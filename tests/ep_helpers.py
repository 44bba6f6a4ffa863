"""Shared by the EmbeddingParallel tests (CPU/gloo with kernel doubles, and 2 GPUs over NCCL): a row-sharded model
and a replicated data-parallel model trained on the same per-rank batches must stay the same model."""
import numpy as np
import torch

CFG_EP = b'''
train_config { train_distribute: EmbeddingParallelStrategy
  optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.05 } } } } }
data_config { batch_size: 64 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "x" input_type: FLOAT }
  input_fields { input_name: "a" input_type: INT64 } input_fields { input_name: "b" input_type: INT64 }
  input_fields { input_name: "c" input_type: INT64 } }
feature_config {
  features { input_names: "x" feature_type: RawFeature embedding_dim: 8 min_val: 0.0 max_val: 4.0 }
  features { input_names: "a" feature_type: IdFeature embedding_dim: 8 hash_bucket_size: 1001 embedding_name: "shared" }
  features { input_names: "b" feature_type: IdFeature embedding_dim: 8 hash_bucket_size: 1001 embedding_name: "shared" }
  features { input_names: "c" feature_type: IdFeature embedding_dim: 8 num_buckets: 37 } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["x", "a", "b", "c"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["x", "a", "b", "c"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [16] } final_dnn { hidden_units: [8] } l2_regularization: 1e-5 }
  embedding_regularization: 1e-5 }
'''


def batch(B, rank, step):
  rng = np.random.default_rng(1000 * rank + step)
  ids = np.concatenate([(rng.zipf(1.3, B) % 5000), (rng.zipf(1.3, B) % 5000), rng.integers(-1, 37, B)]).astype(np.int64)
  dense = rng.uniform(0, 4, (B, 1)).astype(np.float32)
  labels = (rng.uniform(size=B) < 0.3).astype(np.float32)
  return {'sparse_fea': torch.from_numpy(ids), 'dense_fea': torch.from_numpy(dense)}, torch.from_numpy(labels)


def shard_of(full, off, v, rank, world):
  """rows of a table [off, off + v) of the replicated arena that rank owns: row r -> (r mod N, r div N)"""
  return full[off:off + v][rank::world]


def copy_tables(dp_il, ep_il, rank, world):
  """replicated arenas -> this rank's shards (weights and optimizer state)"""
  for dim, a_dp in dp_il.arenas.items():
    a_ep = ep_il.arenas[dim]
    k = a_dp.storage.shape[1] // dim
    for name, (off, _, v) in a_dp.tables.items():
      off_e, local, _ = a_ep.tables[name]
      for j in range(k):   # [w | state0 | state1] column blocks of the interleaved storage
        src = shard_of(a_dp.storage[:, j * dim:(j + 1) * dim], off, v, rank, world)
        a_ep.storage[off_e:off_e + src.shape[0], j * dim:(j + 1) * dim].copy_(src)


def compare(dp_il, ep_il, rank, world, atol):
  worst = 0.0
  for dim, a_dp in dp_il.arenas.items():
    a_ep = ep_il.arenas[dim]
    for name, (off, _, v) in a_dp.tables.items():
      off_e, local, _ = a_ep.tables[name]
      want = shard_of(a_dp.weight, off, v, rank, world)
      got = a_ep.weight[off_e:off_e + want.shape[0]]
      if want.numel():   # (a one-row table has no shard on ranks > 0)
        worst = max(worst, float((want - got).abs().max()))
  assert worst <= atol, 'sharded tables drifted from the replicated ones by %g' % worst
  return worst


def run(make_estimator, dev, rank, world, steps=4, atol=2e-6, lookahead=False, cfg=CFG_EP):
  """make_estimator(config bytes, embedding_parallel) -> EasyRecEstimator on `dev`; cfg: a row-sharded config over
  the inputs of batch()"""
  dp = make_estimator(cfg.replace(b'train_distribute: EmbeddingParallelStrategy', b''), False)
  ep = make_estimator(cfg, None)
  assert ep.embedding_parallel and not dp.embedding_parallel and ep.input_layer.ep
  for dim, a in dp.input_layer.arenas.items():
    assert ep.input_layer.arenas[dim].n_rows < a.n_rows      # (V + N - 1) // N rows per table
  copy_tables(dp.input_layer, ep.input_layer, rank, world)
  ep.model.load_state_dict(dp.model.state_dict())
  ep.trainer.dense_opt.flat_p.copy_(dp.trainer.dense_opt.flat_p)
  losses = []
  batches = []
  for step in range(steps):
    f, l = batch(64, rank, step)
    batches.append(({k: v.to(dev) for k, v in f.items()}, l.to(dev)))
  for step in range(steps):
    f, l = batches[step]
    l_dp, _ = dp.trainer.train_step(f, l)
    # lookahead: the trainer is told the next batch, whose id exchange then runs beside this step
    nxt = batches[step + 1][0] if (lookahead and step + 1 < steps) else None
    l_ep, _ = ep.trainer.train_step(f, l, next_features=nxt)
    losses.append((float(l_dp), float(l_ep)))
    assert abs(float(l_dp) - float(l_ep)) < 1e-5, losses
  worst = compare(dp.input_layer, ep.input_layer, rank, world, atol)
  d = float((dp.trainer.dense_opt.flat_p - ep.trainer.dense_opt.flat_p).abs().max())
  assert d < 1e-5, 'dense parameters differ by %g' % d
  assert losses[-1][0] != losses[0][0]
  ep.input_layer.check_exchange()   # no per-peer block of the fixed-capacity exchange overflowed
  return worst
