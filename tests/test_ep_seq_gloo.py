"""CPU, world 2 and 3 over gloo, kernel doubles: EmbeddingParallel with UN-POOLED HISTORIES - MultiTowerDIN
`seq_att_groups`, in-group `sequence_features`, the `attention` sequence_combiner and the backbone DIN's
`output_seq_and_normal_feature` group.  Every history step is one lookup: er_bucketize_seq (owner, local row; padded
steps ask for nothing) -> K8 -> all-to-alls -> each received row written to its own step's row of the [B*T, sum D]
matrix; backward: local duplicate sums -> owners -> fused update.

The row-sharded model must stay the same model as replicated data parallel on the same per-rank batches (which is the
one-process model of the concatenated batch, tests/test_dp_gloo.py): losses and predictions over several steps within
1e-5, table shards and optimizer slots within 2e-6.  Histories have lengths 0, 1 and T, ids repeat within and across
ranks, and the padded steps of the identity-bucketed histories point at rows no live step reads: those rows stay
bit-unchanged and K8 never requests them."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
B = 12
T_DIN, T_VIEWS = 5, 4
N_LIVE = 20          # live steps of the identity-bucketed histories read rows [0, N_LIVE); padding reads [N_LIVE, 30)

HEAD = b'''
train_config { %s
  optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.05 } } } } }
data_config { batch_size: 12 input_type: DummyInput label_fields: "clk"
  input_fields { input_name: "clk" input_type: FLOAT } input_fields { input_name: "user_id" input_type: INT64 }
  input_fields { input_name: "item_id" input_type: INT64 } input_fields { input_name: "cate_id" input_type: INT64 }
  input_fields { input_name: "price" input_type: FLOAT } input_fields { input_name: "hist_items" input_type: INT64 }
  input_fields { input_name: "hist_cates" input_type: INT64 } input_fields { input_name: "clicks" input_type: INT64 }
  input_fields { input_name: "views" input_type: INT64 } }
feature_config {
  features { input_names: "user_id" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 50 }
  features { input_names: "item_id" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 40 }
  features { input_names: "cate_id" feature_type: IdFeature embedding_dim: 4 num_buckets: 30 }
  features { input_names: "price" feature_type: RawFeature embedding_dim: 4 min_val: 0.0 max_val: 1.0 }
  features { input_names: "hist_items" feature_type: SequenceFeature embedding_dim: 4 hash_bucket_size: 40
             max_seq_len: 5 separator: "|" }
  features { input_names: "hist_cates" feature_type: SequenceFeature embedding_dim: 4 num_buckets: 30 max_seq_len: 5
             separator: "|" }
  features { input_names: "clicks" feature_type: SequenceFeature embedding_dim: 4 num_buckets: 30 max_seq_len: 5
             separator: "|" sequence_combiner { attention {} } }
  features { input_names: "views" feature_type: SequenceFeature embedding_dim: 4 num_buckets: 30 max_seq_len: 4
             separator: "|" } }
'''

# C3's shape (workloads.c3_config_text) with an `attention` combiner in the user group and target attention inside the
# item group: three history launches on one arena (T = 5 for din + clicks, T = 4 for views) beside the id launch
MULTI_TOWER_DIN = HEAD + b'''
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "user" feature_names: ["user_id", "clicks"] wide_deep: DEEP }
  feature_groups { group_name: "item" feature_names: ["item_id", "cate_id", "price"] wide_deep: DEEP
                   sequence_features { group_name: "s" seq_att_map { key: "item_id" hist_seq: "views" }
                                       seq_dnn { hidden_units: [8, 1] } } }
  seq_att_groups { group_name: "din" seq_att_map { key: "item_id" hist_seq: "hist_items" }
                   seq_att_map { key: "cate_id" hist_seq: "hist_cates" } }
  multi_tower { towers { input: "user" dnn { hidden_units: [8] } } towers { input: "item" dnn { hidden_units: [8] } }
                din_towers { input: "din" dnn { hidden_units: [8, 1] } } final_dnn { hidden_units: [4] }
                l2_regularization: 1e-5 }
  embedding_regularization: 1e-5 }
'''

# workloads.c3_backbone_config_text's shape: an output_seq_and_normal_feature group feeding a keras DIN block
BACKBONE_DIN = HEAD + b'''
model_config { model_class: "RankModel"
  feature_groups { group_name: "user" feature_names: ["user_id"] wide_deep: DEEP }
  feature_groups { group_name: "item" feature_names: ["item_id", "cate_id", "price"] wide_deep: DEEP }
  feature_groups { group_name: "seq" feature_names: ["item_id", "cate_id", "hist_items", "hist_cates"] wide_deep: DEEP }
  backbone {
    blocks { name: "user" inputs { feature_group_name: "user" } keras_layer { class_name: "MLP" mlp { hidden_units: [8] } } }
    blocks { name: "item" inputs { feature_group_name: "item" } keras_layer { class_name: "MLP" mlp { hidden_units: [8] } } }
    blocks { name: "seq_input" inputs { feature_group_name: "seq" } input_layer { output_seq_and_normal_feature: true } }
    blocks { name: "din" inputs { block_name: "seq_input" } keras_layer { class_name: "DIN" din {
      attention_dnn { hidden_units: [8, 1] activation: "dice" } need_target_feature: true } } }
    concat_blocks: ["user", "item", "din"]
    top_mlp { hidden_units: [4] } }
  model_params { l2_regularization: 1e-5 }
  embedding_regularization: 1e-5 }
'''

MODELS = {'multi_tower_din': MULTI_TOWER_DIN, 'backbone_din': BACKBONE_DIN}
# identity-bucketed histories: rows >= N_LIVE of their tables are reached only by padded steps
PAD_ONLY = {'multi_tower_din': ('din/hist_cates_embedding', 'clicks_embedding', 'item/views_embedding'),
            'backbone_din': ('hist_cates_embedding',)}


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def batch(rank, step):
  """ids drawn from small ranges (repeats within and across ranks), lengths 0, 1 and T always present, padded steps
  of the identity-bucketed histories pointing at rows [N_LIVE, 30), of the hashed one at ids no live step uses"""
  rng = np.random.default_rng(100 * rank + step)
  ids = np.concatenate([rng.integers(0, 60, B), rng.integers(0, 25, B), rng.integers(0, 30, B)]).astype(np.int64)
  seq = {}
  for name, T, lo, hi in (('hist_items', T_DIN, 0, 25), ('hist_cates', T_DIN, 0, N_LIVE), ('clicks', T_DIN, 0, N_LIVE),
                          ('views', T_VIEWS, 0, N_LIVE)):
    lens = rng.integers(0, T + 1, B).astype(np.int32)
    lens[:3] = [0, 1, T]
    live = rng.integers(lo, hi, (B, T))
    pad = rng.integers(10**6, 10**6 + 50, (B, T)) if name == 'hist_items' else rng.integers(N_LIVE, 30, (B, T))
    h = np.where(np.arange(T)[None, :] < lens[:, None], live, pad).astype(np.int64)
    seq[name] = (torch.from_numpy(h), torch.from_numpy(lens))
  feats = {'sparse_fea': torch.from_numpy(ids), 'dense_fea': torch.from_numpy(rng.uniform(0, 1, (B, 1)).astype(np.float32)),
           'seq_fea': seq}
  return feats, torch.from_numpy((rng.uniform(size=B) < 0.4).astype(np.float32))


def to_dev(feats, labels, dev):
  return ({'sparse_fea': feats['sparse_fea'].to(dev), 'dense_fea': feats['dense_fea'].to(dev),
           'seq_fea': {k: (a.to(dev), b.to(dev)) for k, (a, b) in feats['seq_fea'].items()}}, labels.to(dev))


def compare_storage(dp_il, ep_il, rank, world, atol):
  """every table's shard on this rank - weights and optimizer slots - against the replicated table's rows r = k*N + rank"""
  import ep_helpers
  worst = 0.0
  for dim, a_dp in dp_il.arenas.items():
    a_ep = ep_il.arenas[dim]
    for name, (off, _, v) in a_dp.tables.items():
      off_e, _, _ = a_ep.tables[name]
      want = ep_helpers.shard_of(a_dp.storage, off, v, rank, world)
      if want.numel():
        got = a_ep.storage[off_e:off_e + want.shape[0]]
        worst = max(worst, float((want - got).abs().max()))
  assert worst <= atol, 'sharded tables / optimizer slots drifted from the replicated ones by %g' % worst
  return worst


def pad_only_rows(ep_il, name, rank, world):
  """(arena dim, local rows) of table `name`'s rows >= N_LIVE that this rank owns"""
  for dim, a in ep_il.arenas.items():
    if name in a.tables:
      off_e, _, v = a.tables[name]
      return dim, [off_e + r // world for r in range(N_LIVE, v) if r % world == rank]
  raise KeyError(name)


def check_requests(ep_il, world, model):
  """K8 of every history exchange: no block holds a padded-only row, and counts are the distinct live rows per owner"""
  for dim, subs in ep_il.subcalls.items():
    for sk, sc in subs.items():
      if sc.kind != 'seq':
        continue
      ex = sc.sharded.ex
      rows_l, own = ex.rows_local.cpu().numpy(), ex.owner.cpu().numpy()
      live = rows_l >= 0
      counts = ex.counts.cpu().numpy()
      for o in range(world):
        assert counts[o] == np.unique(rows_l[live & (own == o)]).size
      assert counts[world] == 0
      send = ex.send_rows.cpu().numpy().reshape(world, ex.cap)
      a = ep_il.arenas[dim]
      for name in {slot.table for _, _, slot, _ in sc.items} & set(PAD_ONLY[model]):
        off, local, _ = a.tables[name]
        for o in range(world):
          glob = (send[o][(send[o] >= off) & (send[o] < off + local)] - off) * world + o
          assert (glob < N_LIVE).all(), (name, sorted(set(glob.tolist())))


def _worker(rank, port, ret, world, model, cuda=False):
  """model None: every model; on GPUs each one eager and with the whole step replayed from one CUDA graph"""
  sys.path.insert(0, HERE)
  from test_dp_clip_gloo import _setup
  import torch.distributed as dist
  dev = _setup(rank, port, world, cuda)
  if not cuda:
    import seq_doubles
    seq_doubles.install()   # (_setup installed the other kernel doubles)
  worst = 0.0
  for m in ([model] if model else sorted(MODELS)):
    for graph in ((False, True) if cuda else (False,)):
      worst = max(worst, _run(dev, rank, world, m, cuda, graph))
  ret[rank] = worst
  if cuda:
    dist.barrier()
    os._exit(0)
  dist.destroy_process_group()


def _run(dev, rank, world, model, cuda, graph):
  from easyrec_b200.estimator import EasyRecEstimator
  text = MODELS[model]

  def make(cfg, ep):
    return EasyRecEstimator(cfg, device=dev, seed=5, world_size=world, rank=rank, embedding_parallel=ep,
                            use_cuda_graph=graph and ep is not False)
  dp = make(text % b'', False)
  ep = make(text % b'train_distribute: EmbeddingParallelStrategy', None)
  assert ep.embedding_parallel and ep.input_layer.ep
  kinds = sorted(sc.kind for subs in ep.input_layer.subcalls.values() for sc in subs.values())
  assert kinds == (['seq', 'seq', 'single'] if model == 'multi_tower_din' else ['seq', 'single']), kinds
  import ep_helpers
  ep_helpers.copy_tables(dp.input_layer, ep.input_layer, rank, world)
  ep.model.load_state_dict(dp.model.state_dict())
  ep.trainer.dense_opt.flat_p.copy_(dp.trainer.dense_opt.flat_p)
  pads = [pad_only_rows(ep.input_layer, n, rank, world) for n in PAD_ONLY[model]]
  before = [ep.input_layer.arenas[d].storage[r].clone() for d, r in pads]
  steps = 7 if graph else 4
  losses = []
  for step in range(steps):
    f, l = to_dev(*batch(rank, step), dev)
    l_dp, p_dp = dp.trainer.train_step(f, l)
    l_ep, p_ep = ep.trainer.train_step(f, l)
    losses.append((float(l_dp), float(l_ep)))
    assert abs(float(l_dp) - float(l_ep)) < 1e-5, losses
    assert float((p_dp - p_ep).abs().max()) < 1e-5
    check_requests(ep.input_layer, world, model)
  worst = compare_storage(dp.input_layer, ep.input_layer, rank, world, 5e-6 if cuda else 2e-6)
  for (d, r), b in zip(pads, before):
    assert torch.equal(ep.input_layer.arenas[d].storage[r], b), 'a row only padded steps point at moved'
  d = float((dp.trainer.dense_opt.flat_p - ep.trainer.dense_opt.flat_p).abs().max())
  assert d < 1e-5, d
  assert losses[-1][0] != losses[0][0]
  ep.input_layer.check_exchange()
  if graph:
    assert ep.trainer._graph is not None
  return worst


@pytest.mark.timeout(600)
@pytest.mark.parametrize('model', sorted(MODELS))
@pytest.mark.parametrize('world', [2, 3])
def test_embedding_parallel_over_history_slots_gloo(world, model):
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret, world, model), nprocs=world, join=True)
  assert len(ret) == world


def test_history_table_shared_with_other_features_is_refused_under_embedding_parallel():
  """a table read by history steps and by single-valued slots would need one owner update across two exchanges"""
  from easyrec_b200 import builder
  from easyrec_b200.config import config_util
  text = (MULTI_TOWER_DIN % b'').replace(
      b'embedding_dim: 4 hash_bucket_size: 40 }', b'embedding_dim: 4 hash_bucket_size: 40 embedding_name: "item" }').replace(
      b'hash_bucket_size: 40\n             max_seq_len: 5', b'hash_bucket_size: 40 embedding_name: "item"\n             max_seq_len: 5')
  assert text.count(b'embedding_name: "item"') == 2
  cfg = config_util.get_configs_from_pipeline_file(text)
  with pytest.raises(NotImplementedError, match=r"table\(s\) \['item'\] are read both by history"):
    builder.build_model(cfg, B, 'cpu', world=2, rank=0, shard_tables=True, cpu_generator=torch.Generator().manual_seed(1))
  builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(1))   # (replicated: one table)
  # tf.train.AdamOptimizer's dense decay would run once per exchange of the arena
  adam = (MULTI_TOWER_DIN % b'').replace(b'adagrad_optimizer', b'adam_optimizer')
  with pytest.raises(NotImplementedError, match='adam_optimizer with histories next to other features of embedding_dim 4'):
    builder.build_model(config_util.get_configs_from_pipeline_file(adam), B, 'cpu', world=2, rank=0, shard_tables=True,
                        cpu_generator=torch.Generator().manual_seed(1))
