"""CPU, world 2 and 3 over gloo, kernel doubles (tests/kv_doubles.py for the key-value kernels): key-value tables
(ev_params) trained row-sharded under EmbeddingParallelStrategy.  K1 gives owner = key mod N and key div N, K8 groups and
exchanges the keys, and the owner turns what it received into rows of its own pool.  A model with a key-value item table
(deep and wide) and a key-value tag table next to a static table must train as the same model as one rank on the
concatenated batch: losses and predictions within 1e-5, rows and optimizer slots within 2e-6, compared per key.  The
`.key` / `.val` parts the ranks write restore at world 1 and 3 to the same lookups."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
B = 6

CFG = b'''
train_config { train_distribute: EmbeddingParallelStrategy
  optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.05 } } } } }
data_config { batch_size: 6 input_type: CSVInput label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "u" input_type: INT64 }
  input_fields { input_name: "iid" input_type: INT64 } input_fields { input_name: "tags" input_type: STRING } }
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 23 }
  features { input_names: "iid" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 1000 ev_params { max_capacity: 200 } }
  features { input_names: "tags" feature_type: TagFeature embedding_dim: 4 num_buckets: 40 separator: "|"
             ev_params { max_capacity: 100 } } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["u", "iid", "tags"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["u", "iid"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [8] use_bn: false } final_dnn { hidden_units: [4] use_bn: false } } }
'''


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def batch(rank, step):
  rng = np.random.default_rng(100 * rank + step)
  ids = np.concatenate([rng.integers(0, 50, B), rng.integers(0, 30, B) * 1000003]).astype(np.int64)
  lens = rng.integers(0, 4, B).astype(np.int32)
  tags = rng.integers(0, 40, int(lens.sum())).astype(np.int64)
  labels = rng.integers(0, 2, B).astype(np.float32)
  return ids, tags, lens, labels


def feats(ids, tags, lens, dev):
  return {'sparse_fea': torch.from_numpy(ids).to(dev),
          'tag_fea': {'tags': (torch.from_numpy(tags).to(dev), torch.from_numpy(lens).to(dev), None)}}


def concatenated(world, step):
  parts = [batch(r, step) for r in range(world)]
  ids = np.concatenate([np.concatenate([p[0][f * B:(f + 1) * B] for p in parts]) for f in range(2)])
  return (ids, np.concatenate([p[1] for p in parts]), np.concatenate([p[2] for p in parts]),
          np.concatenate([p[3] for p in parts]))


def kv_rows(il):
  """{table: {global key: [w | state] row}}"""
  out = {}
  for a in il.arenas.values():
    if a.kv is not None:
      keys, rows = a.kv.items()
      out[a.kv.name] = {k: a.storage[r].detach().cpu().numpy().copy() for k, r in zip(keys.tolist(), rows.tolist())}
  return out


def _worker(rank, port, ret, world, tmp, cuda=False):
  """cuda: NCCL and the real kernels on cuda:rank (tests/test_gpu_dp_extra.py); else gloo and the kernel doubles"""
  sys.path.insert(0, HERE)
  from test_dp_clip_gloo import _setup
  dev = _setup(rank, port, world, cuda)
  if not cuda:
    import kv_doubles
    kv_doubles.install()
  from easyrec_b200 import checkpoint
  from easyrec_b200.estimator import EasyRecEstimator
  ep = EasyRecEstimator(CFG, device=dev, seed=5, world_size=world, rank=rank, embedding_parallel=None)
  ref = EasyRecEstimator(CFG, device=dev, seed=5, world_size=1, rank=0, batch_size=B * world)
  assert ep.input_layer.ep and not ref.input_layer.ep
  kv_keys = [k for k in ep.input_layer.arenas if isinstance(k, tuple)]
  assert sorted(kv_keys) == [(1, 'iid_embedding_wide'), (4, 'iid_embedding'), (4, 'tags_embedding')]
  # the static tables: this rank's shard of the reference's rows; the dense parameters: the reference's
  for dim, a in ref.input_layer.arenas.items():
    if isinstance(dim, int):
      for name, (off, _, v) in a.tables.items():
        off_e = ep.input_layer.arenas[dim].tables[name][0]
        src = a.storage[off:off + v][rank::world]
        ep.input_layer.arenas[dim].storage[off_e:off_e + src.shape[0]].copy_(src)
  ep.model.load_state_dict(ref.model.state_dict())
  ep.trainer.dense_opt.flat_p.copy_(ref.trainer.dense_opt.flat_p)
  for step in range(4):
    ids, tags, lens, labels = batch(rank, step)
    l_ep, p_ep = ep.trainer.train_step(feats(ids, tags, lens, dev), torch.from_numpy(labels).to(dev))
    cids, ctags, clens, clabels = concatenated(world, step)
    l_ref, p_ref = ref.trainer.train_step(feats(cids, ctags, clens, dev), torch.from_numpy(clabels).to(dev))
    assert float((p_ep - p_ref[rank * B:(rank + 1) * B]).abs().max()) < 1e-5, (step, p_ep, p_ref)
    mean = torch.tensor([float(l_ep)], device=dev)
    dist.all_reduce(mean)
    assert abs(float(mean) / world - float(l_ref)) < 1e-5, (step, float(mean) / world, float(l_ref))
  ep.input_layer.check_exchange()
  ref.input_layer.check_kv()
  mine, want = kv_rows(ep.input_layer), kv_rows(ref.input_layer)
  worst = 0.0
  for table, rows in want.items():
    got = mine[table]
    assert all(k % world == rank for k in got), table
    assert set(got) == {k for k in rows if k % world == rank}, table
    for k, v in got.items():
      worst = max(worst, float(np.abs(v - rows[k]).max()))
  assert worst <= 2e-6, worst
  for a in ep.input_layer.arenas.values():
    if a.kv is not None:
      checkpoint.save_kv_arena(a, os.path.join(tmp, 'model.ckpt-4'))
  if rank == 0:
    ret['ref'] = want
  ret[rank] = worst
  dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize('world', [2, 3])
def test_key_value_tables_row_sharded_train_as_one_rank_on_the_concatenated_batch_gloo(world, tmp_path):
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret, world, str(tmp_path)), nprocs=world, join=True)
  assert len(ret) == world + 1
  if world != 2:
    return
  # the parts written at world 2: part r holds exactly the keys with key % 2 == r, in the reference's layout
  from easyrec_b200 import _lib, checkpoint, embedding as E
  import kv_doubles
  ck = str(tmp_path / 'model.ckpt-4')
  want = ret['ref']
  var = 'input_layer/iid_embedding/embedding_weights:0'
  for r in range(2):
    keys = np.fromfile(checkpoint.kv_part_path(ck, var, r, 'key'), np.int64)
    assert sorted(keys.tolist()) == sorted(k for k in want['iid_embedding'] if k % 2 == r)
    vals = np.fromfile(checkpoint.kv_part_path(ck, var, r, 'val'), np.float32).reshape(-1, 4)
    for k, v in zip(keys.tolist(), vals):
      np.testing.assert_allclose(v, want['iid_embedding'][k][:4], atol=2e-6, rtol=0)   # (trained at world 2)
  # restore at world 1 and 3: every key's lookup (on its owner, by key div N) reads the trained row and its slot
  kv_doubles.install()
  probe = np.array(sorted(want['iid_embedding']) + [123456789], np.int64)
  for n in (1, 3):
    for r in range(n):
      a = E.Arena(4, 'cpu', n, r)
      a.add_table('iid_embedding', 201, local_rows=201)
      a.kv = E.KvTable('iid_embedding', a, 200, 5, embedding_parallel=True)
      a.materialize(_lib.OPT_ADAGRAD, init_fn=lambda w: w.zero_())
      checkpoint.restore_kv_arena(a, ck)
      mine = probe[probe % n == r]
      rows = torch.empty(mine.size, dtype=torch.int64)
      a.kv.lookup(torch.from_numpy(mine // n), rows, train=False)
      for k, row in zip(mine.tolist(), rows.tolist()):
        got = a.storage[row].numpy()
        if k in want['iid_embedding']:
          np.testing.assert_allclose(got, want['iid_embedding'][k], atol=2e-6, rtol=0)
        else:   # a key no rank trained: the zero row
          assert not got[:4].any()
