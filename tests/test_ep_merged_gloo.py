"""CPU, world 2 and 3 over gloo, kernel doubles: EmbeddingParallel with ONE exchange per arena for its single-valued and
multi-valued (CSR) launches - an IdFeature and a kv-weighted TagFeature reading one table, a `sum` TagFeature, a raw
projection, and a wide group.  With the kv-weighted tag feature's combiner `mean` the wide group's `sum` twin prunes
other lookups (K1 drops a weighted mean lookup whose weight is not > 0, keeps a sum one): the deep and the wide arena
get an exchange each.  With `sum` both arenas have the same combined row plan and share one exchange.

K1 of each launch writes its own range of the exchange's lookup arrays, one K8 runs over all of them, three
all-to-alls per step and exchange (ids, rows, gradients), one owner-side row update and one Adam decay per arena.  The
row-sharded model must stay the same model as replicated data parallel on the same per-rank batches: losses and
predictions within 1e-5, table shards and optimizer slots within 2e-6, with adagrad, lazy Adam and
tf.train.AdamOptimizer, with and without the next batch's id exchange prefetched."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
B = 12
STEPS = 4

CFG = b'''
train_config { %s
  optimizer_config { %s { learning_rate { constant_learning_rate { learning_rate: 0.05 } } } } }
data_config { batch_size: 12 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "u" input_type: INT64 }
  input_fields { input_name: "t1" input_type: STRING } input_fields { input_name: "t2" input_type: STRING }
  input_fields { input_name: "x" input_type: FLOAT } }
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 4 num_buckets: 9 %s }
  features { input_names: "t1" feature_type: TagFeature embedding_dim: 4 num_buckets: 9 %s separator: "|"
             kv_separator: ":" combiner: "%s" }
  features { input_names: "t2" feature_type: TagFeature embedding_dim: 4 hash_bucket_size: 13 separator: "|" combiner: "sum" }
  features { input_names: "x" feature_type: RawFeature embedding_dim: 4 min_val: 0.0 max_val: 2.0 } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["u", "t1", "t2", "x"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["u", "t1", "t2", "x"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [8] use_bn: false } final_dnn { hidden_units: [4] use_bn: false } l2_regularization: 1e-5 }
  embedding_regularization: 1e-5 }
'''
EP = b'train_distribute: EmbeddingParallelStrategy'
SHARED = b'embedding_name: "e"'
OPTS = ('adagrad_optimizer', 'lazy_adam_optimizer', 'adam_optimizer')


# the kv-weighted tag feature's combiner -> exchanges of the deep and the wide arena
EXCHANGES = {'mean': 2, 'sum': 1}


def config(ep, opt, shared=True, comb='mean'):
  e = SHARED if shared else b''
  return CFG % (EP if ep else b'', opt.encode(), e, e, comb.encode())


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _lines(seed, odd_weights=False):
  """odd_weights: t1's kv weights include 0 and negative ones (a mean lookup K1 prunes, a sum lookup it keeps)"""
  rng = np.random.default_rng(seed)
  out = []
  for _ in range(B):
    t1 = '|'.join('%d:%.2f' % (rng.integers(0, 9), rng.choice([0.0, -0.5, rng.uniform(0.2, 2.0)]) if odd_weights else
                               rng.uniform(0.2, 2.0)) for _ in range(rng.integers(0, 4)))
    t2 = '|'.join('w%d' % rng.integers(0, 30) for _ in range(rng.integers(0, 5)))
    out.append('%d,%d,%s,%s,%.3f' % (rng.integers(0, 2), rng.integers(0, 9), t1, t2, rng.uniform(0, 2)))
  return out


def batches(rank, tmp, dev, n=STEPS, odd_weights=False):
  from easyrec_b200.config import config_util
  from easyrec_b200.estimator import EasyRecEstimator
  from easyrec_b200.input import readers
  cfg_text = config(False, 'adagrad_optimizer')
  il = EasyRecEstimator(cfg_text, device='cpu', seed=1).input_layer
  cfg = config_util.get_configs_from_pipeline_file(cfg_text)
  out = []
  for step in range(n):
    path = os.path.join(tmp, 'r%d_s%d.csv' % (rank, step))
    with open(path, 'w') as f:
      f.write('\n'.join(_lines(1000 * rank + step, odd_weights)) + '\n')
    (feats, labels), = list(readers.CSVInput(cfg, il, path))
    out.append(readers.to_device(feats, labels, dev))
  return out


def compare_storage(dp_il, ep_il, rank, world):
  """every table's shard on this rank - weights and optimizer slots - against the replicated rows r = k*N + rank"""
  import ep_helpers
  worst = 0.0
  for dim, a_dp in dp_il.arenas.items():
    a_ep = ep_il.arenas[dim]
    for name, (off, _, v) in a_dp.tables.items():
      off_e, _, _ = a_ep.tables[name]
      want = ep_helpers.shard_of(a_dp.storage, off, v, rank, world)
      if want.numel():
        worst = max(worst, float((want - a_ep.storage[off_e:off_e + want.shape[0]]).abs().max()))
  return worst


def check_structure(il, world, n_exchanges):
  """one exchange per combined row plan of the arenas' non-history launches (each arena's single-valued and tag launch
  in one); K8's counts are the distinct requested (owner, row) pairs over every launch's range; a CSR launch's padding
  is never requested"""
  exchanges = il._exchanges()
  assert len(exchanges) == n_exchanges, len(exchanges)
  assert sum(len(ex.heads) for ex in exchanges) == 2
  for ex in exchanges:
    assert sorted(m.csr for m in ex.launches) == [False, True]
    rows, own, pos = ex.rows_local.cpu().numpy(), ex.owner.cpu().numpy(), ex.pos.cpu().numpy()
    counts = ex.counts.cpu().numpy()
    live = rows >= 0
    for o in range(world):
      assert counts[o] == np.unique(rows[live & (own == o)]).size, (o, counts)
    assert counts[world] == 0
    for m, (_, row_ptr, _) in zip(ex.launches, il._ex_inputs[id(ex)]):
      if m.csr:
        total = int(row_ptr[-1])
        assert 0 < total < m.L
        assert (rows[m.lo + total:m.lo + m.L] == -1).all() and (pos[m.lo + total:m.lo + m.L] == -1).all()


def _run(dev, rank, world, tmp, opt, lookahead, shared, comb, count):
  from easyrec_b200.estimator import EasyRecEstimator
  import ep_helpers

  def make(ep):
    return EasyRecEstimator(config(ep, opt, shared, comb), device=dev, seed=5, world_size=world, rank=rank,
                            embedding_parallel=None if ep else False)
  dp, ep = make(False), make(True)
  assert ep.embedding_parallel and ep.input_layer.ep
  kinds = sorted(sc.kind for subs in ep.input_layer.subcalls.values() for sc in subs.values())
  assert kinds == ['single', 'single', 'tag', 'tag'], kinds
  ep_helpers.copy_tables(dp.input_layer, ep.input_layer, rank, world)
  ep.model.load_state_dict(dp.model.state_dict())
  ep.trainer.dense_opt.flat_p.copy_(dp.trainer.dense_opt.flat_p)
  data = batches(rank, tmp, dev)
  losses = []
  n_a2a = 0
  for step in range(STEPS):
    f, l = data[step]
    l_dp, p_dp = dp.trainer.train_step(f, l)
    nxt = data[step + 1][0] if lookahead and step + 1 < STEPS else None
    count[0] = 0
    l_ep, p_ep = ep.trainer.train_step(f, l, next_features=nxt)
    n_a2a += count[0]
    if not lookahead:
      assert count[0] == 3 * EXCHANGES[comb], count[0]     # ids, rows, gradients
      check_structure(ep.input_layer, world, EXCHANGES[comb])
    elif nxt is not None:
      assert ep.input_layer.prefetch_ready()
    losses.append((float(l_dp), float(l_ep)))
    assert abs(float(l_dp) - float(l_ep)) < 1e-5, losses
    assert float((p_dp - p_ep).abs().max()) < 1e-5
  assert n_a2a == 3 * EXCHANGES[comb] * STEPS, n_a2a       # (a prefetched id exchange moves to the step before)
  worst = compare_storage(dp.input_layer, ep.input_layer, rank, world)
  assert worst <= 2e-6, 'sharded tables / optimizer slots drifted from the replicated ones by %g (%s)' % (worst, opt)
  d = float((dp.trainer.dense_opt.flat_p - ep.trainer.dense_opt.flat_p).abs().max())
  assert d < 1e-5, d
  assert losses[-1][0] != losses[0][0]
  ep.input_layer.check_exchange()
  return worst


def _counting_all_to_all(count):
  import torch.distributed as dist
  inner = dist.all_to_all_single

  def all_to_all_single(*a, **k):
    count[0] += 1
    return inner(*a, **k)
  dist.all_to_all_single = all_to_all_single


def _worker(rank, port, ret, world, tmp, runs, cuda=False):
  sys.path.insert(0, HERE)
  from test_dp_clip_gloo import _setup
  import torch.distributed as dist
  dev = _setup(rank, port, world, cuda)
  count = [0]
  _counting_all_to_all(count)
  worst = 0.0
  for opt, lookahead, shared, comb in runs:
    worst = max(worst, _run(dev, rank, world, tmp, opt, lookahead, shared, comb, count))
  ret[rank] = worst
  if cuda:
    dist.barrier()
    os._exit(0)
  dist.destroy_process_group()


def _spawn(world, tmp, runs):
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret, world, str(tmp), runs), nprocs=world, join=True)
  assert len(ret) == world
  return dict(ret)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('world', [2, 3])
def test_id_and_tag_features_sharing_a_table_row_sharded_equal_replicated_gloo(world, tmp_path):
  _spawn(world, tmp_path, [(opt, lookahead, True, comb) for comb in EXCHANGES for opt in OPTS
                           for lookahead in (False, True)])


@pytest.mark.timeout(600)
@pytest.mark.parametrize('world', [2, 3])
def test_adam_decays_each_row_once_over_disjoint_id_and_tag_tables_gloo(world, tmp_path):
  """tf.train.AdamOptimizer's dense decay of an arena whose id and tag tables are disjoint but share the dim: one
  decay per row and step, as in the replicated model (two exchanges on the arena decayed every row twice)"""
  _spawn(world, tmp_path, [('adam_optimizer', lookahead, False, 'mean') for lookahead in (False, True)])


def _mismatch_worker(rank, port, ret, world, tmp):
  sys.path.insert(0, HERE)
  from test_dp_clip_gloo import _setup
  import torch.distributed as dist
  from easyrec_b200 import _lib
  from easyrec_b200.estimator import EasyRecEstimator
  dev = _setup(rank, port, world, False)
  ep = EasyRecEstimator(config(True, 'adagrad_optimizer'), device=dev, seed=5, world_size=world, rank=rank)
  data = batches(rank, tmp, dev, n=3)
  ep.trainer.train_step(*data[0], next_features=data[1][0])
  ep.trainer.train_step(*data[1])
  ep.input_layer.check_exchange()            # the batch that arrived is the one prefetched

  def altered(feats, what):
    """the same batch with one tag id, or one tag length, changed on every rank"""
    ids, lens, w = feats['tag_fea']['t1']
    ids, lens = ids.clone(), lens.clone()
    if what == 'ids':
      ids[0] = (ids[0] + 1) % 9
    else:
      j = int(np.nonzero(lens.numpy())[0][0])
      lens[j] -= 1
      lens[(j + 1) % B] += 1
    return dict(feats, tag_fea=dict(feats['tag_fea'], t1=(ids, lens, w)))
  raised = []
  for what in ('ids', 'lens'):
    f, l = data[2]
    ep.trainer.train_step(*data[0], next_features=f)
    ep.trainer.train_step(altered(f, what), l)
    try:
      ep.input_layer.check_exchange()
    except _lib.ErError as e:
      assert 'prefetched batch differed' in str(e)
      raised.append(what)
    ep.input_layer.check_exchange()          # (the check resets the counter)
  ret[rank] = raised
  dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_prefetched_exchange_refuses_a_batch_with_other_tag_ids_or_lengths_gloo(tmp_path):
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_mismatch_worker, args=(_free_port(), ret, 2, str(tmp_path)), nprocs=2, join=True)
  assert dict(ret) == {0: ['ids', 'lens'], 1: ['ids', 'lens']}, dict(ret)
