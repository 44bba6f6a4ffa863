"""GPU: the key-value table kernels (csrc/kv_table.cu) on random and adversarial keys, and key-value tables trained
through InputLayer and the Trainer on the real kernels, checked per key (row numbers are not deterministic)."""
import math

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, builder, kernels as K
from easyrec_b200.trainer import Trainer

import kv_doubles
import test_kv_tables_host as H

pytestmark = pytest.mark.gpu
DEV = 'cuda'
DIM = 8
STD = 0.01 / math.sqrt(DIM)


def _index(capacity):
  n = 16
  while n < 2 * capacity:
    n *= 2
  return (torch.full((n,), _lib.KV_EMPTY, dtype=torch.int64, device=DEV), torch.full((n,), -1, dtype=torch.int64, device=DEV),
          torch.zeros(2, dtype=torch.int64, device=DEV))


def _group_of(keys, n_groups):
  return (kv_doubles._mix(np.asarray(keys, np.int64).astype(np.uint64)) & np.uint64(n_groups - 1)).astype(np.int64)


def _cases():
  rng = np.random.default_rng(0)
  chain = [k for k in range(200000) if _group_of([k], 8)[0] == 3][:60]   # 60 keys of one 16-slot group, 128 slots
  return {
      'random': (4096, rng.integers(0, 2**63 - 1, 30000, dtype=np.int64) % 3000 * 7919),
      'one_key': (64, np.full(8192, 12345, np.int64)),
      'probe_chain': (64, np.repeat(np.array(chain, np.int64), 5)),
      'extremes': (16, np.array([0, 2**63 - 2, -1, 0, 2**63 - 2, 5] * 100, np.int64)),
      'full': (1000, rng.permutation(np.repeat(np.arange(1000, dtype=np.int64) * 31 + 2**40, 7))),
  }


@pytest.mark.parametrize('case', list(_cases()))
def test_find_or_insert_gives_every_distinct_key_one_initialised_row(case):
  capacity, keys_np = _cases()[case]
  ik, ir, stats = _index(capacity)
  weight = torch.full((capacity + 1, 3 * DIM), float('nan'), device=DEV)
  w, s0, s1 = weight[:, :DIM], weight[:, DIM:2 * DIM], weight[:, 2 * DIM:]
  keys = torch.tensor(keys_np, device=DEV)
  rows = torch.empty_like(keys)
  K.kv_find_or_insert(ik, ir, capacity, stats, keys, rows, w, s0, s1, 0.25, 99, STD)
  r = rows.cpu().numpy()
  live = keys_np >= 0
  assert (r[~live] == -1).all()
  distinct = np.unique(keys_np[live])
  assert distinct.size <= capacity
  assert (r[live] >= 0).all() and (r[live] < capacity).all()
  first = {}
  for k, row in zip(keys_np[live].tolist(), r[live].tolist()):
    assert first.setdefault(k, row) == row, 'key %d got two rows' % k
  assert len(set(first.values())) == distinct.size, 'two keys share a row'
  assert stats.cpu().tolist() == [distinct.size, 0]
  # find agrees with insert, and a second insert of the same keys claims nothing
  found = torch.empty_like(keys)
  K.kv_find(ik, ir, keys, capacity, found)
  assert np.array_equal(found.cpu().numpy(), r)
  K.kv_find_or_insert(ik, ir, capacity, stats, keys, found, w, s0, s1, 0.25, 99, STD)
  assert np.array_equal(found.cpu().numpy(), r) and stats.cpu().tolist() == [distinct.size, 0]
  # rows hold the generator's values for their key, the state its initial values
  ks = np.array(sorted(first), np.int64)
  rr = torch.tensor([first[k] for k in ks.tolist()], device=DEV)
  np.testing.assert_allclose(w[rr].cpu().numpy(), kv_doubles.init_values(99, ks, DIM, STD), rtol=2e-7, atol=1e-12)
  assert torch.all(s0[rr] == 0.25) and torch.all(s1[rr] == 0)
  # every key the index holds is one of ours
  held = ik.cpu().numpy()
  assert sorted(held[held != _lib.KV_EMPTY].tolist()) == ks.tolist()


def test_keys_beyond_capacity_are_dropped_and_counted():
  capacity = 100
  ik, ir, stats = _index(capacity)
  weight = torch.zeros(capacity + 1, DIM, device=DEV)
  keys = torch.arange(150, dtype=torch.int64, device=DEV) * 3
  rows = torch.empty_like(keys)
  K.kv_find_or_insert(ik, ir, capacity, stats, keys, rows, weight, None, None, 0.0, 1, STD)
  r = rows.cpu().numpy()
  n, dropped = stats.cpu().tolist()
  assert n >= capacity and dropped == (r < 0).sum() and dropped >= 50
  kept = r[r >= 0]
  assert kept.size == capacity and np.unique(kept).size == capacity


def test_bulk_insert_rebuilds_an_index_that_finds_the_given_rows():
  ik, ir, stats = _index(5000)
  keys = torch.unique(torch.randint(0, 1 << 62, (6000,), device=DEV))[:5000]
  keys = keys[torch.randperm(keys.numel(), device=DEV)]
  given = torch.randperm(keys.numel(), device=DEV)
  K.kv_insert_rows(ik, ir, keys, given, stats)
  assert int(stats[1]) == 0
  probe = torch.cat([keys, torch.tensor([-1, (1 << 62) + 7], device=DEV)])
  found = torch.empty_like(probe)
  K.kv_find(ik, ir, probe, 5000, found)
  f = found.cpu()
  assert torch.equal(f[:-2], given.cpu()) and f[-2] == -1 and f[-1] == 5000
  # a repeated key is refused and counted
  K.kv_insert_rows(ik, ir, keys[:3], given[:3], stats)
  assert int(stats[1]) == 3


@pytest.mark.parametrize('kind,opt', [('adagrad', _lib.OPT_ADAGRAD), ('lazy_adam', _lib.OPT_LAZY_ADAM),
                                      ('adam', _lib.OPT_ADAM_ROWS)])
def test_three_steps_on_the_kernels_match_the_float64_restatement(kind, opt):
  il = H.make_layer(opt, device=DEV)
  rng = np.random.default_rng(3)
  steps = []
  for t in range(3):
    feats, batch = H.make_batch(rng, device=DEV)
    R = torch.tensor(rng.integers(-3, 4, (H.B, 3 * H.DIM)) / 4.0, dtype=torch.float32, device=DEV)
    steps.append((batch, R))
    H.train_step(il, feats, R, 0.05, t)
  ref = H.restate(steps, 'adagrad' if kind == 'adagrad' else 'adam')
  for table in ref:
    got = H.per_key(il, table)
    assert set(got) == set(ref[table]) and il.kv_sizes()[table] == len(ref[table])
    for k, (w, s0, s1) in ref[table].items():
      np.testing.assert_allclose(got[k][0], w, atol=1e-6, rtol=0)
      np.testing.assert_allclose(got[k][1], s0, atol=1e-6, rtol=0)
  il.check_kv()


def test_evaluation_on_unseen_keys_reads_zeros_on_the_kernels():
  il = H.make_layer(_lib.OPT_ADAGRAD, device=DEV)
  feats, _ = H.make_batch(np.random.default_rng(5), device=DEV, item_pool=4)
  H.train_step(il, feats, torch.ones(H.B, 3 * H.DIM, device=DEV), 0.05, 0)
  sizes = il.kv_sizes()
  ids = feats['sparse_fea'].clone()
  ids[H.B:H.B + 2] = torch.tensor([987654321, 987654322], device=DEV)
  with torch.no_grad():
    concat, _ = il.lookup({'sparse_fea': ids, 'tag_fea': feats['tag_fea']})['all']
  il.discard_pending()
  assert il.kv_sizes() == sizes and torch.all(concat[:2, H.DIM:2 * H.DIM] == 0)


def test_overflow_raises_naming_the_table_on_the_kernels():
  il = H.make_layer(_lib.OPT_ADAGRAD, device=DEV, capacity=4)
  ids = torch.cat([torch.zeros(H.B, dtype=torch.int64), torch.arange(H.B)]).to(DEV)
  feats = {'sparse_fea': ids, 'tag_fea': {'tags': (torch.zeros(0, dtype=torch.int64, device=DEV),
                                                   torch.zeros(H.B, dtype=torch.int32, device=DEV), None)}}
  H.train_step(il, feats, torch.ones(H.B, 3 * H.DIM, device=DEV), 0.05, 0)
  with pytest.raises(_lib.ErError, match='item_embedding.*max_capacity 4'):
    il.check_kv()


def _batches(n):
  rng = np.random.default_rng(21)
  out = []
  for _ in range(n):
    ids = np.concatenate([rng.integers(0, 60, 8), rng.integers(0, 40, 8) * 1000003])
    tags = rng.integers(0, 15, 16)
    out.append(({'sparse_fea': torch.tensor(ids, device=DEV),
                 'tag_fea': {'tags': (torch.tensor(tags, device=DEV), torch.full((8,), 2, dtype=torch.int32, device=DEV),
                                      None)}},
                torch.tensor(rng.integers(0, 2, 8), dtype=torch.float32, device=DEV)))
  return out


def _train(graph, batches):
  torch.manual_seed(0)
  cfg = H.config(item_ev='ev_params { max_capacity: 1000 }', tag_ev='ev_params { max_capacity: 100 }')
  il, model, _ = builder.build_model(cfg, 8, DEV, cpu_generator=torch.Generator().manual_seed(0))
  tr = Trainer(model, il, 'adagrad', lr=0.05, use_cuda_graph=graph)
  for feats, labels in batches:
    tr.train_step(feats, labels)
  torch.cuda.synchronize()
  out = {}
  for a in il.arenas.values():
    if a.kv is not None:
      keys, rows = a.kv.items()
      st = a.storage.cpu()
      out[a.kv.name] = {k: st[r].numpy().tobytes() for k, r in zip(keys.tolist(), rows.tolist())}
  return out


def test_the_same_batches_train_bit_identical_rows_per_key_eager_and_graph_replayed():
  batches = _batches(6)
  a, b, g = _train(False, batches), _train(False, batches), _train(True, batches)
  assert set(a) == {'iid_embedding', 'iid_embedding_wide', 'tags_embedding'}
  assert a == b
  assert g == a


def test_an_owner_indexes_the_global_keys_of_the_local_keys_it_receives():
  """row-sharded: the owner of rank r of N passes key div N; the index holds and initialises the global key"""
  n, r, capacity = 3, 1, 256
  ik, ir, stats = _index(capacity)
  weight = torch.zeros(capacity + 1, DIM, device=DEV)
  glob = np.array([1, 4, 7, 2**63 - 2 - ((2**63 - 2 - 1) % 3), 1000000000000000003 * 3 + 1], np.int64)
  assert (glob % n == r).all()
  local = torch.tensor(np.append(glob // n, -1), device=DEV)
  rows = torch.empty_like(local)
  K.kv_find_or_insert(ik, ir, capacity, stats, local, rows, weight, None, None, 0.0, 17, 0.0025,
                      init_truncated=False, shard_n=n, shard_rank=r)
  got = rows.cpu().numpy()
  assert got[-1] == -1 and np.unique(got[:-1]).size == glob.size
  held = ik.cpu().numpy()
  assert sorted(held[held != _lib.KV_EMPTY].tolist()) == sorted(glob.tolist())
  np.testing.assert_allclose(weight[rows[:-1]].cpu().numpy(), kv_doubles.init_values(17, glob, DIM, 0.0025, False),
                             rtol=2e-7, atol=1e-12)
  found = torch.empty_like(local)
  K.kv_find(ik, ir, local, capacity, found, shard_n=n, shard_rank=r)
  assert np.array_equal(found.cpu().numpy(), got)
