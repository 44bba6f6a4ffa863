"""GPU: key-value tables (ev_params) on the kernels against exact integer and float64 references.

  K1 at KV_BUCKETS        farm-decimal, mod and identity at num_buckets 2^63 - 1 x shard_n 1/2/3/8/100, single-valued and
                          CSR (cap below and at the total), weighted with a mean slot so that pruned lookups drop; ids
                          0, +-1, -2, 2^63 - 2, 2^63 - 1, INT64_MIN(+1), 17..20-character decimals and ids whose
                          fingerprint is >= 2^63 - 1.  Reference: python integers.
  K8 with 63-bit rows     rows = key div N over [0, 2^63 - 2] for world 1/2/3/8/64/65/200 x n 31/257/212992, with rows that
                          collide under the old `owner << 48 | row` packing, rows that differ only above bit 33, one row
                          with several owners and a warp of one key; caps that fit exactly and one row short.  The checker
                          keys on exact (row, owner) pairs.
  the index kernels       the one-group and two-group index filled past its slots, a probe chain that wraps from the
                          last group to group 0, capacity 2^20 / 2^22 filled by millions of Zipf lookups, dims 1 to 300
                          on interleaved and separate row layouts, the initial-value distribution against scipy's
                          truncated normal and normal, insertion-order independence, and KvTable.load then insert.
  InputLayer              three steps of every row optimizer per key against float64; the emit-form sparse norm of
                          gradient_clipping_by_norm over virtual rows, with and without key-value tables; save and
                          restore (torch checkpoint and embedding parts) then train, bit-identical to an uninterrupted run.
  row-sharded owner chain K1 (shard_n N) -> K8 -> the id all-to-all as a permutation -> kv_find_or_insert on each owner ->
                          the owner's K2 gather -> the requester's pooling K2 -> K7 sums -> the owner's K7 at 1/N, for
                          N = 2 and 3 ranks simulated in one process, against one-rank float64.

The restatements that need no GPU are run against the host doubles in tests/test_kv_tables_host.py."""
import collections
import math
import os

import numpy as np
import pytest
import scipy.stats
import torch

from easyrec_b200 import _lib, checkpoint, embedding as E, input_layer as IL, kernels as K

import kv_doubles
import test_kv_tables_host as H
from test_gpu_lookup_f64 import S32, S64, _guarded, _guards, _weights, L
from easyrec_b200.kernels import _p, _stream

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
KVB = _lib.KV_BUCKETS
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
FARM, MOD, IDENT = _lib.BUCKET_FARM_DECIMAL, _lib.BUCKET_MOD, _lib.BUCKET_IDENTITY
SUM, MEAN = _lib.COMBINER_SUM, _lib.COMBINER_MEAN
NAN_BITS = 0x7FC0DEAD          # the NaN every untouched float of a row buffer holds, compared bit for bit


# ---- K1 at KV_BUCKETS -------------------------------------------------------------------------------------------------
def k1_kv_ref(ids, mode, shard_n, weights=None, combiners=None):
  """K1's rule at num_buckets 2^63 - 1 in python integers -> (rows, owner) lists: the key (fingerprint mod, floored mod
  or identity), then key div N and key mod N; a mean lookup whose weight is not > 0 is dropped (-1, -1)"""
  rows, own = [], []
  for i, v in enumerate(int(x) for x in ids):
    drop = False
    if mode == FARM:
      k = _lib.fingerprint64(str(v)) % KVB
    elif mode == MOD:
      k = v % KVB
    else:
      drop = v == -1
      k = 0 if v < 0 or v >= KVB else v
    if weights is not None and combiners[i] != SUM and not (float(weights[i]) > 0):
      drop = True
    if drop:
      rows.append(-1)
      own.append(-1)
    else:
      rows.append(k // shard_n if shard_n > 1 else k)
      own.append(k % shard_n if shard_n > 1 else 0)
  return rows, own


def kv_edge_ids(rng, n):
  """the edges of the int64 range, 17..20-character decimals, ids whose fingerprint is >= 2^63 - 1, then random"""
  e = [0, 1, -1, -2, 2 ** 63 - 2, I64_MAX, I64_MIN, I64_MIN + 1, 10 ** 16, 10 ** 17 - 1, 10 ** 18, 10 ** 18 + 12345,
       -10 ** 15, -10 ** 16, -10 ** 17, -10 ** 18, I64_MIN + 10 ** 18]
  wide = rng.integers(10 ** 16, I64_MAX, 40, dtype=np.int64).tolist() + (-rng.integers(10 ** 15, I64_MAX, 40,
                                                                                        dtype=np.int64)).tolist()
  high = [v for v in rng.integers(I64_MIN, I64_MAX, 200, dtype=np.int64).tolist()
          if _lib.fingerprint64(str(v)) >= KVB][:30]
  ids = np.array(e + wide + high + rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64).tolist(), np.int64)
  assert len(high) == 30 and all(len(str(v)) >= 17 for v in wide) and any(len(str(v)) == 20 for v in wide)
  return rng.permutation(np.concatenate([ids, ids[:len(e)]]))


def _k1_slots(mode, shard_n, B, T):
  """two slots at KV_BUCKETS: B single lookups pooled by sum, B*T by mean"""
  recs = [dict(num_buckets=KVB, row_offset=0, seg_begin=0, n_seg=B, bucket_mode=mode, combiner=SUM, out_buf=0,
               out_stride=64, out_col=0, shard_n=shard_n),
          dict(num_buckets=KVB, row_offset=0, seg_begin=B, n_seg=B * T, bucket_mode=mode, combiner=MEAN, out_buf=0,
               out_stride=64, out_col=0, shard_n=shard_n)]
  return K.make_slots(recs)


def _k1_call(ids, w, seg_ids, row_ptr, n_seg, cap, sl, alloc):
  sd = K.slots_to_device(sl, DEV)
  # (the device copies stay referenced until the call has run: a freed one could be handed to the next)
  t_ids, t_w, t_sid, t_rp = (None if a is None else torch.from_numpy(a.astype(dt)).to(DEV)
                             for a, dt in ((ids, np.int64), (w, np.float32), (seg_ids, np.int32), (row_ptr, np.int32)))
  rb, rows = _guarded(alloc, torch.int64, S64)
  ob, own = _guarded(alloc, torch.int32, S32)
  args = (_p(t_sid), _p(t_rp), n_seg, cap, _p(sd), len(sl), _p(rows), _p(own), _stream())
  if w is None:
    st = L().er_bucketize(_p(t_ids), *args)
  else:
    st = L().er_bucketize_weighted(_p(t_ids), _p(t_w), *args)
  _lib.check(st, 'er_bucketize')
  _guards(rb, S64, 'rows')
  _guards(ob, S32, 'owner')
  return rows.cpu().numpy().tolist(), own.cpu().numpy().tolist()


@pytest.mark.parametrize('weighted', [False, True], ids=['unweighted', 'weighted'])
@pytest.mark.parametrize('shard_n', [1, 2, 3, 8, 100])
@pytest.mark.parametrize('mode', [FARM, MOD, IDENT], ids=['farm', 'mod', 'identity'])
def test_k1_at_kv_buckets(mode, shard_n, weighted):
  rng = np.random.default_rng(mode * 1000 + shard_n * 2 + weighted)
  ids = kv_edge_ids(rng, 300)
  B, T = 41, 8
  sl = _k1_slots(mode, shard_n, B, T)
  n_seg = B + B * T
  comb_seg = [SUM] * B + [MEAN] * (B * T)
  # single-valued: lookup l is segment l
  x = np.resize(ids, n_seg)
  w = _weights(rng, n_seg) if weighted else None
  got = _k1_call(x, w, None, None, n_seg, n_seg, sl, n_seg)
  want = k1_kv_ref(x, mode, shard_n, w, comb_seg)
  assert got == want, 'single-valued rows / owner'
  # CSR over every id, the cap at the total and five below it
  lens = rng.integers(0, 4, n_seg)
  lens[B] = 0
  rp = np.concatenate([[0], np.cumsum(lens)])
  total = int(rp[-1])
  seg = np.repeat(np.arange(n_seg), lens)
  x = np.resize(ids, total + 8)
  assert total >= ids.size
  w = _weights(rng, total + 8) if weighted else None
  sid = np.concatenate([seg, np.zeros(8, np.int64)])
  for cap in (total, total - 5):
    r, o = _k1_call(x, w, sid, rp, n_seg, cap, sl, total + 8)
    wr, wo = k1_kv_ref(x[:cap], mode, shard_n, None if w is None else w[:cap], [comb_seg[s] for s in seg[:cap]])
    assert r[:cap] == wr and o[:cap] == wo, 'CSR rows / owner (cap %d of %d)' % (cap, total)
    assert set(r[cap:]) == {S64} and set(o[cap:]) == {S32}, 'K1 wrote past the cap'


# ---- K8 with 63-bit rows ----------------------------------------------------------------------------------------------
def k8_case(world, n, seed):
  """(rows, owner) of n lookups: rows = key div world, owner = key mod world for keys across [0, 2^63 - 2], plus the
  adversarial pairs; dropped rows and owners outside [0, world) included"""
  rng = np.random.default_rng(seed)
  pool = rng.integers(0, 2 ** 63 - 1, max(4, n // 6), dtype=np.int64)
  pool[:2] = [0, 2 ** 63 - 2]
  keys = pool[rng.integers(0, pool.size, n)]
  rows, owner = keys // world, keys % world
  special = []
  if world >= 2:   # (x + 2^48 j, 0) and (x, j) pack to one integer under owner << 48 | row
    for x in (5, 2 ** 40 + 3):
      for j in range(1, min(world, 4)):
        special += [(x + (j << 48), 0), (x, j)]
  top = (2 ** 63 - 2) // world
  special += [(top, (2 ** 63 - 2) % world), (top - (1 << 34), 0), (top - (1 << 40), 0), (top - (1 << 50), 0)]
  special += [((1 << 34) + 7, 0), ((1 << 45) + 7, 0), (7, 0)]                 # differ only above bit 33
  special += [(2 ** 52 + 11, o) for o in range(min(world, 6))]               # one row, several owners
  for i, (r, o) in enumerate(special):
    if 2 * i + 1 < n:
      rows[2 * i], owner[2 * i] = r, o
      rows[2 * i + 1], owner[2 * i + 1] = r, o
  k = rng.integers(min(2 * len(special), n - 6), n, max(3, n // 20))
  rows[k[0::3]] = -1
  owner[k[1::3]] = -1
  owner[k[2::3]] = world
  if n >= 128:
    rows[96:128], owner[96:128] = 2 ** 47 + 5, 0                            # a whole warp of one key
  return rows.astype(np.int64), owner.astype(np.int64)


def k8_check(rows, owner, world, cap, send, pos, counts):
  """K8's contract on exact (row, owner) pairs (no packing): counts, positions, send blocks and lost lookups"""
  live = (rows >= 0) & (owner >= 0) & (owner < world)
  pairs = np.stack([rows[live], owner[live]], 1)
  uk, inv = np.unique(pairs, axis=0, return_inverse=True)
  inv = inv.reshape(-1)
  cnt = np.bincount(uk[:, 1], minlength=world)[:world]
  assert np.array_equal(counts[:world], cnt), 'counts[o] must be the distinct rows of owner o'
  assert (pos[~live] == -1).all(), 'a dropped lookup or an owner outside [0, world) got a position'
  p = pos[live]
  # every lookup of one (row, owner) pair has one position
  first = np.full(uk.shape[0], -2, np.int64)
  first[inv[::-1]] = p[::-1]
  assert np.array_equal(first[inv], p), 'lookups of one (row, owner) pair got different positions'
  ok = p >= 0
  assert (send[p[ok]] == rows[live][ok]).all(), 'send_rows[pos[l]] != rows[l]'
  assert (p[ok] // cap == owner[live][ok]).all(), 'position outside the owner block'
  held = first[first >= 0]
  assert np.unique(held).size == held.size, 'two (row, owner) pairs share a position'
  assert held.size == np.minimum(cnt, cap).sum(), 'positions claimed'
  assert (~ok).sum() == counts[world], 'counts[world] must be the number of lost lookups'
  assert (first < 0).sum() == np.maximum(cnt - cap, 0).sum(), 'pairs lost to a full block'
  blk = send.reshape(world, cap)
  filled = np.arange(cap)[None, :] < np.minimum(cnt, cap)[:, None]
  assert (blk[filled] >= 0).all() and (blk[~filled] == -1).all(), 'send_rows blocks: rows first, -1 padding'


@pytest.mark.parametrize('n', [31, 257, 212992])
@pytest.mark.parametrize('world', [1, 2, 3, 8, 64, 65, 200])
def test_k8_on_63_bit_rows(world, n):
  rows, owner = k8_case(world, n, world * 7 + n)
  live = (rows >= 0) & (owner >= 0) & (owner < world)
  cnt = np.bincount(np.unique(np.stack([rows[live], owner[live]], 1), axis=0)[:, 1], minlength=world)[:world]
  mx = int(cnt.max())
  t_rows, t_own = torch.from_numpy(rows).to(DEV), torch.from_numpy(owner.astype(np.int32)).to(DEV)
  ws = K.shard_group_workspace(n, DEV)
  for cap in [mx] + ([mx - 1] if mx >= 2 else []):   # an exact fit, and one row short in the fullest block
    sb, send = _guarded(world * cap, torch.int64, S64)
    pb, pos = _guarded(n, torch.int64, S64)
    cb, counts = _guarded(world + 1, torch.int32, S32)
    _lib.check(L().er_shard_group(_p(t_rows), _p(t_own), n, world, cap, _p(send), _p(pos), _p(counts), _p(ws),
                                  ws.numel(), _stream()), 'er_shard_group')
    for b, s, nm in ((sb, S64, 'send_rows'), (pb, S64, 'pos'), (cb, S32, 'counts')):
      _guards(b, s, nm)
    c = counts.cpu().numpy()
    k8_check(rows, owner, world, cap, send.cpu().numpy(), pos.cpu().numpy(), c)
    assert (c[world] == 0) == (cap == mx)


# ---- the index kernels --------------------------------------------------------------------------------------------------
def group_of(keys, n_groups):
  return (kv_doubles._mix(np.asarray(keys, np.int64).astype(np.uint64)) & np.uint64(n_groups - 1)).astype(np.int64)


def _index(n_index):
  return (torch.full((n_index,), _lib.KV_EMPTY, dtype=torch.int64, device=DEV),
          torch.full((n_index,), -1, dtype=torch.int64, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV))


def index_check(keys, rows, index_keys, index_rows, stats, capacity, n_index, before=None):
  """the documented semantics as a dict model (exact).  Every live key of `keys` is claimed while the index has a free
  slot; a claimed key holds the next row while rows are left, else -1; a lookup reads its key's row and counts in
  stats[1] when that is -1.  `before`: {key: row} held before the call.  Returns {key: row} after it."""
  before = dict(before or {})
  ik, ir = index_keys.tolist(), index_rows.tolist()
  held = {k: r for k, r in zip(ik, ir) if k != _lib.KV_EMPTY}
  assert len(held) == sum(k != _lib.KV_EMPTY for k in ik), 'a key sits in two slots'
  live = [k for k in keys if k >= 0]
  distinct = set(live)
  assert all(held.get(k, r) == r for k, r in before.items()), 'a held key moved or changed its row'
  new = distinct - set(before)
  claimed = set(held) - set(before)
  assert claimed <= new, 'the index holds a key nobody looked up'
  assert len(claimed) == min(len(new), n_index - len(before)), 'every new key is claimed while a slot is free'
  n0 = int(stats[0])
  assert n0 == len(held), 'stats[0] must count the claims'
  given = sorted(r for k, r in held.items() if k in claimed and r >= 0)
  n_before = len(before)
  assert given == list(range(min(n_before, capacity), min(n0, capacity))), 'new keys take the next rows, in order'
  for k, r in zip(keys, rows):
    want = -1 if k < 0 else held.get(k, -1)
    assert r == want, 'key %d: row %d, the index holds %d' % (k, r, want)
  return held


def _insert(ik, ir, stats, capacity, keys, dim=4, truncated=True, stddev=0.01, shard=(1, 0)):
  w = torch.zeros(capacity + 1, dim, device=DEV)
  t = torch.tensor(np.asarray(keys, np.int64), device=DEV)
  rows = torch.empty_like(t)
  K.kv_find_or_insert(ik, ir, capacity, stats, t, rows, w, None, None, 0.0, 5, stddev, truncated,
                      shard_n=shard[0], shard_rank=shard[1])
  return rows.cpu().numpy().tolist(), w


@pytest.mark.parametrize('n_groups', [1, 2])
def test_smallest_indexes_filled_past_their_slots(n_groups):
  n_index = 16 * n_groups
  capacity = n_index // 2
  rng = np.random.default_rng(n_groups)
  distinct = rng.integers(0, 2 ** 63 - 1, 3 * n_index, dtype=np.int64)
  keys = rng.permutation(np.concatenate([distinct, distinct, [-1, -5]])).tolist()
  ik, ir, stats = _index(n_index)
  rows, _ = _insert(ik, ir, stats, capacity, keys)
  held = index_check(keys, rows, ik.cpu(), ir.cpu(), stats.cpu(), capacity, n_index)
  assert len(held) == n_index and sum(r >= 0 for r in held.values()) == capacity
  lost = sum(1 for k, r in zip(keys, rows) if k >= 0 and r < 0)
  assert stats.cpu().tolist() == [n_index, lost]
  # again: nothing claimed, the same rows, every lookup without a row counted again
  rows2, _ = _insert(ik, ir, stats, capacity, keys)
  assert rows2 == rows and stats.cpu().tolist() == [n_index, 2 * lost]
  # find: a held key reads its row, a key claimed beyond capacity and an absent key the zero row
  absent = [k for k in range(10 ** 6, 10 ** 6 + 64) if k not in held][:8]
  probe = torch.tensor(list(held) + absent + [-1], device=DEV)
  found = torch.empty_like(probe)
  K.kv_find(ik, ir, probe, capacity, found)
  want = [r if r >= 0 else capacity for r in held.values()] + [capacity] * len(absent) + [-1]
  assert found.cpu().tolist() == want


def test_probe_chain_wraps_from_the_last_group_to_group_0():
  n_index, capacity = 64, 32
  n_groups = n_index // 16
  cands = np.arange(1, 4000, dtype=np.int64) * 1000003
  last = cands[group_of(cands, n_groups) == n_groups - 1][:21].tolist()
  assert len(last) == 21
  ik, ir, stats = _index(n_index)
  rows, _ = _insert(ik, ir, stats, capacity, last * 3)
  held = index_check(last * 3, rows, ik.cpu(), ir.cpu(), stats.cpu(), capacity, n_index)
  slots = [s for s, k in enumerate(ik.cpu().tolist()) if k != _lib.KV_EMPTY]
  assert slots == list(range(5)) + list(range(48, 64)), 'the chain fills the last group, then wraps to group 0'
  found = torch.empty(len(last), dtype=torch.int64, device=DEV)
  K.kv_find(ik, ir, torch.tensor(last, device=DEV), capacity, found)
  assert found.cpu().tolist() == [held[k] for k in last]


def zipf_keys(rng, distinct, n):
  """n lookups over `distinct` 63-bit keys: Zipf(1.2) draws, so that the head repeats across neighbouring tiles and
  warps, then every key once"""
  pool = np.unique(rng.integers(0, 2 ** 63 - 1, distinct + distinct // 8, dtype=np.int64))[:distinct]
  pool = rng.permutation(pool)
  z = np.minimum(rng.zipf(1.2, n - distinct), distinct) - 1
  z[rng.integers(0, z.size, z.size // 4)] = 0          # a quarter more of the hottest key
  return np.concatenate([pool[z], pool]), pool


@pytest.mark.parametrize('log2_cap', [20, 22])
def test_fill_to_capacity_under_races(log2_cap):
  capacity = 1 << log2_cap
  rng = np.random.default_rng(log2_cap)
  keys, pool = zipf_keys(rng, capacity, 3 * capacity)
  ik, ir, stats = _index(2 * capacity)
  t = torch.from_numpy(keys).to(DEV)
  rows = torch.empty_like(t)
  w = torch.empty(capacity + 1, 1, device=DEV)
  K.kv_find_or_insert(ik, ir, capacity, stats, t, rows, w, None, None, 0.0, 3, 0.01)
  r = rows.cpu().numpy()
  assert stats.cpu().tolist() == [capacity, 0]
  order = np.argsort(keys, kind='stable')
  ks, rs = keys[order], r[order]
  head = np.concatenate([[True], ks[1:] != ks[:-1]])
  start = np.flatnonzero(head)
  assert start.size == capacity
  per_key = rs[start]
  assert (np.maximum.reduceat(rs, start) == per_key).all() and (np.minimum.reduceat(rs, start) == per_key).all(), \
      'lookups of one key got different rows'
  assert np.array_equal(np.sort(per_key), np.arange(capacity)), 'rows are not a permutation of [0, distinct)'
  ikc, irc = ik.cpu().numpy(), ir.cpu().numpy()
  used = ikc != _lib.KV_EMPTY
  assert used.sum() == capacity
  assert np.array_equal(np.sort(ikc[used]), ks[start])
  # the index's own (key, row) pairs are the ones handed out, and the rows hold their keys' initial values
  assert np.array_equal(irc[used][np.argsort(ikc[used])], per_key)
  smp = rng.integers(0, capacity, 4096)
  np.testing.assert_array_max_ulp(w[torch.from_numpy(per_key[smp]).to(DEV), 0].cpu().numpy(),
                                  kv_doubles.init_values(3, ks[start][smp], 1, 0.01)[:, 0], maxulp=1)


def _nan_filled(shape):
  return torch.full(shape, NAN_BITS, dtype=torch.int32, device=DEV).view(torch.float32)


@pytest.mark.parametrize('layout', ['interleaved', 'separate'])
@pytest.mark.parametrize('dim', [1, 3, 16, 17, 64, 300])
def test_new_rows_hold_their_initial_values_and_nothing_else_moves(dim, layout):
  capacity = 200
  pad = 5
  if layout == 'interleaved':   # one [weight | state0 | state1 | pad] row
    buf = _nan_filled((capacity + 1, 3 * dim + pad))
    w, s0, s1 = buf[:, :dim], buf[:, dim:2 * dim], buf[:, 2 * dim:3 * dim]
    bufs = [buf]
  else:
    bufs = [_nan_filled((capacity + 1, dim + pad)) for _ in range(3)]
    w, s0, s1 = (b[:, :dim] for b in bufs)
  before = [b.clone() for b in bufs]
  rng = np.random.default_rng(dim)
  distinct = rng.integers(0, 2 ** 63 - 1, 150, dtype=np.int64)
  keys = torch.tensor(rng.permutation(np.repeat(distinct, 3)), device=DEV)
  rows = torch.empty_like(keys)
  ik, ir, stats = _index(512)
  K.kv_find_or_insert(ik, ir, capacity, stats, keys, rows, w, s0, s1, 0.125, 77, 0.03)
  held = index_check(keys.tolist(), rows.tolist(), ik.cpu(), ir.cpu(), stats.cpu(), capacity, 512)
  ks = np.array(list(held), np.int64)
  rr = torch.tensor(list(held.values()), device=DEV)
  np.testing.assert_array_max_ulp(w[rr].cpu().numpy(), kv_doubles.init_values(77, ks, dim, 0.03), maxulp=1)
  assert bool((s0[rr] == 0.125).all()) and bool((s1[rr] == 0).all())
  # every other float keeps its bits: rows nobody took, the stride padding, the zero row
  for b, old in zip(bufs, before):
    m = torch.zeros(b.shape, dtype=torch.bool, device=DEV)
    m[rr, :3 * dim if layout == 'interleaved' else dim] = True
    assert torch.equal(b.view(torch.int32)[~m], old.view(torch.int32)[~m]), 'a float outside the new rows changed'


def test_initial_values_follow_the_truncated_normal_and_the_normal():
  """about a million keys x 16 columns: KS statistic, mean, variance and range against the distributions themselves
  (scipy), not against a restatement of the kernel's formula"""
  capacity, dim = 1 << 20, 16
  rng = np.random.default_rng(11)
  keys = np.unique(rng.integers(0, 2 ** 63 - 1, capacity + 4096, dtype=np.int64))[:capacity]
  for truncated, sigma in ((True, 0.01 / math.sqrt(dim)), (False, 0.0025)):
    ik, ir, stats = _index(2 * capacity)
    w = torch.empty(capacity + 1, dim, device=DEV)
    t = torch.from_numpy(keys).to(DEV)
    rows = torch.empty_like(t)
    K.kv_find_or_insert(ik, ir, capacity, stats, t, rows, w, None, None, 0.0, 1234, sigma, truncated)
    x = w[:capacity].double().cpu().numpy().reshape(-1) / np.float32(sigma)
    n = x.size
    dist = scipy.stats.truncnorm(-2, 2) if truncated else scipy.stats.norm()
    ks = scipy.stats.kstest(x, dist.cdf).statistic
    assert ks < 1.63 * 1.5 / math.sqrt(n), 'KS statistic %g (n %d)' % (ks, n)       # far beyond the 1% level
    var = dist.var()
    assert abs(x.mean()) < 5 * math.sqrt(var / n), 'mean %g' % x.mean()
    assert abs(x.var() / var - 1) < 5 * math.sqrt(2.0 / n), 'variance %g of %g' % (x.var(), var)
    if truncated:
      # the draws fill [-2, 2] up to about 1/(n phi(2)) of each end: a bound off by 1e-5 in probability misses by 2e-4
      assert x.min() >= -2 * (1 + 2 ** -22) and x.max() <= 2 * (1 + 2 ** -22), 'outside 2 stddev'
      assert x.min() < -2 + 2e-5 and x.max() > 2 - 2e-5, 'range [%r, %r] does not reach +-2 stddev' % (x.min(), x.max())
    else:
      assert 4.5 < -x.min() < 8.3 and 4.5 < x.max() < 8.3, 'range [%r, %r]' % (x.min(), x.max())
    # and the same keys inserted in another order get the same values per key
    perm = rng.permutation(capacity)
    ik2, ir2, st2 = _index(2 * capacity)
    w2 = torch.empty_like(w)
    t2 = t[torch.from_numpy(perm).to(DEV)]
    rows2 = torch.empty_like(t2)
    K.kv_find_or_insert(ik2, ir2, capacity, st2, t2, rows2, w2, None, None, 0.0, 1234, sigma, truncated)
    inv = torch.empty_like(rows2)
    inv[torch.from_numpy(perm).to(DEV)] = rows2
    assert torch.equal(w[rows].view(torch.int32), w2[inv].view(torch.int32)), 'values depend on insertion order'


def _kv_arena(capacity, dim=4, seed=H.SEED):
  a = E.Arena(dim, DEV, 1, 0)
  a.add_table('t', capacity + 1)
  a.kv = E.KvTable('t', a, capacity, seed)
  a.materialize(_lib.OPT_ADAGRAD, init_fn=lambda w: w.zero_())
  return a


def test_load_then_insert_hands_out_rows_after_the_restored_ones():
  capacity = 64
  rng = np.random.default_rng(9)
  keys = rng.integers(0, 2 ** 63 - 1, capacity + 40, dtype=np.int64)
  # at full capacity: every key found at its given row, and a new key gets no row
  a = _kv_arena(capacity)
  given = torch.from_numpy(rng.permutation(capacity))
  a.kv.load(torch.from_numpy(keys[:capacity]), given)
  assert a.kv.stats.cpu().tolist() == [capacity, 0]
  out = torch.empty(capacity + 1, dtype=torch.int64, device=DEV)
  probe = torch.from_numpy(np.append(keys[:capacity], keys[capacity])).to(DEV)
  a.kv.lookup(probe, out, train=True)
  assert out.cpu().tolist() == given.tolist() + [-1]
  assert a.kv.stats.cpu().tolist() == [capacity + 1, 1]
  # restore 40 keys, then insert 30 new ones (and the restored ones again): rows 40..63, then none left
  a = _kv_arena(capacity)
  given = torch.from_numpy(rng.permutation(40))
  a.kv.load(torch.from_numpy(keys[:40]), given)
  before = dict(zip(keys[:40].tolist(), given.tolist()))
  new = keys[40:70]
  mixed = rng.permutation(np.concatenate([new, keys[:40], new]))
  out = torch.empty(mixed.size, dtype=torch.int64, device=DEV)
  a.kv.lookup(torch.from_numpy(mixed).to(DEV), out, train=True)
  held = index_check(mixed.tolist(), out.cpu().tolist(), a.kv.index_keys.cpu(), a.kv.index_rows.cpu(),
                     a.kv.stats.cpu(), capacity, a.kv.index_keys.numel(), before=before)
  assert sorted(r for k, r in held.items() if k not in before and r >= 0) == list(range(40, 64))
  # negative and repeated keys are refused and counted
  a = _kv_arena(capacity)
  with pytest.raises(_lib.ErError, match='negative or repeated'):
    a.kv.load(torch.tensor([3, -4, 5, 3, 3]), torch.arange(5))
  assert int(a.kv.stats[1]) == 3


# ---- InputLayer: every row optimizer per key ----------------------------------------------------------------------------
OPTS = [('sgd', _lib.OPT_SGD), ('adagrad', _lib.OPT_ADAGRAD), ('lazy_adam', _lib.OPT_LAZY_ADAM),
        ('adam', _lib.OPT_ADAM_ROWS), ('momentum', _lib.OPT_MOMENTUM)]
TAG_WEIGHTS = np.array([1.5, 0.5, 0.0, -0.75, 2.0], np.float32)   # (a mean lookup whose weight is not > 0 is pruned)


def make_model_layer(opt, device):
  """a static user table; a key-value item table read by the deep group and, as its dim-1 `_wide` table, by the wide
  group; key-value tag tables pooled by a weighted sum (stags) and a weighted mean (mtags)"""
  D = H.DIM
  feats = [IL.id_feature('user', D, hash_bucket_size=50),
           IL.id_feature('item', D, hash_bucket_size=1000, kv_capacity=64),
           IL.multi_feature('stags', 'tag', D, num_buckets=30, kv_capacity=64),
           IL.multi_feature('mtags', 'tag', D, num_buckets=30, combiner='mean', kv_capacity=64)]
  groups = collections.OrderedDict(all=dict(features=['user', 'item', 'stags', 'mtags']),
                                   wide=dict(features=['user', 'item'], wide=True))
  return IL.InputLayer(feats, groups, H.B, device, embedding_optimizer=opt, generator=torch.Generator(device).manual_seed(1),
                       adagrad_init=0.1, kv_seed=H.SEED, max_tag_lookups=4 * H.B)


def model_batch(rng, device, prune=True):
  """prune=False: positive weights only on the mean tags (the host doubles of K1 take no weights, so they cannot drop
  the lookups the mean prunes before the key-value lookup)"""
  B = H.B
  users, items = rng.integers(0, 100, B), rng.integers(0, 12, B) * 1000003
  batch = dict(items=items)
  feats = {'sparse_fea': torch.tensor(np.concatenate([users, items]), dtype=torch.int64, device=device), 'tag_fea': {}}
  for name in ('stags', 'mtags'):
    lens = rng.integers(0, 4, B).astype(np.int32)
    vals = rng.integers(0, 6, int(lens.sum()))
    w = TAG_WEIGHTS[rng.integers(0, TAG_WEIGHTS.size, vals.size)]
    if name == 'mtags' and not prune:
      w = np.abs(w) + 0.25
    batch[name] = (vals, lens, w)
    feats['tag_fea'][name] = (torch.tensor(vals, dtype=torch.int64, device=device), torch.tensor(lens, device=device),
                              torch.tensor(w, device=device))
  return feats, batch


def model_grads(batch, RR):
  """{table: {key: float64 gradient summed over the step's lookups}}: sum lookups carry w R (w <= 0 included), mean
  lookups w R / sum w over the segment's lookups with w > 0"""
  R, Rw = (x.double().cpu().numpy() for x in RR)
  D = H.DIM
  g = collections.defaultdict(lambda: collections.defaultdict(lambda: 0.0))
  for b, v in enumerate(batch['items']):
    g['item_embedding'][H.item_key(v)] = g['item_embedding'][H.item_key(v)] + R[b, D:2 * D]
    g['item_embedding_wide'][H.item_key(v)] = g['item_embedding_wide'][H.item_key(v)] + Rw[b, 1:2]
  for name, col, mean in (('stags', 2, False), ('mtags', 3, True)):
    vals, lens, w = batch[name]
    off = 0
    for b, n in enumerate(lens):
      v, ww = vals[off:off + n], w[off:off + n].astype(np.float64)
      off += n
      live = ww > 0 if mean else np.ones(n, bool)
      tot = ww[live].sum()
      for k, x in zip(v[live].tolist(), ww[live]):
        t = g[name + '_embedding']
        t[k] = t[k] + (x / tot if mean else x) * R[b, col * D:(col + 1) * D]
  return {t: {k: np.broadcast_to(v, (1 if t.endswith('_wide') else D,)).astype(np.float64) for k, v in d.items()}
          for t, d in g.items()}


def train_model(opt, device, seed=3, prune=True):
  """three steps of make_model_layer -> (layer, [(batch, (R, R_wide))])"""
  il = make_model_layer(opt, device)
  rng = np.random.default_rng(seed)
  steps = []
  for t in range(3):
    feats, batch = model_batch(rng, device, prune)
    R = torch.tensor(rng.integers(-3, 4, (H.B, 4 * H.DIM)) / 4.0, dtype=torch.float32, device=device)
    Rw = torch.tensor(rng.integers(-3, 4, (H.B, 2)) / 4.0, dtype=torch.float32, device=device)
    out = il.lookup(feats)
    concat, wide = out['all'][0], out['wide'][0]
    assert concat.shape == R.shape and wide.shape == Rw.shape
    ((concat * R).sum() + (wide * Rw).sum()).backward()
    il.set_optimizer_step(0.05, t)
    il.backward_update()
    steps.append((batch, (R, Rw)))
  return il, steps


def check_per_key(il, ref, kind, tol):
  """every key-value table per key against the restatement: the row and the optimizer states the rule keeps (state0
  for all but sgd, state1 for the Adam rules; the others must not exist)"""
  want0, want1 = kind != 'sgd', kind in ('adam', 'lazy_adam')
  tables = {a.kv.name: a for a in il.arenas.values() if a.kv is not None}
  assert set(ref) <= set(tables) and all(ref.values())
  for table, a in tables.items():
    assert (a.state0 is not None, a.state1 is not None) == (want0, want1), table
    keys, rows = a.kv.items()
    got = {k: r for k, r in zip(keys.tolist(), rows.tolist())}
    want = ref.get(table, {})
    assert set(got) == set(want) and il.kv_sizes()[table] == len(want), table
    for k, (w, s0, s1) in want.items():
      r = got[k]
      np.testing.assert_allclose(a.weight[r].double().cpu().numpy(), w, atol=tol, rtol=0,
                                 err_msg='%s key %d' % (table, k))
      for st, sr, on in ((a.state0, s0, want0), (a.state1, s1, want1)):
        if on:
          np.testing.assert_allclose(st[r].double().cpu().numpy(), sr, atol=tol, rtol=0,
                                     err_msg='%s key %d state' % (table, k))


@pytest.mark.parametrize('kind,opt', OPTS, ids=[o[0] for o in OPTS])
def test_every_row_optimizer_per_key_against_float64(kind, opt):
  il, steps = train_model(opt, DEV)
  ref = H.restate(steps, kind, grads_of=model_grads)
  assert set(ref) == {'item_embedding', 'item_embedding_wide', 'stags_embedding', 'mtags_embedding'}
  check_per_key(il, ref, kind, 1e-6)
  il.check_kv()


def sparse_sqnorm_ref(batch, R, kv):
  """float64 ||IndexedSlices.values||^2 of make_norm_layer's four columns: one entry per (column, distinct row) - the
  key of a key-value column, the bucket of a static one; item and item2 read one table but are deduplicated apart"""
  R = R.double().cpu().numpy()
  D = H.DIM
  cols = [collections.defaultdict(lambda: np.zeros(D)) for _ in range(4)]
  for b in range(H.B):
    cols[0][_lib.fingerprint64(str(int(batch['users'][b]))) % 50] += R[b, :D]
    for c, v in ((1, int(batch['items'][b])), (2, int(batch['items2'][b]))):
      cols[c][H.item_key(v) if kv else _lib.fingerprint64(str(v)) % 1000] += R[b, c * D:(c + 1) * D]
  off = 0
  for b, n in enumerate(batch['lens']):
    for v in batch['tags'][off:off + n]:
      cols[3][int(v)] += R[b, 3 * D:]
    off += n
  return sum(float((g * g).sum()) for c in cols for g in c.values())


def make_norm_layer(kv, device):
  cap = 64 if kv else 0
  feats = [IL.id_feature('user', H.DIM, hash_bucket_size=50),
           IL.id_feature('item', H.DIM, hash_bucket_size=1000, kv_capacity=cap),
           IL.id_feature('item2', H.DIM, hash_bucket_size=1000, embedding_name='item_embedding', kv_capacity=cap),
           IL.multi_feature('tags', 'tag', H.DIM, num_buckets=30, kv_capacity=cap)]
  groups = collections.OrderedDict(all=dict(features=['user', 'item', 'item2', 'tags']))
  return IL.InputLayer(feats, groups, H.B, device, embedding_optimizer=_lib.OPT_SGD,
                       generator=torch.Generator(device).manual_seed(1), kv_seed=H.SEED, max_tag_lookups=4 * H.B)


def norm_steps(kv, device):
  """(sparse_grad_sqnorm, float64 restatement) of three steps"""
  il = make_norm_layer(kv, device)
  rng = np.random.default_rng(17)
  out = []
  for t in range(3):
    users, items2 = rng.integers(0, 100, H.B), rng.integers(0, 12, H.B) * 1000003
    feats, batch = H.make_batch(rng, device=device)
    feats['sparse_fea'] = torch.cat([torch.from_numpy(users).to(device), feats['sparse_fea'][H.B:],
                                     torch.from_numpy(items2).to(device)])
    batch.update(users=users, items2=items2)
    R = torch.tensor(rng.integers(-3, 4, (H.B, 4 * H.DIM)) / 4.0, dtype=torch.float32, device=device)
    concat, _ = il.lookup(feats)['all']
    (concat * R).sum().backward()
    out.append((float(il.sparse_grad_sqnorm()), sparse_sqnorm_ref(batch, R, kv)))
    il.set_optimizer_step(0.05, t)
    il.backward_update()
  return out


@pytest.mark.parametrize('kv', [True, False], ids=['key_value', 'static'])
def test_emit_form_sparse_norm_against_float64(kv):
  """gradient_clipping_by_norm's sparse part: K7 in emit form over virtual rows row + column * n_rows, per column and
  distinct row.  item and item2 share a table (on a key-value arena n_rows = capacity + 1), and the tags column is CSR"""
  for got, want in norm_steps(kv, DEV):
    assert want > 1.0
    assert abs(got - want) <= 1e-5 * want, 'sparse norm^2 %r, float64 %r' % (got, want)


NORM_LR, CLIP = 16.0, 0.01
NORM_CFG = H.CFG.replace(
    'adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.1 } } }',
    'momentum_optimizer { learning_rate { constant_learning_rate { learning_rate: %g } } momentum_optimizer_value: 0.0 }'
    % NORM_LR).replace('deepfm { dnn { hidden_units: [8] }',
                       'deepfm { l2_regularization: 0.5 dnn { hidden_units: [8] use_bn: false }')


def _norm_estimator(kv, clip):
  from easyrec_b200.estimator import EasyRecEstimator
  ev = 'ev_params { max_capacity: 100 }' if kv else ''
  cfg = NORM_CFG % ('gradient_clipping_by_norm: %g' % clip if clip else '', ev, ev, '')
  assert 'momentum_optimizer' in cfg and 'l2_regularization' in cfg
  return EasyRecEstimator(cfg.encode(), device=DEV, seed=11)


def _step_gradient_sq(est, feats, labels):
  """one step of plain SGD (momentum 0, no clipping); returns float64 (dense, sparse) squared gradient norms, read off
  the update: the dense step carries the l2 term, and every table is read by one column, so a row's step is its
  (column, row) IndexedSlices entry"""
  p0 = est.trainer.dense_opt.flat_p.double().cpu()
  w0 = {d: a.weight.double().cpu() for d, a in est.input_layer.arenas.items() if a.kv is None}
  est.trainer.train_step(feats, labels)
  torch.cuda.synchronize()
  dense = float((((est.trainer.dense_opt.flat_p.double().cpu() - p0) / NORM_LR) ** 2).sum())
  sparse = 0.0
  for d, a in est.input_layer.arenas.items():
    if a.kv is None:
      sparse += float((((a.weight.double().cpu() - w0[d]) / NORM_LR) ** 2).sum())
    else:
      keys, rows = a.kv.items()
      init = kv_doubles.init_values(a.kv.seed, keys.numpy(), a.dim, a.kv.init_stddev, a.kv.init_truncated)
      sparse += float((((a.weight[rows.to(DEV)].double().cpu().numpy() - init) / NORM_LR) ** 2).sum())
  return dense, sparse, p0


@pytest.mark.parametrize('kv', [True, False], ids=['key_value', 'static'])
def test_trainer_global_norm_against_float64(kv):
  """train_config.gradient_clipping_by_norm: last_grad_norm is sqrt(sparse + dense + l2) of the float64 step, and the
  clipped step is the plain one times clip / norm"""
  torch.backends.cuda.matmul.allow_tf32 = False
  feats, labels = _batches(1)[0]
  plain, clipped = _norm_estimator(kv, 0), _norm_estimator(kv, CLIP)
  assert (plain.input_layer.arenas.keys() == clipped.input_layer.arenas.keys() and
          any(a.kv is not None for a in plain.input_layer.arenas.values()) == kv)
  dense, sparse, p0 = _step_gradient_sq(plain, feats, labels)
  assert dense > 0.01 * sparse and sparse > 0.01 * dense, (dense, sparse)
  clipped.trainer.train_step(feats, labels)
  norm = math.sqrt(dense + sparse)
  assert norm > 10 * CLIP
  got = float(clipped.trainer.last_grad_norm)
  assert abs(got - norm) <= 1e-4 * norm, 'last_grad_norm %r, float64 %r (dense %r, sparse %r)' % (got, norm, dense,
                                                                                                 sparse)
  step_plain = plain.trainer.dense_opt.flat_p.double().cpu() - p0
  step_clip = clipped.trainer.dense_opt.flat_p.double().cpu() - p0
  torch.testing.assert_close(step_clip, step_plain * (CLIP / norm), rtol=1e-3, atol=1e-7)


# ---- restore, then train --------------------------------------------------------------------------------------------
def _estimator():
  from easyrec_b200.estimator import EasyRecEstimator
  cfg = H.CFG % ('', 'ev_params { max_capacity: 1000 }', 'ev_params { max_capacity: 100 }', '')
  return EasyRecEstimator(cfg.encode(), device=DEV, seed=11)


def _batches(n):
  rng = np.random.default_rng(21)
  out = []
  for _ in range(n):
    ids = np.concatenate([rng.integers(0, 60, 8), rng.integers(0, 40, 8) * 1000003])
    lens = rng.integers(0, 4, 8).astype(np.int32)
    tags = rng.integers(0, 15, int(lens.sum()))
    out.append(({'sparse_fea': torch.tensor(ids, device=DEV),
                 'tag_fea': {'tags': (torch.tensor(tags, device=DEV), torch.tensor(lens, device=DEV), None)}},
                torch.tensor(rng.integers(0, 2, 8), dtype=torch.float32, device=DEV)))
  return out


def _state(est):
  torch.cuda.synchronize()
  out = {'dense': est.trainer.dense_opt.flat_p.cpu().numpy().tobytes()}
  for d, a in est.input_layer.arenas.items():
    st = a.storage.cpu()
    if a.kv is None:
      out[d] = st.numpy().tobytes()
    else:
      keys, rows = a.kv.items()
      out[d] = {k: st[r].numpy().tobytes() for k, r in zip(keys.tolist(), rows.tolist())}
  return out


def _renumber(est, seed):
  """move every key-value table's keys to a permutation of their rows (storage rows moved with them)"""
  g = torch.Generator().manual_seed(seed)
  for a in est.input_layer.arenas.values():
    if a.kv is not None:
      keys, rows = a.kv.items()
      new = rows[torch.randperm(rows.numel(), generator=g)]
      assert rows.numel() < 3 or not torch.equal(new, rows)
      st = a.storage.clone()
      a.storage[new.to(DEV)] = st[rows.to(DEV)]
      a.kv.load(keys, new)


@pytest.mark.parametrize('renumber', [False, True], ids=['rows_kept', 'rows_permuted'])
@pytest.mark.parametrize('parts', [False, True], ids=['torch_checkpoint', 'embedding_parts'])
def test_restore_then_train_is_bit_identical_to_an_uninterrupted_run(parts, renumber, tmp_path):
  """K7 sums each row's lookups in lookup order whatever the row numbers are, so a restored table continues bit for
  bit, also when its keys come back on other rows"""
  batches = _batches(6)
  whole = _estimator()
  for f, y in batches:
    whole.trainer.train_step(f, y)
  first = _estimator()
  for f, y in batches[:3]:
    first.trainer.train_step(f, y)
  path = first.save(str(tmp_path), embedding_parts=parts)
  assert os.path.isdir(path[:-3] + '-embedding') == parts
  resumed = _estimator().restore(path)
  if renumber:
    _renumber(resumed, 3)
  for f, y in batches[3:]:
    resumed.trainer.train_step(f, y)
  a, b = _state(whole), _state(resumed)
  assert a.keys() == b.keys()
  for k in a:
    assert a[k] == b[k], '%s differs after restore' % (k,)


# ---- the row-sharded owner chain on one GPU ------------------------------------------------------------------------------
def _owner_chain(N, ids, R, lr, capacity=512, dim=8):
  """N ranks in one process: each rank r looks up ids[r] (single-valued, one slot, sum) at KV_BUCKETS with shard_n N.
  Returns ({global key: (owner, initial row, post-step row)}, [pooled [B, dim] per rank])"""
  B = ids[0].size
  sl = K.make_slots([dict(num_buckets=KVB, row_offset=0, seg_begin=0, n_seg=B, bucket_mode=FARM, combiner=SUM,
                          out_buf=0, out_stride=dim, out_col=0, shard_n=N)], dim)
  sd = K.slots_to_device(sl, DEV)
  cap = B
  rows_l, own_l, pos_l, send_l = [], [], [], []
  for r in range(N):   # requester: K1 -> K8
    t = torch.from_numpy(ids[r]).to(DEV)
    rows, own = torch.empty_like(t), torch.empty(B, dtype=torch.int32, device=DEV)
    K.bucketize(t, sd, 1, B, rows=rows, owner=own)
    send = torch.empty(N * cap, dtype=torch.int64, device=DEV)
    pos = torch.empty(B, dtype=torch.int64, device=DEV)
    counts = torch.zeros(N + 1, dtype=torch.int32, device=DEV)
    K.shard_group(rows, own, N, cap, send, pos, counts, K.shard_group_workspace(B, DEV))
    assert int(counts[N]) == 0
    rows_l.append(rows), own_l.append(own), pos_l.append(pos), send_l.append(send)
  # the id all-to-all: owner o receives block o of every requester, requester-major
  recv = [torch.cat([send_l[r][o * cap:(o + 1) * cap] for r in range(N)]) for o in range(N)]
  arenas, owner_rows, send_emb = [], [], []
  n_ex = N * cap
  own_slots = K.slots_to_device(K.make_slots([dict(num_buckets=capacity + 1, row_offset=0, seg_begin=0, n_seg=n_ex,
                                                   bucket_mode=_lib.BUCKET_NONE,
                                                   combiner=SUM | _lib.COMBINER_UNIT_WEIGHTS, out_buf=0,
                                                   out_stride=dim, out_col=0, shard_n=1)], dim), DEV)
  for o in range(N):   # owner: keys -> pool rows, then the gather
    a = E.Arena(dim, DEV, N, o)
    a.add_table('t', capacity + 1)
    a.kv = E.KvTable('t', a, capacity, 99, embedding_parallel=True)
    a.materialize(_lib.OPT_SGD, init_fn=lambda w: w.zero_())
    orow = torch.empty_like(recv[o])
    a.kv.lookup(recv[o], orow, train=True)
    emb = torch.zeros(n_ex, dim, device=DEV)
    K.embedding_fwd(a.weight, dim, orow, own_slots, 1, n_ex, [emb])
    arenas.append(a), owner_rows.append(orow), send_emb.append(emb)
  def per_key(o):
    ks, rs = arenas[o].kv.items()
    w = arenas[o].weight.double().cpu().numpy()
    return {k: w[r].copy() for k, r in zip(ks.tolist(), rs.tolist())}
  init = [per_key(o) for o in range(N)]
  # the row all-to-all back; the requester pools by position
  pool_slots = K.slots_to_device(K.make_slots([dict(num_buckets=n_ex, row_offset=0, seg_begin=0, n_seg=B,
                                                    bucket_mode=_lib.BUCKET_NONE, combiner=SUM, out_buf=0,
                                                    out_stride=dim, out_col=0, shard_n=1)], dim), DEV)
  recv_emb = [torch.cat([send_emb[o][r * cap:(r + 1) * cap] for o in range(N)]) for r in range(N)]
  pooled, send_g = [], []
  for r in range(N):
    out = torch.zeros(B, dim, device=DEV)
    K.embedding_fwd(recv_emb[r], dim, pos_l[r], pool_slots, 1, B, [out])
    pooled.append(out.double().cpu().numpy())
    sums = torch.zeros(n_ex, dim, device=DEV)   # requester K7: the gradient summed per position (emit into a table)
    K.embedding_bwd(sums, None, None, dim, pos_l[r], pool_slots, 1, B, [R[r].contiguous()],
                    K.make_opt(_lib.OPT_SGD, -1.0), K.bwd_workspace(B, DEV, dim), n_rows=n_ex)
    send_g.append(sums)
  for o in range(N):   # the gradient all-to-all, then the owner's K7 at grad_scale 1/N
    recv_g = torch.cat([send_g[r][o * cap:(o + 1) * cap] for r in range(N)])
    a = arenas[o]
    K.embedding_bwd(a.weight, None, None, dim, owner_rows[o], own_slots, 1, n_ex, [recv_g],
                    K.make_opt(_lib.OPT_SGD, lr, grad_scale=1.0 / N), K.bwd_workspace(n_ex, DEV, dim), n_rows=a.n_rows)
  out = {}
  for o in range(N):
    for k, w1 in per_key(o).items():
      assert k not in out, 'key %d on two owners' % k
      out[k] = (o, init[o][k], w1)
  return out, pooled


@pytest.mark.parametrize('N', [2, 3])
def test_row_sharded_owner_chain_against_one_rank_float64(N):
  B, dim, lr = 64, 8, 0.5
  rng = np.random.default_rng(N)
  pool = np.concatenate([rng.integers(I64_MIN, I64_MAX, 40, dtype=np.int64), [0, -1, I64_MAX]])
  ids = [pool[rng.integers(0, pool.size, B)] for _ in range(N)]
  R = [torch.tensor(rng.integers(-4, 5, (B, dim)) / 8.0, dtype=torch.float32, device=DEV) for _ in range(N)]
  got, pooled = _owner_chain(N, ids, R, lr)
  # one rank over the concatenated batch, float64
  keys = {_lib.fingerprint64(str(int(v))) % KVB for x in ids for v in x}
  assert set(got) == keys, 'the owners together hold exactly the one-rank keys'
  table_seed = E._mix64(99 ^ _lib.fingerprint64('t'))
  grads = collections.defaultdict(lambda: np.zeros(dim))
  for r in range(N):
    g = R[r].double().cpu().numpy()
    for b, v in enumerate(ids[r]):
      k = _lib.fingerprint64(str(int(v))) % KVB
      grads[k] += g[b]
      np.testing.assert_array_equal(pooled[r][b], got[k][1], err_msg='rank %d lookup %d' % (r, b))
  for k, (o, w0, w1) in got.items():
    assert o == k % N, 'key %d on owner %d' % (k, o)
    np.testing.assert_array_max_ulp(w0.astype(np.float32),
                                    kv_doubles.init_values(table_seed, [k], dim, 0.0025, truncated=False)[0], maxulp=1)
    want = w0 - lr * grads[k] / N
    bound = 4 * 2.0 ** -24 * (np.abs(w0) + lr * np.abs(grads[k]) / N) + 2.0 ** -140
    assert (np.abs(w1 - want) <= bound).all(), 'key %d: post-step row off the float64 step' % k
