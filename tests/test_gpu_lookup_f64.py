"""GPU: the front half of the sparse path against float64 and exact references, called through the C ABI.

  er_csr_from_lens (K0)   n_seg 1, 2047..2049, 4095, 256*2048 + 1, 3*10^6; all-zero lens, one long segment; seg_ids
                          NULL; n_lookups_cap below, at and above the total (seg_ids past the cap stay untouched)
  er_bucketize[_weighted] every er_bucket_mode x shard_n 1/2/8/100 on non-uniform plans (B- and B*T-segment slots and
                          a slot with n_seg 0), single-valued and CSR with the cap below and above row_ptr[n_seg], with
                          and without weights (the mean / sqrtn prune); IDENTITY at -1, -2, nb - 1, nb and INT64_MIN;
                          mixed plans of 1, 257 and 1024 slots
  er_embedding_fwd (K2)   dims 4/8/16/32/64/128 (vector) and 1/3/6/12 (scalar), single-valued and CSR, every combiner
                          with and without weights (0, negative, NaN and denormal ones), row_stride dim and 3*dim, a
                          table base one float off (scalar fallback, bit-identical), 1 to 8 output buffers with column
                          offsets and pitches, UNIT_WEIGHTS and ONE_ROW slots weighted by raw values, uniform and
                          non-uniform plans, 2048 slots, grid-stride wrap (1.2M single segments at dim 4), the cap,
                          n_seg 0, every seg_scale entry, the refusals
  K1 -> K2 -> K7          the prune: mixed-sign mean / sqrtn segments, CSR and single-valued, every er_opt_kind, the
                          er_mark_rows + er_adam_dense_sweep pair of adam_rows, and the emit form's uniq_rows
  er_shard_group (K8)     world 1/2/8/64/65/200 x n 1/31/257/212992; whole warps of one key, owners -1 and world,
                          caps that overflow by exactly one row, repeat calls on one workspace
  er_sort_rows            n 2,621,440 / 2,621,441 / 4*10^6 (past kMaxTiles tiles) x max_row 1, 2^8, 2^8 + 1, 2^24,
                          2^32 - 2 (1 to 4 passes) x n_dev absent / below / above n, against a stable argsort

References.  Pooled values are float64 restatements of safe_embedding_lookup_sparse built from the fp32 inputs the
kernel received: ids < 0 dropped, for mean / sqrtn weights not > 0 (NaN included) dropped, sum = sum w e, mean =
sum w e / sum w, sqrtn = sum w e / sqrt(sum w^2), an empty segment gives zeros.  Each value carries a bound in
u = 2^-24: a sum of n rounded products is within n u sum|w e| of its float64 value (one u per product, (n - 1) u for
the chain), sum w within (n - 1) u sum|w|, sum w^2 within n u sum w^2; the division and the sqrt add one u each and
pass the operand errors on exactly (a / b: (ea + |a/b| eb) / (|b| - eb)).  Comparisons allow 2 times the bound plus
2^-140.  Segments where fp32 underflows (a live weight below 2^-126, or w^2 that rounds to 0) have no relative bound and
are left to the exact check below.  The header fixes the accumulation order (sequential in lookup order, no FMA), so a
float32 numpy restatement in that order must match every output bit for bit, seg_scale included.  Integer outputs
(row_ptr, seg_ids, rows, owner, send_rows, pos, counts, sorted keys and values) must match exactly.

Hygiene.  Outputs sit in NaN- or sentinel-filled buffers with guards on both sides; the pitch padding, the columns of
other slots and the rows past a slot's n_seg must keep their fill.  Table rows that only pruned, weight-dropped or
past-cap lookups point at hold NaN, as do the row_stride padding columns, so a kernel that read them would return NaN.
Every row handed to a kernel, past the cap included, is inside the table, and the caps sit below the allocated lengths.

Measured on an H100 80GB HBM3 (700 W power limit): the 180 tests run in about 11 s and the process peaks at 0.78 GiB
of reserved device memory.  Worst error / bound (0.5 means the error reached the first-order bound itself, before the
factor 2): K2 pooled values 0.500, the K7 step after K1 -> K2 0.485.
"""
import ctypes

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, kernels as K
from easyrec_b200.kernels import _p, _stream

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
C = 2.0
FLOOR = 2.0 ** -140
G = 64                      # guard elements around every output (keeps 16-byte alignment)
S32 = -0x5A5A5A5B           # sentinels of the integer outputs
S64 = -0x5A5A5A5A5A5A5A5B
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
SUM, MEAN, SQRTN = _lib.COMBINER_SUM, _lib.COMBINER_MEAN, _lib.COMBINER_SQRTN
UNIT = _lib.COMBINER_UNIT_WEIGHTS
FARM, MOD, IDENT, NONE, ONE_ROW = (_lib.BUCKET_FARM_DECIMAL, _lib.BUCKET_MOD, _lib.BUCKET_IDENTITY, _lib.BUCKET_NONE,
                                   _lib.BUCKET_ONE_ROW)
MODES = [FARM, MOD, IDENT, NONE, ONE_ROW]
MODE_IDS = ['farm', 'mod', 'identity', 'none', 'one_row']
SGD, ADAGRAD, LAZY_ADAM, ADAM_ROWS, MOMENTUM = (_lib.OPT_SGD, _lib.OPT_ADAGRAD, _lib.OPT_LAZY_ADAM, _lib.OPT_ADAM_ROWS,
                                                _lib.OPT_MOMENTUM)
KINDS = [SGD, ADAGRAD, LAZY_ADAM, ADAM_ROWS, MOMENTUM]
KIND_IDS = ['sgd', 'adagrad', 'lazy_adam', 'adam_rows', 'momentum']
B1, B2, EPS = 0.9, 0.999, 1e-8
F32 = np.float32
WORST = {}


def L():
  return _lib.load()


def _guarded(n, dtype, fill, g=G):
  buf = torch.full((n + 2 * g,), fill, dtype=dtype, device=DEV)
  return buf, buf[g:g + n]


def _same(a, b, what):
  a, b = torch.as_tensor(a), torch.as_tensor(b)
  if a.dtype.is_floating_point:
    ok = bool((a.view(torch.int32 if a.dtype == torch.float32 else torch.int64) ==
               b.view(torch.int32 if b.dtype == torch.float32 else torch.int64)).all() or
              ((a == b) | (torch.isnan(a) & torch.isnan(b))).all())
  else:
    ok = torch.equal(a, b)
  assert ok, what + ': not bit-identical'


def _guards(buf, fill, what, g=G):
  for part in (buf[:g], buf[-g:]):
    if buf.dtype.is_floating_point:
      assert bool(torch.isnan(part).all()), what + ': wrote into a guard'
    else:
      assert bool((part == fill).all()), what + ': wrote into a guard'


# ---- K0 -------------------------------------------------------------------------------------------------------------
def _csr_case(lens_np, cap, want_seg=True):
  n_seg = lens_np.size
  lens = torch.from_numpy(lens_np.astype(np.int32)).to(DEV)
  rp_buf, rp = _guarded(n_seg + 1, torch.int32, S32)
  alloc = cap + 16
  sid_buf, sid = _guarded(alloc, torch.int32, S32)
  wsb = L().er_csr_workspace_bytes(n_seg)
  ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
  _lib.check(L().er_csr_from_lens(_p(lens), n_seg, _p(rp), _p(sid) if want_seg else None, cap, _p(ws), wsb, _stream()),
             'er_csr_from_lens')
  want_rp = np.concatenate([[0], np.cumsum(lens_np, dtype=np.int64)])
  assert np.array_equal(rp.cpu().numpy(), want_rp), 'row_ptr'
  _guards(rp_buf, S32, 'row_ptr')
  got = sid.cpu().numpy()
  total = int(want_rp[-1])
  n = min(cap, total) if want_seg else 0
  want = np.full(alloc, S32, np.int64)
  want[:n] = np.repeat(np.arange(n_seg), lens_np)[:n]
  assert np.array_equal(got, want), 'seg_ids (positions past min(cap, total) must stay untouched)'
  _guards(sid_buf, S32, 'seg_ids')


@pytest.mark.parametrize('cap_rel', [-7, 0, 5], ids=['cap_below', 'cap_equal', 'cap_above'])
@pytest.mark.parametrize('n_seg', [1, 2047, 2048, 2049, 4095, 256 * 2048 + 1, 3 * 10 ** 6])
def test_csr_from_lens(n_seg, cap_rel):
  rng = np.random.default_rng(n_seg)
  lens = rng.integers(0, 4, n_seg)
  if n_seg == 1:
    lens[0] = 9
  _csr_case(lens, max(int(lens.sum()) + cap_rel, 0))


@pytest.mark.parametrize('case', ['all_zero', 'one_long', 'no_seg_ids'])
def test_csr_from_lens_edges(case):
  if case == 'all_zero':
    _csr_case(np.zeros(5000, np.int64), 3)
    _csr_case(np.zeros(5000, np.int64), 0)
  elif case == 'one_long':
    lens = np.zeros(3000, np.int64)
    lens[1234] = 700001
    _csr_case(lens, 700001)
    _csr_case(lens, 500000)
  else:
    lens = np.random.default_rng(3).integers(0, 5, 10000)
    _csr_case(lens, int(lens.sum()), want_seg=False)


# ---- K1 -------------------------------------------------------------------------------------------------------------
def _fp_mod(ids, nb):
  out = np.empty(ids.size, np.int64)
  cache = {}
  for i, (v, b) in enumerate(zip(ids.tolist(), nb.tolist())):
    h = cache.get(v)
    if h is None:
      h = cache[v] = _lib.fingerprint64(str(v))
    out[i] = h % b
  return out


def _bucket_ref(ids, seg, sl, w):
  """K1's rule restated (include/er_b200.h er_bucket_mode) -> (rows, owner)"""
  f = np.searchsorted(sl['seg_begin'], seg, side='right') - 1
  nb, off, mode = sl['num_buckets'][f], sl['row_offset'][f], sl['bucket_mode'][f]
  sn, comb = sl['shard_n'][f], sl['combiner'][f] & 0xf
  r = np.zeros(ids.size, np.int64)
  drop = np.zeros(ids.size, bool)
  m = mode == FARM
  r[m] = _fp_mod(ids[m], nb[m])
  m = mode == MOD
  r[m] = np.mod(ids[m], nb[m])
  m = mode == IDENT
  drop |= m & (ids == -1)
  r[m] = np.where((ids[m] < 0) | (ids[m] >= nb[m]), 0, ids[m])
  m = mode == NONE
  drop |= m & (ids < 0)
  r[m] = ids[m]
  m = mode == ONE_ROW
  drop |= m & (ids < 0)
  if w is not None:
    with np.errstate(invalid='ignore'):
      drop |= (comb != SUM) & ~(w > 0)
  own = np.where(sn > 1, r % sn, 0)
  r = np.where(sn > 1, r // sn, r)
  return np.where(drop, -1, off + r), np.where(drop, -1, own)


def _weights(rng, n):
  """positive, 0, negative, NaN and denormal lookup weights"""
  w = rng.uniform(0.25, 2.0, n).astype(F32)
  k = rng.integers(0, 8, n)
  w[k == 0] = 0.0
  w[k == 1] = -rng.uniform(0.1, 1.0, (k == 1).sum())
  w[k == 2] = np.nan
  w[k == 3] = F32(3e-41)
  return w


def _k1_run(ids, weights, seg_ids, row_ptr, n_seg, cap, slots_np, alloc):
  sd = K.slots_to_device(slots_np, DEV)
  t_ids = torch.from_numpy(ids).to(DEV)
  t_w = None if weights is None else torch.from_numpy(weights).to(DEV)
  t_sid = None if seg_ids is None else torch.from_numpy(seg_ids.astype(np.int32)).to(DEV)
  t_rp = None if row_ptr is None else torch.from_numpy(row_ptr.astype(np.int32)).to(DEV)
  rb, rows = _guarded(alloc, torch.int64, S64)
  ob, own = _guarded(alloc, torch.int32, S32)
  if t_w is None:
    st = L().er_bucketize(_p(t_ids), _p(t_sid), _p(t_rp), n_seg, cap, _p(sd), len(slots_np), _p(rows), _p(own),
                          _stream())
  else:
    st = L().er_bucketize_weighted(_p(t_ids), _p(t_w), _p(t_sid), _p(t_rp), n_seg, cap, _p(sd), len(slots_np),
                                   _p(rows), _p(own), _stream())
  _lib.check(st, 'er_bucketize')
  _guards(rb, S64, 'rows')
  _guards(ob, S32, 'owner')
  return rows.cpu().numpy(), own.cpu().numpy()


def _k1_check(ids, slots_np, n_seg, rng, weighted):
  """single-valued (seg_ids / row_ptr NULL) and CSR with the cap below and above row_ptr[n_seg]"""
  n = ids.size
  # single-valued: lookup l = segment l
  x = ids[:n_seg] if n >= n_seg else np.resize(ids, n_seg)
  w = _weights(rng, n_seg) if weighted else None
  rows, own = _k1_run(x, w, None, None, n_seg, n_seg, slots_np, n_seg)
  wr, wo = _bucket_ref(x, np.arange(n_seg), slots_np, w)
  assert np.array_equal(rows, wr), 'single-valued rows'
  assert np.array_equal(own, wo), 'single-valued owner'
  # CSR
  lens = rng.integers(0, 4, n_seg)
  rp = np.concatenate([[0], np.cumsum(lens)])
  total = int(rp[-1])
  seg = np.repeat(np.arange(n_seg), lens)
  x = np.resize(ids, total + 8)
  w = _weights(rng, total + 8) if weighted else None
  sid = np.concatenate([seg, np.zeros(8, np.int64)])
  for cap in (max(total - 5, 0), total + 3):
    rows, own = _k1_run(x, w, sid, rp, n_seg, cap, slots_np, total + 8)
    nl = min(cap, total)
    wr, wo = _bucket_ref(x[:nl], seg[:nl], slots_np, None if w is None else w[:nl])
    assert np.array_equal(rows[:nl], wr), 'CSR rows (cap %d of %d)' % (cap, total)
    assert np.array_equal(own[:nl], wo), 'CSR owner'
    assert (rows[nl:] == S64).all() and (own[nl:] == S32).all(), 'K1 wrote past min(cap, row_ptr[n_seg])'


def _edge_ids(nb, rng, n):
  e = np.array([-1, -2, 0, 1, nb - 1, nb, nb + 1, I64_MIN, I64_MIN + 1, I64_MAX, -nb, 2 * nb], np.int64)
  r = rng.integers(-5, 3 * nb + 5, n)
  return rng.permutation(np.concatenate([e, e, r]))


@pytest.mark.parametrize('weighted', [False, True], ids=['unweighted', 'weighted'])
@pytest.mark.parametrize('shard_n', [1, 2, 8, 100])
@pytest.mark.parametrize('mode', MODES, ids=MODE_IDS)
def test_bucketize_modes(mode, shard_n, weighted):
  """4 slots of n_seg B, B*T, 0, B (non-uniform: the binary-search branch), combiners sum / mean / sqrtn / mean"""
  rng = np.random.default_rng(mode * 100 + shard_n + 7 * weighted)
  B, T = 37, 5
  nsegs = [B, B * T, 0, B]
  nbs = [1000, 7, 1, 2 ** 40] if mode != ONE_ROW else [1, 1, 1, 1]
  offs = [0, 1000, 1007, 1008]
  recs, seg = [], 0
  for i in range(4):
    recs.append(dict(num_buckets=nbs[i], row_offset=offs[i], seg_begin=seg, n_seg=nsegs[i], bucket_mode=mode,
                     combiner=[SUM, MEAN, SQRTN, MEAN][i], out_buf=0, out_stride=64, out_col=0, shard_n=shard_n))
    seg += nsegs[i]
  sl = K.make_slots(recs)
  ids = _edge_ids(1000, rng, 600)
  if mode == NONE:
    ids = np.minimum(ids, 2 ** 40)        # (row_offset + id must not wrap)
  _k1_check(ids, sl, seg, rng, weighted)


@pytest.mark.parametrize('n_slots', [1, 257, 1024])
def test_bucketize_plans(n_slots):
  """mixed modes, bucket counts, offsets, combiners and shard counts; segments per slot cycle B, B*T, 0"""
  rng = np.random.default_rng(n_slots)
  B, T = 3, 2
  recs, seg, off = [], 0, 0
  for i in range(n_slots):
    ns = [B, B * T, 0][i % 3] if n_slots > 1 else 50
    mode = MODES[i % 5]
    nb = 1 if mode == ONE_ROW else int(rng.integers(1, 5000))
    recs.append(dict(num_buckets=nb, row_offset=off, seg_begin=seg, n_seg=ns, bucket_mode=mode,
                     combiner=[SUM, MEAN, SQRTN][i % 3], out_buf=0, out_stride=64, out_col=0,
                     shard_n=[1, 2, 8][(i // 5) % 3]))
    seg += ns
    off += nb
  sl = K.make_slots(recs)
  ids = np.minimum(_edge_ids(700, rng, 3 * seg), 2 ** 40)
  _k1_check(ids, sl, seg, rng, weighted=True)


# ---- K2: references ---------------------------------------------------------------------------------------------------
def _pool_f32(table, rows, w, rp, cap, comb_seg, single):
  """the kernel's order restated in float32: (pooled [n_seg, dim], seg_scale [n_seg])"""
  n_seg = comb_seg.size
  dim = table.shape[1]
  acc = np.zeros((n_seg, dim), F32)
  scale = np.zeros(n_seg, F32)
  is_sum = comb_seg == SUM
  with np.errstate(invalid='ignore', divide='ignore', over='ignore', under='ignore'):
    if single:
      r = rows[:n_seg]
      ww = np.ones(n_seg, F32) if w is None else w[:n_seg]
      keep = (r >= 0) & (is_sum | (ww > 0))
      v = table[np.where(keep, r, 0)]
      o = v * ww[:, None] if w is not None else v.copy()
      mean, sq = keep & (comb_seg == MEAN), keep & (comb_seg == SQRTN)
      o[mean] = o[mean] / ww[mean, None]
      scale[mean] = F32(1) / ww[mean]
      d = np.sqrt(ww * ww)
      sqz = sq & (d != 0)
      o[sqz] = o[sqz] / d[sqz, None]
      scale[sqz] = F32(1) / d[sqz]
      o[~keep | (sq & (d == 0))] = 0
      scale[is_sum] = 1
      return o, scale
    b = rp[:-1].astype(np.int64)
    e = np.minimum(rp[1:].astype(np.int64), cap)
    n = np.maximum(e - b, 0)
    wsum = np.zeros(n_seg, F32)
    w2 = np.zeros(n_seg, F32)
    for j in range(int(n.max()) if n_seg else 0):
      s = np.nonzero(n > j)[0]
      idx = b[s] + j
      r = rows[idx]
      ww = np.ones(s.size, F32) if w is None else w[idx]
      live = (r >= 0) & (is_sum[s] | (ww > 0))
      s, r, ww = s[live], r[live], ww[live]
      v = table[r]
      acc[s] = acc[s] + (v * ww[:, None] if w is not None else v)
      wsum[s] = wsum[s] + ww
      w2[s] = w2[s] + ww * ww
    scale[:] = 1
    for cm, den in ((MEAN, wsum), (SQRTN, np.sqrt(w2))):
      m = comb_seg == cm
      nz = m & (den != 0)
      acc[nz] = acc[nz] / den[nz, None]
      scale[nz] = F32(1) / den[nz]
      acc[m & (den == 0)] = 0
      scale[m & (den == 0)] = 0
  return acc, scale


def _pool_f64(table, rows, w, rp, cap, comb_seg, single):
  """safe_embedding_lookup_sparse in float64 -> (value, bound, checkable segments)"""
  n_seg = comb_seg.size
  if single:
    rp = np.arange(n_seg + 1)
    cap = n_seg
  b = rp[:-1].astype(np.int64)
  e = np.minimum(rp[1:].astype(np.int64), cap)
  n_l = int(e.max()) if n_seg else 0
  cnts = np.maximum(e - b, 0)
  seg = np.repeat(np.arange(n_seg), cnts)
  idx = np.repeat(b, cnts) + np.arange(seg.size) - np.repeat(np.cumsum(cnts) - cnts, cnts)
  assert idx.size == 0 or idx.max() < n_l
  r = rows[idx]
  ww = np.ones(idx.size) if w is None else w[idx].astype(np.float64)
  with np.errstate(invalid='ignore'):
    live = (r >= 0) & ((comb_seg[seg] == SUM) | (ww > 0))
  seg, r, ww = seg[live], r[live], ww[live]
  t = torch.from_numpy(table[r].astype(np.float64) * ww[:, None]).to(DEV)
  sg = torch.from_numpy(seg).to(DEV)
  z = torch.zeros(n_seg, table.shape[1], dtype=torch.float64, device=DEV)
  S = z.index_add(0, sg, t)
  A = z.index_add(0, sg, t.abs())
  z1 = torch.zeros(n_seg, dtype=torch.float64, device=DEV)
  tw = torch.from_numpy(ww).to(DEV)
  W = z1.index_add(0, sg, tw)
  WA = z1.index_add(0, sg, tw.abs())
  Q = z1.index_add(0, sg, tw * tw)
  cnt = z1.index_add(0, sg, torch.ones_like(tw))
  tiny = torch.from_numpy((np.abs(ww) < 2.0 ** -126) & (ww != 0)).to(DEV)
  bad = z1.index_add(0, sg, tiny.double()) > 0
  eS = cnt[:, None] * U * A
  comb = torch.from_numpy(comb_seg).to(DEV)
  val, err = S.clone(), eS.clone()
  ok = ~bad
  for cm in (MEAN, SQRTN):
    m = (comb == cm) & (cnt > 0)
    if cm == MEAN:
      d, ed = W, (cnt - 1).clamp_min(0) * U * WA
    else:
      eQ = cnt * U * Q
      d = Q.sqrt()
      ed = d - (Q - eQ).clamp_min(0).sqrt() + U * d
    ok &= ~m | (d - ed > 0) & (Q > 2.0 ** -120)
    dd = torch.where(m, d, torch.ones_like(d))[:, None]
    edd = torch.where(m, ed, torch.zeros_like(ed))[:, None]
    v = S / dd
    e_ = (eS + v.abs() * edd) / (dd - edd).clamp_min(1e-300) + U * v.abs()
    val = torch.where(m[:, None], v, val)
    err = torch.where(m[:, None], e_, err)
  return val, err, ok


# ---- K2: cases --------------------------------------------------------------------------------------------------------
VEC = (4, 8, 16, 32, 64, 128)


class Pool(object):
  """A K2 call: slots cycling over combiners (one UNIT_WEIGHTS slot, one ONE_ROW slot weighted by raw values), n_bufs
  NaN-filled output matrices with pitch padding and gaps between the slots' columns, a table with NaN rows that only
  pruned / past-cap lookups point at and NaN padding columns, lookups past the cap."""

  def __init__(self, dim, single, weighted, stride_mult=1, n_bufs=3, n_slots=6, B=40, T=3, uniform=False, seed=0,
               n_seg_per_slot=None, table_shift=0, max_len=5):
    rng = np.random.default_rng(seed)
    self.dim, self.single, self.weighted = dim, single, weighted
    V, P = 900, 64
    self.V = V
    self.n_rows = V + P
    vec = dim in VEC
    # ---- plan
    recs, seg = [], 0
    cols = [0] * n_bufs
    gap = 4 if vec else 1
    self.slot_info = []
    for i in range(n_slots):
      ns = (n_seg_per_slot or B) if uniform else [B, B * T, B, 0][i % 4]
      comb = [SUM, MEAN, SQRTN][i % 3]
      one_row = (i % 6 == 3) and weighted
      if one_row:
        comb = SUM
      unit = (i % 6 == 4) and weighted
      buf = i % n_bufs
      recs.append(dict(num_buckets=1 if one_row else V, row_offset=0, seg_begin=seg, n_seg=ns,
                       bucket_mode=ONE_ROW if one_row else NONE, combiner=comb | (UNIT if unit else 0), out_buf=buf,
                       out_stride=0, out_col=cols[buf], shard_n=1))
      self.slot_info.append((one_row, unit))
      cols[buf] += dim + gap * ((i // n_bufs) % 2)
      seg += ns
    self.strides = [-(-(c + gap + 1) // 4) * 4 if vec else c + gap + 1 for c in cols]
    self.buf_rows = [max([r['n_seg'] for r in recs if r['out_buf'] == b] + [1]) for b in range(n_bufs)]
    for r in recs:
      r['out_stride'] = self.strides[r['out_buf']]
    self.recs = recs
    self.slots_np = K.make_slots(recs, dim)
    self.sd = K.slots_to_device(self.slots_np, DEV)
    self.n_seg = seg
    comb_seg = np.concatenate([np.full(r['n_seg'], r['combiner'] & 0xf) for r in recs] + [np.zeros(0, np.int64)])
    self.comb_seg = comb_seg.astype(np.int64)
    # ---- table: rows V.. are NaN (only dead lookups point there); the row_stride padding is NaN too
    self.row_stride = dim * stride_mult
    stor = torch.full((self.n_rows * self.row_stride + 8,), float('nan'), device=DEV)
    self.table_full = stor[table_shift:table_shift + self.n_rows * self.row_stride].view(self.n_rows, self.row_stride)
    vals = rng.normal(size=(V, dim)).astype(F32)
    self.table_full[:V, :dim] = torch.from_numpy(vals).to(DEV)
    self.table = self.table_full[:, :dim]
    self.table_np = self.table_full[:, :dim].cpu().numpy()
    # ---- lookups
    seg_slot = np.repeat(np.arange(n_slots), [r['n_seg'] for r in recs])
    if single:
      lens = np.ones(seg, np.int64)
    else:
      lens = rng.integers(0, max_len + 1, seg)
      if seg > 10:
        lens[rng.integers(0, seg, 3)] = 37     # long segments: several rounds of the unrolled loop
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    total = int(rp[-1])
    self.total = total
    self.cap = total if single else max(total - int(lens[-8:].sum()) - 3, 0)
    n_alloc = total + 8
    lk_slot = seg_slot[np.repeat(np.arange(seg), lens)] if seg else np.zeros(0, np.int64)
    lk_slot = np.concatenate([lk_slot, np.zeros(8, np.int64)])
    comb_l = self.comb_seg[np.repeat(np.arange(seg), lens)] if seg else np.zeros(0, np.int64)
    comb_l = np.concatenate([comb_l, np.full(8, MEAN)])
    rows = rng.integers(0, V, n_alloc)
    rows[rng.random(n_alloc) < 0.05] = -1
    if weighted:
      w = rng.normal(size=n_alloc).astype(F32)
      k = rng.integers(0, 10, n_alloc)
      w[k == 0] = 0.0
      w[k == 1] = F32(2e-40)
      pos = comb_l != SUM
      w[pos] = np.abs(w[pos]) + F32(0.25)
      kk = rng.integers(0, 10, n_alloc)
      w[pos & (kk == 0)] = 0.0
      w[pos & (kk == 1)] = -0.5
      w[pos & (kk == 2)] = np.nan
      w[pos & (kk == 3)] = F32(3e-39)
      for i, (one_row, unit) in enumerate(self.slot_info):
        m = lk_slot[:total] == i
        idx = np.nonzero(m)[0]
        if one_row:
          rows[idx] = V - 1
          w[idx] = rng.normal(size=idx.size).astype(F32) * 3
          w[idx[::5]] = 0.0
        if unit:
          w[idx] = 1.0
      with np.errstate(invalid='ignore'):
        dead = (comb_l != SUM) & ~(w > 0)
      rows[dead & (rows >= 0)] = V + rng.integers(0, P, int((dead & (rows >= 0)).sum()))
    else:
      w = None
    past = np.arange(n_alloc) >= self.cap
    rows[past] = V + rng.integers(0, P, int(past.sum()))
    if w is not None:
      w[past] = np.nan
    self.rows_np, self.w_np, self.rp_np = rows, w, rp
    self.rows = torch.from_numpy(rows).to(DEV)
    self.w = None if w is None else torch.from_numpy(w).to(DEV)
    self.rp = None if single else torch.from_numpy(rp.astype(np.int32)).to(DEV)

  def run(self, table=None, n_seg=None):
    n_seg = self.n_seg if n_seg is None else n_seg
    table = self.table if table is None else table
    # guards of at least one output row: a segment given the previous slot lands in them, not outside the buffer
    g = G + -(-max(self.strides) // 4) * 4
    outs = [_guarded(r * s, torch.float32, float('nan'), g) for r, s in zip(self.buf_rows, self.strides)]
    sb, sc = _guarded(max(self.n_seg, 1), torch.float32, float('nan'))
    arr = (ctypes.c_void_p * len(outs))(*[o[1].data_ptr() for o in outs])
    cap = n_seg if self.single else self.cap
    st = L().er_embedding_fwd(table.data_ptr(), self.n_rows, self.dim, table.stride(0), _p(self.rows), _p(self.w),
                              _p(self.rp), n_seg, cap, _p(self.sd), len(self.recs), arr, len(outs), sc.data_ptr(),
                              _stream())
    _lib.check(st, 'er_embedding_fwd')
    for b, _ in outs:
      _guards(b, None, 'K2 output', g)
    _guards(sb, None, 'seg_scale')
    return [o[1].view(r, s) for o, r, s in zip(outs, self.buf_rows, self.strides)], sc

  def expected(self):
    pooled, scale = _pool_f32(self.table_np, self.rows_np, self.w_np, self.rp_np, self.cap, self.comb_seg,
                              self.single)
    bufs = [np.full((r, s), np.nan, F32) for r, s in zip(self.buf_rows, self.strides)]
    for r in self.recs:
      sb = r['seg_begin']
      bufs[r['out_buf']][:r['n_seg'], r['out_col']:r['out_col'] + self.dim] = pooled[sb:sb + r['n_seg']]
    return bufs, scale

  def check(self, outs, sc, what):
    bufs, scale = self.expected()
    for i, (g, e) in enumerate(zip(outs, bufs)):
      _same(g, torch.from_numpy(e).to(DEV), '%s: buffer %d against the float32 restatement' % (what, i))
    _same(sc, torch.from_numpy(scale).to(DEV), what + ': seg_scale')
    # float64 semantics of every slot's segments
    val, err, ok = _pool_f64(self.table_np, self.rows_np, self.w_np, self.rp_np, self.cap, self.comb_seg, self.single)
    got = torch.empty_like(val)
    for r in self.recs:
      sb, ns = r['seg_begin'], r['n_seg']
      got[sb:sb + ns] = outs[r['out_buf']][:ns, r['out_col']:r['out_col'] + self.dim].double()
    e = (got - val).abs()[ok]
    bound = C * err[ok] + FLOOR
    assert bool(torch.isfinite(got[ok]).all()), what + ': non-finite pooled value'
    ratio = float((e / bound).max()) if e.numel() else 0.0
    WORST['K2'] = max(WORST.get('K2', 0.0), ratio)
    assert ratio <= 1.0, '%s: error %.3g x the float64 bound' % (what, ratio)


@pytest.mark.parametrize('weighted', [False, True], ids=['unweighted', 'weighted'])
@pytest.mark.parametrize('path', ['single', 'csr'])
@pytest.mark.parametrize('dim', [4, 8, 16, 32, 64, 128, 1, 3, 6, 12])
def test_pool_dims(dim, path, weighted):
  """every dim on both paths; row_stride 3*dim on every other dim; a non-uniform plan over 3 buffers"""
  stride_mult = 3 if dim in (4, 32, 128, 3, 12) else 1
  p = Pool(dim, path == 'single', weighted, stride_mult=stride_mult, seed=dim * 10 + (path == 'single') + 2 * weighted)
  outs, sc = p.run()
  p.check(outs, sc, 'K2 dim %d %s' % (dim, path))


@pytest.mark.parametrize('path', ['single', 'csr'])
@pytest.mark.parametrize('dim', [4, 16, 128])
def test_pool_table_offset_scalar_fallback(dim, path):
  """a table base one float off 16 bytes takes the scalar kernel: bit-identical to the vector kernel"""
  p0 = Pool(dim, path == 'single', True, seed=77 + dim)
  p1 = Pool(dim, path == 'single', True, seed=77 + dim, table_shift=1)
  assert p1.table.data_ptr() % 16 == 4
  o0, s0 = p0.run()
  o1, s1 = p1.run()
  for a, b in zip(o0, o1):
    _same(a, b, 'scalar fallback against the vector path')
  _same(s0, s1, 'scalar fallback seg_scale')
  p1.check(o1, s1, 'K2 offset table dim %d' % dim)


@pytest.mark.parametrize('n_bufs', [1, 2, 3, 4, 5, 6, 7, 8])
def test_pool_buffers(n_bufs):
  for path in ('single', 'csr'):
    p = Pool(16, path == 'single', True, n_bufs=n_bufs, n_slots=2 * n_bufs + 1, seed=300 + n_bufs)
    outs, sc = p.run()
    p.check(outs, sc, 'K2 %d buffers %s' % (n_bufs, path))


@pytest.mark.parametrize('dim', [16, 6])
@pytest.mark.parametrize('path', ['single', 'csr'])
def test_pool_uniform_plan(path, dim):
  """every slot B segments: the multiply-shift slot lookup"""
  p = Pool(dim, path == 'single', True, n_slots=7, uniform=True, seed=400 + dim)
  outs, sc = p.run()
  p.check(outs, sc, 'K2 uniform %s' % path)


@pytest.mark.parametrize('path', ['single', 'csr'])
def test_pool_2048_slots(path):
  p = Pool(4, path == 'single', True, n_bufs=8, n_slots=2048, B=2, T=2, seed=501)
  outs, sc = p.run()
  p.check(outs, sc, 'K2 2048 slots %s' % path)


def test_pool_grid_stride_wrap():
  """1.2M single segments at dim 4 (more than the grid covers in one sweep), and 600K CSR segments"""
  p = Pool(4, True, True, n_bufs=2, n_slots=2, uniform=True, n_seg_per_slot=600000, seed=601)
  outs, sc = p.run()
  p.check(outs, sc, 'K2 single wrap')
  p = Pool(4, False, True, n_bufs=2, n_slots=3, uniform=True, n_seg_per_slot=200000, seed=602, max_len=2)
  outs, sc = p.run()
  p.check(outs, sc, 'K2 csr wrap')


def test_pool_zero_segments():
  p = Pool(16, False, True, seed=7)
  outs, sc = p.run(n_seg=0)
  for o in outs:
    assert bool(torch.isnan(o).all()), 'n_seg 0 wrote an output'
  assert bool(torch.isnan(sc).all()), 'n_seg 0 wrote seg_scale'


def test_pool_refusals():
  p = Pool(16, False, True, seed=8)
  outs = [torch.empty(p.buf_rows[b] * p.strides[b], device=DEV) for b in range(3)]
  arr = (ctypes.c_void_p * 9)(*([o.data_ptr() for o in outs] * 3))
  t, d = p.table, 16

  def call(table=t.data_ptr(), n_rows=p.n_rows, dim=d, rs=t.stride(0), rows=_p(p.rows), rp=_p(p.rp), n_seg=p.n_seg,
           cap=p.cap, n_slots=len(p.recs), bufs=arr, n_bufs=3):
    return L().er_embedding_fwd(table, n_rows, dim, rs, rows, _p(p.w), rp, n_seg, cap, _p(p.sd), n_slots, bufs, n_bufs,
                                None, _stream())

  bad = [dict(table=None), dict(rows=None), dict(bufs=None), dict(dim=0), dict(rs=8), dict(n_rows=0),
         dict(n_slots=0), dict(n_slots=2049), dict(n_bufs=0), dict(n_bufs=9), dict(n_seg=-1), dict(n_seg=2 ** 31),
         dict(rp=None)]
  for kw in bad:
    assert call(**kw) == _lib.ER_ERR_INVALID_ARG, kw
  nul = (ctypes.c_void_p * 3)(outs[0].data_ptr(), None, outs[2].data_ptr())
  assert call(bufs=nul) == _lib.ER_ERR_INVALID_ARG
  torch.cuda.synchronize()


# ---- K1 -> K2 -> K7: the prune ----------------------------------------------------------------------------------------
class R(object):
  def __init__(self, v, e=None):
    self.v = v
    self.e = torch.zeros_like(v) if e is None else e


def X(t):
  if not torch.is_tensor(t):
    t = torch.tensor(float(F32(t)), dtype=torch.float64, device=DEV)
  return R(t.double())


def _rnd(v, e):
  return R(v, e + U * v.abs())


def add(a, b):
  return _rnd(a.v + b.v, a.e + b.e)


def sub(a, b):
  return _rnd(a.v - b.v, a.e + b.e)


def mul(a, b):
  return _rnd(a.v * b.v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e)


def div(a, b):
  v = a.v / b.v
  lo = b.v.abs() - b.e
  assert bool((lo > 0).all())
  return _rnd(v, (a.e + v.abs() * b.e) / lo)


def sqrt(a):
  v = a.v.sqrt()
  return _rnd(v, v - (a.v - a.e).clamp_min(0.0).sqrt())


def rsqrt(a):
  v = a.v.rsqrt()
  return _rnd(v, (a.v - a.e).rsqrt() - v)


def rule(kind, w, s0, s1, g, lr):
  """TF's row rules as er_embedding_bwd applies them (see test_gpu_optimizer_f64.py)"""
  if kind == ADAGRAD:
    s0 = add(s0, mul(g, g))
    w = sub(w, mul(mul(lr, g), rsqrt(s0)))
  elif kind in (LAZY_ADAM, ADAM_ROWS):
    s0 = add(mul(g, sub(X(1.0), X(B1))), mul(s0, X(B1)))
    s1 = add(mul(mul(g, g), sub(X(1.0), X(B2))), mul(s1, X(B2)))
    w = sub(w, div(mul(lr, s0), add(sqrt(s1), X(EPS))))
  elif kind == MOMENTUM:
    s0 = add(mul(s0, X(B1)), g)
    w = sub(w, mul(lr, s0))
  else:
    w = sub(w, mul(lr, g))
  return w, s0, s1


def _within(got, ref, what):
  err = (got.double() - ref.v).abs()
  bound = C * ref.e + FLOOR
  assert bool(torch.isfinite(got).all()), what + ': non-finite'
  ratio = float((err / bound).max()) if err.numel() else 0.0
  WORST['K7'] = max(WORST.get('K7', 0.0), ratio)
  assert ratio <= 1.0, '%s: error %.3g x bound' % (what, ratio)


@pytest.mark.parametrize('path', ['csr', 'single'])
@pytest.mark.parametrize('kind', KINDS, ids=KIND_IDS)
def test_prune_k1_k2_k7(kind, path):
  """Mean and sqrtn segments mixing weights > 0 with weights 0, < 0 and NaN (and a sum slot whose negative weights are
  kept).  Rows 300..339 are reached only by lookups safe_embedding_lookup_sparse prunes, and some pruned lookups also
  point at live rows.  After K1 (given the weights) -> K2 -> K7, the pruned-only rows are bit-identical to their input
  (for adam_rows: they take er_adam_dense_sweep's decay, as TF's dense Adam gives them), every other row matches a
  float64 step over the surviving lookups only, and the emit form's uniq_rows leaves the pruned-only rows out."""
  rng = np.random.default_rng(40 + kind + 10 * (path == 'single'))
  dim, V, B = 8, 400, 96
  single = path == 'single'
  combs = [MEAN, SQRTN, SUM]
  recs = [dict(num_buckets=V, row_offset=0, seg_begin=f * B, n_seg=B, bucket_mode=NONE, combiner=combs[f], out_buf=0,
               out_stride=3 * dim, out_col=f * dim) for f in range(3)]
  sl = K.make_slots(recs, dim)
  sd = K.slots_to_device(sl, DEV)
  n_seg = 3 * B
  lens = np.ones(n_seg, np.int64) if single else rng.integers(1, 5, n_seg)
  rp = np.concatenate([[0], np.cumsum(lens)])
  n = int(rp[-1])
  seg = np.repeat(np.arange(n_seg), lens)
  ids = rng.integers(0, 300, n)
  w = rng.uniform(0.25, 2.0, n).astype(F32)
  bad = rng.random(n) < (0.4 if single else 0.3)
  w[bad] = rng.choice(np.array([0.0, -0.5, np.nan, -1e-3], F32), int(bad.sum()))
  w[(seg >= 2 * B) & np.isnan(w)] = -2.0                # (a sum slot keeps every weight: no NaN there)
  pruned = bad & (seg < 2 * B)
  to_p = pruned & (rng.random(n) < 0.7)
  ids[to_p] = rng.integers(300, 340, int(to_p.sum()))   # rows only pruned lookups reach
  ids[seg >= 2 * B] = np.minimum(ids[seg >= 2 * B], 299)
  ids[rng.random(n) < 0.03] = -1
  t_ids = torch.from_numpy(ids).to(DEV)
  t_w = torch.from_numpy(w).to(DEV)
  rp_t = None if single else torch.from_numpy(rp.astype(np.int32)).to(DEV)
  sid_t = None if single else torch.from_numpy(seg.astype(np.int32)).to(DEV)
  rows = K.bucketize(t_ids, sd, 3, n_seg, seg_ids=sid_t, row_ptr=rp_t, weights=t_w)
  want_rows, _ = _bucket_ref(ids, seg, sl, w)
  assert np.array_equal(rows.cpu().numpy(), want_rows), 'K1 rows'
  live = want_rows >= 0
  assert not np.isin(np.arange(300, 340), want_rows[live]).any()
  gen = torch.Generator(device=DEV).manual_seed(kind)
  table = torch.randn(V, dim, generator=gen, device=DEV) * 0.5
  st = [None, None]
  if kind in (ADAGRAD, MOMENTUM, LAZY_ADAM, ADAM_ROWS):
    st[0] = torch.rand(V, dim, generator=gen, device=DEV) * 0.2 + 0.05
  if kind in (LAZY_ADAM, ADAM_ROWS):
    st[1] = torch.rand(V, dim, generator=gen, device=DEV) * 0.2 + 1e-3
  init = [table.clone()] + [None if s is None else s.clone() for s in st]
  out = torch.full((B, 3 * dim), float('nan'), device=DEV)
  scale = torch.full((n_seg,), float('nan'), device=DEV)
  K.embedding_fwd(table, dim, rows, sd, 3, n_seg, [out], weights=t_w, row_ptr=rp_t, seg_scale=scale)
  assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(scale).all())
  gout = torch.randn(B, 3 * dim, generator=gen, device=DEV)
  lr, b1p, b2p = 0.05, float(F32(B1 ** 3)), float(F32(B2 ** 3))
  opt = K.make_opt(kind, lr, B1, B2, EPS, b1p, b2p, 1.0)
  K.embedding_bwd(table, st[0], st[1], dim, rows, sd, 3, n_seg, [gout], opt, K.bwd_workspace(n, DEV, dim), weights=t_w,
                  seg_ids=sid_t, row_ptr=rp_t, seg_scale=scale)
  if kind == ADAM_ROWS:
    touched = torch.zeros(V, dtype=torch.uint8, device=DEV)
    K.mark_rows(rows, V, touched, 1)
    K.adam_dense_sweep(table, st[0], st[1], dim, touched, opt)
  got = [table, st[0], st[1]]
  # reference: G[row] = sum over the SURVIVING lookups of gout[segment] * w * seg_scale[segment]
  lv = torch.from_numpy(np.nonzero(live)[0]).to(DEV)
  sg = torch.from_numpy(seg).to(DEV)[lv]
  r = rows[lv]
  f, b = sg // B, sg % B
  gv = gout[b[:, None], f[:, None] * dim + torch.arange(dim, device=DEV)[None, :]]
  coef = mul(X(t_w[lv]), X(scale[sg]))
  term = mul(X(gv), R(coef.v[:, None], coef.e[:, None]))
  z = torch.zeros(V, dim, dtype=torch.float64, device=DEV)
  cnt = torch.zeros(V, dtype=torch.float64, device=DEV).index_add(0, r, torch.ones_like(r, dtype=torch.float64))
  Gs = R(z.index_add(0, r, term.v), z.index_add(0, r, term.e) +
         (cnt - 1).clamp_min(0)[:, None] * U * z.index_add(0, r, term.v.abs()))
  uniq = torch.unique(r)
  lr0 = (div(mul(X(lr), sqrt(sub(X(1.0), X(b2p)))), sub(X(1.0), X(b1p))) if kind in (LAZY_ADAM, ADAM_ROWS) else X(lr))
  gu = R(Gs.v[uniq], Gs.e[uniq])
  ref = rule(kind, X(init[0][uniq]), None if init[1] is None else X(init[1][uniq]),
             None if init[2] is None else X(init[2][uniq]), gu, lr0)
  n_st = {SGD: 0, ADAGRAD: 1, MOMENTUM: 1, LAZY_ADAM: 2, ADAM_ROWS: 2}[kind]
  rest = torch.ones(V, dtype=torch.bool, device=DEV)
  rest[uniq] = False
  for i in range(1 + n_st):
    _within(got[i][uniq], ref[i], 'prune %s %s: live rows [%d]' % (KIND_IDS[kind], path, i))
  if kind == ADAM_ROWS:
    rr = rest.nonzero().flatten()
    mm = mul(X(init[1][rr]), X(B1))
    vv = mul(X(init[2][rr]), X(B2))
    ww = sub(X(init[0][rr]), div(mul(lr0, mm), add(sqrt(vv), X(EPS))))
    for i, refv in enumerate((ww, mm, vv)):
      _within(got[i][rr], refv, 'prune adam_rows %s: untouched rows take the dense decay [%d]' % (path, i))
  else:
    moved = torch.zeros(V, dtype=torch.bool, device=DEV)
    for i in range(1 + n_st):
      moved |= (got[i] != init[i]).any(1)
    moved &= rest
    assert not bool(moved.any()), 'prune %s %s: %d rows no surviving lookup reaches moved (%d of them only pruned ' \
        'lookups reach)' % (KIND_IDS[kind], path, int(moved.sum()), int(moved[300:340].sum()))
  # the emit form: uniq_rows = the distinct rows of the surviving lookups
  ur = torch.full((n,), -7, dtype=torch.int64, device=DEV)
  ug = torch.full((n, dim), float('nan'), device=DEV)
  nu = torch.full((1,), -1, dtype=torch.int32, device=DEV)
  K.embedding_bwd(None, None, None, dim, rows, sd, 3, n_seg, [gout], K.make_opt(SGD, 0.1),
                  K.bwd_workspace(n, DEV, dim), weights=t_w, seg_ids=sid_t, row_ptr=rp_t, seg_scale=scale,
                  uniq_rows=ur, uniq_grads=ug, n_uniq=nu, n_rows=V)
  k = int(nu.item())
  assert torch.equal(ur[:k], uniq), 'emit uniq_rows'


# ---- K8 -------------------------------------------------------------------------------------------------------------
def _shard_case(world, n, seed):
  rng = np.random.default_rng(seed)
  nr = max(4, n // 6)
  rows = rng.integers(0, nr, n)
  owner = rng.integers(0, world, n)
  if n >= 31:
    rows[rng.integers(0, n, max(1, n // 20))] = -1
    k = rng.integers(0, n, max(2, n // 20))
    owner[k[::2]] = -1
    owner[k[1::2]] = world                # outside [0, world): not counted, pos -1
  if n >= 96:
    rows[32:64], owner[32:64] = 3, 0      # a whole warp of one key
    rows[64:96], owner[64:96] = rows[64], owner[64]
  return rows.astype(np.int64), owner.astype(np.int64)


def _shard_check(rows, owner, world, cap, send, pos, counts):
  live = (rows >= 0) & (owner >= 0) & (owner < world)
  keys = owner[live] * (1 << 40) + rows[live]
  uk = np.unique(keys)
  cnt = np.bincount(uk >> 40, minlength=world)[:world]
  assert np.array_equal(counts[:world], cnt), 'counts[o] must be the distinct rows of owner o'
  assert (pos[~live] == -1).all(), 'a dropped lookup or an owner outside [0, world) got a position'
  p = pos[live]
  ok = p >= 0
  assert (send[p[ok]] == rows[live][ok]).all(), 'send_rows[pos[l]] != rows[l]'
  assert (p[ok] // cap == owner[live][ok]).all(), 'position outside the owner block'
  pairs = np.unique(np.stack([keys, p], 1), axis=0)
  assert pairs.shape[0] == uk.size, 'lookups of one key got different positions'
  assert np.unique(p[ok]).size == np.minimum(cnt, cap).sum(), 'positions claimed'
  assert (~ok).sum() == counts[world], 'counts[world] must be the number of lost lookups'
  lost_keys = np.unique(keys[~ok]).size
  assert lost_keys == np.maximum(cnt - cap, 0).sum(), 'rows lost to a full block'
  blk = send.reshape(world, cap)
  m = np.minimum(cnt, cap)
  filled = np.arange(cap)[None, :] < m[:, None]
  assert (blk[filled] >= 0).all() and (blk[~filled] == -1).all(), 'send_rows blocks: rows first, -1 padding'


@pytest.mark.parametrize('n', [1, 31, 257, 212992])
@pytest.mark.parametrize('world', [1, 2, 8, 64, 65, 200])
def test_shard_group(world, n):
  rows, owner = _shard_case(world, n, world * 1000 + n)
  live = (rows >= 0) & (owner >= 0) & (owner < world)
  cnt = np.bincount(np.unique(owner[live] * (1 << 40) + rows[live]) >> 40, minlength=world)[:world]
  mx = int(cnt.max()) if cnt.size else 0
  caps = [max(mx, 1)] + ([mx - 1] if mx >= 2 else [])   # exact fit, and one row over in the fullest block
  t_rows, t_own = torch.from_numpy(rows).to(DEV), torch.from_numpy(owner.astype(np.int32)).to(DEV)
  ws = K.shard_group_workspace(n, DEV)
  for cap in caps:
    for rep in range(2):                                # the same workspace twice
      sb, send = _guarded(world * cap, torch.int64, S64)
      pb, pos = _guarded(n, torch.int64, S64)
      cb, counts = _guarded(world + 1, torch.int32, S32)
      _lib.check(L().er_shard_group(_p(t_rows), _p(t_own), n, world, cap, _p(send), _p(pos), _p(counts), _p(ws),
                                    ws.numel(), _stream()), 'er_shard_group')
      for b, s, nm in ((sb, S64, 'send_rows'), (pb, S64, 'pos'), (cb, S32, 'counts')):
        _guards(b, s, nm)
      c = counts.cpu().numpy()
      _shard_check(rows, owner, world, cap, send.cpu().numpy(), pos.cpu().numpy(), c)
      if cap == mx:
        assert c[world] == 0


# ---- er_sort_rows ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('max_row', [1, 2 ** 8, 2 ** 8 + 1, 2 ** 24, 2 ** 32 - 2])
@pytest.mark.parametrize('n', [2621440, 2621441, 4 * 10 ** 6])
def test_sort_rows(n, max_row):
  """keys = the row (the sentinel max_row for rows < 0, >= max_row or at positions >= n_dev), sorted ascending; vals =
  original positions, stable"""
  gen = torch.Generator(device=DEV).manual_seed(n + max_row)
  rows = torch.randint(-2, max_row + 3, (n,), generator=gen, device=DEV, dtype=torch.int64)
  wsb = L().er_sort_workspace_bytes(n)
  ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
  kb, keys = _guarded(n, torch.int32, S32)
  vb, vals = _guarded(n, torch.int32, S32)
  idx = torch.arange(n, device=DEV)
  for n_dev in (None, n - 1000, n + 5):
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device=DEV)
    _lib.check(L().er_sort_rows(_p(rows), n, _p(nd), max_row, _p(keys), _p(vals), _p(ws), wsb, _stream()),
               'er_sort_rows')
    live = (rows >= 0) & (rows < max_row) & (idx < min(n if n_dev is None else n_dev, n))
    k = torch.where(live, rows, torch.full_like(rows, max_row))
    sk, order = torch.sort(k, stable=True)
    assert torch.equal(keys.long() & 0xFFFFFFFF, sk), 'sorted keys (n_dev %s)' % n_dev
    assert torch.equal(vals.long(), order), 'stable positions (n_dev %s)' % n_dev
    _guards(kb, S32, 'keys')
    _guards(vb, S32, 'vals')


def test_zz_report_worst():
  print('worst error / bound: %s' % ', '.join('%s %.3f' % kv for kv in sorted(WORST.items())))
