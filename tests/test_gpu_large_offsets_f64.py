"""GPU: the sparse kernels on table rows whose float offsets row * row_stride + col pass 2^31 and 2^32, against float64,
against a compact twin, and on aliased device memory (tests/aliased_arena.py: a virtual table of up to 2^32 - 2 rows on
one small physical chunk, every physical word outside the rows' images a sentinel).

  rows          per (dim, row_stride): the rows from two below to two above the one holding float 2^31 and float 2^32
                (with row_stride 3, 9, 12, 48 or 192 one of them runs across the boundary), rows 2^31 - 1 / 2^31 /
                2^31 + 1 at dims 1 and 3, n_rows - 1 (n_rows = 2^32 - 2 at row_stride 1 and 2), and 16 low rows
  er_embedding_fwd (K2)   dims 4/16/64 (vector) and 1/3/6 (scalar) x row_stride dim and 3 dim x single-valued and CSR,
                          sum / mean / sqrtn slots, weights; each high row looked up many times among low rows
  er_embedding_bwd (K7)   every er_opt_kind x separate arrays and [w | state0 | state1] rows x dims 1/3/4/16/64; runs of
                          1 .. 5000 lookups of high rows (warp, CTA, coop > 48, big-bucket > 1024 and hot-row > 4096
                          paths, each asserted reached) and a one-row slot whose row_offset is a high row; also through
                          er_embedding_bwd_presort + er_embedding_bwd_reuse_sort
  emit + er_sparse_apply  the radix engine at n_rows = table rows (up to 2^32 - 2: four sort passes): uniq_rows exactly the
                          high rows, uniq_grads against float64 G, then the owner-side update from that G
  er_mark_rows            an aliased touched mask of 2^32 - 2 bytes, rows 2^31 - 1 .. 2^32 - 3, exact
  er_shard_group (K8)     rows at and above 2^32, up to (2^63 - 1) // world (the largest owner-local row K1 makes from
                          an int64 id), world 2 / 3 / 8, against Python integers
  er_adam_dense_sweep     a real [w | m | v] table just past 2^31 floats (dim 4, row_stride 12: the vector kernel; dim 3,
                          row_stride 9: the scalar kernel), moments on the rows across 2^31 and the last rows
  sensitivity             K2 and K7 handed the table displaced by exactly 2^31 and 2^32 floats (the reservation extended
                          so every address stays mapped): the result checks (not the set-up's) must reject the result

A row index r in [2^31, 2^32) truncated to int32 moves an access 2^32 row_stride floats down.  Tables with such rows
reserve that far below base, and their chunk size has the odd factor 5, which divides none of the row strides used.
So such an access also lands on another physical byte of the chunk, and cannot fault (test_aliased_arena_host.py).

Checks.  (1) float64: K2's pooled values within the bounds of test_gpu_lookup_f64.py; K7's rows and state within the
propagated bound of its row rule (test_gpu_lookup_f64.rule) on G64 = sum g w in float64, whose bound is u |t| per term and
(n - 1) u sum |t| for the sum of n terms in any order.  (2) Bit-identity to a compact twin: the same call on an ordinary
table holding the same row values at small row numbers.  K2 pools in lookup order, so the row number cannot change a bit.
For K7 the twin rows are picked so that every row falls in the same bucket (bucket_bwd.cuh's bucket_of) and in the same
order inside it as its aliased row, and for the radix engine in the same sorted order: every path then sums the same
lookups in the same tree, and only the row number differs.  (3) Hygiene: after each call every physical word outside the
images of the rows in play still holds the sentinel, so a write through a wrapped offset fails the test.

The aliased chunk only serves kernels that visit the rows they are given; the dense sweep visits every row, so it runs
on real memory (and is skipped, saying so, below 12 GiB of free device memory).

Every K7 path returned the twin's bits, so no path depends on the row's value.

Measured on an H100 80GB HBM3 (700 W power limit): the 95 tests run in about 46 s.  Peak device memory is 11.1 GiB
reserved by torch (the sweep's real 8.6 GB table) and 0.94 GiB of arena chunks, and nothing is left allocated after the
run.  An arena maps its chunk at most 256 times; at up to 855 mappings per arena the tests took about twice as long.
Worst error / bound (0.5: the error reached the first-order bound itself, before the factor C): K2 0.498, K7 0.456,
emit uniq_grads 0.482, er_sparse_apply 0.475, the sweep 0.446.
"""
import contextlib

import numpy as np
import pytest
import torch

import aliased_arena as A
from easyrec_b200 import kernels as K
from test_gpu_k7_f64 import bucket_of, num_buckets
from test_gpu_lookup_f64 import (ADAGRAD, ADAM_ROWS, B1, B2, C, EPS, FLOOR, KIND_IDS, KINDS, LAZY_ADAM, MEAN, MOMENTUM,
                                 NONE, ONE_ROW, SGD, SQRTN, SUM, U, R, X, _pool_f64, add, div, mul, rule, sqrt, sub)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32 = np.float32
N_STATE = {SGD: 0, ADAGRAD: 1, MOMENTUM: 1, LAZY_ADAM: 2, ADAM_ROWS: 2}
WORST = {}


@pytest.fixture
def stack():
  """arenas entered here are unmapped and released when the test ends, failed or not"""
  with contextlib.ExitStack() as s:
    yield s
    torch.cuda.synchronize()


# ---- tables -----------------------------------------------------------------------------------------------------------
class Table(object):
  """n_mat = 1 + n_state matrices [n_rows, dim]: 'inter' = one arena of [w | state0 | state1] rows (row_stride
  n_mat * dim), 'sep' = one arena per matrix (row_stride dim).  `mats` are the views handed to the kernels, displaced by
  `shift` floats (0 but in the sensitivity tests); put / get / clean_outside work on the rows' true images."""

  def __init__(self, stack, dim, n_state, layout, shift=0, stride_mult=None):
    self.dim, self.n_mat, self.layout = dim, 1 + n_state, layout
    self.stride = dim * (stride_mult or (self.n_mat if layout == 'inter' else 1))
    self.n_rows = A.table_rows(self.stride)
    assert self.stride % A.ODD, 'row_stride %d: a truncated row index would alias in the chunk' % self.stride
    extent = (self.n_rows * self.stride + shift) * 4
    below = A.below_bytes(self.n_rows, self.stride)
    n_ar = 1 if layout == 'inter' else self.n_mat
    self.arenas = [stack.enter_context(A.AliasedArena(DEV, extent, below_min=below)) for _ in range(n_ar)]
    self.p = self.arenas[0].p
    self.ph = [(ar.phys(torch.float32), ar.phys(torch.int32)) for ar in self.arenas]
    if layout == 'inter':
      t = self.arenas[0].tensor((self.n_rows, self.stride), torch.float32, shift * 4)
      self.mats = [t[:, k * dim:(k + 1) * dim] for k in range(self.n_mat)]
      self.where = [(0, k * dim) for k in range(self.n_mat)]
    else:
      self.mats = [ar.tensor((self.n_rows, self.stride), torch.float32, shift * 4)[:, :dim] for ar in self.arenas]
      self.where = [(k, 0) for k in range(self.n_mat)]

  def rows_for(self, rng, n_low=16):
    """the boundary rows and n_low low rows, all with disjoint images"""
    high = A.boundary_rows(self.dim, self.stride, self.n_rows)
    low = A.with_low_rows(high, self.stride, self.p, n_low, rng)
    return np.array(high, np.int64), np.array(low, np.int64)

  def _idx(self, rows, k):
    a, coff = self.where[k]
    q = self.p // 4
    idx = (np.asarray(rows, np.int64)[:, None] * self.stride + coff + np.arange(self.dim)[None, :]) % q
    return a, torch.from_numpy(idx).to(DEV)

  def put(self, rows, vals):
    for k, v in enumerate(vals):
      a, idx = self._idx(rows, k)
      self.ph[a][0][idx] = v

  def get(self, rows):
    out = []
    for k in range(self.n_mat):
      a, idx = self._idx(rows, k)
      out.append(self.ph[a][0][idx])
    return out

  def clean_outside(self, rows, what):
    torch.cuda.synchronize()
    for a in range(len(self.arenas)):
      pi = self.ph[a][1]
      mask = torch.zeros(pi.numel(), dtype=torch.bool, device=DEV)
      for k in range(self.n_mat):
        if self.where[k][0] == a:
          mask[self._idx(rows, k)[1]] = True
      bad = int(((pi != A.SENTINEL) & ~mask).sum())
      assert bad == 0, '%s: %d physical words outside the rows in play changed' % (what, bad)


class Twin(object):
  """the compact twin: the same layout on ordinary memory, n_rows rows, NaN where no row was put"""

  def __init__(self, dim, n_state, layout, n_rows, stride):
    self.dim, self.n_mat = dim, 1 + n_state
    if layout == 'inter':
      t = torch.full((n_rows, stride), float('nan'), device=DEV)
      self.mats = [t[:, k * dim:(k + 1) * dim] for k in range(self.n_mat)]
    else:
      self.mats = [torch.full((n_rows, stride), float('nan'), device=DEV)[:, :dim] for _ in range(self.n_mat)]

  def put(self, rows, vals):
    r = torch.from_numpy(np.asarray(rows, np.int64)).to(DEV)
    for m, v in zip(self.mats, vals):
      m[r] = v

  def get(self, rows):
    r = torch.from_numpy(np.asarray(rows, np.int64)).to(DEV)
    return [m[r] for m in self.mats]


def _bits_equal(a, b, what):
  a, b = a.contiguous(), b.contiguous()
  same = (a.view(torch.int32) == b.view(torch.int32)) | (torch.isnan(a) & torch.isnan(b))
  n = int((~same).sum())
  assert n == 0, '%s: %d values differ from the compact twin' % (what, n)


def _init_vals(gen, n, dim, kind):
  vals = [torch.randn(n, dim, generator=gen, device=DEV) * 0.5]
  if N_STATE[kind] >= 1:
    vals.append(torch.rand(n, dim, generator=gen, device=DEV) * 0.2 + (0.05 if kind != MOMENTUM else -0.1))
  if N_STATE[kind] == 2:
    vals.append(torch.rand(n, dim, generator=gen, device=DEV) * 0.2 + 1e-3)
  return vals


# ---- K2 ---------------------------------------------------------------------------------------------------------------
def _k2_lookups(rng, high, low, single, B=96):
  """3 slots (sum, mean, sqrtn) of B segments; high rows looked up many times among low rows; a few dropped lookups"""
  n_seg = 3 * B
  lens = np.ones(n_seg, np.int64) if single else rng.integers(0, 6, n_seg)
  if not single:
    lens[rng.integers(0, n_seg, 4)] = 29
  rp = np.concatenate([[0], np.cumsum(lens)])
  n = int(rp[-1])
  pool = np.concatenate([np.repeat(high, 3), low])
  rows = pool[rng.integers(0, pool.size, n)]
  rows[rng.random(n) < 0.04] = -1
  w = rng.uniform(0.25, 2.0, n).astype(F32)
  return n_seg, rp, rows, w


def _k2_run(table, dim, n_rows, rows, w, rp, n_seg, single):
  recs = [dict(num_buckets=n_rows, row_offset=0, seg_begin=f * (n_seg // 3), n_seg=n_seg // 3, bucket_mode=NONE,
               combiner=[SUM, MEAN, SQRTN][f], out_buf=0, out_stride=0, out_col=0) for f in range(3)]
  dpad = -(-dim // 4) * 4
  for f, r in enumerate(recs):
    r['out_stride'], r['out_col'] = 3 * dpad + 4, f * dpad
  sl = K.make_slots(recs, dim)
  sd = K.slots_to_device(sl, DEV)
  out = torch.full((n_seg // 3, 3 * dpad + 4), float('nan'), device=DEV)
  scale = torch.full((n_seg,), float('nan'), device=DEV)
  K.embedding_fwd(table, dim, torch.from_numpy(rows).to(DEV), sd, 3, n_seg, [out],
                  weights=torch.from_numpy(w).to(DEV),
                  row_ptr=None if single else torch.from_numpy(rp.astype(np.int32)).to(DEV), seg_scale=scale)
  torch.cuda.synchronize()
  segs = torch.cat([out[:, f * dpad:f * dpad + dim] for f in range(3)])
  return segs, scale


def _k2_case(stack, dim, stride_mult, single, seed, shift=0):
  rng = np.random.default_rng(seed)
  tab = Table(stack, dim, 0, 'sep', shift=shift, stride_mult=stride_mult)
  high, low = tab.rows_for(rng)
  used = np.concatenate([high, low])
  vals = torch.from_numpy(rng.normal(size=(used.size, dim)).astype(F32)).to(DEV)
  tab.put(used, [vals])
  n_seg, rp, rows, w = _k2_lookups(rng, high, low, single)
  # the twin: used[i] -> row i
  twin = Twin(dim, 0, 'sep', used.size + 1, tab.stride)
  twin.put(np.arange(used.size), [vals])
  lab = np.full(rows.size, -1, np.int64)
  live = rows >= 0
  lab[live] = np.searchsorted(used, rows[live], sorter=np.argsort(used))
  lab[live] = np.argsort(used)[lab[live]]
  assert np.array_equal(used[lab[live]], rows[live])
  got, gsc = _k2_run(tab.mats[0], dim, tab.n_rows, rows, w, rp, n_seg, single)
  tw, tsc = _k2_run(twin.mats[0], dim, used.size + 1, lab, w, rp, n_seg, single)
  what = 'K2 dim %d row_stride %d %s' % (dim, tab.stride, 'single' if single else 'csr')
  _bits_equal(got, tw, what + ': pooled')
  _bits_equal(gsc, tsc, what + ': seg_scale')
  comb = np.repeat([SUM, MEAN, SQRTN], n_seg // 3).astype(np.int64)
  val, err, ok = _pool_f64(twin.mats[0].cpu().numpy(), lab, w, rp, rows.size, comb, single)
  e = (got.double() - val).abs()[ok]
  ratio = float((e / (C * err[ok] + FLOOR)).max())
  WORST['K2'] = max(WORST.get('K2', 0.0), ratio)
  assert bool(torch.isfinite(got).all()) and ratio <= 1.0, '%s: error %.3g x the float64 bound' % (what, ratio)
  _bits_equal(tab.get(used)[0], vals, what + ': the table rows (K2 only reads)')
  tab.clean_outside(used, what)


@pytest.mark.parametrize('path', ['single', 'csr'])
@pytest.mark.parametrize('stride_mult', [1, 3], ids=['stride_dim', 'stride_3dim'])
@pytest.mark.parametrize('dim', [4, 16, 64, 1, 3, 6])
def test_k2(dim, stride_mult, path, stack):
  _k2_case(stack, dim, stride_mult, path == 'single', seed=dim * 10 + stride_mult + 100 * (path == 'single'))


# ---- K7 ---------------------------------------------------------------------------------------------------------------
RUNS = [5000, 1100, 300, 40, 300, 60, 1, 5, 2]   # hot rows > 4096, big buckets > 1024, coop runs > 48, warp / CTA
N_ONE_ROW = 700


def _k7_lookups(rng, high, low):
  """single-valued lookups: slot 0 (NONE) holds runs of RUNS lengths on the high rows and one to three lookups of each
  low row, shuffled, 2% of them dropped, then one more lookup of each row (so every row is updated); slot 1 (ONE_ROW)
  has N_ONE_ROW segments of the row `one` (its row_offset), 5% of them dropped"""
  one = int(high[-1])
  hi = high[:-1]
  lens = np.array([RUNS[i % len(RUNS)] for i in range(hi.size)])
  rows = np.concatenate([np.repeat(hi, lens), np.repeat(low, rng.integers(1, 4, low.size))])
  rows = rows[rng.permutation(rows.size)]
  rows[rng.random(rows.size) < 0.02] = -1
  rows = np.concatenate([rows, hi, low])
  rows1 = np.full(N_ONE_ROW, one, np.int64)
  rows1[rng.random(N_ONE_ROW) < 0.05] = -1
  return np.concatenate([rows, rows1]), rows.size, one


def _k7_plan(dim, n0, n_rows, one_row_offset):
  dpad = -(-dim // 4) * 4 + 4
  recs = [dict(num_buckets=n_rows, row_offset=0, seg_begin=0, n_seg=n0, bucket_mode=NONE, combiner=SUM, out_buf=0,
               out_stride=dpad, out_col=4),
          dict(num_buckets=1, row_offset=one_row_offset, seg_begin=n0, n_seg=N_ONE_ROW, bucket_mode=ONE_ROW,
               combiner=SUM, out_buf=1, out_stride=dpad, out_col=4)]
  sl = K.make_slots(recs, dim)
  return K.slots_to_device(sl, DEV), dpad


def _bucket_twin(rows_u, log2_nb, skip=()):
  """twin rows: the k-th smallest row of bucket b -> the k-th smallest small integer of bucket b"""
  b = bucket_of(rows_u, log2_nb)
  cand = np.arange(1, 1 << 22, dtype=np.int64)
  cand = cand[~np.isin(cand, np.asarray(skip, np.int64))]
  cb = bucket_of(cand, log2_nb)
  out = np.empty_like(rows_u)
  for bv in np.unique(b):
    m = b == bv
    out[m] = cand[cb == bv][:int(m.sum())]
  return out


def _classes(rows_u, cnt, n, warp_mode):
  """the bucketed engine's role for each row: bucket size and run length (bucket_bwd.cuh)"""
  lg = int(num_buckets(n, warp_mode)).bit_length() - 1
  b = bucket_of(rows_u, lg)
  bsize = np.bincount(b, weights=cnt, minlength=1 << lg)[b]
  cls = np.where(bsize <= (128 if warp_mode else 0), 'warp', np.where(bsize <= 1024, 'cta', 'big'))
  cls = np.where((cls == 'cta') & (cnt > 48), 'coop', cls)
  return np.where(cnt > 4096, 'hot', cls), lg


def _k7_call(mats, kind, dim, n_rows, rows_t, sd, n_seg, gbufs, w_t, opt, presort):
  ws = K.bwd_workspace(rows_t.numel(), DEV, dim)
  st = [mats[1] if len(mats) > 1 else None, mats[2] if len(mats) > 2 else None]
  if presort:
    ws0 = K.bwd_workspace(rows_t.numel(), DEV, dim)
    K.embedding_bwd_presort(rows_t, n_rows, dim, ws0, sd, 2)
    K.embedding_bwd(mats[0], st[0], st[1], dim, rows_t, sd, 2, n_seg, gbufs, opt, ws, weights=w_t,
                    sorted_from=(ws0, dim))
  else:
    K.embedding_bwd(mats[0], st[0], st[1], dim, rows_t, sd, 2, n_seg, gbufs, opt, ws, weights=w_t)
  torch.cuda.synchronize()


def _k7_case(stack, dim, kind, layout, seed, shift=0, presort=False):
  rng = np.random.default_rng(seed)
  gen = torch.Generator(device=DEV).manual_seed(seed)
  n_state = N_STATE[kind]
  tab = Table(stack, dim, n_state, layout, shift=shift)
  high, low = tab.rows_for(rng)
  rows, n0, one = _k7_lookups(rng, high, low)
  n = rows.size
  used = np.concatenate([high, low])
  init = _init_vals(gen, used.size, dim, kind)
  tab.put(used, init)
  warp_mode = K.k7_warp_mode(dim)
  live0 = rows[:n0][rows[:n0] >= 0]
  ru, cnt = np.unique(live0, return_counts=True)
  cls, lg = _classes(ru, cnt, n, warp_mode)
  need = {'coop', 'big', 'hot', 'warp' if warp_mode else 'cta'}
  hi_cls = set(cls[np.isin(ru, high)].tolist())
  assert need <= hi_cls, 'high rows reach %s, not %s' % (sorted(hi_cls), sorted(need))
  # twin rows: same bucket, same order inside it; the one-row slot's row after them
  tw_u = _bucket_twin(ru, lg)
  tw_one = int(tw_u.max()) + 1
  tmap = dict(zip(ru.tolist(), tw_u.tolist()))
  tmap[one] = tw_one
  tw_rows = np.array([tmap[int(r)] if r >= 0 else -1 for r in rows], np.int64)
  tw_used = np.array([tmap[int(r)] for r in used], np.int64)
  twin = Twin(dim, n_state, layout, tw_one + 1, tab.stride)
  twin.put(tw_used, init)
  # gradients, weights
  sd, dpad = _k7_plan(dim, n0, tab.n_rows, one)
  sd_t, _ = _k7_plan(dim, n0, tw_one + 1, tw_one)
  # gradients of mean 0.5: a long run's sum does not cancel to where its first-order bound exceeds it
  g0 = torch.randn(n0, dpad, generator=gen, device=DEV) * 0.5 + 0.5
  g1 = torch.randn(N_ONE_ROW, dpad, generator=gen, device=DEV) * 0.5 + 0.5
  w = rng.uniform(0.5, 1.5, n).astype(F32)
  w_t = torch.from_numpy(w).to(DEV)
  lr, b1p, b2p = 0.05, float(F32(B1 ** 3)), float(F32(B2 ** 3))
  opt = K.make_opt(kind, lr, B1, B2, EPS, b1p, b2p, 1.0)       # (momentum rides in beta1)
  # the one-row slot's lookups carry the row of K1's ONE_ROW mode: row_offset
  _k7_call(tab.mats, kind, dim, tab.n_rows, torch.from_numpy(rows).to(DEV), sd, n, [g0, g1], w_t, opt, presort)
  _k7_call(twin.mats, kind, dim, tw_one + 1, torch.from_numpy(tw_rows).to(DEV), sd_t, n, [g0, g1], w_t, opt, presort)
  what = 'K7 %s %s dim %d row_stride %d%s' % (KIND_IDS[kind], layout, dim, tab.stride, ' presort' if presort else '')
  got = tab.get(used)
  ref_t = twin.get(tw_used)
  for k in range(tab.n_mat):
    _bits_equal(got[k], ref_t[k], '%s [%d]' % (what, k))
  Gs = _g64(torch.cat([g0[:, 4:4 + dim], g1[:, 4:4 + dim]]), w_t, rows, used)
  lr0 = (div(mul(X(lr), sqrt(sub(X(1.0), X(b2p)))), sub(X(1.0), X(b1p))) if kind in (LAZY_ADAM, ADAM_ROWS) else X(lr))
  ref = rule(kind, X(init[0]), X(init[1]) if n_state else None, X(init[2]) if n_state == 2 else None, Gs, lr0)
  for k in range(tab.n_mat):
    _within(got[k], ref[k], '%s [%d]' % (what, k), 'K7')
  tab.clean_outside(used, what)


def _g64(g, w_t, rows, used):
  """float64 G of each row of `used` (in that order): the sum over its live lookups l of g[l] * w[l], as an R whose
  bound is u |t| per term and (n - 1) u sum |t| for the sum of n terms in any order"""
  dim = g.shape[1]
  lv = np.nonzero(rows >= 0)[0]
  lv_t = torch.from_numpy(lv).to(DEV)
  term = mul(X(g[lv_t]), R(w_t[lv_t].double()[:, None].expand(-1, dim).contiguous()))
  order = np.argsort(used)
  pos = torch.from_numpy(order[np.searchsorted(used, rows[lv], sorter=order)]).to(DEV)
  z = torch.zeros(used.size, dim, dtype=torch.float64, device=DEV)
  c = torch.zeros(used.size, dtype=torch.float64, device=DEV).index_add(0, pos, torch.ones_like(pos, dtype=torch.float64))
  return R(z.index_add(0, pos, term.v), z.index_add(0, pos, term.e) +
           (c - 1).clamp_min(0)[:, None] * U * z.index_add(0, pos, term.v.abs()))


def _within(got, ref, what, key):
  err = (got.double() - ref.v).abs()
  ratio = float((err / (C * ref.e + FLOOR)).max())
  WORST[key] = max(WORST.get(key, 0.0), ratio)
  assert bool(torch.isfinite(got).all()) and ratio <= 1.0, '%s: error %.3g x the float64 bound' % (what, ratio)


@pytest.mark.parametrize('layout', ['sep', 'inter'])
@pytest.mark.parametrize('kind', KINDS, ids=KIND_IDS)
@pytest.mark.parametrize('dim', [1, 3, 4, 16, 64])
def test_k7(dim, kind, layout, stack):
  _k7_case(stack, dim, kind, layout, seed=1000 + dim * 10 + kind + 7 * (layout == 'inter'))


@pytest.mark.parametrize('dim', [4, 3])
def test_k7_presort_reuse(dim, stack):
  _k7_case(stack, dim, ADAGRAD, 'inter', seed=2000 + dim, presort=True)


# ---- emit form (radix engine) + er_sparse_apply -------------------------------------------------------------------------
@pytest.mark.parametrize('kind', [ADAGRAD, LAZY_ADAM], ids=['adagrad', 'lazy_adam'])
@pytest.mark.parametrize('dim', [1, 3, 4, 64])
def test_emit_then_sparse_apply(dim, kind, stack):
  """the row-sharded owner chain: uniq_rows / uniq_grads from the radix engine at n_rows = the table's rows, then the
  owner's er_sparse_apply on the aliased table; uniq_grads and the updated rows against float64 from g * w"""
  seed = 3000 + dim * 10 + kind
  rng = np.random.default_rng(seed)
  gen = torch.Generator(device=DEV).manual_seed(seed)
  n_state = N_STATE[kind]
  tab = Table(stack, dim, n_state, 'inter')
  high, low = tab.rows_for(rng)
  used = np.concatenate([high, low])
  lens = np.array([[1, 3, 64, 65, 700][i % 5] for i in range(high.size)])
  rows = np.concatenate([np.repeat(high, lens), np.repeat(low, 2)])
  rows = rows[rng.permutation(rows.size)]
  n = rows.size
  rank = {int(r): i for i, r in enumerate(np.sort(used))}     # monotone: the same sorted order
  tw_rows = np.array([rank[int(r)] for r in rows], np.int64)
  dpad = -(-dim // 4) * 4 + 4
  recs = [dict(num_buckets=tab.n_rows, row_offset=0, seg_begin=0, n_seg=n, bucket_mode=NONE, combiner=SUM, out_buf=0,
               out_stride=dpad, out_col=4)]
  sd = K.slots_to_device(K.make_slots(recs, dim), DEV)
  g = torch.randn(n, dpad, generator=gen, device=DEV) * 0.5 + 0.5       # (mean 0.5: as in _k7_case)
  w_t = torch.from_numpy(rng.uniform(0.5, 1.5, n).astype(F32)).to(DEV)
  outs = []
  for rr, nr in ((rows, tab.n_rows), (tw_rows, used.size)):
    ur = torch.full((n,), -7, dtype=torch.int64, device=DEV)
    ug = torch.full((n, dim), float('nan'), device=DEV)
    nu = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    K.embedding_bwd(None, None, None, dim, torch.from_numpy(rr).to(DEV), sd, 1, n, [g], K.make_opt(SGD, 0.1),
                    K.bwd_workspace(n, DEV, dim), weights=w_t, uniq_rows=ur, uniq_grads=ug, n_uniq=nu, n_rows=nr)
    outs.append((ur, ug, nu))
  (ur, ug, nu), (tur, tug, tnu) = outs
  k = int(nu.item())
  assert k == used.size == int(tnu.item())
  assert ur[:k].cpu().numpy().tolist() == np.sort(used).tolist(), 'emit uniq_rows: not the exact rows'
  assert bool((ur[k:] == -7).all()), 'uniq_rows past n_uniq'
  _bits_equal(ug[:k], tug[:k], 'emit uniq_grads dim %d' % dim)
  su = np.sort(used)
  Gs = _g64(g[:, 4:4 + dim], w_t, rows, su)
  _within(ug[:k], Gs, 'emit uniq_grads dim %d' % dim, 'emit')
  # the owner's update
  init = _init_vals(gen, used.size, dim, kind)
  tab.put(su, init)
  twin = Twin(dim, n_state, 'inter', used.size, tab.stride)
  twin.put(np.arange(used.size), init)
  lr, b1p, b2p = 0.05, float(F32(B1 ** 2)), float(F32(B2 ** 2))
  opt = K.make_opt(kind, lr, B1, B2, EPS, b1p, b2p, 1.0)
  st = tab.mats[1:] + [None] * (2 - n_state)
  K.sparse_apply(tab.mats[0], st[0], st[1], dim, ur, ug, nu, opt)
  tst = twin.mats[1:] + [None] * (2 - n_state)
  K.sparse_apply(twin.mats[0], tst[0], tst[1], dim, tur, tug, tnu, opt)
  torch.cuda.synchronize()
  what = 'sparse_apply %s dim %d' % (KIND_IDS[kind], dim)
  got, tw = tab.get(su), twin.get(np.arange(used.size))
  for i in range(tab.n_mat):
    _bits_equal(got[i], tw[i], '%s [%d]' % (what, i))
  lr0 = (div(mul(X(lr), sqrt(sub(X(1.0), X(b2p)))), sub(X(1.0), X(b1p))) if kind == LAZY_ADAM else X(lr))
  ref = rule(kind, X(init[0]), X(init[1]), X(init[2]) if n_state == 2 else None, Gs, lr0)
  for i in range(tab.n_mat):
    _within(got[i], ref[i], '%s [%d]' % (what, i), 'sparse_apply')
  tab.clean_outside(su, what)


# ---- er_mark_rows, er_shard_group -------------------------------------------------------------------------------------
def test_mark_rows(stack):
  n_rows = 2 ** 32 - 2
  ar = stack.enter_context(A.AliasedArena(DEV, n_rows, fill=A.SENTINEL_BYTE, below_min=A.below_bytes(n_rows, 1, 1)))
  touched = ar.tensor((n_rows,), torch.uint8)
  ph = ar.phys(torch.uint8)
  marks = [2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, 2 ** 31 + 4097, 3 * 10 ** 9, 2 ** 32 - 4, n_rows - 1, 0, 5]
  assert A.images_disjoint(marks, 1, ar.p, elem=1)
  rows = torch.tensor(marks + [-1, n_rows, n_rows + 5, 2 ** 33], dtype=torch.int64, device=DEV)
  idx = torch.tensor([m % ar.p for m in marks], dtype=torch.int64, device=DEV)
  for value in (1, 0):
    K.mark_rows(rows, n_rows, touched, value)
    torch.cuda.synchronize()
    assert bool((ph[idx] == value).all()), 'er_mark_rows: a row >= 2^31 was not marked %d' % value
    ph[idx] = A.SENTINEL_BYTE
    assert bool((ph == A.SENTINEL_BYTE).all()), 'er_mark_rows wrote a byte of no row it was given'


@pytest.mark.parametrize('world', [2, 3, 8])
def test_shard_group_rows_past_2_32(world):
  rng = np.random.default_rng(world)
  # owner-local rows as K1 makes them from int64 ids (row = id // world): up to (2^63 - 1) // world
  top = (2 ** 63 - 1) // world
  base = [2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 32 + world, 2 ** 33 + 5, 2 ** 40 + 7, top - 2 ** 32, top]
  rows = [int(base[i]) for i in rng.integers(0, len(base), 600)] + [2 ** 32 + int(x) for x in rng.integers(0, 50, 400)]
  rows += [-1] * 8
  owner = [int(x) for x in rng.integers(0, world, len(rows))]
  n = len(rows)
  cap = 64
  t_rows = torch.tensor(rows, dtype=torch.int64, device=DEV)
  t_own = torch.tensor(owner, dtype=torch.int32, device=DEV)
  send = torch.full((world * cap,), -9, dtype=torch.int64, device=DEV)
  pos = torch.full((n,), -9, dtype=torch.int64, device=DEV)
  counts = torch.full((world + 1,), -9, dtype=torch.int32, device=DEV)
  K.shard_group(t_rows, t_own, world, cap, send, pos, counts, K.shard_group_workspace(n, DEV))
  send, pos, counts = send.tolist(), pos.tolist(), counts.tolist()
  want = [set() for _ in range(world)]
  for r, o in zip(rows, owner):
    if r >= 0:
      want[o].add(r)
  assert counts[:world] == [len(s) for s in want] and counts[world] == 0
  for o in range(world):
    blk = send[o * cap:(o + 1) * cap]
    assert set(blk[:len(want[o])]) == want[o] and blk[len(want[o]):] == [-1] * (cap - len(want[o])), 'owner %d' % o
  for r, o, p in zip(rows, owner, pos):
    if r < 0:
      assert p == -1
    else:
      assert p // cap == o and send[p] == r, 'lookup of row %d: position %d' % (r, p)


# ---- er_adam_dense_sweep on a real table past 2^31 floats -------------------------------------------------------------
@pytest.mark.parametrize('dim', [4, 3], ids=['vector', 'scalar'])
def test_adam_dense_sweep_past_2_31(dim):
  stride = 3 * dim
  n_rows = 2 ** 31 // stride + 1024
  need = n_rows * stride * 4 + n_rows
  free = torch.cuda.mem_get_info()[0]
  if free < need + (3 << 30):
    pytest.skip('needs %.1f GiB of free device memory for a real table past 2^31 floats, %.1f GiB free' %
                ((need + (3 << 30)) / 2 ** 30, free / 2 ** 30))
  gen = torch.Generator(device=DEV).manual_seed(dim)
  t = torch.zeros(n_rows, stride, device=DEV)
  touched = torch.zeros(n_rows, dtype=torch.uint8, device=DEV)
  try:
    r0 = 2 ** 31 // stride
    rows = np.array(sorted({5, 77} | set(range(r0 - 3, r0 + 4)) | set(range(n_rows - 4, n_rows))), np.int64)
    assert any(A.straddles(r, stride, 2 ** 31) for r in rows) or 2 ** 31 % stride == 0
    rt = torch.from_numpy(rows).to(DEV)
    w0 = torch.randn(rows.size, dim, generator=gen, device=DEV)
    m0 = torch.randn(rows.size, dim, generator=gen, device=DEV) * 0.1
    v0 = torch.rand(rows.size, dim, generator=gen, device=DEV) * 0.1 + 1e-3
    m0[1] = 0.0                                            # m = 0, v != 0: still decays v
    t[rt, :dim], t[rt, dim:2 * dim], t[rt, 2 * dim:] = w0, m0, v0
    mark = rt[::3]
    touched[mark] = 1
    lr, b1p, b2p = 0.01, float(F32(B1 ** 4)), float(F32(B2 ** 4))
    opt = K.make_opt(ADAM_ROWS, lr, B1, B2, EPS, b1p, b2p, 1.0)
    K.adam_dense_sweep(t[:, :dim], t[:, dim:2 * dim], t[:, 2 * dim:], dim, touched, opt)
    torch.cuda.synchronize()
    got = [t[rt, :dim], t[rt, dim:2 * dim], t[rt, 2 * dim:]]
    lr0 = div(mul(X(lr), sqrt(sub(X(1.0), X(b2p)))), sub(X(1.0), X(b1p)))
    mm, vv = mul(X(m0), X(B1)), mul(X(v0), X(B2))
    ww = sub(X(w0), div(mul(lr0, mm), add(sqrt(vv), X(EPS))))
    is_t = torch.zeros(rows.size, dtype=torch.bool, device=DEV)
    is_t[::3] = True
    for i, (ref, init) in enumerate(((ww, w0), (mm, m0), (vv, v0))):
      _within(got[i][~is_t], R(ref.v[~is_t], ref.e[~is_t]), 'sweep dim %d [%d]' % (dim, i), 'sweep')
      _bits_equal(got[i][is_t], init[is_t], 'sweep dim %d: touched rows [%d]' % (dim, i))
    t[rt] = 0.0
    nz = sum(int(torch.count_nonzero(c)) for c in t.split(1 << 24))
    assert nz == 0, 'the sweep wrote %d floats of rows whose moments are zero' % nz
  finally:
    del t, touched
    torch.cuda.empty_cache()


# ---- sensitivity -------------------------------------------------------------------------------------------------------
SENSED = 'compact twin|float64 bound|outside the rows in play'   # the result checks, not the set-up's assertions


@pytest.mark.parametrize('shift', [2 ** 31, 2 ** 32], ids=['2^31', '2^32'])
def test_sensitivity_k2(shift, stack):
  """K2 reading a table displaced by `shift` floats, as a wrapped offset would: the checks reject it"""
  with pytest.raises(AssertionError, match=SENSED):
    _k2_case(stack, 16, 1, False, seed=5, shift=shift)


@pytest.mark.parametrize('shift', [2 ** 31, 2 ** 32], ids=['2^31', '2^32'])
def test_sensitivity_k7(shift, stack):
  """K7 updating a table displaced by `shift` floats: the checks reject it"""
  with pytest.raises(AssertionError, match=SENSED):
    _k7_case(stack, 16, ADAGRAD, 'inter', seed=6, shift=shift)


def test_zz_report_worst():
  print('worst error / bound: %s' % ', '.join('%s %.3f' % kv for kv in sorted(WORST.items())))
  print('peak device memory: %.2f GiB reserved by torch, %.3f GiB of arena chunks' % (
      torch.cuda.max_memory_reserved() / 2 ** 30, A.LIVE['peak'] / 2 ** 30))
  assert A.LIVE['bytes'] == 0, 'an arena was left open'
