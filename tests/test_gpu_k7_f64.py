"""GPU: K7's deduplicated per-row gradient sum (er_embedding_bwd) against float64, on every path of both engines.

  G_row = sum over the live lookups l of the row, in ascending lookup order, of coef_l * grad_bufs[..][seg(l)]

  bucketed engine   dims 1/2/3/4/6/8/12/16/32/64/128/300 x a bucket of 1, 32, 33, 127, 128, 129, 1024, 1025 pairs (and
                    16384, 16385, 20000 at dims 1/16/64): the warp role, the CTA role, the big-bucket CTA and its
                    global-memory radix fallback, each asserted reached from a host restatement of num_buckets and
                    bucket_of; warp-chunk run boundaries 31/32/33/64/96/128 at offsets 0, 1, 31, 32, 64 and 96 (one
                    run filling all 128 pairs); the whole-CTA tree at runs 48/49; the hot-row kernel at 4096/4097 and
                    kChunk multiples +- 1; separate and interleaved row_stride layouts
  one-row slots     B = 1500 (not a multiple of 512), three one-row slots in one call, a one-row slot longer than the
                    average slot (beside a 10- or 0-segment slot), slots whose first lookup is dropped, a second call
                    on the same workspace; dims 3/4/16/300
  radix engine      (uniq_rows given) every dim above, runs 1/63/64/65/511/512/513/1025, grad_scale 0.375: uniq_rows and
                    n_uniq exact, uniq_grads = fl(grad_scale G), the table moved by -uniq_grads
  inputs            single-valued and CSR lookups (live count read from row_ptr[n_seg], lookups past it point at rows
                    and segments whose gradients are NaN), dropped (-1) lookups, the sum / mean / sqrtn combiners in
                    one call with and without seg_scale, weights NULL / given / UNIT_WEIGHTS slots, 1 / 3 / 8 gradient buffers with their own
                    pitches and column offsets, n_slots 1 / 257 / 2048, rows 0 and n_rows - 1
  scalar fallback   a table base one float off, row_stride 17 at dim 16, a gradient buffer one float off: bit-identical
                    to the aligned call on every row both sum in lookup order
  presort / reuse   er_embedding_bwd_presort + er_embedding_bwd_reuse_sort against a fresh call, one-row and CSR plans
  exact inputs      gradients in -8..8, coefficients in {+-0.5, +-1, +-2} x {0.5, 1, 2} at dims 1/16/64/300: big and
                    radix-sorted buckets, radix runs and one-row slots around every chunk boundary, where any order
                    sums exactly, so the tree paths must return G64 itself
  limits            dim 4096 runs, dim 4097 is refused

Observing G.  The bucketed engine only updates tables, so every call runs SGD with lr = 1 and grad_scale = 1 on zeroed
touched rows: the kernel then writes fsub(0, G) exactly.  Untouched rows hold a distinct finite pattern and must come
back bit-identical; row_stride padding holds NaN and must stay NaN.

Reference and bound.  G64 = sum g_l w_l s_seg(l) in float64 from the fp32 inputs the kernel received (w = 1 when
weights is NULL or the slot has UNIT_WEIGHTS, s = 1 without seg_scale).  Allowed error, per element:
C F + 2^-140 with F = 2u sum|g w s| + (n - 1) u sum|g w s|, u = 2^-24, C = 2 and n the run length: the first term of F
is the rounding of fl(w s) and fl(g c), the second holds for any summation order (trees, hot-row chunks, one-row
partials).  uniq_grads adds u |G| to F.  On the exact inputs every path must return G64 itself (compared by value:
a shuffle-scan tree starts a sum from its first term, so a zero G may come back as -0).  Where the header promises lookup order - the warp role (buckets of <= 128 pairs), runs of <= 48
in CTA-sorted buckets, and radix runs of <= 64 at dims 64 / 128 and at the scalar dims - a float32 numpy restatement
(c = fl(w s), t = fl(g c), acc = fl(acc + t) from +0 in ascending lookup order) must match bit for bit.  Every call is
made twice and must repeat bit for bit.

Hygiene.  Gradient buffers sit in NaN-filled memory with guards: the pitch padding, other slots' columns and segments
no live lookup uses are NaN, as are the weights and seg_scale entries of dropped lookups and unused segments, so an
over-read turns G into NaN.  Tables and uniq outputs have NaN guards; uniq entries past n_uniq must keep their fill.

Measured on an H100 80GB HBM3 (700 W power limit): the 307 tests run in about 25 s and the process peaks at 0.25 GiB
of reserved device memory.  Worst error / allowed error per path (0.5: the error reached F itself, before the factor
C): warp 0.470, cta 0.488, coop 0.025, big 0.419, big_radix 0.047, hot 0.000, one_row 0.001, radix_vec 0.471,
radix_scalar 0.523, radix_scan 0.518, radix_hot 0.010.
"""
import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, kernels as K

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
C = 2.0
FLOOR = 2.0 ** -140
G = 64                      # guard floats around every buffer (keeps 16-byte alignment)
F32 = np.float32
NAN = F32(np.nan)
SUM, MEAN, SQRTN, UNIT = _lib.COMBINER_SUM, _lib.COMBINER_MEAN, _lib.COMBINER_SQRTN, _lib.COMBINER_UNIT_WEIGHTS
NONE, ONE_ROW = _lib.BUCKET_NONE, _lib.BUCKET_ONE_ROW
WARP_CAP, CAP, BIG_CAP, COOP_RUN, QUEUE_RUN, LONG_RUN = 128, 1024, 16384, 48, 4096, 64
ALL_DIMS = [1, 2, 3, 4, 6, 8, 12, 16, 32, 64, 128, 300]
N_ROWS = 8192              # table rows of most cases
WORST = {}


# ---- host restatements of the bucket placement (csrc/bucket_bwd.cuh) ---------------------------------------------
def num_buckets(n, warp_mode):
  nb = 64
  while nb < 8192 and nb * (80 if warp_mode else 320) < n:
    nb <<= 1
  return nb


def bucket_of(keys, log2_nb):
  k = (np.asarray(keys, np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)
  return (k >> np.uint64(32 - log2_nb)).astype(np.int64)


def _log2(v):
  return int(v).bit_length() - 1


def _aligned_vec(dim, misalign):
  return dim in K.VECTOR_DIMS and not misalign


# ---- a K7 call: lookups, slots, buffers --------------------------------------------------------------------------
class Case(object):
  """rows [cap] (past n_live: lookups past the CSR live count), seg [cap] or None (single-valued), slots as
  (seg_begin, n_seg, bucket_mode) triples covering [0, n_seg)."""

  def __init__(self, rng, dim, n_rows, rows, slots, n_seg, seg=None, n_live=None, wmode='none', scale=False,
               n_bufs=1, comb=SUM, dyadic=False):
    self.dim, self.n_rows, self.n_seg, self.dyadic = dim, n_rows, n_seg, dyadic
    self.rows = np.asarray(rows, np.int64)
    self.cap = self.rows.size
    self.seg = None if seg is None else np.asarray(seg, np.int32)
    self.n_live = self.cap if n_live is None else n_live
    self.csr = seg is not None
    seg_all = np.arange(self.cap) if seg is None else self.seg.astype(np.int64)
    sb = np.array([s[0] for s in slots], np.int64)
    self.slot_sb, self.slot_n = sb, np.array([s[1] for s in slots], np.int64)
    self.mode = np.array([s[2] for s in slots], np.int64)
    nsl = len(slots)
    unit = np.zeros(nsl, bool)
    if wmode == 'unit':
      unit[::2] = True
      unit[self.mode == ONE_ROW] = False
    self.unit = unit
    live = (np.arange(self.cap) < self.n_live) & (self.rows >= 0)
    self.live = live
    f_of = np.searchsorted(sb, seg_all, side='right') - 1
    self.f_of = f_of
    used = np.zeros(n_seg, bool)
    used[seg_all[live]] = True
    # buffers: slot f -> buffer f % n_bufs; its k-th slot at column 4 + k * (dim rounded up to 4, + 4)
    dpad = -(-dim // 4) * 4 + 4
    self.out_buf = np.arange(nsl) % n_bufs
    self.out_col = np.zeros(nsl, np.int64)
    self.out_stride = np.zeros(nsl, np.int64)
    self.bufs_np = []
    for j in range(n_bufs):
      mine = np.nonzero(self.out_buf == j)[0]
      stride = 4 + dpad * max(len(mine), 1) + 4 * (j + 1)
      self.out_col[mine] = 4 + dpad * np.arange(len(mine))
      self.out_stride[mine] = stride
      nb_rows = int(max([self.slot_n[f] for f in mine] + [1]))
      self.bufs_np.append(np.full(nb_rows * stride, NAN, F32))
    s_used = np.nonzero(used)[0]
    fu = np.searchsorted(sb, s_used, side='right') - 1
    for j in range(n_bufs):
      m = self.out_buf[fu] == j
      base = (s_used[m] - sb[fu[m]]) * self.out_stride[fu[m]] + self.out_col[fu[m]]
      idx = base[:, None] + np.arange(dim)[None, :]
      self.bufs_np[j][idx] = (rng.integers(-8, 9, idx.shape) if dyadic else rng.standard_normal(idx.shape)).astype(F32)
    self.weights = None
    if wmode != 'none':
      w = (rng.choice([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0], self.cap) if dyadic else
           rng.uniform(-2.0, 2.0, self.cap)).astype(F32)
      w[rng.random(self.cap) < 0.1] = 0.0
      w[unit[f_of]] = 1.0
      w[~live & ~unit[f_of]] = NAN
      self.weights = w
    self.scale = None
    if scale:
      sc = (rng.choice([0.5, 1.0, 2.0], n_seg) if dyadic else rng.uniform(0.25, 1.5, n_seg)).astype(F32)
      sc[~used] = NAN
      self.scale = sc
    recs = [dict(num_buckets=n_rows, row_offset=0, seg_begin=int(sb[f]), n_seg=int(self.slot_n[f]),
                 bucket_mode=int(self.mode[f]), combiner=int(comb if f % 3 == 0 else (f % 3)) | (UNIT if unit[f] else 0),
                 out_buf=int(self.out_buf[f]), out_stride=int(self.out_stride[f]), out_col=int(self.out_col[f]))
            for f in range(nsl)]
    self.slots_np = K.make_slots(recs, dim)
    self.n_slots = nsl
    self.one_row_path = (not self.csr) and bool((self.mode == ONE_ROW).any())
    self._ref()

  # ---- float64 reference, exact float32 restatement ------------------------------------------------------------
  def _ref(self):
    dim = self.dim
    l = np.nonzero(self.live)[0]
    r = self.rows[l]
    order = np.lexsort((l, r))
    l, r = l[order], r[order]
    s = np.arange(self.cap)[l] if self.seg is None else self.seg[l].astype(np.int64)
    f = self.f_of[l]
    w = np.ones(l.size, F32) if self.weights is None else np.where(self.unit[f], F32(1), self.weights[l]).astype(F32)
    sc = np.ones(l.size, F32) if self.scale is None else self.scale[s]
    c32 = (w * sc).astype(F32) if self.scale is not None else w
    g = np.empty((l.size, dim), F32)
    for j, b in enumerate(self.bufs_np):
      m = self.out_buf[f] == j
      base = (s[m] - self.slot_sb[f[m]]) * self.out_stride[f[m]] + self.out_col[f[m]]
      g[m] = b[base[:, None] + np.arange(dim)[None, :]]
    t64 = g.astype(np.float64) * w.astype(np.float64)[:, None] * sc.astype(np.float64)[:, None]
    t32 = (g * c32[:, None]).astype(F32)
    self.urow, start, cnt = np.unique(r, return_index=True, return_counts=True)
    self.run_len = cnt
    self.G64 = np.add.reduceat(t64, start, axis=0) if l.size else np.zeros((0, dim))
    self.A64 = np.add.reduceat(np.abs(t64), start, axis=0) if l.size else np.zeros((0, dim))
    seq = cnt <= WARP_CAP
    acc = np.zeros((self.urow.size, dim), F32)
    for k in range(int(cnt[seq].max()) if seq.any() else 0):
      m = seq & (cnt > k)
      acc[m] = (acc[m] + t32[start[m] + k]).astype(F32)
    self.seq32 = acc
    self.row_one = np.zeros(self.urow.size, bool)
    if self.one_row_path:
      orow = np.unique(self.rows[self.live & (self.mode[self.f_of] == ONE_ROW)])
      self.row_one = np.isin(self.urow, orow)

  def bound(self):
    n = self.run_len.astype(np.float64)[:, None]
    return C * (2 * U * self.A64 + (n - 1) * U * self.A64) + FLOOR

  # ---- which path each row takes ---------------------------------------------------------------------------------
  def bucket_counts(self):
    keys = self.rows[self.live & ~(self.one_row_path & (self.mode[self.f_of] == ONE_ROW))]
    nb = num_buckets(self.cap, K.k7_warp_mode(self.dim))
    return np.bincount(bucket_of(keys, _log2(nb)), minlength=nb), _log2(nb)

  def paths(self, engine, misalign=False):
    """per touched row: (label, sums in lookup order)"""
    n = self.run_len
    if engine == 'radix':
      if _aligned_vec(self.dim, misalign):
        base = 'radix_vec' if self.dim >= 64 else 'radix_scan'
      else:
        base = 'radix_scan' if self.dim == 1 else 'radix_scalar'
      lab = np.where(n > LONG_RUN, 'radix_hot', base)
      return lab, (lab != 'radix_hot') & (lab != 'radix_scan')
    cnt, lg = self.bucket_counts()
    bc = cnt[bucket_of(self.urow, lg)]
    warp = K.k7_warp_mode(self.dim)
    role = np.where(warp & (bc <= WARP_CAP), 'warp',
                    np.where(bc <= CAP, 'cta', np.where(bc <= BIG_CAP, 'big', 'big_radix')))
    lab = role.astype(object)
    lab[(role != 'warp') & (n > COOP_RUN)] = 'coop'
    lab[np.isin(role, ['big', 'big_radix']) & (n > QUEUE_RUN)] = 'hot'
    lab[self.row_one] = 'one_row'
    exact = (lab == 'warp') | np.isin(role, ['cta', 'big', 'big_radix']) & (n <= COOP_RUN)
    return lab.astype(str), exact & ~self.row_one

  # ---- device side -----------------------------------------------------------------------------------------------
  def upload(self, gbuf_off=False):
    self.bufs_t = []
    views = []
    for j, b in enumerate(self.bufs_np):
      off = 1 if (gbuf_off and j == 0) else 0
      t = torch.full((b.size + 2 * G + off,), float('nan'), dtype=torch.float32, device=DEV)
      t[G + off:G + off + b.size] = torch.from_numpy(b).to(DEV)
      self.bufs_t.append((t, off))
      v = t[G + off:G + off + b.size].view(-1, int(self.out_stride[self.out_buf == j][0]) if (self.out_buf == j).any()
                                           else b.size)
      views.append(v)
    self.sd = K.slots_to_device(self.slots_np, DEV)
    self.rows_t = torch.from_numpy(self.rows).to(DEV)
    self.w_t = None if self.weights is None else torch.from_numpy(self.weights).to(DEV)
    self.sc_t = None if self.scale is None else torch.from_numpy(self.scale).to(DEV)
    self.seg_t = self.rp_t = None
    if self.csr:
      self.seg_t = torch.from_numpy(self.seg).to(DEV)
      lens = np.bincount(self.seg[:self.n_live], minlength=self.n_seg)
      rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
      assert rp[-1] == self.n_live
      self.rp_t = torch.from_numpy(rp).to(DEV)
    return views


def _pattern(n_rows, stride, dim):
  r = np.arange(n_rows, dtype=np.float64)[:, None]
  c = np.arange(stride, dtype=np.float64)[None, :]
  p = (((r * 131 + c * 7) % 1009) / 64.0 - 7.5).astype(F32)
  p[:, dim:] = NAN
  return p


def run(case, engine='bucketed', layout='separate', table_off=False, stride=None, gbuf_off=False, gs=1.0,
        presort=False, ws=None, check=True):
  """One K7 call (twice, bit-identical).  Returns (table [n_rows, stride] float32, uniq tuple or None)."""
  dim, n_rows = case.dim, case.n_rows
  if stride is None:
    stride = dim if layout == 'separate' else 2 * dim + 4
  init = _pattern(n_rows, stride, dim)
  init[case.urow, :dim] = 0.0
  views = case.upload(gbuf_off)
  off = G + (1 if table_off else 0)
  outs = []
  for rep in range(2):
    flat = torch.full((n_rows * stride + 2 * G + 1,), float('nan'), dtype=torch.float32, device=DEV)
    flat[off:off + n_rows * stride] = torch.from_numpy(init.reshape(-1)).to(DEV)
    table = torch.as_strided(flat, (n_rows, dim), (stride, 1), off)
    opt = K.make_opt(_lib.OPT_SGD, 1.0, grad_scale=gs)
    wsk = ws if ws is not None else K.bwd_workspace(case.cap, DEV, dim)
    uq = None
    kw = dict(weights=case.w_t, seg_ids=case.seg_t, row_ptr=case.rp_t, seg_scale=case.sc_t)
    if engine == 'radix':
      ur_buf = torch.full((case.cap + 2 * G,), -7, dtype=torch.int64, device=DEV)
      ug_buf = torch.full((case.cap * dim + 2 * G,), float('nan'), dtype=torch.float32, device=DEV)
      nu = torch.full((1,), -7, dtype=torch.int32, device=DEV)
      kw.update(uniq_rows=ur_buf[G:G + case.cap], uniq_grads=ug_buf[G:G + case.cap * dim].view(case.cap, dim),
                n_uniq=nu)
    if presort:
      pre = K.bwd_workspace(case.cap, DEV, dim)
      K.embedding_bwd_presort(case.rows_t, n_rows, dim, pre, case.sd, case.n_slots, seg_ids=case.seg_t,
                              row_ptr=case.rp_t, n_seg=case.n_seg)
      kw['sorted_from'] = (pre, dim)
    K.embedding_bwd(table, None, None, dim, case.rows_t, case.sd, case.n_slots, case.n_seg, views, opt, wsk, **kw)
    torch.cuda.synchronize()
    got = flat.cpu().numpy()
    assert np.isnan(got[:off]).all() and np.isnan(got[off + n_rows * stride:]).all(), 'wrote into a table guard'
    tab = got[off:off + n_rows * stride].reshape(n_rows, stride)
    if engine == 'radix':
      urb, ugb = ur_buf.cpu().numpy(), ug_buf.cpu().numpy()
      assert (urb[:G] == -7).all() and (urb[-G:] == -7).all(), 'wrote into a uniq_rows guard'
      assert np.isnan(ugb[:G]).all() and np.isnan(ugb[-G:]).all(), 'wrote into a uniq_grads guard'
      uq = (int(nu.item()), urb[G:G + case.cap], ugb[G:G + case.cap * dim].reshape(case.cap, dim))
    outs.append((tab, uq))
  for (t, _), b in zip(case.bufs_t, case.bufs_np):
    assert torch.isnan(t[:G]).all() and torch.isnan(t[-G:]).all(), 'a gradient buffer guard changed'
  (t0, u0), (t1, u1) = outs
  assert np.array_equal(t0.view(np.int32), t1.view(np.int32)), 'a repeated call is not bit-identical'
  if u0 is not None:
    assert u0[0] == u1[0] and np.array_equal(u0[1], u1[1]) and np.array_equal(u0[2].view(np.int32),
                                                                             u1[2].view(np.int32)), \
        'a repeated call is not bit-identical (uniq outputs)'
  if check:
    _check(case, engine, t0, u0, init, gs, misalign=table_off or gbuf_off or stride % 4 != 0)
  return t0, u0


def _check(case, engine, tab, uq, init, gs, misalign):
  dim = case.dim
  untouched = np.ones(case.n_rows, bool)
  untouched[case.urow] = False
  assert np.array_equal(tab[untouched].view(np.int32), init[untouched].view(np.int32)), \
      'rows no live lookup touches changed (%d rows)' % (tab[untouched] != init[untouched]).any(1).sum()
  assert np.isnan(tab[:, dim:]).all(), 'row_stride padding changed'
  lab, exact = case.paths(engine, misalign)
  bound = case.bound()
  got = tab[case.urow, :dim]
  if engine == 'radix':
    n, ur, ug = uq
    assert n == case.urow.size, 'n_uniq %d, expected %d' % (n, case.urow.size)
    assert np.array_equal(ur[:n], case.urow), 'uniq_rows'
    assert np.isnan(ug[n:]).all(), 'uniq_grads past n_uniq changed'
    ug = ug[:n]
    assert np.array_equal(got.view(np.int32), (F32(0) - (ug * F32(1))).astype(F32).view(np.int32)), \
        'table rows are not fsub(0, uniq_grads)'
    _cmp(ug.astype(np.float64), case.G64 * gs, (bound + U * np.abs(case.G64)) * gs, lab, exact, ug,
         (case.seq32 * F32(gs)).astype(F32), 'uniq_grads', (case.G64 * gs).astype(F32) if case.dyadic else None)
  else:
    _cmp(-got.astype(np.float64), case.G64, bound, lab, exact, got, (F32(0) - case.seq32).astype(F32), 'table',
         (F32(0) - case.G64.astype(F32)).astype(F32) if case.dyadic else None)


def _cmp(val, ref, bound, lab, exact, got32, ex32, what, ex_all=None):
  for p in np.unique(lab):
    m = lab == p
    err = np.abs(val[m] - ref[m])
    ratio = err / bound[m]
    bad = ~(ratio <= 1.0)
    assert not bad.any(), '%s, path %s: %d elements off by more than the bound (worst %.3g x bound, first at row %d)' % (
        what, p, bad.sum(), np.nanmax(np.where(np.isnan(ratio), np.inf, ratio)), np.nonzero(bad.any(1))[0][0])
    WORST[p] = max(WORST.get(p, 0.0), float(ratio.max()) if ratio.size else 0.0)
  if ex_all is not None:
    # every order of these sums is exact, so every path must return G; compared by value: the sign of a zero G
    # depends on whether a sum starts from +0 (the shuffle-scan trees start from the first term)
    d = (got32 != ex_all).any(1)
    assert not d.any(), '%s: %d rows differ from the exact G (paths %s)' % (what, d.sum(), sorted(set(lab[d])))
  if exact.any():
    a, b = got32[exact].view(np.int32), ex32[exact].view(np.int32)
    assert np.array_equal(a, b), '%s: %d rows on sequential paths differ from the lookup-order sum (paths %s)' % (
        what, (a != b).any(1).sum(), sorted(set(lab[exact][(a != b).any(1)])))


# ---- row streams with a bucket of a chosen size -------------------------------------------------------------------
def _recipe(size, rng):
  """run lengths that fill a bucket of `size` pairs"""
  if size <= WARP_CAP:
    base, lo, hi = [], 1, 7
  elif size <= CAP + 1:
    base, lo, hi = [COOP_RUN, COOP_RUN + 1], 1, 41
  else:
    base, lo, hi = [COOP_RUN, COOP_RUN + 1, QUEUE_RUN + 1], 20, 401
  out = [x for x in base if x <= size]
  tot = sum(out)
  while tot < size:
    x = min(int(rng.integers(lo, hi)), size - tot)
    out.append(x)
    tot += x
  return out


def stream(rng, dim, recipe, n_bg, n_rows, extra=0, drop=0.05):
  """lookup rows: runs of `recipe` lengths on distinct rows of one bucket (that of row n_rows - 1, whose runs come
  last in it), ascending by row in recipe order, plus n_bg background lookups in other buckets (row 0 among them,
  `drop` of them dropped).  Returns (rows shuffled, the bucket)."""
  cap = sum(recipe) + n_bg + extra
  lg = _log2(num_buckets(cap, K.k7_warp_mode(dim)))
  allr = np.arange(n_rows)
  bk = bucket_of(allr, lg)
  b = bk[-1]
  assert b != bk[0]
  cand = allr[(bk == b) & (allr != n_rows - 1)]
  assert cand.size >= len(recipe) - 1, 'n_rows too small for the recipe'
  rb = np.sort(np.concatenate([rng.choice(cand, len(recipe) - 1, replace=False), [n_rows - 1]]))
  live = np.repeat(rb, recipe)
  pool = allr[(bk != b)]
  pool = np.concatenate([[0], rng.choice(pool, max(1, n_bg // 3), replace=False)])
  bg = rng.choice(pool, n_bg)
  bg[rng.random(n_bg) < drop] = -1
  rows = np.concatenate([live, bg])
  return rows[rng.permutation(rows.size)], b


def _slots_even(n_seg, n_slots, rng, modes=None):
  cuts = np.sort(rng.integers(0, n_seg + 1, n_slots - 1))
  sb = np.concatenate([[0], cuts])
  ns = np.diff(np.concatenate([sb, [n_seg]]))
  return [(int(sb[f]), int(ns[f]), NONE if modes is None else modes[f]) for f in range(n_slots)]


def single_case(rng, dim, rows, n_rows, n_slots=3, **kw):
  return Case(rng, dim, n_rows, rows, _slots_even(rows.size, n_slots, rng), rows.size, **kw)


def csr_case(rng, dim, rows, n_rows, n_slots=3, extra=5, **kw):
  """CSR over `rows` (live); `extra` lookups past the live count point at valid rows and at an empty segment"""
  n_live = rows.size
  lens = []
  tot = 0
  while tot < n_live:
    x = min(int(rng.integers(0, 4)), n_live - tot)
    lens.append(x)
    tot += x
  lens.append(0)
  n_seg = len(lens)
  seg = np.repeat(np.arange(n_seg), lens)
  past_rows = rng.choice(rows[rows >= 0], extra) if extra else np.zeros(0, np.int64)
  all_rows = np.concatenate([rows, past_rows])
  all_seg = np.concatenate([seg, np.full(extra, n_seg - 1)])
  return Case(rng, dim, n_rows, all_rows, _slots_even(n_seg, n_slots, rng), n_seg, seg=all_seg, n_live=n_live, **kw)


def _reached(case, engine, want, misalign=False):
  lab, _ = case.paths(engine, misalign)
  got = set(lab)
  assert set(want) <= got, 'paths %s not reached (reached %s)' % (sorted(set(want) - got), sorted(got))


def _role_of_size(dim, size):
  if K.k7_warp_mode(dim) and size <= WARP_CAP:
    return 'warp'
  return 'cta' if size <= CAP else ('big' if size <= BIG_CAP else 'big_radix')


# ---- bucket roles --------------------------------------------------------------------------------------------------
SIZES = [1, 32, 33, 127, 128, 129, 1024, 1025]
BIG_SIZES = [16384, 16385, 20000]
BIG_DIMS = [1, 16, 64]


@pytest.mark.parametrize('size', SIZES + BIG_SIZES)
@pytest.mark.parametrize('dim', ALL_DIMS)
def test_bucket_roles(dim, size):
  if size in BIG_SIZES and dim not in BIG_DIMS:
    pytest.skip('big buckets at dims %s' % BIG_DIMS)
  rng = np.random.default_rng(dim * 100003 + size)
  n_rows = 65536 if size in BIG_SIZES else N_ROWS
  rows, b = stream(rng, dim, _recipe(size, rng), 300, n_rows)
  case = single_case(rng, dim, rows, n_rows, n_slots=2, wmode='given', scale=size % 2 == 1)
  cnt, _ = case.bucket_counts()
  assert cnt[b] == size, 'the crafted bucket holds %d pairs, not %d' % (cnt[b], size)
  want = [_role_of_size(dim, size)]
  if size > QUEUE_RUN:
    want.append('hot')
  _reached(case, 'bucketed', want)
  run(case, layout=('separate', 'interleaved')[(SIZES + BIG_SIZES).index(size) % 2])


# ---- run lengths at the boundaries -------------------------------------------------------------------------------
WARP_RUNS = [(0, 31), (0, 32), (0, 33), (0, 64), (0, 96), (0, 128), (1, 31), (1, 32), (1, 33), (31, 33), (32, 32),
             (32, 64), (64, 64), (96, 32)]


@pytest.mark.parametrize('prefix,run_len', WARP_RUNS)
@pytest.mark.parametrize('dim', [1, 4, 32])
def test_warp_run_boundaries(dim, prefix, run_len):
  """a run of run_len pairs that starts `prefix` pairs into a warp bucket (after single-lookup runs on smaller rows)"""
  rng = np.random.default_rng(dim * 1000 + prefix * 7 + run_len)
  recipe = [1] * prefix + [run_len]
  rows, b = stream(rng, dim, recipe, 200, N_ROWS)
  case = single_case(rng, dim, rows, N_ROWS, wmode='given')
  cnt, _ = case.bucket_counts()
  assert cnt[b] == prefix + run_len <= WARP_CAP
  lab, exact = case.paths('bucketed')
  i = np.searchsorted(case.urow, N_ROWS - 1)
  assert lab[i] == 'warp' and case.run_len[i] == run_len
  run(case)


@pytest.mark.parametrize('run_len', [48, 49, 4096, 4097, 4607, 4608, 4609, 5121])
@pytest.mark.parametrize('dim', [3, 16, 64, 300])
def test_cta_run_boundaries(dim, run_len):
  """the whole-CTA tree (> 48) in a medium bucket, the hot-row kernel (> 4096, kChunk = 512 lookups per chunk) in a
  big one"""
  rng = np.random.default_rng(dim * 1000 + run_len)
  pad = [2] * (80 if run_len < 100 else 0)   # warp placement: make the bucket a CTA one
  recipe = pad + [run_len]
  rows, b = stream(rng, dim, recipe, 300, N_ROWS)
  case = csr_case(rng, dim, rows, N_ROWS, wmode='unit', scale=True) if run_len % 2 else \
      single_case(rng, dim, rows, N_ROWS, wmode='given')
  lab, _ = case.paths('bucketed')
  i = np.searchsorted(case.urow, N_ROWS - 1)
  want = 'hot' if run_len > QUEUE_RUN else ('coop' if run_len > COOP_RUN else ('cta'))
  assert lab[i] == want and case.run_len[i] == run_len, (lab[i], case.run_len[i])
  run(case, layout='interleaved' if dim == 64 else 'separate')


# ---- radix engine --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('csr', [False, True], ids=['single', 'csr'])
@pytest.mark.parametrize('dim', ALL_DIMS)
def test_radix_engine(dim, csr):
  rng = np.random.default_rng(dim * 17 + csr)
  recipe = [1, 2, 63, 64, 65, 511, 512, 513, 1025, 3]
  rows, _ = stream(rng, dim, recipe, 400, N_ROWS)
  if csr:
    case = csr_case(rng, dim, rows, N_ROWS, wmode='given', scale=True, n_bufs=2)
  else:
    case = single_case(rng, dim, rows, N_ROWS, wmode='unit', n_bufs=3)
  _reached(case, 'radix', ['radix_hot'])
  run(case, engine='radix', gs=0.375, layout='interleaved' if csr else 'separate')


# ---- inputs ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('scale', [False, True], ids=['no_scale', 'seg_scale'])
@pytest.mark.parametrize('wmode', ['none', 'given', 'unit'])
@pytest.mark.parametrize('csr', [False, True], ids=['single', 'csr'])
@pytest.mark.parametrize('dim', [4, 12])
def test_inputs(dim, csr, wmode, scale):
  """four slots with the sum, mean, sqrtn and sum combiners (K7 reads only the UNIT_WEIGHTS flag of a combiner)"""
  rng = np.random.default_rng(dim + 100 * csr + 1000 * len(wmode) + 10000 * scale)
  rows, _ = stream(rng, dim, _recipe(200, rng), 600, N_ROWS, drop=0.15)
  mk = csr_case if csr else single_case
  case = mk(rng, dim, rows, N_ROWS, n_slots=4, wmode=wmode, scale=scale, n_bufs=2)
  run(case)


@pytest.mark.parametrize('n_bufs', [1, 3, 8])
@pytest.mark.parametrize('n_slots', [1, 257, 2048])
@pytest.mark.parametrize('dim', [1, 6])
def test_slots_and_buffers(dim, n_slots, n_bufs):
  rng = np.random.default_rng(dim * 100 + n_slots + n_bufs)
  rows, _ = stream(rng, dim, _recipe(150, rng), 3000, N_ROWS)
  case = single_case(rng, dim, rows, N_ROWS, n_slots=n_slots, wmode='unit', scale=True, n_bufs=n_bufs)
  assert (case.slot_n == 0).any() or n_slots == 1
  run(case, layout='interleaved' if n_bufs == 3 else 'separate')
  if n_slots == 2048:
    case = csr_case(rng, dim, rows, N_ROWS, n_slots=n_slots, wmode='given', n_bufs=n_bufs)
    run(case, engine='radix', gs=0.5)


# ---- one-row slots -------------------------------------------------------------------------------------------------
def one_row_case(rng, dim, plan, n_rows=4096, n_bufs=2, wmode='given', scale=True, dyadic=False):
  """plan: (n_seg, 'one' | 'one0' | 'ids') per slot; a one-row slot reads its own row (a few lookups dropped; 'one0':
  its first lookup among them), the id slots draw from rows below n_rows - 8"""
  rows, slots, sb = [], [], 0
  k = 0
  for n, kind in plan:
    if kind in ('one', 'one0'):
      r = np.full(n, n_rows - 1 - k, np.int64)
      r[rng.random(n) < 0.03] = -1
      r[0] = -1 if kind == 'one0' else r[0]
      k += 1
    else:
      r = rng.integers(0, n_rows - 8, n)
      r[rng.random(n) < 0.05] = -1
    rows.append(r)
    slots.append((sb, n, NONE if kind == 'ids' else ONE_ROW))
    sb += n
  rows = np.concatenate(rows)
  return Case(rng, dim, n_rows, rows, slots, rows.size, wmode=wmode, scale=scale, n_bufs=n_bufs, dyadic=dyadic)


ONE_ROW_PLANS = {
    'b1500': [(1500, 'ids'), (1500, 'one'), (1500, 'ids')],
    'three': [(700, 'one'), (700, 'ids'), (700, 'one'), (700, 'ids'), (700, 'one')],
    'long_beside_short': [(10, 'ids'), (1500, 'one')],
    'long_beside_empty': [(0, 'ids'), (1100, 'one'), (0, 'ids'), (0, 'ids')],
    'first_dropped': [(600, 'one0'), (600, 'ids'), (1300, 'one0')],
}


@pytest.mark.parametrize('plan', sorted(ONE_ROW_PLANS))
@pytest.mark.parametrize('dim', [3, 4, 16, 300])
def test_one_row(dim, plan):
  rng = np.random.default_rng(dim * 31 + len(plan))
  case = one_row_case(rng, dim, ONE_ROW_PLANS[plan])
  _reached(case, 'bucketed', ['one_row'])
  ws = K.bwd_workspace(case.cap, DEV, dim)
  first, _ = run(case, ws=ws)
  again, _ = run(case, ws=ws)   # a second call on the same workspace (its tickets must be back at zero)
  assert np.array_equal(first.view(np.int32), again.view(np.int32))
  run(case, engine='radix', gs=0.75)   # the same lookups through the dedup


# ---- scalar fallback -----------------------------------------------------------------------------------------------
MISALIGN = [(4, 'table_off'), (8, 'table_off'), (16, 'table_off'), (16, 'stride17'), (16, 'gbuf_off'),
            (32, 'gbuf_off'), (64, 'table_off'), (128, 'gbuf_off')]


@pytest.mark.parametrize('engine', ['bucketed', 'radix'])
@pytest.mark.parametrize('dim,how', MISALIGN)
def test_scalar_fallback(dim, how, engine):
  rng = np.random.default_rng(dim * 7 + len(how))
  rows, _ = stream(rng, dim, _recipe(1025, rng), 400, N_ROWS)
  case = single_case(rng, dim, rows, N_ROWS, wmode='given', scale=True, n_bufs=2)
  kw = dict(table_off=how == 'table_off', gbuf_off=how == 'gbuf_off', stride=17 if how == 'stride17' else None)
  mis, _ = run(case, engine=engine, **kw)
  ali, _ = run(case, engine=engine, check=False)
  _, ex_mis = case.paths(engine, misalign=True)
  _, ex_ali = case.paths(engine, misalign=False)
  both = ex_mis & ex_ali
  if engine == 'radix' and dim <= 32:
    # the aligned radix call sums every run of these dims with the warp's shuffle-scan tree: no row is sequential in
    # both calls, and run() has already held the misaligned call to the lookup-order restatement
    assert not both.any()
    return
  assert both.any()
  a, b = mis[case.urow][both, :dim], ali[case.urow][both, :dim]
  assert np.array_equal(a.view(np.int32), b.view(np.int32)), 'the scalar fallback differs from the aligned call'


# ---- presort / reuse -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['one_row', 'csr'])
@pytest.mark.parametrize('dim', [1, 16, 12, 64])
def test_presort_reuse(dim, kind):
  rng = np.random.default_rng(dim + len(kind))
  if kind == 'one_row':
    case = one_row_case(rng, dim, ONE_ROW_PLANS['long_beside_short'] + [(900, 'ids'), (600, 'one')])
  else:
    rows, _ = stream(rng, dim, _recipe(1025, rng), 500, N_ROWS)
    case = csr_case(rng, dim, rows, N_ROWS, wmode='unit', scale=True)
  fresh, _ = run(case)
  reused, _ = run(case, presort=True)
  assert np.array_equal(fresh.view(np.int32), reused.view(np.int32)), 'presort + reuse_sort differs from a fresh call'


# ---- every summation order exact -------------------------------------------------------------------------------------
SHORT_RUNS = [1, 5, 33, 48, 49, 64, 65, 511, 512, 513, 1025]
DYADIC = {   # bucketed runs around kCoopRun, kQueueRun and kChunk multiples; radix runs around kLongRun and kChunk
    'big': (SHORT_RUNS + [4096, 4097, 5121], ['big', 'coop', 'hot']),                  # 16140 pairs: bitonic CTA
    'big_radix': (SHORT_RUNS + [4096, 4097, 4608, 4609], ['big_radix', 'coop', 'hot']),  # 20236: global radix sort
    'radix': (SHORT_RUNS + [4097], ['radix_hot']),
}


@pytest.mark.parametrize('kind', sorted(DYADIC) + ['one_row'])
@pytest.mark.parametrize('dim', [1, 16, 64, 300])
def test_dyadic_exact(dim, kind):
  """gradients in -8..8 and coefficients in {+-0.5, +-1, +-2} x {0.5, 1, 2}: every partial sum of these runs is a
  multiple of 1/4 below 2^18, exact in float32 in any order, so the tree paths (whole-CTA tree, hot-row chunks,
  one-row partials, shuffle scans) must return G64 bit for bit, and a lookup dropped or counted twice at a chunk
  boundary cannot hide under the rounding bound"""
  rng = np.random.default_rng(dim * 7919 + len(kind))
  if kind == 'one_row':
    case = one_row_case(rng, dim, [(1500, 'one0'), (700, 'ids'), (1100, 'one')], dyadic=True)
    want, engines = ['one_row'], ['bucketed', 'radix']
  else:
    recipe, want = DYADIC[kind]
    rows, _ = stream(rng, dim, recipe, 300, 8192)
    case = single_case(rng, dim, rows, 8192, wmode='given', scale=True, n_bufs=2, dyadic=True)
    engines = ['radix' if kind == 'radix' else 'bucketed']
  assert np.array_equal(case.G64, case.G64.astype(F32).astype(np.float64)), 'G is not exact in float32'
  _reached(case, engines[0], want)
  for e in engines:
    run(case, engine=e, gs=0.5 if e == 'radix' else 1.0)


# ---- dim limit -------------------------------------------------------------------------------------------------------
def test_dim_limit():
  rng = np.random.default_rng(4096)
  rows, _ = stream(rng, 4096, [3, 1, 60], 20, 256)
  case = single_case(rng, 4096, rows, 256, wmode='given')
  run(case)
  run(case, engine='radix', gs=0.5)
  case.dim = 4097
  case.bufs_np = [np.zeros(1, F32)]
  t = torch.zeros(256, 4097, device=DEV)
  ws = K.bwd_workspace(case.cap, DEV, 4097)
  with pytest.raises(_lib.ErError, match='dim must be at most 4096'):
    K.embedding_bwd(t, None, None, 4097, torch.from_numpy(case.rows).to(DEV), K.slots_to_device(case.slots_np, DEV),
                    case.n_slots, case.n_seg, [torch.zeros(case.cap, 4100, device=DEV)],
                    K.make_opt(_lib.OPT_SGD, 1.0), ws)


def test_zz_report_worst():
  print('worst error / bound: %s' % ', '.join('%s %.3f' % kv for kv in sorted(WORST.items())))
  print('peak reserved device memory: %.2f GiB' % (torch.cuda.max_memory_reserved() / 2 ** 30))
