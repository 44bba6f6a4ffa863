"""GPU: the optimizer updates against float64, on the state layouts they write through, called through the C ABI.

  er_dense_apply        every kind; segment tables of n = 1, 255..257, 511..513, empty segments first / inside / last,
                        8192 mixed segments, one segment of 10^6 + 3 (every CTA loops over several chunks); per-segment
                        l2 (some zero) and lr_mult, grad_scale != 1, NaN gaps between the segments; rate from lr_dev,
                        hyper_dev or the struct (the losing sources are deliberately wrong); reg_loss_out; ten Adam
                        steps; refusals
  FlatDenseOptimizer    the kernels, biases, gamma and beta of a [624, 256, 128, 64] DNN, three steps, fold_l2 + apply
  er_sparse_apply       every kind x {separate, interleaved Arena} x dims 1/4/6/16/128; -1 rows, the n_uniq clamp from
                        both sides, hyper_dev against the struct
  er_adam_dense_sweep   vector path (dim 16, separate and row_stride 48) and scalar path (dim 6, row_stride 18, m not
                        16-byte aligned); touched NULL / given; rows with m = v = 0 and with m = 0, v != 0
  er_mark_rows          the n_dev clamp, rows < 0 or >= n_rows, value 0
  er_embedding_bwd      the K7 row rule, every kind x {separate, interleaved} x dims 1/4/8/16/32/64/128/6/12 (the d1,
                        warp-mode vector, CTA vector and scalar engines); runs of 65 and 600 lookups of one row on an
                        interleaved arena; the emit form (table NULL, uniq_rows / uniq_grads / n_uniq)

References are float64 restatements of TF's ApplyAdagrad / SparseApplyAdagrad, ApplyAdam / lazy Adam, ApplyMomentum and
plain SGD, evaluated on the fp32 tensors each kernel received.  Each reference value carries a bound on how far the
kernel's fp32 result may lie from it, propagated through the kernel's operation sequence: every rounded operation adds
u = 2^-24 of its result (the kernels use correctly rounded __fmul_rn / __fdiv_rn / __fsqrt_rn / __frsqrt_rn, and the
library is built without fast-math); the error already carried by the operands goes through the operation exactly
(a * b: |a| eb + |b| ea + ea eb; a / b: (ea + |a/b| eb) / (|b| - eb); sqrt and rsqrt: their value at the far end of the
operand's interval).  A fused multiply-add in dense.cu rounds once where the bound counts two, so possible FMA
contraction stays inside it.  A sum of n terms in any order adds (n - 1) u sum|terms| (the hot rows of K7, reg_loss_out,
whose float atomics add the per-warp partials in no fixed order).  Comparisons allow C = 2 times the bound plus 2^-140.
Where the same operations run on the same inputs the results must be bit-identical: the struct, hyper_dev and lr_dev
rate sources, and the update with and without reg_loss_out.

Every output lies inside NaN-filled memory: the gaps between dense segments, the guards around separate tables, the
gradients past n_cap.  Rows an update must not touch are compared bit for bit with their input, whole storage matrix
included, so an update that wrote a state column through the wrong stride, or read a gradient it must not, fails.

Worst error / bound measured on an H100 80GB HBM3 (400 W power limit), the 195 tests in about 7 s at 0.6 GiB peak
device memory (0.5 means the error reached the first-order bound itself, before the slack C): er_dense_apply 0.50 (the
8192-segment and 10^6-element tables included), K7 0.49 for single lookups and 0.49 for the hot rows, er_sparse_apply
0.49, the sweep 0.49, FlatDenseOptimizer 0.48, K7 uniq_grads 0.42, the ten Adam steps 0.42; reg_loss_out 0.027 (its
bound charges one float atomic per warp of the grid), FlatDenseOptimizer reg_loss 0.001.
"""
import ctypes

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, kernels as K
from easyrec_b200.embedding import Arena
from easyrec_b200.kernels import _p, _stream

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
C = 2.0
FLOOR = 2.0 ** -140
G = 64                   # guard elements around every separate output (256 bytes: keeps 16-byte alignment)
SGD, ADAGRAD, LAZY_ADAM, ADAM_ROWS, MOMENTUM = (_lib.OPT_SGD, _lib.OPT_ADAGRAD, _lib.OPT_LAZY_ADAM, _lib.OPT_ADAM_ROWS,
                                                _lib.OPT_MOMENTUM)
KINDS = [SGD, ADAGRAD, LAZY_ADAM, ADAM_ROWS, MOMENTUM]
KIND_IDS = ['sgd', 'adagrad', 'lazy_adam', 'adam_rows', 'momentum']
N_STATE = {SGD: 0, ADAGRAD: 1, MOMENTUM: 1, LAZY_ADAM: 2, ADAM_ROWS: 2}
B1, B2, EPS = 0.9, 0.999, 1e-8
MAX_CTAS = 8 * 132       # er_dense_apply's grid cap (8 waves of the H100's 132 SMs)
WORST = {}


def _f32(x):
  return np.float32(x)


def _adam(kind):
  return kind in (LAZY_ADAM, ADAM_ROWS)


# ---- float64 values with a bound on the fp32 kernel's distance from them ----------------------------------------------
class R(object):
  """v: the float64 reference; e: bound on |fp32 kernel result - v| (same shape)."""

  def __init__(self, v, e=None):
    self.v = v
    self.e = torch.zeros_like(v) if e is None else e

  def __getitem__(self, i):
    return R(self.v[i], self.e[i])


def X(t):
  """an input the kernel holds exactly in fp32"""
  if not torch.is_tensor(t):
    t = torch.tensor(float(_f32(t)), dtype=torch.float64, device=DEV)
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
  assert bool((lo > 0).all()), 'divisor interval contains 0'
  return _rnd(v, (a.e + v.abs() * b.e) / lo)


def sqrt(a):
  v = a.v.sqrt()
  return _rnd(v, v - (a.v - a.e).clamp_min(0.0).sqrt())


def rsqrt(a):
  assert bool((a.v > a.e).all()), 'rsqrt operand interval reaches 0'
  v = a.v.rsqrt()
  return _rnd(v, (a.v - a.e).rsqrt() - v)


def where(m, a, b):
  return R(torch.where(m, a.v, b.v), torch.where(m, a.e, b.e))


def lr_t_of(lr, b1p, b2p):
  """adam_lr_t_of: lr * sqrt(1 - b2^t) / (1 - b1^t), each operation rounded"""
  return div(mul(X(lr), sqrt(sub(X(1.0), X(b2p)))), sub(X(1.0), X(b1p)))


def lr_t_f32(lr, b1p, b2p):
  """the same rate as the fp32 value a caller passes in lr_dev"""
  one = _f32(1.0)
  return float(_f32(_f32(_f32(lr) * np.sqrt(one - _f32(b2p))) / (one - _f32(b1p))))


def rule(kind, w, s0, s1, g, lr):
  """upd_one (csrc/embedding_bwd.cu) and dense_apply_kernel (csrc/dense.cu) on reference values; lr is lr_t for the
  Adam kinds.  Returns (w, s0, s1)."""
  if kind == ADAGRAD:       # ApplyAdagrad: acc += g^2 ; w -= lr * g * rsqrt(acc)
    s0 = add(s0, mul(g, g))
    w = sub(w, mul(mul(lr, g), rsqrt(s0)))
  elif _adam(kind):         # ApplyAdam / lazy Adam on the row: m, v decay-and-add, w -= lr_t * m / (sqrt(v) + eps)
    s0 = add(mul(g, sub(X(1.0), X(B1))), mul(s0, X(B1)))
    s1 = add(mul(mul(g, g), sub(X(1.0), X(B2))), mul(s1, X(B2)))
    w = sub(w, div(mul(lr, s0), add(sqrt(s1), X(EPS))))
  elif kind == MOMENTUM:    # ApplyMomentum: accum = accum * momentum + g ; w -= lr * accum
    s0 = add(mul(s0, X(B1)), g)
    w = sub(w, mul(lr, s0))
  else:
    w = sub(w, mul(lr, g))
  return w, s0, s1


def _within(got, ref, what):
  got = got.double()
  assert bool(torch.isfinite(got).all()), '%s: non-finite result' % what
  err = (got - ref.v).abs()
  bound = C * ref.e + FLOOR
  ratio = float((err / bound).max()) if err.numel() else 0.0
  WORST[what] = max(WORST.get(what, 0.0), ratio)
  assert ratio <= 1.0, '%s: error %.3g x bound (max abs err %.3g)' % (what, ratio, float(err.max()))


def _same(a, b, what):
  assert torch.equal(a, b) or bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all()), what + ': not bit-identical'


def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


def _out(rows, cols):
  """(buffer, view): a [rows, cols] matrix inside a NaN-filled buffer with G guard elements each side"""
  buf = torch.full((2 * G + rows * cols,), float('nan'), device=DEV)
  return buf, buf.as_strided((rows, cols), (cols, 1), G)


def _guards_nan(buf, what):
  assert bool(torch.isnan(buf[:G]).all() and torch.isnan(buf[-G:]).all()), what + ': wrote into a guard'


def _fill_state(kind, mats, gen):
  """w ~ N(0, 0.5); Adagrad accumulators in [0.05, 0.95]; Adam m ~ N(0, 0.1), v in [1e-4, 0.2]; momentum ~ N(0, 0.1)"""
  w, s0, s1 = mats
  w.copy_(torch.randn(w.shape, generator=gen, device=DEV) * 0.5)
  if kind == ADAGRAD:
    s0.copy_(torch.rand(s0.shape, generator=gen, device=DEV) * 0.9 + 0.05)
  elif _adam(kind):
    s0.copy_(torch.randn(s0.shape, generator=gen, device=DEV) * 0.1)
    s1.copy_(torch.rand(s1.shape, generator=gen, device=DEV) * 0.2 + 1e-4)
  elif kind == MOMENTUM:
    s0.copy_(torch.randn(s0.shape, generator=gen, device=DEV) * 0.1)


def _storage(kind, n_rows, dim, layout, gen):
  """([w, s0, s1] with None for the states the kind does not have, guard buffers): three separate matrices inside
  NaN-filled buffers, or the interleaved [w | state0 | state1] rows of Arena.materialize(interleave=True)"""
  if layout == 'interleaved':
    ar = Arena(dim, DEV)
    ar.add_table('t', n_rows)
    ar.materialize(kind, interleave=True)
    assert ar.weight.stride(0) == (1 + N_STATE[kind]) * dim
    mats, bufs = [ar.weight, ar.state0, ar.state1], []
  else:
    mats, bufs = [], []
    for i in range(3):
      if i <= N_STATE[kind]:
        b, v = _out(n_rows, dim)
        bufs.append(b)
        mats.append(v)
      else:
        mats.append(None)
  _fill_state(kind, mats, gen)
  return mats, bufs


def _restore(mats, init):
  for m, i in zip(mats, init):
    if m is not None:
      m.copy_(i)


def _snap(mats):
  return [None if m is None else m.clone() for m in mats]


def _check_rows(kind, got, init, rows, ref, what):
  """the updated rows against the reference, every other row of every matrix bit-identical to its input"""
  names = ('w', 's0', 's1')
  for i in range(1 + N_STATE[kind]):
    keep = torch.ones(got[i].shape[0], dtype=torch.bool, device=DEV)
    keep[rows] = False
    _same(got[i][keep], init[i][keep], '%s %s untouched rows' % (what, names[i]))
    _within(got[i][rows], ref[i], '%s %s' % (what, names[i]))


# ---- er_dense_apply -----------------------------------------------------------------------------------------------
def _dense_apply(p, g, s0, s1, segs_dev, n_segs, max_n, opt, lr_dev=None, reg=None):
  return _lib.load().er_dense_apply(_p(p), _p(g), _p(s0), _p(s1), _p(segs_dev), n_segs, max_n, ctypes.byref(opt),
                                    _p(lr_dev), _p(reg), _stream())


class Dense(object):
  """flat p / g / s0 / s1 buffers with segments of `sizes` separated by NaN gaps of 1..5 floats, a segment table with
  per-segment l2 (about a third zero) and lr_mult in [0.25, 3]"""

  def __init__(self, kind, sizes, seed):
    rng = np.random.default_rng(seed)
    self.kind, self.sizes = kind, list(sizes)
    n = len(sizes)
    gaps = rng.integers(1, 6, n + 1)
    offs = np.zeros(n, np.int64)
    o = int(gaps[0])
    for i, sz in enumerate(sizes):
      offs[i] = o
      o += int(sz) + int(gaps[i + 1])
    self.total = o
    segs = np.zeros(n, dtype=_lib.DENSE_SEG_DTYPE)
    segs['offset'], segs['n'] = offs, sizes
    l2 = rng.uniform(1e-3, 0.3, n).astype(np.float32)
    l2[rng.random(n) < 0.35] = 0.0
    segs['l2'] = l2
    segs['lr_mult'] = rng.uniform(0.25, 3.0, n).astype(np.float32)
    self.segs = segs
    self.segs_dev = torch.from_numpy(segs.view(np.uint8).reshape(-1).copy()).to(DEV)
    self.n_segs, self.max_n = n, max(1, int(max(sizes)))
    sz = np.asarray(sizes, np.int64)
    starts = np.repeat(offs, sz)
    within = np.arange(int(sz.sum())) - np.repeat(np.cumsum(sz) - sz, sz)
    self.idx = torch.from_numpy(starts + within).to(DEV)
    self.l2e = torch.from_numpy(np.repeat(l2, sz)).to(DEV).double()
    self.lrme = torch.from_numpy(np.repeat(segs['lr_mult'], sz)).to(DEV).double()
    self.live = torch.zeros(self.total, dtype=torch.bool, device=DEV)
    self.live[self.idx] = True
    gen = _gen(seed)
    nl = self.idx.numel()
    self.bufs = [torch.full((self.total,), float('nan'), device=DEV) for _ in range(4)]
    self.p, self.g, self.s0, self.s1 = self.bufs
    self.p[self.idx] = torch.randn(nl, generator=gen, device=DEV)
    self.g[self.idx] = torch.randn(nl, generator=gen, device=DEV)
    if kind == ADAGRAD:
      self.s0[self.idx] = torch.rand(nl, generator=gen, device=DEV) * 0.9 + 0.05
    elif _adam(kind):
      self.s0[self.idx] = torch.randn(nl, generator=gen, device=DEV) * 0.1
      self.s1[self.idx] = torch.rand(nl, generator=gen, device=DEV) * 0.2 + 1e-4
    elif kind == MOMENTUM:
      self.s0[self.idx] = torch.randn(nl, generator=gen, device=DEV) * 0.1

  def states(self):
    """the state pointers the kind takes (SGD: both NULL, Adagrad / momentum: state1 NULL)"""
    ns = N_STATE[self.kind]
    return (self.s0 if ns >= 1 else None), (self.s1 if ns >= 2 else None)

  def run(self, opt, lr_dev=None, reg=None):
    s0, s1 = self.states()
    rc = _dense_apply(self.p, self.g, s0, s1, self.segs_dev, self.n_segs, self.max_n, opt, lr_dev, reg)
    _lib.check(rc, 'er_dense_apply')

  def snap(self):
    return [b.clone() for b in self.bufs]

  def restore(self, snap):
    for b, s in zip(self.bufs, snap):
      b.copy_(s)

  def ref(self, lr0, gs, w=None, s0=None, s1=None):
    """(w, s0, s1) over the live elements, from the current buffers (or the given carried references)"""
    i = self.idx
    w = X(self.p[i]) if w is None else w
    s0 = X(self.s0[i]) if s0 is None else s0
    s1 = X(self.s1[i]) if s1 is None else s1
    gr = mul(X(self.g[i]), X(gs))
    gr = where(self.l2e != 0, add(gr, mul(X(self.l2e), w)), gr)
    lr = mul(lr0, X(self.lrme))
    return rule(self.kind, w, s0, s1, gr, lr)

  def reg_depth(self):
    return _reg_depth(self.sizes, self.max_n)

  def check(self, got, init, ref, what):
    ns = N_STATE[self.kind]
    names = ('p', 'g', 's0', 's1')
    for k, (b, b0) in enumerate(zip(got, init)):
      assert bool(torch.isnan(b[~self.live]).all()), '%s: %s written in a gap between segments' % (what, names[k])
      if k == 1 or (k == 2 and ns < 1) or (k == 3 and ns < 2):
        _same(b, b0, '%s %s (read only / not passed)' % (what, names[k]))
    _within(got[0][self.idx], ref[0], what + ' w')
    if ns >= 1:
      _within(got[2][self.idx], ref[1], what + ' s0')
    if ns >= 2:
      _within(got[3][self.idx], ref[2], what + ' s1')


def _reg_depth(sizes, max_n):
  """longest chain of additions behind reg_loss_out: the 3 roundings of a term, a thread's chunks, 5 shuffle levels,
  one atomic per warp of the grid"""
  grid = min(MAX_CTAS, -(-max_n // 256) + len(sizes))
  chunks = sum(-(-int(n) // 256) for n in sizes)
  return 4 + -(-chunks // grid) + 5 + 8 * grid


def _reg_ref(w, l2e, depth):
  """sum l2/2 w^2 over reference weights; the terms are non-negative, so any order is within depth u sum"""
  v = (0.5 * l2e * w.v * w.v).sum()
  e = (l2e * w.v.abs() * w.e + 0.5 * l2e * w.e * w.e).sum() + depth * U * v
  return R(v, e)


def _rng_sizes(n, seed):
  rng = np.random.default_rng(seed)
  s = rng.integers(0, 700, n)
  s[rng.random(n) < 0.1] = 0
  s[rng.random(n) < 0.05] = 1
  return [int(x) for x in s]


TABLES = {
    'one': [1],
    'chunk_edges': [255, 256, 257, 511, 512, 513],
    'empty_segments': [0, 300, 0, 0, 17, 256, 0],
    'max_segments': _rng_sizes(8192, 5),
    'one_million': [1_000_003],
}


@pytest.mark.parametrize('table', list(TABLES))
@pytest.mark.parametrize('kind', KINDS, ids=KIND_IDS)
def test_dense_apply_segment_tables(kind, table):
  """hyper_dev path (what FlatDenseOptimizer passes); the hyper block's grad_scale slot is deliberately wrong: the dense
  update takes grad_scale from the struct.  reg_loss_out against float64; the update without it bit-identical."""
  d = Dense(kind, TABLES[table], seed=len(TABLES[table]) * 10 + kind)
  hy = K.StepHyper(DEV, B1, B2)
  hy.set(0.03, 4, grad_scale=7.0)
  gs = 0.7
  opt = hy.opt(kind, EPS, grad_scale=gs)
  lr0 = lr_t_of(hy.lr, float(hy.b1p), float(hy.b2p)) if _adam(kind) else X(hy.lr)
  init = d.snap()
  ref = d.ref(lr0, gs)
  reg = torch.full((3,), float('nan'), device=DEV)
  reg[1] = 0.0
  d.run(opt, reg=reg[1:2])
  got = d.snap()
  d.check(got, init, ref, 'dense %s' % table)
  assert bool(torch.isnan(reg[0]) and torch.isnan(reg[2])), 'reg_loss_out wrote past its float'
  _within(reg[1:2], _reg_ref(X(init[0][d.idx]), d.l2e, d.reg_depth()), 'dense reg_loss')
  d.restore(init)
  d.run(opt)
  for a, b in zip(d.snap(), got):
    _same(a, b, 'dense %s: update without reg_loss_out' % table)


@pytest.mark.parametrize('kind', KINDS, ids=KIND_IDS)
def test_dense_apply_rate_sources(kind):
  """lr_dev wins over hyper_dev, which wins over the struct; the losing sources hold wrong values.  The struct path forms
  Adam's lr_t from the struct's beta powers exactly as the hyper_dev path forms it from the device block, so the three
  give bit-identical results."""
  d = Dense(kind, [300, 1, 513, 0, 70, 4096], seed=40 + kind)
  lr, b1p, b2p, gs = 0.02, float(_f32(B1 ** 3)), float(_f32(B2 ** 3)), 0.6
  init = d.snap()
  ref = d.ref(lr_t_of(lr, b1p, b2p) if _adam(kind) else X(lr), gs)
  # the struct alone
  d.run(K.make_opt(kind, lr, B1, B2, EPS, b1p, b2p, gs))
  got_s = d.snap()
  d.check(got_s, init, ref, 'dense struct rate')
  # hyper_dev: struct lr and powers wrong, the block's grad_scale wrong (grad_scale is the struct's)
  hdev = torch.tensor([lr, b1p, b2p, 7.0], dtype=torch.float32, device=DEV)
  d.restore(init)
  d.run(K.make_opt(kind, lr * 3, B1, B2, EPS, 0.5, 0.25, gs, hyper_dev=hdev))
  for a, b in zip(d.snap(), got_s):
    _same(a, b, 'dense hyper_dev rate vs struct rate')
  # lr_dev: the effective rate as is; hyper block and struct both wrong
  eff = lr_t_f32(lr, b1p, b2p) if _adam(kind) else lr
  lr_dev = torch.tensor([eff], dtype=torch.float32, device=DEV)
  bad = torch.tensor([lr * 5, 0.3, 0.2, 9.0], dtype=torch.float32, device=DEV)
  d.restore(init)
  d.run(K.make_opt(kind, lr * 3, B1, B2, EPS, 0.5, 0.25, gs, hyper_dev=bad), lr_dev=lr_dev)
  for a, b in zip(d.snap(), got_s):
    _same(a, b, 'dense lr_dev rate vs struct rate')


def test_dense_apply_ten_adam_steps():
  """StepHyper advances the fp32 beta powers; the float64 state is carried from step to step"""
  d = Dense(ADAM_ROWS, [513, 1, 256, 4000, 0, 77], seed=3)
  d.s0[d.idx] = 0.0
  d.s1[d.idx] = 0.0
  hy = K.StepHyper(DEV, B1, B2)
  gen = _gen(33)
  w, m, v = X(d.p[d.idx]), X(d.s0[d.idx]), X(d.s1[d.idx])
  for step in range(10):
    lr = 0.01 * (0.9 ** step)
    hy.set(lr, step)
    d.g[d.idx] = torch.randn(d.idx.numel(), generator=gen, device=DEV)
    init = d.snap()
    w, m, v = d.ref(lr_t_of(hy.lr, float(hy.b1p), float(hy.b2p)), 1.0, w, m, v)
    d.run(hy.opt(ADAM_ROWS, EPS, grad_scale=1.0))
    d.check(d.snap(), init, (w, m, v), 'dense adam step %d' % step)


def test_dense_apply_refusals():
  """refused before launch, with real buffers, and nothing written"""
  lib = _lib.load()
  d = Dense(ADAM_ROWS, [100, 5], seed=9)
  big = np.zeros(8193, dtype=_lib.DENSE_SEG_DTYPE)
  big['offset'], big['n'], big['lr_mult'] = 1, 1, 1.0
  big_dev = torch.from_numpy(big.view(np.uint8).reshape(-1).copy()).to(DEV)
  init = d.snap()
  opt = {k: K.make_opt(k, 0.1, B1, B2, EPS, 0.9, 0.999, 1.0) for k in KINDS}
  cases = [
      ('n_segs 0', d.s0, d.s1, d.segs_dev, 0, 100, ADAM_ROWS),
      ('n_segs 8193', d.s0, d.s1, big_dev, 8193, 100, ADAM_ROWS),
      ('max_seg_n 0', d.s0, d.s1, d.segs_dev, 2, 0, ADAM_ROWS),
      ('adagrad without state0', None, None, d.segs_dev, 2, 100, ADAGRAD),
      ('momentum without state0', None, None, d.segs_dev, 2, 100, MOMENTUM),
      ('adam without state1', d.s0, None, d.segs_dev, 2, 100, ADAM_ROWS),
      ('lazy adam without state1', d.s0, None, d.segs_dev, 2, 100, LAZY_ADAM),
  ]
  for what, s0, s1, segs, n, mx, kind in cases:
    rc = _dense_apply(d.p, d.g, s0, s1, segs, n, mx, opt[kind])
    assert rc == _lib.ER_ERR_INVALID_ARG, '%s: rc %d' % (what, rc)
    assert lib.er_last_error()
  torch.cuda.synchronize()
  for a, b in zip(d.snap(), init):
    _same(a, b, 'refused calls')


# ---- FlatDenseOptimizer -------------------------------------------------------------------------------------------
def _dnn_params(seed):
  gen = torch.Generator().manual_seed(seed)
  units = [624, 256, 128, 64]
  out = []
  for i in range(3):
    fi, fo = units[i], units[i + 1]
    pre = 'dnn/dense_%d/' % i
    out += [(pre + 'kernel', torch.randn(fi, fo, generator=gen) * (1.0 / fi ** 0.5)),
            (pre + 'bias', torch.randn(fo, generator=gen) * 0.1),
            (pre + 'batch_normalization/gamma', 1.0 + 0.1 * torch.randn(fo, generator=gen)),
            (pre + 'batch_normalization/beta', torch.randn(fo, generator=gen) * 0.1)]
  return out


@pytest.mark.parametrize('kind', ['adagrad', 'adam', 'sgd', 'momentum'])
def test_flat_dense_optimizer(kind):
  """three steps with a changing rate, l2 on the kernels only; apply() and fold_l2() + apply(l2_folded=True) both
  against the same carried float64 state, and their reg_loss against float64"""
  from easyrec_b200.trainer import FlatDenseOptimizer
  l2 = float(_f32(0.02))
  opts = []
  for _ in range(2):
    ps = [(n, torch.nn.Parameter(t.to(DEV))) for n, t in _dnn_params(1)]
    opts.append(FlatDenseOptimizer(ps, kind, lr=0.05, l2_of=lambda n, q: l2 if n.endswith('kernel') else 0.0))
  fa, fb = opts
  ek = fa.kind
  idx = torch.cat([torch.arange(o, o + n) for _, o, n in fa.named_ranges()]).to(DEV)
  pad = torch.ones(fa.flat_p.numel(), dtype=torch.bool, device=DEV)
  pad[idx] = False
  l2e = torch.from_numpy(fa._l2_vec_np).to(DEV).double()[idx]
  w = X(fa.flat_p[idx])
  s0 = X(fa.s0[idx]) if fa.s0 is not None else None
  s1 = X(fa.s1[idx]) if fa.s1 is not None else None
  assert fa.s0 is None or bool((fa.s0[idx] == (0.1 if ek == ADAGRAD else 0.0)).all())
  gen = _gen(71)
  n = idx.numel()
  for step, lr in enumerate([0.05, 0.02, 0.08]):
    g = torch.randn(n, generator=gen, device=DEV)
    for fo in opts:
      fo.hyper.set(lr, step)
      fo.flat_g[idx] = g
    reg_a = _reg_ref(w, l2e, _reg_depth(fa.sizes, fa.max_n))
    reg_b = _reg_ref(w, l2e, fb.flat_p.numel() + 4)       # fold_l2 sums with torch: any order of all the terms
    fa.apply()
    fb.fold_l2()
    fb.apply(l2_folded=True)
    gr = mul(X(g), X(1.0))
    gr = where(l2e != 0, add(gr, mul(X(l2e), w)), gr)
    lr0 = lr_t_of(lr, float(fa.hyper.b1p), float(fa.hyper.b2p)) if _adam(ek) else X(lr)
    w, s0, s1 = rule(ek, w, s0, s1, gr, lr0)
    for fo, reg, tag in ((fa, reg_a, 'apply'), (fb, reg_b, 'fold_l2')):
      what = 'flat %s %s step %d' % (kind, tag, step)
      _within(fo.flat_p[idx], w, what + ' w')
      if s0 is not None:
        _within(fo.s0[idx], s0, what + ' s0')
      if s1 is not None:
        _within(fo.s1[idx], s1, what + ' s1')
      assert bool((fo.flat_p[pad] == 0).all()), what + ': alignment padding written'
      _within(fo.reg_loss, reg, what + ' reg_loss')
    for p, (name, off, cnt) in zip(fa.params, fa.named_ranges()):
      assert p.data_ptr() == fa.flat_p[off:].data_ptr(), name


# ---- er_sparse_apply ----------------------------------------------------------------------------------------------
def _sparse_apply(mats, dim, rows, grads, n_uniq, n_cap, opt):
  w, s0, s1 = mats
  rc = _lib.load().er_sparse_apply(_p(w), _p(s0), _p(s1), dim, w.stride(0), _p(rows), _p(grads), _p(n_uniq), n_cap,
                                   ctypes.byref(opt), _stream())
  _lib.check(rc, 'er_sparse_apply')


@pytest.mark.parametrize('dim', [1, 4, 6, 16, 128])
@pytest.mark.parametrize('layout', ['separate', 'interleaved'])
@pytest.mark.parametrize('kind', KINDS, ids=KIND_IDS)
def test_sparse_apply(kind, layout, dim):
  """-1 rows are skipped; *n_uniq < n_cap applies only the first *n_uniq rows, *n_uniq > n_cap stops at n_cap (the
  gradients past n_cap are NaN: reading one would write NaN into a valid row); hyper_dev with a wrong struct gives the
  struct path's bits"""
  V, cap, extra = 300, 64, 16
  gen = _gen(1000 + 100 * kind + dim)
  mats, bufs = _storage(kind, V, dim, layout, gen)
  init = _snap(mats)
  rows = torch.randperm(V, generator=gen, device=DEV)[:cap + extra].to(torch.int64)
  rows[torch.tensor([0, 7, 30, 41, 63], device=DEV)] = -1
  gbuf, gview = _out(cap + extra, dim)
  gview[:cap] = torch.randn(cap, dim, generator=gen, device=DEV)
  lr, b1p, b2p, gs = 0.05, float(_f32(B1 ** 3)), float(_f32(B2 ** 3)), 0.75
  right = K.make_opt(kind, lr, B1, B2, EPS, b1p, b2p, gs)
  hdev = torch.tensor([lr, b1p, b2p, gs], dtype=torch.float32, device=DEV)
  wrong = K.make_opt(kind, lr * 3, B1, B2, EPS, 0.5, 0.25, 9.0, hyper_dev=hdev)
  lr0 = lr_t_of(lr, b1p, b2p) if _adam(kind) else X(lr)
  for nu in (40, cap + 10, None):
    n_eff = cap if nu is None else min(nu, cap)
    nu_dev = None if nu is None else torch.tensor([nu], dtype=torch.int32, device=DEV)
    got = []
    for opt in (right, wrong):
      _restore(mats, init)
      _sparse_apply(mats, dim, rows, gview, nu_dev, cap, opt)
      got.append(_snap(mats))
    for a, b in zip(*got):
      if a is not None:
        _same(a, b, 'sparse_apply hyper_dev vs struct')
    live = rows[:n_eff] >= 0
    r = rows[:n_eff][live]
    g = mul(X(gview[:n_eff][live]), X(gs))
    ref = rule(kind, X(init[0][r]), X(init[1][r]) if init[1] is not None else None,
               X(init[2][r]) if init[2] is not None else None, g, lr0)
    _check_rows(kind, got[0], init, r, ref, 'sparse_apply %s n_uniq=%s' % (layout, nu))
    for b in bufs:
      _guards_nan(b, 'sparse_apply')


# ---- er_adam_dense_sweep and er_mark_rows -------------------------------------------------------------------------
@pytest.mark.parametrize('dim,layout', [(16, 'separate'), (16, 'interleaved'), (6, 'interleaved')],
                         ids=['vector_separate', 'vector_stride48', 'scalar_stride18'])
def test_adam_dense_sweep(dim, layout):
  """m *= b1, v *= b2, w -= lr_t m / (sqrt(v) + eps) on every row not marked touched.  Rows by class (row % 4): m = v = 0
  (left unwritten: bit-identical), m = 0 with v != 0 (v still decays), general, and every other column zero."""
  V = 1000
  gen = _gen(dim * 7 + len(layout))
  mats, bufs = _storage(ADAM_ROWS, V, dim, layout, gen)
  w, m, v = mats
  if layout == 'interleaved':
    assert w.stride(0) == 3 * dim
  cls = torch.arange(V, device=DEV) % 4
  m[cls == 0] = 0.0
  v[cls == 0] = 0.0
  m[cls == 1] = 0.0
  half = (cls == 3).nonzero().flatten()
  m[half[:, None], torch.arange(0, dim, 2, device=DEV)[None, :]] = 0.0
  v[half[:, None], torch.arange(0, dim, 2, device=DEV)[None, :]] = 0.0
  init = _snap(mats)
  lr, b1p, b2p = 0.01, float(_f32(B1 ** 7)), float(_f32(B2 ** 7))
  lr_t = lr_t_of(lr, b1p, b2p)
  tmask = (torch.rand(V, generator=gen, device=DEV) < 0.3).to(torch.uint8)
  hdev = torch.tensor([lr, b1p, b2p, 1.0], dtype=torch.float32, device=DEV)
  for touched in (None, tmask):
    got = []
    for opt in (K.make_opt(ADAM_ROWS, lr, B1, B2, EPS, b1p, b2p),
                K.make_opt(ADAM_ROWS, lr * 3, B1, B2, EPS, 0.5, 0.25, hyper_dev=hdev)):
      _restore(mats, init)
      _lib.check(_lib.load().er_adam_dense_sweep(_p(w), _p(m), _p(v), V, dim, w.stride(0), _p(touched),
                                                 ctypes.byref(opt), _stream()), 'er_adam_dense_sweep')
      got.append(_snap(mats))
    for a, b in zip(*got):
      _same(a, b, 'sweep hyper_dev vs struct')
    swept = torch.ones(V, dtype=torch.bool, device=DEV) if touched is None else touched == 0
    r = swept.nonzero().flatten()
    mm = mul(X(init[1][r]), X(B1))
    vv = mul(X(init[2][r]), X(B2))
    ww = sub(X(init[0][r]), div(mul(lr_t, mm), add(sqrt(vv), X(EPS))))
    what = 'sweep %s touched=%s' % (layout, touched is not None)
    _check_rows(ADAM_ROWS, got[0], init, r, (ww, mm, vv), what)
    z = (cls == 0) & swept
    for a, b in zip(got[0], init):
      _same(a[z], b[z], what + ': all-zero rows')
    dec = (cls == 1) & swept
    assert bool((got[0][2][dec] != init[2][dec]).all()), what + ': v of rows with m = 0 did not decay'
    for b in bufs:
      _guards_nan(b, 'sweep')


def test_mark_rows():
  n_rows, cap = 100, 64
  gen = _gen(5)
  rows = torch.randint(0, n_rows, (cap,), generator=gen, device=DEV)
  rows[torch.tensor([3, 10, 20, 50], device=DEV)] = torch.tensor([-1, 100, 150, -7], device=DEV)
  buf = torch.full((n_rows + 2 * G,), 0xAB, dtype=torch.uint8, device=DEV)
  touched = buf[G:G + n_rows]

  def want(prefill, n, value):
    t = prefill.clone()
    live = rows[:n]
    live = live[(live >= 0) & (live < n_rows)]
    t[live] = value
    return t

  for n_dev in (None, 0, 17, cap, cap + 100):
    n = cap if n_dev is None else min(n_dev, cap)
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device=DEV)
    for value, prefill in ((1, 0), (0, 1)):
      touched.fill_(prefill)
      p0 = touched.clone()
      K.mark_rows(rows, n_rows, touched, value, n_dev=nd)
      assert torch.equal(touched, want(p0, n, value)), (n_dev, value)
      assert bool((buf[:G] == 0xAB).all() and (buf[-G:] == 0xAB).all()), 'mark_rows wrote outside touched'


# ---- er_embedding_bwd: the K7 row rule ----------------------------------------------------------------------------
class K7(object):
  """two CSR slots (mean and sqrtn combiners, lookup weights in [0.25, 2]) over B samples; every live row is looked up
  once except the `hot` rows, looked up hot[i] times each; about 6% of the single lookups are dropped (-1)"""

  def __init__(self, dim, seed, B, V, hot=()):
    rng = np.random.default_rng(seed)
    self.dim, self.B, self.V, self.F = dim, B, V, 2
    F = self.F
    lens = rng.integers(0, 4, B * F).astype(np.int32)
    L = int(lens.sum())
    n_hot = sum(hot)
    assert L > n_hot + 10
    perm = rng.permutation(V)
    singles = perm[len(hot):len(hot) + L - n_hot].astype(np.int64)
    hot_rows = perm[:len(hot)].astype(np.int64)
    rows = np.concatenate([singles] + [np.full(c, r, np.int64) for r, c in zip(hot_rows, hot)])
    drop = rng.random(L - n_hot) < 0.06
    rows[:L - n_hot][drop] = -1
    rows = rows[rng.permutation(L)]
    self.hot_rows = hot_rows
    w = rng.uniform(0.25, 2.0, L).astype(np.float32)
    seg_of = np.repeat(np.arange(B * F), lens)
    scale = np.zeros(B * F, np.float32)
    for s in range(B * F):
      ws = w[seg_of == s].astype(np.float64)
      if ws.size:
        scale[s] = 1.0 / ws.sum() if s < B else 1.0 / np.sqrt((ws * ws).sum())
    stride = -(-F * dim // 4) * 4
    gout = rng.normal(size=(B, stride)).astype(np.float32)
    recs = [dict(num_buckets=V, row_offset=0, seg_begin=f * B, n_seg=B, bucket_mode=_lib.BUCKET_NONE,
                 combiner=[_lib.COMBINER_MEAN, _lib.COMBINER_SQRTN][f], out_buf=0, out_stride=stride,
                 out_col=f * dim) for f in range(F)]
    self.sd = K.slots_to_device(K.make_slots(recs), DEV)
    self.rows = torch.from_numpy(rows).to(DEV)
    self.w = torch.from_numpy(w).to(DEV)
    self.scale = torch.from_numpy(scale).to(DEV)
    self.gout = torch.from_numpy(gout).to(DEV)
    self.row_ptr, self.seg_ids = K.csr_from_lens(torch.from_numpy(lens).to(DEV), L)
    self.L = L
    # G per row: sum over its lookups of gout[segment] * (w * seg_scale), in any order
    seg = torch.from_numpy(seg_of).to(DEV)
    f, b = seg // B, seg % B
    cols = f[:, None] * dim + torch.arange(dim, device=DEV)[None, :]
    gv = self.gout[b[:, None], cols]
    coef = mul(X(self.w), X(self.scale[seg]))
    term = mul(X(gv), R(coef.v[:, None], coef.e[:, None]))
    live = self.rows >= 0
    r = self.rows[live]
    z = torch.zeros(V, dim, dtype=torch.float64, device=DEV)
    sv = z.index_add(0, r, term.v[live])
    se = z.index_add(0, r, term.e[live])
    sa = z.index_add(0, r, term.v[live].abs())
    cnt = torch.zeros(V, dtype=torch.float64, device=DEV).index_add(0, r, torch.ones_like(r, dtype=torch.float64))
    self.uniq = torch.unique(r)
    self.Gsum = R(sv, se + (cnt - 1).clamp_min(0)[:, None] * U * sa)

  def call(self, mats, opt, ws, **kw):
    K.embedding_bwd(mats[0], mats[1], mats[2], self.dim, self.rows, self.sd, self.F, self.B * self.F, [self.gout],
                    opt, ws, weights=self.w, seg_ids=self.seg_ids, row_ptr=self.row_ptr, seg_scale=self.scale, **kw)


def _k7_rule_case(kind, layout, dim, B, V, hot, seed):
  case = K7(dim, seed, B, V, hot)
  gen = _gen(seed)
  mats, bufs = _storage(kind, V, dim, layout, gen)
  init = _snap(mats)
  lr, b1p, b2p, gs = 0.05, float(_f32(B1 ** 4)), float(_f32(B2 ** 4)), 0.75
  case.call(mats, K.make_opt(kind, lr, B1, B2, EPS, b1p, b2p, gs), K.bwd_workspace(case.L, DEV, dim))
  got = _snap(mats)
  r = case.uniq
  g = mul(case.Gsum[r], X(gs))
  lr0 = lr_t_of(lr, b1p, b2p) if _adam(kind) else X(lr)
  ref = rule(kind, X(init[0][r]), X(init[1][r]) if init[1] is not None else None,
             X(init[2][r]) if init[2] is not None else None, g, lr0)
  _check_rows(kind, got, init, r, ref, 'K7 %s dim %d%s' % (layout, dim, ' hot' if hot else ''))
  for b in bufs:
    _guards_nan(b, 'K7')


@pytest.mark.parametrize('dim', [1, 4, 8, 16, 32, 64, 128, 6, 12])
@pytest.mark.parametrize('layout', ['separate', 'interleaved'])
@pytest.mark.parametrize('kind', KINDS, ids=KIND_IDS)
def test_k7_row_rule(kind, layout, dim):
  """each live row looked up once: G = coef g with no sum, so the comparison tests the update rule alone"""
  _k7_rule_case(kind, layout, dim, B=96, V=700, hot=(), seed=500 + 10 * kind + dim)


@pytest.mark.parametrize('dim', [16, 6])
@pytest.mark.parametrize('kind', KINDS, ids=KIND_IDS)
def test_k7_hot_rows_interleaved(kind, dim):
  """runs of 65 and 600 lookups of one row reach bwd_long_* (apply_row_vec at dim 16, apply_scalar at dim 6) on a
  row_stride > dim table; the bound adds the rule's sensitivity to G times the sum-chain bound on G"""
  _k7_rule_case(kind, 'interleaved', dim, B=500, V=2000, hot=(65, 600), seed=900 + 10 * kind + dim)


@pytest.mark.parametrize('dim', [1, 4, 6, 16, 128])
def test_k7_emit_uniq_grads(dim):
  """table NULL: uniq_rows = the distinct live rows ascending, *n_uniq their count, uniq_grads = grad_scale G; nothing
  past n_uniq is written"""
  case = K7(dim, 70 + dim, B=300, V=1500, hot=(65, 3, 2))
  L = case.L
  ur = torch.full((L,), -7, dtype=torch.int64, device=DEV)
  gbuf, ug = _out(L, dim)
  nu = torch.full((1,), -1, dtype=torch.int32, device=DEV)
  gs = 0.375
  case.call([None, None, None], K.make_opt(SGD, 0.1, grad_scale=gs), K.bwd_workspace(L, DEV, dim),
            uniq_rows=ur, uniq_grads=ug, n_uniq=nu, n_rows=case.V)
  n = int(nu.item())
  assert n == case.uniq.numel()
  assert torch.equal(ur[:n], case.uniq)
  assert bool((ur[n:] == -7).all()), 'uniq_rows written past n_uniq'
  assert bool(torch.isnan(ug[n:]).all()), 'uniq_grads written past n_uniq'
  _guards_nan(gbuf, 'uniq_grads')
  _within(ug[:n], mul(case.Gsum[case.uniq], X(gs)), 'K7 emit uniq_grads')
