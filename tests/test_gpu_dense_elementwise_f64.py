"""GPU: the dense towers' elementwise kernels and the vector-sized GEMM against float64 and exact restatements, through
the C ABI where an option or a NULL is only reachable there.

  er_act_fwd / er_act_bwd   all seven kinds on +-0, denormals, FLT_MIN, every power of two 2^-149 .. 2^127 and its
                            neighbours, the expf overflow / underflow points, where 1 - s rounds to 0, where gelu's x^3
                            and x * x overflow, 10^6 draws of N(0, 3); +-inf and NaN against the reference's own fp32
                            expressions; the branch at x = 0 bit for bit; lengths around one grid-stride pass.
  er_dice_fwd / er_dice_bwd units x batch against the i % units broadcast, alpha 0 / 1 / negative, xn over +-90.
  layers.Dice               training forward, dx and d alpha against float64 autograd of utils/activation.py:dice at
                            C3's attention-MLP shapes, a constant column, a variance near eps, a column 1e3 sigma off
                            zero; moving statistics after three steps, then eval.
  er_dropout / Dropout      bit for bit against a numpy restatement of drop_bits; draws placed exactly on the
                            threshold by inverting the splitmix64 finaliser; the layer's counter in eager steps and
                            CUDA-graph replays; a DNN with an activation and dropout on every layer against float64.
  er_gemm_small             every N, M and K in 1..7, the four operand layouts, the slice rule's edges, pitched and
                            misaligned C, bias NULL and not in both kernels, the MMoE gate shapes, refusals.

Bounds are first-order fp32 rounding, u = 2^-24, slack C = 2, following each kernel's order of operations:
  a rounding      u |v| for a result v, 2^-150 where |v| < FLT_MIN (the spacing of the denormals);
  expf / tanhf /  2 ulp: 4u |v|, 2^-148 where |v| < FLT_MIN; an argument error d propagates as slope * d;
  expm1f
  sigmoid         e = expf(-x), d = 1 + e, s = 1 / d: ds = s (2ulp(e) + rnd(d)) / d + rnd(s).  Where expf(-x) may
                  overflow (x < -88.72) the kernel's s is 0, and the bound there is the true value itself (sigmoid and
                  swish values and slopes are below 2.6e-37 there).
  1 - s, 1 - t^2  the error of s (or 2 |t| that of t) plus the rounding: the cancellation where s or t rounds to 1.
  gelu            the argument c (x + k x^3) carries 3 roundings on k x^3, one on the sum and one on c * r, plus the
                  fp32 rounding of the constants c and k; 1 + tanh carries tanhf's 2 ulp near -1 (the left tail).
  dice            each product and difference of y = alpha (1 - p) x + p x and of its three gradient terms rounds once;
                  the layer adds |dy / dxn| times the xn bound of test_gpu_dense_bn (normalisation with eps 1e-9), and
                  dx composes that file's er_bias_bn_act_bwd bound with the error of gxn and of the statistics.
  gemm_small      gamma_k sum |a||b| for an FMA chain of k = k_per_slice, plus n_slice u sum |a||b| for the slices
                  summed in order and u |bias| for the bias add.
Exact: er_dropout (bit for bit, both directions), leaky_relu's forward for x > 0, the branch at 0, non-finite inputs,
gxn where alpha = 1, y of a constant dice column (xn = 0 exactly), gemm_small outputs of a slice that starts past K.
The DNN with dropout is checked with test_gpu_dense.py's rule: no worse than torch fp32 of the same restatement.

Worst error / bound measured on an H100 80GB HBM3 (700 W power limit), 82 tests:
  activations   y / gx: gelu 0.50 / 0.47, leaky_relu 0.48 / 0.48, elu 0.22 / 0.30, selu 0.50 / 0.50, tanh 0.40 / 0.36,
                swish 0.50 / 0.50, sigmoid 0.50 / 0.50 (0.5 = one rounding more than the kernel made, against C = 2);
  er_dice_*     y 0.50, gx_direct 0.50, gxn 0.50, galpha 0.41;
  layers.Dice   y 0.24, dx 0.15, d alpha 0.017, eval y 0.31, moving mean 0.015, moving var 0.075;
  gemm_small    0.31 (shape sweeps), MMoE gate forward 0.025, dX 0.34, dW below 0.001.
"""
import math

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, kernels as K, layers as L
from easyrec_b200.kernels import _p, _stream
from test_gpu_dense_bn import _mean_bound, _sum_bound, _var_bound, _y_bound
from test_gpu_interact_f64 import DEV, U, _gen, _ok, _out, _untouched

pytestmark = pytest.mark.gpu
C = 2.0
FLT_MIN = float(np.finfo(np.float32).tiny)
FLT_MAX = float(np.finfo(np.float32).max)
OVF = FLT_MAX * (1 + U)               # a float64 value at or past this rounds to inf in fp32
WORST = {}
KINDS = ['gelu', 'leaky_relu', 'elu', 'selu', 'tanh', 'swish', 'sigmoid']
GELU_C, GELU_K = math.sqrt(2 / math.pi), 0.044715
SELU_S = 1.0507009873554804934193349852946
SELU_SA = SELU_S * 1.6732632423543772848170429916717


def _cerr(c):
  """relative error of the fp32 rounding of the constant c"""
  return abs(float(np.float32(c)) - c) / abs(c)


E_C, E_K = _cerr(GELU_C), _cerr(GELU_K)
E_K3 = abs(float(np.float32(3.0) * np.float32(GELU_K)) - 3 * GELU_K) / (3 * GELU_K)
E_S, E_SA, E_02 = _cerr(SELU_S), _cerr(SELU_SA), _cerr(0.2)


def _within(got, ref, bound, what):
  """|got - ref| <= bound elementwise: numpy arrays, or tensors (compared on got's device); NaN anywhere fails"""
  if isinstance(got, torch.Tensor):
    ref, bound = (torch.as_tensor(v, dtype=torch.float64, device=got.device) for v in (ref, bound))
    err = (got.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = float(r.max()) if r.numel() else 0.0
  else:
    err = np.abs(np.asarray(got, np.float64) - ref)
    with np.errstate(invalid='ignore', divide='ignore'):
      r = np.where(err == 0, 0.0, err / bound)
    ratio = float(np.max(r)) if r.size else 0.0
  WORST[what] = max(WORST.get(what, 0.0), ratio)
  assert ratio <= 1.0, '%s: error %.3g x bound' % (what, ratio)


def _fn(name, v):
  """np.<name> or torch.<name>, whichever v is"""
  return getattr(torch if isinstance(v, torch.Tensor) else np, name)(v)


def _where(c, a, b):
  if isinstance(c, torch.Tensor):
    return torch.where(c, a, b)
  return np.where(c, a, b)


def _tiny(a):
  """1.0 where |v| = a is below FLT_MIN, else 0.0 (float64)"""
  m = a < FLT_MIN
  return m.double() if isinstance(m, torch.Tensor) else m.astype(np.float64)


def _rnd(v):
  a = abs(v)
  return U * a + _tiny(a) * 2.0 ** -150


def _ulp2(v):
  a = abs(v)
  return 4 * U * a + _tiny(a) * 2.0 ** -148


def _sig(v):
  """float64 s = sigmoid(v), q = 1 - s without cancellation, the error of the kernel's 1 / (1 + expf(-v)) and the mask
  of arguments where that expf may overflow (the kernel's s is 0 there); numpy or torch"""
  with np.errstate(over='ignore'):
    e = _fn('exp', -v)
    s, q = 1.0 / (1.0 + e), 1.0 / (1.0 + _fn('exp', v))
  ovf = e >= FLT_MAX * (1 - 4 * U)
  ds = _where(ovf, s, s * (_ulp2(e) + _rnd(1.0 + e)) / (1.0 + e) + _rnd(s))
  return s, q, ds, ovf


# ---------------------------------------------------------------------------------------------------------------------
# activations
# ---------------------------------------------------------------------------------------------------------------------

def _around(points, k=4):
  """the fp32 values within k ulps of each point, both signs"""
  b = np.abs(np.asarray(points, np.float32)).view(np.int32).astype(np.int64)
  near = (b[:, None] + np.arange(-k, k + 1)[None, :]).ravel()
  near = near[(near >= 0) & (near < 0x7f800000)].astype(np.int32).view(np.float32)
  return np.concatenate([near, -near])


def _act_inputs():
  pts = [0.0, 2.0 ** -149, FLT_MIN, FLT_MAX]
  pts += [2.0 ** e for e in range(-149, 128)]
  pts += [math.log(FLT_MAX), -math.log(2.0 ** -150), -math.log(FLT_MIN),       # expf overflow / underflow / FLT_MIN
          24 * math.log(2), 25 * math.log(2), 9.01,                              # 1 - s and 1 - t^2 round to 0
          FLT_MAX ** (1 / 3), FLT_MAX ** 0.5, (FLT_MAX / 0.134145) ** 0.5]       # gelu: x^3, x x, 0.134 x x overflow
  rng = np.random.default_rng(11)
  return np.concatenate([_around(pts), rng.normal(0, 3, 10 ** 6).astype(np.float32)])


def _act_ref(name, x):
  """float64 value, slope and the kernel's error bounds for both (before the slack C), from fp32 inputs x"""
  with np.errstate(over='ignore', invalid='ignore'):
    if name == 'gelu':
      r = x + GELU_K * x ** 3
      uu = GELU_C * r
      cdf2 = 2.0 / (1.0 + np.exp(-2 * uu))                       # 1 + tanh(uu), no cancellation
      t = np.tanh(uu)
      ea = np.exp(-2 * np.abs(uu))
      sech2 = 4 * ea / (1 + ea) ** 2
      du = GELU_C * (np.abs(GELU_K * x ** 3) * (3 * U + E_K) + U * np.abs(r)) + np.abs(uu) * (U + E_C)
      dt = sech2 * du + _ulp2(t)
      dh = dt + _rnd(cdf2)
      y = 0.5 * x * cdf2
      dy = 0.5 * np.abs(x) * dh + _rnd(y)
      dd = 1 + 3 * GELU_K * x * x
      b = 0.5 * x * sech2 * GELU_C * dd
      s = 0.5 * cdf2 + b
      dsech = 2 * np.abs(t) * dt + _rnd(t * t) + _rnd(sech2)
      ddd = np.abs(3 * GELU_K * x * x) * (2 * U + E_K3) + _rnd(dd)
      ds = (0.5 * dh + 0.5 * np.abs(x) * GELU_C * (np.abs(dd) * dsech + sech2 * ddd) + np.abs(b) * (3 * U + E_C) +
            _rnd(s))
      return y, dy, s, ds
    if name == 'leaky_relu':
      neg = x < 0
      y = np.where(neg, 0.2 * x, x)
      dy = np.where(neg, np.abs(y) * E_02 + _rnd(y), 0.0)
      s = np.where(x > 0, 1.0, 0.2)
      return y, dy, s, np.where(x > 0, 0.0, 0.2 * E_02)
    if name in ('elu', 'selu'):
      neg = x < 0
      a, sa, ea, es = (1.0, 1.0, 0.0, 0.0) if name == 'elu' else (SELU_S, SELU_SA, E_SA, E_S)
      m1, ex = np.expm1(x), np.exp(x)
      y = np.where(neg, sa * m1, a * x)
      dy = np.where(neg, sa * _ulp2(m1) + np.abs(y) * ea, np.abs(y) * es) + (_rnd(y) if name == 'selu' else 0.0)
      s = np.where(neg, sa * ex, a)
      ds = np.where(neg, sa * _ulp2(ex) + np.abs(s) * ea + (_rnd(s) if name == 'selu' else 0.0), np.abs(s) * es)
      return y, dy, s, ds
    if name == 'tanh':
      t = np.tanh(x)
      ea = np.exp(-2 * np.abs(x))
      sech2 = 4 * ea / (1 + ea) ** 2
      return t, _ulp2(t), sech2, 2 * np.abs(t) * _ulp2(t) + _rnd(t * t) + _rnd(sech2)
    s, q, dsg, ovf = _sig(x)
    dq = dsg + _rnd(q)
    if name == 'sigmoid':
      sl = s * q
      return s, dsg, sl, np.where(ovf, sl, q * dsg + s * dq + _rnd(sl))
    # swish: y = x / (1 + e) rounds like s; slope s (1 + x (1 - s))
    y = x * s
    dy = np.where(ovf, np.abs(y), np.abs(x) * (dsg - _rnd(s)) + _rnd(y))
    w = 1 + x * q
    dw = np.abs(x) * dq + _rnd(x * q) + _rnd(w)
    sl = s * w
    return y, dy, sl, np.where(ovf, np.abs(sl), np.abs(w) * dsg + s * dw + _rnd(sl))


def _act_call(lib, x, gy, kind):
  """er_act_fwd / er_act_bwd into NaN-filled buffers; returns (y, gx) after checking nothing else was written"""
  n = x.numel()
  by, y = _out(n)
  bg, gx = _out(n)
  _ok(lib.er_act_fwd(_p(x), n, kind, _p(y), _stream()), 'er_act_fwd')
  _ok(lib.er_act_bwd(_p(x), _p(gy), n, kind, _p(gx), _stream()), 'er_act_bwd')
  _untouched(by, y, 'er_act_fwd')
  _untouched(bg, gx, 'er_act_bwd')
  return y, gx


@pytest.mark.parametrize('name', KINDS)
def test_activations_match_float64(name):
  lib, kind = _lib.load(), K.ACT_KINDS[name]
  x32 = _act_inputs()
  gy32 = np.random.default_rng(12).normal(size=x32.size).astype(np.float32)
  y, gx = _act_call(lib, torch.from_numpy(x32).to(DEV), torch.from_numpy(gy32).to(DEV), kind)
  y, gx = y.double().cpu().numpy(), gx.double().cpu().numpy()
  x, gy = x32.astype(np.float64), gy32.astype(np.float64)
  yr, dy, sr, ds = _act_ref(name, x)
  gr = gy * sr
  dg = np.abs(gy) * ds + _rnd(gr)
  for got, ref, bound, what in ((y, yr, dy, 'y'), (gx, gr, dg, 'gx')):
    big = np.abs(ref) >= OVF                      # fp32 of the true value is inf: the kernel must give that inf
    assert np.array_equal(got[big], np.sign(ref[big]) * np.inf), '%s %s: overflow' % (name, what)
    _within(got[~big], ref[~big], C * bound[~big], '%s %s' % (name, what))
  if name == 'leaky_relu':
    assert np.array_equal(y[x > 0], x[x > 0]), 'leaky_relu must pass positive x through exactly'


def _np32_act(name, x):
  """the reference's own fp32 expressions (utils/activation.py; tf.nn.* kernels) and TF's gradients for gy = 1"""
  f = np.float32
  with np.errstate(all='ignore'):
    sig = f(1) / (f(1) + np.exp(-x))
    if name == 'gelu':
      t = np.tanh(f(GELU_C) * (x + f(GELU_K) * x ** 3))
      cdf = f(0.5) * (f(1) + t)
      return x * cdf, cdf + x * (f(0.5) * (f(1) - t * t) * f(GELU_C) * (f(1) + f(3) * f(GELU_K) * x * x))
    if name == 'leaky_relu':
      return np.where(x > 0, x, x * f(0.2)), np.where(x > 0, f(1), f(0.2))
    if name == 'elu':
      y = np.where(x < 0, np.expm1(x), x)
      return y, np.where(y < 0, y + f(1), f(1))
    if name == 'selu':
      y = np.where(x < 0, f(SELU_SA) * np.expm1(x), f(SELU_S) * x)
      return y, np.where(y < 0, y + f(SELU_SA), f(SELU_S))
    if name == 'tanh':
      y = np.tanh(x)
      return y, f(1) - y * y
    if name == 'swish':
      return x * sig, sig * (f(1) + x * (f(1) - sig))
    return sig, sig * (f(1) - sig)


@pytest.mark.parametrize('name', KINDS)
def test_activations_non_finite_inputs_and_the_branch_at_zero(name):
  """+-inf and NaN give what the reference's fp32 expression gives (NaN included); at +-0 value and slope are pinned
  bit for bit: EluGrad / SeluGrad take the negative branch for x < 0, LeakyReluGrad for x <= 0 (slope 0.2 at 0)."""
  lib, kind = _lib.load(), K.ACT_KINDS[name]
  x = np.array([np.inf, -np.inf, np.nan, 0.0, -0.0], np.float32)
  y, gx = _act_call(lib, torch.from_numpy(x).to(DEV), torch.ones(x.size, device=DEV), kind)
  y, gx = y.cpu().numpy(), gx.cpu().numpy()
  yr, gr = _np32_act(name, x)
  np.testing.assert_array_equal(y[:3], yr[:3].astype(np.float32))
  np.testing.assert_array_equal(gx[:3], gr[:3].astype(np.float32))
  assert np.array_equal(y[3:].view(np.int32), yr[3:].astype(np.float32).view(np.int32)), (name, y[3:], yr[3:])
  slope0 = {'gelu': 0.5, 'leaky_relu': np.float32(0.2), 'elu': 1.0, 'selu': np.float32(SELU_S), 'tanh': 1.0,
            'swish': 0.5, 'sigmoid': 0.25}[name]
  assert np.array_equal(gx[3:], np.full(2, slope0, np.float32)), (name, gx[3:])


@pytest.mark.parametrize('name', ['gelu', 'sigmoid', 'selu'])
def test_activation_lengths_around_one_grid_stride_pass(name):
  """grid_for(n, 1024, 8) = 1056 CTAs x 256 threads = 270,336 elements per pass: every length gives, element by
  element, the bits the kernel gives on one short call (the pattern repeated)."""
  lib, kind = _lib.load(), K.ACT_KINDS[name]
  g = _gen(13)
  pat = torch.randn(4099, device=DEV, generator=g) * 3
  gpat = torch.randn(4099, device=DEV, generator=g)
  ypat, gxpat = _act_call(lib, pat, gpat, kind)
  for n in (1, 255, 270335, 270336, 270337, 10 ** 7 + 3):
    reps = -(-n // 4099)
    y, gx = _act_call(lib, pat.repeat(reps)[:n].contiguous(), gpat.repeat(reps)[:n].contiguous(), kind)
    assert torch.equal(y, ypat.repeat(reps)[:n]) and torch.equal(gx, gxpat.repeat(reps)[:n]), n


# ---------------------------------------------------------------------------------------------------------------------
# dice
# ---------------------------------------------------------------------------------------------------------------------

def _dice_ref(x, xn, a, gy):
  """float64 y, gx_direct, gxn, galpha terms of the kernel's formulas and their first-order bounds (before C)"""
  p, q, dp, _ = _sig(xn)
  dq = dp + _rnd(q)
  A = a * q
  dA = abs(a) * dq + _rnd(A)
  y = A * x + p * x
  dy = abs(x) * dA + _rnd(A * x) + abs(x) * dp + _rnd(p * x) + _rnd(y)
  S = A + p
  gd = gy * S
  dgd = abs(gy) * (dA + dp + _rnd(S)) + _rnd(gd)
  v1 = gy * x
  v2 = v1 * (1 - a)
  dv2 = abs(1 - a) * _rnd(v1) + abs(v1) * _rnd(1 - a) + _rnd(v2)
  v3 = v2 * p
  dv3 = p * dv2 + abs(v2) * dp + _rnd(v3)
  gn = v3 * q
  dgn = q * dv3 + abs(v3) * dq + _rnd(gn)
  ga = v1 * q
  dga = q * _rnd(v1) + abs(v1) * dq + _rnd(ga)
  return (y, dy), (gd, dgd), (gn, dgn), (ga, dga), (p, q)


@pytest.mark.parametrize('units', [1, 3, 32, 33, 128])
@pytest.mark.parametrize('batch', [1, 7, 204800])
def test_dice_kernels_match_float64(batch, units):
  """alpha[c] cycles 0, 1 (gxn exactly 0), negative, random, so a broadcast other than i % units is caught; every other
  row has xn uniform over +-90 (past expf's overflow on the left)."""
  lib = _lib.load()
  g = _gen(batch * 131 + units)
  x = torch.randn(batch, units, device=DEV, generator=g) * 2
  xn = torch.randn(batch, units, device=DEV, generator=g) * 3
  xn[1::2] = torch.rand(xn[1::2].shape, device=DEV, generator=g) * 180 - 90
  alpha = torch.randn(units, device=DEV, generator=g)
  alpha[0::4], alpha[1::4], alpha[2::4] = 0.0, 1.0, -alpha[2::4].abs() - 0.5
  gy = torch.randn(batch, units, device=DEV, generator=g)
  bufs = [_out(batch, units) for _ in range(4)]
  y, gd, gn, ga = (v for _, v in bufs)
  _ok(lib.er_dice_fwd(_p(x), _p(xn), _p(alpha), batch, units, _p(y), _stream()), 'er_dice_fwd')
  _ok(lib.er_dice_bwd(_p(x), _p(xn), _p(alpha), _p(gy), batch, units, _p(gd), _p(gn), _p(ga), _stream()), 'er_dice_bwd')
  for (b, v), what in zip(bufs, ('dice y', 'dice gx_direct', 'dice gxn', 'dice galpha')):
    _untouched(b, v, what)
  assert bool((gn[:, 1::4] == 0).all()), 'gxn must be exactly 0 where alpha = 1'
  a64 = alpha.double()
  step = max(1, (1 << 22) // units)
  for r0 in range(0, batch, step):
    s = slice(r0, r0 + step)
    refs = _dice_ref(x[s].double(), xn[s].double(), a64, gy[s].double())
    for got, (ref, bound), what in zip((y, gd, gn, ga), refs[:4], ('dice y', 'dice gx_direct', 'dice gxn',
                                                                   'dice galpha')):
      _within(got[s], ref, C * bound, what)


def test_dice_wrappers_refuse_mismatched_shapes():
  """kernels.dice_fwd / dice_bwd check x, xn, gy [B, U] and alpha [U] before any launch."""
  x = torch.zeros(8, 4, device=DEV)
  a = torch.zeros(4, device=DEV)
  for bad in ((x, torch.zeros(8, 3, device=DEV), a), (x, torch.zeros(4, 8, device=DEV), a),
              (x, x, torch.zeros(5, device=DEV)), (x, x, torch.zeros(1, 4, device=DEV)), (x.view(-1), x.view(-1), a)):
    with pytest.raises(_lib.ErError):
      K.dice_fwd(*bad)
    with pytest.raises(_lib.ErError):
      K.dice_bwd(*bad, torch.zeros_like(bad[0]))
  with pytest.raises(_lib.ErError):
    K.dice_bwd(x, x, a, torch.zeros(8, 5, device=DEV))


DICE_EPS = float(np.float32(L.DICE_EPS))
MOM = float(np.float32(L.BN_MOMENTUM))


def _dice_layer_inputs(B, U_, g):
  x = torch.randn(B, U_, device=DEV, generator=g)
  if U_ >= 4 and B > 2:
    x[:, 1] = 0.75                                           # constant column: var = 0, xn = 0 exactly
    x[:, 2] = 5.0 + x[:, 2] * 3e-5                           # variance near eps
    x[:, 3] = 1e3 + x[:, 3]                                  # 1e3 sigma off zero
  return x


def _dice_layer_check(lay, x, gy, y, gx, galpha, tag):
  """y, dx and d alpha of one training step against float64 autograd of utils/activation.py:dice"""
  B = x.shape[0]
  x64 = x.double().requires_grad_(True)
  a64 = lay.alphas.detach().double().requires_grad_(True)
  mean = x64.mean(0)
  var = ((x64 - mean) ** 2).mean(0)
  xn = (x64 - mean) / torch.sqrt(var + DICE_EPS)
  p = torch.sigmoid(xn)
  y64 = a64 * (1 - p) * x64 + p * x64
  y64.backward(gy.double())
  xs, gys, a, m, v, xnr = (t.detach() for t in (x64, gy.double(), a64, mean, var, xn))
  r = 1.0 / torch.sqrt(v + DICE_EPS)
  dm = _mean_bound(B, m, v)
  dr = 0.5 * _var_bound(m, v) / (v + DICE_EPS) + 2 * U
  dxn = _y_bound(xs.abs() + m.abs(), m, r, torch.ones_like(m), torch.zeros_like(m), xs, xnr, dm, dr)
  (yr, dy), (gdr, dgd), (gnr, dgn), (gar, dga), (pr, qr) = _dice_ref(xs, xnr, a, gys)
  pq = pr * qr
  _within(y, y64.detach(), C * (dy + abs((1 - a) * xs) * pq * dxn), '%s y' % tag)
  # d alpha: per-element terms (their own bound and the xn error) summed by torch over the batch
  dga_t = dga + abs(gys * xs) * pq * dxn
  _within(galpha, a64.grad, C * (dga_t.sum(0) + _sum_bound(B, (gar ** 2).sum(0))),
          '%s dalpha' % tag)
  # dx = gx_direct + the batch-norm backward of gxn (er_bias_bn_act_bwd, unit gamma)
  dgd_t = dgd + abs(gys * (1 - a)) * pq * dxn
  dgn_t = dgn + abs(gys * xs * (1 - a)) * pq * abs(1 - 2 * pr) * dxn
  xhat = (xs - m) * r
  cond = (abs(xs) + abs(m)) * r
  sg, sgx = gnr.sum(0), (gnr * xhat).sum(0)
  dsg = _sum_bound(B, (gnr ** 2).sum(0))
  dsgx = _sum_bound(B, ((gnr * xhat) ** 2).sum(0), ((gnr.abs() * cond) ** 2).sum(0))
  gz = r * (gnr - sg / B - xhat * sgx / B)
  dgz = r * (3 * U * (abs(gnr) + abs(sg) / B + abs(xhat) * abs(sgx) / B) + dsg / B +   # test_gpu_dense_bn's
             abs(xhat) * dsgx / B + abs(sgx) / B * (U * cond + 2 * U * abs(xhat))) + _rnd(gz)   # gz bound
  dgz += r * (dgn_t + dgn_t.mean(0) + abs(xhat) * (dgn_t * abs(xhat)).mean(0))   # the error of gxn
  dgz += abs(gz) * dr + r * (abs(sgx) / B + (abs(gnr) * r).mean(0) * abs(xhat)) * dxn   # of r and xhat
  _within(gx, x64.grad, C * (dgd_t + dgz + _rnd(gdr + gz)), '%s dx' % tag)


@pytest.mark.parametrize('B,U_', [(204800, 128), (204800, 64), (204800, 32), (1, 8), (2, 8), (777, 5)])
def test_dice_layer_trains_and_evaluates_like_float64(B, U_):
  """Three training steps (y, dx, d alpha each against float64 autograd), the moving statistics after them, then eval
  with those statistics.  alphas: 0, 1, negative and random per column."""
  g = _gen(B + U_)
  lay = L.Dice(U_).to(DEV).train()
  with torch.no_grad():
    lay.alphas.copy_(torch.randn(U_, device=DEV, generator=g))
    lay.alphas[0::4] = 0.0
    lay.alphas[1::4] = 1.0
    lay.alphas[2::4] = -0.7
    if U_ >= 4 and B > 2:
      lay.alphas[1] = 0.0                                    # the constant column: y = 0.5 x exactly
  mm_ref, mv_ref = lay.moving_mean.double(), lay.moving_var.double()
  mm_b, mv_b = torch.zeros_like(mm_ref), torch.zeros_like(mv_ref)
  for step in range(3):
    x = _dice_layer_inputs(B, U_, g).requires_grad_(True)
    gy = torch.randn(B, U_, device=DEV, generator=g)
    lay.alphas.grad = None
    y = lay(x)
    y.backward(gy)
    if U_ >= 4 and B > 2:
      assert torch.equal(y[:, 1], 0.5 * x.detach()[:, 1]), 'a constant column must give xn = 0 exactly'
    if step == 0 or B < 65536:      # (the float64 bounds at 204,800 rows take seconds: one step there)
      _dice_layer_check(lay, x.detach(), gy, y.detach(), x.grad, lay.alphas.grad, 'dice layer')
    mean = x.detach().double().mean(0)
    var = ((x.detach().double() - mean) ** 2).mean(0)
    mm_ref = mm_ref * MOM + mean * (1 - MOM)
    mv_ref = mv_ref * MOM + var * (1 - MOM)
    mm_b = mm_b * MOM + 4 * U * mm_ref.abs() + (1 - MOM) * _mean_bound(B, mean, var)
    mv_b = mv_b * MOM + 4 * U * mv_ref + (1 - MOM) * _var_bound(mean, var) + 1e-300
  _within(lay.moving_mean, mm_ref, C * mm_b + 1e-300, 'dice moving_mean')
  _within(lay.moving_var, mv_ref, C * mv_b, 'dice moving_var')
  lay.eval()
  x = _dice_layer_inputs(B, U_, g)
  with torch.no_grad():
    y = lay(x)
  xs, a = x.double(), lay.alphas.detach().double()
  m, v = lay.moving_mean.double(), lay.moving_var.double()
  r = 1.0 / torch.sqrt(v + DICE_EPS)
  xnr = (xs - m) * r
  dxn = _y_bound(xs.abs() + m.abs(), m, r, torch.ones_like(m), torch.zeros_like(m), xs, xnr, 0.0, 2 * U)
  (yr, dy), _, _, _, (pr, qr) = _dice_ref(xs, xnr, a, torch.zeros_like(xs))
  _within(y, yr, C * (dy + abs((1 - a) * xs) * pr * qr * dxn), 'dice layer y eval')


# ---------------------------------------------------------------------------------------------------------------------
# dropout
# ---------------------------------------------------------------------------------------------------------------------

M64 = (1 << 64) - 1
G1, G2 = 0x9E3779B97F4A7C15, 0xD1B54A32D192ED03
F1, F2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
LAYER_SEEDS = [(0x5EED0001 + k * 0x9E3779B1) & M64 for k in range(3)]   # the first seeds layers.Dropout hands out


def _drop_bits(seed, ctr, idx):
  """drop_bits of csrc/dense.cu in numpy uint64: the top 32 bits of the splitmix64 finaliser of
  seed + ctr * G1 + i * G2 (all mod 2^64)"""
  with np.errstate(over='ignore'):
    z = np.uint64(seed) + np.uint64(ctr & M64) * np.uint64(G1) + np.asarray(idx, np.uint64) * np.uint64(G2)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(F1)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(F2)
    return (z ^ (z >> np.uint64(31))) >> np.uint64(32)


def _thresh(rate):
  """floor(keep * 2^32) for the keep = 1 - rate the kernel forms in double from the fp32 rate; 2^32 at rate 0"""
  return int((1.0 - float(np.float32(rate))) * 4294967296.0)


def _restate(x, rate, seed, ctr):
  """y = x * fp32(1 / keep) where the draw is below the threshold, else +0 (numpy float32)"""
  keep = 1.0 - float(np.float32(rate))
  kept = _drop_bits(seed, ctr, np.arange(x.size, dtype=np.uint64)) < np.uint64(_thresh(rate))
  return np.where(kept, x * np.float32(1.0 / keep), np.float32(0.0)).astype(np.float32), kept


def _unxorshift(v, s):
  x = v
  for _ in range(64 // s + 1):
    x = v ^ (x >> s)
  return x


def _seed_for(draw, ctr, i, low=0x2545F491):
  """a seed under which element i at counter ctr draws exactly `draw`: the finaliser inverted step by step"""
  z = ((draw << 32) | low) & M64
  z = _unxorshift(z, 31) * pow(F2, -1, 1 << 64) & M64
  z = _unxorshift(z, 27) * pow(F1, -1, 1 << 64) & M64
  z = _unxorshift(z, 30)
  return (z - ctr * G1 - i * G2) & M64


def _dropout_call(lib, x, rate, seed, ctr):
  n = x.numel()
  counter = torch.tensor([ctr], dtype=torch.int64, device=DEV)
  buf, y = _out(n)
  _ok(lib.er_dropout(_p(x), n, float(rate), seed, _p(counter), _p(y), _stream()), 'er_dropout')
  _untouched(buf, y, 'er_dropout')
  assert int(counter[0]) == ctr
  return y.cpu().numpy()


@pytest.mark.parametrize('rate', [1e-7, 0.1, 0.3, 0.5, 0.9, 0.999999])
def test_dropout_matches_the_restated_mask_bit_for_bit(rate):
  lib = _lib.load()
  rng = np.random.default_rng(int(rate * 1e7))
  x = rng.normal(size=10 ** 7 + 3).astype(np.float32)
  xd = torch.from_numpy(x).to(DEV)
  for n in (1, 270335, 270336, 270337):
    for k, ctr in enumerate((0, 1, 2 ** 40)):
      seed = LAYER_SEEDS[(n + k) % 3]
      got = _dropout_call(lib, xd[:n], rate, seed, ctr)
      assert np.array_equal(got.view(np.int32), _restate(x[:n], rate, seed, ctr)[0].view(np.int32)), (n, ctr)
  got = _dropout_call(lib, xd, rate, LAYER_SEEDS[0], 2 ** 40)
  want, kept = _restate(x, rate, LAYER_SEEDS[0], 2 ** 40)
  assert np.array_equal(got.view(np.int32), want.view(np.int32))
  assert abs(kept.mean() - (1 - rate)) < 6 * math.sqrt(rate * (1 - rate) / x.size) + 1e-7


@pytest.mark.parametrize('rate', [0.0, 1e-7, 0.1, 0.5, 0.9, 0.999999])
def test_dropout_threshold_boundary_draws(rate):
  """Seeds built so that the chosen element draws exactly thresh - 1 (kept) and thresh (dropped); at rate 0 it draws
  0xffffffff and must be kept (the threshold is 2^32)."""
  lib = _lib.load()
  th = _thresh(rate)
  x = torch.full((300001,), 1.5, device=DEV)
  cases = [(th - 1, True)] + ([(th, False)] if th < 2 ** 32 else [])
  if rate == 0.0:
    assert int(_drop_bits(0x65ca4f3dbb65e528, 0, [0])[0]) == 0xffffffff
    got = _dropout_call(lib, x, 0.0, 0x65ca4f3dbb65e528, 0)
    assert got[0] == 1.5 and np.array_equal(got, np.full(x.numel(), 1.5, np.float32)), 'rate 0 must keep every element'
  for draw, kept in cases:
    for i, ctr in ((0, 0), (7, 3), (270336, 2 ** 40), (300000, 1)):
      seed = _seed_for(draw, ctr, i)
      assert int(_drop_bits(seed, ctr, [i])[0]) == draw
      got = _dropout_call(lib, x, rate, seed, ctr)
      want = _restate(np.full(x.numel(), 1.5, np.float32), rate, seed, ctr)[0]
      assert np.array_equal(got, want)
      assert (got[i] != 0) == kept, (draw, th, i, ctr, got[i])


def test_dropout_layer_counter_in_eager_steps_and_graph_replays():
  """Step k (counter k before it) draws restate(seed, k) in the forward and the backward, and leaves the counter at
  k + 1, both eagerly and when forward + backward replay from one captured CUDA graph."""
  rate, n = 0.3, 270337
  g = _gen(21)
  xs = torch.randn(n, device=DEV, generator=g)
  gs = torch.randn(n, device=DEV, generator=g)
  x_np, g_np = xs.cpu().numpy(), gs.cpu().numpy()
  drop = L.Dropout(rate).to(DEV).train()

  def check(y, gx, k):
    assert np.array_equal(y.detach().cpu().numpy(), _restate(x_np, rate, drop.seed, k)[0]), k
    assert np.array_equal(gx.cpu().numpy(), _restate(g_np, rate, drop.seed, k)[0]), k
    assert int(drop.counter[0]) == k + 1

  for k in range(3):
    x = xs.clone().requires_grad_(True)      # (a layer's input is a fresh tensor every step)
    y = drop(x)
    y.backward(gs)
    check(y, x.grad, k)
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    for _ in range(2):
      drop(xs.clone().requires_grad_(True)).backward(gs)
  torch.cuda.current_stream().wait_stream(side)
  drop.counter.zero_()
  x = xs.clone().requires_grad_(True)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    y = drop(x)
    y.backward(gs)
  assert int(drop.counter[0]) == 0
  for k in range(3):
    graph.replay()
    torch.cuda.synchronize()
    check(y, x.grad, k)


def _no_worse(mine, t32, t64, what, factor=4.0):
  """test_gpu_dense.py's rule: the kernels' error against float64 is no worse than torch fp32's by more than a small
  factor (bulk: 99.9th percentile; tail: maximum)"""
  em, et = (mine.double() - t64).abs().flatten(), (t32.double() - t64).abs().flatten()
  qm = float(torch.quantile(em, 0.999)) if em.numel() > 1000 else float(em.max())
  qt = float(torch.quantile(et, 0.999)) if et.numel() > 1000 else float(et.max())
  scale = float(t64.abs().mean())
  assert qm <= factor * qt + 2e-6 * scale, '%s: p99.9 error %.3g vs torch fp32 %.3g' % (what, qm, qt)
  assert float(em.max()) <= 10 * float(et.max()) + 1e-5 * scale, '%s: max error %.3g vs torch fp32 %.3g' % (
      what, float(em.max()), float(et.max()))


@pytest.mark.parametrize('use_bn', [True, False])
@pytest.mark.parametrize('act', ['gelu', 'elu'])
def test_dnn_with_dropout_on_every_layer_matches_float64(use_bn, act):
  """DNN(48 -> 64 -> 32) with an activation and dropout_ratio on both layers: output and every parameter gradient
  against float64 autograd that applies the restated masks of the step's counters."""
  torch.backends.cuda.matmul.allow_tf32 = False
  gen = torch.Generator().manual_seed(7)
  units = L.Units([64, 32])
  units.activation, units.dropout, units.use_bn = act, (0.3, 0.5), use_bn
  dnn = L.DNN(48, units, generator=gen).to(DEV).train()
  assert all(isinstance(d, L.Dropout) for d in dnn.dropouts)
  B = 512
  x = torch.randn(B, 48, generator=gen).to(DEV).requires_grad_(True)
  gy = torch.randn(B, 32, generator=gen).to(DEV)
  for step in range(2):
    x.grad = None
    dnn.zero_grad(set_to_none=True)
    ctrs = [int(d.counter[0]) for d in dnn.dropouts]
    assert ctrs == [step, step]
    y = dnn(x)
    y.backward(gy)

    def ref(dt):
      leaves = []
      h = x.detach().to(dt).clone().requires_grad_(True)
      h0 = h
      for lay, drop, c in zip(dnn.layers, dnn.dropouts, ctrs):
        p = {k: getattr(lay, k).detach().to(dt).clone().requires_grad_(True)
             for k in ('kernel', 'bias', 'gamma', 'beta') if hasattr(lay, k)}
        leaves.append(p)
        z = h @ p['kernel'] + p['bias']
        if use_bn:
          mu = z.mean(0)
          z = (z - mu) / torch.sqrt(((z - mu) ** 2).mean(0) + float(np.float32(L.BN_EPS))) * p['gamma'] + p['beta']
        z = torch.nn.functional.gelu(z, approximate='tanh') if act == 'gelu' else torch.nn.functional.elu(z)
        _, kept = _restate(np.zeros(z.numel(), np.float32), drop.rate, drop.seed, c)
        mask = torch.from_numpy(kept.reshape(z.shape)).to(DEV, dt) * float(np.float32(1.0 / (1.0 - drop.rate)))
        h = z * mask
      h.backward(gy.to(dt))
      return h.detach(), h0, leaves

    y64, x64, p64 = ref(torch.float64)
    y32, x32, p32 = ref(torch.float32)
    _no_worse(y.detach(), y32, y64, 'dnn y')
    _no_worse(x.grad, x32.grad, x64.grad, 'dnn x.grad')
    for li, (lay, d32, d64) in enumerate(zip(dnn.layers, p32, p64)):
      for k in d64:
        if use_bn and k == 'bias':
          assert bool((lay.bias.grad == 0).all())
          continue
        _no_worse(getattr(lay, k).grad, d32[k].grad, d64[k].grad, 'dnn %s.grad %d' % (k, li))
  assert [int(d.counter[0]) for d in dnn.dropouts] == [2, 2]


# ---------------------------------------------------------------------------------------------------------------------
# er_gemm_small
# ---------------------------------------------------------------------------------------------------------------------

def _slices(M, N, Kd):
  """small_gemm_slices of csrc/small_gemm.cuh"""
  out_ctas = -(-(M * N) // 256)
  if Kd < 512 or out_ctas >= 132:
    return 1
  return max(1, min(-(-264 // out_ctas), Kd // 64))


def _operand(rows, cols, major, g, pad=3):
  """a [rows, cols] fp32 operand, row-major (major='r') or column-major ('c') inside a padded NaN buffer"""
  v = torch.randn(rows, cols, device=DEV, generator=g)
  if major == 'r':
    buf = torch.full((rows, cols + pad), float('nan'), device=DEV)
    buf[:, :cols] = v
    return buf[:, :cols]
  buf = torch.full((cols, rows + pad), float('nan'), device=DEV)
  buf[:, :rows] = v.t()
  return buf[:, :rows].t()


def _gemm_small_check(M, N, Kd, g, lay='rr', bias=True, pitch=0, shift=0, what='gemm_small'):
  lib = _lib.load()
  a = _operand(M, Kd, lay[0], g)
  b = _operand(Kd, N, lay[1], g)
  bi = torch.randn(N, device=DEV, generator=g) if bias else None
  ns = _slices(M, N, Kd)
  nbytes = lib.er_gemm_small_workspace_bytes(M, N, Kd)
  assert nbytes == (4 * ns * M * N if ns > 1 else 0)
  ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=DEV)
  buf, c = _out(M, N, pitch=N + pitch, shift=shift)

  def call():
    _ok(lib.er_gemm_small(_p(a), a.stride(0), a.stride(1), _p(b), b.stride(0), b.stride(1), _p(bi), _p(c), c.stride(0),
                          M, N, Kd, _p(ws), nbytes, _stream()), 'er_gemm_small')
    return c.clone()

  first = call()
  second = call()
  assert torch.equal(first, second), 'er_gemm_small must be deterministic'
  _untouched(buf, c, what)
  a64, b64 = a.double(), b.double()
  ref = a64 @ b64 + (bi.double() if bias else 0.0)
  kps = -(-Kd // ns)
  gam = kps * U / (1 - kps * U)
  bound = (gam + ns * U) * (a64.abs() @ b64.abs()) + (U * (ref.abs() + bi.double().abs()) if bias else 0.0)
  _within(c, ref, C * bound + 1e-300, what)
  return ns


@pytest.mark.parametrize('N', range(1, 8))
def test_gemm_small_every_narrow_n(N):
  g = _gen(N)
  for M, Kd in ((4099, 1000), (20000, 37)):
    _gemm_small_check(M, N, Kd, g, 'rr' if M > 5000 else 'rc')


@pytest.mark.parametrize('M', range(1, 8))
def test_gemm_small_every_short_m_and_k(M):
  g = _gen(100 + M)
  _gemm_small_check(M, 3000, 600, g, 'cr')
  _gemm_small_check(300, 300, M, g, 'cc', bias=False)


@pytest.mark.parametrize('lay', ['rr', 'rc', 'cr', 'cc'])
def test_gemm_small_operand_layouts_and_slice_edges(lay):
  """K = 511 (never sliced) / 512; M N = 33,536 (131 output CTAs: K is sliced) / 33,537 (132: not); M N <= 256 with
  K = 5000 (78 slices of 65: the last starts at 5005 > K and contributes 0); pitched and misaligned C; bias NULL and
  not in the single-slice and the reduce kernel."""
  g = _gen(7)
  assert _gemm_small_check(64, 4, 511, g, lay) == 1
  assert _gemm_small_check(64, 4, 512, g, lay, bias=False, pitch=5, shift=1) > 1
  assert _gemm_small_check(8384, 4, 1024, g, lay) == 3
  assert _gemm_small_check(4791, 7, 1024, g, lay, bias=False, pitch=2, shift=1) == 1
  assert _gemm_small_check(64, 4, 5000, g, lay, shift=1) == 78
  assert _gemm_small_check(1, 1, 5000, g, lay, bias=False) == 78
  assert 77 * 65 >= 5000


@pytest.mark.parametrize('d', [96, 256])
@pytest.mark.parametrize('E', [3, 4, 8])
def test_gemm_small_mmoe_gate_shapes(d, E):
  """the gate layer's forward x[B, d] W[d, E] + b, dX = dY[B, E] W^T[E, d] and dW = X^T[d, B] dY[B, E]"""
  g = _gen(d * E)
  B = 16384
  _gemm_small_check(B, E, d, g, 'rr', what='gemm_small gate fwd')
  _gemm_small_check(B, d, E, g, 'rc', bias=False, what='gemm_small gate dX')
  assert _gemm_small_check(d, E, B, g, 'cr', bias=False, what='gemm_small gate dW') > 1


def test_gemm_small_refusals():
  """A missing or short workspace and an output over 2^31 elements are refused by the argument checks, before any
  launch: the pointers passed are small real buffers that the call never reaches."""
  lib = _lib.load()
  t = torch.zeros(64, device=DEV)
  M, N, Kd = 4, 4, 5000
  need = lib.er_gemm_small_workspace_bytes(M, N, Kd)
  assert need == 4 * 78 * M * N
  ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
  for w, nb in ((None, 0), (ws, need - 4)):
    st = lib.er_gemm_small(_p(t), Kd, 1, _p(t), N, 1, None, _p(t), N, M, N, Kd, _p(w), nb, _stream())
    assert st == _lib.ER_ERR_WORKSPACE and b'workspace' in lib.er_last_error()
  M, N = 65536, 32769
  st = lib.er_gemm_small(_p(t), 1, 1, _p(t), 1, 1, None, _p(t), N, M, N, 1, None, 0, _stream())
  assert st == _lib.ER_ERR_INVALID_ARG and b'too large' in lib.er_last_error()
  st = lib.er_gemm_small(_p(t), 1, 1, _p(t), 1, 1, None, _p(t), 3, 2, 4, 1, None, 0, _stream())
  assert st == _lib.ER_ERR_INVALID_ARG    # ldc < N
  torch.cuda.synchronize()


def test_zz_report_worst_ratios():
  """prints the worst error / bound of every output checked above (pytest -s shows it)"""
  for k in sorted(WORST):
    print('WORST %-28s %.3f' % (k, WORST[k]))
