"""GPU: the batch-norm paths of the dense layer (DenseLayer with use_bn) against float64, each path on its own.

  er_gemm_bn          GEMM whose epilogue produces the training batch statistics: per-half shifted sums, per-tile
                      Welford partials, and the last row tile of a column (picked by a self-resetting ticket
                      counter) merges the tiles.  Taken when K is not split (kernels.gemm_bn).
  er_bias_bn_act_fwd  split-K er_gemm, then the two-pass chunked Welford statistics + normalise + ReLU: the route of
                      long-K, small-batch layers (DeepFM's 624 -> 256 layer at every batch <= 4096), of eval, and of
                      layers without batch norm (gamma = NULL).
  er_bn_act_apply     normalise + ReLU with given statistics, vector kernel and scalar kernel.
  er_bias_bn_act_bwd  column sums of g and g*xhat, then the input gradient, vector kernel and scalar kernel.
  DenseLayer          both forward routes end to end, forward, backward, moving statistics and eval.

Every reference is float64 and computed from the tensors the kernel received or produced: statistics are compared
with the float64 statistics of the kernel's own z (so GEMM error does not blur them), and the ReLU decisions of the
backward pass are the kernel's y > 0.  The scalar kernels are reached with units % 4 == 0 through views one float
past a 16-byte boundary.

Bounds, with u = 2^-24 (fp32 unit roundoff), m / r the statistics used and t = |z| + |bias| + |m|:
  z (er_gemm_bn)  the er_gemm bound of test_gpu_gemm: 4e-6 * sum_k |x||w|.
  mean            4u (8 + sqrt(M / 128)) (|mean| + sigma) + u |mean|: fp32 shifted sums over pieces of <= 64 rows,
                  then the merge over the 128-row tiles (or row chunks) of sums of size |mean|.
  var / rstd      dvar = 1e-5 var + 8u |mean| sigma, |rstd - ref| <= (0.5 dvar / (var + eps) + 2u) rstd.  The
                  |mean| sigma term is the exact variance of inputs perturbed by u relative (the merges combine
                  means rounded at |mean|); the shifted sums and Welford merges stay within 3u |mean| sigma.  A
                  one-pass E[x^2] - E[x]^2 in fp32 errs by ~u mean^2, 100x this bound on the stress columns.
  y               |gamma| r (2u t + dmean + |z + b - m| (drstd + 3u)) + 2u (|beta| + |y|): first-order rounding of
                  each fp32 operation, plus the error of the statistics used.
  column sums     4u (sqrt(B) ||terms||_2 + ||e||_2), e = |g| t r the rounding carried by each g*xhat term.
  gz              first-order rounding of gamma r (g - sum g / B - xhat sum(g xhat) / B) plus the column-sum bounds.
  layer           |err| <= 1e-5 max |ref| per tensor (GEMM error propagated through the normalisation).
Worst error / bound measured on an H100 80GB HBM3 (400 W power limit): er_gemm_bn z 0.16, mean 0.20, rstd 0.46,
moving statistics 0.43; er_bias_bn_act_fwd mean 0.055, rstd 0.46, y 0.087 (training) / 0.50 (eval), moving statistics
0.36; gamma = NULL 1.0 (its bound is the exact rounding bound u |z + b|); er_bn_act_apply 0.47; er_bias_bn_act_bwd gz 0.68,
ggamma 0.31, gbeta / gbias 0.42, vector vs scalar 0.69; layer 0.19 (eval y), 0.13 or less for the rest.
Stress inputs: a bias of 1e3 on every other column (mean ~ 1e3 sigma after the bias add), in er_gemm_bn a column
whose mean is ~1e3 sigma (a constant input column times a weight of 1e3) and a column of zero weights (var = 0
exactly: rstd must be 1/sqrt(eps) in fp32, bit for bit).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, kernels as K, layers as L

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
EPS = float(np.float32(1e-3))     # what the kernels receive (fp32)
MOM = float(np.float32(0.99))
TOL_VAR = 1e-5
ROWS = 16384    # float64 references are formed in blocks of rows: a few hundred MB at most per temporary


def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


def _within(got, ref, bound, what):
  err = (got.double() - ref).abs()
  ratio = float((err / bound).max())
  assert ratio <= 1.0, '%s: error %.3g x bound (max abs err %.3g)' % (what, ratio, float(err.max()))
  return ratio


def _blocks(rows):
  return [slice(r0, r0 + ROWS) for r0 in range(0, rows, ROWS)]


def _col_stats(v, shift=0.0):
  """float64 mean and biased variance of the columns of v + shift (two passes over blocks of rows)"""
  n = v.shape[0]
  mean = sum((v[s].double() + shift).sum(0) for s in _blocks(n)) / n
  return mean, sum(((v[s].double() + shift - mean) ** 2).sum(0) for s in _blocks(n)) / n


def _mean_bound(rows, mean, var):
  return 4 * U * (8 + math.sqrt(rows / 128)) * (mean.abs() + var.sqrt()) + U * mean.abs() + 1e-30


def _var_bound(mean, var):
  return TOL_VAR * var + 8 * U * mean.abs() * var.sqrt()


def _rstd_ref(mean, var):
  """float64 rstd and the bound of an fp32 rstd whose var is within _var_bound"""
  rstd = 1.0 / torch.sqrt(var + EPS)
  return rstd, rstd * (0.5 * _var_bound(mean, var) / (var + EPS) + 2 * U)


def _y_bound(t, m, r, gamma, beta, zb, y_ref, dm, dr):
  return (gamma.abs() * r * (2 * U * t + dm + (zb - m).abs() * (dr + 3 * U)) + 2 * U * (beta.abs() + y_ref.abs()) +
          1e-30)


def _check_y(y, z, b64, m, r, gamma, beta, dm, dr, relu, what):
  """y = act((z + b - m) r gamma + beta) against float64 with the _y_bound, block by block"""
  for s in _blocks(z.shape[0]):
    z64 = z[s].double()
    zb = z64 + b64
    h = (zb - m) * r * gamma + beta
    y_ref = torch.relu(h) if relu else h
    _within(y[s], y_ref, _y_bound(z64.abs() + b64.abs() + m.abs(), m, r, gamma, beta, zb, y_ref, dm, dr), what)


def _misaligned(t):
  """a contiguous copy of t whose data pointer is 4 bytes past a 16-byte boundary"""
  flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
  v = flat[1:].view(t.shape)
  v.copy_(t)
  assert v.data_ptr() % 16 == 4
  return v


# ---------------------------------------------------------------------------------------------------------------------
# er_gemm_bn
# ---------------------------------------------------------------------------------------------------------------------

def _stress_operands(M, N, Kd, g):
  """x [M, Kd], w [Kd, N]: column 0 has zero weights (z = 0, var = 0); column N-1 adds 1e3 x a constant input
  column (mean ~ 1e3 sigma)."""
  x = torch.randn(M, Kd, device=DEV, generator=g)
  x[:, 0] = 1.0
  w = torch.randn(Kd, N, device=DEV, generator=g) / math.sqrt(Kd)
  w[:, 0] = 0.0
  w[0, N - 1] = 1e3
  return x, w


def _check_gemm_bn(x, w, bias, z, save_mean, save_rstd):
  """z against the GEMM bound, save_mean / save_rstd against float64 statistics of z; returns (mean, var)."""
  x64, w64 = x.double(), w.double()
  _within(z, x64 @ w64, 4e-6 * (x64.abs() @ w64.abs()) + 1e-30, 'gemm_bn z')
  mz, var = _col_stats(z)
  mean = mz + (bias.double() if bias is not None else 0.0)
  _within(save_mean, mean, _mean_bound(z.shape[0], mz, var), 'gemm_bn save_mean')
  r, rb = _rstd_ref(mz, var)   # the statistics are taken of z, before the bias
  _within(save_rstd, r, rb, 'gemm_bn save_rstd')
  N = z.shape[1]
  assert float(mz[N - 1].abs()) > 500 * float(var[N - 1].sqrt()), 'stress column lost its offset'
  assert bool((z[:, 0] == 0).all())
  assert float(save_rstd[0]) == float(1.0 / torch.tensor(EPS, dtype=torch.float32).sqrt())   # var == 0 exactly
  if bias is not None:
    assert float(save_mean[0]) == float(bias[0])
  return mean, var


GEMM_BN_SHAPES = ([(M, N) for M in (8, 63, 64, 65, 127, 129, 777, 8192)
                   for N in (8, 16, 17, 32, 33, 64, 65, 128, 129, 200, 1000)] +
                  [(204800, N) for N in (128, 64, 32)])   # 4096 x 50 DIN history rows: 1600 row tiles to merge


@pytest.mark.parametrize('M,N', GEMM_BN_SHAPES)
def test_gemm_bn_statistics_match_float64(M, N):
  """Every MMA width, a second column tile with one live column, 8 column tiles; one half-tile, an empty second
  half, ragged last tiles.  Two calls: bit-identical outputs, moving statistics updated twice."""
  Kd = 40
  assert _lib.load().er_gemm_workspace_bytes(M, N, Kd) == 0
  g = _gen(1009 * M + N)
  x, w = _stress_operands(M, N, Kd, g)
  bias = torch.randn(N, device=DEV, generator=g)
  mm0 = torch.randn(N, device=DEV, generator=g) * 0.1
  mv0 = torch.rand(N, device=DEV, generator=g) + 0.5
  mm, mv = mm0.clone(), mv0.clone()
  first = K.gemm_bn(x, w, bias, mm, mv, 1e-3, 0.99)
  second = K.gemm_bn(x, w, bias, mm, mv, 1e-3, 0.99)
  assert first is not None
  assert all(torch.equal(p, q) for p, q in zip(first, second)), 'er_gemm_bn must be deterministic'
  mean, var = _check_gemm_bn(x, w, bias, *first)
  mm0, mv0 = mm0.double(), mv0.double()
  mz = mean - bias.double()
  dm = _mean_bound(M, mz, var)
  _within(mm, (mm0 * MOM + mean * (1 - MOM)) * MOM + mean * (1 - MOM),
          4 * U * (mm0.abs() + mean.abs()) + 2 * (1 - MOM) * dm, 'gemm_bn moving_mean')
  _within(mv, (mv0 * MOM + var * (1 - MOM)) * MOM + var * (1 - MOM),
          4 * U * (mv0 + var) + 2 * (1 - MOM) * _var_bound(mz, var) + 1e-30, 'gemm_bn moving_var')


def test_gemm_bn_counters_self_reset_and_m_major_operand():
  """The column tickets are left at zero: shape A, then a shape with more column tiles, then A again gives
  bit-identical results.  kernels.gemm_bn keeps one workspace per stream and replaces it (zeroed) only when a call
  needs more bytes, so the repeat of A runs on the workspace whose counters the wider call used.  The A operand is
  also read M-major (a transposed view, NaN in its padding)."""
  g = _gen(5)
  xa, wa = _stress_operands(777, 200, 81, g)
  ba = torch.randn(200, device=DEV, generator=g)
  xb, wb = _stress_operands(300, 1000, 40, g)     # 8 column tiles
  bb = torch.randn(1000, device=DEV, generator=g)
  first = K.gemm_bn(xa, wa, ba, None, None, 1e-3, 0.99)
  other = K.gemm_bn(xb, wb, bb, None, None, 1e-3, 0.99)
  again = K.gemm_bn(xa, wa, ba, None, None, 1e-3, 0.99)
  _check_gemm_bn(xa, wa, ba, *first)
  _check_gemm_bn(xb, wb, bb, *other)
  assert all(torch.equal(p, q) for p, q in zip(first, again)), 'a ticket counter was left non-zero'
  xt = torch.full((81, 780), float('nan'), device=DEV)
  xt[:, :777] = xa.t()
  at = xt[:, :777].t()
  assert at.stride() == (1, 780)
  _check_gemm_bn(at, wa, ba, *K.gemm_bn(at, wa, ba, None, None, 1e-3, 0.99))


def test_gemm_bn_abi_without_moving_statistics():
  lib = _lib.load()
  M, N, Kd = 777, 200, 40
  g = _gen(6)
  x, w = _stress_operands(M, N, Kd, g)
  bias = torch.randn(N, device=DEV, generator=g)
  z = torch.empty(M, N, device=DEV)
  mean = torch.full((N,), float('nan'), device=DEV)
  rstd = torch.full((N,), float('nan'), device=DEV)
  ws = torch.zeros(lib.er_gemm_bn_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)
  bn = _lib.ErBnStats(bias.data_ptr(), mean.data_ptr(), rstd.data_ptr(), None, None, 1e-3, 0.99)
  _lib.check(lib.er_gemm_bn(x.data_ptr(), Kd, 0, w.data_ptr(), N, 1, z.data_ptr(), N, M, N, Kd, ctypes.byref(bn),
                            ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream), 'er_gemm_bn')
  _check_gemm_bn(x, w, bias, z, mean, rstd)


def test_gemm_bn_refuses_split_k_and_more_than_256_column_tiles():
  lib = _lib.load()
  stream = torch.cuda.current_stream().cuda_stream
  # DeepFM's first DNN layer on Criteo at batch 1024: K is split, so the layer takes the two-pass route
  M, N, Kd = 1024, 256, 624
  assert lib.er_gemm_workspace_bytes(M, N, Kd) > 0
  x = torch.randn(M, Kd, device=DEV)
  w = torch.randn(Kd, N, device=DEV)
  assert K.gemm_bn(x, w, None, None, None, 1e-3, 0.99) is None
  z, mean, rstd = torch.empty(M, N, device=DEV), torch.empty(N, device=DEV), torch.empty(N, device=DEV)
  ws = torch.zeros(lib.er_gemm_bn_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)
  bn = _lib.ErBnStats(None, mean.data_ptr(), rstd.data_ptr(), None, None, 1e-3, 0.99)
  st = lib.er_gemm_bn(x.data_ptr(), Kd, 0, w.data_ptr(), N, 1, z.data_ptr(), N, M, N, Kd, ctypes.byref(bn),
                      ws.data_ptr(), ws.numel(), stream)
  assert st == _lib.ER_ERR_INVALID_ARG and b'unsplit K' in lib.er_last_error()
  # N = 32769: 257 column tiles
  M, N, Kd = 8, 32769, 8
  x = torch.randn(M, Kd, device=DEV)
  w = torch.randn(Kd, N + 3, device=DEV)
  z, mean, rstd = torch.empty(M, N, device=DEV), torch.empty(N, device=DEV), torch.empty(N, device=DEV)
  ws = torch.zeros(lib.er_gemm_bn_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)
  bn = _lib.ErBnStats(None, mean.data_ptr(), rstd.data_ptr(), None, None, 1e-3, 0.99)
  st = lib.er_gemm_bn(x.data_ptr(), Kd, 0, w.data_ptr(), N + 3, 1, z.data_ptr(), N, M, N, Kd, ctypes.byref(bn),
                      ws.data_ptr(), ws.numel(), stream)
  assert st == _lib.ER_ERR_INVALID_ARG and b'N too large' in lib.er_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# er_bias_bn_act_fwd / er_bn_act_apply / er_bias_bn_act_bwd
# ---------------------------------------------------------------------------------------------------------------------

BATCHES = (1, 7, 8, 9, 15, 16, 17, 777, 8192, 100003)
UNITS = (1, 5, 31, 32, 33, 256, 1000)


def _epilogue_inputs(B, n, seed):
  g = _gen(seed)
  z = torch.randn(B, n, device=DEV, generator=g)
  bias = torch.randn(n, device=DEV, generator=g)
  bias[0::2] += 1e3
  gamma = torch.rand(n, device=DEV, generator=g) + 0.5
  beta = torch.randn(n, device=DEV, generator=g) * 0.2
  return g, z, bias, gamma, beta


@pytest.mark.parametrize('n', UNITS)
@pytest.mark.parametrize('B', BATCHES)
def test_bias_bn_act_fwd_and_apply_match_float64(B, n):
  """Training (batch statistics, moving statistics), eval, and gamma = NULL (bias + activation only), with and without
  bias, ReLU on and off; then er_bn_act_apply with the training statistics on its vector and its scalar kernel.
  Batch 1 has var = 0."""
  g, z, bias, gamma, beta = _epilogue_inputs(B, n, 31 * B + n)
  ws = K.dense_workspace(B, n, DEV)
  ga64, be64 = gamma.double(), beta.double()
  for b in (None, bias):
    b64 = b.double() if b is not None else torch.zeros(n, dtype=torch.float64, device=DEV)
    mean, var = _col_stats(z, b64)
    dm = _mean_bound(B, mean, var)
    r, rb = _rstd_ref(mean, var)
    for relu in (False, True):
      # no batch norm: one correctly rounded add
      y, _, _ = K.bias_bn_act_fwd(z, b, None, None, None, None, 1e-3, 0.99, True, relu, ws)
      for s in _blocks(B):
        zb = z[s].double() + b64
        _within(y[s], torch.relu(zb) if relu else zb, U * zb.abs() + 1e-30, 'bias_act y')
      # training
      mm0 = torch.randn(n, device=DEV, generator=g) * 0.1
      mv0 = torch.rand(n, device=DEV, generator=g) + 0.5
      mm, mv = mm0.clone(), mv0.clone()
      y, sm, sr = K.bias_bn_act_fwd(z, b, gamma, beta, mm, mv, 1e-3, 0.99, True, relu, ws)
      _within(sm, mean, dm, 'fwd save_mean')
      _within(sr, r, rb, 'fwd save_rstd')
      _within(mm, mm0.double() * MOM + mean * (1 - MOM), 4 * U * (mm0.double().abs() + mean.abs()) + (1 - MOM) * dm,
              'fwd moving_mean')
      _within(mv, mv0.double() * MOM + var * (1 - MOM), 4 * U * (mv0.double() + var) + (1 - MOM) * _var_bound(mean, var),
              'fwd moving_var')
      _check_y(y, z, b64, mean, r, ga64, be64, dm, rb / r, relu, 'fwd y training')
      del y
      # eval: the moving statistics are read, not written
      mme = (b if b is not None else 0.0) + torch.randn(n, device=DEV, generator=g) * 0.1
      mve = torch.rand(n, device=DEV, generator=g) + 0.5
      mme_in, mve_in = mme.clone(), mve.clone()
      ye, _, _ = K.bias_bn_act_fwd(z, b, gamma, beta, mme, mve, 1e-3, 0.99, False, relu, ws)
      assert torch.equal(mme, mme_in) and torch.equal(mve, mve_in)
      re = 1.0 / torch.sqrt(mve.double() + EPS)
      _check_y(ye, z, b64, mme.double(), re, ga64, be64, 0.0, 2 * U, relu, 'fwd y eval')
      del ye
      # er_bn_act_apply with the statistics the training pass saved: vector and scalar kernel
      sm64, sr64 = sm.double(), sr.double()
      _check_y(K.bn_act_apply(z, b, gamma, beta, sm, sr, relu), z, b64, sm64, sr64, ga64, be64, 0.0, 0.0, relu,
               'bn_act_apply y')
      ys = _misaligned(torch.empty_like(z))
      K.bn_act_apply(_misaligned(z), b, gamma, beta, sm, sr, relu, y=ys)
      _check_y(ys, z, b64, sm64, sr64, ga64, be64, 0.0, 0.0, relu, 'bn_act_apply y')
      del ys


def _sum_bound(B, terms_sq, e_sq=0.0):
  """bound of an fp32 column sum of B terms whose squares sum to terms_sq, the terms carrying rounding u*e with
  sum e^2 = e_sq"""
  return 4 * U * (math.sqrt(B) * terms_sq.sqrt() + e_sq ** 0.5) + 1e-30


@pytest.mark.parametrize('n', UNITS)
@pytest.mark.parametrize('B', BATCHES)
def test_bias_bn_act_bwd_vector_and_scalar_match_float64(B, n):
  """BN with ReLU, BN without ReLU, and no BN (gbias = column sum of the masked g), each on the vector kernel
  (units % 4 == 0, aligned) and the scalar kernel (misaligned views of the same data): both within the float64
  bound and within it of each other; two calls are bit-identical; under BN gbias is exactly zero."""
  g, z, bias, gamma, beta = _epilogue_inputs(B, n, 37 * B + n)
  gy = torch.randn(B, n, device=DEV, generator=g)
  ws = K.dense_workspace(B, n, DEV)
  b64, ga64 = bias.double(), gamma.double()
  zm, gym = _misaligned(z), _misaligned(gy)
  for use_bn, relu in ((True, True), (True, False), (False, True)):
    mm = torch.zeros(n, device=DEV)
    mv = torch.ones(n, device=DEV)
    gam = gamma if use_bn else None
    y, sm, sr = K.bias_bn_act_fwd(z, bias, gam, beta if use_bn else None, mm, mv, 1e-3, 0.99, True, relu, ws)
    vec = K.bias_bn_act_bwd(z, bias, gam, y, gy, sm, sr, relu, ws)
    again = K.bias_bn_act_bwd(z, bias, gam, y, gy, sm, sr, relu, ws)
    assert all(p is None or torch.equal(p, q) for p, q in zip(vec, again)), 'er_bias_bn_act_bwd must be deterministic'
    sca = K.bias_bn_act_bwd(zm, bias, gam, _misaligned(y), gym, sm, sr, relu, ws)
    gmask = torch.where(y > 0, gy, torch.zeros_like(gy)) if relu else gy
    m64, r64 = (sm.double(), sr.double()) if use_bn else (None, None)

    def block(s):
      """float64 g, xhat and cond (|xhat| can carry rounding u * cond) of rows s"""
      g64 = gmask[s].double()
      if not use_bn:
        return g64, None, None
      z64 = z[s].double()
      return g64, ((z64 + b64) - m64) * r64, (z64.abs() + b64.abs() + m64.abs()) * r64

    sg = sg_sq = sgx = sgx_sq = e_sq = 0.0
    for s in _blocks(B):
      g64, xhat, cond = block(s)
      sg, sg_sq = sg + g64.sum(0), sg_sq + g64.pow(2).sum(0)
      if use_bn:
        sgx, sgx_sq = sgx + (g64 * xhat).sum(0), sgx_sq + (g64 * xhat).pow(2).sum(0)
        e_sq = e_sq + (g64.abs() * cond).pow(2).sum(0)
    dsg = _sum_bound(B, sg_sq)
    if use_bn:
      dsgx = _sum_bound(B, sgx_sq, e_sq)
      for s in _blocks(B):
        g64, xhat, cond = block(s)
        gz_ref = ga64 * r64 * (g64 - sg / B - xhat * sgx / B)
        gz_bound = (ga64.abs() * r64 * (3 * U * (g64.abs() + sg.abs() / B + xhat.abs() * sgx.abs() / B) + dsg / B +
                                        xhat.abs() * dsgx / B + sgx.abs() / B * (U * cond + 2 * U * xhat.abs())) +
                    U * gz_ref.abs() + 1e-30)
        _within(vec[0][s], gz_ref, gz_bound, 'bwd gz')
        _within(sca[0][s], gz_ref, gz_bound, 'bwd gz')
        _within(vec[0][s], sca[0][s].double(), gz_bound, 'bwd gz vector vs scalar')
    for name, (gz, gbias, ggamma, gbeta) in (('vector', vec), ('scalar', sca)):
      if use_bn:
        _within(ggamma, sgx, dsgx, 'bwd ggamma')
        _within(gbeta, sg, dsg, 'bwd gbeta')
        assert bool((gbias == 0).all()), '%s: gbias must be exactly zero under batch norm' % name
      else:
        assert torch.equal(gz, gmask), '%s: without batch norm gz is the masked g' % name
        _within(gbias, sg, dsg, 'bwd gbias')
    if use_bn:
      _within(vec[2], sca[2].double(), dsgx, 'bwd ggamma vector vs scalar')
      _within(vec[3], sca[3].double(), dsg, 'bwd gbeta vector vs scalar')
    else:
      _within(vec[1], sca[1].double(), dsg, 'bwd gbias vector vs scalar')


def test_vector_and_scalar_epilogue_kernels_are_both_reached():
  """The aligned and the misaligned calls of the two tests above really run different kernels."""
  from torch.profiler import ProfilerActivity, profile
  B, n = 64, 32
  _, z, bias, gamma, beta = _epilogue_inputs(B, n, 1)
  gy = torch.randn(B, n, device=DEV)
  ws = K.dense_workspace(B, n, DEV)
  mm, mv = torch.zeros(n, device=DEV), torch.ones(n, device=DEV)
  y, sm, sr = K.bias_bn_act_fwd(z, bias, gamma, beta, mm, mv, 1e-3, 0.99, True, True, ws)

  def kernels_of(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
      fn()
      torch.cuda.synchronize()
    return ' '.join(e.name for e in prof.events())

  names = kernels_of(lambda: K.bn_act_apply(z, bias, gamma, beta, sm, sr, True))
  assert 'bn_act_apply_vec_kernel' in names and 'bn_act_apply_kernel' not in names, names
  names = kernels_of(lambda: K.bn_act_apply(_misaligned(z), bias, gamma, beta, sm, sr, True))
  assert 'bn_act_apply_kernel' in names and 'bn_act_apply_vec_kernel' not in names, names
  names = kernels_of(lambda: K.bias_bn_act_bwd(z, bias, gamma, y, gy, sm, sr, True, ws))
  assert 'bn_bwd_apply_vec_kernel' in names and 'bn_bwd_apply_kernel' not in names, names
  names = kernels_of(lambda: K.bias_bn_act_bwd(_misaligned(z), bias, gamma, y, gy, sm, sr, True, ws))
  assert 'bn_bwd_apply_kernel' in names and 'bn_bwd_apply_vec_kernel' not in names, names


# ---------------------------------------------------------------------------------------------------------------------
# the layer, both routes
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('B,fused', [(1024, False), (4096, False), (8192, True)])
def test_dense_layer_both_routes_match_float64(B, fused, monkeypatch):
  """DenseLayer(624, 256, bn, relu): at B <= 4096 K is split and the layer runs er_gemm + er_bias_bn_act_fwd; at
  8192 it runs er_gemm_bn + er_bn_act_apply.  A spy on kernels.gemm_bn asserts the route.  Two training steps
  (forward + backward against float64 autograd with the kernel's ReLU decisions), the moving statistics, then eval."""
  assert (_lib.load().er_gemm_workspace_bytes(B, 256, 624) == 0) == fused
  routes = []
  real = K.gemm_bn

  def spy(*args, **kwargs):
    out = real(*args, **kwargs)
    routes.append(out is not None)
    return out

  monkeypatch.setattr(K, 'gemm_bn', spy)
  gen = torch.Generator().manual_seed(B)
  lay = L.DenseLayer(624, 256, use_bn=True, relu=True, generator=gen)
  with torch.no_grad():
    lay.bias.copy_(torch.randn(256, generator=gen) * 0.1)
    lay.gamma.copy_(torch.rand(256, generator=gen) + 0.5)
    lay.beta.copy_(torch.randn(256, generator=gen) * 0.2)
    lay.moving_mean.copy_(torch.randn(256, generator=gen) * 0.1)
    lay.moving_var.copy_(torch.rand(256, generator=gen) + 0.5)
  lay = lay.to(DEV).train()
  params = {k: getattr(lay, k).detach().double() for k in ('kernel', 'bias', 'gamma', 'beta')}
  mm_ref, mv_ref = lay.moving_mean.double(), lay.moving_var.double()
  mm_bound = 4 * U * mm_ref.abs()
  mv_bound = 4 * U * mv_ref
  g = _gen(B)

  def tol(ref):
    return 1e-5 * float(ref.detach().abs().max()) + 1e-30

  for step in range(2):
    x = torch.randn(B, 624, device=DEV, generator=g).requires_grad_(True)
    gy = torch.randn(B, 256, device=DEV, generator=g)
    lay.zero_grad(set_to_none=True)
    y = lay(x)
    y.backward(gy)
    mask = (y > 0).double()
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    x64 = x.detach().double().requires_grad_(True)
    z = x64 @ leaves['kernel'] + leaves['bias']
    mean, var = z.mean(0), ((z - z.mean(0)) ** 2).mean(0)
    y64 = ((z - mean) / torch.sqrt(var + EPS) * leaves['gamma'] + leaves['beta']) * mask
    y64.backward(gy.double())
    _within(y, y64.detach(), tol(y64), 'layer y')
    _within(x.grad, x64.grad, tol(x64.grad), 'layer x.grad')
    for k in ('kernel', 'gamma', 'beta'):
      _within(getattr(lay, k).grad, leaves[k].grad, tol(leaves[k].grad), 'layer %s.grad' % k)
    assert bool((lay.bias.grad == 0).all()), 'bias.grad must be identically zero under batch norm'
    mean, var = mean.detach(), var.detach()
    mm_ref = mm_ref * MOM + mean * (1 - MOM)
    mv_ref = mv_ref * MOM + var * (1 - MOM)
    mm_bound = mm_bound * MOM + 4 * U * mm_ref.abs() + 1e-6 * (1 - MOM) * (mean.abs() + var.sqrt())
    mv_bound = mv_bound * MOM + 4 * U * mv_ref + 1e-5 * (1 - MOM) * var
  assert routes == [fused, fused]
  _within(lay.moving_mean, mm_ref, mm_bound, 'layer moving_mean')
  _within(lay.moving_var, mv_ref, mv_bound, 'layer moving_var')
  lay.eval()
  x = torch.randn(B, 624, device=DEV, generator=g)
  with torch.no_grad():
    y = lay(x)
  assert routes == [fused, fused], 'eval must not compute batch statistics'
  mme, mve = lay.moving_mean.double(), lay.moving_var.double()
  z = x.double() @ params['kernel'] + params['bias']
  y64 = torch.relu((z - mme) / torch.sqrt(mve + EPS) * params['gamma'] + params['beta'])
  _within(y, y64, tol(y64), 'layer y eval')
