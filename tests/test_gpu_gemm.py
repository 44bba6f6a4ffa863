"""GPU: er_gemm (wgmma 3xTF32 dense-layer GEMM) against a float64 matmul of the same fp32 inputs.

Tolerance: |err| <= 4e-6 * sum_k |a_mk||b_kn| + 1e-30 per element -- 3xTF32 drops terms of relative size
2^-21; a plain TF32 product would miss this bound by two orders of magnitude, so the test also proves
the hi/lo split is live.  Covers the three operand layouts of a dense layer (forward, dX, dW), ragged
M/N/K, pitched views, bias, and the split-K path (deterministic: two runs are bit-identical).  N picks the MMA width
(16 / 32 / 64 / 128 columns): every width has a forward and a dW case.  Every shape here has M, N, K >= 8, so
kernels.gemm sends it to er_gemm and not to er_gemm_small.

The layout matrix calls er_gemm directly with explicit operand-major flags: all four (A, B) layouts at every MMA
width, ragged unsplit and split-K, with operands that are views of NaN-filled buffers (a padding element that reaches
the tensor cores unmasked turns the result into NaN).  Output placement covers pitched, odd-pitched and misaligned C
(the scalar-store branches of the epilogue and of the split-K reduction); pitch validation covers pitches shorter
than a row, which must be refused instead of reading the next row."""
import ctypes

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib

pytestmark = pytest.mark.gpu


def _check(a, b, got, bias=None):
  ref = a.double().cpu() @ b.double().cpu()
  if bias is not None:
    ref = ref + bias.double().cpu()
  bound = 4e-6 * (a.abs().double().cpu() @ b.abs().double().cpu()) + 1e-30
  err = (got.double().cpu() - ref).abs()
  worst = float((err / bound).max())
  assert worst <= 1.0, 'error %.3g x bound (max abs err %.3g)' % (worst, float(err.max()))
  return float(err.max())


@pytest.mark.parametrize('M,N,K', [(300, 256, 624), (128, 128, 32), (257, 100, 81), (8192, 64, 128), (1000, 16, 8),
                                   (8, 1024, 40), (300, 32, 624)])
def test_forward_layout(M, N, K):
  from easyrec_b200 import kernels as Kn
  assert min(M, N, K) >= 8   # smaller shapes take er_gemm_small
  g = torch.Generator(device='cuda').manual_seed(M + N + K)
  x = torch.randn(M, K, device='cuda', generator=g)
  w = torch.randn(K, N, device='cuda', generator=g) * 0.1
  bias = torch.randn(N, device='cuda', generator=g)
  _check(x, w, Kn.gemm(x, w))
  _check(x, w, Kn.gemm(x, w, bias=bias), bias)


@pytest.mark.parametrize('M,N,K', [(300, 624, 256), (513, 81, 64), (64, 40, 200)])
def test_dx_layout(M, N, K):
  from easyrec_b200 import kernels as Kn
  g = torch.Generator(device='cuda').manual_seed(1)
  gz = torch.randn(M, K, device='cuda', generator=g)
  w = torch.randn(N, K, device='cuda', generator=g)      # W[in=N, out=K]; dX = gz @ W^T
  _check(gz, w.t(), Kn.gemm(gz, w.t()))


@pytest.mark.parametrize('M,N,K', [(624, 256, 8192), (81, 256, 4100), (256, 128, 300), (64, 9, 1000), (64, 24, 1000),
                                   (96, 48, 3000)])
def test_dw_layout_and_split_k(M, N, K):
  from easyrec_b200 import kernels as Kn
  assert min(M, N, K) >= 8   # smaller shapes take er_gemm_small
  g = torch.Generator(device='cuda').manual_seed(2)
  pitch = (M + 3) // 4 * 4
  x = torch.randn(K, pitch, device='cuda', generator=g)[:, :M]     # pitched view, as the concat buffers are
  gz = torch.randn(K, N, device='cuda', generator=g)
  got = Kn.gemm(x.t(), gz)
  _check(x.t(), gz, got)
  assert torch.equal(got, Kn.gemm(x.t(), gz)), 'split-K reduction must be deterministic'


def test_hi_lo_split_is_live_and_matches_sgemm_level():
  from easyrec_b200 import kernels as Kn
  g = torch.Generator(device='cuda').manual_seed(3)
  x = torch.randn(2048, 512, device='cuda', generator=g)
  w = torch.randn(512, 256, device='cuda', generator=g)
  ref = (x.double() @ w.double())
  err = float((Kn.gemm(x, w).double() - ref).abs().max())
  torch.backends.cuda.matmul.allow_tf32 = False
  err_sgemm = float((torch.mm(x, w).double() - ref).abs().max())
  assert err < 20 * err_sgemm + 1e-5, (err, err_sgemm)
  assert err < 5e-4   # single-pass TF32 is ~2e-2 here; tensor-core fp32 accumulation truncates (K = 512 adds)


# ---- er_gemm called directly: explicit operand layouts, NaN padding, output placement, pitch validation ----

# (a_mn_major, b_mn_major): forward (X, W[in,out]), dX (dY, W), dW (X, dY), and A M-major with B K-major
LAYOUTS = [(0, 1), (0, 0), (1, 1), (1, 0)]


def _ceil4(n):
  return (n + 3) // 4 * 4


def _nan_view(rows, cols, g):
  """[rows, cols] of randn as a view of a NaN-filled buffer whose pitch is cols rounded up to a multiple of 4."""
  buf = torch.full((rows, _ceil4(cols)), float('nan'), device='cuda')
  buf[:, :cols] = torch.randn(rows, cols, device='cuda', generator=g)
  return buf[:, :cols]


def _er_gemm(a, a_mn, b, b_mn, M, N, K, bias=None, c_ptr=None, ldc=None):
  """er_gemm on operands stored as a = [M, K] (a_mn 0) or [K, M] (a_mn 1) and b = [N, K] (b_mn 0) or [K, N]
  (b_mn 1), each with unit inner stride and pitch stride(0).  Writes a new [M, N] tensor, or C at (c_ptr, ldc)."""
  lib = _lib.load()
  out = None
  if c_ptr is None:
    out = torch.empty(M, N, device='cuda')
    c_ptr, ldc = out.data_ptr(), N
  nbytes = lib.er_gemm_workspace_bytes(M, N, K)
  ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda') if nbytes else None
  _lib.check(lib.er_gemm(a.data_ptr(), a.stride(0), a_mn, b.data_ptr(), b.stride(0), b_mn,
                         None if bias is None else bias.data_ptr(), c_ptr, ldc, M, N, K,
                         None if ws is None else ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream),
             'er_gemm')
  return out


def _logical(a, a_mn, b, b_mn):
  """the [M, K] and [K, N] matrices that stored operands represent"""
  return (a.t() if a_mn else a), (b if b_mn else b.t())


@pytest.mark.parametrize('split', [False, True], ids=['ragged', 'splitk_bias'])
@pytest.mark.parametrize('a_mn,b_mn', LAYOUTS)
@pytest.mark.parametrize('N', [9, 16, 17, 32, 33, 64, 65, 128, 129, 300])
def test_layout_matrix_with_nan_padding(N, a_mn, b_mn, split):
  """Every MMA width x every operand layout, ragged in M, N and K, unsplit and split-K (with bias).  Both operands
  lie in NaN-filled buffers: the partial chunks at the K / M / N edges must be masked before the tensor cores."""
  M, K = (200, 2500) if split else (129, 37)
  assert (_lib.load().er_gemm_workspace_bytes(M, N, K) > 0) == split
  g = torch.Generator(device='cuda').manual_seed(16 * N + 4 * a_mn + 2 * b_mn + int(split))
  a = _nan_view(K, M, g) if a_mn else _nan_view(M, K, g)
  b = _nan_view(K, N, g) if b_mn else _nan_view(N, K, g)
  bias = torch.randn(N, device='cuda', generator=g) if split else None
  got = _er_gemm(a, a_mn, b, b_mn, M, N, K, bias)
  assert not bool(torch.isnan(got).any()), 'padding reached the tensor cores'
  A, B = _logical(a, a_mn, b, b_mn)
  _check(A, B, got, bias)


@pytest.mark.parametrize('split', [False, True], ids=['unsplit', 'splitk'])
@pytest.mark.parametrize('pad,col', [(0, 0), (4, 0), (1, 0), (0, 1), (4, 1), (1, 1)])
def test_output_into_pitched_and_misaligned_view(pad, col, split):
  """C at row 1 (and column `col`) of a NaN-filled buffer with ldc = N + pad: ldc % 4 != 0 or a base that is not
  16-byte aligned takes the scalar stores of the epilogue / of the split-K reduction.  The view must hold exactly
  the compact result, and nothing outside it may be written."""
  M, N, K = (200, 132, 2500) if split else (129, 132, 40)
  assert (_lib.load().er_gemm_workspace_bytes(M, N, K) > 0) == split
  g = torch.Generator(device='cuda').manual_seed(7 + pad + 8 * col)
  a, b = _nan_view(M, K, g), _nan_view(K, N, g)
  bias = torch.randn(N, device='cuda', generator=g)
  ref = _er_gemm(a, 0, b, 1, M, N, K, bias)
  ldc = N + pad
  off = ldc + col
  buf = torch.full(((M + 2) * ldc + 8,), float('nan'), device='cuda')
  _er_gemm(a, 0, b, 1, M, N, K, bias, c_ptr=buf.data_ptr() + 4 * off, ldc=ldc)
  view = buf.as_strided((M, N), (ldc, 1), off)
  assert torch.equal(view, ref)
  outside = torch.ones(buf.shape, dtype=torch.bool, device='cuda')
  outside.as_strided((M, N), (ldc, 1), off).fill_(False)
  assert bool(torch.isnan(buf[outside]).all()), 'er_gemm wrote outside C'


@pytest.mark.parametrize('entry', ['er_gemm', 'er_gemm_bn'])
@pytest.mark.parametrize('operand,mn_major', [('a', 0), ('a', 1), ('b', 0), ('b', 1)])
def test_pitch_shorter_than_row_is_refused(entry, operand, mn_major):
  """M = N = K = 81 with one operand given pitch 80 (a multiple of 4, but short of the row): reading it would take
  row r+1's first element as row r's last, so the call must fail.  The buffers hold (rows + 1) x pitch floats, so
  even an admitted call reads inside them.  The same call with pitch 84 is the control."""
  lib = _lib.load()
  M = N = K = 81
  g = torch.Generator(device='cuda').manual_seed(11)
  short = torch.randn((K + 1) * 80, device='cuda', generator=g)   # 81 rows of pitch 80, plus one
  a_mn = mn_major if operand == 'a' else 0
  b_mn = mn_major if operand == 'b' else 1
  a = _nan_view(K, M, g) if a_mn else _nan_view(M, K, g)   # pitch 84: the control's operands
  b = _nan_view(K, N, g) if b_mn else _nan_view(N, K, g)
  c = torch.empty(M, N, device='cuda')
  mean, rstd = torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
  ws = torch.zeros(lib.er_gemm_bn_workspace_bytes(M, N), dtype=torch.uint8, device='cuda')
  bn = _lib.ErBnStats(None, mean.data_ptr(), rstd.data_ptr(), None, None, 1e-3, 0.99)
  stream = torch.cuda.current_stream().cuda_stream

  def call(a_ptr, lda, b_ptr, ldb):
    if entry == 'er_gemm':
      return lib.er_gemm(a_ptr, lda, a_mn, b_ptr, ldb, b_mn, None, c.data_ptr(), N, M, N, K, None, 0, stream)
    return lib.er_gemm_bn(a_ptr, lda, a_mn, b_ptr, ldb, b_mn, c.data_ptr(), N, M, N, K, ctypes.byref(bn),
                          ws.data_ptr(), ws.numel(), stream)

  if operand == 'a':
    st = call(short.data_ptr(), 80, b.data_ptr(), b.stride(0))
  else:
    st = call(a.data_ptr(), a.stride(0), short.data_ptr(), 80)
  torch.cuda.synchronize()
  assert st == _lib.ER_ERR_INVALID_ARG and b'pitch smaller than row' in lib.er_last_error(), \
      '%s admitted a pitch of 80 for a row of 81 (status %d)' % (entry, st)
  assert a.stride(0) == b.stride(0) == 84
  _lib.check(call(a.data_ptr(), 84, b.data_ptr(), 84), entry)
  _check(*_logical(a, a_mn, b, b_mn), c)
