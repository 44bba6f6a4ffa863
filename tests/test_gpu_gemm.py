"""GPU: er_gemm (wgmma 3xTF32 dense-layer GEMM) against a float64 matmul of the same fp32 inputs.

Tolerance: |err| <= 4e-6 * sum_k |a_mk||b_kn| + 1e-30 per element -- 3xTF32 drops terms of relative size
2^-21; a plain TF32 product would miss this bound by two orders of magnitude, so the test also proves
the hi/lo split is live.  Covers the three operand layouts of a dense layer (forward, dX, dW), ragged
M/N/K, pitched views, bias, and the split-K path (deterministic: two runs are bit-identical).  N picks the MMA width
(16 / 32 / 64 / 128 columns): every width has a forward and a dW case."""
import numpy as np
import pytest
import torch

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
                                   (5, 1024, 40), (300, 32, 624)])
def test_forward_layout(M, N, K):
  from easyrec_b200 import kernels as Kn
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


@pytest.mark.parametrize('M,N,K', [(624, 256, 8192), (81, 256, 4100), (256, 128, 300), (64, 1, 1000), (64, 24, 1000),
                                   (96, 48, 3000)])
def test_dw_layout_and_split_k(M, N, K):
  from easyrec_b200 import kernels as Kn
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
