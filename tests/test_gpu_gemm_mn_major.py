"""GPU: er_gemm stages an MN-major operand (M / N contiguous: X and dY in dW, W[in, out] in a forward without
pre-split planes) into exactly the shared-memory bytes a K-major copy of it gives, so every layout of the same
matrices yields the same bits - split along K or not - and a split-K result is the same from run to run."""
import pytest
import torch

from easyrec_b200 import kernels as K

pytestmark = pytest.mark.gpu

# (M, N, K) of dW = X^T.dY: the six C2 tower layers at batch 8192, then a K that is not a multiple of 4, M and N that
# are not multiples of 4, below 128 (MMA widths 16 / 32 / 64) and above it, and an unsplit K
DW_SHAPES = [(624, 256, 8192), (256, 128, 8192), (128, 64, 8192), (81, 256, 8192), (256, 128, 8192), (128, 64, 8192),
             (81, 256, 8195), (200, 33, 8195), (130, 9, 8195), (40, 17, 5001), (97, 300, 2051), (129, 65, 300)]


def _ceil4(n):
  return (n + 3) // 4 * 4


def _pitched(src):
  """src [r, c] copied into a NaN-filled [r, ceil4(c)] buffer: the view er_gemm reads in place (pitch % 4 == 0)"""
  buf = torch.full((src.shape[0], _ceil4(src.shape[1])), float('nan'), device='cuda')
  buf[:, :src.shape[1]] = src
  return buf[:, :src.shape[1]]


def _layouts(a, b):
  """the logical a [M, K] and b [K, N] as (K-major, MN-major) views, each readable in place by er_gemm"""
  a_k, a_mn = _pitched(a), _pitched(a.t().contiguous()).t()
  b_k, b_mn = _pitched(b.t().contiguous()).t(), _pitched(b)
  for t, unit in ((a_k, 1), (a_mn, 0), (b_k, 0), (b_mn, 1)):   # unit: 1 if dim 1 is the contiguous one
    got, _, got_unit = K._gemm_operand(t, 't')
    assert got is t and got_unit == unit
  return (a_k, a_mn), (b_k, b_mn)


def _twice(fn):
  r0, r1 = fn(), fn()
  assert torch.equal(r0, r1), 'split-K result differs between two runs'
  return r0


@pytest.mark.parametrize('M,N,Kd', DW_SHAPES)
def test_dw_layouts_are_bit_identical(M, N, Kd):
  """K.gemm(x.t(), g) (both operands MN-major, as DenseLayer's dW) against the same matrices K-major and mixed"""
  g = torch.Generator(device='cuda').manual_seed(M * 7 + N * 3 + Kd)
  x = torch.randn(Kd, M, device='cuda', generator=g)
  dy = torch.randn(Kd, N, device='cuda', generator=g)
  (a_k, a_mn), (b_k, b_mn) = _layouts(x.t(), dy)
  ref = _twice(lambda: K.gemm(a_k, b_k))
  assert not bool(torch.isnan(ref).any())
  for a, b in ((a_mn, b_mn), (a_mn, b_k), (a_k, b_mn)):
    assert torch.equal(_twice(lambda: K.gemm(a, b)), ref)
  # the same with a bias, added after the slices are summed
  bias = torch.randn(N, device='cuda', generator=g)
  assert torch.equal(_twice(lambda: K.gemm(a_mn, b_mn, bias=bias)), _twice(lambda: K.gemm(a_k, b_k, bias=bias)))


@pytest.mark.parametrize('M,n_in,n_out', [(8192, 624, 256), (8192, 81, 256), (8192, 128, 64), (1000, 33, 17),
                                          (300, 81, 9), (5000, 8, 130)])
def test_forward_mn_major_weight_is_bit_identical(M, n_in, n_out):
  """the forward without planes reads W[in, out] MN-major; a K-major copy of W gives the same bits"""
  g = torch.Generator(device='cuda').manual_seed(M + n_in + n_out)
  x = _pitched(torch.randn(M, n_in, device='cuda', generator=g))
  w = torch.randn(n_in, n_out, device='cuda', generator=g) * 0.05
  bias = torch.randn(n_out, device='cuda', generator=g)
  (_, _), (w_k, w_mn) = _layouts(x, w)
  assert torch.equal(_twice(lambda: K.gemm(x, w_mn, bias=bias)), _twice(lambda: K.gemm(x, w_k, bias=bias)))

