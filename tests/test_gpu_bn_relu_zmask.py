"""GPU: the dense layers' batch-norm + relu backward with the relu mask recomputed from z (er_bn_relu_bwd), which
does not read y.

  er_bn_relu_bwd  bit-identical to er_bias_bn_act_bwd (the same column sums; the mask from z instead of y) and
                  deterministic; gz, ggamma, gbeta within test_gpu_dense_bn.py's float64 bounds (column sums
                  4u (sqrt(B) ||terms||_2 + ||e||_2)).
  mask            bn_pre_act(z) > 0 is exactly y > 0 of the forward kernels, on z within a few ulps of the value where
                  the normalised input crosses 0, and on -0.0.
  layers          every batch-norm layer of a training DNN takes the new path (with and without dropout), and every
                  gradient is bit-identical to the y-mask kernels'.
"""
import math

import numpy as np
import pytest
import torch

from easyrec_b200 import kernels as K
from easyrec_b200 import layers as L

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
EPS = 1e-3


def _within(got, ref, bound, what):
  err = (got.double() - ref).abs()
  ratio = float((err / bound).max())
  assert ratio <= 1.0, '%s: error %.3g x bound (max abs err %.3g)' % (what, ratio, float(err.max()))


def _sum_bound(B, terms_sq, e_sq=0.0):
  return 4 * U * (math.sqrt(B) * terms_sq.sqrt() + e_sq ** 0.5) + 1e-30


def _layer_below(M, N, seed, pitch=0):
  """z, bias, gamma, beta and the fp32 batch statistics of z + bias"""
  g = torch.Generator(device=DEV).manual_seed(seed)
  zbuf = torch.randn(M, N + pitch, device=DEV, generator=g) * 2 + 0.5
  z = zbuf[:, :N]
  bias = torch.randn(N, device=DEV, generator=g) * 0.1
  gamma = 1 + 0.3 * torch.randn(N, device=DEV, generator=g)
  beta = 0.2 * torch.randn(N, device=DEV, generator=g)
  h = (z + bias).double()
  mean = h.mean(0)
  rstd = 1.0 / torch.sqrt(((h - mean) ** 2).mean(0) + EPS)
  return g, z, bias, gamma, beta, mean.float(), rstd.float()


def _ref_sums(gx, y, z, bias, mean, rstd, relu):
  """float64 sums, their bounds, and the float64 masked g / xhat / cond"""
  g64 = torch.where(y > 0, gx, torch.zeros_like(gx)).double() if relu else gx.double()
  m64, r64, b64 = mean.double(), rstd.double(), bias.double()
  z64 = z.double()
  xhat = ((z64 + b64) - m64) * r64
  cond = (z64.abs() + b64.abs() + m64.abs()) * r64
  M = gx.shape[0]
  sg, sgx = g64.sum(0), (g64 * xhat).sum(0)
  dsg = _sum_bound(M, g64.pow(2).sum(0))
  dsgx = _sum_bound(M, (g64 * xhat).pow(2).sum(0), (g64.abs() * cond).pow(2).sum(0))
  return sg, sgx, dsg, dsgx, g64, xhat, cond


# (batch, units): C2's tower widths, a ragged column tile, and a batch of one row chunk per lane
SHAPES = [(8192, 256), (8192, 128), (8192, 64), (1000, 200), (300, 72), (512, 32)]


@pytest.mark.parametrize('relu', [True, False])
@pytest.mark.parametrize('M,N', SHAPES)
def test_bn_relu_bwd_matches_y_mask_path_and_float64(M, N, relu):
  g, z, bias, gamma, beta, _, _ = _layer_below(M, N, 11 * M + N)
  z = z.contiguous()
  ws = K.dense_workspace(M, N, DEV)
  y, mean, rstd = K.bias_bn_act_fwd(z, bias, gamma, beta, torch.zeros(N, device=DEV), torch.ones(N, device=DEV),
                                    EPS, 0.99, True, relu, ws)
  gy = torch.randn(M, N, device=DEV, generator=g)
  old = K.bias_bn_act_bwd(z, bias, gamma, y, gy, mean, rstd, relu, ws)
  new = K.bn_relu_bwd(z, bias, gamma, beta, mean, rstd, gy, relu, ws)
  again = K.bn_relu_bwd(z, bias, gamma, beta, mean, rstd, gy, relu, ws)
  for a, b, c, name in zip(old, new, again, ('gz', 'gbias', 'ggamma', 'gbeta')):
    assert torch.equal(a, b), '%s: the mask from z must give the y-mask path bit for bit' % name
    assert torch.equal(b, c), '%s: er_bn_relu_bwd must be deterministic' % name
  assert bool((new[1] == 0).all())
  sg, sgx, dsg, dsgx, g64, xhat, cond = _ref_sums(gy, y, z, bias, mean, rstd, relu)
  ga64, r64 = gamma.double(), rstd.double()
  gz_ref = ga64 * r64 * (g64 - sg / M - xhat * sgx / M)
  gz_bound = (ga64.abs() * r64 * (3 * U * (g64.abs() + sg.abs() / M + xhat.abs() * sgx.abs() / M) + dsg / M +
                                  xhat.abs() * dsgx / M + sgx.abs() / M * (U * cond + 2 * U * xhat.abs())) +
              U * gz_ref.abs() + 1e-30)
  _within(new[0], gz_ref, gz_bound, 'gz')
  _within(new[2], sgx, dsgx, 'ggamma')
  _within(new[3], sg, dsg, 'gbeta')


def test_mask_from_z_is_exactly_y_positive_near_zero():
  """z a few ulps either side of where (z + b - m) r gamma + beta crosses 0, and z = -0.0 with zero statistics: the
  mask from z (er_bn_relu_bwd) is y > 0 of the forward kernels exactly, so gz is bit-identical to the y-mask kernels'
  (a flipped element would change its own gz and its column's sums)."""
  M, N = 128, 64
  g = torch.Generator(device=DEV).manual_seed(3)
  mean = torch.randn(N, device=DEV, generator=g)
  rstd = 0.5 + torch.rand(N, device=DEV, generator=g)
  gamma = 1 + 0.5 * torch.randn(N, device=DEV, generator=g)
  beta = 0.3 * torch.randn(N, device=DEV, generator=g)
  bias = 0.1 * torch.randn(N, device=DEV, generator=g)
  rstd[:4] = 1.0
  mean[:4] = beta[:4] = bias[:4] = 0.0
  m, r, ga, be, b = (t.cpu().numpy().astype(np.float64) for t in (mean, rstd, gamma, beta, bias))
  z0 = (m - b - be / (r * ga)).astype(np.float32)
  z = np.empty((M, N), np.float32)
  for i in range(M):
    z[i] = z0
    for _ in range(abs(i - M // 2) % 9):
      z[i] = np.nextafter(z[i], np.float32(np.inf) if i >= M // 2 else np.float32(-np.inf))
  z[:, :4] = -0.0            # columns with zero bias, mean and beta: the normalised value of -0.0 is a zero
  z[::2, :4] = 1.0
  z = torch.from_numpy(z).to(DEV)
  gy = torch.randn(M, N, device=DEV, generator=g)
  ws = K.dense_workspace(M, N, DEV)
  for y in (K.bn_act_apply(z, bias, gamma, beta, mean, rstd, True),                     # vector kernel
            K.bn_act_apply(z[:, :N - 1].contiguous(), bias, gamma, beta, mean, rstd, True)):  # scalar kernel
    n = y.shape[1]
    assert 0 < int((y > 0).sum()) < M * n, 'the inputs must straddle 0'
    assert torch.equal(y, K.bn_act_apply(z, bias, gamma, beta, mean, rstd, True)[:, :n])
  y = K.bn_act_apply(z, bias, gamma, beta, mean, rstd, True)
  old = K.bias_bn_act_bwd(z, bias, gamma, y, gy, mean, rstd, True, ws)
  new = K.bn_relu_bwd(z, bias, gamma, beta, mean, rstd, gy, True, ws)
  assert torch.equal(old[0], new[0]), 'mask from z differs from y > 0'


def _run_dnn(monkeypatch, z_mask, build, x):
  """one forward / backward of a fresh DNN; z_mask=False sends every layer to the y-mask kernels"""
  torch.manual_seed(0)
  calls = []
  with monkeypatch.context() as mp:
    real = K.bn_relu_bwd

    def spy(*a, **k):
      calls.append(1)
      return real(*a, **k) if z_mask else None
    mp.setattr(K, 'bn_relu_bwd', spy)
    mp.setattr(L.Dropout, '_next_seed', [0x5EED0001])   # the same dropout seeds in both runs
    net = build().to(DEV).train()
    xx = x.clone().requires_grad_(True)
    out = net(xx)
    (out * torch.linspace(-1, 1, out.shape[1], device=DEV)).sum().backward()
    torch.cuda.synchronize()
  return calls, [xx.grad] + [p.grad for p in net.parameters()]


@pytest.mark.parametrize('units,dropout', [([256, 128, 64], ()), ([128, 64], (0.3, 0.0)), ([64, 30, 16], ())])
def test_dense_layers_take_the_z_mask_path_bit_identically(monkeypatch, units, dropout):
  """Every batch-norm layer of a training DNN runs er_bn_relu_bwd (30 units: the y-mask kernels, units % 4 != 0), and
  all gradients are bit-identical to the y-mask kernels'."""
  x = torch.randn(2048, 96, device=DEV)
  u = L.Units(units)
  u.dropout = dropout
  calls, got = _run_dnn(monkeypatch, True, lambda: L.DNN(96, u), x)
  _, want = _run_dnn(monkeypatch, False, lambda: L.DNN(96, u), x)
  assert len(calls) == len(units)
  for a, b in zip(got, want):
    assert torch.equal(a, b)
