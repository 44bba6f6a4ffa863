"""GPU: fused dense epilogue (bias + batch-norm + relu, fwd/bwd) vs a plain PyTorch fp32 reference of
the same ops and vs the numpy oracle (oracle.dnn_forward/backward).  Tolerances: 2e-5 abs/rel (fp32
reductions over the batch in a different order)."""
import numpy as np
import pytest
import torch

from easyrec_b200 import kernels as K, layers as L
from oracle import oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def torch_ref_dnn(x, layers, training=True, masks=None):
  """plain torch: dense -> BN(batch stats, biased var, eps 1e-3) -> relu.
  masks (optional, one bool tensor per ReLU layer): the ReLU decision is taken from the mask instead of the
  sign of the pre-activation.  Batch norm couples every sample of a column, so ONE unit whose pre-activation
  lies within fp32 noise of zero and takes the other branch shifts that column's gradient sums and with
  them every row of the gradients by O(1/B): two correct fp32 implementations then differ by far more than
  rounding.  Evaluating the reference with the masks of the implementation under test removes that
  discrete ambiguity and leaves a well-posed comparison."""
  mi = 0
  for lay in layers:
    z = x @ lay['W'] + lay['b']
    if 'gamma' in lay:
      if training:
        mu = z.mean(0)
        var = ((z - mu)**2).mean(0)
      else:
        mu, var = lay['mean'], lay['var']
      z = (z - mu) / torch.sqrt(var + 1e-3) * lay['gamma'] + lay['beta']
    if lay['act']:
      if masks is not None:
        x = z * masks[mi].to(z.dtype)
        mi += 1
      else:
        x = torch.relu(z)
    else:
      x = z
  return x


@pytest.mark.parametrize('B,dims,last_plain', [(8192, [624, 256, 128, 64], False), (777, [81, 256, 33, 5], True),
                                               (64, [10, 7], False)])
def test_fused_dnn_matches_torch_and_oracle(B, dims, last_plain):
  torch.backends.cuda.matmul.allow_tf32 = False
  g = torch.Generator().manual_seed(3)
  dnn = L.DNN(dims[0], dims[1:], last_layer_no_activation=last_plain, last_layer_no_batch_norm=last_plain,
              generator=g).to(DEV)
  dnn.train()
  rng = np.random.default_rng(0)
  for lay in dnn.layers:  # non-trivial parameters
    with torch.no_grad():
      lay.bias.copy_(torch.from_numpy(rng.normal(0, 0.1, lay.n_out).astype(np.float32)))
      if lay.use_bn:
        lay.gamma.copy_(torch.from_numpy(rng.uniform(0.5, 1.5, lay.n_out).astype(np.float32)))
        lay.beta.copy_(torch.from_numpy(rng.normal(0, 0.2, lay.n_out).astype(np.float32)))
  x = torch.from_numpy(rng.normal(size=(B, dims[0])).astype(np.float32)).to(DEV).requires_grad_(True)
  gy = torch.from_numpy(rng.normal(size=(B, dims[-1])).astype(np.float32)).to(DEV)
  masks = []
  hooks = [lay.register_forward_hook(lambda m, i, o: masks.append((o > 0).detach())) for lay in dnn.layers if lay.relu]
  y = dnn(x)
  for h in hooks:
    h.remove()
  y.backward(gy)

  # ---- references: torch fp32 and float64, both with the ReLU decisions of the run above ----
  def make(dt):
    out = []
    for lay in dnn.layers:
      d = {'W': lay.kernel.detach().to(dt).clone().requires_grad_(True),
           'b': lay.bias.detach().to(dt).clone().requires_grad_(True), 'act': lay.relu}
      if lay.use_bn:
        d['gamma'] = lay.gamma.detach().to(dt).clone().requires_grad_(True)
        d['beta'] = lay.beta.detach().to(dt).clone().requires_grad_(True)
      out.append(d)
    xr = x.detach().to(dt).clone().requires_grad_(True)
    yr = torch_ref_dnn(xr, out, masks=masks)
    yr.backward(gy.to(dt))
    return out, xr, yr.detach()

  r32, x32, y32 = make(torch.float32)
  r64, x64, y64 = make(torch.float64)

  # Mine and torch's are two fp32 evaluations with different summation orders (wgmma 3xTF32 GEMM + tiled
  # Welford statistics vs cuBLAS SGEMM + torch reductions); both are measured against float64 and mine may
  # not be worse than torch's fp32 by more than a small factor (bulk: 99.9th percentile; tail: maximum).
  def no_worse(mine, t32, t64, what, factor=4.0):
    em, et = (mine.double() - t64).abs().flatten(), (t32.double() - t64).abs().flatten()
    qm = float(torch.quantile(em[:4000000], 0.999)) if em.numel() > 1000 else float(em.max())
    qt = float(torch.quantile(et[:4000000], 0.999)) if et.numel() > 1000 else float(et.max())
    scale = float(t64.abs().mean())
    assert qm <= factor * qt + 2e-6 * scale, '%s: p99.9 error %.3g vs torch fp32 %.3g (scale %.3g)' % (what, qm, qt, scale)
    assert float(em.max()) <= 10 * float(et.max()) + 1e-5 * scale, '%s: max error %.3g vs torch fp32 %.3g' % (
        what, float(em.max()), float(et.max()))

  no_worse(y.detach(), y32, y64, 'y')
  no_worse(x.grad, x32.grad, x64.grad, 'x.grad')
  for li, (lay, d32, d64) in enumerate(zip(dnn.layers, r32, r64)):
    no_worse(lay.kernel.grad, d32['W'].grad, d64['W'].grad, 'kernel grad %d' % li)
    if lay.use_bn:
      no_worse(lay.gamma.grad, d32['gamma'].grad, d64['gamma'].grad, 'gamma grad %d' % li)
      no_worse(lay.beta.grad, d32['beta'].grad, d64['beta'].grad, 'beta grad %d' % li)
      assert float(lay.bias.grad.abs().max()) == 0.0  # identically zero under batch norm
      assert float(d32['b'].grad.abs().max()) < 1e-3   # ... which torch evaluates as rounding noise
    else:
      no_worse(lay.bias.grad, d32['b'].grad, d64['b'].grad, 'bias grad %d' % li)
  # and in absolute terms: the fp32 parity gates of BASELINE.md (1e-4 on activations / logits)
  assert float((y.detach().double() - y64).abs().max()) < 1e-4
  # ---- numpy oracle (its own ReLU decisions: only the forward values, where a flip moves a value by < 1e-6) ----
  ol = []
  for lay in dnn.layers:
    d = {'W': lay.kernel.detach().cpu().numpy(), 'b': lay.bias.detach().cpu().numpy()}
    if lay.use_bn:
      d['gamma'] = lay.gamma.detach().cpu().numpy()
      d['beta'] = lay.beta.detach().cpu().numpy()
    ol.append(d)
  yo, cache = O.dnn_forward(x.detach().cpu().numpy(), ol, True, last_no_act=last_plain, last_no_bn=last_plain)
  np.testing.assert_allclose(y.detach().cpu().numpy(), yo, rtol=2e-4, atol=2e-5)
  gxo, _ = O.dnn_backward(gy.cpu().numpy(), ol, cache)
  # ReLU is discontinuous in its derivative: a pre-activation within fp32 noise of 0 may flip the mask in one
  # implementation and not the other, which changes that sample's whole input gradient.  Compare the samples
  # whose activations all stay clear of zero (the others are a ~1e-4 fraction).
  safe = np.ones(B, bool)
  for c in cache:
    if c['act']:
      safe &= (np.abs(c['h']) > 1e-4).all(axis=1)
  assert safe.mean() > 0.9
  np.testing.assert_allclose(x.grad.cpu().numpy()[safe], gxo[safe], rtol=5e-4, atol=2e-4)


def test_moving_statistics_and_inference_mode():
  torch.backends.cuda.matmul.allow_tf32 = False
  lay = L.DenseLayer(16, 8, use_bn=True, relu=True, generator=torch.Generator().manual_seed(1)).to(DEV)
  x = torch.randn(512, 16, device=DEV)
  lay.train()
  z = x @ lay.kernel + lay.bias
  mu, var = z.mean(0), ((z - z.mean(0))**2).mean(0)
  lay(x)
  assert torch.allclose(lay.moving_mean, 0.01 * mu, atol=1e-6)
  assert torch.allclose(lay.moving_var, 0.99 + 0.01 * var, atol=1e-6)
  lay.eval()
  y = lay(x)
  ref = torch.relu((z - lay.moving_mean) / torch.sqrt(lay.moving_var + 1e-3) * lay.gamma + lay.beta)
  assert torch.allclose(y, ref, atol=1e-5)


def test_single_unit_head_and_rowsum_block_match_float64():
  """the logit head (dense units=1) and the wide block (row sums + sum of squares) vs float64 numpy."""
  from easyrec_b200 import kernels as K
  rng = np.random.default_rng(9)
  for B, W in [(8192, 64), (777, 81), (5, 3)]:
    x = rng.normal(size=(B, W)).astype(np.float32)
    w = rng.normal(size=(W, 1)).astype(np.float32)
    b = rng.normal(size=(1,)).astype(np.float32)
    g = rng.normal(size=(B,)).astype(np.float32)
    tx, tw, tb, tg = (torch.from_numpy(a).to(DEV) for a in (x, w, b, g))
    y = K.dense1_fwd(tx, tw, tb).cpu().numpy()
    np.testing.assert_allclose(y[:, 0], x.astype(np.float64) @ w[:, 0].astype(np.float64) + b[0], rtol=1e-5, atol=1e-5)
    gx, gw, gb = K.dense1_bwd(tx, tw, tg)
    np.testing.assert_allclose(gx.cpu().numpy(), g[:, None] * w[:, 0][None, :], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(gw.cpu().numpy()[:, 0], x.astype(np.float64).T @ g.astype(np.float64), rtol=1e-4, atol=1e-4)
    assert abs(float(gb.item()) - float(g.astype(np.float64).sum())) < 1e-3
    gx2, gw2, gb2 = K.dense1_bwd(tx, tw, tg)
    assert torch.equal(gw, gw2) and torch.equal(gb, gb2)   # deterministic; workspace tickets self-reset
    rs, sq = K.rowsum_block_fwd(tx)
    np.testing.assert_allclose(rs.cpu().numpy(), x.astype(np.float64).sum(1), rtol=1e-5, atol=1e-5)
    assert abs(float(sq.item()) - float((x.astype(np.float64)**2).sum())) <= 2e-6 * float((x.astype(np.float64)**2).sum())
    coef = torch.tensor([0.25], device=DEV)
    gxr = K.rowsum_block_bwd(tx, tg, coef, 2.0).cpu().numpy()
    np.testing.assert_allclose(gxr, g[:, None] + 0.5 * x, rtol=1e-6, atol=1e-6)


def test_concat_cols_into_pitched_buffer_and_split_back():
  from easyrec_b200 import embedding as E, kernels as K
  g = torch.Generator(device=DEV).manual_seed(4)
  mats = [torch.randn(513, w, device=DEV, generator=g) for w in (1, 16, 64)]
  out = K.concat_cols(mats)
  assert out.shape == (513, 81) and out.stride(0) == 84 and out.data_ptr() % 16 == 0
  assert torch.equal(out, torch.cat(mats, 1))
  assert float(out.as_strided((513, 84), (84, 1))[:, 81:].abs().max()) == 0.0   # padding is zero
  back = K.split_cols(out.contiguous(), [1, 16, 64])
  assert all(torch.equal(a, b) for a, b in zip(back, mats))
  leaves = [m.clone().requires_grad_(True) for m in mats]
  y = E.concat_cols(leaves)
  gy = torch.randn(513, 81, device=DEV, generator=g)
  y.backward(gy)
  ref = torch.split(gy, [1, 16, 64], dim=1)
  assert all(torch.equal(l.grad, r) for l, r in zip(leaves, ref))


def test_dropout_kernel_is_bernoulli_keep_scaled_and_its_backward_reuses_the_mask():
  """er_dropout (layers/dnn.py:77-82 tf.nn.dropout): Bernoulli(keep) mask scaled by 1/keep, a function of (seed,
  device counter, index) - the backward recomputes it; a captured graph redraws when the counter advances."""
  from easyrec_b200 import layers as L
  torch.manual_seed(0)
  n, rate = 1 << 20, 0.3
  x = torch.randn(n, device=DEV) + 3.0
  ctr = torch.zeros(1, dtype=torch.int64, device=DEV)
  y = K.dropout(x, rate, 1234, ctr)
  kept = y != 0
  assert abs(float(kept.float().mean()) - 0.7) < 3e-3                       # 5 sigma of a 1M-sample Bernoulli(0.7)
  torch.testing.assert_close(y[kept], x[kept] / 0.7, rtol=1e-6, atol=0)
  assert torch.equal(K.dropout(x, rate, 1234, ctr), y)                      # same (seed, counter): same mask
  ctr.add_(1)
  y2 = K.dropout(x, rate, 1234, ctr)
  both = float(((y2 != 0) & kept).float().mean())
  assert abs(both - 0.49) < 5e-3                                            # independent of the previous step's mask
  assert abs(float(((K.dropout(x, rate, 99, ctr) != 0) & (y2 != 0)).float().mean()) - 0.49) < 5e-3   # and of other layers
  # no run structure: neighbouring elements are independent
  k = kept.float()
  assert abs(float((k[1:] * k[:-1]).mean()) - 0.49) < 5e-3
  # the layer: backward uses the forward's mask, then advances the counter
  drop = L.Dropout(0.5).to(DEV).train()
  xin = (torch.randn(4096, 64, device=DEV) + 2.0).requires_grad_(True)
  h = xin * 1.0
  out = drop(h)
  out.sum().backward()
  torch.testing.assert_close(xin.grad, (out != 0).float() * 2.0)
  assert int(drop.counter[0]) == 1
  drop.eval()
  assert drop(h) is h
