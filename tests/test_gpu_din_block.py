"""GPU: the backbone DIN block.

  er_din_sigmoid_pool_fwd / _bwd against float64, through the C ABI: T and D on both sides of the 32-lane strides,
  lens 0 / 1 / T / random / NULL, scores up to +-80, outputs as views in NaN-filled buffers (everything outside must
  stay NaN), the accumulate_gkeys flag.  Bounds are first-order fp32 rounding, u = 2^-24, slack C = 2 (the conventions
  of test_gpu_interact_f64.py):
    probs    p = 1 / (1 + expf(-a)), a = fp32(scale * s): relative p * C * u * ((1 - p)(|a| + 4) + 2)  (the rounding
             of a, expf's 2 ulp, the add and the divide), absolute floor 2^-126 where expf overflows (p < FLT_MIN);
    out      sum_t p_t k_t in ascending t: C * T * u * sum_t |p_t k_t|;
    g_scores ((scale * p) * (1 - p)) * dp, dp a warp-strided dot: C * 4 * u * |g| + scale p (1 - p) * C * lanes(D) * u *
             sum |gout k|;
    g_keys   p * gout, one rounding: bit-exact; accumulating: within one ulp of prefill + the plain result.
  The golden fixture of layers/keras/din.py (tests/golden/reference_din_block.json) through the kernels.
  The config-built backbone DIN at C3 shape (batch 4096, two length-50 histories, 1M-row item table): logits within
  1e-4 of the same modules run as plain torch on the same looked-up rows and weights, and steps replayed from a CUDA
  graph equal to eager steps."""
import copy
import math

import numpy as np
import pytest
import torch

import host_doubles
from easyrec_b200 import _lib
from easyrec_b200 import interactions as I
from easyrec_b200 import workloads
from easyrec_b200.kernels import _p, _stream
from test_din_block_host import _golden, _score_fn
from test_gpu_interact_f64 import C, DEV, DIN_B, FLOOR, U, _acc_check, _din_inputs, _gen, _lanes, _ok, _out, \
    _untouched, _within

pytestmark = pytest.mark.gpu
SIG_FLOOR = 2.0 ** -126


def _fwd(scores, keys, lens, scale):
  B, T, D = keys.shape
  bp, probs = _out(B, T)
  bo, out = _out(B, D)
  _ok(_lib.load().er_din_sigmoid_pool_fwd(_p(scores), _p(keys), _p(lens), B, T, D, scale, _p(probs), _p(out),
                                          _stream()), 'er_din_sigmoid_pool_fwd')
  _untouched(bp, probs, 'din_sigmoid_pool_fwd probs')
  _untouched(bo, out, 'din_sigmoid_pool_fwd out')
  return probs, out


@pytest.mark.parametrize('T', [1, 31, 32, 33, 50, 200])
@pytest.mark.parametrize('D', [1, 5, 32, 33, 128])
def test_din_sigmoid_pool(T, D):
  lib, B = _lib.load(), DIN_B
  _, keys, scores, lens = _din_inputs(T, D, 10 * T + D + 1)
  scale = float(np.float32(1.0 / math.sqrt(D)))
  probs, out = _fwd(scores, keys, lens, scale)

  valid = torch.arange(T, device=DEV)[None, :] < lens[:, None].long()
  a = scale * scores.double()
  p_ref = torch.where(valid, torch.sigmoid(a), torch.zeros_like(a))
  p_bound = p_ref * C * U * ((1 - p_ref) * (a.abs() + 4) + 2) + SIG_FLOOR
  _within(probs, p_ref, p_bound, 'din_sigmoid_pool_fwd probs')
  assert bool((probs[~valid] == 0).all()), 'steps at or beyond the length must get p = 0 exactly'
  pk = probs.double()[:, :, None] * keys.double()
  _within(out, pk.sum(1), C * T * U * pk.abs().sum(1) + FLOOR, 'din_sigmoid_pool_fwd out')
  assert bool((out[lens == 0] == 0).all()), 'an empty history pools to 0'

  pa, oa = _fwd(scores, keys, torch.full_like(lens, T), scale)
  pn, on = _fwd(scores, keys, None, scale)
  assert torch.equal(pn, pa) and torch.equal(on, oa), 'lens = NULL must equal lens = T'

  gout = torch.randn(B, D, device=DEV, generator=_gen(T * D + 1))
  bs, gs = _out(B, T)
  bk, gk = _out(B, T, D)
  _ok(lib.er_din_sigmoid_pool_bwd(_p(probs), _p(keys), _p(gout), _p(lens), B, T, D, scale, _p(gs), _p(gk), 0,
                                  _stream()), 'er_din_sigmoid_pool_bwd')
  p64, k64, go64 = probs.double(), keys.double(), gout.double()[:, None, :]
  dp = (k64 * go64).sum(-1)
  dp_err = C * _lanes(D) * U * (k64 * go64).abs().sum(-1)
  w = scale * p64 * (1 - p64)
  gs_ref = torch.where(valid, w * dp, torch.zeros_like(dp))
  _within(gs, gs_ref, C * 4 * U * gs_ref.abs() + w * dp_err + FLOOR, 'din_sigmoid_pool_bwd g_scores')
  assert bool((gs[~valid] == 0).all()), 'masked steps must get no gradient'
  assert torch.equal(gk, probs[:, :, None] * gout[:, None, :])
  _untouched(bs, gs, 'din_sigmoid_pool_bwd g_scores')
  _untouched(bk, gk, 'din_sigmoid_pool_bwd g_keys')

  prefill = torch.randn(B, T, D, device=DEV, generator=_gen(6))
  bs2, gs2 = _out(B, T)
  bk2, gk2 = _out(B, T, D)
  gk2.copy_(prefill)
  _ok(lib.er_din_sigmoid_pool_bwd(_p(probs), _p(keys), _p(gout), _p(lens), B, T, D, scale, _p(gs2), _p(gk2), 1,
                                  _stream()), 'er_din_sigmoid_pool_bwd')
  assert torch.equal(gs2, gs)
  _acc_check(gk2, prefill, gk, 'din_sigmoid_pool_bwd accumulate_gkeys')
  _untouched(bk2, gk2, 'din_sigmoid_pool_bwd accumulate')


@pytest.mark.parametrize('name', sorted(_golden()))
def test_golden_through_the_kernels(name):
  """layers/keras/din.py DIN.call, executed from the reference's source, against din_attention /
  din_sigmoid_attention with the fixture's fixed attention function (the block's padding and slicing around them)."""
  from test_din_block_host import _block
  c = _golden()[name]
  mod, keys, query, lens = _block(c)
  fn = _score_fn(c, torch.float32)
  mod.mlp.fn = lambda x: fn(x.cpu()).to(DEV)   # the attention function on the host; concat and pool on the device
  y = mod((keys.to(DEV), lens.to(DEV), query.to(DEV)))
  np.testing.assert_allclose(y.cpu().numpy(), np.array(c['y']), rtol=1e-5, atol=1e-5)


def _c3_batches(n, B=4096, T=50):
  out = []
  for i in range(n):
    f, l = workloads.c3_batch(B, T, 777 + i, 1_000_000)
    out.append(({'sparse_fea': f['sparse_fea'].to(DEV), 'dense_fea': f['dense_fea'].to(DEV),
                 'seq_fea': {k: (a.to(DEV), b.to(DEV)) for k, (a, b) in f['seq_fea'].items()}}, l.to(DEV)))
  return out


def _to_cpu(v):
  if isinstance(v, torch.Tensor):
    return v.detach().cpu()
  if isinstance(v, (list, tuple)):
    return type(v)(_to_cpu(t) for t in v)
  return v


@pytest.mark.parametrize('normalizer', ['softmax', 'sigmoid'])
def test_c3_backbone_din_logits_match_plain_torch(normalizer, monkeypatch):
  from easyrec_b200.estimator import EasyRecEstimator
  torch.backends.cuda.matmul.allow_tf32 = False
  est = EasyRecEstimator(workloads.c3_backbone_config_text(normalizer=normalizer), device=DEV, seed=5,
                         use_cuda_graph=False, default_seq_len=50)
  (feats, labels), = _c3_batches(1)
  assert int(feats['seq_fea']['hist_items'][1].max()) == 50, 'at least one history of full length'
  model = est.model
  model.train()
  il = model.input_layer
  model.backbone.input_layer = None           # (the tables stay where they are: only the dense modules are copied)
  twin_backbone, twin_output = copy.deepcopy(model.backbone).cpu(), copy.deepcopy(model.output).cpu()
  model.backbone.input_layer = twin_backbone.input_layer = il
  with torch.no_grad():
    g = il.lookup(feats)
    logits = model.backbone(g)
    logits = model.output(logits)[:, 0]
  seq, seq_len, target, _ = g['seq']
  assert seq.shape == (4096, 50, 32) and target.shape == (4096, 32)
  host_doubles.install_all(monkeypatch.setattr)
  from test_din_block_host import _din_sigmoid_attention
  monkeypatch.setattr(I, 'din_sigmoid_attention', _din_sigmoid_attention)
  with torch.no_grad():
    ref = twin_output(twin_backbone({k: _to_cpu(v) for k, v in g.items()}))[:, 0]
  err = float((logits.cpu() - ref).abs().max())
  assert err <= 1e-4, 'logits differ from the torch restatement by %.3g' % err


def test_c3_backbone_din_graph_steps_equal_eager_steps():
  from easyrec_b200.estimator import EasyRecEstimator
  torch.backends.cuda.matmul.allow_tf32 = False
  batches = _c3_batches(3)
  runs = []
  for graph in (False, True):
    est = EasyRecEstimator(workloads.c3_backbone_config_text(normalizer='sigmoid'), device=DEV, seed=5,
                           use_cuda_graph=graph, default_seq_len=50)
    losses = [float(est.trainer.train_step(*batches[k % 3])[0]) for k in range(6)]
    assert (not graph) or est.trainer._graph is not None
    runs.append((losses, {d: a.weight.clone() for d, a in est.input_layer.arenas.items()},
                 {k: v.detach().clone() for k, v in est.model.state_dict().items()}))
    del est
    torch.cuda.empty_cache()
  # (the tolerance of test_gpu_models.py's graph test: two estimators built from one seed already differ in the last
  # bit of the first, eager, loss)
  np.testing.assert_allclose(runs[1][0], runs[0][0], rtol=0, atol=1e-6)
  for d in runs[0][1]:
    torch.testing.assert_close(runs[1][1][d], runs[0][1][d], rtol=0, atol=1e-5)
  for k in runs[0][2]:
    torch.testing.assert_close(runs[1][2][k], runs[0][2][k], rtol=0, atol=1e-5, msg=k)
