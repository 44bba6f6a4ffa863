"""Autograd wrappers of the fused interaction kernels (K4 DIN, K5 DCN cross, MMoE, DSSM pieces).

Each Function is one or two calls into liber_b200.so per direction; the matmuls between them run on the
library's own tensor-core GEMM (er_gemm).  Reference code restated by the kernels:
  DIN    layers/sequence_feature_layer.py:150-189, model/multi_tower_din.py:62-97
  cross  model/dcn.py:32-45
  MMoE   layers/mmoe.py:53-83
  DSSM   model/dssm.py:64-71, model/match_model.py:50-69,213-234
"""
import torch

from easyrec_b200 import _lib
from easyrec_b200 import kernels as K
from easyrec_b200.kernels import _p, _stream


class _Gram(torch.autograd.Function):
  """x [B, n, d] -> x x^T [B, n, n] (DLRM / DotInteraction pairwise dot products: model/dlrm.py:52-61,
  layers/keras/interaction.py:47-128) on the library's own batched small-matrix kernel."""

  @staticmethod
  def forward(ctx, x):
    x = _f32(x)
    B, n, d = x.shape
    out = torch.empty(B, n, n, dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().er_gram_fwd(x.data_ptr(), B, n, d, out.data_ptr(), K._stream()), 'er_gram_fwd')
    ctx.save_for_backward(x)
    return out

  @staticmethod
  def backward(ctx, g):
    (x,) = ctx.saved_tensors
    B, n, d = x.shape
    g = _f32(g)
    gx = torch.empty_like(x)
    _lib.check(_lib.load().er_gram_bwd(x.data_ptr(), g.data_ptr(), B, n, d, gx.data_ptr(), K._stream()), 'er_gram_bwd')
    return gx


def gram(x):
  return _Gram.apply(x)


class _MatmulNT(torch.autograd.Function):
  """u [B, H] x i [C, H] -> u i^T [B, C] (the in-batch similarity matrix of MatchModel, model/match_model.py:92-97)
  on the tensor-core GEMM; the transposes are read in place (er_gemm's NT / TN forms)."""

  @staticmethod
  def forward(ctx, u, i):
    u, i = K.gemm_ready(_f32(u)), K.gemm_ready(_f32(i))
    ctx.save_for_backward(u, i)
    return K.gemm(u, i.t())

  @staticmethod
  def backward(ctx, g):
    u, i = ctx.saved_tensors
    g = K.gemm_ready(_f32(g))
    return K.gemm(g, i), K.gemm(g.t(), u)


def matmul_nt(u, i):
  return _MatmulNT.apply(u, i)


def _f32(t):
  if not t.is_cuda or t.dtype != torch.float32:
    raise _lib.ErError('expected a CUDA fp32 tensor (no CPU fallback)')
  return t.contiguous()


class _DinConcat(torch.autograd.Function):
  """din_in[b,t,:] = [q, k, q-k, q*k]."""

  @staticmethod
  def forward(ctx, query, keys):
    query, keys = _f32(query), _f32(keys)
    B, T, D = keys.shape
    out = torch.empty(B, T, 4 * D, dtype=torch.float32, device=keys.device)
    _lib.check(_lib.load().er_din_concat_fwd(_p(query), _p(keys), B, T, D, _p(out), _stream()),
               'er_din_concat_fwd')
    ctx.save_for_backward(query, keys)
    return out

  @staticmethod
  def backward(ctx, g):
    query, keys = ctx.saved_tensors
    B, T, D = keys.shape
    gq = torch.empty_like(query)
    gk = torch.empty_like(keys)
    _lib.check(_lib.load().er_din_concat_bwd(_p(query), _p(keys), _p(_f32(g)), B, T, D, _p(gq), _p(gk), 0,
                                             _stream()), 'er_din_concat_bwd')
    return gq, gk


class _DinPool(torch.autograd.Function):
  """masked softmax over T + weighted sum of the keys."""

  @staticmethod
  def forward(ctx, scores, keys, lens):
    scores, keys = _f32(scores), _f32(keys)
    B, T, D = keys.shape
    probs = torch.empty(B, T, dtype=torch.float32, device=keys.device)
    out = torch.empty(B, D, dtype=torch.float32, device=keys.device)
    _lib.check(_lib.load().er_din_pool_fwd(_p(scores), _p(keys), _p(lens), B, T, D, _p(probs), _p(out),
                                           _stream()), 'er_din_pool_fwd')
    ctx.save_for_backward(probs, keys, lens)
    return out

  @staticmethod
  def backward(ctx, gout):
    probs, keys, lens = ctx.saved_tensors
    B, T, D = keys.shape
    gs = torch.empty_like(probs)
    gk = torch.empty_like(keys)
    _lib.check(_lib.load().er_din_pool_bwd(_p(probs), _p(keys), _p(_f32(gout)), _p(lens), B, T, D, _p(gs),
                                           _p(gk), 0, _stream()), 'er_din_pool_bwd')
    return gs, gk, None


def din_pool(scores, keys, lens):
  """softmax over the first lens[b] steps of scores [B,T] (the rest masked with -2^32 + 1), weighted sum of keys [B,T,D]
  -> [B,D]: the pooling half of target attention, and the `attention` sequence_combiner (layers/input_layer.py:323-339)."""
  return _DinPool.apply(scores, keys, lens)


def din_attention(query, keys, lens, attention_mlp):
  """query [B,D], keys [B,T,D], lens int32 [B]; attention_mlp maps [B,T,4D] -> [B,T,1].
  Returns [B,D] (the caller concatenates the query: multi_tower_din.py:96)."""
  din_in = _DinConcat.apply(query, keys)
  scores = attention_mlp(din_in).reshape(keys.shape[0], keys.shape[1])
  return _DinPool.apply(scores, keys, lens)


class _DinSigmoidPool(torch.autograd.Function):
  """p = sigmoid(scale * scores) on the first lens[b] steps, 0 beyond; weighted sum of the keys."""

  @staticmethod
  def forward(ctx, scores, keys, lens, scale):
    scores, keys = _f32(scores), _f32(keys)
    B, T, D = keys.shape
    probs = torch.empty(B, T, dtype=torch.float32, device=keys.device)
    out = torch.empty(B, D, dtype=torch.float32, device=keys.device)
    _lib.check(_lib.load().er_din_sigmoid_pool_fwd(_p(scores), _p(keys), _p(lens), B, T, D, scale, _p(probs), _p(out),
                                                   _stream()), 'er_din_sigmoid_pool_fwd')
    ctx.save_for_backward(probs, keys, lens)
    ctx.scale = scale
    return out

  @staticmethod
  def backward(ctx, gout):
    probs, keys, lens = ctx.saved_tensors
    B, T, D = keys.shape
    gs = torch.empty_like(probs)
    gk = torch.empty_like(keys)
    _lib.check(_lib.load().er_din_sigmoid_pool_bwd(_p(probs), _p(keys), _p(_f32(gout)), _p(lens), B, T, D, ctx.scale,
                                                   _p(gs), _p(gk), 0, _stream()), 'er_din_sigmoid_pool_bwd')
    return gs, gk, None, None


def din_sigmoid_pool(scores, keys, lens, scale):
  """sigmoid(scale * scores [B,T]) on the first lens[b] steps (0 beyond), weighted sum of keys [B,T,D] -> [B,D]: the
  'sigmoid' attention_normalizer of the keras DIN block (layers/keras/din.py:57-60, scale = 1/sqrt(D))."""
  return _DinSigmoidPool.apply(scores, keys, lens, float(scale))


def din_sigmoid_attention(query, keys, lens, attention_mlp, scale):
  """din_attention with the sigmoid normaliser: [q, k, q-k, q*k] -> attention_mlp -> din_sigmoid_pool."""
  din_in = _DinConcat.apply(query, keys)
  scores = attention_mlp(din_in).reshape(keys.shape[0], keys.shape[1])
  return din_sigmoid_pool(scores, keys, lens, scale)


class _Cross(torch.autograd.Function):
  """x_{l+1} = x0 * (x_l . w) + b + x_l."""

  @staticmethod
  def forward(ctx, x0, xl, w, b):
    x0, xl, w, b = _f32(x0), _f32(xl), _f32(w), _f32(b)
    B, D = xl.shape
    out = torch.empty_like(xl)
    xw = torch.empty(B, dtype=torch.float32, device=xl.device)
    _lib.check(_lib.load().er_cross_fwd(_p(x0), _p(xl), _p(w), _p(b), B, D, _p(out), _p(xw), _stream()),
               'er_cross_fwd')
    ctx.save_for_backward(x0, xl, w, xw)
    return out

  @staticmethod
  def backward(ctx, gout):
    x0, xl, w, xw = ctx.saved_tensors
    B, D = xl.shape
    lib = _lib.load()
    gx0, gxl = torch.empty_like(x0), torch.empty_like(xl)
    gw, gb = torch.empty_like(w), torch.empty_like(w)
    nbytes = lib.er_cross_workspace_bytes(B, D)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=xl.device)
    _lib.check(lib.er_cross_bwd(_p(x0), _p(xl), _p(w), _p(xw), _p(_f32(gout)), B, D, _p(gx0), _p(gxl), _p(gw),
                                _p(gb), 0, _p(ws), nbytes, _stream()), 'er_cross_bwd')
    return gx0, gxl, gw, gb


def cross_layer(x0, xl, w, b):
  return _Cross.apply(x0, xl, w, b)


class _MMoEMix(torch.autograd.Function):
  """out[b,:] = sum_e softmax(gate[b,:])[e] * experts[b,e,:]."""

  @staticmethod
  def forward(ctx, gate_logits, experts):
    gate_logits, experts = _f32(gate_logits), _f32(experts)
    B, E, H = experts.shape
    probs = torch.empty(B, E, dtype=torch.float32, device=experts.device)
    out = torch.empty(B, H, dtype=torch.float32, device=experts.device)
    _lib.check(_lib.load().er_mmoe_mix_fwd(_p(gate_logits), _p(experts), B, E, H, _p(probs), _p(out),
                                           _stream()), 'er_mmoe_mix_fwd')
    ctx.save_for_backward(probs, experts)
    return out

  @staticmethod
  def backward(ctx, gout):
    probs, experts = ctx.saved_tensors
    B, E, H = experts.shape
    gg = torch.empty_like(probs)
    ge = torch.empty_like(experts)
    _lib.check(_lib.load().er_mmoe_mix_bwd(_p(probs), _p(experts), _p(_f32(gout)), B, E, H, _p(gg), _p(ge), 0,
                                           _stream()), 'er_mmoe_mix_bwd')
    return gg, ge


def mmoe_mix(gate_logits, experts):
  return _MMoEMix.apply(gate_logits, experts)


class _L2Norm(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x):
    x = _f32(x)
    B, D = x.shape
    y = torch.empty_like(x)
    inv = torch.empty(B, dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().er_l2norm_fwd(_p(x), B, D, _p(y), _p(inv), _stream()), 'er_l2norm_fwd')
    ctx.save_for_backward(y, inv)
    return y

  @staticmethod
  def backward(ctx, gy):
    y, inv = ctx.saved_tensors
    gx = torch.empty_like(y)
    _lib.check(_lib.load().er_l2norm_bwd(_p(y), _p(inv), _p(_f32(gy)), y.shape[0], y.shape[1], _p(gx),
                                         _stream()), 'er_l2norm_bwd')
    return gx


def l2_normalize(x):
  return _L2Norm.apply(x)


class _InBatchSoftmaxCE(torch.autograd.Function):
  """match_model.py:213-234 (+ duplicate-item masking :50-69): returns (loss, p_bb)."""

  @staticmethod
  def forward(ctx, sim, item_ids, weights):
    sim = _f32(sim)
    B, N = sim.shape
    inv = 1.0 / B if weights is None else 1.0 / float(weights.sum().item())
    rows = torch.empty(B, dtype=torch.float32, device=sim.device)
    pd = torch.empty(B, dtype=torch.float32, device=sim.device)
    g = torch.empty_like(sim)
    _lib.check(_lib.load().er_inbatch_softmax_ce(_p(sim), _p(item_ids), _p(weights), B, N, inv, _p(rows), _p(pd),
                                                 _p(g), _stream()), 'er_inbatch_softmax_ce')
    ctx.save_for_backward(g)
    ctx.mark_non_differentiable(pd)
    return rows.sum(), pd

  @staticmethod
  def backward(ctx, gl, _gp):
    (g,) = ctx.saved_tensors
    return g * gl, None, None


def inbatch_softmax_ce(sim, item_ids=None, weights=None):
  return _InBatchSoftmaxCE.apply(sim, item_ids, weights)
