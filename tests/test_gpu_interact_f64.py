"""GPU: the feature-interaction kernels of csrc/interact2.cu and csrc/interact.cu against float64, called through the C
ABI so that every accumulate flag and every optional NULL pointer is reached.

  DIN        er_din_concat_fwd / _bwd, er_din_pool_fwd / _bwd     T and D on both sides of the 32-lane strides, T = 1,
             D = 1, lens 0 / 1 / T / random / NULL, score spreads of +-80
  DCN        er_cross_fwd / _bwd                                  xw_out NULL, accumulate_gx0, 2^24 + 1 rows (past
                                                                  65535 column-sum chunks of 256 rows)
  MMoE       er_mmoe_mix_fwd / _bwd                               E = 1 (exact), ties, +-50 spreads, accumulate
  DSSM       er_l2norm_fwd / _bwd, er_inbatch_softmax_ce          rows under the 1e-12 clamp, zero and denormal rows;
                                                                  item ids NULL / duplicated / all equal, zero weights
  DLRM       er_gram_fwd / _bwd                                   bit-exact against a float32 emulation
  FM         er_fm_fwd / _bwd, er_fm_block_fwd / _bwd             float4 and scalar paths bit for bit, every J = 1..8
                                                                  and dim/4 = 1..32, refusals
  wide       er_rowsum_block_fwd / _bwd
  logit      er_dense1_fwd / _bwd                                 every JW = 1..8, multi-CTA merge, width 256 refused
  loss       er_sigmoid_ce_fwd_bwd                                logits up to +-1e4, assign-and-scale loss

Every reference is a float64 restatement of the formula, evaluated on the fp32 tensors the kernel received (a backward
kernel's reference uses the forward kernel's outputs it was given).  Outputs are views inside NaN-filled buffers, and
every element outside a view (guards, row pitch) must still be NaN afterwards; pitched inputs carry NaN in their padding,
so a kernel that read it would return NaN.

Bounds are first-order fp32 rounding, u = 2^-24, times a slack C = 2:
  sum / dot   depth * u * sum|terms|, depth = the longest chain of additions in the kernel's order (a lane's
              sequential part + 5 shuffle levels for a warp-strided sum, chunk / warp / CTA stages for column sums).
  expf        2 ulp (4u relative) plus u |arg| from the rounding of the fp32 argument x - max;  logf / log1pf 1 ulp,
              rsqrtf 2 ulp (CUDA's documented bounds; the library is built without fast-math).
  softmax     p_t (r_t + sum_j r_j e_j / sum_j e_j + depth u + u) with r_t the expf bound above.
  products of these are propagated to first order; an absolute floor of 2^-140 covers denormal results, and the
  sigmoid's 2^-126 covers expf overflow below x = -88.7 (the true probability is under FLT_MIN there).
Bit-exact where the kernel's order is fixed and each operation rounds once: DIN concat, g_keys / g_experts / gx0 / gx of
dense1 (single products), the DLRM Gram matrices, FM forward and backward, the rowsum backward, clamped l2norm gradients.
Accumulating outputs must equal prefill + the non-accumulating result to within one ulp of the sum.

Worst error / bound measured on an H100 80GB HBM3 (400 W power limit), the 224 tests in about 10 s: accumulating
outputs 1.0 for cross gx0 (the kernel fuses g*xw into the add: exactly one ulp from prefill + plain), 0.98 MMoE, 0.97
DIN pool, 0.50 DIN concat; l2norm gx 0.51, y 0.15, inv_norm 0.11; DIN concat g_keys 0.50, g_query 0.31; MMoE out 0.49,
probs 0.42, g_gate 0.13; in-batch g_sim 0.47, probs_diag 0.33, loss_rows 0.25; sigmoid CE g_logits 0.41, probs 0.37,
loss 0.053; DIN pool probs 0.39, out 0.11, g_scores 0.10; cross out 0.31, gxl 0.25, xw 0.23, gw 0.012, gb 0.009;
FM block gx 0.19, y 0.13, sumsq 0.020; dense1 y 0.15, gw 0.085, gb 0.013; rowsum y 0.098, sumsq 0.007.
"""
import math

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib
from easyrec_b200.kernels import _p, _stream

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
C = 2.0
FLOOR = 2.0 ** -140
G = 64                   # guard elements before and after every output (256 bytes: keeps 16-byte alignment)
EPS12 = float(np.float32(1e-12))
KPAD = float(np.float32(-2.0 ** 32 + 1))
WORST = {}


def _lib_():
  return _lib.load()


def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


def _cdiv(a, b):
  return -(-a // b)


def _lanes(n):
  """chain length of a warp-strided sum of n terms: each lane's sequential part, then 5 xor-shuffle levels"""
  return _cdiv(n, 32) + 5


def _within(got, ref, bound, what):
  err = (got.double() - ref).abs()
  ratio = float((err / bound).max()) if err.numel() else 0.0
  WORST[what] = max(WORST.get(what, 0.0), ratio)
  assert ratio <= 1.0, '%s: error %.3g x bound (max abs err %.3g)' % (what, ratio, float(err.max()))


def _ok(rc, what):
  _lib.check(rc, what)


def _out(*shape, pitch=None, shift=0):
  """(buffer, view): a view of `shape` inside a NaN-filled buffer with G guard elements each side.  pitch gives the
  2-D view [rows, cols] a row pitch; shift moves its start by that many floats (shift=1: not 16-byte aligned)."""
  cols = shape[-1]
  rows = int(np.prod(shape[:-1])) if len(shape) > 1 else 1
  pitch = pitch or cols
  buf = torch.full((2 * G + rows * pitch + shift,), float('nan'), device=DEV)
  view = buf.as_strided((rows, cols), (pitch, 1), G + shift)
  if pitch == cols:
    view = view.view(*shape)
  return buf, view


def _untouched(buf, view, what):
  c = buf.clone()
  c.as_strided(view.shape, view.stride(), view.storage_offset()).fill_(0.0)
  assert int(torch.isnan(c).sum()) == c.numel() - view.numel(), '%s: wrote outside its output' % what


def _pitched_input(x, pad):
  """x [rows, cols] copied into a row-pitched view (pitch cols + pad) of a NaN-filled buffer"""
  _, v = _out(x.shape[0], x.shape[1], pitch=x.shape[1] + pad)
  v.copy_(x)
  return v


def _acc_check(got, prefill, plain, what):
  """an accumulating output equals prefill + the plain result to within one ulp of the sum (the kernel may fuse the
  product into the add, which rounds once instead of twice)"""
  want = prefill.double() + plain.double()
  mag = torch.maximum(want.abs(), plain.double().abs()).float()
  ulp = (torch.nextafter(mag, torch.full_like(mag, math.inf)) - mag).double()
  _within(got, want, ulp, what)


def _row_blocks(rows, width):
  step = max(1, (1 << 22) // max(1, width))
  return [slice(r, min(rows, r + step)) for r in range(0, rows, step)]


def _softmax_ref(v, depth):
  """float64 softmax over the last axis of v (-inf = masked) and the bound of the kernel's expf(v - max) / sum"""
  m = v.max(-1, keepdim=True).values
  e = torch.exp(v - m)
  s = e.sum(-1, keepdim=True)
  p = e / s
  r = torch.where(e > 0, C * (4 + (v - m).abs()) * U, torch.zeros_like(e))
  e_sum = (r * e).sum(-1, keepdim=True) / s + C * depth * U
  return p, p * (r + e_sum + C * U) + FLOOR


# ---------------------------------------------------------------------------------------------------------------------
# DIN
# ---------------------------------------------------------------------------------------------------------------------

DIN_B = 37      # 8 samples (warps) per CTA: the last CTA of the pool kernels is partial


def _din_inputs(T, D, seed):
  g = _gen(seed)
  B = DIN_B
  q = torch.randn(B, D, device=DEV, generator=g)
  keys = torch.randn(B, T, D, device=DEV, generator=g)
  wide = torch.rand(B, T, device=DEV, generator=g) * 160 - 80          # +-80: only stable after subtracting the max
  scores = torch.where((torch.arange(B, device=DEV) % 2 == 0)[:, None], torch.randn(B, T, device=DEV, generator=g) * 2,
                       wide)
  lens = torch.randint(0, T + 1, (B,), device=DEV, generator=g, dtype=torch.int32)
  lens[0], lens[1], lens[2], lens[3] = 0, 1, T, 0
  return q, keys, scores, lens


@pytest.mark.parametrize('T', [1, 31, 32, 33, 200, 1000])
@pytest.mark.parametrize('D', [1, 5, 32, 33, 128, 200])
def test_din_concat(T, D):
  lib, B = _lib_(), DIN_B
  q, keys, _, _ = _din_inputs(T, D, 10 * T + D)
  buf, out = _out(B, T, 4 * D)
  _ok(lib.er_din_concat_fwd(_p(q), _p(keys), B, T, D, _p(out), _stream()), 'er_din_concat_fwd')
  qe = q[:, None, :].expand(B, T, D)
  assert torch.equal(out, torch.cat([qe, keys, qe - keys, qe * keys], -1))
  _untouched(buf, out, 'din_concat_fwd')

  gin = torch.randn(B, T, 4 * D, device=DEV, generator=_gen(T + D))
  bq, gq = _out(B, D)
  bk, gk = _out(B, T, D)
  _ok(lib.er_din_concat_bwd(_p(q), _p(keys), _p(gin), B, T, D, _p(gq), _p(gk), 0, _stream()), 'er_din_concat_bwd')
  g0, g1, g2, g3 = gin.double().split(D, -1)
  k64, q64 = keys.double(), q.double()[:, None, :]
  _within(gq, (g0 + g2 + g3 * k64).sum(1),
          C * (T + 2) * U * (g0.abs() + g2.abs() + (g3 * k64).abs()).sum(1) + FLOOR, 'din_concat_bwd g_query')
  _within(gk, g1 - g2 + g3 * q64, C * 2 * U * (g1.abs() + g2.abs() + (g3 * q64).abs()) + FLOOR,
          'din_concat_bwd g_keys')
  _untouched(bq, gq, 'din_concat_bwd g_query')
  _untouched(bk, gk, 'din_concat_bwd g_keys')

  prefill = torch.randn(B, T, D, device=DEV, generator=_gen(7))
  bq2, gq2 = _out(B, D)
  bk2, gk2 = _out(B, T, D)
  gk2.copy_(prefill)
  _ok(lib.er_din_concat_bwd(_p(q), _p(keys), _p(gin), B, T, D, _p(gq2), _p(gk2), 1, _stream()), 'er_din_concat_bwd')
  assert torch.equal(gq2, gq)
  _acc_check(gk2, prefill, gk, 'din_concat_bwd accumulate_gkeys')
  _untouched(bk2, gk2, 'din_concat_bwd accumulate')


def _din_pool_fwd(scores, keys, lens):
  lib = _lib_()
  B, T, D = keys.shape
  bp, probs = _out(B, T)
  bo, out = _out(B, D)
  _ok(lib.er_din_pool_fwd(_p(scores), _p(keys), _p(lens), B, T, D, _p(probs), _p(out), _stream()), 'er_din_pool_fwd')
  _untouched(bp, probs, 'din_pool_fwd probs')
  _untouched(bo, out, 'din_pool_fwd out')
  return probs, out


@pytest.mark.parametrize('T', [1, 31, 32, 33, 200, 1000])
@pytest.mark.parametrize('D', [1, 5, 32, 33, 128, 200])
def test_din_pool(T, D):
  lib, B = _lib_(), DIN_B
  _, keys, scores, lens = _din_inputs(T, D, 10 * T + D)
  probs, out = _din_pool_fwd(scores, keys, lens)

  valid = torch.arange(T, device=DEV)[None, :] < lens[:, None].long()
  s64 = torch.where(valid, scores.double(), torch.full_like(scores, KPAD, dtype=torch.float64))
  p_ref, p_bound = _softmax_ref(s64, _lanes(T))
  _within(probs, p_ref, p_bound, 'din_pool_fwd probs')
  empty = lens == 0
  assert bool((probs[~empty][~valid[~empty]] == 0).all()), 'masked steps of a non-empty history must get p = 0'
  uniform = torch.ones((), device=DEV) / T
  assert bool((probs[empty] == uniform).all()), 'an empty history must get p = fp32(1/T) at every step'
  pk = probs.double()[:, :, None] * keys.double()
  _within(out, pk.sum(1), C * T * U * pk.abs().sum(1) + FLOOR, 'din_pool_fwd out')

  full = torch.full_like(lens, T)
  pa, oa = _din_pool_fwd(scores, keys, full)
  pn, on = _din_pool_fwd(scores, keys, None)
  assert torch.equal(pn, pa) and torch.equal(on, oa), 'lens = NULL must equal lens = T'

  gout = torch.randn(B, D, device=DEV, generator=_gen(T * D))
  bs, gs = _out(B, T)
  bk, gk = _out(B, T, D)
  _ok(lib.er_din_pool_bwd(_p(probs), _p(keys), _p(gout), _p(lens), B, T, D, _p(gs), _p(gk), 0, _stream()),
      'er_din_pool_bwd')
  p64, k64, go64 = probs.double(), keys.double(), gout.double()[:, None, :]
  dp = (k64 * go64).sum(-1)
  dp_err = C * _lanes(D) * U * (k64 * go64).abs().sum(-1)
  dot = (p64 * dp).sum(1, keepdim=True)
  dot_err = (p64 * dp_err).sum(1, keepdim=True) + C * T * U * (p64 * dp).abs().sum(1, keepdim=True)
  gs_ref = torch.where(valid, p64 * (dp - dot), torch.zeros_like(dp))
  _within(gs, gs_ref, p64 * (dp_err + dot_err + C * U * (dp - dot).abs()) + C * U * gs_ref.abs() + FLOOR,
          'din_pool_bwd g_scores')
  assert bool((gs[~valid] == 0).all()), 'masked steps must get no gradient'
  assert torch.equal(gk, probs[:, :, None] * gout[:, None, :])
  _untouched(bs, gs, 'din_pool_bwd g_scores')
  _untouched(bk, gk, 'din_pool_bwd g_keys')

  prefill = torch.randn(B, T, D, device=DEV, generator=_gen(5))
  bs2, gs2 = _out(B, T)
  bk2, gk2 = _out(B, T, D)
  gk2.copy_(prefill)
  _ok(lib.er_din_pool_bwd(_p(probs), _p(keys), _p(gout), _p(lens), B, T, D, _p(gs2), _p(gk2), 1, _stream()),
      'er_din_pool_bwd')
  assert torch.equal(gs2, gs)
  _acc_check(gk2, prefill, gk, 'din_pool_bwd accumulate_gkeys')
  _untouched(bk2, gk2, 'din_pool_bwd accumulate')


# ---------------------------------------------------------------------------------------------------------------------
# DCN cross
# ---------------------------------------------------------------------------------------------------------------------

def _cross_run(x0, xl, w, b, gout, accumulate_prefill=None, want_xw=True):
  lib = _lib_()
  B, D = x0.shape
  outs = {}
  bo, out = _out(B, D)
  bx, xw = _out(B)
  _ok(lib.er_cross_fwd(_p(x0), _p(xl), _p(w), _p(b), B, D, _p(out), _p(xw) if want_xw else None, _stream()),
      'er_cross_fwd')
  _untouched(bo, out, 'cross_fwd out')
  outs['out'], outs['xw'] = out, xw
  if not want_xw:
    assert bool(torch.isnan(xw).all()), 'xw_out = NULL: nothing may be written'
    return outs
  nbytes = lib.er_cross_workspace_bytes(B, D)
  ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
  bufs = [_out(B, D), _out(B, D), _out(D), _out(D)]
  gx0, gxl, gw, gb = [v for _, v in bufs]
  if accumulate_prefill is not None:
    gx0.copy_(accumulate_prefill)
  _ok(lib.er_cross_bwd(_p(x0), _p(xl), _p(w), _p(xw), _p(gout), B, D, _p(gx0), _p(gxl), _p(gw), _p(gb),
                       0 if accumulate_prefill is None else 1, _p(ws), nbytes, _stream()), 'er_cross_bwd')
  for (buf, v), name in zip(bufs, ('gx0', 'gxl', 'gw', 'gb')):
    _untouched(buf, v, 'cross_bwd ' + name)
  outs.update(gx0=gx0, gxl=gxl, gw=gw, gb=gb)
  return outs


def _cross_check(x0, xl, w, b, gout, o):
  B, D = x0.shape
  w64, b64 = w.double(), b.double()
  rows_per_chunk = 256 * _cdiv(_cdiv(B, 256), 65535)     # the kernel's column-sum chunks
  depth = rows_per_chunk // 8 + 8 + _cdiv(B, rows_per_chunk)
  z = torch.zeros(D, dtype=torch.float64, device=DEV)
  gw_ref, gw_abs, gw_err, gb_ref, gb_abs = z.clone(), z.clone(), z.clone(), z.clone(), z.clone()
  for s in _row_blocks(B, D):
    x0b, xlb, gob = x0[s].double(), xl[s].double(), gout[s].double()
    xw_ref = (xlb * w64).sum(1, keepdim=True)
    xw_err = C * _lanes(D) * U * (xlb * w64).abs().sum(1, keepdim=True)
    _within(o['xw'][s], xw_ref[:, 0], xw_err[:, 0] + FLOOR, 'cross_fwd xw')
    o_ref = x0b * xw_ref + b64 + xlb
    _within(o['out'][s], o_ref,
            x0b.abs() * xw_err + C * 3 * U * ((x0b * xw_ref).abs() + b64.abs() + xlb.abs()) + FLOOR, 'cross_fwd out')
    assert torch.equal(o['gx0'][s], gout[s] * o['xw'][s][:, None])
    s_ref = (gob * x0b).sum(1, keepdim=True)
    s_err = C * _lanes(D) * U * (gob * x0b).abs().sum(1, keepdim=True)
    _within(o['gxl'][s], gob + w64 * s_ref,
            w64.abs() * s_err + C * 2 * U * (gob.abs() + (w64 * s_ref).abs()) + FLOOR, 'cross_bwd gxl')
    t = xlb * s_ref
    gw_ref += t.sum(0)
    gw_abs += t.abs().sum(0)
    gw_err += (xlb.abs() * s_err).sum(0)
    gb_ref += gob.sum(0)
    gb_abs += gob.abs().sum(0)
  _within(o['gw'], gw_ref, gw_err + C * depth * U * gw_abs + FLOOR, 'cross_bwd gw')
  _within(o['gb'], gb_ref, C * depth * U * gb_abs + FLOOR, 'cross_bwd gb')


@pytest.mark.parametrize('D', [1, 31, 33, 624, 1280])
@pytest.mark.parametrize('B', [1, 255, 256, 257, 65537])
def test_cross(B, D):
  g = _gen(B + D)
  x0, xl, gout = (torch.randn(B, D, device=DEV, generator=g) for _ in range(3))
  w = torch.randn(D, device=DEV, generator=g) / math.sqrt(D)
  b = torch.randn(D, device=DEV, generator=g) * 0.1
  o = _cross_run(x0, xl, w, b, gout)
  _cross_check(x0, xl, w, b, gout, o)

  n = _cross_run(x0, xl, w, b, gout, want_xw=False)
  assert torch.equal(n['out'], o['out']), 'xw_out = NULL must not change out'

  prefill = torch.randn(B, D, device=DEV, generator=g)
  a = _cross_run(x0, xl, w, b, gout, accumulate_prefill=prefill)
  for k in ('out', 'xw', 'gxl', 'gw', 'gb'):
    assert torch.equal(a[k], o[k]), 'accumulate_gx0 changed ' + k
  _acc_check(a['gx0'], prefill, o['gx0'], 'cross_bwd accumulate_gx0')


def test_cross_bwd_past_65535_column_chunks():
  """2^24 + 1 rows: 65537 chunks of 256 rows, more than a grid's y dimension holds.  Positive inputs, so the column
  sums are not cancellations and their relative bound says something."""
  B, D = (1 << 24) + 1, 4
  g = _gen(24)
  x0, xl, gout = (torch.rand(B, D, device=DEV, generator=g) for _ in range(3))
  w = torch.rand(D, device=DEV, generator=g)
  b = torch.rand(D, device=DEV, generator=g)
  o = _cross_run(x0, xl, w, b, gout)
  _cross_check(x0, xl, w, b, gout, o)


# ---------------------------------------------------------------------------------------------------------------------
# MMoE
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('E', [1, 2, 31, 32, 33, 64])
@pytest.mark.parametrize('H', [1, 33, 256])
def test_mmoe_mix(E, H):
  lib, B = _lib_(), 1003
  g = _gen(E * 1000 + H)
  kind = torch.arange(B, device=DEV)[:, None] % 3
  gate = torch.where(kind == 0, torch.round(torch.randn(B, E, device=DEV, generator=g)),   # many ties
                     torch.where(kind == 1, torch.rand(B, E, device=DEV, generator=g) * 100 - 50,
                                 torch.randn(B, E, device=DEV, generator=g) * 3))
  gate[1] = 7.0                                                                              # one row all tied
  experts = torch.randn(B, E, H, device=DEV, generator=g)
  bp, probs = _out(B, E)
  bo, out = _out(B, H)
  _ok(lib.er_mmoe_mix_fwd(_p(gate), _p(experts), B, E, H, _p(probs), _p(out), _stream()), 'er_mmoe_mix_fwd')
  _untouched(bp, probs, 'mmoe_mix_fwd probs')
  _untouched(bo, out, 'mmoe_mix_fwd out')
  p_ref, p_bound = _softmax_ref(gate.double(), _lanes(E))
  _within(probs, p_ref, p_bound, 'mmoe_mix_fwd probs')
  pe = probs.double()[:, :, None] * experts.double()
  _within(out, pe.sum(1), C * E * U * pe.abs().sum(1) + FLOOR, 'mmoe_mix_fwd out')

  gout = torch.randn(B, H, device=DEV, generator=g)
  bg, gg = _out(B, E)
  be, ge = _out(B, E, H)
  _ok(lib.er_mmoe_mix_bwd(_p(probs), _p(experts), _p(gout), B, E, H, _p(gg), _p(ge), 0, _stream()),
      'er_mmoe_mix_bwd')
  _untouched(bg, gg, 'mmoe_mix_bwd g_gate')
  _untouched(be, ge, 'mmoe_mix_bwd g_experts')
  p64, go64 = probs.double(), gout.double()[:, None, :]
  dp = (experts.double() * go64).sum(-1)
  dp_err = C * _lanes(H) * U * (experts.double() * go64).abs().sum(-1)
  dot = (p64 * dp).sum(1, keepdim=True)
  dot_err = (p64 * dp_err).sum(1, keepdim=True) + C * E * U * (p64 * dp).abs().sum(1, keepdim=True)
  gg_ref = p64 * (dp - dot)
  _within(gg, gg_ref, p64 * (dp_err + dot_err + C * U * (dp - dot).abs()) + C * U * gg_ref.abs() + FLOOR,
          'mmoe_mix_bwd g_gate')
  assert torch.equal(ge, probs[:, :, None] * gout[:, None, :])
  if E == 1:
    assert bool((probs == 1).all()) and bool((gg == 0).all()), 'one expert: p = 1 and no gate gradient, exactly'

  prefill = torch.randn(B, E, H, device=DEV, generator=g)
  bg2, gg2 = _out(B, E)
  be2, ge2 = _out(B, E, H)
  ge2.copy_(prefill)
  _ok(lib.er_mmoe_mix_bwd(_p(probs), _p(experts), _p(gout), B, E, H, _p(gg2), _p(ge2), 1, _stream()),
      'er_mmoe_mix_bwd')
  assert torch.equal(gg2, gg)
  _acc_check(ge2, prefill, ge, 'mmoe_mix_bwd accumulate_gexperts')
  _untouched(be2, ge2, 'mmoe_mix_bwd accumulate')


# ---------------------------------------------------------------------------------------------------------------------
# DSSM: l2 normalisation and in-batch softmax cross entropy
# ---------------------------------------------------------------------------------------------------------------------

def _l2_rows(D, seed):
  """rows: 0, norm 1e-7, norm 9e-7 (both under the clamp, sum x^2 = 1e-14 and 8.1e-13), denormals, norm 2e-6 (just
  above), norm 1e3, then N(0, 1) rows"""
  rng = np.random.default_rng(seed)
  rows = [np.zeros(D)]
  for norm in (1e-7, 9e-7, None, 2e-6, 1e3):
    v = rng.standard_normal(D)
    rows.append(v * 1e-40 if norm is None else v / np.linalg.norm(v) * norm)
  rows += list(rng.standard_normal((37, D)))
  x = np.asarray(rows).astype(np.float32)
  assert np.all(np.abs(x[3]) < np.finfo(np.float32).tiny) and np.any(x[3] != 0)
  return torch.from_numpy(x).to(DEV)


@pytest.mark.parametrize('D', [1, 16, 33, 128, 300])
def test_l2norm(D):
  lib = _lib_()
  x = _l2_rows(D, D)
  B = x.shape[0]
  by, y = _out(B, D)
  bi, inv = _out(B)
  _ok(lib.er_l2norm_fwd(_p(x), B, D, _p(y), _p(inv), _stream()), 'er_l2norm_fwd')
  _untouched(by, y, 'l2norm_fwd y')
  _untouched(bi, inv, 'l2norm_fwd inv_norm')
  x64 = x.double()
  ss = (x64 * x64).sum(1)
  assert bool(((ss / EPS12 - 1).abs() > 1e-4).all()), 'keep clear of the ulp-wide band at the clamp'
  clamped = ss < EPS12
  assert clamped[:5].tolist() == [True, True, True, True, False]
  inv_ref = 1.0 / torch.sqrt(torch.clamp(ss, min=EPS12))
  inv_rel = 0.5 * C * _lanes(D) * U + C * 4 * U     # the fp32 sum of squares, then rsqrtf's 2 ulp
  _within(inv, inv_ref, inv_ref * inv_rel, 'l2norm_fwd inv_norm')
  assert bool((inv[clamped] == 1e6).all()), 'a clamped row stores inv_norm = 1/sqrt(1e-12f) rounded to fp32'
  y_ref = x64 * inv_ref[:, None]
  _within(y, y_ref, y_ref.abs() * (inv_rel + C * U) + FLOOR, 'l2norm_fwd y')

  gy = torch.randn(B, D, device=DEV, generator=_gen(D))
  bg, gx = _out(B, D)
  _ok(lib.er_l2norm_bwd(_p(y), _p(inv), _p(gy), B, D, _p(gx), _stream()), 'er_l2norm_bwd')
  _untouched(bg, gx, 'l2norm_bwd gx')
  # TF's gradient, the branch chosen by the float64 sum of squares of x
  y64, i64, g64 = y.double(), inv.double()[:, None], gy.double()
  dot = (g64 * y64).sum(1, keepdim=True)
  dot_err = C * _lanes(D) * U * (g64 * y64).abs().sum(1, keepdim=True)
  full = i64 * (g64 - y64 * dot)
  full_bound = i64 * (C * 2 * U * (g64.abs() + (y64 * dot).abs()) + y64.abs() * dot_err) + C * U * full.abs()
  below = g64 / math.sqrt(EPS12)
  ref = torch.where(clamped[:, None], below, full)
  bound = torch.where(clamped[:, None], C * U * below.abs(), full_bound) + FLOOR
  _within(gx, ref, bound, 'l2norm_bwd gx')
  assert torch.equal(gx[clamped], gy[clamped] * inv[clamped][:, None])


INB_B = [1, 33, 512, 4096]


@pytest.mark.parametrize('B', INB_B)
@pytest.mark.parametrize('cols', ['B', 'B+1', '3B'])
@pytest.mark.parametrize('variant', ['plain', 'dup_ids_weights', 'ids_all_equal'])
def test_inbatch_softmax_ce(B, cols, variant):
  lib = _lib_()
  N = {'B': B, 'B+1': B + 1, '3B': 3 * B}[cols]
  g = _gen(B * 7 + N)
  wide = torch.rand(B, N, device=DEV, generator=g) * 160 - 80
  sim = torch.where((torch.arange(B, device=DEV) % 2 == 0)[:, None], torch.randn(B, N, device=DEV, generator=g) * 3,
                    wide)
  ids = weights = None
  if variant == 'dup_ids_weights':
    ids = torch.randint(0, max(1, B // 8), (B,), device=DEV, generator=g)
    weights = torch.rand(B, device=DEV, generator=g)
    weights[::3] = 0.0
  elif variant == 'ids_all_equal':
    ids = torch.full((B,), 7, dtype=torch.int64, device=DEV)
  wsum = float(weights.double().sum()) if weights is not None else float(B)
  inv_wsum = float(np.float32(1.0 / wsum)) if wsum > 0 else 0.0

  bl, loss = _out(B)
  bp, pd = _out(B)
  bg, gsim = _out(B, N)
  _ok(lib.er_inbatch_softmax_ce(_p(sim), _p(ids), _p(weights), B, N, inv_wsum, _p(loss), _p(pd), _p(gsim),
                                _stream()), 'er_inbatch_softmax_ce')
  for buf, v, name in ((bl, loss, 'loss_rows'), (bp, pd, 'probs_diag'), (bg, gsim, 'g_sim')):
    _untouched(buf, v, 'inbatch_softmax_ce ' + name)

  v = sim.double()
  eye = torch.zeros(B, N, dtype=torch.bool, device=DEV)
  eye[:, :B] = torch.eye(B, dtype=torch.bool, device=DEV)
  masked = torch.zeros_like(eye)
  if ids is not None:      # duplicates of the row's item among the first B columns (never the diagonal, never j >= B)
    masked[:, :B] = (ids[None, :] == ids[:, None]) & ~eye[:, :B]
  v = torch.where(masked, torch.full_like(v, -math.inf), v)
  p, p_bound = _softmax_ref(v, _lanes(N))
  rows = torch.arange(B, device=DEV)
  pbb, pbb_bound = p[rows, rows], p_bound[rows, rows]
  w = weights.double() if weights is not None else torch.ones(B, dtype=torch.float64, device=DEV)
  wi = w * inv_wsum
  lg = torch.log(pbb + EPS12)
  loss_ref = -lg * wi
  _within(pd, pbb, pbb_bound, 'inbatch_softmax_ce probs_diag')
  _within(loss, loss_ref, wi.abs() * ((pbb_bound + C * U * (pbb + EPS12)) / (pbb + EPS12) + C * 2 * U * lg.abs()) +
          C * 2 * U * loss_ref.abs() + FLOOR, 'inbatch_softmax_ce loss_rows')
  coef = -wi * pbb / (pbb + EPS12)
  # the kernel forms -w * inv_wsum * p_bb before dividing by p_bb + 1e-12: for p_bb ~ 1e-40 that product is denormal,
  # rounded to 2^-150 absolute, and the division by ~1e-12 scales that up
  coef_err = (wi.abs() * (pbb_bound * EPS12 / (pbb + EPS12) ** 2 + C * 4 * U * pbb / (pbb + EPS12)) +
              C * 2.0 ** -150 / (pbb + EPS12))
  d = eye.double() - p
  g_ref = coef[:, None] * d
  _within(gsim, g_ref, coef.abs()[:, None] * (p_bound + C * U * d.abs()) + coef_err[:, None] * d.abs() +
          C * 2 * U * g_ref.abs() + FLOOR, 'inbatch_softmax_ce g_sim')
  assert bool((gsim[masked] == 0).all()), 'masked duplicates must get no gradient'
  if weights is not None:
    zero = weights == 0
    assert bool((loss[zero] == 0).all()) and bool((gsim[zero] == 0).all()), 'zero-weight rows contribute nothing'
  if variant == 'ids_all_equal' and N == B:
    assert bool((pd == 1).all()) and bool((loss == 0).all()) and bool((gsim == 0).all()), \
        'every other column masked: p_bb = 1, no loss, no gradient'

  bl2, loss2 = _out(B)
  _ok(lib.er_inbatch_softmax_ce(_p(sim), _p(ids), _p(weights), B, N, inv_wsum, _p(loss2), None, None, _stream()),
      'er_inbatch_softmax_ce')
  assert torch.equal(loss2, loss), 'probs_diag / g_sim = NULL must not change loss_rows'
  _untouched(bl2, loss2, 'inbatch_softmax_ce loss_rows (NULL outputs)')


# ---------------------------------------------------------------------------------------------------------------------
# DLRM Gram matrices: bit-exact against a float32 emulation in the kernel's summation order
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [1, 2, 27, 64])
@pytest.mark.parametrize('d', [1, 3, 16, 128])
def test_gram_bit_exact(n, d):
  lib, B = _lib_(), 37
  g = _gen(n * 1000 + d)
  x = torch.randn(B, n, d, device=DEV, generator=g)
  gout = torch.randn(B, n, n, device=DEV, generator=g)
  bo, out = _out(B, n, n)
  _ok(lib.er_gram_fwd(_p(x), B, n, d, _p(out), _stream()), 'er_gram_fwd')
  _untouched(bo, out, 'gram_fwd')
  bg, gx = _out(B, n, d)
  _ok(lib.er_gram_bwd(_p(x), _p(gout), B, n, d, _p(gx), _stream()), 'er_gram_bwd')
  _untouched(bg, gx, 'gram_bwd')

  xn, gn = x.cpu().numpy(), gout.cpu().numpy()
  acc = np.zeros((B, n, n), np.float32)
  for k in range(d):
    acc = acc + xn[:, :, None, k] * xn[:, None, :, k]      # float32 product, then float32 sum: one rounding each
  assert np.array_equal(out.cpu().numpy(), acc)
  assert torch.equal(out, out.transpose(1, 2))
  gs = gn + gn.transpose(0, 2, 1)
  acc = np.zeros((B, n, d), np.float32)
  for j in range(n):
    acc = acc + gs[:, :, j, None] * xn[:, None, j, :]
  assert np.array_equal(gx.cpu().numpy(), acc)


# ---------------------------------------------------------------------------------------------------------------------
# FM second order (er_fm_fwd / er_fm_bwd) and the FM block
# ---------------------------------------------------------------------------------------------------------------------

def _fm_emulate(x3):
  """float32 emulation of the kernels' order: s = sum_f x, q = sum_f x^2 in field order, y = 0.5 (s^2 - q)"""
  s = torch.zeros_like(x3[:, 0])
  q = torch.zeros_like(x3[:, 0])
  for f in range(x3.shape[1]):
    s = s + x3[:, f]
    q = q + x3[:, f] * x3[:, f]
  return s, 0.5 * (s * s - q)


@pytest.mark.parametrize('D', [4, 8, 16, 5])
def test_fm_fwd_vector_and_scalar_paths(D):
  lib, B, F = _lib_(), 1003, 13
  x3 = torch.randn(B, F, D, device=DEV, generator=_gen(D))
  x = _pitched_input(x3.reshape(B, F * D), 4)           # x_stride > F*D, NaN padding
  s, want = _fm_emulate(x3)
  results = []
  for shift in (0, 1):                                    # shift 1: y not 16-byte aligned, the scalar kernel
    buf, y = _out(B, D, shift=shift)
    _ok(lib.er_fm_fwd(_p(x), B, F, D, x.stride(0), _p(y), _stream()), 'er_fm_fwd')
    _untouched(buf, y, 'fm_fwd')
    assert torch.equal(y, want)
    results.append(y.clone())
  assert torch.equal(results[0], results[1]), 'float4 and scalar paths must agree bit for bit'

  gy = torch.randn(B, D, device=DEV, generator=_gen(D + 1))
  v = gy[:, None, :] * (s[:, None, :] - x3)
  pitch = F * D + 3
  buf, gx = _out(B, F * D, pitch=pitch)
  _ok(lib.er_fm_bwd(_p(x), _p(gy), B, F, D, x.stride(0), _p(gx), pitch, 0, _stream()), 'er_fm_bwd')
  _untouched(buf, gx, 'fm_bwd')
  assert torch.equal(gx.reshape(B, F, D), v)
  prefill = torch.randn(B, F * D, device=DEV, generator=_gen(D + 2))
  buf, gx = _out(B, F * D, pitch=pitch)
  gx.copy_(prefill)
  _ok(lib.er_fm_bwd(_p(x), _p(gy), B, F, D, x.stride(0), _p(gx), pitch, 1, _stream()), 'er_fm_bwd')
  _untouched(buf, gx, 'fm_bwd accumulate')
  assert torch.equal(gx, prefill + v.reshape(B, F * D)), 'accumulate = 1: gx + v rounded once'


# (n_field, dim): J = ceil(n_field * dim / 4 / 32) takes every value 1..8, dim / 4 every value 1..32
FM_BLOCK = [(1, 4), (200, 4), (256, 4), (24, 8), (20, 16), (13, 32), (9, 64), (11, 64), (8, 128), (1, 128), (7, 128)]


def _fm_block_sumsq_depth(B, J):
  """a row (J fields, <= 5 xor levels, 2 component adds, 5 shuffle levels), the rows of a warp, 8 warps, the CTA
  partials a thread adds, 5 shuffle levels, 8 warps"""
  grid = min(_cdiv(B, 8), 4 * 132)
  return J + 12 + _cdiv(B, grid * 8) + 8 + _cdiv(grid, 256) + 5 + 8


@pytest.mark.parametrize('F,dim', FM_BLOCK)
def test_fm_block(F, dim):
  lib, B = _lib_(), 1003
  J = _cdiv(F * dim // 4, 32)
  g = _gen(F * 1000 + dim)
  x3 = torch.randn(B, F, dim, device=DEV, generator=g)
  x = _pitched_input(x3.reshape(B, F * dim), 4)
  ws = torch.zeros(lib.er_fm_block_workspace_bytes(B), dtype=torch.uint8, device=DEV)
  by, y = _out(B, dim)
  bs, sumsq = _out(1)
  _ok(lib.er_fm_block_fwd(_p(x), B, F, dim, x.stride(0), _p(y), _p(sumsq), _p(ws), ws.numel(), _stream()),
      'er_fm_block_fwd')
  _untouched(by, y, 'fm_block_fwd y')
  _untouched(bs, sumsq, 'fm_block_fwd sumsq')
  x64 = x3.double()
  s, q = x64.sum(1), (x64 * x64).sum(1)
  s_err = C * (J + 5) * U * x64.abs().sum(1)
  q_err = C * (J + 6) * U * q
  y_ref = 0.5 * (s * s - q)
  _within(y, y_ref, s.abs() * s_err + 0.5 * (s_err * s_err + q_err) + C * U * (s * s + q) + FLOOR, 'fm_block_fwd y')
  _within(sumsq, q.sum().reshape(1), C * _fm_block_sumsq_depth(B, J) * U * q.sum().reshape(1),
          'fm_block_fwd sumsq')
  by2, y2 = _out(B, dim)
  bs2, sumsq2 = _out(1)
  _ok(lib.er_fm_block_fwd(_p(x), B, F, dim, x.stride(0), _p(y2), _p(sumsq2), _p(ws), ws.numel(), _stream()),
      'er_fm_block_fwd')
  assert torch.equal(y2, y) and torch.equal(sumsq2, sumsq), 'second call on the same workspace (counter reset)'
  by3, y3 = _out(B, dim)
  _ok(lib.er_fm_block_fwd(_p(x), B, F, dim, x.stride(0), _p(y3), None, None, 0, _stream()), 'er_fm_block_fwd')
  assert torch.equal(y3, y), 'sumsq_out = NULL must not change y'

  gy = torch.randn(B, dim, device=DEV, generator=g)
  gp = _pitched_input(torch.randn(B, F * dim, device=DEV, generator=g), 8)
  coef_dev = torch.tensor([0.37], device=DEV)
  coef_mul = 2e-3
  coef = float((coef_dev * torch.tensor(coef_mul, dtype=torch.float32, device=DEV)).item())
  gy64, gp64 = gy.double()[:, None, :], gp.double().reshape(B, F, dim)
  for use_gy in (True, False):
    for use_gp in (True, False):
      for use_coef in (True, False):
        pitch = F * dim + 4
        buf, gx = _out(B, F * dim, pitch=pitch)
        _ok(lib.er_fm_block_bwd(_p(x), _p(gy) if use_gy else None, _p(gp) if use_gp else None,
                                _p(coef_dev) if use_coef else None, coef_mul, B, F, dim, x.stride(0),
                                gp.stride(0) if use_gp else 0, _p(gx), pitch, _stream()), 'er_fm_block_bwd')
        _untouched(buf, gx, 'fm_block_bwd')
        a = gy64 if use_gy else torch.zeros_like(gy64)
        pas = gp64 if use_gp else torch.zeros_like(gp64)
        c = coef if use_coef else 0.0
        ref = pas + a * (s[:, None, :] - x64) + c * x64
        bound = (a.abs() * s_err[:, None, :] + C * 4 * U * (pas.abs() + a.abs() * (s.abs()[:, None, :] + x64.abs()) +
                                                             abs(c) * x64.abs()) + FLOOR)
        _within(gx.reshape(B, F, dim), ref, bound, 'fm_block_bwd gx')


def test_fm_block_refusals():
  """shapes and layouts the FM block cannot take are refused before launch; the buffers are large enough that an
  admitted call would stay inside them, and the outputs stay untouched"""
  lib, B = _lib_(), 64
  x = torch.zeros(B * 1280 + 64, device=DEV)
  ws = torch.zeros(lib.er_fm_block_workspace_bytes(B), dtype=torch.uint8, device=DEV)
  by, y = _out(B * 256 + 64)
  bx, gx = _out(B * 1280 + 64)
  cases = [(4, 12, 48, 0),       # dim / 4 = 3: not a power of two
           (1, 256, 256, 0),     # dim / 4 = 64 > 32
           (9, 128, 1152, 0),    # n_field * dim = 1152 > 1024
           (4, 16, 65, 0),       # row pitch not a multiple of 4 floats
           (4, 16, 64, 1)]       # x 4 bytes past a 16-byte boundary
  for F, dim, stride, shift in cases:
    xp = x.data_ptr() + 4 * shift
    rc = lib.er_fm_block_fwd(xp, B, F, dim, stride, _p(y), None, _p(ws), ws.numel(), _stream())
    assert rc == _lib.ER_ERR_INVALID_ARG, (F, dim, stride, shift, rc)
    rc = lib.er_fm_block_bwd(xp, None, None, None, 0.0, B, F, dim, stride, 0, _p(gx), stride - stride % 4,
                             _stream())
    assert rc == _lib.ER_ERR_INVALID_ARG, (F, dim, stride, shift, rc)
  torch.cuda.synchronize()
  assert bool(torch.isnan(by).all()) and bool(torch.isnan(bx).all()), 'a refused call wrote its output'
  # the control: the same buffers with an admissible shape
  _ok(lib.er_fm_block_fwd(x.data_ptr(), B, 4, 16, 64, _p(y), None, _p(ws), ws.numel(), _stream()), 'er_fm_block_fwd')
  assert bool((y[:B * 16] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# Wide row sum
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('width,B', [(1, 1003), (32, 1003), (33, 1003), (1000, 1003), (33, 65537), (1, 65537)])
def test_rowsum_block(width, B):
  lib = _lib_()
  g = _gen(width + B)
  xs = torch.randn(B, width, device=DEV, generator=g)
  x = _pitched_input(xs, 3)
  ws = torch.zeros(lib.er_fm_block_workspace_bytes(B), dtype=torch.uint8, device=DEV)
  by, y = _out(B)
  bs, sumsq = _out(1)
  _ok(lib.er_rowsum_block_fwd(_p(x), B, width, x.stride(0), _p(y), _p(sumsq), _p(ws), ws.numel(), _stream()),
      'er_rowsum_block_fwd')
  _untouched(by, y, 'rowsum_block_fwd y')
  _untouched(bs, sumsq, 'rowsum_block_fwd sumsq')
  x64 = xs.double()
  _within(y, x64.sum(1), C * _lanes(width) * U * x64.abs().sum(1) + FLOOR, 'rowsum_block_fwd y')
  q = (x64 * x64).sum()
  grid = min(_cdiv(B, 8), 4 * 132)
  depth = _lanes(width) + _cdiv(B, grid * 8) + 8 + _cdiv(grid, 256) + 5 + 8
  _within(sumsq, q.reshape(1), C * depth * U * q.reshape(1), 'rowsum_block_fwd sumsq')
  by2, y2 = _out(B)
  _ok(lib.er_rowsum_block_fwd(_p(x), B, width, x.stride(0), _p(y2), None, None, 0, _stream()),
      'er_rowsum_block_fwd')
  assert torch.equal(y2, y), 'sumsq_out = NULL must not change y'

  gy = torch.randn(B, device=DEV, generator=g)
  coef_dev = torch.tensor([0.37], device=DEV)
  coef_mul = 2e-3
  coef32 = coef_dev * torch.tensor(coef_mul, dtype=torch.float32, device=DEV)
  for use_gy in (True, False):
    for use_coef in (True, False):
      pitch = width + 5
      buf, gx = _out(B, width, pitch=pitch)
      _ok(lib.er_rowsum_block_bwd(_p(x), _p(gy) if use_gy else None, _p(coef_dev) if use_coef else None, coef_mul, B,
                                  width, x.stride(0), _p(gx), pitch, _stream()), 'er_rowsum_block_bwd')
      _untouched(buf, gx, 'rowsum_block_bwd')
      a = gy[:, None] if use_gy else torch.zeros(B, 1, device=DEV)
      c = coef32 if use_coef else torch.zeros(1, device=DEV)
      assert torch.equal(gx, a + c * xs), 'gx = gy + coef * x, each rounded once'


# ---------------------------------------------------------------------------------------------------------------------
# Logit head (dense with one unit)
# ---------------------------------------------------------------------------------------------------------------------

D1_WIDTHS = [1, 31, 32, 33, 64, 65, 97, 129, 161, 193, 255]    # JW = ceil(width / 32) = 1..8, both sides of each edge


def _dense1_bwd_depth(B, width):
  """the rows of a warp, 8 warps, the CTA partials one of `parts` threads adds, then the parts in order"""
  grid = min(_cdiv(B, 8), 132)
  parts = max(1, 256 // (width + 1))
  return _cdiv(B, grid * 8) + 8 + _cdiv(grid, parts) + parts


def _dense1_bwd(x, w, g, need_gx=True, need_gb=True):
  lib = _lib_()
  B, width = x.shape
  ws = torch.zeros(lib.er_dense1_workspace_bytes(width), dtype=torch.uint8, device=DEV)
  bufs = {'gw': _out(width), 'gb': _out(1)}
  if need_gx:
    bufs['gx'] = _out(B, width, pitch=width + 2)
  gx = bufs['gx'][1] if need_gx else None
  _ok(lib.er_dense1_bwd(_p(x), _p(w), _p(g), B, width, x.stride(0), _p(gx), width + 2, _p(bufs['gw'][1]),
                        _p(bufs['gb'][1]) if need_gb else None, _p(ws), ws.numel(), _stream()), 'er_dense1_bwd')
  for name, (buf, v) in bufs.items():
    if name == 'gb' and not need_gb:
      assert bool(torch.isnan(v).all()), 'gb = NULL: nothing may be written'
    else:
      _untouched(buf, v, 'dense1_bwd ' + name)
  return gx, bufs['gw'][1], bufs['gb'][1]


@pytest.mark.parametrize('width,B', [(wd, 1057) for wd in D1_WIDTHS] +
                         [(wd, b) for wd in (1, 33, 255) for b in (1, 7, 9, 1 << 20)])
def test_dense1(width, B):
  lib = _lib_()
  g = _gen(width * 7 + B)
  xs = torch.randn(B, width, device=DEV, generator=g)
  x = _pitched_input(xs, 3)
  w = torch.randn(width, device=DEV, generator=g)
  bias = torch.randn(1, device=DEV, generator=g)
  for b_ in (bias, None):
    buf, y = _out(B)
    _ok(lib.er_dense1_fwd(_p(x), _p(w), _p(b_), B, width, x.stride(0), _p(y), _stream()), 'er_dense1_fwd')
    _untouched(buf, y, 'dense1_fwd')
    b64 = float(b_.item()) if b_ is not None else 0.0
    for s in _row_blocks(B, width):
      xw = xs[s].double() * w.double()
      ref = xw.sum(1) + b64
      _within(y[s], ref, C * (_lanes(width) + 1) * U * (xw.abs().sum(1) + abs(b64)) + FLOOR, 'dense1_fwd y')

  gg = torch.randn(B, device=DEV, generator=g)
  gx, gw, gb = _dense1_bwd(x, w, gg)
  depth = _dense1_bwd_depth(B, width)
  gw_ref = torch.zeros(width, dtype=torch.float64, device=DEV)
  gw_abs = torch.zeros_like(gw_ref)
  for s in _row_blocks(B, width):
    t = gg[s].double()[:, None] * xs[s].double()
    gw_ref += t.sum(0)
    gw_abs += t.abs().sum(0)
    assert torch.equal(gx[s], gg[s][:, None] * w[None, :])
  _within(gw, gw_ref, C * depth * U * gw_abs + FLOOR, 'dense1_bwd gw')
  g64 = gg.double()
  _within(gb, g64.sum().reshape(1), C * depth * U * g64.abs().sum().reshape(1) + FLOOR, 'dense1_bwd gb')

  _, gw2, gb2 = _dense1_bwd(x, w, gg)
  assert torch.equal(gw2, gw) and torch.equal(gb2, gb), 'a repeated call must give the same bits'
  _, gw3, _ = _dense1_bwd(x, w, gg, need_gx=False, need_gb=False)
  assert torch.equal(gw3, gw), 'gx / gb = NULL must not change gw'


def test_dense1_width_256_refused():
  lib, B, width = _lib_(), 64, 256
  x = torch.zeros(B, width, device=DEV)
  w = torch.zeros(width, device=DEV)
  g = torch.zeros(B, device=DEV)
  ws = torch.zeros(lib.er_dense1_workspace_bytes(width), dtype=torch.uint8, device=DEV)
  bw, gw = _out(width)
  bb, gb = _out(1)
  rc = lib.er_dense1_bwd(_p(x), _p(w), _p(g), B, width, width, None, 0, _p(gw), _p(gb), _p(ws), ws.numel(), _stream())
  assert rc == _lib.ER_ERR_INVALID_ARG
  torch.cuda.synchronize()
  assert bool(torch.isnan(bw).all()) and bool(torch.isnan(bb).all())


# ---------------------------------------------------------------------------------------------------------------------
# Sigmoid cross entropy
# ---------------------------------------------------------------------------------------------------------------------

SPECIAL_LOGITS = [0.0, 1e-8, -1e-8, 20.0, -20.0, 88.0, -88.0, 89.0, -89.0, 100.0, -100.0, 1e4, -1e4, 1.0, -1.0]


@pytest.mark.parametrize('B', [1, 1023, 1024, 1025, 1 << 20])
def test_sigmoid_ce(B):
  lib = _lib_()
  g = _gen(B)
  logits = torch.randn(B, device=DEV, generator=g) * 5
  labels = torch.tensor([0.0, 1.0, 0.3], device=DEV)[torch.randint(0, 3, (B,), device=DEV, generator=g)]
  n = min(B, 3 * len(SPECIAL_LOGITS))       # every special logit with every label
  i = torch.arange(n, device=DEV)
  logits[:n] = torch.tensor(SPECIAL_LOGITS, device=DEV)[i % len(SPECIAL_LOGITS)]
  labels[:n] = torch.tensor([0.0, 1.0, 0.3], device=DEV)[i // len(SPECIAL_LOGITS)]
  weights = torch.rand(B, device=DEV, generator=g)
  weights[::5] = 0.0
  x64, z64 = logits.double(), labels.double()
  e = torch.exp(-x64.abs())
  l1p = torch.log1p(e)
  ce = torch.clamp(x64, min=0) - x64 * z64 + l1p
  ce_err = C * (3 * U * (torch.clamp(x64, min=0) + (x64 * z64).abs() + l1p) + 4 * U * e + 2 * U * l1p)
  p = torch.sigmoid(x64)
  p_err = C * (4 * U * (1 - p) * p + 2 * U * p) + 2.0 ** -126
  depth = _cdiv(B, 1024) + 10
  for wts in (weights, None):
    w64 = wts.double() if wts is not None else torch.ones_like(x64)
    inv = float(np.float32(1.0 / float(w64.sum()))) if float(w64.sum()) > 0 else 1.0
    bl, loss = _out(1)
    bp, probs = _out(B)
    bg, gl = _out(B)
    _ok(lib.er_sigmoid_ce_fwd_bwd(_p(logits), _p(labels), _p(wts), B, inv, _p(loss), _p(probs), _p(gl), _stream()),
        'er_sigmoid_ce_fwd_bwd')
    for buf, v, name in ((bl, loss, 'loss'), (bp, probs, 'probs'), (bg, gl, 'g_logits')):
      _untouched(buf, v, 'sigmoid_ce ' + name)
    wl = w64 * ce
    loss_ref = inv * wl.sum()
    _within(loss, loss_ref.reshape(1), (inv * ((w64.abs() * ce_err).sum() + C * depth * U * wl.abs().sum()) +
                                        C * U * loss_ref.abs()).reshape(1) + FLOOR, 'sigmoid_ce loss')
    _within(probs, p, p_err, 'sigmoid_ce probs')
    g_ref = w64 * (p - z64) * inv
    _within(gl, g_ref, (w64 * inv).abs() * (p_err + C * U * (p - z64).abs()) + C * 2 * U * g_ref.abs() + FLOOR,
            'sigmoid_ce g_logits')
    bl2, loss2 = _out(1)
    _ok(lib.er_sigmoid_ce_fwd_bwd(_p(logits), _p(labels), _p(wts), B, inv, _p(loss2), None, None, _stream()),
        'er_sigmoid_ce_fwd_bwd')
    assert torch.equal(loss2, loss), 'probs / g_logits = NULL must not change the loss'
