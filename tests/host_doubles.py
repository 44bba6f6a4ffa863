"""Kernel doubles for the host-side tests (TEST INFRASTRUCTURE): stand-ins with the signatures of the entry points in
easyrec_b200.kernels / interactions whose bodies are the CPU oracle (sparse path), plain torch (dense towers,
interactions) or numpy.  `patch(obj, name, fn)` is pytest's monkeypatch.setattr in fixtures and plain setattr in
spawned worker processes."""
import numpy as np
import torch

from easyrec_b200 import _lib, kernels as K, trainer as T
from oracle import oracle as O


def _slots(slots_dev):
  return np.frombuffer(slots_dev.numpy().tobytes(), dtype=K.SLOT_DTYPE)


def _seg_field(sl, field, n_seg):
  v = np.concatenate([np.full(int(s['n_seg']), s[field]) for s in sl])[:n_seg]
  return v & 0xf if field == 'combiner' else v   # (the ER_COMBINER_UNIT_WEIGHTS flag is a hint for the kernels)


class _Hyper(object):
  """the step scalars as the kernels see them: from er_opt_t.hyper_dev when set (float[4] = lr, beta1^t, beta2^t,
  gradient scale - host memory in these CPU tests), else from the struct"""

  def __init__(self, opt):
    if opt.hyper_dev:
      import ctypes
      h = (ctypes.c_float * 4).from_address(opt.hyper_dev)
      self.lr, self.beta1_power, self.beta2_power, self.grad_scale = float(h[0]), float(h[1]), float(h[2]), float(h[3])
    else:
      self.lr, self.beta1_power, self.beta2_power, self.grad_scale = opt.lr, opt.beta1_power, opt.beta2_power, opt.grad_scale


def install_sparse(patch):
  """bucketize / csr_from_lens / embedding_fwd / embedding_bwd -> the CPU oracle."""
  def csr_from_lens(lens, cap, want_seg_ids=True):
    row_ptr, seg = O.csr_from_lens(lens.numpy())
    seg_ids = np.zeros(max(cap, 1), np.int32)
    seg_ids[:seg.size] = seg
    return torch.from_numpy(row_ptr), torch.from_numpy(seg_ids)

  def bucketize(ids, slots_dev, n_slots, n_seg, seg_ids=None, row_ptr=None, rows=None, owner=None):
    sl = _slots(slots_dev)
    n = ids.numel()
    if row_ptr is None:
      seg_of = np.arange(n)
      live = np.ones(n, bool)
    else:
      total = int(row_ptr[-1])
      seg_of = seg_ids.numpy()[:n].astype(np.int64)
      live = np.arange(n) < total
      seg_of = np.where(live, seg_of, 0)
    per = lambda f: _seg_field(sl, f, n_seg)[seg_of]   # noqa: E731
    r, own = O.bucketize(ids.numpy(), per('bucket_mode'), per('num_buckets'), per('row_offset'), shard_n=per('shard_n'))
    r = np.where(live, r, -1)
    out = rows if rows is not None else torch.empty_like(ids)
    out.copy_(torch.from_numpy(r))
    if owner is not None:
      owner.copy_(torch.from_numpy(np.where(live, own, -1).astype(np.int32)))
    return out

  def _csr(n_seg, rows, row_ptr):
    return np.arange(n_seg + 1, dtype=np.int32) if row_ptr is None else row_ptr.numpy()

  def embedding_fwd(table, dim, rows, slots_dev, n_slots, n_seg, outs, weights=None, row_ptr=None, seg_scale=None,
                    row_stride=None):
    sl = _slots(slots_dev)
    rp = _csr(n_seg, rows, row_ptr)
    pooled, scale = O.embedding_fwd(np.ascontiguousarray(table.numpy()), rows.numpy(), rp, _seg_field(sl, 'combiner', n_seg),
                                    weights=None if weights is None else weights.numpy())
    for s in sl:
      out = outs[int(s['out_buf'])].view(-1)
      for k in range(min(int(s['n_seg']), n_seg - int(s['seg_begin']))):   # (a call may use a prefix of its plan)
        o = k * int(s['out_stride']) + int(s['out_col'])
        out[o:o + dim] = torch.from_numpy(pooled[int(s['seg_begin']) + k])
    if seg_scale is not None:
      seg_scale.copy_(torch.from_numpy(scale))

  def embedding_bwd(table, state0, state1, dim, rows, slots_dev, n_slots, n_seg, grad_bufs, opt, ws, weights=None,
                    seg_ids=None, row_ptr=None, seg_scale=None, row_stride=None, uniq_rows=None, uniq_grads=None,
                    n_uniq=None, n_rows=None, sorted_from=None):
    if sorted_from is not None and K.k7_warp_mode(sorted_from[1]) != K.k7_warp_mode(dim):
      # er_embedding_bwd_reuse_sort's precondition: a placement is reused only by a table of its own placement mode
      raise _lib.ErError('er_embedding_bwd_reuse_sort: a dim-%d placement reused by a dim-%d table (other placement '
                         'mode)' % (sorted_from[1], dim))
    sl = _slots(slots_dev)
    gseg = np.zeros((n_seg, dim), np.float32)
    for s in sl:
      buf = grad_bufs[int(s['out_buf'])].reshape(-1).numpy()
      for k in range(min(int(s['n_seg']), n_seg - int(s['seg_begin']))):
        o = k * int(s['out_stride']) + int(s['out_col'])
        gseg[int(s['seg_begin']) + k] = buf[o:o + dim]
    if table is None:   # emit only: the deduplicated gradient, sorted by row
      nu, ur, ug = O.embedding_bwd(None, None, None, rows.numpy(), None if seg_ids is None else seg_ids.numpy()[:rows.numel()],
                                   gseg, O.OPT_SGD, 0.0, weights=None if weights is None else weights.numpy(),
                                   seg_scale=None if seg_scale is None else seg_scale.numpy(), grad_scale=_Hyper(opt).grad_scale,
                                   want_uniq=True)
      uniq_rows[:nu].copy_(torch.from_numpy(ur))
      uniq_grads[:nu].copy_(torch.from_numpy(ug))
      n_uniq.fill_(nu)
      return
    t = np.ascontiguousarray(table.numpy())
    a = None if state0 is None else np.ascontiguousarray(state0.numpy())
    b = None if state1 is None else np.ascontiguousarray(state1.numpy())
    # the row rule of tf.train.AdamOptimizer on touched rows is the lazy rule (kind 3 -> 2); its dense decay is the
    # adam_dense_sweep double below
    kind = {0: O.OPT_SGD, 1: O.OPT_ADAGRAD, 2: O.OPT_LAZY_ADAM, 3: O.OPT_LAZY_ADAM, 4: O.OPT_MOMENTUM}[int(opt.kind)]
    O.embedding_bwd(t, a, b, rows.numpy(), None if seg_ids is None else seg_ids.numpy()[:rows.numel()], gseg,
                    kind, _Hyper(opt).lr, weights=None if weights is None else weights.numpy(),
                    seg_scale=None if seg_scale is None else seg_scale.numpy(), beta1=opt.beta1, beta2=opt.beta2,
                    eps=opt.eps, beta1_power=_Hyper(opt).beta1_power, beta2_power=_Hyper(opt).beta2_power,
                    grad_scale=_Hyper(opt).grad_scale)
    table.copy_(torch.from_numpy(t))
    if state0 is not None:
      state0.copy_(torch.from_numpy(a))
    if state1 is not None:
      state1.copy_(torch.from_numpy(b))

  def sparse_apply(table, state0, state1, dim, uniq_rows, uniq_grads, n_uniq, opt, row_stride=None):
    n = uniq_rows.numel() if n_uniq is None else int(n_uniq.reshape(-1)[0])
    t = np.ascontiguousarray(table.numpy())
    a = None if state0 is None else np.ascontiguousarray(state0.numpy())
    b = None if state1 is None else np.ascontiguousarray(state1.numpy())
    kind = {0: O.OPT_SGD, 1: O.OPT_ADAGRAD, 2: O.OPT_LAZY_ADAM, 3: O.OPT_LAZY_ADAM}[int(opt.kind)]
    O.embedding_bwd(t, a, b, uniq_rows.numpy()[:n], None, np.ascontiguousarray(uniq_grads.numpy()[:n]), kind, _Hyper(opt).lr,
                    beta1=opt.beta1, beta2=opt.beta2, eps=opt.eps, beta1_power=_Hyper(opt).beta1_power,
                    beta2_power=_Hyper(opt).beta2_power, grad_scale=_Hyper(opt).grad_scale)
    table.copy_(torch.from_numpy(t))
    if state0 is not None:
      state0.copy_(torch.from_numpy(a))
    if state1 is not None:
      state1.copy_(torch.from_numpy(b))

  def mark_rows(rows, n_rows, touched, value, n_dev=None):
    r = rows.numpy()
    n = r.size if n_dev is None else min(int(n_dev.reshape(-1)[0]), r.size)
    r = r[:n]
    touched[torch.from_numpy(r[(r >= 0) & (r < n_rows)])] = value

  def adam_dense_sweep(table, m, v, dim, touched, opt, row_stride=None):
    f = np.float32
    cold = torch.from_numpy(touched.numpy() == 0) if touched is not None else torch.ones(table.shape[0], dtype=torch.bool)
    lr_t = O.adam_lr_t(_Hyper(opt).lr, _Hyper(opt).beta1_power, _Hyper(opt).beta2_power)
    mc = (m[cold].numpy() * f(opt.beta1)).astype(np.float32)
    vc = (v[cold].numpy() * f(opt.beta2)).astype(np.float32)
    m[cold] = torch.from_numpy(mc)
    v[cold] = torch.from_numpy(vc)
    table[cold] = torch.from_numpy(table[cold].numpy() - (lr_t * mc) / (np.sqrt(vc) + f(opt.eps)))
  def shard_group_workspace(n_lookups, device):
    return torch.empty(16, dtype=torch.uint8)

  def shard_group(rows, owner, world, cap, send_rows, pos, counts, ws):
    """er_shard_group: distinct (owner, row) pairs in first-occurrence order (the kernel's order is arbitrary)"""
    r, o = rows.numpy(), owner.numpy()
    send = np.full(world * cap, -1, np.int64)
    p = np.full(r.size, -1, np.int64)
    cnt = np.zeros(world + 1, np.int32)
    seen = {}
    for l in range(r.size):
      if r[l] < 0 or o[l] < 0 or o[l] >= world:   # (an owner outside [0, world) is not counted, as in the kernel)
        continue
      key = (int(o[l]), int(r[l]))
      if key not in seen:
        k = int(cnt[o[l]])
        cnt[o[l]] += 1
        seen[key] = o[l] * cap + k if k < cap else -1
        if k < cap:
          send[o[l] * cap + k] = r[l]
      p[l] = seen[key]
      if p[l] < 0:
        cnt[world] += 1
    send_rows.copy_(torch.from_numpy(send))
    pos.copy_(torch.from_numpy(p))
    counts.copy_(torch.from_numpy(cnt))
  for name, fn in (('csr_from_lens', csr_from_lens), ('bucketize', bucketize), ('embedding_fwd', embedding_fwd),
                   ('embedding_bwd', embedding_bwd), ('mark_rows', mark_rows), ('adam_dense_sweep', adam_dense_sweep),
                   ('sparse_apply', sparse_apply), ('shard_group', shard_group),
                   ('shard_group_workspace', shard_group_workspace)):
    patch(K, name, fn)



def install_dense(patch):
  """dense towers, loss, FM and the flat dense optimizer -> plain torch / the oracle's numpy."""
  def dropout(x, rate, seed, counter, out=None):
    g = torch.Generator().manual_seed((int(seed) + 1000003 * int(counter[0])) % (2**63))
    keep = 1.0 - rate
    mask = (torch.rand(x.shape, generator=g) < keep).to(x.dtype) / keep
    y = x * mask
    if out is not None:
      out.copy_(y)
      return out
    return y
  patch(K, 'dropout', dropout)

  names = {v: k for k, v in K.ACT_KINDS.items() if k != 'prelu'}

  def act_fwd(x, kind):
    return torch.from_numpy(O.activation(x.detach().numpy(), names[kind]).astype(np.float32))

  def act_bwd(x, gy, kind):
    return torch.from_numpy((gy.detach().numpy().astype(np.float64) *
                             O.activation_grad(x.detach().numpy(), names[kind])).astype(np.float32))

  def auc_hist(probs, labels, thresholds, hist):
    # k = number of thresholds strictly below the prediction; negatives in the first T + 1 bins, positives after
    T = thresholds.numel()
    p, lab = probs.detach().reshape(-1).numpy(), labels.detach().reshape(-1).numpy().astype(np.int64) != 0
    k = np.where(np.isnan(p), 0, np.searchsorted(thresholds.numpy(), p, side='left'))   # (a NaN exceeds no threshold)
    hist += torch.from_numpy(np.bincount(k + lab * (T + 1), minlength=2 * (T + 1)).astype(np.int64))
    return hist
  def dice_fwd(x, xn, alpha):
    p = torch.sigmoid(xn)
    return alpha * (1.0 - p) * x + p * x

  def dice_bwd(x, xn, alpha, gy):
    p = torch.sigmoid(xn)
    return gy * (alpha * (1.0 - p) + p), gy * x * (1.0 - alpha) * p * (1.0 - p), gy * x * (1.0 - p)
  patch(K, 'dice_fwd', dice_fwd)
  patch(K, 'dice_bwd', dice_bwd)
  patch(K, 'act_fwd', act_fwd)
  patch(K, 'act_bwd', act_bwd)
  patch(K, 'auc_hist', auc_hist)

  def gemm(a, b, bias=None, out=None):
    r = a @ b
    if bias is not None:
      r = r + bias
    if out is not None:
      out.copy_(r)
      return out
    return r

  def bias_bn_act_fwd(z, bias, gamma, beta, moving_mean, moving_var, eps, momentum, training, relu, ws,
                      y=None, save_mean=None, save_rstd=None):
    h = z if bias is None else z + bias
    mean = rstd = None
    if gamma is not None:
      if training:
        mean = h.mean(0)
        var = ((h - mean) ** 2).mean(0)
        moving_mean.mul_(momentum).add_(mean * (1 - momentum))
        moving_var.mul_(momentum).add_(var * (1 - momentum))
      else:
        mean, var = moving_mean, moving_var
      rstd = 1.0 / torch.sqrt(var + eps)
      h = (h - mean) * rstd * gamma + beta
    return (torch.relu(h) if relu else h), mean, rstd

  def bias_bn_act_bwd(z, bias, gamma, y, gy, mean, rstd, relu, ws):
    g = gy * (y > 0) if relu else gy
    if gamma is None:
      return g, g.sum(0), None, None
    xhat = ((z if bias is None else z + bias) - mean) * rstd
    B = z.shape[0]
    ggamma, gbeta = (g * xhat).sum(0), g.sum(0)
    gx = g * gamma
    gz = rstd / B * (B * gx - gx.sum(0) - xhat * (gx * xhat).sum(0))
    return gz, gz.sum(0), ggamma, gbeta

  def sigmoid_ce(logits, labels, weights=None, inv_count=None, want_grad=True):
    if weights is None and inv_count is None:
      loss, probs, g = O.sigmoid_ce(logits.detach().numpy(), labels.numpy())
      return torch.tensor([loss], dtype=torch.float32), torch.from_numpy(probs), torch.from_numpy(g)
    # the kernel's contract: loss = sum(w * ce) * inv_count, g = w * (p - z) * inv_count
    x, z = logits.detach().numpy().astype(np.float32), labels.numpy().astype(np.float32)
    w = np.ones_like(x) if weights is None else weights.numpy().astype(np.float32)
    inv = np.float32(1.0 / x.size if inv_count is None else inv_count)
    ce = np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))
    p = (1.0 / (1.0 + np.exp(-x))).astype(np.float32)
    return (torch.tensor([float((w * ce).sum(dtype=np.float32) * inv)], dtype=torch.float32), torch.from_numpy(p),
            torch.from_numpy((w * (p - z) * inv).astype(np.float32)))

  def fm_fwd(x, n_field, dim, y=None):
    return torch.from_numpy(O.fm_fwd(np.ascontiguousarray(x.detach().numpy()[:, :n_field * dim]), n_field, dim))

  def fm_bwd(x, gy, n_field, dim, gx=None, accumulate=False):
    w = n_field * dim
    g = torch.from_numpy(O.fm_bwd(np.ascontiguousarray(x.detach().numpy()[:, :w]), np.ascontiguousarray(gy.numpy()), n_field, dim))
    if gx is None:
      return g
    if accumulate:
      gx[:, :w] += g
    else:
      gx[:, :w] = g
    return gx

  def apply(self, l2_folded=False, grad_scale=None):   # FlatDenseOptimizer.apply: l2 + TF Adagrad / Adam / SGD over the flat buffer
    scale = self.grad_scale if grad_scale is None else grad_scale
    assert self.kind in (0, 1, 3, 4), 'this double implements the sgd, adagrad, adam and momentum rules'
    segs = np.frombuffer((self.segs_nol2_dev if l2_folded else self.segs_dev).numpy().tobytes(),
                         dtype=T._lib.DENSE_SEG_DTYPE)
    keep_reg = self.reg_loss.clone()
    self.reg_loss.zero_()
    lr = float(self.lr_dev[0])
    for s in segs:
      o, n = int(s['offset']), int(s['n'])
      w, g = self.flat_p[o:o + n], self.flat_g[o:o + n] * scale
      if s['l2'] > 0:
        self.reg_loss += 0.5 * float(s['l2']) * (w * w).sum()
        g = g + float(s['l2']) * w
      if self.kind == 0:
        w -= lr * float(s['lr_mult']) * g
      elif self.kind == 1:
        self.s0[o:o + n] += g * g
        w -= lr * float(s['lr_mult']) * g / torch.sqrt(self.s0[o:o + n])
      elif self.kind == 4:   # ApplyMomentum: accum = accum * momentum + g ; var -= lr * accum
        self.s0[o:o + n] = self.s0[o:o + n] * self.b1 + g
        w -= lr * float(s['lr_mult']) * self.s0[o:o + n]
      else:   # ApplyAdam: m, v, var -= lr_t*m/(sqrt(v)+eps)
        self.s0[o:o + n] = self.b1 * self.s0[o:o + n] + (1 - self.b1) * g
        self.s1[o:o + n] = self.b2 * self.s1[o:o + n] + (1 - self.b2) * g * g
        w -= lr * float(s['lr_mult']) * self.s0[o:o + n] / (torch.sqrt(self.s1[o:o + n]) + self.eps)
    if l2_folded:   # (the caller computed the regularisation loss when it folded l2 * w into the gradient)
      self.reg_loss.copy_(keep_reg)
  for name, fn in (('gemm', gemm), ('gemm_ready', lambda t: t), ('gemm_bn', lambda *a, **k: None),
                   ('bias_bn_act_fwd', bias_bn_act_fwd), ('bias_bn_act_bwd', bias_bn_act_bwd),
                   ('dense_workspace', lambda b, u, d: torch.zeros(1, dtype=torch.uint8)), ('sigmoid_ce', sigmoid_ce),
                   ('fm_fwd', fm_fwd), ('fm_bwd', fm_bwd)):
    patch(K, name, fn)
  patch(T.FlatDenseOptimizer, 'apply', apply)



def install_interactions(patch):
  """torch-native stand-ins for the fused interaction ops (autograd supplies their backward)."""
  from easyrec_b200 import interactions as I

  def din_attention(query, keys, lens, attention_mlp):
    B, T, D = keys.shape
    q = query[:, None, :].expand(B, T, D)
    scores = attention_mlp(torch.cat([q, keys, q - keys, q * keys], dim=-1)).reshape(B, T)
    mask = torch.arange(T)[None, :] < lens[:, None]
    p = torch.softmax(torch.where(mask, scores, torch.full_like(scores, -2.0**32 + 1)), dim=1)
    return (p[:, :, None] * keys).sum(1)

  def inbatch_softmax_ce(sim, item_ids=None, weights=None):
    B = sim.shape[0]
    if item_ids is not None:
      dup = (item_ids[None, :B] == item_ids[:B, None]).float() - torch.eye(B)
      sim = torch.cat([sim[:, :B] - dup * 1e32, sim[:, B:]], dim=1)
    p = torch.softmax(sim, dim=1)
    diag = p[torch.arange(B), torch.arange(B)]
    w = torch.ones(B) if weights is None else weights
    return -(torch.log(diag + 1e-12) * w).mean() / w.mean(), diag.detach()
  def din_pool(scores, keys, lens):
    T = keys.shape[1]
    mask = torch.arange(T)[None, :] < lens[:, None]
    p = torch.softmax(torch.where(mask, scores, torch.full_like(scores, -2.0**32 + 1)), dim=1)
    return (p[:, :, None] * keys).sum(1)
  patch(I, 'din_pool', din_pool)
  patch(I, 'gram', lambda x: torch.bmm(x, x.transpose(1, 2)))
  patch(I, 'matmul_nt', lambda u, i: u @ i.t())
  patch(I, 'din_attention', din_attention)
  patch(I, 'cross_layer', lambda x0, xl, w, b: x0 * (xl * w).sum(1, keepdim=True) + b + xl)
  patch(I, 'mmoe_mix', lambda g, ex: (torch.softmax(g, dim=1)[:, :, None] * ex).sum(1))
  patch(I, 'l2_normalize', lambda x: x / torch.sqrt(torch.clamp((x * x).sum(1, keepdim=True), min=1e-12)))
  patch(I, 'inbatch_softmax_ce', inbatch_softmax_ce)




def install_all(patch=setattr):
  install_sparse(patch)
  install_dense(patch)
  install_interactions(patch)
