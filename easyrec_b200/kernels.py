"""Thin torch shim over the C ABI: tensors in, `data_ptr()`s + current stream out.

torch is plumbing here (device memory, streams); every function below is one
call into liber_b200.so.  Shapes/dtypes are checked on the host; nothing falls
back to a torch implementation.
"""
import ctypes
import os

import numpy as np
import torch

from easyrec_b200 import _lib, expr
from easyrec_b200._lib import ErOpt, SLOT_DTYPE, c_vp


def _stream():
  return torch.cuda.current_stream().cuda_stream


def _p(t):
  return None if t is None else t.data_ptr()


def _chk(t, dtype, name):
  if t is None:
    return
  if not t.is_cuda:
    raise _lib.ErError('%s must be a CUDA tensor (no CPU fallback)' % name)
  if t.dtype != dtype:
    raise _lib.ErError('%s must be %s, got %s' % (name, dtype, t.dtype))
  if not t.is_contiguous():
    raise _lib.ErError('%s must be contiguous' % name)


def _chk_rows(t, name):
  """table / optimizer-state matrix [n_rows, dim]: fp32, unit inner stride; the row stride may
  exceed dim (interleaved [w | state] rows).  Returns (n_rows, row_stride)."""
  if t is None:
    return None
  if not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1:
    raise _lib.ErError('%s must be a CUDA fp32 [rows, dim] matrix with unit inner stride' % name)
  return t.shape[0], t.stride(0)


def _buf_array(bufs):
  arr = (c_vp * len(bufs))()
  for i, b in enumerate(bufs):
    arr[i] = b.data_ptr()
  return arr


VECTOR_DIMS = (4, 8, 16, 32, 64, 128)


def make_slots(records, dim=None):
  """records: list of dicts with er_slot_t field names -> numpy structured array.

  dim: the arena's embedding dim.  At the vector dims K2 and K7 move rows with 16-byte accesses at
  out_stride * s + out_col of the slot's output buffer, so every out_stride and out_col must then be a multiple of 4
  (include/er_b200.h); the slot table lives in device memory, where the kernels cannot check it."""
  arr = np.zeros(len(records), dtype=SLOT_DTYPE)
  for i, r in enumerate(records):
    for k, v in r.items():
      arr[i][k] = v
    if arr[i]['shard_n'] == 0:
      arr[i]['shard_n'] = 1
  order = np.argsort(arr['seg_begin'], kind='stable')
  if not np.array_equal(order, np.arange(len(records))):
    raise _lib.ErError('slots must be ordered by seg_begin')
  if dim in VECTOR_DIMS:
    bad = np.nonzero((arr['out_stride'] % 4 != 0) | (arr['out_col'] % 4 != 0))[0]
    if bad.size:
      raise _lib.ErError('slot %d: out_stride %d / out_col %d must be multiples of 4 at dim %d' % (
          bad[0], arr[bad[0]]['out_stride'], arr[bad[0]]['out_col'], dim))
  return arr


def slots_to_device(slots_np, device):
  raw = torch.from_numpy(slots_np.view(np.uint8).reshape(-1).copy())
  return raw.to(device)


def csr_from_lens(lens, n_lookups_cap, want_seg_ids=True):
  """lens int32 [n_seg] -> (row_ptr int32 [n_seg+1], seg_ids int32 [cap] | None)."""
  lib = _lib.load()
  _chk(lens, torch.int32, 'lens')
  n_seg = lens.numel()
  row_ptr = torch.empty(n_seg + 1, dtype=torch.int32, device=lens.device)
  seg_ids = (torch.empty(max(n_lookups_cap, 1), dtype=torch.int32, device=lens.device)
             if want_seg_ids else None)
  ws_bytes = lib.er_csr_workspace_bytes(n_seg)
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device=lens.device)
  _lib.check(
      lib.er_csr_from_lens(_p(lens), n_seg, _p(row_ptr), _p(seg_ids), n_lookups_cap, _p(ws),
                           ws_bytes, _stream()), 'er_csr_from_lens')
  return row_ptr, seg_ids


def vocab_index(keys, device):
  """A vocabulary's read-only index on the device: er_kv_insert_rows of entry i's key with row i into an empty index of
  at least twice as many slots.  keys: int64 numpy, distinct and >= 0.  Returns (index_keys, index_rows).  K1 probes
  the index on the GPU; there is no host K1 to read it, so a host device is refused."""
  if not str(device).startswith('cuda'):
    raise NotImplementedError('a vocabulary index is probed by K1 on the GPU; device %s has no K1' % device)
  n_index = 16
  while n_index < 2 * keys.size:
    n_index *= 2
  index_keys = torch.full((n_index,), _lib.KV_EMPTY, dtype=torch.int64, device=device)
  index_rows = torch.full((n_index,), -1, dtype=torch.int64, device=device)
  stats = torch.zeros(2, dtype=torch.int64, device=device)
  kv_insert_rows(index_keys, index_rows, torch.from_numpy(keys).to(device),
                 torch.arange(keys.size, dtype=torch.int64).to(device), stats)
  if int(stats[1]):
    raise _lib.ErError('vocabulary index: %d keys are negative or repeated' % int(stats[1]))
  return index_keys, index_rows


class VocabPlan(object):
  """The vocabularies of one slot plan: `per_slot[i]` is slot i's embedding.Vocab (None for a slot of another mode);
  `dev` holds their er_vocab_t descriptors in slot order, the array the *_vocab forms of K1 are given."""

  def __init__(self, per_slot, device):
    self.per_slot = list(per_slot)
    desc = np.zeros(len(self.per_slot), dtype=_lib.VOCAB_DTYPE)
    for i, v in enumerate(self.per_slot):
      if v is not None:
        desc[i] = (v.index_keys.data_ptr(), v.index_rows.data_ptr(), v.index_keys.numel())
    self.dev = torch.from_numpy(desc.view(np.uint8).copy()).to(device)


def vocab_plan(slots_np, vocabs, device):
  """VocabPlan of a slot plan whose slot i reads vocabulary vocabs[i], or None when no slot is ER_BUCKET_VOCAB.  A
  vocabulary slot without its index is an error: the hashing kernels would read its keys as rows."""
  modes = [int(m) for m in slots_np['bucket_mode']]
  if _lib.BUCKET_VOCAB not in modes:
    return None
  for i, m in enumerate(modes):
    if (m == _lib.BUCKET_VOCAB) != (vocabs[i] is not None):
      raise _lib.ErError('slot %d: a vocabulary goes with bucket mode ER_BUCKET_VOCAB and only with it' % i)
  return VocabPlan(vocabs, device)


def bucketize(ids, slots_dev, n_slots, n_seg, seg_ids=None, row_ptr=None, rows=None,
              owner=None, weights=None, vocabs=None):
  """K1 (er_bucketize).  weights: the lookup weights the lookup will be pooled with (er_bucketize_weighted); mean /
  sqrtn lookups whose weight is not > 0 come out as dropped rows (-1), as safe_embedding_lookup_sparse prunes them.
  vocabs: the VocabPlan of a plan with vocabulary slots (er_bucketize_vocab)."""
  lib = _lib.load()
  _chk(ids, torch.int64, 'ids')
  _chk(weights, torch.float32, 'weights')
  _chk(seg_ids, torch.int32, 'seg_ids')
  _chk(row_ptr, torch.int32, 'row_ptr')
  _chk(owner, torch.int32, 'owner')
  if rows is None:
    rows = torch.empty_like(ids)
  _chk(rows, torch.int64, 'rows')
  if vocabs is not None:
    assert len(vocabs.per_slot) == n_slots and (weights is None or weights.numel() >= ids.numel())
    _lib.check(
        lib.er_bucketize_vocab(_p(ids), _p(weights), _p(seg_ids), _p(row_ptr), n_seg, ids.numel(), _p(slots_dev),
                               n_slots, _p(vocabs.dev), _p(rows), _p(owner), _stream()), 'er_bucketize_vocab')
    return rows
  if weights is None:
    _lib.check(
        lib.er_bucketize(_p(ids), _p(seg_ids), _p(row_ptr), n_seg, ids.numel(), _p(slots_dev),
                         n_slots, _p(rows), _p(owner), _stream()), 'er_bucketize')
    return rows
  assert weights.numel() >= ids.numel()
  _lib.check(
      lib.er_bucketize_weighted(_p(ids), _p(weights), _p(seg_ids), _p(row_ptr), n_seg, ids.numel(),
                                _p(slots_dev), n_slots, _p(rows), _p(owner), _stream()), 'er_bucketize_weighted')
  return rows


def bucketize_seq(ids, lens, batch, seq_len, slots_dev, n_slots, rows=None, owner=None, vocabs=None):
  """K1 over un-pooled histories (er_bucketize_seq): ids int64 [n_features * batch * seq_len] steps, lens int32
  [n_features * batch].  Steps at or beyond their sample's length come out as rows = owner = -1.  vocabs: as in
  bucketize (er_bucketize_seq_vocab)."""
  lib = _lib.load()
  _chk(ids, torch.int64, 'ids')
  _chk(lens, torch.int32, 'lens')
  _chk(owner, torch.int32, 'owner')
  n_features = lens.numel() // batch
  assert lens.numel() == n_features * batch and ids.numel() == lens.numel() * seq_len
  if rows is None:
    rows = torch.empty_like(ids)
  _chk(rows, torch.int64, 'rows')
  assert rows.numel() == ids.numel() and (owner is None or owner.numel() == ids.numel())
  if vocabs is not None:
    assert len(vocabs.per_slot) == n_slots
    _lib.check(
        lib.er_bucketize_seq_vocab(_p(ids), _p(lens), int(batch), int(seq_len), n_features, _p(slots_dev), n_slots,
                                   _p(vocabs.dev), _p(rows), _p(owner), _stream()), 'er_bucketize_seq_vocab')
    return rows
  _lib.check(
      lib.er_bucketize_seq(_p(ids), _p(lens), int(batch), int(seq_len), n_features, _p(slots_dev), n_slots, _p(rows),
                           _p(owner), _stream()), 'er_bucketize_seq')
  return rows


def kv_find_or_insert(index_keys, index_rows, capacity, stats, keys, rows, weight, state0, state1, state0_init, seed,
                      init_stddev, init_truncated=True, shard_n=1, shard_rank=0):
  """er_kv_find_or_insert: rows = the pool rows of the keys `keys * shard_n + shard_rank` (int64 keys from K1, -1
  dropped); a key seen for the first time takes the next row, initialised from (seed, key) and the optimizer state's
  initial values."""
  for t, nm in ((index_keys, 'index_keys'), (index_rows, 'index_rows'), (stats, 'stats'), (keys, 'keys'), (rows, 'rows')):
    _chk(t, torch.int64, nm)
  assert rows.numel() == keys.numel() and index_rows.numel() == index_keys.numel()
  _, stride = _chk_rows(weight, 'weight')
  for st in (state0, state1):
    if st is not None and _chk_rows(st, 'state')[1] != stride:
      raise _lib.ErError('weight and optimizer state must share one row stride')
  _lib.check(_lib.load().er_kv_find_or_insert(
      _p(index_keys), _p(index_rows), index_keys.numel(), int(capacity), _p(stats), _p(keys), keys.numel(),
      int(shard_n), int(shard_rank), _p(rows), _p(weight), _p(state0), _p(state1), stride, weight.shape[1],
      float(state0_init), int(seed) & (2**64 - 1), float(init_stddev), int(bool(init_truncated)), _stream()),
      'er_kv_find_or_insert')
  return rows


def kv_find(index_keys, index_rows, keys, zero_row, rows, shard_n=1, shard_rank=0):
  """er_kv_find: rows = the pool rows of the keys `keys * shard_n + shard_rank`; keys without a row read `zero_row`,
  nothing is inserted."""
  for t, nm in ((index_keys, 'index_keys'), (index_rows, 'index_rows'), (keys, 'keys'), (rows, 'rows')):
    _chk(t, torch.int64, nm)
  assert rows.numel() == keys.numel()
  _lib.check(_lib.load().er_kv_find(_p(index_keys), _p(index_rows), index_keys.numel(), _p(keys), keys.numel(),
                                    int(shard_n), int(shard_rank), int(zero_row), _p(rows), _stream()), 'er_kv_find')
  return rows


def kv_insert_rows(index_keys, index_rows, keys, rows, stats):
  """er_kv_insert_rows: put distinct `keys` into an empty index with the given pool `rows` (restore)."""
  for t, nm in ((index_keys, 'index_keys'), (index_rows, 'index_rows'), (keys, 'keys'), (rows, 'rows'), (stats, 'stats')):
    _chk(t, torch.int64, nm)
  assert rows.numel() == keys.numel()
  _lib.check(_lib.load().er_kv_insert_rows(_p(index_keys), _p(index_rows), index_keys.numel(), _p(keys), _p(rows),
                                           keys.numel(), _p(stats), _stream()), 'er_kv_insert_rows')


def k1_weight_args(ids, weights):
  """Keyword arguments of bucketize() that hand a weighted CSR call's lookup weights to K1, so that the lookups the
  pooling prunes are dropped before K7, er_mark_rows and K8 see them.  Only device tensors take this path: the host
  runs of the input layer (tests/host_doubles.py) stand in for K1 with a double whose bucketize takes no weights."""
  return {'weights': weights} if weights is not None and ids.is_cuda else {}


def k1_vocab_args(call):
  """Keyword arguments of bucketize() / bucketize_seq() that hand a call's vocabularies to K1 (none for a call without
  vocabulary slots, so that the calls of such plans stay what they were)."""
  return {'vocabs': call.vocabs} if getattr(call, 'vocabs', None) is not None else {}


def dropout(x, rate, seed, counter, out=None):
  """er_dropout: x * Bernoulli(1 - rate) / (1 - rate), mask = f(seed, counter[0], index); counter: device int64 [1]."""
  x = x.contiguous()
  _chk(x, torch.float32, 'x')
  _chk(counter, torch.int64, 'counter')
  y = torch.empty_like(x) if out is None else out
  _lib.check(_lib.load().er_dropout(_p(x), x.numel(), float(rate), int(seed) & (2**64 - 1), _p(counter), _p(y), _stream()),
             'er_dropout')
  return y


ACT_KINDS = {'gelu': _lib.ACT_GELU, 'leaky_relu': _lib.ACT_LEAKY_RELU, 'prelu': _lib.ACT_LEAKY_RELU, 'elu': _lib.ACT_ELU,
             'selu': _lib.ACT_SELU, 'tanh': _lib.ACT_TANH, 'swish': _lib.ACT_SWISH, 'sigmoid': _lib.ACT_SIGMOID}


def act_fwd(x, kind):
  """er_act_fwd: y = f(x), f one of the stateless non-relu activations of utils/activation.py:get_activation."""
  x = x.contiguous()
  _chk(x, torch.float32, 'x')
  y = torch.empty_like(x)
  _lib.check(_lib.load().er_act_fwd(_p(x), x.numel(), int(kind), _p(y), _stream()), 'er_act_fwd')
  return y


def act_bwd(x, gy, kind):
  """er_act_bwd: gx = gy * f'(x), the derivative recomputed from the pre-activation."""
  x, gy = x.contiguous(), gy.contiguous()
  _chk(x, torch.float32, 'x')
  _chk(gy, torch.float32, 'gy')
  assert x.numel() == gy.numel()
  gx = torch.empty_like(x)
  _lib.check(_lib.load().er_act_bwd(_p(x), _p(gy), x.numel(), int(kind), _p(gx), _stream()), 'er_act_bwd')
  return gx


def _chk_dice(x, alpha, **same):
  """x [batch, units]; every tensor in `same` the same shape as x; alpha [units]"""
  if x.dim() != 2:
    raise _lib.ErError('x must be [batch, units], got %s' % (tuple(x.shape),))
  for nm, t in same.items():
    if t.shape != x.shape:
      raise _lib.ErError('%s must have the shape of x %s, got %s' % (nm, tuple(x.shape), tuple(t.shape)))
  if alpha.dim() != 1 or alpha.numel() != x.shape[1]:
    raise _lib.ErError('alpha must be [%d], got %s' % (x.shape[1], tuple(alpha.shape)))


def dice_fwd(x, xn, alpha):
  """er_dice_fwd: alpha * (1 - sigmoid(xn)) * x + sigmoid(xn) * x over [batch, units]."""
  for t, nm in ((x, 'x'), (xn, 'xn'), (alpha, 'alpha')):
    _chk(t, torch.float32, nm)
  _chk_dice(x, alpha, xn=xn)
  y = torch.empty_like(x)
  _lib.check(_lib.load().er_dice_fwd(_p(x), _p(xn), _p(alpha), x.shape[0], x.shape[1], _p(y), _stream()), 'er_dice_fwd')
  return y


def dice_bwd(x, xn, alpha, gy):
  """er_dice_bwd -> (gx_direct, gxn, galpha_terms), each [batch, units]."""
  gy = gy.contiguous()
  for t, nm in ((x, 'x'), (xn, 'xn'), (alpha, 'alpha'), (gy, 'gy')):
    _chk(t, torch.float32, nm)
  _chk_dice(x, alpha, xn=xn, gy=gy)
  gd, gn, ga = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
  _lib.check(_lib.load().er_dice_bwd(_p(x), _p(xn), _p(alpha), _p(gy), x.shape[0], x.shape[1], _p(gd), _p(gn), _p(ga),
                                     _stream()), 'er_dice_bwd')
  return gd, gn, ga


def auc_hist(probs, labels, thresholds, hist):
  """er_auc_hist: one batch into the uint64 confusion histograms behind tf.metrics.auc / max_f1 (hist: int64 tensor of
  2 * (T + 1) counters reinterpreted as uint64; they never approach 2^63)."""
  probs, labels = probs.contiguous().view(-1), labels.contiguous().view(-1)
  _chk(probs, torch.float32, 'probs')
  _chk(labels, torch.float32, 'labels')
  _chk(thresholds, torch.float32, 'thresholds')
  _chk(hist, torch.int64, 'hist')
  assert probs.numel() == labels.numel() and hist.numel() == 2 * (thresholds.numel() + 1)
  _lib.check(_lib.load().er_auc_hist(_p(probs), _p(labels), probs.numel(), _p(thresholds), thresholds.numel(), _p(hist),
                                     _stream()), 'er_auc_hist')
  return hist


class ExprPlan(object):
  """The programs of a model's ExprFeatures (expr.Program) packed for er_expr_eval: one device array holding their
  er_expr_t descriptors, then their er_expr_op_t ops; out_cols[e] is the dense_fea column of expression e.  Each program
  is checked on the host: its opcodes, its input indices against n_inputs and the stack it needs."""

  def __init__(self, programs, out_cols, n_inputs, device):
    self.n_expr, self.n_inputs = len(programs), int(n_inputs)
    self.n_ops = sum(len(p.ops) for p in programs)
    self.max_depth = max([p.depth for p in programs] + [0])
    if self.n_ops > _lib.EXPR_MAX_OPS or self.max_depth > _lib.EXPR_MAX_STACK:
      raise _lib.ErError('ExprFeature programs: %d ops and a stack of %d, at most %d and %d'
                         % (self.n_ops, self.max_depth, _lib.EXPR_MAX_OPS, _lib.EXPR_MAX_STACK))
    desc = np.zeros(self.n_expr, dtype=_lib.EXPR_DTYPE)
    ops = np.zeros(self.n_ops, dtype=_lib.EXPR_OP_DTYPE)
    k = 0
    for e, (p, col) in enumerate(zip(programs, out_cols)):
      desc[e] = (k, len(p.ops), col, 0)
      depth = 0
      for op, arg, value in p.ops:
        pushes = op in (expr.EXPR_LOAD, expr.EXPR_CONST)
        if not 0 <= op <= expr.EXPR_OR or (op == expr.EXPR_LOAD and not 0 <= arg < self.n_inputs):
          raise _lib.ErError('ExprFeature program %d: op %d with input %d of %d' % (e, op, arg, self.n_inputs))
        depth += 1 if pushes else (0 if op == expr.EXPR_NEG else -1)
        if depth < 1 or depth > p.depth:
          raise _lib.ErError('ExprFeature program %d: its stack leaves [1, %d]' % (e, p.depth))
        ops[k] = (op, arg if op == expr.EXPR_LOAD else 0, value)
        k += 1
      if depth != 1:
        raise _lib.ErError('ExprFeature program %d leaves %d values' % (e, depth))
    blob = np.concatenate([desc.view(np.uint8), ops.view(np.uint8)]).view(np.int64)
    self.dev = torch.from_numpy(blob.copy()).to(device)


def expr_plan(programs, out_cols, n_inputs, device):
  """ExprPlan on the device.  er_expr_eval runs on the GPU only, so a host device is refused (a plan built with
  ER_PLAN_ONLY=1 only to be inspected is packed all the same)."""
  if not str(device).startswith('cuda') and os.environ.get('ER_PLAN_ONLY') != '1':
    raise NotImplementedError('ExprFeature columns are evaluated by er_expr_eval on the GPU; device %s has none' % device)
  return ExprPlan(programs, out_cols, n_inputs, device)


def expr_eval(plan, inputs, dense):
  """er_expr_eval: inputs float64 [B, n_inputs] -> each ExprFeature's float32 value into its column of dense
  float32 [B, n_dense], in place."""
  _chk(inputs, torch.float64, 'expr inputs')
  _chk(dense, torch.float32, 'dense_fea')
  B = dense.shape[0]
  if inputs.dim() != 2 or inputs.shape[0] != B or inputs.shape[1] != plan.n_inputs:
    raise _lib.ErError('expr inputs must be float64 [%d, %d], got %s' % (B, plan.n_inputs, tuple(inputs.shape)))
  base = plan.dev.data_ptr()
  _lib.check(_lib.load().er_expr_eval(_p(inputs), B, plan.n_inputs, base, plan.n_expr, base + 16 * plan.n_expr,
                                      plan.n_ops, plan.max_depth, _p(dense), dense.shape[1], _stream()),
             'er_expr_eval')
  return dense


def binary_maps(slot_cols, raw_cols, device):
  """the column maps of er_binary_unpack as device int32 tensors, each entry checked against its range on the host (the
  kernel reads them from device memory unchecked)"""
  out = []
  for cols, hi, nm in ((slot_cols, _lib.CRITEO_N_CAT, 'slot_cols'), (raw_cols, _lib.CRITEO_N_DENSE, 'raw_cols')):
    a = np.asarray(cols, np.int64).reshape(-1)
    if a.size and (a.min() < 0 or a.max() >= hi):
      raise _lib.ErError('%s entries must be in [0, %d)' % (nm, hi))
    out.append(torch.from_numpy(a.astype(np.int32)).to(device))
  if out[1].numel() > _lib.CRITEO_N_DENSE:
    raise _lib.ErError('raw_cols has %d entries, at most %d' % (out[1].numel(), _lib.CRITEO_N_DENSE))
  return tuple(out)


def binary_unpack(label, dense, cat, slot_cols, raw_cols, sparse_fea=None, dense_fea=None, labels=None):
  """er_binary_unpack: one CriteoInput batch (label int32 [B], dense fp32 [B, 13], cat int32 [B, 26] holding the uint32
  bits) -> (sparse_fea int64 [n_slot * B] feature-major, dense_fea fp32 [B, n_raw], labels fp32 [B]).  slot_cols /
  raw_cols: device int32 maps from binary_maps.  Outputs are written into the given tensors when passed."""
  B = label.numel()
  _chk(label, torch.int32, 'label')
  _chk(dense, torch.float32, 'dense')
  _chk(cat, torch.int32, 'cat')
  _chk(slot_cols, torch.int32, 'slot_cols')
  _chk(raw_cols, torch.int32, 'raw_cols')
  if dense.numel() != B * _lib.CRITEO_N_DENSE or cat.numel() != B * _lib.CRITEO_N_CAT:
    raise _lib.ErError('dense / cat must hold 13 / 26 values per label')
  n_slot, n_raw = slot_cols.numel(), raw_cols.numel()
  dev = label.device
  sparse_fea = torch.empty(n_slot * B, dtype=torch.int64, device=dev) if sparse_fea is None else sparse_fea
  dense_fea = torch.empty((B, n_raw), dtype=torch.float32, device=dev) if dense_fea is None else dense_fea
  labels = torch.empty(B, dtype=torch.float32, device=dev) if labels is None else labels
  _chk(sparse_fea, torch.int64, 'sparse_fea')
  _chk(dense_fea, torch.float32, 'dense_fea')
  _chk(labels, torch.float32, 'labels')
  assert sparse_fea.numel() == n_slot * B and dense_fea.numel() == B * n_raw and labels.numel() == B
  _lib.check(_lib.load().er_binary_unpack(_p(label), _p(dense), _p(cat), B, _p(slot_cols), n_slot, _p(raw_cols), n_raw,
                                          _p(sparse_fea), _p(dense_fea), _p(labels), _stream()), 'er_binary_unpack')
  return sparse_fea, dense_fea.view(B, n_raw), labels


def shard_group_workspace(n_lookups, device):
  return torch.empty(_lib.load().er_shard_group_workspace_bytes(int(n_lookups)), dtype=torch.uint8, device=device)


def shard_group(rows, owner, world, cap_per_peer, send_rows, pos, counts, ws):
  """K8 (er_shard_group): distinct (owner, row) pairs into fixed-capacity per-owner blocks; see include/er_b200.h."""
  _chk(rows, torch.int64, 'rows')
  _chk(owner, torch.int32, 'owner')
  _chk(send_rows, torch.int64, 'send_rows')
  _chk(pos, torch.int64, 'pos')
  _chk(counts, torch.int32, 'counts')
  assert send_rows.numel() == world * cap_per_peer and pos.numel() == rows.numel() and counts.numel() == world + 1
  _lib.check(_lib.load().er_shard_group(_p(rows), _p(owner), rows.numel(), int(world), int(cap_per_peer), _p(send_rows),
                                        _p(pos), _p(counts), _p(ws), ws.numel(), _stream()), 'er_shard_group')


def embedding_fwd(table, dim, rows, slots_dev, n_slots, n_seg, out_bufs, weights=None,
                  row_ptr=None, seg_scale=None, row_stride=None):
  lib = _lib.load()
  n_rows, row_stride = _chk_rows(table, 'table')
  _chk(rows, torch.int64, 'rows')
  _chk(weights, torch.float32, 'weights')
  _chk(row_ptr, torch.int32, 'row_ptr')
  _chk(seg_scale, torch.float32, 'seg_scale')
  for i, b in enumerate(out_bufs):
    _chk(b, torch.float32, 'out_bufs[%d]' % i)
  _lib.check(
      lib.er_embedding_fwd(_p(table), n_rows, dim, row_stride, _p(rows), _p(weights), _p(row_ptr),
                           n_seg, rows.numel(), _p(slots_dev), n_slots, _buf_array(out_bufs),
                           len(out_bufs), _p(seg_scale), _stream()), 'er_embedding_fwd')


def bwd_workspace(n_lookups_cap, device, dim):
  lib = _lib.load()
  return torch.empty(lib.er_embedding_bwd_workspace_bytes(n_lookups_cap, dim), dtype=torch.uint8,
                     device=device)


def make_opt(kind, lr, beta1=0.9, beta2=0.999, eps=1e-8, beta1_power=0.9, beta2_power=0.999,
             grad_scale=1.0, hyper_dev=None):
  """er_opt_t.  hyper_dev: device float[HYPER_N] the kernels read lr / beta powers / grad_scale from instead of
  the struct fields (which the caller keeps equal to it), so a captured graph follows the schedule."""
  return ErOpt(kind, lr, beta1, beta2, eps, beta1_power, beta2_power, grad_scale, _p(hyper_dev))


class StepHyper(object):
  """The step-varying scalars of the optimizers - learning rate (core/learning_schedules.py:30-75), Adam's
  beta1^t / beta2^t (fp32 accumulators multiplied once per step like TF's `_finish`, compat/adam_s.py:233-245)
  and the sparse gradient scale (1/N for sharded tables x embedding_learning_rate_multiplier) - in ONE device
  float[HYPER_N], refreshed by one 16-byte stream-ordered copy per step (from a fresh pageable host tensor: the
  driver stages it before returning, so the host may run any number of steps ahead of the device)."""

  def __init__(self, device, beta1=0.9, beta2=0.999):
    self.device = device
    self.beta1, self.beta2 = np.float32(beta1), np.float32(beta2)
    self.dev = torch.zeros(_lib.HYPER_N, dtype=torch.float32, device=device)
    self._pow_step = None
    self.b1p = self.b2p = None
    self.lr = 0.0
    self.grad_scale = 1.0

  def _powers(self, step):
    """beta^(step+1) by repeated fp32 multiplication (what the TF variables hold before step `step`)."""
    if self._pow_step is not None and step == self._pow_step + 1:
      self.b1p = np.float32(self.b1p * self.beta1)
      self.b2p = np.float32(self.b2p * self.beta2)
    elif self._pow_step is None or step != self._pow_step:
      b1p, b2p = self.beta1, self.beta2
      for _ in range(int(step)):
        b1p = np.float32(b1p * self.beta1)
        b2p = np.float32(b2p * self.beta2)
      self.b1p, self.b2p = b1p, b2p
    self._pow_step = step

  def set(self, lr, step, grad_scale=1.0):
    self._powers(step)
    self.lr, self.grad_scale = float(np.float32(lr)), float(np.float32(grad_scale))
    h = [0.0] * _lib.HYPER_N
    h[_lib.HYPER_LR] = self.lr
    h[_lib.HYPER_BETA1_POWER] = float(self.b1p)
    h[_lib.HYPER_BETA2_POWER] = float(self.b2p)
    h[_lib.HYPER_GRAD_SCALE] = self.grad_scale
    self.dev.copy_(torch.tensor(h, dtype=torch.float32), non_blocking=True)

  def opt(self, kind, eps=1e-8, grad_scale=None):
    """er_opt_t for `kind` carrying both the values and the device block."""
    return make_opt(kind, self.lr, float(self.beta1), float(self.beta2), eps, float(self.b1p), float(self.b2p),
                    self.grad_scale if grad_scale is None else grad_scale, hyper_dev=self.dev)


def embedding_bwd(table, state0, state1, dim, rows, slots_dev, n_slots, n_seg, grad_bufs, opt,
                  ws, weights=None, seg_ids=None, row_ptr=None, seg_scale=None, row_stride=None,
                  uniq_rows=None, uniq_grads=None, n_uniq=None, n_rows=None, sorted_from=None):
  """sorted_from = (ws, dim) of an earlier embedding_bwd on this stream over the SAME rows tensor, n_rows and placement
  mode (k7_warp_mode): its bucket placement is reused (er_embedding_bwd_reuse_sort)."""
  lib = _lib.load()
  row_stride = dim
  if table is not None:
    n_rows_t, row_stride = _chk_rows(table, 'table')
    n_rows = n_rows if n_rows is not None else n_rows_t
    for st, nm in ((state0, 'state0'), (state1, 'state1')):
      if st is not None and _chk_rows(st, nm)[1] != row_stride:
        raise _lib.ErError('%s must share the table row stride' % nm)
  _chk(rows, torch.int64, 'rows')
  _chk(weights, torch.float32, 'weights')
  _chk(seg_ids, torch.int32, 'seg_ids')
  _chk(row_ptr, torch.int32, 'row_ptr')
  _chk(seg_scale, torch.float32, 'seg_scale')
  _chk(uniq_rows, torch.int64, 'uniq_rows')
  _chk(uniq_grads, torch.float32, 'uniq_grads')
  _chk(n_uniq, torch.int32, 'n_uniq')
  for i, b in enumerate(grad_bufs):
    _chk(b, torch.float32, 'grad_bufs[%d]' % i)
  if sorted_from is not None:
    src_ws, src_dim = sorted_from
    _lib.check(
        lib.er_embedding_bwd_reuse_sort(_p(table), _p(state0), _p(state1), n_rows, dim, row_stride, _p(rows),
                                        _p(weights), _p(seg_ids), _p(row_ptr), n_seg, rows.numel(),
                                        _p(slots_dev), n_slots, _buf_array(grad_bufs), len(grad_bufs),
                                        _p(seg_scale), ctypes.byref(opt), _p(uniq_rows), _p(uniq_grads),
                                        _p(n_uniq), _p(ws), ws.numel(), _p(src_ws), src_ws.numel(), src_dim,
                                        _stream()), 'er_embedding_bwd_reuse_sort')
    return
  _lib.check(
      lib.er_embedding_bwd(_p(table), _p(state0), _p(state1), n_rows, dim, row_stride, _p(rows),
                           _p(weights), _p(seg_ids), _p(row_ptr), n_seg, rows.numel(),
                           _p(slots_dev), n_slots, _buf_array(grad_bufs), len(grad_bufs),
                           _p(seg_scale), ctypes.byref(opt), _p(uniq_rows), _p(uniq_grads),
                           _p(n_uniq), _p(ws), ws.numel(), _stream()), 'er_embedding_bwd')


def k7_warp_mode(dim):
  """mirror of k7_warp_mode in csrc/embedding_bwd.cu: tables whose rows one warp can stage."""
  return dim in (1, 4, 8, 16, 32)


def embedding_bwd_presort(rows, n_rows, dim, ws, slots_dev, n_slots, seg_ids=None, row_ptr=None, n_seg=0):
  """The row-only half of K7's dedup (hashing the lookups into buckets), with the same rows / seg_ids / slots as the
  embedding_bwd it prepares: finish with embedding_bwd(..., sorted_from=(ws, dim))."""
  lib = _lib.load()
  _chk(rows, torch.int64, 'rows')
  _chk(seg_ids, torch.int32, 'seg_ids')
  _lib.check(lib.er_embedding_bwd_presort(_p(rows), n_rows, _p(seg_ids), _p(row_ptr), n_seg, rows.numel(),
                                          _p(slots_dev), n_slots, dim, _p(ws), ws.numel(), _stream()),
             'er_embedding_bwd_presort')


def sparse_apply(table, state0, state1, dim, uniq_rows, uniq_grads, n_uniq, opt, row_stride=None):
  lib = _lib.load()
  _, row_stride = _chk_rows(table, 'table')
  _lib.check(
      lib.er_sparse_apply(_p(table), _p(state0), _p(state1), dim, row_stride, _p(uniq_rows),
                          _p(uniq_grads), _p(n_uniq), uniq_rows.numel(), ctypes.byref(opt),
                          _stream()), 'er_sparse_apply')


def adam_dense_sweep(table, m, v, dim, touched, opt, row_stride=None):
  lib = _lib.load()
  n_rows_t, row_stride = _chk_rows(table, 'table')
  _lib.check(
      lib.er_adam_dense_sweep(_p(table), _p(m), _p(v), n_rows_t, dim,
                              row_stride, _p(touched), ctypes.byref(opt), _stream()),
      'er_adam_dense_sweep')


def mark_rows(rows, n_rows, touched, value, n_dev=None):
  lib = _lib.load()
  _lib.check(
      lib.er_mark_rows(_p(rows), rows.numel(), _p(n_dev), n_rows, _p(touched), value, _stream()),
      'er_mark_rows')


def sort_rows(rows, max_row, n_dev=None):
  lib = _lib.load()
  _chk(rows, torch.int64, 'rows')
  n = rows.numel()
  keys = torch.empty(n, dtype=torch.int32, device=rows.device)
  vals = torch.empty(n, dtype=torch.int32, device=rows.device)
  ws_bytes = lib.er_sort_workspace_bytes(n)
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device=rows.device)
  _lib.check(
      lib.er_sort_rows(_p(rows), n, _p(n_dev), max_row, _p(keys), _p(vals), _p(ws), ws_bytes,
                       _stream()), 'er_sort_rows')
  return keys, vals


def fm_fwd(x, n_field, dim, y=None):
  lib = _lib.load()
  _chk(x, torch.float32, 'x')
  batch = x.shape[0]
  if y is None:
    y = torch.empty(batch, dim, dtype=torch.float32, device=x.device)
  _lib.check(lib.er_fm_fwd(_p(x), batch, n_field, dim, x.stride(0), _p(y), _stream()), 'er_fm_fwd')
  return y


def fm_bwd(x, gy, n_field, dim, gx=None, accumulate=False):
  lib = _lib.load()
  _chk(x, torch.float32, 'x')
  _chk(gy, torch.float32, 'gy')
  batch = x.shape[0]
  if gx is None:
    gx = torch.empty(batch, n_field * dim, dtype=torch.float32, device=x.device)
    accumulate = False
  _lib.check(
      lib.er_fm_bwd(_p(x), _p(gy), batch, n_field, dim, x.stride(0), _p(gx), gx.stride(0),
                    1 if accumulate else 0, _stream()), 'er_fm_bwd')
  return gx


def fm_block_ok(n_field, dim):
  d4 = dim // 4
  return dim % 4 == 0 and 1 <= d4 <= 32 and (d4 & (d4 - 1)) == 0 and n_field * d4 <= 256


_fm_ws = {}


def fm_block_fwd(x, n_field, dim, want_sumsq=True):
  """(y [B, dim], sumsq [1] or None): FM second order and sum(x^2) in one pass over the group matrix."""
  lib = _lib.load()
  if x.dtype != torch.float32 or x.stride(1) != 1:
    raise _lib.ErError('x must be float32 with unit column stride')
  batch = x.shape[0]
  y = torch.empty(batch, dim, dtype=torch.float32, device=x.device)
  sumsq = ws = None
  if want_sumsq:
    sumsq = torch.empty(1, dtype=torch.float32, device=x.device)
    ws = _fm_ws.get(x.device)
    if ws is None:
      ws = torch.zeros(lib.er_fm_block_workspace_bytes(batch), dtype=torch.uint8, device=x.device)
      _fm_ws[x.device] = ws
  _lib.check(lib.er_fm_block_fwd(_p(x), batch, n_field, dim, x.stride(0), _p(y), _p(sumsq), _p(ws),
                                 0 if ws is None else ws.numel(), _stream()), 'er_fm_block_fwd')
  return y, sumsq


def fm_block_bwd(x, gy, g_pass, coef_dev, coef_mul, n_field, dim):
  """gx [B, F*dim] = g_pass + gy*(S - x) + coef*x (any of the three sources may be None)."""
  lib = _lib.load()
  batch = x.shape[0]
  gx = torch.empty(batch, n_field * dim, dtype=torch.float32, device=x.device)
  if g_pass is not None and g_pass.stride(1) != 1:
    g_pass = g_pass.contiguous()
  _lib.check(lib.er_fm_block_bwd(_p(x), _p(gy), _p(g_pass), _p(coef_dev), coef_mul, batch, n_field, dim,
                                 x.stride(0), 0 if g_pass is None else g_pass.stride(0), _p(gx), gx.stride(0),
                                 _stream()), 'er_fm_block_bwd')
  return gx


_blk_ws = {}


def _zero_ws(key, nbytes, device):
  ws = _blk_ws.get((key, device))
  if ws is None or ws.numel() < nbytes:
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=device)   # tickets start at zero, kernels leave them zero
    _blk_ws[(key, device)] = ws
  return ws


def rowsum_block_fwd(x, want_sumsq=True):
  """(y [B], sumsq [1] or None): row sums of a [B, F] matrix and sum(x^2) in one pass."""
  lib = _lib.load()
  batch, width = x.shape
  y = torch.empty(batch, dtype=torch.float32, device=x.device)
  sumsq = ws = None
  if want_sumsq:
    sumsq = torch.empty(1, dtype=torch.float32, device=x.device)
    ws = _zero_ws('rowsum', lib.er_fm_block_workspace_bytes(batch), x.device)
  _lib.check(lib.er_rowsum_block_fwd(_p(x), batch, width, x.stride(0), _p(y), _p(sumsq), _p(ws),
                                     0 if ws is None else ws.numel(), _stream()), 'er_rowsum_block_fwd')
  return y, sumsq


def rowsum_block_bwd(x, gy, coef_dev, coef_mul):
  lib = _lib.load()
  batch, width = x.shape
  gx = torch.empty(batch, width, dtype=torch.float32, device=x.device)
  _lib.check(lib.er_rowsum_block_bwd(_p(x), _p(gy), _p(coef_dev), coef_mul, batch, width, x.stride(0), _p(gx),
                                     gx.stride(0), _stream()), 'er_rowsum_block_bwd')
  return gx


def dense1_fwd(x, w, bias):
  lib = _lib.load()
  batch, width = x.shape
  y = torch.empty(batch, 1, dtype=torch.float32, device=x.device)
  _lib.check(lib.er_dense1_fwd(_p(x), _p(w), _p(bias), batch, width, x.stride(0), _p(y), _stream()), 'er_dense1_fwd')
  return y


def dense1_bwd(x, w, g, need_gx=True):
  lib = _lib.load()
  batch, width = x.shape
  gx = torch.empty(batch, width, dtype=torch.float32, device=x.device) if need_gx else None
  gw = torch.empty(width, 1, dtype=torch.float32, device=x.device)
  gb = torch.empty(1, dtype=torch.float32, device=x.device)
  ws = _zero_ws('dense1', lib.er_dense1_workspace_bytes(width), x.device)
  _lib.check(lib.er_dense1_bwd(_p(x), _p(w), _p(g), batch, width, x.stride(0), _p(gx), width, _p(gw), _p(gb),
                               _p(ws), ws.numel(), _stream()), 'er_dense1_bwd')
  return gx, gw, gb


def _cat_arrays(mats):
  n = len(mats)
  ptrs = (c_vp * n)(*[m.data_ptr() for m in mats])
  widths = (ctypes.c_int32 * n)(*[m.shape[1] for m in mats])
  strides = (ctypes.c_int32 * n)(*[m.stride(0) for m in mats])
  return ptrs, widths, strides, n


def concat_cols(mats, pitch_multiple=4):
  """[B, w_i] matrices -> view [B, sum w] of a pitched buffer [B, ceil_k(sum w)] (padding written as zeros)."""
  lib = _lib.load()
  mats = [m if m.stride(1) == 1 else m.contiguous() for m in mats]
  batch = mats[0].shape[0]
  total = sum(m.shape[1] for m in mats)
  pitch = (total + pitch_multiple - 1) // pitch_multiple * pitch_multiple
  dst = torch.empty(batch, pitch, dtype=torch.float32, device=mats[0].device)
  ptrs, widths, strides, n = _cat_arrays(mats)
  _lib.check(lib.er_concat_cols(ptrs, widths, strides, n, batch, _p(dst), pitch, _stream()), 'er_concat_cols')
  return dst[:, :total]


def split_cols(src, widths):
  """inverse of concat_cols: contiguous [B, w_i] pieces of the columns of src."""
  lib = _lib.load()
  if src.stride(1) != 1:
    src = src.contiguous()
  batch = src.shape[0]
  outs = [torch.empty(batch, w, dtype=torch.float32, device=src.device) for w in widths]
  ptrs, warr, strides, n = _cat_arrays(outs)
  _lib.check(lib.er_split_cols(_p(src), src.stride(0), batch, ptrs, warr, strides, n, _stream()), 'er_split_cols')
  return outs


def sigmoid_ce(logits, labels, weights=None, inv_count=None, want_grad=True):
  """returns (loss [1], probs [B], g_logits [B])."""
  lib = _lib.load()
  _chk(logits, torch.float32, 'logits')
  _chk(labels, torch.float32, 'labels')
  batch = logits.numel()
  if inv_count is None:
    inv_count = 1.0 / batch
  loss = torch.empty(1, dtype=torch.float32, device=logits.device)
  probs = torch.empty(batch, dtype=torch.float32, device=logits.device)
  g = torch.empty(batch, dtype=torch.float32, device=logits.device) if want_grad else None
  _lib.check(
      lib.er_sigmoid_ce_fwd_bwd(_p(logits), _p(labels), _p(weights), batch, inv_count, _p(loss),
                                _p(probs), _p(g), _stream()), 'er_sigmoid_ce_fwd_bwd')
  return loss, probs, g


def _gemm_operand(t, name):
  """2-D fp32 tensor -> (tensor, pitch, contiguous_index) with contiguous_index 1 if dim 1 is the unit-stride one.
  Copies only when the view cannot be read in place (pitch not a multiple of 4 floats / misaligned)."""
  if t.dtype != torch.float32 or t.dim() != 2:
    raise _lib.ErError('%s must be a 2-D float32 tensor' % name)
  for _ in range(2):
    if t.stride(1) == 1 and t.stride(0) % 4 == 0 and t.stride(0) >= t.shape[1] and t.data_ptr() % 16 == 0:
      return t, t.stride(0), 1
    if t.stride(0) == 1 and t.stride(1) % 4 == 0 and t.stride(1) >= t.shape[0] and t.data_ptr() % 16 == 0:
      return t, t.stride(1), 0
    if t.shape[1] % 4:   # pad the pitch: [r, c] -> view of [r, ceil4(c)]
      buf = torch.zeros(t.shape[0], (t.shape[1] + 3) // 4 * 4, dtype=torch.float32, device=t.device)
      buf[:, :t.shape[1]].copy_(t)
      t = buf[:, :t.shape[1]]
    else:
      t = t.contiguous() if not t.is_contiguous() else t.clone()   # clone: a 16-byte aligned allocation
  raise ValueError('%s: cannot be laid out for er_gemm' % name)


def gemm_ready(t):
  """A tensor er_gemm can read in place (and its transpose too): identity for 16-byte aligned rows with a
  pitch that is a multiple of 4 floats, else one padded copy.  Layers call it once in forward and save the
  result, so forward, dX and dW all read the same buffer."""
  return _gemm_operand(t, 'x')[0]


_gemm_ws = {}


def gemm(a, b, bias=None, out=None, planes=None):
  """out[M,N] = a[M,K] @ b[K,N] (+ bias) on the tensor cores (3xTF32).  a / b may be transposed views.
  planes: b's pre-split (hi, lo) planes (DensePlanes.view), read instead of b; the result is bit-identical."""
  lib = _lib.load()
  M, Ka = a.shape
  Kb, N = b.shape
  assert Ka == Kb, (a.shape, b.shape)
  if N < 8 or Ka < 8 or M < 8:
    # vector-sized problems (MMoE gates [d -> num_expert], their dX and dW): er_gemm_small on the CUDA cores, operands
    # read through their strides (transposed views in place); a 128x128 tensor-core tile would be all padding
    return gemm_small(a, b, bias, out)
  a, lda, a_unit = _gemm_operand(a, 'a')      # a_unit == 1: k contiguous -> K-major
  if planes is None:
    b, ldb, b_unit = _gemm_operand(b, 'b')    # b_unit == 1: n contiguous -> MN-major
  if out is None:
    out = torch.empty(M, N, dtype=torch.float32, device=a.device)
  assert out.stride(1) == 1
  nbytes = lib.er_gemm_workspace_bytes(M, N, Ka)
  ws = None
  if nbytes:
    key = (a.device, torch.cuda.current_stream().cuda_stream if a.is_cuda else 0)
    ws = _gemm_ws.get(key)
    if ws is None or ws.numel() < nbytes:
      ws = torch.empty(nbytes, dtype=torch.uint8, device=a.device)
      _gemm_ws[key] = ws
  if planes is not None:
    _lib.check(lib.er_gemm_planes(_p(a), lda, 0 if a_unit else 1, _p(planes[0]), _p(planes[1]), _p(bias), _p(out),
                                  out.stride(0), M, N, Ka, None, _p(ws), 0 if ws is None else ws.numel(), _stream()),
               'er_gemm_planes')
    return out
  _lib.check(lib.er_gemm(_p(a), lda, 0 if a_unit else 1, _p(b), ldb, 1 if b_unit else 0, _p(bias), _p(out),
                         out.stride(0), M, N, Ka, _p(ws), 0 if ws is None else ws.numel(), _stream()), 'er_gemm')
  return out


def gemm_small(a, b, bias=None, out=None):
  """er_gemm_small: out[M,N] = a[M,K] @ b[K,N] (+ bias) for vector-sized shapes; any strides."""
  lib = _lib.load()
  M, Ka = a.shape
  _, N = b.shape
  for t, name in ((a, 'a'), (b, 'b')):
    if not t.is_cuda or t.dtype != torch.float32:
      raise _lib.ErError('%s must be a CUDA fp32 matrix (no CPU fallback)' % name)
  _chk(bias, torch.float32, 'bias')
  if out is None:
    out = torch.empty(M, N, dtype=torch.float32, device=a.device)
  assert out.shape == (M, N) and out.stride(1) == 1 and out.is_cuda and out.dtype == torch.float32
  nbytes = lib.er_gemm_small_workspace_bytes(M, N, Ka)
  ws = None
  if nbytes:
    key = (a.device, torch.cuda.current_stream().cuda_stream, 'small')
    ws = _gemm_ws.get(key)
    if ws is None or ws.numel() < nbytes:
      ws = torch.empty(nbytes, dtype=torch.uint8, device=a.device)
      _gemm_ws[key] = ws
  _lib.check(lib.er_gemm_small(_p(a), a.stride(0), a.stride(1), _p(b), b.stride(0), b.stride(1), _p(bias), _p(out),
                               out.stride(0), M, N, Ka, _p(ws), 0 if ws is None else ws.numel(), _stream()),
             'er_gemm_small')
  return out


_gemm_bn_ws = {}


def gemm_bn(a, b, bias, moving_mean, moving_var, eps, momentum, planes=None):
  """z = a @ b on the tensor cores, with the batch-norm statistics of z + bias from the GEMM epilogue.
  Returns (z, save_mean, save_rstd), or None when the problem would be split along K (caller falls back).
  planes: b's pre-split (hi, lo) planes (DensePlanes.view), read instead of b; the result is bit-identical."""
  lib = _lib.load()
  M, Ka = a.shape
  Kb, N = b.shape
  assert Ka == Kb, (a.shape, b.shape)
  if N < 8 or Ka < 8 or M < 8 or lib.er_gemm_workspace_bytes(M, N, Ka) != 0:
    return None
  a, lda, a_unit = _gemm_operand(a, 'a')
  if planes is None:
    b, ldb, b_unit = _gemm_operand(b, 'b')
  z = torch.empty(M, N, dtype=torch.float32, device=a.device)
  mean = torch.empty(N, dtype=torch.float32, device=a.device)
  rstd = torch.empty(N, dtype=torch.float32, device=a.device)
  nbytes = lib.er_gemm_bn_workspace_bytes(M, N)
  key = (a.device, torch.cuda.current_stream().cuda_stream if a.is_cuda else 0)
  ws = _gemm_bn_ws.get(key)
  if ws is None or ws.numel() < nbytes:
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=a.device)   # counters must start at zero
    _gemm_bn_ws[key] = ws
  bn = _lib.ErBnStats(_p(bias), _p(mean), _p(rstd), _p(moving_mean), _p(moving_var), eps, momentum)
  if planes is not None:
    _lib.check(lib.er_gemm_planes(_p(a), lda, 0 if a_unit else 1, _p(planes[0]), _p(planes[1]), None, _p(z),
                                  z.stride(0), M, N, Ka, ctypes.byref(bn), _p(ws), ws.numel(), _stream()),
               'er_gemm_planes')
    return z, mean, rstd
  _lib.check(lib.er_gemm_bn(_p(a), lda, 0 if a_unit else 1, _p(b), ldb, 1 if b_unit else 0, _p(z), z.stride(0),
                            M, N, Ka, ctypes.byref(bn), _p(ws), ws.numel(), _stream()), 'er_gemm_bn')
  return z, mean, rstd


class DensePlanes(object):
  """Pre-split tf32 hi / lo planes of dense-layer kernels W[in, out], in the layout er_gemm_planes reads: per kernel
  the planes of W^T (rows = out, k = in: the forward's B) and of W (rows = in, k = out: dX's B), in one buffer.
  refresh() re-splits every kernel from its current values in one launch; it reads the tensors' storage, so a
  kernel must stay the same storage (a view that is written in place) for as long as its planes are used."""

  def __init__(self, kernels, device):
    lib = _lib.load()
    self.kernels = list(kernels)
    for w in self.kernels:
      assert w.dim() == 2 and w.dtype == torch.float32 and w.is_cuda and w.is_contiguous()
    jobs = []
    for w in self.kernels:
      n_in, n_out = w.shape
      jobs.append((n_out, n_in, 1, n_out))   # W^T: rows out, k in
      jobs.append((n_in, n_out, n_out, 1))   # W: rows in, k out
    sizes = [int(lib.er_gemm_plane_floats(rows, k)) for rows, k, _, _ in jobs]
    self.buf = torch.empty(2 * sum(sizes), dtype=torch.float32, device=device)
    self.planes = []
    self.jobs = (_lib.ErGemmPlane * len(jobs))()
    off = 0
    for i, ((rows, k, ld_row, ld_k), n) in enumerate(zip(jobs, sizes)):
      hi, lo = self.buf[off:off + n], self.buf[off + n:off + 2 * n]
      off += 2 * n
      self.planes.append((hi, lo))
      self.jobs[i] = _lib.ErGemmPlane(_p(self.kernels[i // 2]), ld_row, ld_k, rows, k, _p(hi), _p(lo))

  def refresh(self):
    _lib.check(_lib.load().er_gemm_split_planes(self.jobs, len(self.planes), _stream()), 'er_gemm_split_planes')

  def view(self, i, transposed):
    """(hi, lo) of kernel i: transposed=False for the forward (B = W), True for dX (B = W^T)."""
    return self.planes[2 * i + (1 if transposed else 0)]


def bn_act_apply(z, bias, gamma, beta, mean, rstd, relu, y=None):
  lib = _lib.load()
  _chk(z, torch.float32, 'z')
  batch, units = z.shape
  if y is None:
    y = torch.empty_like(z)
  _lib.check(lib.er_bn_act_apply(_p(z), _p(bias), _p(gamma), _p(beta), _p(mean), _p(rstd), batch, units,
                                 1 if relu else 0, _p(y), _stream()), 'er_bn_act_apply')
  return y


def dense_workspace(batch, units, device):
  lib = _lib.load()
  # zero-filled: the head of the workspace holds the backward's CTA tickets (self-resetting)
  return torch.zeros(lib.er_dense_workspace_bytes(batch, units), dtype=torch.uint8, device=device)


def bias_bn_act_fwd(z, bias, gamma, beta, moving_mean, moving_var, eps, momentum, training, relu,
                    ws, y=None, save_mean=None, save_rstd=None):
  """y = act(bn(z + bias)) (gamma None: no batch norm). Returns (y, save_mean, save_rstd)."""
  lib = _lib.load()
  _chk(z, torch.float32, 'z')
  batch, units = z.shape
  if y is None:
    y = torch.empty_like(z)
  if gamma is not None and training and save_mean is None:
    save_mean = torch.empty(units, dtype=torch.float32, device=z.device)
    save_rstd = torch.empty(units, dtype=torch.float32, device=z.device)
  _lib.check(
      lib.er_bias_bn_act_fwd(_p(z), _p(bias), _p(gamma), _p(beta), _p(moving_mean), _p(moving_var),
                             batch, units, eps, momentum, 1 if training else 0, 1 if relu else 0,
                             _p(y), _p(save_mean), _p(save_rstd), _p(ws), ws.numel(), _stream()),
      'er_bias_bn_act_fwd')
  return y, save_mean, save_rstd


def bias_bn_act_bwd(z, bias, gamma, y, gy, save_mean, save_rstd, relu, ws):
  """Returns (gz, gbias, ggamma, gbeta)."""
  lib = _lib.load()
  _chk(gy, torch.float32, 'gy')
  batch, units = z.shape
  gz = torch.empty_like(z)
  gbias = torch.empty(units, dtype=torch.float32, device=z.device)
  ggamma = torch.empty(units, dtype=torch.float32, device=z.device) if gamma is not None else None
  gbeta = torch.empty(units, dtype=torch.float32, device=z.device) if gamma is not None else None
  _lib.check(
      lib.er_bias_bn_act_bwd(_p(z), _p(bias), _p(gamma), _p(y), _p(gy), _p(save_mean), _p(save_rstd),
                             batch, units, 1 if relu else 0, _p(gz), _p(gbias), _p(ggamma), _p(gbeta),
                             _p(ws), ws.numel(), _stream()), 'er_bias_bn_act_bwd')
  return gz, gbias, ggamma, gbeta


def bn_relu_bwd(z, bias, gamma, beta, save_mean, save_rstd, gy, relu, ws):
  """bias_bn_act_bwd for batch norm (+ relu) with the relu mask recomputed from z (er_bn_relu_bwd: y is not read).
  Returns (gz, gbias, ggamma, gbeta), or None when the arrays do not suit its vector kernels (units % 4, 16-byte
  alignment): bias_bn_act_bwd then."""
  lib = _lib.load()
  _chk(gy, torch.float32, 'gy')
  batch, units = z.shape
  if units % 4 or any(t is not None and t.data_ptr() % 16 for t in (z, bias, gamma, beta, save_mean, save_rstd, gy)):
    return None
  gz = torch.empty_like(z)
  gbias = torch.empty(units, dtype=torch.float32, device=z.device)
  ggamma = torch.empty(units, dtype=torch.float32, device=z.device)
  gbeta = torch.empty(units, dtype=torch.float32, device=z.device)
  _lib.check(
      lib.er_bn_relu_bwd(_p(z), _p(bias), _p(gamma), _p(beta), _p(save_mean), _p(save_rstd), _p(gy), batch, units,
                         1 if relu else 0, _p(gz), _p(gbias), _p(ggamma), _p(gbeta), _p(ws), ws.numel(), _stream()),
      'er_bn_relu_bwd')
  return gz, gbias, ggamma, gbeta
