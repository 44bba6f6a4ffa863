"""Embedding arenas and the fused lookup / backward-update engine.

Data layout (DESIGN.md "Data layout in HBM"):
  * every table with the same embedding_dim lives back to back in ONE fp32 arena
    [n_rows, dim] (row = dim*4 bytes, 64 B at dim 16), so a whole feature group -- all
    slots, all tables -- is one gather launch and one dedup+update pipeline;
  * optimizer state (adagrad accumulator | adam m, v) are arenas of the same shape;
  * lookups of a batch are the reference's packed CSR (feature-major segments,
    easy_rec/python/input/load_parquet.py:81-90); `rows` are arena row numbers.

This is the host-side counterpart of `feature_column.input_layer` +
`embedding_parallel_lookup` (compat/feature_column/feature_column.py:248-357, 384-414,
643-715): same role, none of its graph.
"""
import math
import os

import numpy as np
import torch

from easyrec_b200 import _lib
from easyrec_b200 import kernels as K


class Slot(object):
  """One (feature column -> output position) pair of an arena."""

  def __init__(self, name, table, bucket_mode, num_buckets, combiner=_lib.COMBINER_SUM,
               out_buf=0, n_seg_per_sample=1):
    self.name = name
    self.table = table            # table name inside the arena (shared embeddings share it)
    self.bucket_mode = bucket_mode
    self.num_buckets = int(num_buckets)
    self.combiner = combiner
    self.out_buf = out_buf        # which output matrix of the arena call
    self.n_seg_per_sample = n_seg_per_sample  # T for sequence slots (un-pooled [B,T,D])
    # True: whatever weights array accompanies the call holds 1.0 for this slot's lookups (plain id / sequence slots
    # next to raw-value slots): the backward skips the per-lookup weight read (ER_COMBINER_UNIT_WEIGHTS)
    self.unit_weights = False
    self.vocab = None             # Vocab of an ER_BUCKET_VOCAB slot


class Arena(object):
  """All tables of one embedding_dim, plus optimizer state, on one device."""

  def __init__(self, dim, device, shard_n=1, shard_rank=0):
    self.dim = dim
    self.device = device
    self.shard_n = shard_n
    self.shard_rank = shard_rank
    self.tables = {}   # name -> (row_offset, n_rows_local, n_rows_global)
    self.n_rows = 0
    self.kv = None     # KvTable: the arena holds one key-value table
    self.weight = None
    self.state0 = None
    self.state1 = None

  def add_table(self, name, n_rows_global, local_rows=None):
    """local_rows: this rank's rows when they are not a share of n_rows_global (a key-value table's pool)"""
    if name in self.tables:
      assert self.tables[name][2] == n_rows_global, 'shared table %s: size mismatch' % name
      return
    # per-worker rows (V + N - 1) // N  (feature_column.py:461-463)
    local = (n_rows_global + self.shard_n - 1) // self.shard_n if local_rows is None else local_rows
    self.tables[name] = (self.n_rows, local, n_rows_global)
    self.n_rows += local

  def materialize(self, opt_kind, init_fn=None, adagrad_init=0.1, generator=None, interleave=True):
    """Allocate the arena.  Default init: truncated_normal(0, 0.01/sqrt(dim))
    (feature_column_v2.py:910-912).

    interleave=True stores a row and its optimizer state side by side, [w | state0 | state1], in
    one storage matrix: the fused row update then touches ONE 128 B line per row at dim 16 +
    adagrad instead of two 64 B half-lines in different DRAM pages -- measured 1.9x more random
    read-modify-writes per second (tools/microbench_gather.cu), while the forward gather of
    the 64 B weight half costs the same as from a dense [V, 16] table."""
    assert self.n_rows > 0
    n_state = {_lib.OPT_SGD: 0, _lib.OPT_ADAGRAD: 1, _lib.OPT_MOMENTUM: 1}.get(opt_kind, 2)
    k = (1 + n_state) if interleave else 1
    self.storage = torch.empty(self.n_rows, k * self.dim, dtype=torch.float32, device=self.device)
    w = self.storage[:, :self.dim]
    plan_only = os.environ.get('ER_PLAN_ONLY') == '1'   # tests of the table PLAN: allocate, do not touch gigabytes
    if plan_only:
      init_fn = lambda t: None   # noqa: E731
    if init_fn is not None:
      init_fn(w)
    else:
      std = 0.01 / math.sqrt(self.dim)
      tmp = torch.empty(self.n_rows, self.dim, dtype=torch.float32, device=self.device)
      torch.nn.init.trunc_normal_(tmp, mean=0.0, std=std, a=-2 * std, b=2 * std,
                                  generator=generator)
      w.copy_(tmp)
      del tmp
    self.weight = w
    self.opt_kind = opt_kind
    self.adagrad_init = adagrad_init

    def state(i, fill):
      if interleave:
        v = self.storage[:, (1 + i) * self.dim:(2 + i) * self.dim]
        if not plan_only:
          v.fill_(fill)
        return v
      return torch.full((self.n_rows, self.dim), fill, dtype=torch.float32, device=self.device)

    self.state0 = self.state1 = None
    if opt_kind == _lib.OPT_ADAGRAD:
      self.state0 = state(0, adagrad_init)
    elif opt_kind == _lib.OPT_MOMENTUM:
      self.state0 = state(0, 0.0)      # the momentum accumulator (slot 'Momentum', zeros)
    elif opt_kind in (_lib.OPT_LAZY_ADAM, _lib.OPT_ADAM_ROWS):
      self.state0 = state(0, 0.0)
      self.state1 = state(1, 0.0)
    # tf.train.AdamOptimizer decays m, v and moves w on EVERY row each step; the rows of this step's lookups are
    # marked here so that the dense sweep skips exactly the rows the fused row update has already written.  A
    # key-value table has no sweep: both of the reference's paths apply _apply_sparse to the gathered rows only
    # (compat/sok_optimizer.py:215-276, and EmbeddingVariable's sparse apply on one worker)
    self.touched = (torch.zeros(self.n_rows, dtype=torch.uint8, device=self.device)
                    if opt_kind == _lib.OPT_ADAM_ROWS and self.kv is None else None)

  def table_view(self, name):
    off, n, _ = self.tables[name]
    return self.weight[off:off + n]


def _mix64(z):
  """splitmix64's finaliser on a python int"""
  m = 2**64 - 1
  z &= m
  z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
  z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
  return z ^ (z >> 31)


class KvTable(object):
  """A key-value table (ev_params) on an arena of its own: `capacity` pool rows, then one zero row that evaluation reads
  for keys it has not seen.  The open-addressing index and its counters live on the device (csrc/kv_table.cu); the
  slots of the table have num_buckets = KV_BUCKETS, so K1 hands over keys, which lookup() turns into pool rows."""

  def __init__(self, name, arena, capacity, seed, embedding_parallel=False):
    self.name = name
    self.arena = arena
    self.capacity = int(capacity)
    self.zero_row = self.capacity
    n_index = 16
    while n_index < 2 * self.capacity:
      n_index *= 2
    dev = arena.device
    self.index_keys = torch.full((n_index,), _lib.KV_EMPTY, dtype=torch.int64, device=dev)
    self.index_rows = torch.full((n_index,), -1, dtype=torch.int64, device=dev)
    self.stats = torch.zeros(2, dtype=torch.int64, device=dev)   # rows handed out, lookups left without a row
    # initial rows depend on (seed, table, key) only: the table's name enters through its fingerprint
    self.seed = _mix64(int(seed) ^ _lib.fingerprint64(name))
    # one worker: the column's initializer, the truncated normal Arena.materialize draws for static tables;
    # EmbeddingParallelStrategy: the DynamicVariable's `random {"stddev": 0.0025}` (feature_column.py:472-480), a
    # normal(0, 0.0025)
    self.init_truncated = not embedding_parallel
    self.init_stddev = 0.0025 if embedding_parallel else 0.01 / math.sqrt(arena.dim)

  def lookup(self, keys, rows, train):
    """rows = the pool rows of `keys`: find-or-insert when training, find only (unseen keys -> the zero row) else.  On
    a row-sharded arena `keys` are the owner-local keys (key div N) this rank received; the index holds global keys."""
    a = self.arena
    if train:
      init0 = a.adagrad_init if a.opt_kind == _lib.OPT_ADAGRAD else 0.0
      return K.kv_find_or_insert(self.index_keys, self.index_rows, self.capacity, self.stats, keys, rows,
                                 a.weight, a.state0, a.state1, init0, self.seed, self.init_stddev, self.init_truncated,
                                 shard_n=a.shard_n, shard_rank=a.shard_rank)
    return K.kv_find(self.index_keys, self.index_rows, keys, self.zero_row, rows, shard_n=a.shard_n,
                     shard_rank=a.shard_rank)

  def size(self):
    """keys that hold a row (reads the device counter back)"""
    return min(int(self.stats[0]), self.capacity)

  def check(self):
    n, dropped = (int(v) for v in self.stats.cpu())
    if dropped or n > self.capacity:
      raise _lib.ErError('key-value table %s: more distinct keys than its max_capacity %d (ev_params); %d lookups had '
                         'no row' % (self.name, self.capacity, dropped))

  def items(self):
    """(global keys, rows) of every key that holds a row, in row order (host tensors)"""
    k, r = self.index_keys.cpu(), self.index_rows.cpu()
    live = (k != _lib.KV_EMPTY) & (r >= 0)
    k, r = k[live], r[live]
    order = torch.argsort(r)
    return k[order], r[order]

  def load(self, keys, rows):
    """rebuild the index from (keys, rows) with the bulk-insert kernel; the caller fills the pool rows"""
    self.index_keys.fill_(_lib.KV_EMPTY)
    self.index_rows.fill_(-1)
    self.stats.zero_()
    if keys.numel():
      K.kv_insert_rows(self.index_keys, self.index_rows, keys.to(self.arena.device), rows.to(self.arena.device),
                       self.stats)
    self.stats[0] = keys.numel()
    if int(self.stats[1]):
      raise _lib.ErError('key-value table %s: restored keys are negative or repeated' % self.name)


class Vocab(object):
  """A vocabulary column's entries on the device: the read-only index K1 probes for ER_BUCKET_VOCAB slots, built once
  with the key-value tables' bulk insert (csrc/kv_table.cu layout).  keys[i] = Fingerprint64(entry i) % (2^63 - 1),
  the key the readers give the feature's raw strings; entry i is row i of the column's table.  The keys must be
  distinct and >= 0 (builder.vocab_keys refuses other vocabularies by name)."""

  def __init__(self, name, keys, device):
    self.name = name
    self.keys = np.asarray(keys, dtype=np.int64)
    if os.environ.get('ER_PLAN_ONLY') == '1' and not str(device).startswith('cuda'):
      # a plan built to be inspected, not run (Arena.materialize): no index, and nothing may probe it
      self.index_keys = self.index_rows = torch.full((16,), _lib.KV_EMPTY, dtype=torch.int64, device=device)
      return
    self.index_keys, self.index_rows = K.vocab_index(self.keys, device)


class ArenaCall(object):
  """The static plan of one fused lookup over an arena for a fixed batch size:
  slot descriptors on the device, output matrices, backward workspace."""

  def __init__(self, arena, slots, batch_size, out_widths, single_valued, max_lookups=None):
    self.arena = arena
    self.slots = slots
    self.batch_size = batch_size
    dim = arena.dim
    recs = []
    seg = 0
    cols = [0] * len(out_widths)
    # row stride of each output matrix: padded to 4 floats so 16 B vector stores stay aligned
    self.out_strides = [((w + 3) // 4) * 4 if dim % 4 == 0 else w for w in out_widths]
    self.out_widths = out_widths
    self.slot_cols = []
    for s in slots:
      off, _, _ = arena.tables[s.table]
      n_seg = batch_size * s.n_seg_per_sample
      # every slot owns its own column range of its output matrix: [B, sum dim] for pooled slots, [B*T, sum dim]
      # for the sequence slots of one group (two hist_seq features of a DIN group sit side by side)
      col = cols[s.out_buf]
      cols[s.out_buf] += dim
      stride = self.out_strides[s.out_buf]
      self.slot_cols.append(col)
      recs.append(dict(num_buckets=s.num_buckets, row_offset=off, seg_begin=seg, n_seg=n_seg,
                       bucket_mode=s.bucket_mode,
                       combiner=s.combiner | (_lib.COMBINER_UNIT_WEIGHTS if s.unit_weights else 0), out_buf=s.out_buf,
                       out_stride=stride, out_col=col, shard_n=arena.shard_n))
      seg += n_seg
    self.n_seg = seg
    self.slots_np = K.make_slots(recs, dim)
    self.slots_dev = K.slots_to_device(self.slots_np, arena.device)
    self.n_slots = len(recs)
    # the vocabularies of the call's ER_BUCKET_VOCAB slots, handed to every K1 of the call (None: no such slot)
    self.vocabs = K.vocab_plan(self.slots_np, [s.vocab for s in slots], arena.device)
    self.single_valued = single_valued
    self.max_lookups = self.n_seg if single_valued else int(max_lookups)
    self.needs_scale = any((s.combiner & 0xf) != _lib.COMBINER_SUM for s in slots)
    self.ws = K.bwd_workspace(self.max_lookups, arena.device, arena.dim)
    self.seg_scale = (torch.empty(self.n_seg, dtype=torch.float32, device=arena.device)
                      if self.needs_scale else None)

  def out_rows(self, buf):
    for s in self.slots:
      if s.out_buf == buf:
        return self.batch_size * s.n_seg_per_sample
    raise KeyError(buf)

  def alloc_outputs(self):
    return [torch.empty(self.out_rows(i), st, dtype=torch.float32, device=self.arena.device)
            for i, st in enumerate(self.out_strides)]


def fused_lookup(call, rows, weights=None, row_ptr=None, outs=None):
  """K2 over one arena.  Returns the call's output matrices as autograd LEAVES
  (requires_grad=True): after loss.backward() their .grad is dL/d(pooled), which
  `fused_backward_update` hands to K7.  The table itself is never a torch Parameter and its
  gradient never materialises as a tensor (reference: IndexedSlices -> apply_gradients,
  compat/optimizers.py:413-416)."""
  a = call.arena
  if outs is None:
    outs = call.alloc_outputs()
  K.embedding_fwd(a.weight, a.dim, rows, call.slots_dev, call.n_slots, call.n_seg, outs,
                  weights=weights, row_ptr=row_ptr, seg_scale=call.seg_scale)
  for o in outs:
    o.requires_grad_(True)
  return outs


def adam_dense_decay(arena, rows, opt, n_dev=None):
  """The dense half of tf.train.AdamOptimizer's sparse apply (builders/optimizer_builder.py:61-66; behaviour
  stated at compat/adam_s.py:74-81): every row WITHOUT a gradient this step still gets m *= b1, v *= b2,
  w -= lr_t*m/(sqrt(v)+eps).  `rows` are the step's looked-up rows (already updated by K7's row rule)."""
  if arena.opt_kind != _lib.OPT_ADAM_ROWS or arena.kv is not None:
    return
  if rows is not None and rows.numel():
    K.mark_rows(rows, arena.n_rows, arena.touched, 1, n_dev=n_dev)
  K.adam_dense_sweep(arena.weight, arena.state0, arena.state1, arena.dim, arena.touched, opt)
  if rows is not None and rows.numel():
    K.mark_rows(rows, arena.n_rows, arena.touched, 0, n_dev=n_dev)


def fused_backward_update(call, rows, outs, opt, weights=None, row_ptr=None, seg_ids=None, sorted_from=None):
  """K7: dedup + segment-sum + optimizer row update from the leaves' gradients.  Runs on the
  caller's thread and stream (not inside the autograd engine), so it is CUDA-graph capturable."""
  a = call.arena
  gbufs = []
  for i, o in enumerate(outs):
    g = o.grad
    if g is None:
      g = torch.zeros_like(o)
    gbufs.append(g.contiguous())
  K.embedding_bwd(a.weight, a.state0, a.state1, a.dim, rows, call.slots_dev, call.n_slots,
                  call.n_seg, gbufs, opt, call.ws, weights=weights, seg_ids=seg_ids,
                  row_ptr=row_ptr, seg_scale=call.seg_scale, sorted_from=sorted_from)
  adam_dense_decay(a, rows, opt, n_dev=None if row_ptr is None else row_ptr[call.n_seg:])


class Placements(object):
  """K7's bucket placements shared by the updates of one step: one per (rows tensor, n_rows, placement mode).  Tables
  looked up with the same rows (the wide dim-1 table next to the deep ones) whose dims share a mode - warp-sized or
  CTA-sized buckets, K.k7_warp_mode - need the same placement, so reusing it (er_embedding_bwd_reuse_sort) only skips
  work and never changes a result.  clear() at the start of every step; `presorted`: presort() launched work that the
  updates' stream has to join."""

  def __init__(self):
    self.clear()

  def presort(self, rows, n_rows, dim, ws, slots_dev, n_slots, seg_ids=None):
    """place the key's lookups into `ws` now, on the current stream, unless the key has a placement"""
    if self.sorted_from(rows, n_rows, dim, ws) is None:
      K.embedding_bwd_presort(rows, n_rows, dim, ws, slots_dev, n_slots, seg_ids=seg_ids)
      self.presorted = True

  def sorted_from(self, rows, n_rows, dim, ws):
    """embedding_bwd's sorted_from: the key's placement (ws, dim), or None when this update into `ws` is the first of
    its key - it places itself and later updates of the key reuse its placement."""
    key = (id(rows), int(n_rows), K.k7_warp_mode(dim))
    hit = self._placed.get(key)
    if hit is None:
      self._placed[key] = (ws, dim)
    return hit

  def clear(self):
    self._placed = {}
    self.presorted = False


class _FM(torch.autograd.Function):
  """K3: layers/fm.py:20-26 on the [B, F*D] group matrix."""

  @staticmethod
  def forward(ctx, x, n_field, dim):
    ctx.n_field, ctx.dim = n_field, dim
    ctx.save_for_backward(x)
    return K.fm_fwd(x, n_field, dim)

  @staticmethod
  def backward(ctx, gy):
    (x,) = ctx.saved_tensors
    gx = torch.empty(x.shape[0], x.shape[1], dtype=torch.float32, device=x.device)
    if x.shape[1] > ctx.n_field * ctx.dim:
      gx.zero_()
    K.fm_bwd(x, gy.contiguous(), ctx.n_field, ctx.dim, gx=gx)
    return gx, None, None


def fm(x, n_field, dim):
  return _FM.apply(x, n_field, dim)


class _FMBlock(torch.autograd.Function):
  """DeepFM's three consumers of the deep group matrix behind one autograd node: FM (layers/fm.py:20-26),
  the deep tower input (returned as a pass-through view) and the embedding regulariser's sum of squares
  (layers/input_layer.py:369-375).  Backward merges the three incoming gradients in one kernel pass, so the
  group matrix (an autograd leaf) receives a single gradient and autograd never runs an accumulation add."""

  @staticmethod
  def forward(ctx, x, n_field, dim):
    ctx.n_field, ctx.dim = n_field, dim
    y, sumsq = K.fm_block_fwd(x, n_field, dim, want_sumsq=True)
    ctx.save_for_backward(x)
    return y, x.view_as(x), sumsq

  @staticmethod
  def backward(ctx, gy, g_pass, g_sumsq):
    (x,) = ctx.saved_tensors
    # d(sumsq)/dx = 2x; g_sumsq stays on the device (no host sync: CUDA-graph capturable)
    gx = K.fm_block_bwd(x, None if gy is None else gy.contiguous(), g_pass,
                        None if g_sumsq is None else g_sumsq.contiguous(), 2.0, ctx.n_field, ctx.dim)
    return gx, None, None


def fm_block(x, n_field, dim):
  """returns (fm [B, dim], x pass-through, sum(x^2) [1])."""
  return _FMBlock.apply(x, n_field, dim)


class _RowsumBlock(torch.autograd.Function):
  """The wide group's two consumers behind one node: reduce_sum over the features (model/deepfm.py:62-63)
  and the embedding regulariser's sum of squares; backward merges both gradients in one pass."""

  @staticmethod
  def forward(ctx, x):
    y, sumsq = K.rowsum_block_fwd(x, want_sumsq=True)
    ctx.save_for_backward(x)
    return y.unsqueeze(1), sumsq

  @staticmethod
  def backward(ctx, gy, g_sumsq):
    (x,) = ctx.saved_tensors
    gx = K.rowsum_block_bwd(x, None if gy is None else gy.contiguous().view(-1),
                            None if g_sumsq is None else g_sumsq.contiguous(), 2.0)
    return gx


def rowsum_block(x):
  """returns (row sums [B, 1], sum(x^2) [1])."""
  return _RowsumBlock.apply(x)


class _ConcatCols(torch.autograd.Function):
  """tf.concat(axis=1) into a buffer whose pitch the next dense layer's GEMM reads in place; the gradient is
  split back into contiguous pieces by one launch."""

  @staticmethod
  def forward(ctx, *mats):
    ctx.widths = [m.shape[1] for m in mats]
    return K.concat_cols(list(mats))

  @staticmethod
  def backward(ctx, g):
    return tuple(K.split_cols(g, ctx.widths))


def concat_cols(mats):
  if len(mats) > 8 or not mats[0].is_cuda:
    return torch.cat(mats, dim=1)
  return _ConcatCols.apply(*mats)


class _SigmoidCE(torch.autograd.Function):
  """tf.losses.sigmoid_cross_entropy (builders/loss_builder.py:36-39), mean over nonzero weights."""

  @staticmethod
  def forward(ctx, logits, labels, weights, inv_count):
    loss, probs, g = K.sigmoid_ce(logits.contiguous(), labels, weights, inv_count)
    ctx.save_for_backward(g)
    ctx.mark_non_differentiable(probs)
    return loss[0], probs

  @staticmethod
  def backward(ctx, gl, _gp):
    (g,) = ctx.saved_tensors
    return g * gl, None, None, None


def sigmoid_cross_entropy(logits, labels, weights=None, inv_count=None):
  if inv_count is None:
    inv_count = 1.0 / logits.numel()
  return _SigmoidCE.apply(logits, labels, weights, inv_count)
