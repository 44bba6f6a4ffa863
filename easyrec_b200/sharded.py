"""Row-sharded embedding tables (model parallel) with all-to-all over NCCL: the GPU counterpart of
`embedding_parallel_lookup` (compat/feature_column/feature_column.py:248-357) and of the EP half of
`optimize_loss` (compat/optimizers.py:294-345).

Shard rule (bit-exact with the reference): owner = row mod N, local row = row div N, each worker holds
(V + N - 1) // N rows of every table (feature_column.py:296,317,461-463); produced by er_bucketize.

`ShardedLookup` / `ShardedExchange` are what `InputLayer` runs for sharded arenas: distinct ids per owner in
FIXED-capacity blocks (K8 er_shard_group), equal-split all-to-alls, nothing read back on the host, the whole exchange
captured in the step's CUDA graph; the single- and multi-valued launches of an arena share one exchange, arenas of one
row plan share ids and one packed row exchange; the id half can be prefetched a step ahead.
"""
import collections
import contextlib
import os

import numpy as np
import torch
import torch.distributed as dist

from easyrec_b200 import _lib
from easyrec_b200 import embedding as E
from easyrec_b200 import kernels as K

# the inputs of one launch's K1: ids, the CSR of a multi-valued launch (seg_ids, row_ptr) and the lookup weights K1
# prunes by, the history lengths of an un-pooled sequence launch
LaunchInput = collections.namedtuple('LaunchInput', ['ids', 'seg_ids', 'row_ptr', 'weights', 'lens'],
                                     defaults=(None,) * 4)


class ShardedExchange(object):
  """The part of the row-sharded lookup that several launches share: K1, K8, the id all-to-all, and ONE packed row
  exchange each way.

  Its members are ShardedLookups, one per (arena, launch).  The launches of the first arena lay out the lookup arrays
  (rows_local / owner / pos): launch k owns lookups [lo_k, lo_k + L_k), its single-valued slots one per segment, a
  multi-valued (CSR) launch its lookup capacity, padded with -1.  Arenas with the SAME row plan (the wide dim-1 tables
  next to the deep ones: same ids, same bucket rules, same owners) repeat those launches over the same ranges; every
  arena owns a column block of the `[N*cap, width]` send / receive matrices, which all its launches pool from and sum
  their gradients into, and gets ONE owner-side row update per step."""

  def __init__(self, world, rank, device):
    self.world, self.rank, self.device = world, rank, device
    self.members = []
    self.launches = []      # the first arena's members, in range order
    self.heads = []         # each arena's first member: its column block and its owner-side update
    self.width = 0
    self.L = 0
    self._l_eff = 0
    self.cap = self.n_ex = 0
    self._built = False
    self._active = []       # members that looked up this step, in call order
    self._summed = 0        # members whose requester-side gradient sums are in send_g
    self._side = torch.cuda.Stream(device=device) if str(device).startswith('cuda') else None
    self._pre = torch.cuda.Stream(device=device) if str(device).startswith('cuda') else None
    self.placements = E.Placements()   # the members' K7 placements, requester and owner side
    self._have_next = False   # K1 / K8 / id all-to-all of the NEXT batch already sit in the *_n buffers
    # global-norm clipping: the owners hold their row update after the gradient exchange until the norm of every
    # rank's received gradients is known (ShardedLookup.apply_held)
    self.hold = False
    self._held = None

  def add(self, member):
    assert not self._built
    a = member.call.arena
    head = next((h for h in self.heads if h.call.arena is a), None)
    k = sum(1 for m in self.members if m.call.arena is a)
    if head is None:
      head = member
      member.col = self.width
      self.width += (a.dim + 3) // 4 * 4    # 16-byte aligned column blocks
      self.heads.append(member)
    member.head, member.col = head, head.col
    if self.members and a is not self.members[0].call.arena:
      ref = self.launches[k]
      assert ref.L == member.L and ref.csr == member.csr and ref.call.arena.n_rows == a.n_rows
      member.lo, member.ref = ref.lo, ref
    else:
      member.lo, member.ref = self.L, member
      self.launches.append(member)
      self.L += member.L
      self._l_eff += member.l_eff
      # distinct rows this rank can ask one peer for: every lookup of the hashed / identity slots in the worst case
      # (rows spread evenly over the owners, `slack` covers the imbalance), ONE row per one-row table, the capacity
      # of a multi-valued launch
      self.cap = min(self.L, (int(np.ceil(member.slack * self._l_eff / self.world)) + 256 + 255) // 256 * 256)
      self.n_ex = self.world * self.cap
    self.members.append(member)

  def build(self):
    if self._built:
      return
    assert all(sum(1 for m in self.members if m.head is h) == len(self.launches) for h in self.heads)
    dev, N = self.device, self.world
    f32, i64 = torch.float32, torch.int64
    self.owner = torch.empty(self.L, dtype=torch.int32, device=dev)
    self.rows_local = torch.empty(self.L, dtype=i64, device=dev)
    self.send_rows = torch.empty(self.n_ex, dtype=i64, device=dev)
    self.recv_rows = torch.empty(self.n_ex, dtype=i64, device=dev)
    self.pos = torch.empty(self.L, dtype=i64, device=dev)
    self.counts = torch.zeros(N + 1, dtype=torch.int32, device=dev)
    self.overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    self.group_ws = K.shard_group_workspace(self.L, dev)
    # the same for the batch AFTER this one (prefetch): ids need no table state, so their exchange runs a step ahead
    self.owner_n = torch.empty(self.L, dtype=torch.int32, device=dev)
    self.rows_local_n = torch.empty(self.L, dtype=i64, device=dev)
    self.send_rows_n = torch.empty(self.n_ex, dtype=i64, device=dev)
    self.recv_rows_n = torch.empty(self.n_ex, dtype=i64, device=dev)
    self.pos_n = torch.empty(self.L, dtype=i64, device=dev)
    self.ids_n = torch.empty(self.L, dtype=i64, device=dev)
    self.counts_n = torch.zeros(N + 1, dtype=torch.int32, device=dev)
    self.mismatch = torch.zeros(1, dtype=i64, device=dev)
    shape = (self.n_ex, self.width)
    self.send_emb, self.recv_emb = torch.zeros(shape, dtype=f32, device=dev), torch.zeros(shape, dtype=f32, device=dev)
    self.send_g, self.recv_g = torch.zeros(shape, dtype=f32, device=dev), torch.zeros(shape, dtype=f32, device=dev)
    for m in self.members:
      m._plan(self)
    self._built = True

  def _k1(self, m, p, ids, rows, owner):
    """K1 of launch m into its range `rows` / `owner`"""
    call = m.call
    if p.lens is not None:
      K.bucketize_seq(ids, p.lens, m.seq[0], m.seq[1], call.slots_dev, call.n_slots, rows=rows, owner=owner)
      return
    if m.csr:
      # multi-valued slots: K1 writes the real lookups only; the padding of the fixed-capacity range asks for nothing
      rows.fill_(-1)
      owner.fill_(-1)
    K.bucketize(ids, call.slots_dev, call.n_slots, call.n_seg, seg_ids=p.seg_ids, row_ptr=p.row_ptr, rows=rows,
                owner=owner, **K.k1_weight_args(ids, p.weights))

  def prefetch(self, inputs):
    """The id half of the NEXT batch's exchange (K1 of every launch -> K8 -> all_to_all(ids)), on a side stream beside
    this step's dense backward: it reads no table, so it may run a whole step ahead.  lookup() of the next step then
    only promotes the results.  inputs() -> [LaunchInput] of the next batch, one per launch; it is called on the
    prefetch branch, so what it computes there (the CSR of the next batch) is ordered with the K1 that reads it.  The
    ids, CSR offsets and weights must be the ones the next lookup() is called with (checked on the device)."""
    self.build()
    N = self.world
    if self._pre is not None:
      self._pre.wait_stream(torch.cuda.current_stream())
    with (torch.cuda.stream(self._pre) if self._pre is not None else contextlib.nullcontext()):
      parts = inputs()
      assert len(parts) == len(self.launches)
      for m, p in zip(self.launches, parts):
        m.ids_n.copy_(p.ids)
        if m.csr:
          m.row_ptr_n.copy_(p.row_ptr)
          m.w_next = p.weights is not None
          if m.w_next:
            m.w_n.copy_(p.weights)
        self._k1(m, p, m.ids_n, m.rows_n, m.owner_n)
      K.shard_group(self.rows_local_n, self.owner_n, N, self.cap, self.send_rows_n, self.pos_n, self.counts_n,
                    self.group_ws)
      self.overflow += self.counts_n[N:]
      dist.all_to_all_single(self.recv_rows_n, self.send_rows_n)
    self._have_next = True

  def join_prefetch(self):
    """the step's stream waits for the prefetch branch (a fork inside a capture must be joined before it ends)"""
    if self._pre is not None:
      torch.cuda.current_stream().wait_stream(self._pre)

  def lookup(self, parts):
    """K1 of every launch into its range -> ONE K8 over all of them -> all_to_all(ids) -> every arena's K2 on the
    owner -> ONE all_to_all(rows).  parts: [LaunchInput] of this batch, one per launch of the first arena, in range
    order.  A CSR launch's weights go to K1 (it drops the mean / sqrtn lookups they prune, so K8 does not request
    those rows); an un-pooled sequence launch's lens make its padded steps request nothing (er_bucketize_seq)."""
    N = self.world
    assert len(parts) == len(self.launches)
    if self._have_next:
      # (inside a capture the prefetch being promoted ran in the PREVIOUS replay or eagerly before this one: ordered
      # by the stream already, and a captured stream may not wait on work outside its capture)
      if self._pre is not None and not torch.cuda.is_current_stream_capturing():
        torch.cuda.current_stream().wait_stream(self._pre)
      for m, p in zip(self.launches, parts):   # the prefetched batch must be the one looked up now
        self.mismatch += (m.ids_n != p.ids).sum()
        if m.csr:
          self.mismatch += (m.row_ptr_n != p.row_ptr).sum()
          if m.w_next and p.weights is not None:   # (bit patterns: a NaN weight equals itself)
            self.mismatch += (m.w_n.view(torch.int32) != p.weights.view(torch.int32)).sum()
          elif m.w_next != (p.weights is not None):
            self.mismatch += 1
      self.pos.copy_(self.pos_n)
      self.recv_rows.copy_(self.recv_rows_n)
      self.rows_local.copy_(self.rows_local_n)
      self._have_next = False
    else:
      for m, p in zip(self.launches, parts):
        self._k1(m, p, p.ids, m.rows, m.owner)
      K.shard_group(self.rows_local, self.owner, N, self.cap, self.send_rows, self.pos, self.counts, self.group_ws)
      self.overflow += self.counts[N:]
      dist.all_to_all_single(self.recv_rows, self.send_rows)
    self.placements.clear()
    if self._side is not None and torch.is_grad_enabled():
      # the row-only halves of the K7s (requester: positions of the single-valued launches, owner: received rows)
      # need no gradient: a parallel branch under the row exchange and the dense forward / backward, joined in the
      # backward
      self._side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(self._side):
        for m in self.members:
          a = m.call.arena
          if not m.csr:
            self.placements.presort(m.pos, self.n_ex, a.dim, m.pool_ws, m.pool_slots, m.call.n_slots)
          if m.head is m:
            self.placements.presort(self.recv_rows, a.n_rows, a.dim, m.owner_ws, m.owner_slots, 1)
    for h in self.heads:
      K.embedding_fwd(h.call.arena.weight, h.call.arena.dim, self.recv_rows, h.owner_slots, 1, self.n_ex, [self.send_emb])
    dist.all_to_all_single(self.recv_emb, self.send_emb)
    self._active, self._summed = [], 0

  def owner_update(self, opt):
    """ONE K7 per arena over the received gradient rows (every launch's sums already added up per position), one
    contribution per source rank summed in rank order, gradient scale 1/N (compat/optimizers.py:315-316); then the
    arena's one dense Adam decay of the step"""
    N = self.world
    struct_scaled = not opt.hyper_dev   # a device-resident grad_scale already carries the 1/N
    if struct_scaled:
      opt.grad_scale = opt.grad_scale / N
    for h in dict.fromkeys(m.head for m in self._active):
      a = h.call.arena
      K.embedding_bwd(a.weight, a.state0, a.state1, a.dim, self.recv_rows, h.owner_slots, 1, self.n_ex, [self.recv_g],
                      opt, h.owner_ws, n_rows=a.n_rows,
                      sorted_from=self.placements.sorted_from(self.recv_rows, a.n_rows, a.dim, h.owner_ws))
      E.adam_dense_decay(a, self.recv_rows, opt)
    if struct_scaled:
      opt.grad_scale = opt.grad_scale * N
    self._active, self._summed = [], 0

  def check(self):
    bad = int(self.mismatch.item())
    if bad:
      self.mismatch.zero_()
      raise _lib.ErError('row-sharded exchange: the prefetched batch differed from the batch looked up in %d ids, '
                         'offsets or weights (train_step(next_features=...) must name the batch of the next call)' % bad)
    lost = int(self.overflow.item())
    if lost:
      self.overflow.zero_()
      raise _lib.ErError('row-sharded exchange: %d lookups exceeded the per-peer capacity %d (x%d peers, %d lookups per '
                         'step); raise ER_EP_SLACK' % (lost, self.cap, self.world, self.L))


class ShardedLookup(object):
  """The exchange of `embedding_parallel_lookup` around ONE fused launch of an InputLayer whose arenas are row-sharded
  (Arena.shard_n > 1): what InputLayer runs instead of K1 + K2 when the pipeline asks for
  `train_distribute: EmbeddingParallelStrategy` (compat/feature_column/feature_column.py:248-357, 416-625).

    forward : K1 (owner = row mod N, local row = row div N) -> K8 er_shard_group: distinct (owner, row) pairs in
              fixed-capacity per-owner blocks (the reference dedups before it sends too, feature_column.py:263) ->
              all_to_all(ids) -> K2 gather on the owner -> all_to_all(rows) -> K2 again, pooling the received rows
              into the call's own output matrices (config-order concat)
    backward: K7 with the plain SGD rule (lr = -1) adds the local duplicates of every position into the send buffer,
              in lookup order -> all_to_all to the owners -> K7 on each owner (one contribution per source rank, summed
              in rank order), gradient scale 1/N (compat/optimizers.py:315-316)

  Every buffer and every split size is fixed when the plan is built (`cap` ids per peer, -1 padded: a padded id
  gathers a zero row and its gradient slot is dropped by K7), so nothing is read back on the host and the exchange
  is captured in the step's CUDA graph with the rest.  A block that overflows loses lookups: counted on the device,
  raised by check().  Launches share a ShardedExchange (its docstring): the single-valued and multi-valued launches
  of an arena, and the arenas of one row plan.  Single-valued slots (the packed sparse_fea / raw projections), the
  ragged (CSR) slots, and un-pooled histories: `seq = (batch, seq_len)` makes every step of the call one lookup and one
  segment, K1 is er_bucketize_seq (padded steps ask for no row) and the pooling K2 writes each received row to its own
  step's row of the call's [batch * seq_len, sum D] matrix; a history launch has an exchange of its own."""

  def __init__(self, call, world, rank, exchange=None, slack=None, seq=None):
    a = call.arena
    assert a.shard_n == world and a.shard_rank == rank
    self.call, self.world, self.rank = call, world, rank
    # lookups of one call: one per segment for single-valued slots, the call's lookup capacity for multi-valued (CSR)
    # slots - TagFeatures, multi-valued sequence steps (the ragged forms of embedding_parallel_lookup,
    # feature_column.py:248-357 `ragged_ids / ragged_lens`)
    self.csr = not call.single_valued
    self.seq = seq
    assert seq is None or (not self.csr and exchange is None)
    self.L = L = call.max_lookups
    self.slack = float(os.environ.get('ER_EP_SLACK', '1.25')) if slack is None else slack
    self.l_eff = L if self.csr else sum(1 if int(r['bucket_mode']) == _lib.BUCKET_ONE_ROW else int(r['n_seg'])
                                        for r in call.slots_np)
    self.sum_opt = K.make_opt(_lib.OPT_SGD, -1.0)   # w - (-1) * sum(g) = the buffer plus the summed gradient
    self._weights = None
    self.ex = exchange or ShardedExchange(world, rank, a.device)
    self.ex.add(self)

  @property
  def cap(self):
    return self.ex.cap

  @property
  def n_ex(self):
    return self.ex.n_ex

  def _plan(self, ex):
    """slot plans over the packed exchange matrices, views of this launch's range (called once by
    ShardedExchange.build)"""
    call, a = self.call, self.call.arena
    dev, D, W = a.device, a.dim, ex.width
    recs = []
    for r in call.slots_np:   # pools the RECEIVED rows (a [N*cap, dim] "table" indexed by position) into the call's layout
      # a one-row table is one position: its lookups stay out of the requester's dedup (weighted column sum instead)
      mode = _lib.BUCKET_ONE_ROW if int(r['bucket_mode']) == _lib.BUCKET_ONE_ROW else _lib.BUCKET_NONE
      recs.append(dict(num_buckets=ex.n_ex, row_offset=0, seg_begin=int(r['seg_begin']), n_seg=int(r['n_seg']),
                       bucket_mode=mode, combiner=int(r['combiner']), out_buf=int(r['out_buf']),
                       out_stride=int(r['out_stride']), out_col=int(r['out_col']), shard_n=1))
    self.pool_slots_np = K.make_slots(recs, D)
    self.pool_slots = K.slots_to_device(self.pool_slots_np, dev)
    if self.head is self:
      own = [dict(num_buckets=a.n_rows, row_offset=0, seg_begin=0, n_seg=ex.n_ex, bucket_mode=_lib.BUCKET_NONE,
                  combiner=_lib.COMBINER_SUM | _lib.COMBINER_UNIT_WEIGHTS, out_buf=0, out_stride=W, out_col=self.col,
                  shard_n=1)]
      self.owner_slots = K.slots_to_device(K.make_slots(own, D), dev)
      self.owner_ws = K.bwd_workspace(ex.n_ex, dev, D)
    self.pool_ws = K.bwd_workspace(self.L, dev, D)
    self.recv_view = ex.recv_emb[:, self.col:self.col + D]   # this arena's received rows: the pooling K2's "table"
    self.sum_view = ex.send_g[:, self.col:self.col + D]      # ... and the requester-side gradient sums
    # this launch's range of the lookup arrays: ONE view object per range, shared by the arenas of the exchange (K7
    # placements are keyed by the tensor object, so the arenas' updates reuse one placement)
    r, lo, hi = self.ref, self.lo, self.lo + self.L
    if r is self:
      self.rows, self.owner, self.pos = ex.rows_local[lo:hi], ex.owner[lo:hi], ex.pos[lo:hi]
      self.rows_n, self.owner_n, self.ids_n = ex.rows_local_n[lo:hi], ex.owner_n[lo:hi], ex.ids_n[lo:hi]
    else:
      self.rows, self.owner, self.pos = r.rows, r.owner, r.pos
    if self.csr:   # what the prefetch saw of the next batch's CSR, compared when it is promoted
      self.row_ptr_n = torch.empty(call.n_seg + 1, dtype=torch.int32, device=dev)
      self.w_n = torch.empty(self.L, dtype=torch.float32, device=dev)
      self.w_next = False

  def forward(self, ids, weights, outs, row_ptr=None, seg_ids=None, lens=None):
    """ids int64 [L] in the call's slot order (None for a launch whose exchange already ran this step); writes the
    pooled rows into `outs` (the call's output matrices).  Multi-valued slots: ids padded to the lookup capacity,
    row_ptr int32 [n_seg + 1] and seg_ids int32 [L] of the CSR (lookups beyond row_ptr[-1] are ignored).  Histories:
    ids [n_features * batch * seq_len] steps and lens int32 [n_features * batch]."""
    ex, call = self.ex, self.call
    ex.build()
    assert (row_ptr is not None) == self.csr and (lens is not None) == (self.seq is not None)
    if ids is not None:
      ex.lookup([LaunchInput(ids, seg_ids, row_ptr, weights if self.csr else None, lens)])
    K.embedding_fwd(self.recv_view, call.arena.dim, self.pos, self.pool_slots, call.n_slots, call.n_seg, outs,
                    weights=weights, row_ptr=row_ptr, seg_scale=call.seg_scale)
    self._weights = weights
    self._seg_ids = seg_ids
    ex._active.append(self)
    return self.rows

  def backward_update(self, outs, opt):
    """each distinct id's gradient row (local duplicates summed first) goes to its owner, which dedups across the
    ranks and applies the fused row update.  Every launch adds its sums into its arena's column block of send_g, in
    the order the launches looked up, so a position read by several launches of one arena holds
    ((0 + sum of the first launch) + sum of the second) + ..., each sum in lookup order; the gradient rows of all
    arenas of the exchange travel together: the last launch to add its sums sends them and runs every owner-side
    update."""
    ex, call, D = self.ex, self.call, self.call.arena.dim
    gbufs = [(o.grad if o.grad is not None else torch.zeros_like(o)).contiguous() for o in outs]
    if gbufs and gbufs[0].is_cuda:
      for g in gbufs:   # (the trainer runs this backward on a side stream: the gradients were produced on the main one)
        g.record_stream(torch.cuda.current_stream())
    if ex._summed == 0:
      if ex.placements.presorted:
        torch.cuda.current_stream().wait_stream(ex._side)
      ex.send_g.zero_()
    K.embedding_bwd(self.sum_view, None, None, D, self.pos, self.pool_slots, call.n_slots, call.n_seg, gbufs,
                    self.sum_opt, self.pool_ws, weights=self._weights, seg_ids=getattr(self, '_seg_ids', None),
                    seg_scale=call.seg_scale, n_rows=self.n_ex,
                    sorted_from=ex.placements.sorted_from(self.pos, self.n_ex, D, self.pool_ws))
    ex._summed += 1
    if ex._summed < len(ex._active):
      return
    dist.all_to_all_single(ex.recv_g, ex.send_g)
    if ex.hold:
      ex._held = opt
      return
    ex.owner_update(opt)

  def apply_held(self):
    """the owner-side updates of a held exchange (after the clip factor went into the gradient scale)"""
    ex = self.ex
    if ex._held is not None:
      opt, ex._held = ex._held, None
      ex.owner_update(opt)

  def check(self):
    """Raises if any step since the last check lost lookups to a full per-peer block (host sync)."""
    self.ex.build()
    self.ex.check()
