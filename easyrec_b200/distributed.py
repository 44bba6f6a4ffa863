"""Data-parallel training over NCCL, one process per GPU (torchrun).

Replicated-table DP = what the reference gets from `HorovodStrategy`
(compat/optimizers.py:285-293): every gradient is averaged over the replicas; the sparse ones
(IndexedSlices) travel as an all-gather of (indices, values).  Here the all-gather moves the
*inputs* of K7 -- each rank's arena rows, per-lookup weights and upstream gradient matrix -- and
every rank then runs the same deterministic dedup + fused row update over the global batch, so
replicas stay bit-identical without a broadcast.  Dense gradients: one flat all-reduce
(`hvd.allreduce(g, Average)`, compat/optimizers.py:289-292).
"""
import numpy as np
import torch
import torch.distributed as dist

from easyrec_b200 import _lib
from easyrec_b200 import embedding as E
from easyrec_b200 import kernels as K


import contextlib


def _null():
  return contextlib.nullcontext()


class GlobalCall(object):
  """Slot plan of one arena call replicated for `world` ranks' gathered lookups."""

  def __init__(self, call, world):
    self.call = call
    self.world = world
    recs = []
    base = call.slots_np
    # (lookup == segment for the slots of a call without CSR lookups: the one-row shortcut applies)
    call.single_one_row_ok = not getattr(call, 'has_csr', False)
    for r in range(world):
      for i in range(call.n_slots):
        s = base[i]
        rows_of_buf = call.out_rows(int(s['out_buf']))
        recs.append(dict(num_buckets=int(s['num_buckets']), row_offset=int(s['row_offset']),
                         seg_begin=int(s['seg_begin']) + r * call.n_seg, n_seg=int(s['n_seg']),
                         # one-row slots do not take part in the gathered dedup (their rows are gathered as -1): every
                         # rank sums its own column block and the [n, dim] sums are all-reduced (OneRowPlan)
                         bucket_mode=(_lib.BUCKET_NONE if int(s['bucket_mode']) == _lib.BUCKET_ONE_ROW
                                      else int(s['bucket_mode'])), combiner=int(s['combiner']),
                         out_buf=int(s['out_buf']), out_stride=int(s['out_stride']),
                         out_col=int(s['out_col']) + r * rows_of_buf * int(s['out_stride']),
                         shard_n=1))
    assert max(r['out_col'] for r in recs) < 2**31
    self.slots_np = K.make_slots(recs, call.arena.dim)
    dev = call.arena.device
    self.slots_dev = K.slots_to_device(self.slots_np, dev)
    self.n_slots = len(recs)
    self.n_seg = call.n_seg * world
    self.max_lookups = call.max_lookups * world
    self.ws = K.bwd_workspace(self.max_lookups, dev, call.arena.dim)
    self.rows = torch.empty(self.max_lookups, dtype=torch.int64, device=dev)
    self.weights = torch.empty(self.max_lookups, dtype=torch.float32, device=dev)
    self.seg_scale = None
    self.grads = [torch.empty(world * call.out_rows(i), st, dtype=torch.float32, device=dev)
                  for i, st in enumerate(call.out_strides)]
    # multi-valued (CSR) slots: every lookup names its segment; rank r's segments follow rank r-1's in the gathered plan
    self.seg_ids = self.seg_off = None
    if getattr(call, 'has_csr', False):
      self.seg_ids = torch.empty(self.max_lookups, dtype=torch.int32, device=dev)
      self.seg_off = (torch.arange(world, dtype=torch.int32, device=dev) * call.n_seg).repeat_interleave(call.max_lookups)
    # one-row slots (RawFeature projections: B lookups of one table row per rank)
    self.one_row = [(int(s['seg_begin']), int(s['n_seg']), int(s['out_buf']), int(s['out_col']), int(s['row_offset']))
                    for s in base if int(s['bucket_mode']) == _lib.BUCKET_ONE_ROW and call.single_one_row_ok]
    if self.one_row:
      self.one_row_rows = torch.tensor([r[4] for r in self.one_row], dtype=torch.int64, device=dev)
      self.one_row_sums = torch.zeros(len(self.one_row), call.arena.dim, dtype=torch.float32, device=dev)
      mask = torch.zeros(call.max_lookups, dtype=torch.bool, device=dev)
      for sb, ns, _, _, _ in self.one_row:
        mask[sb:sb + ns] = True
      self.one_row_mask = mask
      self.rows_send = torch.empty(call.max_lookups, dtype=torch.int64, device=dev)
      # the usual plan lists the raw features side by side: their blocks are ONE [B, n, dim] view of the gradient
      # matrix and their weights one [n, B] view -> two launches for all of them
      o = self.one_row
      dim = call.arena.dim
      self.one_row_block = None
      if all(o[i][1] == o[0][1] and o[i][2] == o[0][2] and o[i][0] == o[0][0] + i * o[0][1] and
             o[i][3] == o[0][3] + i * dim for i in range(len(o))):
        self.one_row_block = (o[0][0], o[0][1], o[0][2], o[0][3], len(o))


class DataParallel(object):

  def __init__(self, input_layer, dense_opt, world, sparse=True):
    """dense_opt: trainer.FlatDenseOptimizer -- its flat gradient buffer is the all-reduce bucket.
    sparse=False (EmbeddingParallel: the tables are row-sharded and exchange their own lookups, sharded.ShardedLookup):
    only the dense gradients are averaged here."""
    self.input_layer = input_layer
    self.world = world
    self.sparse = sparse
    self.placements = E.Placements()   # K7 placements over the gathered rows
    if not sparse:
      self.dense_opt = dense_opt
      dense_opt.grad_scale = 1.0 / world
      self.gcalls = {}
      self._pre = {}
      self._side = None
      self.prephase = False
      return
    input_layer.presort_enabled = False   # K7 runs on the gathered global batch, sorted after the exchange
    self.dense_opt = dense_opt
    dense_opt.grad_scale = 1.0 / world  # mean over replicas, applied inside er_dense_apply
    input_layer.replica_grad_scale = 1.0 / world   # same for the sparse rows (InputLayer.set_optimizer_step)
    plans = getattr(input_layer, 'merged', None) or input_layer.calls
    self.gcalls = {id(c): GlobalCall(c, world) for c in plans.values()}
    self._rows_owner = {}
    self._pre = {}
    self._side = None
    # the early exchange runs on a side stream; CPU runs and the calls it does not cover take the late one
    self.prephase = str(getattr(input_layer, 'device', 'cpu')).startswith('cuda')

  def pre_exchange(self, features):
    """At the head of the step: K1 on this rank's batch, all-gather of the rows and per-lookup weights, and the
    global dedup sort started on a side stream - it needs no gradient, so it runs under the dense forward/backward
    (with N ranks it is N times the single-GPU sort)."""
    self.placements.clear()
    if not self.prephase:
      return
    il = self.input_layer
    self._pre = {}
    owners = {}
    plans = il.precompute_rows(features)   # K1 on the step's stream
    if self._side is None and plans:
      self._side = torch.cuda.Stream(device=plans[0][2].device)
    if plans:
      self._side.wait_stream(torch.cuda.current_stream())
    # the all-gathers of the rows and the global placement run on a side stream: a parallel branch of the step
    # (joined in join_presort) that sits under the lookup and the dense forward / backward
    with torch.cuda.stream(self._side) if plans else _null():
      for dim, m, rows, w in plans:
        g = self.gcalls[id(m)]
        first = owners.get(id(rows))
        if first is None or first.call.arena.n_rows != m.arena.n_rows:
          first = owners[id(rows)] = g
          dist.all_gather_into_tensor(g.rows, self._rows_to_send(g, rows))
          if w is not None:
            dist.all_gather_into_tensor(g.weights, w)
        self._pre[id(m)] = first
      for dim, m, rows, w in plans:
        g = self.gcalls[id(m)]
        self.placements.presort(self._pre[id(m)].rows, m.arena.n_rows, dim, g.ws, g.slots_dev, g.n_slots)

  def sync_dense_grads(self):
    """sum over replicas in one bucket; the 1/world of hvd.allreduce(Average)
    (compat/optimizers.py:289-292) is folded into the dense apply's grad_scale."""
    dist.all_reduce(self.dense_opt.flat_g, op=dist.ReduceOp.SUM)

  def gather_sparse(self, call, rows, w, outs, seg_ids=None):
    """all-gather one arena call's K7 inputs (rows, weights, segment scales, upstream gradients; for a call with
    multi-valued slots also the segment of every lookup) into the GlobalCall buffers; returns the GlobalCall."""
    g = self.gcalls[id(call)]
    if seg_ids is not None:
      # (lookups past a rank's real count carry row -1 and are dropped by K7 whatever segment they name)
      dist.all_gather_into_tensor(g.seg_ids, seg_ids.contiguous())
      g.seg_ids.add_(g.seg_off)
    owner = self._pre.get(id(call))
    if owner is not None:   # rows / weights were gathered (and their sort started) before the step
      g.rows_src = None if owner is g else owner
      self._gather_grads(g, call, outs, w)
      return g
    # arenas with the same row plan (wide dim-1 next to the deep tables) were looked up with the SAME rows /
    # weights tensors: gather those once and let the later call alias the first one's buffers (and its sort)
    first = self._rows_owner.get(id(rows))
    if first is not None and first is not g and first.call.arena.n_rows == call.arena.n_rows:
      g.rows_src = first
    else:
      g.rows_src = None
      self._rows_owner[id(rows)] = g
      dist.all_gather_into_tensor(g.rows, self._rows_to_send(g, rows))
      if w is not None:
        dist.all_gather_into_tensor(g.weights, w)
    self._gather_grads(g, call, outs, w)
    return g

  @staticmethod
  def _rows_to_send(g, rows):
    """this rank's rows with the lookups of one-row slots dropped (-1): those are reduced locally"""
    if not g.one_row:
      return rows
    torch.where(g.one_row_mask[:rows.numel()], torch.full_like(rows, -1), rows, out=g.rows_send[:rows.numel()])
    return g.rows_send[:rows.numel()]

  def _gather_grads(self, g, call, outs, w=None):
    if g.one_row:
      # weighted column sums of this rank's one-row slots, summed over the replicas (mean: the 1/world is in the
      # gradient scale of the row update)
      dim = call.arena.dim
      if g.one_row_block is not None and outs[g.one_row_block[2]].grad is not None:
        sb, ns, buf, col, n = g.one_row_block
        blk = outs[buf].grad[:, col:col + n * dim].reshape(ns, n, dim)
        if w is not None:
          blk = blk * w[sb:sb + n * ns].view(n, ns).t()[:, :, None]
        torch.sum(blk, dim=0, out=g.one_row_sums)
      else:
        for i, (sb, ns, buf, col, _) in enumerate(g.one_row):
          grad = outs[buf].grad
          if grad is None:
            g.one_row_sums[i].zero_()
          elif w is not None:
            torch.sum(grad[:, col:col + dim] * w[sb:sb + ns, None], dim=0, out=g.one_row_sums[i])
          else:
            torch.sum(grad[:, col:col + dim], dim=0, out=g.one_row_sums[i])
      dist.all_reduce(g.one_row_sums, op=dist.ReduceOp.SUM)
    if call.seg_scale is not None:
      if g.seg_scale is None:
        g.seg_scale = torch.empty(g.n_seg, dtype=torch.float32, device=outs[0].device)
      dist.all_gather_into_tensor(g.seg_scale, call.seg_scale)
    for i, o in enumerate(outs):
      grad = o.grad if o.grad is not None else torch.zeros_like(o)
      dist.all_gather_into_tensor(g.grads[i], grad.contiguous())

  def exchange(self, pending):
    """The collectives of one step after the backward: dense flat all-reduce + all-gather of every arena's K7
    inputs."""
    self.sync_dense_grads()
    if not self.sparse:
      return
    self._rows_owner = {}
    for call, rows, w, outs, seg_ids in pending:
      self.gather_sparse(call, rows, w, outs, seg_ids)

  def join_presort(self):
    """main stream waits for the early global sorts (call before apply_sparse)."""
    if self._pre and self._side is not None:
      torch.cuda.current_stream().wait_stream(self._side)

  def apply_sparse(self, pending, opt):
    """The same fused dedup + row update on every rank over the gathered global batch; gradients
    are scaled by 1/world (mean over replicas).  No collectives: CUDA-graph capturable."""
    # mean over replicas: a caller that keeps the step scalars in device memory (InputLayer.hyper) has folded
    # 1/world into them (replica_grad_scale); a plain er_opt_t is scaled here
    struct_scaled = not opt.hyper_dev
    if struct_scaled:
      opt.grad_scale = opt.grad_scale / self.world
    for call, rows, w, outs, seg_ids in pending:
      g = self.gcalls[id(call)]
      a = call.arena
      owner = getattr(g, 'rows_src', None) or g   # the GlobalCall whose buffers hold the gathered rows / weights
      K.embedding_bwd(a.weight, a.state0, a.state1, a.dim, owner.rows, g.slots_dev, g.n_slots, g.n_seg,
                      g.grads, opt, g.ws, weights=owner.weights if w is not None else None,
                      seg_ids=g.seg_ids if seg_ids is not None else None, seg_scale=g.seg_scale,
                      sorted_from=self.placements.sorted_from(owner.rows, a.n_rows, a.dim, g.ws))
      if g.one_row:
        K.sparse_apply(a.weight, a.state0, a.state1, a.dim, g.one_row_rows, g.one_row_sums, None, opt)
      # tf.train.AdamOptimizer: the rows nobody looked up decay too
      E.adam_dense_decay(a, owner.rows if not g.one_row else torch.cat([owner.rows, g.one_row_rows]), opt)
    if struct_scaled:
      opt.grad_scale = opt.grad_scale * self.world
