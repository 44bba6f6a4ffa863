"""Training step driver: the torch-side replacement of the reference's hot loop
(`sess.run(train_op)` under EasyRecEstimator._train_model_fn, model/easy_rec_estimator.py:155-472,
and optimize_loss, compat/optimizers.py:89-450).

One step = K1 bucketize -> K2 gather+pool -> interaction + dense MLP -> loss -> backward ->
K7 dedup + fused row update -> one fused dense-optimizer launch.  The whole step is shape-static,
so it is captured once into a CUDA graph and replayed (launch latency, not HBM, bounds a
batch-8192 step: SURVEY.md section 8d); the learning rate lives in device memory so a schedule
does not need a re-capture.
"""
import ctypes

import numpy as np
import torch

from easyrec_b200 import _lib
from easyrec_b200 import kernels as K
from easyrec_b200 import layers as L


class FlatDenseOptimizer(object):
  """All dense parameters as views of one flat fp32 buffer; gradients are gathered into a flat
  buffer (one multi-tensor copy) and applied by ONE er_dense_apply launch.

  kind 'adagrad': tf.train.AdagradOptimizer (acc0 = 0.1, protos/optimizer.proto:79)
  kind 'adam' / 'lazy_adam': tf.train.AdamOptimizer dense rule, lr_t = lr*sqrt(1-b2^t)/(1-b1^t)
  l2 per tensor: kernel_regularizer l2_regularizer(scale) applied as g += scale * w."""

  def __init__(self, named_params, kind, lr, l2_of=None, beta1=0.9, beta2=0.999, eps=1e-8,
               adagrad_init=0.1):
    self.names = [n for n, _ in named_params]
    self.params = [p for _, p in named_params]
    dev = self.params[0].device
    sizes = [p.numel() for p in self.params]
    self.sizes = sizes
    # every tensor starts on a 16-byte boundary so er_gemm reads the kernels in place (float4 loads)
    total = sum((n + 3) // 4 * 4 for n in sizes)
    self.flat_p = torch.zeros(total, dtype=torch.float32, device=dev)   # (alignment padding between tensors stays 0)
    self.flat_g = torch.zeros(total, dtype=torch.float32, device=dev)
    off = 0
    segs = np.zeros(len(sizes), dtype=_lib.DENSE_SEG_DTYPE)
    self.grad_views = []
    for i, (n, p) in enumerate(named_params):
      v = self.flat_p[off:off + sizes[i]].view_as(p)
      v.copy_(p.data)
      p.data = v
      self.grad_views.append(self.flat_g[off:off + sizes[i]].view_as(p))
      # dense layers write dW straight into this slice (layers._DenseBNAct.backward) when the kernel is
      # used once per step, so the big gradients skip the gather copy
      p._er_grad_out = self.grad_views[-1] if p.dim() == 2 else None
      p._er_uses = 0
      segs[i]['offset'] = off
      segs[i]['n'] = sizes[i]
      segs[i]['l2'] = float(l2_of(n, p)) if l2_of else 0.0
      segs[i]['lr_mult'] = 1.0
      off += (sizes[i] + 3) // 4 * 4
    self.segs_dev = torch.from_numpy(segs.view(np.uint8).reshape(-1).copy()).to(dev)
    # global-norm clipping needs the regularisation gradient l2 * w BEFORE the update rule: l2 per element, and a
    # copy of the segment table without l2 for the apply that follows (the gradient then already carries it)
    l2_vec = np.zeros(total, np.float32)
    for sg in segs:
      l2_vec[int(sg['offset']):int(sg['offset']) + int(sg['n'])] = sg['l2']
    self._l2_vec_np = l2_vec
    self.l2_vec = None
    nol2 = segs.copy()
    nol2['l2'] = 0.0
    self.segs_nol2_dev = torch.from_numpy(nol2.view(np.uint8).reshape(-1).copy()).to(dev)
    self.n_segs = len(sizes)
    self.max_n = max(sizes)
    self.kind = {'adagrad': _lib.OPT_ADAGRAD, 'adam': _lib.OPT_ADAM_ROWS, 'lazy_adam': _lib.OPT_ADAM_ROWS,
                 'sgd': _lib.OPT_SGD, 'momentum': _lib.OPT_MOMENTUM}[kind]
    self.s0 = self.s1 = None
    if self.kind == _lib.OPT_ADAGRAD:
      self.s0 = torch.full((total,), adagrad_init, dtype=torch.float32, device=dev)
    elif self.kind == _lib.OPT_MOMENTUM:
      self.s0 = torch.zeros(total, dtype=torch.float32, device=dev)   # accum; the momentum itself is beta1
    elif self.kind == _lib.OPT_ADAM_ROWS:
      self.s0 = torch.zeros(total, dtype=torch.float32, device=dev)
      self.s1 = torch.zeros(total, dtype=torch.float32, device=dev)
    self.b1, self.b2, self.eps = beta1, beta2, eps
    # lr and Adam's beta powers of the step: the device block shared with the sparse row update (Trainer points
    # this at the input layer's), read by the kernel - lr_t = lr*sqrt(1-b2^t)/(1-b1^t) is formed there
    self.hyper = K.StepHyper(dev, beta1, beta2)
    self.hyper.set(lr, 0)
    self.reg_loss = torch.zeros(1, dtype=torch.float32, device=dev)
    self.grad_scale = 1.0

  @property
  def lr_dev(self):
    """the effective rate of the current step as a [1] tensor (lr, or Adam's lr_t in fp32 like the TF graph)."""
    h = self.hyper
    lr = np.float32(h.lr)
    if self.kind == _lib.OPT_ADAM_ROWS:
      one = np.float32(1.0)
      lr = np.float32(np.float32(lr * np.sqrt(one - h.b2p)) / (one - h.b1p))
    return torch.tensor([float(lr)], dtype=torch.float32)

  def named_ranges(self):
    """(parameter name, offset, numel) of every tensor inside the flat buffers."""
    segs = np.frombuffer(self.segs_dev.cpu().numpy().tobytes(), dtype=_lib.DENSE_SEG_DTYPE)
    return [(n, int(s['offset']), int(s['n'])) for n, s in zip(self.names, segs)]

  def zero_grad(self):
    for p in self.params:
      p.grad = None
      p._er_uses = 0

  def gather_grads(self):
    """p.grad (fresh autograd tensors) -> the flat gradient buffer (one multi-tensor copy)."""
    srcs, dsts = [], []
    for p, v in zip(self.params, self.grad_views):
      if p.grad is None:
        v.zero_()
      elif p.grad.data_ptr() != v.data_ptr():   # else: already produced in place
        srcs.append(p.grad)
        dsts.append(v)
    if srcs:
      torch._foreach_copy_(dsts, srcs)

  def apply(self, l2_folded=False, grad_scale=None):
    """l2_folded: the gradient buffer already holds g + l2 * w (fold_l2): apply without the regulariser.
    grad_scale: instead of self.grad_scale (a buffer that was already averaged over the replicas)."""
    lib = _lib.load()
    opt = self.hyper.opt(self.kind, self.eps, grad_scale=self.grad_scale if grad_scale is None else grad_scale)
    segs = self.segs_nol2_dev if l2_folded else self.segs_dev
    if not l2_folded:
      self.reg_loss.zero_()
    _lib.check(
        lib.er_dense_apply(self.flat_p.data_ptr(), self.flat_g.data_ptr(), K._p(self.s0), K._p(self.s1),
                           segs.data_ptr(), self.n_segs, self.max_n, ctypes.byref(opt),
                           None, None if l2_folded else self.reg_loss.data_ptr(),
                           torch.cuda.current_stream().cuda_stream), 'er_dense_apply')

  def fold_l2(self):
    """flat_g <- flat_g + l2 * w (the gradient of the kernel regularisers, which TF's loss carries) and
    reg_loss <- sum l2/2 * w^2; returns sum(flat_g^2).  For global-norm clipping, which sees the FULL gradient."""
    if self.l2_vec is None:
      self.l2_vec = torch.from_numpy(self._l2_vec_np).to(self.flat_p.device)
    self.reg_loss.copy_((0.5 * self.l2_vec * self.flat_p * self.flat_p).sum().reshape(1))
    self.flat_g.addcmul_(self.l2_vec, self.flat_p)
    return (self.flat_g * self.flat_g).sum()


def _tree_clone(x):
  """device copy of a batch structure: tensors inside dicts / tuples (seq_fea, tag_fea), None passed through."""
  if x is None:
    return None
  if isinstance(x, dict):
    return {k: _tree_clone(v) for k, v in x.items()}
  if isinstance(x, (tuple, list)):
    return tuple(_tree_clone(v) for v in x)
  return x.clone()


def _tree_copy(dst, src, path='features'):
  """src -> the static buffers a captured graph reads; the shapes are part of the capture."""
  if dst is None and src is None:
    return
  if isinstance(dst, dict):
    for k in dst:
      _tree_copy(dst[k], src[k], path + '.' + str(k))
    return
  if isinstance(dst, tuple):
    for i, d in enumerate(dst):
      _tree_copy(d, src[i], '%s[%d]' % (path, i))
    return
  if dst is None or src is None or dst.shape != src.shape:
    raise _lib.ErError('%s: a CUDA-graph captured step needs batches of one fixed shape (got %s, captured %s); '
                       'variable-length inputs (TagFeature lists) train with use_cuda_graph=False'
                       % (path, None if src is None else tuple(src.shape), None if dst is None else tuple(dst.shape)))
  dst.copy_(src, non_blocking=True)


class Trainer(object):

  def __init__(self, model, input_layer, dense_optimizer='adagrad', lr=0.01, lr_fn=None,
               use_cuda_graph=False, world_size=1, beta1=0.9, beta2=0.999, adagrad_init=0.1, dense_lr_fn=None,
               dense_betas=None, clip_norm=0.0):
    self.model = model
    self.input_layer = input_layer
    self.lr = lr
    self.lr_fn = lr_fn or (lambda step: lr)
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    l2 = getattr(model, 'l2_of', None)
    db1, db2 = dense_betas or (beta1, beta2)
    self.dense_opt = FlatDenseOptimizer(named, dense_optimizer, lr, l2_of=l2, beta1=db1, beta2=db2,
                                        adagrad_init=adagrad_init)
    self.beta1, self.beta2 = beta1, beta2
    # the tower kernels' tf32 planes, split at the head of every step's forward and backward (L.use_planes): they are
    # then never stale, whatever wrote the weights between steps (optimizer, checkpoint restore, replica broadcast)
    kernels = L.tower_kernels(model)
    self.planes = K.DensePlanes(kernels, kernels[0].device) if kernels and kernels[0].is_cuda else None
    # dense_lr_fn: a second optimizer_config for everything that is not an embedding table (easy_rec_model.py:446-467):
    # its own schedule and beta powers in its own device block; otherwise one block serves both optimizers
    self.dense_lr_fn = dense_lr_fn
    if dense_lr_fn is None:
      self.dense_opt.hyper = input_layer.hyper   # one device block for both optimizers: one copy per step
    self.world = world_size
    # train_config.gradient_clipping_by_norm (> 0): global-norm clipping of all gradients before the updates
    self.clip_norm = float(clip_norm or 0.0)
    self.last_grad_norm = None
    self.dp = None
    if world_size > 1:
      from easyrec_b200.distributed import DataParallel
      ep = bool(getattr(input_layer, 'ep', False))
      if self.clip_norm and ep:
        # row-sharded tables: the owners hold their update after the gradient all-to-all until the norm of every
        # shard's received gradients has been reduced (compat/optimizers.py:453-470 part_norms)
        input_layer.ep_hold_updates(True)
      self.dp = DataParallel(input_layer, self.dense_opt, world_size, sparse=not ep)
    dev = str(getattr(input_layer, 'device', 'cpu'))
    self._ep_side = torch.cuda.Stream(device=dev) if (self.dp is not None and not self.dp.sparse and
                                                      dev.startswith('cuda')) else None
    self.step = 0
    self.use_cuda_graph = use_cuda_graph
    # the first steps of a graph-mode run execute eagerly as ordinary training steps (allocator pools, lazily
    # created workspaces and handles get their final shape); the step after them is captured WITHOUT being
    # executed and replayed from then on, so every batch is applied exactly once
    self.graph_warmup_steps = 2
    self._eager_steps = 0
    self._prefetch_mode = False
    self._stale_next = False
    self._static_next = None
    self._warm_stream = None
    self._graph = None
    self._step_pending = []
    self._static = None
    self._loss = None
    self._probs = None

  def _set_hyper(self):
    lr = self.lr_fn(self.step)
    self.input_layer.set_optimizer_step(lr, self.step, beta1=self.beta1, beta2=self.beta2)
    if self.dense_lr_fn is not None:
      self.dense_opt.hyper.set(self.dense_lr_fn(self.step), self.step)

  # The step is three segments; only the middle one talks to other ranks (world > 1).  A CUDA graph
  # captures all three, the collectives included.
  def _segment_compute(self, features, labels, next_features=None):
    """lookup -> model -> loss -> backward -> dense grads into the flat buffer."""
    self.dense_opt.zero_grad()
    if self.planes is not None:
      self.planes.refresh()
    with L.use_planes(self.planes):
      logits = self.model(features)
      if next_features is not None:
        # row-sharded tables: the id half of the NEXT batch's exchange reads no table, so it runs beside this step's
        # backward and the next lookup only promotes it (InputLayer.prefetch_exchange)
        self.input_layer.prefetch_exchange(next_features)
      sw = features.get('sample_weight') if isinstance(features, dict) else None
      if sw is not None:   # data_config.sample_weight (input/input.py:140-141 -> EasyRecModel._sample_weight)
        loss, probs = self.model.loss(logits, labels, sample_weight=sw)
      else:
        loss, probs = self.model.loss(logits, labels)
      with L.defer_dw_join():   # kernel-gradient GEMMs overlap the rest of the backward chain
        loss.backward()
    self.dense_opt.gather_grads()
    self._step_pending = list(self.input_layer._pending)
    return loss.detach(), probs

  def _segment_exchange(self):
    if self.dp is not None:
      if not self.dp.sparse:
        # row-sharded tables: their backward (gradient sums, all-to-all to the owners, owner-side row update); on CUDA
        # a parallel branch beside the dense all-reduce + dense optimizer, joined in _segment_update
        if self._ep_side is not None:
          self._ep_side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self._ep_side):   # (no side stream: a no-op)
          self.input_layer.backward_update()
      self.dp.exchange(self._step_pending)   # flat all-reduce + all-gather of K7 inputs
      self.dp.join_presort()

  def _clip_by_global_norm(self):
    """clip_ops.clip_by_global_norm over EVERY gradient, the tables' IndexedSlices included (compat/optimizers.py:
    365-376, norm as _get_grad_norm :453-481): t <- t * clip / max(global_norm, clip).  Runs after the backward pass
    and before any update: the sparse part is a K7 pass in emit form (deduplicated per column, like the IndexedSlices
    TF builds), the factor lands in the device-resident gradient scale the fused row update reads and on the dense
    gradient buffer.  Device-only: captured with the step."""
    il, opt = self.input_layer, self.dense_opt
    if self.dp is not None:
      # data parallel over replicated tables (compat/optimizers.py:285-293 then :365-376): the norm is taken over the
      # REDUCED gradients - the dense ones averaged (the flat buffer holds their sum after the all-reduce), every
      # table's IndexedSlices all-gathered and divided by N, i.e. each rank's per-column slices side by side: the
      # local sums of squares add up over the ranks, over N^2.  One scalar all-reduce; replicas get the same factor.
      n = float(self.world)
      # (row-sharded tables: what each owner received - one entry per source rank and distinct row, summed over all
      # columns of the call, as the reference's single `unique` before the exchange gives it, feature_column.py:263)
      sparse_sq = (il.sparse_grad_sqnorm() if self.dp.sparse else il.ep_recv_sqnorm()).reshape(1)
      import torch.distributed as dist
      dist.all_reduce(sparse_sq, op=dist.ReduceOp.SUM)
      opt.flat_g.mul_(1.0 / n)
      sq = sparse_sq[0] / (n * n) + opt.fold_l2()
    else:
      sq = il.sparse_grad_sqnorm() + opt.fold_l2()
    norm = torch.sqrt(sq)
    scale = self.clip_norm / torch.clamp(norm, min=self.clip_norm)
    opt.flat_g.mul_(scale)
    il.hyper.dev[_lib.HYPER_GRAD_SCALE:_lib.HYPER_GRAD_SCALE + 1].mul_(scale)
    self.last_grad_norm = norm

  def _segment_update(self, loss):
    if self.clip_norm:
      if self._ep_side is not None:
        torch.cuda.current_stream().wait_stream(self._ep_side)   # the gradient exchange of _segment_exchange
      self._clip_by_global_norm()
      if self.dp is not None and not self.dp.sparse:
        self.input_layer.ep_apply_held()       # owner-side K7 with the clipped, 1/N-scaled gradient scale
        self.dense_opt.apply(l2_folded=True, grad_scale=1.0)
      elif self.dp is not None:
        # the gathered K7 reads the clip factor from the device-resident gradient scale (x 1/N, replica_grad_scale);
        # the dense buffer already holds the averaged, regularised, clipped gradient
        self.dp.apply_sparse(self._step_pending, self.input_layer.opt_holder['opt'])
        self.input_layer.discard_pending()
        self.dense_opt.apply(l2_folded=True, grad_scale=1.0)
      else:
        self.input_layer.backward_update()
        self.dense_opt.apply(l2_folded=True)
      return loss + self.dense_opt.reg_loss[0]
    if self.dp is None:
      self.input_layer.backward_update()   # K7: dedup + fused row update, on this thread/stream
    elif self.dp.sparse:
      self.dp.apply_sparse(self._step_pending, self.input_layer.opt_holder['opt'])
      self.input_layer.discard_pending()
    self.dense_opt.apply()                 # one launch: l2 + adagrad/adam over the flat buffer
    if self._ep_side is not None:
      torch.cuda.current_stream().wait_stream(self._ep_side)   # the row-sharded backward of _segment_exchange
    # reported loss = data loss + embedding regularisation (autograd) + dense l2 (from the apply)
    return loss + self.dense_opt.reg_loss[0]

  def _step_body(self, features, labels, next_features=None):
    if self.dp is not None:
      self.dp.pre_exchange(features)   # K1 + all-gather of rows + global dedup sort on a side stream
    loss, probs = self._segment_compute(features, labels, next_features)
    self._segment_exchange()
    out = self._segment_update(loss), probs
    if next_features is not None:
      self.input_layer.join_prefetch()
    return out

  def train_step(self, features, labels, next_features=None):
    """features/labels: device tensors.  Returns (loss [scalar tensor], probs [B]).

    next_features (EmbeddingParallel only, else ignored): the features of the batch the NEXT train_step call will be
    given - its id exchange then runs beside this step instead of at the head of the next one.  A run that passes it
    should pass it on every step but the last; the exchange verifies on the device that the batch it prefetched is the
    one that arrives (InputLayer.check_exchange)."""
    self.model.train()
    self._set_hyper()
    if not bool(getattr(self.input_layer, 'ep', False)):
      next_features = None
    if not self.use_cuda_graph:
      out = self._step_body(features, labels, next_features)
      self.step += 1
      return out
    if self._eager_steps < self.graph_warmup_steps:
      # the eager steps ahead of a capture run on a side stream, like the capture itself: autograd keys the gradient
      # accumulation of a parameter to the stream it first ran on, and the legacy default stream may not take part
      # in a capture (torch's own rule for whole-step capture: "warm up on a side stream")
      cur = torch.cuda.current_stream()
      if self._warm_stream is None:
        self._warm_stream = torch.cuda.Stream(device=cur.device)
      self._warm_stream.wait_stream(cur)
      with torch.cuda.stream(self._warm_stream):
        out = self._step_body(features, labels, next_features)
      cur.wait_stream(self._warm_stream)
      self.step += 1
      self._eager_steps += 1
      return out
    if self._graph is None:
      # row-sharded tables: the captured step always promotes a prefetched id exchange and prefetches the next one;
      # a call that does not name its successor leaves the exchange "stale" and the next call runs it eagerly first
      self._prefetch_mode = bool(getattr(self.input_layer, 'ep', False))
      self._capture(features, labels, next_features)
    else:
      _tree_copy(self._static_feats, features)
      self._static['__labels'].copy_(labels, non_blocking=True)
      if self._prefetch_mode and next_features is not None:
        _tree_copy(self._static_next, next_features)
    if self._prefetch_mode:
      if self._stale_next:   # the previous call did not name this batch: its id exchange runs now, ahead of the replay
        self.input_layer.prefetch_exchange(self._static_feats)
        self.input_layer.join_prefetch()
      self._stale_next = next_features is None
    self._graph.replay()
    if self._prefetch_mode:
      # the replay promoted and prefetched on its own; an EAGER lookup after it (evaluate / predict) must not take
      # the graph's prefetched ids for its own
      self.input_layer.drop_prefetch()
    self.step += 1
    return self._loss, self._probs

  def _capture(self, features, labels, next_features=None):
    """Record one step into a CUDA graph (nothing executes here; train_step replays it).  Every step-varying
    scalar of the optimizers - learning rate, Adam's beta powers, gradient scale - is read by the kernels from
    the device block `input_layer.hyper` that _set_hyper refreshes before each replay, so Adagrad, lazy Adam
    and tf.train.AdamOptimizer rows and any learning-rate schedule replay the same graph."""
    feats = _tree_clone(features)
    self._static = {'__labels': labels.clone()}
    self._static_feats = feats
    self._static_next = _tree_clone(next_features if next_features is not None else features) \
        if self._prefetch_mode else None
    if self._prefetch_mode and not self.input_layer.prefetch_ready():
      self.input_layer.prefetch_exchange(feats)   # eager: the captured lookup promotes a prefetched exchange
      self.input_layer.join_prefetch()
    self._stale_next = False
    torch.cuda.synchronize()
    self._graph = torch.cuda.CUDAGraph()
    n0 = _lib.load().er_launch_count()
    # Data parallel: the collectives (NCCL on the capture stream) are captured with the rest of the step - one
    # graph per step.  capture_error_mode 'thread_local': NCCL's watchdog thread polls CUDA events while this
    # thread captures, which the default global mode treats as a capture violation.
    kw = {} if self.dp is None else {'capture_error_mode': 'thread_local'}
    with torch.cuda.graph(self._graph, **kw):
      self._loss, self._probs = self._step_body(feats, self._static['__labels'], self._static_next)
    # kernels of liber_b200.so inside one replay of the graph
    self.launches_per_step = int(_lib.load().er_launch_count() - n0)
