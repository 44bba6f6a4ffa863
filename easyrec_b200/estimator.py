"""EasyRecEstimator on the fused path: same constructor and train/evaluate/predict surface as the
reference (`model/easy_rec_estimator.py:62-153`, `main.py:102-163,296-400`), body replaced by the
torch/liber_b200 training loop.  tf.estimator plumbing (hooks, Scaffold, SavedModel export, PS/worker)
is out of scope (SURVEY.md section 2.2).
"""
import logging
import os
import time

import numpy as np
import torch

from easyrec_b200 import builder, checkpoint, metrics
from easyrec_b200.config import config_util
from easyrec_b200.input import readers
from easyrec_b200.trainer import Trainer

_DENSE_KIND = {'adagrad_optimizer': 'adagrad', 'adam_optimizer': 'adam', 'lazy_adam_optimizer': 'lazy_adam',
               'momentum_optimizer': 'sgd'}


auc = metrics.auc   # exact ROC AUC; the reference's tf.metrics.auc is a 200-threshold approximation of it


def _with_next(batches, ahead, want_more):
  """(features, labels, next batch or None): the next batch is drawn only when another step will follow, so no batch is
  taken from the input and left untrained."""
  it = iter(batches)
  cur = next(it, None)
  while cur is not None:
    nxt = next(it, None) if (ahead and want_more()) else None
    yield cur[0], cur[1], nxt
    if ahead:
      cur = nxt if nxt is not None else (next(it, None) if want_more() else None)
    else:
      cur = next(it, None)


class _LossReader(object):
  """Every step's loss read back to the host without stalling the device: right after step k is enqueued its loss
  (a device scalar the next step will overwrite) is copied into one of two PINNED host slots on the step's stream and
  an event is recorded; the value is consumed one step later, while step k + 1 already runs.  The host thus works one
  step ahead of the device - batch hand-off, the copies into the step's static buffers and the next launch overlap
  the running step - and still reads every step's result (what a per-step LoggingTensorHook costs the reference,
  easy_rec_estimator.py:384-396, is a sync per step).  flush() returns the newest value (blocks for the last step).
  On a CPU device it reads the value directly."""

  def __init__(self, device):
    self.cuda = str(device).startswith('cuda')
    self.k = 0
    self.value = None
    if self.cuda:
      try:
        self.buf = [torch.empty(1, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.ev = [torch.cuda.Event() for _ in range(2)]
        self.pending = [False, False]
      except RuntimeError as e:   # no page-locked memory to be had: read every loss with a synchronisation instead
        logging.warning('loss reader falls back to synchronous reads: %s', e)
        self.cuda = False

  def _take(self, j):
    if self.pending[j]:
      self.ev[j].synchronize()
      self.value = float(self.buf[j][0])
      self.pending[j] = False

  def push(self, loss):
    """enqueue the read of this step's loss; returns the newest value already on the host (the previous step's)"""
    if not self.cuda:
      self.value = float(loss)
      return self.value
    j = self.k & 1
    self._take(j)                      # (slot reuse: its value was consumed two steps ago, normally a no-op)
    self.buf[j].copy_(loss.detach().reshape(1), non_blocking=True)
    self.ev[j].record()
    self.pending[j] = True
    self.k += 1
    self._take(j ^ 1)                  # the previous step's loss: its step has (nearly) finished
    return self.value

  def flush(self):
    if self.cuda:
      self._take(self.k & 1)           # older slot first, the newest value wins
      self._take((self.k & 1) ^ 1)
    return self.value


class EasyRecEstimator(object):

  def __init__(self, pipeline_config, model_cls=None, run_config=None, params=None, device='cuda:0',
               batch_size=None, use_cuda_graph=False, world_size=1, seed=20240, default_seq_len=50, rank=None,
               embedding_parallel=None):
    if isinstance(pipeline_config, (str, bytes)):
      pipeline_config = config_util.get_configs_from_pipeline_file(pipeline_config)
    self._pipeline_config = pipeline_config
    self._device = device
    self._batch_size = batch_size or pipeline_config.data_config.batch_size
    gen = torch.Generator(device=device).manual_seed(seed) if str(device).startswith('cuda') else None
    # EmbeddingParallel (row-sharded tables + all-to-all) when the config asks for it (train_distribute) or the
    # caller does; otherwise world_size > 1 is data parallel over replicated tables
    self._ep = (builder.embedding_parallel(pipeline_config) if embedding_parallel is None else bool(embedding_parallel)) \
        and world_size > 1
    if rank is None:
      rank = int(os.environ.get('RANK', 0)) if world_size > 1 else 0
    self._rank, self._world = int(rank), int(world_size)
    self._group = None        # gloo group of the end-of-data agreement and the metric reduction (made on first use)
    self.agree_seconds, self.agree_calls = 0.0, 0
    self.input_layer, self.model, self._opt = builder.build_model(
        pipeline_config, self._batch_size, device, generator=gen,
        cpu_generator=torch.Generator().manual_seed(seed), default_seq_len=default_seq_len, world=world_size, rank=rank,
        shard_tables=self._ep)
    # one optimizer_config: tables and dense variables share kind / schedule; two: [0] trains the embedding tables
    # (the fused row rule), [1] everything else (model/easy_rec_estimator.py:216-232)
    dense = self._opt.get('dense')
    d = dense or self._opt
    dense_kind = 'momentum' if (d['kind'] == 'momentum_optimizer' and d.get('momentum', 0.0) > 0) else _DENSE_KIND[d['kind']]
    self.trainer = Trainer(self.model, self.input_layer, dense_kind, lr_fn=self._opt['lr_fn'],
                           use_cuda_graph=use_cuda_graph, world_size=world_size, beta1=self._opt['beta1'],
                           beta2=self._opt['beta2'], adagrad_init=d['acc0'],
                           dense_lr_fn=dense['lr_fn'] if dense else None,
                           dense_betas=(dense['beta1'], dense['beta2']) if dense else None,
                           clip_norm=max(float(pipeline_config.train_config.gradient_clipping_by_norm), 0.0))
    # optimizer_config.embedding_learning_rate_multiplier: gradient multiplier of the embedding tables
    # (model/easy_rec_estimator.py:308-317)
    self.input_layer.emb_grad_mult = float(self._opt.get('emb_lr_mult', 1.0))
    self.global_step = 0

  # -- properties of the reference estimator (easy_rec_estimator.py:97-153) --
  @property
  def embedding_parallel(self):
    return self._ep

  @property
  def rank(self):
    return self._rank

  @property
  def world_size(self):
    return self._world

  def _host_group(self):
    """one gloo group over all ranks, for the small host collectives of train / evaluate / predict"""
    if self._group is None:
      import torch.distributed as dist
      self._group = dist.new_group(backend='gloo')
    return self._group

  def _agree(self, flags, op):
    """element-wise MIN or MAX of this rank's flags over all ranks: one int32 all-reduce on the host"""
    import torch.distributed as dist
    t0 = time.perf_counter()
    t = torch.tensor([int(bool(f)) for f in flags], dtype=torch.int32)
    dist.all_reduce(t, op=dist.ReduceOp.MIN if op == 'min' else dist.ReduceOp.MAX, group=self._host_group())
    self.agree_seconds += time.perf_counter() - t0
    self.agree_calls += 1
    return [bool(x) for x in t.tolist()]

  def _passes(self, input_fn, ahead, want_more, again):
    """this rank's batches over the passes train() makes: (features, labels, next batch of the same pass or None); a
    new pass over input_fn() starts when one ends while again(passes made) holds, unless the pass was empty."""
    epoch = 0
    while True:
      feeder = readers.DeviceFeeder(readers.Prefetcher(input_fn(), depth=2), self._device, depth=2, lookahead=ahead)
      self.last_feeder = feeder
      n = 0
      for item in _with_next(feeder, ahead, want_more):
        n += 1
        yield item
      epoch += 1
      if n == 0 or not again(epoch):
        return

  @property
  def feature_configs(self):
    return config_util.get_feature_configs(self._pipeline_config)

  @property
  def model_config(self):
    return self._pipeline_config.model_config

  @property
  def train_config(self):
    return self._pipeline_config.train_config

  @property
  def eval_config(self):
    return self._pipeline_config.eval_config

  def train(self, input_fn, hooks=None, steps=None, max_steps=None, saving_listeners=None, fetch_loss_every_step=False):
    """input_fn() -> iterable of (features, labels) host batches.  Logs step/loss/steps-per-sec every
    log_step_count_steps like LoggingTensorHook + StepCounterHook (easy_rec_estimator.py:384-396,455-458).
    The batches reach the device through pinned, double-buffered staging (readers.DeviceFeeder) behind a parsing
    thread (readers.Prefetcher).  fetch_loss_every_step: read the loss of EVERY step back to the host (what a per-step
    logging hook costs; bench.py's end-to-end number) - through pinned slots, one step behind the device
    (_LossReader), so the host prepares step k + 1 while step k runs; `last_loss_value` is the newest value read and,
    when train() returns, the last step's.

    world_size > 1: before each step the ranks agree (one host all-reduce over a gloo group) on whether every rank holds
    this step's batch and, with row-sharded tables, the next one; the run stops at the first step some rank cannot
    make, and the next batch's id exchange is prefetched only when every rank has one, so no rank enters a collective
    another rank skips."""
    limit = steps if steps is not None else (max_steps or self.train_config.num_steps or None)
    every = max(int(self.train_config.log_step_count_steps), 1)
    t0, n0 = time.time(), self.global_step
    loss = None
    # data_config.num_epochs: 0 = pass over the data again and again until the step limit (input/input.py:1033-1040
    # dataset.repeat); without a step limit one pass is made
    epochs = int(self._pipeline_config.data_config.num_epochs)
    reader = _LossReader(self._device) if fetch_loss_every_step else None
    # row-sharded tables: train_step is told the NEXT batch, whose id exchange then runs beside the current step
    ahead = 1 if self._ep else 0
    stream = self._passes(input_fn, ahead, lambda: limit is None or self.global_step - n0 + 1 < limit,
                          lambda epoch: limit is not None and not (epochs > 0 and epoch >= epochs))
    try:
      while True:
        item = next(stream, None)   # (a rank whose pass ended has started the next one, when there is one)
        nxt = None if item is None else item[2]
        if self._world > 1:
          have, have_next = self._agree([item is not None, nxt is not None or not ahead], 'min')
          if not have:
            break
          if not have_next:
            nxt = None
        elif item is None:
          break
        # host parsing and the H2D copies run ahead of the device step
        loss, _ = self.trainer.train_step(item[0], item[1], next_features=None if nxt is None else nxt[0])
        self.global_step += 1
        if reader is not None:
          self.last_loss_value = reader.push(loss)
        if self.global_step % every == 0:
          self.input_layer.check_kv()   # a key-value table that ran out of rows stops the run when the loss is logged
          dt = time.time() - t0
          logging.info('global_step = %d, loss = %.6f, global_step/sec = %.2f', self.global_step, float(loss),
                       (self.global_step - n0) / max(dt, 1e-9))
        if limit is not None and self.global_step - n0 >= limit:
          break
    finally:
      stream.close()
    self.input_layer.check_kv()
    if reader is not None and loss is not None:
      self.last_loss_value = reader.flush()      # the last step's loss: every step's result has reached the host
      return self.last_loss_value
    return None if loss is None else float(loss)

  @torch.no_grad()
  def _forward_eval(self, feats):
    self.model.eval()
    self.input_layer.drop_prefetch()   # (an id exchange prefetched for the next TRAINING batch is not this batch's)
    logits = self.model(feats)
    self.input_layer.discard_pending()
    return logits

  def _group_fields(self):
    """eval_config.metrics_set gauc / session_auc -> [(metric name, position of the key feature in the packed
    single-valued ids, reduction)]  (model/rank_model.py:375-421: keys = features[uid_field])."""
    out = []
    by_input = {}
    for fc in self.feature_configs:
      name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
      by_input.setdefault(fc.input_names[0], name)
    for m in self.eval_config.metrics_set:
      which = m.WhichOneof('metric')
      if which in ('gauc', 'session_auc'):
        conf = getattr(m, which)
        field = conf.uid_field if which == 'gauc' else conf.session_id_field
        feat = by_input.get(field, field)
        if feat not in self.input_layer.sparse_names:
          raise ValueError('%s: key field %r is not a single-valued id feature of this model' % (which, field))
        out.append((which, self.input_layer.sparse_names.index(feat), conf.reduction))
    return out

  def _eval_batches(self, input_fn, steps=None):
    """(host features, device features, device labels, own) for evaluate / predict: this rank's batches (at most
    `steps`).  Row-sharded tables with world_size > 1: every forward takes part in the exchange, so a rank whose batches
    are used up repeats a forward of its last batch (own = False: outputs dropped) until every rank is out - one host
    all-reduce per forward decides."""
    gang = self._ep and self._world > 1
    it = iter(input_fn())
    n, had, last = 0, False, None
    while True:
      item = next(it, None) if (steps is None or n < steps) else None
      if gang:
        anyone, stranded = self._agree([item is not None, item is None and not had], 'max')
        if not anyone:
          return
        if stranded:
          raise ValueError('evaluate / predict under row-sharded tables: a rank has no full batch of its own to take '
                           'part in the exchanges of the others')
      elif item is None:
        return
      if item is None:
        yield None, last[0], last[1], False
        continue
      had = True
      n += 1
      last = readers.to_device(item[0], item[1], self._device)
      yield item[0], last[0], last[1], True

  def evaluate(self, input_fn, steps=None, hooks=None, checkpoint_path=None, name=None):
    """One pass over input_fn() (or `steps` batches) -> {metric name: value, 'global_step'} for eval_config.metrics_set
    (no metrics_set: auc).  The streaming metrics (auc at AUC.num_thresholds thresholds as tf.metrics.auc computes it,
    max_f1, the mean / root-mean errors; every task tower of a multi-task model under '<metric>_<tower_name>') are
    accumulated on the device, batch by batch (metrics.MetricSet over er_auc_hist); the grouped AUCs gauc / session_auc
    are computed on the host over the collected predictions, as the reference's py_func does (core/metrics.py:59-106).
    `auc_exact` is the exact ROC AUC of the single binary head (what the thresholded `auc` approximates).

    world_size > 1: each rank evaluates what its input_fn yields, then the metrics are reduced over all ranks - the
    threshold histograms summed, the error totals and counts summed in rank order, `auc_exact` / `gauc` /
    `session_auc` computed over the labels, probabilities and keys of all ranks in rank order - so every rank returns
    the same dict, that of one process evaluating the union of the batches."""
    heads = metrics.heads_of(self.model)
    mset = metrics.MetricSet(self.eval_config.metrics_set, heads, self._device)
    single = len(heads) == 1 and heads[0][0] == '' and heads[0][1] == 'CLASSIFICATION'
    labels_all, probs_all = [], []
    groups = self._group_fields() if single else []
    keys_all = [[] for _ in groups]
    B = self.input_layer.batch_size
    n = 0
    for host, feats, labels, own in self._eval_batches(input_fn, steps):
      logits = self._forward_eval(feats)
      if not own:
        continue
      for k, (_, pos, _) in enumerate(groups):
        keys_all[k].append(readers.host_ids(host, pos, B))
      if heads:
        mset.update(logits, labels)
      if single:
        probs_all.append(torch.sigmoid(logits))
        labels_all.append(labels)
      n += 1
    lab = prob = None
    if probs_all:
      lab, prob = torch.cat(labels_all).cpu().numpy(), torch.cat(probs_all).cpu().numpy()
    keys = [np.concatenate(k) if k else None for k in keys_all]
    if self._world > 1:
      import torch.distributed as dist
      group = self._host_group()
      mset.all_reduce(group)
      parts = [None] * self._world
      dist.all_gather_object(parts, (n, lab, prob, keys), group=group)
      n = sum(p[0] for p in parts)
      got = [p for p in parts if p[1] is not None]
      if got:
        lab, prob = np.concatenate([p[1] for p in got]), np.concatenate([p[2] for p in got])
        keys = [np.concatenate([p[3][k] for p in got]) for k in range(len(groups))]
    out = {'global_step': self.global_step}
    if n and heads:
      out.update(mset.result())
    if lab is not None:
      out['auc_exact'] = metrics.auc(lab, prob)
      for (which, _, reduction), k in zip(groups, keys):
        out[which] = float(metrics.gauc(lab, prob, k, reduction))
    return out

  def predict(self, input_fn, predict_keys=None, hooks=None, checkpoint_path=None, yield_single_examples=True):
    """{'logits', 'probs'} per batch of input_fn(); world_size > 1: this rank's batches (every rank has to iterate to the
    end under row-sharded tables, whose forwards exchange rows)."""
    for _, feats, _, own in self._eval_batches(input_fn):
      logits = self._forward_eval(feats)
      if not own:
        continue
      yield {'logits': logits.cpu().numpy(), 'probs': torch.sigmoid(logits).cpu().numpy()}

  def save(self, model_dir=None, embedding_parts=False):
    """dense parameters + arenas (weights and optimizer state) as one torch checkpoint.  embedding_parts=True
    also writes every table and optimizer slot in the reference's row-sharded layout
    `model.ckpt-<step>-embedding/embed-<var>-part-<rank>.bin` (compat/embedding_parallel_saver.py:99-123),
    which `restore` can read back on a different number of workers."""
    model_dir = model_dir or self._pipeline_config.model_dir
    os.makedirs(model_dir, exist_ok=True)
    path = os.path.join(model_dir, 'model.ckpt-%d.pt' % self.global_step)
    do = self.trainer.dense_opt
    torch.save({'model': self.model.state_dict(),
                'arenas': {d: a.storage for d, a in self.input_layer.arenas.items()},
                'tables': {d: a.tables for d, a in self.input_layer.arenas.items()},
                # key-value tables: the (key, pool row) pairs of their indexes
                'kv': {d: a.kv.items() for d, a in self.input_layer.arenas.items() if a.kv is not None},
                # dense optimizer slots (Adagrad accumulators | Adam m, v), keyed by parameter name: the reference's
                # Saver stores every slot variable, a resumed run continues from them
                'dense_slots': {n: [None if st is None else st[o:o + k].clone() for st in (do.s0, do.s1)]
                                for n, o, k in do.named_ranges()},
                'trainer_step': self.trainer.step,
                'global_step': self.global_step}, path)
    if embedding_parts:
      for a in self.input_layer.arenas.values():
        if a.kv is not None:
          checkpoint.save_kv_arena(a, path[:-3])   # `.key` / `.val` parts
        else:
          checkpoint.save_arena(a, path[:-3])
    return path

  def restore(self, path):
    """`path` as returned by save().  Tables come from the part files next to it when they exist (re-sharded for
    this job's worker count by er_load_embed), else from the arenas stored in the torch checkpoint."""
    ck = torch.load(path, map_location='cpu')
    self.model.load_state_dict(ck['model'])
    self.global_step = int(ck['global_step'])
    # the step counter drives the learning-rate schedule and Adam's beta powers; the dense slots continue
    self.trainer.step = int(ck.get('trainer_step', self.global_step))
    do = self.trainer.dense_opt
    slots = ck.get('dense_slots')
    if slots is not None:
      for n, o, k in do.named_ranges():
        if n not in slots:
          raise KeyError('checkpoint has no optimizer slots for parameter %s' % n)
        for st, saved in zip((do.s0, do.s1), slots[n]):
          if st is not None and saved is not None:
            st[o:o + k].copy_(saved)
    parts = os.path.isdir(path[:-3] + '-embedding')
    for d, a in self.input_layer.arenas.items():
      if parts and a.kv is not None:
        checkpoint.restore_kv_arena(a, path[:-3])
      elif parts:
        checkpoint.restore_arena(a, path[:-3])
      else:
        assert ck['tables'][d] == a.tables, 'checkpoint was written with another table plan'
        a.storage.copy_(ck['arenas'][d])
        if a.kv is not None:
          a.kv.load(*ck['kv'][d])
    return self


def _input_path(cfg, which):
  """what make_input reads for `which` ('train' / 'eval'): the BinaryDataInput of binary_<which>_input when the
  <which>_path oneof holds it, else <which>_input_path"""
  if cfg.WhichOneof(which + '_path') == 'binary_%s_input' % which:
    return getattr(cfg, 'binary_%s_input' % which)
  return getattr(cfg, which + '_input_path')


def train_and_evaluate(pipeline_config_path, train_input_fn=None, eval_input_fn=None, device='cuda:0', **kw):
  """main._train_and_evaluate_impl (main.py:296-400) for the supported model families.  With world_size > 1 every rank
  reads its own shard of train_input_path and eval_input_path, or of binary_train_input and binary_eval_input
  (readers.make_input with this rank and world size)."""
  est = EasyRecEstimator(pipeline_config_path, device=device, **kw)
  cfg = est._pipeline_config
  if train_input_fn is None:
    path = _input_path(cfg, 'train')
    train_input_fn = lambda: readers.make_input(cfg, est.input_layer, path, est.rank, est.world_size)  # noqa: E731
  est.train(train_input_fn)
  epath = _input_path(cfg, 'eval')
  if eval_input_fn is None and epath:
    eval_input_fn = lambda: readers.make_input(cfg, est.input_layer, epath, est.rank, est.world_size)  # noqa: E731
  return est, (est.evaluate(eval_input_fn) if eval_input_fn else {})
