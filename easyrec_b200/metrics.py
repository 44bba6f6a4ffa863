"""Evaluation metrics of the rank models (model/rank_model.py:334-470).

Streaming, on the device (`MetricSet`): the metrics the reference accumulates batch by batch in its eval graph -
`auc` (tf.metrics.auc: confusion counts at `num_thresholds` thresholds, trapezoidal ROC area), `max_f1`
(core/metrics.py:25-56, the same counts at 200 thresholds over the logits), `mean_absolute_error`,
`mean_squared_error`, `root_mean_squared_error`.  One `er_auc_hist` launch per head and batch adds into uint64
histograms in device memory; an evaluate() pass reads 2 * (T + 1) counters back at the end.

Exact, on the host: `auc` (the Mann-Whitney statistic with average ranks over ties = sklearn.metrics.roc_auc_score)
and the grouped AUCs `gauc` / `session_auc` (core/metrics.py:59-106 `_separated_auc_impl`, :260-298), which the
reference computes on the host as well (a py_func over the collected predictions calling sklearn per group)."""
import numpy as np


def _tie_averaged_ranks(scores):
  """1-based ranks, equal scores sharing the mean of their positions."""
  order = np.argsort(scores, kind='mergesort')
  s = scores[order]
  first = np.concatenate([[True], s[1:] != s[:-1]])
  start = np.flatnonzero(first)
  end = np.concatenate([start[1:], [len(s)]])
  mean_rank = 0.5 * (start + end - 1) + 1
  ranks = np.empty(len(s), np.float64)
  ranks[order] = np.repeat(mean_rank, end - start)
  return ranks


def auc(labels, scores):
  labels = np.asarray(labels).reshape(-1).astype(np.float64)
  scores = np.asarray(scores).reshape(-1).astype(np.float64)
  n_pos = labels.sum()
  n_neg = len(labels) - n_pos
  if n_pos == 0 or n_neg == 0:
    return float('nan')
  ranks = _tie_averaged_ranks(scores)
  return float((ranks[labels > 0].sum() - n_pos * (n_pos + 1) / 2) / (n_pos * n_neg))


def gauc(labels, scores, keys, reduction='mean'):
  """AUC per key (user / session), groups with a single class skipped, averaged with weight 1 ('mean'), the
  group's sample count ('mean_by_sample_num') or its positive count ('mean_by_positive_num'); 0.0 when no group
  qualifies.  float32 like the reference's value op."""
  assert reduction in ['mean', 'mean_by_sample_num', 'mean_by_positive_num'], \
      'reduction method must in mean | mean_by_sample_num | mean_by_positive_num'
  labels = np.asarray(labels).reshape(-1).astype(np.float64)
  scores = np.asarray(scores).reshape(-1).astype(np.float64)
  keys = np.asarray(keys).reshape(-1)
  order = np.argsort(keys, kind='mergesort')
  k = keys[order]
  bounds = np.flatnonzero(np.concatenate([[True], k[1:] != k[:-1], [True]]))
  metrics, weights = [], []
  for a, b in zip(bounds[:-1], bounds[1:]):
    idx = order[a:b]
    lab = labels[idx]
    pos = lab.sum()
    if pos == 0 or pos == len(lab):
      continue
    metrics.append(auc(lab, scores[idx]))
    weights.append({'mean': 1, 'mean_by_sample_num': len(lab), 'mean_by_positive_num': pos}[reduction])
  if not metrics:
    return np.float32(0.0)
  return np.average(metrics, weights=weights).astype(np.float32)


# ---- streaming metrics (device accumulators) ---------------------------------------------------------------------
def tf_thresholds(num_thresholds=200):
  """threshold list of tf.metrics.auc (and core/metrics.py:33-38), as the float32 constants the eval graph holds."""
  if not 2 <= int(num_thresholds) <= 4095:
    raise ValueError('auc.num_thresholds must be in [2, 4095], got %d' % num_thresholds)
  kepsilon = 1e-7
  t = [(i + 1) * 1.0 / (num_thresholds - 1) for i in range(num_thresholds - 2)]
  return np.array([0.0 - kepsilon] + t + [1.0 + kepsilon], np.float32)


class ConfusionAtThresholds(object):
  """tp / fn / tn / fp at TF's thresholds, accumulated on the device (er_auc_hist)."""

  def __init__(self, num_thresholds, device):
    import torch
    self.T = int(num_thresholds)
    self.thr = torch.from_numpy(tf_thresholds(self.T)).to(device)
    self.hist = torch.zeros(2 * (self.T + 1), dtype=torch.int64, device=device)

  def update(self, predictions, labels):
    import torch
    from easyrec_b200 import kernels as K
    K.auc_hist(predictions.detach().to(torch.float32), labels.detach().to(torch.float32), self.thr, self.hist)

  def all_reduce(self, group):
    """sum the histograms of all ranks (uint64 counts: exact, in any order)"""
    import torch.distributed as dist
    h = self.hist.cpu()
    dist.all_reduce(h, op=dist.ReduceOp.SUM, group=group)
    self.hist.copy_(h)

  def counts(self):
    """(tp, fn, tn, fp) float32 [T] (TF keeps the accumulators in float32 variables)."""
    h = self.hist.cpu().numpy()
    neg, pos = np.cumsum(h[:self.T + 1]), np.cumsum(h[self.T + 1:])
    tp = (pos[-1] - pos[:self.T]).astype(np.float32)   # predictions above more than i thresholds exceed thr[i]
    fp = (neg[-1] - neg[:self.T]).astype(np.float32)
    return tp, np.float32(pos[-1]) - tp, np.float32(neg[-1]) - fp, fp

  def auc(self):
    """tf.metrics.auc, curve ROC, trapezoidal summation."""
    tp, fn, tn, fp = self.counts()
    eps = np.float32(1e-6)
    y = (tp + eps) / (tp + fn + eps)
    x = fp / (fp + tn + eps)
    return float(np.sum((x[:-1] - x[1:]) * ((y[:-1] + y[1:]) / np.float32(2.0)), dtype=np.float32))

  def max_f1(self):
    """core/metrics.py:40-54: max over thresholds of 2 p r / (p + r + 1e-12); tf.metrics.precision / recall are 0 when
    their denominator is 0."""
    tp, fn, tn, fp = self.counts()
    with np.errstate(divide='ignore', invalid='ignore'):
      prec = np.where(tp + fp > 0, tp / (tp + fp), np.float32(0))
      rec = np.where(tp + fn > 0, tp / (tp + fn), np.float32(0))
    return float(np.max(2 * prec * rec / (prec + rec + np.float32(1e-12))))


class StreamingMean(object):
  """tf.metrics.mean: total and count accumulated on the device."""

  def __init__(self, device):
    import torch
    self.total = torch.zeros((), dtype=torch.float64, device=device)
    self.count = 0

  def update(self, values):
    self.total += values.detach().double().sum()
    self.count += values.numel()

  def all_reduce(self, group):
    """totals and counts of all ranks, summed in rank order: every rank gets the same bits"""
    import torch.distributed as dist
    parts = [None] * dist.get_world_size(group)
    dist.all_gather_object(parts, (float(self.total), self.count), group=group)
    total = 0.0
    for t, _ in parts:
      total += t
    self.total.fill_(total)
    self.count = sum(c for _, c in parts)

  def result(self):
    return float(self.total) / max(self.count, 1)


class MetricSet(object):
  """eval_config.metrics_set over the heads of a model (RankModel._build_metric_impl, model/rank_model.py:334-496;
  MultiTaskModel.build_metric_graph gives every tower's metrics the suffix '_<tower_name>').

  heads: [(suffix, loss_type, label column or None)].  update(logits, labels) per batch, result() at the end.
  The prediction a metric reads follows the reference: auc - probs; max_f1 - LOGITS (rank_model.py:421-426);
  the error metrics - `y` under L2_LOSS (the logits) / SIGMOID_L2_LOSS (their sigmoid), `probs` under CLASSIFICATION."""
  STREAMING = ('auc', 'max_f1', 'mean_absolute_error', 'mean_squared_error', 'root_mean_squared_error')

  def __init__(self, metrics_set, heads, device):
    self.heads = list(heads)
    self.acc = []   # (key, kind, head index, accumulator)
    kinds = [(m.WhichOneof('metric'), m) for m in metrics_set]
    default = not kinds
    if default:   # no metrics_set: auc for the binary heads (a regression head has no default metric)
      kinds = [('auc', None)]
    for which, m in kinds:
      if which not in self.STREAMING:
        continue
      for h, (suffix, loss_type, _) in enumerate(self.heads):
        binary = loss_type == 'CLASSIFICATION'
        if which in ('auc', 'max_f1'):
          if not binary and default:
            continue
          if not binary:
            raise ValueError('%s needs a binary classification head (loss_type %s)' % (which, loss_type))
          T = int(m.auc.num_thresholds) if (which == 'auc' and m is not None) else 200
          a = ConfusionAtThresholds(T, device)
        else:
          a = StreamingMean(device)
        self.acc.append((which + suffix, which, h, a))

  def update(self, logits, labels):
    import torch
    for key, which, h, a in self.acc:
      _, loss_type, col = self.heads[h]
      lg = logits if logits.dim() == 1 else logits[:, h]
      lab = labels if labels.dim() == 1 else labels[:, col if col is not None else h]
      if which == 'max_f1':
        a.update(lg, lab)
      elif which == 'auc':
        a.update(torch.sigmoid(lg), lab)
      else:
        pred = lg if loss_type == 'L2_LOSS' else torch.sigmoid(lg)
        d = lab.to(torch.float32) - pred
        a.update(d.abs() if which == 'mean_absolute_error' else d * d)

  def all_reduce(self, group):
    """every accumulator reduced over the ranks of `group` (torch.distributed, host tensors)"""
    for _, _, _, a in self.acc:
      a.all_reduce(group)

  def result(self):
    out = {}
    for key, which, h, a in self.acc:
      if which == 'auc':
        out[key] = a.auc()
      elif which == 'max_f1':
        out[key] = a.max_f1()
      elif which == 'root_mean_squared_error':
        out[key] = float(np.sqrt(a.result()))
      else:
        out[key] = a.result()
    return out


def heads_of(model):
  """[(suffix, loss_type, label column)] of a built model: one un-suffixed head for the rank models, one per task
  tower ('_<tower_name>', multi_task_model.py:124-141) for the multi-task models; [] for models without a binary /
  regression head (list-wise match models)."""
  towers = list(getattr(model, 'tower_names', []) or [])
  if towers:
    cols = getattr(model, 'label_cols', None) or list(range(len(towers)))
    lts = getattr(model, 'task_loss_types', None) or ['CLASSIFICATION'] * len(towers)
    return [('_' + n, lts[t], cols[t]) for t, n in enumerate(towers)]
  if getattr(model, 'listwise', False):
    return []
  return [('', getattr(model, 'loss_type', 'CLASSIFICATION'), None)]
