"""CPU: CriteoInput, the reference's binary Criteo parts (input/criteo_binary_reader.py, input/criteo_input.py).

* Batches: tests/golden/reference_criteo_batches.json holds the reference's own BinaryDataset batches at world sizes 1-4
  (make_criteo_golden.py).  Every full batch that does not cross a file boundary is bit-identical here; where the
  reference returns more than batch_size samples for a batch that crosses a boundary, the batch here is its first
  batch_size samples (the next batch_size in file order); the last partial batch the reference returns (or fails to
  read) is skipped here.  Parts of unequal sizes follow the cumulative shard rule.
* Columns: the refusals of every feature the files cannot feed without host work.
* Training, kernel doubles: the reference's dlrm_on_criteo.config and share_not_used.config (tables shrunk) trained
  through train_and_evaluate from binary parts equal the same samples written as text and read by CSVInput - losses,
  tables, dense parameters, predictions and the evaluate() dict (with a gauc keyed by a category column)."""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))

import binary_doubles  # noqa: E402
import host_doubles  # noqa: E402
import make_criteo_golden as gen  # noqa: E402
from easyrec_b200 import builder, estimator  # noqa: E402
from easyrec_b200.config import config_util  # noqa: E402
from easyrec_b200.input import readers  # noqa: E402
from test_config import reference_config  # noqa: E402

GOLD = json.load(open(os.path.join(HERE, 'golden', 'reference_criteo_batches.json')))


def small_cfg(features, B=8, extra=''):
  """a DeepFM over `features` (FeatureConfig texts) reading CriteoInput"""
  names = []
  for f in features:
    if 'SequenceFeature' in f:
      continue     # (declared only: a plain group cannot hold it)
    name = f.split('feature_name: "')[1].split('"')[0] if 'feature_name' in f else f.split('input_names: "')[1].split('"')[0]
    names.append('"%s"' % name)
  text = '''model_dir: "/tmp/er_criteo_small"
train_config { optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.1 } } } } }
data_config { batch_size: %d input_type: CriteoInput label_fields: "label" %s
  input_fields { input_name: "label" input_type: INT32 } }
feature_config { %s }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: [%s] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: [%s] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [8] use_bn: false } final_dnn { hidden_units: [4] use_bn: false } } }
''' % (B, extra, '\n'.join('features { %s }' % f for f in features), ', '.join(names), ', '.join(names))
  return config_util.get_configs_from_pipeline_file(text.encode())


# every id slot reads a column of its own, the dense columns in a permuted order; c26 holds the values past 2^31
PLAN = ['input_names: "f3" feature_type: RawFeature embedding_dim: 4 min_val: 0.0 max_val: 10.0',
        'input_names: "c26" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 97',
        'input_names: "f1" feature_type: RawFeature embedding_dim: 4',
        'input_names: "c2" feature_type: IdFeature embedding_dim: 4 num_buckets: 1000000']


def _layer(cfg, B=8):
  il, _, _ = builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  return il


class _Paths(object):
  def __init__(self, label, dense, category):
    self.label_path, self.dense_path, self.category_path = label, dense, category


def _raw(batch):
  """a BinaryBatch -> (label, dense, category uint32) numpy"""
  return batch.label.numpy(), batch.dense.numpy(), batch.cat.numpy().view(np.uint32)


@pytest.mark.parametrize('case', sorted(GOLD['cases']))
def test_batches_replay_the_reference_reader(tmp_path, case):
  B = GOLD['batch_size']
  sizes = GOLD['cases'][case]['sizes']
  labels, denses, cats = gen.write_parts(str(tmp_path), sizes)
  cfg = small_cfg(PLAN, B)
  il = _layer(cfg, B)
  bounds = np.cumsum(sizes)
  same = straddle = partial = 0
  for n, ranks in GOLD['cases'][case]['worlds'].items():
    for r, want in enumerate(ranks):
      rd = readers.CriteoBinaryInput(cfg, il, _Paths(labels, denses, cats), task_index=r, task_num=int(n))
      got = [_raw(b) for b, lab in rd]
      assert all(lab is None for _, lab in rd)
      start, count = readers.criteo_shard(sum(sizes), r, int(n))
      assert len(got) == count // B
      assert got[0][0][0] == start if got else True
      for k, (lab, dense, cat) in enumerate(got):
        ref = want[k]
        first = start + k * B
        np.testing.assert_array_equal(lab, np.arange(first, first + B))
        n_ref = len(ref['label'])
        crosses = bool(((bounds > first) & (bounds < first + B)).any())
        if not crosses:
          assert n_ref == B
          same += 1
        else:
          # the reference keeps the batch's end in the first file's coordinates and reads on in the next file
          f = int(np.searchsorted(bounds, first, side='right'))
          in_next = min(first - (bounds[f - 1] if f else 0) + B, sizes[f + 1])
          assert n_ref == bounds[f] - first + in_next > B
          straddle += 1
        np.testing.assert_array_equal(lab, np.array(ref['label'][:B], np.int32))
        np.testing.assert_array_equal(dense.reshape(-1), np.array(ref['dense'][:B * 13], np.float32))
        np.testing.assert_array_equal(cat.reshape(-1), np.array(ref['category'][:B * 26], np.uint32))
      # the reference's last partial batch (or the failure to read it past the last file it opened) is skipped here
      assert len(want) == len(got) + (1 if count % B else 0)
      if count % B:
        last = want[-1]
        assert 'error' in last or last['label'][0] == start + len(got) * B
        partial += 1
  assert same and straddle and partial


def test_unequal_parts_follow_the_cumulative_rule(tmp_path):
  """the reference's walk to a rank's first file adds the NEXT file's size (criteo_binary_reader.py:87-89); here the
  rank's range is taken in the concatenation of the parts, whatever their sizes"""
  sizes = [5, 30, 7, 19, 1, 12]
  labels, denses, cats = gen.write_parts(str(tmp_path), sizes)
  cfg = small_cfg(PLAN, 4)
  il = _layer(cfg, 4)
  for N in (1, 2, 3, 4):
    seen = set()
    for r in range(N):
      start, count = readers.criteo_shard(sum(sizes), r, N)
      got = list(readers.CriteoBinaryInput(cfg, il, _Paths(labels, denses, cats), task_index=r, task_num=N, batch_size=4))
      assert len(got) == count // 4
      for k, (b, _) in enumerate(got):
        lab, dense, cat = _raw(b)
        want = gen.samples(start + 4 * k, start + 4 * k + 4)
        np.testing.assert_array_equal(lab, want[0])
        np.testing.assert_array_equal(dense, want[1])
        np.testing.assert_array_equal(cat, want[2])
        seen.update(lab.tolist())
      assert count == -(-sum(sizes) // N)
    assert len(seen) >= sum(sizes) // 4 * 4 - 4 * N


def test_unpack_places_columns_by_input_name(tmp_path, monkeypatch):
  binary_doubles.install(monkeypatch.setattr)
  labels, denses, cats = gen.write_parts(str(tmp_path), [16])
  cfg = small_cfg(PLAN, 8)
  il = _layer(cfg, 8)
  rd = readers.CriteoBinaryInput(cfg, il, _Paths(labels, denses, cats))
  assert il.sparse_names == ['c26', 'c2'] and il.raw_names == ['f3', 'f1']
  np.testing.assert_array_equal(rd.slot_cols, [25, 1])
  np.testing.assert_array_equal(rd.raw_cols, [2, 0])
  batch, _ = next(iter(rd))
  feats, lab = readers.to_device(batch, None, 'cpu')
  lab_w, dense_w, cat_w = gen.samples(0, 8)
  ids = cat_w.view(np.int32).astype(np.int64)
  np.testing.assert_array_equal(feats['sparse_fea'].numpy(), np.concatenate([ids[:, 25], ids[:, 1]]))
  assert feats['sparse_fea'].numpy()[0] == -2**31   # uint32 2^31 read as int32
  np.testing.assert_array_equal(feats['dense_fea'].numpy(), dense_w[:, [2, 0]])
  assert lab.dtype == torch.float32 and np.array_equal(lab.numpy(), lab_w.astype(np.float32))
  np.testing.assert_array_equal(readers.host_ids(batch, 1, 8), ids[:, 1])
  # through the feeder on a CPU device: the same batch
  (f2, l2), = list(readers.DeviceFeeder([(batch, None)], 'cpu'))
  assert torch.equal(f2['sparse_fea'], feats['sparse_fea']) and torch.equal(f2['dense_fea'], feats['dense_fea'])
  assert torch.equal(l2, lab)


@pytest.mark.parametrize('feature,what', [
    ('input_names: "f1" feature_type: RawFeature embedding_dim: 4 boundaries: [0.5, 1.0]', 'bucketized'),
    ('input_names: "c3" feature_type: RawFeature embedding_dim: 4', 'dense column'),
    ('input_names: "f4" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 10', 'category column'),
    ('input_names: "c27" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 10', 'f1..f13 / c1..c26'),
    ('input_names: "f14" feature_type: RawFeature embedding_dim: 4', 'f1..f13 / c1..c26'),
    ('input_names: "user" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 10', 'f1..f13 / c1..c26'),
    ('input_names: "c5" feature_type: TagFeature embedding_dim: 4 hash_bucket_size: 10', 'TagFeature'),
    ('input_names: "c5" feature_type: SequenceFeature embedding_dim: 4 hash_bucket_size: 10', 'SequenceFeature'),
    ('feature_name: "cx" input_names: ["c5", "c6"] feature_type: ComboFeature embedding_dim: 4 hash_bucket_size: 10',
     'ComboFeature'),
    ('input_names: "f2" feature_type: RawFeature embedding_dim: 4 raw_input_dim: 2', 'raw_input_dim'),
])
def test_features_the_files_cannot_feed_are_refused_by_name(feature, what):
  cfg = small_cfg(['input_names: "c1" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 10', feature])
  name = feature.split('"')[1]
  il = _layer(cfg)
  with pytest.raises((ValueError, NotImplementedError), match=r'feature %s:.*%s' % (name, what.replace('.', r'\.'))):
    readers.make_input(cfg, il, _Paths(['l'], ['d'], ['c']))


def test_string_paths_and_mismatched_lists_are_refused(tmp_path):
  cfg = small_cfg(PLAN)
  il = _layer(cfg)
  with pytest.raises(ValueError, match='binary_train_input'):
    readers.make_input(cfg, il, 'train.csv')
  labels, denses, cats = gen.write_parts(str(tmp_path), [8, 8])
  with pytest.raises(ValueError, match='as many entries'):
    readers.make_input(cfg, il, _Paths(labels, denses[:1], cats))
  with pytest.raises(ValueError, match='match 2, 1 and 2 files'):
    readers.make_input(cfg, il, _Paths([str(tmp_path / '*label.bin')], [denses[0]], [str(tmp_path / '*category.bin')]))
  with open(cats[1], 'ab') as f:
    f.write(b'\0\0\0\0')
  with pytest.raises(ValueError, match='samples of 104 bytes'):
    readers.make_input(cfg, il, _Paths(labels, denses, cats))
  bad = small_cfg(PLAN, extra='sample_weight: "w"')
  with pytest.raises(NotImplementedError, match='sample_weight'):
    readers.make_input(bad, _layer(bad), _Paths(labels, denses, cats))
  strs = small_cfg(PLAN, extra='input_fields { input_name: "c2" input_type: STRING }')
  with pytest.raises(NotImplementedError, match='feature c2: .*STRING'):
    readers.make_input(strs, _layer(strs), _Paths(labels, denses, cats))


# ---- training from the reference's CriteoInput configs -----------------------------------------------------------------
def write_samples(dirname, n, seed, n_parts=3):
  """n Criteo-like samples as binary parts and the same samples as a CSV file (float32 values written as their
  shortest repr, which reads back to the same float32) -> (BinaryDataInput-like paths, csv path)"""
  rng = np.random.default_rng(seed)
  label = (rng.uniform(size=n) < 0.3).astype(np.int32)
  dense = rng.lognormal(1.0, 1.5, (n, 13)).astype(np.float32)
  cat = rng.integers(0, 2**31, (n, 26)).astype(np.uint32)
  cat[:, :4] %= 7            # small key spaces: gauc groups with several samples
  cuts = np.linspace(0, n, n_parts + 1).astype(int)
  paths = ([], [], [])
  for p in range(n_parts):
    for kind, a, lst in zip(('label', 'dense', 'category'), (label, dense, cat), paths):
      lst.append(os.path.join(dirname, 'p%d_%s.bin' % (p, kind)))
      a[cuts[p]:cuts[p + 1]].tofile(lst[-1])
  csv = os.path.join(dirname, 'all.csv')
  with open(csv, 'w') as f:
    for i in range(n):
      f.write(','.join([str(label[i])] + [str(x) for x in dense[i]] + [str(int(x)) for x in cat[i].view(np.int32)]) + '\n')
  return paths, csv


def criteo_pair(rel, dirname, B, steps, n=None, seed=0):
  """(binary config, csv config) of a reference CriteoInput sample config: tables shrunk, B per batch, `steps` steps,
  gauc on c2; the binary one reads binary_train_input / binary_eval_input, the other the same samples as a CSV file"""
  (lp, dp, cp), csv = write_samples(dirname, n or 6 * B, seed)
  out = []
  for binary in (True, False):
    cfg = config_util.get_configs_from_pipeline_file(reference_config(rel))
    edits = {'data_config.batch_size': B, 'train_config.num_steps': steps, 'model_dir': os.path.join(dirname, 'm%d' % binary)}
    for i, fc in enumerate(config_util.get_feature_configs(cfg)):
      if fc.hash_bucket_size > 0:
        edits['feature_config.features[%d].hash_bucket_size' % i] = 1009
    config_util.edit_config(cfg, edits)
    cfg.eval_config.metrics_set.add().gauc.uid_field = 'c2'
    if binary:
      for msg in (cfg.binary_train_input, cfg.binary_eval_input):
        del msg.label_path[:], msg.dense_path[:], msg.category_path[:]
        msg.label_path.extend(lp)
        msg.dense_path.extend(dp)
        msg.category_path.extend(cp)
    else:
      cfg.data_config.input_type = cfg.data_config.CSVInput
      cfg.train_input_path = csv
      cfg.eval_input_path = csv
    out.append(cfg)
  return out


def _train(cfg, device, record, **kw):
  losses = []
  est_cls = estimator.EasyRecEstimator
  orig = est_cls.__init__

  def init(self, *a, **k):
    orig(self, *a, **k)
    step = self.trainer.train_step

    def train_step(*a2, **k2):
      loss, probs = step(*a2, **k2)
      losses.append(float(loss))
      return loss, probs
    self.trainer.train_step = train_step
  record.setattr(est_cls, '__init__', init)
  est, metrics = estimator.train_and_evaluate(cfg, device=device, seed=3, **kw)
  record.setattr(est_cls, '__init__', orig)
  return est, metrics, losses


def same_training(a, b):
  (ea, ma, la), (eb, mb, lb) = a, b
  assert la == lb and len(la) > 0
  assert ma == mb and 'gauc' in ma and 'auc' in ma
  for (na, pa), (nb, pb) in zip(ea.model.state_dict().items(), eb.model.state_dict().items()):
    assert na == nb and torch.equal(pa, pb), na
  for d in ea.input_layer.arenas:
    assert torch.equal(ea.input_layer.arenas[d].storage, eb.input_layer.arenas[d].storage), d


@pytest.mark.parametrize('rel', ['samples/model_config/dlrm_on_criteo.config', 'samples/model_config/share_not_used.config'])
def test_reference_criteo_configs_train_from_binary_parts_like_from_text(tmp_path, monkeypatch, rel):
  host_doubles.install_all(monkeypatch.setattr)
  binary_doubles.install(monkeypatch.setattr)
  cb, cc = criteo_pair(rel, str(tmp_path), 16, 5)
  assert builder.input_type_name(cb) == 'CriteoInput' and cb.WhichOneof('train_path') == 'binary_train_input'
  a = _train(cb, 'cpu', monkeypatch)
  b = _train(cc, 'cpu', monkeypatch)
  assert len(a[2]) == 5        # 6 batches a pass: 5 steps
  same_training(a, b)
  pa = [p['probs'] for p in a[0].predict(lambda: readers.make_input(cb, a[0].input_layer, cb.binary_eval_input))]
  pb = [p['probs'] for p in b[0].predict(lambda: readers.make_input(cc, b[0].input_layer, cc.eval_input_path))]
  assert len(pa) == 6 and all(np.array_equal(x, y) for x, y in zip(pa, pb))
