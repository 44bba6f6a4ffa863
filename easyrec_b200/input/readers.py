"""Host-side inputs: EasyRec data_config -> packed batches for InputLayer.

Counterpart of input/input.py:806-939 (`_preprocess`) + input/csv_input.py:78-175 +
input/parquet_input.py:201-239 restricted to the feature types of the hot path.  A batch is the reference's packed form (input/parquet_input.py:201-239):
  sparse_fea int64 [n_id*B] feature-major | dense_fea fp32 [B, sum raw_dim] | seq_fea | tag_fea | labels.

String-typed id fields with a hash_bucket_size are bucketed where their bytes are, on the host, by the native
parser: Fingerprint64(bytes) % hash_bucket_size (StringToHashBucketFast, feature_column_v2.py:3915-3921), '' -> -1
(the ignored value of string columns, :2566-2585), and the table plan takes those buckets unchanged; integer
fields go to the device untouched and are hashed there from their decimal text (input/input.py:541-543).
"""
import ctypes
import glob
import os
import re

import numpy as np
import torch

from easyrec_b200 import _lib
from easyrec_b200.config import config_util


def bucketize_raw(x, fc):
  """RawFeature with boundaries: float32 value -> bucket id, as the reference graph computes it:
  (x - min) / (max - min) when max > min (input/input.py:638-640, float32), then the number of boundaries <= x
  (bucketized_column, feature_column_v2.py:2866-2870)."""
  from easyrec_b200 import builder
  x = np.asarray(x, np.float32)
  x = _normalized_raw(x, fc)
  bounds = np.asarray(builder.raw_boundaries(fc), np.float32)
  return np.searchsorted(bounds, x, side='right').astype(np.int64)


def _normalized_raw(x, fc):
  """(x - min) / (max - min) when max > min, then RawFeature.normalizer_fn (input/input.py:638-646), float32"""
  if fc.max_val > fc.min_val:
    x = (x - np.float32(fc.min_val)) / np.float32(fc.max_val - fc.min_val)
  if getattr(fc, 'normalizer_fn', ''):
    from easyrec_b200 import normalizer
    x = normalizer.load(fc.normalizer_fn, 'numpy')(x)
  return x


_STEP_KINDS = (_lib.CSV_I64_STEP_LIST, _lib.CSV_HASH_STEP_LIST)
_LIST_KINDS = (_lib.CSV_I64_LIST, _lib.CSV_HASH_LIST, _lib.CSV_I64_KV_LIST, _lib.CSV_HASH_KV_LIST, _lib.CSV_F32_LIST) + _STEP_KINDS
FP_EMPTY = 0x9ae16a3b2f90404f       # Fingerprint64('')
CROSS_HASH_KEY = 0xDECAFCAFFE       # sparse_ops._DEFAULT_HASH_KEY, what crossed_column(hash_key=None) uses


def fingerprint_cat64(fp1, fp2):
  """tensorflow::FingerprintCat64 on uint64 arrays (platform/fingerprint.h): how the SparseCross kernel folds
  the next column's feature into the running hash."""
  k = np.uint64(0xc6a4a7935bd1e995)
  s47 = np.uint64(47)
  with np.errstate(over='ignore'):
    r = fp1 ^ k
    t = fp2 * k
    r = r ^ ((t ^ (t >> s47)) * k)
    r = r * k
    r = (r ^ (r >> s47)) * k
    return r ^ (r >> s47)


def cross_hash(fingerprints, num_buckets, hash_key=CROSS_HASH_KEY):
  """crossed_column / sparse_cross_hashed over one value per column: `fingerprints` = list of uint64 arrays (a
  string input contributes Fingerprint64(bytes), an integer column its value), folded left to right from hash_key,
  then % num_buckets as uint64 (feature_column_v2.py:4532-4552)."""
  h = np.full(np.asarray(fingerprints[0]).shape, hash_key, np.uint64)
  for fp in fingerprints:
    h = fingerprint_cat64(h, np.asarray(fp).astype(np.uint64))
  return (h % np.uint64(num_buckets)).astype(np.int64)


def string_keys(values):
  """strings -> the 63-bit keys of a vocabulary column, Fingerprint64(bytes) % (2^63 - 1), as the CSV parser keys them
  (er_csv_parse with hash_mod 2^63 - 1); '' and nulls -> -1, the ignored value of string columns
  (feature_column_v2.py:2566-2585)"""
  return np.array([_lib.fingerprint64(v) % _lib.KV_BUCKETS if v else -1 for v in values], np.int64)


def fingerprint_i64(values):
  """Fingerprint64 of the decimal text of int64 values (tf.as_string first, input/input.py:356-376)."""
  v = np.ascontiguousarray(values, np.int64)
  out = np.empty(v.shape, np.uint64)
  _lib.check(_lib.load().er_fingerprint64_i64(v.ctypes.data, v.size, out.ctypes.data), 'er_fingerprint64_i64')
  return out


def _combo_features(pipeline_config, input_layer):
  """feature name -> (input field names, hash_bucket_size) for the ComboFeatures of the plan."""
  out = {}
  for fc in config_util.get_feature_configs(pipeline_config):
    ftype = fc.DESCRIPTOR.fields_by_name['feature_type'].enum_type.values_by_number[fc.feature_type].name
    name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
    if ftype == 'ComboFeature' and name in input_layer.sparse_names:
      out[name] = (list(fc.input_names), fc.hash_bucket_size)
  return out


def bucketize_raw_multi(x, fc):
  """[n, k] values of a k-wide bucketized RawFeature -> ids `bucket + (len(boundaries) + 1) * k_index`, row-major
  (feature_column_v2.py:2849-2870); the matching lens are k per sample."""
  from easyrec_b200 import builder
  x = np.asarray(x, np.float32).reshape(-1, fc.raw_input_dim)
  n_bucket = len(builder.raw_boundaries(fc)) + 1
  ids = bucketize_raw(x, fc) + n_bucket * np.arange(fc.raw_input_dim, dtype=np.int64)[None, :]
  return ids.reshape(-1), np.full(x.shape[0], fc.raw_input_dim, np.int32)


def _bucketized_features(pipeline_config, input_layer):
  """feature name -> FeatureConfig for the RawFeatures the plan treats as bucket ids."""
  from easyrec_b200 import builder
  out = {}
  for fc in config_util.get_feature_configs(pipeline_config):
    name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
    ftype = fc.DESCRIPTOR.fields_by_name['feature_type'].enum_type.values_by_number[fc.feature_type].name
    if ftype == 'RawFeature' and builder.raw_boundaries(fc) is not None and name in input_layer.features:
      out[name] = fc     # a single-valued id slot (raw_input_dim 1) or a fixed-length tag slot (raw_input_dim k)
  return out


def _tag_weight_inputs(pipeline_config):
  """TagFeature with a second input_names entry: that field holds the per-tag weights, split by the feature's own
  separator (input/input.py:477-497) -> {feature name: weight field}."""
  out = {}
  for fc in config_util.get_feature_configs(pipeline_config):
    if len(fc.input_names) > 1 and fc.DESCRIPTOR.fields_by_name['feature_type'].enum_type.values_by_number[
        fc.feature_type].name == 'TagFeature':
      name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
      if fc.HasField('kv_separator'):
        raise ValueError('Tag Feature Error, Cannot set kv_separator and multi input_names in one feature config. '
                         'Feature: %s.' % fc.input_names[0])
      out[name] = fc.input_names[1]
  return out


def _pad_tags(il, name, ids, lens, w):
  """tag feature of a backbone `embedding_layer` block: the reference densifies the ragged tags with '' up to the longest
  list of the BATCH and looks the padding up too (layers/input_layer.py:232-235); weights of the padding are 0.
  (ids, lens, w) numpy -> padded (ids, lens, w); a batch without any tag stays empty (embedding.py:69-72: zeros)."""
  entry = getattr(il, 'pad_tags', {}).get(name)
  if entry is None:
    return ids, lens, w
  pad, use_weights = entry
  if not use_weights:
    w = None                      # combiner mean / sum: reduce over the padded axis, weights unused (embedding.py:11-12)
  n = int(lens.max()) if lens.size else 0
  if n == 0 or bool((lens == n).all()):
    return ids, lens, w
  B = lens.size
  out = np.full((B, n), pad, np.int64)
  mask = np.arange(n)[None, :] < lens[:, None]
  out[mask] = ids
  wp = None
  if w is not None:
    wp = np.zeros((B, n), np.float32)
    wp[mask] = w
    wp = wp.reshape(-1)
  return out.reshape(-1), np.full(B, n, np.int32), wp


def _check_tag_weights(name, lens, wlens):
  """the weight field must hold one value per tag (input/input.py:490-494 asserts equal sizes; the two SparseTensors
  must then share their indices)"""
  if not np.array_equal(lens, wlens):
    raise ValueError('TagFeature Error: The size of %s not equal to the size of its weight input. Please check the input.'
                     % name)


def _expr_inputs(il):
  """the input fields of the ExprFeatures, columns of the batch's expr_fea (InputLayer.expr_inputs)"""
  return getattr(il, 'expr_inputs', ())


def _expr_features(il):
  """the ExprFeatures: raw columns the readers leave to er_expr_eval"""
  return [n for n, f in il.features.items() if getattr(f, 'expr', None) is not None]


def expr_number(x, field, ftype, default):
  """one raw value of an ExprFeature input field -> float64, as input/input.py:507-528 reads it: STRING and DOUBLE
  fields as decimal numbers (tf.string_to_number(.., tf.float64)), INT fields as integers, FLOAT fields rounded to
  float32 (the field's parsed type) and then widened.  An empty value takes the field's default_val; '' there is 0 for a
  number field and not a number for a STRING one.  Raises ValueError naming the field."""
  x = x if x != '' else (default or ('' if ftype == 'STRING' else '0'))
  try:
    t = x.strip(' \t')
    if '_' in t or 'x' in t or 'X' in t or t != t.strip():
      raise ValueError(x)
    if ftype in ('INT32', 'INT64'):
      return float(int(t))
    v = float(t)
    return float(np.float32(v)) if ftype == 'FLOAT' else v
  except ValueError:
    raise ValueError('input field %s (%s): %r is not a number; ExprFeature inputs are read with string_to_number'
                     % (field, ftype, x))


class DummyInput(object):
  """input/dummy_input.py:13-58: a constant in-memory batch, for pipeline-free throughput runs and tests."""

  def __init__(self, input_layer, n_labels=1, seed=0):
    self.il = input_layer
    self.n_labels = n_labels
    self.seed = seed

  def batch(self, step=0):
    il = self.il
    B = il.batch_size
    rng = np.random.default_rng(self.seed + step)
    feats = {}
    if il.sparse_names:
      ids = rng.integers(0, 2**40, len(il.sparse_names) * B, dtype=np.int64)
      feats['sparse_fea'] = torch.from_numpy(ids)
    if il.n_dense:
      feats['dense_fea'] = torch.from_numpy(rng.uniform(0, 1, (B, il.n_dense)).astype(np.float32))
    if _expr_inputs(il):   # small integers: the expressions' comparisons come out both ways, with ties
      feats['expr_fea'] = torch.from_numpy(rng.integers(0, 10, (B, len(_expr_inputs(il)))).astype(np.float64))
    seq, tag = {}, {}
    for f in il.features.values():
      if f.kind == 'seq' and f.name in getattr(il, 'multi_valued_seq', ()):
        # seq_multi_sep: (values of all steps back to back, steps per sample, values per (sample, step))
        lens = rng.integers(1, f.seq_len + 1, B).astype(np.int32)
        steps = np.where(np.arange(f.seq_len)[None, :] < lens[:, None], rng.integers(1, 4, (B, f.seq_len)), 0).astype(np.int32)
        seq[f.name] = (torch.from_numpy(rng.integers(0, 2**40, int(steps.sum()), dtype=np.int64)), torch.from_numpy(lens),
                       torch.from_numpy(steps.reshape(-1)))
      elif f.kind == 'seq':
        lens = rng.integers(1, f.seq_len + 1, B).astype(np.int32)
        seq[f.name] = (torch.from_numpy(rng.integers(0, 2**40, (B, f.seq_len), dtype=np.int64)),
                       torch.from_numpy(lens))
      elif f.kind == 'tag':
        lens = rng.integers(0, 5, B).astype(np.int32)
        tag[f.name] = (torch.from_numpy(rng.integers(0, 2**40, int(lens.sum()), dtype=np.int64)),
                       torch.from_numpy(lens), None)
    if seq:
      feats['seq_fea'] = seq
    if tag:
      feats['tag_fea'] = tag
    labels = (rng.uniform(size=(B, self.n_labels)) < 0.25).astype(np.float32)
    labels = torch.from_numpy(labels if self.n_labels > 1 else labels[:, 0])
    return feats, labels

  def __iter__(self):
    step = 0
    while True:
      yield self.batch(step)
      step += 1


class CSVInput(object):
  """CSVInput (input/csv_input.py): delimiter-separated text, one sample per line, columns in
  data_config.input_fields order; labels from label_fields.  Only Id / Raw / Sequence / Tag features.
  The file bytes go through the library's native parser (er_csv_parse_lines) straight into the batch arrays.

  task_index / task_num: worker `task_index` of `task_num` reads the lines `task_index::task_num` of the file (after the
  header), record by record like the reference's dataset.shard(task_num, task_index) (input/input.py:1018-1023); its
  batches are cut from its own lines in file order.  The parser threads default to the single-process rule divided by
  LOCAL_WORLD_SIZE, so the workers of one host share its cores."""

  def __init__(self, pipeline_config, input_layer, path, batch_size=None, seq_sep='|', engine='native', n_threads=None,
               task_index=0, task_num=1):
    self.cfg = pipeline_config
    self.il = input_layer
    self.path = path
    assert engine in ('native', 'python')
    self.engine = engine
    if not 0 <= task_index < task_num:
      raise ValueError('task_index %d is not in [0, task_num %d)' % (task_index, task_num))
    self.task_index, self.task_num = int(task_index), int(task_num)
    local_world = max(1, int(os.environ.get('LOCAL_WORLD_SIZE', 1)))
    self.n_threads = n_threads or max(1, min(16, (os.cpu_count() or 1) // 2) // local_world)
    dc = pipeline_config.data_config
    self.sep = dc.separator or ','
    self.fields = [f.input_name for f in dc.input_fields]
    self.ftypes = {f.input_name: dc.DESCRIPTOR.nested_types_by_name['Field'].fields_by_name['input_type']
                   .enum_type.values_by_number[f.input_type].name for f in dc.input_fields}
    self.defaults = {f.input_name: f.default_val for f in dc.input_fields}
    self.labels = list(dc.label_fields)
    # data_config.sample_weight: a float field that weighs each sample's loss (input/input.py:140-141)
    self.weight_field = dc.sample_weight if dc.HasField('sample_weight') else None
    self.batch_size = batch_size or input_layer.batch_size
    self.feature_inputs = {}
    self.hash_buckets = {}     # feature -> hash_bucket_size when its STRING field is hashed here, on the host
    self.bucketized = _bucketized_features(pipeline_config, input_layer)
    self.combos = _combo_features(pipeline_config, input_layer)
    self.kv_seps = {}          # TagFeature -> kv_separator: tokens are `id<kv>weight` (input/input.py:447-458)
    self.tag_weights = _tag_weight_inputs(pipeline_config)   # TagFeature -> the field that holds its weights
    # SequenceFeature -> seq_multi_sep: every step is a list of values (input/input.py:686-700)
    self.multi_seps = {(fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]): fc.seq_multi_sep
                       for fc in config_util.get_feature_configs(pipeline_config) if fc.HasField('seq_multi_sep')}
    # fields a cross reads: parsed to raw fingerprints (STRING) or integers (INT), every consumer derives from those
    self.cross_fields = set(f for fields, _ in self.combos.values() for f in fields)
    for fc in config_util.get_feature_configs(pipeline_config):
      name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
      self.feature_inputs[name] = (fc.input_names[0], fc.separator or seq_sep)
      if fc.HasField('kv_separator'):
        self.kv_seps[name] = fc.kv_separator
      if name in self.combos:
        continue
      if fc.hash_bucket_size > 0 and self.ftypes.get(fc.input_names[0]) == 'STRING' and name in input_layer.features:
        assert input_layer.features[name].bucket_mode in (_lib.BUCKET_IDENTITY, _lib.BUCKET_MOD), \
            'feature %s: the table plan must take host-hashed buckets (builder.feature_specs)' % name
        self.hash_buckets[name] = input_layer.features[name].num_buckets   # (2^63 - 1 for a key-value table)
      elif name in input_layer.features and input_layer.features[name].bucket_mode == _lib.BUCKET_VOCAB:
        # a vocabulary column: every raw string becomes its 63-bit key, Fingerprint64 % (2^63 - 1), the same transform
        # as a key-value table's strings; Tag / Sequence fields are read as strings whatever their declared type
        # (input/input.py:118-124)
        self.hash_buckets[name] = _lib.KV_BUCKETS

  def _token(self, x, feature):
    """one id token -> int64: Fingerprint64 % hash_bucket_size for a host-hashed STRING field ('' -> -1, the
    ignored value of string columns, feature_column_v2.py:2566-2585), else the integer it spells
    (input/input.py:544-555 string_to_number)."""
    nb = self.hash_buckets.get(feature)
    if nb:
      return _lib.fingerprint64(x) % nb if x != '' else -1
    return int(x)

  def _combo_column(self, cols, feature):
    """ComboFeature, one row at a time in python ints (the restatement the vectorised path is tested against)."""
    fields, nb = self.combos[feature]
    mask = (1 << 64) - 1
    k = 0xc6a4a7935bd1e995

    def cat(a, b):
      r = a ^ k
      t = (b * k) & mask
      r ^= ((t ^ (t >> 47)) * k) & mask
      r = (r * k) & mask
      r = ((r ^ (r >> 47)) * k) & mask
      return r ^ (r >> 47)
    out = []
    for i in range(len(cols[fields[0]])):
      h = CROSS_HASH_KEY
      for f in fields:
        x = cols[f][i] if cols[f][i] != '' else (self.defaults.get(f) or ('' if self.ftypes[f] == 'STRING' else '0'))
        h = cat(h, _lib.fingerprint64(x if self.ftypes[f] == 'STRING' else str(int(x))))
      out.append(h % nb)
    return np.array(out, np.int64)

  def _id_column(self, col, feature, default):
    if feature in self.bucketized:
      return bucketize_raw([float(x if x != '' else (default or 0)) for x in col], self.bucketized[feature])
    return np.array([self._token(x if x != '' else (default or ('' if feature in self.hash_buckets else '0')), feature)
                     for x in col], np.int64)

  def batches(self):
    return self._batches_native() if self.engine == 'native' else self._batches_python()

  # ---- native path: er_csv_parse fills the batch's column arrays straight from the file bytes ----
  def _column_plan(self):
    """per input field: (kind, width, inner_sep, default) -- what er_csv_parse extracts from it."""
    il = self.il
    plan = {}

    def want(field, spec):
      if plan.setdefault(field, spec) != spec:
        raise ValueError('input field %r is used by features that need different parsings' % field)
    for l in self.labels:
      want(l, (_lib.CSV_F32, 0, b',', 0.0, 0))
    if self.weight_field:
      want(self.weight_field, (_lib.CSV_F32, 0, b',', 1.0, 0))
    def raw_spec(field):
      """a field read by a cross: raw Fingerprint64 of a STRING field / the integer of an INT field."""
      if self.ftypes[field] == 'STRING':
        return (_lib.CSV_HASH, 0, b',', self.defaults.get(field) or '', 0)
      if self.ftypes[field] not in ('INT32', 'INT64'):
        raise NotImplementedError('ComboFeature input %r of type %s (as_string of a float needs its precision)'
                                  % (field, self.ftypes[field]))
      return (_lib.CSV_I64, 0, b',', int(self.defaults.get(field) or 0), 0)
    for n in il.sparse_names:
      src, _ = self.feature_inputs[n]
      if n in self.combos:
        for f in self.combos[n][0]:
          want(f, raw_spec(f))
      elif src in self.cross_fields:
        want(src, raw_spec(src))
      elif n in self.hash_buckets:
        want(src, (_lib.CSV_HASH, 0, b',', self.defaults.get(src) or '', self.hash_buckets[n]))
      elif n in self.bucketized:
        want(src, (_lib.CSV_F32, 0, b',', float(self.defaults.get(src) or 0), 0))
      else:
        want(src, (_lib.CSV_I64, 0, b',', int(self.defaults.get(src) or 0), 0))
    for n in il.raw_names:
      if n in _expr_features(il):
        continue   # (its column is the expression's, filled on the device from expr_fea)
      src, sep = self.feature_inputs[n]
      c0, c1 = il.raw_cols[n]
      if c1 - c0 == 1 and src in _expr_inputs(il) and self.ftypes[src] in ('INT32', 'INT64', 'DOUBLE'):
        # the field is also an ExprFeature input: parsed once, as int64 / float64 below, and rounded to float32 for the
        # raw column - the reference's own cast of an int / double field
        continue
      d = float(self.defaults.get(src) or 0)
      want(src, (_lib.CSV_F32, 0, b',', d, 0) if c1 - c0 == 1 else (_lib.CSV_F32_VEC, c1 - c0, sep.encode(), d, 0))
    for src in _expr_inputs(il):
      t, d = self.ftypes[src], self.defaults.get(src)
      if t in ('INT32', 'INT64'):
        want(src, (_lib.CSV_I64, 0, b',', int(d or 0), 0))
      elif t == 'FLOAT':
        want(src, (_lib.CSV_F32, 0, b',', float(d or 0), 0))
      else:   # STRING / DOUBLE: string_to_number(.., float64); an empty STRING default is not a number
        want(src, (_lib.CSV_F64, 0, b',', d or ('' if t == 'STRING' else '0'), 0))
    for f in il.features.values():
      if f.kind == 'tag' and f.name in self.bucketized:
        src, sep = self.feature_inputs[f.name]
        want(src, (_lib.CSV_F32_VEC, self.bucketized[f.name].raw_input_dim, sep.encode(), float(self.defaults.get(src) or 0), 0))
      elif f.kind in ('seq', 'tag'):
        src, sep = self.feature_inputs[f.name]
        nb = self.hash_buckets.get(f.name, 0)
        if f.kind == 'seq' and f.name in self.multi_seps:
          want(src, (_lib.CSV_HASH_STEP_LIST if nb else _lib.CSV_I64_STEP_LIST, f.seq_len, sep.encode(),
                     self.multi_seps[f.name], nb))
          continue
        if f.name in self.kv_seps:
          kind = _lib.CSV_HASH_KV_LIST if nb else _lib.CSV_I64_KV_LIST
        else:
          kind = _lib.CSV_HASH_LIST if nb else _lib.CSV_I64_LIST
        want(src, (kind, f.seq_len if f.kind == 'seq' else 0, sep.encode(), self.kv_seps.get(f.name, ''), nb))
        if f.kind == 'tag' and f.name in self.tag_weights:
          want(self.tag_weights[f.name], (_lib.CSV_F32_LIST, 0, sep.encode(), 0.0, 0))
    return plan

  def _parse(self, data, size, plan, list_cap, n_batches=1):
    """one er_csv_parse_lines call on `size` bytes at `data` (address or bytes) for up to n_batches * batch_size of this
    worker's lines - the first line of the buffer and every task_num-th one after it -> (n_rows, consumed, lines passed
    over, {field: arrays}), or None when a list column needs a larger array."""
    B = self.batch_size * n_batches
    list_cap = list_cap * n_batches
    cols = (_lib.ErCsvCol * len(self.fields))()
    out, keep = {}, []
    for i, name in enumerate(self.fields):
      kind, width, sep, default, hash_mod = plan.get(name, (_lib.CSV_SKIP, 0, b',', 0, 0))
      c = cols[i]
      c.kind, c.width, c.inner_sep, c.hash_mod = kind, width, sep, hash_mod
      if kind == _lib.CSV_I64:
        c.default_i64 = default
        out[name] = (np.empty(B, np.int64),)
      elif kind in (_lib.CSV_HASH, _lib.CSV_F64):
        keep.append(default.encode())
        c.default_str = keep[-1]
        out[name] = (np.empty(B, np.float64 if kind == _lib.CSV_F64 else np.int64),)
      elif kind == _lib.CSV_F32:
        c.default_f32 = default
        out[name] = (np.empty(B, np.float32),)
      elif kind == _lib.CSV_F32_VEC:
        c.default_f32 = default
        out[name] = (np.empty((B, width), np.float32),)
      elif kind in _STEP_KINDS:
        out[name] = (np.empty(list_cap, np.int64), np.empty(B, np.int32), np.empty(B * width, np.int32))
        c.lens = out[name][1].ctypes.data
        c.step_lens = out[name][2].ctypes.data
        c.list_cap = list_cap
        c.kv_sep = default.encode()       # the plan's default slot carries the separator of the values of a step
      elif kind in _LIST_KINDS:
        cap = B * width if width else list_cap
        out[name] = (np.empty(cap, np.float32 if kind == _lib.CSV_F32_LIST else np.int64), np.empty(B, np.int32))
        c.lens = out[name][1].ctypes.data
        c.list_cap = cap
        if kind in (_lib.CSV_I64_KV_LIST, _lib.CSV_HASH_KV_LIST):
          out[name] += (np.empty(cap, np.float32),)
          c.weights = out[name][2].ctypes.data
          c.kv_sep = default.encode()     # the plan's default slot carries the key / weight separator
      if kind != _lib.CSV_SKIP:
        c.out = out[name][0].ctypes.data
    n_rows, consumed, seen = ctypes.c_int64(0), ctypes.c_size_t(0), ctypes.c_int64(0)
    st = _lib.load().er_csv_parse_lines(data, size, self.sep.encode(), cols, len(self.fields), B, self.n_threads,
                                        self.task_num, 0, ctypes.byref(n_rows), ctypes.byref(consumed),
                                        ctypes.byref(seen))
    if st == _lib.ER_ERR_WORKSPACE:
      return None
    if st != _lib.ER_OK:
      msg = _lib.load().er_last_error().decode()
      m = re.search(r'field (\d+) ', msg)
      raise _lib.ErError('er_csv_parse_lines failed (status %d): %s%s' % (
          st, msg, ' (input field %s)' % self.fields[int(m.group(1)) - 1] if m else ''))
    for i, name in enumerate(self.fields):
      if cols[i].kind in _STEP_KINDS:
        out[name] = (out[name][0][:cols[i].n_vals], out[name][1], out[name][2])
      elif cols[i].kind in _LIST_KINDS:
        out[name] = (out[name][0][:cols[i].n_vals], out[name][1]) + tuple(w[:cols[i].n_vals] for w in out[name][2:])
    return n_rows.value, consumed.value, seen.value, out

  @staticmethod
  def _slice_chunk(cols, plan, k, B):
    """batch k of a chunk parsed in one call: row ranges of the scalar / vector columns, value ranges of the list
    columns (by the running sum of their per-row counts)."""
    out = {}
    for name, arrs in cols.items():
      kind, width = plan[name][0], plan[name][1]
      if kind in _STEP_KINDS:
        vals, lens, steps = arrs
        per_row = steps.reshape(-1, width).sum(1)
        lo, hi = int(per_row[:k * B].sum()), int(per_row[:(k + 1) * B].sum())
        out[name] = (vals[lo:hi], lens[k * B:(k + 1) * B], steps[k * B * width:(k + 1) * B * width])
      elif kind in _LIST_KINDS:
        lens = arrs[1]
        lo, hi = int(lens[:k * B].sum()), int(lens[:(k + 1) * B].sum())
        out[name] = (arrs[0][lo:hi], lens[k * B:(k + 1) * B]) + tuple(w[lo:hi] for w in arrs[2:])
      else:
        out[name] = (arrs[0][k * B:(k + 1) * B],)
    return out

  def _batches_native(self):
    """the file is memory-mapped and parsed in place; one er_csv_parse call takes a CHUNK of several batches (about
    32K lines) so that the parser's threads are started once per chunk, not once per batch, and have enough lines each;
    the last, short chunk of the file is parsed batch by batch.  `line` is the index (after the header) of the file line
    at `off`; before each call `off` moves on to this worker's next line, (task_index - line) mod task_num lines on."""
    import mmap
    B = self.batch_size
    N, me = self.task_num, self.task_index
    line = 0

    def own_line(off, line):
      for _ in range((me - line) % N):     # (at most task_num - 1 other workers' lines)
        nl = mm.find(b'\n', off)
        off = nl + 1 if nl >= 0 else size  # (an unterminated last line of another worker: nothing left)
        line += 1
      return off, line
    plan = self._column_plan()
    list_cap = 16 * B
    chunk = max(1, 32768 // B)
    if os.path.getsize(self.path) == 0:
      return
    with open(self.path, 'rb') as f, mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ) as mm:
      view = np.frombuffer(mm, np.uint8)
      try:
        base, size, off = view.ctypes.data, view.size, 0
        if self.cfg.data_config.with_header:      # the first line names the columns (csv_input.py:139-145)
          off = mm.find(b'\n') + 1 or size
        while chunk > 1:
          off, line = own_line(off, line)
          res = self._parse(base + off, size - off, plan, list_cap, n_batches=chunk)
          if res is None:          # a list column outgrew its array
            list_cap *= 4
            continue
          n_rows, consumed, seen, cols = res
          if n_rows < chunk * B:   # the end of the file is inside this chunk: batch by batch from here
            break
          off += consumed
          line += seen
          for k in range(chunk):
            yield self._pack_columns(self._slice_chunk(cols, plan, k, B))
        while True:
          off, line = own_line(off, line)
          res = self._parse(base + off, size - off, plan, list_cap)
          if res is None:          # a list column outgrew its array
            list_cap *= 4
            continue
          n_rows, consumed, seen, cols = res
          if n_rows < B:           # end of file; a last line without '\n' still counts
            tail = bytes(mm[off:])
            if tail and not tail.endswith(b'\n'):
              res = self._parse(tail + b'\n', len(tail) + 1, plan, max(list_cap, len(tail)))
              if res is not None and res[0] == B:
                yield self._pack_columns(res[3])
            return                 # a ragged last batch does not fit the static plan: skipped
          off += consumed
          line += seen
          yield self._pack_columns(cols)
      finally:
        del view

  def _fingerprints(self, field, cols):
    """uint64 fingerprint of a cross input per sample: the parsed Fingerprint64 of a STRING field, or
    Fingerprint64(as_string(v)) of an INT field."""
    arr = cols[field][0]
    return arr.view(np.uint64) if self.ftypes[field] == 'STRING' else fingerprint_i64(arr)

  def _ids_from_columns(self, n, cols):
    src = self.feature_inputs[n][0]
    if n in self.combos:
      fields, nb = self.combos[n]
      return cross_hash([self._fingerprints(f, cols) for f in fields], nb)
    if n in self.bucketized:
      return bucketize_raw(cols[src][0], self.bucketized[n])
    if n in self.hash_buckets and src in self.cross_fields:   # the field was parsed to raw fingerprints for a cross
      fp = cols[src][0].view(np.uint64)
      return np.where(fp == np.uint64(FP_EMPTY), np.int64(-1), (fp % np.uint64(self.hash_buckets[n])).astype(np.int64))
    return cols[src][0]

  def _pack_columns(self, cols):
    il = self.il
    B = self.batch_size
    feats = {}
    if il.sparse_names:
      feats['sparse_fea'] = torch.from_numpy(np.concatenate([self._ids_from_columns(n, cols) for n in il.sparse_names]))
    if il.raw_names:
      dense = np.zeros((B, il.n_dense), np.float32)
      for n in il.raw_names:
        if n in _expr_features(il):
          continue
        c0, c1 = il.raw_cols[n]
        dense[:, c0:c1] = cols[self.feature_inputs[n][0]][0].reshape(B, c1 - c0)
      feats['dense_fea'] = torch.from_numpy(dense)
    if _expr_inputs(il):
      feats['expr_fea'] = torch.from_numpy(np.stack([cols[f][0].astype(np.float64) for f in _expr_inputs(il)], 1))
    seq, tag = {}, {}
    for f in il.features.values():
      if f.kind not in ('seq', 'tag'):
        continue
      if f.name in self.bucketized:
        v, l = bucketize_raw_multi(cols[self.feature_inputs[f.name][0]][0], self.bucketized[f.name])
        tag[f.name] = (torch.from_numpy(v), torch.from_numpy(l), None)
        continue
      got = cols[self.feature_inputs[f.name][0]]
      vals, lens = got[0], got[1]
      if f.kind == 'seq' and f.name in self.multi_seps:
        seq[f.name] = (torch.from_numpy(vals.copy()), torch.from_numpy(lens), torch.from_numpy(got[2]))
      elif f.kind == 'seq':
        arr = np.zeros((B, f.seq_len), np.int64)
        starts = np.cumsum(lens) - lens
        arr[np.repeat(np.arange(B), lens), np.arange(vals.size) - np.repeat(starts, lens)] = vals
        seq[f.name] = (torch.from_numpy(arr), torch.from_numpy(lens))
      else:
        w = got[2] if len(got) > 2 else None
        if f.name in self.tag_weights:
          w, wlens = cols[self.tag_weights[f.name]]
          _check_tag_weights(f.name, lens, wlens)
        vals, lens, w = _pad_tags(il, f.name, vals, lens, w)
        tag[f.name] = (torch.from_numpy(vals.copy()), torch.from_numpy(lens), None if w is None else torch.from_numpy(w.copy()))
    if seq:
      feats['seq_fea'] = seq
    if tag:
      feats['tag_fea'] = tag
    if self.weight_field:
      feats['sample_weight'] = torch.from_numpy(cols[self.weight_field][0].copy())
    lab = np.stack([cols[l][0] for l in self.labels], 1)
    return feats, torch.from_numpy(lab if lab.shape[1] > 1 else lab[:, 0].copy())

  # ---- pure-python parsing of the same format (engine='python'): the readable restatement the native parser is
  # tested against ----
  def _batches_python(self):
    il = self.il
    B = self.batch_size
    buf = []
    with open(self.path, 'rb') as f:
      if self.cfg.data_config.with_header:
        f.readline()
      for i, line in enumerate(f):
        if i % self.task_num != self.task_index:   # another worker's line
          continue
        buf.append(line.rstrip(b'\r\n').decode('utf-8', errors='surrogateescape').split(self.sep))
        if len(buf) == B:
          yield self._pack(buf)
          buf = []
    # the reference drops nothing; a ragged last batch does not fit the static plan, so it is skipped

  def _pack(self, rows):
    il = self.il
    cols = {name: [r[i] if i < len(r) else '' for r in rows] for i, name in enumerate(self.fields)}
    feats = {}
    ids = []
    for n in il.sparse_names:
      src, _ = self.feature_inputs[n]
      ids.append(self._combo_column(cols, n) if n in self.combos else self._id_column(cols[src], n, self.defaults.get(src)))
    if ids:
      feats['sparse_fea'] = torch.from_numpy(np.concatenate(ids))
    if il.raw_names:
      dense = np.zeros((len(rows), il.n_dense), np.float32)
      for n in il.raw_names:
        if n in _expr_features(il):
          continue
        src, sep = self.feature_inputs[n]
        c0, c1 = il.raw_cols[n]
        for i, x in enumerate(cols[src]):
          x = x if x != '' else (self.defaults.get(src) or '0')
          vals = x.split(sep) if c1 - c0 > 1 else [x]
          dense[i, c0:c0 + len(vals)] = [float(v) for v in vals[:c1 - c0]]
      feats['dense_fea'] = torch.from_numpy(dense)
    if _expr_inputs(il):
      feats['expr_fea'] = torch.from_numpy(np.array(
          [[expr_number(x, f, self.ftypes[f], self.defaults.get(f)) for x in cols[f]] for f in _expr_inputs(il)],
          np.float64).T.copy())
    seq, tag = {}, {}
    for f in il.features.values():
      if f.kind not in ('seq', 'tag'):
        continue
      src, sep = self.feature_inputs[f.name]
      if f.name in self.bucketized:
        k = self.bucketized[f.name].raw_input_dim
        d = float(self.defaults.get(src) or 0)
        mat = np.zeros((len(rows), k), np.float32)
        for i, x in enumerate(cols[src]):
          vals = x.split(sep) if x != '' else [str(d)]
          mat[i, :len(vals[:k])] = [float(v) if v != '' else d for v in vals[:k]]
        v, l = bucketize_raw_multi(mat, self.bucketized[f.name])
        tag[f.name] = (torch.from_numpy(v), torch.from_numpy(l), None)
        continue
      toks = [[t for t in x.split(sep) if t != ''] for x in cols[src]]
      if f.kind == 'seq' and f.name in self.multi_seps:
        # every step token is itself a list: (values of all steps back to back, steps per sample, values per step)
        T, ms = f.seq_len, self.multi_seps[f.name]
        flat, lens, step_lens = [], np.zeros(len(rows), np.int32), np.zeros((len(rows), T), np.int32)
        for i, ts in enumerate(toks):
          ts = ts[:T]  # keep the FIRST max_seq_len steps (utils/shape_utils.py:393-410)
          lens[i] = len(ts)
          for j, t in enumerate(ts):
            vs = [v for v in t.split(ms) if v != '']
            step_lens[i, j] = len(vs)
            flat.extend(self._token(v, f.name) for v in vs)
        seq[f.name] = (torch.from_numpy(np.array(flat, np.int64)), torch.from_numpy(lens),
                       torch.from_numpy(step_lens.reshape(-1)))
      elif f.kind == 'seq':
        T = f.seq_len
        arr = np.zeros((len(rows), T), np.int64)
        lens = np.zeros(len(rows), np.int32)
        for i, ts in enumerate(toks):
          ts = ts[:T]  # keep the FIRST max_seq_len steps (utils/shape_utils.py:393-410)
          lens[i] = len(ts)
          arr[i, :len(ts)] = [self._token(t, f.name) for t in ts]
        seq[f.name] = (torch.from_numpy(arr), torch.from_numpy(lens))
      else:
        lens = np.array([len(ts) for ts in toks], np.int32)
        kv = self.kv_seps.get(f.name)
        w = None
        if kv:   # `id<kv>weight` tokens: both parts mandatory
          pairs = [t.split(kv) for ts in toks for t in ts]
          assert all(len(p_) == 2 for p_ in pairs), 'TagFeature %s: tokens must be key%sweight' % (f.name, kv)
          flat = np.array([self._token(p_[0], f.name) for p_ in pairs], np.int64)
          w = torch.from_numpy(np.array([float(p_[1]) for p_ in pairs], np.float32))
        else:
          flat = np.array([self._token(t, f.name) for ts in toks for t in ts], np.int64)
        if f.name in self.tag_weights:   # the weights come from their own field, split by the same separator
          wt = [[t for t in x.split(sep) if t != ''] for x in cols[self.tag_weights[f.name]]]
          _check_tag_weights(f.name, lens, np.array([len(ts) for ts in wt], np.int32))
          w = torch.from_numpy(np.array([float(t) for ts in wt for t in ts], np.float32))
        flat, lens, wn = _pad_tags(il, f.name, flat, lens, None if w is None else w.numpy())
        tag[f.name] = (torch.from_numpy(flat), torch.from_numpy(lens), None if wn is None else torch.from_numpy(wn))
    if seq:
      feats['seq_fea'] = seq
    if tag:
      feats['tag_fea'] = tag
    if self.weight_field:
      feats['sample_weight'] = torch.from_numpy(np.array([float(x or 1) for x in cols[self.weight_field]], np.float32))
    lab = np.stack([np.array([float(x or 0) for x in cols[l]], np.float32) for l in self.labels], 1)
    labels = torch.from_numpy(lab if lab.shape[1] > 1 else lab[:, 0])
    return feats, labels

  def __iter__(self):
    return self.batches()


class ParquetInput(object):
  """ParquetInput (input/parquet_input.py:201-239 + input/load_parquet.py:81-99): columnar file, one column per
  input field; the batch is the reference's packed form - ids of all sparse features feature-major
  (`sparse_fea`), dense features as one fp32 matrix (`dense_fea`), labels.  Sparse columns may be scalars or
  lists (the reference stores lists, load_parquet.py:139-205); an IdFeature needs exactly one id per cell (ragged
  cells belong to a TagFeature), Tag / Sequence features keep the whole list; a list-valued dense cell
  holds raw_input_dim values (the reference reads x[0] of a list cell, load_parquet.py:108-114, i.e. dim 1).  Like the
  reference's packed path the ids go to the device untouched and are bucketed there (`vals % num_buckets`,
  parquet_input.py:221, or the feature's hash rule).

  `path`: a list of files, or a string of comma-separated patterns, each expanded (sorted) in turn.  Worker task_index
  of task_num reads file j of that list when j % task_num == task_index (parquet_input.py:36-57)."""

  def __init__(self, pipeline_config, input_layer, path, batch_size=None, task_index=0, task_num=1):
    import pyarrow.parquet as pq   # optional dependency of this reader only
    self._pq = pq
    self.cfg = pipeline_config
    self.il = input_layer
    if not 0 <= task_index < task_num:
      raise ValueError('task_index %d is not in [0, task_num %d)' % (task_index, task_num))
    self.all_paths = expand_paths(path)
    self.paths = self.all_paths[task_index::task_num]
    if not self.paths:
      raise ValueError('ParquetInput: %d file(s) for task_num %d workers leave worker %d without a file; write at least '
                       'task_num files' % (len(self.all_paths), task_num, task_index))
    self.labels = list(pipeline_config.data_config.label_fields)
    dc = pipeline_config.data_config
    self.weight_field = dc.sample_weight if dc.HasField('sample_weight') else None
    self.batch_size = batch_size or input_layer.batch_size
    # (the declared types and defaults of the fields: ExprFeature inputs are read by them)
    self.ftypes = {f.input_name: dc.DESCRIPTOR.nested_types_by_name['Field'].fields_by_name['input_type']
                   .enum_type.values_by_number[f.input_type].name for f in dc.input_fields}
    self.defaults = {f.input_name: f.default_val for f in dc.input_fields}
    self.feature_inputs = {}
    for fc in config_util.get_feature_configs(pipeline_config):
      name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
      self.feature_inputs[name] = fc.input_names[0]
      if fc.HasField('kv_separator'):
        raise NotImplementedError('feature %s: kv_separator needs text tokens; Parquet columns carry ids only' % name)
    self.bucketized = _bucketized_features(pipeline_config, input_layer)
    self.combos = _combo_features(pipeline_config, input_layer)
    self.tag_weights = _tag_weight_inputs(pipeline_config)   # TagFeature -> the (list) column that holds its weights
    for fc in config_util.get_feature_configs(pipeline_config):
      if fc.HasField('seq_multi_sep'):
        raise NotImplementedError('feature %s: seq_multi_sep splits text steps; a Parquet column would need nested lists'
                                  % fc.input_names[0])

  @staticmethod
  def _column(col):
    """arrow column -> (values, lens or None): lens is None for scalar columns."""
    import pyarrow as pa
    col = col.combine_chunks() if hasattr(col, 'combine_chunks') else col
    if pa.types.is_list(col.type) or pa.types.is_large_list(col.type):
      offs = col.offsets.to_numpy()
      vals = col.values.to_numpy(zero_copy_only=False)
      return vals[offs[0]:offs[-1]], np.diff(offs).astype(np.int32)
    return col.to_numpy(zero_copy_only=False), None

  def _pack(self, table):
    il = self.il
    n = table.num_rows
    feats = {}
    ids = []
    for name in il.sparse_names:
      if name in self.combos:
        fields, nb = self.combos[name]
        fps = []
        for f in fields:
          vals, lens = self._column(table.column(f))
          if lens is not None:
            raise ValueError('ComboFeature %r: input column %r holds lists' % (name, f))
          fps.append(fingerprint_i64(vals) if np.asarray(vals).dtype.kind in 'iu' else
                     np.array([_lib.fingerprint64(v if v is not None else '') for v in vals], np.uint64))
        ids.append(cross_hash(fps, nb))
        continue
      vals, lens = self._column(table.column(self.feature_inputs[name]))
      if name in self.bucketized:
        ids.append(bucketize_raw(vals, self.bucketized[name]))
      elif lens is None and np.asarray(vals).dtype.kind in 'OUS':
        # string column of a hashed feature: bucket on the host like the CSV reader ('' / null -> -1)
        f = il.features[name]
        if f.bucket_mode == _lib.BUCKET_VOCAB:
          ids.append(string_keys(vals))
          continue
        if f.bucket_mode != _lib.BUCKET_IDENTITY:
          raise ValueError('feature %r: string column %r needs a hash_bucket_size and a STRING input field'
                           % (name, self.feature_inputs[name]))
        ids.append(np.array([_lib.fingerprint64(v) % f.num_buckets if v else -1 for v in vals], np.int64))
      elif lens is None:
        ids.append(np.asarray(vals, np.int64))
      else:
        # list column on a single-valued slot: exactly one id per sample.  The packed path pools whatever the
        # list holds (empty -> zero vector, several -> combined); that is the Tag slot's CSR lookup here.
        if not (lens == 1).all():
          raise ValueError('IdFeature %r has empty or multi-valued cells in %r: declare it as a TagFeature (combiner '
                           '"sum") so that the ragged lists are pooled' % (name, self.feature_inputs[name]))
        ids.append(np.asarray(vals, np.int64))
    if ids:
      feats['sparse_fea'] = torch.from_numpy(np.concatenate(ids))
    if il.raw_names:
      dense = np.zeros((n, il.n_dense), np.float32)
      for name in il.raw_names:
        if name in _expr_features(il):
          continue
        c0, c1 = il.raw_cols[name]
        vals, lens = self._column(table.column(self.feature_inputs[name]))
        dense[:, c0:c1] = np.asarray(vals, np.float32).reshape(n, c1 - c0)
      feats['dense_fea'] = torch.from_numpy(dense)
    if _expr_inputs(il):
      cols = []
      for f in _expr_inputs(il):
        col = table.column(f)
        vals, lens = self._column(col)
        t = self.ftypes.get(f, 'STRING')
        if lens is not None:
          raise ValueError('ExprFeature input column %r holds lists' % f)
        if np.asarray(vals).dtype.kind in 'OUS':
          vals = [expr_number('' if v is None else str(v), f, t, self.defaults.get(f)) for v in vals]
        v = np.asarray(vals, np.float32 if t == 'FLOAT' else np.float64).astype(np.float64)
        nulls = col.is_null().to_numpy(zero_copy_only=False)
        if nulls.any():   # a null is an empty value: the field's default
          v[nulls] = expr_number('', f, t, self.defaults.get(f))
        cols.append(v)
      feats['expr_fea'] = torch.from_numpy(np.stack(cols, 1))
    seq, tag = {}, {}
    for f in il.features.values():
      if f.kind not in ('seq', 'tag'):
        continue
      vals, lens = self._column(table.column(self.feature_inputs[f.name]))
      if f.name in self.bucketized:
        v, l = bucketize_raw_multi(vals, self.bucketized[f.name])
        tag[f.name] = (torch.from_numpy(v), torch.from_numpy(l), None)
        continue
      if f.bucket_mode == _lib.BUCKET_VOCAB:
        if np.asarray(vals).dtype.kind not in 'OUS':
          raise ValueError('feature %r: a vocabulary feature reads strings; column %r holds %s'
                           % (f.name, self.feature_inputs[f.name], np.asarray(vals).dtype))
        vals = string_keys(vals)
      vals = np.array(vals, np.int64)   # owned, writable copy (arrow buffers are read-only)
      if lens is None:
        lens = np.ones(n, np.int32)
      if f.kind == 'seq':
        T = f.seq_len
        arr = np.zeros((n, T), np.int64)
        start = np.cumsum(lens) - lens
        keep = np.minimum(lens, T)   # the FIRST max_seq_len steps (utils/shape_utils.py:393-410)
        for i in range(n):
          arr[i, :keep[i]] = vals[start[i]:start[i] + keep[i]]
        seq[f.name] = (torch.from_numpy(arr), torch.from_numpy(keep.astype(np.int32)))
      else:
        w = None
        if f.name in self.tag_weights:   # a second list column of the same shape (input/input.py:498-501)
          wv, wl = self._column(table.column(self.tag_weights[f.name]))
          _check_tag_weights(f.name, lens, np.ones(n, np.int32) if wl is None else wl)
          w = torch.from_numpy(np.array(wv, np.float32))
        if f.name in getattr(il, 'pad_tags', {}):
          raise NotImplementedError('tag feature %s of an embedding_layer block: string tags come from text inputs' % f.name)
        tag[f.name] = (torch.from_numpy(vals), torch.from_numpy(lens), w)
    if seq:
      feats['seq_fea'] = seq
    if tag:
      feats['tag_fea'] = tag
    if self.weight_field:
      feats['sample_weight'] = torch.from_numpy(
          np.asarray(table.column(self.weight_field).to_numpy(zero_copy_only=False), np.float32).copy())
    lab = np.stack([np.asarray(table.column(l).to_numpy(zero_copy_only=False), np.float32) for l in self.labels], 1)
    labels = torch.from_numpy(lab if lab.shape[1] > 1 else lab[:, 0].copy())
    return feats, labels

  def batches(self):
    """Batch order of the reference loader with one reader process (load_parquet.py:166-301): every file
    yields its own full batches first; its last `rows % batch_size` rows are appended to the rows carried over
    from earlier files, and a batch is cut from that carry as soon as it holds batch_size rows."""
    import pyarrow as pa
    B = self.batch_size
    carry = None
    for path in self.paths:
      pf = self._pq.ParquetFile(path)
      n_full = pf.metadata.num_rows // B * B
      pending, have, done = [], 0, 0
      for rb in pf.iter_batches(batch_size=B):   # record batches stop at row-group boundaries: re-chunk
        pending.append(rb)
        have += rb.num_rows
        while have >= B and done < n_full:
          tab = pa.Table.from_batches(pending)
          yield self._pack(tab.slice(0, B))
          done += B
          rest = tab.slice(B)
          pending = rest.to_batches() if rest.num_rows else []
          have = rest.num_rows
      if have:
        tail = pa.Table.from_batches(pending)
        carry = tail if carry is None else pa.concat_tables([carry, tail])
        if carry.num_rows >= B:
          yield self._pack(carry.slice(0, B).combine_chunks())
          carry = carry.slice(B) if carry.num_rows > B else None
    # the static plan holds exactly batch_size samples: the last partial batch (emitted by the reference unless
    # data_config.drop_remainder) is skipped

  def __iter__(self):
    return self.batches()


_CRITEO_COLUMN = re.compile(r'([fc])([1-9][0-9]*)$')


def criteo_columns(pipeline_config, input_layer):
  """The column maps of a CriteoInput plan -> (slot_cols, raw_cols): the category column of every id slot in
  input_layer.sparse_names order, the dense column of every raw column of dense_fea.  Inputs map by name
  (input/criteo_input.py:76-86): fK is dense column K-1, cK category column K-1, `label` the label.  Only what the files
  can feed without host work is accepted: IdFeatures over cK with hash_bucket_size / num_buckets (bucketed on the
  device like any integer id) and RawFeatures of raw_input_dim 1 over fK; every other use raises naming the feature."""
  from easyrec_b200 import builder
  dc = pipeline_config.data_config
  if list(dc.label_fields) != ['label']:
    raise ValueError('CriteoInput: label_fields must be ["label"], the files\' one label (got %s)' % list(dc.label_fields))
  if dc.HasField('sample_weight'):
    raise NotImplementedError('CriteoInput: sample_weight %r has no source in the binary files' % dc.sample_weight)
  types = builder.input_field_types(pipeline_config)
  col = {}
  for fc in config_util.get_feature_configs(pipeline_config):
    name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
    ftype = builder.ftype_name(fc)
    if ftype not in ('IdFeature', 'RawFeature'):
      raise NotImplementedError('feature %s: a %s needs host work or a source the CriteoInput files do not have; '
                                'only IdFeature and RawFeature are read from them' % (name, ftype))
    src = fc.input_names[0]
    m = _CRITEO_COLUMN.match(src)
    k = int(m.group(2)) if m else 0
    if len(fc.input_names) != 1 or not m or k > (_lib.CRITEO_N_DENSE if m.group(1) == 'f' else _lib.CRITEO_N_CAT):
      raise ValueError('feature %s: input %r is not one of the CriteoInput columns f1..f13 / c1..c26'
                       % (name, ', '.join(fc.input_names)))
    if ftype == 'RawFeature':
      if m.group(1) != 'f':
        raise ValueError('feature %s: a RawFeature reads a dense column f1..f13, not %r' % (name, src))
      if builder.raw_boundaries(fc) is not None:
        raise NotImplementedError('feature %s: a bucketized RawFeature (boundaries) is bucketed on the host; CriteoInput '
                                  'batches are unpacked on the device' % name)
      if fc.raw_input_dim != 1:
        raise ValueError('feature %s: a CriteoInput dense column holds one value, raw_input_dim is %d'
                         % (name, fc.raw_input_dim))
    else:
      if m.group(1) != 'c':
        raise ValueError('feature %s: an IdFeature reads a category column c1..c26, not %r' % (name, src))
      if fc.hash_bucket_size <= 0 and fc.num_buckets <= 0:
        raise NotImplementedError('feature %s: a CriteoInput id needs hash_bucket_size or num_buckets' % name)
      if types.get(src) == 'STRING':
        raise NotImplementedError('feature %s: input field %r is declared STRING, whose ids are hashed from their text on '
                                  'the host; the CriteoInput categories are integers' % (name, src))
    col[name] = k - 1
  slot_cols = [col[n] for n in input_layer.sparse_names]
  raw_cols = [0] * input_layer.n_dense
  for n in input_layer.raw_names:
    raw_cols[input_layer.raw_cols[n][0]] = col[n]
  return np.array(slot_cols, np.int32), np.array(raw_cols, np.int32)


class BinaryBatch(object):
  """One CriteoInput batch as the files hold it: label int32 [B], dense fp32 [B, 13] and cat int32 [B, 26] (the uint32
  bits, read as the reference's declared tf.int32), with the column maps of the reader's plan.  It becomes the batch of
  the other readers - sparse_fea int64 [n_slot * B] feature-major, dense_fea fp32 [B, n_raw], labels fp32 [B] - on the
  device, by er_binary_unpack (DeviceFeeder on its copy stream, to_device)."""

  def __init__(self, label, dense, cat, slot_cols, raw_cols, maps=None):
    self.label, self.dense, self.cat = label, dense, cat
    self.slot_cols, self.raw_cols = slot_cols, raw_cols
    self._maps = {} if maps is None else maps   # device -> the maps there; shared by the batches of one reader

  @property
  def batch_size(self):
    return self.label.numel()

  def ids(self, pos):
    """host int64 ids of id slot `pos` (what sparse_fea[pos * B:(pos + 1) * B] holds after the unpack)"""
    return self.cat[:, int(self.slot_cols[pos])].numpy().astype(np.int64)

  def unpack(self, label, dense, cat, out=(None, None, None)):
    """er_binary_unpack on the current stream over the batch's arrays where they are now (on the device, or the host
    tensors under the kernel doubles) -> (features, labels) in the form of the other readers."""
    from easyrec_b200 import kernels as K
    dev = str(label.device)
    if dev not in self._maps:
      self._maps[dev] = K.binary_maps(self.slot_cols, self.raw_cols, label.device)
    sparse, dense_fea, labels = K.binary_unpack(label, dense, cat, *self._maps[dev], *out)
    feats = {}
    if self.slot_cols.size:
      feats['sparse_fea'] = sparse
    if self.raw_cols.size:
      feats['dense_fea'] = dense_fea
    return feats, labels


def host_ids(feats, pos, batch_size):
  """host int64 ids of id slot `pos` of a host batch (a reader's dict or a BinaryBatch)"""
  if isinstance(feats, BinaryBatch):
    return feats.ids(pos)
  return feats['sparse_fea'][pos * batch_size:(pos + 1) * batch_size].cpu().numpy()


def criteo_parts(binary_paths):
  """BinaryDataInput -> [(label, dense, category) file paths]: entry i of each list expanded with glob and sorted, per
  kind, then appended in list order (input/criteo_input.py:37-52); the three lists must match file for file."""
  n = (len(binary_paths.label_path), len(binary_paths.dense_path), len(binary_paths.category_path))
  if len(set(n)) != 1:
    raise ValueError('CriteoInput: label_path (%d), dense_path (%d) and category_path (%d) must have as many entries' % n)
  parts = []
  for lp, dp, cp in zip(binary_paths.label_path, binary_paths.dense_path, binary_paths.category_path):
    got = [sorted(glob.glob(p)) for p in (lp, dp, cp)]
    if len(set(len(g) for g in got)) != 1:
      raise ValueError('CriteoInput: label_path %r, dense_path %r and category_path %r match %d, %d and %d files'
                       % ((lp, dp, cp) + tuple(len(g) for g in got)))
    parts.extend(zip(*got))
  return parts


def criteo_shard(total, task_index, task_num):
  """(first sample, sample count) of worker task_index of task_num over `total` samples in file order: every worker
  gets ceil(total / task_num) samples in one contiguous range, and the workers at or beyond total % task_num start one
  sample early - so neighbouring ranges overlap and every worker has as many samples
  (criteo_binary_reader.py:61-74)."""
  avg, res = divmod(int(total), int(task_num))
  if res == 0:
    return avg * task_index, avg
  return ((avg + 1) * task_index if task_index < res else avg * task_index + res - 1), avg + 1


class CriteoBinaryInput(object):
  """CriteoInput (input/criteo_input.py + input/criteo_binary_reader.py): per part three flat files - label int32,
  dense 13 x float32 and category 26 x uint32 per sample.  Nothing is parsed: a batch is three byte ranges, read with
  pread straight into its arrays, and yielded as a BinaryBatch that the device unpacks into the readers' batch form.

  binary_paths: the BinaryDataInput of binary_train_input / binary_eval_input.  Worker task_index of task_num reads
  the samples criteo_shard gives it, of the parts concatenated in order; batches are the next batch_size samples in
  file order, across file boundaries, and the last partial batch is skipped (the plan's batch size is fixed)."""

  def __init__(self, pipeline_config, input_layer, binary_paths, task_index=0, task_num=1, batch_size=None):
    if isinstance(binary_paths, (str, bytes)) or not hasattr(binary_paths, 'label_path'):
      raise ValueError('CriteoInput reads the binary parts named by binary_train_input / binary_eval_input '
                       '(BinaryDataInput), not %r' % (binary_paths,))
    if not 0 <= task_index < task_num:
      raise ValueError('task_index %d is not in [0, task_num %d)' % (task_index, task_num))
    self.slot_cols, self.raw_cols = criteo_columns(pipeline_config, input_layer)
    self.batch_size = batch_size or input_layer.batch_size
    self.parts = criteo_parts(binary_paths)
    if not self.parts:
      raise ValueError('CriteoInput: the binary paths match no file')
    self.counts = []
    for paths in self.parts:
      n = os.path.getsize(paths[0]) // 4
      for p, width in zip(paths, (4, 4 * _lib.CRITEO_N_DENSE, 4 * _lib.CRITEO_N_CAT)):
        if os.path.getsize(p) != n * width:
          raise ValueError('CriteoInput: %s holds %d bytes, %d samples of %d bytes expected' % (p, os.path.getsize(p), n, width))
      self.counts.append(n)
    self.starts = np.concatenate([[0], np.cumsum(self.counts, dtype=np.int64)])
    self.start, self.n_samples = criteo_shard(int(self.starts[-1]), task_index, task_num)
    self._maps = {}

  def batches(self):
    B = self.batch_size
    fds = {}
    try:
      for k in range(self.n_samples // B):
        yield self._read(self.start + k * B, B, fds), None
    finally:
      for fd in fds.values():
        os.close(fd)

  def _read(self, pos, n, fds):
    """samples [pos, pos + n) of the concatenated parts, read into fresh arrays"""
    label = np.empty(n, np.int32)
    dense = np.empty((n, _lib.CRITEO_N_DENSE), np.float32)
    cat = np.empty((n, _lib.CRITEO_N_CAT), np.int32)
    arrs = [memoryview(a).cast('B') for a in (label, dense, cat)]
    widths = (4, 4 * _lib.CRITEO_N_DENSE, 4 * _lib.CRITEO_N_CAT)
    done = 0
    f = int(np.searchsorted(self.starts, pos, side='right')) - 1
    while done < n:
      off = pos + done - int(self.starts[f])
      take = min(n - done, self.counts[f] - off)
      for kind, (p, w, buf) in enumerate(zip(self.parts[f], widths, arrs)):
        fd = fds.get((f, kind))
        if fd is None:
          fd = fds[(f, kind)] = os.open(p, os.O_RDONLY)
        dst, at = buf[done * w:(done + take) * w], off * w
        while len(dst):
          got = os.preadv(fd, [dst], at)
          if got <= 0:
            raise IOError('CriteoInput: %s ended before sample %d' % (p, off + take))
          dst, at = dst[got:], at + got
      done += take
      f += 1
    return BinaryBatch(torch.from_numpy(label), torch.from_numpy(dense), torch.from_numpy(cat), self.slot_cols,
                       self.raw_cols, self._maps)

  def __iter__(self):
    return self.batches()


def from_reference_packed(input_layer, fea_dict, sparse_fea_names):
  """The reference's packed feature dict (ParquetInput._to_fea_dict, input/parquet_input.py:201-239) -> the
  InputLayer's batch form.  fea_dict['sparse_fea'] = (vals int64 [L], lens int32 [n_feat * B]) with the lens
  feature-major in `sparse_fea_names` order (load_parquet.py:81-90); 'dense_fea' fp32 [B, sum raw_dim].
  Raw (un-bucketed) ids are expected: the bucket rule runs on the device."""
  il = input_layer
  B = il.batch_size
  vals, lens = fea_dict['sparse_fea']
  vals = np.asarray(vals, np.int64)
  lens = np.asarray(lens, np.int32)
  if lens.size != len(sparse_fea_names) * B:
    raise ValueError('sparse_fea lens has %d entries, expected %d features x batch %d' %
                     (lens.size, len(sparse_fea_names), B))
  counts = lens.reshape(len(sparse_fea_names), B).sum(axis=1)
  ends = np.cumsum(counts)
  if ends[-1] != vals.size:
    raise ValueError('len(all_vals)=%d np.sum(all_lens)=%d' % (vals.size, ends[-1]))
  per = {}
  for i, name in enumerate(sparse_fea_names):
    per[name] = (vals[ends[i] - counts[i]:ends[i]], lens[i * B:(i + 1) * B])
  feats, ids, tag = {}, [], {}
  for name in il.sparse_names:
    v, l = per[name]
    if not (l == 1).all():
      raise ValueError('IdFeature %r has empty or multi-valued cells: declare it as a TagFeature (combiner "sum")' % name)
    ids.append(v)
  if ids:
    feats['sparse_fea'] = torch.from_numpy(np.concatenate(ids))
  for f in il.features.values():
    if f.kind == 'tag':
      v, l = per[f.name]
      tag[f.name] = (torch.from_numpy(v.copy()), torch.from_numpy(l.copy()), None)
    elif f.kind == 'seq':
      raise ValueError('SequenceFeature %r has no packed form in the reference (Id / Tag / Raw only)' % f.name)
  if tag:
    feats['tag_fea'] = tag
  if 'dense_fea' in fea_dict:
    feats['dense_fea'] = torch.from_numpy(np.ascontiguousarray(fea_dict['dense_fea'], np.float32))
  return feats


def expand_paths(path):
  """a list of files as given, or a string of comma-separated patterns: each pattern expanded and sorted in turn (a
  name without wildcards is kept as it is)."""
  if not isinstance(path, str):
    return list(path)
  out = []
  for p in path.strip().split(','):
    out.extend(sorted(glob.glob(p)) if glob.has_magic(p) else [p])
  return out


def make_input(pipeline_config, input_layer, path, task_index=0, task_num=1):
  """reader for data_config.input_type (CSVInput / ParquetInput / CriteoInput / DummyInput); worker task_index of
  task_num reads its shard of `path` (DummyInput: every worker its own constant batches, as before).  CriteoInput takes
  the BinaryDataInput message of binary_train_input / binary_eval_input as `path`."""
  from easyrec_b200 import builder
  dc = pipeline_config.data_config
  if dc.WhichOneof('sampler') is not None:
    # the model itself builds from such a config; its batches (sampled negatives appended to every batch,
    # input/sampler.py) are not something these readers produce
    raise NotImplementedError('data_config.%s: negative samplers are outside the hot-path scope' % dc.WhichOneof('sampler'))
  kind = builder.input_type_name(pipeline_config)
  if kind == 'CriteoInput':
    if isinstance(path, (str, bytes)):
      raise ValueError('CriteoInput reads binary_train_input / binary_eval_input (BinaryDataInput: label_path, dense_path, '
                       'category_path), not the string path %r' % (path,))
    return CriteoBinaryInput(pipeline_config, input_layer, path, task_index=task_index, task_num=task_num)
  if kind.startswith('Parquet'):
    return ParquetInput(pipeline_config, input_layer, path, task_index=task_index, task_num=task_num)
  if kind == 'DummyInput':
    return DummyInput(input_layer, n_labels=max(1, len(dc.label_fields)))
  return CSVInput(pipeline_config, input_layer, path, task_index=task_index, task_num=task_num)


class Prefetcher(object):
  """Runs a batch source in a background thread, `depth` batches ahead of the consumer, so that parsing the
  next batches (er_csv_parse / pyarrow release the GIL) overlaps the device step of the current one - the role of
  `dataset.prefetch(prefetch_size)` in the reference input pipeline (input/input.py:1046-1051).  Order is
  preserved, an exception in the source is re-raised at the consumer, and abandoning the iterator (a step
  limit reached) stops the thread."""

  _END = object()

  def __init__(self, source, depth=2):
    self.source = source
    self.depth = max(int(depth), 1)

  def __iter__(self):
    import queue
    import threading
    q = queue.Queue(maxsize=self.depth)
    stop = threading.Event()

    def put(item):
      while not stop.is_set():
        try:
          q.put(item, timeout=0.1)
          return True
        except queue.Full:
          pass
      return False

    def work():
      try:
        for item in self.source:
          if not put(item):
            return
        put(self._END)
      except BaseException as e:   # handed to the consumer
        put(e)

    t = threading.Thread(target=work, name='easyrec_b200-prefetch', daemon=True)
    t.start()
    try:
      while True:
        item = q.get()
        if item is self._END:
          return
        if isinstance(item, BaseException):
          raise item
        yield item
    finally:
      stop.set()
      try:                      # unblock a producer that waits for room in the queue
        while True:
          q.get_nowait()
      except queue.Empty:
        pass
      t.join(timeout=5.0)


class DeviceFeeder(object):
  """Host batches -> device batches through PINNED staging buffers, `depth` batches ahead of the consumer on a copy
  stream of its own (double buffering at depth 2): while step i runs, batch i+1 is already crossing PCIe - the
  `dataset.prefetch` + H2D of the reference input pipeline (input/input.py:1046-1051, input/load_parquet.py:139-317
  feed the session the same way).  Per slot: pageable host tensor -> pinned buffer (a CPU memcpy) -> cudaMemcpyAsync on
  the copy stream -> an event the compute stream waits on; a slot's device buffers are rewritten only after the
  step that read them has been enqueued and has finished (event recorded when the consumer asks for the next batch).
  On a CPU device it passes the batches through."""

  def __init__(self, source, device, depth=2, lookahead=0):
    """lookahead: how many batches the consumer holds beyond the one it is training on (EasyRecEstimator.train names
    the next batch to train_step so that its id exchange can run early): a slot is recycled only after the step that
    reads it has been enqueued, i.e. `lookahead` requests later."""
    self.source = source
    self.device = device
    self.lookahead = max(int(lookahead), 0)
    self.depth = max(int(depth), 1) + self.lookahead
    self.h2d_bytes = 0   # bytes copied host -> device so far (bench.py reports them per step)

  class _Slot(object):
    def __init__(self):
      self.pinned = {}
      self.dev = {}
      self.ready = None
      self.consumed = None

  def _stage(self, slot, path, t, stream):
    """one tensor: grow-only pinned + device buffers keyed by its place in the batch structure."""
    n = t.numel()
    dev_buf = slot.dev.get(path)
    if dev_buf is None or dev_buf.numel() < n or dev_buf.dtype != t.dtype:
      cap = max(n, 1) if dev_buf is None else max(n, 2 * dev_buf.numel())
      slot.pinned[path] = torch.empty(cap, dtype=t.dtype, pin_memory=True)
      slot.pinned_np = getattr(slot, 'pinned_np', {})
      slot.pinned_np[path] = slot.pinned[path].numpy()
      dev_buf = slot.dev[path] = torch.empty(cap, dtype=t.dtype, device=self.device)
    dev = dev_buf[:n]
    if t.is_pinned() and t.is_contiguous():
      dev.copy_(t.reshape(-1), non_blocking=True)      # the reader already produced page-locked memory
    else:
      # one plain memcpy into the slot's page-locked buffer (numpy: torch's CPU copy forks its whole intra-op
      # thread pool for a 2 MB tensor, 1.2 ms on a 128-thread host against 0.15 ms for the memcpy)
      np.copyto(slot.pinned_np[path][:n], t.detach().reshape(-1).numpy())
      dev.copy_(slot.pinned[path][:n], non_blocking=True)
    self.h2d_bytes += n * t.element_size()
    return dev.view(t.shape)

  def _stage_batch(self, slot, feats, labels, stream):
    if slot.ready is not None and not slot.ready.query():
      slot.ready.synchronize()      # (the previous copy out of this slot's pinned buffers is normally long done)
    with torch.cuda.stream(stream):
      if slot.consumed is not None:
        stream.wait_event(slot.consumed)
      if isinstance(feats, BinaryBatch):
        # the three arrays as read cross PCIe; er_binary_unpack makes the batch form in the slot's own device buffers
        raw = [self._stage(slot, ('__binary', i), t, stream) for i, t in enumerate((feats.label, feats.dense, feats.cat))]
        B, n_raw = feats.batch_size, feats.raw_cols.size
        shapes = ((feats.slot_cols.size * B,), (B, n_raw), (B,))
        if getattr(slot, 'unpacked', None) is None or [tuple(t.shape) for t in slot.unpacked] != list(shapes):
          slot.unpacked = [torch.empty(sh, dtype=dt, device=self.device)
                           for sh, dt in zip(shapes, (torch.int64, torch.float32, torch.float32))]
        slot.batch = feats.unpack(*raw, out=slot.unpacked)
        slot.ready = torch.cuda.Event()
        slot.ready.record(stream)
        return
      out = {}
      for k, v in feats.items():
        if isinstance(v, dict):
          out[k] = {n: tuple(None if t is None else self._stage(slot, (k, n, i), t, stream) for i, t in enumerate(tup))
                    for n, tup in v.items()}
        else:
          out[k] = self._stage(slot, (k,), v, stream)
      lab = self._stage(slot, ('__labels',), labels, stream)
      slot.ready = torch.cuda.Event()
      slot.ready.record(stream)
    slot.batch = (out, lab)

  def __iter__(self):
    if not str(self.device).startswith('cuda'):
      for feats, labels in self.source:
        yield feats.unpack(feats.label, feats.dense, feats.cat) if isinstance(feats, BinaryBatch) else (feats, labels)
      return
    import collections as _c
    stream = torch.cuda.Stream(device=self.device)
    ring = [self._Slot() for _ in range(self.depth)]
    it = iter(self.source)
    queue = _c.deque()
    i = 0
    for _ in range(self.depth):
      nxt = next(it, None)
      if nxt is None:
        break
      self._stage_batch(ring[i % self.depth], nxt[0], nxt[1], stream)
      queue.append(ring[i % self.depth])
      i += 1
    held = _c.deque()
    while queue:
      slot = queue.popleft()
      torch.cuda.current_stream().wait_event(slot.ready)
      yield slot.batch
      held.append(slot)
      if len(held) <= self.lookahead:
        continue
      # the consumer has enqueued the step that reads the oldest held slot: its buffers are free once that step is done
      slot = held.popleft()
      slot.consumed = torch.cuda.Event()
      slot.consumed.record(torch.cuda.current_stream())
      nxt = next(it, None)
      if nxt is not None:
        self._stage_batch(slot, nxt[0], nxt[1], stream)
        queue.append(slot)


def to_device(feats, labels, device):
  if isinstance(feats, BinaryBatch):
    return feats.unpack(*(t.to(device, non_blocking=True) for t in (feats.label, feats.dense, feats.cat)))
  out = {}
  for k, v in feats.items():
    if isinstance(v, dict):
      out[k] = {n: tuple(None if t is None else t.to(device, non_blocking=True) for t in tup)
                for n, tup in v.items()}
    else:
      out[k] = v.to(device, non_blocking=True)
  return out, labels.to(device, non_blocking=True)
