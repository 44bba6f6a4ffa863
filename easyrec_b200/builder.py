"""pipeline config -> (feature specs, feature groups, InputLayer, model).

Host-side counterpart of `FeatureColumnParser` (feature_column/feature_column.py:44-203,259-656)
and of `EasyRecModel.create_class(model_class)` (model/easy_rec_model.py:44-49, main.py:137).
"""
import collections

import numpy as np

from easyrec_b200 import _lib
from easyrec_b200 import input_layer as IL
from easyrec_b200.config import config_util

_OPT_KIND = {'adagrad_optimizer': _lib.OPT_ADAGRAD, 'lazy_adam_optimizer': _lib.OPT_LAZY_ADAM,
             'adam_optimizer': _lib.OPT_ADAM_ROWS, 'momentum_optimizer': _lib.OPT_SGD}


def ev_params(pipeline_config, fc):
  """the EVParams of a feature: its own, else the model's (feature_column/feature_column.py:600-650), else None"""
  if fc.HasField('ev_params'):
    return fc.ev_params
  mc = pipeline_config.model_config
  return mc.ev_params if mc.HasField('ev_params') else None


def vocab_entries(fc):
  """The vocabulary of a feature as a list of byte strings, or None.  The rule is picked in the reference's order,
  hash_bucket_size, then vocab_list, then vocab_file (feature_column/feature_column.py:270-294); vocab_file holds one
  entry per line, keyed on the whole line, and its size is the file's line count (:243-249), a last line without
  '\n' included."""
  if fc.hash_bucket_size > 0:
    return None
  if len(fc.vocab_list) > 0:
    return [v.encode('utf-8') for v in fc.vocab_list]
  if fc.HasField('vocab_file'):
    with open(fc.vocab_file, 'rb') as f:
      lines = f.read().split(b'\n')
    if lines[-1] == b'':
      lines.pop()        # the newline that ends the last line starts no entry
    return lines
  return None


def vocab_keys(name, entries):
  """Entry i of a vocabulary -> its 63-bit key Fingerprint64(entry) % (2^63 - 1), the key the readers give the
  feature's raw strings; K1 reads row i for it.  Repeated entries are refused as TF's vocabulary tables refuse them, and
  two entries whose keys collide are refused because K1 could not tell them apart."""
  if not entries:
    raise ValueError('feature %s: the vocabulary is empty' % name)
  shown = lambda e: e.decode('utf-8', 'replace')   # noqa: E731
  repeated = [shown(e) for e, c in collections.Counter(entries).items() if c > 1]
  if repeated:
    raise ValueError('feature %s: vocabulary entries %s appear more than once (a vocabulary table keys each entry '
                     'once)' % (name, repeated[:10]))
  keys = [_lib.fingerprint64(e) % _lib.KV_BUCKETS for e in entries]
  first = {}
  for e, k in zip(entries, keys):
    if k in first:
      raise NotImplementedError('feature %s: vocabulary entries %r and %r have the same 63-bit key %d '
                                '(Fingerprint64 %% (2^63 - 1)); K1 cannot tell them apart' % (name, shown(first[k]),
                                                                                          shown(e), k))
    first[k] = e
  return tuple(keys)


def vocabulary(pipeline_config, fc, name, field_types, kv):
  """The keys of a feature's vocabulary (vocab_keys) or None; refuses by name what cannot take one"""
  if fc.hash_bucket_size > 0 and (len(fc.vocab_list) > 0 or fc.HasField('vocab_file')):
    raise NotImplementedError('feature %s: hash_bucket_size together with vocab_list / vocab_file: the reference '
                              'hashes and never reads the vocabulary (feature_column/feature_column.py:270-294); keep '
                              'one of them' % name)
  entries = vocab_entries(fc)
  if entries is None:
    return None
  ftype = ftype_name(fc)
  if ftype not in ('IdFeature', 'TagFeature', 'SequenceFeature'):
    raise NotImplementedError('feature %s: vocab_list / vocab_file on a %s; vocabularies are read by IdFeatures, '
                              'TagFeatures and SequenceFeatures' % (name, ftype))
  if kv:
    raise NotImplementedError('feature %s: vocab_list / vocab_file together with ev_params: a vocabulary column has '
                              'a fixed table of len(vocabulary) rows' % name)
  if input_type_name(pipeline_config) == 'CriteoInput':
    raise NotImplementedError('feature %s: vocab_list / vocab_file with CriteoInput, whose category columns are '
                              'integers unpacked on the device' % name)
  if ftype == 'IdFeature' and field_types.get(fc.input_names[0]) != 'STRING':
    # input/input.py:536-555 passes such a field on unconverted, and TF's vocabulary column then refuses the integer
    # tensor (VocabularyListCategoricalColumn._transform_input_tensor: "Column dtype and SparseTensors dtype must be
    # compatible")
    raise ValueError('feature %s: vocab_list / vocab_file on the %s field %s; an IdFeature with a vocabulary reads a '
                     'STRING field' % (name, field_types.get(fc.input_names[0], 'undeclared'), fc.input_names[0]))
  return vocab_keys(name, entries)


def feature_specs(pipeline_config, packed_mod=False, default_seq_len=50):
  """FeatureConfig protos -> FeatureSpec list (config order = packed feature order)."""
  specs = []
  field_types = input_field_types(pipeline_config)
  for fc in config_util.get_feature_configs(pipeline_config):
    name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
    ev = ev_params(pipeline_config, fc)
    # a key-value table (ev_params): a pool of max_capacity rows per rank, filled as keys are trained
    kv = int(ev.max_capacity) if ev is not None else 0
    if kv and ((ftype_name(fc) == 'RawFeature' and fc.embedding_dim == 0 and raw_boundaries(fc) is None) or
               ftype_name(fc) == 'ExprFeature'):
      kv = 0   # a numeric column without a table: ev_params has nothing to apply to
    # a vocabulary column: the readers key its strings, K1 finds their entries (ER_BUCKET_VOCAB)
    vocab = vocabulary(pipeline_config, fc, name, field_types, kv)
    if kv and (ftype_name(fc) not in ('IdFeature', 'TagFeature') or raw_boundaries(fc) is not None or
               (fc.hash_bucket_size <= 0 and fc.num_buckets <= 0)):
      raise NotImplementedError('feature %s: ev_params (key-value tables) on a %s; only IdFeatures and TagFeatures '
                                'with hash_bucket_size or num_buckets take key-value tables' % (name, ftype_name(fc)))
    # a STRING field is hashed where its bytes are, by the reader (Fingerprint64 % hash_bucket_size); integer
    # fields go to the device as int64 and are hashed there from their decimal text (input/input.py:541-543)
    host_hashed = fc.hash_bucket_size > 0 and field_types.get(fc.input_names[0]) == 'STRING'
    # per-feature options that change which row / value a sample reads and are not implemented: refuse
    unsupported = [w for w, on in (
        ('kv_separator on a feature that is not a TagFeature', fc.HasField('kv_separator') and ftype_name(fc) != 'TagFeature'),
        ('seq_multi_sep on a feature that is not a SequenceFeature', fc.HasField('seq_multi_sep') and ftype_name(fc) != 'SequenceFeature'),
        ('normalizer_fn on a feature that is not a RawFeature', fc.HasField('normalizer_fn') and ftype_name(fc) != 'RawFeature'),
        ('sub_feature_type RawFeature', fc.HasField('sub_feature_type') and fc.sub_feature_type != fc.IdFeature)) if on]
    if unsupported:
      raise NotImplementedError('feature %s: %s is outside the hot-path scope' % (name, ', '.join(unsupported)))
    ftype = fc.DESCRIPTOR.fields_by_name['feature_type'].enum_type.values_by_number[fc.feature_type].name
    if ftype == 'IdFeature':
      specs.append(IL.id_feature(name, fc.embedding_dim, hash_bucket_size=fc.hash_bucket_size,
                                 num_buckets=fc.num_buckets, combiner=fc.combiner,
                                 embedding_name=fc.embedding_name, packed_mod=packed_mod, host_hashed=host_hashed,
                                 kv_capacity=kv, vocab=vocab))
    elif ftype == 'ComboFeature':
      # crossed_column over the inputs' string forms (feature_column/feature_column.py:424-455): the reader computes
      # FingerprintCat64 over the inputs' fingerprints % hash_bucket_size (readers.cross_hash); an id slot from there on
      if len(fc.combo_join_sep) > 0 or len(fc.combo_input_seps) > 0:
        raise NotImplementedError('ComboFeature %s: combo_join_sep / combo_input_seps' % name)
      if len(fc.input_names) < 2 or fc.hash_bucket_size <= 0:
        raise ValueError('ComboFeature %s needs at least two input_names and a hash_bucket_size' % name)
      specs.append(IL.id_feature(name, fc.embedding_dim, hash_bucket_size=fc.hash_bucket_size, combiner=fc.combiner,
                                 embedding_name=fc.embedding_name, host_hashed=True))
    elif ftype == 'RawFeature' and raw_boundaries(fc) is not None:
      # bucketized column (feature_column/feature_column.py:364-386): the reader turns the value into its bucket
      # (readers.bucketize_raw), from there on it is an id feature over len(boundaries) + 1 rows
      n_bucket = len(raw_boundaries(fc)) + 1
      if fc.raw_input_dim == 1:
        specs.append(IL.id_feature(name, fc.embedding_dim, num_buckets=n_bucket, combiner=fc.combiner,
                                   embedding_name=fc.embedding_name))
      else:
        # k values per sample -> k ids `bucket + (len(boundaries) + 1) * k_index` (feature_column_v2.py:2849-2870),
        # pooled by the feature's combiner: a fixed-length tag slot
        specs.append(IL.multi_feature(name, 'tag', fc.embedding_dim, num_buckets=n_bucket * fc.raw_input_dim,
                                      combiner=fc.combiner, embedding_name=fc.embedding_name))
    elif ftype == 'RawFeature':
      specs.append(IL.raw_feature(name, fc.embedding_dim, fc.min_val, fc.max_val, fc.raw_input_dim))
    elif ftype == 'ExprFeature':
      # numeric_column(shape=(1,)) of the expression's float32 value, not normalised (feature_column/feature_column.py:
      # 407-422): a raw column without a table, filled on the device by er_expr_eval
      specs.append(IL.raw_feature(name)._replace(expr=expr_feature(fc, name, field_types)))
    elif ftype in ('TagFeature', 'SequenceFeature'):
      specs.append(IL.multi_feature(name, 'tag' if ftype == 'TagFeature' else 'seq', fc.embedding_dim,
                                    hash_bucket_size=fc.hash_bucket_size, num_buckets=fc.num_buckets,
                                    combiner=fc.combiner, embedding_name=fc.embedding_name,
                                    seq_len=((fc.max_seq_len if fc.HasField('max_seq_len') else default_seq_len)
                                             if ftype == 'SequenceFeature' else 1),
                                    packed_mod=packed_mod, host_hashed=host_hashed, kv_capacity=kv, vocab=vocab))
    else:
      raise NotImplementedError('feature_type %s (feature %s) is outside the hot-path scope' % (ftype, name))
  check_vocab_tables(specs)
  return specs


_EXPR_FIELD_TYPES = ('INT32', 'INT64', 'FLOAT', 'DOUBLE', 'STRING')


def expr_feature(fc, name, field_types):
  """(expr.Program, input field names) of an ExprFeature.  Its inputs are read as float64 (input/input.py:507-528:
  STRING fields through string_to_number, the others cast); options the reference never reads for it are refused."""
  from easyrec_b200 import expr
  ignored = [w for w, on in (('embedding_dim', fc.embedding_dim > 0), ('boundaries', len(fc.boundaries) > 0),
                             ('hash_bucket_size', fc.hash_bucket_size > 0)) if on]
  if ignored:
    raise NotImplementedError('ExprFeature %s: %s, which the reference ignores for an ExprFeature (a numeric_column of '
                              'shape (1,), feature_column/feature_column.py:407-422); remove it' % (name, ', '.join(ignored)))
  if not fc.feature_name:
    # input/input.py:508 stores the value under fc.feature_name ('' when unset) while parse_expr_feature
    # (feature_column/feature_column.py:415-418) names the column input_names[0]: the reference would read the raw input
    # field or fail, never the expression
    raise ValueError('ExprFeature %s (expression %r) has no feature_name; the reference trains the expression only '
                     'under its feature_name' % (name, fc.expression))
  if not fc.HasField('expression'):
    raise ValueError('ExprFeature %s has no expression' % name)
  for f in fc.input_names:
    if field_types.get(f) not in _EXPR_FIELD_TYPES:
      raise ValueError('ExprFeature %s: input %s is %s; an expression reads INT32, INT64, FLOAT, DOUBLE or STRING '
                       'fields (input/input.py:513-531)' % (name, f, field_types.get(f, 'not an input field')))
  return expr.compile_expression(name, fc.expression, list(fc.input_names)), tuple(fc.input_names)


def check_vocab_tables(specs):
  """features that share an embedding_name read one table: with a vocabulary among them, they must agree on its row
  count (the reference's shared embedding variable has one shape)"""
  by_table = collections.defaultdict(list)
  for sp in specs:
    if sp.embedding_name:
      by_table[sp.embedding_name].append(sp)
  for table, group in by_table.items():
    if any(sp.vocab is not None for sp in group) and len(set(sp.num_buckets for sp in group)) > 1:
      raise ValueError('embedding_name %s: shared by features with different row counts (%s); a vocabulary column '
                       'has len(vocabulary) rows' % (table, ', '.join('%s: %d' % (sp.name, sp.num_buckets)
                                                                       for sp in group)))


def ftype_name(fc):
  return fc.DESCRIPTOR.fields_by_name['feature_type'].enum_type.values_by_number[fc.feature_type].name


def raw_boundaries(fc):
  """sorted bucket boundaries of a RawFeature, or None: explicit `boundaries`, or - num_buckets > 1 with a
  min/max range - equal-width cuts i / num_buckets on the normalised value
  (feature_column/feature_column.py:364-376)."""
  if len(fc.boundaries) > 0:
    return sorted(fc.boundaries)
  if fc.num_buckets > 1 and fc.max_val > fc.min_val:
    return [x / float(fc.num_buckets) for x in range(0, fc.num_buckets)]
  return None


def feature_groups(model_config):
  groups = collections.OrderedDict()
  for g in model_config.feature_groups:
    wd = g.DESCRIPTOR.fields_by_name['wide_deep'].enum_type.values_by_number[g.wide_deep].name
    seq = []
    for sf in g.sequence_features:
      # target attention inside the group (layers/input_layer.py:96-111 -> layers/sequence_feature_layer.py:190-249):
      # seq_dnn defaults to [128, 64, 32, 1] (:226-230)
      units = IL_units(sf.seq_dnn) if sf.HasField('seq_dnn') else IL_units(None)
      seq.append(dict(name=sf.group_name, maps=[(list(m.key), list(m.hist_seq)) for m in sf.seq_att_map], units=units,
                      need_key=bool(sf.need_key_feature)))
    groups[g.group_name] = dict(features=list(g.feature_names), wide=(wd == 'WIDE'), seq=seq)
  return groups


def IL_units(dnn_config):
  from easyrec_b200 import layers as L
  if dnn_config is None:
    return L.Units([128, 64, 32, 1])
  return L.units_of(dnn_config)


def seq_att_groups(model_config):
  """EasyRecModel.seq_att_groups -> {group: [(keys, hist_seqs), ...]} (layers/seq_input_layer.py:63-101)."""
  out = collections.OrderedDict()
  for g in model_config.seq_att_groups:
    out[g.group_name] = [(list(m.key), list(m.hist_seq)) for m in g.seq_att_map]
  return out


def input_field_types(pipeline_config):
  """input field name -> 'INT32' | 'INT64' | 'STRING' | 'FLOAT' | 'DOUBLE' | ... (data_config.input_fields)."""
  dc = pipeline_config.data_config
  enum = dc.DESCRIPTOR.nested_types_by_name['Field'].fields_by_name['input_type'].enum_type
  return {f.input_name: enum.values_by_number[f.input_type].name for f in dc.input_fields}


def input_type_name(pipeline_config):
  dc = pipeline_config.data_config
  return dc.DESCRIPTOR.fields_by_name['input_type'].enum_type.values_by_number[dc.input_type].name


def optimizer_settings(pipeline_config, index=0):
  """builders/optimizer_builder.py:28-144: kind + constant / exponential-decay schedule of optimizer_config[index].
  With TWO entries the first trains the embedding tables and the second every other variable
  (model/easy_rec_estimator.py:216-232, EasyRecModel.get_grouped_vars model/easy_rec_model.py:446-467): the result
  for index 0 then carries the second one's settings under 'dense'."""
  tc = pipeline_config.train_config
  if len(tc.optimizer_config) == 0:
    return dict(kind='adagrad_optimizer', lr_fn=lambda step: 0.01, beta1=0.9, beta2=0.999, acc0=0.1)
  if index == 0 and len(tc.optimizer_config) == 2:
    out = optimizer_settings(pipeline_config, index=-2)   # (-2 = entry 0 of two, without re-entering this branch)
    out['dense'] = optimizer_settings(pipeline_config, index=1)
    return out
  oc = tc.optimizer_config[index]
  kind = oc.WhichOneof('optimizer')
  if kind is None:
    # builders/optimizer_builder.py:28-144 knows more optimizers (adam_async, ftrl, adamw, ...); only the ones with a
    # fused row rule on this path are accepted
    raise ValueError('unsupported optimizer in train_config.optimizer_config (have: %s)' % sorted(_OPT_KIND))
  o = getattr(oc, kind)
  momentum = float(o.momentum_optimizer_value) if kind == 'momentum_optimizer' else 0.0
  if kind == 'momentum_optimizer' and (momentum < 0 or getattr(o, 'use_nesterov', False)):
    raise ValueError('momentum_optimizer: momentum_optimizer_value %g / use_nesterov are not supported' % momentum)
  lr = o.learning_rate
  which = lr.WhichOneof('learning_rate')
  if which == 'exponential_decay_learning_rate':
    e = lr.exponential_decay_learning_rate

    def lr_fn(step, e=e):
      # core/learning_schedules.py:30-75 exponential_decay_with_burnin, in fp32 like the TF graph it builds:
      # burn-in ramps linearly from burnin_learning_rate to the base rate (or holds the base rate when
      # burnin_learning_rate is 0); the decay clock starts after the burn-in steps.
      f32 = np.float32
      base = f32(e.initial_learning_rate)
      if step < e.burnin_steps:
        if e.burnin_learning_rate == 0:
          v = base
        else:
          slope = (e.initial_learning_rate - e.burnin_learning_rate) / e.burnin_steps
          v = f32(slope) * f32(step) + f32(e.burnin_learning_rate)
      else:
        p = f32(step - e.burnin_steps) / f32(e.decay_steps)
        if e.staircase:
          p = np.floor(p)
        v = base * np.power(f32(e.decay_factor), p, dtype=f32)
      return float(max(f32(v), f32(e.min_learning_rate)))
  elif which == 'constant_learning_rate':
    c = lr.constant_learning_rate.learning_rate
    lr_fn = lambda step, c=c: c  # noqa: E731
  else:
    # builders/optimizer_builder.py:145-215 also knows manual_step / cosine / poly / transformer schedules;
    # they are outside the hot-path scope: refuse instead of training with a made-up rate.
    raise ValueError('unsupported learning_rate schedule: %r' % which)
  # tf.train.MomentumOptimizer(momentum > 0) keeps one accumulator per variable (builders/optimizer_builder.py:91-97);
  # the value travels where Adam's beta1 does (er_opt_t.beta1); momentum 0 is plain SGD, no state
  return dict(kind=kind, lr_fn=lr_fn, beta1=momentum if momentum > 0 else getattr(o, 'beta1', 0.9),
              beta2=getattr(o, 'beta2', 0.999), momentum=momentum,
              acc0=getattr(o, 'initial_accumulator_value', 0.1),
              emb_lr_mult=oc.embedding_learning_rate_multiplier
              if oc.HasField('embedding_learning_rate_multiplier') else 1.0)


_RANK_CLASSES = ('DeepFM', 'DCN', 'DLRM', 'FM', 'MultiTower', 'MultiTowerDIN', 'RankModel', 'WideAndDeep')


def _is_repeated(fd):
  rep = getattr(fd, 'is_repeated', None)     # protobuf >= 5.29 (FieldDescriptor.label is deprecated there)
  if rep is None:
    return fd.label == fd.LABEL_REPEATED
  return rep() if callable(rep) else rep


def _walk_messages(msg, path):
  """(dotted path, message) for every set sub-message, depth first."""
  for fd, value in msg.ListFields():
    if fd.type != fd.TYPE_MESSAGE or fd.message_type.GetOptions().map_entry:
      continue
    rep = _is_repeated(fd)
    items = list(value) if rep else [value]
    for i, v in enumerate(items):
      p = '%s.%s%s' % (path, fd.name, '[%d]' % i if rep else '')
      yield p, v
      for sub in _walk_messages(v, p):
        yield sub


def check_scope(pipeline_config):
  """Refuse configs whose training semantics depend on something this path does not implement, rather than
  training a different model silently.  (Control-plane fields - export, hooks, distribution strategy - do not
  change the arithmetic and are ignored.)"""
  mc = pipeline_config.model_config
  tc = pipeline_config.train_config
  bad = []
  # EVParams first: PAI-TF's admission and eviction, and SOK's cache, cannot be pinned here
  evs = [('model_config.ev_params', mc.ev_params)] if mc.HasField('ev_params') else []
  for fc in config_util.get_feature_configs(pipeline_config):
    if fc.HasField('ev_params'):
      evs.append(('feature %s: ev_params' % (fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]),
                  fc.ev_params))
  for path, ev in evs:
    for field, on, why in (('filter_freq', ev.filter_freq > 0, 'admission by frequency'),
                           ('steps_to_live', ev.steps_to_live > 0, 'eviction'),
                           ('use_cache', ev.use_cache, 'the SOK embedding cache')):
      if on:
        bad.append('%s.%s (%s)' % (path, field, why))
    if ev.max_capacity <= 0:
      bad.append('%s.max_capacity 0' % path)
  dc = pipeline_config.data_config
  if dc.HasField('sample_weight') and mc.model_class in ('DSSM', 'MatchModel'):
    bad.append('data_config.sample_weight with a match model (the list-wise loss normalises by mean(w))')
  for g in mc.feature_groups:
    for sf in g.sequence_features:
      what = [w for w, on in (('allow_key_transform', sf.allow_key_transform), ('transform_dnn', sf.transform_dnn),
                              ('aux_hist_seq', any(len(m.aux_hist_seq) for m in sf.seq_att_map)),
                              ('negative_sampler', g.negative_sampler)) if on]
      if what:
        bad.append('feature_groups[%s].sequence_features[%s]: %s' % (g.group_name, sf.group_name, ', '.join(what)))
    if g.negative_sampler:
      bad.append('feature_groups[%s].negative_sampler' % g.group_name)
    names = g.DESCRIPTOR.fields_by_name['wide_deep'].enum_type.values_by_number
    if names[g.wide_deep].name == 'WIDE_AND_DEEP':
      bad.append('feature_groups[%s].wide_deep WIDE_AND_DEEP' % g.group_name)
  if len(mc.kd) > 0:
    bad.append('model_config.kd (knowledge distillation losses)')
  if mc.HasField('variational_dropout'):
    bad.append('model_config.variational_dropout')
  if len(tc.freeze_gradient) > 0:
    bad.append('train_config.freeze_gradient')
  if tc.fine_tune_checkpoint:
    bad.append('train_config.fine_tune_checkpoint (TF checkpoints cannot be read here; use EasyRecEstimator.restore)')
  if len(tc.optimizer_config) == 2 and mc.model_class == 'WideAndDeep':
    bad.append('two optimizer_config entries with WideAndDeep (wide variables / the rest, wide_and_deep.py:82-110)')
  if len(tc.optimizer_config) > 2:
    bad.append('%d optimizer_config entries (one, or two = embedding + everything else, easy_rec_model.py:446-467)'
               % len(tc.optimizer_config))
  if any(oc.use_moving_average for oc in tc.optimizer_config):
    bad.append('optimizer_config.use_moving_average')
  if mc.model_class in _RANK_CLASSES:
    names = mc.DESCRIPTOR.fields_by_name['loss_type'].enum_type.values_by_number
    if mc.num_class != 1:
      bad.append('num_class %d (only the binary head, num_class 1)' % mc.num_class)
    if names[mc.loss_type].name not in ('CLASSIFICATION', 'L2_LOSS', 'SIGMOID_L2_LOSS'):
      bad.append('loss_type %s (rank models train with CLASSIFICATION = sigmoid cross entropy, L2_LOSS or SIGMOID_L2_LOSS)'
                 % names[mc.loss_type].name)
    extra = [names[l.loss_type].name for l in mc.losses if names[l.loss_type].name != 'CLASSIFICATION' or l.weight != 1.0]
    if extra or len(mc.losses) > 1:
      bad.append('model_config.losses %s' % ([names[l.loss_type].name for l in mc.losses],))
  for path, m in _walk_messages(mc, 'model_config'):
    kind = m.DESCRIPTOR.name
    if kind in ('TaskTower', 'BayesTaskTower'):
      lt = m.DESCRIPTOR.fields_by_name['loss_type'].enum_type.values_by_number[m.loss_type].name
      if len(m.losses) > 0:
        bad.append('%s.losses (per-tower loss list)' % path)
      if m.HasField('task_space_indicator_label'):
        bad.append('%s.task_space_indicator_label (in / out of task-space sample weights)' % path)
      if lt not in ('CLASSIFICATION', 'L2_LOSS', 'SIGMOID_L2_LOSS') or m.num_class != 1:
        bad.append('%s: loss_type %s / num_class %d (task towers train one output with sigmoid cross entropy or an '
                   'L2 loss)' % (path, lt, m.num_class))
    if kind in ('DNN', 'MLP'):
      from easyrec_b200 import layers as L
      for act in ([m.activation] if kind == 'DNN' else [m.activation, m.final_activation]):
        try:
          L.activation_kind(act)
        except NotImplementedError as e:
          bad.append('%s: %s' % (path, e))
  if bad:
    raise NotImplementedError('config is outside the hot-path scope: ' + '; '.join(bad))


def embedding_parallel(pipeline_config):
  """train_config.train_distribute: EmbeddingParallelStrategy (protos/train.proto; main.py / estimator
  `embedding_parallel` property, model/easy_rec_estimator.py:97-153)."""
  tc = pipeline_config.train_config
  names = tc.DESCRIPTOR.fields_by_name['train_distribute'].enum_type.values_by_number
  return names[tc.train_distribute].name == 'EmbeddingParallelStrategy'


def build_model(pipeline_config, batch_size, device, generator=None, cpu_generator=None, world=1, rank=0,
                default_seq_len=50, shard_tables=False):
  """Returns (input_layer, model, optimizer settings) for the config's model_class."""
  from easyrec_b200 import model as model_pkg
  check_scope(pipeline_config)
  mc = pipeline_config.model_config
  # the Parquet inputs bucket ids as `vals % num_buckets` (input/parquet_input.py:221,
  # input/parquet_input_v2.py:96-100) where the feature-column path maps out-of-range ids to 0
  specs = feature_specs(pipeline_config, packed_mod=input_type_name(pipeline_config).startswith('Parquet'),
                        default_seq_len=default_seq_len)
  kv = [s.name for s in specs if s.kv_capacity]
  if kv and world > 1 and not shard_tables:
    raise NotImplementedError(
        'ev_params (key-value tables) of %s with tables replicated over %d data-parallel ranks: replicas would need each '
        'rank\'s gathered update translated to its own rows; train them row-sharded (train_distribute: '
        'EmbeddingParallelStrategy) or on one GPU' % (kv, world))
  groups = feature_groups(mc)
  specs, keras_tables, pad_tags = embedding_layer_tables(mc, specs)
  opt = optimizer_settings(pipeline_config)
  cls = model_pkg.get_model_class(mc.model_class)
  wide_dim = cls.wide_output_dim(mc)
  from easyrec_b200 import backbone
  seq_groups = backbone.seq_output_groups(mc.backbone) if mc.HasField('backbone') else set()
  if generator is None and not str(device).startswith('cuda'):
    generator = cpu_generator   # tables initialised from the caller's seed on a host build too
  il = IL.InputLayer(specs, groups, batch_size, device, wide_output_dim=wide_dim,
                     embedding_optimizer=(_lib.OPT_MOMENTUM if opt.get('momentum', 0.0) > 0 else _OPT_KIND[opt['kind']]),
                     generator=generator,
                     adagrad_init=opt['acc0'], seq_att_groups=seq_att_groups(mc),
                     shard_n=world if (shard_tables and world > 1) else 1, shard_rank=rank if shard_tables else 0,
                     uniform_tables=keras_tables, dense_generator=cpu_generator,
                     multi_valued_seq=[(fc.feature_name if fc.HasField('feature_name') else fc.input_names[0])
                                       for fc in config_util.get_feature_configs(pipeline_config)
                                       if fc.HasField('seq_multi_sep')],
                     seq_combiners={(fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]):
                                    fc.sequence_combiner.WhichOneof('combiner')
                                    for fc in config_util.get_feature_configs(pipeline_config)
                                    if fc.HasField('sequence_combiner')},
                     seq_output_groups=seq_groups,
                     kv_seed=cpu_generator.initial_seed() if cpu_generator is not None else 0,
                     kv_embedding_parallel=embedding_parallel(pipeline_config) or shard_tables)
  il.pad_tags = pad_tags   # tag features of a backbone `embedding_layer` block: the readers pad them with the bucket of ''
  # RawFeature.normalizer_fn: applied to the min-max normalised value on the device (input/input.py:642-646); the
  # readers apply the same function on the host to raw features they bucketize themselves (readers.bucketize_raw)
  from easyrec_b200 import normalizer
  for fc in config_util.get_feature_configs(pipeline_config):
    if fc.HasField('normalizer_fn') and ftype_name(fc) == 'RawFeature':
      name = fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]
      if name in il.raw_cols:
        il.raw_normalizers[name] = normalizer.load(fc.normalizer_fn, 'torch')
  model = cls.from_config(mc, il, generator=cpu_generator)
  if il.attention_modules:
    # the attention MLPs of in-group sequence_features are InputLayer's in the reference (sequence_feature_layer.py);
    # their parameters train with the model's
    import torch
    model.input_attention = torch.nn.ModuleDict({k.replace('/', '__').replace('.', '_'): v
                                                 for k, v in il.attention_modules.items()})
  model = model.to(device)
  if mc.model_class in _RANK_CLASSES:
    model.loss_type = mc.DESCRIPTOR.fields_by_name['loss_type'].enum_type.values_by_number[mc.loss_type].name
  bind_task_labels(model, list(pipeline_config.data_config.label_fields))
  towers = task_towers_of(mc)
  if towers and hasattr(model, 'task_weights') and len(towers) == len(model.task_weights):
    model.task_loss_types = [t.DESCRIPTOR.fields_by_name['loss_type'].enum_type.values_by_number[t.loss_type].name
                             for t in towers]
  return il, model, opt


def task_towers_of(model_config):
  """the task tower messages of a multi-task model_config, in config order (mmoe / dbmtl / simple_multi_task /
  backbone model_params)"""
  which = model_config.WhichOneof('model')
  if which is None:
    return []
  return list(getattr(getattr(model_config, which), 'task_towers', []))


def embedding_layer_tables(model_config, specs):
  """Backbone `embedding_layer` blocks (layers/backbone.py:93-101,314-318 + InputLayer.get_bucketized_features,
  layers/input_layer.py:209-243 + keras EmbeddingLayer, layers/keras/embedding.py:26-81): the features of the block's
  feature group are bucketized by their own rule (`string_to_hash_bucket_fast(v, vocab_f)` for hashed ids, numeric
  inputs taken as already bucketized), offset by the vocabularies before them and looked up in ONE
  `Embedding(sum vocab, embedding_dim)` of the block.  That is the arena layout of this path already: each feature
  gets its own `vocab_f`-row table of the BLOCK's width (back to back in group order = the offsets), Keras' default
  `uniform(-0.05, 0.05)` initialiser instead of the feature columns' truncated normal.

  A TagFeature (string tokens hashed on the host) takes part the way the reference treats it: the ragged tags are
  densified with '' PADDING up to the longest list of the batch, the padding is hashed and looked up like a tag, and the
  step axis is pooled by the block's `combiner` - 'weight' (default): mean over all positions when the feature has no
  weights, sum(w e) / sum(w) with kv weights (padding weighs 0); 'mean'; 'sum' (input_layer.py:232-235,
  embedding.py:9-23, 60-78).  The readers pad such features (pad_tags: feature -> bucket of ''); 'max' / 'min' are refused.

  Returns (specs with those features re-dimensioned, {table name: 0.05}, {tag feature: pad bucket})."""
  if not model_config.HasField('backbone'):
    return specs, {}, {}
  by_name = {s.name: i for i, s in enumerate(specs)}
  groups = {g.group_name: list(g.feature_names) for g in model_config.feature_groups}
  other_use = collections.Counter(n for g in model_config.feature_groups for n in g.feature_names)
  specs, tables, pad_tags = list(specs), {}, {}
  blocks = list(model_config.backbone.blocks) + [b for p in model_config.backbone.packages for b in p.blocks]
  for b in blocks:
    if b.WhichOneof('layer') != 'embedding_layer':
      continue
    if len(b.inputs) != 1 or b.inputs[0].WhichOneof('name') != 'feature_group_name':
      raise ValueError('embedding_layer block %s takes exactly one feature_group_name input' % b.name)
    for n in groups[b.inputs[0].feature_group_name]:
      sp = specs[by_name[n]]
      if sp.vocab is not None:
        raise NotImplementedError('embedding_layer block %s: feature %s has a vocabulary; the block hashes string '
                                  'features into vocabulary-sized buckets (layers/input_layer.py:222-243) instead of '
                                  'looking them up, which is not built' % (b.name, n))
      if sp.kind not in ('id', 'tag'):
        raise NotImplementedError('embedding_layer block %s: feature %s is a %s feature; id / bucketized / tag features '
                                  'go through this block' % (b.name, n, sp.kind))
      if other_use[n] > 1:
        raise NotImplementedError('feature %s is read by embedding_layer block %s and by another feature group: it '
                                  'would need two tables' % (n, b.name))
      table = '%s/%s_embedding' % (b.name, n)
      extra = {}
      if sp.kind == 'tag':
        comb = b.embedding_layer.combiner
        if comb not in ('weight', 'mean', 'sum'):
          raise NotImplementedError('embedding_layer block %s: combiner %r over a tag feature' % (b.name, comb))
        if sp.bucket_mode != _lib.BUCKET_IDENTITY or sp.num_buckets <= 0:
          # (the block hashes the densified STRING tags itself, '' included; integer tags cannot be densified with '')
          raise NotImplementedError('embedding_layer block %s: tag feature %s must be a STRING field with a '
                                    'hash_bucket_size' % (b.name, n))
        extra = dict(combiner='sum' if comb == 'sum' else 'mean')
        # (bucket of the '' padding, whether kv weights count: a callable combiner ignores them, embedding.py:11-12)
        pad_tags[n] = (int(_lib.fingerprint64('') % sp.num_buckets), comb == 'weight')
      specs[by_name[n]] = sp._replace(embedding_dim=int(b.embedding_layer.embedding_dim), embedding_name=table, **extra)
      tables[table] = 0.05
  return specs, tables, pad_tags


def bind_task_labels(model, label_fields):
  """Multi-task towers read the label their `label_name` names; a tower without one takes the label at its own
  position (model/multi_task_model.py:114-122).  Sets model.label_cols = column of each tower in the [B, n_label]
  label matrix the readers build in data_config.label_fields order."""
  names = getattr(model, 'label_names', None)
  if names is None:
    return
  cols = []
  for i, n in enumerate(names):
    if not n:
      if i >= len(label_fields):
        raise ValueError('task tower %d has no label_name and there is no label field at its position' % i)
      cols.append(i)
    elif n in label_fields:
      cols.append(label_fields.index(n))
    else:
      raise ValueError('task tower label_name %r is not one of data_config.label_fields %r' % (n, label_fields))
  model.label_cols = cols
