"""InputLayer: feature groups -> dense tensors, on the fused sm_90a lookup path.

Mirrors the reference surface
  InputLayer(feature_configs, feature_groups, ..., wide_output_dim)       layers/input_layer.py:33-69
  input_layer(features, group_name) -> (concat [B, sum D], [per-feature])   layers/input_layer.py:245-278
  SeqInputLayer(...)(features, seq_group) -> {key, hist_seq_emb, hist_seq_len}  layers/seq_input_layer.py:34-124
with `FeatureColumnParser` (feature_column/feature_column.py:44-203, 259-656) collapsed into a
static *table plan*: which table each feature reads (shared `embedding_name` groups), its bucket
rule, combiner and output column -- fixed at construction, uploaded once as er_slot_t records.

Input contract (the reference's packed form, input/parquet_input.py:201-239, plus sequences):
  features['sparse_fea'] = ids int64 [n_id*B], feature-major, for the single-valued IdFeatures
  features['dense_fea']  = float32 [B, sum raw_input_dim] in raw-feature config order
  features['seq_fea'][name] = (ids int64 [B, T], lens int32 [B])        SequenceFeature
  features['tag_fea'][name] = (ids int64 [L], lens int32 [B], weights fp32 [L] | None)  TagFeature
Outputs keep feature_group CONFIG order (compat/feature_column/feature_column.py:388-414).

Per arena (= embedding_dim) the lookups run as up to three uniform launches -- single-valued slots,
sequence slots (one segment per (sample, position), un-pooled [B,T,D]), CSR tag slots -- and the
backward is ONE dedup + fused row update over all of them, so a table shared by several slots
(key + history of the same id space) gets one optimizer step from the summed gradient, as in TF.
"""
import collections
import os

import numpy as np
import torch

from easyrec_b200 import _lib
from easyrec_b200 import embedding as E
from easyrec_b200 import kernels as K

FeatureSpec = collections.namedtuple(
    'FeatureSpec',
    ['name', 'kind',            # 'id' | 'raw' | 'tag' | 'seq'
     'embedding_dim', 'bucket_mode', 'num_buckets', 'combiner', 'embedding_name',
     'min_val', 'max_val', 'raw_input_dim', 'seq_len'])


def _bucket_rule(hash_bucket_size, num_buckets, packed_mod, host_hashed=False):
  if hash_bucket_size > 0:
    if host_hashed:
      # string-typed field: the reader already computed Fingerprint64(bytes) % hash_bucket_size (er_csv_parse),
      # the device takes the bucket as it is (-1 = empty string = no value)
      return _lib.BUCKET_IDENTITY, hash_bucket_size
    return _lib.BUCKET_FARM_DECIMAL, hash_bucket_size
  if packed_mod:
    return _lib.BUCKET_MOD, num_buckets
  return _lib.BUCKET_IDENTITY, num_buckets


def id_feature(name, embedding_dim, hash_bucket_size=0, num_buckets=0, combiner='sum',
               embedding_name='', packed_mod=False, host_hashed=False):
  """IdFeature: hash_bucket_size -> Fingerprint64(as_string) % size; num_buckets -> identity
  (feature_column/feature_column.py:259-300).  packed_mod: the Parquet packed rule
  `vals % num_buckets` (input/parquet_input.py:221)."""
  mode, nb = _bucket_rule(hash_bucket_size, num_buckets, packed_mod, host_hashed)
  return FeatureSpec(name, 'id', embedding_dim, mode, nb, combiner, embedding_name, 0., 0., 1, 1)


def raw_feature(name, embedding_dim=0, min_val=0.0, max_val=0.0, raw_input_dim=1):
  """RawFeature: (x-min)/(max-min) when max>min (input/input.py:638-640); with embedding_dim>0
  it becomes ids 0..k-1 weighted by the values (input/input.py:648-673)."""
  # raw_input_dim 1: a ONE-row table that every sample hits with weight x (ids are all 0): its gradient is a weighted
  # column sum, which er_embedding_bwd computes without sending B duplicates of one row through the dedup
  mode = _lib.BUCKET_ONE_ROW if raw_input_dim == 1 else _lib.BUCKET_NONE
  return FeatureSpec(name, 'raw', embedding_dim, mode, raw_input_dim, 'sum', '',
                     float(min_val), float(max_val), raw_input_dim, 1)


def multi_feature(name, kind, embedding_dim, hash_bucket_size=0, num_buckets=0, combiner='sum',
                  embedding_name='', seq_len=1, packed_mod=False, host_hashed=False):
  """TagFeature (kind 'tag': multi-valued, pooled by `combiner`, optional kv weights;
  feature_column/feature_column.py:301-360) or SequenceFeature (kind 'seq': un-pooled [B,T,D];
  feature_column_v2.py:4988-5002)."""
  assert kind in ('tag', 'seq')
  mode, nb = _bucket_rule(hash_bucket_size, num_buckets, packed_mod, host_hashed)
  return FeatureSpec(name, kind, embedding_dim, mode, nb, combiner, embedding_name, 0., 0., 1,
                     max(int(seq_len), 1))


_COMBINER = {'sum': _lib.COMBINER_SUM, 'mean': _lib.COMBINER_MEAN, 'sqrtn': _lib.COMBINER_SQRTN}

# The plan's records.  A column of a feature group's concat, `width` wide: kind 'emb' (looked up), 'dense' (raw values,
# no table), 'seqc' (a SequenceFeature pooled by its sequence_combiner) or 'att' (target attention over the group's
# sequence_features: `out_key` names their seq_layout, `need_key` appends the key).  A looked-up column reads `slot`
# into columns [col, col + dim) of the (dim, out_key) output matrix.
GroupColumn = collections.namedtuple('GroupColumn', ['name', 'kind', 'width', 'dim', 'out_key', 'col', 'need_key', 'slot'],
                                     defaults=(None,) * 5)
# a key or history column of a seq_layout, or a sequence column of a seq_group_layout
SeqColumn = collections.namedtuple('SeqColumn', ['name', 'dim', 'out_key', 'col', 'slot'], defaults=(None, None))
# one K7 update of a step: an arena's MergedCall - or, row-sharded with several launches on the arena, one launch's
# _SubCall - with the rows, lookup weights, output matrices and segment ids of the lookup
Pending = collections.namedtuple('Pending', ['call', 'rows', 'weights', 'outs', 'seg_ids'])


class _SubCall(object):
  """One uniform launch over an arena: a list of slots that all have the same segment count."""

  def __init__(self, kind, n_seg_per_slot):
    self.kind = kind               # 'single' | 'seq' | 'tag'
    self.n_seg_per_slot = n_seg_per_slot
    self.items = []                # (out_key, feature name, Slot, source)
    self.call = None               # E.ArenaCall


class MergedCall(object):
  """The arena-wide slot plan used by K7: every sub-call's slots back to back (segments
  renumbered), all output matrices as grad buffers."""

  def __init__(self, arena, subcalls):
    self.arena = arena
    recs = []
    self.buf_of = []   # (subcall index, local out_buf) per merged buffer
    seg = 0
    lookups = 0
    self.sub_lookup_off = []
    self.sub_seg_off = []
    for si, sc in enumerate(subcalls):
      c = sc.call
      base_buf = len(self.buf_of)
      for b in range(len(c.out_strides)):
        self.buf_of.append((si, b))
      self.sub_seg_off.append(seg)
      self.sub_lookup_off.append(lookups)
      for r in c.slots_np:
        recs.append(dict(num_buckets=int(r['num_buckets']), row_offset=int(r['row_offset']),
                         seg_begin=int(r['seg_begin']) + seg, n_seg=int(r['n_seg']),
                         bucket_mode=int(r['bucket_mode']), combiner=int(r['combiner']),
                         out_buf=int(r['out_buf']) + base_buf, out_stride=int(r['out_stride']),
                         out_col=int(r['out_col']), shard_n=int(r['shard_n'])))
      seg += c.n_seg
      lookups += c.max_lookups
    assert len(self.buf_of) <= _lib.MAX_BUFS, 'too many output matrices on one arena'
    self.slots_np = K.make_slots(recs, arena.dim)
    self.slots_dev = K.slots_to_device(self.slots_np, arena.device)
    self.n_slots = len(recs)
    self.n_seg = seg
    self.max_lookups = lookups
    self.out_strides = [subcalls[si].call.out_strides[b] for si, b in self.buf_of]
    self._out_rows = [subcalls[si].call.out_rows(b) for si, b in self.buf_of]
    self.ws = K.bwd_workspace(lookups, arena.device, arena.dim)
    self.has_csr = any(sc.kind in ('tag', 'mseq') for sc in subcalls)
    self.single_valued = not self.has_csr
    self.needs_scale = any(sc.call.needs_scale for sc in subcalls)
    dev = arena.device
    self.rows = torch.empty(lookups, dtype=torch.int64, device=dev) if len(subcalls) > 1 else None
    self.weights = None
    self.seg_ids = torch.empty(lookups, dtype=torch.int32, device=dev) if self.has_csr else None
    if len(subcalls) == 1:
      self.seg_scale = subcalls[0].call.seg_scale   # written in place by K2
    else:
      self.seg_scale = torch.ones(seg, dtype=torch.float32, device=dev) if self.needs_scale else None

  def out_rows(self, buf):
    return self._out_rows[buf]


class InputLayer(object):
  """Builds arenas + fused calls for a set of feature groups and evaluates them.

  groups: OrderedDict group_name -> dict(features=[names...], wide=bool)
  seq_att_groups: OrderedDict name -> list of (key feature names, hist_seq feature names)
      (SeqAttGroupConfig.seq_att_map, protos/feature_config.proto; layers/seq_input_layer.py)
  A group marked wide uses `wide_output_dim` columns per feature with combiner sum
  (feature_column/feature_column.py:616-622)."""

  def __init__(self, features, groups, batch_size, device, wide_output_dim=1,
               embedding_optimizer=_lib.OPT_ADAGRAD, shard_n=1, shard_rank=0, generator=None,
               adagrad_init=0.1, seq_att_groups=None, max_tag_lookups=None, uniform_tables=None,
               dense_generator=None, multi_valued_seq=(), seq_combiners=None, seq_output_groups=()):
    self.features = collections.OrderedDict((f.name, f) for f in features)
    # groups read only by backbone `input_layer { output_seq_and_normal_feature: true }` blocks
    # (layers/common_layers.py:104-131): their SequenceFeatures come out un-pooled as one [B, T, sum D] tensor
    self.seq_output_groups = set(seq_output_groups)
    # SequenceFeatures with seq_multi_sep: every step holds a LIST of values, pooled per step by the feature's
    # combiner (input/input.py:686-700 builds the 3-D SparseTensor; pinned by test/embed_test.py:88-151) - a CSR slot
    # with one segment per (sample, step) instead of one id per step
    self.multi_valued_seq = set(multi_valued_seq)
    # SequenceFeatures of a PLAIN feature group carry a sequence_combiner (layers/input_layer.py:312-347): 'attention' =
    # softmax over the steps of a learned linear score (dense(units=1, no bias)), masked beyond the length, weighted sum
    self.seq_combiners = dict(seq_combiners or {})
    self.groups = groups
    self.seq_att_groups = seq_att_groups or collections.OrderedDict()
    self.batch_size = batch_size
    self.device = device
    self.wide_output_dim = wide_output_dim
    self.sparse_names = [f.name for f in features if f.kind == 'id']
    self.raw_names = [f.name for f in features if f.kind == 'raw']
    self.raw_cols = {}
    c = 0
    for n in self.raw_names:
      self.raw_cols[n] = (c, c + self.features[n].raw_input_dim)
      c += self.features[n].raw_input_dim
    self.n_dense = c
    # ---- table plan -------------------------------------------------------------------
    self.arenas = collections.OrderedDict()          # dim -> Arena
    self.subcalls = collections.OrderedDict()        # dim -> OrderedDict(key -> _SubCall)
    self.group_layout = {}       # group -> [GroupColumn] in concat order
    self.seq_layout = {}         # seq group -> dict(key=[SeqColumn], hist=[SeqColumn], T=steps)
    self.seq_group_layout = {}   # output_seq_and_normal_feature group -> dict(seq=[SeqColumn], T=steps)
    self.attention_modules = collections.OrderedDict()
    self.seqc_order = {}      # group -> names of its sequence-combiner features in config order
    self._shard = (shard_n, shard_rank)
    for gname, g in groups.items():
      self._plan_group(gname, g, dense_generator)
    for sname, maps in self.seq_att_groups.items():
      # the key column lives in the sequence group's own variable scope
      # (layers/seq_input_layer.py:56-75): a table separate from the plain group's
      self._plan_seq_layout(sname, sname, maps)
    for gname, g in groups.items():
      for sub in g.get('seq') or []:
        self._plan_sequence_features(gname, g, sub, dense_generator)
    self._materialize(embedding_optimizer, generator, adagrad_init, uniform_tables)
    self._plan_calls(max_tag_lookups)
    mn = [self.features[n].min_val for n in self.raw_names for _ in range(self.features[n].raw_input_dim)]
    mx = [self.features[n].max_val for n in self.raw_names for _ in range(self.features[n].raw_input_dim)]
    rng = np.array(mx, np.float32) - np.array(mn, np.float32)
    self.raw_has_range = bool((rng > 0).any())
    self.raw_normalizers = collections.OrderedDict()   # feature -> normalizer_fn (set by builder.build_model)
    self.raw_range = torch.tensor(np.where(rng > 0, rng, 1.0), dtype=torch.float32, device=device)
    self.raw_sub = torch.tensor(np.where(rng > 0, np.array(mn, np.float32), 0.0),
                                dtype=torch.float32, device=device)
    # step-varying optimizer scalars live in device memory (K.StepHyper): a captured graph follows the schedule
    self.hyper = K.StepHyper(device)
    self.hyper.set(0.01, 0)
    self.opt_holder = {'opt': self.hyper.opt(embedding_optimizer)}
    # EmbeddingParallel (train_distribute: EmbeddingParallelStrategy): the tables are row-sharded over shard_n ranks
    # and every lookup goes through the all-to-all exchange of sharded.ShardedLookup
    self.ep = shard_n > 1
    if self.ep:
      self._plan_exchanges()
    # embedding_learning_rate_multiplier: the reference multiplies the GRADIENT of every `embedding_weights`
    # variable by it (model/easy_rec_estimator.py:308-317 gradient_multipliers), before the optimizer rule
    self.emb_grad_mult = 1.0
    # 1/N of data-parallel replicas or of row-sharded tables (compat/optimizers.py:289-292,315-316)
    self.replica_grad_scale = 1.0 / shard_n
    self._pending = []        # [Pending] of the last lookup(): what backward_update() applies
    self._rows_cache = {}
    self.placements = E.Placements()
    self._side = None
    self.presort_enabled = True
    self._preset_rows = {}
    self._rows_bufs = {}
    self._pos = {}
    self._next_ids = {}
    self._clip_state = {}

  # ---- table plan: the constructor's stages ---------------------------------------------
  def _add_slot(self, dim, out_key, fname, table, kind, wide=False):
    """one lookup of feature `fname` from `table` into the (dim, out_key) output matrix; returns its Slot"""
    f = self.features[fname]
    B = self.batch_size
    arena = self.arenas.setdefault(dim, E.Arena(dim, self.device, *self._shard))
    arena.add_table(table, f.num_buckets)
    if kind == 'seq' and fname in self.multi_valued_seq:
      kind = 'mseq'
      sk, nseg = ('mseq', f.seq_len), B * f.seq_len
    elif kind == 'seq':
      sk, nseg = ('seq', f.seq_len), B * f.seq_len
    elif kind == 'tag':
      sk, nseg = ('tag',), B
    else:
      sk, nseg = ('single',), B
    subs = self.subcalls.setdefault(dim, collections.OrderedDict())
    sc = subs.setdefault(sk, _SubCall(sk[0], nseg))
    comb = _lib.COMBINER_SUM if (wide or f.kind == 'raw' or kind == 'seq') else _COMBINER[f.combiner]
    slot = E.Slot(out_key + '/' + fname, table, f.bucket_mode, f.num_buckets, comb, out_buf=out_key,
                  n_seg_per_sample=f.seq_len if kind in ('seq', 'mseq') else 1)
    # id and sequence slots never carry per-lookup weights (raw-value and kv-weighted tag slots do)
    slot.unit_weights = f.kind != 'raw' and kind in ('single', 'seq', 'mseq')
    if f.kind == 'raw':
      src = ('raw', self.raw_cols[fname][0])
    elif kind in ('seq', 'mseq'):
      src = ('seq', fname)
    elif kind == 'tag':
      src = ('tag', fname)
    else:
      src = ('id', self.sparse_names.index(fname))
    sc.items.append((out_key, fname, slot, src))
    return slot

  def _plan_group(self, gname, g, dense_generator):
    """the columns of one feature group, in config order"""
    layout, seqc, seq, T = [], [], [], None
    wide = bool(g.get('wide'))
    if gname in self.seq_output_groups:
      if wide:
        raise NotImplementedError('feature group %s: wide_deep WIDE read by output_seq_and_normal_feature' % gname)
      if g.get('seq'):
        raise NotImplementedError('feature group %s: sequence_features in a group read by '
                                  'output_seq_and_normal_feature' % gname)
    for fname in g['features']:
      f = self.features[fname]
      dim = self.wide_output_dim if wide else f.embedding_dim
      if f.kind == 'raw' and dim == 0:
        layout.append(GroupColumn(fname, 'dense', f.raw_input_dim))
        continue
      if f.kind == 'seq' and gname in self.seq_output_groups:
        # InputLayer.get_sequence_feature (layers/input_layer.py:154-192): the un-pooled [B, T, D] lookup, in the
        # table of the column itself (variable_scope('input_layer/' + column name): no group scope, so a feature
        # listed in another group too reads the same table).  T is max_seq_len, fixed so the step can be captured.
        if fname in self.multi_valued_seq:
          raise NotImplementedError('SequenceFeature %s: seq_multi_sep (multi-valued steps) in group %s read by '
                                    'output_seq_and_normal_feature' % (fname, gname))
        if T not in (None, f.seq_len):
          raise NotImplementedError('feature group %s: SequenceFeatures of different max_seq_len (%d, %d) read by '
                                    'output_seq_and_normal_feature' % (gname, T, f.seq_len))
        T = f.seq_len
        # all sequence features of one width write one [B*T, sum D] matrix: the concat costs nothing
        slot = self._add_slot(dim, gname + '#seq', fname, f.embedding_name or fname + '_embedding', 'seq')
        seq.append(SeqColumn(fname, dim, gname + '#seq', slot=slot))
        continue
      if f.kind == 'seq':
        if self.seq_combiners.get(fname) != 'attention' or wide or fname in self.multi_valued_seq:
          raise NotImplementedError('SequenceFeature %s in a plain group needs a sequence_combiner { attention } '
                                    '(or put it in seq_att_groups / sequence_features)' % fname)
        # un-pooled [B*T, D] rows in a matrix of their own; pooled in lookup() by the attention combiner.  In the
        # concat these features follow the plain ones in NAME order, in the per-feature list in config order
        # (input_layer.py:312, 364-367)
        out_key = '%s#seqc/%s' % (gname, fname)
        slot = self._add_slot(dim, out_key, fname, f.embedding_name or fname + '_embedding', 'seq')
        seqc.append(GroupColumn(fname, 'seqc', dim, dim, out_key, slot=slot))
        from easyrec_b200 import layers as L
        att = L.Dense(dim, 1, generator=dense_generator)
        att.bias.requires_grad_(False)       # tf.layers.dense(units=1, use_bias=False, name='attention')
        self.attention_modules[out_key] = att
        continue
      table = (f.embedding_name or fname + '_embedding') + ('_wide' if wide else '')
      kind = 'tag' if f.kind == 'tag' else 'single'
      # one output matrix per (group, launch kind): the single-valued and the CSR launch of a mixed group
      # write their own matrices, the group's concat is assembled from both in config order
      out_key = gname if kind == 'single' else gname + '#tag'
      slot = self._add_slot(dim, out_key, fname, table, kind, wide=wide)
      layout.append(GroupColumn(fname, 'emb', dim, dim, out_key, slot=slot))
    self.seqc_order[gname] = [e.name for e in seqc]
    self.group_layout[gname] = layout + sorted(seqc, key=lambda e: e.name)
    if gname in self.seq_output_groups:
      if not seq:
        raise ValueError('[input_%s] sequence feature is empty (output_seq_and_normal_feature)' % gname)
      self.seq_group_layout[gname] = dict(seq=seq, T=T)

  def _plan_seq_layout(self, sname, scope, maps, own=()):
    """SeqInputLayer (layers/seq_input_layer.py:34-124) over `maps` [(key names, hist_seq names)]: key and history
    columns in tables of the variable scope `scope`; a key that is one of the `own` group columns reuses it"""
    key, hist, T = [], [], None
    for keys, hists in maps:
      for k in keys:
        f = self.features[k]
        mine = next((e for e in own if e.name == k and e.kind == 'emb'), None)
        if mine is not None:
          if mine.out_key != scope:
            raise NotImplementedError('sequence_features key %s is a multi-valued feature of group %s' % (k, scope))
          key.append(SeqColumn(k, mine.dim, mine.out_key, slot=mine.slot))
          continue
        table = f.embedding_name or '%s/%s_embedding' % (scope, k)
        slot = self._add_slot(f.embedding_dim, sname + '/key', k, table, 'single')
        key.append(SeqColumn(k, f.embedding_dim, sname + '/key', slot=slot))
      for h in hists:
        f = self.features[h]
        assert f.kind == 'seq', '%s must be a SequenceFeature' % h
        assert T in (None, f.seq_len), 'hist_seq features of one group must share seq_len'
        T = f.seq_len
        table = f.embedding_name or '%s/%s_embedding' % (scope, h)
        slot = self._add_slot(f.embedding_dim, sname + '/hist', h, table, 'seq')
        hist.append(SeqColumn(h, f.embedding_dim, sname + '/hist', slot=slot))
    self.seq_layout[sname] = lay = dict(key=key, hist=hist, T=T)
    return lay

  def _plan_sequence_features(self, gname, g, sub, dense_generator):
    """feature_groups[...].sequence_features: target attention INSIDE a group (layers/input_layer.py:96-111 ->
    SequenceFeatureLayer, layers/sequence_feature_layer.py:190-249 -> SeqInputLayer with scope_name = the group's):
    a key that is a feature of the same group reuses the group's own embedding output (seq_input_layer.py:63-75);
    histories live in the group's scope; the attended vector (+ the key) is appended to the group's concat"""
    if g.get('wide'):
      raise NotImplementedError('sequence_features in the wide group %s' % gname)
    from easyrec_b200 import layers as L
    sname = '%s/%s' % (gname, sub['name'])
    lay = self._plan_seq_layout(sname, gname, sub['maps'], own=self.group_layout[gname])
    dk, dh = sum(e.dim for e in lay['key']), sum(e.dim for e in lay['hist'])
    if dk != dh:
      raise NotImplementedError('sequence_features %s: key width %d != history width %d (allow_key_transform)'
                                % (sname, dk, dh))
    need_key = bool(sub.get('need_key', True))
    self.group_layout[gname].append(GroupColumn('seq_fea/' + sub['name'], 'att', dh + (dk if need_key else 0),
                                                out_key=sname, need_key=need_key))
    self.attention_modules[sname] = L.DNN(4 * dh, sub['units'], last_layer_no_activation=True,
                                          last_layer_no_batch_norm=True, generator=dense_generator)

  def _materialize(self, embedding_optimizer, generator, adagrad_init, uniform_tables):
    # ER_BUCKET_ONE_ROW promises that no other slot of the arena reads the table (a raw feature listed in two groups
    # of the same width breaks that): such slots go through the ordinary dedup
    for subs in self.subcalls.values():
      uses = collections.Counter(slot.table for sc in subs.values() for _, _, slot, _ in sc.items)
      for sc in subs.values():
        for _, _, slot, _ in sc.items:
          if slot.bucket_mode == _lib.BUCKET_ONE_ROW and (uses[slot.table] > 1 or sc.kind != 'single'):
            slot.bucket_mode = _lib.BUCKET_NONE
    for a in self.arenas.values():
      a.materialize(embedding_optimizer, generator=generator, adagrad_init=adagrad_init)
      # tables of a backbone `embedding_layer` block: Keras Embedding's uniform(-limit, limit) initialiser
      for tname, limit in (uniform_tables or {}).items():
        if tname in a.tables and os.environ.get('ER_PLAN_ONLY') != '1':
          off, local, _ = a.tables[tname]
          rows = torch.empty(local, a.dim, dtype=torch.float32, device=self.device)
          rows.uniform_(-limit, limit, generator=generator)
          a.weight[off:off + local].copy_(rows)

  def _plan_calls(self, max_tag_lookups):
    """one ArenaCall per sub-call (its output matrices in first-use order), one MergedCall per arena"""
    B, device = self.batch_size, self.device
    self.calls = collections.OrderedDict()     # dim -> the single-valued ArenaCall (bench/tests)
    self.merged = collections.OrderedDict()    # dim -> MergedCall
    self._gather_plan = {}
    self.static_ids = {}
    self.static_w = {}
    self.out_index = {}                        # (dim, out_key) -> (subcall key, local buf index)
    for dim, subs in self.subcalls.items():
      for sk, sc in subs.items():
        keys = list(dict.fromkeys(out_key for out_key, _, _, _ in sc.items))
        widths = [0] * len(keys)
        slots = []
        for out_key, _, slot, _ in sc.items:
          slot.out_buf = keys.index(out_key)
          widths[slot.out_buf] += dim
          slots.append(slot)
        if sc.kind == 'tag':
          cap = max_tag_lookups or 8 * B * len(slots)
          sc.call = E.ArenaCall(self.arenas[dim], slots, B, widths, single_valued=False, max_lookups=cap)
        elif sc.kind == 'mseq':
          cap = max_tag_lookups or 4 * B * sk[1] * len(slots)     # room for 4 values per step on average
          sc.call = E.ArenaCall(self.arenas[dim], slots, B, widths, single_valued=False, max_lookups=cap)
        else:
          sc.call = E.ArenaCall(self.arenas[dim], slots, B, widths, single_valued=True)
        for j, k in enumerate(keys):
          self.out_index[(dim, k)] = (sk, j)
        if sc.kind == 'single':
          self.calls[dim] = sc.call
          src = [s for _, _, _, s in sc.items]
          self.static_ids[dim] = torch.zeros(sc.call.n_seg, dtype=torch.int64, device=device)
          has_raw = any(k == 'raw' for k, _ in src)
          self.static_w[dim] = (torch.ones(sc.call.n_seg, dtype=torch.float32, device=device)
                                if has_raw else None)
          sc.call.identity_ids = ([k for k, _ in src] == ['id'] * len(src) and
                                  [i for _, i in src] == list(range(len(self.sparse_names))))
          sc.call.sources = src
      self.merged[dim] = MergedCall(self.arenas[dim], list(subs.values()))
    # every looked-up column reads its position from its own slot's ArenaCall
    cols = {id(slot): c for subs in self.subcalls.values() for sc in subs.values()
            for slot, c in zip(sc.call.slots, sc.call.slot_cols)}

    def resolved(columns):
      return [e if e.slot is None else e._replace(col=cols[id(e.slot)]) for e in columns]
    self.group_layout = {g: resolved(lay) for g, lay in self.group_layout.items()}
    self.seq_layout = {s: dict(lay, key=resolved(lay['key']), hist=resolved(lay['hist']))
                       for s, lay in self.seq_layout.items()}
    self.seq_group_layout = {g: dict(lay, seq=resolved(lay['seq'])) for g, lay in self.seq_group_layout.items()}

  def _plan_exchanges(self):
    """EmbeddingParallel: a ShardedLookup around every sub-call.  The single-valued and multi-valued (CSR) launches of
    an arena form ONE exchange - one K8, one row update per table on the owner - shared by the arenas of the same
    combined row plan (the wide dim-1 tables next to the deep ones); every history launch has an exchange of its own."""
    from easyrec_b200.sharded import ShardedLookup
    shard_n, shard_rank = self._shard
    exchanges = {}       # combined row plan -> the exchange its arenas share (ids once, rows in one packed all-to-all)
    self._ex_plan = []   # (exchange, dim of its first arena, that arena's launches in range order)
    for dim, subs in self.subcalls.items():
      for sk, sc in subs.items():
        if sc.kind != 'seq':
          continue
        # un-pooled histories (one lookup per step, padded steps dropped by K1): an exchange of their own.  The owner
        # applies one row update per exchange, so a table must not be read by a history and by another launch
        mine = set(slot.table for _, _, slot, _ in sc.items)
        for sk2, sc2 in subs.items():
          shared = sorted(mine & set(slot.table for _, _, slot, _ in sc2.items)) if sc2 is not sc else None
          if shared:
            raise NotImplementedError('EmbeddingParallel: table(s) %s are read both by history (SequenceFeature) '
                                      'steps and by other features; give the histories tables of their own'
                                      % shared)
        if len(subs) > 1 and self.arenas[dim].opt_kind == _lib.OPT_ADAM_ROWS:
          # adam_optimizer's dense decay sweeps every row the owner did not update: with two exchanges on one arena
          # each would sweep the rows only the other one updated
          raise NotImplementedError('EmbeddingParallel: adam_optimizer with histories next to other features of '
                                    'embedding_dim %d (their tables share one arena and two exchanges)' % dim)
        sc.sharded = ShardedLookup(sc.call, shard_n, shard_rank, seq=(self.batch_size, sk[1]))
      flat = [sc for sc in subs.values() if sc.kind != 'seq']
      if flat:
        key = tuple(self._rows_key(sc) for sc in flat)
        ex = exchanges.get(key)
        for sc in flat:
          sc.sharded = ShardedLookup(sc.call, shard_n, shard_rank, exchange=ex)
          ex = sc.sharded.ex
        if key not in exchanges:
          exchanges[key] = ex
          self._ex_plan.append((ex, dim, flat))
      if len(subs) == 1:
        self.merged[dim].sharded = next(iter(subs.values())).sharded

  def group_width(self, name):
    """width of the group's concat [B, width]"""
    return sum(e.width for e in self.group_layout[name])

  def discard_pending(self):
    """forget the K7 updates of the last lookup() without applying them (evaluation, or updates applied elsewhere)"""
    self._pending = []

  # ------------------------------------------------------------------
  def set_optimizer_step(self, lr, step, beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0):
    """Per-step hyper-parameters of the fused row update (host-side schedule,
    core/learning_schedules.py:30-75; beta powers as compat/adam_s.py:233-245)."""
    kind = next(iter(self.arenas.values())).opt_kind
    h = self.hyper
    if np.float32(beta1) != h.beta1 or np.float32(beta2) != h.beta2:
      h.beta1, h.beta2, h._pow_step = np.float32(beta1), np.float32(beta2), None
    h.set(lr, step, grad_scale * self.emb_grad_mult * self.replica_grad_scale)
    self.opt_holder['opt'] = h.opt(kind, eps)

  def backward_update(self):
    """After loss.backward(): K7 for every arena looked up since the last call (dedup, segment
    sum and the fused optimizer row update).  The reference's counterpart is
    opt.apply_gradients on the tables' IndexedSlices (compat/optimizers.py:413-416)."""
    if self.ep:
      for m, rows, w, outs, seg_ids in self._pending:
        m.sharded.backward_update(outs, self.opt_holder['opt'])
      self._pending = []
      return
    if self.placements.presorted:
      torch.cuda.current_stream().wait_stream(self._side)   # join the early sorts
    cur = torch.cuda.current_stream() if str(self.device).startswith('cuda') else None
    forked = False
    for idx, (m, rows, w, outs, seg_ids) in enumerate(self._pending):
      # arenas with the same row plan (DeepFM / Wide&Deep: the wide dim-1 and the deep tables) look up the
      # same rows tensor: a later K7 may reuse an earlier one's bucket placement.
      src = self.placements.sorted_from(rows, m.arena.n_rows, m.arena.dim, m.ws)
      if idx > 0 and src is not None and self._side is not None and cur is not None:
        # different arenas, sort already done: this update runs beside the first one on the side stream
        if not forked:
          self._side.wait_stream(cur)
          forked = True
        with torch.cuda.stream(self._side):
          E.fused_backward_update(m, rows, outs, self.opt_holder['opt'], weights=w, seg_ids=seg_ids, sorted_from=src)
      else:
        E.fused_backward_update(m, rows, outs, self.opt_holder['opt'], weights=w, seg_ids=seg_ids, sorted_from=src)
    if forked:
      cur.wait_stream(self._side)
    self._pending = []

  def ep_hold_updates(self, on=True):
    """EmbeddingParallel + global-norm clipping: backward_update() stops after the gradient all-to-all; the owners
    update in ep_apply_held() once the clip factor is in the gradient scale."""
    for ex in self._exchanges():
      ex.hold = bool(on)

  def ep_recv_sqnorm(self):
    """sum of squares of the gradient rows this rank RECEIVED as an owner: one entry per (source rank, distinct row) -
    the IndexedSlices.values of the sharded tables as the reference's backward through hvd.alltoall builds them
    (compat/optimizers.py:453-470 part_norms), times the embedding gradient multiplier squared."""
    total = torch.zeros((), dtype=torch.float32, device=self.device)
    for ex in self._exchanges():
      total = total + (ex.recv_g * ex.recv_g).sum()
    return total * float(self.emb_grad_mult) ** 2

  def ep_apply_held(self):
    for ex in self._exchanges():
      if ex.members:
        ex.members[0].apply_held()

  def check_exchange(self):
    """EmbeddingParallel: raise if a per-peer block of the fixed-capacity exchange overflowed since the last check
    (reads one counter per arena back: call it outside the step loop, e.g. when the loss is logged), or if a prefetched
    batch was not the one looked up.  Every exchange's counters are read and reset before the first error is raised."""
    err = None
    for ex in self._exchanges():
      ex.build()
      try:
        ex.check()
      except _lib.ErError as e:
        err = err or e
    if err is not None:
      raise err

  def sparse_grad_sqnorm(self):
    """sum over the tables of ||IndexedSlices.values||^2 as TF would build them after loss.backward(): the gradient of a
    column's lookup is deduplicated PER COLUMN (embedding_lookup_sparse runs `unique` on its ids), columns that share a
    table are concatenated, not merged (compat/optimizers.py:453-481 l2_loss(grad.values)).  K7 in emit form over
    virtual rows `row + slot * n_rows` produces exactly those per-(column, row) sums; the embedding gradient multiplier
    (model/easy_rec_estimator.py:308-317) is applied first, as optimize_loss does.  Returns a device scalar."""
    total = torch.zeros((), dtype=torch.float32, device=self.device)
    for m, rows, w, outs, seg_ids in self._pending:
      if seg_ids is None and rows.numel() != m.n_seg:
        raise NotImplementedError('gradient_clipping_by_norm: a call whose lookups are not its segments needs seg_ids')
      a = m.arena
      n_l = rows.numel()          # lookups: one per segment for single-valued slots, the lookup capacity for CSR slots
      st = self._clip_state.get(id(m))
      if st is None:
        if a.n_rows * m.n_slots >= 0xFFFFFFFF:
          raise NotImplementedError('gradient_clipping_by_norm: %d rows x %d columns exceed the 32-bit row key' %
                                    (a.n_rows, m.n_slots))
        off = torch.zeros(m.n_seg, dtype=torch.int64)      # per SEGMENT: the virtual-row offset of its column (slot)
        for j, r in enumerate(m.slots_np):
          off[int(r['seg_begin']):int(r['seg_begin']) + int(r['n_seg'])] = j * a.n_rows
        st = dict(off=off.to(self.device), ws=K.bwd_workspace(n_l, self.device, a.dim),
                  ur=torch.empty(n_l, dtype=torch.int64, device=self.device),
                  ug=torch.empty(n_l, a.dim, dtype=torch.float32, device=self.device),
                  nu=torch.zeros(1, dtype=torch.int32, device=self.device),
                  idx=torch.arange(n_l, device=self.device, dtype=torch.int32))
        self._clip_state[id(m)] = st
      # multi-valued slots: every lookup takes the offset of ITS segment's column (the segment ids of the unused tail of
      # the fixed-capacity arrays are undefined: clamped, their rows are -1 anyway)
      off = st['off'] if seg_ids is None else st['off'][seg_ids[:n_l].clamp(0, m.n_seg - 1).long()]
      vr = torch.where(rows < 0, rows, rows + off)
      gbufs = [(o.grad if o.grad is not None else torch.zeros_like(o)).contiguous() for o in outs]
      opt = K.make_opt(_lib.OPT_SGD, 0.0, grad_scale=float(self.emb_grad_mult))
      K.embedding_bwd(None, None, None, a.dim, vr, m.slots_dev, m.n_slots, m.n_seg, gbufs, opt, st['ws'], weights=w,
                      seg_ids=seg_ids, seg_scale=m.seg_scale, uniq_rows=st['ur'], uniq_grads=st['ug'], n_uniq=st['nu'],
                      n_rows=a.n_rows * m.n_slots)
      rowsq = (st['ug'] * st['ug']).sum(dim=1)
      total = total + torch.where(st['idx'] < st['nu'], rowsq, torch.zeros_like(rowsq)).sum()
    return total

  def _rows_buf(self, key, call):
    """persistent output buffer of K1 per row plan (stable address: CUDA graphs, early exchange)."""
    buf = self._rows_bufs.get(key)
    if buf is None:
      buf = torch.empty(call.n_seg, dtype=torch.int64, device=self.device)
      self._rows_bufs[key] = buf
    return buf

  def precompute_rows(self, features):
    """K1 (index hashing / bucketing) of the single-valued slots at the head of the step, ahead of the lookup:
    data-parallel training all-gathers the rows and starts the global dedup sort while the dense forward/backward
    runs.  Returns [(arena dim, ArenaCall, rows, weights)]; the next lookup() reuses them."""
    dense = features.get('dense_fea')
    dense_norm = self.normalize_dense(dense) if dense is not None else None
    out = []
    self._preset_rows = {}
    for dim, subs in self.subcalls.items():
      for sk, sc in subs.items():
        if sc.kind != 'single' or len(subs) != 1:
          continue
        call = sc.call
        key = self._rows_key(sc)
        hit = self._preset_rows.get(key)
        if hit is None:
          cids, w = self._gather_inputs(dim, features.get('sparse_fea'), dense_norm)
          rows = K.bucketize(cids, call.slots_dev, call.n_slots, call.n_seg, rows=self._rows_buf(key, call))
          hit = (rows, w)
          self._preset_rows[key] = hit
        out.append((dim, self.merged[dim], hit[0], hit[1]))
    return out

  def _presort(self):
    """K7's bucket placement needs only the looked-up rows: start it now on a side stream so it runs under the
    dense forward/backward instead of after it (joined in backward_update; captured as a fork/join)."""
    self.placements.clear()
    if not (self._pending and self.presort_enabled and not self.ep and torch.is_grad_enabled() and
            str(self.device).startswith('cuda')):
      return
    if self._side is None:
      self._side = torch.cuda.Stream(device=self.device)
    self._side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(self._side):
      for m, rows, w, outs, seg_ids in self._pending:
        self.placements.presort(rows, m.arena.n_rows, m.arena.dim, m.ws, m.slots_dev, m.n_slots, seg_ids=seg_ids)

  def normalize_dense(self, dense):
    if self.raw_has_range:
      dense = (dense - self.raw_sub) / self.raw_range  # (x - min) / (max - min), input/input.py:638-640
    if self.raw_normalizers:
      # RawFeature.normalizer_fn on the normalised value (input/input.py:642-646), feature by feature
      dense = dense.clone() if not self.raw_has_range else dense
      for name, fn in self.raw_normalizers.items():
        c0, c1 = self.raw_cols[name]
        dense[:, c0:c1] = fn(dense[:, c0:c1])
    return dense

  def prefetch_exchange(self, next_features):
    """EmbeddingParallel: start the id half of the NEXT batch's exchange (K1, K8, id all-to-all) beside the rest of
    this step; the next lookup() promotes it instead of computing it on the critical path.  (The histories' exchanges
    run with their lookup.)"""
    if not self.ep:
      return
    for ex, dim, flat in self._ex_plan:
      ex.prefetch(lambda: self._exchange_inputs(dim, flat, next_features, None, prefetch=True))

  def _exchanges(self):
    seen, out = set(), []
    if self.ep:
      for subs in self.subcalls.values():
        for sc in subs.values():
          if id(sc.sharded.ex) not in seen:
            seen.add(id(sc.sharded.ex))
            out.append(sc.sharded.ex)
    return out

  def join_prefetch(self):
    for ex in self._exchanges():
      ex.join_prefetch()

  def drop_prefetch(self):
    """forget any prefetched id exchange: the next lookup() computes its own (called after a graph replay, whose
    captured promote / prefetch pair does not go through the Python-side flag)"""
    for ex in self._exchanges():
      ex._have_next = False

  def prefetch_ready(self):
    """True when every exchange holds a prefetched id exchange for the next lookup()."""
    ex = self._exchanges()
    return bool(ex) and all(e._have_next for e in ex)

  def _gather_inputs(self, dim, ids, dense_norm, ids_buf=None, want_w=True):
    """ids int64 [n_id*B] feature-major -> (ids, weights) in the single-valued call's slot order.

    Two strided copies per arena (ids of the id slots, normalised values of the raw slots);
    slots that are already in packed order are used in place."""
    call = self.calls[dim]
    if call.identity_ids:
      return ids, None
    B = self.batch_size
    S = call.n_slots
    out_ids = self.static_ids[dim] if ids_buf is None else ids_buf
    out_w = self.static_w[dim] if want_w else None
    plan = self._gather_plan.get(dim)
    if plan is None:
      src = call.sources
      id_pos = [i for i, (k, _) in enumerate(src) if k == 'id']
      id_src = [j for k, j in src if k == 'id']
      raw_pos = [i for i, (k, _) in enumerate(src) if k == 'raw']
      raw_src = [j for k, j in src if k == 'raw']

      def as_slice(v):
        return (v[0], v[-1] + 1) if v and v == list(range(v[0], v[0] + len(v))) else None

      plan = dict(id_pos=as_slice(id_pos), id_src=as_slice(id_src), raw_pos=as_slice(raw_pos),
                  raw_src=as_slice(raw_src),
                  id_pos_t=torch.tensor(id_pos, dtype=torch.int64, device=self.device),
                  id_src_t=torch.tensor(id_src, dtype=torch.int64, device=self.device),
                  raw_pos_t=torch.tensor(raw_pos, dtype=torch.int64, device=self.device),
                  raw_src_t=torch.tensor(raw_src, dtype=torch.int64, device=self.device))
      self._gather_plan[dim] = plan
    o2 = out_ids.view(S, B)
    if plan['id_pos_t'].numel():
      ids2 = ids.view(len(self.sparse_names), B)
      if plan['id_pos'] and plan['id_src']:
        o2[plan['id_pos'][0]:plan['id_pos'][1]].copy_(ids2[plan['id_src'][0]:plan['id_src'][1]])
      else:
        o2.index_copy_(0, plan['id_pos_t'], ids2.index_select(0, plan['id_src_t']))
    if out_w is not None and plan['raw_pos_t'].numel():
      w2 = out_w.view(S, B)
      dt = dense_norm.t()
      if plan['raw_pos'] and plan['raw_src']:
        w2[plan['raw_pos'][0]:plan['raw_pos'][1]].copy_(dt[plan['raw_src'][0]:plan['raw_src'][1]])
      else:
        w2.index_copy_(0, plan['raw_pos_t'], dt.index_select(0, plan['raw_src_t']))
    return out_ids, out_w

  # ------------------------------------------------------------------
  @staticmethod
  def _rows_key(sc):
    """what decides the rows a launch looks up: its slots' bucket rules and offsets and where its ids come from (a
    multi-valued launch: its kind, its features and its lookup capacity too, and which of its slots K1 prunes by
    weight - a weighted mean / sqrtn lookup whose weight is not > 0 reads no row, a sum lookup keeps it, so a mean
    TagFeature in a deep group and its sum twin in a wide group look up different rows)"""
    key = getattr(sc, 'rows_key', None)
    if key is None:
      call = sc.call
      key = (tuple((int(r['num_buckets']), int(r['row_offset']), int(r['seg_begin']), int(r['n_seg']),
                    int(r['bucket_mode']), int(r['shard_n'])) for r in call.slots_np),
             tuple(call.sources) if sc.kind == 'single' else (sc.kind, call.max_lookups) + tuple(
                 src for _, _, _, src in sc.items) + tuple(
                 (int(r['combiner']) & 0xf) != _lib.COMBINER_SUM for r in call.slots_np))
      sc.rows_key = key
    return key

  def _exchange_inputs(self, dim, flat, features, dense_norm, prefetch=False):
    """[LaunchInput] of an exchange's launches `flat` (those of its first arena, `dim`) for the batch `features`, and
    the pooling inputs of each: [(weights, row_ptr, seg_ids)]"""
    from easyrec_b200.sharded import LaunchInput
    parts, pool = [], []
    for sc in flat:
      if sc.kind == 'single':
        if prefetch:
          buf = self._next_ids.get(dim)
          if buf is None:
            buf = self._next_ids[dim] = torch.zeros_like(self.static_ids[dim])
          cids, w = self._gather_inputs(dim, features.get('sparse_fea'), None, ids_buf=buf, want_w=False)
        else:
          cids, w = self._gather_inputs(dim, features.get('sparse_fea'), dense_norm)
        parts.append(LaunchInput(cids))
        pool.append((w, None, None))
        continue
      ids_cap, lens, weights = self._csr_inputs(sc, features)
      row_ptr, seg_ids = K.csr_from_lens(lens.contiguous(), sc.call.max_lookups)
      parts.append(LaunchInput(ids_cap, seg_ids, row_ptr, weights))
      pool.append((weights, row_ptr, seg_ids))
    return parts if prefetch else (parts, pool)

  def _run_subcall(self, dim, sk, sc, features, dense_norm):
    """K1 + K2 of one uniform launch; returns (rows, weights, row_ptr, seg_ids, outs)."""
    call = sc.call
    B = self.batch_size
    if self.ep and sc.kind != 'seq':
      # row-sharded tables: the first launch of an exchange this step runs K1 of all its launches, K8 and the
      # all-to-alls for every arena of its row plan; each launch then pools the received rows by its own plan
      ex = sc.sharded.ex
      hit = self._ex_inputs.get(id(ex))
      if hit is None:
        _, dim0, flat = next(e for e in self._ex_plan if e[0] is ex)
        parts, hit = self._exchange_inputs(dim0, flat, features, dense_norm)
        ex.build()
        ex.lookup(parts)
        self._ex_inputs[id(ex)] = hit
      w, row_ptr, seg_ids = hit[ex.launches.index(sc.sharded.ref)]
      outs = call.alloc_outputs()
      rows = sc.sharded.forward(None, w, outs, row_ptr=row_ptr, seg_ids=seg_ids)
      for o in outs:
        o.requires_grad_(True)
      return rows, w, row_ptr, seg_ids, outs
    if sc.kind == 'single':
      key = self._rows_key(sc)   # arenas with the same row plan (wide dim-1 next to the deep tables) share K1's rows
      hit = self._rows_cache.get(key)
      if hit is None:
        cids, w = self._gather_inputs(dim, features.get('sparse_fea'), dense_norm)
        rows = K.bucketize(cids, call.slots_dev, call.n_slots, call.n_seg, rows=self._rows_buf(key, call))
        self._rows_cache[key] = (rows, w)
      else:
        rows, w = hit
      outs = E.fused_lookup(call, rows, weights=w)
      return rows, w, None, None, outs
    if sc.kind == 'seq' and self.ep:
      # row-sharded tables: er_bucketize_seq (owner, local row; -1 on padded steps) -> K8 -> all-to-alls -> every
      # received row written to its own step's row of the [B*T, sum D] matrix
      T = sc.n_seg_per_slot // B
      seqs = [features['seq_fea'][fname] for _, fname, _, _ in sc.items]
      ids = torch.cat([i.reshape(-1) for i, _ in seqs]) if len(seqs) > 1 else seqs[0][0].reshape(-1)
      lens = torch.cat([n.reshape(-1) for _, n in seqs]) if len(seqs) > 1 else seqs[0][1].reshape(-1)
      outs = call.alloc_outputs()
      rows = sc.sharded.forward(ids.contiguous(), None, outs, lens=lens.to(torch.int32).contiguous())
      for o in outs:
        o.requires_grad_(True)
      return rows, None, None, None, outs
    if sc.kind == 'seq':
      T = sc.n_seg_per_slot // B
      ids_list, pad_list = [], []
      for _, fname, _, _ in sc.items:
        ids, lens = features['seq_fea'][fname]
        ids_list.append(ids.reshape(-1))
        pos = self._pos.get(T)
        if pos is None:
          pos = torch.arange(T, device=self.device, dtype=torch.int32)[None, :]
          self._pos[T] = pos
        pad_list.append((pos >= lens[:, None]).reshape(-1))
      ids = ids_list[0] if len(ids_list) == 1 else torch.cat(ids_list)
      pad = pad_list[0] if len(pad_list) == 1 else torch.cat(pad_list)
      rows = K.bucketize(ids.contiguous(), call.slots_dev, call.n_slots, call.n_seg)
      rows.masked_fill_(pad, -1)   # positions >= seq_len: empty segment -> zero vector
      outs = E.fused_lookup(call, rows)
      return rows, None, None, None, outs
    # tag: CSR
    cap = call.max_lookups
    ids_cap, lens, weights = self._csr_inputs(sc, features)
    row_ptr, seg_ids = K.csr_from_lens(lens.contiguous(), cap)
    rows = torch.full((cap,), -1, dtype=torch.int64, device=self.device)
    K.bucketize(ids_cap, call.slots_dev, call.n_slots, call.n_seg, seg_ids=seg_ids, row_ptr=row_ptr,
                rows=rows, **K.k1_weight_args(ids_cap, weights))
    outs = E.fused_lookup(call, rows, weights=weights, row_ptr=row_ptr)
    return rows, weights, row_ptr, seg_ids, outs

  def _csr_inputs(self, sc, features):
    """a multi-valued launch's ids padded to its lookup capacity, its lengths, and its weights (None: all 1)"""
    ids_list, lens_list, w_list = [], [], []
    any_w = False
    for _, fname, _, _ in sc.items:
      if sc.kind == 'mseq':
        # (values of every step back to back, steps per sample, values per (sample, step) - 0 beyond the length)
        ids, _, lens = features['seq_fea'][fname]
        w = None
      else:
        ids, lens, w = features['tag_fea'][fname]
      ids_list.append(ids)
      lens_list.append(lens)
      w_list.append(w)
      any_w = any_w or (w is not None)
    ids = torch.cat(ids_list) if len(ids_list) > 1 else ids_list[0]
    lens = torch.cat(lens_list) if len(lens_list) > 1 else lens_list[0]
    L = ids.numel()
    cap = sc.call.max_lookups
    assert L <= cap, 'tag lookups %d exceed max_tag_lookups %d' % (L, cap)
    weights = None
    if any_w:
      weights = torch.ones(cap, dtype=torch.float32, device=self.device)
      off = 0
      for i_, w in zip(ids_list, w_list):
        if w is not None:
          weights[off:off + i_.numel()].copy_(w)
        off += i_.numel()
    ids_cap = torch.zeros(cap, dtype=torch.int64, device=self.device)
    ids_cap[:L].copy_(ids)
    return ids_cap, lens, weights

  def has_group(self, group_name):
    return group_name in self.group_layout or group_name in self.seq_layout

  def __call__(self, features, group_name, is_combine=True, is_dict=False):
    """The reference's call form (layers/input_layer.py:245-278; sequence groups: layers/seq_input_layer.py:34-124):

      is_combine=True : (concat [B, sum D] in feature_group config order, [per-feature [B, D] ...][, {feature name: tensor}])
      is_combine=False: (seq_features [(emb [B, T, D], len [B]) ...], plain concat, plain per-feature list)
      a seq_att group : {'key', 'hist_seq_emb', 'hist_seq_len'} (SeqInputLayer)

    Every group of one `features` dict comes out of ONE fused lookup per arena: the first call for a batch runs it, the
    calls for the other groups of the same batch (same dict object) read its outputs."""
    if not self.has_group(group_name):
      raise AssertionError('invalid group_name[%s], list: %s' % (group_name, ','.join(
          list(self.group_layout) + list(self.seq_layout))))
    if getattr(self, '_last_features', None) is not features:
      self._last_groups = self.lookup(features)
      self._last_features = features
    if group_name in self.seq_layout:
      return self.seq_outputs[group_name]
    if group_name in self.seq_group_layout:
      raise NotImplementedError('feature group %s is read by output_seq_and_normal_feature blocks: lookup() returns its '
                                '(seq, seq_len, target, plain features)' % group_name)
    concat, per_feature = self._last_groups[group_name]
    if not is_combine:
      return [], concat, per_feature
    if is_dict:
      names = [e.name for e in self.group_layout[group_name]]
      return concat, per_feature, dict(zip(names, per_feature))
    return concat, per_feature

  def lookup(self, features):
    """Runs K1 + K2 for every arena; returns {group: (concat, [per-feature views])} and fills
    self.seq_outputs {seq group: {key, hist_seq_emb, hist_seq_len}}."""
    dense = features.get('dense_fea')
    dense_norm = self.normalize_dense(dense) if dense is not None else None
    self._rows_cache = dict(self._preset_rows)   # K1 results computed ahead of the step (precompute_rows)
    self._preset_rows = {}
    self._ex_inputs = {}   # EmbeddingParallel: exchange -> its launches' pooling inputs, once it ran for this batch
    self._pending = []
    outs_by_key = {}
    for dim, subs in self.subcalls.items():
      parts = []
      for sk, sc in subs.items():
        rows, w, row_ptr, seg_ids, outs = self._run_subcall(dim, sk, sc, features, dense_norm)
        parts.append((sc, rows, w, seg_ids, outs))
        for (d, k), (skk, j) in self.out_index.items():
          if d == dim and skk == sk:
            outs_by_key[(dim, k)] = outs[j]
      self._queue_update(self.merged[dim], parts)
    self._presort()
    self.seq_outputs = {}
    B = self.batch_size
    for sname, lay in self.seq_layout.items():
      keys = [outs_by_key[(e.dim, e.out_key)][:, e.col:e.col + e.dim] for e in lay['key']]
      hists = [outs_by_key[(e.dim, e.out_key)][:, e.col:e.col + e.dim].reshape(B, lay['T'], e.dim) for e in lay['hist']]
      lens = features['seq_fea'][lay['hist'][0].name][1]
      self.seq_outputs[sname] = dict(
          key=keys[0] if len(keys) == 1 else torch.cat(keys, dim=-1),
          hist_seq_emb=hists[0] if len(hists) == 1 else torch.cat(hists, dim=-1),
          hist_seq_len=lens)
    return {gname: self._group_outputs(gname, features, outs_by_key, dense_norm) for gname in self.group_layout}

  def _queue_update(self, m, parts):
    """the Pending K7 update(s) of one arena's launches `parts` [(sub-call, rows, weights, seg_ids, outs)]: several
    launches are packed into the arena's MergedCall"""
    if self.ep and len(parts) > 1:
      # row-sharded tables: every launch adds its gradient sums to its exchange; the exchange's last launch runs the
      # owner-side updates
      for sc, rows, w, seg_ids, outs in parts:
        self._pending.append(Pending(sc, rows, w, outs, seg_ids))
    elif len(parts) == 1:
      sc, rows, w, seg_ids, outs = parts[0]
      self._pending.append(Pending(m, rows, w, outs, seg_ids))
    else:
      all_outs = []
      any_w = any(p[2] is not None for p in parts)
      if any_w and m.weights is None:
        m.weights = torch.ones(m.max_lookups, dtype=torch.float32, device=self.device)
      for si, (sc, rows, w, seg_ids, outs) in enumerate(parts):
        lo = m.sub_lookup_off[si]
        n = rows.numel()
        m.rows[lo:lo + n].copy_(rows)
        if any_w:
          if w is not None:
            m.weights[lo:lo + n].copy_(w)
          else:
            m.weights[lo:lo + n].fill_(1.0)
        if m.has_csr:
          if seg_ids is not None:
            m.seg_ids[lo:lo + n].copy_(seg_ids[:n] + m.sub_seg_off[si])
          else:
            m.seg_ids[lo:lo + n].copy_(
                torch.arange(m.sub_seg_off[si], m.sub_seg_off[si] + n, device=self.device,
                             dtype=torch.int32))
        if m.needs_scale:
          so = m.sub_seg_off[si]
          if sc.call.seg_scale is not None:
            m.seg_scale[so:so + sc.call.n_seg].copy_(sc.call.seg_scale)
        all_outs.extend(outs)
      self._pending.append(Pending(m, m.rows, m.weights if any_w else None, all_outs,
                                   m.seg_ids if m.has_csr else None))

  def _group_outputs(self, gname, features, outs_by_key, dense_norm):
    """lookup()'s value for one feature group: (concat, [per-feature]), or (seq, seq_len, concat, [per-feature]) for a
    group read by output_seq_and_normal_feature"""
    B = self.batch_size
    layout = self.group_layout[gname]
    per_feature, mats, kinds, reg = [], {}, [], None
    for e in layout:
      if e.kind == 'dense':
        c0, c1 = self.raw_cols[e.name]
        v = dense_norm[:, c0:c1]
      elif e.kind == 'seqc':
        # sequence_combiner { attention } (input_layer.py:323-339): logits = dense(seq, 1, no bias), positions beyond
        # the length masked with -2^32 + 1, softmax over the steps, weighted sum of the step embeddings
        from easyrec_b200 import interactions as I
        mat = outs_by_key[(e.dim, e.out_key)]
        T = self.features[e.name].seq_len
        seq = mat[:, e.col:e.col + e.width].reshape(B, T, e.width).contiguous()
        scores = self.attention_modules[e.out_key](seq.reshape(B * T, e.width)).reshape(B, T)
        v = I.din_pool(scores.contiguous(), seq, features['seq_fea'][e.name][1])
        reg = (reg or []) + [seq]           # embedding_reg_lst takes the un-pooled sequence (input_layer.py:316)
      elif e.kind == 'att':
        # target attention over the group's sequence_features (sequence_feature_layer.py:123-189): softmax of the
        # masked attention-MLP scores over the history, [attended history | key] (need_key_feature)
        from easyrec_b200 import interactions as I
        so = self.seq_outputs[e.out_key]
        key = so['key'].contiguous()
        att = I.din_attention(key, so['hist_seq_emb'].contiguous(), so['hist_seq_len'], self.attention_modules[e.out_key])
        v = torch.cat([att, key], dim=1) if e.need_key else att
        reg = (reg or []) + [so['hist_seq_emb']]
      else:
        mat = outs_by_key[(e.dim, e.out_key)]
        mats[(e.dim, e.out_key)] = mat
        v = mat[:, e.col:e.col + e.width]
      per_feature.append(v)
      kinds.append(e.kind)
    if not layout:   # (only sequence features, read by output_seq_and_normal_feature)
      concat = None
    elif len(mats) == 1 and all(k == 'emb' for k in kinds):
      mat = next(iter(mats.values()))
      width = self.group_width(gname)
      concat = mat if mat.shape[1] == width else mat[:, :width]
    else:
      concat = torch.cat(per_feature, dim=1)
    if reg is not None:
      # the embedding regulariser covers what was LOOKED UP (the group's columns and the histories,
      # input_layer.py:369-375, sequence_feature_layer.py:215-217), not the attended vectors appended to the concat
      concat._er_reg = [v for v, k in zip(per_feature, kinds) if k == 'emb'] + reg
    order = self.seqc_order.get(gname)
    if order and len(order) > 1:
      # the per-feature list keeps the sequence-combiner features in config order (the concat has them by name)
      by_name = {e.name: v for e, v in zip(layout, per_feature) if e.kind == 'seqc'}
      per_feature = [v for e, v in zip(layout, per_feature) if e.kind != 'seqc'] + [by_name[n] for n in order]
    if gname in self.seq_group_layout:
      seq, seq_len = self._seq_group_tensors(gname, features, outs_by_key)
      # the embedding regulariser covers the un-pooled sequence embeddings and the plain embedding columns
      # (input_layer.py:117-151, 176-191)
      seq._er_reg = [seq] + [v for v, k in zip(per_feature, kinds) if k == 'emb']
      return seq, seq_len, concat, per_feature
    return concat, per_feature

  def _seq_group_tensors(self, gname, features, outs_by_key):
    """EnhancedInputLayer.build (layers/common_layers.py:114-127) with concat_seq_feature: the group's sequence
    features side by side on the last axis, [B, T, sum D], and the lengths of the FIRST of them."""
    lay = self.seq_group_layout[gname]
    B, T = self.batch_size, lay['T']
    parts = []   # [matrix, first column, width]: neighbouring columns of one matrix are one view
    for e in lay['seq']:
      mat = outs_by_key[(e.dim, e.out_key)]
      if parts and parts[-1][0] is mat and parts[-1][1] + parts[-1][2] == e.col:
        parts[-1][2] += e.dim
      else:
        parts.append([mat, e.col, e.dim])
    views = [m[:, c:c + w].reshape(B, T, w) for m, c, w in parts]
    seq = views[0] if len(views) == 1 else torch.cat(views, dim=-1)
    return seq, features['seq_fea'][lay['seq'][0].name][1]
