"""GPU: the gradient every table row and attention weight receives through InputLayer, against a float64 restatement.

What is checked is the backward of the glue between the kernels: the column slices and [B, T, D] views of the pooled
matrices, the concats and the per-feature list (sequence-combiner features reordered), the attention paths
(`sequence_combiner { attention }`, in-group target attention with and without the key), the embedding regulariser's
choice of tensors and the merged K7 launch of an arena (row copies, ones-filled weights, segment offsets, seg_scale).

Observing G.  The model is built from pipeline-config text with momentum_optimizer at momentum 0 (plain SGD) and the
step runs at lr = 1: after lookup() and loss.backward() every arena is zeroed and backward_update() writes 0 - G into
every touched row exactly, so G = -weight and untouched rows must stay exactly 0.  Attention parameters are compared
through their .grad.

The loss is  sum_g <R_g, concat_g> + sum_g sum_i <S_gi, per_feature_gi> + sum_s <Q_s, sequence outputs> + the model's
embedding regulariser, with R / S / Q small integers.  Tables hold multiples of 1/16 and lookup weights are powers of
two, so on the linear paths (ids, sum-pooled tags, raw-value weights, shared tables, un-pooled sequences) every
summation order is exact and G must equal the float64 reference bit for bit.  Where mean / sqrtn pooling or a softmax
takes part, the error against float64 may be no worse than a float32 run of the same restatement (test_gpu_dense.py's
rule: a small factor at the 99.9th percentile and at the maximum).

The reference is restated from the config alone: table names by the reference's variable scopes, bucket rows from
oracle.bucketize, `table64[rows]` on a float64 leaf copy of each arena, the sum / mean / sqrtn combiners with the
reference's pruning (rows < 0 dropped; weights <= 0 dropped unless the combiner is sum), the attention combiner and
target attention in plain torch.

The same cases run on the CPU with tests/host_doubles.py in place of the kernels, which rehearses the restatement and the
glue without a device; the restatement's forward is also held against the attention-combiner and DIN restatements of
test_act_metrics_host.py and test_gpu_models.py.

Measured on an H100 80GB HBM3 (700 W power limit): the 15 GPU cases take about 19 s and peak at 0.03 GiB of reserved
device memory.
"""
import collections

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, builder
from easyrec_b200.config import config_util
from oracle import oracle as O

DEV = 'cuda:0'
PAD = -2.0 ** 32 + 1
LAMBDA = 0.5          # embedding_regularization: a power of two keeps the regulariser's gradient exact


# ---- configs ------------------------------------------------------------------------------------------------------
def head(input_type='DummyInput', fields=''):
  return '''
model_dir: "/tmp/x"
train_config { optimizer_config { momentum_optimizer { learning_rate { constant_learning_rate { learning_rate: 1.0 } }
                                                    momentum_optimizer_value: 0.0 } } }
data_config { batch_size: 64 input_type: %s label_fields: "clk" input_fields { input_name: "clk" input_type: FLOAT } %s }
''' % (input_type, fields)


def multi_tower(groups, din=()):
  towers = ' '.join('towers { input: "%s" dnn { hidden_units: [4] } }' % g for g in groups)
  dins = ' '.join('din_towers { input: "%s" dnn { hidden_units: [4, 1] use_bn: false } }' % g for g in din)
  return 'multi_tower { %s %s final_dnn { hidden_units: [4] } }' % (towers, dins)


# 1-3: id features of every bucket rule, a shared embedding_name, raw-value weights, a bucketized raw feature, a dense
# raw column, a sum tag; one feature in two deep groups (the same table) and in the wide group (the dim-1 arena)
IDS = '''
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 8 hash_bucket_size: 500 }
  features { input_names: "a" feature_type: IdFeature embedding_dim: 8 num_buckets: 10 }
  features { input_names: "s" feature_type: IdFeature embedding_dim: 8 hash_bucket_size: 300 }
  features { input_names: "c1" feature_type: IdFeature embedding_dim: 8 num_buckets: 50 embedding_name: "shared" }
  features { input_names: "c2" feature_type: IdFeature embedding_dim: 8 num_buckets: 50 embedding_name: "shared" }
  features { input_names: "p" feature_type: RawFeature embedding_dim: 8 min_val: 0.0 max_val: 1.0 }
  features { input_names: "q" feature_type: RawFeature embedding_dim: 8 raw_input_dim: 3 min_val: 0.0 max_val: 1.0 }
  features { input_names: "bk" feature_type: RawFeature embedding_dim: 4 boundaries: [0.1, 0.5, 0.9] }
  features { input_names: "d" feature_type: RawFeature min_val: 0.0 max_val: 1.0 }
  features { input_names: "t" feature_type: TagFeature embedding_dim: 8 num_buckets: 40 combiner: "sum" }
}
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "deep1" feature_names: ["u", "a", "s", "c1", "c2", "p", "q", "bk", "d", "t"] wide_deep: DEEP }
  feature_groups { group_name: "deep2" feature_names: ["a", "u"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["u", "s", "t", "p"] wide_deep: WIDE }
  %s
  embedding_regularization: %r }
''' % (multi_tower(['deep1', 'deep2', 'wide']), LAMBDA)
IDS_FIELDS = 'input_fields { input_name: "s" input_type: STRING }'

# 4-5: tags of every combiner with and without kv weights next to a single-valued id feature: one arena, one merged
# K7 launch whose single-valued half has no weights
TAGS = '''
feature_config {
  features { input_names: "i" feature_type: IdFeature embedding_dim: 8 num_buckets: 100 embedding_name: "tt" }
  features { input_names: "tm" feature_type: TagFeature embedding_dim: 8 num_buckets: 100 combiner: "mean" embedding_name: "tt" }
  features { input_names: "tq" feature_type: TagFeature embedding_dim: 8 num_buckets: 60 combiner: "sqrtn" }
  features { input_names: "ts" feature_type: TagFeature embedding_dim: 8 num_buckets: 60 combiner: "sum" }
  features { input_names: "tn" feature_type: TagFeature embedding_dim: 8 num_buckets: 100 combiner: "mean" embedding_name: "tt" }
}
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "g" feature_names: ["tm", "i", "tq", "ts", "tn"] wide_deep: DEEP }
  feature_groups { group_name: "w" feature_names: ["tm", "i", "tq"] wide_deep: WIDE }
  %s
  embedding_regularization: %r }
''' % (multi_tower(['g', 'w']), LAMBDA)

# 6: two attention-combined sequences in a plain group (concat by name, per-feature list in config order)
SEQC = '''
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 8 num_buckets: 30 }
  features { input_names: "zz" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 40 max_seq_len: %d
             embedding_name: "seqtab" sequence_combiner { attention {} } }
  features { input_names: "aa" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 40 max_seq_len: %d
             embedding_name: "seqtab" sequence_combiner { attention {} } }
}
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "g" feature_names: ["zz", "u", "aa"] wide_deep: DEEP }
  %s
  embedding_regularization: %r }
'''

# 7: target attention inside a group: the key reuses the group's column and shares its table with the history; two
# histories side by side; a second attention without the key
DIN_GROUP = '''
feature_config {
  features { input_names: "item" feature_type: IdFeature embedding_dim: 8 num_buckets: 200 embedding_name: "items" }
  features { input_names: "cate" feature_type: IdFeature embedding_dim: 4 num_buckets: 20 }
  features { input_names: "h_item" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 200 max_seq_len: %d
             embedding_name: "items" }
  features { input_names: "h_cate" feature_type: SequenceFeature embedding_dim: 4 num_buckets: 20 max_seq_len: %d }
  features { input_names: "h_two" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 200 max_seq_len: %d }
}
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "g" feature_names: ["item", "cate"] wide_deep: DEEP
    sequence_features { group_name: "s1" seq_att_map { key: "item" key: "cate" hist_seq: "h_item" hist_seq: "h_cate" }
                        need_key_feature: true seq_dnn { hidden_units: [8, 1] use_bn: false } }
    sequence_features { group_name: "s2" seq_att_map { key: "item" hist_seq: "h_two" }
                        need_key_feature: false seq_dnn { hidden_units: [8, 1] use_bn: false } } }
  %s
  embedding_regularization: %r }
'''

# 7-8: seq_att_groups (the attention runs in the model: InputLayer hands out key / history / length); a multi-valued
# history (seq_multi_sep) beside a plain one, the key sharing its table with a history
SEQ_ATT = '''
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 8 num_buckets: 30 }
  features { input_names: "item" feature_type: IdFeature embedding_dim: 8 num_buckets: 200 embedding_name: "items" }
  features { input_names: "cate" feature_type: IdFeature embedding_dim: 8 num_buckets: 20 }
  features { input_names: "h_item" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 200 max_seq_len: %d
             embedding_name: "items" }
  features { input_names: "h_cate" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 20 max_seq_len: %d
             seq_multi_sep: "#" combiner: "%s" }
}
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "u" feature_names: ["u"] wide_deep: DEEP }
  seq_att_groups { group_name: "din" seq_att_map { key: "item" hist_seq: "h_item" }
                   seq_att_map { key: "cate" hist_seq: "h_cate" } }
  %s
  embedding_regularization: %r }
'''

# 9: a group read by a backbone input_layer block with output_seq_and_normal_feature: [B, T, sum D] over two widths
SEQ_OUT = '''
feature_config {
  features { input_names: "uid" feature_type: IdFeature embedding_dim: 8 num_buckets: 50 }
  features { input_names: "item" feature_type: IdFeature embedding_dim: 8 num_buckets: 200 }
  features { input_names: "cate" feature_type: IdFeature embedding_dim: 4 num_buckets: 20 }
  features { input_names: "h_item" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 200 max_seq_len: %d }
  features { input_names: "h_cate" feature_type: SequenceFeature embedding_dim: 4 num_buckets: 20 max_seq_len: %d }
}
model_config { model_class: "RankModel"
  feature_groups { group_name: "user" feature_names: ["uid"] wide_deep: DEEP }
  feature_groups { group_name: "seq" feature_names: ["item", "cate", "h_item", "h_cate"] wide_deep: DEEP }
  backbone {
    blocks { name: "user" inputs { feature_group_name: "user" } keras_layer { class_name: "MLP" mlp { hidden_units: [4] } } }
    blocks { name: "seq_input" inputs { feature_group_name: "seq" } input_layer { output_seq_and_normal_feature: true } }
    blocks { name: "din" inputs { block_name: "seq_input" } keras_layer { class_name: "DIN" din {
      attention_dnn { hidden_units: [4, 1] } need_target_feature: true } } }
    concat_blocks: ["user", "din"]
    top_mlp { hidden_units: [4] } }
  embedding_regularization: %r }
'''


# ---- the reference: restated from the config ----------------------------------------------------------------------
def _name(fc):
  return fc.feature_name if fc.HasField('feature_name') else fc.input_names[0]


def _ftype(fc):
  return builder.ftype_name(fc)


class Spec(object):
  """how the reference reads one feature: kind, width, bucket rule (oracle.bucketize mode, bucket count), combiner"""

  def __init__(self, fc, field_types, packed_mod):
    self.name, self.fc, self.k = _name(fc), fc, 1
    t = _ftype(fc)
    self.dim = int(fc.embedding_dim)
    self.combiner = fc.combiner or 'sum'
    self.bounds = list(fc.boundaries)
    if t == 'RawFeature':
      self.kind = 'bucketized' if self.bounds else 'raw'
      self.k, self.T = int(fc.raw_input_dim), 1
      self.mode, self.nb = (2, len(self.bounds) + 1) if self.bounds else (3, self.k)
      return
    self.kind = {'IdFeature': 'id', 'TagFeature': 'tag', 'SequenceFeature': 'seq'}[t]
    if fc.HasField('seq_multi_sep'):
      self.kind = 'mseq'
    if fc.hash_bucket_size > 0:
      # a STRING field arrives hashed by the reader: its bucket is taken as it is (-1 = no value)
      self.mode = 2 if field_types.get(fc.input_names[0]) == 'STRING' else 0
      self.nb = int(fc.hash_bucket_size)
    else:
      self.mode, self.nb = (1 if packed_mod else 2), int(fc.num_buckets)
    self.T = int(fc.max_seq_len) if self.kind in ('seq', 'mseq') else 1
    self.seqc = fc.HasField('sequence_combiner')


def _rows(ids, spec):
  r, _ = O.bucketize(np.asarray(ids, np.int64).reshape(-1), spec.mode, spec.nb, 0)
  return r.reshape(np.asarray(ids).shape)


class Reference(object):
  """The outputs of every group, in dtype `dt`, from float64 leaf copies of the arenas (`leaves`: dim -> [n_rows, dim])
  and copies of the attention parameters.  `touched[dim]` marks the rows a lookup reads."""

  def __init__(self, cfg, il, model, feats, weights, dt):
    self.il, self.dt, self.feats = il, dt, feats
    self.B = il.batch_size
    mc = cfg.model_config
    ftypes = builder.input_field_types(cfg)
    packed = builder.input_type_name(cfg).startswith('Parquet')
    self.specs = collections.OrderedDict((_name(fc), Spec(fc, ftypes, packed))
                                         for fc in config_util.get_feature_configs(cfg))
    self.leaves = {d: w.to(dt).clone().requires_grad_(True) for d, w in weights.items()}
    self.touched = {d: torch.zeros(w.shape[0], dtype=torch.bool) for d, w in weights.items()}
    self.att = {k: [p.detach().cpu().to(dt).clone().requires_grad_(True) for p in m.parameters() if p.requires_grad]
                for k, m in il.attention_modules.items()}
    # packed inputs: single-valued ids (id features and bucketized raw values) and raw values in config order
    single = [n for n, s in self.specs.items() if s.kind == 'id' or (s.kind == 'bucketized' and s.k == 1)]
    ids = feats['sparse_fea'].cpu().numpy().reshape(len(single), self.B) if single else None
    self.ids = {n: ids[i] for i, n in enumerate(single)}
    raw = [n for n, s in self.specs.items() if s.kind == 'raw']
    dense = feats['dense_fea'].cpu().to(dt) if raw else None
    self.raw, c = {}, 0
    for n in raw:
      s = self.specs[n]
      x = dense[:, c:c + s.k]
      if s.fc.max_val > s.fc.min_val:
        x = (x - s.fc.min_val) / (s.fc.max_val - s.fc.min_val)
      self.raw[n] = x
      c += s.k
    self.wide_dim = 1
    self.groups, self.seq_outputs, self.reg = collections.OrderedDict(), collections.OrderedDict(), []
    seq_groups = {g: True for g in getattr(il, 'seq_group_layout', {})}
    for g in mc.feature_groups:
      self.groups[g.group_name] = self._group(g, g.group_name in seq_groups)
    for sg in mc.seq_att_groups:
      lay = self._seq_att(sg.group_name, [(list(m.key), list(m.hist_seq)) for m in sg.seq_att_map], own=None)
      self.seq_outputs[sg.group_name] = lay
      self.reg += [lay['key'], lay['hist_seq_emb']]

  # -- tables and lookups
  def table(self, name, dim):
    off, n, _ = self.il.arenas[dim].tables[name]
    return off, n

  def gather(self, tname, dim, rows):
    """rows (numpy, any shape, -1 = nothing) -> [..., dim], zero where dropped"""
    off, n = self.table(tname, dim)
    r = torch.from_numpy(np.asarray(rows, np.int64))
    live = r >= 0
    assert bool((r[live] < n).all())
    self.touched[dim][(r[live] + off)] = True
    v = self.leaves[dim][torch.where(live, r, torch.zeros_like(r)) + off]
    return v * live[..., None].to(self.dt)

  def pooled(self, spec, tname, dim, ids, lens, w, combiner):
    """safe_embedding_lookup_sparse over CSR lookups: rows < 0 pruned, weights <= 0 pruned unless `combiner` is sum"""
    rows = _rows(ids, spec)
    lens = np.asarray(lens, np.int64)
    seg = np.repeat(np.arange(lens.size), lens)
    wt = torch.ones(len(rows), dtype=self.dt) if w is None else torch.from_numpy(np.asarray(w, np.float32)).to(self.dt)
    keep = rows >= 0
    if combiner != 'sum':
      keep &= (wt.numpy() > 0)
    rows = np.where(keep, rows, -1)
    # a pruned lookup contributes nothing, whatever its weight (a NaN weight of a mean / sqrtn lookup is pruned)
    wt = torch.where(torch.from_numpy(keep), wt, torch.zeros_like(wt))
    e = self.gather(tname, dim, rows) * wt[:, None]
    segt = torch.from_numpy(seg)
    out = torch.zeros(lens.size, dim, dtype=self.dt).index_add(0, segt, e)
    if combiner == 'sum':
      return out
    if combiner == 'mean':
      d = torch.zeros(lens.size, dtype=self.dt).index_add(0, segt, wt)
    else:
      d = torch.sqrt(torch.zeros(lens.size, dtype=self.dt).index_add(0, segt, wt * wt))
    return torch.where(d[:, None] != 0, out / torch.where(d != 0, d, torch.ones_like(d))[:, None], torch.zeros_like(out))

  def lookup(self, name, tname, dim, wide=False):
    """one feature's pooled [B, dim] (plain group) value"""
    s = self.specs[name]
    if s.kind == 'id' or s.kind == 'bucketized':
      return self.gather(tname, dim, _rows(self.ids[name], s))
    if s.kind == 'raw':
      # ids 0 .. k-1 weighted by the normalised values, summed (input/input.py:648-673)
      x = self.raw[name]
      return sum(x[:, j:j + 1] * self.gather(tname, dim, np.full(self.B, j)) for j in range(s.k))
    if s.kind == 'tag':
      ids, lens, w = [None if v is None else v.cpu().numpy() for v in self.feats['tag_fea'][name]]
      return self.pooled(s, tname, dim, ids, lens, w, 'sum' if wide else s.combiner)
    raise AssertionError(name)

  def sequence(self, name, tname, dim):
    """un-pooled [B, T, dim]: steps beyond the length (and multi-valued steps with no value) are zero"""
    s = self.specs[name]
    if s.kind == 'mseq':
      vals, steps, per = [v.cpu().numpy() for v in self.feats['seq_fea'][name]]
      return self.pooled(s, tname, dim, vals, per, None, s.combiner).reshape(self.B, s.T, dim)
    ids, lens = [v.cpu().numpy() for v in self.feats['seq_fea'][name]]
    rows = _rows(ids, s)
    rows = np.where(np.arange(s.T)[None, :] < lens[:, None], rows, -1)
    return self.gather(tname, dim, rows)

  # -- groups
  def _group(self, g, seq_out):
    wide = g.DESCRIPTOR.fields_by_name['wide_deep'].enum_type.values_by_number[g.wide_deep].name == 'WIDE'
    plain, seqc, seq_cols, reg = [], [], [], []
    for n in g.feature_names:
      s = self.specs[n]
      tname = (s.fc.embedding_name or n + '_embedding') + ('_wide' if wide else '')
      dim = self.wide_dim if wide else s.dim
      if s.kind == 'raw' and dim == 0:
        plain.append((n, 'dense', self.raw[n]))
      elif s.kind == 'seq' and seq_out:
        seq_cols.append(self.sequence(n, s.fc.embedding_name or n + '_embedding', s.dim))
      elif s.kind == 'seq':
        # sequence_combiner { attention }: score = seq @ w, masked beyond the length, softmax, weighted sum
        seq = self.sequence(n, s.fc.embedding_name or n + '_embedding', s.dim)
        w = self.att['%s#seqc/%s' % (g.group_name, n)][0]
        lens = self.feats['seq_fea'][n][1].cpu()
        sc = (seq @ w.reshape(-1, 1))[..., 0]
        sc = torch.where(torch.arange(s.T)[None, :] < lens[:, None], sc, torch.full_like(sc, PAD))
        seqc.append((n, (torch.softmax(sc, 1)[:, :, None] * seq).sum(1)))
        reg.append(seq)
      else:
        v = self.lookup(n, tname, dim, wide)
        plain.append((n, 'emb', v))
    cols = [v for _, _, v in plain] + [v for _, v in sorted(seqc, key=lambda t: t[0])]
    per_feature = [v for _, _, v in plain] + [v for _, v in seqc]
    emb = [v for _, k, v in plain if k == 'emb']
    for sf in g.sequence_features:
      own = {n: v for n, k, v in plain if k == 'emb'}
      lay = self._seq_att(g.group_name, [(list(m.key), list(m.hist_seq)) for m in sf.seq_att_map], own=own)
      key, hist, lens = lay['key'], lay['hist_seq_emb'], lay['hist_seq_len']
      att = self.din(key, hist, lens, self.att['%s/%s' % (g.group_name, sf.group_name)])
      v = torch.cat([att, key], 1) if sf.need_key_feature else att
      cols.append(v)
      per_feature.append(v)
      reg.append(hist)
    concat = torch.cat(cols, 1) if cols else None
    if seq_out:
      seq = torch.cat(seq_cols, -1)
      first = [n for n in g.feature_names if self.specs[n].kind == 'seq'][0]
      self.reg += [seq] + emb
      return seq, self.feats['seq_fea'][first][1], concat, per_feature
    # the regulariser sees what was looked up: the embedding columns and the un-pooled sequences
    self.reg += (emb + reg) if reg else [concat]
    return concat, per_feature

  def _seq_att(self, scope, maps, own):
    keys, hists, lens = [], [], None
    for ks, hs in maps:
      for k in ks:
        s = self.specs[k]
        if own is not None and k in own:
          keys.append(own[k])
        else:
          keys.append(self.lookup(k, s.fc.embedding_name or '%s/%s_embedding' % (scope, k), s.dim))
      for h in hs:
        s = self.specs[h]
        hists.append(self.sequence(h, s.fc.embedding_name or '%s/%s_embedding' % (scope, h), s.dim))
        if lens is None:
          lens = self.feats['seq_fea'][h][1]
    return dict(key=torch.cat(keys, -1), hist_seq_emb=torch.cat(hists, -1), hist_seq_len=lens)

  def din(self, key, hist, lens, params):
    """target attention (layers/sequence_feature_layer.py): MLP over [q, k, q - k, q * k], masked softmax, sum"""
    B, T, D = hist.shape
    q = key[:, None, :].expand(B, T, D)
    x = torch.cat([q, hist, q - hist, q * hist], -1).reshape(B * T, 4 * D)
    n = len(params) // 2
    for i in range(n):
      x = x @ params[2 * i] + params[2 * i + 1]
      if i + 1 < n:
        x = torch.relu(x)
    sc = x.reshape(B, T)
    mask = torch.arange(T)[None, :] < lens.cpu()[:, None]
    sc = torch.where(mask, sc, torch.full_like(sc, PAD))
    return (torch.softmax(sc, 1)[:, :, None] * hist).sum(1)


# ---- the loss: the same weights on both sides ---------------------------------------------------------------------
class Weights(object):
  """small-integer weights, one tensor per output, fixed by the output's name"""

  def __init__(self, seed):
    self.seed, self.w = seed, {}

  def __call__(self, key, t):
    if key not in self.w:
      g = torch.Generator().manual_seed(self.seed + 7919 * len(self.w))
      self.w[key] = torch.randint(-3, 4, tuple(t.shape), generator=g).to(torch.float64)
    w = self.w[key]
    assert tuple(w.shape) == tuple(t.shape), key
    return (w.to(t.device, t.dtype) * t).sum()


def loss_of(groups, seq_outputs, W):
  total = 0.0
  for g, out in groups.items():
    if len(out) == 4:
      seq, _, concat, per_feature = out
      total = total + W((g, 'seq'), seq)
    else:
      concat, per_feature = out
    if concat is not None:
      total = total + W((g, 'concat'), concat)
    for i, v in enumerate(per_feature):
      total = total + W((g, 'feature', i), v)
  for s, o in seq_outputs.items():
    total = total + W((s, 'key'), o['key']) + W((s, 'hist'), o['hist_seq_emb'])
  return total


def package_reg_tensors(il, groups, seq_outputs):
  """what the models hand to embedding_reg_loss: each group's output (its `_er_reg` names the looked-up tensors), the
  key and history of each seq_att group"""
  out = []
  for g, o in groups.items():
    out.append(o[0])   # the concat, or the sequence of a group read by output_seq_and_normal_feature
  for s, o in seq_outputs.items():
    out += [o['key'], o['hist_seq_emb']]
  return out


# ---- comparison -------------------------------------------------------------------------------------------------
def no_worse(mine, t32, t64, what, factor=4.0):
  em, et = (mine.double() - t64).abs().flatten(), (t32.double() - t64).abs().flatten()
  qm = float(torch.quantile(em, 0.999)) if em.numel() > 1000 else float(em.max())
  qt = float(torch.quantile(et, 0.999)) if et.numel() > 1000 else float(et.max())
  scale = float(t64.abs().mean()) if t64.numel() else 0.0
  assert qm <= factor * qt + 2e-6 * scale, '%s: p99.9 error %.3g vs float32 restatement %.3g (scale %.3g)' % (
      what, qm, qt, scale)
  assert float(em.max()) <= 10 * float(et.max()) + 1e-5 * scale, '%s: max error %.3g vs float32 restatement %.3g' % (
      what, float(em.max()), float(et.max()))


def _row_names(il, dim):
  names = []
  for t, (off, n, _) in sorted(il.arenas[dim].tables.items(), key=lambda kv: kv[1][0]):
    names += [(t, r) for r in range(n)]
  return names


def run_case(cfg_text, B, make_feats, exact, device=DEV, seed=0, check_plan=None):
  cfg = config_util.get_configs_from_pipeline_file(cfg_text.encode())
  il, model, _ = builder.build_model(cfg, B, device, generator=torch.Generator(device=device).manual_seed(seed + 1),
                                     cpu_generator=torch.Generator().manual_seed(seed + 2))
  assert all(a.opt_kind == _lib.OPT_SGD for a in il.arenas.values())
  assert il.emb_grad_mult == 1.0 and model.embedding_reg == LAMBDA
  assert all(a.n_rows <= 10 ** 4 for a in il.arenas.values())
  gen = torch.Generator().manual_seed(seed + 3)
  with torch.no_grad():
    for a in il.arenas.values():
      # multiples of 1/16: sums of weighted rows, and the regulariser's lambda * x, stay exact
      a.weight.copy_((torch.randint(-8, 9, tuple(a.weight.shape), generator=gen).float() / 16).to(device))
    for m in il.attention_modules.values():
      for p in m.parameters():
        if p.requires_grad:
          p.copy_((torch.randn(p.shape, generator=gen) * 0.5).to(device))
  rng = np.random.default_rng(seed + 4)
  feats = make_feats(rng, B, device)
  if check_plan is not None:
    check_plan(il)
  il.set_optimizer_step(1.0, 0)
  groups = il.lookup(feats)
  weights = {d: a.weight.detach().double().cpu().clone() for d, a in il.arenas.items()}
  W = Weights(seed + 5)
  # (seq_outputs also holds the layouts of in-group target attention: only the seq_att groups are outputs)
  seq_outputs = {g.group_name: il.seq_outputs[g.group_name] for g in cfg.model_config.seq_att_groups}
  loss = loss_of(groups, seq_outputs, W) + model.embedding_reg_loss(package_reg_tensors(il, groups, seq_outputs))
  loss.backward()
  with torch.no_grad():
    for a in il.arenas.values():
      a.weight.zero_()
  il.backward_update()
  G = {d: (-a.weight.detach()).double().cpu() for d, a in il.arenas.items()}
  att_grads = {k: [p.grad.detach().double().cpu() if p.grad is not None else torch.zeros(p.shape, dtype=torch.float64)
                   for p in m.parameters() if p.requires_grad] for k, m in il.attention_modules.items()}

  refs = {}
  for dt in (torch.float64,) + (() if exact else (torch.float32,)):
    ref = Reference(cfg, il, model, feats, weights, dt)
    rl = loss_of(ref.groups, ref.seq_outputs, W) + LAMBDA * 0.5 * sum((t * t).sum() for t in ref.reg)
    rl.backward()
    refs[dt] = ref
  r64 = refs[torch.float64]
  for d in il.arenas:
    g, g64 = G[d], r64.leaves[d].grad
    names = _row_names(il, d)
    untouched = ~r64.touched[d]
    bad = (g[untouched] != 0).any(1) | torch.isnan(g[untouched]).any(1)
    if bool(bad.any()):
      i = int(torch.nonzero(untouched)[torch.nonzero(bad)[0, 0]])
      raise AssertionError('dim %d, table %s row %d: untouched, but received %s' % (d, names[i][0], names[i][1],
                                                                                 g[i].tolist()))
    if exact:
      diff = (g != g64).any(1)
      if bool(diff.any()):
        i = int(torch.nonzero(diff)[0, 0])
        raise AssertionError('dim %d, table %s row %d (exact path): %d rows differ; G %s, float64 %s' % (
            d, names[i][0], names[i][1], int(diff.sum()), g[i].tolist(), g64[i].tolist()))
    else:
      tab = [t for t, _ in names]
      for t in dict.fromkeys(tab):
        sel = torch.tensor([x == t for x in tab])
        no_worse(g[sel], refs[torch.float32].leaves[d].grad[sel], g64[sel], 'dim %d, table %s' % (d, t))
  for k, grads in att_grads.items():
    for j, (got, p64) in enumerate(zip(grads, r64.att[k])):
      if exact:
        raise AssertionError('attention modules make a case inexact')
      no_worse(got, refs[torch.float32].att[k][j].grad, p64.grad, 'attention %s parameter %d' % (k, j))
  return il, r64, G


# ---- batches ------------------------------------------------------------------------------------------------------
def _t(x, dev, dt=torch.int64):
  return torch.as_tensor(np.asarray(x), dtype=dt, device=dev)


def _lens(rng, B, T):
  """lengths 0, 1 and T at the head of the batch, random after"""
  lens = rng.integers(0, T + 1, B)
  lens[:3] = [0, 1, T]
  return lens.astype(np.int32)


def _pow2(rng, n, signs=False):
  w = 2.0 ** rng.integers(-1, 2, n)
  if signs:
    w = w * rng.choice([-1.0, 0.0, 1.0, 1.0, 1.0], n)
  return w.astype(np.float32)


def _tag(rng, B, nb, dev, weighted, max_len=5, drop=False, signs=False):
  lens = rng.integers(0, max_len + 1, B)
  lens[:2] = [0, 3]
  ids = rng.integers(0, nb, int(lens.sum()))
  if drop:
    ids[:3] = -1                       # sample 1: every id dropped
    ids[rng.random(ids.size) < 0.1] = -1
  w = _pow2(rng, ids.size, signs) if weighted else None
  return (_t(ids, dev), _t(lens, dev, torch.int32), None if w is None else _t(w, dev, torch.float32))


def ids_batch(rng, B, dev):
  u = rng.integers(-10 ** 12, 10 ** 12, B)
  a = rng.integers(-3, 14, B)                       # out of range -> bucket 0, -1 dropped
  a[:4] = [-1, 10, 13, 9]
  s = rng.integers(-1, 300, B)                      # host-hashed buckets, -1 = empty string
  c1, c2 = rng.integers(0, 50, B), rng.integers(0, 60, B)
  bk = rng.integers(0, 4, B)
  sparse = np.stack([u, a, s, c1, c2, bk]).astype(np.int64)
  p = 2.0 ** rng.integers(-2, 1, (B, 1))
  q = 2.0 ** rng.integers(-2, 2, (B, 3)) * rng.choice([-1.0, 1.0], (B, 3))
  d = rng.random((B, 1))
  dense = np.concatenate([p, q, d], 1).astype(np.float32)
  return {'sparse_fea': _t(sparse.reshape(-1), dev), 'dense_fea': _t(dense, dev, torch.float32),
          'tag_fea': {'t': _tag(rng, B, 40, dev, True)}}


def tags_batch(rng, B, dev, signs=True):
  """signs: zero and negative kv weights, which K1 prunes under mean / sqrtn (the host double of K1 does not)"""
  return {'sparse_fea': _t(rng.integers(-1, 100, B), dev),
          'tag_fea': {'tm': _tag(rng, B, 100, dev, True, drop=True, signs=signs),
                      'tq': _tag(rng, B, 60, dev, True, drop=True, signs=signs),
                      'ts': _tag(rng, B, 60, dev, False, drop=True),
                      'tn': _tag(rng, B, 100, dev, False, max_len=3, drop=True)}}


def seq_batch(names, nbs, T, mseq=(), n_ids=()):
  def make(rng, B, dev):
    f = {'seq_fea': {}}
    for n, nb in zip(names, nbs):
      lens = _lens(rng, B, T)
      if n in mseq:
        per = rng.integers(0, 4, (B, T)) * (np.arange(T)[None, :] < lens[:, None])
        per[1, 0] = 0                                 # an empty step inside the length
        vals = rng.integers(0, nb, int(per.sum()))
        f['seq_fea'][n] = (_t(vals, dev), _t(lens, dev, torch.int32), _t(per.reshape(-1), dev, torch.int32))
      else:
        f['seq_fea'][n] = (_t(rng.integers(0, nb, (B, T)), dev), _t(lens, dev, torch.int32))
    if n_ids:
      f['sparse_fea'] = _t(np.concatenate([rng.integers(0, nb, B) for nb in n_ids]), dev)
    return f
  return make


# ---- plan checks: every case reaches the path it names -------------------------------------------------------------
def _check_ids(il):
  assert set(il.arenas) == {8, 4, 1}
  modes = {int(r['bucket_mode']) for m in il.merged.values() for r in m.slots_np}
  assert {_lib.BUCKET_FARM_DECIMAL, _lib.BUCKET_IDENTITY, _lib.BUCKET_ONE_ROW} <= modes


def _check_tags(il):
  m = il.merged[8]
  assert len(il.subcalls[8]) > 1 and m.has_csr and m.needs_scale and m.rows is not None


def _check_seqc(il):
  assert len(il.seqc_order['g']) == 2 and [e.name for e in il.group_layout['g']] == ['u', 'aa', 'zz']


def _check_din_group(il):
  assert [e.need_key for e in il.group_layout['g'] if e.kind == 'att'] == [True, False]


# ---- cases --------------------------------------------------------------------------------------------------------
def _check_ids_mod(il):
  _check_ids(il)
  assert any(int(r['bucket_mode']) == _lib.BUCKET_MOD for r in il.merged[8].slots_np)


def case(name, B, T=7, signs=True):
  """(config text, batch maker, exact, plan check) of each case"""
  if name in ('ids', 'ids_parquet'):
    return (head('ParquetInput' if name == 'ids_parquet' else 'DummyInput', IDS_FIELDS) + IDS, ids_batch, True,
            _check_ids_mod if name == 'ids_parquet' else _check_ids)
  if name == 'tags':
    return head() + TAGS, lambda rng, B, dev: tags_batch(rng, B, dev, signs), False, _check_tags
  if name == 'seqc':
    return (head() + SEQC % (T, T, multi_tower(['g']), LAMBDA), seq_batch(['zz', 'aa'], [40, 40], T, n_ids=[30]), False,
            _check_seqc)
  if name == 'din_group':
    return (head() + DIN_GROUP % (T, T, T, multi_tower(['g']), LAMBDA),
            seq_batch(['h_item', 'h_cate', 'h_two'], [200, 20, 200], T, n_ids=[200, 20]), False, _check_din_group)
  if name in ('seq_att_sum', 'seq_att_mean'):
    comb = name.split('_')[-1]
    return (head() + SEQ_ATT % (T, T, comb, multi_tower(['u'], din=['din']), LAMBDA),
            seq_batch(['h_item', 'h_cate'], [200, 20], T, mseq=('h_cate',), n_ids=[30, 200, 20]), comb == 'sum',
            _check_seq_att)
  if name == 'seq_out':
    return (head() + SEQ_OUT % (T, T, LAMBDA), seq_batch(['h_item', 'h_cate'], [200, 20], T, n_ids=[50, 200, 20]),
            True, _check_seq_out)
  raise KeyError(name)


def _check_seq_att(il):
  # a plain and a multi-valued history of one width: two launches, each writing its own matrix
  assert set(il.subcalls[8]) == {('single',), ('seq', il.seq_layout['din']['T']), ('mseq', il.seq_layout['din']['T'])}
  m = il.merged[8]
  assert m.has_csr and m.rows is not None


def _check_seq_out(il):
  assert [e.name for e in il.seq_group_layout['seq']['seq']] == ['h_item', 'h_cate']


CASES = [('ids', 256, 1), ('ids', 100, 1), ('ids_parquet', 256, 1), ('tags', 512, 1), ('tags', 100, 1),
         ('seqc', 256, 1), ('seqc', 256, 7), ('seqc', 100, 50), ('din_group', 256, 7), ('din_group', 256, 50),
         ('seq_att_sum', 256, 1), ('seq_att_sum', 100, 7), ('seq_att_mean', 256, 7), ('seq_out', 256, 7),
         ('seq_out', 64, 50)]


@pytest.mark.gpu
@pytest.mark.parametrize('name,B,T', CASES)
def test_input_layer_gradient_f64(name, B, T):
  text, make, exact, check = case(name, B, T)
  run_case(text, B, make, exact, check_plan=check)


@pytest.mark.parametrize('name', ['ids', 'ids_parquet', 'tags', 'seqc', 'din_group', 'seq_att_sum', 'seq_att_mean',
                                  'seq_out'])
def test_restatement_on_the_host_doubles(name, monkeypatch):
  """The same cases on the CPU, the kernels replaced by tests/host_doubles.py: rehearses the restatement and the glue
  without a device (the double of K1 does not prune by weight, so the tags carry no zero or negative weights here)."""
  import host_doubles
  host_doubles.install_all(monkeypatch.setattr)
  text, make, exact, check = case(name, 64, 7, signs=False)
  run_case(text, 64, make, exact, device='cpu', check_plan=check)


def test_restatement_matches_the_attention_combiner_restatement(monkeypatch):
  """the restatement's forward of a group with two attention-combined sequences against test_act_metrics_host's"""
  import host_doubles
  from test_act_metrics_host import CFG_SEQC, seqc_batch, seqc_expected
  host_doubles.install_all(monkeypatch.setattr)
  cfg = config_util.get_configs_from_pipeline_file(CFG_SEQC)
  il, model, _ = builder.build_model(cfg, 4, 'cpu', cpu_generator=torch.Generator().manual_seed(2))
  with torch.no_grad():
    for m in il.attention_modules.values():
      m.kernel.copy_(torch.randn(m.kernel.shape, generator=torch.Generator().manual_seed(5)))
  feats, _ = seqc_batch()
  u, pooled, unpooled = seqc_expected(il, feats)
  ref = Reference(cfg, il, model, feats, {d: a.weight.detach().double() for d, a in il.arenas.items()}, torch.float64)
  concat, per_feature = ref.groups['g']
  np.testing.assert_allclose(concat.detach().numpy(), np.concatenate([u, pooled['aa'], pooled['zz']], 1), rtol=1e-5,
                             atol=1e-6)
  for got, want in zip(per_feature, (u, pooled['zz'], pooled['aa'])):
    np.testing.assert_allclose(got.detach().numpy(), want, rtol=1e-5, atol=1e-6)
  assert sorted(tuple(r.shape) for r in ref.reg) == [(4, 3, 4), (4, 3, 4), (4, 4)]


def test_restatement_matches_the_din_restatement():
  """Reference.din against test_gpu_models.py's MultiTowerDIN restatement of target attention, in float64"""
  from easyrec_b200 import layers as L
  g = torch.Generator().manual_seed(3)
  B, T, D = 16, 5, 4
  key, hist = torch.randn(B, D, generator=g, dtype=torch.float64), torch.randn(B, T, D, generator=g, dtype=torch.float64)
  lens = torch.tensor([0, 1, T] + [2] * (B - 3), dtype=torch.int32)
  dnn = L.DNN(4 * D, L.units_of(config_util.get_configs_from_pipeline_file(
      (head() + 'model_config { multi_tower { towers { dnn { hidden_units: [8, 1] use_bn: false } } } }').encode())
      .model_config.multi_tower.towers[0].dnn), last_layer_no_activation=True, last_layer_no_batch_norm=True)
  params = [p.detach().double() for p in dnn.parameters()]
  mask = torch.arange(T)[None, :] < lens[:, None]
  he = hist * mask[:, :, None]
  cur = key[:, None, :].expand(-1, T, -1)
  x = torch.cat([cur, he, cur - he, cur * he], -1).reshape(B * T, -1)
  for i, lay in enumerate(dnn.layers):
    x = x @ params[2 * i] + params[2 * i + 1]
    if lay.relu:
      x = torch.relu(x)
  scores = torch.where(mask[:, None, :], x.reshape(B, 1, T), torch.full((B, 1, T), PAD, dtype=torch.float64))
  want = (torch.softmax(scores, -1) @ he).reshape(B, -1)
  ref = Reference.__new__(Reference)
  got = ref.din(key, he, lens, params)
  assert float((got - want).abs().max()) < 1e-12
