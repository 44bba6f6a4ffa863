"""CPU: the glue of InputLayer (table plan, slot descriptors, input gathering, tag CSR path, group layout,
pending list -> backward update) with the four sparse kernels replaced by doubles whose bodies are the CPU
oracle.  The kernels themselves are compared with that oracle on the GPU; what runs here is everything around
them, on a config with every slot flavour: a device-hashed integer id, two TagFeatures (mean / sum) sharing one
table, a k-wide
bucketized RawFeature (fixed-length tag slot) and a RawFeature projection, fed by the native CSV reader.

The expectation is built feature by feature straight from the config semantics (table rows by name, bucket
rules, pooling), independently of the slot plan."""
import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, builder, kernels as K
from easyrec_b200.config import config_util
from easyrec_b200.input import readers
from oracle import oracle as O

import host_doubles  # noqa: E402  (tests/ is on sys.path under pytest's rootdir conftest)

CFG = b'''
data_config { batch_size: 6 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "uid" input_type: INT64 }
  input_fields { input_name: "tags" input_type: STRING } input_fields { input_name: "price" input_type: STRING }
  input_fields { input_name: "age" input_type: FLOAT } input_fields { input_name: "tags2" input_type: STRING } }
feature_config {
  features { input_names: "uid" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 50 }
  features { input_names: "tags" feature_type: TagFeature embedding_dim: 4 num_buckets: 20 separator: "|" combiner: "mean"
             embedding_name: "t" }
  features { input_names: "tags2" feature_type: TagFeature embedding_dim: 4 num_buckets: 20 separator: "|" combiner: "sum"
             embedding_name: "t" }
  features { input_names: "price" feature_type: RawFeature raw_input_dim: 2 separator: "|" embedding_dim: 4
             boundaries: [0.0, 2.0, 4.0, 6.0] combiner: "sum" }
  features { input_names: "age" feature_type: RawFeature embedding_dim: 4 min_val: 0.0 max_val: 100.0 } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["age", "uid", "price", "tags", "tags2"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["uid", "tags"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [8] } final_dnn { hidden_units: [4] } } }
'''
ROWS = [('1', '7', '3|5|5', '-1|1', '10', '5'), ('0', '-12', '', '5|6', '55.5', '1|2'), ('1', '7', '19', '2|2', '0', ''),
        ('0', '123456789012', '0|1|2|3', '7|-3', '100', '19|19|3'), ('1', '0', '4', '0|0', '31', '0'),
        ('0', '99', '6|6', '3.5|4', '77', '7|8|9|10')]


@pytest.fixture
def oracle_kernels(monkeypatch):
  host_doubles.install_sparse(monkeypatch.setattr)
  # torch.empty() returns NaN-filled memory while these tests run: host code that consumes a buffer it never wrote
  # shows up as NaN instead of passing or failing with whatever the allocator left behind
  was = torch.are_deterministic_algorithms_enabled(), torch.utils.deterministic.fill_uninitialized_memory
  torch.use_deterministic_algorithms(True)
  torch.utils.deterministic.fill_uninitialized_memory = True
  yield
  torch.use_deterministic_algorithms(was[0])
  torch.utils.deterministic.fill_uninitialized_memory = was[1]


def _expected_deep(il, rows_txt):
  """[B, 5 features x 4] in feature-group order age, uid, price, tags, tags2 - straight from the config semantics."""
  a = il.arenas[4]
  tab = a.weight.numpy()

  def table(name):
    off, local, _ = a.tables[name if name == 't' else name + '_embedding']
    return tab[off:off + local]
  out = []
  for _, uid, tags, price, age, tags2 in rows_txt:
    e_age = np.float32(float(age) / 100.0) * table('age')[0]                       # projection: x_norm * E[0]
    e_uid = table('uid')[O.fingerprint64(str(int(uid))) % 50]                      # as_string -> hash -> mod
    p = np.array([float(v) for v in price.split('|')], np.float32)
    ids = np.searchsorted(np.array([0, 2, 4, 6], np.float32), p, side='right') + 5 * np.arange(2)
    e_price = table('price')[ids].sum(0)                                           # k ids, sum combiner
    t_ids = [int(v) for v in tags.split('|') if v != '']
    e_tags = table('t')[t_ids].mean(0) if t_ids else np.zeros(4, np.float32)       # mean; empty bag -> zeros
    t2 = [int(v) for v in tags2.split('|') if v != '']
    e_tags2 = table('t')[t2].sum(0) if t2 else np.zeros(4, np.float32)             # same table, sum combiner
    out.append(np.concatenate([e_age, e_uid, e_price, e_tags, e_tags2]))
  return np.array(out, np.float32)


def test_input_layer_glue_with_oracle_kernels(tmp_path, oracle_kernels):
  cfg = config_util.get_configs_from_pipeline_file(CFG)
  il, model, _ = builder.build_model(cfg, 6, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  open(tmp_path / 'd.csv', 'w').write(''.join(','.join(r) + '\n' for r in ROWS))
  (feats, labels), = list(readers.make_input(cfg, il, str(tmp_path / 'd.csv')))
  groups = il.lookup(feats)
  deep, per_feature = groups['deep']
  want = _expected_deep(il, ROWS)
  np.testing.assert_allclose(deep.detach().numpy()[:, :20], want, rtol=1e-6, atol=1e-6)
  assert [tuple(v.shape) for v in per_feature] == [(6, 4)] * 5
  wide, _ = groups['wide']
  assert wide.shape[0] == 6 and wide.shape[1] >= 2
  # ---- backward: every looked-up row moves by the Adagrad rule on the summed gradient ----
  before = il.arenas[4].weight.clone()
  g = torch.from_numpy(np.random.default_rng(1).normal(size=tuple(deep.shape)).astype(np.float32))
  (deep * g).sum().backward()
  il.set_optimizer_step(0.05, 0)
  il.backward_update()
  a = il.arenas[4]
  tab0, G = before.numpy(), np.zeros_like(before.numpy())
  gd = g.numpy()

  def off(name):
    return a.tables[name if name == 't' else name + '_embedding'][0]
  for b, (_, uid, tags, price, age, tags2) in enumerate(ROWS):
    G[off('age')] += np.float32(float(age) / 100.0) * gd[b, 0:4]
    G[off('uid') + O.fingerprint64(str(int(uid))) % 50] += gd[b, 4:8]
    p = np.array([float(v) for v in price.split('|')], np.float32)
    for i in np.searchsorted(np.array([0, 2, 4, 6], np.float32), p, side='right') + 5 * np.arange(2):
      G[off('price') + i] += gd[b, 8:12]
    t_ids = [int(v) for v in tags.split('|') if v != '']
    for i in t_ids:
      G[off('t') + i] += gd[b, 12:16] / len(t_ids)
    for i in [int(v) for v in tags2.split('|') if v != '']:
      G[off('t') + i] += gd[b, 16:20]
  acc = 0.1 + G * G
  want_tab = np.where(G != 0, tab0 - 0.05 * G / np.sqrt(acc), tab0)
  np.testing.assert_allclose(a.weight.numpy(), want_tab, rtol=1e-5, atol=1e-6)
  assert (G != 0).any(1).sum() >= 10
  # ---- per-id weights on a tag slot (weighted mean, sum(w e) / sum(w); the other tag slot keeps weight 1) ----
  ids, lens, _ = feats['tag_fea']['tags']
  w = torch.from_numpy(np.random.default_rng(2).uniform(0.5, 2.0, ids.numel()).astype(np.float32))
  feats['tag_fea']['tags'] = (ids, lens, w)
  deep2, _ = il.lookup(feats)['deep']
  tab = il.arenas[4].weight.numpy()
  toff = il.arenas[4].tables['t'][0]
  o = 0
  for b, n in enumerate(lens.tolist()):
    e = tab[toff + ids[o:o + n].numpy()]
    ww = w[o:o + n].numpy()
    want_b = (e * ww[:, None]).sum(0) / ww.sum() if n else np.zeros(4, np.float32)
    np.testing.assert_allclose(deep2.detach().numpy()[b, 12:16], want_b, rtol=1e-5, atol=1e-6)
    o += n


def test_reference_packed_batch_through_input_layer_matches_embedding_parallel_lookup(oracle_kernels):
  """The reference's own packed batch form and its own lookup result: `embedding_parallel_lookup` executed on the
  numpy shim (tests/golden/reference_lookup.json; ids, lens feature-major, one shared table, sum combiner,
  [B, n_feat * D] output) against readers.from_reference_packed -> InputLayer.lookup on the same table."""
  import json
  import os
  c = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'reference_lookup.json')))['cases']['embedding_parallel_lookup']
  B, F = c['batch_size'], c['n_feature']
  table = np.array(c['table'], np.float32)
  V, D = table.shape
  names = ['f%d' % i for i in range(F)]
  cfg = config_util.get_configs_from_pipeline_file((
      'data_config { batch_size: %d input_type: ParquetInput label_fields: "label" '
      'input_fields { input_name: "label" input_type: FLOAT } %s }\n'
      'feature_config { %s }\n'
      'model_config { model_class: "DeepFM" feature_groups { group_name: "deep" %s wide_deep: DEEP } '
      'feature_groups { group_name: "wide" %s wide_deep: WIDE } deepfm { dnn { hidden_units: [8] } final_dnn { hidden_units: [4] } } }' % (
          B, ' '.join('input_fields { input_name: "%s" input_type: INT64 }' % n for n in names),
          ' '.join('features { input_names: "%s" feature_type: TagFeature embedding_dim: %d num_buckets: %d '
                   'embedding_name: "embedding" combiner: "sum" }' % (n, D, V) for n in names),
          ' '.join('feature_names: "%s"' % n for n in names), ' '.join('feature_names: "%s"' % n for n in names))).encode())
  il, _, _ = builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  off, local, _ = il.arenas[D].tables['embedding']
  assert local == V
  il.arenas[D].weight[off:off + V].copy_(torch.from_numpy(table))
  for rank in c['ranks']:
    feats = readers.from_reference_packed(il, {'sparse_fea': (np.array(rank['ids'], np.int64), np.array(rank['lens'], np.int32))}, names)
    deep, _ = il.lookup(feats)['deep']
    np.testing.assert_allclose(deep.detach().numpy()[:, :F * D], np.array(rank['y'], np.float32), rtol=1e-6, atol=1e-6)


def test_every_column_reads_the_slot_it_was_planned_with(monkeypatch):
  """Each layout column reads the ArenaCall column of its own slot.  The plan has one feature in two groups of the
  same width, in-group sequence_features whose key is a plain column of the group, and a history listed twice (two
  slots of one table, as a reference sample config has it): every one of them keeps its own slot's column."""
  import collections
  from easyrec_b200 import input_layer as IL
  monkeypatch.setenv('ER_PLAN_ONLY', '1')
  feats = [IL.id_feature('item', 8, hash_bucket_size=100), IL.id_feature('cate', 8, num_buckets=30),
           IL.id_feature('user', 8, hash_bucket_size=50), IL.raw_feature('price', 8),
           IL.multi_feature('hist', 'seq', 8, hash_bucket_size=100, seq_len=5)]
  seq = [dict(name='att', maps=[(['cate'], ['hist']), (['cate'], ['hist'])], units=[4, 1], need_key=True)]
  groups = collections.OrderedDict([('user', dict(features=['user', 'item', 'price'])),
                                    ('item', dict(features=['price', 'item', 'cate'], seq=seq))])
  seq_att = collections.OrderedDict([('din', [(['item'], ['hist'])])])
  il = IL.InputLayer(feats, groups, 4, 'cpu', seq_att_groups=seq_att, dense_generator=torch.Generator().manual_seed(0))
  col_of = {id(s): c for subs in il.subcalls.values() for sc in subs.values()
            for s, c in zip(sc.call.slots, sc.call.slot_cols)}
  columns = [e for lay in il.group_layout.values() for e in lay]
  columns += [e for lay in il.seq_layout.values() for e in lay['key'] + lay['hist']]
  looked_up = [e for e in columns if e.slot is not None]
  assert len(looked_up) == 12 and all(e.slot is not None for e in columns if getattr(e, 'kind', None) == 'emb')
  for e in looked_up:
    assert e.slot.name == '%s/%s' % (e.out_key, e.name) and e.col == col_of[id(e.slot)], e
  user, item = il.group_layout['user'], il.group_layout['item']
  assert [(e.name, e.col) for e in user] == [('user', 0), ('item', 8), ('price', 16)]
  assert [(e.name, e.col) for e in item[:3]] == [('price', 0), ('item', 8), ('cate', 16)]
  assert user[1].slot is not item[1].slot and user[2].slot is not item[2].slot
  att = il.seq_layout['item/att']
  assert [e.slot for e in att['key']] == [item[2].slot] * 2 and [e.col for e in att['key']] == [16, 16]
  assert [e.col for e in att['hist']] == [0, 8] and att['hist'][0].slot is not att['hist'][1].slot
  assert item[3] == IL.GroupColumn('seq_fea/att', 'att', 32, out_key='item/att', need_key=True)
  assert il.group_width('user') == 24 and il.group_width('item') == 56
