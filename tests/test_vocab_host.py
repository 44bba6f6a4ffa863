"""CPU, kernel doubles: vocabulary columns (`vocab_list` / `vocab_file`) against a plain-Python restatement of TF's
lookup - categorical_column_with_vocabulary_{list,file} with default_value 0 and no OOV buckets
(feature_column/feature_column.py:277-290,320-333,497-509): a value reads the row of its position in the vocabulary, a
value outside it reads row 0, '' is no value.  The configs and batches here are shared with the GPU and gloo tests."""
import numpy as np
import pytest
import torch

import host_doubles
from easyrec_b200 import _lib, builder
from easyrec_b200.config import config_util
from easyrec_b200.input import readers

B = 8
T = 3
U_VOCAB = ['u%d' % i for i in range(10)]
T_VOCAB = ['red', 'green', 'blue', 'a b', 'été']
I_VOCAB = ['item%d' % i for i in range(12)]


def tf_lookup(vocab, value):
  """TF's vocabulary lookup of one string: its position, 0 outside the vocabulary, None for '' (no value)"""
  if value == '':
    return None
  return vocab.index(value) if value in vocab else 0


def write_vocab_file(path, entries, trailing_newline=True):
  with open(path, 'wb') as f:
    f.write('\n'.join(entries).encode('utf-8') + (b'\n' if trailing_newline else b''))
  return str(path)


def _q(entries):
  return '[%s]' % ', '.join('"%s"' % e for e in entries)


def config(vocab_file, form='vocab', extra_train=''):
  """MultiTowerDIN over a vocabulary IdFeature (STRING), a kv-weighted mean TagFeature and a DIN key + history whose
  vocabulary comes from `vocab_file`.  form 'identity': the same model over identity columns of the same sizes, fed the
  positions (the twin the vocabulary model must train like)."""
  if form == 'vocab':
    u, t, i = ('vocab_list: %s' % _q(U_VOCAB), 'vocab_list: %s' % _q(T_VOCAB), 'vocab_file: "%s"' % vocab_file)
    ft = 'STRING'
  else:
    u, t, i = ('num_buckets: %d' % len(U_VOCAB), 'num_buckets: %d' % len(T_VOCAB), 'num_buckets: %d' % len(I_VOCAB))
    ft = 'INT64'
  return ('''
train_config { %s
  optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.05 } } } } }
data_config { batch_size: %d input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "u" input_type: %s }
  input_fields { input_name: "t" input_type: STRING } input_fields { input_name: "key" input_type: %s }
  input_fields { input_name: "clk" input_type: STRING } }
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 4 %s }
  features { input_names: "t" feature_type: TagFeature embedding_dim: 4 %s separator: "|" kv_separator: ":"
             combiner: "mean" }
  features { input_names: "key" feature_type: IdFeature embedding_dim: 4 %s }
  features { input_names: "clk" feature_type: SequenceFeature embedding_dim: 4 %s separator: "|" max_seq_len: %d } }
model_config { model_class: "MultiTowerDIN"
  seq_att_groups { group_name: "din" seq_att_map { key: "key" hist_seq: "clk" } }
  feature_groups { group_name: "g" feature_names: ["u", "t"] wide_deep: DEEP }
  multi_tower { towers { input: "g" dnn { hidden_units: [8] } } din_towers { input: "din" dnn { hidden_units: [4, 1] } }
                final_dnn { hidden_units: [4] } l2_regularization: 1e-5 }
  embedding_regularization: 1e-5 }
''' % (extra_train, B, ft, ft, u, t, i, i, T)).encode()


def _pick(rng, vocab, extra):
  pool = vocab + extra
  return pool[rng.integers(0, len(pool))]


def raw_batch(seed, n=B, fixed_tags=False):
  """raw strings of one batch: values in and out of the vocabularies, '' among them.  fixed_tags: two non-empty tags per
  sample, so that every batch has one shape (a captured CUDA graph)"""
  rng = np.random.default_rng(seed)
  rows = []
  for _ in range(n):
    u = _pick(rng, U_VOCAB, ['u10', 'zz', ''])
    tags = [(_pick(rng, T_VOCAB, ['purple'] if fixed_tags else ['purple', '']),
             float(rng.choice([0.5, 1.25, 2.0, 0.0, -1.0]))) for _ in range(2 if fixed_tags else rng.integers(0, 4))]
    key = _pick(rng, I_VOCAB, ['item12', ''])
    clk = [_pick(rng, I_VOCAB, ['nope']) for _ in range(rng.integers(1, T + 1))]
    rows.append(dict(u=u, t=tags, key=key, clk=clk, label=float(rng.integers(0, 2))))
  return rows


def csv_lines(rows):
  """the batch as CSV lines of the vocabulary config (empty tag tokens are dropped by the parser)"""
  return ['%d,%s,%s,%s,%s' % (r['label'], r['u'], '|'.join('%s:%g' % tw for tw in r['t'] if tw[0]), r['key'],
                              '|'.join(r['clk'])) for r in rows]


def features(rows, form):
  """(features, labels) of a raw batch: the readers' 63-bit keys for the vocabulary model (form 'vocab'), TF's positions
  restated in Python for its identity twin (form 'identity'; '' -> -1, no value)"""
  def conv(vocab, v):
    if form == 'vocab':
      return int(readers.string_keys([v])[0])
    p = tf_lookup(vocab, v)
    return -1 if p is None else p
  u = [conv(U_VOCAB, r['u']) for r in rows]
  key = [conv(I_VOCAB, r['key']) for r in rows]
  tags = [(conv(T_VOCAB, s), w) for r in rows for s, w in r['t'] if s]   # ('' tokens never reach the batch)
  tag_lens = [sum(1 for s, _ in r['t'] if s) for r in rows]
  seq = np.full((len(rows), T), -1, np.int64)
  for b, r in enumerate(rows):
    seq[b, :len(r['clk'])] = [conv(I_VOCAB, s) for s in r['clk']]
  feats = {'sparse_fea': torch.tensor(u + key, dtype=torch.int64),
           'tag_fea': {'t': (torch.tensor([k for k, _ in tags], dtype=torch.int64),
                             torch.tensor(tag_lens, dtype=torch.int32),
                             torch.tensor([w for _, w in tags], dtype=torch.float32))},
           'seq_fea': {'clk': (torch.from_numpy(seq), torch.tensor([len(r['clk']) for r in rows], dtype=torch.int32))}}
  return feats, torch.tensor([r['label'] for r in rows], dtype=torch.float32)


def tables_and_slots(il):
  """every arena's storage (rows and optimizer slots side by side), as bytes"""
  return {str(k): a.storage.detach().cpu().numpy().tobytes() for k, a in il.arenas.items()}


def train_pair(tmp_path, device, steps=4, graph=False):
  """(losses, tables) of the vocabulary model and of its identity twin trained on the same batches"""
  from easyrec_b200.estimator import EasyRecEstimator
  from easyrec_b200.trainer import Trainer
  vf = write_vocab_file(tmp_path / 'items.txt', I_VOCAB, trailing_newline=False)
  out = []
  for form in ('vocab', 'identity'):
    torch.manual_seed(0)
    est = EasyRecEstimator(config(vf, form), device=device, seed=3)
    tr = Trainer(est.model, est.input_layer, 'adagrad', lr=0.05, use_cuda_graph=graph) if graph else est.trainer
    losses = []
    for step in range(steps):
      feats, labels = readers.to_device(*features(raw_batch(step), form), device)
      losses.append(float(tr.train_step(feats, labels)[0]))
    out.append((losses, tables_and_slots(est.input_layer)))
  return out


@pytest.fixture
def doubles(monkeypatch):
  host_doubles.install_all(monkeypatch.setattr)
  import seq_doubles
  import vocab_doubles
  seq_doubles.install(monkeypatch.setattr)
  vocab_doubles.install(monkeypatch.setattr)


def test_a_host_device_without_k1_refuses_a_vocabulary_model_by_name(tmp_path, monkeypatch):
  """only the GPU's K1 reads a vocabulary index: a host build is refused rather than run on a K1 that would read the
  keys as rows; a plan built only to be inspected (ER_PLAN_ONLY) has no index"""
  host_doubles.install_all(monkeypatch.setattr)
  text = config(write_vocab_file(tmp_path / 'items.txt', I_VOCAB))
  with pytest.raises(NotImplementedError, match='a vocabulary index is probed by K1 on the GPU; device cpu has no K1'):
    _build(text)
  monkeypatch.setenv('ER_PLAN_ONLY', '1')
  il, _, _ = _build(text)
  assert il.features['u'].bucket_mode == _lib.BUCKET_VOCAB and il.arenas[4].tables['u_embedding'][1] == len(U_VOCAB)


def test_vocab_list_and_file_keys_are_the_readers_keys_of_each_entry(tmp_path):
  assert builder.vocab_entries(_fc(b'vocab_list: ["a", "b c", ""]')) == [b'a', b'b c', b'']
  for trailing in (True, False):
    path = write_vocab_file(tmp_path / ('v%d.txt' % trailing), I_VOCAB, trailing)
    entries = builder.vocab_entries(_fc(('vocab_file: "%s"' % path).encode()))
    assert entries == [e.encode() for e in I_VOCAB]            # one entry per line, the last one with or without '\n'
    keys = builder.vocab_keys('f', entries)
    assert list(keys) == readers.string_keys(I_VOCAB).tolist()
    assert all(0 <= k < 2**63 - 1 for k in keys)
  assert readers.string_keys(['', None]).tolist() == [-1, -1]
  # hash_bucket_size wins over a vocabulary in the reference, which never reads it: such configs are refused
  with pytest.raises(NotImplementedError, match='hash_bucket_size together with vocab_list'):
    builder.vocabulary(None, _fc(b'hash_bucket_size: 5 vocab_list: ["a"]'), 'f', {}, 0)
  # vocab_list is read before vocab_file
  fc = _fc(('vocab_list: ["x", "y"] vocab_file: "%s"' % path).encode())
  assert builder.vocab_entries(fc) == [b'x', b'y']


def _fc(text):
  cfg = config_util.get_configs_from_pipeline_file(
      b'feature_config { features { input_names: "f" feature_type: TagFeature embedding_dim: 4 ' + text + b' } }')
  return config_util.get_feature_configs(cfg)[0]


def test_the_csv_reader_keys_every_vocabulary_string(tmp_path):
  vf = write_vocab_file(tmp_path / 'items.txt', I_VOCAB)
  cfg = config_util.get_configs_from_pipeline_file(config(vf))
  specs = builder.feature_specs(cfg)
  assert [(s.name, s.bucket_mode, s.num_buckets) for s in specs] == [
      ('u', _lib.BUCKET_VOCAB, 10), ('t', _lib.BUCKET_VOCAB, 5), ('key', _lib.BUCKET_VOCAB, 12),
      ('clk', _lib.BUCKET_VOCAB, 12)]
  import host_doubles as hd   # noqa: F401  (the reader needs no kernel)
  from easyrec_b200 import input_layer as IL

  class Plan(object):        # what the CSV reader reads of an InputLayer
    features = {s.name: s for s in specs}
    sparse_names = ['u', 'key']
    raw_names = []
    batch_size = B
  rows = raw_batch(7)
  path = tmp_path / 'b.csv'
  path.write_text('\n'.join(csv_lines(rows)) + '\n')
  for engine in ('native', 'python'):
    (feats, labels), = list(readers.CSVInput(cfg, Plan, str(path), engine=engine))
    want, want_labels = features(rows, 'vocab')
    assert torch.equal(feats['sparse_fea'], want['sparse_fea']), engine
    for i in range(3):
      assert torch.equal(feats['tag_fea']['t'][i], want['tag_fea']['t'][i]), (engine, i)
    got_seq, got_lens = feats['seq_fea']['clk']
    assert torch.equal(got_lens, want['seq_fea']['clk'][1])
    live = np.arange(T)[None, :] < got_lens.numpy()[:, None]
    assert np.array_equal(got_seq.numpy()[live], want['seq_fea']['clk'][0].numpy()[live])
    assert torch.equal(labels, want_labels)
  assert IL.FeatureSpec._fields[-1] == 'vocab'


def test_vocabulary_model_trains_like_its_identity_twin_fed_tf_positions(tmp_path, doubles):
  (lv, tv), (li, ti) = train_pair(tmp_path, 'cpu')
  assert lv == li and lv[0] != lv[-1]
  assert tv == ti


def test_the_lookup_reads_the_rows_tf_reads(tmp_path, doubles):
  """one forward on the doubles: every id, tag and history step reads the row of TF's position (OOV -> row 0, ''
  no row, mean pooling over the weights > 0)"""
  from easyrec_b200.estimator import EasyRecEstimator
  vf = write_vocab_file(tmp_path / 'items.txt', I_VOCAB, trailing_newline=False)
  est = EasyRecEstimator(config(vf), device='cpu', seed=3)
  il = est.input_layer
  rows = raw_batch(11)
  feats, _ = features(rows, 'vocab')
  with torch.no_grad():
    concat, _ = il.lookup(feats)['g']
    din = il.seq_outputs['din']
  il.discard_pending()
  tu = il.arenas[4].table_view('u_embedding').numpy()
  tt = il.arenas[4].table_view('t_embedding').numpy()
  tk = il.arenas[4].table_view('din/key_embedding').numpy()
  th = il.arenas[4].table_view('din/clk_embedding').numpy()
  for b, r in enumerate(rows):
    p = tf_lookup(U_VOCAB, r['u'])
    np.testing.assert_array_equal(concat[b, :4].detach().numpy(), np.zeros(4, np.float32) if p is None else tu[p])
    live = [(tf_lookup(T_VOCAB, s), w) for s, w in r['t'] if s and w > 0]
    want = (sum(np.float64(w) * tt[p] for p, w in live) / sum(w for _, w in live)) if live else np.zeros(4)
    np.testing.assert_allclose(concat[b, 4:8].detach().numpy(), want, rtol=1e-6, atol=1e-7)
    p = tf_lookup(I_VOCAB, r['key'])
    np.testing.assert_array_equal(din['key'][b].detach().numpy(), np.zeros(4, np.float32) if p is None else tk[p])
    for t, s in enumerate(r['clk']):
      np.testing.assert_array_equal(din['hist_seq_emb'][b, t].detach().numpy(), th[tf_lookup(I_VOCAB, s)])


def _build(text):
  cfg = config_util.get_configs_from_pipeline_file(text)
  return builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(0))


@pytest.mark.parametrize('edit,err,words', [
    (('vocab_list: %s' % _q(U_VOCAB), 'vocab_list: %s ev_params { max_capacity: 100 }' % _q(U_VOCAB)),
     NotImplementedError, 'feature u: vocab_list / vocab_file together with ev_params'),
    (('vocab_list: %s' % _q(U_VOCAB), 'vocab_list: ["u1", "u2", "u1", "u3", "u2"]'), ValueError,
     "feature u: vocabulary entries ['u1', 'u2'] appear more than once"),
    (('input_name: "u" input_type: STRING', 'input_name: "u" input_type: INT64'), ValueError,
     'feature u: vocab_list / vocab_file on the INT64 field u'),
    (('input_type: CSVInput', 'input_type: CriteoInput'), NotImplementedError,
     'feature u: vocab_list / vocab_file with CriteoInput'),
    (('features { input_names: "key" feature_type: IdFeature embedding_dim: 4',
      'features { input_names: "key" feature_type: IdFeature embedding_dim: 4 embedding_name: "shared"'), None, None),
])
def test_configs_a_vocabulary_cannot_serve_are_refused_by_name(tmp_path, doubles, edit, err, words):
  vf = write_vocab_file(tmp_path / 'items.txt', I_VOCAB)
  text = config(vf).decode()
  assert edit[0] in text
  text = text.replace(edit[0], edit[1], 1)
  if err is None:   # a shared embedding_name whose readers disagree on the row count
    text = text.replace('feature_type: TagFeature embedding_dim: 4', 'feature_type: TagFeature embedding_dim: 4 '
                        'embedding_name: "shared"')
    err, words = ValueError, 'embedding_name shared: shared by features with different row counts (t: 5, key: 12)'
  with pytest.raises(err) as e:
    _build(text.encode())
  assert words in str(e.value)


def test_entries_with_one_key_are_refused_by_name(monkeypatch):
  real = _lib.fingerprint64
  monkeypatch.setattr(_lib, 'fingerprint64', lambda e: 42 if e in (b'b', b'c') else real(e))
  with pytest.raises(NotImplementedError, match="feature f: vocabulary entries 'b' and 'c' have the same 63-bit key 42"):
    builder.vocab_keys('f', [b'a', b'b', b'c'])
  with pytest.raises(ValueError, match='feature f: the vocabulary is empty'):
    builder.vocab_keys('f', [])


def test_vocabulary_refusals_on_features_and_blocks_that_do_not_read_one(tmp_path):
  raw = _fc(b'vocab_list: ["a"]')
  raw.feature_type = raw.RawFeature
  with pytest.raises(NotImplementedError, match='feature f: vocab_list / vocab_file on a RawFeature'):
    builder.vocabulary(None, raw, 'f', {}, 0)
  # a backbone embedding_layer block hashes its features into vocabulary-sized buckets: refused for a vocabulary
  spec = builder.IL.id_feature('u', 4, vocab=(5, 6))
  cfg = config_util.get_configs_from_pipeline_file(b'''
model_config { model_class: "RankModel" feature_groups { group_name: "ids" feature_names: "u" wide_deep: DEEP }
  backbone { blocks { name: "emb" inputs { feature_group_name: "ids" } embedding_layer { embedding_dim: 8 } } } }''')
  with pytest.raises(NotImplementedError, match='embedding_layer block emb: feature u has a vocabulary'):
    builder.embedding_layer_tables(cfg.model_config, [spec])


@pytest.mark.timeout(300)
def test_both_reference_vocab_samples_build_train_and_evaluate(doubles):
  from test_config import reference_configs
  from easyrec_b200.estimator import EasyRecEstimator
  found = 0
  for p, text in sorted(reference_configs().items()):
    if 'vocab_list' not in p:
      continue
    found += 1
    cfg = config_util.get_configs_from_pipeline_file(text)
    est = EasyRecEstimator(cfg, device='cpu', seed=1, batch_size=8)
    hour = est.input_layer.features['hour']
    assert hour.bucket_mode == _lib.BUCKET_VOCAB and hour.num_buckets == 25
    feats, labels = readers.DummyInput(est.input_layer, seed=3).batch()
    assert np.isfinite(float(est.trainer.train_step(feats, labels)[0]))
  assert found == 2
