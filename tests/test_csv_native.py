"""CPU: the native CSV parser (er_csv_parse, through the C ABI) against the pure-python restatement of the same
format, on files with every field kind of the hot path: integer ids (negative, 19 digits), string ids
(Fingerprint64), floats in assorted spellings, empty fields -> defaults, missing trailing fields, \\r\\n line
ends, a sequence field (truncated to max_seq_len), a string tag field (tokens hashed on the host) with empty tokens, a 3-wide raw vector, and a
last line without a newline.  Results must be bit-identical."""
import ctypes
import os

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, builder
from easyrec_b200.config import config_util
from easyrec_b200.input import readers

CFG = b'''
data_config { batch_size: 64 input_type: CSVInput separator: "\\t" label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT }
  input_fields { input_name: "F1" input_type: FLOAT default_val: "2.5" }
  input_fields { input_name: "V3" input_type: STRING }
  input_fields { input_name: "C1" input_type: INT64 default_val: "7" }
  input_fields { input_name: "S1" input_type: STRING }
  input_fields { input_name: "unused" input_type: STRING }
  input_fields { input_name: "H1" input_type: STRING }
  input_fields { input_name: "T1" input_type: STRING } }
feature_config {
  features { input_names: "F1" feature_type: RawFeature embedding_dim: 8 }
  features { input_names: "V3" feature_type: RawFeature embedding_dim: 8 raw_input_dim: 3 separator: "," }
  features { input_names: "C1" feature_type: IdFeature embedding_dim: 8 hash_bucket_size: 1000 }
  features { input_names: "S1" feature_type: IdFeature embedding_dim: 8 hash_bucket_size: 1000 }
  features { input_names: "H1" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 500 max_seq_len: 4 separator: "|" }
  features { input_names: "T1" feature_type: TagFeature embedding_dim: 8 hash_bucket_size: 500 separator: "|" combiner: "mean" }
}
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["F1", "V3", "C1", "S1", "T1"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["C1", "S1"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [16] } final_dnn { hidden_units: [8] } } }
'''


def _file(path, n, rng, crlf=False, last_newline=True):
  lines = []
  for i in range(n):
    f1 = ['', '3', '-0.5', '1e-3', '7.25E+1', '.5'][rng.integers(0, 6)]
    v3 = ','.join('%g' % v for v in rng.normal(size=rng.integers(1, 4)))
    c1 = ['', str(rng.integers(-2**62, 2**62)), '-9223372036854775808', '9223372036854775807', '0'][rng.integers(0, 5)]
    s1 = ['', 'abc', 'user_%d' % rng.integers(0, 50), 'x' * 40][rng.integers(0, 4)]
    h1 = '|'.join(str(v) for v in rng.integers(0, 10**6, rng.integers(0, 7)))
    t1 = ['', '5', '5||6|', '|'.join(str(v) for v in rng.integers(-50, 10**9, rng.integers(1, 6)))][rng.integers(0, 4)]
    fields = ['%d' % rng.integers(0, 2), f1, v3, c1, s1, 'junk', h1, t1]
    if i % 11 == 3:
      fields = fields[:6]          # trailing fields missing altogether
    lines.append('\t'.join(fields))
  text = ('\r\n' if crlf else '\n').join(lines) + (('\r\n' if crlf else '\n') if last_newline else '')
  open(path, 'w', newline='').write(text)


def _same(a, b):
  (fa, la), (fb, lb) = a, b
  assert torch.equal(la, lb) and la.dtype == lb.dtype
  assert sorted(fa) == sorted(fb)
  for k in fa:
    if isinstance(fa[k], dict):
      for n in fa[k]:
        for x, y in zip(fa[k][n], fb[k][n]):
          assert (x is None and y is None) or (torch.equal(x, y) and x.dtype == y.dtype), (k, n)
    else:
      assert torch.equal(fa[k], fb[k]) and fa[k].dtype == fb[k].dtype, k


@pytest.mark.parametrize('crlf,last_newline,threads', [(False, True, 1), (True, False, 4), (False, False, 8)])
def test_native_csv_batches_equal_the_python_restatement(tmp_path, crlf, last_newline, threads):
  cfg = config_util.get_configs_from_pipeline_file(CFG)
  il, _, _ = builder.build_model(cfg, 64, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  path = str(tmp_path / 'd.csv')
  _file(path, 64 * 5 + 17, np.random.default_rng(5), crlf=crlf, last_newline=last_newline)
  native = list(readers.CSVInput(cfg, il, path, n_threads=threads))
  python = list(readers.CSVInput(cfg, il, path, engine='python'))
  assert len(native) == len(python) == 5
  for a, b in zip(native, python):
    _same(a, b)
  feats, _ = native[0]
  # string-typed hashed fields: bucket = Fingerprint64(bytes) % hash_bucket_size on the host (oracle's hash), '' -> -1,
  # and the table plan takes those buckets as they are
  from oracle import oracle as O
  first = [l.rstrip('\r\n').split('\t') for l in open(path, newline='').read().splitlines()[:64]]
  want = [O.fingerprint64(r[4]) % 1000 if len(r) > 4 and r[4] != '' else -1 for r in first]
  s1 = feats['sparse_fea'].reshape(2, 64)[il.sparse_names.index('S1')]
  assert s1.tolist() == want and -1 in want
  assert il.features['S1'].bucket_mode == _lib.BUCKET_IDENTITY and il.features['C1'].bucket_mode == _lib.BUCKET_FARM_DECIMAL
  toks = [t for r in first for t in (r[7].split('|') if len(r) > 7 else []) if t != '']
  assert feats['tag_fea']['T1'][0].tolist() == [O.fingerprint64(t) % 500 for t in toks]
  assert feats['seq_fea']['H1'][0].shape == (64, 4) and int(feats['seq_fea']['H1'][1].max()) == 4
  assert feats['dense_fea'].shape == (64, 4)


def test_native_csv_reports_the_offending_line(tmp_path):
  cfg = config_util.get_configs_from_pipeline_file(CFG)
  il, _, _ = builder.build_model(cfg, 64, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  path = str(tmp_path / 'bad.csv')
  rows = ['1\t2.0\t1,2,3\t%d\ta\tj\t1|2\t3' % i for i in range(64)]
  rows[41] = rows[41].replace('\t41\t', '\t4x1\t')
  open(path, 'w').write('\n'.join(rows) + '\n')
  with pytest.raises(_lib.ErError, match='line 42, field 4 is not a valid integer'):
    list(readers.CSVInput(cfg, il, path))


def test_er_csv_parse_stops_at_max_rows_and_leaves_the_unterminated_tail():
  lib = _lib.load()
  data = b'1,2.5\n3,\n5,7'                     # third line has no newline yet
  ids, vals = np.zeros(2, np.int64), np.zeros(2, np.float32)
  cols = (_lib.ErCsvCol * 2)()
  cols[0].kind, cols[0].out = _lib.CSV_I64, ids.ctypes.data
  cols[1].kind, cols[1].out, cols[1].default_f32 = _lib.CSV_F32, vals.ctypes.data, -1.0
  n, used = ctypes.c_int64(0), ctypes.c_size_t(0)
  assert lib.er_csv_parse(data, len(data), b',', cols, 2, 2, 1, ctypes.byref(n), ctypes.byref(used)) == 0
  assert n.value == 2 and used.value == 9 and ids.tolist() == [1, 3] and vals.tolist() == [2.5, -1.0]
  assert lib.er_csv_parse(data, len(data), b',', cols, 2, 1, 1, ctypes.byref(n), ctypes.byref(used)) == 0
  assert n.value == 1 and used.value == 6


def test_bucketized_raw_features_become_bucket_ids(tmp_path):
  """RawFeature + boundaries / num_buckets (bucketized_column, feature_column/feature_column.py:364-386): the
  readers normalise in float32 and count the boundaries <= x; the table plan sees an id feature with
  len(boundaries) + 1 rows.  Checked against a direct restatement of the TF graph on edge values."""
  import pyarrow as pa
  import pyarrow.parquet as pq
  cfg_text = b'''
data_config { batch_size: 8 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT }
  input_fields { input_name: "hour" input_type: INT32 default_val: "3" }
  input_fields { input_name: "price" input_type: DOUBLE } }
feature_config {
  features { input_names: "hour" feature_type: RawFeature embedding_dim: 8 boundaries: [18.0, 6.0, 12.0] }
  features { input_names: "price" feature_type: RawFeature embedding_dim: 8 min_val: 10.0 max_val: 110.0 num_buckets: 4 }
}
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["hour", "price"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["hour", "price"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [16] } final_dnn { hidden_units: [8] } } }
'''
  cfg = config_util.get_configs_from_pipeline_file(cfg_text)
  il, _, _ = builder.build_model(cfg, 8, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  assert il.sparse_names == ['hour', 'price'] and il.raw_names == []
  assert il.features['hour'].num_buckets == 4 and il.features['price'].num_buckets == 5   # bounds 0, .25, .5, .75
  assert il.arenas[8].tables['hour_embedding'][2] == 4 and il.arenas[8].tables['price_embedding'][2] == 5
  hours = ['0', '5', '6', '11', '12', '18', '23', '']
  prices = ['9.99', '10', '34.9', '35', '60', '85', '109.9', '500']
  open(tmp_path / 'a.csv', 'w').write(''.join('1,%s,%s\n' % hp for hp in zip(hours, prices)))
  want_hour = [0, 0, 1, 1, 2, 3, 3, 0]                      # '' -> default 3 -> below 6
  norm = (np.array([float(p) for p in prices], np.float32) - np.float32(10.0)) / np.float32(100.0)
  want_price = [int((np.array([0, .25, .5, .75], np.float32) <= v).sum()) for v in norm]
  assert want_price == [0, 1, 1, 2, 3, 4, 4, 4]
  for engine in ('native', 'python'):
    (feats, _), = list(readers.CSVInput(cfg, il, str(tmp_path / 'a.csv'), engine=engine))
    assert feats['sparse_fea'].reshape(2, 8).tolist() == [want_hour, want_price], engine
    assert 'dense_fea' not in feats
  pq.write_table(pa.table({'label': np.ones(8, np.float32), 'hour': np.array([int(h or 3) for h in hours], np.int32),
                           'price': np.array([float(p) for p in prices], np.float64)}), str(tmp_path / 'a.parquet'))
  (feats, _), = list(readers.ParquetInput(cfg, il, str(tmp_path / 'a.parquet')))
  assert feats['sparse_fea'].reshape(2, 8).tolist() == [want_hour, want_price]


def test_prefetcher_keeps_order_propagates_errors_and_stops_when_abandoned():
  import threading
  import time
  produced = []

  def source(n, fail_at=None):
    for i in range(n):
      if i == fail_at:
        raise RuntimeError('bad line %d' % i)
      produced.append(i)
      yield i
  assert list(readers.Prefetcher(source(50), depth=3)) == list(range(50))
  with pytest.raises(RuntimeError, match='bad line 7'):
    list(readers.Prefetcher(source(20, fail_at=7)))
  del produced[:]
  it = iter(readers.Prefetcher(source(10**9), depth=2))
  assert [next(it) for _ in range(5)] == [0, 1, 2, 3, 4]
  it.close()                                   # what leaving a `for` loop with `break` does
  n = len(produced)
  time.sleep(0.3)
  assert len(produced) == n and n <= 5 + 2 + 1   # the producer stopped at most depth + 1 items ahead
  assert not [t for t in threading.enumerate() if t.name == 'easyrec_b200-prefetch' and t.is_alive()]
  # the source runs ahead of a slow consumer
  t0 = time.perf_counter()

  def slow(n):
    for i in range(n):
      time.sleep(0.05)
      yield i
  for _ in readers.Prefetcher(slow(10), depth=2):
    time.sleep(0.05)
  assert time.perf_counter() - t0 < 0.85        # overlapped: ~0.55 s, serial would be 1.0 s


def test_er_csv_parse_integer_range_and_spellings():
  lib = _lib.load()

  def parse(tok):
    out = np.array([-77], np.int64)
    cols = (_lib.ErCsvCol * 1)()
    cols[0].kind, cols[0].out, cols[0].default_i64 = _lib.CSV_I64, out.ctypes.data, -77
    data = (tok + '\n').encode()
    n, used = ctypes.c_int64(0), ctypes.c_size_t(0)
    return lib.er_csv_parse(data, len(data), b',', cols, 1, 1, 1, ctypes.byref(n), ctypes.byref(used)), int(out[0])
  assert parse('9223372036854775807') == (0, 2**63 - 1) and parse('-9223372036854775808') == (0, -2**63)
  for bad in ('9223372036854775808', '-9223372036854775809', '18446744073709551616', '99999999999999999999', '1.5', '0x10', '--1'):
    assert parse(bad)[0] == _lib.ER_ERR_INVALID_ARG, bad     # out of int64 range / not an integer: refused like decode_csv
  assert parse('00000000000000000000012') == (0, 12) and parse('+5') == (0, 5) and parse(' 42 ') == (0, 42)
  assert parse('') == (0, -77)                                 # empty -> record default


def test_combo_feature_is_tensorflows_crossed_column_hash(tmp_path):
  """ComboFeature = crossed_column(inputs as strings, hash_bucket_size) (feature_column/feature_column.py:424-455).
  The cross hash is pinned to TensorFlow's own crossed-column test (feature_column_test.py CrossedColumnTest:
  bucketized [-1, .5], [.5, 1.] with boundaries (0, 1) x ['cA'], ['cB', 'cC'], hash_key 5, 5 buckets ->
  (1, 0, 1, 3, 4, 2)); the readers must produce the same buckets from text / Parquet, for STRING and INT inputs,
  and a field shared with a hashed IdFeature must still yield that feature's own bucket."""
  import pyarrow as pa
  import pyarrow.parquet as pq
  from oracle import oracle as O
  import json
  k = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'reference_kats.json')))['crossed_column']
  b = np.array(k['int_column'], np.uint64)               # bucket + 3 * k for the 2-wide bucketized column
  c = np.array([O.fingerprint64(s) for s in k['string_column']], np.uint64)
  assert readers.cross_hash([b, c], k['num_buckets'], hash_key=k['hash_key']).tolist() == k['expected'] == [1, 0, 1, 3, 4, 2]
  assert (readers.fingerprint_i64(np.array([101, 201, 301])) % 10).tolist() == [3, 7, 5]
  cfg_text = b'''
data_config { batch_size: 6 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT }
  input_fields { input_name: "site_id" input_type: STRING }
  input_fields { input_name: "app_id" input_type: STRING default_val: "none" }
  input_fields { input_name: "hour" input_type: INT64 } }
feature_config {
  features { input_names: "site_id" feature_type: IdFeature embedding_dim: 8 hash_bucket_size: 100 }
  features { input_names: ["site_id", "app_id"] feature_name: "site_app" feature_type: ComboFeature embedding_dim: 8 hash_bucket_size: 1000 }
  features { input_names: ["app_id", "hour", "site_id"] feature_name: "app_hour_site" feature_type: ComboFeature embedding_dim: 8 hash_bucket_size: 50 }
}
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["site_id", "site_app", "app_hour_site"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["site_id", "site_app", "app_hour_site"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [16] } final_dnn { hidden_units: [8] } } }
'''
  cfg = config_util.get_configs_from_pipeline_file(cfg_text)
  il, _, _ = builder.build_model(cfg, 6, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  assert il.sparse_names == ['site_id', 'site_app', 'app_hour_site']
  assert all(il.features[n].bucket_mode == _lib.BUCKET_IDENTITY for n in il.sparse_names)
  rows = [('85f751fd', 'ecad2386', '14102100'), ('', 'ecad2386', '-3'), ('1fbe01fe', '', '7'), ('x' * 40, 'y', '0'),
          ('85f751fd', 'ecad2386', '14102100'), ('', '', '12')]
  open(tmp_path / 'a.csv', 'w').write(''.join('1,%s,%s,%s\n' % r for r in rows))

  def cat(a, bb):                                         # FingerprintCat64 in python ints
    m, k = (1 << 64) - 1, 0xc6a4a7935bd1e995
    r = a ^ k
    t = (bb * k) & m
    r ^= ((t ^ (t >> 47)) * k) & m
    r = (r * k) & m
    r = ((r ^ (r >> 47)) * k) & m
    return r ^ (r >> 47)

  def cross(strings, nb):
    h = 0xDECAFCAFFE
    for s_ in strings:
      h = cat(h, O.fingerprint64(s_))
    return h % nb
  want_site = [O.fingerprint64(s_) % 100 if s_ else -1 for s_, _, _ in rows]
  want_sa = [cross([s_, a or 'none'], 1000) for s_, a, _ in rows]
  want_ahs = [cross([a or 'none', str(int(h)), s_], 50) for s_, a, h in rows]
  for engine in ('native', 'python'):
    (feats, _), = list(readers.CSVInput(cfg, il, str(tmp_path / 'a.csv'), engine=engine))
    assert feats['sparse_fea'].reshape(3, 6).tolist() == [want_site, want_sa, want_ahs], engine
  assert want_sa[0] == want_sa[4] and -1 in want_site
  pq.write_table(pa.table({'label': np.ones(6, np.float32), 'site_id': [r[0] for r in rows],
                           'app_id': [r[1] or 'none' for r in rows], 'hour': np.array([int(r[2]) for r in rows], np.int64)}),
                 str(tmp_path / 'a.parquet'))
  (feats, _), = list(readers.ParquetInput(cfg, il, str(tmp_path / 'a.parquet')))
  assert feats['sparse_fea'].reshape(3, 6).tolist() == [want_site, want_sa, want_ahs]


def test_multi_dim_bucketized_raw_feature_reproduces_tensorflows_ids(tmp_path):
  """BucketizedColumnTest: price shape (2,), boundaries [0, 2, 4, 6], [[-1., 1.], [5., 6.]] -> ids [0, 6, 3, 9]; here
  the feature becomes a fixed-length tag slot over 5 * 2 rows fed with exactly those ids, from text and Parquet."""
  import pyarrow as pa
  import pyarrow.parquet as pq
  cfg = config_util.get_configs_from_pipeline_file(b'''
data_config { batch_size: 2 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "price" input_type: STRING }
  input_fields { input_name: "uid" input_type: INT64 } }
feature_config {
  features { input_names: "price" feature_type: RawFeature raw_input_dim: 2 separator: "|" embedding_dim: 8
             boundaries: [0.0, 2.0, 4.0, 6.0] combiner: "mean" }
  features { input_names: "uid" feature_type: IdFeature embedding_dim: 8 num_buckets: 10 } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["price", "uid"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["price", "uid"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [16] } final_dnn { hidden_units: [8] } } }
''')
  il, _, _ = builder.build_model(cfg, 2, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  f = il.features['price']
  assert f.kind == 'tag' and f.num_buckets == 10 and f.bucket_mode == _lib.BUCKET_IDENTITY
  open(tmp_path / 'p.csv', 'w').write('1,-1|1,3\n0,5|6,4\n')
  pq.write_table(pa.table({'label': np.array([1, 0], np.float32), 'uid': np.array([3, 4], np.int64),
                           'price': pa.array([[-1.0, 1.0], [5.0, 6.0]], pa.list_(pa.float32()))}), str(tmp_path / 'p.parquet'))
  got = [list(readers.CSVInput(cfg, il, str(tmp_path / 'p.csv'), engine=e)) for e in ('native', 'python')]
  got.append(list(readers.ParquetInput(cfg, il, str(tmp_path / 'p.parquet'))))
  for (feats, _), in got:
    ids, lens, w = feats['tag_fea']['price']
    assert ids.tolist() == [0, 6, 3, 9] and lens.tolist() == [2, 2] and w is None
    assert feats['sparse_fea'].tolist() == [3, 4]


def test_weighted_tags_with_kv_separator(tmp_path):
  """TagFeature kv_separator (input/input.py:447-458): tokens `id:weight`; ids and fp32 weights come out in step,
  integer keys and hashed string keys alike; a token without its weight is an error."""
  from oracle import oracle as O
  cfg = config_util.get_configs_from_pipeline_file(b'''
data_config { batch_size: 3 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "kv" input_type: STRING }
  input_fields { input_name: "skv" input_type: STRING } }
feature_config {
  features { input_names: "kv" feature_type: TagFeature embedding_dim: 8 num_buckets: 100 separator: "|" kv_separator: ":" combiner: "mean" }
  features { input_names: "skv" feature_type: TagFeature embedding_dim: 8 hash_bucket_size: 30 separator: "|" kv_separator: "=" } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["kv", "skv"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["kv", "skv"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [16] } final_dnn { hidden_units: [8] } } }
''')
  il, _, _ = builder.build_model(cfg, 3, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  open(tmp_path / 'k.csv', 'w').write('1,3:0.5|7:2,cat=1.5\n0,,dog=0.25|cat=4|\n1,99:1e-1,\n')
  for engine in ('native', 'python'):
    (feats, _), = list(readers.CSVInput(cfg, il, str(tmp_path / 'k.csv'), engine=engine))
    ids, lens, w = feats['tag_fea']['kv']
    assert ids.tolist() == [3, 7, 99] and lens.tolist() == [2, 0, 1] and w.dtype == torch.float32
    assert w.tolist() == pytest.approx([0.5, 2.0, 0.1])
    ids, lens, w = feats['tag_fea']['skv']
    assert ids.tolist() == [O.fingerprint64(s) % 30 for s in ('cat', 'dog', 'cat')] and lens.tolist() == [1, 2, 0]
    assert w.tolist() == [1.5, 0.25, 4.0]
  open(tmp_path / 'bad.csv', 'w').write('1,3:0.5|7,cat=1\n0,,\n1,,\n')
  with pytest.raises(_lib.ErError, match='line 1, field 2 is not a valid key:weight list'):
    list(readers.CSVInput(cfg, il, str(tmp_path / 'bad.csv')))


def test_tag_weights_from_a_second_input_field(tmp_path):
  """TagFeature with two input_names (input/input.py:477-501): the second field holds the per-tag weights, split by
  the feature's own separator; it must hold one weight per tag.  Both parser engines, a Parquet list column, and the
  same batch as the `id:weight` spelling of the same data (kv_separator)."""
  head = b'''
data_config { batch_size: 3 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "tags" input_type: STRING }
  input_fields { input_name: "wts" input_type: STRING } }
feature_config {
  features { input_names: ["tags", "wts"] feature_type: TagFeature embedding_dim: 8 num_buckets: 100 separator: "|" combiner: "mean" } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["tags"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["tags"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [16] } final_dnn { hidden_units: [8] } } }
'''
  cfg = config_util.get_configs_from_pipeline_file(head)
  il, _, _ = builder.build_model(cfg, 3, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  open(tmp_path / 'w.csv', 'w').write('1,3|7,0.5|2\n0,,\n1,99||5|,1e-1|-3\n')
  got = {}
  for engine in ('native', 'python'):
    (feats, _), = list(readers.CSVInput(cfg, il, str(tmp_path / 'w.csv'), engine=engine))
    ids, lens, w = feats['tag_fea']['tags']
    assert ids.tolist() == [3, 7, 99, 5] and lens.tolist() == [2, 0, 2] and w.dtype == torch.float32
    assert w.tolist() == pytest.approx([0.5, 2.0, 0.1, -3.0])
    got[engine] = w
  assert torch.equal(got['native'], got['python'])
  # the kv spelling of the same data gives the same batch
  kv = config_util.get_configs_from_pipeline_file(
      head.replace(b'input_names: ["tags", "wts"]', b'input_names: "tags" kv_separator: ":"'))
  il2, _, _ = builder.build_model(kv, 3, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  open(tmp_path / 'kv.csv', 'w').write('1,3:0.5|7:2,\n0,,\n1,99:1e-1|5:-3,\n')
  (f2, _), = list(readers.CSVInput(kv, il2, str(tmp_path / 'kv.csv')))
  for a, b in zip(f2['tag_fea']['tags'], (ids, lens, w)):
    assert torch.equal(a, b)
  # one weight per tag, row by row
  open(tmp_path / 'bad.csv', 'w').write('1,3|7,0.5\n0,,\n1,9,1|2\n')
  for engine in ('native', 'python'):
    with pytest.raises(ValueError, match='TagFeature Error: The size of tags'):
      list(readers.CSVInput(cfg, il, str(tmp_path / 'bad.csv'), engine=engine))
  open(tmp_path / 'nan.csv', 'w').write('1,3|7,0.5|x\n0,,\n1,,\n')
  with pytest.raises(_lib.ErError, match='line 1, field 3 is not a valid float'):
    list(readers.CSVInput(cfg, il, str(tmp_path / 'nan.csv')))
  # kv_separator together with a weight field is the reference's own assertion (input/input.py:443-445)
  both = config_util.get_configs_from_pipeline_file(head.replace(b'separator: "|"', b'separator: "|" kv_separator: ":"'))
  with pytest.raises(ValueError, match='Cannot set kv_separator and multi input_names'):
    readers.CSVInput(both, il, str(tmp_path / 'w.csv'))
  # Parquet: a float list column beside the id list column
  import pyarrow as pa
  import pyarrow.parquet as pq
  pq.write_table(pa.table({'label': pa.array([1.0, 0.0, 1.0], pa.float32()),
                           'tags': pa.array([[3, 7], [], [99, 5]], pa.list_(pa.int64())),
                           'wts': pa.array([[0.5, 2.0], [], [0.1, -3.0]], pa.list_(pa.float32()))}),
                 str(tmp_path / 'w.parquet'))
  (fp, _), = list(readers.ParquetInput(cfg, il, str(tmp_path / 'w.parquet')))
  for a, b in zip(fp['tag_fea']['tags'], (ids, lens, w)):
    assert torch.equal(a, b)


def test_multi_valued_sequence_steps_seq_multi_sep(tmp_path):
  """SequenceFeature with seq_multi_sep (input/input.py:686-700; the lookup pinned by test/embed_test.py:88-151): every
  step holds a list of values pooled by the feature's combiner.  Both parser engines give (values of all steps back to
  back, steps per sample, values per step); through InputLayer with oracle-backed kernels each step's vector is the
  mean of its rows - embed_test's own table and expected output."""
  import host_doubles
  cfg = config_util.get_configs_from_pipeline_file(b'''
data_config { batch_size: 2 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "key" input_type: INT64 }
  input_fields { input_name: "clk" input_type: STRING } input_fields { input_name: "sclk" input_type: STRING } }
feature_config {
  features { input_names: "key" feature_type: IdFeature embedding_dim: 2 num_buckets: 6 embedding_name: "t" }
  features { input_names: "clk" feature_type: SequenceFeature embedding_dim: 2 num_buckets: 6 embedding_name: "t"
             separator: "|" seq_multi_sep: "#" combiner: "mean" max_seq_len: 4 }
  features { input_names: "sclk" feature_type: SequenceFeature embedding_dim: 2 hash_bucket_size: 11
             separator: "|" seq_multi_sep: "#" combiner: "sum" max_seq_len: 2 } }
model_config { model_class: "MultiTowerDIN"
  seq_att_groups { group_name: "din" seq_att_map { key: "key" hist_seq: "clk" } }
  feature_groups { group_name: "u" feature_names: ["key"] wide_deep: DEEP }
  multi_tower { towers { input: "u" dnn { hidden_units: [4] } } din_towers { input: "din" dnn { hidden_units: [4, 1] } }
                final_dnn { hidden_units: [4] } } }
''')
  il, _, _ = builder.build_model(cfg, 2, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  assert il.multi_valued_seq == {'clk', 'sclk'}
  # embed_test.py:88-151: ids '0#1|1#2|2#3|3#4' / '4#5|5' ... with table [[1,2],[3,4],...]: step means [2,3],[4,5],...
  open(tmp_path / 's.csv', 'w').write('1,0,0#1|1#2||2#3|3#4|4#5,a#b|c|d\n0,3,4#5|#|5,\n')
  got = {}
  for engine in ('native', 'python'):
    (feats, _), = list(readers.CSVInput(cfg, il, str(tmp_path / 's.csv'), engine=engine))
    ids, lens, step_lens = feats['seq_fea']['clk']
    assert ids.tolist() == [0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5]            # the first max_seq_len = 4 non-empty steps
    assert lens.tolist() == [4, 3] and step_lens.tolist() == [2, 2, 2, 2, 2, 0, 1, 0]   # '#' alone: a step without values
    sid, slens, ssteps = feats['seq_fea']['sclk']
    from oracle import oracle as O
    assert sid.tolist() == [O.fingerprint64(x) % 11 for x in ('a', 'b', 'c')] and slens.tolist() == [2, 0]
    assert ssteps.tolist() == [2, 1, 0, 0]
    got[engine] = feats
  for a, b in zip(got['native']['seq_fea']['clk'], got['python']['seq_fea']['clk']):
    assert torch.equal(a, b) and a.dtype == b.dtype
  # through the input layer: [B, T, D] with per-step means, zero vectors beyond the length
  import pytest as _pytest
  mp = _pytest.MonkeyPatch()
  try:
    host_doubles.install_sparse(mp.setattr)
    t = il.arenas[2]
    off, n, _ = t.tables['t']
    with torch.no_grad():
      t.weight[off:off + 6].copy_(torch.tensor([[1., 2.], [3., 4.], [5., 6.], [7., 8.], [9., 10.], [11., 12.]]))
    il.lookup(got['native'])
    so = il.seq_outputs['din']
    assert so['hist_seq_len'].tolist() == [4, 3]
    want = torch.tensor([[[2., 3.], [4., 5.], [6., 7.], [8., 9.]], [[10., 11.], [0., 0.], [11., 12.], [0., 0.]]])
    assert torch.allclose(so['hist_seq_emb'], want)
    assert torch.equal(so['key'], torch.tensor([[1., 2.], [7., 8.]]))
  finally:
    mp.undo()


@pytest.mark.parametrize('last_newline', [True, False])
def test_chunked_native_parsing_equals_batch_by_batch(tmp_path, last_newline, monkeypatch):
  """the native engine parses about 32K lines per er_csv_parse call and slices the batches out of the chunk (scalar
  rows, list values by running sums, weights, sequence steps); the end of the file falls back to one batch per call.
  Every batch equals the pure-python engine's, across two whole chunks, the short remainder and a last line without
  a newline that completes a batch."""
  cfg = config_util.get_configs_from_pipeline_file(CFG)
  B = 512
  il, _, _ = builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  chunk = 32768 // B
  n = 2 * chunk * B + 3 * B + (0 if not last_newline else 100)   # without the last newline the final line completes a batch
  path = str(tmp_path / 'big.csv')
  _file(path, n, np.random.default_rng(11), last_newline=last_newline)
  calls = []
  real = readers.CSVInput._parse

  def spy(self, data, size, plan, list_cap, n_batches=1):
    calls.append(n_batches)
    return real(self, data, size, plan, list_cap, n_batches)
  monkeypatch.setattr(readers.CSVInput, '_parse', spy)
  native = list(readers.CSVInput(cfg, il, path, n_threads=4))
  assert calls.count(chunk) >= 3 and calls.count(1) >= 3        # two full chunks + the short one, then batch by batch
  python = list(readers.CSVInput(cfg, il, path, engine='python'))
  assert len(native) == len(python) == 2 * chunk + 3
  for a, b in zip(native, python):
    _same(a, b)


def test_embed_test_seq_multi_embed_verbatim(tmp_path):
  """easy_rec/python/test/embed_test.py:88-151 with its own separators (control characters \\x03 between steps, \\x04
  between the values of a step), table and inputs: '0^D1^C1^D2' and '1^D3^C2^D4^D3^C0' -> hist[0] = [[2,3],[4,5]],
  hist[1] = [[5,6],[7,8],[1,2]], lengths 2 and 3 - through the native parser and the input layer (oracle-backed kernels)."""
  import host_doubles
  cfg = config_util.get_configs_from_pipeline_file(
      b'data_config { batch_size: 2 input_type: CSVInput separator: "," label_fields: "clk"\n'
      b'  input_fields { input_name: "clk" input_type: INT32 default_val: "0" }\n'
      b'  input_fields { input_name: "key" input_type: INT64 }\n'
      b'  input_fields { input_name: "field1" input_type: STRING default_val: "0" } }\n'
      b'feature_config {\n'
      b'  features { input_names: "key" feature_type: IdFeature embedding_dim: 2 num_buckets: 5 embedding_name: "field1_embedding" }\n'
      b'  features { input_names: "field1" feature_type: SequenceFeature separator: "\x03" seq_multi_sep: "\x04"\n'
      b'             embedding_dim: 2 num_buckets: 5 combiner: "mean" max_seq_len: 3 } }\n'
      b'model_config { model_class: "MultiTowerDIN"\n'
      b'  seq_att_groups { group_name: "din" seq_att_map { key: "key" hist_seq: "field1" } }\n'
      b'  feature_groups { group_name: "u" feature_names: ["key"] wide_deep: DEEP }\n'
      b'  multi_tower { towers { input: "u" dnn { hidden_units: [4] } } din_towers { input: "din" dnn { hidden_units: [4, 1] } }\n'
      b'                final_dnn { hidden_units: [4] } } }\n')
  fc = config_util.get_feature_configs(cfg)[1]
  assert fc.separator == '\x03' and fc.seq_multi_sep == '\x04'
  il, _, _ = builder.build_model(cfg, 2, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  open(tmp_path / 'e.csv', 'wb').write(b'0,0,0\x041\x031\x042\n0,1,1\x043\x032\x044\x043\x030\n')
  import pytest as _pytest
  mp = _pytest.MonkeyPatch()
  try:
    host_doubles.install_sparse(mp.setattr)
    for engine in ('native', 'python'):
      (feats, _), = list(readers.CSVInput(cfg, il, str(tmp_path / 'e.csv'), engine=engine))
      ids, lens, steps = feats['seq_fea']['field1']
      assert ids.tolist() == [0, 1, 1, 2, 1, 3, 2, 4, 3, 0] and lens.tolist() == [2, 3] and steps.tolist() == [2, 2, 0, 2, 3, 1]
      t = il.arenas[2]
      hist_tables = [n for n in t.tables if 'field1' in n]
      assert hist_tables, list(t.tables)
      with torch.no_grad():
        for n in hist_tables:     # (the history's table lives in the sequence group's own variable scope)
          off = t.tables[n][0]
          t.weight[off:off + 5].copy_(torch.tensor([[1., 2.], [3., 4.], [5., 6.], [7., 8.], [9., 10.]]))
      il.lookup(feats)
      so = il.seq_outputs['din']
      want = torch.tensor([[[2., 3.], [4., 5.], [0., 0.]], [[5., 6.], [7., 8.], [1., 2.]]])
      assert torch.allclose(so['hist_seq_emb'], want) and so['hist_seq_len'].tolist() == [2, 3]
      il.discard_pending()
  finally:
    mp.undo()


def test_native_and_python_engines_agree_on_random_step_lists_and_weight_fields(tmp_path):
  """randomised lines for the nested kinds added last (SequenceFeature seq_multi_sep: ER_CSV_*_STEP_LIST; TagFeature
  weights in their own field: ER_CSV_F32_LIST): empty fields, empty steps, leading / trailing / doubled separators, more
  steps than max_seq_len, string and integer values, \\r\\n - batch by batch the native parser must equal the
  pure-python restatement (and must not touch memory it does not own: the arrays are exactly sized)."""
  cfg = config_util.get_configs_from_pipeline_file(b"""
data_config { batch_size: 32 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "key" input_type: INT64 }
  input_fields { input_name: "iseq" input_type: STRING } input_fields { input_name: "sseq" input_type: STRING }
  input_fields { input_name: "tags" input_type: STRING } input_fields { input_name: "wts" input_type: STRING } }
feature_config {
  features { input_names: "key" feature_type: IdFeature embedding_dim: 4 num_buckets: 50 }
  features { input_names: "iseq" feature_type: SequenceFeature embedding_dim: 4 num_buckets: 50 separator: "|" seq_multi_sep: "#"
             combiner: "mean" max_seq_len: 5 }
  features { input_names: "sseq" feature_type: SequenceFeature embedding_dim: 4 hash_bucket_size: 37 separator: ";" seq_multi_sep: "^"
             combiner: "sum" max_seq_len: 3 }
  features { input_names: ["tags", "wts"] feature_type: TagFeature embedding_dim: 4 hash_bucket_size: 29 separator: "|" combiner: "mean" } }
model_config { model_class: "MultiTowerDIN"
  seq_att_groups { group_name: "d1" seq_att_map { key: "key" hist_seq: "iseq" } }
  seq_att_groups { group_name: "d2" seq_att_map { key: "key" hist_seq: "sseq" } }
  feature_groups { group_name: "u" feature_names: ["key", "tags"] wide_deep: DEEP }
  multi_tower { towers { input: "u" dnn { hidden_units: [4] } } din_towers { input: "d1" dnn { hidden_units: [4, 1] } }
                din_towers { input: "d2" dnn { hidden_units: [4, 1] } } final_dnn { hidden_units: [4] } } }
""")
  il, _, _ = builder.build_model(cfg, 32, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  rng = np.random.default_rng(123)

  def nested(outer, inner, val, max_steps):
    steps = []
    for _ in range(rng.integers(0, max_steps + 1)):
      vals = [val() for _ in range(rng.integers(0, 4))]
      tok = inner.join(vals)
      if rng.random() < 0.2:
        tok = inner + tok               # leading / doubled inner separators
      if rng.random() < 0.2:
        tok = tok + inner
      steps.append(tok)
    s = outer.join(steps)
    if rng.random() < 0.15:
      s = outer + s + outer
    return s
  lines = []
  for _ in range(32 * 9 + 7):
    n_tag = rng.integers(0, 5)
    tags = '|'.join('t%d' % rng.integers(0, 40) for _ in range(n_tag))
    wts = '|'.join('%.3g' % rng.uniform(-1, 3) for _ in range(n_tag))
    if n_tag and rng.random() < 0.2:
      tags, wts = tags + '|', '|' + wts        # empty tokens are skipped on both sides
    lines.append('%d,%d,%s,%s,%s,%s' % (rng.integers(0, 2), rng.integers(0, 50),
                                       nested('|', '#', lambda: str(rng.integers(0, 50)), 8),
                                       nested(';', '^', lambda: 'w%d' % rng.integers(0, 99), 5), tags, wts))
  path = str(tmp_path / 'r.csv')
  open(path, 'w', newline='').write('\r\n'.join(lines) + '\r\n')
  for threads in (1, 5):
    native = list(readers.CSVInput(cfg, il, path, n_threads=threads))
    python = list(readers.CSVInput(cfg, il, path, engine='python'))
    assert len(native) == len(python) == 9
    for a, b in zip(native, python):
      _same(a, b)
  lens = torch.cat([f['seq_fea']['iseq'][1] for f, _ in native])
  assert int(lens.max()) == 5 and int(lens.min()) == 0          # truncated to max_seq_len; empty histories occur
