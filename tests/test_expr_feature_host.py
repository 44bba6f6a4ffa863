"""CPU, kernel doubles: ExprFeature columns against the reference's own grammar (tests/golden/reference_expr.json, made by
make_expr_golden.py from utils/expr_util.py), the readers' float64 inputs, every refusal, the reference sample config,
and training: a model whose ExprFeatures sit in deep and wide groups must train exactly like its twin that reads the
fixture's values as RawFeatures.  The configs and batches here are shared with the GPU test."""
import json
import os
import re

import numpy as np
import pytest
import torch

import expr_doubles
import host_doubles
from easyrec_b200 import builder, expr as X
from easyrec_b200.config import config_util
from easyrec_b200.input import readers

HERE = os.path.dirname(os.path.abspath(__file__))

# forms the reference rewrites but TF rejects when it builds the graph (numpy, which made the fixture, accepts them), and
# what is refused for another reason: expression -> a fragment of the refusal
REFUSED = {
    'x>y>z': 'compares a bool with a number', 'x==y==z': 'compares a bool with a number',
    'x>True': 'True is not a number', '5<x': 'bare number on the left', 'x**2>1': 'Pow on an input',
    'x//2>1': 'FloorDiv on an input', '+x': 'unary +', '(x>y)>(y>z)': 'orders two bools',
    '(x>y)==1': 'compares a bool with a number',
}


def fixture():
  with open(os.path.join(HERE, 'golden', 'reference_expr.json')) as f:
    d = json.load(f)
  rows = np.array([[int(h, 16) for h in r] for r in d['rows']], np.uint64).view(np.float64)
  return rows, d['cases']


def same_bits(got, want_hex):
  """float32 results against the fixture's bit patterns; a NaN matches any NaN (its sign and payload are the
  platform's)"""
  want = np.array([int(h, 16) for h in want_hex], np.uint32)
  got = np.asarray(got, np.float32)
  nan = np.isnan(want.view(np.float32))
  return bool((np.isnan(got) == nan).all() and (got.view(np.uint32)[~nan] == want[~nan]).all())


def reference_text(source, names):
  """the compiler's text with the reference's spelling of inputs and comparisons"""
  for k, n in enumerate(names):
    source = source.replace('_in(%d)' % k, "parsed_dict['expr_%s']" % n)
  for op, fn in (('_ge', 'greater_equal'), ('_gt', 'greater'), ('_le', 'less_equal'), ('_lt', 'less'),
                 ('_eq', 'equal')):
    source = source.replace(op + '(', 'tf.%s(' % fn)
  return source


def test_the_compiler_and_the_kernel_double_replay_the_reference_grammar():
  rows, cases = fixture()
  seen = 0
  for c in cases:
    e, names = c['expression'], c['input_names']
    if 'reference' in c:
      assert reference_text(X.source(e, names), names) == c['reference'], e
    if 'out' in c and e not in REFUSED:
      p = X.compile_expression('f', e, names)
      assert same_bits(expr_doubles.evaluate(p.ops, rows), c['out']), e
      seen += 1
    else:
      with pytest.raises(ValueError, match='ExprFeature f: expression') as ex:
        X.compile_expression('f', e, names)
      if e in REFUSED:
        assert REFUSED[e] in str(ex.value), (e, str(ex.value))
  assert seen >= 45
  assert set(REFUSED) <= set(c['expression'] for c in cases)


def test_programs_need_at_most_the_kernel_stack():
  # an operand before "(" is dropped and & / | fold flat: the stack grows only through == of bools, & under | and
  # Python's precedence inside an operand
  assert X.compile_expression('f', 'x-(x-(x-(x-(x-(x-(x-(x-(x-x))))))))', ['x']).depth == 2
  assert X.compile_expression('f', '(x>1)&((x>1)&((x>1)&((x>1)&((x>1)&(x>1)))))', ['x']).depth == 3
  deepest = '(x>y)==((y>z)==((x>z)|(z>1)&(x>y-z*x)))'   # (in the fixture: the kernel runs it)
  assert X.compile_expression('f', deepest, ['x', 'y', 'z']).depth == X.MAX_STACK
  with pytest.raises(ValueError, match=r'ExprFeature f: .*a stack of 9 values; er_expr_eval holds 8'):
    X.compile_expression('f', '(x>1)==(' + deepest + ')', ['x', 'y', 'z'])


CFG = '''
train_config { %s
  optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.1 } } } } }
data_config { batch_size: %d input_type: %s separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT }
  input_fields { input_name: "x" input_type: DOUBLE default_val: "1.5" }
  input_fields { input_name: "y" input_type: INT64 default_val: "7" }
  input_fields { input_name: "z" input_type: STRING default_val: "3.25" }
  input_fields { input_name: "r" input_type: FLOAT } input_fields { input_name: "c" input_type: INT64 }
  %s }
feature_config {
  features { input_names: "r" feature_type: RawFeature }
  features { input_names: "c" feature_type: IdFeature embedding_dim: 8 num_buckets: 37 }
  %s }
model_config { model_class: "WideAndDeep"
  feature_groups { group_name: "wide" feature_names: ["c", "e1", "e3"] wide_deep: WIDE }
  feature_groups { group_name: "deep" feature_names: ["r", "c", "e1", "e2"] wide_deep: DEEP }
  wide_and_deep { dnn { hidden_units: [16] use_bn: false } final_dnn { hidden_units: [8] use_bn: false }
                  l2_regularization: 1e-5 } }
'''
# fixture expressions over (x, y, z): two bools and a float
EXPRS = (('e1', '(x>=1)&(x<=5)|(y==2)'), ('e2', 'x*y+z'), ('e3', '(x>y) | (y>z) & (z>x)'))


def config(form, batch_size, extra_train='', input_type='CSVInput', feature=None):
  """form 'expr': e1..e3 are ExprFeatures over x, y, z; 'raw': the twin, e1..e3 RawFeatures over FLOAT fields"""
  if form == 'expr':
    feats = ' '.join('features { feature_name: "%s" input_names: ["x", "y", "z"] feature_type: ExprFeature '
                     'expression: "%s" %s }' % (n, e, feature or '') for n, e in EXPRS)
    fields = ''
  else:
    feats = ' '.join('features { input_names: "%s" feature_type: RawFeature }' % n for n, _ in EXPRS)
    fields = ' '.join('input_fields { input_name: "%s" input_type: FLOAT }' % n for n, _ in EXPRS)
  return (CFG % (extra_train, batch_size, input_type, fields, feats)).encode()


def twin_rows():
  """(inputs float64 [B, 3], values float32 [B, 3] of e1..e3 from the fixture): the fixture rows where e2 is small"""
  rows, cases = fixture()
  by = {c['expression']: c for c in cases}
  vals = np.stack([np.array([int(h, 16) for h in by[e]['out']], np.uint32).view(np.float32) for _, e in EXPRS], 1)
  keep = np.isfinite(vals).all(1) & (np.abs(vals) < 1e4).all(1)
  return rows[keep], vals[keep]


def twin_batches(inputs, values, n_steps, seed):
  """[(expr model batch, raw twin batch, labels)]: the same samples, the ExprFeatures' columns of the expr model's
  dense_fea hold junk that er_expr_eval overwrites"""
  rng = np.random.default_rng(seed)
  out = []
  B = inputs.shape[0]
  for _ in range(n_steps):
    r = rng.uniform(-1, 1, (B, 1)).astype(np.float32)
    c = rng.integers(0, 37, B).astype(np.int64)
    labels = torch.from_numpy((rng.uniform(size=B) < 0.4).astype(np.float32))
    junk = np.full((B, 3), -7.0, np.float32)
    perm = rng.permutation(B)   # the expressions' inputs change from step to step, as a replayed graph must see them
    fx = {'sparse_fea': torch.from_numpy(c), 'dense_fea': torch.from_numpy(np.concatenate([r, junk], 1)),
          'expr_fea': torch.from_numpy(inputs[perm].copy())}
    fr = {'sparse_fea': torch.from_numpy(c.copy()),
          'dense_fea': torch.from_numpy(np.concatenate([r, values[perm]], 1))}
    out.append((fx, fr, labels))
  return out


def same_start(a, b):
  """b <- a's tables, optimizer state and dense parameters (the twins are built alike; this makes it explicit)"""
  for k, arena in a.input_layer.arenas.items():
    b.input_layer.arenas[k].storage.copy_(arena.storage)
  b.model.load_state_dict(a.model.state_dict())
  b.trainer.dense_opt.flat_p.copy_(a.trainer.dense_opt.flat_p)


def assert_same_model(a, b):
  for k, arena in a.input_layer.arenas.items():
    assert torch.equal(arena.storage, b.input_layer.arenas[k].storage), k
  assert torch.equal(a.trainer.dense_opt.flat_p, b.trainer.dense_opt.flat_p)


def run_twins(device, steps=3, use_cuda_graph=False, seed=11, **kw):
  """the expr model and its raw twin trained side by side; kw: EasyRecEstimator's world_size / rank /
  embedding_parallel"""
  from easyrec_b200.estimator import EasyRecEstimator
  inputs, values = twin_rows()
  B = inputs.shape[0]
  ex = EasyRecEstimator(config('expr', B), device=device, seed=3, use_cuda_graph=use_cuda_graph, **kw)
  raw = EasyRecEstimator(config('raw', B), device=device, seed=3, use_cuda_graph=use_cuda_graph, **kw)
  assert ex.input_layer.expr_inputs == ['x', 'y', 'z'] and ex.input_layer.raw_cols == raw.input_layer.raw_cols
  same_start(ex, raw)
  losses = []
  for fx, fr, labels in twin_batches(inputs, values, steps, seed=seed):
    dev = lambda d: {k: v.to(device) for k, v in d.items()}   # noqa: E731
    lx, _ = ex.trainer.train_step(dev(fx), labels.to(device))
    lr, _ = raw.trainer.train_step(dev(fr), labels.to(device))
    assert float(lx) == float(lr) and np.isfinite(float(lx))
    assert torch.equal(ex.trainer.dense_opt.flat_g, raw.trainer.dense_opt.flat_g)
    losses.append(float(lx))
  assert_same_model(ex, raw)
  return ex, raw, losses


def test_expr_features_in_deep_and_wide_groups_train_like_their_raw_twin(monkeypatch):
  host_doubles.install_all(monkeypatch.setattr)
  expr_doubles.install(monkeypatch.setattr)
  ex, raw, _ = run_twins('cpu')
  il = ex.input_layer
  # deep: raw columns without a table; wide: the one-row tables numeric columns get
  assert [e.kind for e in il.group_layout['deep']] == ['dense', 'emb', 'dense', 'dense']
  assert all(il.features[n].embedding_dim == 0 and il.features[n].min_val == il.features[n].max_val == 0
             for n in ('e1', 'e2', 'e3'))


def _write_csv(path, lines):
  with open(path, 'w') as f:
    f.write(''.join(l + '\n' for l in lines))
  return str(path)


# label, x (DOUBLE), y (INT64), z (STRING numbers), r, c; empty x / y / z take 1.5 / 7 / "3.25"
CSV_LINES = ['1,0.1,3,1e3,0.5,4', '0,,,,0.25,5', '1,-0,9007199254740993,9007199254740993,1,6',
             '0,2.5e-310, -4 , 2.5 ,2,7', '1,1e308,0,-0.0,3,8', '0,16777217,16777217,0.30000000000000004,4,9',
             '1,inf,-1,-inf,5,1', '0,nan,2,nan,6,2']


def test_a_double_and_an_int_field_feed_an_expression_and_a_raw_feature_from_one_parse(monkeypatch, tmp_path):
  """the native parser reads such a field once (int64 / float64 for the expression) and rounds it to float32 for the
  raw column, the reference's cast of an int / double field; the python engine reads the two separately"""
  host_doubles.install_all(monkeypatch.setattr)
  expr_doubles.install(monkeypatch.setattr)
  B = len(CSV_LINES)
  text = config('expr', B).replace(
      b'features { input_names: "r" feature_type: RawFeature }',
      b'features { input_names: "r" feature_type: RawFeature } '
      b'features { feature_name: "rx" input_names: "x" feature_type: RawFeature } '
      b'features { feature_name: "ry" input_names: "y" feature_type: RawFeature }').replace(
      b'feature_names: ["r", "c", "e1", "e2"]', b'feature_names: ["r", "rx", "ry", "c", "e1", "e2"]')
  cfg = config_util.get_configs_from_pipeline_file(text)
  il, _, _ = builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  path = _write_csv(tmp_path / 'a.csv', CSV_LINES)
  got = [list(readers.CSVInput(cfg, il, path, engine=e).batches())[0][0] for e in ('native', 'python')]
  x = got[0]['expr_fea'].numpy()
  for feats in got:
    assert np.array_equal(feats['expr_fea'].numpy().view(np.uint64), x.view(np.uint64))
    for name, k in (('rx', 0), ('ry', 1)):
      c0 = il.raw_cols[name][0]
      assert np.array_equal(feats['dense_fea'].numpy()[:, c0], x[:, k].astype(np.float32), equal_nan=True), name


def test_csv_engines_and_parquet_deliver_the_same_float64_inputs(monkeypatch, tmp_path):
  host_doubles.install_all(monkeypatch.setattr)
  expr_doubles.install(monkeypatch.setattr)
  B = len(CSV_LINES)
  cfg = config_util.get_configs_from_pipeline_file(config('expr', B))
  il, _, _ = builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  path = _write_csv(tmp_path / 'a.csv', CSV_LINES)
  want = np.array([[0.1, 3, 1e3], [1.5, 7, 3.25], [-0.0, 9007199254740992.0, 9007199254740993.0],
                   [2.5e-310, -4, 2.5], [1e308, 0, -0.0], [16777217, 16777217, 0.30000000000000004],
                   [np.inf, -1, -np.inf], [np.nan, 2, np.nan]], np.float64)
  got = {}
  for engine in ('native', 'python'):
    (feats, labels), = list(readers.CSVInput(cfg, il, path, engine=engine).batches())
    got[engine] = feats['expr_fea'].numpy()
    assert got[engine].dtype == np.float64 and got[engine].shape == (B, 3)
  pa = pytest.importorskip('pyarrow')
  import pyarrow.parquet as pq
  cols = [l.split(',') for l in CSV_LINES]
  table = pa.table({'label': pa.array([float(c[0]) for c in cols], pa.float32()),
                    'x': pa.array([float(c[1]) if c[1] else None for c in cols], pa.float64()),
                    'y': pa.array([int(c[2]) if c[2] else None for c in cols], pa.int64()),
                    'z': pa.array([c[3] for c in cols], pa.string()),
                    'r': pa.array([float(c[4]) for c in cols], pa.float32()),
                    'c': pa.array([int(c[5]) for c in cols], pa.int64())})
  pq.write_table(table, str(tmp_path / 'a.parquet'))
  pcfg = config_util.get_configs_from_pipeline_file(config('expr', B, input_type='ParquetInput'))
  (feats, labels), = list(readers.ParquetInput(pcfg, il, str(tmp_path / 'a.parquet')).batches())
  got['parquet'] = feats['expr_fea'].numpy()
  for k, v in got.items():
    # (Parquet's null x / y: the column default, as an empty CSV field)
    assert np.array_equal(v.view(np.uint64), want.view(np.uint64)), (k, v)


@pytest.mark.parametrize('engine', ['native', 'python'])
def test_a_value_that_is_not_a_number_raises_naming_the_field(monkeypatch, tmp_path, engine):
  host_doubles.install_all(monkeypatch.setattr)
  expr_doubles.install(monkeypatch.setattr)
  cfg = config_util.get_configs_from_pipeline_file(config('expr', 2))
  il, _, _ = builder.build_model(cfg, 2, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  for bad in ('1,0,0,abc,0,0', '1,0,0,0x10,0,0', '1,0,1.5,0,0,0'):
    path = _write_csv(tmp_path / 'b.csv', ['1,0,0,1,0,0', bad])
    with pytest.raises((ValueError, RuntimeError), match=r'field (z|y)|input field (z|y)'):
      list(readers.CSVInput(cfg, il, path, engine=engine).batches())
  # an empty STRING field whose default is '' is not a number either (string_to_number(''))
  text = config('expr', 2).replace(b'default_val: "3.25"', b'')
  cfg = config_util.get_configs_from_pipeline_file(text)
  path = _write_csv(tmp_path / 'c.csv', ['1,0,0,1,0,0', '1,0,0,,0,0'])
  with pytest.raises((ValueError, RuntimeError), match='z'):
    list(readers.CSVInput(cfg, il, path, engine=engine).batches())


@pytest.mark.parametrize('extra, fragment', [
    ('embedding_dim: 4', 'embedding_dim'), ('boundaries: [1.0, 2.0]', 'boundaries'),
    ('hash_bucket_size: 10', 'hash_bucket_size'), ('vocab_list: ["a"]', 'vocab_list'),
])
def test_options_the_reference_ignores_are_refused_by_name(extra, fragment):
  cfg = config_util.get_configs_from_pipeline_file(config('expr', 4, feature=extra))
  with pytest.raises((NotImplementedError, ValueError), match=r'(?s)e1.*%s' % fragment):
    builder.feature_specs(cfg)


def test_bad_expressions_and_inputs_are_refused_by_name():
  for text, fragment in ((b'expression: "x*y+z"', "'w' is not one of input_names"),
                         (b'input_names: ["x", "y", "z"] feature_type: ExprFeature expression: "x*y+z"',
                          'input q is not an input field')):
    src = config('expr', 4)
    if fragment.startswith("'w'"):
      src = src.replace(text, b'expression: "x*y+w"')
    else:
      src = src.replace(text, b'input_names: ["x", "q"] feature_type: ExprFeature expression: "x>q"')
    with pytest.raises(ValueError, match=re.escape(fragment)):
      builder.feature_specs(config_util.get_configs_from_pipeline_file(src))
  # without feature_name the reference stores the value under '' and names the column input_names[0]: refused
  src = config('expr', 4).replace(b'feature_name: "e2" ', b'')
  with pytest.raises(ValueError, match=r"ExprFeature x \(expression 'x\*y\+z'\) has no feature_name"):
    builder.feature_specs(config_util.get_configs_from_pipeline_file(src))
  src = config('expr', 4).replace(b'expression: "x*y+z"', b'')
  with pytest.raises(ValueError, match='ExprFeature e2 has no expression'):
    builder.feature_specs(config_util.get_configs_from_pipeline_file(src))
  cfg = config_util.get_configs_from_pipeline_file(b'''
data_config { batch_size: 4 input_type: CriteoInput label_fields: "label"
  input_fields { input_name: "label" input_type: INT32 } input_fields { input_name: "f1" input_type: FLOAT }
  input_fields { input_name: "f2" input_type: FLOAT } }
feature_config { features { input_names: "f1" feature_type: RawFeature }
  features { feature_name: "e" input_names: ["f1", "f2"] feature_type: ExprFeature expression: "f1>f2" } }
model_config { model_class: "WideAndDeep" feature_groups { group_name: "deep" feature_names: ["f1", "e"] wide_deep: DEEP }
  wide_and_deep { dnn { hidden_units: [4] } } }''')
  with pytest.raises(NotImplementedError, match='feature e: a ExprFeature'):
    readers.criteo_columns(cfg, None)


def test_a_host_device_without_the_kernel_double_is_refused(monkeypatch):
  host_doubles.install_all(monkeypatch.setattr)
  cfg = config_util.get_configs_from_pipeline_file(config('expr', 4))
  with pytest.raises(NotImplementedError, match='er_expr_eval on the GPU'):
    builder.build_model(cfg, 4, 'cpu', cpu_generator=torch.Generator().manual_seed(0))


def test_the_reference_expr_config_builds_trains_and_evaluates(monkeypatch):
  from easyrec_b200.estimator import EasyRecEstimator
  from test_config import reference_configs
  host_doubles.install_all(monkeypatch.setattr)
  expr_doubles.install(monkeypatch.setattr)
  text, = [t for p, t in reference_configs().items() if os.path.basename(p) == 'multi_tower_on_taobao_for_expr.config']
  cfg = config_util.get_configs_from_pipeline_file(text)
  est = EasyRecEstimator(cfg, device='cpu', seed=1, batch_size=8)
  il = est.input_layer
  assert il.expr_inputs == ['age_level', 'item_age_level']
  assert [e.kind for e in il.group_layout['combo']][-5:] == ['dense'] * 5
  feats, labels = readers.DummyInput(il, seed=3).batch()
  l0, _ = est.trainer.train_step(feats, labels)
  l1, _ = est.trainer.train_step(feats, labels)
  assert np.isfinite(float(l0)) and np.isfinite(float(l1))
  # the five columns hold the expressions of the batch's inputs
  x = feats['expr_fea'].numpy()
  a, i = x[:, 0], x[:, 1]
  want = np.stack([a >= 1, a < i + 5, a == i, (a >= i) & (a <= i + 5), (a >= i) | (a > 5)], 1).astype(np.float32)
  c0 = il.raw_cols['age_satisfy1'][0]
  assert np.array_equal(feats['dense_fea'].numpy()[:, c0:c0 + 5], want)
  ev = est.evaluate(lambda: [(feats, labels)])
  assert 'auc' in ev and np.isfinite(ev['auc'])
