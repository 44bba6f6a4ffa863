"""CPU: the non-relu activations (utils/activation.py:66-118) and the streaming evaluation metrics
(model/rank_model.py:334-496, core/metrics.py:25-56) - oracle restatements against known answers and independent
implementations, and the host logic around the kernels (layers.DNN / keras MLP activation wiring, metrics.MetricSet,
EasyRecEstimator.evaluate) with kernel doubles."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import host_doubles
from easyrec_b200 import builder, kernels as K, layers as L, metrics as M
from easyrec_b200.config import config_util, proto_loader
from oracle import oracle as O


@pytest.fixture
def doubles(monkeypatch):
  host_doubles.install_all(monkeypatch.setattr)


TORCH_ACT = {
    'gelu': lambda x: F.gelu(x, approximate='tanh'), 'leaky_relu': lambda x: F.leaky_relu(x, 0.2), 'elu': F.elu,
    'selu': F.selu, 'tanh': torch.tanh, 'swish': F.silu, 'sigmoid': torch.sigmoid}


def test_oracle_activations_known_answers():
  # closed forms at x = 1 / -1 (gelu: the tanh form the reference defines itself, activation.py:46-60)
  assert O.activation(1.0, 'gelu') == pytest.approx(0.8411919906082768, abs=1e-12)
  assert O.activation(-1.0, 'gelu') == pytest.approx(-0.15880800939172324, abs=1e-12)
  assert O.activation(-1.0, 'leaky_relu') == pytest.approx(-0.2) and O.activation(2.0, 'prelu') == 2.0
  assert O.activation(-1.0, 'elu') == pytest.approx(np.expm1(-1.0))
  assert O.activation(-1.0, 'selu') == pytest.approx(-1.1113307378125625, abs=1e-12)
  assert O.activation(1.0, 'selu') == pytest.approx(1.0507009873554805, abs=1e-15)
  assert O.activation(1.0, 'swish') == pytest.approx(0.7310585786300049, abs=1e-12)
  assert O.activation(0.5, 'tanh') == pytest.approx(np.tanh(0.5)) and O.activation(0.0, 'sigmoid') == 0.5


@pytest.mark.parametrize('name', sorted(TORCH_ACT))
def test_oracle_activations_match_torch_values_and_gradients(name):
  rng = np.random.default_rng(1)
  x = np.concatenate([rng.normal(0, 2, 4000), [0.0, -0.0, 1e-8, -1e-8, 20.0, -20.0]])
  xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
  y = TORCH_ACT[name](xt)
  y.sum().backward()
  np.testing.assert_allclose(O.activation(x, name), y.detach().numpy(), rtol=1e-12, atol=1e-14)
  g = O.activation_grad(x, name)
  nz = x != 0   # (at exactly 0 the one-sided conventions differ between frameworks: TF's are restated, not torch's)
  np.testing.assert_allclose(g[nz], xt.grad.numpy()[nz], rtol=1e-10, atol=1e-13)
  # TF's gradient kernels at 0: EluGrad / SeluGrad take the positive branch for out >= 0, LeakyReluGrad alpha for x <= 0
  at0 = {'elu': 1.0, 'selu': 1.0507009873554805, 'leaky_relu': 0.2}.get(name)
  if at0 is not None:
    assert O.activation_grad(0.0, name) == pytest.approx(at0)


def test_activation_names_resolve_like_get_activation():
  assert L.activation_kind('tf.nn.relu') == 'relu' and L.activation_kind('relu') == 'relu'
  assert L.activation_kind('') is None and L.activation_kind('linear') is None and L.activation_kind(None) is None
  assert L.activation_kind('tf.nn.tanh') == K.ACT_KINDS['tanh'] == L.activation_kind('Tanh')
  assert L.activation_kind('prelu') == L.activation_kind('tf.nn.leaky_relu') == K.ACT_KINDS['leaky_relu']
  assert L.activation_kind('gelu') == K.ACT_KINDS['gelu'] and L.activation_kind('tf.nn.swish') == K.ACT_KINDS['swish']
  assert L.activation_kind('dice') == L.activation_kind('Dice') == 'dice'
  with pytest.raises(NotImplementedError):
    L.activation_kind('softmax')


@pytest.mark.parametrize('name', ['gelu', 'selu', 'tanh'])
def test_dnn_with_a_configured_activation_trains_like_plain_torch(doubles, name):
  """layers.DNN built from a DNN message with `activation` set: the dense / batch-norm stage runs linear, the
  activation is the elementwise pass on top, dropout-free; forward and every gradient equal plain torch autograd."""
  msg = proto_loader.default_schema().DNN()
  msg.hidden_units.extend([12, 6])
  msg.activation = name
  units = L.units_of(msg)
  assert units.activation == name and units[:-1].activation == name
  g = torch.Generator().manual_seed(0)
  dnn = L.DNN(9, units, generator=g)
  dnn.train()
  x = torch.randn(32, 9, generator=g, requires_grad=True)
  y = dnn(x)
  gy = torch.randn(y.shape, generator=g)
  y.backward(gy)
  # plain torch restatement on the same parameters
  xr = x.detach().clone().requires_grad_(True)
  h = xr
  params = []
  for lay in dnn.layers:
    W, b = lay.kernel.detach().clone().requires_grad_(True), lay.bias.detach().clone().requires_grad_(True)
    ga, be = lay.gamma.detach().clone().requires_grad_(True), lay.beta.detach().clone().requires_grad_(True)
    params.append((lay, W, b, ga, be))
    z = h @ W + b
    mu, var = z.mean(0), ((z - z.mean(0)) ** 2).mean(0)
    h = TORCH_ACT[name]((z - mu) / torch.sqrt(var + 1e-3) * ga + be)
  h.backward(gy)
  assert torch.allclose(y, h, atol=1e-5)
  assert torch.allclose(x.grad, xr.grad, atol=1e-4)
  for lay, W, b, ga, be in params:
    assert torch.allclose(lay.kernel.grad, W.grad, atol=1e-4) and torch.allclose(lay.gamma.grad, ga.grad, atol=1e-4)


CFG_ACT = b'''
train_config { optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.05 } } } } }
eval_config { metrics_set { auc { num_thresholds: 500 } } metrics_set { max_f1 {} } metrics_set { mean_squared_error {} }
  metrics_set { mean_absolute_error {} } metrics_set { root_mean_squared_error {} } }
data_config { batch_size: 256 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "a" input_type: INT64 }
  input_fields { input_name: "b" input_type: INT64 } }
feature_config {
  features { input_names: "a" feature_type: IdFeature embedding_dim: 8 num_buckets: 50 }
  features { input_names: "b" feature_type: IdFeature embedding_dim: 8 num_buckets: 50 } }
model_config { model_class: "MultiTower"
  feature_groups { group_name: "g" feature_names: ["a", "b"] wide_deep: DEEP }
  multi_tower { towers { input: "g" dnn { hidden_units: [16] activation: "ACT" } }
                final_dnn { hidden_units: [8] activation: "tf.nn.tanh" } l2_regularization: 1e-6 } }
'''


def _batches(n, B, seed):
  rng = np.random.default_rng(seed)
  for _ in range(n):
    a, b = rng.integers(0, 50, B), rng.integers(0, 50, B)
    lab = ((a + b) % 2 == 0).astype(np.float32)
    yield {'sparse_fea': torch.from_numpy(np.concatenate([a, b]).astype(np.int64))}, torch.from_numpy(lab)


@pytest.mark.parametrize('act', ['gelu', 'swish'])
def test_config_with_activations_trains_and_evaluates_streaming_metrics(doubles, act):
  from easyrec_b200.estimator import EasyRecEstimator
  est = EasyRecEstimator(CFG_ACT.replace(b'ACT', act.encode()), device='cpu', seed=3)
  tower = est.model.tower_dnn[0]
  assert isinstance(tower.acts[0], L.Activation) and tower.acts[0].kind == K.ACT_KINDS[act]
  assert est.model.final_dnn.acts[0].kind == K.ACT_KINDS['tanh'] and not tower.layers[0].relu
  first = est.train(lambda: _batches(1, 256, 0), steps=1)
  last = est.train(lambda: _batches(150, 256, 1), steps=150)
  assert last < first - 0.1, (first, last)
  # evaluate: the streaming metrics against the oracle's definitions over the same predictions
  ev = est.evaluate(lambda: _batches(6, 256, 99))
  logits, labels = [], []
  for f, l in _batches(6, 256, 99):
    logits.append(est._forward_eval(f).numpy())
    labels.append(l.numpy())
  logits, labels = np.concatenate(logits), np.concatenate(labels)
  probs = 1.0 / (1.0 + np.exp(-logits.astype(np.float64)))
  assert ev['auc'] == pytest.approx(O.auc_tf(labels, probs.astype(np.float32), 500), abs=2e-6)
  assert ev['max_f1'] == pytest.approx(O.max_f1(labels, logits), abs=1e-6)
  assert ev['mean_squared_error'] == pytest.approx(np.mean((labels - probs) ** 2), rel=1e-5)
  assert ev['mean_absolute_error'] == pytest.approx(np.mean(np.abs(labels - probs)), rel=1e-5)
  assert ev['root_mean_squared_error'] == pytest.approx(np.sqrt(np.mean((labels - probs) ** 2)), rel=1e-5)
  assert abs(ev['auc'] - ev['auc_exact']) < 5e-3 and ev['auc_exact'] > 0.9


def test_unknown_activations_are_refused_by_the_scope_check():
  cfg = config_util.get_configs_from_pipeline_file(CFG_ACT.replace(b'ACT', b'softmax'))
  with pytest.raises(NotImplementedError, match='softmax'):
    builder.check_scope(cfg)
  builder.check_scope(config_util.get_configs_from_pipeline_file(CFG_ACT.replace(b'ACT', b'dice')))


def test_dice_reproduces_the_reference_function_and_its_gradients(doubles, native):
  """layers.Dice against utils/activation.py:dice executed (tests/golden/reference_activations.json), its backward
  against torch autograd of the restatement, the moving statistics it keeps for evaluation, and the kernels' own gate
  formulas (elementwise.cuh compiled for the CPU) against the same numbers."""
  import ctypes
  d = _act_gold()['cases']['dice']
  x = torch.tensor(d['x'], dtype=torch.float32)
  alphas = torch.tensor(d['alphas'], dtype=torch.float32)
  m = L.Dice(3)
  with torch.no_grad():
    m.alphas.copy_(alphas)
  m.train()
  xi = x.clone().requires_grad_(True)
  y = m(xi)
  np.testing.assert_allclose(y.detach().numpy(), np.array(d['y'], np.float32), rtol=1e-5, atol=1e-6)
  gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(0))
  y.backward(gy)
  xr = x.clone().requires_grad_(True)
  ar = alphas.clone().requires_grad_(True)
  mu, var = xr.mean(0), ((xr - xr.mean(0)) ** 2).mean(0)
  p = torch.sigmoid((xr - mu) / torch.sqrt(var + 1e-9))
  (ar * (1 - p) * xr + p * xr).backward(gy)
  assert torch.allclose(xi.grad, xr.grad, atol=1e-5) and torch.allclose(m.alphas.grad, ar.grad, atol=1e-5)
  # moving statistics (momentum 0.99) feed the evaluation mode
  np.testing.assert_allclose(m.moving_mean.numpy(), 0.01 * x.mean(0).numpy(), rtol=1e-5, atol=1e-7)
  m.eval()
  pe = torch.sigmoid((x - m.moving_mean) / torch.sqrt(m.moving_var + 1e-9))
  assert torch.allclose(m(x), alphas * (1 - pe) * x + pe * x, atol=1e-6)
  # the kernel source's gate given xn: same value, same three gradient terms
  xn = ((x - x.mean(0)) / torch.sqrt(((x - x.mean(0)) ** 2).mean(0) + 1e-9)).numpy().astype(np.float32)
  xv, al = x.numpy().reshape(-1), np.tile(alphas.numpy(), x.shape[0])
  out = np.empty((4, xv.size), np.float32)
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
  gyv = gy.numpy().reshape(-1).copy()
  native.host_dice(vp(xv.copy()), vp(xn.reshape(-1).copy()), vp(al.copy()), vp(gyv), ctypes.c_long(xv.size), vp(out))
  np.testing.assert_allclose(out[0].reshape(x.shape), np.array(d['y'], np.float32), rtol=1e-5, atol=1e-6)
  pn = 1.0 / (1.0 + np.exp(-xn.reshape(-1).astype(np.float64)))
  np.testing.assert_allclose(out[1], gyv * (al * (1 - pn) + pn), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(out[2], gyv * xv * (1 - al) * pn * (1 - pn), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(out[3], gyv * xv * (1 - pn), rtol=1e-5, atol=1e-6)


def test_config_with_dice_trains(doubles):
  from easyrec_b200.estimator import EasyRecEstimator
  est = EasyRecEstimator(CFG_ACT.replace(b'ACT', b'dice'), device='cpu', seed=3)
  dice = est.model.tower_dnn[0].acts[0]
  assert isinstance(dice, L.Dice) and dice.units == 16 and 'tower_dnn.0.acts.0.alphas' in dict(est.model.named_parameters())
  first = est.train(lambda: _batches(1, 256, 0), steps=1)
  last = est.train(lambda: _batches(150, 256, 1), steps=150)
  assert last < first - 0.1 and float(dice.alphas.abs().max()) > 0      # the alphas are trained with the towers
  ev = est.evaluate(lambda: _batches(4, 256, 99))
  assert ev['auc_exact'] > 0.9


# ---- tf.metrics.auc / max_f1 ---------------------------------------------------------------------------------------
def test_oracle_auc_reproduces_tensorflows_own_test_values():
  """tensorflow/python/kernel_tests/metrics_test.py, AUCTest (values recalled from the TF source tree, TF is not
  installable here): testAllCorrect 1, testSomeCorrect 0.5, testAllIncorrect 0, testZeroTruePositivesAndFalseNegatives-
  GivesOneAUC 1 - all with the default 200 thresholds."""
  assert O.auc_tf([0, 1, 1, 0], [0, 1, 1, 0]) == pytest.approx(1.0, abs=1e-6)
  assert O.auc_tf([0, 1, 1, 0], [1, 0, 1, 0]) == pytest.approx(0.5, abs=1e-6)
  assert O.auc_tf([1, 0, 0, 1], [0, 1, 1, 0]) == pytest.approx(0.0, abs=1e-5)
  assert O.auc_tf(np.zeros(4), np.zeros(4)) == pytest.approx(1.0, abs=1e-6)
  t = O.tf_thresholds(200)
  assert t.dtype == np.float32 and len(t) == 200 and t[0] < 0 < t[1] and t[-2] < 1 < t[-1]
  assert t[1] == np.float32(1.0 / 199) and np.all(np.diff(t) > 0)


def test_thresholded_auc_approaches_the_exact_auc():
  rng = np.random.default_rng(5)
  lab = rng.random(50000) < 0.3
  p = np.clip(rng.normal(0.4 + 0.25 * lab, 0.2), 0, 1).astype(np.float32)
  exact = M.auc(lab, p)
  assert abs(O.auc_tf(lab, p, 200) - exact) < 1e-3
  assert abs(O.auc_tf(lab, p, 2000) - exact) < 1e-4


@pytest.mark.parametrize('T', [2, 200, 4095])
def test_streaming_confusion_counts_equal_the_definition(doubles, T):
  rng = np.random.default_rng(T)
  thr = O.tf_thresholds(T)
  assert np.array_equal(M.tf_thresholds(T), thr)
  # predictions sitting exactly on thresholds, outside [0, 1], NaN; labels that truncate to 0 (0.5) and to 1 (1.7)
  p = np.concatenate([rng.random(5000).astype(np.float32), thr[rng.integers(0, T, 500)],
                      np.array([0.0, 1.0, -0.5, 1.5, np.nan], np.float32)])
  lab = rng.choice(np.array([0.0, 1.0, 0.5, 1.7, -1.0], np.float32), p.size)
  acc = M.ConfusionAtThresholds(T, 'cpu')
  order = rng.permutation(p.size)
  for part in np.array_split(order, 7):   # any batching, any order: integer counters
    acc.update(torch.from_numpy(p[part]), torch.from_numpy(lab[part]))
  want = O.confusion_at_thresholds(lab, p, T)
  for got, w in zip(acc.counts(), want):
    assert np.array_equal(got, w.astype(np.float32))
  assert acc.auc() == pytest.approx(O.auc_tf(lab, p, T), abs=1e-6)
  if T == 200:
    assert acc.max_f1() == pytest.approx(O.max_f1(lab, p), abs=1e-7)
  with pytest.raises(ValueError):
    M.tf_thresholds(4096)


def test_metric_set_over_task_towers_uses_each_towers_label_and_loss_type(doubles):
  schema = proto_loader.default_schema()
  ms = []
  for kind in ('auc', 'mean_squared_error'):
    m = schema.EvalMetrics()
    getattr(m, kind).SetInParent()
    ms.append(m)
  heads = [('_ctr', 'CLASSIFICATION', 1), ('_cvr', 'CLASSIFICATION', 0)]
  mset = M.MetricSet(ms, heads, 'cpu')
  rng = np.random.default_rng(0)
  logits = torch.from_numpy(rng.normal(size=(4000, 2)).astype(np.float32))
  labels = torch.from_numpy((rng.random((4000, 2)) < 0.4).astype(np.float32))
  for i in range(0, 4000, 1000):
    mset.update(logits[i:i + 1000], labels[i:i + 1000])
  out = mset.result()
  probs = torch.sigmoid(logits).numpy()
  assert sorted(out) == ['auc_ctr', 'auc_cvr', 'mean_squared_error_ctr', 'mean_squared_error_cvr']
  assert out['auc_ctr'] == pytest.approx(O.auc_tf(labels[:, 1].numpy(), probs[:, 0]), abs=1e-6)
  assert out['auc_cvr'] == pytest.approx(O.auc_tf(labels[:, 0].numpy(), probs[:, 1]), abs=1e-6)
  assert out['mean_squared_error_cvr'] == pytest.approx(np.mean((labels[:, 0].numpy() - probs[:, 1]) ** 2), rel=1e-5)
  # an L2 head reads `y` = the logits and has no auc
  reg = M.MetricSet(ms[1:], [('', 'L2_LOSS', None)], 'cpu')
  reg.update(logits[:, 0], labels[:, 0])
  assert reg.result()['mean_squared_error'] == pytest.approx(np.mean((labels[:, 0].numpy() - logits[:, 0].numpy()) ** 2), rel=1e-5)
  with pytest.raises(ValueError):
    M.MetricSet(ms[:1], [('', 'L2_LOSS', None)], 'cpu')


# ---- the kernels' own source, compiled for the CPU ------------------------------------------------------------------
@pytest.fixture(scope='module')
def native(tmp_path_factory):
  """easyrec_b200/csrc/elementwise.cuh (the formulas the kernels are built from) compiled by g++ into a scratch .so"""
  import ctypes
  import os
  import subprocess
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  so = str(tmp_path_factory.mktemp('native') / 'elementwise_host.so')
  subprocess.check_call(['g++', '-O2', '-shared', '-fPIC', '-x', 'c++', '-I', os.path.join(root, 'include'),
                         '-I', os.path.join(root, 'easyrec_b200', 'csrc'),
                         os.path.join(root, 'tests', 'native', 'elementwise_host.cpp'), '-o', so])
  return ctypes.CDLL(so)


@pytest.mark.parametrize('name', sorted(TORCH_ACT))
def test_kernel_source_activation_formulas_match_the_oracle(native, name):
  import ctypes
  rng = np.random.default_rng(2)
  x = np.concatenate([rng.normal(0, 3, 20000), np.linspace(-30, 30, 2001), [0.0, -0.0, 88.0, -88.0, 1e-20]]).astype(np.float32)
  y, g = np.empty_like(x), np.empty_like(x)
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
  assert native.host_act(K.ACT_KINDS[name], vp(x), ctypes.c_long(x.size), vp(y), vp(g)) == 0
  want, want_g = O.activation(x, name), O.activation_grad(x, name)
  np.testing.assert_allclose(y, want, rtol=2e-6, atol=1e-7)
  np.testing.assert_allclose(g, want_g, rtol=4e-6, atol=1e-6)   # (1 - tanh^2 cancels in fp32 where the slope vanishes)
  assert np.isfinite(y).all() and np.isfinite(g).all()


@pytest.mark.parametrize('T', [2, 200, 4095])
def test_kernel_source_threshold_binning_matches_the_definition(native, T):
  import ctypes
  rng = np.random.default_rng(T + 1)
  thr = O.tf_thresholds(T)
  p = np.concatenate([rng.random(20000).astype(np.float32), thr, np.nextafter(thr, np.float32(2)), np.nextafter(thr, np.float32(-1)),
                      np.array([0.0, 1.0, -3.0, 7.0, np.nan, np.inf, -np.inf], np.float32)])
  lab = rng.choice(np.array([0.0, 1.0, 0.5, 1.7, -1.0, -0.5], np.float32), p.size)
  hist = np.zeros(2 * (T + 1), np.uint64)
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
  native.host_auc_hist(vp(p), vp(lab), ctypes.c_long(p.size), vp(thr), T, vp(hist))
  neg, pos = np.cumsum(hist[:T + 1].astype(np.int64)), np.cumsum(hist[T + 1:].astype(np.int64))
  tp, fn, tn, fp = O.confusion_at_thresholds(lab, p, T)
  assert np.array_equal(pos[-1] - pos[:T], tp) and np.array_equal(neg[-1] - neg[:T], fp)
  assert pos[-1] == tp[0] + fn[0] and neg[-1] == fp[0] + tn[0]


# ---- RawFeature.normalizer_fn (input/input.py:133-137, 642-646) -----------------------------------------------------
CFG_NORM = b'''
data_config { batch_size: 4 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "a" input_type: FLOAT }
  input_fields { input_name: "b" input_type: FLOAT } input_fields { input_name: "c" input_type: FLOAT } }
feature_config {
  features { input_names: "a" feature_type: RawFeature embedding_dim: 4 min_val: 0.0 max_val: 10.0
             normalizer_fn: "lambda x: tf.math.log1p(tf.maximum(x, 0.0))" }
  features { input_names: "b" feature_type: RawFeature embedding_dim: 4 normalizer_fn: "tf.math.sqrt" }
  features { input_names: "c" feature_type: RawFeature embedding_dim: 4 boundaries: [0.5, 1.0, 1.5]
             normalizer_fn: "tf.math.log1p" } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["a", "b", "c"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["c"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [8] } final_dnn { hidden_units: [4] } } }
'''


def test_raw_feature_normalizer_fn_on_the_device_matrix_and_in_the_host_bucketizer(doubles, tmp_path):
  from easyrec_b200 import normalizer
  from easyrec_b200.input import readers
  cfg = config_util.get_configs_from_pipeline_file(CFG_NORM)
  il, _, _ = builder.build_model(cfg, 4, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  assert sorted(il.raw_normalizers) == ['a', 'b']          # `c` is bucketized by the reader, with its normalizer
  a, b, c = [5.0, -2.0, 10.0, 0.0], [4.0, 0.25, 9.0, 0.0], [0.1, 0.7, 2.0, 5.0]
  open(tmp_path / 'n.csv', 'w').write(''.join('1,%g,%g,%g\n' % r for r in zip(a, b, c)))
  (feats, _), = list(readers.CSVInput(cfg, il, str(tmp_path / 'n.csv')))
  # host: log1p(c) against the boundaries -> bucket ids of the `c` slot (the last single-valued slot)
  want_c = np.searchsorted(np.array([0.5, 1.0, 1.5], np.float32), np.log1p(np.array(c, np.float32)), side='right')
  assert feats['sparse_fea'].tolist() == want_c.tolist()
  # device side: the dense matrix after min-max and the normalizers
  dn = il.normalize_dense(feats['dense_fea'])
  np.testing.assert_allclose(dn[:, 0].numpy(), np.log1p(np.maximum(np.array(a, np.float32) / 10.0, 0.0)), rtol=1e-6)
  np.testing.assert_allclose(dn[:, 1].numpy(), np.sqrt(np.array(b, np.float32)), rtol=1e-6)
  assert feats['dense_fea'][:, 1].tolist() == b             # the reader's batch itself is left untouched
  # ... and they reach the projection: out = normalised value * the one-row table
  out = il.lookup(feats)['deep'][0]
  t = il.arenas[4]
  off_a = t.tables[[k for k in t.tables if k.endswith('a_embedding') or '/a' in k][0]][0]
  np.testing.assert_allclose(out[:, :4].detach().numpy(), dn[:, :1].numpy() * t.weight[off_a:off_a + 1].numpy(), rtol=1e-5, atol=1e-7)
  # both backends of one expression agree; unknown tf calls are refused, not guessed
  f_np, f_t = normalizer.load('lambda x: tf.clip_by_value(x * 2.0, 0.0, 1.0)', 'numpy'), \
      normalizer.load('lambda x: tf.clip_by_value(x * 2.0, 0.0, 1.0)', 'torch')
  x = np.linspace(-1, 1, 9).astype(np.float32)
  assert np.array_equal(f_np(x), f_t(torch.from_numpy(x)).numpy())
  with pytest.raises(NotImplementedError):
    normalizer.load('tf.signal.fft', 'numpy')


# ---- er_gemm_small (vector-sized dense layers: MMoE gates, their dX and dW) -------------------------------------------
@pytest.mark.parametrize('M,N,K,form', [(8192, 4, 256, 'fwd'), (8192, 256, 4, 'dx'), (256, 4, 8192, 'dw'), (3, 5, 7, 'fwd'),
                                        (1000, 7, 33, 'fwd'), (33, 7, 1000, 'dw'), (5, 300, 2, 'dx'), (64, 3, 511, 'dw'),
                                        (64, 3, 512, 'dw'), (16384, 3, 96, 'fwd'), (96, 3, 16384, 'dw')])
def test_kernel_source_small_gemm_reads_strided_operands_and_sums_slices_in_order(native, M, N, K, form):
  """small_gemm.cuh compiled for the CPU, driven with the strides kernels.gemm_small passes for the three forms of a
  dense layer: forward (X row-major, W row-major), dX (dY, W^T as a transposed VIEW), dW (X^T as a view, dY)."""
  import ctypes
  rng = np.random.default_rng(M + N + K)
  if form == 'fwd':
    a = torch.from_numpy(rng.normal(size=(M, K + 3)).astype(np.float32))[:, :K]      # a pitched view
    b = torch.from_numpy(rng.normal(size=(K, N)).astype(np.float32))
  elif form == 'dx':
    a = torch.from_numpy(rng.normal(size=(M, K)).astype(np.float32))
    b = torch.from_numpy(rng.normal(size=(N, K)).astype(np.float32)).t()             # W^T read in place
  else:
    a = torch.from_numpy(rng.normal(size=(K, M)).astype(np.float32)).t()             # X^T read in place
    b = torch.from_numpy(rng.normal(size=(K, N)).astype(np.float32))
  bias = torch.from_numpy(rng.normal(size=N).astype(np.float32)) if form == 'fwd' else None
  out = torch.full((M, N + 2), float('nan'))
  L = ctypes.c_long
  native.host_gemm_small.restype = ctypes.c_long
  n_slice = native.host_gemm_small(
      ctypes.c_void_p(a.data_ptr()), L(a.stride(0)), L(a.stride(1)), ctypes.c_void_p(b.data_ptr()), L(b.stride(0)),
      L(b.stride(1)), ctypes.c_void_p(bias.data_ptr() if bias is not None else None), ctypes.c_void_p(out.data_ptr()),
      L(out.stride(0)), L(M), L(N), L(K))
  want = a.double() @ b.double() + (bias.double() if bias is not None else 0.0)
  scale = float(np.sqrt(K))
  assert float((out[:, :N].double() - want).abs().max()) < 6e-6 * scale + 2e-6
  assert torch.isnan(out[:, N:]).all()                       # nothing written beyond the N columns of a pitched output
  assert (n_slice > 1) == (K >= 512 and form == 'dw')         # only the long-K / few-output form is cut into slices
  from easyrec_b200 import _lib
  ws = _lib.load().er_gemm_small_workspace_bytes(M, N, K)
  assert ws == (n_slice * M * N * 4 if n_slice > 1 else 0)    # the library sizes the workspace for the same slicing


# ---- EasyRecEstimator.train(fetch_loss_every_step=True): the pipelined loss read ----------------------------------
def test_loss_reader_returns_every_steps_loss_one_step_behind_and_the_last_on_flush():
  from easyrec_b200 import estimator as E

  class FakeEvent(object):
    def __init__(self):
      self.recorded = self.synced = 0

    def record(self):
      self.recorded += 1

    def synchronize(self):
      assert self.recorded > self.synced     # never waits for an event that was not recorded since its last use
      self.synced = self.recorded

  r = E._LossReader('cpu')
  assert r.push(torch.tensor(0.5)) == 0.5 and r.flush() == 0.5      # host device: read directly
  r = E._LossReader.__new__(E._LossReader)                          # the CUDA branch over stand-in buffers / events
  r.cuda, r.k, r.value = True, 0, None
  r.buf = [torch.empty(1), torch.empty(1)]
  r.ev = [FakeEvent(), FakeEvent()]
  r.pending = [False, False]
  static = torch.zeros(())                                          # the graph's loss output: overwritten every step
  seen = []
  for k in range(7):
    static.fill_(10.0 + k)
    seen.append(r.push(static))
  assert seen == [None, 10.0, 11.0, 12.0, 13.0, 14.0, 15.0]          # one step behind, nothing skipped
  assert r.flush() == 16.0 and r.flush() == 16.0                    # the last step's value; idempotent
  assert [e.recorded for e in r.ev] == [4, 3] and [e.synced for e in r.ev] == [4, 3]


# ---- the reference's own activation code, executed (tests/golden/make_activation_golden.py) ---------------------------
def _act_gold():
  import json
  import os
  return json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_activations.json')))


def test_activations_reproduce_the_reference_functions_executed(native):
  """gelu / swish / dice as utils/activation.py computes them (function bodies run on a numpy shim): the oracle, and
  the kernels' own source compiled for the CPU, give the same values."""
  import ctypes
  g = _act_gold()
  x = np.array(g['x'], np.float32)
  for name in ('gelu', 'swish'):
    want = np.array(g['cases'][name]['y'], np.float32)
    np.testing.assert_allclose(O.activation(x, name), want, rtol=2e-6, atol=1e-7)
    y, s = np.empty_like(x), np.empty_like(x)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
    assert native.host_act(K.ACT_KINDS[name], vp(x), ctypes.c_long(x.size), vp(y), vp(s)) == 0
    np.testing.assert_allclose(y, want, rtol=2e-6, atol=1e-7)
  d = g['cases']['dice']
  np.testing.assert_allclose(O.dice(d['x'], d['alphas']), np.array(d['y'], np.float32), rtol=1e-5, atol=1e-6)


def test_activation_names_follow_get_activation_executed():
  """the config string -> function map recorded by running the reference's get_activation: every name it resolves to a
  stateless function resolves here to the same one; 'linear' / '' mean no activation."""
  tf_name = {'relu': 'tf.nn.relu', K.ACT_KINDS['gelu']: 'gelu', K.ACT_KINDS['leaky_relu']: 'tf.nn.leaky_relu',
             K.ACT_KINDS['elu']: 'tf.nn.elu', K.ACT_KINDS['selu']: 'tf.nn.selu', K.ACT_KINDS['tanh']: 'tf.tanh',
             K.ACT_KINDS['swish']: 'tf.nn.swish', K.ACT_KINDS['sigmoid']: 'tf.nn.sigmoid', None: None}
  for s, fn in _act_gold()['cases']['get_activation']['map'].items():
    got = tf_name[L.activation_kind(s)]
    if fn is not None and fn.startswith('load_by_path('):       # a dotted path: the function it names
      fn = fn[len('load_by_path('):-1].replace('tf.nn.tanh', 'tf.tanh')
    assert got == fn, (s, got, fn)


# ---- sequence_combiner { attention } of a SequenceFeature in a plain feature group (layers/input_layer.py:312-347) ---------
CFG_SEQC = b'''
train_config { optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.1 } } } } }
data_config { batch_size: 4 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "u" input_type: INT64 }
  input_fields { input_name: "zz" input_type: STRING } input_fields { input_name: "aa" input_type: STRING } }
feature_config {
  features { input_names: "zz" feature_type: SequenceFeature embedding_dim: 4 num_buckets: 9 separator: "|" max_seq_len: 3
             sequence_combiner { attention {} } }
  features { input_names: "u" feature_type: IdFeature embedding_dim: 4 num_buckets: 9 }
  features { input_names: "aa" feature_type: SequenceFeature embedding_dim: 4 num_buckets: 9 separator: "|" max_seq_len: 3
             sequence_combiner { attention {} } embedding_name: "zz_embedding" } }
model_config { model_class: "MultiTower"
  feature_groups { group_name: "g" feature_names: ["zz", "u", "aa"] wide_deep: DEEP }
  multi_tower { towers { input: "g" dnn { hidden_units: [8] } } final_dnn { hidden_units: [4] } }
  embedding_regularization: 1e-3 }
'''


def seqc_expected(il, feats):
  """numpy restatement of the group: plain features in config order, then the sequence-combiner features by NAME"""
  t = il.arenas[4]
  B = il.batch_size

  def rows(table, ids):
    off = t.tables[table][0]
    return t.weight[off:off + 9].detach().cpu().numpy()[ids]
  u = rows('u_embedding', feats['sparse_fea'].cpu().numpy())
  pooled, unpooled = {}, {}
  for name, table in (('aa', 'zz_embedding'), ('zz', 'zz_embedding')):
    ids, lens = [x.cpu().numpy() for x in feats['seq_fea'][name]]
    emb = rows(table, ids)                                       # [B, T, D]
    emb = emb * (np.arange(3)[None, :, None] < lens[:, None, None])   # steps beyond the length look up nothing
    w = il.attention_modules['g#seqc/' + name].kernel.detach().cpu().numpy()[:, 0]
    logit = emb @ w
    logit = np.where(np.arange(3)[None, :] < lens[:, None], logit, np.float32(-2.0 ** 32 + 1))
    p = np.exp(logit - logit.max(1, keepdims=True))
    p = p / p.sum(1, keepdims=True)
    pooled[name], unpooled[name] = (p[:, :, None] * emb).sum(1), emb
  return u, pooled, unpooled


def seqc_batch():
  return {'sparse_fea': torch.tensor([1, 5, 0, 8]),
          'seq_fea': {'zz': (torch.tensor([[1, 2, 3], [4, 0, 0], [7, 7, 0], [2, 5, 8]]), torch.tensor([3, 1, 2, 3], dtype=torch.int32)),
                      'aa': (torch.tensor([[8, 0, 0], [3, 3, 3], [1, 6, 0], [0, 0, 0]]), torch.tensor([1, 3, 2, 1], dtype=torch.int32))}}, \
      torch.tensor([1.0, 0.0, 0.0, 1.0])


def test_attention_sequence_combiner_in_a_plain_group(doubles):
  cfg = config_util.get_configs_from_pipeline_file(CFG_SEQC)
  il, model, _ = builder.build_model(cfg, 4, 'cpu', cpu_generator=torch.Generator().manual_seed(2))
  assert [e.name for e in il.group_layout['g']] == ['u', 'aa', 'zz']          # concat: plain features, then by name
  assert il.seqc_order['g'] == ['zz', 'aa']                                  # per-feature list: config order
  with torch.no_grad():
    for m in il.attention_modules.values():
      m.kernel.copy_(torch.randn(m.kernel.shape, generator=torch.Generator().manual_seed(5)))
      assert not m.bias.requires_grad and float(m.bias.abs().sum()) == 0.0   # use_bias=False
  feats, labels = seqc_batch()
  concat, per_feature = il.lookup(feats)['g']
  u, pooled, unpooled = seqc_expected(il, feats)
  np.testing.assert_allclose(concat.detach().numpy(), np.concatenate([u, pooled['aa'], pooled['zz']], 1), rtol=1e-5, atol=1e-6)
  for got, want in zip(per_feature, (u, pooled['zz'], pooled['aa'])):
    np.testing.assert_allclose(got.detach().numpy(), want, rtol=1e-5, atol=1e-6)
  # the embedding regulariser covers the looked-up tensors: u and the UN-POOLED sequences
  reg = concat._er_reg
  assert len(reg) == 3 and sorted(tuple(r.shape) for r in reg) == [(4, 3, 4), (4, 3, 4), (4, 4)]
  want_sq = (u ** 2).sum() + (unpooled['aa'] ** 2).sum() + (unpooled['zz'] ** 2).sum()
  assert float(sum((r * r).sum() for r in reg)) == pytest.approx(float(want_sq), rel=1e-5)
  il.discard_pending()
  # ... and the whole thing trains: table rows, attention vectors and towers move, the loss falls
  from easyrec_b200.estimator import EasyRecEstimator
  est = EasyRecEstimator(CFG_SEQC, device='cpu', seed=2)
  w0 = [m.kernel.detach().clone() for m in est.input_layer.attention_modules.values()]
  losses = [float(est.trainer.train_step(feats, labels)[0]) for _ in range(30)]
  assert losses[-1] < losses[0] - 0.05
  assert all(float((m.kernel - w).abs().max()) > 0 for m, w in zip(est.input_layer.attention_modules.values(), w0))
  # text_cnn (or a missing combiner) stays refused
  bad = config_util.get_configs_from_pipeline_file(CFG_SEQC.replace(b'sequence_combiner { attention {} } }', b'}', 1))
  with pytest.raises(NotImplementedError, match='sequence_combiner'):
    builder.build_model(bad, 4, 'cpu', cpu_generator=torch.Generator().manual_seed(2))


# ---- momentum_optimizer with momentum > 0 (builders/optimizer_builder.py:54-59 -> tf.train.MomentumOptimizer) -----------
def test_oracle_momentum_rule_reproduces_tensorflows_own_test_values():
  """tensorflow/python/training/momentum_test.py testBasic (recalled): lr 2.0, momentum 0.9, grads 0.1 / 0.01 -
  var0 [1, 2] -> [0.8, 1.8] -> 1 - 0.1*2 - (0.9*0.1 + 0.1)*2; var1 [3, 4] -> 3 - 0.01*2 - (0.9*0.01 + 0.01)*2."""
  table = np.array([[1.0, 2.0], [3.0, 4.0]], np.float32)
  acc = np.zeros_like(table)
  g = np.array([[0.1, 0.1], [0.01, 0.01]], np.float32)
  rows, seg = np.array([0, 1], np.int64), np.arange(2, dtype=np.int32)
  O.embedding_bwd(table, acc, None, rows, seg, g, O.OPT_MOMENTUM, 2.0, beta1=0.9)
  np.testing.assert_allclose(table, [[0.8, 1.8], [2.98, 3.98]], rtol=1e-6)
  np.testing.assert_allclose(acc, g, rtol=1e-7)
  O.embedding_bwd(table, acc, None, rows, seg, g, O.OPT_MOMENTUM, 2.0, beta1=0.9)
  np.testing.assert_allclose(table, [[1.0 - 0.2 - 0.38, 2.0 - 0.2 - 0.38], [3.0 - 0.02 - 0.038, 4.0 - 0.02 - 0.038]], rtol=1e-6)
  np.testing.assert_allclose(acc, [[0.19, 0.19], [0.019, 0.019]], rtol=1e-6)
  # sparse apply: duplicates are summed first, rows without a gradient keep weight AND accumulator
  table = np.arange(8, dtype=np.float32).reshape(4, 2)
  acc = np.full((4, 2), 0.5, np.float32)
  O.embedding_bwd(table, acc, None, np.array([2, 0, 2], np.int64), np.arange(3, dtype=np.int32),
                  np.array([[1, 1], [2, 2], [3, 3]], np.float32), O.OPT_MOMENTUM, 0.1, beta1=0.5)
  np.testing.assert_allclose(acc, [[2.25, 2.25], [0.5, 0.5], [4.25, 4.25], [0.5, 0.5]])
  np.testing.assert_allclose(table, [[0 - 0.225, 1 - 0.225], [2, 3], [4 - 0.425, 5 - 0.425], [6, 7]], rtol=1e-6)


def test_momentum_optimizer_config_trains_tables_and_towers_with_the_accumulator_rule(doubles):
  from test_round2_host import CLIP_CFG
  from easyrec_b200 import _lib
  from easyrec_b200.estimator import EasyRecEstimator
  cfg = (CLIP_CFG % b'').replace(b'momentum_optimizer_value: 0.0', b'momentum_optimizer_value: 0.9')
  est = EasyRecEstimator(cfg, device='cpu', seed=11)
  il, tr = est.input_layer, est.trainer
  assert all(a.opt_kind == _lib.OPT_MOMENTUM and a.state0 is not None and a.state1 is None for a in il.arenas.values())
  assert tr.dense_opt.kind == _lib.OPT_MOMENTUM and float(tr.dense_opt.s0.abs().sum()) == 0.0
  rng = np.random.default_rng(0)
  B = 16
  ids = np.stack([rng.integers(0, 6, B), rng.integers(0, 6, B), rng.integers(0, 1000, B)]).astype(np.int64)
  feats = {'sparse_fea': torch.from_numpy(ids.reshape(-1)), 'dense_fea': torch.from_numpy(rng.uniform(0, 2, (B, 1)).astype(np.float32))}
  labels = torch.from_numpy((rng.uniform(size=B) < 0.4).astype(np.float32))
  # plain SGD twin with the same initial weights: its per-step update IS lr * g, the gradient the momentum run sees at
  # step 1; at step 1 both runs therefore move identically (accum = g), and the accumulators equal update / lr
  sgd = EasyRecEstimator(CLIP_CFG % b'', device='cpu', seed=11)
  p0 = tr.dense_opt.flat_p.clone()
  t0 = {d: a.weight.clone() for d, a in il.arenas.items()}
  tr.train_step(feats, labels)
  sgd.trainer.train_step(feats, labels)
  torch.testing.assert_close(tr.dense_opt.flat_p, sgd.trainer.dense_opt.flat_p, rtol=1e-6, atol=1e-7)
  torch.testing.assert_close(tr.dense_opt.s0, (p0 - tr.dense_opt.flat_p) / 0.5, rtol=1e-4, atol=1e-6)
  seen_untouched = False
  for d, a in il.arenas.items():
    torch.testing.assert_close(a.weight, sgd.input_layer.arenas[d].weight, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(a.state0, (t0[d] - a.weight) / 0.5, rtol=1e-4, atol=1e-6)
    untouched = (a.weight == t0[d]).all(1)
    seen_untouched = seen_untouched or bool(untouched.any())
    assert float(a.state0[untouched].abs().sum()) == 0.0                 # rows without a gradient: no state
  # step 2 on the same batch: var -= lr * (0.9 * accum + g2), i.e. further than the SGD twin by lr * 0.9 * accum
  acc1 = {d: a.state0.clone() for d, a in il.arenas.items()}
  w1 = {d: a.weight.clone() for d, a in il.arenas.items()}
  sgd.model.load_state_dict(est.model.state_dict())     # (same weights before step 2 -> same gradient g2)
  for d, a in il.arenas.items():
    sgd.input_layer.arenas[d].weight.copy_(a.weight)
  sgd.trainer.dense_opt.flat_p.copy_(tr.dense_opt.flat_p)
  tr.train_step(feats, labels)
  sgd.trainer.train_step(feats, labels)
  for d, a in il.arenas.items():
    g2 = (w1[d] - sgd.input_layer.arenas[d].weight) / 0.5
    touched = (g2 != 0).any(1)
    torch.testing.assert_close(a.state0[touched], (acc1[d] * 0.9 + g2)[touched], rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(a.weight[touched], (w1[d] - 0.5 * (acc1[d] * 0.9 + g2))[touched], rtol=1e-5, atol=1e-6)


# ---- the reference's own metric tests (easy_rec/python/test/eval_metric_test.py) --------------------------------------
def test_reference_eval_metric_known_answers(doubles):
  """test_max_f1 (:21-33): labels [1,0,0,1], predictions [0.9,0.8,0.7,0.6] -> 2/3; test_gauc / test_session_auc
  (:46-103): two users fed in two updates -> 0.5833333 / 0.5925926 / 0.6 by reduction; all-negative labels -> 0."""
  lab, pred = np.array([1, 0, 0, 1], np.float32), np.array([0.9, 0.8, 0.7, 0.6], np.float32)
  assert O.max_f1(lab, pred) == pytest.approx(2.0 / 3, abs=1e-6)
  acc = M.ConfusionAtThresholds(200, 'cpu')
  acc.update(torch.from_numpy(pred), torch.from_numpy(lab))
  assert acc.max_f1() == pytest.approx(2.0 / 3, abs=1e-6)
  labels = np.array([1, 0, 1, 1, 0, 1, 0, 0, 1])
  probs = np.array([0.9, 0.8, 0.7, 0.6, 0.5, 0.9, 0.8, 0.7, 0.6], np.float32)
  uids = np.array([1, 1, 1, 1, 1, 2, 2, 2, 2])
  for reduction, want in (('mean', 0.5833333), ('mean_by_sample_num', 0.5925926), ('mean_by_positive_num', 0.6)):
    assert float(M.gauc(labels, probs, uids, reduction)) == pytest.approx(want, abs=1e-6)
  assert float(M.gauc(np.zeros(4), pred, np.ones(4))) == 0.0
