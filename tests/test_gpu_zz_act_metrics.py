"""GPU: er_act_fwd / er_act_bwd (the non-relu activations of utils/activation.py:66-118) and er_auc_hist (the
confusion accumulators of tf.metrics.auc / max_f1, model/rank_model.py:360-373, core/metrics.py:25-56) against the
oracle, through the C ABI.  Tolerances: activation values 2e-6 relative / 1e-6 absolute, gradients 1e-5 / 2e-5, against the
float64 oracle (fp32 transcendental functions); the histograms are integers and must match exactly."""
import numpy as np
import pytest
import torch

from easyrec_b200 import kernels as K, layers as L, metrics as M
from oracle import oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAMES = ['gelu', 'leaky_relu', 'elu', 'selu', 'tanh', 'swish', 'sigmoid']


@pytest.mark.parametrize('name', NAMES)
@pytest.mark.parametrize('n', [1, 255, 1000003])
def test_activation_forward_and_backward_match_the_oracle(name, n):
  rng = np.random.default_rng(n)
  x = rng.normal(0, 3, n).astype(np.float32)
  x[:min(n, 5)] = np.array([0.0, -0.0, 30.0, -30.0, 1e-20], np.float32)[:min(n, 5)]
  gy = rng.normal(size=n).astype(np.float32)
  xd, gd = torch.from_numpy(x).to(DEV), torch.from_numpy(gy).to(DEV)
  kind = K.ACT_KINDS[name]
  y = K.act_fwd(xd, kind).cpu().numpy()
  gx = K.act_bwd(xd, gd, kind).cpu().numpy()
  np.testing.assert_allclose(y, O.activation(x, name), rtol=2e-6, atol=1e-6)
  np.testing.assert_allclose(gx, gy.astype(np.float64) * O.activation_grad(x, name), rtol=1e-5, atol=2e-5)   # (|gy| up to 5; 1 - tanh^2 cancels in fp32 where the slope vanishes)


def test_dnn_with_gelu_matches_plain_torch():
  torch.backends.cuda.matmul.allow_tf32 = False
  g = torch.Generator().manual_seed(1)
  units = L.Units([64, 32])
  units.activation = 'gelu'
  dnn = L.DNN(48, units, generator=g).to(DEV)
  dnn.train()
  x = torch.randn(512, 48, generator=g).to(DEV).requires_grad_(True)
  y = dnn(x)
  gy = torch.randn(512, 32, generator=g).to(DEV)
  y.backward(gy)
  xr = x.detach().double().requires_grad_(True)
  h = xr
  for lay in dnn.layers:
    z = h @ lay.kernel.detach().double() + lay.bias.detach().double()
    mu, var = z.mean(0), ((z - z.mean(0)) ** 2).mean(0)
    h = torch.nn.functional.gelu((z - mu) / torch.sqrt(var + 1e-3) * lay.gamma.detach().double() + lay.beta.detach().double(),
                                 approximate='tanh')
  h.backward(gy.double())
  assert float((y.double() - h).abs().max()) < 2e-5
  assert float((x.grad.double() - xr.grad).abs().max()) < 1e-4


@pytest.mark.parametrize('T', [2, 200, 4095])
def test_auc_histograms_are_exact(T):
  rng = np.random.default_rng(T)
  thr = O.tf_thresholds(T)
  acc = M.ConfusionAtThresholds(T, DEV)
  ps, ls = [], []
  for n in (1, 8192, 100003):   # several batches accumulate into the same device counters
    p = rng.random(n).astype(np.float32)
    k = min(n, 300)
    p[:k] = thr[rng.integers(0, T, k)]                       # predictions sitting exactly on thresholds
    if n > 10:
      p[-6:] = np.array([0.0, 1.0, -3.0, 7.0, np.nan, np.inf], np.float32)
    lab = rng.choice(np.array([0.0, 1.0, 0.5, 1.7, -1.0], np.float32), n)
    acc.update(torch.from_numpy(p).to(DEV), torch.from_numpy(lab).to(DEV))
    ps.append(p)
    ls.append(lab)
  p, lab = np.concatenate(ps), np.concatenate(ls)
  for got, want in zip(acc.counts(), O.confusion_at_thresholds(lab, p, T)):
    assert np.array_equal(got, want.astype(np.float32))
  assert acc.auc() == pytest.approx(O.auc_tf(lab, p, T), abs=1e-6)
  if T == 200:
    assert acc.max_f1() == pytest.approx(O.max_f1(lab, p), abs=1e-7)


def test_tensorflows_auc_known_answers_on_the_device():
  """tensorflow/python/kernel_tests/metrics_test.py AUCTest (recalled): all correct 1, some correct 0.5, all wrong 0."""
  for labels, preds, want in (([0, 1, 1, 0], [0, 1, 1, 0], 1.0), ([0, 1, 1, 0], [1, 0, 1, 0], 0.5),
                              ([1, 0, 0, 1], [0, 1, 1, 0], 0.0), ([0, 0, 0, 0], [0, 0, 0, 0], 1.0)):
    acc = M.ConfusionAtThresholds(200, DEV)
    acc.update(torch.tensor(preds, dtype=torch.float32, device=DEV), torch.tensor(labels, dtype=torch.float32, device=DEV))
    assert acc.auc() == pytest.approx(want, abs=1e-5)


def test_reference_max_f1_known_answer_on_the_device():
  """easy_rec/python/test/eval_metric_test.py:21-33: labels [1,0,0,1], predictions [0.9,0.8,0.7,0.6] -> 2/3"""
  acc = M.ConfusionAtThresholds(200, DEV)
  acc.update(torch.tensor([0.9, 0.8, 0.7, 0.6], device=DEV), torch.tensor([1.0, 0.0, 0.0, 1.0], device=DEV))
  assert acc.max_f1() == pytest.approx(2.0 / 3, abs=1e-6)


def test_invalid_metric_arguments_fail_loudly():
  from easyrec_b200 import _lib
  p = torch.zeros(4, device=DEV)
  thr = torch.zeros(5000, device=DEV)
  with pytest.raises((_lib.ErError, AssertionError)):
    K.auc_hist(p, p, thr, torch.zeros(2 * 5001, dtype=torch.int64, device=DEV))
  with pytest.raises(_lib.ErError):
    K.act_fwd(p, 99)


@pytest.mark.parametrize('M,N,K,form', [(8192, 4, 256, 'fwd'), (8192, 256, 4, 'dx'), (256, 4, 8192, 'dw'), (3, 5, 7, 'fwd'),
                                        (1000, 7, 33, 'fwd'), (33, 7, 1000, 'dw'), (16384, 3, 96, 'fwd'), (96, 3, 16384, 'dw')])
def test_small_gemm_matches_float64(M, N, K, form):
  """er_gemm_small through kernels.gemm (what the MMoE gate layers call): forward with bias, dX over W^T and dW over X^T
  read in place; against a float64 product, tolerance 6e-6 * sqrt(K) (a sequential fp32 FMA chain over N(0,1) operands; measured worst case 3e-6 * sqrt(K))."""
  rng = np.random.default_rng(M + N + K)
  if form == 'fwd':
    a = torch.from_numpy(rng.normal(size=(M, K + 4)).astype(np.float32)).to(DEV)[:, :K]
    b = torch.from_numpy(rng.normal(size=(K, N)).astype(np.float32)).to(DEV)
  elif form == 'dx':
    a = torch.from_numpy(rng.normal(size=(M, K)).astype(np.float32)).to(DEV)
    b = torch.from_numpy(rng.normal(size=(N, K)).astype(np.float32)).to(DEV).t()
  else:
    a = torch.from_numpy(rng.normal(size=(K, M)).astype(np.float32)).to(DEV).t()
    b = torch.from_numpy(rng.normal(size=(K, N)).astype(np.float32)).to(DEV)
  bias = torch.from_numpy(rng.normal(size=N).astype(np.float32)).to(DEV) if form == 'fwd' else None
  assert min(M, N, K) < 8
  got = K_gemm(a, b, bias)
  want = a.double() @ b.double() + (bias.double() if bias is not None else 0.0)
  assert float((got.double() - want).abs().max()) < 6e-6 * np.sqrt(K) + 2e-6
  again = K_gemm(a, b, bias)
  assert torch.equal(got, again)                              # deterministic: slices summed in order, no atomics
  out = torch.full((M, N + 4), float('nan'), device=DEV)
  K_gemm(a, b, bias, out=out[:, :N])
  assert torch.equal(out[:, :N], got) and torch.isnan(out[:, N:]).all()


def K_gemm(a, b, bias=None, out=None):
  return K.gemm(a, b, bias=bias, out=out)


def test_mmoe_gate_sized_dense_layer_trains_like_float64():
  """a [d -> 4] dense layer (an MMoE gate): forward, dX and dW all take the vector-sized path"""
  g = torch.Generator().manual_seed(2)
  lay = L.Dense(96, 4, generator=g).to(DEV)
  x = torch.randn(4096, 96, generator=g).to(DEV).requires_grad_(True)
  y = lay(x)
  gy = torch.randn(4096, 4, generator=g).to(DEV)
  y.backward(gy)
  xd = x.detach().double().requires_grad_(True)
  W = lay.kernel.detach().double().requires_grad_(True)
  (xd @ W + lay.bias.detach().double()).backward(gy.double())
  assert float((y.double() - (xd @ W + lay.bias.detach().double())).abs().max()) < 1e-5
  assert float((x.grad.double() - xd.grad).abs().max()) < 1e-5
  assert float((lay.kernel.grad.double() - W.grad).abs().max()) < 2e-4


def test_multi_valued_sequence_steps_on_the_kernels(tmp_path):
  """SequenceFeature with seq_multi_sep through InputLayer on the GPU: test/embed_test.py:88-151's table and expected
  per-step means ([[2,3],[4,5],...]), then one eager training step (CSR backward over (sample, step) segments)."""
  from easyrec_b200 import builder
  from easyrec_b200.config import config_util
  from easyrec_b200.input import readers
  from easyrec_b200.trainer import Trainer
  cfg = config_util.get_configs_from_pipeline_file(b'''
data_config { batch_size: 2 input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "key" input_type: INT64 }
  input_fields { input_name: "clk" input_type: STRING } }
feature_config {
  features { input_names: "key" feature_type: IdFeature embedding_dim: 2 num_buckets: 6 embedding_name: "t" }
  features { input_names: "clk" feature_type: SequenceFeature embedding_dim: 2 num_buckets: 6 embedding_name: "t"
             separator: "|" seq_multi_sep: "#" combiner: "mean" max_seq_len: 4 } }
model_config { model_class: "MultiTowerDIN"
  seq_att_groups { group_name: "din" seq_att_map { key: "key" hist_seq: "clk" } }
  feature_groups { group_name: "u" feature_names: ["key"] wide_deep: DEEP }
  multi_tower { towers { input: "u" dnn { hidden_units: [4] } } din_towers { input: "din" dnn { hidden_units: [4, 1] } }
                final_dnn { hidden_units: [4] } } }
''')
  il, model, _ = builder.build_model(cfg, 2, DEV, cpu_generator=torch.Generator().manual_seed(0))
  open(tmp_path / 's.csv', 'w').write('1,0,0#1|1#2||2#3|3#4|4#5\n0,3,4#5|#|5\n')
  (feats, labels), = list(readers.CSVInput(cfg, il, str(tmp_path / 's.csv')))
  feats, labels = readers.to_device(feats, labels, DEV)
  t = il.arenas[2]
  off, n, _ = t.tables['t']
  with torch.no_grad():
    t.weight[off:off + 6].copy_(torch.tensor([[1., 2.], [3., 4.], [5., 6.], [7., 8.], [9., 10.], [11., 12.]], device=DEV))
  il.lookup(feats)
  so = il.seq_outputs['din']
  want = torch.tensor([[[2., 3.], [4., 5.], [6., 7.], [8., 9.]], [[10., 11.], [0., 0.], [11., 12.], [0., 0.]]], device=DEV)
  assert torch.allclose(so['hist_seq_emb'], want, atol=1e-6) and so['hist_seq_len'].tolist() == [4, 3]
  il.discard_pending()
  before = t.weight[off:off + 6].clone()
  tr = Trainer(model, il, 'adagrad', lr=0.1)
  loss, _ = tr.train_step(feats, labels)
  assert np.isfinite(float(loss))
  changed = (t.weight[off:off + 6] != before).any(1)
  assert int(changed.sum()) >= 3                 # the rows of the keys and of the attended histories moved


@pytest.mark.parametrize('graph', [False, True])
def test_pipelined_loss_read_returns_every_steps_loss(graph):
  """EasyRecEstimator.train(fetch_loss_every_step=True): the losses travel through pinned slots one step behind the
  device; the value train() returns (and last_loss_value) is the LAST step's, equal to a run that synchronises once at the
  end; evaluate() then runs the streaming metrics on the device."""
  from test_act_metrics_host import CFG_ACT, _batches
  from easyrec_b200.estimator import EasyRecEstimator
  cfg = CFG_ACT.replace(b'ACT', b'gelu')
  a = EasyRecEstimator(cfg, device=DEV, seed=3, use_cuda_graph=graph)
  b = EasyRecEstimator(cfg, device=DEV, seed=3, use_cuda_graph=graph)
  la = a.train(lambda: _batches(9, 256, 1), steps=9, fetch_loss_every_step=True)
  lb = b.train(lambda: _batches(9, 256, 1), steps=9)
  assert la == pytest.approx(lb, rel=1e-6) and a.last_loss_value == la and a.global_step == b.global_step == 9
  ev = a.evaluate(lambda: _batches(4, 256, 99))
  assert 0.0 <= ev['auc'] <= 1.0 and 0.0 <= ev['auc_exact'] <= 1.0   # (nine steps in: the scores still sit in a narrow band)
  assert ev['max_f1'] > 0.0 and ev['root_mean_squared_error'] == pytest.approx(np.sqrt(ev['mean_squared_error']), rel=1e-6)


def test_attention_sequence_combiner_on_the_kernels():
  """sequence_combiner { attention } of SequenceFeatures in a plain group (layers/input_layer.py:312-347) through the real
  lookup, er_dense1 and er_din_pool kernels, against the numpy restatement of tests/test_act_metrics_host.py; then one
  training step moves the attention vectors and the table."""
  from test_act_metrics_host import CFG_SEQC, seqc_batch, seqc_expected
  from easyrec_b200 import builder
  from easyrec_b200.config import config_util
  from easyrec_b200.input import readers
  from easyrec_b200.trainer import Trainer
  cfg = config_util.get_configs_from_pipeline_file(CFG_SEQC)
  il, model, _ = builder.build_model(cfg, 4, DEV, cpu_generator=torch.Generator().manual_seed(2))
  with torch.no_grad():
    for m in il.attention_modules.values():
      m.kernel.copy_(torch.randn(m.kernel.shape, generator=torch.Generator().manual_seed(5)).to(DEV))
  feats, labels = seqc_batch()
  feats, labels = readers.to_device(feats, labels, DEV)
  concat, per_feature = il.lookup(feats)['g']
  u, pooled, _ = seqc_expected(il, feats)
  np.testing.assert_allclose(concat.detach().cpu().numpy(), np.concatenate([u, pooled['aa'], pooled['zz']], 1), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(per_feature[1].detach().cpu().numpy(), pooled['zz'], rtol=1e-5, atol=1e-6)
  il.discard_pending()
  w0 = [m.kernel.detach().clone() for m in il.attention_modules.values()]
  t0 = il.arenas[4].weight.clone()
  tr = Trainer(model, il, 'adagrad', lr=0.1)
  loss, _ = tr.train_step(feats, labels)
  assert np.isfinite(float(loss))
  assert all(float((m.kernel - w).abs().max()) > 0 for m, w in zip(il.attention_modules.values(), w0))
  assert float((il.arenas[4].weight - t0).abs().max()) > 0


@pytest.mark.parametrize('dim', [16, 6, 1])
def test_momentum_row_rule_and_dense_apply_track_the_oracle(dim):
  """momentum_optimizer with momentum > 0 (tf.train.MomentumOptimizer): K7's fused row update with the accumulator
  rule against the oracle over three steps (duplicated rows, dropped lookups, rows that appear only once keep their
  accumulator afterwards), and the flat dense apply against numpy."""
  from easyrec_b200 import _lib, embedding as E
  rng = np.random.default_rng(dim)
  V, B, F = 2000, 160, 3
  arena = E.Arena(dim, DEV)
  arena.add_table('t', V)
  arena.materialize(_lib.OPT_MOMENTUM, generator=torch.Generator(device=DEV).manual_seed(1))
  assert arena.state0 is not None and arena.state1 is None and float(arena.state0.abs().sum()) == 0.0
  table = arena.weight.cpu().numpy().copy()
  acc = np.zeros((V, dim), np.float32)
  stride = F * dim
  recs = [dict(num_buckets=V, row_offset=0, seg_begin=f * B, n_seg=B, bucket_mode=3, combiner=0, out_buf=0,
               out_stride=stride, out_col=f * dim) for f in range(F)]
  sd = K.slots_to_device(K.make_slots(recs), DEV)
  pad = (4 - stride % 4) % 4 if dim % 4 == 0 else 0
  ws = K.bwd_workspace(B * F, DEV, dim)
  hyper = K.StepHyper(DEV, 0.9, 0.999)     # beta1 carries the momentum
  for step in range(3):
    rows = rng.integers(0, V if step == 0 else 50, B * F).astype(np.int64)
    rows[rng.integers(0, B * F, 5)] = -1
    gout = rng.normal(0, 0.1, (B, stride + pad)).astype(np.float32)
    lr = 0.05 * (0.8 ** step)
    hyper.set(lr, step, grad_scale=0.5)
    opt = hyper.opt(_lib.OPT_MOMENTUM)
    K.embedding_bwd(arena.weight, arena.state0, None, dim, torch.from_numpy(rows).to(DEV), sd, F, B * F,
                    [torch.from_numpy(gout).to(DEV)], opt, ws)
    gseg = np.concatenate([gout[:, f * dim:(f + 1) * dim] for f in range(F)], 0)
    O.embedding_bwd(table, acc, None, rows, np.arange(B * F, dtype=np.int32), gseg, O.OPT_MOMENTUM, lr, beta1=0.9,
                    grad_scale=0.5)
    np.testing.assert_allclose(arena.weight.cpu().numpy(), table, rtol=0, atol=1e-6)
    np.testing.assert_allclose(arena.state0.cpu().numpy(), acc, rtol=0, atol=1e-6)
  # dense apply: one flat buffer, l2 folded in by the kernel
  import torch.nn as nn
  from easyrec_b200.trainer import FlatDenseOptimizer
  p = nn.Parameter(torch.from_numpy(rng.normal(size=(37, 5)).astype(np.float32)).to(DEV))
  fo = FlatDenseOptimizer([('w/kernel', p)], 'momentum', lr=0.1, beta1=0.9, l2_of=lambda n, q: 0.01)
  w, a = p.detach().cpu().numpy().copy(), np.zeros((37, 5), np.float32)
  for step in range(3):
    g = rng.normal(size=(37, 5)).astype(np.float32)
    fo.grad_views[0].copy_(torch.from_numpy(g).to(DEV))
    fo.hyper.set(0.1, step)
    fo.apply()
    gg = g + np.float32(0.01) * w
    a = a * np.float32(0.9) + gg
    w = w - np.float32(0.1) * a
    np.testing.assert_allclose(p.detach().cpu().numpy(), w, rtol=1e-5, atol=1e-6)


def test_dice_on_the_kernels_matches_the_reference_function_and_torch_autograd():
  """layers.Dice (er_bias_bn_act_* with unit gamma / zero beta at epsilon 1e-9 + er_dice_fwd / er_dice_bwd) against the
  output of utils/activation.py:dice executed (tests/golden/reference_activations.json) and, on a larger matrix, against
  torch autograd of the restatement (values, dx, d alpha)."""
  import json
  import os
  g = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_activations.json')))
  d = g['cases']['dice']
  m = L.Dice(3).to(DEV)
  with torch.no_grad():
    m.alphas.copy_(torch.tensor(d['alphas'], device=DEV))
  m.train()
  y = m(torch.tensor(d['x'], dtype=torch.float32, device=DEV))
  np.testing.assert_allclose(y.detach().cpu().numpy(), np.array(d['y'], np.float32), rtol=1e-5, atol=2e-6)
  gen = torch.Generator().manual_seed(4)
  B, C = 4099, 36
  x = (torch.randn(B, C, generator=gen) * 1.5 + 0.3).to(DEV)
  al = (torch.rand(C, generator=gen) - 0.5).to(DEV)
  gy = torch.randn(B, C, generator=gen).to(DEV)
  m = L.Dice(C).to(DEV)
  with torch.no_grad():
    m.alphas.copy_(al)
  m.train()
  xi = x.clone().requires_grad_(True)
  out = m(xi)
  out.backward(gy)
  xr = x.double().clone().requires_grad_(True)
  ar = al.double().clone().requires_grad_(True)
  mu, var = xr.mean(0), ((xr - xr.mean(0)) ** 2).mean(0)
  p = torch.sigmoid((xr - mu) / torch.sqrt(var + 1e-9))
  ref = ar * (1 - p) * xr + p * xr
  ref.backward(gy.double())
  assert float((out.double() - ref).abs().max()) < 2e-5
  assert float((xi.grad.double() - xr.grad).abs().max()) < 5e-5
  assert float((m.alphas.grad.double() - ar.grad).abs().max()) < 2e-3      # a sum of 4099 terms of size ~1
  np.testing.assert_allclose(m.moving_mean.cpu().numpy(), 0.01 * x.mean(0).cpu().numpy(), rtol=1e-4, atol=1e-6)
