"""CPU, kernel doubles: the backbone DIN - an `input_layer { output_seq_and_normal_feature: true }` block feeding a keras
`DIN` block (layers/common_layers.py:104-131, layers/keras/din.py:16-67).

  * tests/golden/reference_din_block.json (DIN.call executed from the reference's source) against a torch float64
    restatement and against the block itself;
  * the block's output and its input gradients against the float64 restatement;
  * samples/model_config/din_backbone_on_taobao.config (stored copy) builds, trains two steps and evaluates its AUC;
  * every configuration the path does not build is refused, naming the field or the block class."""
import json
import math
import os

import numpy as np
import pytest
import torch

import host_doubles
from easyrec_b200 import backbone as BB
from easyrec_b200 import builder
from easyrec_b200 import interactions as I
from easyrec_b200.config import config_util
from easyrec_b200.input import readers
from test_config import reference_configs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_din_block.json')
PAD = -2.0**32 + 1


def _sample_text(name='din_backbone_on_taobao.config'):
  cfgs = reference_configs()
  return [v for k, v in cfgs.items() if os.path.basename(k) == name][0]


def _din_sigmoid_attention(query, keys, lens, attention_mlp, scale):
  B, T, D = keys.shape
  q = query[:, None, :].expand(B, T, D)
  s = attention_mlp(torch.cat([q, keys, q - keys, q * keys], dim=-1)).reshape(B, T)
  mask = torch.arange(T)[None, :] < lens[:, None]
  p = torch.where(mask, torch.sigmoid(s * scale), torch.zeros_like(s))
  return (p[:, :, None] * keys).sum(1)


@pytest.fixture
def doubles(monkeypatch):
  host_doubles.install_all(monkeypatch.setattr)
  monkeypatch.setattr(I, 'din_sigmoid_attention', _din_sigmoid_attention)


def restate(keys, lens, query, score_fn, normalizer, need_target):
  """layers/keras/din.py:27-67 in torch, any dtype: pad the query, [q, k, q-k, q*k], score, mask with -2^32+1,
  softmax or sigmoid(s / sqrt(D)), weighted sum of keys[:, :, :query width], [| padded query]."""
  B, T, D = keys.shape
  qw = query.shape[-1]
  if qw < D:
    query = torch.nn.functional.pad(query, (0, D - qw))
  q = query[:, None, :].expand(B, T, D)
  s = score_fn(torch.cat([q, keys, q - keys, q * keys], dim=-1)).reshape(B, T)
  s = torch.where(torch.arange(T)[None, :] < lens[:, None].long(), s, torch.full_like(s, PAD))
  p = torch.softmax(s, dim=1) if normalizer == 'softmax' else torch.sigmoid(s / D ** 0.5)
  out = (p[:, :, None] * keys[:, :, :qw]).sum(1)
  return torch.cat([out, query], dim=1) if need_target else out


def _score_fn(case, dtype):
  w1, b1, w2 = (torch.tensor(case[k], dtype=dtype) for k in ('w1', 'b1', 'w2'))
  b2 = float(case['b2'])
  return lambda x: torch.tanh(x @ w1 + b1) @ w2 + b2


class _Fixed(torch.nn.Module):
  def __init__(self, fn):
    super().__init__()
    self.fn = fn

  def forward(self, x):
    return self.fn(x)[:, None]


def _din_conf(normalizer, need_target):
  cfg = config_util.get_configs_from_pipeline_file(_sample_text())
  conf = [b for b in cfg.model_config.backbone.blocks if b.name == 'DIN'][0].keras_layer.din
  conf.attention_normalizer = normalizer
  conf.need_target_feature = need_target
  return conf


def _block(case, dtype=torch.float32):
  """the backbone's DIN module of the case's shape, its attention MLP replaced by the case's fixed function"""
  keys = torch.tensor(case['keys'], dtype=dtype)
  query = torch.tensor(case['query'], dtype=dtype)
  mod = BB.DIN(keys.shape[-1], query.shape[-1], _din_conf(case['normalizer'], case['need_target_feature']))
  mod.mlp = _Fixed(_score_fn(case, dtype))
  return mod, keys, query, torch.tensor(case['lens'], dtype=torch.int32)


def _golden():
  with open(GOLDEN) as f:
    return json.load(f)['cases']


def test_golden_cases_cover_what_the_fixture_promises():
  cases = _golden()
  assert {(c['normalizer'], c['need_target_feature'], len(c['query'][0]) < len(c['keys'][0][0])) for c in cases.values()} \
      == {(n, t, q) for n in ('softmax', 'sigmoid') for t in (True, False) for q in (True, False)}
  for c in cases.values():
    T = len(c['keys'][0])
    assert {0, 1, T} <= set(c['lens'])


@pytest.mark.parametrize('name', sorted(_golden()))
def test_golden_float64_restatement(name):
  c = _golden()[name]
  y = restate(torch.tensor(c['keys'], dtype=torch.float64), torch.tensor(c['lens']),
              torch.tensor(c['query'], dtype=torch.float64), _score_fn(c, torch.float64), c['normalizer'],
              c['need_target_feature'])
  np.testing.assert_allclose(y.numpy(), np.array(c['y']), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('name', sorted(_golden()))
def test_golden_block_under_kernel_doubles(doubles, name):
  c = _golden()[name]
  mod, keys, query, lens = _block(c)
  y = mod((keys, lens, query))
  np.testing.assert_allclose(y.detach().numpy(), np.array(c['y']), rtol=1e-5, atol=1e-5)
  assert y.shape[1] == mod.out_dim


@pytest.mark.parametrize('normalizer', ['softmax', 'sigmoid'])
@pytest.mark.parametrize('qw', [8, 5])
def test_block_output_and_input_gradients_match_float64(doubles, normalizer, qw):
  c = dict(_golden()['%s_target_q8' % normalizer])
  rng = np.random.default_rng(7)
  B, T, D = 6, 9, 8
  c.update(keys=rng.normal(size=(B, T, D)).tolist(), query=rng.normal(size=(B, qw)).tolist(), lens=[0, 1, 9, 4, 9, 2])
  mod, keys, query, lens = _block(c)
  keys.requires_grad_(True)
  query.requires_grad_(True)
  y = mod((keys, lens, query))
  gy = torch.from_numpy(rng.normal(size=tuple(y.shape)).astype(np.float32))
  gk, gq = torch.autograd.grad(y, (keys, query), gy)
  k64 = keys.detach().double().requires_grad_(True)
  q64 = query.detach().double().requires_grad_(True)
  y64 = restate(k64, lens, q64, _score_fn(c, torch.float64), normalizer, True)
  gk64, gq64 = torch.autograd.grad(y64, (k64, q64), gy.double())
  np.testing.assert_allclose(y.detach().numpy(), y64.detach().numpy(), rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(gk.numpy(), gk64.numpy(), rtol=1e-4, atol=1e-5)
  np.testing.assert_allclose(gq.numpy(), gq64.numpy(), rtol=1e-4, atol=1e-5)
  # beyond the length the scores get no gradient: a sigmoid-normalised key there receives nothing at all
  if normalizer == 'sigmoid':
    assert float(gk[0].abs().max()) == 0.0 and float(gk[3, 4:].abs().max()) == 0.0


def test_din_backbone_sample_config_trains_and_evaluates(doubles):
  from easyrec_b200.estimator import EasyRecEstimator
  cfg = config_util.get_configs_from_pipeline_file(_sample_text())
  est = EasyRecEstimator(cfg, device='cpu', seed=1, batch_size=8)
  il = est.input_layer
  assert il.seq_group_layout['sequence']['T'] == 50
  # the history tables carry the feature's name, the target columns share the `normal` group's tables
  tables = set(t for a in il.arenas.values() for t in a.tables)
  assert {'tag_category_list_embedding', 'tag_brand_list_embedding', 'cate_id_embedding', 'brand_embedding'} <= tables
  assert not any('sequence' in t for t in tables)
  din = est.model.backbone.mods['DIN']
  assert din.out_dim == 32 + 32 and not din.sigmoid and din.need_target
  feats, labels = readers.DummyInput(il, n_labels=1, seed=3).batch()
  g = il.lookup(feats)
  seq, seq_len, target, plain = g['sequence']
  assert seq.shape == (8, 50, 32) and target.shape == (8, 32) and len(plain) == 2
  assert torch.equal(seq_len, feats['seq_fea']['tag_category_list'][1])
  assert len(seq._er_reg) == 3      # the un-pooled histories and the two plain columns
  losses = [float(est.trainer.train_step(feats, labels)[0]) for _ in range(2)]
  assert all(np.isfinite(losses))
  ev = est.evaluate(lambda: [(feats, labels)])
  assert 'auc' in ev and 0.0 <= ev['auc'] <= 1.0


def _edit(*pairs):
  text = _sample_text().decode() if isinstance(_sample_text(), bytes) else _sample_text()
  for old, new in pairs:
    assert old in text, old
    text = text.replace(old, new, 1)
  return config_util.get_configs_from_pipeline_file(text.encode())


def _build(cfg):
  return builder.build_model(cfg, 4, 'cpu', cpu_generator=torch.Generator().manual_seed(0))


_TAG_CATE = "input_names: 'tag_category_list'\n     feature_type: SequenceFeature"
_SEQ_INPUT = 'output_seq_and_normal_feature: true'


@pytest.mark.parametrize('edits, exc, pattern', [
    ([(_TAG_CATE, _TAG_CATE + "\n     seq_multi_sep: ';'")], NotImplementedError, 'seq_multi_sep'),
    ([(_TAG_CATE, _TAG_CATE + '\n     sub_feature_type: RawFeature')], NotImplementedError, 'sub_feature_type'),
    ([("blocks {\n      name: 'DIN'", "blocks { name: 'other' inputs { feature_group_name: 'sequence' } keras_layer { "
       "class_name: 'MLP' mlp { hidden_units: [4] } } }\n    blocks {\n      name: 'DIN'")],
     NotImplementedError, 'output_seq_and_normal_feature and by another block'),
    ([("input_names: 'tag_brand_list'\n     feature_type: SequenceFeature\n     separator: '|'\n     "
       "hash_bucket_size: 100000\n     embedding_dim: 16\n     max_seq_len: 50",
       "input_names: 'tag_brand_list'\n     feature_type: SequenceFeature\n     separator: '|'\n     "
       "hash_bucket_size: 100000\n     embedding_dim: 16\n     max_seq_len: 40")], NotImplementedError, 'max_seq_len'),
    ([(_SEQ_INPUT, _SEQ_INPUT + ' concat_seq_feature: false')], NotImplementedError, 'concat_seq_feature'),
    ([('feature_names: "cate_id"\n    feature_names: "brand"\n', '')], ValueError, 'target feature is empty'),
    ([('feature_names: "cate_id"\n    feature_names: "brand"\n',
       'feature_names: "cate_id"\n    feature_names: "brand"\n    feature_names: "pid"\n')], ValueError,
     'target item .* is larger'),
    ([('need_target_feature: true', "need_target_feature: true attention_normalizer: 'tanh'")], ValueError,
     'unsupported attention normalizer'),
])
def test_refusals_name_their_field(edits, exc, pattern):
  cfg = _edit(*edits)
  with pytest.raises(exc, match=pattern):
    _build(cfg)


@pytest.mark.parametrize('name, cls', [('bst_backbone_on_taobao.config', 'BST'), ('cl4srec_on_taobao.config', 'SeqAugment'),
                                       ('text_cnn_on_movielens.config', 'TextCNN')])
def test_other_consumers_of_the_sequence_output_stay_refused_naming_their_class(name, cls):
  cfg = config_util.get_configs_from_pipeline_file(_sample_text(name))
  with pytest.raises(NotImplementedError, match=r'\(%s\) reads the sequence output' % cls):
    _build(cfg)


def test_sigmoid_scale_is_one_over_sqrt_of_the_history_width(doubles, monkeypatch):
  seen = []
  monkeypatch.setattr(I, 'din_sigmoid_attention', lambda q, k, l, m, scale: seen.append(scale) or
                      _din_sigmoid_attention(q, k, l, m, scale))
  mod, keys, query, lens = _block(_golden()['sigmoid_target_q5'])
  mod((keys, lens, query))
  assert seen == [1.0 / math.sqrt(keys.shape[-1])]
