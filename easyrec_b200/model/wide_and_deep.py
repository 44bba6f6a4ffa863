"""WideAndDeep and FM (reference: easy_rec/python/model/wide_and_deep.py:17-80, model/fm.py:14-62): the two smaller
relatives of DeepFM over the same 'wide' / 'deep' groups - the wide group as `wide_output_dim`-wide tables summed over
the features, the deep tower on the fused DNN layers, the FM term on the FM kernel."""
import torch
from torch import nn

from easyrec_b200 import embedding as E
from easyrec_b200 import layers as L
from easyrec_b200 import model as registry
from easyrec_b200.model.rank_model import RankModel


def _sum_features(x, n_feature):
  """tf.add_n over the group's per-feature [B, w] outputs, read from the group's [B, n_feature * w] concat"""
  B = x.shape[0]
  return x.reshape(B, n_feature, -1).sum(dim=1)


@registry.register('WideAndDeep')
class WideAndDeep(RankModel):

  @staticmethod
  def wide_output_dim(model_config):
    # without a final_dnn the wide sum IS a logit: wide_output_dim = num_class (wide_and_deep.py:35-42)
    c = model_config.wide_and_deep
    return int(c.wide_output_dim) if len(c.final_dnn.hidden_units) > 0 else int(model_config.num_class)

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.wide_and_deep
    return cls(input_layer, L.units_of(c.dnn), L.units_of(c.final_dnn) if len(c.final_dnn.hidden_units) > 0 else None,
               l2_reg=c.l2_regularization, embedding_reg=model_config.embedding_regularization, generator=generator)

  def __init__(self, input_layer, dnn_units, final_units, l2_reg=0.0, embedding_reg=0.0, generator=None):
    super().__init__()
    for gname in ('wide', 'deep'):
      assert input_layer.has_group(gname), 'WideAndDeep needs feature groups "wide" and "deep"'
    if any(e.kind != 'emb' for e in input_layer.group_layout['wide']):
      raise NotImplementedError('WideAndDeep: the wide group must hold embedded features only')
    self.input_layer = input_layer
    self.n_wide = len(input_layer.group_layout['wide'])
    self.wide_dim = input_layer.group_width('wide') // self.n_wide
    self.dnn = L.DNN(input_layer.group_width('deep'), dnn_units, generator=generator)
    self.final_dnn = None
    if final_units:
      self.final_dnn = L.DNN(self.wide_dim + self.dnn.out_dim, final_units, generator=generator)
      self.output = L.Dense(self.final_dnn.out_dim, 1, generator)
    else:
      self.output = L.Dense(self.dnn.out_dim, 1, generator)   # `deep_out`
    self.l2_reg, self.embedding_reg = l2_reg, embedding_reg

  def forward(self, features):
    g = self.input_layer.lookup(features)
    wide, deep = g['wide'][0], g['deep'][0]
    self._emb_outputs = (wide, deep)
    wide_fea = _sum_features(wide[:, :self.n_wide * self.wide_dim], self.n_wide)
    deep_fea = self.dnn(deep.contiguous())
    if self.final_dnn is not None:
      return self.output(self.final_dnn(torch.cat([wide_fea, deep_fea], dim=1)))[:, 0]
    return (self.output(deep_fea) + wide_fea)[:, 0]


@registry.register('FM')
class FM(RankModel):
  """wide sum + second-order FM over the deep group's fields + a bias (fm.py:43-62, num_class 1)."""

  @staticmethod
  def wide_output_dim(model_config):
    return int(model_config.num_class)

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.fm
    return cls(input_layer, l2_reg=c.l2_regularization, embedding_reg=model_config.embedding_regularization)

  def __init__(self, input_layer, l2_reg=0.0, embedding_reg=0.0):
    super().__init__()
    lay = input_layer.group_layout['deep']
    if any(e.kind != 'emb' for e in lay) or len({e.width for e in lay}) != 1:
      raise NotImplementedError('FM: the deep group must hold embedded features of one width')
    self.input_layer = input_layer
    self.n_field, self.dim = len(lay), lay[0].width
    self.n_wide = len(input_layer.group_layout['wide'])
    self.fm_bias = nn.Parameter(torch.zeros(1))
    self.l2_reg, self.embedding_reg = l2_reg, embedding_reg

  def forward(self, features):
    g = self.input_layer.lookup(features)
    wide, deep = g['wide'][0], g['deep'][0]
    self._emb_outputs = (wide, deep)
    wide_fea = wide[:, :self.n_wide].sum(dim=1, keepdim=True)
    fm_fea = E.fm(deep.contiguous(), self.n_field, self.dim).sum(dim=1, keepdim=True)
    return (wide_fea + fm_fea + self.fm_bias)[:, 0]
