"""MultiTowerDIN (reference: easy_rec/python/model/multi_tower_din.py:24-130).

towers:      batch_norm(group features) -> DNN                              (:99-111)
din_towers:  target attention over the behaviour sequence                   (:62-97, K4)
             concat[q, k, q-k, q*k] -> DNN(last layer linear, no BN) -> mask -2^32+1 -> softmax
             -> scores @ keys, then concat with the key
final:       concat(all towers) -> final_dnn -> dense(1)                     (:120-128)
"""
import torch
from torch import nn

from easyrec_b200 import interactions as I
from easyrec_b200 import layers as L
from easyrec_b200 import model as registry
from easyrec_b200.model.rank_model import RankModel


@registry.register('MultiTowerDIN')
class MultiTowerDIN(RankModel):

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.multi_tower
    return cls(input_layer, [(t.input, L.units_of(t.dnn)) for t in c.towers],
               [(t.input, L.units_of(t.dnn)) for t in c.din_towers], L.units_of(c.final_dnn),
               l2_reg=c.l2_regularization, embedding_reg=model_config.embedding_regularization,
               generator=generator)

  def __init__(self, input_layer, towers, din_towers, final_units, l2_reg=0.0, embedding_reg=0.0,
               generator=None):
    super().__init__()
    self.input_layer = input_layer
    self.tower_groups = [g for g, _ in towers]
    self.din_groups = [g for g, _ in din_towers]
    self.tower_bn = nn.ModuleList()
    self.tower_dnn = nn.ModuleList()
    total = 0
    for g, units in towers:
      d = input_layer.group_width(g)
      self.tower_bn.append(L.BatchNorm(d))
      self.tower_dnn.append(L.DNN(d, units, generator=generator))
      total += self.tower_dnn[-1].out_dim
    self.din_dnn = nn.ModuleList()
    for g, units in din_towers:
      lay = input_layer.seq_layout[g]
      dk = sum(e.dim for e in lay['key'])
      dh = sum(e.dim for e in lay['hist'])
      assert dk == dh, 'DIN key dim %d != history dim %d' % (dk, dh)
      self.din_dnn.append(L.DNN(4 * dh, units, last_layer_no_activation=True, last_layer_no_batch_norm=True,
                                generator=generator))
      total += dh + dk
    self.final_dnn = L.DNN(total, final_units, generator=generator)
    self.output = L.Dense(self.final_dnn.out_dim, 1, generator)
    self.l2_reg = l2_reg
    self.embedding_reg = embedding_reg

  def forward(self, features):
    groups = self.input_layer.lookup(features)
    seq = self.input_layer.seq_outputs
    feas, reg = [], []
    for g, bn, dnn in zip(self.tower_groups, self.tower_bn, self.tower_dnn):
      x, _ = groups[g]
      reg.append(x)
      feas.append(dnn(bn(x)))
    for g, dnn in zip(self.din_groups, self.din_dnn):
      s = seq[g]
      key, hist, lens = s['key'], s['hist_seq_emb'], s['hist_seq_len']
      reg += [key, hist]
      att = I.din_attention(key.contiguous(), hist.contiguous(), lens, dnn)
      feas.append(torch.cat([att, key], dim=1))
    self._emb_outputs = tuple(reg)
    return self.output(self.final_dnn(torch.cat(feas, dim=1)))[:, 0]


@registry.register('MultiTower')
class MultiTower(MultiTowerDIN):
  """model/multi_tower.py:17-62: per tower batch_normalization -> DNN, concat, final DNN, dense(1) - MultiTowerDIN's
  graph without the attention towers (it reads only `multi_tower.towers`; din / bst towers of the message are not its)."""

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.multi_tower
    return cls(input_layer, [(t.input, L.units_of(t.dnn)) for t in c.towers], [], L.units_of(c.final_dnn),
               l2_reg=c.l2_regularization, embedding_reg=model_config.embedding_regularization, generator=generator)
