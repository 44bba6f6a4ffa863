"""DSSM (reference: easy_rec/python/model/dssm.py:24-106, model/match_model.py:50-139,213-234):
two towers (DNN over all but the last hidden unit, then a linear dense to the last), cosine:
l2-normalise both and divide by temperature; list-wise: U @ I^T [B,B], optional *|sim_w|+sim_b,
duplicate in-batch items masked with -1e32, softmax CE on the diagonal + reg_pos_loss =
mean(relu(-pos_sim)); point-wise: sum(u*i) + sigmoid CE."""
import torch
from torch import nn

from easyrec_b200 import embedding as E
from easyrec_b200 import interactions as I
from easyrec_b200 import layers as L
from easyrec_b200 import model as registry
from easyrec_b200.model.rank_model import RankModel


@registry.register('DSSM')
class DSSM(RankModel):

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.dssm
    loss_name = model_config.DESCRIPTOR.fields_by_name['loss_type'].enum_type.values_by_number[
        model_config.loss_type].name
    simi = c.DESCRIPTOR.fields_by_name['simi_func'].enum_type.values_by_number[c.simi_func].name
    return cls(input_layer, L.units_of(c.user_tower.dnn), L.units_of(c.item_tower.dnn),
               cosine=(simi == 'COSINE'), temperature=c.temperature, scale_simi=c.scale_simi,
               listwise=(loss_name == 'SOFTMAX_CROSS_ENTROPY'), item_id=c.item_id or None,
               l2_reg=c.l2_regularization, embedding_reg=model_config.embedding_regularization,
               generator=generator)

  def __init__(self, input_layer, user_units, item_units, cosine=True, temperature=1.0, scale_simi=True,
               listwise=True, item_id=None, l2_reg=0.0, embedding_reg=0.0, generator=None):
    super().__init__()
    self.input_layer = input_layer
    du = input_layer.group_width('user')
    di = input_layer.group_width('item')
    self.du, self.di = du, di
    self.user_dnn = L.DNN(du, user_units[:-1], generator=generator) if len(user_units) > 1 else nn.Identity()
    self.user_out = L.Dense(user_units[-2] if len(user_units) > 1 else du, user_units[-1], generator)
    self.item_dnn = L.DNN(di, item_units[:-1], generator=generator) if len(item_units) > 1 else nn.Identity()
    self.item_out = L.Dense(item_units[-2] if len(item_units) > 1 else di, item_units[-1], generator)
    self.cosine, self.temperature, self.listwise = cosine, float(temperature), listwise
    self.scale_simi = scale_simi
    if scale_simi:
      self.sim_w = nn.Parameter(torch.ones(1))
      self.sim_b = nn.Parameter(torch.zeros(1))
    self.item_id = item_id
    self.l2_reg = l2_reg
    self.embedding_reg = embedding_reg

  def towers(self, features):
    g = self.input_layer.lookup(features)
    xu, xi = g['user'][0], g['item'][0]
    xu = xu[:, :self.du].contiguous() if xu.shape[1] != self.du else xu
    xi = xi[:, :self.di].contiguous() if xi.shape[1] != self.di else xi
    self._emb_outputs = (xu, xi)
    u = self.user_out(self.user_dnn(xu))
    i = self.item_out(self.item_dnn(xi))
    if self.cosine:
      u, i = I.l2_normalize(u), I.l2_normalize(i)
    return u, i

  def forward(self, features):
    u, i = self.towers(features)
    self._ui = (u, i)
    temp = self.temperature if self.cosine else 1.0
    sim = (I.matmul_nt(u, i) if self.listwise else (u * i).sum(dim=1, keepdim=True)) / temp
    if self.scale_simi:
      sim = sim * self.sim_w.abs() + self.sim_b
    self._item_ids = features.get('item_ids')
    return sim if self.listwise else sim[:, 0]

  accepts_sample_weight = False   # (the list-wise loss normalises by mean(w): not built)

  def loss(self, logits, labels):
    reg = self.embedding_reg_loss(self._emb_outputs)
    if not self.listwise:
      ce, probs = E.sigmoid_cross_entropy(logits, labels)
      return ce + reg, probs
    ce, p_diag = I.inbatch_softmax_ce(logits, self._item_ids)
    u, i = self._ui
    reg_pos = torch.relu(-(u * i).sum(dim=1)).mean()  # match_model.py:228-233
    return ce + reg_pos + reg, p_diag
