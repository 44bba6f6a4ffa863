"""DCN (reference: easy_rec/python/model/dcn.py:24-70): deep tower + cross tower over the same 'all' group,
concat -> final_dnn -> dense(1).  Cross layer v1: x_{l+1} = x0 * (x_l . w) + b + x_l (dcn.py:32-45),
w and b created with tf.get_variable's default initializer (glorot uniform)."""
import math

import torch
from torch import nn

from easyrec_b200 import interactions as I
from easyrec_b200 import layers as L
from easyrec_b200 import model as registry
from easyrec_b200.model.rank_model import RankModel


@registry.register('DCN')
class DCN(RankModel):

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.dcn
    return cls(input_layer, c.deep_tower.input, L.units_of(c.deep_tower.dnn), c.cross_tower.cross_num,
               L.units_of(c.final_dnn), l2_reg=c.l2_regularization,
               embedding_reg=model_config.embedding_regularization, generator=generator)

  def __init__(self, input_layer, group, deep_units, cross_num, final_units, l2_reg=0.0, embedding_reg=0.0,
               generator=None):
    super().__init__()
    self.input_layer = input_layer
    self.group = group
    d = input_layer.group_width(group)
    self.in_dim = d
    self.dnn = L.DNN(d, deep_units, generator=generator)
    lim = math.sqrt(6.0 / (d + d))  # glorot uniform of a [d] variable: fan_in = fan_out = d
    self.cross_w = nn.ParameterList([nn.Parameter(torch.empty(d).uniform_(-lim, lim, generator=generator))
                                     for _ in range(cross_num)])
    self.cross_b = nn.ParameterList([nn.Parameter(torch.empty(d).uniform_(-lim, lim, generator=generator))
                                     for _ in range(cross_num)])
    self.final_dnn = L.DNN(self.dnn.out_dim + d, final_units, generator=generator)
    self.output = L.Dense(self.final_dnn.out_dim, 1, generator)
    self.l2_reg = l2_reg
    self.embedding_reg = embedding_reg

  def forward(self, features):
    x0, _ = self.input_layer.lookup(features)[self.group]
    if x0.shape[1] != self.in_dim:
      x0 = x0[:, :self.in_dim]
    x0 = x0.contiguous()
    self._emb_outputs = (x0,)
    deep = self.dnn(x0)
    x = x0
    for w, b in zip(self.cross_w, self.cross_b):
      x = I.cross_layer(x0, x, w, b)
    return self.output(self.final_dnn(torch.cat([deep, x], dim=1)))[:, 0]
