"""DeepFM on the fused path (reference: easy_rec/python/model/deepfm.py:24-109).

wide  = sum_f wide_f                      [B,1]   (deepfm.py:62-63)
fm    = 0.5((sum_f v)^2 - sum_f v^2)      [B,D]   (layers/fm.py:20-26) over the deep group's features
deep  = DNN(deep concat)                          (deepfm.py:70-72)
with final_dnn: logits = dense(final_dnn(concat[wide, fm, deep]))   (deepfm.py:75-88)
without:        logits = wide + sum_d fm + dense(deep)             (deepfm.py:89-105)
"""
import torch
from torch import nn

from easyrec_b200 import embedding as E
from easyrec_b200 import kernels as K
from easyrec_b200 import layers as L
from easyrec_b200 import model as registry


@registry.register('DeepFM')
class DeepFM(nn.Module):

  @staticmethod
  def wide_output_dim(model_config):
    return model_config.deepfm.wide_output_dim

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.deepfm
    return cls(input_layer, L.units_of(c.dnn), L.units_of(c.final_dnn),
               l2_reg=c.l2_regularization, embedding_reg=model_config.embedding_regularization,
               generator=generator)

  def __init__(self, input_layer, dnn_units, final_units, l2_reg=0.0, embedding_reg=0.0,
               generator=None):
    super().__init__()
    for gname in ('wide', 'deep'):
      if any(e.kind == 'att' for e in input_layer.group_layout.get(gname, [])):
        raise NotImplementedError('DeepFM over a group with sequence_features (the FM fields must share one width)')
    self.input_layer = input_layer
    deep_layout = input_layer.group_layout['deep']
    self.n_field = len(deep_layout)
    self.dim = deep_layout[0].width
    # (a SequenceFeature pooled by its sequence_combiner is one more field of the same width, input_layer.py:312-347)
    assert all(e.width == self.dim and e.kind in ('emb', 'seqc') for e in deep_layout), \
        'FM needs every deep feature embedded with the same dim'
    self.deep_width = self.n_field * self.dim
    self.dnn = L.DNN(self.deep_width, dnn_units, generator=generator)
    self.has_final = len(final_units) > 0
    if self.has_final:
      self.final_dnn = L.DNN(1 + self.dim + self.dnn.out_dim, final_units, generator=generator)
      self.output = L.Dense(self.final_dnn.out_dim, 1, generator)
    else:
      self.output = L.Dense(self.dnn.out_dim, 1, generator)
    self.l2_reg = l2_reg
    self.embedding_reg = embedding_reg

  def forward(self, features):
    g = self.input_layer.lookup(features)
    wide, _ = g['wide']
    deep, _ = g['deep']
    self._wide_sumsq = None
    if wide.is_cuda:
      wide_fea, self._wide_sumsq = E.rowsum_block(wide)
    else:
      wide_fea = wide.sum(dim=1, keepdim=True)
    self._deep_sumsq = None
    if deep.shape[1] == self.deep_width and K.fm_block_ok(self.n_field, self.dim) and deep.is_cuda and \
        not hasattr(deep, '_er_reg'):
      # FM, the tower input and the regulariser's sum of squares from one pass; one merged gradient back
      fm_fea, deep_in, self._deep_sumsq = E.fm_block(deep, self.n_field, self.dim)
    else:
      fm_fea = E.fm(deep, self.n_field, self.dim)
      deep_in = deep[:, :self.deep_width] if deep.shape[1] != self.deep_width else deep
    deep_fea = self.dnn(deep_in)
    if self.has_final:
      all_fea = E.concat_cols([wide_fea, fm_fea, deep_fea])
      logits = self.output(self.final_dnn(all_fea))
    else:
      logits = wide_fea + fm_fea.sum(dim=1, keepdim=True) + self.output(deep_fea)
    self._emb_outputs = (wide, deep)
    return logits[:, 0]

  def l2_of(self, name, param):
    """kernel_regularizer = l2_regularizer(l2_regularization) on every dense kernel
    (layers/dnn.py:57-62, model/deepfm.py:83-87); biases and batch-norm parameters are not
    regularised."""
    return self.l2_reg if name.endswith('kernel') else 0.0

  def regularization_loss(self):
    """l2_regularizer(scale)(w) = scale * sum(w^2)/2 (compat/regularizers.py) on dense kernels
    (layers/dnn.py:57-62) and on the *looked-up* embedding outputs (layers/input_layer.py:369-375)."""
    reg = 0.0
    # dense kernel l2 is applied (and its loss term evaluated) inside the fused dense optimizer
    # launch: see l2_of() and trainer.FlatDenseOptimizer
    if self.embedding_reg > 0:
      wide, deep = self._emb_outputs
      if hasattr(deep, '_er_reg'):
        # sequence-combiner fields: the regulariser covers their un-pooled step embeddings (input_layer.py:316, 369-375)
        deep_sq = sum((t * t).sum() for t in deep._er_reg)
      else:
        deep_sq = self._deep_sumsq[0] if self._deep_sumsq is not None else (deep * deep).sum()
      wide_sq = self._wide_sumsq[0] if self._wide_sumsq is not None else (wide * wide).sum()
      reg = reg + self.embedding_reg * 0.5 * (wide_sq + deep_sq)
    return reg

  def loss(self, logits, labels, sample_weight=None):
    from easyrec_b200.model.rank_model import RankModel
    ce, probs = RankModel.data_loss(self, logits, labels, sample_weight)   # by model_config.loss_type
    return ce + self.regularization_loss(), probs
