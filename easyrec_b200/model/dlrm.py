"""DLRM (reference: easy_rec/python/model/dlrm.py:16-73, protos/dlrm.proto): bot_dnn over the 'dense' group, pairwise
dot products between its output and the per-feature embeddings of the 'sparse' group (`einsum('bne,bme->bnm')`, the
upper triangle row by row, the diagonal kept with arch_interaction_itself), concat [dots | sparse features (| dense
output with arch_with_dense_feature)] - or, arch_interaction_op 'cat', [dense output | sparse features] - then
top_dnn and dense(1).  The reference's own EmbeddingParallel test model
(samples/model_config/dlrm_on_criteo_parquet_ep.config)."""
import torch

from easyrec_b200 import interactions as I
from easyrec_b200 import layers as L
from easyrec_b200 import model as registry
from easyrec_b200.model.rank_model import RankModel


@registry.register('DLRM')
class DLRM(RankModel):

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    if model_config.WhichOneof('model') != 'dlrm':
      raise ValueError('invalid model config: %s' % model_config.WhichOneof('model'))
    c = model_config.dlrm
    return cls(input_layer, L.units_of(c.bot_dnn), L.units_of(c.top_dnn), op=c.arch_interaction_op,
               itself=c.arch_interaction_itself, with_dense=c.arch_with_dense_feature, l2_reg=c.l2_regularization,
               embedding_reg=model_config.embedding_regularization, generator=generator)

  def __init__(self, input_layer, bot_units, top_units, op='dot', itself=False, with_dense=False, l2_reg=0.0,
               embedding_reg=0.0, generator=None):
    super().__init__()
    lay = input_layer.group_layout
    if 'sparse' not in lay:
      raise ValueError('sparse group is not specified')
    if 'dense' not in lay:
      raise ValueError('dense group is not specified')
    if op not in ('dot', 'cat'):
      raise ValueError('arch_interaction_op must be dot or cat, got %r' % op)
    self.input_layer = input_layer
    self.op, self.itself, self.with_dense = op, bool(itself), bool(with_dense)
    self.sparse_dims = [e.width for e in lay['sparse']]
    d_dense = input_layer.group_width('dense')
    self.d_dense = d_dense
    self.bot_dnn = L.DNN(d_dense, bot_units, generator=generator)
    D = self.bot_dnn.out_dim
    n = 1 + len(self.sparse_dims)
    if op == 'dot':
      if any(d != D for d in self.sparse_dims):
        raise ValueError('bot_dnn last hidden[%d] != sparse feature embedding_dim%s' % (D, sorted(set(self.sparse_dims))))
      off = 0 if self.itself else 1
      # upper triangle row by row: interaction[:, i, i + off:] for i = 0 .. n-1 (model/dlrm.py:58-61)
      idx = [i * n + j for i in range(n) for j in range(i + off, n)]
      self.register_buffer('tri_idx', torch.tensor(idx, dtype=torch.int64), persistent=False)
      d_all = len(idx) + sum(self.sparse_dims) + (D if self.with_dense else 0)
    else:
      d_all = D + sum(self.sparse_dims)
    self.n_fea = n
    self.top_dnn = L.DNN(d_all, top_units, generator=generator)
    self.output = L.Dense(self.top_dnn.out_dim, 1, generator)
    self.l2_reg = l2_reg
    self.embedding_reg = embedding_reg

  def forward(self, features):
    g = self.input_layer.lookup(features)
    sparse_cat, sparse = g['sparse']
    dense, _ = g['dense']
    width = sum(self.sparse_dims)
    sparse_cat = sparse_cat[:, :width] if sparse_cat.shape[1] != width else sparse_cat
    dense = dense[:, :self.d_dense] if dense.shape[1] != self.d_dense else dense
    self._emb_outputs = (sparse_cat,) + ((dense,) if dense.requires_grad else ())
    dense_fea = self.bot_dnn(dense.contiguous())
    if self.op == 'cat':
      all_fea = torch.cat([dense_fea, sparse_cat], dim=1)
    else:
      B, D = dense_fea.shape
      stack = torch.cat([dense_fea, sparse_cat], dim=1).reshape(B, self.n_fea, D)
      inter = I.gram(stack.contiguous()).reshape(B, self.n_fea * self.n_fea)
      parts = [inter.index_select(1, self.tri_idx), sparse_cat]
      if self.with_dense:
        parts.append(dense_fea)
      all_fea = torch.cat(parts, dim=1)
    return self.output(self.top_dnn(all_fea.contiguous()))[:, 0]
