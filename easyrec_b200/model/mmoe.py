"""MMoE (reference: easy_rec/python/model/mmoe.py:24-70, layers/mmoe.py:53-83, model/multi_task_model.py):
E expert DNNs on the 'all' group -> per task: softmax(dense(x)) gate, mixture of experts (fused K: mmoe_mix),
tower DNN, dense(num_class).  Loss = sum_task weight * sigmoid CE(label_task)."""
import torch
from torch import nn

from easyrec_b200 import embedding as E
from easyrec_b200 import interactions as I
from easyrec_b200 import layers as L
from easyrec_b200 import model as registry
from easyrec_b200.model.rank_model import RankModel


@registry.register('MMoE')
class MMoE(RankModel):

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.mmoe
    if c.HasField('expert_dnn'):
      experts = [L.units_of(c.expert_dnn)] * c.num_expert
    else:
      experts = [L.units_of(e.dnn) for e in c.experts]
    towers = [(t.tower_name, t.label_name if t.HasField('label_name') else None, L.units_of(t.dnn) if t.HasField('dnn') else [], t.weight)
              for t in c.task_towers]
    group = model_config.feature_groups[0].group_name
    return cls(input_layer, group, experts, towers, l2_reg=c.l2_regularization,
               embedding_reg=model_config.embedding_regularization, generator=generator)

  def __init__(self, input_layer, group, expert_units, towers, l2_reg=0.0, embedding_reg=0.0, generator=None,
               backbone=None):
    super().__init__()
    self.input_layer = input_layer
    self.group = group
    self.backbone = backbone
    d = backbone.out_dim if backbone is not None else input_layer.group_width(group)
    self.in_dim = d
    self.experts = nn.ModuleList([L.DNN(d, u, generator=generator) for u in expert_units])
    h = self.experts[0].out_dim
    self.gates = nn.ModuleList([L.Dense(d, len(expert_units), generator) for _ in towers])
    self.tower_names = [t[0] for t in towers]
    self.label_names = [t[1] for t in towers]
    self.task_weights = [float(t[3]) for t in towers]
    self.tower_dnn = nn.ModuleList([L.DNN(h, t[2], generator=generator) if t[2] else nn.Identity() for t in towers])
    self.tower_out = nn.ModuleList([L.Dense(t[2][-1] if t[2] else h, 1, generator) for t in towers])
    self.l2_reg = l2_reg
    self.embedding_reg = embedding_reg

  def forward(self, features):
    x, _ = self.input_layer.lookup(features)[self.group]
    if self.backbone is None and x.shape[1] != self.in_dim:
      x = x[:, :self.in_dim]
    x = x.contiguous()
    self._emb_outputs = (x,)
    if self.backbone is not None:
      x = self.backbone(x)
    experts = torch.stack([e(x) for e in self.experts], dim=1)  # [B, E, H]
    logits = []
    for gate, dnn, out in zip(self.gates, self.tower_dnn, self.tower_out):
      mix = I.mmoe_mix(gate(x), experts)
      logits.append(out(dnn(mix))[:, 0])
    return torch.stack(logits, dim=1)  # [B, n_task]

  def loss(self, logits, labels, sample_weight=None):
    """labels [B, n_label] in data_config.label_fields order; tower t reads column label_cols[t] (its
    label_name, multi_task_model.py:114-122); multi_task_model.py:201-280: sum_t w_t * CE_t."""
    total = 0.0
    probs = []
    cols = getattr(self, 'label_cols', None) or list(range(len(self.task_weights)))
    for t, w in enumerate(self.task_weights):
      lt = (getattr(self, 'task_loss_types', None) or ['CLASSIFICATION'] * len(self.task_weights))[t]
      ce, p = self.data_loss(logits[:, t].contiguous(), labels[:, cols[t]].contiguous(), sample_weight, loss_type=lt)
      total = total + w * ce
      probs.append(p)
    return total + self.embedding_reg_loss(self._emb_outputs), torch.stack(probs, dim=1)
