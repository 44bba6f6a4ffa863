"""DBMTL, SimpleMultiTask and PLE (reference: easy_rec/python/model/dbmtl.py:17-121, model/simple_multi_task.py:17-56,
model/ple.py:17-128, model/multi_task_model.py): multi-task heads over the 'all' group, composed from the same fused DNN layers and the
MMoE mixture kernel as MMoE; the loss is MMoE's (sum_t weight_t * sigmoid CE on the tower's label)."""
import torch
from torch import nn

from easyrec_b200 import interactions as I
from easyrec_b200 import layers as L
from easyrec_b200 import model as registry
from easyrec_b200.model.mmoe import MMoE


def _towers(task_towers):
  return [(t.tower_name, t.label_name if t.HasField('label_name') else None, float(t.weight)) for t in task_towers]


@registry.register('SimpleMultiTask')
class SimpleMultiTask(MMoE):
  """per task: DNN(features) -> dense(1) (simple_multi_task.py:38-55)."""

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.simple_multi_task
    return cls(input_layer, model_config.feature_groups[0].group_name, _towers(c.task_towers),
               [L.units_of(t.dnn) for t in c.task_towers], l2_reg=c.l2_regularization,
               embedding_reg=model_config.embedding_regularization, generator=generator)

  def __init__(self, input_layer, group, towers, tower_units, l2_reg=0.0, embedding_reg=0.0, generator=None):
    nn.Module.__init__(self)
    self.input_layer, self.group = input_layer, group
    self.in_dim = d = input_layer.group_width(group)
    self.tower_names = [t[0] for t in towers]
    self.label_names = [t[1] for t in towers]
    self.task_weights = [t[2] for t in towers]
    self.tower_dnn = nn.ModuleList([L.DNN(d, u, generator=generator) for u in tower_units])
    self.tower_out = nn.ModuleList([L.Dense(dnn.out_dim, 1, generator) for dnn in self.tower_dnn])
    self.l2_reg, self.embedding_reg = l2_reg, embedding_reg

  def forward(self, features):
    x, _ = self.input_layer.lookup(features)[self.group]
    self._emb_outputs = (x,)
    x = x.contiguous()
    return torch.stack([out(dnn(x))[:, 0] for dnn, out in zip(self.tower_dnn, self.tower_out)], dim=1)


@registry.register('DBMTL')
class DBMTL(MMoE):
  """bottom DNN -> [MMoE experts + per-task gates] -> per-task tower DNN -> "Bayes" relation DNN over
  [tower feature | relation features of the towers it depends on] -> dense(1) (dbmtl.py:44-121)."""

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.dbmtl
    for f in ('bottom_cmbf', 'bottom_uniter'):
      if f in c.DESCRIPTOR.fields_by_name and c.HasField(f):
        raise NotImplementedError('dbmtl.%s' % f)
    return cls(input_layer, model_config.feature_groups[0].group_name, _towers(c.task_towers),
               bottom=L.units_of(c.bottom_dnn) if c.HasField('bottom_dnn') else None,
               expert=L.units_of(c.expert_dnn) if c.HasField('expert_dnn') else None, num_expert=int(c.num_expert),
               tower_units=[L.units_of(t.dnn) if t.HasField('dnn') else None for t in c.task_towers],
               relation_units=[L.units_of(t.relation_dnn) for t in c.task_towers],
               relations=[list(t.relation_tower_names) for t in c.task_towers], l2_reg=c.l2_regularization,
               embedding_reg=model_config.embedding_regularization, generator=generator)

  def __init__(self, input_layer, group, towers, bottom, expert, num_expert, tower_units, relation_units, relations,
               l2_reg=0.0, embedding_reg=0.0, generator=None):
    nn.Module.__init__(self)
    self.input_layer, self.group = input_layer, group
    self.in_dim = d = input_layer.group_width(group)
    self.tower_names = [t[0] for t in towers]
    self.label_names = [t[1] for t in towers]
    self.task_weights = [t[2] for t in towers]
    self.bottom = L.DNN(d, bottom, generator=generator) if bottom else None
    d = self.bottom.out_dim if self.bottom is not None else d
    self.experts = self.gates = None
    if expert:
      assert num_expert > 0, 'dbmtl.expert_dnn needs num_expert'
      self.experts = nn.ModuleList([L.DNN(d, expert, generator=generator) for _ in range(num_expert)])
      self.gates = nn.ModuleList([L.Dense(d, num_expert, generator) for _ in towers])
      d = self.experts[0].out_dim
    self.tower_dnn = nn.ModuleList([L.DNN(d, u, generator=generator) if u else nn.Identity() for u in tower_units])
    tower_dim = [dnn.out_dim if isinstance(dnn, L.DNN) else d for dnn in self.tower_dnn]
    self.relations = []
    rel_dim = {}
    self.relation_dnn = nn.ModuleList()
    for name, td, ru, rel in zip(self.tower_names, tower_dim, relation_units, relations):
      for r in rel:   # a tower may only depend on towers declared before it (dbmtl.py:100-104 reads relation_features)
        if r not in rel_dim:
          raise ValueError('task tower %s: relation tower %r is not defined before it' % (name, r))
      self.relations.append([self.tower_names.index(r) for r in rel])
      self.relation_dnn.append(L.DNN(td + sum(rel_dim[r] for r in rel), ru, generator=generator))
      rel_dim[name] = self.relation_dnn[-1].out_dim
    self.tower_out = nn.ModuleList([L.Dense(dnn.out_dim, 1, generator) for dnn in self.relation_dnn])
    self.l2_reg, self.embedding_reg = l2_reg, embedding_reg

  def forward(self, features):
    x, _ = self.input_layer.lookup(features)[self.group]
    self._emb_outputs = (x,)
    x = x.contiguous()
    if self.bottom is not None:
      x = self.bottom(x)
    if self.experts is not None:
      experts = torch.stack([e(x) for e in self.experts], dim=1)
      inputs = [I.mmoe_mix(gate(x), experts) for gate in self.gates]
    else:
      inputs = [x] * len(self.tower_names)
    rel, logits = [], []
    for i, (dnn, rdnn, out) in enumerate(zip(self.tower_dnn, self.relation_dnn, self.tower_out)):
      parts = [dnn(inputs[i])] + [rel[j] for j in self.relations[i]]
      r = rdnn(parts[0] if len(parts) == 1 else torch.cat(parts, dim=-1))
      rel.append(r)
      logits.append(out(r)[:, 0])
    return torch.stack(logits, dim=1)


@registry.register('PLE')
class PLE(MMoE):
  """Progressive layered extraction (ple.py:36-128): per extraction network, `expert_num_per_task` experts per task on
  that task's features and `share_num` shared experts on the shared features; a task's gate (softmax(dense(task
  features)) over [its experts | shared experts], the MMoE mixture kernel) gives its next features, the shared gate
  (over every expert) the next shared features - dropped in the last network; then tower DNN -> dense(1) per task."""

  @classmethod
  def from_config(cls, model_config, input_layer, generator=None):
    c = model_config.ple
    nets = [dict(per_task=int(n.expert_num_per_task), share=int(n.share_num), task_units=L.units_of(n.task_expert_net),
                 share_units=L.units_of(n.share_expert_net)) for n in c.extraction_networks]
    return cls(input_layer, model_config.feature_groups[0].group_name, _towers(c.task_towers), nets,
               [L.units_of(t.dnn) for t in c.task_towers], l2_reg=c.l2_regularization,
               embedding_reg=model_config.embedding_regularization, generator=generator)

  def __init__(self, input_layer, group, towers, nets, tower_units, l2_reg=0.0, embedding_reg=0.0, generator=None):
    nn.Module.__init__(self)
    self.input_layer, self.group = input_layer, group
    self.in_dim = d = input_layer.group_width(group)
    self.tower_names = [t[0] for t in towers]
    self.label_names = [t[1] for t in towers]
    self.task_weights = [t[2] for t in towers]
    n_task = len(towers)
    self.nets = nn.ModuleList()
    d_task, d_share = [d] * n_task, d
    for li, n in enumerate(nets):
      last = li + 1 == len(nets)
      net = nn.Module()
      net.share = nn.ModuleList([L.DNN(d_share, n['share_units'], generator=generator) for _ in range(n['share'])])
      net.task = nn.ModuleList([nn.ModuleList([L.DNN(d_task[t], n['task_units'], generator=generator)
                                               for _ in range(n['per_task'])]) for t in range(n_task)])
      h = net.task[0][0].out_dim
      if n['share'] and net.share[0].out_dim != h:
        raise ValueError('PLE: task_expert_net and share_expert_net must end in the same width (their outputs are mixed)')
      net.task_gate = nn.ModuleList([L.Dense(d_task[t], n['per_task'] + n['share'], generator) for t in range(n_task)])
      net.share_gate = None if last else L.Dense(d_share, n_task * n['per_task'] + n['share'], generator)
      self.nets.append(net)
      d_task, d_share = [h] * n_task, h
    self.tower_dnn = nn.ModuleList([L.DNN(d_task[t], u, generator=generator) for t, u in enumerate(tower_units)])
    self.tower_out = nn.ModuleList([L.Dense(dnn.out_dim, 1, generator) for dnn in self.tower_dnn])
    self.l2_reg, self.embedding_reg = l2_reg, embedding_reg

  def forward(self, features):
    x, _ = self.input_layer.lookup(features)[self.group]
    self._emb_outputs = (x,)
    x = x.contiguous()
    task_fea, share_fea = [x] * len(self.tower_names), x
    for net in self.nets:
      shared = [e(share_fea) for e in net.share]
      own = [[e(task_fea[t]) for e in net.task[t]] for t in range(len(task_fea))]
      nxt = [I.mmoe_mix(net.task_gate[t](task_fea[t]), torch.stack(own[t] + shared, dim=1)) for t in range(len(task_fea))]
      if net.share_gate is not None:
        every = [e for o in own for e in o] + shared
        share_fea = I.mmoe_mix(net.share_gate(share_fea), torch.stack(every, dim=1))
      task_fea = nxt
    return torch.stack([out(dnn(task_fea[t]))[:, 0] for t, (dnn, out) in enumerate(zip(self.tower_dnn, self.tower_out))],
                       dim=1)
