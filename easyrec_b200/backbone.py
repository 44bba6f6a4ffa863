"""Configurable backbone network (reference: easy_rec/python/layers/backbone.py:215-348, 420-510):
a DAG of named blocks over feature groups, each block a Keras-style layer, a lambda, a recurrent or a
repeat wrapper; `concat_blocks` / `output_blocks` select the outputs, `top_mlp` finishes.

The wiring is host-side (done once); the layers run on liber_b200: `MLP` = layers.DenseLayer stack (wgmma
GEMM + fused batch-norm/activation, layers/keras/blocks.py:33-129), `Cross` = DCN-v2 cross
`x0 * (W x + b) + x` (layers/keras/interaction.py:249-286), `FM` = the FM kernels
(layers/keras/interaction.py:24-44), `MMoE` = expert MLPs + the softmax mixture kernel
(layers/keras/multi_task.py:47-67).  Like the reference, `input_fn` / `input_slice` / `lambda.expression`
are Python source strings evaluated on tensors (backbone.py:240,255,259,274,424-426) -- configs are trusted
input there and here; a small `tf` namespace maps the TensorFlow calls that appear in the sample configs
onto torch.
"""
import math

import torch
from torch import nn

from easyrec_b200 import embedding as E
from easyrec_b200 import interactions as I
from easyrec_b200 import layers as L


class _TF(object):
  """the handful of tf.* calls used by `input_fn` / `lambda` strings in samples/model_config/*.config"""
  float32 = torch.float32

  @staticmethod
  def concat(values, axis=-1):
    return torch.cat(list(values), dim=axis)

  @staticmethod
  def stack(values, axis=0):
    return torch.stack(list(values), dim=axis)

  @staticmethod
  def reduce_sum(x, axis=None, keepdims=False):
    return x.sum() if axis is None else x.sum(dim=axis, keepdim=keepdims)

  @staticmethod
  def reduce_mean(x, axis=None, keepdims=False):
    return x.mean() if axis is None else x.mean(dim=axis, keepdim=keepdims)

  @staticmethod
  def expand_dims(x, axis):
    return x.unsqueeze(axis)

  @staticmethod
  def squeeze(x, axis=None):
    return x.squeeze() if axis is None else x.squeeze(axis)

  @staticmethod
  def reshape(x, shape):
    return x.reshape(*shape)

  @staticmethod
  def multiply(a, b):
    return a * b

  @staticmethod
  def add(a, b):
    return a + b

  @staticmethod
  def subtract(a, b):
    return a - b

  @staticmethod
  def square(x):
    return x * x

  @staticmethod
  def add_n(inputs):
    out = inputs[0]
    for t in inputs[1:]:
      out = out + t
    return out

  @staticmethod
  def unstack(value, num=None, axis=0):
    return list(torch.unbind(value, dim=axis))


_EVAL_ENV = {'tf': _TF, 'torch': torch, '__builtins__': {'len': len, 'range': range, 'list': list, 'sum': sum,
                                                          'int': int, 'float': float, 'tuple': tuple}}


def _eval(src):
  return eval(src, dict(_EVAL_ENV))  # noqa: S307 -- same trust model as the reference (backbone.py:240)


class MLP(nn.Module):
  """layers/keras/blocks.py:33-129: Dense -> BatchNorm -> activation per layer (bias off by default,
  he_uniform kernels); the last layer uses use_final_bn / final_activation / use_final_bias."""

  def __init__(self, n_in, conf, generator=None):
    super().__init__()
    units = list(conf.hidden_units)
    assert units, 'MLP takes at least one hidden unit'
    if conf.use_bn_after_activation:
      raise NotImplementedError('MLP.use_bn_after_activation')
    # activation / final_activation by name (layers/keras/activation.py:97-110 -> utils/activation.py:get_activation);
    # (a pb-message MLP reads the proto default 'relu' for an unset final_activation: Parameter.get_or_default returns a
    # non-empty string field as is, layers/utils.py:224-227)
    kinds = [L.activation_kind(conf.activation), L.activation_kind(conf.final_activation)]
    self.layers = nn.ModuleList()
    self.acts = nn.ModuleList()
    self.dropouts = nn.ModuleList()
    rates = [float(r) for r in conf.dropout_ratio]
    n = len(units)
    for i, u in enumerate(units):
      last = i + 1 == n
      # Dropout(rate) after the layer's activation when 0 < rate < 1; layers beyond the list get none (blocks.py:56-67,
      # 113-117)
      rate = rates[i] if i < len(rates) else 0.0
      if rate >= 1.0:
        raise ValueError('invalid dropout_ratio: %.3f' % rate)
      self.dropouts.append(L.Dropout(rate) if rate > 0.0 else nn.Identity())
      bn = conf.use_final_bn if last else conf.use_bn
      kind = kinds[1] if last else kinds[0]
      lay = L.DenseLayer(n_in, u, bn, kind == 'relu', generator)
      self.acts.append(L._act_module(kind, u))
      lim = math.sqrt(6.0 / n_in)   # he_uniform
      with torch.no_grad():
        lay.kernel.uniform_(-lim, lim, generator=generator)
      use_bias = conf.use_final_bias if last else conf.use_bias
      if not use_bias:
        lay.bias.requires_grad_(False)   # stays zero: tf Dense(use_bias=False)
      self.layers.append(lay)
      n_in = u
    self.out_dim = n_in

  def forward(self, x):
    if isinstance(x, (list, tuple)):
      x = torch.cat(list(x), dim=-1)
    for lay, act, drop in zip(self.layers, self.acts, self.dropouts):
      x = drop(act(lay(x)))
    return x


class Cross(nn.Module):
  """DCN-v2 cross (layers/keras/interaction.py:249-286): x0 * (W x + b [+ diag_scale x]) + x with a full-rank
  W, or W = U V (projection_dim: U [d, p] without bias, V [p, d] with the bias) for the low-rank variant
  (kernel_initializer truncated_normal, bias zeros)."""

  def __init__(self, dim, params, generator=None):
    super().__init__()
    self.diag_scale = float(params.get('diag_scale', 0.0))
    if self.diag_scale < 0:
      raise ValueError('`diag_scale` should be non-negative. Got `diag_scale` = %r' % self.diag_scale)
    proj = params.get('projection_dim')
    self.dense_u = None
    if proj:
      self.dense_u = L.Dense(dim, int(proj), generator)
      self.dense_u.bias.requires_grad_(False)        # Dense(use_bias=False): the zero bias never moves
      self.dense = L.Dense(int(proj), dim, generator)
    else:
      self.dense = L.Dense(dim, dim, generator)
    with torch.no_grad():
      for d in (self.dense_u, self.dense):
        if d is not None:
          nn.init.trunc_normal_(d.kernel, std=0.05, a=-0.1, b=0.1, generator=generator)
    if params.get('use_bias', True) is False:
      self.dense.bias.requires_grad_(False)
    self.out_dim = dim

  def forward(self, inputs):
    x0, x = inputs if isinstance(inputs, (list, tuple)) else (inputs, inputs)
    if x0.shape[-1] != x.shape[-1]:
      raise ValueError('`x0` and `x` dimension mismatch! Got `x0` dimension %d, and x dimension %d. This case is '
                       'not supported yet.' % (x0.shape[-1], x.shape[-1]))
    x = x.contiguous()
    prod = self.dense(x) if self.dense_u is None else self.dense(self.dense_u(x))
    if self.diag_scale:
      prod = prod + self.diag_scale * x
    return x0 * prod + x


class FM(nn.Module):
  """layers/keras/interaction.py:24-44: list of [B, D] (or [B, F, D]) -> 0.5((sum v)^2 - sum v^2);
  use_variant keeps [B, D], else reduce_sum -> [B, 1]."""

  def __init__(self, conf):
    super().__init__()
    self.use_variant = bool(conf.use_variant) if conf is not None else False

  def forward(self, inputs):
    if isinstance(inputs, (list, tuple)):
      n_field, dim = len(inputs), inputs[0].shape[-1]
      x = torch.cat(list(inputs), dim=-1)
    else:
      n_field, dim = inputs.shape[1], inputs.shape[2]
      x = inputs.reshape(inputs.shape[0], n_field * dim)
    y = E.fm(x.contiguous(), n_field, dim)
    return y if self.use_variant else y.sum(dim=1, keepdim=True)


class DotInteraction(nn.Module):
  """DLRM dot interaction (layers/keras/interaction.py:47-128): features [B, F, D] -> all pairwise dot products
  of the lower triangle (with the diagonal when self_interaction), [B, F(F-1)/2] (or [B, F*F] with the upper
  triangle zeroed when skip_gather).  One F x D x F product per sample: the library's batched Gram kernel (er_gram_fwd)."""

  def __init__(self, params):
    super().__init__()
    self.self_interaction = bool(params.get('self_interaction', False))
    self.skip_gather = bool(params.get('skip_gather', False))
    self._idx = {}

  def out_dim(self, n):
    if self.skip_gather:
      return n * n
    return n * (n + 1) // 2 if self.self_interaction else n * (n - 1) // 2

  def forward(self, inputs):
    x = torch.stack(list(inputs), dim=1) if isinstance(inputs, (list, tuple)) else inputs
    n = x.shape[1]
    xa = I.gram(x.contiguous()).reshape(x.shape[0], n * n)
    key = (n, x.device)
    if key not in self._idx:   # static gather indices (row-major lower triangle): no boolean-mask host sync
      keep = torch.tril(torch.ones(n, n, dtype=torch.bool), diagonal=0 if self.self_interaction else -1)
      self._idx[key] = (keep.reshape(-1).nonzero()[:, 0].to(x.device), keep.reshape(1, -1).to(x.device, x.dtype))
    idx, mask = self._idx[key]
    if self.skip_gather:
      return xa * mask
    return xa.index_select(1, idx)


class SENet(nn.Module):
  """FiBiNet SENet (layers/keras/fibinet.py:14-96): per field, per squeeze group -> (max, mean); two dense layers
  (relu, linear) produce one weight per embedding element; re-weight, skip connection, layer norm."""

  def __init__(self, dims, conf, generator=None):
    super().__init__()
    self.g = conf.num_squeeze_group
    assert all(d >= self.g and d % self.g == 0 for d in dims), 'field dims must be divisible by num_squeeze_group'
    emb = sum(dims)
    red = max(1, len(dims) * self.g * 2 // conf.reduction_ratio)
    self.reduce = L.DenseLayer(len(dims) * self.g * 2, red, False, True, generator)
    self.excite = L.Dense(red, emb, generator)
    with torch.no_grad():
      nn.init.kaiming_normal_(self.reduce.kernel.t(), generator=generator)           # he_normal (fan_in)
      nn.init.xavier_normal_(self.excite.kernel, generator=generator)                # glorot_normal
    self.skip = conf.use_skip_connection
    self.ln = nn.LayerNorm(emb, eps=1e-3) if conf.use_output_layer_norm else None   # keras default epsilon
    self.out_dim = emb

  def forward(self, inputs):
    sq = []
    for e in inputs:
      ge = e.reshape(e.shape[0], self.g, e.shape[1] // self.g)
      sq.append(ge.max(dim=-1).values)
      sq.append(ge.mean(dim=-1))
    z = torch.cat(sq, dim=1).contiguous()
    w = self.excite(self.reduce(z))
    x = torch.cat(list(inputs), dim=-1)
    out = x * w
    if self.skip:
      out = out + x
    return self.ln(out) if self.ln is not None else out


class MMoE(nn.Module):
  """layers/keras/multi_task.py:47-67: num_expert expert MLPs on the same input, one softmax gate per task,
  task output = sum_e gate_e * expert_e (the mixture runs in er_mmoe_mix)."""

  def __init__(self, n_in, conf, generator=None):
    super().__init__()
    self.experts = nn.ModuleList([MLP(n_in, conf.expert_mlp, generator) for _ in range(conf.num_expert)])
    self.gates = nn.ModuleList([L.Dense(n_in, conf.num_expert, generator) for _ in range(conf.num_task)])
    self.out_dim = self.experts[0].out_dim

  def forward(self, x):
    ex = torch.stack([e(x) for e in self.experts], dim=1).contiguous()
    return [I.mmoe_mix(g(x), ex) for g in self.gates]


_KERAS_MERGE = {'Add': lambda xs: _TF.add_n(list(xs)), 'Concatenate': lambda xs: torch.cat(list(xs), dim=-1),
                'Multiply': lambda xs: __import__('functools').reduce(lambda a, b: a * b, xs)}


class _Merge(nn.Module):
  """tf.keras.layers.Add / Concatenate / Multiply on a list of tensors (layers/keras/__init__.py falls back to
  tf.keras.layers for class names it does not define itself, utils/load_class.py)."""

  def __init__(self, kind):
    super().__init__()
    self.kind = kind

  def forward(self, inputs):
    return _KERAS_MERGE[self.kind](inputs)


def _shape_of(x):
  if isinstance(x, (list, tuple)):
    return [_shape_of(t) for t in x]
  return tuple(x.shape)


def regularised_groups(backbone_config):
  """feature groups whose looked-up outputs carry the embedding regulariser (layers/input_layer.py:369-375): the ones
  read through InputLayer; the table of an `embedding_layer` block is a plain Keras Embedding without one."""
  out = set()
  for b in backbone_config.blocks:
    if b.WhichOneof('layer') == 'embedding_layer':
      continue
    for inp in b.inputs:
      if inp.WhichOneof('name') == 'feature_group_name':
        out.add(inp.feature_group_name)
  return sorted(out)


def seq_output_groups(backbone_config):
  """feature groups read by `input_layer { output_seq_and_normal_feature: true }` blocks
  (layers/common_layers.py:104-131).  The (seq, seq_len, target) triple of such a block feeds keras `DIN` blocks
  only; a group read this way is read no other way, since its sequence features are looked up un-pooled."""
  blocks = list(backbone_config.blocks) + [b for p in backbone_config.packages for b in p.blocks]
  seq_blocks, groups, other = set(), set(), set()
  for b in blocks:
    reads = [inp.feature_group_name for inp in b.inputs if inp.WhichOneof('name') == 'feature_group_name']
    if b.WhichOneof('layer') == 'input_layer' and b.input_layer.output_seq_and_normal_feature:
      if not b.input_layer.concat_seq_feature:
        raise NotImplementedError('input_layer block %s: concat_seq_feature: false (DIN takes the concatenated '
                                  'sequence)' % b.name)
      seq_blocks.add(b.name)
      groups.update(reads)
    else:
      other.update(reads)
  both = groups & other
  if both:
    raise NotImplementedError('feature group(s) %s read by output_seq_and_normal_feature and by another block'
                              % sorted(both))
  for b in blocks:
    if not any(inp.WhichOneof('name') == 'block_name' and inp.block_name in seq_blocks for inp in b.inputs):
      continue
    cls = b.keras_layer.class_name if b.WhichOneof('layer') == 'keras_layer' else b.WhichOneof('layer')
    if cls != 'DIN':
      raise NotImplementedError('backbone block %s (%s) reads the sequence output of output_seq_and_normal_feature: '
                                'only DIN blocks are built over it' % (b.name, cls))
  return groups


class DIN(nn.Module):
  """keras DIN block (layers/keras/din.py:16-67) over the (seq, seq_len, target) triple of an
  output_seq_and_normal_feature input layer: [q, k, q-k, q*k] over the T steps -> attention MLP (use_final_bn off,
  final bias on, linear final activation forced; BN / dice statistics over all B*T rows) -> scores masked beyond the
  length -> softmax, or sigmoid(s / sqrt(seq width)) -> weighted sum of the keys [-> | target].  A target narrower
  than the history is zero-padded to its width; the pooled vector then keeps the target's width."""

  def __init__(self, seq_width, query_width, conf, generator=None):
    super().__init__()
    if query_width is None:
      raise ValueError('[DIN] target feature is empty (the sequence group has no plain features)')
    if query_width > seq_width:
      raise ValueError('DIN: the embedding size of target item (%d) is larger than the one of sequence (%d)'
                       % (query_width, seq_width))
    if conf.attention_normalizer not in ('softmax', 'sigmoid'):
      raise ValueError('unsupported attention normalizer: ' + conf.attention_normalizer)
    mlp_conf = type(conf.attention_dnn)()
    mlp_conf.CopyFrom(conf.attention_dnn)
    mlp_conf.use_final_bn = False
    mlp_conf.use_final_bias = True
    mlp_conf.final_activation = 'linear'
    self.mlp = MLP(4 * seq_width, mlp_conf, generator)
    if self.mlp.out_dim != 1:
      raise NotImplementedError('DIN attention_dnn must end in one unit (has %d)' % self.mlp.out_dim)
    self.sigmoid = conf.attention_normalizer == 'sigmoid'
    self.need_target = bool(conf.need_target_feature)
    self.seq_width, self.query_width = seq_width, query_width
    self.out_dim = query_width + (seq_width if self.need_target else 0)

  def forward(self, inputs):
    keys, lens, query = inputs
    B, T, D = keys.shape
    if self.query_width < D:
      query = torch.nn.functional.pad(query, (0, D - self.query_width))
    query, keys = query.contiguous(), keys.contiguous()

    def mlp(din_in):
      return self.mlp(din_in.reshape(B * T, 4 * D))
    if self.sigmoid:
      att = I.din_sigmoid_attention(query, keys, lens, mlp, 1.0 / math.sqrt(D))
    else:
      att = I.din_attention(query, keys, lens, mlp)
    if self.query_width < D:
      att = att[:, :self.query_width]   # = the pool over keys[:, :, :query_width]: columns are summed independently
    return torch.cat([att, query], dim=1) if self.need_target else att


class Backbone(nn.Module):
  """Backbone.__call__ + Package.call (backbone.py:215-348,482-510).  Layers are instantiated by a shape-only
  dry run on `meta` tensors, so construction needs no GPU and the optimizer sees every parameter."""

  def __init__(self, config, input_layer, batch_size, generator=None):
    super().__init__()
    self.config = config
    self.input_layer = input_layer
    self.blocks = list(config.blocks)
    if config.packages:
      raise NotImplementedError('backbone packages')
    self.mods = nn.ModuleDict()
    self._gen = generator
    outs = self._run(None, batch_size, build=True)
    if isinstance(outs, (list, tuple)):   # one tensor per task (multi-task models)
      self.n_outputs = len(outs)
      self.out_dims = [o.shape[-1] for o in outs]
      self.out_dim = sum(self.out_dims)
    else:
      self.n_outputs = 1
      self.out_dims = [outs.shape[-1]]
      self.out_dim = outs.shape[-1]

  # -- inputs -----------------------------------------------------------------------------------------
  def _block_input(self, block, outputs, groups):
    ins = []
    for inp in block.inputs:
      which = inp.WhichOneof('name')
      if which == 'feature_group_name':
        v = groups(inp.feature_group_name)
      elif which == 'block_name':
        v = outputs[inp.block_name]
      else:
        raise NotImplementedError('backbone input %s' % which)
      if inp.HasField('input_slice'):     # slice first, then input_fn (layers/backbone.py:253-259)
        v = _eval('lambda x: x' + inp.input_slice.strip())(v)
      if inp.HasField('input_fn'):
        v = _eval(inp.input_fn)(v)
      ins.append(v)
    if block.merge_inputs_into_list:
      out = ins
    elif len(ins) == 1:
      out = ins[0]
    else:   # merge_inputs: lists are extended, tensors concatenated on input_concat_axis
      if any(isinstance(v, (list, tuple)) for v in ins):
        out = [t for v in ins for t in (v if isinstance(v, (list, tuple)) else [v])]
      else:
        out = torch.cat(ins, dim=block.input_concat_axis)
    if block.HasField('extra_input_fn'):
      out = _eval(block.extra_input_fn)(out)
    return out

  # -- layers -----------------------------------------------------------------------------------------
  def _keras(self, name, conf, x, build):
    if build and name not in self.mods:
      cls = conf.class_name
      d = (x[0] if isinstance(x, (list, tuple)) else x).shape[-1]
      if cls == 'MLP':
        n_in = sum(t.shape[-1] for t in x) if isinstance(x, (list, tuple)) else d
        self.mods[name] = MLP(n_in, conf.mlp, self._gen)
      elif cls == 'Cross':
        params = {}
        if conf.HasField('st_params'):
          params = {k: (v.number_value if v.HasField('number_value') else v.bool_value if v.HasField('bool_value')
                        else v.string_value) for k, v in conf.st_params.fields.items()}
        self.mods[name] = Cross(d, params, self._gen)
      elif cls == 'FM':
        self.mods[name] = FM(conf.fm if conf.HasField('fm') else None)
      elif cls == 'MMoE':
        self.mods[name] = MMoE(d, conf.mmoe, self._gen)
      elif cls == 'SENet':
        assert isinstance(x, (list, tuple)), 'SENet takes the feature list (input_layer.only_output_feature_list)'
        self.mods[name] = SENet([t.shape[-1] for t in x], conf.senet, self._gen)
      elif cls in _KERAS_MERGE:       # stock tf.keras.layers merge layers: no parameters
        self.mods[name] = _Merge(cls)
      elif cls == 'DotInteraction':
        params = {}
        if conf.HasField('st_params'):
          params = {k: (v.bool_value if v.HasField('bool_value') else v.number_value)
                    for k, v in conf.st_params.fields.items()}
        self.mods[name] = DotInteraction(params)
      elif cls == 'DIN':
        if not (isinstance(x, (list, tuple)) and len(x) == 3 and x[0].dim() == 3):
          raise NotImplementedError('DIN block %s takes the (seq, seq_len, target) output of an input_layer block with '
                                    'output_seq_and_normal_feature' % name)
        self.mods[name] = DIN(x[0].shape[-1], None if x[2] is None else x[2].shape[-1], conf.din, self._gen)
      else:
        raise NotImplementedError('backbone keras_layer %s' % cls)
    mod = self.mods[name]
    if build:   # shape-only: no kernels
      first = x[0] if isinstance(x, (list, tuple)) else x
      lead = tuple(first.shape[:-1])
      if isinstance(mod, MLP):
        return torch.empty(lead + (mod.out_dim,), device='meta')
      if isinstance(mod, Cross):
        return torch.empty(tuple(first.shape), device='meta')
      if isinstance(mod, FM):
        dim = first.shape[-1]
        return torch.empty((first.shape[0], dim if mod.use_variant else 1), device='meta')
      if isinstance(mod, MMoE):
        return [torch.empty(lead + (mod.out_dim,), device='meta') for _ in mod.gates]
      if isinstance(mod, SENet):
        return torch.empty((first.shape[0], mod.out_dim), device='meta')
      if isinstance(mod, DotInteraction):
        n = len(x) if isinstance(x, (list, tuple)) else first.shape[1]
        return torch.empty((first.shape[0], mod.out_dim(n)), device='meta')
      if isinstance(mod, DIN):
        return torch.empty((first.shape[0], mod.out_dim), device='meta')
    return mod(x)

  def _layer(self, name, conf, x, build):
    which = conf.WhichOneof('layer')
    if which == 'keras_layer':
      return self._keras(name, conf.keras_layer, x, build)
    if which == 'lambda':
      return _eval(getattr(conf, 'lambda').expression)(x)
    if which == 'recurrent':
      rc = conf.recurrent
      fixed = rc.fixed_input_index if rc.HasField('fixed_input_index') else -1
      out = list(x) if fixed >= 0 else x
      for i in range(rc.num_steps):
        o = self._keras('%s_%d' % (name, i), rc.keras_layer, out, build)
        if fixed >= 0:
          j = 0
          for idx in range(len(out)):
            if idx == fixed:
              continue
            out[idx] = o[j] if isinstance(o, (list, tuple)) else o
            j += 1
        else:
          out = o
      if fixed >= 0:
        out = [t for idx, t in enumerate(out) if idx != fixed]
        return out[0] if len(out) == 1 else out
      return out
    if which == 'repeat':
      rp = conf.repeat
      outs = []
      for i in range(rp.num_repeat):
        xi = x
        if rp.HasField('input_slice'):
          xi = _eval('lambda x, i: x' + rp.input_slice.strip())(xi, i)
        if rp.HasField('input_fn'):
          xi = _eval(rp.input_fn)(xi, i)
        outs.append(self._keras('%s_%d' % (name, i), rp.keras_layer, xi, build))
      if len(outs) == 1:
        return outs[0]
      if rp.HasField('output_concat_axis'):
        return torch.cat(outs, dim=rp.output_concat_axis)
      return outs
    raise NotImplementedError('backbone layer %s' % which)

  # -- execution --------------------------------------------------------------------------------------
  def _run(self, group_tensors, batch_size, build=False):
    il = self.input_layer

    def groups(name, as_list=False):
      if build:
        if as_list:
          return [torch.empty(batch_size, e.width, device='meta') for e in il.group_layout[name]]
        return torch.empty(batch_size, il.group_width(name), device='meta')
      return list(group_tensors[name][1]) if as_list else group_tensors[name][0]

    def seq_group(name):
      # EnhancedInputLayer with output_seq_and_normal_feature (layers/common_layers.py:104-131): (seq [B, T, sum D],
      # lengths of the first sequence feature, plain features concatenated or None)
      if build:
        sl = il.seq_group_layout[name]
        return (torch.empty(batch_size, sl['T'], sum(e.dim for e in sl['seq']), device='meta'),
                torch.empty(batch_size, dtype=torch.int32, device='meta'),
                torch.empty(batch_size, il.group_width(name), device='meta') if il.group_layout[name] else None)
      return group_tensors[name][:3]

    outputs = {}
    for block in self.blocks:
      which = block.WhichOneof('layer')
      # EnhancedInputLayer.call (layers/common_layers.py:142-190): the group as one matrix, as its feature list,
      # as a [B, F, D] stack, or as the (matrix, list) pair that later blocks pick apart with input_slice
      ilc = block.input_layer if which == 'input_layer' else None
      mode = 'seq' if ilc and ilc.output_seq_and_normal_feature else \
          'list' if ilc and ilc.only_output_feature_list else '3d' if ilc and ilc.only_output_3d_tensor else \
          'both' if ilc and ilc.output_2d_tensor_and_feature_list else '2d'
      if mode == 'seq':
        getter = seq_group
      elif mode == '2d':
        getter = groups
      elif mode == 'list':
        getter = lambda n: groups(n, True)  # noqa: E731
      elif mode == '3d':
        getter = lambda n: torch.stack(groups(n, True), dim=1)  # noqa: E731
      else:
        getter = lambda n: (groups(n), groups(n, True))  # noqa: E731
      if which == 'embedding_layer':
        # keras EmbeddingLayer over the bucketized features of one group (layers/keras/embedding.py:26-81,
        # layers/backbone.py:314-318): the fused lookup has already produced the group in its concat layout
        # (builder.embedding_layer_tables gave its features the block's width and their own tables)
        name = block.inputs[0].feature_group_name
        outputs[block.name] = groups(name) if block.embedding_layer.concat else groups(name, True)
        continue
      x = self._block_input(block, outputs, getter)
      if which == 'input_layer':
        # (the sequence output returns before dropout / normalisation are applied, common_layers.py:103-105)
        if mode != 'seq' and any(0.0 < r < 1.0 for r in (ilc.dropout_rate, ilc.feature_dropout_rate)) or ilc.do_batch_norm or ilc.do_layer_norm:
          raise NotImplementedError('input_layer block %s: dropout / feature dropout / normalisation' % block.name)
        out = x
      elif which in ('keras_layer', 'lambda', 'recurrent', 'repeat'):
        out = self._layer(block.name, block, x, build)
      elif which is None:   # sequential `layers` or a pure input-merging block
        out = x
        for i, ly in enumerate(block.layers):
          out = self._layer('%s_l%d' % (block.name, i), ly, out, build)
      else:
        raise NotImplementedError('backbone block type %s' % which)
      outputs[block.name] = out
    names = list(self.config.output_blocks) or list(self.config.concat_blocks)
    if not names:   # leaves of the DAG (backbone.py:196-206)
      used = {inp.block_name for b in self.blocks for inp in b.inputs if inp.WhichOneof('name') == 'block_name'}
      names = [b.name for b in self.blocks if b.name not in used]
    outs = []
    for n in names:
      o = outputs[n]
      outs.extend(o if isinstance(o, (list, tuple)) else [o])
    if self.config.concat_blocks and not self.config.output_blocks:
      result = outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)
    else:   # output_blocks / DAG leaves: tensors are handed on as a list (backbone.py:330-348)
      result = outs[0] if len(outs) == 1 else outs
    if self.config.HasField('top_mlp'):
      if isinstance(result, (list, tuple)):
        result = torch.cat(list(result), dim=-1)
      if build:
        if 'backbone_top_mlp' not in self.mods:
          self.mods['backbone_top_mlp'] = MLP(result.shape[-1], self.config.top_mlp, self._gen)
        return torch.empty(tuple(result.shape[:-1]) + (self.mods['backbone_top_mlp'].out_dim,), device='meta')
      result = self.mods['backbone_top_mlp'](result)
    return result

  def forward(self, group_tensors):
    """group_tensors: InputLayer.lookup() result {group: (concat, per-feature list)}."""
    return self._run(group_tensors, self.input_layer.batch_size, build=False)
