"""Dense layers of the interaction stage (K6 of SURVEY.md): fp32, TF-default semantics.

  DNN   layers/dnn.py:50-87   dense(glorot-uniform, zero bias) -> batch_norm -> relu [-> dropout]
  BN    tf.layers.batch_normalization defaults: momentum 0.99, epsilon 1e-3, batch statistics in
        training, *biased* variance for both the normalisation and the moving average (2-D
        inputs take TF's non-fused path)

Per layer: er_gemm (wgmma tensor cores, 3xTF32 operand split so logits stay within 1e-4 of an fp32
CPU run; forward, dX and dW read X / W[in,out] / dY in place) + liber_b200's fused bias/batch-norm/ReLU
epilogue (2 launches forward, 2 backward, deterministic statistics).  There is no torch fallback.
"""
import math
import os

import torch
from torch import nn

from easyrec_b200 import kernels as K

BN_EPS = 1e-3
BN_MOMENTUM = 0.99
_OVERLAP_DW_DX = os.environ.get('ER_OVERLAP_DW_DX', '1') == '1'
_side = {}
_defer = {'on': False, 'dirty': set()}
_planes = {'on': None}


class defer_dw_join(object):
  """Inside this context the side stream that computes the kernel gradients is NOT joined after every layer:
  the dW GEMMs (which nothing in the backward pass consumes) queue up on the side stream while the main
  stream runs the dX / batch-norm chain, and everything is joined once on exit.  The trainer wraps
  loss.backward() in it; code that reads .grad right after a layer's backward must not."""

  def __enter__(self):
    self.prev = _defer['on']
    _defer['on'] = True
    return self

  def __exit__(self, *exc):
    _defer['on'] = self.prev
    if not self.prev:
      for dev in list(_defer['dirty']):
        torch.cuda.current_stream(dev).wait_stream(_side[dev])
      _defer['dirty'].clear()
    return False


def tower_kernels(model):
  """Kernels of the model's dense layers whose forward and dX run on the tensor-core GEMM (both sides at least 8): the
  ones whose tf32 planes a trainer splits once per step (kernels.DensePlanes)."""
  return [m.kernel for m in model.modules()
          if isinstance(m, DenseLayer) and m.kernel.requires_grad and min(m.kernel.shape) >= 8]


class use_planes(object):
  """Inside this context a dense layer whose kernel is in `planes` (a kernels.DensePlanes refreshed from the
  kernels' current values, which must not change inside the context) gives its forward and dX GEMMs the
  pre-split planes instead of the kernel; the products are bit-identical.  The trainer wraps the forward and
  backward pass of each step in it, right after the refresh; any other run splits the kernel in the GEMM."""

  def __init__(self, planes):
    self.planes = planes
    self.index = {id(w): i for i, w in enumerate(planes.kernels)} if planes is not None else {}

  def __enter__(self):
    self.prev = _planes['on']
    _planes['on'] = self
    return self

  def __exit__(self, *exc):
    _planes['on'] = self.prev
    return False


def _kernel_planes(kernel):
  """(forward planes, dX planes) of kernel while a use_planes context covers it, else (None, None)."""
  ctx = _planes['on']
  i = ctx.index.get(id(kernel)) if ctx is not None else None
  if i is None:
    return None, None
  return ctx.planes.view(i, False), ctx.planes.view(i, True)


def _side_stream(device):
  s = _side.get(device)
  if s is None:
    s = torch.cuda.Stream(device=device)
    _side[device] = s
  return s


class _DenseBNAct(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, kernel, bias, gamma, beta, moving_mean, moving_var, training, relu, ws):
    x = K.gemm_ready(x)
    ctx.kernel_param = kernel
    if hasattr(kernel, '_er_uses'):
      kernel._er_uses += 1
    fwd_planes, ctx.dx_planes = _kernel_planes(kernel)
    pk = {} if fwd_planes is None else {'planes': fwd_planes}
    fused = None
    if gamma is not None and training:
      # batch statistics come out of the GEMM epilogue; one elementwise pass normalises + activates
      fused = K.gemm_bn(x, kernel, bias, moving_mean, moving_var, BN_EPS, BN_MOMENTUM, **pk)
    if fused is not None:
      z, mean, rstd = fused
      y = K.bn_act_apply(z, bias, gamma, beta, mean, rstd, relu)
    else:
      z = K.gemm(x, kernel, **pk)
      y, mean, rstd = K.bias_bn_act_fwd(z, bias, gamma, beta, moving_mean, moving_var, BN_EPS,
                                        BN_MOMENTUM, training, relu, ws)
    ctx.relu = relu
    ctx.ws = ws
    ctx.has_bn = gamma is not None
    ctx.save_for_backward(x, kernel, bias, gamma, beta, z, y, mean, rstd)
    return y

  @staticmethod
  def backward(ctx, gy):
    x, kernel, bias, gamma, beta, z, y, mean, rstd = ctx.saved_tensors
    gy = gy.contiguous()
    out = None
    if ctx.has_bn and mean is not None and z.is_cuda:
      # the relu mask recomputed from z (exactly y > 0): y is not read
      out = K.bn_relu_bwd(z, bias, gamma, beta, mean, rstd, gy, ctx.relu, ctx.ws)
    if out is None:
      out = K.bias_bn_act_bwd(z, bias, gamma, y, gy, mean, rstd, ctx.relu, ctx.ws)
    gz, gbias, ggamma, gbeta = out
    # dW goes straight into the optimizer's flat gradient buffer when this kernel is applied once per step
    # (a fresh view object, so AccumulateGrad adopts it instead of cloning)
    kp = ctx.kernel_param
    dst = getattr(kp, '_er_grad_out', None)
    if dst is not None and getattr(kp, '_er_uses', 2) == 1 and kp.grad is None:
      gk = dst.view_as(dst)
    else:
      gk = torch.empty(x.shape[1], gz.shape[1], dtype=torch.float32, device=x.device)
    pk = {} if ctx.dx_planes is None else {'planes': ctx.dx_planes}
    if ctx.needs_input_grad[0] and x.is_cuda and _OVERLAP_DW_DX:
      # dW (split-K, few tiles) and dX (many tiles) are independent: fork dW onto a side stream so the two
      # fill the 132 SMs together (captured as a fork/join inside the step's CUDA graph).  Outputs are
      # allocated on the main stream; the side stream only launches.
      cur = torch.cuda.current_stream()
      side = _side_stream(x.device)
      side.wait_stream(cur)
      with torch.cuda.stream(side):
        K.gemm(x.t(), gz, out=gk)
      gx = K.gemm(gz, kernel.t(), **pk)
      if _defer['on']:
        # joined by defer_dw_join.__exit__; the operands must outlive this function on the side stream
        gz.record_stream(side)
        x.record_stream(side)
        _defer['dirty'].add(x.device)
      else:
        cur.wait_stream(side)
    else:
      K.gemm(x.t(), gz, out=gk)
      gx = K.gemm(gz, kernel.t(), **pk) if ctx.needs_input_grad[0] else None
    return gx, gk, gbias, ggamma, gbeta, None, None, None, None, None


class _Dense1(torch.autograd.Function):
  """tf.layers.dense(units=1): the logit head as a GEMV (one warp per row) instead of a 128-wide GEMM tile."""

  @staticmethod
  def forward(ctx, x, kernel, bias):
    if x.stride(1) != 1:
      x = x.contiguous()
    ctx.save_for_backward(x, kernel)
    return K.dense1_fwd(x, kernel, bias)

  @staticmethod
  def backward(ctx, gy):
    x, kernel = ctx.saved_tensors
    gx, gw, gb = K.dense1_bwd(x, kernel, gy.contiguous().view(-1), need_gx=ctx.needs_input_grad[0])
    return gx, gw, gb


class DenseLayer(nn.Module):
  """tf.layers.dense (kernel [in, out] glorot-uniform, bias zeros) [+ batch_norm] [+ relu]."""

  def __init__(self, n_in, n_out, use_bn, relu, generator=None):
    super().__init__()
    limit = math.sqrt(6.0 / (n_in + n_out))
    w = torch.empty(n_in, n_out)
    w.uniform_(-limit, limit, generator=generator)
    self.kernel = nn.Parameter(w)
    self.bias = nn.Parameter(torch.zeros(n_out))
    self.use_bn = use_bn
    self.relu = relu
    if use_bn:
      self.gamma = nn.Parameter(torch.ones(n_out))
      self.beta = nn.Parameter(torch.zeros(n_out))
      self.register_buffer('moving_mean', torch.zeros(n_out))
      self.register_buffer('moving_var', torch.ones(n_out))
    self.n_out = n_out
    self._ws = None
    self._ws_batch = -1

  def forward(self, x):
    if self._ws is None or self._ws_batch != x.shape[0] or self._ws.device != x.device:
      self._ws = K.dense_workspace(x.shape[0], self.n_out, x.device)
      self._ws_batch = x.shape[0]
    if self.use_bn:
      return _DenseBNAct.apply(x, self.kernel, self.bias, self.gamma, self.beta, self.moving_mean,
                               self.moving_var, self.training, self.relu, self._ws)
    if self.n_out == 1 and not self.relu and x.is_cuda and self.kernel.shape[0] <= 255:
      return _Dense1.apply(x, self.kernel, self.bias)
    return _DenseBNAct.apply(x, self.kernel, self.bias, None, None, None, None, self.training,
                             self.relu, self._ws)


class Dense(DenseLayer):
  """plain tf.layers.dense: no batch norm, no activation (logit heads)."""

  def __init__(self, n_in, n_out, generator=None):
    super().__init__(n_in, n_out, use_bn=False, relu=False, generator=generator)


class _DropoutFn(torch.autograd.Function):
  """y = x * mask / keep; the backward pass recomputes the mask from (seed, counter) - nothing is stored."""

  @staticmethod
  def forward(ctx, x, rate, seed, counter):
    ctx.rate, ctx.seed, ctx.counter = rate, seed, counter
    return K.dropout(x, rate, seed, counter)

  @staticmethod
  def backward(ctx, g):
    return K.dropout(g, ctx.rate, ctx.seed, ctx.counter), None, None, None


class Dropout(nn.Module):
  """tf.nn.dropout(x, keep_prob = 1 - ratio) of DNN.__call__ (layers/dnn.py:77-82): training only.  The mask is a
  counter-based function of (layer seed, step counter, element): the counter is a device scalar advanced once per
  training step by a hook on the upstream gradient (a tiny device add, captured with the step), so a replayed CUDA
  graph draws a fresh mask every step and forward / backward of one step agree."""
  _next_seed = [0x5EED0001]

  def __init__(self, rate):
    super().__init__()
    assert 0.0 <= rate < 1.0, 'invalid dropout_ratio: %.3f' % rate
    self.rate = float(rate)
    self.seed = Dropout._next_seed[0]
    Dropout._next_seed[0] += 0x9E3779B1
    self.register_buffer('counter', torch.zeros(1, dtype=torch.int64))

  def forward(self, x):
    if not self.training or self.rate == 0.0:
      return x
    if x.requires_grad:
      # a hook on the INPUT's gradient runs after this layer's own backward has recomputed the mask: the moment to
      # advance the counter for the next step
      x.register_hook(self._advance)
      return _DropoutFn.apply(x, self.rate, self.seed, self.counter)
    y = K.dropout(x, self.rate, self.seed, self.counter)
    self.counter.add_(1)
    return y

  def _advance(self, grad):
    self.counter.add_(1)
    return grad


def activation_kind(name):
  """activation string of a DNN / MLP config -> None (linear), 'relu' (fused in the dense epilogue) or an er_act_*
  kind.  Names as utils/activation.py:66-118 resolves them: case-insensitive short names, or a `tf.nn.<fn>` /
  `tf.<fn>` path (load_by_path); 'prelu' without arguments is tf.nn.leaky_relu there (:98-101)."""
  if name is None:
    return None
  n = str(name).strip().lower()
  for prefix in ('tf.nn.', 'tf.math.', 'tf.keras.activations.', 'tf.'):
    if n.startswith(prefix):
      n = n[len(prefix):]
      break
  if n in ('', 'linear', 'none'):
    return None
  if n == 'relu':
    return 'relu'
  if n == 'dice':
    return 'dice'
  if n in K.ACT_KINDS:
    return K.ACT_KINDS[n]
  raise NotImplementedError('activation %r (built: relu, linear, dice, %s)' % (name, ', '.join(sorted(K.ACT_KINDS))))


def _act_module(kind, units):
  """the module that follows a layer's (linear) dense / batch-norm stage: nothing for relu (fused there) and linear"""
  if kind in (None, 'relu'):
    return nn.Identity()
  if kind == 'dice':
    return Dice(units)
  return Activation(kind)


class _ActFn(torch.autograd.Function):
  """y = f(x); the backward pass recomputes f'(x) from the saved pre-activation (er_act_bwd)."""

  @staticmethod
  def forward(ctx, x, kind):
    x = x.contiguous()
    ctx.kind = kind
    ctx.save_for_backward(x)
    return K.act_fwd(x, kind)

  @staticmethod
  def backward(ctx, gy):
    (x,) = ctx.saved_tensors
    return K.act_bwd(x, gy.contiguous(), ctx.kind), None


class Activation(nn.Module):
  """one of the stateless non-relu activations of get_activation (utils/activation.py:66-118) on top of a layer whose
  dense / batch-norm epilogue ran in its linear form (layers/dnn.py:70-73, layers/keras/blocks.py:82)."""

  def __init__(self, kind):
    super().__init__()
    assert isinstance(kind, int) and kind > 0
    self.kind = kind

  def forward(self, x):
    return _ActFn.apply(x, self.kind)


DICE_EPS = 1e-9


class _DiceFn(torch.autograd.Function):
  """y = alpha (1 - p) x + p x, p = sigmoid(batch_norm(x)) - the normalisation on the batch-norm kernels (unit gamma, zero
  beta, epsilon 1e-9), the gate and its gradient terms on er_dice_*; d alpha is a column sum of the per-element terms."""

  @staticmethod
  def forward(ctx, x, alpha, ones, zeros, moving_mean, moving_var, training, ws):
    x = x.contiguous()
    xn, mean, rstd = K.bias_bn_act_fwd(x, None, ones, zeros, moving_mean, moving_var, DICE_EPS, BN_MOMENTUM, training,
                                       False, ws)
    ctx.ws = ws
    ctx.save_for_backward(x, xn, alpha, ones, mean, rstd)
    return K.dice_fwd(x, xn, alpha.contiguous())

  @staticmethod
  def backward(ctx, gy):
    x, xn, alpha, ones, mean, rstd = ctx.saved_tensors
    gd, gn, ga = K.dice_bwd(x, xn, alpha.contiguous(), gy.contiguous())
    gz, _, _, _ = K.bias_bn_act_bwd(x, None, ones, xn, gn, mean, rstd, False, ctx.ws)
    return gd + gz, ga.sum(dim=0), None, None, None, None, None, None


class Dice(nn.Module):
  """dice(x) = alphas * (1 - p) * x + p * x, p = sigmoid(batch_normalization(x, center=False, scale=False, epsilon=1e-9))
  (utils/activation.py:13-43; keras layers/keras/activation.py:24-73): alphas start at 0, the normalisation keeps its own
  moving statistics (momentum 0.99) for evaluation."""

  def __init__(self, units):
    super().__init__()
    self.units = units
    self.alphas = nn.Parameter(torch.zeros(units))
    self.register_buffer('ones', torch.ones(units))
    self.register_buffer('zeros', torch.zeros(units))
    self.register_buffer('moving_mean', torch.zeros(units))
    self.register_buffer('moving_var', torch.ones(units))
    self._ws = None
    self._ws_batch = -1

  def forward(self, x):
    if self._ws is None or self._ws_batch != x.shape[0] or self._ws.device != x.device:
      self._ws = K.dense_workspace(x.shape[0], self.units, x.device)
      self._ws_batch = x.shape[0]
    if self.training:
      return _DiceFn.apply(x, self.alphas, self.ones, self.zeros, self.moving_mean, self.moving_var, True, self._ws)
    x = x.contiguous()
    xn, _, _ = K.bias_bn_act_fwd(x, None, self.ones, self.zeros, self.moving_mean, self.moving_var, DICE_EPS, BN_MOMENTUM,
                                 False, False, self._ws)
    return K.dice_fwd(x, xn, self.alphas.detach().contiguous())


class Units(list):
  """hidden_units of a protos/dnn.proto DNN message together with its use_bn flag and dropout_ratio list (slices
  keep them)."""
  use_bn = True
  dropout = ()
  activation = 'relu'

  def __getitem__(self, k):
    v = list.__getitem__(self, k)
    if isinstance(k, slice):
      v = Units(v)
      v.use_bn = self.use_bn
      v.activation = self.activation
      v.dropout = tuple(self.dropout[k])
    return v


def units_of(dnn_config):
  """DNN message -> Units (layers/dnn.py:50-87 reads hidden_units, use_bn and dropout_ratio from the same message)."""
  u = Units(int(x) for x in dnn_config.hidden_units)
  u.use_bn = bool(dnn_config.use_bn)
  u.activation = dnn_config.activation   # 'tf.nn.relu' by default (protos/dnn.proto:11)
  activation_kind(u.activation)          # (unknown names are refused where the config is read)
  u.dropout = tuple(float(r) for r in dnn_config.dropout_ratio)
  if u.dropout and len(u.dropout) != len(u):
    raise ValueError('dropout_ratio needs one entry per hidden layer (layers/dnn.py:78 indexes it by layer)')
  return u


class DNN(nn.Module):
  """layers/dnn.py:50-87.  Inputs of rank 3 ([B, T, d], DIN attention) are flattened to rows, which
  is exactly what tf.layers.batch_normalization does on the last axis."""

  def __init__(self, n_in, hidden_units, use_bn=True, last_layer_no_activation=False,
               last_layer_no_batch_norm=False, generator=None):
    super().__init__()
    use_bn = use_bn and getattr(hidden_units, 'use_bn', True)   # protos/dnn.proto use_bn (default true)
    drop = tuple(getattr(hidden_units, 'dropout', ()))
    kind = activation_kind(getattr(hidden_units, 'activation', 'relu'))
    self.layers = nn.ModuleList()
    self.acts = nn.ModuleList()
    self.dropouts = nn.ModuleList()
    n = len(hidden_units)
    for i, u in enumerate(hidden_units):
      bn = use_bn and (i + 1 < n or not last_layer_no_batch_norm)
      act = i + 1 < n or not last_layer_no_activation
      # relu rides in the dense / batch-norm epilogue; any other activation is an elementwise pass over its linear form
      self.layers.append(DenseLayer(n_in, u, bn, act and kind == 'relu', generator))
      self.acts.append(_act_module(kind, u) if act else nn.Identity())
      # dropout follows the activation of EVERY layer, the last one included (layers/dnn.py:77-82)
      self.dropouts.append(Dropout(drop[i]) if drop and drop[i] > 0 else nn.Identity())
      n_in = u
    self.out_dim = n_in

  def forward(self, x):
    shape = x.shape
    if x.dim() == 3:
      x = x.reshape(-1, shape[-1])
    for layer, act, drop in zip(self.layers, self.acts, self.dropouts):
      x = drop(act(layer(x)))
    if len(shape) == 3:
      x = x.reshape(shape[0], shape[1], -1)
    return x

  def kernels(self):
    return [layer.kernel for layer in self.layers]


class _BNOnly(torch.autograd.Function):
  """tf.layers.batch_normalization on a feature matrix (no dense, no activation):
  model/multi_tower_din.py:103-107.  Same fused kernels with an identity pre-activation."""

  @staticmethod
  def forward(ctx, x, gamma, beta, moving_mean, moving_var, training, ws):
    x = x.contiguous()
    y, mean, rstd = K.bias_bn_act_fwd(x, None, gamma, beta, moving_mean, moving_var, BN_EPS, BN_MOMENTUM,
                                      training, False, ws)
    ctx.ws = ws
    ctx.save_for_backward(x, gamma, y, mean, rstd)
    return y

  @staticmethod
  def backward(ctx, gy):
    x, gamma, y, mean, rstd = ctx.saved_tensors
    gx, _, ggamma, gbeta = K.bias_bn_act_bwd(x, None, gamma, y, gy.contiguous(), mean, rstd, False, ctx.ws)
    return gx, ggamma, gbeta, None, None, None, None


class BatchNorm(nn.Module):

  def __init__(self, units):
    super().__init__()
    self.gamma = nn.Parameter(torch.ones(units))
    self.beta = nn.Parameter(torch.zeros(units))
    self.register_buffer('moving_mean', torch.zeros(units))
    self.register_buffer('moving_var', torch.ones(units))
    self.units = units
    self._ws = None
    self._ws_batch = -1

  def forward(self, x):
    if self._ws is None or self._ws_batch != x.shape[0] or self._ws.device != x.device:
      self._ws = K.dense_workspace(x.shape[0], self.units, x.device)
      self._ws_batch = x.shape[0]
    return _BNOnly.apply(x, self.gamma, self.beta, self.moving_mean, self.moving_var, self.training, self._ws)
