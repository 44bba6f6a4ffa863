"""Golden vectors for the keras DIN block, produced by EXECUTING THE REFERENCE'S OWN CODE.

`DIN.call` (layers/keras/din.py:27-67) is taken from the reference source with `ast` and run against the numpy shim
of make_formula_golden.py (float32), extended by the few ops it calls besides (pad, sigmoid, transpose with a
permutation, squeeze over an axis, sequence_mask with a dtype).  The attention MLP is replaced by a fixed numpy
function whose weights are stored with the case:  score = tanh(x W1 + b1) . w2 + b2  over the [q, k, q-k, q*k] rows.

Cases: softmax and sigmoid normalisers, need_target_feature on and off, a query as wide as the history and a
narrower one (zero-padded by the block), lengths 0, 1 and T in every batch.  Keys beyond a length are NOT zero, so
the masking itself is what the outputs pin.

Run where the reference is mounted:  python tests/golden/make_din_block_golden.py
-> tests/golden/reference_din_block.json, replayed by tests/test_din_block_host.py (torch float64 restatement and the
backbone block under kernel doubles) and tests/test_gpu_din_block.py (CUDA kernels)."""
import json
import logging
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_formula_golden import _make_tf, run  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'reference_din_block.json')
f32 = np.float32


class _Shape(tuple):
  def as_list(self):
    return list(self)


class _TFArray(np.ndarray):
  """an ndarray whose .shape answers TensorShape.as_list() (keys.shape.as_list() in DIN.call)"""

  @property
  def shape(self):
    return _Shape(np.ndarray.shape.__get__(self))

  @shape.setter
  def shape(self, v):
    np.ndarray.shape.__set__(self, v)


def _tf():
  tf = _make_tf({})
  tf.pad = lambda x, paddings: np.pad(x, paddings)
  tf.transpose = lambda x, perm=None: np.transpose(x, perm)
  tf.squeeze = lambda x, axis=None: np.squeeze(x, axis=tuple(axis) if axis is not None else None)

  def sequence_mask(lengths, maxlen=None, dtype=np.bool_):
    lengths = np.asarray(lengths)
    n = int(lengths.max()) if maxlen is None else maxlen
    return (np.arange(n) < lengths[..., None]).astype(dtype)
  tf.sequence_mask = sequence_mask
  def sigmoid(x):
    with np.errstate(over='ignore'):   # exp(2^32 / sqrt(D)) of the masked steps: inf, so the weight is exactly 0
      return (f32(1) / (f32(1) + np.exp(-np.asarray(x, f32), dtype=f32))).astype(f32)
  tf.nn.sigmoid = sigmoid
  return tf


def _attention_fn(w1, b1, w2, b2):
  def f(x, training=None):
    h = np.tanh((x @ w1 + b1).astype(f32)).astype(f32)
    return (h @ w2 + b2).astype(f32)[..., None]     # [B, L, 1]
  return f


def main():
  rng = np.random.default_rng(20261016)
  out = {'generator': 'tests/golden/make_din_block_golden.py', 'mlp': 'score = tanh(x W1 + b1) . w2 + b2', 'cases': {}}
  B, T, D, H = 5, 7, 8, 6
  lens = np.array([0, 1, T, 3, T - 1], np.int32)
  line = None
  for norm in ('softmax', 'sigmoid'):
    for need_target in (True, False):
      for qw in (D, 5):
        keys = rng.normal(size=(B, T, D)).astype(f32)
        query = rng.normal(size=(B, qw)).astype(f32)
        w1 = rng.normal(0, 0.3, (4 * D, H)).astype(f32)
        b1 = rng.normal(0, 0.1, H).astype(f32)
        w2 = rng.normal(0, 0.8, H).astype(f32)
        b2 = f32(rng.normal(0, 0.1))
        layer = types.SimpleNamespace(name='din', din_layer=_attention_fn(w1, b1, w2, b2),
                                      config=types.SimpleNamespace(attention_normalizer=norm,
                                                                   need_target_feature=need_target))
        y, line = run('layers/keras/din.py', 'DIN', 'call', _tf(), layer,
                      (keys.view(_TFArray), lens, query), logging=logging,
                      get_shape_list=lambda x, n=None: list(x.shape), print=lambda *a, **k: None)
        name = '%s_%s_q%d' % (norm, 'target' if need_target else 'notarget', qw)
        out['cases'][name] = {
            'normalizer': norm, 'need_target_feature': need_target, 'keys': keys.tolist(), 'lens': lens.tolist(),
            'query': query.tolist(), 'w1': w1.tolist(), 'b1': b1.tolist(), 'w2': w2.tolist(), 'b2': float(b2),
            'y': np.asarray(y, f32).tolist()}
  out['ref'] = 'layers/keras/din.py:%d' % line
  with open(OUT, 'w') as f:
    json.dump(out, f)
  print('wrote', OUT, len(out['cases']), 'cases')


if __name__ == '__main__':
  main()
