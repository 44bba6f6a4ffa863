"""CPU: the 3xTF32 operand split (easyrec_b200/csrc/tf32_split.cuh, shared by the GEMM's in-kernel staging and the
kernel that pre-splits the tower weights) compiled with g++: hi is x rounded to nearest onto 10 mantissa bits, and
hi + lo == x exactly, over random values, subnormals, signed zeros, values at the rounding boundary and large
exponents up to the largest magnitude whose rounding stays finite."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_FINITE_SPLIT = np.uint32(0x7f7fefff)   # above: the rounding carries into the exponent (hi = inf)


@pytest.fixture(scope='module')
def native(tmp_path_factory):
  so = str(tmp_path_factory.mktemp('native') / 'tf32_split_host.so')
  subprocess.check_call(['g++', '-O2', '-shared', '-fPIC', '-x', 'c++', '-I', os.path.join(ROOT, 'include'),
                         '-I', os.path.join(ROOT, 'easyrec_b200', 'csrc'),
                         os.path.join(ROOT, 'tests', 'native', 'tf32_split_host.cpp'), '-o', so])
  return ctypes.CDLL(so)


def _split(native, x):
  x = np.ascontiguousarray(x, np.float32)
  hi, lo = np.empty_like(x), np.empty_like(x)
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
  native.host_split_tf32(vp(x), ctypes.c_long(x.size), vp(hi), vp(lo))
  return hi, lo


def _tf32_round_nearest(x):
  """round to nearest (ties away from zero in magnitude) onto 10 mantissa bits, from the exact rational value"""
  u = x.view(np.uint32)
  return ((u + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def _inputs():
  rng = np.random.default_rng(5)
  bits = rng.integers(0, 0x7f800000, 200000, dtype=np.uint32)
  bits = bits[bits <= MAX_FINITE_SPLIT]
  edge = []
  for e in (1, 2, 100, 127, 128, 200, 253, 254):   # biased exponents, large ones included
    base = np.uint32(e << 23)
    for m in (0x0, 0x0fff, 0x1000, 0x1001, 0x1fff, 0x2000, 0x3000, 0x7fe000, 0x7fefff, 0x7fffff):
      edge.append(min(base | np.uint32(m), MAX_FINITE_SPLIT))
  sub = np.array([1, 2, 0xfff, 0x1000, 0x1001, 0x2fff, 0x3000, 0x7fffff], np.uint32)   # subnormals
  u = np.concatenate([bits, np.array(edge, np.uint32), sub, np.array([0, MAX_FINITE_SPLIT], np.uint32)])
  u = np.concatenate([u, u | np.uint32(0x80000000)])   # both signs, -0 included
  return u.view(np.float32)


def test_split_is_exact_and_hi_has_ten_mantissa_bits(native):
  x = _inputs()
  hi, lo = _split(native, x)
  assert np.isfinite(hi).all() and np.isfinite(lo).all()
  assert ((hi.view(np.uint32) & np.uint32(0x1fff)) == 0).all(), 'hi keeps more than 10 mantissa bits'
  np.testing.assert_array_equal((hi.astype(np.float64) + lo.astype(np.float64)), x.astype(np.float64))
  np.testing.assert_array_equal(hi + lo, x)
  np.testing.assert_array_equal(hi.view(np.uint32), _tf32_round_nearest(x).view(np.uint32))
  # rounding to nearest: |lo| is at most half a tf32 ulp of |x| (of the smallest normal's, for subnormal x)
  assert (np.abs(lo.astype(np.float64)) <= np.maximum(np.abs(x.astype(np.float64)), 2.0 ** -126) * 2.0 ** -11).all()


def test_split_signed_zero_and_boundary_values(native):
  x = np.array([0.0, -0.0, 1.0 + 2.0 ** -11, 1.0 + 2.0 ** -11 - 2.0 ** -23, 1.0 + 2.0 ** -11 + 2.0 ** -23],
               np.float32)
  hi, lo = _split(native, x)
  assert hi.view(np.uint32)[0] == 0 and hi.view(np.uint32)[1] == 0x80000000   # the sign of zero is kept
  assert hi[2] == np.float32(1.0 + 2.0 ** -10) and lo[2] == np.float32(-2.0 ** -11)   # a tie rounds away from zero
  assert hi[3] == np.float32(1.0) and hi[4] == np.float32(1.0 + 2.0 ** -10)


def test_split_of_the_largest_magnitudes_overflows_to_inf(native):
  """documents the limit stated in tf32_split.cuh: magnitudes that round past the largest finite float give hi = inf"""
  x = np.array([MAX_FINITE_SPLIT + 1, 0x7f7fffff], np.uint32).view(np.float32)
  hi, _ = _split(native, x)
  assert np.isinf(hi).all()
