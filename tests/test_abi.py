"""CPU: the C-ABI library loads and exports exactly what include/er_b200.h declares."""
import ctypes
import os
import re

import pytest
import torch

from easyrec_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
  src = open(os.path.join(ROOT, 'include', 'er_b200.h')).read()
  src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
  return sorted(set(re.findall(r'\b(er_[a-z0-9_]+)\s*\(', src)))


def test_header_symbols_all_exported_and_bound():
  names = _declared()
  assert len(names) >= 15
  lib = ctypes.CDLL(_lib.LIB_PATH)
  for n in names:
    assert hasattr(lib, n), 'missing export: ' + n
  assert sorted(_lib.SIGNATURES) == names


def test_abi_version_and_struct_layout():
  lib = _lib.load()
  assert lib.er_abi_version() == _lib.ABI_VERSION == 3
  assert _lib.SLOT_DTYPE.itemsize == 48
  assert ctypes.sizeof(_lib.ErOpt) == 40 and _lib.ErOpt.hyper_dev.offset == 32


def test_invalid_arguments_fail_loudly_without_gpu():
  lib = _lib.load()
  # null pointers are rejected on the host before any CUDA call
  st = lib.er_fm_fwd(None, 4, 2, 4, 8, None, None)
  assert st == 1 and b'er_fm_fwd' in lib.er_last_error()


@pytest.mark.skipif(torch.cuda.is_available(),
                    reason='placeholder pointers: with a device, test_gpu_gemm checks this on real buffers')
def test_gemm_refuses_pitch_shorter_than_row_without_gpu():
  """A pitch that is a multiple of 4 but short of the row (80 for a row of 81) is refused during validation, for
  either operand and either layout.  The pointers are placeholders, so the test only runs where no device exists:
  if validation ever admitted the call, the launch would fail for want of a device instead of touching memory."""
  lib = _lib.load()
  p = 1 << 20   # 16-byte aligned placeholder address
  bn = _lib.ErBnStats(None, p, p, None, None, 1e-3, 0.99)
  for a_mn, b_mn, lda, ldb in [(0, 1, 80, 84), (1, 1, 80, 84), (0, 0, 84, 80), (0, 1, 84, 80)]:
    st = lib.er_gemm(p, lda, a_mn, p, ldb, b_mn, None, p, 84, 81, 81, 81, None, 0, None)
    assert st == _lib.ER_ERR_INVALID_ARG and b'pitch smaller than row' in lib.er_last_error()
    st = lib.er_gemm_bn(p, lda, a_mn, p, ldb, b_mn, p, 84, 81, 81, 81, ctypes.byref(bn), p, 1 << 20, None)
    assert st == _lib.ER_ERR_INVALID_ARG and b'pitch smaller than row' in lib.er_last_error()


def test_make_slots_refuses_misaligned_vector_plans():
  """At the vector dims K2 and K7 access out_bufs[out_buf] + s*out_stride + out_col 16 bytes at a time, so the plan
  builder refuses an out_stride or out_col that is not a multiple of 4 there; scalar dims take any plan."""
  from easyrec_b200 import kernels as K

  def rec(stride, col):
    return [dict(num_buckets=10, row_offset=0, seg_begin=0, n_seg=4, bucket_mode=_lib.BUCKET_NONE, out_buf=0,
                 out_stride=stride, out_col=col)]

  for dim in K.VECTOR_DIMS:
    K.make_slots(rec(4 * dim, dim), dim)
    for stride, col in ((4 * dim + 2, 0), (4 * dim, 2), (4 * dim + 1, 3)):
      with pytest.raises(_lib.ErError, match='multiples of 4'):
        K.make_slots(rec(stride, col), dim)
  for dim in (1, 3, 6, 12):
    K.make_slots(rec(4 * dim + 1, 3), dim)
  K.make_slots(rec(18, 2))   # no dim: not checked


def test_product_never_imports_oracle():
  pkg = os.path.join(ROOT, 'easyrec_b200')
  for dp, _, files in os.walk(pkg):
    for f in files:
      if f.endswith(('.py', '.cu', '.cuh', '.h', '.cpp')):
        text = open(os.path.join(dp, f)).read()
        assert 'oracle' not in text.lower() or f == '_lib.py' or 'never' in text.lower(), (dp, f)
