"""ctypes binding of liber_b200.so (the C ABI declared in include/er_b200.h).

There is deliberately NO fallback: if the shared library is missing or a call
fails, an exception is raised.  The oracle under /oracle is test infrastructure
and is never imported from here.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# ER_LIB_PATH: another build of the same library (A/B runs of kernel variants)
LIB_PATH = os.environ.get('ER_LIB_PATH') or os.path.join(_HERE, 'lib', 'liber_b200.so')

c_i32, c_i64, c_f32 = ctypes.c_int32, ctypes.c_int64, ctypes.c_float
c_vp, c_sz = ctypes.c_void_p, ctypes.c_size_t

# er_slot_t (include/er_b200.h), 48 bytes
SLOT_DTYPE = np.dtype(
    [('num_buckets', '<i8'), ('row_offset', '<i8'), ('seg_begin', '<i4'),
     ('n_seg', '<i4'), ('bucket_mode', '<i4'), ('combiner', '<i4'),
     ('out_buf', '<i4'), ('out_stride', '<i4'), ('out_col', '<i4'),
     ('shard_n', '<i4')],
    align=True)
assert SLOT_DTYPE.itemsize == 48
# er_dense_seg_t, 24 bytes
DENSE_SEG_DTYPE = np.dtype([('offset', '<i8'), ('n', '<i8'), ('l2', '<f4'), ('lr_mult', '<f4')], align=True)
assert DENSE_SEG_DTYPE.itemsize == 24

BUCKET_FARM_DECIMAL, BUCKET_MOD, BUCKET_IDENTITY, BUCKET_NONE, BUCKET_ONE_ROW = 0, 1, 2, 3, 4
COMBINER_SUM, COMBINER_MEAN, COMBINER_SQRTN = 0, 1, 2
COMBINER_UNIT_WEIGHTS = 16   # flag OR-ed into er_slot_t.combiner: the slot's weights[] entries are all 1.0
OPT_SGD, OPT_ADAGRAD, OPT_LAZY_ADAM, OPT_ADAM_ROWS, OPT_MOMENTUM = 0, 1, 2, 3, 4
# er_act_*: the stateless non-relu activations of utils/activation.py:get_activation
ACT_GELU, ACT_LEAKY_RELU, ACT_ELU, ACT_SELU, ACT_TANH, ACT_SWISH, ACT_SIGMOID = 1, 2, 3, 4, 5, 6, 7
MAX_BUFS = 8
ABI_VERSION = 3
CRITEO_N_DENSE, CRITEO_N_CAT = 13, 26   # ER_CRITEO_N_DENSE / ER_CRITEO_N_CAT: values per sample of a binary part
HYPER_LR, HYPER_BETA1_POWER, HYPER_BETA2_POWER, HYPER_GRAD_SCALE, HYPER_N = 0, 1, 2, 3, 4


class ErOpt(ctypes.Structure):
  """er_opt_t."""
  _fields_ = [('kind', c_i32), ('lr', c_f32), ('beta1', c_f32),
              ('beta2', c_f32), ('eps', c_f32), ('beta1_power', c_f32),
              ('beta2_power', c_f32), ('grad_scale', c_f32), ('hyper_dev', c_vp)]


class ErBnStats(ctypes.Structure):
  """er_bn_stats_t."""
  _fields_ = [('bias', c_vp), ('save_mean', c_vp), ('save_rstd', c_vp), ('moving_mean', c_vp),
              ('moving_var', c_vp), ('eps', c_f32), ('momentum', c_f32)]


class ErGemmPlane(ctypes.Structure):
  """er_gemm_plane_t."""
  _fields_ = [('src', c_vp), ('ld_row', c_i64), ('ld_k', c_i64), ('rows', c_i64), ('k', c_i64), ('hi', c_vp),
              ('lo', c_vp)]


class ErCsvCol(ctypes.Structure):
  """er_csv_col_t."""
  _fields_ = [('kind', c_i32), ('width', c_i32), ('inner_sep', ctypes.c_char), ('kv_sep', ctypes.c_char), ('pad_', ctypes.c_char * 6),
              ('default_i64', c_i64), ('default_f32', c_f32), ('pad2_', c_i32), ('default_str', ctypes.c_char_p),
              ('out', c_vp), ('lens', c_vp), ('list_cap', c_i64), ('n_vals', c_i64), ('hash_mod', ctypes.c_uint64), ('weights', c_vp),
              ('step_lens', c_vp)]


ER_OK, ER_ERR_INVALID_ARG, ER_ERR_WORKSPACE, ER_ERR_CUDA, ER_ERR_UNSUPPORTED = range(5)
CSV_SKIP, CSV_I64, CSV_F32, CSV_HASH, CSV_I64_LIST, CSV_F32_VEC, CSV_HASH_LIST, CSV_I64_KV_LIST, CSV_HASH_KV_LIST, CSV_F32_LIST, \
    CSV_I64_STEP_LIST, CSV_HASH_STEP_LIST = range(12)

# name -> (restype, argtypes); must list every symbol include/er_b200.h declares
SIGNATURES = {
    'er_abi_version': (c_i32, []),
    'er_last_error': (ctypes.c_char_p, []),
    'er_launch_count': (ctypes.c_uint64, []),
    'er_csr_workspace_bytes': (c_sz, [c_i64]),
    'er_csr_from_lens': (c_i32, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_sz,
                                 c_vp]),
    'er_bucketize': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_i32,
                             c_vp, c_vp, c_vp]),
    'er_bucketize_weighted': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_i32,
                                      c_vp, c_vp, c_vp]),
    'er_bucketize_seq': (c_i32, [c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_i32, c_vp, c_vp, c_vp]),
    'er_dropout': (c_i32, [c_vp, c_i64, ctypes.c_float, ctypes.c_uint64, c_vp, c_vp, c_vp]),
    'er_gemm_small_workspace_bytes': (c_sz, [c_i64, c_i64, c_i64]),
    'er_gemm_small': (c_i32, [c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_vp, c_sz,
                              c_vp]),
    'er_dice_fwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_vp, c_vp]),
    'er_dice_bwd': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp]),
    'er_act_fwd': (c_i32, [c_vp, c_i64, c_i32, c_vp, c_vp]),
    'er_act_bwd': (c_i32, [c_vp, c_vp, c_i64, c_i32, c_vp, c_vp]),
    'er_auc_hist': (c_i32, [c_vp, c_vp, c_i64, c_vp, c_i32, c_vp, c_vp]),
    'er_shard_group_workspace_bytes': (c_sz, [c_i64]),
    'er_shard_group': (c_i32, [c_vp, c_vp, c_i64, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_sz, c_vp]),
    'er_fingerprint64_host': (ctypes.c_uint64, [ctypes.c_char_p, c_sz]),
    'er_csv_parse': (c_i32, [c_vp, c_sz, ctypes.c_char, ctypes.POINTER(ErCsvCol), c_i32, c_i64, c_i32,
                             ctypes.POINTER(c_i64), ctypes.POINTER(c_sz)]),
    'er_csv_parse_lines': (c_i32, [c_vp, c_sz, ctypes.c_char, ctypes.POINTER(ErCsvCol), c_i32, c_i64, c_i32, c_i64, c_i64,
                                   ctypes.POINTER(c_i64), ctypes.POINTER(c_sz), ctypes.POINTER(c_i64)]),
    'er_fingerprint64_i64': (c_i32, [c_vp, c_i64, c_vp]),
    'er_binary_unpack': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_vp, c_i32, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp]),
    'er_load_embed': (c_i32, [ctypes.c_char_p, ctypes.c_char_p, c_i32, c_i32, c_i32, c_i64, c_vp, c_vp]),
    'er_embedding_fwd': (c_i32, [
        c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp,
        c_i32, ctypes.POINTER(c_vp), c_i32, c_vp, c_vp
    ]),
    'er_embedding_bwd_workspace_bytes': (c_sz, [c_i64, c_i32]),
    'er_embedding_bwd_presort': (c_i32, [c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_vp, c_i32, c_i32, c_vp, c_sz, c_vp]),
    'er_embedding_bwd_reuse_sort': (c_i32, [
        c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_i64,
        c_i64, c_vp, c_i32, ctypes.POINTER(c_vp), c_i32, c_vp,
        ctypes.POINTER(ErOpt), c_vp, c_vp, c_vp, c_vp, c_sz, c_vp, c_sz, c_i32, c_vp
    ]),
    'er_embedding_bwd': (c_i32, [
        c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_i64,
        c_i64, c_vp, c_i32, ctypes.POINTER(c_vp), c_i32, c_vp,
        ctypes.POINTER(ErOpt), c_vp, c_vp, c_vp, c_vp, c_sz, c_vp
    ]),
    'er_sparse_apply': (c_i32, [
        c_vp, c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_i64,
        ctypes.POINTER(ErOpt), c_vp
    ]),
    'er_adam_dense_sweep': (c_i32, [
        c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp,
        ctypes.POINTER(ErOpt), c_vp
    ]),
    'er_mark_rows': (c_i32, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i32, c_vp]),
    'er_sort_workspace_bytes': (c_sz, [c_i64]),
    'er_sort_rows': (c_i32, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_sz,
                             c_vp]),
    'er_fm_fwd': (c_i32, [c_vp, c_i64, c_i32, c_i32, c_i32, c_vp, c_vp]),
    'er_fm_bwd': (c_i32, [c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_vp, c_i32,
                          c_i32, c_vp]),
    'er_sigmoid_ce_fwd_bwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_f32, c_vp,
                                      c_vp, c_vp, c_vp]),
    'er_dense_workspace_bytes': (c_sz, [c_i64, c_i32]),
    'er_dense_apply': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i64, ctypes.POINTER(ErOpt), c_vp,
                               c_vp, c_vp]),
    'er_concat_cols': (c_i32, [ctypes.POINTER(c_vp), ctypes.POINTER(c_i32), ctypes.POINTER(c_i32), c_i32, c_i64,
                               c_vp, c_i32, c_vp]),
    'er_split_cols': (c_i32, [c_vp, c_i32, c_i64, ctypes.POINTER(c_vp), ctypes.POINTER(c_i32),
                              ctypes.POINTER(c_i32), c_i32, c_vp]),
    'er_rowsum_block_fwd': (c_i32, [c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, c_sz, c_vp]),
    'er_rowsum_block_bwd': (c_i32, [c_vp, c_vp, c_vp, c_f32, c_i64, c_i32, c_i32, c_vp, c_i32, c_vp]),
    'er_dense1_workspace_bytes': (c_sz, [c_i32]),
    'er_dense1_fwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp]),
    'er_dense1_bwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_i32, c_vp, c_vp, c_vp, c_sz, c_vp]),
    'er_gemm_bn_workspace_bytes': (c_sz, [c_i64, c_i64]),
    'er_gemm_bn': (c_i32, [c_vp, c_i64, c_i32, c_vp, c_i64, c_i32, c_vp, c_i64, c_i64, c_i64, c_i64,
                           ctypes.POINTER(ErBnStats), c_vp, c_sz, c_vp]),
    'er_bn_act_apply': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp]),
    'er_fm_block_workspace_bytes': (c_sz, [c_i64]),
    'er_fm_block_fwd': (c_i32, [c_vp, c_i64, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp, c_sz, c_vp]),
    'er_fm_block_bwd': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_f32, c_i64, c_i32, c_i32, c_i32, c_i32, c_vp, c_i32,
                                c_vp]),
    'er_gemm_plane_floats': (c_sz, [c_i64, c_i64]),
    'er_gemm_split_planes': (c_i32, [ctypes.POINTER(ErGemmPlane), c_i32, c_vp]),
    'er_gemm_planes': (c_i32, [c_vp, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64,
                               ctypes.POINTER(ErBnStats), c_vp, c_sz, c_vp]),
    'er_gemm_workspace_bytes': (c_sz, [c_i64, c_i64, c_i64]),
    'er_gemm': (c_i32, [c_vp, c_i64, c_i32, c_vp, c_i64, c_i32, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64,
                        c_vp, c_sz, c_vp]),
    'er_bias_bn_act_fwd': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64,
                                   c_i32, c_f32, c_f32, c_i32, c_i32, c_vp,
                                   c_vp, c_vp, c_vp, c_sz, c_vp]),
    'er_bias_bn_act_bwd': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                   c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp,
                                   c_vp, c_sz, c_vp]),
    'er_din_concat_fwd': (c_i32, [c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp]),
    'er_din_concat_bwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp]),
    'er_din_pool_fwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp]),
    'er_din_pool_bwd': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp]),
    'er_din_sigmoid_pool_fwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_f32, c_vp, c_vp, c_vp]),
    'er_din_sigmoid_pool_bwd': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_f32, c_vp, c_vp, c_i32,
                                        c_vp]),
    'er_cross_fwd': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_vp, c_vp, c_vp]),
    'er_cross_workspace_bytes': (c_sz, [c_i64, c_i32]),
    'er_cross_bwd': (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp, c_i32,
                             c_vp, c_sz, c_vp]),
    'er_mmoe_mix_fwd': (c_i32, [c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp]),
    'er_mmoe_mix_bwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp]),
    'er_gram_fwd': (c_i32, [c_vp, c_i64, c_i32, c_i32, c_vp, c_vp]),
    'er_gram_bwd': (c_i32, [c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp]),
    'er_l2norm_fwd': (c_i32, [c_vp, c_i64, c_i32, c_vp, c_vp, c_vp]),
    'er_l2norm_bwd': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_vp, c_vp]),
    'er_inbatch_softmax_ce': (c_i32, [c_vp, c_vp, c_vp, c_i64, c_i32, c_f32, c_vp, c_vp, c_vp, c_vp]),
}

_lib = None


class ErError(RuntimeError):
  pass


def load():
  """Load liber_b200.so once; raise if it is absent (no CPU fallback exists)."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise ErError(
        'liber_b200.so not found at %s: build it with '
        '`python -c "import __graft_entry__ as g; g.build()"` or '
        '`make -C easyrec_b200/csrc`. There is no CPU fallback.' % LIB_PATH)
  lib = ctypes.CDLL(LIB_PATH)
  for name, (res, args) in SIGNATURES.items():
    fn = getattr(lib, name)  # AttributeError if the symbol is missing
    fn.restype = res
    fn.argtypes = args
  if lib.er_abi_version() != ABI_VERSION:
    raise ErError('liber_b200.so has ABI version %d, this binding needs %d: rebuild it (make -C easyrec_b200/csrc)'
                  % (lib.er_abi_version(), ABI_VERSION))
  _lib = lib
  return lib


def check(status, what):
  if status != 0:
    msg = load().er_last_error()
    raise ErError('%s failed (status %d): %s' %
                  (what, status, msg.decode() if msg else ''))


def fingerprint64(data):
  """Fingerprint64 of a bytes/str object (host side)."""
  if isinstance(data, str):
    data = data.encode('utf-8')
  return int(load().er_fingerprint64_host(data, len(data)))
