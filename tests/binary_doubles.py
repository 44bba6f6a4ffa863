"""numpy restatement of er_binary_unpack (TEST INFRASTRUCTURE): the kernel double of kernels.binary_unpack for the
host-side tests, and the reference the GPU test checks the kernel against."""
import numpy as np
import torch

from easyrec_b200 import kernels as K


def unpack(label, dense, cat, slot_cols, raw_cols):
  """numpy arrays -> (sparse_fea int64 [n_slot * B] feature-major, dense_fea float32 [B, n_raw], labels float32 [B])"""
  B = np.asarray(label).size
  cat = np.asarray(cat).reshape(B, 26).view(np.int32)   # uint32 bits read as int32
  dense = np.asarray(dense, np.float32).reshape(B, 13)
  sparse = cat[:, np.asarray(slot_cols, np.int64)].T.reshape(-1).astype(np.int64)
  return sparse, dense[:, np.asarray(raw_cols, np.int64)].copy(), np.asarray(label, np.int32).astype(np.float32)


def install(patch=setattr):
  def binary_unpack(label, dense, cat, slot_cols, raw_cols, sparse_fea=None, dense_fea=None, labels=None):
    got = unpack(label.numpy(), dense.numpy(), cat.numpy(), slot_cols.numpy(), raw_cols.numpy())
    outs = []
    for arr, out in zip(got, (sparse_fea, dense_fea, labels)):
      t = torch.from_numpy(arr)
      if out is not None:
        out.view(t.shape).copy_(t)
        t = out.view(t.shape)
      outs.append(t)
    return tuple(outs)
  patch(K, 'binary_unpack', binary_unpack)
