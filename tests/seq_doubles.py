"""Kernel double of er_bucketize_seq for the host-side tests (TEST INFRASTRUCTURE), next to tests/host_doubles.py:
the CPU oracle's K1 on every history step, then the padding mask.  Install it after host_doubles.install_all."""
import numpy as np
import torch

from easyrec_b200 import kernels as K
from host_doubles import _seg_field, _slots
from oracle import oracle as O


def bucketize_seq(ids, lens, batch, seq_len, slots_dev, n_slots, rows=None, owner=None):
  """er_bucketize_seq: step l is segment l; rows = owner = -1 at t >= the sample's length (lengths clamped to [0, T])"""
  n = ids.numel()
  sl = _slots(slots_dev)
  per = lambda f: _seg_field(sl, f, n)   # noqa: E731
  r, own = O.bucketize(ids.numpy(), per('bucket_mode'), per('num_buckets'), per('row_offset'), shard_n=per('shard_n'))
  pad = np.tile(np.arange(seq_len), lens.numel()) >= np.repeat(lens.numpy().astype(np.int64), seq_len)
  out = rows if rows is not None else torch.empty_like(ids)
  out.copy_(torch.from_numpy(np.where(pad, -1, r)))
  if owner is not None:
    owner.copy_(torch.from_numpy(np.where(pad, -1, own).astype(np.int32)))
  return out


def install(patch=setattr):
  patch(K, 'bucketize_seq', bucketize_seq)
