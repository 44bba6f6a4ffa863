"""Dict-based doubles of the key-value table kernels (csrc/kv_table.cu) for the host tests (TEST INFRASTRUCTURE), and
the restatement of their initial values.  The doubles keep the same index arrays the kernels do (a key and its pool
row per used entry, in claim order rather than hashed), so that saving and restoring read them alike."""
import numpy as np
import torch
from scipy.special import ndtri

from easyrec_b200 import _lib, kernels as K

_M = np.uint64(0xFFFFFFFFFFFFFFFF)


def _mix(z):
  z = np.asarray(z, dtype=np.uint64)
  with np.errstate(over='ignore'):
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
  return z ^ (z >> np.uint64(31))


def init_values(seed, keys, dim, stddev, truncated=True):
  """float32 [len(keys), dim]: the initial row of each key (kv_init_value in csrc/kv_table.cu), in float64 numpy"""
  k = np.asarray(keys, dtype=np.int64).astype(np.uint64)[:, None]
  with np.errstate(over='ignore'):
    h = _mix(np.uint64(seed) ^ (k * np.uint64(0xD1B54A32D192ED03)))
    c = np.arange(1, dim + 1, dtype=np.uint64)[None, :]
    bits = _mix(h + c * np.uint64(0x9E3779B97F4A7C15))
  u = ((bits >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0**-53
  p = 0.022750131948179195 + u * 0.9544997361036416 if truncated else u
  return (ndtri(p) * np.float64(np.float32(stddev))).astype(np.float32)


def _entries(index_keys, index_rows):
  k, r = index_keys.numpy(), index_rows.numpy()
  used = k != _lib.KV_EMPTY
  return dict(zip(k[used].tolist(), r[used].tolist())), int(used.sum())


def _global(keys, shard_n, shard_rank):
  return [k * shard_n + shard_rank if k >= 0 else -1 for k in keys.numpy().tolist()]


def kv_find_or_insert(index_keys, index_rows, capacity, stats, keys, rows, weight, state0, state1, state0_init, seed,
                      init_stddev, init_truncated=True, shard_n=1, shard_rank=0):
  d, n_used = _entries(index_keys, index_rows)
  out = np.empty(keys.numel(), np.int64)
  for l, k in enumerate(_global(keys, shard_n, shard_rank)):
    if k < 0:
      out[l] = -1
      continue
    r = d.get(k)
    if r is None:   # claimed in the index whether or not the pool has a row left for it
      r = int(stats[0]) if int(stats[0]) < capacity else -1
      stats[0] += 1
      d[k] = r
      index_keys[n_used], index_rows[n_used] = k, r
      n_used += 1
      if r >= 0:
        weight[r] = torch.from_numpy(init_values(seed, [k], weight.shape[1], init_stddev, init_truncated)[0])
        if state0 is not None:
          state0[r] = state0_init
        if state1 is not None:
          state1[r] = 0.0
    if r is None or r < 0:
      r = -1
      stats[1] += 1
    out[l] = r
  rows.copy_(torch.from_numpy(out))
  return rows


def kv_find(index_keys, index_rows, keys, zero_row, rows, shard_n=1, shard_rank=0):
  d, _ = _entries(index_keys, index_rows)
  rows.copy_(torch.tensor([-1 if k < 0 else (d.get(k, -1) if d.get(k, -1) >= 0 else zero_row)
                           for k in _global(keys, shard_n, shard_rank)], dtype=torch.int64))
  return rows


def kv_insert_rows(index_keys, index_rows, keys, rows, stats):
  seen = set()
  for i, (k, r) in enumerate(zip(keys.numpy().tolist(), rows.numpy().tolist())):
    if k < 0 or k in seen:
      stats[1] += 1
      continue
    seen.add(k)
    index_keys[len(seen) - 1], index_rows[len(seen) - 1] = k, r


def _exact_sharding(inner):
  """K1's double with exact integer owner / key div N for the 63-bit buckets of a row-sharded key-value table (the
  kernel divides int64s; the oracle's sharded rule is exact only for table-sized buckets): the double runs unsharded,
  then the keys are split here"""
  def bucketize(ids, slots_dev, n_slots, n_seg, seg_ids=None, row_ptr=None, rows=None, owner=None, **kw):
    sl = np.frombuffer(slots_dev.numpy().tobytes(), dtype=K.SLOT_DTYPE).copy()
    kv = (sl['num_buckets'] == _lib.KV_BUCKETS) & (sl['shard_n'] > 1)
    if not kv.any():
      return inner(ids, slots_dev, n_slots, n_seg, seg_ids=seg_ids, row_ptr=row_ptr, rows=rows, owner=owner, **kw)
    assert kv.all() and (sl['row_offset'] == 0).all(), 'a key-value table has an arena of its own'
    n = int(sl['shard_n'][0])
    sl['shard_n'] = 1
    keys = inner(ids, K.slots_to_device(sl, 'cpu'), n_slots, n_seg, seg_ids=seg_ids, row_ptr=row_ptr, **kw)
    k = keys.numpy()
    out = rows if rows is not None else torch.empty_like(ids)
    out.copy_(torch.from_numpy(np.where(k >= 0, k // n, -1)))
    if owner is not None:
      owner.copy_(torch.from_numpy(np.where(k >= 0, k % n, -1).astype(np.int32)))
    return out
  return bucketize


def install(patch=setattr):
  for name, fn in (('kv_find_or_insert', kv_find_or_insert), ('kv_find', kv_find), ('kv_insert_rows', kv_insert_rows),
                   ('bucketize', _exact_sharding(K.bucketize))):
    patch(K, name, fn)
