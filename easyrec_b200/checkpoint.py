"""Row-sharded embedding checkpoints in the reference's on-disk layout.

EmbeddingParallelSaver (compat/embedding_parallel_saver.py:99-189) keeps the sharded tables OUT of the TF
checkpoint: worker r writes its shard of variable v as raw fp32 to
    <ckpt_path>-embedding/embed-<v with '/' -> '__'>-part-<r>.bin
(row j of part r = global row j * N + r), worker 0 removes stale parts of an earlier, larger job, and the
optimizer slots of those variables are saved the same way (compat/optimizers.py:418-425).  Restore re-shards:
any worker count can read any other's files (LoadEmbed op, ops/src/load_dense_embed.cc:52-136 = er_load_embed).

Variable names follow the TF graph: `<scope>/<table>/embedding_weights:0`, slots `.../Adagrad:0`, `.../Adam:0`
(m) and `.../Adam_1:0` (v)."""
import ctypes
import glob
import os

import numpy as np
import torch

from easyrec_b200 import _lib

_SLOTS = {_lib.OPT_SGD: (), _lib.OPT_ADAGRAD: ('Adagrad',), _lib.OPT_LAZY_ADAM: ('Adam', 'Adam_1'),
          _lib.OPT_ADAM_ROWS: ('Adam', 'Adam_1'), _lib.OPT_MOMENTUM: ('Momentum',)}


def variable_name(table, scope='input_layer', slot=None):
  return '%s/%s/embedding_weights%s:0' % (scope, table, '/' + slot if slot else '')


def part_path(ckpt_path, var_name, part):
  """compat/embedding_parallel_saver.py:104-113."""
  return '%s-embedding/embed-%s-part-%d.bin' % (ckpt_path, var_name.replace('/', '__'), part)


def _part_id(path):
  return int(os.path.basename(path).split('.')[0].split('-')[-1])   # embedding_parallel_saver.py:39-43


def save_embed(rows, ckpt_path, var_name, rank, world):
  """one variable's shard (tensor or array [part_size, dim]) -> its part file; returns the path."""
  path = part_path(ckpt_path, var_name, rank)
  os.makedirs(os.path.dirname(path), exist_ok=True)
  a = rows.detach().cpu().numpy() if isinstance(rows, torch.Tensor) else np.asarray(rows)
  with open(path, 'wb') as f:
    f.write(np.ascontiguousarray(a, np.float32).tobytes())
  if rank == 0:   # clear tables of a run with more workers (:116-122)
    for old in glob.glob(part_path(ckpt_path, var_name, 0).replace('-part-0.bin', '-part-*.bin')):
      if _part_id(old) >= world:
        os.remove(old)
  return path


def load_embed(ckpt_path, var_name, dim, part_size, rank, world):
  """this worker's [part_size, dim] shard of a variable, re-sharded from whatever parts are on disk."""
  out = np.empty((part_size, dim), np.float32)
  n = ctypes.c_int64(0)
  _lib.check(_lib.load().er_load_embed(ckpt_path.encode(), ('embed-' + var_name.replace('/', '__')).encode(), rank, world,
                                       dim, part_size, out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(n)),
             'er_load_embed')
  return out


def _arena_vars(arena, scope):
  """(variable name, tensor view [local rows, dim]) for every table of the arena and its optimizer slots."""
  states = (arena.state0, arena.state1)
  for table, (off, local, _) in arena.tables.items():
    yield variable_name(table, scope), arena.weight[off:off + local]
    for slot, st in zip(_SLOTS[arena.opt_kind], states):
      yield variable_name(table, scope, slot), st[off:off + local]


def save_arena(arena, ckpt_path, scope='input_layer'):
  """every table + optimizer slot of an (un)sharded arena; returns the files written by this rank."""
  return [save_embed(view, ckpt_path, name, arena.shard_rank, arena.shard_n) for name, view in _arena_vars(arena, scope)]


def restore_arena(arena, ckpt_path, scope='input_layer'):
  """fill the arena from the part files of a run with any worker count (re-sharding on the fly)."""
  for name, view in _arena_vars(arena, scope):
    part = load_embed(ckpt_path, name, arena.dim, view.shape[0], arena.shard_rank, arena.shard_n)
    view.copy_(torch.from_numpy(part))


def kv_part_path(ckpt_path, var_name, part, ext):
  """a key-value variable's part: `.key` (int64 keys) or `.val` (fp32 [n, dim] rows in key order)
  (compat/embedding_parallel_saver.py:187-220)"""
  return '%s-embedding/embed-%s-part-%d.%s' % (ckpt_path, var_name.replace('/', '__'), part, ext)


def save_kv_arena(arena, ckpt_path, scope='input_layer'):
  """every variable of a key-value table's arena (the table and its optimizer slots) as this rank's `.key` / `.val`
  parts: the keys that hold a row, and their rows; rank 0 removes the parts of a run with more workers.  Returns the
  files written."""
  keys, rows = arena.kv.items()
  k = keys.numpy().astype(np.int64)
  files = []
  for name, view in _arena_vars(arena, scope):
    kp, vp = (kv_part_path(ckpt_path, name, arena.shard_rank, e) for e in ('key', 'val'))
    os.makedirs(os.path.dirname(kp), exist_ok=True)
    with open(kp, 'wb') as f:
      f.write(k.tobytes())
    with open(vp, 'wb') as f:
      f.write(np.ascontiguousarray(view[rows.to(view.device)].cpu().numpy(), np.float32).tobytes())
    files += [kp, vp]
    if arena.shard_rank == 0:
      for old in glob.glob(kv_part_path(ckpt_path, name, 0, 'key').replace('-part-0.key', '-part-*.key')):
        if _part_id(old) >= arena.shard_n:
          os.remove(old)
          if os.path.exists(old[:-4] + '.val'):
            os.remove(old[:-4] + '.val')
  return files


def load_kv(ckpt_path, var_name, dim, rank, world):
  """(keys int64 [n], vals fp32 [n, dim]): the keys with key % world == rank from every part on disk, in part order, as
  load_kv_embed.cc assigns them (ops/src/load_kv_embed.cc:60-130)"""
  pattern = kv_part_path(ckpt_path, var_name, 0, 'key').replace('-part-0.key', '-part-*.key')
  ks, vs = [], []
  for kp in sorted(glob.glob(pattern), key=_part_id):
    k = np.fromfile(kp, np.int64)
    v = np.fromfile(kp[:-4] + '.val', np.float32)
    if v.size != k.size * dim:
      raise ValueError('%s: %d values for %d keys of dim %d' % (kp[:-4] + '.val', v.size, k.size, dim))
    mine = k % world == rank
    ks.append(k[mine])
    vs.append(v.reshape(-1, dim)[mine])
  if not ks:
    raise FileNotFoundError('no key-value parts %s' % pattern)
  return np.concatenate(ks), np.concatenate(vs)


def restore_kv_arena(arena, ckpt_path, scope='input_layer'):
  """refill a key-value table's arena from the `.key` / `.val` parts of a run with any worker count: this rank keeps
  the keys with key % N == rank; the index is rebuilt by the bulk-insert kernel"""
  kv = arena.kv
  keys = None
  for name, view in _arena_vars(arena, scope):
    k, v = load_kv(ckpt_path, name, arena.dim, arena.shard_rank, arena.shard_n)
    if keys is None:
      keys = k
      if k.size > kv.capacity:
        raise ValueError('key-value table %s: %d keys in the checkpoint exceed max_capacity %d'
                         % (kv.name, k.size, kv.capacity))
      view.zero_()
    elif not np.array_equal(k, keys):
      raise ValueError('%s: its keys differ from the table\'s' % name)
    view[:k.size].copy_(torch.from_numpy(v))
  kv.load(torch.from_numpy(keys), torch.arange(keys.size, dtype=torch.int64))
