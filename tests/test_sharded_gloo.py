"""CPU, world_size 2 and 8 over gloo: the HOST logic of the row-sharded lookup (easyrec_b200/sharded.py
ShardedLookup) - owner grouping into fixed-capacity per-peer blocks, the id / row / gradient all-to-alls, the position
map that pools the received rows, the requester-side duplicate sums and the owner-side 1/N gradient scale
(compat/optimizers.py:315-316).

The CUDA kernels cannot run here, so they are replaced by the oracle-backed doubles of tests/host_doubles.py - the
kernels themselves are compared with that oracle on the GPU (tests/test_gpu_sparse.py, tests/test_gpu_sharded.py on
2 GPUs).  Every rank checks its pooled output and its updated shard against the oracle run on the UNSHARDED table and
the concatenated global batch."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, port, ret, world):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  sys.path.insert(0, HERE)
  import host_doubles
  host_doubles.install_sparse(setattr)
  from easyrec_b200 import _lib, embedding as E, kernels as K
  from easyrec_b200.sharded import ShardedLookup
  from oracle import oracle as O
  B, D = 24, 4
  tables = [('t0', 101), ('t1', 37)]                      # odd sizes: the last shards carry padding rows
  modes = [(_lib.BUCKET_FARM_DECIMAL, 101, 't0'), (_lib.BUCKET_MOD, 37, 't1'), (_lib.BUCKET_FARM_DECIMAL, 101, 't0')]
  slots = [E.Slot('s%d' % i, t, m, nb) for i, (m, nb, t) in enumerate(modes)]
  F = len(slots)
  full = torch.from_numpy(np.random.default_rng(7).normal(0, 0.1, (101 + 37, D)).astype(np.float32))
  g0 = {'t0': 0, 't1': 101}
  arena = E.Arena(D, 'cpu', shard_n=world, shard_rank=rank)
  for name, v in tables:
    arena.add_table(name, v)

  def init_fn(w):
    w.zero_()
    for name, v in tables:
      off = arena.tables[name][0]
      shard = full[g0[name]:g0[name] + v][rank::world]
      w[off:off + shard.shape[0]].copy_(shard)
  arena.materialize(_lib.OPT_ADAGRAD, init_fn=init_fn)
  call = E.ArenaCall(arena, slots, B, [F * D], single_valued=True)
  sl = ShardedLookup(call, world, rank)
  rng = np.random.default_rng(100 + rank)
  ids = (rng.zipf(1.3, F * B) % 5000).astype(np.int64)
  ids[rng.integers(0, F * B, 5)] = -5
  outs = call.alloc_outputs()
  sl.forward(torch.from_numpy(ids), None, outs)
  sl.check()                                              # no lookup lost to a full per-peer block
  out = outs[0]
  mode_l = np.repeat([m for m, _, _ in modes], B)
  nb_l = np.repeat([nb for _, nb, _ in modes], B)
  off_l = np.repeat([g0[t] for _, _, t in modes], B)
  g_rows, _ = O.bucketize(ids, mode_l, nb_l, off_l)
  want = full.numpy()[g_rows].reshape(F, B, D).transpose(1, 0, 2).reshape(B, F * D)
  assert np.array_equal(out.numpy()[:, :F * D], want), 'sharded forward differs'
  gout = rng.normal(0, 0.1, (B, out.shape[1])).astype(np.float32)
  out.grad = torch.from_numpy(gout)
  sl.backward_update(outs, K.make_opt(_lib.OPT_ADAGRAD, 0.05))
  all_rows, all_g = [None] * world, [None] * world
  dist.all_gather_object(all_rows, g_rows)
  dist.all_gather_object(all_g, gout[:, :F * D].reshape(B, F, D).transpose(1, 0, 2).reshape(F * B, D))
  t = full.numpy().copy()
  acc = np.full_like(t, 0.1)
  O.embedding_bwd(t, acc, None, np.concatenate(all_rows), None, np.concatenate(all_g), O.OPT_ADAGRAD, 0.05,
                  grad_scale=1.0 / world)
  touched = 0
  for name, v in tables:
    off = arena.tables[name][0]
    want_shard = t[g0[name]:g0[name] + v][rank::world]
    got = arena.weight[off:off + want_shard.shape[0]].numpy()
    np.testing.assert_allclose(got, want_shard, rtol=0, atol=1e-6)
    touched += int((got != full.numpy()[g0[name]:g0[name] + v][rank::world]).any())
  ret[rank] = touched
  dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize('world', [2, 8])
def test_row_sharded_lookup_matches_unsharded_oracle_gloo(world):
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret, world), nprocs=world, join=True)
  assert len(ret) == world and sum(ret.values()) > 0      # every rank finished; updates really happened
