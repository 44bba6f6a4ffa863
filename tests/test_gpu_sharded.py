"""2 GPUs: the row-sharded (EmbeddingParallel) lookup, sharded.ShardedLookup with NCCL all-to-all, vs the CPU oracle
run on the unsharded table and the concatenated global batch.  Skipped on boxes with fewer than 2 GPUs.

Checks: owner/local-row rule (bit exact, via the pooled values), forward pooled outputs (exact: each
output is a copy/sum of table rows in lookup order), and the post-step shards after the gradient
all-to-all + fused Adagrad with the 1/N scaling of compat/optimizers.py:315-316 (<= 1e-6)."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
WORLD = 2


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, port, ret):
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(rank)
  dev = 'cuda:%d' % rank
  dist.init_process_group('nccl', rank=rank, world_size=WORLD, device_id=torch.device(dev))
  from easyrec_b200 import _lib, embedding as E, kernels as K
  from easyrec_b200.sharded import ShardedLookup
  from oracle import oracle as O
  B, D = 512, 16
  tables = [('t0', 10007), ('t1', 5003)]
  modes = [(_lib.BUCKET_FARM_DECIMAL, 10007, 't0'), (_lib.BUCKET_MOD, 5003, 't1'), (_lib.BUCKET_FARM_DECIMAL, 10007, 't0')]
  slots = [E.Slot('s%d' % i, t, m, nb) for i, (m, nb, t) in enumerate(modes)]
  F = len(slots)
  full = torch.from_numpy(np.random.default_rng(7).normal(0, 0.01, (10007 + 5003, D)).astype(np.float32))
  g0 = {'t0': 0, 't1': 10007}
  arena = E.Arena(D, dev, shard_n=WORLD, shard_rank=rank)
  for name, v in tables:
    arena.add_table(name, v)

  def init_fn(w):
    w.zero_()
    for name, v in tables:
      off = arena.tables[name][0]
      shard = full[g0[name]:g0[name] + v][rank::WORLD]
      w[off:off + shard.shape[0]].copy_(shard)
  arena.materialize(_lib.OPT_ADAGRAD, init_fn=init_fn)
  call = E.ArenaCall(arena, slots, B, [F * D], single_valued=True)
  sl = ShardedLookup(call, WORLD, rank)
  rng = np.random.default_rng(100 + rank)
  ids = (rng.zipf(1.2, F * B) % 50000).astype(np.int64)
  ids[rng.integers(0, F * B, 20)] = -5  # negative ids are valid for hash / floored mod
  outs = call.alloc_outputs()
  sl.forward(torch.from_numpy(ids).to(dev), None, outs)
  sl.check()                            # no lookup lost to a full per-peer block
  out = outs[0]
  # ---- oracle: unsharded rows and pooled outputs ----
  mode_l = np.repeat([m for m, _, _ in modes], B)
  nb_l = np.repeat([nb for _, nb, _ in modes], B)
  off_l = np.repeat([g0[t] for _, _, t in modes], B)
  g_rows, _ = O.bucketize(ids, mode_l, nb_l, off_l)
  want = full.numpy()[g_rows].reshape(F, B, D).transpose(1, 0, 2).reshape(B, F * D)
  assert np.array_equal(out.cpu().numpy(), want), 'sharded forward differs'
  # ---- backward: all ranks' gradients meet on the owners ----
  gout = rng.normal(0, 0.1, (B, F * D)).astype(np.float32)
  out.grad = torch.from_numpy(gout).to(dev)
  sl.backward_update(outs, K.make_opt(_lib.OPT_ADAGRAD, 0.05))
  torch.cuda.synchronize()
  # gather everyone's (rows, grads) on the host and run the oracle on the global batch
  all_rows = [None] * WORLD
  all_g = [None] * WORLD
  dist.all_gather_object(all_rows, g_rows)
  dist.all_gather_object(all_g, gout.reshape(B, F, D).transpose(1, 0, 2).reshape(F * B, D))
  t = full.numpy().copy()
  acc = np.full_like(t, 0.1)
  O.embedding_bwd(t, acc, None, np.concatenate(all_rows), None, np.concatenate(all_g), O.OPT_ADAGRAD, 0.05,
                  grad_scale=1.0 / WORLD)
  for name, v in tables:
    off = arena.tables[name][0]
    want_shard = t[g0[name]:g0[name] + v][rank::WORLD]
    got = arena.weight[off:off + want_shard.shape[0]].cpu().numpy()
    np.testing.assert_allclose(got, want_shard, rtol=0, atol=1e-6)
    assert (got != full.numpy()[g0[name]:g0[name] + v][rank::WORLD]).any()
  ret[rank] = True
  dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_row_sharded_arena_matches_unsharded_oracle_on_2_gpus():
  if torch.cuda.device_count() < WORLD:
    pytest.skip('needs %d GPUs' % WORLD)
  import torch.multiprocessing as mp
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret), nprocs=WORLD, join=True)
  assert len(ret) == WORLD
