"""CPU, world_size 2 over gloo, kernel doubles: train_config.gradient_clipping_by_norm under data parallel over replicated
tables (compat/optimizers.py:285-293 reduce, then :365-376 / :453-481 clip): the norm is taken over the REDUCED gradients -
dense ones averaged, every table's IndexedSlices all-gathered and divided by N (each rank's per-column slices side by
side) - and every gradient is scaled by clip / max(norm, clip).  With plain SGD the clipped step is `scale` times the
unclipped one everywhere; the norm itself is restated independently from one backward pass per rank."""
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


def _setup(rank, port, world, cuda):
  """gloo + kernel doubles on the CPU (this file's tests), NCCL + the real kernels on GPUs (tests/test_gpu_dp_extra.py)"""
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  sys.path.insert(0, HERE)
  if cuda:
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda:%d' % rank))
    torch.backends.cuda.matmul.allow_tf32 = False
    return 'cuda:%d' % rank
  dist.init_process_group('gloo', rank=rank, world_size=world)
  import host_doubles
  host_doubles.install_all()
  torch.use_deterministic_algorithms(True)
  torch.utils.deterministic.fill_uninitialized_memory = True
  return 'cpu'


def _worker(rank, port, ret, world, cuda=False):
  dev = _setup(rank, port, world, cuda)
  from test_round2_host import CLIP_CFG
  from easyrec_b200.estimator import EasyRecEstimator
  B, clipv = 16, 0.05
  rng = np.random.default_rng(10 + rank)                      # a different batch on every rank
  ids = np.stack([rng.integers(0, 6, B), rng.integers(0, 6, B), rng.integers(0, 1000, B)]).astype(np.int64)
  feats = {'sparse_fea': torch.from_numpy(ids.reshape(-1)).to(dev),
           'dense_fea': torch.from_numpy(rng.uniform(0, 2, (B, 1)).astype(np.float32)).to(dev)}
  labels = torch.from_numpy((rng.uniform(size=B) < 0.4).astype(np.float32)).to(dev)

  def make(extra):
    return EasyRecEstimator(CLIP_CFG % extra, device=dev, seed=11, world_size=world, rank=rank, embedding_parallel=False)
  plain, clip, probe = make(b''), make(b'gradient_clipping_by_norm: %g' % clipv), make(b'')
  # -- the norm, restated: this rank's per-column IndexedSlices (unique rows of each column), then over the ranks
  tr, il = probe.trainer, probe.input_layer
  tr._set_hyper()
  probe.model.train()
  tr._segment_compute(feats, labels)
  local_sq = 0.0
  for m, rows, w, outs, seg_ids in il._pending:
    D = m.arena.dim
    r = rows.cpu().numpy()
    for sl in m.slots_np:
      g = outs[int(sl['out_buf'])].grad.cpu().numpy().reshape(-1, int(sl['out_stride']))[:, int(sl['out_col']):int(sl['out_col']) + D]
      lo = int(sl['seg_begin'])
      rr = r[lo:lo + int(sl['n_seg'])]
      ww = np.ones(rr.size, np.float32) if w is None else w.cpu().numpy()[lo:lo + rr.size]
      for u in np.unique(rr[rr >= 0]):
        local_sq += float(((g[rr == u] * ww[rr == u, None]).sum(0).astype(np.float64) ** 2).sum())
  il.discard_pending()
  tot = torch.tensor([local_sq], dtype=torch.float64, device=dev)
  dist.all_reduce(tot)
  g_avg = tr.dense_opt.flat_g.double().clone()
  dist.all_reduce(g_avg)
  g_avg /= world
  l2 = torch.from_numpy(tr.dense_opt._l2_vec_np).double().to(dev)
  want = float(np.sqrt(float(tot[0]) / world ** 2 + float(((g_avg + l2 * tr.dense_opt.flat_p.double()) ** 2).sum())))
  # -- the step
  p0 = plain.trainer.dense_opt.flat_p.clone()
  t0 = {d: a.weight.clone() for d, a in plain.input_layer.arenas.items()}
  plain.trainer.train_step(feats, labels)
  clip.trainer.train_step(feats, labels)
  norm = float(clip.trainer.last_grad_norm)
  assert norm == pytest.approx(want, rel=1e-5) and norm > clipv, (norm, want)
  scale = clipv / norm
  dp_plain = plain.trainer.dense_opt.flat_p - p0
  torch.testing.assert_close(clip.trainer.dense_opt.flat_p - p0, dp_plain * scale, rtol=1e-4, atol=2e-7)
  assert float(dp_plain.abs().max()) > 1e-3
  for d, a in clip.input_layer.arenas.items():
    dt_plain = plain.input_layer.arenas[d].weight - t0[d]
    torch.testing.assert_close(a.weight - t0[d], dt_plain * scale, rtol=1e-4, atol=2e-8)
    assert float(dt_plain.abs().max()) > 1e-4
  # a second step keeps working (the factor does not accumulate in the device-resident gradient scale)
  clip.trainer.train_step(feats, labels)
  assert 0.0 < float(clip.trainer.last_grad_norm) < 10 * norm
  digest = [float(a.storage.double().sum()) for a in clip.input_layer.arenas.values()]
  digest.append(float(clip.trainer.dense_opt.flat_p.double().sum()))
  ret[rank] = tuple(digest) + (norm,)
  if cuda:
    dist.barrier()
    os._exit(0)     # (captured graphs may hold NCCL work: no destroy_process_group)
  dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_global_norm_clipping_under_data_parallel_gloo():
  world = 2
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret, world), nprocs=world, join=True)
  assert len(ret) == world and len(set(ret.values())) == 1, dict(ret)       # replicas identical, same norm everywhere


def _worker_ep(rank, port, ret, world, cuda=False):
  """row-sharded tables (EmbeddingParallel): the sparse part of the norm is what every OWNER received - one gradient
  row per (source rank, distinct row), the columns of the call merged (the reference runs ONE unique over all ids before
  the exchange, feature_column.py:263), divided by N (compat/optimizers.py:306-316) - reduced over the ranks
  (part_norms, :453-470); the owners hold their row update until the factor is known."""
  dev = _setup(rank, port, world, cuda)
  import ep_helpers
  from test_round2_host import CLIP_CFG
  from easyrec_b200.estimator import EasyRecEstimator
  B, clipv = 16, 0.05
  rng = np.random.default_rng(20 + rank)
  ids = np.stack([rng.integers(0, 6, B), rng.integers(0, 6, B), rng.integers(0, 1000, B)]).astype(np.int64)
  feats = {'sparse_fea': torch.from_numpy(ids.reshape(-1)).to(dev),
           'dense_fea': torch.from_numpy(rng.uniform(0, 2, (B, 1)).astype(np.float32)).to(dev)}
  labels = torch.from_numpy((rng.uniform(size=B) < 0.4).astype(np.float32)).to(dev)

  def make(extra, ep):
    return EasyRecEstimator(CLIP_CFG % extra, device=dev, seed=11, world_size=world, rank=rank, embedding_parallel=ep)
  probe = make(b'', False)                                   # replicated tables: the source of weights and of the restatement
  plain, clip = make(b'', True), make(b'gradient_clipping_by_norm: %g' % clipv, True)
  for e in (plain, clip):
    assert e.input_layer.ep
    ep_helpers.copy_tables(probe.input_layer, e.input_layer, rank, world)
    e.model.load_state_dict(probe.model.state_dict())
    e.trainer.dense_opt.flat_p.copy_(probe.trainer.dense_opt.flat_p)
  # -- the norm, restated from one backward pass of the replicated model: per arena, per distinct ROW (all columns)
  tr, il = probe.trainer, probe.input_layer
  tr._set_hyper()
  probe.model.train()
  tr._segment_compute(feats, labels)
  local_sq = 0.0
  for m, rows, w, outs, seg_ids in il._pending:
    D = m.arena.dim
    r = rows.cpu().numpy()
    per_lookup = np.zeros((r.size, D), np.float64)
    for sl in m.slots_np:
      g = outs[int(sl['out_buf'])].grad.cpu().numpy().reshape(-1, int(sl['out_stride']))[:, int(sl['out_col']):int(sl['out_col']) + D]
      lo, n = int(sl['seg_begin']), int(sl['n_seg'])
      ww = np.ones(n, np.float32) if w is None else w.cpu().numpy()[lo:lo + n]
      per_lookup[lo:lo + n] = g * ww[:, None]
    for u in np.unique(r[r >= 0]):
      local_sq += float((per_lookup[r == u].sum(0) ** 2).sum())
  il.discard_pending()
  tot = torch.tensor([local_sq], dtype=torch.float64, device=dev)
  dist.all_reduce(tot)
  g_avg = tr.dense_opt.flat_g.double().clone()
  dist.all_reduce(g_avg)
  g_avg /= world
  l2 = torch.from_numpy(tr.dense_opt._l2_vec_np).double().to(dev)
  want = float(np.sqrt(float(tot[0]) / world ** 2 + float(((g_avg + l2 * tr.dense_opt.flat_p.double()) ** 2).sum())))
  # -- the step: SGD, so clipped = scale * unclipped on every shard and parameter
  p0 = plain.trainer.dense_opt.flat_p.clone()
  t0 = {d: a.weight.clone() for d, a in plain.input_layer.arenas.items()}
  plain.trainer.train_step(feats, labels)
  clip.trainer.train_step(feats, labels)
  norm = float(clip.trainer.last_grad_norm)
  assert norm == pytest.approx(want, rel=1e-5) and norm > clipv, (norm, want)
  scale = clipv / norm
  dp_plain = plain.trainer.dense_opt.flat_p - p0
  torch.testing.assert_close(clip.trainer.dense_opt.flat_p - p0, dp_plain * scale, rtol=1e-4, atol=2e-7)
  moved = 0.0
  for d, a in clip.input_layer.arenas.items():
    dt_plain = plain.input_layer.arenas[d].weight - t0[d]
    torch.testing.assert_close(a.weight - t0[d], dt_plain * scale, rtol=1e-4, atol=2e-8)
    moved = max(moved, float(dt_plain.abs().max()))
  assert moved > 1e-4
  clip.trainer.train_step(feats, labels)          # a second step: the held update was released, nothing accumulates
  clip.input_layer.check_exchange()
  ret[rank] = (norm, float(clip.trainer.dense_opt.flat_p.double().sum()))
  if cuda:
    dist.barrier()
    os._exit(0)     # (captured graphs may hold NCCL work: no destroy_process_group)
  dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_global_norm_clipping_with_row_sharded_tables_gloo():
  world = 2
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker_ep, args=(_free_port(), ret, world), nprocs=world, join=True)
  assert len(ret) == world and len(set(ret.values())) == 1, dict(ret)       # same norm, same dense parameters
