"""2 GPUs: data-parallel DeepFM steps over NCCL (replicated tables, all-gather of K7 inputs).

Checks: (1) replicas stay BIT-identical (tables, optimizer state, dense parameters) - K7 and the dense path
are deterministic and every rank applies the same gathered update; (2) the early exchange (K1 + all-gather
of rows + global dedup sort on a side stream before the step) gives exactly the same model as the plain
exchange after the backward pass; (3) CUDA-graph replay - the collectives captured inside ONE graph per step (NCCL
on the capture stream) - trains exactly the same model as the eager run (2 eager steps, capture, replays: every batch
applied once).  Skipped on boxes with fewer than 2 GPUs."""
import os
import socket

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


def _train(rank, dev, prephase, graph, steps=4):
  import torch.distributed as dist
  from easyrec_b200 import workloads
  from easyrec_b200.trainer import Trainer
  B, V = 512, 50021
  il, model = workloads.build_deepfm_criteo(B, V, dev, dnn=(64, 32), final=(32, 16), seed=11)
  tr = Trainer(model, il, 'adagrad', lr=0.05, use_cuda_graph=graph, world_size=WORLD)
  tr.dp.prephase = prephase   # False: the rows are all-gathered with the gradients after the backward
  for step in range(steps):
    ids, dense, labels = workloads.criteo_batch(B, 100 + 10 * step + rank)
    feats = {'sparse_fea': torch.from_numpy(ids).to(dev), 'dense_fea': torch.from_numpy(dense).to(dev)}
    loss, _ = tr.train_step(feats, torch.from_numpy(labels).to(dev))
  torch.cuda.synchronize()
  state = [il.arenas[16].storage.clone(), il.arenas[1].storage.clone(), tr.dense_opt.flat_p.clone()]
  return float(loss), state


def _worker(rank, port, ret):
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(rank)
  dev = 'cuda:%d' % rank
  dist.init_process_group('nccl', rank=rank, world_size=WORLD, device_id=torch.device(dev))
  torch.backends.cuda.matmul.allow_tf32 = False
  results = {}
  for name, (pre, graph) in {'plain': (False, False), 'early': (True, False), 'graph_one': (True, True)}.items():
    loss, state = _train(rank, dev, pre, graph, steps=6)
    assert loss == loss and abs(loss) < 10
    for t in state:   # replicas identical: max over ranks of |mine - rank0's| must be exactly 0
      ref = t.clone()
      dist.broadcast(ref, src=0)
      assert torch.equal(t, ref), '%s: replicas diverged' % name
    results[name] = state
  for other in ('early', 'graph_one'):
    for a, b in zip(results['plain'], results[other]):
      assert torch.equal(a, b), '%s: a different model than the plain eager exchange' % other
  ret[rank] = True
  dist.destroy_process_group()


@pytest.mark.timeout(400)
def test_dp_replicas_identical_and_early_exchange_equivalent_on_2_gpus():
  if torch.cuda.device_count() < WORLD:
    pytest.skip('needs %d GPUs' % WORLD)
  import torch.multiprocessing as mp
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret), nprocs=WORLD, join=True)
  assert len(ret) == WORLD
