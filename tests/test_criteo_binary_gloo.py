"""CPU, kernel doubles, world 2 and 3 over gloo (and 2 GPUs over NCCL, tests/test_gpu_criteo_binary.py): CriteoInput
workers.  Each worker's batches are the reference reader's for that world size (tests/golden/reference_criteo_batches.json,
first batch_size samples of a batch that crosses a file boundary); training from the binary parts - replicated or
row-sharded tables - equals training on the same per-worker batches handed over as host tensors; the workers stop
together and evaluate() returns the same dict on every worker."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, 'golden'))

import test_criteo_binary_host as H  # noqa: E402
import test_input_shards_gloo as G  # noqa: E402


def _worker(rank, port, ret, world, tmp, mode, cuda=False, graph=False):
  from test_dp_clip_gloo import _setup
  import torch.distributed as dist
  dev = _setup(rank, port, world, cuda)
  import binary_doubles
  import make_criteo_golden as gen
  from easyrec_b200.config import config_util
  from easyrec_b200.estimator import EasyRecEstimator
  from easyrec_b200.input import readers
  if not cuda:
    binary_doubles.install()
  B = H.GOLD['batch_size']
  sizes = H.GOLD['cases']['4x25']['sizes']
  if rank == 0:
    gen.write_parts(tmp, sizes)
  dist.barrier()
  paths = H._Paths(*[[os.path.join(tmp, 'part%d_%s.bin' % (p, k)) for p in range(len(sizes))]
                     for k in ('label', 'dense', 'category')])
  cfg = H.small_cfg(H.PLAN, B)
  if mode == 'ep':
    config_util.edit_config(cfg, {'train_config.train_distribute': 'EmbeddingParallelStrategy'})
  cfg.eval_config.metrics_set.add().auc.SetInParent()
  cfg.eval_config.metrics_set.add().gauc.uid_field = 'c2'
  ests = [EasyRecEstimator(cfg, device=dev, seed=3, world_size=world, rank=rank, use_cuda_graph=graph) for _ in range(2)]
  assert ests[0].embedding_parallel == (mode == 'ep')

  # this worker's batches: the reference reader's for this world size
  mine = list(readers.make_input(cfg, ests[0].input_layer, paths, rank, world))
  want = H.GOLD['cases']['4x25']['worlds'][str(world)][rank]
  assert len(mine) == len(want) - 1      # (the reference's last partial batch is skipped)
  for (b, _), w in zip(mine, want):
    assert b.label.numpy().tolist() == w['label'][:B]
    assert b.cat.numpy().view(np.uint32).reshape(-1).tolist() == w['category'][:B * 26]
  host = []
  for b, _ in mine:
    sp, de, lab = binary_doubles.unpack(b.label.numpy(), b.dense.numpy(), b.cat.numpy(), b.slot_cols, b.raw_cols)
    host.append(({'sparse_fea': torch.from_numpy(sp), 'dense_fea': torch.from_numpy(de)}, torch.from_numpy(lab)))

  losses = [G._record_losses(e) for e in ests]
  ests[0].train(lambda: readers.make_input(cfg, ests[0].input_layer, paths, rank, world))
  ests[1].train(lambda: list(host))
  assert losses[0] == losses[1] and len(losses[0]) == len(mine)
  steps = G._gather(ests[0].global_step)
  assert steps == [len(mine)] * world
  for d, a in ests[0].input_layer.arenas.items():
    assert torch.equal(a.storage, ests[1].input_layer.arenas[d].storage), d
  for (n, p), (_, q) in zip(ests[0].model.state_dict().items(), ests[1].model.state_dict().items()):
    assert torch.equal(p, q), n
  ev = ests[0].evaluate(lambda: readers.make_input(cfg, ests[0].input_layer, paths, rank, world))
  ev_host = ests[1].evaluate(lambda: list(host))
  assert ev == ev_host and 'gauc' in ev
  dicts = G._gather(ev)
  assert all(d == dicts[0] for d in dicts), dicts
  ret[rank] = (len(mine), ev['auc'])
  if cuda:
    dist.barrier()
    os._exit(0)
  dist.destroy_process_group()


@pytest.mark.timeout(900)
@pytest.mark.parametrize('world,mode', [(2, 'dp'), (3, 'dp'), (2, 'ep'), (3, 'ep')])
def test_criteo_workers_read_the_reference_shards_and_train_like_host_batches(tmp_path, world, mode):
  ret = mp.Manager().dict()
  G._spawn(_worker, world, (G._free_port(), ret, world, str(tmp_path), mode))
  assert len(ret) == world and len(set(ret.values())) == 1, dict(ret)
