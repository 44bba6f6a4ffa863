"""CPU, world 2 over gloo, kernel doubles: ExprFeatures in deep and wide groups (tests/test_expr_feature_host.py) trained
data-parallel over replicated tables and row-sharded under EmbeddingParallelStrategy.  An expression's column is local to
its sample's rank, so nothing about it is exchanged: on the same per-rank batches the model must train exactly like its
twin that reads the expressions' values as RawFeatures."""
import os
import socket
import sys

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, port, ret, world, ep):
  sys.path.insert(0, HERE)
  from test_dp_clip_gloo import _setup
  dev = _setup(rank, port, world, False)
  import expr_doubles
  expr_doubles.install()   # (_setup installed the other kernel doubles)
  import test_expr_feature_host as H
  ex, raw, losses = H.run_twins(dev, seed=100 + rank, world_size=world, rank=rank, embedding_parallel=ep)
  assert ex.input_layer.ep == ep
  ret[rank] = losses
  dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize('ep', [False, True], ids=['data_parallel', 'row_sharded'])
def test_expr_features_train_like_their_raw_twin_gloo(ep):
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret, 2, ep), nprocs=2, join=True)
  assert len(ret) == 2
