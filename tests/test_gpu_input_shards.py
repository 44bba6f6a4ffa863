"""2 GPUs over NCCL, real kernels: workers reading their shards of one CSV file / of the Parquet files train the model
one process trains on the union of their batches, and evaluate() returns the union's metrics on every worker - the
worker functions of tests/test_input_shards_gloo.py on cuda devices, eager and graph-replayed, replicated and
row-sharded.  Even shards only: every worker has the same number of batches.  Skipped with fewer than 2 GPUs."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
WORLD = 2
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.timeout(900)
@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('mode,fmt', [('dp', 'csv'), ('ep', 'csv'), ('dp', 'parquet'), ('ep', 'parquet')])
def test_workers_over_shards_train_and_evaluate_like_one_process_on_2_gpus(tmp_path, mode, fmt, graph):
  if torch.cuda.device_count() < WORLD:
    pytest.skip('needs %d GPUs' % WORLD)
  if fmt == 'parquet':
    pytest.importorskip('pyarrow')
  import torch.multiprocessing as mp
  import test_input_shards_gloo as T
  T._prepare(str(tmp_path), WORLD, fmt)
  ret = mp.Manager().dict()
  T._spawn(T._equivalence_worker, WORLD, (T._free_port(), ret, WORLD, str(tmp_path), mode, fmt, True, graph))
  assert len(ret) == WORLD and len(set(v[0] for v in ret.values())) == 1, dict(ret)
