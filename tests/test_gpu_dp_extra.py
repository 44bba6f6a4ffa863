"""2 GPUs over NCCL, real kernels: the multi-GPU additions whose host logic the gloo tests cover on the CPU -
global-norm clipping under data parallel and with row-sharded tables (tests/test_dp_clip_gloo.py) and data parallel over
multi-valued tag slots (tests/test_dp_tags_gloo.py), row-sharded tables with tag / multi-valued sequence slots
(tests/test_ep_tags_gloo.py), row-sharded key-value tables (tests/test_kv_ep_gloo.py) - run by the same worker functions
on cuda devices.  Skipped on boxes with fewer than 2 GPUs."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
WORLD = 2
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _spawn(fn, *extra, n_ret=WORLD):
  if torch.cuda.device_count() < WORLD:
    pytest.skip('needs %d GPUs' % WORLD)
  import torch.multiprocessing as mp
  from test_dp_clip_gloo import _free_port
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(fn, args=(_free_port(), ret, WORLD) + extra + (True,), nprocs=WORLD, join=True)
  assert len(ret) == n_ret
  return dict(ret)


@pytest.mark.timeout(400)
def test_global_norm_clipping_under_data_parallel_on_2_gpus():
  from test_dp_clip_gloo import _worker
  ret = _spawn(_worker)
  assert len(set(ret.values())) == 1, ret


@pytest.mark.timeout(400)
def test_global_norm_clipping_with_row_sharded_tables_on_2_gpus():
  from test_dp_clip_gloo import _worker_ep
  ret = _spawn(_worker_ep)
  assert len(set(ret.values())) == 1, ret


@pytest.mark.timeout(400)
def test_data_parallel_over_tag_slots_on_2_gpus(tmp_path):
  from test_dp_tags_gloo import _worker
  ret = _spawn(_worker, str(tmp_path))
  for worst, dworst, _, _ in ret.values():
    assert worst < 5e-6 and dworst < 5e-6, ret
  assert len(set(v[2:] for v in ret.values())) == 1, ret


@pytest.mark.timeout(400)
def test_embedding_parallel_over_tag_slots_on_2_gpus(tmp_path):
  from test_ep_tags_gloo import _worker
  _spawn(_worker, str(tmp_path))


@pytest.mark.timeout(400)
def test_key_value_tables_row_sharded_on_2_gpus(tmp_path):
  """key-value tables (ev_params) under EmbeddingParallelStrategy through ShardedExchange on the real kernels: the
  ranks train as one rank on the concatenated batch, per key"""
  from test_kv_ep_gloo import _worker
  ret = _spawn(_worker, str(tmp_path), n_ret=WORLD + 1)     # (+ rank 0's one-rank rows)
  assert all(ret[r] <= 2e-6 for r in range(WORLD)), ret
