"""CPU, world 2 and 3 over gloo, kernel doubles: vocabulary features (an IdFeature, a kv-weighted mean TagFeature and a
DIN key + history, tests/test_vocab_host.py) trained data-parallel over replicated tables and row-sharded under
EmbeddingParallelStrategy.  K1 runs on the requester and turns each key into its entry's row, so the row-sharded
exchange (owner = row mod N) and the data-parallel gather are unchanged: on the same per-rank batches the two must stay
the same model."""
import os
import socket
import sys

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
STEPS = 3


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, port, ret, world, tmp):
  sys.path.insert(0, HERE)
  from test_dp_clip_gloo import _setup
  dev = _setup(rank, port, world, False)
  import seq_doubles
  import vocab_doubles
  seq_doubles.install()   # (_setup installed the other kernel doubles)
  vocab_doubles.install()
  import ep_helpers
  import test_vocab_host as V
  from easyrec_b200 import _lib
  from easyrec_b200.estimator import EasyRecEstimator
  vf = V.write_vocab_file(os.path.join(tmp, 'items.txt'), V.I_VOCAB)

  def make(ep, **kw):
    text = V.config(vf, extra_train='train_distribute: EmbeddingParallelStrategy' if ep else '')
    return EasyRecEstimator(text, device=dev, seed=5, embedding_parallel=ep or None, **kw)
  dp = make(False, world_size=world, rank=rank)
  ep = make(True, world_size=world, rank=rank)
  assert ep.input_layer.ep and not dp.input_layer.ep
  assert all(f.bucket_mode == _lib.BUCKET_VOCAB for f in ep.input_layer.features.values())
  ep_helpers.copy_tables(dp.input_layer, ep.input_layer, rank, world)
  ep.model.load_state_dict(dp.model.state_dict())
  ep.trainer.dense_opt.flat_p.copy_(dp.trainer.dense_opt.flat_p)
  for step in range(STEPS):
    feats, labels = V.features(V.raw_batch(100 * rank + step), 'vocab')
    l_dp, _ = dp.trainer.train_step(feats, labels)
    l_ep, _ = ep.trainer.train_step(feats, labels)
    assert abs(float(l_dp) - float(l_ep)) < 1e-5, (step, float(l_dp), float(l_ep))
  worst = ep_helpers.compare(dp.input_layer, ep.input_layer, rank, world, 2e-6)
  d = float((dp.trainer.dense_opt.flat_p - ep.trainer.dense_opt.flat_p).abs().max())
  assert d < 1e-5, d
  ep.input_layer.check_exchange()
  ret[rank] = worst
  dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize('world', [2, 3])
def test_vocabulary_features_train_alike_data_parallel_and_row_sharded_gloo(world, tmp_path):
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret, world, str(tmp_path)), nprocs=world, join=True)
  assert len(ret) == world
