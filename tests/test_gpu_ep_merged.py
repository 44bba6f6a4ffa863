"""The row-sharded exchange shared by an arena's single-valued and multi-valued launches, with the real kernels.

  * tests/test_ep_merged_gloo.py's comparison over NCCL - adagrad, lazy Adam and tf.train.AdamOptimizer against
    replicated data parallel, eager and with the whole step replayed from one CUDA graph, with and without the next
    batch prefetched; on the eager steps without prefetch, the real K1 / K8 make exactly three all-to-alls per step and
    exchange, K8's counts are the distinct requested rows and the CSR padding is never requested.  Skipped on boxes
    with fewer than 2 GPUs.
  * Two ranks on ONE GPU over gloo, eager: K1 of each launch into its range of the lookup arrays (er_bucketize_weighted:
    the kv-weighted tag feature's weights include 0 and negative ones, which its `mean` slot prunes and its `sum` twin
    in the wide group keeps), one K8 over all of them, the pooling K2 and the requester-side K7 of each launch over its
    own range - against one process training the same model on the concatenated batch (no batch norm, no embedding
    regulariser: then the two are the same model), table shards and optimizer slots within 5e-6."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def _graph_worker(rank, port, ret, world, tmp, cuda=True):
  import test_ep_merged_gloo as G
  from test_dp_clip_gloo import _setup
  import torch.distributed as dist
  dev = _setup(rank, port, world, cuda)
  count = [0]
  G._counting_all_to_all(count)
  worst = 0.0
  for comb in G.EXCHANGES:
    for opt in G.OPTS:
      for lookahead in (False, True):
        for graph in (False, True):
          worst = max(worst, _run_graph(G, dev, rank, world, tmp, opt, comb, lookahead, graph, count))
  ret[rank] = worst
  dist.barrier()
  os._exit(0)


def _run_graph(G, dev, rank, world, tmp, opt, comb, lookahead, graph, count):
  from easyrec_b200.estimator import EasyRecEstimator
  import ep_helpers

  def make(ep):
    return EasyRecEstimator(G.config(ep, opt, comb=comb), device=dev, seed=5, world_size=world, rank=rank,
                            embedding_parallel=None if ep else False, use_cuda_graph=graph and ep)
  dp, ep = make(False), make(True)
  ep_helpers.copy_tables(dp.input_layer, ep.input_layer, rank, world)
  ep.model.load_state_dict(dp.model.state_dict())
  ep.trainer.dense_opt.flat_p.copy_(dp.trainer.dense_opt.flat_p)
  steps = 7 if graph else G.STEPS
  data = G.batches(rank, tmp, dev, n=steps)
  for step in range(steps):
    f, l = data[step]
    l_dp, p_dp = dp.trainer.train_step(f, l)
    nxt = data[step + 1][0] if lookahead and step + 1 < steps else None
    count[0] = 0
    l_ep, p_ep = ep.trainer.train_step(f, l, next_features=nxt)
    if not graph and not lookahead:
      assert count[0] == 3 * G.EXCHANGES[comb], count[0]     # ids, rows, gradients
      G.check_structure(ep.input_layer, world, G.EXCHANGES[comb])
    assert abs(float(l_dp) - float(l_ep)) < 1e-5, (opt, step, float(l_dp), float(l_ep))
    assert float((p_dp - p_ep).abs().max()) < 1e-5
  worst = G.compare_storage(dp.input_layer, ep.input_layer, rank, world)
  assert worst <= 5e-6, (opt, comb, lookahead, graph, worst)
  ep.input_layer.check_exchange()
  if graph:
    assert ep.trainer._graph is not None
  return worst


@pytest.mark.timeout(900)
def test_merged_exchange_equals_replicated_data_parallel_on_2_gpus(tmp_path):
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  import torch.multiprocessing as mp
  from test_ep_merged_gloo import _free_port
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_graph_worker, args=(_free_port(), ret, 2, str(tmp_path)), nprocs=2, join=True)
  assert len(ret) == 2


def _one_gpu_config(G, ep, opt, comb, batch):
  text = G.config(ep, opt, comb=comb)
  for a, b in ((b'  embedding_regularization: 1e-5 }', b'  }'), (b'batch_size: 12', b'batch_size: %d' % batch)):
    assert a in text
    text = text.replace(a, b)
  return text


def _one_gpu_worker(rank, port, ret, world, tmp):
  import test_ep_merged_gloo as G
  import torch.distributed as dist
  import ep_helpers
  from easyrec_b200.config import config_util
  from easyrec_b200.estimator import EasyRecEstimator
  from easyrec_b200.input import readers
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  torch.backends.cuda.matmul.allow_tf32 = False
  dev = 'cuda:0'
  worst = 0.0
  for comb in G.EXCHANGES:
    for opt in G.OPTS:
      ep = EasyRecEstimator(_one_gpu_config(G, True, opt, comb, G.B), device=dev, seed=5, world_size=world, rank=rank)
      assert len(ep.input_layer._exchanges()) == G.EXCHANGES[comb]
      whole = _one_gpu_config(G, False, opt, comb, G.B * world)
      one = EasyRecEstimator(whole, device=dev, seed=5)
      ep_helpers.copy_tables(one.input_layer, ep.input_layer, rank, world)
      ep.model.load_state_dict(one.model.state_dict())
      ep.trainer.dense_opt.flat_p.copy_(one.trainer.dense_opt.flat_p)
      mine = G.batches(rank, tmp, dev, odd_weights=True)
      # the concatenated batch of every rank, read by one process
      cfg = config_util.get_configs_from_pipeline_file(whole)
      il = EasyRecEstimator(whole, device='cpu', seed=1).input_layer
      for step in range(G.STEPS):
        path = os.path.join(tmp, 'one_r%d_s%d.csv' % (rank, step))
        with open(path, 'w') as f:
          f.write('\n'.join(sum((G._lines(1000 * r + step, odd_weights=True) for r in range(world)), [])) + '\n')
        (feats, labels), = list(readers.CSVInput(cfg, il, path))
        if step == 0:
          w = feats['tag_fea']['t1'][2]
          assert (w == 0).any() and (w < 0).any()
        one.trainer.train_step(*readers.to_device(feats, labels, dev))
        ep.trainer.train_step(*mine[step])
      w = G.compare_storage(one.input_layer, ep.input_layer, rank, world)
      assert w <= 5e-6, (opt, comb, w)
      d = float((one.trainer.dense_opt.flat_p - ep.trainer.dense_opt.flat_p).abs().max())
      assert d < 1e-5, (opt, comb, d)
      ep.input_layer.check_exchange()
      worst = max(worst, w)
  ret[rank] = worst
  dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_merged_exchange_with_the_real_kernels_two_ranks_on_one_gpu(tmp_path):
  import torch.multiprocessing as mp
  from test_ep_merged_gloo import _free_port
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_one_gpu_worker, args=(_free_port(), ret, 2, str(tmp_path)), nprocs=2, join=True)
  assert len(ret) == 2
