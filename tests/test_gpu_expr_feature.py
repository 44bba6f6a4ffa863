"""GPU: er_expr_eval and ExprFeature training on the device.

  * the kernel replays the reference's grammar (tests/golden/reference_expr.json) bit for bit: every expression the
    compiler accepts, packed into one call, at B = 1, 4096 and 65536 (float64 IEEE ops and one rounding to float32 are
    exact; a NaN matches any NaN);
  * a bad call is refused by ER_REQUIRE before anything is launched;
  * a model with ExprFeatures in deep and wide groups trains exactly like its twin that reads the fixture's values as
    RawFeatures, eagerly and graph-replayed (test_expr_feature_host.py's configs and batches), and the two runs give
    the same losses bit for bit;
  * two row-sharded ranks on one GPU (gloo) train the expr model like its twin."""
import datetime
import os
import socket
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

pytestmark = pytest.mark.gpu


def _accepted():
  import test_expr_feature_host as H
  from easyrec_b200 import expr as X
  rows, cases = H.fixture()
  progs, outs = [], []
  for c in cases:
    if 'out' in c and c['expression'] not in H.REFUSED:
      progs.append(X.compile_expression('f', c['expression'], c['input_names']))
      outs.append(c['out'])
  return rows, progs, outs


@pytest.mark.parametrize('B', [1, 4096, 65536])
def test_er_expr_eval_replays_the_reference_grammar_bit_for_bit(B):
  import test_expr_feature_host as H
  from easyrec_b200 import _lib, kernels as K
  rows, progs, outs = _accepted()
  assert len(progs) >= 45 and max(p.depth for p in progs) == _lib.EXPR_MAX_STACK
  pick = np.arange(B) % rows.shape[0]
  plan = K.expr_plan(progs, list(range(len(progs))), 3, 'cuda:0')
  inputs = torch.from_numpy(np.ascontiguousarray(rows[pick])).cuda()
  dense = torch.full((B, len(progs) + 1), -3.0, dtype=torch.float32, device='cuda:0')
  n0 = _lib.load().er_launch_count()
  K.expr_eval(plan, inputs, dense)
  assert _lib.load().er_launch_count() - n0 == 1
  got = dense.cpu().numpy()
  for e, want in enumerate(outs):
    assert H.same_bits(got[:, e], [want[i] for i in pick]), e
  assert (got[:, -1] == -3.0).all()   # a column no expression names is left alone


def test_a_bad_call_is_refused_before_a_launch():
  from easyrec_b200 import _lib, expr as X, kernels as K
  lib = _lib.load()
  p = X.compile_expression('f', 'x>y', ['x', 'y'])
  plan = K.expr_plan([p], [0], 2, 'cuda:0')
  inputs = torch.zeros((4, 2), dtype=torch.float64, device='cuda:0')
  dense = torch.zeros((4, 1), dtype=torch.float32, device='cuda:0')
  base, s = plan.dev.data_ptr(), torch.cuda.current_stream().cuda_stream
  n0 = lib.er_launch_count()
  for args, msg in (((inputs.data_ptr(), 4, 2, base, 1, base + 16, 3, 9, dense.data_ptr(), 1, s), b'max_depth'),
                    ((inputs.data_ptr(), 4, 2, base, 1, base + 16, 4097, 2, dense.data_ptr(), 1, s), b'n_ops'),
                    ((inputs.data_ptr(), 4, 2, None, 1, base + 16, 3, 2, dense.data_ptr(), 1, s), b'null'),
                    ((None, 4, 2, base, 1, base + 16, 3, 2, dense.data_ptr(), 1, s), b'null inputs'),
                    ((inputs.data_ptr(), 4, 2, base, 1, base + 16, 3, 2, dense.data_ptr(), 0, s), b'dense_pitch'),
                    ((inputs.data_ptr(), 4, 2, base, 2, base + 16, 1, 2, dense.data_ptr(), 1, s), b'at least one op')):
    assert lib.er_expr_eval(*args) == _lib.ER_ERR_INVALID_ARG
    assert msg in lib.er_last_error(), (msg, lib.er_last_error())
  assert lib.er_launch_count() == n0
  # the host refuses programs the kernel would misread before they reach the device
  for bad, msg in (([(0, 2, 0.0)], 'input 2 of 2'), ([(0, 0, 0.0), (2, 0, 0.0)], 'stack leaves'),
                   ([(0, 0, 0.0), (0, 1, 0.0)], 'leaves 2 values'), ([(99, 0, 0.0)], 'op 99')):
    with pytest.raises(_lib.ErError, match=msg):
      K.expr_plan([X.Program(tuple(bad), 'float', 2)], [0], 2, 'cuda:0')
  torch.cuda.synchronize()


def test_expr_features_train_like_their_raw_twin_eager_and_graph_replayed():
  import test_expr_feature_host as H
  torch.backends.cuda.matmul.allow_tf32 = False
  ex, raw, eager = H.run_twins('cuda:0', steps=5)
  ex_g, raw_g, graph = H.run_twins('cuda:0', steps=5, use_cuda_graph=True)
  assert eager == graph
  H.assert_same_model(ex, ex_g)
  # the expression step is one launch more than its twin's
  assert ex_g.trainer.launches_per_step == raw_g.trainer.launches_per_step + 1


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, port, ret):
  import torch.distributed as dist
  sys.path.insert(0, HERE)
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=2, timeout=datetime.timedelta(seconds=300))
  torch.cuda.set_device(0)
  torch.backends.cuda.matmul.allow_tf32 = False
  import test_expr_feature_host as H
  ex, raw, losses = H.run_twins('cuda:0', seed=100 + rank, world_size=2, rank=rank, embedding_parallel=True)
  assert ex.input_layer.ep
  ret[rank] = losses
  dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_row_sharded_ranks_on_one_gpu_train_like_the_raw_twin():
  import torch.multiprocessing as mp
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret), nprocs=2, join=True)
  assert len(ret) == 2
