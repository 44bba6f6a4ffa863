"""GPU, real kernels: CriteoInput.

* er_binary_unpack is bit-exact against its numpy restatement (tests/binary_doubles.py): batch sizes below, at and not a
  multiple of the kernel's 128-row tile; permuted, duplicated and partial column maps, empty ones; category values at
  and past 2^31.  The outputs are prefilled with NaN / a sentinel, so an element left unwritten fails.
* The C2 workload trained from binary parts equals the same samples read from TSV, eager and graph-replayed: the
  unpacked batches, the tables and the dense parameters bit for bit, the reported losses to their last bit.
* Two workers over NCCL (even shards): tests/test_criteo_binary_gloo.py's worker on cuda devices."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import binary_doubles  # noqa: E402
from easyrec_b200 import kernels as K, workloads  # noqa: E402
from easyrec_b200.config import config_util  # noqa: E402
from easyrec_b200.estimator import EasyRecEstimator  # noqa: E402
from easyrec_b200.input import readers  # noqa: E402

SENTINEL = -7777777777


@pytest.mark.parametrize('B', [1, 77, 128, 129, 1000, 4096 + 5])
@pytest.mark.parametrize('slot_cols,raw_cols', [
    (list(range(26)), list(range(13))),
    (list(range(25, -1, -1)), [12, 0, 5, 1, 2, 3, 4, 6, 7, 8, 9, 10, 11]),
    ([3, 3, 0, 25, 3, 7], [4, 4, 0]),
    ([25], []),
    ([], [6]),
])
def test_unpack_is_bit_exact_against_numpy(B, slot_cols, raw_cols):
  rng = np.random.default_rng(B + len(slot_cols))
  label = rng.integers(-3, 3, B).astype(np.int32)
  dense = rng.standard_normal((B, 13)).astype(np.float32)
  cat = rng.integers(0, 2**32, (B, 26), dtype=np.uint64).astype(np.uint32)
  cat[0, :] = 2**31
  cat[-1, :] = 2**32 - 1
  dev = 'cuda:0'
  maps = K.binary_maps(slot_cols, raw_cols, dev)
  outs = (torch.full((len(slot_cols) * B,), SENTINEL, dtype=torch.int64, device=dev),
          torch.full((B, len(raw_cols)), float('nan'), device=dev), torch.full((B,), float('nan'), device=dev))
  got = K.binary_unpack(torch.from_numpy(label).to(dev), torch.from_numpy(dense).to(dev),
                        torch.from_numpy(cat.view(np.int32)).to(dev), *maps, *outs)
  torch.cuda.synchronize()
  want = binary_doubles.unpack(label, dense, cat, slot_cols, raw_cols)
  for g, w in zip(got, want):
    assert np.array_equal(g.cpu().numpy(), w)
  if slot_cols and B > 1:   # (row 0 holds 2^31 in every column: read as int32)
    assert got[0].min().item() == -2**31


def test_column_maps_out_of_range_are_refused():
  with pytest.raises(Exception, match=r'slot_cols entries must be in \[0, 26\)'):
    K.binary_maps([26], [0], 'cuda:0')
  with pytest.raises(Exception, match=r'raw_cols entries must be in \[0, 13\)'):
    K.binary_maps([0], [-1], 'cuda:0')


def _c2_pair(tmp, B, n_batches, vocab=100003):
  """(binary config, TSV config) of C2 over the same samples"""
  lp, dp, cp = workloads.write_c2_binary(os.path.join(tmp, 'c2'), n_batches, B, n_files=3)
  import glob
  label = np.concatenate([np.fromfile(p, np.int32) for p in sorted(glob.glob(lp))])
  dense = np.concatenate([np.fromfile(p, np.float32) for p in sorted(glob.glob(dp))]).reshape(-1, 13)
  cat = np.concatenate([np.fromfile(p, np.uint32) for p in sorted(glob.glob(cp))]).reshape(-1, 26)
  tsv = os.path.join(tmp, 'c2.tsv')
  with open(tsv, 'w') as f:
    for i in range(label.size):
      f.write('\t'.join([str(label[i])] + [str(x) for x in dense[i]] + [str(int(x)) for x in cat[i]]) + '\n')
  cb = config_util.get_configs_from_pipeline_file(workloads.c2_config_text(vocab, B, input_type='CriteoInput'))
  cb.binary_train_input.label_path.append(lp)
  cb.binary_train_input.dense_path.append(dp)
  cb.binary_train_input.category_path.append(cp)
  cc = config_util.get_configs_from_pipeline_file(workloads.c2_config_text(vocab, B))
  return cb, cc, tsv


@pytest.mark.parametrize('graph', [False, True])
def test_c2_from_binary_parts_trains_like_from_tsv(tmp_path, graph):
  torch.backends.cuda.matmul.allow_tf32 = False
  B = 2048
  cb, cc, tsv = _c2_pair(str(tmp_path), B, 6)
  # the batches themselves first: unpacked on the device as the text reader packs them
  il = EasyRecEstimator(cb, device='cuda:0', seed=5).input_layer
  for (fb, lb), (fc, lc) in zip(readers.make_input(cb, il, cb.binary_train_input), readers.make_input(cc, il, tsv)):
    fb, lb = readers.to_device(fb, lb, 'cuda:0')
    assert torch.equal(lb.cpu(), lc)
    for k in ('sparse_fea', 'dense_fea'):
      assert torch.equal(fb[k].cpu(), fc[k]), (k, (fb[k].cpu() != fc[k]).nonzero()[:4], fb[k].cpu()[fb[k].cpu() != fc[k]][:4],
                                               fc[k][fb[k].cpu() != fc[k]][:4])
  out = []
  for cfg, path in ((cb, cb.binary_train_input), (cc, tsv)):
    est = EasyRecEstimator(cfg, device='cuda:0', seed=5, use_cuda_graph=graph)
    losses = []
    step = est.trainer.train_step

    def rec(*a, **k):
      r = step(*a, **k)
      losses.append(r[0].detach().clone())
      return r
    est.trainer.train_step = rec
    est.train(lambda: readers.make_input(cfg, est.input_layer, path))
    torch.cuda.synchronize()
    out.append((est, [float(x) for x in losses]))
  (ea, la), (eb, lb) = out
  # the reported loss adds the l2 term, which er_dense_apply sums with float atomics (reporting only): it may differ in
  # its last bit between two runs of the same batches; the trained state is checked bit for bit below
  assert len(la) == len(lb) == 6 and np.allclose(la, lb, rtol=1e-6, atol=0), (la, lb)
  for d, a in ea.input_layer.arenas.items():
    assert torch.equal(a.storage, eb.input_layer.arenas[d].storage), d
  for (n, p), (_, q) in zip(ea.model.state_dict().items(), eb.model.state_dict().items()):
    assert torch.equal(p, q), n
  assert ea.last_feeder.h2d_bytes == 6 * B * (4 + 52 + 104)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('mode', ['dp', 'ep'])
def test_two_workers_over_nccl_train_like_host_batches(tmp_path, mode, graph):
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  import torch.multiprocessing as mp
  import test_criteo_binary_gloo as T
  import test_input_shards_gloo as G
  ret = mp.Manager().dict()
  G._spawn(T._worker, 2, (G._free_port(), ret, 2, str(tmp_path), mode, True, graph))
  assert len(ret) == 2 and len(set(ret.values())) == 1, dict(ret)
