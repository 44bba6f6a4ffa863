"""er_bucketize_seq (K1 over un-pooled histories) on the device, and the row-sharded history exchange on 2 GPUs.

  * er_bucketize_seq equals er_bucketize followed by the padding mask, bit for bit: every er_bucket_mode, T in
    {1, 31, 32, 33, 50, 200}, shard_n in {1, 2, 3, 8}, uniform and non-uniform slot plans, lengths 0, 1, T and lengths
    outside [0, T] (clamped).  Outputs sit in sentinel-filled buffers with guards on both sides; the ids of padded steps
    are never read (they are poisoned with values that would bucket to live rows).
  * tests/test_ep_seq_gloo.py's models over NCCL with the real kernels, eager and with the whole step replayed from one
    CUDA graph, against replicated data parallel.  Skipped on boxes with fewer than 2 GPUs."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib
from easyrec_b200 import kernels as K

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MODES = (_lib.BUCKET_FARM_DECIMAL, _lib.BUCKET_MOD, _lib.BUCKET_IDENTITY, _lib.BUCKET_NONE, _lib.BUCKET_ONE_ROW)
GUARD = 64
SENT_ROW, SENT_OWN = -7777, -7777


def _guarded(n, dtype, sentinel, dev):
  buf = torch.full((n + 2 * GUARD,), sentinel, dtype=dtype, device=dev)
  return buf, buf[GUARD:GUARD + n]


def _plan(n_features, B, T, mode, shard_n, uniform, rng):
  """one slot per history feature (uniform), or the features' steps split into slots of unequal size"""
  recs, seg = [], 0
  n_steps = B * T
  for f in range(n_features):
    cuts = [0, n_steps] if uniform else sorted({0, n_steps, int(rng.integers(1, max(n_steps, 2)))})
    for a, b in zip(cuts[:-1], cuts[1:]):
      recs.append(dict(num_buckets=int(rng.integers(5, 1000)), row_offset=int(rng.integers(0, 5000)), seg_begin=seg,
                       n_seg=b - a, bucket_mode=mode, combiner=_lib.COMBINER_SUM | _lib.COMBINER_UNIT_WEIGHTS,
                       out_buf=0, out_stride=4, out_col=0, shard_n=shard_n))
      seg += b - a
  return K.make_slots(recs)


def _ids(mode, n, rng):
  if mode == _lib.BUCKET_FARM_DECIMAL:
    return rng.integers(-2**62, 2**62, n)
  if mode == _lib.BUCKET_MOD:
    return rng.integers(-10**6, 10**6, n)
  return rng.integers(-3, 1200, n)   # identity / none / one-row: -1 drops, < -1 and >= nb map per the mode


@pytest.mark.parametrize('T', [1, 31, 32, 33, 50, 200])
def test_bucketize_seq_equals_k1_then_mask(T):
  dev = 'cuda:0'
  rng = np.random.default_rng(T)
  for mode in MODES:
    for shard_n in (1, 2, 3, 8):
      for uniform in (True, False):
        n_features, B = int(rng.integers(1, 4)), int(rng.integers(1, 70))
        n = n_features * B * T
        slots_np = _plan(n_features, B, T, mode, shard_n, uniform, rng)
        slots = K.slots_to_device(slots_np, dev)
        lens = rng.integers(0, T + 1, n_features * B)
        lens[:min(3, lens.size)] = [0, 1, T][:min(3, lens.size)]
        odd = rng.uniform(size=lens.size) < 0.1
        lens = np.where(odd, rng.choice([-5, -1, T + 1, T + 40, 2**31 - 1], lens.size), lens).astype(np.int32)
        ids = _ids(mode, n, rng).astype(np.int64)
        pad = (np.arange(n) % T) >= np.repeat(lens.astype(np.int64), T)
        # K1 then the mask: the reference
        t_ids = torch.from_numpy(ids).to(dev)
        want_rows = torch.empty(n, dtype=torch.int64, device=dev)
        want_own = torch.empty(n, dtype=torch.int32, device=dev)
        K.bucketize(t_ids, slots, len(slots_np), n, rows=want_rows, owner=want_own)
        want_rows, want_own = want_rows.cpu().numpy(), want_own.cpu().numpy()
        want_rows[pad], want_own[pad] = -1, -1
        # the padded steps' ids are poisoned: a kernel that read them would give a different row for a live step
        poisoned = torch.from_numpy(np.where(pad, 7, ids)).to(dev)
        rb, rows = _guarded(n, torch.int64, SENT_ROW, dev)
        ob, own = _guarded(n, torch.int32, SENT_OWN, dev)
        K.bucketize_seq(poisoned, torch.from_numpy(lens).to(dev), B, T, slots, len(slots_np), rows=rows, owner=own)
        rb2, rows2 = _guarded(n, torch.int64, SENT_ROW, dev)
        K.bucketize_seq(poisoned, torch.from_numpy(lens).to(dev), B, T, slots, len(slots_np), rows=rows2)  # owner NULL
        torch.cuda.synchronize()
        for buf, sent in ((rb, SENT_ROW), (ob, SENT_OWN), (rb2, SENT_ROW)):
          g = buf.cpu().numpy()
          assert (g[:GUARD] == sent).all() and (g[-GUARD:] == sent).all(), 'write outside the output'
        ctx = (mode, shard_n, uniform, n_features, B)
        assert np.array_equal(rows.cpu().numpy(), want_rows), ctx
        assert np.array_equal(own.cpu().numpy(), want_own), ctx
        assert np.array_equal(rows2.cpu().numpy(), want_rows), ctx


def test_bucketize_seq_refuses_bad_shapes():
  dev = 'cuda:0'
  slots = K.slots_to_device(_plan(1, 4, 3, _lib.BUCKET_NONE, 1, True, np.random.default_rng(0)), dev)
  ids = torch.zeros(12, dtype=torch.int64, device=dev)
  lens = torch.zeros(4, dtype=torch.int32, device=dev)
  lib = _lib.load()
  rows = torch.empty(12, dtype=torch.int64, device=dev)
  for b, t, f in ((0, 3, 1), (4, 0, 1), (4, 3, 0), (2**20, 2**11, 1)):
    rc = lib.er_bucketize_seq(ids.data_ptr(), lens.data_ptr(), b, t, f, slots.data_ptr(), 1, rows.data_ptr(), None,
                              torch.cuda.current_stream().cuda_stream)
    assert rc == _lib.ER_ERR_INVALID_ARG, (b, t, f)
  rc = lib.er_bucketize_seq(ids.data_ptr(), None, 4, 3, 1, slots.data_ptr(), 1, rows.data_ptr(), None,
                            torch.cuda.current_stream().cuda_stream)
  assert rc == _lib.ER_ERR_INVALID_ARG


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


@pytest.mark.timeout(600)
def test_history_exchange_equals_replicated_data_parallel_on_2_gpus():
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  import torch.multiprocessing as mp
  sys.path.insert(0, HERE)
  import test_ep_seq_gloo as G
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(G._worker, args=(_free_port(), ret, 2, None, True), nprocs=2, join=True)
  assert len(ret) == 2
