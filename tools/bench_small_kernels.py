"""Device timing of the kernels added at the end of round 2 (no GPU lease was left to measure them): er_act_fwd / er_act_bwd
(HBM stream, 8 / 12 bytes per element), er_auc_hist (8 bytes per element) and er_gemm_small (the three forms of an
MMoE gate layer) - CUDA events on the launching stream, a 256 MB write between launches to flush L2, achieved GB/s
against MEASURED_PEAKS.json.  Run on the GPU box:   python tools/bench_small_kernels.py > gpurun_out/small_kernels.txt"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from easyrec_b200 import kernels as K, metrics as M  # noqa: E402

DEV = 'cuda:0'


def timed(fn, iters=20):
  flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=DEV)
  for _ in range(3):
    fn()
  ms = []
  for _ in range(iters):
    flush.fill_(1.0)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    ms.append(a.elapsed_time(b))
  return float(np.median(ms))


def main():
  peak = 3350.0   # H100 SXM data-sheet HBM3 bandwidth (GB/s), used when no measured peak is present
  p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'MEASURED_PEAKS.json')
  if os.path.exists(p):
    peak = float(json.load(open(p)).get('hbm_gbs', peak))
  rows = []
  n = 8192 * 50 * 128          # the DIN attention MLP's first hidden layer at C3 (B 4096 x T 50 ... x 128): 52 M elements
  x = torch.randn(n, device=DEV)
  gy = torch.randn(n, device=DEV)
  for name, kind in sorted(K.ACT_KINDS.items()):
    if name == 'prelu':
      continue
    f = timed(lambda: K.act_fwd(x, kind))
    b = timed(lambda: K.act_bwd(x, gy, kind))
    rows.append(('er_act_fwd[%s]' % name, n, 8 * n, f))
    rows.append(('er_act_bwd[%s]' % name, n, 12 * n, b))
  for n_eval, T in ((8192, 200), (1 << 22, 200), (1 << 22, 4095)):
    acc = M.ConfusionAtThresholds(T, DEV)
    pr, lab = torch.rand(n_eval, device=DEV), (torch.rand(n_eval, device=DEV) < 0.3).float()
    t = timed(lambda: acc.update(pr, lab))
    rows.append(('er_auc_hist[T=%d]' % T, n_eval, 8 * n_eval, t))
  B, d, E = 16384, 1280, 4     # a C5-shaped MMoE gate: [B, d] x [d, 4 experts]
  xg, w, g = torch.randn(B, d, device=DEV), torch.randn(d, E, device=DEV), torch.randn(B, E, device=DEV)
  rows.append(('er_gemm_small fwd [%d,%d]x[%d,%d]' % (B, d, d, E), B * E, 4 * (B * d + d * E + B * E), timed(lambda: K.gemm(xg, w))))
  rows.append(('er_gemm_small dX  [%d,%d]x[%d,%d]' % (B, E, E, d), B * d, 4 * (B * E + d * E + B * d), timed(lambda: K.gemm(g, w.t()))))
  rows.append(('er_gemm_small dW  [%d,%d]x[%d,%d]' % (d, B, B, E), d * E, 4 * (B * d + B * E + d * E), timed(lambda: K.gemm(xg.t(), g))))
  print('kernel | elements | algorithmic bytes | median ms | GB/s | fraction of the HBM peak (%.1f GB/s: MEASURED_PEAKS.json, else the H100 SXM data sheet)' % peak)
  for name, n_el, nbytes, ms in rows:
    gbs = nbytes / (ms * 1e-3) / 1e9
    print('%-44s %10d %12d %8.4f %8.1f %6.3f' % (name, n_el, nbytes, ms, gbs, gbs / peak))


if __name__ == '__main__':
  main()
