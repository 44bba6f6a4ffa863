"""Time the dense-tower GEMMs of the C2 DeepFM step one shape at a time: the forward (er_gemm_bn, batch statistics in
the epilogue, as a DNN layer with batch norm runs it in training), dX = dY.W^T and dW = X^T.dY (er_gemm) of the six
tower layers at batch 8192.  Each row gives the time per call from CUDA events over --iters calls replayed from a CUDA
graph; for dW (split along K = batch) that is everything the call enqueues, the split-K reduction included.  The
forward and dX GEMMs reading the pre-split weight planes (kernels.DensePlanes) are timed beside them and their outputs
are checked to be bit-identical.  Prints one JSON line per shape and the card it ran on."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from easyrec_b200 import kernels as K

B = 8192
LAYERS = [(624, 256), (256, 128), (128, 64), (81, 256), (256, 128), (128, 64)]   # deep tower, final tower


def timeit(fn, iters):
  """kernel time per call without the Python launch overhead: 20 back-to-back calls captured into a CUDA graph,
  the graph replayed iters / 20 times between two events"""
  rep = 20
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    for _ in range(3):
      fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
      for _ in range(rep):
        fn()
  torch.cuda.synchronize()
  for _ in range(3):
    g.replay()
  torch.cuda.synchronize()
  n = max(1, iters // rep)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(n):
    g.replay()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / (n * rep) * 1e3


def card():
  try:
    return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                                    '--format=csv,noheader'], text=True).strip()
  except (OSError, subprocess.CalledProcessError):
    return 'unknown'


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=2000)
  args = ap.parse_args()
  torch.backends.cuda.matmul.allow_tf32 = False
  dev = 'cuda:0'
  g = torch.Generator(device=dev).manual_seed(7)
  presplit = hasattr(K, 'DensePlanes')
  print(json.dumps({'card': card(), 'presplit_available': presplit}))
  tot = {'current': 0.0, 'presplit': 0.0, 'dW': 0.0}
  for kin, kout in LAYERS:
    pitch = (kin + 3) // 4 * 4
    x = torch.randn(B, pitch, device=dev, generator=g)[:, :kin]
    w = torch.randn(kin, kout, device=dev, generator=g) * 0.05
    bias = torch.zeros(kout, device=dev)
    gz = torch.randn(B, kout, device=dev, generator=g)
    mm, mv = torch.zeros(kout, device=dev), torch.ones(kout, device=dev)
    planes = None
    if presplit:
      planes = K.DensePlanes([w], dev)
      planes.refresh()
    cases = [('fwd', lambda p: K.gemm_bn(x, w, bias, mm, mv, 1e-3, 0.99, planes=p)),
             ('dX', lambda p: K.gemm(gz, w.t(), planes=p))] if presplit else \
            [('fwd', lambda p: K.gemm_bn(x, w, bias, mm, mv, 1e-3, 0.99)),
             ('dX', lambda p: K.gemm(gz, w.t()))]
    for name, fn in cases:
      row = {'gemm': name, 'M': B, 'K': kin if name == 'fwd' else kout, 'N': kout if name == 'fwd' else kin}
      row['current_us'] = timeit(lambda: fn(None), args.iters)
      tot['current'] += row['current_us']
      if presplit:
        p = planes.view(0, transposed=(name == 'dX'))
        row['presplit_us'] = timeit(lambda: fn(p), args.iters)
        tot['presplit'] += row['presplit_us']
        mm.zero_(); mv.fill_(1.0)
        r0 = fn(None)
        mm0, mv0 = mm.clone(), mv.clone()
        mm.zero_(); mv.fill_(1.0)
        r1 = fn(p)
        same = all(torch.equal(u, v) for u, v in zip(r0 if isinstance(r0, tuple) else (r0,),
                                                     r1 if isinstance(r1, tuple) else (r1,)))
        row['bit_identical'] = same and torch.equal(mm0, mm) and torch.equal(mv0, mv)
      print(json.dumps(row))
    # dW as DenseLayer's backward runs it: X^T (a transposed view of the pitched activations) times dY
    gk = torch.empty(kin, kout, device=dev)
    row = {'gemm': 'dW', 'M': kin, 'K': B, 'N': kout,
           'current_us': timeit(lambda: K.gemm(x.t(), gz, out=gk), args.iters)}
    tot['dW'] += row['current_us']
    print(json.dumps(row))
  print(json.dumps({'total_current_us': tot['current'], 'total_presplit_us': tot['presplit'] if presplit else None,
                    'total_dW_us': tot['dW']}))


if __name__ == '__main__':
  main()
