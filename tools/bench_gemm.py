"""Time er_gemm (wgmma 3xTF32) against torch.mm fp32 SGEMM on the dense-layer shapes of the C2 DeepFM step."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from easyrec_b200 import kernels as K

torch.backends.cuda.matmul.allow_tf32 = False
B = 8192
shapes = [(624, 256), (256, 128), (128, 64), (81, 256), (64, 1)]


def timeit(fn, n=20):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(n):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / n * 1e3


for kin, kout in shapes:
  pitch = (kin + 3) // 4 * 4
  x = torch.randn(B, pitch, device='cuda')[:, :kin]
  w = torch.randn(kin, kout, device='cuda')
  gz = torch.randn(B, kout, device='cuda')
  for name, a, b in [('fwd', x, w), ('dX ', gz, w.t()), ('dW ', x.t(), gz)]:
    if b.shape[1] % 4 and name != 'fwd':
      pass
    t_er = timeit(lambda: K.gemm(a, b))
    t_th = timeit(lambda: torch.mm(a, b))
    fl = 2.0 * a.shape[0] * a.shape[1] * b.shape[1]
    err = float((K.gemm(a, b) - torch.mm(a, b)).abs().max())
    print('%s [%5d x %4d x %5d]  er_gemm %7.1f us (%6.1f TFLOP/s fp32-equiv)   torch.mm %7.1f us   max|diff| %.2e'
          % (name, a.shape[0], b.shape[1], a.shape[1], t_er, fl / t_er * 1e-6, t_th, err))
