"""Error of er_gemm (3xTF32 on wgmma) vs cuBLAS fp32 SGEMM and single-pass TF32, against float64."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from easyrec_b200 import kernels as K

g = torch.Generator(device='cuda').manual_seed(0)
for M, N, Kd in [(1024, 256, 32), (1024, 256, 128), (1024, 256, 624), (1024, 256, 2048), (256, 256, 8192)]:
  for dist in ('randn', 'pos'):
    a = torch.randn(M, Kd, device='cuda', generator=g)
    b = torch.randn(Kd, N, device='cuda', generator=g)
    if dist == 'pos':
      a, b = a.abs(), b.abs()
    ref = a.double() @ b.double()
    scale = float(ref.abs().mean())
    out = {}
    out['er_gemm'] = K.gemm(a, b)
    torch.backends.cuda.matmul.allow_tf32 = False
    out['sgemm'] = torch.mm(a, b)
    torch.backends.cuda.matmul.allow_tf32 = True
    out['tf32'] = torch.mm(a, b)
    torch.backends.cuda.matmul.allow_tf32 = False
    msg = []
    for k, v in out.items():
      e = (v.double() - ref)
      msg.append('%s max %.2e rms %.2e bias %+.2e' % (k, float(e.abs().max()) / scale, float(e.pow(2).mean().sqrt()) / scale,
                                                    float(e.mean()) / scale))
    print('K=%5d %-5s |ref|~%.1f  ' % (Kd, dist, scale) + ' | '.join(msg), flush=True)
