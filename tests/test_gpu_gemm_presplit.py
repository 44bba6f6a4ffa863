"""GPU: the dense GEMM with a pre-split B (er_gemm_planes reading kernels.DensePlanes) is bit-identical to er_gemm /
er_gemm_bn on the same operands - outputs and batch-norm statistics alike - and the trainer's planes are never stale:
they are split from the weights each step starts with, whatever wrote those weights in between."""
import pytest
import torch

from easyrec_b200 import kernels as K
from easyrec_b200 import layers as L
from easyrec_b200 import workloads
from easyrec_b200.trainer import Trainer

pytestmark = pytest.mark.gpu

# (M, in, out): the C2 towers at batch 8192, then ragged K (not a multiple of 32) and MMA widths 16 / 32 / 64 / 128
SHAPES = [(8192, 624, 256), (8192, 256, 128), (8192, 128, 64), (8192, 81, 256),
          (1000, 17, 33), (777, 33, 17), (300, 624, 81), (513, 81, 624), (129, 40, 200), (64, 8, 8)]


def _pitched(g, rows, cols):
  """[rows, cols] view of a [rows, ceil4(cols) + 4] buffer (the layout of a concat output like [B, 81] in [B, 84])"""
  return torch.randn(rows, (cols + 3) // 4 * 4 + 4, device='cuda', generator=g)[:, :cols]


@pytest.mark.parametrize('M,n_in,n_out', SHAPES)
def test_presplit_forward_and_dx_are_bit_identical(M, n_in, n_out):
  g = torch.Generator(device='cuda').manual_seed(M + n_in + n_out)
  x = _pitched(g, M, n_in)
  w = torch.randn(n_in, n_out, device='cuda', generator=g) * 0.05
  gz = _pitched(g, M, n_out)
  bias = torch.randn(n_out, device='cuda', generator=g)
  planes = K.DensePlanes([w], 'cuda')
  planes.refresh()
  assert torch.equal(K.gemm(x, w, bias=bias), K.gemm(x, w, bias=bias, planes=planes.view(0, False)))
  assert torch.equal(K.gemm(gz, w.t()), K.gemm(gz, w.t(), planes=planes.view(0, True)))
  stats = []
  for p in (None, planes.view(0, False)):
    mm = torch.linspace(-1, 1, n_out, device='cuda')
    mv = torch.linspace(0.5, 2, n_out, device='cuda')
    r = K.gemm_bn(x, w, bias, mm, mv, 1e-3, 0.99, **({} if p is None else {'planes': p}))
    stats.append(None if r is None else r + (mm, mv))
  if stats[0] is None:   # a split K has no epilogue statistics: both forms decline it
    assert stats[1] is None and K._lib.load().er_gemm_workspace_bytes(M, n_out, n_in) > 0
    return
  for a, b in zip(*stats):
    assert torch.equal(a, b)


def test_presplit_split_k_is_bit_identical():
  """a short M over a long K takes the split-K path: the planes are read from the slice's first k-block"""
  g = torch.Generator(device='cuda').manual_seed(3)
  x = torch.randn(64, 4100, device='cuda', generator=g)
  w = torch.randn(4100, 40, device='cuda', generator=g)
  assert K._lib.load().er_gemm_workspace_bytes(64, 40, 4100) > 0
  planes = K.DensePlanes([w], 'cuda')
  planes.refresh()
  assert torch.equal(K.gemm(x, w), K.gemm(x, w, planes=planes.view(0, False)))


def _batch(B, seed):
  ids, dense, labels = workloads.criteo_batch(B, seed)
  return ({'sparse_fea': torch.from_numpy(ids).cuda(), 'dense_fea': torch.from_numpy(dense).cuda()},
          torch.from_numpy(labels).cuda())


def test_trainer_planes_follow_the_weights_each_step_starts_with():
  B = 1024
  il, model = workloads.build_deepfm_criteo(B, 100003, 'cuda', seed=11)
  tr = Trainer(model, il, 'adagrad', lr=0.05)
  kernels = tr.planes.kernels
  assert len(kernels) == 6
  x = torch.randn(B, 624, device='cuda')
  for step in range(2):
    w0 = [w.detach().clone() for w in kernels]
    tr.train_step(*_batch(B, 40 + step))
    torch.cuda.synchronize()
    assert any(not torch.equal(a, w) for a, w in zip(w0, kernels)), 'the step did not move the weights'
    for i, w in enumerate(w0):   # the planes this step used are the split of the weights it started with
      xi = x[:, :w.shape[0]]
      assert torch.equal(K.gemm(xi, w), K.gemm(xi, w, planes=tr.planes.view(i, False)))


def _run(monkeypatch, presplit, restore):
  if not presplit:
    monkeypatch.setattr(L, 'tower_kernels', lambda model: [])
  B = 2048
  il, model = workloads.build_deepfm_criteo(B, 100003, 'cuda', seed=23)
  tr = Trainer(model, il, 'adagrad', lr=0.05, use_cuda_graph=True)
  assert (tr.planes is not None) == presplit
  out = []
  for step in range(5):
    if step == 3:
      # a checkpoint restore between steps writes the weights behind the optimizer's back
      for name, p in model.named_parameters():
        if name in restore:
          p.data.copy_(restore[name])
    loss, probs = tr.train_step(*_batch(B, 70 + step))
    out.append((loss.clone(), probs.clone()))
  torch.cuda.synchronize()
  monkeypatch.undo()
  return out


def test_trainer_with_planes_trains_bit_identically_across_a_restore(monkeypatch):
  """eager warm-up steps, captured graph replays and a weight restore between two replays: losses and predictions
  equal those of a trainer whose GEMMs split the weights themselves"""
  _, model = workloads.build_deepfm_criteo(2048, 100003, 'cuda', seed=99)
  restore = {n: p.detach().clone() for n, p in model.named_parameters() if p.dim() == 2}
  a = _run(monkeypatch, True, restore)
  b = _run(monkeypatch, False, restore)
  for (la, pa), (lb, pb) in zip(a, b):
    assert torch.equal(pa, pb)
    # the reported loss adds the dense l2 term, which er_dense_apply sums with float atomics (any order)
    assert torch.allclose(la, lb, rtol=1e-6, atol=0)
