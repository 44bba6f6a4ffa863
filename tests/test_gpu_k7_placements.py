"""One H100: K7's shared placements (embedding.Placements) on a Wide&Deep config whose wide dim-1 and deep dim-10 arenas
share one row plan - one placement mode each - in both group orders.  Every K7 that reuses a placement is shadowed, on
its own stream and inside the captured step, by a fresh er_embedding_bwd on a copy of the arena with the same rows and
gradients; the two must agree bit for bit in every eager and every graph-replayed step."""
import os
import sys

import pytest
import torch

from easyrec_b200 import embedding as E, kernels as K

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize('order', ['wide_first', 'deep_first'])
def test_reused_placements_equal_fresh_updates_in_eager_and_replayed_steps(order, monkeypatch):
  sys.path.insert(0, HERE)
  import ep_helpers
  from test_k7_placements import CFG
  from easyrec_b200.estimator import EasyRecEstimator
  cfg = CFG % 256
  if order == 'deep_first':
    wide = b'  feature_groups { group_name: "wide" feature_names: ["x", "a", "b", "c"] wide_deep: WIDE }\n'
    cfg = cfg.replace(wide, b'').replace(b'wide_deep: DEEP }\n', b'wide_deep: DEEP }\n' + wide)
  est = EasyRecEstimator(cfg, device=DEV, seed=5, use_cuda_graph=True)
  dims = list(est.input_layer.arenas)
  assert dims == ([1, 10] if order == 'wide_first' else [10, 1])
  mismatch = torch.zeros((), dtype=torch.int64, device=DEV)
  shadows, seen = {}, {}
  real = E.fused_backward_update

  def checked(call, rows, outs, opt, weights=None, row_ptr=None, seg_ids=None, sorted_from=None):
    a = call.arena
    seen.setdefault(a.dim, set()).add((id(rows), sorted_from is not None))
    if sorted_from is None:
      return real(call, rows, outs, opt, weights=weights, row_ptr=row_ptr, seg_ids=seg_ids)
    if a.dim not in shadows:   # (first seen in an eager step: nothing is allocated for the shadow inside the capture)
      shadows[a.dim] = (torch.empty_like(a.storage), K.bwd_workspace(call.max_lookups, a.device, a.dim))
    shadow, ws = shadows[a.dim]
    shadow.copy_(a.storage)
    gbufs = [(o.grad if o.grad is not None else torch.zeros_like(o)).contiguous() for o in outs]
    K.embedding_bwd(shadow[:, :a.dim], shadow[:, a.dim:2 * a.dim], None, a.dim, rows, call.slots_dev, call.n_slots,
                    call.n_seg, gbufs, opt, ws, weights=weights, seg_ids=seg_ids, row_ptr=row_ptr,
                    seg_scale=call.seg_scale)
    real(call, rows, outs, opt, weights=weights, row_ptr=row_ptr, seg_ids=seg_ids, sorted_from=sorted_from)
    mismatch.add_((shadow != a.storage).sum())
  monkeypatch.setattr(E, 'fused_backward_update', checked)

  start = {d: a.storage.clone() for d, a in est.input_layer.arenas.items()}
  for step in range(6):
    f, l = ep_helpers.batch(256, 0, step)
    est.trainer.train_step({k: v.to(DEV) for k, v in f.items()}, l.to(DEV))
  torch.cuda.synchronize()
  assert est.trainer._graph is not None                      # steps 3.. replayed a captured step
  # one row plan, and every update of it reused a placement of its own mode (the presort of the step)
  assert len({r for d in dims for r, _ in seen[d]}) == 1 and all(reused for d in dims for _, reused in seen[d])
  assert int(mismatch) == 0
  for d, a in est.input_layer.arenas.items():
    assert not torch.equal(a.storage, start[d])
