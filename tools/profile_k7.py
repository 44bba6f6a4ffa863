"""Per-kernel durations of er_embedding_bwd on the C2 batch, cold L2 (a 256 MB write between calls), through CUPTI
(torch.profiler).  `emit` profiles the radix engine instead: the call only writes the deduplicated gradient
(uniq_rows / uniq_grads, no table), as gradient clipping by global norm does.
usage: python tools/profile_k7.py [dim16|dim1] [iters] [emit]"""
import collections
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

from easyrec_b200 import _lib, kernels as K, workloads

B, V = 8192, int(os.environ.get('VOCAB', 10_000_000))
DIM = 1 if (len(sys.argv) > 1 and sys.argv[1] == 'dim1') else 16
N = int(sys.argv[2]) if len(sys.argv) > 2 else 10
EMIT = len(sys.argv) > 3 and sys.argv[3] == 'emit'
dev = 'cuda:0'
il, model = workloads.build_deepfm_criteo(B, V, dev, seed=20240)
call, arena = il.calls[DIM], il.arenas[DIM]
flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
gout = torch.randn(B, call.out_strides[0], device=dev) * 1e-3
rows_l, w_l = [], []
for i in range(4):
  ids, dense, _ = workloads.criteo_batch(B, 20240 + i, uniform=os.environ.get('UNIFORM') == '1')
  feats = {'sparse_fea': torch.from_numpy(ids).to(dev), 'dense_fea': torch.from_numpy(dense).to(dev)}
  cids, w = il._gather_inputs(DIM, feats['sparse_fea'], il.normalize_dense(feats['dense_fea']))
  rows_l.append(K.bucketize(cids, call.slots_dev, call.n_slots, call.n_seg).clone())
  w_l.append(w.clone())
opt = K.make_opt(_lib.OPT_ADAGRAD, 0.01)
L = rows_l[0].numel()
uniq = dict(uniq_rows=torch.empty(L, dtype=torch.int64, device=dev), uniq_grads=torch.empty(L, DIM, device=dev),
            n_uniq=torch.zeros(1, dtype=torch.int32, device=dev)) if EMIT else {}


def full(it):
  if EMIT:
    K.embedding_bwd(None, None, None, DIM, rows_l[it % 4], call.slots_dev, call.n_slots, call.n_seg, [gout], opt,
                    call.ws, weights=w_l[it % 4], n_rows=arena.weight.shape[0], **uniq)
  else:
    K.embedding_bwd(arena.weight, arena.state0, None, DIM, rows_l[it % 4], call.slots_dev, call.n_slots, call.n_seg,
                    [gout], opt, call.ws, weights=w_l[it % 4])


for it in range(3):
  full(it)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  for it in range(N):
    flush.fill_(float(it))
    full(it)
  torch.cuda.synchronize()
tot = collections.defaultdict(float)
cnt = collections.Counter()
for e in prof.events():
  if e.device_type == torch.autograd.DeviceType.CUDA and 'FillFunctor' not in e.name:
    tot[e.name] += e.device_time if hasattr(e, 'device_time') else e.cuda_time
    cnt[e.name] += 1
print('dim %d, engine %s: %.1f us of kernels per call' % (DIM, ('radix (emit)' if EMIT else 'bucketed'), sum(tot.values()) / N))
for name, v in sorted(tot.items(), key=lambda kv: -kv[1]):
  print('%8.1f us/call %5.1f x/call %7.1f us each  %s' % (v / N, cnt[name] / N, v / cnt[name], name[:110]))
