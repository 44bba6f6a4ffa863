"""C4 (DSSM two towers) with key-value tables (ev_params) on user_id and item_id against the same model with static
tables, on one GPU:

  python tools/bench_kv_embedding.py [--batch 4096] [--steps 200] [--capacity 20000000]

Both runs train the same 16 rotating zipf batches through EasyRecEstimator's trainer (CUDA graph).  Prints one JSON
line: samples/s of each, the time of the two key-value lookups of one batch repeated on the trained tables (every key
of the batch is already held, so this times finds, not inserts), and the keys held and occupancy of each key-value
table, with the card name and power limit read in the same run.  One GPU only: row-sharded runs are not measured here."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def run(text, batches, steps, warm):
  import torch
  from easyrec_b200.estimator import EasyRecEstimator
  est = EasyRecEstimator(text, device='cuda:0', seed=20240, use_cuda_graph=True)
  for i in range(warm):
    est.trainer.train_step(*batches[i % len(batches)])
  ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  ev0.record()
  for i in range(steps):
    est.trainer.train_step(*batches[i % len(batches)])
  ev1.record()
  torch.cuda.synchronize()
  est.input_layer.check_kv()
  return est, ev0.elapsed_time(ev1) / steps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=4096)
  ap.add_argument('--steps', type=int, default=200)
  ap.add_argument('--warmup', type=int, default=20)
  ap.add_argument('--vocab', type=int, default=25_000_000)
  ap.add_argument('--capacity', type=int, default=20_000_000)
  args = ap.parse_args()

  import torch
  from bench_files_multi import card
  from easyrec_b200 import workloads
  if not torch.cuda.is_available():
    raise SystemExit('bench_kv_embedding.py measures the GPU path: no CUDA device')
  torch.backends.cuda.matmul.allow_tf32 = False
  B = args.batch
  batches = [tuple(x.to('cuda:0') if not isinstance(x, dict) else {k: v.to('cuda:0') for k, v in x.items()}
                   for x in workloads.c4_batch(B, 4040 + i)) for i in range(16)]
  static, static_ms = run(workloads.c4_config_text(B, args.vocab, embedding_parallel=False), batches, args.steps,
                          args.warmup)
  del static
  torch.cuda.empty_cache()
  est, kv_ms = run(workloads.c4_config_text(B, args.vocab, embedding_parallel=False, kv_capacity=args.capacity),
                   batches, args.steps, args.warmup)
  # find-or-insert of one step: the keys K1 writes for each key-value arena, translated again on the warmed table
  il = est.input_layer
  from easyrec_b200 import kernels as K
  work = []
  feats = batches[0][0]
  for ak, call in il.calls.items():
    a = il.arenas[ak]
    if a.kv is not None:
      cids, _ = il._gather_inputs(ak, feats['sparse_fea'], None)
      keys = K.bucketize(cids, call.slots_dev, call.n_slots, call.n_seg)
      work.append((a.kv, keys, torch.empty_like(keys)))
  reps = 200
  ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  ev0.record()
  for _ in range(reps):
    for kv, keys, out in work:
      kv.lookup(keys, out, train=True)
  ev1.record()
  torch.cuda.synchronize()
  sizes = il.kv_sizes()
  gpu = card(0)
  print(json.dumps({
      'metric': 'samples/sec DSSM C4 on one GPU, key-value user_id / item_id tables vs static',
      'card': gpu['name'], 'power_limit_w': gpu['power_limit_w'], 'batch': B, 'steps': args.steps,
      'static': {'samples_per_s': B / (static_ms / 1000.0), 'ms_per_step': static_ms},
      'kv': {'samples_per_s': B / (kv_ms / 1000.0), 'ms_per_step': kv_ms,
             'lookup_of_held_keys_ms_per_step': ev0.elapsed_time(ev1) / reps,
             'keys': sizes, 'capacity': args.capacity,
             'occupancy': {t: n / float(args.capacity) for t, n in sizes.items()}},
      'c2': 'not measured'}))


if __name__ == '__main__':
  main()
