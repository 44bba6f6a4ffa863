"""Times the backbone DIN (workloads.c3_backbone_config_text: input_layer { output_seq_and_normal_feature } -> keras
DIN) against C3's MultiTowerDIN (workloads.c3_config_text) on the same batches: batch 4096, two length-50 histories,
1M-row item table.  Each model trains through its Trainer with the whole step in one CUDA graph; CUDA events bracket K
steps after W warm-up steps, and the models take turns for --rounds rounds so that drift of the shared machine hits
both.  Prints one JSON line with the card name and its power limit.

  python tools/bench_din_backbone.py --steps 200 --warmup 30 --rounds 3"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from easyrec_b200 import workloads  # noqa: E402
from easyrec_b200.estimator import EasyRecEstimator  # noqa: E402


def _card():
  name = torch.cuda.get_device_name(0)
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = 'unknown'
  return name, out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=200)
  ap.add_argument('--warmup', type=int, default=30)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--normalizer', default='softmax', choices=['softmax', 'sigmoid'])
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_din_backbone needs a GPU')
  dev = 'cuda:0'
  B, T, V = 4096, 50, 1_000_000
  batches = []
  for i in range(8):
    f, l = workloads.c3_batch(B, T, 777 + i, V)
    batches.append(({'sparse_fea': f['sparse_fea'].to(dev), 'dense_fea': f['dense_fea'].to(dev),
                     'seq_fea': {k: (a.to(dev), b.to(dev)) for k, (a, b) in f['seq_fea'].items()}}, l.to(dev)))
  models = {'backbone_din': workloads.c3_backbone_config_text(B, V, T, normalizer=args.normalizer),
            'multi_tower_din': workloads.c3_config_text(B, V, T)}
  ests = {k: EasyRecEstimator(text, device=dev, seed=20240, use_cuda_graph=True, default_seq_len=T)
          for k, text in models.items()}
  for est in ests.values():
    for i in range(args.warmup):
      est.trainer.train_step(*batches[i % 8])
  torch.cuda.synchronize()
  ms = {k: [] for k in ests}
  for _ in range(args.rounds):
    for k, est in ests.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for i in range(args.steps):
        est.trainer.train_step(*batches[i % 8])
      e1.record()
      torch.cuda.synchronize()
      ms[k].append(e0.elapsed_time(e1) / args.steps)
  name, limits = _card()
  res = {'card': name, 'power_limit_and_max_sm_clock': limits, 'batch': B, 'seq_len': T, 'item_rows': V,
         'normalizer': args.normalizer, 'steps': args.steps, 'warmup': args.warmup, 'rounds': args.rounds}
  for k, v in ms.items():
    res[k] = {'ms_per_step_median': float(np.median(v)), 'ms_per_step_all': [round(x, 4) for x in v],
              'samples_per_s': B / (float(np.median(v)) / 1000.0),
              'cuda_graph': ests[k].trainer._graph is not None}
  print(json.dumps(res))


if __name__ == '__main__':
  main()
