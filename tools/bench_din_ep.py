"""Times C3 (workloads.c3_config_text: MultiTowerDIN, two behaviour histories, a large item table) with row-sharded
tables (train_distribute: EmbeddingParallelStrategy, histories exchanged step by step) against replicated data parallel
on the same per-rank batches.  Each model trains through its Trainer with the whole step in one CUDA graph; CUDA events
bracket K steps after W warm-up steps, and the two take turns for --rounds rounds so that drift of the shared machine
hits both.  Rank 0 prints one JSON line: samples/s over all ranks, library launches per step, the history steps each
rank looks up per step and the distinct history rows it requests from the owners, and the card name with its power
limit.

  torchrun --nproc_per_node 2 tools/bench_din_ep.py --steps 100 --warmup 20 --rounds 3

Without GPUs the script builds the configs and the batches and stops where the first device is needed."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from easyrec_b200 import workloads  # noqa: E402
from easyrec_b200.config import config_util  # noqa: E402

N_BATCHES = 4


def _card():
  name = torch.cuda.get_device_name(0)
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = 'unknown'
  return name, out


def _to(f, l, dev):
  return ({'sparse_fea': f['sparse_fea'].to(dev), 'dense_fea': f['dense_fea'].to(dev),
           'seq_fea': {k: (a.to(dev), b.to(dev)) for k, (a, b) in f['seq_fea'].items()}}, l.to(dev))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=100)
  ap.add_argument('--warmup', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--batch', type=int, default=4096, help='per rank')
  ap.add_argument('--seq-len', type=int, default=50)
  ap.add_argument('--item-rows', type=int, default=1_000_000)
  args = ap.parse_args()
  world, rank = int(os.environ.get('WORLD_SIZE', '1')), int(os.environ.get('RANK', '0'))
  B, T, V = args.batch, args.seq_len, args.item_rows
  texts = {'row_sharded': workloads.c3_config_text(B, V, T).replace(
               b'train_config {', b'train_config { train_distribute: EmbeddingParallelStrategy', 1),
           'data_parallel': workloads.c3_config_text(B, V, T)}
  for text in texts.values():
    config_util.get_configs_from_pipeline_file(text)
  host = [workloads.c3_batch(B, T, 777 + 1000 * rank + i, V) for i in range(N_BATCHES)]
  hist_steps = [int(sum(int(n.sum()) for _, n in f['seq_fea'].values())) for f, _ in host]
  if not torch.cuda.is_available():
    raise SystemExit('bench_din_ep: configs and %d batches of %d built (%d history steps per batch on average); timing '
                     'needs GPUs: torchrun --nproc_per_node N tools/bench_din_ep.py' % (N_BATCHES, B, np.mean(hist_steps)))
  if world < 2:
    raise SystemExit('bench_din_ep: row sharding needs at least 2 ranks (torchrun --nproc_per_node N, N >= 2)')
  import torch.distributed as dist
  from easyrec_b200.estimator import EasyRecEstimator
  local = int(os.environ.get('LOCAL_RANK', rank))
  torch.cuda.set_device(local)
  dev = 'cuda:%d' % local
  dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device(dev))
  torch.backends.cuda.matmul.allow_tf32 = False
  batches = [_to(f, l, dev) for f, l in host]
  ests = {k: EasyRecEstimator(text, device=dev, seed=20240, world_size=world, rank=rank,
                              embedding_parallel=(k == 'row_sharded'), use_cuda_graph=True, default_seq_len=T)
          for k, text in texts.items()}
  for est in ests.values():
    for i in range(args.warmup):
      est.trainer.train_step(*batches[i % N_BATCHES])
  torch.cuda.synchronize()
  ms = {k: [] for k in ests}
  for _ in range(args.rounds):
    for k, est in ests.items():
      dist.barrier()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for i in range(args.steps):
        est.trainer.train_step(*batches[i % N_BATCHES])
      e1.record()
      torch.cuda.synchronize()
      ms[k].append(e0.elapsed_time(e1) / args.steps)
  # distinct history rows this rank asked the owners for in the last step (K8's per-owner counts of the history calls)
  il = ests['row_sharded'].input_layer
  requested = sum(int(sc.sharded.ex.counts[:world].sum()) for subs in il.subcalls.values() for sc in subs.values()
                  if sc.kind == 'seq')
  il.check_exchange()
  if rank == 0:
    name, limits = _card()
    res = {'card': name, 'power_limit_and_max_sm_clock': limits, 'world': world, 'batch_per_rank': B, 'seq_len': T,
           'item_rows': V, 'steps': args.steps, 'warmup': args.warmup, 'rounds': args.rounds,
           'history_steps_per_rank_per_step': float(np.mean(hist_steps)),
           'history_rows_requested_per_rank_last_step': requested}
    for k, v in ms.items():
      med = float(np.median(v))
      res[k] = {'ms_per_step_median_rank0': med, 'ms_per_step_all_rank0': [round(x, 4) for x in v],
                'samples_per_s': world * B / (med / 1000.0), 'launches_per_step': ests[k].trainer.launches_per_step,
                'cuda_graph': ests[k].trainer._graph is not None}
    print(json.dumps(res))
  dist.barrier()
  dist.destroy_process_group()


if __name__ == '__main__':
  main()
