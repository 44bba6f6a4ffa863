"""Multi-GPU training from files on the C2 workload (DeepFM, Criteo-shaped: 13 dense + 26 sparse, shared table):

  torchrun --nproc_per_node N tools/bench_files_multi.py [--parallelism dp|ep] [--batch 4096] [--steps 50]

Rank 0 writes the C2 TSV and at least N Parquet files (workloads.write_c2_files) to a temporary directory, then every
rank trains through EasyRecEstimator.train(readers.make_input(..., rank, N)): rank r reads lines r::N of the TSV and
Parquet files r::N.  Prints one JSON line: global samples/s from CSV, from Parquet and device-resident (the same
estimator over batches already on the device), the parser threads per rank, the mean time of the per-step end-of-data
agreement, and the card name and power limit read in the same run."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(index):
  import torch
  out = {'name': torch.cuda.get_device_name(index), 'power_limit_w': None}
  try:
    q = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                       capture_output=True, text=True, timeout=20)
    out['power_limit_w'] = float(q.stdout.strip().splitlines()[0])
  except Exception:
    pass
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=4096)
  ap.add_argument('--steps', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--vocab', type=int, default=10_000_000)
  ap.add_argument('--parallelism', choices=('dp', 'ep'), default='ep')
  ap.add_argument('--no-graph', action='store_true')
  args = ap.parse_args()

  import torch
  import torch.distributed as dist
  from easyrec_b200 import workloads
  from easyrec_b200.estimator import EasyRecEstimator
  from easyrec_b200.input import readers
  rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
  local = int(os.environ.get('LOCAL_RANK', 0))
  cuda = torch.cuda.is_available()
  dev = 'cuda:%d' % local if cuda else 'cpu'
  if cuda:
    torch.cuda.set_device(local)
    torch.backends.cuda.matmul.allow_tf32 = False
  if world > 1:
    dist.init_process_group('nccl' if cuda else 'gloo', **({'device_id': torch.device(dev)} if cuda else {}))
  B, steps, warm = args.batch, args.steps, max(args.warmup, 1)
  per_rank = steps + warm + 1
  # the temporary directory of rank 0, announced to the others (ranks share the host's file system)
  box = [tempfile.mkdtemp(prefix='er_files_multi_') if rank == 0 else None]
  if world > 1:
    dist.broadcast_object_list(box, src=0)
  tmp = box[0]
  n_pq = max(world, 1)
  if rank == 0:
    tsv, _ = workloads.write_c2_files(os.path.join(tmp, 'c2'), per_rank * world, B)
    for j in range(n_pq):   # file j holds the batches of worker j
      workloads.write_c2_files(os.path.join(tmp, 'part-%03d' % j), per_rank, B, seed=30000 + 1000 * j)
  if world > 1:
    dist.barrier()
  tsv, pq_glob = os.path.join(tmp, 'c2.tsv'), os.path.join(tmp, 'part-*.parquet')
  ep = world > 1 and args.parallelism == 'ep'

  def build(input_type):
    text = workloads.c2_config_text(args.vocab, B, input_type=input_type)
    return EasyRecEstimator(text, device=dev, seed=20240, use_cuda_graph=cuda and not args.no_graph, world_size=world,
                            rank=rank, embedding_parallel=ep)

  def sync():
    if cuda:
      torch.cuda.synchronize()
    if world > 1:
      dist.barrier()

  def timed(est, input_fn):
    est.train(input_fn, steps=warm)
    sync()
    a0, n0 = est.agree_seconds, est.agree_calls
    t0 = time.perf_counter()
    est.train(input_fn, steps=steps)
    sync()
    dt = time.perf_counter() - t0
    agree_ms = 1000.0 * (est.agree_seconds - a0) / max(est.agree_calls - n0, 1)
    return world * B * steps / dt, agree_ms

  est = build('CSVInput')
  cfg = est._pipeline_config
  csv_reader = readers.make_input(cfg, est.input_layer, tsv, rank, world)
  csv_sps, agree_ms = timed(est, lambda: readers.make_input(cfg, est.input_layer, tsv, rank, world))
  # device-resident: the same estimator over a few of its own batches already on the device
  devb = [readers.to_device(f, l, dev) for _, (f, l) in zip(range(8), readers.make_input(cfg, est.input_layer, tsv, rank,
                                                                                          world))]
  for i in range(warm):
    est.trainer.train_step(*devb[i % len(devb)], next_features=devb[(i + 1) % len(devb)][0] if ep else None)
  sync()
  t0 = time.perf_counter()
  for i in range(steps):
    est.trainer.train_step(*devb[i % len(devb)],
                           next_features=devb[(i + 1) % len(devb)][0] if ep and i + 1 < steps else None)
  sync()
  resident = world * B * steps / (time.perf_counter() - t0)
  del est, devb
  if cuda:
    torch.cuda.empty_cache()
  est = build('ParquetInput')
  cfg_pq = est._pipeline_config
  pq_sps, _ = timed(est, lambda: readers.make_input(cfg_pq, est.input_layer, pq_glob, rank, world))
  if rank == 0:
    print(json.dumps({'metric': 'c2_files_multi_samples_per_s', 'n_gpus': world,
                      'parallelism': '%s%d' % ('ep' if ep else 'dp', world), 'batch_per_gpu': B, 'steps': steps,
                      'from_csv': csv_sps, 'from_parquet': pq_sps, 'device_resident': resident, 'unit': 'samples/s',
                      'parser_threads_per_rank': csv_reader.n_threads, 'agree_ms_per_step': agree_ms,
                      'card': card(local) if cuda else None}))
    shutil.rmtree(tmp, ignore_errors=True)
  if world > 1:
    dist.barrier()
    dist.destroy_process_group()
  return 0


if __name__ == '__main__':
  sys.exit(main())
