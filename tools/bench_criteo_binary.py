"""C2 (DeepFM, Criteo-shaped: 13 dense + 26 sparse, shared table) trained from CriteoInput binary parts:

  python tools/bench_criteo_binary.py [--batch 4096] [--steps 300]
  torchrun --nproc_per_node N tools/bench_criteo_binary.py ...

Rank 0 writes the C2 batches as binary parts (workloads.write_c2_binary) to a temporary directory; every rank trains
through EasyRecEstimator.train(readers.make_input(..., rank, N)) from them, then the same estimator over a few of its
batches already on the device.  Prints one JSON line: global samples/s from the files and device-resident, the reader's
host ms per batch (pread of one batch, nothing else), the er_binary_unpack time per batch (CUDA events over many
launches), the host-to-device bytes per step, and the card name and power limit read in the same run."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=4096)
  ap.add_argument('--steps', type=int, default=300)
  ap.add_argument('--warmup', type=int, default=20)
  ap.add_argument('--vocab', type=int, default=10_000_000)
  ap.add_argument('--files', type=int, default=8)
  ap.add_argument('--parallelism', choices=('dp', 'ep'), default='ep')
  ap.add_argument('--no-graph', action='store_true')
  args = ap.parse_args()

  import torch
  import torch.distributed as dist
  from bench_files_multi import card
  from easyrec_b200 import kernels as K, workloads
  from easyrec_b200.config import config_util
  from easyrec_b200.estimator import EasyRecEstimator
  from easyrec_b200.input import readers
  if not torch.cuda.is_available():
    raise SystemExit('bench_criteo_binary.py measures the GPU path: no CUDA device')
  rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
  local = int(os.environ.get('LOCAL_RANK', 0))
  dev = 'cuda:%d' % local
  torch.cuda.set_device(local)
  torch.backends.cuda.matmul.allow_tf32 = False
  if world > 1:
    dist.init_process_group('nccl', device_id=torch.device(dev))
  B, steps, warm = args.batch, args.steps, max(args.warmup, 1)
  per_rank = steps + warm + 1
  box = [tempfile.mkdtemp(prefix='er_criteo_binary_') if rank == 0 else None]
  if world > 1:
    dist.broadcast_object_list(box, src=0)
  tmp = box[0]
  if rank == 0:
    workloads.write_c2_binary(os.path.join(tmp, 'c2'), per_rank * world, B, n_files=max(args.files, world))
  if world > 1:
    dist.barrier()
  ep = world > 1 and args.parallelism == 'ep'
  cfg = config_util.get_configs_from_pipeline_file(workloads.c2_config_text(args.vocab, B, input_type='CriteoInput'))
  for kind in ('label', 'dense', 'category'):
    getattr(cfg.binary_train_input, kind + '_path').append(os.path.join(tmp, 'c2_part*_%s.bin' % kind))
  est = EasyRecEstimator(cfg, device=dev, seed=20240, use_cuda_graph=not args.no_graph, world_size=world, rank=rank,
                         embedding_parallel=ep)
  paths = cfg.binary_train_input

  def sync():
    torch.cuda.synchronize()
    if world > 1:
      dist.barrier()

  # the reader alone: host time to read one batch
  reader = readers.make_input(cfg, est.input_layer, paths, rank, world)
  it = iter(reader)
  next(it)
  t0 = time.perf_counter()
  n_read = 0
  for _ in range(min(100, reader.n_samples // B - 1)):
    next(it)
    n_read += 1
  read_ms = 1000.0 * (time.perf_counter() - t0) / max(n_read, 1)
  it.close()

  # end to end from the files
  fn = lambda: readers.make_input(cfg, est.input_layer, paths, rank, world)  # noqa: E731
  est.train(fn, steps=warm)
  sync()
  t0 = time.perf_counter()
  est.train(fn, steps=steps)
  sync()
  files_sps = world * B * steps / (time.perf_counter() - t0)
  h2d_per_step = est.last_feeder.h2d_bytes / steps

  # er_binary_unpack alone, on batches already on the device
  raw = next(iter(readers.make_input(cfg, est.input_layer, paths, rank, world)))[0]
  d_raw = [t.to(dev) for t in (raw.label, raw.dense, raw.cat)]
  maps = K.binary_maps(raw.slot_cols, raw.raw_cols, dev)
  outs = K.binary_unpack(*d_raw, *maps)
  for _ in range(20):
    K.binary_unpack(*d_raw, *maps, *outs)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  n_unpack = 2000
  e0.record()
  for _ in range(n_unpack):
    K.binary_unpack(*d_raw, *maps, *outs)
  e1.record()
  torch.cuda.synchronize()
  unpack_us = 1000.0 * e0.elapsed_time(e1) / n_unpack

  # device-resident: the same estimator over a few of its batches already unpacked on the device
  devb = [readers.to_device(f, l, dev) for _, (f, l) in zip(range(8), readers.make_input(cfg, est.input_layer, paths,
                                                                                          rank, world))]
  for i in range(warm):
    est.trainer.train_step(*devb[i % len(devb)], next_features=devb[(i + 1) % len(devb)][0] if ep else None)
  sync()
  t0 = time.perf_counter()
  for i in range(steps):
    est.trainer.train_step(*devb[i % len(devb)],
                           next_features=devb[(i + 1) % len(devb)][0] if ep and i + 1 < steps else None)
  sync()
  resident = world * B * steps / (time.perf_counter() - t0)
  if rank == 0:
    print(json.dumps({'metric': 'c2_criteo_binary_samples_per_s', 'n_gpus': world,
                      'parallelism': '%s%d' % ('ep' if ep else 'dp', world), 'batch_per_gpu': B, 'steps': steps,
                      'from_binary_files': files_sps, 'device_resident': resident, 'unit': 'samples/s',
                      'reader_host_ms_per_batch': read_ms, 'unpack_us_per_batch': unpack_us,
                      'h2d_bytes_per_step': h2d_per_step, 'card': card(local)}))
    shutil.rmtree(tmp, ignore_errors=True)
  if world > 1:
    dist.barrier()
    dist.destroy_process_group()
  return 0


if __name__ == '__main__':
  sys.exit(main())
