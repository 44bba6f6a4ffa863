"""Print the InputLayer plan of every stored reference sample config and of the workload configs as canonical JSON.

    python tools/dump_input_plan.py [--world N] [name-substring ...] > plan.json

The plan is everything the constructor fixes: per arena its tables, per launch its slot records, columns, output
strides and lookup capacity, the arena-wide merged slot plans, every group / sequence layout, `out_index` and the
attention modules' parameter shapes; with --world N > 1 the tables are row-sharded as rank 1 of N and the exchange
each launch joins is listed too.  A config that does not build is recorded with its error.  Two checkouts that print
the same JSON build the same plan.  Runs on the CPU with ER_PLAN_ONLY=1 (tables allocated, not initialised)."""
import argparse
import json
import os
import sys
import tarfile

os.environ['ER_PLAN_ONLY'] = '1'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from easyrec_b200 import builder, workloads  # noqa: E402
from easyrec_b200.config import config_util  # noqa: E402

V = 1000   # vocabulary of the workload configs' large tables


def configs():
  with tarfile.open(os.path.join(ROOT, 'tests', 'golden', 'reference_configs.tar.xz')) as tar:
    out = {m.name: tar.extractfile(m).read() for m in sorted(tar.getmembers(), key=lambda m: m.name) if m.isfile()}
  out['workloads/c2'] = workloads.c2_config_text(V, 16)
  out['workloads/c3'] = workloads.c3_config_text(16, item_vocab=V)
  out['workloads/c3_backbone'] = workloads.c3_backbone_config_text(16, item_vocab=V)
  out['workloads/c4'] = workloads.c4_config_text(16, item_vocab=V, user_vocab=V)
  out['workloads/c5'] = workloads.c5_config_text(16, vocab=V)
  return out


def group_entry(e):
  return [e.name, e.kind, e.width, e.dim, e.out_key, e.col, e.need_key]


def seq_entry(e):
  return [e.name, e.dim, e.out_key, e.col]


def plan(il):
  exchanges = []

  def ex_index(sc):
    sh = getattr(sc, 'sharded', None)
    if sh is None:
      return None
    if not any(x is sh.ex for x in exchanges):
      exchanges.append(sh.ex)
    return [next(i for i, x in enumerate(exchanges) if x is sh.ex), sh.cap, sh.L, sh.seq]

  subcalls = []
  for dim, subs in il.subcalls.items():
    for sk, sc in subs.items():
      c = sc.call
      subcalls.append(dict(dim=dim, key=list(sk), kind=sc.kind, slots=c.slots_np.tobytes().hex(),
                           slot_names=[s.name for s in c.slots], slot_cols=c.slot_cols, out_strides=c.out_strides,
                           out_widths=c.out_widths, max_lookups=c.max_lookups, n_seg=c.n_seg,
                           sources=[list(s) for s in getattr(c, 'sources', [])],
                           identity_ids=getattr(c, 'identity_ids', None), exchange=ex_index(sc)))
  merged = []
  for dim, m in il.merged.items():
    sh = getattr(m, 'sharded', None)
    merged.append(dict(dim=dim, slots=m.slots_np.tobytes().hex(), buf_of=[list(b) for b in m.buf_of],
                       sub_lookup_off=m.sub_lookup_off, sub_seg_off=m.sub_seg_off, max_lookups=m.max_lookups,
                       sharded=None if sh is None else [i for i, x in enumerate(exchanges) if x is sh.ex]))
  return dict(
      arenas=[dict(dim=a.dim, n_rows=a.n_rows, tables=[[n] + list(t) for n, t in a.tables.items()])
              for a in il.arenas.values()],
      subcalls=subcalls, merged=merged,
      calls=list(il.calls), static_w=[d for d, w in il.static_w.items() if w is not None],
      group_layout={g: [group_entry(e) for e in lay] for g, lay in il.group_layout.items()},
      seq_layout={s: dict(key=[seq_entry(e) for e in lay['key']], hist=[seq_entry(e) for e in lay['hist']], T=lay['T'])
                  for s, lay in il.seq_layout.items()},
      seq_group_layout={g: dict(seq=[seq_entry(e) for e in lay['seq']], T=lay['T'])
                        for g, lay in il.seq_group_layout.items()},
      seqc_order=il.seqc_order,
      out_index=[[d, k, list(sk), j] for (d, k), (sk, j) in il.out_index.items()],
      attention_modules={k: {n: list(p.shape) for n, p in m.named_parameters()}
                         for k, m in il.attention_modules.items()})


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--world', type=int, default=1)
  ap.add_argument('only', nargs='*', help='dump only the configs whose name contains one of these')
  args = ap.parse_args()
  out = {}
  for name, text in configs().items():
    if args.only and not any(s in name for s in args.only):
      continue
    try:
      cfg = config_util.get_configs_from_pipeline_file(text)
      il, _, _ = builder.build_model(cfg, 16, 'cpu', cpu_generator=torch.Generator().manual_seed(0),
                                     world=args.world, rank=min(1, args.world - 1), shard_tables=args.world > 1)
      out[name] = plan(il)
    except Exception as e:   # noqa: BLE001 - a refused config is part of the plan: its message must not change
      out[name] = dict(error='%s: %s' % (type(e).__name__, e))
  json.dump(out, sys.stdout, indent=1)   # (key order kept: group and launch order are part of the plan)
  sys.stdout.write('\n')


if __name__ == '__main__':
  main()
