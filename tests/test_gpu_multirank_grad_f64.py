"""GPU: the row gradients of data-parallel and row-sharded training with 2, 3 and 4 ranks on ONE device, against a float64
restatement of every rank's batch over the global tables.

The ranks are processes on cuda:0 that talk over gloo (NCCL refuses two ranks on one device), eagerly: gloo collectives
cannot be captured, so the graph-replayed multi-rank steps stay with the 2-GPU NCCL tests.  gloo takes the CUDA tensors
of every collective these paths make (all_to_all_single, all_gather_into_tensor, all_reduce); none is wrapped.

Observing G is test_gpu_input_layer_grad_f64.py's method carried over to N ranks: momentum_optimizer at momentum 0 and
lr 1, every rank draws the same global tables (multiples of 1/16) from one seed, a row-sharded rank keeps the rows it
owns (local row i = global row i*N + r); the rank looks up its own batch, builds that file's loss with its own R / S / Q
weights plus the embedding regulariser, runs loss.backward(), zeroes every arena or shard and runs the path:

  * EmbeddingParallel (`sharded.py`): InputLayer.backward_update() - requester-side K7 into send_g, the gradient
    all-to-all, the owner-side K7 at 1/N;
  * data parallel (`distributed.py`): DataParallel.exchange(pending), join_presort(), apply_sparse(pending, opt), with
    and without pre_exchange(features) at the head of the step;

and reads G = -weight.  The reference restates each rank's batch in float64 over the global tables (the existing file's
Reference), sums those row gradients over the ranks with a CPU float64 all_reduce and divides by N.

What each case must satisfy:
  * rows no lookup of any rank reads are exactly 0, on every shard, the padding rows of a short last shard included;
  * on the linear paths (ids, shared tables, raw-value weights, sum-pooled tags, un-pooled and sum-pooled histories)
    every sum is exact, so at N = 2 and 4 (1/N a power of two) G equals the reference bit for bit;
  * at N = 3 the row rule scales the exact row sum S once: g = fl(S * fl(1/3)), and fl(1/3) = (1/3)(1 + d1),
    |d1| <= u = 2^-24, then the product rounds once more, (1 + d2).  So |G - S/3| <= (2u + u^2) |S/3|; the float64
    reference S/3 carries one more rounding of 2^-53, hence  |G - ref| <= (2u + u^2 + 2^-52) |ref|  per element, and
    ref == 0 forces G == 0;
  * mean / sqrtn pooling and attention: no worse than a float32 run of the same restatement (summed over the ranks in
    float32), the existing file's no_worse rule;
  * data-parallel replicas hold bit-identical tables (all-gathered and compared);
  * attention parameters: their gradient after the flat dense all-reduce (sync_dense_grads) times grad_scale = 1/N;
  * each case proves from the plan that it reached its path (check_plan).

Row-sharded edges: a per-peer block filled to exactly `cap` distinct rows loses nothing and check_exchange() stays quiet,
one row more and it raises with a count of 1; the prefetched id exchange gives G bit for bit as the plain step, and a
prefetched batch that is not the one looked up raises; with the owners' update held, a power-of-two factor put into the
gradient scale before apply_held() scales G exactly.

The host mirror runs the same workers on the CPU at N = 2 and 3 over gloo with tests/host_doubles.py (and
seq_doubles.py) in place of the kernels: it rehearses the restatement and the rank arithmetic without a device.  The
double of K1 takes no weights, so it prunes no mean / sqrtn lookup by weight: there the tag weights are positive and
carry no NaN.  pre_exchange does nothing on the CPU, so the mirror has no separate early-exchange case.

Measured on an H100 80GB HBM3 (700 W power limit): the three GPU worlds take 16 to 33 s each, about 70 to 90 s in
all, and peak at 0.07 GiB of reserved device memory per process; the worst error / bound at N = 3 is 0.67.  The host
mirror takes about 40 to 60 s.
"""
import datetime
import os
import socket
import sys
import traceback

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -24
BOUND3 = 2 * U + U * U + 2.0 ** -52   # |G - ref| / |ref| at N = 3 (docstring)
HOLD_FACTOR = 0.5


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


# ---- configs ------------------------------------------------------------------------------------------------------
def _configs():
  import test_gpu_input_layer_grad_f64 as S
  # ids: a hashed and identity ids, a shared table read by two features, a one-row raw projection and a raw_input_dim 3
  # one, a sum tag; the same features in a deep (dim 16) and a wide (dim 1) group, so both arenas share one row plan
  # (one exchange, two column blocks); a dim-6 arena (K7's scalar path) beside them, whose one-row raw projection takes
  # data parallel's local sum + all-reduce (an arena with multi-valued slots gathers its one-row lookups instead).
  # num_buckets 10, 50, 40, 100 and hash_bucket_size 500 are not multiples of 3 or 4: the last shards are short
  ids = S.head() + '''
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 16 hash_bucket_size: 500 }
  features { input_names: "a" feature_type: IdFeature embedding_dim: 16 num_buckets: 10 }
  features { input_names: "c1" feature_type: IdFeature embedding_dim: 16 num_buckets: 50 embedding_name: "shared" }
  features { input_names: "c2" feature_type: IdFeature embedding_dim: 16 num_buckets: 50 embedding_name: "shared" }
  features { input_names: "p" feature_type: RawFeature embedding_dim: 16 min_val: 0.0 max_val: 1.0 }
  features { input_names: "q" feature_type: RawFeature embedding_dim: 16 raw_input_dim: 3 min_val: 0.0 max_val: 1.0 }
  features { input_names: "z" feature_type: IdFeature embedding_dim: 6 num_buckets: 100 }
  features { input_names: "r" feature_type: RawFeature embedding_dim: 6 min_val: 0.0 max_val: 1.0 }
  features { input_names: "t" feature_type: TagFeature embedding_dim: 16 num_buckets: 40 combiner: "sum" }
}
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "deep" feature_names: ["u", "a", "c1", "c2", "p", "q", "t"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["u", "a", "c1", "c2", "p", "q", "t"] wide_deep: WIDE }
  feature_groups { group_name: "six" feature_names: ["z", "r"] wide_deep: DEEP }
  %s
  embedding_regularization: %r }
''' % (S.multi_tower(['deep', 'wide', 'six']), S.LAMBDA)
  # histories in tables of their own (a row-sharded table may not be read by history steps and other features): a plain
  # history and a multi-valued one (seq_multi_sep) pooled per step by `combiner`
  din = S.head() + '''
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 8 num_buckets: 30 }
  features { input_names: "item" feature_type: IdFeature embedding_dim: 8 num_buckets: 200 }
  features { input_names: "cate" feature_type: IdFeature embedding_dim: 8 num_buckets: 20 }
  features { input_names: "h_item" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 200 max_seq_len: 7 }
  features { input_names: "h_cate" feature_type: SequenceFeature embedding_dim: 8 num_buckets: 20 max_seq_len: 7
             seq_multi_sep: "#" combiner: "%%s" }
}
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "u" feature_names: ["u"] wide_deep: DEEP }
  seq_att_groups { group_name: "din" seq_att_map { key: "item" hist_seq: "h_item" }
                   seq_att_map { key: "cate" hist_seq: "h_cate" } }
  %s
  embedding_regularization: %r }
''' % (S.multi_tower(['u'], din=['din']), S.LAMBDA)
  # one id feature: the per-peer block capacity
  cap = S.head() + '''
feature_config { features { input_names: "x" feature_type: IdFeature embedding_dim: 8 num_buckets: 4000 } }
model_config { model_class: "MultiTowerDIN"
  feature_groups { group_name: "g" feature_names: ["x"] wide_deep: DEEP }
  %s
  embedding_regularization: %r }
''' % (S.multi_tower(['g']), S.LAMBDA)
  return dict(ids=ids, tags=S.head() + S.TAGS, din_sum=din % 'sum', din_mean=din % 'mean',
              seqc=S.head() + S.SEQC % (7, 7, S.multi_tower(['g']), S.LAMBDA), cap=cap)


EXACT = {'ids': True, 'tags': False, 'din_sum': True, 'din_mean': False, 'seqc': False, 'cap': True}


# ---- per-rank batches ---------------------------------------------------------------------------------------------
def _reshape_ids(x, nb, shape, rank, world):
  """identity ids (x >= 0) of one feature under a cross-rank batch shape: 'owner0' - every id a multiple of N, so rank 0
  owns them all and every other peer's block is empty; 'disjoint' - rank r draws from its own N-th of the range"""
  x = np.asarray(x).copy()
  live = (x >= 0) & (x < nb)
  if shape == 'owner0':
    x[live] -= x[live] % world
  elif shape == 'disjoint':
    k = nb // world
    x[live] = x[live] % k + rank * k
  return x


def _tag_reshaped(t, nb, shape, rank, world, dev):
  ids, lens, w = t
  return (torch.as_tensor(_reshape_ids(ids.cpu().numpy(), nb, shape, rank, world), device=dev), lens, w)


def _emptied(t, dev, B):
  """a bag feature with every bag of this rank empty"""
  w = t[2]
  return (torch.zeros(0, dtype=torch.int64, device=dev), torch.zeros(B, dtype=torch.int32, device=dev),
          None if w is None else torch.zeros(0, dtype=torch.float32, device=dev))


def make_batch(name, rng, B, dev, shape, rank, world, gpu):
  import test_gpu_input_layer_grad_f64 as S
  last = rank == world - 1
  if name == 'ids':
    u = rng.integers(-10 ** 12, 10 ** 12, B)
    a = rng.integers(-3, 14, B)                   # out of range -> bucket 0, -1 dropped
    a[:4] = [-1, 10, 13, 9]
    c1, c2, z = rng.integers(0, 50, B), rng.integers(0, 60, B), rng.integers(-1, 100, B)
    a, c1, c2, z = (_reshape_ids(v, nb, shape, rank, world) for v, nb in ((a, 10), (c1, 50), (c2, 50), (z, 100)))
    p = 2.0 ** rng.integers(-2, 1, (B, 1))
    q = 2.0 ** rng.integers(-2, 2, (B, 3)) * rng.choice([-1.0, 1.0], (B, 3))
    r = 2.0 ** rng.integers(-1, 2, (B, 1)) * rng.choice([-1.0, 1.0], (B, 1))
    t = S._tag(rng, B, 40, dev, True)
    t = _emptied(t, dev, B) if shape == 'empty' and last else _tag_reshaped(t, 40, shape, rank, world, dev)
    return {'sparse_fea': S._t(np.stack([u, a, c1, c2, z]).reshape(-1), dev),
            'dense_fea': S._t(np.concatenate([p, q, r], 1), dev, torch.float32), 'tag_fea': {'t': t}}
  if name == 'tags':
    # zero and negative kv weights, which K1 prunes under mean / sqrtn; NaN weights in `tn`, a mean feature that no
    # sum slot reads (a NaN weight in a sum slot is not pruned)
    i = _reshape_ids(rng.integers(-1, 100, B), 100, shape, rank, world)
    f = {'tm': S._tag(rng, B, 100, dev, True, drop=True, signs=gpu),
         'tq': S._tag(rng, B, 60, dev, True, drop=True, signs=gpu),
         'ts': S._tag(rng, B, 60, dev, False, drop=True),
         'tn': S._tag(rng, B, 100, dev, True, max_len=3, drop=True, signs=gpu)}
    if gpu:
      w = f['tn'][2].clone()
      w[rng.random(w.numel()) < 0.2] = float('nan')
      f['tn'] = (f['tn'][0], f['tn'][1], w)
    nbs = {'tm': 100, 'tq': 60, 'ts': 60, 'tn': 100}
    f = {k: _tag_reshaped(v, nbs[k], shape, rank, world, dev) for k, v in f.items()}
    if shape == 'empty' and last:
      f['ts'] = _emptied(f['ts'], dev, B)
    return {'sparse_fea': S._t(i, dev), 'tag_fea': f}
  if name in ('din_sum', 'din_mean'):
    f = S.seq_batch(['h_item', 'h_cate'], [200, 20], 7, mseq=('h_cate',), n_ids=[30, 200, 20])(rng, B, dev)
    ids = f['sparse_fea'].cpu().numpy().reshape(3, B)
    f['sparse_fea'] = S._t(np.concatenate([_reshape_ids(v, nb, shape, rank, world) for v, nb in zip(ids, (30, 200, 20))]),
                           dev)
    hi, hl = f['seq_fea']['h_item']
    if shape == 'empty' and last:
      hl = torch.zeros_like(hl)                   # every history of this rank is empty
    f['seq_fea']['h_item'] = (torch.as_tensor(_reshape_ids(hi.cpu().numpy(), 200, shape, rank, world), device=dev), hl)
    v, ln, per = f['seq_fea']['h_cate']
    f['seq_fea']['h_cate'] = (torch.as_tensor(_reshape_ids(v.cpu().numpy(), 20, shape, rank, world), device=dev), ln, per)
    return f
  if name == 'seqc':
    f = S.seq_batch(['zz', 'aa'], [40, 40], 7, n_ids=[30])(rng, B, dev)
    f['sparse_fea'] = S._t(_reshape_ids(f['sparse_fea'].cpu().numpy(), 30, shape, rank, world), dev)
    for n in ('zz', 'aa'):
      ids, ln = f['seq_fea'][n]
      if shape == 'empty' and last and n == 'zz':
        ln = torch.zeros_like(ln)
      f['seq_fea'][n] = (torch.as_tensor(_reshape_ids(ids.cpu().numpy(), 40, shape, rank, world), device=dev), ln)
    return f
  if name == 'cap':
    # `shape` distinct even ids (owner 0), the rest of the batch distinct odd ids (owner 1), each looked up once
    n_even = int(shape)
    x = np.concatenate([2 * np.arange(n_even), 2 * np.arange(B - n_even) + 1])
    return {'sparse_fea': S._t(rng.permutation(x), dev)}
  raise KeyError(name)


# ---- plan checks --------------------------------------------------------------------------------------------------
def check_plan(name, path, il, dp):
  if path == 'ep':
    exs = il._exchanges()
    members = [m for ex in exs for m in ex.members]
    if name == 'ids':
      assert {a.dim for a in il.arenas.values()} == {16, 6, 1}
      assert any(len(ex.heads) == 2 and ex.heads[1].col > 0 and ex.heads[1].call.arena.dim == 1 for ex in exs)
    if name == 'tags':
      assert any(m.csr and m.call.seg_scale is not None for m in members)
    if name.startswith('din') or name == 'seqc':
      assert any(m.seq is not None for m in members)
    if name.startswith('din'):
      assert any(m.csr for m in members)
    return
  gcalls = list(dp.gcalls.values())
  if name == 'ids':
    assert any(g.one_row for g in gcalls) and any(g.seg_off is not None for g in gcalls)
    if path == 'dp_pre' and str(il.device).startswith('cuda'):
      assert dp._pre      # the dim-6 arena's rows were gathered at the head of the step
  if name == 'tags':
    assert any(g.seg_off is not None and g.call.seg_scale is not None for g in gcalls)
  if name.startswith('din'):
    assert any(g.seg_off is not None for g in gcalls)


# ---- one case -----------------------------------------------------------------------------------------------------
class Case(object):
  def __init__(self, name, path, shape='rank', B=128, seed=0, prefetch=None, hold=False, slack=None):
    self.name, self.path, self.shape, self.B, self.seed = name, path, shape, B, seed
    self.prefetch, self.hold, self.slack = prefetch, hold, slack   # prefetch: None, 'same' or 'other'

  def __repr__(self):
    return '%s/%s/%s%s%s' % (self.name, self.path, self.shape, '/prefetch-' + self.prefetch if self.prefetch else '',
                             '/hold' if self.hold else '')


def _allreduce_cpu(t):
  import torch.distributed as dist
  t = t.detach().cpu().contiguous().clone()
  dist.all_reduce(t)
  return t


def run(case, rank, world, dev, gpu):
  """runs the case's step on this rank, restates it and returns (G per arena key, comparison data); every collective of
  the case happens here, before any check"""
  import test_gpu_input_layer_grad_f64 as S
  from easyrec_b200 import _lib, builder, trainer as T
  from easyrec_b200.config import config_util
  from easyrec_b200.distributed import DataParallel
  cfg = config_util.get_configs_from_pipeline_file(_configs()[case.name].encode())
  B, seed = case.B, case.seed
  if case.slack is not None:
    os.environ['ER_EP_SLACK'] = str(case.slack)
  try:
    il, model, _ = builder.build_model(cfg, B, dev, generator=torch.Generator(device=dev).manual_seed(seed + 1),
                                       cpu_generator=torch.Generator().manual_seed(seed + 2), world=world, rank=rank,
                                       shard_tables=case.path == 'ep')
  finally:
    os.environ.pop('ER_EP_SLACK', None)
  # the global layout (world 1) the reference reads the tables of
  gil, gmodel, _ = builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(seed + 2))
  assert all(a.opt_kind == _lib.OPT_SGD for a in il.arenas.values()) and il.emb_grad_mult == 1.0
  assert model.embedding_reg == S.LAMBDA and list(il.arenas) == list(gil.arenas)
  assert all(a.n_rows <= 10 ** 4 for a in gil.arenas.values())
  gen = torch.Generator().manual_seed(seed + 3)
  weights = {d: torch.randint(-8, 9, (a.n_rows, a.dim), generator=gen).double() / 16 for d, a in gil.arenas.items()}
  att_params = [p for m in il.attention_modules.values() for p in m.parameters() if p.requires_grad]
  named = [('att%d' % i, p) for i, p in enumerate(att_params)] or [('dummy', torch.nn.Parameter(
      torch.zeros(4, device=dev)))]
  dense_opt = T.FlatDenseOptimizer(named, 'sgd', 1.0)
  dp = DataParallel(il, dense_opt, world, sparse=case.path != 'ep')
  with torch.no_grad():
    for d, a in il.arenas.items():
      a.weight.zero_()
      if case.path == 'ep':
        for name, (off_e, local, v) in a.tables.items():
          off = gil.arenas[d].tables[name][0]
          src = weights[d][off:off + v][rank::world]
          a.weight[off_e:off_e + src.shape[0]].copy_(src.float().to(dev))
      else:
        a.weight.copy_(weights[d].float().to(dev))
    for mods in (il.attention_modules, gil.attention_modules):
      g2 = torch.Generator().manual_seed(seed + 6)
      for m in mods.values():
        for p in m.parameters():
          if p.requires_grad:
            p.copy_((torch.randn(p.shape, generator=g2) * 0.5).to(p.device))
  # this rank's batch: from (seed, rank), or from the seed alone when every rank reads the same batch
  rng = np.random.default_rng([seed, 0 if case.shape == 'same' else rank + 1])
  feats = make_batch(case.name, rng, B, dev, case.shape, rank, world, gpu)
  il.set_optimizer_step(1.0, 0)     # (after DataParallel: its 1/N is part of the device-resident gradient scale)
  if case.hold:
    il.ep_hold_updates(True)
  if case.prefetch:
    other = make_batch(case.name, np.random.default_rng([seed, 77, rank]), B, dev, case.shape, rank, world, gpu)
    il.prefetch_exchange(feats if case.prefetch == 'same' else other)
    assert all(ex._have_next for ex, _, _ in il._ex_plan)   # (a history's exchange runs with its lookup)
  if case.path == 'dp_pre':
    dp.pre_exchange(feats)
  groups = il.lookup(feats)
  check_plan(case.name, case.path, il, dp)
  seq_outputs = {g.group_name: il.seq_outputs[g.group_name] for g in cfg.model_config.seq_att_groups}
  W = S.Weights(1000 * seed + 10 * rank + 5)
  loss = S.loss_of(groups, seq_outputs, W) + model.embedding_reg_loss(S.package_reg_tensors(il, groups, seq_outputs))
  loss.backward()
  with torch.no_grad():
    for a in il.arenas.values():
      a.weight.zero_()
  dense_opt.gather_grads()
  pending = list(il._pending)
  if case.path == 'ep':
    il.backward_update()
    dp.exchange(pending)        # the dense all-reduce only
    if case.hold:
      il.hyper.dev[_lib.HYPER_GRAD_SCALE:_lib.HYPER_GRAD_SCALE + 1].mul_(HOLD_FACTOR)
      il.ep_apply_held()
  else:
    dp.exchange(pending)
    dp.join_presort()
    dp.apply_sparse(pending, il.opt_holder['opt'])
    il.discard_pending()
  scale = HOLD_FACTOR if case.hold else 1.0
  G = {d: (-a.weight.detach()).double().cpu() / scale for d, a in il.arenas.items()}
  att = [v.double().cpu() * dense_opt.grad_scale for v in dense_opt.grad_views[:len(att_params)]]
  lost = None
  if case.path == 'ep':
    try:
      il.check_exchange()
    except _lib.ErError as e:
      lost = str(e)
  out = dict(G=G, att=att, lost=lost, il=il, gil=gil, cap=il._exchanges()[0].cap if case.path == 'ep' else None)
  # -- the restatement of this rank's batch, summed over the ranks
  exact = EXACT[case.name]
  for dt in (torch.float64,) + (() if exact else (torch.float32,)):
    ref = S.Reference(cfg, gil, gmodel, feats, weights, dt)
    rl = S.loss_of(ref.groups, ref.seq_outputs, W) + S.LAMBDA * 0.5 * sum((t * t).sum() for t in ref.reg)
    rl.backward()
    out[dt] = dict(G={d: _allreduce_cpu(ref.leaves[d].grad) / world for d in weights},
                   att=[_allreduce_cpu(p.grad) / world for k in ref.att for p in ref.att[k]])
    if dt == torch.float64:
      out['touched'] = {d: _allreduce_cpu(ref.touched[d].to(torch.int32)) > 0 for d in weights}
  if case.path != 'ep':
    import torch.distributed as dist
    out['replicas'] = {}
    for d, g in G.items():
      w = il.arenas[d].weight.detach().cpu().contiguous().view(torch.int32)
      allw = [torch.empty_like(w) for _ in range(world)]
      dist.all_gather(allw, w)
      out['replicas'][d] = all(torch.equal(x, allw[0]) for x in allw)
  return out


def _local_map(il, gil, d, rank, world):
  """for every row of this rank's shard of arena d: its global row, -1 on a padding row"""
  m = torch.full((il.arenas[d].n_rows,), -1, dtype=torch.int64)
  for name, (off_e, local, v) in il.arenas[d].tables.items():
    off = gil.arenas[d].tables[name][0]
    g = torch.arange(v, dtype=torch.int64)[rank::world] + off
    m[off_e:off_e + g.numel()] = g
  return m


def compare(case, out, rank, world):
  """the checks of one case; returns the worst error / bound at N = 3 on its exact paths (0 elsewhere)"""
  import test_gpu_input_layer_grad_f64 as S
  il, gil, exact = out['il'], out['gil'], EXACT[case.name]
  r64, r32 = out[torch.float64], out.get(torch.float32)
  worst = 0.0
  assert out['lost'] is None, out['lost']
  for d in out['G']:
    g = out['G'][d]
    if case.path == 'ep':
      m = _local_map(il, gil, d, rank, world)
      live = m >= 0
      idx = torch.where(live, m, torch.zeros_like(m))
      g64 = torch.where(live[:, None], r64['G'][d][idx], torch.zeros_like(g))
      touched = live & out['touched'][d][idx]
      g32 = None if r32 is None else torch.where(live[:, None], r32['G'][d][idx], torch.zeros_like(g, dtype=torch.float32))
      names = [(n, i) for n, (off_e, local, v) in sorted(il.arenas[d].tables.items(), key=lambda kv: kv[1][0])
               for i in range(local)]
    else:
      assert out['replicas'][d], 'dim %s: the replicas hold different tables' % d
      g64, touched, g32 = r64['G'][d], out['touched'][d], None if r32 is None else r32['G'][d]
      names = S._row_names(gil, d)
    bad = (g[~touched] != 0).any(1) | torch.isnan(g[~touched]).any(1)
    if bool(bad.any()):
      i = int(torch.nonzero(~touched)[torch.nonzero(bad)[0, 0]])
      raise AssertionError('%r dim %s, table %s local row %d: untouched, but received %s' % (
          case, d, names[i][0], names[i][1], g[i].tolist()))
    if exact and world in (1, 2, 4):
      diff = (g != g64).any(1)
      if bool(diff.any()):
        i = int(torch.nonzero(diff)[0, 0])
        raise AssertionError('%r dim %s, table %s local row %d (exact path): %d rows differ; G %s, float64 %s' % (
            case, d, names[i][0], names[i][1], int(diff.sum()), g[i].tolist(), g64[i].tolist()))
    elif exact:
      err, bound = (g - g64).abs(), BOUND3 * g64.abs()
      over = err > bound
      if bool(over.any()):
        i = int(torch.nonzero(over.any(1))[0, 0])
        raise AssertionError('%r dim %s, table %s local row %d: |G - ref| above (2u + u^2 + 2^-52)|ref|; G %s, float64 '
                             '%s' % (case, d, names[i][0], names[i][1], g[i].tolist(), g64[i].tolist()))
      pos = bound > 0
      if bool(pos.any()):
        worst = max(worst, float((err[pos] / bound[pos]).max()))
    else:
      tab = [t for t, _ in names]
      for t in dict.fromkeys(tab):
        sel = torch.tensor([x == t for x in tab])
        S.no_worse(g[sel], g32[sel], g64[sel], '%r dim %s, table %s' % (case, d, t))
  for j, (got, p64) in enumerate(zip(out['att'], r64['att'])):
    S.no_worse(got.reshape(p64.shape), r32['att'][j], p64, '%r attention parameter %d' % (case, j))
  return worst


def cases(world, gpu):
  """the cases of one world; every rank runs them in this order"""
  names = ['ids', 'tags', 'din_sum', 'din_mean', 'seqc']
  paths = ['ep', 'dp', 'dp_pre'] if gpu else ['ep', 'dp']
  out = [Case(n, p) for n in names for p in paths]
  for shape in ('same', 'disjoint', 'owner0', 'empty'):
    out += [Case(n, p, shape) for n in (names if gpu else ['ids', 'tags', 'din_sum']) for p in ('ep', 'dp')]
  out += [Case(n, 'ep', prefetch='same') for n in ('ids', 'tags', 'din_sum')]
  out += [Case(n, 'ep', hold=True) for n in ('ids', 'tags', 'din_sum')]
  return out


def _worker(rank, port, ret, world, gpu):
  import torch.distributed as dist
  sys.path.insert(0, HERE)
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
  if gpu:
    dev = 'cuda:0'
    torch.cuda.set_device(0)
    torch.backends.cuda.matmul.allow_tf32 = False
  else:
    import host_doubles
    import seq_doubles
    host_doubles.install_all()
    seq_doubles.install()
    dev = 'cpu'
  errors, worst, plain = [], 0.0, {}
  for case in cases(world, gpu):
    out = run(case, rank, world, dev, gpu)
    try:
      worst = max(worst, compare(case, out, rank, world))
      key = (case.name, case.shape)
      if case.path == 'ep' and not case.prefetch and not case.hold:
        plain[key] = out['G']
      if case.prefetch:       # the prefetched id exchange: the same G, bit for bit, as the plain step
        for d, g in out['G'].items():
          assert torch.equal(g, plain[key][d]), '%r dim %s: G differs from the step without prefetch' % (case, d)
    except AssertionError:
      errors.append('rank %d: %s' % (rank, traceback.format_exc(limit=2)))
  # a prefetched batch that is not the one looked up
  out = run(Case('ids', 'ep', prefetch='other'), rank, world, dev, gpu)
  if out['lost'] is None or 'prefetched batch differed' not in out['lost']:
    errors.append('rank %d: a prefetched batch other than the looked-up one was not reported: %r' % (rank, out['lost']))
  if world == 2:
    # the per-peer block capacity: B = 1024 single-valued lookups, slack 0.01 -> cap = 512 rows per peer
    full = Case('cap', 'ep', shape=512, B=1024, slack=0.01)
    out = run(full, rank, world, dev, gpu)
    try:
      assert out['cap'] == 512, out['cap']
      compare(full, out, rank, world)
    except AssertionError:
      errors.append('rank %d: %s' % (rank, traceback.format_exc(limit=2)))
    out = run(Case('cap', 'ep', shape=513, B=1024, slack=0.01), rank, world, dev, gpu)
    if out['lost'] is None or not out['lost'].startswith('row-sharded exchange: 1 lookups exceeded the per-peer '
                                                         'capacity 512'):
      errors.append('rank %d: one row past the per-peer capacity was not reported as 1 lost lookup: %r' % (
          rank, out['lost']))
  peak = torch.cuda.max_memory_reserved() / 2 ** 30 if gpu else 0.0
  ret[rank] = (errors, worst, peak)
  dist.destroy_process_group()


def _spawn(world, gpu):
  import torch.multiprocessing as mp
  mgr = mp.Manager()
  ret = mgr.dict()
  mp.spawn(_worker, args=(_free_port(), ret, world, gpu), nprocs=world, join=True)
  assert len(ret) == world
  errors = [e for r in range(world) for e in ret[r][0]]
  assert not errors, '\n'.join(errors)
  worst = max(ret[r][1] for r in range(world))
  print('world %d: worst error / bound at N = 3 %.3f, peak reserved %.3f GiB per process' % (
      world, worst, max(ret[r][2] for r in range(world))))
  assert worst <= 1.0
  return worst


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize('world', [2, 3, 4])
def test_multirank_row_gradients_f64(world):
  _spawn(world, gpu=True)


@pytest.mark.timeout(600)
@pytest.mark.parametrize('world', [2, 3])
def test_multirank_restatement_on_the_host_doubles(world):
  _spawn(world, gpu=False)
