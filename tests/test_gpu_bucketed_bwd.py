"""GPU parity of K7 on the bucketed dedup (bucket_bwd.cuh: hash the lookups into buckets by row, one warp sorts each
bucket on (row, lookup) in registers, the run kernels sum and apply) against the CPU oracle, through the C ABI.

Equal rows come out adjacent and in ascending lookup order, as from the radix sort, so short runs are summed in the
oracle's sequential order and hot rows by fixed chunked trees (tolerance stated).  Covered: every dim class (vector
4..128, scalar 1 and 6), CSR with weights and mean / sqrtn scaling, dropped lookups, duplicates of one row that overflow a warp's
128 pairs (CTA sort), a CTA's 16384 pairs (global-memory radix fallback), one-row slots (ER_BUCKET_ONE_ROW), the
presort + reuse split, clustered rows (identity ids), device-side lookup counts, and agreement with the radix engine
(uniq_rows output) at the C2 size.
"""
import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, kernels as K
from oracle import oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def t(a):
  return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _case(kind, dim, rng, V, B, F, with_csr=False, hot=(), one_row=False, clustered=False):
  combs = ([0, 1, 2] * F)[:F] if with_csr else [0] * F
  n_tab = V + (F if one_row else 0)
  table = rng.normal(size=(n_tab, dim)).astype(np.float32)
  s0 = np.full((n_tab, dim), 0.1, np.float32) if kind == _lib.OPT_ADAGRAD else np.zeros((n_tab, dim), np.float32)
  s1 = np.zeros((n_tab, dim), np.float32)
  if with_csr:
    lens = rng.integers(0, 5, B * F).astype(np.int32)
    L = int(lens.sum())
  else:
    lens = np.ones(B * F, np.int32)
    L = B * F
  rows = (rng.integers(0, min(V, 300), L) if clustered else rng.integers(0, V, L)).astype(np.int64)
  for row, count in hot:
    rows[rng.choice(L, min(count, L), replace=False)] = row
  rows[rng.integers(0, L, L // 25 + 1)] = -1
  modes = [3] * F
  offs = [0] * F
  if one_row:   # the last two slots are one-row tables appended behind the V shared rows
    for f in (F - 2, F - 1):
      modes[f] = _lib.BUCKET_ONE_ROW
      offs[f] = V + f
      sl = slice(f * B, (f + 1) * B)
      rows[sl] = np.where(rows[sl] < 0, -1, V + f)
  w = rng.uniform(0.1, 2.0, L).astype(np.float32) if (with_csr or one_row) else None
  stride = F * dim + (4 - F * dim % 4) % 4
  gout = rng.normal(size=(B, stride)).astype(np.float32)
  recs = [dict(num_buckets=V, row_offset=offs[f], seg_begin=f * B, n_seg=B, bucket_mode=modes[f], combiner=combs[f],
               out_buf=0, out_stride=stride, out_col=f * dim) for f in range(F)]
  sd = K.slots_to_device(K.make_slots(recs), DEV)
  return dict(table=table, s0=s0, s1=s1, lens=lens, L=L, rows=rows, w=w, stride=stride, gout=gout, sd=sd, combs=combs,
              n_tab=n_tab)


def _run(kind, dim, c, B, F, with_csr, presort=False):
  d_table, d_s0, d_s1, d_rows = t(c['table']), t(c['s0']), t(c['s1']), t(c['rows'])
  row_ptr = seg_ids = scale = None
  L = c['L']
  if with_csr:
    row_ptr, seg_ids = K.csr_from_lens(t(c['lens']), L)
    scale = torch.empty(B * F, device=DEV)
    out = torch.empty(B, c['stride'], device=DEV)
    K.embedding_fwd(d_table, dim, d_rows, c['sd'], F, B * F, [out], weights=t(c['w']), row_ptr=row_ptr, seg_scale=scale)
  opt = K.make_opt(kind, 0.05, beta1_power=0.9**4, beta2_power=0.999**4, grad_scale=0.5)
  ws = K.bwd_workspace(L, DEV, dim)
  src = None
  if presort:
    K.embedding_bwd_presort(d_rows, c['n_tab'], dim, ws, c['sd'], F, seg_ids=seg_ids, row_ptr=row_ptr, n_seg=B * F)
    src = (ws, dim)
  K.embedding_bwd(d_table, d_s0 if kind != _lib.OPT_SGD else None,
                  d_s1 if kind == _lib.OPT_LAZY_ADAM else None, dim, d_rows, c['sd'], F, B * F, [t(c['gout'])], opt,
                  ws, weights=None if c['w'] is None else t(c['w']), seg_ids=seg_ids, row_ptr=row_ptr, seg_scale=scale,
                  sorted_from=src)
  torch.cuda.synchronize()
  table, s0, s1 = c['table'].copy(), c['s0'].copy(), c['s1'].copy()
  gseg = np.concatenate([c['gout'][:, f * dim:(f + 1) * dim] for f in range(F)], 0)
  _, seg_of = O.csr_from_lens(c['lens'])
  oscale = None
  if with_csr:
    _, oscale = O.embedding_fwd(c['table'], c['rows'], O.csr_from_lens(c['lens'])[0],
                                np.repeat(np.array(c['combs'], np.int32), B), weights=c['w'])
  okind = {_lib.OPT_SGD: O.OPT_SGD, _lib.OPT_ADAGRAD: O.OPT_ADAGRAD, _lib.OPT_LAZY_ADAM: O.OPT_LAZY_ADAM}[kind]
  O.embedding_bwd(table, s0, s1, c['rows'], seg_of, gseg, okind, 0.05, weights=c['w'], seg_scale=oscale,
                  beta1_power=0.9**4, beta2_power=0.999**4, grad_scale=0.5)
  return (d_table.cpu().numpy(), d_s0.cpu().numpy(), d_s1.cpu().numpy()), (table, s0, s1)


def _check(got, want, long_rows=()):
  cold = np.ones(want[0].shape[0], bool)
  cold[list(long_rows)] = False
  for g, w_ in zip(got, want):
    # short runs, summed in the oracle's order
    np.testing.assert_allclose(g[cold], w_[cold], rtol=2e-6, atol=2e-6)
    if long_rows:   # fixed-tree sums of hundreds..tens of thousands of N(0,1) gradients
      np.testing.assert_allclose(g[~cold], w_[~cold], rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize('kind', [_lib.OPT_SGD, _lib.OPT_ADAGRAD, _lib.OPT_LAZY_ADAM])
@pytest.mark.parametrize('dim,with_csr', [(16, False), (16, True), (1, False), (32, True), (6, True), (4, False),
                                          (64, False), (128, True), (8, False)])
def test_bucketed_bwd_matches_the_oracle(kind, dim, with_csr):
  rng = np.random.default_rng(kind * 1000 + dim)
  B, F, V = 700, 3, 5000
  hot = [(5, 300), (9, 70), (11, 65), (12, 64)]      # hot-row kernel runs, and both sides of its 64-lookup boundary
  c = _case(kind, dim, rng, V, B, F, with_csr=with_csr, hot=hot)
  got, want = _run(kind, dim, c, B, F, with_csr)
  _check(got, want, long_rows=[5, 9, 11, 12])
  # untouched rows did not move at all
  touched = np.unique(c['rows'][c['rows'] >= 0])
  mask = np.ones(V, bool)
  mask[touched] = False
  assert np.array_equal(got[0][mask], c['table'][mask])


@pytest.mark.parametrize('dim', [16, 1, 6])
def test_big_buckets_and_beyond_shared_memory(dim):
  """2000 and 6000 duplicates of one row (buckets sorted by a CTA in shared memory) and 20000 of a third (more than
  the 16384 pairs a CTA can hold: global-memory radix fallback)."""
  rng = np.random.default_rng(dim)
  B, F, V = 12000, 4, 200000
  hot = [(17, 2000), (123456, 6000), (99, 20000)]
  c = _case(_lib.OPT_ADAGRAD, dim, rng, V, B, F, hot=hot)
  got, want = _run(_lib.OPT_ADAGRAD, dim, c, B, F, False)
  _check(got, want, long_rows=[17, 123456, 99])
  assert not np.array_equal(got[0][[17, 123456, 99]], c['table'][[17, 123456, 99]])


@pytest.mark.parametrize('dim', [16, 1])
@pytest.mark.parametrize('presort', [False, True])
def test_one_row_slots_take_the_column_sum_path(dim, presort):
  rng = np.random.default_rng(40 + dim)
  B, F, V = 1500, 5, 3000
  c = _case(_lib.OPT_ADAGRAD, dim, rng, V, B, F, hot=[(7, 100)], one_row=True)
  got, want = _run(_lib.OPT_ADAGRAD, dim, c, B, F, False, presort=presort)
  one = [V + F - 2, V + F - 1]
  _check(got, want, long_rows=[7] + one)
  for r in one:    # 1500 weighted gradient rows into ONE table row: tight relative to the summed magnitude
    assert np.abs(got[0][r] - want[0][r]).max() < 1e-5


def test_clustered_rows_and_device_side_counts():
  """identity-style ids (all rows < 300 of a 1M-row table) spread over the buckets; CSR count read on the device."""
  rng = np.random.default_rng(3)
  B, F, V = 2000, 3, 1_000_000
  c = _case(_lib.OPT_LAZY_ADAM, 16, rng, V, B, F, with_csr=True, clustered=True)
  got, want = _run(_lib.OPT_LAZY_ADAM, 16, c, B, F, True)
  runs = np.bincount(c['rows'][c['rows'] >= 0])
  _check(got, want, long_rows=list(np.flatnonzero(runs > 32)))


def _reuse_case(V, B, F, dim):
  r2 = np.random.default_rng(dim)
  table = t(r2.normal(size=(V, dim)).astype(np.float32))
  acc = t(np.full((V, dim), 0.1, np.float32))
  stride = (F * dim + 3) // 4 * 4
  gout = t(r2.normal(size=(B, stride)).astype(np.float32))
  recs = [dict(num_buckets=V, row_offset=0, seg_begin=f * B, n_seg=B, bucket_mode=3, combiner=0, out_buf=0,
               out_stride=stride, out_col=f * dim) for f in range(F)]
  return table, acc, gout, K.slots_to_device(K.make_slots(recs), DEV)


def _reuse_rows(V, B, F):
  rng = np.random.default_rng(21)
  rows = (rng.zipf(1.2, B * F) % V).astype(np.int64)
  rows[rng.integers(0, B * F, 30)] = -1
  rows[rng.integers(0, B * F, 200)] = 7
  return t(rows)


def _presort_then_two_tables_equals_fresh_calls(first, second):
  """the second table reuses the placement of the first call, of the same placement mode: bit for bit a fresh call"""
  V, B, F = 3000, 400, 5
  d_rows = _reuse_rows(V, B, F)
  res = {}
  for mode in ('fresh', 'reuse'):
    out = []
    ws_first = K.bwd_workspace(B * F, DEV, first)
    for dim in (first, second):
      table, acc, gout, sd = _reuse_case(V, B, F, dim)
      ws = ws_first if dim == first else K.bwd_workspace(B * F, DEV, dim)
      src = None
      if mode == 'reuse':
        if dim == first:
          K.embedding_bwd_presort(d_rows, V, first, ws_first, sd, F)
        src = (ws_first, first)
      K.embedding_bwd(table, acc, None, dim, d_rows, sd, F, B * F, [gout], K.make_opt(_lib.OPT_ADAGRAD, 0.05), ws,
                      sorted_from=src)
      out.append((table.cpu(), acc.cpu()))
    res[mode] = out
  for (ta, aa), (tb, ab) in zip(res['fresh'], res['reuse']):
    assert torch.equal(ta, tb) and torch.equal(aa, ab)


def test_presort_then_two_tables_equals_fresh_calls():
  """DeepFM's plan: the wide dim-1 table reuses the placement of the deep dim-16 call (warp-sized buckets)."""
  _presort_then_two_tables_equals_fresh_calls(16, 1)


def test_presort_then_two_cta_mode_tables_equals_fresh_calls():
  """the same with CTA-sized buckets: a dim-10 table reuses the placement of a dim-64 call."""
  _presort_then_two_tables_equals_fresh_calls(64, 10)


@pytest.mark.parametrize('placed,dim', [(16, 64), (64, 16)])
def test_reuse_across_placement_modes_is_refused(placed, dim):
  """A warp-mode placement is no placement for a CTA-mode table, nor the other way round: ER_ERR_UNSUPPORTED, and
  neither the table nor its optimizer state moves."""
  V, B, F = 3000, 400, 5
  d_rows = _reuse_rows(V, B, F)
  _, _, _, sd_placed = _reuse_case(V, B, F, placed)
  ws_placed = K.bwd_workspace(B * F, DEV, placed)
  K.embedding_bwd_presort(d_rows, V, placed, ws_placed, sd_placed, F)
  table, acc, gout, sd = _reuse_case(V, B, F, dim)
  table0, acc0 = table.clone(), acc.clone()
  with pytest.raises(_lib.ErError, match=r'\(status %d\)' % _lib.ER_ERR_UNSUPPORTED):
    K.embedding_bwd(table, acc, None, dim, d_rows, sd, F, B * F, [gout], K.make_opt(_lib.OPT_ADAGRAD, 0.05),
                    K.bwd_workspace(B * F, DEV, dim), sorted_from=(ws_placed, placed))
  torch.cuda.synchronize()
  assert torch.equal(table, table0) and torch.equal(acc, acc0)


def test_c2_size_bucketed_equals_radix_engine_and_is_deterministic():
  """B=8192 x 39 slots over a 10M-row table, Zipf ids + 13 one-row slots: the bucketed engine, the radix engine
  (selected by asking for the uniq_rows output) and a repeat of the bucketed call agree."""
  B, F, D, V = 8192, 39, 16, 10_000_000
  rng = np.random.default_rng(8)
  ids = (rng.zipf(1.05, 26 * B).astype(np.int64) - 1) % (2**40)
  ids = ids * 26 + np.repeat(np.arange(26, dtype=np.int64), B)
  recs = [dict(num_buckets=1, row_offset=f, seg_begin=f * B, n_seg=B, bucket_mode=_lib.BUCKET_ONE_ROW, combiner=0,
               out_buf=0, out_stride=F * D, out_col=f * D) for f in range(13)]
  recs += [dict(num_buckets=V, row_offset=13, seg_begin=f * B, n_seg=B, bucket_mode=_lib.BUCKET_FARM_DECIMAL, combiner=0,
                out_buf=0, out_stride=F * D, out_col=f * D) for f in range(13, F)]
  sd = K.slots_to_device(K.make_slots(recs), DEV)
  all_ids = t(np.concatenate([np.zeros(13 * B, np.int64), ids]))
  rows = K.bucketize(all_ids, sd, F, B * F)
  assert int(rows[:13 * B].max()) == 12 and int(rows[13 * B:].min()) >= 13
  g = torch.Generator(device=DEV).manual_seed(1)
  table0 = torch.randn(V + 13, D, device=DEV, generator=g) * 0.01
  gout = torch.randn(B, F * D, device=DEV, generator=g) * 0.01
  w = torch.cat([torch.rand(13 * B, device=DEV, generator=g), torch.ones(26 * B, device=DEV)])
  ws = K.bwd_workspace(B * F, DEV, D)
  outs = []
  for engine in ('bucket', 'bucket', 'radix'):
    table, acc = table0.clone(), torch.full((V + 13, D), 0.1, device=DEV)
    kw = {}
    if engine == 'radix':
      kw = dict(uniq_rows=torch.empty(B * F, dtype=torch.int64, device=DEV), uniq_grads=torch.empty(B * F, D, device=DEV),
                n_uniq=torch.zeros(1, dtype=torch.int32, device=DEV))
    K.embedding_bwd(table, acc, None, D, rows, sd, F, B * F, [gout], K.make_opt(_lib.OPT_ADAGRAD, 0.01), ws, weights=w, **kw)
    outs.append((table, acc))
  assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])       # deterministic
  changed_b = (outs[0][0] != table0).any(1)
  changed_r = (outs[2][0] != table0).any(1)
  assert torch.equal(changed_b, changed_r) and int(changed_b.sum()) == int(torch.unique(rows).numel())
  # different (both fixed) orders of fp32 additions inside hot rows: small relative to the accumulated gradient
  assert float((outs[0][0] - outs[2][0]).abs().max()) < 2e-6
  assert float((outs[0][1] - outs[2][1]).abs().max() / outs[2][1].abs().max()) < 1e-5
