"""CPU, kernel doubles, world 2 and 3 over gloo: multi-worker training from files.

* Shard rule: worker r of N reads the lines r::N of a CSV file (after the header) - dataset.shard(N, r) of the reference
  (input/input.py:1018-1023) - and cuts its batches from them in file order: its batches are those of the unsharded
  reader over a file holding only those lines, bit for bit, for both engines.  Parquet files are dealt out by
  `file index % N == r` (parquet_input.py:36-57).
* Training: N workers at batch B over one file train the model one process trains at batch N*B over the same lines
  (step k of the workers together is lines [kNB, (k+1)NB)), replicated or row-sharded, on a model without batch norm.
* End of data: the workers agree before every step, so uneven shards stop every worker at the same step; evaluate() and
  predict() cover every worker's full batches (row-sharded workers that ran out keep joining the exchange).
* Metrics: evaluate() returns one dict on every worker, that of one process evaluating the union of their batches."""
import ctypes
import os
import socket
import sys
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from easyrec_b200 import _lib, builder
from easyrec_b200.config import config_util
from easyrec_b200.input import readers

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import test_csv_native as csvn  # noqa: E402
import test_ep_tags_gloo as tags  # noqa: E402

# DeepFM without batch norm over an id sharing its table with a key:weight tag, a hashed string tag and a raw value
TRAIN_CFG = b'''
%s
train_config { optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.1 } } } } }
data_config { batch_size: %d input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "u" input_type: INT64 }
  input_fields { input_name: "t1" input_type: STRING } input_fields { input_name: "t2" input_type: STRING }
  input_fields { input_name: "x" input_type: FLOAT } }
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 4 num_buckets: 9 embedding_name: "e" }
  features { input_names: "t1" feature_type: TagFeature embedding_dim: 4 num_buckets: 9 embedding_name: "e" separator: "|"
             kv_separator: ":" combiner: "mean" }
  features { input_names: "t2" feature_type: TagFeature embedding_dim: 4 hash_bucket_size: 13 separator: "|" combiner: "sum" }
  features { input_names: "x" feature_type: RawFeature embedding_dim: 4 min_val: 0.0 max_val: 2.0 } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["u", "t1", "t2", "x"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["u", "t2"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [8] use_bn: false } final_dnn { hidden_units: [4] use_bn: false } l2_regularization: 1e-3 }
  }
eval_config { metrics_set { auc {} } metrics_set { max_f1 {} } metrics_set { mean_absolute_error {} }
  metrics_set { root_mean_squared_error {} } metrics_set { gauc { uid_field: "u" } } }
'''

# the same model over Parquet columns: scalar id, list-valued tag, dense value
PARQUET_CFG = b'''
%s
train_config { optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.1 } } } } }
data_config { batch_size: %d input_type: ParquetInput label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "u" input_type: INT64 }
  input_fields { input_name: "tg" input_type: INT64 } input_fields { input_name: "x" input_type: FLOAT } }
feature_config {
  features { input_names: "u" feature_type: IdFeature embedding_dim: 4 num_buckets: 9 embedding_name: "e" }
  features { input_names: "tg" feature_type: TagFeature embedding_dim: 4 num_buckets: 9 embedding_name: "e" combiner: "mean" }
  features { input_names: "x" feature_type: RawFeature embedding_dim: 4 min_val: 0.0 max_val: 2.0 } }
model_config { model_class: "DeepFM"
  feature_groups { group_name: "deep" feature_names: ["u", "tg", "x"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["u", "tg"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [8] use_bn: false } final_dnn { hidden_units: [4] use_bn: false } l2_regularization: 1e-3 }
  }
eval_config { metrics_set { auc {} } metrics_set { max_f1 {} } metrics_set { mean_squared_error {} } }
'''


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _spawn(fn, world, args, timeout=420):
  """run fn(rank, *args) in `world` processes; a worker that has not finished after `timeout` seconds fails the test"""
  ctx = mp.start_processes(fn, args=args, nprocs=world, join=False, start_method='spawn')
  deadline = time.time() + timeout
  while not ctx.join(timeout=5):
    if time.time() > deadline:
      for p in ctx.processes:
        if p.is_alive():
          p.kill()
      pytest.fail('workers still running after %d s: a rank is blocked in a collective' % timeout)


def _train_lines(n, seed):
  rng = np.random.default_rng(seed)
  out = []
  for _ in range(n):
    t1 = '|'.join('%d:%.2f' % (rng.integers(0, 9), rng.uniform(0.2, 2.0)) for _ in range(rng.integers(0, 4)))
    t2 = '|'.join('w%d' % rng.integers(0, 30) for _ in range(rng.integers(0, 5)))
    out.append('%d,%d,%s,%s,%.3f' % (rng.integers(0, 2), rng.integers(0, 9), t1, t2, rng.uniform(0, 2)))
  return out


def _write(path, lines, header=None, last_newline=True):
  text = '\n'.join(([header] if header else []) + lines) + ('\n' if last_newline else '')
  open(path, 'w', newline='').write(text)


def _with_header(cfg):
  return cfg.replace(b'data_config {', b'data_config { with_header: true', 1)


# ---- shard rule ------------------------------------------------------------------------------------------------------
def _check_shards(cfg_bytes, B, lines, tmp, header, last_newline, engines=('native', 'python'), worlds=(2, 3)):
  cfg_bytes = _with_header(cfg_bytes) if header else cfg_bytes
  cfg = config_util.get_configs_from_pipeline_file(cfg_bytes)
  il, _, _ = builder.build_model(cfg, B, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  path = os.path.join(tmp, 'all.csv')
  _write(path, lines, 'h' if header else None, last_newline)
  total = 0
  for N in worlds:
    for r in range(N):
      mine = lines[r::N]
      own = os.path.join(tmp, 'own_%d_%d.csv' % (N, r))
      # (the last line of the whole file lacks its '\n' only in the file whose last line it is)
      _write(own, mine, 'h' if header else None, last_newline or (len(lines) - 1) % N != r)
      want = list(readers.CSVInput(cfg, il, own, engine='native'))
      assert len(want) == len(mine) // B
      for engine in engines:
        got = list(readers.CSVInput(cfg, il, path, engine=engine, n_threads=3, task_index=r, task_num=N))
        assert len(got) == len(want), (N, r, engine)
        for a, b in zip(got, want):
          csvn._same(a, b)
      total += len(want)
  return total


@pytest.mark.parametrize('header,last_newline', [(False, True), (True, False), (True, True), (False, False)])
def test_csv_worker_reads_lines_r_mod_n_scalar_string_history_tag_columns(tmp_path, header, last_newline):
  """hashed string ids, 19-digit integers, defaults, missing trailing fields, a 3-wide raw vector, a history, a
  string tag; the line count leaves the last line to a different worker per N"""
  B = 16
  p = str(tmp_path / 'gen.csv')
  csvn._file(p, 16 * 6 * 3 + 5, np.random.default_rng(4), last_newline=True)
  lines = open(p, newline='').read().split('\n')[:-1]
  assert _check_shards(csvn.CFG.replace(b'batch_size: 64', b'batch_size: 16'), B, lines, str(tmp_path), header,
                       last_newline) > 0


@pytest.mark.parametrize('header,last_newline', [(False, False), (True, True)])
def test_csv_worker_reads_lines_r_mod_n_kv_tags_and_multi_valued_steps(tmp_path, header, last_newline):
  """key:weight tags, plain hashed tags and a SequenceFeature with seq_multi_sep (every step a list)"""
  lines = tags._lines(12 * 7 + 2, 9)
  assert _check_shards(tags.CFG % b'', 12, lines, str(tmp_path), header, last_newline) > 0


def test_csv_worker_shards_across_the_native_chunk_boundary(tmp_path):
  """more than 32K lines per worker: the native engine's chunked calls carry the file's line index from one chunk to
  the next (scalar, hashed, history and tag columns, the last partial batch skipped)"""
  B = 500
  p = str(tmp_path / 'gen.csv')
  csvn._file(p, 100003, np.random.default_rng(8), last_newline=True)
  lines = open(p, newline='').read().split('\n')[:-1]
  cfg = csvn.CFG.replace(b'batch_size: 64', b'batch_size: 500')
  assert _check_shards(cfg, B, lines, str(tmp_path), False, False, engines=('native',), worlds=(2, 3)) >= 5 * 66


def test_native_lines_seen_accounting_matches_the_python_split():
  """er_csv_parse_lines keeps every stride-th line from line `phase`, stops after max_rows kept lines and reports the
  complete lines it passed over; the unterminated tail is never counted"""
  lib = _lib.load()
  text = b''.join(b'%d\n' % i for i in range(23)) + b'99'
  py_lines = text.split(b'\n')[:-1]            # complete lines only, as the python engine's split sees them
  for stride in (1, 2, 3, 5):
    for phase in range(stride):
      for max_rows in (0, 1, 3, 100):
        out = np.full(64, -7, np.int64)
        col = _lib.ErCsvCol()
        col.kind, col.out = _lib.CSV_I64, out.ctypes.data
        n, used, seen = ctypes.c_int64(), ctypes.c_size_t(), ctypes.c_int64()
        assert lib.er_csv_parse_lines(text, len(text), b',', ctypes.byref(col), 1, max_rows, 2, stride, phase,
                                      ctypes.byref(n), ctypes.byref(used), ctypes.byref(seen)) == 0
        kept = list(range(phase, len(py_lines), stride))[:max_rows]
        assert out[:n.value].tolist() == [int(py_lines[i]) for i in kept]
        passed = (kept[-1] + 1) if len(kept) == max_rows and max_rows else (0 if max_rows == 0 else len(py_lines))
        assert seen.value == passed and used.value == sum(len(l) + 1 for l in py_lines[:passed]), (stride, phase, max_rows)
  col = _lib.ErCsvCol()
  col.kind, col.out = _lib.CSV_I64, np.zeros(4, np.int64).ctypes.data
  n, used, seen = ctypes.c_int64(), ctypes.c_size_t(), ctypes.c_int64()
  assert lib.er_csv_parse_lines(text, len(text), b',', ctypes.byref(col), 1, 4, 1, 3, 3, ctypes.byref(n),
                                ctypes.byref(used), ctypes.byref(seen)) == _lib.ER_ERR_INVALID_ARG


# ---- Parquet ---------------------------------------------------------------------------------------------------------
def _parquet_files(directory, n_files, rows, seed=0, prefix='part'):
  import pyarrow as pa
  import pyarrow.parquet as pq
  rng = np.random.default_rng(seed)
  paths = []
  for k in range(n_files):
    tab = pa.table({'label': pa.array((rng.uniform(size=rows) < 0.4).astype(np.float32)),
                    'u': pa.array(rng.integers(0, 9, rows).astype(np.int64)),
                    'tg': pa.array([[int(v) for v in rng.integers(0, 9, int(m))] for m in rng.integers(0, 4, rows)],
                                   pa.list_(pa.int64())),
                    'x': pa.array(rng.uniform(0, 2, rows).astype(np.float32))})
    paths.append(os.path.join(directory, '%s-%02d.parquet' % (prefix, k)))
    pq.write_table(tab, paths[-1], row_group_size=5)
  return paths


def test_parquet_files_are_dealt_by_index_and_a_worker_without_a_file_is_an_error(tmp_path):
  pytest.importorskip('pyarrow')
  paths = _parquet_files(str(tmp_path), 5, 8)
  cfg = config_util.get_configs_from_pipeline_file(PARQUET_CFG % (b'', 4))
  il, _, _ = builder.build_model(cfg, 4, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
  pattern = os.path.join(str(tmp_path), 'part-*.parquet')
  assert readers.ParquetInput(cfg, il, pattern).paths == paths
  for N in (2, 3, 5):
    for r in range(N):
      got = readers.make_input(cfg, il, pattern, r, N)
      assert got.paths == paths[r::N]
      want = list(readers.ParquetInput(cfg, il, paths[r::N]))
      mine = list(got)
      assert len(mine) == len(want) > 0
      for a, b in zip(mine, want):
        csvn._same(a, b)
  # comma-separated patterns are expanded one after the other, each sorted
  two = ','.join([os.path.join(str(tmp_path), 'part-0[34].parquet'), os.path.join(str(tmp_path), 'part-0[0-2].parquet')])
  assert readers.ParquetInput(cfg, il, two, task_index=1, task_num=2).paths == [paths[4], paths[1]]
  with pytest.raises(ValueError, match='5 file.*task_num 6'):
    readers.make_input(cfg, il, pattern, 5, 6)


# ---- training / evaluation over gloo ---------------------------------------------------------------------------------
def _ep_flag(mode):
  return b'train_config { train_distribute: EmbeddingParallelStrategy }' if mode == 'ep' else b''


def _record_losses(est):
  losses = []
  real = est.trainer.train_step

  def step(*a, **k):
    out = real(*a, **k)
    losses.append(float(out[0]))
    return out
  est.trainer.train_step = step
  return losses


def _copy_weights(src, dst, rank, world, ep):
  """the replicated model `src` (world 1) -> `dst` (this worker; row-sharded tables take their rows r::N)"""
  import ep_helpers
  if ep:
    ep_helpers.copy_tables(src.input_layer, dst.input_layer, rank, world)
  else:
    for d, a in src.input_layer.arenas.items():
      dst.input_layer.arenas[d].storage.copy_(a.storage)
  dst.model.load_state_dict(src.model.state_dict())
  dst.trainer.dense_opt.flat_p.copy_(src.trainer.dense_opt.flat_p)


def _drift(one, est, rank, world, ep):
  """largest difference of tables + optimizer slots, and of dense parameters + their slots"""
  import ep_helpers
  worst = 0.0
  for dim, a in one.input_layer.arenas.items():
    b = est.input_layer.arenas[dim]
    if not ep:
      worst = max(worst, float((a.storage - b.storage).abs().max()))
      continue
    for name, (off, _, v) in a.tables.items():
      off_e = b.tables[name][0]
      want = ep_helpers.shard_of(a.storage, off, v, rank, world)
      if want.numel():
        worst = max(worst, float((want - b.storage[off_e:off_e + want.shape[0]]).abs().max()))
  do1, do2 = one.trainer.dense_opt, est.trainer.dense_opt
  dworst = float((do1.flat_p - do2.flat_p).abs().max())
  for s1, s2 in ((do1.s0, do2.s0), (do1.s1, do2.s1)):
    if s1 is not None:
      dworst = max(dworst, float((s1 - s2).abs().max()))
  return worst, dworst


def _gather(obj):
  import torch.distributed as dist
  out = [None] * dist.get_world_size()
  dist.all_gather_object(out, obj)
  return out


def _close(a, b, tol=1e-6):
  assert sorted(a) == sorted(b), (a, b)
  for k in a:
    assert abs(a[k] - b[k]) <= tol or (np.isnan(a[k]) and np.isnan(b[k])), (k, a[k], b[k])


def _equivalence_worker(rank, port, ret, world, tmp, mode, fmt, cuda=False, graph=False):
  from test_dp_clip_gloo import _setup
  import torch.distributed as dist
  dev = _setup(rank, port, world, cuda)
  from easyrec_b200.estimator import EasyRecEstimator, train_and_evaluate
  ep = mode == 'ep'
  B = 8
  base = TRAIN_CFG if fmt == 'csv' else PARQUET_CFG
  cfg_n, cfg_1 = base % (_ep_flag(mode), B), base % (b'', B * world)
  est = EasyRecEstimator(cfg_n, device=dev, seed=3, world_size=world, rank=rank, use_cuda_graph=graph)
  one = EasyRecEstimator(cfg_1, device=dev, seed=3)
  assert est.embedding_parallel == ep
  _copy_weights(one, est, rank, world, ep)
  c_n, c_1 = est._pipeline_config, one._pipeline_config
  if fmt == 'csv':
    train, evalp = os.path.join(tmp, 'train.csv'), os.path.join(tmp, 'eval.csv')
    train_1, eval_1 = train, evalp
  else:
    train = evalp = os.path.join(tmp, 'part-*.parquet')
    train_1 = eval_1 = os.path.join(tmp, 'union.parquet')

  # -- evaluation and prediction with the same weights: one dict on every worker, that of the union
  ev = est.evaluate(lambda: readers.make_input(c_n, est.input_layer, evalp, rank, world))
  ev1 = one.evaluate(lambda: readers.make_input(c_1, one.input_layer, eval_1))
  dicts = _gather(ev)
  assert all(d == dicts[0] for d in dicts), dicts
  _close(ev, ev1)
  if fmt == 'csv':
    mine = np.concatenate([p['probs'] for p in est.predict(lambda: readers.make_input(c_n, est.input_layer, evalp,
                                                                                      rank, world))])
    allp = np.concatenate([p['probs'] for p in one.predict(lambda: readers.make_input(c_1, one.input_layer, eval_1))])
    assert mine.shape == allp[rank::world].shape and np.abs(mine - allp[rank::world]).max() <= 1e-6

  # -- training, step by step
  l_n, l_1 = _record_losses(est), _record_losses(one)
  est.train(lambda: readers.make_input(c_n, est.input_layer, train, rank, world))
  one.train(lambda: readers.make_input(c_1, one.input_layer, train_1))
  assert len(l_n) == len(l_1) > 0 and est.global_step == one.global_step
  mean = torch.tensor(l_n, dtype=torch.float64)
  dist.all_reduce(mean)
  mean = (mean / world).numpy()
  assert np.abs(mean - np.array(l_1)).max() <= 1e-5, (mean, l_1)
  worst, dworst = _drift(one, est, rank, world, ep)
  assert worst <= 2e-6 and dworst <= 2e-6, (worst, dworst)

  # -- train_and_evaluate reads this worker's shards of train_input_path / eval_input_path
  if fmt == 'csv' and not cuda:
    path = os.path.join(tmp, 'pipeline.config')
    if rank == 0:
      open(path, 'wb').write(cfg_n + b'train_input_path: "%s" eval_input_path: "%s"\n' % (train.encode(), evalp.encode()))
    dist.barrier()
    a, ev_a = train_and_evaluate(path, device=dev, seed=5, world_size=world, rank=rank)
    b = EasyRecEstimator(path, device=dev, seed=5, world_size=world, rank=rank)
    b.train(lambda: readers.make_input(b._pipeline_config, b.input_layer, train, rank, world))
    ev_b = b.evaluate(lambda: readers.make_input(b._pipeline_config, b.input_layer, evalp, rank, world))
    assert ev_a == ev_b and a.global_step == b.global_step == len(l_1)
    for d, x in a.input_layer.arenas.items():
      assert torch.equal(x.storage, b.input_layer.arenas[d].storage)
  ret[rank] = (len(l_n), worst, dworst)
  if cuda:
    dist.barrier()
    os._exit(0)
  dist.destroy_process_group()


def _prepare(tmp, world, fmt, B=8, steps=4, eval_steps=3):
  if fmt == 'csv':
    _write(os.path.join(tmp, 'train.csv'), _train_lines(world * B * steps, 11))
    _write(os.path.join(tmp, 'eval.csv'), _train_lines(world * B * eval_steps, 12))
    return
  import pyarrow as pa
  import pyarrow.parquet as pq
  paths = _parquet_files(tmp, world, B * steps, seed=13)
  # one process at batch N*B sees the workers' step k side by side: rows of file 0 step k, file 1 step k, ...
  tabs = [pq.read_table(p) for p in paths]
  parts = [t.slice(k * B, B) for k in range(steps) for t in tabs]
  pq.write_table(pa.concat_tables(parts), os.path.join(tmp, 'union.parquet'))


@pytest.mark.timeout(900)
@pytest.mark.parametrize('world,mode,fmt', [(2, 'dp', 'csv'), (3, 'dp', 'csv'), (2, 'ep', 'csv'), (3, 'ep', 'csv'),
                                            (2, 'dp', 'parquet'), (2, 'ep', 'parquet')])
def test_workers_over_shards_train_and_evaluate_like_one_process_over_the_file(tmp_path, world, mode, fmt):
  if fmt == 'parquet':
    pytest.importorskip('pyarrow')
  _prepare(str(tmp_path), world, fmt)
  ret = mp.Manager().dict()
  _spawn(_equivalence_worker, world, (_free_port(), ret, world, str(tmp_path), mode, fmt))
  assert len(ret) == world and len(set(v[0] for v in ret.values())) == 1, dict(ret)


def _uneven_worker(rank, port, ret, world, tmp, mode, B, n_lines):
  from test_dp_clip_gloo import _setup
  dev = _setup(rank, port, world, False)
  from easyrec_b200.estimator import EasyRecEstimator
  ep = mode == 'ep'
  est = EasyRecEstimator(TRAIN_CFG % (_ep_flag(mode), B), device=dev, seed=3, world_size=world, rank=rank)
  ref = EasyRecEstimator(TRAIN_CFG % (b'', B), device=dev, seed=3)
  _copy_weights(ref, est, rank, world, ep)
  cfg = est._pipeline_config
  path = os.path.join(tmp, 'uneven.csv')
  # evaluation covers every worker's full batches: the union of them, evaluated by one process
  ev = est.evaluate(lambda: readers.make_input(cfg, est.input_layer, path, rank, world))
  ev1 = ref.evaluate(lambda: readers.make_input(ref._pipeline_config, ref.input_layer, os.path.join(tmp, 'union.csv')))
  dicts = _gather(ev)
  assert all(d == dicts[0] for d in dicts), dicts
  _close(ev, ev1)
  n_pred = sum(1 for _ in est.predict(lambda: readers.make_input(cfg, est.input_layer, path, rank, world)))
  # training: every worker makes the steps the shortest shard allows
  est.train(lambda: readers.make_input(cfg, est.input_layer, path, rank, world))
  ret[rank] = (est.global_step, n_pred)
  import torch.distributed as dist
  dist.destroy_process_group()


@pytest.mark.timeout(900)
@pytest.mark.parametrize('world,mode', [(2, 'dp'), (2, 'ep'), (3, 'dp'), (3, 'ep')])
def test_uneven_shards_stop_training_together_and_evaluate_every_batch(tmp_path, world, mode):
  B, k = 8, 4
  n_lines = world * k * B - (world - 1)       # worker 0: k full batches, the others k - 1
  lines = _train_lines(n_lines, 21)
  _write(str(tmp_path / 'uneven.csv'), lines)
  own = [lines[r::world] for r in range(world)]
  _write(str(tmp_path / 'union.csv'), sum((o[:len(o) // B * B] for o in own), []))
  ret = mp.Manager().dict()
  _spawn(_uneven_worker, world, (_free_port(), ret, world, str(tmp_path), mode, B, n_lines), timeout=420)
  assert sorted(ret.keys()) == list(range(world))
  assert all(ret[r][0] == k - 1 for r in range(world)), dict(ret)
  assert [ret[r][1] for r in range(world)] == [k] + [k - 1] * (world - 1), dict(ret)
