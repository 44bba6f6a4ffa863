"""CPU: key-value embedding tables (ev_params) through InputLayer, the builder and the checkpoints, with the sparse
kernels replaced by the oracle's doubles and the key-value kernels by the dict-based doubles of kv_doubles.

Every row is checked per KEY against a float64 numpy restatement built from the keys alone: initial values from
(seed, table, key), then the optimizer's row rule on the summed gradient of the key's lookups.  Row numbers are never
compared: the kernels hand them out in claim order, which is not deterministic."""
import collections
import math
import os

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, builder, checkpoint, embedding as E, input_layer as IL, kernels as K
from easyrec_b200.config import config_util

import host_doubles  # noqa: E402  (tests/ is on sys.path under pytest's rootdir conftest)
import kv_doubles

B = 8
DIM = 4
SEED = 7


@pytest.fixture
def doubles(monkeypatch):
  host_doubles.install_sparse(monkeypatch.setattr)
  kv_doubles.install(monkeypatch.setattr)


def make_layer(opt, device='cpu', capacity=64, item_buckets=1000, adagrad_init=0.1):
  feats = [IL.id_feature('user', DIM, hash_bucket_size=50),
           IL.id_feature('item', DIM, hash_bucket_size=item_buckets, kv_capacity=capacity),
           IL.multi_feature('tags', 'tag', DIM, num_buckets=30, kv_capacity=capacity)]
  groups = collections.OrderedDict(all=dict(features=['user', 'item', 'tags']))
  return IL.InputLayer(feats, groups, B, device, embedding_optimizer=opt, generator=torch.Generator(device).manual_seed(1),
                       adagrad_init=adagrad_init, kv_seed=SEED, max_tag_lookups=4 * B)


def make_batch(rng, device='cpu', item_pool=12):
  users = rng.integers(0, 100, B)
  items = rng.integers(0, item_pool, B) * 1000003
  lens = rng.integers(0, 4, B).astype(np.int32)
  tags = rng.integers(0, 6, int(lens.sum()))
  feats = {'sparse_fea': torch.tensor(np.concatenate([users, items]), dtype=torch.int64, device=device),
           'tag_fea': {'tags': (torch.tensor(tags, dtype=torch.int64, device=device),
                                torch.tensor(lens, device=device), None)}}
  return feats, dict(items=items, tags=tags, lens=lens)


def train_step(il, feats, R, lr, t, **kw):
  concat, _ = il.lookup(feats)['all']
  (concat * R).sum().backward()
  il.set_optimizer_step(lr, t, **kw)
  il.backward_update()


def item_key(v):
  return _lib.fingerprint64(str(int(v))) % _lib.KV_BUCKETS


def table_seed(table):
  return E._mix64(SEED ^ _lib.fingerprint64(table))


def key_grads(batch, R):
  """{table: {key: summed float64 gradient}} of one step"""
  R = R.double().cpu().numpy()
  g = {'item_embedding': collections.defaultdict(lambda: np.zeros(DIM)),
       'tags_embedding': collections.defaultdict(lambda: np.zeros(DIM))}
  for b, v in enumerate(batch['items']):
    g['item_embedding'][item_key(v)] += R[b, DIM:2 * DIM]
  off = 0
  for b, n in enumerate(batch['lens']):
    for v in batch['tags'][off:off + n]:
      g['tags_embedding'][int(v)] += R[b, 2 * DIM:3 * DIM]
    off += n
  return g


def per_key(il, table):
  """{key: (row, state0, state1)} of a key-value table, as float64"""
  a = il.arenas[(DIM, table)]
  keys, rows = a.kv.items()
  out = {}
  for k, r in zip(keys.tolist(), rows.tolist()):
    st = [None if s is None else s[r].double().cpu().numpy() for s in (a.state0, a.state1)]
    out[k] = (a.weight[r].double().cpu().numpy(), st[0], st[1])
  return out


def restate(steps, kind, lr=0.05, b1=0.9, b2=0.999, eps=1e-8, acc0=0.1, grads_of=key_grads):
  """float64: {table: {key: [w, s0, s1]}} after `steps` [(batch, R)].  kind: 'sgd', 'adagrad', 'momentum' (momentum b1)
  or 'adam' / 'lazy_adam' (both the touched-row rule on a key-value table).  grads_of(batch, R) -> {table: {key: summed
  gradient}}: every key a step looked up, a zero gradient included"""
  ref = {}
  for t, (batch, R) in enumerate(steps):
    for table, grads in grads_of(batch, R).items():
      for k, g in grads.items():
        if k not in ref.setdefault(table, {}):
          dim = g.size
          w0 = kv_doubles.init_values(table_seed(table), [k], dim, 0.01 / math.sqrt(dim))[0].astype(np.float64)
          ref[table][k] = [w0, np.full(dim, acc0 if kind == 'adagrad' else 0.0), np.zeros(dim)]
        w, s0, s1 = ref[table][k]
        if kind == 'sgd':
          w = w - lr * g
        elif kind == 'momentum':
          s0 = b1 * s0 + g
          w = w - lr * s0
        elif kind == 'adagrad':
          s0 = s0 + g * g
          w = w - lr * g / np.sqrt(s0)
        else:
          s0 = b1 * s0 + (1 - b1) * g
          s1 = b2 * s1 + (1 - b2) * g * g
          lr_t = lr * math.sqrt(1 - b2 ** (t + 1)) / (1 - b1 ** (t + 1))
          w = w - lr_t * s0 / (np.sqrt(s1) + eps)
        ref[table][k] = [w, s0, s1]
  return ref


@pytest.mark.parametrize('kind,opt', [('adagrad', _lib.OPT_ADAGRAD), ('lazy_adam', _lib.OPT_LAZY_ADAM),
                                      ('adam', _lib.OPT_ADAM_ROWS), ('sgd', _lib.OPT_SGD),
                                      ('momentum', _lib.OPT_MOMENTUM)])
def test_three_steps_match_a_float64_restatement_per_key(doubles, kind, opt):
  import test_gpu_kv_f64 as G
  il, steps = G.train_model(opt, 'cpu', prune=False)
  ref = restate(steps, kind, grads_of=G.model_grads)
  G.check_per_key(il, ref, kind, 1e-6)
  if kind == 'adam':
    # adam_optimizer on a key-value table is the touched-row rule: no dense sweep, keys a step did not see stay put
    assert il.arenas[(DIM, 'item_embedding')].touched is None
    untouched = set(ref['item_embedding']) - set(G.model_grads(*steps[-1])['item_embedding'])
    assert untouched, 'the batches should leave some item key out of the last step'


def test_ids_that_collide_in_a_static_table_get_their_own_rows(doubles):
  nb = 3
  a, b = next((i, j) for i in range(50) for j in range(i + 1, 50)
              if _lib.fingerprint64(str(i)) % nb == _lib.fingerprint64(str(j)) % nb)
  il = make_layer(_lib.OPT_ADAGRAD, item_buckets=nb)
  ids = np.concatenate([np.zeros(B, np.int64), np.array([a, b] * (B // 2), np.int64)])
  feats = {'sparse_fea': torch.tensor(ids), 'tag_fea': {'tags': (torch.zeros(0, dtype=torch.int64),
                                                                  torch.zeros(B, dtype=torch.int32), None)}}
  R = torch.zeros(B, 3 * DIM)
  R[0::2, DIM:2 * DIM] = 1.0     # only the lookups of `a` carry a gradient
  train_step(il, feats, R, 0.1, 0)
  got = per_key(il, 'item_embedding')
  ka, kb = item_key(a), item_key(b)
  assert set(got) == {ka, kb}
  std = 0.01 / math.sqrt(DIM)
  init = kv_doubles.init_values(table_seed('item_embedding'), [ka, kb], DIM, std)
  assert not np.array_equal(init[0], init[1])
  np.testing.assert_array_equal(got[kb][0], init[1])             # b: trained with a zero gradient
  assert np.abs(got[ka][0] - init[0]).min() > 1e-3               # a: moved by the step
  np.testing.assert_allclose(got[ka][1], 0.1 + (B // 2) ** 2, rtol=1e-6)


def test_evaluation_reads_zero_rows_for_unseen_keys_and_inserts_nothing(doubles):
  il = make_layer(_lib.OPT_ADAGRAD)
  rng = np.random.default_rng(5)
  feats, _ = make_batch(rng, item_pool=4)
  train_step(il, feats, torch.ones(B, 3 * DIM), 0.05, 0)
  sizes = il.kv_sizes()
  ids = feats['sparse_fea'].clone()
  ids[B:B + 2] = torch.tensor([987654321, 987654322])                     # unseen item ids
  seen = per_key(il, 'item_embedding')
  with torch.no_grad():
    concat, _ = il.lookup({'sparse_fea': ids, 'tag_fea': {'tags': (torch.tensor([29, 28]), torch.tensor(
        [2] + [0] * (B - 1), dtype=torch.int32), None)}})['all']
  il.discard_pending()
  assert il.kv_sizes() == sizes
  assert torch.all(concat[:2, DIM:2 * DIM] == 0) and torch.all(concat[0, 2 * DIM:] == 0)
  for b in range(2, B):
    np.testing.assert_array_equal(concat[b, DIM:2 * DIM].double().numpy(), seen[item_key(int(ids[B + b]))][0])


def test_overflowing_max_capacity_raises_naming_the_table(doubles):
  il = make_layer(_lib.OPT_ADAGRAD, capacity=4)
  ids = np.concatenate([np.zeros(B, np.int64), np.arange(B, dtype=np.int64)])
  feats = {'sparse_fea': torch.tensor(ids), 'tag_fea': {'tags': (torch.zeros(0, dtype=torch.int64),
                                                                  torch.zeros(B, dtype=torch.int32), None)}}
  train_step(il, feats, torch.ones(B, 3 * DIM), 0.05, 0)
  assert il.kv_sizes()['item_embedding'] == 4
  with pytest.raises(_lib.ErError, match='item_embedding.*max_capacity 4'):
    il.check_kv()
  with pytest.raises(_lib.ErError, match='item_embedding'):
    il.check_exchange()


CFG = '''
train_config { %s optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.1 } } } } }
data_config { batch_size: 8 input_type: CSVInput label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "uid" input_type: INT64 }
  input_fields { input_name: "iid" input_type: INT64 } input_fields { input_name: "tags" input_type: STRING } }
feature_config {
  features { input_names: "uid" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 50 }
  features { input_names: "iid" feature_type: IdFeature embedding_dim: 4 hash_bucket_size: 100 %s }
  features { input_names: "tags" feature_type: TagFeature embedding_dim: 4 num_buckets: 20 separator: "|" %s } }
model_config { model_class: "DeepFM" %s
  feature_groups { group_name: "deep" feature_names: ["uid", "iid", "tags"] wide_deep: DEEP }
  feature_groups { group_name: "wide" feature_names: ["uid", "iid"] wide_deep: WIDE }
  deepfm { dnn { hidden_units: [8] } final_dnn { hidden_units: [4] } } }
'''


def config(item_ev='', tag_ev='', model_ev='', train=''):
  return config_util.get_configs_from_pipeline_file((CFG % (train, item_ev, tag_ev, model_ev)).encode())


def build(cfg, **kw):
  os.environ['ER_PLAN_ONLY'] = '1'
  try:
    return builder.build_model(cfg, 8, 'cpu', cpu_generator=torch.Generator().manual_seed(0), **kw)
  finally:
    del os.environ['ER_PLAN_ONLY']


def test_builder_plans_key_value_tables_from_feature_and_model_ev_params():
  il, _, _ = build(config(item_ev='ev_params { max_capacity: 1000 }'))
  assert {k for k in il.arenas if isinstance(k, tuple)} == {(4, 'iid_embedding'), (1, 'iid_embedding_wide')}
  assert il.features['iid'].num_buckets == _lib.KV_BUCKETS and il.features['iid'].kv_capacity == 1000
  assert il.arenas[(4, 'iid_embedding')].n_rows == 1001                    # the pool and the zero row
  assert il.features['uid'].kv_capacity == 0 and il.features['uid'].num_buckets == 50
  # the model's ev_params covers every column; a feature's own overrides it
  il, _, _ = build(config(tag_ev='ev_params { max_capacity: 30 }', model_ev='ev_params { max_capacity: 500 }'))
  assert il.features['uid'].kv_capacity == 500 and il.features['tags'].kv_capacity == 30
  assert il.features['tags'].num_buckets == _lib.KV_BUCKETS and il.features['tags'].bucket_mode == _lib.BUCKET_IDENTITY


@pytest.mark.parametrize('ev,field', [('filter_freq: 2', 'filter_freq'), ('steps_to_live: 10', 'steps_to_live'),
                                      ('use_cache: true', 'use_cache'), ('max_capacity: 0', 'max_capacity')])
@pytest.mark.parametrize('where', ['feature', 'model'])
def test_ev_params_that_cannot_be_pinned_are_refused_by_name(ev, field, where):
  text = 'ev_params { %s }' % ev
  cfg = config(item_ev=text) if where == 'feature' else config(model_ev=text)
  with pytest.raises(NotImplementedError, match='ev_params.%s' % field):
    build(cfg)


def test_key_value_tables_on_data_parallel_ranks_are_refused_by_name():
  cfg = config(item_ev='ev_params { max_capacity: 100 }')
  with pytest.raises(NotImplementedError, match='ev_params.*data-parallel.*EmbeddingParallelStrategy'):
    build(cfg, world=2, rank=0)
  il, _, _ = build(cfg, world=2, rank=1, shard_tables=True)      # row-sharded: built
  a = il.arenas[(4, 'iid_embedding')]
  assert (a.shard_n, a.shard_rank, a.n_rows, a.kv.init_stddev, a.kv.init_truncated) == (2, 1, 101, 0.0025, False)


def test_model_ev_params_leave_numeric_columns_without_a_table_alone():
  text = CFG.replace('input_fields { input_name: "tags" input_type: STRING }',
                     'input_fields { input_name: "tags" input_type: STRING } '
                     'input_fields { input_name: "x" input_type: FLOAT }').replace(
      'separator: "|" %s } }', 'separator: "|" %s }\n features { input_names: "x" feature_type: RawFeature } }')
  cfg = config_util.get_configs_from_pipeline_file((text % ('', '', '', 'ev_params { max_capacity: 50 }')).encode())
  il, _, _ = build(cfg)
  assert il.features['x'].kv_capacity == 0 and il.features['iid'].kv_capacity == 50


def test_ev_params_on_a_column_that_takes_no_key_value_table_is_refused_by_name():
  text = CFG.replace('input_fields { input_name: "tags" input_type: STRING }',
                     'input_fields { input_name: "tags" input_type: STRING } '
                     'input_fields { input_name: "x" input_type: FLOAT }').replace(
      'separator: "|" %s } }', 'separator: "|" %s }\n features { input_names: "x" feature_type: RawFeature '
      'embedding_dim: 4 boundaries: [0.5] ev_params { max_capacity: 10 } } }')
  cfg = config_util.get_configs_from_pipeline_file((text % ('', '', '', '')).encode())
  with pytest.raises(NotImplementedError, match='feature x: ev_params'):
    build(cfg)


def _trained(doubles_rng_seed=11):
  il = make_layer(_lib.OPT_ADAGRAD)
  rng = np.random.default_rng(doubles_rng_seed)
  for t in range(2):
    feats, _ = make_batch(rng)
    train_step(il, feats, torch.tensor(rng.normal(size=(B, 3 * DIM)), dtype=torch.float32), 0.05, t)
  return il


@pytest.mark.parametrize('world', [1, 2, 3])
def test_key_value_parts_have_the_reference_layout_and_reshard_by_key(doubles, tmp_path, world):
  il = _trained()
  a = il.arenas[(DIM, 'item_embedding')]
  ck = str(tmp_path / 'model.ckpt-2')
  files = checkpoint.save_kv_arena(a, ck)
  var = 'input_layer/item_embedding/embedding_weights:0'
  kp = '%s-embedding/embed-%s-part-0.key' % (ck, var.replace('/', '__'))
  assert kp in files and kp[:-4] + '.val' in files
  assert any(f.endswith('embedding_weights__Adagrad:0-part-0.val') for f in files)
  keys = np.fromfile(kp, np.int64)
  vals = np.fromfile(kp[:-4] + '.val', np.float32).reshape(-1, DIM)
  ref = per_key(il, 'item_embedding')
  assert sorted(keys.tolist()) == sorted(ref)
  for k, v in zip(keys.tolist(), vals):
    np.testing.assert_array_equal(v, ref[k][0].astype(np.float32))
  # restore on `world` ranks: rank r keeps exactly the keys with key % world == r, rows and slots per key
  seen = set()
  for r in range(world):
    arena = E.Arena(DIM, 'cpu', world, r)
    arena.add_table('item_embedding', 65)
    arena.kv = E.KvTable('item_embedding', arena, 64, SEED)
    arena.materialize(_lib.OPT_ADAGRAD, init_fn=lambda w: w.zero_())
    checkpoint.restore_kv_arena(arena, ck)
    k2, r2 = arena.kv.items()
    assert all(k % world == r for k in k2.tolist())
    seen |= set(k2.tolist())
    for k, row in zip(k2.tolist(), r2.tolist()):
      np.testing.assert_array_equal(arena.weight[row].double().numpy(), ref[k][0])
      np.testing.assert_array_equal(arena.state0[row].double().numpy(), ref[k][1])
    assert int(arena.kv.stats[0]) == k2.numel()
  assert seen == set(ref)
  # a stale part of a larger job is removed when rank 0 saves again
  open(kp.replace('part-0', 'part-5'), 'wb').close()
  open(kp.replace('part-0.key', 'part-5.val'), 'wb').close()
  checkpoint.save_kv_arena(a, ck)
  assert not os.path.exists(kp.replace('part-0', 'part-5'))


def test_restored_index_reads_the_same_rows(doubles):
  il = _trained()
  a = il.arenas[(DIM, 'item_embedding')]
  keys, rows = a.kv.items()
  il2 = make_layer(_lib.OPT_ADAGRAD)
  a2 = il2.arenas[(DIM, 'item_embedding')]
  a2.storage.copy_(a.storage)
  a2.kv.load(keys, rows)
  assert il2.kv_sizes()['item_embedding'] == keys.numel()
  probe = torch.cat([keys, torch.tensor([123456789])])
  out = torch.empty_like(probe)
  with torch.no_grad():
    a2.kv.lookup(probe, out, train=False)
  assert out[:-1].tolist() == rows.tolist() and int(out[-1]) == a2.kv.zero_row


def test_a_table_shared_by_static_and_key_value_features_is_refused():
  feats = [IL.id_feature('a', DIM, hash_bucket_size=50, embedding_name='t'),
           IL.id_feature('b', DIM, hash_bucket_size=50, embedding_name='t', kv_capacity=10)]
  with pytest.raises(ValueError, match='table t: read by features with different ev_params'):
    IL.InputLayer(feats, collections.OrderedDict(g=dict(features=['a', 'b'])), B, 'cpu')


# ---- the restatements of test_gpu_kv_f64 against the doubles --------------------------------------------------------------
@pytest.mark.parametrize('shard_n', [1, 3, 100])
@pytest.mark.parametrize('mode', [_lib.BUCKET_FARM_DECIMAL, _lib.BUCKET_MOD, _lib.BUCKET_IDENTITY])
def test_k1_kv_restatement_on_the_host_doubles(doubles, mode, shard_n):
  import test_gpu_kv_f64 as G
  ids = G.kv_edge_ids(np.random.default_rng(mode), 50)
  sl = G._k1_slots(mode, shard_n, ids.size, 0)[:1]      # one summed slot, a lookup per segment
  rows, owner = torch.empty(ids.size, dtype=torch.int64), torch.empty(ids.size, dtype=torch.int32)
  K.bucketize(torch.from_numpy(ids), K.slots_to_device(sl, 'cpu'), 1, ids.size, rows=rows, owner=owner)
  assert (rows.tolist(), owner.tolist()) == G.k1_kv_ref(ids, mode, shard_n)


@pytest.mark.parametrize('world,n', [(1, 31), (3, 257), (65, 257), (200, 31)])
def test_k8_checker_on_the_host_double(doubles, world, n):
  import test_gpu_kv_f64 as G
  rows, owner = G.k8_case(world, n, world + n)
  live = (rows >= 0) & (owner >= 0) & (owner < world)
  mx = int(np.bincount(np.unique(np.stack([rows[live], owner[live]], 1), axis=0)[:, 1], minlength=world).max())
  for cap in (mx - 1, mx):
    send, pos = torch.empty(world * cap, dtype=torch.int64), torch.empty(n, dtype=torch.int64)
    counts = torch.empty(world + 1, dtype=torch.int32)
    K.shard_group(torch.from_numpy(rows), torch.from_numpy(owner.astype(np.int32)), world, cap, send, pos, counts,
                    K.shard_group_workspace(n, 'cpu'))
    G.k8_check(rows, owner, world, cap, send.numpy(), pos.numpy(), counts.numpy())
  # and it refuses the old packing's answer: two pairs that pack to one integer under owner << 48 | row share a position
  if world >= 2:
    p = pos.numpy().copy()
    p[1], p[2] = p[0], p[0]      # k8_case puts (5 + 2^48, 0) at 0 and 1, (5, 1) at 2 and 3
    with pytest.raises(AssertionError):
      G.k8_check(rows, owner, world, mx, send.numpy(), p, counts.numpy())


def test_index_model_on_the_kv_doubles(doubles):
  import test_gpu_kv_f64 as G
  rng = np.random.default_rng(4)
  capacity, n_index = 40, 128
  keys = rng.permutation(np.concatenate([rng.integers(0, 2 ** 63 - 1, 50, dtype=np.int64)] * 2 + [[-1]])).tolist()
  ik, ir = torch.full((n_index,), _lib.KV_EMPTY, dtype=torch.int64), torch.full((n_index,), -1, dtype=torch.int64)
  stats = torch.zeros(2, dtype=torch.int64)
  rows = torch.empty(len(keys), dtype=torch.int64)
  w = torch.zeros(capacity + 1, DIM)
  K.kv_find_or_insert(ik, ir, capacity, stats, torch.tensor(keys), rows, w, None, None, 0.0, 5, 0.01)
  held = G.index_check(keys, rows.tolist(), ik, ir, stats, capacity, n_index)
  assert len(held) == 50 and stats.tolist() == [50, sum(1 for k, r in zip(keys, rows.tolist()) if k >= 0 and r < 0)]


@pytest.mark.parametrize('kv', [True, False], ids=['key_value', 'static'])
def test_sparse_norm_restatement_on_the_host_doubles(doubles, kv):
  import test_gpu_kv_f64 as G
  for got, want in G.norm_steps(kv, 'cpu'):
    assert abs(got - want) <= 1e-5 * want
