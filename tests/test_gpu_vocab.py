"""GPU: vocabulary columns on the kernels.  K1's ER_BUCKET_VOCAB mode (er_bucketize_vocab, er_bucketize_seq_vocab)
against a Python dict on single-valued, weighted CSR and padded-sequence slot plans, vocabularies of 1 to 10^6 entries
and shard_n 1, 2 and 8; a model with vocabulary features against the same model over identity columns fed TF's
positions, eager and graph-replayed; and a checkpoint round trip."""
import glob
import os

import numpy as np
import pytest
import torch

from easyrec_b200 import _lib, builder, embedding as E, kernels as K
from easyrec_b200.config import config_util
from easyrec_b200.input import readers
from easyrec_b200.trainer import Trainer

import test_vocab_host as V

pytestmark = pytest.mark.gpu
DEV = 'cuda'
NB_HASH, NB_ID = 1000, 50


def _vocab_keys(rng, n):
  keys = np.unique(rng.integers(0, 2**63 - 1, int(n * 1.05) + 8, dtype=np.int64))
  return rng.permutation(keys)[:n]


def _ids(rng, keys, n):
  """hits, misses, -1 and other negatives of one vocabulary"""
  kind = rng.integers(0, 10, n)
  hits = keys[rng.integers(0, keys.size, n)]
  miss = rng.integers(0, 2**63 - 1, n, dtype=np.int64)
  miss = np.where(np.isin(miss, keys), -1, miss)
  return np.where(kind < 5, hits, np.where(kind < 8, miss, np.where(kind < 9, -1, -rng.integers(2, 2**40, n))))


def _plan(sizes, shard_n, n_seg, combiners):
  """slots vocab A, hashed, vocab B, identity - each with its own row offset"""
  recs, off = [], 3
  for i, (mode, nb) in enumerate(((_lib.BUCKET_VOCAB, sizes[0]), (_lib.BUCKET_FARM_DECIMAL, NB_HASH),
                                  (_lib.BUCKET_VOCAB, sizes[1]), (_lib.BUCKET_IDENTITY, NB_ID))):
    recs.append(dict(num_buckets=nb, row_offset=off, seg_begin=i * n_seg, n_seg=n_seg, bucket_mode=mode,
                     combiner=combiners[i], shard_n=shard_n))
    off += (nb + shard_n - 1) // shard_n
  return K.make_slots(recs)


def _expect_vocab(ids, pos_of, offset, shard_n, drop_w):
  """the dict's rows and owners of one vocabulary slot's lookups"""
  rows, owner = np.empty(ids.size, np.int64), np.empty(ids.size, np.int32)
  for j, v in enumerate(ids.tolist()):
    if v < 0 or drop_w[j]:
      rows[j], owner[j] = -1, -1
      continue
    p = pos_of.get(v, 0)
    rows[j], owner[j] = offset + p // shard_n, p % shard_n
  return rows, owner


SIZES = [(1, 1), (7, 1000), (1000, 3), (1000000, 50000)]


@pytest.mark.parametrize('shard_n', [1, 2, 8])
@pytest.mark.parametrize('sizes', SIZES, ids=['%dx%d' % s for s in SIZES])
@pytest.mark.parametrize('layout', ['single', 'csr', 'seq'])
def test_k1_vocabulary_lookups_are_the_dicts_rows_bit_for_bit(layout, sizes, shard_n):
  rng = np.random.default_rng(sizes[0] * 31 + sizes[1] + shard_n)
  vk = [_vocab_keys(rng, n) for n in sizes]
  vocabs = [E.Vocab('a', vk[0], DEV), None, E.Vocab('b', vk[1], DEV), None]
  Bn, Tn = 512, 5
  n_seg = Bn * Tn if layout == 'seq' else Bn
  mean, sm = _lib.COMBINER_MEAN, _lib.COMBINER_SUM
  sl = _plan(sizes, shard_n, n_seg, [sm, mean, mean, sm] if layout == 'csr' else [sm] * 4)
  plan = K.vocab_plan(sl, vocabs, DEV)
  slots = K.slots_to_device(sl, DEV)
  # lookups per segment, and the slot of each lookup
  lens = rng.integers(0, 5, 4 * n_seg).astype(np.int32) if layout == 'csr' else np.ones(4 * n_seg, np.int32)
  slot_of = np.repeat(np.repeat(np.arange(4), n_seg), lens)
  n = int(lens.sum())
  ids = np.empty(n, np.int64)
  for f in range(4):
    m = slot_of == f
    ids[m] = _ids(rng, vk[f // 2], int(m.sum())) if f in (0, 2) else rng.integers(-3, 2**40, int(m.sum()))
  w = rng.choice(np.array([1.5, 0.25, 0.0, -1.0, np.nan], np.float32), n)
  ids_d, w_d = torch.tensor(ids, device=DEV), torch.tensor(w, device=DEV)
  rows, owner = torch.full((n + 64,), -9, dtype=torch.int64, device=DEV), torch.full((n + 64,), -9, dtype=torch.int32, device=DEV)
  ref_rows, ref_owner = rows.clone(), owner.clone()
  seq_lens = None
  if layout == 'single':
    K.bucketize(ids_d, slots, 4, 4 * n_seg, rows=rows[:n], owner=owner[:n], vocabs=plan)
    K.bucketize(ids_d, slots, 4, 4 * n_seg, rows=ref_rows[:n], owner=ref_owner[:n])
    drop_w = np.zeros(n, bool)
  elif layout == 'csr':
    cap = n + 64
    ids_cap = torch.cat([ids_d, torch.full((64,), 5, dtype=torch.int64, device=DEV)])
    w_cap = torch.cat([w_d, torch.ones(64, device=DEV)])
    row_ptr, seg_ids = K.csr_from_lens(torch.tensor(lens, device=DEV), cap)
    K.bucketize(ids_cap, slots, 4, 4 * n_seg, seg_ids=seg_ids, row_ptr=row_ptr, rows=rows, owner=owner, weights=w_cap,
                vocabs=plan)
    K.bucketize(ids_cap, slots, 4, 4 * n_seg, seg_ids=seg_ids, row_ptr=row_ptr, rows=ref_rows, owner=ref_owner,
                weights=w_cap)
    drop_w = (slot_of == 2) & ~(w > 0)     # the mean vocabulary slot prunes weights that are not > 0
  else:
    seq_lens = rng.integers(-1, Tn + 2, 4 * Bn).astype(np.int32)
    lt = torch.tensor(seq_lens, device=DEV)
    K.bucketize_seq(ids_d, lt, Bn, Tn, slots, 4, rows=rows[:n], owner=owner[:n], vocabs=plan)
    K.bucketize_seq(ids_d, lt, Bn, Tn, slots, 4, rows=ref_rows[:n], owner=ref_owner[:n])
    drop_w = np.zeros(n, bool)
  got_r, got_o = rows.cpu().numpy(), owner.cpu().numpy()
  ref_r, ref_o = ref_rows.cpu().numpy(), ref_owner.cpu().numpy()
  assert (got_r[n:] == -9).all() and (got_o[n:] == -9).all()   # nothing past the lookups is written
  pad = np.zeros(n, bool)
  if seq_lens is not None:
    pad = np.tile(np.arange(Tn), 4 * Bn) >= np.repeat(np.clip(seq_lens, 0, Tn), Tn)
  for f in range(4):
    m = slot_of == f
    if f in (0, 2):
      er, eo = _expect_vocab(ids[m], {int(k): p for p, k in enumerate(vk[f // 2])}, int(sl[f]['row_offset']), shard_n,
                             drop_w[m])
      er[pad[m]], eo[pad[m]] = -1, -1
    else:   # every other slot: er_bucketize's rows and owners
      er, eo = ref_r[:n][m], ref_o[:n][m]
    assert np.array_equal(got_r[:n][m], er), (f, layout)
    assert np.array_equal(got_o[:n][m], eo), (f, layout)


def _train(tmp_path, form, graph, steps=4):
  vf = V.write_vocab_file(tmp_path / 'items.txt', V.I_VOCAB, trailing_newline=False)
  torch.manual_seed(0)
  cfg = config_util.get_configs_from_pipeline_file(V.config(vf, form))
  il, model, _ = builder.build_model(cfg, V.B, DEV, cpu_generator=torch.Generator().manual_seed(0))
  tr = Trainer(model, il, 'adagrad', lr=0.05, use_cuda_graph=graph)
  losses = []
  for step in range(steps):
    feats, labels = readers.to_device(*V.features(V.raw_batch(step, fixed_tags=graph), form), DEV)
    losses.append(tr.train_step(feats, labels)[0].item())
  torch.cuda.synchronize()
  return losses, V.tables_and_slots(il)


@pytest.mark.parametrize('graph', [False, True], ids=['eager', 'graph'])
def test_vocabulary_model_trains_bit_identically_to_its_identity_twin(tmp_path, graph):
  lv, tv = _train(tmp_path, 'vocab', graph)
  li, ti = _train(tmp_path, 'identity', graph)
  assert lv == li and lv[0] != lv[-1]
  assert tv == ti


def test_checkpoint_round_trip_of_a_vocabulary_model(tmp_path):
  from easyrec_b200.estimator import EasyRecEstimator
  vf = V.write_vocab_file(tmp_path / 'items.txt', V.I_VOCAB)
  batches = [readers.to_device(*V.features(V.raw_batch(s), 'vocab'), DEV) for s in range(4)]

  def make():
    return EasyRecEstimator(V.config(vf), device=DEV, seed=3)
  a = make()
  for feats, labels in batches[:2]:
    a.trainer.train_step(feats, labels)
  path = a.save(str(tmp_path / 'ck'), embedding_parts=True)
  # the u table is the identity column's len(vocabulary) rows
  part = glob.glob(os.path.join(path[:-3] + '-embedding', '*u_embedding*part-0.bin'))
  assert part and os.path.getsize(sorted(part)[0]) == len(V.U_VOCAB) * 4 * 4
  la = [a.trainer.train_step(f, l)[0].item() for f, l in batches[2:]]
  b = make()
  b.restore(path)
  lb = [b.trainer.train_step(f, l)[0].item() for f, l in batches[2:]]
  torch.cuda.synchronize()
  assert la == lb
  assert V.tables_and_slots(a.input_layer) == V.tables_and_slots(b.input_layer)
