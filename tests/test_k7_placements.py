"""K7's shared bucket placements (embedding.Placements): one placement per (rows tensor, n_rows, placement mode), so a
table reuses only a placement it would have made itself.  The rule object on its own, then a Wide&Deep config whose wide
dim-1 group is listed before a deep dim-10 group over the same features (the two placement modes on one row plan),
trained on the CPU over gloo with the kernel doubles: data parallel against one process on the concatenated batch, and
row-sharded against replicated data parallel.  The embedding_bwd double refuses a reuse across modes as
er_embedding_bwd_reuse_sort does."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from easyrec_b200 import embedding as E, kernels as K

HERE = os.path.dirname(os.path.abspath(__file__))

# (wide before deep: the dim-1 arena is looked up, and updated, first)
CFG = b'''
train_config { optimizer_config { adagrad_optimizer { learning_rate { constant_learning_rate { learning_rate: 0.1 } } } } }
data_config { batch_size: %d input_type: CSVInput separator: "," label_fields: "label"
  input_fields { input_name: "label" input_type: FLOAT } input_fields { input_name: "x" input_type: FLOAT }
  input_fields { input_name: "a" input_type: INT64 } input_fields { input_name: "b" input_type: INT64 }
  input_fields { input_name: "c" input_type: INT64 } }
feature_config {
  features { input_names: "x" feature_type: RawFeature embedding_dim: 10 min_val: 0.0 max_val: 4.0 }
  features { input_names: "a" feature_type: IdFeature embedding_dim: 10 hash_bucket_size: 1001 embedding_name: "shared" }
  features { input_names: "b" feature_type: IdFeature embedding_dim: 10 hash_bucket_size: 1001 embedding_name: "shared" }
  features { input_names: "c" feature_type: IdFeature embedding_dim: 10 num_buckets: 37 } }
model_config { model_class: "WideAndDeep"
  feature_groups { group_name: "wide" feature_names: ["x", "a", "b", "c"] wide_deep: WIDE }
  feature_groups { group_name: "deep" feature_names: ["x", "a", "b", "c"] wide_deep: DEEP }
  wide_and_deep { dnn { hidden_units: [16] use_bn: false } final_dnn { hidden_units: [8] use_bn: false }
                  l2_regularization: 1e-5 } }
'''


def test_one_placement_per_rows_n_rows_and_mode(monkeypatch):
  launched = []
  monkeypatch.setattr(K, 'embedding_bwd_presort', lambda rows, n_rows, dim, ws, *a, **k: launched.append((dim, ws)))
  p = E.Placements()
  rows, other_rows = torch.zeros(4, dtype=torch.int64), torch.zeros(4, dtype=torch.int64)
  ws = {d: 'ws%d' % d for d in (1, 4, 10, 16, 64)}
  # presort: one launch per key; dims 16 and 1 share the warp mode, 10 and 64 the CTA mode
  for d in (16, 1, 10, 64):
    p.presort(rows, 100, d, ws[d], None, 3)
  p.presort(rows, 200, 4, ws[4], None, 3)                 # another n_rows: a placement of its own
  assert launched == [(16, 'ws16'), (10, 'ws10'), (4, 'ws4')]
  assert p.sorted_from(rows, 100, 1, ws[1]) == ('ws16', 16)
  assert p.sorted_from(rows, 100, 16, ws[16]) == ('ws16', 16)
  assert p.sorted_from(rows, 100, 64, ws[64]) == ('ws10', 10)
  assert p.sorted_from(rows, 200, 16, ws[16]) == ('ws4', 4)
  # without a presort the first update of a key places (None) and the later ones of its mode reuse it
  assert p.sorted_from(other_rows, 100, 10, 'own10') is None
  assert p.sorted_from(other_rows, 100, 1, 'own1') is None
  assert p.sorted_from(other_rows, 100, 64, 'own64') == ('own10', 10)
  assert p.sorted_from(other_rows, 100, 16, 'own16') == ('own1', 1)
  assert p.sorted_from(other_rows, 300, 16, 'own16b') is None
  p.clear()
  assert p.sorted_from(rows, 100, 1, ws[1]) is None
  p.presort(rows, 100, 16, ws[16], None, 3)               # (the key was placed by the update above: no launch)
  p.presort(rows, 100, 10, ws[10], None, 3)
  assert launched[3:] == [(10, 'ws10')]


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _cat_batches(parts):
  """per-rank batches -> the concatenated batch (sparse_fea is feature-major: [n_id, B] per rank)"""
  n_id = parts[0][0]['sparse_fea'].numel() // parts[0][1].numel()
  ids = torch.cat([f['sparse_fea'].view(n_id, -1) for f, _ in parts], dim=1).reshape(-1)
  return ({'sparse_fea': ids, 'dense_fea': torch.cat([f['dense_fea'] for f, _ in parts])},
          torch.cat([l for _, l in parts]))


def _dp_worker(rank, port, ret, world):
  sys.path.insert(0, HERE)
  from test_dp_clip_gloo import _setup
  import ep_helpers
  _setup(rank, port, world, False)
  from easyrec_b200.estimator import EasyRecEstimator
  B, steps = 16, 3
  dp = EasyRecEstimator(CFG % B, device='cpu', seed=3, world_size=world, rank=rank, embedding_parallel=False)
  one = EasyRecEstimator(CFG % (B * world), device='cpu', seed=3)     # the same model on the concatenated batch
  assert list(dp.input_layer.arenas) == [1, 10]
  for d, a in dp.input_layer.arenas.items():
    one.input_layer.arenas[d].storage.copy_(a.storage)
  one.model.load_state_dict(dp.model.state_dict())
  one.trainer.dense_opt.flat_p.copy_(dp.trainer.dense_opt.flat_p)
  for step in range(steps):
    parts = [ep_helpers.batch(B, r, step) for r in range(world)]
    dp.trainer.train_step(*parts[rank])
    one.trainer.train_step(*_cat_batches(parts))
  worst = max(float((a.storage - one.input_layer.arenas[d].storage).abs().max())
              for d, a in dp.input_layer.arenas.items())
  dworst = float((dp.trainer.dense_opt.flat_p - one.trainer.dense_opt.flat_p).abs().max())
  ret[rank] = (worst, dworst, float(sum(a.storage.double().sum() for a in dp.input_layer.arenas.values())))
  dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_data_parallel_over_both_placement_modes_equals_one_process_on_the_concatenated_batch():
  world = 2
  ret = mp.Manager().dict()
  mp.spawn(_dp_worker, args=(_free_port(), ret, world), nprocs=world, join=True)
  assert len(ret) == world
  for worst, dworst, _ in ret.values():
    assert worst < 2e-6 and dworst < 2e-6, dict(ret)          # tables (weights and accumulators) and dense parameters
  assert len(set(v[2] for v in ret.values())) == 1, dict(ret)   # replicas bit-identical


def _ep_worker(rank, port, ret, world):
  sys.path.insert(0, HERE)
  from test_dp_clip_gloo import _setup
  import ep_helpers
  _setup(rank, port, world, False)
  from easyrec_b200.estimator import EasyRecEstimator

  def make(cfg, ep):
    return EasyRecEstimator(cfg, device='cpu', seed=5, world_size=world, rank=rank, embedding_parallel=ep)
  cfg = (CFG % 64).replace(b'train_config { ', b'train_config { train_distribute: EmbeddingParallelStrategy ')
  ret[rank] = ep_helpers.run(make, 'cpu', rank, world, cfg=cfg)
  dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_row_sharded_over_both_placement_modes_equals_replicated_data_parallel_gloo():
  world = 2
  ret = mp.Manager().dict()
  mp.spawn(_ep_worker, args=(_free_port(), ret, world), nprocs=world, join=True)
  assert len(ret) == world
