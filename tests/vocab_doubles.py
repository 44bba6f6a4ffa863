"""Doubles of K1's vocabulary mode (ER_BUCKET_VOCAB: er_bucketize_vocab, er_bucketize_seq_vocab) and of the vocabulary
index build for the host tests (TEST INFRASTRUCTURE).  They restate the rule as a dict lookup - the key of a lookup ->
the position of its entry, 0 when no entry has it, -1 for a key < 0 - turn the vocabulary slots into identity slots over
len(vocabulary) rows, which pass those positions through, and hand the call to whatever K1 double is installed.  Install
them after host_doubles.install_all (and seq_doubles.install)."""
import numpy as np
import torch

from easyrec_b200 import _lib, kernels as K
from host_doubles import _slots


def vocab_ids(ids, sl, seg_of, vocabs):
  """(ids, slots) with the vocabulary lookups restated; seg_of: the segment of each lookup"""
  if vocabs is None:
    return ids, sl
  sl = sl.copy()
  slot_of = np.searchsorted(sl['seg_begin'], seg_of, side='right') - 1
  out = ids.copy()
  for i, v in enumerate(vocabs.per_slot):
    if int(sl[i]['bucket_mode']) != _lib.BUCKET_VOCAB:
      continue
    pos = {int(k): p for p, k in enumerate(v.keys)}
    sel = np.nonzero(slot_of == i)[0]
    out[sel] = [pos.get(int(k), 0) if k >= 0 else -1 for k in ids[sel]]
    sl[i]['bucket_mode'] = _lib.BUCKET_IDENTITY
  return out, sl


def install(patch=setattr):
  inner, inner_seq = K.bucketize, K.bucketize_seq

  def bucketize(ids, slots_dev, n_slots, n_seg, seg_ids=None, row_ptr=None, rows=None, owner=None, vocabs=None, **kw):
    if vocabs is None:
      return inner(ids, slots_dev, n_slots, n_seg, seg_ids=seg_ids, row_ptr=row_ptr, rows=rows, owner=owner, **kw)
    n = ids.numel()
    seg_of = np.arange(n) if row_ptr is None else seg_ids.numpy()[:n].astype(np.int64)
    if row_ptr is not None:
      seg_of = np.where(np.arange(n) < int(row_ptr[-1]), seg_of, 0)
    vids, sl = vocab_ids(ids.numpy(), _slots(slots_dev), seg_of, vocabs)
    return inner(torch.from_numpy(vids), K.slots_to_device(sl, 'cpu'), n_slots, n_seg, seg_ids=seg_ids, row_ptr=row_ptr,
                 rows=rows, owner=owner, **kw)

  def bucketize_seq(ids, lens, batch, seq_len, slots_dev, n_slots, rows=None, owner=None, vocabs=None):
    vids, sl = vocab_ids(ids.numpy(), _slots(slots_dev), np.arange(ids.numel()), vocabs)
    return inner_seq(torch.from_numpy(vids), lens, batch, seq_len, K.slots_to_device(sl, 'cpu'), n_slots, rows=rows,
                     owner=owner)

  def vocab_index(keys, device):
    # the doubles read Vocab.keys; the index itself is never probed on the host
    empty = torch.full((16,), _lib.KV_EMPTY, dtype=torch.int64, device=device)
    return empty, empty.clone()
  patch(K, 'bucketize', bucketize)
  patch(K, 'bucketize_seq', bucketize_seq)
  patch(K, 'vocab_index', vocab_index)
