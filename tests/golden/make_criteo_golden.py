"""Golden batches from the reference's own CriteoInput reader, run unmodified.

input/criteo_binary_reader.py imports only the standard library and numpy, so it is loaded by file path (the `easy_rec`
package itself cannot be imported without TensorFlow) and `BinaryDataset` reads the parts written by `write_parts`
at world sizes 1-4, drop_last=False, batch size B.  Sample i of a case holds label i, dense values i + j / 16 and
category values 32 i + c, the last one 2^31 + i (uint32 values past the int32 range).  The parts of a case are equal in
size: the reference's walk to a rank's first file is only right then (DESIGN.md section 4).

  python tests/golden/make_criteo_golden.py <EasyRec checkout>/easy_rec/python
    ->  tests/golden/reference_criteo_batches.json, replayed by tests/test_criteo_binary_host.py"""
import importlib.util
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'reference_criteo_batches.json')
B = 8
# name -> samples per part; 100 and 102 samples: total % N is 0 and non-zero among N = 1..4
CASES = {'4x25': [25] * 4, '3x34': [34] * 3}
WORLDS = (1, 2, 3, 4)


def samples(lo, hi):
  """(label int32 [n], dense float32 [n, 13], category uint32 [n, 26]) of samples lo..hi-1"""
  i = np.arange(lo, hi, dtype=np.int64)
  label = i.astype(np.int32)
  dense = (i[:, None] + np.arange(13)[None, :] / 16.0).astype(np.float32)
  cat = (32 * i[:, None] + np.arange(26)[None, :]).astype(np.uint32)
  cat[:, 25] = (np.uint64(2**31) + i.astype(np.uint64)).astype(np.uint32)
  return label, dense, cat


def write_parts(dirname, sizes):
  """part p -> <dirname>/part<p>_{label,dense,category}.bin; returns the (label, dense, category) path lists"""
  out = ([], [], [])
  lo = 0
  for p, n in enumerate(sizes):
    arrs = samples(lo, lo + n)
    for kind, a, lst in zip(('label', 'dense', 'category'), arrs, out):
      path = os.path.join(dirname, 'part%d_%s.bin' % (p, kind))
      a.tofile(path)
      lst.append(path)
    lo += n
  return out


def _batch(ds, k):
  """batch k of a BinaryDataset, or the error reading it raises: a last partial batch that ends where a file ends goes
  on reading a file the dataset never opened"""
  try:
    dense, cat, lab = ds[k]
  except TypeError as e:
    return {'error': '%s: %s' % (type(e).__name__, e)}
  return {'label': lab.reshape(-1).tolist(), 'dense': dense.reshape(-1).tolist(), 'category': cat.reshape(-1).tolist()}


def main(ref):
  spec = importlib.util.spec_from_file_location('criteo_binary_reader', os.path.join(ref, 'input', 'criteo_binary_reader.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  gold = {'batch_size': B, 'cases': {}}
  for name, sizes in CASES.items():
    with tempfile.TemporaryDirectory() as d:
      labels, denses, cats = write_parts(d, sizes)
      worlds = {}
      for n in WORLDS:
        ranks = []
        for r in range(n):
          ds = mod.BinaryDataset(labels, denses, cats, batch_size=B, drop_last=False, prefetch=1, global_rank=r,
                                 global_size=n)
          ranks.append([_batch(ds, k) for k in range(len(ds))])
        worlds[str(n)] = ranks
      gold['cases'][name] = {'sizes': sizes, 'worlds': worlds}
  with open(OUT, 'w') as f:
    json.dump(gold, f, separators=(',', ':'))
  print('wrote', OUT)


if __name__ == '__main__':
  main(sys.argv[1])
