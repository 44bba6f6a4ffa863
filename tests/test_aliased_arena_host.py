"""The arithmetic of tests/aliased_arena.py on the host: the chunk size, the reservation around base, the row choice of
test_gpu_large_offsets_f64.py and the disjointness of the rows' physical images."""
import numpy as np
import pytest

import aliased_arena as A

GRANS = [2 << 20, 512 << 10]
# (dim, row_stride) of test_gpu_large_offsets_f64.py: separate arrays and [w | state...] rows
LAYOUTS = sorted({(d, s) for d in (1, 3, 4, 6, 16, 64) for s in (d, 2 * d, 3 * d)})


@pytest.mark.parametrize('gran', GRANS)
@pytest.mark.parametrize('extent', [1, 16 * A.GIB, 48 * A.GIB, 2 ** 32 * 4 * 3, 800 * A.GIB])
def test_chunk_and_reservation(extent, gran):
  p = A.chunk_bytes(extent, gran)
  below, above, n_maps = A.layout(extent, p)
  assert p % gran == 0 and p % A.ODD == 0 and (p & (p - 1)) != 0, 'P = ODD * 2^k * granularity'
  for d in (2 ** 31 * 4, 2 ** 32 * 4, 2 ** 32, 2 ** 31):
    assert d % p != 0, 'a wrap of %d bytes must reach another physical byte' % d
  assert n_maps <= A.MAX_MAPS
  assert below % p == 0 and above % p == 0 and below + above == n_maps * p
  assert A.covers_wraps(below, above)
  assert above >= extent + p, 'the whole table and one chunk of slack lie above base'
  if p > 3 * gran:                                      # the smallest P that fits
    assert A.layout(extent, p // 2)[2] > A.MAX_MAPS
  assert A.chunk_bytes(extent, gran, min_bytes=4 * p) >= 4 * p


def test_wrapped_offsets_land_in_the_range():
  """every address a 32-bit wrap of an element offset produces lies inside [base - below, base + above)"""
  p = A.chunk_bytes(48 * A.GIB, 2 << 20)
  below, above, _ = A.layout(48 * A.GIB, p)
  for off in (2 ** 31, 2 ** 31 + 5, 2 ** 32 - 1, 2 ** 32, 3 * 2 ** 31, 2 ** 33 + 64 * 192):
    for wrapped in (((off + 2 ** 31) % 2 ** 32) - 2 ** 31, off % 2 ** 32):
      assert -below <= wrapped * 4 < above
      if wrapped != off:
        assert (wrapped * 4) % p != (off * 4) % p, 'a wrapped offset must reach another physical byte'
    for wrapped_b in (((off * 4 + 2 ** 31) % 2 ** 32) - 2 ** 31, (off * 4) % 2 ** 32):
      assert -below <= wrapped_b < above


@pytest.mark.parametrize('dim,row_stride', LAYOUTS)
def test_row_choice(dim, row_stride):
  n_rows = A.table_rows(row_stride)
  extent = n_rows * row_stride * 4
  assert extent <= 32 * A.GIB + row_stride * 4 * 64
  assert (n_rows - 1) * row_stride < 2 ** 33 + 64 * row_stride < 2.5 * 2 ** 32, 'a wrap never moves by 3 * 2^32 floats'
  p = A.chunk_bytes(extent, 2 << 20)
  high = A.boundary_rows(dim, row_stride, n_rows)
  assert max(high) == n_rows - 1
  for b in (2 ** 31, 2 ** 32):
    if n_rows * row_stride <= b:
      assert row_stride == 1 and b == 2 ** 32         # a K7 table of 2^32 - 2 rows of one float ends below 2^32
      continue
    offs = [r * row_stride for r in high]
    assert any(o + row_stride <= b for o in offs) and any(o >= b for o in offs), 'rows on both sides of %d' % b
    if b % row_stride:
      assert any(A.straddles(r, row_stride, b) for r in high), 'a row from below %d to above it' % b
  if dim in (1, 3) and n_rows > 2 ** 31 + 1:
    assert {2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1} <= set(high)
  if row_stride <= 2:
    assert n_rows == 2 ** 32 - 2
  # a row index truncated to int32 (r - 2^32 for r in [2^31, 2^32)) moves 2^32 row_stride floats down: the range maps
  # the address, and it is another physical byte
  below_min = A.below_bytes(n_rows, row_stride)
  p = A.chunk_bytes(extent, 2 << 20, below_min=below_min)
  below, above, n_maps = A.layout(extent, p, below_min)
  assert n_maps <= A.MAX_MAPS and row_stride % A.ODD
  wrapped_rows = [r for r in high if 2 ** 31 <= r < 2 ** 32]
  assert bool(wrapped_rows) == (n_rows > 2 ** 31)
  for r in wrapped_rows:
    for c in (0, row_stride - 1):
      good, bad = (r * row_stride + c) * 4, ((r - 2 ** 32) * row_stride + c) * 4
      assert -below <= bad < above, 'row %d truncated to int32 falls outside the reservation' % r
      assert good % p != bad % p, 'row %d truncated to int32 reaches its own physical byte' % r
  for off in (max(high) * row_stride, 2 ** 31, 2 ** 32):    # the element-offset wraps stay inside too
    for wrapped in (((off + 2 ** 31) % 2 ** 32) - 2 ** 31, off % 2 ** 32):
      assert -below <= wrapped * 4 < above
  low = A.with_low_rows(high, row_stride, p, 24, np.random.default_rng(row_stride))
  rows = high + low
  assert len(set(rows)) == len(rows) and A.images_disjoint(rows, row_stride, p)
  # the images of the row set, element by element, are pairwise distinct
  imgs = {A.image(r, c, row_stride, p) for r in rows for c in range(row_stride)}
  assert len(imgs) == len(rows) * row_stride


def test_images_disjoint_detects_overlap():
  p = 3 * (2 << 20)
  assert A.images_disjoint([0, 1, 2], 4, p)
  assert not A.images_disjoint([0, p // 16], 4, p)              # the same physical bytes
  assert not A.images_disjoint([p // 20, 0], 5, p)              # a row wrapping the chunk's end onto row 0
  assert A.images_disjoint([p // 20, 1], 5, p)
