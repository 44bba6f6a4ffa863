"""Aliased device memory: a huge virtual table backed by one small physical allocation.

The sparse kernels index tables of up to 2^32 - 2 rows, so a float offset row * row_stride + col passes 2^31 and 2^32
in the tables the project trains (a 200M-row item table at dim 16 with interleaved Adagrad state holds 6.4e9 floats).
Testing those offsets on real memory needs tens of GiB per case.  An AliasedArena instead reserves a virtual range and
maps ONE physical chunk of P bytes into it back to back with the CUDA driver's virtual memory management API
(cuMemCreate / cuMemAddressReserve / cuMemMap / cuMemSetAccess), so byte x of the range lies on physical byte x mod P:

  reservation  [base - below, base + above),  above >= max(extent, 16 GiB) + P,  both multiples of P,
               below >= 8 GiB, and >= 2^31 row_stride elem bytes when the table has rows past 2^31
  P            ODD * 2^k * granularity, ODD = 5: never a power of two, and no divisor of a row stride in play

Why a kernel that computes a wrong offset is seen, and cannot fault:
  * a wrapped int32 element offset lies in [-8 GiB, 8 GiB) bytes of base, a wrapped uint32 one in [0, 16 GiB), a wrapped
    32-bit byte offset in [-2 GiB, 4 GiB); a row index r in [2^31, 2^32) truncated to int32 (r - 2^32, e.g. `int r =
    rows[i]`, or a signed cast of K7's uint32 row) lies 2^32 row_stride elements lower, at least -2^31 row_stride
    elements from base: the reservation maps all of them, so the access lands in the chunk;
  * a displacement of 2^31 or 2^32 floats (2^33 / 2^34 bytes), of 2^32 bytes, or of 2^32 rows (2^34 row_stride bytes)
    is not a multiple of P, since ODD divides no power of two and no row stride the tests use (the tables refuse a
    stride ODD divides): it reaches a different physical byte than the right address;
  * a test places its rows so that their images (row * row_stride + col) * 4 mod P are pairwise disjoint and fills
    every other physical byte with a sentinel: a write to a wrong address changes a byte it must not.

The arithmetic (choice of P, the layout, the images, the row choice) is plain Python below, checked on the host by
test_aliased_arena_host.py; AliasedArena is the device part.
"""
import ctypes

GIB = 1 << 30
BELOW = 8 * GIB          # int32 element offsets wrap to at most 2^31 floats below base
ABOVE_MIN = 16 * GIB     # uint32 element offsets wrap to below 2^32 floats above base
ODD = 5                  # odd factor of P: divides no power of two and none of the row strides the tests use
MAX_MAPS = 256           # mappings of the chunk per arena (each costs a driver call); P grows instead
SENTINEL = 0x3E5A5A5A    # fill of every physical word no row image covers (a finite float, 0.2132...)
SENTINEL_BYTE = 0x5A     # the same fill for byte-sized arenas (touched masks)
LIVE = {'bytes': 0, 'peak': 0}   # physical bytes of the open arenas, and their peak


def _ceil_to(x, m):
  return -(-x // m) * m


def below_bytes(n_rows=0, row_stride=1, elem=4):
  """bytes the reservation must reach below base: 8 GiB for wrapped int32 element offsets, and for a table with rows
  past 2^31 also the 2^32 row_stride elements a row index truncated to int32 moves down by (row 2^31 -> -2^31)"""
  return max(BELOW, 2 ** 31 * row_stride * elem if n_rows > 2 ** 31 else 0)


def chunk_bytes(extent, gran, max_maps=MAX_MAPS, min_bytes=0, below_min=BELOW):
  """The smallest P = ODD * 2^k * gran, P >= min_bytes, that maps the reservation of `extent` bytes (and below_min
  bytes below base) in at most max_maps mappings."""
  k = 0
  while True:
    p = ODD * (1 << k) * gran
    if p >= min_bytes and layout(extent, p, below_min)[2] <= max_maps:
      return p
    k += 1


def layout(extent, p, below_min=BELOW):
  """(below, above, n_maps) of the reservation around base for a range of `extent` bytes and chunk P"""
  below = _ceil_to(max(BELOW, below_min), p)
  above = _ceil_to(max(extent, ABOVE_MIN) + p, p)
  return below, above, (below + above) // p


def image(row, col, row_stride, p, elem=4):
  """physical byte of element (row, col) of a [*, row_stride] matrix at base"""
  return ((row * row_stride + col) * elem) % p


def images_disjoint(rows, row_stride, p, elem=4):
  """True when the physical byte ranges of the given rows (row_stride elements each) do not overlap"""
  span = row_stride * elem
  iv = []
  for r in rows:
    a = image(r, 0, row_stride, p, elem)
    if a + span <= p:
      iv.append((a, a + span))
    else:                                          # the row wraps around the end of the chunk
      iv.append((a, p))
      iv.append((0, a + span - p))
  iv.sort()
  return all(iv[i][1] <= iv[i + 1][0] for i in range(len(iv) - 1))


def covers_wraps(below, above):
  """True when the reservation [base - below, base + above) holds every address a 32-bit wrap can produce"""
  return below >= 2 ** 31 * 4 and above >= 2 ** 32 * 4 and above >= 2 ** 32


def table_rows(row_stride):
  """n_rows of the aliased tables at this row stride: 2^32 - 2 (K7's largest) while the table stays below 2^33 floats,
  else enough rows to reach 2^33 floats.  Every offset then stays below 2^33 + 64 row_stride, so a 32-bit wrap of the
  offset moves it by 2^32 or 2^33 floats; a truncated row index moves it by 2^32 row_stride floats.  With ODD not
  dividing row_stride, P divides none of these."""
  return 2 ** 32 - 2 if row_stride <= 2 else 2 ** 33 // row_stride + 64


def boundary_rows(dim, row_stride, n_rows):
  """Rows whose float offsets sit just below, across and just above 2^31 and 2^32: for each boundary B the rows from two
  before to two after the one holding float B (with a stride that does not divide B the row B // row_stride starts below
  B and ends above it).  At dims 1 and 3 also rows 2^31 - 1, 2^31, 2^31 + 1, and always n_rows - 1."""
  out = []
  for b in (2 ** 31, 2 ** 32):
    r0 = b // row_stride
    out += [r for r in range(r0 - 2, r0 + 3) if 0 <= r < n_rows]
  if dim in (1, 3):
    out += [r for r in (2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1) if r < n_rows]
  out.append(n_rows - 1)
  return sorted(set(out))


def straddles(row, row_stride, b):
  return row * row_stride < b < (row + 1) * row_stride


def with_low_rows(high, row_stride, p, n_low, rng, lo_max=1 << 20, elem=4):
  """high rows plus n_low random rows below lo_max whose images miss every chosen row's"""
  rows = list(high)
  assert images_disjoint(rows, row_stride, p, elem), 'boundary rows overlap in the chunk: raise P'
  low = []
  while len(low) < n_low:
    r = int(rng.integers(0, lo_max))
    if r in rows or not images_disjoint(rows + [r], row_stride, p, elem):
      continue
    rows.append(r)
    low.append(r)
  return sorted(low)


# ---- the device part ----------------------------------------------------------------------------------------------
class _Prop(ctypes.Structure):
  """CUmemAllocationProp"""
  _fields_ = [('type', ctypes.c_int), ('requestedHandleTypes', ctypes.c_int), ('loc_type', ctypes.c_int),
              ('loc_id', ctypes.c_int), ('win32HandleMetaData', ctypes.c_void_p), ('compressionType', ctypes.c_ubyte),
              ('gpuDirectRDMACapable', ctypes.c_ubyte), ('usage', ctypes.c_ushort), ('reserved', ctypes.c_ubyte * 4)]


class _Access(ctypes.Structure):
  """CUmemAccessDesc"""
  _fields_ = [('loc_type', ctypes.c_int), ('loc_id', ctypes.c_int), ('flags', ctypes.c_int)]


_CU_MEM_ALLOCATION_TYPE_PINNED = 1
_CU_MEM_LOCATION_TYPE_DEVICE = 1
_CU_MEM_ACCESS_FLAGS_PROT_READWRITE = 3
_CU_MEM_ALLOC_GRANULARITY_MINIMUM = 0
_cu = None


def _driver():
  global _cu
  if _cu is None:
    _cu = ctypes.CDLL('libcuda.so.1')
    for nm in ('cuMemAddressReserve', 'cuMemMap', 'cuMemSetAccess', 'cuMemUnmap', 'cuMemAddressFree', 'cuMemCreate',
               'cuMemRelease', 'cuMemGetAllocationGranularity'):
      getattr(_cu, nm).restype = ctypes.c_int
  return _cu


def _ck(rc, what):
  if rc != 0:
    raise RuntimeError('%s failed: CUresult %d' % (what, rc))


class _Iface(object):
  def __init__(self, ptr, shape, typestr):
    self.__cuda_array_interface__ = {'shape': tuple(shape), 'typestr': typestr, 'data': (ptr, False), 'version': 2,
                                     'strides': None}


class AliasedArena(object):
  """A virtual range of `extent` bytes at `base` (plus the wrap margins) on one physical chunk of `p` bytes.

  tensor(shape, dtype) views base zero-copy; phys(dtype) views the chunk (mapping 0).  Use as a context manager, so
  that close() (unmap, free the range, release the chunk) runs when a test fails too."""

  def __init__(self, device, extent, max_maps=MAX_MAPS, min_bytes=0, fill=SENTINEL, below_min=BELOW):
    import torch
    self.torch = torch
    self.device = torch.device(device)
    torch.zeros(1, device=self.device)            # the primary context, current on this thread
    torch.cuda.synchronize(self.device)
    cu = _driver()
    prop = _Prop()
    prop.type = _CU_MEM_ALLOCATION_TYPE_PINNED
    prop.loc_type = _CU_MEM_LOCATION_TYPE_DEVICE
    prop.loc_id = self.device.index or 0
    gran = ctypes.c_size_t()
    _ck(cu.cuMemGetAllocationGranularity(ctypes.byref(gran), ctypes.byref(prop), _CU_MEM_ALLOC_GRANULARITY_MINIMUM),
        'cuMemGetAllocationGranularity')
    self.gran = gran.value
    self.p = chunk_bytes(extent, self.gran, max_maps, min_bytes, below_min)
    self.below, self.above, self.n_maps = layout(extent, self.p, below_min)
    if self.n_maps > max_maps:
      raise ValueError('%d mappings of the chunk: at most %d' % (self.n_maps, max_maps))
    self.size = self.below + self.above
    self._handle = self._lo = None
    self._mapped = 0
    try:
      h = ctypes.c_ulonglong()
      _ck(cu.cuMemCreate(ctypes.byref(h), ctypes.c_size_t(self.p), ctypes.byref(prop), ctypes.c_ulonglong(0)),
          'cuMemCreate')
      self._handle = h.value
      LIVE['bytes'] += self.p
      LIVE['peak'] = max(LIVE['peak'], LIVE['bytes'])
      lo = ctypes.c_ulonglong()
      # alignment 0: the granularity (P itself is not a power of two, and the mappings need no more)
      _ck(cu.cuMemAddressReserve(ctypes.byref(lo), ctypes.c_size_t(self.size), ctypes.c_size_t(0),
                                 ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)), 'cuMemAddressReserve')
      self._lo = lo.value
      acc = _Access(_CU_MEM_LOCATION_TYPE_DEVICE, prop.loc_id, _CU_MEM_ACCESS_FLAGS_PROT_READWRITE)
      for i in range(self.n_maps):
        _ck(cu.cuMemMap(ctypes.c_ulonglong(self._lo + i * self.p), ctypes.c_size_t(self.p), ctypes.c_size_t(0),
                        ctypes.c_ulonglong(self._handle), ctypes.c_ulonglong(0)), 'cuMemMap')
        self._mapped += 1
      _ck(cu.cuMemSetAccess(ctypes.c_ulonglong(self._lo), ctypes.c_size_t(self.size), ctypes.byref(acc),
                            ctypes.c_size_t(1)), 'cuMemSetAccess')
      self.base = self._lo + self.below
      self.fill(fill)
      self._self_check()
    except BaseException:
      self.close()
      raise

  def tensor(self, shape, dtype, byte_offset=0):
    """a zero-copy view [shape] at base + byte_offset (the aliased table)"""
    torch = self.torch
    ts = {torch.float32: '<f4', torch.uint8: '|u1', torch.int32: '<i4', torch.int64: '<i8'}[dtype]
    ptr = self.base + byte_offset
    t = torch.as_tensor(_Iface(ptr, shape, ts), device=self.device)
    if t.data_ptr() != ptr:
      raise RuntimeError('torch.as_tensor copied the aliased range')
    return t

  def phys(self, dtype):
    """the P physical bytes as a flat tensor (mapping 0 of the range)"""
    torch = self.torch
    n = self.p // torch.empty(0, dtype=dtype).element_size()
    ts = {torch.float32: '<f4', torch.uint8: '|u1', torch.int32: '<i4'}[dtype]
    t = torch.as_tensor(_Iface(self._lo, (n,), ts), device=self.device)
    assert t.data_ptr() == self._lo
    return t

  def fill(self, value):
    torch = self.torch
    if value == SENTINEL:
      self.phys(torch.int32).fill_(SENTINEL)
    else:
      self.phys(torch.uint8).fill_(value)

  def _self_check(self):
    """a word written through the last mapping reads back through mapping 0, and through base at its image"""
    torch = self.torch
    ph = self.phys(torch.int32)
    keep = ph[:2].clone()
    k = self.n_maps - 1
    far = torch.as_tensor(_Iface(self._lo + k * self.p, (2,), '<i4'), device=self.device)
    far.copy_(torch.tensor([0x12345678, -0x2468ACE], dtype=torch.int32))
    if not torch.equal(ph[:2].cpu(), torch.tensor([0x12345678, -0x2468ACE], dtype=torch.int32)):
      raise RuntimeError('a write through mapping %d did not reach mapping 0' % k)
    ph[:2] = keep
    torch.cuda.synchronize(self.device)

  def close(self):
    """unmap, free the range and release the chunk; every step is tried even when an earlier one fails, and the first
    failure is raised at the end"""
    cu = _driver()
    failed = []

    def step(rc, what):
      if rc != 0:
        failed.append('%s failed: CUresult %d' % (what, rc))

    if self._lo is not None:
      try:
        self.torch.cuda.synchronize(self.device)
      except Exception as e:                       # still release what the driver holds
        failed.append('synchronize: %s' % e)
      # the mappings are unmapped one by one, as they were made
      for i in range(self._mapped):
        step(cu.cuMemUnmap(ctypes.c_ulonglong(self._lo + i * self.p), ctypes.c_size_t(self.p)), 'cuMemUnmap')
      self._mapped = 0
      step(cu.cuMemAddressFree(ctypes.c_ulonglong(self._lo), ctypes.c_size_t(self.size)), 'cuMemAddressFree')
      self._lo = None
    if self._handle is not None:
      step(cu.cuMemRelease(ctypes.c_ulonglong(self._handle)), 'cuMemRelease')
      self._handle = None
      LIVE['bytes'] -= self.p
    if failed:
      raise RuntimeError('; '.join(failed))

  def __enter__(self):
    return self

  def __exit__(self, *exc):
    self.close()
    return False
