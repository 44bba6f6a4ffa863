// The open-addressing index of 63-bit keys shared by the key-value tables (csrc/kv_table.cu) and K1's vocabulary
// lookup (ER_BUCKET_VOCAB, csrc/bucketize.cu).
//
// Layout: keys[n_index] (ER_KV_EMPTY = free) and rows[n_index], n_index a power of two >= 16.  A key's probe sequence
// is the 16-slot (128-byte) groups g, g + 1, ... from g = mix(key) mod (n_index / 16); a 16-lane tile loads one group
// per step and compares all 16 keys with one ballot.  Slots are claimed with a 64-bit atomicCAS and never freed, so
// every thread that looks up one key walks the same slots, sees each one's final value (either in its load or as its
// CAS result), and stops on the same slot.
#pragma once
#include "common.cuh"

namespace er {

constexpr int kKvTile = 16;

__device__ __forceinline__ uint64_t kv_mix(uint64_t z) {   // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

struct KvIndex {
  long long* keys;
  int64_t* rows;
  int64_t n_groups;   // n_index / 16, a power of two
};

// The slot of `k`, or -1 (find: absent; insert: every slot holds another key).  Called by all 16 lanes of the tile
// (lane t of the tile at warp lane base + t, tmask = the tile's lanes) with the same k; uniform over the tile.  `won`:
// this call claimed the slot.  A key is claimed whether or not the pool has a row left for it, so every lookup of one
// key lands on the same slot; the claimer decides the row.
template <bool kInsert>
__device__ __forceinline__ int64_t kv_probe(const KvIndex& ix, int64_t k, int t, int base, unsigned tmask, bool& won) {
  won = false;
  const int64_t gmask = ix.n_groups - 1;
  const int64_t g0 = (int64_t)(kv_mix((uint64_t)k) & (uint64_t)gmask);
  for (int64_t i = 0; i < ix.n_groups; ++i) {
    const int64_t s0 = ((g0 + i) & gmask) * kKvTile;
    const long long v = *(volatile const long long*)(ix.keys + s0 + t);
    const unsigned hit = (__ballot_sync(tmask, v == (long long)k) >> base) & 0xFFFFu;
    if (hit) return s0 + __ffs(hit) - 1;
    unsigned empty = (__ballot_sync(tmask, v == (long long)ER_KV_EMPTY) >> base) & 0xFFFFu;
    if constexpr (!kInsert) {
      if (empty) return -1;   // a key is never stored past a free slot of its sequence
    } else {
      while (empty) {
        const int j = __ffs(empty) - 1;
        long long old = 0;
        if (t == j) old = atomicCAS((unsigned long long*)(ix.keys + s0 + j), (unsigned long long)ER_KV_EMPTY,
                                    (unsigned long long)k);
        old = __shfl_sync(tmask, old, base + j);
        if (old == (long long)ER_KV_EMPTY) {
          won = true;
          return s0 + j;
        }
        if (old == (long long)k) return s0 + j;
        empty &= empty - 1;   // another key took it: the next free slot of this group
      }
    }
  }
  return -1;
}

// The find side: the slot of `k` in an index nobody writes during the call, or -1.
__device__ __forceinline__ int64_t kv_find_slot(const KvIndex& ix, int64_t k, int t, int base, unsigned tmask) {
  bool won;
  return kv_probe<false>(ix, k, t, base, tmask, won);
}

}  // namespace er
