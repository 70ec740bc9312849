// First-occurrence table of the device-side unique (unique.cu) and of the fused full-neighbor hop (full_hop.cu): an
// open-addressing table keyed by id that keeps the minimum index under which the id was inserted.
#pragma once
#include "common.cuh"

namespace eu {

// slot = {id + 1, min index}; key 0 = free; id 2^64-1 (tag overflow) lives in the extra slot [mask + 1]
__device__ __forceinline__ void uq_insert(HashSlot* tab, unsigned long long mask, unsigned long long id, unsigned long long i) {
  const unsigned long long tag = id + 1;
  if (tag == 0ull) { atomicMin(&tab[mask + 1].row, i); return; }
  unsigned long long h = mix64(id) & mask;
  while (true) {
    const unsigned long long prev = atomicCAS(&tab[h].key, 0ull, tag);
    if (prev == 0ull || prev == tag) { atomicMin(&tab[h].row, i); return; }
    h = (h + 1) & mask;
  }
}

__device__ __forceinline__ unsigned long long uq_first(const HashSlot* tab, unsigned long long mask, unsigned long long id) {
  const unsigned long long tag = id + 1;
  if (tag == 0ull) return tab[mask + 1].row;
  unsigned long long h = mix64(id) & mask;
  while (true) {
    const ulonglong2 s = *reinterpret_cast<const ulonglong2*>(tab + h);
    if (s.x == tag) return s.y;
    h = (h + 1) & mask;
  }
}

// Insert from a warp whose active lanes hold consecutive indices i: runs of equal ids (default fill, hubs, a node listed by
// many rows) would hammer one slot, so only the lowest lane of each group of equal ids -- the group's minimum index --
// inserts.
__device__ __forceinline__ void uq_insert_warp(HashSlot* tab, unsigned long long mask, unsigned long long id, unsigned long long i) {
  const unsigned peers = __match_any_sync(__activemask(), id);
  if ((threadIdx.x & 31) != __ffs(peers) - 1) return;
  uq_insert(tab, mask, id, i);
}

static __global__ void k_uq_clear(HashSlot* tab, int64_t slots) {
  for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < slots; s += (int64_t)gridDim.x * blockDim.x) {
    tab[s].key = 0ull; tab[s].row = kEmptyRow;
  }
}

// table slots for n inserted ids: the power of two >= 2n, at least 64 (one more slot holds id 2^64-1)
inline int64_t uq_table_cap(int64_t n) {
  int64_t cap = 64;
  while (cap < 2 * n) cap <<= 1;
  return cap;
}

}  // namespace eu
