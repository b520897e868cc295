// One launch over a host table of entries of any sizes (bt_adamw_step, bt_grad_pack, bt_grad_ordered_sum): each entry
// is cut into chunks of a kernel's fixed element count, block b takes chunk b of the whole table, and the host stores
// each entry's first chunk (the prefix sums of the chunk counts) as its chunk0.
#pragma once
#include <stdint.h>

namespace bt {

// The entry of block `chunk`: the last one whose first chunk is <= chunk (entries of no chunks are never chosen when a
// later entry starts at the same chunk).
template <class Entry>
__device__ __forceinline__ int entry_of_chunk(const Entry* __restrict__ entries, int n_entries, int64_t chunk) {
  int lo = 0, hi = n_entries - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (entries[mid].chunk0 <= chunk) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

}  // namespace bt
