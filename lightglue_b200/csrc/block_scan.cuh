// Ordered compaction by a 1024-thread block: one step over 1024 consecutive flags.
#pragma once

// Every thread of the block calls this with its flag (0 or 1) for element `base + tid`.  Returns the element's slot,
// `carry` plus the number of set flags before it in this step; `carry` (shared, 0 before the first step) is then
// advanced past the step.  warp_sums is shared scratch of 32 ints.  Ends with the block synchronised.
__device__ __forceinline__ int block_scan_step(int flag, int tid, int* warp_sums, int* carry) {
  int incl = flag;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, off);
    if ((tid & 31) >= off) incl += t;
  }
  if ((tid & 31) == 31) warp_sums[tid >> 5] = incl;
  __syncthreads();
  if (tid < 32) {
    int w = warp_sums[tid];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, off);
      if (tid >= off) w += t;
    }
    warp_sums[tid] = w;
  }
  __syncthreads();
  const int c = *carry;
  const int slot = c + ((tid >> 5) ? warp_sums[(tid >> 5) - 1] : 0) + incl - 1;
  __syncthreads();
  if (tid == 0) *carry = c + warp_sums[31];
  __syncthreads();
  return slot;
}
