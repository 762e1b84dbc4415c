// rle.cuh — device pieces of cocoapi's run-length "counts" strings, shared by the instance-mask encoder (mask_post.cu) and the
// label-map encoder (label_rle.cu).
#pragma once
#include "common.cuh"

namespace ape {

// block-wide exclusive sum over 256 threads; returns this thread's offset, *sum the total.  s_warp holds 8 ints.
__device__ __forceinline__ int block_excl_scan_256(int v, int *s_warp, int *sum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int before = 0, total = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    before += i < warp ? s_warp[i] : 0;
    total += s_warp[i];
  }
  __syncthreads();  // s_warp is reused by the next call
  *sum = total;
  return before + incl - v;
}

// cocoapi rleToString of one count (see ape_rle_to_string): number of characters, and the characters when out != NULL
__device__ __forceinline__ int rle_chars(long long x, uint8_t *out, int room) {
  int n = 0;
  bool more = true;
  while (more) {
    int c = (int)(x & 0x1f);
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    if (more) c |= 0x20;
    if (out && n < room) out[n] = (uint8_t)(c + 48);
    ++n;
  }
  return n;
}

}  // namespace ape
