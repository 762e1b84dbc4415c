// nms.cu — greedy hard-NMS over score-sorted boxes (torchvision.ops.nms semantics), used by
//   the two-stage proposal selection   ape/modeling/ape_deta/deformable_transformer_vl.py:591-596
//   the final class-aware NMS           ape/modeling/ape_deta/fast_rcnn.py:192 (detectron2 batched_nms)
// Two launches: (1) upper-triangular IoU>thr bit matrix, 64x64 boxes per CTA; (2) one CTA scans the
// sorted list in chunks of 64: one warp resolves the 64x64 diagonal block in registers, then all threads OR
// the rows of the boxes kept in that chunk into the suppression bitset out of shared memory (the rows of the
// next chunk are prefetched with cp.async meanwhile) — the serial dependency is 64 register steps per chunk.
// IoU arithmetic is written with explicit round-to-nearest intrinsics (no FMA contraction):
//   inter / (area_a + area_b - inter) > thr, widths/heights clamped at 0, as torchvision's devIoU.
#include "common.cuh"

namespace ape {
namespace {

__device__ __forceinline__ bool iou_gt(const float4 a, const float4 b, float thr) {
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  const float w = fmaxf(__fsub_rn(right, left), 0.f), h = fmaxf(__fsub_rn(bottom, top), 0.f);
  const float inter = __fmul_rn(w, h);
  const float sa = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  const float sb = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter)) > thr;
}

// grid (col_blocks, row_blocks), 64 threads; mask[row * col_blocks + cb] bit j = IoU(row, cb*64+j) > thr, j > row
__global__ void __launch_bounds__(64) nms_mask_kernel(const float4 *__restrict__ boxes, int n, const int *__restrict__ n_dev,
                                                      float thr, unsigned long long *__restrict__ mask, int col_blocks) {
  const int rb = blockIdx.y, cb = blockIdx.x;
  if (cb < rb) return;  // lower triangle never read
  if (n_dev) n = min(n, max(*n_dev, 0));  // only the first *n_dev boxes are real (static-shape callers)
  if (cb * 64 >= n) return;
  __shared__ float4 cols[64];
  const int t = threadIdx.x;
  const int col = cb * 64 + t;
  if (col < n) cols[t] = boxes[col];
  __syncthreads();
  const int row = rb * 64 + t;
  if (row >= n) return;
  const float4 a = boxes[row];
  const int ncols = min(64, n - cb * 64);
  unsigned long long bits = 0;
  for (int j = (rb == cb) ? t + 1 : 0; j < ncols; ++j)
    if (iou_gt(a, cols[j], thr)) bits |= 1ull << j;
  mask[(size_t)row * col_blocks + cb] = bits;
}

// single CTA, 1024 threads; keep[i] = 1 iff sorted box i survives; *count = number kept.
// Per chunk of 64 boxes: (a) warp 0 resolves the 64x64 diagonal block with the rows in registers (lane i holds
// rows i and i+32; the row broadcasts are shuffles that do not depend on the running bitset, so only a test +
// predicated OR per box sits on the serial chain); (b) all threads OR the rows of the kept boxes into the
// suppression bitset from SHARED memory — the chunk's rows were fetched with cp.async while the previous chunk
// was being resolved (double buffer), so no global-memory latency sits between chunks.
__device__ __forceinline__ void cp_async8(void *smem, const void *gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__global__ void __launch_bounds__(1024) nms_scan_kernel(const unsigned long long *__restrict__ mask, int n, const int *__restrict__ n_dev,
                                                        int pitch, unsigned char *__restrict__ keep, int *__restrict__ count) {
  extern __shared__ unsigned long long s_dyn[];
  if (n_dev) n = min(n, max(*n_dev, 0));
  const int col_blocks = (n + 63) / 64;  // active chunks; rows of `mask` are `pitch` words apart
  unsigned long long *removed = s_dyn;                      // col_blocks words
  unsigned long long *rows[2] = {s_dyn + pitch, s_dyn + pitch + 64 * (size_t)pitch};  // [64][pitch] each
  __shared__ unsigned long long s_keepbits;
  const int t = threadIdx.x, nt = blockDim.x;
  for (int w = t; w < col_blocks; w += nt) removed[w] = 0;
  auto prefetch = [&](int c, int buf) {
    // rows base..base+63, words c..col_blocks-1 (word c = the diagonal block)
    const int base = c * 64, nb = min(64, n - base), nw = col_blocks - c;
    for (int i = t; i < nb * nw; i += nt) {
      const int r = i / nw, w = c + (i - r * nw);
      cp_async8(&rows[buf][r * pitch + w], mask + (size_t)(base + r) * pitch + w);
    }
    cp_async_commit();
  };
  if (col_blocks > 0) prefetch(0, 0);
  int total = 0;
  for (int c = 0; c < col_blocks; ++c) {
    const int buf = c & 1;
    const int base = c * 64, nb = min(64, n - base);
    cp_async_wait_all();
    __syncthreads();  // chunk c's rows are in rows[buf]; removed[] of the previous chunk is complete
    if (c + 1 < col_blocks) prefetch(c + 1, buf ^ 1);
    if (t < 32) {
      const unsigned long long r0 = (t < nb) ? rows[buf][t * pitch + c] : 0ull;
      const unsigned long long r1 = (t + 32 < nb) ? rows[buf][(t + 32) * pitch + c] : 0ull;
      unsigned long long rem = removed[c], kept = 0;
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const unsigned long long row = __shfl_sync(0xffffffffu, i < 32 ? r0 : r1, i & 31);
        if (i < nb && !((rem >> i) & 1ull)) {
          kept |= 1ull << i;
          rem |= row;  // diagonal block: bits j > i only
        }
      }
      if (t == 0) s_keepbits = kept;
      total += __popcll(kept);
    }
    __syncthreads();
    const unsigned long long kept = s_keepbits;
    if (t < nb) keep[base + t] = (unsigned char)((kept >> t) & 1ull);
    // suppress later chunks: thread (g, wl) ORs rows g, g+8, .. of the chunk for word c+1+wl (+128, ..)
    const int g = t >> 7, wl = t & 127;
    for (int w = c + 1 + wl; w < col_blocks; w += 128) {
      unsigned long long acc = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int i = g + 8 * j;
        if ((kept >> i) & 1ull) acc |= rows[buf][i * pitch + w];
      }
      if (acc) atomicOr(&removed[w], acc);
    }
  }
  if (t == 0) *count = total;
}

// Fallback for very long lists (the double-buffered rows do not fit shared memory): same algorithm, rows read
// straight from global memory.
__global__ void __launch_bounds__(256) nms_scan_big_kernel(const unsigned long long *__restrict__ mask, int n, const int *__restrict__ n_dev,
                                                           int pitch, unsigned char *__restrict__ keep, int *__restrict__ count) {
  extern __shared__ unsigned long long removed[];  // col_blocks words
  if (n_dev) n = min(n, max(*n_dev, 0));
  const int col_blocks = (n + 63) / 64;
  __shared__ unsigned long long s_diag[64];
  __shared__ unsigned long long s_keepbits;
  __shared__ int s_total;
  const int t = threadIdx.x;
  for (int w = t; w < col_blocks; w += blockDim.x) removed[w] = 0;
  if (t == 0) s_total = 0;
  __syncthreads();
  for (int c = 0; c < col_blocks; ++c) {
    const int base = c * 64;
    const int nb = min(64, n - base);
    if (t < nb) s_diag[t] = mask[(size_t)(base + t) * pitch + c];
    __syncthreads();
    if (t == 0) {
      unsigned long long rem = removed[c], kept = 0;
      for (int i = 0; i < nb; ++i) {
        if (!((rem >> i) & 1ull)) {
          kept |= 1ull << i;
          rem |= s_diag[i];
        }
      }
      s_keepbits = kept;
      s_total += __popcll(kept);
    }
    __syncthreads();
    const unsigned long long kept = s_keepbits;
    if (t < nb) keep[base + t] = (unsigned char)((kept >> t) & 1ull);
    for (int w = c + 1 + t; w < col_blocks; w += blockDim.x) {
      unsigned long long acc = removed[w], k = kept;
      while (k) {
        const int i = __ffsll((long long)k) - 1;
        k &= k - 1;
        acc |= mask[(size_t)(base + i) * pitch + w];
      }
      removed[w] = acc;
    }
    __syncthreads();
  }
  if (t == 0) *count = s_total;
}


// ---------------------------------------------------------------------------------------------------------------
// Class-aware NMS for the open-vocabulary head when (almost) every (query, class) pair is a candidate
// (test_score_thresh = 0.0 with 900 queries x 1203 names = 1.08 M pairs: fast_rcnn.py:129-192 -> batched_nms, which
// torchvision runs class by class above 25 000 boxes on CUDA, `_batched_nms_vanilla`).  Every class sees the SAME Q boxes
// (boxes are per query), so one Q x Q IoU bit matrix serves all classes; the per-class work is "sort the queries by this
// class's score, greedy scan with the shared matrix".  Kernel 1 builds the matrix (one ballot per 32 pairs); kernel 2 is
// persistent: the matrix lives in shared memory, one WARP owns a class: compaction of the candidates (score > thresh),
// bitonic sort of 64-bit (score, index) keys in shared memory, scan with the suppression bitset in registers (lane w
// = word w), result written class-major: out[c][q] = score if (q, c) survives else -inf.
__global__ void __launch_bounds__(256) cw_mask_kernel(const float4 *__restrict__ boxes, int Q, int W, float thr,
                                                      unsigned *__restrict__ mask) {
  const int task = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (task >= Q * W) return;
  const int i = task / W, w = task - i * W;
  const int j = w * 32 + lane;
  bool bit = false;
  if (j < Q && j != i) bit = iou_gt(boxes[i], boxes[j], thr);
  const unsigned bits = __ballot_sync(0xffffffffu, bit);
  if (lane == 0) mask[task] = bits;
}

__device__ __forceinline__ unsigned ordered_bits(float f) {
  const unsigned u = __float_as_uint(f);
  return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}

constexpr int kCwWarps = 8, kCwMaxQ = 1024;

__global__ void __launch_bounds__(kCwWarps * 32) cw_scan_kernel(const unsigned *__restrict__ mask, const float *__restrict__ scores,
                                                                long long ld, const unsigned char *__restrict__ row_valid, int Q,
                                                                int N, int W, float score_thresh, float *__restrict__ out) {
  extern __shared__ unsigned long long s_cw[];
  unsigned long long *keys = s_cw + (size_t)(threadIdx.x >> 5) * kCwMaxQ;           // this warp's sort buffer
  unsigned *s_mask = reinterpret_cast<unsigned *>(s_cw + (size_t)kCwWarps * kCwMaxQ);  // [Q][W]
  for (int i = threadIdx.x; i < Q * W; i += blockDim.x) s_mask[i] = mask[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  const float ninf = __int_as_float(0xff800000);
  for (int c = blockIdx.x * kCwWarps + warp; c < N; c += gridDim.x * kCwWarps) {
    // 1. candidates of this class, compacted (order irrelevant: the keys are sorted next)
    int n = 0;
    for (int q0 = 0; q0 < Q; q0 += 32) {
      const int q = q0 + lane;
      float sc = 0.f;
      bool cand = false;
      if (q < Q && (!row_valid || row_valid[q])) {
        sc = scores[(size_t)q * ld + c];
        cand = sc > score_thresh;
      }
      const unsigned m = __ballot_sync(0xffffffffu, cand);
      if (cand) keys[n + __popc(m & lt)] = ((unsigned long long)ordered_bits(sc) << 32) | (unsigned)(0xffffffffu - (unsigned)q);
      n += __popc(m);
    }
    int np2 = 32;
    while (np2 < n) np2 <<= 1;
    for (int i = n + lane; i < np2; i += 32) keys[i] = 0ull;
    __syncwarp();
    // 2. bitonic sort, descending: higher score first, ties -> lower query index first
    for (int k = 2; k <= np2; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int t = lane; t < (np2 >> 1); t += 32) {
          const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // element with bit j clear
          const int p = i | j;
          const unsigned long long a = keys[i], b = keys[p];
          const bool desc = (i & k) == 0;
          if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[p] = a; }
        }
        __syncwarp();
      }
    }
    // 3. greedy scan: `removed` / `kept` bitsets live in registers, lane w = word w
    unsigned removed = 0, kept = 0;
    unsigned long long key = n > 0 ? keys[0] : 0ull;
    for (int i = 0; i < n; ++i) {
      const unsigned long long next = (i + 1 < n) ? keys[i + 1] : 0ull;  // independent of the chain below
      const unsigned q = 0xffffffffu - (unsigned)(key & 0xffffffffull);
      const unsigned r = __shfl_sync(0xffffffffu, removed, q >> 5);
      if (!((r >> (q & 31)) & 1u)) {  // warp-uniform
        if (lane == (int)(q >> 5)) kept |= 1u << (q & 31);
        if (lane < W) removed |= s_mask[q * W + lane];
      }
      key = next;
    }
    // 4. class-major output row
    float *orow = out + (size_t)c * Q;
    for (int q0 = 0; q0 < Q; q0 += 32) {
      const unsigned kb = __shfl_sync(0xffffffffu, kept, q0 >> 5);
      const int q = q0 + lane;
      if (q < Q) orow[q] = ((kb >> lane) & 1u) ? scores[(size_t)q * ld + c] : ninf;
    }
    __syncwarp();
  }
}

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int64_t ape_nms_workspace_bytes(int n) {
  const int64_t cb = (n + 63) / 64;
  return (int64_t)n * cb * 8;
}

static int nms_launch(const float *boxes_sorted, int n, const int *n_dev, float iou_threshold, void *workspace, uint8_t *keep,
                      int *count, void *stream) {
  if (n < 0) return fail(APE_ERR_INVALID_ARG, "nms: n=%d", n);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (n == 0) {
    if (count) cudaMemsetAsync(count, 0, sizeof(int), st);
    return APE_OK;
  }
  if (!boxes_sorted || !workspace || !keep || !count) return fail(APE_ERR_NULL_PTR, "nms: null pointer argument");
  if (reinterpret_cast<uintptr_t>(boxes_sorted) & 15) return fail(APE_ERR_INVALID_ARG, "nms: boxes must be 16-byte aligned");
  const int cb = (n + 63) / 64;
  if ((size_t)cb * 8 > 200 * 1024) return fail(APE_ERR_UNSUPPORTED, "nms: n=%d too large for the single-CTA scan", n);
  if (n_dev) cudaMemsetAsync(keep, 0, (size_t)n, st);  // entries past *n_dev are never visited
  nms_mask_kernel<<<dim3(cb, cb), 64, 0, st>>>(reinterpret_cast<const float4 *>(boxes_sorted), n, n_dev, iou_threshold,
                                               reinterpret_cast<unsigned long long *>(workspace), cb);
  if (int rc = check_launch("nms_mask_kernel")) return rc;
  const size_t smem = (size_t)cb * 8 * (1 + 2 * 64);
  if (smem <= 200 * 1024) {
    if (smem > 48 * 1024) {
      cudaError_t e = cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return fail((int)e, "nms: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    }
    nms_scan_kernel<<<1, 1024, smem, st>>>(reinterpret_cast<const unsigned long long *>(workspace), n, n_dev, cb, keep, count);
    return check_launch("nms_scan_kernel");
  }
  const size_t smem_big = (size_t)cb * 8;
  if (smem_big > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(nms_scan_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_big);
    if (e != cudaSuccess) return fail((int)e, "nms: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  nms_scan_big_kernel<<<1, 256, smem_big, st>>>(reinterpret_cast<const unsigned long long *>(workspace), n, n_dev, cb, keep, count);
  return check_launch("nms_scan_kernel");
}

extern "C" int ape_nms_sorted(const float *boxes_sorted, int n, float iou_threshold, void *workspace, uint8_t *keep,
                              int *count, void *stream) {
  return nms_launch(boxes_sorted, n, nullptr, iou_threshold, workspace, keep, count, stream);
}

extern "C" int ape_nms_sorted_dev(const float *boxes_sorted, int n_max, const int *n_dev, float iou_threshold, void *workspace,
                                  uint8_t *keep, int *count, void *stream) {
  if (!n_dev) return fail(APE_ERR_NULL_PTR, "nms: null n_dev");
  return nms_launch(boxes_sorted, n_max, n_dev, iou_threshold, workspace, keep, count, stream);
}

extern "C" int64_t ape_nms_classwise_workspace_bytes(int Q) { return (int64_t)Q * ((Q + 31) / 32) * 4; }

extern "C" int ape_nms_classwise(const float *boxes, const float *scores, int64_t ld_scores, const uint8_t *row_valid, int Q,
                                 int N, float score_thresh, float iou_threshold, void *workspace, float *out, void *stream) {
  if (Q < 0 || N < 0 || Q > kCwMaxQ) return fail(APE_ERR_UNSUPPORTED, "nms_classwise: Q=%d N=%d (Q <= %d)", Q, N, kCwMaxQ);
  if (Q == 0 || N == 0) return APE_OK;
  if (!boxes || !scores || !workspace || !out) return fail(APE_ERR_NULL_PTR, "nms_classwise: null pointer argument");
  if (reinterpret_cast<uintptr_t>(boxes) & 15) return fail(APE_ERR_INVALID_ARG, "nms_classwise: boxes must be 16-byte aligned");
  if (ld_scores < N) return fail(APE_ERR_INVALID_ARG, "nms_classwise: ld_scores < N");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int W = (Q + 31) / 32;
  cw_mask_kernel<<<(Q * W + 7) / 8, 256, 0, st>>>(reinterpret_cast<const float4 *>(boxes), Q, W, iou_threshold,
                                                  reinterpret_cast<unsigned *>(workspace));
  if (int rc = check_launch("cw_mask_kernel")) return rc;
  const size_t smem = (size_t)kCwWarps * kCwMaxQ * 8 + (size_t)Q * W * 4;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(cw_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return fail((int)e, "nms_classwise: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  int sms = 0, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) sms = 132;
  const int ctas = min(sms, (N + kCwWarps - 1) / kCwWarps);
  cw_scan_kernel<<<ctas, kCwWarps * 32, smem, st>>>(reinterpret_cast<const unsigned *>(workspace), scores, ld_scores, row_valid, Q,
                                                    N, W, score_thresh, out);
  return check_launch("cw_scan_kernel");
}
