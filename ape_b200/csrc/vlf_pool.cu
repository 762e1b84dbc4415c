// vlf_pool.cu — language-side attention pooling of VisionLanguageFusion for ONE language token
// (the "name" prompt case; BiMultiHeadAttention.forward, ape/layers/fuse_helper.py:67-166, restructured as
// in ape_b200/layers/vision_language_fusion.py:single_token).  For every head h:
//     t[s]   = v_s . qa[h] + qc[h]                       (scores of all S vision tokens against the one key)
//     w[s]   = clamp(t[s] - max_all(t), -5e4, 5e4)        (stable_softmax_2d + clamps, fuse_helper.py:88-97)
//     wl[s]  = clamp(w[s] - max_s(w), -5e4, 5e4)          (:99-108)
//     p      = softmax_s(wl);   pooled[h,:] = sum_s p[s] * v_s
// Three launches, v is read twice (16-bit), nothing of size S x 2048 is ever formed:
//   (1) scores + per-CTA maxima: ~300 CTAs each own a strip of tokens, one warp per token, qa in registers;
//   (2) fold maxima (per head and global);  (3) per-CTA partial sums of exp() and exp()*v over the same strips.
// The caller folds the [strips] partials (deterministic order) and applies the tiny projections.
#include "common.cuh"

namespace ape {
namespace {

constexpr int kMaxHeads = 8;
constexpr int kMaxStrip = 512;  // tokens per CTA (both passes); bounds the exp() staging buffer

__device__ __forceinline__ void load8f(const float *p, float *f) {
  const float4 a = *reinterpret_cast<const float4 *>(p), b = *reinterpret_cast<const float4 *>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <typename T>
__device__ __forceinline__ void load_row8(const T *p, float *f) {
  if constexpr (sizeof(T) == 4) load8f(reinterpret_cast<const float *>(p), f);
  else Elem<T>::unpack(*reinterpret_cast<const uint4 *>(p), f);
}

// Pass 1.  grid (nct, B), 256 threads; the CTA owns tokens [blockIdx.x*strip, +strip), one warp per token,
// lane = 8 channels (C == 256), the 8x8 slice of qa a lane needs lives in registers.  The 8 per-head partial
// dot products of a lane are reduced over the warp with a halving butterfly (9 shuffles instead of 40).
template <typename T>
__global__ void __launch_bounds__(256)
vlf_scores_kernel(const T *__restrict__ v, const float *__restrict__ qa, const float *__restrict__ qc,
                  float *__restrict__ scores, float *__restrict__ blockmax, int S, int NH, int strip) {
  pdl_prologue();
  constexpr int C = 256;
  __shared__ float s_max[8][kMaxHeads];
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float q[kMaxHeads][8];
#pragma unroll
  for (int h = 0; h < kMaxHeads; ++h) {
    if (h < NH) load8f(qa + ((size_t)b * NH + h) * C + lane * 8, q[h]);
    else {
#pragma unroll
      for (int k = 0; k < 8; ++k) q[h][k] = 0.f;
    }
  }
  // after the butterfly lane L holds head (L>>2)&7's total (see below); its bias:
  const int myh = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
  const float myqc = myh < NH ? qc[b * NH + myh] : 0.f;
  const int s0 = blockIdx.x * strip, s1 = min(S, s0 + strip);
  float wmax = -INFINITY;
  // one token: 8 per-head partial dot products per lane, reduced over the warp by the halving butterfly; lane L ends with head
  // myh's total
  auto score = [&](const float *f, int s) {
    float a[kMaxHeads];
#pragma unroll
    for (int h = 0; h < kMaxHeads; ++h) {
      a[h] = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) a[h] = fmaf(f[k], q[h][k], a[h]);
    }
    // halving butterfly: bit 4 of the lane picks heads {0..3} / {4..7}, bit 3 the pair, bit 2 the head
    float c4[4];
    const bool hi16 = lane & 16;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float send = hi16 ? a[i] : a[i + 4], keep = hi16 ? a[i + 4] : a[i];
      c4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
    float c2[2];
    const bool hi8 = lane & 8;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float send = hi8 ? c4[i] : c4[i + 2], keep = hi8 ? c4[i + 2] : c4[i];
      c2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    const bool hi4 = lane & 4;
    float c1 = (hi4 ? c2[1] : c2[0]) + __shfl_xor_sync(0xffffffffu, hi4 ? c2[0] : c2[1], 4);
    c1 += __shfl_xor_sync(0xffffffffu, c1, 2);
    c1 += __shfl_xor_sync(0xffffffffu, c1, 1);
    const float t = c1 + myqc;
    if ((lane & 3) == 0 && myh < NH) scores[((size_t)b * NH + myh) * S + s] = t;
    wmax = fmaxf(wmax, t);
  };
  // two tokens per iteration: both rows are requested before either is reduced (the loop is bound by the latency of one
  // 512-byte row load per warp at two CTAs per SM: 32 us for the 45 MB of the 1024^2 encoder, 4.5x the HBM time)
  for (int s = s0 + warp; s < s1; s += 16) {
    const bool two = s + 8 < s1;  // warp-uniform
    float f0[8], f1[8];
    load_row8<T>(v + ((size_t)b * S + s) * C + lane * 8, f0);
    if (two) load_row8<T>(v + ((size_t)b * S + s + 8) * C + lane * 8, f1);
    score(f0, s);
    if (two) score(f1, s + 8);
  }
  if ((lane & 3) == 0) s_max[warp][myh] = wmax;
  __syncthreads();
  if (threadIdx.x < NH) {
    float m = s_max[0][threadIdx.x];
    for (int w = 1; w < 8; ++w) m = fmaxf(m, s_max[w][threadIdx.x]);
    blockmax[((size_t)b * gridDim.x + blockIdx.x) * NH + threadIdx.x] = m;
  }
}

// maxes[0] = global max over everything; maxes[1 + b*NH + h] = max over s of scores[b,h,:].  One CTA,
// one warp per (b, h) pair (round-robin), lanes stride over the per-CTA maxima of pass 1.
__global__ void __launch_bounds__(1024)
vlf_max_kernel(const float *__restrict__ blockmax, int B, int nblk, int NH, float *__restrict__ maxes) {
  pdl_prologue();
  __shared__ float s_row[64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = warp; t < B * NH; t += 32) {
    const int b = t / NH, h = t % NH;
    float m = -INFINITY;
    for (int i = lane; i < nblk; i += 32) m = fmaxf(m, blockmax[((size_t)b * nblk + i) * NH + h]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) {
      maxes[1 + t] = m;
      s_row[t] = m;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float g = -INFINITY;
    for (int i = 0; i < B * NH; ++i) g = fmaxf(g, s_row[i]);
    maxes[0] = g;
  }
}

// Pass 2.  grid (nct, B), 256 threads, same strips as pass 1.  exp() of the strip's scores is staged in shared
// memory, then one warp per token: lane = 8 channels, 8x8 fp32 accumulators; warps are folded through shared
// memory in a fixed order.  partial[b, cta, h, 0..C-1] = sum_s e*v, [.., C] = sum_s e.
template <typename T>
__global__ void __launch_bounds__(256)
vlf_pool_kernel(const T *__restrict__ v, const float *__restrict__ scores, const float *__restrict__ maxes,
                float *__restrict__ partial, int S, int NH, int strip, int stable_2d) {
  pdl_prologue();
  constexpr int C = 256;
  __shared__ __align__(16) float s_e[kMaxStrip][kMaxHeads];
  __shared__ __align__(16) float s_red[8][C];
  __shared__ float s_se[8][kMaxHeads];
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s0 = blockIdx.x * strip, n = min(strip, S - s0);
  const float gmax = stable_2d ? maxes[0] : 0.f;
  for (int i = threadIdx.x; i < n * kMaxHeads; i += 256) {
    const int h = i / n, r = i - h * n;  // consecutive threads -> consecutive tokens of one head (coalesced)
    float e = 0.f;
    if (h < NH) {
      const float t = scores[((size_t)b * NH + h) * S + s0 + r];
      const float w = fminf(fmaxf(t - gmax, -50000.f), 50000.f);
      const float rmax = fminf(fmaxf(maxes[1 + b * NH + h] - gmax, -50000.f), 50000.f);
      e = expf(fminf(fmaxf(w - rmax, -50000.f), 50000.f));
    }
    s_e[r][h] = e;
  }
  __syncthreads();
  float acc[kMaxHeads][8], se[kMaxHeads];
#pragma unroll
  for (int h = 0; h < kMaxHeads; ++h) {
    se[h] = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[h][k] = 0.f;
  }
  auto accumulate = [&](const float *f, int r) {
    float e[8];
    load8f(&s_e[r][0], e);
#pragma unroll
    for (int h = 0; h < kMaxHeads; ++h) {
      se[h] += e[h];
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[h][k] = fmaf(e[h], f[k], acc[h][k]);
    }
  };
  for (int r = warp; r < n; r += 16) {  // two rows in flight per warp (same fixed accumulation order: r, then r + 8)
    const bool two = r + 8 < n;
    float f0[8], f1[8];
    load_row8<T>(v + ((size_t)b * S + s0 + r) * C + lane * 8, f0);
    if (two) load_row8<T>(v + ((size_t)b * S + s0 + r + 8) * C + lane * 8, f1);
    accumulate(f0, r);
    if (two) accumulate(f1, r + 8);
  }
  if (lane == 0) {
#pragma unroll
    for (int h = 0; h < kMaxHeads; ++h) s_se[warp][h] = se[h];
  }
  float *dst = partial + ((size_t)b * gridDim.x + blockIdx.x) * NH * (C + 1);
#pragma unroll
  for (int h = 0; h < kMaxHeads; ++h) {
    if (h < NH) {  // CTA-uniform
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 8; ++k) s_red[warp][lane * 8 + k] = acc[h][k];
      __syncthreads();
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += s_red[w][threadIdx.x];
      dst[h * (C + 1) + threadIdx.x] = t;
      if (threadIdx.x == 0) {
        float u = 0.f;
        for (int w = 0; w < 8; ++w) u += s_se[w][h];
        dst[h * (C + 1) + C] = u;
      }
    }
  }
}

int strips_for(int S, int *strip_out) {
  int nct = 132 * 2;  // two strips per SM of an H100 SXM
  int strip = (S + nct - 1) / nct;
  if (strip > kMaxStrip) strip = kMaxStrip;
  if (strip < 8) strip = 8;
  *strip_out = strip;
  return (S + strip - 1) / strip;
}

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int64_t ape_vlf_pool_workspace_bytes(int B, int S, int C, int NH) {
  int strip;
  const int64_t nct = strips_for(S, &strip);
  return ((int64_t)B * NH * S + (int64_t)B * nct * NH + 1 + (int64_t)B * NH + (int64_t)B * nct * NH * (C + 1)) * 4;
}

extern "C" int ape_vlf_pool(const void *v, const float *qa, const float *qc, void *workspace, float **partial_out,
                            int *strips_out, int B, int S, int C, int NH, int stable_softmax_2d, int dtype, void *stream) {
  if (B <= 0 || S <= 0 || NH <= 0 || NH > kMaxHeads || C != 256 || B * NH > 64 || B > 65535)
    return fail(APE_ERR_UNSUPPORTED, "vlf_pool: B=%d S=%d C=%d NH=%d not supported (C must be 256, NH <= 8)", B, S, C, NH);
  if (!v || !qa || !qc || !workspace) return fail(APE_ERR_NULL_PTR, "vlf_pool: null pointer argument");
  if ((reinterpret_cast<uintptr_t>(v) & 15) || (reinterpret_cast<uintptr_t>(qa) & 15))
    return fail(APE_ERR_INVALID_ARG, "vlf_pool: v / qa must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int strip;
  const int nct = strips_for(S, &strip);
  float *scores = reinterpret_cast<float *>(workspace);
  float *blockmax = scores + (size_t)B * NH * S;
  float *maxes = blockmax + (size_t)B * nct * NH;
  float *partial = maxes + 1 + (size_t)B * NH;
  const dim3 grid(nct, B);
  if (dtype == APE_DTYPE_F32) APE_LAUNCH((vlf_scores_kernel<float>), grid, 256, 0, st, (const float *)v, qa, qc, scores, blockmax, S, NH, strip);
  else if (dtype == APE_DTYPE_F16) APE_LAUNCH((vlf_scores_kernel<__half>), grid, 256, 0, st, (const __half *)v, qa, qc, scores, blockmax, S, NH, strip);
  else APE_LAUNCH((vlf_scores_kernel<__nv_bfloat16>), grid, 256, 0, st, (const __nv_bfloat16 *)v, qa, qc, scores, blockmax, S, NH, strip);
  if (int rc = check_launch("vlf_scores_kernel")) return rc;
  APE_LAUNCH((vlf_max_kernel), 1, 1024, 0, st, blockmax, B, nct, NH, maxes);
  if (int rc = check_launch("vlf_max_kernel")) return rc;
  if (dtype == APE_DTYPE_F32) APE_LAUNCH((vlf_pool_kernel<float>), grid, 256, 0, st, (const float *)v, scores, maxes, partial, S, NH, strip, stable_softmax_2d);
  else if (dtype == APE_DTYPE_F16) APE_LAUNCH((vlf_pool_kernel<__half>), grid, 256, 0, st, (const __half *)v, scores, maxes, partial, S, NH, strip, stable_softmax_2d);
  else APE_LAUNCH((vlf_pool_kernel<__nv_bfloat16>), grid, 256, 0, st, (const __nv_bfloat16 *)v, scores, maxes, partial, S, NH, strip, stable_softmax_2d);
  if (partial_out) *partial_out = partial;
  if (strips_out) *strips_out = nct;
  return check_launch("vlf_pool_kernel");
}
