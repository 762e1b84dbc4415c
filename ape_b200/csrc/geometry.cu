// geometry.cu — the per-image-size geometry of the deformable transformer, built on the device from the image sizes.
//
// The padded batch has a fixed shape (Hp, Wp) and fixed level shapes; only the valid (h, w) of each image changes from call to
// call.  ape_pad_geometry turns those sizes, held in device memory, into everything DeformableDetrTransformerVL.geometry returns
// that depends on them, so a CUDA graph captured once serves every image size that fits the padded shape.  Each output restates
// the torch code it replaces with the same fp32 operations in the same order (see include/ape_b200.h); the file is compiled
// without fast-math, so divisions are IEEE and sinf / cosf / logf are the precise ones torch's kernels call.
#include "common.cuh"

namespace {

constexpr int kMaxLevels = 8;
constexpr int kTok = 32;  // tokens per CTA
constexpr int kThreads = 256;

struct Levels {
  int h[kMaxLevels], w[kMaxLevels], start[kMaxLevels];
  int L, S;
};

// Rows (or columns) of a level whose nearest source pixel lies inside the image: F.interpolate(mode="nearest") maps destination
// index i to min(floor(i * (float)in / out), in - 1) (upsample_nearest2d's nearest_neighbor_compute_source_index).  The map is
// non-decreasing in i, so the valid indices are a prefix and this is its length.
__device__ int nearest_valid(int in, int out, int valid) {
  const float scale = (float)in / (float)out;
  int n = 0;
  for (int i = 0; i < out; ++i) n += min((int)floorf((float)i * scale), in - 1) < valid;
  return n;
}

template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void __launch_bounds__(kThreads) pad_geometry_kernel(
    const int *__restrict__ sizes, int Hp, int Wp, Levels lv, const float *__restrict__ dim_t, const float *__restrict__ level_embeds,
    int E, float offset, float eps, float scale, int normalize, uint8_t *__restrict__ mask_flatten, T *__restrict__ pos_lvl,
    float *__restrict__ pos_flatten, float *__restrict__ valid_ratios, float *__restrict__ reference_points,
    float *__restrict__ output_proposals, uint8_t *__restrict__ proposal_invalid) {
  __shared__ int s_vh[kMaxLevels], s_vw[kMaxLevels];
  __shared__ float s_rw[kMaxLevels], s_rh[kMaxLevels];
  __shared__ int s_lvl[kTok], s_i[kTok], s_j[kTok];
  ape::pdl_prologue();
  const int b = blockIdx.y, L = lv.L, S = lv.S, tid = threadIdx.x;
  // the sizes only change values, never addresses: clamped to [1, Hp] x [1, Wp]
  const int h = min(max(sizes[2 * b], 1), Hp), w = min(max(sizes[2 * b + 1], 1), Wp);
  if (tid < 2 * L) {
    const int l = tid >> 1;
    if (tid & 1)
      s_vw[l] = nearest_valid(Wp, lv.w[l], w);
    else
      s_vh[l] = nearest_valid(Hp, lv.h[l], h);
  }
  const int tok0 = blockIdx.x * kTok;
  if (tid < kTok && tok0 + tid < S) {
    const int s = tok0 + tid;
    int l = 0;
    while (l + 1 < L && s >= lv.start[l + 1]) ++l;
    s_lvl[tid] = l;
    s_i[tid] = (s - lv.start[l]) / lv.w[l];
    s_j[tid] = (s - lv.start[l]) % lv.w[l];
  }
  __syncthreads();
  if (tid < L) {  // get_valid_ratio: sum(~mask).float() / W, which torch computes as a product with the scalar's reciprocal
    s_rw[tid] = (float)s_vw[tid] * (1.f / (float)lv.w[tid]);
    s_rh[tid] = (float)s_vh[tid] * (1.f / (float)lv.h[tid]);
    if (blockIdx.x == 0) {
      valid_ratios[((long long)b * L + tid) * 2 + 0] = s_rw[tid];
      valid_ratios[((long long)b * L + tid) * 2 + 1] = s_rh[tid];
    }
  }
  __syncthreads();
  const int ntok = min(kTok, S - tok0);

  // per token: padding mask, reference points, anchor proposal
  if (tid < ntok) {
    const int l = s_lvl[tid], i = s_i[tid], j = s_j[tid];
    const long long bs = (long long)b * S + tok0 + tid;
    const bool pad = !(i < s_vh[l] && j < s_vw[l]);
    mask_flatten[bs] = pad;
    // get_reference_points: linspace(0.5, n - 0.5, n) is i + 0.5 exactly (its step is exactly 1), / (valid ratio * n),
    // then times the valid ratios of every level
    const float rx = ((float)j + 0.5f) / (s_rw[l] * (float)lv.w[l]);
    const float ry = ((float)i + 0.5f) / (s_rh[l] * (float)lv.h[l]);
    float2 *ref = reinterpret_cast<float2 *>(reference_points) + bs * L;
    for (int k = 0; k < L; ++k) ref[k] = make_float2(rx * s_rw[k], ry * s_rh[k]);
    // geometry()'s anchors: (linspace(0, n - 1, n) + 0.5) / valid count, wh = 0.05 * 2^lvl, the (0.01, 0.99) test on all four,
    // log(p / (1 - p)), inf where padded or invalid
    float p[4];
    p[0] = ((float)j + 0.5f) / (float)s_vw[l];
    p[1] = ((float)i + 0.5f) / (float)s_vh[l];
    p[2] = p[3] = 0.05f * (float)(1 << l);
    bool ok = true;
    for (int k = 0; k < 4; ++k) ok = ok && p[k] > 0.01f && p[k] < 0.99f;
    const bool invalid = pad || !ok;
    float4 o;
    o.x = invalid ? INFINITY : logf(p[0] / (1.f - p[0]));
    o.y = invalid ? INFINITY : logf(p[1] / (1.f - p[1]));
    o.z = invalid ? INFINITY : logf(p[2] / (1.f - p[2]));
    o.w = invalid ? INFINITY : logf(p[3] / (1.f - p[3]));
    reinterpret_cast<float4 *>(output_proposals)[bs] = o;
    proposal_invalid[bs] = invalid;
  }

  // per (token, channel pair): PositionEmbeddingSine of the level's mask, + level embedding.  The mask is a rectangle of vh valid
  // rows and vw valid columns, so the cumulative sums are closed forms: y = min(i + 1, vh) in a valid column (0 in a padded one),
  // its last row vh (0); x likewise.
  const int F = E / 2, P = E / 2;
  for (int idx = tid; idx < ntok * P; idx += kThreads) {
    const int t = idx / P, c = 2 * (idx - t * P);  // channels c, c + 1: sin and cos of one dim_t pair
    const int l = s_lvl[t], i = s_i[t], j = s_j[t];
    const int vh = s_vh[l], vw = s_vw[l];
    const bool yaxis = c < F;
    const int k = yaxis ? c : c - F;
    float v, last;
    if (yaxis) {
      v = j < vw ? (float)min(i + 1, vh) : 0.f;
      last = j < vw ? (float)vh : 0.f;
    } else {
      v = i < vh ? (float)min(j + 1, vw) : 0.f;
      last = i < vh ? (float)vw : 0.f;
    }
    if (normalize) v = (v + offset) / (last + eps) * scale;
    // dim_t[k + 1] == dim_t[k] (the table pairs its entries), so one quotient serves the sine and the cosine
    const float q = v / dim_t[k];
    const float e0 = sinf(q), e1 = cosf(q);
    const long long o = ((long long)b * S + tok0 + t) * E + c;
    if (pos_flatten) *reinterpret_cast<float2 *>(pos_flatten + o) = make_float2(e0, e1);
    const float *lvl = level_embeds + (long long)l * E + c;
    pos_lvl[o] = from_f32<T>(e0 + lvl[0]);
    pos_lvl[o + 1] = from_f32<T>(e1 + lvl[1]);
  }
}

// One warp per row: a row whose mask byte is set is overwritten with +0.0; the others are not touched, so an all-false mask costs
// the read of the mask alone.
template <typename T>
__global__ void __launch_bounds__(kThreads) zero_masked_rows_kernel(T *__restrict__ x, long long ld, const uint8_t *__restrict__ mask,
                                                                    long long rows, int cols) {
  ape::pdl_prologue();
  const long long r = (long long)blockIdx.x * (kThreads / 32) + threadIdx.x / 32;
  if (r >= rows || !mask[r]) return;
  T *row = x + r * ld;
  for (int c = threadIdx.x % 32; c < cols; c += 32) row[c] = T(0);
}

// Phase one of the region prompt: *empty is 1 on entry (set by the launcher); any CTA that finds a set byte of the map writes 0.
// Every writer writes the same value, so the result does not depend on the order.
__global__ void __launch_bounds__(kThreads) region_empty_kernel(const uint8_t *__restrict__ map, long long n, uint8_t *__restrict__ empty) {
  ape::pdl_prologue();
  const long long n16 = n / 16, stride = (long long)gridDim.x * kThreads;
  bool set = false;
  const uint4 *v = reinterpret_cast<const uint4 *>(map);
  for (long long k = (long long)blockIdx.x * kThreads + threadIdx.x; k < n16; k += stride) {
    const uint4 q = v[k];
    set |= (q.x | q.y | q.z | q.w) != 0u;
  }
  for (long long k = n16 * 16 + (long long)blockIdx.x * kThreads + threadIdx.x; k < n; k += stride) set |= map[k] != 0;
  if (__syncthreads_or(set) && threadIdx.x == 0) *empty = 0;
}

struct RegionLevels {
  int h[kMaxLevels], w[kMaxLevels], start[kMaxLevels];
  float sh[kMaxLevels], sw[kMaxLevels];  // (float)Hp / h_l and (float)Wp / w_l, divided on the host (IEEE, as torch's host code)
  int L, S;
};

// The two source taps of destination index d along one axis of F.interpolate(mode="bilinear", align_corners=False), with the
// fp32 operations of torch's CUDA kernel (upsample_bilinear2d_out_frame: FADD d + 0.5, FFMA by the scale minus 0.5, clamp at 0,
// truncate, lambda = src - index): the first tap always has a nonzero weight (1 - lambda > 0); the second counts when lambda is
// nonzero, and is the first again at the last source row or column.
__device__ __forceinline__ void bilinear_taps(int d, float scale, int n_in, int &t0, int &t1) {
  float src = __fmaf_rn((float)d + 0.5f, scale, -0.5f);
  src = src < 0.f ? 0.f : src;
  const int i = min((int)src, n_in - 1);
  const float lambda = src - (float)i;
  t0 = i;
  t1 = lambda != 0.f && i < n_in - 1 ? i + 1 : i;
}

// One thread per token: region = the whole batch is empty, or a tap with nonzero weight reads a set byte of the image's map.
__global__ void __launch_bounds__(kThreads) region_prompt_kernel(const uint8_t *__restrict__ map, int Hp, int Wp, RegionLevels lv,
                                                                 const uint8_t *__restrict__ empty,
                                                                 const float *__restrict__ output_proposals,
                                                                 const uint8_t *__restrict__ proposal_invalid,
                                                                 float *__restrict__ out_proposals, uint8_t *__restrict__ out_invalid,
                                                                 uint8_t *__restrict__ region) {
  ape::pdl_prologue();
  const int s = blockIdx.x * kThreads + threadIdx.x, b = blockIdx.y;
  if (s >= lv.S) return;
  int l = 0;
  while (l + 1 < lv.L && s >= lv.start[l + 1]) ++l;
  const int i = (s - lv.start[l]) / lv.w[l], j = (s - lv.start[l]) % lv.w[l];
  bool in = *empty != 0;
  if (!in) {
    int r0, r1, c0, c1;
    bilinear_taps(i, lv.sh[l], Hp, r0, r1);
    bilinear_taps(j, lv.sw[l], Wp, c0, c1);
    const uint8_t *m = map + (long long)b * Hp * Wp;
    in = (m[(long long)r0 * Wp + c0] | m[(long long)r0 * Wp + c1] | m[(long long)r1 * Wp + c0] | m[(long long)r1 * Wp + c1]) != 0;
  }
  const long long bs = (long long)b * lv.S + s;
  const float4 p = reinterpret_cast<const float4 *>(output_proposals)[bs];
  reinterpret_cast<float4 *>(out_proposals)[bs] = in ? p : make_float4(INFINITY, INFINITY, INFINITY, INFINITY);
  out_invalid[bs] = proposal_invalid[bs] | !in;
  if (region) region[bs] = in;
}

}  // namespace

using namespace ape;

extern "C" int ape_pad_geometry(const int *sizes, int B, int Hp, int Wp, const int *level_hw, int L, const float *dim_t,
                                const float *level_embeds, int E, float offset, float eps, float scale, int normalize,
                                uint8_t *mask_flatten, void *pos_lvl, int pos_dtype, float *pos_flatten, float *valid_ratios,
                                float *reference_points, float *output_proposals, uint8_t *proposal_invalid, void *stream) {
  if (B <= 0) return fail(APE_ERR_INVALID_ARG, "pad_geometry: B=%d", B);
  if (L < 1 || L > kMaxLevels) return fail(APE_ERR_INVALID_ARG, "pad_geometry: L=%d outside [1, %d]", L, kMaxLevels);
  if (Hp <= 0 || Wp <= 0) return fail(APE_ERR_INVALID_ARG, "pad_geometry: padded shape %dx%d", Hp, Wp);
  if (E <= 0 || E % 2) return fail(APE_ERR_INVALID_ARG, "pad_geometry: E=%d must be even and positive", E);
  if (!level_hw) return fail(APE_ERR_NULL_PTR, "pad_geometry: null level shapes");
  if (pos_dtype != APE_DTYPE_F32 && pos_dtype != APE_DTYPE_F16 && pos_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_UNSUPPORTED, "pad_geometry: pos dtype %d (fp32 / fp16 / bf16 only)", pos_dtype);
  if (!sizes || !dim_t || !level_embeds || !mask_flatten || !pos_lvl || !valid_ratios || !reference_points || !output_proposals ||
      !proposal_invalid)
    return fail(APE_ERR_NULL_PTR, "pad_geometry: null pointer");
  Levels lv{};
  lv.L = L;
  long long S = 0;
  for (int l = 0; l < L; ++l) {
    const int h = level_hw[2 * l], w = level_hw[2 * l + 1];
    if (h < 1 || h > Hp || w < 1 || w > Wp)
      return fail(APE_ERR_INVALID_ARG, "pad_geometry: level %d of %dx%d does not fit the %dx%d padded shape", l, h, w, Hp, Wp);
    lv.h[l] = h;
    lv.w[l] = w;
    lv.start[l] = (int)S;
    S += (long long)h * w;
  }
  if (S * E > INT32_MAX) return fail(APE_ERR_INVALID_ARG, "pad_geometry: %lld tokens x %d channels", S, E);
  if ((reinterpret_cast<uintptr_t>(pos_flatten) & 7) || (reinterpret_cast<uintptr_t>(reference_points) & 7) ||
      (reinterpret_cast<uintptr_t>(output_proposals) & 15))
    return fail(APE_ERR_INVALID_ARG, "pad_geometry: pos_flatten / reference_points must be 8-byte, output_proposals 16-byte aligned");
  lv.S = (int)S;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)((S + kTok - 1) / kTok), (unsigned)B);
  if (pos_dtype == APE_DTYPE_F16)
    APE_LAUNCH(pad_geometry_kernel<__half>, grid, kThreads, 0, st, sizes, Hp, Wp, lv, dim_t, level_embeds, E, offset, eps, scale,
               normalize, mask_flatten, reinterpret_cast<__half *>(pos_lvl), pos_flatten, valid_ratios, reference_points,
               output_proposals, proposal_invalid);
  else if (pos_dtype == APE_DTYPE_BF16)
    APE_LAUNCH(pad_geometry_kernel<__nv_bfloat16>, grid, kThreads, 0, st, sizes, Hp, Wp, lv, dim_t, level_embeds, E, offset, eps,
               scale, normalize, mask_flatten, reinterpret_cast<__nv_bfloat16 *>(pos_lvl), pos_flatten, valid_ratios,
               reference_points, output_proposals, proposal_invalid);
  else
    APE_LAUNCH(pad_geometry_kernel<float>, grid, kThreads, 0, st, sizes, Hp, Wp, lv, dim_t, level_embeds, E, offset, eps, scale,
               normalize, mask_flatten, reinterpret_cast<float *>(pos_lvl), pos_flatten, valid_ratios, reference_points,
               output_proposals, proposal_invalid);
  return check_launch("pad_geometry_kernel");
}

extern "C" int ape_zero_masked_rows(void *x, int64_t ld, const uint8_t *mask, int64_t rows, int cols, int dtype, void *stream) {
  if (rows < 0 || cols < 0 || ld < cols) return fail(APE_ERR_INVALID_ARG, "zero_masked_rows: rows %lld, cols %d, ld %lld", (long long)rows,
                                                     cols, (long long)ld);
  if (rows == 0 || cols == 0) return APE_OK;
  if (!x || !mask) return fail(APE_ERR_NULL_PTR, "zero_masked_rows: null pointer");
  const unsigned grid = (unsigned)((rows + kThreads / 32 - 1) / (kThreads / 32));
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == APE_DTYPE_F32)
    APE_LAUNCH(zero_masked_rows_kernel<uint32_t>, grid, kThreads, 0, st, reinterpret_cast<uint32_t *>(x), (long long)ld, mask,
               (long long)rows, cols);
  else if (dtype == APE_DTYPE_F16 || dtype == APE_DTYPE_BF16)
    APE_LAUNCH(zero_masked_rows_kernel<uint16_t>, grid, kThreads, 0, st, reinterpret_cast<uint16_t *>(x), (long long)ld, mask,
               (long long)rows, cols);
  else
    return fail(APE_ERR_UNSUPPORTED, "zero_masked_rows: dtype %d (fp32 / fp16 / bf16 only)", dtype);
  return check_launch("zero_masked_rows_kernel");
}

extern "C" int ape_region_prompt_empty(const uint8_t *map, int64_t n, uint8_t *empty, void *stream) {
  if (n < 0) return fail(APE_ERR_INVALID_ARG, "region_prompt_empty: n=%lld", (long long)n);
  if (!empty || (n > 0 && !map)) return fail(APE_ERR_NULL_PTR, "region_prompt_empty: null pointer");
  if (reinterpret_cast<uintptr_t>(map) & 15) return fail(APE_ERR_INVALID_ARG, "region_prompt_empty: map must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(empty, 1, 1, st);
  if (e != cudaSuccess) return fail((int)e, "region_prompt_empty: %s", cudaGetErrorString(e));
  if (n == 0) return APE_OK;
  // 16 bytes per thread and pass; enough CTAs to fill the SMs a few times over, fewer for a small map
  const long long per_cta = 16LL * kThreads * 4;
  const long long ctas = (n + per_cta - 1) / per_cta;
  const unsigned grid = (unsigned)(ctas < 1024 ? ctas : 1024);
  APE_LAUNCH(region_empty_kernel, grid, kThreads, 0, st, map, (long long)n, empty);
  return check_launch("region_empty_kernel");
}

extern "C" int ape_region_prompt(const uint8_t *map, int B, int Hp, int Wp, const int *level_hw, int L, const uint8_t *empty,
                                 const float *output_proposals, const uint8_t *proposal_invalid, float *out_proposals,
                                 uint8_t *out_invalid, uint8_t *region, void *stream) {
  if (B <= 0 || B > 65535) return fail(APE_ERR_INVALID_ARG, "region_prompt: B=%d outside [1, 65535]", B);
  if (L < 1 || L > kMaxLevels) return fail(APE_ERR_INVALID_ARG, "region_prompt: L=%d outside [1, %d]", L, kMaxLevels);
  if (Hp <= 0 || Wp <= 0) return fail(APE_ERR_INVALID_ARG, "region_prompt: padded shape %dx%d", Hp, Wp);
  if (!level_hw) return fail(APE_ERR_NULL_PTR, "region_prompt: null level shapes");
  if (!map || !empty || !output_proposals || !proposal_invalid || !out_proposals || !out_invalid)
    return fail(APE_ERR_NULL_PTR, "region_prompt: null pointer");
  if ((reinterpret_cast<uintptr_t>(output_proposals) & 15) || (reinterpret_cast<uintptr_t>(out_proposals) & 15))
    return fail(APE_ERR_INVALID_ARG, "region_prompt: output_proposals / out_proposals must be 16-byte aligned");
  RegionLevels lv{};
  lv.L = L;
  long long S = 0;
  for (int l = 0; l < L; ++l) {
    const int h = level_hw[2 * l], w = level_hw[2 * l + 1];
    if (h < 1 || h > Hp || w < 1 || w > Wp)
      return fail(APE_ERR_INVALID_ARG, "region_prompt: level %d of %dx%d does not fit the %dx%d padded shape", l, h, w, Hp, Wp);
    lv.h[l] = h;
    lv.w[l] = w;
    lv.start[l] = (int)S;
    lv.sh[l] = (float)Hp / (float)h;
    lv.sw[l] = (float)Wp / (float)w;
    S += (long long)h * w;
  }
  if (S > INT32_MAX / 4) return fail(APE_ERR_INVALID_ARG, "region_prompt: %lld tokens", S);
  lv.S = (int)S;
  const dim3 grid((unsigned)((S + kThreads - 1) / kThreads), (unsigned)B);
  APE_LAUNCH(region_prompt_kernel, grid, kThreads, 0, (cudaStream_t)stream, map, Hp, Wp, lv, empty, output_proposals,
             proposal_invalid, out_proposals, out_invalid, region);
  return check_launch("region_prompt_kernel");
}
