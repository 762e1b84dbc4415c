// semseg.cu — semantic label maps without the class-score maps (DeformableDETRSegmVL._semantic, model.sem_seg_format = "label").
//
// The reference's semantic branch (ape/modeling/ape_deta/deformable_detr_segm_vl.py:875-918 `_postprocess_semantic`, then
// detectron2 sem_seg_postprocess) forms, for the K kept queries of one image,
//   m_q  = sigmoid(resize1(logit_q))                     resize1: mask-logit grid h x w -> padded image Hp x Wp
//   S[c] = sum_q cls[q, c] m_q                           [N, Hp, Wp] fp32 (5 GB at 1203 classes and 1024^2)
//   out  = resize2(S[:, :img_h, :img_w])                 resize2: cropped image -> output size out_h x out_w
// and the evaluator keeps only out.argmax(0).  Both resizes are bilinear (align_corners=False), hence linear, so
//   out[c] = sum_q cls[q, c] A_q,   A_q = resize2(crop(m_q)),
// i.e. one GEMM at the OUTPUT resolution on operands resampled once, with the class argmax taken in its epilogue:
//   semseg_resample_kernel     A [rows * out_w, Kp] 16-bit, pixel-major, for one band of output rows (bounded workspace)
//   gemm_tc_kernel<EpiArgmax>  (gemm_tc.cu, ape_gemm_tn_argmax) A cls^T -> u64 key per pixel (common.cuh argmax_key)
//   semseg_keys_init_kernel    keys <- one constant key ("-inf", or the stuff_prob_thing constant of class 0)
//   semseg_keys_decode_kernel  keys -> int64 label, fp32 score
// Index, clamp and lambda arithmetic is ATen's upsample_bilinear2d (area_pixel_compute_source_index, scale = in / out in fp32).
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "resize.cuh"

namespace ape {
namespace {

// sigmoid(resize1(plane))(Y, X) for the padded-grid point given by its row / column lerps
template <typename TL>
__device__ __forceinline__ float up_sigmoid(const TL *plane, int w, const Lerp &ry, const Lerp &rx) {
  return 1.f / (1.f + expf(-up_value(plane, w, ry, rx)));
}

// the 8 queries of blockIdx.y at output pixel (y, x) -> one 16-byte store into `row`, the pixel's row of A
template <typename TL, typename TO>
__device__ __forceinline__ void resample_px(const TL *__restrict__ logits, const long long *__restrict__ index, TO *__restrict__ row,
                                            int K, int h, int w, float s1h, float s1w, int img_h, int img_w, float s2h, float s2w, int y,
                                            int x) {
  const int k0 = blockIdx.y * 8;
  const Lerp ry = lerp_at(s2h, y, img_h), rx = lerp_at(s2w, x, img_w);  // resize2 over the crop of the padded map
  const Lerp ay0 = lerp_at(s1h, ry.i0, h), ay1 = lerp_at(s1h, ry.i1, h);  // resize1 at the two padded rows it reads
  const Lerp bx0 = lerp_at(s1w, rx.i0, w), bx1 = lerp_at(s1w, rx.i1, w);  // ... and the two padded columns
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] = 0.f;  // pad columns K..Kp
    if (k0 + i < K) {
      const TL *plane = logits + (size_t)__ldg(index + k0 + i) * h * w;
      const float m00 = up_sigmoid(plane, w, ay0, bx0), m01 = up_sigmoid(plane, w, ay0, bx1);
      const float m10 = up_sigmoid(plane, w, ay1, bx0), m11 = up_sigmoid(plane, w, ay1, bx1);
      v[i] = ry.l0 * (rx.l0 * m00 + rx.l1 * m01) + ry.l1 * (rx.l0 * m10 + rx.l1 * m11);
    }
  }
  *reinterpret_cast<uint4 *>(row + k0) = Elem<TO>::pack(v);
}

// A[(y - row0) * out_w + x, k] for output rows [row0, row0 + rows), k < Kp; thread = one pixel x 8 queries (one 16-byte store)
template <typename TL, typename TO>
__global__ void __launch_bounds__(256) semseg_resample_kernel(const TL *__restrict__ logits, const long long *__restrict__ index,
                                                              TO *__restrict__ A, long long lda, int K, int h, int w, float s1h,
                                                              float s1w, int img_h, int img_w, float s2h, float s2w, int out_w,
                                                              int row0, int rows) {
  pdl_prologue();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)rows * out_w) return;
  resample_px(logits, index, A + (size_t)pix * lda, K, h, w, s1h, s1w, img_h, img_w, s2h, s2w, row0 + (int)(pix / out_w),
              (int)(pix % out_w));
}

// The same for a map whose sizes are on the device (ape_semseg_resample_dev): A row i is pixel p0 + i of the row-major
// out_h x out_w map.  Pixels past the map's end return, so the work follows the real size, not the capacity.
template <typename TL, typename TO>
__global__ void __launch_bounds__(256) semseg_resample_dev_kernel(const TL *__restrict__ logits, const long long *__restrict__ index,
                                                                  TO *__restrict__ A, long long lda, int K, int h, int w, float s1h,
                                                                  float s1w, int Hp, int Wp, const int *__restrict__ dims, int cap,
                                                                  long long p0, int n) {
  pdl_prologue();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= n) return;
  const DevSizes d = dev_sizes(dims, Hp, Wp, cap);
  const long long g = p0 + pix;
  if (g >= (long long)d.oh * d.ow) return;
  const float s2h = __fdiv_rn((float)d.ih, (float)d.oh), s2w = __fdiv_rn((float)d.iw, (float)d.ow);  // the host's IEEE divisions
  resample_px(logits, index, A + (size_t)pix * lda, K, h, w, s1h, s1w, d.ih, d.iw, s2h, s2w, (int)(g / d.ow), (int)(g % d.ow));
}

__global__ void __launch_bounds__(256) semseg_keys_init_kernel(unsigned long long *__restrict__ keys, long long n,
                                                               unsigned long long key) {
  pdl_prologue();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) keys[i] = key;
}

// ape_semseg_keys_init_dev: the keys of the map's out_h x out_w pixels, and the number of those pixels in each band of `band`
// (the rows the argmax GEMM of that band reads, ape_gemm_tn_argmax_dev)
__global__ void __launch_bounds__(256) semseg_keys_init_dev_kernel(unsigned long long *__restrict__ keys, const int *__restrict__ dims,
                                                                   int cap, unsigned long long key, long long band, int nbands,
                                                                   int *__restrict__ band_rows) {
  pdl_prologue();
  const DevSizes d = dev_sizes(dims, 1, 1, cap);
  const long long n = (long long)d.oh * d.ow;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) keys[i] = key;
  if (blockIdx.x == 0)
    for (int t = threadIdx.x; t < nbands; t += blockDim.x) band_rows[t] = (int)max(0LL, min(band, n - t * band));
}

// dims (ape_semseg_keys_decode_dev): n is the map's out_h x out_w from the device, within the capacity n
__global__ void __launch_bounds__(256) semseg_keys_decode_kernel(const unsigned long long *__restrict__ keys, long long n,
                                                                 long long *__restrict__ label, float *__restrict__ score,
                                                                 const int *__restrict__ dims, int cap) {
  pdl_prologue();
  if (dims) {
    const DevSizes d = dev_sizes(dims, 1, 1, cap);
    n = min(n, (long long)d.oh * d.ow);
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    label[i] = (long long)(0xFFFFFFFFu - (uint32_t)k);
    score[i] = argmax_key_value(k);
  }
}

template <typename TL, typename TO>
void launch_resample(dim3 grid, cudaStream_t st, const void *logits, const int64_t *index, void *A, long long lda, int K, int h,
                     int w, float s1h, float s1w, int img_h, int img_w, float s2h, float s2w, int out_w, int row0, int rows) {
  auto kernel = semseg_resample_kernel<TL, TO>;
  APE_LAUNCH(kernel, grid, 256, 0, st, (const TL *)logits, (const long long *)index, (TO *)A, lda, K, h, w,
             s1h, s1w, img_h, img_w, s2h, s2w, out_w, row0, rows);
}

int grid_1d(long long n) { return (int)std::min<long long>((n + 255) / 256, 132LL * 16); }

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int ape_semseg_resample(const void *logits, const int64_t *index, void *A, int64_t lda, int K, int h, int w, int Hp,
                                   int Wp, int img_h, int img_w, int out_h, int out_w, int row0, int rows, int logit_dtype,
                                   int a_dtype, void *stream) {
  if (logit_dtype != APE_DTYPE_F32 && logit_dtype != APE_DTYPE_F16 && logit_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "semseg_resample: logit dtype %d", logit_dtype);
  if (a_dtype != APE_DTYPE_F16 && a_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "semseg_resample: the operand must be fp16 or bf16 (got dtype %d)", a_dtype);
  if (K <= 0 || h <= 0 || w <= 0 || Hp <= 0 || Wp <= 0 || img_h <= 0 || img_w <= 0 || img_h > Hp || img_w > Wp || out_h <= 0 ||
      out_w <= 0 || row0 < 0 || rows <= 0 || (long long)row0 + rows > out_h)
    return fail(APE_ERR_INVALID_ARG, "semseg_resample: bad geometry K=%d logits %dx%d, padded %dx%d, image %dx%d, output %dx%d, rows %d+%d",
                K, h, w, Hp, Wp, img_h, img_w, out_h, out_w, row0, rows);
  const int Kp = (K + 7) / 8 * 8;
  if (Kp / 8 > 65535 || (long long)rows * out_w > 0x7fffffffLL)
    return fail(APE_ERR_INVALID_ARG, "semseg_resample: band too large (K=%d, %d x %d pixels)", K, rows, out_w);
  if (lda < Kp || lda % 8) return fail(APE_ERR_INVALID_ARG, "semseg_resample: row pitch %lld must be >= %d and a multiple of 8", (long long)lda, Kp);
  if (!logits || !index || !A) return fail(APE_ERR_NULL_PTR, "semseg_resample: null pointer");
  if (reinterpret_cast<uintptr_t>(A) & 15) return fail(APE_ERR_INVALID_ARG, "semseg_resample: A must be 16-byte aligned");
  const float s1h = (float)h / (float)Hp, s1w = (float)w / (float)Wp;              // area_pixel_compute_scale
  const float s2h = (float)img_h / (float)out_h, s2w = (float)img_w / (float)out_w;
  const dim3 grid((unsigned)(((long long)rows * out_w + 255) / 256), (unsigned)(Kp / 8));
  cudaStream_t st = (cudaStream_t)stream;
#define APE_SEMSEG_RESAMPLE(TL, TO) \
  launch_resample<TL, TO>(grid, st, logits, index, A, lda, K, h, w, s1h, s1w, img_h, img_w, s2h, s2w, out_w, row0, rows)
  if (a_dtype == APE_DTYPE_F16) {
    if (logit_dtype == APE_DTYPE_F32) APE_SEMSEG_RESAMPLE(float, __half);
    else if (logit_dtype == APE_DTYPE_F16) APE_SEMSEG_RESAMPLE(__half, __half);
    else APE_SEMSEG_RESAMPLE(__nv_bfloat16, __half);
  } else {
    if (logit_dtype == APE_DTYPE_F32) APE_SEMSEG_RESAMPLE(float, __nv_bfloat16);
    else if (logit_dtype == APE_DTYPE_F16) APE_SEMSEG_RESAMPLE(__half, __nv_bfloat16);
    else APE_SEMSEG_RESAMPLE(__nv_bfloat16, __nv_bfloat16);
  }
#undef APE_SEMSEG_RESAMPLE
  return check_launch("semseg_resample_kernel");
}

extern "C" int ape_semseg_keys_init(uint64_t *keys, int64_t n, float value, int column, void *stream) {
  if (n < 0 || column < 0) return fail(APE_ERR_INVALID_ARG, "semseg_keys_init: bad n=%lld column=%d", (long long)n, column);
  if (n == 0) return APE_OK;
  if (!keys) return fail(APE_ERR_NULL_PTR, "semseg_keys_init: null pointer");
  if (reinterpret_cast<uintptr_t>(keys) & 7) return fail(APE_ERR_INVALID_ARG, "semseg_keys_init: keys must be 8-byte aligned");
  const float v = value + 0.f;
  uint32_t u;
  memcpy(&u, &v, 4);
  APE_LAUNCH(semseg_keys_init_kernel, grid_1d(n), 256, 0, (cudaStream_t)stream, (unsigned long long *)keys, (long long)n,
             argmax_key_bits(u, (uint32_t)column));
  return check_launch("semseg_keys_init_kernel");
}

extern "C" int ape_semseg_keys_decode(const uint64_t *keys, int64_t n, int64_t *label, float *score, void *stream) {
  if (n < 0) return fail(APE_ERR_INVALID_ARG, "semseg_keys_decode: bad n=%lld", (long long)n);
  if (n == 0) return APE_OK;
  if (!keys || !label || !score) return fail(APE_ERR_NULL_PTR, "semseg_keys_decode: null pointer");
  if ((reinterpret_cast<uintptr_t>(keys) | reinterpret_cast<uintptr_t>(label)) & 7 || reinterpret_cast<uintptr_t>(score) & 3)
    return fail(APE_ERR_INVALID_ARG, "semseg_keys_decode: misaligned buffers");
  APE_LAUNCH(semseg_keys_decode_kernel, grid_1d(n), 256, 0, (cudaStream_t)stream, (const unsigned long long *)keys, (long long)n,
             (long long *)label, score, (const int *)nullptr, 0);
  return check_launch("semseg_keys_decode_kernel");
}

// ---- device-held sizes ------------------------------------------------------------------------------------------------------
extern "C" int ape_semseg_resample_dev(const void *logits, const int64_t *index, void *A, int64_t lda, int K, int h, int w, int Hp,
                                       int Wp, const int *sizes, int cap, int64_t p0, int n, int logit_dtype, int a_dtype, void *stream) {
  if (logit_dtype != APE_DTYPE_F32 && logit_dtype != APE_DTYPE_F16 && logit_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "semseg_resample_dev: logit dtype %d", logit_dtype);
  if (a_dtype != APE_DTYPE_F16 && a_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "semseg_resample_dev: the operand must be fp16 or bf16 (got dtype %d)", a_dtype);
  if (K <= 0 || h <= 0 || w <= 0 || Hp <= 0 || Wp <= 0 || cap <= 0 || (long long)cap * cap > (1LL << 30) || p0 < 0 || n <= 0 ||
      p0 + n > (long long)cap * cap)
    return fail(APE_ERR_INVALID_ARG, "semseg_resample_dev: bad geometry K=%d logits %dx%d, padded %dx%d, capacity %d, pixels %lld+%d",
                K, h, w, Hp, Wp, cap, (long long)p0, n);
  const int Kp = (K + 7) / 8 * 8;
  if (Kp / 8 > 65535) return fail(APE_ERR_INVALID_ARG, "semseg_resample_dev: K=%d too large", K);
  if (lda < Kp || lda % 8) return fail(APE_ERR_INVALID_ARG, "semseg_resample_dev: row pitch %lld must be >= %d and a multiple of 8", (long long)lda, Kp);
  if (!logits || !index || !A || !sizes) return fail(APE_ERR_NULL_PTR, "semseg_resample_dev: null pointer");
  if (reinterpret_cast<uintptr_t>(A) & 15) return fail(APE_ERR_INVALID_ARG, "semseg_resample_dev: A must be 16-byte aligned");
  const float s1h = (float)h / (float)Hp, s1w = (float)w / (float)Wp;  // area_pixel_compute_scale
  const dim3 grid((unsigned)((n + 255) / 256), (unsigned)(Kp / 8));
  cudaStream_t st = (cudaStream_t)stream;
#define APE_SEMSEG_RESAMPLE_DEV(TL, TO)                                                                                          \
  APE_LAUNCH((semseg_resample_dev_kernel<TL, TO>), grid, 256, 0, st, (const TL *)logits, (const long long *)index, (TO *)A,     \
             (long long)lda, K, h, w, s1h, s1w, Hp, Wp, sizes, cap, (long long)p0, n)
  if (a_dtype == APE_DTYPE_F16) {
    if (logit_dtype == APE_DTYPE_F32) APE_SEMSEG_RESAMPLE_DEV(float, __half);
    else if (logit_dtype == APE_DTYPE_F16) APE_SEMSEG_RESAMPLE_DEV(__half, __half);
    else APE_SEMSEG_RESAMPLE_DEV(__nv_bfloat16, __half);
  } else {
    if (logit_dtype == APE_DTYPE_F32) APE_SEMSEG_RESAMPLE_DEV(float, __nv_bfloat16);
    else if (logit_dtype == APE_DTYPE_F16) APE_SEMSEG_RESAMPLE_DEV(__half, __nv_bfloat16);
    else APE_SEMSEG_RESAMPLE_DEV(__nv_bfloat16, __nv_bfloat16);
  }
#undef APE_SEMSEG_RESAMPLE_DEV
  return check_launch("semseg_resample_dev_kernel");
}

extern "C" int ape_semseg_keys_init_dev(uint64_t *keys, const int *sizes, int cap, float value, int column, int64_t band, int nbands,
                                        int *band_rows, void *stream) {
  if (cap <= 0 || (long long)cap * cap > (1LL << 30) || column < 0 || band <= 0 || nbands <= 0 || band * nbands < (long long)cap * cap)
    return fail(APE_ERR_INVALID_ARG, "semseg_keys_init_dev: bad capacity %d, column %d, %d bands of %lld", cap, column, nbands,
                (long long)band);
  if (!keys || !sizes || !band_rows) return fail(APE_ERR_NULL_PTR, "semseg_keys_init_dev: null pointer");
  if (reinterpret_cast<uintptr_t>(keys) & 7) return fail(APE_ERR_INVALID_ARG, "semseg_keys_init_dev: keys must be 8-byte aligned");
  const float v = value + 0.f;
  uint32_t u;
  memcpy(&u, &v, 4);
  APE_LAUNCH(semseg_keys_init_dev_kernel, grid_1d((long long)cap * cap), 256, 0, (cudaStream_t)stream, (unsigned long long *)keys,
             sizes, cap, argmax_key_bits(u, (uint32_t)column), (long long)band, nbands, band_rows);
  return check_launch("semseg_keys_init_dev_kernel");
}

extern "C" int ape_semseg_keys_decode_dev(const uint64_t *keys, const int *sizes, int cap, int64_t *label, float *score, void *stream) {
  if (cap <= 0 || (long long)cap * cap > (1LL << 30)) return fail(APE_ERR_INVALID_ARG, "semseg_keys_decode_dev: capacity %d", cap);
  if (!keys || !sizes || !label || !score) return fail(APE_ERR_NULL_PTR, "semseg_keys_decode_dev: null pointer");
  if ((reinterpret_cast<uintptr_t>(keys) | reinterpret_cast<uintptr_t>(label)) & 7 || reinterpret_cast<uintptr_t>(score) & 3)
    return fail(APE_ERR_INVALID_ARG, "semseg_keys_decode_dev: misaligned buffers");
  const long long n = (long long)cap * cap;
  APE_LAUNCH(semseg_keys_decode_kernel, grid_1d(n), 256, 0, (cudaStream_t)stream, (const unsigned long long *)keys, n,
             (long long *)label, score, sizes, cap);
  return check_launch("semseg_keys_decode_kernel");
}
