// norm_rope.cu — row-wise kernels around the tensor-core GEMMs of the ViT / transformer blocks:
//   * LayerNorm over the last dim (fp32 statistics, 16-bit or fp32 IO, optional row gather so that
//     window partition / un-partition (utils_eva02.py:19-63) costs no extra pass),
//   * 2-D rotary embedding applied in place to the q and k thirds of a fused [M, 3C] qkv buffer
//     (VisionRotaryEmbeddingFast, utils_eva02.py:307-346; rotate_half :248-252).
// All HBM-bound: one warp per row, 128-bit loads, data held in registers between the two passes.
#include <cuda_fp8.h>

#include "common.cuh"

namespace ape {
namespace {

template <typename T>
struct Vec8 {  // 8 elements of T as raw storage
  static constexpr int kBytes = 8 * sizeof(T);
};

template <typename T>
__device__ __forceinline__ void load8(const T *p, float *f) {
  if constexpr (sizeof(T) == 4) {
    const float4 a = *reinterpret_cast<const float4 *>(p), b = *reinterpret_cast<const float4 *>(p + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  } else {
    const uint4 v = *reinterpret_cast<const uint4 *>(p);
    Elem<T>::unpack(v, f);
  }
}
template <typename T>
__device__ __forceinline__ void store8(T *p, const float *f) {
  if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4 *>(p) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4 *>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
  } else {
    *reinterpret_cast<uint4 *>(p) = Elem<T>::pack(f);
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per row.  MAXV = max 8-element vectors per lane (C <= 256 * MAXV).
// y[out_row(r)] = LN(x[r]) * w + b;  out_row = gather ? row_map[r] : r.
template <typename TI, typename TO, int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const TI *__restrict__ x, long long ldx, TO *__restrict__ y, long long ldy,
                 const float *__restrict__ w, const float *__restrict__ b, const int *__restrict__ row_map,
                 int rows, int C, float eps) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const TI *xr = x + (size_t)warp * ldx;
  // rows are padded to a multiple of 8 elements (host-checked pitch); elements >= C are ignored on
  // input and written as 0 (keeps the K-padding of the next GEMM's operand clean, e.g. C = 2730)
  const int nvec = (C + 7) >> 3;
  float v[MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
      load8<TI>(xr + 8 * j, v[i]);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (8 * j + k >= C) v[i][k] = 0.f;
        sum += v[i][k];
      }
    }
  }
  const float mean = warp_sum(sum) / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = (8 * j + k < C) ? v[i][k] - mean : 0.f;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
  const int orow = row_map ? row_map[warp] : warp;
  TO *yr = y + (size_t)orow * ldy;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
      float o[8];
      if (8 * j + 8 <= C) {
        const float4 w0 = __ldg(reinterpret_cast<const float4 *>(w + 8 * j)), w1 = __ldg(reinterpret_cast<const float4 *>(w + 8 * j) + 1);
        const float4 b0 = __ldg(reinterpret_cast<const float4 *>(b + 8 * j)), b1 = __ldg(reinterpret_cast<const float4 *>(b + 8 * j) + 1);
        const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = (v[i][k] - mean) * rstd * ww[k] + bb[k];
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k)
          o[k] = (8 * j + k < C) ? (v[i][k] - mean) * rstd * __ldg(w + 8 * j + k) + __ldg(b + 8 * j + k) : 0.f;
      }
      store8<TO>(yr + 8 * j, o);
    }
  }
}

// layernorm_kernel with an e4m3 output (the A operand of ape_gemm_tn_e4m3): the warp holds the whole row, so the row's
// absolute maximum of t = LN(x) * w + b comes for free; y = e4m3(t / s) with s = max|t| / 448, and scale[out_row] = s.
template <typename TI, int MAXV>
__global__ void __launch_bounds__(256)
layernorm_e4m3_kernel(const TI *__restrict__ x, long long ldx, uint8_t *__restrict__ y, long long ldy, float *__restrict__ scale,
                      const float *__restrict__ w, const float *__restrict__ b, const int *__restrict__ row_map,
                      int rows, int C, float eps) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const TI *xr = x + (size_t)warp * ldx;
  const int nvec = (C + 7) >> 3;
  float v[MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
      load8<TI>(xr + 8 * j, v[i]);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (8 * j + k >= C) v[i][k] = 0.f;
        sum += v[i][k];
      }
    }
  }
  const float mean = warp_sum(sum) / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = (8 * j + k < C) ? v[i][k] - mean : 0.f;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {  // t in place of x, the same arithmetic as layernorm_kernel
    const int j = lane + 32 * i;
    if (j < nvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        v[i][k] = (8 * j + k < C) ? (v[i][k] - mean) * rstd * __ldg(w + 8 * j + k) + __ldg(b + 8 * j + k) : 0.f;
        amax = fmaxf(amax, fabsf(v[i][k]));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float s = amax / 448.f;  // 448: the largest finite e4m3 value
  const int orow = row_map ? row_map[warp] : warp;
  uint8_t *yr = y + (size_t)orow * ldy;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
      uint32_t q[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2 lo = make_float2(0.f, 0.f), hi = make_float2(0.f, 0.f);
        if (s > 0.f) {
          lo = make_float2(v[i][4 * h] / s, v[i][4 * h + 1] / s);
          hi = make_float2(v[i][4 * h + 2] / s, v[i][4 * h + 3] / s);
        }
        q[h] = (uint32_t)__nv_cvt_float2_to_fp8x2(lo, __NV_SATFINITE, __NV_E4M3) |
               ((uint32_t)__nv_cvt_float2_to_fp8x2(hi, __NV_SATFINITE, __NV_E4M3) << 16);
      }
      *reinterpret_cast<uint2 *>(yr + 8 * j) = make_uint2(q[0], q[1]);
    }
  }
  if (lane == 0) scale[orow] = s;
}

// Extended row kernel for the deformable encoder (C <= 256 * MAXV):
//   t  = LN(x; w, b, eps)                       (norms[1] of the previous layer, deformable_transformer_vl.py:36-54)
//   t  = LN(t; w2, b2, eps2)       if w2        (layer_norm_v of the VisionLanguageFusion that follows, fuse_helper.py:224)
//   y  = t + col_add[c]            if col_add   (gamma_v * delta_v: one vector per image for "name" prompts)
//   y2 = y + row_add[row]          if y2        (query + query_pos, the operand of the sampling-offset / attention-weight GEMM)
// so the activations make one trip through HBM where the module sequence makes four.
// NORM = false (no w): t = x, and y is written only when non-null: the first layer of an encoder without fusion layers, whose
// input needs nothing but `query + query_pos` (deformable_transformer.py:78-102).
template <typename TI, typename TO, int MAXV, bool NORM = true>
__global__ void __launch_bounds__(256)
layernorm_ex_kernel(const TI *__restrict__ x, long long ldx, TO *__restrict__ y, long long ldy, const float *__restrict__ w,
                    const float *__restrict__ b, float eps, const float *__restrict__ w2, const float *__restrict__ b2,
                    float eps2, const float *__restrict__ col_add, long long col_add_stride, int rows_per_image,
                    const TO *__restrict__ row_add, long long ld_add, TO *__restrict__ y2, long long ldy2, int rows, int C) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const TI *xr = x + (size_t)warp * ldx;
  const int nvec = C >> 3;  // host guarantees C % 8 == 0
  float v[MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
      load8<TI>(xr + 8 * j, v[i]);
#pragma unroll
      for (int k = 0; k < 8; ++k) sum += v[i][k];
    }
  }
  if constexpr (NORM) {
  float mean = warp_sum(sum) / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (lane + 32 * i < nvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = v[i][k] - mean;
        sq += d * d;
      }
    }
  float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
      float ww[8], bb[8];
      load8<float>(w + 8 * j, ww);
      load8<float>(b + 8 * j, bb);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        v[i][k] = (v[i][k] - mean) * rstd * ww[k] + bb[k];
        sum += v[i][k];
      }
    }
  }
  if (w2) {
    mean = warp_sum(sum) / (float)C;
    sq = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
      if (lane + 32 * i < nvec) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float d = v[i][k] - mean;
          sq += d * d;
        }
      }
    rstd = rsqrtf(warp_sum(sq) / (float)C + eps2);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int j = lane + 32 * i;
      if (j < nvec) {
        float ww[8], bb[8];
        load8<float>(w2 + 8 * j, ww);
        load8<float>(b2 + 8 * j, bb);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[i][k] = (v[i][k] - mean) * rstd * ww[k] + bb[k];
      }
    }
  }
  }  // NORM
  const float *ca = col_add ? col_add + (size_t)(warp / rows_per_image) * col_add_stride : nullptr;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + 32 * i;
    if (j < nvec) {
      if (ca) {
        float cc[8];
        load8<float>(ca + 8 * j, cc);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[i][k] += cc[k];
      }
      if (NORM || y) store8<TO>(y + (size_t)warp * ldy + 8 * j, v[i]);
      if (y2) {
        float a[8], o[8];
        load8<TO>(row_add + (size_t)warp * ld_add + 8 * j, a);
        // y2 is computed from the ROUNDED y so that it equals `y + row_add` evaluated on the stored tensors
        float r[8];
        if constexpr (sizeof(TO) == 4) {
#pragma unroll
          for (int k = 0; k < 8; ++k) r[k] = v[i][k];
        } else {
          Elem<TO>::unpack(Elem<TO>::pack(v[i]), r);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = r[k] + a[k];
        store8<TO>(y2 + (size_t)warp * ldy2 + 8 * j, o);
      }
    }
  }
}

// Wide rows (1024 < C <= 4096, e.g. the 2730-wide SwiGLU hidden): one CTA of 256 threads per row, each thread keeps
// up to two 8-element vectors in registers, statistics through warp shuffles + 8 shared-memory partials; the row
// makes exactly one trip in and one trip out.
__device__ __forceinline__ float block_sum_256(float v, float *s_part) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // s_part may still be read from the previous reduction
  if (lane == 0) s_part[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += s_part[i];
  return t;
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(256)
layernorm_wide_kernel(const TI *__restrict__ x, long long ldx, TO *__restrict__ y, long long ldy,
                      const float *__restrict__ w, const float *__restrict__ b, const int *__restrict__ row_map,
                      int rows, int C, float eps) {
  pdl_prologue();
  __shared__ float s_part[8];
  const int row = blockIdx.x;
  const bool wb_aligned = ((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
  const TI *xr = x + (size_t)row * ldx;
  const int nvec = (C + 7) >> 3;
  float v[2][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int j = threadIdx.x + 256 * i;
    if (j < nvec) {
      load8<TI>(xr + 8 * j, v[i]);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (8 * j + k >= C) v[i][k] = 0.f;
        sum += v[i][k];
      }
    }
  }
  const float mean = block_sum_256(sum, s_part) / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int j = threadIdx.x + 256 * i;
    if (j < nvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = (8 * j + k < C) ? v[i][k] - mean : 0.f;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(block_sum_256(sq, s_part) / (float)C + eps);
  TO *yr = y + (size_t)(row_map ? row_map[row] : row) * ldy;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int j = threadIdx.x + 256 * i;
    if (j < nvec) {
      float o[8];
      if (8 * j + 8 <= C && wb_aligned) {
        float ww[8], bb[8];
        load8<float>(w + 8 * j, ww);
        load8<float>(b + 8 * j, bb);
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = (v[i][k] - mean) * rstd * ww[k] + bb[k];
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k)
          o[k] = (8 * j + k < C) ? (v[i][k] - mean) * rstd * __ldg(w + 8 * j + k) + __ldg(b + 8 * j + k) : 0.f;
      }
      store8<TO>(yr + 8 * j, o);
    }
  }
}

// In-place 2-D RoPE on the q and k parts of qkv [M, 3*C] (C = heads*hd); cos/sin [npos, hd] fp32;
// token m uses position pos_map ? pos_map[m] : m % npos.  t' = t*cos + rotate_half(t)*sin with
// rotate_half pairing (2i, 2i+1) -> (-t[2i+1], t[2i]).  One thread per 8 channels.
template <typename T>
__global__ void __launch_bounds__(256)
rope_qk_kernel(T *__restrict__ qkv, long long ld, const float *__restrict__ cosr, const float *__restrict__ sinr,
               const int *__restrict__ pos_map, int M, int C, int hd, int npos) {
  pdl_prologue();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int vec_per_row = 2 * C / 8;  // q and k only
  if (idx >= (long long)M * vec_per_row) return;
  const int m = (int)(idx / vec_per_row), j = (int)(idx % vec_per_row);
  const int col = j * 8;           // column inside [0, 2C)
  const int d = col % hd;          // channel inside the head (hd % 8 == 0)
  const int pos = pos_map ? pos_map[m] : m % npos;
  T *p = qkv + (size_t)m * ld + col;
  float t[8], o[8];
  load8<T>(p, t);
  const float *c = cosr + (size_t)pos * hd + d, *s = sinr + (size_t)pos * hd + d;
#pragma unroll
  for (int i = 0; i < 8; i += 2) {
    o[i] = t[i] * c[i] - t[i + 1] * s[i];
    o[i + 1] = t[i + 1] * c[i + 1] + t[i] * s[i + 1];
  }
  store8<T>(p, o);
}

template <typename TI, typename TO>
int launch_ln(const void *x, long long ldx, void *y, long long ldy, const float *w, const float *b, const int *row_map,
              int rows, int C, float eps, cudaStream_t st) {
  const int blocks = (rows + 7) / 8;
  const bool aligned = (reinterpret_cast<uintptr_t>(w) & 15) == 0 && (reinterpret_cast<uintptr_t>(b) & 15) == 0;
  if (C <= 256 && aligned)
    APE_LAUNCH((layernorm_kernel<TI, TO, 1>), blocks, 256, 0, st, (const TI *)x, ldx, (TO *)y, ldy, w, b, row_map, rows, C, eps);
  else if (C <= 1024 && aligned)
    APE_LAUNCH((layernorm_kernel<TI, TO, 4>), blocks, 256, 0, st, (const TI *)x, ldx, (TO *)y, ldy, w, b, row_map, rows, C, eps);
  else  // one CTA per row, row held in registers (also valid in place)
    APE_LAUNCH((layernorm_wide_kernel<TI, TO>), rows, 256, 0, st, (const TI *)x, ldx, (TO *)y, ldy, w, b, row_map, rows, C, eps);
  return check_launch("layernorm_kernel");
}

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int ape_layernorm(const void *x, int64_t ldx, void *y, int64_t ldy, const float *weight, const float *bias,
                             const int *row_map, int rows, int C, float eps, int in_dtype, int out_dtype, void *stream) {
  if (rows < 0 || C <= 0 || C > 4096) return fail(APE_ERR_INVALID_ARG, "layernorm: rows=%d C=%d (C <= 4096)", rows, C);
  if (ldx < ((C + 7) & ~7) || ldy < ((C + 7) & ~7))
    return fail(APE_ERR_INVALID_ARG, "layernorm: row pitch must cover C rounded up to 8 elements");
  if (rows == 0) return APE_OK;
  if (!x || !y || !weight || !bias) return fail(APE_ERR_NULL_PTR, "layernorm: null pointer argument");
  const int ie = dtype_size(in_dtype), oe = dtype_size(out_dtype);
  if ((ldx * ie) % 16 || (ldy * oe) % 16 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15))
    return fail(APE_ERR_INVALID_ARG, "layernorm: rows must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define APE_LN(TI, TO) return launch_ln<TI, TO>(x, ldx, y, ldy, weight, bias, row_map, rows, C, eps, st)
  if (in_dtype == APE_DTYPE_F32) {
    if (out_dtype == APE_DTYPE_F32) APE_LN(float, float);
    if (out_dtype == APE_DTYPE_F16) APE_LN(float, __half);
    if (out_dtype == APE_DTYPE_BF16) APE_LN(float, __nv_bfloat16);
  } else if (in_dtype == APE_DTYPE_F16) {
    if (out_dtype == APE_DTYPE_F32) APE_LN(__half, float);
    if (out_dtype == APE_DTYPE_F16) APE_LN(__half, __half);
  } else if (in_dtype == APE_DTYPE_BF16) {
    if (out_dtype == APE_DTYPE_F32) APE_LN(__nv_bfloat16, float);
    if (out_dtype == APE_DTYPE_BF16) APE_LN(__nv_bfloat16, __nv_bfloat16);
  }
#undef APE_LN
  return fail(APE_ERR_UNSUPPORTED, "layernorm: dtype pair (%d -> %d) not supported", in_dtype, out_dtype);
}

extern "C" int ape_layernorm_e4m3(const void *x, int64_t ldx, void *y, int64_t ldy, float *scale, const float *weight,
                                  const float *bias, const int *row_map, int rows, int C, float eps, int in_dtype, void *stream) {
  if (rows < 0 || C <= 0 || C > 1024) return fail(APE_ERR_INVALID_ARG, "layernorm_e4m3: rows=%d C=%d (C <= 1024)", rows, C);
  if (ldx < ((C + 7) & ~7) || ldy < ((C + 7) & ~7))
    return fail(APE_ERR_INVALID_ARG, "layernorm_e4m3: row pitch must cover C rounded up to 8 elements");
  if (in_dtype != APE_DTYPE_F32 && in_dtype != APE_DTYPE_F16 && in_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_UNSUPPORTED, "layernorm_e4m3: input dtype %d not supported", in_dtype);
  if (rows == 0) return APE_OK;
  if (!x || !y || !scale || !weight || !bias) return fail(APE_ERR_NULL_PTR, "layernorm_e4m3: null pointer argument");
  if ((ldx * dtype_size(in_dtype)) % 16 || ldy % 16 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15))
    return fail(APE_ERR_INVALID_ARG, "layernorm_e4m3: rows must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int blocks = (rows + 7) / 8;
#define APE_LN8(TI)                                                                                                        \
  do {                                                                                                                     \
    if (C <= 256)                                                                                                          \
      APE_LAUNCH((layernorm_e4m3_kernel<TI, 1>), blocks, 256, 0, st, (const TI *)x, ldx, (uint8_t *)y, ldy, scale, weight, bias, \
                 row_map, rows, C, eps);                                                                                   \
    else                                                                                                                   \
      APE_LAUNCH((layernorm_e4m3_kernel<TI, 4>), blocks, 256, 0, st, (const TI *)x, ldx, (uint8_t *)y, ldy, scale, weight, bias, \
                 row_map, rows, C, eps);                                                                                   \
  } while (0)
  if (in_dtype == APE_DTYPE_F32) APE_LN8(float);
  else if (in_dtype == APE_DTYPE_F16) APE_LN8(__half);
  else APE_LN8(__nv_bfloat16);
#undef APE_LN8
  return check_launch("layernorm_e4m3_kernel");
}

extern "C" int ape_layernorm_ex(const void *x, int64_t ldx, void *y, int64_t ldy, const float *weight, const float *bias,
                                float eps, const float *weight2, const float *bias2, float eps2, const float *col_add,
                                int64_t col_add_stride, int rows_per_image, const void *row_add, int64_t ld_add, void *y2,
                                int64_t ldy2, int rows, int C, int in_dtype, int out_dtype, void *stream) {
  if (rows < 0 || C <= 0 || C > 1024 || C % 8 != 0) return fail(APE_ERR_INVALID_ARG, "layernorm_ex: rows=%d C=%d (C %% 8 == 0, C <= 1024)", rows, C);
  if (ldx < C || ldy < C || (y2 && (ldy2 < C || ld_add < C)))
    return fail(APE_ERR_INVALID_ARG, "layernorm_ex: row pitch smaller than C");
  if (rows == 0) return APE_OK;
  const bool norm = weight != nullptr;  // no weight: no normalisation (then weight2 must be null too, and y may be)
  if (!norm && (bias || weight2 || !(y || y2)))
    return fail(APE_ERR_INVALID_ARG, "layernorm_ex: without weight, bias and weight2 must be null and y or y2 given");
  if (!x || (norm && (!y || !bias)) || (weight2 && !bias2) || (y2 && !row_add) || (col_add && rows_per_image <= 0))
    return fail(APE_ERR_NULL_PTR, "layernorm_ex: null pointer argument");
  const int ie = dtype_size(in_dtype), oe = dtype_size(out_dtype);
  const uintptr_t al = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(y2) |
                       reinterpret_cast<uintptr_t>(row_add) | reinterpret_cast<uintptr_t>(weight) | reinterpret_cast<uintptr_t>(bias) |
                       reinterpret_cast<uintptr_t>(weight2) | reinterpret_cast<uintptr_t>(bias2) | reinterpret_cast<uintptr_t>(col_add);
  if ((ldx * ie) % 16 || (ldy * oe) % 16 || (ldy2 * oe) % 16 || (ld_add * oe) % 16 || (col_add_stride * 4) % 16 || (al & 15))
    return fail(APE_ERR_INVALID_ARG, "layernorm_ex: rows / vectors must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int blocks = (rows + 7) / 8;
#define APE_LNX(TI, TO)                                                                                                   \
  do {                                                                                                                    \
    if (!norm && C <= 256)                                                                                                \
      APE_LAUNCH((ape::layernorm_ex_kernel<TI, TO, 1, false>), blocks, 256, 0, st, (const TI *)x, ldx, (TO *)y, ldy, weight, bias, eps, \
          weight2, bias2, eps2, col_add, col_add_stride, rows_per_image > 0 ? rows_per_image : 1, (const TO *)row_add, ld_add, (TO *)y2, \
          ldy2, rows, C);                                                                                                 \
    else if (!norm)                                                                                                       \
      APE_LAUNCH((ape::layernorm_ex_kernel<TI, TO, 4, false>), blocks, 256, 0, st, (const TI *)x, ldx, (TO *)y, ldy, weight, bias, eps, \
          weight2, bias2, eps2, col_add, col_add_stride, rows_per_image > 0 ? rows_per_image : 1, (const TO *)row_add, ld_add, (TO *)y2, \
          ldy2, rows, C);                                                                                                 \
    else if (C <= 256)                                                                                                    \
      APE_LAUNCH((ape::layernorm_ex_kernel<TI, TO, 1>), blocks, 256, 0, st, (const TI *)x, ldx, (TO *)y, ldy, weight, bias, eps, weight2, bias2, eps2, \
          col_add, col_add_stride, rows_per_image > 0 ? rows_per_image : 1, (const TO *)row_add, ld_add, (TO *)y2, ldy2, rows, C);  \
    else                                                                                                                  \
      APE_LAUNCH((ape::layernorm_ex_kernel<TI, TO, 4>), blocks, 256, 0, st, (const TI *)x, ldx, (TO *)y, ldy, weight, bias, eps, weight2, bias2, eps2, \
          col_add, col_add_stride, rows_per_image > 0 ? rows_per_image : 1, (const TO *)row_add, ld_add, (TO *)y2, ldy2, rows, C);  \
    return check_launch("layernorm_ex_kernel");                                                                          \
  } while (0)
  if (in_dtype == APE_DTYPE_F16 && out_dtype == APE_DTYPE_F16) APE_LNX(__half, __half);
  if (in_dtype == APE_DTYPE_BF16 && out_dtype == APE_DTYPE_BF16) APE_LNX(__nv_bfloat16, __nv_bfloat16);
  if (in_dtype == APE_DTYPE_F32 && out_dtype == APE_DTYPE_F32) APE_LNX(float, float);
  if (in_dtype == APE_DTYPE_F32 && out_dtype == APE_DTYPE_F16) APE_LNX(float, __half);
  if (in_dtype == APE_DTYPE_F32 && out_dtype == APE_DTYPE_BF16) APE_LNX(float, __nv_bfloat16);
#undef APE_LNX
  return fail(APE_ERR_UNSUPPORTED, "layernorm_ex: dtype pair (%d -> %d) not supported", in_dtype, out_dtype);
}

extern "C" int ape_rope_qk(void *qkv, int64_t ld, const float *cos_table, const float *sin_table, const int *pos_map,
                           int M, int C, int head_dim, int npos, int dtype, void *stream) {
  if (M < 0 || C <= 0 || head_dim <= 0 || head_dim % 8 != 0 || C % head_dim != 0 || npos <= 0)
    return fail(APE_ERR_INVALID_ARG, "rope: M=%d C=%d head_dim=%d npos=%d", M, C, head_dim, npos);
  if (M == 0) return APE_OK;
  if (!qkv || !cos_table || !sin_table) return fail(APE_ERR_NULL_PTR, "rope: null pointer argument");
  if ((ld * dtype_size(dtype)) % 16 || (reinterpret_cast<uintptr_t>(qkv) & 15))
    return fail(APE_ERR_INVALID_ARG, "rope: rows must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long n = (long long)M * (2 * C / 8);
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (dtype == APE_DTYPE_F32)
    APE_LAUNCH((rope_qk_kernel<float>), blocks, 256, 0, st, (float *)qkv, ld, cos_table, sin_table, pos_map, M, C, head_dim, npos);
  else if (dtype == APE_DTYPE_F16)
    APE_LAUNCH((rope_qk_kernel<__half>), blocks, 256, 0, st, (__half *)qkv, ld, cos_table, sin_table, pos_map, M, C, head_dim, npos);
  else if (dtype == APE_DTYPE_BF16)
    APE_LAUNCH((rope_qk_kernel<__nv_bfloat16>), blocks, 256, 0, st, (__nv_bfloat16 *)qkv, ld, cos_table, sin_table, pos_map, M, C, head_dim, npos);
  else
    return fail(APE_ERR_INVALID_ARG, "rope: unknown dtype %d", dtype);
  return check_launch("rope_qk_kernel");
}

// ---- GroupNorm over token-major (NHWC) activations ------------------------------------------------
// The neck's ChannelMapper (detrex; configs/…1080k.py:42-55) applies GroupNorm(32, 256) to each 1x1-conv
// output.  With activations kept as [B, HW, C] rows (what the encoder consumes) the statistics of a group
// span all HW rows x C/G channels.  Deterministic two-level reduction: (1) each CTA reduces a strip of rows
// to per-group partial (sum, sum of squares), (2) one small kernel folds the partials in a fixed order and
// emits mean / rstd, (3) normalise.  One thread owns 8 consecutive channels (= one group when C/G == 8).
namespace ape {
namespace {

constexpr int kGnRowsPerCta = 64;

template <typename T>
__global__ void __launch_bounds__(256)
gn_partial_kernel(const T *__restrict__ x, long long ldx, int rows_per_image, int C, int cpg,
                  float *__restrict__ partial /* [B, strips, C/8, 2] */) {
  pdl_prologue();
  const int vec_per_row = C / 8;
  const int b = blockIdx.y, strip = blockIdx.x;
  const int r0 = strip * kGnRowsPerCta, r1 = min(rows_per_image, r0 + kGnRowsPerCta);
  // thread t: vector column v = t % vec_per_row, row offset t / vec_per_row (host guarantees 256 % vec_per_row == 0)
  const int v = threadIdx.x % vec_per_row, ro = threadIdx.x / vec_per_row, rstep = 256 / vec_per_row;
  float s = 0.f, ss = 0.f;
  for (int r = r0 + ro; r < r1; r += rstep) {
    float f[8];
    load8<T>(x + ((size_t)b * rows_per_image + r) * ldx + 8 * v, f);
#pragma unroll
    for (int k = 0; k < 8; ++k) { s += f[k]; ss += f[k] * f[k]; }
  }
  __shared__ float sh[256][2];
  sh[threadIdx.x][0] = s;
  sh[threadIdx.x][1] = ss;
  __syncthreads();
  if (threadIdx.x < vec_per_row) {
    float a = 0.f, c = 0.f;
    for (int j = threadIdx.x; j < 256; j += vec_per_row) { a += sh[j][0]; c += sh[j][1]; }
    float *dst = partial + (((size_t)b * gridDim.x + strip) * vec_per_row + threadIdx.x) * 2;
    dst[0] = a;
    dst[1] = c;
  }
}

// one warp per (b, group): lanes stride over the strips (fixed assignment -> deterministic), fp64 fold
__global__ void gn_finalize_kernel(const float *__restrict__ partial, int B, int strips, int vec_per_row, int vec_per_group,
                                   float count, float eps, float *__restrict__ stats /* [B, G, 2] mean, rstd */) {
  pdl_prologue();
  const int idx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int G = vec_per_row / vec_per_group;
  if (idx >= B * G) return;
  const int b = idx / G, g = idx % G;
  double s = 0.0, ss = 0.0;
  for (int st = lane; st < strips; st += 32)
    for (int v = 0; v < vec_per_group; ++v) {
      const float2 p = *reinterpret_cast<const float2 *>(partial + (((size_t)b * strips + st) * vec_per_row + g * vec_per_group + v) * 2);
      s += p.x;
      ss += p.y;
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  if (lane == 0) {
    const double mean = s / count;
    const double var = fmax(ss / count - mean * mean, 0.0);
    stats[idx * 2] = (float)mean;
    stats[idx * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(256)
gn_apply_kernel(const TI *__restrict__ x, long long ldx, TO *__restrict__ y, long long ldy, long long y_batch_stride,
                const float *__restrict__ w, const float *__restrict__ bias, const float *__restrict__ stats, int rows_per_image,
                long long total_rows, int C, int vec_per_group) {
  pdl_prologue();
  const int vec_per_row = C / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total_rows * vec_per_row) return;
  const long long row = idx / vec_per_row;
  const int v = (int)(idx % vec_per_row);
  const int b = (int)(row / rows_per_image);
  const int G = vec_per_row / vec_per_group;
  const float mean = stats[(b * G + v / vec_per_group) * 2], rstd = stats[(b * G + v / vec_per_group) * 2 + 1];
  float f[8], o[8];
  load8<TI>(x + (size_t)row * ldx + 8 * v, f);
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = (f[k] - mean) * rstd * __ldg(w + 8 * v + k) + __ldg(bias + 8 * v + k);
  store8<TO>(y + (size_t)b * y_batch_stride + (size_t)(row - (long long)b * rows_per_image) * ldy + 8 * v, o);
}

}  // namespace
}  // namespace ape

extern "C" int64_t ape_groupnorm_workspace_bytes(int B, int rows_per_image, int C) {
  const int64_t strips = (rows_per_image + ape::kGnRowsPerCta - 1) / ape::kGnRowsPerCta;
  return ((int64_t)B * strips * (C / 8) * 2 + (int64_t)B * C) * 4;
}

extern "C" int ape_groupnorm_nhwc(const void *x, int64_t ldx, void *y, int64_t ldy, int64_t y_batch_stride,
                                  const float *weight, const float *bias, void *workspace, int B, int rows_per_image, int C, int groups, float eps, int in_dtype,
                                  int out_dtype, void *stream) {
  using namespace ape;
  if (B < 0 || rows_per_image <= 0 || C <= 0 || groups <= 0 || C % groups != 0 || (C / groups) % 8 != 0 || 256 % (C / 8) != 0)
    return fail(APE_ERR_UNSUPPORTED, "groupnorm: C=%d groups=%d (channels per group must be a multiple of 8, C/8 must divide 256)", C, groups);
  if (B == 0) return APE_OK;
  if (!x || !y || !weight || !bias || !workspace) return fail(APE_ERR_NULL_PTR, "groupnorm: null pointer argument");
  if (y_batch_stride == 0) y_batch_stride = (int64_t)rows_per_image * ldy;
  if ((ldx * dtype_size(in_dtype)) % 16 || (ldy * dtype_size(out_dtype)) % 16 || (y_batch_stride * dtype_size(out_dtype)) % 16 ||
      (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15))
    return fail(APE_ERR_INVALID_ARG, "groupnorm: rows must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int strips = (rows_per_image + kGnRowsPerCta - 1) / kGnRowsPerCta;
  const int vpr = C / 8, vpg = C / groups / 8;
  float *partial = reinterpret_cast<float *>(workspace);
  float *stats = partial + (size_t)B * strips * vpr * 2;
  if (in_dtype == APE_DTYPE_F32) APE_LAUNCH((gn_partial_kernel<float>), dim3(strips, B), 256, 0, st, (const float *)x, ldx, rows_per_image, C, C / groups, partial);
  else if (in_dtype == APE_DTYPE_F16) APE_LAUNCH((gn_partial_kernel<__half>), dim3(strips, B), 256, 0, st, (const __half *)x, ldx, rows_per_image, C, C / groups, partial);
  else APE_LAUNCH((gn_partial_kernel<__nv_bfloat16>), dim3(strips, B), 256, 0, st, (const __nv_bfloat16 *)x, ldx, rows_per_image, C, C / groups, partial);
  if (int rc = check_launch("gn_partial_kernel")) return rc;
  APE_LAUNCH((gn_finalize_kernel), (B * groups + 3) / 4, 128, 0, st, partial, B, strips, vpr, vpg, (float)rows_per_image * (C / groups), eps, stats);
  if (int rc = check_launch("gn_finalize_kernel")) return rc;
  const long long total_rows = (long long)B * rows_per_image;
  const unsigned blocks = (unsigned)((total_rows * vpr + 255) / 256);
#define APE_GN(TI, TO) APE_LAUNCH((gn_apply_kernel<TI, TO>), blocks, 256, 0, st, (const TI *)x, ldx, (TO *)y, ldy, y_batch_stride, weight, bias, stats, rows_per_image, total_rows, C, vpg)
  if (in_dtype == APE_DTYPE_F32 && out_dtype == APE_DTYPE_F32) APE_GN(float, float);
  else if (in_dtype == APE_DTYPE_F16 && out_dtype == APE_DTYPE_F16) APE_GN(__half, __half);
  else if (in_dtype == APE_DTYPE_BF16 && out_dtype == APE_DTYPE_BF16) APE_GN(__nv_bfloat16, __nv_bfloat16);
  else if (in_dtype == APE_DTYPE_F16 && out_dtype == APE_DTYPE_F32) APE_GN(__half, float);
  else if (in_dtype == APE_DTYPE_BF16 && out_dtype == APE_DTYPE_F32) APE_GN(__nv_bfloat16, float);
  else return fail(APE_ERR_UNSUPPORTED, "groupnorm: dtype pair (%d -> %d) not supported", in_dtype, out_dtype);
#undef APE_GN
  return check_launch("gn_apply_kernel");
}


// ---- small fp32 GEMV: y[b, n] = W[n, :] . x[b, :] + bias[n] ---------------------------------------------------------------
// The language side of VisionLanguageFusion for "name" prompts is two affine maps of ONE 1024-wide token per encoder layer
// (vision_language_fusion.py:_folded_language_maps: [2312, 1024] and [1024, 2048] fp32 matrices); PyTorch runs them as cuBLAS
// GEMV kernels.  One warp per output row, 128-bit loads of the weight row, up to 4 input rows held against it.
namespace ape {
namespace {
__global__ void __launch_bounds__(256) gemv_f32_kernel(const float *__restrict__ W, const float *__restrict__ x,
                                                       const float *__restrict__ bias, float *__restrict__ y, int B, int N, int K) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  const float4 *w4 = reinterpret_cast<const float4 *>(W + (size_t)warp * K);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
  for (int k = lane; k < K / 4; k += 32) {
    const float4 w = __ldg(w4 + k);
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      if (b < B) {
        const float4 xv = __ldg(reinterpret_cast<const float4 *>(x + (size_t)b * K) + k);
        acc[b] = fmaf(w.x, xv.x, fmaf(w.y, xv.y, fmaf(w.z, xv.z, fmaf(w.w, xv.w, acc[b]))));
      }
    }
  }
#pragma unroll
  for (int b = 0; b < 4; ++b) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[b] += __shfl_xor_sync(0xffffffffu, acc[b], o);
  }
  if (lane == 0) {
    const float bb = bias != nullptr ? __ldg(bias + warp) : 0.f;
    for (int b = 0; b < B && b < 4; ++b) y[(size_t)b * N + warp] = acc[b] + bb;
  }
}
}  // namespace
}  // namespace ape

extern "C" int ape_gemv_f32(const float *W, const float *x, const float *bias, float *y, int B, int N, int K, void *stream) {
  using namespace ape;
  if (!W || !x || !y) return fail(APE_ERR_NULL_PTR, "gemv: null pointer");
  if (B <= 0 || B > 4 || N <= 0 || K <= 0 || K % 4) return fail(APE_ERR_UNSUPPORTED, "gemv: B=%d (1..4) N=%d K=%d (multiple of 4)", B, N, K);
  if ((reinterpret_cast<uintptr_t>(W) | reinterpret_cast<uintptr_t>(x)) & 15) return fail(APE_ERR_INVALID_ARG, "gemv: W / x must be 16-byte aligned");
  APE_LAUNCH(gemv_f32_kernel, (N + 7) / 8, 256, 0, (cudaStream_t)stream, W, x, bias, y, B, N, K);
  return check_launch("gemv_f32_kernel");
}


// ---- decoder reference-point update ---------------------------------------------------------------------------------------
// DeformableDetrTransformerDecoderVL.forward (deformable_transformer_vl.py:268-300, boxes as reference points):
//   new_ref = sigmoid(bbox_embed(output) + inverse_sigmoid(ref))                 detrex inverse_sigmoid, eps 1e-3
//   ref_in  = new_ref[:, :, None] * cat([valid_ratios, valid_ratios], -1)[:, None]   (input of the next layer's cross attention)
// Nine elementwise launches per decoder layer in PyTorch; one here, with the same fp32 operations in the same order
// (clamp, clamp, clamp, divide, logf, add, 1 / (1 + expf(-x)), multiply) so that the results are the same bits.
namespace ape {
namespace {
__global__ void __launch_bounds__(256) ref_update_kernel(const float *__restrict__ delta, const float *__restrict__ ref,
                                                         const float *__restrict__ valid_ratios, float *__restrict__ new_ref,
                                                         float *__restrict__ ref_in, int rows, int Q, int L, float eps) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (row, coordinate)
  if (i >= rows * 4) return;
  const int row = i >> 2, c = i & 3, b = row / Q;
  float x = fminf(fmaxf(__ldg(ref + i), 0.f), 1.f);
  const float x1 = fmaxf(x, eps), x2 = fmaxf(1.f - x, eps);
  const float y = __ldg(delta + i) + logf(x1 / x2);
  const float r = 1.f / (1.f + expf(-y));
  new_ref[i] = r;
  for (int l = 0; l < L; ++l) ref_in[((size_t)row * L + l) * 4 + c] = r * __ldg(valid_ratios + ((size_t)b * L + l) * 2 + (c & 1));
}
}  // namespace
}  // namespace ape

extern "C" int ape_ref_update(const float *delta, const float *ref, const float *valid_ratios, float *new_ref, float *ref_in, int B,
                              int Q, int L, float eps, void *stream) {
  using namespace ape;
  if (!delta || !ref || !valid_ratios || !new_ref || !ref_in) return fail(APE_ERR_NULL_PTR, "ref_update: null pointer");
  if (B <= 0 || Q <= 0 || L <= 0) return fail(APE_ERR_INVALID_ARG, "ref_update: B=%d Q=%d L=%d", B, Q, L);
  const int n = B * Q * 4;
  APE_LAUNCH(ref_update_kernel, (n + 255) / 256, 256, 0, (cudaStream_t)stream, delta, ref, valid_ratios, new_ref, ref_in, B * Q, Q, L, eps);
  return check_launch("ref_update_kernel");
}


// ---- text tower, length-packed prompts ------------------------------------------------------------------------------------
// First residual of the packed text tower (TextTransformer: token_embedding(text) + positional_embedding,
// eva02_clip/transformer.py:722-724) over rows that hold the prompts back to back: x[r] = tok_emb[tok[r]] + pos_emb[pos[r]],
// one fp32 add as in the module sequence, so real rows carry the same bits.  Pad rows (pos < 0) are zeros; so is a row whose
// token id or position lies outside its table (nothing is read out of bounds).  One thread per 4 channels.
namespace ape {
namespace {
__global__ void __launch_bounds__(256) text_embed_packed_kernel(const float *__restrict__ tok_emb, const float *__restrict__ pos_emb,
                                                                const int *__restrict__ tok, const int *__restrict__ pos,
                                                                float *__restrict__ x, int rows, int D, int vocab, int ctx) {
  pdl_prologue();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int vec_per_row = D / 4;
  if (idx >= (long long)rows * vec_per_row) return;
  const int r = (int)(idx / vec_per_row), j = (int)(idx % vec_per_row);
  const int t = tok[r], q = pos[r];
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  if (q >= 0 && q < ctx && t >= 0 && t < vocab) {
    const float4 a = __ldg(reinterpret_cast<const float4 *>(tok_emb + (size_t)t * D) + j);
    const float4 b = __ldg(reinterpret_cast<const float4 *>(pos_emb + (size_t)q * D) + j);
    o = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
  reinterpret_cast<float4 *>(x + (size_t)r * D)[j] = o;
}

// out[i] = x[rows[i]]: the end-of-text rows of the packed prompts, ahead of ln_final and the text projection
__global__ void __launch_bounds__(256) rows_gather_kernel(const float *__restrict__ x, long long ldx, const long long *__restrict__ rows,
                                                          float *__restrict__ out, long long ldo, int n, int D) {
  pdl_prologue();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int vec_per_row = D / 4;
  if (idx >= (long long)n * vec_per_row) return;
  const int i = (int)(idx / vec_per_row), j = (int)(idx % vec_per_row);
  reinterpret_cast<float4 *>(out + (size_t)i * ldo)[j] = reinterpret_cast<const float4 *>(x + (size_t)rows[i] * ldx)[j];
}
}  // namespace
}  // namespace ape

extern "C" int ape_text_embed_packed(const float *token_embedding, const float *positional_embedding, const int *tok, const int *pos,
                                     float *x, int rows, int D, int vocab, int ctx, void *stream) {
  using namespace ape;
  if (rows < 0 || D <= 0 || D % 4 || vocab <= 0 || ctx <= 0)
    return fail(APE_ERR_INVALID_ARG, "text_embed_packed: rows=%d D=%d (multiple of 4) vocab=%d ctx=%d", rows, D, vocab, ctx);
  if (rows == 0) return APE_OK;
  if (!token_embedding || !positional_embedding || !tok || !pos || !x) return fail(APE_ERR_NULL_PTR, "text_embed_packed: null pointer argument");
  if ((reinterpret_cast<uintptr_t>(token_embedding) | reinterpret_cast<uintptr_t>(positional_embedding) | reinterpret_cast<uintptr_t>(x)) & 15)
    return fail(APE_ERR_INVALID_ARG, "text_embed_packed: tables and x must be 16-byte aligned");
  const long long n = (long long)rows * (D / 4);
  APE_LAUNCH(text_embed_packed_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, token_embedding, positional_embedding,
             tok, pos, x, rows, D, vocab, ctx);
  return check_launch("text_embed_packed_kernel");
}

extern "C" int ape_rows_gather(const float *x, int64_t ldx, const int64_t *rows, float *out, int64_t ldo, int n, int D, void *stream) {
  using namespace ape;
  if (n < 0 || D <= 0 || D % 4 || ldx < D || ldo < D) return fail(APE_ERR_INVALID_ARG, "rows_gather: n=%d D=%d (multiple of 4, pitches >= D)", n, D);
  if (n == 0) return APE_OK;
  if (!x || !rows || !out) return fail(APE_ERR_NULL_PTR, "rows_gather: null pointer argument");
  if (ldx % 4 || ldo % 4 || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15))
    return fail(APE_ERR_INVALID_ARG, "rows_gather: rows must be 16-byte aligned");
  const long long nv = (long long)n * (D / 4);
  APE_LAUNCH(rows_gather_kernel, (unsigned)((nv + 255) / 256), 256, 0, (cudaStream_t)stream, x, (long long)ldx,
             reinterpret_cast<const long long *>(rows), out, (long long)ldo, n, D);
  return check_launch("rows_gather_kernel");
}
