// msda_bwd.cu — multi-scale deformable attention, backward (sm_90a).
//
// Replaces torch.ops.ape.ms_deform_attn_backward
//   (ape/layers/csrc/vision.cpp:78, ms_deform_attn.h:42-61, host ms_deform_attn_cuda.cu:84-160,
//    kernels ms_deform_im2col_cuda.cuh:301-920 + the per-sample arithmetic of ms_deform_attn_col2im_bilinear :86-146).
//
//   grad_value[b, corner(s), h, :] += bilinear_w(corner) * attn * grad_out[b,q,h,:]
//   grad_attn[b,q,h,l,p]            = sum_c grad_out * bilinear(value)
//   grad_loc[b,q,h,l,p,(x,y)]       = (W_l, H_l) * attn * sum_c grad_out * d bilinear / d(w_im, h_im)
//
// Design (same mapping as the forward kernel, not the reference's thread-per-scalar kernels with their six
// shared-memory reduction variants): a row is one (b, q, h); LPR lanes own 16 bytes of its channels each.  Phase 1: the
// CTA turns its tile's sampling locations into records in shared memory.  Phase 2: every lane walks the L*P samples of
// its row — 4 corner loads (128-bit), 4 dot products with its chunk of grad_out, the three per-sample gradients reduced
// over the row's LPR lanes with shuffles (no shared-memory reduction, no __syncthreads per sample), and one VECTOR
// atomic per corner for grad_value (red.global.add.v4.f32).  All arithmetic in fp32 for every dtype; grad_value is
// accumulated in an fp32 buffer (the reference accumulates with atomicAdd in the tensor's own dtype, half included).
#include "common.cuh"

namespace ape {
namespace {

constexpr int kBwdMaxLevels = 16;

struct BwdParams {
  const void *value, *loc, *attn, *grad_out;
  const int64_t *shapes, *starts;
  float *grad_value;  // fp32 [B,S,H,D], pre-zeroed
  void *grad_loc, *grad_attn;
  int B, S, H, L, Q, P;
  int ht_log2;
};

// flags: 1 = x1 distinct texel, 2 = y1 distinct texel, 4 = left column valid, 8 = right column valid,
//        16 = top row valid, 32 = bottom row valid (all validity bits are 0 for an out-of-range sample)
struct __align__(16) BRec {
  unsigned off_flags;  // (byte offset of corner (y0, x0) in `value`, in 16-byte units) << 6 | flags
  float a, lh, lw;
};

__device__ __forceinline__ BRec make_brec(float x, float y, float a, int Hl, int Wl, int start, int h, int H, int row_bytes) {
  const float h_im = y * (float)Hl - 0.5f;
  const float w_im = x * (float)Wl - 0.5f;
  const bool in_range = h_im > -1.f && w_im > -1.f && h_im < (float)Hl && w_im < (float)Wl;
  const int h_low = __float2int_rd(h_im), w_low = __float2int_rd(w_im);
  const int hc = min(max(h_low, -1), Hl - 1), wc = min(max(w_low, -1), Wl - 1);
  const int y0 = max(hc, 0), x0 = max(wc, 0);
  const int y1 = min(hc + 1, Hl - 1), x1 = min(wc + 1, Wl - 1);
  BRec r;
  unsigned f = (x1 != x0 ? 1 : 0) | (y1 != y0 ? 2 : 0);
  if (in_range) f |= (w_low >= 0 ? 4 : 0) | (w_low < Wl - 1 ? 8 : 0) | (h_low >= 0 ? 16 : 0) | (h_low < Hl - 1 ? 32 : 0);
  r.off_flags = ((unsigned)(((start + y0 * Wl + x0) * H + h) * (row_bytes >> 4)) << 6) | f;
  r.a = in_range ? a : 0.f;
  r.lh = in_range ? h_im - floorf(h_im) : 0.f;
  r.lw = in_range ? w_im - floorf(w_im) : 0.f;
  return r;
}

__device__ __forceinline__ void red_add_v4(float *p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

template <typename T, int LPR>
__global__ void __launch_bounds__(LPR >= 4 ? 256 : 64 * LPR) msda_bwd_kernel(const BwdParams p) {
  using E = Elem<T>;
  constexpr int VEC = E::kVec;
  constexpr int NT = LPR >= 4 ? 256 : 64 * LPR;
  constexpr int R = NT / LPR;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int s_lvl[kBwdMaxLevels * 3];
  __shared__ int s_dy[kBwdMaxLevels];
  const int LP = p.L * p.P;
  const int lps = LP | 1;
  BRec *s_rec = reinterpret_cast<BRec *>(smem_raw);
  const int tid = threadIdx.x;
  if (tid < p.L) {
    s_lvl[tid * 3 + 0] = (int)p.shapes[tid * 2 + 0];
    s_lvl[tid * 3 + 1] = (int)p.shapes[tid * 2 + 1];
    s_lvl[tid * 3 + 2] = (int)p.starts[tid];
    s_dy[tid] = (int)p.shapes[tid * 2 + 1] * p.H * LPR * 16;
  }
  __syncthreads();
  const int HT = 1 << p.ht_log2, QT = R >> p.ht_log2, head_tiles = p.H >> p.ht_log2;
  const int b = blockIdx.y;
  const int q0 = (blockIdx.x / head_tiles) * QT, h0 = (blockIdx.x % head_tiles) * HT;
  const T *loc = reinterpret_cast<const T *>(p.loc);
  const T *attn = reinterpret_cast<const T *>(p.attn);
  for (int i = tid; i < R * LP; i += NT) {
    const int r = i / LP, s = i - r * LP;
    const int q = q0 + (r >> p.ht_log2), h = h0 + (r & (HT - 1));
    BRec rec = {0u, 0.f, 0.f, 0.f};
    if (q < p.Q) {
      const int l = s / p.P;
      const size_t e = (((size_t)b * p.Q + q) * p.H + h) * LP + s;
      const float2 xy = E::load2(loc + 2 * e);
      rec = make_brec(xy.x, xy.y, E::load1(attn + e), s_lvl[l * 3], s_lvl[l * 3 + 1], s_lvl[l * 3 + 2], h, p.H, LPR * 16);
    }
    s_rec[r * lps + s] = rec;
  }
  __syncthreads();

  const int r = tid / LPR, c = tid % LPR;
  const int q = q0 + (r >> p.ht_log2), h = h0 + (r & (HT - 1));
  const bool active = q < p.Q;  // whole row groups are active / inactive together; shuffles below stay inside a group
  const size_t row = ((size_t)b * p.Q + (active ? q : 0)) * p.H + h;
  float g[VEC];
  {
    uint4 gv = make_uint4(0u, 0u, 0u, 0u);
    if (active) gv = *(reinterpret_cast<const uint4 *>(p.grad_out) + row * LPR + c);
    E::unpack(gv, g);
  }
  const char *vb = reinterpret_cast<const char *>(p.value) + ((size_t)b * p.S * p.H * LPR + c) * 16;
  float *gvb = p.grad_value + ((size_t)b * p.S * p.H * LPR + c) * (16 / sizeof(T)) ;  // same element index as vb
  const BRec *recs = s_rec + r * lps;
  const unsigned dxb = (unsigned)(p.H * LPR * 16);
  T *gloc = reinterpret_cast<T *>(p.grad_loc);
  T *gattn = reinterpret_cast<T *>(p.grad_attn);

#pragma unroll 1
  for (int l = 0; l < p.L; ++l) {
    const unsigned dyb = (unsigned)s_dy[l];
    const float Wf = (float)s_lvl[l * 3 + 1], Hf = (float)s_lvl[l * 3];
#pragma unroll 1
    for (int pp = 0; pp < p.P; ++pp) {
      const BRec rc = recs[l * p.P + pp];
      const unsigned f = rc.off_flags;
      const unsigned o0 = (f >> 6) << 4;
      const unsigned ox = (f & 1) ? dxb : 0u, oy = (f & 2) ? dyb : 0u;
      const bool L_ok = f & 4, R_ok = f & 8, T_ok = f & 16, B_ok = f & 32;
      const unsigned off[4] = {o0, o0 + ox, o0 + oy, o0 + oy + ox};
      const bool ok[4] = {T_ok && L_ok, T_ok && R_ok, B_ok && L_ok, B_ok && R_ok};
      const float lh = rc.lh, lw = rc.lw, hh = 1.f - lh, hw = 1.f - lw;
      const float wgt[4] = {hh * hw, hh * lw, lh * hw, lh * lw};
      float dot[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        dot[k] = 0.f;
        if (ok[k]) {  // uniform inside the row group (same record)
          float v[VEC];
          E::unpack(ldg_nc_v4(reinterpret_cast<const uint4 *>(vb + off[k])), v);
#pragma unroll
          for (int i = 0; i < VEC; ++i) dot[k] = fmaf(g[i], v[i], dot[k]);
          // grad_value: w_k * attn * grad_out, one vector reduction per 4 channels
          const float s = wgt[k] * rc.a;
          float *dst = gvb + (size_t)off[k] / sizeof(T);
#pragma unroll
          for (int i = 0; i < VEC; i += 4) red_add_v4(dst + i, s * g[i], s * g[i + 1], s * g[i + 2], s * g[i + 3]);
        }
      }
      // per-sample gradients, summed over this lane's channels (ms_deform_im2col_cuda.cuh:114-145)
      float ga = wgt[0] * dot[0] + wgt[1] * dot[1] + wgt[2] * dot[2] + wgt[3] * dot[3];
      float gh = -hw * dot[0] - lw * dot[1] + hw * dot[2] + lw * dot[3];
      float gw = -hh * dot[0] + hh * dot[1] - lh * dot[2] + lh * dot[3];
#pragma unroll
      for (int o = 1; o < LPR; o <<= 1) {
        ga += __shfl_xor_sync(0xffffffffu, ga, o);
        gh += __shfl_xor_sync(0xffffffffu, gh, o);
        gw += __shfl_xor_sync(0xffffffffu, gw, o);
      }
      if (active && c == 0) {
        const size_t e = row * LP + l * p.P + pp;
        gattn[e] = E::from_f(ga);
        gloc[2 * e] = E::from_f(Wf * gw * rc.a);
        gloc[2 * e + 1] = E::from_f(Hf * gh * rc.a);
      }
    }
  }
}

template <typename T, int LPR>
int launch_bwd(const BwdParams &p, cudaStream_t st) {
  constexpr int NT = LPR >= 4 ? 256 : 64 * LPR, R = NT / LPR;
  const size_t smem = (size_t)R * ((p.L * p.P) | 1) * sizeof(BRec);
  auto k = msda_bwd_kernel<T, LPR>;
  if (smem > 40 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "msda_bwd: cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
  }
  const int QT = R >> p.ht_log2;
  dim3 grid((unsigned)(((p.Q + QT - 1) / QT) * (p.H >> p.ht_log2)), (unsigned)p.B);
  k<<<grid, NT, smem, st>>>(p);
  return check_launch("msda_bwd_kernel");
}

template <typename T>
int dispatch_bwd(int lpr, const BwdParams &p, cudaStream_t st) {
  switch (lpr) {
    case 1: return launch_bwd<T, 1>(p, st);
    case 2: return launch_bwd<T, 2>(p, st);
    case 4: return launch_bwd<T, 4>(p, st);
    case 8: return launch_bwd<T, 8>(p, st);
    case 16: return launch_bwd<T, 16>(p, st);
    case 32: return launch_bwd<T, 32>(p, st);
  }
  return fail(APE_ERR_UNSUPPORTED, "msda_bwd: lanes-per-row %d", lpr);
}

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int ape_msda_bwd(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc, const void *attn,
                            const void *grad_out, float *grad_value_f32, void *grad_loc, void *grad_attn, int B, int S, int H,
                            int D, int L, int Q, int P, int dtype, void *stream) {
  if (dtype != APE_DTYPE_F32 && dtype != APE_DTYPE_F16 && dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "msda_bwd: unknown dtype %d", dtype);
  if (B < 0 || S < 0 || Q < 0 || H <= 0 || D <= 0 || L <= 0 || P <= 0 || L > kBwdMaxLevels || B > 65535)
    return fail(APE_ERR_INVALID_ARG, "msda_bwd: bad sizes B=%d S=%d H=%d D=%d L=%d Q=%d P=%d", B, S, H, D, L, Q, P);
  if ((long long)S * H * D * dtype_size(dtype) >= (1LL << 30)) return fail(APE_ERR_UNSUPPORTED, "msda_bwd: one image's value tensor must stay below 1 GiB (26-bit offsets in 16-byte units)");
  if (B == 0 || Q == 0) return APE_OK;
  if (!value || !shapes || !starts || !loc || !attn || !grad_out || !grad_value_f32 || !grad_loc || !grad_attn)
    return fail(APE_ERR_NULL_PTR, "msda_bwd: null pointer argument");
  const int row_bytes = D * dtype_size(dtype);
  const int lpr = row_bytes / 16;
  if (row_bytes % 16 != 0 || lpr > 32 || (lpr & (lpr - 1)) || (H & (H - 1)))
    return fail(APE_ERR_UNSUPPORTED, "msda_bwd: head dim * element size must be a power-of-two multiple of 16 B (<= 512), H a power of two");
  if ((reinterpret_cast<uintptr_t>(value) | reinterpret_cast<uintptr_t>(grad_out) | reinterpret_cast<uintptr_t>(grad_value_f32)) & 15)
    return fail(APE_ERR_INVALID_ARG, "msda_bwd: value / grad_out / grad_value must be 16-byte aligned");
  BwdParams p{};
  p.value = value; p.loc = loc; p.attn = attn; p.grad_out = grad_out; p.shapes = shapes; p.starts = starts;
  p.grad_value = grad_value_f32; p.grad_loc = grad_loc; p.grad_attn = grad_attn;
  p.B = B; p.S = S; p.H = H; p.L = L; p.Q = Q; p.P = P;
  const int R = (lpr >= 4 ? 256 : 64 * lpr) / lpr;
  int ht = Q >= 4 * R ? 1 : H;
  while (ht > R) ht >>= 1;
  int lg = 0;
  while ((1 << lg) < ht) ++lg;
  p.ht_log2 = lg;
  if ((size_t)R * ((L * P) | 1) * 16 > 200 * 1024) return fail(APE_ERR_UNSUPPORTED, "msda_bwd: L*P=%d too large for shared memory", L * P);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (dtype) {
    case APE_DTYPE_F32: return dispatch_bwd<float>(lpr, p, st);
    case APE_DTYPE_F16: return dispatch_bwd<__half>(lpr, p, st);
    default: return dispatch_bwd<__nv_bfloat16>(lpr, p, st);
  }
}
