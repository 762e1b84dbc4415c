// msda_fwd.cu — multi-scale deformable attention forward for sm_90a (H100).
//
// Replaces torch.ops.ape.ms_deform_attn_forward
//   (ape/layers/csrc/MsDeformAttn/ms_deform_attn_cuda.cu:21-81, kernel
//    ape/layers/csrc/MsDeformAttn/ms_deform_im2col_cuda.cuh:237-299)
// and, in the fused entry point, the softmax + sampling-location arithmetic of
//   ape/layers/multi_scale_deform_attn.py:283-311.
//
// Design (GPU-first, not a translation of the reference's thread-per-scalar kernel):
//   * a "row" is one (b, q, h) output vector of D channels.  One lane owns 16 bytes of a row
//     (4 fp32 / 8 fp16|bf16 channels), so a row is LPR = D*sizeof(T)/16 lanes and every corner
//     fetch is one 128-bit load per lane — a full 128 B line per fp32 row of D=32.
//   * a CTA owns a tile of QT queries x HT heads.  Phase 1: all threads cooperatively read the
//     tile's sampling locations / attention weights with coalesced streaming loads and turn each
//     sample into 4 corner indices (int32, in 16-byte units, -1 = outside) and 4 fp32 weights
//     (bilinear x attention) staged in shared memory.  Phase 2: every lane walks the L*P samples
//     of its row, reads index/weight quads with two broadcast LDS.128, issues U*4 independent
//     LDG.128 gathers before consuming them, and accumulates in fp32 registers.  No shuffles
//     are needed because a lane owns its channels outright.
//   * HT=1 makes a CTA's rows 32..64 consecutive queries of ONE head, so neighbouring queries
//     (pixels, in the encoder) re-use each other's texels out of L1; HT=H keeps all heads of a few
//     queries together (better when queries are spatially unrelated, e.g. the decoder).
//   * spatial_shapes / level_start_index stay int64 device tensors at the boundary (as in the
//     reference op) and are converted once per CTA into int32 shared memory.
//   * the output is written exactly once with 128-bit stores; no pre-zeroing
//     (the reference does at::zeros + overwrite, ms_deform_attn_cuda.cu:55).
#include "common.cuh"

namespace ape {
namespace {

constexpr int kMaxLevels = 16;

struct MsdaParams {
  const void *value;
  const int64_t *shapes;
  const int64_t *starts;
  const void *loc;    // plain: sampling locations; fused: raw offsets
  const void *attn;   // plain: attention weights;  fused: raw logits
  const float *ref;   // fused only
  void *out;
  int64_t offs_row_stride;   // fused: elements between consecutive (b,q) rows of `loc`
  int64_t logit_row_stride;  // fused: elements between consecutive (b,q) rows of `attn`
  int B, S, H, L, Q, P;
  int ht_log2;  // log2(heads per CTA)
  int ref_dim;  // fused: 2 or 4
  int vec4;     // fused: P == 4 and offsets / logits rows allow 16 / 8-byte vector loads
};

__host__ __device__ constexpr int threads_for(int lpr) { return lpr >= 4 ? 256 : 64 * lpr; }

// floor(i / d) for 0 <= i < 2^20 given inv = 1/d (float): (i + 0.5) * inv never lands on the wrong
// side of an integer for these ranges, and costs 3 instructions instead of a ~20-instruction idiv.
__device__ __forceinline__ int fast_div(int i, float inv) { return __float2int_rz(((float)i + 0.5f) * inv); }

// One sampling point -> one 16-byte record {corner(y0,x0) byte offset | flags, hh*a, lh*a, lw}.
// Follows ms_deform_im2col_cuda.cuh:279-291 (in-range test) and :36-80 (corner validity, weights); `x`,`y` are
// normalised locations.  Coordinates are clamped into the level so every offset is a valid address; corners or
// samples the reference skips get weight 0 (the only observable difference: a NaN/Inf texel next to the border is
// multiplied by 0 instead of being skipped — finite inputs give identical results).
// flags (low 4 bits of the offset, which is a multiple of the >=16-byte row): 1 = x1 is a distinct texel,
// 2 = y1 is a distinct texel, 4 = left corners valid, 8 = right corners valid.  The vertical validity and the
// attention weight are folded into hh_a / lh_a; keeping lw in fp32 makes the 4 products identical to the
// uncompressed form up to reassociation.  16 bytes per sample instead of 32 halves the shared memory a CTA pins,
// which is L1 capacity returned to the gathered texels.
struct __align__(16) Sample {
  int off_flags;
  float hh_a, lh_a, lw;
};

// core of make_sample: corner (y0, x0) inside the level, flags and weights (off_flags holds the flags only)
__device__ __forceinline__ Sample make_sample_xy(float x, float y, float a, int Hl, int Wl, int &y0, int &x0) {
  const float h_im = y * (float)Hl - 0.5f;
  const float w_im = x * (float)Wl - 0.5f;
  const bool in_range = h_im > -1.f && w_im > -1.f && h_im < (float)Hl && w_im < (float)Wl;
  const float hf = floorf(h_im), wf = floorf(w_im);
  const float lh = h_im - hf, lw = w_im - wf;
  const float hh = 1.f - lh;
  // saturating float->int conversions (NaN -> 0), then clamp into the level
  const int h_low = __float2int_rd(h_im), w_low = __float2int_rd(w_im);
  const bool hl_ok = in_range && h_low >= 0, hh_ok = in_range && h_low < Hl - 1;
  const bool wl_ok = w_low >= 0, wh_ok = w_low < Wl - 1;
  const int hc = min(max(h_low, -1), Hl - 1), wc = min(max(w_low, -1), Wl - 1);
  y0 = max(hc, 0);
  x0 = max(wc, 0);
  const int y1 = min(hc + 1, Hl - 1), x1 = min(wc + 1, Wl - 1);
  Sample r;
  r.off_flags = (x1 != x0 ? 1 : 0) | (y1 != y0 ? 2 : 0) | (wl_ok ? 4 : 0) | (wh_ok ? 8 : 0);
  r.hh_a = hl_ok ? hh * a : 0.f;
  r.lh_a = hh_ok ? lh * a : 0.f;
  r.lw = in_range ? lw : 0.f;
  return r;
}

__device__ __forceinline__ Sample make_sample(float x, float y, float a, int Hl, int Wl, int start,
                                              int h, int H, int row_bytes) {
  int y0, x0;
  Sample r = make_sample_xy(x, y, a, Hl, Wl, y0, x0);
  r.off_flags |= ((start + y0 * Wl + x0) * H + h) * row_bytes;
  return r;
}

// 4 consecutive elements / 4 consecutive (x, y) pairs of the offsets / logits tensors as fp32 (one or two vector
// loads instead of 4 / 8 scalar ones; the host checks the alignment and passes vec4 = true).
template <typename TO>
__device__ __forceinline__ void load4(const TO *p, float *f) {
  if constexpr (sizeof(TO) == 4) {
    const float4 v = *reinterpret_cast<const float4 *>(p);
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  } else {
    const uint2 v = *reinterpret_cast<const uint2 *>(p);
    float g[8];
    Elem<TO>::unpack(make_uint4(v.x, v.y, 0u, 0u), g);
    f[0] = g[0]; f[1] = g[1]; f[2] = g[2]; f[3] = g[3];
  }
}
template <typename TO>
__device__ __forceinline__ void load8(const TO *p, float *f) {
  if constexpr (sizeof(TO) == 4) {
    const float4 a = *reinterpret_cast<const float4 *>(p), b = *reinterpret_cast<const float4 *>(p + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  } else {
    Elem<TO>::unpack(*reinterpret_cast<const uint4 *>(p), f);
  }
}

// Phase 2: gather + accumulate + store for one lane.  The host guarantees P % U == 0.
// s_dy[l] = byte distance between vertically adjacent texels of level l (W_l * H * row_bytes).
template <typename T, int LPR, int U>
__device__ __forceinline__ void gather_rows(const MsdaParams &p, const Sample *s_rec, const int *s_dy, int lps, int b,
                                            int q, int h) {
  using E = Elem<T>;
  constexpr int VEC = E::kVec;
  const int r = threadIdx.x / LPR, c = threadIdx.x % LPR;
  if (q < 0 || q >= p.Q) return;

  const char *vb = reinterpret_cast<const char *>(p.value) + ((size_t)b * p.S * p.H * LPR + c) * 16;
  const Sample *row = s_rec + r * lps;
  const unsigned dxb = (unsigned)(p.H * LPR * 16);

  float acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[i] = 0.f;

#pragma unroll 1
  for (int l = 0; l < p.L; ++l) {
    const unsigned dyb = (unsigned)s_dy[l];
#pragma unroll 1
    for (int pp = 0; pp < p.P; pp += U) {
      Sample sm[U];
#pragma unroll
      for (int u = 0; u < U; ++u) sm[u] = row[l * p.P + pp + u];
      uint4 v[U][4];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const unsigned o0 = (unsigned)sm[u].off_flags & ~15u;
        const unsigned ox = (sm[u].off_flags & 1) ? dxb : 0u, oy = (sm[u].off_flags & 2) ? dyb : 0u;
        v[u][0] = ldg_nc_v4(reinterpret_cast<const uint4 *>(vb + o0));
        v[u][1] = ldg_nc_v4(reinterpret_cast<const uint4 *>(vb + o0 + ox));
        v[u][2] = ldg_nc_v4(reinterpret_cast<const uint4 *>(vb + o0 + oy));
        v[u][3] = ldg_nc_v4(reinterpret_cast<const uint4 *>(vb + o0 + oy + ox));
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float hw = (sm[u].off_flags & 4) ? 1.f - sm[u].lw : 0.f;
        const float lw = (sm[u].off_flags & 8) ? sm[u].lw : 0.f;
        const float ww[4] = {sm[u].hh_a * hw, sm[u].hh_a * lw, sm[u].lh_a * hw, sm[u].lh_a * lw};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float f[VEC];
          E::unpack(v[u][k], f);
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] = fmaf(ww[k], f[i], acc[i]);
        }
      }
    }
  }
  uint4 *ob = reinterpret_cast<uint4 *>(p.out) + (((size_t)b * p.Q + q) * p.H + h) * LPR + c;
  stg_stream_v4(ob, E::pack(acc));
}

// grid = (q_tiles * head_tiles, B); dynamic smem = R*lps*16 bytes.
template <typename T, int LPR, int U>
__global__ void __launch_bounds__(threads_for(LPR))
msda_fwd_kernel(const MsdaParams p) {
  using E = Elem<T>;
  constexpr int NT = threads_for(LPR);
  constexpr int R = NT / LPR;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int s_lvl[kMaxLevels * 3];
  __shared__ int s_dy[kMaxLevels];

  const int LP = p.L * p.P;
  const int lps = LP | 1;  // odd stride (in 16 B units): conflict-free broadcast reads
  Sample *s_rec = reinterpret_cast<Sample *>(smem_raw);

  const int tid = threadIdx.x;
  if (tid < p.L) {
    s_lvl[tid * 3 + 0] = (int)p.shapes[tid * 2 + 0];
    s_lvl[tid * 3 + 1] = (int)p.shapes[tid * 2 + 1];
    s_lvl[tid * 3 + 2] = (int)p.starts[tid];
    s_dy[tid] = (int)p.shapes[tid * 2 + 1] * p.H * LPR * 16;
  }
  __syncthreads();

  const int HT = 1 << p.ht_log2;
  const int QT = R >> p.ht_log2;
  const int head_tiles = p.H >> p.ht_log2;
  const int b = blockIdx.y;
  const int q0 = (blockIdx.x / head_tiles) * QT;
  const int h0 = (blockIdx.x % head_tiles) * HT;

  const T *loc = reinterpret_cast<const T *>(p.loc);
  const T *attn = reinterpret_cast<const T *>(p.attn);
  const float inv_lp = 1.f / (float)LP, inv_p = 1.f / (float)p.P;
  for (int i = tid; i < R * LP; i += NT) {
    const int r = fast_div(i, inv_lp), s = i - r * LP;  // exact for i < 2^20
    const int q = q0 + (r >> p.ht_log2), h = h0 + (r & (HT - 1));
    Sample rec = {0, 0.f, 0.f, 0.f};
    if (q < p.Q) {
      const int l = fast_div(s, inv_p);
      const size_t e = (((size_t)b * p.Q + q) * p.H + h) * LP + s;
      const float2 xy = E::load2(loc + 2 * e);
      const float a = E::load1(attn + e);
      rec = make_sample(xy.x, xy.y, a, s_lvl[l * 3], s_lvl[l * 3 + 1], s_lvl[l * 3 + 2], h, p.H, LPR * 16);
    }
    s_rec[r * lps + s] = rec;
  }
  __syncthreads();
  {
    const int r = tid / LPR;
    gather_rows<T, LPR, U>(p, s_rec, s_dy, lps, b, q0 + (r >> p.ht_log2), h0 + (r & (HT - 1)));
  }
}

// Fused variant: softmax(logits) over L*P, loc = f(ref, offsets), then the same gather.
// TO = element type of the offsets/logits tensors (output of the sampling_offsets /
// attention_weights linears).
template <typename T, typename TO, int LPR, int U>
__global__ void __launch_bounds__(threads_for(LPR))
msda_fused_fwd_kernel(const MsdaParams p) {
  pdl_prologue();
  using EO = Elem<TO>;
  constexpr int NT = threads_for(LPR);
  constexpr int R = NT / LPR;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int s_lvl[kMaxLevels * 3];
  __shared__ int s_dy[kMaxLevels];
  __shared__ float s_max[R], s_rinv[R];

  const int LP = p.L * p.P;
  const int lps = LP | 1;
  Sample *s_rec = reinterpret_cast<Sample *>(smem_raw);
  float *s_logit = reinterpret_cast<float *>(smem_raw + (size_t)R * lps * sizeof(Sample));

  const int tid = threadIdx.x;
  if (tid < p.L) {
    s_lvl[tid * 3 + 0] = (int)p.shapes[tid * 2 + 0];
    s_lvl[tid * 3 + 1] = (int)p.shapes[tid * 2 + 1];
    s_lvl[tid * 3 + 2] = (int)p.starts[tid];
    s_dy[tid] = (int)p.shapes[tid * 2 + 1] * p.H * LPR * 16;
  }
  const int HT = 1 << p.ht_log2;
  const int QT = R >> p.ht_log2;
  const int head_tiles = p.H >> p.ht_log2;
  const int b = blockIdx.y;
  const int q0 = (blockIdx.x / head_tiles) * QT;
  const int h0 = (blockIdx.x % head_tiles) * HT;

  const TO *offs = reinterpret_cast<const TO *>(p.loc);
  const TO *logits = reinterpret_cast<const TO *>(p.attn);

  // stage logits (coalesced), then one thread per row reduces max / sum(exp)
  const float inv_lp = 1.f / (float)LP, inv_p = 1.f / (float)p.P;
  const bool vec4 = p.vec4 != 0;  // P == 4 and 8/16-byte aligned rows: one thread per (row, level), vector loads
  if (vec4) {
    const float inv_l = 1.f / (float)p.L;
    for (int i = tid; i < R * p.L; i += NT) {
      const int r = fast_div(i, inv_l), l = i - r * p.L;
      const int q = q0 + (r >> p.ht_log2), h = h0 + (r & (HT - 1));
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (q < p.Q) load4<TO>(logits + ((size_t)b * p.Q + q) * p.logit_row_stride + h * LP + l * 4, v);
#pragma unroll
      for (int k = 0; k < 4; ++k) s_logit[r * lps + l * 4 + k] = v[k];
    }
  } else {
    for (int i = tid; i < R * LP; i += NT) {
      const int r = fast_div(i, inv_lp), s = i - r * LP;
      const int q = q0 + (r >> p.ht_log2), h = h0 + (r & (HT - 1));
      float v = 0.f;
      if (q < p.Q) v = EO::load1(logits + ((size_t)b * p.Q + q) * p.logit_row_stride + (size_t)h * LP + s);
      s_logit[r * lps + s] = v;
    }
  }
  __syncthreads();
  if (tid < R) {
    const float *row = s_logit + tid * lps;
    float m = row[0];
    for (int s = 1; s < LP; ++s) m = fmaxf(m, row[s]);
    float sum = 0.f;
    for (int s = 0; s < LP; ++s) sum += __expf(row[s] - m);
    s_max[tid] = m;
    s_rinv[tid] = 1.f / sum;
  }
  __syncthreads();

  if (vec4) {
    const float inv_l = 1.f / (float)p.L;
    for (int i = tid; i < R * p.L; i += NT) {
      const int r = fast_div(i, inv_l), l = i - r * p.L;
      const int q = q0 + (r >> p.ht_log2), h = h0 + (r & (HT - 1));
      Sample *dst = s_rec + r * lps + l * 4;
      if (q >= p.Q) {
#pragma unroll
        for (int k = 0; k < 4; ++k) dst[k] = Sample{0, 0.f, 0.f, 0.f};
        continue;
      }
      const int Hl = s_lvl[l * 3], Wl = s_lvl[l * 3 + 1], start = s_lvl[l * 3 + 2];
      const size_t bq = (size_t)b * p.Q + q;
      float o[8];
      load8<TO>(offs + bq * p.offs_row_stride + (h * LP + l * 4) * 2, o);
      const float *rp = p.ref + (bq * p.L + l) * p.ref_dim;
      const float mx = s_max[r], ri = s_rinv[r];
      float sx, sy;  // loc = ref + off * (sx, sy)
      if (p.ref_dim == 2) {  // multi_scale_deform_attn.py:298-303: ref + off / (W_l, H_l)
        sx = 1.f / (float)Wl;
        sy = 1.f / (float)Hl;
      } else {               // :304-311: ref_xy + off / P * ref_wh * 0.5
        sx = rp[2] * 0.125f;
        sy = rp[3] * 0.125f;
      }
      const float rx = rp[0], ry = rp[1];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float a = __expf(s_logit[r * lps + l * 4 + k] - mx) * ri;
        dst[k] = make_sample(fmaf(o[2 * k], sx, rx), fmaf(o[2 * k + 1], sy, ry), a, Hl, Wl, start, h, p.H, LPR * 16);
      }
    }
  } else {
    for (int i = tid; i < R * LP; i += NT) {
      const int r = fast_div(i, inv_lp), s = i - r * LP;
      const int q = q0 + (r >> p.ht_log2), h = h0 + (r & (HT - 1));
      Sample rec = {0, 0.f, 0.f, 0.f};
      if (q < p.Q) {
        const int l = fast_div(s, inv_p);
        const int Hl = s_lvl[l * 3], Wl = s_lvl[l * 3 + 1];
        const size_t bq = (size_t)b * p.Q + q;
        const float2 o = EO::load2(offs + bq * p.offs_row_stride + ((size_t)h * LP + s) * 2);
        const float a = __expf(s_logit[r * lps + s] - s_max[r]) * s_rinv[r];
        const float *rp = p.ref + (bq * p.L + l) * p.ref_dim;
        float x, y;
        if (p.ref_dim == 2) {
          // multi_scale_deform_attn.py:298-303: ref + off / (W_l, H_l)
          x = rp[0] + o.x / (float)Wl;
          y = rp[1] + o.y / (float)Hl;
        } else {
          // multi_scale_deform_attn.py:304-311: ref_xy + off / P * ref_wh * 0.5
          x = rp[0] + o.x / (float)p.P * rp[2] * 0.5f;
          y = rp[1] + o.y / (float)p.P * rp[3] * 0.5f;
        }
        rec = make_sample(x, y, a, Hl, Wl, s_lvl[l * 3 + 2], h, p.H, LPR * 16);
      }
      s_rec[r * lps + s] = rec;
    }
  }
  __syncthreads();
  {
    const int r = tid / LPR;
    gather_rows<T, LPR, U>(p, s_rec, s_dy, lps, b, q0 + (r >> p.ht_log2), h0 + (r & (HT - 1)));
  }
}

// Scalar fallback for shapes the vector path does not cover (D*sizeof(T) not a power-of-two
// multiple of 16 B, L > 16, or tiles that do not fit shared memory).  One thread per output
// scalar, fp32 accumulation.  Correctness path only.
template <typename T>
__global__ void __launch_bounds__(256)
msda_fwd_scalar_kernel(const MsdaParams p, int D, long long n) {
  using E = Elem<T>;
  const T *value = reinterpret_cast<const T *>(p.value);
  const T *loc = reinterpret_cast<const T *>(p.loc);
  const T *attn = reinterpret_cast<const T *>(p.attn);
  T *out = reinterpret_cast<T *>(p.out);
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % D);
    const long long row = idx / D;  // (b*Q+q)*H+h
    const int h = (int)(row % p.H);
    const int b = (int)(row / ((long long)p.H * p.Q));
    const T *vb = value + (size_t)b * p.S * p.H * D;
    float acc = 0.f;
    const int LP = p.L * p.P;
    for (int l = 0; l < p.L; ++l) {
      const int Hl = (int)p.shapes[2 * l], Wl = (int)p.shapes[2 * l + 1], st = (int)p.starts[l];
      for (int pt = 0; pt < p.P; ++pt) {
        const size_t e = (size_t)row * LP + l * p.P + pt;
        const float x = E::to_f(loc[2 * e]), y = E::to_f(loc[2 * e + 1]), a = E::to_f(attn[e]);
        const Sample sm = make_sample(x, y, a, Hl, Wl, st, h, p.H, 16);  // offsets in units of 16 -> (s,h) row index * 16
        const size_t r0 = (size_t)(((unsigned)sm.off_flags & ~15u) >> 4);
        const size_t rx = (sm.off_flags & 1) ? (size_t)p.H : 0, ry = (sm.off_flags & 2) ? (size_t)Wl * p.H : 0;
        const float hw = (sm.off_flags & 4) ? 1.f - sm.lw : 0.f, lw = (sm.off_flags & 8) ? sm.lw : 0.f;
        const float w00 = sm.hh_a * hw, w01 = sm.hh_a * lw, w10 = sm.lh_a * hw, w11 = sm.lh_a * lw;
        if (w00 != 0.f) acc = fmaf(w00, E::to_f(vb[r0 * D + c]), acc);
        if (w01 != 0.f) acc = fmaf(w01, E::to_f(vb[(r0 + rx) * D + c]), acc);
        if (w10 != 0.f) acc = fmaf(w10, E::to_f(vb[(r0 + ry) * D + c]), acc);
        if (w11 != 0.f) acc = fmaf(w11, E::to_f(vb[(r0 + ry + rx) * D + c]), acc);
      }
    }
    out[idx] = E::from_f(acc);
  }
}

// ---- host dispatch ---------------------------------------------------------------------------
template <typename K>
int set_smem(K kernel, size_t bytes) {
  if (bytes <= 40 * 1024) return APE_OK;  // static shared memory counts against the 48 KB default too
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(smem=%zu): %s", bytes, cudaGetErrorString(e));
  return APE_OK;
}

template <typename T, int LPR, int U>
int launch_plain(const MsdaParams &p, cudaStream_t st) {
  constexpr int NT = threads_for(LPR), R = NT / LPR;
  const int lps = (p.L * p.P) | 1;
  const size_t smem = (size_t)R * lps * 16;
  auto k = msda_fwd_kernel<T, LPR, U>;
  if (int rc = set_smem(k, smem)) return rc;
  const int QT = R >> p.ht_log2;
  dim3 grid((unsigned)(((p.Q + QT - 1) / QT) * (p.H >> p.ht_log2)), (unsigned)p.B);
  k<<<grid, NT, smem, st>>>(p);
  return check_launch("msda_fwd_kernel");
}

template <typename T, typename TO, int LPR, int U>
int launch_fused(const MsdaParams &p, cudaStream_t st) {
  constexpr int NT = threads_for(LPR), R = NT / LPR;
  const int lps = (p.L * p.P) | 1;
  const size_t smem = (size_t)R * lps * 20;
  auto k = msda_fused_fwd_kernel<T, TO, LPR, U>;
  if (int rc = set_smem(k, smem)) return rc;
  const int QT = R >> p.ht_log2;
  dim3 grid((unsigned)(((p.Q + QT - 1) / QT) * (p.H >> p.ht_log2)), (unsigned)p.B);
  APE_LAUNCH(k, grid, NT, smem, st, p);
  return check_launch("msda_fused_fwd_kernel");
}

template <typename T, int U>
int dispatch_lpr_plain(int lpr, const MsdaParams &p, cudaStream_t st) {
  switch (lpr) {
    case 1: return launch_plain<T, 1, U>(p, st);
    case 2: return launch_plain<T, 2, U>(p, st);
    case 4: return launch_plain<T, 4, U>(p, st);
    case 8: return launch_plain<T, 8, U>(p, st);
    case 16: return launch_plain<T, 16, U>(p, st);
    case 32: return launch_plain<T, 32, U>(p, st);
  }
  return fail(APE_ERR_UNSUPPORTED, "msda: lanes-per-row %d", lpr);
}

template <typename T, typename TO>
int dispatch_lpr_fused(int lpr, const MsdaParams &p, cudaStream_t st) {
  if (p.P % 2 != 0) {
    switch (lpr) {
      case 2: return launch_fused<T, TO, 2, 1>(p, st);
      case 4: return launch_fused<T, TO, 4, 1>(p, st);
      case 8: return launch_fused<T, TO, 8, 1>(p, st);
      case 16: return launch_fused<T, TO, 16, 1>(p, st);
    }
  } else {
    switch (lpr) {
      case 2: return launch_fused<T, TO, 2, 2>(p, st);
      case 4: return launch_fused<T, TO, 4, 2>(p, st);
      case 8: return launch_fused<T, TO, 8, 2>(p, st);
      case 16: return launch_fused<T, TO, 16, 2>(p, st);
    }
  }
  return fail(APE_ERR_UNSUPPORTED, "msda_fused: lanes-per-row %d (head dim * elem size must be 32..256 B)", lpr);
}

template <typename T>
int launch_scalar(const MsdaParams &p, int D, cudaStream_t st) {
  const long long n = (long long)p.B * p.Q * p.H * D;
  long long blocks = (n + 255) / 256;
  if (blocks > 132LL * 64) blocks = 132LL * 64;
  if (blocks < 1) blocks = 1;
  msda_fwd_scalar_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(p, D, n);
  return check_launch("msda_fwd_scalar_kernel");
}

bool is_pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }
int ilog2(int x) { int l = 0; while ((1 << l) < x) ++l; return l; }

int validate(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc,
             const void *attn, void *out, int B, int S, int H, int D, int L, int Q, int P, int dtype) {
  if (dtype != APE_DTYPE_F32 && dtype != APE_DTYPE_F16 && dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "msda: unknown dtype %d", dtype);
  if (B < 0 || S < 0 || Q < 0 || H <= 0 || D <= 0 || L <= 0 || P <= 0)
    return fail(APE_ERR_INVALID_ARG, "msda: bad sizes B=%d S=%d H=%d D=%d L=%d Q=%d P=%d", B, S, H, D, L, Q, P);
  if ((long long)S * H * D >= (1LL << 31))
    return fail(APE_ERR_UNSUPPORTED, "msda: S*H*D=%lld exceeds int32 indexing", (long long)S * H * D);
  if (B > 65535) return fail(APE_ERR_UNSUPPORTED, "msda: B=%d > 65535", B);
  if (B == 0 || Q == 0) return APE_OK;
  if (!value || !shapes || !starts || !loc || !attn || !out)
    return fail(APE_ERR_NULL_PTR, "msda: null pointer argument");
  return APE_OK;
}

// default tile mapping: one head per CTA when there are enough queries for neighbouring
// queries to share texels (encoder: queries are pixels); all heads together otherwise.
int default_ht(int H, int Q, int R) {
  if (!is_pow2(H)) return 1;
  if (Q >= 4 * R) return 1;
  int ht = H;
  while (ht > R) ht >>= 1;
  return ht;
}

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int ape_msda_fwd_variant(const void *value, const int64_t *shapes, const int64_t *starts,
                                    const void *loc, const void *attn, void *out, int B, int S, int H,
                                    int D, int L, int Q, int P, int dtype, int variant, void *stream) {
  if (int rc = validate(value, shapes, starts, loc, attn, out, B, S, H, D, L, Q, P, dtype)) return rc;
  if (B == 0 || Q == 0) return APE_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MsdaParams p{};
  p.value = value; p.shapes = shapes; p.starts = starts; p.loc = loc; p.attn = attn; p.out = out;
  p.B = B; p.S = S; p.H = H; p.L = L; p.Q = Q; p.P = P;

  const int esize = dtype_size(dtype);
  const int row_bytes = D * esize;
  const int lpr = row_bytes / 16;
  const bool vec_ok = (row_bytes % 16 == 0) && is_pow2(lpr) && lpr <= 32 && L <= kMaxLevels;
  bool scalar = !vec_ok || (variant >= 0 && (variant & 0x1000));
  const int LP = L * P;
  int ht = 0, unroll = (P % 4 == 0) ? 4 : (P % 2 == 0) ? 2 : 1;
  if (!scalar) {
    const int R = threads_for(lpr) / lpr;
    const size_t smem = (size_t)R * ((L * P) | 1) * 16;
    if (smem > 200 * 1024) scalar = true;
    ht = default_ht(H, Q, R);
    if (variant >= 0) {
      const int vh = variant & 0xff, vu = (variant >> 8) & 0xf;
      if (vh) {
        if (!is_pow2(vh) || H % vh != 0 || vh > R)
          return fail(APE_ERR_INVALID_ARG, "msda: heads_per_cta=%d invalid for H=%d R=%d", vh, H, R);
        ht = vh;
      }
      if (vu) {
        if ((vu != 1 && vu != 2 && vu != 4) || P % vu != 0)
          return fail(APE_ERR_INVALID_ARG, "msda: unroll=%d must be 1, 2 or 4 and divide P=%d", vu, P);
        unroll = vu;
      }
    }
  }
  if (scalar) {
    switch (dtype) {
      case APE_DTYPE_F32: return launch_scalar<float>(p, D, st);
      case APE_DTYPE_F16: return launch_scalar<__half>(p, D, st);
      default: return launch_scalar<__nv_bfloat16>(p, D, st);
    }
  }
  p.ht_log2 = ilog2(ht);
#define APE_MSDA_DISPATCH(T)                                            \
  switch (unroll) {                                                     \
    case 1: return dispatch_lpr_plain<T, 1>(lpr, p, st);                \
    case 2: return dispatch_lpr_plain<T, 2>(lpr, p, st);                \
    default: return dispatch_lpr_plain<T, 4>(lpr, p, st);               \
  }
  switch (dtype) {
    case APE_DTYPE_F32: APE_MSDA_DISPATCH(float)
    case APE_DTYPE_F16: APE_MSDA_DISPATCH(__half)
    default: APE_MSDA_DISPATCH(__nv_bfloat16)
  }
#undef APE_MSDA_DISPATCH
}

extern "C" int ape_msda_fwd(const void *value, const int64_t *shapes, const int64_t *starts,
                            const void *loc, const void *attn, void *out, int B, int S, int H, int D,
                            int L, int Q, int P, int dtype, void *stream) {
  return ape_msda_fwd_variant(value, shapes, starts, loc, attn, out, B, S, H, D, L, Q, P, dtype, -1, stream);
}

extern "C" int ape_msda_fused_fwd(const void *value, const int64_t *shapes, const int64_t *starts,
                                  const void *offsets, int64_t offs_row_stride, const void *logits,
                                  int64_t logit_row_stride, const float *ref, int ref_dim, void *out,
                                  int B, int S, int H, int D, int L, int Q, int P, int dtype,
                                  int offs_dtype, void *stream) {
  if (int rc = validate(value, shapes, starts, offsets, logits, out, B, S, H, D, L, Q, P, dtype)) return rc;
  if (offs_dtype != APE_DTYPE_F32 && offs_dtype != APE_DTYPE_F16 && offs_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "msda_fused: unknown offs_dtype %d", offs_dtype);
  if (ref_dim != 2 && ref_dim != 4)
    return fail(APE_ERR_INVALID_ARG, "msda_fused: last dim of reference_points must be 2 or 4, got %d", ref_dim);
  if (offs_row_stride < (int64_t)H * L * P * 2 || logit_row_stride < (int64_t)H * L * P)
    return fail(APE_ERR_INVALID_ARG, "msda_fused: row strides smaller than a row");
  if (B == 0 || Q == 0) return APE_OK;
  if (!ref) return fail(APE_ERR_NULL_PTR, "msda_fused: null reference_points");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MsdaParams p{};
  p.value = value; p.shapes = shapes; p.starts = starts; p.loc = offsets; p.attn = logits; p.ref = ref;
  p.out = out; p.offs_row_stride = offs_row_stride; p.logit_row_stride = logit_row_stride;
  p.B = B; p.S = S; p.H = H; p.L = L; p.Q = Q; p.P = P; p.ref_dim = ref_dim;
  {
    const int eo = dtype_size(offs_dtype);
    p.vec4 = P == 4 && (reinterpret_cast<uintptr_t>(offsets) & 15) == 0 && (offs_row_stride * eo) % 16 == 0 &&
             (reinterpret_cast<uintptr_t>(logits) & (4 * eo - 1)) == 0 && (logit_row_stride * eo) % (4 * eo) == 0;
  }
  const int row_bytes = D * dtype_size(dtype);
  const int lpr = row_bytes / 16;
  if (row_bytes % 16 != 0 || !is_pow2(lpr) || L > kMaxLevels)
    return fail(APE_ERR_UNSUPPORTED, "msda_fused: D=%d dtype=%d L=%d not supported", D, dtype, L);
  const int R = threads_for(lpr) / lpr;
  if ((size_t)R * ((L * P) | 1) * 20 > 200 * 1024)
    return fail(APE_ERR_UNSUPPORTED, "msda_fused: L*P=%d too large for shared memory", L * P);
  p.ht_log2 = ilog2(default_ht(H, Q, R));
#define APE_FUSED_DISPATCH(T)                                                           \
  switch (offs_dtype) {                                                                 \
    case APE_DTYPE_F32: return dispatch_lpr_fused<T, float>(lpr, p, st);                \
    case APE_DTYPE_F16: return dispatch_lpr_fused<T, __half>(lpr, p, st);               \
    default: return dispatch_lpr_fused<T, __nv_bfloat16>(lpr, p, st);                   \
  }
  switch (dtype) {
    case APE_DTYPE_F32: APE_FUSED_DISPATCH(float)
    case APE_DTYPE_F16: APE_FUSED_DISPATCH(__half)
    default: APE_FUSED_DISPATCH(__nv_bfloat16)
  }
#undef APE_FUSED_DISPATCH
}
