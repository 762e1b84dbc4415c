// vlf_fold.cu — VisionLanguageFusion for N > 1 language tokens (phrase / expression / fused-vocabulary prompts) in the
// folded form of BiAttentionBlock.folded (ape_b200/layers/vision_language_fusion.py).  Per head h and language token n the
// language side is folded into 256-vectors of the vision space:
//     qa[h,n] = scale W_q,h^T k[h,n],   qc[h,n] = scale b_q,h . k[h,n],   U[h,n] = W_out_v,h val_l[h,n]
// so that nothing of width 2048 is ever formed over the S vision tokens:
//   vision side   out_s = v_s + gamma (sum_h sum_n softmax_n(v_s . qa[h,n] + qc[h,n]) U[h,n] + b_out_v)   (vlf_fold_vision)
//   language side pooled[h,n] = sum_s softmax_s(v_s . qa[h,n]) v_s    (qc cancels; split over S, vlf_fold_pool + combine)
// The +-5e4 clamps and the global-max shift of fuse_helper.py:88-110 are softmax-invariant translations as long as they do
// not bind (see attn_xfwd.cu); both kernels evaluate the unclamped softmaxes, as ape_attn_cross_fwd does.
//
// Operands: v [B*S, 256] 16-bit (row pitch ldv), qa / U [B, NH, N, 256] 16-bit contiguous, qc [B, NH, N] fp32.  Every
// 64 x 64 operand box is a TMA load with the 128-byte swizzle (attn.cuh's maps); rows past a (b, h) block of keys belong to
// the next block or lie past the tensor (zero fill) and are masked.
//
// vlf_fold_vision_kernel: one CTA = 64 rows of v (one consumer warpgroup, O = 64 x 256 fp32 = 128 registers per thread, as
// ape_attn_cross_fwd's 256-channel heads) + one TMA producer warp.  The eight heads are normalised separately but summed
// into ONE accumulator, so each head's P is normalised before its P.U MMA: with more than one key block a statistics pass
// (Q K^T only: row max and sum) precedes the P.U pass; with N <= 64 the one score block serves both.
// vlf_fold_pool_kernel: queries are the B * NH * N rows of qa (all heads of an image share the keys and values v), keys =
// values = v, one shared-memory tile per key block serves as both MMA operands.  The S keys of an image are split into
// `nsplit` chunks so that small N still fills the machine; each CTA writes its unnormalised O and (max, sum) and
// vlf_fold_combine_kernel folds the chunks in a fixed order (deterministic).
#include <algorithm>

#include "attn.cuh"

namespace ape {
namespace {

using attn::ex2;
using attn::pack2;

constexpr int C = 256, NCH = 4, KB = 64;  // channels, 64-channel chunks, keys per block
constexpr float kLog2e = 1.4426950408889634f;

struct alignas(1024) VisionSmem {
  uint8_t q[NCH][64 * 128];
  uint8_t k[2][NCH][KB * 128];
  uint8_t u[2][NCH][KB * 128];
  uint64_t q_full, k_full[2], k_empty[2], u_full[2], u_empty[2];
};

struct alignas(1024) PoolSmem {
  uint8_t q[NCH][64 * 128];
  uint8_t kv[2][NCH][KB * 128];
  uint64_t q_full, kv_full[2], kv_empty[2];
};

// DEV (vlf_fold_vision_dev_kernel): the text is padded to N tokens per (b, h) block and only the first *n_dev (clamped to
// [1, N]) are keys; the key blocks past them are not loaded, and whether the statistics pass runs is decided from N alone, so
// the kernel's arithmetic follows the padded shape whatever the prompt.
template <typename T, bool DEV>
__device__ __forceinline__ void fold_vision(const CUtensorMap &map_v, const CUtensorMap &map_qa, const CUtensorMap &map_u,
                                            const T *resid, long long ldv, const float *__restrict__ qc, const float *__restrict__ gamma,
                                            const float *__restrict__ bias, T *out, long long ldo, int S, int N, int NH,
                                            const int *n_dev) {
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  VisionSmem &s = *reinterpret_cast<VisionSmem *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x, b = blockIdx.y;
  const int nkb = (N + KB - 1) / KB;
  const bool two_pass = nkb > 1;

  if (warp == 4 && lane == 0) {
    tc::prefetch_tensormap(&map_v);
    tc::prefetch_tensormap(&map_qa);
    tc::prefetch_tensormap(&map_u);
    tc::mbar_init(&s.q_full, 1);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&s.k_full[i], 1);
      tc::mbar_init(&s.k_empty[i], 4);  // one arrival per consumer warp
      tc::mbar_init(&s.u_full[i], 1);
      tc::mbar_init(&s.u_empty[i], 4);
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  int n_live = N, nkb_live = nkb;  // keys in use and their blocks (a kernel before this one writes *n_dev)
  if constexpr (DEV) {
    n_live = min(max(*n_dev, 1), N);
    nkb_live = (n_live + KB - 1) / KB;
  }

  if (warp == 4) {
    // ===================== TMA producer: Q once, then per head [K blocks (statistics pass)] + (K, U) blocks =====================
    if (lane == 0) {
      tc::mbar_expect_tx(&s.q_full, NCH * 64 * 128);
#pragma unroll
      for (int c = 0; c < NCH; ++c) tc::tma_load_2d(s.q[c], &map_v, &s.q_full, c * 64, b * S + tile * 64);
      int kj = 0, uj = 0;
      auto load_k = [&](int row) {
        const int i = kj & 1, n = kj >> 1;
        tc::mbar_wait(&s.k_empty[i], (n & 1) ^ 1);
        tc::mbar_expect_tx(&s.k_full[i], NCH * KB * 128);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tc::tma_load_2d(s.k[i][c], &map_qa, &s.k_full[i], c * 64, row);
        ++kj;
      };
      for (int h = 0; h < NH; ++h) {
        const int row0 = (b * NH + h) * N;
        if (two_pass)
          for (int j = 0; j < nkb_live; ++j) load_k(row0 + j * KB);
        for (int j = 0; j < nkb_live; ++j) {
          load_k(row0 + j * KB);
          const int i = uj & 1, n = uj >> 1;
          tc::mbar_wait(&s.u_empty[i], (n & 1) ^ 1);
          tc::mbar_expect_tx(&s.u_full[i], NCH * KB * 128);
#pragma unroll
          for (int c = 0; c < NCH; ++c) tc::tma_load_2d(s.u[i][c], &map_u, &s.u_full[i], c * 64, row0 + j * KB);
          ++uj;
        }
      }
    }
    __syncwarp();
    return;
  }

  // ===================== consumer warpgroup: rows 16 * warp + lane / 4 + 8 hh (hh = 0, 1) =====================
  const int tq = lane & 3;
  float o[NCH][32];
#pragma unroll
  for (int c = 0; c < NCH; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
  tc::mbar_wait(&s.q_full, 0);
  int kj = 0, uj = 0;

  // scores of key block j of head h in the log2 domain: (v . qa + qc) * log2(e), keys >= n_live at -inf
  auto scores = [&](float (&sc)[32], const float *qch, int j) {
    const int i = kj & 1, n = kj >> 1;
    tc::mbar_wait(&s.k_full[i], n & 1);
    tc::wgmma_fence();
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const uint64_t dq = tc::make_smem_desc_sw128(tc::smem_u32(s.q[c]));
      const uint64_t dk = tc::make_smem_desc_sw128(tc::smem_u32(s.k[i][c]));
#pragma unroll
      for (int k = 0; k < 4; ++k) tc::Wgmma<64, T>::template ss<0>(sc, dq + 2 * k, dk + 2 * k, (c | k) != 0);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::fence_regs<32>(sc);
    if (lane == 0) tc::mbar_arrive(&s.k_empty[i]);
    ++kj;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = j * KB + 8 * jj + 2 * tq + e;
        const float bq = key < n_live ? __ldg(qch + key) : 0.f;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float &x = sc[4 * jj + 2 * hh + e];
          x = key < n_live ? (x + bq) * kLog2e : -INFINITY;
        }
      }
  };
  auto quad_max = [&](const float (&sc)[32], int hh) {
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) mx = fmaxf(mx, sc[4 * jj + 2 * hh + e]);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    return fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
  };

  for (int h = 0; h < NH; ++h) {
    const float *qch = qc + ((size_t)b * NH + h) * N;
    float m[2] = {-INFINITY, -INFINITY}, inv[2] = {0.f, 0.f};
    if (two_pass) {  // statistics pass: exact row max and sum of the head's softmax
      float l[2] = {0.f, 0.f};
      for (int j = 0; j < nkb_live; ++j) {
        float sc[32];
        scores(sc, qch, j);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const float m_new = fmaxf(m[hh], quad_max(sc, hh));  // finite from block 0 on: key 0 is always valid
          l[hh] *= m[hh] == -INFINITY ? 0.f : ex2(m[hh] - m_new);
          m[hh] = m_new;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) l[hh] += ex2(sc[4 * jj + 2 * hh + e] - m_new);
        }
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
        inv[hh] = 1.f / l[hh];
      }
    }
    for (int j = 0; j < nkb_live; ++j) {
      float sc[32];
      scores(sc, qch, j);
      if (!two_pass) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) m[hh] = quad_max(sc, hh);
      }
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int e = 0; e < 2; ++e) sc[4 * jj + 2 * hh + e] = ex2(sc[4 * jj + 2 * hh + e] - m[hh]);
      if (!two_pass) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float l = 0.f;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) l += sc[4 * jj + 2 * hh] + sc[4 * jj + 2 * hh + 1];
          l += __shfl_xor_sync(0xffffffffu, l, 1);
          l += __shfl_xor_sync(0xffffffffu, l, 2);
          inv[hh] = 1.f / l;
        }
      }
      uint32_t pa[4][4];  // normalised P of this head as the A operand of four m64k16 MMAs
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          pa[jj >> 1][2 * (jj & 1) + hh] = pack2<T>(sc[4 * jj + 2 * hh] * inv[hh], sc[4 * jj + 2 * hh + 1] * inv[hh]);
      const int i = uj & 1, n = uj >> 1;
      tc::mbar_wait(&s.u_full[i], n & 1);
#pragma unroll
      for (int c = 0; c < NCH; ++c) tc::fence_regs<32>(o[c]);
      tc::wgmma_fence();
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const uint64_t du = tc::make_smem_desc_sw128(tc::smem_u32(s.u[i][c]));
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) tc::Wgmma<64, T>::template rs<1>(o[c], pa[kk], du + 128 * kk, 1);
      }
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < NCH; ++c) tc::fence_regs<32>(o[c]);
      if (lane == 0) tc::mbar_arrive(&s.u_empty[i]);
      ++uj;
    }
  }

  // ===================== epilogue: out = v + gamma * (O + b_out_v), one rounding =====================
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = tile * 64 + warp * 16 + (lane >> 2) + 8 * hh;
    if (r >= S) continue;
    const size_t row = (size_t)b * S + r;
    const T *src = resid + row * ldv;
    T *dst = out + row * ldo;
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int col = c * 64 + 8 * jj + 2 * tq;
        const uint32_t raw = *reinterpret_cast<const uint32_t *>(src + col);
        const T *t2 = reinterpret_cast<const T *>(&raw);
        const float2 g = *reinterpret_cast<const float2 *>(gamma + col), bo = *reinterpret_cast<const float2 *>(bias + col);
        const float y0 = fmaf(g.x, o[c][4 * jj + 2 * hh] + bo.x, Elem<T>::to_f(t2[0]));
        const float y1 = fmaf(g.y, o[c][4 * jj + 2 * hh + 1] + bo.y, Elem<T>::to_f(t2[1]));
        *reinterpret_cast<uint32_t *>(dst + col) = pack2<T>(y0, y1);
      }
  }
}

template <typename T>
__global__ void __launch_bounds__(160, 1)
vlf_fold_vision_kernel(const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_qa,
                       const __grid_constant__ CUtensorMap map_u, const T *resid, long long ldv, const float *__restrict__ qc,
                       const float *__restrict__ gamma, const float *__restrict__ bias, T *out, long long ldo, int S, int N,
                       int NH) {
  fold_vision<T, false>(map_v, map_qa, map_u, resid, ldv, qc, gamma, bias, out, ldo, S, N, NH, nullptr);
}

template <typename T>
__global__ void __launch_bounds__(160, 1)
vlf_fold_vision_dev_kernel(const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_qa,
                           const __grid_constant__ CUtensorMap map_u, const T *resid, long long ldv, const float *__restrict__ qc,
                           const float *__restrict__ gamma, const float *__restrict__ bias, T *out, long long ldo, int S, int N,
                           int NH, const int *n_dev) {
  fold_vision<T, true>(map_v, map_qa, map_u, resid, ldv, qc, gamma, bias, out, ldo, S, N, NH, n_dev);
}

// grid (ceil(R / 64), nsplit, B), R = NH * N query rows per image; chunk c covers keys [c * chunk, min(S, (c + 1) * chunk)).
// DEV (vlf_fold_pool_dev_kernel): rows r of token r % N >= *n_dev (clamped to [1, N]) are padding; a tile of padding rows
// alone returns at once, and the combine writes zeros for them without reading their partials.
template <typename T, bool DEV>
__device__ __forceinline__ void fold_pool(const CUtensorMap &map_qa, const CUtensorMap &map_v, float *__restrict__ part_o,
                                          float2 *__restrict__ part_ml, int S, int R, int chunk, int N, const int *n_dev) {
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  PoolSmem &s = *reinterpret_cast<PoolSmem *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x, split = blockIdx.y, b = blockIdx.z, nsplit = gridDim.y;
  const int k0 = split * chunk, nk = min(chunk, S - k0);  // nk >= 1: the host sizes chunks so none is empty
  const int nkb = (nk + KB - 1) / KB;

  if (warp == 4 && lane == 0) {
    tc::prefetch_tensormap(&map_qa);
    tc::prefetch_tensormap(&map_v);
    tc::mbar_init(&s.q_full, 1);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&s.kv_full[i], 1);
      tc::mbar_init(&s.kv_empty[i], 4);
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if constexpr (DEV) {  // every row of the tile is a padding token: nothing of it is read
    const int n_live = min(max(*n_dev, 1), N);
    bool live = false;
    for (int r = tile * 64; r < min(R, tile * 64 + 64) && !live; ++r) live = r % N < n_live;
    if (!live) return;
  }

  if (warp == 4) {
    if (lane == 0) {
      tc::mbar_expect_tx(&s.q_full, NCH * 64 * 128);
#pragma unroll
      for (int c = 0; c < NCH; ++c) tc::tma_load_2d(s.q[c], &map_qa, &s.q_full, c * 64, b * R + tile * 64);
      for (int j = 0; j < nkb; ++j) {
        const int i = j & 1, n = j >> 1;
        tc::mbar_wait(&s.kv_empty[i], (n & 1) ^ 1);
        tc::mbar_expect_tx(&s.kv_full[i], NCH * KB * 128);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tc::tma_load_2d(s.kv[i][c], &map_v, &s.kv_full[i], c * 64, b * S + k0 + j * KB);
      }
    }
    __syncwarp();
    return;
  }

  const int tq = lane & 3;
  float o[NCH][32];
#pragma unroll
  for (int c = 0; c < NCH; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  tc::mbar_wait(&s.q_full, 0);
  for (int j = 0; j < nkb; ++j) {
    const int i = j & 1, n = j >> 1;
    float sc[32];
    tc::mbar_wait(&s.kv_full[i], n & 1);
    tc::wgmma_fence();
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const uint64_t dq = tc::make_smem_desc_sw128(tc::smem_u32(s.q[c]));
      const uint64_t dk = tc::make_smem_desc_sw128(tc::smem_u32(s.kv[i][c]));
#pragma unroll
      for (int k = 0; k < 4; ++k) tc::Wgmma<64, T>::template ss<0>(sc, dq + 2 * k, dk + 2 * k, (c | k) != 0);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::fence_regs<32>(sc);
    if ((j + 1) * KB > nk) {  // the chunk's last, partial block: keys past the chunk (next chunk / image, zero fill) masked
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (j * KB + 8 * jj + 2 * tq + e >= nk) sc[4 * jj + e] = sc[4 * jj + 2 + e] = -INFINITY;
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) mx = fmaxf(mx, sc[4 * jj + 2 * hh + e]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hh], mx * kLog2e);
      alpha[hh] = m_run[hh] == -INFINITY ? 0.f : ex2(m_run[hh] - m_new);
      m_run[hh] = m_new;
      m_use[hh] = m_new == -INFINITY ? 0.f : m_new;
      l[hh] *= alpha[hh];
    }
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int q = 0; q < 32; ++q) o[c][q] *= alpha[(q >> 1) & 1];
    uint32_t pa[4][4];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float e0 = ex2(fmaf(sc[4 * jj + 2 * hh], kLog2e, -m_use[hh]));
        const float e1 = ex2(fmaf(sc[4 * jj + 2 * hh + 1], kLog2e, -m_use[hh]));
        l[hh] += e0 + e1;
        pa[jj >> 1][2 * (jj & 1) + hh] = pack2<T>(e0, e1);
      }
#pragma unroll
    for (int c = 0; c < NCH; ++c) tc::fence_regs<32>(o[c]);
    tc::wgmma_fence();
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const uint64_t dv = tc::make_smem_desc_sw128(tc::smem_u32(s.kv[i][c]));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) tc::Wgmma<64, T>::template rs<1>(o[c], pa[kk], dv + 128 * kk, 1);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NCH; ++c) tc::fence_regs<32>(o[c]);
    if (lane == 0) tc::mbar_arrive(&s.kv_empty[i]);  // the tile served as keys and values; both MMAs are done
  }

  // partials of the chunk: unnormalised O (fp32) and (max in the log2 domain, sum) per query row
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    const int r = tile * 64 + warp * 16 + (lane >> 2) + 8 * hh;
    if (r >= R) continue;
    const size_t prow = ((size_t)b * nsplit + split) * R + r;
    float *dst = part_o + prow * C + 2 * tq;
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<float2 *>(dst + c * 64 + 8 * jj) = make_float2(o[c][4 * jj + 2 * hh], o[c][4 * jj + 2 * hh + 1]);
    if (tq == 0) part_ml[prow] = make_float2(m_run[hh], l[hh]);
  }
}

template <typename T>
__global__ void __launch_bounds__(160, 1)
vlf_fold_pool_kernel(const __grid_constant__ CUtensorMap map_qa, const __grid_constant__ CUtensorMap map_v,
                     float *__restrict__ part_o, float2 *__restrict__ part_ml, int S, int R, int chunk) {
  fold_pool<T, false>(map_qa, map_v, part_o, part_ml, S, R, chunk, 1, nullptr);
}

template <typename T>
__global__ void __launch_bounds__(160, 1)
vlf_fold_pool_dev_kernel(const __grid_constant__ CUtensorMap map_qa, const __grid_constant__ CUtensorMap map_v,
                         float *__restrict__ part_o, float2 *__restrict__ part_ml, int S, int R, int chunk, int N, const int *n_dev) {
  fold_pool<T, true>(map_qa, map_v, part_o, part_ml, S, R, chunk, N, n_dev);
}

// One CTA of 256 threads per query row (b, h, n): pooled[b * N + n, h * 256 + col] = sum_c w_c O_c / sum_c w_c l_c with
// w_c = 2^(m_c - max_c m_c), chunks in ascending order.
template <typename T>
__global__ void __launch_bounds__(256)
vlf_fold_combine_kernel(const float *__restrict__ part_o, const float2 *__restrict__ part_ml, T *__restrict__ pooled,
                        long long ldp, int R, int N, int nsplit) {
  pdl_prologue();
  const int b = blockIdx.y, r = blockIdx.x, col = threadIdx.x;
  const size_t base = (size_t)b * nsplit * R + r;
  float mx = -INFINITY;
  for (int c = 0; c < nsplit; ++c) mx = fmaxf(mx, part_ml[base + (size_t)c * R].x);
  float acc = 0.f, den = 0.f;
  for (int c = 0; c < nsplit; ++c) {
    const float2 ml = part_ml[base + (size_t)c * R];
    const float w = ex2(ml.x - mx);
    den = fmaf(w, ml.y, den);
    acc = fmaf(w, part_o[(base + (size_t)c * R) * C + col], acc);
  }
  const int h = r / N, n = r - h * N;
  pooled[((size_t)b * N + n) * ldp + h * C + col] = Elem<T>::from_f(acc / den);
}

// The combine of vlf_fold_pool_dev_kernel: padding rows (token >= *n_dev, clamped to [1, N]) are written as zeros, so every row
// of the pooled output is finite whatever the prompt; the others as vlf_fold_combine_kernel.
template <typename T>
__global__ void __launch_bounds__(256)
vlf_fold_combine_dev_kernel(const float *__restrict__ part_o, const float2 *__restrict__ part_ml, T *__restrict__ pooled,
                            long long ldp, int R, int N, int nsplit, const int *__restrict__ n_dev) {
  pdl_prologue();
  const int b = blockIdx.y, r = blockIdx.x, col = threadIdx.x;
  const int h = r / N, n = r - h * N;
  T *dst = pooled + ((size_t)b * N + n) * ldp + h * C + col;
  if (n >= min(max(*n_dev, 1), N)) {
    *dst = Elem<T>::from_f(0.f);
    return;
  }
  const size_t base = (size_t)b * nsplit * R + r;
  float mx = -INFINITY;
  for (int c = 0; c < nsplit; ++c) mx = fmaxf(mx, part_ml[base + (size_t)c * R].x);
  float acc = 0.f, den = 0.f;
  for (int c = 0; c < nsplit; ++c) {
    const float2 ml = part_ml[base + (size_t)c * R];
    const float w = ex2(ml.x - mx);
    den = fmaf(w, ml.y, den);
    acc = fmaf(w, part_o[(base + (size_t)c * R) * C + col], acc);
  }
  *dst = Elem<T>::from_f(acc / den);
}

// Key chunks of the pooling: enough CTAs for two per SM of an H100 SXM, at least 1024 keys each.
int pool_splits(int B, int S, int R, int *chunk) {
  const int tiles = (R + 63) / 64 * B;
  int nsplit = std::max(1, std::min((264 + tiles - 1) / tiles, (S + 1023) / 1024));
  *chunk = ((S + nsplit - 1) / nsplit + KB - 1) / KB * KB;
  return (S + *chunk - 1) / *chunk;  // every chunk holds at least one key
}

int check_common(const char *what, int B, int S, int N, int NH, int dtype) {
  if (dtype != APE_DTYPE_F16 && dtype != APE_DTYPE_BF16) return fail(APE_ERR_INVALID_ARG, "%s: fp16 / bf16 only (dtype %d)", what, dtype);
  if (B <= 0 || B > 65535 || S <= 0 || N <= 0 || NH <= 0 || (long long)B * S >= (1LL << 31) ||
      (long long)B * NH * N >= (1LL << 31) || (S + 63) / 64 > 2147483647 / 64)
    return fail(APE_ERR_UNSUPPORTED, "%s: B=%d S=%d N=%d NH=%d out of range", what, B, S, N, NH);
  return APE_OK;
}

// the shared-memory opt-in, once per kernel instantiation (the caller's static flag)
template <typename K>
int set_smem(bool &set, K kernel, size_t bytes, const char *what) {
  if (!set) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return fail((int)e, "%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
    set = true;
  }
  return APE_OK;
}

template <typename T>
int launch_vision(const CUtensorMap &mv, const CUtensorMap &mqa, const CUtensorMap &mu, const void *v, int64_t ldv, const float *qc,
                  const float *gamma, const float *bias, void *out, int64_t ldo, int B, int S, int N, int NH, cudaStream_t st,
                  const int *n_dev = nullptr) {
  const dim3 grid((unsigned)((S + 63) / 64), (unsigned)B);
  if (n_dev) {
    auto k = vlf_fold_vision_dev_kernel<T>;
    static bool set = false;
    if (int rc = set_smem(set, k, sizeof(VisionSmem) + 1024, "vlf_fold_vision_dev")) return rc;
    APE_LAUNCH(k, grid, 160, sizeof(VisionSmem) + 1024, st, mv, mqa, mu, (const T *)v, (long long)ldv, qc, gamma, bias, (T *)out,
               (long long)ldo, S, N, NH, n_dev);
    return check_launch("vlf_fold_vision_dev_kernel");
  }
  auto k = vlf_fold_vision_kernel<T>;
  static bool set = false;
  if (int rc = set_smem(set, k, sizeof(VisionSmem) + 1024, "vlf_fold_vision")) return rc;
  APE_LAUNCH(k, grid, 160, sizeof(VisionSmem) + 1024, st, mv, mqa, mu, (const T *)v, (long long)ldv, qc, gamma, bias, (T *)out,
             (long long)ldo, S, N, NH);
  return check_launch("vlf_fold_vision_kernel");
}

template <typename T>
int launch_pool(const CUtensorMap &mqa, const CUtensorMap &mv, float *part_o, float2 *part_ml, void *pooled, int64_t ldp, int B,
                int S, int N, int R, int nsplit, int chunk, cudaStream_t st, const int *n_dev = nullptr) {
  if (n_dev) {
    auto k = vlf_fold_pool_dev_kernel<T>;
    static bool set = false;
    if (int rc = set_smem(set, k, sizeof(PoolSmem) + 1024, "vlf_fold_pool_dev")) return rc;
    APE_LAUNCH(k, dim3((unsigned)((R + 63) / 64), (unsigned)nsplit, (unsigned)B), 160, sizeof(PoolSmem) + 1024, st, mqa, mv, part_o,
               part_ml, S, R, chunk, N, n_dev);
    if (int rc = check_launch("vlf_fold_pool_dev_kernel")) return rc;
    APE_LAUNCH((vlf_fold_combine_dev_kernel<T>), dim3((unsigned)R, (unsigned)B), 256, 0, st, (const float *)part_o,
               (const float2 *)part_ml, (T *)pooled, (long long)ldp, R, N, nsplit, n_dev);
    return check_launch("vlf_fold_combine_dev_kernel");
  }
  auto k = vlf_fold_pool_kernel<T>;  // T is not in the kernel's signature: the flag must live here, per T
  static bool set = false;
  if (int rc = set_smem(set, k, sizeof(PoolSmem) + 1024, "vlf_fold_pool")) return rc;
  APE_LAUNCH(k, dim3((unsigned)((R + 63) / 64), (unsigned)nsplit, (unsigned)B), 160, sizeof(PoolSmem) + 1024, st, mqa, mv, part_o,
             part_ml, S, R, chunk);
  if (int rc = check_launch("vlf_fold_pool_kernel")) return rc;
  APE_LAUNCH((vlf_fold_combine_kernel<T>), dim3((unsigned)R, (unsigned)B), 256, 0, st, (const float *)part_o,
             (const float2 *)part_ml, (T *)pooled, (long long)ldp, R, N, nsplit);
  return check_launch("vlf_fold_combine_kernel");
}

}  // namespace
}  // namespace ape

using namespace ape;

static int fold_vision_impl(const void *v, int64_t ldv, const void *qa, const void *u, const float *qc, const float *gamma,
                            const float *bias, void *out, int64_t ldo, int B, int S, int N, int NH, int C_, int dtype, void *stream,
                            const int *n_dev) {
  if (int rc = check_common("vlf_fold_vision", B, S, N, NH, dtype)) return rc;
  if (C_ != C) return fail(APE_ERR_UNSUPPORTED, "vlf_fold_vision: %d channels (256 only)", C_);
  if (!v || !qa || !u || !qc || !gamma || !bias || !out) return fail(APE_ERR_NULL_PTR, "vlf_fold_vision: null pointer argument");
  if (ldv < C || ldo < C || ldv % 8 || ldo % 8 ||
      ((reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(qa) | reinterpret_cast<uintptr_t>(u) |
        reinterpret_cast<uintptr_t>(out)) & 15) || ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(bias)) & 7))
    return fail(APE_ERR_INVALID_ARG, "vlf_fold_vision: v / out rows of >= 256 elements, 16-byte aligned; gamma / bias 8-byte aligned");
  CUtensorMap mv, mqa, mu;
  if (int rc = attn::make_map(&mv, v, dtype, (long long)B * S, C, ldv)) return rc;
  if (int rc = attn::make_map(&mqa, qa, dtype, (long long)B * NH * N, C, C)) return rc;
  if (int rc = attn::make_map(&mu, u, dtype, (long long)B * NH * N, C, C)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == APE_DTYPE_F16) return launch_vision<__half>(mv, mqa, mu, v, ldv, qc, gamma, bias, out, ldo, B, S, N, NH, st, n_dev);
  return launch_vision<__nv_bfloat16>(mv, mqa, mu, v, ldv, qc, gamma, bias, out, ldo, B, S, N, NH, st, n_dev);
}

extern "C" int ape_vlf_fold_vision(const void *v, int64_t ldv, const void *qa, const void *u, const float *qc, const float *gamma,
                                   const float *bias, void *out, int64_t ldo, int B, int S, int N, int NH, int C_, int dtype,
                                   void *stream) {
  return fold_vision_impl(v, ldv, qa, u, qc, gamma, bias, out, ldo, B, S, N, NH, C_, dtype, stream, nullptr);
}

extern "C" int ape_vlf_fold_vision_dev(const void *v, int64_t ldv, const void *qa, const void *u, const float *qc, const float *gamma,
                                       const float *bias, void *out, int64_t ldo, int B, int S, int N, int NH, const int *n_dev, int C_,
                                       int dtype, void *stream) {
  if (!n_dev) return fail(APE_ERR_NULL_PTR, "vlf_fold_vision_dev: null n_dev");
  if (reinterpret_cast<uintptr_t>(n_dev) & 3) return fail(APE_ERR_INVALID_ARG, "vlf_fold_vision_dev: n_dev must be a 4-byte aligned int32");
  return fold_vision_impl(v, ldv, qa, u, qc, gamma, bias, out, ldo, B, S, N, NH, C_, dtype, stream, n_dev);
}

extern "C" int64_t ape_vlf_fold_pool_workspace_bytes(int B, int S, int N, int NH) {
  if (B <= 0 || S <= 0 || N <= 0 || NH <= 0) return 0;
  int chunk;
  const int R = NH * N, nsplit = pool_splits(B, S, R, &chunk);
  return (int64_t)B * nsplit * R * (C + 2) * 4;
}

static int fold_pool_impl(const void *v, int64_t ldv, const void *qa, void *workspace, void *pooled, int64_t ldp, int B, int S, int N,
                          int NH, int C_, int dtype, void *stream, const int *n_dev) {
  if (int rc = check_common("vlf_fold_pool", B, S, N, NH, dtype)) return rc;
  if (C_ != C) return fail(APE_ERR_UNSUPPORTED, "vlf_fold_pool: %d channels (256 only)", C_);
  if (!v || !qa || !workspace || !pooled) return fail(APE_ERR_NULL_PTR, "vlf_fold_pool: null pointer argument");
  if (ldv < C || ldv % 8 || ldp < (int64_t)NH * C ||
      ((reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(qa) | reinterpret_cast<uintptr_t>(workspace)) & 15))
    return fail(APE_ERR_INVALID_ARG, "vlf_fold_pool: v rows of >= 256 elements, 16-byte aligned operands, ldp >= NH * 256");
  const int R = NH * N;
  int chunk;
  const int nsplit = pool_splits(B, S, R, &chunk);
  if ((long long)B * nsplit > 65535 * 64LL || nsplit > 65535) return fail(APE_ERR_UNSUPPORTED, "vlf_fold_pool: %d splits", nsplit);
  CUtensorMap mqa, mv;
  if (int rc = attn::make_map(&mqa, qa, dtype, (long long)B * R, C, C)) return rc;
  if (int rc = attn::make_map(&mv, v, dtype, (long long)B * S, C, ldv)) return rc;
  float *part_o = reinterpret_cast<float *>(workspace);
  float2 *part_ml = reinterpret_cast<float2 *>(part_o + (size_t)B * nsplit * R * C);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == APE_DTYPE_F16) return launch_pool<__half>(mqa, mv, part_o, part_ml, pooled, ldp, B, S, N, R, nsplit, chunk, st, n_dev);
  return launch_pool<__nv_bfloat16>(mqa, mv, part_o, part_ml, pooled, ldp, B, S, N, R, nsplit, chunk, st, n_dev);
}

extern "C" int ape_vlf_fold_pool(const void *v, int64_t ldv, const void *qa, void *workspace, void *pooled, int64_t ldp, int B,
                                 int S, int N, int NH, int C_, int dtype, void *stream) {
  return fold_pool_impl(v, ldv, qa, workspace, pooled, ldp, B, S, N, NH, C_, dtype, stream, nullptr);
}

// The split over S and the combine order come from (B, S, N, NH): with N the padded token count they do not depend on *n_dev.
extern "C" int ape_vlf_fold_pool_dev(const void *v, int64_t ldv, const void *qa, void *workspace, void *pooled, int64_t ldp, int B,
                                     int S, int N, int NH, const int *n_dev, int C_, int dtype, void *stream) {
  if (!n_dev) return fail(APE_ERR_NULL_PTR, "vlf_fold_pool_dev: null n_dev");
  if (reinterpret_cast<uintptr_t>(n_dev) & 3) return fail(APE_ERR_INVALID_ARG, "vlf_fold_pool_dev: n_dev must be a 4-byte aligned int32");
  return fold_pool_impl(v, ldv, qa, workspace, pooled, ldp, B, S, N, NH, C_, dtype, stream, n_dev);
}
