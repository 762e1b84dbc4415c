// attn.cuh — flash-attention forward on the Hopper (sm_90a) tensor cores, shared by the ViT / text-tower self-attention
// (attn_fwd.cu) and the vision-language cross attention with wide heads (attn_xfwd.cu).
//
// One CTA = QM = 64 * CWG queries of one (sequence, head); it walks the keys in blocks of 64.  Roles:
//   warpgroups 0..CWG-1  consumers : warpgroup g owns query rows 64g..64g+63.  Per key block j:
//                                    S_j = Q K_j^T   (wgmma m64n64k16, Q and K_j K-major in shared memory, fp32 in registers)
//                                    online softmax in the exp2 domain on the accumulator fragment (a row lives in the 4
//                                    lanes of a quad), P_j rounded to 16 bit;
//                                    O += P_j V_j    (wgmma m64n64k16 per 64-channel chunk of the head, B = V_j in its
//                                                     natural [key][channel] layout = MN-major operand)
//   warp 4 * CWG         producer  : TMA loads of Q once, then K_j / V_j into double buffers (mbarrier full / empty).
// P_IN_SMEM selects where the P.V MMA reads P from: the warpgroup's registers (the S fragment repacked as the A operand,
// no shared-memory traffic) or a 128-byte-swizzled shared-memory tile written by the softmax threads.
// Head dim HD = 64 * NC: Q, K_j, V_j are NC swizzled 64-column chunks each; O is NC x 32 fp32 registers per thread.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "tc.cuh"

namespace ape {
namespace attn {

constexpr int KN = 64;  // keys per block

template <int NC, int CWG, bool P_IN_SMEM>
struct alignas(1024) Smem {
  uint8_t q[NC][CWG * 64 * 128];
  uint8_t k[2][NC][KN * 128];
  uint8_t v[2][NC][KN * 128];
  uint8_t p[P_IN_SMEM ? CWG : 1][P_IN_SMEM ? 64 * 128 : 16];
  uint64_t q_full, k_full[2], k_empty[2], v_full[2], v_empty[2];
};

struct Params {
  void *out;
  long long ldo;                // elements
  int q_seq_rows, kv_seq_rows;  // rows between the starts of consecutive sequences in Q / K,V
  int q_col0, k_col0, v_col0;   // column of head 0 in each tensor (the fused qkv buffer: 0, C, 2C)
  int n_valid;                  // keys >= n_valid of every sequence are masked out
  int q_store_rows;             // query rows >= this (inside a sequence) are not written (packed sequences)
  int causal;                   // key t attends only to keys <= t (text tower, eva02_clip/transformer.py:714-720)
  int heads;
  float *stats_out;             // [rows, heads, 2] (sum, sum of squares) of each row's stored output values, or nullptr
  float scale_log2;             // softmax scale * log2(e)
  const int *out_row_map;       // ROW_MAP kernels: query row r is stored at out / stats_out row out_row_map[r]; -1 = not stored
  const int *seg_start;         // SEG kernels: query row r of the launch also ignores the keys before position seg_start[r]
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (std::is_same<T, __half>::value) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
  } else {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
  }
}

// SEG: several short sequences share one tile (the text tower's length-packed prompts).  Query row r attends key k of its
// tile iff seg_start[r] <= k and k passes the causal / n_valid mask: the causal mask with a lower bound per row.
template <typename T, int NC, int CWG, bool P_IN_SMEM, bool ROW_MAP = false, bool SEG = false>
__global__ void __launch_bounds__(CWG * 128 + 32, NC == 1 ? 2 : 1)
attn_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
            const __grid_constant__ CUtensorMap map_v, const Params p) {
  constexpr int QM = 64 * CWG, HD = 64 * NC;
  using S = Smem<NC, CWG, P_IN_SMEM>;
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  S &s = *reinterpret_cast<S *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qblk = blockIdx.x, head = blockIdx.y, seq = blockIdx.z;
  const int qrow0 = seq * p.q_seq_rows + qblk * QM;  // first query row of this tile
  const int krow0 = seq * p.kv_seq_rows;
  // key blocks that hold at least one key some row of this tile attends to
  const int nkv = ((p.causal ? min(p.n_valid, (qblk + 1) * QM) : p.n_valid) + KN - 1) / KN;

  if (warp == 4 * CWG && lane == 0) {
    tc::prefetch_tensormap(&map_q);
    tc::prefetch_tensormap(&map_k);
    tc::prefetch_tensormap(&map_v);
    tc::mbar_init(&s.q_full, 1);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      tc::mbar_init(&s.k_full[b], 1);
      tc::mbar_init(&s.k_empty[b], 4 * CWG);  // one arrival per consumer warp
      tc::mbar_init(&s.v_full[b], 1);
      tc::mbar_init(&s.v_empty[b], 4 * CWG);
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // barriers are set up; the previous kernel's output (q / k / v) may be read from here on

  if (warp == 4 * CWG) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      tc::mbar_expect_tx(&s.q_full, NC * QM * 128);
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int g = 0; g < CWG; ++g)  // the box is 64 rows x 64 channels
          tc::tma_load_2d(s.q[c] + g * 64 * 128, &map_q, &s.q_full, p.q_col0 + head * HD + c * 64, qrow0 + g * 64);
      for (int j = 0; j < nkv; ++j) {
        const int b = j & 1, n = j >> 1;
        tc::mbar_wait(&s.k_empty[b], (n & 1) ^ 1);
        tc::mbar_expect_tx(&s.k_full[b], NC * KN * 128);
#pragma unroll
        for (int c = 0; c < NC; ++c) tc::tma_load_2d(s.k[b][c], &map_k, &s.k_full[b], p.k_col0 + head * HD + c * 64, krow0 + j * KN);
        tc::mbar_wait(&s.v_empty[b], (n & 1) ^ 1);
        tc::mbar_expect_tx(&s.v_full[b], NC * KN * 128);
#pragma unroll
        for (int c = 0; c < NC; ++c) tc::tma_load_2d(s.v[b][c], &map_v, &s.v_full[b], p.v_col0 + head * HD + c * 64, krow0 + j * KN);
      }
    }
    __syncwarp();
    return;
  }

  // ===================== consumers: warpgroup g, rows r = 16 * (warp % 4) + lane / 4 + 8 h (h = 0, 1) =====================
  const int g = warp >> 2, w4 = warp & 3, tq = lane & 3;
  int qpos[2];  // position of the thread's two query rows inside the sequence
#pragma unroll
  for (int h = 0; h < 2; ++h) qpos[h] = qblk * QM + g * 64 + w4 * 16 + (lane >> 2) + 8 * h;
  int seg_lo[2] = {0, 0};  // SEG: first key position of the thread's two rows
  if constexpr (SEG) {
#pragma unroll
    for (int h = 0; h < 2; ++h) seg_lo[h] = p.seg_start[(size_t)seq * p.q_seq_rows + qpos[h]];
  }
  float o[NC][32];
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  tc::mbar_wait(&s.q_full, 0);

  for (int j = 0; j < nkv; ++j) {
    const int b = j & 1, n = j >> 1;
    float sc[32];
    tc::mbar_wait(&s.k_full[b], n & 1);
    tc::wgmma_fence();
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const uint64_t dq = tc::make_smem_desc_sw128(tc::smem_u32(s.q[c] + g * 64 * 128));
      const uint64_t dk = tc::make_smem_desc_sw128(tc::smem_u32(s.k[b][c]));
#pragma unroll
      for (int k = 0; k < 4; ++k) tc::Wgmma<64, T>::template ss<0>(sc, dq + 2 * k, dk + 2 * k, (c | k) != 0);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::fence_regs<32>(sc);
    if (lane == 0) tc::mbar_arrive(&s.k_empty[b]);  // K_j may be replaced by K_{j+2}

    // masking: padded keys (>= n_valid) and, causal, keys after the query's own position score -inf: ex2(-inf) = 0.
    // Only blocks that hold such a key for some row of the warpgroup run the compares (the last partial block of n_valid,
    // and the causal diagonal); in every other block they would leave all scores as they are.
    const bool mask = (j + 1) * KN > p.n_valid || (p.causal && (j + 1) * KN - 1 > qblk * QM + g * 64);
    if (mask) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int kvalid = (p.causal ? min(p.n_valid, qpos[h] + 1) : p.n_valid) - j * KN;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * jj + 2 * tq + e >= kvalid) sc[4 * jj + 2 * h + e] = -INFINITY;
      }
    }
    if constexpr (SEG) {
      // the lower bound, likewise only where it masks something: a warp runs the compares of a block when one of its 16
      // rows starts after the block's first key
      if (__any_sync(0xffffffffu, max(seg_lo[0], seg_lo[1]) > j * KN)) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int klo = seg_lo[h] - j * KN;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * jj + 2 * tq + e < klo) sc[4 * jj + 2 * h + e] = -INFINITY;
        }
      }
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) mx = fmaxf(mx, sc[4 * jj + 2 * h + e]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx * p.scale_log2);
      alpha[h] = m_run[h] == -INFINITY ? 0.f : ex2(m_run[h] - m_new);
      m_run[h] = m_new;
      m_use[h] = m_new == -INFINITY ? 0.f : m_new;  // a row with no key yet: every exponential is 0
      l[h] *= alpha[h];
    }
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] *= alpha[(i >> 1) & 1];
    uint32_t pa[4][4];  // P_j as the A operand of four m64k16 MMAs (16 keys each)
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float e0 = ex2(fmaf(sc[4 * jj + 2 * h], p.scale_log2, -m_use[h]));
        const float e1 = ex2(fmaf(sc[4 * jj + 2 * h + 1], p.scale_log2, -m_use[h]));
        l[h] += e0 + e1;
        pa[jj >> 1][2 * (jj & 1) + h] = pack2<T>(e0, e1);
      }
    if constexpr (P_IN_SMEM) {
      // rows of 64 keys = 128 bytes, 16-byte chunk jj of row r at (jj ^ (r % 8)) (the swizzle TMA would write)
      const uint32_t pbase = tc::smem_u32(s.p[g]);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = w4 * 16 + (lane >> 2) + 8 * h;
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(pbase + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * tq),
                       "r"(pa[jj >> 1][2 * (jj & 1) + h]) : "memory");
        }
      tc::fence_proxy_async();
      asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");  // the whole P tile of the warpgroup is written
    }
    tc::mbar_wait(&s.v_full[b], n & 1);
#pragma unroll
    for (int c = 0; c < NC; ++c) tc::fence_regs<32>(o[c]);
    tc::wgmma_fence();
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const uint64_t dv = tc::make_smem_desc_sw128(tc::smem_u32(s.v[b][c]));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // B (MN-major): +16 key rows = 2 KB per step
        if constexpr (P_IN_SMEM) {
          const uint64_t dp = tc::make_smem_desc_sw128(tc::smem_u32(s.p[g]));
          tc::Wgmma<64, T>::template ss<1>(o[c], dp + 2 * kk, dv + 128 * kk, 1);
        } else {
          tc::Wgmma<64, T>::template rs<1>(o[c], pa[kk], dv + 128 * kk, 1);
        }
      }
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NC; ++c) tc::fence_regs<32>(o[c]);
    if (lane == 0) tc::mbar_arrive(&s.v_empty[b]);  // V_j (and the P tile) may be replaced
  }

  // ===================== epilogue: O / l, 16-bit, optional per-(row, head) statistics =====================
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    const float inv = 1.f / l[h];
    // packed sequences: rows past the sequence belong to the next one and must not be written
    bool store_row = qpos[h] < p.q_store_rows;
    size_t row = (size_t)seq * p.q_seq_rows + qpos[h];
    if constexpr (ROW_MAP) {  // e.g. padded windows back to raster order; pad rows map to -1
      const int mapped = store_row ? p.out_row_map[row] : -1;
      store_row = mapped >= 0;
      row = (size_t)(store_row ? mapped : 0);
    }
    T *dst = reinterpret_cast<T *>(p.out) + row * p.ldo + head * HD + 2 * tq;
    float st_sum = 0.f, st_sq = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const uint32_t pk = pack2<T>(o[c][4 * jj + 2 * h] * inv, o[c][4 * jj + 2 * h + 1] * inv);
        if (store_row) *reinterpret_cast<uint32_t *>(dst + c * 64 + 8 * jj) = pk;
        if (p.stats_out != nullptr) {  // statistics of the values as stored, for the LayerNorm folded into the next GEMM
          const T *t2 = reinterpret_cast<const T *>(&pk);
          const float f0 = Elem<T>::to_f(t2[0]), f1 = Elem<T>::to_f(t2[1]);
          st_sum += f0 + f1;
          st_sq += f0 * f0 + f1 * f1;
        }
      }
    if (p.stats_out != nullptr) {
      st_sum += __shfl_xor_sync(0xffffffffu, st_sum, 1);
      st_sq += __shfl_xor_sync(0xffffffffu, st_sq, 1);
      st_sum += __shfl_xor_sync(0xffffffffu, st_sum, 2);
      st_sq += __shfl_xor_sync(0xffffffffu, st_sq, 2);
      if (tq == 0 && store_row)
        *reinterpret_cast<float2 *>(p.stats_out + (row * p.heads + head) * 2) = make_float2(st_sum, st_sq);
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [rows, cols] 16-bit row-major tensor with pitch `ld` elements, box = 64 channels x 64 rows, 128-byte swizzle; rows past
// the tensor read as zeros.
inline int make_map(CUtensorMap *map, const void *base, int dtype, long long rows, long long cols, long long ld) {
  static EncodeTiledFn enc = [] {
    void *ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      return reinterpret_cast<EncodeTiledFn>(ptr);
    return (EncodeTiledFn) nullptr;
  }();
  if (!enc) return fail(APE_ERR_UNSUPPORTED, "attn: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)KN};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, dtype == APE_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                   const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(APE_ERR_INVALID_ARG, "attn: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return APE_OK;
}

// grid = (query rows per sequence / (64 * CWG), heads, sequences)
template <typename T, int NC, int CWG, bool P_IN_SMEM, bool ROW_MAP = false, bool SEG = false>
int launch(const CUtensorMap &mq, const CUtensorMap &mk, const CUtensorMap &mv, const Params &p, dim3 grid, cudaStream_t st) {
  const size_t smem = sizeof(Smem<NC, CWG, P_IN_SMEM>) + 1024;
  auto k = attn_kernel<T, NC, CWG, P_IN_SMEM, ROW_MAP, SEG>;
  static bool set = false;
  if (!set) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "attn: cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
    set = true;
  }
  APE_LAUNCH(k, grid, CWG * 128 + 32, smem, st, mq, mk, mv, p);
  return check_launch("attn_kernel");
}

}  // namespace attn
}  // namespace ape
