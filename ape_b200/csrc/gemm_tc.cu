// gemm_tc.cu — C[M,N] = A[M,K] · W[N,K]^T (+bias, activation, residual) on the Hopper (sm_90a) tensor cores:
// TMA-staged 128-byte-swizzled operand tiles, wgmma issued by two consumer warpgroups with fp32 accumulators in
// registers, epilogue straight from the accumulator fragments.  Hand-written (no CUTLASS/cuBLAS).
//
// This is the dense workhorse behind the reference's nn.Linear calls on the detection path:
//   ViT q/k/v/proj and SwiGLU w1/w2/w3      ape/modeling/backbone/vit_eva_clip.py:225-232,266-267,125-132
//   encoder/decoder FFN and MSDA projections  ape/modeling/ape_deta/deformable_transformer_vl.py:36-54,
//                                              ape/layers/multi_scale_deform_attn.py:278-295,353
//   VisionLanguageAlign contraction            ape/layers/vision_language_align.py:36-48
// `W` is consumed in nn.Linear's own [out_features, in_features] layout: both operands are K-major.
//
// Kernel shape (persistent, warp-specialised, 288 threads, 1 CTA / SM):
//   warps 0-7  consumers : warpgroup g owns rows 64g..64g+63 of the 128 x BN tile: 4 x wgmma m64nBNk16 per k-block,
//                          one k-block in flight (the stage of the previous one is released when it has completed),
//                          then bias / activation / residual / rotary / LayerNorm fold in registers and direct stores
//   warp 8     producer  : STAGES-deep ring of {A 128x64, B BNx64} 16-bit tiles, mbarrier full/empty; it runs ahead
//                          into the next tile's k-blocks while the consumers finish the epilogue of the current one
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"
#include "tc.cuh"

namespace ape {
namespace {

constexpr int BM = 128, BK = 64, WG_K = 16;
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 32;

enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_SWIGLU = 3, ACT_CLAMP = 4 };

struct GemmParams {
  void *C;
  const float *bias;
  const void *residual;
  long long ldc, ldr;
  int M, N, K;
  int m_blocks, n_blocks, k_blocks;
  int out_dtype;  // APE_DTYPE_*
  int res_dtype;  // APE_DTYPE_* of `residual` (fp32-output GEMMs may add a 16-bit residual and vice versa)
  int act;
  int n_fastest;  // tile order: consecutive tiles walk the column blocks of one row group (A stays hot in L2)
  int vec_out;    // C rows allow paired (2-element) stores
  int vec_res;    // residual rows allow paired loads
  // optional 2-D rotary embedding on output columns [0, rope_cols) (q and k thirds of a fused qkv projection;
  // VisionRotaryEmbeddingFast, utils_eva02.py:248-252,346), applied after the bias in fp32: 64-channel heads
  const float *rope_cos, *rope_sin;  // [npos, 64]
  const int *rope_pos;               // [M] row -> position, or nullptr: row % rope_npos
  int rope_cols, rope_npos;
  // LayerNorm folded around the GEMM (sub-LN of the EVA-02 block, vit_eva_clip.py:266,130: inner_attn_ln before proj, ffn_ln
  // before w3).  The producer of A (attention / SwiGLU epilogue) leaves per-row partial (sum, sum of squares) of the 16-bit
  // values it wrote; this GEMM runs on the RAW A with weights pre-scaled by gamma and finishes
  //   LN(a) W^T = rstd * (a (gamma .* W)^T  -  mean * colsum)  +  (beta W^T + b)
  // in the epilogue: no LayerNorm launch and no extra trip of the activations through HBM.
  const float *ln_part;    // [M, ln_nparts, 2] partial (sum, sumsq) per row, fixed order (deterministic), or nullptr
  const float *ln_colsum;  // [N] sum_k of the 16-bit pre-scaled weight row
  int ln_nparts;
  float ln_inv_c, ln_eps;
  // SwiGLU epilogue: per-row (sum, sumsq) of every 64-column slab of the 16-bit output, [M, stats_nslab, 2]
  float *stats_out;
  int stats_nslab;
  // implicit-GEMM 3x3 convolution (stride 1, zero padding 1) over an NHWC image: an m block is a conv_tw x conv_th pixel
  // tile of one image, k block kb = (filter tap kb / conv_cblks, 64-channel block kb % conv_cblks); map_a is 4-D
  int conv;  // 0 = plain GEMM
  int conv_tw, conv_th, conv_tiles_x, conv_tiles_img, conv_cblks, conv_W, conv_H;
  // development aid (ape_gemm_set_trace): 8 clock64 stamps per CTA — 0 entry, 1 set-up done, 2 first operands landed,
  // 3 last MMA issued, 4 first accumulator complete, 5 last accumulator complete, 6 epilogue drained, 7 exit
  long long *trace;
};

__device__ __forceinline__ void trace_stamp(const GemmParams &p, int slot) {
  if (p.trace != nullptr) p.trace[(size_t)blockIdx.x * 8 + slot] = clock64();
}

template <int BN, int STAGES>
struct alignas(1024) GemmSmem {
  uint8_t a[STAGES][BM * BK * 2];
  uint8_t b[STAGES][BN * BK * 2];
  uint64_t full[STAGES], empty[STAGES];
};

__device__ __forceinline__ float act1(float v, int act) {
  if (act == ACT_RELU) return fmaxf(v, 0.f);
  if (act == ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  if (act == ACT_CLAMP) return fminf(fmaxf(v, -50000.f), 50000.f);  // vision_language_align.py:49-51
  return v;
}

__device__ __forceinline__ float ld16(const uint16_t *p, bool half) {
  const uint16_t u = __ldg(p);
  return half ? __half2float(__ushort_as_half(u)) : __uint_as_float((uint32_t)u << 16);
}

// Element offset of output row m: the row itself, or for the convolution the NHWC pixel the tile row stands for.
__device__ __forceinline__ size_t out_row_offset(const GemmParams &p, int m) {
  if (!p.conv) return (size_t)m * p.ldc;
  const int m_blk = m / BM, r = m - m_blk * BM;
  const int img = m_blk / p.conv_tiles_img, t = m_blk - img * p.conv_tiles_img;
  const int ty = t / p.conv_tiles_x, tx = t - ty * p.conv_tiles_x;
  const int x = tx * p.conv_tw + r % p.conv_tw, y = ty * p.conv_th + r / p.conv_tw;
  return (((size_t)img * p.conv_H + y) * p.conv_W + x) * p.ldc;
}

template <typename TO>
__device__ __forceinline__ void store_pair(TO *dst, float v0, float v1, bool ok1, bool vec) {
  if (vec && ok1) {
    if constexpr (sizeof(TO) == 4) {
      *reinterpret_cast<float2 *>(dst) = make_float2(v0, v1);
    } else if constexpr (std::is_same<TO, __half>::value) {
      *reinterpret_cast<__half2 *>(dst) = __floats2half2_rn(v0, v1);
    } else {
      *reinterpret_cast<__nv_bfloat162 *>(dst) = __floats2bfloat162_rn(v0, v1);
    }
  } else {
    dst[0] = Elem<TO>::from_f(v0);
    if (ok1) dst[1] = Elem<TO>::from_f(v1);
  }
}

// Epilogue of one warpgroup for its 64 rows x BN columns of tile (m_blk, n_blk), from the wgmma accumulator fragment:
// thread (warp w, lane l) holds rows r0 = 16 w + l/4 and r0 + 8, column pairs 8 j + 2 (l % 4) + {0, 1}.  Adjacent column
// pairs are exactly what SwiGLU (interleaved gate / up) and the rotary embedding (rotate_half pairs) combine.
template <typename TO, int BN>
__device__ __forceinline__ void epilogue(const GemmParams &p, const float *acc, int m_blk, int n_blk, int wg, int lane) {
  const int warp4 = (threadIdx.x >> 5) & 3, tq = lane & 3;
  const int c_base = n_blk * BN + 2 * tq;
  const bool swiglu = p.act == ACT_SWIGLU;
  TO *C = reinterpret_cast<TO *>(p.C);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m_blk * BM + wg * 64 + warp4 * 16 + (lane >> 2) + 8 * h;
    const bool row_ok = m < p.M;
    const int mr = row_ok ? m : p.M - 1;  // rows past M read a valid row and store nothing
    float ln_rstd = 1.f, ln_shift = 0.f;  // ln_shift = rstd * mean
    if (p.ln_part != nullptr) {  // row statistics from the producer's partials, summed in a fixed order
      const float2 *pp = reinterpret_cast<const float2 *>(p.ln_part) + (size_t)mr * p.ln_nparts;
      float sum = 0.f, sq = 0.f;
      for (int i = 0; i < p.ln_nparts; ++i) {
        const float2 t = __ldg(pp + i);
        sum += t.x;
        sq += t.y;
      }
      const float mean = sum * p.ln_inv_c;
      ln_rstd = rsqrtf(fmaxf(sq * p.ln_inv_c - mean * mean, 0.f) + p.ln_eps);
      ln_shift = ln_rstd * mean;
    }
    const float *rcos = nullptr, *rsin = nullptr;
    if (p.rope_cos != nullptr) {
      const int pos = p.rope_pos ? __ldg(p.rope_pos + mr) : mr % p.rope_npos;
      rcos = p.rope_cos + (size_t)pos * 64;
      rsin = p.rope_sin + (size_t)pos * 64;
    }
    TO *crow = C + out_row_offset(p, mr);
    float st_sum = 0.f, st_sq = 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = c_base + 8 * j;
      const bool ok0 = n < p.N, ok1 = n + 1 < p.N;
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (ok0) {
        if (p.ln_part != nullptr) {  // rstd * acc - rstd * mean * colsum; the bias below is beta W^T + b
          v0 = fmaf(ln_rstd, v0, -ln_shift * __ldg(p.ln_colsum + n));
          if (ok1) v1 = fmaf(ln_rstd, v1, -ln_shift * __ldg(p.ln_colsum + n + 1));
        }
        if (p.bias != nullptr) {
          v0 += __ldg(p.bias + n);
          if (ok1) v1 += __ldg(p.bias + n + 1);
        }
      }
      if (swiglu) {
        // interleaved (gate, up) column pair -> silu(gate) * up, output column n / 2 (vit_eva_clip.py:126-128); N is even
        const float o = v0 / (1.f + __expf(-v0)) * v1;
        const TO ot = Elem<TO>::from_f(o);
        if (ok0 && row_ok) crow[n / 2] = ot;
        if (p.stats_out != nullptr) {  // statistics of the values as stored (16-bit), columns beyond N/2 excluded
          const float f = ok0 ? Elem<TO>::to_f(ot) : 0.f;
          st_sum += f;
          st_sq = fmaf(f, f, st_sq);
          if ((j & 15) == 15) {  // 128 accumulator columns = one 64-column output slab complete
            st_sum += __shfl_xor_sync(0xffffffffu, st_sum, 1);
            st_sq += __shfl_xor_sync(0xffffffffu, st_sq, 1);
            st_sum += __shfl_xor_sync(0xffffffffu, st_sum, 2);
            st_sq += __shfl_xor_sync(0xffffffffu, st_sq, 2);
            const int slab_idx = (n_blk * BN + 8 * (j - 15)) / 128;
            if (tq == 0 && row_ok && slab_idx < p.stats_nslab)
              *reinterpret_cast<float2 *>(p.stats_out + ((size_t)m * p.stats_nslab + slab_idx) * 2) = make_float2(st_sum, st_sq);
            st_sum = 0.f;
            st_sq = 0.f;
          }
        }
        continue;
      }
      if (rcos != nullptr && n < p.rope_cols) {  // rotate_half pair (n, n+1) -> (-t[n+1], t[n])
        const float2 c = __ldg(reinterpret_cast<const float2 *>(rcos + (n & 63)));
        const float2 s = __ldg(reinterpret_cast<const float2 *>(rsin + (n & 63)));
        const float t0 = v0, t1 = v1;
        v0 = t0 * c.x - t1 * s.x;
        v1 = t1 * c.y + t0 * s.y;
      }
      v0 = act1(v0, p.act);
      v1 = act1(v1, p.act);
      if (p.residual != nullptr && ok0) {
        if (p.res_dtype == APE_DTYPE_F32) {
          const float *res = reinterpret_cast<const float *>(p.residual) + (size_t)mr * p.ldr + n;
          if (p.vec_res && ok1) {
            const float2 r2 = __ldg(reinterpret_cast<const float2 *>(res));
            v0 += r2.x;
            v1 += r2.y;
          } else {
            v0 += __ldg(res);
            if (ok1) v1 += __ldg(res + 1);
          }
        } else {
          const uint16_t *res = reinterpret_cast<const uint16_t *>(p.residual) + (size_t)mr * p.ldr + n;
          const bool half = p.res_dtype == APE_DTYPE_F16;
          v0 += ld16(res, half);
          if (ok1) v1 += ld16(res + 1, half);
        }
      }
      if (ok0 && row_ok) store_pair<TO>(crow + n, v0, v1, ok1, p.vec_out);
    }
  }
}

// CL = cluster size along M (1 or 2).  With CL == 2 the two CTAs of a cluster work on vertically adjacent 128-row tiles
// of the same BN-column block: each loads half of the B (weight) tile and TMA-multicasts it into both CTAs' shared
// memory, which halves the weight traffic from L2 per CTA.  A stage may only be refilled when the consumers of BOTH CTAs
// have finished reading it, so every consumer warp arrives on the "empty" barrier of both CTAs.
template <int BN, int STAGES, int CL, typename TI>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  if (threadIdx.x == 0) trace_stamp(p, 0);
  using Smem = GemmSmem<BN, STAGES>;
  Smem &s = *reinterpret_cast<Smem *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr uint32_t STAGE_BYTES = (BM + BN) * BK * 2;

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  // work items: (m group of CL row blocks, n block); CTA `rank` of the cluster takes row block CL*m_group + rank
  const int rank = CL > 1 ? (int)tc::cluster_ctarank() : 0;
  const int m_groups = (p.m_blocks + CL - 1) / CL;
  const int num_tiles = m_groups * p.n_blocks;
  const int first = blockIdx.x / CL, stride = gridDim.x / CL;
  // t-th tile of this CTA: tiles first, first + stride, ... of the (row group, column block) grid
  auto tile_at = [&](int t, int &m_blk, int &n_blk) -> bool {
    const int tile = first + t * stride;
    if (tile >= num_tiles) return false;
    const int mg = p.n_fastest ? tile / p.n_blocks : tile % m_groups;
    n_blk = p.n_fastest ? tile % p.n_blocks : tile / m_groups;
    m_blk = mg * CL + rank;
    return true;
  };

  if (warp == kConsumerWarps && lane == 0) {
    tc::prefetch_tensormap(&map_a);
    tc::prefetch_tensormap(&map_b);
#pragma unroll
    for (int i = 0; i < STAGES; ++i) {
      tc::mbar_init(&s.full[i], 1);
      tc::mbar_init(&s.empty[i], kConsumerWarps * CL);  // one arrival per consumer warp of each CTA of the cluster
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  if (CL > 1) tc::cluster_sync_all();  // peer barriers are initialised before any multicast / remote arrive can reach them
  pdl_wait();  // set-up done: operands / residual of the previous kernel may be read, C may be written from here on
  if (threadIdx.x == 0) trace_stamp(p, 1);

  if (warp == kConsumerWarps) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      uint32_t stage = 0, phase = 0;
      int m_blk, n_blk;
      for (int t = 0; tile_at(t, m_blk, n_blk); ++t) {
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          tc::mbar_wait(&s.empty[stage], phase ^ 1);
          tc::mbar_expect_tx(&s.full[stage], STAGE_BYTES);
          if (p.conv) {
            const int img = m_blk / p.conv_tiles_img, tt = m_blk - img * p.conv_tiles_img;
            const int ty = tt / p.conv_tiles_x, tx = tt - ty * p.conv_tiles_x;
            const int tap = kb / p.conv_cblks, cb = kb - tap * p.conv_cblks;
            tc::tma_load_4d(s.a[stage], &map_a, &s.full[stage], cb * BK, tx * p.conv_tw + tap % 3 - 1, ty * p.conv_th + tap / 3 - 1, img);
          } else {
            tc::tma_load_2d(s.a[stage], &map_a, &s.full[stage], kb * BK, m_blk * BM);
          }
          if (CL == 1) {
            tc::tma_load_2d(s.b[stage], &map_b, &s.full[stage], kb * BK, n_blk * BN);
          } else {
            constexpr int HALF_ROWS = BN / CL;
            tc::tma_load_2d_multicast(s.b[stage] + rank * HALF_ROWS * BK * 2, &map_b, &s.full[stage], kb * BK,
                                      n_blk * BN + rank * HALF_ROWS, (uint16_t)((1u << CL) - 1));
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers (two warpgroups) =====================
    const int wg = warp / 4;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    auto release = [&](uint32_t st) {  // the MMAs that read stage `st` have completed (in this warp's view of the group)
      if (lane == 0) {
        tc::mbar_arrive(&s.empty[st]);
        if (CL > 1) tc::mbar_arrive_cluster(tc::mapa_u32(&s.empty[st], (uint32_t)(rank ^ 1)));
      }
    };
    uint32_t stage = 0, phase = 0;
    int m_blk, n_blk;
    for (int t = 0; tile_at(t, m_blk, n_blk); ++t) {
      uint32_t prev = 0;
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        tc::mbar_wait(&s.full[stage], phase);
        if (kb == 0 && t == 0 && threadIdx.x == 0) trace_stamp(p, 2);
        const uint64_t da = tc::make_smem_desc_sw128(tc::smem_u32(s.a[stage] + wg * 64 * BK * 2));
        const uint64_t db = tc::make_smem_desc_sw128(tc::smem_u32(s.b[stage]));
        tc::fence_regs<BN / 2>(acc);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WG_K; ++k)  // advance 16 elements (32 B) along K inside the 128-byte swizzle row
          tc::Wgmma<BN, TI>::template ss<0>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        tc::wgmma_commit();
        tc::fence_regs<BN / 2>(acc);
        if (kb > 0) {
          tc::wgmma_wait<1>();
          release(prev);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::fence_regs<BN / 2>(acc);
      release(prev);
      if (threadIdx.x == 0) {
        trace_stamp(p, 3);
        if (t == 0) trace_stamp(p, 4);
        trace_stamp(p, 5);
      }
      if (p.out_dtype == APE_DTYPE_F32) epilogue<float, BN>(p, acc, m_blk, n_blk, wg, lane);
      else if (p.out_dtype == APE_DTYPE_F16) epilogue<__half, BN>(p, acc, m_blk, n_blk, wg, lane);
      else epilogue<__nv_bfloat16, BN>(p, acc, m_blk, n_blk, wg, lane);
    }
    if (threadIdx.x == 0) trace_stamp(p, 6);
  }
  __syncthreads();
  if (CL > 1) tc::cluster_sync_all();  // no CTA leaves while its peer can still signal its barriers
  if (threadIdx.x == 0) trace_stamp(p, 7);
}

// ---- host ----------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encoder() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void *ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// [rows, K] 16-bit row-major matrix with pitch `ld` elements; box = 64 (K) x box_rows, 128 B swizzle.
int make_map(CUtensorMap *map, const void *base, int dtype, long long rows, long long K, long long ld, int box_rows,
             int box_cols = BK) {
  EncodeTiledFn enc = get_encoder();
  if (!enc) return fail(APE_ERR_UNSUPPORTED, "gemm: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * (dtype == APE_DTYPE_F32 ? 4 : 2)};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, dtype == APE_DTYPE_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                        : dtype == APE_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                   const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(APE_ERR_INVALID_ARG, "gemm: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return APE_OK;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

template <int BN, int STAGES, int CL, typename TI>
int launch_gemm(const CUtensorMap &ma, const CUtensorMap &mb, GemmParams &p, cudaStream_t st) {
  using Smem = GemmSmem<BN, STAGES>;
  const size_t smem = sizeof(Smem) + 1024;
  auto k = gemm_tc_kernel<BN, STAGES, CL, TI>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "gemm: cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
    attr_set = true;
  }
  p.n_blocks = (p.N + BN - 1) / BN;
  p.n_fastest = p.n_blocks <= 8;  // few column blocks: keep the A rows of a group hot instead of re-reading A per column block
  const int groups = (p.m_blocks + CL - 1) / CL * p.n_blocks;
  const int max_clusters = num_sms() / CL;
  const int clusters = groups < max_clusters ? groups : max_clusters;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(clusters * CL));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  cudaError_t e = cudaLaunchKernelEx(&cfg, k, ma, mb, p);
  if (e != cudaSuccess) return fail((int)e, "gemm_tc_kernel launch: %s", cudaGetErrorString(e));
  return check_launch("gemm_tc_kernel");
}

// 4 stages of 48 KB (BN = 256) or 6 of 32 KB (BN = 128): 192 KB of the 227 KB a block may use.
template <int CL, typename TI>
int launch_bn(int bn, const CUtensorMap &ma, const CUtensorMap &mb, GemmParams &p, cudaStream_t st) {
  if (bn == 256) return launch_gemm<256, 4, CL, TI>(ma, mb, p, st);
  return launch_gemm<128, 6, CL, TI>(ma, mb, p, st);
}

int launch_any(int bn, bool cluster, int in_dtype, const CUtensorMap &ma, const CUtensorMap &mb, GemmParams &p, cudaStream_t st) {
  if (in_dtype == APE_DTYPE_BF16)
    return cluster ? launch_bn<2, __nv_bfloat16>(bn, ma, mb, p, st) : launch_bn<1, __nv_bfloat16>(bn, ma, mb, p, st);
  return cluster ? launch_bn<2, __half>(bn, ma, mb, p, st) : launch_bn<1, __half>(bn, ma, mb, p, st);
}

}  // namespace
}  // namespace ape

using namespace ape;

struct RopeArgs {
  const float *cos, *sin;
  const int *pos;
  int cols, npos;
};

struct FuseArgs {  // LayerNorm fold (consume) / SwiGLU row statistics (produce); see GemmParams
  const float *ln_part, *ln_colsum;
  int ln_nparts;
  float ln_inv_c, ln_eps;
  float *stats_out;
  int stats_nslab;
};

static long long *g_gemm_trace = nullptr;

// Development aid: device buffer of 8 * grid long long receiving clock64 stamps of the next single-CTA / multicast GEMM
// launches (see GemmParams::trace); nullptr switches it off.  Not for concurrent use.
extern "C" void ape_gemm_set_trace(long long *device_buffer) { g_gemm_trace = device_buffer; }

static int gemm_impl(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc,
                     const float *bias, const void *residual, int64_t ldr, int res_dtype, int M, int N, int K, int in_dtype,
                     int out_dtype, int act, int tile_n, const RopeArgs *rope, void *stream, const FuseArgs *fuse = nullptr) {
  if (residual && res_dtype != APE_DTYPE_F32 && res_dtype != APE_DTYPE_F16 && res_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "gemm: bad res_dtype %d", res_dtype);
  if (in_dtype != APE_DTYPE_F16 && in_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "gemm: operands must be fp16 or bf16 (got dtype %d)", in_dtype);
  if (out_dtype != APE_DTYPE_F32 && out_dtype != APE_DTYPE_F16 && out_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "gemm: bad out_dtype %d", out_dtype);
  if (act < 0 || act > ACT_CLAMP) return fail(APE_ERR_INVALID_ARG, "gemm: bad activation %d", act);
  if (M < 0 || N <= 0 || K <= 0) return fail(APE_ERR_INVALID_ARG, "gemm: bad sizes M=%d N=%d K=%d", M, N, K);
  if (M == 0) return APE_OK;
  if (!A || !W || !C) return fail(APE_ERR_NULL_PTR, "gemm: null pointer argument");
  if ((lda * 2) % 16 || (ldw * 2) % 16 || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15))
    return fail(APE_ERR_INVALID_ARG, "gemm: A/W base and row pitch must be 16-byte aligned (TMA)");
  if (lda < K || ldw < K) return fail(APE_ERR_INVALID_ARG, "gemm: row pitch smaller than K");
  if (act == ACT_SWIGLU && ((N & 1) || residual)) return fail(APE_ERR_INVALID_ARG, "gemm: swiglu needs even N, no residual");
  // default tile width 128: a 128 x 256 tile holds 128 fp32 accumulators per consumer thread, more than the 168 registers a
  // thread of this 288-thread block may use leave room for next to the epilogue (it spills); 256 stays selectable
  const int bn = (tile_n & 0xfff) > 0 ? (tile_n & 0xfff) : 128;
  if (bn != 128 && bn != 256) return fail(APE_ERR_INVALID_ARG, "gemm: tile_n must be 128 or 256");
  if (tile_n & 0x2000) return fail(APE_ERR_UNSUPPORTED, "gemm: tile_n flag 0x2000 (CTA-pair MMA) is not available on sm_90a");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // kernel variant: single CTA, or a cluster of 2 along M sharing the weight tile by TMA multicast.  The cluster pays off
  // when the K loop is long (K >= 2048: w3, FFN2, the 3x3 convolutions), where the weight tile is the larger share of the
  // operand traffic; bit 0x1000 forces the single CTA, bit 0x4000 the cluster.
  const int m_blocks = (M + BM - 1) / BM;
  const bool cluster = m_blocks >= 2 && (tile_n & 0x1000) == 0 && ((tile_n & 0x4000) != 0 || K >= 2048);
  CUtensorMap ma, mb;
  if (int rc = make_map(&ma, A, in_dtype, M, K, lda, BM)) return rc;
  if (int rc = make_map(&mb, W, in_dtype, N, K, ldw, cluster ? bn / 2 : bn)) return rc;
  GemmParams p{};
  p.C = C; p.bias = bias; p.residual = residual; p.ldc = ldc; p.ldr = ldr;
  p.M = M; p.N = N; p.K = K;
  p.m_blocks = m_blocks;
  p.k_blocks = (K + BK - 1) / BK;
  p.out_dtype = out_dtype; p.act = act; p.res_dtype = res_dtype;
  p.trace = g_gemm_trace;
  const int oe = out_dtype == APE_DTYPE_F32 ? 4 : 2;
  p.vec_out = (ldc % 2) == 0 && (reinterpret_cast<uintptr_t>(C) % (2 * oe)) == 0;
  p.vec_res = residual != nullptr && (ldr % 2) == 0 && (reinterpret_cast<uintptr_t>(residual) % 8) == 0;
  const int n_out = act == ACT_SWIGLU ? N / 2 : N;
  if (fuse) {
    if (fuse->ln_part) {
      if (out_dtype != APE_DTYPE_F32 || !fuse->ln_colsum || fuse->ln_nparts <= 0 || act == ACT_SWIGLU)
        return fail(APE_ERR_INVALID_ARG, "gemm+ln: needs an fp32 output, column sums and partial statistics");
      p.ln_part = fuse->ln_part; p.ln_colsum = fuse->ln_colsum; p.ln_nparts = fuse->ln_nparts;
      p.ln_inv_c = fuse->ln_inv_c; p.ln_eps = fuse->ln_eps;
    }
    if (fuse->stats_out) {
      if (oe != 2 || act != ACT_SWIGLU || fuse->stats_nslab != (n_out + 63) / 64)
        return fail(APE_ERR_INVALID_ARG, "gemm+stats: needs the SwiGLU epilogue with a 16-bit output and stats_nslab = ceil(N/2/64)");
      p.stats_out = fuse->stats_out; p.stats_nslab = fuse->stats_nslab;
    }
  }
  if (rope) {
    if (oe != 2 || act != ACT_NONE || rope->cols % 64 != 0 || rope->cols > N || rope->npos <= 0 || !rope->cos || !rope->sin)
      return fail(APE_ERR_INVALID_ARG, "gemm+rope: needs a 16-bit output, no activation, rope_cols a multiple of 64 <= N");
    p.rope_cos = rope->cos; p.rope_sin = rope->sin; p.rope_pos = rope->pos; p.rope_cols = rope->cols; p.rope_npos = rope->npos;
  }
  return launch_any(bn, cluster, in_dtype, ma, mb, p, st);
}

extern "C" int ape_gemm_tn(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc,
                           const float *bias, const void *residual, int64_t ldr, int M, int N, int K, int in_dtype,
                           int out_dtype, int act, int tile_n, void *stream) {
  return gemm_impl(A, lda, W, ldw, C, ldc, bias, residual, ldr, out_dtype, M, N, K, in_dtype, out_dtype, act, tile_n, nullptr,
                   stream);
}

extern "C" int ape_gemm_tn_ex(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc,
                              const float *bias, const void *residual, int64_t ldr, int res_dtype, int M, int N, int K,
                              int in_dtype, int out_dtype, int act, int tile_n, void *stream) {
  return gemm_impl(A, lda, W, ldw, C, ldc, bias, residual, ldr, res_dtype, M, N, K, in_dtype, out_dtype, act, tile_n, nullptr,
                   stream);
}

extern "C" int ape_gemm_tn_fused(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc, const float *bias,
                                 const void *residual, int64_t ldr, int res_dtype, int M, int N, int K, int in_dtype, int out_dtype,
                                 int act, int tile_n, const float *ln_part, int ln_nparts, const float *ln_colsum, float ln_inv_c,
                                 float ln_eps, float *stats_out, int stats_nslab, void *stream) {
  FuseArgs f{ln_part, ln_colsum, ln_nparts, ln_inv_c, ln_eps, stats_out, stats_nslab};
  return gemm_impl(A, lda, W, ldw, C, ldc, bias, residual, ldr, res_dtype, M, N, K, in_dtype, out_dtype, act, tile_n, nullptr,
                   stream, &f);
}

// 4-D tensor map over an NHWC image [B, H, W, C] (16-bit): box = 64 channels x bw x bh pixels of one image, 128 B swizzle.
static int make_map_nhwc(CUtensorMap *map, const void *base, int dtype, int B, int H, int W, int C, int bw, int bh) {
  EncodeTiledFn enc = get_encoder();
  if (!enc) return fail(APE_ERR_UNSUPPORTED, "conv: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)bh, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, dtype == APE_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                   const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(APE_ERR_INVALID_ARG, "conv: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return APE_OK;
}

// 3x3 convolution, stride 1, zero padding 1, no dilation / groups, over NHWC activations as an implicit GEMM on the wgmma
// kernel: M = B*H*W output pixels, N = Cout, K = 9*Cin walked as (filter tap, 64-channel block).  The A tile of tap
// (dy, dx) is the 128-pixel tile shifted by (dy-1, dx-1): one 4-D TMA box, out-of-image parts arrive as zeros.
extern "C" int ape_conv3x3_nhwc(const void *x, const void *w, void *y, const float *bias, int B, int H, int W, int Cin, int Cout,
                                int dtype, int act, void *stream) {
  if (dtype != APE_DTYPE_F16 && dtype != APE_DTYPE_BF16) return fail(APE_ERR_INVALID_ARG, "conv3x3: fp16 / bf16 only");
  if (B <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return fail(APE_ERR_INVALID_ARG, "conv3x3: bad sizes");
  if (Cin % 64 || Cout % 8) return fail(APE_ERR_UNSUPPORTED, "conv3x3: Cin must be a multiple of 64 and Cout of 8 (got %d, %d)", Cin, Cout);
  if (act != ACT_NONE && act != ACT_RELU && act != ACT_GELU) return fail(APE_ERR_INVALID_ARG, "conv3x3: activation %d", act);
  int tw = 128;
  while (tw > 8 && W % tw) tw >>= 1;
  const int th = 128 / tw;
  if (W % tw || H % th) return fail(APE_ERR_UNSUPPORTED, "conv3x3: %dx%d image is not a whole number of %dx%d pixel tiles", H, W, th, tw);
  if (!x || !w || !y) return fail(APE_ERR_NULL_PTR, "conv3x3: null pointer argument");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(y)) & 15)
    return fail(APE_ERR_INVALID_ARG, "conv3x3: tensors must be 16-byte aligned");
  const int K = 9 * Cin, M = B * H * W, N = Cout;
  const int bn = 128;
  const int m_blocks = M / BM;
  const bool cluster = m_blocks >= 2 && m_blocks % 2 == 0;  // K = 9 * Cin is a long loop: share the weight tile (see gemm_impl)
  CUtensorMap ma, mb;
  if (int rc = make_map_nhwc(&ma, x, dtype, B, H, W, Cin, tw, th)) return rc;
  if (int rc = make_map(&mb, w, dtype, N, K, K, cluster ? bn / 2 : bn)) return rc;
  GemmParams p{};
  p.C = y; p.bias = bias; p.ldc = N; p.M = M; p.N = N; p.K = K;
  p.m_blocks = m_blocks;
  p.k_blocks = K / BK;
  p.out_dtype = dtype; p.res_dtype = dtype; p.act = act;
  p.vec_out = 1;
  p.conv = 1; p.conv_tw = tw; p.conv_th = th; p.conv_tiles_x = W / tw; p.conv_tiles_img = (W / tw) * (H / th); p.conv_cblks = Cin / 64;
  p.conv_W = W; p.conv_H = H;
  return launch_any(bn, cluster, dtype, ma, mb, p, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ape_gemm_tn_rope(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc,
                                const float *bias, int M, int N, int K, int in_dtype, int out_dtype, const float *cos_table,
                                const float *sin_table, const int *pos_map, int npos, int head_dim, int rope_cols,
                                int tile_n, void *stream) {
  if (head_dim != 64) return fail(APE_ERR_UNSUPPORTED, "gemm+rope: head_dim %d (only 64)", head_dim);
  if ((reinterpret_cast<uintptr_t>(cos_table) | reinterpret_cast<uintptr_t>(sin_table)) & 15)
    return fail(APE_ERR_INVALID_ARG, "gemm+rope: cos / sin tables must be 16-byte aligned");
  RopeArgs r{cos_table, sin_table, pos_map, rope_cols, npos};
  return gemm_impl(A, lda, W, ldw, C, ldc, bias, nullptr, 0, out_dtype, M, N, K, in_dtype, out_dtype, ACT_NONE, tile_n, &r, stream);
}
