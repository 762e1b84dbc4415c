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
// Kernel shape (persistent, warp-specialised, 384 threads, 1 CTA / SM):
//   warps 0-7   consumers : warpgroup g owns rows 64g..64g+63 of the 128 x BN tile: 4 x wgmma m64nBNk16 per k-block,
//                           one k-block in flight (the stage of the previous one is released when it has completed),
//                           then bias / activation / residual / rotary / LayerNorm fold in registers and direct stores
//   warps 8-11  producer  : one thread keeps a STAGES-deep ring of {A 128x64, B BNx64} 16-bit tiles filled by TMA
//                           (mbarrier full/empty); it runs ahead into the next tile's k-blocks while the consumers finish
//                           the epilogue of the current one.  The warpgroup gives its registers to the consumers
//                           (setmaxnreg 40 / 232), so BN = 256 holds its 128 accumulators per thread without spilling.
// gemm_pp_kernel is the ping-pong form of the same kernel for single-CTA BN = 128 GEMMs with many tiles: each consumer
// warpgroup owns whole tiles, and their main loops alternate so that one's epilogue runs under the other's MMAs.
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"
#include "tc.cuh"

namespace ape {
namespace {

constexpr int BM = 128, BK = 64, WG_K = 16;
constexpr int kConsumerWarps = 8;
// gemm_tc_kernel and gemm_pp_kernel: two consumer warpgroups and a producer warpgroup (setmaxnreg works per warpgroup)
constexpr int kThreads = 32 * kConsumerWarps + 128;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;  // 40 x 128 + 232 x 256 <= the 168 x 384 registers of the launch

enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_SWIGLU = 3, ACT_CLAMP = 4 };
enum Res { RES_NONE = 0, RES_F32 = 1, RES_16 = 2 };  // RES_16: a residual of the operand type

// The epilogue of a kernel instantiation, fixed at compile time: output fp32 (or the 16-bit operand type), activation,
// residual, LayerNorm fold, rotary embedding, SwiGLU row statistics.  A runtime-generic epilogue tests every feature for
// each of the 64 accumulator values of a thread; it compiled to ~29 k SASS instructions per kernel, more than the
// instruction caches hold, and its issue time exceeded the main loop of the short-K GEMMs.  Bias is a uniform runtime test.
template <bool OUT32, int ACT, int RES, bool LN = false, bool ROPE = false, bool STATS = false>
struct Epi {
  static constexpr bool out32 = OUT32, ln = LN, rope = ROPE, stats = STATS;
  static constexpr int act = ACT, res = RES;
};

struct GemmParams {
  void *C;
  const float *bias;
  const void *residual;
  long long ldc, ldr;
  int M, N, K;
  int m_blocks, n_blocks, k_blocks;
  int band;     // tile order: row groups per raster band (see tile_at)
  int vec_out;  // C rows allow paired (2-element) stores
  int fast;     // C, residual, bias and column sums allow paired accesses: tiles inside M x N take the unguarded epilogue
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
  // class-argmax epilogue (EpiArgmax): C is the u64 key per row; output column n stands for class n + argmax_col_base
  int argmax_col_base;
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

template <int ACT>
__device__ __forceinline__ float act1(float v) {
  if constexpr (ACT == ACT_RELU) return fmaxf(v, 0.f);
  if constexpr (ACT == ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  if constexpr (ACT == ACT_CLAMP) return fminf(fmaxf(v, -50000.f), 50000.f);  // vision_language_align.py:49-51
  return v;
}

// (p[n], p[n + 1]) of an fp32 vector: one 8-byte load when VEC (n even, base 8-byte aligned), else p[n + 1] only if ok1
template <bool VEC>
__device__ __forceinline__ float2 ld_pair(const float *p, int n, bool ok1) {
  if constexpr (VEC) return __ldg(reinterpret_cast<const float2 *>(p + n));
  return make_float2(__ldg(p + n), ok1 ? __ldg(p + n + 1) : 0.f);
}
template <bool VEC, typename T>
__device__ __forceinline__ float2 ld_res_pair(const T *p, bool ok1) {
  if constexpr (VEC) return Elem<T>::load2(p);
  return make_float2(Elem<T>::load1(p), ok1 ? Elem<T>::load1(p + 1) : 0.f);
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
// FULL: the tile lies inside M x N and p.fast holds, so no row or column test and paired loads throughout; edge tiles
// (and outputs / residuals / vectors without 8-byte pairs) take the guarded instantiation.
template <class E, typename TI, int BN, bool FULL>
__device__ __forceinline__ void epilogue(const GemmParams &p, const float *acc, int m_blk, int n_blk, int wg, int lane) {
  using TO = std::conditional_t<E::out32, float, TI>;
  constexpr bool swiglu = E::act == ACT_SWIGLU;
  const int warp4 = (threadIdx.x >> 5) & 3, tq = lane & 3;
  const int c_base = n_blk * BN + 2 * tq;
  TO *C = reinterpret_cast<TO *>(p.C);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m_blk * BM + wg * 64 + warp4 * 16 + (lane >> 2) + 8 * h;
    const bool row_ok = FULL || m < p.M;
    const int mr = row_ok ? m : p.M - 1;  // rows past M read a valid row and store nothing
    float ln_rstd = 1.f, ln_shift = 0.f;  // ln_shift = rstd * mean
    if constexpr (E::ln) {  // row statistics from the producer's partials, summed in a fixed order
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
    int rope_row = 0;  // first table element of the row's position (an offset, not two pointers: it keeps BN = 128 spill-free)
    if constexpr (E::rope) rope_row = (p.rope_pos ? __ldg(p.rope_pos + mr) : mr % p.rope_npos) * 64;
    TO *crow = C + out_row_offset(p, mr);
    const float *res32 = reinterpret_cast<const float *>(p.residual) + (size_t)mr * p.ldr;
    const TI *res16 = reinterpret_cast<const TI *>(p.residual) + (size_t)mr * p.ldr;
    float st_sum = 0.f, st_sq = 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = c_base + 8 * j;
      const bool ok0 = FULL || n < p.N, ok1 = FULL || n + 1 < p.N;
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (ok0) {
        if constexpr (E::ln) {  // rstd * acc - rstd * mean * colsum; the bias below is beta W^T + b
          const float2 cs = ld_pair<FULL>(p.ln_colsum, n, ok1);
          v0 = fmaf(ln_rstd, v0, -ln_shift * cs.x);
          if (ok1) v1 = fmaf(ln_rstd, v1, -ln_shift * cs.y);
        }
        if (p.bias != nullptr) {  // with the LN fold, paired bias loads cost the cluster kernel 8 bytes of spill
          const float2 b = ld_pair<FULL && !E::ln>(p.bias, n, ok1);
          v0 += b.x;
          if (ok1) v1 += b.y;
        }
      }
      if constexpr (swiglu) {
        // interleaved (gate, up) column pair -> silu(gate) * up, output column n / 2 (vit_eva_clip.py:126-128); N is even
        const float o = v0 / (1.f + __expf(-v0)) * v1;
        const TO ot = Elem<TO>::from_f(o);
        if (ok0 && row_ok) crow[n / 2] = ot;
        if constexpr (E::stats) {  // statistics of the values as stored (16-bit), columns beyond N/2 excluded
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
      } else {
        if constexpr (E::rope) {
          if (n < p.rope_cols) {  // rotate_half pair (n, n+1) -> (-t[n+1], t[n])
            const float2 c = __ldg(reinterpret_cast<const float2 *>(p.rope_cos + rope_row + (n & 63)));
            const float2 s = __ldg(reinterpret_cast<const float2 *>(p.rope_sin + rope_row + (n & 63)));
            const float t0 = v0, t1 = v1;
            v0 = t0 * c.x - t1 * s.x;
            v1 = t1 * c.y + t0 * s.y;
          }
        }
        v0 = act1<E::act>(v0);
        v1 = act1<E::act>(v1);
        if constexpr (E::res != RES_NONE) {
          if (ok0) {
            const float2 r = E::res == RES_F32 ? ld_res_pair<FULL>(res32 + n, ok1) : ld_res_pair<FULL>(res16 + n, ok1);
            v0 += r.x;
            if (ok1) v1 += r.y;
          }
        }
        if (ok0 && row_ok) store_pair<TO>(crow + n, v0, v1, ok1, FULL || p.vec_out);
      }
    }
  }
}

// Class-argmax epilogue of the semantic label maps (semseg.cu): rows are pixels, columns classes, and nothing is stored but
// the running maximum of each row.  A thread takes the first maximum over its 2 x BN/8 columns of a row, the quad (the four
// threads that share the row) combines by shuffles, and one 64-bit atomicMax per (row, tile) merges it into the u64 key of
// the row (argmax_key: larger value first, then lower class, so the key is torch.argmax over all column tiles).
struct EpiArgmax {
  static constexpr bool out32 = true, ln = false, rope = false, stats = false;
  static constexpr int act = ACT_NONE, res = RES_NONE;
};
// The same epilogue for a map whose size is on the device (ape_gemm_tn_argmax_dev): M is the capacity, and `residual`, which no
// argmax epilogue reads, points at the number of rows in use (device int32), so GemmParams and the other kernels stay as they were
struct EpiArgmaxDev : EpiArgmax {};
template <class E>
constexpr bool kArgmax = std::is_same<E, EpiArgmax>::value || std::is_same<E, EpiArgmaxDev>::value;
template <class E>
constexpr bool kDevRows = std::is_same<E, EpiArgmaxDev>::value;

// row blocks that hold rows of A: all of them, or (kDevRows) those below the device count at p.residual.  Read after pdl_wait(): a kernel before this
// one writes the count.
template <class E>
__device__ __forceinline__ int live_m_blocks(const GemmParams &p) {
  if constexpr (kDevRows<E>) return (min(max(*static_cast<const int *>(p.residual), 0), p.M) + BM - 1) / BM;
  return p.m_blocks;
}

template <int BN>
__device__ __forceinline__ void argmax_epilogue(const GemmParams &p, const float *acc, int m_blk, int n_blk, int wg, int lane) {
  const int warp4 = (threadIdx.x >> 5) & 3, tq = lane & 3;
  const int c_base = n_blk * BN + 2 * tq;
  unsigned long long *keys = reinterpret_cast<unsigned long long *>(p.C);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m_blk * BM + wg * 64 + warp4 * 16 + (lane >> 2) + 8 * h;
    float best = -INFINITY;
    int col = -1;  // -1: no column of this thread lies inside N
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {  // columns in increasing order, strict >: the first maximum
      const int n = c_base + 8 * j;
      const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (n < p.N && (col < 0 || v0 > best)) { best = v0; col = n; }
      if (n + 1 < p.N && v1 > best) { best = v1; col = n + 1; }
    }
#pragma unroll
    for (int s = 1; s <= 2; s <<= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, s);
      const int oc = __shfl_xor_sync(0xffffffffu, col, s);
      if (oc >= 0 && (col < 0 || ob > best || (ob == best && oc < col))) { best = ob; col = oc; }
    }
    if (tq == 0 && col >= 0 && m < p.M) atomicMax(keys + m, argmax_key(best, col + p.argmax_col_base));
  }
}

// CL = cluster size along M (1 or 2).  With CL == 2 the two CTAs of a cluster work on vertically adjacent 128-row tiles
// of the same BN-column block: each loads half of the B (weight) tile and TMA-multicasts it into both CTAs' shared
// memory, which halves the weight traffic from L2 per CTA.  A stage may only be refilled when the consumers of BOTH CTAs
// have finished reading it, so every consumer warp arrives on the "empty" barrier of both CTAs.
template <int BN, int STAGES, int CL, typename TI, class E>
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
  int m_groups = (p.m_blocks + CL - 1) / CL;
  int num_tiles = m_groups * p.n_blocks;
  const int first = blockIdx.x / CL, stride = gridDim.x / CL;
  // t-th tile of this CTA: tiles first, first + stride, ... of the (row group, column block) grid, walked in bands of
  // p.band row groups; inside a band the row group changes fastest.  The tiles resident at one time then cover a few row
  // groups across all column blocks, so each A row block is read from HBM once, not once per column block.
  auto tile_at = [&](int t, int &m_blk, int &n_blk) -> bool {
    const int tile = first + t * stride;
    if (tile >= num_tiles) return false;
    const int per_band = p.band * p.n_blocks;
    const int band = tile / per_band, r = tile - band * per_band;
    const int rows = min(p.band, m_groups - band * p.band);
    n_blk = r / rows;
    m_blk = (band * p.band + r - n_blk * rows) * CL + rank;
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
  if constexpr (kDevRows<E>) {
    m_groups = (live_m_blocks<E>(p) + CL - 1) / CL;
    num_tiles = m_groups * p.n_blocks;
  }

  if (warp >= kConsumerWarps) {
    // ===================== TMA producer (one thread of the producer warpgroup) =====================
    tc::setmaxnreg_dec<kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0) {
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
    tc::setmaxnreg_inc<kConsumerRegs>();  // BN = 256: 128 accumulators
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
      if constexpr (kArgmax<E>) {
        argmax_epilogue<BN>(p, acc, m_blk, n_blk, wg, lane);
      } else {
        // BN = 256 as two 128-column halves, one after the other (as gemm_pp_kernel does with its row halves): a single
        // epilogue over all 128 accumulators hoists the bias and residual loads of every column ahead of the stores and
        // spills.  Accumulators 64 h .. 64 h + 63 are columns 128 h .. 128 h + 127 of the tile.
#pragma unroll
        for (int h = 0; h < BN / 128; ++h) {
          const int nb = n_blk * (BN / 128) + h;
          if (!E::rope && p.fast && (m_blk + 1) * BM <= p.M && (nb + 1) * 128 <= p.N) epilogue<E, TI, 128, true>(p, acc + 64 * h, m_blk, nb, wg, lane);
          else epilogue<E, TI, 128, false>(p, acc + 64 * h, m_blk, nb, wg, lane);
        }
      }
    }
    if (threadIdx.x == 0) trace_stamp(p, 6);
  }
  __syncthreads();
  if (CL > 1) tc::cluster_sync_all();  // no CTA leaves while its peer can still signal its barriers
  if (threadIdx.x == 0) trace_stamp(p, 7);
}

// Ping-pong variant (single CTA, BN = 128, 384 threads): the same operand ring and the same epilogues, but each consumer
// warpgroup owns whole 128 x 128 tiles — warpgroup g takes the CTA's tiles t with t % 2 == g — so one warpgroup's epilogue
// runs while the other's MMAs keep the tensor cores busy.
//   warps 0-7   consumers : warpgroup g, 128 accumulators per thread (two m64n128 halves: tile rows 0-63 and 64-127)
//   warps 8-11  producer  : one thread issues TMA; the warpgroup gives its registers to the consumers (setmaxnreg works
//                           per warpgroup, hence a whole warpgroup)
// Synchronisation rules:
//  1. mbar_wait(bar, parity) passes as soon as the barrier is not in phase `parity`, so a wait for a phase one ahead of
//     the barrier's current one passes on a stage TMA has not written.  Each warpgroup skips the other's k-blocks (K = 256
//     with 6 stages: warpgroup 1's first tile uses stages 4, 5, 0, 1), so (stage, phase) come from the CTA's running
//     k-block index t * k_blocks + kb, never from a counter per warpgroup, and the order handoff (rule 2) makes a
//     warpgroup wait on the full barriers of tile t only after the other has passed its waits of tile t - 1: every
//     earlier fill of the stage has then landed, and the next one needs this warpgroup's release.
//  2. Order handoff on named barriers kOrderBar + g (256 threads: one warpgroup waits with bar.sync, the other arrives):
//     warpgroup g starts the main loop of tile t only after the other warpgroup has issued the last MMA of tile t - 1.
//     Every arrive (after tile t, if tile t + 1 exists) is matched by the sync before tile t + 1.
//  3. empty[i] counts 4 arrivals, one per warp of the single warpgroup that reads the stage.
//  4. The epilogue takes warp4 from threadIdx.x (consumers keep warps 0-7) and the row half from its `wg` argument.
//     trace_stamp slots keep their meaning; thread 0 belongs to warpgroup 0.
//  5. PDL as in gemm_tc_kernel: launch_dependents at entry, griddepcontrol.wait before the first TMA load and store.
constexpr int kOrderBar = 1;  // named barriers 1 and 2

template <typename TI, class E>
__global__ void __launch_bounds__(kThreads, 1)
gemm_pp_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GemmParams p) {
  constexpr int BN = 128, STAGES = 6;
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  if (threadIdx.x == 0) trace_stamp(p, 0);
  using Smem = GemmSmem<BN, STAGES>;
  Smem &s = *reinterpret_cast<Smem *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr uint32_t STAGE_BYTES = (BM + BN) * BK * 2;

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  // the tile order of gemm_tc_kernel with CL = 1 (grouped raster in bands of p.band row blocks, row block fastest)
  const int num_tiles = p.m_blocks * p.n_blocks;
  auto tile_at = [&](int t, int &m_blk, int &n_blk) -> bool {
    const int tile = blockIdx.x + t * gridDim.x;
    if (tile >= num_tiles) return false;
    const int per_band = p.band * p.n_blocks;
    const int band = tile / per_band, r = tile - band * per_band;
    const int rows = min(p.band, p.m_blocks - band * p.band);
    n_blk = r / rows;
    m_blk = band * p.band + r - n_blk * rows;
    return true;
  };

  if (warp == kConsumerWarps && lane == 0) {
    tc::prefetch_tensormap(&map_a);
    tc::prefetch_tensormap(&map_b);
#pragma unroll
    for (int i = 0; i < STAGES; ++i) {
      tc::mbar_init(&s.full[i], 1);
      tc::mbar_init(&s.empty[i], 4);  // rule 3
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (threadIdx.x == 0) trace_stamp(p, 1);

  if (warp >= kConsumerWarps) {
    // ===================== TMA producer: every tile of the CTA in order, one ring =====================
    tc::setmaxnreg_dec<kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0) {
      uint32_t stage = 0, phase = 0;
      int m_blk, n_blk;
      for (int t = 0; tile_at(t, m_blk, n_blk); ++t) {
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          tc::mbar_wait(&s.empty[stage], phase ^ 1);
          tc::mbar_expect_tx(&s.full[stage], STAGE_BYTES);
          tc::tma_load_2d(s.a[stage], &map_a, &s.full[stage], kb * BK, m_blk * BM);
          tc::tma_load_2d(s.b[stage], &map_b, &s.full[stage], kb * BK, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers: warpgroup wg, tiles wg, wg + 2, ... =====================
    tc::setmaxnreg_inc<kConsumerRegs>();  // 128 accumulators
    const int wg = warp / 4;
    float acc[BN];  // acc[0, 64): tile rows 0-63, acc[64, 128): rows 64-127
#pragma unroll
    for (int i = 0; i < BN; ++i) acc[i] = 0.f;
    auto release = [&](uint32_t st) {  // the MMAs that read stage `st` have completed (in this warp's view of the group)
      if (lane == 0) tc::mbar_arrive(&s.empty[st]);
    };
    int m_blk, n_blk;
    for (int t = wg; tile_at(t, m_blk, n_blk); t += 2) {
      if (t > 0) tc::named_bar_sync(kOrderBar + wg, 256);  // rule 2: the other warpgroup issued tile t - 1
      const uint32_t g0 = (uint32_t)t * p.k_blocks;       // rule 1: the CTA's running k-block index
      uint32_t stage = g0 % STAGES, phase = (g0 / STAGES) & 1, prev = 0;
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        tc::mbar_wait(&s.full[stage], phase);
        if (kb == 0 && t == 0 && threadIdx.x == 0) trace_stamp(p, 2);
        const uint64_t da = tc::make_smem_desc_sw128(tc::smem_u32(s.a[stage]));
        const uint64_t da_hi = tc::make_smem_desc_sw128(tc::smem_u32(s.a[stage] + 64 * BK * 2));
        const uint64_t db = tc::make_smem_desc_sw128(tc::smem_u32(s.b[stage]));
        tc::fence_regs<BN>(acc);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WG_K; ++k) {
          tc::Wgmma<BN, TI>::template ss<0>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
          tc::Wgmma<BN, TI>::template ss<0>(acc + 64, da_hi + 2 * k, db + 2 * k, (kb | k) != 0);
        }
        tc::wgmma_commit();
        tc::fence_regs<BN>(acc);
        if (kb > 0) {
          tc::wgmma_wait<1>();
          release(prev);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      int m_nx, n_nx;
      if (tile_at(t + 1, m_nx, n_nx)) tc::named_bar_arrive(kOrderBar + (wg ^ 1), 256);  // rule 2: hand over
      tc::wgmma_wait<0>();
      tc::fence_regs<BN>(acc);
      release(prev);
      if (threadIdx.x == 0) {
        trace_stamp(p, 3);
        if (t == 0) trace_stamp(p, 4);
        trace_stamp(p, 5);
      }
      if constexpr (kArgmax<E>) {
        argmax_epilogue<BN>(p, acc, m_blk, n_blk, 0, lane);
        argmax_epilogue<BN>(p, acc + 64, m_blk, n_blk, 1, lane);
      } else if (!E::rope && p.fast && (m_blk + 1) * BM <= p.M && (n_blk + 1) * BN <= p.N) {
        epilogue<E, TI, BN, true>(p, acc, m_blk, n_blk, 0, lane);
        epilogue<E, TI, BN, true>(p, acc + 64, m_blk, n_blk, 1, lane);
      } else {
        epilogue<E, TI, BN, false>(p, acc, m_blk, n_blk, 0, lane);
        epilogue<E, TI, BN, false>(p, acc + 64, m_blk, n_blk, 1, lane);
      }
    }
    if (threadIdx.x == 0) trace_stamp(p, 6);
  }
  __syncthreads();
  if (threadIdx.x == 0) trace_stamp(p, 7);
}

// FP8 form (ape_gemm_tn_e4m3): e4m3 A [M, K] and W [N, K] with an fp32 scale per row of each, C = (A W^T) * a_scale[m] *
// w_scale[n], then the epilogue E of the 16-bit kernels (TO: the 16-bit output type).  The tiles of gemm_tc_kernel with
// CL = 1, BN = 128, and a single producer warp (288 threads): a 128-byte swizzle row holds 128 e4m3 values, so one k-block
// is 128 of K, the stage sizes are those of the 16-bit kernel, and a warpgroup issues 4 x m64n128k32 per k-block.
// Hopper's FP8 MMA does not keep full fp32 precision when it accumulates over a long K, so each k-block's 4 MMAs go into a
// scratch fragment (the first with scale_d = 0) that is added to the fp32 accumulator in registers once they have
// completed: one promotion per 128 of K, as CUTLASS's FP8 kernels without "fast accumulation" do.  The second fragment is
// why this is the cooperative form (64 + 64 accumulators per thread); a ping-pong warpgroup already holds 128.
constexpr int BK8 = 128;
constexpr int kFp8Threads = 32 * kConsumerWarps + 32;  // producer: warp 8

template <typename TO, class E>
__global__ void __launch_bounds__(kFp8Threads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GemmParams p,
                const float *__restrict__ a_scale, const float *__restrict__ w_scale) {
  constexpr int BN = 128, STAGES = 6;
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  using Smem = GemmSmem<BN, STAGES>;  // BK x 16 bit = BK8 x 8 bit per row: the same bytes
  Smem &s = *reinterpret_cast<Smem *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr uint32_t STAGE_BYTES = (BM + BN) * BK8;

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int num_tiles = p.m_blocks * p.n_blocks;
  auto tile_at = [&](int t, int &m_blk, int &n_blk) -> bool {  // gemm_tc_kernel's order with CL = 1
    const int tile = blockIdx.x + t * gridDim.x;
    if (tile >= num_tiles) return false;
    const int per_band = p.band * p.n_blocks;
    const int band = tile / per_band, r = tile - band * per_band;
    const int rows = min(p.band, p.m_blocks - band * p.band);
    n_blk = r / rows;
    m_blk = band * p.band + r - n_blk * rows;
    return true;
  };

  if (warp == kConsumerWarps && lane == 0) {
    tc::prefetch_tensormap(&map_a);
    tc::prefetch_tensormap(&map_b);
#pragma unroll
    for (int i = 0; i < STAGES; ++i) {
      tc::mbar_init(&s.full[i], 1);
      tc::mbar_init(&s.empty[i], kConsumerWarps);
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == kConsumerWarps) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      uint32_t stage = 0, phase = 0;
      int m_blk, n_blk;
      for (int t = 0; tile_at(t, m_blk, n_blk); ++t) {
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          tc::mbar_wait(&s.empty[stage], phase ^ 1);
          tc::mbar_expect_tx(&s.full[stage], STAGE_BYTES);
          tc::tma_load_2d(s.a[stage], &map_a, &s.full[stage], kb * BK8, m_blk * BM);
          tc::tma_load_2d(s.b[stage], &map_b, &s.full[stage], kb * BK8, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63 of the tile =====================
    const int wg = warp / 4, warp4 = warp & 3, tq = lane & 3;
    float acc[BN / 2], part[BN / 2];
    uint32_t stage = 0, phase = 0;
    int m_blk, n_blk;
    for (int t = 0; tile_at(t, m_blk, n_blk); ++t) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        tc::mbar_wait(&s.full[stage], phase);
        const uint64_t da = tc::make_smem_desc_sw128(tc::smem_u32(s.a[stage] + wg * 64 * BK8));
        const uint64_t db = tc::make_smem_desc_sw128(tc::smem_u32(s.b[stage]));
        tc::fence_regs<BN / 2>(part);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK8 / 32; ++k)  // 32 elements (32 B) along K per instruction
          tc::Wgmma<BN, __nv_fp8_e4m3>::template ss<0>(part, da + 2 * k, db + 2 * k, k != 0);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::fence_regs<BN / 2>(part);
        if (lane == 0) tc::mbar_arrive(&s.empty[stage]);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];  // promotion into the fp32 accumulator
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      // dequantise: acc * a_scale[m] * w_scale[n] in fp32 (rows past M read row M - 1, columns past N scale by 0)
      const int m0 = m_blk * BM + wg * 64 + warp4 * 16 + (lane >> 2);
      const float sa0 = __ldg(a_scale + min(m0, p.M - 1)), sa1 = __ldg(a_scale + min(m0 + 8, p.M - 1));
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n_blk * BN + 8 * j + 2 * tq;
        const float sw0 = n < p.N ? __ldg(w_scale + n) : 0.f, sw1 = n + 1 < p.N ? __ldg(w_scale + n + 1) : 0.f;
        acc[4 * j] = acc[4 * j] * sa0 * sw0;
        acc[4 * j + 1] = acc[4 * j + 1] * sa0 * sw1;
        acc[4 * j + 2] = acc[4 * j + 2] * sa1 * sw0;
        acc[4 * j + 3] = acc[4 * j + 3] * sa1 * sw1;
      }
      if (p.fast && (m_blk + 1) * BM <= p.M && (n_blk + 1) * BN <= p.N) epilogue<E, TO, BN, true>(p, acc, m_blk, n_blk, wg, lane);
      else epilogue<E, TO, BN, false>(p, acc, m_blk, n_blk, wg, lane);
    }
  }
  __syncthreads();
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

// [rows, K] 16-bit row-major matrix with pitch `ld` elements; box = 64 (K) x box_rows, 128 B swizzle.  An e4m3 matrix
// (APE_DTYPE_E4M3) is mapped as bytes, and its box of box_cols = BK8 elements is the same 128-byte row.
int make_map(CUtensorMap *map, const void *base, int dtype, long long rows, long long K, long long ld, int box_rows,
             int box_cols = BK) {
  EncodeTiledFn enc = get_encoder();
  if (!enc) return fail(APE_ERR_UNSUPPORTED, "gemm: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * (dtype == APE_DTYPE_F32 ? 4 : dtype == APE_DTYPE_E4M3 ? 1 : 2)};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, dtype == APE_DTYPE_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                        : dtype == APE_DTYPE_E4M3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
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

// PP: the ping-pong kernel (BN = 128, STAGES = 6, CL = 1 only)
template <int BN, int STAGES, int CL, typename TI, class E, bool PP = false>
int launch_gemm(const CUtensorMap &ma, const CUtensorMap &mb, GemmParams &p, cudaStream_t st) {
  static_assert(!PP || (BN == 128 && STAGES == 6 && CL == 1), "gemm_pp_kernel is BN = 128, 6 stages, single CTA");
  using Smem = GemmSmem<BN, STAGES>;
  const size_t smem = sizeof(Smem) + 1024;
  auto k = PP ? gemm_pp_kernel<TI, E> : gemm_tc_kernel<BN, STAGES, CL, TI, E>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "gemm: cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
    attr_set = true;
  }
  p.n_blocks = (p.N + BN - 1) / BN;
  const int m_groups = (p.m_blocks + CL - 1) / CL;
  const int groups = m_groups * p.n_blocks;
  const int max_clusters = num_sms() / CL;
  const int clusters = groups < max_clusters ? groups : max_clusters;
  // raster band: the fewest row groups whose tiles across all column blocks occupy every resident CTA.  Its A rows
  // (band x 128 x K) and the whole of W stay in L2 for the model's shapes (W is at most 11 MB: the ViT SwiGLU w12).
  p.band = std::min(m_groups, (clusters + p.n_blocks - 1) / p.n_blocks);
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
// pp: the ping-pong kernel (gemm_impl selects it only for bn = 128 without a cluster)
template <int CL, typename TI, class E>
int launch_bn(int bn, bool pp, const CUtensorMap &ma, const CUtensorMap &mb, GemmParams &p, cudaStream_t st) {
  if (bn == 256) return launch_gemm<256, 4, CL, TI, E>(ma, mb, p, st);
  if constexpr (CL == 1)
    if (pp) return launch_gemm<128, 6, 1, TI, E, true>(ma, mb, p, st);
  return launch_gemm<128, 6, CL, TI, E>(ma, mb, p, st);
}

struct EpiKey {
  bool out32;
  int act, res;
  bool ln, rope, stats;
};

// The epilogues with a kernel, X(out32, act, residual, ln, rope, stats), each for fp16 and bf16 operands; a 16-bit output
// or residual has the operand type.  Any other combination is rejected.
//   model call sites                                                     tests/test_gemm_gpu.py adds
//   16-bit  none             most projections, heads, 1x1 / 3x3 convs     16-bit + 16-bit residual, any of none/relu/gelu
//   16-bit  relu             encoder / decoder FFN1, MLP heads           fp32 + relu / gelu / swiglu
//   16-bit  gelu             text-tower MLP
//   16-bit  + fp32 residual  MSDA output projection, MLP with residual
//   16-bit  swiglu (+stats)  ViT w12
//   16-bit  rope             ViT qkv with fused rotary embedding
//   fp32    none / clamp     class / box heads, mask logits, text projection, vision-language logits
//   fp32    + fp32 / 16-bit residual   ViT proj / w3 / patch embed, encoder FFN2, text blocks, decoder self-attention out
//   fp32    LN fold + fp32 residual    ViT proj / w3 after the sub-LayerNorms
#define APE_GEMM_EPILOGUES(X)                                                                                            \
  X(false, ACT_NONE, RES_NONE, false, false, false) X(false, ACT_RELU, RES_NONE, false, false, false)                   \
  X(false, ACT_GELU, RES_NONE, false, false, false) X(false, ACT_NONE, RES_F32, false, false, false)                    \
  X(false, ACT_NONE, RES_16, false, false, false) X(false, ACT_RELU, RES_16, false, false, false)                       \
  X(false, ACT_GELU, RES_16, false, false, false) X(false, ACT_SWIGLU, RES_NONE, false, false, false)                   \
  X(false, ACT_SWIGLU, RES_NONE, false, false, true) X(false, ACT_NONE, RES_NONE, false, true, false)                   \
  X(true, ACT_NONE, RES_NONE, false, false, false) X(true, ACT_RELU, RES_NONE, false, false, false)                     \
  X(true, ACT_GELU, RES_NONE, false, false, false) X(true, ACT_SWIGLU, RES_NONE, false, false, false)                   \
  X(true, ACT_CLAMP, RES_NONE, false, false, false) X(true, ACT_NONE, RES_F32, false, false, false)                     \
  X(true, ACT_NONE, RES_16, false, false, false) X(true, ACT_NONE, RES_F32, true, false, false)

template <int CL, typename TI>
int launch_epi(int bn, bool pp, const EpiKey &k, const CUtensorMap &ma, const CUtensorMap &mb, GemmParams &p, cudaStream_t st) {
#define APE_EPI_CASE(o, a, r, l, ro, s)                                                                                  \
  if (k.out32 == o && k.act == a && k.res == r && k.ln == l && k.rope == ro && k.stats == s)                           \
    return launch_bn<CL, TI, Epi<o, a, r, l, ro, s>>(bn, pp, ma, mb, p, st);
  APE_GEMM_EPILOGUES(APE_EPI_CASE)
#undef APE_EPI_CASE
  return fail(APE_ERR_UNSUPPORTED, "gemm: no kernel for the epilogue (fp32 out %d, act %d, residual %d, ln %d, rope %d, stats %d)",
              (int)k.out32, k.act, k.res, (int)k.ln, (int)k.rope, (int)k.stats);
}

int launch_any(int bn, bool cluster, bool pp, int in_dtype, const EpiKey &k, const CUtensorMap &ma, const CUtensorMap &mb,
               GemmParams &p, cudaStream_t st) {
  if (in_dtype == APE_DTYPE_BF16)
    return cluster ? launch_epi<2, __nv_bfloat16>(bn, false, k, ma, mb, p, st) : launch_epi<1, __nv_bfloat16>(bn, pp, k, ma, mb, p, st);
  return cluster ? launch_epi<2, __half>(bn, false, k, ma, mb, p, st) : launch_epi<1, __half>(bn, pp, k, ma, mb, p, st);
}

// Ping-pong pays off when most CTAs get a tile for each consumer warpgroup; with fewer tiles (the 900-row decoder
// GEMMs) the cooperative kernel, which splits one tile over both warpgroups, finishes a CTA's single tile sooner.
bool use_pingpong(int tiles) { return tiles >= 2 * num_sms(); }

// 128 x 256 tiles on single CTAs for long-K wide GEMMs (the ViT-L w3, 4096 x 1024 x 2730): each CTA's 43-k-block main
// loop is long against its exposed epilogue, and the 128 tiles fill the SMs in one round; it took 46 us where the 128 x 128
// cluster of two took 110 (tests/perf_gemm_256.py, DESIGN.md §5).  Elsewhere 128 stays: at K = 512 to 1024 the 128 x 128
// ping-pong kernel, which hides each epilogue under the other warpgroup's MMAs, beat the cooperative 128 x 256 tile on
// qkv, w12 and the pyramid deconvolutions, and the cooperative 128 x 128 tile beat it on proj.  A cluster of two was
// slower than a single CTA at both widths on every shape measured, although it halves the weight traffic from L2.
bool use_wide(int N, int K) { return N >= 1024 && K >= 2048; }

template <typename TO, class E>
int launch_fp8(const CUtensorMap &ma, const CUtensorMap &mb, GemmParams &p, const float *a_scale, const float *w_scale,
               cudaStream_t st) {
  constexpr int BN = 128;
  const size_t smem = sizeof(GemmSmem<BN, 6>) + 1024;
  auto k = gemm_fp8_kernel<TO, E>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "gemm_e4m3: cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
    attr_set = true;
  }
  p.n_blocks = (p.N + BN - 1) / BN;
  const int tiles = p.m_blocks * p.n_blocks;
  const int ctas = std::min(tiles, num_sms());
  p.band = std::min(p.m_blocks, (ctas + p.n_blocks - 1) / p.n_blocks);  // raster band as in launch_gemm
  APE_LAUNCH(k, ctas, kFp8Threads, smem, st, ma, mb, p, a_scale, w_scale);
  return check_launch("gemm_fp8_kernel");
}

// The e4m3 epilogues: 16-bit output + bias (ViT qkv), SwiGLU with and without the row statistics (ViT w12).
template <typename TO>
int launch_fp8_epi(int act, bool stats, const CUtensorMap &ma, const CUtensorMap &mb, GemmParams &p, const float *a_scale,
                   const float *w_scale, cudaStream_t st) {
  if (act == ACT_NONE && !stats) return launch_fp8<TO, Epi<false, ACT_NONE, RES_NONE>>(ma, mb, p, a_scale, w_scale, st);
  if (act == ACT_SWIGLU && !stats) return launch_fp8<TO, Epi<false, ACT_SWIGLU, RES_NONE>>(ma, mb, p, a_scale, w_scale, st);
  if (act == ACT_SWIGLU) return launch_fp8<TO, Epi<false, ACT_SWIGLU, RES_NONE, false, false, true>>(ma, mb, p, a_scale, w_scale, st);
  return fail(APE_ERR_UNSUPPORTED, "gemm_e4m3: no kernel for activation %d (none or swiglu only)", act);
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
  const bool force_pp = (tile_n & 0x8000) != 0, force_coop = (tile_n & 0x10000) != 0;
  const int m_blocks = (M + BM - 1) / BM;
  // Tile width: 128, or 128 x 256 on a single CTA where use_wide says so.  An explicit width in tile_n (128 or 256)
  // overrides the rule, and bits 0x8000 / 0x10000 (below) pin the 128-wide kernels unless a width is given.
  const bool wide = (tile_n & 0xfff) == 0 && !force_pp && !force_coop && use_wide(N, K);
  const int bn = (tile_n & 0xfff) > 0 ? (tile_n & 0xfff) : wide ? 256 : 128;
  if (bn != 128 && bn != 256) return fail(APE_ERR_INVALID_ARG, "gemm: tile_n must be 128 or 256");
  if (tile_n & 0x2000) return fail(APE_ERR_UNSUPPORTED, "gemm: tile_n flag 0x2000 (CTA-pair MMA) is not available on sm_90a");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // kernel variant: single CTA, or a cluster of 2 along M sharing the weight tile by TMA multicast.  The 128-wide
  // GEMMs with a long K loop (K >= 2048: FFN2 and the 3x3 convolutions) take the cluster, where the weight tile is the
  // larger share of the operand traffic; bit 0x1000 forces the single CTA, bit 0x4000 the cluster.
  // A single-CTA BN = 128 GEMM runs the ping-pong kernel when there are enough tiles (use_pingpong); bit 0x8000 forces
  // it (single CTA), bit 0x10000 forces the cooperative kernel.
  if (force_pp && (force_coop || bn != 128 || (tile_n & 0x4000)))
    return fail(APE_ERR_INVALID_ARG, "gemm: tile_n flag 0x8000 (ping-pong) needs tile width 128, no cluster and no 0x10000");
  const bool cluster = m_blocks >= 2 && !force_pp && (tile_n & 0x1000) == 0 && ((tile_n & 0x4000) != 0 || (!wide && K >= 2048));
  const bool pp = !cluster && bn == 128 && !force_coop && (force_pp || use_pingpong(m_blocks * ((N + bn - 1) / bn)));
  CUtensorMap ma, mb;
  if (int rc = make_map(&ma, A, in_dtype, M, K, lda, BM)) return rc;
  if (int rc = make_map(&mb, W, in_dtype, N, K, ldw, cluster ? bn / 2 : bn)) return rc;
  GemmParams p{};
  p.C = C; p.bias = bias; p.residual = residual; p.ldc = ldc; p.ldr = ldr;
  p.M = M; p.N = N; p.K = K;
  p.m_blocks = m_blocks;
  p.k_blocks = (K + BK - 1) / BK;
  p.trace = g_gemm_trace;
  const int oe = out_dtype == APE_DTYPE_F32 ? 4 : 2;
  if (oe == 2 && out_dtype != in_dtype)
    return fail(APE_ERR_UNSUPPORTED, "gemm: a 16-bit output must have the operand dtype (out %d, operands %d)", out_dtype, in_dtype);
  if (residual && res_dtype != APE_DTYPE_F32 && res_dtype != in_dtype)
    return fail(APE_ERR_UNSUPPORTED, "gemm: a 16-bit residual must have the operand dtype (residual %d, operands %d)", res_dtype, in_dtype);
  const auto pairs = [](const void *ptr, long long ld, int esize) {  // rows start on 2-element boundaries
    return (ld % 2) == 0 && (reinterpret_cast<uintptr_t>(ptr) % (2 * esize)) == 0;
  };
  p.vec_out = pairs(C, ldc, oe);
  p.fast = p.vec_out && (!residual || pairs(residual, ldr, res_dtype == APE_DTYPE_F32 ? 4 : 2)) &&
           reinterpret_cast<uintptr_t>(bias) % 8 == 0 && (!fuse || reinterpret_cast<uintptr_t>(fuse->ln_colsum) % 8 == 0);
  EpiKey key{oe == 4, act, !residual ? RES_NONE : res_dtype == APE_DTYPE_F32 ? RES_F32 : RES_16, false, rope != nullptr, false};
  const int n_out = act == ACT_SWIGLU ? N / 2 : N;
  if (fuse) {
    if (fuse->ln_part) {
      if (out_dtype != APE_DTYPE_F32 || !fuse->ln_colsum || fuse->ln_nparts <= 0 || act == ACT_SWIGLU)
        return fail(APE_ERR_INVALID_ARG, "gemm+ln: needs an fp32 output, column sums and partial statistics");
      p.ln_part = fuse->ln_part; p.ln_colsum = fuse->ln_colsum; p.ln_nparts = fuse->ln_nparts;
      p.ln_inv_c = fuse->ln_inv_c; p.ln_eps = fuse->ln_eps;
      key.ln = true;
    }
    if (fuse->stats_out) {
      if (oe != 2 || act != ACT_SWIGLU || fuse->stats_nslab != (n_out + 63) / 64)
        return fail(APE_ERR_INVALID_ARG, "gemm+stats: needs the SwiGLU epilogue with a 16-bit output and stats_nslab = ceil(N/2/64)");
      p.stats_out = fuse->stats_out; p.stats_nslab = fuse->stats_nslab;
      key.stats = true;
    }
  }
  if (rope) {
    if (oe != 2 || act != ACT_NONE || rope->cols % 64 != 0 || rope->cols > N || rope->npos <= 0 || !rope->cos || !rope->sin)
      return fail(APE_ERR_INVALID_ARG, "gemm+rope: needs a 16-bit output, no activation, rope_cols a multiple of 64 <= N");
    p.rope_cos = rope->cos; p.rope_sin = rope->sin; p.rope_pos = rope->pos; p.rope_cols = rope->cols; p.rope_npos = rope->npos;
  }
  return launch_any(bn, cluster, pp, in_dtype, key, ma, mb, p, st);
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
  p.vec_out = 1;
  p.fast = reinterpret_cast<uintptr_t>(bias) % 8 == 0;
  p.conv = 1; p.conv_tw = tw; p.conv_th = th; p.conv_tiles_x = W / tw; p.conv_tiles_img = (W / tw) * (H / th); p.conv_cblks = Cin / 64;
  p.conv_W = W; p.conv_H = H;
  const EpiKey key{false, act, RES_NONE, false, false, false};
  return launch_any(bn, cluster, false, dtype, key, ma, mb, p, reinterpret_cast<cudaStream_t>(stream));
}

// keys[m] = max over n of argmax_key((A W^T)[m, n], n + col_base): the class argmax of every pixel row, merged into keys that
// the caller initialised (ape_semseg_keys_init).  Single-CTA BN = 128 kernel; K is the padded number of kept queries.
// E = EpiArgmaxDev (ape_gemm_tn_argmax_dev): the same over the first *m_dev rows, M being the capacity.
template <class E>
static int gemm_argmax(const void *A, int64_t lda, const void *W, int64_t ldw, uint64_t *keys, int M, const int *m_dev, int N, int K,
                       int col_base, int in_dtype, void *stream) {
  if (in_dtype != APE_DTYPE_F16 && in_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "gemm_argmax: operands must be fp16 or bf16 (got dtype %d)", in_dtype);
  if (M < 0 || N <= 0 || K <= 0 || col_base < 0 || (long long)col_base + N > 0x7fffffffLL)
    return fail(APE_ERR_INVALID_ARG, "gemm_argmax: bad sizes M=%d N=%d K=%d col_base=%d", M, N, K, col_base);
  if (M == 0) return APE_OK;
  if (!A || !W || !keys || (kDevRows<E> && !m_dev)) return fail(APE_ERR_NULL_PTR, "gemm_argmax: null pointer argument");
  if ((lda * 2) % 16 || (ldw * 2) % 16 || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15))
    return fail(APE_ERR_INVALID_ARG, "gemm_argmax: A/W base and row pitch must be 16-byte aligned (TMA)");
  if (lda < K || ldw < K) return fail(APE_ERR_INVALID_ARG, "gemm_argmax: row pitch smaller than K");
  if (reinterpret_cast<uintptr_t>(keys) & 7) return fail(APE_ERR_INVALID_ARG, "gemm_argmax: keys must be 8-byte aligned");
  constexpr int bn = 128;
  CUtensorMap ma, mb;
  if (int rc = make_map(&ma, A, in_dtype, M, K, lda, BM)) return rc;
  if (int rc = make_map(&mb, W, in_dtype, N, K, ldw, bn)) return rc;
  GemmParams p{};
  p.C = keys; p.M = M; p.N = N; p.K = K;
  p.m_blocks = (M + BM - 1) / BM;
  p.k_blocks = (K + BK - 1) / BK;
  p.trace = g_gemm_trace;
  p.argmax_col_base = col_base;
  p.residual = m_dev;  // EpiArgmaxDev's row count (nullptr otherwise, as before)
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // the device row count is read by the cooperative kernel's tile walk only, so EpiArgmaxDev always takes that kernel; both
  // kernels give every key the same MMA sequence and the keys merge by atomicMax, so the keys are the same either way
  if constexpr (!kDevRows<E>) {
    if (use_pingpong(p.m_blocks * ((N + bn - 1) / bn))) {
      if (in_dtype == APE_DTYPE_BF16) return launch_gemm<bn, 6, 1, __nv_bfloat16, E, true>(ma, mb, p, st);
      return launch_gemm<bn, 6, 1, __half, E, true>(ma, mb, p, st);
    }
  }
  if (in_dtype == APE_DTYPE_BF16) return launch_gemm<bn, 6, 1, __nv_bfloat16, E>(ma, mb, p, st);
  return launch_gemm<bn, 6, 1, __half, E>(ma, mb, p, st);
}

extern "C" int ape_gemm_tn_argmax(const void *A, int64_t lda, const void *W, int64_t ldw, uint64_t *keys, int M, int N, int K,
                                  int col_base, int in_dtype, void *stream) {
  return gemm_argmax<EpiArgmax>(A, lda, W, ldw, keys, M, nullptr, N, K, col_base, in_dtype, stream);
}

extern "C" int ape_gemm_tn_argmax_dev(const void *A, int64_t lda, const void *W, int64_t ldw, uint64_t *keys, int M, const int *m_rows,
                                      int N, int K, int col_base, int in_dtype, void *stream) {
  return gemm_argmax<EpiArgmaxDev>(A, lda, W, ldw, keys, M, m_rows, N, K, col_base, in_dtype, stream);
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

extern "C" int ape_gemm_tn_e4m3(const void *A, int64_t lda, const void *W, int64_t ldw, const float *a_scale,
                                const float *w_scale, void *C, int64_t ldc, const float *bias, int M, int N, int K, int out_dtype,
                                int act, float *stats_out, int stats_nslab, void *stream) {
  if (out_dtype != APE_DTYPE_F16 && out_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_UNSUPPORTED, "gemm_e4m3: output must be fp16 or bf16 (got dtype %d)", out_dtype);
  if (act != ACT_NONE && act != ACT_SWIGLU)
    return fail(APE_ERR_UNSUPPORTED, "gemm_e4m3: no kernel for activation %d (none or swiglu only)", act);
  if (M < 0 || N <= 0 || K <= 0) return fail(APE_ERR_INVALID_ARG, "gemm_e4m3: bad sizes M=%d N=%d K=%d", M, N, K);
  if (K % 16) return fail(APE_ERR_INVALID_ARG, "gemm_e4m3: K must be a multiple of 16 (got %d)", K);
  if (M == 0) return APE_OK;
  if (!A || !W || !C) return fail(APE_ERR_NULL_PTR, "gemm_e4m3: null pointer argument");
  if (!a_scale || !w_scale) return fail(APE_ERR_NULL_PTR, "gemm_e4m3: null scale pointer (a_scale [M] and w_scale [N] are required)");
  if (lda % 16 || ldw % 16 || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15))
    return fail(APE_ERR_INVALID_ARG, "gemm_e4m3: A/W base and row pitch must be 16-byte aligned (TMA)");
  if (lda < K || ldw < K) return fail(APE_ERR_INVALID_ARG, "gemm_e4m3: row pitch smaller than K");
  if ((reinterpret_cast<uintptr_t>(a_scale) | reinterpret_cast<uintptr_t>(w_scale)) & 3)
    return fail(APE_ERR_INVALID_ARG, "gemm_e4m3: scales must be 4-byte aligned fp32");
  if (act == ACT_SWIGLU && (N & 1)) return fail(APE_ERR_INVALID_ARG, "gemm_e4m3: swiglu needs even N");
  const int n_out = act == ACT_SWIGLU ? N / 2 : N;
  if (stats_out && (act != ACT_SWIGLU || stats_nslab != (n_out + 63) / 64))
    return fail(APE_ERR_INVALID_ARG, "gemm_e4m3+stats: needs the SwiGLU epilogue and stats_nslab = ceil(N/2/64)");
  CUtensorMap ma, mb;
  if (int rc = make_map(&ma, A, APE_DTYPE_E4M3, M, K, lda, BM, BK8)) return rc;
  if (int rc = make_map(&mb, W, APE_DTYPE_E4M3, N, K, ldw, 128, BK8)) return rc;
  GemmParams p{};
  p.C = C; p.bias = bias; p.ldc = ldc;
  p.M = M; p.N = N; p.K = K;
  p.m_blocks = (M + BM - 1) / BM;
  p.k_blocks = (K + BK8 - 1) / BK8;
  p.vec_out = (ldc % 2) == 0 && (reinterpret_cast<uintptr_t>(C) % 4) == 0;
  p.fast = p.vec_out && reinterpret_cast<uintptr_t>(bias) % 8 == 0;
  p.stats_out = stats_out;
  p.stats_nslab = stats_out ? stats_nslab : 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (out_dtype == APE_DTYPE_BF16) return launch_fp8_epi<__nv_bfloat16>(act, stats_out != nullptr, ma, mb, p, a_scale, w_scale, st);
  return launch_fp8_epi<__half>(act, stats_out != nullptr, ma, mb, p, a_scale, w_scale, st);
}
