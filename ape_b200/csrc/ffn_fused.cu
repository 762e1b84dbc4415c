// ffn_fused.cu — the encoder / decoder feed-forward block in one kernel on the Hopper (sm_90a) tensor cores:
//   out[M, 256] (fp32) = relu(X W1^T + b1) W2^T + b2 + X
// X [M, 256], W1 [F, 256] and W2 [256, F] 16-bit in nn.Linear's own layouts, b1 / b2 fp32.  The [M, F] hidden activation
// never leaves the SM: for the APE-L_D encoder (M = 87 296, F = 2048) the two-GEMM path writes and re-reads 358 MB of it
// per layer.
//
// One CTA = 128 rows of X; it walks the hidden dimension in chunks of 64 (the flash-attention loop of attn.cuh with
// relu(S + b1) in place of the softmax).  Roles (384 threads; O, S and P need more than the 168 registers a thread of a
// 384-thread block gets, so the producer warpgroup hands registers to the consumers with setmaxnreg):
//   warpgroups 0, 1  consumers : warpgroup g owns rows 64g..64g+63 and a 64 x 256 fp32 O in registers.  Per chunk j:
//                                S_j = X W1_j^T      (wgmma m64n64k16 x 16, X and W1_j K-major in shared memory)
//                                P_j = relu(S_j + b1_j) rounded to 16 bit, repacked as the register A operand
//                                O  += P_j W2_j^T    (wgmma m64n256k16 x 4, W2_j = 256 rows x 64 hidden, K-major)
//                                the O MMAs of chunk j and the S MMAs of chunk j+1 are issued back to back
//   warpgroup 2      producer  : one thread issues TMA loads of X once, then W1_j / W2_j into double buffers (mbarrier full / empty).
// Arithmetic: the same k-ordered wgmma chains, the same fp32 epilogue operations and the same 16-bit rounding of the hidden
// activation as gemm_tc.cu's FFN1 (ReLU epilogue) followed by FFN2 (bias + 16-bit residual, fp32 output), so the result is
// the two-GEMM result.
// CL = 2 (selectable, not the default: measured slower): a cluster of two CTAs on adjacent row tiles; each loads half of
// every weight chunk and multicasts it to both, halving the weight traffic from L2 (every 128-row tile streams all of W1
// and W2).
#include "attn.cuh"  // make_map (64 x 64 swizzled boxes), pack2
#include "common.cuh"
#include "tc.cuh"

namespace ape {
namespace {

constexpr int E = 256, BM = 128, HC = 64;  // embedding width, rows per CTA, hidden chunk
constexpr int kThreads = 384;

struct alignas(1024) FfnSmem {
  uint8_t x[E / 64][BM * 128];     // X tile: 4 column chunks of 128 rows x 64 (128 B, swizzled)
  uint8_t w1[2][E / 64][HC * 128];  // W1_j: 4 column chunks of 64 hidden rows x 64
  uint8_t w2[2][E * 128];           // W2_j: 256 output rows x 64 hidden (one K-major 256-row tile)
  uint64_t x_full, w1_full[2], w1_empty[2], w2_full[2], w2_empty[2];
};

struct FfnParams {
  const float *b1, *b2;  // fp32 [F], [256], or nullptr
  const void *x;         // residual: the X the MMAs read
  float *out;
  long long ldx, ldo;
  int M, F;
};

template <typename T, int CL>
__global__ void __launch_bounds__(kThreads, 1)
ffn_fused_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w1,
                 const __grid_constant__ CUtensorMap map_w2, const FfnParams p) {
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  FfnSmem &s = *reinterpret_cast<FfnSmem *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = CL > 1 ? (int)tc::cluster_ctarank() : 0;
  const int row0 = blockIdx.x * BM;
  const int nch = p.F / HC;

  if (warp == 8 && lane == 0) {
    tc::prefetch_tensormap(&map_x);
    tc::prefetch_tensormap(&map_w1);
    tc::prefetch_tensormap(&map_w2);
    tc::mbar_init(&s.x_full, 1);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      tc::mbar_init(&s.w1_full[b], 1);
      tc::mbar_init(&s.w1_empty[b], 8 * CL);  // one arrival per consumer warp of each CTA of the cluster
      tc::mbar_init(&s.w2_full[b], 1);
      tc::mbar_init(&s.w2_empty[b], 8 * CL);
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  if (CL > 1) tc::cluster_sync_all();  // peer barriers are initialised before any multicast / remote arrive can reach them
  pdl_wait();  // X (the previous kernel's output) may be read and out written from here on

  if (warp >= 8) {
    // ===================== TMA producer =====================
    tc::setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      tc::mbar_expect_tx(&s.x_full, E * BM * 2);
#pragma unroll
      for (int c = 0; c < E / 64; ++c)
#pragma unroll
        for (int h = 0; h < 2; ++h) tc::tma_load_2d(s.x[c] + h * 64 * 128, &map_x, &s.x_full, c * 64, row0 + h * 64);
      for (int j = 0; j < nch; ++j) {
        const int b = j & 1, n = j >> 1;
        tc::mbar_wait(&s.w1_empty[b], (n & 1) ^ 1);
        tc::mbar_expect_tx(&s.w1_full[b], E * HC * 2);
        if (CL == 1) {
#pragma unroll
          for (int c = 0; c < E / 64; ++c) tc::tma_load_2d(s.w1[b][c], &map_w1, &s.w1_full[b], c * 64, j * HC);
        } else {
#pragma unroll
          for (int c = 2 * rank; c < 2 * rank + 2; ++c)
            tc::tma_load_2d_multicast(s.w1[b][c], &map_w1, &s.w1_full[b], c * 64, j * HC, (uint16_t)3);
        }
        tc::mbar_wait(&s.w2_empty[b], (n & 1) ^ 1);
        tc::mbar_expect_tx(&s.w2_full[b], E * HC * 2);
        if (CL == 1) {
#pragma unroll
          for (int q = 0; q < E / 64; ++q) tc::tma_load_2d(s.w2[b] + q * 64 * 128, &map_w2, &s.w2_full[b], j * HC, q * 64);
        } else {
#pragma unroll
          for (int q = 2 * rank; q < 2 * rank + 2; ++q)
            tc::tma_load_2d_multicast(s.w2[b] + q * 64 * 128, &map_w2, &s.w2_full[b], j * HC, q * 64, (uint16_t)3);
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers: warpgroup g, rows 16 * (warp % 4) + lane / 4 + 8 h (h = 0, 1) =====================
    tc::setmaxnreg_inc<232>();
    const int g = warp >> 2, tq = lane & 3;
    auto release = [&](uint64_t *bar) {  // the MMAs that read this buffer have completed (in this warp's view)
      if (lane == 0) {
        tc::mbar_arrive(bar);
        if (CL > 1) tc::mbar_arrive_cluster(tc::mapa_u32(bar, (uint32_t)(rank ^ 1)));
      }
    };
    auto issue_s = [&](float *sc, int b) {  // S = X W1_j^T, k in order
#pragma unroll
      for (int c = 0; c < E / 64; ++c) {
        const uint64_t dx = tc::make_smem_desc_sw128(tc::smem_u32(s.x[c] + g * 64 * 128));
        const uint64_t dw = tc::make_smem_desc_sw128(tc::smem_u32(s.w1[b][c]));
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::Wgmma<64, T>::template ss<0>(sc, dx + 2 * k, dw + 2 * k, (c | k) != 0);
      }
    };
    float o[E / 2];
#pragma unroll
    for (int i = 0; i < E / 2; ++i) o[i] = 0.f;
    float sc[32];
    tc::mbar_wait(&s.x_full, 0);
    tc::mbar_wait(&s.w1_full[0], 0);
    tc::wgmma_fence();
    issue_s(sc, 0);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::fence_regs<32>(sc);
    release(&s.w1_empty[0]);

    for (int j = 0; j < nch; ++j) {
      const int b = j & 1, n = j >> 1;
      // P_j = relu(S_j + b1) in 16 bit: act1(acc + bias) of the GEMM epilogue, then its paired round-to-nearest
      uint32_t pa[4][4];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float2 bb = make_float2(0.f, 0.f);
        if (p.b1 != nullptr) bb = __ldg(reinterpret_cast<const float2 *>(p.b1 + j * HC + 8 * jj + 2 * tq));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v0 = sc[4 * jj + 2 * h], v1 = sc[4 * jj + 2 * h + 1];
          if (p.b1 != nullptr) {
            v0 += bb.x;
            v1 += bb.y;
          }
          pa[jj >> 1][2 * (jj & 1) + h] = attn::pack2<T>(fmaxf(v0, 0.f), fmaxf(v1, 0.f));
        }
      }
      tc::mbar_wait(&s.w2_full[b], n & 1);
      tc::fence_regs<E / 2>(o);
      tc::wgmma_fence();
      const uint64_t dw2 = tc::make_smem_desc_sw128(tc::smem_u32(s.w2[b]));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) tc::Wgmma<256, T>::template rs<0>(o, pa[kk], dw2 + 2 * kk, (j | kk) != 0);
      tc::wgmma_commit();
      if (j + 1 < nch) {  // S_{j+1} queues behind O_j on the tensor cores
        const int b1 = b ^ 1;
        tc::mbar_wait(&s.w1_full[b1], ((j + 1) >> 1) & 1);
        issue_s(sc, b1);
        tc::wgmma_commit();
        tc::wgmma_wait<1>();
        tc::fence_regs<E / 2>(o);
        release(&s.w2_empty[b]);
        tc::wgmma_wait<0>();
        tc::fence_regs<32>(sc);
        release(&s.w1_empty[b1]);
      } else {
        tc::wgmma_wait<0>();
        tc::fence_regs<E / 2>(o);
        release(&s.w2_empty[b]);
      }
    }

    // ===================== epilogue: (O + b2) + X, fp32 paired stores; rows >= M are not written =====================
    const T *xg = reinterpret_cast<const T *>(p.x);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = row0 + g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (m < p.M) {
        const T *xr = xg + (size_t)m * p.ldx + 2 * tq;
        float *dst = p.out + (size_t)m * p.ldo + 2 * tq;
#pragma unroll
        for (int jj = 0; jj < E / 8; ++jj) {
          float v0 = o[4 * jj + 2 * h], v1 = o[4 * jj + 2 * h + 1];
          if (p.b2 != nullptr) {
            const float2 bb = __ldg(reinterpret_cast<const float2 *>(p.b2 + 8 * jj + 2 * tq));
            v0 += bb.x;
            v1 += bb.y;
          }
          const float2 r = Elem<T>::load2(xr + 8 * jj);
          v0 += r.x;
          v1 += r.y;
          *reinterpret_cast<float2 *>(dst + 8 * jj) = make_float2(v0, v1);
        }
      }
    }
  }
  __syncthreads();
  if (CL > 1) tc::cluster_sync_all();  // no CTA leaves while its peer can still signal its barriers
}

template <typename T, int CL>
int launch(const CUtensorMap &mx, const CUtensorMap &m1, const CUtensorMap &m2, const FfnParams &p, cudaStream_t st) {
  const size_t smem = sizeof(FfnSmem) + 1024;
  auto k = ffn_fused_kernel<T, CL>;
  static bool set = false;
  if (!set) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "ffn_fused: cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
    set = true;
  }
  const int tiles = (p.M + BM - 1) / BM;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)((tiles + CL - 1) / CL * CL));
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
  cudaError_t e = cudaLaunchKernelEx(&cfg, k, mx, m1, m2, p);
  if (e != cudaSuccess) return fail((int)e, "ffn_fused_kernel launch: %s", cudaGetErrorString(e));
  return check_launch("ffn_fused_kernel");
}

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int ape_ffn_fused(const void *x, int64_t ldx, const void *w1, int64_t ldw1, const float *b1, const void *w2,
                             int64_t ldw2, const float *b2, float *out, int64_t ldo, int M, int E_, int F, int dtype,
                             int variant, void *stream) {
  if (dtype != APE_DTYPE_F16 && dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "ffn_fused: operands must be fp16 or bf16 (got dtype %d)", dtype);
  if (E_ != E) return fail(APE_ERR_UNSUPPORTED, "ffn_fused: embedding width %d (only %d)", E_, E);
  if (F <= 0 || F % HC) return fail(APE_ERR_UNSUPPORTED, "ffn_fused: hidden width %d is not a positive multiple of %d", F, HC);
  if (M < 0) return fail(APE_ERR_INVALID_ARG, "ffn_fused: bad row count %d", M);
  if (variant < 0 || variant > 2) return fail(APE_ERR_INVALID_ARG, "ffn_fused: bad variant %d", variant);
  if (ldo == 0) ldo = E;
  if (M == 0) return APE_OK;
  if (!x || !w1 || !w2 || !out) return fail(APE_ERR_NULL_PTR, "ffn_fused: null pointer argument");
  if (((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w1) | reinterpret_cast<uintptr_t>(w2)) & 15) ||
      ldx % 8 || ldw1 % 8 || ldw2 % 8)
    return fail(APE_ERR_INVALID_ARG, "ffn_fused: x / w1 / w2 base and row pitch must be 16-byte aligned (TMA)");
  if (ldx < E || ldw1 < E || ldw2 < F || ldo < E) return fail(APE_ERR_INVALID_ARG, "ffn_fused: row pitch smaller than the row");
  if ((reinterpret_cast<uintptr_t>(out) & 7) || ldo % 2 ||
      ((reinterpret_cast<uintptr_t>(b1) | reinterpret_cast<uintptr_t>(b2)) & 7))
    return fail(APE_ERR_INVALID_ARG, "ffn_fused: out (and its row pitch) and b1 / b2 must allow 8-byte pairs");
  CUtensorMap mx, m1, m2;
  if (int rc = attn::make_map(&mx, x, dtype, M, E, ldx)) return rc;
  if (int rc = attn::make_map(&m1, w1, dtype, F, E, ldw1)) return rc;
  if (int rc = attn::make_map(&m2, w2, dtype, E, F, ldw2)) return rc;
  FfnParams p{b1, b2, x, out, ldx, ldo, M, F};
  // variant 0 = default = 1: one CTA per row tile; 2: clusters of two.  On an H100 at 400 W the cluster was the slower one at
  // both the encoder (87 296 rows: 581 vs 460 us, fp16) and the decoder shape (900 rows: 88 vs 61 us).
  const bool cluster = variant == 2;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == APE_DTYPE_BF16)
    return cluster ? launch<__nv_bfloat16, 2>(mx, m1, m2, p, st) : launch<__nv_bfloat16, 1>(mx, m1, m2, p, st);
  return cluster ? launch<__half, 2>(mx, m1, m2, p, st) : launch<__half, 1>(mx, m1, m2, p, st);
}
