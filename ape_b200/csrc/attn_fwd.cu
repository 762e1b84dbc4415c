// attn_fwd.cu — softmax attention core of the EVA-02 ViT blocks (Attention.forward, ape/modeling/backbone/
// vit_eva_clip.py:218-319: q·k^T·scale -> softmax -> ·v, 16 heads x 64, window (N=1024) and global (N=4096) blocks)
// and of the EVA02-CLIP text tower (causal, 77-token prompts packed at a row stride): flash-attention forward with wgmma
// (attn.cuh), Q/K/V tiles staged by TMA straight out of the fused [M, 3C] qkv buffer the qkv GEMM wrote (no head split
// copies).  One CTA = 128 queries (two consumer warpgroups) of one (sequence, head).
#include <stdlib.h>

#include "attn.cuh"

namespace ape {
namespace {
constexpr int QM = 128, HD = 64;
constexpr int kDefaultAttnVariant = 1;
}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int ape_attn_fwd_ex(const void *qkv, int64_t ld, void *out, int64_t ldo, int num_seq, int n, int n_valid, int heads,
                               int head_dim, float scale, int dtype, float *stats_out, int seq_stride, int causal, int64_t total_rows,
                               void *stream);

// Kernel structure used by ape_attn_fwd*: 0 = P written to shared memory and read from there by the P.V MMA, 1 = P kept in
// registers as the MMA's A operand.  set >= 0 selects it for the process (tests / tuning); returns the value in force.  The
// initial value comes from APE_ATTN_VARIANT or the built-in default.
extern "C" int ape_attn_variant(int set) {
  static int current = [] {
    const char *e = getenv("APE_ATTN_VARIANT");
    return e != nullptr ? atoi(e) : kDefaultAttnVariant;
  }();
  if (set >= 0) current = set ? 1 : 0;
  return current;
}

extern "C" int ape_attn_fwd(const void *qkv, int64_t ld, void *out, int64_t ldo, int num_seq, int n, int heads,
                            int head_dim, float scale, int dtype, void *stream) {
  return ape_attn_fwd_ex(qkv, ld, out, ldo, num_seq, n, n, heads, head_dim, scale, dtype, nullptr, 0, 0, 0, stream);
}

extern "C" int ape_attn_fwd_ex(const void *qkv, int64_t ld, void *out, int64_t ldo, int num_seq, int n, int n_valid, int heads,
                               int head_dim, float scale, int dtype, float *stats_out, int seq_stride, int causal, int64_t total_rows,
                               void *stream) {
  if (n_valid <= 0 || n_valid > n) return fail(APE_ERR_INVALID_ARG, "attn: n_valid=%d must be in [1, n=%d]", n_valid, n);
  if (seq_stride <= 0) seq_stride = n;
  if (seq_stride < n_valid) return fail(APE_ERR_INVALID_ARG, "attn: seq_stride=%d smaller than n_valid=%d", seq_stride, n_valid);
  if (total_rows <= 0) total_rows = (int64_t)(num_seq - 1) * seq_stride + n;
  if (total_rows < (int64_t)(num_seq - 1) * seq_stride + n_valid) return fail(APE_ERR_INVALID_ARG, "attn: total_rows too small");
  if (dtype != APE_DTYPE_F16 && dtype != APE_DTYPE_BF16) return fail(APE_ERR_INVALID_ARG, "attn: fp16 / bf16 only (dtype %d)", dtype);
  if (head_dim != HD) return fail(APE_ERR_UNSUPPORTED, "attn: head_dim %d (only 64)", head_dim);
  if (num_seq < 0 || n <= 0 || n % QM != 0 || heads <= 0 || heads > 65535 || num_seq > 65535)
    return fail(APE_ERR_UNSUPPORTED, "attn: num_seq=%d n=%d heads=%d (n must be a multiple of 128)", num_seq, n, heads);
  if (num_seq == 0) return APE_OK;
  if (!qkv || !out) return fail(APE_ERR_NULL_PTR, "attn: null pointer argument");
  const int C = heads * HD;
  if (ld < 3 * C || ldo < C || (ld * 2) % 16 || (ldo * 2) % 16 || (reinterpret_cast<uintptr_t>(qkv) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15))
    return fail(APE_ERR_INVALID_ARG, "attn: qkv [rows, >= 3*heads*64] / out [rows, >= heads*64] with 16-byte aligned rows");
  CUtensorMap map;  // rows past the buffer read as zeros (TMA)
  if (int rc = attn::make_map(&map, qkv, dtype, total_rows, 3 * C, ld)) return rc;
  attn::Params p{};
  p.out = out; p.ldo = ldo; p.heads = heads; p.stats_out = stats_out;
  p.q_seq_rows = seq_stride; p.kv_seq_rows = seq_stride;
  p.q_col0 = 0; p.k_col0 = C; p.v_col0 = 2 * C;
  p.n_valid = n_valid; p.causal = causal ? 1 : 0;
  p.q_store_rows = seq_stride >= n ? n : n_valid;
  p.scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid((unsigned)(n / QM), (unsigned)heads, (unsigned)num_seq);
  const bool p_smem = ape_attn_variant(-1) == 0;
  if (dtype == APE_DTYPE_F16)
    return p_smem ? attn::launch<__half, 1, 2, true>(map, map, map, p, grid, st) : attn::launch<__half, 1, 2, false>(map, map, map, p, grid, st);
  return p_smem ? attn::launch<__nv_bfloat16, 1, 2, true>(map, map, map, p, grid, st)
                : attn::launch<__nv_bfloat16, 1, 2, false>(map, map, map, p, grid, st);
}
