// attn_xfwd.cu — cross attention with wide heads: the two softmax attentions of VisionLanguageFusion for phrase / text
// prompts (BiMultiHeadAttention.forward, ape/layers/fuse_helper.py:67-166):
//   vision  <- language :  out_v = softmax_t( q_s . k_t ) value_l     queries = S vision tokens, keys = N_t phrases
//   language <- vision  :  out_l = softmax_s( k_t . q_s ) value_v     queries = N_t phrases,      keys = S vision tokens
// 8 heads of 256 channels (embed_dim 2048), N_t up to 5 000, S up to 196 416 (BASELINE.json configs[3]); the reference
// materialises the S x N_t score matrix per head in fp32 (31 GB at that size) and applies both softmaxes to it.  Here each
// direction is one flash-attention pass (attn.cuh): the scores never leave registers.
//
// Equivalence with the reference's op sequence: it subtracts the GLOBAL maximum of the score matrix (a constant: both
// softmaxes are invariant to it) and clamps scores and shifted scores to +-5e4 (fuse_helper.py:88-110).  A clamp only
// changes a score that lies more than 5e4 below its row / global maximum, whose softmax weight is exp(-5e4) = 0 in fp32
// either way; the results are identical unless a WHOLE row sits 5e4 below the global maximum, which LayerNormed inputs
// (|q.k| is bounded by |q||k| of normalised vectors times the projection norms) cannot produce.
//
// Separate Q / K / V tensors (three tensor maps), different row counts for queries and keys, padded key rows masked.
// HD = 64: 128 queries per CTA (two consumer warpgroups).  HD = 256: the O accumulator is 128 fp32 registers per thread,
// so a CTA is one consumer warpgroup of 64 queries (160 KB of shared memory for Q and double-buffered K / V).
#include "attn.cuh"

using namespace ape;

extern "C" int ape_attn_cross_fwd(const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv, void *out,
                                  int64_t ldo, int num_seq, int nq, int nkv, int n_valid, int heads, int head_dim, float scale,
                                  int dtype, void *stream) {
  if (dtype != APE_DTYPE_F16 && dtype != APE_DTYPE_BF16) return fail(APE_ERR_INVALID_ARG, "attn_x: fp16 / bf16 only (dtype %d)", dtype);
  if (head_dim != 64 && head_dim != 256) return fail(APE_ERR_UNSUPPORTED, "attn_x: head_dim %d (64 or 256)", head_dim);
  if (num_seq < 0 || nq <= 0 || nq % 128 || nkv <= 0 || nkv % 64 || n_valid <= 0 || n_valid > nkv || heads <= 0 || heads > 65535 ||
      num_seq > 65535)
    return fail(APE_ERR_UNSUPPORTED, "attn_x: num_seq=%d nq=%d nkv=%d n_valid=%d heads=%d (nq %% 128 == 0, nkv %% 64 == 0)", num_seq, nq,
                nkv, n_valid, heads);
  if (num_seq == 0) return APE_OK;
  if (!q || !k || !v || !out) return fail(APE_ERR_NULL_PTR, "attn_x: null pointer argument");
  const int C = heads * head_dim;
  if (ldq < C || ldk < C || ldv < C || ldo < C || (ldq * 2) % 16 || (ldk * 2) % 16 || (ldv * 2) % 16 || (ldo * 2) % 16 ||
      ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(out)) & 15))
    return fail(APE_ERR_INVALID_ARG, "attn_x: operands [rows, >= heads*head_dim] with 16-byte aligned rows");
  CUtensorMap mq, mk, mv;
  if (int rc = attn::make_map(&mq, q, dtype, (long long)num_seq * nq, C, ldq)) return rc;
  if (int rc = attn::make_map(&mk, k, dtype, (long long)num_seq * nkv, C, ldk)) return rc;
  if (int rc = attn::make_map(&mv, v, dtype, (long long)num_seq * nkv, C, ldv)) return rc;
  attn::Params p{};
  p.out = out; p.ldo = ldo; p.heads = heads;
  p.q_seq_rows = nq; p.kv_seq_rows = nkv;
  p.n_valid = n_valid; p.q_store_rows = nq;
  p.scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (head_dim == 64) {
    const dim3 grid((unsigned)(nq / 128), (unsigned)heads, (unsigned)num_seq);
    if (dtype == APE_DTYPE_F16) return attn::launch<__half, 1, 2, false>(mq, mk, mv, p, grid, st);
    return attn::launch<__nv_bfloat16, 1, 2, false>(mq, mk, mv, p, grid, st);
  }
  const dim3 grid((unsigned)(nq / 64), (unsigned)heads, (unsigned)num_seq);
  if (dtype == APE_DTYPE_F16) return attn::launch<__half, 4, 1, false>(mq, mk, mv, p, grid, st);
  return attn::launch<__nv_bfloat16, 4, 1, false>(mq, mk, mv, p, grid, st);
}
