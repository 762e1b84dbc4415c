/*
 * ape_b200.h — C-ABI of libape_b200.so, the sm_90a (H100) kernels behind APE's
 * detection forward pass.
 *
 * Every entry point is `extern "C"`, takes plain device pointers and sizes, a
 * `cudaStream_t` passed as `void*`, never allocates, never synchronises, and is
 * safe to call under CUDA-graph capture.  Return value: 0 = ok, <0 = invalid
 * argument (text in ape_last_error()), >0 = a cudaError_t from the launch.
 *
 * Reference interfaces replaced (paths relative to the APE repository):
 *   ape_msda_fwd            <- torch.ops.ape.ms_deform_attn_forward
 *                              ape/layers/csrc/vision.cpp:76-79 (registration)
 *                              ape/layers/csrc/MsDeformAttn/ms_deform_attn.h:21-40 (dispatch)
 *                              ape/layers/csrc/MsDeformAttn/ms_deform_attn_cuda.cu:21-81 (host)
 *                              ape/layers/csrc/MsDeformAttn/ms_deform_im2col_cuda.cuh:237-299 (kernel)
 *   ape_msda_fused_fwd      <- MultiScaleDeformableAttention.forward tail
 *                              ape/layers/multi_scale_deform_attn.py:283-348
 *                              (softmax + sampling-location arithmetic + gather in one launch)
 * The Python side that binds these (ctypes) and registers the reference's
 * operator names lives in ape_b200/_lib.py and ape_b200/ops.py; the binding a
 * reference maintainer would add is shown in INTEGRATION.md.
 */
#ifndef APE_B200_H_
#define APE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define APE_ABI_VERSION 3

/* element types accepted by the kernels (value of the `dtype` argument) */
#define APE_DTYPE_F32 0
#define APE_DTYPE_F16 1
#define APE_DTYPE_BF16 2
#define APE_DTYPE_E4M3 3 /* FP8 e4m3 (torch.float8_e4m3fn): ape_gemm_tn_e4m3 operands, ape_layernorm_e4m3 output */

/* status codes (<0); positive return values are cudaError_t */
#define APE_OK 0
#define APE_ERR_INVALID_ARG (-1)
#define APE_ERR_UNSUPPORTED (-2)
#define APE_ERR_NULL_PTR (-3)

int ape_abi_version(void);

/* Text of the last non-zero status returned on the calling thread ("" if none). */
const char *ape_last_error(void);

/* Number of kernels this library has launched since load (all threads). */
uint64_t ape_launch_count(void);

/*
 * Multi-scale deformable attention, forward.
 *
 *   out[b,q,h,:] = sum_{l<L} sum_{p<P} attn[b,q,h,l,p] *
 *                  bilinear_zero_pad(value_l[b,:,h,:], loc[b,q,h,l,p] * (W_l,H_l) - 0.5)
 *
 * value   [B,S,H,D]      contiguous, dtype
 * spatial_shapes [L,2]   int64 (H_l, W_l), DEVICE memory (as in the reference op)
 * level_start    [L]     int64, DEVICE memory
 * loc     [B,Q,H,L,P,2]  contiguous, dtype, (x,y) normalised to [0,1]
 * attn    [B,Q,H,L,P]    contiguous, dtype
 * out     [B,Q,H*D]      contiguous, dtype; fully overwritten (no pre-zeroing needed)
 *
 * Accumulation is always fp32 (the reference accumulates in `dtype`,
 * ms_deform_im2col_cuda.cuh:270).  Sample kept iff h_im>-1 && w_im>-1 &&
 * h_im<H_l && w_im<W_l (…cuh:285-291), per-corner validity as …cuh:56-78.
 */
int ape_msda_fwd(const void *value, const int64_t *spatial_shapes, const int64_t *level_start,
                 const void *loc, const void *attn, void *out, int B, int S, int H, int D, int L,
                 int Q, int P, int dtype, void *stream);

/*
 * Same contract as ape_msda_fwd but selects a kernel variant explicitly
 * (used by bench.py / tests to sweep mappings; `variant` < 0 = default).
 *   variant = heads_per_cta (1,2,4,8) | unroll<<8 ; 0x1000 = scalar fallback kernel
 */
int ape_msda_fwd_variant(const void *value, const int64_t *spatial_shapes, const int64_t *level_start,
                         const void *loc, const void *attn, void *out, int B, int S, int H, int D,
                         int L, int Q, int P, int dtype, int variant, void *stream);

/*
 * Fused tail of MultiScaleDeformableAttention.forward (multi_scale_deform_attn.py:283-348):
 * takes the raw outputs of the sampling_offsets / attention_weights linears and the
 * reference points, performs softmax over L*P, the sampling-location arithmetic and
 * the gather in one launch (sampling locations and attention weights never touch HBM).
 *
 * value     [B,S,H,D]        dtype
 * offsets   [B,Q,H,L,P,2]    offs_dtype (raw linear output), row stride `offs_row_stride` elements per (b,q)
 * logits    [B,Q,H,L*P]      offs_dtype (raw linear output), row stride `logit_row_stride` elements per (b,q)
 * ref       [B,Q,L,ref_dim]  fp32, ref_dim 2 (points) or 4 (boxes cx,cy,w,h)
 *   ref_dim 2: loc = ref + off / (W_l,H_l)                      (…py:298-303)
 *   ref_dim 4: loc = ref_xy + off / P * ref_wh * 0.5            (…py:304-311)
 * out       [B,Q,H*D]        dtype
 */
int ape_msda_fused_fwd(const void *value, const int64_t *spatial_shapes, const int64_t *level_start,
                       const void *offsets, int64_t offs_row_stride, const void *logits,
                       int64_t logit_row_stride, const float *ref, int ref_dim, void *out, int B,
                       int S, int H, int D, int L, int Q, int P, int dtype, int offs_dtype,
                       void *stream);

/*
 * Second-generation fused kernel for calls with many queries (the encoder: Q = S = 87 296 at 1024^2), 16-bit value, D = 32,
 * P = 4.  `value2` is the PAIR layout [B][S][H][2][D]: entry (s, h) = channels of token s followed by those of token s+1, one
 * aligned 128-byte line, so a bilinear sample costs two full L1 lines instead of four half-used ones; the four corners of
 * the P points of one level are blended with packed 16-bit FMAs, levels are summed in fp32 (the reference's half kernel
 * accumulates everything in half, ms_deform_im2col_cuda.cuh:270,290).  Same sampling semantics as ape_msda_fused_fwd.
 *   ape_msda_pair_values     value [B,S,H*D] (row pitch ld elements) -> value2; token_mask [B*S] bytes or NULL zeroes masked
 *                            tokens (key_padding_mask, multi_scale_deform_attn.py:286-287)
 *   ape_msda_pair_supported  1 if the geometry is covered (host_shapes int32 [L,2] on the HOST: every level >= 2 wide)
 *   ape_msda_pair_fused_fwd  heads_per_cta: 0 = auto (1 for Q >= 128: a CTA's 32 rows are queries of one head);
 *                            tile_w: for Q == S the CTA's queries form a tile_w x (32 / heads_per_cta / tile_w) PIXEL tile of one
 *                            level (texel re-use in both directions); 0 = consecutive queries, -1 = auto (8);
 *                            head_major: CTA order (0: heads of one tile adjacent, 1: tiles of one head adjacent)
 */
int ape_msda_pair_values(const void *value, int64_t ld, void *value2, const uint8_t *token_mask, int B, int S, int H, int D,
                         int dtype, void *stream);
int ape_msda_pair_supported(const int *host_shapes, int L, int H, int D, int P, int dtype);
int ape_msda_pair_fused_fwd(const void *value2, const int64_t *spatial_shapes, const int64_t *level_start,
                            const int *host_shapes, const void *offsets, int64_t offs_row_stride, const void *logits,
                            int64_t logit_row_stride, const float *ref, int ref_dim, void *out, int B, int S, int H, int D,
                            int L, int Q, int P, int dtype, int offs_dtype, int heads_per_cta, int tile_w, int head_major,
                            void *stream);

/*
 * Multi-scale deformable attention, backward  <- torch.ops.ape.ms_deform_attn_backward
 *   (ape/layers/csrc/vision.cpp:78, ms_deform_attn.h:42-61, ms_deform_attn_cuda.cu:84-160,
 *    ms_deform_im2col_cuda.cuh:86-146 per-sample arithmetic, :301-920 kernels).
 * Inputs as ape_msda_fwd plus grad_out [B,Q,H*D] (dtype).  Outputs: grad_value_f32 [B,S,H,D] ALWAYS fp32 and pre-zeroed by
 * the caller (vector atomics accumulate into it; the caller casts to dtype), grad_loc [B,Q,H,L,P,2] and grad_attn
 * [B,Q,H,L,P] in dtype, fully overwritten.  fp32 arithmetic for every dtype.
 */
int ape_msda_bwd(const void *value, const int64_t *spatial_shapes, const int64_t *level_start, const void *loc,
                 const void *attn, const void *grad_out, float *grad_value_f32, void *grad_loc, void *grad_attn, int B,
                 int S, int H, int D, int L, int Q, int P, int dtype, void *stream);

/*
 * Tensor-core linear layer: C[M,N] = act(A[M,K] * W[N,K]^T + bias) (+ residual), TMA + wgmma.
 * Replaces the nn.Linear (cuBLAS) calls of the detection path (vit_eva_clip.py:225-232,266-267,125-132;
 * deformable_transformer_vl.py:36-54; multi_scale_deform_attn.py:278-295,353; vision_language_align.py:36-48).
 *
 * A [M,K] and W [N,K] (nn.Linear weight layout) are fp16 or bf16 (in_dtype), K contiguous, row pitches
 * lda / ldw in elements (16-byte aligned rows).  fp32 accumulation in registers (wgmma).
 * bias: fp32 [N] or NULL.  residual: [M,N] of out_dtype with pitch ldr, or NULL.
 * act: 0 none, 1 ReLU, 2 GELU(erf), 3 SwiGLU over interleaved (gate, up) column pairs -> C is [M, N/2],
 *      4 clamp to +-50000 (VisionLanguageAlign, vision_language_align.py:49-51).
 * out_dtype: APE_DTYPE_* of C (pitch ldc elements).  tile_n: 0 = auto, or 128 / 256 (| 0x1000 forces a single CTA, | 0x4000 a
 * cluster of two CTAs sharing the weight tile by TMA multicast; without either the cluster is used for K >= 2048).
 */
int ape_gemm_tn(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc, const float *bias,
                const void *residual, int64_t ldr, int M, int N, int K, int in_dtype, int out_dtype, int act,
                int tile_n, void *stream);

/* ape_gemm_tn with the residual in its own element type (res_dtype): the engine keeps the residual stream / pre-LayerNorm
 * sums in fp32 (out_dtype F32) while GEMM operands and LayerNorm outputs are 16-bit, so e.g. a 16-bit residual is added
 * into an fp32 output (encoder: query + output_proj(...)) or an fp32 residual into an fp32 output (ViT: x + proj(...)). */
int ape_gemm_tn_ex(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc, const float *bias,
                   const void *residual, int64_t ldr, int res_dtype, int M, int N, int K, int in_dtype, int out_dtype,
                   int act, int tile_n, void *stream);

/*
 * ape_gemm_tn_ex with a LayerNorm folded around it (the sub-LayerNorms of the EVA-02 block, vit_eva_clip.py:266,130):
 *   consume: ln_part [M, ln_nparts, 2] per-row partial (sum, sum of squares) of the RAW 16-bit A written by its producer;
 *            W must hold gamma .* W, ln_colsum [N] its row sums (of the 16-bit values), bias = beta W^T + b; the epilogue forms
 *            rstd * (A W'^T - mean * colsum) + bias (+ residual); fp32 output only.  ln_inv_c = 1 / C, ln_eps as the LayerNorm.
 *   produce: stats_out [M, ceil(N/2/64), 2] with act = SwiGLU: (sum, sum of squares) of every 64-column slab of the output.
 * Either half may be disabled with NULL.
 */
int ape_gemm_tn_fused(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc, const float *bias,
                      const void *residual, int64_t ldr, int res_dtype, int M, int N, int K, int in_dtype, int out_dtype,
                      int act, int tile_n, const float *ln_part, int ln_nparts, const float *ln_colsum, float ln_inv_c,
                      float ln_eps, float *stats_out, int stats_nslab, void *stream);

/*
 * FP8 linear layer: C[M, N] = act((A W^T) * a_scale[m] * w_scale[n] + bias), e4m3 x e4m3 on the wgmma tensor cores.
 * A [M, K] and W [N, K] are e4m3 bytes (torch.float8_e4m3fn), K contiguous, row pitches lda / ldw in elements (= bytes),
 * 16-byte aligned; K a multiple of 16.  a_scale fp32 [M] and w_scale fp32 [N] are required (dequantised value = q * scale).
 * The products of e4m3 values are exact; they are summed in fp32, promoted from the tensor cores' accumulator into an fp32
 * register accumulator every 128 of K.  The scales are applied first, in fp32, then the epilogue of ape_gemm_tn_fused:
 * bias fp32 [N] or NULL, and act 0 (none) or 3 (SwiGLU over interleaved column pairs, C [M, N/2]; stats_out as in
 * ape_gemm_tn_fused, or NULL).  out_dtype fp16 or bf16 (pitch ldc elements).  Other epilogues: APE_ERR_UNSUPPORTED.
 */
int ape_gemm_tn_e4m3(const void *A, int64_t lda, const void *W, int64_t ldw, const float *a_scale, const float *w_scale, void *C,
                     int64_t ldc, const float *bias, int M, int N, int K, int out_dtype, int act, float *stats_out,
                     int stats_nslab, void *stream);

/*
 * 3x3 convolution (stride 1, zero padding 1) over NHWC activations as an implicit GEMM on the wgmma kernel: the 3x3
 * convolutions of SimpleFeaturePyramid (vit_eva_clip.py:804-847) and of the mask head (deformable_detr_segm_vl.py:741-747).
 * x [B,H,W,Cin], w [Cout,3,3,Cin] (= the Conv2d weight permuted (0,2,3,1)), y [B,H,W,Cout], bias fp32 [Cout] or NULL;
 * fp16 / bf16, fp32 accumulation; act 0 / 1 (ReLU) / 2 (GELU).  Cin % 64 == 0; the image must be a whole number of
 * tw x (128/tw) pixel tiles, tw the largest power of two <= 128 dividing W.
 */
int ape_conv3x3_nhwc(const void *x, const void *w, void *y, const float *bias, int B, int H, int W, int Cin, int Cout,
                     int dtype, int act, void *stream);

/*
 * ape_gemm_tn with the 2-D rotary embedding of the ViT (VisionRotaryEmbeddingFast, utils_eva02.py:248-252,346) fused into
 * the epilogue: C = A W^T + bias, then t' = t*cos + rotate_half(t)*sin on output columns [0, rope_cols) — the q and k
 * thirds of the fused qkv projection (vit_eva_clip.py:225-262) — in fp32 before the single rounding to the 16-bit
 * output.  cos/sin fp32 [npos, 64]; row m uses position pos_map[m] (int32, device) or m % npos when NULL; head_dim 64.
 */
int ape_gemm_tn_rope(const void *A, int64_t lda, const void *W, int64_t ldw, void *C, int64_t ldc, const float *bias,
                     int M, int N, int K, int in_dtype, int out_dtype, const float *cos_table, const float *sin_table,
                     const int *pos_map, int npos, int head_dim, int rope_cols, int tile_n, void *stream);

/*
 * The transformer FFN block (detrex FFN(num_fcs=2): Linear -> ReLU -> Linear + identity) in one launch:
 *   out[M, E] (fp32) = relu(x w1^T + b1) w2^T + b2 + x
 * x [M, E] (pitch ldx), w1 [F, E] (pitch ldw1), w2 [E, F] (pitch ldw2) 16-bit of one dtype in nn.Linear's layouts, 16-byte
 * aligned bases and pitches; b1 fp32 [F], b2 fp32 [E] (NULL = no bias); out fp32, pitch ldo (0 = E), 8-byte pairs.
 * E must be 256 and F a multiple of 64 (APE_ERR_UNSUPPORTED otherwise).  The [M, F] hidden activation stays on chip; the
 * result equals ape_gemm_tn_ex(x, w1, act relu, 16-bit out) followed by ape_gemm_tn_ex(h, w2, + b2, 16-bit residual x, fp32 out)
 * bit for bit.  variant: 0 = default (= 1), 1 = one CTA per 128-row tile, 2 = clusters of two row tiles sharing the weight
 * chunks by TMA multicast (A/B runs).
 */
int ape_ffn_fused(const void *x, int64_t ldx, const void *w1, int64_t ldw1, const float *b1, const void *w2, int64_t ldw2,
                  const float *b2, float *out, int64_t ldo, int M, int E, int F, int dtype, int variant, void *stream);

/*
 * Development aid (no reference counterpart): when device_buffer is not NULL, every CTA of the following ape_gemm_tn*
 * launches writes 8 clock64() stamps to device_buffer[8 * blockIdx.x ..]:
 * entry, set-up done, first operands landed, last MMA issued, first / last accumulator complete, epilogue drained, exit.
 * NULL switches it off.  Process-wide, not for concurrent use.
 */
void ape_gemm_set_trace(long long *device_buffer);

/*
 * LayerNorm over the last dimension (nn.LayerNorm / inner_attn_ln / ffn_ln of vit_eva_clip.py:505-523,266,130;
 * norms of the detrex transformer layers).  fp32 statistics; x [rows, C] pitch ldx (in_dtype), y pitch ldy
 * (out_dtype); weight/bias fp32 [C].  Pitches must cover C rounded up to 8 elements; padding elements
 * are written as 0.  row_map (int32 [rows], device) or NULL: output row of input row r (window partition).
 */
int ape_layernorm(const void *x, int64_t ldx, void *y, int64_t ldy, const float *weight, const float *bias,
                  const int *row_map, int rows, int C, float eps, int in_dtype, int out_dtype, void *stream);

/*
 * ape_layernorm with an e4m3 output and a scale per row, the A operand of ape_gemm_tn_e4m3: with t the fp32 LayerNorm output
 * of row r (after weight and bias, as ape_layernorm computes it), s = max|t| / 448 (0 for an all-zero row) and
 * y[out_row] = e4m3(t / s), rounded to nearest even and saturating (0 where s = 0), scale[out_row] = s.  C <= 1024; y pitch
 * ldy bytes, a multiple of 16 covering C rounded up to 8; padding bytes are written as 0.  row_map as in ape_layernorm.
 */
int ape_layernorm_e4m3(const void *x, int64_t ldx, void *y, int64_t ldy, float *scale, const float *weight, const float *bias,
                       const int *row_map, int rows, int C, float eps, int in_dtype, void *stream);

/*
 * Extended LayerNorm for the deformable encoder (C % 8 == 0, C <= 1024); one pass over the activations for
 *   t = LN(x; weight, bias, eps)                 norms[1] of a detrex BaseTransformerLayer (deformable_transformer_vl.py:36-54)
 *   t = LN(t; weight2, bias2, eps2)  if weight2  layer_norm_v of the next VisionLanguageFusion (fuse_helper.py:224)
 *   y = t + col_add[image, :]        if col_add  gamma_v * delta_v of that fusion (one fp32 [C] vector per image for
 *                                                "name" prompts; col_add_stride elements between images, rows_per_image rows each)
 *   y2 = y + row_add[row, :]         if y2       query + query_pos (multi_scale_deform_attn.py:262-263); row_add / y2 in out_dtype
 * weight NULL: no normalisation (t = x; bias and weight2 must be NULL) and y may be NULL, so that only y2 = x + row_add is
 * written: the first layer of an encoder without fusion layers (deformable_transformer.py:78-102).
 */
int ape_layernorm_ex(const void *x, int64_t ldx, void *y, int64_t ldy, const float *weight, const float *bias, float eps,
                     const float *weight2, const float *bias2, float eps2, const float *col_add, int64_t col_add_stride,
                     int rows_per_image, const void *row_add, int64_t ld_add, void *y2, int64_t ldy2, int rows, int C,
                     int in_dtype, int out_dtype, void *stream);

/*
 * GroupNorm over token-major activations x [B, rows_per_image, C] (the neck's GroupNorm(32, 256) after each
 * 1x1 conv, configs/…1080k.py:42-55): statistics per (image, group) over all rows x C/groups channels, fp32,
 * deterministic.  y_batch_stride: elements between images of y (0 = rows_per_image * ldy), so the result can be
 * written straight into its slice of the flattened multi-level feature tensor.
 * workspace: ape_groupnorm_workspace_bytes(B, rows_per_image, C) bytes.
 */
int64_t ape_groupnorm_workspace_bytes(int B, int rows_per_image, int C);
int ape_groupnorm_nhwc(const void *x, int64_t ldx, void *y, int64_t ldy, int64_t y_batch_stride, const float *weight,
                       const float *bias, void *workspace, int B, int rows_per_image, int C, int groups, float eps,
                       int in_dtype, int out_dtype, void *stream);

/*
 * In-place 2-D rotary embedding on the q and k thirds of a fused qkv buffer [M, 3*C] (pitch ld):
 * t' = t*cos + rotate_half(t)*sin (VisionRotaryEmbeddingFast, utils_eva02.py:248-252,346).
 * cos/sin fp32 [npos, head_dim]; token m uses row pos_map[m] (int32, device) or m % npos when NULL.
 */
int ape_rope_qk(void *qkv, int64_t ld, const float *cos_table, const float *sin_table, const int *pos_map, int M,
                int C, int head_dim, int npos, int dtype, void *stream);

/*
 * First residual of the text tower over length-packed prompts (TextTransformer.forward, eva02_clip/transformer.py:722-724):
 * x[r, :] = token_embedding[tok[r], :] + positional_embedding[pos[r], :], all fp32, x [rows, D] contiguous, D % 4 == 0,
 * tables [vocab, D] / [ctx, D] contiguous and 16-byte aligned; tok / pos int32 [rows] (device).  A row with pos[r] < 0 (a
 * pad row of a tile) is written as zeros, and so is a row whose token id or position lies outside its table.
 */
int ape_text_embed_packed(const float *token_embedding, const float *positional_embedding, const int *tok, const int *pos,
                          float *x, int rows, int D, int vocab, int ctx, void *stream);
/* out[i, :] = x[rows[i], :] for i < n: fp32 rows of D elements (D % 4 == 0, pitches ldx / ldo in elements, 16-byte aligned
 * rows), rows int64 [n] on the device, every entry a row of x.  The text tower reads its end-of-text rows with it. */
int ape_rows_gather(const float *x, int64_t ldx, const int64_t *rows, float *out, int64_t ldo, int n, int D, void *stream);

/*
 * Softmax attention core of the ViT blocks (Attention.forward, ape/modeling/backbone/vit_eva_clip.py:218-319, the
 * part xformers / F.scaled_dot_product_attention computes there): out = softmax(q k^T * scale) v per (sequence, head),
 * flash-attention style on the wgmma tensor cores.  qkv [num_seq * n, >= 3*heads*64] (pitch ld elements): columns
 * [0,C) = q, [C,2C) = k, [2C,3C) = v with C = heads*64, head h at columns h*64 (the layout the fused qkv GEMM writes,
 * RoPE already applied); sequence s owns rows [s*n, (s+1)*n).  out [num_seq * n, >= C] (pitch ldo).  fp16 or bf16,
 * head_dim 64, n a multiple of 128; fp32 softmax statistics and accumulation.
 */
int ape_attn_fwd(const void *qkv, int64_t ld, void *out, int64_t ldo, int num_seq, int n, int heads, int head_dim,
                 float scale, int dtype, void *stream);
/* Same with sequences padded to n rows: only the first n_valid keys of every sequence take part in the softmax (the rows
 * beyond must hold finite values, e.g. zeros).  Used for the self-attention over the 900 decoder queries
 * (deformable_transformer_vl.py:142-147: nn.MultiheadAttention, 8 heads x 32 — heads zero-padded to 64 channels). */
/* stats_out (or NULL): fp32 [rows, heads, 2] — per row and head the (sum, sum of squares) of the 64 output values as stored,
 * consumed by ape_gemm_tn_fused to fold the LayerNorm that follows (inner_attn_ln, vit_eva_clip.py:266) into the projection.
 * seq_stride (0 = n): rows between consecutive sequences; sequences may be packed tighter than the 128-row tile (the text
 * tower packs 77-token prompts at a stride of 80 rows): rows of a tile past n_valid are then neither attended nor written.
 * causal: key t only sees keys <= t (eva02_clip/transformer.py:714-720).  total_rows (0 = derived): rows of the qkv buffer. */
int ape_attn_fwd_ex(const void *qkv, int64_t ld, void *out, int64_t ldo, int num_seq, int n, int n_valid, int heads,
                    int head_dim, float scale, int dtype, float *stats_out, int seq_stride, int causal, int64_t total_rows,
                    void *stream);
/* ape_attn_fwd_ex with a scattered output: out_row_map (int32, device, one entry per query row of the launch, i.e.
 * (num_seq - 1) * seq_stride + the rows stored per sequence) gives the row of out and of stats_out that query row r is
 * stored at; -1 leaves nothing written for that row.  Lets the padded 14x14 windows of the APE-Ti ViT (vit_eva02.py)
 * write their attention output straight back into raster token order, skipping the pad tokens.  Mapped rows must lie
 * inside out / stats_out and be distinct. */
int ape_attn_fwd_mapped(const void *qkv, int64_t ld, void *out, int64_t ldo, int num_seq, int n, int n_valid, int heads,
                        int head_dim, float scale, int dtype, float *stats_out, int seq_stride, int causal, int64_t total_rows,
                        const int *out_row_map, void *stream);
/* ape_attn_fwd_ex over tiles that hold several short sequences each (the text tower's length-packed prompts): seg_start
 * (int32, device, one entry per query row of the launch) gives, for query row r of a tile, the position inside that tile
 * where r's own sequence starts; r attends key k of its tile iff seg_start[r] <= k <= r.  A pad row carries its own position
 * and so attends only itself (finite output).  n = n_valid = 128, seq_stride 0 or 128, causal != 0: anything else is
 * APE_ERR_UNSUPPORTED.  With seg_start[r] = 0 everywhere the result equals ape_attn_fwd_ex(causal = 1) bit for bit. */
int ape_attn_fwd_seg(const void *qkv, int64_t ld, void *out, int64_t ldo, int num_seq, int n, int n_valid, int heads,
                     int head_dim, float scale, int dtype, float *stats_out, int seq_stride, int causal, int64_t total_rows,
                     const int *seg_start, void *stream);

/* Kernel structure behind ape_attn_fwd*: 0 = P written to shared memory and read from there by the P.V wgmma, 1 = P kept in
 * registers as the A operand of the P.V wgmma.  set >= 0 selects it for the process; returns the value in force
 * (initially APE_ATTN_VARIANT or the built-in default). */
int ape_attn_variant(int set);

/*
 * Cross attention with separate Q / K / V tensors and 64- or 256-channel heads: the two softmax attentions of
 * VisionLanguageFusion for phrase / text prompts (BiMultiHeadAttention.forward, ape/layers/fuse_helper.py:67-166: 8 heads x 256;
 * vision <- language: queries = S vision tokens, keys = N_t phrases; language <- vision: the transposed roles), one
 * flash-attention pass per direction — the S x N_t score matrix (31 GB in fp32 at 1536^2 / 5 000 phrases) is never formed.
 * q [num_seq * nq, >= heads*head_dim], k / v [num_seq * nkv, ...], out like q; nq a multiple of 128, nkv a multiple of 64 (rows
 * padded by the caller with finite values), only the first n_valid keys of every sequence count.  fp16 / bf16, fp32 softmax
 * statistics and accumulation.  The reference's global-max shift and +-5e4 clamps are softmax-invariant for LayerNormed
 * inputs (see csrc/attn_xfwd.cu).
 */
int ape_attn_cross_fwd(const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv, void *out, int64_t ldo,
                       int num_seq, int nq, int nkv, int n_valid, int heads, int head_dim, float scale, int dtype, void *stream);

/*
 * Language-side attention pooling of VisionLanguageFusion for a single language token ("name" prompts):
 * softmax over the S vision tokens of scores t[s,h] = v_s . qa[h] + qc[h] (with the reference's global-max shift
 * and +-5e4 clamps, fuse_helper.py:88-110) and the p-weighted sum of v.  v [B,S,C] dtype; qa [B,NH,C], qc [B,NH] fp32.
 * Results are left as per-strip partials in the workspace: *partial_out -> [B, *strips_out, NH, C+1] fp32
 * (last column = sum of exp).  workspace: ape_vlf_pool_workspace_bytes(B,S,C,NH) bytes.
 */
int64_t ape_vlf_pool_workspace_bytes(int B, int S, int C, int NH);
int ape_vlf_pool(const void *v, const float *qa, const float *qc, void *workspace, float **partial_out, int *strips_out,
                 int B, int S, int C, int NH, int stable_softmax_2d, int dtype, void *stream);

/*
 * Greedy hard NMS over boxes already sorted by descending score (torchvision.ops.nms semantics; replaces the
 * nms call inside batched_nms of deformable_transformer_vl.py:591-596 and fast_rcnn.py:192).
 * boxes_sorted [n,4] fp32 xyxy (16-byte aligned); keep [n] bytes (1 = survives); *count = survivors (device int).
 * workspace: ape_nms_workspace_bytes(n) bytes of device memory.
 */
int64_t ape_nms_workspace_bytes(int n);
int ape_nms_sorted(const float *boxes_sorted, int n, float iou_threshold, void *workspace, uint8_t *keep, int *count,
                   void *stream);
/* Same, for static-shape callers (CUDA graphs): buffers are sized for n_max boxes, only the first min(n_max, *n_dev)
 * (device int) are real; keep[i] = 0 for the rest.  workspace: ape_nms_workspace_bytes(n_max). */
int ape_nms_sorted_dev(const float *boxes_sorted, int n_max, const int *n_dev, float iou_threshold, void *workspace,
                       uint8_t *keep, int *count, void *stream);

/*
 * Class-aware NMS when (almost) every (query, class) pair is a candidate (test_score_thresh 0.0: 900 queries x 1203 names;
 * fast_rcnn.py:129-192 -> batched_nms, class by class as torchvision's _batched_nms_vanilla).  All classes share the Q
 * per-query boxes, so one Q x Q IoU bit matrix serves every class; one warp sorts and scans one class.
 * boxes [Q,4] fp32 xyxy (16-byte aligned), scores [Q,N] fp32 (row pitch ld_scores), row_valid [Q] bytes or NULL,
 * candidates = valid rows with score > score_thresh.  out [N,Q] fp32 CLASS-major: the score where (q, c) survives, -inf
 * elsewhere (a top-k over it yields the detections in descending score order).  Q <= 1024.
 * workspace: ape_nms_classwise_workspace_bytes(Q).
 */
int64_t ape_nms_classwise_workspace_bytes(int Q);
int ape_nms_classwise(const float *boxes, const float *scores, int64_t ld_scores, const uint8_t *row_valid, int Q, int N,
                      float score_thresh, float iou_threshold, void *workspace, float *out, void *stream);

/*
 * Input pipeline of the predictor (SURVEY.md 8(f) row 3): the ResizeShortestEdge of DefaultPredictor.__call__
 * (ape/engine/defaults.py:203-230 -> detectron2 ResizeTransform.apply_image -> PIL Image.resize(BILINEAR) for uint8 images)
 * on the device, BIT-EXACT with Pillow's libImaging/Resample.c (triangle filter widened by the down-scaling factor, 22-bit
 * fixed-point taps, uint8 intermediate between the horizontal and the vertical pass).
 *   ape_resample_ksize      taps per output sample for one axis (host)
 *   ape_resample_coeffs_u8  HOST tables of one axis: bounds [out,2] int32 (first source sample, tap count), kk [out,ksize] int32
 *   ape_resample_u8         src [H,W,C] uint8 (row pitch src_pitch bytes) -> out float32 planes [C][new_h][new_w] with element
 *                           strides (plane_stride, row_stride); tmp [H,new_w,C] uint8 workspace; tables as DEVICE copies;
 *                           flip_channels: source channel c lands in plane C-1-c (BGR -> RGB, defaults.py:218-220)
 */
int ape_resample_ksize(int in_size, int out_size);
int ape_resample_coeffs_u8(int in_size, int out_size, int *bounds_host, int *kk_host);
int ape_resample_u8(const uint8_t *src, int64_t src_pitch, uint8_t *tmp, float *out, int64_t plane_stride, int64_t row_stride,
                    const int *bounds_h, const int *kk_h, int ksize_h, const int *bounds_v, const int *kk_v, int ksize_v, int H,
                    int W, int C, int new_h, int new_w, int flip_channels, void *stream);

/* Decoder reference-point update (deformable_transformer_vl.py:268-300, 4-d reference points): new_ref [B,Q,4] =
 * sigmoid(delta + inverse_sigmoid(ref, eps)) and ref_in [B,Q,L,4] = new_ref[:,:,None] * cat(valid_ratios, valid_ratios)[:,None]
 * (valid_ratios [B,L,2]); all fp32, same operation order as the PyTorch sequence. */
int ape_ref_update(const float *delta, const float *ref, const float *valid_ratios, float *new_ref, float *ref_in, int B, int Q,
                   int L, float eps, void *stream);

/* y[b,n] = W[n,:] . x[b,:] + bias[n] in fp32 for 1..4 input rows (the folded language-side maps of VisionLanguageFusion for one
 * language token, ape/layers/fuse_helper.py:67-166 restructured): W [N,K] row-major, K a multiple of 4, W / x 16-byte aligned. */
int ape_gemv_f32(const float *W, const float *x, const float *bias, float *y, int B, int N, int K, void *stream);

/*
 * Instance-mask post-processing for the detections that survive the final selection (deformable_detr_segm_vl.py:569-603 and
 * detectron2 detector_postprocess / paste_masks_in_image), without the full-resolution fp32 maps:
 *   ape_mask_crop   logits [Q,h,w] dtype (one image), index [K] int64 kept queries, boxes [K,4] fp32 xyxy in padded-image
 *                   pixels -> out [K,S,S] bytes = (ROIAlign(S, scale 1, sampling_ratio 0, aligned) of (bilinear upsample to
 *                   Hp x Wp, align_corners=False, > 0) >= 0.5), i.e. BitMasks(sigmoid(mask) > 0.5).crop_and_resize(boxes, S).
 *                   workspace: ape_mask_crop_workspace_bytes(K, Hp, Wp) (one bit per upsampled pixel).
 *   ape_mask_paste  masks [N,S,S] bytes (0 / 1), boxes [N,4] fp32 in OUTPUT-image pixels -> out [N,img_h,img_w] bytes (bool):
 *                   bilinear grid_sample (zeros padding, align_corners=False) of the mask inside its box >= threshold.
 * boxes 16-byte aligned.
 */
int64_t ape_mask_crop_workspace_bytes(int K, int Hp, int Wp);
int ape_mask_crop(const void *logits, const int64_t *index, const float *boxes, void *workspace, uint8_t *out, int K, int h, int w,
                  int Hp, int Wp, int S, int dtype, void *stream);
int ape_mask_paste(const uint8_t *masks, const float *boxes, uint8_t *out, int N, int S, int img_h, int img_w, float threshold,
                   void *stream);
/*
 * The pasted masks as COCO run-length codes without ever writing the dense masks (the evaluators encode every pasted mask with
 * cocoapi's mask_util.encode(np.array(mask[:, :, None], order="F")) right away: ape/evaluation/d3_evaluation.py:466-468,
 * refcoco_evaluation.py:450-452, detectron2 instances_to_coco_json): runs of equal pixels in COLUMN-major order.
 *   ape_mask_paste_rle  pass 1 (positions == NULL): col_count [N,img_w] int32 <- run boundaries per (mask, column);
 *                       pass 2: positions <- the boundary positions x*img_h + y, in order, at col_offset [N,img_w] int64 =
 *                       exclusive scan of col_count over the whole array.  Same pixel arithmetic as ape_mask_paste.
 *   ape_rle_to_string   HOST: run lengths (first run = zeros) -> cocoapi's compressed "counts" string (rleToString); returns
 *                       the number of characters (out holds up to 7 per count).
 */
int ape_mask_paste_rle(const uint8_t *masks, const float *boxes, int N, int S, int img_h, int img_w, float threshold,
                       int *col_count, const int64_t *col_offset, int *positions, void *stream);
int ape_rle_to_string(const uint32_t *counts, int m, char *out);
/*
 * The kept instance masks of the packed selection rows as COCO run-length codes in fixed-size slots, with no count read back
 * by the host: CUDA-graph capturable, and the result is one fixed-shape tensor for one collective.  Replaces, per image, the
 * reference's paste_masks_in_image (detectron2 detector_postprocess), then mask_util.encode / instances_to_coco_json (the
 * evaluator's encoding of every pasted mask), then the pickled comm.gather of those codes (lvis_evaluation.py:103-104).
 *   ape_mask_pack  logits [B,Q,h,w] dtype; rows [B,topk,13] fp32 as DeformableDETRSegmVL.forward_packed writes them (x1, y1,
 *                  x2, y2 in image pixels, score, class, query index, candidates, kept nk, image h, w, output h, w); out_hw
 *                  HOST int32 [B,2] = the output sizes (the same as the rows' last two columns).  For each slot < nk whose
 *                  box is non-empty after detector_postprocess's rescale and clip: ape_mask_crop over the padded size Hp x Wp,
 *                  then the paste into the rescaled box at threshold 0.5 encoded as cocoapi's rleToString "counts".
 *                  out [B,topk,60+slot] bytes per slot: the 13 fp32 columns; int32 kind (0 no mask, 1 counts characters,
 *                  2 the S x S mask as bits: pixel y*S+x at byte >> 3, bit & 7) and int32 length; the slot, zero after the length.
 *                  A code longer than slot bytes is stored as bits.  slot: a multiple of 4 of at least S*S/8.
 *                  workspace: ape_mask_pack_workspace_bytes(topk, Hp, Wp, max output width, S, slot), 256-byte aligned;
 *                  rows and out 4-byte aligned.
 */
int64_t ape_mask_pack_workspace_bytes(int topk, int Hp, int Wp, int max_w, int S, int slot);
int ape_mask_pack(const void *logits, const float *rows, const int *out_hw, void *workspace, uint8_t *out, int B, int topk, int Q,
                  int h, int w, int Hp, int Wp, int S, int slot, int dtype, void *stream);

/*
 * Semantic label maps without the [N,H,W] class-score maps.  Replaces, for one image, the semantic tail of
 * deformable_detr_segm_vl.py:875-918 (`_postprocess_semantic`: bilinear upsample of the kept mask logits to the padded size,
 * sigmoid, einsum("qc,qhw->chw") with the class scores) + detectron2 sem_seg_postprocess (crop to the image, bilinear resize
 * to the output size) + the evaluator's argmax over classes.  Both resizes are linear, so the class contraction runs at the
 * output resolution on operands resampled once:
 *   ape_semseg_resample     A [rows*out_w, lda] (a_dtype fp16 / bf16) for output rows [row0, row0+rows):
 *                           A[p, k] = resize2(crop(sigmoid(resize1(logits[index[k]]))))(p), k < K; columns K..Kp-1 zero,
 *                           Kp = K rounded up to 8 <= lda, lda a multiple of 8, A 16-byte aligned.  logits [Q,h,w]
 *                           (logit_dtype fp32 / fp16 / bf16), index [K] int64; resize1 h x w -> Hp x Wp, crop img_h x img_w,
 *                           resize2 -> out_h x out_w, both upsample_bilinear2d (align_corners=False) arithmetic in fp32.
 *   ape_semseg_keys_init    keys [n] <- the key of (value, column): value = -INFINITY for "no class yet", or the constant
 *                           class 0 takes (stuff_prob_thing, deformable_detr_segm_vl.py:655-664) with the GEMM started at class 1.
 *   ape_gemm_tn_argmax      keys[m] = max(keys[m], max_n key((A W^T)[m, n], col_base + n)), A [M,K], W [N,K] (classes x
 *                           padded queries) 16-bit of one dtype, same alignment rules as ape_gemm_tn; nothing else is stored.
 *   ape_semseg_keys_decode  label [n] int64 = the class of keys[i], score [n] fp32 = its value.
 * key(v, c) = (order-preserving bits of v) << 32 | (0xFFFFFFFF - c): ties resolve to the lowest class, as torch.argmax.
 */
int ape_semseg_resample(const void *logits, const int64_t *index, void *A, int64_t lda, int K, int h, int w, int Hp, int Wp,
                        int img_h, int img_w, int out_h, int out_w, int row0, int rows, int logit_dtype, int a_dtype, void *stream);
int ape_semseg_keys_init(uint64_t *keys, int64_t n, float value, int column, void *stream);
int ape_gemm_tn_argmax(const void *A, int64_t lda, const void *W, int64_t ldw, uint64_t *keys, int M, int N, int K, int col_base,
                       int in_dtype, void *stream);
int ape_semseg_keys_decode(const uint64_t *keys, int64_t n, int64_t *label, float *score, void *stream);

/*
 * A label map as cocoapi run-length codes, one per label present, without a mask per label.  Replaces detectron2's
 * SemSegEvaluator.process -> encode_json_sem_seg: np.unique, then for each label mask_util.encode(np.array((L == c)[:, :, None],
 * order="F")).  label int64 [H,W] row-major, H*W <= 2^27, labels in [0, 65535].  A "codes body" is P x (int32 label, int32
 * character offset from the first character, int32 character length) in ascending label order, then the rleToString
 * characters of every label.  Deterministic: the output does not depend on the order of atomics.
 *   ape_label_rle_sizes            sizes (device int32 [3]) <- P labels present, m boundaries (t >= 1 with L(t) != L(t-1) in
 *                                  column-major order t = x*H + y), number of labels outside [0, 65535] (0 or 1).  workspace:
 *                                  ape_label_rle_workspace_bytes(W, 0, 0).
 *   ape_label_rle                  out <- the codes body; sizes is a HOST copy of what ape_label_rle_sizes wrote for this map
 *                                  (labels outside [0, 65535]: APE_ERR_INVALID_ARG).  out holds ape_label_rle_out_bytes(P, m);
 *                                  out_info (device int32 [3]) <- 1, bytes written, P.  workspace:
 *                                  ape_label_rle_workspace_bytes(W, P, 2m+1) (P x W int32 and about 3 int32 per boundary).
 *   ape_label_rle_pack             one image's semantic slot of `slot` bytes with no host read-back (CUDA-graph capturable):
 *                                  labels in [0, num_labels).  The slot is zeroed, then holds the codes body (kind 1) when it
 *                                  fits, else the map as uint16 [H,W] row-major (kind 2) when 2*H*W <= slot, else nothing
 *                                  (kind 3).  A map whose boundaries alone rule out codes that fit skips their passes.
 *                                  out_info (device int32 [3]) <- kind, bytes used (kind 3: the bytes the smaller form needs, a
 *                                  lower bound for codes; 0 for labels outside [0, num_labels)), P.  slot a multiple of 4,
 *                                  >= 16; workspace: ape_label_rle_pack_workspace_bytes(W, num_labels, slot).
 * Workspaces 256-byte aligned, out 4-byte aligned.
 */
int64_t ape_label_rle_workspace_bytes(int W, int P, int64_t events);
int64_t ape_label_rle_out_bytes(int P, int m);
int ape_label_rle_sizes(const int64_t *label, int H, int W, void *workspace, int *sizes, void *stream);
int ape_label_rle(const int64_t *label, int H, int W, const int *sizes, void *workspace, uint8_t *out, int *out_info, void *stream);
int64_t ape_label_rle_pack_workspace_bytes(int W, int num_labels, int slot);
int ape_label_rle_pack(const int64_t *label, int H, int W, int num_labels, int slot, void *workspace, uint8_t *out, int *out_info,
                       void *stream);

/*
 * Panoptic merge without the [K,H,W] mask stacks.  Replaces, for one image, the per-pixel part of
 * deformable_detr_segm_vl.py:919-998 (`_postprocess_panoptic`, after the upsample of :569 and detectron2 sem_seg_postprocess):
 *   v_k = resize2(crop(resize1(logits[index[k]]))), p_k = sigmoid(v_k), id = the first k maximising scores[k] * p_k
 * with resize1 h x w -> Hp x Wp, crop img_h x img_w, resize2 -> out_h x out_w, both upsample_bilinear2d (align_corners=False)
 * arithmetic in fp32, the sigmoid after both.  logits [Q,h,w] (logit_dtype fp32 / fp16 / bf16), index [K] int64 in [0, Q),
 * scores [K] fp32; a query whose score is -INFINITY takes no part (it never wins and its counts stay 0).
 *   ids    [out_h, out_w] int32: id where p_id >= prob, else -1 (also where no query takes part).
 *   counts [3, K] int32: mask_area[k] = #{pixels whose id is k}, inter_area[k] = #{... and p_k >= prob},
 *          original_area[k] = #{pixels with p_k >= prob}.  Zeroed by the call itself.
 * 0 <= K <= APE_PANOPTIC_MAX_K (per-CTA shared-memory histograms of 3*K int32).  Two kernels, no allocation, no
 * synchronisation: capturable in a CUDA graph.
 */
#define APE_PANOPTIC_MAX_K 4096
int ape_panoptic_winners(const void *logits, const int64_t *index, const float *scores, int *ids, int *counts, int K, int h, int w,
                         int Hp, int Wp, int img_h, int img_w, int out_h, int out_w, float prob, int logit_dtype, void *stream);

/*
 * One image's panoptic slot from what ape_panoptic_winners wrote (ids [out_h, out_w], counts [3, K]) and classes [K] int32, with
 * no host read-back.  Replaces the segment bookkeeping and painting of deformable_detr_segm_vl.py:958-995: for k in order, query k
 * takes part iff mask_area, original_area and inter_area are > 0 and !((double)mask_area / original_area < overlap_threshold)
 * (and 0 <= classes[k] < num_classes); isthing = classes[k] < num_things; a stuff class that already has a segment maps to it,
 * otherwise the next id (1, 2, ...) is assigned; category_id = classes[k] - num_things + 1 for stuff when stuff_first, else
 * classes[k].  Queries whose score was -inf have all-zero counts and take no part.  The slot (slot_bytes, a multiple of 4, at
 * least 32 + 12 K + 2 out_h out_w; 4-byte aligned) is written completely:
 *   int32 [8]          1, segments S, out_h, out_w, K, bytes used (32 + 12 K + 2 out_h out_w), 0, 0
 *   int32 [K][3]       (id, isthing, category_id) of segments 1..S in id order; rows >= S zero
 *   uint16 [out_h, out_w]  segment id of each pixel (0 = none), row-major; then zeros to the slot's end
 * workspace (256-byte aligned): ape_panoptic_pack_workspace_bytes(K, num_classes); ids 8-byte aligned.  Two kernels, no allocation,
 * no synchronisation: capturable in a CUDA graph.  Deterministic.
 */
int64_t ape_panoptic_pack_workspace_bytes(int K, int num_classes);
int ape_panoptic_pack(const int *ids, const int *counts, const int *classes, int K, int num_classes, int num_things, int stuff_first,
                      double overlap_threshold, int out_h, int out_w, void *workspace, uint8_t *slot, int slot_bytes, void *stream);

/*
 * Per-image-size geometry of the deformable transformer for a padded batch (DeformableDetrTransformerVL.geometry and the sine
 * position embedding, deformable_transformer_vl.py:435-477 and the anchor part of :321-353), built on the device from the image
 * sizes so that one CUDA graph serves every size inside the padded shape.
 *   sizes         int32 [B, 2] (h, w) in device memory, clamped to [1, Hp] x [1, Wp] (values only, never addresses)
 *   level_hw      HOST int [L, 2], 1 <= L <= 8, each level inside Hp x Wp; S = sum h_l w_l tokens, levels flattened in order
 *   dim_t         fp32 [E / 2]: PositionEmbeddingSine's temperature ** (2 * (k // 2) / (E / 2)), computed by the caller; its
 *                 entries come in equal pairs (dim_t[2m] == dim_t[2m + 1]) and the kernel reads the first of each
 *   level_embeds  fp32 [L, E]
 * Level l's padding mask is F.interpolate(mode="nearest") of the pixel mask: row i is valid iff
 * min(floor(i * ((float)Hp / h_l)), Hp - 1) < h (columns likewise).  Outputs (written completely):
 *   mask_flatten      bool [B, S]             padded tokens
 *   pos_lvl           pos_dtype [B, S, E]     (pos + level_embeds[l]) rounded to pos_dtype (fp32 / fp16 / bf16)
 *   pos_flatten       fp32 [B, S, E] or NULL  pos: channels [0, E/2) from the row sums y, [E/2, E) from the column sums x, each
 *                                             as (sin, cos) of ((c + offset) / (last + eps) * scale) / dim_t[k] (c alone when
 *                                             normalize is 0), precise sinf / cosf
 *   valid_ratios      fp32 [B, L, 2]          (valid columns * (1 / w_l), valid rows * (1 / h_l)): torch divides a tensor by a
 *                                             scalar as a product with the scalar's fp32 reciprocal
 *   reference_points  fp32 [B, S, L, 2]       ((j + 0.5) / (ratio_w * w_l), (i + 0.5) / (ratio_h * h_l)) * the ratios of every level
 *   output_proposals  fp32 [B, S, 4]          log(p / (1 - p)) of ((j + 0.5) / valid_w, (i + 0.5) / valid_h, 0.05 * 2^l, 0.05 * 2^l),
 *                                             inf where padded or any p outside (0.01, 0.99)
 *   proposal_invalid  bool [B, S, 1]          padded or outside (0.01, 0.99)
 * pos_flatten and reference_points 8-byte, output_proposals 16-byte aligned.  One kernel, no allocation, no synchronisation:
 * capturable in a CUDA graph.  Deterministic; every fp32 operation is the torch code's, in its order.
 */
int ape_pad_geometry(const int *sizes, int B, int Hp, int Wp, const int *level_hw, int L, const float *dim_t, const float *level_embeds,
                     int E, float offset, float eps, float scale, int normalize, uint8_t *mask_flatten, void *pos_lvl, int pos_dtype,
                     float *pos_flatten, float *valid_ratios, float *reference_points, float *output_proposals,
                     uint8_t *proposal_invalid, void *stream);

/*
 * In place: x[r, 0:cols] = +0.0 for every row r < rows with mask[r] != 0 (row pitch ld elements; dtype fp32 / fp16 / bf16).  Rows
 * whose mask is 0 are not written, so an all-false mask costs its read alone.  Replaces `value.masked_fill(key_padding_mask[..., None],
 * 0)` of MultiScaleDeformableAttention.forward (ape/layers/multi_scale_deform_attn.py:322-323) on the engine path.  One kernel, no
 * allocation, no synchronisation: capturable in a CUDA graph.
 */
int ape_zero_masked_rows(void *x, int64_t ld, const uint8_t *mask, int64_t rows, int cols, int dtype, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* APE_B200_H_ */
