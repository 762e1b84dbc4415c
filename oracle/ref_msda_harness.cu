/*
 * oracle/ref_msda_harness.cu — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Thin extern "C" launcher around the REFERENCE's own forward kernel, compiled from the
 * reference sources where they lie (this file only #includes
 * /root/reference/ape/layers/csrc/MsDeformAttn/ms_deform_im2col_cuda.cuh; no reference
 * source is copied into this repository).  Built by oracle/Makefile into
 * oracle/_ref/libref_msda.so (git-ignored; travels to the GPU box) and used there as
 *   (1) a second oracle for the CUDA parity tests (tests/test_msda_gpu.py), and
 *   (2) the "kernel to beat": the reference's 2020-era SIMT kernel recompiled for sm_90a,
 *       timed beside ours by bench.py on identical tensors.
 * The launcher plays the role of ms_deform_attn_cuda_forward
 * (ape/layers/csrc/MsDeformAttn/ms_deform_attn_cuda.cu:21-81) minus the ATen plumbing:
 * one call to ms_deformable_im2col_cuda<scalar_t> per batch chunk of `im2col_step`.
 */
#include REF_IM2COL_HEADER

#include <cuda_fp16.h>

template <typename T>
static int run(cudaStream_t st, const void *value, const int64_t *shapes, const int64_t *starts,
               const void *loc, const void *attn, void *out, int B, int S, int H, int D, int L, int Q,
               int P, int im2col_step) {
  const int step = B < im2col_step ? B : im2col_step;
  if (step <= 0 || B % step != 0) return -1;
  const size_t per_value = (size_t)S * H * D, per_loc = (size_t)Q * H * L * P * 2,
               per_attn = (size_t)Q * H * L * P, per_out = (size_t)Q * H * D;
  for (int n = 0; n < B / step; ++n) {
    ms_deformable_im2col_cuda<T>(st, (const T *)value + n * step * per_value, shapes, starts,
                                 (const T *)loc + n * step * per_loc,
                                 (const T *)attn + n * step * per_attn, step, S, H, D, L, Q, P,
                                 (T *)out + n * step * per_out);
  }
  return (int)cudaGetLastError();
}

extern "C" int ref_msda_forward(const void *value, const int64_t *shapes, const int64_t *starts,
                                const void *loc, const void *attn, void *out, int B, int S, int H,
                                int D, int L, int Q, int P, int dtype, int im2col_step, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0) return run<float>(st, value, shapes, starts, loc, attn, out, B, S, H, D, L, Q, P, im2col_step);
  if (dtype == 1) return run<c10::Half>(st, value, shapes, starts, loc, attn, out, B, S, H, D, L, Q, P, im2col_step);
  return -2; /* the reference has no bf16 path (AT_DISPATCH_FLOATING_TYPES_AND_HALF) */
}
