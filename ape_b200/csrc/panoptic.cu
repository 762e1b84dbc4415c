// panoptic.cu — per-pixel winners and segment areas of the panoptic merge without the [K, H, W] mask stacks
// (DeformableDETRSegmVL._panoptic on the engine path, modeling/postprocess.py postprocess_panoptic_winners).
//
// The reference's panoptic branch (ape/modeling/ape_deta/deformable_detr_segm_vl.py:569 and :919-998 `_postprocess_panoptic`,
// with detectron2 sem_seg_postprocess) forms, for the K kept queries of one image,
//   v_k  = resize2(crop(resize1(logit_k)))          resize1: h x w -> padded Hp x Wp; crop img_h x img_w; resize2 -> out_h x out_w
//   p_k  = sigmoid(v_k)                              [K, out_h, out_w] fp32, several times over (1 to 4 GB each at K = 300)
//   id   = argmax_k score_k * p_k                    first maximum, as torch.argmax
// and keeps, besides the map, only three areas per query (mask, intersection with p >= prob, p >= prob).  One thread here
// owns one output pixel and walks the K queries: it resamples v_k from the logits (4 padded-grid points x 4 logit taps, the
// L1 serves the overlap between neighbouring pixels), keeps the running first maximum, and counts into per-CTA shared
// histograms, which are added to the global counts with one atomic per non-zero bin when the CTA ends.
//   panoptic_zero_kernel     counts <- 0 (a kernel, so that the pair is one capturable sequence on the stream)
//   panoptic_winners_kernel  ids [out_h, out_w] int32, counts [3, K] int32
#include <algorithm>

#include "common.cuh"
#include "resize.cuh"

namespace ape {
namespace {

constexpr int kTileW = 32, kTileH = 8;  // one warp = 32 adjacent pixels of a row; one CTA = 8 rows
constexpr int kThreads = kTileW * kTileH;

__global__ void __launch_bounds__(256) panoptic_zero_kernel(int *__restrict__ counts, int n) {
  pdl_prologue();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) counts[i] = 0;
}

// hist [3][K] in shared memory: 0 mask_area (pixels the query wins), 1 inter_area (... where its p >= prob), 2 original_area
// (pixels where its p >= prob).  Queries whose score is -inf take no part: they never win and are not counted.
template <typename TL>
__global__ void __launch_bounds__(kThreads) panoptic_winners_kernel(const TL *__restrict__ logits, const long long *__restrict__ index,
                                                                    const float *__restrict__ scores, int *__restrict__ ids,
                                                                    int *__restrict__ counts, int K, int h, int w, float s1h,
                                                                    float s1w, int img_h, int img_w, float s2h, float s2w, int out_h,
                                                                    int out_w, float prob, int tiles_x, int tiles) {
  extern __shared__ int hist[];
  for (int i = threadIdx.x; i < 3 * K; i += kThreads) hist[i] = 0;
  pdl_prologue();
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int y = (t / tiles_x) * kTileH + (int)(threadIdx.x >> 5);
    if (y >= out_h) continue;  // warp-uniform: the ballots below see all 32 lanes
    const int x = (t % tiles_x) * kTileW + lane;
    const bool valid = x < out_w;
    const Lerp ry = lerp_at(s2h, y, img_h), rx = lerp_at(s2w, min(x, out_w - 1), img_w);  // resize2 over the crop
    const Lerp ay0 = lerp_at(s1h, ry.i0, h), ay1 = lerp_at(s1h, ry.i1, h);  // resize1 at the two padded rows it reads
    const Lerp bx0 = lerp_at(s1w, rx.i0, w), bx1 = lerp_at(s1w, rx.i1, w);  // ... and the two padded columns
    float best = -INFINITY, best_p = 0.f;
    int id = -1;
    for (int k = 0; k < K; ++k) {
      const float score = __ldg(scores + k);
      if (score == -INFINITY) continue;  // uniform across the CTA
      const TL *plane = logits + (size_t)__ldg(index + k) * h * w;
      const float m00 = up_value(plane, w, ay0, bx0), m01 = up_value(plane, w, ay0, bx1);
      const float m10 = up_value(plane, w, ay1, bx0), m11 = up_value(plane, w, ay1, bx1);
      const float v = ry.l0 * (rx.l0 * m00 + rx.l1 * m01) + ry.l1 * (rx.l0 * m10 + rx.l1 * m11);
      const float p = 1.f / (1.f + expf(-v));
      const float s = score * p;
      if (s > best) {  // strict: the first maximum wins
        best = s;
        best_p = p;
        id = k;
      }
      const unsigned hit = __ballot_sync(0xffffffffu, valid && p >= prob);
      if (lane == 0 && hit) atomicAdd(&hist[2 * K + k], __popc(hit));
    }
    if (valid) {
      const bool solid = id >= 0 && best_p >= prob;
      ids[(size_t)y * out_w + x] = solid ? id : -1;
      if (id >= 0) {
        atomicAdd(&hist[id], 1);
        if (solid) atomicAdd(&hist[K + id], 1);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * K; i += kThreads)
    if (hist[i]) atomicAdd(counts + i, hist[i]);
}

template <typename TL>
void launch_winners(int grid, size_t smem, cudaStream_t st, const void *logits, const int64_t *index, const float *scores, int *ids,
                    int *counts, int K, int h, int w, float s1h, float s1w, int img_h, int img_w, float s2h, float s2w, int out_h,
                    int out_w, float prob, int tiles_x, int tiles) {
  auto kernel = panoptic_winners_kernel<TL>;
  APE_LAUNCH(kernel, grid, kThreads, smem, st, (const TL *)logits, (const long long *)index, scores, ids, counts, K, h, w, s1h, s1w,
             img_h, img_w, s2h, s2w, out_h, out_w, prob, tiles_x, tiles);
}

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int ape_panoptic_winners(const void *logits, const int64_t *index, const float *scores, int *ids, int *counts, int K, int h,
                                    int w, int Hp, int Wp, int img_h, int img_w, int out_h, int out_w, float prob, int logit_dtype,
                                    void *stream) {
  if (logit_dtype != APE_DTYPE_F32 && logit_dtype != APE_DTYPE_F16 && logit_dtype != APE_DTYPE_BF16)
    return fail(APE_ERR_INVALID_ARG, "panoptic_winners: logit dtype %d", logit_dtype);
  if (K < 0 || K > APE_PANOPTIC_MAX_K)
    return fail(APE_ERR_INVALID_ARG, "panoptic_winners: K=%d outside [0, %d] (the per-CTA shared histograms)", K, APE_PANOPTIC_MAX_K);
  if (h <= 0 || w <= 0 || Hp <= 0 || Wp <= 0 || img_h <= 0 || img_w <= 0 || img_h > Hp || img_w > Wp || out_h <= 0 || out_w <= 0 ||
      (long long)out_h * out_w > 0x7fffffffLL)
    return fail(APE_ERR_INVALID_ARG, "panoptic_winners: bad geometry logits %dx%d, padded %dx%d, image %dx%d, output %dx%d", h, w, Hp,
                Wp, img_h, img_w, out_h, out_w);
  if (!ids || (K > 0 && (!logits || !index || !scores || !counts))) return fail(APE_ERR_NULL_PTR, "panoptic_winners: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (K > 0) {
    APE_LAUNCH(panoptic_zero_kernel, std::min((3 * K + 255) / 256, 64), 256, 0, st, counts, 3 * K);
    const int rc = check_launch("panoptic_zero_kernel");
    if (rc != APE_OK) return rc;
  }
  const float s1h = (float)h / (float)Hp, s1w = (float)w / (float)Wp;  // area_pixel_compute_scale
  const float s2h = (float)img_h / (float)out_h, s2w = (float)img_w / (float)out_w;
  const int tiles_x = (out_w + kTileW - 1) / kTileW;
  const int tiles = tiles_x * ((out_h + kTileH - 1) / kTileH);
  // a few waves of 8 resident CTAs per SM: enough CTAs to balance the tiles, few enough that the histogram flushes stay small
  const int grid = std::max(1, std::min(tiles, 32 * std::max(sms, 1)));
  const size_t smem = (size_t)3 * K * sizeof(int);
#define APE_PANOPTIC(TL) \
  launch_winners<TL>(grid, smem, st, logits, index, scores, ids, counts, K, h, w, s1h, s1w, img_h, img_w, s2h, s2w, out_h, out_w, prob, \
                     tiles_x, tiles)
  if (logit_dtype == APE_DTYPE_F32) APE_PANOPTIC(float);
  else if (logit_dtype == APE_DTYPE_F16) APE_PANOPTIC(__half);
  else APE_PANOPTIC(__nv_bfloat16);
#undef APE_PANOPTIC
  return check_launch("panoptic_winners_kernel");
}
