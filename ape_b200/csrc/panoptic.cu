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
//
// ape_panoptic_pack turns those into one image's panoptic slot of forward_packed without reading anything back to the host
// (the reference's loop over the kept queries, deformable_detr_segm_vl.py:958-995, and the painting of the map):
//   panoptic_segments_kernel  one CTA: which queries make a segment, their ids, the lookup table query -> segment id, the slot's
//                             header and segment table
//   panoptic_paint_kernel     map [out_h, out_w] uint16 = lut[ids] (0 where ids is -1) into the slot, then zeros to its end
#include <algorithm>
#include <climits>

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
                                                                    int out_w, float prob, int tiles_x, int tiles,
                                                                    const int *__restrict__ dims, int Hp, int Wp) {
  extern __shared__ int hist[];
  for (int i = threadIdx.x; i < 3 * K; i += kThreads) hist[i] = 0;
  pdl_prologue();
  if (dims) {  // ape_panoptic_winners_dev: sizes from the device, the output within the out_h x out_w capacity
    const DevSizes d = dev_sizes(dims, Hp, Wp, min(out_h, out_w));
    img_h = d.ih;
    img_w = d.iw;
    out_h = d.oh;
    out_w = d.ow;
    s2h = __fdiv_rn((float)img_h, (float)out_h);  // the host's IEEE divisions
    s2w = __fdiv_rn((float)img_w, (float)out_w);
    tiles_x = (out_w + kTileW - 1) / kTileW;
    tiles = tiles_x * ((out_h + kTileH - 1) / kTileH);
  }
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
                    int out_w, float prob, int tiles_x, int tiles, const int *dims, int Hp, int Wp) {
  auto kernel = panoptic_winners_kernel<TL>;
  APE_LAUNCH(kernel, grid, kThreads, smem, st, (const TL *)logits, (const long long *)index, scores, ids, counts, K, h, w, s1h, s1w,
             img_h, img_w, s2h, s2w, out_h, out_w, prob, tiles_x, tiles, dims, Hp, Wp);
}

// ---- the panoptic slot ----------------------------------------------------------------------------------------------------
constexpr int kSegThreads = 1024;
constexpr int kSegPer = APE_PANOPTIC_MAX_K / kSegThreads;  // consecutive queries per thread, so that the scan runs in query order
constexpr int kSlotHead = 8;                                // int32 header words

// The reference's loop, for k in order: a query with all three areas > 0 and mask_area / original_area not below the threshold
// takes part; a thing query, or the first such query of its stuff class, opens the next segment id; a later query of a stuff class
// joins the segment of that class's first one.  In parallel: the first query of each stuff class is a minimum (atomicMin, so it
// does not depend on the order of the atomics), the ids a block scan over the openers.
__global__ void __launch_bounds__(kSegThreads) panoptic_segments_kernel(const int *__restrict__ counts, const int *__restrict__ classes,
                                                                        int K, int num_classes, int num_things, int stuff_first,
                                                                        double overlap, int out_h, int out_w, int map_bytes,
                                                                        int *__restrict__ first, int *__restrict__ lut,
                                                                        int *__restrict__ slot, const int *__restrict__ dims) {
  __shared__ int s_id[APE_PANOPTIC_MAX_K];  // segment id of every query that opens one
  __shared__ int s_warp[kSegThreads / 32];
  pdl_prologue();
  if (dims) {  // ape_panoptic_pack_dev: the output size from the device, within the out_h x out_w capacity
    const DevSizes d = dev_sizes(dims, 1, 1, min(out_h, out_w));
    out_h = d.oh;
    out_w = d.ow;
    map_bytes = 2 * out_h * out_w;
  }
  for (int c = threadIdx.x; c < num_classes; c += kSegThreads) first[c] = INT_MAX;
  __syncthreads();
  const int k0 = threadIdx.x * kSegPer;
  int cls[kSegPer];
  bool valid[kSegPer];
#pragma unroll
  for (int j = 0; j < kSegPer; ++j) {
    const int k = k0 + j;
    valid[j] = false;
    cls[j] = 0;
    if (k < K) {
      const int area = counts[k], inter = counts[K + k], orig = counts[2 * K + k], c = classes[k];
      // the reference skips a query iff area / orig < threshold, the quotient of two ints correctly rounded to a double: the
      // same IEEE division here (a NaN threshold then skips nothing, as there); a class outside [0, num_classes) takes no part
      valid[j] = area > 0 && orig > 0 && inter > 0 && !((double)area / (double)orig < overlap) && c >= 0 && c < num_classes;
      cls[j] = c;
      if (valid[j] && c >= num_things) atomicMin(first + c, k);
    }
  }
  __syncthreads();
  int opens = 0;
  bool open[kSegPer];
#pragma unroll
  for (int j = 0; j < kSegPer; ++j) {
    open[j] = valid[j] && (cls[j] < num_things || __ldcg(first + cls[j]) == k0 + j);
    opens += open[j];
  }
  // exclusive scan of the openers over the CTA (32 warps)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = opens;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int before = 0, segments = 0;
#pragma unroll 8
  for (int i = 0; i < kSegThreads / 32; ++i) {
    const int v = s_warp[i];
    before += i < warp ? v : 0;
    segments += v;
  }
  int id = before + incl - opens;
#pragma unroll
  for (int j = 0; j < kSegPer; ++j) {
    const int k = k0 + j;
    if (!open[j]) continue;
    s_id[k] = ++id;
    const bool thing = cls[j] < num_things;
    int *row = slot + kSlotHead + 3 * (id - 1);
    row[0] = id;
    row[1] = thing ? 1 : 0;
    row[2] = thing || !stuff_first ? cls[j] : cls[j] - num_things + 1;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < kSegPer; ++j) {
    const int k = k0 + j;
    if (k >= K) break;
    lut[k] = open[j] ? s_id[k] : valid[j] ? s_id[__ldcg(first + cls[j])] : 0;  // a repeat takes its class's segment
  }
  for (int i = kSlotHead + 3 * segments + threadIdx.x; i < kSlotHead + 3 * K; i += kSegThreads) slot[i] = 0;  // unused rows
  if (threadIdx.x == 0) {
    slot[0] = 1;
    slot[1] = segments;
    slot[2] = out_h;
    slot[3] = out_w;
    slot[4] = K;
    slot[5] = 4 * kSlotHead + 12 * K + map_bytes;
    slot[6] = 0;
    slot[7] = 0;
  }
}

// lut of the segment ids at two pixels as one little-endian word of two uint16 (0 past the map's end and where ids is -1)
__device__ __forceinline__ uint32_t paint_pair(const int *__restrict__ ids, const int *__restrict__ lut, long long p, long long HW) {
  int a = -1, b = -1;
  if (p + 1 < HW) {
    const int2 v = __ldg(reinterpret_cast<const int2 *>(ids + p));  // p is even, ids 8-byte aligned
    a = v.x;
    b = v.y;
  } else if (p < HW) {
    a = __ldg(ids + p);
  }
  const uint32_t lo = a >= 0 ? (uint32_t)__ldg(lut + a) & 0xffffu : 0u;
  const uint32_t hi = b >= 0 ? (uint32_t)__ldg(lut + b) & 0xffffu : 0u;
  return lo | hi << 16;
}

// map words w = [0, words) of the slot from its map on (word w = pixels 2w, 2w+1): 16-byte stores from the first 16-byte
// boundary, single words before it (head < 4) and after the last whole vector
// dims: HW from the device size row, within the capacity cap x cap
__global__ void __launch_bounds__(256) panoptic_paint_kernel(const int *__restrict__ ids, const int *__restrict__ lut, long long HW,
                                                             uint32_t *__restrict__ map, long long words, int head,
                                                             const int *__restrict__ dims, int cap) {
  pdl_prologue();
  if (dims) {
    const DevSizes d = dev_sizes(dims, 1, 1, cap);
    HW = (long long)d.oh * d.ow;
  }
  const long long vecs = (words - head) / 4, tail = head + 4 * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < vecs; i += (long long)gridDim.x * blockDim.x) {
    const long long w = head + 4 * i;
    uint4 v;
    v.x = paint_pair(ids, lut, 2 * w, HW);
    v.y = paint_pair(ids, lut, 2 * w + 2, HW);
    v.z = paint_pair(ids, lut, 2 * w + 4, HW);
    v.w = paint_pair(ids, lut, 2 * w + 6, HW);
    *reinterpret_cast<uint4 *>(map + w) = v;
  }
  if (blockIdx.x == 0 && threadIdx.x < 8) {
    const long long w = threadIdx.x < 4 ? (long long)threadIdx.x : tail + threadIdx.x - 4;
    if ((threadIdx.x < 4 && w < head) || (threadIdx.x >= 4 && w < words)) map[w] = paint_pair(ids, lut, 2 * w, HW);
  }
}

}  // namespace
}  // namespace ape

using namespace ape;

namespace {
// dims == nullptr: the host sizes; else the device size row, out_h x out_w being the capacity (grid and checks)
int panoptic_winners_run(const void *logits, const int64_t *index, const float *scores, int *ids, int *counts, int K, int h, int w,
                         int Hp, int Wp, int img_h, int img_w, int out_h, int out_w, float prob, int logit_dtype, const int *dims,
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
                     tiles_x, tiles, dims, Hp, Wp)
  if (logit_dtype == APE_DTYPE_F32) APE_PANOPTIC(float);
  else if (logit_dtype == APE_DTYPE_F16) APE_PANOPTIC(__half);
  else APE_PANOPTIC(__nv_bfloat16);
#undef APE_PANOPTIC
  return check_launch("panoptic_winners_kernel");
}
}  // namespace

extern "C" int ape_panoptic_winners(const void *logits, const int64_t *index, const float *scores, int *ids, int *counts, int K, int h,
                                    int w, int Hp, int Wp, int img_h, int img_w, int out_h, int out_w, float prob, int logit_dtype,
                                    void *stream) {
  return panoptic_winners_run(logits, index, scores, ids, counts, K, h, w, Hp, Wp, img_h, img_w, out_h, out_w, prob, logit_dtype,
                              nullptr, stream);
}

extern "C" int ape_panoptic_winners_dev(const void *logits, const int64_t *index, const float *scores, int *ids, int *counts, int K,
                                        int h, int w, int Hp, int Wp, const int *sizes, int cap, float prob, int logit_dtype,
                                        void *stream) {
  if (!sizes) return fail(APE_ERR_NULL_PTR, "panoptic_winners_dev: null sizes");
  if (cap <= 0) return fail(APE_ERR_INVALID_ARG, "panoptic_winners_dev: capacity %d", cap);
  // the host-side image size only has to pass the checks: the kernel reads the real one
  return panoptic_winners_run(logits, index, scores, ids, counts, K, h, w, Hp, Wp, 1, 1, cap, cap, prob, logit_dtype, sizes, stream);
}

namespace {
int64_t pan_align(int64_t n) { return (n + 255) / 256 * 256; }
}  // namespace

// workspace: first valid query per class int32 [num_classes], then the lookup table query -> segment id int32 [K]
extern "C" int64_t ape_panoptic_pack_workspace_bytes(int K, int num_classes) {
  if (K < 0 || K > APE_PANOPTIC_MAX_K || num_classes < 0) return 0;
  return pan_align(4LL * std::max(num_classes, 1)) + pan_align(4LL * std::max(K, 1));
}

namespace {
int panoptic_pack_run(const int *ids, const int *counts, const int *classes, int K, int num_classes, int num_things, int stuff_first,
                      double overlap_threshold, int out_h, int out_w, long long need, void *workspace, uint8_t *slot, int slot_bytes,
                      const int *dims, int cap, void *stream) {
  if (K < 0 || K > APE_PANOPTIC_MAX_K)
    return fail(APE_ERR_INVALID_ARG, "panoptic_pack: K=%d outside [0, %d]", K, APE_PANOPTIC_MAX_K);
  if (num_classes < 0 || num_things < 0) return fail(APE_ERR_INVALID_ARG, "panoptic_pack: num_classes %d, num_things %d", num_classes, num_things);
  if (out_h <= 0 || out_w <= 0) return fail(APE_ERR_INVALID_ARG, "panoptic_pack: bad output size %dx%d", out_h, out_w);
  const long long HW = (long long)out_h * out_w;
  if (slot_bytes < 0 || slot_bytes % 4 != 0 || need > slot_bytes)
    return fail(APE_ERR_INVALID_ARG, "panoptic_pack: slot of %d bytes (a multiple of 4 of at least %lld for K=%d and %dx%d)", slot_bytes,
                need, K, out_h, out_w);
  if (!ids || !workspace || !slot || (K > 0 && (!counts || !classes))) return fail(APE_ERR_NULL_PTR, "panoptic_pack: null pointer");
  if ((reinterpret_cast<uintptr_t>(workspace) & 255) || (reinterpret_cast<uintptr_t>(slot) & 3) || (reinterpret_cast<uintptr_t>(ids) & 7))
    return fail(APE_ERR_INVALID_ARG, "panoptic_pack: workspace must be 256-byte, slot 4-byte and ids 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  int *first = reinterpret_cast<int *>(workspace);
  int *lut = reinterpret_cast<int *>(reinterpret_cast<char *>(workspace) + pan_align(4LL * std::max(num_classes, 1)));
  APE_LAUNCH(panoptic_segments_kernel, 1, kSegThreads, 0, st, counts, classes, K, num_classes, num_things, stuff_first ? 1 : 0,
             overlap_threshold, out_h, out_w, (int)std::min(2 * HW, 0x7fffffffLL), first, lut, reinterpret_cast<int *>(slot), dims);
  int rc = check_launch("panoptic_segments_kernel");
  if (rc != APE_OK) return rc;
  uint8_t *map = slot + 4LL * kSlotHead + 12LL * K;
  const long long words = (slot_bytes - (map - slot)) / 4;
  const int head = (int)std::min<long long>(((16 - (reinterpret_cast<uintptr_t>(map) & 15)) & 15) / 4, words);
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long blocks = ((words - head) / 4 + 255) / 256;
  const int grid = (int)std::max(1LL, std::min(blocks, 8LL * std::max(sms, 1)));
  APE_LAUNCH(panoptic_paint_kernel, grid, 256, 0, st, ids, (const int *)lut, HW, reinterpret_cast<uint32_t *>(map), words, head, dims, cap);
  return check_launch("panoptic_paint_kernel");
}
}  // namespace

extern "C" int ape_panoptic_pack(const int *ids, const int *counts, const int *classes, int K, int num_classes, int num_things,
                                 int stuff_first, double overlap_threshold, int out_h, int out_w, void *workspace, uint8_t *slot,
                                 int slot_bytes, void *stream) {
  const long long need = 4LL * kSlotHead + 12LL * K + 2LL * out_h * out_w;
  return panoptic_pack_run(ids, counts, classes, K, num_classes, num_things, stuff_first, overlap_threshold, out_h, out_w, need, workspace,
                           slot, slot_bytes, nullptr, 0, stream);
}

extern "C" int ape_panoptic_pack_dev(const int *ids, const int *counts, const int *classes, int K, int num_classes, int num_things,
                                     int stuff_first, double overlap_threshold, const int *sizes, int cap, void *workspace, uint8_t *slot,
                                     int slot_bytes, void *stream) {
  if (!sizes) return fail(APE_ERR_NULL_PTR, "panoptic_pack_dev: null sizes");
  if (cap <= 0 || (long long)cap * cap > 0x3fffffffLL) return fail(APE_ERR_INVALID_ARG, "panoptic_pack_dev: capacity %d", cap);
  // the slot must hold the header and the table; a map larger than the rest of the slot is cut at the slot's end
  return panoptic_pack_run(ids, counts, classes, K, num_classes, num_things, stuff_first, overlap_threshold, cap, cap,
                           4LL * kSlotHead + 12LL * K, workspace, slot, slot_bytes, sizes, cap, stream);
}
