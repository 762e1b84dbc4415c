// mask_post.cu — instance-mask post-processing of the detections that survive the final selection
// (DeformableDETRSegmVL.forward, ape/modeling/ape_deta/deformable_detr_segm_vl.py:569-603 and _postprocess_instance ->
// detectron2 detector_postprocess):
//
//   mask_pred = F.interpolate(mask_pred, size=padded image, mode="bilinear", align_corners=False)     :569-572 (all 900 queries)
//   box_mask  = mask_pred[filter_inds].sigmoid() > 0.5                                                  :590-598
//   box_mask  = BitMasks(box_mask).crop_and_resize(pred_boxes, 128)        ROIAlign(128, scale 1, ratio 0, aligned) >= 0.5
//   pred_masks = paste_masks_in_image(box_mask, rescaled boxes, (H_out, W_out), 0.5)     bilinear grid_sample >= 0.5
//
// The reference materialises [900, 1024, 1024] fp32 (3.8 GB) for the first line alone; the library formulation used here
// in round 1 (kept queries only) still wrote the upsampled fp32 maps, their sigmoid, the comparison, a float copy for
// roi_align and, for the paste, an [N, H, W, 2] sampling grid.  Three kernels replace all of it:
//
//   mask_binarize_kernel   upsampled logit > 0 for the kept queries only, ONE BIT per pixel ([K, Hp, Wp/32] words; a warp
//                          ballots a word), never the fp32 maps.  Bilinear arithmetic = ATen's upsample_bilinear2d
//                          (align_corners=False: src = scale * (dst + 0.5) - 0.5 clamped at 0, fp32).
//   mask_roialign_kernel   torchvision's roi_align arithmetic (aligned=True, adaptive sampling grid ceil(roi / 128)) over
//                          the bit masks, thresholded at 0.5 -> [K, 128, 128] bytes.
//   mask_paste_kernel      detectron2's _do_paste_mask (grid_sample bilinear, zeros padding, align_corners=False) of a
//                          128 x 128 mask into its box, thresholded -> bool [N, H_out, W_out]; four pixels per thread, the
//                          sampling grid exists only in registers.
// sigmoid(x) > 0.5 is evaluated as x > 0 (identical except for |x| < 6e-8, where fp32 sigmoid rounds to 0.5 exactly).
#include "common.cuh"
#include "rle.cuh"

namespace ape {
namespace {

template <typename T>
__device__ __forceinline__ float ldf(const T *p) {
  return Elem<T>::to_f(__ldg(p));
}

// bits[k][Y][X / 32] bit (X % 32) = bilinear_upsample(logits[index[k]])(Y, X) > 0
// SKIP (the packed path, mask_pack_* below): slot k does nothing unless live[k].  The extra parameter comes last so that the
// other parameters keep their places and the SKIP = false kernels compile to what they were before it existed.
template <typename T, bool SKIP>
__global__ void __launch_bounds__(256) mask_binarize_kernel(const T *__restrict__ logits, const long long *__restrict__ index,
                                                            uint32_t *__restrict__ bits, int h, int w, int Hp, int Wp,
                                                            float scale_h, float scale_w, const int *__restrict__ live) {
  pdl_prologue();
  if (SKIP && !__ldg(live + blockIdx.z)) return;
  const int words = (Wp + 31) >> 5;
  const int lane = threadIdx.x & 31;
  const int word = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int Y = blockIdx.y, k = blockIdx.z;
  if (word >= words) return;
  const int X = word * 32 + lane;
  bool on = false;
  if (X < Wp) {
    const T *src = logits + (size_t)__ldg(index + k) * h * w;
    float sy = fmaxf(scale_h * ((float)Y + 0.5f) - 0.5f, 0.f);
    float sx = fmaxf(scale_w * ((float)X + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
    const float ly = sy - (float)y0, lx = sx - (float)x0;
    const float hy = 1.f - ly, hx = 1.f - lx;
    const float v = hy * (hx * ldf(src + (size_t)y0 * w + x0) + lx * ldf(src + (size_t)y0 * w + x1)) +
                    ly * (hx * ldf(src + (size_t)y1 * w + x0) + lx * ldf(src + (size_t)y1 * w + x1));
    on = v > 0.f;
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, on);
  if (lane == 0) bits[((size_t)k * Hp + Y) * words + word] = bal;
}

__device__ __forceinline__ float bit_at(const uint32_t *m, int words, int y, int x) {
  return (float)((__ldg(m + (size_t)y * words + (x >> 5)) >> (x & 31)) & 1u);
}

// torchvision roi_align (aligned = true, spatial_scale 1, sampling_ratio 0) of the k-th bit mask over box k, >= 0.5
template <bool SKIP>
__global__ void __launch_bounds__(256) mask_roialign_kernel(const uint32_t *__restrict__ bits, const float *__restrict__ boxes,
                                                            uint8_t *__restrict__ out, int Hp, int Wp, int S,
                                                            const int *__restrict__ live) {
  pdl_prologue();
  if (SKIP && !__ldg(live + blockIdx.y)) return;
  const int k = blockIdx.y;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * S) return;
  const int ph = idx / S, pw = idx - ph * S;
  const int words = (Wp + 31) >> 5;
  const uint32_t *m = bits + (size_t)k * Hp * words;
  const float4 b = __ldg(reinterpret_cast<const float4 *>(boxes) + k);
  const float roi_start_w = b.x - 0.5f, roi_start_h = b.y - 0.5f;
  const float roi_width = (b.z - 0.5f) - roi_start_w, roi_height = (b.w - 0.5f) - roi_start_h;
  const float bin_h = roi_height / (float)S, bin_w = roi_width / (float)S;
  const int grid_h = (int)ceilf(roi_height / (float)S), grid_w = (int)ceilf(roi_width / (float)S);
  const float count = (float)max(grid_h * grid_w, 1);
  float acc = 0.f;
  for (int iy = 0; iy < grid_h; ++iy) {
    const float yy = roi_start_h + ph * bin_h + ((float)iy + .5f) * bin_h / (float)grid_h;
    for (int ix = 0; ix < grid_w; ++ix) {
      const float xx = roi_start_w + pw * bin_w + ((float)ix + .5f) * bin_w / (float)grid_w;
      float y = yy, x = xx;
      if (y < -1.f || y > (float)Hp || x < -1.f || x > (float)Wp) continue;  // bilinear_interpolate: outside -> 0
      if (y <= 0.f) y = 0.f;
      if (x <= 0.f) x = 0.f;
      int y_low = (int)y, x_low = (int)x, y_high, x_high;
      if (y_low >= Hp - 1) { y_high = y_low = Hp - 1; y = (float)y_low; } else y_high = y_low + 1;
      if (x_low >= Wp - 1) { x_high = x_low = Wp - 1; x = (float)x_low; } else x_high = x_low + 1;
      const float ly = y - (float)y_low, lx = x - (float)x_low, hy = 1.f - ly, hx = 1.f - lx;
      acc += hy * hx * bit_at(m, words, y_low, x_low) + hy * lx * bit_at(m, words, y_low, x_high) +
             ly * hx * bit_at(m, words, y_high, x_low) + ly * lx * bit_at(m, words, y_high, x_high);
    }
  }
  out[(size_t)k * S * S + idx] = (acc / count) >= 0.5f ? 1 : 0;
}

// detectron2 _do_paste_mask for ONE output pixel: grid_sample(mask_n, normalised (x, y) relative to box b, bilinear, zeros padding,
// align_corners = false) >= threshold.  Shared by the dense paste and the run-length kernels, so both see the same booleans.
__device__ __forceinline__ bool paste_px(const uint8_t *__restrict__ m, const float4 &b, int S, int y, int x, float threshold) {
  const float gy = ((float)y + 0.5f - b.y) / (b.w - b.y) * 2.f - 1.f;
  const float iy = ((gy + 1.f) * (float)S - 1.f) / 2.f;  // grid_sampler_unnormalize, align_corners = false
  const float fy = floorf(iy);
  const int y_n = (int)fy, y_s = y_n + 1;
  const float wy_s = iy - fy, wy_n = (fy + 1.f) - iy;  // (iy - iy_nw), (iy_se - iy) as ATen's grid_sampler
  const float gx = ((float)x + 0.5f - b.x) / (b.z - b.x) * 2.f - 1.f;
  const float ixf = ((gx + 1.f) * (float)S - 1.f) / 2.f;
  const float fx = floorf(ixf);
  const int x_w = (int)fx, x_e = x_w + 1;
  const float wx_e = ixf - fx, wx_w = (fx + 1.f) - ixf;
  float v = 0.f;
  // isfinite: a degenerate box gives inf / nan coordinates, which grid_sample treats as out of bounds
  if (isfinite(ixf) && isfinite(iy) && x_e >= 0 && x_w < S && y_s >= 0 && y_n < S) {
    const bool wn = y_n >= 0, ws = y_s < S, ww = x_w >= 0, we = x_e < S;
    if (wn && ww) v += (float)__ldg(m + y_n * S + x_w) * (wx_w * wy_n);
    if (wn && we) v += (float)__ldg(m + y_n * S + x_e) * (wx_e * wy_n);
    if (ws && ww) v += (float)__ldg(m + y_s * S + x_w) * (wx_w * wy_s);
    if (ws && we) v += (float)__ldg(m + y_s * S + x_e) * (wx_e * wy_s);
  }
  return v >= threshold;
}

__global__ void __launch_bounds__(256) mask_paste_kernel(const uint8_t *__restrict__ masks, const float *__restrict__ boxes,
                                                         uint8_t *__restrict__ out, int S, int img_h, int img_w, float threshold) {
  pdl_prologue();
  const int n = blockIdx.z, y = blockIdx.y;
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (x4 >= img_w) return;
  const float4 b = __ldg(reinterpret_cast<const float4 *>(boxes) + n);
  const uint8_t *m = masks + (size_t)n * S * S;
  uint8_t r[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) r[i] = paste_px(m, b, S, y, x4 + i, threshold) ? 1 : 0;
  uint8_t *dst = out + ((size_t)n * img_h + y) * img_w + x4;
  if (x4 + 4 <= img_w && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
    *reinterpret_cast<uint32_t *>(dst) = (uint32_t)r[0] | ((uint32_t)r[1] << 8) | ((uint32_t)r[2] << 16) | ((uint32_t)r[3] << 24);
  } else {
    for (int i = 0; i < 4 && x4 + i < img_w; ++i) dst[i] = r[i];
  }
}

// ---- pasted masks as COCO run-length codes, without the dense masks -------------------------------------------------------
// The evaluators turn every pasted mask into cocoapi's RLE right away (mask_util.encode(np.array(mask[:, :, None], order="F")),
// ape/evaluation/{d3,refcoco}_evaluation.py:466-468 and detectron2's instances_to_coco_json for COCO / LVIS): runs of equal
// pixels in COLUMN-major order, the first run counting zeros.  300 pasted 1024^2 masks are 314 MB of booleans to write, copy to
// the host and scan there; their run boundaries are a few hundred kilobytes.  Two passes over (mask, column) CTAs, each pixel
// recomputed from the 128 x 128 mask with the paste arithmetic above:
//   pass 1  number of boundaries in the column (a pixel differs from its predecessor in column-major order; the predecessor of
//           the first pixel of a column is the last pixel of the previous column, of the very first pixel a 0)
//   (exclusive scan of the per-column numbers, on the caller's side)
//   pass 2  the positions j = x * H + y of the boundaries, written in order at the column's offset.
// Run lengths are the differences of consecutive positions (plus the leading and the trailing run).
// SKIP: mask n does nothing unless live[n] (its counts and positions are then left unwritten).
template <bool WRITE, bool SKIP>
__global__ void __launch_bounds__(256) mask_rle_kernel(const uint8_t *__restrict__ masks, const float *__restrict__ boxes, int S,
                                                       int img_h, int img_w, float threshold, int *__restrict__ col_count,
                                                       const long long *__restrict__ col_offset, int *__restrict__ positions,
                                                       const int *__restrict__ live) {
  pdl_prologue();
  if (SKIP && !__ldg(live + blockIdx.y)) return;
  const int n = blockIdx.y, x = blockIdx.x;
  const float4 b = __ldg(reinterpret_cast<const float4 *>(boxes) + n);
  const uint8_t *m = masks + (size_t)n * S * S;
  long long out0 = 0;
  if (WRITE) out0 = col_offset[(size_t)n * img_w + x];
  // value of the pixel before this column's first one in column-major order
  const bool carry_in = x > 0 ? paste_px(m, b, S, img_h - 1, x - 1, threshold) : false;
  {  // columns the box does not reach are all zeros: at most the boundary that ends a run of the previous column
    const float gx = ((float)x + 0.5f - b.x) / (b.z - b.x) * 2.f - 1.f;
    const float ixf = ((gx + 1.f) * (float)S - 1.f) / 2.f;
    const float fx = floorf(ixf);
    if (!(isfinite(ixf) && (int)fx + 1 >= 0 && (int)fx < S)) {
      if (threadIdx.x == 0) {
        if (WRITE) { if (carry_in) positions[out0] = x * img_h; }
        else col_count[(size_t)n * img_w + x] = carry_in ? 1 : 0;
      }
      return;
    }
  }
  __shared__ int s_warp[8];
  __shared__ int s_last[8];
  __shared__ int s_base;
  __shared__ int s_carry;
  if (threadIdx.x == 0) { s_base = 0; s_carry = carry_in ? 1 : 0; }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int y0 = 0; y0 < img_h; y0 += 256) {  // 256 rows per step, boundaries kept in row order
    const int y = y0 + threadIdx.x;
    const bool cur = y < img_h ? paste_px(m, b, S, y, x, threshold) : false;
    if (lane == 31) s_last[warp] = cur ? 1 : 0;
    __syncthreads();
    bool prev = __shfl_up_sync(0xffffffffu, cur ? 1 : 0, 1) != 0;
    if (lane == 0) prev = (warp == 0 ? s_carry : s_last[warp - 1]) != 0;
    const bool flag = y < img_h && cur != prev;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int before = s_base;
    for (int w = 0; w < warp; ++w) before += s_warp[w];
    if (WRITE && flag) positions[out0 + before + __popc(bal & ((1u << lane) - 1))] = x * img_h + y;
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int w = 0; w < 8; ++w) t += s_warp[w];
      s_base += t;
      s_carry = s_last[7];  // the step is full (y0 + 255 < img_h) whenever another step follows
    }
    __syncthreads();
  }
  if (!WRITE && threadIdx.x == 0) col_count[(size_t)n * img_w + x] = s_base;
}

// ---- the kept masks of the packed selection rows as COCO run-length codes in fixed-size slots -----------------------------
// Input: the rows of DeformableDETRSegmVL.forward_packed, [topk, 13] fp32 per image (x1, y1, x2, y2, score, class, query index,
// candidates, kept nk, image h, w, output h, w).  Everything the host path reads back (nk, the run totals) stays on the device:
// every slot gets a CTA, and the slots that hold nothing return after reading a flag.  Output row of a slot (PACK_ROW bytes
// before the SLOT bytes): the 13 fp32 columns, then int32 kind (0 nothing, 1 "counts" characters, 2 the 128 x 128 mask as bits)
// and int32 length, then the slot.
constexpr int PACK_COLS = 13, PACK_HEAD = 4 * PACK_COLS + 8;
constexpr int SLOT_EMPTY = 0, SLOT_CHARS = 1, SLOT_BITS = 2;

// detector_postprocess (detr.py) on one row: box * (output / image size, a double rounded to fp32), clamped to the output,
// kept iff width and height are > 0.  live[k] = k < nk and kept; the crop box is the row's box, the paste box the rescaled one.
__global__ void __launch_bounds__(256) mask_pack_prep_kernel(const float *__restrict__ rows, int topk, long long *__restrict__ index,
                                                             float4 *__restrict__ crop_box, float4 *__restrict__ paste_box,
                                                             int *__restrict__ live) {
  pdl_prologue();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= topk) return;
  const float *r = rows + (size_t)k * PACK_COLS;
  const int nk = (int)r[8];
  int ok = 0;
  if (k < nk) {
    const float h = r[9], w = r[10], oh = r[11], ow = r[12];
    const float sx = (float)((double)ow / (double)w), sy = (float)((double)oh / (double)h);
    const float x1 = fminf(fmaxf(__fmul_rn(r[0], sx), 0.f), ow), y1 = fminf(fmaxf(__fmul_rn(r[1], sy), 0.f), oh);
    const float x2 = fminf(fmaxf(__fmul_rn(r[2], sx), 0.f), ow), y2 = fminf(fmaxf(__fmul_rn(r[3], sy), 0.f), oh);
    ok = __fsub_rn(x2, x1) > 0.f && __fsub_rn(y2, y1) > 0.f;
    index[k] = (long long)r[6];
    crop_box[k] = make_float4(r[0], r[1], r[2], r[3]);
    paste_box[k] = make_float4(x1, y1, x2, y2);
  }
  live[k] = ok;
}

// One CTA per slot: exclusive scan of the slot's column counts -> col_offset (the slot's positions start at n * slot), the
// number of boundaries, and chars[n] = whether they fit: m boundaries make m + 1 counts of at least one character each, so a slot
// with m >= slot boundaries goes straight to bits and the positions workspace stays at slot int32 per slot.
__global__ void __launch_bounds__(256) mask_pack_scan_kernel(const int *__restrict__ col_count, const int *__restrict__ live, int W,
                                                             int slot, long long *__restrict__ col_offset, int *__restrict__ total,
                                                             int *__restrict__ chars) {
  pdl_prologue();
  const int n = blockIdx.x;
  if (!__ldg(live + n)) {
    if (threadIdx.x == 0) chars[n] = 0;
    return;
  }
  __shared__ int s_warp[8];
  long long base = 0;
  for (int x0 = 0; x0 < W; x0 += 256) {
    const int x = x0 + threadIdx.x;
    const int v = x < W ? col_count[(size_t)n * W + x] : 0;
    int sum;
    const int off = block_excl_scan_256(v, s_warp, &sum);
    if (x < W) col_offset[(size_t)n * W + x] = (long long)n * slot + base + off;
    base += sum;
  }
  if (threadIdx.x == 0) {
    total[n] = (int)min(base, 0x7fffffffLL);
    chars[n] = base < slot;
  }
}

// One CTA per slot: the row, the slot word and the slot.  Counts from the boundary positions p (c_i = p_i - p_{i-1}, with
// p_{-1} = 0 and a last boundary at H * W), delta-coded and written at their scanned character offsets; a code longer than the
// slot is replaced by the slot's 128 x 128 mask, bit (y * S + x) at byte >> 3, bit & 7.  Bytes after the length are zero.
__global__ void __launch_bounds__(256) mask_pack_encode_kernel(const float *__restrict__ rows, const int *__restrict__ live,
                                                               const int *__restrict__ chars, const int *__restrict__ total,
                                                               const int *__restrict__ positions, const uint8_t *__restrict__ masks,
                                                               int S, int H, int W, int slot, uint8_t *__restrict__ out) {
  pdl_prologue();
  const int n = blockIdx.x, tid = threadIdx.x;
  uint8_t *dst = out + (size_t)n * (PACK_HEAD + slot);
  uint8_t *body = dst + PACK_HEAD;
  if (tid < PACK_COLS) reinterpret_cast<float *>(dst)[tid] = rows[(size_t)n * PACK_COLS + tid];
  __shared__ int s_warp[8];
  int kind = SLOT_EMPTY, len = 0;
  if (__ldg(live + n)) {
    kind = SLOT_BITS;
    if (__ldg(chars + n)) {
      const int m = total[n] + 1;
      const long long HW = (long long)H * W;
      const int *p = positions + (size_t)n * slot;
      auto P = [&](int j) -> long long { return j < 0 ? 0 : j >= m - 1 ? HW : (long long)p[j]; };
      int base = 0;
      for (int i0 = 0; i0 < m && base <= slot; i0 += 256) {  // base is the same in every thread
        const int i = i0 + tid;
        long long x = 0;
        int nc = 0;
        if (i < m) {
          x = P(i) - P(i - 1);
          if (i > 2) x -= P(i - 2) - P(i - 3);
          nc = rle_chars(x, nullptr, 0);
        }
        int sum;
        const int off = base + block_excl_scan_256(nc, s_warp, &sum);
        if (i < m && off < slot) rle_chars(x, body + off, slot - off);
        base += sum;
      }
      if (base <= slot) {
        kind = SLOT_CHARS;
        len = base;
      }
    }
    __syncthreads();  // the characters of a code that did not fit are overwritten below
    if (kind == SLOT_BITS) {
      const uint8_t *m = masks + (size_t)n * S * S;
      len = (S * S + 7) / 8;
      for (int j = tid; j < len; j += blockDim.x) {
        uint32_t b = 0;
        for (int t = 0; t < 8; ++t) {
          const int px = j * 8 + t;
          if (px < S * S && __ldg(m + px)) b |= 1u << t;
        }
        body[j] = (uint8_t)b;
      }
    }
  }
  for (int j = len + tid; j < slot; j += blockDim.x) body[j] = 0;
  if (tid == 0) {
    reinterpret_cast<int *>(dst + 4 * PACK_COLS)[0] = kind;
    reinterpret_cast<int *>(dst + 4 * PACK_COLS)[1] = len;
  }
}

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int64_t ape_mask_crop_workspace_bytes(int K, int Hp, int Wp) {
  if (K < 0 || Hp <= 0 || Wp <= 0) return 0;
  return (int64_t)K * Hp * ((Wp + 31) / 32) * 4;
}

extern "C" int ape_mask_crop(const void *logits, const int64_t *index, const float *boxes, void *workspace, uint8_t *out, int K,
                             int h, int w, int Hp, int Wp, int S, int dtype, void *stream) {
  if (K == 0) return APE_OK;
  if (!logits || !index || !boxes || !workspace || !out) return fail(APE_ERR_NULL_PTR, "mask_crop: null pointer");
  if (K < 0 || K > 65535 || h <= 0 || w <= 0 || Hp <= 0 || Wp <= 0 || Hp > 65535 || S <= 0 || S > 1024)
    return fail(APE_ERR_INVALID_ARG, "mask_crop: bad geometry K=%d %dx%d -> %dx%d, S=%d", K, h, w, Hp, Wp, S);
  if (reinterpret_cast<uintptr_t>(boxes) & 15) return fail(APE_ERR_INVALID_ARG, "mask_crop: boxes must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int words = (Wp + 31) / 32;
  const float sh = (float)h / (float)Hp, sw = (float)w / (float)Wp;  // area_pixel_compute_scale, align_corners = false
  dim3 g1((words + 7) / 8, Hp, K);
  uint32_t *bits = reinterpret_cast<uint32_t *>(workspace);
  if (dtype == APE_DTYPE_F32)
    APE_LAUNCH((mask_binarize_kernel<float, false>), g1, 256, 0, st, (const float *)logits, (const long long *)index, bits, h, w, Hp, Wp, sh, sw,
               (const int *)nullptr);
  else if (dtype == APE_DTYPE_F16)
    APE_LAUNCH((mask_binarize_kernel<__half, false>), g1, 256, 0, st, (const __half *)logits, (const long long *)index, bits, h, w, Hp, Wp, sh,
               sw, (const int *)nullptr);
  else if (dtype == APE_DTYPE_BF16)
    APE_LAUNCH((mask_binarize_kernel<__nv_bfloat16, false>), g1, 256, 0, st, (const __nv_bfloat16 *)logits, (const long long *)index, bits, h, w,
               Hp, Wp, sh, sw, (const int *)nullptr);
  else
    return fail(APE_ERR_INVALID_ARG, "mask_crop: dtype %d", dtype);
  int rc = check_launch("mask_binarize_kernel");
  if (rc) return rc;
  APE_LAUNCH((mask_roialign_kernel<false>), dim3((S * S + 255) / 256, K), 256, 0, st, (const uint32_t *)bits, boxes, out, Hp, Wp, S,
             (const int *)nullptr);
  return check_launch("mask_roialign_kernel");
}

extern "C" int ape_mask_paste(const uint8_t *masks, const float *boxes, uint8_t *out, int N, int S, int img_h, int img_w,
                              float threshold, void *stream) {
  if (N == 0) return APE_OK;
  if (!masks || !boxes || !out) return fail(APE_ERR_NULL_PTR, "mask_paste: null pointer");
  if (N < 0 || N > 65535 || S <= 0 || img_h <= 0 || img_w <= 0 || img_h > 65535)
    return fail(APE_ERR_INVALID_ARG, "mask_paste: bad geometry N=%d S=%d image %dx%d", N, S, img_h, img_w);
  if (reinterpret_cast<uintptr_t>(boxes) & 15) return fail(APE_ERR_INVALID_ARG, "mask_paste: boxes must be 16-byte aligned");
  APE_LAUNCH(mask_paste_kernel, dim3(((img_w + 3) / 4 + 255) / 256, img_h, N), 256, 0, (cudaStream_t)stream, masks, boxes, out, S,
             img_h, img_w, threshold);
  return check_launch("mask_paste_kernel");
}

// pass 1 (positions == NULL): col_count [N, img_w] int32 <- boundaries per column; pass 2: positions <- boundary positions at
// col_offset [N, img_w] int64 (exclusive scan of col_count over the whole [N, img_w] array).
extern "C" int ape_mask_paste_rle(const uint8_t *masks, const float *boxes, int N, int S, int img_h, int img_w, float threshold,
                                  int *col_count, const int64_t *col_offset, int *positions, void *stream) {
  if (N == 0) return APE_OK;
  if (!masks || !boxes) return fail(APE_ERR_NULL_PTR, "mask_paste_rle: null pointer");
  if (N < 0 || N > 65535 || S <= 0 || img_h <= 0 || img_w <= 0 || (long long)img_h * img_w > 0x7fffffffLL)
    return fail(APE_ERR_INVALID_ARG, "mask_paste_rle: bad geometry N=%d S=%d image %dx%d", N, S, img_h, img_w);
  if (reinterpret_cast<uintptr_t>(boxes) & 15) return fail(APE_ERR_INVALID_ARG, "mask_paste_rle: boxes must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (positions == nullptr) {
    if (!col_count) return fail(APE_ERR_NULL_PTR, "mask_paste_rle: null col_count");
    APE_LAUNCH((mask_rle_kernel<false, false>), dim3(img_w, N), 256, 0, st, masks, boxes, S, img_h, img_w, threshold, col_count,
               (const long long *)nullptr, (int *)nullptr, (const int *)nullptr);
  } else {
    if (!col_offset) return fail(APE_ERR_NULL_PTR, "mask_paste_rle: null col_offset");
    APE_LAUNCH((mask_rle_kernel<true, false>), dim3(img_w, N), 256, 0, st, masks, boxes, S, img_h, img_w, threshold, (int *)nullptr,
               (const long long *)col_offset, positions, (const int *)nullptr);
  }
  return check_launch("mask_rle_kernel");
}

namespace {
// workspace of ape_mask_pack, every part 256-byte aligned; reused image after image
struct PackWs {
  long long *index;
  float4 *crop_box, *paste_box;
  int *live, *chars, *total, *col_count, *positions;
  long long *col_offset;
  uint32_t *bits;
  uint8_t *masks;
  int64_t bytes;
};

PackWs pack_ws(void *base, int topk, int Hp, int Wp, int max_w, int S, int slot) {
  PackWs w{};
  int64_t off = 0;
  auto take = [&](int64_t n) {
    const int64_t o = off;
    off += (n + 255) / 256 * 256;
    return reinterpret_cast<char *>(reinterpret_cast<uintptr_t>(base) + o);
  };
  w.index = reinterpret_cast<long long *>(take(8LL * topk));
  w.crop_box = reinterpret_cast<float4 *>(take(16LL * topk));
  w.paste_box = reinterpret_cast<float4 *>(take(16LL * topk));
  w.live = reinterpret_cast<int *>(take(4LL * topk));
  w.chars = reinterpret_cast<int *>(take(4LL * topk));
  w.total = reinterpret_cast<int *>(take(4LL * topk));
  w.col_count = reinterpret_cast<int *>(take(4LL * topk * max_w));
  w.col_offset = reinterpret_cast<long long *>(take(8LL * topk * max_w));
  w.positions = reinterpret_cast<int *>(take(4LL * topk * slot));
  w.bits = reinterpret_cast<uint32_t *>(take(ape_mask_crop_workspace_bytes(topk, Hp, Wp)));
  w.masks = reinterpret_cast<uint8_t *>(take((int64_t)topk * S * S));
  w.bytes = off;
  return w;
}
}  // namespace

extern "C" int64_t ape_mask_pack_workspace_bytes(int topk, int Hp, int Wp, int max_w, int S, int slot) {
  if (topk <= 0 || Hp <= 0 || Wp <= 0 || max_w <= 0 || S <= 0 || slot <= 0) return 0;
  return pack_ws(nullptr, topk, Hp, Wp, max_w, S, slot).bytes;
}

extern "C" int ape_mask_pack(const void *logits, const float *rows, const int *out_hw, void *workspace, uint8_t *out, int B, int topk,
                             int Q, int h, int w, int Hp, int Wp, int S, int slot, int dtype, void *stream) {
  if (B == 0 || topk == 0) return APE_OK;
  if (!logits || !rows || !out_hw || !workspace || !out) return fail(APE_ERR_NULL_PTR, "mask_pack: null pointer");
  if (B < 0 || topk < 0 || topk > 65535 || Q <= 0 || h <= 0 || w <= 0 || Hp <= 0 || Wp <= 0 || Hp > 65535 || S <= 0 || S > 1024)
    return fail(APE_ERR_INVALID_ARG, "mask_pack: bad geometry B=%d topk=%d Q=%d %dx%d -> %dx%d, S=%d", B, topk, Q, h, w, Hp, Wp, S);
  if (slot % 4 != 0 || slot < (S * S + 7) / 8)
    return fail(APE_ERR_INVALID_ARG, "mask_pack: slot of %d bytes (a multiple of 4 that holds the %d x %d mask as bits)", slot, S, S);
  if ((reinterpret_cast<uintptr_t>(rows) | reinterpret_cast<uintptr_t>(out)) & 3)
    return fail(APE_ERR_INVALID_ARG, "mask_pack: rows and out must be 4-byte aligned");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(APE_ERR_INVALID_ARG, "mask_pack: workspace must be 256-byte aligned");
  if (dtype != APE_DTYPE_F32 && dtype != APE_DTYPE_F16 && dtype != APE_DTYPE_BF16) return fail(APE_ERR_INVALID_ARG, "mask_pack: dtype %d", dtype);
  int max_w = 0;
  for (int b = 0; b < B; ++b) {
    const int oh = out_hw[2 * b], ow = out_hw[2 * b + 1];
    if (oh <= 0 || ow <= 0 || (long long)oh * ow > 0x7fffffffLL)
      return fail(APE_ERR_INVALID_ARG, "mask_pack: bad output size %dx%d of image %d", oh, ow, b);
    max_w = max(max_w, ow);
  }
  const PackWs ws = pack_ws(workspace, topk, Hp, Wp, max_w, S, slot);
  cudaStream_t st = (cudaStream_t)stream;
  const int words = (Wp + 31) / 32;
  const float sh = (float)h / (float)Hp, sw = (float)w / (float)Wp;  // as ape_mask_crop
  const size_t esize = dtype == APE_DTYPE_F32 ? 4 : 2;
  int rc;
  for (int b = 0; b < B; ++b) {
    const int H = out_hw[2 * b], W = out_hw[2 * b + 1];
    const float *r = rows + (size_t)b * topk * PACK_COLS;
    const void *lg = reinterpret_cast<const char *>(logits) + (size_t)b * Q * h * w * esize;
    APE_LAUNCH(mask_pack_prep_kernel, (topk + 255) / 256, 256, 0, st, r, topk, ws.index, ws.crop_box, ws.paste_box, ws.live);
    if ((rc = check_launch("mask_pack_prep_kernel"))) return rc;
    const dim3 g1((words + 7) / 8, Hp, topk);
    if (dtype == APE_DTYPE_F32)
      APE_LAUNCH((mask_binarize_kernel<float, true>), g1, 256, 0, st, (const float *)lg, (const long long *)ws.index, ws.bits, h, w, Hp,
                 Wp, sh, sw, (const int *)ws.live);
    else if (dtype == APE_DTYPE_F16)
      APE_LAUNCH((mask_binarize_kernel<__half, true>), g1, 256, 0, st, (const __half *)lg, (const long long *)ws.index, ws.bits, h, w, Hp,
                 Wp, sh, sw, (const int *)ws.live);
    else
      APE_LAUNCH((mask_binarize_kernel<__nv_bfloat16, true>), g1, 256, 0, st, (const __nv_bfloat16 *)lg, (const long long *)ws.index,
                 ws.bits, h, w, Hp, Wp, sh, sw, (const int *)ws.live);
    if ((rc = check_launch("mask_binarize_kernel"))) return rc;
    APE_LAUNCH((mask_roialign_kernel<true>), dim3((S * S + 255) / 256, topk), 256, 0, st, (const uint32_t *)ws.bits,
               (const float *)ws.crop_box, ws.masks, Hp, Wp, S, (const int *)ws.live);
    if ((rc = check_launch("mask_roialign_kernel"))) return rc;
    APE_LAUNCH((mask_rle_kernel<false, true>), dim3(W, topk), 256, 0, st, (const uint8_t *)ws.masks, (const float *)ws.paste_box, S, H, W,
               0.5f, ws.col_count, (const long long *)nullptr, (int *)nullptr, (const int *)ws.live);
    if ((rc = check_launch("mask_rle_kernel"))) return rc;
    APE_LAUNCH(mask_pack_scan_kernel, topk, 256, 0, st, (const int *)ws.col_count, (const int *)ws.live, W, slot, ws.col_offset,
               ws.total, ws.chars);
    if ((rc = check_launch("mask_pack_scan_kernel"))) return rc;
    APE_LAUNCH((mask_rle_kernel<true, true>), dim3(W, topk), 256, 0, st, (const uint8_t *)ws.masks, (const float *)ws.paste_box, S, H, W,
               0.5f, (int *)nullptr, (const long long *)ws.col_offset, ws.positions, (const int *)ws.chars);
    if ((rc = check_launch("mask_rle_kernel"))) return rc;
    APE_LAUNCH(mask_pack_encode_kernel, topk, 256, 0, st, r, (const int *)ws.live, (const int *)ws.chars, (const int *)ws.total,
               (const int *)ws.positions, (const uint8_t *)ws.masks, S, H, W, slot, out + (size_t)b * topk * (PACK_HEAD + slot));
    if ((rc = check_launch("mask_pack_encode_kernel"))) return rc;
  }
  return APE_OK;
}

// cocoapi rleToString (maskApi.c): run lengths -> the compressed ASCII string of the "counts" field (HOST function).
// Every count from the fourth on is stored as the difference to the count two places earlier; 5 bits per character plus a
// continuation bit, offset 48.  Returns the number of characters written (out must hold 7 * m), < 0 on bad arguments.
extern "C" int ape_rle_to_string(const uint32_t *counts, int m, char *out) {
  if (m < 0 || (m > 0 && (!counts || !out))) return fail(APE_ERR_INVALID_ARG, "rle_to_string: bad arguments");
  int p = 0;
  for (int i = 0; i < m; ++i) {
    long long x = (long long)counts[i];
    if (i > 2) x -= (long long)counts[i - 2];
    bool more = true;
    while (more) {
      char c = (char)(x & 0x1f);
      x >>= 5;
      more = (c & 0x10) ? x != -1 : x != 0;
      if (more) c |= 0x20;
      c += 48;
      out[p++] = c;
    }
  }
  return p;
}
