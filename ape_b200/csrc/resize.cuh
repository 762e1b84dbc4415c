// resize.cuh — ATen's upsample_bilinear2d (align_corners = false) arithmetic for kernels that resample mask logits on the fly
// (semseg.cu, panoptic.cu): area_pixel_compute_source_index with scale = in / out in fp32, the index clamp and the lambdas.
#pragma once
#include "common.cuh"

namespace ape {

// source indices and weights of one output index of upsample_bilinear2d (align_corners = false)
struct Lerp {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Lerp lerp_at(float scale, int dst, int in_size) {
  const float src = fmaxf(scale * ((float)dst + 0.5f) - 0.5f, 0.f);
  Lerp r;
  r.i0 = (int)src;
  r.i1 = r.i0 + (r.i0 < in_size - 1 ? 1 : 0);
  r.l1 = src - (float)r.i0;
  r.l0 = 1.f - r.l1;
  return r;
}

template <typename T>
__device__ __forceinline__ float ldf(const T *p) {
  return Elem<T>::to_f(__ldg(p));
}

// resize1(plane)(Y, X) for the padded-grid point given by its row / column lerps
template <typename TL>
__device__ __forceinline__ float up_value(const TL *plane, int w, const Lerp &ry, const Lerp &rx) {
  const TL *r0 = plane + (size_t)ry.i0 * w, *r1 = plane + (size_t)ry.i1 * w;
  return ry.l0 * (rx.l0 * ldf(r0 + rx.i0) + rx.l1 * ldf(r0 + rx.i1)) +
         ry.l1 * (rx.l0 * ldf(r1 + rx.i0) + rx.l1 * ldf(r1 + rx.i1));
}

}  // namespace ape
