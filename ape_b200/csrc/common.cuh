// common.cuh — shared helpers for libape_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <utility>

#include "ape_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libape_b200 is written for sm_90a (H100) only"
#endif

namespace ape {

// ---- status plumbing -------------------------------------------------------------------------
char *last_error_buf();  // thread-local, 512 bytes
void count_launch(int n = 1);

inline int fail(int code, const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

inline int check_launch(const char *what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail((int)e, "%s: %s", what, cudaGetErrorString(e));
  count_launch();
  return APE_OK;
}

inline int dtype_size(int dtype) { return dtype == APE_DTYPE_F32 ? 4 : 2; }

// ---- programmatic dependent launch -------------------------------------------------------------
// Every kernel of the library starts with pdl_prologue(): it tells the scheduler that the NEXT kernel of the stream may be
// launched (its CTAs start as SM resources free up and run their own set-up), then waits until the PREVIOUS kernel has
// completed and flushed its writes — before this kernel reads or writes any global memory.  Launches go through APE_LAUNCH,
// which sets cudaLaunchAttributeProgrammaticStreamSerialization; between two kernels of the library the launch latency and
// the prologue (barrier set-up of the TMA / wgmma kernels) then overlap the tail of the previous kernel, in
// eager mode and inside captured CUDA graphs alike.  A predecessor that is not one of ours never triggers early, so the
// dependency degrades to ordinary stream order.  APE_PDL=0 in the environment disables the attribute (A/B runs).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() {
  pdl_launch_dependents();
  pdl_wait();
}

bool pdl_enabled();  // abi.cu

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args &&...args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
#define APE_LAUNCH(kernel, grid, block, smem, stream, ...) \
  (void)ape::launch_pdl(kernel, dim3(grid), dim3(block), (size_t)(smem), stream, __VA_ARGS__)

// ---- device helpers --------------------------------------------------------------------------
// 128-bit read-only gather load (goes through L1; texels are re-used by neighbouring queries).
__device__ __forceinline__ uint4 ldg_nc_v4(const uint4 *p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// streaming loads: read exactly once, keep them out of L1 so gathered texels stay resident.
__device__ __forceinline__ float2 ldg_stream_f2(const float2 *p) {
  float2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ float ldg_stream_f1(const float *p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t ldg_stream_u32(const uint32_t *p) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ uint16_t ldg_stream_u16(const uint16_t *p) {
  uint16_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void stg_stream_v4(uint4 *p, uint4 v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// ---- sizes held on the device (the *_dev entry points of the packed result stages) ------------
// One image's row (image h, w, output h, w) of an int32 [B, 4] device tensor.  The image is clamped to [1, Hp] x [1, Wp] (the
// pad), the output to [1, cap] x [1, cap] (the buffers' capacity): a bad size changes values, never addresses.
struct DevSizes {
  int ih, iw, oh, ow;
};
__device__ __forceinline__ DevSizes dev_sizes(const int *row, int Hp, int Wp, int cap) {
  DevSizes s;
  s.ih = min(max(row[0], 1), Hp);
  s.iw = min(max(row[1], 1), Wp);
  s.oh = min(max(row[2], 1), cap);
  s.ow = min(max(row[3], 1), cap);
  return s;
}

// ---- class-argmax keys (semantic label maps: gemm_tc.cu EpiArgmax, semseg.cu) ---------------------
// (order-preserving bits of the fp32 value) << 32 | (0xFFFFFFFF - column): the unsigned maximum of such keys is the largest
// value and, among equal values, the lowest column, i.e. torch.argmax.  -0 is folded into +0 (argmax compares them equal).
__host__ __device__ __forceinline__ unsigned long long argmax_key_bits(uint32_t u, uint32_t col) {
  const uint32_t o = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)o << 32) | (0xFFFFFFFFu - col);
}
__device__ __forceinline__ unsigned long long argmax_key(float v, int col) {
  return argmax_key_bits(__float_as_uint(v + 0.f), (uint32_t)col);
}
__device__ __forceinline__ float argmax_key_value(unsigned long long key) {
  const uint32_t o = (uint32_t)(key >> 32);
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// element traits: conversion of packed 16-bit pairs to fp32 and back.
template <typename T>
struct Elem;
template <>
struct Elem<float> {
  static constexpr int kVec = 4;  // elements per 16 bytes
  __device__ static __forceinline__ float load1(const float *p) { return ldg_stream_f1(p); }
  __device__ static __forceinline__ float2 load2(const float *p) {
    return ldg_stream_f2(reinterpret_cast<const float2 *>(p));
  }
  __device__ static __forceinline__ void unpack(const uint4 &v, float *f) {
    f[0] = __uint_as_float(v.x);
    f[1] = __uint_as_float(v.y);
    f[2] = __uint_as_float(v.z);
    f[3] = __uint_as_float(v.w);
  }
  __device__ static __forceinline__ uint4 pack(const float *f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                      __float_as_uint(f[3]));
  }
  __device__ static __forceinline__ float to_f(float x) { return x; }
  __device__ static __forceinline__ float from_f(float x) { return x; }
};
template <>
struct Elem<__half> {
  static constexpr int kVec = 8;
  __device__ static __forceinline__ float load1(const __half *p) {
    return __half2float(__ushort_as_half(ldg_stream_u16(reinterpret_cast<const uint16_t *>(p))));
  }
  __device__ static __forceinline__ float2 load2(const __half *p) {
    uint32_t u = ldg_stream_u32(reinterpret_cast<const uint32_t *>(p));
    return __half22float2(*reinterpret_cast<__half2 *>(&u));
  }
  __device__ static __forceinline__ void unpack(const uint4 &v, float *f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 t = __half22float2(*reinterpret_cast<const __half2 *>(&w[i]));
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
  }
  __device__ static __forceinline__ uint4 pack(const float *f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 t = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t *>(&t);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
  __device__ static __forceinline__ float to_f(__half x) { return __half2float(x); }
  __device__ static __forceinline__ __half from_f(float x) { return __float2half_rn(x); }
};
template <>
struct Elem<__nv_bfloat16> {
  static constexpr int kVec = 8;
  __device__ static __forceinline__ float load1(const __nv_bfloat16 *p) {
    uint32_t u = ldg_stream_u16(reinterpret_cast<const uint16_t *>(p));
    return __uint_as_float(u << 16);
  }
  __device__ static __forceinline__ float2 load2(const __nv_bfloat16 *p) {
    uint32_t u = ldg_stream_u32(reinterpret_cast<const uint32_t *>(p));
    return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
  }
  __device__ static __forceinline__ void unpack(const uint4 &v, float *f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ static __forceinline__ uint4 pack(const float *f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 t = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t *>(&t);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
  __device__ static __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
  __device__ static __forceinline__ __nv_bfloat16 from_f(float x) { return __float2bfloat16_rn(x); }
};

}  // namespace ape
