// Shared helpers for the psalm_b200 CUDA kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/psalm_b200.h"

namespace psalm {

void set_error(const char* fmt, ...);

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return PSALM_E_CUDA;
  }
  return PSALM_OK;
}

#define PSALM_REQUIRE(cond, ...)            \
  do {                                      \
    if (!(cond)) {                          \
      psalm::set_error(__VA_ARGS__);        \
      return PSALM_E_ARG;                   \
    }                                       \
  } while (0)

inline size_t dtype_size(int dt) { return dt == PSALM_F32 ? 4 : 2; }

// cudaFuncSetAttribute / cluster-occupancy probes are PER DEVICE: a once-per-process flag would leave the second
// GPU of a process unconfigured (kernels needing > 48 KB of dynamic shared memory then fail to launch there).
struct PerDevice {
  int v[64];
  bool set[64];
  PerDevice() { for (int i = 0; i < 64; ++i) { v[i] = 0; set[i] = false; } }
  static int dev() { int d = 0; cudaGetDevice(&d); return d & 63; }
  bool first() { const int d = dev(); if (set[d]) return false; set[d] = true; return true; }
};

// ---- element conversion -------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// unpack a 32-bit word holding two 16-bit floats into two fp32
template <typename T> __device__ __forceinline__ void unpack2(uint32_t w, float& lo, float& hi);
template <> __device__ __forceinline__ void unpack2<__nv_bfloat16>(uint32_t w, float& lo, float& hi) {
  lo = __uint_as_float(w << 16);
  hi = __uint_as_float(w & 0xffff0000u);
}
template <> __device__ __forceinline__ void unpack2<__half>(uint32_t w, float& lo, float& hi) {
  __half2 h = *reinterpret_cast<__half2*>(&w);
  float2 f = __half22float2(h);
  lo = f.x;
  hi = f.y;
}
template <typename T> __device__ __forceinline__ uint32_t pack2(float lo, float hi);
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// acc.xy += v.xy * w, one rounding per lane (Hopper has no packed fp32 FMA)
__device__ __forceinline__ void ffma2(float2& acc, const float2 v, const float w) {
  acc.x = fmaf(v.x, w, acc.x);
  acc.y = fmaf(v.y, w, acc.y);
}

// 16-byte vector of CH elements of T (CH = 4 for fp32, 8 for 16-bit types), as fp32 lanes
template <typename T> struct Vec16 {
  static constexpr int CH = 16 / sizeof(T);
};

template <typename T>
__device__ __forceinline__ void load16_as_f32(const T* p, float (&f)[16 / sizeof(T)]) {
  if constexpr (sizeof(T) == 4) {
    float4 v = __ldg(reinterpret_cast<const float4*>(p));
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  } else {
    uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
    unpack2<T>(v.x, f[0], f[1]);
    unpack2<T>(v.y, f[2], f[3]);
    unpack2<T>(v.z, f[4], f[5]);
    unpack2<T>(v.w, f[6], f[7]);
  }
}

// same, as CH/2 float2 pairs (operands of the packed FFMA2 path)
template <typename T>
__device__ __forceinline__ void load16_as_f32x2(const T* p, float2 (&f)[8 / sizeof(T)]) {
  if constexpr (sizeof(T) == 4) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(p));
    f[0] = make_float2(v.x, v.y);
    f[1] = make_float2(v.z, v.w);
  } else {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
    unpack2<T>(v.x, f[0].x, f[0].y);
    unpack2<T>(v.y, f[1].x, f[1].y);
    unpack2<T>(v.z, f[2].x, f[2].y);
    unpack2<T>(v.w, f[3].x, f[3].y);
  }
}

template <typename T>
__device__ __forceinline__ void store16_from_f32(T* p, const float (&f)[16 / sizeof(T)]) {
  if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  } else {
    uint4 v;
    v.x = pack2<T>(f[0], f[1]);
    v.y = pack2<T>(f[2], f[3]);
    v.z = pack2<T>(f[4], f[5]);
    v.w = pack2<T>(f[6], f[7]);
    *reinterpret_cast<uint4*>(p) = v;
  }
}

}  // namespace psalm
