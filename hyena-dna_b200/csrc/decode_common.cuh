// Device helpers shared by the one-position decoding kernels (decode.cuh) and the multi-position ones (decode_extend.cuh).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace hy {
namespace dec {

// the 3-tap causal short filter of one channel at one position: w0 p[t-2] + w1 p[t-1] + w2 p[t] + b
__device__ __forceinline__ float short3(float w0, float w1, float w2, float b, float pm2, float pm1, float p0) {
  return fmaf(w0, pm2, fmaf(w1, pm1, fmaf(w2, p0, b)));
}

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// ---- the stored history h: float (the default), __half or __nv_bfloat16 (decode_args.h).  Every value is computed in
// fp32 and rounded to nearest even once, when it is stored (hround); every read widens it back to fp32 exactly (hwiden).
// For float both are the identity, so the fp32 instantiations are the kernels as they were.
template <class T> __device__ __forceinline__ T hround(float x);
template <> __device__ __forceinline__ float hround<float>(float x) { return x; }
template <> __device__ __forceinline__ __half hround<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 hround<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

__device__ __forceinline__ float hwiden(float x) { return x; }
__device__ __forceinline__ float hwiden(__half x) { return __half2float(x); }
__device__ __forceinline__ float hwiden(__nv_bfloat16 x) { return __bfloat162float(x); }

// 4 consecutive history positions starting at a multiple of 4 (16 bytes of float, 8 bytes of a 16-bit type), widened
__device__ __forceinline__ float4 hld4(const float* p) { return ld4(p); }
__device__ __forceinline__ float4 hld4(const __half* p) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 hld4(const __nv_bfloat16* p) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

// the vector of 4 history positions the shift kernel moves: float4, or 8 bytes of a 16-bit type
template <class T> struct HVec4 { using type = uint2; };
template <> struct HVec4<float> { using type = float4; };

}  // namespace dec
}  // namespace hy
