// Device helpers shared by the one-position decoding kernels (decode.cuh) and the multi-position ones (decode_extend.cuh).
#pragma once
#include <cuda_runtime.h>

namespace hy {
namespace dec {

// the 3-tap causal short filter of one channel at one position: w0 p[t-2] + w1 p[t-1] + w2 p[t] + b
__device__ __forceinline__ float short3(float w0, float w1, float w2, float b, float pm2, float pm1, float p0) {
  return fmaf(w0, pm2, fmaf(w1, pm1, fmaf(w2, p0, b)));
}

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

}  // namespace dec
}  // namespace hy
