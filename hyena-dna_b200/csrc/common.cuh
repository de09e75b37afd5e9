// Shared helpers for the sm_90a Hyena long-convolution kernels.
//
// Nothing in this directory includes torch headers: the library is a plain C-ABI
// shared object (include/hyena_b200.h) and PyTorch only hands it device pointers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace hy {

// ---------------------------------------------------------------- complex helpers
// A complex value is one float2; a complex multiply is two FMAs and two multiplies.
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
// a * conj(b)
__device__ __forceinline__ float2 cmulc(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, a.y * b.y), fmaf(a.y, b.x, -a.x * b.y));
}
// a * (c - i s) with compile-time friendly real constants c, s
__device__ __forceinline__ float2 cmul_cs(float2 a, float c, float s) {
  return make_float2(fmaf(a.x, c, a.y * s), fmaf(a.y, c, -a.x * s));
}
// elementwise (not complex) product / fma of two sample pairs
__device__ __forceinline__ float2 pmul(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 pfma(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 cconj(float2 a) { return make_float2(a.x, -a.y); }
// -i * a
__device__ __forceinline__ float2 cmul_negi(float2 a) { return make_float2(a.y, -a.x); }
// +i * a
__device__ __forceinline__ float2 cmul_i(float2 a) { return make_float2(-a.y, a.x); }

// ---------------------------------------------------------------- compile-time loop
template <int I> struct IC { static constexpr int value = I; };
template <int I, int N, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (I < N) {
    f(IC<I>{});
    static_for<I + 1, N>(f);
  }
}

__host__ __device__ constexpr int ilog2c(int n) { return n <= 1 ? 0 : 1 + ilog2c(n >> 1); }
__host__ __device__ constexpr int brev(int x, int bits) {
  int r = 0;
  for (int i = 0; i < bits; ++i) r |= ((x >> i) & 1) << (bits - 1 - i);
  return r;
}

// ---------------------------------------------------------------- twiddle tables (device memory)
// tw1024[j] = exp(-2*pi*i * j / 1024)      j in [0,1024)   (also the "hi" table of the 2^20 roots)
// twlo[j]   = exp(-2*pi*i * j / 2^20)      j in [0,1024)   ("lo" table: W_{2^20}^e = tw1024[e>>10] * twlo[e&1023])
struct Twiddles {
  const float2* tw1024;
  const float2* twlo;
};

// W_{2^20}^{e20}, e20 in [0, 2^20)
__device__ __forceinline__ float2 root20(const Twiddles& T, uint32_t e20) {
  float2 hi = __ldg(T.tw1024 + (e20 >> 10));
  float2 lo = __ldg(T.twlo + (e20 & 1023u));
  return cmul(hi, lo);
}

// ---------------------------------------------------------------- cache-hinted global access
__device__ __forceinline__ float2 ld_stream2(const float2* p) {   // read-once data: do not keep in L1
  float2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ float ld_stream1(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}

// ---------------------------------------------------------------- cp.async (LDGSTS) helpers
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  const int n = valid ? 16 : 0;                      // src-size 0: the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

}  // namespace hy
