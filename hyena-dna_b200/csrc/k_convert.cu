// Conversions between the reference's filter-spectrum convention and this library's packed spectrum.
//
// The reference extension takes `filter = torch.fft.rfft(k, n=fft_size)` -- (H, fft_size/2+1) complex64, natural bin
// order, unnormalised (src/ops/fftconv.py:64-65, csrc/fftconv/fftconv.cpp:53-61) -- and returns
// `dfilter` with irfft(dfilter, n=fft_size, norm='forward')[:L] == dk (fftconv.cpp:134-143,235;
// src/ops/fftconv.py:94-98).  The kernels here work on the packed half-size spectrum Z[k] = FFT_M(x[2m] + i x[2m+1])
// stored in [k1][k2] order (fft_passes.cuh).  For fft_size == 2M both carry the same information:
//     X[f] = E[f] + W_N^f O[f],   Z[f] = E[f] + i O[f],   E[f] = (X[f] + conj X[M-f]) / 2,   N = 2M.
// For sequences shorter than the library's minimum transform (fft_size < 2M = 2048) the conversion goes through the time
// domain with a direct DFT (at most 1024 points per channel).
#include "launch.h"

namespace hy {

__device__ __forceinline__ size_t packed_index(uint32_t f, int logM1, int logM2) {
  const uint32_t k1 = f & ((1u << logM1) - 1u), k2 = f >> logM1;
  return ((size_t)k1 << logM2) + k2;
}

// X (H, M+1) natural -> Z (H, M) packed
__global__ void rfft_to_packed_kernel(const float2* __restrict__ X, float2* __restrict__ Z, int H, int logM, int logM1) {
  const uint32_t M = 1u << logM;
  const int logM2 = logM - logM1;
  const size_t total = (size_t)H * M;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t f = (uint32_t)(i & (M - 1));
    const size_t h = i >> logM;
    const float2* Xh = X + h * (size_t)(M + 1);
    const float2 a = Xh[f], b = cconj(Xh[M - f]);
    const float2 E = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y + b.y));
    float s, c;
    sincospif((float)f / (float)M, &s, &c);                      // W_N^{-f} = exp(+i pi f / M)
    const float2 d = make_float2(0.5f * (a.x - b.x), 0.5f * (a.y - b.y));
    const float2 O = make_float2(d.x * c - d.y * s, d.x * s + d.y * c);
    Z[h * (size_t)M + packed_index(f, logM1, logM2)] = make_float2(E.x - O.y, E.y + O.x);   // E + i O
  }
}

// Z (H, M) packed -> X (H, M+1) natural, scaled
__global__ void packed_to_rfft_kernel(const float2* __restrict__ Z, float2* __restrict__ X, int H, int logM, int logM1,
                                      float scale) {
  const uint32_t M = 1u << logM;
  const int logM2 = logM - logM1;
  const size_t total = (size_t)H * (M + 1);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t h = i / (M + 1);
    const uint32_t f = (uint32_t)(i - h * (M + 1));
    const float2* Zh = Z + h * (size_t)M;
    const uint32_t fa = f & (M - 1), fb = (M - f) & (M - 1);
    const float2 a = Zh[packed_index(fa, logM1, logM2)], b = cconj(Zh[packed_index(fb, logM1, logM2)]);
    const float2 E = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y + b.y));
    const float2 O = make_float2(0.5f * (a.y - b.y), -0.5f * (a.x - b.x));       // (a - b) / (2i)
    float s, c;
    sincospif((float)f / (float)M, &s, &c);                      // W_N^f = exp(-i pi f / M) = c - i s
    const float2 WO = make_float2(O.x * c + O.y * s, O.y * c - O.x * s);
    X[i] = make_float2(scale * (E.x + WO.x), scale * (E.y + WO.y));
  }
}

// direct inverse real DFT: k[h][t] = (1/N) sum_f X~[f] exp(+2 pi i f t / N), t < L   (N <= 2048)
__global__ void rfft_to_time_small_kernel(const float2* __restrict__ X, float* __restrict__ k, int H, int L, int N) {
  const int half = N / 2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)H * L; i += (size_t)gridDim.x * blockDim.x) {
    const int h = (int)(i / L), t = (int)(i - (size_t)h * L);
    const float2* Xh = X + (size_t)h * (half + 1);
    float acc = Xh[0].x + ((t & 1) ? -Xh[half].x : Xh[half].x);
    for (int f = 1; f < half; ++f) {
      float s, c;
      sincospif(2.f * (float)((f * t) & (N - 1)) / (float)N, &s, &c);
      acc += 2.f * (Xh[f].x * c - Xh[f].y * s);
    }
    k[i] = acc / (float)N;
  }
}

// direct real DFT of x (H, L) zero padded to N: X[h][f] = scale * sum_t x[t] exp(-2 pi i f t / N), f <= N/2
__global__ void time_to_rfft_small_kernel(const float* __restrict__ x, float2* __restrict__ X, int H, int L, int N, float scale) {
  const int half = N / 2;
  const size_t total = (size_t)H * (half + 1);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int h = (int)(i / (half + 1)), f = (int)(i - (size_t)h * (half + 1));
    const float* xh = x + (size_t)h * L;
    float re = 0.f, im = 0.f;
    for (int t = 0; t < L; ++t) {
      float s, c;
      sincospif(2.f * (float)((f * t) & (N - 1)) / (float)N, &s, &c);
      re = fmaf(xh[t], c, re);
      im = fmaf(-xh[t], s, im);
    }
    X[i] = make_float2(scale * re, scale * im);
  }
}

static int blocks_for(size_t n) { size_t b = (n + 255) / 256; return (int)(b > 132 * 16 ? 132 * 16 : (b ? b : 1)); }

cudaError_t launch_rfft_to_packed(const float2* X, float2* Z, int H, int logM, int logM1, cudaStream_t s) {
  prof_begin(K_CONVERT, s);
  rfft_to_packed_kernel<<<blocks_for((size_t)H << logM), 256, 0, s>>>(X, Z, H, logM, logM1);
  prof_end(K_CONVERT, s);
  return cudaGetLastError();
}
cudaError_t launch_packed_to_rfft(const float2* Z, float2* X, int H, int logM, int logM1, float scale, cudaStream_t s) {
  prof_begin(K_CONVERT, s);
  packed_to_rfft_kernel<<<blocks_for((size_t)H << logM), 256, 0, s>>>(Z, X, H, logM, logM1, scale);
  prof_end(K_CONVERT, s);
  return cudaGetLastError();
}
cudaError_t launch_rfft_to_time_small(const float2* X, float* k, int H, int L, int N, cudaStream_t s) {
  prof_begin(K_CONVERT, s);
  rfft_to_time_small_kernel<<<blocks_for((size_t)H * L), 256, 0, s>>>(X, k, H, L, N);
  prof_end(K_CONVERT, s);
  return cudaGetLastError();
}
cudaError_t launch_time_to_rfft_small(const float* x, float2* X, int H, int L, int N, float scale, cudaStream_t s) {
  prof_begin(K_CONVERT, s);
  time_to_rfft_small_kernel<<<blocks_for((size_t)H * (N / 2 + 1)), 256, 0, s>>>(x, X, H, L, N, scale);
  prof_end(K_CONVERT, s);
  return cudaGetLastError();
}

}  // namespace hy
