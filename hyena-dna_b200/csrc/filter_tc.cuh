// Implicit filter (forward and backward) on the Hopper tensor cores (wgmma), sm_90a.
//
// The filter MLP of filter_params.h (reference src/models/sequence/hyena.py:96-155,199-238), with the three
// GEMM-shaped layers run as wgmma.mma_async ... .tf32 with fp32 accumulators in registers:
//
//   tile = 128 positions; 512 threads = four warpgroups, warpgroup w owns rows 64 (w & 1) .. of the tile and column
//          half (w >> 1) of every layer (wgmma M = 64)
//   layer 1,2 : D[128 x 64]  = act[128 x 64] * W^T      (N = 64,  K = 64)
//   layer 3   : D[128 x 128] = act[128 x 64] * W3_h^T   (N = 128, K = 64) per half of 128 channels
//
// fp32 accuracy on tf32 tensor cores: every fp32 operand x is split x = hi + lo with hi = rna_tf32(x),
// lo = rna_tf32(x - hi), and each product is issued three times (hi*hi + lo*hi + hi*lo, the lo*lo term is
// below 2^-22 relative): "3xTF32".  Plain TF32 would put ~5e-4 relative error into k and hence into y.
//
// Operands are written to shared memory by the CUDA cores (the activations are produced in registers by the
// previous epilogue, so there is nothing for TMA to fetch) in the canonical no-swizzle K-major core-matrix
// layout: element (r, k) of an R x 64 fp32 operand sits at byte (r/8)*2048 + (k/4)*128 + (r%8)*16 + (k%4)*4,
// i.e. 8-row x 16-byte core matrices, LBO (K direction) = 128 B, SBO (M/N direction) = 2048 B.
#pragma once
#include "fft_passes.cuh"
#include "filter_params.h"
#include "tc_prims.cuh"

namespace hy {
namespace tc {

constexpr int kTileM = 128;
constexpr uint32_t kSBO = 2048, kLBO = 128;
constexpr int kImgW64 = 64 * 64;            // floats of a 64-row operand image
constexpr int kImgW128 = 128 * 64;          // floats of a 128-row operand image

__host__ __device__ constexpr uint32_t op_off(int r, int k) {   // byte offset inside an operand image
  return (uint32_t)((r >> 3) * 2048 + (k >> 2) * 128 + (r & 7) * 16 + (k & 3) * 4);
}

// shared memory map (bytes)
constexpr uint32_t kOffAhi = 0, kOffAlo = 32768, kOffW1hi = 65536, kOffW1lo = 81920, kOffW2hi = 98304,
                   kOffW2lo = 114688, kOffW3hi = 131072, kOffW3lo = 163840, kOffMisc = 196608;
// misc: W0[64][16] | b0[64] | b1[64] | b2[64] | freq[64]
constexpr uint32_t kMiscFloats = 64 * 16 + 4 * 64;
constexpr size_t kSmemBytes = kOffMisc + kMiscFloats * 4 + 16;

__host__ __device__ constexpr size_t wimg_floats(int D) { return 4 * (size_t)kImgW64 + (size_t)((D + 127) / 128) * 2 * kImgW128; }

// Accurate sinf / sincosf are ~100 instructions each with their large-argument paths; inlined 48x per tile they made
// the epilogue instruction-fetch bound (ncu: stall_no_instruction 5.1 per issue).  One out-of-line copy each.
__device__ __noinline__ float sin_ni(float x) { return sinf(x); }
__device__ __noinline__ float cos_ni(float x) { return cosf(x); }

// Inline sin / cos for the epilogues: three-term Cody-Waite reduction by pi/2 (FMA) + the classic degree-7 / degree-8 minimax
// polynomials on [-pi/4, pi/4], branch free.  <= 1.5 ulp for |x| <= 1e3 and <= 7e-8 absolute everywhere below the guard (checked
// against fp64 over 1e7 arguments; libm's fp32 sin has the same absolute error) -- the accuracy class of sinf / torch.sin, which the
// reference uses (hyena.py:105).  ~22 instructions with no call: the 16-32 evaluations of an epilogue are independent, so they
// overlap (the out-of-line sinf serialised them: one ~120-cycle dependent chain per call, 0.5 instructions per scheduler-cycle).
// Arguments here are freq * pre-activation (|x| <~ 1e2); beyond the guard the library function runs.
__device__ __forceinline__ void sincos_core(float x, float& sn, float& cs, int& q) {
  const float fq = rintf(x * 0.636619772367581343f);
  q = (int)fq;
  float r = fmaf(fq, -1.5707963705062866f, x);
  r = fmaf(fq, 4.371138828673793e-08f, r);
  r = fmaf(fq, 1.7763568394002505e-15f, r);
  const float s = r * r;
  float ps = fmaf(-1.95152959e-4f, s, 8.33216087e-3f);
  ps = fmaf(ps, s, -1.66666546e-1f);
  sn = fmaf(ps, s * r, r);
  float pc = fmaf(2.44331571e-5f, s, -1.38873163e-3f);
  pc = fmaf(pc, s, 4.16666457e-2f);
  pc = fmaf(pc, s, -0.5f);
  cs = fmaf(pc, s, 1.0f);
}
__device__ __forceinline__ float sin_acc(float x) {
  if (fabsf(x) > 30000.f) return sin_ni(x);
  float sn, cs; int q;
  sincos_core(x, sn, cs, q);
  const float v = (q & 1) ? cs : sn;
  return (q & 2) ? -v : v;
}
__device__ __forceinline__ float cos_acc(float x) {
  if (fabsf(x) > 30000.f) return cos_ni(x);
  float sn, cs; int q;
  sincos_core(x, sn, cs, q);
  const float v = (q & 1) ? sn : cs;
  return ((q + 1) & 2) ? -v : v;
}

// Fragment coordinates of this thread (see tc_prims.cuh): rows r0 and r0 + 8 of the tile, columns
// cbase + 8 (i >> 2) + 2 t + (i & 1) for accumulator element i, cbase = (column half of the warpgroup) * N / 2.
struct Frag {
  int r0, t, rh, ch;
  __device__ Frag(int tid) {
    const int warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    rh = wg & 1; ch = wg >> 1; t = lane & 3;
    r0 = 64 * rh + 16 * (warp & 3) + (lane >> 2);
  }
  __device__ int row(int i) const { return r0 + ((i & 2) ? 8 : 0); }
  __device__ int col(int i, int n_half) const { return ch * n_half + 8 * (i >> 2) + 2 * t + (i & 1); }
};

// D (+)= A * B^T over K = 64 as 3xTF32 for this warpgroup's 64 rows: the eight hi*hi products go to `m`, the sixteen
// lo*hi / hi*lo products (2^-11 times smaller, their truncation bias is negligible) to `c`; the caller adds the two.
// The tensor core adds into its accumulator with truncation, so a chain of n MMAs biases the sum by ~n 2^-24 towards
// zero: with all 24 products chained into one accumulator the filter came out several times less accurate than the
// reference's fp32 path.  a_* / b_* are the operand images already offset to this warpgroup's rows / columns.
template <int R>
__device__ __forceinline__ void layer_ss(float (&m)[R], float (&c)[R], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                         uint32_t b_lo, uint32_t acc0) {
  // four base descriptors, stepped by K (2 core matrices = 256 B = 16 descriptor units per k8 block): 32 precomputed
  // 64-bit descriptors would hold 64 registers and push the accumulators of the callers into local memory
  const uint64_t ah = make_desc_ls(a_hi, kLBO, kSBO), al = make_desc_ls(a_lo, kLBO, kSBO);
  const uint64_t bh = make_desc_ls(b_hi, kLBO, kSBO), bl = make_desc_ls(b_lo, kLBO, kSBO);
  constexpr uint64_t kStep = 2 * kLBO >> 4;
  wgmma_fence();
  fence_regs(m); fence_regs(c);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) wgmma_ss(m, ah + ks * kStep, bh + ks * kStep, (acc0 | ks) ? 1u : 0u);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    wgmma_ss(c, al + ks * kStep, bh + ks * kStep, (acc0 | ks) ? 1u : 0u);
    wgmma_ss(c, ah + ks * kStep, bl + ks * kStep, 1u);
  }
  wgmma_commit();
}
template <int R>
__device__ __forceinline__ void layer_wait(float (&m)[R], float (&c)[R]) {
  wgmma_wait<0>();
  fence_regs(m); fence_regs(c);
}

// hi / lo operand images of the activation pair (r, k), (r, k + 1), k even
__device__ __forceinline__ void store_pair_split(unsigned char* smem, int r, int k, float x0, float x1) {
  float2 hi, lo;
  split_tf32(x0, hi.x, lo.x);
  split_tf32(x1, hi.y, lo.y);
  const uint32_t off = op_off(r, k);
  *reinterpret_cast<float2*>(smem + kOffAhi + off) = hi;
  *reinterpret_cast<float2*>(smem + kOffAlo + off) = lo;
}
// all 16 fragment elements of a 64-column layer
__device__ __forceinline__ void store_frag16(unsigned char* smem, const Frag& f, const float (&a)[16]) {
#pragma unroll
  for (int i = 0; i < 16; i += 2) store_pair_split(smem, f.row(i), f.col(i, 32), a[i], a[i + 1]);
}
__device__ __forceinline__ uint32_t a_rows(uint32_t img, const Frag& f) { return img + (uint32_t)f.rh * 8u * kSBO; }

// ---------------------------------------------------------------------------------------------- prep
// Split the weights into tf32 hi/lo operand images (global memory, in shared-memory image order):
// [W1 hi][W1 lo][W2 hi][W2 lo] then per 128-channel half h: [W3_h hi][W3_h lo] (rows >= D are zero).
__global__ void filter_tc_prep_kernel(const float* __restrict__ W1, const float* __restrict__ W2,
                                      const float* __restrict__ W3, int D, float* __restrict__ wimg) {
  const int nh = (D + 127) / 128;
  const int total = 2 * kImgW64 + nh * kImgW128;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    float x;
    float* hi_img;
    float* lo_img;
    int r, k;
    if (i < 2 * kImgW64) {
      const int w = i / kImgW64, e = i % kImgW64;
      r = e / 64; k = e % 64;
      x = (w == 0 ? W1 : W2)[r * 64 + k];
      hi_img = wimg + w * 2 * kImgW64;
      lo_img = hi_img + kImgW64;
    } else {
      const int j = i - 2 * kImgW64, h = j / kImgW128, e = j % kImgW128;
      r = e / 64; k = e % 64;
      const int c = h * 128 + r;
      x = (c < D) ? W3[(size_t)c * 64 + k] : 0.f;
      hi_img = wimg + 4 * kImgW64 + (size_t)h * 2 * kImgW128;
      lo_img = hi_img + kImgW128;
    }
    float hi, lo;
    split_tf32(x, hi, lo);
    hi_img[op_off(r, k) / 4] = hi;
    lo_img[op_off(r, k) / 4] = lo;
  }
}

// ---------------------------------------------------------------------------------------------- forward
constexpr int kThreads = 512;

__global__ void __launch_bounds__(kThreads, 1)
filter_tc_fwd_kernel(const FilterParams P, const float* __restrict__ wimg, float* __restrict__ kout, int ntiles) {
  extern __shared__ __align__(1024) unsigned char smem[];
  float* misc = reinterpret_cast<float*>(smem + kOffMisc);
  float* W0s = misc;                    // [64][16]
  float* b0s = misc + 64 * 16;
  float* b1s = b0s + 64;
  float* b2s = b1s + 64;
  float* frs = b2s + 64;
  const int tid = threadIdx.x;
  const Frag f(tid);
  const uint32_t sbase = smem_u32(smem);
  const int nh = (P.D + 127) / 128;

  // ---- one-time setup: resident weights
  for (int i = tid; i < 4 * kImgW64 / 4; i += kThreads)   // W1/W2 hi/lo images: 64 KB, 16 bytes per cp.async
    cp_async16(smem + kOffW1hi + 16 * i, wimg + 4 * i, true);
  for (int i = tid; i < 64 * 16; i += kThreads) {
    const int r = i / 16, e = i % 16;
    W0s[i] = (e < P.E) ? __ldg(P.W0 + r * P.E + e) : 0.f;
  }
  if (tid < 64) {
    b0s[tid] = __ldg(P.b0 + tid); b1s[tid] = __ldg(P.b1 + tid); b2s[tid] = __ldg(P.b2 + tid);
    frs[tid] = __ldg(P.freq + tid);
  }
  cp_async_wait_all();
  __syncthreads();
  const uint32_t a_hi = a_rows(sbase + kOffAhi, f), a_lo = a_rows(sbase + kOffAlo, f);

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tb = tile * kTileM;
    // prefetch output-layer half 0 (the buffer is free: the MMAs that read it completed last tile)
    {
      const float* src = wimg + 4 * kImgW64;
      for (int i = tid; i < 2 * kImgW128 / 4; i += kThreads) cp_async16(smem + kOffW3hi + 16 * i, src + 4 * i, true);
    }
    // ---- layer 0 on the CUDA cores: a1 = sin(f * (W0 z + b0))
    {
      float a[16];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int t = tb + f.r0 + 8 * h;
        float z[kMaxE];
#pragma unroll
        for (int e = 0; e < kMaxE; ++e) z[e] = (t < P.L && e < P.E) ? __ldg(P.z + (size_t)t * P.z_stride + e) : 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          if (((i >> 1) & 1) != h) continue;
          const int c = f.col(i, 32);
          float acc = b0s[c];
#pragma unroll
          for (int e = 0; e < kMaxE; ++e) acc = fmaf(W0s[c * 16 + e], z[e], acc);
          a[i] = sin_acc(frs[c] * acc);
        }
      }
      store_frag16(smem, f, a);
    }
    fence_async_smem();
    __syncthreads();
    // ---- layers 1 and 2 on the tensor cores
#pragma unroll
    for (int layer = 0; layer < 2; ++layer) {
      float m[16], c[16];
      const uint32_t bh = sbase + (layer ? kOffW2hi : kOffW1hi) + (uint32_t)f.ch * 4u * kSBO;
      const uint32_t bl = sbase + (layer ? kOffW2lo : kOffW1lo) + (uint32_t)f.ch * 4u * kSBO;
      layer_ss(m, c, a_hi, a_lo, bh, bl, 0u);
      layer_wait(m, c);
      __syncthreads();                                   // every warpgroup has read the A images
      const float* bs = layer ? b2s : b1s;
      float a[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int col = f.col(i, 32);
        a[i] = sin_acc(frs[col] * ((m[i] + c[i]) + bs[col]));
      }
      store_frag16(smem, f, a);
      fence_async_smem();
      __syncthreads();
    }
    // ---- output layer, 128 channels at a time, modulation in the epilogue
    float tpos[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int t = tb + f.r0 + 8 * h;
      tpos[h] = t < P.L ? __ldg(P.t + t) : 0.f;
    }
    for (int hh = 0; hh < nh; ++hh) {
      cp_async_wait_all();                               // this thread's pieces of half hh have landed
      fence_async_smem();
      __syncthreads();
      float m[32], c[32];
      layer_ss(m, c, a_hi, a_lo, sbase + kOffW3hi + (uint32_t)f.ch * 8u * kSBO, sbase + kOffW3lo + (uint32_t)f.ch * 8u * kSBO, 0u);
      layer_wait(m, c);
      __syncthreads();                                   // the W3 buffer (and, after the last half, the A images) is free
      if (hh + 1 < nh) {                                 // stream the next half while this one is written out
        const float* src = wimg + 4 * kImgW64 + (size_t)(hh + 1) * 2 * kImgW128;
        for (int i = tid; i < 2 * kImgW128 / 4; i += kThreads) cp_async16(smem + kOffW3hi + 16 * i, src + 4 * i, true);
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int ch = hh * 128 + f.col(i, 64);
        const int h = (i >> 1) & 1;
        const int t = tb + f.r0 + 8 * h;
        if (ch < P.D && t < P.L) {
          float x = m[i] + c[i];
          if (P.modulate) x *= (expf(-tpos[h] * fabsf(__ldg(P.deltas + ch))) + P.shift);
          kout[(size_t)ch * P.L + t] = x;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- backward, stage 1
// Per 128-position tile, all GEMMs with M = positions (same fragment mapping and operand images as forward):
//   recompute pre1..3 / a1..3;  da3 = dh W3 (dh = dk * modulation, K = channels in chunks of 64);
//   dp3 = da3 f cos(f pre3);  da2 = dp3 W2;  dp2 = ...;  da1 = dp2 W1;  dp1 = ...
// and writes, feature-major (64, L): a1, a2, a3, dp1, dp2, dp3, X = sum_l da_l cos(f pre_l) pre_l, plus dh (D, L).
// Stage 2 (below) turns those into the parameter gradients with GEMMs whose reduction dimension is the sequence: dW3 = dh a3, dW2 = dp3^T a2, dW1 = dp2^T a1, dW0 = dp1^T z, db_l = colsum(dp_l),
// dfreq = colsum(X), dz = dp1 W0.
//
// Streamed operand images (global, built by filter_tc_prep_bwd_kernel), item i lives in stream buffer i & 1:
//   items 0..nq-1: W3^T chunk q  [64 features x 64 channels of chunk q];  item nq: W2^T;  item nq+1: W1^T
constexpr int kScratchArrays = 7;

__host__ __device__ constexpr size_t wimg_bwd_floats(int D) {
  return 4 * (size_t)kImgW64 + (size_t)((D + 63) / 64 + 2) * 2 * kImgW64;
}

__global__ void filter_tc_prep_bwd_kernel(const float* __restrict__ W1, const float* __restrict__ W2,
                                          const float* __restrict__ W3, int D, float* __restrict__ wimg) {
  const int nq = (D + 63) / 64;
  const int total = (2 + nq + 2) * kImgW64;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int item = i / kImgW64, e = i % kImgW64;
    const int r = e / 64, k = e % 64;
    float x;
    float* hi_img = wimg + (size_t)item * 2 * kImgW64;
    if (item == 0) x = W1[r * 64 + k];
    else if (item == 1) x = W2[r * 64 + k];
    else if (item < 2 + nq) {                  // W3^T chunk q: (feature r, channel k of the chunk)
      const int c = (item - 2) * 64 + k;
      x = (c < D) ? W3[(size_t)c * 64 + r] : 0.f;
    } else if (item == 2 + nq) x = W2[k * 64 + r];     // W2^T
    else x = W1[k * 64 + r];                           // W1^T
    float hi, lo;
    split_tf32(x, hi, lo);
    hi_img[op_off(r, k) / 4] = hi;
    hi_img[kImgW64 + op_off(r, k) / 4] = lo;
  }
}

__device__ __forceinline__ void stream_item(unsigned char* smem, const float* wimg, int item, int tid) {
  const float* src = wimg + (size_t)(2 + item) * 2 * kImgW64;
  unsigned char* dst = smem + kOffW3hi + (item & 1) * 32768;
  for (int i = tid; i < 2 * kImgW64 / 4; i += kThreads) cp_async16(dst + 16 * i, src + 4 * i, true);
}

// 16 fragment elements of one layer into a feature-major (64, L) array
__device__ __forceinline__ void store_feat16(float* arr, size_t L, const Frag& f, int tb, const float (&a)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int t = tb + f.row(i);
    if (t < (int)L) arr[(size_t)f.col(i, 32) * L + t] = a[i];
  }
}

__global__ void __launch_bounds__(kThreads, 1)
filter_tc_bwd_kernel(const FilterParams P, const float* __restrict__ wimg, const float* __restrict__ dk,
                     float* __restrict__ dh, float* __restrict__ scratch, int ntiles) {
  extern __shared__ __align__(1024) unsigned char smem[];
  float* misc = reinterpret_cast<float*>(smem + kOffMisc);
  float* W0s = misc;
  float* b0s = misc + 64 * 16;
  float* b1s = b0s + 64;
  float* b2s = b1s + 64;
  float* frs = b2s + 64;
  const int tid = threadIdx.x;
  const Frag f(tid);
  const uint32_t sbase = smem_u32(smem);
  const int nq = (P.D + 63) / 64;
  const size_t L = (size_t)P.L;
  const size_t arr = L * 64;                             // floats per scratch array

  for (int i = tid; i < 4 * kImgW64 / 4; i += kThreads) cp_async16(smem + kOffW1hi + 16 * i, wimg + 4 * i, true);
  for (int i = tid; i < 64 * 16; i += kThreads) {
    const int r = i / 16, e = i % 16;
    W0s[i] = (e < P.E) ? __ldg(P.W0 + r * P.E + e) : 0.f;
  }
  if (tid < 64) {
    b0s[tid] = __ldg(P.b0 + tid); b1s[tid] = __ldg(P.b1 + tid); b2s[tid] = __ldg(P.b2 + tid);
    frs[tid] = __ldg(P.freq + tid);
  }
  cp_async_wait_all();
  __syncthreads();
  const uint32_t a_hi = a_rows(sbase + kOffAhi, f), a_lo = a_rows(sbase + kOffAlo, f);
  const uint32_t bcol = (uint32_t)f.ch * 4u * kSBO;      // this warpgroup's 32 columns of a 64-row B image
  // Live across the dk chunk loop are only what the epilogues after it cannot get back cheaply: pre2, pre3, the
  // accumulators and the next chunk's dk.  The frequencies are read from shared memory at each use and pre1 (five FMAs
  // per element) is recomputed after the loop, in the same order, so that nothing spills at 128 registers.
  auto fr = [&](int i) { return frs[f.col(i, 32)]; };
  // pre1 = W0 z + b0 of fragment element i's row t (z of rows t >= L reads as zero)
  auto layer0 = [&](int i, const float (&z)[kMaxE]) {
    const int c = f.col(i, 32);
    float acc = b0s[c];
#pragma unroll
    for (int e = 0; e < kMaxE; ++e) acc = fmaf(W0s[c * 16 + e], z[e], acc);
    return acc;
  };
  auto load_z = [&](int t, float (&z)[kMaxE]) {
#pragma unroll
    for (int e = 0; e < kMaxE; ++e) z[e] = (t < P.L && e < P.E) ? __ldg(P.z + (size_t)t * P.z_stride + e) : 0.f;
  };

  // dk of chunk q is pulled into L2 while chunk q - 1's MMAs run (a register prefetch would spill)
  auto prefetch_dk = [&](int q, int tb) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int ch = q * 64 + f.col(i, 32), t = tb + f.row(i);
      if (ch < P.D && t < P.L) asm volatile("prefetch.global.L2 [%0];" ::"l"(dk + (size_t)ch * L + t));
    }
  };

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tb = tile * kTileM;
    prefetch_dk(0, tb);                                  // lands during the forward recompute
    stream_item(smem, wimg, 0, tid);
    stream_item(smem, wimg, 1, tid);

    // ---- forward recompute
    float pre2[16], pre3[16], a[16];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float z[kMaxE];
      load_z(tb + f.r0 + 8 * h, z);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (((i >> 1) & 1) != h) continue;
        a[i] = sin_acc(fr(i) * layer0(i, z));
      }
    }
    store_frag16(smem, f, a);
    store_feat16(scratch + 0 * arr, L, f, tb, a);
    fence_async_smem();
    __syncthreads();
    {
      float m[16], c[16];
      layer_ss(m, c, a_hi, a_lo, sbase + kOffW1hi + bcol, sbase + kOffW1lo + bcol, 0u);
      layer_wait(m, c);
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 16; ++i) { pre2[i] = (m[i] + c[i]) + b1s[f.col(i, 32)]; a[i] = sin_acc(fr(i) * pre2[i]); }
    }
    store_frag16(smem, f, a);
    store_feat16(scratch + 1 * arr, L, f, tb, a);
    fence_async_smem();
    __syncthreads();
    {
      float m[16], c[16];
      layer_ss(m, c, a_hi, a_lo, sbase + kOffW2hi + bcol, sbase + kOffW2lo + bcol, 0u);
      layer_wait(m, c);
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 16; ++i) { pre3[i] = (m[i] + c[i]) + b2s[f.col(i, 32)]; a[i] = sin_acc(fr(i) * pre3[i]); }
    }
    store_feat16(scratch + 2 * arr, L, f, tb, a);

    // ---- da3 = dh W3, 64 channels per MMA group; dh = dk * (exp(-t|delta|) + shift) also goes to HBM (stage 2 needs it)
    float tpos[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int t = tb + f.r0 + 8 * h;
      tpos[h] = t < P.L ? __ldg(P.t + t) : 0.f;
    }
    float m[16], c[16];
    for (int q = 0; q < nq; ++q) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int ch = q * 64 + f.col(i, 32), t = tb + f.row(i);
        float x = 0.f;
        if (ch < P.D && t < P.L) {
          x = __ldg(dk + (size_t)ch * L + t);
          if (P.modulate) x *= (expf(-tpos[(i >> 1) & 1] * fabsf(__ldg(P.deltas + ch))) + P.shift);
          dh[(size_t)ch * L + t] = x;
        }
        a[i] = x;
      }
      store_frag16(smem, f, a);                          // the previous MMA group has completed (waited below)
      cp_async_wait_all();
      fence_async_smem();
      __syncthreads();
      const uint32_t sb = sbase + kOffW3hi + (q & 1) * 32768;
      layer_ss(m, c, a_hi, a_lo, sb + bcol, sb + 16384u + bcol, q > 0 ? 1u : 0u);
      if (q + 1 < nq) prefetch_dk(q + 1, tb);
      layer_wait(m, c);
      __syncthreads();
      stream_item(smem, wimg, q + 2, tid);               // refill the buffer this group just released
    }

    // ---- layer 3 -> 2 -> 1 backward through the sine activations
    float X[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float cs = cos_acc(fr(i) * pre3[i]);
      const float g = (m[i] + c[i]) * cs;
      X[i] = g * pre3[i];
      a[i] = g * fr(i);
    }
    store_feat16(scratch + 5 * arr, L, f, tb, a);
    store_frag16(smem, f, a);
    cp_async_wait_all();
    fence_async_smem();
    __syncthreads();
    {                                                    // da2 = dp3 W2   (B = W2^T image, item nq)
      const uint32_t sb = sbase + kOffW3hi + (nq & 1) * 32768;
      layer_ss(m, c, a_hi, a_lo, sb + bcol, sb + 16384u + bcol, 0u);
      layer_wait(m, c);
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float cs = cos_acc(fr(i) * pre2[i]);
      const float g = (m[i] + c[i]) * cs;
      X[i] = fmaf(g, pre2[i], X[i]);
      a[i] = g * fr(i);
    }
    store_feat16(scratch + 4 * arr, L, f, tb, a);
    store_frag16(smem, f, a);
    fence_async_smem();
    __syncthreads();
    {                                                    // da1 = dp2 W1   (B = W1^T image, item nq+1)
      const uint32_t sb = sbase + kOffW3hi + ((nq + 1) & 1) * 32768;
      layer_ss(m, c, a_hi, a_lo, sb + bcol, sb + 16384u + bcol, 0u);
      layer_wait(m, c);
      __syncthreads();                                   // A images and stream buffers are free for the next tile
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float z[kMaxE];
      load_z(tb + f.r0 + 8 * h, z);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (((i >> 1) & 1) != h) continue;
        const float pre1 = layer0(i, z);
        const float cs = cos_acc(fr(i) * pre1);
        const float g = (m[i] + c[i]) * cs;
        X[i] = fmaf(g, pre1, X[i]);
        a[i] = g * fr(i);
      }
    }
    store_feat16(scratch + 3 * arr, L, f, tb, a);
    store_feat16(scratch + 6 * arr, L, f, tb, X);
  }
}

// ---------------------------------------------------------------------------------------------- backward, stage 2
// All parameter gradients of the filter are reductions over the sequence of the stage-1 arrays.  They run as three
// channel-major weight-gradient GEMMs (proj_gemm.cuh wgrad_ych_kernel: dW^T = sum_pos Y[n][pos] X[m][pos], 3xTF32,
// running sums in registers, fixed-order split-K partials), on operands the scratch order a1 a2 a3 dp1 dp2 dp3 X
// makes contiguous:
//   P1  X = dh (D rows),               Y = a3:          dW3[c][j] = T[j][c]
//   P2  X = [dp2; dp3] (128 rows),     Y = [a1; a2]:    dW1 = block (0, 0), dW2 = block (1, 1) (the off-diagonal blocks
//                                                        are not needed)
//   P3  X = [dp1; dp2; dp3; X],        Y = [zT; 1]:     dW0[j][e] = T[e][j], db0 / db1 / db2 / dfreq = T[E][64 l + j]
// then filter_red_finish_kernel sums each call's partials in split order and adds them into the gradients.
// [zT; 1] (E + 1, L) is built next to the partials by filter_red_ones_kernel.
__global__ void filter_red_ones_kernel(const float* __restrict__ zT, int E, int L, float* __restrict__ zt1) {
  const size_t nz = (size_t)E * L, total = nz + (size_t)L;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    zt1[i] = i < nz ? __ldg(zT + i) : 1.f;
}

struct RedFinish {
  const float* p1; const float* p2; const float* p3;   // (s1, 64, D), (s2, 128, 128), (s3, E + 1, 256) partials
  int s1, s2, s3;
  float* dW0; float* db0; float* dW1; float* db1; float* dW2; float* db2; float* dW3; float* dfreq;
  int D, E;
};

__device__ __forceinline__ float sum_splits(const float* p, size_t stride, int splits) {
  float s = 0.f;
  for (int k = 0; k < splits; ++k) s += __ldg(p + (size_t)k * stride);
  return s;
}

// one thread per gradient element: dW3 (D x 64), dW1, dW2 (64 x 64), dW0 (64 x E), db0, db1, db2, dfreq (64 each),
// numbered so that consecutive threads read consecutive partials
__global__ void filter_red_finish_kernel(const RedFinish r) {
  const int n3 = r.D * 64, n12 = 64 * 64, n0 = 64 * r.E;
  const int total = n3 + 2 * n12 + n0 + 4 * 64;
  const size_t st1 = (size_t)64 * r.D, st2 = 128 * 128, st3 = (size_t)(r.E + 1) * 256;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int q = i;
    if (q < n3) {
      const int j = q / r.D, c = q % r.D;
      r.dW3[c * 64 + j] += sum_splits(r.p1 + q, st1, r.s1);
      continue;
    }
    q -= n3;
    if (q < 2 * n12) {
      const int l = q / n12, k = (q % n12) / 64, j = q % 64;     // l = 0: dW1 = dp2 a1^T, l = 1: dW2 = dp3 a2^T
      (l ? r.dW2 : r.dW1)[j * 64 + k] += sum_splits(r.p2 + (size_t)(64 * l + k) * 128 + 64 * l + j, st2, r.s2);
      continue;
    }
    q -= 2 * n12;
    if (q < n0) {
      const int e = q / 64, j = q % 64;
      r.dW0[j * r.E + e] += sum_splits(r.p3 + (size_t)e * 256 + j, st3, r.s3);
      continue;
    }
    q -= n0;
    const int l = q / 64, j = q % 64;
    float* dst = l == 0 ? r.db0 : l == 1 ? r.db1 : l == 2 ? r.db2 : r.dfreq;
    dst[j] += sum_splits(r.p3 + (size_t)r.E * 256 + q, st3, r.s3);
  }
}

}  // namespace tc
}  // namespace hy
