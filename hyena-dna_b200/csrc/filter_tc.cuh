// Implicit filter (forward and backward) on the Hopper tensor cores (wgmma), sm_90a.
//
// Same math as filter_fwd_kernel (filter_mlp.cuh; reference src/models/sequence/hyena.py:96-155,199-238),
// but the three GEMM-shaped layers run as wgmma.mma_async ... .tf32 with fp32 accumulators in registers:
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
#include "filter_mlp.cuh"
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
  wgmma_fence();
  fence_regs(m); fence_regs(c);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    wgmma_ss(m, make_desc_ls(a_hi + ks * 2 * kLBO, kLBO, kSBO), make_desc_ls(b_hi + ks * 2 * kLBO, kLBO, kSBO), (acc0 | ks) ? 1u : 0u);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    wgmma_ss(c, make_desc_ls(a_lo + ks * 2 * kLBO, kLBO, kSBO), make_desc_ls(b_hi + ks * 2 * kLBO, kLBO, kSBO), (acc0 | ks) ? 1u : 0u);
    wgmma_ss(c, make_desc_ls(a_hi + ks * 2 * kLBO, kLBO, kSBO), make_desc_ls(b_lo + ks * 2 * kLBO, kLBO, kSBO), 1u);
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
// Stage 2 (host side, hyena-dna_b200/ops.py) turns those into the parameter gradients with GEMMs whose reduction
// dimension is the sequence: dW3 = dh a3, dW2 = dp3^T a2, dW1 = dp2^T a1, dW0 = dp1^T z, db_l = colsum(dp_l),
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
  float fr[16];                                          // this thread's frequencies
#pragma unroll
  for (int i = 0; i < 16; ++i) fr[i] = frs[f.col(i, 32)];

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tb = tile * kTileM;
    stream_item(smem, wimg, 0, tid);
    stream_item(smem, wimg, 1, tid);

    // ---- forward recompute
    float pre1[16], pre2[16], pre3[16], a[16];
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
        pre1[i] = acc;
        a[i] = sin_acc(fr[i] * acc);
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
      for (int i = 0; i < 16; ++i) { pre2[i] = (m[i] + c[i]) + b1s[f.col(i, 32)]; a[i] = sin_acc(fr[i] * pre2[i]); }
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
      for (int i = 0; i < 16; ++i) { pre3[i] = (m[i] + c[i]) + b2s[f.col(i, 32)]; a[i] = sin_acc(fr[i] * pre3[i]); }
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
    float nx[16];                                        // dk of the next chunk, loaded one MMA group ahead
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int ch = f.col(i, 32), t = tb + f.row(i);
      nx[i] = (ch < P.D && t < P.L) ? __ldg(dk + (size_t)ch * L + t) : 0.f;
    }
    for (int q = 0; q < nq; ++q) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int ch = q * 64 + f.col(i, 32), t = tb + f.row(i);
        float x = nx[i];
        if (ch < P.D && t < P.L) {
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
      if (q + 1 < nq) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int ch = (q + 1) * 64 + f.col(i, 32), t = tb + f.row(i);
          nx[i] = (ch < P.D && t < P.L) ? __ldg(dk + (size_t)ch * L + t) : 0.f;
        }
      }
      layer_wait(m, c);
      __syncthreads();
      stream_item(smem, wimg, q + 2, tid);               // refill the buffer this group just released
    }

    // ---- layer 3 -> 2 -> 1 backward through the sine activations
    float X[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float cs = cos_acc(fr[i] * pre3[i]);
      const float g = (m[i] + c[i]) * cs;
      X[i] = g * pre3[i];
      a[i] = g * fr[i];
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
      const float cs = cos_acc(fr[i] * pre2[i]);
      const float g = (m[i] + c[i]) * cs;
      X[i] = fmaf(g, pre2[i], X[i]);
      a[i] = g * fr[i];
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
    for (int i = 0; i < 16; ++i) {
      const float cs = cos_acc(fr[i] * pre1[i]);
      const float g = (m[i] + c[i]) * cs;
      X[i] = fmaf(g, pre1[i], X[i]);
      a[i] = g * fr[i];
    }
    store_feat16(scratch + 3 * arr, L, f, tb, a);
    store_feat16(scratch + 6 * arr, L, f, tb, X);
  }
}

// ---------------------------------------------------------------------------------------------- backward, stage 2
// All parameter gradients of the filter are reductions over the sequence.  With the stage-1 arrays stored feature-
// major every operand is K-major with K = position, so they are three accumulating wgmma GEMM groups whose fp32
// accumulators stay in registers (persistent CTAs, split over the sequence, an atomic flush every kRedChain K blocks):
//   G1  dW3[c][j]      = sum_t dh[c][t] a3[j][t]                       M = 128 channels per tile (<= 2 tiles), N = 64
//   G2  [dp3;dp2] x [a2;a1;1]^T : block(0,0) = dW2, block(1,1) = dW1, column 128 = (db2 ; db1)     M = 128, N = 144
//   G3  [dp1;X]  x [z;1]^T      : rows 0..63 -> (dW0 | db0), rows 64..127 col 8 -> dfreq             M = 128, N = 16
// K block = 32 positions (operand images: K-major, SBO 1024 B, LBO 128 B), 3xTF32 like everywhere else.
constexpr int kRedKB = 32;
constexpr int kRedThreads = 512;
constexpr int kRedItems = 12;                // ceil(8 * roundup8(256 + 7*64 + emb_dim) / 512)
constexpr uint32_t kRedSBO = 1024;
__host__ __device__ constexpr uint32_t red_off(int r, int k) {
  return (uint32_t)((r >> 3) * 1024 + (k >> 2) * 128 + (r & 7) * 16 + (k & 3) * 4);
}
constexpr uint32_t kRedImg128 = 128 * kRedKB * 4;      // bytes of a 128-row image (16 KB)
// shared memory map (bytes); every operand has a hi image followed by a lo image
constexpr uint32_t kRedOffDh = 0;                                  // 2 tiles x (hi 16K + lo 16K) = 64 KB
constexpr uint32_t kRedOffAs = 65536;                              // [dp3;dp2]   32 KB
constexpr uint32_t kRedOffAx = kRedOffAs + 32768;                  // [dp1;X]     32 KB
constexpr uint32_t kRedOffB3 = kRedOffAx + 32768;                  // a3 (64 rows): hi 8K + lo 8K
constexpr uint32_t kRedOffBs = kRedOffB3 + 16384;                  // [a2;a1;ones16] 144 rows: hi 18K + lo 18K
constexpr uint32_t kRedOffBz = kRedOffBs + 36864;                  // [z pad 8; ones 8] 16 rows: hi 2K + lo 2K
constexpr uint32_t kRedOffMisc = kRedOffBz + 4096;
constexpr size_t kRedSmemBytes = kRedOffMisc + 64;

// D (+)= A * B^T over one K block of 32 positions as 3xTF32, all products into one accumulator (restarted every
// kRedChain blocks, see below)
template <int R>
__device__ __forceinline__ void issue_red(float (&d)[R], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, uint32_t first_acc) {
  uint32_t acc = first_acc;
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    const uint32_t a = (pass == 1) ? a_lo : a_hi;
    const uint32_t b = (pass == 2) ? b_lo : b_hi;
#pragma unroll
    for (int ks = 0; ks < kRedKB / 8; ++ks) {
      wgmma_ss(d, make_desc_ls(a + ks * 2 * kLBO, kLBO, kRedSBO), make_desc_ls(b + ks * 2 * kLBO, kLBO, kRedSBO), acc);
      acc = 1;
    }
  }
}

// four consecutive positions of a feature row (zero beyond L); vector load when rows are 16-byte aligned
__device__ __forceinline__ float4 load4_row(const float* __restrict__ src, size_t t, size_t L, bool v4) {
  float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
  if (v4 && t + 3 < L) return __ldg(reinterpret_cast<const float4*>(src + t));
  if (t < L) x.x = __ldg(src + t);
  if (t + 1 < L) x.y = __ldg(src + t + 1);
  if (t + 2 < L) x.z = __ldg(src + t + 2);
  if (t + 3 < L) x.w = __ldg(src + t + 3);
  return x;
}

struct RedArgs {
  const float* dh;        // (D, L)
  const float* scratch;   // (7, 64, L): a1 a2 a3 dp1 dp2 dp3 X
  const float* zT;        // (E, L)
  float* dW0; float* db0; float* dW1; float* db1; float* dW2; float* db2; float* dW3; float* dfreq;
  int L, D, E;
};

// Work items: (row, 4-position piece) pairs, 8 pieces per row; item w = tid + kRedThreads*it, so every item of a thread
// has the same piece index (tid >> 3) & 7.  Inside every group of 64 items the ROW runs fastest (row = 8 (w >> 6) + (w & 7),
// piece = (w >> 3) & 7), so the eight lanes of a quarter warp write the eight 16-byte rows of ONE core matrix = 128
// contiguous bytes (conflict free), and a warp reads 64 contiguous bytes of each of eight rows.
struct RedItem { const float* src; uint32_t off; uint32_t lo_off; };
__device__ __forceinline__ RedItem red_item(const RedArgs& R, int it, int tid) {
  const size_t L = (size_t)R.L;
  const int nrow = R.D + 7 * 64 + R.E;                   // dh rows, six (64,L) arrays + X, z rows
  const int pc = (tid >> 3) & 7;
  const int row = (((tid + kRedThreads * it) >> 6) << 3) + (tid & 7);
  RedItem m{nullptr, 0u, 0u};
  uint32_t img = 0, lo = 0;
  int r = 0;
  if (row < R.D) {
    m.src = R.dh + (size_t)row * L; img = kRedOffDh + (row >> 7) * 32768; lo = 16384; r = row & 127;
  } else if (row < nrow) {
    const int q = row - R.D;
    if (q < 7 * 64) {
      const int arr = q >> 6, f = q & 63;                // scratch order: a1 a2 a3 dp1 dp2 dp3 X
      m.src = R.scratch + ((size_t)arr * 64 + f) * L;
      switch (arr) {
        case 0: img = kRedOffBs; lo = 18432; r = 64 + f; break;     // a1  -> B_s rows 64..127
        case 1: img = kRedOffBs; lo = 18432; r = f; break;          // a2  -> B_s rows 0..63
        case 2: img = kRedOffB3; lo = 8192; r = f; break;           // a3
        case 3: img = kRedOffAx; lo = 16384; r = f; break;          // dp1 -> A_x rows 0..63
        case 4: img = kRedOffAs; lo = 16384; r = 64 + f; break;     // dp2 -> A_s rows 64..127
        case 5: img = kRedOffAs; lo = 16384; r = f; break;          // dp3 -> A_s rows 0..63
        default: img = kRedOffAx; lo = 16384; r = 64 + f; break;    // X   -> A_x rows 64..127
      }
    } else {
      const int e = q - 7 * 64;                          // z feature e -> B_z row e
      m.src = R.zT + (size_t)e * L; img = kRedOffBz; lo = 2048; r = e;
    }
  }
  m.off = img + red_off(r, 4 * pc);
  m.lo_off = lo;
  return m;
}

// K blocks per accumulator chain.  The tensor core truncates every add into its accumulator, so a chain of n MMAs biases
// the sum towards zero by ~n 2^-24 of its magnitude: one chain through a CTA's whole slice of a 2^20-position sequence
// (~250 blocks x 12 MMAs) put same-sign sums 8.5e-5 (relative) off, 100x the error of an fp32 library GEMM.  So every
// kRedChain blocks the accumulators are flushed into the gradients with round-to-nearest atomic adds and restarted.
// Shorter chains trade the bias for more atomic adds per gradient element (their own rounding) and time: on an H100
// (400 W) at L = 2^20, D = 256 the kernel took 5.4 ms with one chain, 5.65 ms with 8 blocks, 6.0 ms with 4, 7.3 ms with 2.
constexpr int kRedChain = 8;

// accumulators -> gradients (fragment element i: row f.row(i) of the group, column f.col(i, n_half))
__device__ __forceinline__ void red_flush(const RedArgs& R, const Frag& f, int nmt, const float (&g1)[2][16],
                                          const float (&g2)[36], const float (&g3)[4]) {
  for (int mt = 0; mt < nmt; ++mt) {                       // G1: dW3 rows c = 128 mt + row, 64 columns
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int c = mt * 128 + f.row(i);
      if (c < R.D) atomicAdd(R.dW3 + (size_t)c * 64 + f.col(i, 32), g1[mt][i]);
    }
  }
  // G2: rows < 64: cols 0..63 -> dW2[row][j]; rows >= 64: cols 64..127 -> dW1[row-64][j]; col 128 -> db2 / db1
#pragma unroll
  for (int i = 0; i < 36; ++i) {
    const int r = f.row(i), n = f.col(i, 72);
    if (n == 128) atomicAdd(((r < 64) ? R.db2 : R.db1) + (r & 63), g2[i]);
    else if (r < 64 && n < 64) atomicAdd(R.dW2 + r * 64 + n, g2[i]);
    else if (r >= 64 && n >= 64 && n < 128) atomicAdd(R.dW1 + (r - 64) * 64 + (n - 64), g2[i]);
  }
  // G3: rows < 64: cols 0..E-1 -> dW0[row][e], col 8 -> db0[row]; rows >= 64: col 8 -> dfreq[row-64]
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = f.row(i), n = f.col(i, 8);
    if (r < 64) {
      if (n < R.E) atomicAdd(R.dW0 + r * R.E + n, g3[i]);
      else if (n == 8) atomicAdd(R.db0 + r, g3[i]);
    } else if (n == 8) {
      atomicAdd(R.dfreq + (r - 64), g3[i]);
    }
  }
}

__global__ void __launch_bounds__(kRedThreads, 1) filter_tc_red_kernel(const RedArgs R, int nblocks) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x;
  const Frag f(tid);
  const uint32_t sbase = smem_u32(smem);
  const int nmt = (R.D + 127) / 128;                       // channel tiles (host guarantees <= 2)
  const size_t L = (size_t)R.L;
  const bool v4 = (R.L & 3) == 0;
  const int pc = (tid >> 3) & 7;

  // zero every image once (rows that are never loaded -- channel padding, z padding -- stay zero), then the ones rows
  for (uint32_t i = tid; i < kRedOffMisc / 16; i += kRedThreads) reinterpret_cast<float4*>(smem)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  for (int i = tid; i < 16 * kRedKB; i += kRedThreads) {   // [a2;a1;ones16]: rows 128..143 hi = 1
    const int r = 128 + i / kRedKB, k = i % kRedKB;
    *reinterpret_cast<float*>(smem + kRedOffBs + red_off(r, k)) = 1.f;
  }
  for (int i = tid; i < 8 * kRedKB; i += kRedThreads) {    // [z;ones8]: rows 8..15 hi = 1
    const int r = 8 + i / kRedKB, k = i % kRedKB;
    *reinterpret_cast<float*>(smem + kRedOffBz + red_off(r, k)) = 1.f;
  }
  __syncthreads();

  // accumulators of this warpgroup: rows 64 rh .. of every group, column half ch
  float g1[2][16], g2[36], g3[4];
  const uint32_t arow = (uint32_t)f.rh * 8u * kRedSBO;
  bool first = true;                                       // no MMA issued yet
  int chain = 0;                                           // K blocks in the accumulators since their last flush
  for (int blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
    const size_t t = (size_t)blk * kRedKB + 4 * pc;
    if (!first) {                                          // previous MMAs have read the images
      wgmma_wait<0>();
      fence_regs(g1[0]); fence_regs(g1[1]); fence_regs(g2); fence_regs(g3);
      __syncthreads();
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      constexpr int kH = kRedItems / 2;
      float4 x[kH];
      RedItem m[kH];
#pragma unroll
      for (int j = 0; j < kH; ++j) {                       // all loads of this half block in flight at once
        m[j] = red_item(R, half * kH + j, tid);
        x[j] = m[j].src ? load4_row(m[j].src, t, L, v4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < kH; ++j) {
        if (m[j].src) {
          float4 hi, lo;
          split_tf32(x[j].x, hi.x, lo.x); split_tf32(x[j].y, hi.y, lo.y);
          split_tf32(x[j].z, hi.z, lo.z); split_tf32(x[j].w, hi.w, lo.w);
          *reinterpret_cast<float4*>(smem + m[j].off) = hi;
          *reinterpret_cast<float4*>(smem + m[j].off + m[j].lo_off) = lo;
        }
      }
    }
    fence_async_smem();
    __syncthreads();
    const uint32_t acc0 = chain ? 1u : 0u;
    wgmma_fence();
    fence_regs(g1[0]); fence_regs(g1[1]); fence_regs(g2); fence_regs(g3);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
      if (mt < nmt)
        issue_red(g1[mt], sbase + kRedOffDh + mt * 32768 + arow, sbase + kRedOffDh + mt * 32768 + 16384 + arow,
                  sbase + kRedOffB3 + f.ch * 4 * kRedSBO, sbase + kRedOffB3 + 8192 + f.ch * 4 * kRedSBO, acc0);
    issue_red(g2, sbase + kRedOffAs + arow, sbase + kRedOffAs + 16384 + arow, sbase + kRedOffBs + f.ch * 9 * kRedSBO,
              sbase + kRedOffBs + 18432 + f.ch * 9 * kRedSBO, acc0);
    issue_red(g3, sbase + kRedOffAx + arow, sbase + kRedOffAx + 16384 + arow, sbase + kRedOffBz + f.ch * kRedSBO,
              sbase + kRedOffBz + 2048 + f.ch * kRedSBO, acc0);
    wgmma_commit();
    first = false;
    if (++chain == kRedChain) {                            // the images stay untouched until the barrier at the loop top
      wgmma_wait<0>();
      fence_regs(g1[0]); fence_regs(g1[1]); fence_regs(g2); fence_regs(g3);
      red_flush(R, f, nmt, g1, g2, g3);
      chain = 0;
    }
  }
  if (chain == 0) return;
  wgmma_wait<0>();
  fence_regs(g1[0]); fence_regs(g1[1]); fence_regs(g2); fence_regs(g3);
  red_flush(R, f, nmt, g1, g2, g3);
}

}  // namespace tc
}  // namespace hy
