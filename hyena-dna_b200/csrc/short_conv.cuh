// Backward of the 3-tap depthwise short filter (src/models/sequence/hyena.py:363-369, :394).
//
// Forward (fused into the FFT column passes): s[t] = w0 P(t-2) + w1 P(t-1) + w2 P(t) + b for t in [0,L),
// P(t) = p[t] + in_bias inside [0,L) and 0 outside (p = in_proj output before its bias).
// Backward, given ds = d loss / d s  (B,3D,L):
//   dp[t]  = w2 ds[t] + w1 ds[t+1] + w0 ds[t+2]          (ds[t>=L] = 0)
//   dw_j   = sum_{b,t} ds[t] P(t-2+j),  db = sum ds,  d in_bias = sum dp
// Left-padded rows (row_start non-null, short_conv_bwd_rows_kernel): positions t < row_start[b] are padding that the forward
// zeroed before the filter, so dp is 0 there (the transposed filter would carry ds[rs], ds[rs+1] into rs-1, rs-2) and they
// stay out of d in_bias; a pad sample of a window reads 0.
// Packed sequences (seg_base non-null, short_conv_bwd_packed_kernel): row b is one sequence of the packed (3D, total) ds and
// dp, addressed as in the *_PACKED FFT modes.  ds is read and dp written at t >= row_start[b] only, so the transposed filter
// stops at the sequence's last position and nothing of the previous sequence is touched.  dsw / dsb come from pass 3.
#pragma once
#include "fft_passes.cuh"

namespace hy {

constexpr int kScSpan = 8192;     // positions per CTA

struct ShortBwdArgs {
  const float* ds;      // (B,3D,L)
  const float* p;       // (B,3D,L), or null when dsw / dsb were already accumulated by pass 3
  const float* in_bias; // (3D) or null
  const float* sw;      // (3D,3)
  float* dp;            // (B,3D,L)
  float* dsw;           // (3D,3)  atomicAdd
  float* dsb;           // (3D)    atomicAdd
  float* dib;           // (3D)    atomicAdd (d in_proj.bias) or null
  int L, C3, vec;
  const int* row_start; // (B) first real position of each row, or null (plain kernel)
  const long long* seg_base;   // (B) packed sequences: offset of row b's position 0 in a channel, or null
  long long cstride;           // packed sequences: channel stride (total positions)
};

#ifdef HY_FILTER_KERNEL_TU
template <bool ROWS>
__device__ __forceinline__ void short_conv_bwd_body(const ShortBwdArgs& a) {
  const int ch = blockIdx.y, b = blockIdx.z;
  const int L = a.L;
  const bool vec = a.vec;
  const float* ds = a.ds + row_off(b, ch, a.C3, L);
  const float* p = a.p ? a.p + row_off(b, ch, a.C3, L) : nullptr;
  float* dp = a.dp + row_off(b, ch, a.C3, L);
  const float w0 = __ldg(a.sw + 3 * ch), w1 = __ldg(a.sw + 3 * ch + 1), w2 = __ldg(a.sw + 3 * ch + 2);
  const float ib = a.in_bias ? __ldg(a.in_bias + ch) : 0.f;
  [[maybe_unused]] int rs = 0;
  if constexpr (ROWS) rs = __ldg(a.row_start + b);
  float r[5] = {0.f, 0.f, 0.f, 0.f, 0.f};      // dw0, dw1, dw2, db, dib
  const int tbeg = blockIdx.x * kScSpan;
  const int tend = min(L, tbeg + kScSpan);
  for (int t0 = tbeg + 2 * threadIdx.x; t0 < tend; t0 += 512) {
    float2 d0 = load_pair(ds, t0, L, vec);
    float2 d1 = (t0 + 2 < L) ? load_pair(ds, t0 + 2, L, vec) : make_float2(0.f, 0.f);
    float2 o;
    o.x = fmaf(w2, d0.x, fmaf(w1, d0.y, w0 * d1.x));
    o.y = fmaf(w2, d0.y, fmaf(w1, d1.x, w0 * d1.y));
    if constexpr (ROWS) o = mask_pair(o, t0, rs);
    store_pair(dp, t0, L, vec, o);
    if (a.p) {
      float P[4];
      load_window(p, t0, L, vec, ib, P);
      if constexpr (ROWS) mask_window(P, t0, rs);
      r[0] = fmaf(d0.x, P[0], fmaf(d0.y, P[1], r[0]));
      r[1] = fmaf(d0.x, P[1], fmaf(d0.y, P[2], r[1]));
      r[2] = fmaf(d0.x, P[2], fmaf(d0.y, P[3], r[2]));
      r[3] += d0.x + d0.y;
    }
    r[4] += o.x + ((t0 + 1 < L) ? o.y : 0.f);
  }
  __shared__ float red[8][5];
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    float s = r[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][j] = s;
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    if (threadIdx.x < 3) { if (a.p) atomicAdd(a.dsw + 3 * ch + threadIdx.x, s); }
    else if (threadIdx.x == 3) { if (a.p) atomicAdd(a.dsb + ch, s); }
    else if (a.dib) atomicAdd(a.dib + ch, s);
  }
}

__global__ void __launch_bounds__(256) short_conv_bwd_packed_kernel(const ShortBwdArgs a) {
  const int ch = blockIdx.y, b = blockIdx.z;
  const int L = a.L;
  const int rs = __ldg(a.row_start + b);
  const int tbeg = blockIdx.x * kScSpan;
  const int tend = min(L, tbeg + kScSpan);
  if (tend <= rs) return;                      // the whole span is before the sequence (uniform per CTA)
  const long long off = __ldg(a.seg_base + b) + (long long)ch * a.cstride;
  const float* ds = a.ds + off;
  float* dp = a.dp + off;
  const float w0 = __ldg(a.sw + 3 * ch), w1 = __ldg(a.sw + 3 * ch + 1), w2 = __ldg(a.sw + 3 * ch + 2);
  float r = 0.f;                               // d in_bias
  for (int t0 = tbeg + 2 * threadIdx.x; t0 < tend; t0 += 512) {
    if (t0 + 1 < rs) continue;
    const float2 d0 = load_pair_seg(ds, t0, L, rs);
    const float2 d1 = (t0 + 2 < L) ? load_pair_seg(ds, t0 + 2, L, rs) : make_float2(0.f, 0.f);
    float2 o;
    o.x = fmaf(w2, d0.x, fmaf(w1, d0.y, w0 * d1.x));
    o.y = fmaf(w2, d0.y, fmaf(w1, d1.x, w0 * d1.y));
    o = mask_pair(o, t0, rs);
    store_pair_seg(dp, t0, L, rs, o);
    r += o.x + ((t0 + 1 < L) ? o.y : 0.f);
  }
  if (!a.dib) return;
  __shared__ float red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = r;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w];
    atomicAdd(a.dib + ch, s);
  }
}

__global__ void __launch_bounds__(256) short_conv_bwd_kernel(const ShortBwdArgs a) { short_conv_bwd_body<false>(a); }
__global__ void __launch_bounds__(256) short_conv_bwd_rows_kernel(const ShortBwdArgs a) { short_conv_bwd_body<true>(a); }

#endif  // HY_FILTER_KERNEL_TU

}  // namespace hy
