// Extending a decode cache by n >= 1 positions at once (chunked prefill, continuation scoring).
//
// Output j of a chunk that starts at position t is, per recurrence o (decode.cuh for one position):
//     out_o[t+j] = sum_{s<=t+j} k_o[t+j-s] g_o[s] + bias_o g_o[t+j],      g_o = v_o * x_{O-1-o},
// a Toeplitz product of the whole history g_o[0, t+n) (the chunk's own g_o included) with the filter.
//   decode_ext_hist_kernel     the 3-tap short filter of the n positions for all (O+1) D in_proj channels, carried in from
//                              the cache's tail; g_0 into h[0][t, t+n); the tail shifted to the last two positions
//   decode_ext_dot_kernel      direct Toeplitz product, split into partial sums over 1024-position chunks: a CTA stages the
//                              history chunk of up to 8 batch rows and the filter window (chunk + tile taps) in shared
//                              memory, so both are read once per launch; each thread keeps an 8-output register block
//   decode_ext_combine_kernel  fixed-order sum of the partials (or the FFT route's convolution), + bias g, the gates:
//                              g_{o+1} into the next recurrence's history, or y_pre = out * x_0 after the last recurrence
//   decode_branch_combine_kernel the combine of a branched cache: + the parent row's F[t-b+j] (decode_args.h); the hist and
//                              dot kernels run unchanged on a branch's history row with shifted arguments
// fp32 arithmetic, no atomics: every sum has a fixed order for a given (B, D, t, n), so an extend is bitwise reproducible.
// The kernels that touch the history are templates over its element type T (decode.cuh): stores round, reads widen.
#pragma once
#include <cuda_runtime.h>

#include "decode_args.h"
#include "decode_common.cuh"

namespace hy {
namespace dec {

// one CTA per (b, d): channels d, D + d, ..., O D + d of positions [t, t+n)
template <class T>
__global__ void __launch_bounds__(256) decode_ext_hist_kernel(const ExtHistArgsT<T> a) {
  const int row = blockIdx.x;                    // b * D + d
  const int b = row / a.D, d = row - b * a.D;
  const int nj = a.C / a.D;
  for (int idx = threadIdx.x; idx < nj * a.n; idx += blockDim.x) {
    const int i = idx / a.n, j = idx - i * a.n;
    const int c = i * a.D + d;
    const size_t bc = (size_t)b * a.C + c;
    const float* pc = a.p + bc * a.n;
    const float ib = a.in_bias ? __ldg(a.in_bias + c) : 0.f;
    const float* tl = a.tail + bc * 2;
    const float pm2 = j >= 2 ? pc[j - 2] + ib : tl[j];          // j = 0, 1: positions t-2, t-1 come from the tail
    const float pm1 = j >= 1 ? pc[j - 1] + ib : tl[1];
    a.s[bc * a.n + j] = short3(__ldg(a.sw + 3 * c), __ldg(a.sw + 3 * c + 1), __ldg(a.sw + 3 * c + 2), __ldg(a.sb + c), pm2,
                               pm1, pc[j] + ib);
  }
  __syncthreads();                               // every read of the tail is done; s of this row is visible to the CTA
  const float* sv = a.s + ((size_t)b * a.C + a.C - a.D + d) * a.n;
  const float* sg = a.s + ((size_t)b * a.C + a.gate + d) * a.n;
  T* h = a.h + (size_t)row * a.ld + a.t;
  for (int j = threadIdx.x; j < a.n; j += blockDim.x) h[j] = hround<T>(sv[j] * sg[j]);
  if ((int)threadIdx.x < nj) {
    const int c = threadIdx.x * a.D + d;
    const size_t bc = (size_t)b * a.C + c;
    const float* pc = a.p + bc * a.n;
    const float ib = a.in_bias ? __ldg(a.in_bias + c) : 0.f;
    float* tl = a.tail + bc * 2;
    const float t0 = a.n >= 2 ? pc[a.n - 2] + ib : tl[1];
    tl[0] = t0;
    tl[1] = pc[a.n - 1] + ib;
  }
}

// shared-memory index with one pad word per 32: lanes that walk consecutive positions from starts 4 or 32 words apart hit
// distinct banks
__device__ __forceinline__ int sk(int x) { return x + (x >> 5); }

// part[b][d][j][g] = sum over the chunks of group g, s <= t+j, of h[b][d][s] k[t+j-s]   for the outputs of tile
// [j0, j0 + NT) and the batch rows [z*BG, z*BG + BG).
//
// Within a 1024-position chunk starting at s0, output j0 + r at position s0 + q takes the tap m = t + j0 - s0 + r - q, stored
// reversed at krev[ld-1-m].  The window staged in shared memory is krev[A4 .. A4 + kChunk + NT + 4) with
// A4 = ld - t - j0 + s0 - NT - R, which is 16-byte aligned for R = (-t) mod 4 (the misaligned offset of decode_dot_kernel:
// here it is folded into the shared-memory index instead of funnelling registers), so that tap sits at window index
// q + NT - 1 - r + R.  Taps with m < 0 (s > t + j: not yet causal) fall past the row end and are staged as zeros.
//
// Thread layout: warp w serves the 8-output column jc = w / WPC (WPC = 8 / (NT/8) warps per column); its lanes split the
// chunk into consecutive runs of QL positions.  Along a run the 8 taps a lane needs slide by one per position: one new
// shared-memory load per position feeds 8 * BG FMAs.  The lanes' sums are reduced by a butterfly, the column's warps in a
// fixed order through shared memory.
template <int BG, int NT, class T>
__global__ void __launch_bounds__(32 * kExtWarps, 1) decode_ext_dot_kernel(const ExtDotArgsT<T> a) {
  constexpr int RJ = kExtRJ;
  constexpr int JT = NT / RJ;
  constexpr int WPC = kExtWarps / JT;
  constexpr int QL = kChunk / (32 * WPC);
  constexpr int WS = kChunk + NT + 4;
  static_assert(JT * WPC == kExtWarps && QL * 32 * WPC == kChunk, "tile shape");
  __shared__ float hs[BG][kChunk + kChunk / 32];
  __shared__ float ws[WS + WS / 32 + 1];
  __shared__ float red[WPC > 1 ? BG * RJ : 1][kExtWarps];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int jc = warp / WPC, wq = warp - jc * WPC;
  const int qa = (wq * 32 + lane) * QL;
  const int cb = NT - 1 - jc * RJ + a.R;
  const int d = blockIdx.y, b0 = blockIdx.z * BG;
  const int g = blockIdx.x / a.njt, j0 = (blockIdx.x - g * a.njt) * NT;
  const int L = a.t + a.n;
  const float* krow = a.k + (size_t)d * a.kstride;

  float acc[BG][RJ];
#pragma unroll
  for (int i = 0; i < BG; ++i)
#pragma unroll
    for (int r = 0; r < RJ; ++r) acc[i][r] = 0.f;

  const int c_end = min((g + 1) * a.cpb, a.nchunk);
  for (int c = g * a.cpb; c < c_end; ++c) {
    const int s0 = c * kChunk;
    if (s0 > a.t + j0 + NT - 1) break;           // every tap of this tile at these positions is causally masked
    __syncthreads();                             // the previous chunk's readers are done
    for (int v = threadIdx.x; v < BG * (kChunk / 4); v += blockDim.x) {
      const int i = v / (kChunk / 4), q = (v - i * (kChunk / 4)) * 4;
      const int b = b0 + i, s = s0 + q;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b < a.B && s < L) {                    // s < L <= ld, ld % 4 == 0: the whole vector lies inside the row
        x = hld4(a.h + ((size_t)b * a.D + d) * a.ld + s);
        if (s + 4 > L) {                         // positions >= t + n hold no history yet
          x.y = s + 1 < L ? x.y : 0.f;
          x.z = s + 2 < L ? x.z : 0.f;
          x.w = 0.f;
        }
      }
      hs[i][sk(q)] = x.x; hs[i][sk(q + 1)] = x.y; hs[i][sk(q + 2)] = x.z; hs[i][sk(q + 3)] = x.w;
    }
    const long long A4 = (long long)a.ld - a.t - j0 + s0 - NT - a.R;
    for (int v = threadIdx.x; v < WS / 4; v += blockDim.x) {
      const long long idx = A4 + 4 * v;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx >= 0 && idx < a.ld) x = ld4(krow + idx);
      ws[sk(4 * v)] = x.x; ws[sk(4 * v + 1)] = x.y; ws[sk(4 * v + 2)] = x.z; ws[sk(4 * v + 3)] = x.w;
    }
    __syncthreads();
    float wv[RJ];                                // wv[r] = tap of output jc*RJ + r at position qa + q
#pragma unroll
    for (int r = 0; r < RJ; ++r) wv[r] = ws[sk(qa + cb - r)];
#pragma unroll
    for (int q = 0; q < QL; ++q) {
#pragma unroll
      for (int i = 0; i < BG; ++i) {
        const float hv = hs[i][sk(qa + q)];
#pragma unroll
        for (int r = 0; r < RJ; ++r) acc[i][r] = fmaf(hv, wv[r], acc[i][r]);
      }
      if (q + 1 < QL) {
#pragma unroll
        for (int r = RJ - 1; r > 0; --r) wv[r] = wv[r - 1];
        wv[0] = ws[sk(qa + q + 1 + cb)];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < BG; ++i)
#pragma unroll
    for (int r = 0; r < RJ; ++r)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[i][r] += __shfl_xor_sync(0xffffffffu, acc[i][r], o);
  if constexpr (WPC == 1) {
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < BG; ++i)
#pragma unroll
        for (int r = 0; r < RJ; ++r) {
          const int b = b0 + i, j = j0 + jc * RJ + r;
          if (b < a.B && j < a.n) a.part[(((size_t)b * a.D + d) * a.n + j) * a.groups + g] = acc[i][r];
        }
    }
  } else {                                       // one column (JT == 1): its 8 warps in a fixed order
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < BG; ++i)
#pragma unroll
        for (int r = 0; r < RJ; ++r) red[i * RJ + r][warp] = acc[i][r];
    }
    __syncthreads();
    if ((int)threadIdx.x < BG * RJ) {
      const int i = threadIdx.x / RJ, r = threadIdx.x - i * RJ;
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kExtWarps; ++w) s += red[threadIdx.x][w];
      const int b = b0 + i, j = j0 + r;
      if (b < a.B && j < a.n) a.part[(((size_t)b * a.D + d) * a.n + j) * a.groups + g] = s;
    }
  }
}

// fixed-order sum of the partials of output j of one (b, channel) row
template <class T>
__device__ __forceinline__ float ext_partial_sum(const ExtCombineArgsT<T>& a, int row, int j) {
  const float* pp = a.part + (size_t)row * a.prow + (size_t)j * a.pj;
  float acc = 0.f;
  for (int g = 0; g < a.groups; ++g) acc += pp[g];
  return acc;
}

// everything of output j once acc = sum_{s<t+j} k[t+j-s] g[s] is known: + bias g, times the gate, into h_next or y
template <class T>
__device__ __forceinline__ void ext_combine_epilogue(const ExtCombineArgsT<T>& a, int row, int b, int d, int j, float acc) {
  const float gv = hwiden(a.h[(size_t)row * a.ld + a.t + j]);
  const float y = fmaf(__ldg(a.fbias + (size_t)d * a.fstride), gv, acc);
  const float x = a.s[((size_t)b * a.C + a.xch + d) * a.n + j];
  if (a.last) a.y[(size_t)row * a.n + j] = y * x;
  else a.h_next[(size_t)row * a.ld + a.t + j] = hround<T>(y * x);
}

// one thread per (b, d, j)
template <class T>
__global__ void __launch_bounds__(256) decode_ext_combine_kernel(const ExtCombineArgsT<T> a) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.B * a.D * a.n) return;
  const int row = (int)(idx / a.n), j = (int)(idx - (long long)row * a.n);
  const int b = row / a.D, d = row - b * a.D;
  ext_combine_epilogue(a, row, b, d, j, ext_partial_sum(a, row, j));
}

// the combine of a branched cache (decode_args.h BranchCombineArgs): the partials over the branch's positions [b, t+j), then
// F[parent[row b]][d][t-b+j] (the shared context before b), then the same epilogue; one thread per (b, d, j)
template <class T>
__global__ void __launch_bounds__(256) decode_branch_combine_kernel(const BranchCombineArgsT<T> w) {
  const ExtCombineArgsT<T>& a = w.c;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.B * a.D * a.n) return;
  const int row = (int)(idx / a.n), j = (int)(idx - (long long)row * a.n);
  const int b = row / a.D, d = row - b * a.D;
  const float* f = w.f + ((size_t)__ldg(w.parent + b) * a.D + d) * a.ld;
  ext_combine_epilogue(a, row, b, d, j, ext_partial_sum(a, row, j) + f[a.t + j]);
}

}  // namespace dec
}  // namespace hy
