// Incremental decoding of the causal Hyena operator: one output position at a time from a cached history.
//
// Output t of a causal recurrence (src/models/sequence/hyena.py:414-423 with fftconv_ref, :59-88) is
//     out[t] = sum_{s<=t} k[t-s] g[s] + bias g[t],      g = v * x_gate (short-filtered in_proj channels),
// so a step is one dot product per (b, channel) over the stored history g[0..t) plus O(1) work at position t.
//   decode_hist_kernel     after a prefill of P positions: g[0..P) of recurrence 0 and the short-filter tail
//   decode_admit_kernel    the same for prompts placed into chosen rows of a running cache so that they end at its position
//                          (PACKED: prompts packed back to back, cu_seqlens; also a packed prefill at t = P into rows 0..N-1)
//   decode_shift_kernel    in-place shift of every history row by a multiple of 4 positions (compaction, room for a prompt)
//   decode_dot_kernel      split over positions: one warp per (1024-position chunk, channel), each k row read once for
//                          all batch rows of its group; the filter is stored time-reversed so that h and k both stream in
//                          ascending order (k[t-s] = krev[ld-1-t+s]); the k offset's misalignment R = (ld-1-t) mod 4 is a
//                          template parameter: two aligned float4 loads are funnelled into the four values a lane needs
//   decode_step_kernel     one warp per (b, channel): fixed-order reduction of the chunk partials, the short filter of
//                          position t from the tail (recurrence 0), the gates, g[t] into the history, the epilogue
//   decode_win_step_kernel decode_step_kernel inside an open window [b, b + Wc): the partials cover only [b, t) (the dot
//                          kernel run on h + b with t - b) and the precomputed F[t-b] = sum_{s<b} k[t-s] g[s] is added
//   decode_branch_step_kernel the same for a branched cache (decode_args.h BranchStepArgs): each batch row is a branch with
//                          its own history from b on, and F is read from the row of the branch's parent
//   *_dev_kernel           the same steps with the position read on the device (decode_args.h DevPos), for a step captured
//                          once in a CUDA graph and replayed at every position; decode_pos_advance_kernel moves it
// fp32 arithmetic, no atomics: every sum has a fixed order, so a step is bitwise reproducible.  Every kernel that reads or
// writes the history is a template over its element type T (float, __half, __nv_bfloat16; decode_args.h): a value is
// rounded once when it is stored, g^ = round(g), and every read and the step's own s = t term use g^ widened to fp32.
#pragma once
#include <cuda_runtime.h>

#include "decode_args.h"
#include "decode_common.cuh"

namespace hy {
namespace dec {

// g[t] = short(v)[t] * short(x_gate)[t] for t < P into h (row stride ld); tail = P(P-2), P(P-1) of every channel.
// ROWS: row b is left-padded, its positions t < s = row_start[b] read as the short filter's padding before t = 0 (0, no
// in_proj bias): g is 0 there, and a pad position in the tail is 0.
// Grid: (B * D rows, up to 64 position CTAs per row); the rows go on x, which has no 65535 limit.
template <bool ROWS, class T>
__device__ __forceinline__ void hist_body(const HistArgsT<T>& a) {
  const int row = blockIdx.x;                    // b * D + d
  const int b = row / a.D, d = row - b * a.D;
  const int s = ROWS ? __ldg(a.row_start + b) : 0;
  const int cv = a.C - a.D + d, cg = a.gate + d;
  const float* pv = a.p + ((size_t)b * a.C + cv) * a.P;
  const float* pg = a.p + ((size_t)b * a.C + cg) * a.P;
  const float ibv = a.in_bias ? __ldg(a.in_bias + cv) : 0.f, ibg = a.in_bias ? __ldg(a.in_bias + cg) : 0.f;
  const float v0 = __ldg(a.sw + 3 * cv), v1 = __ldg(a.sw + 3 * cv + 1), v2 = __ldg(a.sw + 3 * cv + 2), vb = __ldg(a.sb + cv);
  const float g0 = __ldg(a.sw + 3 * cg), g1 = __ldg(a.sw + 3 * cg + 1), g2 = __ldg(a.sw + 3 * cg + 2), gb = __ldg(a.sb + cg);
  T* h = a.h + (size_t)row * a.ld;
  for (int t = blockIdx.y * blockDim.x + threadIdx.x; t < a.P; t += gridDim.y * blockDim.x) {
    if (ROWS) {
      if (t < s) { h[t] = hround<T>(0.f); continue; }
      const float vm2 = t - 2 >= s ? pv[t - 2] + ibv : 0.f, vm1 = t - 1 >= s ? pv[t - 1] + ibv : 0.f, vp = pv[t] + ibv;
      const float gm2 = t - 2 >= s ? pg[t - 2] + ibg : 0.f, gm1 = t - 1 >= s ? pg[t - 1] + ibg : 0.f, gp = pg[t] + ibg;
      h[t] = hround<T>(short3(v0, v1, v2, vb, vm2, vm1, vp) * short3(g0, g1, g2, gb, gm2, gm1, gp));
    } else {
      const float vm2 = t >= 2 ? pv[t - 2] + ibv : 0.f, vm1 = t >= 1 ? pv[t - 1] + ibv : 0.f, vp = pv[t] + ibv;
      const float gm2 = t >= 2 ? pg[t - 2] + ibg : 0.f, gm1 = t >= 1 ? pg[t - 1] + ibg : 0.f, gp = pg[t] + ibg;
      h[t] = hround<T>(short3(v0, v1, v2, vb, vm2, vm1, vp) * short3(g0, g1, g2, gb, gm2, gm1, gp));
    }
  }
  // tail of channels d, D + d, ..., O D + d (one thread each, first CTA of the row)
  const int nj = a.C / a.D;
  if (blockIdx.y == 0 && (int)threadIdx.x < nj) {
    const int c = threadIdx.x * a.D + d;
    const float* pc = a.p + ((size_t)b * a.C + c) * a.P;
    const float ib = a.in_bias ? __ldg(a.in_bias + c) : 0.f;
    float* tl = a.tail + ((size_t)b * a.C + c) * 2;
    tl[0] = (ROWS ? a.P - 2 >= s : a.P >= 2) ? pc[a.P - 2] + ib : 0.f;
    tl[1] = pc[a.P - 1] + ib;
  }
}

template <class T>
__global__ void __launch_bounds__(256) decode_hist_kernel(const HistArgsT<T> a) { hist_body<false>(a); }
template <class T>
__global__ void __launch_bounds__(256) decode_hist_rows_kernel(const HistArgsT<T> a) { hist_body<true>(a); }

// Admission of prompt i into cache row rows[i] at the placement offset off = t - P (AdmitArgs): the arithmetic of hist_body
// on the prompt's positions j = tau - off, written at cache positions tau in [off, t), and 0 at tau < off + s (s the prompt's
// first real position, 0 without row_start) in the same pass, so no separate memset runs.  A row whose history is zero
// before its first real position decodes like the unpadded prompt (time invariance, DESIGN.md section 4.15).  The tail of
// all C channels of row rows[i] is the prompt's last two positions, a pad position there 0.
// PACKED: the prompts are packed back to back in p (1, C, T); position j of prompt i is read at p[c T + seg_base[i] + j]
// (64-bit), and only at j >= s = row_start[i] = P - n_i, so nothing before a prompt is read.  Otherwise wp.seg_base and
// wp.cstride are unused and the kernel is the plain admission (AdmitArgs in wp.adm).
// Grid: (k * D rows, up to 64 position CTAs per row); the rows go on x, which has no 65535 limit.
template <bool PACKED, class T>
__global__ void __launch_bounds__(256) decode_admit_kernel(const AdmitPackedArgsT<T> wp) {
  const AdmitArgsT<T>& w = wp.adm;
  const HistArgsT<T>& a = w.hist;
  const int row = blockIdx.x;                    // i * D + d
  const int i = row / a.D, d = row - i * a.D;
  const int s = a.row_start ? __ldg(a.row_start + i) : 0;
  const int s0 = w.off + s;                      // first real position in cache positions
  const int r = __ldg(w.rows + i);
  const int cv = a.C - a.D + d, cg = a.gate + d;
  const long long sbase = PACKED ? __ldg(wp.seg_base + i) : 0;
  const float* pv = PACKED ? a.p + (cv * wp.cstride + sbase) : a.p + ((size_t)i * a.C + cv) * a.P;
  const float* pg = PACKED ? a.p + (cg * wp.cstride + sbase) : a.p + ((size_t)i * a.C + cg) * a.P;
  const float ibv = a.in_bias ? __ldg(a.in_bias + cv) : 0.f, ibg = a.in_bias ? __ldg(a.in_bias + cg) : 0.f;
  const float v0 = __ldg(a.sw + 3 * cv), v1 = __ldg(a.sw + 3 * cv + 1), v2 = __ldg(a.sw + 3 * cv + 2), vb = __ldg(a.sb + cv);
  const float g0 = __ldg(a.sw + 3 * cg), g1 = __ldg(a.sw + 3 * cg + 1), g2 = __ldg(a.sw + 3 * cg + 2), gb = __ldg(a.sb + cg);
  T* h = a.h + ((size_t)r * a.D + d) * a.ld;
  for (int t = blockIdx.y * blockDim.x + threadIdx.x; t < w.t; t += gridDim.y * blockDim.x) {
    if (t < s0) { h[t] = hround<T>(0.f); continue; }
    const int j = t - w.off;
    const float vm2 = j - 2 >= s ? pv[j - 2] + ibv : 0.f, vm1 = j - 1 >= s ? pv[j - 1] + ibv : 0.f, vp = pv[j] + ibv;
    const float gm2 = j - 2 >= s ? pg[j - 2] + ibg : 0.f, gm1 = j - 1 >= s ? pg[j - 1] + ibg : 0.f, gp = pg[j] + ibg;
    h[t] = hround<T>(short3(v0, v1, v2, vb, vm2, vm1, vp) * short3(g0, g1, g2, gb, gm2, gm1, gp));
  }
  // tail of channels d, D + d, ..., O D + d (one thread each, first CTA of the row)
  const int nj = a.C / a.D;
  if (blockIdx.y == 0 && (int)threadIdx.x < nj) {
    const int c = threadIdx.x * a.D + d;
    const float* pc = PACKED ? a.p + (c * wp.cstride + sbase) : a.p + ((size_t)i * a.C + c) * a.P;
    const float ib = a.in_bias ? __ldg(a.in_bias + c) : 0.f;
    float* tl = a.tail + ((size_t)r * a.C + c) * 2;
    tl[0] = a.P - 2 >= s ? pc[a.P - 2] + ib : 0.f;
    tl[1] = pc[a.P - 1] + ib;
  }
}

// In-place shift of one history row per CTA (ShiftArgs) over the 4-position vectors V of [0, round4(t)) (a float4, or 8
// bytes of a 16-bit history); shift is a multiple of 4, so whole vectors move.  Left (shift = -m): h[tau] = h[tau + m], tiles in ascending order.  Right (shift = d): h[tau + d] =
// h[tau], tiles in descending order, then [0, d) zeroed.  Each tile's loads complete (__syncthreads) before its stores, and
// no later tile reads a word an earlier tile stored (left: later tiles read above every earlier destination; right: below
// it), so the shift is race-free without a scratch copy.  Plain loads: the row is written in place (no read-only path).
template <class T>
__global__ void __launch_bounds__(kShiftThreads) decode_shift_kernel(const ShiftArgsT<T> a) {
  using V = typename HVec4<T>::type;
  V* h = reinterpret_cast<V*>(a.h + (size_t)blockIdx.x * a.ld);
  const int n4 = (a.t + 3) >> 2;
  constexpr int kTile = kShiftThreads * kShiftVec;
  V v[kShiftVec];
  if (a.shift < 0) {
    const int m4 = (-a.shift) >> 2, w4 = n4 - m4;          // destinations [0, w4) <- sources [m4, n4)
    for (int q0 = 0; q0 < w4; q0 += kTile) {
#pragma unroll
      for (int u = 0; u < kShiftVec; ++u) {
        const int q = q0 + u * kShiftThreads + threadIdx.x;
        if (q < w4) v[u] = h[q + m4];
      }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < kShiftVec; ++u) {
        const int q = q0 + u * kShiftThreads + threadIdx.x;
        if (q < w4) h[q] = v[u];
      }
    }
  } else {
    const int d4 = a.shift >> 2;                           // destinations [d4, d4 + n4) <- sources [0, n4)
    for (int q1 = n4; q1 > 0; q1 -= kTile) {
#pragma unroll
      for (int u = 0; u < kShiftVec; ++u) {
        const int q = q1 - 1 - (u * kShiftThreads + (int)threadIdx.x);
        if (q >= 0) v[u] = h[q];
      }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < kShiftVec; ++u) {
        const int q = q1 - 1 - (u * kShiftThreads + (int)threadIdx.x);
        if (q >= 0) h[q + d4] = v[u];
      }
    }
    // every load happened before the last tile's barrier, and the stores went to [d4, d4 + n4): [0, d4) is free
    for (int q = threadIdx.x; q < d4; q += kShiftThreads) h[q] = V{};
  }
}

// part[b][d][chunk] = sum_{s in chunk, s < t} h[b][d][s] k[t-s]   for the batch rows [z*BG, z*BG + BG)
template <int BG, int R, class T>
__device__ __forceinline__ void dot_body(const DotArgsT<T> a) {
  const int lane = threadIdx.x & 31;
  const int d = blockIdx.y * kDotWarps + (threadIdx.x >> 5);
  if (d >= a.D) return;
  const int chunk = blockIdx.x, b0 = blockIdx.z * BG;
  // k[t-s] = krow[ld-1-t+s]; (ld-1-t) - R is a multiple of 4, so kb is 16-byte aligned
  const float* kb = a.k + (size_t)d * a.kstride + (a.ld - 1 - a.t - R);
  float acc[BG];
#pragma unroll
  for (int i = 0; i < BG; ++i) acc[i] = 0.f;
#pragma unroll
  for (int j = 0; j < kChunk / 128; ++j) {
    const int s0 = chunk * kChunk + j * 128 + lane * 4;
    if (s0 < a.t) {
      const float4 ka = ld4(kb + s0);
      float4 kv = ka;
      if (R != 0) {
        const float4 kc = ld4(kb + s0 + 4);
        if (R == 1) kv = make_float4(ka.y, ka.z, ka.w, kc.x);
        if (R == 2) kv = make_float4(ka.z, ka.w, kc.x, kc.y);
        if (R == 3) kv = make_float4(ka.w, kc.x, kc.y, kc.z);
      }
      const bool full = s0 + 4 <= a.t;
#pragma unroll
      for (int i = 0; i < BG; ++i) {
        const int b = b0 + i;
        if (b < a.B) {
          float4 hv = hld4(a.h + ((size_t)b * a.D + d) * a.ld + s0);
          if (!full) {                           // positions >= t hold no history yet
            hv.y = s0 + 1 < a.t ? hv.y : 0.f;
            hv.z = s0 + 2 < a.t ? hv.z : 0.f;
            hv.w = 0.f;
          }
          acc[i] = fmaf(hv.x, kv.x, acc[i]);
          acc[i] = fmaf(hv.y, kv.y, acc[i]);
          acc[i] = fmaf(hv.z, kv.z, acc[i]);
          acc[i] = fmaf(hv.w, kv.w, acc[i]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < BG; ++i) {
    float s = acc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const int b = b0 + i;
    if (lane == 0 && b < a.B) a.part[((size_t)b * a.D + d) * a.nchunk_max + chunk] = s;
  }
}

template <int BG, int R, class T>
__global__ void __launch_bounds__(32 * kDotWarps) decode_dot_kernel(const DotArgsT<T> a) { dot_body<BG, R>(a); }

// decode_dot_kernel with t (and the history offset) read from the device position: the grid covers a fixed chunk bound and
// the CTAs of chunks at or past t leave at once (the combine reads only the ceil(t / kChunk) partials below them)
template <int BG, class T>
__global__ void __launch_bounds__(32 * kDotWarps) decode_dot_dev_kernel(DotArgsT<T> a, const DevPos p) {
  const int t0 = p.pos[0];
  const int off = p.mode == kPosWindow ? p.pos[1] : p.mode == kPosBranch ? p.pos[2] : 0;
  a.t = t0 - off;
  if ((int)blockIdx.x * kChunk >= a.t) return;
  if (p.mode == kPosWindow) a.h += off;
  switch ((a.ld - 1 - a.t) & 3) {
    case 0: dot_body<BG, 0>(a); break;
    case 1: dot_body<BG, 1>(a); break;
    case 2: dot_body<BG, 2>(a); break;
    default: dot_body<BG, 3>(a); break;
  }
}

// fixed-order reduction of the chunk partials of one (b, channel) row: lane-strided chains, then a butterfly
template <class T>
__device__ __forceinline__ float reduce_partials(const StepArgsT<T>& a, int row, int lane) {
  float acc = 0.f;
  const float* part = a.part + (size_t)row * a.nchunk_max;
  for (int i = lane; i < a.nchunk; i += 32) acc += part[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// everything of a step at position t once acc = sum_{s<t} k[t-s] g[s] is known (one warp per (b, channel) row); the
// s = t term and the bias use the stored g^[t], as every later read of it does
template <class T>
__device__ __forceinline__ void step_epilogue(const StepArgsT<T>& a, int row, int b, int d, int lane, float acc) {
  float v, gate, x0;
  if (a.v_in == nullptr) {
    // recurrence 0: lane j < O+1 runs the short filter of channel j D + d from the tail and p_t, and shifts the tail
    float s = 0.f;
    if (lane <= a.order) {
      const int c = lane * a.D + d;
      const size_t bc = (size_t)b * a.C + c;
      const float pt = a.p_t[bc] + (a.in_bias ? __ldg(a.in_bias + c) : 0.f);
      float* tl = a.tail + bc * 2;
      const float pm2 = tl[0], pm1 = tl[1];
      s = short3(__ldg(a.sw + 3 * c), __ldg(a.sw + 3 * c + 1), __ldg(a.sw + 3 * c + 2), __ldg(a.sb + c), pm2, pm1, pt);
      a.s_t[bc] = s;
      tl[0] = pm1;
      tl[1] = pt;
    }
    v = __shfl_sync(0xffffffffu, s, a.order);
    gate = __shfl_sync(0xffffffffu, s, a.gate / a.D);
    x0 = __shfl_sync(0xffffffffu, s, 0);
  } else {
    v = a.v_in[row];
    gate = a.s_t[(size_t)b * a.C + a.gate + d];
    x0 = a.s_t[(size_t)b * a.C + d];
  }
  if (lane == 0) {
    const T gs = hround<T>(v * gate);
    a.h[(size_t)row * a.ld + a.t] = gs;
    const float g = hwiden(gs);
    const float k0 = a.k[(size_t)d * a.kstride + a.ld - 1];
    float y = fmaf(k0, g, acc);
    y = fmaf(a.fbias[(size_t)d * a.fstride], g, y);
    a.out[row] = a.last ? y * x0 : y;
  }
}

template <class T>
__global__ void __launch_bounds__(32 * kStepWarps) decode_step_kernel(const StepArgsT<T> a) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kStepWarps + (threadIdx.x >> 5);      // b * D + d
  if (row >= a.B * a.D) return;
  const int b = row / a.D, d = row - b * a.D;
  const float acc = reduce_partials(a, row, lane);
  step_epilogue(a, row, b, d, lane, acc);
}

// a step inside an open window: the partials of the window positions [b, t), then F[t-b] (the history before b), then
// the same epilogue as decode_step_kernel; the summation order is fixed, so a windowed step is bitwise reproducible
template <class T>
__global__ void __launch_bounds__(32 * kStepWarps) decode_win_step_kernel(const WinStepArgsT<T> w) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kStepWarps + (threadIdx.x >> 5);      // b * D + d
  if (row >= w.st.B * w.st.D) return;
  const int b = row / w.st.D, d = row - b * w.st.D;
  const float acc = reduce_partials(w.st, row, lane) + w.win[(size_t)row * w.wstride + w.j];
  step_epilogue(w.st, row, b, d, lane, acc);
}

// a step of a branched cache: the partials of the branch's own positions [b, t), then F[parent[row b]][d][t-b] (the shared
// context before b), then the same epilogue on the branch's history row (stride H); fixed order, bitwise reproducible
template <class T>
__global__ void __launch_bounds__(32 * kStepWarps) decode_branch_step_kernel(const BranchStepArgsT<T> w) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kStepWarps + (threadIdx.x >> 5);      // b * D + d
  if (row >= w.st.B * w.st.D) return;
  const int b = row / w.st.D, d = row - b * w.st.D;
  const float* f = w.f + ((size_t)__ldg(w.parent + b) * w.st.D + d) * w.st.ld;
  const float acc = reduce_partials(w.st, row, lane) + f[w.st.t];
  step_epilogue(w.st, row, b, d, lane, acc);
}

// the combine kernels of a device-position step: t (and win_b, base) from pos, then the same bodies as above
template <class T>
__device__ __forceinline__ void dev_position(StepArgsT<T>& st, int t) {
  st.t = t;
  st.nchunk = (t + kChunk - 1) / kChunk;
}

template <class T>
__global__ void __launch_bounds__(32 * kStepWarps) decode_step_dev_kernel(StepArgsT<T> a, const int* pos) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kStepWarps + (threadIdx.x >> 5);      // b * D + d
  if (row >= a.B * a.D) return;
  dev_position(a, pos[0]);
  const int b = row / a.D, d = row - b * a.D;
  const float acc = reduce_partials(a, row, lane);
  step_epilogue(a, row, b, d, lane, acc);
}

// the partials cover [win_b, t); st.t stays absolute (g_t is written at h[t]) while the partial count follows t - win_b
template <class T>
__global__ void __launch_bounds__(32 * kStepWarps) decode_win_step_dev_kernel(WinStepArgsT<T> w, const int* pos) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kStepWarps + (threadIdx.x >> 5);      // b * D + d
  if (row >= w.st.B * w.st.D) return;
  const int t = pos[0], j = t - pos[1];
  dev_position(w.st, j);
  w.st.t = t;
  const int b = row / w.st.D, d = row - b * w.st.D;
  const float acc = reduce_partials(w.st, row, lane) + w.win[(size_t)row * w.wstride + j];
  step_epilogue(w.st, row, b, d, lane, acc);
}

template <class T>
__global__ void __launch_bounds__(32 * kStepWarps) decode_branch_step_dev_kernel(BranchStepArgsT<T> w, const int* pos) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kStepWarps + (threadIdx.x >> 5);      // b * D + d
  if (row >= w.st.B * w.st.D) return;
  dev_position(w.st, pos[0] - pos[2]);
  const int b = row / w.st.D, d = row - b * w.st.D;
  const float* f = w.f + ((size_t)__ldg(w.parent + b) * w.st.D + d) * w.st.ld;
  const float acc = reduce_partials(w.st, row, lane) + f[w.st.t];
  step_epilogue(w.st, row, b, d, lane, acc);
}

// the end of a device-position step: one thread, launched after every kernel of the step has read pos
__global__ void decode_pos_advance_kernel(int* pos) { pos[0] += 1; }

}  // namespace dec
}  // namespace hy
