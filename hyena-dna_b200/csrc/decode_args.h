// Argument blocks of the incremental-decoding kernels (decode.cuh); host-includable.
//
// Cache layout (one HyenaOperator, O = order, C = (O+1) D in_proj channels, F = (O-1) D filter channels, Lcap positions,
// ld = Lcap rounded up to a multiple of 4):
//   k     (F, ld) + 4 floats  the filter, time-reversed: k[c][j] is stored at k[c*ld + ld-1-j]; the 4 trailing floats are
//                             padding that the aligned vector loads of the last row may touch (never used)
//   h     (O-1, B, D, ld)     the gated input g_o of every recurrence o, by position
//   tail  (B, C, 2)           in_proj outputs (with bias) of the last two positions: the 3-tap short filter's state
//   s_t   (B, C)              short-filter outputs of the current position (written by recurrence 0, read by the later ones)
//   part  (B, D, ceil(Lcap/1024)) partial dot products of one step
// A windowed step (WinStepArgs below) also reads the window's history tail F (O-1, B, D, W), kept beside the cache.
// Extending by n positions (Ext* below) uses per-call scratch: the short-filter outputs (B, C, n) and the partials of the
// direct Toeplitz kernel (B, D, n, ext_groups()).  The cache layout is the same.
#pragma once

namespace hy {
namespace dec {

constexpr int kChunk = 1024;              // positions per partial: one warp, 32 lanes x 8 float4
constexpr int kDotWarps = 8;              // channels per CTA of the dot kernel (one warp each)
constexpr int kStepWarps = 8;             // (b, channel) pairs per CTA of the combine kernel
constexpr int kMaxOrder = 31;             // the combine kernel gives one lane to each of the O+1 in_proj channel groups

inline int ld_for(int Lcap) { return (Lcap + 3) & ~3; }
inline int chunks_for(int Lcap) { return (Lcap + kChunk - 1) / kChunk; }

struct HistArgs {
  const float* p;        // (B, C, P) in_proj output without its bias, channel-major
  const float* in_bias;  // (C) or null
  const float* sw;       // (C, 3) short_filter.weight
  const float* sb;       // (C) short_filter.bias
  float* h;              // (B, D, ld): history of recurrence 0, positions [0, P) written
  float* tail;           // (B, C, 2)
  int B, D, C, P, ld;
  int gate;              // channel offset of the gate of recurrence 0: (O-1) D
};

struct DotArgs {
  const float* h;        // (B, D, ld) history of this recurrence
  const float* k;        // reversed filter row of channel d of this recurrence: k + d * kstride
  float* part;           // (B, D, nchunk_max)
  int B, D, t, ld, kstride, nchunk_max;
};

struct StepArgs {
  const float* part;     // (B, D, nchunk_max) partials of sum_{s<t} h[s] k[t-s]
  int nchunk, nchunk_max;
  const float* k;        // reversed filter row of channel d: k + d * kstride (k[0] at index ld-1)
  const float* fbias;    // effective filter bias of channel d: fbias[d * fstride]
  int kstride, fstride, ld;
  const float* p_t;      // (B, C) in_proj output of position t without its bias (recurrence 0 only)
  const float* in_bias;  // (C) or null
  const float* sw;       // (C, 3)
  const float* sb;       // (C)
  float* tail;           // (B, C, 2)
  float* s_t;            // (B, C)
  const float* v_in;     // (B, D) output of the previous recurrence, null for recurrence 0
  float* h;              // (B, D, ld) history of this recurrence: g_t is written at position t
  float* out;            // (B, D) recurrence output; times x0 when `last`
  int B, D, C, order, t;
  int gate;              // channel offset of this recurrence's gate: (O-1-o) D
  int last;
};

// A windowed step at position t in the window [b, b + Wc) (b a multiple of 4): st.part / st.nchunk hold the partials of
// sum_{b<=s<t} h[s] k[t-s] (decode_dot_kernel on h + b with t - b), and win the precomputed history tail
// F[j] = sum_{s<b} k[b+j-s] h[s] of the window positions j in [0, Wc)
struct WinStepArgs {
  StepArgs st;
  const float* win;      // (B, D, wstride) F of this recurrence
  int wstride;           // W >= Wc
  int j;                 // t - b
};

// A step whose position is read on the device (a captured CUDA graph replays it at every position): pos = [t, win_b, base]
// (int32).  The dot kernel runs on a grid of a fixed chunk bound; it takes its t and history offset from pos by `mode`:
constexpr int kPosPlain = 0;              // t = pos[0] over h
constexpr int kPosWindow = 1;             // t = pos[0] - pos[1] over h + pos[1]
constexpr int kPosBranch = 2;             // t = pos[0] - pos[2] over the branch rows h
struct DevPos {
  const int* pos;        // [t, win_b, base]
  int mode;              // kPos*
};

// ---- extending a cache by n positions at once (decode_extend.cuh)
constexpr int kExtRJ = 8;                 // outputs per thread of the direct Toeplitz kernel (register block)
constexpr int kExtWarps = 8;              // warps per CTA of the direct Toeplitz kernel
constexpr int kExtTargetCtas = 4096;      // the direct kernel merges 1024-position chunks per CTA down to about this many CTAs

inline int ext_tile(int n) { return n <= 8 ? 8 : 64; }        // outputs per CTA of the direct kernel (8 or 64)
inline int ext_bg(int B) { return B <= 1 ? 1 : B <= 2 ? 2 : B <= 4 ? 4 : 8; }

// chunks per CTA of the direct kernel for (B, D, history t, n new positions); the partials have ext_groups() entries per
// output: ceil(chunks / chunks_per_cta)
inline int ext_chunks_per_cta(int B, int D, int t, int n) {
  const int nchunk = chunks_for(t + n);
  const int njt = (n + ext_tile(n) - 1) / ext_tile(n), bg = ext_bg(B);
  const long long base = (long long)njt * D * ((B + bg - 1) / bg);
  long long want = kExtTargetCtas / base;
  if (want < 1) want = 1;
  if (want > nchunk) want = nchunk;
  return (int)((nchunk + want - 1) / want);
}
inline int ext_groups(int B, int D, int t, int n) {
  const int cpb = ext_chunks_per_cta(B, D, t, n);
  return (chunks_for(t + n) + cpb - 1) / cpb;
}

struct ExtHistArgs {
  const float* p;        // (B, C, n) in_proj output of positions [t, t+n) without its bias, channel-major
  const float* in_bias;  // (C) or null
  const float* sw;       // (C, 3)
  const float* sb;       // (C)
  float* tail;           // (B, C, 2): read as the state before position t, left as the state after position t+n-1
  float* s;              // (B, C, n) short-filter outputs of the n positions
  float* h;              // (B, D, ld) history of recurrence 0: g_0 of positions [t, t+n) written
  int B, D, C, t, n, ld;
  int gate;              // channel offset of the gate of recurrence 0: (O-1) D
};

struct ExtDotArgs {
  const float* h;        // (B, D, ld) history of this recurrence, positions [0, t+n) valid
  const float* k;        // reversed filter row of channel d of this recurrence: k + d * kstride
  float* part;           // (B, D, n, groups)
  int B, D, t, n, ld, kstride;
  int R;                 // (-t) mod 4: misalignment of every filter window (see decode_ext_dot_kernel)
  int njt;               // output tiles of the kernel's tile size: ceil(n / NT)
  int cpb, nchunk, groups;
};

struct ExtCombineArgs {
  const float* part;     // sum over g < groups of part[row * prow + j * pj + g] = sum_{s<=t+j} k[t+j-s] g_o[s]
  long long prow;
  int pj, groups;
  const float* fbias;    // effective filter bias of channel d: fbias[d * fstride]
  int fstride;
  const float* h;        // (B, D, ld) history of this recurrence (g_o[t+j] for the bias term)
  const float* s;        // (B, C, n) short-filter outputs (the gates)
  float* h_next;         // (B, D, ld) history of the next recurrence: g_{o+1} = out * x_{O-2-o}, or null when `last`
  float* y;              // (B, D, n): out * x_0 when `last`
  int B, D, C, t, n, ld;
  int xch;               // channel offset of the gate that multiplies the output: (O-2-o) D
  int last;
};

// ---- decoding a branched cache (DecodeCache.fork): branches of one context that share its history tail F
// A branch row holds g_o of positions [b, b + Hc) only, with row stride H (b and H multiples of 4, Hc <= H).  The kernels run
// on it with ld = H, t - b in place of t and the filter pointer moved by ld_parent - H: every tap index ld-1-t+s then lands on
// the same absolute filter element as in the unbranched call.  F (P, D, H) of a recurrence holds, per parent row, the
// contribution of the context before b to the positions [b, b + Hc); parent[row b] selects the F row of branch b.
struct BranchStepArgs {
  StepArgs st;           // st.ld = H, st.t = t - b, st.k shifted; st.part holds the partials over [b, t)
  const float* f;        // (P, D, H) F of this recurrence
  const int* parent;     // (B) F row of each branch
};

struct BranchCombineArgs {
  ExtCombineArgs c;      // c.ld = H, c.t = t - b
  const float* f;        // (P, D, H) F of this recurrence
  const int* parent;     // (B) F row of each branch
};

}  // namespace dec
}  // namespace hy
