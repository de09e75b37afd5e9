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

}  // namespace dec
}  // namespace hy
