// In-register radix-R (R = 1,2,4,...,32) complex FFT and the two-stage block FFT built on it.
//
// Every index below is a compile-time constant after template expansion: the 32 complex
// values a thread owns stay in registers, twiddles W_32^j become FFMA immediates, and the
// "bit reversal" of the decimation-in-frequency butterflies is pure register renaming.
#pragma once
#include "common.cuh"

namespace hy {

// cos(2*pi*j/32), j in [0,8]
__host__ __device__ constexpr float qcos32(int j) {
  constexpr float t[9] = {1.0f, 0.9807852804032304f, 0.9238795325112867f, 0.8314696123025452f, 0.7071067811865476f,
                          0.5555702330196022f, 0.3826834323650898f, 0.19509032201612825f, 0.0f};
  return t[j];
}
__host__ __device__ constexpr float cos32(int j) {
  j &= 31;
  return j <= 8 ? qcos32(j) : j <= 16 ? -qcos32(16 - j) : j <= 24 ? -qcos32(j - 16) : qcos32(32 - j);
}
__host__ __device__ constexpr float sin32(int j) { return cos32(j + 24); }

// a * W_32^J (forward, W = exp(-2 pi i/32)) or a * conj(W_32^J) (INV)
template <int J, bool INV>
__device__ __forceinline__ float2 mul_w32(float2 a) {
  constexpr int j = J & 31;
  if constexpr (j == 0) return a;
  else if constexpr (j == 16) return make_float2(-a.x, -a.y);
  else if constexpr (j == 8) return INV ? cmul_i(a) : cmul_negi(a);
  else if constexpr (j == 24) return INV ? cmul_negi(a) : cmul_i(a);
  else {
    constexpr float c = cos32(j);
    constexpr float s = INV ? -sin32(j) : sin32(j);      // multiply by (c - i s)
    return cmul_cs(a, c, s);
  }
}

// One decimation-in-frequency pass over the sub-array v[BASE .. BASE+N), recursing down to N = 1.
// On return element X[k] of each length-N0 transform sits at v[BASE + brev(k)].
template <int N, int BASE, bool INV, int TOTAL>
__device__ __forceinline__ void dif(float2 (&v)[TOTAL]) {
  if constexpr (N >= 2) {
    constexpr int H = N / 2;
    static_for<0, H>([&](auto i_) {
      constexpr int i = decltype(i_)::value;
      float2 a = v[BASE + i], b = v[BASE + i + H];
      v[BASE + i] = cadd(a, b);
      v[BASE + i + H] = mul_w32<i * (32 / N), INV>(csub(a, b));
    });
    dif<H, BASE, INV, TOTAL>(v);
    dif<H, BASE + H, INV, TOTAL>(v);
  }
}

// Same, but the caller promises v[BASE+H .. BASE+N) == 0 on entry (zero-padded upper half):
// the first butterfly layer degenerates to a copy and one twiddle multiply.
template <int N, int BASE, bool INV, int TOTAL>
__device__ __forceinline__ void dif_upper_zero(float2 (&v)[TOTAL]) {
  if constexpr (N >= 2) {
    constexpr int H = N / 2;
    static_for<0, H>([&](auto i_) {
      constexpr int i = decltype(i_)::value;
      v[BASE + i + H] = mul_w32<i * (32 / N), INV>(v[BASE + i]);
    });
    dif<H, BASE, INV, TOTAL>(v);
    dif<H, BASE + H, INV, TOTAL>(v);
  }
}

// ------------------------------------------------------------------------------------------
// Geometry of an N-point FFT spread over N/32 threads (N >= 32), each owning 32 points.
//   stage 1: thread q holds x[R2*n1 + q] in v[n1]; radix-32 over n1; twiddle W_N^{q*k1'}
//   exchange through shared memory (row pitch P = R2+1 complex, conflict free)
//   stage 2: thread q owns the G2 = 32/R2 work items k1' = q + R2*i; radix-R2 over n2
//   result:  X[R2*s + q] ("natural slot s") sits in v[slot<LOGN>(s)]
// For N < 32 a thread owns 32/N whole transforms: transform gi lives in v[gi*N .. gi*N+N) and
// X[k] of transform gi sits in v[gi*N + brev(k)].
template <int LOGN>
struct Geo {
  static constexpr int N = 1 << LOGN;
  static constexpr int R2 = N >= 32 ? N / 32 : 1;
  static constexpr int LOGR2 = ilog2c(R2);
  static constexpr int G2 = 32 / R2;
  static constexpr int P = R2 + 1;                 // exchange row pitch (complex elements)
  static constexpr int THREADS = N >= 32 ? N / 32 : 1;
  __host__ __device__ static constexpr int slot(int s) {
    if (N < 32) return 0;   // not used
    if (R2 == 1) return brev(s, 5);
    return (s % G2) * R2 + brev(s / G2, LOGR2);
  }
  // exchange footprint of one transform, in complex elements (without the per-transform pad)
  __host__ __device__ static constexpr int ex_elems() { return R2 == 1 ? 0 : 32 * P; }
};

// v[idx(s)] *= lo[s & 7] * hi[s >> 3] for s in [0,32) (hi[0] is taken as 1), the 32 twiddles base * step^s of a geometric
// sequence split as (base * step^j, j < 8) x (step^{8m}, m < 4).  The callers read all eleven factors straight from the
// twiddle tables (one or two correctly rounded table entries each), so that every twiddle carries at most one table
// product and ONE further rounding -- round 1 built them by chained multiplications (up to five roundings), which showed up
// as ~1.3x the error of the reference's cuFFT path at L = 2^20 (tests/test_gpu_parity_full.py).
// idx is a constexpr functor s -> register index.  CONJ multiplies by the conjugates instead.
template <bool CONJ, class IDX>
__device__ __forceinline__ void mul_twiddles(float2 (&v)[32], const float2 (&lo_)[8], const float2 (&hi_)[4], IDX) {
  float2 lo[8], hi[4];
#pragma unroll
  for (int j = 0; j < 8; ++j) lo[j] = CONJ ? cconj(lo_[j]) : lo_[j];
#pragma unroll
  for (int j = 1; j < 4; ++j) hi[j] = CONJ ? cconj(hi_[j]) : hi_[j];
  static_for<0, 32>([&](auto s_) {
    constexpr int s = decltype(s_)::value;
    constexpr int r = IDX::at(s);
    float2 w = lo[s & 7];
    if constexpr ((s >> 3) > 0) w = cmul(w, hi[s >> 3]);
    v[r] = cmul(v[r], w);
  });
}

// W_{2^20}^{(eb + j*es) << sh} for j < 8 and W^{(8 m es) << sh} for m in 1..3, exponents modulo 2^logM
__device__ __forceinline__ void twiddle_factors20(const Twiddles& T, uint32_t eb, uint32_t es, int logM, float2 (&lo)[8],
                                                  float2 (&hi)[4]) {
  const int sh = 20 - logM;
  const uint32_t mask = (1u << logM) - 1u;
#pragma unroll
  for (int j = 0; j < 8; ++j) lo[j] = root20(T, ((eb + (uint32_t)j * es) & mask) << sh);
  hi[0] = make_float2(1.f, 0.f);
#pragma unroll
  for (int m = 1; m < 4; ++m) hi[m] = root20(T, ((8u * (uint32_t)m * es) & mask) << sh);
}

// the same from the 1024-entry table alone: W_1024^{(j e1)} and W_1024^{(8 m e1)}
__device__ __forceinline__ void twiddle_factors10(const float2* __restrict__ tw1024, uint32_t e1, float2 (&lo)[8], float2 (&hi)[4]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) lo[j] = __ldg(tw1024 + (((uint32_t)j * e1) & 1023u));
  hi[0] = make_float2(1.f, 0.f);
#pragma unroll
  for (int m = 1; m < 4; ++m) hi[m] = __ldg(tw1024 + ((8u * (uint32_t)m * e1) & 1023u));
}

template <int LOGN> struct SlotIdx { __host__ __device__ static constexpr int at(int s) { return Geo<LOGN>::slot(s); } };
struct Brev5Idx { __host__ __device__ static constexpr int at(int s) { return brev(s, 5); } };
struct IdentIdx { __host__ __device__ static constexpr int at(int s) { return s; } };

// Two-stage N-point FFT (N = 2^LOGN >= 32) of the 32 values in v (input: natural slot s in v[s]).
//   ex    : this transform's exchange area in shared memory (Geo::ex_elems() complex)
//   q     : this thread's index inside the transform, [0, R2)
//   SYNC  : functor called between the exchange write and read (warp or CTA barrier)
// Output: natural slot s (element R2*s + q) in v[Geo<LOGN>::slot(s)].
template <int LOGN, bool INV, bool UPPER_ZERO, class SYNC>
__device__ __forceinline__ void block_fft(float2 (&v)[32], float2* ex, int q, const float2* __restrict__ tw1024,
                                          SYNC sync) {
  using G = Geo<LOGN>;
  static_assert(LOGN >= 5 && LOGN <= 10, "two-stage FFT covers 32..1024 points");
  if constexpr (UPPER_ZERO) dif_upper_zero<32, 0, INV, 32>(v); else dif<32, 0, INV, 32>(v);
  if constexpr (G::R2 > 1) {
    // twiddle W_N^{q*k1'}: geometric in k1' with ratio W_N^q; exponents taken from the 1024-table
    constexpr int SH = 10 - LOGN;                         // W_N^e = tw1024[e << SH]
    const uint32_t e1 = (uint32_t)q << SH;
    float2 lo[8], hi[4];
    twiddle_factors10(tw1024, e1, lo, hi);
    mul_twiddles<INV>(v, lo, hi, Brev5Idx{});
    // exchange: ex[k1' * P + q]
    static_for<0, 32>([&](auto k_) {
      constexpr int k1 = decltype(k_)::value;
      ex[k1 * G::P + q] = v[brev(k1, 5)];
    });
    sync();
    static_for<0, G::G2>([&](auto i_) {
      constexpr int i = decltype(i_)::value;
      static_for<0, G::R2>([&](auto n_) {
        constexpr int n2 = decltype(n_)::value;
        v[i * G::R2 + n2] = ex[(q + G::R2 * i) * G::P + n2];
      });
    });
    static_for<0, G::G2>([&](auto i_) {
      constexpr int i = decltype(i_)::value;
      dif<G::R2, i * G::R2, INV, 32>(v);
    });
  }
}

}  // namespace hy
