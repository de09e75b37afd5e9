// Projection GEMMs of the operator on the Hopper tensor cores (wgmma), fp32 accuracy via 3xTF32.
//
// in_proj / out_proj and their input gradients (src/models/sequence/hyena.py:350-351, :391, :440) are all of the form
//     OUT[pos][n] = sum_k ACT[pos][k] * W[n][k]            pos = up to 2^20 sequence positions, K <= 768, N <= 768
// with the activation either row-major (pos, k) (u, dy) or channel-major (k, pos) (y_pre, ds/dp), and the output either
// channel-major (n, pos) (p, dy_pre: what the FFT passes read) or row-major (pos, n) (y, du).  One persistent,
// warp-specialised kernel (proj_gemm_kernel):
//
//   tile      128 positions x 128 outputs, K streamed in chunks of 32; two consumer warpgroups of 64 positions each
//   A operand the activation chunk: global -> shared-memory staging ring by TMA (one tiled copy per chunk, issued by a
//             producer warp, four chunks in flight) -> registers in the wgmma A-fragment layout -> (hi, lo) tf32 split.
//             The MMAs read A from registers, so only B goes through the shared-memory port.
//   B operand the weights, pre-split once per call into hi / lo images in the canonical no-swizzle K-major
//             core-matrix layout (proj_prep_kernel), streamed by TMA bulk copies into the same ring of stages
//   D         fp32 accumulators in registers, restarted for every K chunk (12 MMAs, the 8 small correction products
//             first so that only the 4 hi*hi MMAs add at full scale) and added into a second register set with
//             round-to-nearest adds.  Reason: the tensor core adds into its accumulator with truncation, so a long chain
//             biases the result by ~(number of MMAs) x 2^-24 towards zero.
//   3xTF32    x = hi + lo, hi = rna_tf32(x), lo = rna_tf32(x - hi);  D += Ahi Bhi + Alo Bhi + Ahi Blo   (lo*lo < 2^-22)
//
// Optional fused prologue (FIR): the activation is ds (B, C, L) and the GEMM consumes dp = transposed 3-tap depthwise
// filter of ds (dp[t] = w2 ds[t] + w1 ds[t+1] + w0 ds[t+2], hyena.py:363-369 backward), so dp never exists in HBM.
//
// Optional GELU transforms (template argument FN, the block MLP fc1 -> gelu -> fc2 with the hidden activation `a` kept
// channel-major (B, H, L); hyena-dna_b200/mlp.py):
//   ACT_CH  prologue: the GEMM consumes gelu(act)            (fc2 forward: gelu(a) never exists in HBM)
//   OUT_CH  epilogue: OUT = acc * gelu'(aux), aux (B, N, L)  (fc2 input gradient: da = (dy W2) o gelu'(a))
//   wgrad   the converter warps build the B images from gelu(X)  (fc2 weight gradient)
//
// Weight gradients (wgrad_kernel) at the end of the file.
#pragma once
#include <cuda.h>      // CUtensorMap (types only: the encode function is looked up at run time, no libcuda link)

#include "common.cuh"
#include "tc_prims.cuh"

namespace hy {

// Elementwise activations fused into the projection GEMMs: torch's fp32 GELU (approximate="tanh" / "none") and its
// analytic derivative, in the same formulas (ATen ActivationGeluKernel.cu) with the accurate tanhf / erff / expf.
enum ActFn { FN_NONE = 0, FN_GELU_TANH = 1, FN_GELU_ERF = 2 };

template <int FN>
__device__ __forceinline__ float act_fn(float x) {
  static_assert(FN == FN_GELU_TANH || FN == FN_GELU_ERF, "GELU variant");
  if constexpr (FN == FN_GELU_TANH) {
    constexpr float kBeta = (float)(M_SQRT2 * M_2_SQRTPI * 0.5), kKappa = 0.044715f;
    const float inner = kBeta * (x + kKappa * (x * x * x));
    return 0.5f * x * (1.f + tanhf(inner));
  } else {
    return x * 0.5f * (1.f + erff(x * (float)M_SQRT1_2));
  }
}

template <int FN>
__device__ __forceinline__ float act_grad(float x) {
  static_assert(FN == FN_GELU_TANH || FN == FN_GELU_ERF, "GELU variant");
  if constexpr (FN == FN_GELU_TANH) {
    constexpr float kBeta = (float)(M_SQRT2 * M_2_SQRTPI * 0.5), kKappa = 0.044715f;
    const float x_sq = x * x;
    const float th = tanhf(kBeta * (x + kKappa * (x_sq * x)));
    const float left = 0.5f * x, right = 1.f + th;
    const float left_derivative = 0.5f * right;
    const float right_derivative = left * (1.f - th * th) * (kBeta * (1.f + 3.f * kKappa * x_sq));
    return left_derivative + right_derivative;
  } else {
    constexpr float kBeta = (float)(M_2_SQRTPI * M_SQRT1_2 * 0.5);
    const float cdf = 0.5f * (1.f + erff(x * (float)M_SQRT1_2));
    const float pdf = expf(-0.5f * x * x) * kBeta;
    return cdf + x * pdf;
  }
}

namespace pg {

constexpr int kKC = 32;                 // K chunk (one chunk = 4 MMAs of K = 8 per product)
constexpr int kThreads = 288;           // 9 warps: 0-7 two consumer warpgroups, 8 TMA producer
constexpr uint32_t kSBO = 1024, kLBO = 128;
constexpr uint32_t kAPitchCh = 132 * 4; // ACT_CH staging row: 128 positions + one look-ahead quad (fused FIR)
constexpr uint32_t kAStageBytes = 32 * kAPitchCh;      // 16.5 KB (>= the 16 KB an ACT_ROW tile needs)

// byte offset of element (n, k) inside one (rows x 32) operand image
__host__ __device__ constexpr uint32_t img_off(int n, int k) {
  return (uint32_t)((n >> 3) * 1024 + (k >> 2) * 128 + (n & 7) * 16 + (k & 3) * 4);
}

enum ActLayout { ACT_ROW = 0 /* (B, L, K): k contiguous */, ACT_CH = 1 /* (B, K, L): position contiguous */ };
enum OutLayout { OUT_CH = 0 /* (B, N, L) */, OUT_ROW = 1 /* (B, L, N) */ };

struct Args {
  const float* act;      // activation, layout per template
  const float* wimg;     // weight images from proj_prep_kernel: [n_tile][k_chunk][hi | lo][NT x 32]
  float* out;
  const float* bias;     // (N) added in the epilogue, or null
  const float* fir;      // (K, 3) taps of the transposed short filter applied to the activation (ACT_CH only), or null
  int B, L, K, N;        // batch, positions per batch (tensor pitch), reduction size, outputs
  int l0, ln;            // positions [l0, l0 + ln) of every batch are processed (host-side chunking of long sequences)
  int kchunks;           // ceil(K / 32)
  int ntiles_n;          // ceil(N / NT)
  int mtiles_per_b;      // ceil(ln / 128)
  int vec;               // 1: the activation qualifies for TMA (16-byte aligned rows): `tmap` is valid
  const float* aux;      // (B, N, L) pre-activation read by the gradient epilogue (OUT_CH with FN != FN_NONE), or null
};

// ------------------------------------------------------------------------------------------------ weight images
// B[n][k] = transposed ? W[k * ldw + n] : W[n * ldw + k];  rows n >= N and columns k >= K are zero
__global__ void proj_prep_kernel(const float* __restrict__ W, int ldw, int transposed, int N, int K, int NT,
                                 float* __restrict__ img) {
  const int kch = (K + kKC - 1) / kKC, ntn = (N + NT - 1) / NT;
  const size_t total = (size_t)ntn * kch * NT * kKC;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int kk = (int)(i % kKC);
    const int nn = (int)((i / kKC) % NT);
    const int kc = (int)((i / ((size_t)kKC * NT)) % kch);
    const int nt = (int)(i / ((size_t)kKC * NT * kch));
    const int n = nt * NT + nn, k = kc * kKC + kk;
    float x = 0.f;
    if (n < N && k < K) x = transposed ? W[(size_t)k * ldw + n] : W[(size_t)n * ldw + k];
    float hi, lo;
    tc::split_tf32(x, hi, lo);
    float* base = img + ((size_t)nt * kch + kc) * 2 * NT * kKC;
    base[img_off(nn, kk) / 4] = hi;
    base[(size_t)NT * kKC + img_off(nn, kk) / 4] = lo;
  }
}

__host__ __device__ constexpr size_t wimg_floats(int N, int K, int NT) {
  return (size_t)((N + NT - 1) / NT) * ((K + kKC - 1) / kKC) * 2 * NT * kKC;
}

// ------------------------------------------------------------------------------------------------ the kernel
// Activation staging slot (17 KB, 1024-byte aligned):
//   ACT_ROW  128 rows x 32 floats (128-byte rows), 16-byte pieces XOR-swizzled by the row (= TMA SWIZZLE_128B): the
//            A-fragment loads (8 rows x 4 consecutive k per warp) are bank-conflict free
//   ACT_CH   32 channel rows x 132 floats (128 positions + 4 look-ahead samples for the fused FIR), dense
constexpr uint32_t kSStageBytes = 17408;
static_assert(kSStageBytes >= 32 * kAPitchCh && kSStageBytes >= 128 * 128 && kSStageBytes % 1024 == 0, "staging slot");

template <int NT> struct Cfg {
  static constexpr int STAGES = 4;                                     // weight stages = staging slots
  static constexpr uint32_t STAGE_BYTES = 2u * NT * kKC * 4u;          // hi + lo image of one K chunk
  static constexpr size_t OFF_A = (size_t)STAGES * STAGE_BYTES;        // activation staging ring
  static constexpr size_t OFF_BAR = OFF_A + (size_t)STAGES * kSStageBytes;
  static constexpr size_t OFF_FIR = OFF_BAR + 256;
  static constexpr size_t SMEM = OFF_FIR;                              // + 12 K bytes of taps when the FIR is fused
  static_assert(NT == 128, "one m64n128 accumulator per consumer warpgroup");
};

// Warp roles (288 threads):
//   warps 0-3, 4-7  consumer warpgroups, positions [0, 64) and [64, 128) of the tile: staged activation -> A fragments
//                   (-> fused FIR) -> (hi, lo) split -> wgmma against the weight stage -> register accumulators -> stores
//   warp 8          producer: per chunk one TMA bulk copy of the weight images and one tiled TMA copy of the activation
//                   tile (lane 0); stages the activation by hand when it does not qualify for TMA (all lanes)
// FN != FN_NONE: GELU prologue (ACT_CH -> OUT_ROW) or GELU-gradient epilogue (ACT_ROW -> OUT_CH), see the top of the file
template <int NT, int ACT, int OUT, int FN = FN_NONE>
__global__ void __launch_bounds__(kThreads, 1) proj_gemm_kernel(const Args a, const __grid_constant__ CUtensorMap tmap) {
  static_assert(FN == FN_NONE || (ACT == ACT_CH && OUT == OUT_ROW) || (ACT == ACT_ROW && OUT == OUT_CH),
                "the GELU transforms exist for the fc2 forward and input-gradient layouts only");
  using C = Cfg<NT>;
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  float* fir_s = reinterpret_cast<float*>(smem + C::OFF_FIR);     // (K, 3) taps, FIR only
  const uint32_t sbase = tc::smem_u32(smem);
  const uint32_t bar0 = tc::smem_u32(bars);
  auto FULL = [&](int s) { return bar0 + 8u * s; };
  auto EMPTY = [&](int s) { return bar0 + 8u * (4 + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool use_fir = (ACT == ACT_CH) && a.fir != nullptr;
  if (use_fir)
    for (int i = tid; i < 3 * a.K; i += kThreads) fir_s[i] = __ldg(a.fir + i);
  if (tid == 0) {
    for (int s = 0; s < 4; ++s) { tc::mbar_init(FULL(s), 1); tc::mbar_init(EMPTY(s), 8); }
  }
  __syncthreads();

  const int mtiles = a.B * a.mtiles_per_b;
  const int ntiles = mtiles * a.ntiles_n;
  const int lend = a.l0 + a.ln;
  auto tile_pos = [&](int tile, int& b, int& lt, int& nt) {
    const int mt = tile / a.ntiles_n;
    nt = tile - mt * a.ntiles_n;
    b = mt / a.mtiles_per_b;
    lt = a.l0 + (mt - b * a.mtiles_per_b) * 128;
  };

  if (warp == 8) {
    // ================================================================== producer
    // Out-of-range coordinates are zero-filled by the copy engine (end of the tensor: exactly the zero padding the fused
    // FIR needs; K tail).  Activations that do not qualify for TMA (rows not 16-byte aligned) are staged by the 32 lanes
    // with plain loads and stores instead.
    if (lane == 0 && a.vec) tc::tma_prefetch_desc(&tmap);
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      int b, lt, nt;
      tile_pos(tile, b, lt, nt);
      for (int kc = 0; kc < a.kchunks; ++kc, ++it) {
        const int s = (int)(it & 3u);
        const int k0 = kc * kKC;
        tc::mbar_wait_u(EMPTY(s), ((it >> 2) & 1u) ^ 1u);
        const float* wsrc = a.wimg + ((size_t)nt * a.kchunks + kc) * (C::STAGE_BYTES / 4);
        const uint32_t st_u = sbase + (uint32_t)C::OFF_A + (uint32_t)s * kSStageBytes;
        if (a.vec) {
          if (lane == 0) {
            const uint32_t abytes = (ACT == ACT_ROW) ? 128u * 128u : 32u * kAPitchCh;
            tc::mbar_arrive_expect_tx(FULL(s), C::STAGE_BYTES + abytes);
            tc::bulk_g2s(sbase + s * C::STAGE_BYTES, wsrc, C::STAGE_BYTES, FULL(s));
            if constexpr (ACT == ACT_ROW) tc::tma_load_2d(st_u, &tmap, k0, b * a.L + lt, FULL(s));
            else tc::tma_load_2d(st_u, &tmap, lt, b * a.K + k0, FULL(s));
          }
          continue;
        }
        unsigned char* st = smem + C::OFF_A + (size_t)s * kSStageBytes;
        if constexpr (ACT == ACT_ROW) {
#pragma unroll 1
          for (int i = 0; i < 4; ++i) {
            const int r = lane + 32 * i, l = lt + r;
            const float* src = a.act + ((size_t)b * a.L + (l < lend ? l : 0)) * a.K + k0;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              float4 v;
              v.x = (l < lend && k0 + 4 * c + 0 < a.K) ? __ldg(src + 4 * c + 0) : 0.f;
              v.y = (l < lend && k0 + 4 * c + 1 < a.K) ? __ldg(src + 4 * c + 1) : 0.f;
              v.z = (l < lend && k0 + 4 * c + 2 < a.K) ? __ldg(src + 4 * c + 2) : 0.f;
              v.w = (l < lend && k0 + 4 * c + 3 < a.K) ? __ldg(src + 4 * c + 3) : 0.f;
              *reinterpret_cast<float4*>(st + r * 128 + ((c ^ (r & 7)) << 4)) = v;
            }
          }
        } else {
          const int j = lane;
          const bool kv = k0 + j < a.K;
          const float* src = a.act + ((size_t)b * a.K + (kv ? k0 + j : 0)) * a.L + lt;
          float* dst = reinterpret_cast<float*>(st + j * kAPitchCh);
          for (int e = 0; e < 132; ++e) dst[e] = (kv && lt + e < a.L) ? __ldg(src + e) : 0.f;
        }
        __syncwarp();
        if (lane == 0) {
          tc::mbar_arrive_expect_tx(FULL(s), C::STAGE_BYTES);
          tc::bulk_g2s(sbase + s * C::STAGE_BYTES, wsrc, C::STAGE_BYTES, FULL(s));
        }
      }
    }
    return;
  }

  // ================================================================== consumers: warpgroup wg = positions [64 wg, 64 wg + 64)
  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const int r0 = 64 * wg + 16 * (warp & 3) + g;                  // fragment rows r0, r0 + 8 of the tile
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int b, lt, nt;
    tile_pos(tile, b, lt, nt);
    float sum[64], acc[64];
    for (int kc = 0; kc < a.kchunks; ++kc, ++it) {
      const int s = (int)(it & 3u);
      tc::mbar_wait_u(FULL(s), (it >> 2) & 1u);                    // weights and activation of this chunk have landed
      const unsigned char* st = smem + C::OFF_A + (size_t)s * kSStageBytes;
      const int k0 = kc * kKC;
      uint32_t ahi[4][4], alo[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int row = r0 + ((q & 1) ? 8 : 0), k = 8 * ks + t + ((q & 2) ? 4 : 0);
          float x;
          if constexpr (ACT == ACT_ROW) {
            x = *reinterpret_cast<const float*>(st + row * 128 + (((k >> 2) ^ (row & 7)) << 4) + (k & 3) * 4);
          } else {
            const float* sp = reinterpret_cast<const float*>(st + k * kAPitchCh) + row;
            if constexpr (FN != FN_NONE) {
              x = act_fn<FN>(sp[0]);       // zero-filled staging (tails of K and L) stays zero: gelu(0) = 0
            } else if (!use_fir) {
              x = sp[0];
            } else {
              // dp[t] = w2 ds[t] + w1 ds[t+1] + w0 ds[t+2]; ds beyond the tensor end is staged as zero, a position
              // beyond the processed range produces a value nobody stores; channels >= K are staged as zero
              const float* w = fir_s + 3 * (k0 + k < a.K ? k0 + k : 0);
              x = fmaf(w[2], sp[0], fmaf(w[1], sp[1], w[0] * sp[2]));
            }
          }
          float hh, lw;
          tc::split_tf32(x, hh, lw);
          ahi[ks][q] = __float_as_uint(hh); alo[ks][q] = __float_as_uint(lw);
        }
      }
      // a fresh accumulation per chunk: the correction products (lo*hi, hi*lo; 2^-11 of the result) first, the four
      // hi*hi products last, so that only those add at full scale; chunks are summed with round-to-nearest adds
      const uint32_t bhi = sbase + s * C::STAGE_BYTES, blo = bhi + C::STAGE_BYTES / 2;
      tc::wgmma_fence();
      tc::fence_regs(acc);
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        tc::wgmma_rs_n128(acc, alo[ks], tc::make_desc_ls(bhi + ks * 2 * kLBO, kLBO, kSBO), ks ? 1u : 0u);
        tc::wgmma_rs_n128(acc, ahi[ks], tc::make_desc_ls(blo + ks * 2 * kLBO, kLBO, kSBO), 1u);
      }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        tc::wgmma_rs_n128(acc, ahi[ks], tc::make_desc_ls(bhi + ks * 2 * kLBO, kLBO, kSBO), 1u);
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
      tc::fence_regs(acc);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(EMPTY(s));                    // weight stage and staging slot are free
      if (kc == 0) {
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = acc[i];
      } else {
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] += acc[i];
      }
    }
    // epilogue: element i of the fragment = (row r0 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 t + (i & 1))
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int l = lt + r0 + 8 * h;
      if (l >= lend) continue;
      float pre[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        if constexpr (OUT == OUT_CH && FN != FN_NONE) {
          // gradient epilogue: the pre-activation values of eight column pairs are fetched together, so that their
          // loads are in flight at once instead of each one stalling the multiply that consumes it
          if (j % 8 == 0) {
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int n = nt * NT + 8 * (j + (i >> 1)) + 2 * t + (i & 1);
              pre[i] = n < a.N ? __ldg(a.aux + ((size_t)b * a.N + n) * a.L + l) : 0.f;
            }
          }
        }
        const int n = nt * NT + 8 * j + 2 * t;
        float v0 = sum[4 * j + 2 * h], v1 = sum[4 * j + 2 * h + 1];
        if constexpr (OUT == OUT_CH && FN != FN_NONE) {
          float* dst = a.out + ((size_t)b * a.N + n) * a.L + l;
          if (n < a.N) dst[0] = v0 * act_grad<FN>(pre[2 * (j % 8)]);
          if (n + 1 < a.N) dst[a.L] = v1 * act_grad<FN>(pre[2 * (j % 8) + 1]);
        } else if constexpr (OUT == OUT_CH) {
          float* dst = a.out + ((size_t)b * a.N + n) * a.L + l;
          if (n < a.N) dst[0] = v0 + (a.bias ? __ldg(a.bias + n) : 0.f);
          if (n + 1 < a.N) dst[a.L] = v1 + (a.bias ? __ldg(a.bias + n + 1) : 0.f);
        } else {
          float* dst = a.out + ((size_t)b * a.L + l) * a.N + n;
          if (a.bias) {
            if (n < a.N) v0 += __ldg(a.bias + n);
            if (n + 1 < a.N) v1 += __ldg(a.bias + n + 1);
          }
          if (n + 1 < a.N && (a.N & 1) == 0) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
          else {
            if (n < a.N) dst[0] = v0;
            if (n + 1 < a.N) dst[1] = v1;
          }
        }
      }
    }
  }
}

}  // namespace pg

// ================================================================================================ weight gradients
// dW[m][n] = sum_{b,pos} X[b][m][pos] * Y[b][pos][n]: the reduction runs over the (up to 2^20) sequence positions.
// Computed as its transpose, T[n][m] = sum_pos Y[pos][n] X[m][pos], so that both operands sit in their natural layout
// (wgmma takes tf32 operands K-major only):
//   A operand = Y^T: 128 columns n of Y per tile, two consumer warpgroups of 64; each thread loads its A fragments
//               (Y[pos][n] of the staged chunk), (hi, lo) split in registers
//   B operand = X:   128 rows m per tile, K = position contiguous in memory = K-major; four converter warps turn the
//               staged rows into hi / lo K-major core-matrix images (one 16-byte piece = four consecutive positions of
//               one row; optional transposed short filter on the fly from six staged samples)
//   staging   both tiles of a chunk arrive by TMA into shared-memory rings, four chunks in flight
//   split-K   CTA = (n tile, m tile, slice of the position chunks), one partial per CTA, summed in fixed order by
//             wgrad_reduce_kernel (deterministic, no atomics).
//   accuracy  the tensor core adds into its accumulator with truncation: a chain of n MMAs biases the sum by ~n 2^-24
//             towards zero, and a slice here is thousands of MMAs long.  So the accumulator is restarted every kSeg chunks
//             (the correction products of a chunk first, its hi*hi products last) and added into a running sum in
//             registers with round-to-nearest adds; the CTA writes its partial once, at the end of its slice.
//   registers acc 64 + sum 64 + A fragments 32 + next chunk's Y 16 per consumer thread: whole warpgroups, and moves
//             registers from the converter and producer warpgroups to the consumers (setmaxnreg).
//   overlap   the next chunk's Y values are loaded while this chunk's MMAs run; the converters fill the other image pair.
namespace wg {

constexpr int kThreads = 512;             // warpgroups: 0, 1 consumers; 2 X -> B images; 3 TMA producer (one warp)
constexpr int kRegConsumer = 184, kRegConvert = 88, kRegProducer = 56;   // setmaxnreg; 128 each at launch
static_assert(2 * kRegConsumer + kRegConvert + kRegProducer <= 4 * 128, "register file of one CTA");
constexpr int kSeg = 4;                   // chunks per accumulation segment (48 chained MMAs)
constexpr int kStg = 4;                   // staged chunks in flight
constexpr uint32_t kYPitch = 128 * 4;     // staged Y row: 128 columns, dense (= the TMA box)
constexpr uint32_t kYStage = 32 * kYPitch;            // 32 positions
constexpr uint32_t kXPitch = 36 * 4;      // staged X row: 32 positions + one look-ahead quad (fused FIR)
constexpr uint32_t kXStage = 128 * kXPitch;           // 128 rows
constexpr uint32_t kImg = 128 * 32 * 4;               // one 128 x 32 operand image (16 KB)
constexpr uint32_t kOffY = 0, kOffX = kOffY + kStg * kYStage;
constexpr uint32_t kOffImg = (kOffX + kStg * kXStage + 1023u) & ~1023u;                       // images: [2][hi | lo]
constexpr uint32_t kOffBar = kOffImg + 2 * 2 * kImg;
constexpr size_t kSmem = kOffBar + 256;
static_assert(kOffImg % 1024 == 0, "operand images must start on a core-matrix group boundary");
static_assert(kYStage % 128 == 0 && kXStage % 128 == 0, "TMA destinations are 128-byte aligned");
static_assert(kSmem <= 227 * 1024, "shared memory budget");

struct Args {
  const float* X;       // (B, M, L)
  const float* Y;       // (B, L, N)
  const float* fir;     // (M, 3) or null
  float* part;          // (splits, N, M) partial sums of the TRANSPOSED product
  int B, L, M, N;
  int chunks_per_b;     // ceil(L / 32)
  int mtiles, ntiles, splits;
  int vec;              // 1: both tensors qualify for TMA (16-byte aligned rows): the tensor maps are valid
  unsigned zero;        // 0 at run time (tc::mbar_arrive_after_loads)
};

// Staging: one producer thread issues, per chunk of 32 positions, ONE tiled TMA copy of the Y tile (box 128 n x 32 pos of
// the (N, L, B) tensor) and one of the X tile (box 36 pos x 128 m of the (L, M, B) tensor; four look-ahead samples for
// the fused FIR), completion on an mbarrier per stage.  Out-of-range rows / columns / positions are zero-filled by the
// copy engine (tails of M, N and L; the 3-D maps keep a tile from running into the next batch).
// FN != FN_NONE: the product is taken with gelu(X) (fir must be null), applied by the converter warps.
template <int FN = FN_NONE>
__global__ void __launch_bounds__(kThreads, 1) wgrad_kernel(const Args a, const __grid_constant__ CUtensorMap tmapX,
                                                            const __grid_constant__ CUtensorMap tmapY) {
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  // barriers: b_full[2] b_empty[2] s_full[4] y_empty[4] x_empty[4]
  const uint32_t sbase = tc::smem_u32(smem), bar0 = tc::smem_u32(bars);
  auto B_FULL = [&](int s) { return bar0 + 8u * s; };
  auto B_EMPTY = [&](int s) { return bar0 + 8u * (2 + s); };
  auto S_FULL = [&](int j) { return bar0 + 8u * (4 + j); };
  auto Y_EMPTY = [&](int j) { return bar0 + 8u * (8 + j); };
  auto X_EMPTY = [&](int j) { return bar0 + 8u * (12 + j); };
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) { tc::mbar_init(B_FULL(s), 128); tc::mbar_init(B_EMPTY(s), 8); }
    for (int j = 0; j < kStg; ++j) { tc::mbar_init(S_FULL(j), 1); tc::mbar_init(Y_EMPTY(j), 256); tc::mbar_init(X_EMPTY(j), 128); }
  }
  __syncthreads();

  // work item of this CTA
  const int split = blockIdx.x % a.splits;
  const int tile = blockIdx.x / a.splits;
  const int nt = tile / a.mtiles, mt = tile - nt * a.mtiles;
  const int n0 = nt * 128, m0 = mt * 128;
  const int nrows = min(128, a.N - n0);                                 // valid accumulator rows
  const int mcols = min(128, a.M - m0);                                 // valid accumulator columns
  const long long total_chunks = (long long)a.B * a.chunks_per_b;
  const long long c_begin = total_chunks * split / a.splits, c_end = total_chunks * (split + 1) / a.splits;
  const long long nchunks = c_end - c_begin;

  if (warp < 8) {
    // ---------------------------------------------------------------- consumers: rows n [64 wg, 64 wg + 64) of the tile
    tc::setmaxnreg_inc<kRegConsumer>();
    const int wgi = warp >> 2, g = lane >> 2, t = lane & 3;
    const int nl0 = 64 * wgi + 16 * (warp & 3) + g;                     // fragment rows nl0, nl0 + 8
    float acc[64], sum[64], yv[4][4];
#pragma unroll
    for (int i = 0; i < 64; ++i) sum[i] = 0.f;
    // this thread's A-fragment values of chunk q from the staged Y tile; the slot is released once they have arrived
    auto load_y = [&](long long q) {
      const int ss = (int)(q % kStg);
      tc::mbar_wait_u(S_FULL(ss), (uint32_t)(q / kStg) & 1u);            // the producer's copies of this chunk have landed
      const unsigned char* st = smem + kOffY + (size_t)ss * kYStage;
      uint32_t dep = 0;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int nl = nl0 + ((e & 1) ? 8 : 0), k = 8 * ks + t + ((e & 2) ? 4 : 0);
          yv[ks][e] = *reinterpret_cast<const float*>(st + k * kYPitch + nl * 4);
          dep |= __float_as_uint(yv[ks][e]);
        }
      }
      tc::mbar_arrive_after_loads(Y_EMPTY(ss), dep, a.zero);            // staged Y tile consumed: the producer may refill it
    };
    if (nchunks > 0) load_y(0);
    for (long long q = 0; q < nchunks; ++q) {
      uint32_t ahi[4][4], alo[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float h, lw;
          tc::split_tf32(yv[ks][e], h, lw);
          ahi[ks][e] = __float_as_uint(h); alo[ks][e] = __float_as_uint(lw);
        }
      }
      const uint32_t it = (uint32_t)q;
      const int s = it & 1;
      tc::mbar_wait_u(B_FULL(s), (it >> 1) & 1);
      const uint32_t bhi = sbase + kOffImg + s * 2 * kImg, blo = bhi + kImg;
      const uint32_t cont = (it % kSeg) != 0;                           // 0: this chunk starts a segment
      tc::wgmma_fence();
      tc::fence_regs(acc);
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {                                  // corrections: lo * hi, hi * lo
        tc::wgmma_rs_n128(acc, alo[ks], tc::make_desc_ls(bhi + ks * 2 * pg::kLBO, pg::kLBO, pg::kSBO), (cont | ks) ? 1u : 0u);
        tc::wgmma_rs_n128(acc, ahi[ks], tc::make_desc_ls(blo + ks * 2 * pg::kLBO, pg::kLBO, pg::kSBO), 1u);
      }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)                                    // main: hi * hi
        tc::wgmma_rs_n128(acc, ahi[ks], tc::make_desc_ls(bhi + ks * 2 * pg::kLBO, pg::kLBO, pg::kSBO), 1u);
      tc::wgmma_commit();
      if (q + 1 < nchunks) load_y(q + 1);                               // under this chunk's MMAs
      tc::wgmma_wait<0>();
      tc::fence_regs(acc);
      tc::fence_frags(ahi);                                             // read by the MMAs up to here
      tc::fence_frags(alo);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(B_EMPTY(s));                       // the image pair is free
      if (it % kSeg == kSeg - 1 || q + 1 == nchunks) {                  // end of a segment: sum += acc (round to nearest)
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = acc[i] + sum[i];
      }
    }
    // the CTA's partial, written once (zero for an empty slice)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int nl = nl0 + 8 * h;
      if (nl >= nrows) continue;
      float* dst = a.part + ((size_t)split * a.N + n0 + nl) * a.M + m0;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int ml = 8 * j + 2 * t;
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (ml + e < mcols) dst[ml + e] = sum[4 * j + 2 * h + e];
      }
    }
  } else if (warp < 12) {
    // ---------------------------------------------------------------- B side: X rows -> K-major hi / lo images
    tc::setmaxnreg_dec<kRegConvert>();
    const int t = tid - 256;
    const bool use_fir = a.fir != nullptr;
    // this thread converts pieces (row r, quad k4) with r % 8 == t % 8: the eight lanes of a quarter warp then write one
    // contiguous 128-byte core matrix (bank-conflict free); 1024 pieces per chunk, 8 per thread
    const int rlo = t & 7, kq = (t >> 3) & 7, rhi0 = t >> 6;            // rows r = rlo + 8 * (rhi0 + 2 i), i < 8
    float w[8][3];
    if (use_fir) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int m = m0 + rlo + 8 * (rhi0 + 2 * i);
#pragma unroll
        for (int j = 0; j < 3; ++j) w[i][j] = (m < a.M) ? __ldg(a.fir + 3 * m + j) : 0.f;
      }
    }
    for (long long q = 0; q < nchunks; ++q) {
      const int ss = (int)(q % kStg);
      tc::mbar_wait_u(S_FULL(ss), (uint32_t)(q / kStg) & 1u);
      const unsigned char* st = smem + kOffX + (size_t)ss * kXStage;
      const uint32_t it = (uint32_t)q;
      const int s = it & 1;
      tc::mbar_wait_u(B_EMPTY(s), ((it >> 1) & 1) ^ 1);                 // the MMAs that read this image pair are done
      unsigned char* hi_img = smem + kOffImg + (size_t)s * 2 * kImg;
      unsigned char* lo_img = hi_img + kImg;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = rlo + 8 * (rhi0 + 2 * i);
        const float* row = reinterpret_cast<const float*>(st + r * kXPitch) + 4 * kq;
        float4 v = *reinterpret_cast<const float4*>(row);
        if (use_fir) {
          const float2 nx = *reinterpret_cast<const float2*>(row + 4);
          const float x4 = nx.x, x5 = nx.y;
          float4 o;
          o.x = fmaf(w[i][2], v.x, fmaf(w[i][1], v.y, w[i][0] * v.z));
          o.y = fmaf(w[i][2], v.y, fmaf(w[i][1], v.z, w[i][0] * v.w));
          o.z = fmaf(w[i][2], v.z, fmaf(w[i][1], v.w, w[i][0] * x4));
          o.w = fmaf(w[i][2], v.w, fmaf(w[i][1], x4, w[i][0] * x5));
          v = o;
        }
        if constexpr (FN != FN_NONE) {                                 // zero fill outside the tensor stays zero
          v.x = act_fn<FN>(v.x); v.y = act_fn<FN>(v.y); v.z = act_fn<FN>(v.z); v.w = act_fn<FN>(v.w);
        }
        float4 h, lw;
        tc::split_tf32(v.x, h.x, lw.x); tc::split_tf32(v.y, h.y, lw.y);
        tc::split_tf32(v.z, h.z, lw.z); tc::split_tf32(v.w, h.w, lw.w);
        const uint32_t off = pg::img_off(r, 4 * kq);
        *reinterpret_cast<float4*>(hi_img + off) = h;
        *reinterpret_cast<float4*>(lo_img + off) = lw;
      }
      tc::mbar_arrive(X_EMPTY(ss));                                     // staged rows consumed
      tc::fence_async_smem();
      tc::mbar_arrive(B_FULL(s));
    }
  } else {
    // ---------------------------------------------------------------- producer: Y and X tiles of every chunk (TMA)
    tc::setmaxnreg_dec<kRegProducer>();
    if (warp != 12) return;
    if (lane == 0 && a.vec) { tc::tma_prefetch_desc(&tmapX); tc::tma_prefetch_desc(&tmapY); }
    int sb_ = (int)(c_begin / a.chunks_per_b), sl_ = (int)(c_begin - (long long)sb_ * a.chunks_per_b) * 32;
    for (long long q = 0; q < nchunks; ++q) {
      const int ss = (int)(q % kStg);
      const uint32_t par = ((uint32_t)(q / kStg) & 1u) ^ 1u;
      const int b = sb_, l0 = sl_;
      sl_ += 32;
      if (sl_ >= a.chunks_per_b * 32) { sl_ = 0; ++sb_; }
      tc::mbar_wait_u(Y_EMPTY(ss), par);
      tc::mbar_wait_u(X_EMPTY(ss), par);
      if (a.vec) {
        if (lane == 0) {
          tc::mbar_arrive_expect_tx(S_FULL(ss), kYStage + kXStage);
          tc::tma_load_3d(sbase + kOffY + ss * kYStage, &tmapY, n0, l0, b, S_FULL(ss));
          tc::tma_load_3d(sbase + kOffX + ss * kXStage, &tmapX, l0, m0, b, S_FULL(ss));
        }
      } else {
        // rows that do not qualify for TMA: the 32 lanes stage the tiles with plain loads (zero fill outside the tensors)
        float* ys = reinterpret_cast<float*>(smem + kOffY + (size_t)ss * kYStage);
        for (int i = lane; i < 32 * 128; i += 32) {
          const int k = i >> 7, n = i & 127, l = l0 + k;
          ys[i] = (l < a.L && n0 + n < a.N) ? __ldg(a.Y + ((size_t)b * a.L + l) * a.N + n0 + n) : 0.f;
        }
        float* xs = reinterpret_cast<float*>(smem + kOffX + (size_t)ss * kXStage);
        for (int i = lane; i < 128 * 36; i += 32) {
          const int r = i / 36, e = i - r * 36, l = l0 + e;
          xs[i] = (m0 + r < a.M && l < a.L) ? __ldg(a.X + ((size_t)b * a.M + m0 + r) * a.L + l) : 0.f;
        }
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(S_FULL(ss));
      }
    }
  }
}

// dW = sum over splits of part^T (fixed order: deterministic).  part is (splits, N, M); dW is (M, N), or (N, M) when
// `transposed` (then no transposition is left to do)
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dW, int splits, int M, int N,
                                    int transposed, float beta) {
  const size_t total = (size_t)M * N;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    // i indexes the OUTPUT; fetch part[n][m]
    size_t src;
    if (transposed) src = i;                                            // dW (N, M) == part layout
    else { const int m = (int)(i / N), n = (int)(i - (size_t)m * N); src = (size_t)n * M + m; }
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += part[(size_t)k * total + src];
    dW[i] = (beta != 0.f) ? fmaf(beta, dW[i], s) : s;
  }
}

}  // namespace wg
}  // namespace hy
