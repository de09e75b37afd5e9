// Block glue either side of the mixer (SURVEY.md S8 f1): residual add + LayerNorm in one pass, forward and backward.
//
// Reference: flash-attention/flash_attn/modules/block.py:111-148 (pre-norm Block: dropout -> add -> LayerNorm with
// residual_in_fp32; dropout p = 0 in every HyenaDNA config) and flash_attn.ops.layer_norm.dropout_add_layer_norm, the
// fused op that Block calls with fused_dropout_add_ln=True (src/models/sequence/long_conv_lm.py:139-200 builds the
// blocks, :377-396 runs them and applies the final norm the same way).
//
//   forward   r = x (+ res);  mean, rstd over the D features of a row;  y = (r - mean) * rstd * w + b
//             one warp per row, the row lives in registers (two sweeps: mean, then centred sum of squares);
//             HBM traffic 4 x 4 D bytes per row (x, res in; r, y out) + 8 bytes of statistics
//   backward  g = dy * w;  dr = rstd * (g - mean_D(g) - xhat * mean_D(g * xhat)) + dres;  dx = dres_in = dr
//             dw += sum_rows dy * xhat,  db += sum_rows dy: per-CTA partials written to a (CTAs, 2, D) scratch and
//             summed in fixed order by ln_reduce_kernel (deterministic, no atomics).  Register path: per-lane sums over
//             the CTA's rows, combined across its warps in shared memory.  Generic path: per-thread column sums over a
//             contiguous block of rows, no shared memory.
// fp32 throughout (residual_in_fp32 semantics).  Memory-bound elementwise work: coalesced float4 rows, grid = a multiple
// of the SM count, no shared-memory staging needed.
#pragma once
#include "common.cuh"
#include "layernorm_args.h"

namespace hy {
namespace ln {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// NV float4 per lane cover D (D % 4 == 0, D <= 128 * NV)
template <int NV>
__global__ void __launch_bounds__(32 * kWarps) add_ln_fwd_kernel(const FwdArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int D4 = a.D >> 2;
  float4 w4[NV], b4[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    w4[i] = c < D4 ? __ldg(reinterpret_cast<const float4*>(a.w) + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    b4[i] = (c < D4 && a.b) ? __ldg(reinterpret_cast<const float4*>(a.b) + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float invD = 1.0f / (float)a.D;
  for (long long row = (long long)blockIdx.x * kWarps + warp; row < a.rows; row += (long long)gridDim.x * kWarps) {
    const float4* xr = reinterpret_cast<const float4*>(a.x + row * a.D);
    const float4* rr = a.res ? reinterpret_cast<const float4*>(a.res + row * a.D) : nullptr;
    float4 v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < D4) {
        v[i] = __ldg(xr + c);
        if (rr) { const float4 r = __ldg(rr + c); v[i].x += r.x; v[i].y += r.y; v[i].z += r.z; v[i].w += r.w; }
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
      }
    }
    const float mean = warp_sum(s) * invD;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < D4) {
        const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
        q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
    }
    const float rstd = rsqrtf(warp_sum(q) * invD + a.eps);
    if (lane == 0) { a.mean[row] = mean; a.rstd[row] = rstd; }
    float4* ro = a.res_out ? reinterpret_cast<float4*>(a.res_out + row * a.D) : nullptr;
    float4* yo = reinterpret_cast<float4*>(a.y + row * a.D);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < D4) {
        if (ro) ro[c] = v[i];
        float4 o;
        o.x = fmaf((v[i].x - mean) * rstd, w4[i].x, b4[i].x);
        o.y = fmaf((v[i].y - mean) * rstd, w4[i].y, b4[i].y);
        o.z = fmaf((v[i].z - mean) * rstd, w4[i].z, b4[i].z);
        o.w = fmaf((v[i].w - mean) * rstd, w4[i].w, b4[i].w);
        yo[c] = o;
      }
    }
  }
}

// any D: scalar accesses, the row is read twice (not the HyenaDNA shapes; kept so that the entry point has no shape hole)
__global__ void __launch_bounds__(32 * kWarps) add_ln_fwd_generic_kernel(const FwdArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float invD = 1.0f / (float)a.D;
  for (long long row = (long long)blockIdx.x * kWarps + warp; row < a.rows; row += (long long)gridDim.x * kWarps) {
    const float* xr = a.x + row * a.D;
    const float* rr = a.res ? a.res + row * a.D : nullptr;
    float s = 0.f;
    for (int c = lane; c < a.D; c += 32) s += xr[c] + (rr ? rr[c] : 0.f);
    const float mean = warp_sum(s) * invD;
    float q = 0.f;
    for (int c = lane; c < a.D; c += 32) { const float d = xr[c] + (rr ? rr[c] : 0.f) - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) * invD + a.eps);
    if (lane == 0) { a.mean[row] = mean; a.rstd[row] = rstd; }
    for (int c = lane; c < a.D; c += 32) {
      const float r = xr[c] + (rr ? rr[c] : 0.f);
      if (a.res_out) a.res_out[row * a.D + c] = r;
      a.y[row * a.D + c] = fmaf((r - mean) * rstd, __ldg(a.w + c), a.b ? __ldg(a.b + c) : 0.f);
    }
  }
}

template <int NV>
__global__ void __launch_bounds__(32 * kWarps) add_ln_bwd_kernel(const BwdArgs a) {
  extern __shared__ float sh[];                       // [kWarps][2][D]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int D4 = a.D >> 2;
  float4 w4[NV], aw[NV], ab[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    w4[i] = c < D4 ? __ldg(reinterpret_cast<const float4*>(a.w) + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    aw[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    ab[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float invD = 1.0f / (float)a.D;
  for (long long row = (long long)blockIdx.x * kWarps + warp; row < a.rows; row += (long long)gridDim.x * kWarps) {
    const float mean = __ldg(a.mean + row), rstd = __ldg(a.rstd + row);
    const float4* dyr = reinterpret_cast<const float4*>(a.dy + row * a.D);
    const float4* rr = reinterpret_cast<const float4*>(a.r + row * a.D);
    const float4* dr = a.dres ? reinterpret_cast<const float4*>(a.dres + row * a.D) : nullptr;
    float4 g[NV], xh[NV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      g[i] = xh[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < D4) {
        const float4 d = __ldg(dyr + c), r = __ldg(rr + c);
        xh[i] = make_float4((r.x - mean) * rstd, (r.y - mean) * rstd, (r.z - mean) * rstd, (r.w - mean) * rstd);
        aw[i].x = fmaf(d.x, xh[i].x, aw[i].x); aw[i].y = fmaf(d.y, xh[i].y, aw[i].y);
        aw[i].z = fmaf(d.z, xh[i].z, aw[i].z); aw[i].w = fmaf(d.w, xh[i].w, aw[i].w);
        ab[i].x += d.x; ab[i].y += d.y; ab[i].z += d.z; ab[i].w += d.w;
        g[i] = make_float4(d.x * w4[i].x, d.y * w4[i].y, d.z * w4[i].z, d.w * w4[i].w);
        s1 += (g[i].x + g[i].y) + (g[i].z + g[i].w);
        s2 += fmaf(g[i].x, xh[i].x, g[i].y * xh[i].y) + fmaf(g[i].z, xh[i].z, g[i].w * xh[i].w);
      }
    }
    const float m1 = warp_sum(s1) * invD, m2 = warp_sum(s2) * invD;
    float4* dxo = reinterpret_cast<float4*>(a.dx + row * a.D);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < D4) {
        float4 o;
        o.x = rstd * (g[i].x - m1 - xh[i].x * m2); o.y = rstd * (g[i].y - m1 - xh[i].y * m2);
        o.z = rstd * (g[i].z - m1 - xh[i].z * m2); o.w = rstd * (g[i].w - m1 - xh[i].w * m2);
        if (dr) { const float4 e = __ldg(dr + c); o.x += e.x; o.y += e.y; o.z += e.z; o.w += e.w; }
        dxo[c] = o;
      }
    }
  }
  // per-CTA partials: warps in fixed order
  float* mine = sh + (size_t)warp * 2 * a.D;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < D4) {
      reinterpret_cast<float4*>(mine)[c] = aw[i];
      reinterpret_cast<float4*>(mine + a.D)[c] = ab[i];
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * a.D; j += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int wv = 0; wv < kWarps; ++wv) t += sh[(size_t)wv * 2 * a.D + j];
    a.part[(size_t)blockIdx.x * 2 * a.D + j] = t;
  }
}

// any D and any alignment, scalar accesses, no shared memory (so no limit on D).  Two independent sweeps: dx row by row
// (one warp per row, grid-stride, as the forward); then dw / db by columns over a contiguous block of rows per CTA, each
// thread summing its columns in row order into part[CTA] -- fixed order, deterministic, no atomics
__global__ void __launch_bounds__(32 * kWarps) add_ln_bwd_generic_kernel(const BwdArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float invD = 1.0f / (float)a.D;
  for (long long row = (long long)blockIdx.x * kWarps + warp; row < a.rows; row += (long long)gridDim.x * kWarps) {
    const float mean = __ldg(a.mean + row), rstd = __ldg(a.rstd + row);
    const float* dyr = a.dy + row * a.D;
    const float* rr = a.r + row * a.D;
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < a.D; c += 32) {
      const float xh = (rr[c] - mean) * rstd, g = dyr[c] * __ldg(a.w + c);
      s1 += g; s2 = fmaf(g, xh, s2);
    }
    const float m1 = warp_sum(s1) * invD, m2 = warp_sum(s2) * invD;
    for (int c = lane; c < a.D; c += 32) {
      const float xh = (rr[c] - mean) * rstd, g = dyr[c] * __ldg(a.w + c);
      a.dx[row * a.D + c] = rstd * (g - m1 - xh * m2) + (a.dres ? a.dres[row * a.D + c] : 0.f);
    }
  }
  const long long per = (a.rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = min(a.rows, (long long)blockIdx.x * per), r1 = min(a.rows, r0 + per);
  float* out = a.part + (size_t)blockIdx.x * 2 * a.D;
  for (int c = threadIdx.x; c < a.D; c += blockDim.x) {
    float sw = 0.f, sb = 0.f;
#pragma unroll 4
    for (long long row = r0; row < r1; ++row) {
      const float d = a.dy[row * a.D + c];
      sw = fmaf(d, (a.r[row * a.D + c] - __ldg(a.mean + row)) * __ldg(a.rstd + row), sw);
      sb += d;
    }
    out[c] = sw;
    out[a.D + c] = sb;
  }
}

// dw[j] (+)= sum over CTAs of part[cta][0][j]; db likewise (fixed order)
__global__ void ln_reduce_kernel(const float* __restrict__ part, int nparts, int D, float* __restrict__ dw,
                                 float* __restrict__ db) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= 2 * D) return;
  float t = 0.f;
  for (int p = 0; p < nparts; ++p) t += part[(size_t)p * 2 * D + j];
  if (j < D) dw[j] = t;
  else if (db) db[j - D] = t;
}

}  // namespace ln
}  // namespace hy
