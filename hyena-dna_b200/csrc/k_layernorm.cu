// Launchers of the residual-add + LayerNorm kernels (layernorm.cuh).
#include "launch.h"
#include "layernorm.cuh"

namespace hy {

static int ln_grid(long long rows) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long want = (rows + ln::kWarps - 1) / ln::kWarps;
  long long cap = 8LL * sms;                         // 8 CTAs of 8 warps per SM: a whole number of waves
  return (int)(want < cap ? (want < 1 ? 1 : want) : cap);
}
int ln_partials(long long rows) { return ln_grid(rows); }

static bool aligned16p(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

cudaError_t launch_add_ln_fwd(const ln::FwdArgs& a, cudaStream_t s) {
  const int grid = ln_grid(a.rows);
  const bool vec = (a.D % 4 == 0) && a.D <= 128 * ln::kMaxV && aligned16p(a.x) && aligned16p(a.y) && aligned16p(a.w) &&
                   (!a.res || aligned16p(a.res)) && (!a.res_out || aligned16p(a.res_out)) && (!a.b || aligned16p(a.b));
  prof_begin(K_ADD_LN, s);
  if (!vec) ln::add_ln_fwd_generic_kernel<<<grid, 32 * ln::kWarps, 0, s>>>(a);
  else if (a.D <= 128) ln::add_ln_fwd_kernel<1><<<grid, 32 * ln::kWarps, 0, s>>>(a);
  else if (a.D <= 256) ln::add_ln_fwd_kernel<2><<<grid, 32 * ln::kWarps, 0, s>>>(a);
  else if (a.D <= 512) ln::add_ln_fwd_kernel<4><<<grid, 32 * ln::kWarps, 0, s>>>(a);
  else ln::add_ln_fwd_kernel<8><<<grid, 32 * ln::kWarps, 0, s>>>(a);
  prof_end(K_ADD_LN, s);
  return cudaGetLastError();
}

cudaError_t launch_add_ln_bwd(ln::BwdArgs a, float* dw, float* db, cudaStream_t s) {
  const int grid = ln_grid(a.rows);
  const bool vec = (a.D % 4 == 0) && a.D <= 128 * ln::kMaxV && aligned16p(a.dy) && aligned16p(a.r) && aligned16p(a.dx) &&
                   aligned16p(a.w) && (!a.dres || aligned16p(a.dres));
  prof_begin(K_ADD_LN, s);
  if (!vec) {
    ln::add_ln_bwd_generic_kernel<<<grid, 32 * ln::kWarps, 0, s>>>(a);
  } else {
    const size_t sh = (size_t)ln::kWarps * 2 * a.D * sizeof(float);     // <= 64 KB at D = 1024
    cudaError_t e = cudaSuccess;
    if (a.D <= 128) { e = set_smem(ln::add_ln_bwd_kernel<1>, sh); if (e == cudaSuccess) ln::add_ln_bwd_kernel<1><<<grid, 32 * ln::kWarps, sh, s>>>(a); }
    else if (a.D <= 256) { e = set_smem(ln::add_ln_bwd_kernel<2>, sh); if (e == cudaSuccess) ln::add_ln_bwd_kernel<2><<<grid, 32 * ln::kWarps, sh, s>>>(a); }
    else if (a.D <= 512) { e = set_smem(ln::add_ln_bwd_kernel<4>, sh); if (e == cudaSuccess) ln::add_ln_bwd_kernel<4><<<grid, 32 * ln::kWarps, sh, s>>>(a); }
    else { e = set_smem(ln::add_ln_bwd_kernel<8>, sh); if (e == cudaSuccess) ln::add_ln_bwd_kernel<8><<<grid, 32 * ln::kWarps, sh, s>>>(a); }
    if (e != cudaSuccess) return e;
  }
  prof_end(K_ADD_LN, s);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  prof_begin(K_ADD_LN, s);
  ln::ln_reduce_kernel<<<(2 * a.D + 255) / 256, 256, 0, s>>>(a.part, grid, a.D, dw, db);
  prof_end(K_ADD_LN, s);
  return cudaGetLastError();
}

}  // namespace hy
