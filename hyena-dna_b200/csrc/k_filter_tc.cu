#include "launch.h"
#include "filter_tc.cuh"
namespace hy {

size_t filter_tc_wimg_bytes(int D) {
  const size_t a = tc::wimg_floats(D), b = tc::wimg_bwd_floats(D);
  return (a > b ? a : b) * sizeof(float);
}

cudaError_t launch_filter_bwd_tc(const FilterParams& P, float* wimg, const float* dk, float* dh, float* scratch,
                                 cudaStream_t s) {
  cudaError_t e = set_smem(tc::filter_tc_bwd_kernel, tc::kSmemBytes);
  if (e != cudaSuccess) return e;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  prof_begin(K_FILTER_TC_PREP, s);
  tc::filter_tc_prep_bwd_kernel<<<64, 256, 0, s>>>(P.W1, P.W2, P.W3, P.D, wimg);
  prof_end(K_FILTER_TC_PREP, s);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int ntiles = (P.L + tc::kTileM - 1) / tc::kTileM;
  const int grid = ntiles < sms ? ntiles : sms;
  prof_begin(K_FILTER_TC_BWD, s);
  tc::filter_tc_bwd_kernel<<<grid, tc::kThreads, tc::kSmemBytes, s>>>(P, wimg, dk, dh, scratch, ntiles);
  prof_end(K_FILTER_TC_BWD, s);
  return cudaGetLastError();
}

cudaError_t launch_filter_fwd_tc(const FilterParams& P, float* wimg, float* kout, cudaStream_t s) {
  cudaError_t e = set_smem(tc::filter_tc_fwd_kernel, tc::kSmemBytes);
  if (e != cudaSuccess) return e;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  prof_begin(K_FILTER_TC_PREP, s);
  tc::filter_tc_prep_kernel<<<64, 256, 0, s>>>(P.W1, P.W2, P.W3, P.D, wimg);
  prof_end(K_FILTER_TC_PREP, s);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int ntiles = (P.L + tc::kTileM - 1) / tc::kTileM;
  const int grid = ntiles < sms ? ntiles : sms;
  prof_begin(K_FILTER_TC_FWD, s);
  tc::filter_tc_fwd_kernel<<<grid, tc::kThreads, tc::kSmemBytes, s>>>(P, wimg, kout, ntiles);
  prof_end(K_FILTER_TC_FWD, s);
  return cudaGetLastError();
}

// work: [zT; 1] (E + 1, L), then the partials of the three GEMMs of stage 2 (filter_tc.cuh), each 16-byte aligned
static size_t ones_floats(int L, int E) { return ((size_t)(E + 1) * L + 3) & ~(size_t)3; }

size_t filter_red_work_bytes(int L, int D, int E) {
  return ones_floats(L, E) * sizeof(float) + proj_wgrad_scratch_bytes(D, 64) + proj_wgrad_scratch_bytes(128, 128) +
         proj_wgrad_scratch_bytes(256, E + 1);
}

cudaError_t launch_filter_stage2(const RedLaunch& r, float* work, cudaStream_t s) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t arr = (size_t)64 * r.L;                   // floats per stage-1 array: a1 a2 a3 dp1 dp2 dp3 X
  float* zt1 = work;
  float* p1 = zt1 + ones_floats(r.L, r.E);
  float* p2 = p1 + proj_wgrad_scratch_bytes(r.D, 64) / sizeof(float);
  float* p3 = p2 + proj_wgrad_scratch_bytes(128, 128) / sizeof(float);
  prof_begin(K_FILTER_TC_RED, s);
  tc::filter_red_ones_kernel<<<2 * sms, 256, 0, s>>>(r.zT, r.E, r.L, zt1);
  prof_end(K_FILTER_TC_RED, s);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  tc::RedFinish f{p1, p2, p3, 0, 0, 0, r.dW0, r.db0, r.dW1, r.db1, r.dW2, r.db2, r.dW3, r.dfreq, r.D, r.E};
  e = launch_wgrad_part(r.dh, r.scratch + 2 * arr, 1, nullptr, 1, r.L, r.D, 64, p1, s, 0, K_FILTER_TC_RED, &f.s1);
  if (e != cudaSuccess) return e;
  e = launch_wgrad_part(r.scratch + 4 * arr, r.scratch, 1, nullptr, 1, r.L, 128, 128, p2, s, 0, K_FILTER_TC_RED, &f.s2);
  if (e != cudaSuccess) return e;
  e = launch_wgrad_part(r.scratch + 3 * arr, zt1, 1, nullptr, 1, r.L, 256, r.E + 1, p3, s, 0, K_FILTER_TC_RED, &f.s3);
  if (e != cudaSuccess) return e;
  const int total = r.D * 64 + 2 * 64 * 64 + 64 * r.E + 4 * 64;
  prof_begin(K_FILTER_TC_RED, s);
  tc::filter_red_finish_kernel<<<(total + 255) / 256, 256, 0, s>>>(f);
  prof_end(K_FILTER_TC_RED, s);
  return cudaGetLastError();
}

}  // namespace hy
