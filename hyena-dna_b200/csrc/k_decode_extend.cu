// Launchers of the multi-position decoding kernels (decode_extend.cuh).
#include "launch.h"
#include "decode_extend.cuh"

namespace hy {

template <class T>
cudaError_t launch_decode_ext_hist(const dec::ExtHistArgsT<T>& a, cudaStream_t s) {
  prof_begin(K_DECODE_EXT_HIST, s);
  dec::decode_ext_hist_kernel<T><<<a.B * a.D, 256, 0, s>>>(a);
  prof_end(K_DECODE_EXT_HIST, s);
  return cudaGetLastError();
}

template <int BG, int NT, class T>
static void ext_dot(const dec::ExtDotArgsT<T>& a, dim3 grid, cudaStream_t s) {
  dec::decode_ext_dot_kernel<BG, NT, T><<<grid, 32 * dec::kExtWarps, 0, s>>>(a);
}

template <int NT, class T>
static void ext_dot_bg(const dec::ExtDotArgsT<T>& a, int BG, dim3 grid, cudaStream_t s) {
  switch (BG) {
    case 1: ext_dot<1, NT>(a, grid, s); break;
    case 2: ext_dot<2, NT>(a, grid, s); break;
    case 4: ext_dot<4, NT>(a, grid, s); break;
    default: ext_dot<8, NT>(a, grid, s); break;
  }
}

// grid: (groups x output tiles, D, batch groups); the tile size and batch group follow n and B (decode_args.h)
template <class T>
cudaError_t launch_decode_ext_dot(const dec::ExtDotArgsT<T>& a, cudaStream_t s) {
  const int BG = dec::ext_bg(a.B), NT = dec::ext_tile(a.n);
  dim3 grid(a.groups * a.njt, a.D, (a.B + BG - 1) / BG);
  prof_begin(K_DECODE_EXT_DOT, s);
  if (NT == 8) ext_dot_bg<8>(a, BG, grid, s);
  else ext_dot_bg<64>(a, BG, grid, s);
  prof_end(K_DECODE_EXT_DOT, s);
  return cudaGetLastError();
}

template <class T>
cudaError_t launch_decode_ext_combine(const dec::ExtCombineArgsT<T>& a, cudaStream_t s) {
  const long long n = (long long)a.B * a.D * a.n;
  prof_begin(K_DECODE_EXT_COMBINE, s);
  dec::decode_ext_combine_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a);
  prof_end(K_DECODE_EXT_COMBINE, s);
  return cudaGetLastError();
}

template <class T>
cudaError_t launch_decode_branch_combine(const dec::BranchCombineArgsT<T>& a, cudaStream_t s) {
  const long long n = (long long)a.c.B * a.c.D * a.c.n;
  prof_begin(K_DECODE_EXT_COMBINE, s);
  dec::decode_branch_combine_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a);
  prof_end(K_DECODE_EXT_COMBINE, s);
  return cudaGetLastError();
}

// the history element types (decode_args.h): float, and the 16-bit histories
#define HY_DECODE_EXT_INSTANTIATE(T)                                                                 \
  template cudaError_t launch_decode_ext_hist<T>(const dec::ExtHistArgsT<T>&, cudaStream_t);         \
  template cudaError_t launch_decode_ext_dot<T>(const dec::ExtDotArgsT<T>&, cudaStream_t);           \
  template cudaError_t launch_decode_ext_combine<T>(const dec::ExtCombineArgsT<T>&, cudaStream_t);   \
  template cudaError_t launch_decode_branch_combine<T>(const dec::BranchCombineArgsT<T>&, cudaStream_t);
HY_DECODE_EXT_INSTANTIATE(float)
HY_DECODE_EXT_INSTANTIATE(__half)
HY_DECODE_EXT_INSTANTIATE(__nv_bfloat16)
#undef HY_DECODE_EXT_INSTANTIATE

}  // namespace hy
