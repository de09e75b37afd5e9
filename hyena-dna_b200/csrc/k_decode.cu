// Launchers of the incremental-decoding kernels (decode.cuh).
#include "launch.h"
#include "decode.cuh"

namespace hy {

template <class T>
cudaError_t launch_decode_hist(const dec::HistArgsT<T>& a, cudaStream_t s) {
  const int per_row = (a.P + 255) / 256;
  dim3 grid(a.B * a.D, per_row < 64 ? per_row : 64);
  prof_begin(K_DECODE_HIST, s);
  if (a.row_start) dec::decode_hist_rows_kernel<T><<<grid, 256, 0, s>>>(a);
  else dec::decode_hist_kernel<T><<<grid, 256, 0, s>>>(a);
  prof_end(K_DECODE_HIST, s);
  return cudaGetLastError();
}

// the history fill of admitted prompts: counted and timed as decode_hist (the kind list callers enumerate stays as it is)
template <class T>
cudaError_t launch_decode_admit(const dec::AdmitArgsT<T>& a, cudaStream_t s) {
  const int per_row = (a.t + 255) / 256;
  dim3 grid(a.hist.B * a.hist.D, per_row < 64 ? per_row : 64);
  prof_begin(K_DECODE_HIST, s);
  dec::decode_admit_kernel<false, T><<<grid, 256, 0, s>>>(dec::AdmitPackedArgsT<T>{a, nullptr, 0});
  prof_end(K_DECODE_HIST, s);
  return cudaGetLastError();
}

// packed prompts (cu_seqlens): the same kernel in its packed mode, with the same grid and kind
template <class T>
cudaError_t launch_decode_admit_packed(const dec::AdmitPackedArgsT<T>& a, cudaStream_t s) {
  const int per_row = (a.adm.t + 255) / 256;
  dim3 grid(a.adm.hist.B * a.adm.hist.D, per_row < 64 ? per_row : 64);
  prof_begin(K_DECODE_HIST, s);
  dec::decode_admit_kernel<true, T><<<grid, 256, 0, s>>>(a);
  prof_end(K_DECODE_HIST, s);
  return cudaGetLastError();
}

// counted by launch_count under no kind, as the position advance: it belongs to no existing kernel class
template <class T>
cudaError_t launch_decode_shift(const dec::ShiftArgsT<T>& a, long long rows, cudaStream_t s) {
  dec::decode_shift_kernel<T><<<(unsigned)rows, dec::kShiftThreads, 0, s>>>(a);
  count_launch();
  return cudaGetLastError();
}

template <int BG, class T>
static cudaError_t dot_bg(const dec::DotArgsT<T>& a, int R, dim3 grid, cudaStream_t s) {
  const int threads = 32 * dec::kDotWarps;
  switch (R) {
    case 0: dec::decode_dot_kernel<BG, 0, T><<<grid, threads, 0, s>>>(a); break;
    case 1: dec::decode_dot_kernel<BG, 1, T><<<grid, threads, 0, s>>>(a); break;
    case 2: dec::decode_dot_kernel<BG, 2, T><<<grid, threads, 0, s>>>(a); break;
    default: dec::decode_dot_kernel<BG, 3, T><<<grid, threads, 0, s>>>(a); break;
  }
  return cudaGetLastError();
}

// the split dot product over dot.t positions in nchunk chunks
template <class T>
static cudaError_t launch_dot(const dec::DotArgsT<T>& dot, int nchunk, int kind, cudaStream_t s) {
  const int BG = dot.B <= 1 ? 1 : dot.B <= 2 ? 2 : dot.B <= 4 ? 4 : 8;
  const int R = (dot.ld - 1 - dot.t) & 3;
  dim3 grid(nchunk, (dot.D + dec::kDotWarps - 1) / dec::kDotWarps, (dot.B + BG - 1) / BG);
  prof_begin(kind, s);
  cudaError_t e = BG == 1 ? dot_bg<1>(dot, R, grid, s) : BG == 2 ? dot_bg<2>(dot, R, grid, s)
                : BG == 4 ? dot_bg<4>(dot, R, grid, s) : dot_bg<8>(dot, R, grid, s);
  prof_end(kind, s);
  return e;
}

// one recurrence of one step: the split dot product over the history (skipped at t = 0), then the combine kernel
template <class T>
cudaError_t launch_decode_step(const dec::DotArgsT<T>& dot, const dec::StepArgsT<T>& st, cudaStream_t s) {
  if (st.nchunk > 0) {
    cudaError_t e = launch_dot(dot, st.nchunk, K_DECODE_STEP, s);
    if (e != cudaSuccess) return e;
  }
  const int rows = st.B * st.D;
  prof_begin(K_DECODE_STEP, s);
  dec::decode_step_kernel<T><<<(rows + dec::kStepWarps - 1) / dec::kStepWarps, 32 * dec::kStepWarps, 0, s>>>(st);
  prof_end(K_DECODE_STEP, s);
  return cudaGetLastError();
}

// one recurrence of a windowed step: the dot product over the window positions [b, t) (skipped at t = b), then the
// windowed combine kernel
template <class T>
cudaError_t launch_decode_win_step(const dec::DotArgsT<T>& dot, const dec::WinStepArgsT<T>& w, cudaStream_t s) {
  if (w.st.nchunk > 0) {
    cudaError_t e = launch_dot(dot, w.st.nchunk, K_DECODE_WIN_STEP, s);
    if (e != cudaSuccess) return e;
  }
  const int rows = w.st.B * w.st.D;
  prof_begin(K_DECODE_WIN_STEP, s);
  dec::decode_win_step_kernel<T><<<(rows + dec::kStepWarps - 1) / dec::kStepWarps, 32 * dec::kStepWarps, 0, s>>>(w);
  prof_end(K_DECODE_WIN_STEP, s);
  return cudaGetLastError();
}

// one recurrence of a branch step: the dot product over the branch's positions [b, t) (skipped at t = b), then the branch
// combine kernel; counted as a windowed step (a window whose F is selected per row)
template <class T>
cudaError_t launch_decode_branch_step(const dec::DotArgsT<T>& dot, const dec::BranchStepArgsT<T>& w, cudaStream_t s) {
  if (w.st.nchunk > 0) {
    cudaError_t e = launch_dot(dot, w.st.nchunk, K_DECODE_WIN_STEP, s);
    if (e != cudaSuccess) return e;
  }
  const int rows = w.st.B * w.st.D;
  prof_begin(K_DECODE_WIN_STEP, s);
  dec::decode_branch_step_kernel<T><<<(rows + dec::kStepWarps - 1) / dec::kStepWarps, 32 * dec::kStepWarps, 0, s>>>(w);
  prof_end(K_DECODE_WIN_STEP, s);
  return cudaGetLastError();
}

// ---- device-position steps: fixed grids, the position read by the kernels (decode.cuh *_dev_kernel)
template <class T>
static cudaError_t launch_dot_dev(const dec::DotArgsT<T>& dot, const dec::DevPos& p, int nchunk, int kind, cudaStream_t s) {
  const int BG = dot.B <= 1 ? 1 : dot.B <= 2 ? 2 : dot.B <= 4 ? 4 : 8;
  const int threads = 32 * dec::kDotWarps;
  dim3 grid(nchunk, (dot.D + dec::kDotWarps - 1) / dec::kDotWarps, (dot.B + BG - 1) / BG);
  prof_begin(kind, s);
  switch (BG) {
    case 1: dec::decode_dot_dev_kernel<1, T><<<grid, threads, 0, s>>>(dot, p); break;
    case 2: dec::decode_dot_dev_kernel<2, T><<<grid, threads, 0, s>>>(dot, p); break;
    case 4: dec::decode_dot_dev_kernel<4, T><<<grid, threads, 0, s>>>(dot, p); break;
    default: dec::decode_dot_dev_kernel<8, T><<<grid, threads, 0, s>>>(dot, p); break;
  }
  prof_end(kind, s);
  return cudaGetLastError();
}

static dim3 step_grid(int B, int D) { return dim3((B * D + dec::kStepWarps - 1) / dec::kStepWarps); }

template <class T>
cudaError_t launch_decode_step_dev(const dec::DotArgsT<T>& dot, const dec::StepArgsT<T>& st, const int* pos, int nchunk,
                                   cudaStream_t s) {
  cudaError_t e = launch_dot_dev(dot, dec::DevPos{pos, dec::kPosPlain}, nchunk, K_DECODE_STEP, s);
  if (e != cudaSuccess) return e;
  prof_begin(K_DECODE_STEP, s);
  dec::decode_step_dev_kernel<T><<<step_grid(st.B, st.D), 32 * dec::kStepWarps, 0, s>>>(st, pos);
  prof_end(K_DECODE_STEP, s);
  return cudaGetLastError();
}

template <class T>
cudaError_t launch_decode_win_step_dev(const dec::DotArgsT<T>& dot, const dec::WinStepArgsT<T>& w, const int* pos, int nchunk,
                                       cudaStream_t s) {
  cudaError_t e = launch_dot_dev(dot, dec::DevPos{pos, dec::kPosWindow}, nchunk, K_DECODE_WIN_STEP, s);
  if (e != cudaSuccess) return e;
  prof_begin(K_DECODE_WIN_STEP, s);
  dec::decode_win_step_dev_kernel<T><<<step_grid(w.st.B, w.st.D), 32 * dec::kStepWarps, 0, s>>>(w, pos);
  prof_end(K_DECODE_WIN_STEP, s);
  return cudaGetLastError();
}

template <class T>
cudaError_t launch_decode_branch_step_dev(const dec::DotArgsT<T>& dot, const dec::BranchStepArgsT<T>& w, const int* pos,
                                          int nchunk, cudaStream_t s) {
  cudaError_t e = launch_dot_dev(dot, dec::DevPos{pos, dec::kPosBranch}, nchunk, K_DECODE_WIN_STEP, s);
  if (e != cudaSuccess) return e;
  prof_begin(K_DECODE_WIN_STEP, s);
  dec::decode_branch_step_dev_kernel<T><<<step_grid(w.st.B, w.st.D), 32 * dec::kStepWarps, 0, s>>>(w, pos);
  prof_end(K_DECODE_WIN_STEP, s);
  return cudaGetLastError();
}

// counted by launch_count but under no kind: it is not a step kernel
cudaError_t launch_decode_pos_advance(int* pos, cudaStream_t s) {
  dec::decode_pos_advance_kernel<<<1, 1, 0, s>>>(pos);
  count_launch();
  return cudaGetLastError();
}

// the history element types (decode_args.h): float, and the 16-bit histories
#define HY_DECODE_INSTANTIATE(T)                                                                                          \
  template cudaError_t launch_decode_hist<T>(const dec::HistArgsT<T>&, cudaStream_t);                                     \
  template cudaError_t launch_decode_admit<T>(const dec::AdmitArgsT<T>&, cudaStream_t);                                   \
  template cudaError_t launch_decode_admit_packed<T>(const dec::AdmitPackedArgsT<T>&, cudaStream_t);                      \
  template cudaError_t launch_decode_shift<T>(const dec::ShiftArgsT<T>&, long long, cudaStream_t);                        \
  template cudaError_t launch_decode_step<T>(const dec::DotArgsT<T>&, const dec::StepArgsT<T>&, cudaStream_t);            \
  template cudaError_t launch_decode_win_step<T>(const dec::DotArgsT<T>&, const dec::WinStepArgsT<T>&, cudaStream_t);     \
  template cudaError_t launch_decode_branch_step<T>(const dec::DotArgsT<T>&, const dec::BranchStepArgsT<T>&, cudaStream_t); \
  template cudaError_t launch_decode_step_dev<T>(const dec::DotArgsT<T>&, const dec::StepArgsT<T>&, const int*, int,      \
                                                 cudaStream_t);                                                           \
  template cudaError_t launch_decode_win_step_dev<T>(const dec::DotArgsT<T>&, const dec::WinStepArgsT<T>&, const int*,    \
                                                     int, cudaStream_t);                                                  \
  template cudaError_t launch_decode_branch_step_dev<T>(const dec::DotArgsT<T>&, const dec::BranchStepArgsT<T>&,          \
                                                        const int*, int, cudaStream_t);
HY_DECODE_INSTANTIATE(float)
HY_DECODE_INSTANTIATE(__half)
HY_DECODE_INSTANTIATE(__nv_bfloat16)
#undef HY_DECODE_INSTANTIATE

}  // namespace hy
