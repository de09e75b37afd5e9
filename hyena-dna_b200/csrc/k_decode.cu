// Launchers of the incremental-decoding kernels (decode.cuh).
#include "launch.h"
#include "decode.cuh"

namespace hy {

cudaError_t launch_decode_hist(const dec::HistArgs& a, cudaStream_t s) {
  const int per_row = (a.P + 255) / 256;
  dim3 grid(per_row < 64 ? per_row : 64, a.B * a.D);
  prof_begin(K_DECODE_HIST, s);
  dec::decode_hist_kernel<<<grid, 256, 0, s>>>(a);
  prof_end(K_DECODE_HIST, s);
  return cudaGetLastError();
}

template <int BG>
static cudaError_t dot_bg(const dec::DotArgs& a, int R, dim3 grid, cudaStream_t s) {
  const int threads = 32 * dec::kDotWarps;
  switch (R) {
    case 0: dec::decode_dot_kernel<BG, 0><<<grid, threads, 0, s>>>(a); break;
    case 1: dec::decode_dot_kernel<BG, 1><<<grid, threads, 0, s>>>(a); break;
    case 2: dec::decode_dot_kernel<BG, 2><<<grid, threads, 0, s>>>(a); break;
    default: dec::decode_dot_kernel<BG, 3><<<grid, threads, 0, s>>>(a); break;
  }
  return cudaGetLastError();
}

// the split dot product over dot.t positions in nchunk chunks
static cudaError_t launch_dot(const dec::DotArgs& dot, int nchunk, int kind, cudaStream_t s) {
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
cudaError_t launch_decode_step(const dec::DotArgs& dot, const dec::StepArgs& st, cudaStream_t s) {
  if (st.nchunk > 0) {
    cudaError_t e = launch_dot(dot, st.nchunk, K_DECODE_STEP, s);
    if (e != cudaSuccess) return e;
  }
  const int rows = st.B * st.D;
  prof_begin(K_DECODE_STEP, s);
  dec::decode_step_kernel<<<(rows + dec::kStepWarps - 1) / dec::kStepWarps, 32 * dec::kStepWarps, 0, s>>>(st);
  prof_end(K_DECODE_STEP, s);
  return cudaGetLastError();
}

// one recurrence of a windowed step: the dot product over the window positions [b, t) (skipped at t = b), then the
// windowed combine kernel
cudaError_t launch_decode_win_step(const dec::DotArgs& dot, const dec::WinStepArgs& w, cudaStream_t s) {
  if (w.st.nchunk > 0) {
    cudaError_t e = launch_dot(dot, w.st.nchunk, K_DECODE_WIN_STEP, s);
    if (e != cudaSuccess) return e;
  }
  const int rows = w.st.B * w.st.D;
  prof_begin(K_DECODE_WIN_STEP, s);
  dec::decode_win_step_kernel<<<(rows + dec::kStepWarps - 1) / dec::kStepWarps, 32 * dec::kStepWarps, 0, s>>>(w);
  prof_end(K_DECODE_WIN_STEP, s);
  return cudaGetLastError();
}

// one recurrence of a branch step: the dot product over the branch's positions [b, t) (skipped at t = b), then the branch
// combine kernel; counted as a windowed step (a window whose F is selected per row)
cudaError_t launch_decode_branch_step(const dec::DotArgs& dot, const dec::BranchStepArgs& w, cudaStream_t s) {
  if (w.st.nchunk > 0) {
    cudaError_t e = launch_dot(dot, w.st.nchunk, K_DECODE_WIN_STEP, s);
    if (e != cudaSuccess) return e;
  }
  const int rows = w.st.B * w.st.D;
  prof_begin(K_DECODE_WIN_STEP, s);
  dec::decode_branch_step_kernel<<<(rows + dec::kStepWarps - 1) / dec::kStepWarps, 32 * dec::kStepWarps, 0, s>>>(w);
  prof_end(K_DECODE_WIN_STEP, s);
  return cudaGetLastError();
}

// ---- device-position steps: fixed grids, the position read by the kernels (decode.cuh *_dev_kernel)
static cudaError_t launch_dot_dev(const dec::DotArgs& dot, const dec::DevPos& p, int nchunk, int kind, cudaStream_t s) {
  const int BG = dot.B <= 1 ? 1 : dot.B <= 2 ? 2 : dot.B <= 4 ? 4 : 8;
  const int threads = 32 * dec::kDotWarps;
  dim3 grid(nchunk, (dot.D + dec::kDotWarps - 1) / dec::kDotWarps, (dot.B + BG - 1) / BG);
  prof_begin(kind, s);
  switch (BG) {
    case 1: dec::decode_dot_dev_kernel<1><<<grid, threads, 0, s>>>(dot, p); break;
    case 2: dec::decode_dot_dev_kernel<2><<<grid, threads, 0, s>>>(dot, p); break;
    case 4: dec::decode_dot_dev_kernel<4><<<grid, threads, 0, s>>>(dot, p); break;
    default: dec::decode_dot_dev_kernel<8><<<grid, threads, 0, s>>>(dot, p); break;
  }
  prof_end(kind, s);
  return cudaGetLastError();
}

static dim3 step_grid(int B, int D) { return dim3((B * D + dec::kStepWarps - 1) / dec::kStepWarps); }

cudaError_t launch_decode_step_dev(const dec::DotArgs& dot, const dec::StepArgs& st, const int* pos, int nchunk,
                                   cudaStream_t s) {
  cudaError_t e = launch_dot_dev(dot, dec::DevPos{pos, dec::kPosPlain}, nchunk, K_DECODE_STEP, s);
  if (e != cudaSuccess) return e;
  prof_begin(K_DECODE_STEP, s);
  dec::decode_step_dev_kernel<<<step_grid(st.B, st.D), 32 * dec::kStepWarps, 0, s>>>(st, pos);
  prof_end(K_DECODE_STEP, s);
  return cudaGetLastError();
}

cudaError_t launch_decode_win_step_dev(const dec::DotArgs& dot, const dec::WinStepArgs& w, const int* pos, int nchunk,
                                       cudaStream_t s) {
  cudaError_t e = launch_dot_dev(dot, dec::DevPos{pos, dec::kPosWindow}, nchunk, K_DECODE_WIN_STEP, s);
  if (e != cudaSuccess) return e;
  prof_begin(K_DECODE_WIN_STEP, s);
  dec::decode_win_step_dev_kernel<<<step_grid(w.st.B, w.st.D), 32 * dec::kStepWarps, 0, s>>>(w, pos);
  prof_end(K_DECODE_WIN_STEP, s);
  return cudaGetLastError();
}

cudaError_t launch_decode_branch_step_dev(const dec::DotArgs& dot, const dec::BranchStepArgs& w, const int* pos, int nchunk,
                                          cudaStream_t s) {
  cudaError_t e = launch_dot_dev(dot, dec::DevPos{pos, dec::kPosBranch}, nchunk, K_DECODE_WIN_STEP, s);
  if (e != cudaSuccess) return e;
  prof_begin(K_DECODE_WIN_STEP, s);
  dec::decode_branch_step_dev_kernel<<<step_grid(w.st.B, w.st.D), 32 * dec::kStepWarps, 0, s>>>(w, pos);
  prof_end(K_DECODE_WIN_STEP, s);
  return cudaGetLastError();
}

// counted by launch_count but under no kind: it is not a step kernel
cudaError_t launch_decode_pos_advance(int* pos, cudaStream_t s) {
  dec::decode_pos_advance_kernel<<<1, 1, 0, s>>>(pos);
  count_launch();
  return cudaGetLastError();
}

}  // namespace hy
