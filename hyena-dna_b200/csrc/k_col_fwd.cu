// Pass-1 dispatch over the input mode; the kernels live in k_col_fwd_m*.cu (one translation unit per mode).
#include "launch.h"
namespace hy {
cudaError_t launch_col_fwd(int mode, const PassArgs& a, int rows, cudaStream_t s) {
  switch (mode) {
    case COL_FILTER: return launch_col_fwd_mode<COL_FILTER>(a, rows, s);
    case COL_GATE: return launch_col_fwd_mode<COL_GATE>(a, rows, s);
    case COL_DC: return launch_col_fwd_mode<COL_DC>(a, rows, s);
    case COL_PLAIN: return launch_col_fwd_mode<COL_PLAIN>(a, rows, s);
    case COL_GATE_ROWS: return launch_col_fwd_mode<COL_GATE_ROWS>(a, rows, s);
    case COL_DC_ROWS: return launch_col_fwd_mode<COL_DC_ROWS>(a, rows, s);
    case COL_GATE_PACKED: return launch_col_fwd_mode<COL_GATE_PACKED>(a, rows, s);
    case COL_DC_PACKED: return launch_col_fwd_mode<COL_DC_PACKED>(a, rows, s);
    case COL_PLAIN_WIN: return launch_col_fwd_mode<COL_PLAIN_WIN>(a, rows, s);
  }
  return cudaErrorInvalidValue;
}
}  // namespace hy
