// Pass-3 dispatch over the output mode; the kernels live in k_col_inv_m*.cu (one translation unit per mode).
#include "launch.h"
namespace hy {
cudaError_t launch_col_inv(int mode, const PassArgs& a, int rows, cudaStream_t s) {
  switch (mode) {
    case INV_CONV_FWD: return launch_col_inv_mode<INV_CONV_FWD>(a, rows, s);
    case INV_BWD_DG: return launch_col_inv_mode<INV_BWD_DG>(a, rows, s);
    case INV_DK: return launch_col_inv_mode<INV_DK>(a, rows, s);
    case INV_PLAIN_FWD: return launch_col_inv_mode<INV_PLAIN_FWD>(a, rows, s);
    case INV_PLAIN_BWD: return launch_col_inv_mode<INV_PLAIN_BWD>(a, rows, s);
    case INV_CONV_FWD_ROWS: return launch_col_inv_mode<INV_CONV_FWD_ROWS>(a, rows, s);
    case INV_BWD_DG_ROWS: return launch_col_inv_mode<INV_BWD_DG_ROWS>(a, rows, s);
    case INV_CONV_FWD_PACKED: return launch_col_inv_mode<INV_CONV_FWD_PACKED>(a, rows, s);
    case INV_BWD_DG_PACKED: return launch_col_inv_mode<INV_BWD_DG_PACKED>(a, rows, s);
    case INV_CONV_FWD_WIN: return launch_col_inv_mode<INV_CONV_FWD_WIN>(a, rows, s);
    case INV_PLAIN_FWD_WIN: return launch_col_inv_mode<INV_PLAIN_FWD_WIN>(a, rows, s);
  }
  return cudaErrorInvalidValue;
}
}  // namespace hy
