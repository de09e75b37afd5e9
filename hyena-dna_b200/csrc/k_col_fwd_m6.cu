#define HY_MODE 6
#include "k_col_fwd.inc"
