#define HY_MODE 8
#include "k_col_fwd.inc"
