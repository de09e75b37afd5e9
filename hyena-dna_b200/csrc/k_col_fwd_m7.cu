#define HY_MODE 7
#include "k_col_fwd.inc"
