#define HY_MODE 4
#include "k_col_fwd.inc"
