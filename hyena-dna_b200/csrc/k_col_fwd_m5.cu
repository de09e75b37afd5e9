#define HY_MODE 5
#include "k_col_fwd.inc"
