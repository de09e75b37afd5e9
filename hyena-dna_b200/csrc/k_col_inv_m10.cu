#define HY_MODE 10
#include "k_col_inv.inc"
