#define HY_MODE 7
#include "k_col_inv.inc"
