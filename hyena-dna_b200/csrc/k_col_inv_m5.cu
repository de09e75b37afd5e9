#define HY_MODE 5
#include "k_col_inv.inc"
