#define HY_MODE 9
#include "k_col_inv.inc"
