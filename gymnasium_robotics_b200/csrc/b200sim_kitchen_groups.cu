// The kitchen bring-up build with the two-level broad phase (bounding-volume groups, DESIGN.md section 3): same translation unit as
// b200sim_kitchen.cu compiled with -DB200_KITCHEN_GROUPS semantics; kernels fetch_kernel_groups<W, 31>, unit
// kernel_unit_kitchen_groups.
#define B200_KITCHEN_GROUPS 1
#include "b200sim_kitchen.cu"
