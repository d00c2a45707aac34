// Bring-up build of the step kernel for models with joint equalities and condim-6 contacts (Franka Kitchen, BASELINE config
// 5b): same sources as b200sim.cu compiled with -DB200_KITCHEN (two-sided dof rows, six base rows per contact, task kind 8),
// a separate translation unit so that the validated builds stay untouched.  The device model of such a model is built here
// too (the contact record is larger, so the scratch layout differs).  The candidate-pair list (3 708 pairs for the kitchen)
// is regrouped into bounding-volume groups there and scanned in two levels (sim_core.cuh `collision`, DESIGN.md 3).
// b200sim_kitchen_groups.cu includes this file with B200_KITCHEN_GROUPS defined: the same build with the two-level broad phase
// (dmodel.h / sim_core.cuh); its kernels and unit carry the suffix _groups so that both builds live in one library and
// `b200sim_create` can pick either (B200SIM_KITCHEN_GROUPS=1; both builds are validated against each other on the GPU).
#define B200_KITCHEN 1
#if defined(B200_HULL)
#define fetch_kernel fetch_kernel_hull
#define KITCHEN_UNIT kernel_unit_kitchen_hull
#elif defined(B200_KITCHEN_GROUPS)
#define fetch_kernel fetch_kernel_groups
#define KITCHEN_UNIT kernel_unit_kitchen_groups
#else
#define KITCHEN_UNIT kernel_unit_kitchen
#endif
#include <cuda_runtime.h>
#include <stdint.h>

#include "step_kernel.cuh"

// NVP = 31 (not 30): the instantiations must not share a symbol with the NVP = 30 kernels of b200sim.cu
#ifdef B200_KITCHEN_GROUPS
#define B200_KITCHEN_VARIANTS(X) X(7, 31) X(10, 31) X(11, 31)   // 11: fits since the pair list left shared memory
#else
#define B200_KITCHEN_VARIANTS(X) X(7, 31) X(10, 31)
#endif

B200_KERNEL_UNIT(KITCHEN_UNIT, B200_KITCHEN_VARIANTS)
