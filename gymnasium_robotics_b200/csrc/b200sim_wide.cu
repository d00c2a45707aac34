// Wide build of the step kernel: models with 33..36 dofs (Adroit hammer / relocate).  Same sources as b200sim.cu, compiled
// with 64-bit dof masks (B200_WIDE) and the bordered register Cholesky (NVP = 32 + 4); a separate translation unit so that
// the ordinary builds keep their 32-bit masks and register budgets.
#define B200_WIDE 1
#include <cuda_runtime.h>
#include <stdint.h>

#include "step_kernel.cuh"

#define B200_WIDE_VARIANTS(X) X(7, 36) X(10, 36) X(13, 36) X(14, 36)
B200_KERNEL_UNIT(kernel_unit_wide, B200_WIDE_VARIANTS)
