// Ant build of the step kernel: the AntMaze models (NVP = 14) compiled with -DB200_ANT, for the handles whose Ant keywords need more
// than the plain build's observation (b200sim_set_ant_info, maze touch_mode 2..4): contact_force_range as the clip range, the Ant-v4
// (111,) contact-force observation, and the per-step info row written from lane 0 in the same launch.  A translation unit of its own
// (kernels fetch_kernel_ant<W, 14>, unit kernel_unit_ant) so that the plain build's kernels stay instruction-identical.
#define B200_ANT 1
#define fetch_kernel fetch_kernel_ant
#include <cuda_runtime.h>
#include <stdint.h>

#include "step_kernel.cuh"

// the block sizes the plain build instantiates for NVP = 14 (b200sim_create picks among them the same way)
#define B200_ANT_VARIANTS(X) X(7, 14) X(8, 14) X(14, 14) X(16, 14) X(28, 14) X(32, 14)
B200_KERNEL_UNIT(kernel_unit_ant, B200_ANT_VARIANTS)
