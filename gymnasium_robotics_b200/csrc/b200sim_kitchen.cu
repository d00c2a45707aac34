// Bring-up build of the step kernel for models with joint equalities and condim-6 contacts (Franka Kitchen, BASELINE config
// 5b): same sources as b200sim.cu compiled with -DB200_KITCHEN (two-sided dof rows, six base rows per contact, task kind 8),
// a separate translation unit so that the validated builds stay untouched.  The device model of such a model is built here
// too (the contact record is larger, so the scratch layout differs).  The candidate-pair list (3 708 pairs for the kitchen)
// is regrouped into bounding-volume groups there and scanned in two levels (sim_core.cuh `collision`, DESIGN.md 3).
// b200sim_kitchen_groups.cu includes this file with B200_KITCHEN_GROUPS defined: the same build with the two-level broad phase
// (dmodel.h / sim_core.cuh); its kernels and entry points carry the suffix _groups so that both builds live in one library and
// `b200sim_create` can pick either (B200SIM_KITCHEN_GROUPS=1; both builds are validated against each other on the GPU).
#define B200_KITCHEN 1
#if defined(B200_HULL)
#define fetch_kernel fetch_kernel_hull
#define KITCHEN_FN(name) b200sim_kitchen_hull_##name
#elif defined(B200_KITCHEN_GROUPS)
#define fetch_kernel fetch_kernel_groups
#define KITCHEN_FN(name) b200sim_kitchen_groups_##name
#else
#define KITCHEN_FN(name) b200sim_kitchen_##name
#endif
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "step_kernel.cuh"

// NVP = 31 (not 30): the instantiations must not share a symbol with the NVP = 30 kernels of b200sim.cu
#ifdef B200_KITCHEN_GROUPS
#define B200_KITCHEN_VARIANTS(X) X(7, 31) X(10, 31) X(11, 31)   // 11: fits since the pair list left shared memory; chosen only by B200SIM_WPB=11 until measured
#else
#define B200_KITCHEN_VARIANTS(X) X(7, 31) X(10, 31)
#endif

extern "C" int KITCHEN_FN(build)(const b200_model_view* view, const double* eq_data, const float* ref, int penv_body,
                                     std::vector<uint32_t>* buf, std::string* err) {
  return dm_build(*view, eq_data, ref, *buf, *err, penv_body);
}

extern "C" int KITCHEN_FN(setattr)(int wpb, int smem_bytes) {
  cudaError_t e = cudaErrorInvalidValue;
#define B200_SETATTR(W, V) if (wpb == W) e = cudaFuncSetAttribute(fetch_kernel<W, V>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
  B200_KITCHEN_VARIANTS(B200_SETATTR)
#undef B200_SETATTR
  return e == cudaSuccess ? 0 : -1;
}

extern "C" int KITCHEN_FN(launch)(int wpb, int blocks, size_t smem_bytes, void* stream, const uint32_t* model_dev, const FetchTask* task,
                                      int mode, int nraw, int N, const StepIO* io) {
  int matched = 0;
#define B200_LAUNCH(W, V)                                                                                        \
  if (wpb == W) { matched = 1; fetch_kernel<W, V><<<blocks, W * 32, smem_bytes, (cudaStream_t)stream>>>(model_dev, *task, mode, nraw, N, *io); }
  B200_KITCHEN_VARIANTS(B200_LAUNCH)
#undef B200_LAUNCH
  return matched ? 0 : -1;
}
