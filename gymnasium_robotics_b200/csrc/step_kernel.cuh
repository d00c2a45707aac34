// The step kernel: one warp integrates one env for a whole env-step (all sub-steps on chip); WPB warps share one copy of
// the model constants that a single thread stages into shared memory with a TMA bulk copy (cp.async.bulk + mbarrier).
// Included by each kernel build (translation unit): b200sim.cu (32-bit dof masks, NVP <= 30), b200sim_wide.cu (B200_WIDE: 64-bit
// dof masks, NVP = 36), the three b200sim_kitchen*.cu and b200sim_ant.cu (B200_ANT); each one names its instantiations once, in B200_KERNEL_UNIT.
#pragma once
#include <cuda_runtime.h>
#include "fetch_task.cuh"

#ifdef B200_STAGE_TIMING
static __device__ unsigned long long g_stage_cycles[TM_COUNT];
#endif

static __device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Everything one launch reads and writes per env.  Output rows are addressed with explicit strides, so the same kernel serves
// the five separate [N, dim] arrays of the classic entry points and the packed [N, W] rows of b200sim_set_packed (one row per env:
// obs | achieved | desired | reward | success | terminated | truncated, SURVEY.md 8e).  TimeLimit lives here too: `elapsed` is
// the library-owned per-env step counter, incremented by a MODE_STEP launch; truncated = elapsed >= max_steps
// (gymnasium TimeLimit), terminated = success for the tasks that end an episode on success (maze_v4.py:390-398 with
// continuing_task = False), else False (robot_env.py:106-112).
struct StepIO {
  float* state; const float* actions; const unsigned char* mask;
  float *obs, *achieved, *desired, *reward, *success;
  int obs_stride, goal_stride, scalar_stride;
  float *term_f, *trunc_f;                 // fp32 copies of the flags inside a packed row (NULL = none), scalar_stride apart
  unsigned char *terminated, *truncated;   // [N] byte flags (NULL = none)
  int* elapsed; int max_steps, term_on_success;
  int* info;
  unsigned long long* overflow_count;      // device counter of env-steps that ran into a capacity limit (NULL = none)
};

// The observation noise of a handle (b200sim_set_obs_noise): one scale per observation entry (NULL = no noise), the per-env
// episode counters, the key and the global index of env 0.  A kernel parameter of the kitchen builds only: the other builds' kernels
// take exactly the parameters they took before it existed.
struct ObsNoiseArgs {
  const float* scale; const int* episode; unsigned long long seed; int env_offset;
};
#ifdef B200_KITCHEN
#define B200_KITCHEN_PARAM , ObsNoiseArgs noise_args
#define B200_KITCHEN_ARG , noise_args
#elif defined(B200_ANT)
#define B200_KITCHEN_PARAM , AntInfoArgs ant_args
#define B200_KITCHEN_ARG , ant_args
#else
#define B200_KITCHEN_PARAM
#define B200_KITCHEN_ARG
#endif

template <int WPB, int NVP>
__global__ void __launch_bounds__(WPB * 32) fetch_kernel(const uint32_t* __restrict__ model_g, FetchTask task, int mode, int nraw,
                                                         int N, StepIO io B200_KITCHEN_PARAM) {
  extern __shared__ __align__(128) uint32_t smem[];
  __shared__ __align__(8) unsigned long long bar;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // ---- stage the model constants: TMA 1-D bulk copy global -> shared, completion on an mbarrier
  const int model_words = ((const DMHead*)model_g)->hot_words;  // header + HOT arrays (uniform scalar load)
  const uint32_t bytes = (uint32_t)model_words * 4u;
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem)),
                 "l"(model_g), "r"(bytes), "r"(smem_u32(&bar))
                 : "memory");
  }
  {
    uint32_t done = 0;
    while (!done) {
      asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n selp.u32 %0, 1, 0, p;\n}"
                   : "=r"(done)
                   : "r"(smem_u32(&bar))
                   : "memory");
    }
  }
  const DMHead* h = (const DMHead*)smem;
  const int env = blockIdx.x * WPB + warp;
  const bool active = env < N && !(io.mask && !io.mask[env]);  // warp-uniform
  Ctx c;
#ifdef B200_STAGE_TIMING
  long long tim[TM_COUNT];
  for (int k = 0; k < TM_COUNT; k++) tim[k] = 0;
  c.tim = tim;
  const long long t_begin = clock64();
#endif
  c.mg = model_g; c.mw = smem; c.h = h; c.lane = lane;
  c.s = (float*)(smem + model_words) + (size_t)warp * h->scr_words;
  const size_t e = active ? (size_t)env : 0;
  const float* act = io.actions ? io.actions + e * task.nact : nullptr;  // only dereferenced in MODE_STEP by active warps
  float* success = io.success + e * io.scalar_stride;
  int iters = 0;
#ifdef B200_KITCHEN
  // the noise of the observation this launch returns: the episode that observation belongs to and the step count after the launch
  // (a step increments `elapsed` below; a refresh -- after a reset, after set_state -- leaves it)
  const bool noisy = active && noise_args.scale;
  const ObsNoiseKey noise_key = {noise_args.scale, noise_args.seed, (uint32_t)(noise_args.env_offset + env), noisy ? (uint32_t)noise_args.episode[e] : 0u,
                                 noisy ? (uint32_t)(io.elapsed[e] + (mode == MODE_STEP ? 1 : 0)) : 0u};
  fetch_env_step<NVP, (WPB >= 28)>(c, task, active, mode, nraw, io.state + e * task.st_stride, act, io.obs + e * io.obs_stride, io.achieved + e * io.goal_stride,
                      io.desired + e * io.goal_stride, io.reward + e * io.scalar_stride, success, &iters, noisy ? &noise_key : nullptr);
#elif defined(B200_ANT)
  AntForces antf = {ant_args.cf_lo, ant_args.cf_hi, 0.f};
  fetch_env_step<NVP, (WPB >= 28)>(c, task, active, mode, nraw, io.state + e * task.st_stride, act, io.obs + e * io.obs_stride, io.achieved + e * io.goal_stride,
                      io.desired + e * io.goal_stride, io.reward + e * io.scalar_stride, success, &iters, &antf);
  if (active && lane == 0)
    ant_info(c, task, ant_args, mode, mode == MODE_STEP ? task.n_substeps > 0 : (mode == MODE_RAW && nraw > 0), io.state + e * task.st_stride, act,
             antf.sq, e);
#else
  // (WPB >= 28: at most 72 registers per thread, the driver rebuilds its context before each stage call -- stage_ctx)
  fetch_env_step<NVP, (WPB >= 28)>(c, task, active, mode, nraw, io.state + e * task.st_stride, act, io.obs + e * io.obs_stride, io.achieved + e * io.goal_stride,
                      io.desired + e * io.goal_stride, io.reward + e * io.scalar_stride, success, &iters);
#endif
  if (active && lane == 0) {
    // episode bookkeeping of the env-step (TimeLimit wrapper + compute_terminated), flags in both output forms; refresh / raw
    // launches leave the flags of the rows they rewrite alone (a same-step autoreset keeps the flags of the finished episode)
    if (mode == MODE_STEP) {
      bool term = io.term_on_success && *success != 0.f, trunc = false;
      if (io.elapsed) { int el = io.elapsed[e] + 1; io.elapsed[e] = el; trunc = io.max_steps > 0 && el >= io.max_steps; }
      if (io.terminated) io.terminated[e] = term ? 1 : 0;
      if (io.truncated) io.truncated[e] = trunc ? 1 : 0;
      if (io.term_f) io.term_f[e * io.scalar_stride] = term ? 1.f : 0.f;
      if (io.trunc_f) io.trunc_f[e * io.scalar_stride] = trunc ? 1.f : 0.f;
    }
    if (io.info) io.info[e] = iters;
    if (io.overflow_count && (iters >> 16)) atomicAdd(io.overflow_count, 1ull);
  }
#ifdef B200_STAGE_TIMING
  if (lane == 0 && active) {
    long long sum = 0;
    for (int k = 0; k < TM_OTHER; k++) sum += tim[k];
    tim[TM_OTHER] = clock64() - t_begin - sum;
    for (int k = 0; k < TM_COUNT; k++) atomicAdd(&g_stage_cycles[k], (unsigned long long)tim[k]);
  }
#endif
}

// One kernel build: its model builder (the scratch layout depends on the unit's defines) and its fetch_kernel<WPB, NVP>
// instantiations.  b200sim_create picks the unit of a model once and keeps it on the handle.
struct KernelUnit {
  int (*build)(const b200_model_view& view, const double* eq_data, const float* ref, int penv_body, std::vector<uint32_t>& buf,
               std::string& err);
  bool (*has)(int wpb, int nvp);                                // an instantiation <wpb, nvp> exists
  cudaError_t (*setattr)(int wpb, int nvp, int smem_bytes);     // cudaErrorInvalidValue when it does not
  bool (*launch)(int wpb, int nvp, int blocks, size_t smem_bytes, cudaStream_t stream, const uint32_t* model_dev, const FetchTask& task,
                 int mode, int nraw, int N, const StepIO& io, const ObsNoiseArgs& noise_args, const AntInfoArgs& ant_args);
};   // launch: false (nothing launched) when it does not; noise_args reach the kitchen units' kernels only, ant_args the ant unit's

#define B200_UNIT_HAS(W, V) || (wpb == W && nvp == V)
#define B200_UNIT_SETATTR(W, V) \
  if (wpb == W && nvp == V) return cudaFuncSetAttribute(fetch_kernel<W, V>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
#define B200_UNIT_LAUNCH(W, V)                                                                           \
  if (wpb == W && nvp == V) {                                                                            \
    fetch_kernel<W, V><<<blocks, W * 32, smem_bytes, stream>>>(model_dev, task, mode, nraw, N, io B200_KITCHEN_ARG); \
    return true;                                                                                         \
  }

// Defines `const KernelUnit NAME` from the unit's instantiation list VARIANTS(X): one X(WPB, NVP) per kernel.
#define B200_KERNEL_UNIT(NAME, VARIANTS)                                                                                              \
  static int unit_build(const b200_model_view& view, const double* eq_data, const float* ref, int penv_body, std::vector<uint32_t>& buf, \
                        std::string& err) {                                                                                          \
    return dm_build(view, eq_data, ref, buf, err, penv_body);                                                                       \
  }                                                                                                                                  \
  static bool unit_has(int wpb, int nvp) { return false VARIANTS(B200_UNIT_HAS); }                                                   \
  static cudaError_t unit_setattr(int wpb, int nvp, int smem_bytes) {                                                                \
    VARIANTS(B200_UNIT_SETATTR)                                                                                                      \
    return cudaErrorInvalidValue;                                                                                                    \
  }                                                                                                                                  \
  static bool unit_launch(int wpb, int nvp, int blocks, size_t smem_bytes, cudaStream_t stream, const uint32_t* model_dev,           \
                          const FetchTask& task, int mode, int nraw, int N, const StepIO& io, const ObsNoiseArgs& noise_args,        \
                          const AntInfoArgs& ant_args) {                                                                             \
    VARIANTS(B200_UNIT_LAUNCH)                                                                                                       \
    return false;                                                                                                                    \
  }                                                                                                                                  \
  extern const KernelUnit NAME = {unit_build, unit_has, unit_setattr, unit_launch};
