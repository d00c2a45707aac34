// TEST-ONLY: the host emulation (hostsim.cpp, compiled in whole) plus the FrankaKitchen observation-noise entry points of
// rng_mode="device" (csrc/fetch_task.cuh kitchen_observe, b200sim_set_obs_noise).  Kitchen flavors only (-DB200_KITCHEN).
#include "hostsim.cpp"

#ifndef B200_KITCHEN
#error "kitchen_noise.cpp is the kitchen flavors' emulation: compile it with -DB200_KITCHEN"
#endif

// the 59 uniforms in [-1, 1) of the stream (seed; env, episode, step t), entry j = word j % 4 of block j / 4 (rs_obs_noise_block):
// what the kitchen step kernel scales and adds
extern "C" void hostsim_kitchen_noise(unsigned long long seed, unsigned env, unsigned episode, unsigned t, float* out) {
  for (int b = 0; 4 * b < 59; b++) {
    float u[4];
    rs_obs_noise_block(seed, env, episode, t, (uint32_t)b, u);
    for (int w = 0; w < 4 && 4 * b + w < 59; w++) out[4 * b + w] = u[w];
  }
}

// hostsim_env_step of a kitchen env with the observation noise of b200sim_set_obs_noise (scale NULL: noise-free): scale [nobs], the
// env's global index, episode counter and step counter after the call -- the key the step kernel builds (csrc/step_kernel.cuh)
extern "C" int hostsim_kitchen_env_step(void* p, const FetchTask* t, int mode, int nraw, const float* scale, unsigned long long seed,
                                        unsigned env, unsigned episode, unsigned step, float* st, const float* action, float* obs,
                                        float* achieved, float* desired, float* reward, float* success) {
  const ObsNoiseKey key = {scale, seed, env, episode, step};
  int it = 0;
  warp_call(((HostSim*)p)->ctx, [&](const Ctx& c) {
    fetch_env_step<HOST_NVP>(c, *t, true, mode, nraw, st, action, obs, achieved, desired, reward, success, &it, scale ? &key : nullptr);
  });
  return it;
}
