// TEST-ONLY: the host emulation (hostsim.cpp, compiled in whole) as the ant kernel build (-DB200_ANT, csrc/b200sim_ant.cu) plus the
// entry point of b200sim_set_ant_info: one env's launch with the Ant's keywords, and its info row.
#include "hostsim.cpp"

#ifndef B200_ANT
#error "ant_info.cpp is the ant build's emulation: compile it with -DB200_ANT"
#endif

// hostsim_env_step of an ant-build env, followed by what fetch_kernel_ant's lane 0 does after it (ant_info): `a` as
// b200sim_set_ant_info leaves it, with rows / origin pointing at this env's row [9] / reset position [2] (or NULL)
extern "C" int hostsim_ant_env_step(void* p, const FetchTask* t, int mode, int nraw, const AntInfoArgs* a, float* st, const float* action,
                                    float* obs, float* achieved, float* desired, float* reward, float* success) {
  int it = 0;
  warp_call(((HostSim*)p)->ctx, [&](const Ctx& c) {
    AntForces f = {a->cf_lo, a->cf_hi, 0.f};
    fetch_env_step<HOST_NVP>(c, *t, true, mode, nraw, st, action, obs, achieved, desired, reward, success, &it, &f);
    if (c.lane == 0)
      ant_info(c, *t, *a, mode, mode == MODE_STEP ? t->n_substeps > 0 : (mode == MODE_RAW && nraw > 0), st, action, f.sq, 0);
  });
  return it;
}
