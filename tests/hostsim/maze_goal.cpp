// TEST-ONLY: the maze goal update of b200sim_set_goal_update (csrc/reset_sample.cuh rs_maze_goal_update), compiled for the host with
// the same flags as the host emulation, so that the CPU tests run the code the update kernel runs.
#include "../../gymnasium_robotics_b200/csrc/reset_sample.cuh"

// goal [2] in/out; returns the number of candidates drawn (0: the goal stays)
extern "C" int hostsim_maze_goal_update(const float* goal_xy, int n_goal, float scaling, float noise, float radius, unsigned long long seed,
                                        unsigned env, unsigned episode, unsigned step, const float* ach, float* goal) {
  return rs_maze_goal_update(goal_xy, n_goal, scaling, noise, radius, seed, env, episode, step, ach, goal);
}
