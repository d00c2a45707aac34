// TEST-ONLY: AntMaze-v3's goal redraw of b200sim_set_goal_redraw (csrc/reset_sample.cuh rs_maze_goal_redraw), compiled for the host
// with the same flags as the host emulation, so that the CPU tests run the code the redraw kernel runs.
#include "../../gymnasium_robotics_b200/csrc/reset_sample.cuh"

// goal [2] in/out, reward out (written only when the goal changed); returns 1 when the goal changed
extern "C" int hostsim_maze_goal_redraw(const float* goal_xy, int n_goal, float scaling, float noise, float radius, int dense,
                                        unsigned long long seed, unsigned env, unsigned episode, unsigned step, const float* ach, float* goal,
                                        float* reward) {
  return rs_maze_goal_redraw(goal_xy, n_goal, scaling, noise, radius, dense, seed, env, episode, step, ach, goal, reward);
}
