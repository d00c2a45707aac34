// In-kernel reset sampling (SURVEY.md 8f row 1): the draws of the reference's reset path on the device, one counter-based
// stream per (seed, env, episode) so that resets need no host round trip and are independent of batch size and sharding.
//
//   Fetch: object start xy by rejection (envs/fetch/fetch_env.py:386-392) and goal (envs/fetch/fetch_env.py:153-166).
//
// The generator is Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11), written out here;
// it is the "throughput" RNG mode -- distribution-equal to the reference's numpy PCG64 stream, not value-equal (the
// value-equal mode stays on the host: gymnasium_robotics_b200/fetch.py `_sample_reset`, rng_mode="numpy").
// Compiles for the device (b200sim.cu) and for the host (tests/hostsim/hostsim.cpp: the CPU test backend calls the same code).
#pragma once
#include <stdint.h>
#include <math.h>

#include "../../include/b200sim.h"

#ifdef __CUDACC__
#define RS_HD __host__ __device__ inline
#else
#define RS_HD inline
#endif

RS_HD void rs_mulhilo(uint32_t a, uint32_t b, uint32_t* hi, uint32_t* lo) {
  uint64_t p = (uint64_t)a * (uint64_t)b;
  *hi = (uint32_t)(p >> 32); *lo = (uint32_t)p;
}

// counter c[4], key k[2] -> out[4]
RS_HD void rs_philox4x32_10(const uint32_t c[4], const uint32_t k[2], uint32_t out[4]) {
  uint32_t c0 = c[0], c1 = c[1], c2 = c[2], c3 = c[3], k0 = k[0], k1 = k[1];
  for (int r = 0; r < 10; r++) {
    uint32_t hi0, lo0, hi1, lo1;
    rs_mulhilo(0xD2511F53u, c0, &hi0, &lo0);
    rs_mulhilo(0xCD9E8D57u, c2, &hi1, &lo1);
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

RS_HD float rs_u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }   // [0, 1), 24 bits

// 128 candidate positions at most (the loop ends at the first accepted one, typically inside block 0 or 1): a rejected last
// one has probability (pi 0.1^2 / (2 obj_range)^2)^128 -- 1e-58 for obj_range 0.15, 3e-14 for FetchSlide's 0.1
#define RS_FETCH_OBJ_BLOCKS 64
#define RS_FETCH_GOAL_BLOCK 64

// draws of one Fetch reset: obj_xy (only when has_object) and goal
RS_HD void rs_fetch_reset_draw(const b200sim_fetch_reset_t& p, unsigned long long seed, uint32_t env, uint32_t episode, float obj_xy[2],
                               float goal[3]) {
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  uint32_t ctr[4] = {env, episode, 0u, 0x5EEDu}, r[4];
  if (p.has_object) {
    // fetch_env.py:386-392: redraw until the object is at least 0.1 from the gripper in the plane
    bool done = false;
    for (int b = 0; b < RS_FETCH_OBJ_BLOCKS && !done; b++) {
      ctr[2] = (uint32_t)b;
      rs_philox4x32_10(ctr, key, r);
      for (int h = 0; h < 2 && !done; h++) {
        float dx = (2.0f * rs_u01(r[2 * h]) - 1.0f) * p.obj_range, dy = (2.0f * rs_u01(r[2 * h + 1]) - 1.0f) * p.obj_range;
        obj_xy[0] = p.gripper_xpos[0] + dx; obj_xy[1] = p.gripper_xpos[1] + dy;
        done = sqrtf(dx * dx + dy * dy) >= 0.1f;
      }
    }
  }
  ctr[2] = RS_FETCH_GOAL_BLOCK;
  rs_philox4x32_10(ctr, key, r);
  for (int k = 0; k < 3; k++) goal[k] = p.gripper_xpos[k] + (2.0f * rs_u01(r[k]) - 1.0f) * p.target_range;   // fetch_env.py:155-157 / :164-166
  if (p.has_object) {
    for (int k = 0; k < 3; k++) goal[k] += p.target_offset[k];                                                // :158
    goal[2] = p.height_offset;                                                                                // :159
    if (p.target_in_the_air && rs_u01(r[3]) < 0.5f) {                                                         // :160-161
      ctr[2] = RS_FETCH_GOAL_BLOCK + 1;
      rs_philox4x32_10(ctr, key, r);
      goal[2] += rs_u01(r[0]) * 0.45f;
    }
  }
}

// one env's state record <- rest record + draws
RS_HD void rs_fetch_reset_record(const b200sim_fetch_reset_t& p, unsigned long long seed, uint32_t env, uint32_t episode, const float* rest,
                                 int stride, int st_qpos, int st_goal, float* rec) {
  float xy[2] = {0.f, 0.f}, goal[3];
  rs_fetch_reset_draw(p, seed, env, episode, xy, goal);
  for (int k = 0; k < stride; k++) rec[k] = rest[k];
  if (p.has_object) { rec[st_qpos + p.obj_qadr] = xy[0]; rec[st_qpos + p.obj_qadr + 1] = xy[1]; }
  for (int k = 0; k < 3; k++) rec[st_goal + k] = goal[k];
}

// Generic form for reset_model functions that are a fixed list of uniform draws written into the env's record (the Adroit envs:
// adroit_hammer.py:372-378 board height; adroit_relocate.py:354-373 ball xy + target xyz; adroit_door.py:359-371 frame xyz):
// slot k of the list <- lo[k] + (hi[k] - lo[k]) * u, u = word k % 4 of Philox block k / 4 of the (seed; env, episode) stream.
RS_HD void rs_uniform_reset_record(const b200sim_uniform_reset_t& p, unsigned long long seed, uint32_t env, uint32_t episode, const float* rest,
                                   int stride, float* rec) {
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  uint32_t ctr[4] = {env, episode, 0u, 0x0A11u}, r[4] = {0u, 0u, 0u, 0u};
  for (int k = 0; k < stride; k++) rec[k] = rest[k];
  float euler[3] = {0.f, 0.f, 0.f};
  for (int k = 0; k < p.n; k++) {
    if ((k & 3) == 0) { ctr[2] = (uint32_t)(k >> 2); rs_philox4x32_10(ctr, key, r); }
    float v = p.lo[k] + (p.hi[k] - p.lo[k]) * rs_u01(r[k & 3]);
    if (p.slot[k] >= 0) rec[p.slot[k]] = v; else euler[-1 - p.slot[k]] = v;   // slot -1 - j: Euler angle j of the orientation below
  }
  if (p.quat_slot >= 0) {
    // adroit_pen.py:379-384: body_quat <- euler2quat(angles) = qx(e0) * qy(e1) * qz(e2) (utils/rotations.py:87-113)
    float ca = cosf(0.5f * euler[0]), sa = sinf(0.5f * euler[0]), cb = cosf(0.5f * euler[1]), sb = sinf(0.5f * euler[1]);
    float cc = cosf(0.5f * euler[2]), sc = sinf(0.5f * euler[2]);
    float w = ca * cb, x = sa * cb, y = ca * sb, z = sa * sb;       // qx * qy
    float* q = rec + p.quat_slot;
    q[0] = w * cc - z * sc; q[1] = x * cc + y * sc; q[2] = y * cc - x * sc; q[3] = z * cc + w * sc;   // (* qz)
  }
}

// Maze reset (envs/maze/maze_v4.py:299-358 MazeEnv.reset with generate_target_goal :256-274, generate_reset_pos :276-297,
// add_xy_position_noise :360-373): goal = a goal cell + noise, start = a reset cell farther than `p.separation` from the goal + noise
// (0: half a cell, 0.5 * scaling; AntMaze-v3's envs/maze/maze.py:194 uses 0.5).
// `goal_xy` / `reset_xy` are the cell-centre tables ([n, 2]); an index is (word * n) >> 32 (bias < n / 2^32).
#define RS_MAZE_POS_BLOCKS 32   // 128 candidate reset cells at most
RS_HD void rs_maze_reset_draw(const b200sim_maze_reset_t& p, const float* goal_xy, const float* reset_xy, unsigned long long seed, uint32_t env,
                              uint32_t episode, float goal[2], float pos[2]) {
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  uint32_t ctr[4] = {env, episode, 0u, 0x3A2Eu}, r[4];
  const float amp = p.noise * p.scaling;
  const float sep = p.separation > 0.f ? p.separation : 0.5f * p.scaling;
  rs_philox4x32_10(ctr, key, r);
  uint32_t gi = (uint32_t)(((uint64_t)r[0] * (uint64_t)p.n_goal) >> 32);
  goal[0] = goal_xy[2 * gi] + (2.0f * rs_u01(r[1]) - 1.0f) * amp;
  goal[1] = goal_xy[2 * gi + 1] + (2.0f * rs_u01(r[2]) - 1.0f) * amp;
  bool done = false;
  pos[0] = goal[0]; pos[1] = goal[1];
  for (int b = 1; b <= RS_MAZE_POS_BLOCKS && !done; b++) {
    ctr[2] = (uint32_t)b;
    rs_philox4x32_10(ctr, key, r);
    for (int h = 0; h < 4 && !done; h++) {
      uint32_t ri = (uint32_t)(((uint64_t)r[h] * (uint64_t)p.n_reset) >> 32);
      pos[0] = reset_xy[2 * ri]; pos[1] = reset_xy[2 * ri + 1];
      float dx = pos[0] - goal[0], dy = pos[1] - goal[1];
      done = !(sqrtf(dx * dx + dy * dy) <= sep);     // maze_v4.py:289-296, maze.py:193-198
    }
  }
  ctr[2] = RS_MAZE_POS_BLOCKS + 1;
  rs_philox4x32_10(ctr, key, r);
  pos[0] += (2.0f * rs_u01(r[0]) - 1.0f) * amp;
  pos[1] += (2.0f * rs_u01(r[1]) - 1.0f) * amp;
}

// Goal update of a continuing maze task (envs/maze/maze_v4.py:400-418 update_goal, called at the end of every step when
// reset_target=True): while the achieved position `ach` lies within `radius` of the goal, the goal becomes a new goal cell + noise.
// The distance is antmaze_observe's (csrc/fetch_task.cuh), rounding for rounding, so the update fires exactly when the step's
// success column is 1.  Candidate c comes from one Philox block at counter (env, episode, step, RS_MAZE_GOAL_TAG | c << 16), step
// being the env's step counter after the step: word 0 picks the cell as in rs_maze_reset_draw, words 1 and 2 the noise.  Each
// product and sum of a candidate is rounded on its own (no FMA contraction), so a restatement in fp32 gives the same bits.
// Returns the number of candidates drawn, 0 when the goal stays.
#define RS_MAZE_GOAL_TAG 0x60A1u
// 64 candidates at most; when all are rejected the goal is the last one.  A candidate is rejected when it lands within 0.45 of `ach`:
// the noise boxes (side 0.5 x scaling) of the goal cells are disjoint, and a disc of radius 0.45 covers at most one box's worth of
// them at scaling 1 (PointMaze) and 0.16 of one box at scaling 4 (AntMaze), so with n >= 2 goal cells one candidate is rejected
// with probability <= 1/2 resp. 0.08, and all 64 with probability <= 5e-20 resp. 5e-71
#define RS_MAZE_GOAL_CANDIDATES 64
RS_HD float rs_maze_goal_distance(const float ach[2], const float goal[2]) {
  float dx = ach[0] - goal[0], dy = ach[1] - goal[1];
#ifdef __CUDA_ARCH__
  return sqrtf(fmaf(dy, dy, __fmul_rn(dx, dx)));
#else
  return sqrtf(dx * dx + dy * dy);
#endif
}
// MAX_CANDIDATES 1 is AntMaze-v3's single draw (rs_maze_goal_redraw below).
template <int MAX_CANDIDATES = RS_MAZE_GOAL_CANDIDATES>
RS_HD int rs_maze_goal_update(const float* goal_xy, int n_goal, float scaling, float noise, float radius, unsigned long long seed,
                              uint32_t env, uint32_t episode, uint32_t step, const float ach[2], float goal[2]) {
  if (!(rs_maze_goal_distance(ach, goal) <= radius)) return 0;
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  const float amp = noise * scaling;
  int c = 0;
  while (c < MAX_CANDIDATES) {
    uint32_t ctr[4] = {env, episode, step, RS_MAZE_GOAL_TAG | ((uint32_t)c << 16)}, r[4];
    rs_philox4x32_10(ctr, key, r);
    c++;
    uint32_t gi = (uint32_t)(((uint64_t)r[0] * (uint64_t)n_goal) >> 32);
    const float nx = 2.0f * rs_u01(r[1]) - 1.0f, ny = 2.0f * rs_u01(r[2]) - 1.0f;   // exact
#ifdef __CUDA_ARCH__
    goal[0] = __fadd_rn(goal_xy[2 * gi], __fmul_rn(nx, amp));
    goal[1] = __fadd_rn(goal_xy[2 * gi + 1], __fmul_rn(ny, amp));
#else
    goal[0] = goal_xy[2 * gi] + nx * amp;
    goal[1] = goal_xy[2 * gi + 1] + ny * amp;
#endif
    if (!(rs_maze_goal_distance(ach, goal) <= radius)) break;
  }
  return c;
}

// Goal redraw of a continuing AntMaze-v3 task (envs/maze/maze.py:283-302: compute_terminated draws generate_target_goal +
// add_xy_position_noise once, with no rejection, for an env within the radius of its goal).  The draw is candidate 0 of
// rs_maze_goal_update and is kept even when it lands within the radius.  ant_maze_v3.py:94-97 computes the reward after that, so
// `reward` is the step's reward against the new goal: reward_kernel's formula (b200sim.cu) on rs_maze_goal_distance, which rounds as
// reward_kernel does, so the two agree bit for bit.  Returns 1 when the goal changed (`goal` and `reward` written), 0 otherwise.
RS_HD int rs_maze_goal_redraw(const float* goal_xy, int n_goal, float scaling, float noise, float radius, int dense, unsigned long long seed,
                              uint32_t env, uint32_t episode, uint32_t step, const float ach[2], float goal[2], float* reward) {
  if (!rs_maze_goal_update<1>(goal_xy, n_goal, scaling, noise, radius, seed, env, episode, step, ach, goal)) return 0;
  const float d = rs_maze_goal_distance(ach, goal);
  *reward = dense ? expf(-d) : (d <= radius ? 1.f : 0.f);
  return 1;
}

RS_HD void rs_maze_reset_record(const b200sim_maze_reset_t& p, const float* goal_xy, const float* reset_xy, unsigned long long seed, uint32_t env,
                                uint32_t episode, const float* rest, int stride, int st_qpos, int st_goal, float* rec) {
  float goal[2], pos[2];
  rs_maze_reset_draw(p, goal_xy, reset_xy, seed, env, episode, goal, pos);
  for (int k = 0; k < stride; k++) rec[k] = rest[k];
  rec[st_qpos] = pos[0]; rec[st_qpos + 1] = pos[1];      // ant_maze_v5.py:285 / point_maze.py:380: init_qpos[:2] = reset_pos
  rec[st_goal] = goal[0]; rec[st_goal + 1] = goal[1];
}

// Shadow-Hand manipulation reset (envs/shadow_dexterous_hand/manipulate.py:154-224 _reset_sim, :226-279 _sample_goal).  The reset
// is a loop in the reference -- draw a start pose, settle 10 x n_substeps, accept when the object rests on the palm -- so it is
// two entry points: the pose draw of one attempt (record <- rest record + pose, goal kept) and, after the settle launches, the
// goal draw from the settled pose.  rot modes: 0 none, 1 "z", 2 "parallel", 3 "xyz" (also the initial rotation of "ignore").
RS_HD void rs_qmul(float* r, const float* a, const float* b) {
  float w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  float y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
RS_HD void rs_qnormalize(float* q) {
  float n = 1.0f / sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] *= n; q[1] *= n; q[2] *= n; q[3] *= n;
}
// utils/rotations.py:340-346 quat_from_angle_and_axis
RS_HD void rs_angle_axis(float* q, float angle, float ax, float ay, float az) {
  float n = 1.0f / sqrtf(ax * ax + ay * ay + az * az), s = sinf(0.5f * angle);
  q[0] = cosf(0.5f * angle); q[1] = s * ax * n; q[2] = s * ay * n; q[3] = s * az * n;
  rs_qnormalize(q);
}
// one rotation draw in the reference's order: angle ~ U(-pi, pi), then (parallel) a table index or (xyz) an axis ~ U(-1, 1)^3
RS_HD void rs_hand_rotation(int mode, const uint32_t r[4], const uint32_t r2[4], const float* parallel, float* q) {
  const float PI = 3.14159265358979323846f;
  float angle = (2.0f * rs_u01(r[0]) - 1.0f) * PI;
  if (mode == 1) rs_angle_axis(q, angle, 0.f, 0.f, 1.f);
  else if (mode == 2) {
    float z[4];
    rs_angle_axis(z, angle, 0.f, 0.f, 1.f);
    uint32_t k = (uint32_t)(((uint64_t)r[1] * 24u) >> 32);
    rs_qmul(q, z, parallel + 4 * k);                                   // manipulate.py:184-187 / :252-255
  } else rs_angle_axis(q, angle, 2.0f * rs_u01(r2[0]) - 1.0f, 2.0f * rs_u01(r2[1]) - 1.0f, 2.0f * rs_u01(r2[2]) - 1.0f);
}
RS_HD void rs_hand_pose_record(const b200sim_hand_reset_t& p, const float* parallel, unsigned long long seed, uint32_t env, uint32_t episode,
                               uint32_t attempt, const float* rest, int stride, int st_qpos, int st_goal, int ngoal, float* rec) {
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  uint32_t ctr[4] = {env, episode, 4u * attempt, 0x4A2Du}, r[4], r2[4], r3[4];
  rs_philox4x32_10(ctr, key, r);
  ctr[2] = 4u * attempt + 1u; rs_philox4x32_10(ctr, key, r2);
  ctr[2] = 4u * attempt + 2u; rs_philox4x32_10(ctr, key, r3);
  float goal[8];
  for (int k = 0; k < ngoal && k < 8; k++) goal[k] = rec[st_goal + k];
  for (int k = 0; k < stride; k++) rec[k] = rest[k];
  for (int k = 0; k < ngoal && k < 8; k++) rec[st_goal + k] = goal[k];
  float* pose = rec + st_qpos + p.obj_qadr;
  if (p.randomize_rotation && p.rot_mode != 0) {                        // manipulate.py:176-197
    float off[4], q[4];
    rs_hand_rotation(p.rot_mode, r, r2, parallel, off);
    rs_qmul(q, pose + 3, off);
    for (int k = 0; k < 4; k++) pose[3 + k] = q[k];
  }
  if (p.randomize_position) {                                            // :200-202: += normal(size=3, scale=0.005), Box-Muller
    const float TWO_PI = 6.28318530717958647692f;
    float u1 = 1.0f - rs_u01(r3[0]), u2 = rs_u01(r3[1]), u3 = 1.0f - rs_u01(r3[2]), u4 = rs_u01(r3[3]);
    float m1 = sqrtf(-2.0f * logf(u1)), m2 = sqrtf(-2.0f * logf(u3));
    pose[0] += 0.005f * m1 * cosf(TWO_PI * u2); pose[1] += 0.005f * m1 * sinf(TWO_PI * u2); pose[2] += 0.005f * m2 * cosf(TWO_PI * u4);
  }
  rs_qnormalize(pose + 3);                                               // :204
}
RS_HD void rs_hand_goal(const b200sim_hand_reset_t& p, const float* parallel, unsigned long long seed, uint32_t env, uint32_t episode,
                        int st_qpos, int st_goal, float* rec) {
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  uint32_t ctr[4] = {env, episode, 0x400u, 0x4A2Du}, r[4], r2[4], r3[4];
  rs_philox4x32_10(ctr, key, r);
  ctr[2] = 0x401u; rs_philox4x32_10(ctr, key, r2);
  ctr[2] = 0x402u; rs_philox4x32_10(ctr, key, r3);
  const float* pose = rec + st_qpos + p.obj_qadr;
  float* g = rec + st_goal;
  for (int k = 0; k < 3; k++) {
    g[k] = pose[k];
    if (p.goal_random_position) g[k] += p.pos_lo[k] + (p.pos_hi[k] - p.pos_lo[k]) * rs_u01(r3[k]);   // manipulate.py:231-241
  }
  if (p.goal_rot_mode == 0) for (int k = 0; k < 4; k++) g[3 + k] = pose[3 + k];                        // :269-270 ("ignore" / "fixed")
  else rs_hand_rotation(p.goal_rot_mode, r, r2, parallel, g + 3);                                      // :247-268
  rs_qnormalize(g + 3);                                                                                // :276
}

// HandReach goal (envs/shadow_dexterous_hand/reach.py:95-121): the thumb tip and one other finger tip (uniform choice of four)
// meet at palm + (0, -0.09, 0.05) + N(0, 0.005^2): each of the two goals sits 5 mm before the meeting point on the line from its
// initial goal; with probability 0.1 the goal is the initial finger-tip configuration.
RS_HD void rs_reach_reset_record(const b200sim_reach_reset_t& p, unsigned long long seed, uint32_t env, uint32_t episode, const float* rest,
                                 int stride, int st_goal, float* rec) {
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  uint32_t ctr[4] = {env, episode, 0u, 0x2EAC4u}, r[4], r2[4];
  rs_philox4x32_10(ctr, key, r);
  ctr[2] = 1u; rs_philox4x32_10(ctr, key, r2);
  for (int k = 0; k < stride; k++) rec[k] = rest[k];
  float* g = rec + st_goal;
  for (int k = 0; k < 15; k++) g[k] = p.initial_goal[k];
  if (rs_u01(r[1]) < 0.1f) return;                                           // reach.py:118-120
  const float TWO_PI = 6.28318530717958647692f;
  float m1 = sqrtf(-2.0f * logf(1.0f - rs_u01(r2[0]))), m2 = sqrtf(-2.0f * logf(1.0f - rs_u01(r2[2])));
  float meet[3] = {p.meeting[0] + 0.005f * m1 * cosf(TWO_PI * rs_u01(r2[1])), p.meeting[1] + 0.005f * m1 * sinf(TWO_PI * rs_u01(r2[1])),
                   p.meeting[2] + 0.005f * m2 * cosf(TWO_PI * rs_u01(r2[3]))};
  int finger = (int)(((uint64_t)r[0] * 4u) >> 32);                           // :99-101 (the thumb is entry 4 of the five tips)
  const int sel[2] = {4, finger};
  for (int j = 0; j < 2; j++) {
    float* gj = g + 3 * sel[j];
    float d[3] = {meet[0] - gj[0], meet[1] - gj[1], meet[2] - gj[2]};
    float n = 0.005f / sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    for (int k = 0; k < 3; k++) gj[k] = meet[k] - n * d[k];                  // :111-116
  }
}

// Bad-state detection and recovery at env-step granularity.  mj_step checks qpos / qvel / qacc for NaN and |x| > mjMAXVAL = 1e10
// before and after the forward pass and answers with a warning + mj_resetData ([ext] engine_forward.c mj_checkPos / mj_checkVel /
// mj_checkAcc; SURVEY.md section 5 "failure detection"); here one thread scans its env's state record after the step and, when
// a rest record is given, puts the env back to it except for the `keep` ranges (goal, per-episode model poses).
RS_HD int rs_check_record(float* rec, int stride, const float* rest, const b200sim_keep_t& keep) {
  int bad = 0;
  for (int k = 0; k < stride; k++) { float v = rec[k]; if (!(fabsf(v) <= 1e10f)) bad = 1; }   // NaN fails the comparison too
  if (bad && rest) {
    for (int k = 0; k < stride; k++) {
      bool kept = false;
      for (int r = 0; r < keep.n; r++) if (k >= keep.start[r] && k < keep.start[r] + keep.len[r]) kept = true;
      if (!kept || !(fabsf(rec[k]) <= 1e10f)) rec[k] = rest[k];
    }
  }
  return bad;
}
