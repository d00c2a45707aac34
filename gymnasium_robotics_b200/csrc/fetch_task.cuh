// Fetch task layer executed inside the step kernel: action application, sub-step loop, observation, reward.
// Restates (batched, fp32) the per-step Python of the reference:
//   BaseRobotEnv.step                 gymnasium_robotics/envs/robot_env.py:114-152
//   MujocoFetchEnv._set_action        envs/fetch/fetch_env.py:85-105, 305-310 ; utils/mujoco_utils.py:34-71, 83-107
//   MujocoFetchEnv._step_callback     envs/fetch/fetch_env.py:295-303
//   generate_mujoco_observations      envs/fetch/fetch_env.py:312-360 ; rotations.mat2euler utils/rotations.py:162-184
//   compute_reward / _is_success      envs/fetch/fetch_env.py:74-80, 168-170
#pragma once
#include "sim_core.cuh"

#define FETCH_MAX_ROBOT_JNT 16

struct FetchTask {
  int has_object, block_gripper, n_substeps, reward_dense;
  int grip_site, obj_site, frame_site;  // "robot0:grip", "object0", body frame of robot0:gripper_link
  int nrobot;
  int robot_qadr[FETCH_MAX_ROBOT_JNT], robot_dadr[FETCH_MAX_ROBOT_JNT];
  int finger_qadr[2];
  int nobs;
  float distance_threshold, dt;
  // task family (TASK_FETCH / TASK_ANTMAZE), action and goal widths, maze success radius
  int kind, nact, ngoal;
  float success_radius;
  int obs_qpos_start;   // maze tasks: first qpos entry that is part of `observation` (Ant 2, Point 0)
  float vel_clip;       // maze tasks: |qvel| clip applied before stepping (Point 5.0, 0 = none)
  // hand manipulation tasks: object free joint addresses, which goal parts count, rotation threshold
  int obj_qadr, obj_dadr, goal_flags;
  float rotation_threshold;
  int touch_mode;       // 0 = no touch observation, 1 = sensordata, 2 = boolean, 3 = log(x + 1)
  int tip_site[5];      // HandReach: fingertip sites "robot0:S_{ff,mf,rf,lf,th}tip"; Adroit hammer: [0] = "tool", [1] = "nail_goal"
  int penv_body;        // runtime body with a per-env body_pos (-1 = none)
  // state record layout (floats, per env): qpos | qvel | warm | ctrl | mocap(7) | pose(7) | goal(ngoal) | penv body pose(3 + 4)
  int st_qpos, st_qvel, st_warm, st_ctrl, st_mocap, st_pose, st_goal, st_stride, st_penv;
};
// TASK_ANTMAZE covers both maze agents (Ant, Point)
enum { TASK_FETCH = 0, TASK_ANTMAZE = 1, TASK_HAND = 2, TASK_HAND_REACH = 3, TASK_ADROIT_HAMMER = 4, TASK_ADROIT_RELOCATE = 5,
       TASK_ADROIT_PEN = 6, TASK_ADROIT_DOOR = 7, TASK_KITCHEN = 8 };
#define TASK_IS_ADROIT(k) ((k) >= TASK_ADROIT_HAMMER && (k) <= TASK_ADROIT_DOOR)
enum { GOAL_USE_POS = 1, GOAL_USE_ROT = 2, GOAL_IGNORE_Z = 4 };

enum { MODE_STEP = 0, MODE_REFRESH = 1, MODE_RAW = 2 };

HD void site_pose(const Ctx& c, int site, float* pos, float* quat) {
  int b = MI(site_body)[site];
  float t[3];
  qrot(t, SF(xquat) + 4 * b, MF(site_pos) + 3 * site);
  for (int k = 0; k < 3; k++) pos[k] = SF(xpos)[3 * b + k] + t[k];
  if (quat) qmul(quat, SF(xquat) + 4 * b, MF(site_quat) + 4 * site);
}

HD void load_state(const Ctx& c, const FetchTask& t, const float* st) {
  const DMHead* h = c.h;
  LANES(i, h->nq) SF(qpos)[i] = st[t.st_qpos + i];
  LANES(i, h->nv) { SF(qvel)[i] = st[t.st_qvel + i]; SF(qacc)[i] = st[t.st_warm + i]; }  // qacc doubles as the warm start
  LANES(i, h->nu) SF(ctrl)[i] = st[t.st_ctrl + i];
  LANES(i, 3 * h->nmocap) SF(mocap_pos)[i] = st[t.st_mocap + i];
  LANES(i, 4 * h->nmocap) SF(mocap_quat)[i] = st[t.st_mocap + 3 + i];
  if (h->penv_body > 0) LANES(i, 7) SF(penv_pos)[i] = st[t.st_penv + i];
  if (c.lane == 0) { SI(counters)[CNT_ITERS] = 0; SI(counters)[CNT_OVERFLOW] = 0; }
  SYNC();
}

HD void store_state(const Ctx& c, const FetchTask& t, float* st) {
  const DMHead* h = c.h;
  LANES(i, h->nq) st[t.st_qpos + i] = SF(qpos)[i];
  LANES(i, h->nv) { st[t.st_qvel + i] = SF(qvel)[i]; st[t.st_warm + i] = SF(qacc)[i]; }
  LANES(i, h->nu) st[t.st_ctrl + i] = SF(ctrl)[i];
  LANES(i, 3 * h->nmocap) st[t.st_mocap + i] = SF(mocap_pos)[i];
  LANES(i, 4 * h->nmocap) st[t.st_mocap + 3 + i] = SF(mocap_quat)[i];
  if (c.lane == 0 && t.kind == TASK_FETCH) {
    float p[3], q[4];
    site_pose(c, t.frame_site, p, q);  // data.xpos / data.xquat of the welded body as of the last forward pass
    for (int k = 0; k < 3; k++) st[t.st_pose + k] = p[k];
    for (int k = 0; k < 4; k++) st[t.st_pose + 3 + k] = q[k];
  }
}

HD void site_vel(const Ctx& c, int site, const float* pos, float* velp, float* velr) {
  const float* V = SF(cvel) + 6 * MI(site_body)[site];
  float r[3] = {pos[0] - c.h->ref[0], pos[1] - c.h->ref[1], pos[2] - c.h->ref[2]}, t[3];
  cross3(t, V, r);
  velp[0] = V[3] + t[0]; velp[1] = V[4] + t[1]; velp[2] = V[5] + t[2];
  if (velr) { velr[0] = V[0]; velr[1] = V[1]; velr[2] = V[2]; }
}

// squared-distance accumulation with ONE rounding sequence on the device (round-to-nearest fused multiply-add per term), the same in the
// step kernel and in reward_kernel: `reward == compute_reward(achieved_goal, desired_goal)` bit for bit
#ifdef __CUDA_ARCH__
#define B200_SQACC(d2, e) d2 = fmaf((e), (e), d2)
#else
#define B200_SQACC(d2, e) d2 += (e) * (e)
#endif
HD void fetch_observe(const Ctx& c, const FetchTask& t, const float* goal, float* obs, float* achieved, float* desired,
                      float* reward, float* success) {
  pass_V(c, SF(qvel), SF(cvel));  // site velocities: Jacobian of the last forward pass times the current qvel
  if (c.lane == 0) {
    // (written straight to the observation row: a local staging array indexed by a running count would be local memory)
    float grip[3], gvel[3];
    float* o = obs;
    int n = 0;
    site_pose(c, t.grip_site, grip, nullptr);
    site_vel(c, t.grip_site, grip, gvel, nullptr);
    for (int k = 0; k < 3; k++) gvel[k] *= t.dt;
    for (int k = 0; k < 3; k++) o[n++] = grip[k];
    float ag[3] = {grip[0], grip[1], grip[2]};
    const float* gs_q = SF(qpos);
    const float* gs_v = SF(qvel);
    float gstate[2] = {gs_q[t.robot_qadr[t.nrobot - 2]], gs_q[t.robot_qadr[t.nrobot - 1]]};
    float gv[2] = {gs_v[t.robot_dadr[t.nrobot - 2]] * t.dt, gs_v[t.robot_dadr[t.nrobot - 1]] * t.dt};
    if (t.has_object) {
      float op[3], oq[4], m[9], vp[3], vr[3];
      site_pose(c, t.obj_site, op, oq);
      q2mat(m, oq);
      site_vel(c, t.obj_site, op, vp, vr);
      for (int k = 0; k < 3; k++) o[n++] = op[k];
      for (int k = 0; k < 3; k++) o[n++] = op[k] - grip[k];
      o[n++] = gstate[0]; o[n++] = gstate[1];
      // mat2euler
      float cy = sqrtf(m[8] * m[8] + m[5] * m[5]);
      float ex, ey, ez;
      if (cy > 8.8817841970012523e-16f) { ez = -atan2f(m[1], m[0]); ey = -atan2f(-m[2], cy); ex = -atan2f(m[5], m[8]); }
      else { ez = -atan2f(-m[3], m[4]); ey = -atan2f(-m[2], cy); ex = 0.f; }
      o[n++] = ex; o[n++] = ey; o[n++] = ez;
      for (int k = 0; k < 3; k++) o[n++] = vp[k] * t.dt - gvel[k];
      for (int k = 0; k < 3; k++) o[n++] = vr[k] * t.dt;
      for (int k = 0; k < 3; k++) ag[k] = op[k];
    } else { o[n++] = gstate[0]; o[n++] = gstate[1]; }
    for (int k = 0; k < 3; k++) o[n++] = gvel[k];
    o[n++] = gv[0]; o[n++] = gv[1];
    float d2 = 0;
    for (int k = 0; k < 3; k++) { achieved[k] = ag[k]; desired[k] = goal[k]; float e = ag[k] - goal[k]; B200_SQACC(d2, e); }
    float d = sqrtf(d2);
    *reward = t.reward_dense ? -d : -(d > t.distance_threshold ? 1.f : 0.f);
    *success = d < t.distance_threshold ? 1.f : 0.f;
  }
}

#ifdef B200_ANT
// The ant build's contact forces (b200sim_set_ant_info): the clip range contact_force_range in, the warp's sum of the squares of the
// clipped forces of every body out (the contact cost's; the world row is zero)
struct AntForces { float lo, hi, sq; };
#endif
// AntMaze: obs = ant qpos[2:] | qvel [| clipped contact forces], achieved = qpos[:2]; reward exp(-d) (dense) or d <= r (sparse)
// (reference: envs/maze/ant_maze_v5.py:295-320, envs/maze/maze_v4.py:381-398).
// touch_mode == 1 (AntMaze-v5 on Gymnasium's Ant-v5 [ext], ant_maze_v5.py:99: observation (105,) = 27 + 13 x 6): appended are the
// per-body external contact forces `data.cfrc_ext[1:]` clipped to contact_force_range = (-1, 1): for every body the sum of the
// contact forces acting on it as a spatial force [torque(3); force(3)] about the subtree com of its tree root, world axes, from
// the contacts and constraint forces of the LAST forward pass (Ant-v5 calls mj_rnePostConstraint after mj_step).  The group's
// spatial force about `ref` is sum_k F_k w_k over its contacts' base rows (what pass_F feeds into J^T f); body B of the pair
// receives +, body A -.  A refresh (no sub-step) reports zeros, as the reference's reset observation does (mj_resetData).
HD void antmaze_observe(const Ctx& c, const FetchTask& t, const float* goal, float* obs, float* achieved, float* desired,
                        float* reward, float* success, bool stepped
#ifdef B200_ANT
                        , AntForces* ant = nullptr
#endif
                        ) {
  const DMHead* h = c.h;
  const int q0 = t.obs_qpos_start;
  LANES(i, h->nq - q0) obs[i] = SF(qpos)[q0 + i];
  LANES(i, h->nv) obs[h->nq - q0 + i] = SF(qvel)[i];
#ifdef B200_ANT
  // touch_mode 3: cfrc_ext[1:] appended (Ant-v5), 4: all of cfrc_ext, world row first (Ant-v4 use_contact_forces, (111,)), 2: none; the
  // forces are clipped to contact_force_range and computed in every case, for the contact cost (the sum of their squares)
  const float cf_lo = ant ? ant->lo : -1.f, cf_hi = ant ? ant->hi : 1.f;
  float* cf = t.touch_mode >= 3 ? obs + (h->nq - q0 + h->nv) : nullptr;
  if (t.touch_mode == 4) { LANES(k, 6) cf[k] = 0.f; cf += 6; }
  float cf_sq = 0.f;
#define B200_CF_PUT(dst, v) do { const float v_ = (v); if (cf) dst = v_; cf_sq += v_ * v_; } while (0)
#define B200_CF_LO cf_lo
#define B200_CF_HI cf_hi
  {
#else
#define B200_CF_PUT(dst, v) dst = v
#define B200_CF_LO -1.f
#define B200_CF_HI 1.f
  if (t.touch_mode == 1) {
    float* cf = obs + (h->nq - q0 + h->nv);
#endif
    const int* cnt = SI(counters);
    const int ngrp = stepped ? cnt[CNT_NGRP] : 0;
    LANES(i, stepped ? cnt[CNT_NCON] : 0) {   // base-row forces of every contact (parked in the JV slots, as pass_F does)
      float* cr = SF(con) + i * CON_WORDS;
      float F[C_NB];
      contact_base_forces(cr, con_dim(cr), F);
      for (int k = 0; k < C_NB; k++) cr[C_JV + k] = F[k];
    }
    SYNC();
    LANES(idx, ngrp * 6) {
      int g = idx / 6, a = idx - 6 * g;
      float* gr = SF(group) + g * GRP_WORDS;
      float acc = 0;
      for (int i = grp_start(gr), i1 = i + grp_count(gr); i < i1; i++) {
        const float* cr = SF(con) + i * CON_WORDS;
        int dim = con_dim(cr);
        const float* F = cr + C_JV;
        acc += F[0] * cr[C_W + a];
        if (dim > 1) acc += F[1] * cr[C_W + 6 + a] + F[2] * cr[C_W + 12 + a];
        if (dim > 3 && a < 3) acc += F[3] * cr[C_W + 3 + a];
      }
      gr[G_V + a] = acc;
    }
    SYNC();
    LANES(b1, h->nmjb - 1) {
      if (!stepped) {   // a refresh computes no kinematics: xpos / xquat below would be whatever the shared memory last held
        for (int k = 0; k < 6; k++) B200_CF_PUT(cf[6 * b1 + k], 0.f);
        continue;
      }
      const int b = b1 + 1;      // MJCF body: the row layout of data.cfrc_ext (fused bodies keep their own rows)
      float acc[6] = {0, 0, 0, 0, 0, 0};
      for (int g = 0; g < ngrp; g++) {
        const float* gr = SF(group) + g * GRP_WORDS;
        if (grp_count(gr) == 0) continue;   // weld groups carry no contact
        int ba = grp_bodies(gr) & 0xff, bb = grp_bodies(gr) >> 8;
        float sg = b == bb ? 1.f : (b == ba ? -1.f : 0.f);
        if (sg != 0.f) for (int k = 0; k < 6; k++) acc[k] += sg * gr[G_V + k];
      }
      // subtree com of the tree root of body b (positions of the last forward pass)
      int root = GI(mjb_rt)[b];
      while (MI(body_parent)[root] != 0) root = MI(body_parent)[root];
      uint32_t sub = MU(body_sub)[root];
      float com[3] = {0, 0, 0}, mass = 0;
      while (sub) {
        int k = ffs_pop(sub);
        float ip[3], mk = MF(body_mass)[k];
        qrot(ip, SF(xquat) + 4 * k, MF(body_ipos) + 3 * k);
        for (int a = 0; a < 3; a++) com[a] += mk * (SF(xpos)[3 * k + a] + ip[a]);
        mass += mk;
      }
      float off[3], tq[3];
      for (int a = 0; a < 3; a++) off[a] = com[a] / mass - h->ref[a];
      cross3(tq, off, acc + 3);   // torque about the com = torque about ref - (com - ref) x force
      for (int a = 0; a < 3; a++) {
        B200_CF_PUT(cf[6 * b1 + a], fminf(fmaxf(acc[a] - tq[a], B200_CF_LO), B200_CF_HI));
        B200_CF_PUT(cf[6 * b1 + 3 + a], fminf(fmaxf(acc[3 + a], B200_CF_LO), B200_CF_HI));
      }
    }
  }
#ifdef B200_ANT
  if (ant) ant->sq = wsum(cf_sq);
#endif
#undef B200_CF_PUT
#undef B200_CF_LO
#undef B200_CF_HI
  if (c.lane == 0) {
    float dx = SF(qpos)[0] - goal[0], dy = SF(qpos)[1] - goal[1];
    // the same rounding sequence as reward_kernel's loop over the goal entries (b200sim.cu): round(dx^2), then one fused multiply-add --
    // `reward == compute_reward(achieved_goal, desired_goal)` holds bit for bit (core.py:61-62), dense exp(-d) rewards included
#ifdef __CUDA_ARCH__
    float d = sqrtf(fmaf(dy, dy, __fmul_rn(dx, dx)));
#else
    float d = sqrtf(dx * dx + dy * dy);
#endif
    achieved[0] = SF(qpos)[0]; achieved[1] = SF(qpos)[1]; desired[0] = goal[0]; desired[1] = goal[1];
    *reward = t.reward_dense ? expf(-d) : (d <= t.success_radius ? 1.f : 0.f);
    *success = d <= t.success_radius ? 1.f : 0.f;
  }
}

HD void quat_to_euler(const float* q, float* e) {
  float n = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  float m[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (n > 2.220446e-16f) {
    float sc = 2.0f / n, w = q[0], x = q[1], y = q[2], z = q[3];
    m[0] = 1 - sc * (y * y + z * z); m[1] = sc * (x * y - w * z); m[2] = sc * (x * z + w * y);
    m[3] = sc * (x * y + w * z); m[4] = 1 - sc * (x * x + z * z); m[5] = sc * (y * z - w * x);
    m[6] = sc * (x * z - w * y); m[7] = sc * (y * z + w * x); m[8] = 1 - sc * (x * x + y * y);
  }
  float cy = sqrtf(m[8] * m[8] + m[5] * m[5]);
  if (cy > 8.8817841970012523e-16f) { e[2] = -atan2f(m[1], m[0]); e[1] = -atan2f(-m[2], cy); e[0] = -atan2f(m[5], m[8]); }
  else { e[2] = -atan2f(-m[3], m[4]); e[1] = -atan2f(-m[2], cy); e[0] = 0.f; }
}
HD void euler_to_quat(const float* e, float* q) {
  float ai = 0.5f * e[2], aj = -0.5f * e[1], ak = 0.5f * e[0];
  float si = sinf(ai), sj = sinf(aj), sk = sinf(ak), ci = cosf(ai), cj = cosf(aj), ck = cosf(ak);
  float cc = ci * ck, cs = ci * sk, sc = si * ck, ss = si * sk;
  q[0] = cj * cc + sj * ss; q[3] = cj * sc - sj * cs; q[2] = -(cj * ss + sj * cc); q[1] = cj * cs - sj * sc;
}

// Shadow-hand block manipulation: obs = robot qpos | robot qvel | object qvel | object qpos, achieved = object qpos (7)
// (reference: envs/shadow_dexterous_hand/manipulate.py:298-314, :88-138)
HD void hand_goal_distance(const FetchTask& t, const float* a, const float* g, float* d_pos, float* d_rot) {
  *d_pos = 0.f; *d_rot = 0.f;
  if (t.goal_flags & GOAL_USE_POS) { float e[3] = {a[0] - g[0], a[1] - g[1], a[2] - g[2]}; *d_pos = sqrtf(dot3(e, e)); }
  if (t.goal_flags & GOAL_USE_ROT) {
    float qa[4] = {a[3], a[4], a[5], a[6]};
    if (t.goal_flags & GOAL_IGNORE_Z) {
      // ignore_z_target_rotation (manipulate.py:97-106; the pen): both quaternions to Euler angles (R = Rx Ry Rz,
      // utils/rotations.py:162-184, 245-271), the achieved z angle replaced by the goal's, back to a quaternion (:140-159)
      float ea[3], eb[3];
      quat_to_euler(a + 3, ea);
      quat_to_euler(g + 3, eb);
      ea[2] = eb[2];
      euler_to_quat(ea, qa);
    }
    // w component of qa * conj(g)
    float w = qa[0] * g[3] + qa[1] * g[4] + qa[2] * g[5] + qa[3] * g[6];
    *d_rot = 2.f * acosf(fminf(fmaxf(w, -1.f), 1.f));
  }
}
HD float hand_reward(const FetchTask& t, float d_pos, float d_rot, float* success) {
  float s = (d_pos < t.distance_threshold ? 1.f : 0.f) * (d_rot < t.rotation_threshold ? 1.f : 0.f);
  if (success) *success = s;
  return t.reward_dense ? -(10.f * d_pos + d_rot) : s - 1.f;
}
HD void hand_observe(const Ctx& c, const FetchTask& t, const float* goal, float* obs, float* achieved, float* desired,
                     float* reward, float* success) {
  const DMHead* h = c.h;
  const int nrq = t.obj_qadr, nrv = t.obj_dadr;  // robot joints come first, the object's free joint last
  LANES(i, nrq) obs[i] = SF(qpos)[i];
  LANES(i, nrv) obs[nrq + i] = SF(qvel)[i];
  LANES(i, 6) obs[nrq + nrv + i] = SF(qvel)[nrv + i];
  LANES(i, 7) { float v = SF(qpos)[nrq + i]; obs[nrq + nrv + 6 + i] = v; achieved[i] = v; desired[i] = goal[i]; }
  if (c.lane == 0) {
    float dp, dr;
    hand_goal_distance(t, SF(qpos) + nrq, goal, &dp, &dr);
    *reward = hand_reward(t, dp, dr, success);
  }
  (void)h;
}

// HandReach: obs = robot qpos | robot qvel | 5 fingertip site positions (as of the last forward pass), which are also the
// achieved goal; reward / success on the 15-dim distance (reference: envs/shadow_dexterous_hand/reach.py:88-130, 284-300)
HD void reach_observe(const Ctx& c, const FetchTask& t, const float* goal, float* obs, float* achieved, float* desired,
                      float* reward, float* success) {
  const DMHead* h = c.h;
  LANES(i, h->nq) obs[i] = SF(qpos)[i];
  LANES(i, h->nv) obs[h->nq + i] = SF(qvel)[i];
  float d2 = 0.f;
#ifdef B200_WARP_CODE
  // lane k < 5 holds the error of finger tip k; the squared distance is then accumulated over the 15 entries IN ORDER by every lane
  // (15 shuffles, once per env-step): the rounding sequence of reward_kernel's loop, so that the dense reward equals compute_reward bit for bit
  float e3[3] = {0.f, 0.f, 0.f};
  LANES(k, 5) {
    float p[3];
    site_pose(c, t.tip_site[k], p, nullptr);
    for (int a = 0; a < 3; a++) {
      obs[h->nq + h->nv + 3 * k + a] = p[a]; achieved[3 * k + a] = p[a]; desired[3 * k + a] = goal[3 * k + a];
      e3[a] = p[a] - goal[3 * k + a];
    }
  }
  for (int k = 0; k < 5; k++)
    for (int a = 0; a < 3; a++) { float e = __shfl_sync(0xffffffffu, e3[a], k); B200_SQACC(d2, e); }
  float d = sqrtf(d2);
#else
  LANES(k, 5) {
    float p[3];
    site_pose(c, t.tip_site[k], p, nullptr);
    for (int a = 0; a < 3; a++) {
      obs[h->nq + h->nv + 3 * k + a] = p[a]; achieved[3 * k + a] = p[a]; desired[3 * k + a] = goal[3 * k + a];
      float e = p[a] - goal[3 * k + a];
      B200_SQACC(d2, e);
    }
  }
  float d = sqrtf(wsum(d2));
#endif
  if (c.lane == 0) {
    *reward = t.reward_dense ? -d : -(d > t.distance_threshold ? 1.f : 0.f);
    *success = d < t.distance_threshold ? 1.f : 0.f;
  }
}

// Touch sensors as of the last forward pass (public MuJoCo semantics, restated in oracle/oracle.c `sensors`): sum of the
// normal forces of the contacts that involve the sensor's body and whose ray from the contact point along the contact
// normal (flipped when the sensor's body is the second one) hits the site volume.  Appended to the observation by
// MujocoManipulateTouchSensorsEnv._get_obs (envs/shadow_dexterous_hand/manipulate_touch_sensors.py:107-138).
HD bool ray_hits_site(int type, const float* size, const float* p, const float* d) {
  if (type == B200_GEOM_SPHERE) {
    float r = size[0], b = dot3(p, d), cc = dot3(p, p) - r * r;
    if (cc <= 0) return true;
    return b * b - cc >= 0 && -b >= 0;
  }
  if (type == B200_GEOM_CYLINDER) {
    // slab |z| <= half length, then the infinite cylinder x^2 + y^2 <= r^2 over the slab's parameter interval
    float t0 = 0, t1 = 1e30f, r = size[0], hl = size[1];
    if (fabsf(d[2]) < 1e-12f) { if (fabsf(p[2]) > hl) return false; }
    else {
      float a = (-hl - p[2]) / d[2], b = (hl - p[2]) / d[2];
      if (a > b) { float t = a; a = b; b = t; }
      t0 = fmaxf(t0, a); t1 = fminf(t1, b);
      if (t0 > t1) return false;
    }
    float A = d[0] * d[0] + d[1] * d[1], B = p[0] * d[0] + p[1] * d[1], C = p[0] * p[0] + p[1] * p[1] - r * r;
    if (A < 1e-20f) return C <= 0;
    float disc = B * B - A * C;
    if (disc < 0) return false;
    float sq = sqrtf(disc), ta = (-B - sq) / A, tb = (-B + sq) / A;
    return fmaxf(t0, ta) <= fminf(t1, tb);
  }
  float t0 = 0, t1 = 1e30f;
  for (int k = 0; k < 3; k++) {
    if (fabsf(d[k]) < 1e-12f) { if (fabsf(p[k]) > size[k]) return false; continue; }
    float a = (-size[k] - p[k]) / d[k], b = (size[k] - p[k]) / d[k];
    if (a > b) { float t = a; a = b; b = t; }
    t0 = fmaxf(t0, a); t1 = fminf(t1, b);
    if (t0 > t1) return false;
  }
  return true;
}
HD void touch_observe(const Ctx& c, const FetchTask& t, float* out, int nmax = 1 << 30) {
  const DMHead* h = c.h;
  const int ncon = SI(counters)[CNT_NCON];
  LANES(k, (h->nsensor < nmax ? h->nsensor : nmax)) {
    int site = GI(sensor_site)[k], body = GI(sensor_body)[k], type = GI(sensor_type)[k];
    float size[3] = {GF(sensor_size)[3 * k], GF(sensor_size)[3 * k + 1], GF(sensor_size)[3 * k + 2]};
    float total = 0.f, sp[3], sq[4];
    bool posed = false;
    for (int i = 0; i < ncon; i++) {
      const float* cr = SF(con) + i * CON_WORDS;
      const float* cx = SF(conx) + i * CX_WORDS;
      int p = ((const int*)cx)[CX_PAIR];
      int g1 = PAIR_I(pair_geom1)[p], g2 = PAIR_I(pair_geom2)[p];
      int b1 = MI(geom_body)[g1], b2 = g2 < 0 ? 0 : MI(geom_body)[g2];
      if (b1 != body && b2 != body) continue;
      float F[C_NB];
      contact_base_forces(cr, con_dim(cr), F);
      if (!(F[0] > 0)) continue;
      if (!posed) { site_pose(c, site, sp, sq); posed = true; }
      float rel[3] = {cx[CX_POS] - sp[0], cx[CX_POS + 1] - sp[1], cx[CX_POS + 2] - sp[2]};
      float sg = b2 == body ? -1.f : 1.f, dir[3] = {sg * cr[C_W + 3], sg * cr[C_W + 4], sg * cr[C_W + 5]};  // contact normal
      float qc[4] = {sq[0], -sq[1], -sq[2], -sq[3]}, loc[3], dl[3];
      qrot(loc, qc, rel); qrot(dl, qc, dir);
      if (ray_hits_site(type, size, loc, dl)) total += F[0];
    }
    out[k] = t.touch_mode == 2 ? (total > 0.f ? 1.f : 0.f) : (t.touch_mode == 3 ? logf(total + 1.f) : total);
  }
}

// AdroitHandHammer (envs/adroit_hand/adroit_hammer.py:291-357): every derived quantity is the one of the last forward pass
// (data.xpos / site_xpos / sensordata after mj_step), qpos / qvel are the integrated ones.
HD void adroit_hammer_observe(const Ctx& c, const FetchTask& t, float* obs, float* achieved, float* desired, float* reward,
                              float* success) {
  const DMHead* h = c.h;
  const int nq = h->nq, nv = h->nv, nr = nq - 6;
  LANES(i, nr) obs[i] = SF(qpos)[i];
  LANES(i, 6) obs[nr + i] = fminf(fmaxf(SF(qvel)[nv - 6 + i], -1.f), 1.f);
  float v2 = 0.f;
  LANES(i, nv) v2 += SF(qvel)[i] * SF(qvel)[i];
  v2 = wsum(v2);
  float touch = 0.f;
  if (h->nsensor > 0) {   // sensordata of "S_nail" (the model keeps only this sensor), clipped to [-1, 1]
    float tv[1] = {0.f};
    FetchTask tt = t; tt.touch_mode = 1;
    touch_observe(c, tt, tv, 1);
    touch = fminf(fmaxf(tv[0], -1.f), 1.f);
  }
  if (c.lane == 0) {
    float palm[3], hamm[3], hq[4], head[3], nail[3], goal[3], e[3];
    site_pose(c, t.grip_site, palm, nullptr);
    site_pose(c, t.obj_site, hamm, hq);
    site_pose(c, t.tip_site[0], head, nullptr);
    site_pose(c, t.frame_site, nail, nullptr);
    site_pose(c, t.tip_site[1], goal, nullptr);
    quat_to_euler(hq, e);
    float* o = obs + nr + 6;
    for (int k = 0; k < 3; k++) { o[k] = palm[k]; o[3 + k] = hamm[k]; o[6 + k] = e[k]; o[9 + k] = nail[k]; achieved[k] = nail[k]; desired[k] = goal[k]; }
    o[12] = touch;
    float dg[3] = {nail[0] - goal[0], nail[1] - goal[1], nail[2] - goal[2]}, dp[3] = {palm[0] - hamm[0], palm[1] - hamm[1], palm[2] - hamm[2]},
          dh[3] = {head[0] - nail[0], head[1] - nail[1], head[2] - nail[2]};
    float gd = sqrtf(dot3(dg, dg));
    bool ok = gd < 0.01f;
    float r = ok ? 10.f : -0.1f;
    if (t.reward_dense) {
      r = -0.1f * sqrtf(dot3(dp, dp)) - sqrtf(dot3(dh, dh)) - 10.f * gd - 1e-2f * sqrtf(v2);
      if (hamm[2] > 0.04f && head[2] > 0.04f) r += 2.f;
      if (gd < 0.020f) r += 25.f;
      if (gd < 0.010f) r += 75.f;
    }
    *reward = r; *success = ok ? 1.f : 0.f;
  }
}

// AdroitHandRelocate (envs/adroit_hand/adroit_relocate.py:288-345): obs = qpos[:-6] | palm - ball | palm - target | ball - target;
// the target is a per-env world site position (site_pos redrawn by reset_model, :354-373) kept in the goal slot of the state
HD void adroit_relocate_observe(const Ctx& c, const FetchTask& t, const float* goal, float* obs, float* achieved, float* desired,
                                float* reward, float* success) {
  const DMHead* h = c.h;
  const int nr = h->nq - 6;
  LANES(i, nr) obs[i] = SF(qpos)[i];
  if (c.lane == 0) {
    float palm[3], ball[3];
    site_pose(c, t.grip_site, palm, nullptr);
    site_pose(c, t.obj_site, ball, nullptr);
    float po[3], pt[3], ot[3];
    for (int k = 0; k < 3; k++) {
      po[k] = palm[k] - ball[k]; pt[k] = palm[k] - goal[k]; ot[k] = ball[k] - goal[k];
      obs[nr + k] = po[k]; obs[nr + 3 + k] = pt[k]; obs[nr + 6 + k] = ot[k];
      achieved[k] = ball[k]; desired[k] = goal[k];
    }
    float gd = sqrtf(dot3(ot, ot));
    bool ok = gd < 0.1f;
    float r = ok ? 10.f : -0.1f;
    if (t.reward_dense) {
      r = -0.1f * sqrtf(dot3(po, po));
      if (ball[2] > 0.04f) r += 1.0f - 0.5f * sqrtf(dot3(pt, pt)) - 0.5f * gd;
      if (gd < 0.1f) r += 10.f;
      if (gd < 0.05f) r += 20.f;
    }
    *reward = r; *success = ok ? 1.f : 0.f;
  }
}

// AdroitHandPen (envs/adroit_hand/adroit_pen.py:288-378): obs = qpos[:-6] | pen pos | pen qvel | pen direction | desired
// direction | pen pos - desired pos | direction difference (45).  Directions are (top site - bottom site) / length; the two
// lengths are measured once at reset in the reference (:392-399) and are model constants (distance_threshold = pen length,
// rotation_threshold = target length here).  The target pen is a static body whose quaternion is per-env state.
HD void adroit_pen_observe(const Ctx& c, const FetchTask& t, float* obs, float* achieved, float* desired, float* reward,
                           float* success) {
  const DMHead* h = c.h;
  const int nr = h->nq - 6, nv = h->nv;
  LANES(i, nr) obs[i] = SF(qpos)[i];
  LANES(i, 6) obs[nr + 3 + i] = SF(qvel)[nv - 6 + i];
  if (c.lane == 0) {
    float pos[3], loc[3], ot[3], ob[3], tt[3], tb[3], oo[3], dd[3];
    site_pose(c, t.obj_site, pos, nullptr);
    site_pose(c, t.frame_site, loc, nullptr);
    site_pose(c, t.tip_site[0], ot, nullptr); site_pose(c, t.tip_site[1], ob, nullptr);
    site_pose(c, t.tip_site[2], tt, nullptr); site_pose(c, t.tip_site[3], tb, nullptr);
    const float il = 1.0f / t.distance_threshold, it = 1.0f / t.rotation_threshold;
    float dl[3];
    for (int k = 0; k < 3; k++) {
      oo[k] = (ot[k] - ob[k]) * il; dd[k] = (tt[k] - tb[k]) * it; dl[k] = pos[k] - loc[k];
      obs[nr + k] = pos[k]; obs[nr + 9 + k] = oo[k]; obs[nr + 12 + k] = dd[k]; obs[nr + 15 + k] = dl[k]; obs[nr + 18 + k] = oo[k] - dd[k];
      achieved[k] = oo[k]; desired[k] = dd[k];
    }
    float gd = sqrtf(dot3(dl, dl)), sim = dot3(oo, dd);
    bool ok = gd < 0.075f && sim > 0.95f;
    float r = ok ? 10.f : -0.1f;
    if (t.reward_dense) {
      r = -gd + sim;
      if (gd < 0.075f && sim > 0.9f) r += 10.f;
      if (gd < 0.075f && sim > 0.95f) r += 50.f;
      if (pos[2] < 0.075f) r -= 5.f;
    }
    *reward = r; *success = ok ? 1.f : 0.f;
  }
}

// AdroitHandDoor (envs/adroit_hand/adroit_door.py:279-344): obs = qpos[1:-2] | latch | door hinge | palm | handle | palm - handle |
// door_open (+-1) (39); obj_qadr = qpos address of "door_hinge" (the latch is the last joint)
HD void adroit_door_observe(const Ctx& c, const FetchTask& t, float* obs, float* achieved, float* desired, float* reward,
                            float* success) {
  const DMHead* h = c.h;
  const int nq = h->nq, nv = h->nv, nr = nq - 3;
  LANES(i, nr) obs[i] = SF(qpos)[1 + i];
  float v2 = 0.f;
  LANES(i, nv) v2 += SF(qvel)[i] * SF(qvel)[i];
  v2 = wsum(v2);
  if (c.lane == 0) {
    float palm[3], handle[3], dp[3];
    site_pose(c, t.grip_site, palm, nullptr);
    site_pose(c, t.frame_site, handle, nullptr);
    const float door = SF(qpos)[t.obj_qadr], latch = SF(qpos)[nq - 1];
    obs[nr] = latch; obs[nr + 1] = door;
    for (int k = 0; k < 3; k++) { dp[k] = palm[k] - handle[k]; obs[nr + 2 + k] = palm[k]; obs[nr + 5 + k] = handle[k]; obs[nr + 8 + k] = dp[k]; achieved[k] = palm[k]; desired[k] = handle[k]; }
    obs[nr + 11] = door > 1.0f ? 1.f : -1.f;
    bool ok = door >= 1.35f;
    float r = ok ? 10.f : -0.1f;
    if (t.reward_dense) {
      r = -0.1f * sqrtf(dot3(dp, dp)) - 0.1f * (door - 1.57f) * (door - 1.57f) - 1e-5f * v2;
      if (door > 0.2f) r += 2.f;
      if (door > 1.0f) r += 8.f;
      if (door > 1.35f) r += 10.f;
    }
    *reward = r; *success = ok ? 1.f : 0.f;
  }
}

#ifdef B200_KITCHEN
#include "reset_sample.cuh"
// FrankaKitchen observation noise (franka_env.py:114-124, kitchen_env.py:374-385; b200sim_set_obs_noise): block b of the
// Philox4x32-10 stream (seed; env, episode, step t) holds the uniforms of observation entries 4 b .. 4 b + 3, each in [-1, 1).
// `t` is the env's step counter after the launch, so that a refresh after set_state(elapsed = t) redraws the noise step t drew.
// t < 2^28, b < 16; the tag 0x0B5E is used by no other draw (reset_sample.cuh).
#define RS_OBS_NOISE_TAG 0x0B5Eu
RS_HD void rs_obs_noise_block(unsigned long long seed, uint32_t env, uint32_t episode, uint32_t t, uint32_t b, float u[4]) {
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  const uint32_t ctr[4] = {env, episode, (t << 4) | b, RS_OBS_NOISE_TAG};
  uint32_t r[4];
  rs_philox4x32_10(ctr, key, r);
  for (int w = 0; w < 4; w++) u[w] = 2.0f * rs_u01(r[w]) - 1.0f;   // exact in fp32: (k - 2^23) / 2^23
}
// One env's noise stream in one launch: `scale` holds one amplitude per observation entry, env is the global env index
struct ObsNoiseKey {
  const float* scale;
  unsigned long long seed;
  uint32_t env, episode, t;
};
// FrankaKitchen-v1 (envs/franka_kitchen/franka_env.py:92-128, kitchen_env.py:371-423): the kernel runs do_simulation(ctrl, 40)
// and returns the observation robot qpos | robot qvel | object qpos | object qvel (the first nu joints are the robot's) and
// the full, noise-free qpos as `achieved` (the task bookkeeping reads the true state, kitchen_env.py:356-369).  Without `noise`
// the observation is noise-free and the host adds the noise (rng_mode "numpy" / "torch"); with it (rng_mode "device") the
// kernel adds u * scale[j] to entry j, u = uniform j % 4 of block j / 4 of the env's stream, one lane per block.  The
// position targets and the bookkeeping are batched host-side tensor code (gymnasium_robotics_b200/kitchen.py), as they are
// Python in the reference.
HD void kitchen_observe(const Ctx& c, const FetchTask& t, float* obs, float* achieved, float* desired, float* reward, float* success,
                        const ObsNoiseKey* noise) {
  const DMHead* h = c.h;
  const int nr = h->nu, nq = h->nq, nv = h->nv;
  if (noise) {
    LANES(b, (t.nobs + 3) >> 2) {
      float u[4];
      rs_obs_noise_block(noise->seed, noise->env, noise->episode, noise->t, (uint32_t)b, u);
      for (int w = 0; w < 4; w++) {
        const int j = 4 * b + w;
        if (j >= t.nobs) break;
        const float v = j < nr ? SF(qpos)[j] : (j < 2 * nr ? SF(qvel)[j - nr] : (j < nr + nq ? SF(qpos)[j - nr] : SF(qvel)[j - nq]));
#ifdef __CUDA_ARCH__
        obs[j] = v + __fmul_rn(u[w], noise->scale[j]);   // the product rounded on its own, as the host build rounds it
#else
        obs[j] = v + u[w] * noise->scale[j];
#endif
      }
    }
  } else {
    LANES(i, nr) { obs[i] = SF(qpos)[i]; obs[nr + i] = SF(qvel)[i]; }
    LANES(i, nq - nr) obs[2 * nr + i] = SF(qpos)[nr + i];
    LANES(i, nv - nr) obs[2 * nr + (nq - nr) + i] = SF(qvel)[nr + i];
  }
  LANES(i, nq) { achieved[i] = SF(qpos)[i]; desired[i] = 0.f; }
  if (c.lane == 0) { *reward = 0.f; *success = 0.f; }
}
#endif

// one env, one warp.  `st` is this env's state record; outputs are this env's rows.  `active` is warp-uniform: idle
// warps run the same control flow (for the block-wide alignment barriers) but touch no memory.
// REBUILD: rebuild the context before each stage call (stage_ctx).  Kitchen builds: `noise`, the env's observation noise (NULL =
// none); the ant build: `ant`, the contact-force clip range in, the contact forces' sum of squares out; these parameters exist in
// those builds only, so that the other builds' kernels keep their source and parameters.
template <int NVP, bool REBUILD = false>
HD void fetch_env_step(const Ctx& c, const FetchTask& t, bool active, int mode, int nraw, float* st, const float* action, float* obs,
                       float* achieved, float* desired, float* reward, float* success, int* iters_out
#ifdef B200_KITCHEN
                       , const ObsNoiseKey* noise = nullptr
#endif
#ifdef B200_ANT
                       , AntForces* ant = nullptr
#endif
                       ) {
  const DMHead* h = c.h;
  if (active) {
    load_state(c, t, st);
    if (NVP >= 30 && mode == MODE_STEP && (t.kind == TASK_HAND || t.kind == TASK_HAND_REACH || TASK_IS_ADROIT(t.kind))) {
      // (Adroit: a = act_mean + clip(a) * act_rng, adroit_hammer.py:292-293 -- the same arithmetic)
      // MujocoHandEnv._set_action (hand_env.py:42-61, absolute control): ctrl = centre + clip(a) * half range, clipped
      LANES(i, h->nu) {
        float lo = MF(act_ctrlrange)[2 * i], hi = MF(act_ctrlrange)[2 * i + 1];
        float a = fminf(fmaxf(action[i], -1.f), 1.f);
        SF(ctrl)[i] = fminf(fmaxf(0.5f * (hi + lo) + a * (0.5f * (hi - lo)), lo), hi);
      }
      SYNC();
    } else if (mode == MODE_STEP && t.kind == TASK_FETCH) {
      // _set_action: clip, scale, mocap <- last forward pose of the welded body + delta, position actuators relative
      float a[4];
      for (int k = 0; k < 4; k++) a[k] = fminf(fmaxf(action[k], -1.f), 1.f);
      if (c.lane == 0) {
        for (int k = 0; k < 3; k++) SF(mocap_pos)[k] = st[t.st_pose + k] + 0.05f * a[k];
        const float rot[4] = {1.f, 0.f, 1.f, 0.f};
        for (int k = 0; k < 4; k++) SF(mocap_quat)[k] = st[t.st_pose + 3 + k] + rot[k];
        float g = t.block_gripper ? 0.f : a[3];
        for (int i = 0; i < h->nu; i++) SF(ctrl)[i] = SF(qpos)[MI(jnt_qposadr)[MI(act_trnid)[i]]] + g;
      }
      SYNC();
    } else if (mode == MODE_STEP) {
      // do_simulation(action, frame_skip): ctrl = action (clamped to ctrlrange inside the actuation stage);
      // PointEnv.step first clips the action and the velocity (envs/maze/point.py:52-77)
      LANES(i, h->nu) SF(ctrl)[i] = action[i];
      if (t.vel_clip > 0) {
        LANES(i, h->nu) SF(ctrl)[i] = fminf(fmaxf(action[i], -1.f), 1.f);
        LANES(i, h->nv) SF(qvel)[i] = fminf(fmaxf(SF(qvel)[i], -t.vel_clip), t.vel_clip);
      }
      SYNC();
    }
  }
  int nsub = mode == MODE_STEP ? t.n_substeps : (mode == MODE_RAW ? nraw : 0);
  for (int s = 0; s < nsub; s++) {
    forward<NVP, REBUILD>(c, active);
    TIC();
    if (NVP >= 30) ALIGN(); TOC(TM_BARRIER);
    if (h->integrator == B200_INT_RK4) rk4_substep<NVP, REBUILD>(c, active);
    else if (active) euler_step<NVP>(stage_ctx<REBUILD>(c));
    TOC(TM_INTEG);
  }
  // touch sensors read the contacts and forces of the last forward pass: a refresh (no sub-step) runs one first,
  // block-uniformly (forward() contains the block-wide alignment barriers); the warm start is left untouched
  const bool touch_fwd = NVP >= 30 && ((t.kind == TASK_HAND && t.touch_mode != 0) || t.kind == TASK_ADROIT_HAMMER) && nsub == 0;
  if (touch_fwd) {
    forward<NVP, REBUILD>(c, active);
    if (active) { LANES(i, h->nv) SF(qacc)[i] = st[t.st_warm + i]; SYNC(); }
  }
  if (!active) return;
  if (t.kind == TASK_FETCH) {
    if (mode == MODE_REFRESH || (mode == MODE_STEP && t.block_gripper) || nsub == 0) {
      if (mode == MODE_STEP && t.block_gripper) {
        if (c.lane == 0) { SF(qpos)[t.finger_qadr[0]] = 0.f; SF(qpos)[t.finger_qadr[1]] = 0.f; }
        SYNC();
      }
      kinematics(c);
      com_quantities(c);
    }
    fetch_observe(c, t, st + t.st_goal, obs, achieved, desired, reward, success);
  } else if (NVP >= 30 && t.kind == TASK_HAND_REACH) {
    if (nsub == 0) kinematics(c);   // refresh after a reset: site positions of the new state
    reach_observe(c, t, st + t.st_goal, obs, achieved, desired, reward, success);
  } else if (NVP >= 30 && t.kind == TASK_ADROIT_HAMMER) {
    adroit_hammer_observe(c, t, obs, achieved, desired, reward, success);
#ifdef B200_KITCHEN
  } else if (NVP >= 30 && t.kind == TASK_KITCHEN) {
    kitchen_observe(c, t, obs, achieved, desired, reward, success, noise);
#endif
  } else if (NVP >= 30 && t.kind == TASK_ADROIT_DOOR) {
    if (nsub == 0) kinematics(c);
    adroit_door_observe(c, t, obs, achieved, desired, reward, success);
  } else if (NVP >= 30 && t.kind == TASK_ADROIT_PEN) {
    if (nsub == 0) kinematics(c);
    adroit_pen_observe(c, t, obs, achieved, desired, reward, success);
  } else if (NVP >= 30 && t.kind == TASK_ADROIT_RELOCATE) {
    if (nsub == 0) kinematics(c);   // refresh after a reset: body / site positions of the new state
    adroit_relocate_observe(c, t, st + t.st_goal, obs, achieved, desired, reward, success);
  } else if (NVP >= 30 && t.kind == TASK_HAND) {
    hand_observe(c, t, st + t.st_goal, obs, achieved, desired, reward, success);
    if (t.touch_mode) touch_observe(c, t, obs + t.obj_qadr + h->nv + 7);
  } else {
#ifdef B200_ANT
    antmaze_observe(c, t, st + t.st_goal, obs, achieved, desired, reward, success, nsub > 0, ant);
#else
    antmaze_observe(c, t, st + t.st_goal, obs, achieved, desired, reward, success, nsub > 0);
#endif
  }
  store_state(c, t, st);
  if (iters_out && c.lane == 0) *iters_out = SI(counters)[CNT_ITERS] | (SI(counters)[CNT_OVERFLOW] << 16);
}

// The Ant's keywords and per-step info of a handle (b200sim_set_ant_info): contact_force_range, the cost and reward weights, the healthy
// z range, the Ant version's info rules, the [N, 9] info rows (NULL = none) and the [N, 2] reset positions of Ant-v5's
// distance_from_origin.  A kernel parameter of the ant build only (b200sim_ant.cu, csrc/step_kernel.cuh), as ObsNoiseArgs is of the kitchen builds.
struct AntInfoArgs {
  float cf_lo, cf_hi, forward_w, ctrl_w, contact_w, healthy_reward, z_lo, z_hi;
  int v4, survive_always, contact_in_ctrl;   // Ant-v4 rules; terminate_when_unhealthy and use_contact_forces under them
  float* rows; const float* origin;
};
#ifdef B200_ANT
// Lane 0 of an ant-build env after its launch.  The torso's xy of the last forward pass (the last RK4 stage of a step; qpos[0:2] after a
// refresh, which runs mj_forward on the new state) is kept in the two record words after the goal; a step's velocity is the change of
// it over dt = timestep x frame_skip.  A step writes the info row of Ant.step [ext] (ant_v3.py:76-145 with the v4 / v5 changes): v5
// x, y = qpos[0:2], distance from the reset position, reward_forward = forward_reward_weight * vx, reward_ctrl = -ctrl_cost (the
// action as passed, before the ctrlrange clamp), reward_contact = -contact_cost, reward_survive = healthy_reward * is_healthy; v4 x, y
// = the torso's xpos and its distance from the world origin, reward_forward = vx, reward_ctrl = -contact_cost under
// use_contact_forces (Ant-v4's info bug, fixed in v5), reward_survive = healthy_reward * (is_healthy or terminate_when_unhealthy).  A
// refresh writes the reset info (v5: x, y and distance 0; v4: none) with the other columns 0.
HD void ant_info(const Ctx& c, const FetchTask& t, const AntInfoArgs& a, int mode, bool stepped, float* st, const float* action,
                 float contact_sq, size_t e) {
  const DMHead* h = c.h;
  const float* qp = SF(qpos);
  float* stale = st + t.st_goal + t.ngoal;
  const int tb = 3 * GI(mjb_rt)[1];   // MJCF body 1, the torso (main_body)
  const float x = stepped ? SF(xpos)[tb] : qp[0], y = stepped ? SF(xpos)[tb + 1] : qp[1];
  if (a.rows && mode != MODE_RAW) {
    float r[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (mode == MODE_STEP) {
      const float vx = (x - stale[0]) / t.dt, vy = (y - stale[1]) / t.dt;
      float ctrl = 0.f;
      for (int i = 0; i < t.nact; i++) ctrl += action[i] * action[i];
      ctrl *= a.ctrl_w;
      const float contact = a.contact_w * contact_sq;
      bool healthy = qp[2] >= a.z_lo && qp[2] <= a.z_hi;
      for (int i = 0; i < h->nq; i++) healthy = healthy && isfinite(qp[i]);
      for (int i = 0; i < h->nv; i++) healthy = healthy && isfinite(SF(qvel)[i]);
      r[3] = vx; r[4] = vy; r[7] = -contact;
      r[8] = (healthy || (a.v4 && a.survive_always)) ? a.healthy_reward : 0.f;
      if (a.v4) {
        r[0] = x; r[1] = y; r[2] = sqrtf(x * x + y * y); r[5] = vx; r[6] = a.contact_in_ctrl ? -contact : -ctrl;
      } else {
        const float dx = qp[0] - a.origin[2 * e], dy = qp[1] - a.origin[2 * e + 1];
        r[0] = qp[0]; r[1] = qp[1]; r[2] = sqrtf(dx * dx + dy * dy); r[5] = a.forward_w * vx; r[6] = -ctrl;
      }
    } else if (!a.v4) {
      r[0] = qp[0]; r[1] = qp[1];
    }
    for (int k = 0; k < 9; k++) a.rows[9 * e + k] = r[k];
  }
  stale[0] = x; stale[1] = y;
}
#endif
