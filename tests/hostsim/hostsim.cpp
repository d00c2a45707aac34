// TEST-ONLY host emulation of the CUDA physics core: compiles gymnasium_robotics_b200/csrc/sim_core.cuh with
// WARP_W == 1 (one "lane" runs every strided loop) so the fp32 kernel arithmetic can be compared with the fp64 oracle
// on a machine without a GPU.  Never linked into the product library; the product path is CUDA only.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <string>
#include <type_traits>
#ifdef B200_HOST_WARP
#include "hostwarp.h"   // WARP_W == 32: the lane-parallel code paths on 32 lock-step fibers
#endif
#include "../../gymnasium_robotics_b200/csrc/fetch_task.cuh"

// run f(ctx) once (WARP_W == 1) or on the 32 lanes of the emulated warp
#if defined(B200_HOST_WARP) && defined(B200_STAGE_TIMING)
static long long g_stage_rounds[TM_COUNT];   // lane 0's per-stage collective counts, accumulated over calls
extern "C" int hostsim_stage_rounds(long long* out, int reset) {
  for (int k = 0; k < TM_COUNT; k++) { out[k] = g_stage_rounds[k]; if (reset) g_stage_rounds[k] = 0; }
  return TM_COUNT;
}
#endif
template <class F> static void warp_call(const Ctx& base, F f) {
#if defined(B200_HOST_WARP) && defined(B200_STAGE_TIMING)
  hw_run([&](int lane) {
    long long tim[TM_COUNT] = {0};
    Ctx c = base; c.lane = lane; c.tim = tim; f(c);
    if (lane == 0) for (int k = 0; k < TM_COUNT; k++) g_stage_rounds[k] += tim[k];
  });
#elif defined(B200_HOST_WARP)
  hw_run([&](int lane) { Ctx c = base; c.lane = lane; f(c); });
#else
  f(base);
#endif
}

#ifdef B200_WIDE
static const bool kWide = true;   // 64-bit dof masks: the tables carry two words per mask
#else
static const bool kWide = false;
#endif
// the padded dof count of the product kernel build this flavor stands for: the wide build's bordered Cholesky (32 + 4 rows), the
// kitchen builds' 31, else 32 (the WARP_W == 1 flavors solve with the shared-memory Cholesky whatever the size)
#if defined(B200_WIDE)
#define HOST_NVP 36
#elif defined(B200_KITCHEN)
#define HOST_NVP 31
#else
#define HOST_NVP 32
#endif

struct HostSim {
  std::vector<uint8_t> blob;
  b200_model_view view;
  std::vector<uint32_t> model;
  std::vector<float> scratch;
  Ctx ctx;
  std::string err;
};

// the problem the Newton solver is given, as tests/devsim's problem op runs it: every stage forward<nvp> runs up to the first
// direction solve (kinematics ... newton_begin, build_H), with HF and CX derived from nvp
template <bool HF, bool CX> static void problem_stages(const Ctx& c) {
  kinematics(c); com_quantities(c); mass_matrix(c);
  collision<HF, CX>(c);
  make_constraint<HF>(c);
  smooth_forces(c);
  newton_begin<HF>(c);
  build_H<HF>(c);
}

extern "C" {
void* hostsim_create(const void* blob, size_t n, const double* eq_data, const float* ref, int penv_body, int ngrp_cap) {
  HostSim* s = new HostSim;
  s->blob.assign((const uint8_t*)blob, (const uint8_t*)blob + n);
  if (b200_model_parse(s->blob.data(), n, &s->view) != 0) { delete s; return nullptr; }
  if (dm_build(s->view, eq_data, ref, s->model, s->err, penv_body, kWide, ngrp_cap) != 0) { fprintf(stderr, "hostsim: %s\n", s->err.c_str()); delete s; return nullptr; }
  const DMHead* h = (const DMHead*)s->model.data();
  s->scratch.assign(h->scr_words, 0.f);
  s->ctx.mg = s->model.data(); s->ctx.mw = s->model.data(); s->ctx.h = h; s->ctx.s = s->scratch.data(); s->ctx.lane = 0;
  return s;
}
void hostsim_destroy(void* p) { delete (HostSim*)p; }
float* hostsim_scratch(void* p) { return ((HostSim*)p)->scratch.data(); }
int hostsim_scr_words(void* p) { return ((HostSim*)p)->ctx.h->scr_words; }
int hostsim_npair(void* p) { return ((HostSim*)p)->ctx.h->npair; }
#ifdef B200_KITCHEN_GROUPS
int hostsim_nbgrp(void* p) { return ((HostSim*)p)->ctx.h->nbgrp; }
#endif
int hostsim_offset(void* p, const char* name) {
  const DMHead* h = ((HostSim*)p)->ctx.h;
#define X(nm, words) if (strcmp(name, #nm) == 0) return h->s_##nm;
  DM_SCRATCH_PERSIST(X)
#undef X
#define X(nm) if (strcmp(name, #nm) == 0) return h->s_##nm;
  DM_SCRATCH_UNION(X)
#undef X
  return -1;
}
void hostsim_forward(void* p) { warp_call(((HostSim*)p)->ctx, [](const Ctx& c) { forward<HOST_NVP>(c, true); }); }
void hostsim_step(void* p, int n) { warp_call(((HostSim*)p)->ctx, [n](const Ctx& c) { for (int i = 0; i < n; i++) { forward<HOST_NVP>(c, true); euler_step<HOST_NVP>(c); } }); }
void hostsim_kinematics(void* p) { warp_call(((HostSim*)p)->ctx, [](const Ctx& c) { kinematics(c); com_quantities(c); mass_matrix(c); }); }
// the collision stage alone, with HF and CX derived from nvp as forward<NVP> derives them (the broad phase reads the pair list of the
// kitchen groups build through ctx.mg, the whole model)
void hostsim_collide(void* p, int nvp) {
  const Ctx& base = ((HostSim*)p)->ctx;
  const bool hf = nvp >= 30, cx = nvp == 22 || nvp >= 30;
  if (hf) warp_call(base, [](const Ctx& c) { collision<true, true>(c); });
  else if (cx) warp_call(base, [](const Ctx& c) { collision<false, true>(c); });
  else warp_call(base, [](const Ctx& c) { collision<false, false>(c); });
}
void hostsim_problem(void* p, int nvp) {
  const Ctx& base = ((HostSim*)p)->ctx;
  const bool hf = nvp >= 30, cx = nvp == 22 || nvp >= 30;
  if (hf) warp_call(base, [](const Ctx& c) { problem_stages<true, true>(c); });
  else if (cx) warp_call(base, [](const Ctx& c) { problem_stages<false, true>(c); });
  else warp_call(base, [](const Ctx& c) { problem_stages<false, false>(c); });
}
// the rows' JV slots <- J search (rows_from_vec<HF>) on a scratch that hostsim_problem left
void hostsim_jv(void* p, int nvp) {
  const Ctx& base = ((HostSim*)p)->ctx;
  if (nvp >= 30) warp_call(base, [](const Ctx& c) { rows_from_vec<true>(c, SF(search)); });
  else warp_call(base, [](const Ctx& c) { rows_from_vec<false>(c, SF(search)); });
}
// build_H<HF> alone, on a scratch that hostsim_problem left
void hostsim_build_h(void* p, int nvp) {
  const Ctx& base = ((HostSim*)p)->ctx;
  if (nvp >= 30) warp_call(base, [](const Ctx& c) { build_H<true>(c); });
  else warp_call(base, [](const Ctx& c) { build_H<false>(c); });
}
// touch_observe with touch_mode 1 (the sensordata values) on a scratch that hostsim_problem left, its contact records possibly edited
// (tests/devsim STAGE_TOUCH): nsensor floats into out
void hostsim_touch(void* p, float* out) {
  FetchTask t;
  memset(&t, 0, sizeof(t));
  t.touch_mode = 1;
  warp_call(((HostSim*)p)->ctx, [&](const Ctx& c) { touch_observe(c, t, out); });
}
// ray_hits_site on n rays given in the site frame: p, d [n][3] -> hit [n] (the site-frame test touch_observe runs per contact)
void hostsim_ray_hits(int type, const float* size, int n, const float* p, const float* d, int* hit) {
  for (int i = 0; i < n; i++) hit[i] = ray_hits_site(type, size, p + 3 * i, d + 3 * i) ? 1 : 0;
}
int hostsim_model_offset(void* p, const char* name) {
  const DMHead* h = ((HostSim*)p)->ctx.h;
#define X(nm, w, kind) if (strcmp(name, #nm) == 0) return h->o_##nm;
  DM_ARRAYS(X)
#undef X
  return -1;
}
const uint32_t* hostsim_model(void* p) { return ((HostSim*)p)->model.data(); }
// this flavor's contact-record and group layout (dmodel.h): C_MU, C_U, C_DIMGRP, CON_WORDS, GRP_WORDS, G_RANGE, C_W, C_D, CX_POS, CX_PAIR,
// CX_WORDS
void hostsim_layout(int* out) {
  out[0] = C_MU; out[1] = C_U; out[2] = C_DIMGRP; out[3] = CON_WORDS; out[4] = GRP_WORDS; out[5] = G_RANGE;
  out[6] = C_W; out[7] = C_D; out[8] = CX_POS; out[9] = CX_PAIR; out[10] = CX_WORDS;
}
int hostsim_task_size() { return (int)sizeof(FetchTask); }
// one env's launch.  The kitchen flavors take `noise`, the env's observation-noise key as the step kernel builds it (NULL:
// noise-free); the ant flavor takes `a`, the Ant's keywords as b200sim_set_ant_info leaves them with rows / origin pointing at this
// env's info row [9] / reset position [2] (or NULL), and runs what fetch_kernel_ant's lane 0 runs after the step (ant_info).  Like
// fetch_env_step's, these parameters exist in those flavors only.
int hostsim_env_step(void* p, const FetchTask* t, int mode, int nraw, float* st, const float* action, float* obs, float* achieved,
                     float* desired, float* reward, float* success
#ifdef B200_KITCHEN
                     , const ObsNoiseKey* noise
#endif
#ifdef B200_ANT
                     , const AntInfoArgs* a
#endif
                     ) {
  int it = 0;
  warp_call(((HostSim*)p)->ctx, [&](const Ctx& c) {
#if defined(B200_KITCHEN)
    fetch_env_step<HOST_NVP>(c, *t, true, mode, nraw, st, action, obs, achieved, desired, reward, success, &it, noise);
#elif defined(B200_ANT)
    AntForces f = {a->cf_lo, a->cf_hi, 0.f};
    fetch_env_step<HOST_NVP>(c, *t, true, mode, nraw, st, action, obs, achieved, desired, reward, success, &it, &f);
    if (c.lane == 0)
      ant_info(c, *t, *a, mode, mode == MODE_STEP ? t->n_substeps > 0 : (mode == MODE_RAW && nraw > 0), st, action, f.sq, 0);
#else
    fetch_env_step<HOST_NVP>(c, *t, true, mode, nraw, st, action, obs, achieved, desired, reward, success, &it);
#endif
  });
  return it;
}
// x <- (A + hh diag(dadd))^-1 x with spd_solve<nvp> for an nv-dof system: A packed lower-triangular (nv (nv + 1) / 2 words), dadd
// optional, scratchH the solver's work area (the column buffers of the register Cholesky); A == scratchH is the Newton solve's
// in-place call.  Only the header's nv is read.  Returns -1 for an nvp this flavor does not instantiate.
int hostsim_spd(int nvp, int nv, const float* A, const float* dadd, float hh, float* x, float* scratchH) {
  DMHead head;
  memset(&head, 0, sizeof(head));
  head.nv = nv;
  Ctx base;
  memset(&base, 0, sizeof(base));
  base.h = &head;
  int ok = 0;
  auto run = [&](auto tag) {
    constexpr int V = decltype(tag)::value;
    ok = 1;
    warp_call(base, [&](const Ctx& c) { spd_solve<V>(c, A, dadd, hh, x, scratchH); });
  };
  switch (nvp) {
#if defined(B200_WIDE)
    case 36: run(std::integral_constant<int, 36>()); break;
#elif defined(B200_KITCHEN)
    case 31: run(std::integral_constant<int, 31>()); break;
#else
    case 14: run(std::integral_constant<int, 14>()); break;
    case 15: run(std::integral_constant<int, 15>()); break;
    case 21: run(std::integral_constant<int, 21>()); break;
    case 22: run(std::integral_constant<int, 22>()); break;
    case 30: run(std::integral_constant<int, 30>()); break;
    case 32: run(std::integral_constant<int, 32>()); break;
#endif
    default: break;
  }
  return ok ? 0 : -1;
}
}
// in-kernel reset sampling (csrc/reset_sample.cuh), the same code the CUDA reset kernel runs
#include "../../gymnasium_robotics_b200/csrc/reset_sample.cuh"
extern "C" void hostsim_philox4x32_10(const uint32_t* ctr, const uint32_t* key, uint32_t* out) { rs_philox4x32_10(ctr, key, out); }
extern "C" void hostsim_fetch_reset_record(const b200sim_fetch_reset_t* p, unsigned long long seed, unsigned env, unsigned episode, const float* rest,
                                           int stride, int st_qpos, int st_goal, float* rec) {
  rs_fetch_reset_record(*p, seed, env, episode, rest, stride, st_qpos, st_goal, rec);
}
extern "C" void hostsim_uniform_reset_record(const b200sim_uniform_reset_t* p, unsigned long long seed, unsigned env, unsigned episode, const float* rest,
                                             int stride, float* rec) {
  rs_uniform_reset_record(*p, seed, env, episode, rest, stride, rec);
}
extern "C" void hostsim_maze_reset_record(const b200sim_maze_reset_t* p, const float* goal_xy, const float* reset_xy, unsigned long long seed, unsigned env,
                                          unsigned episode, const float* rest, int stride, int st_qpos, int st_goal, float* rec) {
  rs_maze_reset_record(*p, goal_xy, reset_xy, seed, env, episode, rest, stride, st_qpos, st_goal, rec);
}
extern "C" void hostsim_hand_pose_record(const b200sim_hand_reset_t* p, const float* parallel, unsigned long long seed, unsigned env, unsigned episode,
                                         unsigned attempt, const float* rest, int stride, int st_qpos, int st_goal, int ngoal, float* rec) {
  rs_hand_pose_record(*p, parallel, seed, env, episode, attempt, rest, stride, st_qpos, st_goal, ngoal, rec);
}
extern "C" void hostsim_hand_goal(const b200sim_hand_reset_t* p, const float* parallel, unsigned long long seed, unsigned env, unsigned episode,
                                  int st_qpos, int st_goal, float* rec) {
  rs_hand_goal(*p, parallel, seed, env, episode, st_qpos, st_goal, rec);
}
extern "C" void hostsim_reach_reset_record(const b200sim_reach_reset_t* p, unsigned long long seed, unsigned env, unsigned episode, const float* rest,
                                           int stride, int st_goal, float* rec) {
  rs_reach_reset_record(*p, seed, env, episode, rest, stride, st_goal, rec);
}
// the maze goal update of b200sim_set_goal_update: goal [2] in/out; returns the number of candidates drawn (0: the goal stays)
extern "C" int hostsim_maze_goal_update(const float* goal_xy, int n_goal, float scaling, float noise, float radius, unsigned long long seed,
                                        unsigned env, unsigned episode, unsigned step, const float* ach, float* goal) {
  return rs_maze_goal_update(goal_xy, n_goal, scaling, noise, radius, seed, env, episode, step, ach, goal);
}
// AntMaze-v3's goal redraw of b200sim_set_goal_redraw: goal [2] in/out, reward out (written only when the goal changed); returns 1
// when the goal changed
extern "C" int hostsim_maze_goal_redraw(const float* goal_xy, int n_goal, float scaling, float noise, float radius, int dense,
                                        unsigned long long seed, unsigned env, unsigned episode, unsigned step, const float* ach, float* goal,
                                        float* reward) {
  return rs_maze_goal_redraw(goal_xy, n_goal, scaling, noise, radius, dense, seed, env, episode, step, ach, goal, reward);
}
#ifdef B200_KITCHEN
// the 59 uniforms in [-1, 1) of the stream (seed; env, episode, step t), entry j = word j % 4 of block j / 4 (rs_obs_noise_block):
// what the kitchen step kernel scales and adds
extern "C" void hostsim_kitchen_noise(unsigned long long seed, unsigned env, unsigned episode, unsigned t, float* out) {
  for (int b = 0; 4 * b < 59; b++) {
    float u[4];
    rs_obs_noise_block(seed, env, episode, t, (uint32_t)b, u);
    for (int w = 0; w < 4 && 4 * b + w < 59; w++) out[4 * b + w] = u[w];
  }
}
#endif
extern "C" int hostsim_check_record(float* rec, int stride, const float* rest, const b200sim_keep_t* keep) {
  b200sim_keep_t k;
  k.n = 0;
  if (keep) k = *keep;
  return rs_check_record(rec, stride, rest, k);
}
#ifdef B200_HOST_WARP
extern "C" long hostsim_collectives() { return g_hw.collectives; }   // scheduler rounds so far = warp collectives executed (2 per shuffle / ballot, 1 per __syncwarp)
#endif
extern "C" int hostsim_model_words(void* p) { return ((HostSim*)p)->ctx.h->nwords; }
extern "C" int hostsim_hot_words(void* p) { return ((HostSim*)p)->ctx.h->hot_words; }
