/* CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  Not part of the product path.
 *
 * A from-scratch fp64, single-env restatement of the documented `mj_step` pipeline that the reference
 * reaches through `mujoco.mj_step(model, data, nstep=n_substeps)` at
 * gymnasium_robotics/envs/robot_env.py:340-341 (and mj_forward at fetch_env.py:303,401).
 *
 * PARITY UNPINNED: the arithmetic of this path lives in the un-vendored `mujoco` wheel
 * (pyproject.toml:27 `mujoco>=2.2.0`), which is absent from this environment, and the reference's own
 * tests hold no post-step golden vectors (SURVEY.md section 8c).  This file restates the *published*
 * algorithm (MuJoCo "Computation" chapter; SURVEY.md Appendix B) and is validated against closed-form
 * physics in tests/test_oracle_physics.py.  Deviations from MuJoCo are listed in DESIGN.md.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may load it.
 *
 * Pipeline per sub-step (Appendix B numbering):
 *   1 kinematics  2 com/cdof  3 tendons  4 CRB mass matrix  5 collision  6 constraint rows
 *   7 smooth forces (passive, RNE bias, actuation)  8 Newton solver (pyramidal cones, exact line search)
 *   9 touch sensors  10 semi-implicit Euler with implicit joint damping (or RK4)
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200sim_model.h"

typedef double real;
#define MINVAL 1e-15
#define MAXCON 96
#define MAXEFC 640
#define MINIMP 0.0001
#define MAXIMP 0.9999

enum { ROW_EQ = 0, ROW_FRICTION = 1, ROW_LIMIT = 2, ROW_CONTACT = 3 };

typedef struct {
  real dist, pos[3], frame[9], includemargin, friction[5], solref[2], solimp[5];
  int dim, geom1, geom2, body1, body2, pair, efc_address;
} Contact;

typedef struct oracle_sim {
  void* blob;
  b200_model_view m;
  int nbody, nq, nv, nu, ngeom, nsite, nmocap;
  /* mutable model copies (the reference edits these after load) */
  real *eq_data, *act_gainprm, *act_biasprm, *body_pos, *body_quat, *jnt_range;
  /* state */
  real time;
  real *qpos, *qvel, *ctrl, *mocap_pos, *mocap_quat, *qacc_warmstart, *qacc;
  /* derived */
  real *xpos, *xquat, *xmat, *xipos, *ximat, *xanchor, *xaxis, *geom_xpos, *geom_xmat, *site_xpos, *site_xmat;
  real *subtree_com, *cinert, *crb, *cdof, *cdof_dot, *cvel, *cacc, *cfrc;
  real *M, *L; /* dense nv*nv */
  real *qfrc_bias, *qfrc_passive, *qfrc_actuator, *qfrc_smooth, *qacc_smooth, *qfrc_constraint, *actuator_force;
  real *ten_length, *ten_J;
  real *sensordata;
  /* contacts + constraint rows */
  int ncon, nefc;
  Contact con[MAXCON];
  real *J; /* MAXEFC * nv */
  real efc_pos[MAXEFC], efc_margin[MAXEFC], efc_D[MAXEFC], efc_R[MAXEFC], efc_aref[MAXEFC], efc_vel[MAXEFC],
      efc_force[MAXEFC], efc_floss[MAXEFC], efc_diagA[MAXEFC], efc_KBIP[MAXEFC][4];
  int efc_type[MAXEFC], efc_id[MAXEFC];
  /* solver stats */
  int solver_iter, warn_overflow, noslip_enabled, noslip_iter;
  long total_newton_iter, total_substeps;
  real solver_fwdinv;
} oracle_sim;

/* ------------------------------------------------------------------------------------------------ */
/* small vector helpers */
static inline real dot3(const real* a, const real* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static inline void cross3(real* r, const real* a, const real* b) {
  real x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
static inline void copy3(real* r, const real* a) { r[0] = a[0]; r[1] = a[1]; r[2] = a[2]; }
static inline void sub3(real* r, const real* a, const real* b) { r[0] = a[0] - b[0]; r[1] = a[1] - b[1]; r[2] = a[2] - b[2]; }
static inline void add3(real* r, const real* a, const real* b) { r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2]; }
static inline void addscl3(real* r, const real* a, real s) { r[0] += a[0] * s; r[1] += a[1] * s; r[2] += a[2] * s; }
static inline real norm3(const real* a) { return sqrt(dot3(a, a)); }
static inline real normalize3(real* a) {
  real n = norm3(a);
  if (n < MINVAL) { a[0] = 1; a[1] = 0; a[2] = 0; return 0; }
  a[0] /= n; a[1] /= n; a[2] /= n;
  return n;
}
static inline void mulmatvec3(real* r, const real* m, const real* v) { /* r = M v (row-major) */
  real x = m[0] * v[0] + m[1] * v[1] + m[2] * v[2], y = m[3] * v[0] + m[4] * v[1] + m[5] * v[2],
       z = m[6] * v[0] + m[7] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
static inline void mulmatTvec3(real* r, const real* m, const real* v) { /* r = M^T v */
  real x = m[0] * v[0] + m[3] * v[1] + m[6] * v[2], y = m[1] * v[0] + m[4] * v[1] + m[7] * v[2],
       z = m[2] * v[0] + m[5] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
static inline void mulquat(real* r, const real* a, const real* b) {
  real w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  real x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  real y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  real z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
static inline void normalize4(real* q) {
  real n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (n < MINVAL) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
static inline void quat2mat(real* m, const real* q) {
  real w = q[0], x = q[1], y = q[2], z = q[3];
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2 * (x * y - w * z); m[2] = 2 * (x * z + w * y);
  m[3] = 2 * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2 * (y * z - w * x);
  m[6] = 2 * (x * z - w * y); m[7] = 2 * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
static inline void rotvecquat(real* r, const real* v, const real* q) {
  real m[9];
  quat2mat(m, q);
  mulmatvec3(r, m, v);
}
static inline void axisangle2quat(real* q, const real* axis, real angle) {
  real s = sin(angle * 0.5);
  q[0] = cos(angle * 0.5); q[1] = axis[0] * s; q[2] = axis[1] * s; q[3] = axis[2] * s;
}
/* spatial vectors are [angular(3); linear(3)] about the kinematic-tree root's subtree com */
static inline void cross_motion(real* r, const real* v, const real* s) {
  real a[3], b[3], c[3];
  cross3(a, v, s);         /* w x s_ang */
  cross3(b, v, s + 3);     /* w x s_lin */
  cross3(c, v + 3, s);     /* v_lin x s_ang */
  r[0] = a[0]; r[1] = a[1]; r[2] = a[2];
  r[3] = b[0] + c[0]; r[4] = b[1] + c[1]; r[5] = b[2] + c[2];
}
static inline void cross_force(real* r, const real* v, const real* f) {
  real a[3], b[3], c[3];
  cross3(a, v, f);         /* w x f_ang */
  cross3(b, v + 3, f + 3); /* v_lin x f_lin */
  cross3(c, v, f + 3);     /* w x f_lin */
  r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2];
  r[3] = c[0]; r[4] = c[1]; r[5] = c[2];
}
/* 10-number spatial inertia: [Ixx Iyy Izz Ixy Ixz Iyz | m*r(3) | m], r = com offset from the reference point */
static inline void mul_inert_vec(real* res, const real* I, const real* v) {
  const real* mo = I + 6;
  real t[3];
  res[0] = I[0] * v[0] + I[3] * v[1] + I[4] * v[2];
  res[1] = I[3] * v[0] + I[1] * v[1] + I[5] * v[2];
  res[2] = I[4] * v[0] + I[5] * v[1] + I[2] * v[2];
  cross3(t, mo, v + 3); /* m r x v_lin */
  res[0] += t[0]; res[1] += t[1]; res[2] += t[2];
  cross3(t, v, mo);     /* w x m r */
  res[3] = I[9] * v[3] + t[0]; res[4] = I[9] * v[4] + t[1]; res[5] = I[9] * v[5] + t[2];
}

/* ------------------------------------------------------------------------------------------------ */
static real* dalloc(size_t n) { return (real*)calloc(n > 0 ? n : 1, sizeof(real)); }
static real* ddup(const double* src, size_t n) {
  real* p = dalloc(n);
  for (size_t i = 0; i < n; i++) p[i] = src[i];
  return p;
}

void oracle_reset_data(oracle_sim* s);

oracle_sim* oracle_create(const void* blob, size_t nbytes) {
  oracle_sim* s = (oracle_sim*)calloc(1, sizeof(oracle_sim));
  s->blob = malloc(nbytes);
  memcpy(s->blob, blob, nbytes);
  if (b200_model_parse(s->blob, nbytes, &s->m) != 0) { free(s->blob); free(s); return NULL; }
  const b200_model_view* m = &s->m;
  int nb = m->nbody, nv = m->nv, nq = m->nq;
  s->nbody = nb; s->nq = nq; s->nv = nv; s->nu = m->nu; s->ngeom = m->ngeom; s->nsite = m->nsite; s->nmocap = m->nmocap;
  s->eq_data = ddup(m->eq_data, (size_t)m->neq * 11);
  s->act_gainprm = ddup(m->act_gainprm, (size_t)m->nu * 3);
  s->act_biasprm = ddup(m->act_biasprm, (size_t)m->nu * 3);
  s->body_pos = ddup(m->body_pos, (size_t)nb * 3);
  s->jnt_range = ddup(m->jnt_range, (size_t)m->njnt * 2);
  s->body_quat = ddup(m->body_quat, (size_t)nb * 4);
  s->qpos = dalloc(nq); s->qvel = dalloc(nv); s->ctrl = dalloc(m->nu); s->mocap_pos = dalloc(3 * m->nmocap);
  s->mocap_quat = dalloc(4 * m->nmocap); s->qacc_warmstart = dalloc(nv); s->qacc = dalloc(nv);
  s->xpos = dalloc(3 * nb); s->xquat = dalloc(4 * nb); s->xmat = dalloc(9 * nb); s->xipos = dalloc(3 * nb);
  s->ximat = dalloc(9 * nb); s->xanchor = dalloc(3 * m->njnt); s->xaxis = dalloc(3 * m->njnt);
  s->geom_xpos = dalloc(3 * m->ngeom); s->geom_xmat = dalloc(9 * m->ngeom);
  s->site_xpos = dalloc(3 * m->nsite); s->site_xmat = dalloc(9 * m->nsite);
  s->subtree_com = dalloc(3 * nb); s->cinert = dalloc(10 * nb); s->crb = dalloc(10 * nb);
  s->cdof = dalloc(6 * nv); s->cdof_dot = dalloc(6 * nv); s->cvel = dalloc(6 * nb); s->cacc = dalloc(6 * nb); s->cfrc = dalloc(6 * nb);
  s->M = dalloc((size_t)nv * nv); s->L = dalloc((size_t)nv * nv);
  s->qfrc_bias = dalloc(nv); s->qfrc_passive = dalloc(nv); s->qfrc_actuator = dalloc(nv); s->qfrc_smooth = dalloc(nv);
  s->qacc_smooth = dalloc(nv); s->qfrc_constraint = dalloc(nv); s->actuator_force = dalloc(m->nu);
  s->ten_length = dalloc(m->ntendon); s->ten_J = dalloc((size_t)m->ntendon * nv);
  s->sensordata = dalloc(m->nsensor);
  s->J = dalloc((size_t)MAXEFC * nv);
  oracle_reset_data(s);
  s->noslip_enabled = 1;   /* honours <option noslip_iterations>; oracle_set_noslip(s, 0) switches the pass off */
  return s;
}

void oracle_destroy(oracle_sim* s) {
  if (!s) return;
  real* ptrs[] = {s->eq_data, s->act_gainprm, s->act_biasprm, s->body_pos, s->body_quat, s->jnt_range, s->qpos, s->qvel, s->ctrl, s->mocap_pos,
                  s->mocap_quat, s->qacc_warmstart, s->qacc, s->xpos, s->xquat, s->xmat, s->xipos, s->ximat, s->xanchor,
                  s->xaxis, s->geom_xpos, s->geom_xmat, s->site_xpos, s->site_xmat, s->subtree_com, s->cinert, s->crb,
                  s->cdof, s->cdof_dot, s->cvel, s->cacc, s->cfrc, s->M, s->L, s->qfrc_bias, s->qfrc_passive,
                  s->qfrc_actuator, s->qfrc_smooth, s->qacc_smooth, s->qfrc_constraint, s->actuator_force, s->ten_length,
                  s->ten_J, s->sensordata, s->J};
  for (size_t i = 0; i < sizeof(ptrs) / sizeof(ptrs[0]); i++) free(ptrs[i]);
  free(s->blob);
  free(s);
}

/* mj_resetData: qpos = qpos0, everything else zero, mocap pose from the model body pose */
void oracle_reset_data(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  for (int i = 0; i < s->nq; i++) s->qpos[i] = m->qpos0[i];
  memset(s->qvel, 0, sizeof(real) * s->nv);
  memset(s->qacc, 0, sizeof(real) * s->nv);
  memset(s->qacc_warmstart, 0, sizeof(real) * s->nv);
  memset(s->ctrl, 0, sizeof(real) * s->nu);
  for (int i = 0; i < m->nmocap; i++) {
    int b = m->mocap_body[i];
    for (int k = 0; k < 3; k++) s->mocap_pos[3 * i + k] = s->body_pos[3 * b + k];
    for (int k = 0; k < 4; k++) s->mocap_quat[4 * i + k] = m->body_quat[4 * b + k];
  }
  s->time = 0;
  s->ncon = 0; s->nefc = 0;
}

/* ------------------------------------------------------------------------------------------------ */
/* 1. kinematics */
static void kinematics(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  s->xpos[0] = s->xpos[1] = s->xpos[2] = 0;
  s->xquat[0] = 1; s->xquat[1] = s->xquat[2] = s->xquat[3] = 0;
  quat2mat(s->xmat, s->xquat);
  for (int b = 1; b < s->nbody; b++) {
    real *xp = s->xpos + 3 * b, *xq = s->xquat + 4 * b;
    int p = m->body_parent[b], jn = m->body_jntnum[b], ja = m->body_jntadr[b];
    if (m->body_mocapid[b] >= 0) {
      int id = m->body_mocapid[b];
      copy3(xp, s->mocap_pos + 3 * id);
      memcpy(xq, s->mocap_quat + 4 * id, 4 * sizeof(real));
      normalize4(xq);
    } else if (jn == 1 && m->jnt_type[ja] == B200_JNT_FREE) {
      int a = m->jnt_qposadr[ja];
      copy3(xp, s->qpos + a);
      memcpy(xq, s->qpos + a + 3, 4 * sizeof(real));
      normalize4(xq);
      copy3(s->xanchor + 3 * ja, xp);
      s->xaxis[3 * ja] = 0; s->xaxis[3 * ja + 1] = 0; s->xaxis[3 * ja + 2] = 1;
    } else {
      real t[3];
      mulmatvec3(t, s->xmat + 9 * p, s->body_pos + 3 * b);
      add3(xp, s->xpos + 3 * p, t);
      real bq[4] = {s->body_quat[4 * b], s->body_quat[4 * b + 1], s->body_quat[4 * b + 2], s->body_quat[4 * b + 3]};
      mulquat(xq, s->xquat + 4 * p, bq);
      for (int j = ja; j < ja + jn; j++) {
        real jp[3] = {m->jnt_pos[3 * j], m->jnt_pos[3 * j + 1], m->jnt_pos[3 * j + 2]};
        real jax[3] = {m->jnt_axis[3 * j], m->jnt_axis[3 * j + 1], m->jnt_axis[3 * j + 2]};
        real *anc = s->xanchor + 3 * j, *ax = s->xaxis + 3 * j;
        rotvecquat(t, jp, xq); add3(anc, xp, t);
        rotvecquat(ax, jax, xq);
        real dq = s->qpos[m->jnt_qposadr[j]] - m->qpos0[m->jnt_qposadr[j]];
        if (m->jnt_type[j] == B200_JNT_SLIDE) {
          addscl3(xp, ax, dq);
        } else if (m->jnt_type[j] == B200_JNT_HINGE) {
          real ql[4], nq[4];
          axisangle2quat(ql, jax, dq);
          mulquat(nq, xq, ql);
          memcpy(xq, nq, sizeof(nq));
          rotvecquat(t, jp, xq);
          sub3(xp, anc, t);
        }
      }
      normalize4(xq);
    }
    quat2mat(s->xmat + 9 * b, xq);
    real t[3], iq[4], bi[4] = {m->body_iquat[4 * b], m->body_iquat[4 * b + 1], m->body_iquat[4 * b + 2], m->body_iquat[4 * b + 3]};
    real ip[3] = {m->body_ipos[3 * b], m->body_ipos[3 * b + 1], m->body_ipos[3 * b + 2]};
    mulmatvec3(t, s->xmat + 9 * b, ip); add3(s->xipos + 3 * b, xp, t);
    mulquat(iq, xq, bi); quat2mat(s->ximat + 9 * b, iq);
  }
  copy3(s->xipos, s->xpos); quat2mat(s->ximat, s->xquat);
  for (int g = 0; g < s->ngeom; g++) {
    int b = m->geom_body[g];
    real t[3], gq[4], q[4] = {m->geom_quat[4 * g], m->geom_quat[4 * g + 1], m->geom_quat[4 * g + 2], m->geom_quat[4 * g + 3]};
    real gp[3] = {m->geom_pos[3 * g], m->geom_pos[3 * g + 1], m->geom_pos[3 * g + 2]};
    mulmatvec3(t, s->xmat + 9 * b, gp); add3(s->geom_xpos + 3 * g, s->xpos + 3 * b, t);
    mulquat(gq, s->xquat + 4 * b, q); quat2mat(s->geom_xmat + 9 * g, gq);
  }
  for (int i = 0; i < s->nsite; i++) {
    int b = m->site_body[i];
    real t[3], gq[4], q[4] = {m->site_quat[4 * i], m->site_quat[4 * i + 1], m->site_quat[4 * i + 2], m->site_quat[4 * i + 3]};
    real gp[3] = {m->site_pos[3 * i], m->site_pos[3 * i + 1], m->site_pos[3 * i + 2]};
    mulmatvec3(t, s->xmat + 9 * b, gp); add3(s->site_xpos + 3 * i, s->xpos + 3 * b, t);
    mulquat(gq, s->xquat + 4 * b, q); quat2mat(s->site_xmat + 9 * i, gq);
  }
}

/* 2. com-based quantities */
static void com_pos(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  int nb = s->nbody;
  real* mass_sub = dalloc(nb);
  for (int b = 0; b < nb; b++) {
    mass_sub[b] = m->body_mass[b];
    for (int k = 0; k < 3; k++) s->subtree_com[3 * b + k] = m->body_mass[b] * s->xipos[3 * b + k];
  }
  for (int b = nb - 1; b > 0; b--) {
    int p = m->body_parent[b];
    mass_sub[p] += mass_sub[b];
    for (int k = 0; k < 3; k++) s->subtree_com[3 * p + k] += s->subtree_com[3 * b + k];
  }
  for (int b = 0; b < nb; b++) {
    if (mass_sub[b] < MINVAL) copy3(s->subtree_com + 3 * b, s->xipos + 3 * b);
    else for (int k = 0; k < 3; k++) s->subtree_com[3 * b + k] /= mass_sub[b];
  }
  free(mass_sub);
  for (int b = 1; b < nb; b++) {
    const real* c = s->subtree_com + 3 * m->body_rootid[b];
    real r[3];
    sub3(r, s->xipos + 3 * b, c);
    real mass = m->body_mass[b];
    const real* R = s->ximat + 9 * b;
    real d[3] = {m->body_inertia[3 * b], m->body_inertia[3 * b + 1], m->body_inertia[3 * b + 2]};
    real I[9];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) I[3 * i + j] = R[3 * i] * d[0] * R[3 * j] + R[3 * i + 1] * d[1] * R[3 * j + 1] + R[3 * i + 2] * d[2] * R[3 * j + 2];
    real rr = dot3(r, r);
    real* ci = s->cinert + 10 * b;
    ci[0] = I[0] + mass * (rr - r[0] * r[0]); ci[1] = I[4] + mass * (rr - r[1] * r[1]); ci[2] = I[8] + mass * (rr - r[2] * r[2]);
    ci[3] = I[1] - mass * r[0] * r[1]; ci[4] = I[2] - mass * r[0] * r[2]; ci[5] = I[5] - mass * r[1] * r[2];
    ci[6] = mass * r[0]; ci[7] = mass * r[1]; ci[8] = mass * r[2]; ci[9] = mass;
  }
  memset(s->cinert, 0, 10 * sizeof(real));
  for (int j = 0; j < m->njnt; j++) {
    int b = m->jnt_body[j], d = m->jnt_dofadr[j];
    const real* c = s->subtree_com + 3 * m->body_rootid[b];
    real off[3];
    sub3(off, c, s->xanchor + 3 * j);
    if (m->jnt_type[j] == B200_JNT_FREE) {
      memset(s->cdof + 6 * d, 0, 36 * sizeof(real));
      for (int k = 0; k < 3; k++) s->cdof[6 * (d + k) + 3 + k] = 1;
      for (int k = 0; k < 3; k++) {
        real ax[3] = {s->xmat[9 * b + k], s->xmat[9 * b + 3 + k], s->xmat[9 * b + 6 + k]};
        copy3(s->cdof + 6 * (d + 3 + k), ax);
        cross3(s->cdof + 6 * (d + 3 + k) + 3, ax, off);
      }
    } else if (m->jnt_type[j] == B200_JNT_SLIDE) {
      memset(s->cdof + 6 * d, 0, 3 * sizeof(real));
      copy3(s->cdof + 6 * d + 3, s->xaxis + 3 * j);
    } else {
      copy3(s->cdof + 6 * d, s->xaxis + 3 * j);
      cross3(s->cdof + 6 * d + 3, s->xaxis + 3 * j, off);
    }
  }
}

/* 3. fixed tendons */
static void tendons(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  int nv = s->nv;
  memset(s->ten_J, 0, sizeof(real) * m->ntendon * nv);
  for (int t = 0; t < m->ntendon; t++) {
    real len = 0;
    for (int w = m->ten_adr[t]; w < m->ten_adr[t] + m->ten_num[t]; w++) {
      int d = m->wrap_dof[w];
      int j = m->dof_jnt[d];
      len += m->wrap_coef[w] * s->qpos[m->jnt_qposadr[j]];
      s->ten_J[t * nv + d] += m->wrap_coef[w];
    }
    s->ten_length[t] = len;
  }
}

/* 4. composite rigid body -> dense M */
static void crb(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  int nv = s->nv, nb = s->nbody;
  memcpy(s->crb, s->cinert, sizeof(real) * 10 * nb);
  for (int b = nb - 1; b > 0; b--) {
    int p = m->body_parent[b];
    if (p > 0) for (int k = 0; k < 10; k++) s->crb[10 * p + k] += s->crb[10 * b + k];
  }
  memset(s->M, 0, sizeof(real) * nv * nv);
  for (int i = 0; i < nv; i++) {
    real buf[6];
    mul_inert_vec(buf, s->crb + 10 * m->dof_body[i], s->cdof + 6 * i);
    for (int j = i; j >= 0; j = m->dof_parent[j]) {
      real v = 0;
      for (int k = 0; k < 6; k++) v += s->cdof[6 * j + k] * buf[k];
      s->M[i * nv + j] = s->M[j * nv + i] = v;
    }
    s->M[i * nv + i] += m->dof_armature[i];
  }
}

/* dense Cholesky A = L L^T (lower), returns 0 on success */
static int cholesky(real* L, const real* A, int n) {
  for (int i = 0; i < n; i++) {
    for (int j = 0; j <= i; j++) {
      real sum = A[i * n + j];
      for (int k = 0; k < j; k++) sum -= L[i * n + k] * L[j * n + k];
      if (i == j) {
        if (sum < MINVAL) sum = MINVAL;
        L[i * n + i] = sqrt(sum);
      } else L[i * n + j] = sum / L[j * n + j];
    }
    for (int j = i + 1; j < n; j++) L[i * n + j] = 0;
  }
  return 0;
}
static void chol_solve(real* x, const real* L, const real* b, int n) {
  for (int i = 0; i < n; i++) {
    real sum = b[i];
    for (int k = 0; k < i; k++) sum -= L[i * n + k] * x[k];
    x[i] = sum / L[i * n + i];
  }
  for (int i = n - 1; i >= 0; i--) {
    real sum = x[i];
    for (int k = i + 1; k < n; k++) sum -= L[k * n + i] * x[k];
    x[i] = sum / L[i * n + i];
  }
}

/* ------------------------------------------------------------------------------------------------ */
/* Jacobians via cdof: point velocity = lin + ang x (p - com_root) */
static void jac_point(const oracle_sim* s, int body, const real* point, real* jacp, real* jacr) {
  const b200_model_view* m = &s->m;
  int nv = s->nv;
  if (jacp) memset(jacp, 0, sizeof(real) * 3 * nv);
  if (jacr) memset(jacr, 0, sizeof(real) * 3 * nv);
  if (body <= 0) return;
  real off[3];
  sub3(off, point, s->subtree_com + 3 * m->body_rootid[body]);
  /* last dof of the body or of its nearest ancestor with dofs */
  int b = body;
  while (b > 0 && m->body_dofnum[b] == 0) b = m->body_parent[b];
  if (b <= 0) return;
  for (int d = m->body_dofadr[b] + m->body_dofnum[b] - 1; d >= 0; d = m->dof_parent[d]) {
    const real* c = s->cdof + 6 * d;
    if (jacr) { jacr[d] = c[0]; jacr[nv + d] = c[1]; jacr[2 * nv + d] = c[2]; }
    if (jacp) {
      real t[3];
      cross3(t, c, off);
      jacp[d] = c[3] + t[0]; jacp[nv + d] = c[4] + t[1]; jacp[2 * nv + d] = c[5] + t[2];
    }
  }
}

void oracle_jac_site(const oracle_sim* s, int site, real* jacp, real* jacr) {
  jac_point(s, s->m.site_body[site], s->site_xpos + 3 * site, jacp, jacr);
}

/* ------------------------------------------------------------------------------------------------ */
/* 5. collision */
static void make_frame(real* f) { /* f[0:3] = normal given; build two tangents */
  normalize3(f);
  real* y = f + 3;
  y[0] = y[1] = y[2] = 0;
  if (f[1] < 0.5 && f[1] > -0.5) y[1] = 1; else y[2] = 1;
  real d = dot3(f, y);
  addscl3(y, f, -d);
  normalize3(y);
  cross3(f + 6, f, y);
}

static Contact* add_contact(oracle_sim* s, int pair, real dist, const real* pos, const real* normal) {
  const b200_model_view* m = &s->m;
  if (s->ncon >= MAXCON) { s->warn_overflow++; return NULL; }
  Contact* c = &s->con[s->ncon++];
  memset(c, 0, sizeof(*c));
  c->dist = dist; copy3(c->pos, pos); copy3(c->frame, normal);
  make_frame(c->frame);
  c->pair = pair; c->geom1 = m->pair_geom1[pair]; c->geom2 = m->pair_geom2[pair];
  c->body1 = m->geom_body[c->geom1]; c->body2 = m->geom_body[c->geom2];
  c->dim = m->pair_condim[pair];
  c->includemargin = m->pair_margin[pair] - m->pair_gap[pair];
  for (int k = 0; k < 5; k++) { c->friction[k] = m->pair_friction[5 * pair + k]; c->solimp[k] = m->pair_solimp[5 * pair + k]; }
  c->solref[0] = m->pair_solref[2 * pair]; c->solref[1] = m->pair_solref[2 * pair + 1];
  return c;
}

/* plane (geom1) vs box (geom2): up to 4 corners below plane+margin */
static void collide_plane_box(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *pp = s->geom_xpos + 3 * g1, *pm = s->geom_xmat + 9 * g1, *bp = s->geom_xpos + 3 * g2, *bm = s->geom_xmat + 9 * g2;
  const double* sz = m->geom_size + 3 * g2;
  real n[3] = {pm[2], pm[5], pm[8]}, dif[3];
  sub3(dif, bp, pp);
  real dist0 = dot3(dif, n);
  int cnt = 0;
  for (int i = 0; i < 8 && cnt < 4; i++) {
    real loc[3] = {(i & 1 ? sz[0] : -sz[0]), (i & 2 ? sz[1] : -sz[1]), (i & 4 ? sz[2] : -sz[2])}, vec[3];
    mulmatvec3(vec, bm, loc);
    real ldist = dot3(n, vec);
    if (dist0 + ldist > margin || ldist > 0) continue;
    real d = dist0 + ldist, pos[3];
    add3(pos, bp, vec);
    addscl3(pos, n, -d * 0.5);
    add_contact(s, pair, d, pos, n);
    cnt++;
  }
}

/* plane vs sphere / capsule */
static void collide_plane_sphere(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *pp = s->geom_xpos + 3 * g1, *pm = s->geom_xmat + 9 * g1, *c = s->geom_xpos + 3 * g2;
  real n[3] = {pm[2], pm[5], pm[8]}, dif[3];
  sub3(dif, c, pp);
  real r = m->geom_size[3 * g2], d = dot3(dif, n) - r;
  if (d > margin) return;
  real pos[3];
  copy3(pos, c);
  addscl3(pos, n, -r - d * 0.5);
  add_contact(s, pair, d, pos, n);
}
static void collide_plane_capsule(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *pp = s->geom_xpos + 3 * g1, *pm = s->geom_xmat + 9 * g1, *c = s->geom_xpos + 3 * g2, *cm = s->geom_xmat + 9 * g2;
  real n[3] = {pm[2], pm[5], pm[8]}, ax[3] = {cm[2], cm[5], cm[8]};
  real r = m->geom_size[3 * g2], h = m->geom_size[3 * g2 + 1];
  for (int side = -1; side <= 1; side += 2) {
    real e[3], dif[3];
    copy3(e, c);
    addscl3(e, ax, side * h);
    sub3(dif, e, pp);
    real d = dot3(dif, n) - r;
    if (d > margin) continue;
    real pos[3];
    copy3(pos, e);
    addscl3(pos, n, -r - d * 0.5);
    add_contact(s, pair, d, pos, n);
  }
}

/* ---- box-box: separating-axis test + reference-face clipping (own formulation; <= 4 contacts per pair) */
typedef struct { real p[3]; real d; } ClipPt;

static int clip_poly(real (*in)[2], int n, real (*out)[2], int axis, real bound, int sign) {
  /* keep points with sign*coord <= bound, 2-D Sutherland-Hodgman against one edge of the reference rectangle */
  int k = 0;
  for (int i = 0; i < n; i++) {
    real* a = in[i];
    real* b = in[(i + 1) % n];
    real da = sign * a[axis] - bound, db = sign * b[axis] - bound;
    if (da <= 0) { out[k][0] = a[0]; out[k][1] = a[1]; k++; }
    if ((da < 0 && db > 0) || (da > 0 && db < 0)) {
      real t = da / (da - db);
      out[k][0] = a[0] + t * (b[0] - a[0]); out[k][1] = a[1] + t * (b[1] - a[1]); k++;
    }
  }
  return k;
}

static void collide_box_box(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *pa = s->geom_xpos + 3 * g1, *Ra = s->geom_xmat + 9 * g1, *pb = s->geom_xpos + 3 * g2, *Rb = s->geom_xmat + 9 * g2;
  real ha[3] = {m->geom_size[3 * g1], m->geom_size[3 * g1 + 1], m->geom_size[3 * g1 + 2]};
  real hb[3] = {m->geom_size[3 * g2], m->geom_size[3 * g2 + 1], m->geom_size[3 * g2 + 2]};
  real d[3], da[3], db[3];
  sub3(d, pb, pa);
  mulmatTvec3(da, Ra, d); /* centre offset in A's frame */
  mulmatTvec3(db, Rb, d);
  /* C[i][j] = a_i . b_j */
  real C[3][3], Q[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      C[i][j] = Ra[i] * Rb[j] + Ra[3 + i] * Rb[3 + j] + Ra[6 + i] * Rb[6 + j];
      Q[i][j] = fabs(C[i][j]);
    }
  /* face axes */
  real best = -1e300; int code = -1; real bestsign = 1;
  for (int i = 0; i < 3; i++) {
    real sep = fabs(da[i]) - (ha[i] + hb[0] * Q[i][0] + hb[1] * Q[i][1] + hb[2] * Q[i][2]);
    if (sep > margin) return;
    if (sep > best) { best = sep; code = i; bestsign = da[i] < 0 ? -1 : 1; }
  }
  for (int j = 0; j < 3; j++) {
    real sep = fabs(db[j]) - (hb[j] + ha[0] * Q[0][j] + ha[1] * Q[1][j] + ha[2] * Q[2][j]);
    if (sep > margin) return;
    if (sep > best) { best = sep; code = 3 + j; bestsign = db[j] < 0 ? -1 : 1; }
  }
  /* edge axes a_i x b_j (normalised); an edge axis wins only if clearly better than the best face axis */
  real ebest = -1e300; int ecode = -1; real eaxis[3] = {0, 0, 0};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      real ai[3] = {Ra[i], Ra[3 + i], Ra[6 + i]}, bj[3] = {Rb[j], Rb[3 + j], Rb[6 + j]}, ax[3];
      cross3(ax, ai, bj);
      real l = norm3(ax);
      if (l < 1e-6) continue;
      ax[0] /= l; ax[1] /= l; ax[2] /= l;
      real ra = 0, rb = 0;
      for (int k = 0; k < 3; k++) {
        real ak[3] = {Ra[k], Ra[3 + k], Ra[6 + k]}, bk[3] = {Rb[k], Rb[3 + k], Rb[6 + k]};
        ra += ha[k] * fabs(dot3(ak, ax));
        rb += hb[k] * fabs(dot3(bk, ax));
      }
      real dd = dot3(d, ax);
      real sep = fabs(dd) - (ra + rb);
      if (sep > margin) return;
      if (sep > ebest) { ebest = sep; ecode = 3 * i + j; copy3(eaxis, ax); if (dd < 0) { eaxis[0] = -ax[0]; eaxis[1] = -ax[1]; eaxis[2] = -ax[2]; } }
    }
  if (ecode >= 0 && ebest > best + 1e-3 * (fabs(best) + 1e-3) && ebest > 0.95 * best + 0.0 && ebest > best) {
    /* edge-edge: closest points between the supporting edges */
    int i = ecode / 3, j = ecode % 3;
    real n[3];
    copy3(n, eaxis); /* from A to B */
    real ea[3] = {Ra[i], Ra[3 + i], Ra[6 + i]}, eb[3] = {Rb[j], Rb[3 + j], Rb[6 + j]};
    /* point on A's edge: centre + sum over k != i of sign(n.a_k) ha_k a_k ; on B's: centre - sign(n.b_k) hb_k b_k */
    real PA[3], PB[3];
    copy3(PA, pa); copy3(PB, pb);
    for (int k = 0; k < 3; k++) {
      real ak[3] = {Ra[k], Ra[3 + k], Ra[6 + k]}, bk[3] = {Rb[k], Rb[3 + k], Rb[6 + k]};
      if (k != i) addscl3(PA, ak, (dot3(n, ak) > 0 ? 1 : -1) * ha[k]);
      if (k != j) addscl3(PB, bk, (dot3(n, bk) > 0 ? -1 : 1) * hb[k]);
    }
    /* closest points of the two lines PA + s ea, PB + t eb */
    real w[3];
    sub3(w, PA, PB);
    real a = 1, b = dot3(ea, eb), c = 1, dd = dot3(ea, w), e = dot3(eb, w), den = a * c - b * b;
    real sp = den > 1e-12 ? (b * e - c * dd) / den : 0, tp = den > 1e-12 ? (a * e - b * dd) / den : 0;
    if (sp > ha[i]) sp = ha[i]; if (sp < -ha[i]) sp = -ha[i];
    if (tp > hb[j]) tp = hb[j]; if (tp < -hb[j]) tp = -hb[j];
    real qa[3], qb[3], pos[3];
    copy3(qa, PA); addscl3(qa, ea, sp);
    copy3(qb, PB); addscl3(qb, eb, tp);
    pos[0] = 0.5 * (qa[0] + qb[0]); pos[1] = 0.5 * (qa[1] + qb[1]); pos[2] = 0.5 * (qa[2] + qb[2]);
    add_contact(s, pair, ebest, pos, n);
    return;
  }
  /* face contact.  Reference box = the one owning the best axis; incident = the other. */
  const real *pr, *Rr, *pi, *Ri; real hr[3], hi[3]; int ax; real sgn; int flip;
  if (code < 3) { pr = pa; Rr = Ra; pi = pb; Ri = Rb; copy3(hr, ha); copy3(hi, hb); ax = code; sgn = bestsign; flip = 0; }
  else { pr = pb; Rr = Rb; pi = pa; Ri = Ra; copy3(hr, hb); copy3(hi, ha); ax = code - 3; sgn = -bestsign; flip = 1; }
  /* reference face normal (world), pointing from the reference box toward the incident box */
  real nr[3] = {Rr[ax] * sgn, Rr[3 + ax] * sgn, Rr[6 + ax] * sgn};
  /* incident face: the face of the incident box most anti-parallel to nr */
  int iax = 0; real bestd = -1;
  real nloc[3];
  mulmatTvec3(nloc, Ri, nr);
  for (int k = 0; k < 3; k++) if (fabs(nloc[k]) > bestd) { bestd = fabs(nloc[k]); iax = k; }
  real isgn = nloc[iax] > 0 ? -1 : 1;
  int u = (iax + 1) % 3, v = (iax + 2) % 3;
  /* incident face vertices in world, then in the reference face's 2-D frame */
  int ru = (ax + 1) % 3, rv = (ax + 2) % 3;
  real poly[8][2], tmp[8][2], depth_c[4][3];
  real au[3] = {Rr[ru], Rr[3 + ru], Rr[6 + ru]}, av[3] = {Rr[rv], Rr[3 + rv], Rr[6 + rv]};
  real fc[3]; /* incident face centre */
  copy3(fc, pi);
  { real t[3] = {Ri[iax], Ri[3 + iax], Ri[6 + iax]}; addscl3(fc, t, isgn * hi[iax]); }
  real iu[3] = {Ri[u], Ri[3 + u], Ri[6 + u]}, iv[3] = {Ri[v], Ri[3 + v], Ri[6 + v]};
  static const int su[4] = {1, -1, -1, 1}, sv[4] = {1, 1, -1, -1};
  for (int k = 0; k < 4; k++) {
    real p[3], rel[3];
    copy3(p, fc); addscl3(p, iu, su[k] * hi[u]); addscl3(p, iv, sv[k] * hi[v]);
    sub3(rel, p, pr);
    poly[k][0] = dot3(rel, au); poly[k][1] = dot3(rel, av);
    copy3(depth_c[k], p);
  }
  /* plane of the incident face in reference coords: height(x,y) is affine -> evaluate from 3 vertices */
  real h0, hx, hy;
  {
    real r0[3], r1[3], r3[3];
    sub3(r0, depth_c[0], pr); sub3(r1, depth_c[1], pr); sub3(r3, depth_c[3], pr);
    real z0 = dot3(r0, nr) - hr[ax], z1 = dot3(r1, nr) - hr[ax], z3 = dot3(r3, nr) - hr[ax];
    /* solve z = h0 + hx*x + hy*y through vertices 0,1,3 */
    real x0 = poly[0][0], y0 = poly[0][1], x1 = poly[1][0], y1 = poly[1][1], x3 = poly[3][0], y3 = poly[3][1];
    real det = (x1 - x0) * (y3 - y0) - (x3 - x0) * (y1 - y0);
    if (fabs(det) < 1e-14) { hx = hy = 0; h0 = z0; }
    else {
      hx = ((z1 - z0) * (y3 - y0) - (z3 - z0) * (y1 - y0)) / det;
      hy = ((x1 - x0) * (z3 - z0) - (x3 - x0) * (z1 - z0)) / det;
      h0 = z0 - hx * x0 - hy * y0;
    }
  }
  int n = 4;
  n = clip_poly(poly, n, tmp, 0, hr[ru], 1);
  n = clip_poly(tmp, n, poly, 0, hr[ru], -1);
  n = clip_poly(poly, n, tmp, 1, hr[rv], 1);
  n = clip_poly(tmp, n, poly, 1, hr[rv], -1);
  /* candidates */
  real cand[8][4]; int nc = 0;
  for (int k = 0; k < n && k < 8; k++) {
    real z = h0 + hx * poly[k][0] + hy * poly[k][1];
    if (z > margin) continue;
    cand[nc][0] = poly[k][0]; cand[nc][1] = poly[k][1]; cand[nc][2] = z; cand[nc][3] = 0; nc++;
  }
  if (nc == 0) return;
  /* reduce to <= 4: deepest, farthest from it, farthest from that line, farthest on the other side */
  int sel[4], ns = 0;
  if (nc <= 4) { for (int k = 0; k < nc; k++) sel[ns++] = k; }
  else {
    int i0 = 0;
    for (int k = 1; k < nc; k++) if (cand[k][2] < cand[i0][2]) i0 = k;
    int i1 = -1; real bd = -1;
    for (int k = 0; k < nc; k++) { real dx = cand[k][0] - cand[i0][0], dy = cand[k][1] - cand[i0][1], q = dx * dx + dy * dy; if (k != i0 && q > bd) { bd = q; i1 = k; } }
    real ex = cand[i1][0] - cand[i0][0], ey = cand[i1][1] - cand[i0][1];
    int i2 = -1, i3 = -1; real bp = 0, bn = 0;
    for (int k = 0; k < nc; k++) {
      if (k == i0 || k == i1) continue;
      real cr = ex * (cand[k][1] - cand[i0][1]) - ey * (cand[k][0] - cand[i0][0]);
      if (cr > bp) { bp = cr; i2 = k; }
      if (cr < bn) { bn = cr; i3 = k; }
    }
    sel[ns++] = i0; sel[ns++] = i1;
    if (i2 >= 0) sel[ns++] = i2;
    if (i3 >= 0) sel[ns++] = i3;
    /* keep a deterministic order: ascending candidate index */
    for (int a = 0; a < ns; a++) for (int b = a + 1; b < ns; b++) if (sel[b] < sel[a]) { int t = sel[a]; sel[a] = sel[b]; sel[b] = t; }
  }
  real nout[3] = {flip ? -nr[0] : nr[0], flip ? -nr[1] : nr[1], flip ? -nr[2] : nr[2]}; /* geom1 -> geom2 */
  for (int k = 0; k < ns; k++) {
    real* c = cand[sel[k]];
    real pos[3];
    copy3(pos, pr);
    addscl3(pos, au, c[0]); addscl3(pos, av, c[1]);
    addscl3(pos, nr, hr[ax] + 0.5 * c[2]); /* midway between the reference face and the incident point */
    add_contact(s, pair, c[2], pos, nout);
  }
}

/* ---- sphere / capsule vs box (own formulation): closest point on the box to a point, in the box frame */
static real point_box(const real* p, const real* bp, const real* bm, const double* h, real* closest, real* normal) {
  /* returns signed distance from p to the box surface; normal points from the box surface towards p */
  real rel[3], loc[3], q[3];
  sub3(rel, p, bp);
  mulmatTvec3(loc, bm, rel);
  int inside = 1;
  for (int k = 0; k < 3; k++) { q[k] = loc[k] < -h[k] ? -h[k] : (loc[k] > h[k] ? h[k] : loc[k]); if (q[k] != loc[k]) inside = 0; }
  real nl[3] = {0, 0, 0}, dist;
  if (!inside) {
    real d[3] = {loc[0] - q[0], loc[1] - q[1], loc[2] - q[2]};
    dist = norm3(d);
    nl[0] = d[0] / dist; nl[1] = d[1] / dist; nl[2] = d[2] / dist;
  } else {
    int ax = 0; real best = 1e300;
    for (int k = 0; k < 3; k++) { real pen = h[k] - fabs(loc[k]); if (pen < best) { best = pen; ax = k; } }
    dist = -best;
    nl[ax] = loc[ax] < 0 ? -1 : 1;
    q[ax] = nl[ax] * h[ax];
  }
  mulmatvec3(closest, bm, q); add3(closest, closest, bp);
  mulmatvec3(normal, bm, nl);
  return dist;
}

static void sphere_box_contact(oracle_sim* s, int pair, const real* center, real r, int gbox, real margin) {
  const b200_model_view* m = &s->m;
  real closest[3], nrm[3];
  real d = point_box(center, s->geom_xpos + 3 * gbox, s->geom_xmat + 9 * gbox, m->geom_size + 3 * gbox, closest, nrm) - r;
  if (d > margin) return;
  /* contact normal from geom1 (sphere/capsule) to geom2 (box) = -nrm ; position midway between the two surfaces */
  real n[3] = {-nrm[0], -nrm[1], -nrm[2]}, pos[3];
  copy3(pos, closest);
  addscl3(pos, nrm, 0.5 * d);
  add_contact(s, pair, d, pos, n);
}

static void collide_sphere_box(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  sphere_box_contact(s, pair, s->geom_xpos + 3 * g1, m->geom_size[3 * g1], g2, margin);
}

/* capsule (geom1) vs box (geom2): both end spheres if both are within the margin, else the sphere at the point of the
 * segment closest to the box (golden-section search on the convex distance function) */
static void collide_capsule_box(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *c = s->geom_xpos + 3 * g1, *cm = s->geom_xmat + 9 * g1;
  real ax[3] = {cm[2], cm[5], cm[8]}, r = m->geom_size[3 * g1], h = m->geom_size[3 * g1 + 1];
  const real *bp = s->geom_xpos + 3 * g2, *bm = s->geom_xmat + 9 * g2;
  const double* bh = m->geom_size + 3 * g2;
  real e0[3], e1[3], cl[3], nn[3];
  copy3(e0, c); addscl3(e0, ax, -h);
  copy3(e1, c); addscl3(e1, ax, h);
  real d0 = point_box(e0, bp, bm, bh, cl, nn) - r, d1 = point_box(e1, bp, bm, bh, cl, nn) - r;
  if (d0 <= margin && d1 <= margin) {
    sphere_box_contact(s, pair, e0, r, g2, margin);
    sphere_box_contact(s, pair, e1, r, g2, margin);
    return;
  }
  const real gr = 0.6180339887498949;
  real lo = -h, hi = h, x1 = hi - gr * (hi - lo), x2 = lo + gr * (hi - lo), p[3];
  copy3(p, c); addscl3(p, ax, x1); real f1 = point_box(p, bp, bm, bh, cl, nn);
  copy3(p, c); addscl3(p, ax, x2); real f2 = point_box(p, bp, bm, bh, cl, nn);
  for (int it = 0; it < 24; it++) {
    if (f1 < f2) { hi = x2; x2 = x1; f2 = f1; x1 = hi - gr * (hi - lo); copy3(p, c); addscl3(p, ax, x1); f1 = point_box(p, bp, bm, bh, cl, nn); }
    else { lo = x1; x1 = x2; f1 = f2; x2 = lo + gr * (hi - lo); copy3(p, c); addscl3(p, ax, x2); f2 = point_box(p, bp, bm, bh, cl, nn); }
  }
  real t = 0.5 * (lo + hi);
  copy3(p, c); addscl3(p, ax, t);
  real fmin = point_box(p, bp, bm, bh, cl, nn);
  if (fmin - r > margin) return;
  /* flat zone {f <= fmin + tol} of the convex distance function: a capsule lying (nearly) parallel on a face gets one
   * contact at each end of the zone instead of one at an arbitrary point of it */
  const real tol = 2e-5;
  real ta = t, tb = t, a0 = -h, b0 = h;
  copy3(p, c); addscl3(p, ax, a0);
  if (point_box(p, bp, bm, bh, cl, nn) <= fmin + tol) ta = a0;
  else { real in = t; for (int it = 0; it < 14; it++) { real mid = 0.5 * (a0 + in); copy3(p, c); addscl3(p, ax, mid);
      if (point_box(p, bp, bm, bh, cl, nn) <= fmin + tol) in = mid; else a0 = mid; } ta = in; }
  copy3(p, c); addscl3(p, ax, b0);
  if (point_box(p, bp, bm, bh, cl, nn) <= fmin + tol) tb = b0;
  else { real in = t; for (int it = 0; it < 14; it++) { real mid = 0.5 * (b0 + in); copy3(p, c); addscl3(p, ax, mid);
      if (point_box(p, bp, bm, bh, cl, nn) <= fmin + tol) in = mid; else b0 = mid; } tb = in; }
  if (tb - ta > r) {
    copy3(p, c); addscl3(p, ax, ta); sphere_box_contact(s, pair, p, r, g2, margin);
    copy3(p, c); addscl3(p, ax, tb); sphere_box_contact(s, pair, p, r, g2, margin);
  } else {
    copy3(p, c); addscl3(p, ax, t);
    sphere_box_contact(s, pair, p, r, g2, margin);
  }
}

/* sphere/capsule (geom1) vs sphere/capsule (geom2): closest points of the two axis segments (a sphere is a segment of
 * zero length), then a sphere-sphere contact there.  Parallel overlapping segments give one contact at the middle of
 * the overlap. */
static void segment_closest(const real* p1, const real* a1, real h1, const real* p2, const real* a2, real h2, real* s_out, real* t_out) {
  real w[3];
  sub3(w, p1, p2);
  real cx[3];
  cross3(cx, a1, a2);   /* den = |a1 x a2|^2 = sin^2 theta (not 1 - b^2: no cancellation, and exact for non-unit axes too) */
  real b = dot3(a1, a2), d = dot3(a1, w), e = dot3(a2, w), den = dot3(cx, cx), sp, tp;
  if (h1 <= 0 && h2 <= 0) { *s_out = 0; *t_out = 0; return; }
  if (h1 <= 0) { sp = 0; tp = e; }
  else if (h2 <= 0) { tp = 0; sp = -d; }
  else if (den > 1e-9) {
    sp = (b * e - d) / den;
    if (sp < -h1) sp = -h1; if (sp > h1) sp = h1;
    tp = e + b * sp;
    if (tp < -h2) { tp = -h2; sp = b * tp - d; }
    else if (tp > h2) { tp = h2; sp = b * tp - d; }
  } else {
    /* parallel: interval of segment 1 (in its own coordinate) facing segment 2 */
    real mid2 = -d, /* centre of segment 2 projected on axis 1, relative to p1 */ lo = mid2 - h2, hi = mid2 + h2;
    if (lo < -h1) lo = -h1; if (hi > h1) hi = h1;
    if (lo > hi) sp = mid2 < 0 ? -h1 : h1; else sp = 0.5 * (lo + hi);
    tp = e + b * sp;
  }
  if (sp < -h1) sp = -h1; if (sp > h1) sp = h1;
  if (tp < -h2) tp = -h2; if (tp > h2) tp = h2;
  *s_out = sp; *t_out = tp;
}
static void collide_round_round(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *c1 = s->geom_xpos + 3 * g1, *m1 = s->geom_xmat + 9 * g1, *c2 = s->geom_xpos + 3 * g2, *m2 = s->geom_xmat + 9 * g2;
  real a1[3] = {m1[2], m1[5], m1[8]}, a2[3] = {m2[2], m2[5], m2[8]};
  real r1 = m->geom_size[3 * g1], r2 = m->geom_size[3 * g2];
  real h1 = m->geom_type[g1] == B200_GEOM_CAPSULE ? m->geom_size[3 * g1 + 1] : 0;
  real h2 = m->geom_type[g2] == B200_GEOM_CAPSULE ? m->geom_size[3 * g2 + 1] : 0;
  real sp, tp, q1[3], q2[3], n[3];
  segment_closest(c1, a1, h1, c2, a2, h2, &sp, &tp);
  copy3(q1, c1); addscl3(q1, a1, sp);
  copy3(q2, c2); addscl3(q2, a2, tp);
  sub3(n, q2, q1);
  real len = sqrt(dot3(n, n)), d = len - r1 - r2;
  if (d > margin) return;
  if (len < 1e-12) { n[0] = 0; n[1] = 0; n[2] = 1; } else { n[0] /= len; n[1] /= len; n[2] /= len; }
  real pos[3];
  copy3(pos, q1);
  addscl3(pos, n, r1 + 0.5 * d);
  add_contact(s, pair, d, pos, n);
}


/* ---- general convex pairs (cylinder / ellipsoid against box, capsule, sphere, cylinder, ellipsoid): Minkowski portal
 * refinement on the support functions (Snethen, "XenoCollide", Game Programming Gems 7 -- the published algorithm that
 * MuJoCo's convex collider wraps through libccd: tolerance opt.mpr_tolerance = 1e-6, at most opt.mpr_iterations = 50 rounds);
 * one contact per pair, both shapes inflated by margin / 2, dist = margin - depth.  Everything is evaluated relative to the
 * first geom's centre (the fp32 twin in csrc/sim_core.cuh needs that; here it only keeps the two implementations alike). */
typedef struct { int type; real pos[3]; const real* mat; const double* size; real infl; const double* hv; int nhv; } CvxShape;
static void cvx_support(const CvxShape* g, const real* d, real* out) {
  real l[3], sl[3] = {0, 0, 0};
  mulmatTvec3(l, g->mat, d);
  const double* z = g->size;
  switch (g->type) {
    case B200_GEOM_SPHERE: { real n = norm3(l); if (n > 0) { sl[0] = z[0] * l[0] / n; sl[1] = z[0] * l[1] / n; sl[2] = z[0] * l[2] / n; } break; }
    case B200_GEOM_CAPSULE: { real n = norm3(l); if (n > 0) { sl[0] = z[0] * l[0] / n; sl[1] = z[0] * l[1] / n; sl[2] = z[0] * l[2] / n; } sl[2] += l[2] >= 0 ? z[1] : -z[1]; break; }
    case B200_GEOM_CYLINDER: { real n = sqrt(l[0] * l[0] + l[1] * l[1]); if (n > 1e-12) { sl[0] = z[0] * l[0] / n; sl[1] = z[0] * l[1] / n; } sl[2] = l[2] >= 0 ? z[1] : -z[1]; break; }
    case B200_GEOM_ELLIPSOID: { real a = z[0] * l[0], b = z[1] * l[1], c = z[2] * l[2], n = sqrt(a * a + b * b + c * c); if (n > 0) { sl[0] = z[0] * a / n; sl[1] = z[1] * b / n; sl[2] = z[2] * c / n; } break; }
    case B200_GEOM_MESH: {   /* reduced convex hull (mjcf.py hull_vertices): the vertex that is farthest along l, first one on ties */
      int best = 0; real bd = -1e300;
      for (int i = 0; i < g->nhv; i++) { real dd = g->hv[3 * i] * l[0] + g->hv[3 * i + 1] * l[1] + g->hv[3 * i + 2] * l[2]; if (dd > bd) { bd = dd; best = i; } }
      if (g->nhv > 0) { sl[0] = g->hv[3 * best]; sl[1] = g->hv[3 * best + 1]; sl[2] = g->hv[3 * best + 2]; }
      break;
    }
    default: /* box */ sl[0] = l[0] >= 0 ? z[0] : -z[0]; sl[1] = l[1] >= 0 ? z[1] : -z[1]; sl[2] = l[2] >= 0 ? z[2] : -z[2]; break;
  }
  mulmatvec3(out, g->mat, sl);
  real n = norm3(d);
  for (int k = 0; k < 3; k++) out[k] += g->pos[k] + (n > 0 ? g->infl * d[k] / n : 0);
}
typedef struct { real v[3], a[3], b[3]; } CvxPt; /* point of A - B and its witnesses */
static void cvx_msupport(const CvxShape* A, const CvxShape* B, const real* d, CvxPt* p) {
  real nd[3] = {-d[0], -d[1], -d[2]};
  cvx_support(A, d, p->a); cvx_support(B, nd, p->b);
  sub3(p->v, p->a, p->b);
}
/* returns 1 and (depth, dir from A to B, pos) when the inflated shapes overlap */
static int cvx_mpr(const CvxShape* A, const CvxShape* B, real tol, int maxit, real* depth, real* dir_out, real* pos) {
  CvxPt v0, v1, v2, v3, v4;
  real dir[3], va[3], vb[3], t[3];
  copy3(v0.a, A->pos); copy3(v0.b, B->pos); sub3(v0.v, v0.a, v0.b);
  if (norm3(v0.v) < 1e-12) v0.v[0] = 1e-5;
  for (int k = 0; k < 3; k++) dir[k] = -v0.v[k];
  normalize3(dir);
  cvx_msupport(A, B, dir, &v1);
  if (dot3(v1.v, dir) <= 0) return 0;
  cross3(dir, v0.v, v1.v);
  if (norm3(dir) < 1e-12) {
    /* the origin lies on the ray v0 -> v1: the centres' line is the contact normal */
    for (int k = 0; k < 3; k++) dir_out[k] = -v0.v[k];
    normalize3(dir_out);
    *depth = dot3(v1.v, dir_out);
    for (int k = 0; k < 3; k++) pos[k] = 0.5 * (v1.a[k] + v1.b[k]);
    return 1;
  }
  normalize3(dir);
  cvx_msupport(A, B, dir, &v2);
  if (dot3(v2.v, dir) <= 0) return 0;
  sub3(va, v1.v, v0.v); sub3(vb, v2.v, v0.v); cross3(dir, va, vb); normalize3(dir);
  if (dot3(dir, v0.v) > 0) { CvxPt tmp = v1; v1 = v2; v2 = tmp; for (int k = 0; k < 3; k++) dir[k] = -dir[k]; }
  /* portal discovery */
  for (int it = 0;; it++) {
    if (it > maxit) return 0;
    cvx_msupport(A, B, dir, &v3);
    if (dot3(v3.v, dir) <= 0) return 0;
    int cont = 0;
    cross3(t, v1.v, v3.v);
    if (dot3(t, v0.v) < 0) { v2 = v3; cont = 1; }
    else { cross3(t, v3.v, v2.v); if (dot3(t, v0.v) < 0) { v1 = v3; cont = 1; } }
    if (!cont) break;
    sub3(va, v1.v, v0.v); sub3(vb, v2.v, v0.v); cross3(dir, va, vb); normalize3(dir);
  }
  /* portal refinement; once the portal has passed the origin the shapes overlap and the loop continues to the surface */
  int hit = 0;
  for (int it = 0;; it++) {
    sub3(va, v2.v, v1.v); sub3(vb, v3.v, v1.v); cross3(dir, va, vb); normalize3(dir);
    if (dot3(dir, v1.v) >= 0) hit = 1;
    cvx_msupport(A, B, dir, &v4);
    real d4 = dot3(v4.v, dir);
    if (!hit && d4 < 0) return 0;
    real m1 = d4 - dot3(v1.v, dir), m2 = d4 - dot3(v2.v, dir), m3 = d4 - dot3(v3.v, dir);
    real mn = m1 < m2 ? (m1 < m3 ? m1 : m3) : (m2 < m3 ? m2 : m3);
    if (mn <= tol || it >= maxit) {
      if (!hit) return 0;
      break;
    }
    cross3(t, v4.v, v0.v);
    if (dot3(v1.v, t) > 0) { if (dot3(v2.v, t) > 0) v1 = v4; else v3 = v4; }
    else { if (dot3(v3.v, t) > 0) v2 = v4; else v1 = v4; }
  }
  /* depth = distance of the origin from the portal plane along its normal; witnesses by barycentric weights of the
   * portal tetrahedron (v0 is interior, so its weight only matters before normalisation) */
  *depth = dot3(dir, v1.v);
  copy3(dir_out, dir);
  real b0, b1, b2, b3, sum;
  cross3(t, v1.v, v2.v); b0 = dot3(t, v3.v);
  cross3(t, v3.v, v2.v); b1 = dot3(t, v0.v);
  cross3(t, v0.v, v1.v); b2 = dot3(t, v3.v);
  cross3(t, v2.v, v1.v); b3 = dot3(t, v0.v);
  sum = b0 + b1 + b2 + b3;
  if (sum <= 0) {
    b0 = 0;
    cross3(t, v2.v, v3.v); b1 = dot3(t, dir);
    cross3(t, v3.v, v1.v); b2 = dot3(t, dir);
    cross3(t, v1.v, v2.v); b3 = dot3(t, dir);
    sum = b1 + b2 + b3;
  }
  if (!(fabs(sum) > 0)) return 0;
  for (int k = 0; k < 3; k++)
    pos[k] = 0.5 * (b0 * (v0.a[k] + v0.b[k]) + b1 * (v1.a[k] + v1.b[k]) + b2 * (v2.a[k] + v2.b[k]) + b3 * (v3.a[k] + v3.b[k])) / sum;
  return 1;
}
static void collide_convex(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  CvxShape A = {m->geom_type[g1], {0, 0, 0}, s->geom_xmat + 9 * g1, m->geom_size + 3 * g1, 0.5 * margin, NULL, 0};
  CvxShape B = {m->geom_type[g2], {0, 0, 0}, s->geom_xmat + 9 * g2, m->geom_size + 3 * g2, 0.5 * margin, NULL, 0};
  if (A.type == B200_GEOM_MESH) { A.hv = m->hull_vert + 3 * m->geom_hull[2 * g1]; A.nhv = m->geom_hull[2 * g1 + 1]; }
  if (B.type == B200_GEOM_MESH) { B.hv = m->hull_vert + 3 * m->geom_hull[2 * g2]; B.nhv = m->geom_hull[2 * g2 + 1]; }
  sub3(B.pos, s->geom_xpos + 3 * g2, s->geom_xpos + 3 * g1);
  real depth, dir[3], pos[3];
  if (!cvx_mpr(&A, &B, 1e-6, 50, &depth, dir, pos)) return;
  add3(pos, pos, s->geom_xpos + 3 * g1);
  add_contact(s, pair, margin - depth, pos, dir);
}
/* plane vs cylinder: deepest point of the lower rim, the same rim direction on the other cap, and two more points of
 * the lower rim at +-120 degrees (own point selection; MuJoCo's mjc_PlaneCylinder picks up to four points differently) */
static void collide_plane_cylinder(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *pp = s->geom_xpos + 3 * g1, *pm = s->geom_xmat + 9 * g1, *c = s->geom_xpos + 3 * g2, *cm = s->geom_xmat + 9 * g2;
  real n[3] = {pm[2], pm[5], pm[8]}, ax[3] = {cm[2], cm[5], cm[8]};
  real r = m->geom_size[3 * g2], h = m->geom_size[3 * g2 + 1];
  real an = dot3(ax, n);
  if (an > 0) { ax[0] = -ax[0]; ax[1] = -ax[1]; ax[2] = -ax[2]; an = -an; }   /* ax points towards the plane */
  real rad[3] = {-n[0] + an * ax[0], -n[1] + an * ax[1], -n[2] + an * ax[2]};  /* rim direction of steepest descent */
  real rl = norm3(rad);
  if (rl < 1e-9) { real y[3] = {0, 0, 0}; if (fabs(ax[0]) < 0.5) y[0] = 1; else y[1] = 1; cross3(rad, ax, y); rl = norm3(rad); }
  for (int k = 0; k < 3; k++) rad[k] /= rl;
  real side[3];
  cross3(side, ax, rad);
  const real cs[4] = {1, 1, -0.5, -0.5}, sn[4] = {0, 0, 0.8660254037844386, -0.8660254037844386}, cap[4] = {1, -1, 1, 1};
  for (int i = 0; i < 4; i++) {
    real p[3], dif[3];
    for (int k = 0; k < 3; k++) p[k] = c[k] + cap[i] * h * ax[k] + r * (cs[i] * rad[k] + sn[i] * side[k]);
    sub3(dif, p, pp);
    real d = dot3(dif, n);
    if (d > margin) continue;
    addscl3(p, n, -0.5 * d);
    add_contact(s, pair, d, p, n);
  }
}
/* plane vs ellipsoid: the support point of the ellipsoid against the plane normal */
static void collide_plane_ellipsoid(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *pp = s->geom_xpos + 3 * g1, *pm = s->geom_xmat + 9 * g1;
  real n[3] = {pm[2], pm[5], pm[8]}, nn[3] = {-n[0], -n[1], -n[2]}, p[3], dif[3];
  CvxShape E = {B200_GEOM_ELLIPSOID, {0, 0, 0}, s->geom_xmat + 9 * g2, m->geom_size + 3 * g2, 0, NULL, 0};
  copy3(E.pos, s->geom_xpos + 3 * g2);
  cvx_support(&E, nn, p);
  sub3(dif, p, pp);
  real d = dot3(dif, n);
  if (d > margin) return;
  addscl3(p, n, -0.5 * d);
  add_contact(s, pair, d, p, n);
}

/* plane vs hull (mesh geoms compiled with mesh_hull): the hull vertices within the margin of the plane, the deepest first, at most four
 * (own point selection; ties keep the lower vertex index) */
static void collide_plane_hull(oracle_sim* s, int pair, real margin) {
  const b200_model_view* m = &s->m;
  int g1 = m->pair_geom1[pair], g2 = m->pair_geom2[pair];
  const real *pp = s->geom_xpos + 3 * g1, *pm = s->geom_xmat + 9 * g1, *c = s->geom_xpos + 3 * g2, *cm = s->geom_xmat + 9 * g2;
  real n[3] = {pm[2], pm[5], pm[8]};
  const double* hv = m->hull_vert + 3 * m->geom_hull[2 * g2];
  int nhv = m->geom_hull[2 * g2 + 1];
  real last = -1e300; int lasti = -1;
  for (int k = 0; k < 4; k++) {
    /* the next vertex in (distance, index) order after (last, lasti) */
    int best = -1; real bd = 1e300;
    for (int i = 0; i < nhv; i++) {
      real p[3], dif[3];
      mulmatvec3(p, cm, hv + 3 * i);
      for (int a = 0; a < 3; a++) dif[a] = p[a] + c[a] - pp[a];
      real d = dot3(dif, n);
      if ((d > last || (d == last && i > lasti)) && d < bd) { bd = d; best = i; }
    }
    if (best < 0 || bd > margin) break;
    real p[3];
    mulmatvec3(p, cm, hv + 3 * best);
    for (int a = 0; a < 3; a++) p[a] += c[a];
    addscl3(p, n, -0.5 * bd);
    add_contact(s, pair, bd, p, n);
    last = bd; lasti = best;
  }
}

static void collision(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  s->ncon = 0;
  for (int p = 0; p < m->npair; p++) {
    int g1 = m->pair_geom1[p], g2 = m->pair_geom2[p];
    int t1 = m->geom_type[g1], t2 = m->geom_type[g2];
    real margin = m->pair_margin[p];
    /* bounding-sphere / plane-distance rejection */
    if (t1 == B200_GEOM_PLANE) {
      const real* pm = s->geom_xmat + 9 * g1;
      real n[3] = {pm[2], pm[5], pm[8]}, dif[3];
      sub3(dif, s->geom_xpos + 3 * g2, s->geom_xpos + 3 * g1);
      if (dot3(dif, n) > margin + m->geom_rbound[g2]) continue;
    } else {
      real dif[3];
      sub3(dif, s->geom_xpos + 3 * g2, s->geom_xpos + 3 * g1);
      real bound = margin + m->geom_rbound[g1] + m->geom_rbound[g2];
      if (dot3(dif, dif) > bound * bound) continue;
    }
    if (t1 == B200_GEOM_PLANE && t2 == B200_GEOM_BOX) collide_plane_box(s, p, margin);
    else if (t1 == B200_GEOM_PLANE && t2 == B200_GEOM_SPHERE) collide_plane_sphere(s, p, margin);
    else if (t1 == B200_GEOM_PLANE && t2 == B200_GEOM_CAPSULE) collide_plane_capsule(s, p, margin);
    else if (t1 == B200_GEOM_BOX && t2 == B200_GEOM_BOX) collide_box_box(s, p, margin);
    else if (t1 == B200_GEOM_SPHERE && t2 == B200_GEOM_BOX) collide_sphere_box(s, p, margin);
    else if (t1 == B200_GEOM_CAPSULE && t2 == B200_GEOM_BOX) collide_capsule_box(s, p, margin);
    else if ((t1 == B200_GEOM_SPHERE || t1 == B200_GEOM_CAPSULE) && (t2 == B200_GEOM_SPHERE || t2 == B200_GEOM_CAPSULE))
      collide_round_round(s, p, margin);
    else if (t1 == B200_GEOM_PLANE && t2 == B200_GEOM_CYLINDER) collide_plane_cylinder(s, p, margin);
    else if (t1 == B200_GEOM_PLANE && t2 == B200_GEOM_ELLIPSOID) collide_plane_ellipsoid(s, p, margin);
    else if (t1 == B200_GEOM_PLANE && t2 == B200_GEOM_MESH && m->n_geom_hull > 0) collide_plane_hull(s, p, margin);
    else if (t1 >= B200_GEOM_SPHERE && t1 <= B200_GEOM_MESH && t2 >= B200_GEOM_SPHERE && t2 <= B200_GEOM_MESH &&
             ((t1 != B200_GEOM_MESH && t2 != B200_GEOM_MESH) || m->n_geom_hull > 0))
      collide_convex(s, p, margin);   /* any pair with a cylinder, an ellipsoid or a hull (mesh geom with a vertex table) */
    /* other pair types (height fields): not restated (DESIGN.md lists them) */
  }
}

/* ------------------------------------------------------------------------------------------------ */
/* 6. constraint rows */
static void get_impedance(const real* solimp_in, real pos, real margin, real* imp, real* impP) {
  real si[5] = {solimp_in[0], solimp_in[1], solimp_in[2], solimp_in[3], solimp_in[4]};
  for (int k = 0; k < 2; k++) { if (si[k] < MINIMP) si[k] = MINIMP; if (si[k] > MAXIMP) si[k] = MAXIMP; }
  if (si[2] < 0) si[2] = 0;
  if (si[3] < MINIMP) si[3] = MINIMP; if (si[3] > MAXIMP) si[3] = MAXIMP;
  if (si[4] < 1) si[4] = 1;
  if (si[0] == si[1] || si[2] <= MINVAL) { *imp = 0.5 * (si[0] + si[1]); *impP = 0; return; }
  real x = (pos - margin) / si[2];
  if (x < 0) x = -x;
  if (x >= 1) { *imp = si[1]; *impP = 0; return; }
  if (x <= 0) { *imp = si[0]; *impP = 0; return; }
  real y;
  if (si[4] == 1) y = x;
  else if (x <= si[3]) y = pow(x, si[4]) / pow(si[3], si[4] - 1);
  else y = 1 - pow(1 - x, si[4]) / pow(1 - si[3], si[4] - 1);
  *imp = si[0] + y * (si[1] - si[0]);
  *impP = 0;
}

static int add_row(oracle_sim* s, int type, int id, real pos, real margin, real floss, real diagA, const real* solref,
                   const real* solimp) {
  if (s->nefc >= MAXEFC) { s->warn_overflow++; return -1; }
  int i = s->nefc++;
  memset(s->J + (size_t)i * s->nv, 0, sizeof(real) * s->nv);
  s->efc_type[i] = type; s->efc_id[i] = id; s->efc_pos[i] = pos; s->efc_margin[i] = margin; s->efc_floss[i] = floss;
  s->efc_diagA[i] = diagA;
  real h = s->m.opt[B200_OPT_TIMESTEP];
  real imp, impP;
  get_impedance(solimp, pos, margin, &imp, &impP);
  real dmax = solimp[1];
  if (dmax < MINIMP) dmax = MINIMP; if (dmax > MAXIMP) dmax = MAXIMP;
  real K, B;
  if (solref[0] > 0) {
    real tc = solref[0] < 2 * h ? 2 * h : solref[0]; /* refsafe */
    real dr = solref[1];
    real kd = dmax * dmax * tc * tc * dr * dr, bd = dmax * tc;
    K = 1 / (kd > MINVAL ? kd : MINVAL);
    B = 2 / (bd > MINVAL ? bd : MINVAL);
  } else { K = -solref[0] / (dmax * dmax); B = -solref[1] / dmax; }
  if (type == ROW_FRICTION) K = 0;
  s->efc_KBIP[i][0] = K; s->efc_KBIP[i][1] = B; s->efc_KBIP[i][2] = imp; s->efc_KBIP[i][3] = impP;
  real R = (1 - imp) / imp * diagA;
  if (R < MINVAL) R = MINVAL;
  s->efc_R[i] = R; s->efc_D[i] = 1 / R;
  return i;
}

static void make_constraint(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  int nv = s->nv;
  s->nefc = 0;
  real* jp1 = dalloc(3 * nv), *jr1 = dalloc(3 * nv), *jp2 = dalloc(3 * nv), *jr2 = dalloc(3 * nv);
  /* equality */
  for (int e = 0; e < m->neq; e++) {
    if (!m->eq_active[e]) continue;
    const real* data = s->eq_data + 11 * e;
    real solref[2] = {m->eq_solref[2 * e], m->eq_solref[2 * e + 1]}, solimp[5];
    for (int k = 0; k < 5; k++) solimp[k] = m->eq_solimp[5 * e + k];
    if (m->eq_type[e] == B200_EQ_WELD) {
      /* objects are body-frame sites (or -1 = world).  data: [anchor(3) on obj2 | relpos(3) on obj1 | relquat(4) | torquescale] */
      int s1 = m->eq_obj1[e], s2 = m->eq_obj2[e];
      real p1[3], p2[3], q1[4] = {1, 0, 0, 0}, q2[4] = {1, 0, 0, 0}, t[3];
      int b1 = 0, b2 = 0;
      const real idm[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
      const real *x1 = idm, *x2 = idm;
      real z3[3] = {0, 0, 0};
      const real *o1 = z3, *o2 = z3;
      real sq1[4], sq2[4];
      if (s1 >= 0) { b1 = m->site_body[s1]; x1 = s->site_xmat + 9 * s1; o1 = s->site_xpos + 3 * s1;
        real q[4] = {m->site_quat[4 * s1], m->site_quat[4 * s1 + 1], m->site_quat[4 * s1 + 2], m->site_quat[4 * s1 + 3]};
        mulquat(sq1, s->xquat + 4 * b1, q); memcpy(q1, sq1, sizeof(q1)); }
      if (s2 >= 0) { b2 = m->site_body[s2]; x2 = s->site_xmat + 9 * s2; o2 = s->site_xpos + 3 * s2;
        real q[4] = {m->site_quat[4 * s2], m->site_quat[4 * s2 + 1], m->site_quat[4 * s2 + 2], m->site_quat[4 * s2 + 3]};
        mulquat(sq2, s->xquat + 4 * b2, q); memcpy(q2, sq2, sizeof(q2)); }
      mulmatvec3(t, x1, data + 3); add3(p1, o1, t);
      mulmatvec3(t, x2, data + 0); add3(p2, o2, t);
      real cpos[6];
      sub3(cpos, p1, p2);
      jac_point(s, b1, p1, jp1, jr1);
      jac_point(s, b2, p2, jp2, jr2);
      real ts = data[10];
      real quat[4], quat1[4] = {q2[0], -q2[1], -q2[2], -q2[3]}, quat2[4];
      mulquat(quat, q1, data + 6);
      mulquat(quat2, quat1, quat);
      cpos[3] = ts * quat2[1]; cpos[4] = ts * quat2[2]; cpos[5] = ts * quat2[3];
      real iw_t = m->eq_invweight[2 * e], iw_r = m->eq_invweight[2 * e + 1];
      int rows[6];
      for (int k = 0; k < 6; k++) rows[k] = add_row(s, ROW_EQ, e, cpos[k], 0, 0, k < 3 ? iw_t : iw_r, solref, solimp);
      for (int k = 0; k < 3; k++) if (rows[k] >= 0)
        for (int d = 0; d < nv; d++) s->J[(size_t)rows[k] * nv + d] = jp1[k * nv + d] - jp2[k * nv + d];
      for (int d = 0; d < nv; d++) {
        real axis[3] = {jr1[d] - jr2[d], jr1[nv + d] - jr2[nv + d], jr1[2 * nv + d] - jr2[2 * nv + d]};
        real qa[4] = {0, axis[0], axis[1], axis[2]}, t1[4], t2[4];
        mulquat(t1, quat1, qa);
        mulquat(t2, t1, quat);
        for (int k = 0; k < 3; k++) if (rows[3 + k] >= 0) s->J[(size_t)rows[3 + k] * nv + d] = 0.5 * ts * t2[1 + k];
      }
    } else if (m->eq_type[e] == B200_EQ_JOINT) {
      int j1 = m->eq_obj1[e], j2 = m->eq_obj2[e];
      int a1 = m->jnt_qposadr[j1], d1 = m->jnt_dofadr[j1];
      real pos = s->qpos[a1] - m->qpos0[a1], deriv = 0;
      if (j2 >= 0) {
        int a2 = m->jnt_qposadr[j2];
        real dif = s->qpos[a2] - m->qpos0[a2];
        pos -= data[0] + data[1] * dif + data[2] * dif * dif + data[3] * dif * dif * dif + data[4] * dif * dif * dif * dif;
        deriv = data[1] + 2 * data[2] * dif + 3 * data[3] * dif * dif + 4 * data[4] * dif * dif * dif;
      } else pos -= data[0];
      int i = add_row(s, ROW_EQ, e, pos, 0, 0, m->eq_invweight[2 * e], solref, solimp);
      if (i >= 0) {
        s->J[(size_t)i * nv + d1] = 1;
        if (j2 >= 0) s->J[(size_t)i * nv + m->jnt_dofadr[j2]] = -deriv;
      }
    }
  }
  /* dof frictionloss */
  for (int d = 0; d < nv; d++) {
    if (m->dof_frictionloss[d] <= 0) continue;
    real sr[2] = {m->dof_solref_fri[2 * d], m->dof_solref_fri[2 * d + 1]}, si[5];
    for (int k = 0; k < 5; k++) si[k] = m->dof_solimp_fri[5 * d + k];
    int i = add_row(s, ROW_FRICTION, d, 0, 0, m->dof_frictionloss[d], m->dof_invweight0[d], sr, si);
    if (i >= 0) s->J[(size_t)i * nv + d] = 1;
  }
  /* joint limits */
  for (int j = 0; j < m->njnt; j++) {
    if (!m->jnt_limited[j] || m->jnt_type[j] == B200_JNT_FREE) continue;
    real q = s->qpos[m->jnt_qposadr[j]], margin = m->jnt_margin[j];
    real sr[2] = {m->jnt_solref[2 * j], m->jnt_solref[2 * j + 1]}, si[5];
    for (int k = 0; k < 5; k++) si[k] = m->jnt_solimp[5 * j + k];
    for (int side = -1; side <= 1; side += 2) {
      real dist = side * (s->jnt_range[2 * j + (side + 1) / 2] - q);
      if (dist < margin) {
        int i = add_row(s, ROW_LIMIT, j, dist, margin, 0, m->dof_invweight0[m->jnt_dofadr[j]], sr, si);
        if (i >= 0) s->J[(size_t)i * nv + m->jnt_dofadr[j]] = -side;
      }
    }
  }
  /* tendon limits */
  for (int t = 0; t < m->ntendon; t++) {
    if (!m->ten_limited[t]) continue;
    real margin = m->ten_margin[t];
    real sr[2] = {m->ten_solref[2 * t], m->ten_solref[2 * t + 1]}, si[5];
    for (int k = 0; k < 5; k++) si[k] = m->ten_solimp[5 * t + k];
    for (int side = -1; side <= 1; side += 2) {
      real dist = side * (m->ten_range[2 * t + (side + 1) / 2] - s->ten_length[t]);
      if (dist < margin) {
        int i = add_row(s, ROW_LIMIT, m->njnt + t, dist, margin, 0, m->ten_invweight0[t], sr, si);
        if (i >= 0) for (int d = 0; d < nv; d++) s->J[(size_t)i * nv + d] = -side * s->ten_J[t * nv + d];
      }
    }
  }
  /* contacts (pyramidal) */
  for (int c = 0; c < s->ncon; c++) {
    Contact* con = &s->con[c];
    con->efc_address = -1;
    if (con->dist >= con->includemargin) continue; /* excluded by gap */
    jac_point(s, con->body1, con->pos, jp1, jr1);
    jac_point(s, con->body2, con->pos, jp2, jr2);
    int dim = con->dim;
    /* contact-frame Jacobian rows: 3 translational (+ up to 3 rotational) */
    real* Jc = dalloc((size_t)6 * nv);
    for (int k = 0; k < 3; k++)
      for (int d = 0; d < nv; d++) {
        real vp = 0, vr = 0;
        for (int a = 0; a < 3; a++) {
          vp += con->frame[3 * k + a] * (jp2[a * nv + d] - jp1[a * nv + d]);
          vr += con->frame[3 * k + a] * (jr2[a * nv + d] - jr1[a * nv + d]);
        }
        Jc[k * nv + d] = vp; Jc[(3 + k) * nv + d] = vr;
      }
    real tran = m->pair_invweight[2 * con->pair], rot = m->pair_invweight[2 * con->pair + 1];
    con->efc_address = s->nefc;
    if (dim == 1) {
      int i = add_row(s, ROW_CONTACT, c, con->dist, con->includemargin, 0, tran, con->solref, con->solimp);
      if (i >= 0) memcpy(s->J + (size_t)i * nv, Jc, sizeof(real) * nv);
    } else {
      int first = -1;
      for (int k = 1; k < dim; k++) {
        real mu = con->friction[k - 1];
        real dA = tran + mu * mu * (k < 3 ? tran : rot);
        for (int sg = 1; sg >= -1; sg -= 2) {
          int i = add_row(s, ROW_CONTACT, c, con->dist, con->includemargin, 0, dA, con->solref, con->solimp);
          if (i < 0) continue;
          if (first < 0) first = i;
          for (int d = 0; d < nv; d++) s->J[(size_t)i * nv + d] = Jc[d] + sg * mu * Jc[k * nv + d];
        }
      }
      /* pyramid regularisation: every edge shares R = 2 mu^2 R(first row), mu = friction[0] / sqrt(impratio) */
      if (first >= 0) {
        real mu = con->friction[0] / sqrt(m->opt[B200_OPT_IMPRATIO]);
        real Rpy = 2 * mu * mu * s->efc_R[first];
        if (Rpy < MINVAL) Rpy = MINVAL;
        for (int i = first; i < s->nefc; i++) { s->efc_R[i] = Rpy; s->efc_D[i] = 1 / Rpy; }
      }
    }
    free(Jc);
  }
  free(jp1); free(jr1); free(jp2); free(jr2);
}

/* ------------------------------------------------------------------------------------------------ */
/* 7. velocity-dependent terms and smooth forces */
static void com_vel(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  memset(s->cvel, 0, 6 * sizeof(real));
  for (int b = 1; b < s->nbody; b++) {
    real v[6];
    memcpy(v, s->cvel + 6 * m->body_parent[b], sizeof(v));
    int da = m->body_dofadr[b], dn = m->body_dofnum[b];
    int d = da;
    while (d < da + dn) {
      int j = m->dof_jnt[d];
      if (m->jnt_type[j] == B200_JNT_FREE) {
        for (int k = 0; k < 3; k++) { memset(s->cdof_dot + 6 * (d + k), 0, 6 * sizeof(real)); for (int a = 0; a < 6; a++) v[a] += s->cdof[6 * (d + k) + a] * s->qvel[d + k]; }
        for (int k = 3; k < 6; k++) cross_motion(s->cdof_dot + 6 * (d + k), v, s->cdof + 6 * (d + k));
        for (int k = 3; k < 6; k++) for (int a = 0; a < 6; a++) v[a] += s->cdof[6 * (d + k) + a] * s->qvel[d + k];
        d += 6;
      } else {
        cross_motion(s->cdof_dot + 6 * d, v, s->cdof + 6 * d);
        for (int a = 0; a < 6; a++) v[a] += s->cdof[6 * d + a] * s->qvel[d];
        d += 1;
      }
    }
    memcpy(s->cvel + 6 * b, v, sizeof(v));
  }
}

static void rne_bias(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  real g[3] = {m->opt[B200_OPT_GRAVITY], m->opt[B200_OPT_GRAVITY + 1], m->opt[B200_OPT_GRAVITY + 2]};
  s->cacc[0] = s->cacc[1] = s->cacc[2] = 0; s->cacc[3] = -g[0]; s->cacc[4] = -g[1]; s->cacc[5] = -g[2];
  memset(s->cfrc, 0, 6 * sizeof(real));
  for (int b = 1; b < s->nbody; b++) {
    real* a = s->cacc + 6 * b;
    memcpy(a, s->cacc + 6 * m->body_parent[b], 6 * sizeof(real));
    for (int d = m->body_dofadr[b]; d < m->body_dofadr[b] + m->body_dofnum[b]; d++)
      for (int k = 0; k < 6; k++) a[k] += s->cdof_dot[6 * d + k] * s->qvel[d];
    real Ia[6], Iv[6], vxIv[6];
    mul_inert_vec(Ia, s->cinert + 10 * b, a);
    mul_inert_vec(Iv, s->cinert + 10 * b, s->cvel + 6 * b);
    cross_force(vxIv, s->cvel + 6 * b, Iv);
    for (int k = 0; k < 6; k++) s->cfrc[6 * b + k] = Ia[k] + vxIv[k];
  }
  for (int b = s->nbody - 1; b > 0; b--) {
    int p = m->body_parent[b];
    if (p > 0) for (int k = 0; k < 6; k++) s->cfrc[6 * p + k] += s->cfrc[6 * b + k];
  }
  for (int d = 0; d < s->nv; d++) {
    real v = 0;
    for (int k = 0; k < 6; k++) v += s->cdof[6 * d + k] * s->cfrc[6 * m->dof_body[d] + k];
    s->qfrc_bias[d] = v;
  }
}

static void passive(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  for (int d = 0; d < s->nv; d++) s->qfrc_passive[d] = -m->dof_damping[d] * s->qvel[d];
  for (int j = 0; j < m->njnt; j++) {
    if (m->jnt_stiffness[j] == 0 || m->jnt_type[j] == B200_JNT_FREE) continue;
    int a = m->jnt_qposadr[j];
    s->qfrc_passive[m->jnt_dofadr[j]] -= m->jnt_stiffness[j] * (s->qpos[a] - m->qpos_spring[a]);
  }
}

static void actuation(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  memset(s->qfrc_actuator, 0, sizeof(real) * s->nv);
  for (int i = 0; i < s->nu; i++) {
    real c = s->ctrl[i];
    if (m->act_ctrllimited[i]) { if (c < m->act_ctrlrange[2 * i]) c = m->act_ctrlrange[2 * i]; if (c > m->act_ctrlrange[2 * i + 1]) c = m->act_ctrlrange[2 * i + 1]; }
    int j = m->act_trnid[i];
    real gear = m->act_gear[i];
    real len = gear * s->qpos[m->jnt_qposadr[j]], vel = gear * s->qvel[m->jnt_dofadr[j]];
    real f = s->act_gainprm[3 * i] * c + s->act_biasprm[3 * i] + s->act_biasprm[3 * i + 1] * len + s->act_biasprm[3 * i + 2] * vel;
    if (m->act_forcelimited[i]) { if (f < m->act_forcerange[2 * i]) f = m->act_forcerange[2 * i]; if (f > m->act_forcerange[2 * i + 1]) f = m->act_forcerange[2 * i + 1]; }
    s->actuator_force[i] = f;
    s->qfrc_actuator[m->jnt_dofadr[j]] += gear * f;
  }
}

/* ------------------------------------------------------------------------------------------------ */
/* 8. Newton solver (primal, pyramidal) */
typedef struct { real cost, d1, d2; } LsPoint;

static real constraint_update(oracle_sim* s, const real* jar, real* force, int* active) {
  real cost = 0;
  for (int i = 0; i < s->nefc; i++) {
    real D = s->efc_D[i], R = s->efc_R[i], x = jar[i];
    switch (s->efc_type[i]) {
      case ROW_EQ: force[i] = -D * x; active[i] = 1; cost += 0.5 * D * x * x; break;
      case ROW_FRICTION: {
        real f = s->efc_floss[i];
        if (x <= -R * f) { force[i] = f; active[i] = 0; cost += -0.5 * R * f * f - f * x; }
        else if (x >= R * f) { force[i] = -f; active[i] = 0; cost += -0.5 * R * f * f + f * x; }
        else { force[i] = -D * x; active[i] = 1; cost += 0.5 * D * x * x; }
      } break;
      default:
        if (x < 0) { force[i] = -D * x; active[i] = 1; cost += 0.5 * D * x * x; }
        else { force[i] = 0; active[i] = 0; }
    }
  }
  return cost;
}

static LsPoint ls_eval(const oracle_sim* s, real alpha, const real* jar, const real* jv, const real* qg) {
  LsPoint p;
  p.cost = qg[0] + alpha * qg[1] + alpha * alpha * qg[2];
  p.d1 = qg[1] + 2 * alpha * qg[2];
  p.d2 = 2 * qg[2];
  for (int i = 0; i < s->nefc; i++) {
    real D = s->efc_D[i], R = s->efc_R[i], x = jar[i] + alpha * jv[i], v = jv[i];
    int quad = 0;
    if (s->efc_type[i] == ROW_EQ) quad = 1;
    else if (s->efc_type[i] == ROW_FRICTION) {
      real f = s->efc_floss[i];
      if (x <= -R * f) { p.cost += -0.5 * R * f * f - f * x; p.d1 += -f * v; }
      else if (x >= R * f) { p.cost += -0.5 * R * f * f + f * x; p.d1 += f * v; }
      else quad = 1;
    } else quad = x < 0;
    if (quad) { p.cost += 0.5 * D * x * x; p.d1 += D * x * v; p.d2 += D * v * v; }
  }
  return p;
}

/* exact line search on the convex piecewise-quadratic: safeguarded Newton on phi'(alpha) */
static real linesearch(const oracle_sim* s, const real* jar, const real* jv, const real* qg, real gtol, int maxit) {
  LsPoint p0 = ls_eval(s, 0, jar, jv, qg);
  if (p0.d1 >= 0 || p0.d2 <= 0) return 0; /* not a descent direction */
  real lo = 0, hi = -1, alpha = -p0.d1 / p0.d2, best = 0, bestcost = p0.cost;
  for (int it = 0; it < maxit; it++) {
    LsPoint p = ls_eval(s, alpha, jar, jv, qg);
    if (p.cost <= bestcost) { bestcost = p.cost; best = alpha; } /* never accept an increase (round-off only) */
    if (fabs(p.d1) < gtol) break;
    if (p.d1 < 0) lo = alpha; else hi = alpha;
    real next = alpha - p.d1 / p.d2;
    if (hi > 0 && (next <= lo || next >= hi)) next = 0.5 * (lo + hi);
    if (next == alpha) break;
    alpha = next;
  }
  return best;
}

static void solve_newton(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  int nv = s->nv, ne = s->nefc;
  real tol = m->opt[B200_OPT_TOLERANCE], meaninertia = m->opt[B200_OPT_MEANINERTIA];
  real scale = 1.0 / (meaninertia * (nv > 1 ? nv : 1));
  real *Ma = dalloc(nv), *jar = dalloc(ne), *force = dalloc(ne), *grad = dalloc(nv), *search = dalloc(nv), *Mv = dalloc(nv),
       *jv = dalloc(ne), *H = dalloc((size_t)nv * nv), *Lh = dalloc((size_t)nv * nv), *tmp = dalloc(nv);
  int* active = (int*)calloc(ne + 1, sizeof(int));
  real* qacc = s->qacc;
#define MULM(out, vec) for (int i_ = 0; i_ < nv; i_++) { real a_ = 0; for (int j_ = 0; j_ < nv; j_++) a_ += s->M[i_ * nv + j_] * (vec)[j_]; (out)[i_] = a_; }
#define MULJ(out, vec) for (int i_ = 0; i_ < ne; i_++) { real a_ = 0; for (int j_ = 0; j_ < nv; j_++) a_ += s->J[(size_t)i_ * nv + j_] * (vec)[j_]; (out)[i_] = a_; }
  /* warm start: pick the cheaper of qacc_warmstart and qacc_smooth */
  real cost_ws = 0, cost_sm = 0;
  for (int pass = 0; pass < 2; pass++) {
    const real* cand = pass == 0 ? s->qacc_warmstart : s->qacc_smooth;
    MULM(Ma, cand);
    MULJ(jar, cand);
    for (int i = 0; i < ne; i++) jar[i] -= s->efc_aref[i];
    real c = constraint_update(s, jar, force, active);
    for (int i = 0; i < nv; i++) c += 0.5 * (Ma[i] - s->qfrc_smooth[i]) * (cand[i] - s->qacc_smooth[i]);
    if (pass == 0) cost_ws = c; else cost_sm = c;
  }
  int use_ws = m->opt_int[B200_OPTI_WARMSTART] && cost_ws < cost_sm;
  memcpy(qacc, use_ws ? s->qacc_warmstart : s->qacc_smooth, sizeof(real) * nv);
  MULM(Ma, qacc);
  MULJ(jar, qacc);
  for (int i = 0; i < ne; i++) jar[i] -= s->efc_aref[i];
  real cost = 0;
  int iter = 0;
  for (;; iter++) {
    real ccost = constraint_update(s, jar, force, active);
    real gauss = 0;
    for (int i = 0; i < nv; i++) gauss += 0.5 * (Ma[i] - s->qfrc_smooth[i]) * (qacc[i] - s->qacc_smooth[i]);
    real newcost = ccost + gauss;
    /* gradient and Newton direction */
    for (int i = 0; i < nv; i++) {
      real a = Ma[i] - s->qfrc_smooth[i];
      for (int r = 0; r < ne; r++) a -= s->J[(size_t)r * nv + i] * force[r];
      grad[i] = a;
    }
    real gnorm = 0;
    for (int i = 0; i < nv; i++) gnorm += grad[i] * grad[i];
    gnorm = sqrt(gnorm);
    if (iter > 0) {
      real improvement = scale * (cost - newcost), gradient = scale * gnorm;
      cost = newcost;
      if (improvement < tol || gradient < tol) break;
    } else cost = newcost;
    if (iter >= m->opt_int[B200_OPTI_ITERATIONS]) break;
    memcpy(H, s->M, sizeof(real) * nv * nv);
    for (int r = 0; r < ne; r++) {
      if (!active[r]) continue;
      const real* Jr = s->J + (size_t)r * nv;
      real D = s->efc_D[r];
      for (int i = 0; i < nv; i++) {
        if (Jr[i] == 0) continue;
        real di = D * Jr[i];
        for (int j = 0; j < nv; j++) H[i * nv + j] += di * Jr[j];
      }
    }
    cholesky(Lh, H, nv);
    chol_solve(tmp, Lh, grad, nv);
    for (int i = 0; i < nv; i++) search[i] = -tmp[i];
    /* line search */
    MULM(Mv, search);
    MULJ(jv, search);
    real qg[3] = {gauss, 0, 0}, snorm = 0;
    for (int i = 0; i < nv; i++) { qg[1] += search[i] * (Ma[i] - s->qfrc_smooth[i]); qg[2] += 0.5 * search[i] * Mv[i]; snorm += search[i] * search[i]; }
    snorm = sqrt(snorm);
    if (snorm < MINVAL) break;
    real gtol = tol * m->opt[B200_OPT_LS_TOLERANCE] * snorm / scale;
    real alpha = linesearch(s, jar, jv, qg, gtol, m->opt_int[B200_OPTI_LS_ITERATIONS]);
    if (alpha == 0) break;
    for (int i = 0; i < nv; i++) { qacc[i] += alpha * search[i]; Ma[i] += alpha * Mv[i]; }
    for (int i = 0; i < ne; i++) jar[i] += alpha * jv[i];
  }
  s->solver_iter = iter;
  s->total_newton_iter += iter;
  constraint_update(s, jar, force, active);
  memcpy(s->efc_force, force, sizeof(real) * ne);
  for (int i = 0; i < nv; i++) {
    real a = 0;
    for (int r = 0; r < ne; r++) a += s->J[(size_t)r * nv + i] * force[r];
    s->qfrc_constraint[i] = a;
  }
  free(Ma); free(jar); free(force); free(grad); free(search); free(Mv); free(jv); free(H); free(Lh); free(tmp); free(active);
#undef MULM
#undef MULJ
}

/* 8b. Noslip post-pass [ext: mj_solNoSlip, enabled by <option noslip_iterations="N"> -- the Adroit models ask for 20,
 * gymnasium_robotics/envs/assets/adroit_hand/adroit_assets.xml:3].  After the main solve the forces of the FRICTION dimensions are
 * re-solved by projected Gauss-Seidel on the UNREGULARISED dual problem min_f 1/2 f^T A f + f^T b, A = J M^-1 J^T (no R on the
 * diagonal), b = J qacc_smooth - aref, everything else held fixed:
 *   - dof frictionloss rows: one-dimensional Newton step, clamped to [-frictionloss, +frictionloss];
 *   - pyramidal contacts: for every pair of opposing edges (f+, f-) of a friction direction the sum f+ + f- (their share of the
 *     normal force) is kept and the difference is re-solved on the segment |y| <= mid, f+ = mid + y, f- = mid - y
 *     (K1 = A++ + A-- - 2 A+-, K0 = mid (A++ - A--) + bc+ - bc-, y = -K0 / K1);
 *   - limit rows, equality rows and frictionless contacts are not touched.
 * Stops after N sweeps or when the cost decrease of a sweep, scaled by 1 / (meaninertia max(1, nv)), falls under noslip_tolerance
 * (1e-6, MuJoCo's default).  Restated from memory of the published algorithm (SURVEY.md Appendix B.1 grades it LOW confidence);
 * pinned here by a closed-form stick test (tests/test_oracle_physics.py).  `oracle_set_noslip(s, 0)` switches it off so that
 * the CUDA path, which does not run the pass (DESIGN.md deviation 12), can be compared like for like. */
static void solve_noslip(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  int nv = s->nv, ne = s->nefc, niter = m->opt_int[B200_OPTI_NOSLIP_ITERATIONS];
  if (niter <= 0 || ne == 0 || !s->noslip_enabled) return;
  int any = 0;
  for (int i = 0; i < ne; i++) if (s->efc_type[i] == ROW_FRICTION) any = 1;
  for (int c = 0; c < s->ncon; c++) if (s->con[c].efc_address >= 0 && s->con[c].dim > 1) any = 1;
  if (!any) return;
  real *X = dalloc((size_t)ne * nv), *A = dalloc((size_t)ne * ne), *b = dalloc(ne), *f = dalloc(ne);
  for (int i = 0; i < ne; i++) chol_solve(X + (size_t)i * nv, s->L, s->J + (size_t)i * nv, nv);   /* X_i = M^-1 J_i^T */
  for (int i = 0; i < ne; i++)
    for (int j = 0; j < ne; j++) {
      real a = 0;
      for (int d = 0; d < nv; d++) a += s->J[(size_t)i * nv + d] * X[(size_t)j * nv + d];
      A[(size_t)i * ne + j] = a;
    }
  for (int i = 0; i < ne; i++) {
    real a = -s->efc_aref[i];
    for (int d = 0; d < nv; d++) a += s->J[(size_t)i * nv + d] * s->qacc_smooth[d];
    b[i] = a; f[i] = s->efc_force[i];
  }
  real scale = 1.0 / (m->opt[B200_OPT_MEANINERTIA] * (nv > 1 ? nv : 1));
#define RES(i) ({ real r_ = b[i]; for (int j_ = 0; j_ < ne; j_++) r_ += A[(size_t)(i) * ne + j_] * f[j_]; r_; })
  int it = 0;
  for (; it < niter; it++) {
    real improvement = 0;
    for (int i = 0; i < ne; i++) {
      if (s->efc_type[i] != ROW_FRICTION) continue;
      real Aii = A[(size_t)i * ne + i];
      if (Aii < MINVAL) continue;
      real res = RES(i), old = f[i], fl = s->efc_floss[i];
      real nw = old - res / Aii;
      if (nw < -fl) nw = -fl; else if (nw > fl) nw = fl;
      real d = nw - old;
      f[i] = nw;
      improvement -= 0.5 * d * d * Aii + d * res;
    }
    for (int c = 0; c < s->ncon; c++) {
      const Contact* con = &s->con[c];
      if (con->efc_address < 0 || con->dim == 1) continue;
      for (int k = 1; k < con->dim; k++) {
        int j = con->efc_address + 2 * (k - 1);
        real A00 = A[(size_t)j * ne + j], A11 = A[(size_t)(j + 1) * ne + j + 1], A01 = A[(size_t)j * ne + j + 1];
        real r0 = RES(j), r1 = RES(j + 1), o0 = f[j], o1 = f[j + 1];
        real bc0 = r0 - A00 * o0 - A01 * o1, bc1 = r1 - A01 * o0 - A11 * o1;
        real mid = 0.5 * (o0 + o1), K1 = A00 + A11 - 2 * A01, K0 = mid * (A00 - A11) + bc0 - bc1;
        real n0, n1;
        if (K1 < MINVAL) { n0 = n1 = mid; }
        else {
          real y = -K0 / K1;
          if (y < -mid) { n0 = 0; n1 = 2 * mid; } else if (y > mid) { n0 = 2 * mid; n1 = 0; } else { n0 = mid + y; n1 = mid - y; }
        }
        real d0 = n0 - o0, d1 = n1 - o1;
        f[j] = n0; f[j + 1] = n1;
        improvement -= 0.5 * (d0 * d0 * A00 + d1 * d1 * A11 + 2 * d0 * d1 * A01) + d0 * r0 + d1 * r1;
      }
    }
    if (improvement * scale < 1e-6) { it++; break; }
  }
#undef RES
  s->noslip_iter = it;
  memcpy(s->efc_force, f, sizeof(real) * ne);
  for (int d = 0; d < nv; d++) {
    real a = 0;
    for (int r = 0; r < ne; r++) a += s->J[(size_t)r * nv + d] * f[r];
    s->qfrc_constraint[d] = a;
  }
  /* qacc = qacc_smooth + M^-1 qfrc_constraint */
  real* t = dalloc(nv);
  chol_solve(t, s->L, s->qfrc_constraint, nv);
  for (int d = 0; d < nv; d++) s->qacc[d] = s->qacc_smooth[d] + t[d];
  free(t); free(X); free(A); free(b); free(f);
}

/* 9. touch sensors (public MuJoCo semantics): sum of the normal forces of the active contacts that involve the sensor's
 * body and whose ray -- from the contact point along the contact normal, flipped when the sensor's body is the second
 * body -- hits the site volume (always true for a contact point inside the volume).  Site shapes: sphere, box. */
static int ray_hits_site(int type, const double* size, const real* p, const real* d) { /* p, d in the site frame */
  if (type == B200_GEOM_SPHERE) {
    real r = size[0], b = dot3(p, d), c = dot3(p, p) - r * r;
    if (c <= 0) return 1;              /* starts inside */
    real disc = b * b - c;
    return disc >= 0 && -b >= 0;       /* nearest root t = -b - sqrt(disc) >= 0 when the ray points at the sphere */
  }
  if (type == B200_GEOM_CYLINDER) { /* slab |z| <= half length, then x^2 + y^2 <= r^2 over the slab's interval */
    real t0 = 0, t1 = 1e30, r = size[0], hl = size[1];
    if (fabs(d[2]) < 1e-12) { if (fabs(p[2]) > hl) return 0; }
    else {
      real a = (-hl - p[2]) / d[2], b = (hl - p[2]) / d[2];
      if (a > b) { real t = a; a = b; b = t; }
      if (a > t0) t0 = a;
      if (b < t1) t1 = b;
      if (t0 > t1) return 0;
    }
    real A = d[0] * d[0] + d[1] * d[1], B = p[0] * d[0] + p[1] * d[1], C = p[0] * p[0] + p[1] * p[1] - r * r;
    if (A < 1e-20) return C <= 0;
    real disc = B * B - A * C;
    if (disc < 0) return 0;
    real sq = sqrt(disc), ta = (-B - sq) / A, tb = (-B + sq) / A;
    return (t0 > ta ? t0 : ta) <= (t1 < tb ? t1 : tb);
  }
  /* box: slab test for t >= 0 */
  real t0 = 0, t1 = 1e30;
  for (int k = 0; k < 3; k++) {
    if (fabs(d[k]) < 1e-12) { if (fabs(p[k]) > size[k]) return 0; continue; }
    real a = (-size[k] - p[k]) / d[k], b = (size[k] - p[k]) / d[k];
    if (a > b) { real t = a; a = b; b = t; }
    if (a > t0) t0 = a;
    if (b < t1) t1 = b;
    if (t0 > t1) return 0;
  }
  return 1;
}
static void sensors(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  for (int k = 0; k < m->nsensor; k++) {
    int site = m->sensor_site[k], body = m->sensor_body[k];
    int type = m->n_sensor_type == m->nsensor ? m->sensor_type[k] : B200_GEOM_BOX;
    real total = 0;
    for (int c = 0; c < s->ncon; c++) {
      Contact* con = &s->con[c];
      if (con->efc_address < 0 || (con->body1 != body && con->body2 != body)) continue;
      int nrow = con->dim == 1 ? 1 : 2 * (con->dim - 1);
      real fn = 0;
      for (int r = 0; r < nrow; r++) fn += s->efc_force[con->efc_address + r];
      if (fn <= 0) continue;
      real rel[3], loc[3], dir[3], dl[3];
      sub3(rel, con->pos, s->site_xpos + 3 * site);
      mulmatTvec3(loc, s->site_xmat + 9 * site, rel);
      real sg = con->body2 == body ? -1 : 1;
      for (int a = 0; a < 3; a++) dir[a] = sg * con->frame[a];
      mulmatTvec3(dl, s->site_xmat + 9 * site, dir);
      if (!ray_hits_site(type, m->sensor_size + 3 * k, loc, dl)) continue;
      total += fn;
    }
    s->sensordata[k] = total;
  }
}

/* ------------------------------------------------------------------------------------------------ */
void oracle_forward(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  int nv = s->nv;
  kinematics(s);
  com_pos(s);
  tendons(s);
  crb(s);
  collision(s);
  make_constraint(s);
  com_vel(s);
  passive(s);
  rne_bias(s);
  actuation(s);
  for (int i = 0; i < nv; i++) s->qfrc_smooth[i] = s->qfrc_passive[i] - s->qfrc_bias[i] + s->qfrc_actuator[i];
  cholesky(s->L, s->M, nv);
  chol_solve(s->qacc_smooth, s->L, s->qfrc_smooth, nv);
  if (s->nefc == 0) {
    memcpy(s->qacc, s->qacc_smooth, sizeof(real) * nv);
    memset(s->qfrc_constraint, 0, sizeof(real) * nv);
    s->solver_iter = 0;
  } else {
    /* reference acceleration */
    for (int i = 0; i < s->nefc; i++) {
      real v = 0;
      for (int d = 0; d < nv; d++) v += s->J[(size_t)i * nv + d] * s->qvel[d];
      s->efc_vel[i] = v;
      s->efc_aref[i] = -s->efc_KBIP[i][1] * v - s->efc_KBIP[i][0] * s->efc_KBIP[i][2] * (s->efc_pos[i] - s->efc_margin[i]);
    }
    solve_newton(s);
    solve_noslip(s);
  }
  sensors(s);
  (void)m;
}

static void integrate_pos(oracle_sim* s, real* qpos, const real* qvel, real h) {
  const b200_model_view* m = &s->m;
  for (int j = 0; j < m->njnt; j++) {
    int a = m->jnt_qposadr[j], d = m->jnt_dofadr[j];
    if (m->jnt_type[j] == B200_JNT_FREE) {
      for (int k = 0; k < 3; k++) qpos[a + k] += h * qvel[d + k];
      real w[3] = {qvel[d + 3], qvel[d + 4], qvel[d + 5]};
      real ang = normalize3(w) * h;
      if (ang != 0) {
        real dq[4], nq[4];
        axisangle2quat(dq, w, ang);
        mulquat(nq, qpos + a + 3, dq);
        memcpy(qpos + a + 3, nq, sizeof(nq));
      }
      normalize4(qpos + a + 3);
    } else qpos[a] += h * qvel[d];
  }
}

static void euler(oracle_sim* s) {
  const b200_model_view* m = &s->m;
  int nv = s->nv;
  real h = m->opt[B200_OPT_TIMESTEP];
  int damped = 0;
  for (int d = 0; d < nv; d++) if (m->dof_damping[d] > 0) damped = 1;
  real* qacc = dalloc(nv);
  if (damped) {
    real *A = dalloc((size_t)nv * nv), *L = dalloc((size_t)nv * nv), *rhs = dalloc(nv);
    memcpy(A, s->M, sizeof(real) * nv * nv);
    for (int d = 0; d < nv; d++) { A[d * nv + d] += h * m->dof_damping[d]; rhs[d] = s->qfrc_smooth[d] + s->qfrc_constraint[d]; }
    cholesky(L, A, nv);
    chol_solve(qacc, L, rhs, nv);
    free(A); free(L); free(rhs);
  } else memcpy(qacc, s->qacc, sizeof(real) * nv);
  for (int d = 0; d < nv; d++) s->qvel[d] += h * qacc[d];
  integrate_pos(s, s->qpos, s->qvel, h);
  s->time += h;
  memcpy(s->qacc_warmstart, s->qacc, sizeof(real) * nv);
  free(qacc);
}

static void rk4(oracle_sim* s) {
  /* classical RK4 over (qpos, qvel); one full forward per stage; ctrl held constant */
  const b200_model_view* m = &s->m;
  int nv = s->nv, nq = s->nq;
  real h = m->opt[B200_OPT_TIMESTEP];
  static const real A[3] = {0.5, 0.5, 1.0}, B[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};
  real *q0 = dalloc(nq), *v0 = dalloc(nv), *X[4], *F[4], *dX = dalloc(nv), *dF = dalloc(nv);
  for (int i = 0; i < 4; i++) { X[i] = dalloc(nv); F[i] = dalloc(nv); }
  memcpy(q0, s->qpos, sizeof(real) * nq); memcpy(v0, s->qvel, sizeof(real) * nv);
  real t0 = s->time;
  memcpy(X[0], s->qvel, sizeof(real) * nv); memcpy(F[0], s->qacc, sizeof(real) * nv);
  for (int i = 1; i < 4; i++) {
    memcpy(s->qpos, q0, sizeof(real) * nq);
    integrate_pos(s, s->qpos, X[i - 1], A[i - 1] * h);
    for (int d = 0; d < nv; d++) s->qvel[d] = v0[d] + A[i - 1] * h * F[i - 1][d];
    memcpy(X[i], s->qvel, sizeof(real) * nv);
    s->time = t0 + A[i - 1] * h;
    oracle_forward(s);
    memcpy(F[i], s->qacc, sizeof(real) * nv);
  }
  memset(dX, 0, sizeof(real) * nv); memset(dF, 0, sizeof(real) * nv);
  for (int i = 0; i < 4; i++) for (int d = 0; d < nv; d++) { dX[d] += B[i] * X[i][d]; dF[d] += B[i] * F[i][d]; }
  memcpy(s->qpos, q0, sizeof(real) * nq);
  for (int d = 0; d < nv; d++) s->qvel[d] = v0[d] + h * dF[d];
  integrate_pos(s, s->qpos, dX, h);
  s->time = t0 + h;
  memcpy(s->qacc_warmstart, s->qacc, sizeof(real) * nv);
  for (int i = 0; i < 4; i++) { free(X[i]); free(F[i]); }
  free(q0); free(v0); free(dX); free(dF);
}

void oracle_step(oracle_sim* s, int nstep) {
  for (int k = 0; k < nstep; k++) {
    oracle_forward(s);
    if (s->m.opt_int[B200_OPTI_INTEGRATOR] == B200_INT_RK4) rk4(s); else euler(s);
    s->total_substeps++;
  }
}

/* ------------------------------------------------------------------------------------------------ */
/* accessors for the ctypes wrapper */
#define ACC(name, field) real* oracle_##name(oracle_sim* s) { return s->field; }
ACC(qpos, qpos) ACC(qvel, qvel) ACC(ctrl, ctrl) ACC(mocap_pos, mocap_pos) ACC(mocap_quat, mocap_quat)
ACC(qacc_warmstart, qacc_warmstart) ACC(qacc, qacc) ACC(xpos, xpos) ACC(xquat, xquat) ACC(xmat, xmat)
ACC(site_xpos, site_xpos) ACC(site_xmat, site_xmat) ACC(geom_xpos, geom_xpos) ACC(geom_xmat, geom_xmat)
ACC(eq_data, eq_data) ACC(act_gainprm, act_gainprm) ACC(act_biasprm, act_biasprm) ACC(body_pos, body_pos) ACC(body_quat, body_quat)
ACC(M, M) ACC(qfrc_bias, qfrc_bias) ACC(qfrc_smooth, qfrc_smooth) ACC(qacc_smooth, qacc_smooth)
ACC(qfrc_constraint, qfrc_constraint) ACC(efc_J, J) ACC(efc_force, efc_force) ACC(efc_aref, efc_aref)
ACC(efc_pos, efc_pos) ACC(efc_D, efc_D) ACC(efc_R, efc_R) ACC(sensordata, sensordata) ACC(subtree_com, subtree_com)
ACC(cdof, cdof) ACC(qfrc_actuator, qfrc_actuator) ACC(qfrc_passive, qfrc_passive)
real* oracle_time(oracle_sim* s) { return &s->time; }
/* per constraint row: type (ROW_*), object (equality, dof, joint or njnt + tendon, contact), and K, B, imp, impP of aref */
int* oracle_efc_type(oracle_sim* s) { return s->efc_type; }
int* oracle_efc_id(oracle_sim* s) { return s->efc_id; }
real* oracle_efc_KBIP(oracle_sim* s) { return &s->efc_KBIP[0][0]; }
real* oracle_efc_margin(oracle_sim* s) { return s->efc_margin; }
/* translational and rotational Jacobian (3 x nv each) of a point fixed to a body, at the current kinematics */
void oracle_jac_point(const oracle_sim* s, int body, const real* point, real* jacp, real* jacr) { jac_point(s, body, point, jacp, jacr); }
int oracle_ncon(const oracle_sim* s) { return s->ncon; }
int oracle_nefc(const oracle_sim* s) { return s->nefc; }
int oracle_solver_iter(const oracle_sim* s) { return s->solver_iter; }
long oracle_total_newton_iter(const oracle_sim* s) { return s->total_newton_iter; }
int oracle_overflow(const oracle_sim* s) { return s->warn_overflow; }
void oracle_set_noslip(oracle_sim* s, int on) { s->noslip_enabled = on ? 1 : 0; }
int oracle_noslip_iter(const oracle_sim* s) { return s->noslip_iter; }
int oracle_size(const oracle_sim* s, int which) { return s->m.sizes[which]; }
/* Per-body external contact force, the contact part of mj_rnePostConstraint [ext] (Gymnasium's Ant-v5 calls it after mj_step and
 * reads data.cfrc_ext: gymnasium_robotics/envs/maze/ant_maze_v5.py:99 "(105,) = 27 + 13 x 6"): for every contact with constraint
 * rows, the contact force in the contact frame (mj_contactForce: pyramid edges f -> normal = sum f, friction k = mu_k (f+ - f-))
 * rotated to world axes, taken as a spatial force [torque; force] about the subtree com of the body's tree root, subtracted from
 * the first body and added to the second.  out: nbody x 6. */
void oracle_cfrc_ext(const oracle_sim* s, real* out) {
  const b200_model_view* m = &s->m;
  /* rows = MJCF (unfused) bodies when the blob carries the tables, else the runtime bodies */
  const int rows = m->n_mjbody_rt > 0 ? m->n_mjbody_rt : s->nbody;
  memset(out, 0, sizeof(real) * 6 * rows);
  for (int c = 0; c < s->ncon; c++) {
    const Contact* con = &s->con[c];
    if (con->efc_address < 0) continue;
    real f[6] = {0, 0, 0, 0, 0, 0};
    if (con->dim == 1) f[0] = s->efc_force[con->efc_address];
    else for (int k = 1; k < con->dim; k++) {
      real fp = s->efc_force[con->efc_address + 2 * (k - 1)], fm = s->efc_force[con->efc_address + 2 * (k - 1) + 1];
      f[0] += fp + fm; f[k] = con->friction[k - 1] * (fp - fm);
    }
    real F[3] = {0, 0, 0}, T[3] = {0, 0, 0};
    for (int a = 0; a < 3; a++) { addscl3(F, con->frame + 3 * a, f[a]); addscl3(T, con->frame + 3 * a, f[3 + a]); }
    for (int side = 0; side < 2; side++) {
      int rb = side ? con->body2 : con->body1, g = side ? con->geom2 : con->geom1;
      if (rb == 0) continue;
      int row = (m->n_geom_mjbody == s->ngeom && g >= 0) ? m->geom_mjbody[g] : rb;
      real sg = side ? 1 : -1, r[3], tq[3];
      sub3(r, con->pos, s->subtree_com + 3 * m->body_rootid[rb]);
      cross3(tq, r, F);
      for (int a = 0; a < 3; a++) { out[6 * row + a] += sg * (T[a] + tq[a]); out[6 * row + 3 + a] += sg * F[a]; }
    }
  }
}
int oracle_cfrc_rows(const oracle_sim* s) { return s->m.n_mjbody_rt > 0 ? s->m.n_mjbody_rt : s->nbody; }
/* contact k -> out[0]=dist, out[1:4]=pos, out[4:13]=frame, out[13]=dim, out[14]=geom1, out[15]=geom2, out[16]=efc_address,
 * out[17]=pair */
void oracle_contact(const oracle_sim* s, int k, real* out) {
  const Contact* c = &s->con[k];
  out[0] = c->dist; memcpy(out + 1, c->pos, 3 * sizeof(real)); memcpy(out + 4, c->frame, 9 * sizeof(real));
  out[13] = c->dim; out[14] = c->geom1; out[15] = c->geom2; out[16] = c->efc_address; out[17] = c->pair;
}
/* the collision stage alone, from the current geom_xpos / geom_xmat (no kinematics): the contact list that contacts() reads.
 * Tests of the narrow phase set the geom poses directly, so that both sides collide exactly the same inputs. */
void oracle_collision(oracle_sim* s) { collision(s); }
