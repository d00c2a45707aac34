// b200sim physics core: one warp integrates one env.  Hand-written for sm_90a; the same source compiles on the
// host with WARP_W == 1 for the test-only emulation harness in tests/hostsim (never part of the product library).
//
// Replaces `mujoco.mj_step(model, data, nstep=n_substeps)` (reference: gymnasium_robotics/envs/robot_env.py:340-341)
// for the model features listed in DESIGN.md.  Formulation (differs from the oracle on purpose):
//   * spatial quantities are expressed about one fixed world point `ref` (not per-tree subtree coms);
//   * kinematics by pointer jumping over the body tree (log depth);
//   * tree recursions (CRB, velocities, RNE, J*v, J^T f) via ancestor / subtree bit masks, no sequential passes;
//   * constraint Jacobian is never materialised: each base row is a spatial 6-vector `w` plus a body pair, pyramid
//     edges are combinations of a contact's base rows, and H = M + J^T D J is assembled from per-body-pair 6x6 blocks;
//   * dense packed Cholesky for H and for (M + h*B).
#pragma once
#include "dmodel.h"

// B200_WARP_CODE: the 32-lane code paths (shuffle reductions, scans, the register Cholesky).  nvcc compiles them for the device;
// the test-only build -DB200_HOST_WARP (tests/hostsim/hostwarp.h) compiles the same lines for the host with the warp intrinsics
// emulated by 32 lock-step fibers, so that the CPU suite can execute the lane-parallel logic itself, not only its WARP_W == 1
// counterpart.
#if defined(__CUDACC__) || defined(B200_HOST_WARP)
#define B200_WARP_CODE 1
#endif
#ifdef __CUDACC__
// internal linkage: b200sim.cu and b200sim_wide.cu compile these sources with different dof-mask widths
#define HD static __device__ __forceinline__
#define HDN static __device__ __noinline__
#define STAGE static __device__ __noinline__  // pipeline stages are real calls: keeps the kernel inside the instruction caches
#define ASSUME_SHARED_PTR(p) __builtin_assume(__isShared(p))
#define ASSUME_SHARED(c) do { __builtin_assume(__isShared((c).s)); __builtin_assume(__isShared((c).mw)); __builtin_assume(__isShared((c).h)); } while (0)
#define WARP_W 32
#define SYNC() __syncwarp()
// block-wide alignment points: keep the warps of a block inside the same code window (instruction-cache locality)
#define ALIGN() __syncthreads()
#define ALIGN_OR(p) __syncthreads_or(p)
#elif defined(B200_HOST_WARP)
#define HD static inline
#define HDN static
#define STAGE static
#define ASSUME_SHARED(c) do { } while (0)
#define ASSUME_SHARED_PTR(p) do { } while (0)
#define WARP_W 32
#define SYNC() __syncwarp()
#define ALIGN() __syncwarp()                          // one warp stands for the block
#define ALIGN_OR(p) (__ballot_sync(0xffffffffu, (p)) != 0u)
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
#else
#define HD static inline
#define HDN static
#define STAGE static
#define ASSUME_SHARED(c) do { } while (0)
#define ASSUME_SHARED_PTR(p) do { } while (0)
#define WARP_W 1
#define SYNC() do { } while (0)
#define ALIGN() do { } while (0)
#define ALIGN_OR(p) (p)
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
#endif

#define B200_MINVAL 1e-15f
#define B200_MINIMP 0.0001f
#define B200_MAXIMP 0.9999f

struct Ctx {
  const uint32_t* mg;  // whole model buffer in global memory (COLD arrays are read from here)
  const uint32_t* mw;  // header + HOT arrays staged in shared memory
  const DMHead* h;
  float* s;            // this env's scratch (shared memory)
  int lane;
#ifdef B200_STAGE_TIMING
  long long* tim;      // experiments only: per-thread cycle counters per stage
#endif
};
#ifdef B200_STAGE_TIMING
enum { TM_KIN = 0, TM_COM_M, TM_COLL, TM_CONSTR, TM_SMOOTH, TM_NBEGIN, TM_NCHECK, TM_BUILDH, TM_NDIR, TM_NMOVE, TM_INTEG, TM_BARRIER, TM_OTHER, TM_MV_MULM, TM_MV_ROWS, TM_MV_LS, TM_CK_PASSF, TM_MV_UPD, TM_COUNT };
#define TIC() long long t0_ = clock64()
#define TOC(k) do { long long t1_ = clock64(); c.tim[k] += t1_ - t0_; t0_ = t1_; } while (0)
// the convergence check ends newton_begin and newton_move: its cycles move from that stage's counter to TM_NCHECK
#define CHECK_TIC() long long tc_ = clock64()
#define CHECK_TOC(stage) do { long long d_ = clock64() - tc_; c.tim[TM_NCHECK] += d_; c.tim[stage] -= d_; } while (0)
#else
#define TIC() do { } while (0)
#define TOC(k) do { } while (0)
#define CHECK_TIC() do { } while (0)
#define CHECK_TOC(stage) do { } while (0)
#endif
#ifdef __CUDACC__
// the step kernel's dynamic shared memory (`smem` in step_kernel.cuh): model header + HOT arrays, then one scratch per warp
extern __shared__ __align__(128) uint32_t b200_smem[];
#endif
// The context handed to a stage call by the driver loops (forward(), the sub-step loop of fetch_env_step).  In a block of 28 or
// 32 warps a thread gets at most 72 / 64 registers, and the stages use nearly all of them, so a scratch pointer the driver kept
// live across the ~50 stage calls of a sub-step was spilled to local memory (which, beside a 231 KB shared-memory carve-out, is
// L2) and reloaded after every call.  There (REBUILD) the driver rebuilds the context before each call instead, from the header
// words in shared memory and the warp index.  With 128 registers nothing is spilled and the rebuild only adds instructions
// (FetchPickAndPlace at 32 warps: -6 % step-kernel time; the 7..16-warp kernels were slower with it, DESIGN.md section 6).
template <bool REBUILD>
HD Ctx stage_ctx(const Ctx& c) {
#ifdef __CUDACC__
  if (REBUILD) {
    // (%tid.x read afresh: threadIdx.x would be merged with the kernel's own lane and warp values, which then stay live)
    uint32_t tid;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
    Ctx r = c;
    const DMHead* h = (const DMHead*)b200_smem;
    r.s = (float*)(b200_smem + h->hot_words) + (tid >> 5) * h->scr_words;
    r.lane = (int)(tid & 31);
    return r;
  }
#endif
  return c;
}
#define MI(name) ((const int*)(c.mw + c.h->o_##name))
#define MU(name) ((const uint32_t*)(c.mw + c.h->o_##name))
#define MF(name) ((const float*)(c.mw + c.h->o_##name))
#ifdef B200_KITCHEN_GROUPS
#define PAIR_I(name) ((const int*)(c.mg + c.h->o_##name))    // two-level kitchen build: the pair list stays in global memory (dmodel.h)
#define PAIR_F(name) ((const float*)(c.mg + c.h->o_##name))
#else
#define PAIR_I(name) MI(name)
#define PAIR_F(name) MF(name)
#endif
#define GI(name) ((const int*)(c.mg + c.h->o_##name))
#define GF(name) ((const float*)(c.mg + c.h->o_##name))
#define SF(name) (c.s + c.h->s_##name)
#define SI(name) ((int*)(c.s + c.h->s_##name))
#define LANES(i, n) for (int i = c.lane; i < (n); i += WARP_W)

// ---------------------------------------------------------------------------------------------------------------
// warp helpers
HD float wsum(float v) {
#ifdef B200_WARP_CODE
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
  return v;
}
HD float wmax(float v) {
#ifdef B200_WARP_CODE
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
#endif
  return v;
}
HD int wsumi(int v) {
#ifdef B200_WARP_CODE
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
  return v;
}
// exclusive prefix sum of v over lanes; *total = sum
HD int wexscan(int v, int lane, int* total) {
#ifdef B200_WARP_CODE
  int x = v;
  for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  *total = __shfl_sync(0xffffffffu, x, 31);
  return x - v;
#else
  (void)lane; *total = v; return 0;
#endif
}
HD int ffs_pop(uint32_t& m) {  // index of lowest set bit, and clear it
#ifdef __CUDACC__
  int b = __ffs(m) - 1;
#else
  int b = __builtin_ctz(m);
#endif
  m &= m - 1;
  return b;
}
// dof masks: 32 bits in the ordinary builds, 64 bits in the wide build (B200_WIDE: models with 33..40 dofs, stored as two
// words per entry in the model tables and in the group records); body masks stay 32 bits (<= 32 runtime bodies)
#ifdef B200_WIDE
typedef unsigned long long dmask_t;
HD int ffs_pop(dmask_t& m) {
#ifdef __CUDACC__
  int b = __ffsll((long long)m) - 1;
#else
  int b = __builtin_ctzll(m);
#endif
  m &= m - 1;
  return b;
}
#define DM(name, i) ((dmask_t)MU(name)[2 * (i)] | ((dmask_t)MU(name)[2 * (i) + 1] << 32))
HD dmask_t grp_mask(const float* gr) { const uint32_t* u = (const uint32_t*)gr; return (dmask_t)u[G_MASK] | ((dmask_t)u[G_MASK + 1] << 32); }
HD dmask_t grp_sign(const float* gr) { const uint32_t* u = (const uint32_t*)gr; return (dmask_t)u[G_SIGN] | ((dmask_t)u[G_SIGN + 1] << 32); }
HD void grp_set_masks(int* gi, dmask_t mask, dmask_t sign) {
  uint32_t* u = (uint32_t*)gi;
  u[G_MASK] = (uint32_t)mask; u[G_MASK + 1] = (uint32_t)(mask >> 32); u[G_SIGN] = (uint32_t)sign; u[G_SIGN + 1] = (uint32_t)(sign >> 32);
}
#else
typedef uint32_t dmask_t;
#define DM(name, i) (MU(name)[i])
HD dmask_t grp_mask(const float* gr) { return ((const uint32_t*)gr)[G_MASK]; }
HD dmask_t grp_sign(const float* gr) { return ((const uint32_t*)gr)[G_SIGN]; }
HD void grp_set_masks(int* gi, dmask_t mask, dmask_t sign) { ((uint32_t*)gi)[G_MASK] = mask; ((uint32_t*)gi)[G_SIGN] = sign; }
#endif
#define DBIT(m, j) ((int)(((m) >> (j)) & 1))
// G_RANGE of a group record: first contact (8 bits), contact count (8 bits), MJCF bodies A | B << 8 (16 bits)
HD int grp_start(const float* gr) { return ((const int*)gr)[G_RANGE] & 0xff; }
HD int grp_count(const float* gr) { return (((const int*)gr)[G_RANGE] >> 8) & 0xff; }
HD int grp_bodies(const float* gr) { return (int)(((const uint32_t*)gr)[G_RANGE] >> 16); }

// ---------------------------------------------------------------------------------------------------------------
// small math
HD float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
HD void cross3(float* r, const float* a, const float* b) {
  float x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
HD float dot6(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5]; }
HD void qmul(float* r, const float* a, const float* b) {
  float w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  float x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  float y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  float z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
HD void qnormalize(float* q) {
  float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (n < 1e-12f) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  float inv = 1.0f / n;
  q[0] *= inv; q[1] *= inv; q[2] *= inv; q[3] *= inv;
}
HD void q2mat(float* m, const float* q) {
  float w = q[0], x = q[1], y = q[2], z = q[3];
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2 * (x * y - w * z); m[2] = 2 * (x * z + w * y);
  m[3] = 2 * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2 * (y * z - w * x);
  m[6] = 2 * (x * z - w * y); m[7] = 2 * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
HD void qrot(float* r, const float* q, const float* v) {  // r = R(q) v
  float t[3], u[3] = {q[1], q[2], q[3]};
  cross3(t, u, v);
  t[0] = 2 * t[0]; t[1] = 2 * t[1]; t[2] = 2 * t[2];
  float c2[3];
  cross3(c2, u, t);
  r[0] = v[0] + q[0] * t[0] + c2[0]; r[1] = v[1] + q[0] * t[1] + c2[1]; r[2] = v[2] + q[0] * t[2] + c2[2];
}
HD void mulmv(float* r, const float* m, const float* v) {
  float x = m[0] * v[0] + m[1] * v[1] + m[2] * v[2], y = m[3] * v[0] + m[4] * v[1] + m[5] * v[2], z = m[6] * v[0] + m[7] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
HD void mulmtv(float* r, const float* m, const float* v) {
  float x = m[0] * v[0] + m[3] * v[1] + m[6] * v[2], y = m[1] * v[0] + m[4] * v[1] + m[7] * v[2], z = m[2] * v[0] + m[5] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
HD void cross_motion(float* r, const float* v, const float* s) {
  float a[3], b[3], cc[3];
  cross3(a, v, s); cross3(b, v, s + 3); cross3(cc, v + 3, s);
  r[0] = a[0]; r[1] = a[1]; r[2] = a[2]; r[3] = b[0] + cc[0]; r[4] = b[1] + cc[1]; r[5] = b[2] + cc[2];
}
HD void cross_force(float* r, const float* v, const float* f) {
  float a[3], b[3], cc[3];
  cross3(a, v, f); cross3(b, v + 3, f + 3); cross3(cc, v, f + 3);
  r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2]; r[3] = cc[0]; r[4] = cc[1]; r[5] = cc[2];
}
HD void mul_inert(float* res, const float* I, const float* v) {  // 10-number inertia about `ref`
  const float* mo = I + 6;
  float t[3];
  res[0] = I[0] * v[0] + I[3] * v[1] + I[4] * v[2];
  res[1] = I[3] * v[0] + I[1] * v[1] + I[5] * v[2];
  res[2] = I[4] * v[0] + I[5] * v[1] + I[2] * v[2];
  cross3(t, mo, v + 3);
  res[0] += t[0]; res[1] += t[1]; res[2] += t[2];
  cross3(t, v, mo);
  res[3] = I[9] * v[3] + t[0]; res[4] = I[9] * v[4] + t[1]; res[5] = I[9] * v[5] + t[2];
}
HD int pidx(int i, int j) { return i >= j ? (i * (i + 1)) / 2 + j : (j * (j + 1)) / 2 + i; }

// ---------------------------------------------------------------------------------------------------------------
// 1. kinematics (pointer jumping)
STAGE void kinematics(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  int nb = h->nb;
  float *A = SF(kinA), *B = SF(kinB);
  const float *qpos = SF(qpos);
  LANES(b, nb) {
    float lp[3] = {0, 0, 0}, lq[4] = {1, 0, 0, 0};
    int anc = 0;
    if (b > 0) {
      anc = MI(body_parent)[b];
      int mid = MI(body_mocapid)[b], jn = MI(body_jntnum)[b], ja = MI(body_jntadr)[b];
      if (mid >= 0) {
        for (int k = 0; k < 3; k++) lp[k] = SF(mocap_pos)[3 * mid + k];
        for (int k = 0; k < 4; k++) lq[k] = SF(mocap_quat)[4 * mid + k];
        qnormalize(lq);
      } else if (jn == 1 && MI(jnt_type)[ja] == B200_JNT_FREE) {
        int a = MI(jnt_qposadr)[ja];
        for (int k = 0; k < 3; k++) lp[k] = qpos[a + k];
        for (int k = 0; k < 4; k++) lq[k] = qpos[a + 3 + k];
        qnormalize(lq);
      } else {
        // one body may carry a per-env pose (Adroit: model.body_pos[nail_board] / body_pos[Object] / body_quat[target] are
        // redrawn at every reset): 3 + 4 floats of the state record
        const float* bp = (b == c.h->penv_body) ? SF(penv_pos) : MF(body_pos) + 3 * b;
        const float* bqm = (b == c.h->penv_body) ? SF(penv_pos) + 3 : MF(body_quat) + 4 * b;
        for (int k = 0; k < 3; k++) lp[k] = bp[k];
        for (int k = 0; k < 4; k++) lq[k] = bqm[k];
        for (int j = ja; j < ja + jn; j++) {
          const float* jp = MF(jnt_pos) + 3 * j;
          const float* jax = MF(jnt_axis) + 3 * j;
          float dq = qpos[MI(jnt_qposadr)[j]] - MF(jnt_qpos0)[j];
          if (MI(jnt_type)[j] == B200_JNT_SLIDE) {
            float ax[3];
            qrot(ax, lq, jax);
            lp[0] += ax[0] * dq; lp[1] += ax[1] * dq; lp[2] += ax[2] * dq;
          } else {
            float anc_l[3], t[3], ql[4], nq[4], sn, cs;
#ifdef __CUDACC__
            sincosf(0.5f * dq, &sn, &cs);
#else
            sn = sinf(0.5f * dq); cs = cosf(0.5f * dq);
#endif
            qrot(t, lq, jp);
            anc_l[0] = lp[0] + t[0]; anc_l[1] = lp[1] + t[1]; anc_l[2] = lp[2] + t[2];
            ql[0] = cs; ql[1] = jax[0] * sn; ql[2] = jax[1] * sn; ql[3] = jax[2] * sn;
            qmul(nq, lq, ql);
            lq[0] = nq[0]; lq[1] = nq[1]; lq[2] = nq[2]; lq[3] = nq[3];
            qrot(t, lq, jp);
            lp[0] = anc_l[0] - t[0]; lp[1] = anc_l[1] - t[1]; lp[2] = anc_l[2] - t[2];
          }
        }
      }
    }
    float* o = A + 8 * b;
    o[0] = lp[0]; o[1] = lp[1]; o[2] = lp[2]; o[3] = lq[0]; o[4] = lq[1]; o[5] = lq[2]; o[6] = lq[3];
    ((int*)o)[7] = anc;
  }
  SYNC();
  for (int it = 0; it < h->kin_iters; it++) {
    LANES(b, nb) {
      const float* me = A + 8 * b;
      float* o = B + 8 * b;
      int anc = ((const int*)me)[7];
      if (anc != 0) {
        const float* pa = A + 8 * anc;
        float t[3], q[4];
        qrot(t, pa + 3, me);
        qmul(q, pa + 3, me + 3);
        o[0] = pa[0] + t[0]; o[1] = pa[1] + t[1]; o[2] = pa[2] + t[2];
        o[3] = q[0]; o[4] = q[1]; o[5] = q[2]; o[6] = q[3];
        ((int*)o)[7] = ((const int*)pa)[7];
      } else {
        for (int k = 0; k < 7; k++) o[k] = me[k];
        ((int*)o)[7] = 0;
      }
    }
    SYNC();
    float* t = A; A = B; B = t;
  }
  LANES(b, nb) {
    const float* me = A + 8 * b;
    float q[4] = {me[3], me[4], me[5], me[6]};
    qnormalize(q);
    float* xp = SF(xpos) + 3 * b;
    float* xq = SF(xquat) + 4 * b;
    xp[0] = me[0]; xp[1] = me[1]; xp[2] = me[2];
    xq[0] = q[0]; xq[1] = q[1]; xq[2] = q[2]; xq[3] = q[3];
  }
  SYNC();
}

// 2. spatial inertias and motion axes about `ref`; geom centres
STAGE void com_quantities(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  const float* ref = h->ref;
  LANES(b, h->nb) {
    float* ci = SF(cinert) + 10 * b;
    if (b == 0) { for (int k = 0; k < 10; k++) ci[k] = 0; continue; }
    float ip[3], r[3], iq[4], Ri[9];
    qrot(ip, SF(xquat) + 4 * b, MF(body_ipos) + 3 * b);
    for (int k = 0; k < 3; k++) r[k] = SF(xpos)[3 * b + k] + ip[k] - ref[k];
    qmul(iq, SF(xquat) + 4 * b, MF(body_iquat) + 4 * b);
    q2mat(Ri, iq);
    const float* d = MF(body_inertia) + 3 * b;
    float mass = MF(body_mass)[b];
    float I00 = Ri[0] * d[0] * Ri[0] + Ri[1] * d[1] * Ri[1] + Ri[2] * d[2] * Ri[2];
    float I11 = Ri[3] * d[0] * Ri[3] + Ri[4] * d[1] * Ri[4] + Ri[5] * d[2] * Ri[5];
    float I22 = Ri[6] * d[0] * Ri[6] + Ri[7] * d[1] * Ri[7] + Ri[8] * d[2] * Ri[8];
    float I01 = Ri[0] * d[0] * Ri[3] + Ri[1] * d[1] * Ri[4] + Ri[2] * d[2] * Ri[5];
    float I02 = Ri[0] * d[0] * Ri[6] + Ri[1] * d[1] * Ri[7] + Ri[2] * d[2] * Ri[8];
    float I12 = Ri[3] * d[0] * Ri[6] + Ri[4] * d[1] * Ri[7] + Ri[5] * d[2] * Ri[8];
    float rr = dot3(r, r);
    ci[0] = I00 + mass * (rr - r[0] * r[0]); ci[1] = I11 + mass * (rr - r[1] * r[1]); ci[2] = I22 + mass * (rr - r[2] * r[2]);
    ci[3] = I01 - mass * r[0] * r[1]; ci[4] = I02 - mass * r[0] * r[2]; ci[5] = I12 - mass * r[1] * r[2];
    ci[6] = mass * r[0]; ci[7] = mass * r[1]; ci[8] = mass * r[2]; ci[9] = mass;
  }
  LANES(j, h->njnt) {
    int b = MI(jnt_body)[j], d = MI(jnt_dofadr)[j], t = MI(jnt_type)[j];
    float R[9], bq[4], xp[3];
    for (int k = 0; k < 4; k++) bq[k] = SF(xquat)[4 * b + k];
    for (int k = 0; k < 3; k++) xp[k] = SF(xpos)[3 * b + k];
    // a body with several joints (Adroit: two arm hinges on the forearm, 3 slides + 3 hinges on the hammer): joint j acts
    // in the frame reached before the later joints of the same body, so those are undone from the final body pose
    for (int k = MI(body_jntadr)[b] + MI(body_jntnum)[b] - 1; k > j; k--) {
      float dq = SF(qpos)[MI(jnt_qposadr)[k]] - MF(jnt_qpos0)[k], ax[3];
      if (MI(jnt_type)[k] == B200_JNT_SLIDE) {
        qrot(ax, bq, MF(jnt_axis) + 3 * k);
        xp[0] -= ax[0] * dq; xp[1] -= ax[1] * dq; xp[2] -= ax[2] * dq;
      } else {
        float anc[3], tt[3], ql[4], nq[4], sn, cs;
#ifdef __CUDACC__
        sincosf(-0.5f * dq, &sn, &cs);
#else
        sn = sinf(-0.5f * dq); cs = cosf(-0.5f * dq);
#endif
        qrot(tt, bq, MF(jnt_pos) + 3 * k);
        anc[0] = xp[0] + tt[0]; anc[1] = xp[1] + tt[1]; anc[2] = xp[2] + tt[2];
        const float* ja = MF(jnt_axis) + 3 * k;
        ql[0] = cs; ql[1] = ja[0] * sn; ql[2] = ja[1] * sn; ql[3] = ja[2] * sn;
        qmul(nq, bq, ql);
        bq[0] = nq[0]; bq[1] = nq[1]; bq[2] = nq[2]; bq[3] = nq[3];
        qrot(tt, bq, MF(jnt_pos) + 3 * k);
        xp[0] = anc[0] - tt[0]; xp[1] = anc[1] - tt[1]; xp[2] = anc[2] - tt[2];
      }
    }
    q2mat(R, bq);
    float* cd = SF(cdof) + 6 * d;
    if (t == B200_JNT_FREE) {
      float off[3] = {ref[0] - xp[0], ref[1] - xp[1], ref[2] - xp[2]};
      for (int k = 0; k < 3; k++) { for (int a = 0; a < 6; a++) cd[6 * k + a] = 0; cd[6 * k + 3 + k] = 1; }
      for (int k = 0; k < 3; k++) {
        float ax[3] = {R[k], R[3 + k], R[6 + k]};
        float* o = cd + 6 * (3 + k);
        o[0] = ax[0]; o[1] = ax[1]; o[2] = ax[2];
        cross3(o + 3, ax, off);
      }
    } else {
      float ax[3];
      mulmv(ax, R, MF(jnt_axis) + 3 * j);
      if (t == B200_JNT_SLIDE) { cd[0] = cd[1] = cd[2] = 0; cd[3] = ax[0]; cd[4] = ax[1]; cd[5] = ax[2]; }
      else {
        float jp[3], off[3];
        mulmv(jp, R, MF(jnt_pos) + 3 * j);
        for (int k = 0; k < 3; k++) off[k] = ref[k] - (xp[k] + jp[k]);
        cd[0] = ax[0]; cd[1] = ax[1]; cd[2] = ax[2];
        cross3(cd + 3, ax, off);
      }
    }
  }
  LANES(g, h->ngeom) {
    int b = MI(geom_body)[g];
    float t[3];
    qrot(t, SF(xquat) + 4 * b, MF(geom_pos) + 3 * g);
    for (int k = 0; k < 3; k++) SF(geom_xpos)[3 * g + k] = SF(xpos)[3 * b + k] + t[k];
  }
  SYNC();
}

// 4. mass matrix, packed lower triangle
STAGE void mass_matrix(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  int nv = h->nv, nM = nv * (nv + 1) / 2;
  float* M = SF(M);
  LANES(i, nM) M[i] = 0;
  SYNC();
  LANES(i, nv) {
    float crb[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    uint32_t sub = MU(body_sub)[MI(dof_body)[i]];
    while (sub) { int b = ffs_pop(sub); const float* ci = SF(cinert) + 10 * b; for (int k = 0; k < 10; k++) crb[k] += ci[k]; }
    float buf[6];
    mul_inert(buf, crb, SF(cdof) + 6 * i);
    dmask_t anc = DM(dof_anc, i);
    int row = i * (i + 1) / 2;
    while (anc) { int j = ffs_pop(anc); M[row + j] = dot6(SF(cdof) + 6 * j, buf); }
    M[row + i] += MF(dof_armature)[i];
  }
  SYNC();
}

// velocity pass: b6[b] = sum_{j in ancdof(b)} cdof_j * vec_j
STAGE void pass_V(const Ctx c, const float* vec, float* out) {
  ASSUME_SHARED(c);
  ASSUME_SHARED_PTR(vec); ASSUME_SHARED_PTR(out);
  LANES(b, c.h->nb) {
    float v[6] = {0, 0, 0, 0, 0, 0};
    dmask_t m = DM(body_ancdof, b);
    while (m) { int j = ffs_pop(m); const float* cd = SF(cdof) + 6 * j; float q = vec[j]; for (int k = 0; k < 6; k++) v[k] += cd[k] * q; }
    for (int k = 0; k < 6; k++) out[6 * b + k] = v[k];
  }
  SYNC();
}

// 7. smooth forces: fsmooth = passive - bias + actuation
STAGE void smooth_forces(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  int nv = h->nv, nb = h->nb;
  const float *qvel = SF(qvel), *qpos = SF(qpos);
  LANES(j, nv) {
    float vp[6] = {0, 0, 0, 0, 0, 0}, vj[6];
    dmask_t m = DM(dof_pre, j);
    while (m) { int i = ffs_pop(m); const float* cd = SF(cdof) + 6 * i; float q = qvel[i]; for (int k = 0; k < 6; k++) vp[k] += cd[k] * q; }
    for (int k = 0; k < 6; k++) vj[k] = SF(cdof)[6 * j + k] * qvel[j];
    cross_motion(SF(d6) + 6 * j, vp, vj);
  }
  SYNC();
  LANES(b, nb) {
    float* f = SF(b6) + 6 * b;
    if (b == 0) { for (int k = 0; k < 6; k++) f[k] = 0; continue; }
    float a[6] = {0, 0, 0, -h->gravity[0], -h->gravity[1], -h->gravity[2]};
    float v[6] = {0, 0, 0, 0, 0, 0};  // spatial velocity of this body (kept in registers)
    dmask_t m = DM(body_ancdof, b);
    while (m) {
      int j = ffs_pop(m);
      const float* d = SF(d6) + 6 * j;
      const float* cd = SF(cdof) + 6 * j;
      float q = qvel[j];
      for (int k = 0; k < 6; k++) { a[k] += d[k]; v[k] += cd[k] * q; }
    }
    float Ia[6], Iv[6], x[6];
    mul_inert(Ia, SF(cinert) + 10 * b, a);
    mul_inert(Iv, SF(cinert) + 10 * b, v);
    cross_force(x, v, Iv);
    for (int k = 0; k < 6; k++) f[k] = Ia[k] + x[k];
  }
  SYNC();
  LANES(j, nv) {
    float fs[6] = {0, 0, 0, 0, 0, 0};
    uint32_t sub = MU(body_sub)[MI(dof_body)[j]];
    while (sub) { int b = ffs_pop(sub); const float* f = SF(b6) + 6 * b; for (int k = 0; k < 6; k++) fs[k] += f[k]; }
    float bias = dot6(SF(cdof) + 6 * j, fs);
    float f = -MF(dof_damping)[j] * qvel[j] - bias;
    int jn = MI(dof_jnt)[j];
    if (MI(jnt_type)[jn] != B200_JNT_FREE) {
      float st = MF(jnt_stiffness)[jn];
      if (st != 0) f -= st * (qpos[MI(jnt_qposadr)[jn]] - MF(jnt_qspring)[jn]);
      for (int a = 0; a < h->nu; a++) {
        if (MI(act_trnid)[a] != jn) continue;
        float ct = SF(ctrl)[a];
        if (MI(act_ctrllimited)[a]) ct = fminf(fmaxf(ct, MF(act_ctrlrange)[2 * a]), MF(act_ctrlrange)[2 * a + 1]);
        float gear = MF(act_gear)[a];
        float len = gear * qpos[MI(jnt_qposadr)[jn]], vel = gear * qvel[j];
        const float* bp = MF(act_bias) + 3 * a;
        float af = MF(act_gain)[a] * ct + bp[0] + bp[1] * len + bp[2] * vel;
        if (MI(act_forcelimited)[a]) af = fminf(fmaxf(af, MF(act_forcerange)[2 * a]), MF(act_forcerange)[2 * a + 1]);
        f += gear * af;
      }
    }
    SF(fsmooth)[j] = f;
  }
  SYNC();
}

// impedance and reference-acceleration constants of the soft-constraint model (used when rows are created)
// (the five solimp numbers travel by value: a pointer to a caller's local array would force that array into local memory)
HDN float impedance5(float s0, float s1, float s2, float s3, float s4, float pos, float margin) {
  float d0 = fminf(fmaxf(s0, B200_MINIMP), B200_MAXIMP), d1 = fminf(fmaxf(s1, B200_MINIMP), B200_MAXIMP);
  float width = fmaxf(s2, 0.f), mid = fminf(fmaxf(s3, B200_MINIMP), B200_MAXIMP), power = fmaxf(s4, 1.f);
  if (d0 == d1 || width <= B200_MINVAL) return 0.5f * (d0 + d1);
  float x = fabsf((pos - margin) / width);
  if (x >= 1) return d1;
  if (x <= 0) return d0;
  float y;
  if (power == 1) y = x;
  else if (power == 2) y = x <= mid ? x * x / mid : 1 - (1 - x) * (1 - x) / (1 - mid);
  else y = x <= mid ? powf(x, power) / powf(mid, power - 1) : 1 - powf(1 - x, power) / powf(1 - mid, power - 1);
  return d0 + y * (d1 - d0);
}
HD float impedance(const float* solimp, float pos, float margin) {
  return impedance5(solimp[0], solimp[1], solimp[2], solimp[3], solimp[4], pos, margin);
}
// K and B of the reference acceleration (refsafe), given solref and dmax = solimp[1]
HD void ref_kb(const Ctx& c, const float* solref, float dmax_in, float* K, float* B) {
  float dmax = fminf(fmaxf(dmax_in, B200_MINIMP), B200_MAXIMP);
  if (solref[0] > 0) {
    float tc = fmaxf(solref[0], 2 * c.h->timestep), dr = solref[1];
    *K = 1.0f / fmaxf(dmax * dmax * tc * tc * dr * dr, B200_MINVAL);
    *B = 2.0f / fmaxf(dmax * tc, B200_MINVAL);
  } else { *K = -solref[0] / (dmax * dmax); *B = -solref[1] / dmax; }
}

// ---------------------------------------------------------------------------------------------------------------
// 5. collision (plane-box, box-box; same decision logic as oracle/oracle.c, fp32)
// Result of one candidate pair (at most 4 contacts): 29 words on the lane's stack.  A/B-timed when it was chosen:
// keeping the result in a shared-memory slot forces the lanes to park it in 28 registers before the contact records -- which the
// slots overlay -- are written, which was measurably slower in the 72-register build.  What does move to shared memory is
// the box-box routine's working set (BoxScratch): it is dead when the routine returns, so no parking is needed, and with it the
// stack frame -- whose size x 132 k threads is what the local-memory write-back traffic scales with -- shrinks.
struct ContactOut { float pos[4][3]; float nrm[4][3]; float dist[4]; int cnt; };
// clipping buffers of collide_box_box: one slot per working lane in SHARED memory (dmodel.h DM_CSLOT_WORDS)
struct BoxScratch { float poly[8][2]; float tmp[8][3]; };
static_assert(sizeof(BoxScratch) <= DM_CSLOT_WORDS * 4, "BoxScratch must fit a narrow-phase lane slot");

HD void geom_pose(const Ctx& c, int g, float* pos, float* mat) {
  int b = MI(geom_body)[g];
  float q[4];
  qmul(q, SF(xquat) + 4 * b, MF(geom_quat) + 4 * g);
  q2mat(mat, q);
  pos[0] = SF(geom_xpos)[3 * g]; pos[1] = SF(geom_xpos)[3 * g + 1]; pos[2] = SF(geom_xpos)[3 * g + 2];
}

HD void collide_plane_box(const Ctx& c, int g1, int g2, float margin, ContactOut& o) {
  float pp[3], pm[9], bp[3], bm[9];
  geom_pose(c, g1, pp, pm); geom_pose(c, g2, bp, bm);
  const float* sz = MF(geom_size) + 3 * g2;
  float n[3] = {pm[2], pm[5], pm[8]}, dif[3] = {bp[0] - pp[0], bp[1] - pp[1], bp[2] - pp[2]};
  float dist0 = dot3(dif, n);
  o.cnt = 0;
  for (int i = 0; i < 8; i++) {
    float loc[3] = {(i & 1) ? sz[0] : -sz[0], (i & 2) ? sz[1] : -sz[1], (i & 4) ? sz[2] : -sz[2]}, vec[3];
    mulmv(vec, bm, loc);
    float ld = dot3(n, vec);
    if (dist0 + ld > margin || ld > 0 || o.cnt >= 4) continue;
    float d = dist0 + ld;
    int k = o.cnt++;
    o.dist[k] = d;
    for (int a = 0; a < 3; a++) { o.pos[k][a] = bp[a] + vec[a] - n[a] * d * 0.5f; o.nrm[k][a] = n[a]; }
  }
}

HD int clip_poly(const float (*in)[2], int n, float (*out)[2], int axis, float bound, float sign) {
  int k = 0;
  for (int i = 0; i < n; i++) {
    const float* a = in[i];
    const float* b = in[(i + 1 == n) ? 0 : i + 1];
    float da = sign * a[axis] - bound, db = sign * b[axis] - bound;
    if (da <= 0) { out[k][0] = a[0]; out[k][1] = a[1]; k++; }
    if ((da < 0 && db > 0) || (da > 0 && db < 0)) {
      float t = da / (da - db);
      out[k][0] = a[0] + t * (b[0] - a[0]); out[k][1] = a[1] + t * (b[1] - a[1]); k++;
    }
  }
  return k;
}

HDN void collide_box_box(const Ctx c, int g1, int g2, float margin, ContactOut& o, BoxScratch& bs) {
  ASSUME_SHARED(c);
  float pa[3], Ra[9], pb[3], Rb[9];
  geom_pose(c, g1, pa, Ra); geom_pose(c, g2, pb, Rb);
  const float* ha = MF(geom_size) + 3 * g1;
  const float* hb = MF(geom_size) + 3 * g2;
  o.cnt = 0;
  float d[3] = {pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]}, da[3], db[3];
  mulmtv(da, Ra, d); mulmtv(db, Rb, d);
  float C[3][3], Q[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) { C[i][j] = Ra[i] * Rb[j] + Ra[3 + i] * Rb[3 + j] + Ra[6 + i] * Rb[6 + j]; Q[i][j] = fabsf(C[i][j]); }
  float best = -1e30f, bestsign = 1; int code = -1;
  for (int i = 0; i < 3; i++) {
    float sep = fabsf(da[i]) - (ha[i] + hb[0] * Q[i][0] + hb[1] * Q[i][1] + hb[2] * Q[i][2]);
    if (sep > margin) return;
    if (sep > best) { best = sep; code = i; bestsign = da[i] < 0 ? -1.f : 1.f; }
  }
  for (int j = 0; j < 3; j++) {
    float sep = fabsf(db[j]) - (hb[j] + ha[0] * Q[0][j] + ha[1] * Q[1][j] + ha[2] * Q[2][j]);
    if (sep > margin) return;
    if (sep > best) { best = sep; code = 3 + j; bestsign = db[j] < 0 ? -1.f : 1.f; }
  }
  float ebest = -1e30f; int ecode = -1; float eaxis[3] = {0, 0, 0};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      float ai[3] = {Ra[i], Ra[3 + i], Ra[6 + i]}, bj[3] = {Rb[j], Rb[3 + j], Rb[6 + j]}, ax[3];
      cross3(ax, ai, bj);
      float l = sqrtf(dot3(ax, ax));
      if (l < 1e-6f) continue;
      float il = 1.0f / l;
      ax[0] *= il; ax[1] *= il; ax[2] *= il;
      float ra = 0, rb = 0;
      for (int k = 0; k < 3; k++) {
        float ak[3] = {Ra[k], Ra[3 + k], Ra[6 + k]}, bk[3] = {Rb[k], Rb[3 + k], Rb[6 + k]};
        ra += ha[k] * fabsf(dot3(ak, ax)); rb += hb[k] * fabsf(dot3(bk, ax));
      }
      float dd = dot3(d, ax), sep = fabsf(dd) - (ra + rb);
      if (sep > margin) return;
      if (sep > ebest) { ebest = sep; ecode = 3 * i + j; float sg = dd < 0 ? -1.f : 1.f; eaxis[0] = sg * ax[0]; eaxis[1] = sg * ax[1]; eaxis[2] = sg * ax[2]; }
    }
  // (runtime-indexed columns / entries are picked with selects so that the matrices stay in registers: an array indexed by a
  // runtime value, or reached through a pointer chosen at run time, would live in local memory)
#define B200_SEL3(a0, a1, a2, i) ((i) == 0 ? (a0) : ((i) == 1 ? (a1) : (a2)))
#define B200_COL(out, R, i) do { out[0] = B200_SEL3(R[0], R[1], R[2], i); out[1] = B200_SEL3(R[3], R[4], R[5], i); out[2] = B200_SEL3(R[6], R[7], R[8], i); } while (0)
  if (ecode >= 0 && ebest > best + 1e-3f * (fabsf(best) + 1e-3f) && ebest > 0.95f * best && ebest > best) {
    int i = ecode / 3, j = ecode - 3 * i;
    float n[3] = {eaxis[0], eaxis[1], eaxis[2]};
    float ea[3], eb[3];
    B200_COL(ea, Ra, i); B200_COL(eb, Rb, j);
    float PA[3] = {pa[0], pa[1], pa[2]}, PB[3] = {pb[0], pb[1], pb[2]};
#pragma unroll
    for (int k = 0; k < 3; k++) {
      float ak[3] = {Ra[k], Ra[3 + k], Ra[6 + k]}, bk[3] = {Rb[k], Rb[3 + k], Rb[6 + k]};
      if (k != i) { float sg = (dot3(n, ak) > 0 ? 1.f : -1.f) * ha[k]; PA[0] += ak[0] * sg; PA[1] += ak[1] * sg; PA[2] += ak[2] * sg; }
      if (k != j) { float sg = (dot3(n, bk) > 0 ? -1.f : 1.f) * hb[k]; PB[0] += bk[0] * sg; PB[1] += bk[1] * sg; PB[2] += bk[2] * sg; }
    }
    float w[3] = {PA[0] - PB[0], PA[1] - PB[1], PA[2] - PB[2]};
    float b = dot3(ea, eb), dd = dot3(ea, w), e = dot3(eb, w), den = 1 - b * b;
    float sp = den > 1e-12f ? (b * e - dd) / den : 0, tp = den > 1e-12f ? (e - b * dd) / den : 0;
    sp = fminf(fmaxf(sp, -ha[i]), ha[i]); tp = fminf(fmaxf(tp, -hb[j]), hb[j]);
    o.cnt = 1; o.dist[0] = ebest; o.nrm[0][0] = n[0]; o.nrm[0][1] = n[1]; o.nrm[0][2] = n[2];
    for (int k = 0; k < 3; k++) o.pos[0][k] = 0.5f * (PA[k] + ea[k] * sp + PB[k] + eb[k] * tp);
    return;
  }
  // reference box (owner of the separating face) and incident box, copied with selects
  const bool flipb = code >= 3;
  const int ax = flipb ? code - 3 : code, flip = flipb ? 1 : 0;
  const float sgn = flipb ? -bestsign : bestsign;
  float pr[3], pi[3], Rr[9], Ri[9];
#pragma unroll
  for (int k = 0; k < 3; k++) { pr[k] = flipb ? pb[k] : pa[k]; pi[k] = flipb ? pa[k] : pb[k]; }
#pragma unroll
  for (int k = 0; k < 9; k++) { Rr[k] = flipb ? Rb[k] : Ra[k]; Ri[k] = flipb ? Ra[k] : Rb[k]; }
  const float* hr = flipb ? hb : ha;   // half sizes: shared-memory tables, runtime indices are fine there
  const float* hi = flipb ? ha : hb;
  float nr[3];
  B200_COL(nr, Rr, ax);
  nr[0] *= sgn; nr[1] *= sgn; nr[2] *= sgn;
  float nloc[3];
  mulmtv(nloc, Ri, nr);
  int iax = 0; float bestd = -1;
#pragma unroll
  for (int k = 0; k < 3; k++) if (fabsf(nloc[k]) > bestd) { bestd = fabsf(nloc[k]); iax = k; }
  float isgn = B200_SEL3(nloc[0], nloc[1], nloc[2], iax) > 0 ? -1.f : 1.f;
  int u = (iax + 1) % 3, v = (iax + 2) % 3, ru = (ax + 1) % 3, rv = (ax + 2) % 3;
  float au[3], av[3], iu[3], iv[3], ia[3];
  B200_COL(au, Rr, ru); B200_COL(av, Rr, rv); B200_COL(iu, Ri, u); B200_COL(iv, Ri, v); B200_COL(ia, Ri, iax);
  const float hia = hi[iax] * isgn, hiu = hi[u], hiv = hi[v], hrax = hr[ax];
  float fc[3] = {pi[0] + ia[0] * hia, pi[1] + ia[1] * hia, pi[2] + ia[2] * hia};
  float (*poly)[2] = bs.poly;
  float (*tmp)[2] = (float (*)[2])bs.tmp;
  float zc[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    float su = (k == 0 || k == 3) ? 1.f : -1.f, sv = (k < 2) ? 1.f : -1.f;
    float rel[3];
    for (int a = 0; a < 3; a++) rel[a] = fc[a] + iu[a] * su * hiu + iv[a] * sv * hiv - pr[a];
    poly[k][0] = dot3(rel, au); poly[k][1] = dot3(rel, av);
    zc[k] = dot3(rel, nr) - hrax;
  }
  float h0, hx, hy;
  {
    float x0 = poly[0][0], y0 = poly[0][1], x1 = poly[1][0], y1 = poly[1][1], x3 = poly[3][0], y3 = poly[3][1];
    float z0 = zc[0], z1 = zc[1], z3 = zc[3];
    float det = (x1 - x0) * (y3 - y0) - (x3 - x0) * (y1 - y0);
    if (fabsf(det) < 1e-14f) { hx = hy = 0; h0 = z0; }
    else {
      hx = ((z1 - z0) * (y3 - y0) - (z3 - z0) * (y1 - y0)) / det;
      hy = ((x1 - x0) * (z3 - z0) - (x3 - x0) * (z1 - z0)) / det;
      h0 = z0 - hx * x0 - hy * y0;
    }
  }
  int n = 4;
  n = clip_poly(poly, n, tmp, 0, hr[ru], 1.f);
  n = clip_poly(tmp, n, poly, 0, hr[ru], -1.f);
  n = clip_poly(poly, n, tmp, 1, hr[rv], 1.f);
  n = clip_poly(tmp, n, poly, 1, hr[rv], -1.f);
  float (*cand)[3] = bs.tmp;   // the clipping result is in `poly`: `tmp` is free again
  int nc = 0;
  for (int k = 0; k < n && k < 8; k++) {
    float z = h0 + hx * poly[k][0] + hy * poly[k][1];
    if (z > margin) continue;
    cand[nc][0] = poly[k][0]; cand[nc][1] = poly[k][1]; cand[nc][2] = z; nc++;
  }
  if (nc == 0) return;
  // at most four of the candidates, in ascending candidate order: kept as a bit mask (no index array)
  uint32_t keep = (1u << nc) - 1u;
  if (nc > 4) {
    int i0 = 0;
    for (int k = 1; k < nc; k++) if (cand[k][2] < cand[i0][2]) i0 = k;
    int i1 = -1; float bd = -1;
    for (int k = 0; k < nc; k++) { float dx = cand[k][0] - cand[i0][0], dy = cand[k][1] - cand[i0][1], q = dx * dx + dy * dy; if (k != i0 && q > bd) { bd = q; i1 = k; } }
    float ex = cand[i1][0] - cand[i0][0], ey = cand[i1][1] - cand[i0][1];
    int i2 = -1, i3 = -1; float bp = 0, bn = 0;
    for (int k = 0; k < nc; k++) {
      if (k == i0 || k == i1) continue;
      float cr = ex * (cand[k][1] - cand[i0][1]) - ey * (cand[k][0] - cand[i0][0]);
      if (cr > bp) { bp = cr; i2 = k; }
      if (cr < bn) { bn = cr; i3 = k; }
    }
    keep = (1u << i0) | (1u << i1);
    if (i2 >= 0) keep |= 1u << i2;
    if (i3 >= 0) keep |= 1u << i3;
  }
  float fs = flip ? -1.f : 1.f;
  int ns = 0;
  while (keep) {
    const float* cd = cand[ffs_pop(keep)];
    o.dist[ns] = cd[2];
    o.nrm[ns][0] = fs * nr[0]; o.nrm[ns][1] = fs * nr[1]; o.nrm[ns][2] = fs * nr[2];
    for (int a = 0; a < 3; a++) o.pos[ns][a] = pr[a] + au[a] * cd[0] + av[a] * cd[1] + nr[a] * (hrax + 0.5f * cd[2]);
    ns++;
  }
  o.cnt = ns;
#undef B200_COL
#undef B200_SEL3
}

// ---- sphere / capsule against planes and boxes (same decision logic as oracle/oracle.c)
HD void collide_plane_sphere(const Ctx& c, int g1, int g2, float margin, ContactOut& o) {
  float pp[3], pm[9];
  geom_pose(c, g1, pp, pm);
  const float* ce = SF(geom_xpos) + 3 * g2;
  float n[3] = {pm[2], pm[5], pm[8]}, dif[3] = {ce[0] - pp[0], ce[1] - pp[1], ce[2] - pp[2]};
  float r = MF(geom_size)[3 * g2], d = dot3(dif, n) - r;
  o.cnt = 0;
  if (d > margin) return;
  o.cnt = 1; o.dist[0] = d;
  for (int a = 0; a < 3; a++) { o.pos[0][a] = ce[a] - n[a] * (r + 0.5f * d); o.nrm[0][a] = n[a]; }
}
HD void collide_plane_capsule(const Ctx& c, int g1, int g2, float margin, ContactOut& o) {
  float pp[3], pm[9], cp[3], cm[9];
  geom_pose(c, g1, pp, pm); geom_pose(c, g2, cp, cm);
  float n[3] = {pm[2], pm[5], pm[8]}, ax[3] = {cm[2], cm[5], cm[8]};
  float r = MF(geom_size)[3 * g2], hl = MF(geom_size)[3 * g2 + 1];
  o.cnt = 0;
  for (int side = -1; side <= 1; side += 2) {
    float e[3] = {cp[0] + ax[0] * side * hl, cp[1] + ax[1] * side * hl, cp[2] + ax[2] * side * hl};
    float dif[3] = {e[0] - pp[0], e[1] - pp[1], e[2] - pp[2]};
    float d = dot3(dif, n) - r;
    if (d > margin) continue;
    int k = o.cnt++;
    o.dist[k] = d;
    for (int a = 0; a < 3; a++) { o.pos[k][a] = e[a] - n[a] * (r + 0.5f * d); o.nrm[k][a] = n[a]; }
  }
}
// signed distance from p to the surface of a box (pose bp/bm, half sizes h); normal points from the surface towards p
HD float point_box(const float* p, const float* bp, const float* bm, const float* h, float* closest, float* normal) {
  float rel[3] = {p[0] - bp[0], p[1] - bp[1], p[2] - bp[2]}, loc[3], q[3];
  mulmtv(loc, bm, rel);
  bool inside = true;
  for (int k = 0; k < 3; k++) { q[k] = fminf(fmaxf(loc[k], -h[k]), h[k]); if (q[k] != loc[k]) inside = false; }
  float nl[3] = {0, 0, 0}, dist;
  if (!inside) {
    float d[3] = {loc[0] - q[0], loc[1] - q[1], loc[2] - q[2]};
    dist = sqrtf(dot3(d, d));
    float inv = 1.0f / dist;
    nl[0] = d[0] * inv; nl[1] = d[1] * inv; nl[2] = d[2] * inv;
  } else {
    int ax = 0; float best = 1e30f;
    for (int k = 0; k < 3; k++) { float pen = h[k] - fabsf(loc[k]); if (pen < best) { best = pen; ax = k; } }
    dist = -best;
    float sg = loc[ax] < 0 ? -1.f : 1.f;
    if (ax == 0) { nl[0] = sg; q[0] = sg * h[0]; } else if (ax == 1) { nl[1] = sg; q[1] = sg * h[1]; } else { nl[2] = sg; q[2] = sg * h[2]; }
  }
  mulmv(closest, bm, q);
  closest[0] += bp[0]; closest[1] += bp[1]; closest[2] += bp[2];
  mulmv(normal, bm, nl);
  return dist;
}
HD void sphere_box_contact(const float* center, float r, const float* bp, const float* bm, const float* bh, float margin, ContactOut& o) {
  if (o.cnt >= 4) return;
  float closest[3], nrm[3];
  float d = point_box(center, bp, bm, bh, closest, nrm) - r;
  if (d > margin) return;
  int k = o.cnt++;
  o.dist[k] = d;
  for (int a = 0; a < 3; a++) { o.nrm[k][a] = -nrm[a]; o.pos[k][a] = closest[a] + nrm[a] * 0.5f * d; }
}
// signed distance of a point given in the box frame (the distance part of point_box, no transforms)
HD float box_sdist(const float* loc, const float* h) {
  float dx = fabsf(loc[0]) - h[0], dy = fabsf(loc[1]) - h[1], dz = fabsf(loc[2]) - h[2];
  if (dx <= 0 && dy <= 0 && dz <= 0) return fmaxf(dx, fmaxf(dy, dz));   // inside: minus the smallest penetration
  float ex = fmaxf(dx, 0.f), ey = fmaxf(dy, 0.f), ez = fmaxf(dz, 0.f);
  return sqrtf(ex * ex + ey * ey + ez * ez);
}
HDN void capsule_box_contacts(const float* cp, const float* ax, float r, float hl, const float* bp, const float* bm, const float* bh,
                              float margin, ContactOut& o) {
  // the search runs in the box frame: segment p(t) = cl + t dl, t in [-hl, hl] (rotated once; every evaluation of the convex
  // distance function is then a handful of operations)
  float rel[3] = {cp[0] - bp[0], cp[1] - bp[1], cp[2] - bp[2]}, cl[3], dl[3], p[3];
  mulmtv(cl, bm, rel); mulmtv(dl, bm, ax);
#define B200_SEG(t_) (p[0] = fmaf(dl[0], (t_), cl[0]), p[1] = fmaf(dl[1], (t_), cl[1]), p[2] = fmaf(dl[2], (t_), cl[2]), box_sdist(p, bh))
  // no point of the segment is closer than the centre's distance minus the half length (the distance is 1-Lipschitz)
  if (box_sdist(cl, bh) - hl - r > margin) return;
  float d0 = B200_SEG(-hl) - r, d1 = B200_SEG(hl) - r;
  if (d0 <= margin && d1 <= margin) {
    float e0[3] = {cp[0] - ax[0] * hl, cp[1] - ax[1] * hl, cp[2] - ax[2] * hl}, e1[3] = {cp[0] + ax[0] * hl, cp[1] + ax[1] * hl, cp[2] + ax[2] * hl};
    sphere_box_contact(e0, r, bp, bm, bh, margin, o);
    sphere_box_contact(e1, r, bp, bm, bh, margin, o);
    return;
  }
  const float gr = 0.6180339887498949f;
  float lo = -hl, hi = hl, x1 = hi - gr * (hi - lo), x2 = lo + gr * (hi - lo);
  float f1 = B200_SEG(x1), f2 = B200_SEG(x2);
  for (int it = 0; it < 24; it++) {
    if (f1 < f2) { hi = x2; x2 = x1; f2 = f1; x1 = hi - gr * (hi - lo); f1 = B200_SEG(x1); }
    else { lo = x1; x1 = x2; f1 = f2; x2 = lo + gr * (hi - lo); f2 = B200_SEG(x2); }
  }
  float t = 0.5f * (lo + hi);
  float fmin = B200_SEG(t);
  if (fmin - r > margin) return;
  // flat zone {f <= fmin + tol} of the convex distance function: a capsule lying (nearly) parallel on a face gets one
  // contact at each end of the zone instead of one at an arbitrary point of it (same rule as oracle/oracle.c)
  const float tol = 2e-5f;
  float tz[2];
  for (int side = 0; side < 2; side++) {
    float out = side ? hl : -hl, in = t;
    if (B200_SEG(out) <= fmin + tol) in = out;
    else for (int it = 0; it < 14; it++) {
      float mid = 0.5f * (out + in);
      if (B200_SEG(mid) <= fmin + tol) in = mid; else out = mid;
    }
    tz[side] = in;
  }
#undef B200_SEG
  if (tz[1] - tz[0] > r) {
    for (int a = 0; a < 3; a++) p[a] = cp[a] + ax[a] * tz[0];
    sphere_box_contact(p, r, bp, bm, bh, margin, o);
    for (int a = 0; a < 3; a++) p[a] = cp[a] + ax[a] * tz[1];
    sphere_box_contact(p, r, bp, bm, bh, margin, o);
  } else {
    for (int a = 0; a < 3; a++) p[a] = cp[a] + ax[a] * t;
    sphere_box_contact(p, r, bp, bm, bh, margin, o);
  }
}
// sphere or capsule geom g1 against box geom g2, or (g2 < 0) against the maze wall cells around it
HD void collide_round_box(const Ctx& c, int g1, int g2, float margin, ContactOut& o) {
  const DMHead* h = c.h;
  o.cnt = 0;
  float cp[3], cm[9];
  geom_pose(c, g1, cp, cm);
  bool capsule = MI(geom_type)[g1] == B200_GEOM_CAPSULE;
  float r = MF(geom_size)[3 * g1], hl = MF(geom_size)[3 * g1 + 1], ax[3] = {cm[2], cm[5], cm[8]};
  if (g2 >= 0) {
    float bp[3], bm[9];
    geom_pose(c, g2, bp, bm);
    if (capsule) capsule_box_contacts(cp, ax, r, hl, bp, bm, MF(geom_size) + 3 * g2, margin, o);
    else sphere_box_contact(cp, r, bp, bm, MF(geom_size) + 3 * g2, margin, o);
    return;
  }
  float reach = MF(geom_rbound)[g1] + margin, s = h->grid_scale;
  if (cp[2] - reach > h->grid_top) return;
  int j0 = (int)floorf((cp[0] - reach + h->grid_xc) / s), j1 = (int)floorf((cp[0] + reach + h->grid_xc) / s);
  int i0 = (int)floorf((h->grid_yc - (cp[1] + reach)) / s), i1 = (int)floorf((h->grid_yc - (cp[1] - reach)) / s);
  const float idm[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  float bh[3] = {0.5f * s, 0.5f * s, 0.5f * h->grid_top};
  for (int i = i0; i <= i1; i++)
    for (int j = j0; j <= j1; j++) {
      if (i < 0 || j < 0 || i >= h->grid_len || j >= h->grid_wid) continue;
      int bit = i * h->grid_wid + j;
      if (!((MU(grid_walls)[bit >> 5] >> (bit & 31)) & 1u)) continue;
      float bp[3] = {(j + 0.5f) * s - h->grid_xc, h->grid_yc - (i + 0.5f) * s, 0.5f * h->grid_top};
      if (capsule) capsule_box_contacts(cp, ax, r, hl, bp, idm, bh, margin, o);
      else sphere_box_contact(cp, r, bp, idm, bh, margin, o);
    }
}

// sphere/capsule against sphere/capsule: closest points of the two axis segments, then a sphere-sphere contact
// (same decision logic as oracle/oracle.c collide_round_round)
HDN void collide_round_round(const Ctx c, int g1, int g2, float margin, ContactOut& o) {
  ASSUME_SHARED(c);
  o.cnt = 0;
  float p1[3], m1[9], p2[3], m2[9];
  geom_pose(c, g1, p1, m1); geom_pose(c, g2, p2, m2);
  float a1[3] = {m1[2], m1[5], m1[8]}, a2[3] = {m2[2], m2[5], m2[8]};
  float r1 = MF(geom_size)[3 * g1], r2 = MF(geom_size)[3 * g2];
  float h1 = MI(geom_type)[g1] == B200_GEOM_CAPSULE ? MF(geom_size)[3 * g1 + 1] : 0.f;
  float h2 = MI(geom_type)[g2] == B200_GEOM_CAPSULE ? MF(geom_size)[3 * g2 + 1] : 0.f;
  float w[3] = {p1[0] - p2[0], p1[1] - p2[1], p1[2] - p2[2]};
  // den = |a1 x a2|^2 = sin^2 theta: 1 - (a1.a2)^2 cancels to nothing below theta ~ 3e-4 in fp32 and is not sin^2 theta for axes
  // that are unit only to 1e-7 (identical axes gave den ~ 1e-7, a "non-parallel" solve and a contact millimetres off)
  float cx[3];
  cross3(cx, a1, a2);
  float b = dot3(a1, a2), d = dot3(a1, w), e = dot3(a2, w), den = dot3(cx, cx), sp = 0, tp = 0;
  if (h1 <= 0 && h2 <= 0) { sp = 0; tp = 0; }
  else if (h1 <= 0) { sp = 0; tp = e; }
  else if (h2 <= 0) { tp = 0; sp = -d; }
  else if (den > 1e-9f) {
    sp = fminf(fmaxf((b * e - d) / den, -h1), h1);
    tp = e + b * sp;
    if (tp < -h2) { tp = -h2; sp = b * tp - d; }
    else if (tp > h2) { tp = h2; sp = b * tp - d; }
  } else {
    float mid2 = -d, lo = fmaxf(mid2 - h2, -h1), hi = fminf(mid2 + h2, h1);
    sp = lo > hi ? (mid2 < 0 ? -h1 : h1) : 0.5f * (lo + hi);
    tp = e + b * sp;
  }
  sp = fminf(fmaxf(sp, -h1), h1); tp = fminf(fmaxf(tp, -h2), h2);
  float q1[3], n[3];
  for (int k = 0; k < 3; k++) { q1[k] = p1[k] + a1[k] * sp; n[k] = p2[k] + a2[k] * tp - q1[k]; }
  float len = sqrtf(dot3(n, n)), dist = len - r1 - r2;
  if (dist > margin) return;
  if (len < 1e-12f) { n[0] = 0; n[1] = 0; n[2] = 1; } else { float il = 1.0f / len; n[0] *= il; n[1] *= il; n[2] *= il; }
  o.cnt = 1; o.dist[0] = dist;
  for (int k = 0; k < 3; k++) { o.nrm[0][k] = n[k]; o.pos[0][k] = q1[k] + n[k] * (r1 + 0.5f * dist); }
}


// ---- general convex pairs (a cylinder or an ellipsoid against a box / capsule / sphere / cylinder / ellipsoid): Minkowski
// portal refinement on the support functions (Snethen's XenoCollide -- the published algorithm behind MuJoCo's convex
// collider: tolerance 1e-6, at most 50 rounds), one contact per pair, both shapes inflated by margin / 2, dist = margin -
// depth.  Same decision logic as oracle/oracle.c cvx_mpr; evaluated relative to the first geom's centre so that fp32
// keeps its resolution.  A point of A - B is kept as (v, witness on A); the witness on B is a - v.
#ifdef B200_HULL
struct CvxShape { int type; float pos[3], mat[9], size[3], infl; const float* hv; int nhv; };   // hv: hull vertices (global memory)
#else
struct CvxShape { int type; float pos[3], mat[9], size[3], infl; };
#endif
struct CvxPt { float v[3], a[3]; };
HD void cvx_support(const CvxShape& g, const float* d, float* out) {
  float l[3], sl[3] = {0, 0, 0};
  mulmtv(l, g.mat, d);
  const float* z = g.size;
  if (g.type == B200_GEOM_BOX) { sl[0] = l[0] >= 0 ? z[0] : -z[0]; sl[1] = l[1] >= 0 ? z[1] : -z[1]; sl[2] = l[2] >= 0 ? z[2] : -z[2]; }
#ifdef B200_HULL
  else if (g.type == B200_GEOM_MESH) {   // reduced convex hull: the vertex farthest along l, the first one on ties (as oracle/oracle.c)
    int best = 0; float bd = -3.0e38f;
    for (int i = 0; i < g.nhv; i++) { float dd = g.hv[3 * i] * l[0] + g.hv[3 * i + 1] * l[1] + g.hv[3 * i + 2] * l[2]; if (dd > bd) { bd = dd; best = i; } }
    if (g.nhv > 0) { sl[0] = g.hv[3 * best]; sl[1] = g.hv[3 * best + 1]; sl[2] = g.hv[3 * best + 2]; }
  }
#endif
  else if (g.type == B200_GEOM_CYLINDER) {
    float n = sqrtf(l[0] * l[0] + l[1] * l[1]);
    if (n > 1e-12f) { float i = z[0] / n; sl[0] = i * l[0]; sl[1] = i * l[1]; }
    sl[2] = l[2] >= 0 ? z[1] : -z[1];
  } else if (g.type == B200_GEOM_ELLIPSOID) {
    float a = z[0] * l[0], b = z[1] * l[1], cc = z[2] * l[2], n = sqrtf(a * a + b * b + cc * cc);
    if (n > 0) { float i = 1.0f / n; sl[0] = z[0] * a * i; sl[1] = z[1] * b * i; sl[2] = z[2] * cc * i; }
  } else {  // sphere, capsule
    float n = sqrtf(dot3(l, l));
    if (n > 0) { float i = z[0] / n; sl[0] = i * l[0]; sl[1] = i * l[1]; sl[2] = i * l[2]; }
    if (g.type == B200_GEOM_CAPSULE) sl[2] += l[2] >= 0 ? z[1] : -z[1];
  }
  mulmv(out, g.mat, sl);
  float n = sqrtf(dot3(d, d)), e = n > 0 ? g.infl / n : 0.f;
  for (int k = 0; k < 3; k++) out[k] += g.pos[k] + e * d[k];
}
HD void cvx_msupport(const CvxShape& A, const CvxShape& B, const float* d, CvxPt& p) {
  float nd[3] = {-d[0], -d[1], -d[2]}, b[3];
  cvx_support(A, d, p.a); cvx_support(B, nd, b);
  p.v[0] = p.a[0] - b[0]; p.v[1] = p.a[1] - b[1]; p.v[2] = p.a[2] - b[2];
}
HD void cvx_portal_dir(const CvxPt& o, const CvxPt& p, const CvxPt& q, float* dir) {  // normalised (p - o) x (q - o)
  float va[3] = {p.v[0] - o.v[0], p.v[1] - o.v[1], p.v[2] - o.v[2]}, vb[3] = {q.v[0] - o.v[0], q.v[1] - o.v[1], q.v[2] - o.v[2]};
  cross3(dir, va, vb);
  float n = sqrtf(dot3(dir, dir)), i = n > 1e-30f ? 1.0f / n : 0.f;
  dir[0] *= i; dir[1] *= i; dir[2] *= i;
}
HDN void collide_convex(const Ctx c, int g1, int g2, float margin, ContactOut& o) {
  ASSUME_SHARED(c);
  o.cnt = 0;
  CvxShape A, B;
  float p1[3], p2[3];
  geom_pose(c, g1, p1, A.mat); geom_pose(c, g2, p2, B.mat);
  A.type = MI(geom_type)[g1]; B.type = MI(geom_type)[g2];
#ifdef B200_HULL
  A.hv = GF(hull_vert) + 3 * GI(geom_hull)[2 * g1]; A.nhv = GI(geom_hull)[2 * g1 + 1];
  B.hv = GF(hull_vert) + 3 * GI(geom_hull)[2 * g2]; B.nhv = GI(geom_hull)[2 * g2 + 1];
#endif
  for (int k = 0; k < 3; k++) { A.pos[k] = 0.f; B.pos[k] = p2[k] - p1[k]; A.size[k] = MF(geom_size)[3 * g1 + k]; B.size[k] = MF(geom_size)[3 * g2 + k]; }
  A.infl = B.infl = 0.5f * margin;
  const float tol = 1e-6f; const int maxit = 50;
  CvxPt v0, v1, v2, v3, v4;
  float dir[3], t[3];
  for (int k = 0; k < 3; k++) { v0.a[k] = 0.f; v0.v[k] = -B.pos[k]; }
  if (dot3(v0.v, v0.v) < 1e-24f) v0.v[0] = 1e-5f;
  { float i = rsqrtf(dot3(v0.v, v0.v)); dir[0] = -v0.v[0] * i; dir[1] = -v0.v[1] * i; dir[2] = -v0.v[2] * i; }
  cvx_msupport(A, B, dir, v1);
  if (dot3(v1.v, dir) <= 0) return;
  cross3(t, v0.v, v1.v);
  float depth, pos[3];
  if (dot3(t, t) < 1e-24f) {
    // the origin lies on the ray v0 -> v1: the centres' line is the contact normal
    depth = dot3(v1.v, dir);
    for (int k = 0; k < 3; k++) pos[k] = v1.a[k] - 0.5f * v1.v[k];
  } else {
    { float i = rsqrtf(dot3(t, t)); dir[0] = t[0] * i; dir[1] = t[1] * i; dir[2] = t[2] * i; }
    cvx_msupport(A, B, dir, v2);
    if (dot3(v2.v, dir) <= 0) return;
    cvx_portal_dir(v0, v1, v2, dir);
    if (dot3(dir, v0.v) > 0) { CvxPt tmp = v1; v1 = v2; v2 = tmp; dir[0] = -dir[0]; dir[1] = -dir[1]; dir[2] = -dir[2]; }
    // (the two search loops leave through `break` only -- a miss is a flag tested after the loop, not a return from inside it)
    bool miss = false;
    for (int it = 0;; it++) {  // portal discovery
      if (it > maxit) { miss = true; break; }
      cvx_msupport(A, B, dir, v3);
      if (dot3(v3.v, dir) <= 0) { miss = true; break; }
      bool cont = false;
      cross3(t, v1.v, v3.v);
      if (dot3(t, v0.v) < 0) { v2 = v3; cont = true; }
      else { cross3(t, v3.v, v2.v); if (dot3(t, v0.v) < 0) { v1 = v3; cont = true; } }
      if (!cont) break;
      cvx_portal_dir(v0, v1, v2, dir);
    }
    if (miss) return;
    bool hit = false;
    for (int it = 0;; it++) {  // refinement; past the origin the shapes overlap and the loop runs on to the surface
      cvx_portal_dir(v1, v2, v3, dir);
      if (dot3(dir, v1.v) >= 0) hit = true;
      cvx_msupport(A, B, dir, v4);
      float d4 = dot3(v4.v, dir);
      if (!hit && d4 < 0) { miss = true; break; }
      float mn = fminf(fminf(d4 - dot3(v1.v, dir), d4 - dot3(v2.v, dir)), d4 - dot3(v3.v, dir));
      if (mn <= tol || it >= maxit) { miss = !hit; break; }
      cross3(t, v4.v, v0.v);
      if (dot3(v1.v, t) > 0) { if (dot3(v2.v, t) > 0) v1 = v4; else v3 = v4; }
      else { if (dot3(v3.v, t) > 0) v2 = v4; else v1 = v4; }
    }
    if (miss) return;
    depth = dot3(dir, v1.v);
    float b0, b1, b2, b3, sum;
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
    if (!(fabsf(sum) > 0)) return;
    float is = 1.0f / sum;
    // midpoint of the two witnesses: a - v / 2 per portal vertex
    for (int k = 0; k < 3; k++)
      pos[k] = (b0 * (v0.a[k] - 0.5f * v0.v[k]) + b1 * (v1.a[k] - 0.5f * v1.v[k]) + b2 * (v2.a[k] - 0.5f * v2.v[k]) + b3 * (v3.a[k] - 0.5f * v3.v[k])) * is;
  }
  o.cnt = 1; o.dist[0] = margin - depth;
  for (int k = 0; k < 3; k++) { o.nrm[0][k] = dir[k]; o.pos[0][k] = pos[k] + p1[k]; }
}
// plane vs cylinder / ellipsoid (same point selection as oracle/oracle.c)
HDN void collide_plane_convex(const Ctx c, int g1, int g2, float margin, ContactOut& o) {
  ASSUME_SHARED(c);
  o.cnt = 0;
  float pp[3], pm[9], cp[3], cm[9];
  geom_pose(c, g1, pp, pm); geom_pose(c, g2, cp, cm);
  float n[3] = {pm[2], pm[5], pm[8]};
  const float* sz = MF(geom_size) + 3 * g2;
#ifdef B200_HULL
  if (MI(geom_type)[g2] == B200_GEOM_MESH) {
    // plane vs hull: the hull vertices within the margin of the plane, the deepest first, at most four ((distance, index) order)
    const float* hv = GF(hull_vert) + 3 * GI(geom_hull)[2 * g2];
    const int nhv = GI(geom_hull)[2 * g2 + 1];
    float last = -3.0e38f; int lasti = -1;
    for (int k = 0; k < 4; k++) {
      int best = -1; float bd = 3.0e38f;
      for (int i = 0; i < nhv; i++) {
        float p[3];
        mulmv(p, cm, hv + 3 * i);
        float dif[3] = {p[0] + cp[0] - pp[0], p[1] + cp[1] - pp[1], p[2] + cp[2] - pp[2]};
        float d = dot3(dif, n);
        if ((d > last || (d == last && i > lasti)) && d < bd) { bd = d; best = i; }
      }
      if (best < 0 || bd > margin) break;
      float p[3];
      mulmv(p, cm, hv + 3 * best);
      int k2 = o.cnt++;
      o.dist[k2] = bd;
      for (int a = 0; a < 3; a++) { o.nrm[k2][a] = n[a]; o.pos[k2][a] = p[a] + cp[a] - 0.5f * bd * n[a]; }
      last = bd; lasti = best;
    }
    return;
  }
#endif
  if (MI(geom_type)[g2] == B200_GEOM_ELLIPSOID) {
    float l[3], nn[3] = {-n[0], -n[1], -n[2]}, sl[3] = {0, 0, 0}, p[3];
    mulmtv(l, cm, nn);
    float a = sz[0] * l[0], b = sz[1] * l[1], cc = sz[2] * l[2], nl = sqrtf(a * a + b * b + cc * cc);
    if (nl > 0) { sl[0] = sz[0] * a / nl; sl[1] = sz[1] * b / nl; sl[2] = sz[2] * cc / nl; }
    mulmv(p, cm, sl);
    float dif[3] = {p[0] + cp[0] - pp[0], p[1] + cp[1] - pp[1], p[2] + cp[2] - pp[2]};
    float d = dot3(dif, n);
    if (d > margin) return;
    o.cnt = 1; o.dist[0] = d;
    for (int k = 0; k < 3; k++) { o.nrm[0][k] = n[k]; o.pos[0][k] = p[k] + cp[k] - 0.5f * d * n[k]; }
    return;
  }
  float ax[3] = {cm[2], cm[5], cm[8]}, r = sz[0], hl = sz[1];
  float an = dot3(ax, n);
  if (an > 0) { ax[0] = -ax[0]; ax[1] = -ax[1]; ax[2] = -ax[2]; an = -an; }
  float rad[3] = {-n[0] + an * ax[0], -n[1] + an * ax[1], -n[2] + an * ax[2]};
  float rl = sqrtf(dot3(rad, rad));
  if (rl < 1e-9f) { float y[3] = {0, 0, 0}; if (fabsf(ax[0]) < 0.5f) y[0] = 1; else y[1] = 1; cross3(rad, ax, y); rl = sqrtf(dot3(rad, rad)); }
  { float i = 1.0f / rl; rad[0] *= i; rad[1] *= i; rad[2] *= i; }
  float side[3];
  cross3(side, ax, rad);
  for (int i = 0; i < 4; i++) {
    float cs = i < 2 ? 1.f : -0.5f, sn = i < 2 ? 0.f : (i == 2 ? 0.8660254037844386f : -0.8660254037844386f), cap = i == 1 ? -1.f : 1.f;
    float p[3];
    for (int k = 0; k < 3; k++) p[k] = cp[k] + cap * hl * ax[k] + r * (cs * rad[k] + sn * side[k]);
    float dif[3] = {p[0] - pp[0], p[1] - pp[1], p[2] - pp[2]};
    float d = dot3(dif, n);
    if (d > margin) continue;
    int k2 = o.cnt++;
    o.dist[k2] = d;
    for (int k = 0; k < 3; k++) { o.nrm[k2][k] = n[k]; o.pos[k2][k] = p[k] - 0.5f * d * n[k]; }
  }
}

HD void make_frame(float* f) {
  float n = sqrtf(dot3(f, f)), inv = n > 1e-12f ? 1.0f / n : 0.f;
  f[0] *= inv; f[1] *= inv; f[2] *= inv;
  float* y = f + 3;
  y[0] = y[1] = y[2] = 0;
  if (f[1] < 0.5f && f[1] > -0.5f) y[1] = 1; else y[2] = 1;
  float d = dot3(f, y);
  y[0] -= f[0] * d; y[1] -= f[1] * d; y[2] -= f[2] * d;
  float ny = 1.0f / sqrtf(dot3(y, y));
  y[0] *= ny; y[1] *= ny; y[2] *= ny;
  cross3(f + 6, f, y);
}

// HF: model family with hand features (frictionloss rows, tendon limits, round-round pairs, touch sensors); compiled out
// of the other kernel instantiations to keep their instruction stream short
// CX: builds that carry the general convex collider (cylinder / ellipsoid geoms)
template <bool HF, bool CX>
STAGE void collision(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  int* cnt = SI(counters);
  // broad-phase candidates: pair indices, one byte each (models with up to 255 candidate pairs) or two (Adroit door: 278)
  unsigned char* cand = (unsigned char*)SI(cand);
  unsigned short* cand16 = (unsigned short*)SI(cand);
  const bool wide_cand = h->npair > 255;
  if (c.lane == 0) { cnt[CNT_NCON] = 0; cnt[CNT_NCAND] = 0; cnt[CNT_NGRP] = 0; }
  SYNC();
#if defined(B200_KITCHEN_GROUPS) && !defined(B200_KITCHEN_FLATSCAN)
  // broad phase, level 1: lanes over the bounding-volume groups (dmodel.h) -- one sphere fixed to a body against one anchor
  // geom (plane / the box itself / its bounding sphere); the survivors' pair runs are listed as (first pair, running count)
  uint32_t* surv = (uint32_t*)SI(surv);
  int nsurv = 0, npexp = 0;   // warp-uniform
  for (int base = 0; base < h->nbgrp; base += WARP_W) {
    int g = base + c.lane;
    bool hit = false;
    int npg = 0;
    if (g < h->nbgrp) {
      int b = MI(bg_body)[g], an = MI(bg_anchor)[g];
      float r = MF(bg_radius)[g], cw[3], rel[3];
      qrot(cw, SF(xquat) + 4 * b, MF(bg_center) + 3 * g);
      const float* xa = SF(geom_xpos) + 3 * an;
      for (int k = 0; k < 3; k++) rel[k] = SF(xpos)[3 * b + k] + cw[k] - xa[k];
      int ta = MI(geom_type)[an];
      if (ta == B200_GEOM_PLANE) hit = dot3(rel, MF(geom_size) + 3 * an) <= r;
      else if (ta == B200_GEOM_BOX) {
        float bp[3], bm[9], loc[3];
        geom_pose(c, an, bp, bm);
        mulmtv(loc, bm, rel);
        hit = box_sdist(loc, MF(geom_size) + 3 * an) <= r;
      } else { float bound = r + MF(geom_rbound)[an]; hit = dot3(rel, rel) <= bound * bound; }
      if (hit) npg = MI(bg_count)[g];
    }
    int total, slot = wexscan(hit ? 1 : 0, c.lane, &total);
    int ptotal, poff = wexscan(npg, c.lane, &ptotal);
    if (hit && nsurv + slot < DM_NSURV_MAX) surv[nsurv + slot] = (uint32_t)MI(bg_start)[g] | ((uint32_t)(npexp + poff) << 16);
    if (nsurv + total > DM_NSURV_MAX) {
      // more surviving groups than slots: the tail is dropped and flagged like a candidate overflow; the running count
      // must end at the last kept group
      int keep = DM_NSURV_MAX - nsurv;
      int kept_pairs = 0;
#ifdef B200_WARP_CODE
      kept_pairs = __shfl_sync(0xffffffffu, poff + npg, 31 - __clz(__ballot_sync(0xffffffffu, hit && slot < keep)));
#else
      kept_pairs = (hit && slot < keep) ? npg : 0;
#endif
      if (keep <= 0) kept_pairs = 0;
      if (c.lane == 0) cnt[CNT_OVERFLOW] |= 1;
      nsurv = DM_NSURV_MAX; npexp += kept_pairs;
    } else { nsurv += total; npexp += ptotal; }
  }
  if (c.lane == 0) surv[nsurv] = (uint32_t)npexp << 16;   // end marker
  SYNC();
  // level 2: lanes over the pairs of the surviving groups (the entry holding the i-th expanded pair by bisection)
  for (int base = 0; base < npexp; base += WARP_W) {
    int ei = base + c.lane, p = h->npair;
    if (ei < npexp) {
      int lo = 0, hi = nsurv;   // surv[lo].count <= ei < surv[hi].count
      while (hi - lo > 1) { int mid = (lo + hi) >> 1; if ((int)(surv[mid] >> 16) <= ei) lo = mid; else hi = mid; }
      p = (int)(surv[lo] & 0xffffu) + ei - (int)(surv[lo] >> 16);
    }
    bool hit = false;
    if (p < h->npair) {
#else
  // broad phase: lanes over the static pair list, ordered compaction
  for (int base = 0; base < h->npair; base += WARP_W) {
    int p = base + c.lane;
    bool hit = false;
    if (p < h->npair) {
#endif
      int g1 = PAIR_I(pair_geom1)[p], g2 = PAIR_I(pair_geom2)[p];
      float margin = PAIR_F(pair_margin)[p];
      const float *x1 = SF(geom_xpos) + 3 * g1, *x2 = SF(geom_xpos) + 3 * g2;
      float dif[3] = {x2[0] - x1[0], x2[1] - x1[1], x2[2] - x1[2]};
      if (g2 < 0) {
        // maze walls: any wall cell within reach of the geom's bounding sphere?
        float reach = MF(geom_rbound)[g1] + margin, s = h->grid_scale;
        const float* x = SF(geom_xpos) + 3 * g1;
        if (x[2] - reach <= h->grid_top) {
          int j0 = (int)floorf((x[0] - reach + h->grid_xc) / s), j1 = (int)floorf((x[0] + reach + h->grid_xc) / s);
          int i0 = (int)floorf((h->grid_yc - (x[1] + reach)) / s), i1 = (int)floorf((h->grid_yc - (x[1] - reach)) / s);
          for (int i = i0; i <= i1; i++)
            for (int j = j0; j <= j1; j++) {
              if (i < 0 || j < 0 || i >= h->grid_len || j >= h->grid_wid) continue;
              int bit = i * h->grid_wid + j;
              if ((MU(grid_walls)[bit >> 5] >> (bit & 31)) & 1u) hit = true;
            }
        }
      } else if (MI(geom_type)[g1] == B200_GEOM_PLANE) {
        // planes live on the world body: dm_build stores the world normal in the (otherwise unused) size slot
        const float* n = MF(geom_size) + 3 * g1;
        hit = dot3(dif, n) <= margin + MF(geom_rbound)[g2];
      } else {
        float bound = margin + MF(geom_rbound)[g1] + MF(geom_rbound)[g2];
        hit = dot3(dif, dif) <= bound * bound;
#ifdef B200_KITCHEN
        // large boxes (counters, doors): the bounding sphere of a box is loose, so test the other geom's bounding sphere
        // against the box itself (distance of its centre in the box frame); still conservative
        for (int side = 0; side < 2 && hit; side++) {
          int gb = side ? g1 : g2, go = side ? g2 : g1;
          if (MI(geom_type)[gb] != B200_GEOM_BOX) continue;
          float bp[3], bm[9], rel[3], loc[3];
          geom_pose(c, gb, bp, bm);
          const float* xo = SF(geom_xpos) + 3 * go;
          rel[0] = xo[0] - bp[0]; rel[1] = xo[1] - bp[1]; rel[2] = xo[2] - bp[2];
          mulmtv(loc, bm, rel);
          hit = box_sdist(loc, MF(geom_size) + 3 * gb) <= margin + MF(geom_rbound)[go];
        }
#endif
      }
    }
    int total, slot = wexscan(hit ? 1 : 0, c.lane, &total);
    int basec = cnt[CNT_NCAND];
    SYNC();
    if (hit && basec + slot < h->ncand_max) { if (wide_cand) cand16[basec + slot] = (unsigned short)p; else cand[basec + slot] = (unsigned char)p; }
    if (c.lane == 0) { int nn = basec + total; if (nn > h->ncand_max) { nn = h->ncand_max; cnt[CNT_OVERFLOW] |= 1; } cnt[CNT_NCAND] = nn; }
    SYNC();
  }
  // narrow phase: one lane per candidate pair (lock-step over identical pair types in the common case), `nslot` pairs per
  // round: every working lane owns a BoxScratch slot in shared memory (the result record itself stays on the lane's stack)
  int ncand = cnt[CNT_NCAND];
  const int nslotA = h->ncslotA, nslotAB = nslotA + h->ncslotB;
  // no __isShared assumption on this per-lane select between two scratch regions: with one, nvcc 12.9 miscompiled the kernel
  // (invalid __shared__ reads in the next broad phase on the GPU)
  BoxScratch& bs = *(BoxScratch*)(c.lane < nslotA ? c.s + h->s_cslotA + c.lane * DM_CSLOT_WORDS
                                                  : c.s + h->s_cslotB + ((c.lane < nslotAB ? c.lane : nslotA) - nslotA) * DM_CSLOT_WORDS);
  for (int base = 0, nslot = 0; base < ncand; base += nslot) {
    // region B is the contact-record array itself: usable as long as no record has been written (always in the first round)
    nslot = cnt[CNT_NCON] == 0 ? nslotAB : nslotA;
    if (nslot > WARP_W) nslot = WARP_W;   // (the one-lane host emulation walks the candidates one by one)
    int ci = base + c.lane;
    ContactOut o;
    o.cnt = 0;
    int p = -1;
    if (c.lane < nslot && ci < ncand) {
      p = wide_cand ? (int)cand16[ci] : (int)cand[ci];
      int g1 = PAIR_I(pair_geom1)[p], g2 = PAIR_I(pair_geom2)[p];
      float margin = PAIR_F(pair_margin)[p];
      int t1 = MI(geom_type)[g1], t2 = g2 < 0 ? B200_GEOM_BOX : MI(geom_type)[g2];
#ifdef B200_HULL
      const bool cv1 = t1 == B200_GEOM_CYLINDER || t1 == B200_GEOM_ELLIPSOID || t1 == B200_GEOM_MESH,
                 cv2 = t2 == B200_GEOM_CYLINDER || t2 == B200_GEOM_ELLIPSOID || t2 == B200_GEOM_MESH;
#else
      const bool cv1 = t1 == B200_GEOM_CYLINDER || t1 == B200_GEOM_ELLIPSOID, cv2 = t2 == B200_GEOM_CYLINDER || t2 == B200_GEOM_ELLIPSOID;
#endif
      if (CX && (cv1 || cv2)) {
        if (t1 == B200_GEOM_PLANE) collide_plane_convex(c, g1, g2, margin, o);
        else collide_convex(c, g1, g2, margin, o);
      } else if (t1 == B200_GEOM_PLANE) {
        if (t2 == B200_GEOM_BOX) collide_plane_box(c, g1, g2, margin, o);
        else if (t2 == B200_GEOM_SPHERE) collide_plane_sphere(c, g1, g2, margin, o);
        else collide_plane_capsule(c, g1, g2, margin, o);
      } else if (t1 == B200_GEOM_BOX) collide_box_box(c, g1, g2, margin, o, bs);
      else if (t2 == B200_GEOM_BOX) collide_round_box(c, g1, g2, margin, o);
      else if (HF) collide_round_round(c, g1, g2, margin, o);
      // contacts beyond the gap are not turned into constraints
      float inc = margin - GF(pair_gap)[p];
      int k2 = 0;
      for (int k = 0; k < o.cnt; k++) if (o.dist[k] < inc) { if (k2 != k) { o.dist[k2] = o.dist[k]; for (int a = 0; a < 3; a++) { o.pos[k2][a] = o.pos[k][a]; o.nrm[k2][a] = o.nrm[k][a]; } } k2++; }
      o.cnt = k2;
    }
    int ocnt = o.cnt;
    int gtotal, gslot = wexscan(ocnt > 0 ? 1 : 0, c.lane, &gtotal);
    int basec = cnt[CNT_NCON], baseg = cnt[CNT_NGRP];
    int gid = baseg + gslot;
    // a geom pair beyond the group capacity is dropped with all its contacts BEFORE the contacts are numbered: every
    // counted contact record is then really written (a counted but unwritten record would be finalised from stale words)
    if (ocnt > 0 && gid >= h->ngrp_max - DM_NWELD_MAX) ocnt = 0;
    int total, slot = wexscan(ocnt, c.lane, &total);
    // (the slots of region B overlay the contact records written below: BoxScratch is dead by now)
    SYNC();
    int kept = 0;
    for (int k = 0; k < ocnt; k++) {
      // raw contact (position, normal, distance, pair) parked in its record; finalised by one lane per contact below
      int id = basec + slot + k;
      if (id >= h->ncon_max) break;
      float* cr = SF(con) + id * CON_WORDS;
      cr[0] = o.pos[k][0]; cr[1] = o.pos[k][1]; cr[2] = o.pos[k][2];
      cr[3] = o.nrm[k][0]; cr[4] = o.nrm[k][1]; cr[5] = o.nrm[k][2];
      cr[6] = o.dist[k];
      ((int*)cr)[7] = p;
      ((int*)cr)[C_DIMGRP] = gid << 8;
      kept++;
    }
    if (ocnt > 0) {
      int* gi = (int*)(SF(group) + gid * GRP_WORDS);
      int ba = MI(geom_body)[PAIR_I(pair_geom1)[p]], bb = PAIR_I(pair_geom2)[p] < 0 ? 0 : MI(geom_body)[PAIR_I(pair_geom2)[p]];
      dmask_t ma = DM(body_ancdof, ba), mb = DM(body_ancdof, bb);
      // the pair's two MJCF (unfused) bodies, A | B << 8 (world / maze walls: 0): rows of per-body contact forces
      const int bodies = GI(geom_mjb)[PAIR_I(pair_geom1)[p]] | ((PAIR_I(pair_geom2)[p] < 0 ? 0 : GI(geom_mjb)[PAIR_I(pair_geom2)[p]]) << 8);
      ((uint32_t*)gi)[G_RANGE] = (uint32_t)(basec + slot) | (uint32_t)kept << 8 | (uint32_t)bodies << 16;
      grp_set_masks(gi, ma ^ mb, mb);
    }
    if (c.lane == 0) {
      int nn = basec + total; if (nn > h->ncon_max) { nn = h->ncon_max; cnt[CNT_OVERFLOW] |= 2; }
      int ng = baseg + gtotal; if (ng > h->ngrp_max - DM_NWELD_MAX) { ng = h->ngrp_max - DM_NWELD_MAX; cnt[CNT_OVERFLOW] |= 4; }
      cnt[CNT_NCON] = nn; cnt[CNT_NGRP] = ng;
    }
    SYNC();
  }
  // contact records: frame, spatial row vectors about `ref`, friction, impedance / regulariser / reference-acceleration
  // constants -- one lane per contact
  LANES(id, cnt[CNT_NCON]) {
    float* cr = SF(con) + id * CON_WORDS;
    const float pos[3] = {cr[0], cr[1], cr[2]}, dist = cr[6];
    float fr9[9] = {cr[3], cr[4], cr[5], 0, 0, 0, 0, 0, 0};
    const int p = ((const int*)cr)[7], gid8 = ((const int*)cr)[C_DIMGRP];
    make_frame(fr9);
    float r[3] = {pos[0] - h->ref[0], pos[1] - h->ref[1], pos[2] - h->ref[2]};
    for (int a = 0; a < 3; a++) { float* w = cr + C_W + 6 * a; cross3(w, r, fr9 + 3 * a); w[3] = fr9[3 * a]; w[4] = fr9[3 * a + 1]; w[5] = fr9[3 * a + 2]; }
    const float* fr = GF(pair_friction) + 3 * p;
    int dim = GI(pair_condim)[p];
    float mu0 = fr[0];
    cr[C_MU] = mu0; cr[C_MU + 1] = fr[1];
#ifdef B200_KITCHEN
    cr[C_MU + 2] = fr[2];   // rolling friction (condim 6)
#endif
    float incl = PAIR_F(pair_margin)[p] - GF(pair_gap)[p];
    float solimp[5] = {GF(pair_solimp)[5 * p], GF(pair_solimp)[5 * p + 1], GF(pair_solimp)[5 * p + 2], GF(pair_solimp)[5 * p + 3], GF(pair_solimp)[5 * p + 4]};
    float solref[2] = {GF(pair_solref)[2 * p], GF(pair_solref)[2 * p + 1]};
    float imp = impedance(solimp, dist, incl);
    float K, Bc;
    ref_kb(c, solref, solimp[1], &K, &Bc);
    float tran = GF(pair_invweight)[2 * p];
    float R;
    if (dim == 1) R = fmaxf((1 - imp) / imp * tran, B200_MINVAL);
    else {
      float R0 = fmaxf((1 - imp) / imp * (tran + mu0 * mu0 * tran), B200_MINVAL);
      float mu = mu0 * rsqrtf(h->impratio);
      R = fmaxf(2 * mu * mu * R0, B200_MINVAL);
    }
    cr[C_D] = 1.0f / R;
    cr[C_U] = K * imp * (dist - incl); cr[C_U + 1] = 0; cr[C_U + 2] = 0; cr[C_U + 3] = 0;
#ifdef B200_KITCHEN
    cr[C_U + 4] = 0; cr[C_U + 5] = 0;
#endif
    cr[C_JV] = Bc;
    ((int*)cr)[C_DIMGRP] = dim | gid8;
    if (HF && h->nsensor > 0) {
      float* cx = SF(conx) + id * CX_WORDS;
      cx[CX_POS] = pos[0]; cx[CX_POS + 1] = pos[1]; cx[CX_POS + 2] = pos[2];
      ((int*)cx)[CX_PAIR] = p;
    }
  }
  SYNC();
}

// ---------------------------------------------------------------------------------------------------------------
// 6. constraint rows
// spatial vector of contact base row k (about ref): k<3 translational rows are cached in C_W, k==3 is the torsional row
#ifdef B200_KITCHEN
// base row k: 0..2 translational (cached), 3 torsional = (n, 0), 4 / 5 rolling = (t1, 0) / (t2, 0)
HD void con_w(const float* cr, int k, float* w) {
  if (k < 3) { const float* s = cr + C_W + 6 * k; w[0] = s[0]; w[1] = s[1]; w[2] = s[2]; w[3] = s[3]; w[4] = s[4]; w[5] = s[5]; }
  else { const float* s = cr + C_W + 6 * (k - 3) + 3; w[0] = s[0]; w[1] = s[1]; w[2] = s[2]; w[3] = w[4] = w[5] = 0; }
}
HD float con_mu(const float* cr, int k) { return k < 3 ? cr[C_MU] : (k == 3 ? cr[C_MU + 1] : cr[C_MU + 2]); }  // base row k >= 1
#else
HD void con_w(const float* cr, int k, float* w) {
  if (k < 3) { const float* s = cr + C_W + 6 * k; w[0] = s[0]; w[1] = s[1]; w[2] = s[2]; w[3] = s[3]; w[4] = s[4]; w[5] = s[5]; }
  else { w[0] = cr[C_W + 3]; w[1] = cr[C_W + 4]; w[2] = cr[C_W + 5]; w[3] = w[4] = w[5] = 0; }
}
HD float con_mu(const float* cr, int k) { return k < 3 ? cr[C_MU] : cr[C_MU + 1]; }  // base row k >= 1
#endif
// C_DIMGRP: condim (8 bits), group (8 bits), and from the solver's first check on the activity of the contact's edges at the
// current point (bit 0: u_n < 0 of a frictionless contact; pyramid: bit 2 (k - 1) u_n + mu u_k < 0, bit 2 (k - 1) + 1 u_n - mu u_k < 0)
HD int con_dim(const float* cr) { return ((const int*)cr)[C_DIMGRP] & 0xff; }
HD int con_grp(const float* cr) { return (((const int*)cr)[C_DIMGRP] >> 8) & 0xff; }
HD uint32_t con_act(const float* cr) { return ((const uint32_t*)cr)[C_DIMGRP] >> 16; }

template <bool HF>
STAGE void make_constraint(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  int* cnt = SI(counters);
  if (c.lane == 0) { cnt[CNT_NDR] = 0; cnt[CNT_NWELD] = 0; }
  SYNC();
  // weld equalities (at most DM_NWELD_MAX): every lane evaluates the warp-uniform poses, lane k < 6 then builds row k
  for (int e = 0; e < h->neq; e++) {
    if (!MI(eq_active)[e] || MI(eq_type)[e] != B200_EQ_WELD) continue;
    const int nw = cnt[CNT_NWELD], gid = cnt[CNT_NGRP];
    float* wr = SF(weld) + nw * WELD_WORDS;
    const float* data = MF(eq_data) + 11 * e;
    int s1 = MI(eq_obj1)[e], s2 = MI(eq_obj2)[e], b1 = 0, b2 = 0;
    float p1[3] = {0, 0, 0}, p2[3] = {0, 0, 0}, q1[4] = {1, 0, 0, 0}, q2[4] = {1, 0, 0, 0}, t[3];
    if (s1 >= 0) { b1 = MI(site_body)[s1]; qmul(q1, SF(xquat) + 4 * b1, MF(site_quat) + 4 * s1); qrot(t, SF(xquat) + 4 * b1, MF(site_pos) + 3 * s1); for (int k = 0; k < 3; k++) p1[k] = SF(xpos)[3 * b1 + k] + t[k]; }
    if (s2 >= 0) { b2 = MI(site_body)[s2]; qmul(q2, SF(xquat) + 4 * b2, MF(site_quat) + 4 * s2); qrot(t, SF(xquat) + 4 * b2, MF(site_pos) + 3 * s2); for (int k = 0; k < 3; k++) p2[k] = SF(xpos)[3 * b2 + k] + t[k]; }
    qrot(t, q1, data + 3); for (int k = 0; k < 3; k++) p1[k] += t[k];
    qrot(t, q2, data + 0); for (int k = 0; k < 3; k++) p2[k] += t[k];
    const float ts = data[10];
    float quat[4], quat1[4] = {q2[0], -q2[1], -q2[2], -q2[3]}, quat2[4];
    qmul(quat, q1, data + 6);
    qmul(quat2, quat1, quat);
    // rows: J = J(body1 at p1) - J(body2 at p2); translational rows about the anchor of the side that carries dofs
    const bool use1 = b1 > 0 && DM(body_ancdof, b1) != 0;
    float r[3];
    for (int k = 0; k < 3; k++) r[k] = (use1 ? p1[k] : p2[k]) - h->ref[k];
    float K, Bc;
    ref_kb(c, MF(eq_solref) + 2 * e, MF(eq_solimp)[5 * e + 1], &K, &Bc);
    LANES(k, 6) {
      float* w = wr + W_W + 6 * k;
      float cp;
      if (k < 3) {
        float e3[3] = {k == 0 ? 1.f : 0.f, k == 1 ? 1.f : 0.f, k == 2 ? 1.f : 0.f};
        cross3(w, r, e3); w[3] = e3[0]; w[4] = e3[1]; w[5] = e3[2];
        cp = k == 0 ? p1[0] - p2[0] : (k == 1 ? p1[1] - p2[1] : p1[2] - p2[2]);
      } else {
        const int kk = k - 3;
        for (int a = 0; a < 3; a++) {  // column a of the 3x3 map (relative angular velocity -> residual rate)
          float qa[4] = {0, a == 0 ? 1.f : 0.f, a == 1 ? 1.f : 0.f, a == 2 ? 1.f : 0.f}, t1[4], t2[4];
          qmul(t1, quat1, qa); qmul(t2, t1, quat);
          w[a] = 0.5f * ts * (kk == 0 ? t2[1] : (kk == 1 ? t2[2] : t2[3])); w[3 + a] = 0;
        }
        cp = ts * (kk == 0 ? quat2[1] : (kk == 1 ? quat2[2] : quat2[3]));
      }
      float imp = impedance(MF(eq_solimp) + 5 * e, cp, 0.f);
      float R = fmaxf((1 - imp) / imp * MF(eq_invweight)[2 * e + (k < 3 ? 0 : 1)], B200_MINVAL);
      wr[W_D + k] = 1.0f / R; wr[W_JAR + k] = K * imp * cp;
    }
    if (c.lane == 0) {
      wr[W_B] = Bc;
      ((int*)wr)[W_GRP] = gid;  // one group per weld; row value = w . (V[b1] - V[b2]) => A = b2, B = b1
      int* gi = (int*)(SF(group) + gid * GRP_WORDS);
      dmask_t ma = DM(body_ancdof, b2), mb = DM(body_ancdof, b1);
      gi[G_RANGE] = 0;
      grp_set_masks(gi, ma ^ mb, mb);
    }
    SYNC();
    if (c.lane == 0) { cnt[CNT_NGRP] = gid + 1; cnt[CNT_NWELD] = nw + 1; }
    SYNC();
  }
  // joint limits -> dof rows (ordered compaction over joints, lower side first)
  for (int base = 0; base < h->njnt; base += WARP_W) {
    int j = base + c.lane;
    // (the lower-side row first, then the upper-side one: two scalars each instead of runtime-indexed arrays)
    int nrow = 0; float dist0 = 0, dist1 = 0, sgn0 = 0, sgn1 = 0;
    if (j < h->njnt && MI(jnt_limited)[j] && MI(jnt_type)[j] != B200_JNT_FREE) {
      float q = SF(qpos)[MI(jnt_qposadr)[j]], margin = MF(jnt_margin)[j];
      float dl = q - MF(jnt_range)[2 * j], du = MF(jnt_range)[2 * j + 1] - q;
      if (dl < margin) { dist0 = dl; sgn0 = 1.f; nrow = 1; }
      if (du < margin) { if (nrow) { dist1 = du; sgn1 = -1.f; } else { dist0 = du; sgn0 = -1.f; } nrow++; }
    }
    int total, slot = wexscan(nrow, c.lane, &total);
    int basec = cnt[CNT_NDR];
    SYNC();
#pragma unroll
    for (int k = 0; k < 2; k++) {
      int id = basec + slot + k;
      if (k >= nrow || id >= h->ndr_max) continue;
      const float distk = k ? dist1 : dist0, sgnk = k ? sgn1 : sgn0;
      float* dr = SF(dofrow) + id * DR_WORDS;
      int* di = (int*)dr;
      int d = MI(jnt_dofadr)[j];
      float margin = MF(jnt_margin)[j];
      float solimp[5] = {GF(jnt_solimp)[5 * j], GF(jnt_solimp)[5 * j + 1], GF(jnt_solimp)[5 * j + 2], GF(jnt_solimp)[5 * j + 3], GF(jnt_solimp)[5 * j + 4]};
      float solref[2] = {GF(jnt_solref)[2 * j], GF(jnt_solref)[2 * j + 1]};
      float imp = impedance(solimp, distk, margin);
      float K, Bc;
      ref_kb(c, solref, solimp[1], &K, &Bc);
      float R = fmaxf((1 - imp) / imp * MF(dof_invweight0)[d], B200_MINVAL);
      di[DR_DOF] = d; dr[DR_COEF] = sgnk; di[DR_DOF2] = -1; dr[DR_COEF2] = 0;
      dr[DR_D] = 1.0f / R; dr[DR_JAR] = K * imp * (distk - margin); dr[DR_JV] = Bc;
    }
    if (c.lane == 0) { int nn = basec + total; if (nn > h->ndr_max) { nn = h->ndr_max; cnt[CNT_OVERFLOW] |= 8; } cnt[CNT_NDR] = nn; }
    SYNC();
  }
  // limits of fixed tendons (length = sum coef * qpos over <= 2 joints) -> dof rows, lower side first
  if (HF) for (int base = 0; base < h->nten; base += WARP_W) {
    int t = base + c.lane;
    int nrow = 0; float dist0 = 0, dist1 = 0, sgn0 = 0, sgn1 = 0;
    if (t < h->nten) {
      float len = MF(ten_coef)[2 * t] * SF(qpos)[MI(ten_qadr)[2 * t]];
      if (MI(ten_dof)[2 * t + 1] >= 0) len += MF(ten_coef)[2 * t + 1] * SF(qpos)[MI(ten_qadr)[2 * t + 1]];
      float margin = MF(ten_margin)[t];
      float dl = len - MF(ten_range)[2 * t], du = MF(ten_range)[2 * t + 1] - len;
      if (dl < margin) { dist0 = dl; sgn0 = 1.f; nrow = 1; }
      if (du < margin) { if (nrow) { dist1 = du; sgn1 = -1.f; } else { dist0 = du; sgn0 = -1.f; } nrow++; }
    }
    int total, slot = wexscan(nrow, c.lane, &total);
    int basec = cnt[CNT_NDR];
    SYNC();
#pragma unroll
    for (int k = 0; k < 2; k++) {
      int id = basec + slot + k;
      if (k >= nrow || id >= h->ndr_max) continue;
      const float distk = k ? dist1 : dist0, sgnk = k ? sgn1 : sgn0;
      float* dr = SF(dofrow) + id * DR_WORDS;
      int* di = (int*)dr;
      float margin = MF(ten_margin)[t];
      float solimp[5] = {GF(ten_solimp)[5 * t], GF(ten_solimp)[5 * t + 1], GF(ten_solimp)[5 * t + 2], GF(ten_solimp)[5 * t + 3], GF(ten_solimp)[5 * t + 4]};
      float solref[2] = {GF(ten_solref)[2 * t], GF(ten_solref)[2 * t + 1]};
      float imp = impedance(solimp, distk, margin);
      float K, Bc;
      ref_kb(c, solref, solimp[1], &K, &Bc);
      float R = fmaxf((1 - imp) / imp * GF(ten_invweight)[t], B200_MINVAL);
      di[DR_DOF] = MI(ten_dof)[2 * t]; dr[DR_COEF] = sgnk * MF(ten_coef)[2 * t];
      di[DR_DOF2] = MI(ten_dof)[2 * t + 1]; dr[DR_COEF2] = sgnk * MF(ten_coef)[2 * t + 1];
      dr[DR_D] = 1.0f / R; dr[DR_JAR] = K * imp * (distk - margin); dr[DR_JV] = Bc;
    }
    if (c.lane == 0) { int nn = basec + total; if (nn > h->ndr_max) { nn = h->ndr_max; cnt[CNT_OVERFLOW] |= 8; } cnt[CNT_NDR] = nn; }
    SYNC();
  }
#ifdef B200_KITCHEN
  // joint equalities q1 - q1_0 = poly(q2 - q2_0) (oven knobs <-> burners of the kitchen model) as two-sided dof rows:
  // coefficients (1, -poly'), D < 0 marks the row as two-sided for the solver stages  [bring-up build only]
  if (c.lane == 0) {
    for (int e = 0; e < h->neq; e++) {
      if (!MI(eq_active)[e] || MI(eq_type)[e] != B200_EQ_JOINT) continue;
      int id = cnt[CNT_NDR];
      if (id >= h->ndr_max) { cnt[CNT_OVERFLOW] |= 8; break; }
      const float* data = MF(eq_data) + 11 * e;
      int j1 = MI(eq_obj1)[e], j2 = MI(eq_obj2)[e];
      float pos = SF(qpos)[MI(jnt_qposadr)[j1]] - MF(jnt_qpos0)[j1], deriv = 0.f;
      if (j2 >= 0) {
        float dif = SF(qpos)[MI(jnt_qposadr)[j2]] - MF(jnt_qpos0)[j2];
        pos -= data[0] + dif * (data[1] + dif * (data[2] + dif * (data[3] + dif * data[4])));
        deriv = data[1] + dif * (2 * data[2] + dif * (3 * data[3] + dif * 4 * data[4]));
      } else pos -= data[0];
      float* dr = SF(dofrow) + id * DR_WORDS;
      int* di = (int*)dr;
      float imp = impedance(MF(eq_solimp) + 5 * e, pos, 0.f);
      float K, Bc;
      ref_kb(c, MF(eq_solref) + 2 * e, MF(eq_solimp)[5 * e + 1], &K, &Bc);
      float R = fmaxf((1 - imp) / imp * MF(eq_invweight)[2 * e], B200_MINVAL);
      di[DR_DOF] = MI(jnt_dofadr)[j1]; dr[DR_COEF] = 1.f;
      di[DR_DOF2] = j2 >= 0 ? MI(jnt_dofadr)[j2] : -1; dr[DR_COEF2] = -deriv;
      dr[DR_D] = -1.0f / R; dr[DR_JAR] = K * imp * pos; dr[DR_JV] = Bc;
      cnt[CNT_NDR] = id + 1;
    }
  }
  SYNC();
#endif
  // dof frictionloss rows: position residual 0, so the row value starts at 0
  if (HF) { LANES(d, h->nfric) SF(fric)[d] = 0.f; SYNC(); }
}

// base-row generalized forces of a contact from its base-row values U (pyramid edges f = -D * min(0, u_n +- mu u_k)).  Returns
// the activity of the edges, in the layout of con_act(): the solver stores it in the record for build_H.
HD uint32_t contact_base_forces(const float* cr, int dim, const float (&U)[C_NB], float* F) {
  float D = cr[C_D], un = U[0];
#pragma unroll
  for (int k = 0; k < C_NB; k++) F[k] = 0;
  if (dim == 1) { F[0] = un < 0 ? -D * un : 0.f; return un < 0 ? 1u : 0u; }
  uint32_t act = 0;
#pragma unroll
  for (int k = 1; k < C_NB; k++) {   // (statically indexed so that U and F stay in registers)
    if (k >= dim) continue;
    float mu = con_mu(cr, k), uk = U[k];
    float xp = un + mu * uk, xm = un - mu * uk;
    float fp = xp < 0 ? -D * xp : 0.f, fm = xm < 0 ? -D * xm : 0.f;
    act |= (xp < 0 ? 1u : 0u) << (2 * k - 2) | (xm < 0 ? 1u : 0u) << (2 * k - 1);
    F[0] += fp + fm;
    F[k] = mu * (fp - fm);
  }
  return act;
}
// the same from the values stored in the record
HD void contact_base_forces(const float* cr, int dim, float* F) {
  float U[C_NB];
#pragma unroll
  for (int k = 0; k < C_NB; k++) U[k] = cr[C_U + k];
  contact_base_forces(cr, dim, U, F);
}
// the solver's contact update: the base-row forces of the new values U parked in the JV slots (read by pass_F, rewritten by the
// next J * search product) and the edge activity in the record (read by build_H)
HD void contact_park_forces(float* cr, const float (&U)[C_NB]) {
  int* dg = (int*)cr + C_DIMGRP;
  float F[C_NB];
  const uint32_t act = contact_base_forces(cr, *dg & 0xff, U, F);
#pragma unroll
  for (int k = 0; k < C_NB; k++) cr[C_JV + k] = F[k];
  *dg = (int)(((uint32_t)*dg & 0xffffu) | act << 16);
}

// JV slots of every row <- J * vec (the search direction); the opening passes J qvel / J qacc are fused in rows_begin()
template <bool HF>
STAGE void rows_from_vec(const Ctx c, const float* vec) {
  ASSUME_SHARED(c);
  ASSUME_SHARED_PTR(vec);
  const int* cnt = SI(counters);
  int ngrp = cnt[CNT_NGRP];
  // per-group relative spatial velocity dV_g = sum_{j in S_g} sigma_gj cdof_j vec_j  (lane = (group, component))
  LANES(idx, ngrp * 6) {
    int g = idx / 6, a = idx - 6 * g;
    float* gr = SF(group) + g * GRP_WORDS;
    dmask_t S = grp_mask(gr), sg = grp_sign(gr);
    float acc = 0;
    while (S) { int j = ffs_pop(S); float t = SF(cdof)[6 * j + a] * vec[j]; acc += DBIT(sg, j) ? t : -t; }
    gr[G_V + a] = acc;
  }
  SYNC();
  LANES(i, cnt[CNT_NCON]) {
    float* cr = SF(con) + i * CON_WORDS;
    int dim = con_dim(cr), nbase = dim == 1 ? 1 : dim;
    const float* dV = SF(group) + con_grp(cr) * GRP_WORDS + G_V;
    for (int k = 0; k < nbase; k++) {
      float w[6];
      con_w(cr, k, w);
      cr[C_JV + k] = dot6(w, dV);
    }
  }
  LANES(i, cnt[CNT_NWELD] * 6) {
    float* wr = SF(weld) + (i / 6) * WELD_WORDS;
    int k = i % 6;
    const float* dV = SF(group) + ((const int*)wr)[W_GRP] * GRP_WORDS + G_V;
    wr[W_JV + k] = dot6(wr + W_W + 6 * k, dV);
  }
  LANES(i, cnt[CNT_NDR]) {
    float* dr = SF(dofrow) + i * DR_WORDS;
    const int* di = (const int*)dr;
    float val = dr[DR_COEF] * vec[di[DR_DOF]];
    if (di[DR_DOF2] >= 0) val += dr[DR_COEF2] * vec[di[DR_DOF2]];
    dr[DR_JV] = val;
  }
  if (HF) LANES(d, c.h->nfric) SF(fric)[c.h->nfric + d] = vec[d];
  SYNC();
}

// the two row passes that open the solver, fused: rows <- rows + B * (J qvel) + J qacc (same arithmetic and order as
// two separate passes row += B * (J qvel), row += J qacc); the second group velocity is parked at 6 g in the H region,
// which build_H fills later)
template <bool HF>
STAGE void rows_begin(const Ctx c, const float* qvel, const float* qacc) {
  ASSUME_SHARED(c);
  ASSUME_SHARED_PTR(qvel); ASSUME_SHARED_PTR(qacc);
  const int* cnt = SI(counters);
  int ngrp = cnt[CNT_NGRP];
  float* dA = SF(H);
  LANES(idx, ngrp * 6) {
    int g = idx / 6, a = idx - 6 * g;
    float* gr = SF(group) + g * GRP_WORDS;
    dmask_t S = grp_mask(gr), sg = grp_sign(gr);
    float acc = 0, acc2 = 0;
    while (S) {
      int j = ffs_pop(S);
      float cd = SF(cdof)[6 * j + a], t = cd * qvel[j], t2 = cd * qacc[j];
      bool pos = DBIT(sg, j);
      acc += pos ? t : -t; acc2 += pos ? t2 : -t2;
    }
    gr[G_V + a] = acc; dA[idx] = acc2;
  }
  SYNC();
  LANES(i, cnt[CNT_NCON]) {
    float* cr = SF(con) + i * CON_WORDS;
    int dim = con_dim(cr), nbase = dim == 1 ? 1 : dim;
    const float* gr = SF(group) + con_grp(cr) * GRP_WORDS;
    const float* gA = dA + 6 * con_grp(cr);
    float Bc = cr[C_JV];
    float U[C_NB];
#pragma unroll
    for (int k = 0; k < C_NB; k++) {   // (statically indexed so that U stays in registers)
      U[k] = 0.f;
      if (k >= nbase) continue;
      float w[6];
      con_w(cr, k, w);
      float u = cr[C_U + k];
      u += Bc * dot6(w, gr + G_V);
      u += dot6(w, gA);
      cr[C_U + k] = u;
      U[k] = u;
    }
    contact_park_forces(cr, U);   // for the solver's first check (Bc is not read again)
  }
  LANES(i, cnt[CNT_NWELD] * 6) {
    float* wr = SF(weld) + (i / 6) * WELD_WORDS;
    int k = i % 6;
    const int g = ((const int*)wr)[W_GRP];
    const float* gr = SF(group) + g * GRP_WORDS;
    float u = wr[W_JAR + k];
    u += wr[W_B] * dot6(wr + W_W + 6 * k, gr + G_V);
    u += dot6(wr + W_W + 6 * k, dA + 6 * g);
    wr[W_JAR + k] = u;
  }
  LANES(i, cnt[CNT_NDR]) {
    float* dr = SF(dofrow) + i * DR_WORDS;
    const int* di = (const int*)dr;
    float v1 = dr[DR_COEF] * qvel[di[DR_DOF]], v2 = dr[DR_COEF] * qacc[di[DR_DOF]];
    if (di[DR_DOF2] >= 0) { v1 += dr[DR_COEF2] * qvel[di[DR_DOF2]]; v2 += dr[DR_COEF2] * qacc[di[DR_DOF2]]; }
    float u = dr[DR_JAR];
    u += dr[DR_JV] * v1;
    u += v2;
    dr[DR_JAR] = u;
  }
  if (HF) LANES(d, c.h->nfric) {
    float* fr = SF(fric);
    float u = fr[d];
    u += MF(dof_fricB)[d] * qvel[d];
    u += qacc[d];
    fr[d] = u;
  }
  SYNC();
}

// ---------------------------------------------------------------------------------------------------------------
// 8. Newton solver pieces
// fcon = J^T f from the base-row forces that the contact update parked in the JV slots (contact_park_forces, followed by a
// SYNC): per-group spatial force, then one 6-dot per (dof, group)
template <bool HF>
HD void pass_F(const Ctx c, float* out) {
  // (no ASSUME_SHARED_PTR(out): with it, nvcc 12.9 compiled the check inlined into newton_begin / newton_move as unreachable
  // and dropped it; tests/test_newton_fused_check.py looks for the check in both)
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  const int* cnt = SI(counters);
  int ngrp = cnt[CNT_NGRP], nweld = cnt[CNT_NWELD], ndr = cnt[CNT_NDR];
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
#ifdef B200_KITCHEN
      if (dim > 4 && a < 3) acc += F[4] * cr[C_W + 6 + 3 + a] + F[5] * cr[C_W + 12 + 3 + a];
#endif
    }
    for (int i = 0; i < nweld; i++) {
      const float* wr = SF(weld) + i * WELD_WORDS;
      if (((const int*)wr)[W_GRP] != g) continue;
      for (int k = 0; k < 6; k++) acc -= wr[W_D + k] * wr[W_JAR + k] * wr[W_W + 6 * k + a];
    }
    gr[G_V + a] = acc;
  }
  SYNC();
  LANES(j, h->nv) {
    float q = 0;
    const float* cd = SF(cdof) + 6 * j;
    for (int g = 0; g < ngrp; g++) {
      const float* gr = SF(group) + g * GRP_WORDS;
      if (!DBIT(grp_mask(gr), j)) continue;
      float d = dot6(cd, gr + G_V);
      q += DBIT(grp_sign(gr), j) ? d : -d;
    }
    for (int i = 0; i < ndr; i++) {
      const float* dr = SF(dofrow) + i * DR_WORDS;
      const int* di = (const int*)dr;
      float x = dr[DR_JAR];
#ifdef B200_KITCHEN
      float f = (dr[DR_D] < 0 || x < 0) ? -fabsf(dr[DR_D]) * x : 0.f;   // D < 0: two-sided (equality) row
#else
      float f = x < 0 ? -dr[DR_D] * x : 0.f;
#endif
      if (di[DR_DOF] == j) q += dr[DR_COEF] * f;
      if (di[DR_DOF2] == j) q += dr[DR_COEF2] * f;
    }
    if (HF && h->nfric) {
      // Huber-type friction row: force -D x clamped to +-frictionloss
      float fl = MF(dof_frictionloss)[j];
      q += fminf(fmaxf(-MF(dof_fricD)[j] * SF(fric)[j], -fl), fl);
    }
    out[j] = q;
  }
  SYNC();
}

STAGE void mulM(const Ctx c, const float* v, float* out) {
  ASSUME_SHARED(c);
  ASSUME_SHARED_PTR(v); ASSUME_SHARED_PTR(out);
  int nv = c.h->nv;
  const float* M = SF(M);
  LANES(i, nv) {
    float a = 0;
    const int row = i * (i + 1) / 2;
    for (int j = 0; j <= i; j++) a += M[row + j] * v[j];                           // row part of the packed lower triangle
    for (int j = i + 1, idx = row + 2 * i + 1; j < nv; idx += ++j) a += M[idx] * v[j];   // column part: idx = j (j + 1) / 2 + i
    out[i] = a;
  }
  SYNC();
}

// H = M + sum_g S_g^T K_g S_g  (+ dof rows on the diagonal blocks)
template <bool HF>
STAGE void build_H(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  const int* cnt = SI(counters);
  int nv = h->nv, nM = nv * (nv + 1) / 2, nweld = cnt[CNT_NWELD], ngrp = cnt[CNT_NGRP], ndr = cnt[CNT_NDR];
  float* H = SF(H);
  LANES(i, nM) H[i] = SF(M)[i];
  // K blocks in the dead solver scratch after H (room for >= 1, dmodel.h), in chunks of as many groups as fit it: every H entry
  // still sums its groups in ascending order
  float* Kc = H + nM;
  const int kcap = (h->s_grad - h->s_H - nM) / 21;
  for (int g0 = 0; g0 < ngrp; g0 += kcap) {
    const int g1 = ngrp - g0 < kcap ? ngrp : g0 + kcap;
    // lane e < 21 owns packed entry e = (r, s) of every group's 6x6
    LANES(e, 21) {
      int r = 0; while ((r + 1) * (r + 2) / 2 <= e) r++;
      const int s = e - r * (r + 1) / 2;
      for (int g = g0; g < g1; g++) {
        float* K = Kc + 21 * (g - g0);
        const float* gr = SF(group) + g * GRP_WORDS;
        float acc = 0;
        for (int i = grp_start(gr), i1 = i + grp_count(gr); i < i1; i++) {
          const float* cr = SF(con) + i * CON_WORDS;
          const int dim = con_dim(cr);
          const uint32_t act = con_act(cr);
          float D = cr[C_D];
          float wnr = cr[C_W + r], wns = cr[C_W + s];
          if (dim == 1) { if (act & 1u) acc += D * wnr * wns; continue; }
          float Wnn = 0;
          for (int k = 1; k < dim; k++) {
            float ap = (act >> (2 * k - 2)) & 1u ? 1.f : 0.f, am = (act >> (2 * k - 1)) & 1u ? 1.f : 0.f;
            if (ap + am == 0.f) continue;
            float mu = con_mu(cr, k);
            float wkr, wks;
            if (k < 3) { wkr = cr[C_W + 6 * k + r]; wks = cr[C_W + 6 * k + s]; }
#ifdef B200_KITCHEN
            else { wkr = r < 3 ? cr[C_W + 6 * (k - 3) + 3 + r] : 0.f; wks = s < 3 ? cr[C_W + 6 * (k - 3) + 3 + s] : 0.f; }
#else
            else { wkr = r < 3 ? cr[C_W + 3 + r] : 0.f; wks = s < 3 ? cr[C_W + 3 + s] : 0.f; }
#endif
            Wnn += ap + am;
            float Wnk = mu * (ap - am), Wkk = mu * mu * (ap + am);
            acc += D * (Wnk * (wnr * wks + wkr * wns) + Wkk * wkr * wks);
          }
          acc += D * Wnn * wnr * wns;
        }
        for (int i = 0; i < nweld; i++) {
          const float* wr = SF(weld) + i * WELD_WORDS;
          if (((const int*)wr)[W_GRP] != g) continue;
          for (int k = 0; k < 6; k++) acc += wr[W_D + k] * wr[W_W + 6 * k + r] * wr[W_W + 6 * k + s];
        }
        K[e] = acc;
      }
    }
    SYNC();
    // lane i owns row i of H: for every group whose chains contain dof i, y = K cdof_i (registers), then
    // H_ij += sigma_i sigma_j cdof_j . y for the group's dofs j <= i
    LANES(i, nv) {
      const float* cd = SF(cdof) + 6 * i;
      const int row = i * (i + 1) / 2;
      for (int g = g0; g < g1; g++) {
        const float* gr = SF(group) + g * GRP_WORDS;
        const dmask_t S = grp_mask(gr), mb = grp_sign(gr);
        if (!DBIT(S, i)) continue;
        const float* K = Kc + 21 * (g - g0);
        float y[6];
#pragma unroll
        for (int r = 0; r < 6; r++) {
          float a = 0;
#pragma unroll
          for (int s2 = 0; s2 < 6; s2++) a += K[pidx(r, s2)] * cd[s2];
          y[r] = a;
        }
        float si = DBIT(mb, i) ? 1.f : -1.f;
        dmask_t m2 = S & (((dmask_t)2 << i) - (dmask_t)1);  // j <= i
        while (m2) {
          int j = ffs_pop(m2);
          float sj = DBIT(mb, j) ? 1.f : -1.f;
          H[row + j] += si * sj * dot6(SF(cdof) + 6 * j, y);
        }
      }
    }
    SYNC();
  }
  SYNC();
  // dof friction rows in their quadratic zone (|x| < R * frictionloss)
  if (HF) {
    LANES(d, h->nfric) {
      float D = MF(dof_fricD)[d], x = SF(fric)[d];
      if (D > 0 && fabsf(x) * D < MF(dof_frictionloss)[d]) H[d * (d + 1) / 2 + d] += D;
    }
    SYNC();
  }
  if (HF) {
    // dof rows (active ones): lane = dof; a row over (d1, d2) adds to the two diagonals and to the entry (max, min),
    // which the lane of the larger dof owns
    LANES(j, nv) {
      float diag = 0.f;
      for (int i = 0; i < ndr; i++) {
        const float* dr = SF(dofrow) + i * DR_WORDS;
        const int* di = (const int*)dr;
#ifdef B200_KITCHEN
        if (!(dr[DR_JAR] < 0 || dr[DR_D] < 0)) continue;
        const float Dr = fabsf(dr[DR_D]);
#else
        if (!(dr[DR_JAR] < 0)) continue;
        const float& Dr = dr[DR_D];   // (a reference: loaded where used, as before the kitchen branch existed)
#endif
        int d1 = di[DR_DOF], d2 = di[DR_DOF2];
        if (d1 == j) diag += Dr * dr[DR_COEF] * dr[DR_COEF];
        if (d2 == j) diag += Dr * dr[DR_COEF2] * dr[DR_COEF2];
        if (d2 >= 0 && (d1 > d2 ? d1 : d2) == j) H[j * (j + 1) / 2 + (d1 > d2 ? d2 : d1)] += Dr * dr[DR_COEF] * dr[DR_COEF2];
      }
      H[j * (j + 1) / 2 + j] += diag;
    }
  } else if (c.lane == 0) {
    // few limit rows (arm / legged models): one lane walks them
    for (int i = 0; i < ndr; i++) {
      const float* dr = SF(dofrow) + i * DR_WORDS;
      const int* di = (const int*)dr;
      if (!(dr[DR_JAR] < 0)) continue;
      int d1 = di[DR_DOF], d2 = di[DR_DOF2];
      H[pidx(d1, d1)] += dr[DR_D] * dr[DR_COEF] * dr[DR_COEF];
      if (d2 >= 0) { H[pidx(d2, d2)] += dr[DR_D] * dr[DR_COEF2] * dr[DR_COEF2]; H[pidx(d1, d2)] += dr[DR_D] * dr[DR_COEF] * dr[DR_COEF2]; }
    }
  }
  SYNC();
}

// in-place packed Cholesky H = L L^T, one lane per row
STAGE void cholesky(const Ctx c, float* H) {
  ASSUME_SHARED(c);
  int n = c.h->nv;
  for (int k = 0; k < n; k++) {
    float hkk = H[k * (k + 1) / 2 + k];
    float d = sqrtf(fmaxf(hkk, 1e-30f)), inv = 1.0f / d;
    SYNC();
    LANES(i, n) { if (i == k) H[i * (i + 1) / 2 + k] = d; else if (i > k) H[i * (i + 1) / 2 + k] *= inv; }
    SYNC();
    LANES(i, n) {
      if (i <= k) continue;
      int row = i * (i + 1) / 2;
      float lik = H[row + k];
      for (int j = k + 1; j <= i; j++) H[row + j] -= lik * H[j * (j + 1) / 2 + k];
    }
    SYNC();
  }
}
// x <- (L L^T)^-1 x
STAGE void chol_solve(const Ctx c, const float* L, float* x) {
  ASSUME_SHARED(c);
  int n = c.h->nv;
  for (int k = 0; k < n; k++) {
    if (c.lane == (k % WARP_W)) x[k] = x[k] / L[k * (k + 1) / 2 + k];
    SYNC();
    float xk = x[k];
    LANES(i, n) if (i > k) x[i] -= L[i * (i + 1) / 2 + k] * xk;
    SYNC();
  }
  for (int k = n - 1; k >= 0; k--) {
    if (c.lane == (k % WARP_W)) x[k] = x[k] / L[k * (k + 1) / 2 + k];
    SYNC();
    float xk = x[k];
    LANES(i, k) x[i] -= L[k * (k + 1) / 2 + i] * xk;
    SYNC();
  }
}

// x <- (A + hh*diag(dadd))^-1 x for the packed SPD matrix A.  CUDA: register-resident right-looking Cholesky, lane i owns
// the full symmetric row i (lower part ends up as L, the frozen upper part gives L^T), columns travel by warp shuffle;
// NVP is nv padded to a compile-time size (identity padding).  Host emulation: the shared-memory routines above.
#ifdef B200_WARP_CODE
// Models with more than 32 dofs (wide build, NVP = 32 + KB): lane i owns row i of the leading 32 x 32 block as before and,
// in addition, its entries of the KB border rows (c[r] = H[32 + r][i]); the KB x KB corner block is replicated in every
// lane.  The border rows ride along the right-looking elimination (one extra shuffle per border row and step), the corner
// becomes the Schur complement and is factorised redundantly in registers; the two triangular solves pick the border up
// through KB warp reductions (forward) and a lane-local correction (backward).
template <int NVP>
static __device__ __noinline__ void spd_solve(const Ctx c, const float* A, const float* dadd, float hh, float* x, float* scratchH) {
  ASSUME_SHARED(c);
  __builtin_assume(__isShared(A)); __builtin_assume(__isShared(x)); if (dadd) __builtin_assume(__isShared(dadd));
  __builtin_assume(__isShared(scratchH));
  constexpr int NA = NVP > 32 ? 32 : NVP, KB = NVP > 32 ? NVP - 32 : 0, KS = KB > 0 ? KB : 1;
  const int nv = c.h->nv, i = c.lane;
  const unsigned FULL = 0xffffffffu;
  float h[NA];
  const int rowi = i * (i + 1) / 2;
  const bool live = i < nv;
  // branch-free loads (clamped index + select) so the warp stays converged for the shuffles below
#pragma unroll
  for (int j = 0; j < NA; j++) {
    const bool in = live && j < nv;
    int idx = (j <= i) ? rowi + j : j * (j + 1) / 2 + i;
    idx = in ? idx : 0;
    float v = A[idx];
    v = in ? v : ((i == j) ? 1.f : 0.f);
    h[j] = v;
  }
  float cb[KS], S[KS][KS], bb[KS];   // border entries of this lane, replicated corner block, border right-hand side
#pragma unroll
  for (int r = 0; r < KB; r++) {
    const int row = 32 + r, ro = row * (row + 1) / 2;
    const bool in = row < nv;
    cb[r] = (in && live) ? A[ro + i] : 0.f;
#pragma unroll
    for (int q = 0; q < KB; q++) {
      const int col = 32 + q;
      const bool in2 = in && col < nv;
      float v = A[in2 ? (q <= r ? ro + col : col * (col + 1) / 2 + row) : 0];
      S[r][q] = in2 ? v : (r == q ? 1.f : 0.f);
    }
    bb[r] = in ? x[row] : 0.f;
  }
  if (dadd != nullptr) {
    float dd = hh * dadd[live ? i : 0];
#pragma unroll
    for (int j = 0; j < NA; j++) h[j] += (live && i == j) ? dd : 0.f;
#pragma unroll
    for (int r = 0; r < KB; r++) S[r][r] += (32 + r < nv) ? hh * dadd[32 + r < nv ? 32 + r : 0] : 0.f;
  }
  float b = 0.f;
  if (live) b = x[i];  // predicated load: idle lanes never touch x
  float dinv = 1.f;
  // column k of L travels through shared memory (one store per lane, 128-bit broadcast loads) instead of one shuffle per
  // (row, column) pair; two alternating buffers in the dead `scratchH` region (A has been loaded into registers above;
  // when A == scratchH the warp-level barrier below orders the overwrite)
  constexpr int NA4 = (NA + 3) & ~3;
  float* colbuf = scratchH;
  __syncwarp();
#pragma unroll
  for (int k = 0; k < NA; k++) {
    float hkk = __shfl_sync(FULL, h[k], k);
    float inv = rsqrtf(fmaxf(hkk, 1e-30f));
    float lik = (i > k) ? h[k] * inv : 0.f;
    dinv = (i == k) ? inv : dinv;
    h[k] = (i > k) ? lik : h[k];
    if (k + 1 < NA) {
      float* col = colbuf + (k & 1) * NA4;
      if (i < NA4) col[i] = lik;
      __syncwarp();
      const float4* c4 = (const float4*)col;
#pragma unroll
      for (int q = (k + 1) / 4; q < NA4 / 4; q++) {
        const float4 v = c4[q];
        if (4 * q + 0 > k && 4 * q + 0 < NA) h[4 * q + 0] = fmaf(-lik, v.x, h[4 * q + 0]);
        if (4 * q + 1 > k && 4 * q + 1 < NA) h[4 * q + 1] = fmaf(-lik, v.y, h[4 * q + 1]);
        if (4 * q + 2 > k && 4 * q + 2 < NA) h[4 * q + 2] = fmaf(-lik, v.z, h[4 * q + 2]);
        if (4 * q + 3 > k && 4 * q + 3 < NA) h[4 * q + 3] = fmaf(-lik, v.w, h[4 * q + 3]);
      }
    }
    float lr[KS];
#pragma unroll
    for (int r = 0; r < KB; r++) {
      lr[r] = __shfl_sync(FULL, cb[r] * inv, k);            // L[32 + r][k]
      cb[r] = (i == k) ? lr[r] : fmaf(-lr[r], lik, cb[r]);   // lanes <= k: lik = 0, their (final) entries stay
    }
#pragma unroll
    for (int r = 0; r < KB; r++)
#pragma unroll
      for (int q = 0; q < KB; q++) S[r][q] = fmaf(-lr[r], lr[q], S[r][q]);
  }
  // corner block: S = L_S L_S^T in place (lower triangle), replicated
  float sinv[KS];
#pragma unroll
  for (int k = 0; k < KB; k++) {
    float inv = rsqrtf(fmaxf(S[k][k], 1e-30f));
    sinv[k] = inv;
#pragma unroll
    for (int r = k + 1; r < KB; r++) S[r][k] *= inv;
#pragma unroll
    for (int r = k + 1; r < KB; r++)
#pragma unroll
      for (int q = k + 1; q <= r; q++) S[r][q] = fmaf(-S[r][k], S[q][k], S[r][q]);
  }
#pragma unroll
  for (int k = 0; k < NA; k++) {  // L y = b
    float yk = __shfl_sync(FULL, b * dinv, k);
    float bn = fmaf(-h[k], yk, b);
    b = (i > k) ? bn : ((i == k) ? yk : b);
  }
  // border: y_B = L_S^-1 (b_B - W y_A), z_B = L_S^-T y_B
#pragma unroll
  for (int r = 0; r < KB; r++) bb[r] -= wsum(cb[r] * b);
#pragma unroll
  for (int k = 0; k < KB; k++) {
    bb[k] *= sinv[k];
#pragma unroll
    for (int r = k + 1; r < KB; r++) bb[r] = fmaf(-S[r][k], bb[k], bb[r]);
  }
#pragma unroll
  for (int k = KB - 1; k >= 0; k--) {
    bb[k] *= sinv[k];
#pragma unroll
    for (int r = 0; r < k; r++) bb[r] = fmaf(-S[k][r], bb[k], bb[r]);
  }
#pragma unroll
  for (int r = 0; r < KB; r++) b = fmaf(-cb[r], bb[r], b);   // y_A - W^T z_B
  float sacc = 0.f, z = 0.f;
#pragma unroll
  for (int k = NA - 1; k >= 0; k--) {  // L^T z = y, with l_kj = h_j[k] * dinv_j for k > j
    float zk = __shfl_sync(FULL, (b - dinv * sacc) * dinv, k);
    float sn = fmaf(h[k], zk, sacc);
    sacc = (i < k) ? sn : sacc;
    z = (i == k) ? zk : z;
  }
  __syncwarp();
  if (i < nv && i < NA) x[i] = z;
#pragma unroll
  for (int r = 0; r < KB; r++) if (i == r && 32 + r < nv) x[32 + r] = bb[r];
  __syncwarp();
}
#else
template <int NVP>
static inline void spd_solve(const Ctx& c, const float* A, const float* dadd, float hh, float* x, float* scratchH) {
  int nv = c.h->nv, nM = nv * (nv + 1) / 2;
  for (int i = 0; i < nM; i++) scratchH[i] = A[i];
  if (dadd) for (int i = 0; i < nv; i++) scratchH[i * (i + 1) / 2 + i] += hh * dadd[i];
  cholesky(c, scratchH);
  chol_solve(c, scratchH, x);
}
#endif

// the step alpha and the improvement cost(0) - cost(alpha), returned by value (the caller's improvement lives on its stack)
struct LsStep { float alpha, improve; };
#ifndef B200_KITCHEN
// Line search over the constraint edges, held in registers.  Every constraint row expands into one or more edges (x0, v, D):
// the pyramid edges of a contact are x = u_n +- mu u_k, then come the six rows of each weld and the dof rows.  D < 0 marks a
// two-sided (equality) row, D == 0 an empty slot (a contact's unused pyramid edges, and the slots past the last edge).  Lane
// `lane` owns edge slots lane + WARP_W j, j < LSE * 32 / WARP_W -- the lane assignment of a strided loop over the edges -- and
// builds them once per Newton move; every cost evaluation then reads them from registers.  LSE (edge slots per lane of a
// 32-lane warp) is fixed per kernel build (dmodel.h DM_LS_E); b200sim_create refuses models with more edges than that.
struct LsVal { float cost, d1, d2; };

// x_n + mu (+-x_k), rounded once on the device (nvcc has always fused this product into the addition, FFMA) and twice on the host
// (ISO C++ does not contract): the register build keeps the edge values of both bit for bit, whatever the surrounding code
HD float pyramid_edge(float xn, float mu, float xk) {
#ifdef __CUDACC__
  return fmaf(mu, xk, xn);
#else
  return xn + mu * xk;
#endif
}

// cost(alpha) - gauss constant, first and second derivative.  Each lane adds its slots in ascending order, as the strided loop
// over a shared edge list did, so the sums do not depend on where the edges are kept.
template <bool HF, int NS>
HD LsVal ls_eval(const Ctx c, const float (&ex)[NS], const float (&ev)[NS], const float (&eD)[NS], int nedge, float alpha, float g1,
                 float g2) {
  float cost = 0, d1 = 0, d2 = 0;
#pragma unroll
  for (int j = 0; j < NS; j++) {
    if (WARP_W * j >= nedge) break;   // warp-uniform: no lane has an edge in slot j or later
    float x0 = ex[j], v = ev[j], D = eD[j];
    float x = fmaf(alpha, v, x0), Da = fabsf(D);
    if (D < 0 || (x < 0 && D > 0)) { float dx = Da * x; cost = fmaf(0.5f * dx, x, cost); d1 = fmaf(dx, v, d1); d2 = fmaf(Da * v, v, d2); }
  }
  if (HF) LANES(d, c.h->nfric) {
    float D = MF(dof_fricD)[d];
    if (D > 0) {
      float fl = MF(dof_frictionloss)[d], v = SF(fric)[c.h->nfric + d], x = SF(fric)[d] + alpha * v, Rf = fl / D;
      if (x <= -Rf) { cost += fl * (-0.5f * Rf - x); d1 -= fl * v; }
      else if (x >= Rf) { cost += fl * (-0.5f * Rf + x); d1 += fl * v; }
      else { cost += 0.5f * D * x * x; d1 += D * x * v; d2 += D * v * v; }
    }
  }
  LsVal r;
  r.cost = wsum(cost) + alpha * g1 + alpha * alpha * g2;
  r.d1 = wsum(d1) + g1 + 2 * alpha * g2;
  r.d2 = wsum(d2) + 2 * g2;
  return r;
}

// inlined into newton_move: one call boundary less per move (the 32-warp kernels run 1 % faster than with a call of its own)
template <bool HF, int LSE>
HD LsStep linesearch(const Ctx c, float g1, float g2, float gtol, int maxit) {
  ASSUME_SHARED(c);
  constexpr int NS = LSE * 32 / WARP_W;   // slots per lane
  const DMHead* h = c.h;
  const int* cnt = SI(counters);
  const int epc = h->edges_per_con, ncon = cnt[CNT_NCON], nweld6 = cnt[CNT_NWELD] * 6, ndr = cnt[CNT_NDR];
  const int nce = epc * ncon, nwe = nce + nweld6, nedge = nwe + ndr;
  float ex[NS], ev[NS], eD[NS];
  // contact and pyramid edge of slot j, q = e / epc and r = e % epc, advanced by WARP_W per slot (two divisions in all)
  const int qs = WARP_W / epc, rs = WARP_W % epc;
  int q = c.lane / epc, r = c.lane % epc;
#pragma unroll
  for (int j = 0; j < NS; j++) {
    const int e = c.lane + WARP_W * j;
    float x0 = 0.f, v = 0.f, D = 0.f;
    if (j > 0) { q += qs; r += rs; if (r >= epc) { r -= epc; q++; } }
    if (WARP_W * j < nedge) {   // warp-uniform: slots past the last edge stay empty
      if (e < nce) {   // contact q, pyramid edge r = base row 1 + r / 2, + for even r
        const float* cr = SF(con) + q * CON_WORDS;
        const int k = r, dim = con_dim(cr);
        const float un = cr[C_U], vn = cr[C_JV];
        if (dim == 1) {
          if (k == 0) { x0 = un; v = vn; D = cr[C_D]; }
        } else if (k < 2 * (dim - 1)) {
          const int b = 1 + (k >> 1);
          const float mu = con_mu(cr, b), su = (k & 1) ? -cr[C_U + b] : cr[C_U + b], sv = (k & 1) ? -cr[C_JV + b] : cr[C_JV + b];
          x0 = pyramid_edge(un, mu, su); v = pyramid_edge(vn, mu, sv);
          D = cr[C_D];
        }
      } else if (e < nwe) {
        const int i = e - nce;
        const float* wr = SF(weld) + (i / 6) * WELD_WORDS;
        x0 = wr[W_JAR + i % 6]; v = wr[W_JV + i % 6]; D = -wr[W_D + i % 6];
      } else if (e < nedge) {
        const float* dr = SF(dofrow) + (e - nwe) * DR_WORDS;
        x0 = dr[DR_JAR]; v = dr[DR_JV]; D = dr[DR_D];
      }
    }
    ex[j] = x0; ev[j] = v; eD[j] = D;
  }
  const LsVal p0 = ls_eval<HF>(c, ex, ev, eD, nedge, 0.f, g1, g2);
  if (p0.d1 >= 0 || p0.d2 <= 0) return LsStep{0.f, 0.f};
  gtol = fmaxf(gtol, 1e-5f * fabsf(p0.d1));  // single-precision floor on the derivative test
  float lo = 0, hi = -1, alpha = -p0.d1 / p0.d2, best = 0, bestcost = p0.cost;
  for (int it = 0; it < maxit; it++) {
    const LsVal p = ls_eval<HF>(c, ex, ev, eD, nedge, alpha, g1, g2);
    if (p.cost <= bestcost) { bestcost = p.cost; best = alpha; }
    if (fabsf(p.d1) < gtol) break;
    if (p.d1 < 0) lo = alpha; else hi = alpha;
    float next = alpha - p.d1 / p.d2;
    if (hi > 0 && (next <= lo || next >= hi)) next = 0.5f * (lo + hi);
    if (next == alpha) break;
    alpha = next;
  }
  return LsStep{best, p0.cost - bestcost};
}

#else
// The kitchen builds (B200_KITCHEN) keep the line search over a flat edge list in shared memory: with up to 10 edges per contact
// the register version above ran their step kernel 1.6 % slower (DESIGN.md section 3).  ls_edges() expands every constraint row
// into (x0, v, D) triples once per Newton move into the scratch that H and d6 occupied before the direction solve; ls_eval()
// then walks the triples with all 32 lanes.  LSE is unused here.
template <bool HF>
STAGE int ls_edges(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  const int* cnt = SI(counters);
  const int epc = h->edges_per_con, ncon = cnt[CNT_NCON], nweld6 = cnt[CNT_NWELD] * 6, ndr = cnt[CNT_NDR];
  float* E = SF(H);
  LANES(i, ncon) {
    const float* cr = SF(con) + i * CON_WORDS;
    float* e = E + 3 * epc * i;
    int dim = con_dim(cr);
    float D = cr[C_D], un = cr[C_U], vn = cr[C_JV];
    int ne = 0;
    if (dim == 1) { e[0] = un; e[1] = vn; e[2] = D; ne = 1; }
    else for (int k = 1; k < dim; k++) {
      float mu = con_mu(cr, k), uk = mu * cr[C_U + k], vk = mu * cr[C_JV + k];
      e[3 * ne] = un + uk; e[3 * ne + 1] = vn + vk; e[3 * ne + 2] = D; ne++;
      e[3 * ne] = un - uk; e[3 * ne + 1] = vn - vk; e[3 * ne + 2] = D; ne++;
    }
    for (; ne < epc; ne++) e[3 * ne + 2] = 0.f;
  }
  float* W = E + 3 * epc * ncon;
  LANES(i, nweld6) {
    const float* wr = SF(weld) + (i / 6) * WELD_WORDS;
    int k = i % 6;
    W[3 * i] = wr[W_JAR + k]; W[3 * i + 1] = wr[W_JV + k]; W[3 * i + 2] = -wr[W_D + k];
  }
  float* R = W + 3 * nweld6;
  LANES(i, ndr) {
    const float* dr = SF(dofrow) + i * DR_WORDS;
    R[3 * i] = dr[DR_JAR]; R[3 * i + 1] = dr[DR_JV]; R[3 * i + 2] = dr[DR_D];
  }
  SYNC();
  return epc * ncon + nweld6 + ndr;
}

// cost(alpha) - gauss constant, first and second derivative
template <bool HF>
STAGE void ls_eval(const Ctx c, int nedge, float alpha, float g1, float g2, float* out) {
  ASSUME_SHARED(c);
  float cost = 0, d1 = 0, d2 = 0;
  const float* E = SF(H);
  LANES(i, nedge) {
    float x0 = E[3 * i], v = E[3 * i + 1], D = E[3 * i + 2];
    float x = fmaf(alpha, v, x0), Da = fabsf(D);
    if (D < 0 || (x < 0 && D > 0)) { float dx = Da * x; cost = fmaf(0.5f * dx, x, cost); d1 = fmaf(dx, v, d1); d2 = fmaf(Da * v, v, d2); }
  }
  if (HF) LANES(d, c.h->nfric) {
    float D = MF(dof_fricD)[d];
    if (D > 0) {
      float fl = MF(dof_frictionloss)[d], v = SF(fric)[c.h->nfric + d], x = SF(fric)[d] + alpha * v, Rf = fl / D;
      if (x <= -Rf) { cost += fl * (-0.5f * Rf - x); d1 -= fl * v; }
      else if (x >= Rf) { cost += fl * (-0.5f * Rf + x); d1 += fl * v; }
      else { cost += 0.5f * D * x * x; d1 += D * x * v; d2 += D * v * v; }
    }
  }
  out[0] = wsum(cost) + alpha * g1 + alpha * alpha * g2;
  out[1] = wsum(d1) + g1 + 2 * alpha * g2;
  out[2] = wsum(d2) + 2 * g2;
}

template <bool HF, int LSE>
STAGE LsStep linesearch(const Ctx c, float g1, float g2, float gtol, int maxit) {
  ASSUME_SHARED(c);
  float p0[3], p[3];
  const int nedge = ls_edges<HF>(c);
  ls_eval<HF>(c, nedge, 0.f, g1, g2, p0);
  if (p0[1] >= 0 || p0[2] <= 0) return LsStep{0.f, 0.f};
  gtol = fmaxf(gtol, 1e-5f * fabsf(p0[1]));  // single-precision floor on the derivative test
  float lo = 0, hi = -1, alpha = -p0[1] / p0[2], best = 0, bestcost = p0[0];
  for (int it = 0; it < maxit; it++) {
    ls_eval<HF>(c, nedge, alpha, g1, g2, p);
    if (p[0] <= bestcost) { bestcost = p[0]; best = alpha; }
    if (fabsf(p[1]) < gtol) break;
    if (p[1] < 0) lo = alpha; else hi = alpha;
    float next = alpha - p[1] / p[2];
    if (hi > 0 && (next <= lo || next >= hi)) next = 0.5f * (lo + hi);
    if (next == alpha) break;
    alpha = next;
  }
  return LsStep{best, p0[0] - bestcost};
}

#endif

// Newton solver, split so that the iteration loop can be driven block-uniformly (see forward()).  The convergence check ends
// the stage that brings the solver to its point (newton_begin, newton_move), right after the contact update that parked the
// base-row forces and the edge activity: no sweep over the contacts, stage call or block barrier of its own.

// gradient and convergence tests at the current point after `iter` moves, the last of which improved the cost by
// `improvement`; returns 1 when the solver is finished
template <bool HF>
HD int newton_check(const Ctx c, int iter, float improvement) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  int nv = h->nv;
  float *Ma = SF(Ma), *grad = SF(grad), *fs = SF(fsmooth), *fcon = SF(fcon);
  float scale = 1.0f / (h->meaninertia * (float)(nv > 1 ? nv : 1));
  float tol = fmaxf(h->tolerance, 1e-6f);  // single-precision floor for the convergence tests
  TIC();
  pass_F<HF>(c, fcon);
  TOC(TM_CK_PASSF);
  float g2sum = 0, f2sum = 0;
  LANES(i, nv) {
    float g = Ma[i] - fs[i] - fcon[i], f = fabsf(Ma[i]) + fabsf(fs[i]) + fabsf(fcon[i]);
    grad[i] = g; g2sum += g * g; f2sum += f * f;
  }
  SYNC();
  float gnorm = sqrtf(wsum(g2sum)), fnorm = sqrtf(wsum(f2sum));
  // single-precision floor: the gradient cannot be resolved below ~eps32 * (|M a| + |f_smooth| + |f_constraint|)
  if (gnorm < 2e-6f * fnorm) return 1;
  if (iter > 0 && (scale * improvement < tol || scale * gnorm < tol)) return 1;
  if (iter >= h->iterations || iter >= 12) return 1;
  return 0;
}

// opening of the solve and the check at iteration 0; returns 1 when the warm start is already converged
template <bool HF>
STAGE int newton_begin(const Ctx c) {
  ASSUME_SHARED(c);
  // qacc holds the warm start (previous sub-step's solution); rows become J a - aref = J a + B (J qvel) + K imp r
  mulM(c, SF(qacc), SF(Ma));
  rows_begin<HF>(c, SF(qvel), SF(qacc));
  CHECK_TIC();
  const int done = newton_check<HF>(c, 0, 0.f);
  CHECK_TOC(TM_NBEGIN);
  return done;
}

// Newton direction; returns 0 if the direction vanished
template <int NVP>
STAGE void newton_direction(const Ctx c) {
  ASSUME_SHARED(c);
  int nv = c.h->nv;
  LANES(i, nv) SF(search)[i] = -SF(grad)[i];
  SYNC();
  spd_solve<NVP>(c, SF(H), nullptr, 0.f, SF(search), SF(H));
}

// exact line search and move number iter, then the check at the new point; returns 0 to go on, 1 when the solver has converged,
// 2 when it must stop (no progress possible: the point is the one already checked)
template <bool HF, int LSE>
STAGE int newton_move(const Ctx c, int iter) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  int nv = h->nv;
  int* cnt = SI(counters);
  float *a = SF(qacc), *Ma = SF(Ma), *Mv = SF(Mv), *search = SF(search), *fs = SF(fsmooth);
  float scale = 1.0f / (h->meaninertia * (float)(nv > 1 ? nv : 1));
  TIC();
  mulM(c, search, Mv);
  TOC(TM_MV_MULM);
  rows_from_vec<HF>(c, search);
  TOC(TM_MV_ROWS);
  float q1 = 0, q2 = 0, sn = 0;
  LANES(i, nv) { q1 += search[i] * (Ma[i] - fs[i]); q2 += 0.5f * search[i] * Mv[i]; sn += search[i] * search[i]; }
  q1 = wsum(q1); q2 = wsum(q2); sn = sqrtf(wsum(sn));
  if (sn < 1e-20f) return 2;
  float gtol = h->tolerance * h->ls_tolerance * sn / scale;
  TOC(TM_MV_ROWS);
  const LsStep ls = linesearch<HF, LSE>(c, q1, q2, gtol, h->ls_iterations < 20 ? h->ls_iterations : 20);
  const float alpha = ls.alpha;
  TOC(TM_MV_LS);
  if (alpha == 0.f) return 2;
  LANES(i, nv) { a[i] += alpha * search[i]; Ma[i] += alpha * Mv[i]; }
  LANES(i, cnt[CNT_NCON]) {
    float* cr = SF(con) + i * CON_WORDS;
    float U[C_NB];
#pragma unroll
    for (int k = 0; k < C_NB; k++) { U[k] = cr[C_U + k] + alpha * cr[C_JV + k]; cr[C_U + k] = U[k]; }
    contact_park_forces(cr, U);
  }
  LANES(i, cnt[CNT_NWELD] * 6) { float* wr = SF(weld) + (i / 6) * WELD_WORDS; wr[W_JAR + i % 6] += alpha * wr[W_JV + i % 6]; }
  LANES(i, cnt[CNT_NDR]) { float* dr = SF(dofrow) + i * DR_WORDS; dr[DR_JAR] += alpha * dr[DR_JV]; }
  if (HF) LANES(d, h->nfric) SF(fric)[d] += alpha * SF(fric)[h->nfric + d];
  SYNC();
  if (c.lane == 0) cnt[CNT_ITERS] += 1;
  TOC(TM_MV_UPD);
  CHECK_TIC();
  const int done = newton_check<HF>(c, iter + 1, ls.improve);
  CHECK_TOC(TM_NMOVE);
  return done;
}

// the solve of the implicit-damping Euler step: SF(search) <- (M + h B)^-1 (f_smooth + f_constraint)
template <int NVP>
STAGE void euler_solve(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  float* x = SF(search);
  LANES(i, h->nv) x[i] = SF(fsmooth)[i] + SF(fcon)[i];
  SYNC();
  spd_solve<NVP>(c, SF(M), MF(dof_damping), h->timestep, x, SF(H));
}

// ---------------------------------------------------------------------------------------------------------------
// forward dynamics (mj_forward) and one Euler sub-step
// One forward pass.  `active` is warp-uniform; idle warps (no env, or masked out) only take part in the block-wide
// alignment barriers, so every warp of the block executes the same barrier sequence.  The Newton loop runs until every
// warp of the block has converged (converged warps idle through the remaining rounds).
template <int NVP, bool REBUILD = false>
HD void forward(const Ctx c, bool active) {
  constexpr bool HF = NVP >= 30;
  constexpr bool CX = NVP == 22 || NVP >= 30;   // NVP 22 = the 21-dof arm build plus the convex collider (FetchSlide)
  constexpr int kLsE = DM_LS_E(NVP);   // line-search edge slots per lane
  // HF: the hand build (NVP >= 30, 14 warps per block) is faster with a barrier after every stage (DESIGN.md 3, "Hand build").
  // REBUILD (the 28- and 32-warp kernels): no alignment after the collision stage and between the Newton direction and the move;
  // with the convergence check inside the move, FetchPickAndPlace at 32 warps runs 1.4 % faster without them (DESIGN.md 6)
  TIC();
  ALIGN(); TOC(TM_BARRIER);
  if (active) kinematics(stage_ctx<REBUILD>(c));
  TOC(TM_KIN); if (HF) ALIGN(); TOC(TM_BARRIER);
  if (active) { com_quantities(stage_ctx<REBUILD>(c)); mass_matrix(stage_ctx<REBUILD>(c)); }
  TOC(TM_COM_M); ALIGN(); TOC(TM_BARRIER);
  if (active) collision<HF, CX>(stage_ctx<REBUILD>(c));
  TOC(TM_COLL); if (!REBUILD) ALIGN(); TOC(TM_BARRIER);
  if (active) make_constraint<HF>(stage_ctx<REBUILD>(c));
  TOC(TM_CONSTR); if (HF) ALIGN(); TOC(TM_BARRIER);
  if (active) smooth_forces(stage_ctx<REBUILD>(c));
  TOC(TM_SMOOTH); if (HF) ALIGN(); TOC(TM_BARRIER);
  int done = 1;
  if (active) done = newton_begin<HF>(stage_ctx<REBUILD>(c));
  TOC(TM_NBEGIN);
  for (int iter = 0;; iter++) {
    bool more = ALIGN_OR(!done);
    TOC(TM_BARRIER);
    if (!more) break;
    if (!done) build_H<HF>(stage_ctx<REBUILD>(c));
    TOC(TM_BUILDH); if (HF) ALIGN(); TOC(TM_BARRIER);
    if (!done) newton_direction<NVP>(stage_ctx<REBUILD>(c));
    TOC(TM_NDIR); if (!REBUILD) ALIGN(); TOC(TM_BARRIER);
    if (!done) done = newton_move<HF, kLsE>(stage_ctx<REBUILD>(c), iter);
    TOC(TM_NMOVE);
  }
}

// qpos <- qpos (+) dt * vel  (free-joint quaternions on the manifold)
STAGE void integrate_pos(const Ctx c, float* qpos, const float* qvel, float hh) {
  ASSUME_SHARED(c);
  ASSUME_SHARED_PTR(qpos); ASSUME_SHARED_PTR(qvel);
  const DMHead* h = c.h;
  LANES(j, h->njnt) {
    int a = MI(jnt_qposadr)[j], d = MI(jnt_dofadr)[j];
    if (MI(jnt_type)[j] == B200_JNT_FREE) {
      for (int k = 0; k < 3; k++) qpos[a + k] += hh * qvel[d + k];
      float w[3] = {qvel[d + 3], qvel[d + 4], qvel[d + 5]};
      float n = sqrtf(dot3(w, w));
      float q[4] = {qpos[a + 3], qpos[a + 4], qpos[a + 5], qpos[a + 6]};
      if (n > 0) {
        float ang = 0.5f * n * hh, sn = sinf(ang), cs = cosf(ang), inv = 1.0f / n;
        float dq[4] = {cs, w[0] * inv * sn, w[1] * inv * sn, w[2] * inv * sn}, nq[4];
        qmul(nq, q, dq);
        q[0] = nq[0]; q[1] = nq[1]; q[2] = nq[2]; q[3] = nq[3];
      }
      qnormalize(q);
      qpos[a + 3] = q[0]; qpos[a + 4] = q[1]; qpos[a + 5] = q[2]; qpos[a + 6] = q[3];
    } else qpos[a] += hh * qvel[d];
  }
  SYNC();
}

template <int NVP>
STAGE void euler_step(const Ctx c) {
  ASSUME_SHARED(c);
  const DMHead* h = c.h;
  int nv = h->nv;
  float hh = h->timestep;
  float* x = SF(search);  // qacc itself is next sub-step's warm start
  if (h->any_damping) {
    euler_solve<NVP>(c);
  } else {
    LANES(i, nv) x[i] = SF(qacc)[i];
    SYNC();
  }
  LANES(i, nv) SF(qvel)[i] += hh * x[i];
  SYNC();
  integrate_pos(c, SF(qpos), SF(qvel), hh);
}

// one classical RK4 sub-step over (qpos, qvel), ctrl held constant, one forward pass per stage, no implicit damping
// (reference: `integrator="RK4"` of the Ant model, gymnasium_robotics/envs/mujoco/assets/ant.xml:3).  The first
// stage's forward pass has already been done by the caller.
template <int NVP, bool REBUILD = false>
HD void rk4_substep(const Ctx c, bool active) {
  const DMHead* h = c.h;
  const int nv = h->nv, nq = h->nq;
  const float hh = h->timestep;
  const float A[3] = {0.5f, 0.5f, 1.0f}, B[4] = {1.0f / 6, 1.0f / 3, 1.0f / 3, 1.0f / 6};
  if (active) {
    LANES(i, nq) SF(rk_q0)[i] = SF(qpos)[i];
    LANES(i, nv) { SF(rk_v0)[i] = SF(qvel)[i]; SF(rk_dx)[i] = B[0] * SF(qvel)[i]; SF(rk_df)[i] = B[0] * SF(qacc)[i]; }
    SYNC();
  }
  for (int st = 1; st < 4; st++) {
    if (active) {
      float a = A[st - 1] * hh;
      LANES(i, nq) SF(qpos)[i] = SF(rk_q0)[i];
      SYNC();
      integrate_pos(c, SF(qpos), SF(qvel), a);           // X_{st-1} is the current qvel
      LANES(i, nv) SF(qvel)[i] = SF(rk_v0)[i] + a * SF(qacc)[i];
      SYNC();
    }
    forward<NVP, REBUILD>(c, active);
    if (active) {
      LANES(i, nv) { SF(rk_dx)[i] += B[st] * SF(qvel)[i]; SF(rk_df)[i] += B[st] * SF(qacc)[i]; }
      SYNC();
    }
  }
  if (active) {
    LANES(i, nq) SF(qpos)[i] = SF(rk_q0)[i];
    LANES(i, nv) SF(qvel)[i] = SF(rk_v0)[i] + hh * SF(rk_df)[i];
    SYNC();
    integrate_pos(c, SF(qpos), SF(rk_dx), hh);
  }
}
