// Device model: the fp32 constant tables one thread block stages into shared memory, and the per-env
// scratch layout.  Built on the host from the fp64 blob (include/b200sim_model.h) by dm_build().
//
// Replaces the `mujoco.MjModel` object of the reference (gymnasium_robotics/envs/robot_env.py:293).
#pragma once
#include <stdint.h>
#include <string.h>
#include <math.h>
#include <vector>
#include <string>
#include <map>
#include <set>
#include <utility>

#include "../../include/b200sim_model.h"

#define DM_MAX_BODY 32   // one lane per body / 32-bit body masks
#define DM_MAX_NV 40     // dof masks: one word per entry up to 32 dofs, two words (wide kernel build, B200_WIDE) up to 40
#define DM_NDOFROW_MIN 8
#define DM_NCAND_MAX 96   // broad-phase candidate slots (one byte each: pair index < 256)
#define DM_NWELD_MAX 1
// box-box working set of one narrow-phase lane in shared memory (sim_core.cuh `BoxScratch`: the clipping polygons, 8 x 2 + 8 x 3
// words).  The slots overlay scratch that is dead while the narrow phase runs: region A = the body-force / dof-term buffers of the
// smooth-force stage (b6 .. d6), region B = the contact records, as long as the narrow phase has not written one.
#define DM_CSLOT_WORDS 40
// Line-search edge slots per lane of a 32-lane warp, per kernel build: sim_core.cuh `linesearch` keeps every constraint edge of
// the env in registers, edge e in slot e / 32 of lane e % 32.  The arm and legged builds (NVP <= 22) carry at most 20 contacts
// of 6 pyramid edges, one weld (6 rows) and 8 dof rows = 134 edges; the hand and Adroit builds (NVP 30, 36; 32 in the test
// emulation) up to 48 dof rows = 174.  dm_ls_edges() is a model's bound.  The kitchen builds keep a shared-memory edge list.
#ifdef B200_KITCHEN
#define DM_LS_E(NVP) 0
#else
#define DM_LS_E(NVP) ((NVP) >= 30 ? 6 : 5)
#endif

// (name, words-per-element, kind) ; kind selects the element count.  HOT arrays are staged into shared memory by every
// block; COLD arrays (per-pair contact parameters, read only when a contact is created) stay in global memory.
// Kitchen build with the two-level broad phase (-DB200_KITCHEN_GROUPS on top of -DB200_KITCHEN; the plain kitchen build keeps the
// flat scan, its bit-exact reference): the flat pair list (3 708 entries, 44 KB) leaves shared memory -- it is only read for the pairs of the
// bounding-volume groups that survive the first broad-phase level -- and the group table (one bounding sphere on one body
// against one anchor geom, a contiguous run of pairs) is staged instead.
#ifdef B200_KITCHEN_GROUPS
#define DM_PAIR_HOT(X)
#define DM_PAIR_COLD(X) X(pair_geom1, 1, npair) X(pair_geom2, 1, npair) X(pair_margin, 1, npair)
#define DM_BGRP_HOT(X) X(bg_body, 1, nbgrp) X(bg_anchor, 1, nbgrp) X(bg_start, 1, nbgrp) X(bg_count, 1, nbgrp) X(bg_center, 3, nbgrp) X(bg_radius, 1, nbgrp)
#ifndef DM_NSURV_MAX
#define DM_NSURV_MAX 96   // bounding-volume groups that may survive the first level per env per sub-step (tests override it)
#endif
#else
#define DM_PAIR_HOT(X) X(pair_geom1, 1, npair) X(pair_geom2, 1, npair) X(pair_margin, 1, npair)
#define DM_PAIR_COLD(X)
#define DM_BGRP_HOT(X)
#endif
// builds with the support-map narrow phase for mesh geoms (-DB200_HULL): per geom (first vertex, count) into the reduced-hull vertex
// table of the blob (mjcf.py hull_vertices); read only by the narrow phase of a pair with such a geom
#ifdef B200_HULL
#define DM_HULL_COLD(X) X(geom_hull, 2, ngeom) X(hull_vert, 3, nhullv)
#else
#define DM_HULL_COLD(X)
#endif
#define DM_ARRAYS_HOT(X) \
  X(body_parent, 1, nb) X(body_jntadr, 1, nb) X(body_jntnum, 1, nb) X(body_dofadr, 1, nb) X(body_dofnum, 1, nb) \
  X(body_mocapid, 1, nb) X(body_ancdof, MW, nb) X(body_sub, 1, nb) X(body_pos, 3, nb) X(body_quat, 4, nb) \
  X(body_ipos, 3, nb) X(body_iquat, 4, nb) X(body_mass, 1, nb) X(body_inertia, 3, nb) \
  X(jnt_type, 1, njnt) X(jnt_body, 1, njnt) X(jnt_qposadr, 1, njnt) X(jnt_dofadr, 1, njnt) X(jnt_limited, 1, njnt) \
  X(jnt_pos, 3, njnt) X(jnt_axis, 3, njnt) X(jnt_range, 2, njnt) X(jnt_margin, 1, njnt) X(jnt_stiffness, 1, njnt) \
  X(jnt_qpos0, 1, njnt) X(jnt_qspring, 1, njnt) \
  X(dof_body, 1, nv) X(dof_jnt, 1, nv) X(dof_anc, MW, nv) X(dof_pre, MW, nv) X(dof_armature, 1, nv) \
  X(dof_damping, 1, nv) X(dof_frictionloss, 1, nv) X(dof_invweight0, 1, nv) \
  X(geom_type, 1, ngeom) X(geom_body, 1, ngeom) X(geom_pos, 3, ngeom) X(geom_quat, 4, ngeom) X(geom_size, 3, ngeom) \
  X(geom_rbound, 1, ngeom) \
  DM_PAIR_HOT(X) DM_BGRP_HOT(X) \
  X(site_body, 1, nsite) X(site_pos, 3, nsite) X(site_quat, 4, nsite) \
  X(act_trnid, 1, nu) X(act_ctrllimited, 1, nu) X(act_forcelimited, 1, nu) X(act_gear, 1, nu) X(act_gain, 1, nu) \
  X(act_bias, 3, nu) X(act_ctrlrange, 2, nu) X(act_forcerange, 2, nu) \
  X(eq_type, 1, neq) X(eq_obj1, 1, neq) X(eq_obj2, 1, neq) X(eq_active, 1, neq) X(eq_data, 11, neq) X(eq_solref, 2, neq) \
  X(eq_solimp, 5, neq) X(eq_invweight, 2, neq) \
  X(mocap_body, 1, nmocap) X(grid_walls, 1, ngridw) \
  X(dof_fricD, 1, nfric) X(dof_fricB, 1, nfric) \
  X(ten_dof, 2, nten) X(ten_qadr, 2, nten) X(ten_coef, 2, nten) X(ten_range, 2, nten) X(ten_margin, 1, nten)
#define DM_ARRAYS_COLD(X) \
  X(jnt_solref, 2, njnt) X(jnt_solimp, 5, njnt) /* read only when a limit row is created */ \
  DM_PAIR_COLD(X) \
  X(pair_condim, 1, npair) X(pair_friction, 3, npair) X(pair_gap, 1, npair) X(pair_solref, 2, npair) \
  X(pair_solimp, 5, npair) X(pair_invweight, 2, npair) \
  X(ten_solref, 2, nten) X(ten_solimp, 5, nten) X(ten_invweight, 1, nten) \
  X(sensor_site, 1, nsensor) X(sensor_body, 1, nsensor) X(sensor_type, 1, nsensor) X(sensor_size, 3, nsensor) \
  X(geom_mjb, 1, ngeom) X(mjb_rt, 1, nmjb) /* MJCF (unfused) body of a geom / runtime body of an MJCF body: cfrc_ext rows */ \
  DM_HULL_COLD(X)
#define DM_ARRAYS(X) DM_ARRAYS_HOT(X) DM_ARRAYS_COLD(X)

// per-env scratch that lives for the whole sub-step (name, words expression)
#define DM_SCRATCH_PERSIST(X) \
  X(qpos, nq) X(qvel, nv) X(qacc, nv) X(ctrl, nu) X(mocap_pos, 3 * nmocap) X(mocap_quat, 4 * nmocap) \
  X(xpos, 3 * nb) X(xquat, 4 * nb) X(cdof, 6 * nv) X(M, nv * (nv + 1) / 2) X(fsmooth, nv) X(fcon, nv) \
  X(rk_q0, nrkq) X(rk_v0, nrkv) X(rk_dx, nrkv) X(rk_df, nrkv) \
  X(con, ncon_max * CON_WORDS) X(dofrow, ndr_max * DR_WORDS) X(weld, DM_NWELD_MAX * WELD_WORDS) \
  X(group, ngrp_max * grp_words) X(counters, 8) X(fric, 2 * nfric) X(conx, ncx * CX_WORDS) X(penv_pos, npenv)
// time-shared region `uni`: kinematics {kinA, kinB} -> dynamics {cinert, b6, d6, geom_xpos, cand} -> solver {H, d6, grad,
// search, Ma, Mv} -> observation {cvel}.  d6 keeps one offset in both phases that use it.
#ifdef B200_KITCHEN_GROUPS
#define DM_SCRATCH_UNION(X) X(kinA) X(kinB) X(cinert) X(b6) X(d6) X(geom_xpos) X(cand) X(surv) X(H) X(grad) X(search) X(Ma) X(Mv) X(cvel)
#else
#define DM_SCRATCH_UNION(X) X(kinA) X(kinB) X(cinert) X(b6) X(d6) X(geom_xpos) X(cand) X(H) X(grad) X(search) X(Ma) X(Mv) X(cvel)
#endif
#define DM_SCRATCH(X) DM_SCRATCH_PERSIST(X)

// contact record (words): up to 4 base rows (normal, two tangents, torsion).  W = spatial vectors of the three
// translational rows about `ref`; the torsional row is (W0[3:6], 0).  During row set-up JV[0] holds B of the reference
// acceleration and U holds K*imp*r (normal row) / 0; afterwards U = J a - aref and JV = J search.
#ifdef B200_KITCHEN
// bring-up build (DESIGN.md section 7, step ii): condim 6 = two rolling base rows next to the torsional one; the rotational rows
// need no extra vectors (row k >= 3 is (W[k - 3][3:6], 0)), only a third friction coefficient and six U / JV slots
enum { C_W = 0 /*18*/, C_MU = 18 /*slide, torsion, roll*/, C_D = 21, C_U = 22 /*6*/, C_JV = 28 /*6*/, C_DIMGRP = 34, CON_WORDS = 36 };
#define C_NB 6
#else
enum { C_W = 0 /*18*/, C_MU = 18 /*slide, torsion*/, C_D = 20, C_U = 21 /*4*/, C_JV = 25 /*4*/, C_DIMGRP = 29, CON_WORDS = 30 };
#define C_NB 4
#endif
// dof row (joint limit or fixed-tendon limit over <= 2 dofs): JAR holds K*imp*r and JV holds B during set-up.
// Dof frictionloss rows are always present, one per dof, with constant D and B: they live in the per-dof arrays
// `fric` (FR_JAR, FR_JV) instead of generic rows.
enum { FR_JAR = 0, FR_JV = 1 };
// contact extras kept only by models with touch sensors: world position and pair index
enum { CX_POS = 0, CX_PAIR = 3, CX_WORDS = 4 };
enum { DR_DOF = 0, DR_COEF = 1, DR_D = 2, DR_JAR = 3, DR_JV = 4, DR_DOF2 = 5, DR_COEF2 = 6, DR_WORDS = 7 };
// weld: 6 rows w[6]; D[6], JAR[6] (K*imp*r during set-up), JV[6], B (one value), group
enum { W_W = 0, W_D = 36, W_JAR = 42, W_JV = 48, W_B = 54, W_GRP = 55, WELD_WORDS = 56 };
// group = one geom pair in contact (its contacts are contiguous) or one weld: one word G_RANGE = first contact | contact count << 8
// | the two MJCF body ids << 16 (A | B << 8, A = body of the pair's first geom: per-body contact forces, Ant-v5 cfrc_ext), dof
// mask S = anc(A) xor anc(B) with sign mask (bit set: dof on the B side), a 6-vector used for dV (J*v) and F (J^T f).  The
// group's 6x6 block K of H is not stored: build_H assembles the blocks in dead solver scratch, as many groups at a time as fit.
#ifdef B200_WIDE
enum { G_RANGE = 0, G_MASK = 1, G_SIGN = 3, G_V = 5, GRP_WORDS = 11 };   // two-word masks
#else
enum { G_RANGE = 0, G_MASK = 1, G_SIGN = 2, G_V = 3, GRP_WORDS = 9 };
#endif
enum { ROWT_EQ = 0, ROWT_FRICTION = 1, ROWT_LIMIT = 2 };
enum { CNT_NCON = 0, CNT_NDR = 1, CNT_NGRP = 2, CNT_NCAND = 3, CNT_NWELD = 4, CNT_ITERS = 5, CNT_OVERFLOW = 6 };

struct DMHead {
  int nb, njnt, nq, nv, nu, ngeom, nsite, nmocap, neq, npair;
  int nwords;      // size of the model buffer (header included) in 4-byte words
  int hot_words;   // leading part staged into shared memory (header + HOT arrays)
  int scr_words;   // per-env scratch size in words
  int iterations, ls_iterations, integrator, any_damping, kin_iters, ncon_max, ngrp_max, ndr_max;
  int edges_per_con, any_convex_pair, mask_words, penv_body;   // mask_words: 1, or 2 when nv > 32 (wide kernel build); penv_body: runtime body whose body_pos is per-env state (-1 = none)   // pyramid edges of the widest contact (2 * (condim - 1)): line-search edge slots
  int nten, nfric, ncand_max, nsensor;   // nsensor: touch sensors (site volume + body)   // limited fixed tendons; nfric = nv when any dof has frictionloss, else 0
  int grid_len, grid_wid, ngridw, any_round_pair;   // maze wall grid (0 x 0 when the model has none)
  int nmjb;        // MJCF bodies before fusing (rows of per-body outputs such as cfrc_ext)
  int s_cslotA, ncslotA, s_cslotB, ncslotB;   // narrow-phase lane slots (DM_CSLOT_WORDS each): two scratch regions, ncslotA + ncslotB <= 32
  float grid_scale, grid_top, grid_xc, grid_yc;  // cell size, wall top height, map centre offsets
  float timestep, gravity[3], tolerance, impratio, meaninertia, ls_tolerance, ref[3];
#define X(name, w, kind) int o_##name;
  DM_ARRAYS(X)
#undef X
#define X(name, words) int s_##name;
  DM_SCRATCH_PERSIST(X)
#undef X
#define X(name) int s_##name;
  DM_SCRATCH_UNION(X)
#undef X
#ifdef B200_KITCHEN_GROUPS
  int nbgrp;   // bounding-volume groups of the two-level broad phase (after the fields the common host code reads)
#endif
};

// ---------------------------------------------------------------------------------------------------------------
// host-side builder
static inline uint32_t f2w(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
// most line-search edges an env of this model can have: every contact with the widest pyramid, the welds, the dof rows
static inline int dm_ls_edges(const DMHead& h) { return h.edges_per_con * h.ncon_max + 6 * DM_NWELD_MAX + h.ndr_max; }

static inline int dm_build(const b200_model_view& m, const double* eq_data_override, const float ref[3],
                           std::vector<uint32_t>& buf, std::string& err, int penv_body = -1, bool force_wide = false,
                           int ngrp_cap = 0 /* tests: smaller contact-group capacity to exercise the overflow path */) {
  DMHead h;
  memset(&h, 0, sizeof(h));
  h.nb = m.nbody; h.njnt = m.njnt; h.nq = m.nq; h.nv = m.nv; h.nu = m.nu; h.nsite = m.nsite;
  h.nmocap = m.nmocap; h.neq = m.neq;
  // pair list on the device: ordinary pairs, plus one grid pair (geom2 = -1) per geom that can touch maze walls
  std::vector<int> psrc;       // source pair index in the blob
  std::vector<int> pgrid;      // 1 = grid pair
  {
    std::vector<char> seen(m.ngeom, 0);
    for (int p = 0; p < m.npair; p++) {
      bool isgrid = m.n_pair_grid == m.npair && m.pair_grid[p];
      if (!isgrid) { psrc.push_back(p); pgrid.push_back(0); }
      else if (!seen[m.pair_geom1[p]]) { seen[m.pair_geom1[p]] = 1; psrc.push_back(p); pgrid.push_back(1); }
    }
  }
#ifdef B200_KITCHEN_GROUPS
  // Two-level broad phase: the pairs are regrouped by (body of geom1, body of geom2); inside such a bucket every geom of
  // the anchor side (the world body's geoms, else the side with fewer geoms) gets one group = its pairs, contiguous in
  // the device pair list, behind ONE bounding sphere fixed to the other body that encloses the bounding spheres of all
  // its partner geoms (+ the largest pair margin).  A group whose sphere misses the anchor geom cannot hold a candidate
  // pair, so the set of candidates is the flat scan's; only their order follows the regrouped list.
  struct BGroup { int body, anchor, start, count; double c[3], r; };
  std::vector<BGroup> bgs;
  {
    std::map<std::pair<int, int>, std::vector<int>> buckets;
    for (size_t p = 0; p < psrc.size(); p++) {
      if (pgrid[p]) { err = "maze-grid pairs are not part of the kitchen build"; return -1; }
      buckets[std::make_pair(m.geom_body[m.pair_geom1[psrc[p]]], m.geom_body[m.pair_geom2[psrc[p]]])].push_back(psrc[p]);
    }
    std::vector<int> order;
    for (auto& kv : buckets) {
      const std::vector<int>& ps = kv.second;
      std::set<int> GA, GB;
      for (int sp : ps) { GA.insert(m.pair_geom1[sp]); GB.insert(m.pair_geom2[sp]); }
      int ba = kv.first.first, bb = kv.first.second;
      bool anchorB = ba == 0 ? false : (bb == 0 ? true : GB.size() <= GA.size());   // anchor side; the sphere sits on the other body
      const std::set<int>& anchors = anchorB ? GB : GA;
      for (int an : anchors) {
        BGroup g;
        g.body = anchorB ? ba : bb; g.anchor = an; g.start = (int)order.size(); g.count = 0;
        std::vector<int> partner;
        double mg = 0;
        for (int sp : ps) {
          if ((anchorB ? m.pair_geom2[sp] : m.pair_geom1[sp]) != an) continue;
          order.push_back(sp); g.count++;
          partner.push_back(anchorB ? m.pair_geom1[sp] : m.pair_geom2[sp]);
          if (m.pair_margin[sp] > mg) mg = m.pair_margin[sp];
        }
        for (int k = 0; k < 3; k++) { g.c[k] = 0; for (int pg : partner) g.c[k] += m.geom_pos[3 * pg + k] / partner.size(); }
        g.r = 0;
        for (int pg : partner) {
          double d2 = 0;
          for (int k = 0; k < 3; k++) { double d = m.geom_pos[3 * pg + k] - g.c[k]; d2 += d * d; }
          double rr = sqrt(d2) + m.geom_rbound[pg];
          if (rr > g.r) g.r = rr;
        }
        g.r = (g.r + mg) * (1.0 + 1e-5) + 1e-6;   // fp32 slack: the group test must never reject what the pair test accepts
        bgs.push_back(g);
      }
    }
    psrc = order;
  }
  h.nbgrp = (int)bgs.size();
#endif
  h.npair = (int)psrc.size();
  h.edges_per_con = 1;
  for (size_t p = 0; p < psrc.size(); p++) {
    int cd = m.pair_condim[psrc[p]], ne = cd == 1 ? 1 : 2 * (cd - 1);
    if (ne > h.edges_per_con) h.edges_per_con = ne;
  }
  std::vector<int> gmap(m.ngeom, -1), gsrc;
  for (size_t p = 0; p < psrc.size(); p++) {
    int ga = m.pair_geom1[psrc[p]], gb = m.pair_geom2[psrc[p]];
    if (gmap[ga] < 0) { gmap[ga] = (int)gsrc.size(); gsrc.push_back(ga); }
    if (!pgrid[p] && gmap[gb] < 0) { gmap[gb] = (int)gsrc.size(); gsrc.push_back(gb); }
  }
  h.ngeom = (int)gsrc.size();
  if (m.n_grid_dims >= 2 && m.grid_dims[0] > 0) {
    h.grid_len = m.grid_dims[0]; h.grid_wid = m.grid_dims[1]; h.ngridw = (h.grid_len * h.grid_wid + 31) / 32;
    h.grid_scale = (float)m.grid_param[0]; h.grid_top = (float)(m.grid_param[1] * m.grid_param[0]);
    h.grid_xc = (float)m.grid_param[2]; h.grid_yc = (float)m.grid_param[3];
  }
  h.nmjb = m.n_mjbody_rt > 0 ? m.n_mjbody_rt : m.nbody;   // blobs without the table: runtime bodies stand for themselves
  h.nsensor = m.nsensor;
  if (m.nsensor > 0 && m.n_sensor_type != m.nsensor) { err = "model blob lacks sensor_type"; return -1; }
  h.ncand_max = DM_NCAND_MAX;
  // models with several hundred candidate pairs (Adroit door: 278, large door / frame bounding spheres) fill 96 slots on
  // ~12 % of random-action env-steps (measured in the emulation): twice the slots for them
  if (m.npair > 255) h.ncand_max = 2 * DM_NCAND_MAX;
  if (h.npair > 65535) { err = "more than 65535 candidate geom pairs"; return -1; }
  h.ncon_max = m.nmocap > 0 ? 16 : 20;   // contacts kept per env per sub-step
  h.ngrp_max = m.nmocap > 0 ? 10 : 14;   // geom pairs in contact (+ welds) per env per sub-step
#ifdef B200_KITCHEN
  h.ncon_max = 24; h.ngrp_max = 18;      // the arm sweeping through kettle, knobs and doors (emulation soak: 15 / 13 seen)
#endif
  if (ngrp_cap > DM_NWELD_MAX && ngrp_cap < h.ngrp_max) h.ngrp_max = ngrp_cap;
  if (h.nb > DM_MAX_BODY) { err = "model has more than 32 runtime bodies"; return -1; }
  if (h.nv > DM_MAX_NV) { err = "model has more than 40 dofs"; return -1; }
  h.mask_words = (h.nv > 32 || force_wide) ? 2 : 1;
  h.penv_body = (penv_body > 0 && penv_body < h.nb) ? penv_body : -1;
  std::vector<int> tsrc;   // limited fixed tendons (unlimited ones have no effect without springs)
  for (int t = 0; t < m.ntendon; t++) {
    if (!m.ten_limited[t]) continue;
    if (m.ten_num[t] < 1 || m.ten_num[t] > 2) { err = "fixed tendons over more than 2 joints are not supported by the CUDA path"; return -1; }
    tsrc.push_back(t);
  }
  h.nten = (int)tsrc.size();
  for (int d = 0; d < m.nv; d++) if (m.dof_frictionloss[d] > 0) h.nfric = m.nv;
  {
    int nlim = 0;
    for (int j = 0; j < m.njnt; j++) if (m.jnt_limited[j] && m.jnt_type[j] != B200_JNT_FREE) nlim++;
    int want = nlim + h.nten;   // at most one side of every limit can be active at a time
    // models with tendon-coupled, friction-loaded joints (the Shadow hand) sit at many limits at once; the arm / legged
    // models keep the small table that lets 32 envs share one thread block
#ifdef B200_KITCHEN
    for (int e = 0; e < m.neq; e++) if (m.eq_type[e] == B200_EQ_JOINT) want++;   // one (always active) row per joint equality
    if (want > DM_NDOFROW_MIN) h.nten = h.nten > 0 ? h.nten : 0;
    h.ndr_max = want < DM_NDOFROW_MIN ? DM_NDOFROW_MIN : (want > 48 ? 48 : want);
#else
    h.ndr_max = (h.nten > 0 || h.nfric > 0) ? (want < DM_NDOFROW_MIN ? DM_NDOFROW_MIN : (want > 48 ? 48 : want)) : DM_NDOFROW_MIN;
#endif
  }
  int nweld = 0;
  for (int e = 0; e < m.neq; e++) if (m.eq_type[e] == B200_EQ_WELD) nweld++;
  if (nweld > DM_NWELD_MAX) { err = "too many weld constraints"; return -1; }
  h.iterations = m.opt_int[B200_OPTI_ITERATIONS]; h.ls_iterations = m.opt_int[B200_OPTI_LS_ITERATIONS];
  h.integrator = m.opt_int[B200_OPTI_INTEGRATOR];
  h.timestep = (float)m.opt[B200_OPT_TIMESTEP];
  for (int k = 0; k < 3; k++) { h.gravity[k] = (float)m.opt[B200_OPT_GRAVITY + k]; h.ref[k] = ref[k]; }
  h.tolerance = (float)m.opt[B200_OPT_TOLERANCE]; h.impratio = (float)m.opt[B200_OPT_IMPRATIO];
  h.meaninertia = (float)m.opt[B200_OPT_MEANINERTIA]; h.ls_tolerance = (float)m.opt[B200_OPT_LS_TOLERANCE];
  for (int d = 0; d < m.nv; d++) if (m.dof_damping[d] > 0) h.any_damping = 1;
  // offsets
  int nb = h.nb, njnt = h.njnt, nq = h.nq, nv = h.nv, nu = h.nu, ngeom = h.ngeom, nsite = h.nsite, nmocap = h.nmocap,
      neq = h.neq, npair = h.npair, ngridw = h.ngridw, ncon_max = h.ncon_max, ngrp_max = h.ngrp_max, ndr_max = h.ndr_max,
      nten = h.nten, nfric = h.nfric, nsensor = h.nsensor, ncx = h.nsensor > 0 ? h.ncon_max : 0, MW = h.mask_words,
      grp_words = MW == 2 ? 11 : 9, npenv = h.penv_body > 0 ? 8 : 0, nmjb = h.nmjb;
#ifdef B200_HULL
  int nhullv = m.n_hull_vert / 3;
  if (m.n_geom_hull != 2 * m.ngeom) { err = "model blob lacks the hull vertex table (compile with mesh_hull)"; return -1; }
#endif
#ifdef B200_KITCHEN_GROUPS
  int nbgrp = h.nbgrp;
#endif
  int nrkq = h.integrator == B200_INT_RK4 ? nq : 0, nrkv = h.integrator == B200_INT_RK4 ? nv : 0;
  int off = (int)((sizeof(DMHead) + 3) / 4);
#define X(name, w, kind) h.o_##name = off; off += (w) * (kind);
  DM_ARRAYS_HOT(X)
#undef X
  off = (off + 3) & ~3;  // 16-byte multiple for the bulk copy
  h.hot_words = off;
#define X(name, w, kind) h.o_##name = off; off += (w) * (kind);
  DM_ARRAYS_COLD(X)
#undef X
  off = (off + 3) & ~3;
  h.nwords = off;
  int so = 0;
#define X(name, words) h.s_##name = so; so += (words); so = (so + 1) & ~1;
  DM_SCRATCH_PERSIST(X)
#undef X
  {
    so = (so + 3) & ~3;   // 16-byte aligned: the register Cholesky reads its column buffers (in the dead H region) as float4
    int nM = nv * (nv + 1) / 2, u = so;
    int d6off = 16 * nb > nM ? 16 * nb : nM;
    // room for a line-search edge list (x0, v, D per edge slot) over H and d6.  Only the kitchen builds still use it (the others keep
    // their edges in registers); it stays for all because it sizes this region for AntMaze and PointMaze too, and with it their
    // scratch (scr_words, hence the accepted block sizes) and their narrow-phase slots in region A
    int need = 3 * (h.edges_per_con * ncon_max + 6 * DM_NWELD_MAX + ndr_max) - 6 * nv;
    if (need > d6off) d6off = need;
    // and so do two solver temporaries that are dead by the time H is built: the per-group J qacc of rows_begin (6 per group,
    // from H's start) and the packed 6x6 blocks of the groups build_H is adding (21 words each after H: room for one at least)
    need = (nM + 21 > 6 * ngrp_max ? nM + 21 : 6 * ngrp_max) - 6 * nv;
    if (need > d6off) d6off = need;
    d6off = (d6off + 1) & ~1;
    h.s_kinA = u; h.s_kinB = u + 8 * nb;
    h.s_cinert = u; h.s_b6 = u + 10 * nb; h.s_d6 = u + d6off;
    int after = u + d6off + 6 * nv;
    h.s_geom_xpos = after; h.s_cand = after + 3 * ngeom;
    h.s_H = u; h.s_grad = after; h.s_search = after + nv; h.s_Ma = after + 2 * nv; h.s_Mv = after + 3 * nv;
    h.s_cvel = u;
    int endA = after + 3 * ngeom + (h.npair > 255 ? h.ncand_max / 2 : h.ncand_max / 4), endB = after + 4 * nv;   // candidate slots: 1 or 2 bytes
#ifdef B200_KITCHEN_GROUPS
    h.s_surv = endA; endA += DM_NSURV_MAX + 1;   // surviving groups: (first pair | running pair count << 16) + one end marker
#endif
    so = endA > endB ? endA : endB;
    h.s_cslotA = h.s_b6; h.ncslotA = (h.s_d6 + 6 * nv - h.s_b6) / DM_CSLOT_WORDS;
    h.s_cslotB = h.s_con; h.ncslotB = (ncon_max * CON_WORDS) / DM_CSLOT_WORDS;

    if (h.ncslotA > 32) h.ncslotA = 32;
    if (h.ncslotA + h.ncslotB > 32) h.ncslotB = 32 - h.ncslotA;
    if (h.ncslotA < 1) { err = "no scratch for a narrow-phase lane slot"; return -1; }
  }
  h.scr_words = (so + 3) & ~3;
  (void)nq;
  buf.assign(h.nwords, 0);
  auto F = [&](int o, int i, double v) { buf[o + i] = f2w((float)v); };
  auto I = [&](int o, int i, int v) { buf[o + i] = (uint32_t)v; };
  // masks
  typedef unsigned long long u64;
  std::vector<u64> anc(nv, 0), pre(nv, 0), bodyanc(nb, 0);
  std::vector<uint32_t> sub(nb, 0);
  auto PUTM = [&](int o, int i, u64 v) { buf[o + MW * i] = (uint32_t)v; if (MW == 2) buf[o + 2 * i + 1] = (uint32_t)(v >> 32); };
  for (int d = 0; d < nv; d++) {
    int p = m.dof_parent[d];
    anc[d] = (p >= 0 ? anc[p] : (u64)0) | ((u64)1 << d);
  }
  for (int b = 1; b < nb; b++) {
    // dofs of this body and of all ancestors
    int a = b;
    while (a > 0 && m.body_dofnum[a] == 0) a = m.body_parent[a];
    bodyanc[b] = a > 0 ? anc[m.body_dofadr[a] + m.body_dofnum[a] - 1] : (u64)0;
  }
  for (int b = nb - 1; b >= 0; b--) {
    sub[b] |= 1u << b;
    if (b > 0) sub[m.body_parent[b]] |= sub[b];
  }
  for (int d = 0; d < nv; d++) {
    int b = m.dof_body[d], j = m.dof_jnt[d];
    u64 mask = bodyanc[m.body_parent[b]];  // all dofs of ancestor bodies
    // earlier dofs of the same body: every earlier joint of the body; for a free joint's rotational dofs only the
    // three translational dofs (body-fixed axes: no rot-rot terms, see DESIGN.md "velocity products")
    for (int e = m.body_dofadr[b]; e < d; e++) {
      if (m.dof_jnt[e] != j) mask |= (u64)1 << e;
      else if (m.jnt_type[j] == B200_JNT_FREE && d - m.jnt_dofadr[j] >= 3 && e - m.jnt_dofadr[j] < 3) mask |= (u64)1 << e;
    }
    pre[d] = mask;
  }
  {
    int maxdepth = 1;
    std::vector<int> depth(nb, 0);
    for (int b = 1; b < nb; b++) { depth[b] = depth[m.body_parent[b]] + 1; if (depth[b] > maxdepth) maxdepth = depth[b]; }
    h.kin_iters = 0;
    while ((1 << h.kin_iters) < maxdepth) h.kin_iters++;
  }
  for (int b = 0; b < nb; b++) {
    I(h.o_body_parent, b, m.body_parent[b]); I(h.o_body_jntadr, b, m.body_jntadr[b]); I(h.o_body_jntnum, b, m.body_jntnum[b]);
    I(h.o_body_dofadr, b, m.body_dofadr[b]); I(h.o_body_dofnum, b, m.body_dofnum[b]); I(h.o_body_mocapid, b, m.body_mocapid[b]);
    PUTM(h.o_body_ancdof, b, bodyanc[b]); buf[h.o_body_sub + b] = sub[b];
    for (int k = 0; k < 3; k++) { F(h.o_body_pos, 3 * b + k, m.body_pos[3 * b + k]); F(h.o_body_ipos, 3 * b + k, m.body_ipos[3 * b + k]);
      F(h.o_body_inertia, 3 * b + k, m.body_inertia[3 * b + k]); }
    for (int k = 0; k < 4; k++) { F(h.o_body_quat, 4 * b + k, m.body_quat[4 * b + k]); F(h.o_body_iquat, 4 * b + k, m.body_iquat[4 * b + k]); }
    F(h.o_body_mass, b, m.body_mass[b]);
  }
  for (int j = 0; j < njnt; j++) {
    if (m.jnt_type[j] == B200_JNT_BALL) { err = "ball joints are not supported"; return -1; }
    I(h.o_jnt_type, j, m.jnt_type[j]); I(h.o_jnt_body, j, m.jnt_body[j]); I(h.o_jnt_qposadr, j, m.jnt_qposadr[j]);
    I(h.o_jnt_dofadr, j, m.jnt_dofadr[j]); I(h.o_jnt_limited, j, m.jnt_limited[j]);
    for (int k = 0; k < 3; k++) { F(h.o_jnt_pos, 3 * j + k, m.jnt_pos[3 * j + k]); F(h.o_jnt_axis, 3 * j + k, m.jnt_axis[3 * j + k]); }
    for (int k = 0; k < 2; k++) { F(h.o_jnt_range, 2 * j + k, m.jnt_range[2 * j + k]); F(h.o_jnt_solref, 2 * j + k, m.jnt_solref[2 * j + k]); }
    for (int k = 0; k < 5; k++) F(h.o_jnt_solimp, 5 * j + k, m.jnt_solimp[5 * j + k]);
    F(h.o_jnt_margin, j, m.jnt_margin[j]); F(h.o_jnt_stiffness, j, m.jnt_stiffness[j]);
    F(h.o_jnt_qpos0, j, m.qpos0[m.jnt_qposadr[j]]); F(h.o_jnt_qspring, j, m.qpos_spring[m.jnt_qposadr[j]]);
    if (m.jnt_type[j] == B200_JNT_FREE && m.body_jntnum[m.jnt_body[j]] != 1) { err = "free joint must be the only joint of its body"; return -1; }
  }
  for (int d = 0; d < nv; d++) {
    I(h.o_dof_body, d, m.dof_body[d]); I(h.o_dof_jnt, d, m.dof_jnt[d]); PUTM(h.o_dof_anc, d, anc[d]); PUTM(h.o_dof_pre, d, pre[d]);
    F(h.o_dof_armature, d, m.dof_armature[d]); F(h.o_dof_damping, d, m.dof_damping[d]);
    F(h.o_dof_frictionloss, d, m.dof_frictionloss[d]); F(h.o_dof_invweight0, d, m.dof_invweight0[d]);
    if (nfric) {
      // constant row parameters of the dof-friction constraint (pos = 0, margin = 0): D = 1/R, B of the reference acceleration
      double fl = m.dof_frictionloss[d];
      const double* si = m.dof_solimp_fri + 5 * d; const double* sr = m.dof_solref_fri + 2 * d;
      double d0 = fmin(fmax(si[0], 0.0001), 0.9999), d1 = fmin(fmax(si[1], 0.0001), 0.9999), width = fmax(si[2], 0.0);
      double imp = (d0 == d1 || width <= 1e-15) ? 0.5 * (d0 + d1) : d0;   // x = |pos - margin| / width = 0
      double R = fmax((1 - imp) / imp * m.dof_invweight0[d], 1e-15);
      double B = sr[0] > 0 ? 2.0 / fmax(d1 * fmax(sr[0], 2 * m.opt[B200_OPT_TIMESTEP]), 1e-15) : -sr[1] / d1;
      F(h.o_dof_fricD, d, fl > 0 ? 1.0 / R : 0.0); F(h.o_dof_fricB, d, B);
    }
  }
  for (int t = 0; t < nten; t++) {
    int st = tsrc[t], adr = m.ten_adr[st];
    for (int k = 0; k < 2; k++) {
      bool has = k < m.ten_num[st];
      int d = has ? m.wrap_dof[adr + k] : -1;
      if (has && m.jnt_type[m.dof_jnt[d]] == B200_JNT_FREE) { err = "tendon over a free joint"; return -1; }
      I(h.o_ten_dof, 2 * t + k, d); I(h.o_ten_qadr, 2 * t + k, has ? m.jnt_qposadr[m.dof_jnt[d]] : 0);
      F(h.o_ten_coef, 2 * t + k, has ? m.wrap_coef[adr + k] : 0.0);
      F(h.o_ten_range, 2 * t + k, m.ten_range[2 * st + k]); F(h.o_ten_solref, 2 * t + k, m.ten_solref[2 * st + k]);
    }
    F(h.o_ten_margin, t, m.ten_margin[st]); F(h.o_ten_invweight, t, m.ten_invweight0[st]);
    for (int k = 0; k < 5; k++) F(h.o_ten_solimp, 5 * t + k, m.ten_solimp[5 * st + k]);
  }
  for (int g = 0; g < ngeom; g++) {
    int sg = gsrc[g];
    I(h.o_geom_type, g, m.geom_type[sg]); I(h.o_geom_body, g, m.geom_body[sg]);
    for (int k = 0; k < 3; k++) { F(h.o_geom_pos, 3 * g + k, m.geom_pos[3 * sg + k]); F(h.o_geom_size, 3 * g + k, m.geom_size[3 * sg + k]); }
    if (m.geom_type[sg] == B200_GEOM_PLANE) {
      // a plane's size is never used by the collision routines: the slot carries its world normal (planes sit on the world body)
      if (m.geom_body[sg] != 0) { err = "plane geoms must belong to the world body"; return -1; }
      const double* q = m.geom_quat + 4 * sg;
      F(h.o_geom_size, 3 * g + 0, 2 * (q[1] * q[3] + q[0] * q[2])); F(h.o_geom_size, 3 * g + 1, 2 * (q[2] * q[3] - q[0] * q[1]));
      F(h.o_geom_size, 3 * g + 2, q[0] * q[0] - q[1] * q[1] - q[2] * q[2] + q[3] * q[3]);
    }
    for (int k = 0; k < 4; k++) F(h.o_geom_quat, 4 * g + k, m.geom_quat[4 * sg + k]);
    F(h.o_geom_rbound, g, m.geom_rbound[sg]);
    I(h.o_geom_mjb, g, m.n_geom_mjbody == m.ngeom ? m.geom_mjbody[sg] : m.geom_body[sg]);
#ifdef B200_HULL
    I(h.o_geom_hull, 2 * g, m.geom_hull[2 * sg]); I(h.o_geom_hull, 2 * g + 1, m.geom_hull[2 * sg + 1]);
    if (m.geom_type[sg] == B200_GEOM_MESH && m.geom_hull[2 * sg + 1] < 4) { err = "mesh geom without a hull vertex table"; return -1; }
#else
    if (m.geom_type[sg] == B200_GEOM_MESH) { err = "mesh geoms need the hull build of the library (models compiled without mesh_hull carry box proxies)"; return -1; }
#endif
  }
#ifdef B200_HULL
  for (int i = 0; i < 3 * nhullv; i++) F(h.o_hull_vert, i, m.hull_vert[i]);
#endif
  for (int p = 0; p < npair; p++) {
    int sp = psrc[p];
    I(h.o_pair_geom1, p, gmap[m.pair_geom1[sp]]); I(h.o_pair_geom2, p, pgrid[p] ? -1 : gmap[m.pair_geom2[sp]]); I(h.o_pair_condim, p, m.pair_condim[sp]);
    int t1 = m.geom_type[m.pair_geom1[sp]], t2 = m.geom_type[m.pair_geom2[sp]];
    bool r1 = t1 == B200_GEOM_SPHERE || t1 == B200_GEOM_CAPSULE, r2 = t2 == B200_GEOM_SPHERE || t2 == B200_GEOM_CAPSULE;
    bool c1 = t1 == B200_GEOM_CYLINDER || t1 == B200_GEOM_ELLIPSOID, c2 = t2 == B200_GEOM_CYLINDER || t2 == B200_GEOM_ELLIPSOID;
    bool v1 = r1 || c1 || t1 == B200_GEOM_BOX, v2 = r2 || c2 || t2 == B200_GEOM_BOX;   // convex primitives
    bool ok = (t1 == B200_GEOM_PLANE && (t2 == B200_GEOM_BOX || r2 || c2)) || (t1 == B200_GEOM_BOX && t2 == B200_GEOM_BOX) ||
              (r1 && t2 == B200_GEOM_BOX) || (r1 && r2) || ((c1 || c2) && v1 && v2);
#ifdef B200_HULL
    {  // hull geoms: plane-hull has its own routine, every other pair with a hull goes through the portal-refinement collider
      bool m1 = t1 == B200_GEOM_MESH, m2 = t2 == B200_GEOM_MESH;
      if ((t1 == B200_GEOM_PLANE && m2) || ((m1 || m2) && (v1 || m1) && (v2 || m2))) { ok = true; c1 = c1 || m1; c2 = c2 || m2; }
    }
#endif
    if (r1 && r2) h.any_round_pair = 1;
    if (c1 || c2) h.any_convex_pair = 1;   // served by the general convex collider (kernel builds with CX)

    if (!ok) { err = "collision pair type not supported by the CUDA path yet"; return -1; }
#ifdef B200_KITCHEN
    if (m.pair_condim[sp] != 1 && m.pair_condim[sp] != 3 && m.pair_condim[sp] != 4 && m.pair_condim[sp] != 6) { err = "condim must be 1, 3, 4 or 6"; return -1; }
#else
    if (m.pair_condim[sp] != 1 && m.pair_condim[sp] != 3 && m.pair_condim[sp] != 4) { err = "condim must be 1, 3 or 4 on the CUDA path"; return -1; }
#endif
    F(h.o_pair_friction, 3 * p + 0, m.pair_friction[5 * sp + 0]); F(h.o_pair_friction, 3 * p + 1, m.pair_friction[5 * sp + 2]);
    F(h.o_pair_friction, 3 * p + 2, m.pair_friction[5 * sp + 3]);
    F(h.o_pair_margin, p, m.pair_margin[sp]); F(h.o_pair_gap, p, m.pair_gap[sp]);
    for (int k = 0; k < 2; k++) { F(h.o_pair_solref, 2 * p + k, m.pair_solref[2 * sp + k]); F(h.o_pair_invweight, 2 * p + k, m.pair_invweight[2 * sp + k]); }
    for (int k = 0; k < 5; k++) F(h.o_pair_solimp, 5 * p + k, m.pair_solimp[5 * sp + k]);
  }
#ifdef B200_KITCHEN_GROUPS
  for (int g = 0; g < nbgrp; g++) {
    I(h.o_bg_body, g, bgs[g].body); I(h.o_bg_anchor, g, gmap[bgs[g].anchor]); I(h.o_bg_start, g, bgs[g].start); I(h.o_bg_count, g, bgs[g].count);
    for (int k = 0; k < 3; k++) F(h.o_bg_center, 3 * g + k, bgs[g].c[k]);
    F(h.o_bg_radius, g, bgs[g].r);
  }
#endif
#ifdef B200_KITCHEN
  // the kitchen builds' line search walks an edge list in the solver scratch (the other builds are checked by b200sim_create)
  if (3 * dm_ls_edges(h) > h.s_grad - h.s_H) { err = "line-search edge list does not fit the solver scratch"; return -1; }
#endif
  for (int k = 0; k < nsensor; k++) {
    I(h.o_sensor_site, k, m.sensor_site[k]); I(h.o_sensor_body, k, m.sensor_body[k]); I(h.o_sensor_type, k, m.sensor_type[k]);
    for (int a = 0; a < 3; a++) F(h.o_sensor_size, 3 * k + a, m.sensor_size[3 * k + a]);
  }
  for (int i = 0; i < h.grid_len * h.grid_wid; i++) if (m.grid_walls[i]) buf[h.o_grid_walls + i / 32] |= 1u << (i % 32);
  for (int s = 0; s < nsite; s++) {
    I(h.o_site_body, s, m.site_body[s]);
    for (int k = 0; k < 3; k++) F(h.o_site_pos, 3 * s + k, m.site_pos[3 * s + k]);
    for (int k = 0; k < 4; k++) F(h.o_site_quat, 4 * s + k, m.site_quat[4 * s + k]);
  }
  for (int a = 0; a < nu; a++) {
    I(h.o_act_trnid, a, m.act_trnid[a]); I(h.o_act_ctrllimited, a, m.act_ctrllimited[a]); I(h.o_act_forcelimited, a, m.act_forcelimited[a]);
    F(h.o_act_gear, a, m.act_gear[a]); F(h.o_act_gain, a, m.act_gainprm[3 * a]);
    for (int k = 0; k < 3; k++) F(h.o_act_bias, 3 * a + k, m.act_biasprm[3 * a + k]);
    for (int k = 0; k < 2; k++) { F(h.o_act_ctrlrange, 2 * a + k, m.act_ctrlrange[2 * a + k]); F(h.o_act_forcerange, 2 * a + k, m.act_forcerange[2 * a + k]); }
  }
  for (int e = 0; e < neq; e++) {
#ifdef B200_KITCHEN
    // work in progress (DESIGN.md section 7, step i): joint equalities become two-sided dof rows; only the emulation build
    // of the Kitchen bring-up compiles this, the product library still refuses the model
    if (m.eq_type[e] != B200_EQ_WELD && m.eq_type[e] != B200_EQ_JOINT) { err = "only weld and joint equalities are supported"; return -1; }
#else
    if (m.eq_type[e] != B200_EQ_WELD) { err = "only weld equalities are supported by the CUDA path yet"; return -1; }
#endif
    I(h.o_eq_type, e, m.eq_type[e]); I(h.o_eq_obj1, e, m.eq_obj1[e]); I(h.o_eq_obj2, e, m.eq_obj2[e]); I(h.o_eq_active, e, m.eq_active[e]);
    const double* data = eq_data_override ? eq_data_override + 11 * e : m.eq_data + 11 * e;
    for (int k = 0; k < 11; k++) F(h.o_eq_data, 11 * e + k, data[k]);
    for (int k = 0; k < 2; k++) { F(h.o_eq_solref, 2 * e + k, m.eq_solref[2 * e + k]); F(h.o_eq_invweight, 2 * e + k, m.eq_invweight[2 * e + k]); }
    for (int k = 0; k < 5; k++) F(h.o_eq_solimp, 5 * e + k, m.eq_solimp[5 * e + k]);
  }
  for (int i = 0; i < nmocap; i++) I(h.o_mocap_body, i, m.mocap_body[i]);
  for (int b = 0; b < nmjb; b++) I(h.o_mjb_rt, b, m.n_mjbody_rt > 0 ? m.mjbody_rt[b] : b);
  if (nmjb > 255) { err = "more than 255 MJCF bodies"; return -1; }
  memcpy(buf.data(), &h, sizeof(h));
  return 0;
}
