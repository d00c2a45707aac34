// TEST-ONLY device harness: runs one stage of the kernel source on the GPU, on its own, so that the suite can compare that stage
// with an fp64 reference instead of a whole env-step.  Compiled with the product's nvcc flags (gymnasium_robotics_b200._lib.NVCC_FLAGS)
// and the defines of one product translation unit per library; never linked into the product.
//
// One warp per block and one case per block, so one launch runs a whole batch of cases.  Each block copies its case from global
// into dynamic shared memory (the stages assume shared-memory operands), runs the stage, and copies everything back -- the
// operands and the work areas, so that the host can check what the stage wrote and what it must have left alone.
//
// spd: spd_solve<NVP>, the register Cholesky of the Newton direction (A == scratchH, in place) and of the implicit-damping Euler
// step (A = M, dadd = dof damping, scratchH = the dead H region).  Only the header's nv is read, so a zeroed header with nv set
// stands for the model, and any nv up to NVP can be solved.
//
// collide / kin: whole stages on a real model (dm_build on the host with this library's defines), staged as the step kernel
// stages it (step_kernel.cuh): header + HOT arrays in shared memory, the COLD arrays -- the kitchen groups build's pair list among
// them -- read from the global model, one env's scratch after the hot words.  The host hands in a whole scratch image per case
// and gets the whole image back.  collide = collision<HF, CX> with HF and CX derived from NVP as forward<NVP> derives them;
// kin = kinematics, com_quantities and mass_matrix.
//
// problem / jv: the problem the Newton solver is given.  problem = every stage forward<NVP> runs up to the first direction solve:
// kinematics, com_quantities, mass_matrix, collision<HF, CX>, make_constraint<HF>, smooth_forces, newton_begin<HF> (M qacc of the
// warm start, rows_begin, the check: fcon through pass_F and grad) and build_H<HF>.  jv = rows_from_vec<HF>(c, SF(search)) on an image
// that problem returned: with a unit vector in search it reads one column of the kernel's implicit J into the rows' JV slots.
//
// touch: touch_observe (touch_mode 1, the sensordata values) on an image that problem returned, or on such an image with its contact
// records edited on the host: nsensor floats per case into `out`.  The records hold the base-row values U of the warm-start qacc that
// newton_begin left, so the forces the sensors sum are a deterministic function of the injected state.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../gymnasium_robotics_b200/csrc/fetch_task.cuh"
#include <string>
#include <vector>

// header words in front of the operands, rounded to 16 bytes (the register Cholesky reads its column buffers as float4)
#define DEVSIM_HEAD_WORDS ((int)((sizeof(DMHead) + 15) / 16 * 4))

// shared memory of one block: header | A (la) | x (lx) | dadd (lx) | scratchH (lh); la, lx, lh are multiples of 4
template <int NVP>
__global__ void __launch_bounds__(32) spd_kernel(const int* __restrict__ nv, float* A, const float* __restrict__ dadd, float hh, int use_dadd,
                                                  float* x, float* H, int la, int lx, int lh, int inplace) {
  const int e = blockIdx.x, lane = threadIdx.x;
  for (int k = lane; k < DEVSIM_HEAD_WORDS; k += 32) b200_smem[k] = 0u;
  __syncwarp();
  DMHead* head = (DMHead*)b200_smem;
  if (lane == 0) head->nv = nv[e];
  float* sA = (float*)(b200_smem + DEVSIM_HEAD_WORDS);
  float* sX = sA + la;
  float* sD = sX + lx;
  float* sH = sD + lx;
  for (int k = lane; k < la; k += 32) sA[k] = A[(size_t)e * la + k];
  for (int k = lane; k < lx; k += 32) { sX[k] = x[(size_t)e * lx + k]; sD[k] = dadd[(size_t)e * lx + k]; }
  for (int k = lane; k < lh; k += 32) sH[k] = H[(size_t)e * lh + k];
  __syncwarp();
  Ctx c;
  c.mg = b200_smem; c.mw = b200_smem; c.h = head; c.s = sH; c.lane = lane;
#ifdef B200_STAGE_TIMING
  c.tim = nullptr;
#endif
  spd_solve<NVP>(c, sA, use_dadd ? sD : nullptr, hh, sX, inplace ? sA : sH);
  __syncwarp();
  for (int k = lane; k < la; k += 32) A[(size_t)e * la + k] = sA[k];
  for (int k = lane; k < lx; k += 32) x[(size_t)e * lx + k] = sX[k];
  for (int k = lane; k < lh; k += 32) H[(size_t)e * lh + k] = sH[k];
}

static char g_err[512];

extern "C" const char* devsim_last_error() { return g_err; }

#define DEVSIM_OK(call)                                                                                 \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess) {                                                                            \
      snprintf(g_err, sizeof(g_err), "%s: %s", #call, cudaGetErrorString(e_));                          \
      rc = -2;                                                                                          \
      goto done;                                                                                        \
    }                                                                                                   \
  } while (0)

// ncase cases in one launch; host arrays nv[ncase], A[ncase][la], dadd[ncase][lx], x[ncase][lx], H[ncase][lh]; A, x and H are
// overwritten with their contents after the solve.  Returns 0, -1 for an NVP this library does not instantiate, -2 on a CUDA error
// (devsim_last_error()).
extern "C" int devsim_spd(int nvp, int ncase, const int* nv, float* A, const float* dadd, float hh, int use_dadd, float* x, float* H,
                          int la, int lx, int lh, int inplace) {
  int rc = 0;
  int* d_nv = nullptr;
  float *d_A = nullptr, *d_D = nullptr, *d_x = nullptr, *d_H = nullptr;
  const size_t smem = (size_t)(DEVSIM_HEAD_WORDS + la + 2 * lx + lh) * 4;
  g_err[0] = 0;
  DEVSIM_OK(cudaMalloc(&d_nv, sizeof(int) * ncase));
  DEVSIM_OK(cudaMalloc(&d_A, sizeof(float) * ncase * la));
  DEVSIM_OK(cudaMalloc(&d_D, sizeof(float) * ncase * lx));
  DEVSIM_OK(cudaMalloc(&d_x, sizeof(float) * ncase * lx));
  DEVSIM_OK(cudaMalloc(&d_H, sizeof(float) * ncase * lh));
  DEVSIM_OK(cudaMemcpy(d_nv, nv, sizeof(int) * ncase, cudaMemcpyHostToDevice));
  DEVSIM_OK(cudaMemcpy(d_A, A, sizeof(float) * ncase * la, cudaMemcpyHostToDevice));
  DEVSIM_OK(cudaMemcpy(d_D, dadd, sizeof(float) * ncase * lx, cudaMemcpyHostToDevice));
  DEVSIM_OK(cudaMemcpy(d_x, x, sizeof(float) * ncase * lx, cudaMemcpyHostToDevice));
  DEVSIM_OK(cudaMemcpy(d_H, H, sizeof(float) * ncase * lh, cudaMemcpyHostToDevice));
  {
    int matched = 0;
#define DEVSIM_SPD(V)                                                                                                        \
    if (nvp == V) {                                                                                                          \
      matched = 1;                                                                                                           \
      DEVSIM_OK(cudaFuncSetAttribute(spd_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                \
      spd_kernel<V><<<ncase, 32, smem>>>(d_nv, d_A, d_D, hh, use_dadd, d_x, d_H, la, lx, lh, inplace);                      \
    }
#if defined(B200_WIDE)
    DEVSIM_SPD(36)
#elif defined(B200_KITCHEN)
    DEVSIM_SPD(31)
#else
    DEVSIM_SPD(14) DEVSIM_SPD(15) DEVSIM_SPD(21) DEVSIM_SPD(22) DEVSIM_SPD(30)
#endif
#undef DEVSIM_SPD
    if (!matched) { snprintf(g_err, sizeof(g_err), "devsim_spd: NVP %d is not instantiated in this library", nvp); rc = -1; goto done; }
  }
  DEVSIM_OK(cudaGetLastError());
  DEVSIM_OK(cudaDeviceSynchronize());
  DEVSIM_OK(cudaMemcpy(A, d_A, sizeof(float) * ncase * la, cudaMemcpyDeviceToHost));
  DEVSIM_OK(cudaMemcpy(x, d_x, sizeof(float) * ncase * lx, cudaMemcpyDeviceToHost));
  DEVSIM_OK(cudaMemcpy(H, d_H, sizeof(float) * ncase * lh, cudaMemcpyDeviceToHost));
done:
  cudaFree(d_nv); cudaFree(d_A); cudaFree(d_D); cudaFree(d_x); cudaFree(d_H);
  return rc;
}

enum { DEVSIM_COLLIDE = 0, DEVSIM_KIN = 1, DEVSIM_PROBLEM = 2, DEVSIM_JV = 3, DEVSIM_BUILD_H = 4, DEVSIM_TOUCH = 5 };

template <int NVP>
__global__ void __launch_bounds__(32) stage_kernel(const uint32_t* __restrict__ model, int stage, float* scratch, float* out) {
  const int e = blockIdx.x, lane = threadIdx.x;
  const DMHead* hg = (const DMHead*)model;
  const int hot = hg->hot_words, sw = hg->scr_words;
  for (int k = lane; k < hot; k += 32) b200_smem[k] = model[k];
  float* s = (float*)(b200_smem + hot);
  for (int k = lane; k < sw; k += 32) s[k] = scratch[(size_t)e * sw + k];
  __syncwarp();
  Ctx c;
  c.mg = model; c.mw = b200_smem; c.h = (const DMHead*)b200_smem; c.s = s; c.lane = lane;
#ifdef B200_STAGE_TIMING
  c.tim = nullptr;
#endif
  constexpr bool HF = NVP >= 30;
  constexpr bool CX = NVP == 22 || NVP >= 30;
  if (stage == DEVSIM_COLLIDE) collision<HF, CX>(c);
  else if (stage == DEVSIM_KIN) { kinematics(c); com_quantities(c); mass_matrix(c); }
  else if (stage == DEVSIM_PROBLEM) {
    kinematics(c); com_quantities(c); mass_matrix(c);
    collision<HF, CX>(c);
    make_constraint<HF>(c);
    smooth_forces(c);
    newton_begin<HF>(c);
    build_H<HF>(c);
  } else if (stage == DEVSIM_JV) rows_from_vec<HF>(c, SF(search));
  else if (stage == DEVSIM_TOUCH) {
    FetchTask t;
    memset(&t, 0, sizeof(t));
    t.touch_mode = 1;
    touch_observe(c, t, out + (size_t)e * c.h->nsensor);
  } else build_H<HF>(c);
  __syncwarp();
  for (int k = lane; k < sw; k += 32) scratch[(size_t)e * sw + k] = s[k];
}

__global__ void ray_hits_kernel(int type, float s0, float s1, float s2, int n, const float* p, const float* d, int* hit) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const float size[3] = {s0, s1, s2};
  if (i < n) hit[i] = ray_hits_site(type, size, p + 3 * i, d + 3 * i) ? 1 : 0;
}

#ifdef B200_WIDE
static const bool kWide = true;   // 64-bit dof masks, as hostsim's wide flavor builds them
#else
static const bool kWide = false;
#endif

struct DevModel {
  std::vector<uint8_t> blob;
  b200_model_view view;
  std::vector<uint32_t> model;
};

extern "C" {
// the device model of a blob as this library's unit builds it (NULL on a refusal: devsim_last_error())
void* devsim_model_create(const void* blob, size_t n, const double* eq_data, const float* ref, int penv_body, int ngrp_cap) {
  DevModel* d = new DevModel;
  std::string err;
  d->blob.assign((const uint8_t*)blob, (const uint8_t*)blob + n);
  if (b200_model_parse(d->blob.data(), n, &d->view) != 0) { snprintf(g_err, sizeof(g_err), "not a model blob"); delete d; return nullptr; }
  if (dm_build(d->view, eq_data, ref, d->model, err, penv_body, kWide, ngrp_cap) != 0) {
    snprintf(g_err, sizeof(g_err), "dm_build: %s", err.c_str());
    delete d;
    return nullptr;
  }
  return d;
}
void devsim_model_destroy(void* p) { delete (DevModel*)p; }
// the device model words, writable: devsim_stage uploads them for every run, so a test may edit a table for the runs that follow
uint32_t* devsim_model_words(void* p) { return ((DevModel*)p)->model.data(); }
int devsim_scr_words(void* p) { return ((const DMHead*)((DevModel*)p)->model.data())->scr_words; }
int devsim_model_nwords(void* p) { return ((const DMHead*)((DevModel*)p)->model.data())->nwords; }
// this library's contact-record and group layout (dmodel.h): C_MU, C_U, C_DIMGRP, CON_WORDS, GRP_WORDS, G_RANGE, C_W, C_D, CX_POS, CX_PAIR,
// CX_WORDS
void devsim_layout(int* out) {
  out[0] = C_MU; out[1] = C_U; out[2] = C_DIMGRP; out[3] = CON_WORDS; out[4] = GRP_WORDS; out[5] = G_RANGE;
  out[6] = C_W; out[7] = C_D; out[8] = CX_POS; out[9] = CX_PAIR; out[10] = CX_WORDS;
}
// scratch offset of a named per-env array (DM_SCRATCH_PERSIST / DM_SCRATCH_UNION), or model offset of a model array (DM_ARRAYS)
int devsim_offset(void* p, const char* name, int model_array) {
  const DMHead* h = (const DMHead*)((DevModel*)p)->model.data();
  if (model_array) {
#define X(nm, w, kind) if (strcmp(name, #nm) == 0) return h->o_##nm;
    DM_ARRAYS(X)
#undef X
    return -1;
  }
#define X(nm, words) if (strcmp(name, #nm) == 0) return h->s_##nm;
  DM_SCRATCH_PERSIST(X)
#undef X
#define X(nm) if (strcmp(name, #nm) == 0) return h->s_##nm;
  DM_SCRATCH_UNION(X)
#undef X
  return -1;
}

// ray_hits_site on n rays given in the site frame: p, d [n][3] host arrays -> hit [n].  Returns 0, -2 on a CUDA error.
int devsim_ray_hits(int type, const float* size, int n, const float* p, const float* d, int* hit) {
  int rc = 0;
  float *d_p = nullptr, *d_d = nullptr;
  int* d_h = nullptr;
  g_err[0] = 0;
  if (n <= 0) return 0;
  DEVSIM_OK(cudaMalloc(&d_p, sizeof(float) * 3 * n));
  DEVSIM_OK(cudaMalloc(&d_d, sizeof(float) * 3 * n));
  DEVSIM_OK(cudaMalloc(&d_h, sizeof(int) * n));
  DEVSIM_OK(cudaMemcpy(d_p, p, sizeof(float) * 3 * n, cudaMemcpyHostToDevice));
  DEVSIM_OK(cudaMemcpy(d_d, d, sizeof(float) * 3 * n, cudaMemcpyHostToDevice));
  ray_hits_kernel<<<(n + 127) / 128, 128>>>(type, size[0], size[1], size[2], n, d_p, d_d, d_h);
  DEVSIM_OK(cudaGetLastError());
  DEVSIM_OK(cudaMemcpy(hit, d_h, sizeof(int) * n, cudaMemcpyDeviceToHost));
done:
  cudaFree(d_p); cudaFree(d_d); cudaFree(d_h);
  return rc;
}

// run one stage (DEVSIM_COLLIDE, DEVSIM_KIN, DEVSIM_PROBLEM, DEVSIM_JV, DEVSIM_BUILD_H, DEVSIM_TOUCH) of the NVP = nvp instantiation on ncase scratch
// images [ncase][scr_words], one block each; the images are overwritten with the scratch after the stage, and DEVSIM_TOUCH writes
// out[ncase][nsensor] (NULL for the other stages).  Returns 0, -1 for an NVP this library does not instantiate, -2 on a CUDA error.
int devsim_stage(void* p, int nvp, int stage, int ncase, float* scratch, float* out) {
  int rc = 0;
  const DevModel* d = (const DevModel*)p;
  const DMHead* h = (const DMHead*)d->model.data();
  uint32_t* d_m = nullptr;
  float *d_s = nullptr, *d_o = nullptr;
  const size_t smem = ((size_t)h->hot_words + h->scr_words) * 4, sb = (size_t)ncase * h->scr_words * 4;
  const size_t ob = stage == DEVSIM_TOUCH ? (size_t)ncase * h->nsensor * 4 : 0;
  g_err[0] = 0;
  DEVSIM_OK(cudaMalloc(&d_m, d->model.size() * 4));
  DEVSIM_OK(cudaMalloc(&d_s, sb));
  if (ob) DEVSIM_OK(cudaMalloc(&d_o, ob));
  DEVSIM_OK(cudaMemcpy(d_m, d->model.data(), d->model.size() * 4, cudaMemcpyHostToDevice));
  DEVSIM_OK(cudaMemcpy(d_s, scratch, sb, cudaMemcpyHostToDevice));
  {
    int matched = 0;
#define DEVSIM_STAGE(V)                                                                                                      \
    if (nvp == V) {                                                                                                          \
      matched = 1;                                                                                                           \
      DEVSIM_OK(cudaFuncSetAttribute(stage_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));              \
      stage_kernel<V><<<ncase, 32, smem>>>(d_m, stage, d_s, d_o);                                                            \
    }
#if defined(B200_WIDE)
    DEVSIM_STAGE(36)
#elif defined(B200_KITCHEN)
    DEVSIM_STAGE(31)
#else
    DEVSIM_STAGE(14) DEVSIM_STAGE(15) DEVSIM_STAGE(21) DEVSIM_STAGE(22) DEVSIM_STAGE(30)
#endif
#undef DEVSIM_STAGE
    if (!matched) { snprintf(g_err, sizeof(g_err), "devsim_stage: NVP %d is not instantiated in this library", nvp); rc = -1; goto done; }
  }
  DEVSIM_OK(cudaGetLastError());
  DEVSIM_OK(cudaDeviceSynchronize());
  DEVSIM_OK(cudaMemcpy(scratch, d_s, sb, cudaMemcpyDeviceToHost));
  if (ob) DEVSIM_OK(cudaMemcpy(out, d_o, ob, cudaMemcpyDeviceToHost));
done:
  cudaFree(d_m); cudaFree(d_s); cudaFree(d_o);
  return rc;
}
}
