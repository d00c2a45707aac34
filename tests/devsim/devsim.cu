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
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../gymnasium_robotics_b200/csrc/fetch_task.cuh"

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
