// harness.cu — routine-level test harness for the engine's dense linear algebra (tests/test_dense_algebra.py).
//
// TEST INFRASTRUCTURE ONLY. This translation unit includes the kernel source itself, so the routines under test are the
// ones the engine runs, compiled the way it ships (nvcc with __graft_entry__.NVCC_FLAGS) or, with -DB200MJ_CPU_EMU, the
// way the CPU emulation compiles them (tests/emu/cuda_emu.h). Nothing under dm_control_b200/ loads it.
//
// One warp runs one case. The host packs each case as an image of its shared-memory workspace (matrices, vectors,
// integer lists, sentinels) plus a row of integer parameters; the warp copies its image into its slice of dynamic shared
// memory, calls the routine on pointers into that slice, and copies the whole slice back, so the caller also sees
// whatever the routine wrote where it should not have.
#include "../../dm_control_b200/csrc/b200mj.cu"

enum { OP_CHOL = 1, OP_MULTI = 2, OP_TN = 3, OP_PROD = 4, OP_RSQRT = 5 };
// parameter row of one case (NPAR ints); offsets are in doubles from the start of the case's image, -1 = none
enum { P_OP, P_N, P_A, P_L, P_DINV, P_B, P_Y, P_FWIN, P_FWOUT, P_BKIN, P_BKOUT, P_K, P_LD, P_XB, P_XX, P_J, P_SD, P_ALIST,
       P_NACT, P_COLBUF, P_NEG, P_V, P_OUT, P_OUT2, P_NROWS, NPAR = 32 };

#define AT(p) (P[p] >= 0 ? ws + P[p] : nullptr)

template <int N>
__device__ void run_tn(const int* P, double* ws, int lane) {
  tn_factor<N>(AT(P_A), AT(P_L), AT(P_DINV), lane, AT(P_B), AT(P_Y), AT(P_J), AT(P_SD),
               reinterpret_cast<const int*>(AT(P_ALIST)), P[P_NACT], AT(P_COLBUF));
  if (P[P_BKIN] >= 0) tn_back<N>(AT(P_L), AT(P_DINV), AT(P_BKIN), AT(P_BKOUT), lane, P[P_NEG]);
  if (P[P_FWIN] >= 0) tn_forward<N>(AT(P_L), AT(P_DINV), AT(P_FWIN), AT(P_FWOUT), lane);
}

template <int N>
__device__ void run_tn_prod(const int* P, double* ws, int lane) {
  constexpr int LD = N | 1;
  if (lane < N) ws[P[P_OUT] + lane] = tn_symv_row<N>(AT(P_A), AT(P_V), lane);
  if (lane < P[P_NROWS]) ws[P[P_OUT2] + lane] = tn_dot_row<N>(AT(P_J) + lane * LD, AT(P_V));
}

__global__ void alg_kernel(const int* params, const double* in, double* out, int stride, int ncases) {
  B200MJ_DYN_SMEM
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, c = blockIdx.x * (blockDim.x >> 5) + w;
  if (c >= ncases) return;
  const int* P = params + (size_t)c * NPAR;
  double* ws = smem + (size_t)w * stride;
  for (int i = lane; i < stride; i += 32) ws[i] = in[(size_t)c * stride + i];
  __syncwarp();
  const int n = P[P_N];
  switch (P[P_OP]) {
    case OP_CHOL:
      chol_factor(AT(P_A), AT(P_L), AT(P_DINV), n, lane, AT(P_B), AT(P_Y));
      if (P[P_FWIN] >= 0) chol_forward(AT(P_L), AT(P_DINV), AT(P_FWIN), AT(P_FWOUT), n, lane);
      if (P[P_BKIN] >= 0) chol_back(AT(P_L), AT(P_DINV), AT(P_BKIN), AT(P_BKOUT), n, lane);
      break;
    case OP_MULTI:
      chol_factor(AT(P_A), AT(P_L), AT(P_DINV), n, lane, nullptr, nullptr);
      chol_solve_multi(AT(P_L), AT(P_DINV), n, AT(P_B), AT(P_Y), P[P_LD], P[P_K], lane, AT(P_XB), AT(P_XX));
      break;
    case OP_TN:
      switch (n) {
#define TN_CASE(NV) case NV: run_tn<NV>(P, ws, lane); break;
        B200MJ_NV_LIST(TN_CASE)
#undef TN_CASE
      }
      break;
    case OP_PROD:
      if (P[P_LD] == 0) {          // compile-time size
        switch (n) {
#define TN_CASE(NV) case NV: run_tn_prod<NV>(P, ws, lane); break;
          B200MJ_NV_LIST(TN_CASE)
#undef TN_CASE
        }
      } else {
        FOR_LANES(i, n) ws[P[P_OUT] + i] = symv_row(AT(P_A), AT(P_V), n, i);
        FOR_LANES(r, P[P_NROWS]) ws[P[P_OUT2] + r] = dot_rows(AT(P_J) + r * P[P_LD], AT(P_V), n);
      }
      break;
    case OP_RSQRT:
      FOR_LANES(i, n) ws[P[P_OUT] + i] = pos_rsqrt(ws[P[P_V] + i]);
      break;
  }
  __syncwarp();
  for (int i = lane; i < stride; i += 32) out[(size_t)c * stride + i] = ws[i];
}
#undef AT

// params [ncases][NPAR], in / out [ncases][stride] doubles: device pointers (host pointers under the emulation).
// Returns 0, or the CUDA error of the launch.
extern "C" int alg_run(const int* params, const double* in, double* out, int stride, int ncases, int warps) {
  const size_t smem = (size_t)warps * stride * sizeof(double);
  if (smem > SMEM_MAX || stride % 2) return -1;
  cudaFuncSetAttribute(alg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  B200MJ_LAUNCH(alg_kernel, (ncases + warps - 1) / warps, 32 * warps, smem, (cudaStream_t)0, params, in, out, stride, ncases);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)0);
  return (int)e;
}

extern "C" int alg_npar() { return NPAR; }
