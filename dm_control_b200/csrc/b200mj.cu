// b200mj.cu — H100 (sm_90a) batched forward-dynamics engine: ONE WARP PER ENVIRONMENT.
//
// Stands where the un-vendored `mujoco.mj_step / mj_step1 / mj_step2 / mj_forward` calls stand in
// dm_control/mujoco/engine.py:147-176,306-343. Stage list: SURVEY.md §8a. C ABI: include/b200mj.h.
//
// Layout: batched state is row-major [batch, n] in HBM, so the warp that owns environment e reads its
// row with consecutive lanes on consecutive doubles (coalesced). Everything between the load of
// (qpos, qvel, act, qacc_warmstart, ctrl) and the store of the new state + observation-contract outputs
// lives in a per-warp shared-memory workspace (struct Lay) — `nstep` physics steps are fused into one
// launch. Lanes parallelise over bodies of a tree level, dofs, geom pairs or constraint rows; reductions
// are fixed-order xor-shuffle trees so results are bit-reproducible run to run.
//
// No CPU fallback exists: if this library is missing the Python facade raises.

#ifdef B200MJ_CPU_EMU
// tests/emu/cuda_emu.h: lock-step CPU emulation of the warp / CTA primitives so that the `-m "not gpu"` tests can run
// THIS source for logic errors without a GPU. Test infrastructure only: the product library is built by nvcc without
// this macro, and nothing in dm_control_b200/ ever loads the emulation build.
#include "cuda_emu.h"
#define B200MJ_DYN_SMEM        // cuda_emu.h defines `smem` at namespace scope (a block-scope extern of a thread_local trips g++ in templates)
#else
#include <cuda_runtime.h>
#define B200MJ_DYN_SMEM extern __shared__ double smem[];
#define B200MJ_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

#include "../../include/b200mj.h"
#include "../../include/b200mj_model_fields.h"
#include "../../include/b200mj_convex.h"

#define FULL 0xffffffffu
#define FOR_LANES(i, n) _Pragma("unroll 1") for (int i = lane; i < (n); i += 32)
// dynamic shared memory one CTA may opt into on sm_90 (228 KB per SM, 1 KB of which is reserved per CTA)
#define SMEM_MAX (227 * 1024)

// ------------------------------------------------------------------------------------------------
// device model view + workspace layout
// ------------------------------------------------------------------------------------------------
struct DevModel {
#define DECL_I(name) const int* name;
#define DECL_R(name) const double* name;
  B200MJ_MODEL_FIELDS(DECL_I, DECL_R)
#undef DECL_I
#undef DECL_R
  int nq, nv, nu, na, nbody, njnt, ngeom, nsite, ntendon, neq, nsensor, nsensordata, npair, nlevel, nconmax, njmax;
  // actuator moments by dof (CSR, built by b200mj_model_create): joint and fixed-tendon transmissions have constant
  // moment arms, so qfrc_actuator[i] = sum over dof_act_id[dof_act_adr[i] .. dof_act_adr[i+1]) of coef * force
  const int* dof_act_adr; const int* dof_act_id; const double* dof_act_coef;
  // per-environment geoms (b200mj_model_set_variable_geoms): geom_varid[g] = slot k of io.var_geom_pos / var_geom_size, or -1
  const int* geom_varid; int nvargeom;
  int ldv;          // padded row length of nv-wide matrices (odd => conflict-free column walks)
  int integrator, iterations, ls_iterations, disableflags, solver;
  int any_damping, acc_sensors;
  int cvx_warp;     // convex pairs resolved by the whole warp (cvx_pair_warp; B200MJ_CVX_WARP=0: one pair per lane, cvx_pair)
  double timestep, gravity[3], tolerance, ls_tolerance, impratio, meaninertia;
};

// offsets (in doubles) into one environment's workspace
struct Lay {
  int total;                             // doubles per environment
  int qpos, qvel, act, ctrl, qaccws, actdot;
  int xpos, xquat, xmat, xipos, xanchor, xaxis, gxpos, gxmat, scom, slinvel;
  int cinert, crb, cdof, cdofdot, cvel, cacc, cfrc, cfrcext;
  int tenlen, tenJ, actforce;
  int M, H, dinv;
  int J, efcD, efcSD, aref, jar, jv, force, eqflag, actlist;
  int bias, passive, qfact, smooth, qaccs, qacc, qcon, Ma, grad, search, Mv, tmpv;
  int con;                               // contact records, 16 doubles each
  int cq;                                // collision: queue of candidate pairs that passed the bounding tests (64 ints)
  int gcache, grb, gmg, gty;             // collision, models with many candidate pairs per geom: per-geom bounding radius / margin / type staged once per step
  int rk;                                // RK4 scratch: X0q, X0v, X0a, accv, acca, accd
  int sens;                              // sensordata staging
  int vold;                              // last-step acceleration kernel: qvel before integration (for rne_post_constraint)
  int colbuf;                            // compile-time-size algebra: column broadcast buffer (TN_COLBUF_DOUBLES)
  int pgsA, pgsX, pgsB;                  // PGS solver (fused kernel only): A = J M^-1 J' + R [nj x nj], M^-1 J' [nj x ld], b [nj]
  // dual form of the Newton direction (runtime-size acceleration kernels, nv >= 32, row buckets of at most 32 rows):
  // dV = rows of M^-1 J' [rows x ld]; dS = scratch [rows^2 + tri(rows) + 3 rows] for A = J M^-1 J', the factor of the
  // active block R + A_aa and its right-hand side (aliases H, which is free between chol(M) and the Euler step)
  int dual, dV, dS, drows;
  int jalias;                            // dual form, small buckets: the workspace copy of J lives in H's storage (free once J M^-1 is there); J M^-1 is computed from the handover row
  int mglobal;                           // runtime-size acceleration kernels, nv >= 32: M stays in the handover row (no workspace copy)
};

// Per-environment row of the L2-resident handover buffer between the split position and acceleration kernels
// (offsets in doubles).
struct Hand { int M, J, efcD, aref, eqflag, bias, passive, tenlen, tenJ, counts, total; };
// Second row, written only in the last physics step: what the acceleration-stage sensors need from the position stage.
// X(field, doubles), with the model `m` and the contact count `ncon` in scope. The struct, its layout, the position
// kernel's dump, the acceleration kernel's reload and the sensor-carrying acceleration workspace all expand this list.
#define HAND2_FIELDS(X) X(xpos, 3 * m.nbody) X(xquat, 4 * m.nbody) X(xmat, 9 * m.nbody) X(xipos, 3 * m.nbody) \
  X(scom, 3 * m.nbody) X(cinert, 10 * m.nbody) X(cdof, 6 * m.nv) X(cdofdot, 6 * m.nv) X(cvel, 6 * m.nbody) X(con, ncon * CON_STRIDE)
#define HAND2_DECL(f, n) int f;
struct Hand2 { HAND2_FIELDS(HAND2_DECL) int total; };
#undef HAND2_DECL
// the handover buffers of the split path and their row layouts: rows [hand_batch + SHADOW_ROWS][H.total], rows2 likewise
struct Handover { Hand H; Hand2 H2; double* rows; double* rows2; };

// Row-bucket compaction (split path): the position kernel appends every environment to the list of its row-count
// bucket (count[b] = entries so far, list[b * cap ..]); the acceleration launch of a bucket then runs dense CTAs of
// several warps over that list instead of one single-warp CTA per environment of which most exit at once.
struct Compact { int* count; int* list; int cap; int nbucket; int rows_cap[4]; int shadow_row; };
#define SHADOW_ROWS 16   // private handover rows for the shadow warps of a launch's last CTA: [2 groups][8 warps]

struct b200mj_model {
  DevModel dm;
  Lay lay;
  Lay lay_pos;                // compact workspace of the split position kernels
  // acceleration kernel: row-count buckets (workspace sized for rows_cap[b] constraint rows), plain and
  // sensor-carrying (last physics step of a fused step) variants
  int nbucket; int rows_cap[4]; Lay lay_acc_b[4], lay_accs_b[4]; size_t smem_acc_b[4], smem_accs_b[4];
  Handover ho; int hand_batch;
  // environment groups x row buckets run on their own streams (independent work: hides each launch's tail)
  cudaStream_t gmain[2], gaux[2][4]; cudaEvent_t ev_fork, ev_join[2], ev_pos[2], ev_acc[2][4]; int streams_ok;
  int convex_pairs;                // some candidate pair needs cvx_capsule_box / cvx_pair (else: primitive-only position kernels)
  int* d_bcount; int* d_blist;     // compaction: counters [2 groups][4 buckets], lists [2 groups][4 buckets][hand_batch]
  // the trailing mj_step1 of the last split-path step left a complete handover for this (io, batch): see B200MJ_STEP_REUSE_POS
  const double* reuse_qpos; int reuse_batch; int reuse_flags; int reuse_ok; int reuse_has_dump;
  int epb_pos, pos_big;
  size_t smem_pos;
  int* d_idata;
  double* d_rdata;
  int* d_xi; double* d_xr;      // derived tables (dof_act_*)
  int* d_varid;                 // geom -> variable-geom slot
  int envs_per_block;
  size_t smem_per_env;
  int tn_nv;                  // nv when a compile-time-size acceleration kernel exists for this model, else 0
  int nkey;
  struct {                    // environment overrides for tests (read_test_hooks)
    int tn, split, dual_min_nv, buckets[3], nbuckets, epb_pos, acc_warps, envs_per_block;
  } hooks;
};

// ------------------------------------------------------------------------------------------------
// small device math
// ------------------------------------------------------------------------------------------------
// a * b + c with one rounding, written out where it matters for speed. The library is built with -fmad=false: the
// compiler's own contraction of a * b + c depends on the kernel a routine is inlined into, so the fused and the split
// kernels would round the same routine differently. Spelled out, every kernel computes it the same way.
#ifdef B200MJ_CPU_EMU
#define MADD(a, b, c) ((a) * (b) + (c))
#else
#define MADD(a, b, c) __fma_rn((a), (b), (c))
#endif
__device__ __forceinline__ double dot3(const double* a, const double* b) { return MADD(a[2], b[2], MADD(a[1], b[1], a[0]*b[0])); }
__device__ __forceinline__ void cross3(double* r, const double* a, const double* b) {
  double x = MADD(a[1], b[2], -(a[2]*b[1])), y = MADD(a[2], b[0], -(a[0]*b[2])), z = MADD(a[0], b[1], -(a[1]*b[0]));
  r[0] = x; r[1] = y; r[2] = z;
}
__device__ __forceinline__ double norm3(const double* a) { return sqrt(dot3(a, a)); }
__device__ __forceinline__ double normalize3(double* a) {
  double n = norm3(a);
  if (n < BMJ_MINVAL) { a[0] = 1; a[1] = 0; a[2] = 0; } else { a[0] /= n; a[1] /= n; a[2] /= n; }
  return n;
}
__device__ __forceinline__ void mul_quat(double* r, const double* a, const double* b) {
  double w = MADD(-a[3], b[3], MADD(-a[2], b[2], MADD(-a[1], b[1], a[0]*b[0])));
  double x = MADD(-a[3], b[2], MADD(a[2], b[3], MADD(a[1], b[0], a[0]*b[1])));
  double y = MADD(a[3], b[1], MADD(a[2], b[0], MADD(-a[1], b[3], a[0]*b[2])));
  double z = MADD(a[3], b[0], MADD(-a[2], b[1], MADD(a[1], b[2], a[0]*b[3])));
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
// mju_normalize4 semantics: a quaternion whose norm is already within mjMINVAL of 1 is left untouched, which makes
// the operation idempotent — mj_kinematics normalises qpos in place at every position stage, and step(n) must stay
// bit-identical to n x step() (engine_test.py:627-663) although the latter passes through one more position stage
// per call.
__device__ __forceinline__ void normalize4(double* q) {
  double n = sqrt(q[0]*q[0] + q[1]*q[1] + q[2]*q[2] + q[3]*q[3]);
  if (n < BMJ_MINVAL) { q[0] = 1; q[1] = q[2] = q[3] = 0; }
  else if (fabs(n - 1) > BMJ_MINVAL) { double inv = 1 / n; q[0] *= inv; q[1] *= inv; q[2] *= inv; q[3] *= inv; }
}
__device__ __forceinline__ void quat2mat(double* m, const double* q) {
  double q00 = q[0]*q[0], q11 = q[1]*q[1], q22 = q[2]*q[2], q33 = q[3]*q[3];
  m[0] = q00 + q11 - q22 - q33; m[4] = q00 - q11 + q22 - q33; m[8] = q00 - q11 - q22 + q33;
  m[1] = 2*(q[1]*q[2] - q[0]*q[3]); m[2] = 2*(q[1]*q[3] + q[0]*q[2]);
  m[3] = 2*(q[1]*q[2] + q[0]*q[3]); m[5] = 2*(q[2]*q[3] - q[0]*q[1]);
  m[6] = 2*(q[1]*q[3] - q[0]*q[2]); m[7] = 2*(q[2]*q[3] + q[0]*q[1]);
}
__device__ __forceinline__ void mat_vec(double* r, const double* m, const double* v) {
  double x = MADD(m[2], v[2], MADD(m[1], v[1], m[0]*v[0])), y = MADD(m[5], v[2], MADD(m[4], v[1], m[3]*v[0])),
         z = MADD(m[8], v[2], MADD(m[7], v[1], m[6]*v[0]));
  r[0] = x; r[1] = y; r[2] = z;
}
__device__ __forceinline__ void matT_vec(double* r, const double* m, const double* v) {
  double x = MADD(m[6], v[2], MADD(m[3], v[1], m[0]*v[0])), y = MADD(m[7], v[2], MADD(m[4], v[1], m[1]*v[0])),
         z = MADD(m[8], v[2], MADD(m[5], v[1], m[2]*v[0]));
  r[0] = x; r[1] = y; r[2] = z;
}
__device__ __forceinline__ void rot_vec_quat(double* r, const double* v, const double* q) {
  double m[9]; quat2mat(m, q); mat_vec(r, m, v);
}
__device__ __forceinline__ void axis_angle2quat(double* q, const double* axis, double angle) {
  if (angle == 0) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  double s, c; sincos(angle * 0.5, &s, &c);
  q[0] = c; q[1] = axis[0]*s; q[2] = axis[1]*s; q[3] = axis[2]*s;
}
__device__ __forceinline__ void quat_integrate(double* q, const double* w, double h) {
  double ax[3] = {w[0], w[1], w[2]};
  double n = norm3(ax);
  if (n < BMJ_MINVAL) return;
  ax[0] /= n; ax[1] /= n; ax[2] /= n;
  double dq[4], r[4];
  axis_angle2quat(dq, ax, h * n);
  normalize4(q);
  mul_quat(r, q, dq);
  q[0] = r[0]; q[1] = r[1]; q[2] = r[2]; q[3] = r[3];
}
__device__ __forceinline__ void mul_inert_vec(double* r, const double* i, const double* v) {
  r[0] = MADD(i[7], v[5], MADD(-i[8], v[4], MADD(i[4], v[2], MADD(i[3], v[1], i[0]*v[0]))));
  r[1] = MADD(-i[6], v[5], MADD(i[8], v[3], MADD(i[5], v[2], MADD(i[1], v[1], i[3]*v[0]))));
  r[2] = MADD(i[6], v[4], MADD(-i[7], v[3], MADD(i[2], v[2], MADD(i[5], v[1], i[4]*v[0]))));
  r[3] = MADD(i[9], v[3], MADD(-i[7], v[2], i[8]*v[1]));
  r[4] = MADD(i[9], v[4], MADD(-i[8], v[0], i[6]*v[2]));
  r[5] = MADD(i[9], v[5], MADD(-i[6], v[1], i[7]*v[0]));
}
__device__ __forceinline__ void cross_motion(double* r, const double* vel, const double* v) {
  double a[3], b[3], c[3];
  cross3(a, vel, v); cross3(b, vel, v + 3); cross3(c, vel + 3, v);
  r[0] = a[0]; r[1] = a[1]; r[2] = a[2]; r[3] = b[0] + c[0]; r[4] = b[1] + c[1]; r[5] = b[2] + c[2];
}
__device__ __forceinline__ void cross_force(double* r, const double* vel, const double* f) {
  double a[3], b[3], c[3];
  cross3(a, vel, f); cross3(b, vel + 3, f + 3); cross3(c, vel, f + 3);
  r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2]; r[3] = c[0]; r[4] = c[1]; r[5] = c[2];
}
__device__ __forceinline__ double clampd(double x, double lo, double hi) { return x < lo ? lo : (x > hi ? hi : x); }
__device__ __forceinline__ bool bad_value(double x) { return isnan(x) || x > BMJ_MAXVAL || x < -BMJ_MAXVAL; }

__device__ __noinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
// exclusive prefix sum over lanes; *total = sum over all lanes
__device__ __forceinline__ int warp_excl_scan(int v, int lane, int* total) {
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(FULL, x, o); if (lane >= o) x += y; }
  *total = __shfl_sync(FULL, x, 31);
  return x - v;
}

struct Ctx {
  const DevModel& m; const Lay& L; double* ws; int lane; int disableflags;
  int newton_sync;      // every warp of the CTA takes the same number of Newton trips (multi-warp acceleration CTAs)
  // where the position/velocity stage deposits what the acceleration stage consumes: the workspace itself in the
  // fused kernel, this environment's row of the L2-resident handover buffer in the split position kernel
  double *pM, *pJ, *pD, *pAref, *pBias, *pPassive; int* pEq; double* stage;
  const double* Jg;     // acceleration stage: this environment's constraint Jacobian in the handover row (L.jalias)
  const double* Mc;     // acceleration stage: the joint-space inertia, read-only — the workspace copy, or (L.mglobal) the handover row in L2
  int env; const double* var_pos; const double* var_size;      // per-environment geoms (set_env)
  __device__ void set_env(int e, const b200mj_io& io) { env = e; var_pos = io.var_geom_pos; var_size = io.var_geom_size; }
  __device__ Ctx(const DevModel& m_, const Lay& L_, double* ws_, int lane_, int df, int ns) : m(m_), L(L_), ws(ws_), lane(lane_), disableflags(df), newton_sync(ns), env(0), var_pos(nullptr), var_size(nullptr) {
    pM = ws_ + L_.M; pJ = ws_ + L_.J; pD = ws_ + L_.efcD; pAref = ws_ + L_.aref; pBias = ws_ + L_.bias; pPassive = ws_ + L_.passive;
    pEq = reinterpret_cast<int*>(ws_ + L_.eqflag); stage = ws_ + L_.J; Mc = pM; Jg = pJ;
  }
};
#define W(name) (c.ws + c.L.name)

// ------------------------------------------------------------------------------------------------
// dense Cholesky in the workspace: A (n x n, row stride ld) -> lower factor Lm, same stride
// ------------------------------------------------------------------------------------------------
// coalesced copy between a handover row in global memory and the workspace: 16-byte accesses, four in flight per
// lane (a rolled 8-byte loop would serialise one L2/DRAM latency per element). Regions are 16-byte aligned and padded
// to an even number of doubles by the layout builder.
__device__ __forceinline__ void copy_row(double* dst, const double* src, int n, int lane) {
  const int n2 = (n + 1) >> 1;
  double2* d2 = reinterpret_cast<double2*>(dst); const double2* s2 = reinterpret_cast<const double2*>(src);
  int i = lane;
  _Pragma("unroll 1") for (; i + 96 < n2; i += 128) {
    double2 a = s2[i], b = s2[i + 32], c = s2[i + 64], d = s2[i + 96];
    d2[i] = a; d2[i + 32] = b; d2[i + 64] = c; d2[i + 96] = d;
  }
  _Pragma("unroll 1") for (; i < n2; i += 32) d2[i] = s2[i];
}

// dot product of two workspace rows with four independent accumulators (breaks the DFMA dependency chain)
__device__ __forceinline__ double dot_rows(const double* a, const double* b, int n) {
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
  int k = 0;
  _Pragma("unroll 1") for (; k + 4 <= n; k += 4) { s0 = MADD(a[k], b[k], s0); s1 = MADD(a[k + 1], b[k + 1], s1); s2 = MADD(a[k + 2], b[k + 2], s2); s3 = MADD(a[k + 3], b[k + 3], s3); }
  _Pragma("unroll 1") for (; k < n; k++) s0 = MADD(a[k], b[k], s0);
  return (s0 + s1) + (s2 + s3);
}

// Symmetric nv x nv matrices (M, the Newton Hessian, their Cholesky factors) are stored as PACKED lower triangles:
// element (i, j <= i) at tri(i) + j. Rows stay contiguous (what the left-looking factorisation and the triangular
// solves walk), lane-strided row starts tri(lane) hit distinct banks (triangular numbers are a permutation mod 2^k),
// and two packed triangles cost 0.52 of one dense matrix: the acceleration kernels hold 16 instead of 11
// environments per SM.
__device__ __forceinline__ int tri(int i) { return (i * (i + 1)) >> 1; }

// row i of (symmetric S) * v from the packed lower triangle; accumulation order identical to dot_rows
__device__ __forceinline__ double symv_row(const double* Sp, const double* v, int n, int i) {
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
  const double* Si = Sp + tri(i);        // row i, columns <= i
  const double* Sc = Sp + i;             // column i below the diagonal: Sc[tri(k)], k > i
  int k = 0, tk = 0;
  _Pragma("unroll 1") for (; k + 4 <= n; k += 4) {
    const int t1 = tk + k + 1, t2 = t1 + k + 2, t3 = t2 + k + 3;
    s0 = MADD(k <= i ? Si[k] : Sc[tk], v[k], s0);
    s1 = MADD(k + 1 <= i ? Si[k + 1] : Sc[t1], v[k + 1], s1);
    s2 = MADD(k + 2 <= i ? Si[k + 2] : Sc[t2], v[k + 2], s2);
    s3 = MADD(k + 3 <= i ? Si[k + 3] : Sc[t3], v[k + 3], s3);
    tk = t3 + k + 4;
  }
  _Pragma("unroll 1") for (; k < n; k++) { s0 = MADD(k <= i ? Si[k] : Sc[tk], v[k], s0); tk += k + 1; }
  return (s0 + s1) + (s2 + s3);
}

// forward substitution L y = b (L packed, n <= 64); b and y may alias
__device__ __noinline__ void chol_forward(const double* Lm, const double* dinv, const double* b, double* y, int n, int lane) {
  if (n <= 32) {
    double xi = lane < n ? b[lane] : 0.0;
    const double* Li = Lm + tri(lane);
    _Pragma("unroll 1") for (int j = 0; j < n; j++) {
      double yj = __shfl_sync(FULL, xi, j) * dinv[j];
      if (lane == j) xi = yj; else if (lane > j && lane < n) xi = MADD(-Li[j], yj, xi);
    }
    __syncwarp();
    if (lane < n) y[lane] = xi;
    __syncwarp();
    return;
  }
  const int i1 = lane + 32;
  const double* L0 = Lm + tri(lane); const double* L1 = Lm + tri(i1);
  double x0 = lane < n ? b[lane] : 0.0, x1 = i1 < n ? b[i1] : 0.0;
  _Pragma("unroll 1") for (int j = 0; j < n; j++) {
    double v = __shfl_sync(FULL, j < 32 ? x0 : x1, j & 31);
    double yj = v * dinv[j];
    if (j < 32) { if (lane == j) x0 = yj; else if (lane > j && lane < n) x0 -= L0[j] * yj; if (i1 < n) x1 -= L1[j] * yj; }
    else { if (i1 == j) x1 = yj; else if (i1 > j && i1 < n) x1 -= L1[j] * yj; }
  }
  __syncwarp();
  if (lane < n) y[lane] = x0;
  if (i1 < n) y[i1] = x1;
  __syncwarp();
}

// backward substitution L^T x = y (L packed, n <= 64); y and x may alias
__device__ __noinline__ void chol_back(const double* Lm, const double* dinv, const double* y, double* x, int n, int lane) {
  if (n <= 32) {
    double xi = lane < n ? y[lane] : 0.0;
    int tj = tri(n - 1);
    _Pragma("unroll 1") for (int j = n - 1; j >= 0; j--) {
      double xj = __shfl_sync(FULL, xi, j) * dinv[j];
      if (lane == j) xi = xj; else if (lane < j) xi = MADD(-Lm[tj + lane], xj, xi);
      tj -= j;
    }
    __syncwarp();
    if (lane < n) x[lane] = xi;
    __syncwarp();
    return;
  }
  const int i1 = lane + 32;
  double x0 = lane < n ? y[lane] : 0.0, x1 = i1 < n ? y[i1] : 0.0;
  int tj = tri(n - 1);
  _Pragma("unroll 1") for (int j = n - 1; j >= 0; j--) {
    double v = __shfl_sync(FULL, j < 32 ? x0 : x1, j & 31);
    double xj = v * dinv[j];
    if (j < 32) { if (lane == j) x0 = xj; else if (lane < j) x0 -= Lm[tj + lane] * xj; }
    else { if (i1 == j) x1 = xj; else if (i1 < j) x1 -= Lm[tj + i1] * xj; if (lane < n) x0 -= Lm[tj + lane] * xj; }
    tj -= j;
  }
  __syncwarp();
  if (lane < n) x[lane] = x0;
  if (i1 < n) x[i1] = x1;
  __syncwarp();
}

// Cholesky factor of a packed symmetric matrix, A -> Lm (may alias), dinv[j] = 1 / L[j][j] (neither the factor nor
// the triangular solves divide). When a right-hand side b is given, y = L^-1 b comes out as well (b, y may alias).
//
// n < 32: left-looking by blocks of four columns, one row per lane. The part of the four dot products that lies
// left of the block shares its loads of the lane's own row (5 loads per 4 multiply-adds instead of 8), the four
// accumulators are the independent chains that hide the DFMA latency, and inside the block the new columns stay in
// registers: pivots and the 6 cross terms travel by shuffle, so there is one shared-memory round trip per block
// instead of one per column. The right-hand side rides along as row n of the matrix on the spare lane n — the
// forward substitution costs no extra pass.
__device__ __noinline__ void chol_factor(const double* A, double* Lm, double* dinv, int n, int lane, const double* b, double* y) {
  if (n < 32) {
    const bool isrow = lane < n, isrhs = (b != nullptr) && lane == n, live = isrow || isrhs;
    const int ti = tri(lane);
    const double* Ai = isrow ? A + ti : (isrhs ? b : A);   // this lane's row of A (read at the block's columns)
    double* Li = isrow ? Lm + ti : (isrhs ? y : Lm);       // this lane's row of L (idle lanes read row 0, never write)
    int tj0 = 0;                                           // tri(j0)
    _Pragma("unroll 1") for (int j0 = 0; j0 < n; j0 += 4) {
      const int j1 = min(j0 + 1, n - 1), j2 = min(j0 + 2, n - 1), j3 = min(j0 + 3, n - 1);   // tail block: clamp
      const double* r0 = Lm + tj0; const double* r1 = Lm + tri(j1); const double* r2 = Lm + tri(j2); const double* r3 = Lm + tri(j3);
      double t0 = 0, t1 = 0, t2 = 0, t3 = 0;
      _Pragma("unroll 1") for (int k = 0; k < j0; k += 4) {      // j0 is a multiple of 4
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const double a = Li[k + q];
          t0 = MADD(a, r0[k + q], t0); t1 = MADD(a, r1[k + q], t1); t2 = MADD(a, r2[k + q], t2); t3 = MADD(a, r3[k + q], t3);
        }
      }
      const bool on0 = live && lane >= j0, on1 = live && lane >= j0 + 1 && j0 + 1 < n,
                 on2 = live && lane >= j0 + 2 && j0 + 2 < n, on3 = live && lane >= j0 + 3 && j0 + 3 < n;
      t0 = on0 ? Ai[j0] - t0 : 0.0; t1 = on1 ? Ai[j0 + 1] - t1 : 0.0; t2 = on2 ? Ai[j0 + 2] - t2 : 0.0; t3 = on3 ? Ai[j0 + 3] - t3 : 0.0;
      double l0, l1 = 0, l2 = 0;
      {
        double piv = __shfl_sync(FULL, t0, j0);
        if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
        const double inv = rsqrt(piv);
        l0 = t0 * inv;
        if (lane == j0) { Li[j0] = piv * inv; dinv[j0] = inv; } else if (on0) Li[j0] = l0;
      }
      if (j0 + 1 < n) {
        t1 -= l0 * __shfl_sync(FULL, l0, j0 + 1);
        double piv = __shfl_sync(FULL, t1, j0 + 1);
        if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
        const double inv = rsqrt(piv);
        l1 = t1 * inv;
        if (lane == j0 + 1) { Li[j0 + 1] = piv * inv; dinv[j0 + 1] = inv; } else if (on1) Li[j0 + 1] = l1;
      }
      if (j0 + 2 < n) {
        t2 -= l0 * __shfl_sync(FULL, l0, j0 + 2);
        t2 -= l1 * __shfl_sync(FULL, l1, j0 + 2);
        double piv = __shfl_sync(FULL, t2, j0 + 2);
        if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
        const double inv = rsqrt(piv);
        l2 = t2 * inv;
        if (lane == j0 + 2) { Li[j0 + 2] = piv * inv; dinv[j0 + 2] = inv; } else if (on2) Li[j0 + 2] = l2;
      }
      if (j0 + 3 < n) {
        t3 -= l0 * __shfl_sync(FULL, l0, j0 + 3);
        t3 -= l1 * __shfl_sync(FULL, l1, j0 + 3);
        t3 -= l2 * __shfl_sync(FULL, l2, j0 + 3);
        double piv = __shfl_sync(FULL, t3, j0 + 3);
        if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
        const double inv = rsqrt(piv);
        if (lane == j0 + 3) { Li[j0 + 3] = piv * inv; dinv[j0 + 3] = inv; } else if (on3) Li[j0 + 3] = t3 * inv;
      }
      __syncwarp();
      tj0 += 4 * j0 + 10;      // tri(j0 + 4) - tri(j0)
    }
    return;
  }
  // n >= 32: two rows per lane (lane, lane + 32), left-looking by blocks of four columns like the path above: the part
  // of the eight dot products left of the block shares its loads (2 own-row + 4 pivot-row loads per 8 multiply-adds; one
  // column at a time with a dot product per row took 4 loads per 2), the eight accumulators are independent chains,
  // and inside the block pivots and cross terms travel by shuffle. Rows 0..31 are finished once the block start passes
  // 32: from there on only the second row of every lane is updated.
  const int i0 = lane, i1 = lane + 32, ti0 = tri(i0), ti1 = tri(i1);
  // the right-hand side rides along as row n (the second row of lane n - 32) when there is a spare row: y = L^-1 b for free
  const bool ride = b != nullptr && n < 64, isrhs = ride && i1 == n;
  const bool in1 = i1 < n || isrhs;
  const double* A0 = A + ti0; const double* A1 = isrhs ? b : (in1 ? A + ti1 : A);
  double* L0 = Lm + ti0; double* L1 = isrhs ? y : (in1 ? Lm + ti1 : Lm);      // idle second rows read row 0, never write
  int tj0 = 0;
  _Pragma("unroll 1") for (int j0 = 0; j0 < n; j0 += 4) {
    const int j1 = min(j0 + 1, n - 1), j2 = min(j0 + 2, n - 1), j3 = min(j0 + 3, n - 1);
    const double* r0 = Lm + tj0; const double* r1 = Lm + tri(j1); const double* r2 = Lm + tri(j2); const double* r3 = Lm + tri(j3);
    double s0 = 0, s1 = 0, s2 = 0, s3 = 0, u0 = 0, u1 = 0, u2 = 0, u3 = 0;      // s: row i0, u: row i1
    const bool low = j0 < 32;                                                   // warp-uniform
    if (low) {
      _Pragma("unroll 1") for (int k = 0; k < j0; k += 4) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const double b0 = r0[k + q], b1 = r1[k + q], b2 = r2[k + q], b3 = r3[k + q];
          const double a0 = L0[k + q], a1 = L1[k + q];      // rows above the block read finished entries: their sums are discarded below
          s0 += a0 * b0; s1 += a0 * b1; s2 += a0 * b2; s3 += a0 * b3;
          u0 += a1 * b0; u1 += a1 * b1; u2 += a1 * b2; u3 += a1 * b3;
        }
      }
    } else {
      _Pragma("unroll 1") for (int k = 0; k < j0; k += 4) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const double a1 = L1[k + q];
          u0 += a1 * r0[k + q]; u1 += a1 * r1[k + q]; u2 += a1 * r2[k + q]; u3 += a1 * r3[k + q];
        }
      }
    }
    // (row, column) pairs of this block that exist: row >= column, column < n
    const bool c1 = j0 + 1 < n, c2 = j0 + 2 < n, c3 = j0 + 3 < n;
    const bool p00 = low && i0 >= j0, p01 = low && c1 && i0 >= j0 + 1, p02 = low && c2 && i0 >= j0 + 2, p03 = low && c3 && i0 >= j0 + 3;
    const bool p10 = in1 && i1 >= j0, p11 = in1 && c1 && i1 >= j0 + 1, p12 = in1 && c2 && i1 >= j0 + 2, p13 = in1 && c3 && i1 >= j0 + 3;
    s0 = p00 ? A0[j0] - s0 : 0.0; s1 = p01 ? A0[j0 + 1] - s1 : 0.0; s2 = p02 ? A0[j0 + 2] - s2 : 0.0; s3 = p03 ? A0[j0 + 3] - s3 : 0.0;
    u0 = p10 ? A1[j0] - u0 : 0.0; u1 = p11 ? A1[j0 + 1] - u1 : 0.0; u2 = p12 ? A1[j0 + 2] - u2 : 0.0; u3 = p13 ? A1[j0 + 3] - u3 : 0.0;
    // value of row j of this block (rows j0..j0+3 live in the first rows of lanes j when j < 32, else in the second rows of lanes j - 32)
#define ROWVAL(sv, uv, j) __shfl_sync(FULL, low ? (sv) : (uv), (j) & 31)
    double m0, m1 = 0, m2 = 0, n0, n1 = 0, n2 = 0;      // scaled columns: m = first row, n = second row
    {
      double piv = ROWVAL(s0, u0, j0);
      if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
      const double inv = rsqrt(piv);
      m0 = s0 * inv; n0 = u0 * inv;
      if (p00) L0[j0] = (i0 == j0) ? piv * inv : m0;
      if (p10) L1[j0] = (i1 == j0) ? piv * inv : n0;
      if (lane == (j0 & 31)) dinv[j0] = inv;
    }
    if (c1) {
      const double x = ROWVAL(m0, n0, j0 + 1);
      s1 -= m0 * x; u1 -= n0 * x;
      double piv = ROWVAL(s1, u1, j0 + 1);
      if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
      const double inv = rsqrt(piv);
      m1 = s1 * inv; n1 = u1 * inv;
      if (p01) L0[j0 + 1] = (i0 == j0 + 1) ? piv * inv : m1;
      if (p11) L1[j0 + 1] = (i1 == j0 + 1) ? piv * inv : n1;
      if (lane == ((j0 + 1) & 31)) dinv[j0 + 1] = inv;
    }
    if (c2) {
      const double x0 = ROWVAL(m0, n0, j0 + 2), x1 = ROWVAL(m1, n1, j0 + 2);
      s2 -= m0 * x0; u2 -= n0 * x0; s2 -= m1 * x1; u2 -= n1 * x1;
      double piv = ROWVAL(s2, u2, j0 + 2);
      if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
      const double inv = rsqrt(piv);
      m2 = s2 * inv; n2 = u2 * inv;
      if (p02) L0[j0 + 2] = (i0 == j0 + 2) ? piv * inv : m2;
      if (p12) L1[j0 + 2] = (i1 == j0 + 2) ? piv * inv : n2;
      if (lane == ((j0 + 2) & 31)) dinv[j0 + 2] = inv;
    }
    if (c3) {
      const double x0 = ROWVAL(m0, n0, j0 + 3), x1 = ROWVAL(m1, n1, j0 + 3), x2 = ROWVAL(m2, n2, j0 + 3);
      s3 -= m0 * x0; u3 -= n0 * x0; s3 -= m1 * x1; u3 -= n1 * x1; s3 -= m2 * x2; u3 -= n2 * x2;
      double piv = ROWVAL(s3, u3, j0 + 3);
      if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
      const double inv = rsqrt(piv);
      if (p03) L0[j0 + 3] = (i0 == j0 + 3) ? piv * inv : s3 * inv;
      if (p13) L1[j0 + 3] = (i1 == j0 + 3) ? piv * inv : u3 * inv;
      if (lane == ((j0 + 3) & 31)) dinv[j0 + 3] = inv;
    }
#undef ROWVAL
    __syncwarp();
    tj0 += 4 * j0 + 10;
  }
  if (b && !ride) chol_forward(Lm, dinv, b, y, n, lane);
}

// M X = B for K right-hand sides at once (M = L L^T, L packed, n <= 64; B, X: K rows of stride ld, may alias).
// The K substitutions share every load of L and run as independent dependency chains, eight at a time: one pass of
// 2 n steps serves eight right-hand sides (a single substitution is latency-bound: one shuffle + one DFMA per step).
// Lanes own rows `lane` and `lane + 32` of the unknowns. Serves the dual form of the Newton direction (rows of M^-1 J').
// `xb` / `xx` (optional): one more right-hand side / solution living elsewhere (qacc_smooth = M^-1 qfrc_smooth rides along with
// the rows of J M^-1: no separate forward / backward pass).
__device__ __noinline__ void chol_solve_multi(const double* Lm, const double* dinv, int n, const double* Bm, double* Xm, int ld, int K, int lane,
                                              const double* xb, double* xx) {
  const int Kall = K + (xb ? 1 : 0);
  const int i0 = lane, i1 = lane + 32;
  const bool in0 = i0 < n, in1 = i1 < n;
  const double* L0 = Lm + tri(i0); const double* L1 = Lm + tri(i1);
  _Pragma("unroll 1") for (int r0 = 0; r0 < Kall; r0 += 8) {
    double a0[8], a1[8];
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int r = r0 + q;
      const double* src = r < K ? Bm + r * ld : xb;
      a0[q] = (r < Kall && in0) ? src[i0] : 0.0;
      a1[q] = (r < Kall && in1) ? src[i1] : 0.0;
    }
    // forward: L y = b
    _Pragma("unroll 1") for (int j = 0; j < n; j++) {
      const double dj = dinv[j];
      const double l0 = (in0 && i0 > j) ? L0[j] : 0.0, l1 = (in1 && i1 > j) ? L1[j] : 0.0;
      if (j < 32) {
#pragma unroll
        for (int q = 0; q < 8; q++) {
          const double v = __shfl_sync(FULL, a0[q], j) * dj;
          a0[q] = (lane == j) ? v : a0[q] - l0 * v;
          a1[q] -= l1 * v;
        }
      } else {
#pragma unroll
        for (int q = 0; q < 8; q++) {
          const double v = __shfl_sync(FULL, a1[q], j - 32) * dj;
          a1[q] = (i1 == j) ? v : a1[q] - l1 * v;
        }
      }
    }
    // backward: L^T x = y
    int tj = tri(n - 1);
    _Pragma("unroll 1") for (int j = n - 1; j >= 0; j--) {
      const double dj = dinv[j];
      const double l0 = (i0 < j) ? Lm[tj + i0] : 0.0, l1 = (i1 < j) ? Lm[tj + i1] : 0.0;     // i0 < j <= n - 1
      if (j >= 32) {
#pragma unroll
        for (int q = 0; q < 8; q++) {
          const double v = __shfl_sync(FULL, a1[q], j - 32) * dj;
          a1[q] = (i1 == j) ? v : a1[q] - l1 * v;
          a0[q] -= l0 * v;
        }
      } else {
#pragma unroll
        for (int q = 0; q < 8; q++) {
          const double v = __shfl_sync(FULL, a0[q], j) * dj;
          a0[q] = (lane == j) ? v : a0[q] - l0 * v;
        }
      }
      tj -= j;
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int r = r0 + q;
      double* dst = r < K ? Xm + r * ld : xx;
      if (r < Kall && in0) dst[i0] = a0[q];
      if (r < Kall && in1) dst[i1] = a1[q];
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// Compile-time-size dense algebra for the acceleration kernels (nv = N known at compile time, N <= 31).
//
// The runtime-size routines above walk the packed triangle in shared memory with rolled loops: 87 % of their
// instructions are address arithmetic, loop control and LDS, and every one waits on the one before (a profile put most
// of the acceleration kernel's stall samples there). Here one lane owns one ROW of the
// matrix in REGISTERS (N doubles), every loop is fully unrolled, so each multiply-add is one DFMA with register
// operands and an immediate-offset broadcast load:
//   * tn_factor: right-looking Cholesky. Column j is published once through a 2 x 32-double shared buffer
//     (STS, __syncwarp, then lane-invariant LDS.128 broadcasts), the trailing update is N-1-j independent DFMAs per
//     lane. The Newton Hessian  H = M + sum_active D_r J_r^T J_r  is assembled straight into the row registers, and the right-hand side rides along as row N on the spare lane N, so
//     the forward substitution costs nothing.
//   * tn_back / tn_forward: triangular solves with the column (row) of L in registers, pre-scaled by 1/L_jj and with
//     the diagonal zeroed: one shuffle + one DFMA per unknown, nothing else.
// ------------------------------------------------------------------------------------------------
#define TN_COLBUF_DOUBLES 64

// 1/sqrt(x) for x in [mjMINVAL, huge): hardware seed + one cubic step, no special-case slow path (the library
// rsqrt() carries a subroutine call for denormals / infinities, and a call inside the unrolled factorisation makes
// ptxas mirror the whole register-resident row into local memory).
__device__ __forceinline__ double pos_rsqrt(double x) {
#ifdef B200MJ_CPU_EMU
  return 1.0 / sqrt(x);
#else
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  // one third-order step: e = 1 - x y^2, y <- y (1 + e/2 + 3 e^2 / 8): 2^-22 seed -> full double precision
  const double e = fma(-x, y * y, 1.0);
  const double p = fma(0.375, e, 0.5);
  y = fma(y * e, p, y);
  return y;
#endif
}

// a zero the compiler cannot see through: keeps ptxas from cloning the 20 KB tn_factor per call site (instruction cache)
__device__ __forceinline__ int opaque_zero() {
#ifdef B200MJ_CPU_EMU
  return 0;
#else
  int z; asm volatile("mov.s32 %0, 0;" : "=r"(z)); return z;
#endif
}

template <int N>
__device__ __noinline__ void tn_factor(const double* Msrc, double* Lm, double* dinv, int lane, const double* b, double* y,
                                       const double* J, const double* SD, const int* alist, int nact, double* colbuf) {
  constexpr int LD = N | 1;
  double a[N];
  const bool isrow = lane < N, isrhs = (b != nullptr) && lane == N;
  const int ti = tri(isrow ? lane : 0);
  {
    const double* src = isrow ? Msrc + ti : (isrhs ? b : Msrc);
    const int cnt = isrow ? lane + 1 : (isrhs ? N : 0);
#pragma unroll
    for (int k = 0; k < N; k++) a[k] = k < cnt ? src[k] : 0.0;
  }
  // Newton Hessian: += sum over active rows of D_r J_r^T J_r (lower triangle is what counts)
  _Pragma("unroll 1") for (int t = 0; t < nact; t++) {
    const int r = alist[t];
    const double* Jr = J + r * LD;
    const double sj = isrow ? SD[r] * Jr[lane] : 0.0;
#pragma unroll
    for (int k = 0; k < N; k++) a[k] = MADD(sj, Jr[k], a[k]);
  }
#pragma unroll
  for (int j = 0; j < N; j++) {
    double* cb = colbuf + (j & 1) * 32;      // double-buffered: one __syncwarp per column is enough
    cb[lane] = a[j];                         // raw column j (lanes < j hold upper-triangle junk that nobody reads)
    __syncwarp();
    double piv = cb[j];
    if (piv < BMJ_MINVAL) piv = BMJ_MINVAL;
    const double inv = pos_rsqrt(piv);
    const double lj = (lane == j ? piv : a[j]) * inv;      // L[i][j]; the diagonal is sqrt(piv)
    a[j] = lj;
    if (lane == j) dinv[j] = inv;
    const double cc = lj * inv;                            // raw_i / piv : a[i][k] -= raw_i raw_k / piv
    int k = j + 1;
    if (k < N && (k & 1)) { a[k] = MADD(-cc, cb[k], a[k]); k++; }
#pragma unroll
    for (; k + 1 < N; k += 2) {
      const double2 s2 = *reinterpret_cast<const double2*>(cb + k);
      a[k] = MADD(-cc, s2.x, a[k]); a[k + 1] = MADD(-cc, s2.y, a[k + 1]);
    }
    if (k < N) a[k] = MADD(-cc, cb[k], a[k]);
  }
  if (isrow) {
#pragma unroll
    for (int k = 0; k < N; k++) if (k <= lane) Lm[ti + k] = a[k];
  } else if (isrhs) {
#pragma unroll
    for (int k = 0; k < N; k++) y[k] = a[k];
  }
  __syncwarp();
}

// L^T x = y with column `lane` of L in registers; x = -x when negate (Newton search direction). y, x may alias.
template <int N>
__device__ __noinline__ void tn_back(const double* Lm, const double* dinv, const double* y, double* x, int lane, int negate) {
  const bool on = lane < N;
  const int li = on ? lane : 0;
  const double d = on ? dinv[li] : 0.0;
  double c[N];
#pragma unroll
  for (int i = 0; i < N; i++) c[i] = (on && i > lane) ? Lm[((i * (i + 1)) >> 1) + li] * d : 0.0;
  double z = on ? y[li] * d : 0.0;
#pragma unroll
  for (int i = N - 1; i >= 1; i--) { const double xi = __shfl_sync(FULL, z, i); z = MADD(-c[i], xi, z); }
  __syncwarp();
  if (on) x[li] = negate ? -z : z;
  __syncwarp();
}

// L y = b with row `lane` of L in registers. b, y may alias.
template <int N>
__device__ __noinline__ void tn_forward(const double* Lm, const double* dinv, const double* b, double* y, int lane) {
  const bool on = lane < N;
  const int li = on ? lane : 0, ti = tri(li);
  const double d = on ? dinv[li] : 0.0;
  double r[N];
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = (on && k < lane) ? Lm[ti + k] * d : 0.0;
  double z = on ? b[li] * d : 0.0;
#pragma unroll
  for (int j = 0; j < N - 1; j++) { const double yj = __shfl_sync(FULL, z, j); z = MADD(-r[j], yj, z); }
  __syncwarp();
  if (on) y[li] = z;
  __syncwarp();
}

// row `lane` of (symmetric M, packed lower triangle) * v ; v is 16-byte aligned
template <int N>
__device__ __forceinline__ double tn_symv_row(const double* Mp, const double* v, int lane) {
  const int li = lane < N ? lane : N - 1, ti = tri(li);
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
#pragma unroll
  for (int k = 0; k + 1 < N; k += 2) {
    const double2 v2 = *reinterpret_cast<const double2*>(v + k);
    const double m0 = Mp[k <= li ? ti + k : ((k * (k + 1)) >> 1) + li];
    const double m1 = Mp[k + 1 <= li ? ti + k + 1 : (((k + 1) * (k + 2)) >> 1) + li];
    if ((k & 2) == 0) { s0 = MADD(m0, v2.x, s0); s1 = MADD(m1, v2.y, s1); } else { s2 = MADD(m0, v2.x, s2); s3 = MADD(m1, v2.y, s3); }
  }
  if (N & 1) s0 = MADD(Mp[N - 1 <= li ? ti + N - 1 : (((N - 1) * N) >> 1) + li], v[N - 1], s0);
  return (s0 + s1) + (s2 + s3);
}

// dot product of one Jacobian row (this lane's) with a 16-byte-aligned nv-vector
template <int N>
__device__ __forceinline__ double tn_dot_row(const double* row, const double* v) {
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
#pragma unroll
  for (int k = 0; k + 1 < N; k += 2) {
    const double2 v2 = *reinterpret_cast<const double2*>(v + k);
    if ((k & 2) == 0) { s0 = MADD(row[k], v2.x, s0); s1 = MADD(row[k + 1], v2.y, s1); } else { s2 = MADD(row[k], v2.x, s2); s3 = MADD(row[k + 1], v2.y, s3); }
  }
  if (N & 1) s0 = MADD(row[N - 1], v[N - 1], s0);
  return (s0 + s1) + (s2 + s3);
}

// bottom-up accumulation child -> parent for a [nbody, width] table. Bodies are numbered parents-first, so one
// reverse sweep does it; lane i owns component i (width <= 10), which keeps the summation order fixed.
__device__ __noinline__ void tree_accumulate_raw(const int* parentid, int nbody, double* tab, int width, bool into_world, int lane) {
  if (lane < width) {
    _Pragma("unroll 1") for (int b = nbody - 1; b > 0; b--) {
      int p = parentid[b];
      if (p > 0 || into_world) tab[p * width + lane] += tab[b * width + lane];
    }
  }
  __syncwarp();
}
#define tree_accumulate(c, tab, width, into_world) \
  tree_accumulate_raw((c).m.body_parentid, (c).m.nbody, tab, width, into_world, (c).lane)

// ------------------------------------------------------------------------------------------------
// position stage
// ------------------------------------------------------------------------------------------------
// geom_pos / geom_size / bounding radius of geom g in environment `env`: the model's, or this environment's own
// (corridor walls and platforms differ per environment while the topology is shared; arenas/corridors.py:394-440)
__device__ __forceinline__ void geom_pos_of(const Ctx& c, int g, double* gp) {
  const DevModel& m = c.m;
  const int k = (m.nvargeom > 0 && c.var_pos) ? m.geom_varid[g] : -1;
  const double* src = k >= 0 ? c.var_pos + ((size_t)c.env * m.nvargeom + k) * 3 : m.geom_pos + 3 * g;
  gp[0] = src[0]; gp[1] = src[1]; gp[2] = src[2];
}
__device__ __forceinline__ double geom_size_of(const Ctx& c, int g, double* sz) {
  const DevModel& m = c.m;
  const int k = (m.nvargeom > 0 && c.var_size) ? m.geom_varid[g] : -1;
  if (k < 0) { sz[0] = m.geom_size[3 * g]; sz[1] = m.geom_size[3 * g + 1]; sz[2] = m.geom_size[3 * g + 2]; return m.geom_rbound[g]; }
  const double* src = c.var_size + ((size_t)c.env * m.nvargeom + k) * 3;
  sz[0] = src[0]; sz[1] = src[1]; sz[2] = src[2];
  const int t = m.geom_type[g];
  if (t == BMJ_GEOM_SPHERE) return sz[0];
  if (t == BMJ_GEOM_CAPSULE) return sz[0] + sz[1];
  if (t == BMJ_GEOM_CYLINDER) return sqrt(sz[0] * sz[0] + sz[1] * sz[1]);
  if (t == BMJ_GEOM_ELLIPSOID) return fmax(sz[0], fmax(sz[1], sz[2]));
  if (t == BMJ_GEOM_BOX) return sqrt(sz[0] * sz[0] + sz[1] * sz[1] + sz[2] * sz[2]);
  return m.geom_rbound[g];
}

__device__ __forceinline__ void kinematics(const Ctx& c) {
  const DevModel& m = c.m; int lane = c.lane;
  double* qpos = W(qpos); double* xpos = W(xpos); double* xquat = W(xquat); double* xmat = W(xmat);
  if (lane == 0) {
    xpos[0] = xpos[1] = xpos[2] = 0; xquat[0] = 1; xquat[1] = xquat[2] = xquat[3] = 0;
    for (int i = 0; i < 9; i++) xmat[i] = (i % 4 == 0) ? 1.0 : 0.0;
  }
  FOR_LANES(j, m.njnt) {
    int t = m.jnt_type[j];
    if (t == BMJ_JNT_FREE) normalize4(qpos + m.jnt_qposadr[j] + 3);
    else if (t == BMJ_JNT_BALL) normalize4(qpos + m.jnt_qposadr[j]);
    else if (t == BMJ_JNT_HINGE) {
      // sin / cos of every hinge's half angle, all joints at once (lanes = joints): inside the level loop below only a
      // few lanes are busy, and sincos was a third of its serial chain. Parked in this joint's xanchor slot, which the
      // level loop overwrites after it has read them.
      const double angle = qpos[m.jnt_qposadr[j]] - m.qpos0[m.jnt_qposadr[j]];
      double sn = 0, cs = 1;
      if (angle != 0) sincos(angle * 0.5, &sn, &cs);
      W(xanchor)[3 * j] = sn; W(xanchor)[3 * j + 1] = cs;
    }
  }
  __syncwarp();
  _Pragma("unroll 1") for (int l = 1; l < m.nlevel; l++) {
    int a0 = m.level_adr[l], a1 = m.level_adr[l + 1];
    _Pragma("unroll 1") for (int k = a0 + lane; k < a1; k += 32) {
      int b = m.level_body[k], p = m.body_parentid[b];
      double pos[3], quat[4], tmp[3], bp[3] = {m.body_pos[3*b], m.body_pos[3*b+1], m.body_pos[3*b+2]};
      double bq[4] = {m.body_quat[4*b], m.body_quat[4*b+1], m.body_quat[4*b+2], m.body_quat[4*b+3]};
      mat_vec(tmp, xmat + 9 * p, bp);
      for (int i = 0; i < 3; i++) pos[i] = xpos[3 * p + i] + tmp[i];
      mul_quat(quat, xquat + 4 * p, bq);
      int j0 = m.body_jntadr[b], jn = m.body_jntnum[b];
      _Pragma("unroll 1") for (int j = j0; j < j0 + jn; j++) {
        int qa = m.jnt_qposadr[j], t = m.jnt_type[j];
        double* anchor = W(xanchor) + 3 * j; double* axis = W(xaxis) + 3 * j;
        double jax[3] = {m.jnt_axis[3*j], m.jnt_axis[3*j+1], m.jnt_axis[3*j+2]};
        double jp[3] = {m.jnt_pos[3*j], m.jnt_pos[3*j+1], m.jnt_pos[3*j+2]};
        const double hs = anchor[0], hc = anchor[1];       // hinge: sin, cos of the half angle (pre-pass above)
        if (t == BMJ_JNT_FREE) {
          for (int i = 0; i < 3; i++) pos[i] = qpos[qa + i];
          for (int i = 0; i < 4; i++) quat[i] = qpos[qa + 3 + i];
          for (int i = 0; i < 3; i++) anchor[i] = pos[i];
          rot_vec_quat(axis, jax, quat);
          continue;
        }
        rot_vec_quat(tmp, jp, quat);
        for (int i = 0; i < 3; i++) anchor[i] = pos[i] + tmp[i];
        double ax[3]; rot_vec_quat(ax, jax, quat);
        for (int i = 0; i < 3; i++) axis[i] = ax[i];
        if (t == BMJ_JNT_SLIDE) {
          double q = qpos[qa] - m.qpos0[qa];
          for (int i = 0; i < 3; i++) pos[i] += ax[i] * q;
        } else {
          double ql[4], r[4];
          if (t == BMJ_JNT_HINGE) {     // axis_angle2quat with the precomputed sin / cos (hs == 0 <=> angle == 0)
            if (hs == 0) { ql[0] = 1; ql[1] = ql[2] = ql[3] = 0; }
            else { ql[0] = hc; ql[1] = jax[0] * hs; ql[2] = jax[1] * hs; ql[3] = jax[2] * hs; }
          } else for (int i = 0; i < 4; i++) ql[i] = qpos[qa + i];
          mul_quat(r, quat, ql);
          for (int i = 0; i < 4; i++) quat[i] = r[i];
          rot_vec_quat(tmp, jp, quat);
          for (int i = 0; i < 3; i++) pos[i] = anchor[i] - tmp[i];
        }
      }
      normalize4(quat);
      for (int i = 0; i < 3; i++) xpos[3 * b + i] = pos[i];
      for (int i = 0; i < 4; i++) xquat[4 * b + i] = quat[i];
      quat2mat(xmat + 9 * b, quat);
    }
    __syncwarp();
  }
  // inertial frames' origins and geom frames
  FOR_LANES(b, m.nbody) {
    double tmp[3], ip[3] = {m.body_ipos[3*b], m.body_ipos[3*b+1], m.body_ipos[3*b+2]};
    mat_vec(tmp, xmat + 9 * b, ip);
    for (int i = 0; i < 3; i++) W(xipos)[3 * b + i] = xpos[3 * b + i] + tmp[i];
  }
  FOR_LANES(g, m.ngeom) {
    int b = m.geom_bodyid[g];
    double tmp[3], q[4], gp[3];
    geom_pos_of(c, g, gp);
    double gq[4] = {m.geom_quat[4*g], m.geom_quat[4*g+1], m.geom_quat[4*g+2], m.geom_quat[4*g+3]};
    mat_vec(tmp, xmat + 9 * b, gp);
    for (int i = 0; i < 3; i++) W(gxpos)[3 * g + i] = xpos[3 * b + i] + tmp[i];
    mul_quat(q, xquat + 4 * b, gq);
    quat2mat(W(gxmat) + 9 * g, q);
  }
  __syncwarp();
}

__device__ __forceinline__ void site_frame(const Ctx& c, int s, double* pos, double* mat) {
  const DevModel& m = c.m;
  int b = m.site_bodyid[s];
  double tmp[3], q[4], sp[3] = {m.site_pos[3*s], m.site_pos[3*s+1], m.site_pos[3*s+2]};
  double sq[4] = {m.site_quat[4*s], m.site_quat[4*s+1], m.site_quat[4*s+2], m.site_quat[4*s+3]};
  mat_vec(tmp, W(xmat) + 9 * b, sp);
  for (int i = 0; i < 3; i++) pos[i] = W(xpos)[3 * b + i] + tmp[i];
  mul_quat(q, W(xquat) + 4 * b, sq);
  quat2mat(mat, q);
}

__device__ __forceinline__ void geom_frame(const Ctx& c, int g, double* pos, double* mat) {
  const DevModel& m = c.m;
  int b = m.geom_bodyid[g];
  double tmp[3], q[4], gp[3];
  geom_pos_of(c, g, gp);
  double gq[4] = {m.geom_quat[4*g], m.geom_quat[4*g+1], m.geom_quat[4*g+2], m.geom_quat[4*g+3]};
  mat_vec(tmp, W(xmat) + 9 * b, gp);
  for (int i = 0; i < 3; i++) pos[i] = W(xpos)[3 * b + i] + tmp[i];
  mul_quat(q, W(xquat) + 4 * b, gq);
  quat2mat(mat, q);
}

__device__ __forceinline__ void com_pos(const Ctx& c) {
  const DevModel& m = c.m; int lane = c.lane;
  double* sc = W(scom); double* xipos = W(xipos);
  FOR_LANES(b, m.nbody) { double ms = m.body_mass[b]; for (int i = 0; i < 3; i++) sc[3 * b + i] = ms * xipos[3 * b + i]; }
  __syncwarp();
  tree_accumulate(c, sc, 3, true);
  FOR_LANES(b, m.nbody) {
    double sm = m.body_subtreemass[b];
    if (sm < BMJ_MINVAL) for (int i = 0; i < 3; i++) sc[3 * b + i] = xipos[3 * b + i];
    else for (int i = 0; i < 3; i++) sc[3 * b + i] /= sm;
  }
  __syncwarp();
  FOR_LANES(b, m.nbody) {
    double* ci = W(cinert) + 10 * b;
    if (b == 0) { for (int i = 0; i < 10; i++) ci[i] = 0; continue; }
    double q[4], mat[9], iq[4] = {m.body_iquat[4*b], m.body_iquat[4*b+1], m.body_iquat[4*b+2], m.body_iquat[4*b+3]};
    mul_quat(q, W(xquat) + 4 * b, iq);
    quat2mat(mat, q);
    int root = m.body_rootid[b];
    double dif[3];
    for (int i = 0; i < 3; i++) dif[i] = xipos[3 * b + i] - sc[3 * root + i];
    double mass = m.body_mass[b], in0 = m.body_inertia[3*b], in1 = m.body_inertia[3*b+1], in2 = m.body_inertia[3*b+2];
    double t[9];
    for (int r = 0; r < 3; r++) for (int cc = 0; cc < 3; cc++)
      t[3 * r + cc] = mat[3 * r] * in0 * mat[3 * cc] + mat[3 * r + 1] * in1 * mat[3 * cc + 1] + mat[3 * r + 2] * in2 * mat[3 * cc + 2];
    ci[0] = t[0] + mass * (dif[1]*dif[1] + dif[2]*dif[2]);
    ci[1] = t[4] + mass * (dif[0]*dif[0] + dif[2]*dif[2]);
    ci[2] = t[8] + mass * (dif[0]*dif[0] + dif[1]*dif[1]);
    ci[3] = t[1] - mass * dif[0]*dif[1];
    ci[4] = t[2] - mass * dif[0]*dif[2];
    ci[5] = t[5] - mass * dif[1]*dif[2];
    ci[6] = mass * dif[0]; ci[7] = mass * dif[1]; ci[8] = mass * dif[2]; ci[9] = mass;
  }
  FOR_LANES(j, m.njnt) {
    int b = m.jnt_bodyid[j], root = m.body_rootid[b], da = m.jnt_dofadr[j], t = m.jnt_type[j];
    double off[3];
    for (int i = 0; i < 3; i++) off[i] = sc[3 * root + i] - W(xanchor)[3 * j + i];
    double* cd = W(cdof) + 6 * da;
    if (t == BMJ_JNT_FREE) {
      for (int k = 0; k < 3; k++) { for (int i = 0; i < 6; i++) cd[6 * k + i] = 0; cd[6 * k + 3 + k] = 1; }
      cd += 18;
    }
    if (t == BMJ_JNT_FREE || t == BMJ_JNT_BALL) {
      const double* xm = W(xmat) + 9 * b;
      for (int k = 0; k < 3; k++) {
        double ax[3] = {xm[k], xm[3 + k], xm[6 + k]};
        for (int i = 0; i < 3; i++) cd[6 * k + i] = ax[i];
        cross3(cd + 6 * k + 3, ax, off);
      }
    } else if (t == BMJ_JNT_SLIDE) {
      for (int i = 0; i < 3; i++) { cd[i] = 0; cd[3 + i] = W(xaxis)[3 * j + i]; }
    } else {
      double ax[3] = {W(xaxis)[3*j], W(xaxis)[3*j+1], W(xaxis)[3*j+2]};
      for (int i = 0; i < 3; i++) cd[i] = ax[i];
      cross3(cd + 3, ax, off);
    }
  }
  // fixed tendons: length and (dense) Jacobian row
  FOR_LANES(t, m.ntendon) {
    double* row = W(tenJ) + t * m.ldv;
    _Pragma("unroll 1") for (int i = 0; i < m.nv; i++) row[i] = 0;
    double len = 0;
    _Pragma("unroll 1") for (int w = m.tendon_adr[t]; w < m.tendon_adr[t] + m.tendon_num[t]; w++) {
      int j = m.wrap_objid[w];
      len += m.wrap_prm[w] * W(qpos)[m.jnt_qposadr[j]];
      row[m.jnt_dofadr[j]] += m.wrap_prm[w];
    }
    W(tenlen)[t] = len;
  }
  __syncwarp();
}

__device__ __forceinline__ void crb_and_factor(const Ctx& c) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  double* crb = W(crb); double* M = c.pM;
  _Pragma("unroll 1") for (int i = lane; i < 10 * m.nbody; i += 32) crb[i] = W(cinert)[i];
  _Pragma("unroll 1") for (int i = lane; i < tri(nv); i += 32) M[i] = 0;
  __syncwarp();
  tree_accumulate(c, crb, 10, false);
  FOR_LANES(i, nv) {
    double buf[6], cd[6];
    for (int k = 0; k < 6; k++) cd[k] = W(cdof)[6 * i + k];
    mul_inert_vec(buf, crb + 10 * m.dof_bodyid[i], cd);
    for (int j = i; j >= 0; j = m.dof_parentid[j]) {
      const double* cj = W(cdof) + 6 * j;
      double s = 0;
      for (int k = 0; k < 6; k++) s += cj[k] * buf[k];
      if (j == i) s += m.dof_armature[i];
      M[tri(i) + j] = s;      // packed lower triangle: j walks the ancestors of i, so j <= i
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// collision (narrow phase per candidate pair; lanes = pairs; ordered compaction keeps pair order)
// ------------------------------------------------------------------------------------------------
#define MAXPC 4   // contacts one geom pair can emit
// Raw contacts are staged in shared memory (lane-strided, inside the not-yet-used Jacobian buffer) rather than in
// a per-thread array: dynamic indexing would push that array to local memory. Slot k, field f of this lane:
//   stg[(k*7 + f)*32]   f = 0 dist, 1..3 pos, 4..6 normal ;  tangent hint: stg[(28 + f)*32]
#define STG(k, f) stg[((k) * 7 + (f)) * 32]
#define STG_TAN(f) stg[(28 + (f)) * 32]
#define STAGE_DOUBLES (31 * 32)

__device__ __forceinline__ void stage_contact(double* stg, int& n, double dist, const double* pos, const double* nrm) {
  STG(n, 0) = dist;
  for (int i = 0; i < 3; i++) { STG(n, 1 + i) = pos[i]; STG(n, 4 + i) = nrm[i]; }
  n++;
}
__device__ __forceinline__ void raw_plane_sphere(double* stg, int& n, double margin, const double* ppos, const double* nrm, const double* spos, double radius) {
  double dif[3] = {spos[0] - ppos[0], spos[1] - ppos[1], spos[2] - ppos[2]};
  double cdist = dot3(dif, nrm);
  if (cdist > margin + radius) return;
  double dist = cdist - radius, pos[3];
  for (int i = 0; i < 3; i++) pos[i] = spos[i] - nrm[i] * (radius + 0.5 * dist);
  stage_contact(stg, n, dist, pos, nrm);
}
__device__ __forceinline__ void raw_sphere_sphere(double* stg, int& n, double margin, const double* p1, double r1, const double* p2, double r2) {
  double dif[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  double cdist = norm3(dif);
  if (cdist > margin + r1 + r2) return;
  double dist = cdist - r1 - r2, nrm[3], pos[3];
  if (cdist < BMJ_MINVAL) { nrm[0] = 1; nrm[1] = nrm[2] = 0; }
  else for (int i = 0; i < 3; i++) nrm[i] = dif[i] / cdist;
  for (int i = 0; i < 3; i++) pos[i] = p1[i] + nrm[i] * (r1 + 0.5 * dist);
  stage_contact(stg, n, dist, pos, nrm);
}

// ------------------------------------------------------------------------------------------------
// cvx_pair (include/b200mj_convex.h) with the WHOLE WARP on one pair: same arithmetic, same answer, a fifth of the
// latency. A convex contact costs up to ~900 support evaluations in sequence (12 frame axes + a 96-point lattice for the
// start directions, three descents of <= 32 steps with <= 8 step halvings each, MPR before and after); with one pair
// per lane a single touching ellipsoid kept its environment — and, through the phase barriers, its CTA and the whole
// launch — waiting (on the CMU corridor, a visible share of each control step). Here the 108 start-direction evaluations run one per
// lane, the three descents run side by side in three groups of eight lanes and every group evaluates its eight halvings
// of a step at once; selections replicate the scalar code's order (first index among equal minima, first accepted
// halving), so the contact is bit-identical to cvx_pair's (tests/test_convex_pairs.py, emulated kernel vs oracle).
// The two MPR passes stay sequential and are executed redundantly by all lanes (no divergence, no broadcast).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int first_bit(unsigned b) { return __popc((b & (0u - b)) - 1u); }
__device__ __forceinline__ void warp_argmin(double& h, int& k) {      // smallest h, smallest k among equals; h >= 1e300 / NaN never win
  if (!(h < 1e300)) { h = 1e300; k = 1 << 20; }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const double oh = __shfl_xor_sync(FULL, h, off); const int ok = __shfl_xor_sync(FULL, k, off);
    if (oh < h || (oh == h && ok < k)) { h = oh; k = ok; }
  }
}

__device__ __noinline__ int cvx_pair_warp(int lane, int t1, const double* p1, const double* m1, const double* s1, int t2, const double* p2,
                                          const double* m2, const double* s2, double margin, double* dist, double* pos, double* nrm) {
  CvxGeom g1 = {t1, p1, m1, s1, 0.5 * margin}, g2 = {t2, p2, m2, s2, 0.5 * margin};
  double depth;
  if (!cvx_mpr(g1, g2, (const double*)0, &depth, nrm, pos)) return 0;
  double start[9] = {nrm[0], nrm[1], nrm[2], nrm[0], nrm[1], nrm[2], nrm[0], nrm[1], nrm[2]};
  {   // best frame axis of the two geoms: k = lane < 12
    double hk = 1e300; int kk = lane;
    if (lane < 12) {
      const double* mm = lane < 6 ? m1 : m2;
      const int ax = (lane % 6) >> 1; const double sg = (lane & 1) ? -1.0 : 1.0;
      const double dk[3] = {sg * mm[ax], sg * mm[3 + ax], sg * mm[6 + ax]};
      CvxSup sk; cvx_support(g1, g2, dk, sk);
      hk = cvx_dot(sk.v, dk);
    }
    warp_argmin(hk, kk);
    if (kk < 12) {
      const double* mm = kk < 6 ? m1 : m2;
      const int ax = (kk % 6) >> 1; const double sg = (kk & 1) ? -1.0 : 1.0;
      start[3] = sg * mm[ax]; start[4] = sg * mm[3 + ax]; start[5] = sg * mm[6 + ax];
    }
  }
  {   // best point of the 96-point Fibonacci lattice: k = lane, lane + 32, lane + 64
    double hb = 1e300; int kb = 1 << 20;
    _Pragma("unroll 1") for (int k = lane; k < 96; k += 32) {
      const double z = 1.0 - (2.0 * k + 1.0) / 96.0, rr = sqrt(1.0 - z * z), ph = 2.399963229728653 * k;
      const double dk[3] = {rr * cos(ph), rr * sin(ph), z};
      CvxSup sk; cvx_support(g1, g2, dk, sk);
      const double hk = cvx_dot(sk.v, dk);
      if (hk < hb) { hb = hk; kb = k; }
    }
    warp_argmin(hb, kb);
    if (kb < 96) {
      const double z = 1.0 - (2.0 * kb + 1.0) / 96.0, rr = sqrt(1.0 - z * z), ph = 2.399963229728653 * kb;
      start[6] = rr * cos(ph); start[7] = rr * sin(ph); start[8] = z;
    }
  }
  // three descents side by side: group = lane / 8 (the fourth group repeats the third and is ignored), eight halvings per step at once
  const int grp = lane >> 3, c = grp < 3 ? grp : 2, hf = lane & 7;
  double d[3] = {start[3 * c], start[3 * c + 1], start[3 * c + 2]};
  CvxSup sf; cvx_support(g1, g2, d, sf);
  double hd = cvx_dot(sf.v, d), eta = 0;
  bool active = true;
  _Pragma("unroll 1") for (int it = 0; it < 32; it++) {
    double g[3] = {sf.v[0] - hd * d[0], sf.v[1] - hd * d[1], sf.v[2] - hd * d[2]};
    if (active && cvx_dot(g, g) < 1e-20) active = false;
    if (!__any_sync(FULL, active)) break;
    if (active && it == 0) {
      const double nd[3] = {-d[0], -d[1], -d[2]};
      CvxSup sb; cvx_support(g1, g2, nd, sb);
      const double hb = cvx_dot(sb.v, nd);
      eta = 2.0 / (hb - hd > 1e-9 ? hb - hd : 1e-9);
    }
    double eh = eta;
    for (int q = 0; q < hf; q++) eh *= 0.5;                 // the scalar code's `eta *= 0.5`, hf times
    double dn[3] = {d[0] - eh * g[0], d[1] - eh * g[1], d[2] - eh * g[2]};
    cvx_normalize(dn);
    CvxSup sn; cvx_support(g1, g2, dn, sn);
    const double hn = cvx_dot(sn.v, dn);
    const unsigned acc = (__ballot_sync(FULL, active && hn < hd - 1e-14) >> (8 * grp)) & 0xffu;
    if (active && acc == 0) active = false;
    const int src = (active ? 8 * grp + first_bit(acc) : lane);
    // the accepted candidate of this group (its first accepted halving) becomes the group's state
    const double a_dn0 = __shfl_sync(FULL, dn[0], src), a_dn1 = __shfl_sync(FULL, dn[1], src), a_dn2 = __shfl_sync(FULL, dn[2], src);
    const double a_hn = __shfl_sync(FULL, hn, src), a_eh = __shfl_sync(FULL, eh, src);
    CvxSup a_sn;
#pragma unroll
    for (int i = 0; i < 3; i++) { a_sn.v[i] = __shfl_sync(FULL, sn.v[i], src); a_sn.a[i] = __shfl_sync(FULL, sn.a[i], src); a_sn.b[i] = __shfl_sync(FULL, sn.b[i], src); }
    if (active) {
      const double a_dn[3] = {a_dn0, a_dn1, a_dn2};
      const double gn[3] = {a_sn.v[0] - a_hn * a_dn[0], a_sn.v[1] - a_hn * a_dn[1], a_sn.v[2] - a_hn * a_dn[2]};
      const double dd[3] = {a_dn[0] - d[0], a_dn[1] - d[1], a_dn[2] - d[2]}, dg[3] = {gn[0] - g[0], gn[1] - g[1], gn[2] - g[2]};
      const double sy = cvx_dot(dd, dg), ss = cvx_dot(dd, dd);
      d[0] = a_dn[0]; d[1] = a_dn[1]; d[2] = a_dn[2]; sf = a_sn; hd = a_hn;
      eta = (sy > 1e-12 * ss && ss > 0) ? ss / sy : 2 * a_eh;
    }
  }
  // the lowest end point wins, first descent first
  double dbest[3] = {nrm[0], nrm[1], nrm[2]}, hbest = 1e300;
  CvxSup sbest; cvx_support(g1, g2, dbest, sbest);
#pragma unroll
  for (int cc = 0; cc < 3; cc++) {
    const double h_c = __shfl_sync(FULL, hd, 8 * cc);
    double d_c[3]; CvxSup s_c;
#pragma unroll
    for (int i = 0; i < 3; i++) { d_c[i] = __shfl_sync(FULL, d[i], 8 * cc); s_c.v[i] = __shfl_sync(FULL, sf.v[i], 8 * cc); s_c.a[i] = __shfl_sync(FULL, sf.a[i], 8 * cc); s_c.b[i] = __shfl_sync(FULL, sf.b[i], 8 * cc); }
    if (h_c < hbest) { hbest = h_c; dbest[0] = d_c[0]; dbest[1] = d_c[1]; dbest[2] = d_c[2]; sbest = s_c; }
  }
  if (hbest < depth - 1e-9) {
    const double nd[3] = {-dbest[0], -dbest[1], -dbest[2]};
    CvxSup sb; cvx_support(g1, g2, nd, sb);
    const double ext = cvx_dot(sb.v, nd);
    double d2 = 1e300, n2[3], p2v[3];
    int hit = 0;
    if (ext > 1e-12) {
      const double inner[3] = {0.5 * ext * nd[0], 0.5 * ext * nd[1], 0.5 * ext * nd[2]};
      hit = cvx_mpr(g1, g2, inner, &d2, n2, p2v);
    }
    if (hit && d2 <= hbest + 1e-9) {
      depth = d2;
      for (int i = 0; i < 3; i++) { nrm[i] = n2[i]; pos[i] = p2v[i]; }
    } else {
      depth = hbest;
      for (int i = 0; i < 3; i++) { nrm[i] = dbest[i]; pos[i] = 0.5 * (sbest.a[i] + sbest.b[i]); }
    }
  }
  *dist = margin - depth;
  return 1;
}

// geom-type pairs that narrowphase<true> resolves with cvx_pair (everything without a closed form; t1 <= t2)
__device__ __forceinline__ bool pair_is_mpr(int t1, int t2) {
  if (t1 == BMJ_GEOM_PLANE || t1 == BMJ_GEOM_SPHERE && (t2 == BMJ_GEOM_SPHERE || t2 == BMJ_GEOM_CAPSULE || t2 == BMJ_GEOM_BOX)) return false;
  if (t1 == BMJ_GEOM_CAPSULE && (t2 == BMJ_GEOM_CAPSULE || t2 == BMJ_GEOM_BOX)) return false;
  return t1 >= BMJ_GEOM_SPHERE && t2 <= BMJ_GEOM_BOX;
}

// returns the number of raw contacts staged for this lane's pair (normal points from geom1 to geom2)
// CVX = false: the model's candidate pairs are all analytic primitive pairs (decided at model_create), so the convex routines
// (cvx_capsule_box / cvx_pair: ~50 registers and 0.8 KB of stack in the position kernels) are compiled out.
template <bool CVX>
__device__ __noinline__ int narrowphase(double* stg, int t1, int t2, double margin, const double* p1, const double* m1, const double* s1,
                                        const double* p2, const double* m2, const double* s2) {
  int n = 0;
  STG_TAN(0) = 0; STG_TAN(1) = 0; STG_TAN(2) = 0;
  if (t1 == BMJ_GEOM_PLANE) {
    double nr[3] = {m1[2], m1[5], m1[8]};
    if (t2 == BMJ_GEOM_SPHERE) { raw_plane_sphere(stg, n, margin, p1, nr, p2, s2[0]); return n; }
    if (t2 == BMJ_GEOM_CAPSULE) {
      double ax[3] = {m2[2], m2[5], m2[8]}, e[3];
      for (int i = 0; i < 3; i++) e[i] = p2[i] + ax[i] * s2[1];
      raw_plane_sphere(stg, n, margin, p1, nr, e, s2[0]);
      for (int i = 0; i < 3; i++) e[i] = p2[i] - ax[i] * s2[1];
      raw_plane_sphere(stg, n, margin, p1, nr, e, s2[0]);
      if (n) for (int i = 0; i < 3; i++) STG_TAN(i) = ax[i];
      return n;
    }
    if (t2 == BMJ_GEOM_ELLIPSOID) {
      double nl[3]; matT_vec(nl, m2, nr);
      double sv[3] = {nl[0] * s2[0], nl[1] * s2[1], nl[2] * s2[2]};
      double len = norm3(sv);
      if (len < BMJ_MINVAL) return 0;
      double loc[3] = {-s2[0] * sv[0] / len, -s2[1] * sv[1] / len, -s2[2] * sv[2] / len}, pt[3];
      mat_vec(pt, m2, loc);
      for (int i = 0; i < 3; i++) pt[i] += p2[i];
      double dif[3] = {pt[0] - p1[0], pt[1] - p1[1], pt[2] - p1[2]};
      double dist = dot3(dif, nr);
      if (dist > margin) return 0;
      double pos[3];
      for (int i = 0; i < 3; i++) pos[i] = pt[i] - nr[i] * dist * 0.5;
      stage_contact(stg, n, dist, pos, nr);
      return n;
    }
    if (t2 == BMJ_GEOM_BOX) {
      double dif[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
      double dist0 = dot3(dif, nr);
      for (int k = 0; k < 8 && n < MAXPC; k++) {
        double loc[3] = {(k & 1 ? s2[0] : -s2[0]), (k & 2 ? s2[1] : -s2[1]), (k & 4 ? s2[2] : -s2[2])}, corner[3];
        mat_vec(corner, m2, loc);
        double ldist = dot3(nr, corner);
        if (dist0 + ldist > margin || ldist > 0) continue;
        double dist = dist0 + ldist, pos[3];
        for (int i = 0; i < 3; i++) pos[i] = p2[i] + corner[i] - nr[i] * dist * 0.5;
        stage_contact(stg, n, dist, pos, nr);
      }
      return n;
    }
    if (t2 == BMJ_GEOM_CYLINDER) {
      double ax[3] = {m2[2], m2[5], m2[8]};
      double dif[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
      double dist0 = dot3(dif, nr), prjaxis = dot3(nr, ax);
      if (prjaxis > 0) { for (int i = 0; i < 3; i++) ax[i] = -ax[i]; prjaxis = -prjaxis; }
      double vec[3], len_sq = 0;
      for (int i = 0; i < 3; i++) { vec[i] = ax[i] * prjaxis - nr[i]; len_sq += vec[i] * vec[i]; }
      double len = sqrt(len_sq);
      if (len < 1e-12) { vec[0] = m2[0] * s2[0]; vec[1] = m2[3] * s2[0]; vec[2] = m2[6] * s2[0]; }
      else for (int i = 0; i < 3; i++) vec[i] *= s2[0] / len;
      double prjvec = dot3(vec, nr), axl[3], pos[3];
      for (int i = 0; i < 3; i++) axl[i] = ax[i] * s2[1];
      double prjax = prjaxis * s2[1];
      if (dist0 + prjax + prjvec > margin) return 0;
      double dist = dist0 + prjax + prjvec;
      for (int i = 0; i < 3; i++) pos[i] = p2[i] + vec[i] + axl[i] - nr[i] * dist * 0.5;
      stage_contact(stg, n, dist, pos, nr);
      if (dist0 - prjax + prjvec <= margin) {
        dist = dist0 - prjax + prjvec;
        for (int i = 0; i < 3; i++) pos[i] = p2[i] + vec[i] - axl[i] - nr[i] * dist * 0.5;
        stage_contact(stg, n, dist, pos, nr);
      }
      double prjvec1 = -prjvec * 0.5;
      if (dist0 + prjax + prjvec1 <= margin) {
        double v1[3]; cross3(v1, vec, ax);
        double l1 = norm3(v1);
        if (l1 > BMJ_MINVAL) {
          for (int i = 0; i < 3; i++) v1[i] *= s2[0] * sqrt(3.0) * 0.5 / l1;
          for (int sgn = -1; sgn <= 1 && n < MAXPC; sgn += 2) {
            dist = dist0 + prjax + prjvec1;
            for (int i = 0; i < 3; i++) pos[i] = p2[i] + sgn * v1[i] + axl[i] - vec[i] * 0.5 - nr[i] * dist * 0.5;
            stage_contact(stg, n, dist, pos, nr);
          }
        }
      }
      return n;
    }
    return 0;
  }
  if (t1 == BMJ_GEOM_SPHERE) {
    if (t2 == BMJ_GEOM_SPHERE) { raw_sphere_sphere(stg, n, margin, p1, s1[0], p2, s2[0]); return n; }
    if (t2 == BMJ_GEOM_CAPSULE) {
      double ax[3] = {m2[2], m2[5], m2[8]}, w[3] = {p1[0] - p2[0], p1[1] - p2[1], p1[2] - p2[2]};
      double x = clampd(dot3(ax, w), -s2[1], s2[1]), nearp[3];
      for (int i = 0; i < 3; i++) nearp[i] = p2[i] + ax[i] * x;
      raw_sphere_sphere(stg, n, margin, p1, s1[0], nearp, s2[0]);
      return n;
    }
    if (t2 == BMJ_GEOM_BOX) {
      double w[3] = {p1[0] - p2[0], p1[1] - p2[1], p1[2] - p2[2]}, loc[3], cl[3], nl[3], dist;
      matT_vec(loc, m2, w);
      bool inside = true;
      for (int i = 0; i < 3; i++) { cl[i] = clampd(loc[i], -s2[i], s2[i]); if (cl[i] != loc[i]) inside = false; }
      if (!inside) {
        double dl[3] = {loc[0] - cl[0], loc[1] - cl[1], loc[2] - cl[2]};
        double dn = norm3(dl);
        if (dn - s1[0] > margin) return 0;
        dist = dn - s1[0];
        for (int i = 0; i < 3; i++) nl[i] = -dl[i] / dn;
      } else {
        double bd = s2[0] - fabs(loc[0]); int best = 0;
        if (s2[1] - fabs(loc[1]) < bd) { bd = s2[1] - fabs(loc[1]); best = 1; }
        if (s2[2] - fabs(loc[2]) < bd) { bd = s2[2] - fabs(loc[2]); best = 2; }
        double sg0 = loc[0] > 0 ? -1 : 1, sg1 = loc[1] > 0 ? -1 : 1, sg2 = loc[2] > 0 ? -1 : 1;
        nl[0] = best == 0 ? sg0 : 0; nl[1] = best == 1 ? sg1 : 0; nl[2] = best == 2 ? sg2 : 0;
        dist = -bd - s1[0];
      }
      double nw[3], pos[3]; mat_vec(nw, m2, nl);
      for (int i = 0; i < 3; i++) pos[i] = p1[i] + nw[i] * (s1[0] + 0.5 * dist);
      stage_contact(stg, n, dist, pos, nw);
      return n;
    }
  }
  if constexpr (CVX) {
    if (t1 == BMJ_GEOM_CAPSULE && t2 == BMJ_GEOM_BOX) {
      double out[14];
      const int nc = cvx_capsule_box(p1, m1, s1, p2, m2, s2, margin, out);
      if (nc > 0) stage_contact(stg, n, out[0], out + 1, out + 4);
      if (nc > 1) stage_contact(stg, n, out[7], out + 8, out + 11);
      return n;
    }
    if (!(t1 == BMJ_GEOM_CAPSULE && t2 == BMJ_GEOM_CAPSULE)) {
      // every remaining pair of convex primitives (an ellipsoid, a cylinder or two boxes involved): MPR, one contact
      if (t1 >= BMJ_GEOM_SPHERE && t2 <= BMJ_GEOM_BOX) {
        double dist, pos[3], nrm[3];
        if (cvx_pair(t1, p1, m1, s1, t2, p2, m2, s2, margin, &dist, pos, nrm)) stage_contact(stg, n, dist, pos, nrm);
      }
      return n;
    }
  } else if (!(t1 == BMJ_GEOM_CAPSULE && t2 == BMJ_GEOM_CAPSULE)) return 0;   // unreachable: see pair_needs_convex()
  if (t1 == BMJ_GEOM_CAPSULE && t2 == BMJ_GEOM_CAPSULE) {
    double a1[3] = {m1[2], m1[5], m1[8]}, a2[3] = {m2[2], m2[5], m2[8]};
    double dif[3] = {p1[0] - p2[0], p1[1] - p2[1], p1[2] - p2[2]};
    double ma = dot3(a1, a1), mb = -dot3(a1, a2), mc = dot3(a2, a2);
    double u = -dot3(a1, dif), v = dot3(a2, dif);
    double det = ma * mc - mb * mb, len1 = s1[1], len2 = s2[1];
    if (fabs(det) >= BMJ_MINVAL) {
      double x1 = (mc * u - mb * v) / det, x2 = (ma * v - mb * u) / det;
      if (x1 > len1) { x1 = len1; x2 = (v - mb * len1) / mc; }
      else if (x1 < -len1) { x1 = -len1; x2 = (v + mb * len1) / mc; }
      if (x2 > len2) { x2 = len2; x1 = clampd((u - mb * len2) / ma, -len1, len1); }
      else if (x2 < -len2) { x2 = -len2; x1 = clampd((u + mb * len2) / ma, -len1, len1); }
      double v1[3], v2[3];
      for (int i = 0; i < 3; i++) { v1[i] = p1[i] + a1[i] * x1; v2[i] = p2[i] + a2[i] * x2; }
      raw_sphere_sphere(stg, n, margin, v1, s1[0], v2, s2[0]);
      return n;
    }
    for (int e = 0; e < 2 && n < 2; e++) {
      double x1 = e == 0 ? len1 : -len1, v1[3], v2[3];
      for (int i = 0; i < 3; i++) v1[i] = p1[i] + a1[i] * x1;
      double w[3] = {v1[0] - p2[0], v1[1] - p2[1], v1[2] - p2[2]};
      double x2 = dot3(w, a2);
      if (x2 < -len2 || x2 > len2) continue;
      for (int i = 0; i < 3; i++) v2[i] = p2[i] + a2[i] * x2;
      raw_sphere_sphere(stg, n, margin, v1, s1[0], v2, s2[0]);
    }
    for (int e = 0; e < 2 && n < 2; e++) {
      double x2 = e == 0 ? len2 : -len2, v1[3], v2[3];
      for (int i = 0; i < 3; i++) v2[i] = p2[i] + a2[i] * x2;
      double w[3] = {v2[0] - p1[0], v2[1] - p1[1], v2[2] - p1[2]};
      double x1 = dot3(w, a1);
      if (x1 <= -len1 || x1 >= len1) continue;
      for (int i = 0; i < 3; i++) v1[i] = p1[i] + a1[i] * x1;
      raw_sphere_sphere(stg, n, margin, v1, s1[0], v2, s2[0]);
    }
    if (n == 0) {
      double x1 = clampd(u / ma, -len1, len1), v1[3], v2[3];
      for (int i = 0; i < 3; i++) v1[i] = p1[i] + a1[i] * x1;
      double w[3] = {v1[0] - p2[0], v1[1] - p2[1], v1[2] - p2[2]};
      double x2 = clampd(dot3(w, a2), -len2, len2);
      for (int i = 0; i < 3; i++) v2[i] = p2[i] + a2[i] * x2;
      raw_sphere_sphere(stg, n, margin, v1, s1[0], v2, s2[0]);
    }
    return n;
  }
  return 0;
}

__device__ __forceinline__ void make_frame(double* frame, const double* normal, const double* tangent) {
  double x[3] = {normal[0], normal[1], normal[2]};
  normalize3(x);
  double y[3] = {tangent[0], tangent[1], tangent[2]};
  if (norm3(y) < 0.5) {
    y[0] = y[1] = y[2] = 0;
    if (x[1] < 0.5 && x[1] > -0.5) y[1] = 1; else y[2] = 1;
  }
  double dp = dot3(x, y);
  for (int i = 0; i < 3; i++) y[i] -= dp * x[i];
  normalize3(y);
  double z[3]; cross3(z, x, y);
  for (int i = 0; i < 3; i++) { frame[i] = x[i]; frame[3 + i] = y[i]; frame[6 + i] = z[i]; }
}

// contact record: [0] dist, [1..3] pos, [4..12] frame, [13] mu, [14] (geom1,geom2), [15] (dim, efc_address)
#define CON_STRIDE 16
__device__ __forceinline__ int* con_ints(double* rec) { return reinterpret_cast<int*>(rec + 14); }

template <bool CVX>
__device__ __forceinline__ int collision(const Ctx& c, int* warn_contactfull) {
  const DevModel& m = c.m; int lane = c.lane;
  int ncon = 0;
  if (c.disableflags & (BMJ_DSBL_CONTACT | BMJ_DSBL_CONSTRAINT)) return 0;
  double* stg = c.stage + lane;   // staging: the Jacobian buffer (fused kernel) / the not-yet-written dynamics block (split)
  // Two phases, interleaved: the bounding tests of 32 candidate pairs at a time append the survivors to a queue (in pair
  // order), and the narrow phase runs over 32 queued pairs at a time. Few of a model's candidate pairs pass the bounds
  // in any one step (CMU corridor: 2 113 candidates, a few dozen survivors), and the narrow phase is divergent code: run
  // per 32 candidates, every chunk with one survivor paid for a whole pass. Contacts come out in pair order as before.
  int* queue = reinterpret_cast<int*>(W(cq));
  // With many candidate pairs per geom the per-pair chain  pair -> geom -> (type, margin, size / per-environment size ->
  // bounding radius)  through global memory is what the bounding tests wait for (long-scoreboard stalls 4.1 per issue in
  // the CMU corridor capture): stage the three per-geom quantities in shared memory once.
  const bool gc = c.L.gcache != 0;
  int* gty = reinterpret_cast<int*>(W(gty));
  if (gc) {
    FOR_LANES(g, m.ngeom) { double sz[3]; W(grb)[g] = geom_size_of(c, g, sz); W(gmg)[g] = m.geom_margin[g]; gty[g] = m.geom_type[g]; }
    __syncwarp();
  }
  int qn = 0, base = 0;
  _Pragma("unroll 1") while (base < m.npair || qn > 0) {
    _Pragma("unroll 1") while (qn < 32 && base < m.npair) {
      const int p = base + lane;
      bool keep = false;
      if (p < m.npair) {
        const int g1 = m.pair_geom1[p], g2 = m.pair_geom2[p];
        const int t1 = gc ? gty[g1] : m.geom_type[g1], t2 = gc ? gty[g2] : m.geom_type[g2];
        const double margin = gc ? fmax(W(gmg)[g1], W(gmg)[g2]) : fmax(m.geom_margin[g1], m.geom_margin[g2]);
        const double* p1 = W(gxpos) + 3 * g1; const double* p2 = W(gxpos) + 3 * g2;
        const double* m1 = W(gxmat) + 9 * g1; const double* m2 = W(gxmat) + 9 * g2;
        double dif[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
        double s1[3], s2[3];
        double rb1, rb2;
        if (gc) { rb1 = W(grb)[g1]; rb2 = W(grb)[g2]; }      // sizes: only boxes that pass the sphere test need them (below)
        else { rb1 = geom_size_of(c, g1, s1); rb2 = geom_size_of(c, g2, s2); }
        if (t1 == BMJ_GEOM_PLANE) {
          double nr[3] = {m1[2], m1[5], m1[8]};
          keep = dot3(dif, nr) <= rb2 + margin;
        } else {
          double bound = rb1 + rb2 + margin;
          keep = dot3(dif, dif) <= bound * bound;
          // boxes (corridor walls: long, thin, with a bounding sphere that reaches most of the walker): the other geom's
          // bounding sphere against the box's slabs, in the box frame — conservative, so the contact set is unchanged
          if (keep && t2 == BMJ_GEOM_BOX) {
            if (gc) geom_size_of(c, g2, s2);
            double loc[3]; matT_vec(loc, m2, dif);
            const double r = rb1 + margin;
            keep = fabs(loc[0]) <= s2[0] + r && fabs(loc[1]) <= s2[1] + r && fabs(loc[2]) <= s2[2] + r;
          }
          if (keep && t1 == BMJ_GEOM_BOX) {
            if (gc) geom_size_of(c, g1, s1);
            double loc[3]; matT_vec(loc, m1, dif);
            const double r = rb2 + margin;
            keep = fabs(loc[0]) <= s1[0] + r && fabs(loc[1]) <= s1[1] + r && fabs(loc[2]) <= s1[2] + r;
          }
        }
      }
      const unsigned bal = __ballot_sync(FULL, keep);
      if (keep) queue[qn + __popc(bal & ((1u << lane) - 1))] = p;
      qn += __popc(bal);
      base += 32;
    }
    __syncwarp();
    const int take = qn < 32 ? qn : 32;
    int n = 0, g1 = 0, g2 = 0;
    bool mpr_lane = false;      // this lane's pair has no closed form: resolved below by the whole warp (cvx_pair_warp)
    if (lane < take) {
      const int p = queue[lane];
      g1 = m.pair_geom1[p]; g2 = m.pair_geom2[p];
      const int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
      if constexpr (CVX) mpr_lane = m.cvx_warp && pair_is_mpr(t1, t2);
      if (mpr_lane) { STG_TAN(0) = 0; STG_TAN(1) = 0; STG_TAN(2) = 0; }
      else {
        const double margin = fmax(m.geom_margin[g1], m.geom_margin[g2]);
        double s1[3], s2[3];
        geom_size_of(c, g1, s1); geom_size_of(c, g2, s2);
        n = narrowphase<CVX>(stg, t1, t2, margin, W(gxpos) + 3 * g1, W(gxmat) + 9 * g1, s1, W(gxpos) + 3 * g2, W(gxmat) + 9 * g2, s2);
      }
    }
    if constexpr (CVX) {
      unsigned todo = __ballot_sync(FULL, mpr_lane);
      _Pragma("unroll 1") while (todo) {
        const int src = first_bit(todo);
        todo &= todo - 1;
        const int a = __shfl_sync(FULL, g1, src), b = __shfl_sync(FULL, g2, src);
        const double margin = fmax(m.geom_margin[a], m.geom_margin[b]);
        double s1[3], s2[3], dist, cpos[3], cnrm[3];
        geom_size_of(c, a, s1); geom_size_of(c, b, s2);
        const int hit = cvx_pair_warp(lane, m.geom_type[a], W(gxpos) + 3 * a, W(gxmat) + 9 * a, s1, m.geom_type[b], W(gxpos) + 3 * b, W(gxmat) + 9 * b, s2,
                                      margin, &dist, cpos, cnrm);
        if (lane == src && hit) stage_contact(stg, n, dist, cpos, cnrm);
      }
    }
    // the queue's remainder moves to the front
    const int rest = qn - take;
    const int moved = lane < rest ? queue[take + lane] : 0;
    __syncwarp();
    if (lane < rest) queue[lane] = moved;
    qn = rest;
    int total;
    int off = warp_excl_scan(n, lane, &total);
    if (total == 0) continue;
    _Pragma("unroll 1") for (int k = 0; k < n; k++) {
      int idx = ncon + off + k;
      if (idx >= m.nconmax) continue;
      double* rec = W(con) + idx * CON_STRIDE;
      rec[0] = STG(k, 0);
      double nrm[3], tan[3];
      for (int i = 0; i < 3; i++) { rec[1 + i] = STG(k, 1 + i); nrm[i] = STG(k, 4 + i); tan[i] = STG_TAN(i); }
      make_frame(rec + 4, nrm, tan);
      int pr1 = m.geom_priority[g1], pr2 = m.geom_priority[g2];
      int condim; double mu;
      if (pr1 != pr2) { int gp = pr1 > pr2 ? g1 : g2; condim = m.geom_condim[gp]; mu = m.geom_friction[3 * gp]; }
      else { condim = max(m.geom_condim[g1], m.geom_condim[g2]); mu = fmax(m.geom_friction[3 * g1], m.geom_friction[3 * g2]); }
      rec[13] = mu;
      int* ii = con_ints(rec);
      ii[0] = g1; ii[1] = g2; ii[2] = condim; ii[3] = -1;
    }
    ncon += total;
    if (ncon > m.nconmax) { ncon = m.nconmax; *warn_contactfull = 1; break; }
  }
  __syncwarp();
  return ncon;
}

// ------------------------------------------------------------------------------------------------
// constraint rows: Jacobian, regulariser D = 1/R and reference acceleration, fused
// ------------------------------------------------------------------------------------------------
struct RowPrm { double R, aref; };
// impedance d(r), stiffness/damping from solref, regulariser R and reference acceleration for one row
__device__ __noinline__ RowPrm row_params_raw(double sr0, double sr1, double si0, double si1, double si2, double si3, double si4,
                                              double pos, double margin, double diag, double vel, double timestep, int refsafe) {
  double d0 = clampd(si0, BMJ_MINIMP, BMJ_MAXIMP), dmax = clampd(si1, BMJ_MINIMP, BMJ_MAXIMP);
  double width = fmax(BMJ_MINVAL, si2), mid = clampd(si3, BMJ_MINIMP, BMJ_MAXIMP), power = fmax(1.0, si4);
  double x = fabs(pos - margin) / width, imp;
  if (x >= 1) imp = dmax;
  else if (x <= 0) imp = d0;
  else {
    double y;
    if (power == 1) y = x;
    else if (x <= mid) y = pow(x / mid, power) * mid;
    else y = 1 - pow((1 - x) / (1 - mid), power) * (1 - mid);
    imp = d0 + y * (dmax - d0);
  }
  double K, B;
  if (sr0 > 0) {
    double tc = sr0, dr = sr1;
    if (refsafe) tc = fmax(tc, 2 * timestep);
    K = 1 / fmax(BMJ_MINVAL, dmax * dmax * tc * tc * dr * dr);
    B = 2 / fmax(BMJ_MINVAL, dmax * tc);
  } else { K = -sr0 / fmax(BMJ_MINVAL, dmax * dmax); B = -sr1 / fmax(BMJ_MINVAL, dmax); }
  RowPrm r;
  r.R = fmax(BMJ_MINVAL, (1 - imp) * diag / imp);
  r.aref = -B * vel - K * imp * (pos - margin);
  return r;
}
__device__ __forceinline__ void row_params(const Ctx& c, const double* solref, const double* solimp, double pos, double margin,
                                           double diag, double vel, double* R, double* aref, double* imp_out) {
  RowPrm r = row_params_raw(solref[0], solref[1], solimp[0], solimp[1], solimp[2], solimp[3], solimp[4], pos, margin, diag, vel,
                            c.m.timestep, !(c.disableflags & BMJ_DSBL_REFSAFE));
  *R = r.R; *aref = r.aref; *imp_out = 0;
}

__device__ __forceinline__ int make_constraint(const Ctx& c, int ncon, int* warn_cnstrfull) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  double* J = c.pJ; double* qvel = W(qvel);
  int nefc = 0;
  if (c.disableflags & BMJ_DSBL_CONSTRAINT) return 0;
  // ---- equality (all lanes build one row at a time) ----
  if (!(c.disableflags & BMJ_DSBL_EQUALITY)) {
    _Pragma("unroll 1") for (int e = 0; e < m.neq; e++) {
      if (!m.eq_active0[e]) continue;
      if (nefc >= m.njmax) { *warn_cnstrfull = 1; return nefc; }
      const double* data = m.eq_data + 11 * e;
      int o1 = m.eq_obj1id[e], o2 = m.eq_obj2id[e], et = m.eq_type[e];
      double pos, diag, deriv = 0;
      if (et == BMJ_EQ_TENDON) {
        pos = W(tenlen)[o1] - m.tendon_length0[o1]; diag = m.tendon_invweight0[o1];
        if (o2 >= 0) {
          double dif = W(tenlen)[o2] - m.tendon_length0[o2];
          pos -= data[0] + data[1]*dif + data[2]*dif*dif + data[3]*dif*dif*dif + data[4]*dif*dif*dif*dif;
          deriv = data[1] + 2*data[2]*dif + 3*data[3]*dif*dif + 4*data[4]*dif*dif*dif;
          diag += m.tendon_invweight0[o2];
        } else pos -= data[0];
      } else {  // joint
        int qa1 = m.jnt_qposadr[o1];
        pos = W(qpos)[qa1] - m.qpos0[qa1]; diag = m.dof_invweight0[m.jnt_dofadr[o1]];
        if (o2 >= 0) {
          int qa2 = m.jnt_qposadr[o2];
          double dif = W(qpos)[qa2] - m.qpos0[qa2];
          pos -= data[0] + data[1]*dif + data[2]*dif*dif + data[3]*dif*dif*dif + data[4]*dif*dif*dif*dif;
          deriv = data[1] + 2*data[2]*dif + 3*data[3]*dif*dif + 4*data[4]*dif*dif*dif;
          diag += m.dof_invweight0[m.jnt_dofadr[o2]];
        } else pos -= data[0];
      }
      double part = 0;
      FOR_LANES(i, nv) {
        double v;
        if (et == BMJ_EQ_TENDON) v = W(tenJ)[o1 * ld + i] - (o2 >= 0 ? deriv * W(tenJ)[o2 * ld + i] : 0.0);
        else v = (i == m.jnt_dofadr[o1] ? 1.0 : 0.0) - ((o2 >= 0 && i == m.jnt_dofadr[o2]) ? deriv : 0.0);
        J[nefc * ld + i] = v;
        part += v * qvel[i];
      }
      double vel = warp_sum(part), R, aref, imp;
      row_params(c, m.eq_solref + 2 * e, m.eq_solimp + 5 * e, pos, 0.0, diag, vel, &R, &aref, &imp);
      if (lane == 0) { c.pD[nefc] = 1 / R; c.pAref[nefc] = aref; c.pEq[nefc] = 1; }
      nefc++;
    }
  }
  __syncwarp();
  // ---- joint limits (one lane per joint; ordered compaction) ----
  if (!(c.disableflags & BMJ_DSBL_LIMIT)) {
    _Pragma("unroll 1") for (int base = 0; base < m.njnt; base += 32) {
      int j = base + lane;
      int cnt = 0; double dist[2]; int side[2];
      if (j < m.njnt && m.jnt_limited[j]) {
        int t = m.jnt_type[j];
        if (t == BMJ_JNT_SLIDE || t == BMJ_JNT_HINGE) {
          double value = W(qpos)[m.jnt_qposadr[j]], margin = m.jnt_margin[j];
          for (int s = -1; s <= 1; s += 2) {
            double d = s * (m.jnt_range[2 * j + (s + 1) / 2] - value);
            if (d < margin) { dist[cnt] = d; side[cnt] = s; cnt++; }
          }
        }
      }
      int total, off = warp_excl_scan(cnt, lane, &total);
      _Pragma("unroll 1") for (int k = 0; k < cnt; k++) {
        int r = nefc + off + k;
        if (r >= m.njmax) continue;
        int da = m.jnt_dofadr[j];
        double* row = J + r * ld;
        _Pragma("unroll 1") for (int i = 0; i < nv; i++) row[i] = 0;
        row[da] = -side[k];
        double vel = -side[k] * qvel[da], R, aref, imp;
        row_params(c, m.jnt_solref + 2 * j, m.jnt_solimp + 5 * j, dist[k], m.jnt_margin[j], m.dof_invweight0[da], vel, &R, &aref, &imp);
        c.pD[r] = 1 / R; c.pAref[r] = aref; c.pEq[r] = 0;
      }
      nefc += total;
      if (nefc > m.njmax) { nefc = m.njmax; *warn_cnstrfull = 1; return nefc; }
    }
  }
  __syncwarp();
  // ---- contacts (lanes = dofs) ----
  _Pragma("unroll 1") for (int ci = 0; ci < ncon; ci++) {
    double* rec = W(con) + ci * CON_STRIDE;
    int* ii = con_ints(rec);
    int g1 = ii[0], g2 = ii[1], dim = ii[2];
    double margin = fmax(m.geom_margin[g1], m.geom_margin[g2]), gap = fmax(m.geom_gap[g1], m.geom_gap[g2]);
    double includemargin = margin - gap, dist = rec[0];
    if (dist >= includemargin) continue;
    int nrow = dim == 1 ? 1 : 4;   // condim 1 or 3 (pyramidal); model_create rejects 4/6
    if (nefc + nrow > m.njmax) { *warn_cnstrfull = 1; break; }
    int b1 = m.geom_bodyid[g1], b2 = m.geom_bodyid[g2];
    double pos[3] = {rec[1], rec[2], rec[3]};
    double fr[9];
    for (int i = 0; i < 9; i++) fr[i] = rec[4 + i];
    double mu = rec[13];
    double off1[3], off2[3];
    int r1 = m.body_rootid[b1], r2 = m.body_rootid[b2];
    for (int i = 0; i < 3; i++) { off1[i] = pos[i] - W(scom)[3 * r1 + i]; off2[i] = pos[i] - W(scom)[3 * r2 + i]; }
    double pv[3] = {0, 0, 0};
    _Pragma("unroll 1") for (int i = lane; i < nv; i += 32) {
      unsigned w1 = (unsigned)m.body_dofmask[2 * b1 + (i >> 5)], w2 = (unsigned)m.body_dofmask[2 * b2 + (i >> 5)];
      bool in1 = (w1 >> (i & 31)) & 1, in2 = (w2 >> (i & 31)) & 1;
      double jd[3] = {0, 0, 0};
      if (in1 || in2) {
        const double* cd = W(cdof) + 6 * i;
        double tmp[3];
        if (in2) { cross3(tmp, cd, off2); for (int k = 0; k < 3; k++) jd[k] += cd[3 + k] + tmp[k]; }
        if (in1) { cross3(tmp, cd, off1); for (int k = 0; k < 3; k++) jd[k] -= cd[3 + k] + tmp[k]; }
      }
      double jn = dot3(fr, jd);
      if (dim == 1) { J[nefc * ld + i] = jn; pv[0] += jn * qvel[i]; }
      else {
        double jt1 = dot3(fr + 3, jd), jt2 = dot3(fr + 6, jd);
        J[nefc * ld + i] = jn + mu * jt1; J[(nefc + 1) * ld + i] = jn - mu * jt1;
        J[(nefc + 2) * ld + i] = jn + mu * jt2; J[(nefc + 3) * ld + i] = jn - mu * jt2;
        pv[0] += jn * qvel[i]; pv[1] += jt1 * qvel[i]; pv[2] += jt2 * qvel[i];
      }
    }
    double vn = warp_sum(pv[0]);
    // contact parameter mixing (solref / solimp)
    double solref[2], solimp[5];
    int pr1 = m.geom_priority[g1], pr2 = m.geom_priority[g2];
    if (pr1 != pr2) {
      int gp = pr1 > pr2 ? g1 : g2;
      for (int i = 0; i < 2; i++) solref[i] = m.geom_solref[2 * gp + i];
      for (int i = 0; i < 5; i++) solimp[i] = m.geom_solimp[5 * gp + i];
    } else {
      double s1 = m.geom_solmix[g1], s2 = m.geom_solmix[g2], mix;
      if (s1 >= BMJ_MINVAL && s2 >= BMJ_MINVAL) mix = s1 / (s1 + s2);
      else if (s1 < BMJ_MINVAL && s2 < BMJ_MINVAL) mix = 0.5;
      else if (s1 < BMJ_MINVAL) mix = 0.0; else mix = 1.0;
      if (m.geom_solref[2 * g1] > 0 && m.geom_solref[2 * g2] > 0)
        for (int i = 0; i < 2; i++) solref[i] = mix * m.geom_solref[2 * g1 + i] + (1 - mix) * m.geom_solref[2 * g2 + i];
      else
        for (int i = 0; i < 2; i++) solref[i] = fmin(m.geom_solref[2 * g1 + i], m.geom_solref[2 * g2 + i]);
      for (int i = 0; i < 5; i++) solimp[i] = mix * m.geom_solimp[5 * g1 + i] + (1 - mix) * m.geom_solimp[5 * g2 + i];
    }
    double tran = m.body_invweight0[2 * b1] + m.body_invweight0[2 * b2];
    if (dim == 1) {
      double R, aref, imp;
      row_params(c, solref, solimp, dist, includemargin, tran, vn, &R, &aref, &imp);
      if (lane == 0) { c.pD[nefc] = 1 / R; c.pAref[nefc] = aref; c.pEq[nefc] = 0; }
    } else {
      double vt1 = warp_sum(pv[1]), vt2 = warp_sum(pv[2]);
      double mureg = mu / sqrt(fmax(BMJ_MINVAL, m.impratio));
      if (lane < 4) {
        double vel = vn + ((lane & 1) ? -mu : mu) * (lane < 2 ? vt1 : vt2);
        double R, aref, imp;
        // every edge: same pos / margin / diagApprox (tran + mu^2 tran); shared R_py = 2 mu^2 R(first edge)
        row_params(c, solref, solimp, dist, includemargin, tran + mu * mu * tran, vel, &R, &aref, &imp);
        double Rpy = fmax(BMJ_MINVAL, 2 * mureg * mureg * R);
        c.pD[nefc + lane] = 1 / Rpy; c.pAref[nefc + lane] = aref; c.pEq[nefc + lane] = 0;
      }
    }
    if (lane == 0) ii[3] = nefc;
    nefc += nrow;
  }
  __syncwarp();
  return nefc;
}

// ------------------------------------------------------------------------------------------------
// velocity stage: cvel, cdof_dot, passive forces, RNE bias
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fwd_velocity(const Ctx& c) {
  const DevModel& m = c.m; int lane = c.lane;
  double* cvel = W(cvel); double* cacc = W(cacc); double* cfrc = W(cfrc); double* qvel = W(qvel);
  if (lane < 6) {   // world body: zero velocity / force; gravity enters as a base acceleration (one writer per element)
    cvel[lane] = 0; cfrc[lane] = 0;
    cacc[lane] = (lane >= 3 && !(c.disableflags & BMJ_DSBL_GRAVITY)) ? -m.gravity[lane - 3] : 0.0;
  }
  __syncwarp();
  _Pragma("unroll 1") for (int l = 1; l < m.nlevel; l++) {
    int a0 = m.level_adr[l], a1 = m.level_adr[l + 1];
    _Pragma("unroll 1") for (int k = a0 + lane; k < a1; k += 32) {
      int b = m.level_body[k], p = m.body_parentid[b];
      double cv[6], ca[6];
      for (int i = 0; i < 6; i++) { cv[i] = cvel[6 * p + i]; ca[i] = cacc[6 * p + i]; }
      int j0 = m.body_jntadr[b], jn = m.body_jntnum[b];
      _Pragma("unroll 1") for (int j = j0; j < j0 + jn; j++) {
        int da = m.jnt_dofadr[j], t = m.jnt_type[j];
        double* cdd = W(cdofdot); const double* cd = W(cdof);
        if (t == BMJ_JNT_FREE) {
          for (int i = 0; i < 18; i++) cdd[6 * da + i] = 0;
          for (int q = 0; q < 3; q++) for (int i = 0; i < 6; i++) cv[i] += cd[6 * (da + q) + i] * qvel[da + q];
          da += 3;
        }
        if (t == BMJ_JNT_FREE || t == BMJ_JNT_BALL) {
          for (int q = 0; q < 3; q++) { double r[6]; cross_motion(r, cv, cd + 6 * (da + q)); for (int i = 0; i < 6; i++) cdd[6 * (da + q) + i] = r[i]; }
          for (int q = 0; q < 3; q++) for (int i = 0; i < 6; i++) cv[i] += cd[6 * (da + q) + i] * qvel[da + q];
        } else {
          double r[6]; cross_motion(r, cv, cd + 6 * da);
          for (int i = 0; i < 6; i++) { cdd[6 * da + i] = r[i]; cv[i] += cd[6 * da + i] * qvel[da]; }
        }
      }
      int d0 = m.body_dofadr[b], dn = m.body_dofnum[b];
      _Pragma("unroll 1") for (int q = d0; q < d0 + dn; q++) for (int i = 0; i < 6; i++) ca[i] += W(cdofdot)[6 * q + i] * qvel[q];
      for (int i = 0; i < 6; i++) { cvel[6 * b + i] = cv[i]; cacc[6 * b + i] = ca[i]; }
    }
    __syncwarp();
  }
  // body forces for all bodies at once (lanes = bodies) rather than inside the level loop, where few lanes are busy
  FOR_LANES(b, m.nbody) {
    if (b == 0) continue;
    double t1[6], t2[6], t3[6];
    mul_inert_vec(t1, W(cinert) + 10 * b, cacc + 6 * b);
    mul_inert_vec(t2, W(cinert) + 10 * b, cvel + 6 * b);
    cross_force(t3, cvel + 6 * b, t2);
    for (int i = 0; i < 6; i++) cfrc[6 * b + i] = t1[i] + t3[i];
  }
  __syncwarp();
  tree_accumulate(c, cfrc, 6, false);
  FOR_LANES(k, m.nv) {
    int b = m.dof_bodyid[k];
    double s = 0;
    for (int i = 0; i < 6; i++) s += W(cdof)[6 * k + i] * cfrc[6 * b + i];
    c.pBias[k] = s;
    double ps = 0;
    if (!(c.disableflags & BMJ_DSBL_PASSIVE)) {
      int j = m.dof_jntid[k], t = m.jnt_type[j];
      if ((t == BMJ_JNT_SLIDE || t == BMJ_JNT_HINGE) && m.jnt_stiffness[j] != 0) {
        int qa = m.jnt_qposadr[j];
        ps -= m.jnt_stiffness[j] * (W(qpos)[qa] - m.qpos_spring[qa]);
      }
      ps -= m.dof_damping[k] * qvel[k];
    }
    c.pPassive[k] = ps;
  }
  __syncwarp();
}

__device__ __forceinline__ void subtree_vel(const Ctx& c) {
  const DevModel& m = c.m; int lane = c.lane;
  double* sl = W(slinvel);
  FOR_LANES(b, m.nbody) {
    int root = m.body_rootid[b];
    double dif[3], tmp[3];
    for (int i = 0; i < 3; i++) dif[i] = W(xipos)[3 * b + i] - W(scom)[3 * root + i];
    cross3(tmp, dif, W(cvel) + 6 * b);
    for (int i = 0; i < 3; i++) sl[3 * b + i] = m.body_mass[b] * (W(cvel)[6 * b + 3 + i] - tmp[i]);
  }
  __syncwarp();
  tree_accumulate(c, sl, 3, true);
  FOR_LANES(b, m.nbody) { double sm = fmax(BMJ_MINVAL, m.body_subtreemass[b]); for (int i = 0; i < 3; i++) sl[3 * b + i] /= sm; }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// acceleration stage
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fwd_actuation(const Ctx& c) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  bool off = c.disableflags & BMJ_DSBL_ACTUATION;
  FOR_LANES(a, m.nu) {
    double force = 0;
    int aa = m.actuator_actadr[a];
    if (aa >= 0) W(actdot)[aa] = 0;
    if (!off) {
      double ctrl = W(ctrl)[a];
      if (m.actuator_ctrllimited[a] && !(c.disableflags & BMJ_DSBL_CLAMPCTRL))
        ctrl = clampd(ctrl, m.actuator_ctrlrange[2 * a], m.actuator_ctrlrange[2 * a + 1]);
      double input = ctrl;
      int dt = m.actuator_dyntype[a];
      if (dt == BMJ_DYN_INTEGRATOR) { W(actdot)[aa] = ctrl; input = W(act)[aa]; }
      else if (dt == BMJ_DYN_FILTER) { double tau = fmax(BMJ_MINVAL, m.actuator_dynprm[a]); W(actdot)[aa] = (ctrl - W(act)[aa]) / tau; input = W(act)[aa]; }
      double gear = m.actuator_gear[a], length, velocity;
      if (m.actuator_trntype[a] == BMJ_TRN_JOINT) {
        int j = m.actuator_trnid[a];
        length = gear * W(qpos)[m.jnt_qposadr[j]]; velocity = gear * W(qvel)[m.jnt_dofadr[j]];
      } else {
        int t = m.actuator_trnid[a];
        length = gear * W(tenlen)[t];
        double s = 0; _Pragma("unroll 1") for (int i = 0; i < nv; i++) s += gear * W(tenJ)[t * ld + i] * W(qvel)[i];
        velocity = s;
      }
      const double* gp = m.actuator_gainprm + 3 * a; const double* bp = m.actuator_biasprm + 3 * a;
      double gain = gp[0];
      if (m.actuator_gaintype[a] == BMJ_GAIN_AFFINE) gain += gp[1] * length + gp[2] * velocity;
      double bias = 0;
      if (m.actuator_biastype[a] == BMJ_BIAS_AFFINE) bias = bp[0] + bp[1] * length + bp[2] * velocity;
      force = gain * input + bias;
      if (m.actuator_forcelimited[a]) force = clampd(force, m.actuator_forcerange[2 * a], m.actuator_forcerange[2 * a + 1]);
    }
    W(actforce)[a] = force;
  }
  __syncwarp();
  // qfrc_actuator = moment^T force: the nonzero moment arms of every dof in actuator order (same summation order
  // as the dense nu-loop this replaces; the skipped terms are exact zeros)
  FOR_LANES(i, nv) {
    double s = 0;
    const int a0 = m.dof_act_adr[i], a1 = m.dof_act_adr[i + 1];
    _Pragma("unroll 1") for (int k = a0; k < a1; k++) s += m.dof_act_coef[k] * W(actforce)[m.dof_act_id[k]];
    W(qfact)[i] = s;
  }
  __syncwarp();
}

template <int NVT>
__device__ __forceinline__ void fwd_acceleration(const Ctx& c, const b200mj_io& io, int env) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv;
  FOR_LANES(i, nv) {
    double s = W(passive)[i] - W(bias)[i] + W(qfact)[i];
    if (io.qfrc_applied) s += io.qfrc_applied[(size_t)env * nv + i];
    W(smooth)[i] = s;
  }
  if (io.xfrc_applied) {
    _Pragma("unroll 1") for (int b = 1; b < m.nbody; b++) {
      const double* xf = io.xfrc_applied + ((size_t)env * m.nbody + b) * 6;
      double f[6]; bool any = false;
      for (int i = 0; i < 6; i++) { f[i] = xf[i]; any |= (f[i] != 0); }
      if (!any) continue;
      int root = m.body_rootid[b];
      double off[3];
      for (int i = 0; i < 3; i++) off[i] = W(xipos)[3 * b + i] - W(scom)[3 * root + i];
      FOR_LANES(i, nv) {
        unsigned w = (unsigned)m.body_dofmask[2 * b + (i >> 5)];
        if (!((w >> (i & 31)) & 1)) continue;
        const double* cd = W(cdof) + 6 * i;
        double tmp[3]; cross3(tmp, cd, off);
        double s = 0;
        for (int k = 0; k < 3; k++) s += (cd[3 + k] + tmp[k]) * f[k] + cd[k] * f[3 + k];
        W(smooth)[i] += s;
      }
    }
  }
  __syncwarp();
  // factor M into the H buffer (free until the Newton solver assembles its Hessian there)
  if constexpr (NVT > 0) {
    tn_factor<NVT>(W(M), W(H), W(dinv), lane, W(smooth), W(qaccs), W(J), W(efcSD), reinterpret_cast<const int*>(W(actlist)), opaque_zero(), W(colbuf));
    tn_back<NVT>(W(H), W(dinv), W(qaccs), W(qaccs), lane, 0);
  } else {
    if (c.L.dual) {
      chol_factor(c.Mc, W(H), W(dinv), nv, lane, nullptr, nullptr);      // qacc_smooth: one more right-hand side of dual_prepare's substitution pass
    } else {
      chol_factor(c.Mc, W(H), W(dinv), nv, lane, W(smooth), W(qaccs));
      chol_back(W(H), W(dinv), W(qaccs), W(qaccs), nv, lane);
    }
  }
}

// --- Newton solver ---------------------------------------------------------------------------------
struct Primal { double cost, gauss; int nact, changed; };

// Ma = M qacc ; jar = J qacc - aref
template <int NVT>
__device__ __forceinline__ void compute_Ma_jar(const Ctx& c, int nefc) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  if constexpr (NVT > 0) {
    if (lane < NVT) W(Ma)[lane] = tn_symv_row<NVT>(W(M), W(qacc), lane);
    FOR_LANES(r, nefc) W(jar)[r] = tn_dot_row<NVT>(W(J) + r * ld, W(qacc)) - W(aref)[r];
  } else {
    FOR_LANES(i, nv) W(Ma)[i] = symv_row(c.Mc, W(qacc), nv, i);
    FOR_LANES(r, nefc) W(jar)[r] = dot_rows(W(J) + r * ld, W(qacc), nv) - W(aref)[r];
  }
  __syncwarp();
}

__device__ __forceinline__ Primal constraint_update(const Ctx& c, int nefc) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  const int* eqf = reinterpret_cast<const int*>(W(eqflag));
  int* alist = reinterpret_cast<int*>(W(actlist));
  double cpart = 0;
  int nact = 0, changed = 0;
  _Pragma("unroll 1") for (int base = 0; base < nefc; base += 32) {
    int r = base + lane;
    bool act = false;
    if (r < nefc) {
      double jar = W(jar)[r], D = W(efcD)[r];
      act = eqf[r] || jar < 0;
      changed |= ((W(efcSD)[r] != 0.0) != act);
      W(efcSD)[r] = act ? D : 0.0;
      W(force)[r] = act ? -D * jar : 0.0;
      if (act) cpart += 0.5 * D * jar * jar;
    }
    unsigned bal = __ballot_sync(FULL, act);
    if (act) alist[nact + __popc(bal & ((1u << lane) - 1))] = r;
    nact += __popc(bal);
  }
  __syncwarp();
  double gpart = 0;
  FOR_LANES(i, nv) {
    double s = 0;
    _Pragma("unroll 1") for (int a = 0; a < nact; a++) { int r = alist[a]; s += W(J)[r * ld + i] * W(force)[r]; }
    W(qcon)[i] = s;
    gpart += (W(Ma)[i] - W(smooth)[i]) * (W(qacc)[i] - W(qaccs)[i]);
  }
  Primal p;
  p.gauss = 0.5 * warp_sum(gpart);
  p.cost = warp_sum(cpart) + p.gauss;
  p.nact = nact;
  p.changed = __any_sync(FULL, changed);
  __syncwarp();
  return p;
}

// --- dual form of the Newton direction (c.L.dual) --------------------------------------------------------------------
// The Hessian of the primal problem is H = M + J_a' D_a J_a over the active rows a. With few rows and many dofs the
// Woodbury identity gives the same direction from an nact x nact system instead of an nv x nv factorisation:
//   H^-1 g = u - V_a' (R_a + A_aa)^-1 J_a u,   u = M^-1 g = qacc - qacc_smooth - V' force,
//   V = J M^-1 (rows, computed once per physics step from chol(M)),  A = J M^-1 J',  R = 1 / D.
// The CMU humanoid (nv = 62) has ~10 rows in a typical step and the Newton solver refactors on almost every iteration:
// ~3.5 factorisations of 62 x 62 per physics step become one eight-at-a-time substitution pass and 3.5 factorisations
// of ~5 x 5. Same iterates as the primal form up to rounding (tests/test_gpu_parity.py, tests/test_emu_kernel_parity.py).
__device__ __forceinline__ void dual_prepare(const Ctx& c, int nefc) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  const double* Jsrc = c.L.jalias ? c.Jg : W(J);
  chol_solve_multi(W(H), W(dinv), nv, Jsrc, W(dV), ld, nefc, lane, W(smooth), W(qaccs));      // + qacc_smooth (fwd_acceleration left it to this pass)
  if (nefc == 0) return;
  if (c.L.jalias) { copy_row(W(J), c.Jg, nefc * ld, lane); __syncwarp(); }      // over the factor of M, which nothing reads any more
  double* A = W(dS);                                                    // may alias H: chol(M) is dead from here on
  _Pragma("unroll 1") for (int r = 0; r < nefc; r++) {
    if (lane <= r) { const double a = dot_rows(W(J) + r * ld, W(dV) + lane * ld, nv); A[r * nefc + lane] = a; A[lane * nefc + r] = a; }
  }
  __syncwarp();
}

// search = -H^-1 grad through the dual form (grad: newton_gradient)
__device__ __forceinline__ void newton_direction_dual(const Ctx& c, int nefc, int nact, bool refactor) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  const int* alist = reinterpret_cast<const int*>(W(actlist));
  double* A = W(dS); double* S = A + nefc * nefc; double* sdinv = S + tri(c.L.drows); double* t = sdinv + c.L.drows; double* y = t + c.L.drows;
  FOR_LANES(i, nv) {
    double u0 = W(qacc)[i] - W(qaccs)[i], u1 = 0;
    int a = 0;
    _Pragma("unroll 1") for (; a + 2 <= nact; a += 2) { const int r0 = alist[a], r1 = alist[a + 1]; u0 -= W(dV)[r0 * ld + i] * W(force)[r0]; u1 -= W(dV)[r1 * ld + i] * W(force)[r1]; }
    if (a < nact) { const int r0 = alist[a]; u0 -= W(dV)[r0 * ld + i] * W(force)[r0]; }
    W(tmpv)[i] = u0 + u1;
  }
  __syncwarp();
  if (nact > 0) {
    FOR_LANES(a, nact) t[a] = dot_rows(W(J) + alist[a] * ld, W(tmpv), nv);
    if (refactor) {
      FOR_LANES(a, nact) {
        const int ra = alist[a]; const double* Ar = A + ra * nefc; double* Sa = S + tri(a);
        _Pragma("unroll 1") for (int b = 0; b < a; b++) Sa[b] = Ar[alist[b]];
        Sa[a] = Ar[ra] + 1.0 / W(efcD)[ra];
      }
      __syncwarp();
      chol_factor(S, S, sdinv, nact, lane, t, y);
    } else { __syncwarp(); chol_forward(S, sdinv, t, y, nact, lane); }
    chol_back(S, sdinv, y, y, nact, lane);
  }
  // search = -(u - V_a' y), and M search = -(M u - J_a' y) = -(grad - J_a' y) for free: the line search needs no product with M
  FOR_LANES(i, nv) {
    double s0 = W(tmpv)[i], s1 = 0, m0 = W(grad)[i], m1 = 0;
    int a = 0;
    _Pragma("unroll 1") for (; a + 2 <= nact; a += 2) {
      const int r0 = alist[a], r1 = alist[a + 1];
      s0 -= W(dV)[r0 * ld + i] * y[a]; s1 -= W(dV)[r1 * ld + i] * y[a + 1];
      m0 -= W(J)[r0 * ld + i] * y[a]; m1 -= W(J)[r1 * ld + i] * y[a + 1];
    }
    if (a < nact) { const int r0 = alist[a]; s0 -= W(dV)[r0 * ld + i] * y[a]; m0 -= W(J)[r0 * ld + i] * y[a]; }
    W(search)[i] = -(s0 + s1); W(Mv)[i] = -(m0 + m1);
  }
  __syncwarp();
}

// (re)assemble H = M + J^T diag(SD) J and factor it only when the active set changed; search = -H^-1 grad.
// The gradient comes first and alone: the stopping tests need only its norm, so the trip that ends the iteration
// (one per physics step) skips the factorisation / substitutions of a direction nobody would use.
__device__ __forceinline__ double newton_gradient(const Ctx& c) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv;
  double gpart = 0;
  FOR_LANES(i, nv) { double g = W(Ma)[i] - W(smooth)[i] - W(qcon)[i]; W(grad)[i] = g; gpart += g * g; }
  const double gnorm = sqrt(warp_sum(gpart));
  __syncwarp();
  return gnorm;
}

template <int NVT>
__device__ __forceinline__ void newton_direction(const Ctx& c, int nefc, int nact, bool refactor) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  if constexpr (NVT == 0) { if (c.L.dual) { newton_direction_dual(c, nefc, nact, refactor); return; } }
  if constexpr (NVT > 0) {
    if (refactor) tn_factor<NVT>(W(M), W(H), W(dinv), lane, W(grad), W(search), W(J), W(efcSD), reinterpret_cast<const int*>(W(actlist)), nact, W(colbuf));
    else tn_forward<NVT>(W(H), W(dinv), W(grad), W(search), lane);
    tn_back<NVT>(W(H), W(dinv), W(search), W(search), lane, 1);
    return;
  }
  if (refactor) {
    const int* alist = reinterpret_cast<const int*>(W(actlist));
    // lane j owns column j (and j+32) of the lower triangle; rows in register blocks of 8
    _Pragma("unroll 1") for (int j = lane; j < nv; j += 32) {
      _Pragma("unroll 1") for (int i0 = (j & ~7); i0 < nv; i0 += 8) {
        double acc[8];
        const int t0 = tri(i0) + j;      // packed (i0 + q, j) sits at t0 + q * i0 + q (q + 1) / 2; rows above the diagonal are skipped
#pragma unroll
        for (int q = 0; q < 8; q++) acc[q] = (i0 + q < nv && i0 + q >= j) ? c.Mc[t0 + q * i0 + ((q * (q + 1)) >> 1)] : 0.0;
        _Pragma("unroll 1") for (int a = 0; a < nact; a++) {
          int r = alist[a];
          const double* Jr = W(J) + r * ld;
          double sj = W(efcSD)[r] * Jr[j];
#pragma unroll
          for (int q = 0; q < 8; q++) if (i0 + q < nv) acc[q] += Jr[i0 + q] * sj;
        }
#pragma unroll
        for (int q = 0; q < 8; q++) if (i0 + q < nv && i0 + q >= j) W(H)[t0 + q * i0 + ((q * (q + 1)) >> 1)] = acc[q];
      }
    }
    __syncwarp();
    chol_factor(W(H), W(H), W(dinv), nv, lane, W(grad), W(search));   // in place, forward substitution included
  } else chol_forward(W(H), W(dinv), W(grad), W(search), nv, lane);
  chol_back(W(H), W(dinv), W(search), W(search), nv, lane);
  FOR_LANES(i, nv) W(search)[i] = -W(search)[i];
  __syncwarp();
}

__device__ __forceinline__ void ls_eval(const Ctx& c, int nefc, double alpha, const double* qg, double* d1, double* d2) {
  int lane = c.lane;
  const int* eqf = reinterpret_cast<const int*>(W(eqflag));
  double q1 = 0, q2 = 0;
  FOR_LANES(r, nefc) {
    double jar = W(jar)[r], jv = W(jv)[r];
    double x = jar + alpha * jv;
    if (eqf[r] || x < 0) { double D = W(efcD)[r]; q1 += D * jar * jv; q2 += 0.5 * D * jv * jv; }
  }
  q1 = warp_sum(q1) + qg[1]; q2 = warp_sum(q2) + qg[2];
  *d1 = 2 * alpha * q2 + q1;
  *d2 = 2 * q2;
}

template <int NVT>
__device__ __forceinline__ double line_search(const Ctx& c, int nefc, const Primal& pr) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  double sp = 0;
  FOR_LANES(i, nv) sp += W(search)[i] * W(search)[i];
  double snorm = sqrt(warp_sum(sp));
  if (snorm < BMJ_MINVAL) return 0;
  double gtol = m.tolerance * m.ls_tolerance * snorm * (m.meaninertia * max(1, nv));
  double g1 = 0, g2 = 0;
  if constexpr (NVT > 0) {
    if (lane < NVT) {
      double s = tn_symv_row<NVT>(W(M), W(search), lane);
      W(Mv)[lane] = s;
      g1 += W(search)[lane] * (W(Ma)[lane] - W(smooth)[lane]); g2 += 0.5 * W(search)[lane] * s;
    }
    FOR_LANES(r, nefc) W(jv)[r] = tn_dot_row<NVT>(W(J) + r * ld, W(search));
  } else {
    const bool have_mv = c.L.dual != 0;      // the dual form of the direction delivers M search as well (newton_direction_dual)
    FOR_LANES(i, nv) {
      double s = have_mv ? W(Mv)[i] : symv_row(c.Mc, W(search), nv, i);
      W(Mv)[i] = s;
      g1 += W(search)[i] * (W(Ma)[i] - W(smooth)[i]); g2 += 0.5 * W(search)[i] * s;
    }
    FOR_LANES(r, nefc) W(jv)[r] = dot_rows(W(J) + r * ld, W(search), nv);
  }
  double qg[3] = {pr.gauss, warp_sum(g1), warp_sum(g2)};
  __syncwarp();
  double d1, d2;
  ls_eval(c, nefc, 0.0, qg, &d1, &d2);
  if (d1 >= 0 || d2 <= 0) return 0;
  double lo = 0, dlo = d1, hi = 0, dhi = 0; bool have_hi = false;
  double alpha = -d1 / d2, best = 0;
  _Pragma("unroll 1") for (int it = 0; it < m.ls_iterations; it++) {
    double e1, e2;
    ls_eval(c, nefc, alpha, qg, &e1, &e2);
    best = alpha;
    if (fabs(e1) < gtol) break;
    if (e1 < 0) { lo = alpha; dlo = e1; } else { hi = alpha; dhi = e1; have_hi = true; }
    double next = alpha - e1 / e2;
    if (have_hi) { if (!(next > lo && next < hi)) next = lo + (hi - lo) * (-dlo) / (dhi - dlo); }
    else if (next <= lo) next = 2 * alpha + 1e-12;
    if (next == alpha) break;
    alpha = next;
  }
  return best;
}

// CTA-wide phase alignment: all warps of a CTA run the same code region at the same time so that instruction
// lines are fetched from L2 once per CTA, not once per warp (the pass footprint is ~5x the 32 KB L1.5 I-cache).
// The fused and position kernels take these barriers at coarse points (pass start, stage boundaries around the solver)
// whenever a CTA holds more than one warp.
#define PHASE_SYNC() do { if (blockDim.x > 32) __syncthreads(); } while (0)

template <int NVT>
__device__ __forceinline__ int solve_newton(const Ctx& c, int nefc) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv;
  Primal pr; pr.cost = 0; pr.gauss = 0; pr.nact = 0; pr.changed = 1;
  const bool active = nefc > 0;
  if constexpr (NVT == 0) { if (c.L.dual) dual_prepare(c, nefc); }
  if (active) {
    // start point: the warm start if it has lower cost than the unconstrained acceleration (MuJoCo's rule).
    // candidates: 0 = qacc_warmstart, 1 = qacc_smooth, 2 = qacc_warmstart restored (only when it won)
    bool warm = !(c.disableflags & BMJ_DSBL_WARMSTART);
    double cost_warm = 0;
    _Pragma("unroll 1") for (int cand = warm ? 0 : 1; cand < 3; cand++) {
      if (cand == 0) {
        FOR_LANES(i, nv) W(qacc)[i] = W(qaccws)[i];
        __syncwarp();
        compute_Ma_jar<NVT>(c, nefc);
      } else if (cand == 1) {
        // park the warm-start products (Mv / jv are free until the first line search); for the unconstrained
        // candidate M qacc_smooth = qfrc_smooth by construction, so only J qacc_smooth is a product
        FOR_LANES(i, nv) { W(Mv)[i] = W(Ma)[i]; W(qacc)[i] = W(qaccs)[i]; W(Ma)[i] = W(smooth)[i]; }
        FOR_LANES(r, nefc) W(jv)[r] = W(jar)[r];
        __syncwarp();
        if constexpr (NVT > 0) { FOR_LANES(r, nefc) W(jar)[r] = tn_dot_row<NVT>(W(J) + r * m.ldv, W(qacc)) - W(aref)[r]; }
        else { FOR_LANES(r, nefc) W(jar)[r] = dot_rows(W(J) + r * m.ldv, W(qacc), nv) - W(aref)[r]; }
        __syncwarp();
      } else {
        if (!(warm && cost_warm < pr.cost)) break;
        FOR_LANES(i, nv) { W(qacc)[i] = W(qaccws)[i]; W(Ma)[i] = W(Mv)[i]; }
        FOR_LANES(r, nefc) W(jar)[r] = W(jv)[r];
        __syncwarp();
      }
      pr = constraint_update(c, nefc);
      if (cand == 0) cost_warm = pr.cost;
    }
  } else {
    FOR_LANES(i, nv) { W(qacc)[i] = W(qaccs)[i]; W(qcon)[i] = 0; }
    __syncwarp();
  }
  double scale = 1 / (m.meaninertia * max(1, nv));
  int iter = 0;
  bool refactor = true, done = !active;
  double oldcost = 0;
  while (true) {
    // every warp of the CTA takes the same number of trips: finished environments idle at the barrier
    if (c.newton_sync) { if (!__syncthreads_or(!done)) break; } else if (done) break;
    if (!done) {
      const double gnorm = newton_gradient(c);
      bool stop = false;
      if (iter > 0) {
        double improvement = scale * (oldcost - pr.cost), gradient = scale * gnorm;
        if (improvement < m.tolerance || gradient < m.tolerance) stop = true;
      }
      if (iter >= m.iterations) stop = true;
      double alpha = 0;
      if (!stop) { newton_direction<NVT>(c, nefc, pr.nact, refactor); alpha = line_search<NVT>(c, nefc, pr); if (alpha == 0) stop = true; }
      if (stop) done = true;
      else {
        FOR_LANES(i, nv) { W(qacc)[i] += alpha * W(search)[i]; W(Ma)[i] += alpha * W(Mv)[i]; }
        FOR_LANES(r, nefc) W(jar)[r] += alpha * W(jv)[r];
        __syncwarp();
        oldcost = pr.cost;
        pr = constraint_update(c, nefc);
        refactor = pr.changed != 0;
        iter++;
      }
    }
  }
  return iter;
}

// --- dual solver: projected Gauss-Seidel (mj_solPGS; oracle/mjoracle.cpp solve_pgs has the statement of the method) ----
// Runs in the fused kernel only (b200mj_step falls back to it for PGS models): the dense nefc x nefc matrix lives in
// the workspace. Rows are swept in order, one at a time, by the whole warp (lanes = columns of the row).
__device__ __forceinline__ int solve_pgs(const Ctx& c, int nefc) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv;
  if (nefc == 0) {
    FOR_LANES(i, nv) { W(qacc)[i] = W(qaccs)[i]; W(qcon)[i] = 0; }
    __syncwarp();
    return 0;
  }
  double* A = W(pgsA); double* X = W(pgsX); double* B = W(pgsB); double* f = W(force);
  const int* eqf = reinterpret_cast<const int*>(W(eqflag));
  // X_r = M^-1 J_r'  (W(H), W(dinv) hold the factor of M from fwd_acceleration)
  _Pragma("unroll 1") for (int r = 0; r < nefc; r++) {
    chol_forward(W(H), W(dinv), W(J) + r * ld, X + r * ld, nv, lane);
    chol_back(W(H), W(dinv), X + r * ld, X + r * ld, nv, lane);
  }
  _Pragma("unroll 1") for (int i = 0; i < nefc; i++) {
    FOR_LANES(j, nefc) A[i * nefc + j] = dot_rows(W(J) + i * ld, X + j * ld, nv) + (i == j ? 1.0 / W(efcD)[i] : 0.0);
  }
  FOR_LANES(r, nefc) B[r] = dot_rows(W(J) + r * ld, W(qaccs), nv) - W(aref)[r];
  __syncwarp();
  // warm start: forces implied by qacc_warmstart, kept only if their dual cost is negative
  if (!(c.disableflags & BMJ_DSBL_WARMSTART)) {
    FOR_LANES(r, nefc) {
      const double jar = dot_rows(W(J) + r * ld, W(qaccws), nv) - W(aref)[r];
      f[r] = (eqf[r] || jar < 0) ? -W(efcD)[r] * jar : 0.0;
    }
    __syncwarp();
    double part = 0;
    FOR_LANES(i, nefc) part += f[i] * (0.5 * dot_rows(A + i * nefc, f, nefc) + B[i]);
    const double cost = warp_sum(part);
    __syncwarp();
    if (cost > 0) { FOR_LANES(r, nefc) f[r] = 0; }
  } else { FOR_LANES(r, nefc) f[r] = 0; }
  __syncwarp();
  const double scale = 1 / (m.meaninertia * max(1, nv));
  int iter = 0;
  _Pragma("unroll 1") while (iter < m.iterations) {
    double improvement = 0;
    _Pragma("unroll 1") for (int i = 0; i < nefc; i++) {
      double part = 0;
      FOR_LANES(j, nefc) part += A[i * nefc + j] * f[j];
      const double res = B[i] + warp_sum(part);
      const double Aii = A[i * nefc + i], old = f[i];
      double fi = old - res / Aii;
      if (!eqf[i] && fi < 0) fi = 0;
      const double delta = fi - old;
      improvement -= 0.5 * delta * delta * Aii + delta * res;
      __syncwarp();
      if (lane == 0) f[i] = fi;
      __syncwarp();
    }
    iter++;
    if (improvement * scale < m.tolerance) break;
  }
  FOR_LANES(i, nv) {
    double sum = 0;
    _Pragma("unroll 1") for (int r = 0; r < nefc; r++) sum += W(J)[r * ld + i] * f[r];
    W(qcon)[i] = sum;
    W(tmpv)[i] = W(smooth)[i] + sum;
  }
  __syncwarp();
  chol_forward(W(H), W(dinv), W(tmpv), W(qacc), nv, lane);
  chol_back(W(H), W(dinv), W(qacc), W(qacc), nv, lane);
  return iter;
}

// cacc / cfrc_int with qacc + external contact forces (for accelerometer / force / torque sensors)
__device__ __forceinline__ void rne_post_constraint(const Ctx& c, const b200mj_io& io, int env, int ncon) {
  const DevModel& m = c.m; int lane = c.lane;
  double* cext = W(cfrcext); double* cacc = W(cacc); double* cint = W(cfrc);
  _Pragma("unroll 1") for (int i = lane; i < 6 * m.nbody; i += 32) cext[i] = 0;
  __syncwarp();
  if (io.xfrc_applied) {
    FOR_LANES(b, m.nbody) {
      if (b == 0) continue;
      const double* xf = io.xfrc_applied + ((size_t)env * m.nbody + b) * 6;
      int root = m.body_rootid[b];
      double dif[3], tq[3], f[3] = {xf[0], xf[1], xf[2]};
      for (int i = 0; i < 3; i++) dif[i] = W(xipos)[3 * b + i] - W(scom)[3 * root + i];
      cross3(tq, dif, f);
      for (int i = 0; i < 3; i++) { cext[6 * b + i] += xf[3 + i] + tq[i]; cext[6 * b + 3 + i] += f[i]; }
    }
    __syncwarp();
  }
  // contacts: serial over contacts (lane 0) keeps the accumulation order fixed
  if (lane == 0) {
    _Pragma("unroll 1") for (int ci = 0; ci < ncon; ci++) {
      double* rec = W(con) + ci * CON_STRIDE; int* ii = con_ints(rec);
      int adr = ii[3]; if (adr < 0) continue;
      double f[3] = {0, 0, 0}, mu = rec[13];
      if (ii[2] == 1) f[0] = W(force)[adr];
      else for (int k = 1; k < 3; k++) { double fp = W(force)[adr + 2 * (k - 1)], fn = W(force)[adr + 2 * (k - 1) + 1]; f[0] += fp + fn; f[k] = (fp - fn) * mu; }
      double fw[3]; matT_vec(fw, rec + 4, f);
      int bb[2] = {m.geom_bodyid[ii[0]], m.geom_bodyid[ii[1]]};
      for (int side = 0; side < 2; side++) {
        int b = bb[side]; if (b <= 0) continue;
        double sgn = side == 0 ? -1 : 1; int root = m.body_rootid[b];
        double dif[3], tq[3];
        for (int i = 0; i < 3; i++) dif[i] = rec[1 + i] - W(scom)[3 * root + i];
        cross3(tq, dif, fw);
        for (int i = 0; i < 3; i++) { cext[6 * b + i] += sgn * tq[i]; cext[6 * b + 3 + i] += sgn * fw[i]; }
      }
    }
  }
  if (lane < 6) {
    cint[lane] = 0;
    cacc[lane] = (lane >= 3 && !(c.disableflags & BMJ_DSBL_GRAVITY)) ? -m.gravity[lane - 3] : 0.0;
  }
  __syncwarp();
  _Pragma("unroll 1") for (int l = 1; l < m.nlevel; l++) {
    int a0 = m.level_adr[l], a1 = m.level_adr[l + 1];
    _Pragma("unroll 1") for (int k = a0 + lane; k < a1; k += 32) {
      int b = m.level_body[k], p = m.body_parentid[b];
      double ca[6];
      for (int i = 0; i < 6; i++) ca[i] = cacc[6 * p + i];
      int d0 = m.body_dofadr[b], dn = m.body_dofnum[b];
      _Pragma("unroll 1") for (int q = d0; q < d0 + dn; q++) for (int i = 0; i < 6; i++) ca[i] += W(cdofdot)[6 * q + i] * W(qvel)[q] + W(cdof)[6 * q + i] * W(qacc)[q];
      double t1[6], t2[6], t3[6];
      mul_inert_vec(t1, W(cinert) + 10 * b, ca);
      mul_inert_vec(t2, W(cinert) + 10 * b, W(cvel) + 6 * b);
      cross_force(t3, W(cvel) + 6 * b, t2);
      for (int i = 0; i < 6; i++) { cacc[6 * b + i] = ca[i]; cint[6 * b + i] = t1[i] + t3[i] - cext[6 * b + i]; }
    }
    __syncwarp();
  }
  tree_accumulate(c, cint, 6, true);
}

// ---- ray / convex zone test of the touch sensor (MuJoCo: mju_rayGeom(...) >= 0): does p + t v, t >= 0, meet the site? ----
struct Interval { double lo, hi; bool ok; };
__device__ __forceinline__ void iv_clip(Interval& a, double lo, double hi) {
  if (lo > hi) { double t = lo; lo = hi; hi = t; }
  a.lo = fmax(a.lo, lo); a.hi = fmin(a.hi, hi);
  if (a.lo > a.hi) a.ok = false;
}
__device__ __forceinline__ void iv_quadric(Interval& r, double a, double b, double c) {   // a t^2 + 2 b t + c <= 0
  if (a < BMJ_MINVAL) { if (c > 0) r.ok = false; return; }
  double det = b * b - a * c;
  if (det < 0) { r.ok = false; return; }
  double sq = sqrt(det);
  iv_clip(r, (-b - sq) / a, (-b + sq) / a);
}
__device__ __forceinline__ void iv_slab(Interval& r, double p, double v, double half) {
  if (fabs(v) < BMJ_MINVAL) { if (fabs(p) > half) r.ok = false; return; }
  iv_clip(r, (-half - p) / v, (half - p) / v);
}
__device__ __noinline__ bool ray_hits_zone(int type, const double* sz, const double* p, const double* v) {
  Interval r; r.lo = -1e300; r.hi = 1e300; r.ok = true;
  if (type == BMJ_GEOM_SPHERE) iv_quadric(r, dot3(v, v), dot3(p, v), dot3(p, p) - sz[0] * sz[0]);
  else if (type == BMJ_GEOM_ELLIPSOID) {
    double ps[3] = {p[0] / sz[0], p[1] / sz[1], p[2] / sz[2]}, vs[3] = {v[0] / sz[0], v[1] / sz[1], v[2] / sz[2]};
    iv_quadric(r, dot3(vs, vs), dot3(ps, vs), dot3(ps, ps) - 1);
  } else if (type == BMJ_GEOM_BOX) { for (int i = 0; i < 3; i++) iv_slab(r, p[i], v[i], sz[i]); }
  else if (type == BMJ_GEOM_CYLINDER || type == BMJ_GEOM_CAPSULE) {
    iv_quadric(r, v[0]*v[0] + v[1]*v[1], p[0]*v[0] + p[1]*v[1], p[0]*p[0] + p[1]*p[1] - sz[0]*sz[0]);
    iv_slab(r, p[2], v[2], sz[1]);
    if (type == BMJ_GEOM_CAPSULE) {
      if (r.ok && r.hi >= 0) return true;
      for (int s = -1; s <= 1; s += 2) {
        Interval q; q.lo = -1e300; q.hi = 1e300; q.ok = true;
        double pc[3] = {p[0], p[1], p[2] - s * sz[1]};
        iv_quadric(q, dot3(v, v), dot3(pc, v), dot3(pc, pc) - sz[0] * sz[0]);
        if (q.ok && q.hi >= 0) return true;
      }
      return false;
    }
  } else return false;
  return r.ok && r.hi >= 0;
}

// ------------------------------------------------------------------------------------------------
// sensors (stage 1 = position, 2 = velocity, 3 = acceleration); results staged in the workspace
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void sensors(const Ctx& c, int stage_mask, int ncon) {
  const DevModel& m = c.m; int lane = c.lane;
  if (c.disableflags & BMJ_DSBL_SENSOR) return;
  FOR_LANES(s, m.nsensor) {
    if (!((stage_mask >> (m.sensor_needstage[s] - 1)) & 1)) continue;
    double* out = W(sens) + m.sensor_adr[s];
    int id = m.sensor_objid[s], st = m.sensor_type[s];
    if (st == BMJ_SENS_JOINTPOS) out[0] = W(qpos)[m.jnt_qposadr[id]];
    else if (st == BMJ_SENS_JOINTVEL) out[0] = W(qvel)[m.jnt_dofadr[id]];
    else if (st == BMJ_SENS_ACTUATORFRC) out[0] = W(actforce)[id];
    else if (st == BMJ_SENS_SUBTREECOM) for (int i = 0; i < 3; i++) out[i] = W(scom)[3 * id + i];
    else if (st == BMJ_SENS_SUBTREELINVEL) for (int i = 0; i < 3; i++) out[i] = W(slinvel)[3 * id + i];
    else if (st == BMJ_SENS_FRAMEPOS) {
      double p[3], pm[9];
      int ot = m.sensor_objtype[s];
      if (ot == BMJ_OBJ_SITE) site_frame(c, id, p, pm);
      else if (ot == BMJ_OBJ_GEOM) geom_frame(c, id, p, pm);
      else if (ot == BMJ_OBJ_BODY) for (int i = 0; i < 3; i++) p[i] = W(xipos)[3 * id + i];
      else for (int i = 0; i < 3; i++) p[i] = W(xpos)[3 * id + i];
      int rid = m.sensor_refid[s];
      if (rid < 0) { for (int i = 0; i < 3; i++) out[i] = p[i]; }
      else {
        double rp[3], rm[9]; int rt = m.sensor_reftype[s];
        if (rt == BMJ_OBJ_SITE) site_frame(c, rid, rp, rm);
        else if (rt == BMJ_OBJ_GEOM) geom_frame(c, rid, rp, rm);
        else if (rt == BMJ_OBJ_BODY) {
          for (int i = 0; i < 3; i++) rp[i] = W(xipos)[3 * rid + i];
          double q[4], iq[4] = {m.body_iquat[4*rid], m.body_iquat[4*rid+1], m.body_iquat[4*rid+2], m.body_iquat[4*rid+3]};
          mul_quat(q, W(xquat) + 4 * rid, iq); quat2mat(rm, q);
        } else { for (int i = 0; i < 3; i++) rp[i] = W(xpos)[3 * rid + i]; for (int i = 0; i < 9; i++) rm[i] = W(xmat)[9 * rid + i]; }
        double dif[3] = {p[0] - rp[0], p[1] - rp[1], p[2] - rp[2]};
        matT_vec(out, rm, dif);
      }
    } else if (st == BMJ_SENS_VELOCIMETER || st == BMJ_SENS_GYRO || st == BMJ_SENS_ACCELEROMETER || st == BMJ_SENS_FORCE || st == BMJ_SENS_TORQUE) {
      double sp[3], sm[9]; site_frame(c, id, sp, sm);
      int b = m.site_bodyid[id], root = m.body_rootid[b];
      double dif[3], tmp[3];
      for (int i = 0; i < 3; i++) dif[i] = sp[i] - W(scom)[3 * root + i];
      const double* cv = W(cvel) + 6 * b;
      if (st == BMJ_SENS_GYRO) matT_vec(out, sm, cv);
      else if (st == BMJ_SENS_VELOCIMETER) {
        cross3(tmp, dif, cv); double lin[3] = {cv[3] - tmp[0], cv[4] - tmp[1], cv[5] - tmp[2]}; matT_vec(out, sm, lin);
      } else if (st == BMJ_SENS_ACCELEROMETER) {
        const double* ca = W(cacc) + 6 * b;
        cross3(tmp, dif, ca); double lin[3] = {ca[3] - tmp[0], ca[4] - tmp[1], ca[5] - tmp[2]}, acc[3], va[3], vl[3], corr[3];
        matT_vec(acc, sm, lin);
        cross3(tmp, dif, cv); double vlin[3] = {cv[3] - tmp[0], cv[4] - tmp[1], cv[5] - tmp[2]};
        matT_vec(va, sm, cv); matT_vec(vl, sm, vlin);
        cross3(corr, va, vl);
        for (int i = 0; i < 3; i++) out[i] = acc[i] + corr[i];
      } else if (st == BMJ_SENS_FORCE) matT_vec(out, sm, W(cfrc) + 6 * b + 3);
      else {
        const double* cf = W(cfrc) + 6 * b;
        cross3(tmp, dif, cf + 3); double tq[3] = {cf[0] - tmp[0], cf[1] - tmp[1], cf[2] - tmp[2]}; matT_vec(out, sm, tq);
      }
    } else if (st == BMJ_SENS_TOUCH) {
      double sp[3], sm[9]; site_frame(c, id, sp, sm);
      int b = m.site_bodyid[id]; double total = 0;
      double sz[3] = {m.site_size[3*id], m.site_size[3*id+1], m.site_size[3*id+2]}; int stp = m.site_type[id];
      _Pragma("unroll 1") for (int ci = 0; ci < ncon; ci++) {
        double* rec = W(con) + ci * CON_STRIDE; int* ii = con_ints(rec);
        if (ii[3] < 0) continue;
        if (m.geom_bodyid[ii[0]] != b && m.geom_bodyid[ii[1]] != b) continue;
        double nf = 0;
        if (ii[2] == 1) nf = W(force)[ii[3]]; else for (int k = 0; k < 4; k++) nf += W(force)[ii[3] + k];
        if (nf <= 0) continue;
        double dif[3] = {rec[1] - sp[0], rec[2] - sp[1], rec[3] - sp[2]}, loc[3], ray[3] = {rec[4], rec[5], rec[6]}, vloc[3];
        matT_vec(loc, sm, dif);
        if (m.geom_bodyid[ii[1]] == b) { ray[0] = -ray[0]; ray[1] = -ray[1]; ray[2] = -ray[2]; }
        matT_vec(vloc, sm, ray);
        bool in = ray_hits_zone(stp, sz, loc, vloc);
        if (in) total += nf;
      }
      out[0] = total;
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// integration
// ------------------------------------------------------------------------------------------------
// qpos <- integrate(qpos, a*vel, h)
__device__ __forceinline__ void integrate_pos(const Ctx& c, double* qpos, const double* vel, double a, double h) {
  const DevModel& m = c.m; int lane = c.lane;
  FOR_LANES(j, m.njnt) {
    int qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j], t = m.jnt_type[j];
    if (t == BMJ_JNT_FREE) {
      for (int i = 0; i < 3; i++) qpos[qa + i] += h * (a * vel[da + i]);
      double w[3] = {a * vel[da + 3], a * vel[da + 4], a * vel[da + 5]};
      quat_integrate(qpos + qa + 3, w, h);
    } else if (t == BMJ_JNT_BALL) { double w[3] = {a * vel[da], a * vel[da + 1], a * vel[da + 2]}; quat_integrate(qpos + qa, w, h); }
    else qpos[qa] += h * (a * vel[da]);
  }
  __syncwarp();
}

__device__ __forceinline__ void advance_act(const Ctx& c, double* act, const double* actdot, double scale, double h) {
  const DevModel& m = c.m; int lane = c.lane;
  FOR_LANES(a, m.nu) {
    int aa = m.actuator_actadr[a];
    if (aa < 0) continue;
    double v = act[aa] + h * (scale * actdot[aa]);
    if (m.actuator_actlimited[a]) v = clampd(v, m.actuator_actrange[2 * a], m.actuator_actrange[2 * a + 1]);
    act[aa] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool check_bad(const Ctx& c, const double* v, int n) {
  int lane = c.lane; int badf = 0;
  FOR_LANES(i, n) if (bad_value(v[i])) badf = 1;
  return __any_sync(FULL, badf);
}

__device__ __forceinline__ void reset_state(const Ctx& c, double* time) {
  const DevModel& m = c.m; int lane = c.lane;
  FOR_LANES(i, m.nq) W(qpos)[i] = m.qpos0[i];
  FOR_LANES(i, m.nv) { W(qvel)[i] = 0; W(qaccws)[i] = 0; }
  FOR_LANES(i, m.na) W(act)[i] = 0;
  *time = 0;
  __syncwarp();
}

template <int NVT>
__device__ __forceinline__ void euler_step(const Ctx& c, double* time) {
  const DevModel& m = c.m; int lane = c.lane; int nv = m.nv, ld = m.ldv; double h = m.timestep;
  advance_act(c, W(act), W(actdot), 1.0, h);
  if (NVT > 0 && m.any_damping && !(c.disableflags & BMJ_DSBL_EULERDAMP)) {
    if constexpr (NVT > 0) {
      // M is dead after the solver: M + h diag(damping) is formed in place
      FOR_LANES(i, nv) { W(tmpv)[i] = W(smooth)[i] + W(qcon)[i]; W(M)[tri(i) + i] += h * m.dof_damping[i]; }
      __syncwarp();
      tn_factor<NVT>(W(M), W(H), W(dinv), lane, W(tmpv), W(tmpv), W(J), W(efcSD), reinterpret_cast<const int*>(W(actlist)), opaque_zero(), W(colbuf));
      tn_back<NVT>(W(H), W(dinv), W(tmpv), W(tmpv), lane, 0);
      FOR_LANES(i, nv) W(qvel)[i] += h * W(tmpv)[i];
    }
  } else if (m.any_damping && !(c.disableflags & BMJ_DSBL_EULERDAMP)) {
    copy_row(W(H), c.Mc, tri(nv), lane);
    FOR_LANES(i, nv) W(tmpv)[i] = W(smooth)[i] + W(qcon)[i];
    __syncwarp();
    FOR_LANES(i, nv) W(H)[tri(i) + i] += h * m.dof_damping[i];
    __syncwarp();
    chol_factor(W(H), W(H), W(dinv), nv, lane, W(tmpv), W(tmpv));
    chol_back(W(H), W(dinv), W(tmpv), W(tmpv), nv, lane);
    FOR_LANES(i, nv) W(qvel)[i] += h * W(tmpv)[i];
  } else FOR_LANES(i, nv) W(qvel)[i] += h * W(qacc)[i];
  FOR_LANES(i, nv) W(qaccws)[i] = W(qacc)[i];
  __syncwarp();
  integrate_pos(c, W(qpos), W(qvel), 1.0, h);
  *time += h;
}

__device__ __forceinline__ void write_outputs(const Ctx& c, const b200mj_io& io, int env, int ncon, int nefc, int niter,
                                              bool posvel, bool acc, bool want_sens) {
  const DevModel& m = c.m; int lane = c.lane;
  size_t e = (size_t)env;
#define OUT(ptr, src, n) if (io.ptr) { _Pragma("unroll 1") for (int i = lane; i < (n); i += 32) io.ptr[e * (n) + i] = (src)[i]; }
  if (posvel) {
    OUT(xpos, W(xpos), 3 * m.nbody) OUT(xquat, W(xquat), 4 * m.nbody) OUT(xmat, W(xmat), 9 * m.nbody)
    OUT(xipos, W(xipos), 3 * m.nbody)
    OUT(subtree_com, W(scom), 3 * m.nbody) OUT(subtree_linvel, W(slinvel), 3 * m.nbody) OUT(cvel, W(cvel), 6 * m.nbody)
    OUT(qfrc_bias, c.pBias, m.nv) OUT(qfrc_passive, c.pPassive, m.nv)
    if (io.geom_xpos || io.geom_xmat) {   // recomputed: the staged geom frames share storage with the Hessian
      FOR_LANES(g, m.ngeom) {
        double p[3], mm[9]; geom_frame(c, g, p, mm);
        if (io.geom_xpos) for (int i = 0; i < 3; i++) io.geom_xpos[(e * m.ngeom + g) * 3 + i] = p[i];
        if (io.geom_xmat) for (int i = 0; i < 9; i++) io.geom_xmat[(e * m.ngeom + g) * 9 + i] = mm[i];
      }
    }
    if (io.site_xpos || io.site_xmat) {
      FOR_LANES(s, m.nsite) {
        double p[3], mm[9]; site_frame(c, s, p, mm);
        if (io.site_xpos) for (int i = 0; i < 3; i++) io.site_xpos[(e * m.nsite + s) * 3 + i] = p[i];
        if (io.site_xmat) for (int i = 0; i < 9; i++) io.site_xmat[(e * m.nsite + s) * 9 + i] = mm[i];
      }
    }
    if (io.qM) _Pragma("unroll 1") for (int i = lane; i < m.nv * m.nv; i += 32) { int r = i / m.nv, q = i % m.nv; io.qM[e * m.nv * m.nv + i] = c.pM[r >= q ? tri(r) + q : tri(q) + r]; }
    if (io.ncon && lane == 0) io.ncon[e] = ncon;
    if (io.nefc && lane == 0) io.nefc[e] = nefc;
    FOR_LANES(k, ncon) {
      double* rec = W(con) + k * CON_STRIDE; int* ii = con_ints(rec);
      size_t o = e * m.nconmax + k;
      if (io.contact_geom) { io.contact_geom[2 * o] = ii[0]; io.contact_geom[2 * o + 1] = ii[1]; }
      if (io.contact_efc_address) io.contact_efc_address[o] = ii[3];
      if (io.contact_dist) io.contact_dist[o] = rec[0];
      if (io.contact_pos) for (int i = 0; i < 3; i++) io.contact_pos[3 * o + i] = rec[1 + i];
      if (io.contact_frame) for (int i = 0; i < 9; i++) io.contact_frame[9 * o + i] = rec[4 + i];
    }
  }
  if (acc) {
    OUT(qacc, W(qacc), m.nv) OUT(qfrc_actuator, W(qfact), m.nv) OUT(actuator_force, W(actforce), m.nu)
    OUT(qfrc_constraint, W(qcon), m.nv)
    if (io.efc_force) FOR_LANES(r, nefc) io.efc_force[e * m.njmax + r] = W(force)[r];
    if (io.solver_niter && lane == 0) io.solver_niter[e] = niter;
  }
  if (want_sens) { OUT(sensordata, W(sens), m.nsensordata) }
#undef OUT
}

// the state a physics step advances, workspace -> io (NVT: compile-time nv of the acceleration kernels, 0: runtime)
template <int NVT>
__device__ __forceinline__ void store_state(const Ctx& c, const b200mj_io& io, size_t e, double time) {
  const DevModel& m = c.m; int lane = c.lane; const int nv = NVT > 0 ? NVT : m.nv;
  FOR_LANES(i, m.nq) io.qpos[e * m.nq + i] = W(qpos)[i];
  FOR_LANES(i, nv) { io.qvel[e * nv + i] = W(qvel)[i]; if (io.qacc_warmstart) io.qacc_warmstart[e * nv + i] = W(qaccws)[i]; }
  FOR_LANES(i, m.na) io.act[e * m.na + i] = W(act)[i];
  if (io.time && lane == 0) io.time[e] = time;
}

// adds a launch's warning counts (indexed by BMJ_WARN_*) to the environment's counters
__device__ __forceinline__ void add_warnings(const b200mj_io& io, size_t e, int lane, const int (&n)[BMJ_NWARNING]) {
  if (!io.warning || lane != 0) return;
  int* w = io.warning + e * BMJ_NWARNING;
  _Pragma("unroll") for (int k = 0; k < BMJ_NWARNING; k++) if (n[k]) w[k] += n[k];
}

enum { MODE_STEP = 0, MODE_FORWARD = 1 };

// One launch = one warp per environment, `nstep` physics steps fused. Every stage function is inlined exactly
// once into the single pass loop below (model / layout operands then come straight from the constant bank).
//   pass kinds: [posvel + acc + integrate] x nstep  (RK4: 4 passes per step), then for the reference's legacy
//   ordering one trailing [posvel] pass (= mj_step1 on the new state); MODE_FORWARD = one [posvel + acc] pass.
// CVX: as for the position kernels (the primitive-only build shares narrowphase<false> with them, so the two paths stay bit-identical).
template <bool CVX>
__global__ void __launch_bounds__(256)
step_kernel(const __grid_constant__ DevModel m, const __grid_constant__ Lay L, const __grid_constant__ b200mj_io io,
            int batch, int nstep, int flags, int mode, int extra_disable, const uint8_t* env_mask) {
  B200MJ_DYN_SMEM
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int env = blockIdx.x * (blockDim.x >> 5) + warp;
  // warps past the end of the batch shadow the last environment (same control flow => same barrier count)
  // and never store; so do the warps of environments outside env_mask (masked reset / forward)
  const bool live = env < batch && (env_mask == nullptr || env_mask[env < batch ? env : 0] != 0);
  if (env >= batch) env = batch - 1;
  Ctx c(m, L, smem + (size_t)warp * L.total, lane, m.disableflags | extra_disable, 0);
  c.set_env(env, io);
  size_t e = (size_t)env;
  // ---- load state ----
  FOR_LANES(i, m.nq) W(qpos)[i] = io.qpos[e * m.nq + i];
  FOR_LANES(i, m.nv) { W(qvel)[i] = io.qvel[e * m.nv + i]; W(qaccws)[i] = io.qacc_warmstart ? io.qacc_warmstart[e * m.nv + i] : 0.0; }
  FOR_LANES(i, m.na) W(act)[i] = io.act[e * m.na + i];
  FOR_LANES(i, m.nu) W(ctrl)[i] = io.ctrl ? io.ctrl[e * m.nu + i] : 0.0;
  if (io.sensordata) FOR_LANES(i, m.nsensordata) W(sens)[i] = io.sensordata[e * m.nsensordata + i];
  double time = io.time ? io.time[e] : 0.0;
  int warn[BMJ_NWARNING] = {};
  __syncwarp();
  const bool want_sens = (flags & B200MJ_STEP_SENSORS) != 0;
  const bool forward = mode == MODE_FORWARD;
  const bool legacy = (flags & B200MJ_STEP_LEGACY) != 0;
  const bool full_final = (flags & B200MJ_STEP_FULL_FINAL) != 0;
  const bool rk4 = m.integrator == BMJ_INT_RK4;
  // ---- control check (mj_step / mj_step2 / mj_forward all start from a finite ctrl) ----
  if (check_bad(c, W(ctrl), m.nu)) { warn[BMJ_WARN_BADCTRL]++; FOR_LANES(i, m.nu) W(ctrl)[i] = 0; __syncwarp(); }

  int step_idx = 0, sub = 0;             // sub: Runge-Kutta stage 0..3 (always 0 for Euler)
  int r_ncon = 0, r_nefc = 0, r_niter = 0;   // reported statistics (first evaluation of a step)
  while (true) {
    const bool final_pass = !forward && step_idx >= nstep;      // trailing mj_step1 of the legacy ordering
    if (final_pass && !legacy) break;
    const bool last = forward || step_idx == nstep - 1;
    if (!forward && sub == 0) {
      if (check_bad(c, W(qpos), m.nq)) { warn[BMJ_WARN_BADQPOS]++; reset_state(c, &time); }
      if (check_bad(c, W(qvel), m.nv)) { warn[BMJ_WARN_BADQVEL]++; reset_state(c, &time); }
    }
    // ---------------- position + velocity stage ----------------
    PHASE_SYNC();
    kinematics(c);
    com_pos(c);
    crb_and_factor(c);
    int ncon = 0, nefc = 0, niter = 0;
    if (!final_pass || full_final) {
      int wfull = 0, cfull = 0;
      ncon = collision<CVX>(c, &wfull);
      nefc = make_constraint(c, ncon, &cfull);
      warn[BMJ_WARN_CONTACTFULL] += wfull; warn[BMJ_WARN_CNSTRFULL] += cfull;
    }
    fwd_velocity(c);
    const bool out_posvel = final_pass || forward || (!legacy && last && sub == 0);
    if (out_posvel) subtree_vel(c);
    // ---------------- acceleration stage ----------------
    if (!final_pass) {
      fwd_actuation(c);
      fwd_acceleration<0>(c, io, env);
      PHASE_SYNC();
      niter = m.solver == BMJ_SOL_PGS ? solve_pgs(c, nefc) : solve_newton<0>(c, nefc);
    }
    if (sub == 0) { r_ncon = ncon; r_nefc = nefc; if (!final_pass) r_niter = niter; }
    const bool out_acc = !final_pass && sub == 0 && last;
    const int smask = want_sens ? ((out_posvel ? 3 : 0) | (out_acc ? 4 : 0)) : 0;
    PHASE_SYNC();
    if ((smask & 4) && m.acc_sensors) rne_post_constraint(c, io, env, ncon);
    if (smask) sensors(c, smask, ncon);
    if (live && (out_posvel || out_acc)) write_outputs(c, io, env, r_ncon, r_nefc, r_niter, out_posvel, out_acc, want_sens && out_posvel);
    if (final_pass || forward) break;
    // ---------------- integration ----------------
    if (sub == 0 && check_bad(c, W(qacc), m.nv)) { warn[BMJ_WARN_BADQACC]++; reset_state(c, &time); step_idx++; continue; }
    if (!rk4) { euler_step<0>(c, &time); step_idx++; }
    else {
      // classic RK4 over (qpos, qvel, act): stage `sub` has just produced F_sub = (qvel, qacc, act_dot)
      const int nq = m.nq, nv = m.nv, na = m.na; const double h = m.timestep;
      double* X0q = W(rk); double* X0v = X0q + nq; double* X0a = X0v + nv;
      double* accv = X0a + na; double* acca = accv + nv; double* accd = acca + nv;
      const double Bw = (sub == 0 || sub == 3) ? 1.0 / 6 : 1.0 / 3;
      if (sub == 0) {
        FOR_LANES(i, nq) X0q[i] = W(qpos)[i];
        FOR_LANES(i, nv) { X0v[i] = W(qvel)[i]; accv[i] = 0; acca[i] = 0; }
        FOR_LANES(i, na) { X0a[i] = W(act)[i]; accd[i] = 0; }
      }
      FOR_LANES(i, nv) { accv[i] += Bw * W(qvel)[i]; acca[i] += Bw * W(qacc)[i]; }
      FOR_LANES(i, na) accd[i] += Bw * W(actdot)[i];
      __syncwarp();
      const bool fin = sub == 3;
      const double a = fin ? 1.0 : (sub == 2 ? 1.0 : 0.5);
      FOR_LANES(i, nq) W(qpos)[i] = X0q[i];
      FOR_LANES(i, na) W(act)[i] = X0a[i];
      __syncwarp();
      integrate_pos(c, W(qpos), fin ? accv : W(qvel), a, h);      // stage velocity, or the weighted sum at the end
      advance_act(c, W(act), fin ? accd : W(actdot), a, h);
      FOR_LANES(i, nv) { W(qvel)[i] = X0v[i] + h * (a * (fin ? acca[i] : W(qacc)[i])); if (fin) W(qaccws)[i] = W(qacc)[i]; }
      __syncwarp();
      if (fin) { time += h; sub = 0; step_idx++; } else sub++;
    }
  }
  if (!live) return;
  if (forward) {
    FOR_LANES(i, m.nq) io.qpos[e * m.nq + i] = W(qpos)[i];   // quaternions were normalised in place
  } else {
    if (!legacy && want_sens) { FOR_LANES(i, m.nsensordata) if (io.sensordata) io.sensordata[e * m.nsensordata + i] = W(sens)[i]; }
    store_state<0>(c, io, e, time);
  }
  add_warnings(io, e, lane, warn);
}

// ------------------------------------------------------------------------------------------------
// Split path: the same stage functions in two smaller kernels. A pass is  [pos_kernel -> acc_kernel];
// M, efc_J, efc_D, aref, bias, passive (and the tendon tables) travel through an L2-resident handover row, the
// state through the io arrays. Smaller code footprint and workspace per kernel => 2x the resident warps.
// Used for the first nstep-1 physics steps of a fused step() when no applied forces are routed in; the last step
// (acceleration-stage sensors, outputs, trailing mj_step1) stays with the fused kernel above.
// ------------------------------------------------------------------------------------------------
// FINAL = the trailing mj_step1 of the legacy ordering (subtree velocities, position/velocity sensors, outputs);
// otherwise the position/velocity half of a physics step, optionally dumping what the acceleration-stage sensors need.
// BUILD picks the narrow phase and the launch bounds:
//   POS_CVX (160, 2): at most five phase-aligned warps per CTA and a 204-register budget, so that two CTAs share an SM
//     (shared memory allows no more); the rarely taken convex narrow phase (cvx_mpr) would otherwise set the kernel's
//     register count to 255 and halve occupancy
//   POS_PRIM (160, 3): models whose candidate pairs are all analytic primitive pairs (no convex code, no stack spills):
//     three CTAs per SM
//   POS_BIG (224, 1): large models (CMU corridor: 30 KB of position workspace per environment, one CTA per SM either
//     way): up to seven phase-aligned warps in that one CTA and the full register budget
enum { POS_PRIM, POS_CVX, POS_BIG };
template <bool FINAL, int BUILD>
__global__ void __launch_bounds__(BUILD == POS_BIG ? 224 : 160, BUILD == POS_PRIM ? 3 : BUILD == POS_CVX ? 2 : 1)
pos_kernel(const __grid_constant__ DevModel m, const __grid_constant__ Lay L, const __grid_constant__ Handover ho,
           const __grid_constant__ b200mj_io io, int batch, int flags, int dump, int env0, const __grid_constant__ Compact cp) {
  constexpr bool CVX = BUILD != POS_PRIM;
  B200MJ_DYN_SMEM
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int env = env0 + blockIdx.x * (blockDim.x >> 5) + warp;      // this launch covers environments [env0, batch)
  // The warps of a CTA are phase-aligned by barriers between the stages (the kernel executes ~84 KB of SASS per
  // pass against a 32 KB L1.5 I-cache: unaligned warps spent 44 % of their stalls on instruction fetch). Warps past
  // the end of the batch shadow the last environment so that every warp reaches every barrier; they recompute and
  // rewrite identical values and skip the warning counters.
  const bool live = env < batch;
  if (!live) env = batch - 1;
  Ctx c(m, L, smem + (size_t)warp * L.total, lane, m.disableflags, 0);
  c.set_env(env, io);
  size_t e = (size_t)env;
  // A shadow warp gets a handover row of its own: the stages read back what they wrote there (raw-contact staging, Jacobian rows), so
  // sharing the live environment's row would race; the io arrays are only ever overwritten with identical values.
  const size_t hr = live ? e : (size_t)(cp.shadow_row + warp);
  const Hand& H = ho.H;
  double* hrow = ho.rows + hr * H.total;
  c.pM = hrow + H.M; c.pJ = hrow + H.J; c.pD = hrow + H.efcD; c.pAref = hrow + H.aref; c.pBias = hrow + H.bias;
  c.pPassive = hrow + H.passive; c.pEq = reinterpret_cast<int*>(hrow + H.eqflag);
  c.stage = hrow + H.J;         // raw-contact staging: the row's Jacobian block (L2), written only later by make_constraint
  FOR_LANES(i, m.nq) W(qpos)[i] = io.qpos[e * m.nq + i];
  FOR_LANES(i, m.nv) W(qvel)[i] = io.qvel[e * m.nv + i];
  const bool want_sens = FINAL && (flags & B200MJ_STEP_SENSORS) != 0;
  __syncwarp();
  int warn[BMJ_NWARNING] = {};
  warn[BMJ_WARN_BADQPOS] = check_bad(c, W(qpos), m.nq);
  warn[BMJ_WARN_BADQVEL] = check_bad(c, W(qvel), m.nv);
  if (warn[BMJ_WARN_BADQPOS] || warn[BMJ_WARN_BADQVEL]) {
    FOR_LANES(i, m.nq) W(qpos)[i] = m.qpos0[i];
    FOR_LANES(i, m.nv) { W(qvel)[i] = 0; io.qvel[e * m.nv + i] = 0; if (io.qacc_warmstart) io.qacc_warmstart[e * m.nv + i] = 0; }
    FOR_LANES(i, m.na) io.act[e * m.na + i] = 0;
    if (io.time && lane == 0) io.time[e] = 0;
    __syncwarp();
  }
  PHASE_SYNC();
  kinematics(c);
  int wfull = 0, cfull = 0, ncon = 0, nefc = 0;
  const bool with_constraints = !FINAL || (flags & B200MJ_STEP_FULL_FINAL) != 0;
  PHASE_SYNC();
  if (with_constraints) ncon = collision<CVX>(c, &wfull);   // before com_pos: staging lives in the block com_pos starts to fill
  PHASE_SYNC();
  com_pos(c);
  crb_and_factor(c);
  PHASE_SYNC();
  if (with_constraints) nefc = make_constraint(c, ncon, &cfull);
  PHASE_SYNC();
  fwd_velocity(c);
  PHASE_SYNC();
  if (FINAL) {
    // (the sensor block shares storage with cacc / cfrc, which fwd_velocity has finished with; the acceleration-stage values of the last physics step are kept)
    if (io.sensordata) FOR_LANES(i, m.nsensordata) W(sens)[i] = io.sensordata[e * m.nsensordata + i];
    subtree_vel(c);
    if (want_sens) sensors(c, 3, ncon);
    write_outputs(c, io, env, ncon, nefc, 0, true, false, want_sens);
  }
  if (!FINAL || with_constraints) {
    // hand over the small tables the actuation stage needs and the row counts (the trailing step1 does so too: the
    // next call may start from its handover, B200MJ_STEP_REUSE_POS)
    FOR_LANES(t, m.ntendon) hrow[H.tenlen + t] = W(tenlen)[t];
    copy_row(hrow + H.tenJ, W(tenJ), m.ntendon * m.ldv, lane);
    if (lane == 0) { int* cnt = reinterpret_cast<int*>(hrow + H.counts); cnt[0] = ncon; cnt[1] = nefc; }
    if (dump) {
      double* d2 = ho.rows2 + hr * ho.H2.total;
#define DUMP(f, n) copy_row(d2 + ho.H2.f, W(f), (n), lane);
      HAND2_FIELDS(DUMP)
#undef DUMP
    }
  }
  FOR_LANES(i, m.nq) io.qpos[e * m.nq + i] = W(qpos)[i];      // quaternions were normalised in place
  if (!FINAL || with_constraints) {
    // bucket lists for the acceleration launches: one shared-memory ticket per environment, one global atomic per CTA
    // and bucket (every warp of the CTA gets here: the shadows of environments past the batch end take no ticket)
    int* cta = reinterpret_cast<int*>(smem + (size_t)(blockDim.x >> 5) * L.total);      // 8 ints behind the workspaces (64 bytes reserved)
    if (threadIdx.x < 4) cta[threadIdx.x] = 0;
    __syncthreads();
    int b = 0, my = 0;
    if (live && lane == 0) {
      while (b + 1 < cp.nbucket && nefc > cp.rows_cap[b]) b++;
      my = atomicAdd(&cta[b], 1);
    }
    __syncthreads();
    if (threadIdx.x < 4) cta[4 + threadIdx.x] = cta[threadIdx.x] ? atomicAdd(&cp.count[threadIdx.x], cta[threadIdx.x]) : 0;
    __syncthreads();
    if (live && lane == 0) cp.list[(size_t)b * cp.cap + cta[4 + b] + my] = env;
  }
  if (live) {
    warn[BMJ_WARN_CONTACTFULL] = wfull; warn[BMJ_WARN_CNSTRFULL] = cfull;
    add_warnings(io, e, lane, warn);
  }
}

// LAST = last physics step of a fused step(): acceleration-stage sensors and outputs are produced here.
// NVT = 0: nv at run time (any model; CTAs of up to 8 warps). Otherwise nv fixed at compile time (register-resident
// algebra, tn_* above), one instantiation per nv of B200MJ_NV_LIST — the dofs of the benchmark configurations (cheetah 9,
// quadruped 22, humanoid 27) and a few common small sizes — built for at most 4 warps per CTA. Same arguments, same
// handover format.
#define B200MJ_NV_LIST(X) X(6) X(9) X(12) X(18) X(22) X(27)
template <bool LAST, int NVT>
__global__ void __launch_bounds__(NVT > 0 ? 128 : 256, NVT > 0 ? 4 : 0)
acc_kernel(const __grid_constant__ DevModel m, const __grid_constant__ Lay L, const __grid_constant__ Handover ho,
           const __grid_constant__ b200mj_io io, int first_pass, int flags, const int* bucket_count, const int* bucket_list) {
  B200MJ_DYN_SMEM
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // One launch per row-count bucket: the CTAs walk the bucket's environment list (*bucket_count entries), which the
  // position kernel filled. The warps of a multi-warp CTA are phase-aligned by barriers (load -> M^-1 -> every Newton
  // trip -> Euler), so that instruction lines are fetched once per CTA: the unrolled algebra executes 83 KB of SASS
  // against a 32 KB L1.5 I-cache. Warps past the end of the list then shadow its last entry (same control flow, no stores).
  const bool sync = blockDim.x > 32;
  const int n = bucket_count[0];
  int k = blockIdx.x * (blockDim.x >> 5) + warp;
  bool live = true;
  if (k >= n) {
    if (!sync || blockIdx.x * (blockDim.x >> 5) >= n) return;
    live = false; k = n - 1;
  }
  const int env = bucket_list[k];
  size_t e = (size_t)env;
  const Hand& H = ho.H;
  const double* hrow = ho.rows + e * H.total;
  const int* cnt = reinterpret_cast<const int*>(hrow + H.counts);
  const int ncon = cnt[0], nefc = cnt[1];
  Ctx c(m, L, smem + (size_t)warp * L.total, lane, m.disableflags, sync);
  c.set_env(env, io);
  const int nv = NVT > 0 ? NVT : m.nv, ld = NVT > 0 ? (NVT | 1) : m.ldv;
  // ---- load state + handover ----
  FOR_LANES(i, m.nq) W(qpos)[i] = io.qpos[e * m.nq + i];
  FOR_LANES(i, nv) { W(qvel)[i] = io.qvel[e * nv + i]; W(qaccws)[i] = io.qacc_warmstart ? io.qacc_warmstart[e * nv + i] : 0.0;
                     W(bias)[i] = hrow[H.bias + i]; W(passive)[i] = hrow[H.passive + i]; }
  FOR_LANES(i, m.na) W(act)[i] = io.act[e * m.na + i];
  FOR_LANES(i, m.nu) W(ctrl)[i] = io.ctrl ? io.ctrl[e * m.nu + i] : 0.0;
  if (L.mglobal) c.Mc = hrow + H.M;      // read where the position kernel left it (L2): one factorisation, one product and the Euler copy
  else copy_row(W(M), hrow + H.M, tri(nv), lane);
  c.Jg = hrow + H.J;
  if (!L.jalias) copy_row(W(J), hrow + H.J, nefc * ld, lane);      // (jalias: dual_prepare brings it in once the factor of M is dead)
  FOR_LANES(r, nefc) { W(efcD)[r] = hrow[H.efcD + r]; W(aref)[r] = hrow[H.aref + r];
                       reinterpret_cast<int*>(W(eqflag))[r] = reinterpret_cast<const int*>(hrow + H.eqflag)[r]; W(efcSD)[r] = 0; }
  FOR_LANES(t, m.ntendon) W(tenlen)[t] = hrow[H.tenlen + t];
  copy_row(W(tenJ), hrow + H.tenJ, m.ntendon * ld, lane);
  const bool want_sens = LAST && (flags & B200MJ_STEP_SENSORS) != 0;
  double time = io.time ? io.time[e] : 0.0;
  __syncwarp();
  int warn[BMJ_NWARNING] = {};
  if (check_bad(c, W(ctrl), m.nu)) { warn[BMJ_WARN_BADCTRL] = first_pass; FOR_LANES(i, m.nu) W(ctrl)[i] = 0; __syncwarp(); }
  fwd_actuation(c);
  b200mj_io io_noforce = io; io_noforce.qfrc_applied = nullptr; io_noforce.xfrc_applied = nullptr;
  if (sync) __syncthreads();
  fwd_acceleration<NVT>(c, io_noforce, env);
  if (sync) __syncthreads();
  int niter = solve_newton<NVT>(c, nefc);
  if (LAST && live) write_outputs(c, io, env, ncon, nefc, niter, false, true, false);
  if (want_sens) FOR_LANES(i, nv) W(vold)[i] = W(qvel)[i];
  if (sync) __syncthreads();
  if (check_bad(c, W(qacc), nv)) { warn[BMJ_WARN_BADQACC] = 1; reset_state(c, &time); }
  else euler_step<NVT>(c, &time);
  if (!live) return;      // shadows: no stores (the sensor epilogue below has no barriers)
  store_state<NVT>(c, io, e, time);
  add_warnings(io, e, lane, warn);
  if (want_sens) {
    // Acceleration-stage sensors of the step just taken (MuJoCo evaluates them in mj_forward, before the state
    // advances): the solver's storage is dead now, so the position-stage dump is loaded over it (a workspace that
    // held both at once allowed 6 instead of 14 environments per SM).
    __syncwarp();
    FOR_LANES(i, nv) W(qvel)[i] = W(vold)[i];
    const double* d2 = ho.rows2 + e * ho.H2.total;
#define UNDUMP(f, n) copy_row(W(f), d2 + ho.H2.f, (n), lane);
    HAND2_FIELDS(UNDUMP)
#undef UNDUMP
    if (io.sensordata) FOR_LANES(i, m.nsensordata) W(sens)[i] = io.sensordata[e * m.nsensordata + i];
    __syncwarp();
    if (m.acc_sensors) rne_post_constraint(c, io_noforce, env, ncon);
    sensors(c, 4, ncon);
    if (io.sensordata) FOR_LANES(i, m.nsensordata) io.sensordata[e * m.nsensordata + i] = W(sens)[i];
  }
}

// ------------------------------------------------------------------------------------------------
// host side of the C ABI
// ------------------------------------------------------------------------------------------------
static int64_t g_launches = 0;

typedef decltype(&step_kernel<true>) step_kernel_fn;
typedef decltype(&pos_kernel<false, POS_CVX>) pos_kernel_fn;
typedef decltype(&acc_kernel<false, 0>) acc_kernel_fn;

static step_kernel_fn step_kernel_for(const b200mj_model* M) { return M->convex_pairs ? step_kernel<true> : step_kernel<false>; }

// final: the trailing mj_step1
static pos_kernel_fn pos_kernel_for(const b200mj_model* M, bool final) {
  if (M->pos_big) return final ? pos_kernel<true, POS_BIG> : pos_kernel<false, POS_BIG>;
  if (M->convex_pairs) return final ? pos_kernel<true, POS_CVX> : pos_kernel<false, POS_CVX>;
  return final ? pos_kernel<true, POS_PRIM> : pos_kernel<false, POS_PRIM>;
}

// the acceleration kernel for a compile-time size of nvt dofs (0: the runtime-size kernel), or nullptr where
// B200MJ_NV_LIST has no kernel for nvt
static acc_kernel_fn acc_kernel_for(int nvt, bool last) {
  switch (nvt) {
#define NV_CASE(n) case n: return last ? acc_kernel<true, n> : acc_kernel<false, n>;
    NV_CASE(0) B200MJ_NV_LIST(NV_CASE)
#undef NV_CASE
    default: return nullptr;
  }
}

// Lets every kernel the model's current layout can launch use up to SMEM_MAX of dynamic shared memory. Runs again
// whenever the layout is rebuilt: a change of capacities can move the model to another position-kernel build.
static void allow_shared_memory(const b200mj_model* M) {
  const void* kernels[] = {(const void*)step_kernel_for(M), (const void*)pos_kernel_for(M, false), (const void*)pos_kernel_for(M, true),
                           (const void*)acc_kernel_for(M->tn_nv, false), (const void*)acc_kernel_for(M->tn_nv, true)};
  for (const void* k : kernels) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
}

// Environment overrides, read once per model. Each is a test hook that steers a model onto a path it would not take by
// itself; unset, the engine makes every one of these choices from the model:
//   B200MJ_TN=0              runtime-size acceleration kernels although a compile-time-size one exists (the fused,
//                            split and TN comparisons of test_emu_kernel_parity.py, test_gpu_engine.py and test_dual_newton.py)
//   B200MJ_SPLIT=0           the fused kernel only (test_launch_knobs_do_not_change_results,
//                            test_fused_and_split_paths_agree_bitwise)
//   B200MJ_DUAL_MIN_NV=n     dual Newton direction from n dofs on (default 32; 0: never), forced onto the 27-dof humanoid
//                            by test_dual_newton.py
//   B200MJ_CVX_WARP=0        one convex pair per lane (cvx_pair), the bitwise reference for cvx_pair_warp
//                            (test_engine_convex_contacts_equal_the_oracles_bitwise, test_launch_knobs_do_not_change_results)
//   B200MJ_BUCKETS=a,b[,c]   acceleration row-bucket capacities below njmax
//   B200MJ_EPB_POS=n         warps per position-kernel CTA
//   B200MJ_ACC_WARPS=n       warps per compile-time-size acceleration CTA, at most 4 (default 4)
//   B200MJ_ENVS_PER_BLOCK=n  warps per fused-kernel CTA
//                            (these four: launch invariance, test_launch_knobs_do_not_change_results)
static void read_test_hooks(b200mj_model* M) {
  auto num = [](const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; };
  M->hooks.tn = num("B200MJ_TN", 1);
  M->hooks.split = num("B200MJ_SPLIT", 1);
  M->hooks.dual_min_nv = num("B200MJ_DUAL_MIN_NV", 32);
  M->dm.cvx_warp = num("B200MJ_CVX_WARP", 1);
  M->hooks.nbuckets = 0;
  if (const char* e = getenv("B200MJ_BUCKETS")) {
    const int got = sscanf(e, "%d,%d,%d", &M->hooks.buckets[0], &M->hooks.buckets[1], &M->hooks.buckets[2]);
    if (got >= 2) M->hooks.nbuckets = got;
  }
  M->hooks.epb_pos = num("B200MJ_EPB_POS", 0);
  M->hooks.acc_warps = num("B200MJ_ACC_WARPS", 4);
  if (M->hooks.acc_warps < 1 || M->hooks.acc_warps > 8) M->hooks.acc_warps = 4;
  M->hooks.envs_per_block = num("B200MJ_ENVS_PER_BLOCK", 0);
}

static void build_layout(b200mj_model* M) {
  DevModel& m = M->dm; Lay& L = M->lay;
  int o = 0;
  auto take = [&](int n) { int r = o; o += (n + 1) & ~1; return r; };   // keep 16-byte alignment
  int nv = m.nv, nb = m.nbody, ld = m.ldv, nj = m.njmax;
  const int ntri = nv * (nv + 1) / 2;   // packed lower triangle (M, H)
  // efc_J; with candidate pairs at least STAGE_DOUBLES, where the narrow phase stages its raw contacts
  const int jcap = (m.npair > 0 && nj * ld < STAGE_DOUBLES) ? STAGE_DOUBLES : nj * ld;
  L.qpos = take(m.nq); L.qvel = take(nv); L.act = take(m.na); L.ctrl = take(m.nu); L.qaccws = take(nv); L.actdot = take(m.na);
  L.xpos = take(3 * nb); L.xquat = take(4 * nb); L.xmat = take(9 * nb); L.xipos = take(3 * nb);
  L.scom = take(3 * nb); L.slinvel = take(3 * nb);
  L.cinert = take(10 * nb); L.cdof = take(6 * nv); L.cdofdot = take(6 * nv);
  L.cvel = take(6 * nb); L.cfrcext = take(m.acc_sensors ? 6 * nb : 0);
  // Position/velocity-stage temporaries that are dead once the acceleration stage starts share their storage
  // with the Newton Hessian / Cholesky buffer H (lifetimes: DESIGN.md "workspace").
  int h0 = o;
  L.crb = take(10 * nb); L.cacc = take(6 * nb); L.cfrc = take(6 * nb);
  L.gxpos = take(3 * m.ngeom); L.gxmat = take(9 * m.ngeom); L.xanchor = take(3 * m.njnt); L.xaxis = take(3 * m.njnt);
  if (o - h0 < ntri) take(ntri - (o - h0));
  L.H = h0;
  L.tenlen = take(m.ntendon); L.tenJ = take(m.ntendon * ld); L.actforce = take(m.nu);
  L.M = take(ntri); L.dinv = take(nv);
  L.J = take(jcap); L.efcD = take(nj); L.efcSD = take(nj); L.aref = take(nj); L.jar = take(nj); L.jv = take(nj);
  L.force = take(nj); L.eqflag = take((nj + 1) / 2); L.actlist = take((nj + 1) / 2);
  L.bias = take(nv); L.passive = take(nv); L.qfact = take(nv); L.smooth = take(nv); L.qaccs = take(nv); L.qacc = take(nv);
  L.qcon = take(nv); L.Ma = take(nv); L.grad = take(nv); L.search = take(nv); L.Mv = take(nv); L.tmpv = take(nv);
  L.con = take(m.nconmax * CON_STRIDE); L.cq = take(m.npair > 0 ? 32 : 0);
  L.gcache = (m.npair >= 16 * m.ngeom && m.ngeom > 0) ? 1 : 0;
  L.grb = take(L.gcache ? m.ngeom : 0); L.gmg = take(L.gcache ? m.ngeom : 0); L.gty = take(L.gcache ? (m.ngeom + 1) / 2 : 0);
  L.rk = take(m.integrator == BMJ_INT_RK4 ? (m.nq + 3 * nv + 2 * m.na + 8) : 0);
  L.sens = take(m.nsensordata);
  const bool pgs = m.solver == BMJ_SOL_PGS;
  L.pgsA = take(pgs ? nj * nj : 0); L.pgsX = take(pgs ? nj * ld : 0); L.pgsB = take(pgs ? nj : 0);
  L.total = o;
  M->smem_per_env = (size_t)o * sizeof(double);
  // One CTA per SM holding as many environments (= warps) as the 227 KB of shared memory allow, at most 8: the
  // warps of a CTA are phase-aligned with barriers and so share their instruction fetches.
  int best = (int)(SMEM_MAX / (M->smem_per_env ? M->smem_per_env : 1));
  if (best > 8) best = 8;
  if (M->hooks.envs_per_block >= 1 && M->hooks.envs_per_block <= best) best = M->hooks.envs_per_block;
  M->envs_per_block = best;

  // ---- split kernels: compact layouts + handover rows ----
  {
    Lay& P = M->lay_pos; memset(&P, 0, sizeof(P));
    o = 0;
    // Lifetimes (pos_kernel): kinematics -> collision -> com_pos -> crb_and_factor -> make_constraint -> fwd_velocity [-> subtree_vel,
    // sensors]. Storage shared along that line, so that three 5-warp CTAs fit one SM (humanoid: 14.3 KB per environment, was 19.2):
    //   [gxpos gxmat]      dead after collision  ==  crb (crb_and_factor), then cacc, cfrc (fwd_velocity), then slinvel, sens (trailing step1)
    //   [xanchor xaxis]    dead after com_pos    ==  cdofdot (fwd_velocity)
    // The narrow phase stages its raw contacts in the (not yet written) Jacobian block of the environment's handover row in L2.
    P.qpos = take(m.nq); P.qvel = take(nv);
    P.xpos = take(3 * nb); P.xquat = take(4 * nb); P.xmat = take(9 * nb); P.xipos = take(3 * nb);
    P.scom = take(3 * nb); P.cinert = take(10 * nb); P.cdof = take(6 * nv); P.cvel = take(6 * nb);
    {
      const int a0 = o;
      P.xanchor = take(3 * m.njnt); P.xaxis = take(3 * m.njnt);
      const int a1 = o;
      o = a0; P.cdofdot = take(6 * nv);
      if (o < a1) o = a1;
    }
    {
      const int b0 = o;
      P.gxpos = take(3 * m.ngeom); P.gxmat = take(9 * m.ngeom);
      const int b1 = o;
      o = b0; P.crb = take(10 * nb);
      const int b2 = o;
      o = b0; P.cacc = take(6 * nb); P.cfrc = take(6 * nb);
      const int b3 = o;
      o = b0; P.slinvel = take(3 * nb); P.sens = take(m.nsensordata);
      if (o < b1) o = b1;
      if (o < b2) o = b2;
      if (o < b3) o = b3;
    }
    P.tenlen = take(m.ntendon); P.tenJ = take(m.ntendon * ld);
    P.con = take(m.nconmax * CON_STRIDE); P.cq = take(m.npair > 0 ? 32 : 0);
    P.gcache = (m.npair >= 16 * m.ngeom && m.ngeom > 0) ? 1 : 0;      // CMU corridor: 2 113 pairs over 73 geoms
    P.grb = take(P.gcache ? m.ngeom : 0); P.gmg = take(P.gcache ? m.ngeom : 0); P.gty = take(P.gcache ? (m.ngeom + 1) / 2 : 0);
    P.total = o;
    M->smem_pos = (size_t)o * sizeof(double);
    // dual form of the Newton direction in the runtime-size kernels from dual_min_nv dofs on (32: the two-rows-per-lane
    // factorisation)
    const int dual_min_nv = M->hooks.dual_min_nv;
    const int ncon = m.nconmax;      // HAND2_FIELDS: room for every contact
    auto tri_host = [](int i) { return (i * (i + 1)) / 2; };
    auto acc_layout = [&](Lay& A, int rows, bool with_sens) {
      memset(&A, 0, sizeof(A));
      o = 0;
      A.qpos = take(m.nq); A.qvel = take(nv); A.act = take(m.na); A.ctrl = take(m.nu); A.qaccws = take(nv); A.actdot = take(m.na);
      A.tenlen = take(m.ntendon); A.tenJ = take(m.ntendon * ld); A.actforce = take(m.nu);
      A.force = take(rows); A.qacc = take(nv); A.vold = take(with_sens ? nv : 0); A.colbuf = take(M->tn_nv ? TN_COLBUF_DOUBLES : 0);
      // Everything below is dead once the state has been integrated; the sensor-carrying variant then re-uses the
      // storage for the position-stage dump that rne_post_constraint and the acceleration-stage sensors read.
      const int u0 = o;
      A.mglobal = (!M->tn_nv && nv >= 32) ? 1 : 0;
      A.M = take(A.mglobal ? 0 : ntri); A.H = take(ntri); A.dinv = take(nv);
      // dual form with few rows: J's workspace copy aliases H (dual_prepare), so that seven CMU environments fit an SM
      const bool dual = dual_min_nv > 0 && !M->tn_nv && nv >= dual_min_nv && rows <= 32 && m.solver == BMJ_SOL_NEWTON;
      const int dneed = rows * rows + tri_host(rows) + 3 * rows + 2;      // dS
      A.jalias = (dual && rows * ld + dneed <= ntri) ? 1 : 0;
      A.J = A.jalias ? A.H : take(rows * ld); A.efcD = take(rows); A.efcSD = take(rows); A.aref = take(rows); A.jar = take(rows); A.jv = take(rows);
      A.eqflag = take((rows + 1) / 2); A.actlist = take((rows + 1) / 2);
      A.bias = take(nv); A.passive = take(nv); A.qfact = take(nv); A.smooth = take(nv); A.qaccs = take(nv);
      A.qcon = take(nv); A.Ma = take(nv); A.grad = take(nv); A.search = take(nv); A.Mv = take(nv); A.tmpv = take(nv);
      if (dual) {
        A.dual = 1; A.drows = rows; A.dV = take(rows * ld);
        A.dS = A.jalias ? A.H + ((rows * ld + 1) & ~1) : (dneed <= ntri ? A.H : take(dneed));
      }
      if (with_sens) {
        const int acc_end = o;
        o = u0;
#define TAKE_DUMP(f, n) A.f = take(n);
        HAND2_FIELDS(TAKE_DUMP)
#undef TAKE_DUMP
        A.cacc = take(6 * nb); A.cfrc = take(6 * nb); A.cfrcext = take(6 * nb);
        A.sens = take(m.nsensordata);
        if (o < acc_end) o = acc_end;
      }
      A.total = o;
      return (size_t)o * sizeof(double);
    };
    // row-count buckets: most environments carry far fewer rows than njmax (humanoid: mean 10, max 43 of 64)
    // {10, 16, 32, njmax} gave a shorter kernel group than {10, 24, njmax} on the humanoid workload
    int caps[4] = {10, 16, 32, nj};
    int ncap = 4;
    // large capacities (CMU corridor, njmax 200; 91 % of the environments carry <= 12 rows, 99.6 % <= 32): every populated bucket launch
    // costs one per-environment latency and the launches cannot share SMs (shared memory), so three buckets measured
    // faster per control step than four
    if (nj > 96) { caps[0] = 12; caps[1] = 32; caps[2] = nj; ncap = 3; }
    if (M->hooks.nbuckets) {
      ncap = M->hooks.nbuckets + 1;
      for (int k = 0; k < M->hooks.nbuckets; k++) caps[k] = M->hooks.buckets[k];
      caps[ncap - 1] = nj;
    }
    M->nbucket = 0;
    for (int k = 0; k < ncap; k++) {
      int cap = caps[k] < nj ? caps[k] : nj;
      if (M->nbucket > 0 && cap <= M->rows_cap[M->nbucket - 1]) continue;
      int bi = M->nbucket++;
      M->rows_cap[bi] = cap;
      M->smem_acc_b[bi] = acc_layout(M->lay_acc_b[bi], cap, false);
      M->smem_accs_b[bi] = acc_layout(M->lay_accs_b[bi], cap, true);
      if (cap == nj) break;
    }
    Hand& Hd = M->ho.H;
    o = 0;
    Hd.M = take(ntri); Hd.J = take(jcap); Hd.efcD = take(nj); Hd.aref = take(nj); Hd.eqflag = take((nj + 1) / 2);
    Hd.bias = take(nv); Hd.passive = take(nv); Hd.tenlen = take(m.ntendon); Hd.tenJ = take(m.ntendon * ld); Hd.counts = take(2);
    Hd.total = o;
    Hand2& H2 = M->ho.H2;
    o = 0;
#define TAKE_H2(f, n) H2.f = take(n);
    HAND2_FIELDS(TAKE_H2)
#undef TAKE_H2
    H2.total = o;
    auto pick = [](size_t per_env) { int e = (int)((SMEM_MAX - 64) / (per_env ? per_env : 1)); return e > 8 ? 8 : e; };   // 64: CTA scratch of the bucket compaction
    // several small CTAs per SM: no phase barriers in the split kernels
    // position kernels: CTAs of up to 5 phase-aligned warps, two CTAs per SM when they fit
    M->epb_pos = pick(M->smem_pos) > 5 ? 5 : pick(M->smem_pos);
    // one 5-warp CTA per SM and room for more warps: the POS_BIG kernels (up to 7 warps, __launch_bounds__(224, 1))
    M->pos_big = 0;
    if (2 * 5 * M->smem_pos + 2 * 64 > SMEM_MAX && pick(M->smem_pos) > 5) { M->pos_big = 1; M->epb_pos = pick(M->smem_pos) > 7 ? 7 : pick(M->smem_pos); }
    const int v = M->hooks.epb_pos;
    if (v >= 1 && v <= pick(M->smem_pos) && v <= (M->pos_big ? 7 : 5)) M->epb_pos = v;   // __launch_bounds__(160, ..)
  }
}

// one field of the compiled-model blob on the host: its first element and its length
template <class T> struct HostField { const T* p; int n; };
struct HostModel {
#define HOST_I(name) HostField<int> name;
#define HOST_R(name) HostField<double> name;
  B200MJ_MODEL_FIELDS(HOST_I, HOST_R)
#undef HOST_I
#undef HOST_R
};
#define COUNT_FIELD(name) + 1
static const int NFIELDS = 0 B200MJ_MODEL_FIELDS(COUNT_FIELD, COUNT_FIELD);
#undef COUNT_FIELD

extern "C" {

const char* b200mj_version(void) { return "b200mj 0.1.0 (sm_90a, warp-per-env fp64)"; }

const char* b200mj_error_string(int code) {
  switch (code) {
    case 0: return "ok";
    case -1: return "bad argument";
    case -2: return "CUDA allocation / copy failed";
    case -3: return "model feature outside the supported subset (condim 4/6, frictionloss, nv > 64, CG solver, elliptic cones, mesh / hfield geoms)";
    case -4: return "per-environment workspace exceeds 227 KB of shared memory: lower nconmax / njmax";
    case -5: return "kernel launch failed";
    default: return "unknown error";
  }
}

int64_t b200mj_launch_count(void) { return g_launches; }
int64_t b200mj_workspace_bytes(const b200mj_model* m) { return m ? (int64_t)m->smem_per_env : -1; }
int b200mj_envs_per_block(const b200mj_model* m) { return m ? m->envs_per_block : -1; }

int b200mj_describe(const b200mj_model* M, char* buf, int n) {
  if (!M || !buf || n <= 0) return -1;
  int w = snprintf(buf, n, "{\"fused_workspace_bytes\": %zu, \"fused_envs_per_cta\": %d, \"pos_workspace_bytes\": %zu, \"pos_envs_per_cta\": %d, "
                   "\"handover_bytes_per_env\": %zu, \"acc_buckets\": [", M->smem_per_env, M->envs_per_block, M->smem_pos, M->epb_pos,
                   (size_t)(M->ho.H.total + M->ho.H2.total) * sizeof(double));
  for (int b = 0; b < M->nbucket && w < n; b++)
    w += snprintf(buf + w, n - w, "%s{\"rows\": %d, \"workspace_bytes\": %zu, \"last_step_workspace_bytes\": %zu}", b ? ", " : "",
                  M->rows_cap[b], M->smem_acc_b[b], M->smem_accs_b[b]);
  if (w < n) w += snprintf(buf + w, n - w, "]}");
  return w < n ? 0 : -1;
}

int b200mj_model_create(const int32_t* idata, int ni, const double* rdata, int nr, b200mj_model** out) {
  if (!idata || !rdata || !out || ni <= 0 || nr <= 0) return -1;
  // the blob starts with one (offset, length) pair per field of b200mj_model_fields.h: refuse a malformed directory,
  // else locate every field on the host
  if (ni < 2 * NFIELDS) return -1;
  HostModel h;
  int k = 0;
#define LOCATE(name, base, lo, hi) { const long off = idata[2 * k], len = idata[2 * k + 1]; k++; \
    if (off < (lo) || len < 0 || off + len > (hi)) return -1; h.name = {base + off, (int)len}; }
#define LOCATE_I(name) LOCATE(name, idata, 2 * NFIELDS, ni)
#define LOCATE_R(name) LOCATE(name, rdata, 0, nr)
  B200MJ_MODEL_FIELDS(LOCATE_I, LOCATE_R)
#undef LOCATE_I
#undef LOCATE_R
#undef LOCATE
  b200mj_model* M = new b200mj_model();
  memset(M, 0, sizeof(*M));
  if (cudaMalloc(&M->d_idata, (size_t)ni * sizeof(int)) != cudaSuccess) { delete M; return -2; }
  if (cudaMalloc(&M->d_rdata, (size_t)nr * sizeof(double)) != cudaSuccess) { cudaFree(M->d_idata); delete M; return -2; }
  if (cudaMemcpy(M->d_idata, idata, (size_t)ni * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(M->d_rdata, rdata, (size_t)nr * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaFree(M->d_idata); cudaFree(M->d_rdata); delete M; return -2;
  }
  DevModel& m = M->dm;
#define DEV_I(name) m.name = M->d_idata + (h.name.p - idata);
#define DEV_R(name) m.name = M->d_rdata + (h.name.p - rdata);
  B200MJ_MODEL_FIELDS(DEV_I, DEV_R)
#undef DEV_I
#undef DEV_R
  const int* sz = h.sizes.p; const int* opti = h.opt_int.p; const double* optr = h.opt_real.p;
  m.nq = sz[BMJ_NQ]; m.nv = sz[BMJ_NV]; m.nu = sz[BMJ_NU]; m.na = sz[BMJ_NA]; m.nbody = sz[BMJ_NBODY];
  m.njnt = sz[BMJ_NJNT]; m.ngeom = sz[BMJ_NGEOM]; m.nsite = sz[BMJ_NSITE]; m.ntendon = sz[BMJ_NTENDON];
  m.neq = sz[BMJ_NEQ]; m.nsensor = sz[BMJ_NSENSOR]; m.nsensordata = sz[BMJ_NSENSORDATA];
  m.npair = sz[BMJ_NPAIR]; m.nlevel = sz[BMJ_NLEVEL]; m.nconmax = sz[BMJ_NCONMAX]; m.njmax = sz[BMJ_NJMAX];
  m.ldv = m.nv | 1;
  m.integrator = opti[BMJ_OPT_INTEGRATOR]; m.iterations = opti[BMJ_OPT_ITERATIONS]; m.solver = opti[BMJ_OPT_SOLVER];
  m.ls_iterations = opti[BMJ_OPT_LS_ITERATIONS]; m.disableflags = opti[BMJ_OPT_DISABLEFLAGS];
  m.timestep = optr[BMJ_OPT_TIMESTEP];
  for (int i = 0; i < 3; i++) m.gravity[i] = optr[BMJ_OPT_GRAVITY_X + i];
  m.tolerance = optr[BMJ_OPT_TOLERANCE]; m.ls_tolerance = optr[BMJ_OPT_LS_TOLERANCE];
  m.impratio = optr[BMJ_OPT_IMPRATIO]; m.meaninertia = optr[BMJ_OPT_MEANINERTIA];
  m.any_damping = 0;
  for (int i = 0; i < m.nv; i++) if (h.dof_damping.p[i] > 0) m.any_damping = 1;
  m.acc_sensors = 0;
  for (int i = 0; i < h.sensor_type.n; i++) { int t = h.sensor_type.p[i]; if (t == BMJ_SENS_ACCELEROMETER || t == BMJ_SENS_FORCE || t == BMJ_SENS_TORQUE) m.acc_sensors = 1; }
  bool unsupported = m.nv > 64 || (opti[BMJ_OPT_SOLVER] != BMJ_SOL_NEWTON && opti[BMJ_OPT_SOLVER] != BMJ_SOL_PGS) || opti[BMJ_OPT_CONE] != 0 ||
                     (m.integrator != BMJ_INT_EULER && m.integrator != BMJ_INT_RK4);
  for (int i = 0; i < h.geom_condim.n; i++) if (h.geom_condim.p[i] != 1 && h.geom_condim.p[i] != 3) unsupported = true;
  // geom types without a narrow-phase function here (height fields, meshes) must not slip through as contact-free geoms
  for (int i = 0; i < h.geom_type.n; i++) if (h.geom_type.p[i] == BMJ_GEOM_HFIELD || h.geom_type.p[i] >= BMJ_GEOM_MESH) unsupported = true;
  for (int i = 0; i < h.dof_frictionloss.n; i++) if (h.dof_frictionloss.p[i] != 0) unsupported = true;
  if (unsupported) { b200mj_model_destroy(M); return -3; }
  // does any candidate pair reach the convex routines (see narrowphase<CVX>)? If not the position kernels are the primitive-only builds.
  M->convex_pairs = 0;
  for (int p = 0; p < m.npair; p++) {
    const int t1 = h.geom_type.p[h.pair_geom1.p[p]], t2 = h.geom_type.p[h.pair_geom2.p[p]];
    const bool analytic = t1 == BMJ_GEOM_PLANE || (t1 == BMJ_GEOM_SPHERE && (t2 == BMJ_GEOM_SPHERE || t2 == BMJ_GEOM_CAPSULE || t2 == BMJ_GEOM_BOX)) ||
                          (t1 == BMJ_GEOM_CAPSULE && t2 == BMJ_GEOM_CAPSULE);
    if (!analytic) M->convex_pairs = 1;
  }
  {   // actuator moment arms by dof (constant for joint and fixed-tendon transmissions)
    const int nv = m.nv, nu = m.nu;
    int* adr = new int[nv + 1];
    int* ids = new int[(size_t)nv * (nu > 0 ? nu : 1)];
    double* coef = new double[(size_t)nv * (nu > 0 ? nu : 1)];
    const int* jnt_dofadr = h.jnt_dofadr.p;
    int n = 0;
    for (int i = 0; i < nv; i++) {
      adr[i] = n;
      for (int a = 0; a < nu; a++) {
        double mom = 0; bool any = false;
        const double gear = h.actuator_gear.p[a];
        if (h.actuator_trntype.p[a] == BMJ_TRN_JOINT) { if (jnt_dofadr[h.actuator_trnid.p[a]] == i) { mom = gear; any = true; } }
        else {
          const int t = h.actuator_trnid.p[a];
          double tj = 0;
          for (int w = h.tendon_adr.p[t]; w < h.tendon_adr.p[t] + h.tendon_num.p[t]; w++)
            if (jnt_dofadr[h.wrap_objid.p[w]] == i) { tj += h.wrap_prm.p[w]; any = true; }
          mom = gear * tj;
        }
        if (any) { ids[n] = a; coef[n] = mom; n++; }
      }
    }
    adr[nv] = n;
    const int nn = n > 0 ? n : 1;
    bool ok = cudaMalloc(&M->d_xi, (size_t)(nv + 1 + nn) * sizeof(int)) == cudaSuccess &&
              cudaMalloc(&M->d_xr, (size_t)nn * sizeof(double)) == cudaSuccess;
    if (ok) ok = cudaMemcpy(M->d_xi, adr, (size_t)(nv + 1) * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess &&
                 cudaMemcpy(M->d_xi + nv + 1, ids, (size_t)nn * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess &&
                 cudaMemcpy(M->d_xr, coef, (size_t)nn * sizeof(double), cudaMemcpyHostToDevice) == cudaSuccess;
    delete[] adr; delete[] ids; delete[] coef;
    if (!ok) { b200mj_model_destroy(M); return -2; }
    m.dof_act_adr = M->d_xi; m.dof_act_id = M->d_xi + nv + 1; m.dof_act_coef = M->d_xr;
  }
  read_test_hooks(M);
  M->nkey = sz[BMJ_NKEY];
  M->tn_nv = (M->hooks.tn && acc_kernel_for(m.nv, false)) ? m.nv : 0;
  build_layout(M);
  if (M->envs_per_block < 1) { b200mj_model_destroy(M); return -4; }
  for (int g = 0; g < 2; g++) {
    cudaStreamCreateWithFlags(&M->gmain[g], cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&M->ev_join[g], cudaEventDisableTiming); cudaEventCreateWithFlags(&M->ev_pos[g], cudaEventDisableTiming);
    for (int b = 0; b < 4; b++) { cudaStreamCreateWithFlags(&M->gaux[g][b], cudaStreamNonBlocking); cudaEventCreateWithFlags(&M->ev_acc[g][b], cudaEventDisableTiming); }
  }
  cudaEventCreateWithFlags(&M->ev_fork, cudaEventDisableTiming);
  M->streams_ok = 1;
  allow_shared_memory(M);
  *out = M;
  return 0;
}

void b200mj_model_destroy(b200mj_model* M) {
  if (!M) return;
  cudaFree(M->d_idata); cudaFree(M->d_rdata);
  if (M->d_xi) cudaFree(M->d_xi);
  if (M->d_xr) cudaFree(M->d_xr);
  if (M->d_varid) cudaFree(M->d_varid);
  if (M->ho.rows) cudaFree(M->ho.rows);
  if (M->ho.rows2) cudaFree(M->ho.rows2);
  if (M->d_bcount) cudaFree(M->d_bcount);
  if (M->d_blist) cudaFree(M->d_blist);
  if (M->streams_ok) {
    for (int g = 0; g < 2; g++) {
      cudaStreamDestroy(M->gmain[g]); cudaEventDestroy(M->ev_join[g]); cudaEventDestroy(M->ev_pos[g]);
      for (int b = 0; b < 4; b++) { cudaStreamDestroy(M->gaux[g][b]); cudaEventDestroy(M->ev_acc[g][b]); }
    }
    cudaEventDestroy(M->ev_fork);
  }
  delete M;
}

int b200mj_model_set_disableflags(b200mj_model* M, int disableflags) {
  if (!M) return -1;
  M->dm.disableflags = disableflags;
  M->reuse_ok = 0;
  return 0;
}

int b200mj_model_set_capacity(b200mj_model* M, int nconmax, int njmax) {
  if (!M || nconmax < 0 || njmax < 0) return -1;
  M->dm.nconmax = nconmax; M->dm.njmax = njmax;
  build_layout(M);
  allow_shared_memory(M);
  // the handover rows are sized by the layout: drop them, the next b200mj_step allocates for the new capacities
  if (M->ho.rows) cudaFree(M->ho.rows);
  if (M->ho.rows2) cudaFree(M->ho.rows2);
  M->ho.rows = M->ho.rows2 = nullptr; M->hand_batch = 0; M->reuse_ok = 0;
  return M->envs_per_block < 1 ? -4 : 0;
}

// masked state reset (b200mj_reset): one thread per (environment, state element)
extern "C" __global__ void b200mj_reset_kernel(const __grid_constant__ DevModel m, const __grid_constant__ b200mj_io io, int batch,
                                               const uint8_t* env_mask, const double* key_qpos) {
  const int per = m.nq + 2 * m.nv + m.na + m.nu + 1;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)batch * per) return;
  const int e = (int)(idx / per); int k = (int)(idx % per);
  if (env_mask && !env_mask[e]) return;
  if (k < m.nq) { io.qpos[(size_t)e * m.nq + k] = key_qpos ? key_qpos[k] : m.qpos0[k]; return; }
  k -= m.nq;
  if (k < m.nv) { io.qvel[(size_t)e * m.nv + k] = 0; return; }
  k -= m.nv;
  if (k < m.nv) { if (io.qacc_warmstart) io.qacc_warmstart[(size_t)e * m.nv + k] = 0; return; }
  k -= m.nv;
  if (k < m.na) { io.act[(size_t)e * m.na + k] = 0; return; }
  k -= m.na;
  if (k < m.nu) { if (io.ctrl) const_cast<double*>(io.ctrl)[(size_t)e * m.nu + k] = 0; return; }
  if (io.time) io.time[e] = 0;
}

// mj_contactForce for one contact id of every environment (one thread per environment)
extern "C" __global__ void b200mj_contact_force_kernel(const __grid_constant__ DevModel m, const __grid_constant__ b200mj_io io,
                                                       int batch, int cid, double* out6) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= batch) return;
  double f[6] = {0, 0, 0, 0, 0, 0};
  const int ncon = io.ncon ? io.ncon[e] : 0;
  if (cid >= 0 && cid < ncon && io.contact_efc_address && io.contact_geom && io.efc_force) {
    const size_t o = (size_t)e * m.nconmax + cid;
    const int adr = io.contact_efc_address[o];
    if (adr >= 0) {
      const int g1 = io.contact_geom[2 * o], g2 = io.contact_geom[2 * o + 1];
      const int pr1 = m.geom_priority[g1], pr2 = m.geom_priority[g2];
      int condim; double mu;
      if (pr1 != pr2) { const int gp = pr1 > pr2 ? g1 : g2; condim = m.geom_condim[gp]; mu = m.geom_friction[3 * gp]; }
      else { condim = max(m.geom_condim[g1], m.geom_condim[g2]); mu = fmax(m.geom_friction[3 * g1], m.geom_friction[3 * g2]); }
      const double* ef = io.efc_force + (size_t)e * m.njmax + adr;
      if (condim == 1) f[0] = ef[0];
      else {   // pyramid edges (+t1, -t1, +t2, -t2): mju_decodePyramid
        f[0] = ef[0] + ef[1] + ef[2] + ef[3];
        f[1] = (ef[0] - ef[1]) * mu;
        f[2] = (ef[2] - ef[3]) * mu;
      }
    }
  }
  for (int i = 0; i < 6; i++) out6[(size_t)e * 6 + i] = f[i];
}

static int launch(const b200mj_model* M, const b200mj_io* io, int batch, int nstep, int flags, int mode, int extra, void* stream,
                  const uint8_t* env_mask = nullptr) {
  if (!M || !io || batch <= 0 || nstep < 0) return -1;
  const_cast<b200mj_model*>(M)->reuse_ok = 0;      // the fused kernel leaves no handover behind
  if (!io->qpos || !io->qvel || (M->dm.na > 0 && !io->act)) return -1;
  int epb = M->envs_per_block;
  int grid = (batch + epb - 1) / epb;
  const size_t smem = M->smem_per_env * epb;
  B200MJ_LAUNCH(step_kernel_for(M), grid, 32 * epb, smem, (cudaStream_t)stream, M->dm, M->lay, *io, batch, nstep, flags, mode, extra, env_mask);
  g_launches++;
  return cudaGetLastError() == cudaSuccess ? 0 : -5;
}

int b200mj_step(const b200mj_model* Mc, const b200mj_io* io, int batch, int nstep, int flags, void* stream) {
  b200mj_model* M = const_cast<b200mj_model*>(Mc);
  if (!M || !io || batch <= 0 || nstep < 0) return -1;
  // Split path: Euler, legacy ordering, no applied forces routed in, workspaces fit. Everything else (RK4, the
  // non-legacy ordering, qfrc/xfrc_applied) runs through the fused kernel.
  bool can_split = M->hooks.split && nstep >= 1 && (flags & B200MJ_STEP_LEGACY) && M->dm.integrator == BMJ_INT_EULER &&
                   M->dm.solver == BMJ_SOL_NEWTON &&
                   !io->qfrc_applied && !io->xfrc_applied && M->epb_pos >= 1 && M->smem_accs_b[M->nbucket - 1] <= SMEM_MAX &&
                   io->qpos && io->qvel && (M->dm.na == 0 || io->act);
  if (!can_split) return launch(M, io, batch, nstep, flags, MODE_STEP, 0, stream);
  if (M->hand_batch < batch) {
    if (M->ho.rows) cudaFree(M->ho.rows);
    if (M->ho.rows2) cudaFree(M->ho.rows2);
    M->ho.rows = M->ho.rows2 = nullptr; M->hand_batch = 0; M->reuse_ok = 0;
    if (cudaMalloc(&M->ho.rows, (size_t)(batch + SHADOW_ROWS) * M->ho.H.total * sizeof(double)) != cudaSuccess) return -2;
    if (cudaMalloc(&M->ho.rows2, (size_t)(batch + SHADOW_ROWS) * M->ho.H2.total * sizeof(double)) != cudaSuccess) return -2;
    if (M->d_bcount) cudaFree(M->d_bcount);
    if (M->d_blist) cudaFree(M->d_blist);
    M->d_bcount = M->d_blist = nullptr;
    if (cudaMalloc(&M->d_bcount, (size_t)2 * 4 * sizeof(int)) != cudaSuccess) return -2;
    if (cudaMalloc(&M->d_blist, (size_t)2 * 4 * batch * sizeof(int)) != cudaSuccess) return -2;
    cudaMemset(M->d_bcount, 0, (size_t)2 * 4 * sizeof(int));
    M->hand_batch = batch;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const bool want_sens = (flags & B200MJ_STEP_SENSORS) != 0;
  // Every physics step is split; the last one uses the sensor-carrying acceleration kernel and the trailing mj_step1 is
  // the FINAL position kernel.
  // B200MJ_STEP_REUSE_POS: the previous call's trailing mj_step1 wrote this state's handover rows already
  // (the trailing mj_step1 dumps what the acceleration-stage sensors need only when the call had one physics step: a
  // call whose first step is also its last must then find that dump, or recompute the position stage)
  const bool reuse = (flags & B200MJ_STEP_REUSE_POS) && M->reuse_ok && M->reuse_qpos == io->qpos &&
                     M->reuse_batch == batch && M->reuse_flags == (flags & ~B200MJ_STEP_REUSE_POS) &&
                     (nstep > 1 || !want_sens || M->reuse_has_dump);
  M->reuse_ok = 0;
  // Environment groups (2 for batches >= 2048): the launch sequence of each group is independent of the other's, so
  // groups run on their own streams and one group's position kernel fills the tail of the other's acceleration kernels.
  // On the humanoid workload 2 groups measured faster than 1 and 3 (with the earlier, larger workspaces 2 groups were
  // slower: too few warps of each kind fitted an SM side by side).
  const int ngroups = batch >= 2048 ? 2 : 1;
  // Row-bucket compaction: acceleration CTAs of several warps over dense per-bucket environment lists. Each group has
  // one set of bucket counters and lists, refilled by every position launch and read by the acceleration launches of
  // the same physics step. Reuse across steps is ordered by the group stream: every bucket stream joins back into it
  // (ev_acc) before the next position launch and its counter reset are queued there. The trailing mj_step1 fills them
  // for the next call's first acceleration launches (B200MJ_STEP_REUSE_POS). The launch sequence is the same in every
  // call, so a captured CUDA graph of this function stays valid.
  // On the humanoid workload 4 phase-aligned warps per CTA gave the shortest kernel group of one-warp CTAs and compacted
  // CTAs of 2, 3, 4 and 8 warps. The compile-time-size kernels are built for at most 4 warps per CTA (__launch_bounds__(128, 4)).
  if (ngroups > 1) cudaEventRecord(M->ev_fork, st);
  for (int g = 0; g < ngroups; g++) {
    const int e0 = (int)((long long)batch * g / ngroups), e1 = (int)((long long)batch * (g + 1) / ngroups), cnt = e1 - e0;
    cudaStream_t sm = (g == 0) ? st : M->gmain[g];
    if (g > 0) cudaStreamWaitEvent(sm, M->ev_fork, 0);
    const int gp = (cnt + M->epb_pos - 1) / M->epb_pos;
    int* gcount = M->d_bcount + (size_t)g * 4;
    int* glist = M->d_blist + (size_t)g * 4 * M->hand_batch;
    auto compact = [&]() {
      Compact cp; memset(&cp, 0, sizeof(cp));
      cp.shadow_row = M->hand_batch + g * 8;
      cp.count = gcount; cp.list = glist; cp.cap = M->hand_batch; cp.nbucket = M->nbucket;
      for (int b = 0; b < M->nbucket; b++) cp.rows_cap[b] = M->rows_cap[b];
      cudaMemsetAsync(cp.count, 0, 4 * sizeof(int), sm);
      return cp;
    };
    for (int s = 0; s < nstep; s++) {
      const bool last = s == nstep - 1;
      if (!(reuse && s == 0)) {
        const Compact cp = compact();
        B200MJ_LAUNCH(pos_kernel_for(M, false), gp, 32 * M->epb_pos, M->smem_pos * M->epb_pos + 64, sm, M->dm, M->lay_pos, M->ho, *io,
                      e1, flags, last && want_sens, e0, cp);
        g_launches++;
      }
      if (M->nbucket > 1) cudaEventRecord(M->ev_pos[g], sm);
      for (int b = 0; b < M->nbucket; b++) {
        cudaStream_t sb = b == 0 ? sm : M->gaux[g][b];     // buckets are independent: let them share the SMs
        if (b > 0) cudaStreamWaitEvent(sb, M->ev_pos[g], 0);
        const size_t ws = (last ? M->smem_accs_b[b] : M->smem_acc_b[b]);
        // warps per CTA: as many as fit SMEM_MAX, at most acc_warps
        const int want = M->tn_nv ? M->hooks.acc_warps : 8;      // runtime-size kernels (__launch_bounds__(256)): whatever fills the SM
        int cap = (int)(SMEM_MAX / ws); if (cap > want) cap = want; if (M->tn_nv && cap > 4) cap = 4; if (cap < 1) cap = 1;
        // as many resident warps per SM as SMEM_MAX allows (CMU corridor, 37 KB per warp: two CTAs of 3 instead of one of 4); ties: the larger CTA
        int wpc = 1, best = 0;
        for (int w = cap; w >= 1; w--) { const int res = (int)(SMEM_MAX / ((w * ws) + 1024)) * w; if (res > best) { best = res; wpc = w; } }
        const int grid = (cnt + wpc - 1) / wpc;
        const int* bl = glist + (size_t)b * M->hand_batch;
        const Lay& la = last ? M->lay_accs_b[b] : M->lay_acc_b[b];
        B200MJ_LAUNCH(acc_kernel_for(M->tn_nv, last), grid, 32 * wpc, ws * wpc, sb, M->dm, la, M->ho, *io, s == 0, flags, gcount + b, bl);
        if (b > 0) cudaEventRecord(M->ev_acc[g][b], sb);
        g_launches++;
      }
      for (int b = 1; b < M->nbucket; b++) cudaStreamWaitEvent(sm, M->ev_acc[g][b], 0);   // join after the main-stream bucket is queued
    }
    const Compact cp = compact();      // the lists of the next call's first physics step
    B200MJ_LAUNCH(pos_kernel_for(M, true), gp, 32 * M->epb_pos, M->smem_pos * M->epb_pos + 64, sm, M->dm, M->lay_pos, M->ho, *io,
                  e1, flags, want_sens && nstep == 1, e0, cp);
    g_launches++;
    if (g > 0) { cudaEventRecord(M->ev_join[g], sm); cudaStreamWaitEvent(st, M->ev_join[g], 0); }
  }
  if (cudaGetLastError() != cudaSuccess) return -5;
  if (flags & B200MJ_STEP_FULL_FINAL) { M->reuse_ok = 1; M->reuse_qpos = io->qpos; M->reuse_batch = batch; M->reuse_flags = flags & ~B200MJ_STEP_REUSE_POS; M->reuse_has_dump = want_sens && nstep == 1; }
  return 0;
}

int b200mj_forward(const b200mj_model* M, const b200mj_io* io, int batch, int extra_disableflags, int flags, void* stream) {
  return launch(M, io, batch, 0, flags, MODE_FORWARD, extra_disableflags, stream);
}

int b200mj_forward_masked(const b200mj_model* M, const b200mj_io* io, int batch, const uint8_t* env_mask, int extra_disableflags,
                          int flags, void* stream) {
  return launch(M, io, batch, 0, flags, MODE_FORWARD, extra_disableflags, stream, env_mask);
}

int b200mj_reset(const b200mj_model* M, const b200mj_io* io, int batch, const uint8_t* env_mask, int keyframe, void* stream) {
  if (!M || !io || batch <= 0 || !io->qpos || !io->qvel || (M->dm.na > 0 && !io->act)) return -1;
  const DevModel& m = M->dm;
  const double* key = nullptr;
  if (keyframe >= 0) {
    if (keyframe >= M->nkey) return -1;
    key = m.key_qpos + (size_t)keyframe * m.nq;
  }
  const long long total = (long long)batch * (m.nq + 2 * m.nv + m.na + m.nu + 1);
  B200MJ_LAUNCH(b200mj_reset_kernel, (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, M->dm, *io, batch, env_mask, key);
  g_launches++;
  if (cudaGetLastError() != cudaSuccess) return -5;
  // mj_forward with actuation disabled (engine.py:325-327), sensors on, for the environments just reset
  return launch(M, io, batch, 0, B200MJ_STEP_SENSORS, MODE_FORWARD, BMJ_DSBL_ACTUATION, stream, env_mask);
}

int b200mj_contact_force(const b200mj_model* M, const b200mj_io* io, int batch, int contact_id, double* out6, void* stream) {
  if (!M || !io || !out6 || batch <= 0) return -1;
  B200MJ_LAUNCH(b200mj_contact_force_kernel, (batch + 127) / 128, 128, 0, (cudaStream_t)stream, M->dm, *io, batch, contact_id, out6);
  g_launches++;
  return cudaGetLastError() == cudaSuccess ? 0 : -5;
}

int b200mj_subtree_vel(const b200mj_model* M, const b200mj_io* io, int batch, int flags, void* stream) {
  // zero physics steps in the legacy ordering = the trailing mj_step1 alone: position / velocity stage (with collision
  // when B200MJ_STEP_FULL_FINAL), mj_subtreeVel, position- and velocity-stage sensors, outputs; the state is unchanged
  return launch(M, io, batch, 0, flags | B200MJ_STEP_LEGACY, MODE_STEP, 0, stream);
}

int b200mj_model_set_variable_geoms(b200mj_model* M, const int32_t* geom_ids, int n) {
  if (!M || n < 0 || (n > 0 && !geom_ids)) return -1;
  const int ng = M->dm.ngeom;
  int* varid = new int[ng > 0 ? ng : 1];
  for (int g = 0; g < ng; g++) varid[g] = -1;
  for (int k = 0; k < n; k++) { if (geom_ids[k] < 0 || geom_ids[k] >= ng) { delete[] varid; return -1; } varid[geom_ids[k]] = k; }
  if (!M->d_varid && cudaMalloc(&M->d_varid, (size_t)(ng > 0 ? ng : 1) * sizeof(int)) != cudaSuccess) { delete[] varid; return -2; }
  const bool ok = cudaMemcpy(M->d_varid, varid, (size_t)ng * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess;
  delete[] varid;
  if (!ok) return -2;
  M->dm.geom_varid = M->d_varid; M->dm.nvargeom = n; M->reuse_ok = 0;
  return 0;
}

int b200mj_step_host(const b200mj_model* M, const b200mj_io* io, int batch, int nstep, int flags, const double* ctrl_host,
                     double* ctrl_dev, const double* obs_dev, double* obs_host, int nobs, void* stream) {
  if (!M || !io || !ctrl_host || !ctrl_dev) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemcpyAsync(ctrl_dev, ctrl_host, (size_t)batch * M->dm.nu * sizeof(double), cudaMemcpyHostToDevice, s) != cudaSuccess) return -2;
  b200mj_io io2 = *io; io2.ctrl = ctrl_dev;
  int rc = b200mj_step(M, &io2, batch, nstep, flags, stream);
  if (rc) return rc;
  if (obs_dev && obs_host && nobs > 0)
    if (cudaMemcpyAsync(obs_host, obs_dev, (size_t)batch * nobs * sizeof(double), cudaMemcpyDeviceToHost, s) != cudaSuccess) return -2;
  return cudaStreamSynchronize(s) == cudaSuccess ? 0 : -5;
}

}  // extern "C"
