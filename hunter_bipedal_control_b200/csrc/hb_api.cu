// libhunter_b200.so -- C ABI (include/hunter_b200.h) over the sm_90a kernels. Host side: context, scratch, launches.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>

#include "../../include/hunter_b200.h"
#include "hb_common.cuh"
#include "hb_mpc.cuh"
#include "hb_planner.h"
#include <algorithm>
#include <string>
#include <utility>
#include <atomic>
#include <mutex>
#include <cstring>
#include <thread>
#include <vector>
#include "hb_qp.cuh"
#include "hb_rbd.cuh"
#include "hb_sqp.cuh"
#include "hb_wbc.cuh"
#include "hb_hoqp.cuh"
#include "hb_rollout.cuh"

using namespace hb;

// ---------------------------------------------------------------------------------------------- kernels
namespace {

constexpr int QP_STRIDE_H = NWBC * NWBC, QP_STRIDE_A = WBC_ROWS * NWBC;

// input cost R = blkdiag(R_f, J0' R_v J0) with J0 the contact Jacobian at initialState (LeggedInterface.cpp:263-288)
__global__ void init_input_cost_kernel(double* Rout) {
  __shared__ double J0[12 * 16];
  const int lane = threadIdx.x;
  if (lane < 16) {
    double q[NQ], e[NQ];
    const double q0[NQ] = {HB_INITIAL_STATE[6], HB_INITIAL_STATE[7], HB_INITIAL_STATE[8], HB_INITIAL_STATE[9], HB_INITIAL_STATE[10], HB_INITIAL_STATE[11],
                           HB_INITIAL_STATE[12], HB_INITIAL_STATE[13], HB_INITIAL_STATE[14], HB_INITIAL_STATE[15], HB_INITIAL_STATE[16], HB_INITIAL_STATE[17],
                           HB_INITIAL_STATE[18], HB_INITIAL_STATE[19], HB_INITIAL_STATE[20], HB_INITIAL_STATE[21]};
    for (int i = 0; i < NQ; ++i) { q[i] = q0[i]; e[i] = (i == lane) ? 1.0 : 0.0; }
    KinOut<double> o;
    kin_pass<double>(q, e, o);
    for (int r = 0; r < 12; ++r) J0[r * 16 + lane] = o.cvel[r];
  }
  __syncthreads();
  const double rts[24] = {HB_R_TASKSPACE_DIAG[0], HB_R_TASKSPACE_DIAG[1], HB_R_TASKSPACE_DIAG[2], HB_R_TASKSPACE_DIAG[3], HB_R_TASKSPACE_DIAG[4], HB_R_TASKSPACE_DIAG[5],
                          HB_R_TASKSPACE_DIAG[6], HB_R_TASKSPACE_DIAG[7], HB_R_TASKSPACE_DIAG[8], HB_R_TASKSPACE_DIAG[9], HB_R_TASKSPACE_DIAG[10], HB_R_TASKSPACE_DIAG[11],
                          HB_R_TASKSPACE_DIAG[12], HB_R_TASKSPACE_DIAG[13], HB_R_TASKSPACE_DIAG[14], HB_R_TASKSPACE_DIAG[15], HB_R_TASKSPACE_DIAG[16], HB_R_TASKSPACE_DIAG[17],
                          HB_R_TASKSPACE_DIAG[18], HB_R_TASKSPACE_DIAG[19], HB_R_TASKSPACE_DIAG[20], HB_R_TASKSPACE_DIAG[21], HB_R_TASKSPACE_DIAG[22], HB_R_TASKSPACE_DIAG[23]};
  for (int idx = lane; idx < NU * NU; idx += 32) {
    const int i = idx / NU, j = idx - i * NU;
    double v = 0.0;
    if (i < 12 && i == j) v = rts[i];
    if (i >= 12 && j >= 12) for (int r = 0; r < 12; ++r) v += J0[r * 16 + 6 + i - 12] * rts[12 + r] * J0[r * 16 + 6 + j - 12];
    Rout[idx] = v;
  }
}

__global__ void qp_batch_kernel(int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA,
                                size_t strideH, size_t strideA, size_t strideB, const int32_t* m_per, double rho, int max_iter, double* x,
                                int32_t* status, int32_t* iters) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int inst = blockIdx.x * wpb + warp;
  if (inst >= B) return;
  double* base = reinterpret_cast<double*>(smem_raw) + (size_t)warp * qp_workspace_doubles(n);
  QpWorkspace w;
  qp_carve(base, n, w);
  const int mi = m_per ? m_per[inst] : m;
  QpResult r = qp_solve_warp(n, mi, H + inst * strideH, g + (size_t)inst * n, A + inst * strideA, lbA + inst * strideB, ubA + inst * strideB,
                             rho, max_iter, x + (size_t)inst * n, w);
  if (lane_id() == 0) { if (status) status[inst] = r.status; if (iters) iters[inst] = r.iters; }
}

__global__ void wbc_assemble_kernel(int B, hb_wbc_settings ws, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                                    const uint8_t* stance_mode, double* H, double* g, double* A, double* lbA, double* ubA, int32_t* m_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int inst = blockIdx.x * wpb + warp;
  if (inst >= B) return;
  WbcShared& sh = reinterpret_cast<WbcShared*>(smem_raw)[warp];
  const int m = wbc_assemble_warp(x_des + (size_t)inst * NX, u_des + (size_t)inst * NU, rbd + (size_t)inst * 32, mode[inst],
                                  stance_mode ? stance_mode[inst] != 0 : false, ws, sh, H + (size_t)inst * QP_STRIDE_H, g + (size_t)inst * NWBC,
                                  A + (size_t)inst * QP_STRIDE_A, lbA + (size_t)inst * WBC_ROWS, ubA + (size_t)inst * WBC_ROWS);
  if (lane_id() == 0) m_out[inst] = m;
}

// Fused WeightedWbc step (K5+K6): assembly terms, reduced QP (tau and swing forces eliminated), interior point, expansion to
// the reference's 38-vector [qdd, F, tau]. Shared memory per warp: QP workspace for n<=28 with the Hessian as a packed triangle (the
// assembly scratch aliases the factorisation area, which is dead until the first Newton step) + the reduced constraint matrix.
constexpr int WZ_N = 28, WZ_ME = 6, WZ_MI = 40, WZ_ROWS = 36;
__host__ __device__ constexpr size_t wbc_fused_doubles() { return qp_workspace_doubles(WZ_N, WZ_ME, WZ_MI, true) + WZ_ROWS * WZ_N + 2 * WZ_ROWS + 3 * WZ_N + 16 + 8; }
// One warp per block and one block per instance: 8 blocks per SM put a 1024-instance batch in one wave on 132 SMs (8 x 132 >= 1024;
// at 7 a tail wave of 100 blocks costs almost as much as the full one). The runtime reserves 1 KB of shared memory per block.
static_assert(8 * (wbc_fused_doubles() * sizeof(double) + 1024) <= 228 * 1024, "wbc_fused_kernel must fit 8 blocks per SM");

__global__ void __launch_bounds__(32, 8) wbc_fused_kernel(int B, hb_wbc_settings ws, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, const uint8_t* stance_mode,
                                 double rho, int max_iter, double* sol, int32_t* status, int32_t* iters) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
  const int inst = blockIdx.x * wpb + warp;
  if (inst >= B) return;
  double* base = reinterpret_cast<double*>(smem_raw) + (size_t)warp * wbc_fused_doubles();
  QpWorkspace w;
  qp_carve(base, WZ_N, w, WZ_ME, WZ_MI, true);
  double* p = base + qp_workspace_doubles(WZ_N, WZ_ME, WZ_MI, true);
  double* Az = p; p += WZ_ROWS * WZ_N;
  double* lbz = p; p += WZ_ROWS;
  double* ubz = p; p += WZ_ROWS;
  double* gz = p; p += WZ_N;
  double* xz = p; p += WZ_N;
  double* nlej = p; p += WZ_N;
  int* stcol = reinterpret_cast<int*>(p);
  static_assert(sizeof(WbcShared) <= sizeof(double) * (WZ_N * 29 + WZ_N * 7 + WZ_ME * 7 + WZ_N + WZ_ME + 6 * WZ_N + 5 * WZ_ME + 8 * WZ_MI), "assembly scratch must fit in the aliased area");
  WbcShared& sh = *reinterpret_cast<WbcShared*>(w.K);   // K, V, S, vectors: dead until the QP starts
  const int md = mode[inst];
  int nw = 0;
  wbc_assemble_warp(x_des + (size_t)inst * NX, u_des + (size_t)inst * NU, rbd + (size_t)inst * 32, md, stance_mode ? stance_mode[inst] != 0 : false, ws, sh,
                    nullptr, nullptr, nullptr, nullptr, nullptr, &nw);
  int m = 0;
  const int nz = wbc_reduced_build(sh, md, nw, stance_mode ? stance_mode[inst] != 0 : false, rho, ws, u_des + (size_t)inst * NU, w.H, gz, Az, lbz, ubz, stcol, m);
  if (lane < NJ) nlej[lane] = sh.nle[6 + lane];
  __syncwarp();
  // the workspace is carved for n = 28 (leading dimension 29); smaller problems (nz = 22, 16) use the same leading dimension
  QpResult r = qp_solve_warp<true>(nz, m, nullptr, gz, Az, lbz, ubz, 0.0, max_iter, xz, w);
  __syncwarp();
  double* out = sol + (size_t)inst * NWBC;
  if (lane < NQ) out[lane] = xz[lane];
  if (lane < 12) {
    double f = 0.0;
    for (int c = 0; c < nz - NQ; ++c) if (stcol[c] == lane) f = xz[NQ + c];
    out[NQ + lane] = f;
  }
  if (lane < NJ) {
    double t = nlej[lane];
    for (int c = 0; c < nz; ++c) t += Az[(6 + lane) * nz + c] * xz[c];
    out[NQ + 12 + lane] = t;
  }
  if (lane == 0) { if (status) status[inst] = r.status; if (iters) iters[inst] = r.iters; }
}

// ---------------------------------------------------------------------------------------------- hierarchical WBC (row N4)
__global__ void __launch_bounds__(32) hoqp_kernel(int B, const hb_hoqp_problem* problems, double* scratch, int max_iter, double* x, double* slack, int32_t* status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int inst = blockIdx.x;
  if (inst >= B) return;
  HoqpShared& sh = *reinterpret_cast<HoqpShared*>(smem_raw);
  QpWorkspace w;
  qp_carve(reinterpret_cast<double*>(smem_raw + sizeof(HoqpShared)), HQ_NQ, w, 1, HQ_ROWS);
  const int st = hoqp_solve_warp(problems[inst], sh, w, scratch + (size_t)inst * HQ_SCRATCH, max_iter, x + (size_t)inst * HQ_N, slack ? slack + (size_t)inst * HQ_STK : nullptr);
  if (status && threadIdx.x == 0) status[inst] = st;
}

// The three tasks of HierarchicalWbc::update from the WBC terms of one instance (decision vector [qdd(16), F(12), tau(10)]):
//   task0 = formulateFloatingBaseEomTask + formulateTorqueLimitsTask + formulateFrictionConeTask + formulateNoContactMotionTask
//   task1 = formulateBaseAccelTask          task2 = formulateContactForceTask * 0.1 + formulateSwingLegTask * 1     (WbcBase.cpp:138-338)
__global__ void __launch_bounds__(32) hwbc_tasks_kernel(int B, hb_wbc_settings ws, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                                                        hb_hoqp_problem* problems) {
  __shared__ WbcShared sh;
  const int inst = blockIdx.x, lane = threadIdx.x;
  if (inst >= B) return;
  const int md_ = mode[inst];
  int nw = 0;
  wbc_assemble_warp(x_des + (size_t)inst * NX, u_des + (size_t)inst * NU, rbd + (size_t)inst * 32, md_, false, ws, sh, nullptr, nullptr, nullptr, nullptr, nullptr, &nw);
  hb_hoqp_problem& pb = problems[inst];
  bool fl[4]; int nc = 0;
  for (int c = 0; c < 4; ++c) { fl[c] = contact_flag(md_, c); nc += fl[c]; }
  const int nsw = 4 - nc;
  const int ma0 = 16 + 3 * nsw + 3 * nc, md0 = 20 + 5 * nc, ma1 = 6, ma2 = 12 + 3 * nsw;
  if (lane == 0) { pb.n = NWBC; pb.levels = 3; pb.ma[0] = ma0; pb.md[0] = md0; pb.ma[1] = ma1; pb.md[1] = 0; pb.ma[2] = ma2; pb.md[2] = 0; }
  for (int idx = lane; idx < HB_HOQP_MAX_EQ * NWBC; idx += 32) { (&pb.a[0][0][0])[idx] = 0.0; (&pb.a[1][0][0])[idx] = 0.0; (&pb.a[2][0][0])[idx] = 0.0; }
  for (int idx = lane; idx < HB_HOQP_MAX_IN * NWBC; idx += 32) (&pb.d[0][0][0])[idx] = 0.0;
  __syncwarp();
  // task0 equalities: EoM rows [M | -J' | -S'] x = -nle
  for (int idx = lane; idx < 16 * NWBC; idx += 32) {
    const int i = idx / NWBC, j = idx - i * NWBC;
    double a;
    if (j < NQ) a = sh.M[i * 16 + j];
    else if (j < NQ + 12) a = -sh.J[(j - NQ) * 16 + i];
    else a = (i >= 6 && j - NQ - 12 == i - 6) ? -1.0 : 0.0;
    pb.a[0][i][j] = a;
  }
  if (lane < 16) pb.b[0][lane] = -sh.nle[lane];
  if (lane == 0) {
    int r = 16;
    for (int c = 0; c < 4; ++c) if (!fl[c]) for (int a = 0; a < 3; ++a) { pb.a[0][r][NQ + 3 * c + a] = 1.0; pb.b[0][r] = 0.0; ++r; }      // zero swing force
    for (int c = 0; c < 4; ++c) if (fl[c]) for (int a = 0; a < 3; ++a) {                                                                  // no contact motion
      for (int j = 0; j < NQ; ++j) pb.a[0][r][j] = sh.J[(3 * c + a) * 16 + j];
      pb.b[0][r] = -sh.dJv[3 * c + a]; ++r;
    }
    // task0 inequalities: torque limits, friction pyramid
    int q = 0;
    for (int sgn = 0; sgn < 2; ++sgn) for (int j = 0; j < NJ; ++j) { pb.d[0][q][NQ + 12 + j] = sgn == 0 ? 1.0 : -1.0; pb.f[0][q] = ws.torque_limits[j % 5]; ++q; }
    const double mu = ws.friction_coefficient;
    const double pyr[5][3] = {{0, 0, -1}, {1, 0, -mu}, {-1, 0, -mu}, {0, 1, -mu}, {0, -1, -mu}};
    for (int c = 0; c < 4; ++c) if (fl[c]) for (int k = 0; k < 5; ++k) { for (int a = 0; a < 3; ++a) pb.d[0][q][NQ + 3 * c + a] = pyr[k][a]; pb.f[0][q] = 0.0; ++q; }
    // task2 first part: 0.1 * (F = F_des)
    for (int j = 0; j < 12; ++j) { pb.a[2][j][NQ + j] = 0.1; pb.b[2][j] = 0.1 * u_des[(size_t)inst * NU + j]; }
  }
  // task1: base acceleration rows (the weighted formulation's base rows with the weight divided out); task2 second part: swing rows
  const int nswr = 3 * nsw;
  for (int idx = lane; idx < 6 * NQ; idx += 32) { const int i = idx / NQ, j = idx - i * NQ; pb.a[1][i][j] = sh.Aw[(nswr + i) * 16 + j] / ws.weight_base_accel; }
  if (lane < 6) pb.b[1][lane] = sh.bw[nswr + lane] / ws.weight_base_accel;
  for (int idx = lane; idx < nswr * NQ; idx += 32) { const int i = idx / NQ, j = idx - i * NQ; pb.a[2][12 + i][j] = sh.Aw[i * 16 + j] / ws.weight_swing_leg; }
  if (lane < nswr) pb.b[2][12 + lane] = sh.bw[lane] / ws.weight_swing_leg;
}

// LeggedRobotInitializer::compute (initialization/LeggedRobotInitializer.cpp:67-77)
__global__ void cold_start_kernel(int B, int N, const double* x0, const int32_t* mode, double* xt, double* ut) {
  const int inst = blockIdx.x;
  const double* x = x0 + (size_t)inst * NX;
  for (int idx = threadIdx.x; idx < (N + 1) * NX; idx += blockDim.x) xt[(size_t)inst * (N + 1) * NX + idx] = x[idx % NX];
  for (int idx = threadIdx.x; idx < N * NU; idx += blockDim.x) {
    const int k = idx / NU, j = idx - k * NU;
    const int md = mode[(size_t)inst * (N + 1) + k];
    int ns = 0;
    for (int c = 0; c < 4; ++c) ns += contact_flag(md, c);
    double v = 0.0;
    if (j < 12 && (j % 3) == 2 && contact_flag(md, j / 3)) v = c_model.total_mass * HB_GRAVITY / ns;
    ut[(size_t)inst * N * NU + idx] = v;
  }
}

// index k of the interval [tk[k], tk[k+1]) of a grid with n intervals that holds t (clamped to 0 .. n-1), and the interpolation weight
__device__ __forceinline__ int grid_interval(const double* tk, int n, double t, double& al) {
  int lo = 0, hi = n;                     // invariant: tk[lo] <= t (or lo == 0), tk[hi] > t (or hi == n)
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (tk[mid] <= t) lo = mid; else hi = mid; }
  const double d = tk[lo + 1] - tk[lo];
  double a = d > 0.0 ? (t - tk[lo]) / d : 0.0;
  al = a < 0.0 ? 0.0 : (a > 1.0 ? 1.0 : a);
  return lo;
}

// Warm start of the next solve from the resident primal solution (ocs2::SqpSolver::initializeStateInputTrajectories; mpc.coldStart
// false, task.info:146): x[0] = measured state; interval i takes u[i] = previous input at t_i and x[i+1] = previous state at t_{i+1}
// while t_{i+1} lies inside the previous horizon, otherwise the initializer (weight-compensating input, state kept,
// LeggedRobotInitializer.cpp:67-77). One block per instance; the previous trajectories are staged in shared memory so that the
// update can be done in place. With event-node grids (tk_new != null) both the previous and the new node times are arbitrary:
// tk_res / nn_res hold the previous grid and are replaced by the new one at the end.
__global__ void __launch_bounds__(128) warm_shift_kernel(int B, int N, double dt, const double* t0_new, double* t0_res, const double* x0,
                                                          const int32_t* mode, double* xt, double* ut, const double* tk_new, const int32_t* nn_new,
                                                          double* tk_res, int32_t* nn_res) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* px = reinterpret_cast<double*>(smem_raw);
  double* pu = px + (size_t)(N + 1) * NX;
  __shared__ double ptk[HB_MAX_HORIZON + 1];
  const int inst = blockIdx.x;
  const bool grid = tk_new != nullptr;
  double* x = xt + (size_t)inst * (N + 1) * NX; double* u = ut + (size_t)inst * N * NU;
  for (int i = threadIdx.x; i < (N + 1) * NX; i += blockDim.x) px[i] = x[i];
  for (int i = threadIdx.x; i < N * NU; i += blockDim.x) pu[i] = u[i];
  const int np = grid ? nn_res[inst] : N;                        // intervals of the previous grid
  const int nw = grid ? nn_new[inst] : N;                        // intervals of the new grid
  const double* tn_ = grid ? tk_new + (size_t)inst * (N + 1) : nullptr;
  if (grid) for (int i = threadIdx.x; i <= N; i += blockDim.x) ptk[i] = tk_res[(size_t)inst * (N + 1) + i];
  __syncthreads();
  const double tp = grid ? ptk[0] : t0_res[inst], tn = t0_new[inst], t_end = grid ? ptk[np] : tp + N * dt;
  auto new_time = [&](int k) { return grid ? tn_[k < nw ? k : nw] : tn + k * dt; };
  auto locate = [&](double t, double& al) {
    if (grid) return grid_interval(ptk, np, t, al);
    double s = (t - tp) / dt; s = s < 0.0 ? 0.0 : (s > (double)N ? (double)N : s);
    int k = (int)floor(s); if (k >= N) k = N - 1;
    al = s - k;
    return k;
  };
  auto prev_state = [&](double t, int j) { double al; const int k = locate(t, al); return (1.0 - al) * px[k * NX + j] + al * px[(k + 1) * NX + j]; };
  auto prev_input = [&](double t, int j) {
    double al; const int k = locate(t, al);
    const int k1 = (k + 1 < np) ? k + 1 : np - 1;
    return (1.0 - al) * pu[k * NU + j] + al * pu[k1 * NU + j];
  };
  // first interval that falls back to the initializer: smallest i with t_{i+1} > t_end (1e-9 guards the grid-aligned case)
  int istar = nw;
  for (int i = 0; i < nw; ++i) if (new_time(i + 1) > t_end + 1e-9) { istar = i; break; }
  for (int idx = threadIdx.x; idx < (N + 1) * NX; idx += blockDim.x) {
    const int k = idx / NX, j = idx - k * NX;
    const int ks = k <= istar ? k : istar;                 // the initializer keeps the state of node istar
    x[idx] = (ks == 0) ? x0[(size_t)inst * NX + j] : prev_state(new_time(ks), j);
  }
  for (int idx = threadIdx.x; idx < N * NU; idx += blockDim.x) {
    const int k = idx / NU, j = idx - k * NU;
    double v;
    if (k < istar) v = prev_input(new_time(k), j);
    else {
      const int md = mode[(size_t)inst * (N + 1) + k];
      int ns = 0;
      for (int c = 0; c < 4; ++c) ns += contact_flag(md, c);
      v = (j < 12 && (j % 3) == 2 && contact_flag(md, j / 3)) ? c_model.total_mass * HB_GRAVITY / ns : 0.0;
    }
    u[idx] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) { t0_res[inst] = tn; if (grid) nn_res[inst] = nw; }
  if (grid) for (int i = threadIdx.x; i <= N; i += blockDim.x) tk_res[(size_t)inst * (N + 1) + i] = tn_[i];
}

// MPC_MRT_Interface::evaluatePolicy with the feed-forward policy (LeggedController.cpp:154-156, task.info:93):
// linear interpolation of the state / input trajectories at t0 + t_rel; mode = mode in force at that time.
__global__ void policy_eval_kernel(int B, int N, double dt, double t_rel, const double* xt, const double* ut, const int32_t* mode, double* x_des,
                                   double* u_des, int32_t* mode_out, const double* tk, const int32_t* nn, const double* t_abs, const double* t0res) {
  const int inst = blockIdx.x * blockDim.x / 32 + (threadIdx.x >> 5);
  if (inst >= B) return;
  const int lane = threadIdx.x & 31;
  if (t_abs) t_rel = t_abs[inst] - t0res[inst];        // evaluation at an absolute time per instance (500 Hz WBC ticks between MPC updates)
  int k, na = N;
  double al;
  if (tk) {      // event-node grid: node times of this instance
    const double* t = tk + (size_t)inst * (N + 1);
    na = nn[inst];
    k = grid_interval(t, na, t[0] + t_rel, al);
  } else {
    double s = t_rel / dt;
    if (s < 0.0) s = 0.0;
    if (s > (double)N) s = (double)N;
    k = (int)floor(s);
    if (k >= N) k = N - 1;
    al = s - k;
  }
  const double* x = xt + (size_t)inst * (N + 1) * NX;
  const double* u = ut + (size_t)inst * N * NU;
  if (lane < NX) {
    x_des[(size_t)inst * NX + lane] = (1.0 - al) * x[k * NX + lane] + al * x[(k + 1) * NX + lane];
    const int k1 = (k + 1 < na) ? k + 1 : na - 1;   // the input trajectory repeats its last sample at the final node
    u_des[(size_t)inst * NU + lane] = (1.0 - al) * u[k * NU + lane] + al * u[k1 * NU + lane];
  }
  if (lane == 0 && mode_out) mode_out[inst] = mode[(size_t)inst * (N + 1) + k];
}

// torque law (LeggedController.cpp:181-184): feed-forward joint torques = tail(10) of the WBC solution
__global__ void torque_kernel(int B, const double* sol, double* torque) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < B * NJ) { const int i = idx / NJ, j = idx - i * NJ; torque[idx] = sol[(size_t)i * NWBC + 28 + j]; }
}

// joint command law (LeggedController.cpp:186-257), one thread per instance; joints are visited in order because the limit
// protection of joint j only affects the commands of joints >= j within the same cycle
__global__ void joint_command_kernel(int B, hb_pd_gains g, double dt, const double* x_des, const double* u_des, const double* sol,
                                     const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded, uint8_t* estop, double* command,
                                     double* out_tau) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const double* xd = x_des + (size_t)inst * NX; const double* ud = u_des + (size_t)inst * NU;
  const double* ws = sol + (size_t)inst * NWBC; const double* r = rbd + (size_t)inst * 32;
  const bool is_loaded = loaded ? loaded[inst] != 0 : true;
  bool stop = estop ? estop[inst] != 0 : false;
  const int mode = mode_cmd[inst];
  for (int j = 0; j < NJ; ++j) {
    const double q = r[6 + j], qd = r[NQ + 6 + j];
    if (!stop && is_loaded && (q > c_model.joint_upper[j] + 0.02 || q < c_model.joint_lower[j] - 0.02)) stop = true;
    double pd, vd, kp, kd, ff;
    if (!is_loaded) {
      pd = xd[12 + j]; vd = ud[12 + j]; kp = g.kp_position; kd = (j == 4 || j == 9) ? g.kd_feet : g.kd_position; ff = 0.0;
    } else {
      const double qdd = ws[6 + j];
      pd = xd[12 + j] + 0.5 * qdd * dt * dt; vd = ud[12 + j] + qdd * dt; ff = ws[28 + j];
      const bool contact = contact_flag(mode, j / 5);
      if (j == 0 || j == 1 || j == 5 || j == 6) { kp = contact ? g.kp_small_stance : g.kp_small_swing; kd = g.kd_small; }
      else if (j == 4 || j == 9) { kp = contact ? g.kp_small_stance : g.kp_small_swing; kd = g.kd_feet; }
      else { kp = contact ? g.kp_big_stance : g.kp_big_swing; kd = g.kd_big; }
    }
    if (stop) { pd = 0.0; vd = 0.0; kp = 0.0; kd = 1.0; ff = 0.0; }
    double* c = command + ((size_t)inst * NJ + j) * 5;
    c[0] = pd; c[1] = vd; c[2] = kp; c[3] = kd; c[4] = ff;
    out_tau[(size_t)inst * NJ + j] = ff + kp * (pd - q) + kd * (vd - qd);
  }
  if (estop) estop[inst] = stop ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------- state estimator (row N3)
// KalmanFilterEstimate::update (legged_estimation/src/LinearKalmanFilter.cpp:72-185), one warp per instance. The constant matrices
// of the filter are never formed: A = I + dt E (position <- velocity), C = rows of +-1 (foot - base position, base velocity,
// foot height), so A P A' and C M are index arithmetic. With S = C Pm C' + R = L L', Y = L^-1 C Pm and z = L^-1 (y - C x):
//   x <- x + Y' z ,  P <- Pm - Y' Y   ( = (I - Pm C' S^-1 C) Pm, symmetric by construction).
struct KfShared {
  double P[18 * 18], Pm[18 * 18], T[28 * 18], S[28 * 29], Y[28 * 18];
  double x[18], ey[28], z[28], sdi[28], qd[18], rd[28];
};
// row r of C applied to the 18 rows of a matrix stored row-major with leading dimension ld: (C M)[r][c]
__device__ __forceinline__ double kf_c_row(const double* M, int ld, int r, int c) {
  if (r < 12) return M[(r % 3) * ld + c] - M[(6 + r) * ld + c];
  if (r < 24) return M[(3 + (r % 3)) * ld + c];
  return M[(8 + 3 * (r - 24)) * ld + c];
}
__global__ void __launch_bounds__(32) kf_update_kernel(int B, hb_kf_params prm, double dt, hb_kf_state* state, const double* quat, const double* angl,
                                                       const double* accl, const double* jpos, const double* jvel, const uint8_t* cflag, double* rbd_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  KfShared& sh = *reinterpret_cast<KfShared*>(smem_raw);
  const int inst = blockIdx.x, lane = threadIdx.x;
  hb_kf_state& st = state[inst];
  // ---- updateImu: quaternion -> ZYX angles, local angular velocity -> Euler rates -> global angular velocity (every lane, registers)
  const double qx = quat[4 * inst], qy = quat[4 * inst + 1], qz = quat[4 * inst + 2], qw = quat[4 * inst + 3];
  double zyx[3];
  zyx[0] = atan2(2.0 * (qx * qy + qw * qz), qw * qw + qx * qx - qy * qy - qz * qz);
  zyx[1] = asin(fmin(-2.0 * (qx * qz - qw * qy), .99999));
  zyx[2] = atan2(2.0 * (qy * qz + qw * qx), qw * qw - qx * qx - qy * qy + qz * qz);
  double sz, cz, sy, cy, sx, cx;
  sincos(zyx[0], &sz, &cz); sincos(zyx[1], &sy, &cy); sincos(zyx[2], &sx, &cx);
  const double wlx = angl[3 * inst], wly = angl[3 * inst + 1], wlz = angl[3 * inst + 2];
  const double dzr = (sx * wly + cx * wlz) / cy, dyr = cx * wly - sx * wlz, dxr = wlx + sy * dzr;   // yaw, pitch, roll rates
  const double wg[3] = {-sz * dyr + cy * cz * dxr, cz * dyr + cy * sz * dxr, dzr - sy * dxr};
  // ---- contact kinematics with the base at the origin and zero base linear velocity (:84-100)
  double q[NQ], v[NQ];
  q[0] = q[1] = q[2] = 0.0; q[3] = zyx[0]; q[4] = zyx[1]; q[5] = zyx[2];
  v[0] = v[1] = v[2] = 0.0;
  {
    const double r = (cz * wg[0] + sz * wg[1]) / cy;      // getEulerAnglesZyxDerivativesFromGlobalAngularVelocity
    v[5] = r; v[4] = -sz * wg[0] + cz * wg[1]; v[3] = wg[2] + sy * r;
  }
  for (int j = 0; j < NJ; ++j) { q[6 + j] = jpos[(size_t)inst * NJ + j]; v[6 + j] = jvel[(size_t)inst * NJ + j]; }
  KinOut<double> ko;
  kin_pass<double>(q, v, ko);
  // world acceleration (:133-134)
  double acc[3];
  {
    const double R[9] = {cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx, sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx, -sy, cy * sx, cy * cx};
    const double a0 = accl[3 * inst], a1 = accl[3 * inst + 1], a2 = accl[3 * inst + 2];
    acc[0] = R[0] * a0 + R[1] * a1 + R[2] * a2; acc[1] = R[3] * a0 + R[4] * a1 + R[5] * a2; acc[2] = R[6] * a0 + R[7] * a1 + R[8] * a2 - 9.81;
  }
  // ---- noise covariances (diagonal), prediction of the state
  for (int i = lane; i < 324; i += 32) sh.P[i] = st.P[i];
  if (lane < 18) {
    const double xo = st.x_hat[lane];
    double xn = xo;
    if (lane < 3) xn = xo + dt * st.x_hat[3 + lane] + 0.5 * dt * dt * acc[lane];
    else if (lane < 6) xn = xo + dt * acc[lane - 3];
    sh.x[lane] = xn;
    double qv;
    if (lane < 3) qv = (dt / 20.0) * prm.imu_process_noise_position;
    else if (lane < 6) qv = (dt * (double)9.81f / 20.0) * prm.imu_process_noise_velocity;
    else qv = dt * prm.foot_process_noise_position * (cflag[4 * inst + (lane - 6) / 3] ? 1.0 : 100.0);
    sh.qd[lane] = qv;
  }
  if (lane < 28) {
    double rv;
    if (lane < 12) rv = prm.foot_sensor_noise_position * (cflag[4 * inst + lane / 3] ? 1.0 : 100.0);
    else if (lane < 24) rv = prm.foot_sensor_noise_velocity * (cflag[4 * inst + (lane - 12) / 3] ? 1.0 : 100.0);
    else rv = prm.foot_height_sensor_noise * (cflag[4 * inst + lane - 24] ? 1.0 : 100.0);
    sh.rd[lane] = rv;
  }
  __syncwarp();
  // Pm = A P A' + Q
  for (int idx = lane; idx < 324; idx += 32) {
    const int r = idx / 18, c = idx - 18 * r;
    double s = sh.P[idx];
    if (r < 3) s += dt * sh.P[(r + 3) * 18 + c];
    if (c < 3) s += dt * sh.P[r * 18 + c + 3];
    if (r < 3 && c < 3) s += dt * dt * sh.P[(r + 3) * 18 + c + 3];
    if (r == c) s += sh.qd[r];
    sh.Pm[idx] = s;
  }
  // innovation y - C x (:137-143): ps = -eePos (+ footRadius on z), vs = -eeVel, feet heights
  if (lane < 28) {
    double y;
    if (lane < 12) y = -ko.cpos[lane] + ((lane % 3) == 2 ? prm.foot_radius : 0.0);
    else if (lane < 24) y = -ko.cvel[lane - 12];
    else y = st.feet_heights[lane - 24];
    sh.ey[lane] = y - kf_c_row(sh.x, 1, lane, 0);
  }
  __syncwarp();
  // T = C Pm (28 x 18), S = T C' + R (28 x 28, ld 29; C' applied to the columns = C applied to the rows of T')
  for (int idx = lane; idx < 28 * 18; idx += 32) { const int r = idx / 18, c = idx - 18 * r; sh.T[idx] = kf_c_row(sh.Pm, 18, r, c); }
  __syncwarp();
  for (int idx = lane; idx < 28 * 28; idx += 32) {
    const int i = idx / 28, j = idx - 28 * i;
    const double* Ti = sh.T + i * 18;
    double s;
    if (j < 12) s = Ti[j % 3] - Ti[6 + j];
    else if (j < 24) s = Ti[3 + (j % 3)];
    else s = Ti[8 + 3 * (j - 24)];
    if (i == j) s += sh.rd[i];
    sh.S[i * 29 + j] = s;
  }
  __syncwarp();
  warp_chol_inv(sh.S, 28, 29, sh.sdi, lane);
  // Y = L^-1 T (28 x 18), z = L^-1 ey
  for (int idx = lane; idx < 28 * 18; idx += 32) {
    const int i = idx / 18, c = idx - 18 * i;
    double s = sh.sdi[i] * sh.T[i * 18 + c];
    for (int k = 0; k < i; ++k) s = fma(sh.S[k * 29 + i], sh.T[k * 18 + c], s);
    sh.Y[idx] = s;
  }
  warp_li_mv(sh.S, 28, 29, sh.sdi, sh.ey, sh.z, lane);
  __syncwarp();
  if (lane < 18) {
    double s = sh.x[lane];
    for (int k = 0; k < 28; ++k) s = fma(sh.Y[k * 18 + lane], sh.z[k], s);
    sh.x[lane] = s;
  }
  for (int idx = lane; idx < 324; idx += 32) {
    const int r = idx / 18, c = idx - 18 * r;
    double s = 0.5 * (sh.Pm[idx] + sh.Pm[c * 18 + r]);
    for (int k = 0; k < 28; ++k) s = fma(-sh.Y[k * 18 + r], sh.Y[k * 18 + c], s);
    sh.P[idx] = s;
  }
  __syncwarp();
  // :151-156: once the xy position is observed well enough, decouple it and shrink its covariance
  const bool decouple = sh.P[0] * sh.P[19] - sh.P[1] * sh.P[18] > 0.000001;
  for (int idx = lane; idx < 324; idx += 32) {
    const int r = idx / 18, c = idx - 18 * r;
    double vP = sh.P[idx];
    if (decouple) { if ((r < 2) != (c < 2)) vP = 0.0; else if (r < 2 && c < 2) vP /= 10.0; }
    st.P[idx] = vP;
  }
  if (lane < 18) st.x_hat[lane] = sh.x[lane];
  // ---- rbd state (StateEstimateBase.cpp:73-106): [zyx, p, q_j, omega_world, v, qd_j]
  double* rb = rbd_out + (size_t)inst * 32;
  if (lane < 3) { rb[lane] = zyx[lane]; rb[3 + lane] = sh.x[lane]; rb[16 + lane] = wg[lane]; rb[19 + lane] = sh.x[3 + lane]; }
  if (lane < NJ) { rb[6 + lane] = q[6 + lane]; rb[22 + lane] = v[6 + lane]; }
}

// ---------------------------------------------------------------------------------------------- contact-force estimate (row N3, second half)
// StateEstimateBase::estContactForce (legged_estimation/src/StateEstimateBase.cpp:130-206): generalised-momentum observer
//   p = M v,  pSCg = beta p + S' tau_cmd + C' v - g,  low-pass (gamma = exp(-lambda dt), beta = (1 - gamma) / (gamma dt)),  tau_d = beta p - filtered,
// then per foot the least-norm 6-D wrench w with (S_leg J_foot') w = S_leg tau_d (5 joint rows of the leg, toe frame Jacobian in world axes).
// One warp per instance; the terms Pinocchio provides are obtained as
//   M v  = inverse dynamics with acceleration v at zero velocity, no gravity;   g = inverse dynamics at rest with gravity;
//   C' v = d/dq (1/2 v' M(q) v) at fixed v (lane i = dual sweep seeded on q_i; valid for any C with dM/dt = C + C', as Pinocchio's).
struct ObsShared { double p[NQ], g[NQ], ctv[NQ], taud[NQ], Jf[2 * 5 * 6]; };
__global__ void __launch_bounds__(32) contact_force_kernel(int B, double lambda, double dt_in, hb_observer_state* state, const double* rbd, const double* tau_cmd,
                                                           double* est, double* disturbance) {
  __shared__ ObsShared sh;
  const int inst = blockIdx.x, lane = threadIdx.x;
  const double dt = dt_in > 1.0 ? 0.002 : dt_in;
  const double gama = exp(-lambda * dt), beta = (1.0 - gama) / (gama * dt);
  const double* r = rbd + (size_t)inst * 32;
  double q[NQ], v[NQ];
  for (int i = 0; i < 3; ++i) { q[i] = r[3 + i]; q[3 + i] = r[i]; v[i] = r[NQ + 3 + i]; }
  for (int j = 0; j < NJ; ++j) { q[6 + j] = r[6 + j]; v[6 + j] = r[NQ + 6 + j]; }
  {
    double sz, cz, sy, cy;
    sincos(q[3], &sz, &cz); sincos(q[4], &sy, &cy);
    const double dxr = (cz * r[NQ] + sz * r[NQ + 1]) / cy;      // getEulerAnglesZyxDerivativesFromGlobalAngularVelocity
    v[5] = dxr; v[4] = -sz * r[NQ] + cz * r[NQ + 1]; v[3] = r[NQ + 2] + sy * dxr;
  }
  if (lane < 3) sh.ctv[lane] = 0.0;                 // the kinetic energy does not depend on the base position
  else if (lane < NQ) {
    D1 qd[NQ], vd[NQ];
    for (int i = 0; i < NQ; ++i) { qd[i] = D1(q[i], i == lane ? 1.0 : 0.0); vd[i] = D1(v[i], 0.0); }
    KinOut<D1> o;
    kin_pass<D1>(qd, vd, o);
    sh.ctv[lane] = o.ke.d;
  } else if (lane == 16) {
    double zero[NQ], tau[NQ];
    for (int i = 0; i < NQ; ++i) zero[i] = 0.0;
    rnea_pass(q, zero, v, false, tau, nullptr);
    for (int i = 0; i < NQ; ++i) sh.p[i] = tau[i];
  } else if (lane == 17) {
    double zero[NQ], tau[NQ];
    for (int i = 0; i < NQ; ++i) zero[i] = 0.0;
    rnea_pass(q, zero, zero, true, tau, nullptr);
    for (int i = 0; i < NQ; ++i) sh.g[i] = tau[i];
  } else if (lane < 20) {
    // toe-frame Jacobian of leg `leg` with respect to its five joints, world axes: column j = [a_j x (p_toe - o_j) ; a_j]
    const int leg = lane - 18;
    double R[9], ax0[9], pj[3], o[5][3], a[5][3];
    base_frame(q, R, ax0);
    for (int i = 0; i < 3; ++i) pj[i] = q[i];
    for (int j = 0; j < 5; ++j) {
      const int b = 1 + 5 * leg + j;
      double d[3];
      rot_const(R, &c_model.joint_xyz[3 * b], d);
      for (int i = 0; i < 3; ++i) { pj[i] += d[i]; o[j][i] = pj[i]; }
      joint_rotate(R, c_model.joint_axis[b], q[5 + b], a[j]);
    }
    double off[3], toe[3];
    rot_const(R, &c_model.contact_offset[3 * leg], off);
    for (int i = 0; i < 3; ++i) toe[i] = pj[i] + off[i];
    for (int j = 0; j < 5; ++j) {
      double rr[3], lin[3];
      for (int i = 0; i < 3; ++i) rr[i] = toe[i] - o[j][i];
      cross(a[j], rr, lin);
      for (int i = 0; i < 3; ++i) { sh.Jf[(leg * 5 + j) * 6 + i] = lin[i]; sh.Jf[(leg * 5 + j) * 6 + 3 + i] = a[j][i]; }
    }
  }
  __syncwarp();
  hb_observer_state& st = state[inst];
  if (lane < NQ) {
    const double p = sh.p[lane];
    const double pscg = beta * p + (lane >= 6 ? tau_cmd[(size_t)inst * NJ + lane - 6] : 0.0) + sh.ctv[lane] - sh.g[lane];
    const double filt = (1.0 - gama) * pscg + gama * st.p_filtered[lane];
    st.p_filtered[lane] = filt;
    const double td = beta * p - filt;
    sh.taud[lane] = td;
    if (disturbance) disturbance[(size_t)inst * NQ + lane] = td;
  }
  __syncwarp();
  double* e = est + (size_t)inst * 16;
  if (lane < 2) {
    // least-norm solution of A w = b, A = S J' (5 x 6): w = A' (A A')^-1 b (the reference takes the SVD solve; same result at full row rank)
    const double* A = sh.Jf + lane * 30;          // row j = joint j of the leg, 6 columns
    double Gm[5][6];
    for (int i = 0; i < 5; ++i) {
      for (int j = 0; j < 5; ++j) { double s = 0.0; for (int c = 0; c < 6; ++c) s += A[i * 6 + c] * A[j * 6 + c]; Gm[i][j] = s; }
      Gm[i][5] = sh.taud[6 + 5 * lane + i];
    }
    for (int c = 0; c < 5; ++c) {
      int pv = c; double best = fabs(Gm[c][c]);
      for (int rr = c + 1; rr < 5; ++rr) if (fabs(Gm[rr][c]) > best) { best = fabs(Gm[rr][c]); pv = rr; }
      if (pv != c) for (int j = 0; j < 6; ++j) { const double t = Gm[c][j]; Gm[c][j] = Gm[pv][j]; Gm[pv][j] = t; }
      const double inv = 1.0 / Gm[c][c];
      for (int rr = c + 1; rr < 5; ++rr) { const double f = Gm[rr][c] * inv; for (int j = c; j < 6; ++j) Gm[rr][j] -= f * Gm[c][j]; }
    }
    double y[5];
    for (int rr = 4; rr >= 0; --rr) { double s = Gm[rr][5]; for (int j = rr + 1; j < 5; ++j) s -= Gm[rr][j] * y[j]; y[rr] = s / Gm[rr][rr]; }
    double w[6], n3 = 0.0, n6 = 0.0;
    for (int c = 0; c < 6; ++c) { double s = 0.0; for (int j = 0; j < 5; ++j) s += A[j * 6 + c] * y[j]; w[c] = s; n6 += s * s; if (c < 3) n3 += s * s; }
    for (int c = 0; c < 6; ++c) e[6 * lane + c] = w[c];
    e[12 + lane] = sqrt(n3);
    e[14 + lane] = sqrt(n6);
  }
}

// ---------------------------------------------------------------------------------------------- closed-loop rollout pieces (row N2)
// Actuation model of the simulated hardware (legged_gazebo/src/LeggedHWSim.cpp:166-192): every write pushes the hybrid joint command
// (posDes, velDes, kp, kd, ff) with its time stamp on a buffer, drops the entries older than `delay` from the far end, and applies the
// OLDEST remaining one: tau = kp (posDes - q) + kd (velDes - qd) + ff with the CURRENT joint state. One thread per instance; the deque is a
// ring of HB_ACT_CAPACITY entries (a full ring drops its oldest entry first).
__global__ void actuation_kernel(int B, double delay, const double* time, hb_actuation_state* state, const double* command, const double* rbd, double* tau) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  hb_actuation_state& st = state[inst];
  const double t = time[inst];
  int cnt = st.count, head = st.head;             // head = newest entry; entries head, head+1, ... (mod capacity) are older and older
  while (cnt > 0 && st.stamp[(head + cnt - 1) % HB_ACT_CAPACITY] + delay < t) --cnt;
  if (cnt == HB_ACT_CAPACITY) --cnt;
  head = (head + HB_ACT_CAPACITY - 1) % HB_ACT_CAPACITY;
  st.stamp[head] = t;
  for (int k = 0; k < NJ * 5; ++k) st.cmd[head][k] = command[(size_t)inst * NJ * 5 + k];
  ++cnt;
  st.count = cnt; st.head = head;
  const double* c = st.cmd[(head + cnt - 1) % HB_ACT_CAPACITY];
  const double* r = rbd + (size_t)inst * 32;
  for (int j = 0; j < NJ; ++j) tau[(size_t)inst * NJ + j] = c[5 * j + 2] * (c[5 * j] - r[6 + j]) + c[5 * j + 3] * (c[5 * j + 1] - r[NQ + 6 + j]) + c[5 * j + 4];
}

// One step of a batched rigid-body simulation of the robot on flat ground (stands in for the Gazebo / MuJoCo plant of the reference's
// closed loop, legged_gazebo / legged_mujoco): forward dynamics M(q) qdd = S' tau + J_c' F_c - nle with compliant point contacts at the four
// contact frames (normal spring-damper, viscous tangential friction clipped to the cone), semi-implicit Euler over `substeps` substeps.
// Same rigid-body passes as the WBC assembly: lanes 0-15 unit-velocity sweeps -> J_c columns, lanes 0-15 RNEA with unit accelerations ->
// M columns, lane 16 -> nle; 16 x 16 Cholesky in shared memory. One warp per instance.
struct SimShared { double q[NQ], v[NQ], J[12 * NQ], M[NQ * 17], nle[NQ], rhs[NQ], t1[NQ], t2[NQ], kdi[NQ], F[12], cpos[12], cvel[12]; };
__global__ void __launch_bounds__(32) sim_step_kernel(int B, hb_sim_params prm, double* rbd_io, const double* tau, double* contact_force, uint8_t* contact_flag) {
  __shared__ SimShared sh;
  const int inst = blockIdx.x, lane = threadIdx.x;
  double* r = rbd_io + (size_t)inst * 32;
  if (lane == 0) {
    for (int i = 0; i < 3; ++i) { sh.q[i] = r[3 + i]; sh.q[3 + i] = r[i]; sh.v[i] = r[NQ + 3 + i]; }
    for (int j = 0; j < NJ; ++j) { sh.q[6 + j] = r[6 + j]; sh.v[6 + j] = r[NQ + 6 + j]; }
    double sz, cz, sy, cy;
    sincos(sh.q[3], &sz, &cz); sincos(sh.q[4], &sy, &cy);
    const double dxr = (cz * r[NQ] + sz * r[NQ + 1]) / cy;
    sh.v[5] = dxr; sh.v[4] = -sz * r[NQ] + cz * r[NQ + 1]; sh.v[3] = r[NQ + 2] + sy * dxr;
  }
  __syncwarp();
  const double h = prm.dt / (prm.substeps > 0 ? prm.substeps : 1);
  for (int sub = 0; sub < (prm.substeps > 0 ? prm.substeps : 1); ++sub) {
    if (lane < NQ) {
      double q[NQ], e[NQ];
      for (int i = 0; i < NQ; ++i) { q[i] = sh.q[i]; e[i] = (i == lane) ? 1.0 : 0.0; }
      KinOut<double> o;
      kin_pass<double>(q, e, o);
      for (int rr = 0; rr < 12; ++rr) sh.J[rr * NQ + lane] = o.cvel[rr];
      if (lane == 0) for (int rr = 0; rr < 12; ++rr) sh.cpos[rr] = o.cpos[rr];
    }
    __syncwarp();
    if (lane < 12) { double s = 0.0; for (int i = 0; i < NQ; ++i) s += sh.J[lane * NQ + i] * sh.v[i]; sh.cvel[lane] = s; }
    __syncwarp();
    if (lane < 4) {
      const double depth = prm.ground_height - sh.cpos[3 * lane + 2];
      double fz = 0.0, fx = 0.0, fy = 0.0;
      if (depth > 0.0) {
        fz = prm.ground_stiffness * depth - prm.ground_damping * sh.cvel[3 * lane + 2];
        if (fz < 0.0) fz = 0.0;
        fx = -prm.tangential_damping * sh.cvel[3 * lane]; fy = -prm.tangential_damping * sh.cvel[3 * lane + 1];
        const double ft = sqrt(fx * fx + fy * fy), fmax_ = prm.friction_mu * fz;
        if (ft > fmax_) { const double sc = ft > 0.0 ? fmax_ / ft : 0.0; fx *= sc; fy *= sc; }
      }
      sh.F[3 * lane] = fx; sh.F[3 * lane + 1] = fy; sh.F[3 * lane + 2] = fz;
    }
    if (lane < 17) {
      double q[NQ], v[NQ], a[NQ], tq[NQ];
      for (int i = 0; i < NQ; ++i) { q[i] = sh.q[i]; v[i] = lane == 16 ? sh.v[i] : 0.0; a[i] = (i == lane) ? 1.0 : 0.0; }
      rnea_pass(q, v, a, lane == 16, tq, nullptr);
      if (lane < 16) { for (int rr = 0; rr < NQ; ++rr) sh.M[rr * 17 + lane] = tq[rr]; }
      else { for (int rr = 0; rr < NQ; ++rr) sh.nle[rr] = tq[rr]; }
    }
    __syncwarp();
    if (lane < NQ) {
      // joint side of the plant as in the reference's MuJoCo model (mujoco/model/hunter/hunter.xml:6): rotor armature on the diagonal of M,
      // viscous joint damping
      double s = -sh.nle[lane] + (lane >= 6 ? tau[(size_t)inst * NJ + lane - 6] - prm.joint_damping * sh.v[lane] : 0.0);
      for (int rr = 0; rr < 12; ++rr) s += sh.J[rr * NQ + lane] * sh.F[rr];
      sh.rhs[lane] = s;
      if (lane >= 6) sh.M[lane * 17 + lane] += prm.joint_armature;
      for (int j = lane + 1; j < NQ; ++j) { const double a = 0.5 * (sh.M[lane * 17 + j] + sh.M[j * 17 + lane]); sh.M[j * 17 + lane] = a; }   // lower triangle, symmetrised
    }
    __syncwarp();
    warp_chol_inv(sh.M, NQ, 17, sh.kdi, lane);
    warp_li_mv(sh.M, NQ, 17, sh.kdi, sh.rhs, sh.t1, lane);
    warp_lit_mv(sh.M, NQ, 17, sh.kdi, sh.t1, sh.t2, lane);      // t2 = qdd
    if (lane < NQ) { const double vn = sh.v[lane] + h * sh.t2[lane]; sh.v[lane] = vn; sh.q[lane] += h * vn; }
    __syncwarp();
  }
  if (lane == 0) {
    for (int i = 0; i < 3; ++i) { r[3 + i] = sh.q[i]; r[i] = sh.q[3 + i]; r[NQ + 3 + i] = sh.v[i]; }
    for (int j = 0; j < NJ; ++j) { r[6 + j] = sh.q[6 + j]; r[NQ + 6 + j] = sh.v[6 + j]; }
    double sz, cz, sy, cy;
    sincos(sh.q[3], &sz, &cz); sincos(sh.q[4], &sy, &cy);
    const double d0 = sh.v[3], d1 = sh.v[4], d2 = sh.v[5];      // yaw, pitch, roll rates -> world angular velocity
    r[NQ] = -sz * d1 + cz * cy * d2; r[NQ + 1] = cz * d1 + sz * cy * d2; r[NQ + 2] = d0 - sy * d2;
  }
  if (lane < 12 && contact_force) contact_force[(size_t)inst * 12 + lane] = sh.F[lane];
  if (lane < 4 && contact_flag) contact_flag[(size_t)inst * 4 + lane] = sh.F[3 * lane + 2] > 0.0 ? 1 : 0;
}

// computeCentroidalStateFromRbdModel (LeggedController.cpp:336)
__global__ void rbd_to_centroidal_kernel(int B, const double* rbd, double* x) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  rbd_to_centroidal(rbd + (size_t)inst * 32, x + (size_t)inst * NX);
}

// Expansion of the compact reference description onto the node grid (SwitchedModelReferenceManager::modifyReferences
// products evaluated where the solver needs them: TargetTrajectories::getDesiredState, ModeSchedule::modeAtTime,
// SwingTrajectoryPlanner::get{X,Y,Z}{position,velocity}Constraint; CubicSpline.cpp:46-124).
// Packed upload of hb_reference (host-pointer cycle): only the used entries of the fixed-capacity struct cross PCIe (about 3 KB instead of
// 17.7 KB per instance). Stream layout per instance, 8-byte words: header {n_events, n_targets, n_segments[12], 2 pad} (8 words),
// event_times, modes (as int32 pairs, padded), target_times, target_states, segments. `offs` (B + 1 words offsets) leads the stream.
struct RefPackHeader { int32_t n_events, n_targets, nseg[12], pad[2]; };
static_assert(sizeof(RefPackHeader) == 64, "header is 8 words");
__global__ void reference_unpack_kernel(int B, const long long* offs, const double* stream, hb_reference* refs) {
  const int inst = blockIdx.x;
  if (inst >= B) return;
  const double* p = stream + offs[inst];
  const RefPackHeader hd = *reinterpret_cast<const RefPackHeader*>(p);
  hb_reference& r = refs[inst];
  const int ne = min(max(hd.n_events, 0), HB_MAX_EVENTS), nt = min(max(hd.n_targets, 0), HB_MAX_TARGETS);
  p += 8;
  if (threadIdx.x == 0) { r.n_events = ne; r.n_targets = nt; for (int q = 0; q < 12; ++q) r.n_segments[q / 3][q % 3] = min(max(hd.nseg[q], 0), HB_MAX_SEGMENTS); }
  for (int i = threadIdx.x; i < ne; i += blockDim.x) r.event_times[i] = p[i];
  p += ne;
  const int32_t* pm = reinterpret_cast<const int32_t*>(p);
  for (int i = threadIdx.x; i <= ne; i += blockDim.x) r.modes[i] = pm[i];
  p += (ne + 2) / 2;
  for (int i = threadIdx.x; i < nt; i += blockDim.x) r.target_times[i] = p[i];
  p += nt;
  for (int i = threadIdx.x; i < nt * 22; i += blockDim.x) r.target_states[i / 22][i % 22] = p[i];
  p += nt * 22;
  for (int q = 0; q < 12; ++q) {
    const int ns = min(max(hd.nseg[q], 0), HB_MAX_SEGMENTS);
    double* dst = &r.segments[q / 3][q % 3][0][0];
    for (int i = threadIdx.x; i < ns * 6; i += blockDim.x) dst[i] = p[i];
    p += ns * 6;
  }
}

// The same copy without the host pass: when the caller's hb_reference array is pinned (cudaHostAlloc / cudaHostRegister) the block reads the
// USED entries straight out of host memory through the mapped alias (zero-copy), so no host core packs and only the used bytes cross PCIe.
__global__ void reference_gather_pinned_kernel(int B, const hb_reference* __restrict__ src, hb_reference* refs, unsigned long long* stat) {
  const int inst = blockIdx.x;
  if (inst >= B) return;
  const hb_reference& h = src[inst];
  hb_reference& r = refs[inst];
  __shared__ int cnt[14];
  __shared__ int bad;
  if (threadIdx.x == 0) { bad = 0; cnt[0] = min(max(h.n_events, 0), HB_MAX_EVENTS); if (cnt[0] != h.n_events) bad = 1; }
  __syncthreads();
  if (threadIdx.x == 1) { const int nt = h.n_targets; cnt[1] = min(max(nt, 0), HB_MAX_TARGETS); if (nt < 1 || nt > HB_MAX_TARGETS) bad = 1; }
  if (threadIdx.x >= 2 && threadIdx.x < 14) {
    const int q = threadIdx.x - 2, ns = h.n_segments[q / 3][q % 3];
    cnt[threadIdx.x] = min(max(ns, 0), HB_MAX_SEGMENTS);
    if (ns < 0 || ns > HB_MAX_SEGMENTS) bad = 1;
  }
  __syncthreads();
  const int ne = cnt[0], nt = cnt[1];
  if (threadIdx.x == 0) { r.n_events = ne; r.n_targets = nt; }
  if (threadIdx.x >= 2 && threadIdx.x < 14) { const int q = threadIdx.x - 2; r.n_segments[q / 3][q % 3] = cnt[threadIdx.x]; }
  // the checks of references_valid() ride on the copy: the values are in registers anyway
  bool ok = true;
  for (int i = threadIdx.x; i < ne; i += blockDim.x) {
    const double t = h.event_times[i];
    r.event_times[i] = t;
    if (!(t == t) || (i > 0 && t < h.event_times[i - 1])) ok = false;
  }
  for (int i = threadIdx.x; i <= ne; i += blockDim.x) { const int32_t m = h.modes[i]; r.modes[i] = m; if (m < 0 || m > 3) ok = false; }
  for (int i = threadIdx.x; i < nt; i += blockDim.x) {
    const double t = h.target_times[i];
    r.target_times[i] = t;
    if (!(t == t) || (i > 0 && !(t > h.target_times[i - 1]))) ok = false;
  }
  for (int i = threadIdx.x; i < nt * 22; i += blockDim.x) r.target_states[i / 22][i % 22] = h.target_states[i / 22][i % 22];
  // the twelve (foot, axis) segment lists in one flattened loop: all loads of the block are in flight together (PCIe round trips overlap)
  for (int i = threadIdx.x; i < 12 * HB_MAX_SEGMENTS * 6; i += blockDim.x) {
    const int q = i / (HB_MAX_SEGMENTS * 6), e = i - q * (HB_MAX_SEGMENTS * 6);
    if (e < cnt[2 + q] * 6) {
      const double* sp = &h.segments[q / 3][q % 3][0][0];
      const double v = sp[e];
      (&r.segments[q / 3][q % 3][0][0])[e] = v;
      if (e % 6 == 1 && !(v > sp[e - 1])) ok = false;       // segment end time after its start time
    }
  }
  if (!ok) bad = 1;
  __syncthreads();
  if (threadIdx.x == 0) {
    if (bad) atomicAdd(stat, 1ull);
    int words = 7 + ne + (ne + 2) / 2 + 23 * nt;
    for (int q = 0; q < 12; ++q) words += 6 * cnt[2 + q];
    atomicAdd(stat + 1, (unsigned long long)words);
  }
}

// Time discretisation with event nodes (row S1; ocs2::timeDiscretizationWithEvents as SqpSolver::run calls it): nodes step by dt from the
// initial time; a step that would pass a mode-switch time lands on it instead (the pre-event interval is shortened) and the grid
// re-anchors there; the last node is the final time; nodes closer than dt_min to their predecessor replace it. OCS2's duplicated
// pre- / post-event node pair (identity jump map, no cost, no constraint on it) is collapsed into one node that carries the post-event
// mode. One thread per instance; nn[inst] = number of intervals (<= N, the capacity); status 1 = capacity exhausted (last interval stretched).
__global__ void time_grid_kernel(int B, int N, double dt, double T, const double* t0, const hb_reference* refs, double* tk, int32_t* nn, int32_t* status) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const hb_reference& rf = refs[inst];
  const int nev = min(max(rf.n_events, 0), HB_MAX_EVENTS);
  double* t = tk + (size_t)inst * (N + 1);
  const double ti = t0[inst], tf = ti + T, dt_min = 1e-9;
  int ei = 0;
  while (ei < nev && rf.event_times[ei] <= ti + 1e-9) ++ei;      // switches at (or before) the initial time are in force already
  int n = 0, st = 0;
  double cur = ti;
  t[0] = ti;
  while (cur < tf) {
    double nx = cur + dt;
    if (ei < nev && nx >= rf.event_times[ei]) { nx = rf.event_times[ei]; ++ei; }
    if (nx >= tf) nx = tf;
    if (nx > cur + dt_min || n == 0) {
      if (n == N) { t[N] = tf; st = 1; break; }
      ++n;
    }
    t[n] = nx;
    cur = nx;
  }
  for (int k = n + 1; k <= N; ++k) t[k] = t[n];
  nn[inst] = n;
  if (status) status[inst] = st;
}

__global__ void reference_expand_kernel(int B, int N, double dt, const double* t0, const hb_reference* refs, double* x_ref, double* swing,
                                        int32_t* mode, const double* tk) {
  const int inst = blockIdx.x;
  const hb_reference& rf = refs[inst];
  // counts are clamped to the capacities of hb_reference: a malformed struct cannot index out of bounds (the host-pointer entry
  // points reject it with HB_EINVAL before it gets here; device-pointer callers own their data)
  const int n_events = min(max(rf.n_events, 0), HB_MAX_EVENTS), n_targets = min(max(rf.n_targets, 1), HB_MAX_TARGETS);
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    const double t = tk ? tk[(size_t)inst * (N + 1) + k] : t0[inst] + k * dt;
    // mode in force on the interval starting at t (post-event mode when t coincides with an event)
    int idx = 0;
    while (idx < n_events && rf.event_times[idx] <= t + 1e-9) ++idx;
    mode[(size_t)inst * (N + 1) + k] = rf.modes[idx];
    // target state: linear interpolation, clamped
    double* xr = x_ref + ((size_t)inst * (N + 1) + k) * NX;
    if (n_targets <= 1 || t <= rf.target_times[0]) { for (int i = 0; i < NX; ++i) xr[i] = rf.target_states[0][i]; }
    else if (t >= rf.target_times[n_targets - 1]) { for (int i = 0; i < NX; ++i) xr[i] = rf.target_states[n_targets - 1][i]; }
    else {
      int s = 0;
      while (s + 2 < n_targets && rf.target_times[s + 1] <= t) ++s;
      const double span = rf.target_times[s + 1] - rf.target_times[s];
      const double al = span > 0.0 ? (t - rf.target_times[s]) / span : 0.0;
      for (int i = 0; i < NX; ++i) xr[i] = (1.0 - al) * rf.target_states[s][i] + al * rf.target_states[s + 1][i];
    }
    // swing references: cubic Hermite segments
    double* sw = swing + ((size_t)inst * (N + 1) + k) * 24;
    for (int c = 0; c < 4; ++c)
      for (int a = 0; a < 3; ++a) {
        const int ns = min(max(rf.n_segments[c][a], 0), HB_MAX_SEGMENTS);
        double pos = 0.0, vel = 0.0;
        if (ns > 0) {
          int s = 0;
          while (s + 1 < ns && t >= rf.segments[c][a][s][1]) ++s;
          const double* sg = rf.segments[c][a][s];
          const double Tr = sg[1] - sg[0], T = Tr > 0.0 ? Tr : 1.0, tn = (t - sg[0]) / T;
          const double dp = sg[4] - sg[2], dvv = sg[5] - sg[3];
          const double c0 = sg[2], c1 = sg[3] * T, c2 = -(3.0 * sg[3] + dvv) * T + 3.0 * dp, c3 = (2.0 * sg[3] + dvv) * T - 2.0 * dp;
          pos = ((c3 * tn + c2) * tn + c1) * tn + c0;
          vel = ((3.0 * c3 * tn + 2.0 * c2) * tn + c1) / T;
        }
        sw[6 * c + a] = pos; sw[6 * c + 3 + a] = vel;
      }
  }
}

// InverseKinematics::computeFootPos: contact frame positions at the configuration of x (one thread per instance)
__global__ void contact_positions_kernel(int B, const double* x, double* pos) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  double q[NQ], v[NQ];
  for (int i = 0; i < NQ; ++i) { q[i] = x[(size_t)inst * NX + 6 + i]; v[i] = 0.0; }
  KinOut<double> o;
  kin_pass<double>(q, v, o);
  for (int i = 0; i < 12; ++i) pos[(size_t)inst * 12 + i] = o.cpos[i];
}

// plan_prepare_kernel unpacks t0 / x0 from the plan inputs and evaluates computeFootPos at x0 (the planner's current_feet input).
__global__ void plan_prepare_kernel(int B, const hb_plan_input* in, double* t0, double* x0, double* feet) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const hb_plan_input& p = in[inst];
  double q[NQ], v[NQ];
  for (int i = 0; i < NX; ++i) x0[(size_t)inst * NX + i] = p.x0[i];
  for (int i = 0; i < NQ; ++i) { q[i] = p.x0[6 + i]; v[i] = 0.0; }
  t0[inst] = p.t0;
  KinOut<double> o;
  kin_pass<double>(q, v, o);
  for (int i = 0; i < 12; ++i) feet[(size_t)inst * 12 + i] = o.cpos[i];
}

// Device planner (row N1): the same source as the host planner (csrc/hb_planner.h), four threads per instance (eight instances per 32-thread block). Thread 0 of an
// instance builds the two-sample target in shared memory, thread r plans foot r on it (the feet are independent), thread 0 resamples it,
// then threads 0 and 1 run the IK of the left / right leg on the resampled target, then thread 0 writes the schedule and the targets.
// Same functions as the host planner, so the plan is the same. The targets (2.9 KB each) live in shared memory only: no thread keeps
// a copy on its stack.
__global__ void __launch_bounds__(32) plan_references_coop_kernel(int B, const hb_plan_input* in, const double* feet, double* latest_stance,
                                                                  hb_reference* out, int32_t* status, hbplan::PlanConsts pc) {
  __shared__ hbplan::Target s_tg[8], s_old[8];
  __shared__ int s_rc[8];
  const int g = threadIdx.x >> 2, r = threadIdx.x & 3;
  const int inst = blockIdx.x * 8 + g;
  const bool active = inst < B;
  hb_plan_input p;
  hbplan::ModeSchedule ms;
  hb_reference* o = out + (active ? inst : 0);
  double t_lo = 0.0, t_hi = 0.0, tf = 0.0;
  int rc = 0;
  if (r == 0) s_rc[g] = 0;
  __syncwarp();
  if (active) {
    p = in[inst];
    if (feet) for (int i = 0; i < 12; ++i) p.feet_pos[i] = feet[(size_t)inst * 12 + i];
    if (!(p.horizon > 0.0) || !(p.prev_event < p.gait_start) || p.gait < 0 || p.gait > 3) rc = -1;
    tf = p.t0 + p.horizon; t_lo = p.t0 - 1e-9; t_hi = tf + 1e-9;
    if (rc == 0 && !hbplan::tile_gait(p.gait, p.prev_event, p.gait_start, p.t0 - p.horizon, tf + p.horizon, ms)) rc = -5;
    if (rc == 0 && r == 0) s_tg[g] = hbplan::cmd_vel_to_target(pc, p.cmd_vel, p.t0, p.x0, p.time_to_target);
  }
  __syncwarp();
  if (active && rc == 0) {     // rc is the same on the four threads of an instance here
    // phase A: foot r on the two-sample target
    const double body_vel_cmd[6] = {p.cmd_vel[0], p.cmd_vel[1], p.cmd_vel[2], p.cmd_vel[3], 0.0, 0.0};
    hbplan::SwingOut so{o, t_lo, t_hi, false};
    for (int a = 0; a < 3; ++a) o->n_segments[r][a] = 0;
    if (!hbplan::plan_swing(ms, s_tg[g], p.t0, p.feet_pos, body_vel_cmd, latest_stance + (size_t)inst * 12, so, r, r + 1) || so.overflow) rc = -5;
  }
  __syncwarp();                // every foot has read the two-sample target before thread 0 resamples it in place
  if (active) {
    if (rc == 0 && r == 0 && p.joint_ik && hbplan::joint_refs_resample(pc, p.t0, tf, s_tg[g], s_old[g]) < 0) rc = -5;
    if (rc != 0) atomicMin(&s_rc[g], rc);
  }
  __syncwarp();
  // phase B: IK per leg on the shared target (segments of every foot are in place after the barrier)
  if (active && s_rc[g] == 0 && p.joint_ik && s_tg[g].n > 2 && r < 2) hbplan::joint_refs_leg(pc, o, r, p.x0, s_tg[g]);
  __syncwarp();
  if (active && r == 0) {
    int frc = s_rc[g];
    if (frc == 0) frc = hbplan::write_schedule_and_targets(ms, s_tg[g], t_lo, t_hi, o);
    if (frc != 0) {
      o->n_events = 0; o->modes[0] = 3; o->n_targets = 1; o->target_times[0] = p.t0;
      for (int i = 0; i < 22; ++i) o->target_states[0][i] = (i < 6) ? 0.0 : p.x0[i];
      for (int c = 0; c < 4; ++c) for (int a = 0; a < 3; ++a) o->n_segments[c][a] = 0;
    }
    if (status) status[inst] = frc;
  }
}

// parity probe of the SHIPPING linearisation (lin_half of K0): flow map value, the full Jacobian tiles rebuilt from the compact
// record (rows 3..11 of df/dx, the force / joint-velocity blocks of df/du) and the contact kinematics with their Jacobians.
struct ProbeShared { LinHalf h[2]; ChainModel cm; double rec[LIN_STRIDE]; double dummy[LIN_STRIDE]; };
__global__ void __launch_bounds__(32) probe_flow_map_kernel(int B, const double* x, const double* u, double* f, double* A, double* Bm, double* ee) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ProbeShared& ps = *reinterpret_cast<ProbeShared*>(smem_raw);
  const int inst = blockIdx.x, lane = threadIdx.x, half = lane >> 4, hl = lane & 15;
  chain_model_load(ps.cm, threadIdx.x, blockDim.x);
  LinHalf& sh = ps.h[half];
  for (int i = hl; i < NX; i += 16) { sh.x[i] = x[(size_t)inst * NX + i]; sh.u[i] = u[(size_t)inst * NU + i]; }
  __syncwarp();
  // both halves linearise the same node; only half 0 writes the record (half 1 runs with act = false into a dummy record)
  double* rec = half == 0 ? ps.rec : ps.dummy;
  lin_half(sh, ps.cm, sh.x, hl, half == 0, rec + LIN_F1, rec + LIN_A1, rec + LIN_BF1, rec + LIN_BV1, true, rec);
  __syncwarp();
  const double im = 1.0 / c_model.total_mass;
  if (lane < NX) f[(size_t)inst * NX + lane] = ps.rec[LIN_F1 + lane];
  for (int idx = lane; idx < TS; idx += 32) {
    const int i = idx / NX, j = idx - i * NX;
    double a = 0.0, b = 0.0;
    if (i >= 3 && i < 12) a = ps.rec[LIN_A1 + (i - 3) * NX + j];
    if (j < 12) {
      if (i < 3) b = (j % 3 == i) ? im : 0.0;
      else if (i < 6) b = ps.rec[LIN_BF1 + (i - 3) * 12 + j];
    } else {
      if (i >= 6 && i < 12) b = ps.rec[LIN_BV1 + (i - 6) * NJ + j - 12];
      else if (i >= 12) b = (i == j) ? 1.0 : 0.0;
    }
    A[(size_t)inst * TS + idx] = a; Bm[(size_t)inst * TS + idx] = b;
  }
  if (ee) {
    double* o = ee + (size_t)inst * (24 + 3 * 12 * NX);
    if (lane < 12) { o[lane] = ps.rec[LIN_EPOS + lane]; o[12 + lane] = ps.rec[LIN_EVEL + lane]; }
    for (int idx = lane; idx < 12 * NX; idx += 32) {
      const int r = idx / NX, j = idx - r * NX;
      double dp = 0.0;
      if (j >= 6 && j < 9) dp = (j - 6 == r % 3) ? 1.0 : 0.0;
      else if (j >= 9) dp = ps.rec[LIN_DPQ + r * NDIR + j - 9];
      o[24 + idx] = dp;
      o[24 + 12 * NX + idx] = ps.rec[LIN_DVX + idx];
      o[24 + 24 * NX + idx] = (j >= 12) ? ps.rec[LIN_DVV + r * NJ + j - 12] : 0.0;
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------- context
struct hb_ctx {
  hb_config cfg;
  hb_wbc_settings wbc;       // WBC gains / limits / weights in force (task.info values by default; hb_wbc_set_settings, hb_load_task_info)
  int device;
  cudaStream_t stream;
  cudaStream_t stream_main, stream_aux;   // the chunked host-pointer calls pipeline their chunks over these
  int base;                               // instance offset into the per-instance scratch (chunked calls)
  int64_t launches;
  // MPC scratch
  double *dxt, *dut, *perf;
  double *lin, *proj, *rk;   // node records of the SQP pipeline (K0 -> K1 -> K2/K3)
  int32_t* flags;
  // WBC scratch: the control step's desired state / input / mode, the fused WBC's status and iterations when the caller passes none
  double *xdes, *udes;
  int32_t *wstatus, *witers, *wmode;
  double* hoqp_scratch; hb_hoqp_problem* hoqp_prob;   // hierarchical WBC (allocated by its first call)
  // hb_resident_cycle_batch_dev: references expanded over the horizon and, with event_nodes, the node grid they are expanded on
  double *cyc_xref, *cyc_swing, *cyc_tk;
  int32_t *cyc_mode, *cyc_nn;
  // resident primal solution (hb_resident_cycle_batch): solve time, trajectories, node modes (policy evaluation between MPC solves),
  // node times / interval counts (event-node grids)
  double *res_t0, *res_xt, *res_ut, *res_tk;
  int32_t *res_mode, *res_nn;
  int res_valid;                      // number of instances holding a previous solution
  double* res_sol; int res_sol_valid;   // last good WBC solution per instance (WeightedWbc fallback, W5)
  double* res_stance;                 // the device planner's latest stance positions (row N1)
  // hb_rollout_batch_dev's scratch, allocated at max_batch by its first call: commands, plan inputs -> planner -> cycle, the tick's WBC
  // solution / joint command / torques, the states held instances are put back to, the tick time
  void* ro_mem;
  hb_rollout_command* ro_cmd; hb_plan_input* ro_in; hb_reference* ro_refs; hb_solve_info* ro_info; int32_t* ro_pstat;
  double *ro_t0, *ro_x0, *ro_feet, *ro_sol, *ro_jcmd, *ro_jtau, *ro_tau, *ro_held, *ro_tnow;
  // host-call staging, sized on demand by the calls that use it (grow): the device arena Staging carves, and the pinned host buffer of
  // hb_resident_cycle_batch's packed references / reference verdicts
  void* arena; size_t arena_cap;
  void* pinned; size_t pinned_cap;
  int last_cuda;
  size_t last_h2d_bytes;     // bytes of packed references uploaded by the last hb_resident_cycle_batch
  // optional per-kernel event timing (hb_profile_enable / hb_profile_read)
  int prof_on, prof_n;
  cudaEvent_t* prof_ev;   // 2 * PROF_MAX events
  int* prof_kind;
};

namespace {

enum { HB_OK = 0, HB_EINVAL = -1, HB_ECUDA = -2, HB_ENOMEM = -3, HB_ECAP = -4, HB_EPLAN = -5, HB_ECOMM = -6 };

#define CK(call)                                   \
  do {                                             \
    cudaError_t e__ = (call);                      \
    if (e__ != cudaSuccess) { if (ctx) ctx->last_cuda = (int)e__; return HB_ECUDA; } \
  } while (0)

constexpr int PROF_MAX = 4096;
enum { K_UNPROFILED = -1, K_BACKWARD = 0, K_FORWARD_LS = 1, K_WBC_ASSEMBLE = 2, K_QP = 3, K_OTHER = 4, K_LIN = 5, K_LQ = 6, K_NKINDS = 7 };

template <class T> cudaError_t dalloc(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)); }

inline void prof_begin(hb_ctx* ctx, int kind) {
  if (ctx->prof_on && ctx->prof_n < PROF_MAX) { ctx->prof_kind[ctx->prof_n] = kind; cudaEventRecord(ctx->prof_ev[2 * ctx->prof_n], ctx->stream); }
}
inline void prof_end(hb_ctx* ctx) {
  if (ctx->prof_on && ctx->prof_n < PROF_MAX) { cudaEventRecord(ctx->prof_ev[2 * ctx->prof_n + 1], ctx->stream); ctx->prof_n++; }
}

// One kernel launch on ctx->stream: counted (hb_launch_count), timed under `kind` when profiling is on (K_UNPROFILED: never), launch
// error checked.
template <class... P, class... A>
int launch(hb_ctx* ctx, int kind, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  if (kind != K_UNPROFILED) prof_begin(ctx, kind);
  kernel<<<grid, block, smem, ctx->stream>>>(std::forward<A>(args)...);
  if (kind != K_UNPROFILED) prof_end(ctx);
  ctx->launches++;
  CK(cudaGetLastError());
  return HB_OK;
}

int set_device(hb_ctx* ctx) { return cudaSetDevice(ctx->device) == cudaSuccess ? HB_OK : HB_ECUDA; }

// The growth policy of the context's on-demand buffers (the staging arena, the pinned host buffer): grow only, to 5/4 of the request so
// that a packed reference stream a little longer than the last one does not reallocate, contents not kept. Every host-pointer call waits
// for its copies before it returns, so no copy still reads the buffer that is freed.
int grow(hb_ctx* ctx, void** buf, size_t* cap, size_t bytes, bool pinned_host) {
  if (bytes <= *cap) return HB_OK;
  if (*buf) { if (pinned_host) cudaFreeHost(*buf); else cudaFree(*buf); }
  *buf = nullptr; *cap = 0;
  const size_t want = bytes + bytes / 4;
  const cudaError_t e = pinned_host ? cudaHostAlloc(buf, want, cudaHostAllocDefault) : cudaMalloc(buf, want);
  if (e != cudaSuccess) { *buf = nullptr; ctx->last_cuda = (int)e; cudaGetLastError(); return HB_ENOMEM; }
  *cap = want;
  return HB_OK;
}

// Device side of one staged argument. Converts to its device pointer once Staging::reserve has placed it (null for a null pass-through
// argument); at(i) points at instance i (element i of a buf slice).
template <class T> struct Dev {
  void* const* p;
  size_t per;
  operator T*() const { return static_cast<T*>(*p); }
  T* at(size_t i) const { return static_cast<T*>(*p) + i * per; }
};

// Staging of one host-pointer call. The call declares its host arguments with their elements per instance; reserve() then places all of
// them in the context's device arena (grown on demand, freed by hb_destroy) before any copy is enqueued, and h2d / d2h copy instances
// [lo, hi) of every argument on ctx->stream. Slices start on 256-byte boundaries, as separate cudaMalloc's would.
//   in / inout   copied in (inout: and back)
//   out          the device always gets a buffer; copied back only when the caller passed a host pointer
//   *_or_null    a null host pointer stays a null device pointer
//   tmp / buf    device only: per instance (tmp) or n elements for the whole call (buf)
class Staging {
 public:
  Staging(hb_ctx* ctx, int B) : ctx_(ctx), B_((size_t)B) {}
  template <class T> Dev<const T> in(const T* h, size_t per) { return add<const T>(h, nullptr, per, B_, true); }
  template <class T> Dev<T> inout(T* h, size_t per) { return add<T>(h, h, per, B_, true); }
  template <class T> Dev<T> out(T* h, size_t per) { return add<T>(nullptr, h, per, B_, true); }
  template <class T> Dev<const T> in_or_null(const T* h, size_t per) { return add<const T>(h, nullptr, per, B_, h != nullptr); }
  template <class T> Dev<T> inout_or_null(T* h, size_t per) { return add<T>(h, h, per, B_, h != nullptr); }
  template <class T> Dev<T> tmp(size_t per) { return add<T>(nullptr, nullptr, per, B_, true); }
  template <class T> Dev<T> buf(size_t n) { Dev<T> d = add<T>(nullptr, nullptr, n, 1, true); d.per = 1; return d; }

  int reserve() {
    size_t total = 0;
    for (int k = 0; k < n_; ++k) if (s_[k].used) { s_[k].off = total; total += (s_[k].bytes * s_[k].count + 255) & ~(size_t)255; }
    const int rc = grow(ctx_, &ctx_->arena, &ctx_->arena_cap, total, false);
    if (rc) return rc;
    for (int k = 0; k < n_; ++k) if (s_[k].used) s_[k].dev = static_cast<char*>(ctx_->arena) + s_[k].off;
    return HB_OK;
  }
  int h2d(size_t lo, size_t hi) { return copy(lo, hi, true); }
  int d2h(size_t lo, size_t hi) { return copy(lo, hi, false); }
  // the whole batch in one piece: reserve, copy in, call(), copy out, wait
  template <class F> int run(F&& call) {
    int rc = reserve();
    if (!rc) rc = h2d(0, B_);
    if (!rc) rc = call();
    if (!rc) rc = d2h(0, B_);
    if (rc) return rc;
    hb_ctx* ctx = ctx_;
    CK(cudaStreamSynchronize(ctx->stream));
    return HB_OK;
  }

 private:
  struct Slot { const void* src; void* dst; size_t bytes, count, off; void* dev; bool used; };
  template <class T> Dev<T> add(const void* src, void* dst, size_t per, size_t count, bool used) {
    Slot& s = s_[n_++];
    s = Slot{src, dst, per * sizeof(T), count, 0, nullptr, used};
    return Dev<T>{&s.dev, per};
  }
  int copy(size_t lo, size_t hi, bool to_dev) {
    hb_ctx* ctx = ctx_;
    for (int k = 0; k < n_; ++k) {
      const Slot& s = s_[k];
      const size_t off = lo * s.bytes, n = (hi - lo) * s.bytes;
      if (to_dev && s.src) CK(cudaMemcpyAsync(static_cast<char*>(s.dev) + off, static_cast<const char*>(s.src) + off, n, cudaMemcpyHostToDevice, ctx->stream));
      if (!to_dev && s.dst) CK(cudaMemcpyAsync(static_cast<char*>(s.dst) + off, static_cast<char*>(s.dev) + off, n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    return HB_OK;
  }
  hb_ctx* ctx_;
  size_t B_;
  Slot s_[16];   // the largest call (hb_resident_plan_cycle_batch) declares 11
  int n_ = 0;
};

// The pipelined host-pointer calls: chunk c of nchunk covers instances [B c / nchunk, B (c + 1) / nchunk) on stream_main (even c) or
// stream_aux (odd c), so the copies of one chunk overlap the kernels of the other. ctx->stream / ctx->base point at the chunk while
// body(c, lo, hi) runs and are restored after the last one; both streams are drained before the first error is returned.
template <class F> int chunked(hb_ctx* ctx, int B, int nchunk, F&& body) {
  int rc = HB_OK;
  for (int c = 0; c < nchunk && rc == HB_OK; ++c) {
    const size_t lo = (size_t)B * c / nchunk, hi = (size_t)B * (c + 1) / nchunk;
    ctx->stream = (c % 2 == 0) ? ctx->stream_main : ctx->stream_aux;
    ctx->base = (int)lo;
    rc = body(c, lo, hi);
  }
  ctx->stream = ctx->stream_main;
  ctx->base = 0;
  cudaError_t e1 = cudaStreamSynchronize(ctx->stream_aux), e0 = cudaStreamSynchronize(ctx->stream_main);
  if (rc) return rc;
  if (e0 != cudaSuccess || e1 != cudaSuccess) { ctx->last_cuda = (int)(e0 != cudaSuccess ? e0 : e1); return HB_ECUDA; }
  return HB_OK;
}

// chunk count of the host-pointer cycles: cfg.e2e_chunks when set (one chunk below 64 instances per chunk), otherwise two from 4096
// instances on when the call has host work and copies to hide behind the other chunk's kernels (`overlap`)
int cycle_chunks(const hb_ctx* ctx, int B, bool overlap) {
  const int c = ctx->cfg.e2e_chunks;
  return c > 0 ? (B >= 64 * c ? c : 1) : ((overlap && B >= 4096) ? 2 : 1);
}

// Caller-supplied hb_reference structs (host-pointer entry points): counts within the capacities, monotone times, positive segment
// lengths, modes in 0..3. The device expansion indexes with these counts, so a malformed struct is rejected here with HB_EINVAL.
bool references_valid(int B, const hb_reference* refs) {
  for (int i = 0; i < B; ++i) {
    const hb_reference& r = refs[i];
    if (r.n_events < 0 || r.n_events > HB_MAX_EVENTS || r.n_targets < 1 || r.n_targets > HB_MAX_TARGETS) return false;
    for (int k = 0; k <= r.n_events; ++k) if (r.modes[k] < 0 || r.modes[k] > 3) return false;
    for (int k = 0; k < r.n_events; ++k) if (!(r.event_times[k] == r.event_times[k]) || (k > 0 && r.event_times[k] < r.event_times[k - 1])) return false;
    for (int k = 0; k < r.n_targets; ++k) if (!(r.target_times[k] == r.target_times[k]) || (k > 0 && !(r.target_times[k] > r.target_times[k - 1]))) return false;
    for (int c = 0; c < 4; ++c)
      for (int a = 0; a < 3; ++a) {
        const int ns = r.n_segments[c][a];
        if (ns < 0 || ns > HB_MAX_SEGMENTS) return false;
        for (int q = 0; q < ns; ++q) if (!(r.segments[c][a][q][1] > r.segments[c][a][q][0])) return false;
      }
  }
  return true;
}

}  // namespace

extern "C" {

int hb_default_config(hb_config* cfg) {
  if (!cfg) return HB_EINVAL;
  cfg->horizon_N = 100;
  cfg->dt = 0.01;
  cfg->max_batch = 1024;
  cfg->wbc_rho = 1e-8;      // Tikhonov weight of the WBC QP: its optimum is the least-norm one to O(rho) (DESIGN.md section 2, item 4)
  cfg->qp_max_iter = 40;
  cfg->line_search_max_trials = 14;
  cfg->time_horizon = 0.0;
  cfg->event_nodes = 0;
  cfg->e2e_chunks = 0;
  return HB_OK;
}

const char* hb_strerror(int code) {
  switch (code) {
    case HB_OK: return "ok";
    case HB_EINVAL: return "invalid argument";
    case HB_ECUDA: return "CUDA error";
    case HB_ENOMEM: return "out of memory";
    case HB_ECAP: return "batch exceeds context capacity";
    case HB_EPLAN: return "reference planner: swing phase without take-off / touch-down time, or reference capacity exceeded";
    case HB_ECOMM: return "NCCL not available or a collective failed (hb_shard_last_error)";
    default: return "unknown error";
  }
}

int hb_create(const hb_config* cfg, int device, hb_ctx** out) {
  // horizon cap: the warm shift stages one instance's previous trajectories in shared memory ((2N+1) x 22 doubles <= 227 KB)
  if (!cfg || !out || cfg->horizon_N < 1 || cfg->horizon_N > HB_MAX_HORIZON || cfg->max_batch < 1 || !(cfg->dt > 0.0) || cfg->time_horizon < 0.0) return HB_EINVAL;
  hb_ctx* ctx = new (std::nothrow) hb_ctx();
  if (!ctx) return HB_ENOMEM;
  memset(ctx, 0, sizeof(*ctx));
  ctx->cfg = *cfg;
  ctx->device = device;
  hb_default_wbc_settings(&ctx->wbc);
  // every failure below goes through hb_destroy (streams and partial allocations are released there)
  if (cudaSetDevice(device) != cudaSuccess) { hb_destroy(ctx); return HB_ECUDA; }
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { ctx->stream = nullptr; hb_destroy(ctx); return HB_ECUDA; }
  ctx->stream_main = ctx->stream;
  if (cudaStreamCreateWithFlags(&ctx->stream_aux, cudaStreamNonBlocking) != cudaSuccess) { ctx->stream_aux = nullptr; hb_destroy(ctx); return HB_ECUDA; }
  // model constants
  Model* m = new Model();
  memset(m, 0, sizeof(Model));
  for (int b = 0; b < NBODY; ++b) {
    for (int i = 0; i < 3; ++i) { m->joint_xyz[3 * b + i] = HB_JOINT_XYZ[3 * b + i]; m->com[3 * b + i] = HB_BODY_COM[3 * b + i]; }
    for (int i = 0; i < 9; ++i) m->inertia[9 * b + i] = HB_BODY_INERTIA[9 * b + i];
    m->mass[b] = HB_BODY_MASS[b];
    int code = 0;
    for (int i = 0; i < 3; ++i) if (HB_JOINT_AXIS[3 * b + i] != 0.0) code = (HB_JOINT_AXIS[3 * b + i] > 0 ? 1 : -1) * (i + 1);
    m->joint_axis[b] = code;
  }
  m->total_mass = HB_TOTAL_MASS;
  for (int i = 0; i < 12; ++i) m->contact_offset[i] = HB_CONTACT_OFFSET[i];
  for (int j = 0; j < NJ; ++j) { m->joint_lower[j] = HB_JOINT_LOWER[j]; m->joint_upper[j] = HB_JOINT_UPPER[j]; m->joint_vel_limit[j] = HB_JOINT_VEL_LIMIT[j]; m->torque_limit[j] = HB_WBC_TORQUE_LIMITS[j % 5]; }
  for (int i = 0; i < NX; ++i) m->Q[i] = HB_Q_DIAG[i];
  cudaError_t e = cudaMemcpyToSymbol(c_model, m, sizeof(Model));
  if (e == cudaSuccess) {
    double* dR = nullptr;
    e = dalloc(&dR, NU * NU);
    if (e == cudaSuccess) {
      init_input_cost_kernel<<<1, 32, 0, ctx->stream>>>(dR);
      e = cudaStreamSynchronize(ctx->stream);
      if (e == cudaSuccess) e = cudaMemcpy(m->R, dR, sizeof(double) * NU * NU, cudaMemcpyDeviceToHost);
      if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_model, m, sizeof(Model));
      cudaFree(dR);
    }
  }
  if (e == cudaSuccess) {
    double tab[32 * LQ_LANE_TAB] = {};
    for (int l = 0; l < 32; ++l) {
      double* t = tab + l * LQ_LANE_TAB;
      if (l < NX) t[0] = m->Q[l];
      if (l < 12) t[1] = m->R[l * NU + l];
      if (l >= 12 && l < NU) for (int j = 0; j < NJ; ++j) t[2 + j] = m->R[l * NU + 12 + j];
      if (l < 10) { t[12] = m->joint_lower[l]; t[13] = m->joint_upper[l]; }
      else if (l < 20) { t[12] = -m->joint_vel_limit[l - 10]; t[13] = m->joint_vel_limit[l - 10]; }
    }
    e = cudaMemcpyToSymbol(g_lq_lane, tab, sizeof(tab));
  }
  delete m;
  if (e != cudaSuccess) { ctx->last_cuda = (int)e; hb_destroy(ctx); return HB_ECUDA; }
  const size_t B = cfg->max_batch, N = cfg->horizon_N;
  bool ok = true;
  // the node records of the SQP pipeline (31 KB per instance and interval) are allocated by the first MPC solve: contexts that only run the
  // WBC / QP / planner / estimator entry points never pay for them
  ok = ok && dalloc(&ctx->dxt, B * (N + 1) * NX) == cudaSuccess && dalloc(&ctx->dut, B * N * NU) == cudaSuccess;
  ok = ok && dalloc(&ctx->perf, B * 4) == cudaSuccess && dalloc(&ctx->flags, B) == cudaSuccess;
  ok = ok && dalloc(&ctx->xdes, B * NX) == cudaSuccess && dalloc(&ctx->udes, B * NU) == cudaSuccess;
  ok = ok && dalloc(&ctx->wstatus, B) == cudaSuccess && dalloc(&ctx->witers, B) == cudaSuccess && dalloc(&ctx->wmode, B) == cudaSuccess;
  ok = ok && dalloc(&ctx->cyc_xref, B * (N + 1) * NX) == cudaSuccess && dalloc(&ctx->cyc_swing, B * (N + 1) * 24) == cudaSuccess;
  ok = ok && dalloc(&ctx->cyc_mode, B * (N + 1)) == cudaSuccess && dalloc(&ctx->cyc_tk, B * (N + 1)) == cudaSuccess && dalloc(&ctx->cyc_nn, B) == cudaSuccess;
  ok = ok && dalloc(&ctx->res_xt, B * (N + 1) * NX) == cudaSuccess && dalloc(&ctx->res_ut, B * N * NU) == cudaSuccess && dalloc(&ctx->res_t0, B) == cudaSuccess;
  ok = ok && dalloc(&ctx->res_mode, B * (N + 1)) == cudaSuccess && dalloc(&ctx->res_tk, B * (N + 1)) == cudaSuccess && dalloc(&ctx->res_nn, B) == cudaSuccess;
  ok = ok && dalloc(&ctx->res_sol, B * NWBC) == cudaSuccess && dalloc(&ctx->res_stance, B * 12) == cudaSuccess;
  // host-pointer calls stage through ctx->arena, which the first such call sizes: contexts driven through device pointers never pay for it
  if (!ok) { hb_destroy(ctx); return HB_ENOMEM; }
  {
    cudaError_t fe = cudaSuccess;
    auto attr = [&](const void* fn, size_t bytes) { if (fe == cudaSuccess) fe = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes); };
    attr((const void*)probe_flow_map_kernel, sizeof(ProbeShared));
    attr((const void*)qp_batch_kernel, 200 * 1024);
    attr((const void*)wbc_fused_kernel, wbc_fused_doubles() * sizeof(double));
    attr((const void*)hoqp_kernel, hoqp_smem_bytes());
    attr((const void*)lin_kernel, 4 * sizeof(LinHalf) + sizeof(ChainModel));
    attr((const void*)lq_kernel, sizeof(LqShared));
    attr((const void*)riccati_kernel, sizeof(RicShared));
    attr((const void*)forward_linesearch2_kernel, sizeof(Fw2Shared));
    attr((const void*)warm_shift_kernel, sizeof(double) * ((N + 1) * NX + N * NU));
    // the one-block-per-instance kernels fit 8 blocks per SM only with the full shared-memory carveout; do not leave it to the driver
    for (const void* fn : {(const void*)wbc_fused_kernel, (const void*)riccati_kernel})
      if (fe == cudaSuccess) fe = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    if (fe != cudaSuccess) { ctx->last_cuda = (int)fe; hb_destroy(ctx); return HB_ECUDA; }
  }
  *out = ctx;
  return HB_OK;
}

int hb_destroy(hb_ctx* ctx) {
  if (!ctx) return HB_EINVAL;
  cudaSetDevice(ctx->device);
  void* ptrs[] = {ctx->lin, ctx->proj, ctx->rk, ctx->dxt, ctx->dut, ctx->perf, ctx->flags, ctx->xdes, ctx->udes, ctx->wstatus, ctx->witers, ctx->wmode,
                  ctx->hoqp_scratch, ctx->hoqp_prob, ctx->cyc_xref, ctx->cyc_swing, ctx->cyc_tk, ctx->cyc_mode, ctx->cyc_nn, ctx->res_t0, ctx->res_xt,
                  ctx->res_ut, ctx->res_tk, ctx->res_mode, ctx->res_nn, ctx->res_sol, ctx->res_stance, ctx->arena, ctx->ro_mem};
  for (void* p : ptrs) if (p) cudaFree(p);
  if (ctx->pinned) cudaFreeHost(ctx->pinned);
  if (ctx->prof_ev) { for (int i = 0; i < 2 * PROF_MAX; ++i) cudaEventDestroy(ctx->prof_ev[i]); delete[] ctx->prof_ev; delete[] ctx->prof_kind; }
  if (ctx->stream_aux) cudaStreamDestroy(ctx->stream_aux);
  if (ctx->stream_main) cudaStreamDestroy(ctx->stream_main);
  else if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return HB_OK;
}

int hb_sync(hb_ctx* ctx) {
  if (!ctx) return HB_EINVAL;
  CK(cudaStreamSynchronize(ctx->stream));
  return HB_OK;
}
int hb_profile_enable(hb_ctx* ctx, int on) {
  if (!ctx) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  if (on && !ctx->prof_ev) {
    ctx->prof_ev = new (std::nothrow) cudaEvent_t[2 * PROF_MAX];
    ctx->prof_kind = new (std::nothrow) int[PROF_MAX];
    if (!ctx->prof_ev || !ctx->prof_kind) return HB_ENOMEM;
    for (int i = 0; i < 2 * PROF_MAX; ++i) CK(cudaEventCreate(&ctx->prof_ev[i]));
  }
  ctx->prof_on = on ? 1 : 0;
  ctx->prof_n = 0;
  return HB_OK;
}

int hb_profile_read(hb_ctx* ctx, double* ms_per_kind, int64_t* count_per_kind) {
  if (!ctx || !ms_per_kind || !count_per_kind) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  CK(cudaStreamSynchronize(ctx->stream));
  for (int k = 0; k < K_NKINDS; ++k) { ms_per_kind[k] = 0.0; count_per_kind[k] = 0; }
  for (int i = 0; i < ctx->prof_n; ++i) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ctx->prof_ev[2 * i], ctx->prof_ev[2 * i + 1]));
    ms_per_kind[ctx->prof_kind[i]] += ms;
    count_per_kind[ctx->prof_kind[i]]++;
  }
  ctx->prof_n = 0;
  return HB_OK;
}

const char* hb_last_cuda_error(const hb_ctx* ctx) { return ctx ? cudaGetErrorString((cudaError_t)ctx->last_cuda) : "no context"; }

int64_t hb_launch_count(const hb_ctx* ctx) { return ctx ? ctx->launches : 0; }
int64_t hb_last_reference_upload_bytes(const hb_ctx* ctx) { return ctx ? (int64_t)ctx->last_h2d_bytes : 0; }
void* hb_stream(hb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

// ------------------------------------------------------------------------------------------ device-pointer entry points
static int launch_qp(hb_ctx* ctx, int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA,
                     size_t sH, size_t sA, size_t sB, const int32_t* m_per, double* x, int32_t* status, int32_t* iters) {
  if (n < 1 || n > QP_MAX_N || m < 0 || m > QP_MAX_M) return HB_EINVAL;
  const size_t per_warp = qp_workspace_doubles(n) * sizeof(double);
  int wpb = (int)((200 * 1024) / per_warp);
  if (wpb < 1) return HB_EINVAL;
  if (wpb > 1) wpb = 1;   // one warp per CTA: the shared-memory footprint, not the thread count, bounds residency
  const int blocks = (B + wpb - 1) / wpb;
  return launch(ctx, K_QP, qp_batch_kernel, blocks, 32 * wpb, per_warp * wpb, B, n, m, H, g, A, lbA, ubA, sH, sA, sB, m_per, ctx->cfg.wbc_rho,
                ctx->cfg.qp_max_iter, x, status, iters);
}

int hb_wbc_qp_batch_dev(hb_ctx* ctx, int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA,
                        const double* ubA, double* x, int32_t* status, int32_t* iters) {
  if (!ctx || B < 0 || !H || !g || !A || !lbA || !ubA || !x) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch_qp(ctx, B, n, m, H, g, A, lbA, ubA, (size_t)n * n, (size_t)m * n, (size_t)m, nullptr, x, status, iters);
}

int hb_wbc_solve_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                           const uint8_t* stance_mode, double* sol, int32_t* status) {
  if (!ctx || B < 0 || !x_des || !u_des || !rbd || !mode || !sol) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_QP, wbc_fused_kernel, B, 32, wbc_fused_doubles() * sizeof(double), B, ctx->wbc, x_des, u_des, rbd, mode, stance_mode,
                ctx->cfg.wbc_rho, ctx->cfg.qp_max_iter, sol, status ? status : ctx->wstatus + ctx->base, ctx->witers + ctx->base);
}

int hb_wbc_assemble_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                              const uint8_t* stance_mode, double* H, double* g, double* A, double* lbA, double* ubA, int32_t* m_rows) {
  if (!ctx || B < 0 || !x_des || !u_des || !rbd || !mode || !H || !g || !A || !lbA || !ubA || !m_rows) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  const int wpb = 4;
  return launch(ctx, K_WBC_ASSEMBLE, wbc_assemble_kernel, (B + wpb - 1) / wpb, 32 * wpb, sizeof(WbcShared) * wpb, B, ctx->wbc, x_des, u_des, rbd, mode,
                stance_mode, H, g, A, lbA, ubA, m_rows);
}

int hb_wbc_qp_rows_batch_dev(hb_ctx* ctx, int B, int n, int m_alloc, const int32_t* m_rows, const double* H, const double* g, const double* A,
                             const double* lbA, const double* ubA, double* x, int32_t* status, int32_t* iters) {
  if (!ctx || B < 0 || !m_rows || !H || !g || !A || !lbA || !ubA || !x) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch_qp(ctx, B, n, m_alloc, H, g, A, lbA, ubA, (size_t)n * n, (size_t)m_alloc * n, (size_t)m_alloc, m_rows, x, status, iters);
}

static int hoqp_reserve(hb_ctx* ctx) {
  if (ctx->hoqp_scratch) return HB_OK;
  const size_t Bc = ctx->cfg.max_batch;
  if (dalloc(&ctx->hoqp_scratch, Bc * HQ_SCRATCH) != cudaSuccess || dalloc(&ctx->hoqp_prob, Bc) != cudaSuccess) {
    cudaGetLastError();
    if (ctx->hoqp_scratch) cudaFree(ctx->hoqp_scratch);
    ctx->hoqp_scratch = nullptr; ctx->hoqp_prob = nullptr;
    return HB_ENOMEM;
  }
  return HB_OK;
}

int hb_hoqp_solve_batch_dev(hb_ctx* ctx, int B, const hb_hoqp_problem* problems, double* x, double* slack, int32_t* status) {
  if (!ctx || B < 0 || !problems || !x) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  const int rc = hoqp_reserve(ctx);
  if (rc) return rc;
  return launch(ctx, K_QP, hoqp_kernel, B, 32, hoqp_smem_bytes(), B, problems, ctx->hoqp_scratch, 2 * ctx->cfg.qp_max_iter, x, slack, status);
}

static int hwbc_tasks_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, hb_hoqp_problem* problems) {
  return launch(ctx, K_WBC_ASSEMBLE, hwbc_tasks_kernel, B, 32, 0, B, ctx->wbc, x_des, u_des, rbd, mode, problems);
}

int hb_hierarchical_wbc_solve_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, double* sol,
                                        int32_t* status) {
  if (!ctx || B < 0 || !x_des || !u_des || !rbd || !mode || !sol) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  int rc = hoqp_reserve(ctx);
  if (rc) return rc;
  rc = hwbc_tasks_dev(ctx, B, x_des, u_des, rbd, mode, ctx->hoqp_prob);
  if (rc) return rc;
  return hb_hoqp_solve_batch_dev(ctx, B, ctx->hoqp_prob, sol, nullptr, status);
}

int hb_mpc_cold_start_batch_dev(hb_ctx* ctx, int B, const double* x0, const int32_t* mode, double* x_traj, double* u_traj) {
  if (!ctx || B < 0 || !x0 || !mode || !x_traj || !u_traj) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, cold_start_kernel, B, 128, 0, B, ctx->cfg.horizon_N, x0, mode, x_traj, u_traj);
}

static int mpc_solve_impl(hb_ctx* ctx, int B, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                          double* x_traj, double* u_traj, hb_solve_info* info, const double* tk, const int32_t* nn) {
  if (!ctx || B < 0 || !x0 || !x_ref || !swing_ref || !mode || !x_traj || !u_traj || ((tk == nullptr) != (nn == nullptr))) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  if (!ctx->lin) {
    const size_t Bc = ctx->cfg.max_batch, Nc = ctx->cfg.horizon_N;
    if (dalloc(&ctx->lin, Bc * Nc * LIN_STRIDE) != cudaSuccess || dalloc(&ctx->proj, Bc * Nc * PJ_STRIDE) != cudaSuccess || dalloc(&ctx->rk, Bc * Nc * RK_STRIDE) != cudaSuccess) {
      cudaGetLastError();
      if (ctx->lin) cudaFree(ctx->lin);
      if (ctx->proj) cudaFree(ctx->proj);
      ctx->lin = ctx->proj = ctx->rk = nullptr;
      return HB_ENOMEM;
    }
  }
  SqpArgs a;
  a.tk = tk; a.nn = nn;
  a.B = B; a.N = ctx->cfg.horizon_N; a.dt = ctx->cfg.dt; a.x_ref = x_ref; a.swing = swing_ref; a.mode = mode; a.xt = x_traj; a.ut = u_traj;
  {
    const size_t o = (size_t)ctx->base, Nn = (size_t)ctx->cfg.horizon_N;
    a.lin = ctx->lin + o * Nn * LIN_STRIDE; a.proj = ctx->proj + o * Nn * PJ_STRIDE; a.rk = ctx->rk + o * Nn * RK_STRIDE;
    a.dxt = ctx->dxt + o * (Nn + 1) * NX; a.dut = ctx->dut + o * Nn * NU; a.perf = ctx->perf + o * 4; a.flags = ctx->flags + o; a.x0 = x0;
  }
  const int N = a.N, NP = (N + 1) / 2;
  const long long nw = (long long)B * NP;
  int rc = launch(ctx, K_LIN, lin_kernel, (unsigned)((nw + 1) / 2), 64, 4 * sizeof(LinHalf) + sizeof(ChainModel), a);
  if (!rc) rc = launch(ctx, K_LQ, lq_kernel, (unsigned)((long long)B * N), 32, sizeof(LqShared), a);
  if (!rc) rc = launch(ctx, K_BACKWARD, riccati_kernel, B, 64, sizeof(RicShared), a);
  if (!rc) rc = launch(ctx, K_FORWARD_LS, forward_linesearch2_kernel, B, 32, sizeof(Fw2Shared), a, ctx->cfg.line_search_max_trials, info);
  return rc;
}

int hb_mpc_solve_batch_dev(hb_ctx* ctx, int B, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                           double* x_traj, double* u_traj, hb_solve_info* info) {
  return mpc_solve_impl(ctx, B, x0, x_ref, swing_ref, mode, x_traj, u_traj, info, nullptr, nullptr);
}

int hb_mpc_solve_grid_batch_dev(hb_ctx* ctx, int B, const double* x0, const double* node_times, const int32_t* n_intervals, const double* x_ref,
                                const double* swing_ref, const int32_t* mode, double* x_traj, double* u_traj, hb_solve_info* info) {
  if (!node_times || !n_intervals) return HB_EINVAL;
  return mpc_solve_impl(ctx, B, x0, x_ref, swing_ref, mode, x_traj, u_traj, info, node_times, n_intervals);
}

static int policy_eval_impl(hb_ctx* ctx, int B, double t_rel, const double* x_traj, const double* u_traj, const int32_t* mode, double* x_des,
                            double* u_des, int32_t* mode_out, const double* tk, const int32_t* nn) {
  if (!ctx || B < 0 || !x_traj || !u_traj || !mode || !x_des || !u_des || ((tk == nullptr) != (nn == nullptr))) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  const int wpb = 4;
  return launch(ctx, K_UNPROFILED, policy_eval_kernel, (B + wpb - 1) / wpb, 32 * wpb, 0, B, ctx->cfg.horizon_N, ctx->cfg.dt, t_rel, x_traj, u_traj, mode,
                x_des, u_des, mode_out, tk, nn, nullptr, nullptr);
}

int hb_policy_eval_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* x_traj, const double* u_traj, const int32_t* mode, double* x_des,
                             double* u_des, int32_t* mode_out) {
  return policy_eval_impl(ctx, B, t_rel, x_traj, u_traj, mode, x_des, u_des, mode_out, nullptr, nullptr);
}

int hb_policy_eval_grid_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* node_times, const int32_t* n_intervals, const double* x_traj,
                                  const double* u_traj, const int32_t* mode, double* x_des, double* u_des, int32_t* mode_out) {
  if (!node_times || !n_intervals) return HB_EINVAL;
  return policy_eval_impl(ctx, B, t_rel, x_traj, u_traj, mode, x_des, u_des, mode_out, node_times, n_intervals);
}

int hb_time_grid_batch_dev(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* node_times, int32_t* n_intervals, int32_t* status) {
  if (!ctx || B < 0 || !t0 || !refs || !node_times || !n_intervals) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  const double T = ctx->cfg.time_horizon > 0.0 ? ctx->cfg.time_horizon : ctx->cfg.horizon_N * ctx->cfg.dt;
  return launch(ctx, K_UNPROFILED, time_grid_kernel, (B + 127) / 128, 128, 0, B, ctx->cfg.horizon_N, ctx->cfg.dt, T, t0, refs, node_times, n_intervals, status);
}

static int control_step_impl(hb_ctx* ctx, int B, double t_rel, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                             const double* rbd, double* x_traj, double* u_traj, hb_solve_info* info, double* wbc_sol, double* torque,
                             int32_t* wbc_status, const double* tk, const int32_t* nn) {
  if (!ctx || !rbd || !wbc_sol) return HB_EINVAL;
  int rc = mpc_solve_impl(ctx, B, x0, x_ref, swing_ref, mode, x_traj, u_traj, info, tk, nn);
  if (rc) return rc;
  if (B == 0) return HB_OK;
  double* xdes = ctx->xdes + (size_t)ctx->base * NX; double* udes = ctx->udes + (size_t)ctx->base * NU; int32_t* wmode = ctx->wmode + ctx->base;
  rc = policy_eval_impl(ctx, B, t_rel, x_traj, u_traj, mode, xdes, udes, wmode, tk, nn);
  if (rc) return rc;
  rc = hb_wbc_solve_batch_dev(ctx, B, xdes, udes, rbd, wmode, nullptr, wbc_sol, wbc_status);
  if (!rc && torque) rc = launch(ctx, K_UNPROFILED, torque_kernel, (B * NJ + 127) / 128, 128, 0, B, wbc_sol, torque);
  return rc;
}

int hb_control_step_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                              const double* rbd, double* x_traj, double* u_traj, hb_solve_info* info, double* wbc_sol, double* torque,
                              int32_t* wbc_status) {
  return control_step_impl(ctx, B, t_rel, x0, x_ref, swing_ref, mode, rbd, x_traj, u_traj, info, wbc_sol, torque, wbc_status, nullptr, nullptr);
}

// WeightedWbc::update fallback (WeightedWbc.cpp:57-64): a QP that did not solve returns the previous solution of that instance; a solved
// one becomes the new "previous". `have_prev` is 0 on the first cycle after a cold start (the reference then returns the unsolved iterate).
__global__ void wbc_fallback_kernel(int B, int have_prev, const int32_t* status, double* sol, double* prev, double* torque) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * NWBC) return;
  const int i = idx / NWBC, j = idx - i * NWBC;
  if (status[i] != 0 && have_prev) {
    const double v = prev[idx];
    sol[idx] = v;
    if (torque && j >= 28) torque[(size_t)i * NJ + j - 28] = v;
  } else {
    prev[idx] = sol[idx];
  }
}

// store the solve time of a cold-started resident solution
__global__ void set_times_kernel(int B, int N, const double* t0_new, double* t0_res, const double* tk_new, const int32_t* nn_new, double* tk_res,
                                 int32_t* nn_res) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  t0_res[i] = t0_new[i];
  if (tk_new) {
    nn_res[i] = nn_new[i];
    for (int k = 0; k <= N; ++k) tk_res[(size_t)i * (N + 1) + k] = tk_new[(size_t)i * (N + 1) + k];
  }
}

// hb_resident_cycle_batch_dev; with run_wbc = false the cycle ends after the SQP iteration (hb_rollout_batch_dev: the 500 Hz tick at the
// same time is the WBC of that cycle, so the cycle's own would be thrown away)
static int resident_cycle_impl(hb_ctx* ctx, int B, int cold_start, double t_rel, const double* t0, const double* x0, const hb_reference* refs,
                               const double* rbd, hb_solve_info* info, double* wbc_sol, double* torque, int32_t* wbc_status, bool run_wbc) {
  if (!ctx || B < 0 || !t0 || !x0 || !refs || !rbd) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (ctx->base + B > ctx->cfg.max_batch) return HB_ECAP;
  if (!cold_start && ctx->res_valid < ctx->base + B) return HB_EINVAL;     // no previous solution to shift
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N, o = (size_t)ctx->base;
  double* xref = ctx->cyc_xref + o * (N + 1) * NX; double* swing = ctx->cyc_swing + o * (N + 1) * 24; int32_t* mode = ctx->cyc_mode + o * (N + 1);
  double* xt = ctx->res_xt + o * (N + 1) * NX; double* ut = ctx->res_ut + o * N * NU; double* tres = ctx->res_t0 + o;
  // event-node grids (cfg.event_nodes): per-instance node times, kept resident beside the primal solution
  const bool grid = ctx->cfg.event_nodes != 0;
  double* tk = grid ? ctx->cyc_tk + o * (N + 1) : nullptr; int32_t* nn = grid ? ctx->cyc_nn + o : nullptr;
  double* tkres = grid ? ctx->res_tk + o * (N + 1) : nullptr; int32_t* nnres = grid ? ctx->res_nn + o : nullptr;
  int rc = HB_OK;
  if (grid) {
    rc = hb_time_grid_batch_dev(ctx, B, t0, refs, tk, nn, nullptr);
    if (rc) return rc;
    rc = hb_reference_expand_grid_batch_dev(ctx, B, tk, refs, xref, swing, mode);
  } else {
    rc = hb_reference_expand_batch_dev(ctx, B, t0, refs, xref, swing, mode);
  }
  if (rc) return rc;
  if (cold_start) {
    rc = hb_mpc_cold_start_batch_dev(ctx, B, x0, mode, xt, ut);
    if (!rc) rc = launch(ctx, K_UNPROFILED, set_times_kernel, (B + 127) / 128, 128, 0, B, (int)N, t0, tres, tk, nn, tkres, nnres);
  } else {
    const size_t smem = sizeof(double) * ((N + 1) * NX + N * NU);     // opted in at hb_create
    rc = launch(ctx, K_UNPROFILED, warm_shift_kernel, B, 128, smem, B, (int)N, ctx->cfg.dt, t0, tres, x0, mode, xt, ut, tk, nn, tkres, nnres);
  }
  if (rc) return rc;
  CK(cudaMemcpyAsync(ctx->res_mode + o * (N + 1), mode, sizeof(int32_t) * B * (N + 1), cudaMemcpyDeviceToDevice, ctx->stream));
  if (ctx->res_valid < ctx->base + B) ctx->res_valid = ctx->base + B;
  if (!run_wbc) return mpc_solve_impl(ctx, B, x0, xref, swing, mode, xt, ut, info, tk, nn);
  rc = control_step_impl(ctx, B, t_rel, x0, xref, swing, mode, rbd, xt, ut, info, wbc_sol, torque, wbc_status, tk, nn);
  if (rc) return rc;
  if (wbc_status) {
    const int have_prev = (!cold_start && ctx->res_sol_valid >= ctx->base + B) ? 1 : 0;
    rc = launch(ctx, K_UNPROFILED, wbc_fallback_kernel, (B * NWBC + 127) / 128, 128, 0, B, have_prev, wbc_status, wbc_sol, ctx->res_sol + o * NWBC, torque);
    if (rc) return rc;
    if (ctx->res_sol_valid < ctx->base + B) ctx->res_sol_valid = ctx->base + B;
  }
  return HB_OK;
}

int hb_resident_cycle_batch_dev(hb_ctx* ctx, int B, int cold_start, double t_rel, const double* t0, const double* x0, const hb_reference* refs,
                                const double* rbd, hb_solve_info* info, double* wbc_sol, double* torque, int32_t* wbc_status) {
  if (!wbc_sol) return HB_EINVAL;
  return resident_cycle_impl(ctx, B, cold_start, t_rel, t0, x0, refs, rbd, info, wbc_sol, torque, wbc_status, true);
}

int hb_plan_references_batch_dev(hb_ctx* ctx, int B, const hb_plan_input* in, const double* feet, double* latest_stance, hb_reference* out,
                                 int32_t* status) {
  if (!ctx || B < 0 || !in || !latest_stance || !out) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  static const hbplan::PlanConsts pc = hbplan::make_consts();
  return launch(ctx, K_UNPROFILED, plan_references_coop_kernel, (B + 7) / 8, 32, 0, B, in, feet, latest_stance, out, status, pc);
}

int hb_default_kf_params(hb_kf_params* p) {
  if (!p) return HB_EINVAL;
  p->foot_radius = 0.02; p->imu_process_noise_position = 0.02; p->imu_process_noise_velocity = 0.02; p->foot_process_noise_position = 0.5;
  p->foot_sensor_noise_position = 0.5; p->foot_sensor_noise_velocity = 0.1; p->foot_height_sensor_noise = 0.01;
  return HB_OK;
}

int hb_kf_reset(int B, hb_kf_state* state) {
  if (B < 0 || !state) return HB_EINVAL;
  for (int i = 0; i < B; ++i) {
    memset(&state[i], 0, sizeof(hb_kf_state));
    for (int k = 0; k < 18; ++k) state[i].P[k * 18 + k] = 100.0;
  }
  return HB_OK;
}

int hb_estimator_update_batch_dev(hb_ctx* ctx, int B, const hb_kf_params* params, double dt, hb_kf_state* state, const double* quat,
                                  const double* ang_vel_local, const double* lin_acc_local, const double* joint_pos, const double* joint_vel,
                                  const uint8_t* contact_flag, double* rbd_out) {
  if (!ctx || B < 0 || !params || !state || !quat || !ang_vel_local || !lin_acc_local || !joint_pos || !joint_vel || !contact_flag || !rbd_out) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, kf_update_kernel, B, 32, sizeof(KfShared), B, *params, dt, state, quat, ang_vel_local, lin_acc_local, joint_pos,
                joint_vel, contact_flag, rbd_out);
}

int hb_default_wbc_settings(hb_wbc_settings* s) {
  if (!s) return HB_EINVAL;
  for (int j = 0; j < 5; ++j) s->torque_limits[j] = HB_WBC_TORQUE_LIMITS[j];
  s->friction_coefficient = HB_WBC_FRICTION_MU;
  s->swing_kp = HB_WBC_SWING_KP; s->swing_kd = HB_WBC_SWING_KD;
  s->base_accel_kp = 40.0; s->base_accel_kd = 4.0;            // task.info:310-314; loaded (WbcBase.cpp:386-393) but used by no task
  s->base_height_kp = HB_WBC_BASE_HEIGHT_KP; s->base_height_kd = HB_WBC_BASE_HEIGHT_KD;
  s->base_angular_kp = HB_WBC_BASE_ANGULAR_KP; s->base_angular_kd = HB_WBC_BASE_ANGULAR_KD;
  s->weight_swing_leg = HB_WBC_WEIGHT_SWING; s->weight_base_accel = HB_WBC_WEIGHT_BASE; s->weight_contact_force = HB_WBC_WEIGHT_FORCE;
  return HB_OK;
}

int hb_wbc_get_settings(const hb_ctx* ctx, hb_wbc_settings* s) {
  if (!ctx || !s) return HB_EINVAL;
  *s = ctx->wbc;
  return HB_OK;
}

int hb_wbc_set_settings(hb_ctx* ctx, const hb_wbc_settings* s) {
  if (!ctx || !s) return HB_EINVAL;
  for (int j = 0; j < 5; ++j) if (!(s->torque_limits[j] > 0.0)) return HB_EINVAL;
  if (!(s->friction_coefficient > 0.0) || !(s->weight_swing_leg > 0.0) || !(s->weight_base_accel > 0.0) || s->weight_contact_force < 0.0) return HB_EINVAL;
  ctx->wbc = *s;      // passed by value with the next launch: nothing in flight is affected
  return HB_OK;
}

int hb_wbc_set_kp_kd(hb_ctx* ctx, double swing_kp, double swing_kd) {
  if (!ctx) return HB_EINVAL;
  ctx->wbc.swing_kp = swing_kp; ctx->wbc.swing_kd = swing_kd;
  return HB_OK;
}

namespace {
// Minimal reader of the boost property-tree INFO subset the reference's task.info uses: `key value`, `key { ... }`, `(i,j) value`,
// `;` comments. Values are collected under dotted paths ("swingLegTask.kp", "torqueLimitsTask.(0,0)").
struct InfoMap {
  std::vector<std::pair<std::string, std::string>> kv;
  const std::string* find(const std::string& k) const { for (const auto& e : kv) if (e.first == k) return &e.second; return nullptr; }
  bool number(const std::string& k, double* out) const {
    const std::string* v = find(k);
    if (!v) return false;
    char* end = nullptr;
    const double d = strtod(v->c_str(), &end);
    if (end == v->c_str()) { if (*v == "true") { *out = 1.0; return true; } if (*v == "false") { *out = 0.0; return true; } return false; }
    *out = d;
    return true;
  }
};
bool info_parse(const char* path, InfoMap& out) {
  FILE* f = fopen(path, "r");
  if (!f) return false;
  std::vector<std::string> tok;
  std::string cur;
  int ch;
  bool comment = false;
  auto flush = [&]() { if (!cur.empty()) { tok.push_back(cur); cur.clear(); } };
  while ((ch = fgetc(f)) != EOF) {
    if (comment) { if (ch == '\n') comment = false; continue; }
    if (ch == ';') { flush(); comment = true; continue; }
    if (ch == '{' || ch == '}') { flush(); tok.push_back(std::string(1, (char)ch)); continue; }
    if (ch == ' ' || ch == '\t' || ch == '\n' || ch == '\r') { flush(); continue; }
    cur.push_back((char)ch);
  }
  flush();
  fclose(f);
  std::vector<std::string> path_stack;
  size_t i = 0;
  while (i < tok.size()) {
    const std::string& t = tok[i];
    if (t == "}") { if (path_stack.empty()) return false; path_stack.pop_back(); ++i; continue; }
    if (t == "{") return false;
    if (i + 1 < tok.size() && tok[i + 1] == "{") { path_stack.push_back(t); i += 2; continue; }
    if (i + 1 >= tok.size() || tok[i + 1] == "}") { ++i; continue; }      // key without a value
    std::string key;
    for (const auto& p : path_stack) { key += p; key += '.'; }
    key += t;
    out.kv.emplace_back(key, tok[i + 1]);
    i += 2;
  }
  return path_stack.empty();
}
}  // namespace

int hb_parse_task_info(const char* path, hb_task_info* out) {
  if (!path || !out) return HB_EINVAL;
  InfoMap m;
  if (!info_parse(path, m)) return HB_EINVAL;
  memset(out, 0, sizeof(*out));
  hb_default_wbc_settings(&out->wbc);
  hb_kf_params kf; hb_default_kf_params(&kf);
  memcpy(out->kalman, &kf, sizeof(kf));
  out->contact_force_cutoff_frequency = 250.0; out->contact_threshold = 75.0;
  out->sqp_dt = 0.015; out->sqp_iteration = 1; out->mpc_time_horizon = 0.8; out->mpc_cold_start = 0;
  double v;
  int found = 0;
  hb_wbc_settings& w = out->wbc;
  for (int j = 0; j < 5; ++j) { char k[64]; snprintf(k, sizeof(k), "torqueLimitsTask.(%d,0)", j); if (m.number(k, &v)) { w.torque_limits[j] = v; found |= 1; } }
  if (m.number("frictionConeTask.frictionCoefficient", &v)) { w.friction_coefficient = v; found |= 1; }
  if (m.number("swingLegTask.kp", &v)) { w.swing_kp = v; found |= 1; }
  if (m.number("swingLegTask.kd", &v)) { w.swing_kd = v; found |= 1; }
  if (m.number("baseAccelTask.kp", &v)) { w.base_accel_kp = v; found |= 1; }
  if (m.number("baseAccelTask.kd", &v)) { w.base_accel_kd = v; found |= 1; }
  if (m.number("baseHeightTask.kp", &v)) { w.base_height_kp = v; found |= 1; }
  if (m.number("baseHeightTask.kd", &v)) { w.base_height_kd = v; found |= 1; }
  if (m.number("baseAngularTask.kp", &v)) { w.base_angular_kp = v; found |= 1; }
  if (m.number("baseAngularTask.kd", &v)) { w.base_angular_kd = v; found |= 1; }
  if (m.number("weight.swingLeg", &v)) { w.weight_swing_leg = v; found |= 1; }
  if (m.number("weight.baseAccel", &v)) { w.weight_base_accel = v; found |= 1; }
  if (m.number("weight.contactForce", &v)) { w.weight_contact_force = v; found |= 1; }
  const char* kfk[7] = {"footRadius", "imuProcessNoisePosition", "imuProcessNoiseVelocity", "footProcessNoisePosition", "footSensorNoisePosition",
                        "footSensorNoiseVelocity", "footHeightSensorNoise"};
  for (int j = 0; j < 7; ++j) if (m.number(std::string("kalmanFilter.") + kfk[j], &v)) { out->kalman[j] = v; found |= 2; }
  if (m.number("contactForceEsimation.cutoffFrequency", &v)) { out->contact_force_cutoff_frequency = v; found |= 4; }
  if (m.number("contactForceEsimation.contactThreshold", &v)) { out->contact_threshold = v; found |= 4; }
  if (m.number("sqp.dt", &v)) { out->sqp_dt = v; found |= 8; }
  if (m.number("sqp.sqpIteration", &v)) { out->sqp_iteration = (int32_t)v; found |= 8; }
  if (m.number("mpc.timeHorizon", &v)) { out->mpc_time_horizon = v; found |= 16; }
  if (m.number("mpc.coldStart", &v)) { out->mpc_cold_start = v != 0.0; found |= 16; }
  out->found = found;
  return HB_OK;
}

int hb_load_task_info(hb_ctx* ctx, const char* path) {
  if (!ctx || !path) return HB_EINVAL;
  hb_task_info ti;
  int rc = hb_parse_task_info(path, &ti);
  if (rc) return rc;
  return hb_wbc_set_settings(ctx, &ti.wbc);
}

int hb_default_sim_params(hb_sim_params* p) {
  if (!p) return HB_EINVAL;
  p->dt = 0.002; p->substeps = 4; p->ground_height = 0.0; p->ground_stiffness = 3.0e4; p->ground_damping = 3.0e2; p->tangential_damping = 3.0e2; p->friction_mu = 0.7;
  p->joint_armature = 0.1; p->joint_damping = 1.0;       // mujoco/model/hunter/hunter.xml:6 (default joint armature / damping of the reference's plant)
  return HB_OK;
}

int hb_actuation_reset(int B, hb_actuation_state* state) {
  if (B < 0 || !state) return HB_EINVAL;
  memset(state, 0, sizeof(hb_actuation_state) * (size_t)B);       // cmdBuffer_ cleared (LeggedHWSim.cpp:171-174)
  return HB_OK;
}

int hb_actuation_batch_dev(hb_ctx* ctx, int B, double delay, const double* time, hb_actuation_state* state, const double* command, const double* rbd,
                           double* tau) {
  if (!ctx || B < 0 || !time || !state || !command || !rbd || !tau || delay < 0.0) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, actuation_kernel, (B + 63) / 64, 64, 0, B, delay, time, state, command, rbd, tau);
}

int hb_sim_step_batch_dev(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, double* contact_force, uint8_t* contact_flag) {
  if (!ctx || B < 0 || !params || !rbd || !tau || !(params->dt > 0.0) || params->substeps < 1 || params->substeps > 1000) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, sim_step_kernel, B, 32, 0, B, *params, rbd, tau, contact_force, contact_flag);
}

// hb_resident_wbc_batch_dev; no_prev = true: the fallback has no previous solution yet (first tick after a cold start whose cycle ran no WBC)
static int resident_wbc_impl(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode, double* x_des, double* u_des,
                             int32_t* mode_out, double* wbc_sol, double* torque, int32_t* wbc_status, bool no_prev) {
  if (!ctx || B < 0 || !t_now || !rbd || !x_des || !u_des || !mode_out || !wbc_sol) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (ctx->base + B > ctx->res_valid) return HB_EINVAL;             // no resident solution to evaluate
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N, o = (size_t)ctx->base;
  const bool grid = ctx->cfg.event_nodes != 0;
  const int wpb = 4;
  int rc = launch(ctx, K_UNPROFILED, policy_eval_kernel, (B + wpb - 1) / wpb, 32 * wpb, 0, B, (int)N, ctx->cfg.dt, 0.0, ctx->res_xt + o * (N + 1) * NX,
                  ctx->res_ut + o * N * NU, ctx->res_mode + o * (N + 1), x_des, u_des, mode_out, grid ? ctx->res_tk + o * (N + 1) : nullptr,
                  grid ? ctx->res_nn + o : nullptr, t_now, ctx->res_t0 + o);
  if (!rc) rc = hb_wbc_solve_batch_dev(ctx, B, x_des, u_des, rbd, mode_out, stance_mode, wbc_sol, wbc_status);
  if (!rc && torque) rc = launch(ctx, K_UNPROFILED, torque_kernel, (B * NJ + 127) / 128, 128, 0, B, wbc_sol, torque);
  if (rc) return rc;
  if (wbc_status) {
    const int have_prev = (!no_prev && ctx->res_sol_valid >= ctx->base + B) ? 1 : 0;
    rc = launch(ctx, K_UNPROFILED, wbc_fallback_kernel, (B * NWBC + 127) / 128, 128, 0, B, have_prev, wbc_status, wbc_sol, ctx->res_sol + o * NWBC, torque);
    if (rc) return rc;
    if (ctx->res_sol_valid < ctx->base + B) ctx->res_sol_valid = ctx->base + B;
  }
  return HB_OK;
}

int hb_resident_wbc_batch_dev(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode, double* x_des, double* u_des,
                              int32_t* mode_out, double* wbc_sol, double* torque, int32_t* wbc_status) {
  return resident_wbc_impl(ctx, B, t_now, rbd, stance_mode, x_des, u_des, mode_out, wbc_sol, torque, wbc_status, false);
}

int hb_default_rollout_params(hb_rollout_params* p) {
  if (!p) return HB_EINVAL;
  memset(p, 0, sizeof(*p));
  p->period = 0.002; p->mpc_every = 5; p->actuation_delay = 0.009;
  hb_default_sim_params(&p->sim);
  hb_default_pd_gains(&p->gains);
  for (int j = 0; j < NJ; ++j) p->torque_limit[j] = HB_WBC_TORQUE_LIMITS[j % 5];
  return HB_OK;
}

// hb_rollout_batch_dev's scratch: one allocation at max_batch, carved into 256-byte aligned slices
static int rollout_reserve(hb_ctx* ctx) {
  if (ctx->ro_mem) return HB_OK;
  const size_t Bc = ctx->cfg.max_batch;
  size_t total = 0;
  auto slice = [&](size_t per) { const size_t o = total; total += (per * Bc + 255) & ~(size_t)255; return o; };
  const size_t o_cmd = slice(sizeof(hb_rollout_command)), o_in = slice(sizeof(hb_plan_input)), o_refs = slice(sizeof(hb_reference));
  const size_t o_info = slice(sizeof(hb_solve_info)), o_pstat = slice(sizeof(int32_t)), o_t0 = slice(sizeof(double)), o_x0 = slice(sizeof(double) * NX);
  const size_t o_feet = slice(sizeof(double) * 12), o_sol = slice(sizeof(double) * NWBC), o_jcmd = slice(sizeof(double) * NJ * 5);
  const size_t o_jtau = slice(sizeof(double) * NJ), o_tau = slice(sizeof(double) * NJ), o_held = slice(sizeof(double) * 32), o_tnow = slice(sizeof(double));
  if (cudaMalloc(&ctx->ro_mem, total) != cudaSuccess) { cudaGetLastError(); ctx->ro_mem = nullptr; return HB_ENOMEM; }
  char* b = static_cast<char*>(ctx->ro_mem);
  ctx->ro_cmd = reinterpret_cast<hb_rollout_command*>(b + o_cmd); ctx->ro_in = reinterpret_cast<hb_plan_input*>(b + o_in);
  ctx->ro_refs = reinterpret_cast<hb_reference*>(b + o_refs); ctx->ro_info = reinterpret_cast<hb_solve_info*>(b + o_info);
  ctx->ro_pstat = reinterpret_cast<int32_t*>(b + o_pstat);
  double** dp[] = {&ctx->ro_t0, &ctx->ro_x0, &ctx->ro_feet, &ctx->ro_sol, &ctx->ro_jcmd, &ctx->ro_jtau, &ctx->ro_tau, &ctx->ro_held, &ctx->ro_tnow};
  const size_t offs[] = {o_t0, o_x0, o_feet, o_sol, o_jcmd, o_jtau, o_tau, o_held, o_tnow};
  for (int k = 0; k < 9; ++k) *dp[k] = reinterpret_cast<double*>(b + offs[k]);
  return HB_OK;
}

int hb_rollout_batch_dev(hb_ctx* ctx, int B, int64_t tick0, int n_ticks, const hb_rollout_params* p, const hb_rollout_command* cmd, double* rbd,
                         hb_actuation_state* act, uint8_t* estop, hb_rollout_stats* stats, double* log) {
  if (!ctx || B < 0 || n_ticks < 0 || tick0 < 0 || !p || !cmd || !rbd || !act || !estop || !stats) return HB_EINVAL;
  if (p->mpc_every < 1 || !(p->period > 0.0) || p->log_every < 0 || !(p->actuation_delay >= 0.0) || !(p->sim.dt > 0.0) || p->sim.substeps < 1 ||
      p->sim.substeps > 1000 || tick0 + n_ticks > INT32_MAX)
    return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  for (int i = 0; i < B; ++i) {
    const hb_rollout_command& c = cmd[i];
    if (c.gait < 0 || c.gait > 3 || c.n_cmd < 1 || c.n_cmd > HB_ROLLOUT_MAX_CMDS || !(c.gait_start == c.gait_start)) return HB_EINVAL;
    for (int k = 0; k < c.n_cmd; ++k) if (!(c.cmd_time[k] == c.cmd_time[k]) || (k > 0 && c.cmd_time[k] < c.cmd_time[k - 1])) return HB_EINVAL;
  }
  const bool cold = tick0 == 0;
  if (!cold && ctx->res_valid < B) return HB_EINVAL;       // no resident solution to continue from
  if (n_ticks == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  int rc = rollout_reserve(ctx);
  if (rc) return rc;
  CK(cudaMemcpyAsync(ctx->ro_cmd, cmd, sizeof(hb_rollout_command) * B, cudaMemcpyHostToDevice, ctx->stream));
  const double horizon = (ctx->cfg.event_nodes && ctx->cfg.time_horizon > 0.0) ? ctx->cfg.time_horizon : ctx->cfg.horizon_N * ctx->cfg.dt;
  const int n_log = (log && p->log_every > 0) ? (n_ticks + p->log_every - 1) / p->log_every : 0;
  const unsigned grid = (B + 63) / 64;
  for (int k = 0; k < n_ticks && !rc; ++k) {
    const int64_t a = tick0 + k;
    const double t = (double)a * p->period;           // a product, never an accumulated sum: a stepwise caller reproduces it exactly
    const bool mpc = a % p->mpc_every == 0, first_cold = cold && k == 0;
    double* log_row = (n_log && k % p->log_every == 0) ? log + (size_t)(k / p->log_every) * 32 : nullptr;
    rc = launch(ctx, K_UNPROFILED, rollout_tick_begin_kernel, grid, 64, 0, B, (int)a, t, p->min_base_height, rbd, ctx->ro_held, stats, ctx->ro_tnow,
                log_row, (size_t)n_log * 32);
    if (!rc && mpc) {
      if (first_cold) CK(cudaMemsetAsync(ctx->res_stance, 0, sizeof(double) * B * 12, ctx->stream));   // latestStanceposition_ starts at zero
      rc = launch(ctx, K_UNPROFILED, rollout_plan_inputs_kernel, grid, 64, 0, B, t, horizon, ctx->ro_cmd, rbd, ctx->ro_in);
      if (!rc) rc = launch(ctx, K_UNPROFILED, plan_prepare_kernel, grid, 64, 0, B, ctx->ro_in, ctx->ro_t0, ctx->ro_x0, ctx->ro_feet);
      if (!rc) rc = hb_plan_references_batch_dev(ctx, B, ctx->ro_in, ctx->ro_feet, ctx->res_stance, ctx->ro_refs, ctx->ro_pstat);
      if (!rc) rc = resident_cycle_impl(ctx, B, first_cold, 0.0, ctx->ro_t0, ctx->ro_x0, ctx->ro_refs, rbd, ctx->ro_info, nullptr, nullptr, nullptr, false);
    }
    // the cycle ran no WBC, so after a cold start the first tick's fallback has no previous solution, as the cycle's own would not have
    if (!rc) rc = resident_wbc_impl(ctx, B, ctx->ro_tnow, rbd, nullptr, ctx->xdes, ctx->udes, ctx->wmode, ctx->ro_sol, nullptr, ctx->wstatus, first_cold);
    if (!rc) rc = hb_joint_command_batch_dev(ctx, B, &p->gains, p->period, ctx->xdes, ctx->udes, ctx->ro_sol, ctx->wmode, rbd, nullptr, estop, ctx->ro_jcmd,
                                             ctx->ro_jtau);
    if (!rc) rc = hb_actuation_batch_dev(ctx, B, p->actuation_delay, ctx->ro_tnow, act, ctx->ro_jcmd, rbd, ctx->ro_tau);
    if (!rc) rc = launch(ctx, K_UNPROFILED, rollout_saturate_kernel, (B * NJ + 127) / 128, 128, 0, B, *p, ctx->ro_tau);
    if (!rc) rc = hb_sim_step_batch_dev(ctx, B, &p->sim, rbd, ctx->ro_tau, nullptr, nullptr);
    if (!rc) rc = launch(ctx, K_UNPROFILED, rollout_tick_end_kernel, grid, 64, 0, B, (int)a, mpc ? 1 : 0, ctx->ro_info, ctx->ro_pstat, ctx->wstatus, estop, ctx->ro_tau, ctx->ro_held, rbd, stats);
  }
  return rc;
}

int hb_observer_reset(int B, hb_observer_state* state) {
  if (B < 0 || !state) return HB_EINVAL;
  memset(state, 0, sizeof(hb_observer_state) * (size_t)B);      // pSCgZinvlast_ starts at zero (StateEstimateBase.cpp:58-59)
  return HB_OK;
}

int hb_contact_force_estimate_batch_dev(hb_ctx* ctx, int B, double cutoff_frequency, double dt, hb_observer_state* state, const double* rbd,
                                        const double* tau_cmd, double* est_contact_force, double* disturbance_torque) {
  if (!ctx || B < 0 || !state || !rbd || !tau_cmd || !est_contact_force || !(cutoff_frequency > 0.0) || !(dt > 0.0)) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, contact_force_kernel, B, 32, 0, B, cutoff_frequency, dt, state, rbd, tau_cmd, est_contact_force, disturbance_torque);
}

int hb_default_pd_gains(hb_pd_gains* g) {
  if (!g) return HB_EINVAL;
  g->kp_position = 10.0; g->kd_position = 3.0;
  g->kp_big_stance = 40.0; g->kp_big_swing = 30.0; g->kd_big = 2.0;
  g->kp_small_stance = 30.0; g->kp_small_swing = 20.0; g->kd_small = 2.0;
  g->kd_feet = 0.01;
  return HB_OK;
}

int hb_joint_command_batch_dev(hb_ctx* ctx, int B, const hb_pd_gains* gains, double period, const double* x_des, const double* u_des,
                               const double* wbc_sol, const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded, uint8_t* estop,
                               double* command, double* output_torque) {
  if (!ctx || B < 0 || !gains || !x_des || !u_des || !wbc_sol || !mode_cmd || !rbd || !command || !output_torque) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, joint_command_kernel, (B + 63) / 64, 64, 0, B, *gains, period, x_des, u_des, wbc_sol, mode_cmd, rbd, loaded, estop,
                command, output_torque);
}

int hb_rbd_to_centroidal_batch_dev(hb_ctx* ctx, int B, const double* rbd, double* x) {
  if (!ctx || B < 0 || !rbd || !x) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, rbd_to_centroidal_kernel, (B + 63) / 64, 64, 0, B, rbd, x);
}

int hb_reference_expand_batch_dev(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* x_ref, double* swing_ref, int32_t* mode) {
  if (!ctx || B < 0 || !t0 || !refs || !x_ref || !swing_ref || !mode) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, reference_expand_kernel, B, 128, 0, B, ctx->cfg.horizon_N, ctx->cfg.dt, t0, refs, x_ref, swing_ref, mode, nullptr);
}

int hb_reference_expand_grid_batch_dev(hb_ctx* ctx, int B, const double* node_times, const hb_reference* refs, double* x_ref, double* swing_ref,
                                       int32_t* mode) {
  if (!ctx || B < 0 || !node_times || !refs || !x_ref || !swing_ref || !mode) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, reference_expand_kernel, B, 128, 0, B, ctx->cfg.horizon_N, ctx->cfg.dt, nullptr, refs, x_ref, swing_ref, mode, node_times);
}

int hb_contact_positions_batch_dev(hb_ctx* ctx, int B, const double* x, double* pos) {
  if (!ctx || B < 0 || !x || !pos) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, contact_positions_kernel, (B + 63) / 64, 64, 0, B, x, pos);
}

int hb_probe_flow_map_dev(hb_ctx* ctx, int B, const double* x, const double* u, double* f, double* A, double* Bm, double* ee) {
  if (!ctx || B < 0 || !x || !u || !f || !A || !Bm) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (set_device(ctx)) return HB_ECUDA;
  return launch(ctx, K_UNPROFILED, probe_flow_map_kernel, B, 32, sizeof(ProbeShared), B, x, u, f, A, Bm, ee);
}

// ------------------------------------------------------------------------------------------ host-pointer entry points
// Each call checks its arguments, declares its host inputs and outputs to a Staging (per-instance element counts) and runs the
// device-pointer entry point on the staged slices.
#define H2D(dst, src, n) CK(cudaMemcpyAsync(dst, src, (n), cudaMemcpyHostToDevice, ctx->stream))
#define D2H(dst, src, n) CK(cudaMemcpyAsync(dst, src, (n), cudaMemcpyDeviceToHost, ctx->stream))

int hb_wbc_qp_batch(hb_ctx* ctx, int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA,
                    double* x, int32_t* status, int32_t* iters) {
  if (!ctx || B < 0 || !H || !g || !A || !lbA || !ubA || !x) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (n < 1 || n > QP_MAX_N || m < 0 || m > QP_MAX_M) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto dH = s.in(H, (size_t)n * n); auto dA = s.in(A, (size_t)m * n); auto dg = s.in(g, n); auto dlb = s.in(lbA, m); auto dub = s.in(ubA, m);
  auto dx = s.out(x, n); auto dst = s.out(status, 1); auto dit = s.out(iters, 1);
  return s.run([&] { return hb_wbc_qp_batch_dev(ctx, B, n, m, dH, dg, dA, dlb, dub, dx, dst, dit); });
}

int hb_wbc_assemble_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                          const uint8_t* stance_mode, double* H, double* g, double* A, double* lbA, double* ubA, int32_t* m_rows) {
  if (!ctx || B < 0 || !x_des || !u_des || !rbd || !mode || !H || !g || !A || !lbA || !ubA || !m_rows) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto md = s.in(mode, 1); auto sm = s.in_or_null(stance_mode, 1);
  auto dH = s.out(H, QP_STRIDE_H); auto dA = s.out(A, QP_STRIDE_A); auto dg = s.out(g, NWBC); auto dlb = s.out(lbA, WBC_ROWS);
  auto dub = s.out(ubA, WBC_ROWS); auto dm = s.out(m_rows, 1);
  return s.run([&] { return hb_wbc_assemble_batch_dev(ctx, B, xd, ud, r, md, sm, dH, dg, dA, dlb, dub, dm); });
}

int hb_wbc_solve_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                       const uint8_t* stance_mode, double* sol, int32_t* status) {
  if (!ctx || B < 0 || !x_des || !u_des || !rbd || !mode || !sol) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto md = s.in(mode, 1); auto sm = s.in_or_null(stance_mode, 1);
  auto dsol = s.out(sol, NWBC); auto dst = s.out(status, 1);
  return s.run([&] { return hb_wbc_solve_batch_dev(ctx, B, xd, ud, r, md, sm, dsol, dst); });
}

int hb_hoqp_solve_batch(hb_ctx* ctx, int B, const hb_hoqp_problem* problems, double* x, double* slack, int32_t* status) {
  if (!ctx || B < 0 || !problems || !x) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  for (int i = 0; i < B; ++i) {
    const hb_hoqp_problem& p = problems[i];
    if (p.n < 1 || p.n > HB_HOQP_N || p.levels < 1 || p.levels > HB_HOQP_MAX_LEVELS) return HB_EINVAL;
    int stk = 0;
    for (int l = 0; l < p.levels; ++l) { if (p.ma[l] < 0 || p.ma[l] > HB_HOQP_MAX_EQ || p.md[l] < 0 || p.md[l] > HB_HOQP_MAX_IN) return HB_EINVAL; stk += p.md[l]; }
    if (stk > HB_HOQP_MAX_STACKED) return HB_EINVAL;
  }
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto pb = s.in(problems, 1); auto dx = s.out(x, HQ_N); auto dsl = s.out(slack, HQ_STK); auto dst = s.out(status, 1);
  return s.run([&] { return hb_hoqp_solve_batch_dev(ctx, B, pb, dx, dsl, dst); });
}

int hb_hierarchical_wbc_tasks_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                                    hb_hoqp_problem* problems) {
  if (!ctx || B < 0 || !x_des || !u_des || !rbd || !mode || !problems) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto md = s.in(mode, 1); auto pb = s.out(problems, 1);
  return s.run([&] { return hwbc_tasks_dev(ctx, B, xd, ud, r, md, pb); });
}

int hb_hierarchical_wbc_solve_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, double* sol,
                                    int32_t* status) {
  if (!ctx || B < 0 || !x_des || !u_des || !rbd || !mode || !sol) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto md = s.in(mode, 1);
  auto dsol = s.out(sol, NWBC); auto dst = s.out(status, 1);
  return s.run([&] { return hb_hierarchical_wbc_solve_batch_dev(ctx, B, xd, ud, r, md, dsol, dst); });
}

int hb_mpc_cold_start_batch(hb_ctx* ctx, int B, const double* x0, const int32_t* mode, double* x_traj, double* u_traj) {
  if (!ctx || B < 0 || !x0 || !mode || !x_traj || !u_traj) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(x0, NX); auto md = s.in(mode, N + 1); auto xt = s.out(x_traj, (N + 1) * NX); auto ut = s.out(u_traj, N * NU);
  return s.run([&] { return hb_mpc_cold_start_batch_dev(ctx, B, d0, md, xt, ut); });
}

int hb_mpc_solve_batch(hb_ctx* ctx, int B, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode, double* x_traj,
                       double* u_traj, hb_solve_info* info) {
  if (!ctx || B < 0 || !x0 || !x_ref || !swing_ref || !mode || !x_traj || !u_traj) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(x0, NX); auto xr = s.in(x_ref, (N + 1) * NX); auto sw = s.in(swing_ref, (N + 1) * 24); auto md = s.in(mode, N + 1);
  auto xt = s.inout(x_traj, (N + 1) * NX); auto ut = s.inout(u_traj, N * NU); auto inf = s.out(info, 1);
  return s.run([&] { return hb_mpc_solve_batch_dev(ctx, B, d0, xr, sw, md, xt, ut, inf); });
}

int hb_mpc_solve_grid_batch(hb_ctx* ctx, int B, const double* x0, const double* node_times, const int32_t* n_intervals, const double* x_ref,
                            const double* swing_ref, const int32_t* mode, double* x_traj, double* u_traj, hb_solve_info* info) {
  if (!ctx || B < 0 || !x0 || !node_times || !n_intervals || !x_ref || !swing_ref || !mode || !x_traj || !u_traj) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  const size_t N = ctx->cfg.horizon_N;
  for (int i = 0; i < B; ++i) {      // a grid the kernels can walk: 1 <= n <= N intervals of positive length
    if (n_intervals[i] < 1 || n_intervals[i] > (int)N) return HB_EINVAL;
    for (int k = 0; k < n_intervals[i]; ++k) if (!(node_times[(size_t)i * (N + 1) + k + 1] > node_times[(size_t)i * (N + 1) + k])) return HB_EINVAL;
  }
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto d0 = s.in(x0, NX); auto xr = s.in(x_ref, (N + 1) * NX); auto sw = s.in(swing_ref, (N + 1) * 24); auto md = s.in(mode, N + 1);
  auto xt = s.inout(x_traj, (N + 1) * NX); auto ut = s.inout(u_traj, N * NU); auto tk = s.in(node_times, N + 1); auto nn = s.in(n_intervals, 1);
  auto inf = s.out(info, 1);
  return s.run([&] { return hb_mpc_solve_grid_batch_dev(ctx, B, d0, tk, nn, xr, sw, md, xt, ut, inf); });
}

int hb_time_grid_batch(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* node_times, int32_t* n_intervals, int32_t* status) {
  if (!ctx || B < 0 || !t0 || !refs || !node_times || !n_intervals) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (!references_valid(B, refs)) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(t0, 1); auto rf = s.in(refs, 1); auto tk = s.out(node_times, N + 1); auto nn = s.out(n_intervals, 1); auto st = s.out(status, 1);
  return s.run([&] { return hb_time_grid_batch_dev(ctx, B, d0, rf, tk, nn, st); });
}

int hb_reference_expand_grid_batch(hb_ctx* ctx, int B, const double* node_times, const hb_reference* refs, double* x_ref, double* swing_ref,
                                   int32_t* mode) {
  if (!ctx || B < 0 || !node_times || !refs || !x_ref || !swing_ref || !mode) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (!references_valid(B, refs)) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto tk = s.in(node_times, N + 1); auto rf = s.in(refs, 1);
  auto xr = s.out(x_ref, (N + 1) * NX); auto sw = s.out(swing_ref, (N + 1) * 24); auto md = s.out(mode, N + 1);
  return s.run([&] { return hb_reference_expand_grid_batch_dev(ctx, B, tk, rf, xr, sw, md); });
}

int hb_resident_write_batch(hb_ctx* ctx, int B, const double* t0, const double* x_traj, const double* u_traj, const int32_t* mode, const double* node_times,
                            const int32_t* n_intervals) {
  if (!ctx || B < 0 || !t0 || !x_traj || !u_traj) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  const bool grid = ctx->cfg.event_nodes != 0;
  if (grid && (!node_times || !n_intervals)) return HB_EINVAL;      // an event-node context shifts between grids: the snapshot needs its grid
  const size_t N = ctx->cfg.horizon_N;
  if (grid) for (int i = 0; i < B; ++i) if (n_intervals[i] < 1 || n_intervals[i] > (int)N) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  H2D(ctx->res_t0, t0, sizeof(double) * B); H2D(ctx->res_xt, x_traj, sizeof(double) * B * (N + 1) * NX); H2D(ctx->res_ut, u_traj, sizeof(double) * B * N * NU);
  if (mode) H2D(ctx->res_mode, mode, sizeof(int32_t) * B * (N + 1));
  if (grid) { H2D(ctx->res_tk, node_times, sizeof(double) * B * (N + 1)); H2D(ctx->res_nn, n_intervals, sizeof(int32_t) * B); }
  int rc = hb_sync(ctx);
  if (rc) return rc;
  if (ctx->res_valid < B) ctx->res_valid = B;
  return HB_OK;
}

int hb_resident_read_grid_batch(hb_ctx* ctx, int B, double* node_times, int32_t* n_intervals) {
  if (!ctx || B < 0 || !node_times || !n_intervals) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->res_valid || !ctx->cfg.event_nodes) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N;
  D2H(node_times, ctx->res_tk, sizeof(double) * B * (N + 1)); D2H(n_intervals, ctx->res_nn, sizeof(int32_t) * B);
  return hb_sync(ctx);
}

int hb_control_step_batch(hb_ctx* ctx, int B, double t_rel, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                          const double* rbd, double* x_traj, double* u_traj, hb_solve_info* info, double* wbc_sol, double* torque,
                          int32_t* wbc_status) {
  if (!ctx || B < 0 || !x0 || !x_ref || !swing_ref || !mode || !rbd || !x_traj || !u_traj) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(x0, NX); auto xr = s.in(x_ref, (N + 1) * NX); auto sw = s.in(swing_ref, (N + 1) * 24); auto md = s.in(mode, N + 1);
  auto xt = s.inout(x_traj, (N + 1) * NX); auto ut = s.inout(u_traj, N * NU); auto r = s.in(rbd, 32);
  auto inf = s.out(info, 1); auto sol = s.out(wbc_sol, NWBC); auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1);
  const int rc = s.reserve();
  if (rc) return rc;
  // Two half-batches on two streams: the copies of one half overlap the kernels of the other (pinned host memory assumed).
  return chunked(ctx, B, B >= 256 ? 2 : 1, [&](int, size_t lo, size_t hi) -> int {
    int r2 = s.h2d(lo, hi);
    if (!r2) r2 = hb_control_step_batch_dev(ctx, (int)(hi - lo), t_rel, d0.at(lo), xr.at(lo), sw.at(lo), md.at(lo), r.at(lo), xt.at(lo), ut.at(lo),
                                            inf.at(lo), sol.at(lo), tau.at(lo), st.at(lo));
    return r2 ? r2 : s.d2h(lo, hi);
  });
}

// words (8 bytes) one packed instance needs
static inline size_t ref_pack_words(const hb_reference& r) {
  size_t w = 8 + (size_t)r.n_events + ((size_t)r.n_events + 2) / 2 + (size_t)r.n_targets * 23;
  for (int c = 0; c < 4; ++c) for (int a = 0; a < 3; ++a) w += (size_t)r.n_segments[c][a] * 6;
  return w;
}
// one instance's packed stream at p (ref_pack_words(r) words)
static inline void ref_pack_one(const hb_reference& r, double* p) {
  RefPackHeader hd;
  memset(&hd, 0, sizeof(hd));
  hd.n_events = r.n_events; hd.n_targets = r.n_targets;
  for (int q = 0; q < 12; ++q) hd.nseg[q] = r.n_segments[q / 3][q % 3];
  memcpy(p, &hd, sizeof(hd)); p += 8;
  memcpy(p, r.event_times, sizeof(double) * r.n_events); p += r.n_events;
  memcpy(p, r.modes, sizeof(int32_t) * (r.n_events + 1)); p += (r.n_events + 2) / 2;
  memcpy(p, r.target_times, sizeof(double) * r.n_targets); p += r.n_targets;
  memcpy(p, r.target_states, sizeof(double) * 22 * r.n_targets); p += 22 * r.n_targets;
  for (int q = 0; q < 12; ++q) { const int ns = r.n_segments[q / 3][q % 3]; memcpy(p, &r.segments[q / 3][q % 3][0][0], sizeof(double) * 6 * ns); p += 6 * ns; }
}
// pack refs[lo, hi) into the pinned staging area dst (offsets first, then the per-instance streams); returns the words used.
// Memory-bound on one core (5.3 MB read from the 17 KB-strided structs and 5.3 MB written per 1024 trot references), inside the caller's
// end-to-end time. Spreading the copies over host threads spawned per call was measured and rejected: on a host with a CPU quota the
// thread start-up costs more than the copies.
static size_t ref_pack(const hb_reference* refs, size_t lo, size_t hi, double* dst) {
  const size_t n = hi - lo;
  long long* offs = reinterpret_cast<long long*>(dst);
  size_t w = n + 1;
  for (size_t i = 0; i < n; ++i) {
    offs[i] = (long long)w;
    ref_pack_one(refs[lo + i], dst + w);
    w += ref_pack_words(refs[lo + i]);
  }
  offs[n] = (long long)w;
  return w;
}

int hb_resident_cycle_batch(hb_ctx* ctx, int B, int cold_start, double t_rel, const double* t0, const double* x0, const hb_reference* refs,
                            const double* rbd, hb_solve_info* info, double* wbc_sol, double* torque, int32_t* wbc_status) {
  if (!ctx || B < 0 || !t0 || !x0 || !refs || !rbd) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (!cold_start && ctx->res_valid < B) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  // a pinned (page-locked, mapped) reference array is read by the device directly
  const hb_reference* refs_dev = nullptr;
  {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, refs) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer) refs_dev = static_cast<const hb_reference*>(at.devicePointer);
    else cudaGetLastError();
  }
  // Chunks on two streams, as in hb_control_step_batch; only the small per-instance inputs and results cross PCIe.
  // Automatic choice: with a pageable reference array the host packs the used entries, and from 4096 instances on two chunks hide that pass
  // and the copies behind the other chunk's kernels; below, the half-batch kernels of the sequential stages run no faster than the full
  // batch. With a pinned array there is no host pass to hide and one chunk is used at every size.
  const int nchunk = cycle_chunks(ctx, B, !refs_dev);
  // pinned path: validation and byte count happen on the device while it copies (no per-instance host work at all); the verdict, two words
  // per chunk {invalid structs, words read}, comes back with the results. Pageable path: the used entries are packed into the context's
  // pinned host buffer, copied, and unpacked on the device.
  size_t pack_words = 0;
  if (!refs_dev) {
    if (!references_valid(B, refs)) return HB_EINVAL;
    for (int i = 0; i < B; ++i) pack_words += ref_pack_words(refs[i]);
    pack_words += (size_t)B + 2 * (size_t)nchunk + 8;
  }
  const size_t stat_words = refs_dev ? 2 * (size_t)nchunk : 0;
  Staging s(ctx, B);
  auto d0 = s.in(t0, 1); auto dx0 = s.in(x0, NX); auto r = s.in(rbd, 32); auto rf = s.tmp<hb_reference>(1);
  auto d_pack = s.buf<double>(pack_words); auto d_stat = s.buf<unsigned long long>(stat_words);
  auto inf = s.out(info, 1); auto sol = s.out(wbc_sol, NWBC); auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1);
  int rc = s.reserve();
  if (!rc) rc = grow(ctx, &ctx->pinned, &ctx->pinned_cap, refs_dev ? sizeof(unsigned long long) * stat_words : sizeof(double) * pack_words, true);
  if (rc) return rc;
  double* h_pack = static_cast<double*>(ctx->pinned);
  unsigned long long* h_stat = static_cast<unsigned long long*>(ctx->pinned);
  size_t pack_base = 0;
  ctx->last_h2d_bytes = 0;
  rc = chunked(ctx, B, nchunk, [&](int c, size_t lo, size_t hi) -> int {
    const int n = (int)(hi - lo);
    int r2 = s.h2d(lo, hi);
    if (r2) return r2;
    if (refs_dev) {
      CK(cudaMemsetAsync(d_stat.at(2 * c), 0, 2 * sizeof(unsigned long long), ctx->stream));
      r2 = launch(ctx, K_UNPROFILED, reference_gather_pinned_kernel, n, 128, 0, n, refs_dev + lo, rf.at(lo), d_stat.at(2 * c));
      if (r2) return r2;
      D2H(h_stat + 2 * c, d_stat.at(2 * c), 2 * sizeof(unsigned long long));
    } else {
      const size_t words = ref_pack(refs, lo, hi, h_pack + pack_base);
      H2D(d_pack.at(pack_base), h_pack + pack_base, sizeof(double) * words);
      r2 = launch(ctx, K_UNPROFILED, reference_unpack_kernel, n, 128, 0, n, reinterpret_cast<const long long*>(d_pack.at(pack_base)), d_pack.at(pack_base), rf.at(lo));
      if (r2) return r2;
      pack_base += words;
      ctx->last_h2d_bytes += sizeof(double) * words;
    }
    r2 = hb_resident_cycle_batch_dev(ctx, n, cold_start, t_rel, d0.at(lo), dx0.at(lo), rf.at(lo), r.at(lo), inf.at(lo), sol.at(lo), tau.at(lo), st.at(lo));
    return r2 ? r2 : s.d2h(lo, hi);
  });
  if (rc) return rc;
  if (refs_dev) {
    unsigned long long invalid = 0, words = 0;
    for (int c = 0; c < nchunk; ++c) { invalid += h_stat[2 * c]; words += h_stat[2 * c + 1]; }
    ctx->last_h2d_bytes = sizeof(double) * (size_t)words;
    if (invalid) { ctx->res_valid = 0; return HB_EINVAL; }      // malformed structs: counts were clamped on the device, the outputs are not meaningful
  }
  return HB_OK;
}

int hb_plan_references_gpu(hb_ctx* ctx, int B, const hb_plan_input* in, double* latest_stance, hb_reference* out, int32_t* status) {
  if (!ctx || B < 0 || !in || !latest_stance || !out) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto din = s.in(in, 1); auto ls = s.inout(latest_stance, 12); auto dout = s.out(out, 1); auto st = s.out(status, 1);
  return s.run([&] { return hb_plan_references_batch_dev(ctx, B, din, nullptr, ls, dout, st); });
}

int hb_resident_plan_cycle_batch(hb_ctx* ctx, int B, int cold_start, double t_rel, const hb_plan_input* in, const double* rbd, hb_solve_info* info,
                                 double* wbc_sol, double* torque, int32_t* wbc_status, int32_t* plan_status) {
  if (!ctx || B < 0 || !in || !rbd) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (!cold_start && ctx->res_valid < B) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  const int nchunk = cycle_chunks(ctx, B, true);
  Staging s(ctx, B);
  auto din = s.in(in, 1); auto r = s.in(rbd, 32);
  auto d0 = s.tmp<double>(1); auto dx0 = s.tmp<double>(NX); auto feet = s.tmp<double>(12); auto rf = s.tmp<hb_reference>(1);   // planner -> cycle
  auto inf = s.out(info, 1); auto sol = s.out(wbc_sol, NWBC); auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1); auto pst = s.out(plan_status, 1);
  const int rc = s.reserve();
  if (rc) return rc;
  return chunked(ctx, B, nchunk, [&](int, size_t lo, size_t hi) -> int {
    const int n = (int)(hi - lo);
    int r2 = s.h2d(lo, hi);
    if (r2) return r2;
    if (cold_start) CK(cudaMemsetAsync(ctx->res_stance + lo * 12, 0, sizeof(double) * n * 12, ctx->stream));   // latestStanceposition_ starts at zero
    r2 = launch(ctx, K_UNPROFILED, plan_prepare_kernel, (n + 63) / 64, 64, 0, n, din.at(lo), d0.at(lo), dx0.at(lo), feet.at(lo));
    if (!r2) r2 = hb_plan_references_batch_dev(ctx, n, din.at(lo), feet.at(lo), ctx->res_stance + lo * 12, rf.at(lo), pst.at(lo));
    if (!r2) r2 = hb_resident_cycle_batch_dev(ctx, n, cold_start, t_rel, d0.at(lo), dx0.at(lo), rf.at(lo), r.at(lo), inf.at(lo), sol.at(lo), tau.at(lo), st.at(lo));
    return r2 ? r2 : s.d2h(lo, hi);
  });
}

int hb_resident_read_batch(hb_ctx* ctx, int B, double* t0, double* x_traj, double* u_traj) {
  if (!ctx || B < 0) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->res_valid) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N;
  if (t0) D2H(t0, ctx->res_t0, sizeof(double) * B);
  if (x_traj) D2H(x_traj, ctx->res_xt, sizeof(double) * B * (N + 1) * NX);
  if (u_traj) D2H(u_traj, ctx->res_ut, sizeof(double) * B * N * NU);
  return hb_sync(ctx);
}

int hb_joint_command_batch(hb_ctx* ctx, int B, const hb_pd_gains* gains, double period, const double* x_des, const double* u_des,
                           const double* wbc_sol, const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded, uint8_t* estop,
                           double* command, double* output_torque) {
  if (!ctx || B < 0 || !gains || !x_des || !u_des || !wbc_sol || !mode_cmd || !rbd || !command || !output_torque) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto xd = s.in(x_des, NX); auto ud = s.in(u_des, NU); auto r = s.in(rbd, 32); auto sol = s.in(wbc_sol, NWBC); auto md = s.in(mode_cmd, 1);
  auto ld = s.in_or_null(loaded, 1); auto es = s.inout_or_null(estop, 1); auto cmd = s.out(command, NJ * 5); auto tau = s.out(output_torque, NJ);
  return s.run([&] { return hb_joint_command_batch_dev(ctx, B, gains, period, xd, ud, sol, md, r, ld, es, cmd, tau); });
}

int hb_estimator_update_batch(hb_ctx* ctx, int B, const hb_kf_params* params, double dt, hb_kf_state* state, const double* quat,
                              const double* ang_vel_local, const double* lin_acc_local, const double* joint_pos, const double* joint_vel,
                              const uint8_t* contact_flag, double* rbd_out) {
  if (!ctx || B < 0 || !params || !state || !quat || !ang_vel_local || !lin_acc_local || !joint_pos || !joint_vel || !contact_flag || !rbd_out) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto kf = s.inout(state, 1); auto q = s.in(quat, 4); auto w = s.in(ang_vel_local, 3); auto a = s.in(lin_acc_local, 3);
  auto jp = s.in(joint_pos, NJ); auto jv = s.in(joint_vel, NJ); auto fl = s.in(contact_flag, 4); auto ro = s.out(rbd_out, 32);
  return s.run([&] { return hb_estimator_update_batch_dev(ctx, B, params, dt, kf, q, w, a, jp, jv, fl, ro); });
}

int hb_actuation_batch(hb_ctx* ctx, int B, double delay, const double* time, hb_actuation_state* state, const double* command, const double* rbd,
                       double* tau) {
  if (!ctx || B < 0 || !time || !state || !command || !rbd || !tau) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto st = s.inout(state, 1); auto tm = s.in(time, 1); auto cmd = s.in(command, NJ * 5); auto r = s.in(rbd, 32); auto t = s.out(tau, NJ);
  return s.run([&] { return hb_actuation_batch_dev(ctx, B, delay, tm, st, cmd, r, t); });
}

int hb_sim_step_batch(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, double* contact_force, uint8_t* contact_flag) {
  if (!ctx || B < 0 || !params || !rbd || !tau) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto r = s.inout(rbd, 32); auto t = s.in(tau, NJ); auto cf = s.out(contact_force, 12); auto fl = s.out(contact_flag, 4);
  return s.run([&] { return hb_sim_step_batch_dev(ctx, B, params, r, t, cf, fl); });
}

int hb_resident_wbc_batch(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode, double* x_des, double* u_des,
                          int32_t* mode_out, double* wbc_sol, double* torque, int32_t* wbc_status) {
  if (!ctx || B < 0 || !t_now || !rbd || !x_des || !u_des || !mode_out || !wbc_sol) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (B > ctx->res_valid) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto tn = s.in(t_now, 1); auto r = s.in(rbd, 32); auto sm = s.in_or_null(stance_mode, 1);
  auto xd = s.out(x_des, NX); auto ud = s.out(u_des, NU); auto md = s.out(mode_out, 1); auto sol = s.out(wbc_sol, NWBC);
  auto tau = s.out(torque, NJ); auto st = s.out(wbc_status, 1);    // always passed: the fallback and its bookkeeping run on every call
  return s.run([&] { return hb_resident_wbc_batch_dev(ctx, B, tn, r, sm, xd, ud, md, sol, tau, st); });
}

int hb_contact_force_estimate_batch(hb_ctx* ctx, int B, double cutoff_frequency, double dt, hb_observer_state* state, const double* rbd,
                                    const double* tau_cmd, double* est_contact_force, double* disturbance_torque) {
  if (!ctx || B < 0 || !state || !rbd || !tau_cmd || !est_contact_force) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto st = s.inout(state, 1); auto r = s.in(rbd, 32); auto t = s.in(tau_cmd, NJ); auto est = s.out(est_contact_force, 16);
  auto dist = s.out(disturbance_torque, NQ);
  return s.run([&] { return hb_contact_force_estimate_batch_dev(ctx, B, cutoff_frequency, dt, st, r, t, est, dist); });
}

int hb_rbd_to_centroidal_batch(hb_ctx* ctx, int B, const double* rbd, double* x) {
  if (!ctx || B < 0 || !rbd || !x) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto r = s.in(rbd, 32); auto dx = s.out(x, NX);
  return s.run([&] { return hb_rbd_to_centroidal_batch_dev(ctx, B, r, dx); });
}

int hb_reference_expand_batch(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* x_ref, double* swing_ref, int32_t* mode) {
  if (!ctx || B < 0 || !t0 || !refs || !x_ref || !swing_ref || !mode) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (!references_valid(B, refs)) return HB_EINVAL;
  if (set_device(ctx)) return HB_ECUDA;
  const size_t N = ctx->cfg.horizon_N;
  Staging s(ctx, B);
  auto d0 = s.in(t0, 1); auto rf = s.in(refs, 1);
  auto xr = s.out(x_ref, (N + 1) * NX); auto sw = s.out(swing_ref, (N + 1) * 24); auto md = s.out(mode, N + 1);
  return s.run([&] { return hb_reference_expand_batch_dev(ctx, B, d0, rf, xr, sw, md); });
}

int hb_contact_positions_batch(hb_ctx* ctx, int B, const double* x, double* pos) {
  if (!ctx || B < 0 || !x || !pos) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto dx = s.in(x, NX); auto dp = s.out(pos, 12);
  return s.run([&] { return hb_contact_positions_batch_dev(ctx, B, dx, dp); });
}

static std::atomic<int> g_plan_threads{0};   // 0 = hardware_concurrency (hb_plan_set_threads)
static int plan_range(int lo, int hi, const hb_plan_input* in, double* latest_stance, hb_reference* out) {
  static const hbplan::PlanConsts pc = hbplan::make_consts();
  for (int i = lo; i < hi; ++i) {
    const int rc = hbplan::plan_one(pc, in[i], latest_stance + (size_t)i * 12, out + i, true);
    if (rc) return rc;
  }
  return HB_OK;
}

int hb_plan_set_threads(int n_threads) {
  if (n_threads < 0) return HB_EINVAL;
  g_plan_threads.store(n_threads);
  return HB_OK;
}

int hb_plan_references(int B, const hb_plan_input* in, double* latest_stance, hb_reference* out) {
  if (B < 0 || !in || !latest_stance || !out) return HB_EINVAL;
  // instances are independent: spread them over the host cores (the planner feeds ~1e5 solves/s per GPU; one core plans ~2e4/s)
  unsigned hw = std::thread::hardware_concurrency();
  if (const int forced = g_plan_threads.load()) hw = (unsigned)forced;
  int nt = (int)std::min<unsigned>(hw ? hw : 1u, (unsigned)((B + 63) / 64));
  if (nt <= 1) return plan_range(0, B, in, latest_stance, out);
  std::vector<std::thread> pool;
  std::vector<int> rcs(nt, HB_OK);
  for (int t = 0; t < nt; ++t) {
    const int lo = (int)((long long)B * t / nt), hi = (int)((long long)B * (t + 1) / nt);
    pool.emplace_back([=, &rcs]() { rcs[t] = plan_range(lo, hi, in, latest_stance, out); });
  }
  for (auto& th : pool) th.join();
  for (int t = 0; t < nt; ++t) if (rcs[t]) return rcs[t];
  return HB_OK;
}

int hb_gait_select(int B, hb_gait_selector* state, const int32_t* gait_type, const double* cmd_vel, const double* target_state0, int32_t* level,
                   int32_t* insert) {
  if (B < 0 || !state || !gait_type || !cmd_vel || !target_state0 || !level || !insert) return HB_EINVAL;
  for (int i = 0; i < B; ++i) {
    if (state[i].head < 0 || state[i].head >= 50 || state[i].count < 0 || state[i].count > 50) return HB_EINVAL;
    int ins = 0;
    level[i] = hbplan::gait_select(state + i, gait_type[i], cmd_vel + (size_t)i * 4, target_state0 + (size_t)i * 22, &ins);
    insert[i] = ins;
  }
  return HB_OK;
}

int hb_probe_flow_map(hb_ctx* ctx, int B, const double* x, const double* u, double* f, double* A, double* Bm, double* ee) {
  if (!ctx || B < 0 || !x || !u || !f || !A || !Bm) return HB_EINVAL;
  if (B == 0) return HB_OK;
  if (B > ctx->cfg.max_batch) return HB_ECAP;
  if (set_device(ctx)) return HB_ECUDA;
  Staging s(ctx, B);
  auto dx = s.in(x, NX); auto du = s.in(u, NU);
  auto df = s.out(f, NX); auto dA = s.out(A, TS); auto dB = s.out(Bm, TS); auto dee = s.out(ee, 24 + 36 * NX);
  return s.run([&] { return hb_probe_flow_map_dev(ctx, B, dx, du, df, dA, dB, dee); });
}

}  // extern "C"

#include "hb_shard.cuh"
