// Hierarchical QP (HoQP) on the device, one warp per instance: legged::HoQp (legged_wbc/src/HoQp.cpp:21-198) and the three-level cascade of
// legged::HierarchicalWbc::update (legged_wbc/src/HierarchicalWbc.cpp:18-31). SURVEY 8f row N4.
//
// Level k (task: A_k x = b_k in the least-squares sense, D_k x <= f_k softened by slacks v >= 0) is solved in the null space Z of all
// higher-priority equality tasks, x = x_prev + Z z:
//     min 1/2 ||A_k (x_prev + Z z) - b_k||^2 + 1/2 ||v||^2
//     s.t. -v <= 0,   D_prev (x_prev + Z z) <= f_prev + v_prev*  (stacked higher levels, their slack solutions frozen),   D_k (x_prev + Z z) - v <= f_k
// exactly the (H, c, D, f) of HoQp::buildHMatrix / buildCVector / buildDMatrix / buildFVector, handed to the batched interior point
// (qp_solve_warp replaces qpOASES as in the weighted WBC). Then Z <- Z kernel(A_k Z) (HoQp::buildZMatrix: Eigen FullPivLU::kernel; here a
// Gauss-Jordan elimination with complete pivoting -- any basis of the same null space gives the same x).
#pragma once
#include "hb_common.cuh"
#include "hb_qp.cuh"
#include "../../include/hunter_b200.h"

namespace hb {

constexpr int HQ_N = HB_HOQP_N, HQ_MA = HB_HOQP_MAX_EQ, HQ_MD = HB_HOQP_MAX_IN, HQ_STK = HB_HOQP_MAX_STACKED;
constexpr int HQ_NQ = HQ_N + HQ_MD;                // variables of a lifted level problem (z, v)
constexpr int HQ_ROWS = 2 * HQ_MD + HQ_STK;         // rows of a lifted level problem
constexpr int HQ_LDZ = HQ_N + 1, HQ_LDA = HQ_N + 1;
// global scratch per instance (doubles): lifted H, c, D, lb, ub, z; stacked D, f, slack
constexpr size_t HQ_SCRATCH = (size_t)HQ_NQ * HQ_NQ + HQ_NQ + (size_t)HQ_ROWS * HQ_NQ + 2 * HQ_ROWS + HQ_NQ + (size_t)HQ_STK * HQ_N + 2 * HQ_STK;

struct HoqpShared {
  double Z[HQ_N * HQ_LDZ];       // current null-space basis (n x nx)
  double AZ[HQ_MA * HQ_LDA];     // A_k Z (ma x nx), then its reduced row echelon form
  double Zn[HQ_N * HQ_LDZ];      // next basis while it is formed
  double x[HQ_N], r[HQ_MA];
  int pcol[HQ_MA], prow[HQ_MA], isp[HQ_N], freec[HQ_N];
};
__host__ __device__ inline size_t hoqp_smem_bytes() { return sizeof(HoqpShared) + qp_workspace_doubles(HQ_NQ, 1, HQ_ROWS) * sizeof(double); }

// Solve one hierarchy. Returns 0, or the first failing level's QP status * 10 + level.
__device__ inline int hoqp_solve_warp(const hb_hoqp_problem& pb, HoqpShared& sh, QpWorkspace& w, double* scratch, int max_iter, double* x_out,
                                      double* slack_out) {
  const int lane = lane_id();
  const int n = min(max(pb.n, 1), HQ_N), L = min(max(pb.levels, 0), HB_HOQP_MAX_LEVELS);
  double* Hq = scratch; double* cq = Hq + (size_t)HQ_NQ * HQ_NQ; double* Dq = cq + HQ_NQ; double* lbq = Dq + (size_t)HQ_ROWS * HQ_NQ; double* ubq = lbq + HQ_ROWS;
  double* zq = ubq + HQ_ROWS; double* stkD = zq + HQ_NQ; double* stkf = stkD + (size_t)HQ_STK * HQ_N; double* stks = stkf + HQ_STK;
  for (int idx = lane; idx < n * HQ_LDZ; idx += 32) { const int i = idx / HQ_LDZ, j = idx - i * HQ_LDZ; sh.Z[idx] = (i == j) ? 1.0 : 0.0; }
  for (int i = lane; i < n; i += 32) sh.x[i] = 0.0;
  __syncwarp();
  int nx = n, nstk = 0, status = 0;
  for (int lvl = 0; lvl < L; ++lvl) {
    const int ma = min(max(pb.ma[lvl], 0), HQ_MA), md = min(max(pb.md[lvl], 0), HQ_MD);
    const double* A = &pb.a[lvl][0][0]; const double* bvec = pb.b[lvl]; const double* D = &pb.d[lvl][0][0]; const double* fvec = pb.f[lvl];
    if (nstk + md > HQ_STK) { status = 20 + lvl; break; }
    double* slk = stks + nstk;                     // slack solution of this level goes to the end of the stack
    if (nx > 0) {
      // AZ = A Z, r = A x - b
      for (int idx = lane; idx < ma * nx; idx += 32) {
        const int i = idx / nx, j = idx - i * nx;
        double s = 0.0;
        for (int k = 0; k < n; ++k) s = fma(A[i * HQ_N + k], sh.Z[k * HQ_LDZ + j], s);
        sh.AZ[i * HQ_LDA + j] = s;
      }
      for (int i = lane; i < ma; i += 32) { double s = -bvec[i]; for (int k = 0; k < n; ++k) s = fma(A[i * HQ_N + k], sh.x[k], s); sh.r[i] = s; }
      __syncwarp();
      const int nq = nx + md, nr = 2 * md + nstk;
      // lifted Hessian and gradient (HoQp::buildHMatrix / buildCVector)
      for (int idx = lane; idx < nq * nq; idx += 32) {
        const int i = idx / nq, j = idx - i * nq;
        double s = 0.0;
        if (i < nx && j < nx) { for (int k = 0; k < ma; ++k) s = fma(sh.AZ[k * HQ_LDA + i], sh.AZ[k * HQ_LDA + j], s); if (i == j) s += 1e-12; }
        else if (i == j) s = 1.0;
        Hq[idx] = s;
      }
      for (int i = lane; i < nq; i += 32) {
        double s = 0.0;
        if (i < nx) for (int k = 0; k < ma; ++k) s = fma(sh.AZ[k * HQ_LDA + i], sh.r[k], s);
        cq[i] = s;
      }
      // lifted inequality rows (HoQp::buildDMatrix / buildFVector)
      for (int idx = lane; idx < nr * nq; idx += 32) {
        const int i = idx / nq, j = idx - i * nq;
        double s = 0.0;
        if (i < md) s = (j == nx + i) ? -1.0 : 0.0;
        else if (i < md + nstk) { if (j < nx) { const double* dr = stkD + (size_t)(i - md) * HQ_N; for (int k = 0; k < n; ++k) s = fma(dr[k], sh.Z[k * HQ_LDZ + j], s); } }
        else { const int ii = i - md - nstk; if (j < nx) { for (int k = 0; k < n; ++k) s = fma(D[ii * HQ_N + k], sh.Z[k * HQ_LDZ + j], s); } else s = (j == nx + ii) ? -1.0 : 0.0; }
        Dq[idx] = s;
      }
      for (int i = lane; i < nr; i += 32) {
        double u = 0.0;
        if (i >= md && i < md + nstk) { const double* dr = stkD + (size_t)(i - md) * HQ_N; double s = 0.0; for (int k = 0; k < n; ++k) s = fma(dr[k], sh.x[k], s); u = stkf[i - md] - s + stks[i - md]; }
        else if (i >= md + nstk) { const int ii = i - md - nstk; double s = 0.0; for (int k = 0; k < n; ++k) s = fma(D[ii * HQ_N + k], sh.x[k], s); u = fvec[ii] - s; }
        lbq[i] = -1e20; ubq[i] = u;
      }
      __syncwarp();
      const QpResult qr = qp_solve_warp(nq, nr, Hq, cq, Dq, lbq, ubq, 1e-10, max_iter, zq, w);
      __syncwarp();
      if (qr.status != 0 && status == 0) status = 10 * qr.status + lvl;
      // x <- x + Z z ; slack of this level
      double xn = 0.0;
      if (lane < n) { xn = sh.x[lane]; for (int j = 0; j < nx; ++j) xn = fma(sh.Z[lane * HQ_LDZ + j], zq[j], xn); }
      double xn2 = 0.0;
      if (lane + 32 < n) { xn2 = sh.x[lane + 32]; for (int j = 0; j < nx; ++j) xn2 = fma(sh.Z[(lane + 32) * HQ_LDZ + j], zq[j], xn2); }
      __syncwarp();
      if (lane < n) sh.x[lane] = xn;
      if (lane + 32 < n) sh.x[lane + 32] = xn2;
      for (int i = lane; i < md; i += 32) slk[i] = zq[nx + i];
    } else {
      // nothing left to decide: the slacks absorb whatever the higher priorities leave
      for (int i = lane; i < md; i += 32) { double s = -fvec[i]; for (int k = 0; k < n; ++k) s = fma(D[i * HQ_N + k], sh.x[k], s); slk[i] = s > 0.0 ? s : 0.0; }
    }
    // stack this level's inequalities (Task::operator+, Task.h:46-58)
    for (int idx = lane; idx < md * n; idx += 32) { const int i = idx / n, k = idx - i * n; stkD[(size_t)(nstk + i) * HQ_N + k] = D[i * HQ_N + k]; }
    for (int i = lane; i < md; i += 32) stkf[nstk + i] = fvec[i];
    nstk += md;
    __syncwarp();
    // Z <- Z kernel(A Z): reduced row echelon form of AZ with complete pivoting
    if (ma > 0 && nx > 0) {
      double amax = 0.0;
      for (int idx = lane; idx < ma * nx; idx += 32) amax = fmax(amax, fabs(sh.AZ[(idx / nx) * HQ_LDA + idx % nx]));
      amax = warp_max(amax);
      const double tol = 1e-9 * fmax(amax, 1e-300);
      for (int j = lane; j < nx; j += 32) sh.isp[j] = 0;
      __syncwarp();
      int rank = 0;
      unsigned long long rowused = 0ull;
      for (int step = 0; step < min(ma, nx); ++step) {
        double best = -1.0; int bi = 0, bj = 0;
        for (int idx = lane; idx < ma * nx; idx += 32) {
          const int i = idx / nx, j = idx - i * nx;
          if (((rowused >> i) & 1ull) || sh.isp[j]) continue;
          const double a = fabs(sh.AZ[i * HQ_LDA + j]);
          if (a > best) { best = a; bi = i; bj = j; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const double ob = __shfl_xor_sync(HB_FULL_MASK, best, o);
          const int oi = __shfl_xor_sync(HB_FULL_MASK, bi, o), oj = __shfl_xor_sync(HB_FULL_MASK, bj, o);
          if (ob > best || (ob == best && (oi < bi || (oi == bi && oj < bj)))) { best = ob; bi = oi; bj = oj; }
        }
        if (!(best > tol)) break;
        const double inv = 1.0 / sh.AZ[bi * HQ_LDA + bj];
        __syncwarp();
        for (int j = lane; j < nx; j += 32) sh.AZ[bi * HQ_LDA + j] *= inv;
        __syncwarp();
        for (int idx = lane; idx < ma * nx; idx += 32) {
          const int i = idx / nx, j = idx - i * nx;
          if (i == bi || j == bj) continue;
          sh.AZ[i * HQ_LDA + j] -= sh.AZ[i * HQ_LDA + bj] * sh.AZ[bi * HQ_LDA + j];
        }
        __syncwarp();
        for (int i = lane; i < ma; i += 32) if (i != bi) sh.AZ[i * HQ_LDA + bj] = 0.0;
        if (lane == 0) { sh.pcol[rank] = bj; sh.prow[rank] = bi; sh.isp[bj] = 1; }
        rowused |= 1ull << bi;
        ++rank;
        __syncwarp();
      }
      int nfree = 0;
      for (int j = 0; j < nx; ++j) if (!sh.isp[j]) { if (lane == 0) sh.freec[nfree] = j; ++nfree; }
      __syncwarp();
      // column c of the new basis: Z[:, f] - sum_i Z[:, pcol_i] R[prow_i][f]
      for (int idx = lane; idx < n * nfree; idx += 32) {
        const int k = idx / nfree, c = idx - k * nfree, fcol = sh.freec[c];
        double s = sh.Z[k * HQ_LDZ + fcol];
        for (int i = 0; i < rank; ++i) s = fma(-sh.Z[k * HQ_LDZ + sh.pcol[i]], sh.AZ[sh.prow[i] * HQ_LDA + fcol], s);
        sh.Zn[k * HQ_LDZ + c] = s;
      }
      __syncwarp();
      for (int idx = lane; idx < n * nfree; idx += 32) { const int k = idx / nfree, c = idx - k * nfree; sh.Z[k * HQ_LDZ + c] = sh.Zn[k * HQ_LDZ + c]; }
      nx = nfree;
      __syncwarp();
    }
  }
  for (int i = lane; i < n; i += 32) x_out[i] = sh.x[i];
  if (slack_out) for (int i = lane; i < HQ_STK; i += 32) slack_out[i] = i < nstk ? stks[i] : 0.0;
  return status;
}

}  // namespace hb

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
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
}  // namespace
