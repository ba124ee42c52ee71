// K5: WeightedWbc problem assembly on the device (legged_wbc/src/WbcBase.cpp:54-338, WeightedWbc.cpp:18-94),
// one warp per instance. Lane-level parallelism (see hb_rbd.cuh):
//   pass A  lanes 0-15: unit velocities at the measured q -> contact Jacobian columns J_c (12x16)
//           lanes 16-31: unit velocities at the planned q -> centroidal momentum matrix columns A(q_des) (6x16)
//   pass B  lane 0: dual pass at (q_meas; direction v_meas)  -> p_c, v_c, dJ_c/dt v   (WbcBase.cpp:91-109)
//           lane 1: dual pass at (q_des;  direction v_des)   -> p_c, v_c, dA/dt v      (WbcBase.cpp:119-136)
//   pass C  lanes 0-15: RNEA with unit accelerations -> M(q) columns (CRBA, WbcBase.cpp:88-89); lane 16: nle (WbcBase.cpp:90)
// The QP (H, g, A, lbA, ubA) is written in the reference's own layout (qpOASES row-major, WeightedWbc.cpp:27-41).
#pragma once
#include "hb_common.cuh"
#include "hb_qp.cuh"
#include "hb_rbd.cuh"
#include "../../include/hunter_b200.h"

namespace hb {

constexpr int WBC_ROWS = 60;     // allocated rows of A per instance
constexpr double QP_INFTY = 1e20;  // qpOASES::INFTY

struct WbcShared {
  double J[12 * 16];
  double Ad[6 * 16];
  double M[16 * 16];
  double nle[16];
  double q[16], v[16], qd[16], vd[16];
  double pos_m[12], vel_m[12], dJv[12], pos_d[12], vel_d[12];
  double Adv[6], com_d[3];
  double Aw[18 * 16];   // weighted task rows acting on qdd (swing: <=12, base: 6)
  double bw[18];
  double misc[32];
};

// rotationMatrixToRotationVector(R_ref R_meas^T)  (rotationErrorInWorld, WbcBase.cpp:281)
__device__ inline void rotation_error_world(const double* Rref, const double* Rmeas, double* err) {
  double E[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) E[3 * i + j] = Rref[3 * i] * Rmeas[3 * j] + Rref[3 * i + 1] * Rmeas[3 * j + 1] + Rref[3 * i + 2] * Rmeas[3 * j + 2];
  const double sk[3] = {E[7] - E[5], E[2] - E[6], E[3] - E[1]};
  double c = 0.5 * (E[0] + E[4] + E[8] - 1.0);
  c = fmin(1.0, fmax(-1.0, c));
  const double ang = acos(c);
  const double sn = sqrt(sk[0] * sk[0] + sk[1] * sk[1] + sk[2] * sk[2]);
  double f = 0.5;
  if (ang > 1e-8 && sn > 1e-12) f = ang / sn;
  for (int i = 0; i < 3; ++i) err[i] = f * sk[i];
}

// Assemble one instance. Outputs may be global or shared. Returns the number of constraint rows m.
__device__ inline int wbc_assemble_warp(const double* __restrict__ x_des, const double* __restrict__ u_des,
                                        const double* __restrict__ rbd, int mode, bool stance_mode, const hb_wbc_settings& ws, WbcShared& sh,
                                        double* H, double* g, double* A, double* lbA, double* ubA, int* nw_out = nullptr) {
  const int lane = lane_id();
  const Model& md = c_model;
  // ---- measured q, v (WbcBase.cpp:72-79)
  if (lane == 0) {
    for (int i = 0; i < 3; ++i) { sh.q[i] = rbd[3 + i]; sh.q[3 + i] = rbd[i]; sh.v[i] = rbd[NQ + 3 + i]; }
    for (int j = 0; j < NJ; ++j) { sh.q[6 + j] = rbd[6 + j]; sh.v[6 + j] = rbd[NQ + 6 + j]; }
    double sz, cz, sy, cy;
    sincos(sh.q[3], &sz, &cz); sincos(sh.q[4], &sy, &cy);
    const double w0 = rbd[NQ], w1 = rbd[NQ + 1], w2 = rbd[NQ + 2];
    const double dxr = (cz * w0 + sz * w1) / cy;
    sh.v[5] = dxr; sh.v[4] = -sz * w0 + cz * w1; sh.v[3] = w2 + sy * dxr;
    for (int i = 0; i < NQ; ++i) sh.qd[i] = x_des[6 + i];
  }
  __syncwarp();
  // ---- pass A
  {
    double q[NQ], e[NQ];
    const bool meas = lane < 16;
    const int k = lane & 15;
    for (int i = 0; i < NQ; ++i) { q[i] = meas ? sh.q[i] : sh.qd[i]; e[i] = (i == k) ? 1.0 : 0.0; }
    KinOut<double> o;
    kin_pass<double>(q, e, o);
    if (meas) { for (int r = 0; r < 12; ++r) sh.J[r * 16 + k] = o.cvel[r]; }
    else { for (int r = 0; r < 6; ++r) sh.Ad[r * 16 + k] = o.h[r]; }
  }
  __syncwarp();
  // ---- planned generalised velocity: v_b = A_b^-1 (m hbar - A_j qj_dot)  (mapping_.getPinocchioJointVelocity, WbcBase.cpp:130)
  if (lane == 0) {
    double Ab[36], rhs[6], vb[6];
    for (int r = 0; r < 6; ++r) {
      for (int c = 0; c < 6; ++c) Ab[6 * r + c] = sh.Ad[r * 16 + c];
      double s = md.total_mass * x_des[r];
      for (int j = 0; j < NJ; ++j) s -= sh.Ad[r * 16 + 6 + j] * u_des[12 + j];
      rhs[r] = s;
    }
    solve6_cmm(Ab, rhs, vb);
    for (int i = 0; i < 6; ++i) sh.vd[i] = vb[i];
    for (int j = 0; j < NJ; ++j) sh.vd[6 + j] = u_des[12 + j];
  }
  __syncwarp();
  // ---- pass B (dual pass along q_dot = v)
  if (lane < 2) {
    D1 q[NQ], v[NQ];
    for (int i = 0; i < NQ; ++i) {
      const double qi = lane == 0 ? sh.q[i] : sh.qd[i], vi = lane == 0 ? sh.v[i] : sh.vd[i];
      q[i] = D1(qi, vi); v[i] = D1(vi, 0.0);
    }
    KinOut<D1> o;
    kin_pass<D1>(q, v, o);
    if (lane == 0) { for (int r = 0; r < 12; ++r) { sh.pos_m[r] = o.cpos[r].v; sh.vel_m[r] = o.cvel[r].v; sh.dJv[r] = o.cvel[r].d; } }
    else {
      for (int r = 0; r < 12; ++r) { sh.pos_d[r] = o.cpos[r].v; sh.vel_d[r] = o.cvel[r].v; }
      for (int r = 0; r < 6; ++r) sh.Adv[r] = o.h[r].d;
      for (int r = 0; r < 3; ++r) sh.com_d[r] = o.com[r].v;
    }
  }
  // ---- pass C (RNEA columns)
  if (lane < 17) {
    double q[NQ], v[NQ], a[NQ], tau[NQ];
    for (int i = 0; i < NQ; ++i) { q[i] = sh.q[i]; v[i] = lane == 16 ? sh.v[i] : 0.0; a[i] = (i == lane) ? 1.0 : 0.0; }
    rnea_pass(q, v, a, lane == 16, tau, nullptr);
    if (lane < 16) { for (int r = 0; r < NQ; ++r) sh.M[r * 16 + lane] = tau[r]; }
    else { for (int r = 0; r < NQ; ++r) sh.nle[r] = tau[r]; }
  }
  __syncwarp();
  // symmetrise M (WbcBase.cpp:88-89 copies the upper triangle; numerically the same matrix)
  for (int idx = lane; idx < 256; idx += 32) {
    const int i = idx >> 4, j = idx & 15;
    if (j < i) { const double a = 0.5 * (sh.M[i * 16 + j] + sh.M[j * 16 + i]); sh.M[i * 16 + j] = a; }
  }
  __syncwarp();
  for (int idx = lane; idx < 256; idx += 32) { const int i = idx >> 4, j = idx & 15; if (j > i) sh.M[i * 16 + j] = sh.M[j * 16 + i]; }
  __syncwarp();
  // ---- desired base kinematics (computeBaseKinematicsFromCentroidalModel, WbcBase.cpp:134-135) and task rows
  int nw = 0;  // number of weighted rows (uniform)
  bool fl[4];
  int nc = 0;
  for (int c = 0; c < 4; ++c) { fl[c] = contact_flag(mode, c); nc += fl[c]; }
  if (stance_mode) nw = 6;
  else nw = 3 * (4 - nc) + 6;
  if (lane == 0) {
    for (int i = 0; i < 18 * 16; ++i) sh.Aw[i] = 0.0;
    if (stance_mode) {
      for (int i = 0; i < 6; ++i) { sh.Aw[i * 16 + i] = ws.weight_base_accel; sh.bw[i] = 0.0; }
    } else {
      // normalised centroidal momentum rate at the plan (getNormalizedCentroidalMomentumRate)
      double hd[6] = {0, 0, 0, 0, 0, 0};
      for (int c = 0; c < 4; ++c) {
        const double* F = u_des + 3 * c;
        const double r0 = sh.pos_d[3 * c] - sh.com_d[0], r1 = sh.pos_d[3 * c + 1] - sh.com_d[1], r2 = sh.pos_d[3 * c + 2] - sh.com_d[2];
        hd[0] += F[0]; hd[1] += F[1]; hd[2] += F[2];
        hd[3] += r1 * F[2] - r2 * F[1]; hd[4] += r2 * F[0] - r0 * F[2]; hd[5] += r0 * F[1] - r1 * F[0];
      }
      hd[2] -= md.total_mass * HB_GRAVITY;
      double Ab[36], rhs[6], qbdd[6];
      for (int r = 0; r < 6; ++r) { for (int c = 0; c < 6; ++c) Ab[6 * r + c] = sh.Ad[r * 16 + c]; rhs[r] = hd[r] - sh.Adv[r]; }
      solve6_cmm(Ab, rhs, qbdd);
      // euler axes at the plan and at the measurement
      double Rd[9], axd[9], Rm[9], axm[9];
      base_frame<double>(sh.qd, Rd, axd);
      base_frame<double>(sh.q, Rm, axm);
      double baseVelW[3], baseAccW[3], wm[3], dJw_v[3];
      {
        const double* vd = sh.vd;
        double w1[3], w2[3], t1[3], t2[3];
        for (int i = 0; i < 3; ++i) { w1[i] = axd[i] * vd[3]; w2[i] = w1[i] + axd[3 + i] * vd[4]; }
        cross(w1, &axd[3], t1); cross(w2, &axd[6], t2);
        for (int i = 0; i < 3; ++i) {
          baseVelW[i] = w2[i] + axd[6 + i] * vd[5];
          baseAccW[i] = axd[i] * qbdd[3] + axd[3 + i] * qbdd[4] + axd[6 + i] * qbdd[5] + t1[i] * vd[4] + t2[i] * vd[5];
        }
      }
      {
        const double* vm = sh.v;
        double w1[3], w2[3], t1[3], t2[3];
        for (int i = 0; i < 3; ++i) { w1[i] = axm[i] * vm[3]; w2[i] = w1[i] + axm[3 + i] * vm[4]; }
        cross(w1, &axm[3], t1); cross(w2, &axm[6], t2);
        for (int i = 0; i < 3; ++i) { wm[i] = w2[i] + axm[6 + i] * vm[5]; dJw_v[i] = t1[i] * vm[4] + t2[i] * vm[5]; }
      }
      int r = 0;
      // swing leg task (WbcBase.cpp:297-323), weight 100
      for (int c = 0; c < 4; ++c) if (!fl[c]) for (int a = 0; a < 3; ++a) {
        const double acc = ws.swing_kp * (sh.pos_d[3 * c + a] - sh.pos_m[3 * c + a]) + ws.swing_kd * (sh.vel_d[3 * c + a] - sh.vel_m[3 * c + a]);
        for (int j = 0; j < NQ; ++j) sh.Aw[r * 16 + j] = ws.weight_swing_leg * sh.J[(3 * c + a) * 16 + j];
        sh.bw[r] = ws.weight_swing_leg * (acc - sh.dJv[3 * c + a]);
        ++r;
      }
      // base xy acceleration (WbcBase.cpp:228-240)
      for (int a = 0; a < 2; ++a) { sh.Aw[r * 16 + a] = ws.weight_base_accel; sh.bw[r] = ws.weight_base_accel * qbdd[a]; ++r; }
      // base height (WbcBase.cpp:243-256)
      sh.Aw[r * 16 + 2] = ws.weight_base_accel;
      sh.bw[r] = ws.weight_base_accel * (qbdd[2] + ws.base_height_kp * (sh.qd[2] - sh.q[2]) + ws.base_height_kd * (sh.vd[2] - sh.v[2]));
      ++r;
      // base angular motion (WbcBase.cpp:259-290)
      double err[3];
      rotation_error_world(Rd, Rm, err);
      for (int a = 0; a < 3; ++a) {
        for (int i = 0; i < 3; ++i) sh.Aw[r * 16 + 3 + i] = ws.weight_base_accel * axm[3 * i + a];
        sh.bw[r] = ws.weight_base_accel * (baseAccW[a] + ws.base_angular_kp * err[a] + ws.base_angular_kd * (baseVelW[a] - wm[a]) - dJw_v[a]);
        ++r;
      }
    }
  }
  __syncwarp();
  if (nw_out) *nw_out = nw;
  if (H == nullptr) return 16 + 3 * (4 - nc) + 20 + 5 * nc + 3 * (4 - nc);   // terms only (fused path builds the reduced QP from sh)
  // ---- H = Aw'Aw, g = -Aw'bw (WeightedWbc.cpp:38-41); only the qdd block is non-zero
  // formulateContactForceTask * weightContactForce (WbcBase.cpp:325-338, WeightedWbc.cpp:87-91; not in stance mode): rows w_f [0 | I_12 | 0] x = w_f F_des
  const double wf2 = stance_mode ? 0.0 : ws.weight_contact_force * ws.weight_contact_force;
  for (int idx = lane; idx < NWBC * NWBC; idx += 32) {
    const int i = idx / NWBC, j = idx - i * NWBC;
    double s = 0.0;
    if (i < NQ && j < NQ) for (int r = 0; r < nw; ++r) s += sh.Aw[r * 16 + i] * sh.Aw[r * 16 + j];
    if (i == j && i >= NQ && i < NQ + 12) s += wf2;
    H[idx] = s;
  }
  for (int i = lane; i < NWBC; i += 32) {
    double s = 0.0;
    if (i < NQ) for (int r = 0; r < nw; ++r) s += sh.Aw[r * 16 + i] * sh.bw[r];
    else if (i < NQ + 12) s = wf2 * u_des[i - NQ];
    g[i] = -s;
  }
  // ---- constraints (WeightedWbc.cpp:68-71): EoM (16 eq) + swing force = 0 (3 per swing contact) + torque limits (20)
  //      + friction pyramid (5 per stance contact) + 3 zero rows per swing contact
  const int n_sw = 4 - nc;
  const int r_sw = 16, r_tq = 16 + 3 * n_sw, r_fr = r_tq + 20, r_zero = r_fr + 5 * nc, m = r_zero + 3 * n_sw;
  for (int idx = lane; idx < m * NWBC; idx += 32) A[idx] = 0.0;
  __syncwarp();
  for (int idx = lane; idx < 16 * NWBC; idx += 32) {
    const int i = idx / NWBC, j = idx - i * NWBC;
    double a;
    if (j < NQ) a = sh.M[i * 16 + j];
    else if (j < NQ + 12) a = -sh.J[(j - NQ) * 16 + i];
    else a = (i >= 6 && j - NQ - 12 == i - 6) ? -1.0 : 0.0;
    A[idx] = a;
  }
  for (int i = lane; i < 16; i += 32) { lbA[i] = -sh.nle[i]; ubA[i] = -sh.nle[i]; }
  if (lane == 0) {
    int r = r_sw;
    for (int c = 0; c < 4; ++c) if (!fl[c]) for (int a = 0; a < 3; ++a) { A[r * NWBC + NQ + 3 * c + a] = 1.0; lbA[r] = 0.0; ubA[r] = 0.0; ++r; }
    for (int sgn = 0; sgn < 2; ++sgn) for (int j = 0; j < NJ; ++j) {
      A[r * NWBC + NQ + 12 + j] = sgn == 0 ? 1.0 : -1.0; lbA[r] = -QP_INFTY; ubA[r] = ws.torque_limits[j % 5]; ++r;
    }
    const double mu = ws.friction_coefficient;
    const double pyr[5][3] = {{0, 0, -1}, {1, 0, -mu}, {-1, 0, -mu}, {0, 1, -mu}, {0, -1, -mu}};
    for (int c = 0; c < 4; ++c) if (fl[c]) for (int k = 0; k < 5; ++k) {
      for (int a = 0; a < 3; ++a) A[r * NWBC + NQ + 3 * c + a] = pyr[k][a];
      lbA[r] = -QP_INFTY; ubA[r] = 0.0; ++r;
    }
    for (int k = 0; k < 3 * n_sw; ++k) { lbA[r] = -QP_INFTY; ubA[r] = 0.0; ++r; }
  }
  __syncwarp();
  return m;
}

// Reduced WeightedWbc QP for the fused path: tau = M_j qdd - J_j' F + nle_j and F_swing = 0 are substituted, leaving
//   z = [qdd(16), F_stance(3 n_st)],  6 equalities (base rows of the EoM), 10 two-sided torque rows, 5 friction rows per
// stance contact. The Tikhonov term rho ||[qdd, F, tau]||^2 of the full problem is carried over exactly (rho I + rho T'T).
// Hz is written into `Hw` as its packed lower triangle (tri_row; Hz is exactly symmetric: entry (i, j) and (j, i) are the same products
// summed in the same order), rows of Az have stride nz. Returns nz; m_out = number of rows.
__device__ inline int wbc_reduced_build(const WbcShared& sh, int mode, int nw, bool stance_mode, double rho, const hb_wbc_settings& ws, const double* __restrict__ u_des,
                                        double* Hw, double* gz, double* Az, double* lbz, double* ubz, int* stcol /*12*/, int& m_out) {
  const int lane = lane_id();
  int nst = 0;
  for (int j = 0; j < 12; ++j) if (contact_flag(mode, j / 3)) { if (lane == 0) stcol[nst] = j; ++nst; }
  const int nz = NQ + nst;
  const int nc = nst / 3;
  const int m = 6 + NJ + 5 * nc;
  __syncwarp();
  // rows: 6 base EoM equalities, 10 torque rows T = [M_j, -J_j,st'], 5 friction rows per stance contact
  for (int idx = lane; idx < m * nz; idx += 32) {
    const int r = idx / nz, c = idx - r * nz;
    double v = 0.0;
    if (r < 6 + NJ) v = (c < NQ) ? sh.M[r * 16 + c] : -sh.J[stcol[c - NQ] * 16 + r];
    else {
      const int fr = r - 6 - NJ, ci = fr / 5, k = fr - 5 * ci;     // stance contact ci occupies columns NQ+3ci .. NQ+3ci+2
      const int cc = c - NQ - 3 * ci;
      if (cc >= 0 && cc < 3) {
        const double mu = ws.friction_coefficient;
        const double pyr[5][3] = {{0, 0, -1}, {1, 0, -mu}, {-1, 0, -mu}, {0, 1, -mu}, {0, -1, -mu}};
        v = pyr[k][cc];
      }
    }
    Az[idx] = v;
  }
  for (int r = lane; r < m; r += 32) {
    if (r < 6) { lbz[r] = -sh.nle[r]; ubz[r] = -sh.nle[r]; }
    else if (r < 6 + NJ) { const int j = r - 6; lbz[r] = -ws.torque_limits[j % 5] - sh.nle[6 + j]; ubz[r] = ws.torque_limits[j % 5] - sh.nle[6 + j]; }
    else { lbz[r] = -QP_INFTY; ubz[r] = 0.0; }
  }
  __syncwarp();
  const double* Tm = Az + 6 * nz;   // torque rows double as the map tau = T z + nle_j
  const double wf2 = stance_mode ? 0.0 : ws.weight_contact_force * ws.weight_contact_force;
  for (int idx = lane; idx < nz * nz; idx += 32) {
    const int i = idx / nz, j = idx - i * nz;
    if (j > i) continue;
    double s = (i == j) ? rho : 0.0;
    if (i == j && i >= NQ) s += wf2;                      // contact-force task on the stance forces (swing forces are eliminated at zero)
    if (i < NQ && j < NQ) for (int r = 0; r < nw; ++r) s += sh.Aw[r * 16 + i] * sh.Aw[r * 16 + j];
    double t = 0.0;
    for (int r = 0; r < NJ; ++r) t += Tm[r * nz + i] * Tm[r * nz + j];
    Hw[tri_row(i) + j] = s + rho * t;
  }
  for (int i = lane; i < nz; i += 32) {
    double s = 0.0;
    if (i < NQ) for (int r = 0; r < nw; ++r) s -= sh.Aw[r * 16 + i] * sh.bw[r];
    else s = -wf2 * u_des[stcol[i - NQ]];
    double t = 0.0;
    for (int r = 0; r < NJ; ++r) t += Tm[r * nz + i] * sh.nle[6 + r];
    gz[i] = s + rho * t;
  }
  __syncwarp();
  m_out = m;
  return nz;
}

}  // namespace hb

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
constexpr int QP_STRIDE_H = NWBC * NWBC, QP_STRIDE_A = WBC_ROWS * NWBC;

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

// torque law (LeggedController.cpp:181-184): feed-forward joint torques = tail(10) of the WBC solution
__global__ void torque_kernel(int B, const double* sol, double* torque) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < B * NJ) { const int i = idx / NJ, j = idx - i * NJ; torque[idx] = sol[(size_t)i * NWBC + 28 + j]; }
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
}  // namespace
