// K5: WeightedWbc problem assembly on the device (legged_wbc/src/WbcBase.cpp:54-338, WeightedWbc.cpp:18-94),
// one warp per instance. Lane-level parallelism (see hb_rbd.cuh; the measured q, v are its rbd_to_qv):
//   pass A  lanes 0-15: unit velocities at the measured q -> contact Jacobian columns J_c (12x16)
//           lanes 16-31: unit velocities at the planned q -> centroidal momentum matrix columns A(q_des) (6x16)
//   pass B  lane 0: dual pass at (q_meas; direction v_meas)  -> p_c, v_c, dJ_c/dt v   (WbcBase.cpp:91-109)
//           lane 1: dual pass at (q_des;  direction v_des)   -> p_c, v_c, dA/dt v      (WbcBase.cpp:119-136)
//   pass C  lanes 0-15: RNEA with unit accelerations -> M(q) columns (CRBA, WbcBase.cpp:88-89); lane 16: nle (WbcBase.cpp:90)
// Each WbcBase::formulate*Task (WbcBase.cpp:138-338) is written once, here: wbc_terms_warp (the terms above and the motion tasks on qdd at
// unit weight), wbc_task0_eq, wbc_task0_ineq, wbc_task12_rows; wbc_rows counts their rows. WeightedWbc weights the motion tasks
// (wbc_weight_rows) and writes its QP in the reference's own layout (qpOASES row-major, WeightedWbc.cpp:27-41) or the reduced QP of the
// fused path (wbc_reduced_build); HierarchicalWbc stacks the unweighted tasks by priority (hb_hoqp.cuh).
#pragma once
#include "hb_common.cuh"
#include "hb_planner.h"
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
  double At[18 * 16];   // motion task rows acting on qdd (swing: <=12, base: 6), at unit weight until wbc_weight_rows
  double bt[18];
  double misc[32];
  double frame[36];     // WBC maps: contact c's surface frame n, t1, t2 at frame[9c ..]; n_z = 0 marks flat ground (wbc_contact_frames)
};

// row counts of the tasks for one contact mode
struct WbcRows {
  int nc, nsw;   // stance and swing contacts
  int eq;        // task0 equalities the weighted QP keeps: EoM (16), zero force of each swing contact (3 nsw)
  int md0;       // task0 inequalities: torque limits (20), friction pyramid of each stance contact (5 nc)
  int nt;        // motion task rows in At, bt: swing legs (3 nsw) and base acceleration (6); 6 in stance mode
  int ma2;       // hierarchical task2: contact forces (12), swing legs (3 nsw)
  int m;         // weighted QP constraints: eq + md0 + 3 nsw zero rows
};
__device__ inline WbcRows wbc_rows(int mode, bool stance_mode) {
  int nc = 0;
  for (int c = 0; c < 4; ++c) nc += contact_flag(mode, c);
  const int nsw = 4 - nc, eq = 16 + 3 * nsw, md0 = 2 * NJ + 5 * nc;
  return {nc, nsw, eq, md0, stance_mode ? 6 : 3 * nsw + 6, 12 + 3 * nsw, eq + md0 + 3 * nsw};
}
// task0 equalities of the hierarchical formulation: EoM (16), zero force or no motion of each contact (3 x 4)
constexpr int WBC_MA0 = 28;

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

// The surface frame (n, t1, t2) of each contact on WBC map m (WBC maps, hunter_b200.h; hbplan::map_frame), lane c < 4 for contact c at its
// measured position sh.pos_m. Where the ground is flat the contact keeps the flat rows: its n_z is written 0, which no frame has
// (n_z = 1 / L > 0).
__device__ inline void wbc_contact_frames(const hb_terrain& m, WbcShared& sh) {
  const int c = lane_id();
  if (c >= 4) return;
  double* f = sh.frame + 9 * c;
  if (!hbplan::map_frame(m, sh.pos_m[3 * c], sh.pos_m[3 * c + 1], f)) f[2] = 0.0;
}

// The surface frames the friction rows of instance `inst` read (wbc_task0_ineq): sh.frame when the instance has a WBC map, null (flat
// rows) otherwise
__device__ __forceinline__ const double* wbc_frames(const InstanceView<hb_terrain>& maps, int inst, const WbcShared& sh) {
  return maps.of(inst) ? sh.frame : nullptr;
}

// The WBC terms of one instance in sh, and the motion task rows at unit weight in sh.At, sh.bt: formulateSwingLegTask (3 rows per swing
// contact, in contact order), then formulateBaseAccelTask (6); in stance mode formulateStanceBaseAccelTask (6 identity rows, b = 0).
// Returns the number of task rows. stance_mode is read where it is used (wbc_fused_kernel passes its shared copy: held in a register
// across the passes, it spilled). maps: the WBC maps (the kernels' __grid_constant__ parameter); with a map, instance inst's contact
// frames go to sh.frame after pass C.
__device__ inline int wbc_terms_warp(const double* __restrict__ x_des, const double* __restrict__ u_des, const double* __restrict__ rbd,
                                     int mode, const bool& stance_mode, const hb_wbc_settings& ws, const InstanceView<hb_terrain>& maps, int inst,
                                     WbcShared& sh) {
  const int lane = lane_id();
  const Model& md = c_model;
  // ---- measured q, v (WbcBase.cpp:72-79)
  if (lane == 0) {
    rbd_to_qv(rbd, sh.q, sh.v);
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
  // ---- contact frames on the WBC map (pass B's measured contact positions)
  if (const hb_terrain* m = maps.of(inst)) wbc_contact_frames(*m, sh);
  // symmetrise M (WbcBase.cpp:88-89 copies the upper triangle; numerically the same matrix)
  for (int idx = lane; idx < 256; idx += 32) {
    const int i = idx >> 4, j = idx & 15;
    if (j < i) { const double a = 0.5 * (sh.M[i * 16 + j] + sh.M[j * 16 + i]); sh.M[i * 16 + j] = a; }
  }
  __syncwarp();
  for (int idx = lane; idx < 256; idx += 32) { const int i = idx >> 4, j = idx & 15; if (j > i) sh.M[i * 16 + j] = sh.M[j * 16 + i]; }
  __syncwarp();
  // ---- desired base kinematics (computeBaseKinematicsFromCentroidalModel, WbcBase.cpp:134-135) and task rows
  if (lane == 0) {
    bool fl[4];   // contact flags before the rows: contact_flag in the loop condition changes how the base rows below are contracted
    for (int c = 0; c < 4; ++c) fl[c] = contact_flag(mode, c);
    for (int i = 0; i < 18 * 16; ++i) sh.At[i] = 0.0;
    if (stance_mode) {
      for (int i = 0; i < 6; ++i) { sh.At[i * 16 + i] = 1.0; sh.bt[i] = 0.0; }
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
      // swing leg task (WbcBase.cpp:297-323)
      for (int c = 0; c < 4; ++c) if (!fl[c]) for (int a = 0; a < 3; ++a) {
        const double acc = ws.swing_kp * (sh.pos_d[3 * c + a] - sh.pos_m[3 * c + a]) + ws.swing_kd * (sh.vel_d[3 * c + a] - sh.vel_m[3 * c + a]);
        for (int j = 0; j < NQ; ++j) sh.At[r * 16 + j] = sh.J[(3 * c + a) * 16 + j];
        sh.bt[r] = acc - sh.dJv[3 * c + a];
        ++r;
      }
      // base xy acceleration (WbcBase.cpp:228-240)
      for (int a = 0; a < 2; ++a) { sh.At[r * 16 + a] = 1.0; sh.bt[r] = qbdd[a]; ++r; }
      // base height (WbcBase.cpp:243-256)
      sh.At[r * 16 + 2] = 1.0;
      sh.bt[r] = qbdd[2] + ws.base_height_kp * (sh.qd[2] - sh.q[2]) + ws.base_height_kd * (sh.vd[2] - sh.v[2]);
      ++r;
      // base angular motion (WbcBase.cpp:259-290)
      double err[3];
      rotation_error_world(Rd, Rm, err);
      for (int a = 0; a < 3; ++a) {
        for (int i = 0; i < 3; ++i) sh.At[r * 16 + 3 + i] = axm[3 * i + a];
        sh.bt[r] = baseAccW[a] + ws.base_angular_kp * err[a] + ws.base_angular_kd * (baseVelW[a] - wm[a]) - dJw_v[a];
        ++r;
      }
    }
  }
  __syncwarp();
  return wbc_rows(mode, stance_mode).nt;
}

// formulateWeightedTasks (WeightedWbc.cpp:73-81): the motion task rows times their weights, in place -- weight_swing_leg on the swing
// rows, weight_base_accel on the base rows. The contact-force task is weighted where its rows are formed.
__device__ inline void wbc_weight_rows(WbcShared& sh, const WbcRows& n, bool stance_mode, const hb_wbc_settings& ws) {
  const int lane = lane_id(), nsr = stance_mode ? 0 : 3 * n.nsw;
  for (int idx = lane; idx < n.nt * 16; idx += 32) sh.At[idx] *= (idx >> 4) < nsr ? ws.weight_swing_leg : ws.weight_base_accel;
  for (int r = lane; r < n.nt; r += 32) sh.bt[r] *= r < nsr ? ws.weight_swing_leg : ws.weight_base_accel;
  __syncwarp();
}

// The WBC settings instance `inst` runs: its controller setting's (hb_rollout_set_controller_settings) when the view has one, the context's
// `ws` otherwise. Lane 0 stages them in `dst`, shared memory of the warp, which every lane reads after the call.
__device__ inline const hb_wbc_settings& wbc_select_settings(const hb_wbc_settings& ws, InstanceView<hb_controller_setting> cs, int inst,
                                                             hb_wbc_settings& dst) {
  if (lane_id() == 0) {
    const hb_controller_setting* c = cs.of(inst);
    if (c) dst = c->wbc;
    else dst = ws;
  }
  __syncwarp();
  return dst;
}

// ---- the tasks on the decision vector [qdd(16), F(12), tau(10)], rows of NWBC columns at leading dimension lda. Rows of task0 after the
// 16 EoM rows come per contact in contact order: the swing contacts' first, then the stance contacts'.
// the k-th contact (contact order) whose contact flag is `stance`
__device__ inline int wbc_nth_contact(int mode, bool stance, int k) {
  int c = 0;
  for (; c < 3; ++c) if (contact_flag(mode, c) == stance && k-- == 0) break;
  return c;
}

// task0 equality rows 0 .. rows-1 (rows <= WBC_MA0): formulateFloatingBaseEomTask [M | -J' | -S'] x = -nle (16 rows), zero force of each
// swing contact (3 nsw), formulateNoContactMotionTask J_c qdd = -dJ_c v of each stance contact (3 nc). WeightedWbc keeps the first n.eq.
__device__ inline void wbc_task0_eq(const WbcShared& sh, int mode, const WbcRows& n, int rows, double* A, int lda, double* b) {
  const int lane = lane_id(), nsw = n.nsw;
  for (int idx = lane; idx < rows * NWBC; idx += 32) {
    const int i = idx / NWBC, j = idx - i * NWBC;
    double a = 0.0;
    if (i < 16) {
      if (j < NQ) a = sh.M[i * 16 + j];
      else if (j < NQ + 12) a = -sh.J[(j - NQ) * 16 + i];
      else a = (i >= 6 && j - NQ - 12 == i - 6) ? -1.0 : 0.0;
    } else if (i < 16 + 3 * nsw) {
      const int k = i - 16, c = wbc_nth_contact(mode, false, k / 3);
      a = (j == NQ + 3 * c + k % 3) ? 1.0 : 0.0;
    } else {
      const int k = i - 16 - 3 * nsw, c = wbc_nth_contact(mode, true, k / 3);
      a = j < NQ ? sh.J[(3 * c + k % 3) * 16 + j] : 0.0;
    }
    A[i * lda + j] = a;
  }
  for (int i = lane; i < rows; i += 32) {
    double v = 0.0;
    if (i < 16) v = -sh.nle[i];
    else if (i >= 16 + 3 * nsw) { const int k = i - 16 - 3 * nsw; v = -sh.dJv[3 * wbc_nth_contact(mode, true, k / 3) + k % 3]; }
    b[i] = v;
  }
}

// task0 inequality row q (formulateTorqueLimitsTask: 20 rows, then formulateFrictionConeTask: 5 pyramid rows per stance contact): its
// nonzeros are coef[0 .. len) from column col0; returns its bound f. frames (nullable: flat): the contacts' surface frames on a WBC map
// (WbcShared::frame); a contact with a frame gets the pyramid about its normal, -n, +-t1 - mu n, +-t2 - mu n.
__device__ inline double wbc_task0_ineq(const hb_wbc_settings& ws, int mode, int q, int& col0, int& len, double* coef, const double* frames) {
  if (q < 2 * NJ) {
    const int j = q % NJ;
    col0 = NQ + 12 + j; len = 1; coef[0] = q < NJ ? 1.0 : -1.0; coef[1] = 0.0; coef[2] = 0.0;
    return ws.torque_limits[j % 5];
  }
  const int fr = q - 2 * NJ, k = fr % 5;
  const double mu = ws.friction_coefficient;   // pyramid rows {0,0,-1}, {1,0,-mu}, {-1,0,-mu}, {0,1,-mu}, {0,-1,-mu}
  const int c = wbc_nth_contact(mode, true, fr / 5);
  col0 = NQ + 3 * c; len = 3;
  const double* f = frames ? frames + 9 * c : nullptr;
  if (f && f[2] != 0.0) {
    const double* t = f + (k < 3 ? 3 : 6);
    for (int a = 0; a < 3; ++a) coef[a] = k == 0 ? -f[a] : (k & 1 ? t[a] : -t[a]) - hbplan::mul_rn(mu, f[a]);
    return 0.0;
  }
  coef[0] = k == 1 ? 1.0 : (k == 2 ? -1.0 : 0.0);
  coef[1] = k == 3 ? 1.0 : (k == 4 ? -1.0 : 0.0);
  coef[2] = k == 0 ? -1.0 : -mu;
  return 0.0;
}

// HierarchicalWbc's task1 (lvl 1): the 6 base-acceleration rows; task2 (lvl 2): 0.1 * (F = F_des), then the 3 rows of each swing contact.
// The motion rows are the unit-weight rows At, bt (stride 16) of wbc_terms_warp. Returns the number of rows.
__device__ inline int wbc_task12_rows(int lvl, const double* At, const double* bt, const WbcRows& n, const double* u_des, double* A, int lda, double* b) {
  const int lane = lane_id(), nswr = 3 * n.nsw;
  const int ma = lvl == 1 ? 6 : n.ma2;
  for (int idx = lane; idx < ma * NWBC; idx += 32) {
    const int i = idx / NWBC, j = idx - i * NWBC;
    double a = 0.0;
    if (lvl == 1) { if (j < NQ) a = At[(nswr + i) * 16 + j]; }
    else if (i < 12) a = (j == NQ + i) ? 0.1 : 0.0;
    else if (j < NQ) a = At[(i - 12) * 16 + j];
    A[i * lda + j] = a;
  }
  for (int i = lane; i < ma; i += 32) b[i] = lvl == 1 ? bt[nswr + i] : (i < 12 ? 0.1 * u_des[i] : bt[i - 12]);
  return ma;
}

// Reduced WeightedWbc QP for the fused path: tau = M_j qdd - J_j' F + nle_j and F_swing = 0 are substituted, leaving
//   z = [qdd(16), F_stance(3 n_st)],  6 equalities (base rows of the EoM), 10 two-sided torque rows, 5 friction rows per
// stance contact (their limits and pyramid coefficients from wbc_task0_ineq). The Tikhonov term rho ||[qdd, F, tau]||^2 of the full
// problem is carried over exactly (rho I + rho T'T).
// Hz is written into `Hw` as its packed lower triangle (tri_row; Hz is exactly symmetric: entry (i, j) and (j, i) are the same products
// summed in the same order), rows of Az have stride nz. Returns nz; m_out = number of rows. frames: as wbc_task0_ineq's.
__device__ inline int wbc_reduced_build(const WbcShared& sh, const WbcRows& n, int mode, bool stance_mode, double rho, const hb_wbc_settings& ws,
                                        const double* frames, const double* __restrict__ u_des, double* Hw, double* gz, double* Az, double* lbz,
                                        double* ubz, int* stcol /*12*/, int& m_out) {
  const int lane = lane_id();
  if (lane == 0) for (int j = 0, k = 0; j < 12; ++j) if (contact_flag(mode, j / 3)) stcol[k++] = j;
  const int nz = NQ + 3 * n.nc, m = 6 + NJ + 5 * n.nc, nw = n.nt;
  __syncwarp();
  // rows: 6 base EoM equalities, 10 torque rows T = [M_j, -J_j,st'], 5 friction rows per stance contact
  for (int idx = lane; idx < m * nz; idx += 32) {
    const int r = idx / nz, c = idx - r * nz;
    double v = 0.0;
    if (r < 6 + NJ) v = (c < NQ) ? sh.M[r * 16 + c] : -sh.J[stcol[c - NQ] * 16 + r];
    else {
      const int fr = r - 6 - NJ, ci = fr / 5;     // stance contact ci occupies columns NQ+3ci .. NQ+3ci+2
      const int cc = c - NQ - 3 * ci;
      if (cc >= 0 && cc < 3) { int c0, len; double coef[3]; wbc_task0_ineq(ws, mode, 2 * NJ + fr, c0, len, coef, frames); v = coef[cc]; }
    }
    Az[idx] = v;
  }
  for (int r = lane; r < m; r += 32) {
    int c0, len; double coef[3];
    if (r < 6) { lbz[r] = -sh.nle[r]; ubz[r] = -sh.nle[r]; }
    else if (r < 6 + NJ) { const int j = r - 6; const double lim = wbc_task0_ineq(ws, mode, j, c0, len, coef, nullptr); lbz[r] = -lim - sh.nle[6 + j]; ubz[r] = lim - sh.nle[6 + j]; }
    else { lbz[r] = -QP_INFTY; ubz[r] = wbc_task0_ineq(ws, mode, NJ + r - 6, c0, len, coef, frames); }
  }
  __syncwarp();
  const double* Tm = Az + 6 * nz;   // torque rows double as the map tau = T z + nle_j
  const double wf2 = stance_mode ? 0.0 : ws.weight_contact_force * ws.weight_contact_force;
  for (int idx = lane; idx < nz * nz; idx += 32) {
    const int i = idx / nz, j = idx - i * nz;
    if (j > i) continue;
    double s = (i == j) ? rho : 0.0;
    if (i == j && i >= NQ) s += wf2;                      // contact-force task on the stance forces (swing forces are eliminated at zero)
    if (i < NQ && j < NQ) for (int r = 0; r < nw; ++r) s += sh.At[r * 16 + i] * sh.At[r * 16 + j];
    double t = 0.0;
    for (int r = 0; r < NJ; ++r) t += Tm[r * nz + i] * Tm[r * nz + j];
    Hw[tri_row(i) + j] = s + rho * t;
  }
  for (int i = lane; i < nz; i += 32) {
    double s = 0.0;
    if (i < NQ) for (int r = 0; r < nw; ++r) s -= sh.At[r * 16 + i] * sh.bt[r];
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

__global__ void wbc_assemble_kernel(int B, hb_wbc_settings ws, const __grid_constant__ InstanceView<hb_terrain> maps, const double* x_des,
                                    const double* u_des, const double* rbd, const int32_t* mode, const uint8_t* stance_mode, double* H, double* g,
                                    double* A, double* lbA, double* ubA, int32_t* m_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int inst = blockIdx.x * wpb + warp;
  if (inst >= B) return;
  WbcShared& sh = reinterpret_cast<WbcShared*>(smem_raw)[warp];
  const int md = mode[inst];
  const bool stance = stance_mode ? stance_mode[inst] != 0 : false;
  const double* ud = u_des + (size_t)inst * NU;
  wbc_terms_warp(x_des + (size_t)inst * NX, ud, rbd + (size_t)inst * 32, md, stance, ws, maps, inst, sh);
  const WbcRows n = wbc_rows(md, stance);
  wbc_weight_rows(sh, n, stance, ws);
  const int lane = lane_id();
  H += (size_t)inst * QP_STRIDE_H; g += (size_t)inst * NWBC; A += (size_t)inst * QP_STRIDE_A; lbA += (size_t)inst * WBC_ROWS; ubA += (size_t)inst * WBC_ROWS;
  // H = At'At, g = -At'bt (WeightedWbc.cpp:38-41) on the qdd block, plus formulateContactForceTask * weightContactForce (WbcBase.cpp:325-338,
  // not in stance mode): rows w_f [0 | I_12 | 0] x = w_f F_des
  const double wf2 = stance ? 0.0 : ws.weight_contact_force * ws.weight_contact_force;
  for (int idx = lane; idx < NWBC * NWBC; idx += 32) {
    const int i = idx / NWBC, j = idx - i * NWBC;
    double s = 0.0;
    if (i < NQ && j < NQ) for (int r = 0; r < n.nt; ++r) s += sh.At[r * 16 + i] * sh.At[r * 16 + j];
    if (i == j && i >= NQ && i < NQ + 12) s += wf2;
    H[idx] = s;
  }
  for (int i = lane; i < NWBC; i += 32) {
    double s = 0.0;
    if (i < NQ) for (int r = 0; r < n.nt; ++r) s += sh.At[r * 16 + i] * sh.bt[r];
    else if (i < NQ + 12) s = wf2 * ud[i - NQ];
    g[i] = -s;
  }
  // constraints (WeightedWbc.cpp:68-71): the n.eq task0 equalities (lbA = ubA = b), every task0 inequality (lbA = -inf, ubA = f), 3 zero
  // rows per swing contact
  for (int idx = lane; idx < n.m * NWBC; idx += 32) A[idx] = 0.0;
  __syncwarp();
  wbc_task0_eq(sh, md, n, n.eq, A, NWBC, lbA);
  for (int q = lane; q < n.md0; q += 32) {
    int c0, len; double coef[3];
    const int r = n.eq + q;
    ubA[r] = wbc_task0_ineq(ws, md, q, c0, len, coef, wbc_frames(maps, inst, sh));
    lbA[r] = -QP_INFTY;
    for (int k = 0; k < len; ++k) A[r * NWBC + c0 + k] = coef[k];
  }
  for (int r = n.eq + n.md0 + lane; r < n.m; r += 32) { lbA[r] = -QP_INFTY; ubA[r] = 0.0; }
  __syncwarp();
  for (int i = lane; i < n.eq; i += 32) ubA[i] = lbA[i];
  if (lane == 0) m_out[inst] = n.m;
}

// Fused WeightedWbc step (K5+K6): assembly terms, reduced QP (tau and swing forces eliminated), interior point, expansion to
// the reference's 38-vector [qdd, F, tau]. Shared memory per warp: QP workspace for n<=28 with the Hessian as a packed triangle (the
// assembly scratch aliases the factorisation area, which is dead until the first Newton step) + the reduced constraint matrix.
constexpr int WZ_N = 28, WZ_ME = 6, WZ_MI = 40, WZ_ROWS = 36;
__host__ __device__ constexpr size_t wbc_fused_doubles() { return qp_workspace_doubles(WZ_N, WZ_ME, WZ_MI, true) + WZ_ROWS * WZ_N + 2 * WZ_ROWS + 3 * WZ_N + 16 + 8; }
// One warp per block and one block per instance: 8 blocks per SM put a 1024-instance batch in one wave on 132 SMs (8 x 132 >= 1024;
// at 7 a tail wave of 100 blocks costs almost as much as the full one). The runtime reserves 1 KB of shared memory per block.
static_assert(8 * (wbc_fused_doubles() * sizeof(double) + 1024) <= 228 * 1024, "wbc_fused_kernel must fit 8 blocks per SM");

// The assembly scratch and the WBC settings the warp's instance runs (wbc_select_settings), aliased over the QP's factorisation area
struct WbcStaged { WbcShared sh; hb_wbc_settings ws; bool stance; };

__global__ void __launch_bounds__(32, 8) wbc_fused_kernel(int B, hb_wbc_settings ws_ctx, InstanceView<hb_controller_setting> cs,
                                 const __grid_constant__ InstanceView<hb_terrain> maps, const double* x_des, const double* u_des, const double* rbd,
                                 const int32_t* mode, const uint8_t* stance_mode, double rho, int max_iter, double* sol, int32_t* status, int32_t* iters) {
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
  static_assert(sizeof(WbcStaged) <= sizeof(double) * (WZ_N * 29 + WZ_N * 7 + WZ_ME * 7 + WZ_N + WZ_ME + 6 * WZ_N + 5 * WZ_ME + 8 * WZ_MI), "assembly scratch must fit in the aliased area");
  WbcStaged& stg = *reinterpret_cast<WbcStaged*>(w.K);   // K, V, S, vectors: dead until the QP starts
  WbcShared& sh = stg.sh;
  if (lane == 0) stg.stance = stance_mode ? stance_mode[inst] != 0 : false;
  const hb_wbc_settings& ws = wbc_select_settings(ws_ctx, cs, inst, stg.ws);
  const int md = mode[inst];
  wbc_terms_warp(x_des + (size_t)inst * NX, u_des + (size_t)inst * NU, rbd + (size_t)inst * 32, md, stg.stance, ws, maps, inst, sh);
  const bool stance = stg.stance;
  const WbcRows n = wbc_rows(md, stance);
  wbc_weight_rows(sh, n, stance, ws);
  int m = 0;
  // the frames are read here, before the QP takes over the aliased area
  const int nz = wbc_reduced_build(sh, n, md, stance, rho, ws, wbc_frames(maps, inst, sh), u_des + (size_t)inst * NU, w.H, gz, Az, lbz, ubz, stcol, m);
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
