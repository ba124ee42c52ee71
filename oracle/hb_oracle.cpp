// ORACLE (test infrastructure only) -- see hb_oracle.hpp for the scope statement. PARITY UNPINNED for solver rows.
#include "hb_oracle.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <thread>
#include <vector>

#include "hb_rbd.hpp"

using namespace hbo;

namespace {

constexpr int NX = HB_NX, NU = HB_NU, NQ = HB_NQ, NJ = HB_NJ, NC = HB_NC;
constexpr int ND = NX + NU;  // tangent directions of the brute-force AD
using D44 = Dual<ND>;

double g_R[NU * NU];
bool g_init = false;
// WBC gains / limits / weights: the shipped task.info values unless a test overrides them (hbo_set_wbc_settings), mirroring what
// WbcBase::loadTasksSetting / WeightedWbc::loadTasksSetting / setKpKd make configurable at run time
struct WbcSettings { double torque[5], mu, swing_kp, swing_kd, accel_kp, accel_kd, height_kp, height_kd, angular_kp, angular_kd, weight_swing, weight_base, weight_force; };
WbcSettings g_wbc = {{HB_WBC_TORQUE_LIMITS[0], HB_WBC_TORQUE_LIMITS[1], HB_WBC_TORQUE_LIMITS[2], HB_WBC_TORQUE_LIMITS[3], HB_WBC_TORQUE_LIMITS[4]},
                     HB_WBC_FRICTION_MU, HB_WBC_SWING_KP, HB_WBC_SWING_KD, 40.0, 4.0, HB_WBC_BASE_HEIGHT_KP, HB_WBC_BASE_HEIGHT_KD, HB_WBC_BASE_ANGULAR_KP,
                     HB_WBC_BASE_ANGULAR_KD, HB_WBC_WEIGHT_SWING, HB_WBC_WEIGHT_BASE, HB_WBC_WEIGHT_FORCE};

// MotionPhaseDefinition.h:55-87
inline void mode_to_flags(int mode, bool* f) {
  f[0] = f[2] = (mode == 2 || mode == 3);
  f[1] = f[3] = (mode == 1 || mode == 3);
}

// ---------------------------------------------------------------- centroidal flow map (M1, App. C.2)
// x = [h/m (6), q (16)], u = [F (12), qj_dot (10)]
template <class T>
void flow_map_T(const T* x, const T* u, T* f, T* epos, T* evel, T* vgen_out = nullptr) {
  Kin<T> kin;
  forward_kinematics(x + 6, kin);
  T com[3];
  center_of_mass(kin, com);
  // momentum carried by the joint velocities: A_j * qj_dot
  T vg[NQ];
  for (int i = 0; i < 6; ++i) vg[i] = T(0.0);
  for (int j = 0; j < NJ; ++j) vg[6 + j] = u[12 + j];
  Vel<T> vel;
  velocities(kin, vg, vel);
  T hj[6];
  centroidal_momentum(kin, vel, com, hj);
  // base block A_b (6 columns)
  T Ab[6 * NQ];
  for (int c = 0; c < 6; ++c) {
    T e[NQ];
    for (int i = 0; i < NQ; ++i) e[i] = T(i == c ? 1.0 : 0.0);
    Vel<T> ve;
    velocities(kin, e, ve);
    T h[6];
    centroidal_momentum(kin, ve, com, h);
    for (int r = 0; r < 6; ++r) Ab[r * NQ + c] = h[r];
  }
  T rhs[6], vb[6];
  for (int i = 0; i < 6; ++i) rhs[i] = x[i] * HB_TOTAL_MASS - hj[i];
  solve6(Ab, rhs, vb);  // mapping_.getPinocchioJointVelocity (WbcBase.cpp:130)
  for (int i = 0; i < 6; ++i) vg[i] = vb[i];
  velocities(kin, vg, vel);
  T r[NC][3];
  for (int c = 0; c < NC; ++c) {
    contact_position(kin, c, r[c]);
    if (epos) for (int i = 0; i < 3; ++i) epos[3 * c + i] = r[c][i];
    if (evel) contact_velocity(kin, vel, c, evel + 3 * c);
  }
  // normalised centroidal momentum rate (getNormalizedCentroidalMomentumRate, call site WbcBase.cpp:134)
  for (int i = 0; i < 6; ++i) f[i] = T(0.0);
  for (int c = 0; c < NC; ++c) {
    T rc[3], l[3];
    for (int i = 0; i < 3; ++i) rc[i] = r[c][i] - com[i];
    cross3(rc, u + 3 * c, l);
    for (int i = 0; i < 3; ++i) { f[i] += u[3 * c + i] * (1.0 / HB_TOTAL_MASS); f[3 + i] += l[i] * (1.0 / HB_TOTAL_MASS); }
  }
  f[2] = f[2] - HB_GRAVITY;
  for (int i = 0; i < 6; ++i) f[6 + i] = vb[i];
  for (int j = 0; j < NJ; ++j) f[12 + j] = u[12 + j];
  if (vgen_out) for (int i = 0; i < NQ; ++i) vgen_out[i] = vg[i];
}

struct FlowLin {
  double f[NX], A[NX * NX], B[NX * NU];
  double epos[12], evel[12], dpos_dx[12 * NX], dvel_dx[12 * NX], dvel_du[12 * NU];
};

void flow_map_lin(const double* x, const double* u, FlowLin& o) {
  D44 xd[NX], ud[NU], fd[NX], ep[12], ev[12];
  for (int i = 0; i < NX; ++i) xd[i] = D44::seed(x[i], i);
  for (int i = 0; i < NU; ++i) ud[i] = D44::seed(u[i], NX + i);
  flow_map_T<D44>(xd, ud, fd, ep, ev);
  for (int i = 0; i < NX; ++i) {
    o.f[i] = fd[i].v;
    for (int j = 0; j < NX; ++j) o.A[i * NX + j] = fd[i].d[j];
    for (int j = 0; j < NU; ++j) o.B[i * NU + j] = fd[i].d[NX + j];
  }
  for (int i = 0; i < 12; ++i) {
    o.epos[i] = ep[i].v; o.evel[i] = ev[i].v;
    for (int j = 0; j < NX; ++j) { o.dpos_dx[i * NX + j] = ep[i].d[j]; o.dvel_dx[i * NX + j] = ev[i].d[j]; }
    for (int j = 0; j < NU; ++j) o.dvel_du[i * NU + j] = ev[i].d[NX + j];
  }
}

// ---------------------------------------------------------------- penalties (App. C.4; relaxedBarrierPenaltyVis.py:15-19)
struct Pen { double v, d1, d2; };
inline Pen relaxed_barrier(double h, double mu, double delta) {
  Pen p;
  if (h > delta) { p.v = -mu * std::log(h); p.d1 = -mu / h; p.d2 = mu / (h * h); }
  else {
    double z = (h - 2.0 * delta) / delta;
    p.v = mu * (-std::log(delta) + 0.5 * z * z - 0.5);
    p.d1 = mu * (h - 2.0 * delta) / (delta * delta);
    p.d2 = mu / (delta * delta);
  }
  return p;
}
// DoubleSidedPenalty: p(h-lo) + p(hi-h)  (LeggedInterface.cpp:340-353)
inline Pen double_sided(double h, double lo, double hi, double mu, double delta) {
  Pen a = relaxed_barrier(h - lo, mu, delta), b = relaxed_barrier(hi - h, mu, delta);
  return {a.v + b.v, a.d1 - b.d1, a.d2 + b.d2};
}

// weightCompensatingInput (common/utils.h:75-93)
void weight_compensating_input(int mode, double* u) {
  bool fl[4]; mode_to_flags(mode, fl);
  int n = fl[0] + fl[1] + fl[2] + fl[3];
  for (int i = 0; i < NU; ++i) u[i] = 0.0;
  if (n > 0) for (int c = 0; c < NC; ++c) if (fl[c]) u[3 * c + 2] = HB_TOTAL_MASS * HB_GRAVITY / n;
}

struct NodeLQ {
  double Ad[NX * NX], Bd[NX * NU], b[NX];
  double Q[NX * NX], R[NU * NU], P[NU * NX], q[NX], r[NU];
  double C[16 * NX], D[16 * NU], e[16];
  int m;
  double cost;  // unscaled stage cost
};

// Stage cost and state-input equality constraints at (x,u). If lin != nullptr also their LQ model.
// epos/evel and Jacobians come from the flow-map evaluation at the same point.
void node_cost_constraints(const double* x, const double* u, const double* xref, const double* swing, int mode,
                           const double* epos, const double* evel, const FlowLin* lin, NodeLQ& o) {
  bool fl[4]; mode_to_flags(mode, fl);
  const bool L = lin != nullptr;
  if (L) {
    std::fill(o.Q, o.Q + NX * NX, 0.0); std::fill(o.R, o.R + NU * NU, 0.0); std::fill(o.P, o.P + NU * NX, 0.0);
    std::fill(o.q, o.q + NX, 0.0); std::fill(o.r, o.r + NU, 0.0);
    std::fill(o.C, o.C + 16 * NX, 0.0); std::fill(o.D, o.D + 16 * NU, 0.0);
  }
  double cost = 0.0;
  // --- M2 quadratic tracking cost
  double unom[NU]; weight_compensating_input(mode, unom);
  double dx[NX], du[NU];
  for (int i = 0; i < NX; ++i) dx[i] = x[i] - xref[i];
  for (int i = 0; i < NU; ++i) du[i] = u[i] - unom[i];
  for (int i = 0; i < NX; ++i) cost += 0.5 * HB_Q_DIAG[i] * dx[i] * dx[i];
  for (int i = 0; i < NU; ++i) {
    double s = 0.0;
    for (int j = 0; j < NU; ++j) s += g_R[i * NU + j] * du[j];
    cost += 0.5 * du[i] * s;
    if (L) o.r[i] += s;
  }
  if (L) {
    for (int i = 0; i < NX; ++i) { o.Q[i * NX + i] += HB_Q_DIAG[i]; o.q[i] += HB_Q_DIAG[i] * dx[i]; }
    for (int i = 0; i < NU * NU; ++i) o.R[i] += g_R[i];
  }
  // --- M6 friction cone soft constraint on stance contacts (FrictionConeConstraint.cpp:78-233)
  for (int c = 0; c < NC; ++c) {
    if (!fl[c]) continue;
    const double Fx = u[3 * c], Fy = u[3 * c + 1], Fz = u[3 * c + 2];
    const double t2 = Fx * Fx + Fy * Fy + HB_FRICTION_REGULARIZATION, tn = std::sqrt(t2), t32 = tn * t2;
    const double h = HB_FRICTION_MU * Fz - tn;
    Pen p = relaxed_barrier(h, HB_FRICTION_BARRIER_MU, HB_FRICTION_BARRIER_DELTA);
    cost += p.v;
    if (L) {
      const double gr[3] = {-Fx / tn, -Fy / tn, HB_FRICTION_MU};
      double Hh[9] = {-(Fy * Fy + HB_FRICTION_REGULARIZATION) / t32, Fx * Fy / t32, 0, Fx * Fy / t32,
                      -(Fx * Fx + HB_FRICTION_REGULARIZATION) / t32, 0, 0, 0, 0};
      for (int i = 0; i < 3; ++i) {
        o.r[3 * c + i] += p.d1 * gr[i];
        for (int j = 0; j < 3; ++j) o.R[(3 * c + i) * NU + 3 * c + j] += p.d2 * gr[i] * gr[j] + p.d1 * Hh[3 * i + j];
      }
      // hessianDiagonalShift on the full input and state diagonals (FrictionConeConstraint.cpp:218-230)
      for (int i = 0; i < NU; ++i) o.R[i * NU + i] += p.d1 * (-HB_FRICTION_HESSIAN_SHIFT);
      for (int i = 0; i < NX; ++i) o.Q[i * NX + i] += p.d1 * (-HB_FRICTION_HESSIAN_SHIFT);
    }
  }
  // --- M7 xy swing reference soft constraint (XYReferenceConstraintCppAd.cpp:71-98, LeggedRobotPreComputation.cpp:109-119)
  for (int c = 0; c < NC; ++c) {
    if (fl[c]) continue;
    for (int a = 0; a < 2; ++a) {
      const double h = evel[3 * c + a] - swing[6 * c + 3 + a] + HB_XY_POSITION_GAIN * (epos[3 * c + a] - swing[6 * c + a]);
      cost += 0.5 * HB_SOFT_SWING_WEIGHT * h * h;
      if (L) {
        double gx[NX], gu[NU];
        for (int j = 0; j < NX; ++j) gx[j] = lin->dvel_dx[(3 * c + a) * NX + j] + HB_XY_POSITION_GAIN * lin->dpos_dx[(3 * c + a) * NX + j];
        for (int j = 0; j < NU; ++j) gu[j] = lin->dvel_du[(3 * c + a) * NU + j];
        const double w = HB_SOFT_SWING_WEIGHT;
        for (int i = 0; i < NX; ++i) { o.q[i] += w * h * gx[i]; for (int j = 0; j < NX; ++j) o.Q[i * NX + j] += w * gx[i] * gx[j]; }
        for (int i = 0; i < NU; ++i) {
          o.r[i] += w * h * gu[i];
          for (int j = 0; j < NU; ++j) o.R[i * NU + j] += w * gu[i] * gu[j];
          for (int j = 0; j < NX; ++j) o.P[i * NX + j] += w * gu[i] * gx[j];
        }
      }
    }
  }
  // --- M8 state-input limits (LeggedInterface.cpp:317-357)
  for (int j = 0; j < NJ; ++j) {
    Pen p = double_sided(x[12 + j], HB_JOINT_LOWER[j], HB_JOINT_UPPER[j], HB_LIMIT_POS_MU, HB_LIMIT_POS_DELTA);
    cost += p.v;
    if (L) { o.q[12 + j] += p.d1; o.Q[(12 + j) * NX + 12 + j] += p.d2; }
    Pen pv = double_sided(u[12 + j], -HB_JOINT_VEL_LIMIT[j], HB_JOINT_VEL_LIMIT[j], HB_LIMIT_VEL_MU, HB_LIMIT_VEL_DELTA);
    cost += pv.v;
    if (L) { o.r[12 + j] += pv.d1; o.R[(12 + j) * NU + 12 + j] += pv.d2; }
  }
  for (int c = 0; c < NC; ++c) {
    Pen p = double_sided(u[3 * c + 2], 0.0, HB_LIMIT_FORCE_MAX, HB_LIMIT_FORCE_MU, HB_LIMIT_FORCE_DELTA);
    cost += p.v;
    if (L) { o.r[3 * c + 2] += p.d1; o.R[(3 * c + 2) * NU + 3 * c + 2] += p.d2; }
  }
  o.cost = cost;
  // --- equality constraints M3/M4/M5
  int m = 0;
  for (int c = 0; c < NC; ++c) {
    if (fl[c]) {
      // zero velocity with z-position pull (LeggedInterface.cpp:436-446): v + diag(0,0,3) p + (0,0,-0.06)
      for (int a = 0; a < 3; ++a) {
        double val = evel[3 * c + a];
        if (a == 2) val += HB_ZEROVEL_Z_GAIN * epos[3 * c + 2] + HB_ZEROVEL_Z_OFFSET;
        o.e[m] = val;
        if (L) {
          for (int j = 0; j < NX; ++j) o.C[m * NX + j] = lin->dvel_dx[(3 * c + a) * NX + j] + (a == 2 ? HB_ZEROVEL_Z_GAIN * lin->dpos_dx[(3 * c + 2) * NX + j] : 0.0);
          for (int j = 0; j < NU; ++j) o.D[m * NU + j] = lin->dvel_du[(3 * c + a) * NU + j];
        }
        ++m;
      }
    } else {
      // zero force (ZeroForceConstraint.cpp:60-93)
      for (int a = 0; a < 3; ++a) {
        o.e[m] = u[3 * c + a];
        if (L) o.D[m * NU + 3 * c + a] = 1.0;
        ++m;
      }
      // normal velocity (NormalVelocityConstraintCppAd.cpp:71-98, LeggedRobotPreComputation.cpp:96-106)
      o.e[m] = evel[3 * c + 2] - swing[6 * c + 5] + HB_POSITION_ERROR_GAIN * (epos[3 * c + 2] - swing[6 * c + 2]);
      if (L) {
        for (int j = 0; j < NX; ++j) o.C[m * NX + j] = lin->dvel_dx[(3 * c + 2) * NX + j] + HB_POSITION_ERROR_GAIN * lin->dpos_dx[(3 * c + 2) * NX + j];
        for (int j = 0; j < NU; ++j) o.D[m * NU + j] = lin->dvel_du[(3 * c + 2) * NU + j];
      }
      ++m;
    }
  }
  o.m = m;
}

// RK2 (Heun) flow and sensitivities (S2)
void rk2_step(const double* x, const double* u, double dt, double* xnext) {
  double f1[NX], f2[NX], x2[NX];
  flow_map_T<double>(x, u, f1, nullptr, nullptr);
  for (int i = 0; i < NX; ++i) x2[i] = x[i] + dt * f1[i];
  flow_map_T<double>(x2, u, f2, nullptr, nullptr);
  for (int i = 0; i < NX; ++i) xnext[i] = x[i] + 0.5 * dt * (f1[i] + f2[i]);
}

void node_lq(double dt, const double* x, const double* u, const double* xn, const double* xref, const double* swing,
             int mode, NodeLQ& o) {
  static thread_local FlowLin k1, k2;
  flow_map_lin(x, u, k1);
  double x2[NX];
  for (int i = 0; i < NX; ++i) x2[i] = x[i] + dt * k1.f[i];
  flow_map_lin(x2, u, k2);
  // A2 <- A2 (I + dt A1); B2 <- B2 + dt A2 B1
  double A2A1[NX * NX], A2B1[NX * NU];
  for (int i = 0; i < NX; ++i)
    for (int j = 0; j < NX; ++j) {
      double s = 0.0, t = 0.0;
      for (int k = 0; k < NX; ++k) { s += k2.A[i * NX + k] * k1.A[k * NX + j]; t += k2.A[i * NX + k] * k1.B[k * NU + j]; }
      A2A1[i * NX + j] = s; A2B1[i * NU + j] = t;
    }
  for (int i = 0; i < NX; ++i) {
    for (int j = 0; j < NX; ++j) o.Ad[i * NX + j] = (i == j ? 1.0 : 0.0) + 0.5 * dt * (k1.A[i * NX + j] + k2.A[i * NX + j] + dt * A2A1[i * NX + j]);
    for (int j = 0; j < NU; ++j) o.Bd[i * NU + j] = 0.5 * dt * (k1.B[i * NU + j] + k2.B[i * NU + j] + dt * A2B1[i * NU + j]);
    o.b[i] = x[i] + 0.5 * dt * (k1.f[i] + k2.f[i]) - xn[i];
  }
  node_cost_constraints(x, u, xref, swing, mode, k1.epos, k1.evel, &k1, o);
}

// ---------------------------------------------------------------- small dense helpers (row-major)
inline void mm(const double* A, const double* B, double* C, int m, int k, int n) {  // C[m x n] = A[m x k] B[k x n]
  for (int i = 0; i < m; ++i)
    for (int j = 0; j < n; ++j) { double s = 0.0; for (int l = 0; l < k; ++l) s += A[i * k + l] * B[l * n + j]; C[i * n + j] = s; }
}
inline void mtm(const double* A, const double* B, double* C, int k, int m, int n) {  // C[m x n] = A^T[m x k] B[k x n], A is k x m
  for (int i = 0; i < m; ++i)
    for (int j = 0; j < n; ++j) { double s = 0.0; for (int l = 0; l < k; ++l) s += A[l * m + i] * B[l * n + j]; C[i * n + j] = s; }
}

struct Projection { double Px[NU * NX], Pu[NU * NU], pe[NU]; int nt; };  // du = Px dx + Pu w + pe, w in R^nt

// Least-squares projection of the state-input equalities C dx + D du + e = 0 (S4). D is rank deficient for Hunter
// (two point contacts on one rigid foot), so the projection is defined through the normal equations
// D^T D du = -D^T (C dx + e), solved by Gauss-Jordan elimination with diagonal pivoting and a rank threshold.
void project_constraints(const NodeLQ& lq, Projection& pr) {
  const int m = lq.m;
  double G[NU][NU + NX + 1];
  for (int i = 0; i < NU; ++i) {
    for (int j = 0; j < NU; ++j) { double s = 0.0; for (int r = 0; r < m; ++r) s += lq.D[r * NU + i] * lq.D[r * NU + j]; G[i][j] = s; }
    for (int j = 0; j < NX; ++j) { double s = 0.0; for (int r = 0; r < m; ++r) s += lq.D[r * NU + i] * lq.C[r * NX + j]; G[i][NU + j] = -s; }
    double s = 0.0; for (int r = 0; r < m; ++r) s += lq.D[r * NU + i] * lq.e[r];
    G[i][NU + NX] = -s;
  }
  double dmax = 0.0;
  for (int i = 0; i < NU; ++i) dmax = std::max(dmax, G[i][i]);
  const double tol = 1e-9 * std::max(dmax, 1e-300);
  bool piv[NU] = {false};
  for (int step = 0; step < NU; ++step) {
    int p = -1; double best = tol;
    for (int i = 0; i < NU; ++i) if (!piv[i] && G[i][i] > best) { best = G[i][i]; p = i; }
    if (p < 0) break;
    piv[p] = true;
    const double inv = 1.0 / G[p][p];
    for (int j = 0; j < NU + NX + 1; ++j) G[p][j] *= inv;
    for (int i = 0; i < NU; ++i) {
      if (i == p) continue;
      const double f = G[i][p];
      if (f == 0.0) continue;
      for (int j = 0; j < NU + NX + 1; ++j) G[i][j] -= f * G[p][j];
    }
  }
  std::fill(pr.Px, pr.Px + NU * NX, 0.0); std::fill(pr.Pu, pr.Pu + NU * NU, 0.0); std::fill(pr.pe, pr.pe + NU, 0.0);
  int nt = 0;
  int freeidx[NU];
  for (int i = 0; i < NU; ++i) if (!piv[i]) freeidx[nt++] = i;
  for (int i = 0; i < NU; ++i) {
    if (piv[i]) {
      for (int j = 0; j < NX; ++j) pr.Px[i * NX + j] = G[i][NU + j];
      pr.pe[i] = G[i][NU + NX];
      for (int c = 0; c < nt; ++c) pr.Pu[i * NU + c] = -G[i][freeidx[c]];
    }
  }
  for (int c = 0; c < nt; ++c) pr.Pu[freeidx[c] * NU + c] = 1.0;
  pr.nt = nt;
}

struct NodeGain {  // closed-loop maps of one node in original coordinates
  double Kx[NX * NX], kx[NX];  // dx+ = Kx dx + kx
  double Ku[NU * NX], ku[NU];  // du  = Ku dx + ku
  double gq[NX], gu_w[NU], Kw[NU * NX], kw[NU];  // armijo pieces: projected gradients q~, r~ and w = Kw dx + kw
  int nt;
};

// Cholesky solve of SPD system (n<=22), in place on copies
bool chol_solve(const double* Hin, int n, const double* rhs, int nrhs, double* out) {
  double Lm[NU * NU];
  for (int i = 0; i < n; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = Hin[i * n + j];
      for (int k = 0; k < j; ++k) s -= Lm[i * n + k] * Lm[j * n + k];
      if (i == j) { if (!(s > 0.0)) return false; Lm[i * n + i] = std::sqrt(s); }
      else Lm[i * n + j] = s / Lm[j * n + j];
    }
  for (int c = 0; c < nrhs; ++c) {
    double y[NU];
    for (int i = 0; i < n; ++i) { double s = rhs[i * nrhs + c]; for (int k = 0; k < i; ++k) s -= Lm[i * n + k] * y[k]; y[i] = s / Lm[i * n + i]; }
    for (int i = n - 1; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < n; ++k) s -= Lm[k * n + i] * out[k * nrhs + c]; out[i * nrhs + c] = s / Lm[i * n + i]; }
  }
  return true;
}

// One backward Riccati step (S5, App. C.5 step 3) on the projected model; updates S (NXxNX), s (NX).
bool riccati_step(const NodeLQ& lq, const Projection& pr, double dt, double* S, double* s, NodeGain& g) {
  const int nt = pr.nt;
  // scaled cost (S3): stage cost times dt
  double Q[NX * NX], R[NU * NU], P[NU * NX], q[NX], r[NU];
  for (int i = 0; i < NX * NX; ++i) Q[i] = dt * lq.Q[i];
  for (int i = 0; i < NU * NU; ++i) R[i] = dt * lq.R[i];
  for (int i = 0; i < NU * NX; ++i) P[i] = dt * lq.P[i];
  for (int i = 0; i < NX; ++i) q[i] = dt * lq.q[i];
  for (int i = 0; i < NU; ++i) r[i] = dt * lq.r[i];
  // compact Pu to NU x nt
  double Pu[NU * NU];
  for (int i = 0; i < NU; ++i) for (int c = 0; c < nt; ++c) Pu[i * nt + c] = pr.Pu[i * NU + c];
  // At = A + B Px ; Bt = B Pu ; bt = b + B pe
  double At[NX * NX], Bt[NX * NU], bt[NX], T1[NX * NX];
  mm(lq.Bd, pr.Px, T1, NX, NU, NX);
  for (int i = 0; i < NX * NX; ++i) At[i] = lq.Ad[i] + T1[i];
  mm(lq.Bd, Pu, Bt, NX, NU, nt);
  for (int i = 0; i < NX; ++i) { double t = lq.b[i]; for (int j = 0; j < NU; ++j) t += lq.Bd[i * NU + j] * pr.pe[j]; bt[i] = t; }
  // projected cost
  double RPx[NU * NX], PRPx[NU * NX], rRpe[NU];
  mm(R, pr.Px, RPx, NU, NU, NX);
  for (int i = 0; i < NU * NX; ++i) PRPx[i] = P[i] + RPx[i];
  for (int i = 0; i < NU; ++i) { double t = r[i]; for (int j = 0; j < NU; ++j) t += R[i * NU + j] * pr.pe[j]; rRpe[i] = t; }
  double Qt[NX * NX], qt[NX], Pt[NU * NX], Rt[NU * NU], rt[NU], T2[NX * NX], T3[NU * NU];
  // Qt = Q + Px^T P + P^T Px + Px^T R Px
  mtm(pr.Px, P, T1, NU, NX, NX);       // Px^T P
  mtm(pr.Px, RPx, T2, NU, NX, NX);     // Px^T R Px
  for (int i = 0; i < NX; ++i) for (int j = 0; j < NX; ++j) Qt[i * NX + j] = Q[i * NX + j] + T1[i * NX + j] + T1[j * NX + i] + T2[i * NX + j];
  for (int i = 0; i < NX; ++i) {
    double t = q[i];
    for (int j = 0; j < NU; ++j) t += pr.Px[j * NX + i] * rRpe[j] + P[j * NX + i] * pr.pe[j];
    qt[i] = t;
  }
  mtm(Pu, PRPx, Pt, NU, nt, NX);       // nt x NX
  mm(R, Pu, T3, NU, NU, nt);           // NU x nt
  mtm(Pu, T3, Rt, NU, nt, nt);         // nt x nt
  for (int c = 0; c < nt; ++c) { double t = 0.0; for (int j = 0; j < NU; ++j) t += Pu[j * nt + c] * rRpe[j]; rt[c] = t; }
  // Riccati
  double SA[NX * NX], SB[NX * NU], sb[NX];
  mm(S, At, SA, NX, NX, NX);
  mm(S, Bt, SB, NX, NX, nt);
  for (int i = 0; i < NX; ++i) { double t = s[i]; for (int j = 0; j < NX; ++j) t += S[i * NX + j] * bt[j]; sb[i] = t; }
  double Huu[NU * NU], Hux[NU * NX], hu[NU];
  mtm(Bt, SB, Huu, NX, nt, nt);
  for (int i = 0; i < nt * nt; ++i) Huu[i] += Rt[i];
  mtm(Bt, SA, Hux, NX, nt, NX);
  for (int i = 0; i < nt * NX; ++i) Hux[i] += Pt[i];
  for (int c = 0; c < nt; ++c) { double t = rt[c]; for (int j = 0; j < NX; ++j) t += Bt[j * nt + c] * sb[j]; hu[c] = t; }
  for (int i = 0; i < nt; ++i) for (int j = 0; j < i; ++j) { double a = 0.5 * (Huu[i * nt + j] + Huu[j * nt + i]); Huu[i * nt + j] = Huu[j * nt + i] = a; }
  double K[NU * NX], kff[NU], rhs[NU * (NX + 1)], sol[NU * (NX + 1)];
  for (int c = 0; c < nt; ++c) { for (int j = 0; j < NX; ++j) rhs[c * (NX + 1) + j] = -Hux[c * NX + j]; rhs[c * (NX + 1) + NX] = -hu[c]; }
  if (nt > 0 && !chol_solve(Huu, nt, rhs, NX + 1, sol)) return false;
  for (int c = 0; c < nt; ++c) { for (int j = 0; j < NX; ++j) K[c * NX + j] = sol[c * (NX + 1) + j]; kff[c] = sol[c * (NX + 1) + NX]; }
  // S <- Qt + At^T S At + Hux^T K ; s <- qt + At^T (s + S bt) + Hux^T kff
  double Sn[NX * NX], sn[NX];
  mtm(At, SA, Sn, NX, NX, NX);
  mtm(Hux, K, T1, nt, NX, NX);
  for (int i = 0; i < NX * NX; ++i) Sn[i] += Qt[i] + T1[i];
  for (int i = 0; i < NX; ++i) {
    double t = qt[i];
    for (int j = 0; j < NX; ++j) t += At[j * NX + i] * sb[j];
    for (int c = 0; c < nt; ++c) t += Hux[c * NX + i] * kff[c];
    sn[i] = t;
  }
  for (int i = 0; i < NX; ++i) for (int j = 0; j < NX; ++j) S[i * NX + j] = 0.5 * (Sn[i * NX + j] + Sn[j * NX + i]);
  for (int i = 0; i < NX; ++i) s[i] = sn[i];
  // closed loop in original coordinates
  double PuK[NU * NX];
  mm(Pu, K, PuK, NU, nt, NX);
  for (int i = 0; i < NU * NX; ++i) g.Ku[i] = pr.Px[i] + PuK[i];
  for (int i = 0; i < NU; ++i) { double t = pr.pe[i]; for (int c = 0; c < nt; ++c) t += Pu[i * nt + c] * kff[c]; g.ku[i] = t; }
  mm(Bt, K, T1, NX, nt, NX);
  for (int i = 0; i < NX * NX; ++i) g.Kx[i] = At[i] + T1[i];
  for (int i = 0; i < NX; ++i) { double t = bt[i]; for (int c = 0; c < nt; ++c) t += Bt[i * nt + c] * kff[c]; g.kx[i] = t; }
  for (int i = 0; i < NX; ++i) g.gq[i] = qt[i];
  for (int c = 0; c < nt; ++c) { g.gu_w[c] = rt[c]; g.kw[c] = kff[c]; for (int j = 0; j < NX; ++j) g.Kw[c * NX + j] = K[c * NX + j]; }
  g.nt = nt;
  return true;
}

struct Perf { double merit, dynSSE, eqSSE; };
inline double dt_of(const hbo_horizon& hz, int k) { return hz.dts ? hz.dts[k] : hz.dt; }
inline double total_violation(const Perf& p) { return std::sqrt(p.dynSSE + p.eqSSE); }

// computePerformance (S6): merit = sum dt*cost, SSE = dt*||defect||^2, dt*||eq||^2
Perf performance(const hbo_horizon& hz, const double* xt, const double* ut, const double* x_ref, const double* swing,
                 const int32_t* mode) {
  Perf pf{0.0, 0.0, 0.0};
  NodeLQ tmp;
  for (int k = 0; k < hz.N; ++k) {
    const double dtk = dt_of(hz, k);
    const double* x = xt + k * NX; const double* u = ut + k * NU;
    double f1[NX], f2[NX], x2[NX], ep[12], ev[12];
    flow_map_T<double>(x, u, f1, ep, ev);
    for (int i = 0; i < NX; ++i) x2[i] = x[i] + dtk * f1[i];
    flow_map_T<double>(x2, u, f2, nullptr, nullptr);
    double d2 = 0.0;
    for (int i = 0; i < NX; ++i) { double d = x[i] + 0.5 * dtk * (f1[i] + f2[i]) - xt[(k + 1) * NX + i]; d2 += d * d; }
    node_cost_constraints(x, u, x_ref + k * NX, swing + k * 24, mode[k], ep, ev, nullptr, tmp);
    double e2 = 0.0;
    for (int i = 0; i < tmp.m; ++i) e2 += tmp.e[i] * tmp.e[i];
    pf.merit += dtk * tmp.cost; pf.dynSSE += dtk * d2; pf.eqSSE += dtk * e2;
  }
  return pf;
}

// max_trials caps the line search's trials like hb_config.line_search_max_trials; record (nullable) receives one row per trial evaluated
void mpc_iteration(const hbo_horizon& hz, const double* x0, const double* x_ref, const double* swing, const int32_t* mode,
                   double* xt, double* ut, hbo_solve_info* info, int max_trials = 14, hbo_ls_trial* record = nullptr) {
  const int N = hz.N;
  for (int i = 0; i < NX; ++i) xt[i] = x0[i];
  std::vector<NodeGain> gains(N);
  double S[NX * NX], s[NX];
  std::fill(S, S + NX * NX, 0.0); std::fill(s, s + NX, 0.0);  // no terminal cost (App. B)
  Perf base{0.0, 0.0, 0.0};
  static thread_local NodeLQ lq;
  Projection pr;
  bool ok = true;
  for (int k = N - 1; k >= 0; --k) {
    const double dtk = dt_of(hz, k);
    node_lq(dtk, xt + k * NX, ut + k * NU, xt + (k + 1) * NX, x_ref + k * NX, swing + k * 24, mode[k], lq);
    double d2 = 0.0, e2 = 0.0;
    for (int i = 0; i < NX; ++i) d2 += lq.b[i] * lq.b[i];
    for (int i = 0; i < lq.m; ++i) e2 += lq.e[i] * lq.e[i];
    base.merit += dtk * lq.cost; base.dynSSE += dtk * d2; base.eqSSE += dtk * e2;
    project_constraints(lq, pr);
    ok = ok && riccati_step(lq, pr, dtk, S, s, gains[k]);
  }
  // forward pass
  std::vector<double> dx((N + 1) * NX, 0.0), du(N * NU, 0.0);
  double armijo = 0.0;
  for (int k = 0; k < N; ++k) {
    const NodeGain& g = gains[k];
    const double* d = &dx[k * NX];
    for (int i = 0; i < NU; ++i) { double t = g.ku[i]; for (int j = 0; j < NX; ++j) t += g.Ku[i * NX + j] * d[j]; du[k * NU + i] = t; }
    for (int i = 0; i < NX; ++i) { double t = g.kx[i]; for (int j = 0; j < NX; ++j) t += g.Kx[i * NX + j] * d[j]; dx[(k + 1) * NX + i] = t; }
    for (int i = 0; i < NX; ++i) armijo += g.gq[i] * d[i];
    for (int c = 0; c < g.nt; ++c) { double w = g.kw[c]; for (int j = 0; j < NX; ++j) w += g.Kw[c * NX + j] * d[j]; armijo += g.gu_w[c] * w; }
  }
  // filter line search (App. C.5 step 4)
  const double gamma_c = 1e-6, armijoFactor = 1e-4, alpha_decay = 0.5, alpha_min = 1e-4;
  const double v0 = total_violation(base);
  std::vector<double> xn((N + 1) * NX), un(N * NU);
  double alpha = 1.0; bool accepted = false; Perf pn = base; int trials = 0;
  bool finite = ok;
  for (double v : dx) finite = finite && std::isfinite(v);
  for (double v : du) finite = finite && std::isfinite(v);
  if (finite) {
    while (alpha >= alpha_min && trials < max_trials) {
      for (size_t i = 0; i < xn.size(); ++i) xn[i] = xt[i] + alpha * dx[i];
      for (size_t i = 0; i < un.size(); ++i) un[i] = ut[i] + alpha * du[i];
      pn = performance(hz, xn.data(), un.data(), x_ref, swing, mode);
      const double v1 = total_violation(pn);
      const double am = alpha * armijo;
      bool acc;
      int branch;
      if (v1 > HB_SQP_G_MAX) { branch = HBO_LS_VIOLATION; acc = v1 < (1.0 - gamma_c) * v0; }
      else if (v1 < HB_SQP_G_MIN && v0 < HB_SQP_G_MIN && am < 0.0) { branch = HBO_LS_ARMIJO; acc = pn.merit < base.merit + armijoFactor * am; }
      else { branch = HBO_LS_FILTER; acc = pn.merit < (base.merit - gamma_c * v0) || v1 < (1.0 - gamma_c) * v0; }
      acc = std::isfinite(pn.merit) && std::isfinite(v1) && acc;
      if (record) record[trials] = hbo_ls_trial{alpha, pn.merit, v1, branch, acc ? 1 : 0};
      ++trials;
      if (acc) { accepted = true; break; }
      alpha *= alpha_decay;
    }
  }
  if (accepted) {
    std::copy(xn.begin(), xn.end(), xt);
    std::copy(un.begin(), un.end(), ut);
  }
  if (info) {
    info->alpha = accepted ? alpha : 0.0;
    info->merit0 = base.merit; info->viol0 = v0;
    info->merit1 = accepted ? pn.merit : base.merit; info->viol1 = accepted ? total_violation(pn) : v0;
    info->armijo = armijo; info->status = finite ? 0 : 3; info->n_trials = trials;
  }
}

// ---------------------------------------------------------------- WBC (W1-W3)
void rbd_to_qv(const double* rbd, double* q, double* v) {
  // WbcBase.cpp:72-79; rbd = [zyx(3), p(3), qj(10), omega_world(3), v(3), qj_dot(10)] (StateEstimateBase.cpp:73-106)
  for (int i = 0; i < 3; ++i) { q[i] = rbd[3 + i]; q[3 + i] = rbd[i]; v[i] = rbd[NQ + 3 + i]; }
  for (int j = 0; j < NJ; ++j) { q[6 + j] = rbd[6 + j]; v[6 + j] = rbd[NQ + 6 + j]; }
  // euler rates from world angular velocity: solve T rates = omega
  const double cz = std::cos(q[3]), sz = std::sin(q[3]), cy = std::cos(q[4]), sy = std::sin(q[4]);
  const double w[3] = {rbd[NQ], rbd[NQ + 1], rbd[NQ + 2]};
  // T = [[0,-sz,cz cy],[0,cz,sz cy],[1,0,-sy]]
  const double dx = (cz * w[0] + sz * w[1]) / cy;  // roll rate
  const double dy = -sz * w[0] + cz * w[1];        // pitch rate
  const double dz = w[2] + sy * dx;                // yaw rate
  v[3] = dz; v[4] = dy; v[5] = dx;
}

// rotationMatrixToRotationVector(R_ref R_meas^T)  (rotationErrorInWorld, WbcBase.cpp:281; App. C.1)
void rotation_error_world(const double* Rref, const double* Rmeas, double* err) {
  double E[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double s = 0.0; for (int k = 0; k < 3; ++k) s += Rref[3 * i + k] * Rmeas[3 * j + k]; E[3 * i + j] = s; }
  const double sk[3] = {E[7] - E[5], E[2] - E[6], E[3] - E[1]};
  double c = 0.5 * (E[0] + E[4] + E[8] - 1.0);
  c = std::min(1.0, std::max(-1.0, c));
  const double ang = std::acos(c);
  const double sn = std::sqrt(sk[0] * sk[0] + sk[1] * sk[1] + sk[2] * sk[2]);  // = 2 sin(ang)
  double f = 0.5;
  if (ang > 1e-8 && sn > 1e-12) f = ang / sn;
  for (int i = 0; i < 3; ++i) err[i] = f * sk[i];
}

struct WbcQP { double H[38 * 38], g[38], A[60 * 38], lbA[60], ubA[60]; int m; };
constexpr double QP_INF = 1e20;  // qpOASES::INFTY

// `terms` (optional) receives the pieces the hierarchical WBC stacks by priority instead of by weight: the weighted task rows
// (Aw 24x38, bw 24, row count), the contact Jacobian (12x16) and dJ/dt v (12).
struct WbcTerms { double Aw[24 * 38], bw[24], J[12 * NQ], dJv[12]; int rw; };
void wbc_assemble(const double* x_des, const double* u_des, const double* rbd, int mode, bool stance_mode, WbcQP& qp, WbcTerms* terms = nullptr) {
  bool fl[4]; mode_to_flags(mode, fl);
  int nc = fl[0] + fl[1] + fl[2] + fl[3];
  const int NV = 38;
  // ---- updateMeasured (WbcBase.cpp:70-117)
  double q[NQ], v[NQ];
  rbd_to_qv(rbd, q, v);
  Kin<double> kin; forward_kinematics(q, kin);
  double M[NQ * NQ], nle[NQ], zero[NQ] = {0};
  for (int c = 0; c < NQ; ++c) {
    double e[NQ] = {0}, col[NQ]; e[c] = 1.0;
    rnea(q, zero, e, false, col, &kin);
    for (int r = 0; r < NQ; ++r) M[r * NQ + c] = col[r];
  }
  for (int i = 0; i < NQ; ++i) for (int j = 0; j < i; ++j) { double a = 0.5 * (M[i * NQ + j] + M[j * NQ + i]); M[i * NQ + j] = M[j * NQ + i] = a; }
  rnea(q, v, zero, true, nle, &kin);
  // contact Jacobians and dJ*v via first-order AD along q_dot = v
  double J[12 * NQ], dJv[12], pos_m[12], vel_m[12];
  {
    for (int c = 0; c < NQ; ++c) {
      double e[NQ] = {0}; e[c] = 1.0;
      Vel<double> ve; velocities(kin, e, ve);
      for (int i = 0; i < NC; ++i) { double vc[3]; contact_velocity(kin, ve, i, vc); for (int a = 0; a < 3; ++a) J[(3 * i + a) * NQ + c] = vc[a]; }
    }
    using D1 = Dual<1>;
    D1 qd[NQ], vd[NQ];
    for (int i = 0; i < NQ; ++i) { qd[i].v = q[i]; qd[i].d[0] = v[i]; vd[i] = D1(v[i]); }
    Kin<D1> kd; forward_kinematics(qd, kd);
    Vel<D1> ud; velocities(kd, vd, ud);
    for (int i = 0; i < NC; ++i) {
      D1 pc[3], vc[3]; contact_position(kd, i, pc); contact_velocity(kd, ud, i, vc);
      for (int a = 0; a < 3; ++a) { pos_m[3 * i + a] = pc[a].v; vel_m[3 * i + a] = vc[a].v; dJv[3 * i + a] = vc[a].d[0]; }
    }
  }
  // base angular Jacobian rows (LOCAL_WORLD_ALIGNED): omega = T(euler) rates -> cols 3..5 = world axes; dJ*v = dT/dt rates
  double Jw[3 * NQ] = {0}, dJw_v[3];
  for (int i = 0; i < 3; ++i) for (int a = 0; a < 3; ++a) Jw[a * NQ + 3 + i] = kin.ax[3 + i][a];
  {
    double w1[3], w2[3], t1[3], t2[3];
    for (int i = 0; i < 3; ++i) { w1[i] = kin.ax[3][i] * v[3]; w2[i] = w1[i] + kin.ax[4][i] * v[4]; }
    cross3(w1, kin.ax[4], t1); cross3(w2, kin.ax[5], t2);
    for (int i = 0; i < 3; ++i) dJw_v[i] = t1[i] * v[4] + t2[i] * v[5];
  }
  // ---- updateDesired (WbcBase.cpp:119-136) + computeBaseKinematicsFromCentroidalModel (App. C.2)
  double f_des[NX], pos_d[12], vel_d[12], vdes[NQ];
  flow_map_T<double>(x_des, u_des, f_des, pos_d, vel_d, vdes);
  double basePose[6], baseVel[6], baseAcc[6];
  for (int i = 0; i < 6; ++i) basePose[i] = x_des[6 + i];
  {
    const double* qd = x_des + 6;
    Kin<double> kd; forward_kinematics(qd, kd);
    double com[3]; center_of_mass(kd, com);
    double A[6 * NQ]; centroidal_matrix(kd, com, A);
    // Adot*v = d/dt (A(q) v) at fixed v, along q_dot = v
    using D1 = Dual<1>;
    D1 q1[NQ], v1[NQ];
    for (int i = 0; i < NQ; ++i) { q1[i].v = qd[i]; q1[i].d[0] = vdes[i]; v1[i] = D1(vdes[i]); }
    Kin<D1> k1; forward_kinematics(q1, k1);
    D1 c1[3]; center_of_mass(k1, c1);
    Vel<D1> u1; velocities(k1, v1, u1);
    D1 h1[6]; centroidal_momentum(k1, u1, c1, h1);
    double rhs[6], qbdd[6];
    for (int i = 0; i < 6; ++i) rhs[i] = HB_TOTAL_MASS * f_des[i] - h1[i].d[0];  // joint accelerations are zero (WbcBase.cpp:133)
    solve6(A, rhs, qbdd);
    for (int i = 0; i < 3; ++i) { baseVel[i] = vdes[i]; baseAcc[i] = qbdd[i]; }
    // angular velocity / acceleration in world from euler rates and second derivatives
    double w1[3], w2[3], t1[3], t2[3];
    for (int i = 0; i < 3; ++i) { w1[i] = kd.ax[3][i] * vdes[3]; w2[i] = w1[i] + kd.ax[4][i] * vdes[4]; }
    cross3(w1, kd.ax[4], t1); cross3(w2, kd.ax[5], t2);
    for (int i = 0; i < 3; ++i) {
      baseVel[3 + i] = kd.ax[3][i] * vdes[3] + kd.ax[4][i] * vdes[4] + kd.ax[5][i] * vdes[5];
      baseAcc[3 + i] = kd.ax[3][i] * qbdd[3] + kd.ax[4][i] * qbdd[4] + kd.ax[5][i] * qbdd[5] + t1[i] * vdes[4] + t2[i] * vdes[5];
    }
  }
  // ---- constraints: EoM + torque limits + friction (WeightedWbc.cpp:68-71)
  std::fill(qp.A, qp.A + 60 * NV, 0.0);
  int row = 0;
  // formulateFloatingBaseEomTask (WbcBase.cpp:138-149): [M, -J^T, -S^T] x = -nle
  for (int i = 0; i < NQ; ++i) {
    for (int j = 0; j < NQ; ++j) qp.A[row * NV + j] = M[i * NQ + j];
    for (int j = 0; j < 12; ++j) qp.A[row * NV + NQ + j] = -J[j * NQ + i];
    if (i >= 6) qp.A[row * NV + NQ + 12 + (i - 6)] = -1.0;
    qp.lbA[row] = qp.ubA[row] = -nle[i];
    ++row;
  }
  // formulateFrictionConeTask equality part: swing contact forces = 0 (WbcBase.cpp:190-203)
  for (int c = 0; c < NC; ++c) if (!fl[c]) for (int a = 0; a < 3; ++a) { qp.A[row * NV + NQ + 3 * c + a] = 1.0; qp.lbA[row] = qp.ubA[row] = 0.0; ++row; }
  // formulateTorqueLimitsTask (WbcBase.cpp:151-167)
  for (int sgn = 0; sgn < 2; ++sgn) for (int j = 0; j < NJ; ++j) {
    qp.A[row * NV + NQ + 12 + j] = sgn == 0 ? 1.0 : -1.0; qp.lbA[row] = -QP_INF; qp.ubA[row] = g_wbc.torque[j % 5]; ++row;
  }
  // friction pyramid on stance contacts, then 3*(4-nc) all-zero rows (WbcBase.cpp:205-221)
  const double mu = g_wbc.mu;
  const double pyr[5][3] = {{0, 0, -1}, {1, 0, -mu}, {-1, 0, -mu}, {0, 1, -mu}, {0, -1, -mu}};
  for (int c = 0; c < NC; ++c) if (fl[c]) for (int r = 0; r < 5; ++r) {
    for (int a = 0; a < 3; ++a) qp.A[row * NV + NQ + 3 * c + a] = pyr[r][a];
    qp.lbA[row] = -QP_INF; qp.ubA[row] = 0.0; ++row;
  }
  for (int r = 0; r < 3 * (NC - nc); ++r) { qp.lbA[row] = -QP_INF; qp.ubA[row] = 0.0; ++row; }
  qp.m = row;
  // ---- weighted tasks (WeightedWbc.cpp:73-94)
  double Aw[36 * 38]; double bw[36]; int rw = 0;
  std::fill(Aw, Aw + 36 * NV, 0.0);
  if (stance_mode) {
    for (int i = 0; i < 6; ++i) { Aw[rw * NV + i] = g_wbc.weight_base; bw[rw] = 0.0; ++rw; }
  } else {
    // swing leg task (WbcBase.cpp:297-323)
    for (int c = 0; c < NC; ++c) if (!fl[c]) for (int a = 0; a < 3; ++a) {
      const double acc = g_wbc.swing_kp * (pos_d[3 * c + a] - pos_m[3 * c + a]) + g_wbc.swing_kd * (vel_d[3 * c + a] - vel_m[3 * c + a]);
      for (int j = 0; j < NQ; ++j) Aw[rw * NV + j] = g_wbc.weight_swing * J[(3 * c + a) * NQ + j];
      bw[rw] = g_wbc.weight_swing * (acc - dJv[3 * c + a]); ++rw;
    }
    // base xy acceleration (WbcBase.cpp:228-240)
    for (int a = 0; a < 2; ++a) { Aw[rw * NV + a] = g_wbc.weight_base; bw[rw] = g_wbc.weight_base * baseAcc[a]; ++rw; }
    // base height (WbcBase.cpp:243-256)
    Aw[rw * NV + 2] = g_wbc.weight_base;
    bw[rw] = g_wbc.weight_base * (baseAcc[2] + g_wbc.height_kp * (basePose[2] - q[2]) + g_wbc.height_kd * (baseVel[2] - v[2]));
    ++rw;
    // base angular motion (WbcBase.cpp:259-290)
    double Rm[9], Rr[9], err[3], wm[3];
    euler_zyx_to_R(q + 3, Rm); euler_zyx_to_R(basePose + 3, Rr);
    rotation_error_world(Rr, Rm, err);
    for (int i = 0; i < 3; ++i) wm[i] = kin.ax[3][i] * v[3] + kin.ax[4][i] * v[4] + kin.ax[5][i] * v[5];
    for (int a = 0; a < 3; ++a) {
      for (int j = 0; j < NQ; ++j) Aw[rw * NV + j] = g_wbc.weight_base * Jw[a * NQ + j];
      bw[rw] = g_wbc.weight_base * (baseAcc[3 + a] + g_wbc.angular_kp * err[a] + g_wbc.angular_kd * (baseVel[3 + a] - wm[a]) - dJw_v[a]);
      ++rw;
    }
    // contact force task (WbcBase.cpp:325-338) * weightContactForce (0 in the shipped task.info:328-333)
    if (g_wbc.weight_force != 0.0) for (int j = 0; j < 12; ++j) { Aw[rw * NV + NQ + j] = g_wbc.weight_force; bw[rw] = g_wbc.weight_force * u_des[j]; ++rw; }
  }
  if (terms) {
    const int rt = rw < 24 ? rw : 24;      // the swing / base rows (the hierarchical formulation builds its own contact-force task)
    std::memcpy(terms->Aw, Aw, sizeof(double) * 24 * NV); std::memcpy(terms->bw, bw, sizeof(double) * 24); terms->rw = rt;
    std::memcpy(terms->J, J, sizeof(J)); std::memcpy(terms->dJv, dJv, sizeof(dJv));
  }
  for (int i = 0; i < NV; ++i) {
    for (int j = 0; j < NV; ++j) { double s = 0.0; for (int r = 0; r < rw; ++r) s += Aw[r * NV + i] * Aw[r * NV + j]; qp.H[i * NV + j] = s; }
    double s = 0.0; for (int r = 0; r < rw; ++r) s += Aw[r * NV + i] * bw[r];
    qp.g[i] = -s;
  }
}

// ---------------------------------------------------------------- dense QP: primal-dual interior point (stands in for W4)
// min 1/2 x'(H + rho I)x + g'x  s.t. lbA <= A x <= ubA. Rows with lbA == ubA are equalities, |bound| >= 1e19 is infinite.
// Dense LU with partial pivoting on the reduced KKT system; Mehrotra predictor-corrector.
bool lu_solve(std::vector<double>& Mx, int n, std::vector<double>& rhs) {
  std::vector<int> perm(n);
  for (int i = 0; i < n; ++i) perm[i] = i;
  for (int c = 0; c < n; ++c) {
    int p = c; double best = std::fabs(Mx[c * n + c]);
    for (int r = c + 1; r < n; ++r) if (std::fabs(Mx[r * n + c]) > best) { best = std::fabs(Mx[r * n + c]); p = r; }
    if (best == 0.0 || !std::isfinite(best)) return false;
    if (p != c) { for (int j = 0; j < n; ++j) std::swap(Mx[c * n + j], Mx[p * n + j]); std::swap(rhs[c], rhs[p]); }
    for (int r = c + 1; r < n; ++r) {
      const double f = Mx[r * n + c] / Mx[c * n + c];
      if (f == 0.0) continue;
      for (int j = c; j < n; ++j) Mx[r * n + j] -= f * Mx[c * n + j];
      rhs[r] -= f * rhs[c];
    }
  }
  for (int r = n - 1; r >= 0; --r) { double s = rhs[r]; for (int j = r + 1; j < n; ++j) s -= Mx[r * n + j] * rhs[j]; rhs[r] = s / Mx[r * n + r]; }
  return true;
}

int qp_solve(int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA, double rho,
             double* x, int* iters_out) {
  // split rows
  std::vector<int> eq; std::vector<double> beq;
  std::vector<std::vector<double>> Din; std::vector<double> fin;
  for (int r = 0; r < m; ++r) {
    const double* a = A + r * n;
    double nrm = 0.0; for (int j = 0; j < n; ++j) nrm = std::max(nrm, std::fabs(a[j]));
    const bool lo = lbA[r] > -1e19, hi = ubA[r] < 1e19;
    if (nrm == 0.0) { if ((lo && lbA[r] > 1e-12) || (hi && ubA[r] < -1e-12)) return 2; continue; }
    if (lo && hi && lbA[r] == ubA[r]) { eq.push_back(r); beq.push_back(ubA[r]); continue; }
    if (hi) { Din.emplace_back(a, a + n); fin.push_back(ubA[r]); }
    if (lo) { std::vector<double> t(n); for (int j = 0; j < n; ++j) t[j] = -a[j]; Din.push_back(t); fin.push_back(-lbA[r]); }
  }
  const int me = (int)eq.size(), mi = (int)Din.size();
  std::vector<double> xx(n, 0.0), y(me, 0.0), s(mi, 1.0), z(mi, 1.0);
  auto Dx = [&](const std::vector<double>& v, int r) { double t = 0.0; for (int j = 0; j < n; ++j) t += Din[r][j] * v[j]; return t; };
  for (int r = 0; r < mi; ++r) { s[r] = std::max(1.0, fin[r] - Dx(xx, r)); z[r] = 1.0; }
  const int nk = n + me;
  int it = 0; int status = 1;
  const int max_it = 60;
  for (; it < max_it; ++it) {
    // residuals
    std::vector<double> rd(n), rp(me), rs(mi);
    for (int i = 0; i < n; ++i) {
      double t = g[i] + rho * xx[i];
      for (int j = 0; j < n; ++j) t += H[i * n + j] * xx[j];
      for (int r = 0; r < me; ++r) t += A[eq[r] * n + i] * y[r];
      for (int r = 0; r < mi; ++r) t += Din[r][i] * z[r];
      rd[i] = t;
    }
    for (int r = 0; r < me; ++r) { double t = -beq[r]; for (int j = 0; j < n; ++j) t += A[eq[r] * n + j] * xx[j]; rp[r] = t; }
    double mu = 0.0;
    for (int r = 0; r < mi; ++r) { rs[r] = Dx(xx, r) + s[r] - fin[r]; mu += s[r] * z[r]; }
    if (mi > 0) mu /= mi;
    double rn = 0.0;
    for (double v : rd) rn = std::max(rn, std::fabs(v));
    for (double v : rp) rn = std::max(rn, std::fabs(v));
    for (double v : rs) rn = std::max(rn, std::fabs(v));
    if (!std::isfinite(rn)) { status = 3; break; }
    {
      // termination: relative residuals 1e-11, complementarity 1e-13 (tighter than the CUDA solver's 1e-10 / 1e-12)
      double gs = 1.0, bs = 1.0, rdn = 0.0, rpn = 0.0;
      for (int i = 0; i < n; ++i) gs = std::max(gs, 1.0 + std::fabs(g[i]));
      for (double v : beq) bs = std::max(bs, 1.0 + std::fabs(v));
      for (double v : fin) bs = std::max(bs, 1.0 + std::fabs(v));
      for (double v : rd) rdn = std::max(rdn, std::fabs(v));
      for (double v : rp) rpn = std::max(rpn, std::fabs(v));
      for (double v : rs) rpn = std::max(rpn, std::fabs(v));
      if (rdn < 1e-11 * gs && rpn < 1e-11 * bs && mu < 1e-13) { status = 0; break; }
    }
    // KKT matrix
    std::vector<double> K0(nk * nk, 0.0);
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) K0[i * nk + j] = H[i * n + j] + (i == j ? rho : 0.0);
    for (int r = 0; r < mi; ++r) {
      const double w = z[r] / s[r];
      for (int i = 0; i < n; ++i) { const double di = Din[r][i]; if (di == 0.0) continue; for (int j = 0; j < n; ++j) K0[i * nk + j] += w * di * Din[r][j]; }
    }
    for (int r = 0; r < me; ++r) for (int j = 0; j < n; ++j) { K0[(n + r) * nk + j] = A[eq[r] * n + j]; K0[j * nk + n + r] = A[eq[r] * n + j]; }
    auto solve_dir = [&](const std::vector<double>& rc, std::vector<double>& dx, std::vector<double>& dy, std::vector<double>& ds, std::vector<double>& dz) {
      std::vector<double> rhs(nk), Kc = K0;
      for (int i = 0; i < n; ++i) {
        double t = -rd[i];
        for (int r = 0; r < mi; ++r) t += Din[r][i] * ((rc[r] - z[r] * rs[r]) / s[r]);
        rhs[i] = t;
      }
      for (int r = 0; r < me; ++r) rhs[n + r] = -rp[r];
      if (!lu_solve(Kc, nk, rhs)) return false;
      for (int i = 0; i < n; ++i) dx[i] = rhs[i];
      for (int r = 0; r < me; ++r) dy[r] = rhs[n + r];
      for (int r = 0; r < mi; ++r) { ds[r] = -rs[r] - Dx(dx, r); dz[r] = -(rc[r] + z[r] * ds[r]) / s[r]; }
      return true;
    };
    auto max_step = [&](const std::vector<double>& ds, const std::vector<double>& dz) {
      double a = 1.0;
      for (int r = 0; r < mi; ++r) { if (ds[r] < 0.0) a = std::min(a, -s[r] / ds[r]); if (dz[r] < 0.0) a = std::min(a, -z[r] / dz[r]); }
      return a;
    };
    std::vector<double> dx(n), dy(me), ds(mi), dz(mi), rc(mi);
    for (int r = 0; r < mi; ++r) rc[r] = s[r] * z[r];
    if (!solve_dir(rc, dx, dy, ds, dz)) { status = 3; break; }
    double sigma = 0.0;
    if (mi > 0) {
      const double a_aff = max_step(ds, dz);
      double mu_aff = 0.0;
      for (int r = 0; r < mi; ++r) mu_aff += (s[r] + a_aff * ds[r]) * (z[r] + a_aff * dz[r]);
      mu_aff /= mi;
      sigma = std::pow(mu_aff / mu, 3.0);
      for (int r = 0; r < mi; ++r) rc[r] = s[r] * z[r] + ds[r] * dz[r] - sigma * mu;
      if (!solve_dir(rc, dx, dy, ds, dz)) { status = 3; break; }
    }
    const double a = std::min(1.0, 0.995 * max_step(ds, dz));
    for (int i = 0; i < n; ++i) xx[i] += a * dx[i];
    for (int r = 0; r < me; ++r) y[r] += a * dy[r];
    for (int r = 0; r < mi; ++r) { s[r] += a * ds[r]; z[r] += a * dz[r]; }
  }
  for (int i = 0; i < n; ++i) x[i] = xx[i];
  if (iters_out) *iters_out = it;
  return status;
}

template <class F>
void parallel_for(int B, int threads, F fn) {
  if (threads <= 1) { for (int i = 0; i < B; ++i) fn(i); return; }
  std::vector<std::thread> th;
  for (int t = 0; t < threads; ++t) th.emplace_back([=]() { for (int i = t; i < B; i += threads) fn(i); });
  for (auto& t : th) t.join();
}

}  // namespace

extern "C" {

void hbo_init(void) {
  if (g_init) return;
  // initializeInputCostWeight (LeggedInterface.cpp:263-288): R = blkdiag(R_f, J0^T R_v J0), J0 at initialState
  double q[NQ];
  for (int i = 0; i < NQ; ++i) q[i] = HB_INITIAL_STATE[6 + i];
  Kin<double> kin; forward_kinematics(q, kin);
  double J0[12 * NJ];
  for (int j = 0; j < NJ; ++j) {
    double e[NQ] = {0}; e[6 + j] = 1.0;
    Vel<double> ve; velocities(kin, e, ve);
    for (int c = 0; c < NC; ++c) { double vc[3]; contact_velocity(kin, ve, c, vc); for (int a = 0; a < 3; ++a) J0[(3 * c + a) * NJ + j] = vc[a]; }
  }
  std::fill(g_R, g_R + NU * NU, 0.0);
  for (int i = 0; i < 12; ++i) g_R[i * NU + i] = HB_R_TASKSPACE_DIAG[i];
  for (int i = 0; i < NJ; ++i) for (int j = 0; j < NJ; ++j) {
    double s = 0.0; for (int r = 0; r < 12; ++r) s += J0[r * NJ + i] * HB_R_TASKSPACE_DIAG[12 + r] * J0[r * NJ + j];
    g_R[(12 + i) * NU + 12 + j] = s;
  }
  g_init = true;
}

// 17 doubles in the order of hb_wbc_settings (include/hunter_b200.h); NULL restores the shipped values
void hbo_set_wbc_settings(const double* s) {
  static const WbcSettings defaults = g_wbc;
  if (!s) { g_wbc = defaults; return; }
  std::memcpy(&g_wbc, s, sizeof(WbcSettings));
}

void hbo_input_cost_R(double* R) { hbo_init(); std::memcpy(R, g_R, sizeof(g_R)); }

void hbo_rbd(const double* q, const double* v, double* M, double* nle, double* J, double* dJv, double* A, double* com,
             double* h, double* cpos) {
  Kin<double> kin; forward_kinematics(q, kin);
  double zero[NQ] = {0};
  for (int c = 0; c < NQ; ++c) {
    double e[NQ] = {0}, col[NQ]; e[c] = 1.0;
    rnea(q, zero, e, false, col, &kin);
    for (int r = 0; r < NQ; ++r) M[r * NQ + c] = col[r];
    Vel<double> ve; velocities(kin, e, ve);
    for (int i = 0; i < NC; ++i) { double vc[3]; contact_velocity(kin, ve, i, vc); for (int a = 0; a < 3; ++a) J[(3 * i + a) * NQ + c] = vc[a]; }
  }
  rnea(q, v, zero, true, nle, &kin);
  center_of_mass(kin, com);
  centroidal_matrix(kin, com, A);
  Vel<double> vel; velocities(kin, v, vel);
  centroidal_momentum(kin, vel, com, h);
  for (int i = 0; i < NC; ++i) contact_position(kin, i, cpos + 3 * i);
  using D1 = Dual<1>;
  D1 qd[NQ], vd[NQ];
  for (int i = 0; i < NQ; ++i) { qd[i].v = q[i]; qd[i].d[0] = v[i]; vd[i] = D1(v[i]); }
  Kin<D1> kd; forward_kinematics(qd, kd);
  Vel<D1> ud; velocities(kd, vd, ud);
  for (int i = 0; i < NC; ++i) { D1 vc[3]; contact_velocity(kd, ud, i, vc); for (int a = 0; a < 3; ++a) dJv[3 * i + a] = vc[a].d[0]; }
}

// Terms of the momentum observer (StateEstimateBase.cpp:130-206, Pinocchio calls :157-166 restated): p = M v, generalised gravity g,
// C' v = (dM/dt - C) v with dM/dt v from a dual number seeded ALONG v and C v from inverse dynamics (a different route than the device
// code, which differentiates the kinetic energy per coordinate), and the 6-D toe-frame Jacobians (LOCAL_WORLD_ALIGNED) of both feet.
void hbo_observer_terms(const double* q, const double* v, double* p, double* g, double* ctv, double* Jfoot /*2 x 6 x 16*/) {
  double zero[NQ] = {0};
  Kin<double> kin; forward_kinematics(q, kin);
  rnea(q, zero, v, false, p, &kin);
  rnea(q, zero, zero, true, g, &kin);
  double cv[NQ];
  rnea(q, v, zero, false, cv, &kin);
  using D1 = Dual<1>;
  D1 qd[NQ], zd[NQ], vd[NQ], pd[NQ];
  for (int i = 0; i < NQ; ++i) { qd[i].v = q[i]; qd[i].d[0] = v[i]; zd[i] = D1(0.0); vd[i] = D1(v[i]); }
  rnea<D1>(qd, zd, vd, false, pd);
  for (int i = 0; i < NQ; ++i) ctv[i] = pd[i].d[0] - cv[i];
  for (int f = 0; f < 2; ++f) {
    for (int c = 0; c < NQ; ++c) {
      double e[NQ] = {0}; e[c] = 1.0;
      Vel<double> ve; velocities(kin, e, ve);
      double vc[3]; contact_velocity(kin, ve, f, vc);
      const int b = HB_CONTACT_BODY[f];
      for (int a = 0; a < 3; ++a) { Jfoot[(f * 6 + a) * NQ + c] = vc[a]; Jfoot[(f * 6 + 3 + a) * NQ + c] = ve.w[b][a]; }
    }
  }
}

// computeCentroidalStateFromRbdModel (LeggedController.cpp:336; App. C.2)
void hbo_rbd_to_centroidal(const double* rbd, double* x) {
  double q[NQ], v[NQ];
  rbd_to_qv(rbd, q, v);
  Kin<double> kin; forward_kinematics(q, kin);
  double com[3]; center_of_mass(kin, com);
  Vel<double> vel; velocities(kin, v, vel);
  double h[6]; centroidal_momentum(kin, vel, com, h);
  for (int i = 0; i < 6; ++i) x[i] = h[i] / HB_TOTAL_MASS;
  for (int i = 0; i < NQ; ++i) x[6 + i] = q[i];
}

void hbo_flow_map(const double* x, const double* u, double* f, double* A, double* B) {
  if (A || B) {
    FlowLin l; flow_map_lin(x, u, l);
    std::memcpy(f, l.f, sizeof(l.f));
    if (A) std::memcpy(A, l.A, sizeof(l.A));
    if (B) std::memcpy(B, l.B, sizeof(l.B));
  } else {
    flow_map_T<double>(x, u, f, nullptr, nullptr);
  }
}

void hbo_ee_kinematics(const double* x, const double* u, double* pos, double* vel, double* dpos_dx, double* dvel_dx, double* dvel_du) {
  FlowLin l; flow_map_lin(x, u, l);
  std::memcpy(pos, l.epos, sizeof(l.epos)); std::memcpy(vel, l.evel, sizeof(l.evel));
  if (dpos_dx) std::memcpy(dpos_dx, l.dpos_dx, sizeof(l.dpos_dx));
  if (dvel_dx) std::memcpy(dvel_dx, l.dvel_dx, sizeof(l.dvel_dx));
  if (dvel_du) std::memcpy(dvel_du, l.dvel_du, sizeof(l.dvel_du));
}

void hbo_node_lq(double dt, const double* x, const double* u, const double* xn, const double* xref, const double* swing, int mode,
                 double* Ad, double* Bd, double* b, double* Q, double* R, double* P, double* q, double* r, double* C, double* D,
                 double* e, int* m, double* cost) {
  hbo_init();
  static thread_local NodeLQ lq;
  node_lq(dt, x, u, xn, xref, swing, mode, lq);
  std::memcpy(Ad, lq.Ad, sizeof(lq.Ad)); std::memcpy(Bd, lq.Bd, sizeof(lq.Bd)); std::memcpy(b, lq.b, sizeof(lq.b));
  std::memcpy(Q, lq.Q, sizeof(lq.Q)); std::memcpy(R, lq.R, sizeof(lq.R)); std::memcpy(P, lq.P, sizeof(lq.P));
  std::memcpy(q, lq.q, sizeof(lq.q)); std::memcpy(r, lq.r, sizeof(lq.r));
  std::memcpy(C, lq.C, sizeof(lq.C)); std::memcpy(D, lq.D, sizeof(lq.D)); std::memcpy(e, lq.e, sizeof(lq.e));
  *m = lq.m; *cost = lq.cost;
}

void hbo_mpc_iteration(const hbo_horizon* hz, int max_trials, const double* x0, const double* x_ref, const double* swing, const int32_t* mode,
                       double* x_traj, double* u_traj, hbo_solve_info* info, hbo_ls_trial* trials) {
  hbo_init();
  mpc_iteration(*hz, x0, x_ref, swing, mode, x_traj, u_traj, info, max_trials, trials);
}

// LeggedRobotInitializer::compute (initialization/LeggedRobotInitializer.cpp:67-77): x_{k+1} = x_k, u = weight compensation
void hbo_mpc_cold_start(const hbo_horizon* hz, const double* x0, const int32_t* mode, double* x_traj, double* u_traj) {
  for (int k = 0; k <= hz->N; ++k) for (int i = 0; i < NX; ++i) x_traj[k * NX + i] = x0[i];
  for (int k = 0; k < hz->N; ++k) weight_compensating_input(mode[k], u_traj + k * NU);
}

void hbo_wbc_assemble(const double* x_des, const double* u_des, const double* rbd, int mode, int stance_mode, double* H, double* g,
                      double* A, double* lbA, double* ubA, int* m) {
  static thread_local WbcQP qp;
  wbc_assemble(x_des, u_des, rbd, mode, stance_mode != 0, qp);
  std::memcpy(H, qp.H, sizeof(qp.H)); std::memcpy(g, qp.g, sizeof(qp.g));
  std::memcpy(A, qp.A, sizeof(double) * qp.m * 38);
  std::memcpy(lbA, qp.lbA, sizeof(double) * qp.m); std::memcpy(ubA, qp.ubA, sizeof(double) * qp.m);
  *m = qp.m;
}

void hbo_wbc_terms(const double* x_des, const double* u_des, const double* rbd, int mode, double* Aw, double* bw, int* rw, double* J, double* dJv) {
  static thread_local WbcQP qp;
  static thread_local WbcTerms t;
  wbc_assemble(x_des, u_des, rbd, mode, false, qp, &t);
  std::memcpy(Aw, t.Aw, sizeof(t.Aw)); std::memcpy(bw, t.bw, sizeof(t.bw)); *rw = t.rw;
  std::memcpy(J, t.J, sizeof(t.J)); std::memcpy(dJv, t.dJv, sizeof(t.dJv));
}

int hbo_qp_solve(int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA, double rho,
                 double* x, int* iters) {
  return qp_solve(n, m, H, g, A, lbA, ubA, rho, x, iters);
}

int hbo_wbc_solve(const double* x_des, const double* u_des, const double* rbd, int mode, int stance_mode, double rho, double* sol) {
  static thread_local WbcQP qp;
  wbc_assemble(x_des, u_des, rbd, mode, stance_mode != 0, qp);
  return qp_solve(38, qp.m, qp.H, qp.g, qp.A, qp.lbA, qp.ubA, rho, sol, nullptr);
}

void hbo_mpc_iteration_batch(const hbo_horizon* hz, int B, int threads, const double* x0, const double* x_ref, const double* swing,
                             const int32_t* mode, double* x_traj, double* u_traj, hbo_solve_info* info) {
  hbo_init();
  const int N = hz->N;
  parallel_for(B, threads, [=](int i) {
    mpc_iteration(*hz, x0 + (size_t)i * NX, x_ref + (size_t)i * (N + 1) * NX, swing + (size_t)i * (N + 1) * 24, mode + (size_t)i * (N + 1),
                  x_traj + (size_t)i * (N + 1) * NX, u_traj + (size_t)i * N * NU, info ? info + i : nullptr);
  });
}

void hbo_wbc_solve_batch(int B, int threads, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                         const uint8_t* stance_mode, double rho, double* sol, int32_t* status) {
  parallel_for(B, threads, [=](int i) {
    int st = hbo_wbc_solve(x_des + (size_t)i * NX, u_des + (size_t)i * NU, rbd + (size_t)i * 32, mode[i], stance_mode ? stance_mode[i] : 0, rho,
                           sol + (size_t)i * 38);
    if (status) status[i] = st;
  });
}

void hbo_wbc_qp_batch(int B, int threads, int n, int m, const double* H, const double* g, const double* A, const double* lbA,
                      const double* ubA, double rho, double* x, int32_t* status) {
  parallel_for(B, threads, [=](int i) {
    int st = qp_solve(n, m, H + (size_t)i * n * n, g + (size_t)i * n, A + (size_t)i * m * n, lbA + (size_t)i * m, ubA + (size_t)i * m, rho,
                      x + (size_t)i * n, nullptr);
    if (status) status[i] = st;
  });
}

}  // extern "C"
