// Lane-level pieces of the SQP iteration shared by the node-parallel pipeline in hb_sqp.cuh (what ocs2::SqpSolver::run does for
// sqpIteration = 1, legged_controllers/src/LeggedController.cpp:378-379,406; SURVEY 8a rows M1-M12, S1-S7):
//   penalties (relaxed barrier, double sided), and the VALUE-only evaluations the filter line search runs with one lane per
//   horizon node: the centroidal flow map (flow_map_lane) and the stage cost / equality-constraint values (node_values_lane).
#pragma once
#include "hb_common.cuh"
#include "hb_planner.h"
#include "hb_rbd.cuh"

namespace hb {

constexpr int TS = NX * NX;        // one 22x22 tile
constexpr int NDIR = 13;           // non-trivial configuration directions: euler(3) + joints(10)

// ------------------------------------------------------------------ penalties (SURVEY App. C.4)
struct Pen { double v, d1, d2; };
__device__ __forceinline__ Pen relaxed_barrier(double h, double mu, double delta) {
  Pen p;
  if (h > delta) { p.v = -mu * log(h); p.d1 = -mu / h; p.d2 = mu / (h * h); }
  else {
    const double z = (h - 2.0 * delta) / delta;
    p.v = mu * (-log(delta) + 0.5 * z * z - 0.5);
    p.d1 = mu * (h - 2.0 * delta) / (delta * delta);
    p.d2 = mu / (delta * delta);
  }
  return p;
}
__device__ __forceinline__ Pen double_sided(double h, double lo, double hi, double mu, double delta) {
  const Pen a = relaxed_barrier(h - lo, mu, delta), b = relaxed_barrier(hi - h, mu, delta);
  Pen p; p.v = a.v + b.v; p.d1 = a.d1 - b.d1; p.d2 = a.d2 + b.d2;
  return p;
}

// ------------------------------------------------------------------ centroidal flow map, one lane = one evaluation
// (used by the line search: lane-per-node). x = [hbar(6), q(16)], u = [F(12), qj_dot(10)]   (SURVEY App. C.2)
// ONE sweep over the kinematic tree per evaluation. The base twist solves A_b v_b = m hbar - A_j qj_dot; instead of probing the columns of
// the centroidal momentum matrix with unit velocities (five sweeps in round 1: joint momentum, three Euler-rate columns, contact
// velocities) the sweep runs with the base at rest and accumulates, next to the joint momentum A_j qj_dot, the rotational inertia of the
// whole robot about the origin. For a rigid motion (v0, w) of the base the momentum is [m (v0 + w x (com - p0)); I_C w] with
// I_C = I_O - m (|com|^2 1 - com com'), so A[:, 0:3] = [m I; 0] (computeFloatingBaseCentroidalMomentumMatrixInverse) and the Euler-rate
// columns are [m w_c x (com - p0); I_C w_c] with w_c the world axis of Euler rate c. Velocities are linear in v, so the contact
// velocities are the base-at-rest ones plus v0 + W x (cpos - p0).
__device__ inline void flow_map_lane(const double* x, const double* u, double* f, double* epos, double* evel) {
  const Model& md = c_model;
  const double m = md.total_mass;
  double R0[9], ax0[9];
  {
    double sz, cz, sy, cy, sx, cx;
    sincos_t(x[9], sz, cz); sincos_t(x[10], sy, cy); sincos_t(x[11], sx, cx);
    R0[0] = cz * cy; R0[1] = cz * sy * sx - sz * cx; R0[2] = cz * sy * cx + sz * sx;
    R0[3] = sz * cy; R0[4] = sz * sy * sx + cz * cx; R0[5] = sz * sy * cx - cz * sx;
    R0[6] = -sy;     R0[7] = cy * sx;                R0[8] = cy * cx;
    ax0[0] = 0.0; ax0[1] = 0.0; ax0[2] = 1.0;
    ax0[3] = -sz; ax0[4] = cz; ax0[5] = 0.0;
    ax0[6] = cz * cy; ax0[7] = sz * cy; ax0[8] = -sy;
  }
  const double p0[3] = {x[6], x[7], x[8]};
  double P[3] = {0, 0, 0}, Lo[3] = {0, 0, 0}, mc[3] = {0, 0, 0};
  double IO[6] = {0, 0, 0, 0, 0, 0};    // xx xy xz yy yz zz about the origin
  double cp[12], cvj[12];
  // mass, first moment and rotational inertia of body b (world frame, about the origin)
  auto add_inertia = [&](int b, const double* R, const double* cw) {
    const double mb = md.mass[b];
    const double* I = &md.inertia[9 * b];
    double T[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) T[3 * i + k] = R[3 * i] * I[k] + R[3 * i + 1] * I[3 + k] + R[3 * i + 2] * I[6 + k];
    const double c2 = cw[0] * cw[0] + cw[1] * cw[1] + cw[2] * cw[2];
    IO[0] += T[0] * R[0] + T[1] * R[1] + T[2] * R[2] + mb * (c2 - cw[0] * cw[0]);
    IO[1] += T[0] * R[3] + T[1] * R[4] + T[2] * R[5] - mb * cw[0] * cw[1];
    IO[2] += T[0] * R[6] + T[1] * R[7] + T[2] * R[8] - mb * cw[0] * cw[2];
    IO[3] += T[3] * R[3] + T[4] * R[4] + T[5] * R[5] + mb * (c2 - cw[1] * cw[1]);
    IO[4] += T[3] * R[6] + T[4] * R[7] + T[5] * R[8] - mb * cw[1] * cw[2];
    IO[5] += T[6] * R[6] + T[7] * R[7] + T[8] * R[8] + mb * (c2 - cw[2] * cw[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) mc[i] += cw[i] * mb;
  };
  {
    double r[3], cw[3];
    rot_const(R0, &md.com[0], r);
#pragma unroll
    for (int i = 0; i < 3; ++i) cw[i] = p0[i] + r[i];
    add_inertia(0, R0, cw);                       // the base is at rest: no momentum
  }
  for (int leg = 0; leg < 2; ++leg) {
    double R[9], p[3], w[3] = {0, 0, 0}, vl[3] = {0, 0, 0};
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = R0[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) p[i] = p0[i];
    for (int j = 0; j < 5; ++j) {
      const int b = 1 + 5 * leg + j;
      double d[3], wxd[3], a[3], sj, cj;
      rot_const(R, &md.joint_xyz[3 * b], d);
      cross(w, d, wxd);
#pragma unroll
      for (int i = 0; i < 3; ++i) { p[i] += d[i]; vl[i] += wxd[i]; }
      sincos_t(x[11 + b], sj, cj);
      joint_rotate_sc(R, md.joint_axis[b], sj, cj, a);
      const double vb = u[11 + b];
#pragma unroll
      for (int i = 0; i < 3; ++i) w[i] += a[i] * vb;
      double r[3], wxr[3], vc[3], cw[3], l[3], wl[3], Iwl[3], Iw[3];
      rot_const(R, &md.com[3 * b], r);
      cross(w, r, wxr);
      const double mb = md.mass[b];
#pragma unroll
      for (int i = 0; i < 3; ++i) { vc[i] = (vl[i] + wxr[i]) * mb; cw[i] = p[i] + r[i]; }
      cross(cw, vc, l);
      rotT(R, w, wl);
      const double* I = &md.inertia[9 * b];
#pragma unroll
      for (int i = 0; i < 3; ++i) Iwl[i] = wl[0] * I[3 * i] + wl[1] * I[3 * i + 1] + wl[2] * I[3 * i + 2];
      rot(R, Iwl, Iw);
#pragma unroll
      for (int i = 0; i < 3; ++i) { P[i] += vc[i]; Lo[i] += l[i] + Iw[i]; }
      add_inertia(b, R, cw);
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {  // toe (contact leg), heel (contact 2+leg)
      const int c = leg + 2 * t;
      double off[3], wxo[3];
      rot_const(R, &md.contact_offset[3 * c], off);
      cross(w, off, wxo);
#pragma unroll
      for (int i = 0; i < 3; ++i) { cp[3 * c + i] = p[i] + off[i]; cvj[3 * c + i] = vl[i] + wxo[i]; }
    }
  }
  const double im = 1.0 / m;
  double com[3], cxP[3], hj[6];
#pragma unroll
  for (int i = 0; i < 3; ++i) com[i] = mc[i] * im;
  cross(com, P, cxP);
#pragma unroll
  for (int i = 0; i < 3; ++i) { hj[i] = P[i]; hj[3 + i] = Lo[i] - cxP[i]; }
  // inertia about the centre of mass
  const double cc = com[0] * com[0] + com[1] * com[1] + com[2] * com[2];
  const double Ic[9] = {IO[0] - m * (cc - com[0] * com[0]), IO[1] + m * com[0] * com[1], IO[2] + m * com[0] * com[2],
                        IO[1] + m * com[0] * com[1], IO[3] - m * (cc - com[1] * com[1]), IO[4] + m * com[1] * com[2],
                        IO[2] + m * com[0] * com[2], IO[4] + m * com[1] * com[2], IO[5] - m * (cc - com[2] * com[2])};
  const double rb[3] = {com[0] - p0[0], com[1] - p0[1], com[2] - p0[2]};
  double Ae[6][3];  // Euler-rate columns of A
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double* wc = &ax0[3 * c];
    double wxr[3];
    cross(wc, rb, wxr);
#pragma unroll
    for (int i = 0; i < 3; ++i) { Ae[i][c] = m * wxr[i]; Ae[3 + i][c] = Ic[3 * i] * wc[0] + Ic[3 * i + 1] * wc[1] + Ic[3 * i + 2] * wc[2]; }
  }
  double rl[3], ra[3];
  for (int i = 0; i < 3; ++i) { rl[i] = m * x[i] - hj[i]; ra[i] = m * x[3 + i] - hj[3 + i]; }
  // 3x3 solve A22 th = ra (Cramer)
  const double a = Ae[3][0], b = Ae[3][1], c = Ae[3][2], d = Ae[4][0], e = Ae[4][1], g = Ae[4][2], h = Ae[5][0], k = Ae[5][1], l = Ae[5][2];
  const double det = a * (e * l - g * k) - b * (d * l - g * h) + c * (d * k - e * h);
  const double id = 1.0 / det;
  double th[3];
  th[0] = ((e * l - g * k) * ra[0] - (b * l - c * k) * ra[1] + (b * g - c * e) * ra[2]) * id;
  th[1] = (-(d * l - g * h) * ra[0] + (a * l - c * h) * ra[1] - (a * g - c * d) * ra[2]) * id;
  th[2] = ((d * k - e * h) * ra[0] - (a * k - b * h) * ra[1] + (a * e - b * d) * ra[2]) * id;
  double vb[6];
  for (int i = 0; i < 3; ++i) { vb[i] = (rl[i] - Ae[i][0] * th[0] - Ae[i][1] * th[1] - Ae[i][2] * th[2]) / m; vb[3 + i] = th[i]; }
  if (evel) {
    double W[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) W[i] = ax0[i] * th[0] + ax0[3 + i] * th[1] + ax0[6 + i] * th[2];
#pragma unroll
    for (int cc2 = 0; cc2 < NC; ++cc2) {
      const double rr[3] = {cp[3 * cc2] - p0[0], cp[3 * cc2 + 1] - p0[1], cp[3 * cc2 + 2] - p0[2]};
      double wxr[3];
      cross(W, rr, wxr);
#pragma unroll
      for (int i = 0; i < 3; ++i) evel[3 * cc2 + i] = cvj[3 * cc2 + i] + vb[i] + wxr[i];
    }
  }
  if (epos) for (int i = 0; i < 12; ++i) epos[i] = cp[i];
  double fl[3] = {0, 0, 0}, fa[3] = {0, 0, 0};
  for (int cc2 = 0; cc2 < NC; ++cc2) {
    const double* F = u + 3 * cc2;
    const double r0 = cp[3 * cc2] - com[0], r1 = cp[3 * cc2 + 1] - com[1], r2 = cp[3 * cc2 + 2] - com[2];
    fl[0] += F[0]; fl[1] += F[1]; fl[2] += F[2];
    fa[0] += r1 * F[2] - r2 * F[1]; fa[1] += r2 * F[0] - r0 * F[2]; fa[2] += r0 * F[1] - r1 * F[0];
  }
  for (int i = 0; i < 3; ++i) { f[i] = fl[i] * im; f[3 + i] = fa[i] * im; }
  f[2] -= HB_GRAVITY;
  for (int i = 0; i < 6; ++i) f[6 + i] = vb[i];
  for (int j = 0; j < NJ; ++j) f[12 + j] = u[12 + j];
}

// Value of a sum of relaxed log barriers that share (mu, delta): -mu sum log(h_i) over the arguments above delta is -mu log(prod h_i) -- ONE
// logarithm per group instead of one per constraint (52 per node in the line search); arguments at or below delta take the quadratic
// extension term by term. The products stay far inside the double range (<= 20 factors of at most a few hundred each).
struct BarrierSum {
  double prod = 1.0, quad = 0.0;
  __device__ __forceinline__ void add(double h, double delta) {
    if (h > delta) prod *= h;
    else { const double z = (h - 2.0 * delta) / delta; quad += -log(delta) + 0.5 * z * z - 0.5; }
  }
  __device__ __forceinline__ double value(double mu) const { return mu * (quad - log(prod)); }
};

// Stance force (Fx, Fy, Fz) in the surface frame f = (n, t1, t2) of hbplan::surface_frame: the local force t_R_w F = (t1.F, t2.F, n.F)
// of FrictionConeConstraint.cpp:82, which the friction cone bounds on an MPC cone map
__device__ __forceinline__ void cone_local_force(const double* f, double& Fx, double& Fy, double& Fz) {
  const double lx = f[3] * Fx + f[4] * Fy + f[5] * Fz, ly = f[6] * Fx + f[7] * Fy + f[8] * Fz, lz = f[0] * Fx + f[1] * Fy + f[2] * Fz;
  Fx = lx; Fy = ly; Fz = lz;
}

// Stage cost (unscaled) and equality-constraint values of one node, one lane = one node (values only). sth (nullable): the node's four
// stance heights on an MPC map (SqpArgs::sth), which the stance z rows subtract as K1's do. cgr (nullable): the node's four ground
// gradients on an MPC cone map (SqpArgs::cgr); a stance contact on sloped ground has its cone about that ground's frame, as K1's has.
__device__ inline void node_values_lane(const double* x, const double* u, const double* xref, const double* swing, int mode,
                                        const double* epos, const double* evel, const double* sth, const double* cgr, double& cost,
                                        double& eq_sq) {
  const Model& md = c_model;
  bool fl[4]; int ns = 0;
  for (int c = 0; c < 4; ++c) { fl[c] = contact_flag(mode, c); ns += fl[c]; }
  double cst = 0.0;
  for (int i = 0; i < NX; ++i) { const double d = x[i] - xref[i]; cst += 0.5 * md.Q[i] * d * d; }
  double du[NU];
  const double fz = ns > 0 ? md.total_mass * HB_GRAVITY / ns : 0.0;
  for (int i = 0; i < NU; ++i) du[i] = u[i];
  for (int c = 0; c < 4; ++c) if (fl[c]) du[3 * c + 2] -= fz;
  for (int i = 0; i < NU; ++i) { double s = 0.0; for (int j = 0; j < NU; ++j) s += md.R[i * NU + j] * du[j]; cst += 0.5 * du[i] * s; }
  double e2 = 0.0;
  BarrierSum fric, lpos, lvel, lforce;
  for (int c = 0; c < 4; ++c) {
    if (fl[c]) {
      const double Fx = u[3 * c], Fy = u[3 * c + 1], Fz = u[3 * c + 2];
      double h, f[9];
      if (cgr && hbplan::surface_frame(cgr[2 * c], cgr[2 * c + 1], f)) {
        // the cone on the local force; written apart from the flat statement, which keeps its own instructions
        double lx = Fx, ly = Fy, lz = Fz;
        cone_local_force(f, lx, ly, lz);
        h = fma(HB_FRICTION_MU, lz, -sqrt(fma(lx, lx, fma(ly, ly, (double)HB_FRICTION_REGULARIZATION))));
      } else h = HB_FRICTION_MU * Fz - sqrt(Fx * Fx + Fy * Fy + HB_FRICTION_REGULARIZATION);
      fric.add(h, HB_FRICTION_BARRIER_DELTA);
      const double e0 = evel[3 * c], e1 = evel[3 * c + 1];
      double e2z = evel[3 * c + 2] + HB_ZEROVEL_Z_GAIN * epos[3 * c + 2] + HB_ZEROVEL_Z_OFFSET;
      if (sth) e2z -= HB_ZEROVEL_Z_GAIN * sth[c];
      e2 += e0 * e0 + e1 * e1 + e2z * e2z;
    } else {
      for (int a = 0; a < 2; ++a) {
        const double h = evel[3 * c + a] - swing[6 * c + 3 + a] + HB_XY_POSITION_GAIN * (epos[3 * c + a] - swing[6 * c + a]);
        cst += 0.5 * HB_SOFT_SWING_WEIGHT * h * h;
      }
      const double en = evel[3 * c + 2] - swing[6 * c + 5] + HB_POSITION_ERROR_GAIN * (epos[3 * c + 2] - swing[6 * c + 2]);
      e2 += u[3 * c] * u[3 * c] + u[3 * c + 1] * u[3 * c + 1] + u[3 * c + 2] * u[3 * c + 2] + en * en;
    }
  }
  for (int j = 0; j < NJ; ++j) {
    lpos.add(x[12 + j] - md.joint_lower[j], HB_LIMIT_POS_DELTA); lpos.add(md.joint_upper[j] - x[12 + j], HB_LIMIT_POS_DELTA);
    lvel.add(u[12 + j] + md.joint_vel_limit[j], HB_LIMIT_VEL_DELTA); lvel.add(md.joint_vel_limit[j] - u[12 + j], HB_LIMIT_VEL_DELTA);
  }
  for (int c = 0; c < 4; ++c) { lforce.add(u[3 * c + 2], HB_LIMIT_FORCE_DELTA); lforce.add(HB_LIMIT_FORCE_MAX - u[3 * c + 2], HB_LIMIT_FORCE_DELTA); }
  cst += fric.value(HB_FRICTION_BARRIER_MU) + lpos.value(HB_LIMIT_POS_MU) + lvel.value(HB_LIMIT_VEL_MU) + lforce.value(HB_LIMIT_FORCE_MU);
  cost = cst; eq_sq = e2;
}


}  // namespace hb

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
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
}  // namespace
