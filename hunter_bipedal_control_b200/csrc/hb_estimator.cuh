// State estimation on the device (SURVEY 8f row N3): the linear Kalman filter of legged_estimation and the generalised-momentum
// contact-force observer of StateEstimateBase. One warp per instance.
#pragma once
#include "hb_common.cuh"
#include "hb_planner.h"
#include "hb_qp.cuh"
#include "hb_rbd.cuh"
#include "hb_rollout.cuh"
#include "../../include/hunter_b200.h"

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
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
// the filter state of one instance: hb_estimator_update_batch passes hb_kf_state[], the estimated episodes their hb_estimation_state[]
__device__ __forceinline__ hb_kf_state& kf_of(hb_kf_state& s) { return s; }
__device__ __forceinline__ hb_kf_state& kf_of(hb_estimation_state& s) { return s.kf; }
// The contact positions fk (12) with the base at the origin, at the ZYX angles zyx and the joint readings jp: the filter's kinematics (:84-100),
// which are Pinocchio's at (pos, zyx, q) less pos. Not inlined: kf_update_kernel's fusion and odometry_fuse_kernel run this one compiled body,
// so that the episode and hb_estimator_fuse_odometry give the same bits (inlined into each kernel, kin_pass's sums may round differently).
__device__ __noinline__ void odom_contact_positions(const double* zyx, const double* jp, double* fk) {
  double q[NQ], v[NQ];
  for (int i = 0; i < NQ; ++i) { q[i] = i < 3 ? 0.0 : (i < 6 ? zyx[i - 3] : jp[i - 6]); v[i] = 0.0; }
  KinOut<double> o;
  kin_pass<double>(q, v, o);
  for (int i = 0; i < 12; ++i) fk[i] = o.cpos[i];
}
// KalmanFilterEstimate::updateFromTopic (:186-235) with the camera at the base origin: x_hat[i] after the fusion of the message position pos,
// for i outside the velocity rows 3..5; fk from odom_contact_positions.
__device__ __forceinline__ double odom_fused_state(int i, const double* pos, const double* fk, double foot_radius) {
  if (i < 3) return pos[i];
  const int k = (i - 6) % 3;
  const double p = pos[k] + fk[i - 6];
  return k == 2 ? p - foot_radius : p;
}
// Odom (estimated episodes with hb_rollout_set_odometry): odom_pos / odom_has (B x 3 / B) are the odometry messages of the tick, and an
// instance with odom_has[i] != 0 is fused after the filter step (odom_fused_state; feet heights of the contact feet follow, velocity and P
// stay). Without Odom the pointers are not read and the kernel has no call to odom_contact_positions, whose call site costs registers.
// maps: the estimator maps (hb_estimator_set_maps). An instance with a map measures foot c's height (row 24 + c) as the map's height under
// the predicted foot, hbplan::map_height at x[6 + 3c], x[7 + 3c], in place of feet_heights[c], which it then does not read; the fusion
// above still writes it.
template <class State, bool Odom>
__global__ void __launch_bounds__(32) kf_update_kernel(int B, hb_kf_params prm, double dt, State* state, const double* quat, const double* angl,
                                                       const double* accl, const double* jpos, const double* jvel, const uint8_t* cflag, double* rbd_out,
                                                       const double* odom_pos, const uint8_t* odom_has, InstanceView<hb_terrain> maps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  KfShared& sh = *reinterpret_cast<KfShared*>(smem_raw);
  const int inst = blockIdx.x, lane = threadIdx.x;
  hb_kf_state& st = kf_of(state[inst]);
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
  const double rates[3] = {dzr, dyr, dxr};
  double wg[3];
  world_omega_from_zyx_rates(sz, cz, sy, cy, rates, wg);
  // ---- contact kinematics with the base at the origin and zero base linear velocity (:84-100)
  double q[NQ], v[NQ];
  q[0] = q[1] = q[2] = 0.0; q[3] = zyx[0]; q[4] = zyx[1]; q[5] = zyx[2];
  v[0] = v[1] = v[2] = 0.0;
  zyx_rates_from_world_omega(sz, cz, sy, cy, wg, &v[3]);
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
  // innovation y - C x (:137-143): ps = -eePos (+ footRadius on z), vs = -eeVel, feet heights (on a map: the ground under the predicted foot)
  const hb_terrain* map = maps.of(inst);
  if (lane < 28) {
    double y;
    if (lane < 12) y = -ko.cpos[lane] + ((lane % 3) == 2 ? prm.foot_radius : 0.0);
    else if (lane < 24) y = -ko.cvel[lane - 12];
    else if (map) y = hbplan::map_height(map, sh.x[6 + 3 * (lane - 24)], sh.x[7 + 3 * (lane - 24)]);
    else y = st.feet_heights[lane - 24];
    sh.ey[lane] = y - kf_c_row(sh.x, 1, lane, 0);
  }
  // the fused state of this lane's row, written after the filter step
  const bool fuse = Odom && odom_has[inst];
  double xf = 0.0;
  if (fuse && lane < 18 && (lane < 3 || lane >= 6)) {
    double fk[12];
    odom_contact_positions(zyx, &q[6], fk);
    xf = odom_fused_state(lane, odom_pos + (size_t)inst * 3, fk, prm.foot_radius);
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
  // :169-173: updateFromTopic after the decoupling; a contact foot's height follows its fused position
  const bool fused_row = fuse && (lane < 3 || lane >= 6);
  const double xo = fused_row ? xf : (lane < 18 ? sh.x[lane] : 0.0);
  if (lane < 18) st.x_hat[lane] = xo;
  if (fused_row && lane >= 6 && lane < 18 && (lane - 6) % 3 == 2 && cflag[4 * inst + (lane - 6) / 3]) st.feet_heights[(lane - 6) / 3] = xo;
  // ---- rbd state (StateEstimateBase.cpp:73-106, updateLinear after the fusion): [zyx, p, q_j, omega_world, v, qd_j]
  double* rb = rbd_out + (size_t)inst * 32;
  if (lane < 3) { rb[lane] = zyx[lane]; rb[3 + lane] = xo; rb[16 + lane] = wg[lane]; rb[19 + lane] = sh.x[3 + lane]; }
  if (lane < NJ) { rb[6 + lane] = q[6 + lane]; rb[22 + lane] = v[6 + lane]; }
}

// hb_estimator_fuse_odometry: kf_update_kernel's fusion on its outputs, one thread per instance. The filter's angles and joint readings are
// the estimated rbd's.
__global__ void odometry_fuse_kernel(int B, double foot_radius, hb_kf_state* state, const double* pos, const uint8_t* has, const uint8_t* cflag,
                                     double* rbd) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B || !has[inst]) return;
  hb_kf_state& st = state[inst];
  double* rb = rbd + (size_t)inst * 32;
  const double* p = pos + (size_t)inst * 3;
  double fk[12];
  odom_contact_positions(rb, rb + 6, fk);
  for (int i = 0; i < 18; ++i) if (i < 3 || i >= 6) st.x_hat[i] = odom_fused_state(i, p, fk, foot_radius);
  for (int c = 0; c < 4; ++c) if (cflag[4 * inst + c]) st.feet_heights[c] = st.x_hat[8 + 3 * c];
  for (int k = 0; k < 3; ++k) rb[3 + k] = p[k];
}

// StateEstimateBase::estContactForce (legged_estimation/src/StateEstimateBase.cpp:130-206): generalised-momentum observer
//   p = M v,  pSCg = beta p + S' tau_cmd + C' v - g,  low-pass (gamma = exp(-lambda dt), beta = (1 - gamma) / (gamma dt)),  tau_d = beta p - filtered,
// then per foot the least-norm 6-D wrench w with (S_leg J_foot') w = S_leg tau_d (5 joint rows of the leg, toe frame Jacobian in world axes).
// One warp per instance; the terms Pinocchio provides are obtained as
//   M v  = inverse dynamics with acceleration v at zero velocity, no gravity;   g = inverse dynamics at rest with gravity;
//   C' v = d/dq (1/2 v' M(q) v) at fixed v (lane i = dual sweep seeded on q_i; valid for any C with dM/dt = C + C', as Pinocchio's).
// One observer step of one instance on its warp (every lane calls it): p_filtered (16) advanced, est (16) and disturbance (16, nullable)
// written, from the rbd r (32) and the torques tau (10). Not inlined: contact_force_kernel and the estimated episodes' contact_observe_kernel
// run this one compiled body, so that the episode and hb_contact_force_estimate_batch give the same bits (as odom_contact_positions).
struct ObsShared { double p[NQ], g[NQ], ctv[NQ], taud[NQ], Jf[2 * 5 * 6]; };
__device__ __noinline__ void observer_step(ObsShared& sh, int lane, double lambda, double dt_in, double* p_filtered, const double* r, const double* tau,
                                           double* e, double* disturbance) {
  const double dt = dt_in > 1.0 ? 0.002 : dt_in;
  const double gama = exp(-lambda * dt), beta = (1.0 - gama) / (gama * dt);
  double q[NQ], v[NQ];
  rbd_to_qv(r, q, v);
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
  if (lane < NQ) {
    const double p = sh.p[lane];
    const double pscg = beta * p + (lane >= 6 ? tau[lane - 6] : 0.0) + sh.ctv[lane] - sh.g[lane];
    const double filt = (1.0 - gama) * pscg + gama * p_filtered[lane];
    p_filtered[lane] = filt;
    const double td = beta * p - filt;
    sh.taud[lane] = td;
    if (disturbance) disturbance[lane] = td;
  }
  __syncwarp();
  if (lane < 2) {
    // least-norm solution of A w = b, A = S J' (5 x 6), as the reference's SVD solve gives it: Householder QR of A' = Q [R; 0], then
    // w = Q [R^-T b; 0]. A loses rank inside the joint limits (knee ~0.0208 rad, where the hip-pitch, knee and ankle origins line up,
    // cond(A) ~ 1.8 / |knee - k*|); this solve is backward stable, so the error in w grows like cond(A) eps, where the normal equations
    // A A' y = b it replaces squared the condition number.
    const double* A = sh.Jf + lane * 30;          // row j = joint j of the leg, 6 columns
    double M[6][5], vd[5], bt[5], rd[5];          // M = A'; below the diagonal: Householder vectors (leading entries vd), rd = diag R
#pragma unroll
    for (int c = 0; c < 6; ++c)
#pragma unroll
      for (int j = 0; j < 5; ++j) M[c][j] = A[j * 6 + c];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      double nn = 0.0;
#pragma unroll
      for (int i = k; i < 6; ++i) nn = fma(M[i][k], M[i][k], nn);
      const double n = sqrt(nn), x0 = M[k][k];
      const double alpha = x0 >= 0.0 ? -n : n;    // reflect onto -sign(x0) |x| e_k: v_0 = x0 - alpha has no cancellation
      vd[k] = x0 - alpha;
      bt[k] = n > 0.0 ? 1.0 / (n * (n + fabs(x0))) : 0.0;      // 2 / (v' v)
      rd[k] = alpha;
#pragma unroll
      for (int j = k + 1; j < 5; ++j) {
        double s = vd[k] * M[k][j];
#pragma unroll
        for (int i = k + 1; i < 6; ++i) s = fma(M[i][k], M[i][j], s);
        s *= bt[k];
        M[k][j] -= s * vd[k];
#pragma unroll
        for (int i = k + 1; i < 6; ++i) M[i][j] = fma(-s, M[i][k], M[i][j]);
      }
    }
    double w[6];                                  // R' y = b (forward), then w = H_0 ... H_4 [y; 0]
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      double s = sh.taud[6 + 5 * lane + i];
#pragma unroll
      for (int j = 0; j < i; ++j) s = fma(-M[j][i], w[j], s);
      w[i] = s / rd[i];
    }
    w[5] = 0.0;
#pragma unroll
    for (int k = 4; k >= 0; --k) {
      double s = vd[k] * w[k];
#pragma unroll
      for (int i = k + 1; i < 6; ++i) s = fma(M[i][k], w[i], s);
      s *= bt[k];
      w[k] -= s * vd[k];
#pragma unroll
      for (int i = k + 1; i < 6; ++i) w[i] = fma(-s, M[i][k], w[i]);
    }
    double n3 = 0.0, n6 = 0.0;
    for (int c = 0; c < 6; ++c) { n6 += w[c] * w[c]; if (c < 3) n3 += w[c] * w[c]; }
    for (int c = 0; c < 6; ++c) e[6 * lane + c] = w[c];
    e[12 + lane] = sqrt(n3);
    e[14 + lane] = sqrt(n6);
  }
}
__global__ void __launch_bounds__(32) contact_force_kernel(int B, double lambda, double dt_in, hb_observer_state* state, const double* rbd, const double* tau_cmd,
                                                           double* est, double* disturbance) {
  __shared__ ObsShared sh;
  const int inst = blockIdx.x;
  observer_step(sh, threadIdx.x, lambda, dt_in, state[inst].p_filtered, rbd + (size_t)inst * 32, tau_cmd + (size_t)inst * NJ, est + (size_t)inst * 16,
                disturbance ? disturbance + (size_t)inst * NQ : nullptr);
}

// Step (4) of an estimated tick with contact detection (hunter_b200.h): the observer of each instance with a record, on its estimated rbd
// with its stored effort, into its stored output. One warp per instance; the others return.
__global__ void __launch_bounds__(32) contact_observe_kernel(int B, double dt, InstanceView<hb_contact_detection> set, ContactDetectState* st,
                                                             const double* rbd) {
  __shared__ ObsShared sh;
  const int inst = blockIdx.x;
  const hb_contact_detection* r = set.of(inst);
  if (!r) return;
  ContactDetectState& d = st[inst];
  observer_step(sh, threadIdx.x, r->cutoff_frequency, dt, d.p_filtered, rbd + (size_t)inst * 32, d.effort, d.force, nullptr);
}
}  // namespace
