// Device rigid-body routines for the fixed Hunter tree (what the reference gets from Pinocchio / ocs2_centroidal_model /
// CppAD-generated code: legged_wbc/src/WbcBase.cpp:85-135, legged_interface/src/dynamics/LeggedRobotDynamicsAD.cpp:57-71).
//
// Design: every routine is plain per-lane scalar code templated on the scalar type. The warp gets its parallelism from
// WHAT each lane evaluates, not from cooperation inside the routine:
//   * lane k evaluates with the unit generalised velocity e_k   -> column k of the centroidal momentum matrix A(q)
//                                                                   and of the contact Jacobians J_c(q)
//   * lane k evaluates with a first-order dual number seeded in direction q_k (velocity held fixed)
//                                                                -> d h/dq_k, d com/dq_k, d p_c/dq_k, d (J_c v)/dq_k
//   * lane k evaluates RNEA with unit acceleration e_k            -> column k of the joint-space inertia matrix M(q)
//   * lane k evaluates node k of the horizon (line search)        -> defects / constraint values / costs of 32 nodes at once
// Generalised coordinates: q = [p(3), yaw, pitch, roll, q_j(10)], v = q_dot (SURVEY App. C.1). World axes throughout.
// The state layout is written here once, for every kernel: rbd_to_qv / qv_to_rbd between a measured rbd state and (q, v), on the two
// Euler-rate maps zyx_rates_from_world_omega / world_omega_from_zyx_rates; contact_positions gives the contact frames at a configuration.
#pragma once
#include "hb_common.cuh"

namespace hb {

// first-order dual number (value, one tangent)
struct D1 {
  double v, d;
  __device__ __forceinline__ D1() {}
  __device__ __forceinline__ D1(double a) : v(a), d(0.0) {}
  __device__ __forceinline__ D1(double a, double b) : v(a), d(b) {}
};
__device__ __forceinline__ D1 operator+(D1 a, D1 b) { return D1(a.v + b.v, a.d + b.d); }
__device__ __forceinline__ D1 operator-(D1 a, D1 b) { return D1(a.v - b.v, a.d - b.d); }
__device__ __forceinline__ D1 operator-(D1 a) { return D1(-a.v, -a.d); }
__device__ __forceinline__ D1 operator*(D1 a, D1 b) { return D1(a.v * b.v, fma(a.d, b.v, a.v * b.d)); }
__device__ __forceinline__ D1 operator*(D1 a, double b) { return D1(a.v * b, a.d * b); }
__device__ __forceinline__ D1 operator*(double b, D1 a) { return D1(a.v * b, a.d * b); }
__device__ __forceinline__ D1 operator+(D1 a, double b) { return D1(a.v + b, a.d); }
__device__ __forceinline__ D1 operator-(D1 a, double b) { return D1(a.v - b, a.d); }
__device__ __forceinline__ void sincos_t(double a, double& s, double& c) { sincos(a, &s, &c); }
__device__ __forceinline__ void sincos_t(D1 a, D1& s, D1& c) {
  double sv, cv;
  sincos(a.v, &sv, &cv);
  s = D1(sv, cv * a.d);
  c = D1(cv, -sv * a.d);
}
__device__ __forceinline__ double val(double a) { return a; }
__device__ __forceinline__ double val(D1 a) { return a.v; }

template <class T> __device__ __forceinline__ void cross(const T* a, const T* b, T* c) {
  const T c0 = a[1] * b[2] - a[2] * b[1];
  const T c1 = a[2] * b[0] - a[0] * b[2];
  const T c2 = a[0] * b[1] - a[1] * b[0];
  c[0] = c0; c[1] = c1; c[2] = c2;
}
// y = R x, R row-major 3x3, x constant vector
template <class T> __device__ __forceinline__ void rot_const(const T* R, const double* x, T* y) {
  y[0] = R[0] * x[0] + R[1] * x[1] + R[2] * x[2];
  y[1] = R[3] * x[0] + R[4] * x[1] + R[5] * x[2];
  y[2] = R[6] * x[0] + R[7] * x[1] + R[8] * x[2];
}
template <class T> __device__ __forceinline__ void rot(const T* R, const T* x, T* y) {
  const T y0 = R[0] * x[0] + R[1] * x[1] + R[2] * x[2];
  const T y1 = R[3] * x[0] + R[4] * x[1] + R[5] * x[2];
  const T y2 = R[6] * x[0] + R[7] * x[1] + R[8] * x[2];
  y[0] = y0; y[1] = y1; y[2] = y2;
}
template <class T> __device__ __forceinline__ void rotT(const T* R, const T* x, T* y) {
  const T y0 = R[0] * x[0] + R[3] * x[1] + R[6] * x[2];
  const T y1 = R[1] * x[0] + R[4] * x[1] + R[7] * x[2];
  const T y2 = R[2] * x[0] + R[5] * x[1] + R[8] * x[2];
  y[0] = y0; y[1] = y1; y[2] = y2;
}

// Base rotation and the world axes of the three Euler rates (yaw about e_z, pitch about Rz e_y, roll about Rz Ry e_x).
template <class T>
__device__ __forceinline__ void base_frame(const T* q, T* R, T* ax /*9: axes of yaw,pitch,roll as rows*/) {
  T sz, cz, sy, cy, sx, cx;
  sincos_t(q[3], sz, cz); sincos_t(q[4], sy, cy); sincos_t(q[5], sx, cx);
  R[0] = cz * cy; R[1] = cz * sy * sx - sz * cx; R[2] = cz * sy * cx + sz * sx;
  R[3] = sz * cy; R[4] = sz * sy * sx + cz * cx; R[5] = sz * sy * cx - cz * sx;
  R[6] = -sy;     R[7] = cy * sx;                R[8] = cy * cx;
  ax[0] = T(0.0); ax[1] = T(0.0); ax[2] = T(1.0);
  ax[3] = -sz; ax[4] = cz; ax[5] = T(0.0);
  ax[6] = cz * cy; ax[7] = sz * cy; ax[8] = -sy;
}

// R <- R * Rot(axis, th) for a signed coordinate axis code (+-1 x, +-2 y, +-3 z); returns the world joint axis in a[].
template <class T> __device__ __forceinline__ void joint_rotate(T* R, int code, const T& th, T* a) {
  T s, c;
  sincos_t(th, s, c);
  const int ax = code < 0 ? -code : code;
  if (code < 0) s = -s;
  const double sg = code < 0 ? -1.0 : 1.0;
  if (ax == 1) {
    for (int r = 0; r < 3; ++r) {
      a[r] = R[3 * r] * sg;
      const T c1 = R[3 * r + 1], c2 = R[3 * r + 2];
      R[3 * r + 1] = c * c1 + s * c2; R[3 * r + 2] = c * c2 - s * c1;
    }
  } else if (ax == 2) {
    for (int r = 0; r < 3; ++r) {
      a[r] = R[3 * r + 1] * sg;
      const T c0 = R[3 * r], c2 = R[3 * r + 2];
      R[3 * r] = c * c0 - s * c2; R[3 * r + 2] = s * c0 + c * c2;
    }
  } else {
    for (int r = 0; r < 3; ++r) {
      a[r] = R[3 * r + 2] * sg;
      const T c0 = R[3 * r], c1 = R[3 * r + 1];
      R[3 * r] = c * c0 + s * c1; R[3 * r + 1] = c * c1 - s * c0;
    }
  }
}

template <class T>
struct KinOut {
  T h[6];      // centroidal momentum [linear; angular about the CoM] = A(q) v
  T com[3];    // centre of mass
  T cpos[12];  // contact positions
  T cvel[12];  // contact velocities J_c(q) v
  T ke;        // kinetic energy 1/2 v' M(q) v
};

// R <- R * Rot(axis) given the sine / cosine of the joint angle; returns the world joint axis in a[].
template <class T> __device__ __forceinline__ void joint_rotate_sc(T* R, int code, T s, const T& c, T* a) {
  const int ax = code < 0 ? -code : code;
  if (code < 0) s = -s;
  const double sg = code < 0 ? -1.0 : 1.0;
  if (ax == 1) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      a[r] = R[3 * r] * sg;
      const T c1 = R[3 * r + 1], c2 = R[3 * r + 2];
      R[3 * r + 1] = c * c1 + s * c2; R[3 * r + 2] = c * c2 - s * c1;
    }
  } else if (ax == 2) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      a[r] = R[3 * r + 1] * sg;
      const T c0 = R[3 * r], c2 = R[3 * r + 2];
      R[3 * r] = c * c0 - s * c2; R[3 * r + 2] = s * c0 + c * c2;
    }
  } else {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      a[r] = R[3 * r + 2] * sg;
      const T c0 = R[3 * r], c1 = R[3 * r + 1];
      R[3 * r] = c * c0 + s * c1; R[3 * r + 1] = c * c1 - s * c0;
    }
  }
}

// One sweep over the tree: positions, velocities, CoM and centroidal momentum for generalised (q, v).
// Functor form (no runtime-indexed local arrays): qf(i), vf(i) return coordinate / velocity i; scf(k, s, c) returns the sine and
// cosine of angle k (0..2 = yaw, pitch, roll; 3..12 = joints), so that callers can share one sincos evaluation per configuration;
// of.h(r,x), of.com(r,x), of.cpos(i,x), of.cvel(i,x) receive the results.
template <class T, class QF, class VF, class SCF, class OF>
__device__ __forceinline__ void kin_pass_f(QF qf, VF vf, SCF scf, OF of) {
  const Model& md = c_model;
  T R0[9], ax0[9];
  {
    T sz, cz, sy, cy, sx, cx;
    scf(0, sz, cz); scf(1, sy, cy); scf(2, sx, cx);
    R0[0] = cz * cy; R0[1] = cz * sy * sx - sz * cx; R0[2] = cz * sy * cx + sz * sx;
    R0[3] = sz * cy; R0[4] = sz * sy * sx + cz * cx; R0[5] = sz * sy * cx - cz * sx;
    R0[6] = -sy;     R0[7] = cy * sx;                R0[8] = cy * cx;
    ax0[0] = T(0.0); ax0[1] = T(0.0); ax0[2] = T(1.0);
    ax0[3] = -sz; ax0[4] = cz; ax0[5] = T(0.0);
    ax0[6] = cz * cy; ax0[7] = sz * cy; ax0[8] = -sy;
  }
  T w0[3], P[3], Lo[3], mc[3];
  T ke = T(0.0);
  {
    const T v3 = vf(3), v4 = vf(4), v5 = vf(5);
#pragma unroll
    for (int i = 0; i < 3; ++i) w0[i] = ax0[i] * v3 + ax0[3 + i] * v4 + ax0[6 + i] * v5;
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) { P[i] = T(0.0); Lo[i] = T(0.0); mc[i] = T(0.0); }
  auto add_body = [&](int b, const T* R, const T* p, const T* w, const T* vl) {
    T r[3], wxr[3], vc[3], cw[3], l[3], wl[3], Iwl[3], Iw[3];
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
    for (int i = 0; i < 3; ++i) { P[i] = P[i] + vc[i]; Lo[i] = Lo[i] + l[i] + Iw[i]; mc[i] = mc[i] + cw[i] * mb; }
    // kinetic energy of the body (dead code for sinks that ignore it)
    ke = ke + ((vl[0] + wxr[0]) * vc[0] + (vl[1] + wxr[1]) * vc[1] + (vl[2] + wxr[2]) * vc[2] + wl[0] * Iwl[0] + wl[1] * Iwl[1] + wl[2] * Iwl[2]) * 0.5;
  };
  T p0[3] = {qf(0), qf(1), qf(2)}, v0[3] = {vf(0), vf(1), vf(2)};
  add_body(0, R0, p0, w0, v0);
  for (int leg = 0; leg < 2; ++leg) {
    T R[9], p[3], w[3], vl[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = R0[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) { p[i] = p0[i]; w[i] = w0[i]; vl[i] = v0[i]; }
    for (int j = 0; j < 5; ++j) {
      const int b = 1 + 5 * leg + j;
      T d[3], wxd[3], a[3], sj, cj;
      rot_const(R, &md.joint_xyz[3 * b], d);
      cross(w, d, wxd);
#pragma unroll
      for (int i = 0; i < 3; ++i) { p[i] = p[i] + d[i]; vl[i] = vl[i] + wxd[i]; }
      scf(2 + b, sj, cj);
      joint_rotate_sc(R, md.joint_axis[b], sj, cj, a);
      const T vb = vf(5 + b);
#pragma unroll
      for (int i = 0; i < 3; ++i) w[i] = w[i] + a[i] * vb;
      add_body(b, R, p, w, vl);
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {  // toe (contact leg), heel (contact 2+leg)
      const int c = leg + 2 * t;
      T off[3], wxo[3];
      rot_const(R, &md.contact_offset[3 * c], off);
      cross(w, off, wxo);
#pragma unroll
      for (int i = 0; i < 3; ++i) { of.cpos(3 * c + i, p[i] + off[i]); of.cvel(3 * c + i, vl[i] + wxo[i]); }
    }
  }
  const double im = 1.0 / md.total_mass;
  T com[3], cxP[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) { com[i] = mc[i] * im; of.com(i, com[i]); }
  cross(com, P, cxP);
#pragma unroll
  for (int i = 0; i < 3; ++i) { of.h(i, P[i]); of.h(3 + i, Lo[i] - cxP[i]); }
  of.ke(ke);
}

// ---- chain-split sweep (used by the node linearisation): a lane evaluates the base frame and ONE leg chain only.
// Bodies outside the chain do not depend on the chain's joint coordinates / velocities, so a joint-seeded lane needs nothing else;
// base-seeded quantities are the sum of a (base + left chain) lane and a (right chain) lane. The model constants of the chain pass
// live in shared memory because lanes of one warp walk different chains (constant memory would serialise the diverging addresses).
struct ChainModel {
  double joint_xyz[NBODY * 3], com[NBODY * 3], inertia[NBODY * 9], mass[NBODY], contact_offset[NC * 3];
  int joint_axis[NBODY];
};
__device__ __forceinline__ void chain_model_load(ChainModel& cm, int tid, int nthreads) {
  const Model& md = c_model;
  for (int i = tid; i < NBODY * 3; i += nthreads) { cm.joint_xyz[i] = md.joint_xyz[i]; cm.com[i] = md.com[i]; }
  for (int i = tid; i < NBODY * 9; i += nthreads) cm.inertia[i] = md.inertia[i];
  for (int i = tid; i < NBODY; i += nthreads) { cm.mass[i] = md.mass[i]; cm.joint_axis[i] = md.joint_axis[i]; }
  for (int i = tid; i < NC * 3; i += nthreads) cm.contact_offset[i] = md.contact_offset[i];
}

template <class T> struct ChainOut {
  T P[3], Lo[3], mc[3];   // partial sums over the bodies visited: linear momentum, angular momentum about the origin, mass * position
  T cpos[6], cvel[6];     // toe (contact `leg`) then heel (contact 2 + leg) of this chain
};

template <class T, class QF, class VF, class SCF>
__device__ __forceinline__ void kin_chain_f(const ChainModel& md, int leg, bool with_base, QF qf, VF vf, SCF scf, ChainOut<T>& o) {
  T R[9], ax0[9];
  {
    T sz, cz, sy, cy, sx, cx;
    scf(0, sz, cz); scf(1, sy, cy); scf(2, sx, cx);
    R[0] = cz * cy; R[1] = cz * sy * sx - sz * cx; R[2] = cz * sy * cx + sz * sx;
    R[3] = sz * cy; R[4] = sz * sy * sx + cz * cx; R[5] = sz * sy * cx - cz * sx;
    R[6] = -sy;     R[7] = cy * sx;                R[8] = cy * cx;
    ax0[0] = T(0.0); ax0[1] = T(0.0); ax0[2] = T(1.0);
    ax0[3] = -sz; ax0[4] = cz; ax0[5] = T(0.0);
    ax0[6] = cz * cy; ax0[7] = sz * cy; ax0[8] = -sy;
  }
  T w[3], p[3] = {qf(0), qf(1), qf(2)}, vl[3] = {vf(0), vf(1), vf(2)};
  {
    const T v3 = vf(3), v4 = vf(4), v5 = vf(5);
#pragma unroll
    for (int i = 0; i < 3; ++i) w[i] = ax0[i] * v3 + ax0[3 + i] * v4 + ax0[6 + i] * v5;
  }
  T P[3], Lo[3], mc[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) { P[i] = T(0.0); Lo[i] = T(0.0); mc[i] = T(0.0); }
  auto add_body = [&](int b) {
    T r[3], wxr[3], vc[3], cw[3], l[3], wl[3], Iwl[3], Iw[3];
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
    for (int i = 0; i < 3; ++i) { P[i] = P[i] + vc[i]; Lo[i] = Lo[i] + l[i] + Iw[i]; mc[i] = mc[i] + cw[i] * mb; }
  };
  if (with_base) add_body(0);
  for (int j = 0; j < 5; ++j) {
    const int b = 1 + 5 * leg + j;
    T d[3], wxd[3], a[3], sj, cj;
    rot_const(R, &md.joint_xyz[3 * b], d);
    cross(w, d, wxd);
#pragma unroll
    for (int i = 0; i < 3; ++i) { p[i] = p[i] + d[i]; vl[i] = vl[i] + wxd[i]; }
    scf(2 + b, sj, cj);
    joint_rotate_sc(R, md.joint_axis[b], sj, cj, a);
    const T vb = vf(5 + b);
#pragma unroll
    for (int i = 0; i < 3; ++i) w[i] = w[i] + a[i] * vb;
    add_body(b);
  }
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int c = leg + 2 * t;
    T off[3], wxo[3];
    rot_const(R, &md.contact_offset[3 * c], off);
    cross(w, off, wxo);
#pragma unroll
    for (int i = 0; i < 3; ++i) { o.cpos[3 * t + i] = p[i] + off[i]; o.cvel[3 * t + i] = vl[i] + wxo[i]; }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) { o.P[i] = P[i]; o.Lo[i] = Lo[i]; o.mc[i] = mc[i]; }
}

template <class T> struct KinOutSink {
  KinOut<T>& o;
  __device__ __forceinline__ void h(int i, const T& x) { o.h[i] = x; }
  __device__ __forceinline__ void com(int i, const T& x) { o.com[i] = x; }
  __device__ __forceinline__ void cpos(int i, const T& x) { o.cpos[i] = x; }
  __device__ __forceinline__ void cvel(int i, const T& x) { o.cvel[i] = x; }
  __device__ __forceinline__ void ke(const T& x) { o.ke = x; }
};

// Array form (used where the lane-private copy of q, v is needed anyway)
template <class T>
__device__ void kin_pass(const T* q, const T* v, KinOut<T>& o) {
  KinOutSink<T> sink{o};
  kin_pass_f<T>([&](int i) { return q[i]; }, [&](int i) { return v[i]; },
                [&](int k, T& s, T& c) { sincos_t(q[3 + k], s, c); }, sink);
}

// ---- the state layout: rbd [zyx, p, q_j, omega_world, v, qd_j] <-> q = [p, zyx, q_j], v = [v, zyx rates, qd_j].
// omega_world = T(zyx) [yaw, pitch, roll rates]; both directions take the sines and cosines of yaw (sz, cz) and pitch (sy, cy).
// getEulerAnglesZyxDerivativesFromGlobalAngularVelocity: rates = T^-1 w
__device__ __forceinline__ void zyx_rates_from_world_omega(double sz, double cz, double sy, double cy, const double* w, double* rates) {
  const double w0 = w[0], w1 = w[1], w2 = w[2];
  const double dxr = (cz * w0 + sz * w1) / cy;
  rates[2] = dxr; rates[1] = -sz * w0 + cz * w1; rates[0] = w2 + sy * dxr;
}
// w = T rates
__device__ __forceinline__ void world_omega_from_zyx_rates(double sz, double cz, double sy, double cy, const double* rates, double* w) {
  const double d0 = rates[0], d1 = rates[1], d2 = rates[2];
  w[0] = -sz * d1 + cz * cy * d2; w[1] = cz * d1 + sz * cy * d2; w[2] = d0 - sy * d2;
}
__device__ __forceinline__ void rbd_to_qv(const double* r, double* q, double* v) {
  for (int i = 0; i < 3; ++i) { q[i] = r[3 + i]; q[3 + i] = r[i]; v[i] = r[NQ + 3 + i]; }
  for (int j = 0; j < NJ; ++j) { q[6 + j] = r[6 + j]; v[6 + j] = r[NQ + 6 + j]; }
  double sz, cz, sy, cy;
  sincos(q[3], &sz, &cz); sincos(q[4], &sy, &cy);
  zyx_rates_from_world_omega(sz, cz, sy, cy, &r[NQ], &v[3]);
}
__device__ __forceinline__ void qv_to_rbd(const double* q, const double* v, double* r) {
  for (int i = 0; i < 3; ++i) { r[3 + i] = q[i]; r[i] = q[3 + i]; r[NQ + 3 + i] = v[i]; }
  for (int j = 0; j < NJ; ++j) { r[6 + j] = q[6 + j]; r[NQ + 6 + j] = v[6 + j]; }
  double sz, cz, sy, cy;
  sincos(q[3], &sz, &cz); sincos(q[4], &sy, &cy);
  world_omega_from_zyx_rates(sz, cz, sy, cy, &v[3], &r[NQ]);
}

// InverseKinematics::computeFootPos: the contact frame positions (12) at the configuration q
__device__ __forceinline__ void contact_positions(const double* qs, double* pos) {
  double q[NQ], v[NQ];
  for (int i = 0; i < NQ; ++i) { q[i] = qs[i]; v[i] = 0.0; }
  KinOut<double> o;
  kin_pass<double>(q, v, o);
  for (int i = 0; i < 12; ++i) pos[i] = o.cpos[i];
}

// computeCentroidalStateFromRbdModel (LeggedController.cpp:336): rbd -> x [h_lin/m, h_ang/m, p, zyx, q_j]
__device__ __forceinline__ void rbd_to_centroidal(const double* r, double* x) {
  double q[NQ], v[NQ];
  rbd_to_qv(r, q, v);
  KinOut<double> o;
  kin_pass<double>(q, v, o);
  for (int i = 0; i < 6; ++i) x[i] = o.h[i] / c_model.total_mass;
  for (int i = 0; i < NQ; ++i) x[6 + i] = q[i];
}

// The base of rnea_pass for the coordinates q, v, a: its orientation R0, the world axes of its yaw / pitch / roll rotations ax0 (rows), its
// world angular velocity w0 and acceleration wd0, and the acceleration pd0 of its origin.
__device__ __forceinline__ void rnea_base_motion(const double* q, const double* v, const double* a, double* R0, double* ax0, double* w0, double* wd0,
                                                 double* pd0) {
  base_frame(q, R0, ax0);
  double w1[3], w2[3], t1[3], t2[3];
  for (int i = 0; i < 3; ++i) { w1[i] = ax0[i] * v[3]; w2[i] = w1[i] + ax0[3 + i] * v[4]; }
  cross(w1, &ax0[3], t1);
  cross(w2, &ax0[6], t2);
  for (int i = 0; i < 3; ++i) {
    w0[i] = w2[i] + ax0[6 + i] * v[5];
    wd0[i] = ax0[i] * a[3] + ax0[3 + i] * a[4] + ax0[6 + i] * a[5] + t1[i] * v[4] + t2[i] * v[5];
    pd0[i] = a[i];
  }
}

// Newton-Euler wrench of one rigid body, world frame: orientation R, angular velocity w and acceleration wd, acceleration pd of its frame
// origin; mass mb, CoM com and inertia I about the CoM (both in the body frame, I row-major). F = mb (pd + wd x r + w x (w x r)) (+ mb g e_z
// with gravity) and the moment about the frame origin n = R (I wd_l + w_l x I w_l) + r x F, with r = R com and w_l, wd_l = R' w, R' wd.
__device__ __forceinline__ void rigid_body_wrench(const double* R, const double* w, const double* wd, const double* pd, double mb, const double* com,
                                                  const double* I, bool gravity, double* F, double* n) {
  double r[3], t[3], t2[3], t3[3], wl[3], wdl[3], Iw[3], Iwd[3], Nl[3], N[3], rxF[3];
  rot_const(R, com, r);
  cross(wd, r, t); cross(w, r, t2); cross(w, t2, t3);
  for (int i = 0; i < 3; ++i) F[i] = (pd[i] + t[i] + t3[i]) * mb;
  if (gravity) F[2] += mb * HB_GRAVITY;
  rotT(R, w, wl); rotT(R, wd, wdl);
  for (int i = 0; i < 3; ++i) {
    Iw[i] = wl[0] * I[3 * i] + wl[1] * I[3 * i + 1] + wl[2] * I[3 * i + 2];
    Iwd[i] = wdl[0] * I[3 * i] + wdl[1] * I[3 * i + 1] + wdl[2] * I[3 * i + 2];
  }
  cross(wl, Iw, Nl);
  for (int i = 0; i < 3; ++i) Nl[i] += Iwd[i];
  rot(R, Nl, N);
  cross(r, F, rxF);
  for (int i = 0; i < 3; ++i) n[i] = N[i] + rxF[i];
}

// The inertial parameters rnea_pass reads for body b: its mass, its CoM and its inertia about the CoM (body frame, row-major).
// NominalBodies reads the model; LinkBodies reads a table of 13 doubles per body, [m, c(3), I(9)] (a varied robot's bodies, sim_step_kernel).
struct NominalBodies {
  __device__ __forceinline__ double mass(int b) const { return c_model.mass[b]; }
  __device__ __forceinline__ const double* com(int b) const { return &c_model.com[3 * b]; }
  __device__ __forceinline__ const double* inertia(int b) const { return &c_model.inertia[9 * b]; }
};
constexpr int LINK_BODY = 13;
struct LinkBodies {
  const double* t;
  __device__ __forceinline__ double mass(int b) const { return t[LINK_BODY * b]; }
  __device__ __forceinline__ const double* com(int b) const { return t + LINK_BODY * b + 1; }
  __device__ __forceinline__ const double* inertia(int b) const { return t + LINK_BODY * b + 4; }
};

// Recursive Newton-Euler in the coordinates above: tau = M(q) a + C(q,v) v + g(q)   (float64, per lane), with the bodies' inertial
// parameters from `bodies` (the model's by default; the kinematics are always the model's).
// Also returns the classical acceleration of the four contact points (= J_c a + dJ_c/dt v).
template <class Bodies = NominalBodies>
__device__ void rnea_pass(const double* q, const double* v, const double* a, bool gravity, double* tau, double* cacc, Bodies bodies = Bodies()) {
  const Model& md = c_model;
  double R0[9], ax0[9], w0[3], wd0[3], pd0[3];
  rnea_base_motion(q, v, a, R0, ax0, w0, wd0, pd0);
  auto body_wrench = [&](int b, const double* R, const double* w, const double* wd, const double* pd, double* F, double* n) {
    rigid_body_wrench(R, w, wd, pd, bodies.mass(b), bodies.com(b), bodies.inertia(b), gravity, F, n);
  };
  double f0[3], n0[3];
  body_wrench(0, R0, w0, wd0, pd0, f0, n0);
  for (int leg = 0; leg < 2; ++leg) {
    double R[9], w[3], wd[3], pd[3];
    for (int i = 0; i < 9; ++i) R[i] = R0[i];
    for (int i = 0; i < 3; ++i) { w[i] = w0[i]; wd[i] = wd0[i]; pd[i] = pd0[i]; }
    double dj[5][3], aj[5][3], Fj[5][3], nj[5][3];
    for (int j = 0; j < 5; ++j) {
      const int b = 1 + 5 * leg + j;
      double t[3], t2[3], t3[3], t4[3];
      rot_const(R, &md.joint_xyz[3 * b], dj[j]);
      cross(wd, dj[j], t); cross(w, dj[j], t2); cross(w, t2, t3);
      for (int i = 0; i < 3; ++i) pd[i] += t[i] + t3[i];
      joint_rotate(R, md.joint_axis[b], q[5 + b], aj[j]);
      cross(w, aj[j], t4);
      for (int i = 0; i < 3; ++i) { wd[i] += aj[j][i] * a[5 + b] + t4[i] * v[5 + b]; w[i] += aj[j][i] * v[5 + b]; }
      body_wrench(b, R, w, wd, pd, Fj[j], nj[j]);
    }
    if (cacc) {
      for (int t = 0; t < 2; ++t) {
        const int c = leg + 2 * t;
        double o[3], t1[3], t2[3], t3[3];
        rot_const(R, &md.contact_offset[3 * c], o);
        cross(wd, o, t1); cross(w, o, t2); cross(w, t2, t3);
        for (int i = 0; i < 3; ++i) cacc[3 * c + i] = pd[i] + t1[i] + t3[i];
      }
    }
    double f[3] = {0, 0, 0}, n[3] = {0, 0, 0};
    for (int j = 4; j >= 0; --j) {
      const int b = 1 + 5 * leg + j;
      for (int i = 0; i < 3; ++i) { f[i] += Fj[j][i]; n[i] += nj[j][i]; }
      tau[5 + b] = aj[j][0] * n[0] + aj[j][1] * n[1] + aj[j][2] * n[2];
      double dxf[3];
      cross(dj[j], f, dxf);
      for (int i = 0; i < 3; ++i) n[i] += dxf[i];  // moment about the parent origin
    }
    for (int i = 0; i < 3; ++i) { f0[i] += f[i]; n0[i] += n[i]; }
  }
  for (int i = 0; i < 3; ++i) {
    tau[i] = f0[i];
    tau[3 + i] = ax0[3 * i] * n0[0] + ax0[3 * i + 1] * n0[1] + ax0[3 * i + 2] * n0[2];
  }
}

// Solve A_b y = r for the base block of the centroidal momentum matrix (row-major, ld 6). A_b = [m I, A12; 0, A22]
// (computeFloatingBaseCentroidalMomentumMatrixInverse uses the same structure): one 3x3 adjugate and one division instead of a pivoted
// 6x6 elimination with twelve divisions on the dependent chain.
__device__ __forceinline__ void solve6_cmm(const double* A, const double* r, double* y) {
  const double a = A[21], b = A[22], c = A[23], d = A[27], e = A[28], g = A[29], h = A[33], k = A[34], l = A[35];
  const double c00 = e * l - g * k, c01 = d * l - g * h, c02 = d * k - e * h;
  const double id = 1.0 / (a * c00 - b * c01 + c * c02);
  y[3] = (c00 * r[3] - (b * l - c * k) * r[4] + (b * g - c * e) * r[5]) * id;
  y[4] = (-c01 * r[3] + (a * l - c * h) * r[4] - (a * g - c * d) * r[5]) * id;
  y[5] = (c02 * r[3] - (a * k - b * h) * r[4] + (a * e - b * d) * r[5]) * id;
#pragma unroll
  for (int i = 0; i < 3; ++i) y[i] = (r[i] - A[6 * i + 3] * y[3] - A[6 * i + 4] * y[4] - A[6 * i + 5] * y[5]) / A[7 * i];
}

}  // namespace hb

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
// computeCentroidalStateFromRbdModel (LeggedController.cpp:336)
__global__ void rbd_to_centroidal_kernel(int B, const double* rbd, double* x) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  rbd_to_centroidal(rbd + (size_t)inst * 32, x + (size_t)inst * NX);
}

// InverseKinematics::computeFootPos: contact frame positions at the configuration of x (one thread per instance)
__global__ void contact_positions_kernel(int B, const double* x, double* pos) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  contact_positions(x + (size_t)inst * NX + 6, pos + (size_t)inst * 12);
}
}  // namespace
