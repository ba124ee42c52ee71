// The CPU oracle told where the ground under the stance feet is, for its stance heights and its friction cones: mpc_map_oracle.cpp (the
// oracle, oracle/hb_oracle.cpp compiled as it is, given the stance heights of hunter_b200.h's "MPC maps") given surface frames as well,
// the cones of "MPC cone maps". Test infrastructure only; tests/mpc_cone_ref.py builds and loads it.
//
// The oracle's friction cone (M6) of stance contact c is the statement `Pen p = relaxed_barrier(h, HB_FRICTION_BARRIER_MU,
// HB_FRICTION_BARRIER_DELTA);` followed by its cost, gradient, Hessian and diagonal-shift terms. This unit compiles the oracle with
//   - HB_FRICTION_BARRIER_MU expanding to 0 for a contact with a frame (its own cone then adds zeros), the constant otherwise;
//   - HB_FRICTION_BARRIER_DELTA expanding to the constant followed by a second statement, hbc::cone(...), which adds the cone of a
//     contact with a frame restated from FrictionConeConstraint.cpp:78-233: the local force Fl = t_R_w F, h = mu Fl_z - sqrt(Fl_x^2 +
//     Fl_y^2 + reg), the relaxed barrier of h, g = t_R_w' g_l and H = t_R_w' H_l t_R_w, the Hessian diagonal shift unchanged.
// Its expressions are the oracle's in the oracle's order, so an identity frame adds what the oracle adds: the oracle's bits. The frame of
// a node's contact is found from the swing-reference pointer the oracle hands its node evaluation (swing + 24 k), as the heights are.
// Frames are t_R_w, rows t1, t2, n (9 doubles per contact); null frames: the oracle's cones.
#include <cmath>
#include <cstddef>

#include "../include/hunter_model_constants.h"
// the frame rule as the device runs it: every product rounded on its own, none contracted into an fma by the host compiler
#pragma GCC push_options
#pragma GCC optimize("fp-contract=off")
#include "../hunter_bipedal_control_b200/csrc/hb_planner.h"
#pragma GCC pop_options

namespace hbc {
constexpr double kMu = HB_FRICTION_BARRIER_MU, kDelta = HB_FRICTION_BARRIER_DELTA;
thread_local const double* swing0 = nullptr;    // the swing references of node 0 of the call in progress
thread_local const double* frames = nullptr;    // that call's frames, nodes x 4 x 9; null: every cone about world z
inline const double* frame(const double* swing, int c) { return frames ? frames + ((size_t)((swing - swing0) / 24) * 4 + c) * 9 : nullptr; }
// the barrier weight the oracle's own cone statement uses: 0 where hbc::cone adds the cone instead
inline double oracle_mu(const double* swing, int c) { return frame(swing, c) ? 0.0 : kMu; }

// The cone of stance contact c on its frame (nothing without one), added to the oracle's node terms o (NodeLQ) and cost; lin: whether
// the oracle forms the LQ model (node_cost_constraints' L).
template <class O>
void cone(const double* swing, int c, const double* u, bool lin, O& o, double& cost) {
  const double* R = frame(swing, c);
  if (!R) return;
  constexpr int nx = sizeof(o.q) / sizeof(double), nu = sizeof(o.r) / sizeof(double);
  const double F[3] = {u[3 * c], u[3 * c + 1], u[3 * c + 2]};
  double Fl[3];
  for (int a = 0; a < 3; ++a) Fl[a] = R[3 * a] * F[0] + R[3 * a + 1] * F[1] + R[3 * a + 2] * F[2];
  const double Fx = Fl[0], Fy = Fl[1], Fz = Fl[2];
  const double t2 = Fx * Fx + Fy * Fy + HB_FRICTION_REGULARIZATION, tn = std::sqrt(t2), t32 = tn * t2;
  const double h = HB_FRICTION_MU * Fz - tn;
  // relaxed barrier (relaxedBarrierPenaltyVis.py:15-19)
  double v, d1, d2;
  if (h > kDelta) { v = -kMu * std::log(h); d1 = -kMu / h; d2 = kMu / (h * h); }
  else {
    const double z = (h - 2.0 * kDelta) / kDelta;
    v = kMu * (-std::log(kDelta) + 0.5 * z * z - 0.5); d1 = kMu * (h - 2.0 * kDelta) / (kDelta * kDelta); d2 = kMu / (kDelta * kDelta);
  }
  cost += v;
  if (!lin) return;
  const double gl[3] = {-Fx / tn, -Fy / tn, HB_FRICTION_MU};
  const double Hl[9] = {-(Fy * Fy + HB_FRICTION_REGULARIZATION) / t32, Fx * Fy / t32, 0, Fx * Fy / t32,
                        -(Fx * Fx + HB_FRICTION_REGULARIZATION) / t32, 0, 0, 0, 0};
  double gr[3], HR[9], Hh[9];
  for (int i = 0; i < 3; ++i) gr[i] = gl[0] * R[i] + gl[1] * R[3 + i] + gl[2] * R[6 + i];                       // t_R_w' g_l
  for (int a = 0; a < 3; ++a)
    for (int j = 0; j < 3; ++j) HR[3 * a + j] = Hl[3 * a] * R[j] + Hl[3 * a + 1] * R[3 + j] + Hl[3 * a + 2] * R[6 + j];   // H_l t_R_w
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Hh[3 * i + j] = R[i] * HR[j] + R[3 + i] * HR[3 + j] + R[6 + i] * HR[6 + j];       // t_R_w' H_l t_R_w
  for (int i = 0; i < 3; ++i) {
    o.r[3 * c + i] += d1 * gr[i];
    for (int j = 0; j < 3; ++j) o.R[(3 * c + i) * nu + 3 * c + j] += d2 * gr[i] * gr[j] + d1 * Hh[3 * i + j];
  }
  for (int i = 0; i < nu; ++i) o.R[i * nu + i] += d1 * (-HB_FRICTION_HESSIAN_SHIFT);
  for (int i = 0; i < nx; ++i) o.Q[i * nx + i] += d1 * (-HB_FRICTION_HESSIAN_SHIFT);
}

// the frames of one call, set for its duration on the calling thread
struct Scope {
  Scope(const double* swing, const double* f) { swing0 = swing; frames = f; }
  ~Scope() { swing0 = nullptr; frames = nullptr; }
};
}  // namespace hbc

#undef HB_FRICTION_BARRIER_MU
#undef HB_FRICTION_BARRIER_DELTA
#define HB_FRICTION_BARRIER_MU hbc::oracle_mu(swing, c)
#define HB_FRICTION_BARRIER_DELTA hbc::kDelta); hbc::cone(swing, c, u, L, o, cost
#include "mpc_map_oracle.cpp"

extern "C" {
// The surface frame (n, t1, t2) of map m at (x, y): hbplan::map_frame, the rule the WBC and both MPC kernels use. Returns whether the
// ground is sloped there (f written only then).
int hbc_map_frame(const hb_terrain* m, double x, double y, double* f) { return hbplan::map_frame(*m, x, y, f) ? 1 : 0; }

// hbt_node_lq with the node's four frames (4 x 9, nullable)
void hbc_node_lq(double dt, const double* x, const double* u, const double* xn, const double* xref, const double* swing, int mode,
                 double* Ad, double* Bd, double* b, double* Q, double* R, double* P, double* q, double* r, double* C, double* D,
                 double* e, int* m, double* cost, const double* stance_h, const double* frames) {
  hbc::Scope s(swing, frames);
  hbt_node_lq(dt, x, u, xn, xref, swing, mode, Ad, Bd, b, Q, R, P, q, r, C, D, e, m, cost, stance_h);
}

// hbt_mpc_iteration with (N+1) x 4 x 9 frames (nullable)
void hbc_mpc_iteration(const hbo_horizon* hz, int max_trials, const double* x0, const double* x_ref, const double* swing, const int32_t* mode,
                       double* x_traj, double* u_traj, hbo_solve_info* info, hbo_ls_trial* trials, const double* stance_h, const double* frames) {
  hbc::Scope s(swing, frames);
  hbt_mpc_iteration(hz, max_trials, x0, x_ref, swing, mode, x_traj, u_traj, info, trials, stance_h);
}

// hbt_mpc_iteration_batch with B x (N+1) x 4 x 9 frames (nullable)
void hbc_mpc_iteration_batch(const hbo_horizon* hz, int B, const double* x0, const double* x_ref, const double* swing, const int32_t* mode,
                             double* x_traj, double* u_traj, hbo_solve_info* info, const double* stance_h, const double* frames) {
  const size_t N = (size_t)hz->N;
  for (int i = 0; i < B; ++i) {
    const double* sw = swing + (size_t)i * (N + 1) * 24;
    hbc::Scope s(sw, frames ? frames + (size_t)i * (N + 1) * 36 : nullptr);
    hbt_mpc_iteration(hz, 14, x0 + (size_t)i * NX, x_ref + (size_t)i * (N + 1) * NX, sw, mode + (size_t)i * (N + 1),
                      x_traj + (size_t)i * (N + 1) * NX, u_traj + (size_t)i * N * NU, info ? info + i : nullptr, nullptr,
                      stance_h ? stance_h + (size_t)i * (N + 1) * 4 : nullptr);
  }
}
}
