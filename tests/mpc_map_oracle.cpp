// The CPU oracle (oracle/hb_oracle.cpp, compiled as it is) told where the ground under the stance feet is: the stance heights of
// hunter_b200.h's "MPC maps". Test infrastructure only; tests/mpc_map_ref.py builds and loads it.
//
// The oracle's stance z row (M4) is the one statement `if (a == 2) val += HB_ZEROVEL_Z_GAIN * epos[3 * c + 2] + HB_ZEROVEL_Z_OFFSET;`
// of node_cost_constraints. This unit compiles the oracle with HB_ZEROVEL_Z_OFFSET expanding to the constant followed by a second statement,
// `if (a == 2 && heights) val -= HB_ZEROVEL_Z_GAIN * h`, with h the height of the row's contact c at the row's node: the row becomes
// (v_z + 3 p_z - 0.06) - 3 h, the device's order of operations, and holds the foot at 0.02 + h; the row's Jacobian is unchanged. The node is
// found from the swing-reference pointer the oracle hands its node evaluation (swing + 24 k, in the linearisation and in the line search
// alike). Without heights the first statement is the oracle's own, and +0 heights subtract +0: the oracle's bits either way.
#include <cstddef>

#include "../include/hunter_model_constants.h"

namespace hbt {
constexpr double kZeroVelZOffset = HB_ZEROVEL_Z_OFFSET;
thread_local const double* swing0 = nullptr;    // the swing references of node 0 of the call in progress
thread_local const double* heights = nullptr;   // that call's stance heights, nodes x 4; null: flat ground
inline double height(const double* swing, int c) { return heights ? heights[(size_t)((swing - swing0) / 24) * 4 + c] : 0.0; }
// the heights of one call, set for its duration on the calling thread
struct Scope {
  Scope(const double* swing, const double* h) { swing0 = swing; heights = h; }
  ~Scope() { swing0 = nullptr; heights = nullptr; }
};
}  // namespace hbt

#undef HB_ZEROVEL_Z_OFFSET
#define HB_ZEROVEL_Z_OFFSET hbt::kZeroVelZOffset; if (a == 2 && hbt::heights) val -= HB_ZEROVEL_Z_GAIN * hbt::height(swing, c)
#include "../oracle/hb_oracle.cpp"

extern "C" {
// hbo_node_lq with the four heights of the node's contacts (nullable)
void hbt_node_lq(double dt, const double* x, const double* u, const double* xn, const double* xref, const double* swing, int mode,
                 double* Ad, double* Bd, double* b, double* Q, double* R, double* P, double* q, double* r, double* C, double* D,
                 double* e, int* m, double* cost, const double* stance_h) {
  hbt::Scope s(swing, stance_h);
  hbo_node_lq(dt, x, u, xn, xref, swing, mode, Ad, Bd, b, Q, R, P, q, r, C, D, e, m, cost);
}

// hbo_mpc_iteration with (N+1) x 4 heights (nullable)
void hbt_mpc_iteration(const hbo_horizon* hz, int max_trials, const double* x0, const double* x_ref, const double* swing, const int32_t* mode,
                       double* x_traj, double* u_traj, hbo_solve_info* info, hbo_ls_trial* trials, const double* stance_h) {
  hbt::Scope s(swing, stance_h);
  hbo_mpc_iteration(hz, max_trials, x0, x_ref, swing, mode, x_traj, u_traj, info, trials);
}

// hbo_mpc_iteration_batch (one thread) with B x (N+1) x 4 heights (nullable)
void hbt_mpc_iteration_batch(const hbo_horizon* hz, int B, const double* x0, const double* x_ref, const double* swing, const int32_t* mode,
                             double* x_traj, double* u_traj, hbo_solve_info* info, const double* stance_h) {
  const size_t N = (size_t)hz->N;
  for (int i = 0; i < B; ++i) {
    const double* sw = swing + (size_t)i * (N + 1) * 24;
    hbt::Scope s(sw, stance_h ? stance_h + (size_t)i * (N + 1) * 4 : nullptr);
    hbo_mpc_iteration(hz, 14, x0 + (size_t)i * NX, x_ref + (size_t)i * (N + 1) * NX, sw, mode + (size_t)i * (N + 1),
                      x_traj + (size_t)i * (N + 1) * NX, u_traj + (size_t)i * N * NU, info ? info + i : nullptr, nullptr);
  }
}
}
