// ORACLE (test infrastructure only). CPU float64 restatement of the reference's per-control-step
// NMPC iteration + WeightedWbc QP for the Hunter biped. Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this; the product path never does.
//
// PARITY UNPINNED for the solver rows (SURVEY §8c): OCS2 (SqpMpc / HPIPM), Pinocchio, CppAD and qpOASES are
// not vendored in the reference and cannot be built offline, and the reference holds no golden vectors for this
// path. What IS pinned: rigid-body quantities against the reference's vendored MuJoCo 3.0.1 model
// (tests/golden/rbd_mujoco.json), derivatives against finite differences, QPs by KKT residuals, Riccati by a
// dense KKT solve. Every function cites the reference file:line it restates.
#pragma once
#include <cstdint>

#ifdef __cplusplus
extern "C" {
#endif

// node-sampled references for one MPC instance (same layout the CUDA path consumes)
//   x_ref   [(N+1) x 22]   target state at node times          (cost M2: LeggedRobotQuadraticTrackingCost.h:73-80)
//   swing   [(N+1) x 4 x 6] per contact [px,py,pz,vx,vy,vz] of the swing reference (LeggedRobotPreComputation.cpp:96-119)
//   mode    [(N+1)]        mode number (MotionPhaseDefinition.h:55-87) in force on interval k
typedef struct {
  int N;
  double dt;          // uniform interval length, used when dts == NULL
  const double* dts;  // optional: N interval lengths dt_k = t_{k+1} - t_k (non-uniform grids: OCS2's time discretisation re-anchors
                      // the grid at every mode switch, SURVEY 8a row S1)
} hbo_horizon;

typedef struct {
  double alpha;           // accepted step size (0 = no step)
  double merit0, merit1;  // merit before / after
  double viol0, viol1;    // total constraint violation before / after
  double armijo;          // descent metric
  int status;             // 0 ok, 3 NaN
  int n_trials;
} hbo_solve_info;

// one trial of the filter line search (App. C.5 step 4): the branch that decided it and the decision
enum { HBO_LS_VIOLATION = 0, HBO_LS_ARMIJO = 1, HBO_LS_FILTER = 2 };
typedef struct {
  double alpha, merit, viol;  // step length, merit and total violation of the trial
  int branch;                 // HBO_LS_*: violation (viol > g_max), Armijo (viol, viol0 < g_min and a descent metric < 0), filter
  int accepted;               // 1: the step was taken at this trial
} hbo_ls_trial;

void hbo_init(void);
// rigid-body probes (for pinning against MuJoCo / finite differences)
void hbo_rbd(const double* q, const double* v, double* M /*16x16*/, double* nle /*16*/, double* J /*12x16*/,
             double* dJv /*12*/, double* A /*6x16*/, double* com /*3*/, double* h /*6*/, double* cpos /*12*/);
void hbo_rbd_to_centroidal(const double* rbd /*32*/, double* x /*22*/);
void hbo_observer_terms(const double* q, const double* v, double* p /*16*/, double* g /*16*/, double* ctv /*16*/, double* Jfoot /*2x6x16*/);
void hbo_flow_map(const double* x, const double* u, double* f /*22*/, double* A /*22x22*/, double* B /*22x22*/);
void hbo_ee_kinematics(const double* x, const double* u, double* pos /*12*/, double* vel /*12*/, double* dpos_dx /*12x22*/,
                       double* dvel_dx /*12x22*/, double* dvel_du /*12x22*/);
void hbo_input_cost_R(double* R /*22x22*/);
void hbo_set_wbc_settings(const double* s /*17 doubles, order of hb_wbc_settings; NULL = shipped task.info values*/);
// node LQ model (for inspection): returns sizes via pointers
void hbo_node_lq(double t_dt, const double* x, const double* u, const double* xn, const double* xref, const double* swing,
                 int mode, double* Ad, double* Bd, double* b, double* Q, double* R, double* P, double* q, double* r,
                 double* C, double* D, double* e, int* m, double* cost);
// one SQP iteration (S1-S7) on one instance; x_traj[(N+1)x22], u_traj[Nx22] in/out. max_trials (>= 1) caps the line search like
// hb_config.line_search_max_trials (14: alpha = 1, 1/2, ... >= 1e-4, the cap alpha_min reaches first); trials (nullable, max_trials rows)
// receives one row per trial evaluated, info->n_trials in all
void hbo_mpc_iteration(const hbo_horizon* hz, int max_trials, const double* x0, const double* x_ref, const double* swing, const int32_t* mode,
                       double* x_traj, double* u_traj, hbo_solve_info* info, hbo_ls_trial* trials);
void hbo_mpc_cold_start(const hbo_horizon* hz, const double* x0, const int32_t* mode, double* x_traj, double* u_traj);
// WBC (W1-W4)
void hbo_wbc_terms(const double* x_des, const double* u_des, const double* rbd, int mode, double* Aw, double* bw, int* rw, double* J, double* dJv);
void hbo_wbc_assemble(const double* x_des, const double* u_des, const double* rbd, int mode, int stance_mode,
                      double* H /*38x38*/, double* g /*38*/, double* A /*60x38 row-major*/, double* lbA, double* ubA, int* m);
int hbo_qp_solve(int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA,
                 double rho, double* x, int* iters);
int hbo_wbc_solve(const double* x_des, const double* u_des, const double* rbd, int mode, int stance_mode, double rho,
                  double* sol /*38*/);
// batched helpers with OpenMP-free std::thread parallelism (CPU baseline timing)
void hbo_mpc_iteration_batch(const hbo_horizon* hz, int B, int threads, const double* x0, const double* x_ref, const double* swing,
                             const int32_t* mode, double* x_traj, double* u_traj, hbo_solve_info* info);
void hbo_wbc_solve_batch(int B, int threads, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                         const uint8_t* stance_mode, double rho, double* sol, int32_t* status);
void hbo_wbc_qp_batch(int B, int threads, int n, int m, const double* H, const double* g, const double* A, const double* lbA,
                      const double* ubA, double rho, double* x, int32_t* status);

#ifdef __cplusplus
}
#endif
