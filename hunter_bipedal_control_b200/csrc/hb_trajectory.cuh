// The resident primal solution on the device: the initializer (cold start), the warm shift of the previous solution onto the next
// solve's grid, and the policy evaluation between MPC solves.
#pragma once
#include "hb_common.cuh"

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
// Input j of the initializer at a node of mode md (LeggedRobotInitializer::compute, LeggedRobotInitializer.cpp:67-77): the stance feet
// share the robot's weight in z, everything else is zero.
__device__ __forceinline__ double initializer_input(int md, int j) {
  int ns = 0;
  for (int c = 0; c < 4; ++c) ns += contact_flag(md, c);
  return (j < 12 && (j % 3) == 2 && contact_flag(md, j / 3)) ? c_model.total_mass * HB_GRAVITY / ns : 0.0;
}

// LeggedRobotInitializer::compute (initialization/LeggedRobotInitializer.cpp:67-77)
__global__ void cold_start_kernel(int B, int N, const double* x0, const int32_t* mode, double* xt, double* ut) {
  const int inst = blockIdx.x;
  const double* x = x0 + (size_t)inst * NX;
  for (int idx = threadIdx.x; idx < (N + 1) * NX; idx += blockDim.x) xt[(size_t)inst * (N + 1) * NX + idx] = x[idx % NX];
  for (int idx = threadIdx.x; idx < N * NU; idx += blockDim.x) {
    const int k = idx / NU, j = idx - k * NU;
    ut[(size_t)inst * N * NU + idx] = initializer_input(mode[(size_t)inst * (N + 1) + k], j);
  }
}

// index k of the interval [tk[k], tk[k+1]) of a grid with n intervals that holds t (clamped to 0 .. n-1), and the interpolation weight
__device__ __forceinline__ int grid_interval(const double* tk, int n, double t, double& al) {
  int lo = 0, hi = n;                     // invariant: tk[lo] <= t (or lo == 0), tk[hi] > t (or hi == n)
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (tk[mid] <= t) lo = mid; else hi = mid; }
  const double d = tk[lo + 1] - tk[lo];
  double a = d > 0.0 ? (t - tk[lo]) / d : 0.0;
  al = a < 0.0 ? 0.0 : (a > 1.0 ? 1.0 : a);
  return lo;
}

// The same on the uniform grid of n intervals, with s = (t - t_0) / dt the caller computes: s clamped to [0, n], k = floor(s) capped at
// n - 1, weight s - k
__device__ __forceinline__ int uniform_interval(double s, int n, double& al) {
  if (s < 0.0) s = 0.0;
  if (s > (double)n) s = (double)n;
  int k = (int)floor(s);
  if (k >= n) k = n - 1;
  al = s - k;
  return k;
}

// One solution of B instances as the kernels store it (the resident solution, or the adopted policy of the MRT split): solve time, node
// times and interval counts (event-node grids; null on uniform ones), state / input trajectories, node modes
struct SolutionRows {
  double *t0, *xt, *ut, *tk;
  int32_t *mode, *nn;
};

// Warm start of the next solve from the resident primal solution (ocs2::SqpSolver::initializeStateInputTrajectories; mpc.coldStart
// false, task.info:146): x[0] = measured state; interval i takes u[i] = previous input at t_i and x[i+1] = previous state at t_{i+1}
// while t_{i+1} lies inside the previous horizon, otherwise the initializer (weight-compensating input, state kept,
// LeggedRobotInitializer.cpp:67-77). One block per instance; the previous trajectories are staged in shared memory so that the
// update can be done in place. With event-node grids (tk_new != null) both the previous and the new node times are arbitrary:
// res.tk / res.nn hold the previous grid and are replaced by the new one at the end.
__global__ void __launch_bounds__(128) warm_shift_kernel(int B, int N, double dt, const double* t0_new, const double* x0, const int32_t* mode,
                                                          const double* tk_new, const int32_t* nn_new, SolutionRows res) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* px = reinterpret_cast<double*>(smem_raw);
  double* pu = px + (size_t)(N + 1) * NX;
  __shared__ double ptk[HB_MAX_HORIZON + 1];
  const int inst = blockIdx.x;
  const bool grid = tk_new != nullptr;
  double* x = res.xt + (size_t)inst * (N + 1) * NX; double* u = res.ut + (size_t)inst * N * NU;
  for (int i = threadIdx.x; i < (N + 1) * NX; i += blockDim.x) px[i] = x[i];
  for (int i = threadIdx.x; i < N * NU; i += blockDim.x) pu[i] = u[i];
  const int np = grid ? res.nn[inst] : N;                        // intervals of the previous grid
  const int nw = grid ? nn_new[inst] : N;                        // intervals of the new grid
  const double* tn_ = grid ? tk_new + (size_t)inst * (N + 1) : nullptr;
  if (grid) for (int i = threadIdx.x; i <= N; i += blockDim.x) ptk[i] = res.tk[(size_t)inst * (N + 1) + i];
  __syncthreads();
  const double tp = grid ? ptk[0] : res.t0[inst], tn = t0_new[inst], t_end = grid ? ptk[np] : tp + N * dt;
  auto new_time = [&](int k) { return grid ? tn_[k < nw ? k : nw] : tn + k * dt; };
  auto locate = [&](double t, double& al) {
    if (grid) return grid_interval(ptk, np, t, al);
    return uniform_interval((t - tp) / dt, N, al);
  };
  auto prev_state = [&](double t, int j) { double al; const int k = locate(t, al); return (1.0 - al) * px[k * NX + j] + al * px[(k + 1) * NX + j]; };
  auto prev_input = [&](double t, int j) {
    double al; const int k = locate(t, al);
    const int k1 = (k + 1 < np) ? k + 1 : np - 1;
    return (1.0 - al) * pu[k * NU + j] + al * pu[k1 * NU + j];
  };
  // first interval that falls back to the initializer: smallest i with t_{i+1} > t_end (1e-9 guards the grid-aligned case)
  int istar = nw;
  for (int i = 0; i < nw; ++i) if (new_time(i + 1) > t_end + 1e-9) { istar = i; break; }
  for (int idx = threadIdx.x; idx < (N + 1) * NX; idx += blockDim.x) {
    const int k = idx / NX, j = idx - k * NX;
    const int ks = k <= istar ? k : istar;                 // the initializer keeps the state of node istar
    x[idx] = (ks == 0) ? x0[(size_t)inst * NX + j] : prev_state(new_time(ks), j);
  }
  for (int idx = threadIdx.x; idx < N * NU; idx += blockDim.x) {
    const int k = idx / NU, j = idx - k * NU;
    u[idx] = k < istar ? prev_input(new_time(k), j) : initializer_input(mode[(size_t)inst * (N + 1) + k], j);
  }
  __syncthreads();
  if (threadIdx.x == 0) { res.t0[inst] = tn; if (grid) res.nn[inst] = nw; }
  if (grid) for (int i = threadIdx.x; i <= N; i += blockDim.x) res.tk[(size_t)inst * (N + 1) + i] = tn_[i];
}

// The per-instance source choice of policy_eval_kernel: an instance with an MPC latency lat.of(inst) >= 1 evaluates `adopted` instead of
// the solution the kernel was given. An unset lat: every instance evaluates the given one.
struct PolicyChoice {
  InstanceView<int32_t> lat;
  SolutionRows adopted;
};

// MPC_MRT_Interface::updatePolicy, one warp per instance: the resident solution `from` is copied into the adopted policy `to` of the
// instances that adopt. With lat set (the episodes), an instance with latency d = *lat.of(inst) >= 1 adopts on tick `tick` iff tick >= d
// and (tick - d) % every == 0, and every such instance adopts when tick < 0 (the cold tick's adoption after its cycle); with lat unset,
// the instances with update[inst] != 0 adopt (update null: all).
__global__ void policy_adopt_kernel(int B, int N, InstanceView<int32_t> lat, long long tick, int every, const uint8_t* update, SolutionRows from,
                                    SolutionRows to) {
  const int inst = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (inst >= B) return;
  const int lane = threadIdx.x & 31;
  if (lat.recs) {
    const int32_t* d = lat.of(inst);
    if (!d || *d < 1 || (tick >= 0 && (tick < *d || (tick - *d) % every != 0))) return;
  } else if (update && !update[inst]) {
    return;
  }
  const size_t nx = (size_t)(N + 1) * NX, nu = (size_t)N * NU, i = (size_t)inst;
  for (size_t k = lane; k < nx; k += 32) to.xt[i * nx + k] = from.xt[i * nx + k];
  for (size_t k = lane; k < nu; k += 32) to.ut[i * nu + k] = from.ut[i * nu + k];
  for (int k = lane; k <= N; k += 32) to.mode[i * (N + 1) + k] = from.mode[i * (N + 1) + k];
  if (from.tk) for (int k = lane; k <= N; k += 32) to.tk[i * (N + 1) + k] = from.tk[i * (N + 1) + k];
  if (lane == 0) {
    to.t0[inst] = from.t0[inst];
    if (from.nn) to.nn[inst] = from.nn[inst];
  }
}

// MPC_MRT_Interface::evaluatePolicy with the feed-forward policy (LeggedController.cpp:154-156, task.info:93): linear interpolation of
// the state / input trajectories of s at t0 + t_rel (s.t0 read only with t_abs); mode = the node mode of the interval holding that time
// (the interval ending there at a node where the mode changes). choice: see PolicyChoice.
__global__ void policy_eval_kernel(int B, int N, double dt, double t_rel, SolutionRows s, double* x_des, double* u_des, int32_t* mode_out,
                                   const double* t_abs, PolicyChoice choice) {
  const int inst = blockIdx.x * blockDim.x / 32 + (threadIdx.x >> 5);
  if (inst >= B) return;
  const int lane = threadIdx.x & 31;
  const int32_t* d = choice.lat.of(inst);
  if (d && *d >= 1) s = choice.adopted;
  if (t_abs) t_rel = t_abs[inst] - s.t0[inst];        // evaluation at an absolute time per instance (500 Hz WBC ticks between MPC updates)
  int k, na = N;
  double al;
  if (s.tk) {      // event-node grid: node times of this instance
    const double* t = s.tk + (size_t)inst * (N + 1);
    na = s.nn[inst];
    k = grid_interval(t, na, t[0] + t_rel, al);
  } else {
    k = uniform_interval(t_rel / dt, N, al);
  }
  const double* x = s.xt + (size_t)inst * (N + 1) * NX;
  const double* u = s.ut + (size_t)inst * N * NU;
  if (lane < NX) {
    x_des[(size_t)inst * NX + lane] = (1.0 - al) * x[k * NX + lane] + al * x[(k + 1) * NX + lane];
    const int k1 = (k + 1 < na) ? k + 1 : na - 1;   // the input trajectory repeats its last sample at the final node
    u_des[(size_t)inst * NU + lane] = (1.0 - al) * u[k * NU + lane] + al * u[k1 * NU + lane];
  }
  // mode in force at t: ModeSchedule::modeAtTime finds a switch at t by lower_bound, so the earlier mode holds AT a switching time; a node
  // whose mode differs from its predecessor's starts a new mode, and exactly at that node the interval ending there still holds
  if (lane == 0 && mode_out) {
    const int32_t* md = s.mode + (size_t)inst * (N + 1);
    mode_out[inst] = (al == 0.0 && k > 0 && md[k] != md[k - 1]) ? md[k - 1] : md[k];
  }
}

// store the solve time (and, with tk_new, the node grid) of a cold-started resident solution res
__global__ void set_times_kernel(int B, int N, const double* t0_new, const double* tk_new, const int32_t* nn_new, SolutionRows res) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  res.t0[i] = t0_new[i];
  if (tk_new) {
    res.nn[i] = nn_new[i];
    for (int k = 0; k <= N; ++k) res.tk[(size_t)i * (N + 1) + k] = tk_new[(size_t)i * (N + 1) + k];
  }
}
}  // namespace
