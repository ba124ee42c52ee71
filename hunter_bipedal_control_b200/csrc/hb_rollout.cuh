// Closed-loop episodes (hb_rollout_batch_dev, SURVEY 8f row N2): the per-instance kernels the episode loop adds around the device planner,
// the resident cycle, the 500 Hz WBC tick, the joint command law, the actuation model and the plant. One thread per instance.
#pragma once
#include "hb_common.cuh"
#include "hb_rbd.cuh"

namespace hb {

// Plan inputs of the MPC cycle at time t, with the defaults of api.make_plan_inputs: x0 = the centroidal restatement of the measured rbd,
// cmd_vel of the last command segment that has started (the first one before that), prev_event = min(t, gait_start) - 0.5, IK joint
// references. feet_pos is left zero: plan_prepare_kernel computes the feet from x0.
__global__ void rollout_plan_inputs_kernel(int B, double t, double horizon, const hb_rollout_command* cmd, const double* rbd, hb_plan_input* in) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const hb_rollout_command& c = cmd[inst];
  hb_plan_input& p = in[inst];
  p.t0 = t; p.horizon = horizon; p.time_to_target = horizon;
  p.gait_start = c.gait_start; p.prev_event = (c.gait_start < t ? c.gait_start : t) - 0.5;
  int j = 0;
  for (int k = 1; k < c.n_cmd; ++k) if (c.cmd_time[k] <= t) j = k;
  for (int i = 0; i < 4; ++i) p.cmd_vel[i] = c.cmd_vel[j][i];
  rbd_to_centroidal(rbd + (size_t)inst * 32, p.x0);
  for (int i = 0; i < 12; ++i) p.feet_pos[i] = 0.0;
  p.gait = c.gait; p.joint_ik = 1;
}

// failure bits of a state entering a tick; the orientation and height checks are only meaningful on a finite state
__device__ __forceinline__ int rollout_state_check(const double* r, double min_base_height) {
  for (int i = 0; i < 32; ++i) if (!isfinite(r[i])) return HB_ROLLOUT_FAIL_NONFINITE;
  int why = 0;
  if (r[2] > M_PI_2 || r[2] < -M_PI_2) why |= HB_ROLLOUT_FAIL_ORIENTATION;     // zyx[2] = roll: SafetyChecker::checkOrientation
  if (min_base_height != 0.0 && r[5] < min_base_height) why |= HB_ROLLOUT_FAIL_HEIGHT;
  return why;
}

// Start of tick `tick` (absolute): the state entering it is checked (an instance that fails is held from this tick on), `held` takes the
// state every held instance is put back to, the tick time goes to every instance (policy evaluation, actuation stamp), and the state is
// logged when log_row is set. A non-finite state can only enter the first tick of a call (the end kernel never leaves one behind); with no
// finite state of that instance known, the nominal standing pose replaces it.
__global__ void rollout_tick_begin_kernel(int B, int tick, double t, double min_base_height, double* rbd, double* held, hb_rollout_stats* stats,
                                          double* t_now, double* log_row, size_t log_stride) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  double* r = rbd + (size_t)inst * 32;
  double* h = held + (size_t)inst * 32;
  hb_rollout_stats& s = stats[inst];
  const int why = rollout_state_check(r, min_base_height);
  if (why && s.fail_tick < 0) { s.fail_tick = tick; s.fail_reason = why; }
  if (why & HB_ROLLOUT_FAIL_NONFINITE) {
    const double nominal[NQ] = {0.0, 0.0, 0.0, 0.0, 0.0, HB_INITIAL_STATE[8], HB_INITIAL_STATE[12], HB_INITIAL_STATE[13], HB_INITIAL_STATE[14],
                                HB_INITIAL_STATE[15], HB_INITIAL_STATE[16], HB_INITIAL_STATE[17], HB_INITIAL_STATE[18], HB_INITIAL_STATE[19],
                                HB_INITIAL_STATE[20], HB_INITIAL_STATE[21]};
    for (int i = 0; i < 32; ++i) r[i] = i < NQ ? nominal[i] : 0.0;
  }
  for (int i = 0; i < 32; ++i) h[i] = r[i];
  t_now[inst] = t;
  if (log_row) for (int i = 0; i < 32; ++i) log_row[inst * log_stride + i] = r[i];
}

// actuator saturation of the applied torques (B x 10); NaN passes through as in numpy.clip
__global__ void rollout_saturate_kernel(int B, hb_rollout_params p, double* tau) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * NJ) return;
  const double lim = p.torque_limit[idx % NJ], v = tau[idx];
  tau[idx] = v < -lim ? -lim : (v > lim ? lim : v);
}

// End of tick `tick`, after the plant step: the tick's outputs count for instances that were up when it began; the emergency stop the joint
// command raised fails the instance at this tick; failed instances are put back to `held`; a non-finite new state fails the instance at the
// next tick (the state entering it) and is put back too, so no non-finite state reaches the planner or a solver.
__global__ void rollout_tick_end_kernel(int B, int tick, int mpc_tick, const hb_solve_info* info, const int32_t* plan_status, const int32_t* wbc_status,
                                        const uint8_t* estop, const double* tau, const double* held, double* rbd, hb_rollout_stats* stats) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  hb_rollout_stats& s = stats[inst];
  double* r = rbd + (size_t)inst * 32;
  if (s.fail_tick < 0) {
    if (mpc_tick) { s.mpc_bad += info[inst].status != 0; s.plan_rejects += plan_status[inst] != 0; }
    s.wbc_fallbacks += wbc_status[inst] != 0;
    double m = s.max_abs_torque;
    for (int j = 0; j < NJ; ++j) { const double a = fabs(tau[(size_t)inst * NJ + j]); if (a > m) m = a; }
    s.max_abs_torque = m;
    if (estop[inst]) { s.fail_tick = tick; s.fail_reason = HB_ROLLOUT_FAIL_ESTOP; }
  }
  bool restore = s.fail_tick >= 0;
  if (!restore) {
    for (int i = 0; i < 32; ++i) if (!isfinite(r[i])) restore = true;
    if (restore) { s.fail_tick = tick + 1; s.fail_reason = HB_ROLLOUT_FAIL_NONFINITE; }
  }
  if (restore) for (int i = 0; i < 32; ++i) r[i] = held[(size_t)inst * 32 + i];
}

}  // namespace hb
