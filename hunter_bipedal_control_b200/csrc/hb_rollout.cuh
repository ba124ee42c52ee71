// Closed-loop episodes (hb_rollout_batch_dev, SURVEY 8f row N2): the joint command law, the actuation model and the plant, and the
// per-instance kernels the episode loop adds around them, the device planner, the resident cycle and the 500 Hz WBC tick.
#pragma once
#include "hb_bridge.cuh"
#include "hb_common.cuh"
#include "hb_planner.h"
#include "hb_qp.cuh"
#include "hb_rbd.cuh"
#include "../../include/hunter_b200.h"

namespace hb {

// The publisher state of a teleoperated instance (teleoperation, hunter_b200.h; per-instance context state, zero when cleared): the
// filtered command last (vx, vy, vz, yaw rate) and 1 + the index of the goal in force it last saw (0: none), so that a goal a message
// replaced is not captured again
struct TeleopState { double last[4]; int32_t goal_seen, pad; };
// The captured-target source of an instance whose target a teleop message wrote: beyond every goal index, so the planner plans on it
constexpr int32_t TELEOP_CAPTURED = HB_MAX_GOALS;

// The contact detection state of an instance (contact detection, hunter_b200.h; per-instance context state): the observer's filtered
// momentum and last output, the effort it reads next (the last tick's applied torque) and the flags the filter last used
struct ContactDetectState { double p_filtered[16], force[16], effort[10]; uint8_t flags[4]; int32_t pad; };
// The contact detection of the estimated episodes: the setting and the states (indexed as the setting's records); an empty view detects none
struct ContactDetect {
  InstanceView<hb_contact_detection> set;
  ContactDetectState* st;
};
// The cleared state: no momentum, no effort, no flags used, the output the constructor fills with 50 (StateEstimateBase.cpp:61-62)
__host__ __device__ inline void contact_detect_clear(ContactDetectState& d) {
  for (int i = 0; i < 16; ++i) { d.p_filtered[i] = 0.0; d.force[i] = 50.0; }
  for (int j = 0; j < 10; ++j) d.effort[j] = 0.0;
  for (int c = 0; c < 4; ++c) d.flags[c] = 0;
  d.pad = 0;
}

// whether the joystick of record s sends a message on absolute tick a: inside a window, on its period from the window's start
__device__ __forceinline__ bool teleop_message(const hb_teleop_setting& s, int a) {
  for (int w = 0; w < s.n_window && w < HB_MAX_TELEOP_WINDOWS; ++w)
    if (s.on_tick[w] <= a && a < s.off_tick[w] && (a - s.on_tick[w]) % s.period_ticks == 0) return true;
  return false;
}

// Plan inputs of the MPC cycle at time t, with the defaults of api.make_plan_inputs: x0 = the centroidal restatement of the measured rbd,
// cmd_vel of the last command segment that has started (the first one before that), prev_event = min(t, gait_start) - 0.5, IK joint
// references. feet_pos is left zero: plan_prepare_kernel computes the feet from x0. With est (estimated episodes) x0[9] is the unwrapped
// observation yaw (LeggedController.cpp:335-337).
// Goals (hb_goal_schedule, hunter_b200.h) of the instances that have one: the goal in force at t is captured, target and index, when it differs
// from the captured one (captured_idx -1: none); reset (an episode's tick 0) forgets the captured goal first. The planner reads them.
// Teleoperated instances (a record in teleop; publisher state pub): the goal capture compares with the goal they last saw, then a message
// due on tick a runs the publisher step and captures the cmd_vel target of last (source TELEOP_CAPTURED); they plan with cmd_vel = last.
// Both captures of an instance with a record in maps build their targets on that height map (height maps, hunter_b200.h).
__global__ void rollout_plan_inputs_kernel(int B, int a, double t, double horizon, const hb_rollout_command* cmd, const double* rbd,
                                           const hb_estimation_state* est, hb_plan_input* in, InstanceView<hb_goal_schedule> goals,
                                           InstanceView<hb_teleop_setting> teleop, TeleopState* pub, int reset, hb_target* captured,
                                           int32_t* captured_idx, hbplan::PlanConsts pc, InstanceView<hb_terrain> maps) {
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
  if (est) p.x0[9] = est[inst].yaw_obs;
  for (int i = 0; i < 12; ++i) p.feet_pos[i] = 0.0;
  p.gait = c.gait; p.joint_ik = 1;
  const hb_teleop_setting* tp = teleop.of(inst);
  TeleopState* ts = tp ? pub + inst : nullptr;
  if (ts && reset) {
    for (int i = 0; i < 4; ++i) ts->last[i] = 0.0;
    ts->goal_seen = 0;
    captured_idx[inst] = -1;
  }
  if (const hb_goal_schedule* sp = goals.of(inst)) {
    const hb_goal_schedule& s = *sp;
    int g = -1;
    for (int k = 0; k < s.n_goal; ++k) if (s.time[k] <= t) g = k;
    const int had = ts ? ts->goal_seen - 1 : reset ? -1 : captured_idx[inst];
    if (g >= 0 && g != had) {
      hbplan::goal_to_target(pc, t, p.x0, s.goal[g], captured[inst], maps.of(inst));
      if (ts) captured_idx[inst] = g;
    }
    if (ts) ts->goal_seen = (g >= 0 ? g : had) + 1;
    else captured_idx[inst] = g >= 0 ? g : had;
  }
  if (ts) {
    if (teleop_message(*tp, a)) {     // TargetTrajectoriesPublisher's cmdVelCallback
      double* last = ts->last;
      for (int k : {0, 1, 3}) {
        const double lim = tp->change_limit[k == 3 ? 2 : k];
        double d = p.cmd_vel[k] - last[k];
        d = d > 0 ? fmin(d, lim) : fmax(d, -lim);
        last[k] += d;
      }
      last[2] = 0.0;
      hbplan::cmd_vel_to_target(pc, last, t, p.x0, horizon, captured[inst], maps.of(inst));
      captured_idx[inst] = TELEOP_CAPTURED;
    }
    for (int i = 0; i < 4; ++i) p.cmd_vel[i] = ts->last[i];
  }
}

// failure bits of a state entering a tick; the orientation and height checks are only meaningful on a finite state. ter (nullable): the
// terrain of the instance, above which the base height is measured; null measures it from z = 0.
__device__ __forceinline__ int rollout_state_check(const double* r, double min_base_height, const hb_terrain* ter) {
  for (int i = 0; i < 32; ++i) if (!isfinite(r[i])) return HB_ROLLOUT_FAIL_NONFINITE;
  int why = 0;
  if (r[2] > M_PI_2 || r[2] < -M_PI_2) why |= HB_ROLLOUT_FAIL_ORIENTATION;     // zyx[2] = roll: SafetyChecker::checkOrientation
  if (min_base_height != 0.0) {
    double z = r[5];
    if (ter) { double gx, gy; z -= hbplan::terrain_height<false>(*ter, r[3], r[4], &gx, &gy); }
    if (z < min_base_height) why |= HB_ROLLOUT_FAIL_HEIGHT;
  }
  return why;
}

// The world wrench (force, couple) the push schedule s puts on the plant step of the tick at time t: the active pushes added in ascending j
// to zeros, so that a host restatement reproduces it bit for bit
__device__ __forceinline__ void push_wrench(const hb_push_schedule& s, double t, double* w) {
  for (int c = 0; c < 6; ++c) w[c] = 0.0;
  for (int j = 0; j < s.n_push; ++j) {
    if (!(s.t_start[j] <= t && t < s.t_start[j] + s.duration[j])) continue;
    for (int c = 0; c < 3; ++c) { w[c] += s.force[j][c]; w[3 + c] += s.torque[j][c]; }
  }
}

// Start of tick `tick` (absolute): the state entering it is checked (an instance that fails is held from this tick on), `held` takes the
// state every held instance is put back to, the tick time goes to every instance (policy evaluation, actuation stamp), and the state is
// logged when log_row is set. A non-finite state can only enter the first tick of a call (the end kernel never leaves one behind); with no
// finite state of that instance known, the nominal standing pose replaces it. With wrench set, the tick's push wrench (B x 6) is written
// for the plant step: from the instance's push schedule, zeros without one. The base height of an instance with a terrain is measured
// above it.
__global__ void rollout_tick_begin_kernel(int B, int tick, double t, double min_base_height, double* rbd, double* held, hb_rollout_stats* stats,
                                          double* t_now, double* log_row, size_t log_stride, InstanceView<hb_push_schedule> pushes, double* wrench,
                                          InstanceView<hb_terrain> terrain) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  double* r = rbd + (size_t)inst * 32;
  double* h = held + (size_t)inst * 32;
  hb_rollout_stats& s = stats[inst];
  const int why = rollout_state_check(r, min_base_height, terrain.of(inst));
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
  if (wrench) {
    double* w = wrench + (size_t)inst * 6;
    if (const hb_push_schedule* ps = pushes.of(inst)) push_wrench(*ps, t, w);
    else for (int c = 0; c < 6; ++c) w[c] = 0.0;
  }
}

// actuator saturation of the applied torques (B x 10); NaN passes through as in numpy.clip. An instance with a hardware record in `hw`
// saturates at its limits in place of p.torque_limit.
__global__ void rollout_saturate_kernel(int B, hb_rollout_params p, InstanceView<hb_hardware_setting> hw, double* tau) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * NJ) return;
  const hb_hardware_setting* h = hw.of(idx / NJ);
  const double lim = h ? h->torque_limit[idx % NJ] : p.torque_limit[idx % NJ], v = tau[idx];
  tau[idx] = v < -lim ? -lim : (v > lim ? lim : v);
}

// End of tick `tick`, after the plant step: the tick's outputs count for instances that were up when it began; the emergency stop the joint
// command raised fails the instance at this tick; failed instances are put back to `held`; a non-finite new state fails the instance at the
// next tick (the state entering it) and is put back too, so no non-finite state reaches the planner or a solver. An instance with contact
// detection (det) stores the tick's applied torque as its next effort: here, after the plant step, because a bridged instance's applied
// torque is the plant's (motor bridge, hunter_b200.h).
__global__ void rollout_tick_end_kernel(int B, int tick, int mpc_tick, const hb_solve_info* info, const int32_t* plan_status, const int32_t* wbc_status,
                                        const uint8_t* estop, const double* tau, const double* held, double* rbd, hb_rollout_stats* stats, ContactDetect det) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  if (det.set.of(inst)) for (int j = 0; j < NJ; ++j) det.st[inst].effort[j] = tau[(size_t)inst * NJ + j];
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

// ---- recorded channels (hb_rollout_set_channel, hunter_b200.h)
// Elements per row of each channel and the size of one element, by HB_CHANNEL_* index
constexpr int CHANNEL_WIDTH[HB_CHANNELS] = {NJ, NJ * 5, NX, NU, NWBC, 1, 12, 4, 30, 3};
constexpr int CHANNEL_BYTES[HB_CHANNELS] = {8, 8, 8, 8, 8, 4, 8, 1, 8, 4};
// The channels one recorded tick writes, in ascending channel order: channel[k]'s elements are the instance's elements first[k] ..
// first[k + 1] - 1 of width in all; dst[k] is that channel's row for the tick at instance 0, and stride[k] its elements per instance.
struct RecordSlots {
  int n, width;
  int channel[HB_CHANNELS], first[HB_CHANNELS];
  size_t stride[HB_CHANNELS];
  void* dst[HB_CHANNELS];
};
// What the tick computed, in the episode's scratch (instance-major): sensors only in estimated episodes, contact forces only when a
// contact channel is recorded, info and plan status only on an MPC tick.
struct RecordSources {
  const double *tau, *jcmd, *xdes, *udes, *sol, *cforce;
  const int32_t *mode, *wstatus, *pstat;
  const uint8_t* cflag;
  const hb_solve_info* info;
  const double *quat, *gyro, *acc, *jpos, *jvel;
  int mpc;
};

// One recorded tick: one thread per recorded element of every instance, so that consecutive threads write consecutive addresses of an
// instance's row. Reads only; the tick's values are copied as they are.
__global__ void rollout_record_kernel(int B, const __grid_constant__ RecordSlots s, const __grid_constant__ RecordSources src) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)B * s.width) return;
  const int inst = (int)(idx / s.width);
  int e = (int)(idx % s.width), k = 0;
  while (k + 1 < s.n && e >= s.first[k + 1]) ++k;
  e -= s.first[k];
  const size_t at = (size_t)inst * s.stride[k] + e;
  double* d = static_cast<double*>(s.dst[k]);
  switch (s.channel[k]) {
    case HB_CHANNEL_TORQUE: d[at] = src.tau[(size_t)inst * NJ + e]; break;
    case HB_CHANNEL_JOINT_COMMAND: d[at] = src.jcmd[(size_t)inst * NJ * 5 + e]; break;
    case HB_CHANNEL_X_DES: d[at] = src.xdes[(size_t)inst * NX + e]; break;
    case HB_CHANNEL_U_DES: d[at] = src.udes[(size_t)inst * NU + e]; break;
    case HB_CHANNEL_WBC_SOLUTION: d[at] = src.sol[(size_t)inst * NWBC + e]; break;
    case HB_CHANNEL_MODE: static_cast<int32_t*>(s.dst[k])[at] = src.mode[inst]; break;
    case HB_CHANNEL_CONTACT_FORCE: d[at] = src.cforce[(size_t)inst * 12 + e]; break;
    case HB_CHANNEL_CONTACT_FLAG: static_cast<uint8_t*>(s.dst[k])[at] = src.cflag[(size_t)inst * 4 + e]; break;
    case HB_CHANNEL_SENSORS:
      d[at] = e < 4 ? src.quat[(size_t)inst * 4 + e] : e < 7 ? src.gyro[(size_t)inst * 3 + e - 4] : e < 10 ? src.acc[(size_t)inst * 3 + e - 7]
              : e < 20 ? src.jpos[(size_t)inst * NJ + e - 10] : src.jvel[(size_t)inst * NJ + e - 20];
      break;
    case HB_CHANNEL_STATUS:
      static_cast<int32_t*>(s.dst[k])[at] = e == 0 ? src.wstatus[inst] : !src.mpc ? -1 : e == 1 ? src.info[inst].status : src.pstat[inst];
      break;
  }
}

// ---- episode snapshots (hb_episode_save_async / hb_episode_restore, hunter_b200.h)
constexpr int EPISODE_MAX_SEGMENTS = 20;
// One per-instance buffer of a snapshot row: the context's buffer (instance-major, `bytes` per instance, a multiple of 4) and the row's
// 8-byte words first .. first + ceil(bytes / 8) - 1 that hold it. A null buffer is one the context never allocated: a save writes `fill`
// in each of its 4-byte units, a restore skips it. by_row: the buffer is indexed by the row instead of the context instance (the headers a
// save stages).
struct EpisodeSegment {
  char* buf;
  uint32_t bytes, first, fill;
  int32_t by_row;
};
struct EpisodeSegments {
  int n;
  uint32_t row_words;
  EpisodeSegment seg[EPISODE_MAX_SEGMENTS];
};

// Save (restore == 0): row i <- instance src[i] of every segment. Restore: instance i <- row src[i]. src null: i. One thread per 8-byte
// word of the B rows written or read, so that consecutive threads touch consecutive addresses of a row and of a segment; the copy goes in
// 4-byte units because int32 segments (node modes, interval counts, goal index) leave the context's per-instance strides 4-byte aligned.
// The padding of a row is written as zeros.
__global__ void episode_copy_kernel(int B, const __grid_constant__ EpisodeSegments t, const int32_t* src, int restore, uint32_t* rows) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)B * t.row_words) return;
  const int i = (int)(idx / t.row_words);
  const uint32_t w = (uint32_t)(idx % t.row_words);
  int k = 0;
  while (k + 1 < t.n && w >= t.seg[k + 1].first) ++k;
  const EpisodeSegment& s = t.seg[k];
  const uint32_t off = (w - s.first) * 8;
  const bool two = off + 4 < s.bytes;
  const int other = src ? src[i] : i;
  uint32_t* row = rows + ((size_t)(restore ? other : i) * t.row_words + w) * 2;
  if (restore) {
    if (!s.buf) return;
    uint32_t* c = reinterpret_cast<uint32_t*>(s.buf + (size_t)i * s.bytes + off);
    c[0] = row[0];
    if (two) c[1] = row[1];
  } else {
    const uint32_t* c = s.buf ? reinterpret_cast<const uint32_t*>(s.buf + (size_t)(s.by_row ? i : other) * s.bytes + off) : nullptr;
    row[0] = c ? c[0] : s.fill;
    row[1] = !two ? 0u : c ? c[1] : s.fill;
  }
}

// ---- estimated episodes (hb_rollout_estimated_batch_dev, hb_sim_read_sensors_batch_dev)

// Philox4x32-10 (Salmon et al., SC'11): counter c encrypted under key (k0, k1), in place. Written out rather than taken from curand so that
// the noise is a documented function a test can restate.
__device__ __forceinline__ void philox4x32_10(uint32_t k0, uint32_t k1, uint32_t c[4]) {
  for (int round = 0; round < 10; ++round) {
    if (round) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1;
    c[0] = n0; c[1] = (uint32_t)p1; c[2] = n2; c[3] = (uint32_t)p0;
  }
}

// Noise block numbers: each sensor channel owns fixed blocks of 4 normals, so a channel with sigma 0 draws nothing and shifts no other one.
enum { NOISE_BLOCK_ORIENTATION = 0, NOISE_BLOCK_GYRO = 1, NOISE_BLOCK_ACCEL = 2, NOISE_BLOCK_JOINT_POS = 3, NOISE_BLOCK_JOINT_VEL = 6 };

// v[0..m) += sigma x normals of blocks block0, block0 + 1, ...: counter (block, tick, stream_lo, stream_hi), key (seed_lo, seed_hi); the 4 words
// w of a block are u = (w + 0.5) 2^-32 and Box-Muller turns (u0, u1) and (u2, u3) into normals 0, 1 and 2, 3.
__device__ __forceinline__ void add_sensor_noise(double sigma, uint64_t seed, int block0, uint32_t tick, uint64_t stream, double* v, int m) {
  if (!(sigma > 0.0)) return;
  double n[4];
  for (int j = 0; j < m; ++j) {
    if (j % 4 == 0) {
      uint32_t c[4] = {(uint32_t)(block0 + j / 4), tick, (uint32_t)stream, (uint32_t)(stream >> 32)};
      philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), c);
      for (int h = 0; h < 2; ++h) {
        const double u0 = ((double)c[2 * h] + 0.5) * 0x1p-32, u1 = ((double)c[2 * h + 1] + 0.5) * 0x1p-32;
        const double r = sqrt(-2.0 * log(u0));
        double s, co;
        sincos(2.0 * M_PI * u1, &s, &co);
        n[2 * h] = r * co; n[2 * h + 1] = r * s;
      }
    }
    v[j] += sigma * n[j % 4];
  }
}

// v[0..m) += off[0..m), skipping the entries equal to 0.0 so that a -0.0 reading keeps its sign (simulated hardware, hunter_b200.h)
__device__ __forceinline__ void add_sensor_offset(const double* off, double* v, int m) {
  for (int j = 0; j < m; ++j) if (off[j] != 0.0) v[j] += off[j];
}

// The simulated robot's sensors at absolute tick `tick` from the true rbd r (LeggedHWSim::readSim, LeggedHWSim.cpp:116-130, and the joint
// encoders). The accelerometer differences the world base velocity over the last plant step (accel_dt) where Gazebo reads the instantaneous
// acceleration; unprimed, it reads gravity only. Updates base_vel_prev / primed. hw (nullable): the robot's hardware record, whose offsets
// are added before the noise and whose sigmas replace nz's. mb (nullable): the robot's motor bridge, whose encoders the joint readings pass
// after the noise.
__device__ __forceinline__ void read_sensors(const hb_sensor_noise& nz, const hb_hardware_setting* hw, const hb_motor_bridge* mb, uint32_t tick,
                                             double accel_dt, const double* r, hb_estimation_state& e, double* quat, double* gyro, double* acc,
                                             double* jp, double* jv) {
  double sz, cz, sy, cy, sx, cx;
  sincos(r[0], &sz, &cz); sincos(r[1], &sy, &cy); sincos(r[2], &sx, &cx);
  const double R[9] = {cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx, sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx, -sy, cy * sx, cy * cx};
  double aw[3] = {0.0, 0.0, 0.0};
  if (e.primed) for (int i = 0; i < 3; ++i) aw[i] = (r[NQ + 3 + i] - e.base_vel_prev[i]) / accel_dt;
  aw[2] += 9.81;
  double ang[3] = {r[0], r[1], r[2]}, g[3], a[3], q[NJ], qd[NJ];
  for (int i = 0; i < 3; ++i) {
    g[i] = R[i] * r[NQ] + R[3 + i] * r[NQ + 1] + R[6 + i] * r[NQ + 2];           // R' omega_world: RelativeAngularVel
    a[i] = R[i] * aw[0] + R[3 + i] * aw[1] + R[6 + i] * aw[2];
  }
  for (int j = 0; j < NJ; ++j) { q[j] = r[6 + j]; qd[j] = r[NQ + 6 + j]; }
  for (int i = 0; i < 3; ++i) { e.base_vel_prev[i] = r[NQ + 3 + i]; }
  e.primed = 1;
  if (hw) {
    add_sensor_offset(hw->orientation_offset, ang, 3); add_sensor_offset(hw->gyro_bias, g, 3); add_sensor_offset(hw->accel_bias, a, 3);
    add_sensor_offset(hw->encoder_offset, q, NJ);
  }
  const uint64_t st = e.noise_stream;
  add_sensor_noise(hw ? hw->sigma_orientation : nz.orientation, nz.seed, NOISE_BLOCK_ORIENTATION, tick, st, ang, 3);
  add_sensor_noise(hw ? hw->sigma_angular_velocity : nz.angular_velocity, nz.seed, NOISE_BLOCK_GYRO, tick, st, g, 3);
  add_sensor_noise(hw ? hw->sigma_linear_acceleration : nz.linear_acceleration, nz.seed, NOISE_BLOCK_ACCEL, tick, st, a, 3);
  add_sensor_noise(hw ? hw->sigma_joint_position : nz.joint_position, nz.seed, NOISE_BLOCK_JOINT_POS, tick, st, q, NJ);
  add_sensor_noise(hw ? hw->sigma_joint_velocity : nz.joint_velocity, nz.seed, NOISE_BLOCK_JOINT_VEL, tick, st, qd, NJ);
  if (mb) for (int j = 0; j < NJ; ++j) bridge_feedback(*mb, j, &q[j], &qd[j]);
  // quaternion (x, y, z, w) of R = Rz(yaw) Ry(pitch) Rx(roll)
  double hsz, hcz, hsy, hcy, hsx, hcx;
  sincos(0.5 * ang[0], &hsz, &hcz); sincos(0.5 * ang[1], &hsy, &hcy); sincos(0.5 * ang[2], &hsx, &hcx);
  quat[0] = hcz * hcy * hsx - hsz * hsy * hcx; quat[1] = hcz * hsy * hcx + hsz * hcy * hsx;
  quat[2] = hsz * hcy * hcx - hcz * hsy * hsx; quat[3] = hcz * hcy * hcx + hsz * hsy * hsx;
  for (int i = 0; i < 3; ++i) { gyro[i] = g[i]; acc[i] = a[i]; }
  for (int j = 0; j < NJ; ++j) { jp[j] = q[j]; jv[j] = qd[j]; }
}

// ---- odometry (hb_rollout_set_odometry): the tracking camera of each instance, read with its sensors
enum { NOISE_BLOCK_ODOM_DRIFT = 9, NOISE_BLOCK_ODOM_POSITION = 10 };
// The camera state of one instance (per-instance context state): the true base positions of the last HB_ODOM_MAX_DELAY + 1 ticks, by tick
// modulo that count, and the bias
struct OdomCamera { double hist[HB_ODOM_MAX_DELAY + 1][3]; double bias[3]; };
// A camera read: the setting, the camera states (indexed as the setting's records) and where the tick's messages go (pos B x 3, has B).
// With has null there is no read.
struct OdomRead {
  InstanceView<hb_odometry_setting> set;
  OdomCamera* cam;
  double* pos;
  uint8_t* has;
};

// The camera of instance inst at absolute tick `tick` from its true rbd r (hunter_b200.h, odometry): records the base position, and writes
// the message due on this tick (has 1, pos) or none (has 0, pos 0).
__device__ __forceinline__ void read_odometry(const OdomRead& o, int inst, uint64_t seed, uint32_t tick, uint64_t stream, const double* r) {
  const hb_odometry_setting* s = o.set.of(inst);
  double pos[3] = {0.0, 0.0, 0.0};
  uint8_t has = 0;
  if (s && s->period_ticks > 0) {
    OdomCamera& c = o.cam[inst];
    if (tick == 0) {
      for (int k = 0; k < HB_ODOM_MAX_DELAY + 1; ++k) c.hist[k][0] = c.hist[k][1] = c.hist[k][2] = 0.0;
      c.bias[0] = c.bias[1] = c.bias[2] = 0.0;
    }
    for (int k = 0; k < 3; ++k) c.hist[tick % (HB_ODOM_MAX_DELAY + 1)][k] = r[3 + k];
    if (tick % (uint32_t)s->period_ticks == 0 && tick >= (uint32_t)s->delay_ticks) {
      add_sensor_noise(s->sigma_drift, seed, NOISE_BLOCK_ODOM_DRIFT, tick, stream, c.bias, 3);
      const double* p = c.hist[(tick - (uint32_t)s->delay_ticks) % (HB_ODOM_MAX_DELAY + 1)];
      for (int k = 0; k < 3; ++k) pos[k] = p[k] + c.bias[k];
      add_sensor_noise(s->sigma_position, seed, NOISE_BLOCK_ODOM_POSITION, tick, stream, pos, 3);
      has = 1;
    }
  }
  for (int k = 0; k < 3; ++k) o.pos[(size_t)inst * 3 + k] = pos[k];
  o.has[inst] = has;
}

// Contact detection's rule (hunter_b200.h) on the flags f (4, in/out) of an instance with record r at time t: phase times of the schedule of
// e, then estContactState on the observer output force
__device__ __forceinline__ void detect_contacts(const hb_contact_detection& r, const hb_estimation_state& e, double t, const double* force, uint8_t* f) {
  double s[4], en[4];
  hbplan::contact_phase_times(e.has_plan, e.n_events, e.event_times, e.modes, t, s, en);
  hbplan::contact_state(r, t, s, en, force, f);
}

// Sensor read of B instances, one thread each. With cflag (the episode tick) the filter's contact flags come from the stored schedule of the
// latest plan at flag_time, the previous observation's time (LeggedController.cpp:296-297), all 1 before the first plan (:298-304); an
// instance with contact detection (det) then has them replaced by the rule on its stored observer output, its state cleared first on tick 0.
// With odom set (an estimated episode with odometry) each instance's camera is read too. An instance with a record in `hw` reads its
// sensors on it, and one with a record in `bridge` its joints through the bridge's encoders.
__global__ void sensor_read_kernel(int B, hb_sensor_noise nz, InstanceView<hb_hardware_setting> hw, InstanceView<hb_motor_bridge> bridge, uint32_t tick,
                                   double accel_dt, double flag_time, const double* rbd, hb_estimation_state* est, double* quat, double* gyro,
                                   double* acc, double* jp, double* jv, uint8_t* cflag, OdomRead odom, ContactDetect det) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  hb_estimation_state& e = est[inst];
  read_sensors(nz, hw.of(inst), bridge.of(inst), tick, accel_dt, rbd + (size_t)inst * 32, e, quat + (size_t)inst * 4, gyro + (size_t)inst * 3, acc + (size_t)inst * 3,
               jp + (size_t)inst * NJ, jv + (size_t)inst * NJ);
  if (cflag) {
    const int mode = e.has_plan ? hbplan::mode_at(e.n_events, e.event_times, e.modes, flag_time) : 3;
    uint8_t* f = cflag + (size_t)inst * 4;
    for (int c = 0; c < 4; ++c) f[c] = contact_flag(mode, c) ? 1 : 0;
    if (const hb_contact_detection* r = det.set.of(inst)) {
      ContactDetectState& d = det.st[inst];
      if (tick == 0) contact_detect_clear(d);
      detect_contacts(*r, e, flag_time, d.force, f);
      for (int c = 0; c < 4; ++c) d.flags[c] = f[c];
    }
  }
  if (odom.has) read_odometry(odom, inst, nz.seed, tick, e.noise_stream, rbd + (size_t)inst * 32);
}

// hb_contact_state_estimate_async: the rule alone, one thread per instance (records: the staged records of the call)
__global__ void contact_state_kernel(int B, double t, const hb_estimation_state* est, const double* force, InstanceView<hb_contact_detection> records,
                                     uint8_t* flags) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  if (const hb_contact_detection* r = records.of(inst)) detect_contacts(*r, est[inst], t, force + (size_t)inst * 16, flags + (size_t)inst * 4);
}

// hb_sim_read_odometry: the camera read alone, one thread per instance
__global__ void odometry_read_kernel(int B, uint64_t seed, uint32_t tick, const double* rbd, const hb_estimation_state* est, OdomRead odom) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  read_odometry(odom, inst, seed, tick, est[inst].noise_stream, rbd + (size_t)inst * 32);
}

// angles::normalize_angle_positive / normalize_angle / shortest_angular_distance (ROS angles): fmod and one subtraction, all exact
__device__ __forceinline__ double shortest_angular_distance(double from, double to) {
  const double two_pi = 2.0 * M_PI;
  double a = fmod(fmod(to - from, two_pi) + two_pi, two_pi);
  if (a > M_PI) a -= two_pi;
  return a;
}

// The observation step after the filter (LeggedController.cpp:334-337): yaw_obs follows the filter's wrapped yaw by the shortest angular
// distance. Errors of the estimate against the true state entering the tick count while the instance has not failed; est_log takes the
// estimated rbd. The squares and sums are rounded one operation at a time (no contraction) so that a restatement reproduces them.
__global__ void est_observe_kernel(int B, const double* rbd, const double* est_rbd, const hb_rollout_stats* stats, hb_estimation_state* est,
                                   hb_estimation_stats* est_stats, double* log_row, size_t log_stride) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const double* r = rbd + (size_t)inst * 32;
  const double* e = est_rbd + (size_t)inst * 32;
  hb_estimation_state& s = est[inst];
  s.yaw_obs = s.yaw_obs + shortest_angular_distance(s.yaw_obs, e[0]);
  if (est_stats && stats[inst].fail_tick < 0) {
    hb_estimation_stats& es = est_stats[inst];
    const double d0 = e[NQ + 3] - r[NQ + 3], d1 = e[NQ + 4] - r[NQ + 4], d2 = e[NQ + 5] - r[NQ + 5], dz = fabs(e[5] - r[5]);
    const double sq = __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2)), ve = sqrt(sq);
    if (ve > es.max_vel_err) es.max_vel_err = ve;
    if (dz > es.max_height_err) es.max_height_err = dz;
    es.sum_sq_vel_err = __dadd_rn(es.sum_sq_vel_err, sq);
    es.sum_sq_height_err = __dadd_rn(es.sum_sq_height_err, __dmul_rn(dz, dz));
    es.count += 1;
  }
  if (log_row) for (int i = 0; i < 32; ++i) log_row[inst * log_stride + i] = e[i];
}

// After an MPC cycle of an estimated episode: the mode schedule the cycle used becomes the instance's own, so that the filter's contact
// flags survive the end of the call (the next call reads no context scratch of this one)
__global__ void est_schedule_kernel(int B, const hb_reference* refs, hb_estimation_state* est) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const hb_reference& f = refs[inst];
  hb_estimation_state& s = est[inst];
  const int n = f.n_events < HB_MAX_EVENTS ? f.n_events : HB_MAX_EVENTS;
  s.n_events = n;
  for (int i = 0; i < n; ++i) s.event_times[i] = f.event_times[i];
  for (int i = 0; i <= n; ++i) s.modes[i] = f.modes[i];
  s.has_plan = 1;
}

}  // namespace hb

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
// joint command law (LeggedController.cpp:186-257), one thread per instance; joints are visited in order because the limit
// protection of joint j only affects the commands of joints >= j within the same cycle. An instance with a controller setting in `cs` runs
// its gains in place of `gains`.
__global__ void joint_command_kernel(int B, hb_pd_gains gains, InstanceView<hb_controller_setting> cs, double dt, const double* x_des,
                                     const double* u_des, const double* sol, const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded,
                                     uint8_t* estop, double* command, double* out_tau) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const hb_controller_setting* rec = cs.of(inst);
  hb_pd_gains g = gains;
  if (rec) g = rec->gains;
  const double* xd = x_des + (size_t)inst * NX; const double* ud = u_des + (size_t)inst * NU;
  const double* ws = sol + (size_t)inst * NWBC; const double* r = rbd + (size_t)inst * 32;
  const bool is_loaded = loaded ? loaded[inst] != 0 : true;
  bool stop = estop ? estop[inst] != 0 : false;
  const int mode = mode_cmd[inst];
  for (int j = 0; j < NJ; ++j) {
    const double q = r[6 + j], qd = r[NQ + 6 + j];
    if (!stop && is_loaded && (q > c_model.joint_upper[j] + 0.02 || q < c_model.joint_lower[j] - 0.02)) stop = true;
    double pd, vd, kp, kd, ff;
    if (!is_loaded) {
      pd = xd[12 + j]; vd = ud[12 + j]; kp = g.kp_position; kd = (j == 4 || j == 9) ? g.kd_feet : g.kd_position; ff = 0.0;
    } else {
      const double qdd = ws[6 + j];
      pd = xd[12 + j] + 0.5 * qdd * dt * dt; vd = ud[12 + j] + qdd * dt; ff = ws[28 + j];
      const bool contact = contact_flag(mode, j / 5);
      if (j == 0 || j == 1 || j == 5 || j == 6) { kp = contact ? g.kp_small_stance : g.kp_small_swing; kd = g.kd_small; }
      else if (j == 4 || j == 9) { kp = contact ? g.kp_small_stance : g.kp_small_swing; kd = g.kd_feet; }
      else { kp = contact ? g.kp_big_stance : g.kp_big_swing; kd = g.kd_big; }
    }
    if (stop) { pd = 0.0; vd = 0.0; kp = 0.0; kd = 1.0; ff = 0.0; }
    double* c = command + ((size_t)inst * NJ + j) * 5;
    c[0] = pd; c[1] = vd; c[2] = kp; c[3] = kd; c[4] = ff;
    out_tau[(size_t)inst * NJ + j] = ff + kp * (pd - q) + kd * (vd - qd);
  }
  if (estop) estop[inst] = stop ? 1 : 0;
}

// The hybrid joint command's PD law (LeggedHWSim.cpp:181-186): one body for the actuation model and the motor bridge's motor PD, so that a
// neutral bridge reproduces the actuation model bit for bit. The roundings are written out, as the compiler contracts
// kp (pos - q) + kd (vel - qd) + ff: otherwise the contraction could differ between the call sites.
__device__ __forceinline__ double hybrid_pd(double pos, double vel, double kp, double kd, double ff, double q, double qd) {
  return __dadd_rn(__fma_rn(kp, __dsub_rn(pos, q), __dmul_rn(kd, __dsub_rn(vel, qd))), ff);
}

// Actuation model of the simulated hardware (legged_gazebo/src/LeggedHWSim.cpp:166-192): every write pushes the hybrid joint command
// (posDes, velDes, kp, kd, ff) with its time stamp on a buffer, drops the entries older than `delay` from the far end, and applies the
// OLDEST remaining one: tau = kp (posDes - q) + kd (velDes - qd) + ff with the CURRENT joint state. One thread per instance; the deque is a
// ring of HB_ACT_CAPACITY entries (a full ring drops its oldest entry first). An instance with a hardware record in `hw` runs its delay in
// place of `delay_all`. An instance with a record in `bridge` writes the oldest entry's decoded motor command to its row of mcmd (B x 50)
// instead of a torque to tau; the plant runs its PD.
__global__ void actuation_kernel(int B, double delay_all, InstanceView<hb_hardware_setting> hw, InstanceView<hb_motor_bridge> bridge, const double* time,
                                 hb_actuation_state* state, const double* command, const double* rbd, double* tau, double* mcmd) {
  const int inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= B) return;
  const hb_hardware_setting* h = hw.of(inst);
  const double delay = h ? h->actuation_delay : delay_all;
  hb_actuation_state& st = state[inst];
  const double t = time[inst];
  int cnt = st.count, head = st.head;             // head = newest entry; entries head, head+1, ... (mod capacity) are older and older
  while (cnt > 0 && st.stamp[(head + cnt - 1) % HB_ACT_CAPACITY] + delay < t) --cnt;
  if (cnt == HB_ACT_CAPACITY) --cnt;
  head = (head + HB_ACT_CAPACITY - 1) % HB_ACT_CAPACITY;
  st.stamp[head] = t;
  for (int k = 0; k < NJ * 5; ++k) st.cmd[head][k] = command[(size_t)inst * NJ * 5 + k];
  ++cnt;
  st.count = cnt; st.head = head;
  const double* c = st.cmd[(head + cnt - 1) % HB_ACT_CAPACITY];
  if (const hb_motor_bridge* mb = bridge.of(inst)) {
    for (int j = 0; j < NJ; ++j) bridge_command(*mb, j, c + 5 * j, mcmd + ((size_t)inst * NJ + j) * 5);
    return;
  }
  const double* r = rbd + (size_t)inst * 32;
  for (int j = 0; j < NJ; ++j) tau[(size_t)inst * NJ + j] = hybrid_pd(c[5 * j], c[5 * j + 1], c[5 * j + 2], c[5 * j + 3], c[5 * j + 4], r[6 + j], r[NQ + 6 + j]);
}

// One step of a batched rigid-body simulation of the robot on the ground (stands in for the Gazebo / MuJoCo plant of the reference's
// closed loop, legged_gazebo / legged_mujoco): forward dynamics M(q) qdd = S' tau + J_c' F_c - nle with compliant point contacts at the four
// contact frames (normal spring-damper, viscous tangential friction clipped to the cone), semi-implicit Euler over `substeps` substeps.
// Same rigid-body passes as the WBC assembly: lanes 0-15 unit-velocity sweeps -> J_c columns, lanes 0-15 RNEA with unit accelerations ->
// M columns, lane 16 -> nle; 16 x 16 Cholesky in shared memory. One warp per instance. wrench (B x 6, nullable): an external world force at
// the base origin and a world couple, which enter as the generalised forces Q_p = f, Q_zyx = T' tau with omega_world = T(zyx) zyx_dot
// (world_omega_from_zyx_rates, hb_rbd.cuh); null adds nothing. var: the plants of the instances that have one (varied plants,
// hunter_b200.h); the others run the nominal plant. terrain: the ground under the instances that have one (terrain, hunter_b200.h); the
// others stand on flat ground at prm.ground_height. links: the bodies of the instances that have them (link variations, hunter_b200.h),
// formed once per call into `body` (LinkBodies' table); the others read the model's.
struct SimShared {
  double q[NQ], v[NQ], J[12 * NQ], M[NQ * 17], nle[NQ], rhs[NQ], t1[NQ], t2[NQ], kdi[NQ], F[12], cpos[12], cvel[12], body[NBODY * LINK_BODY];
};

// Body b of a link variation l as LinkBodies reads it (out: 13 doubles): m' = s_m m, c' = c + shift, I' = s_I I, each one rounded operation.
// Returns whether the body equals the model's.
__device__ __forceinline__ bool link_body(const hb_link_variation& l, int b, double* out) {
  const Model& md = c_model;
  out[0] = __dmul_rn(l.mass_scale[b], md.mass[b]);
  bool same = out[0] == md.mass[b];
  for (int i = 0; i < 3; ++i) { out[1 + i] = __dadd_rn(md.com[3 * b + i], l.com_shift[b][i]); same &= out[1 + i] == md.com[3 * b + i]; }
  for (int i = 0; i < 9; ++i) { out[4 + i] = __dmul_rn(l.inertia_scale[b], md.inertia[9 * b + i]); same &= out[4 + i] == md.inertia[9 * b + i]; }
  return same;
}

// One RNEA lane of a varied robot on the body table t (LinkBodies). Not inlined, as payload_rnea: the nominal lanes keep their code. Its
// roundings can differ from the inlined nominal pass's, so a robot whose bodies all equal the model's runs the nominal pass.
__device__ __noinline__ void link_rnea(const double* q, const double* v, const double* a, bool gravity, const double* t, double* tau) {
  rnea_pass(q, v, a, gravity, tau, nullptr, LinkBodies{t});
}

// The payload of a varied plant in one RNEA lane: rnea_pass's base-body wrench for a rigid body fixed to the base with mass m, CoM c and
// inertia I (base frame), added to the base rows of tau (the joint rows get nothing from a body on the base). Not inlined: inlined after
// rnea_pass it keeps q, v, a live across that pass and sim_step_kernel spills (255 registers); called, the kernel stays without spills.
__device__ __noinline__ void payload_rnea(const double* q, const double* v, const double* a, bool gravity, double m, const double* c, const double* I,
                                             double* tau) {
  double R0[9], ax0[9], w0[3], wd0[3], pd0[3], F[3], n[3];
  rnea_base_motion(q, v, a, R0, ax0, w0, wd0, pd0);
  rigid_body_wrench(R0, w0, wd0, pd0, m, c, I, gravity, F, n);
  for (int i = 0; i < 3; ++i) {
    tau[i] += F[i];
    tau[3 + i] += ax0[3 * i] * n[0] + ax0[3 * i + 1] * n[1] + ax0[3 * i + 2] * n[2];
  }
}

// The contact force F (3) of one contact point at position p, velocity v on a slope of the terrain with height h and gradient (gx, gy)
// at p (the sloped path of terrain, hunter_b200.h): normal spring-damper along the surface normal, viscous tangential friction in the
// tangent plane clipped to mu times the normal force. Returns the normal force.
__device__ __forceinline__ double sloped_contact(const double* p, const double* v, double h, double gx, double gy, double kg, double dg, double ct,
                                                 double mu, double* F) {
  const double L = sqrt(1.0 + gx * gx + gy * gy);
  const double n[3] = {-gx / L, -gy / L, 1.0 / L};
  const double depth = (h - p[2]) / L;
  F[0] = F[1] = F[2] = 0.0;
  if (!(depth > 0.0)) return 0.0;
  const double vn = v[0] * n[0] + v[1] * n[1] + v[2] * n[2];
  double fn = kg * depth - dg * vn;
  if (fn < 0.0) fn = 0.0;
  double ft[3];
  for (int c = 0; c < 3; ++c) ft[c] = -ct * (v[c] - vn * n[c]);
  const double tl = sqrt(ft[0] * ft[0] + ft[1] * ft[1] + ft[2] * ft[2]), fmax_ = mu * fn;
  if (tl > fmax_) { const double sc = tl > 0.0 ? fmax_ / tl : 0.0; for (int c = 0; c < 3; ++c) ft[c] *= sc; }
  for (int c = 0; c < 3; ++c) F[c] = fn * n[c] + ft[c];
  return fn;
}

// The motor bridge's side of a plant step (motor bridge, hunter_b200.h): the bridged instances (rec; an empty view bridges none), their
// decoded motor commands (cmd, B x 50), their torque limits (lim_rows, B x 10, when given; otherwise the hardware record's, or lim) and
// where the mean over the substeps of the clipped torque goes (applied, B x 10, nullable).
struct MotorDrive {
  InstanceView<hb_motor_bridge> rec;
  const double* cmd;
  const double* lim_rows;
  InstanceView<hb_hardware_setting> hw;
  double lim[NJ];
  double* applied;
};

// The torque the motor of joint j of bridged instance inst applies at joint state q, qd: the hybrid PD law in the motor frame, back to the
// joint frame, clipped to the instance's limit. Not inlined, as payload_rnea, to keep sim_step_kernel without spills.
__device__ __noinline__ double bridge_motor_torque(const MotorDrive& d, const hb_motor_bridge& b, int inst, int j, double q, double qd) {
  const double* m = d.cmd + ((size_t)inst * NJ + j) * 5;
  const hb_hardware_setting* h = d.hw.of(inst);
  const double lim = d.lim_rows ? d.lim_rows[(size_t)inst * NJ + j] : h ? h->torque_limit[j] : d.lim[j], dir = (double)b.direction[j];
  const double t = dir * hybrid_pd(m[0], m[1], m[2], m[3], m[4], dir * q + b.zero[j], dir * qd);
  return t < -lim ? -lim : (t > lim ? lim : t);
}

// Friction loss of joint j of a joint model (joint models, hunter_b200.h) at velocity v: -f_j clamp(v / v_s, -1, 1)
__device__ __forceinline__ double joint_friction(const hb_joint_model& m, int j, double v) {
  const double x = v / m.friction_velocity;
  return -m.friction_loss[j] * (x < -1.0 ? -1.0 : (x > 1.0 ? 1.0 : x));
}

// The range stop of joint j of a joint model at q, v with m_jj the joint's diagonal of M + armature: 0 inside the range (and at a bound),
// min(0, -m_jj (k r + b v)) past the upper end, max(0, m_jj (k r - b v)) past the lower end; it never pulls the joint towards the stop.
__device__ __forceinline__ double joint_stop(const hb_joint_model& m, int j, double q, double v, double mjj) {
  if (q > m.upper[j]) { const double t = -mjj * (m.stop_stiffness * (q - m.upper[j]) + m.stop_damping * v); return t < 0.0 ? t : 0.0; }
  if (q < m.lower[j]) { const double t = mjj * (m.stop_stiffness * (m.lower[j] - q) - m.stop_damping * v); return t > 0.0 ? t : 0.0; }
  return 0.0;
}

// The views are __grid_constant__ (read in place, never copied): as plain by-value parameters they cost the kernel two registers.
// joints: the joint models of the instances that have one (joint models, hunter_b200.h); the others have no stops and no friction loss.
__global__ void __launch_bounds__(32) sim_step_kernel(int B, hb_sim_params prm, double* rbd_io, const double* tau, const double* wrench,
                                                      const __grid_constant__ InstanceView<hb_plant_variation> var,
                                                      const __grid_constant__ InstanceView<hb_terrain> terrain, const __grid_constant__ MotorDrive drive,
                                                      const __grid_constant__ InstanceView<hb_link_variation> links,
                                                      const __grid_constant__ InstanceView<hb_joint_model> joints, double* contact_force,
                                                      uint8_t* contact_flag) {
  __shared__ SimShared sh;
  const int inst = blockIdx.x, lane = threadIdx.x;
  const hb_plant_variation* pv = var.of(inst);      // null: the nominal plant
  const hb_terrain* ter = terrain.of(inst);         // null: flat ground at prm.ground_height
  const hb_motor_bridge* mb = drive.rec.of(inst);   // null: the joints receive tau
  const hb_link_variation* lv = links.of(inst);     // null: the model's bodies (also for a record whose bodies equal the model's)
  bool touch = false;                    // lanes 0-3: the normal force of their contact in the last substep is positive
  double applied = 0.0;                  // lanes 6-15 of a bridged instance: the sum over the substeps of the motor's clipped torque
  double* r = rbd_io + (size_t)inst * 32;
  if (lane == 0) rbd_to_qv(r, sh.q, sh.v);
  if (lv && !__any_sync(HB_FULL_MASK, lane < NBODY && !link_body(*lv, lane, &sh.body[LINK_BODY * lane]))) lv = nullptr;
  __syncwarp();
  const double h = prm.dt / (prm.substeps > 0 ? prm.substeps : 1);
  for (int sub = 0; sub < (prm.substeps > 0 ? prm.substeps : 1); ++sub) {
    if (lane < NQ) {
      double q[NQ], e[NQ];
      for (int i = 0; i < NQ; ++i) { q[i] = sh.q[i]; e[i] = (i == lane) ? 1.0 : 0.0; }
      KinOut<double> o;
      kin_pass<double>(q, e, o);
      for (int rr = 0; rr < 12; ++rr) sh.J[rr * NQ + lane] = o.cvel[rr];
      if (lane == 0) for (int rr = 0; rr < 12; ++rr) sh.cpos[rr] = o.cpos[rr];
    }
    __syncwarp();
    if (lane < 12) { double s = 0.0; for (int i = 0; i < NQ; ++i) s += sh.J[lane * NQ + i] * sh.v[i]; sh.cvel[lane] = s; }
    __syncwarp();
    if (lane < 4) {
      double gh = prm.ground_height, gx = 0.0, gy = 0.0;
      if (ter) gh = hbplan::terrain_height<false>(*ter, sh.cpos[3 * lane], sh.cpos[3 * lane + 1], &gx, &gy);
      if (gx == 0.0 && gy == 0.0) {      // flat ground, or a level patch of the terrain: the flat contact at its height
        const double depth = gh - sh.cpos[3 * lane + 2];
        double fz = 0.0, fx = 0.0, fy = 0.0;
        if (depth > 0.0) {
          double kg = prm.ground_stiffness, dg = prm.ground_damping, mu = prm.friction_mu;
          if (pv) { kg *= pv->stiffness_scale; dg *= pv->damping_scale; mu *= pv->friction_scale; }
          fz = kg * depth - dg * sh.cvel[3 * lane + 2];
          if (fz < 0.0) fz = 0.0;
          fx = -prm.tangential_damping * sh.cvel[3 * lane]; fy = -prm.tangential_damping * sh.cvel[3 * lane + 1];
          const double ft = sqrt(fx * fx + fy * fy), fmax_ = mu * fz;
          if (ft > fmax_) { const double sc = ft > 0.0 ? fmax_ / ft : 0.0; fx *= sc; fy *= sc; }
        }
        sh.F[3 * lane] = fx; sh.F[3 * lane + 1] = fy; sh.F[3 * lane + 2] = fz;
        touch = fz > 0.0;
      } else {
        double kg = prm.ground_stiffness, dg = prm.ground_damping, mu = prm.friction_mu;
        if (pv) { kg *= pv->stiffness_scale; dg *= pv->damping_scale; mu *= pv->friction_scale; }
        touch = sloped_contact(&sh.cpos[3 * lane], &sh.cvel[3 * lane], gh, gx, gy, kg, dg, prm.tangential_damping, mu, &sh.F[3 * lane]) > 0.0;
      }
    }
    if (lane < 17) {
      double q[NQ], v[NQ], a[NQ], tq[NQ];
      for (int i = 0; i < NQ; ++i) { q[i] = sh.q[i]; v[i] = lane == 16 ? sh.v[i] : 0.0; a[i] = (i == lane) ? 1.0 : 0.0; }
      if (lv) link_rnea(q, v, a, lane == 16, sh.body, tq);
      else rnea_pass(q, v, a, lane == 16, tq, nullptr);
      if (pv && (lane < 6 || lane == 16) && pv->payload_mass > 0.0)
        payload_rnea(q, v, a, lane == 16, pv->payload_mass, pv->payload_com, pv->payload_inertia, tq);
      if (lane < 16) { for (int rr = 0; rr < NQ; ++rr) sh.M[rr * 17 + lane] = tq[rr]; }
      else { for (int rr = 0; rr < NQ; ++rr) sh.nle[rr] = tq[rr]; }
    }
    __syncwarp();
    if (lane < NQ) {
      // joint side of the plant as in the reference's MuJoCo model (mujoco/model/hunter/hunter.xml:6): rotor armature on the diagonal of M,
      // viscous joint damping. A varied plant's motor strength scales the torque first, as one rounded product (never contracted into
      // the damping term), so that strength s on tau is strength 1 on s * tau. A bridged joint's motor runs its PD on this substep's state.
      double tj = 0.0;
      if (lane >= 6 && mb) {
        tj = bridge_motor_torque(drive, *mb, inst, lane - 6, sh.q[lane], sh.v[lane]);
        applied = sub ? applied + tj : tj;
      } else if (lane >= 6) {
        tj = tau[(size_t)inst * NJ + lane - 6];
      }
      if (pv && lane >= 6) tj = __dmul_rn(pv->motor_strength[lane - 6], tj);
      // a joint model's terms (joint models, hunter_b200.h), skipped where they do not act: the friction loss after the damping, the stop
      // after the armature
      const hb_joint_model* jm = lane >= 6 ? joints.of(inst) : nullptr;
      double jt = lane >= 6 ? tj - prm.joint_damping * sh.v[lane] : 0.0;
      if (jm && jm->friction_loss[lane - 6] != 0.0) jt += joint_friction(*jm, lane - 6, sh.v[lane]);
      double s = -sh.nle[lane] + jt;
      for (int rr = 0; rr < 12; ++rr) s += sh.J[rr * NQ + lane] * sh.F[rr];
      if (wrench && lane < 6) {
        const double* w = wrench + (size_t)inst * 6;
        if (lane < 3) s += w[lane];
        else {
          double sz, cz, sy, cy;
          sincos(sh.q[3], &sz, &cz); sincos(sh.q[4], &sy, &cy);
          // rows yaw, pitch, roll of T' (couple), T the map of world_omega_from_zyx_rates
          s += lane == 3 ? w[5] : (lane == 4 ? -sz * w[3] + cz * w[4] : cz * cy * w[3] + sz * cy * w[4] - sy * w[5]);
        }
      }
      if (lane >= 6) sh.M[lane * 17 + lane] += prm.joint_armature;
      if (jm && (sh.q[lane] > jm->upper[lane - 6] || sh.q[lane] < jm->lower[lane - 6]))
        s += joint_stop(*jm, lane - 6, sh.q[lane], sh.v[lane], sh.M[lane * 17 + lane]);
      sh.rhs[lane] = s;
      for (int j = lane + 1; j < NQ; ++j) { const double a = 0.5 * (sh.M[lane * 17 + j] + sh.M[j * 17 + lane]); sh.M[j * 17 + lane] = a; }   // lower triangle, symmetrised
    }
    __syncwarp();
    warp_chol_inv(sh.M, NQ, 17, sh.kdi, lane);
    warp_li_mv(sh.M, NQ, 17, sh.kdi, sh.rhs, sh.t1, lane);
    warp_lit_mv(sh.M, NQ, 17, sh.kdi, sh.t1, sh.t2, lane);      // t2 = qdd
    if (lane < NQ) { const double vn = sh.v[lane] + h * sh.t2[lane]; sh.v[lane] = vn; sh.q[lane] += h * vn; }
    __syncwarp();
  }
  if (lane == 0) qv_to_rbd(sh.q, sh.v, r);
  if (lane >= 6 && lane < NQ && mb && drive.applied) drive.applied[(size_t)inst * NJ + lane - 6] = applied / (prm.substeps > 0 ? prm.substeps : 1);
  if (lane < 12 && contact_force) contact_force[(size_t)inst * 12 + lane] = sh.F[lane];
  if (lane < 4 && contact_flag) contact_flag[(size_t)inst * 4 + lane] = touch ? 1 : 0;
}
}  // namespace
