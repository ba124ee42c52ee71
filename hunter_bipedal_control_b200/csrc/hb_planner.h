// Host-side reference preprocessing of one MPC solve (SURVEY 8a rows P1, P3, P5), mirroring the reference's own objects:
//   P1  GaitSchedule::{insertModeSequenceTemplate, tileModeSequenceTemplate}      legged_interface/src/gait/GaitSchedule.cpp:57-161
//       gait templates                                                            legged_controllers/config/hunter/gait.info (hb_planner_settings.gait)
//   P3  SwingTrajectoryPlanner::{update, calNextFootPos, genSwingTrajs}           legged_interface/src/foot_planner/SwingTrajectoryPlanner.cpp:164-358
//       CubicSpline nodes (time, position, velocity)                              legged_interface/src/foot_planner/CubicSpline.cpp:46-70
//   P5  cmdVelToTargetTrajectories / targetPoseToTargetTrajectories               legged_controllers/src/TargetTrajectoriesPublisher.cpp:41-130
// The output is the compact hb_reference consumed by hb_reference_expand_batch (device).
//   P4  calculateJointRef + InverseKinematics::computeIK                        legged_interface/src/SwitchedModelReferenceManager.cpp:251-300,
//                                                                                 src/foot_planner/InverseKinematics.cpp:20-231
//   P2  calculateVelAbs / walkGait (speed-based gait selection)                   legged_interface/src/SwitchedModelReferenceManager.cpp:185-249
//
// Everything here is fixed-capacity, allocation-free code that compiles for the host (hb_plan_references, threaded over instances)
// AND for the device (plan_references_coop_kernel, four threads per instance; row N1): the same source, so both produce the same plan.
#pragma once
#include <math.h>
#include <string.h>

#include "../../include/hunter_b200.h"
#include "../../include/hunter_model_constants.h"

#if defined(__CUDACC__)
#define HBP_HD __host__ __device__
#define HBP_HDI __host__ __device__ __forceinline__
#else
#define HBP_HD
#define HBP_HDI inline
#endif

namespace hbplan {

constexpr int MAX_PHASES = 128;     // phases of the tiled schedule kept around one solve (about 3 horizons + one gait period)

// model constants the planner needs, passed by value to the device kernel (host static arrays are not visible to device code)
struct PlanConsts {
  double joint_xyz[33], joint_axis[33], contact_offset[12], lower[10], upper[10], default_joints[10];
};
inline PlanConsts make_consts() {
  PlanConsts pc;
  for (int i = 0; i < 33; ++i) { pc.joint_xyz[i] = HB_JOINT_XYZ[i]; pc.joint_axis[i] = HB_JOINT_AXIS[i]; }
  for (int i = 0; i < 12; ++i) pc.contact_offset[i] = HB_CONTACT_OFFSET[i];
  for (int i = 0; i < 10; ++i) { pc.lower[i] = HB_JOINT_LOWER[i]; pc.upper[i] = HB_JOINT_UPPER[i]; pc.default_joints[i] = HB_DEFAULT_JOINT_STATE[i]; }
  return pc;
}

HBP_HD inline double dmin(double a, double b) { return a < b ? a : b; }
HBP_HD inline double dmax(double a, double b) { return a > b ? a : b; }

// a product rounded on its own: never contracted into an fma by the device compiler, so host and device round alike
HBP_HD inline double mul_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

// The one terrain lookup (terrain, hunter_b200.h) of the plant, the height check and the planner's height maps. RN: every product of
// the interpolation is rounded on its own (mul_rn), so that the host and the device get the same bits (the planner); without it the
// device compiler contracts them as it always has (the plant and the height check, whose instructions this form leaves unchanged).
template <bool RN> HBP_HDI double terrain_mul(double a, double b) { return RN ? mul_rn(a, b) : a * b; }

// One axis of a terrain lookup: the grid coordinate of the world coordinate x, clamped to [0, n - 1], split into the cell index
// i <= n - 2 and the fraction a of the cell. Returns whether x was clamped (off the grid, where the gradient along this axis is zero).
// A NaN coordinate clamps to 0, so no index leaves the grid.
HBP_HDI bool terrain_axis(double x, double origin, double spacing, int n, int* i, double* a) {
  double u = (x - origin) / spacing;
  bool clamped = false;
  if (!(u >= 0.0)) { u = 0.0; clamped = true; }
  else if (u > (double)(n - 1)) { u = (double)(n - 1); clamped = true; }
  int c = (int)floor(u);
  if (c > n - 2) c = n - 2;
  *i = c; *a = u - (double)c;
  return clamped;
}

// Height h of the terrain at world (x, y) and its gradient (gx, gy), bilinear on the cell, as hunter_b200.h documents it
template <bool RN> HBP_HDI double terrain_height(const hb_terrain& t, double x, double y, double* gx, double* gy) {
  int i, j;
  double a, b;
  const bool cx = terrain_axis(x, t.origin[0], t.spacing, t.nx, &i, &a), cy = terrain_axis(y, t.origin[1], t.spacing, t.ny, &j, &b);
  const double h00 = t.height[j][i], h01 = t.height[j][i + 1], h10 = t.height[j + 1][i], h11 = t.height[j + 1][i + 1];
  const double h0 = h00 + terrain_mul<RN>(a, h01 - h00), h1 = h10 + terrain_mul<RN>(a, h11 - h10);
  const double d0 = h01 - h00, d1 = h11 - h10;
  *gx = cx ? 0.0 : (d0 + terrain_mul<RN>(b, d1 - d0)) / t.spacing;
  *gy = cy ? 0.0 : (h1 - h0) / t.spacing;
  return h0 + terrain_mul<RN>(b, h1 - h0);
}

// h(x, y) of a planner height map (height maps, hunter_b200.h): the terrain lookup with its products rounded on their own
HBP_HD inline double map_height(const hb_terrain* m, double x, double y) {
  double gx, gy;
  return terrain_height<true>(*m, x, y, &gx, &gy);
}

// The surface frame of ground with gradient (gx, gy): f = (n, t1, t2) with n = (-gx, -gy, 1) / L, L = sqrt(1 + gx^2 + gy^2),
// t1 = (1, 0, gx) / sqrt(1 + gx^2) and t2 = n x t1, each product rounded on its own (mul_rn) as the map lookup's, so that host and device
// frames have the same bits. Returns whether the ground is sloped; a zero gradient is flat ground, and f is then left as it is.
HBP_HD inline bool surface_frame(double gx, double gy, double* f) {
  if (gx == 0.0 && gy == 0.0) return false;
  const double L = sqrt(1.0 + mul_rn(gx, gx) + mul_rn(gy, gy)), Lt = sqrt(1.0 + mul_rn(gx, gx));
  const double n0 = -gx / L, n1 = -gy / L, n2 = 1.0 / L, t0 = 1.0 / Lt, t2 = gx / Lt;
  f[0] = n0; f[1] = n1; f[2] = n2;
  f[3] = t0; f[4] = 0.0; f[5] = t2;
  f[6] = mul_rn(n1, t2) - mul_rn(n2, 0.0);
  f[7] = mul_rn(n2, t0) - mul_rn(n0, t2);
  f[8] = mul_rn(n0, 0.0) - mul_rn(n1, t0);
  return true;
}

// The surface frame of map m at world (x, y) (surface_frame of the lookup's gradient): the friction cones of the WBC maps and the MPC
// cone maps (hunter_b200.h) are about it. Returns whether the ground is sloped there; f is written only then.
HBP_HD inline bool map_frame(const hb_terrain& m, double x, double y, double* f) {
  double gx, gy;
  terrain_height<true>(m, x, y, &gx, &gy);
  return surface_frame(gx, gy, f);
}

struct Vec3 { double x, y, z; };
HBP_HD inline Vec3 operator+(Vec3 a, Vec3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
HBP_HD inline Vec3 operator-(Vec3 a, Vec3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
HBP_HD inline Vec3 operator*(double s, Vec3 a) { return {s * a.x, s * a.y, s * a.z}; }
HBP_HD inline Vec3 cross(Vec3 a, Vec3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

// getRotationMatrixFromZyxEulerAngles applied to a vector
HBP_HD inline Vec3 rot_zyx(const double* e, Vec3 v) {
  const double cz = cos(e[0]), sz = sin(e[0]), cy = cos(e[1]), sy = sin(e[1]), cx = cos(e[2]), sx = sin(e[2]);
  const double R[9] = {cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx, sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx, -sy, cy * sx, cy * cx};
  return {R[0] * v.x + R[1] * v.y + R[2] * v.z, R[3] * v.x + R[4] * v.y + R[5] * v.z, R[6] * v.x + R[7] * v.y + R[8] * v.z};
}

// MotionPhaseDefinition.h:55-87
HBP_HD inline bool contact_flag(int mode, int c) { return (c & 1) ? (mode == 1 || mode == 3) : (mode == 2 || mode == 3); }

struct ModeSchedule { int n_events; double events[MAX_PHASES]; int modes[MAX_PHASES + 1]; };   // n_events + 1 modes

// The compiled-in template of gait 0..3 (legged_controllers/config/hunter/gait.info, ModeSequenceTemplate): hb_default_planner_settings.
// The entries beyond n_phase are left as they are.
HBP_HD inline void gait_template(int gait, hb_gait_template& g) {
  int32_t* modes = g.modes; double* times = g.switching_times;
  switch (gait) {
    case 1: modes[0] = 2; modes[1] = 1; times[0] = 0.0; times[1] = 0.3; times[2] = 0.6; g.n_phase = 2; break;                 // trot
    case 2: modes[0] = 2; modes[1] = 3; modes[2] = 1; modes[3] = 3;
            times[0] = 0.0; times[1] = 0.25; times[2] = 0.3; times[3] = 0.55; times[4] = 0.6; g.n_phase = 4; break;           // standing_trot
    case 3: modes[0] = 2; modes[1] = 0; modes[2] = 1; modes[3] = 0;
            times[0] = 0.0; times[1] = 0.15; times[2] = 0.2; times[3] = 0.35; times[4] = 0.4; g.n_phase = 4; break;           // flying_trot
    default: modes[0] = 3; times[0] = 0.0; times[1] = 0.5; g.n_phase = 1; break;                                                // stance
  }
}

// What one instance's plan reads of its hb_planner_settings: the template of its gait and swing_trajectory_config (168 B, staged per
// instance in shared memory by the device planner).
struct PlanSettings {
  hb_gait_template tmpl;
  double swing_height, swing_time_scale, next_stance_z, feet_bias_x1, feet_bias_x2, feet_bias_y, feet_bias_z;
};

// The settings of an instance planning gait `gait` (0..3): from its record s, or with s null the compiled-in values (task.info's
// swing_trajectory_config, next_position_z at the loader's default), which hb_default_planner_settings records give as well.
HBP_HD inline void plan_settings(const hb_planner_settings* s, int gait, PlanSettings& ps) {
  if (s) {
    ps.tmpl = s->gait[gait];
    ps.swing_height = s->swing_height; ps.swing_time_scale = s->swing_time_scale; ps.next_stance_z = s->next_stance_z;
    ps.feet_bias_x1 = s->feet_bias_x1; ps.feet_bias_x2 = s->feet_bias_x2; ps.feet_bias_y = s->feet_bias_y; ps.feet_bias_z = s->feet_bias_z;
    return;
  }
  gait_template(gait, ps.tmpl);
  ps.swing_height = HB_SWING_HEIGHT; ps.swing_time_scale = HB_SWING_TIME_SCALE; ps.next_stance_z = HB_NEXT_POSITION_Z;
  ps.feet_bias_x1 = HB_FEET_BIAS_X1; ps.feet_bias_x2 = HB_FEET_BIAS_X2; ps.feet_bias_y = HB_FEET_BIAS_Y; ps.feet_bias_z = HB_FEET_BIAS_Z;
}

// hb_default_planner_settings: every gait's compiled-in template (unused entries zero) and the compiled-in swing settings
inline void default_settings(hb_planner_settings& s) {
  memset(&s, 0, sizeof(s));
  for (int g = 0; g < 4; ++g) gait_template(g, s.gait[g]);
  PlanSettings ps;
  plan_settings(nullptr, 0, ps);
  s.swing_height = ps.swing_height; s.swing_time_scale = ps.swing_time_scale; s.next_stance_z = ps.next_stance_z;
  s.feet_bias_x1 = ps.feet_bias_x1; s.feet_bias_x2 = ps.feet_bias_x2; s.feet_bias_y = ps.feet_bias_y; s.feet_bias_z = ps.feet_bias_z;
}

// A schedule that is STANCE (two phases split at `prev_event`, like the reference's initialModeSchedule {STANCE, STANCE},
// reference.info:21-32) until `start`, then the template tiled up to `final_time` and closed by a STANCE phase:
// GaitSchedule.cpp:57-93 (insert; the last mode before insertion is STANCE, so no extra transition phase) and :123-161 (tile).
// Like GaitSchedule::getModeSchedule (:95-121), which drops the phases older than its lower bound, whole template periods that end
// before `t_keep` are skipped; the schedule inside [t_keep, final_time] is unchanged. Returns false when MAX_PHASES is exceeded.
HBP_HD inline bool tile_gait(const hb_gait_template& g, double prev_event, double start, double t_keep, double final_time, ModeSchedule& ms) {
  const int32_t* tm = g.modes; const double* tt = g.switching_times;
  const int np = g.n_phase;
  const double period = tt[np];
  if (start < t_keep) start += floor((t_keep - start) / period) * period;
  int ne = 0;
  ms.modes[0] = 3; ms.events[ne++] = prev_event;
  ms.modes[1] = 3; ms.events[ne++] = start;
  while (ms.events[ne - 1] < final_time) {
    if (ne + np + 1 > MAX_PHASES) return false;
    for (int i = 0; i < np; ++i) {
      ms.modes[ne] = tm[i];
      ms.events[ne] = ms.events[ne - 1] + (tt[i + 1] - tt[i]);
      ++ne;
    }
  }
  ms.modes[ne] = 3;
  ms.n_events = ne;
  return true;
}

// ModeSchedule::modeAtTime: lower_bound on the event times (an event time itself belongs to the earlier mode)
HBP_HD inline int mode_at(int n_events, const double* events, const int* modes, double t) {
  int idx = 0;
  while (idx < n_events && events[idx] < t) ++idx;
  return modes[idx];
}
HBP_HD inline int mode_at(const ModeSchedule& ms, double t) {
  return mode_at(ms.n_events, ms.events, ms.modes, t);
}

struct Target { int n; double t[HB_MAX_TARGETS]; double x[HB_MAX_TARGETS][22]; };

// cmdVelToTargetTrajectories (TargetTrajectoriesPublisher.cpp:102-130) with targetPoseToTargetTrajectories (:41-62), written into the
// sample count n, times tm and states x of a target: the planner's Target, or a caller's hb_target (the teleop capture writes global
// memory, not a stack copy). With a height map (nullable) both samples' body heights are taken above the map (height maps, hunter_b200.h).
HBP_HD inline void cmd_vel_target(const PlanConsts& pc, const double* cmd /*vx,vy,vz,wz*/, double time, const double* state, double time_to_target,
                                  int& n, double* tm, double (*x)[22], const hb_terrain* map) {
  const double* pose = state + 6;
  Vec3 v = rot_zyx(pose + 3, {cmd[0], cmd[1], cmd[2]});
  if (fabs(v.x) < 0.06) v.x = 0.0;
  else if (fabs(v.y) < 0.06) v.y = 0.0;
  double target[6] = {pose[0] + v.x * time_to_target, pose[1] + v.y * time_to_target, HB_COM_HEIGHT, pose[3] + cmd[3] * time_to_target, 0.0, 0.0};
  double cur[6] = {pose[0], pose[1], pose[2], pose[3], 0.0, 0.0};
  double com = HB_COM_HEIGHT;
  if (map) { com = HB_COM_HEIGHT + map_height(map, pose[0], pose[1]); target[2] = HB_COM_HEIGHT + map_height(map, target[0], target[1]); }
  double dz = com - pose[2];
  dz = dz > 0 ? dmin(dz, 0.04) : dmax(dz, -0.04);      // changeLimit_[2] (TargetTrajectoriesPublisher.h:97)
  cur[2] = pose[2] + dz;
  n = 2;
  tm[0] = time; tm[1] = time + time_to_target;
  for (int k = 0; k < 2; ++k) {
    for (int i = 0; i < 22; ++i) x[k][i] = 0.0;
    for (int i = 0; i < 6; ++i) x[k][6 + i] = (k == 0) ? cur[i] : target[i];
    for (int j = 0; j < 10; ++j) x[k][12 + j] = pc.default_joints[j];
    x[k][0] = v.x; x[k][1] = v.y; x[k][2] = v.z;    // stateTrajectory[.].head(3) = cmdVelRot (:127-128)
  }
}
HBP_HD inline Target cmd_vel_to_target(const PlanConsts& pc, const double* cmd, double time, const double* state, double time_to_target,
                                        const hb_terrain* map = nullptr) {
  Target tg;
  cmd_vel_target(pc, cmd, time, state, time_to_target, tg.n, tg.t, tg.x, map);
  return tg;
}
HBP_HD inline void cmd_vel_to_target(const PlanConsts& pc, const double* cmd, double time, const double* state, double time_to_target, hb_target& tg,
                                     const hb_terrain* map = nullptr) {
  cmd_vel_target(pc, cmd, time, state, time_to_target, tg.n, tg.time, tg.state, map);
}

// goalToTargetTrajectories with estimateTimeToTarget (TargetTrajectoriesPublisher.cpp:29-38, :83-100) and targetPoseToTargetTrajectories
// (:41-62), written into a caller's hb_target (the device capture writes global memory, not a stack copy). The yaw difference is not
// wrapped, as in the reference. A zero reaching time would give two samples at one time: the single target sample is kept instead.
// With a height map (nullable) the body height is taken above the map, and the goal sample's differs by the map's rise to the goal.
HBP_HD inline void goal_to_target(const PlanConsts& pc, double time, const double* state, const double* goal /*x, y, yaw*/, hb_target& tg,
                                  const hb_terrain* map = nullptr) {
  const double* pose = state + 6;
  const double h = map ? map_height(map, pose[0], pose[1]) : 0.0;
  double dz = (map ? HB_COM_HEIGHT + h : HB_COM_HEIGHT) - pose[2];
  dz = dz > 0 ? dmin(dz, 0.04) : dmax(dz, -0.04);      // changeLimit_[2] (TargetTrajectoriesPublisher.h:97)
  const double z = pose[2] + dz;
  const double zg = map ? z + (map_height(map, goal[0], goal[1]) - h) : z;
  const double dx = goal[0] - pose[0], dy = goal[1] - pose[1];
  const double reach = dmax(fabs(goal[2] - pose[3]) / HB_TARGET_ROTATION_VELOCITY, sqrt(mul_rn(dx, dx) + mul_rn(dy, dy)) / HB_TARGET_DISPLACEMENT_VELOCITY);
  const double cur[6] = {pose[0], pose[1], z, pose[3], 0.0, 0.0}, target[6] = {goal[0], goal[1], zg, goal[2], 0.0, 0.0};
  tg.n = reach > 0.0 ? 2 : 1;
  tg.time[0] = time; tg.time[1] = time + reach;
  for (int k = 0; k < tg.n; ++k) {
    const double* p = (tg.n == 1 || k == 1) ? target : cur;
    for (int i = 0; i < 6; ++i) { tg.state[k][i] = 0.0; tg.state[k][6 + i] = p[i]; }
    for (int j = 0; j < 10; ++j) tg.state[k][12 + j] = pc.default_joints[j];
  }
}

// the planner's copy of a caller's target (its n samples; n clamped to the capacity, so that a malformed record cannot index out of bounds)
HBP_HD inline void target_from(const hb_target& src, Target& tg) {
  tg.n = src.n < 1 ? 1 : (src.n > HB_MAX_TARGETS ? HB_MAX_TARGETS : src.n);
  for (int k = 0; k < tg.n; ++k) {
    tg.t[k] = src.time[k];
    for (int i = 0; i < 22; ++i) tg.x[k][i] = src.state[k][i];
  }
}

// TargetTrajectories::getDesiredState: piecewise-linear, clamped at both ends
HBP_HD inline void target_state(const Target& tg, double t, double* x) {
  if (tg.n <= 1 || t <= tg.t[0]) { memcpy(x, tg.x[0], sizeof(double) * 22); return; }
  if (t >= tg.t[tg.n - 1]) { memcpy(x, tg.x[tg.n - 1], sizeof(double) * 22); return; }
  int s = 0;
  while (s + 2 < tg.n && tg.t[s + 1] <= t) ++s;
  const double a = (t - tg.t[s]) / (tg.t[s + 1] - tg.t[s]);
  for (int i = 0; i < 22; ++i) x[i] = (1.0 - a) * tg.x[s][i] + a * tg.x[s + 1][i];
}

struct Node { double t, p, v; };
struct Seg { double t0, t1, p0, v0, p1, v1; };

// The planned segments go straight into the output hb_reference, restricted to the window [t_lo, t_hi] the solver can see.
struct SwingOut { hb_reference* ref; double t_lo, t_hi; bool overflow; };
HBP_HD inline void emit(SwingOut& so, int c, int a, const Seg& g) {
  if (g.t1 <= so.t_lo || g.t0 >= so.t_hi) return;
  int& n = so.ref->n_segments[c][a];
  if (n >= HB_MAX_SEGMENTS) { so.overflow = true; return; }
  double* d = so.ref->segments[c][a][n++];
  d[0] = g.t0; d[1] = g.t1; d[2] = g.p0; d[3] = g.v0; d[4] = g.p1; d[5] = g.v1;
}

// SwingTrajectoryPlanner::findIndex (SwingTrajectoryPlanner.cpp:394-419)
HBP_HD inline void find_index(int index, const bool* stock, int n, int& start_idx, int& final_idx) {
  start_idx = 0;
  for (int ip = index - 1; ip >= 0; --ip) if (stock[ip] != stock[index]) { start_idx = ip; break; }
  final_idx = n - 2;
  for (int ip = index + 1; ip < n; ++ip) if (stock[ip] != stock[index]) { final_idx = ip - 1; break; }
}

// SwingTrajectoryPlanner::threadSaftyGetStartStopTime (:510-532) on a stored schedule (n_events, events, modes): for each contact c the start
// and stop [s[c], e[c]] of the run of equal contact flags around t, as update (:164-260) stores them per phase: events[find_index(p)]. The
// phase is lookup::findIndexInTimeArray's (mode_at's: an event time belongs to the earlier phase), clamped to n_events - 1. Without a plan,
// or with a schedule of one phase (where the reference indexes events[-1]), both are t. n_events is clamped to HB_MAX_EVENTS.
HBP_HD inline void contact_phase_times(int has_plan, int n_events, const double* events, const int* modes, double t, double* s, double* e) {
  const int n = n_events < HB_MAX_EVENTS ? n_events : HB_MAX_EVENTS;
  if (!has_plan || n < 1) {
    for (int c = 0; c < 4; ++c) s[c] = e[c] = t;
    return;
  }
  int idx = 0;
  while (idx < n && events[idx] < t) ++idx;
  if (idx > n - 1) idx = n - 1;
  for (int c = 0; c < 4; ++c) {
    bool stock[HB_MAX_EVENTS + 1];
    for (int p = 0; p <= n; ++p) stock[p] = contact_flag(modes[p], c);
    int si, fi;
    find_index(idx, stock, n + 1, si, fi);
    s[c] = events[si]; e[c] = events[fi];
  }
}

// StateEstimateBase::estContactState (StateEstimateBase.cpp:208-226) with the record r: flags (in: the schedule's, out: the detected ones)
// at time t, phase times s, e (contact_phase_times) and the observer's output force (16, hb_contact_force_estimate_batch's layout), whose
// F_z of leg c % 2 decides a swing foot late in its phase and a stance foot early in its phase. The comparisons are strict.
HBP_HD inline void contact_state(const hb_contact_detection& r, double t, const double* s, const double* e, const double* force, uint8_t* flags) {
  for (int c = 0; c < 4; ++c) {
    const bool cmd = flags[c] != 0;
    const double P = e[c] - s[c], fz = force[6 * (c % 2) + 2];
    if (!cmd && t - s[c] > r.swing_fraction * P) flags[c] = fz > r.threshold ? 1 : 0;
    if (cmd && t - s[c] < r.stance_fraction * P) flags[c] = fz > r.threshold ? 1 : 0;
  }
}

// SwingTrajectoryPlanner::calNextFootPos (:289-312). body_vel_cmd = [vx, vy, vz, wz, 0, 0] as set from /cmd_vel_filtered
// (SwitchedModelReferenceManager.cpp:91-101): its tail(3) = (wz, 0, 0) is used as the commanded angular velocity, as the reference does.
// With a height map (nullable) the centrifugal term reads the body height above the map, and the foothold stands on the map.
HBP_HD inline Vec3 next_foot_pos(const PlanSettings& s, int foot, double current_time, double stop_time, double next_middle_time, const double* next_middle_body_pos,
                          const double* current_body_pos, Vec3 current_body_vel, const double* body_vel_cmd, const hb_terrain* map) {
  // feet_bias_ (SwingTrajectoryPlanner.cpp:76-79): toes x1, heels x2, +y on the left
  const Vec3 bias{foot < 2 ? s.feet_bias_x1 : s.feet_bias_x2, (foot & 1) ? -s.feet_bias_y : s.feet_bias_y, s.feet_bias_z};
  const Vec3 roted_bias = rot_zyx(next_middle_body_pos + 3, bias);
  const Vec3 vel_cmd_linear = rot_zyx(current_body_pos + 3, {body_vel_cmd[0], body_vel_cmd[1], body_vel_cmd[2]});
  const Vec3 vel_cmd_angular = rot_zyx(current_body_pos + 3, {body_vel_cmd[3], body_vel_cmd[4], body_vel_cmd[5]});
  Vec3 vel_linear = current_body_vel; vel_linear.z = 0.0;
  const double k = 0.03;
  const Vec3 p_shoulder = (stop_time - current_time) * (0.5 * vel_linear + 0.5 * vel_cmd_linear) + roted_bias;
  const Vec3 p_symmetry = (next_middle_time - stop_time) * vel_linear + k * (vel_linear - vel_cmd_linear);
  const double body_z = map ? current_body_pos[2] - map_height(map, current_body_pos[0], current_body_pos[1]) : current_body_pos[2];
  const Vec3 p_centrifugal = (0.5 * sqrt(body_z / 9.81)) * cross(vel_linear, vel_cmd_angular);
  Vec3 r = Vec3{current_body_pos[0], current_body_pos[1], current_body_pos[2]} + p_shoulder + p_symmetry + p_centrifugal;
  r.z = map ? s.next_stance_z + map_height(map, r.x, r.y) : s.next_stance_z;
  return r;
}

// SwingTrajectoryPlanner::genSwingTrajs (:314-358): x/y three-node, z four-node Hermite splines with the reference's shape constants.
// The z shape is that of ground at z = 0 (its node heights are fractions of the absolute apex). With a height map (nullable) it is built
// on ends lowered by h_lo = min(a.z, b.z) - next_stance_z, the lower end's ground, and h_lo is added back to the node positions.
HBP_HD inline void gen_swing(const PlanSettings& s, SwingOut& sp, int foot, double t0, double t1, Vec3 a, Vec3 b, const hb_terrain* map) {
  const double xy_a1 = 0.417, xy_l1 = 0.650, xy_k1 = 1.770;
  const double pa[3] = {a.x, a.y, a.z}, pb[3] = {b.x, b.y, b.z};
  for (int ax = 0; ax < 2; ++ax) {
    const Node n0{t0, pa[ax], 0.0}, n1{(1 - xy_a1) * t0 + xy_a1 * t1, (1 - xy_l1) * pa[ax] + xy_l1 * pb[ax], xy_k1 * (pb[ax] - pa[ax]) / (t1 - t0)}, n2{t1, pb[ax], 0.0};
    emit(sp, foot, ax, Seg{n0.t, n1.t, n0.p, n0.v, n1.p, n1.v});
    emit(sp, foot, ax, Seg{n1.t, n2.t, n1.p, n1.v, n2.p, n2.v});
  }
  double h_lo = 0.0;
  if (map) { h_lo = dmin(a.z, b.z) - s.next_stance_z; a.z = a.z - h_lo; b.z = b.z - h_lo; }
  const double scaling = dmin(1.0, (t1 - t0) / s.swing_time_scale);
  const double max_z = dmax(a.z, b.z) + scaling * s.swing_height;
  const double z_a1 = 0.251, z_l1 = 0.749, z_k1 = 1.338, z_a2 = 0.630, z_l2 = 0.570, z_k2 = 1.633, z_k3 = 0.0;
  Node n0{t0, a.z, 0.0};
  Node n1{(1 - z_a1) * t0 + z_a1 * t1, z_l1 * max_z, z_k1 * (z_l1 * (max_z - a.z)) / (z_a1 * (t1 - t0))};
  Node n2{(1 - z_a2) * t0 + z_a2 * t1, z_l2 * max_z + (1 - z_l2) * b.z, z_k2 * z_l2 * (b.z - max_z) / ((1 - z_a2) * (t1 - t0))};
  Node n3{t1, b.z, z_k3 * z_l2 * (b.z - max_z) / ((1 - z_a2) * (t1 - t0))};
  if (map) { n0.p = n0.p + h_lo; n1.p = n1.p + h_lo; n2.p = n2.p + h_lo; n3.p = n3.p + h_lo; }
  emit(sp, foot, 2, Seg{n0.t, n1.t, n0.p, n0.v, n1.p, n1.v});
  emit(sp, foot, 2, Seg{n1.t, n2.t, n1.p, n1.v, n2.p, n2.v});
  emit(sp, foot, 2, Seg{n2.t, n3.t, n2.p, n2.v, n3.p, n3.v});
}

// SwingTrajectoryPlanner::update (:164-286). latest_stance (4x3) is the planner's state (in/out).
// Returns false where the reference would throw (swing phase without a defined take-off / touch-down, :421-458).
// The feet are independent of each other: [j_begin, j_end) selects the ones this call plans (the host planner passes 0..4, the
// cooperative device kernel one foot per thread). With a height map (nullable) every lift-off point stands on the map: its z is
// next_stance_z + h at its (x, y).
HBP_HD inline bool plan_swing(const PlanSettings& s, const ModeSchedule& ms, const Target& tg, double init_time, const double* current_feet /*12*/, const double* body_vel_cmd /*6*/,
                              double* latest_stance /*12*/, SwingOut& sp, const hb_terrain* map, int j_begin = 0, int j_end = 4) {
  const int np = ms.n_events + 1;
  const int mode_now = mode_at(ms, init_time + 0.001);
  for (int i = j_begin; i < j_end; ++i) {
    if (contact_flag(mode_now, i)) for (int a = 0; a < 3; ++a) latest_stance[3 * i + a] = current_feet[3 * i + a];
    latest_stance[3 * i + 2] = map ? s.next_stance_z + map_height(map, latest_stance[3 * i], latest_stance[3 * i + 1]) : s.next_stance_z;
  }
  for (int j = j_begin; j < j_end; ++j) {
    bool stock[MAX_PHASES + 1];
    for (int p = 0; p < np; ++p) stock[p] = contact_flag(ms.modes[p], j);
    Vec3 last{latest_stance[3 * j], latest_stance[3 * j + 1], latest_stance[3 * j + 2]}, next = last;
    int last_final_idx = 0;
    for (int p = 0; p < np; ++p) {
      int si, fi;
      find_index(p, stock, np, si, fi);
      if (!stock[p]) {
        if (si < 0 || fi >= np - 1) return false;      // checkThatIndicesAreValid
        const double t_start = ms.events[si], t_final = ms.events[fi];
        if (init_time < t_final && fi > last_final_idx) {
          last = next;
          double next_middle_time;
          if (fi < np - 1) {
            int si2, fi2;
            find_index(fi + 1, stock, np, si2, fi2);
            next_middle_time = 0.5 * (t_final + ms.events[fi2]);
          } else next_middle_time = t_final;
          double xm[22], xc[22];
          target_state(tg, next_middle_time, xm);
          target_state(tg, init_time, xc);
          const Vec3 body_vel{tg.x[0][0], tg.x[0][1], tg.x[0][2]};
          next = next_foot_pos(s, j, init_time, t_final, next_middle_time, xm + 6, xc + 6, body_vel, body_vel_cmd, map);
          last_final_idx = fi;
        }
        // every phase of a swing interval pushes the same spline set (one MultiCubicSpline per phase index in the reference);
        // only emit it once per swing interval
        if (p == 0 || stock[p - 1]) gen_swing(s, sp, j, t_start, t_final, last, next, map);
      } else {
        if (p == 0 || !stock[p - 1]) {
          const double t_start = ms.events[si], t_final = (fi >= 0 && fi < ms.n_events) ? ms.events[fi] : ms.events[ms.n_events - 1];
          const double pn[3] = {next.x, next.y, next.z};
          for (int a = 0; a < 3; ++a) emit(sp, j, a, Seg{t_start, t_final, pn[a], 0.0, pn[a], 0.0});
        }
      }
    }
  }
  return true;
}

// ------------------------------------------------------------------------------------------------------------------------------
// P4: joint references by inverse kinematics (SwitchedModelReferenceManager::calculateJointRef, SwitchedModelReferenceManager.cpp:251-300;
// InverseKinematics::{computeIK, computeTranslationIK, computeRotationIK}, foot_planner/InverseKinematics.cpp:20-231).
// The Eigen solvers the reference calls are restated by what they compute:
//   ColPivHouseholderQR(threshold 0.01)::solve  -> pivot on the largest residual column norm, rank = #pivots > 0.01 * first pivot,
//                                                  least squares on the pivot columns, zeros elsewhere (basic solution);
//   FullPivLU::kernel                           -> e_j - sum_P (J_P^-1 J_j)_p e_p for every non-pivot column j, pivot columns P chosen by
//                                                  complete pivoting.

struct LegKin { double toe[3]; double R[9]; double Jl[15]; double Ja[15]; };   // Jl, Ja: 3x5 row-major, world axes

HBP_HD inline void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
HBP_HD inline void rot_zyx_mat(const double* e, double* R) {
  const double cz = cos(e[0]), sz = sin(e[0]), cy = cos(e[1]), sy = sin(e[1]), cx = cos(e[2]), sx = sin(e[2]);
  const double M[9] = {cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx, sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx, -sy, cy * sx, cy * cx};
  memcpy(R, M, sizeof(M));
}
HBP_HD inline void axis_angle(const double* a, double q, double* R) {   // Rodrigues, unit axis
  const double c = cos(q), s = sin(q), v = 1.0 - c;
  const double M[9] = {c + a[0] * a[0] * v, a[0] * a[1] * v - a[2] * s, a[0] * a[2] * v + a[1] * s,
                       a[1] * a[0] * v + a[2] * s, c + a[1] * a[1] * v, a[1] * a[2] * v - a[0] * s,
                       a[2] * a[0] * v - a[1] * s, a[2] * a[1] * v + a[0] * s, c + a[2] * a[2] * v};
  memcpy(R, M, sizeof(M));
}

// forward kinematics and frame Jacobian of the toe contact frame of leg (0 left, 1 right): pose = [p(3), zyx(3)], qj = 5 leg joints
HBP_HD inline void leg_kin(const PlanConsts& pc, int leg, const double* pose, const double* qj, LegKin& k) {
  double R[9], o[3] = {pose[0], pose[1], pose[2]}, orig[5][3], ax[5][3];
  rot_zyx_mat(pose + 3, R);
  for (int i = 0; i < 5; ++i) {
    const int b = 1 + 5 * leg + i;
    const double* xyz = pc.joint_xyz + 3 * b; const double* a = pc.joint_axis + 3 * b;
    for (int r = 0; r < 3; ++r) o[r] += R[3 * r] * xyz[0] + R[3 * r + 1] * xyz[1] + R[3 * r + 2] * xyz[2];
    for (int r = 0; r < 3; ++r) { orig[i][r] = o[r]; ax[i][r] = R[3 * r] * a[0] + R[3 * r + 1] * a[1] + R[3 * r + 2] * a[2]; }
    double Rj[9], Rn[9];
    axis_angle(a, qj[i], Rj);
    mat3_mul(R, Rj, Rn);
    memcpy(R, Rn, sizeof(Rn));
  }
  const double* off = pc.contact_offset + 3 * leg;      // contacts 0 / 1 = left / right toe
  for (int r = 0; r < 3; ++r) k.toe[r] = o[r] + R[3 * r] * off[0] + R[3 * r + 1] * off[1] + R[3 * r + 2] * off[2];
  memcpy(k.R, R, sizeof(R));
  for (int i = 0; i < 5; ++i) {
    const double d[3] = {k.toe[0] - orig[i][0], k.toe[1] - orig[i][1], k.toe[2] - orig[i][2]};
    k.Jl[i] = ax[i][1] * d[2] - ax[i][2] * d[1];
    k.Jl[5 + i] = ax[i][2] * d[0] - ax[i][0] * d[2];
    k.Jl[10 + i] = ax[i][0] * d[1] - ax[i][1] * d[0];
    for (int r = 0; r < 3; ++r) k.Ja[5 * r + i] = ax[i][r];
  }
}

// x = ColPivHouseholderQR(A (m x n, row-major, m <= 3, n <= 5), threshold).solve(b)
HBP_HD inline void qrcp_solve(const double* A, int m, int n, const double* b, double threshold, double* x) {
  double Q[3][3];            // orthonormal directions of the chosen columns
  double coef[3];            // b components along them
  int piv[3]; double R[3][3] = {{0}};
  bool used[5] = {false, false, false, false, false};
  double first = 0.0; int rank = 0;
  const int kmax = m < n ? m : n;
  for (int k = 0; k < kmax; ++k) {
    int best = -1; double bn = -1.0; double bres[3] = {0, 0, 0};
    for (int j = 0; j < n; ++j) {
      if (used[j]) continue;
      double r[3] = {0, 0, 0};
      for (int i = 0; i < m; ++i) r[i] = A[i * n + j];
      for (int t = 0; t < k; ++t) { double d = 0; for (int i = 0; i < m; ++i) d += Q[t][i] * r[i]; for (int i = 0; i < m; ++i) r[i] -= d * Q[t][i]; }
      double nn = 0; for (int i = 0; i < m; ++i) nn += r[i] * r[i];
      if (nn > bn) { bn = nn; best = j; for (int i = 0; i < m; ++i) bres[i] = r[i]; }
    }
    const double pv = sqrt(bn > 0 ? bn : 0.0);
    if (k == 0) first = pv;
    if (!(pv > threshold * first) || pv == 0.0) break;
    used[best] = true; piv[k] = best;
    for (int i = 0; i < m; ++i) Q[k][i] = bres[i] / pv;
    for (int t = 0; t <= k; ++t) { double d = 0; for (int i = 0; i < m; ++i) d += Q[t][i] * A[i * n + best]; R[t][k] = d; }
    double d = 0; for (int i = 0; i < m; ++i) d += Q[k][i] * b[i];
    coef[k] = d;
    rank = k + 1;
  }
  for (int j = 0; j < n; ++j) x[j] = 0.0;
  for (int k = rank - 1; k >= 0; --k) {          // back substitution R y = Q^T b on the pivot columns
    double v = coef[k];
    for (int t = k + 1; t < rank; ++t) v -= R[k][t] * x[piv[t]];
    x[piv[k]] = v / R[k][k];
  }
}

// FullPivLU(J (3x5)).kernel(): returns the kernel dimension (5 - rank), N is 5 x dim row-major (ld 3)
HBP_HD inline int fullpiv_kernel(const double* J, double* N) {
  double M[3][5]; int colp[5] = {0, 1, 2, 3, 4};
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 5; ++j) M[i][j] = J[5 * i + j];
  int rank = 0; double maxpiv = 0.0;
  for (int k = 0; k < 3; ++k) {
    int bi = k, bj = k; double bv = -1.0;
    for (int i = k; i < 3; ++i) for (int j = k; j < 5; ++j) if (fabs(M[i][j]) > bv) { bv = fabs(M[i][j]); bi = i; bj = j; }
    if (bv <= 0.0) break;
    if (k == 0) maxpiv = bv;
    for (int j = 0; j < 5; ++j) { const double t = M[k][j]; M[k][j] = M[bi][j]; M[bi][j] = t; }
    for (int i = 0; i < 3; ++i) { const double t = M[i][k]; M[i][k] = M[i][bj]; M[i][bj] = t; }
    { const int t = colp[k]; colp[k] = colp[bj]; colp[bj] = t; }
    // Eigen's default rank threshold: |pivot| > eps * diagonal size * max pivot
    if (bv > 2.220446049250313e-16 * 3.0 * maxpiv) rank = k + 1; else break;
    for (int i = k + 1; i < 3; ++i) { const double f = M[i][k] / M[k][k]; for (int j = k; j < 5; ++j) M[i][j] -= f * M[k][j]; }
  }
  const int dim = 5 - rank;
  for (int i = 0; i < 15; ++i) N[i] = 0.0;
  for (int c = 0; c < dim; ++c) {
    // solve U11 y = -U12[:, c] (upper triangular, rank x rank)
    double y[3] = {0, 0, 0};
    for (int k = rank - 1; k >= 0; --k) {
      double v = -M[k][rank + c];
      for (int t = k + 1; t < rank; ++t) v -= M[k][t] * y[t];
      y[k] = v / M[k][k];
    }
    for (int k = 0; k < rank; ++k) N[3 * colp[k] + c] = y[k];
    N[3 * colp[rank + c] + c] = 1.0;
  }
  return dim;
}

// pinocchio::log3
HBP_HD inline void log3(const double* R, double* w) {
  const double tr = R[0] + R[4] + R[8];
  const double PI_ = 3.14159265358979323846;
  double theta;
  if (tr >= 3.0) theta = 0.0; else if (tr <= -1.0) theta = PI_; else theta = acos((tr - 1.0) * 0.5);
  const double v[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
  if (theta >= PI_ - 1e-2) {
    // near pi: axis from the diagonal, signs from the skew part
    const double c = cos(theta) , s = sin(theta), t1 = 1.0 - c;
    const double k = theta;
    (void)s;
    for (int i = 0; i < 3; ++i) {
      const double d = (R[4 * i] - c) / t1;
      const double a = sqrt(d > 0 ? d : 0.0);
      w[i] = k * (v[i] >= 0 ? a : -a);
    }
    return;
  }
  const double f = (theta > 1e-8) ? theta / (2.0 * sin(theta)) : 0.5 * (1.0 + theta * theta / 6.0);
  for (int i = 0; i < 3; ++i) w[i] = f * v[i];
}

HBP_HD inline double norm3(const double* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

// InverseKinematics::computeTranslationIK (InverseKinematics.cpp:37-127)
HBP_HD inline void translation_ik(const PlanConsts& pc, int leg, const double* pose, double* qj, const double* des) {
  const double err_tol = 0.01, conv_tol = 0.001, dt = 0.7; const int max_it = 5;
  LegKin k; leg_kin(pc, leg, pose, qj, k);
  double err[3] = {k.toe[0] - des[0], k.toe[1] - des[1], k.toe[2] - des[2]};
  double last = norm3(err);
  if (last < err_tol) return;
  int it = 0;
  while (true) {
    double vi[5], nq[5];
    qrcp_solve(k.Jl, 3, 5, err, 0.01, vi);
    for (int i = 0; i < 5; ++i) {
      nq[i] = qj[i] - dt * vi[i];
      nq[i] = dmax(pc.lower[5 * leg + i], nq[i]);
      nq[i] = dmin(pc.upper[5 * leg + i], nq[i]);
    }
    LegKin kn; leg_kin(pc, leg, pose, nq, kn);
    for (int r = 0; r < 3; ++r) err[r] = kn.toe[r] - des[r];
    const double en = norm3(err);
    if (en > last) break;
    if (fabs(en - last) < conv_tol) break;
    last = en;
    for (int i = 0; i < 5; ++i) qj[i] = nq[i];
    k = kn;
    if (en < err_tol) break;
    if (++it >= max_it) break;
  }
}

// InverseKinematics::computeRotationIK (:135-231): orientation error reduced inside the kernel of the translational Jacobian
HBP_HD inline void rotation_ik(const PlanConsts& pc, int leg, const double* pose, double* qj, const double* Rdes) {
  const double err_tol = 0.01, conv_tol = 0.001, dt = 0.7; const int max_it = 5;
  auto rot_err = [&](const LegKin& k, double* e) {
    double M[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) M[3 * i + j] = Rdes[i] * k.R[j] + Rdes[3 + i] * k.R[3 + j] + Rdes[6 + i] * k.R[6 + j];   // Rdes^T R
    log3(M, e);
  };
  LegKin k; leg_kin(pc, leg, pose, qj, k);
  double err[3]; rot_err(k, err);
  double last = norm3(err);
  if (last < err_tol) return;
  int it = 0;
  while (true) {
    // LOCAL frame Jacobians: rows rotated by R^T (the kernel of the linear part is unchanged by the rotation)
    double Jll[15], Jal[15];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 5; ++c) {
      Jll[5 * r + c] = k.R[r] * k.Jl[c] + k.R[3 + r] * k.Jl[5 + c] + k.R[6 + r] * k.Jl[10 + c];
      Jal[5 * r + c] = k.R[r] * k.Ja[c] + k.R[3 + r] * k.Ja[5 + c] + k.R[6 + r] * k.Ja[10 + c];
    }
    double Nk[15];
    const int dim = fullpiv_kernel(Jll, Nk);
    double JN[9] = {0}, y[3] = {0, 0, 0}, vi[5] = {0, 0, 0, 0, 0};
    if (dim > 0) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < dim; ++c) { double d = 0; for (int j = 0; j < 5; ++j) d += Jal[5 * r + j] * Nk[3 * j + c]; JN[r * dim + c] = d; }
      qrcp_solve(JN, 3, dim, err, 0.01, y);
      for (int j = 0; j < 5; ++j) { double d = 0; for (int c = 0; c < dim; ++c) d += Nk[3 * j + c] * y[c]; vi[j] = -d; }
    }
    double nq[5];
    for (int i = 0; i < 5; ++i) {
      nq[i] = qj[i] + dt * vi[i];
      nq[i] = dmax(pc.lower[5 * leg + i], nq[i]);
      nq[i] = dmin(pc.upper[5 * leg + i], nq[i]);
    }
    LegKin kn; leg_kin(pc, leg, pose, nq, kn);
    rot_err(kn, err);
    const double en = norm3(err);
    if (en > last) break;
    if (fabs(en - last) < conv_tol) break;
    last = en;
    for (int i = 0; i < 5; ++i) qj[i] = nq[i];
    k = kn;
    if (en < err_tol) break;
    if (++it >= max_it) break;
  }
}

HBP_HD inline double swing_value(const hb_reference* ref, int c, int a, double t) {
  const int n = ref->n_segments[c][a];
  int s = 0;
  while (s + 1 < n && t > ref->segments[c][a][s][1]) ++s;       // an event time belongs to the earlier phase (lookup::findIndexInTimeArray)
  const double* g = ref->segments[c][a][s];
  const double T = g[1] - g[0], tn = (t - g[0]) / T, dp = g[4] - g[2], dv = g[5] - g[3];
  const double c0 = g[2], c1 = g[3] * T, c2 = -(3.0 * g[3] + dv) * T + 3.0 * dp, c3 = (2.0 * g[3] + dv) * T - 2.0 * dp;
  return ((c3 * tn + c2) * tn + c1) * tn + c0;
}

// SwitchedModelReferenceManager::calculateJointRef (:251-300): resample the target every 0.15 s and replace the joint part by IK on the
// planned toe positions, each sample seeded by the previous one. Returns false when the sample count exceeds HB_MAX_TARGETS.
// Step 1 of calculateJointRef: the resampled target (sample times, interpolated states, default joints in sample 0).
// Returns the number of samples n (0: horizon too short, the two-sample target stays; -1: more than HB_MAX_TARGETS samples).
// `old` is scratch for the input samples (the device kernel passes shared memory, so that no thread holds a Target on its stack).
HBP_HD inline int joint_refs_resample(const PlanConsts& pc, double init_time, double final_time, Target& tg, Target& old) {
  if (tg.n <= 1) return 0;
  const double step = 0.15;
  const int n = (int)floor((final_time - init_time) / step) + 1;
  if (n <= 2) return 0;
  if (n > HB_MAX_TARGETS) return -1;
  old = tg;
  tg.n = n;
  for (int i = 0; i < n; ++i) {
    // Eigen LinSpaced: low + i * (high - low) / (n - 1), the last point set to high
    tg.t[i] = (i == n - 1) ? final_time : init_time + i * ((final_time - init_time) / (n - 1));
    target_state(old, tg.t[i], tg.x[i]);
  }
  for (int j = 0; j < 10; ++j) tg.x[0][12 + j] = pc.default_joints[j];
  return n;
}

// Step 2 for one leg: IK at every sample, seeded by the previous sample's solution of the same leg (the legs do not interact).
HBP_HD inline void joint_refs_leg(const PlanConsts& pc, const hb_reference* sp, int leg, const double* init_state, Target& tg) {
  double Rdes[9];
  rot_zyx_mat(init_state + 9, Rdes);
  double qj[5];
  for (int k = 0; k < 5; ++k) qj[k] = tg.x[0][12 + 5 * leg + k];
  for (int i = 0; i < tg.n; ++i) {
    const double des[3] = {swing_value(sp, leg, 0, tg.t[i]), swing_value(sp, leg, 1, tg.t[i]), swing_value(sp, leg, 2, tg.t[i])};
    translation_ik(pc, leg, tg.x[i] + 6, qj, des);
    rotation_ik(pc, leg, tg.x[i] + 6, qj, Rdes);
    for (int k = 0; k < 5; ++k) tg.x[i][12 + 5 * leg + k] = qj[k];
  }
}

// SwitchedModelReferenceManager::calculateJointRef (:251-300): resample the target every 0.15 s and replace the joint part by IK on the
// planned toe positions, each sample seeded by the previous one. Returns false when the sample count exceeds HB_MAX_TARGETS.
HBP_HD inline bool joint_references(const PlanConsts& pc, const hb_reference* sp, double init_time, double final_time, const double* init_state, Target& tg) {
  Target old;
  const int n = joint_refs_resample(pc, init_time, final_time, tg, old);
  if (n < 0) return false;
  if (n == 0) return true;
  joint_refs_leg(pc, sp, 0, init_state, tg);
  joint_refs_leg(pc, sp, 1, init_state, tg);
  return true;
}

// ------------------------------------------------------------------------------------------------------------------------------
// P2: speed-based gait selection (SwitchedModelReferenceManager::{calculateVelAbs, walkGait, trotGait}, :185-249).
// Returns the gait level after the update (0 stance, 1 trot, 3 "flying trot" level which inserts no template in the reference) and sets
// *insert to 1 when the reference would insert a template on this call (stance or trot), 0 otherwise. The reference leaves velAvg_
// uninitialised before the first call; here the history starts empty, which gives the same values from the first call on.
HBP_HD inline int gait_select(hb_gait_selector* st, int gait_type, const double* cmd_vel /*vx,vy,vz,wz*/, const double* target0 /*22*/, int* insert) {
  Vec3 c = rot_zyx(target0 + 9, {cmd_vel[0], cmd_vel[1], cmd_vel[2]});
  const double vc[4] = {c.x, c.y, 0.0, cmd_vel[3] / 3.0};
  const double ve[4] = {target0[0], target0[1], 0.0, target0[3] / 3.0};
  double s2 = 0.0;
  for (int i = 0; i < 4; ++i) { const double m = 0.5 * vc[i] + 0.5 * ve[i]; s2 += m * m; }
  const double vel_abs = sqrt(s2);
  st->history[st->head] = vel_abs;                       // ring buffer of the 50 most recent samples
  st->head = (st->head + 1) % 50;
  if (st->count < 50) st->count++;
  double sum = 0.0;
  for (int i = 0; i < st->count; ++i) sum += st->history[i];
  st->vel_avg = sum / st->count;
  *insert = 0;
  if (gait_type == 0) {                                  // walkGait
    if (st->vel_avg <= 0.02) { if (st->gait_level != 0) { *insert = 1; st->gait_level = 0; } }
    else if (st->vel_avg > 0.03 && st->vel_avg < 0.4) { if (st->gait_level != 1) { *insert = 1; st->gait_level = 1; } }
    else if (st->vel_avg >= 0.4) { if (st->gait_level != 3) st->gait_level = 3; }
  } else if (gait_type == 2) {                           // trotGait
    if (st->gait_level != 1) { *insert = 1; st->gait_level = 1; }
  }
  return st->gait_level;
}

// mode schedule restricted to the window (events strictly inside), keeping the mode in force at t_lo; target samples
HBP_HD inline int write_schedule_and_targets(const ModeSchedule& ms, const Target& tg, double t_lo, double t_hi, hb_reference* out) {
  int first = 0;
  while (first < ms.n_events && ms.events[first] <= t_lo) ++first;
  int last = first;
  while (last < ms.n_events && ms.events[last] < t_hi) ++last;
  const int ne = last - first;
  if (ne > HB_MAX_EVENTS) return -5;
  out->n_events = ne;
  for (int i = 0; i < ne; ++i) out->event_times[i] = ms.events[first + i];
  for (int i = 0; i <= ne; ++i) out->modes[i] = ms.modes[first + i];
  out->n_targets = tg.n;
  for (int k = 0; k < tg.n; ++k) { out->target_times[k] = tg.t[k]; memcpy(out->target_states[k], tg.x[k], sizeof(double) * 22); }
  return 0;
}

// One instance, start to finish: schedule, target (the given one, or the cmd_vel target when target is null), swing planner, IK joint
// references, compact output; with the planner settings `settings` (null: the compiled-in ones) and the height map `map` (null: none).
// Returns 0, -1 (invalid input) or -5 (schedule / reference capacity exceeded, or a swing phase without take-off / touch-down time).
HBP_HD inline int plan_one(const PlanConsts& pc, const hb_plan_input& p, const hb_target* target, const hb_planner_settings* settings,
                           const hb_terrain* map, double* latest_stance /*12, in/out*/, hb_reference* out, bool zero_fill) {
  if (!(p.horizon > 0.0) || !(p.prev_event < p.gait_start) || p.gait < 0 || p.gait > 3) return -1;
  const double tf = p.t0 + p.horizon;
  if (zero_fill) memset(out, 0, sizeof(*out));
  PlanSettings ps;
  plan_settings(settings, p.gait, ps);
  ModeSchedule ms;
  // the reference tiles over [t0 - T, tf + T] (SwitchedModelReferenceManager.cpp:147)
  if (!tile_gait(ps.tmpl, p.prev_event, p.gait_start, p.t0 - p.horizon, tf + p.horizon, ms)) return -5;
  Target tg;
  if (target) target_from(*target, tg);
  else tg = cmd_vel_to_target(pc, p.cmd_vel, p.t0, p.x0, p.time_to_target, map);
  const double body_vel_cmd[6] = {p.cmd_vel[0], p.cmd_vel[1], p.cmd_vel[2], p.cmd_vel[3], 0.0, 0.0};
  SwingOut so{out, p.t0 - 1e-9, tf + 1e-9, false};
  for (int c = 0; c < 4; ++c) for (int a = 0; a < 3; ++a) out->n_segments[c][a] = 0;
  if (!plan_swing(ps, ms, tg, p.t0, p.feet_pos, body_vel_cmd, latest_stance, so, map) || so.overflow) return -5;
  if (p.joint_ik && !joint_references(pc, out, p.t0, tf, p.x0, tg)) return -5;
  return write_schedule_and_targets(ms, tg, so.t_lo, so.t_hi, out);
}

}  // namespace hbplan
