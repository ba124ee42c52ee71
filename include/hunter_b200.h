/* hunter_b200.h -- C ABI of libhunter_b200.so: batched NMPC iteration + WeightedWbc QP for the Hunter biped on H100.
 *
 * Every entry point replaces one operator of the reference's per-control-step path (SURVEY.md 8b); the reference-side
 * bindings (C++ adapters deriving from ocs2::MPC_BASE / legged::WbcBase) are shown in INTEGRATION.md.
 *
 *   hb_wbc_solve_batch      <-> legged::WeightedWbc::update            legged_wbc/src/WeightedWbc.cpp:18-66,
 *                               legged::WbcBase::update               legged_wbc/include/legged_wbc/WbcBase.h:43-44
 *   hb_wbc_qp_batch         <-> qpOASES::QProblem::init + getPrimalSolution   legged_wbc/src/WeightedWbc.cpp:44-55
 *   hb_hierarchical_wbc_solve_batch <-> legged::HierarchicalWbc::update   legged_wbc/src/HierarchicalWbc.cpp:18-31
 *   hb_hoqp_solve_batch     <-> legged::HoQp (null-space cascade)          legged_wbc/src/HoQp.cpp:21-198
 *   hb_mpc_solve_batch      <-> ocs2::MPC_MRT_Interface::advanceMpc -> SqpMpc/SqpSolver::run (one SQP iteration)
 *                               legged_controllers/src/LeggedController.cpp:378-379,406
 *   hb_mpc_cold_start_batch <-> LeggedRobotInitializer::compute       legged_interface/src/initialization/LeggedRobotInitializer.cpp:67-77
 *   hb_policy_eval_batch    <-> MPC_MRT_Interface::evaluatePolicy     legged_controllers/src/LeggedController.cpp:154-156
 *   hb_control_step_batch   <-> LeggedController::update MPC->policy->WBC->torque law   LeggedController.cpp:137-257
 *   hb_resident_cycle_batch <-> SqpSolver::run with its resident primalSolution_ (warm start) + the rest of LeggedController::update
 *   hb_resident_plan_cycle_batch <-> ReferenceManager::preSolverRun (planner on the device) + hb_resident_cycle_batch
 *   hb_estimator_update_batch <-> KalmanFilterEstimate::update        legged_estimation/src/LinearKalmanFilter.cpp:72-185
 *   hb_contact_force_estimate_batch <-> StateEstimateBase::estContactForce   legged_estimation/src/StateEstimateBase.cpp:130-206
 *   hb_joint_command_batch  <-> joint command / torque law            LeggedController.cpp:186-257
 *   hb_plan_references      <-> GaitSchedule tiling + SwingTrajectoryPlanner::update + cmdVelToTargetTrajectories + calculateJointRef
 *   hb_gait_select          <-> SwitchedModelReferenceManager::calculateVelAbs + walkGait/trotGait   :185-249
 *   hb_rbd_to_centroidal_batch <-> CentroidalModelRbdConversions::computeCentroidalStateFromRbdModel  LeggedController.cpp:336
 *   hb_reference_expand_batch  <-> SwitchedModelReferenceManager::modifyReferences (gait tiling, swing planner, target
 *                               interpolation, evaluated on the node grid)   legged_interface/src/SwitchedModelReferenceManager.cpp:136-171
 *
 * Conventions: plain pointers and sizes only; no exceptions cross the ABI. Return 0 on success, <0 on misuse / CUDA error
 * (hb_strerror). Per-instance status words: 0 converged, 1 iteration cap, 2 infeasible / ill-posed, 3 NaN
 * (the raw QP adds 4, beyond its row capacity: see hb_wbc_qp_batch_dev).
 * All arithmetic is IEEE float64 (the reference is all-double: ocs2::scalar_t).
 * Layouts (row-major, instance-major): state x[22] = [h_lin/m, h_ang/m, p, zyx, q_j]; input u[22] = [F0..F3, qj_dot];
 * rbd[32] = [zyx, p, q_j, omega_world, v, qj_dot]; WBC solution sol[38] = [qdd(16), F(12), tau(10)].
 * The *_host entry points take host pointers (pinned or pageable) and copy through the context's staging buffers;
 * the *_dev entry points take device pointers and run asynchronously on the context's stream (hb_sync to wait).
 */
#ifndef HUNTER_B200_H
#define HUNTER_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct hb_ctx hb_ctx;

typedef struct {
  int32_t horizon_N;     /* shooting intervals (BASELINE: 100; shipped task.info: ~54)            */
  double dt;             /* node spacing [s] (BASELINE: 0.01; task.info:82 0.015)                 */
  int32_t max_batch;     /* capacity of the context's scratch buffers                             */
  double wbc_rho;        /* Tikhonov weight that defines the least-norm WBC optimum (qpOASES setToMPC regularisation) */
  int32_t qp_max_iter;   /* interior-point iteration cap                                          */
  int32_t line_search_max_trials; /* trials of the filter line search, alpha = 1, 1/2, ...; >= 1 (hb_create rejects less:
                                     a line search of no trials never steps). Default 14; alpha >= 1e-4 ends the search at
                                     14 trials, so caps above 14 act as 14                                               */
  double time_horizon;   /* mpc.timeHorizon [s] (task.info:144 0.8); 0 = horizon_N * dt. Used by the event-node grid */
  int32_t event_nodes;   /* 1: the resident cycle discretises [t0, t0 + time_horizon] like ocs2::timeDiscretizationWithEvents
                            (steps of dt, a node on every mode switch, grid re-anchored there, last node = final time); horizon_N is
                            then the node capacity. 0: uniform grid t0 + k dt (BASELINE configs)                          */
  int32_t e2e_chunks;    /* host-pointer cycle calls split the batch into this many chunks pipelined over two streams (copies of one
                            chunk overlap kernels of the other); 0 = automatic                                            */
} hb_config;

typedef struct {
  double alpha;          /* accepted step length (0 = step rejected, iterate kept)                */
  double merit0, merit1; /* merit before / after                                                  */
  double viol0, viol1;   /* sqrt(dynamics SSE + equality SSE) before / after                      */
  double armijo;         /* descent metric of the projected subproblem                            */
  int32_t status;        /* 0 ok, 3 NaN                                                           */
  int32_t n_trials;      /* line-search trials evaluated                                          */
} hb_solve_info;

/* compact per-instance reference description consumed by hb_reference_expand_batch */
#define HB_MAX_EVENTS 32
#define HB_MAX_TARGETS 16
#define HB_MAX_SEGMENTS 24
#define HB_MAX_HORIZON 512   /* hb_create rejects longer horizons (shared-memory staging of one instance's trajectories) */
typedef struct {
  int32_t n_events;                       /* mode schedule: modes[i] holds on (event_times[i-1], event_times[i]] */
  double event_times[HB_MAX_EVENTS];
  int32_t modes[HB_MAX_EVENTS + 1];
  int32_t n_targets;                      /* target trajectory samples (time, state)                              */
  double target_times[HB_MAX_TARGETS];
  double target_states[HB_MAX_TARGETS][22];
  int32_t n_segments[4][3];               /* per contact, per axis: cubic Hermite segments [t0,t1,p0,v0,p1,v1]    */
  double segments[4][3][HB_MAX_SEGMENTS][6];
} hb_reference;

/* inputs of the host-side reference planner (one MPC solve of one instance) */
typedef struct {
  double t0;              /* solver init time                                                             */
  double horizon;         /* final time = t0 + horizon                                                    */
  double time_to_target;  /* TIME_TO_TARGET of the cmd_vel target (TargetTrajectoriesPublisher.cpp:107)   */
  double gait_start;      /* time at which the gait template starts (STANCE before)                       */
  double prev_event;      /* an event time inside the initial stance (< gait_start)                       */
  double x0[22];          /* current observation state                                                    */
  double cmd_vel[4];      /* filtered command: vx, vy, vz, yaw rate (body frame)                          */
  double feet_pos[12];    /* current contact positions in world (hb_contact_positions_batch)              */
  int32_t gait;           /* 0 stance, 1 trot, 2 standing_trot, 3 flying_trot (gait.info; hb_planner_settings) */
  int32_t joint_ik;       /* 1: resample the target every 0.15 s and fill joint references by IK (calculateJointRef,
                             SwitchedModelReferenceManager.cpp:251-300); 0: keep the two-sample target with default joints */
} hb_plan_input;

/* A target trajectory of one instance (the TargetTrajectories the planner tracks: the two-sample target cmdVelToTargetTrajectories or
 * goalToTargetTrajectories publishes, or any other): piecewise-linear in time between the samples, held before the first and after the
 * last. The input trajectory is zero, as in every target the reference publishes. */
typedef struct {
  int32_t n;                              /* samples, 1..HB_MAX_TARGETS                                            */
  double time[HB_MAX_TARGETS];            /* absolute times, strictly ascending                                    */
  double state[HB_MAX_TARGETS][22];       /* state samples (layout of x)                                           */
} hb_target;

/* ---- planner settings: how each gait steps and swings, the reference's run-time planner configuration ----
 * gait[g] is the ModeSequenceTemplate of gait g (hb_plan_input.gait, hb_rollout_command.gait), the templates of gait.info in its `list`
 * order (legged_controllers/config/hunter/gait.info; loadModeSequenceTemplate, ModeSequenceTemplate.cpp:59-83); the swing fields are
 * swing_trajectory_config (task.info:21-34; loadSwingTrajectorySettings, SwingTrajectoryPlanner.cpp:549-561). The template is tiled as
 * the compiled-in one is: mode modes[k] holds for switching_times[k + 1] - switching_times[k], the period is switching_times[n_phase].
 * Swing apex: max(lift-off z, touch-down z) + min(1, swing duration / swing_time_scale) * swing_height; every planned foothold and every
 * stance foot stands at next_stance_z; the nominal foothold offset of foot c from the base is (x, +-feet_bias_y, feet_bias_z), with
 * x = feet_bias_x1 for the toes (contacts 0, 1) and feet_bias_x2 for the heels (2, 3), +y for the left contacts (0, 2).
 * Validity (the setters and hb_plan_references_settings return -1 otherwise): for each gait n_phase in 1..HB_GAIT_MAX_PHASES, modes[k] in
 * 0..3 and switching_times[0..n_phase] finite, starting at 0 and strictly ascending (the entries beyond n_phase are not read);
 * swing_height finite and >= 0, swing_time_scale finite and > 0, the other swing fields finite.
 * A valid template may still be too short for the planner's capacities: more than 128 phases tiled over [t0 - T, t0 + 2T] (T the
 * horizon), more than HB_MAX_EVENTS events inside the horizon or more than HB_MAX_SEGMENTS swing segments per foot and axis. Such a
 * plan fails with status -5, like any plan over the capacities, and the episodes count it in plan_rejects. */
#define HB_GAIT_MAX_PHASES 8
typedef struct {                     /* ModeSequenceTemplate (gait.info)                                                          */
  int32_t n_phase;                   /* 1..HB_GAIT_MAX_PHASES                                                                     */
  int32_t modes[HB_GAIT_MAX_PHASES]; /* 0 FLY, 1 R, 2 L, 3 STANCE (MotionPhaseDefinition.h:57-60)                                 */
  double switching_times[HB_GAIT_MAX_PHASES + 1];   /* [0] == 0, strictly ascending; the period is [n_phase]                      */
} hb_gait_template;                  /* 112 B */
typedef struct {
  hb_gait_template gait[4];          /* indexed by hb_plan_input.gait / hb_rollout_command.gait                                   */
  double swing_height, swing_time_scale, next_stance_z;           /* swing_trajectory_config                                       */
  double feet_bias_x1, feet_bias_x2, feet_bias_y, feet_bias_z;
} hb_planner_settings;               /* 504 B */
/* The shipped settings (host only): gait.info's four templates and task.info's swing block, the values compiled into the planner. */
int hb_default_planner_settings(hb_planner_settings* s);
/* hb_planner_settings from a task.info and a gait.info file (host only), with the INFO reader of hb_parse_task_info: swing_trajectory_config's
 * swingHeight, swingTimeScale, feet_bias_x1/x2/y/z and next_position_z (the key the reference loads; the shipped task.info names it
 * next_stance_position_z, so the loader's default 0.02 applies, SwingTrajectoryPlanner.cpp:560), and for g = 0..3 the template named by
 * `list.[g]` of gait_info (modeSequence names FLY, R, L, STANCE; switchingTimes). As in hb_parse_task_info, a key or template that is absent
 * keeps its default (hb_default_planner_settings). -1: a NULL argument, a file missing or malformed, an unknown mode name, a template whose
 * mode and time counts do not match (n modes, n + 1 times) or that has more than HB_GAIT_MAX_PHASES phases, or a result that is not valid. */
int hb_parse_planner_settings(const char* task_info, const char* gait_info, hb_planner_settings* out);

/* ---- height maps: the ground the planner is told about, the reference's terrainHeight as a function of (x, y) ----
 * A height map is an hb_terrain record (terrain, below) that the planner reads; the reference plans with terrainHeight = 0 everywhere
 * (SwitchedModelReferenceManager.cpp:152). For an instance with a map m, h(x, y) is the terrain lookup of m (the grid, clamping and
 * bilinear rules of terrain, below) with each of its products rounded on its own, so the host and the device get the same bits. Map
 * heights are measured from the ground the planner otherwise assumes: an all-zero map is the planner without one, and over a plant whose
 * flat ground is at sim.ground_height = g the map of a terrain H is H - g. With a map the planner changes in these places only:
 *  - lift-off: every stance foot's latest stance point has z = next_stance_z + h at its (x, y);
 *  - touch-down: every planned foothold r has r.z = next_stance_z + h(r.x, r.y);
 *  - swing z: the four-node z spline is built on its ends lowered by h_lo = min(lift-off z, touch-down z) - next_stance_z, with the shape
 *    of swing_trajectory_config, and h_lo is added back to its node positions (velocities are differences and stay);
 *  - centrifugal term of the foothold: sqrt((z - h(x, y)) / g) with (x, y, z) the body position it reads;
 *  - body height of the targets: with the pose p = x[6:12] and z' = p[2] + clamp(HB_COM_HEIGHT + h(p[0], p[1]) - p[2], -0.04, 0.04), the
 *    cmd_vel target's sample 0 has height z' and its sample 1 HB_COM_HEIGHT + h at sample 1's (x, y); the goal target's sample 0 has z'
 *    and its goal sample z' + (h(goal x, y) - h(p[0], p[1])), also when it is the only sample. The teleop messages' target is the cmd_vel
 *    target.
 * A map of zeros gives the plans and targets of no map bit for bit; an instance without a map plans as before. The IK joint references
 * follow the swing splines and the targets. Maps are read by every device planner path (hb_plan_set_maps) and by the host calls
 * hb_plan_references_maps, hb_goal_to_target_maps and hb_cmd_vel_to_target_maps. The MPC, WBC, joint law and estimator do not read them;
 * the estimator is told about the ground by estimator maps (below), records of this type set on their own. */

/* ---- estimator maps: the ground the Kalman filter is told about, its feet heights as a function of (x, y) ----
 * An estimator map is an hb_terrain record that the filter reads; the reference measures each foot's height as feetHeights_, zero unless
 * updateFromTopic writes it (LinearKalmanFilter.cpp:62, 143, 227). For an instance with a map m, the update's measurement row 24 + c is
 * y = h_m(x[6 + 3c], x[7 + 3c]) at the predicted state x (the prediction does not move the feet: the previous estimate's foot xy), with h_m
 * the height-map lookup (height maps, above; the same bits on the host and the device). C, R, Q and the decoupling do not change, and the
 * row stays the foot's z: it has no -grad h . (x, y) coupling (no linearisation of the ground; the foot xy is measured kinematically by
 * rows 0..11, and a step of the map is a one-cell ramp whose gradient would make such a row jump between ticks). Map heights are measured
 * from the ground the filter otherwise assumes (z = 0), as a height map's: over a plant whose flat ground is at g the map of a terrain H is
 * H - g, so one record serves both settings. A mapped update does not read feet_heights; the odometry fusion still writes it, and with a
 * camera and a map the map wins. An all-zero map is the filter without one bit for bit while feet_heights is +0 (every episode without
 * odometry: hb_kf_reset sets +0 and only the fusion writes it). Maps are read by hb_estimator_update_batch_dev, hb_estimator_update_batch
 * and hb_rollout_estimated_batch_dev (hb_estimator_set_maps); the truth episodes, the planner, the plant and hb_estimator_fuse_odometry
 * do not read them. */

/* ---- MPC maps: the ground the MPC's stance feet are held on ----
 * An MPC map is an hb_terrain record that the MPC's stance-foot equality reads. The reference's row (LeggedInterface.cpp:436-446) is
 * v_c + diag(0, 0, 3) p_c + (0, 0, -0.06) = 0: its z row pulls every stance contact towards z = 0.02, flat ground. For an instance with a
 * map m, at node k and each contact c in stance there, h = h_m(x, y) at the swing reference's position of c at the node (swing_ref[k][6c],
 * [6c + 1]: for a stance phase the planner's stance position, the foot's current position for the current stance and the planned foothold
 * for later ones), with h_m the height-map lookup (height maps, above; one record means the same ground to the planner, the filter and
 * the MPC). The z row is then (v_z + 3 p_z - 0.06) - 3 h, so the stance foot is held at 0.02 + h; the linearisation's row and the line
 * search's violation use the same h. h depends on the reference, not on the iterate: the row's Jacobian is unchanged and has no grad h
 * coupling (a step of the map is a one-cell ramp, as for estimator maps). Swing rows, friction cones (MPC cone maps, below), costs, the
 * WBC, the planner, the filter and the plant do not read MPC maps. An all-zero map (h = +0) is the solve without one bit for bit. Map heights are measured
 * from the flat ground the MPC otherwise assumes (z = 0), as height maps' are. Maps are read by every MPC path (hb_mpc_set_maps). */

/* ---- WBC maps: the ground the WBC's friction pyramids stand on ----
 * A WBC map is an hb_terrain record that the WBC's friction constraint reads. The reference's pyramid (WbcBase::formulateFrictionConeTask,
 * WbcBase.cpp:205-221) is about the world z axis: rows (0, 0, -1), (+-1, 0, -mu), (0, +-1, -mu) on each stance contact's force. For an
 * instance with a map m, each stance contact c gets the frame of m at its measured position (the contact position of the forward
 * kinematics at the rbd state the WBC is given: in estimated episodes the estimate, so the lookup drifts with the estimate unless
 * odometry is set): with (gx, gy) the gradient of the height-map lookup (height maps, above) at (x_c, y_c),
 *   L = sqrt(1 + gx^2 + gy^2),  n = (-gx, -gy, 1) / L,  t1 = (1, 0, gx) / sqrt(1 + gx^2),  t2 = n x t1,
 * every product rounded on its own as the lookup's. The contact's five rows become -n, t1 - mu n, -t1 - mu n, t2 - mu n, -t2 - mu n, each
 * with bound 0, mu the instance's friction_coefficient (the context's hb_wbc_settings or its controller setting). Where gx == 0 and
 * gy == 0 (a zero map, a plateau cell, a point off the grid on both axes) the rows are the flat rows unchanged, the plant's own flat-path
 * rule, so an all-zero map is the WBC without one bit for bit. The normal is the bilinear gradient the plant's sloped contact pushes along:
 * a foot on a step's one-cell ramp gets the ramp's steep normal, as it does in the plant; there is no smoothing over the foot. Every other
 * WBC row (EoM, torque limits, zero swing forces, no contact motion, swing-leg, base and contact-force tasks), the MPC's friction cone
 * (MPC cone maps, below), the planner, the filter and the plant do not read WBC maps. Maps are read by every WBC path (hb_wbc_set_maps). */

/* ---- MPC cone maps: the ground the MPC's friction cones stand on ----
 * An MPC cone map is an hb_terrain record that the MPC's friction cone (FrictionConeConstraint) reads. The reference's cone is
 * h = mu F_z - sqrt(F_x^2 + F_y^2 + reg) on the local force t_R_w F of each stance contact (FrictionConeConstraint.cpp:78-233), with
 * t_R_w the identity: a cone about the world z axis. For an instance with a cone map m, at node k and each contact c in stance there,
 * t_R_w has the rows t1, t2 and n of the WBC maps' frame (above) at the swing reference's position of c at the node (swing_ref[k][6c],
 * [6c + 1], where MPC maps look up the stance height). The cone is then h = mu Fl_z - sqrt(Fl_x^2 + Fl_y^2 + reg) with
 * Fl = (t1.F, t2.F, n.F), its input gradient t_R_w' g_l and its input Hessian t_R_w' H_l t_R_w, the reference's chain through
 * dF_du = t_R_w; the linearisation and the line search's trial cost use the same frame. mu, reg, the relaxed barrier and the Hessian
 * diagonal shift are unchanged. Where gx == 0 and gy == 0 (a zero map, a plateau cell, a point off the grid on both axes) and for a swing
 * contact the cone's statements are those without a map, so an all-zero map is the solve without one bit for bit. The frame depends on
 * the reference, not on the iterate. The normal-force limits on u[3c + 2] stay on world z: they are the reference's box on that input,
 * and the tilted cone itself keeps the force's normal component positive (mu Fl_z >= sqrt(reg)). The stance z row (MPC maps, above), the
 * swing rows, the costs, the WBC, the planner, the filter and the plant do not read cone maps. Cone maps are read by every MPC path (hb_mpc_set_cone_maps). */

/* state of the speed-based gait selection of one instance (SwitchedModelReferenceManager velAbsHistory_/velAvg_/gaitLevel_);
 * zero-initialise, then set gait_level = -1 ("no template chosen yet") or the level in force */
typedef struct {
  double history[50];
  double vel_avg;
  int32_t head, count;
  int32_t gait_level;
  int32_t reserved;
} hb_gait_selector;

/* joint PD gains of the command law (dynamic_reconfigure parameters, legged_controllers/cfg/Tutorials.cfg:6-16,
 * LeggedController.cpp:431-447) */
typedef struct {
  double kp_position, kd_position;            /* before the controller is loaded                     */
  double kp_big_stance, kp_big_swing, kd_big; /* hip pitch / knee (joints 2,3,7,8)                   */
  double kp_small_stance, kp_small_swing, kd_small; /* hip roll / yaw (0,1,5,6) and ankle kp (4,9)   */
  double kd_feet;                             /* ankle (4,9)                                         */
} hb_pd_gains;

/* ---- state estimator (SURVEY 8f row N3): linear Kalman filter of legged_estimation/src/LinearKalmanFilter.cpp:72-185 ---- */
typedef struct {
  double x_hat[18];        /* base position(3), base linear velocity(3), four contact positions(12), world frame */
  double P[18 * 18];       /* covariance, row-major                                                              */
  double feet_heights[4];  /* terrain height under each contact (measurement rows 24..27; not read on an estimator map) */
} hb_kf_state;

typedef struct {           /* task.info:336-345 */
  double foot_radius, imu_process_noise_position, imu_process_noise_velocity, foot_process_noise_position;
  double foot_sensor_noise_position, foot_sensor_noise_velocity, foot_height_sensor_noise;
} hb_kf_params;

/* state of the generalised-momentum observer behind the contact-force estimate (pSCgZinvlast_, StateEstimateBase.h:125) */
typedef struct { double p_filtered[16]; } hb_observer_state;
int hb_observer_reset(int B, hb_observer_state* state);   /* host only: zeros (StateEstimateBase.cpp:58-59) */

/* ---- run-time WBC settings: what WbcBase::loadTasksSetting / WeightedWbc::loadTasksSetting read from task.info
 * (legged_wbc/src/WbcBase.cpp:352-411, WeightedWbc.cpp:96-111) and WbcBase::setKpKd changes (WbcBase.h:65-69) ---- */
typedef struct {
  double torque_limits[5];            /* torqueLimitsTask (motor 1..5 of a leg)                    task.info:290-297 */
  double friction_coefficient;        /* frictionConeTask.frictionCoefficient                      :299-302          */
  double swing_kp, swing_kd;          /* swingLegTask                                              :304-308          */
  double base_accel_kp, base_accel_kd;   /* baseAccelTask (loaded by the reference, used by no task) :310-314        */
  double base_height_kp, base_height_kd; /* baseHeightTask                                          :316-320         */
  double base_angular_kp, base_angular_kd; /* baseAngularTask                                       :322-326         */
  double weight_swing_leg, weight_base_accel, weight_contact_force;   /* weight                     :328-333         */
} hb_wbc_settings;

/* what hb_parse_task_info extracts from a task.info file (boost property-tree INFO format): the WBC block above, the estimator
 * parameters and the solver discretisation. `found` has one bit per section that was present (1 WBC, 2 kalmanFilter,
 * 4 contactForceEsimation, 8 sqp, 16 mpc); absent sections keep the defaults. */
typedef struct {
  hb_wbc_settings wbc;
  double kalman[7];                   /* hb_kf_params in declaration order (kalmanFilter, task.info:336-345)                */
  double contact_force_cutoff_frequency, contact_threshold;   /* contactForceEsimation                   :347-351          */
  double sqp_dt;                      /* sqp.dt                                                            :82               */
  int32_t sqp_iteration;              /* sqp.sqpIteration                                                  :83               */
  double mpc_time_horizon;            /* mpc.timeHorizon                                                   :144              */
  int32_t mpc_cold_start;             /* mpc.coldStart                                                     :146              */
  int32_t found;
} hb_task_info;

int hb_default_wbc_settings(hb_wbc_settings* s);
int hb_parse_task_info(const char* path, hb_task_info* out);          /* host only; -1: file missing or malformed */
/* the WBC settings in force for this context (defaults: the shipped task.info values compiled into include/hunter_model_constants.h) */
int hb_wbc_get_settings(const hb_ctx* ctx, hb_wbc_settings* s);
int hb_wbc_set_settings(hb_ctx* ctx, const hb_wbc_settings* s);
int hb_wbc_set_kp_kd(hb_ctx* ctx, double swing_kp, double swing_kd);   /* WbcBase::setKpKd */
/* The controller's whole-body controller (LeggedController::wbc_), per context. A new context is weighted.
 * Entry points that run the controller's WBC follow it: hb_control_step_batch(_dev), hb_resident_cycle_batch(_dev),
 * hb_resident_plan_cycle_batch, hb_resident_wbc_batch(_dev), hb_rollout_batch_dev and hb_rollout_estimated_batch_dev. Entry points named
 * after one class ignore it: hb_wbc_solve_batch(_dev) is always WeightedWbc, hb_hierarchical_wbc_solve_batch(_dev) always HierarchicalWbc.
 * Under HB_WBC_HIERARCHICAL, stance_mode arguments are accepted and have no effect (WbcBase::setStanceMode is read only by
 * WeightedWbc::formulateWeightedTasks), and the previous-solution fallback of the weighted path applies to a status != 0 (the reference's
 * HoQp applies whatever iterate qpOASES holds; see DESIGN §1 "Hierarchical WBC in the loop"). hb_wbc_set_settings, hb_wbc_set_kp_kd and
 * hb_load_task_info apply to both formulations and leave the choice as it is. */
#define HB_WBC_WEIGHTED 0       /* legged::WeightedWbc (default) */
#define HB_WBC_HIERARCHICAL 1   /* legged::HierarchicalWbc       */
int hb_wbc_set_formulation(hb_ctx* ctx, int32_t formulation);   /* -1 for any other value; the previous choice is kept */
int hb_wbc_get_formulation(const hb_ctx* ctx, int32_t* formulation);
int hb_load_task_info(hb_ctx* ctx, const char* path);                  /* hb_parse_task_info + hb_wbc_set_settings */

/* ---- hierarchical QP (SURVEY 8f row N4): legged::HoQp / legged::HierarchicalWbc ---- */
#define HB_HOQP_MAX_LEVELS 3
#define HB_HOQP_N 38            /* decision variables (the WBC's [qdd, F, tau])                             */
#define HB_HOQP_MAX_EQ 32       /* rows of a (equality task) per level                                      */
#define HB_HOQP_MAX_IN 40       /* rows of d (inequality task) per level                                    */
#define HB_HOQP_MAX_STACKED 80  /* inequality rows of all levels together                                   */
typedef struct {                /* one hierarchy: level 0 has the highest priority (Task a x = b, d x <= f; legged_wbc/include/legged_wbc/Task.h) */
  int32_t n, levels;
  int32_t ma[HB_HOQP_MAX_LEVELS], md[HB_HOQP_MAX_LEVELS];
  double a[HB_HOQP_MAX_LEVELS][HB_HOQP_MAX_EQ][HB_HOQP_N], b[HB_HOQP_MAX_LEVELS][HB_HOQP_MAX_EQ];
  double d[HB_HOQP_MAX_LEVELS][HB_HOQP_MAX_IN][HB_HOQP_N], f[HB_HOQP_MAX_LEVELS][HB_HOQP_MAX_IN];
} hb_hoqp_problem;

/* ---- closed-loop rollout (SURVEY 8f row N2): actuation model of the simulated hardware and a batched rigid-body plant ---- */
#define HB_ACT_CAPACITY 16
typedef struct {           /* command buffer of one robot (LeggedHWSim::cmdBuffer_, legged_gazebo/src/LeggedHWSim.cpp:166-186) */
  int32_t count, head;     /* entries in the ring; index of the newest one                                  */
  double stamp[HB_ACT_CAPACITY];
  double cmd[HB_ACT_CAPACITY][50];   /* per joint: posDes, velDes, kp, kd, ff                               */
} hb_actuation_state;
typedef struct {
  double dt;                /* control period covered by one call [s] (500 Hz loop: 0.002)                  */
  int32_t substeps;         /* semi-implicit Euler substeps per call                                        */
  double ground_height;     /* flat ground z                                                                */
  double ground_stiffness, ground_damping;   /* normal spring-damper per contact point [N/m], [N s/m]       */
  double tangential_damping;                 /* viscous tangential friction [N s/m], clipped to mu * F_z    */
  double friction_mu;
  double joint_armature;    /* rotor inertia added to the joint diagonal of M [kg m^2] (mujoco/model/hunter/hunter.xml:6: 0.1) */
  double joint_damping;     /* viscous joint damping [N m s/rad] (hunter.xml:6: 1)                           */
} hb_sim_params;
int hb_default_sim_params(hb_sim_params* p);
int hb_actuation_reset(int B, hb_actuation_state* state);   /* host only */

/* ---- closed-loop episodes (hb_rollout_batch_dev): planner + MPC cycle at mpc_every ticks, 500 Hz WBC tick, joint command law, actuation
 * delay, saturation and plant, for a batch of robots in one call ---- */
#define HB_ROLLOUT_MAX_CMDS 8
typedef struct {                 /* the command of one instance: gait and a piecewise-constant cmd_vel                            */
  int32_t gait;                  /* 0..3 as hb_plan_input.gait                                                                    */
  double gait_start;             /* as hb_plan_input.gait_start                                                                   */
  int32_t n_cmd;                 /* 1..HB_ROLLOUT_MAX_CMDS                                                                        */
  double cmd_time[HB_ROLLOUT_MAX_CMDS];      /* ascending; cmd_vel[j] holds from cmd_time[j] on (cmd_vel[0] also before cmd_time[0]) */
  double cmd_vel[HB_ROLLOUT_MAX_CMDS][4];
} hb_rollout_command;
typedef struct {
  double period;                 /* one WBC tick [s] (0.002); tick k of a call runs at t = (tick0 + k) * period                   */
  int32_t mpc_every;             /* an MPC cycle on every tick with (tick0 + k) % mpc_every == 0 (5: 100 Hz, task.info mpcDesiredFrequency) */
  double actuation_delay;        /* command delay of the actuation model [s] (legged_gazebo/config/default.yaml:2, 0.009)         */
  hb_sim_params sim;             /* the plant; sim.dt is the time it advances per tick                                            */
  hb_pd_gains gains;             /* joint command law                                                                             */
  double torque_limit[10];       /* actuator saturation of the applied torques (default: HB_WBC_TORQUE_LIMITS per leg)             */
  double min_base_height;        /* failure when the base z falls below it; 0 disables the check                                  */
  int32_t log_every;             /* 0: no log                                                                                     */
} hb_rollout_params;
#define HB_ROLLOUT_FAIL_ESTOP 1        /* the joint command law raised the emergency stop                                       */
#define HB_ROLLOUT_FAIL_ORIENTATION 2  /* |roll| > pi/2 (SafetyChecker::checkOrientation, SafetyChecker.h:34-43)                 */
#define HB_ROLLOUT_FAIL_HEIGHT 4       /* base z < min_base_height (base z above the terrain for an instance with one)         */
#define HB_ROLLOUT_FAIL_NONFINITE 8    /* an rbd entry is not finite                                                           */
typedef struct {                 /* per-instance outcome, in/out: start an episode with zeros and fail_tick = -1                  */
  int32_t fail_tick;             /* absolute tick of the first failure, -1: never failed                                          */
  int32_t fail_reason;           /* HB_ROLLOUT_FAIL_* bits of that tick                                                           */
  int32_t mpc_bad, wbc_fallbacks, plan_rejects;   /* counts of info.status != 0, wbc_status != 0, plan_status != 0                */
  double max_abs_torque;         /* over the applied (saturated) torques, before a plant variation's motor_strength scales them
                                    (with a motor bridge: the mean over the tick's substeps of the motor's clipped torque)        */
} hb_rollout_stats;
int hb_default_rollout_params(hb_rollout_params* p);       /* host only */

/* ---- per-robot episode settings: pushes, plant variations and terrains (hb_rollout_set_pushes / _plant_variations / _terrains) ----
 * Each sets one record per robot on the context: from then on both episode calls apply record i to instance i of their batch for i < B.
 * The records are a host array, validated on the host and copied to the context in stream order on the context's stream; the caller may
 * free it when the call returns. B == 0 clears the setting (the array may be NULL). -1: B < 0, a NULL array with B > 0, or a record
 * outside its documented range; -4: B > max_batch. A rejected call keeps the previous setting and enqueues nothing. Instances at or beyond
 * B run the nominal plant (no push, no variation) on the flat ground of sim.ground_height. The device copy is allocated at max_batch by
 * the first call that sets records and freed by hb_destroy. Settings add no launch to an episode. */

/* The record type of each per-robot setting call, for hb_check_setting_records: hb_push_schedule for hb_rollout_set_pushes,
 * hb_plant_variation for _plant_variations, hb_terrain for _terrains, hb_goal_schedule for _goals, hb_odometry_setting for _odometry,
 * hb_controller_setting for _controller_settings, hb_hardware_setting for _hardware, hb_planner_settings for hb_plan_set_settings,
 * hb_target for hb_plan_set_targets and int32_t latency ticks for hb_rollout_set_mpc_latencies. */
#define HB_SETTING_PUSHES 0
#define HB_SETTING_PLANT_VARIATIONS 1
#define HB_SETTING_TERRAINS 2
#define HB_SETTING_GOALS 3
#define HB_SETTING_ODOMETRY 4
#define HB_SETTING_CONTROLLERS 5
#define HB_SETTING_HARDWARE 6
#define HB_SETTING_PLANNER 7
#define HB_SETTING_TARGETS 8
#define HB_SETTING_LATENCIES 9
#define HB_SETTING_MOTOR_BRIDGE 11     /* hb_motor_bridge for hb_rollout_set_motor_bridge (10 stays unassigned: callers have used it as an unknown kind) */
/* The record check of the setting call of `kind`, without a context (host only, no GPU needed): records (B of the kind's type) are judged
 * by that call's rules for a record, and a record passes iff the call accepts it (the call's other checks, such as B against max_batch,
 * need its context). 0: every record passes, *first_bad = -1. -1: *first_bad is the index of the first record that fails, or -1 for an
 * unknown kind, B < 0 or NULL records with B > 0; -1 also for a NULL first_bad. */
int hb_check_setting_records(int32_t kind, int B, const void* records, int32_t* first_bad);

/* ---- pushed episodes: scheduled external wrenches on the base, applied by the plant of both episode calls ----
 * Push j acts on the plant step of absolute tick a iff t_start[j] <= t && t < t_start[j] + duration[j], with t = (double)a * period (the
 * episode's tick time). During that step the wrench is constant over all substeps, so a push is quantised to whole ticks. Overlapping
 * pushes add up: each of the 6 wrench components starts from 0.0 and the active pushes are added in ascending j. A world force f at the
 * base frame origin (rbd[3:6]) and a world couple tau enter the plant as generalised forces on the base coordinates (p, zyx): Q_p = f and
 * Q_zyx = T' tau, where omega_world = T(zyx) (dyaw, dpitch, droll) is the map behind rbd[16:19], i.e. Q_yaw = tau_z,
 * Q_pitch = -sz tau_x + cz tau_y, Q_roll = cz cy tau_x + sz cy tau_y - sy tau_z, evaluated at each substep's orientation. A push on
 * another point r of the body is the force f plus the couple r x f. The controllers are not told about the push. */
#define HB_MAX_PUSHES 4
typedef struct {                      /* external pushes on one robot's base                                                  */
  int32_t n_push;                     /* 0..HB_MAX_PUSHES; 0 = undisturbed                                                    */
  double t_start[HB_MAX_PUSHES];      /* absolute time [s]                                                                    */
  double duration[HB_MAX_PUSHES];     /* [s], >= 0                                                                            */
  double force[HB_MAX_PUSHES][3];     /* world frame [N], applied at the base frame origin (rbd[3:6])                         */
  double torque[HB_MAX_PUSHES][3];    /* world frame couple [N m]                                                             */
} hb_push_schedule;
/* Sets the push schedules of the context's episodes (a per-robot episode setting, above). -1 also for n_push outside 0..HB_MAX_PUSHES, a
 * non-finite t_start / force / torque, a negative or non-finite duration. */
int hb_rollout_set_pushes(hb_ctx* ctx, int B, const hb_push_schedule* pushes);

/* ---- varied plants: a plant of its own for each robot of the episodes (payload on the base, ground contact, motor strength) ----
 * The variation acts on the simulated plant only; the planner, MPC, WBC, joint command law, actuation model and estimator keep the nominal
 * model and are not told about it. With s the variation of an instance, its plant step differs from hb_sim_step_batch in:
 *  - ground contact: k = sim.ground_stiffness * s.stiffness_scale, d = sim.ground_damping * s.damping_scale and
 *    mu = sim.friction_mu * s.friction_scale, each product formed once and used where the unvaried step uses the parameter (tangential
 *    damping is not varied);
 *  - motors: joint j receives the generalised force s.motor_strength[j] * tau[j], after the episode's saturation (hb_rollout_stats'
 *    max_abs_torque counts the saturated command, before this scaling);
 *  - payload (when payload_mass > 0): a rigid body fixed to the base, mass m, CoM c and inertia I_c (base frame). With the base coordinates
 *    (p, zyx), omega = T(zyx) zyx_dot, r = R(zyx) c and I_w = R I_c R': column k < 6 of M gains [F; T' n], the payload wrench about the
 *    base origin for a unit acceleration of coordinate k with v = 0 and no gravity (F = m (pdd + omega_dot x r), n = I_w omega_dot + r x F);
 *    nle gains the same for the actual velocity with no acceleration and gravity on: omega_dot0 = (omega_1 x a_pitch) dpitch +
 *    (omega_2 x a_roll) droll (the velocity-product term of the base's angular acceleration), F = m (omega_dot0 x r + omega x (omega x r))
 *    + m g e_z, n = I_w omega_dot0 + omega x I_w omega + r x F. Joint columns are unchanged.
 * The default variation (hb_default_plant_variation: no payload, every scale 1) is the unvaried plant bit for bit, as is an instance with no
 * variation set. */
typedef struct {                 /* the plant of one robot, relative to hb_sim_params and the nominal model            */
  double payload_mass;           /* [kg], >= 0; 0 = no payload (then payload_com and payload_inertia must be all zero) */
  double payload_com[3];         /* payload CoM in the base frame [m], relative to the base frame origin (rbd[3:6])  */
  double payload_inertia[9];     /* about the payload CoM, base frame, row-major, symmetric positive semidefinite     */
  double friction_scale;         /* mu = friction_scale * sim.friction_mu, >= 0                                       */
  double stiffness_scale;        /* ground_stiffness scaled, > 0                                                      */
  double damping_scale;          /* ground_damping scaled, >= 0                                                       */
  double motor_strength[10];     /* joint j receives motor_strength[j] * tau[j], >= 0 (0 = a dead motor)              */
} hb_plant_variation;            /* 208 B */
int hb_default_plant_variation(hb_plant_variation* v);      /* host only: no payload, every scale 1 */
/* Sets the plant variations of the context's episodes (a per-robot episode setting, above). -1 also for a field outside its range above:
 * any non-finite value, an inertia that is not exactly symmetric or has a negative principal minor (Sylvester's criterion, in double), a
 * zero mass with a nonzero CoM or inertia. */
int hb_rollout_set_plant_variations(hb_ctx* ctx, int B, const hb_plant_variation* v);

/* ---- link variations: each robot's own bodies in the episodes (link masses, centres of mass and inertias) ----
 * Like a plant variation, the setting acts on the simulated plant only; the planner, MPC, WBC, joint command law, actuation model and
 * estimator keep the nominal model and are not told about it. Record i acts on instance i of both episode calls; instances at or beyond B
 * run the nominal bodies bit for bit. The bodies are those of the model (HB_NBODY = 11): 0 is the base with the imu merged in, 1-5 are
 * leg_l1 .. leg_l5 and 6-10 leg_r1 .. leg_r5, l5 and r5 carrying their welded toe and heel bodies. With r the record of an instance and
 * m_b, c_b, I_b the model's mass, CoM (body frame) and rotational inertia about the CoM (body frame) of body b, the plant's body b has
 *   m' = mass_scale[b] m_b,   c' = c_b + com_shift[b],   I' = inertia_scale[b] I_b (every entry),
 * each value formed once, as one rounded product or sum, so that scale 1 and shift 0 give the nominal value exactly. These values enter
 * every rigid-body term of the plant's dynamics: the 16 columns of M(q) and nle(q, v). The kinematics (contact points, J_c), the armature,
 * the joint damping, the contacts, the wrench path and a plant variation's payload (which adds on top) are unchanged.
 * hb_default_link_variation's record (every scale 1, every shift 0) is the unvaried plant bit for bit, as is an instance with no record.
 * The setting has no state of its own (hb_episode_state_bytes does not count it) and adds no launch to an episode: the plant kernel forms
 * a varied instance's bodies once per step and reads the model's for the others, and for a record whose bodies all equal the model's. Every other entry point ignores it; hb_sim_step_links
 * takes records explicitly. */
typedef struct {                 /* the bodies of one robot, relative to the nominal model                                        */
  double mass_scale[11];         /* m' = mass_scale[b] m_b, finite, > 0                                                            */
  double com_shift[11][3];       /* c' = c_b + com_shift[b], body frame [m], finite                                                */
  double inertia_scale[11];      /* I' = inertia_scale[b] I_b, finite, > 0                                                         */
} hb_link_variation;             /* 440 B */
#define HB_SETTING_LINK_VARIATIONS 13         /* hb_link_variation for hb_rollout_set_link_variations (hb_check_setting_records)     */
#define HB_SETTING_HEIGHT_MAPS 14             /* hb_terrain for hb_plan_set_maps (hb_check_setting_records), the rules of _TERRAINS  */
#define HB_SETTING_ESTIMATOR_MAPS 15          /* hb_terrain for hb_estimator_set_maps (hb_check_setting_records), as _TERRAINS      */
#define HB_SETTING_MPC_MAPS 17                /* hb_terrain for hb_mpc_set_maps (hb_check_setting_records), as _TERRAINS; 16 unused */
#define HB_SETTING_WBC_MAPS 18                /* hb_terrain for hb_wbc_set_maps (hb_check_setting_records), as _TERRAINS            */
#define HB_SETTING_MPC_CONE_MAPS 19           /* hb_terrain for hb_mpc_set_cone_maps (hb_check_setting_records), as _TERRAINS       */
int hb_default_link_variation(hb_link_variation* r);      /* host only: every scale 1, every shift 0 */
/* Sets the link variations of the context's episodes (a per-robot episode setting, above). -1 also for a value that is not finite, a
 * mass_scale <= 0 or an inertia_scale <= 0. */
int hb_rollout_set_link_variations(hb_ctx* ctx, int B, const hb_link_variation* r);

/* ---- joint models: each robot's joint range stops and friction loss in the episodes' plant ----
 * The reference's plants give every leg joint a range and a friction loss: mujoco/model/hunter/hunter.xml:59-124 (range, which MuJoCo 3's
 * autolimits makes a limit constraint, and frictionloss="0.2") and legged_hunter_description/urdf/hunter_sim.urdf (<limit lower upper>,
 * enforced by Gazebo's ODE, and <dynamics friction="0.2">). A joint model adds both to the simulated plant, per robot. Like a link
 * variation it acts on the plant only: the planner, MPC, WBC, joint command law, actuation model, estimator and the emergency-stop check
 * keep their behaviour and are not told about it. Record i acts on instance i of both episode calls; instances at or beyond B, and
 * instances without a record, run the plant without these terms bit for bit.
 * For joint j (lanes 6-15 of the plant step, coordinate 6 + j) in each substep, at the substep's q_j and v_j, after the joint torque and
 * the viscous damping have been summed into the joint's right-hand side, s = tau_j - joint_damping v_j:
 *   (1) friction loss, when f_j != 0: s -= f_j clamp(v_j / v_s, -1, 1), regularised Coulomb friction (the bridged joints' motor torque
 *       takes the place of tau_j, and the term follows in the same place);
 *   (2) the contact Jacobian's forces and the wrench are added as without a record; joint_armature is added to the diagonal of M;
 *   (3) range stop, with m_jj the joint's diagonal entry of M + armature in this substep (a link variation's bodies included; a payload
 *       only changes the base block): past the upper end, r = q_j - upper_j > 0, s += min(0, -m_jj (k r + b v_j)); past the lower end,
 *       r = lower_j - q_j > 0, s += max(0, m_jj (k r - b v_j)). The stop never pulls a joint towards it (as the ground's normal force is
 *       clipped at 0). A joint at its bound exactly (r = 0) gets no stop term.
 * Then the step solves (M + A) qdd = rhs and integrates as before. A term whose condition is false is skipped, not added as zero, so a
 * record with every f_j = 0 and every bound infinite (any k, b) is the plant without a record bit for bit.
 * Stability rule: the plant integrates explicitly (semi-implicit Euler, h = sim.dt / sim.substeps), and the effective inertia of a joint is
 * at least joint_armature (the joint block's Schur complement of M + A is at least A). Each joint's total viscous gain must therefore
 * satisfy h (sim.joint_damping + f_j / v_s) <= sim.joint_armature. A plant step or an episode call whose sim params break this rule for
 * any record it reads returns -1 before any launch. The stop's gains are not part of the rule: they scale with m_jj.
 * Deviations from the reference's simulators: MuJoCo solves friction loss and limits as soft constraints in its solver, scaled by 1/A_jj of
 * the constraint's inverse inertia; here they are explicit penalty terms scaled by m_jj. No parity with MuJoCo's solver is claimed.
 * The setting has no state of its own (hb_episode_state_bytes does not count it) and adds no launch to an episode. */
typedef struct {                 /* the joints of one robot's plant                                                                */
  double friction_loss[10];      /* f_j [N m], finite, >= 0                                            (hunter.xml frictionloss: 0.2) */
  double friction_velocity;      /* v_s [rad/s], finite, > 0: the regularisation velocity                                          */
  double lower[10], upper[10];   /* stop range [rad], not NaN, lower < upper; -inf / +inf: no stop on that side                     */
  double stop_stiffness;         /* k [1/s^2], finite, >= 0                                                                        */
  double stop_damping;           /* b [1/s], finite, >= 0                                                                          */
} hb_joint_model;                /* 264 B */
#define HB_SETTING_JOINT_MODELS 21            /* hb_joint_model for hb_rollout_set_joint_models (hb_check_setting_records)          */
/* host only: f_j = 0.2 (hunter.xml, hunter_sim.urdf), v_s = 0.01 rad/s, the ranges HB_JOINT_LOWER / HB_JOINT_UPPER (those of hunter.xml
 * and hunter_sim.urdf), and k, b from MuJoCo's default solref (timeconst tc = 0.02, dampratio zeta = 1) and solimp (d_max = 0.95) past the
 * impedance width, where MuJoCo's reference acceleration is a_ref = -b v - k r with b = 2 / (d_max tc) and k = 1 / (d_max tc^2 zeta^2)
 * (MuJoCo documentation, Computation > Constraint model > Reference acceleration, and Modeling > Solver parameters): b = 105.26.. 1/s,
 * k = 2631.57.. 1/s^2. At hb_default_sim_params, h (1 + 0.2 / 0.01) = 0.0105 <= 0.1. */
int hb_default_joint_model(hb_joint_model* r);
/* Sets the joint models of the context's episodes (a per-robot episode setting, above). -1 also for a friction loss that is not finite
 * and >= 0, a friction_velocity that is not finite and > 0, a NaN bound, lower >= upper, a stop gain that is not finite and >= 0. The
 * stability rule above is checked by each episode call against its params. */
int hb_rollout_set_joint_models(hb_ctx* ctx, int B, const hb_joint_model* r);

/* ---- terrain: the ground under each robot of the episodes, a height field on a regular world-frame grid ----
 * The terrain acts on the simulated plant and on the height failure check only; the planner, MPC, WBC, joint command law, actuation
 * model and estimator keep assuming flat ground at z = 0 and are not told about it. The planner can be told where the ground is by a
 * height map (height maps, above; hb_plan_set_maps), the estimator's feet heights by an estimator map (estimator maps, above;
 * hb_estimator_set_maps), the MPC's stance feet by an MPC map (MPC maps, above; hb_mpc_set_maps), the WBC's friction pyramids by a
 * WBC map (WBC maps, above; hb_wbc_set_maps) and the MPC's friction cones by an MPC cone map (MPC cone maps, above;
 * hb_mpc_set_cone_maps), records of this type each set on its own.
 * Height and gradient at a world point (x, y): u = (x - origin[0]) / spacing clamped to [0, nx - 1], i = min(floor(u), nx - 2),
 * a = u - i; the same for y gives w, j and b. With lerp(p, q, s) = p + s (q - p): h0 = lerp(h[j][i], h[j][i+1], a),
 * h1 = lerp(h[j+1][i], h[j+1][i+1], a), h = lerp(h0, h1, b); g_x = lerp(h[j][i+1] - h[j][i], h[j+1][i+1] - h[j+1][i], b) / spacing,
 * g_y = (h1 - h0) / spacing. A coordinate that was clamped (u < 0 or u > nx - 1, likewise for y) has a zero gradient component, so the
 * edge heights continue outward as flat ground. A plateau (four equal corners) gives its height exactly.
 * Contact of each contact point p (velocity v) in each substep, with k, d and mu those of the instance (scaled by its plant variation):
 *  - flat path, g_x = g_y = 0 exactly: the flat-ground contact with h in place of sim.ground_height, the same expressions bit for bit;
 *  - sloped path otherwise: n = (-g_x, -g_y, 1) / L, L = sqrt(1 + g_x^2 + g_y^2), depth = (h - p_z) / L, active iff depth > 0;
 *    v_n = v.n, f_n = max(0, k depth - d v_n), v_t = v - v_n n, f_t = -sim.tangential_damping v_t scaled down to length mu f_n when it
 *    is longer, F = f_n n + f_t.
 *  contact_flag is 1 iff f_n > 0 (on the flat path: F_z > 0, as without a terrain).
 * Failure check: for an instance with a terrain, HB_ROLLOUT_FAIL_HEIGHT tests base z - h(base x, base y) < min_base_height on a finite
 * state; instances without one keep the absolute test. Friction is viscous only: on a slope of angle theta a standing robot creeps at
 * about m g sin(theta) / (n_contacts tangential_damping). Terrains add no launch to an episode. */
#define HB_TERRAIN_MAX 64
typedef struct {                      /* the ground under one robot: a height field on a regular world-frame grid                 */
  int32_t nx, ny;                     /* samples along world x and y, 2..HB_TERRAIN_MAX each                                       */
  double origin[2];                   /* world (x, y) of sample (0, 0) [m]                                                         */
  double spacing;                     /* sample spacing [m], > 0                                                                   */
  double height[HB_TERRAIN_MAX][HB_TERRAIN_MAX];  /* height[j][i] = ground z at (origin[0] + i spacing, origin[1] + j spacing);
                                         only j < ny, i < nx are read                                                              */
} hb_terrain;                         /* 32 800 B */
/* Sets the terrains of the context's episodes (a per-robot episode setting, above; the device copy takes 33.6 MB at 1024). -1 also for
 * nx or ny outside 2..HB_TERRAIN_MAX, a non-finite origin, a spacing that is not finite and > 0, a non-finite height among the used
 * samples. */
int hb_rollout_set_terrains(hb_ctx* ctx, int B, const hb_terrain* t);

/* ---- goals: a schedule of goal poses per robot, the reference's /move_base_simple/goal command (goalToTargetTrajectories) ----
 * Which goal is in force: on an MPC tick at time t, goal j is in force when j is the last index with time[j] <= t.
 * Capture: when the goal in force differs from the one the instance last captured, that tick builds the target once,
 * hb_goal_to_target(t, x0, goal[j]), with x0 the tick's plan-input state (the true state, or in estimated episodes the estimate with
 * x0[9] = yaw_obs), and the instance captures it. This is the publisher's behaviour: it converts a goal once, on the observation it
 * holds when the goal arrives.
 * Later MPC ticks plan on the captured target until another goal comes into force (the swing planner still reads the command's cmd_vel,
 * as the reference reads /cmd_vel_filtered apart from the target). Before its first goal an instance plans on its cmd_vel target.
 * The captured target and goal index are per-instance context state, like the planner's latest stance positions: they are cleared by an
 * episode call with tick0 == 0 and by every hb_rollout_set_goals call, so a split episode continues exactly. An instance without goals
 * (n_goal == 0, or at or beyond B) runs exactly as with no goals set. Goals add no launch to an episode. */
#define HB_MAX_GOALS 8
typedef struct {                      /* the goal poses of one robot                                                          */
  int32_t n_goal;                     /* 0..HB_MAX_GOALS                                                                       */
  double time[HB_MAX_GOALS];          /* absolute time [s] the goal is given, ascending                                        */
  double goal[HB_MAX_GOALS][3];       /* world x, y [m] and yaw [rad], the yaw in the unwrapped convention of x[9]             */
} hb_goal_schedule;
/* Sets the goal schedules of the context's episodes (a per-robot episode setting, above) and clears every captured goal. -1 also for
 * n_goal outside 0..HB_MAX_GOALS, a non-finite time or goal entry, times that descend. */
int hb_rollout_set_goals(hb_ctx* ctx, int B, const hb_goal_schedule* goals);

/* ---- MPC latency: the solve time of each robot's MPC cycle, as the MRT interface of the reference sees it (MPC_MRT_Interface) ----
 * An instance with latency d >= 1 ticks tracks its own adopted policy: a copy of the resident solution (solve time, node times, interval
 * count, state / input trajectories, node modes). Every MPC cycle still writes the resident solution, which stays the solver's warm start.
 * Adoption (MPC_MRT_Interface::updatePolicy): on absolute tick a, before that tick's MPC cycle, the instance adopts the resident solution
 * iff a >= d and (a - d) % mpc_every == 0, so the solution of the cycle at tick c comes into force at tick c + d (with d == mpc_every, just
 * before the next cycle overwrites it). On the cold tick (tick0 == 0, first tick of the call) every instance with d >= 1 adopts right after
 * the cycle, so the controller starts with a policy (the reference shows its stance override until the first solve; a deviation).
 * The policy evaluation of every tick, and the WBC, joint command law and fallback after it, read the adopted policy for d >= 1 and the
 * resident solution for d == 0; the joint command law takes its planned contact from the adopted policy's mode (the reference reads the
 * reference manager's newest schedule there; a deviation). The plan inputs, the planner, the warm start, the estimator's contact flags
 * and goal capture read the newest plan, as the reference's reference manager does.
 * The adopted policy is per-instance context state like the captured goals, so a split episode continues exactly; the resident
 * snapshots (hb_resident_read_batch / hb_resident_write_batch) do not include it, the episode snapshots (hb_episode_save_async, below)
 * do. Range: 0 <= d <= mpc_every; an episode call whose setting has an
 * entry above its mpc_every returns -1 before any launch, and so does a warm call (tick0 > 0) in which an instance with d >= 1 has never
 * adopted a policy. With no setting, or every latency 0, the episode calls issue exactly the launches they issue without one; with a
 * latency set they add one launch on each tick where an instance within the setting adopts, and one on the cold tick. */
/* Sets the MPC latencies of the context's episodes, ticks[i] for instance i (a per-robot episode setting, above; instances at or beyond B
 * run with latency 0). -1 also for a negative entry. */
int hb_rollout_set_mpc_latencies(hb_ctx* ctx, int B, const int32_t* ticks);

/* ---- odometry: a simulated tracking camera per robot, fused into the estimate (KalmanFilterEstimate::updateFromTopic) ----
 * Only the estimated episodes read this setting; hb_rollout_batch_dev has no estimator and ignores it. An instance with period_ticks == 0,
 * or at or beyond B, has no camera and runs exactly as with no setting.
 * The camera of instance i at absolute tick a, in the tick's sensor read: at a == 0 its state (position history and bias) is cleared;
 * the true base position entering the tick (rbd[3:6]) is recorded in history slot a % (HB_ODOM_MAX_DELAY + 1); a message is due iff
 * a % period_ticks == 0 and a >= delay_ticks, and then bias += sigma_drift n_d and pos = p(a - delay_ticks) + bias + sigma_position n_p,
 * each of the two terms added in that order. The normals are the sensor noise's Philox4x32-10 scheme (hb_sensor_noise, below): key
 * hb_sensor_noise.seed, counter (block, tick, noise_stream), 3 normals of block 9 for n_d and of block 10 for n_p (blocks 0-8 are the
 * sensors'); a sigma of 0 draws nothing. The history and bias are per-instance context state, allocated at max_batch by the first call that
 * sets records, freed by hb_destroy and cleared by every such call and by a read at tick 0, so a split episode continues exactly, also
 * between a reading and its delayed arrival.
 * The fusion (updateFromTopic), after the filter's predict / correct step and its xy decoupling, on a tick with a message:
 * x_hat[0:3] = pos; for each contact c, x_hat[6+3c : 9+3c] = pos + fk_c and then x_hat[8+3c] -= foot_radius, with fk_c the contact
 * position at the filter's ZYX angles and joint readings with the base at the origin (the filter's own kinematics), and feet_heights[c] =
 * x_hat[8+3c] where contact_flag[c]; the velocity x_hat[3:6] and P are left untouched. The estimated rbd then takes pos as its position,
 * and everything downstream (est_stats, est_log, yaw_obs, planner, MPC, WBC, joint law, goal capture) sees the fused estimate. Once
 * messages arrive, the filter's feet heights follow the camera instead of staying 0, as in the reference.
 * Deviations from the reference: the camera is mounted at the base frame origin (base2sensor = identity: the robot's URDF has no camera
 * link, and the tf lookup by stamp is not modelled); world2odom is the identity, which the reference never changes; messages arrive on whole
 * ticks; the message's orientation is not used (with an identity mount the reference does not use it either). Pinocchio's kinematics at
 * (pos, zyx, q) is restated as pos + fk_c: the same value, rounded as one more addition per coordinate.
 * Odometry adds no launch to an episode. */
#define HB_ODOM_MAX_DELAY 15
typedef struct {            /* the tracking camera of one robot                                                                     */
  int32_t period_ticks;     /* a message every period_ticks ticks, >= 0; 0 = no camera (the instance runs as with no setting)      */
  int32_t delay_ticks;      /* 0..HB_ODOM_MAX_DELAY: a message carries the pose of delay_ticks ticks earlier                        */
  double sigma_position;    /* white noise per message and axis [m], >= 0                                                           */
  double sigma_drift;       /* random-walk increment of the camera's bias per message and axis [m], >= 0                            */
} hb_odometry_setting;
/* Sets the tracking cameras of the context's estimated episodes (a per-robot episode setting, above) and clears every camera's state. -1
 * also for a negative period_ticks or delay_ticks, a delay_ticks above HB_ODOM_MAX_DELAY, or a sigma that is negative or not finite. */
int hb_rollout_set_odometry(hb_ctx* ctx, int B, const hb_odometry_setting* s);

/* ---- controller settings: the controller's run-time tuning per robot (the WBC block of task.info, WbcBase::setKpKd, and the joint PD
 * gains of LeggedController's dynamic_reconfigure, LeggedController.cpp:433-447) ----
 * Record i acts on instance i of both episode calls: its wbc replaces the context's WBC settings (hb_wbc_set_settings, hb_wbc_set_kp_kd,
 * hb_load_task_info) in the tick's WBC under both formulations (the three weights act only under HB_WBC_WEIGHTED, as the context's do), and
 * its gains replace p->gains in the joint command law (the episodes run the loaded branch: kp_position / kd_position are carried and read
 * by nothing, as those of p->gains). Instances at or beyond B keep the context's settings and p->gains, bit for bit as with no setting.
 * Every other entry point ignores this setting: the control step, the resident cycle and tick, hb_wbc_solve_batch, hb_hierarchical_wbc_*,
 * hb_joint_command_batch, hb_policy_wbc and the adapters run the context's settings and the gains they are given.
 * The setting adds no launch to an episode; the fused WBC kernels and the joint command law read the record of their own instance. */
typedef struct {
  hb_wbc_settings wbc;   /* in place of the context's WBC settings, for this robot */
  hb_pd_gains gains;     /* in place of hb_rollout_params.gains, for this robot     */
} hb_controller_setting;
/* Sets the controller settings of the context's episodes (a per-robot episode setting, above). -1 also for a field that is not finite, or
 * for a record hb_wbc_set_settings would reject (a torque limit, friction_coefficient, weight_swing_leg or weight_base_accel <= 0,
 * weight_contact_force < 0), a negative WBC task kp / kd, or a negative PD gain. */
int hb_rollout_set_controller_settings(hb_ctx* ctx, int B, const hb_controller_setting* s);

/* ---- simulated hardware: each robot's actuators and sensors between the controller and the plant (LeggedHWSim) ----
 * Like a plant variation, the setting acts on the simulated robot only; the planner, MPC, WBC, joint command law and estimator are not
 * told about it. Record i acts on instance i of the episodes; instances at or beyond B run the call's values, bit for bit as with no
 * setting. With r the record of an instance:
 *  - actuation: the actuation model's drop rule (hb_actuation_batch_dev) runs with r.actuation_delay in place of p->actuation_delay: the
 *    oldest entries with stamp + delay < t are dropped, and the oldest remaining one is applied. Everything else about the ring is unchanged,
 *    so a delay of HB_ACT_CAPACITY - 1 periods or more applies the oldest entry of the full ring (the ring holds HB_ACT_CAPACITY commands), as
 *    a per-call delay does.
 *  - saturation: the applied torque of joint j is clipped to +-r.torque_limit[j] in place of p->torque_limit[j]; hb_rollout_stats'
 *    max_abs_torque counts the clipped value, before a plant variation's motor_strength.
 *  - sensors (hb_rollout_estimated_batch_dev only): each reading is formed as (1) the true value, as hb_sim_read_sensors_batch_dev forms it;
 *    (2) plus its offset; (3) plus sigma x its Philox normals, with r's sigma in place of the call's hb_sensor_noise sigma of that channel,
 *    and the call's seed, the instance's noise_stream and the same blocks. The offsets: orientation_offset is added to the ZYX angles
 *    before the quaternion is formed; gyro_bias to R' omega_world; accel_bias to R' (a_world + (0, 0, 9.81)); encoder_offset to q_j; the
 *    joint velocities get none. An offset entry equal to 0.0 (either sign) adds nothing, so a reading of -0.0 stays -0.0 and a record with
 *    zero offsets reads bit for bit what the call's values read. The tracking camera (odometry) is unchanged.
 * hb_rollout_batch_dev has no sensors and reads only the delay and the limits. Every other entry point ignores this setting: the control
 * step, the resident cycle and tick, hb_actuation_batch(_dev), hb_sim_read_sensors(_batch_dev) and the adapters; hb_actuation_hw and
 * hb_sim_read_sensors_hw take records explicitly. The setting adds no launch to an episode: the actuation, saturation and sensor kernels
 * that run every tick read the record of their own instance. hb_default_hardware_setting's record, with the noise sigmas of the call,
 * reproduces the unset episode bit for bit. */
typedef struct {                 /* the simulated hardware of one robot (LeggedHWSim), which the controllers are not told about */
  double actuation_delay;        /* [s], finite, >= 0: in place of hb_rollout_params.actuation_delay                       */
  double torque_limit[10];       /* [N m], finite, > 0: in place of hb_rollout_params.torque_limit                          */
  double sigma_orientation, sigma_angular_velocity, sigma_linear_acceleration,
         sigma_joint_position, sigma_joint_velocity;   /* finite, >= 0: in place of the call's hb_sensor_noise sigmas (its seed stays the key) */
  double orientation_offset[3];  /* IMU mounting error on the ZYX angles [rad]                                             */
  double gyro_bias[3];           /* body frame [rad/s]                                                                      */
  double accel_bias[3];          /* body frame [m/s^2]                                                                      */
  double encoder_offset[10];     /* joint zero offsets [rad]                                                                */
} hb_hardware_setting;           /* 280 B */
/* host only: actuation_delay 0.009 s and torque_limit HB_WBC_TORQUE_LIMITS per leg (hb_default_rollout_params' values), every sigma and
 * offset 0 */
int hb_default_hardware_setting(hb_hardware_setting* s);
/* Sets the simulated hardware of the context's episodes (a per-robot episode setting, above). -1 also for a field that is not finite, a
 * negative actuation_delay, a torque_limit <= 0 or a negative sigma. */
int hb_rollout_set_hardware(hb_ctx* ctx, int B, const hb_hardware_setting* s);

/* ---- motor bridge: each robot's joint path through the real Hunter's driver (legged_bridge_hw) in place of LeggedHWSim's torque law ----
 * Like the hardware setting, it acts on the simulated robot only; the planner, MPC, WBC, joint command law and estimator are not told
 * about it. Record i acts on instance i of the episodes; instances at or beyond B run the unbridged path bit for bit. The bridge has no
 * state of its own (hb_episode_state_bytes does not count it). With r the record of an instance, joint j:
 *  - command (BridgeHW::write, BridgeHW.cpp:67-88, then the motor protocol, motor_control.c:146-225): the actuation model's drop rule is
 *    unchanged (the hardware record's delay included); the oldest remaining entry (posDes, velDes, kp, kd, ff) is mapped to the motor frame
 *    in double: kp_m = s kp, kd_m = s kd, pos_m = d posDes + z, vel_m = d velDes, ff_m = (s ff) d, with s = command_scale[j],
 *    d = direction[j], z = zero[j]. Each is clamped to its range: kp_m to [0, kp_max], kd_m to [0, kd_max], pos_m, vel_m and ff_m to
 *    +-pos_max, +-vel_max, +-ff_max. With quantise = 1 each is first rounded to float32, clamped in float32, encoded as the protocol does,
 *    code = (int)((x - min) * (2^bits - 1) / span), truncated, with 12 / 9 / 16 / 12 / 12 bits for kp / kd / pos / vel / ff, and decoded
 *    as (float)code * span / (2^bits - 1) + min, every float32 operation rounded on its own (span = max - min in float32). Deviation: the
 *    firmware's decode is not public; it is assumed to be the map the driver uses for feedback. A NaN value encodes as code 0 (what a
 *    float-to-int truncation on the GPU gives); +-inf clamps to the range's end. With quantise = 0 the values are clamped in double and
 *    neither rounded nor encoded (a NaN stays NaN).
 *  - motor PD (on the motor, at its own rate): on every plant substep, the joint receives tau = d (kp_m (pos_m - (d q + z)) + kd_m
 *    (vel_m - d qd) + ff_m) with that substep's q, qd: the same PD law as the unbridged actuation, evaluated in the motor frame. Deviation:
 *    the driver's loop runs at the plant's substep rate (sim.dt / sim.substeps, 2 kHz by default). tau is clipped to the instance's torque
 *    limit (the hardware record's, or hb_rollout_params.torque_limit) and then scaled by a plant variation's motor_strength, as unbridged.
 *    The episode's saturation step does not act on the instance: the plant clips. The applied torque that HB_CHANNEL_TORQUE records and
 *    hb_rollout_stats.max_abs_torque counts is the mean over the tick's substeps of the clipped tau, before motor_strength.
 *  - encoders (hb_rollout_estimated_batch_dev only; motor_control.c:484-500, BridgeHW.cpp:35-43): the joint readings are formed as (1) the
 *    true q, qd; (2) plus the hardware record's encoder offset and the noise, as unbridged; (3) to the motor frame, d q + z and d qd; (4)
 *    clamped to +-pos_max / +-vel_max and, with quantise = 1, rounded to float32, encoded in 16 / 12 bits and decoded as above; (5) back to
 *    the joint frame, (p - z) d: in float32 with quantise = 1 (the driver's values are float32), in double without. Deviation: no current
 *    or torque feedback, which nothing in the episode loop reads.
 * A record with scale 1, directions +-1, zero 0, quantise 0 and ranges that never bind, on a plant with one substep, gives the unbridged
 * episode bit for bit. hb_rollout_batch_dev has no sensors and reads only the command side. The setting adds no launch to an episode:
 * the actuation, plant and sensor kernels that run every tick read the record of their own instance. Every other entry point ignores it;
 * hb_actuation_bridge, hb_sim_step_bridge and hb_sim_read_sensors_bridge take records explicitly. */
typedef struct {                 /* one robot's joint path through legged_bridge_hw, which the controllers are not told about   */
  double command_scale[10];      /* multiplies kp, kd and ff, >= 0 (BridgeHW.cpp:74-85: 0.7 on joints 0, 1, 5, 6; 1 elsewhere)    */
  int32_t direction[10];         /* +1 or -1: motor angle = direction * q + zero (BridgeHW.h:118)                                */
  double zero[10];               /* motor angle of joint angle 0 [rad] (baseMotor_, BridgeHW.h:120: 0)                           */
  double kp_max[10];             /* protocol range of kp: [0, kp_max], > 0 (motor_control.c:11-35: 500)                          */
  double kd_max[10];             /* [0, kd_max], > 0 (5)                                                                         */
  double pos_max[10];            /* +-pos_max [rad], > 0 (12.5)                                                                  */
  double vel_max[10];            /* +-vel_max [rad/s], > 0 (18)                                                                  */
  double ff_max[10];             /* +-ff_max [N m], > 0 (30 on X motors, 90 on D motors: joints 2, 3, 7, 8, transmit.cpp:434-500) */
  int32_t quantise;              /* 1: the protocol's float32 codes; 0: clamps only, in double                                  */
} hb_motor_bridge;               /* 608 B */
/* host only: the reference's record: the scales, directions and zeros above, each joint's X or D motor ranges, quantise = 1 */
int hb_default_motor_bridge(hb_motor_bridge* r);
/* Sets the motor bridges of the context's episodes (a per-robot episode setting, above). -1 also for a direction other than +-1, a
 * non-finite value, a negative command_scale, a maximum <= 0, or quantise outside {0, 1}. */
int hb_rollout_set_motor_bridge(hb_ctx* ctx, int B, const hb_motor_bridge* r);
/* The bridge's codec on the host, the same functions the kernels run (host only, no context, no GPU): hb_motor_bridge_encode maps
 * command (B x 10 x 5, joint frame, as hb_joint_command_batch writes it) to the decoded motor command out (B x 10 x 5: pos_m, vel_m,
 * kp_m, kd_m, ff_m in the motor frame) of records r (B); hb_motor_bridge_feedback maps joint readings q, qd (B x 10) through steps (3) to
 * (5) of the encoders to q_out, qd_out. -1: B < 0, a NULL pointer with B > 0, or a record hb_rollout_set_motor_bridge rejects. */
int hb_motor_bridge_encode(int B, const hb_motor_bridge* r, const double* command, double* out);
int hb_motor_bridge_feedback(int B, const hb_motor_bridge* r, const double* q, const double* qd, double* q_out, double* qd_out);

/* ---- teleoperation: each robot driven as the joystick drives the reference (joy_teleop.launch, TargetTrajectoriesPublisher) ----
 * The operator's velocity command reaches the robot as /cmd_vel messages at the teleop rate while the deadman button is held, and the
 * publisher limits the change per message and converts each message once into a target. Record i acts on instance i of both episode
 * calls; instances at or beyond B run without it: the cmd_vel segment in force, and the cmd_vel target rebuilt on every MPC tick.
 * Messages: instance i receives a message on absolute MPC tick a iff on_tick[w] <= a < off_tick[w] and (a - on_tick[w]) % period_ticks
 * == 0 for some window w < n_window. An episode call returns -1 before any launch when a record's period_ticks or any on_tick[w] is not a
 * multiple of its mpc_every, so messages fall on MPC ticks only.
 * Publisher step (TargetTrajectoriesPublisher.h:97-131), on each message with cmd the cmd_vel segment in force at t: for k = vx, vy, yaw
 * rate in that order, d = cmd[k] - last[k], d = d > 0 ? min(d, change_limit) : max(d, -change_limit), last[k] += d; last[vz] = 0; then the
 * target is hb_cmd_vel_to_target(t, x0, last) with x0 the tick's plan-input state (the true state, or in estimated episodes the estimate
 * with x0[9] = yaw_obs), as goal capture uses it.
 * Planning: a teleoperated instance plans with cmd_vel = last (its swing planner's body velocity command, /cmd_vel_filtered) on its
 * captured target. Before its first message last = 0 and it plans on the cmd_vel target of last, rebuilt each MPC tick (deviation: the
 * reference's starting() target is the zero state). The latest message wins: the goal capture (goals, above) and the messages write one
 * captured target; on one tick the goal is captured first and the message second; a goal a message has replaced is not captured again;
 * outside the windows the last target stays in force, as when the operator lets go of the stick.
 * last, the goal last seen, the captured target and its source are per-instance context state: they are cleared by an episode call with
 * tick0 == 0 and by every hb_rollout_set_teleop call, the clearing call (B == 0) included, so a split episode continues exactly and no
 * message's target outlives the setting. hb_rollout_set_goals with schedules forgets the captured target and the goal last seen, and keeps
 * last: a teleoperated instance then captures the new goal in force as an instance without teleop does. Teleop adds no launch to an
 * episode.
 * Deviations: joy_node also publishes when an axis changes (coalesced to 50 ms), here messages come at the autorepeat rate only; the
 * reference drops messages while its observation time is 0, here the controller has published from tick 0. */
#define HB_MAX_TELEOP_WINDOWS 4
typedef struct {                              /* the joystick and the target publisher of one robot                                   */
  int32_t period_ticks;                       /* message period [ticks], >= 1 (50: autorepeat_rate 10 Hz at the 500 Hz tick)          */
  int32_t n_window;                           /* 0..HB_MAX_TELEOP_WINDOWS; 0: no message ever (the instance keeps last = 0)           */
  int32_t on_tick[HB_MAX_TELEOP_WINDOWS];     /* the deadman is held over absolute ticks [on_tick[w], off_tick[w]): on_tick >= 0,     */
  int32_t off_tick[HB_MAX_TELEOP_WINDOWS];    /* on_tick < off_tick, and off_tick[w] <= on_tick[w + 1] (ascending, not overlapping)   */
  double change_limit[3];                     /* per-message change of vx, vy [m/s] and yaw rate [rad/s], > 0; +inf: no limit         */
} hb_teleop_setting;                          /* 64 B */
#define HB_SETTING_TELEOP 12                  /* hb_teleop_setting for hb_rollout_set_teleop (hb_check_setting_records)                */
/* host only: period_ticks 50, one window [0, INT32_MAX), change_limit (0.1, 0.05, 0.3) (changeLimit_, TargetTrajectoriesPublisher.h:97) */
int hb_default_teleop_setting(hb_teleop_setting* s);
/* Sets the teleoperation of the context's episodes (a per-robot episode setting, above) and clears every instance's publisher state and
 * captured target (also with B == 0, once a setting has been made). -1 also for a period_ticks < 1, n_window outside 0..HB_MAX_TELEOP_WINDOWS, a window outside the rules above, or a
 * change_limit that is not > 0 (NaN). */
int hb_rollout_set_teleop(hb_ctx* ctx, int B, const hb_teleop_setting* s);

/* ---- estimated episodes (hb_rollout_estimated_batch_dev): the controllers read the Kalman filter's estimate from synthesised, noisy
 * sensors instead of the plant's true state (LeggedController::updateStateEstimation, LeggedController.cpp:280-349) ---- */
typedef struct {                 /* standard deviations of additive Gaussian sensor noise; 0 = that channel is exact and draws nothing */
  uint64_t seed;                 /* Philox4x32-10 key                                                                              */
  double orientation;            /* on each ZYX angle before the quaternion [rad]                                                  */
  double angular_velocity;       /* gyro, body frame [rad/s]                                                                       */
  double linear_acceleration;    /* accelerometer, body frame [m/s^2]                                                              */
  double joint_position, joint_velocity;   /* encoders [rad], [rad/s]                                                             */
} hb_sensor_noise;
typedef struct {
  hb_kf_params kf;               /* hb_default_kf_params, or hb_parse_task_info(...).kalman                                        */
  hb_sensor_noise noise;
} hb_estimation_params;
typedef struct {                 /* per instance, in/out, device memory for the episode call; hb_estimation_reset starts it       */
  hb_kf_state kf;
  uint64_t noise_stream;         /* Philox counter words 2-3: the instance's noise stream, independent of its batch position       */
  double base_vel_prev[3];       /* world base velocity at the last sensor read (accelerometer finite difference)                  */
  int32_t primed;                /* 0: no previous read, the accelerometer reads gravity only                                      */
  double yaw_obs;                /* unwrapped yaw handed to the MPC (currentObservation_.state(9))                                 */
  int32_t has_plan, n_events;    /* mode schedule of the latest plan (contact flags of the filter); has_plan = 0: all feet trusted */
  double event_times[HB_MAX_EVENTS];
  int32_t modes[HB_MAX_EVENTS + 1];
} hb_estimation_state;
typedef struct {                 /* per instance, in/out; counts while the instance has not failed (as hb_rollout_stats)            */
  double max_vel_err, max_height_err;          /* |v_hat - v| (world base linear velocity), |z_hat - z|, against the true state entering the tick */
  double sum_sq_vel_err, sum_sq_height_err;
  int32_t count;                               /* ticks counted                                                                  */
} hb_estimation_stats;
int hb_default_estimation_params(hb_estimation_params* p);  /* host only: default filter, no noise, seed 0 */
/* host only: x_hat = 0, P = 100 I, feet heights 0 (hb_kf_reset), noise_stream = first_stream + i, primed = has_plan = 0, yaw_obs = 0 */
int hb_estimation_reset(int B, uint64_t first_stream, hb_estimation_state* state);

int hb_default_kf_params(hb_kf_params* p);
/* x_hat = 0, P = 100 I, heights = 0 (KalmanFilterEstimate constructor, LinearKalmanFilter.cpp:24-63); host only */
int hb_kf_reset(int B, hb_kf_state* state);
int hb_default_pd_gains(hb_pd_gains* g);
int hb_default_config(hb_config* cfg);
int hb_create(const hb_config* cfg, int device, hb_ctx** out);
int hb_destroy(hb_ctx* ctx);
int hb_sync(hb_ctx* ctx);
const char* hb_strerror(int code);
/* text of the last CUDA runtime error seen by this context (diagnostics for return code -2) */
const char* hb_last_cuda_error(const hb_ctx* ctx);
/* number of kernel launches issued through this context since creation (bench.py reports it as gpu_launches) */
int64_t hb_launch_count(const hb_ctx* ctx);
/* bytes of reference data the last hb_resident_cycle_batch moved host -> device (only the used entries of hb_reference are uploaded) */
int64_t hb_last_reference_upload_bytes(const hb_ctx* ctx);
/* per-kernel device timing with CUDA events on the context's stream (used by bench.py for the roofline line):
 * kinds 0 = Riccati sweep, 1 = forward pass + line search, 2 = WBC assembly, 3 = interior-point QP, 4 = other,
 *       5 = node linearisation (kinematics), 6 = node LQ model + projection */
int hb_profile_enable(hb_ctx* ctx, int on);
int hb_profile_read(hb_ctx* ctx, double* ms_per_kind /*7*/, int64_t* count_per_kind /*7*/);
/* the context's CUDA stream as a cudaStream_t cast to void* (for event timing on the launching stream) */
void* hb_stream(hb_ctx* ctx);

/* ---- device-pointer (asynchronous) entry points ---- */
/* Batched dense QP, one problem per warp: min 1/2 x'(H + wbc_rho I) x + g'x  s.t.  lbA <= A x <= ubA, with 1 <= n <= 80 and 0 <= m <= 160
 * (HB_EINVAL otherwise). H (n x n, row-major, exactly symmetric: the residuals read all of it, the factorisation its lower triangle).
 * Rows: all-zero rows are dropped; |bound| >= 1e19 means no bound on that side; lbA == ubA (exactly) makes an equality row; a row with
 * two finite bounds lbA < ubA is two-sided. Row capacity: at most 32 equality rows and 96 one-sided entries, where a two-sided row
 * counts as two entries; zero rows and rows without finite bounds count towards neither.
 * status[i] (nullable): 0 solved; 1 iteration cap (qp_max_iter) reached, x = last iterate; 2 an all-zero row whose bounds exclude 0
 * (lbA > 1e-12 or ubA < -1e-12), or a failed factorisation; 3 non-finite iterate; 4 more rows than the capacity above.
 * With status 2 from a zero row and with status 4, x = 0 and iters = 0. iters[i] (nullable): interior-point iterations. */
int hb_wbc_qp_batch_dev(hb_ctx* ctx, int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA,
                        const double* ubA, double* x, int32_t* status, int32_t* iters);
int hb_wbc_solve_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                           const uint8_t* stance_mode, double* sol, int32_t* status);
/* WbcBase::formulate*Task + WeightedWbc::formulateConstraints / formulateWeightedTasks (legged_wbc/src/WbcBase.cpp:138-338,
 * WeightedWbc.cpp:68-94) in the layout WeightedWbc::update hands to qpOASES (WeightedWbc.cpp:24-42): H = A_w' A_w (38 x 38), g = -A_w' b_w,
 * A (60 rows allocated, m_rows[i] used, row-major 60 x 38), lbA / ubA (60, -1e20 = qpOASES -INFTY). Feeds the raw QP sweep
 * (BASELINE configs[4]) and the assembly parity test; the product path (hb_wbc_solve_batch) never materialises these matrices. */
int hb_wbc_assemble_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                              const uint8_t* stance_mode /*nullable*/, double* H, double* g, double* A, double* lbA, double* ubA,
                              int32_t* m_rows);
/* hb_wbc_qp_batch_dev with a per-problem row count: A / lbA / ubA are allocated with m_alloc rows, problem i uses its first m_rows[i] */
int hb_wbc_qp_rows_batch_dev(hb_ctx* ctx, int B, int n, int m_alloc, const int32_t* m_rows, const double* H, const double* g,
                             const double* A, const double* lbA, const double* ubA, double* x, int32_t* status, int32_t* iters);
/* HoQp cascade (legged_wbc/src/HoQp.cpp:21-198): x (B x 38, first n entries used) = solution of the lowest level (HoQp::getSolutions),
 * slack (B x 80, nullable) = stacked slack solutions in level order, status[i] = 0 or 10 * (QP status) + level of the first failing level */
int hb_hoqp_solve_batch_dev(hb_ctx* ctx, int B, const hb_hoqp_problem* problems, double* x, double* slack /*nullable*/, int32_t* status /*nullable*/);
/* legged::HierarchicalWbc::update (legged_wbc/src/HierarchicalWbc.cpp:18-31): task0 = floating-base EoM + torque limits + friction cone +
 * no contact motion, task1 = base acceleration, task2 = 0.1 * contact force + swing leg; sol (B x 38) = [qdd, F, tau]. One fused kernel per
 * call: the tasks never leave the chip and each level is solved at its own shape. status[i] as hb_hoqp_solve_batch_dev's, plus 21 / 22
 * when level 0 / 1 leaves more than 28 free variables to the next level (level 0 leaves at most 22 while its EoM rows have full rank). */
int hb_hierarchical_wbc_solve_batch_dev(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                                        double* sol, int32_t* status /*nullable*/);
int hb_mpc_cold_start_batch_dev(hb_ctx* ctx, int B, const double* x0, const int32_t* mode, double* x_traj, double* u_traj);
int hb_mpc_solve_batch_dev(hb_ctx* ctx, int B, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                           double* x_traj, double* u_traj, hb_solve_info* info);
/* ---- time discretisation with event nodes (SURVEY 8a row S1) ----
 * hb_time_grid_batch: node times (B x (horizon_N + 1)) and interval counts (B) of every instance from its mode-switch times
 * (hb_reference.event_times); status[i] = 1 when the capacity horizon_N was exhausted (last interval stretched to the final time).
 * The *_grid_* entry points are the grid-aware forms of their uniform counterparts: interval k of instance i has length
 * node_times[i][k+1] - node_times[i][k]; nodes beyond n_intervals[i] are ignored. */
int hb_time_grid_batch_dev(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* node_times, int32_t* n_intervals,
                           int32_t* status /*nullable*/);
int hb_reference_expand_grid_batch_dev(hb_ctx* ctx, int B, const double* node_times, const hb_reference* refs, double* x_ref, double* swing_ref,
                                       int32_t* mode);
int hb_mpc_solve_grid_batch_dev(hb_ctx* ctx, int B, const double* x0, const double* node_times, const int32_t* n_intervals, const double* x_ref,
                                const double* swing_ref, const int32_t* mode, double* x_traj, double* u_traj, hb_solve_info* info);
int hb_policy_eval_grid_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* node_times, const int32_t* n_intervals, const double* x_traj,
                                  const double* u_traj, const int32_t* mode, double* x_des, double* u_des, int32_t* mode_out);
int hb_policy_eval_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* x_traj, const double* u_traj, const int32_t* mode,
                             double* x_des, double* u_des, int32_t* mode_out);
int hb_control_step_batch_dev(hb_ctx* ctx, int B, double t_rel, const double* x0, const double* x_ref, const double* swing_ref,
                              const int32_t* mode, const double* rbd, double* x_traj, double* u_traj, hb_solve_info* info,
                              double* wbc_sol, double* torque, int32_t* wbc_status);
/* joint command law (LeggedController.cpp:186-257): posDes = q_mpc + 0.5 qdd dt^2, velDes = qd_mpc + qdd dt, gains by joint class
 * and planned contact state of the leg, feed-forward = WBC torque; joint-limit protection sets the per-instance emergency stop flag
 * (in/out) which turns the command into pure damping (0,0,0,1,0). loaded[i] = 0 selects the pre-load position hold (:211-222).
 * command: B x 10 x 5 = (posDes, velDes, kp, kd, ff) per joint; output_torque: B x 10 = ff + kp (posDes - q) + kd (velDes - qd). */
int hb_joint_command_batch_dev(hb_ctx* ctx, int B, const hb_pd_gains* gains, double period, const double* x_des, const double* u_des,
                               const double* wbc_sol, const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded, uint8_t* estop,
                               double* command, double* output_torque);
/* Resident closed-loop cycle: the context keeps the primal solution on the device like ocs2::SqpSolver keeps primalSolution_.
 * One call = reference expansion (hb_reference -> node grid) + warm start (previous solution interpolated on the new grid, tail from
 * the initializer; mpc.coldStart false, task.info:146 -- or the initializer everywhere when cold_start != 0) + one SQP iteration +
 * policy evaluation at t0 + t_rel + WeightedWbc + torque law. Only t0, x0, refs, rbd go in and info / wbc_sol / torque / status come
 * out; hb_resident_read_batch copies the resident trajectories out when the caller wants them (PrimalSolution). The WeightedWbc
 * fallback is applied on the device: an instance whose QP did not solve (wbc_status != 0) returns its previous solution and torques
 * (WeightedWbc.cpp:57-64) from the second cycle on. */
int hb_resident_cycle_batch_dev(hb_ctx* ctx, int B, int cold_start, double t_rel, const double* t0, const double* x0,
                                const hb_reference* refs, const double* rbd, hb_solve_info* info, double* wbc_sol, double* torque,
                                int32_t* wbc_status);
/* device planner (SURVEY 8f row N1): the same planner source as hb_plan_references, four cooperating threads per instance. feet != NULL
 * overrides in[i].feet_pos (B x 12, e.g. from hb_contact_positions_batch_dev); status[i] = 0, -1 or -5 like hb_plan_references. */
int hb_plan_references_batch_dev(hb_ctx* ctx, int B, const hb_plan_input* in, const double* feet, double* latest_stance,
                                 hb_reference* out, int32_t* status /*nullable*/);
/* Explicit planner targets of the context (hb_plan_references_targets on the device): while set, hb_plan_references_batch_dev,
 * hb_plan_references_gpu and hb_resident_plan_cycle_batch plan instance i < B on targets[i] instead of its cmd_vel target; instances at
 * or beyond B keep theirs. The episode calls do not read it (they take goals, hb_rollout_set_goals). Setting conventions of the
 * per-robot episode settings (below): host array validated and copied in stream order, B == 0 clears, -4 for B > max_batch, a rejected
 * call keeps the previous setting. -1 also for n outside 1..HB_MAX_TARGETS, times that are not strictly ascending, a non-finite
 * time[k] or state[k][.] with k < n. */
int hb_plan_set_targets(hb_ctx* ctx, int B, const hb_target* targets);
/* Planner settings of the context (hb_planner_settings, above): instance i < B of every device planner path -- hb_plan_references_batch_dev,
 * hb_plan_references_gpu, hb_resident_plan_cycle_batch, hb_rollout_batch_dev and hb_rollout_estimated_batch_dev -- plans with settings[i]
 * in place of the compiled-in templates and swing settings; instances at or beyond B, and every instance while none is set, plan with the
 * compiled-in values bit for bit (hb_default_planner_settings gives the same plans). One setting serves every path, so an episode can be
 * written as a loop of those calls. Setting conventions of the per-robot episode settings (below): host array validated and copied in
 * stream order, B == 0 clears (settings may be NULL), -1 also for a record that is not valid, -4 for B > max_batch, a rejected call keeps
 * the previous setting. The setting adds no launch to any call. */
int hb_plan_set_settings(hb_ctx* ctx, int B, const hb_planner_settings* settings);
/* Height maps of the context (height maps, above): instance i < B of every device planner path -- hb_plan_references_batch_dev,
 * hb_plan_references_gpu, hb_resident_plan_cycle_batch, hb_rollout_batch_dev and hb_rollout_estimated_batch_dev, the goal and teleop
 * captures of the episodes included -- plans on maps[i]; instances at or beyond B, and every instance while none is set, plan without a
 * map. The contract of hb_plan_set_settings: host array validated and copied in stream order, B == 0 clears (maps may be NULL), -1 for a
 * record hb_rollout_set_terrains rejects, -4 for B > max_batch, a rejected call keeps the previous setting, no launch added. Maps are a
 * setting, not episode state: snapshots do not hold them. */
int hb_plan_set_maps(hb_ctx* ctx, int B, const hb_terrain* maps);
/* Estimator maps of the context (estimator maps, above): instance i < B of every estimator path -- hb_estimator_update_batch_dev,
 * hb_estimator_update_batch and hb_rollout_estimated_batch_dev -- measures its feet heights on maps[i]; instances at or beyond B, and every
 * instance while none is set, run the filter without a map. One setting serves the public filter call and the episode, so an estimated
 * episode can be written as a loop of public calls. The contract of hb_plan_set_maps: host array validated and copied in stream order,
 * B == 0 clears (maps may be NULL), -1 for a record hb_rollout_set_terrains rejects, -4 for B > max_batch, a rejected call keeps the
 * previous setting, no launch added. Maps are a setting, not episode state: hb_episode_state_bytes and snapshots do not count them. */
int hb_estimator_set_maps(hb_ctx* ctx, int B, const hb_terrain* maps);
/* MPC maps of the context (MPC maps, above): instance i < B of every MPC path -- hb_mpc_solve_batch(_dev), hb_mpc_solve_grid_batch(_dev),
 * hb_control_step_batch(_dev), hb_resident_cycle_batch(_dev), hb_resident_plan_cycle_batch (the MRT split's solves included),
 * hb_rollout_batch_dev and hb_rollout_estimated_batch_dev -- holds its stance feet on maps[i]; instances at or beyond B, and every
 * instance while none is set, solve without a map. One setting serves every path, so an episode can be written as a loop of public
 * calls. The contract of hb_plan_set_maps: host array validated and copied in stream order, B == 0 clears (maps may be NULL), -1 for a
 * record hb_rollout_set_terrains rejects, -4 for B > max_batch, a rejected call keeps the previous setting. While a map is set, each solve
 * runs one more launch (the stance heights, once per solve); unset, the launches are those without the setting. Maps are a setting, not
 * episode state: hb_episode_state_bytes and snapshots do not count them. */
int hb_mpc_set_maps(hb_ctx* ctx, int B, const hb_terrain* maps);
/* WBC maps of the context (WBC maps, above): instance i < B of every WBC path -- hb_wbc_solve_batch(_dev), hb_wbc_assemble_batch(_dev),
 * hb_hierarchical_wbc_solve_batch(_dev), hb_hierarchical_wbc_tasks_batch, hb_control_step_batch(_dev), hb_resident_cycle_batch(_dev),
 * hb_resident_plan_cycle_batch, hb_resident_wbc_batch(_dev), hb_policy_wbc(_async), hb_rollout_batch_dev and hb_rollout_estimated_batch_dev
 * -- tilts its stance contacts' friction pyramids on maps[i]; instances at or beyond B, and every instance while none is set, keep the
 * flat pyramids. One setting serves every path, so an episode can be written as a loop of public calls. The contract of hb_plan_set_maps:
 * host array validated and copied in stream order, B == 0 clears (maps may be NULL), -1 for a record hb_rollout_set_terrains rejects, -4
 * for B > max_batch, a rejected call keeps the previous setting. No launch is added, set or not. Maps are a setting, not episode state:
 * hb_episode_state_bytes and snapshots do not count them. */
int hb_wbc_set_maps(hb_ctx* ctx, int B, const hb_terrain* maps);
/* MPC cone maps of the context (MPC cone maps, above): instance i < B of every MPC path -- the paths of hb_mpc_set_maps -- has its stance
 * contacts' friction cones about maps[i]'s surface frames; instances at or beyond B, and every instance while none is set, keep the cones
 * about world z. A setting of its own, apart from the MPC maps, so that either can be measured alone. The contract of hb_plan_set_maps:
 * host array validated and copied in stream order, B == 0 clears (maps may be NULL), -1 for a record hb_rollout_set_terrains rejects, -4
 * for B > max_batch, a rejected call keeps the previous setting. No launch is added, set or not. Maps are a setting, not episode state:
 * hb_episode_state_bytes and snapshots do not count them. */
int hb_mpc_set_cone_maps(hb_ctx* ctx, int B, const hb_terrain* maps);

/* ---- contact detection: the Kalman filter's contact flags from the momentum observer instead of the plan's schedule alone ----
 * Without it an estimated episode tells the filter the schedule's flags (LeggedController.cpp:296-304), which are wrong where a foot
 * lands late (a step down) or early (a step up). With a record r for an instance, each estimated tick runs StateEstimateBase::
 * estContactForce (the observer of hb_contact_force_estimate_batch) and replaces the schedule's flags by StateEstimateBase::estContactState
 * (StateEstimateBase.cpp:208-226), which the reference computes every input of and never calls. At time t with the schedule's flag
 * cmd[c] of contact c (ordered l_f1, r_f1, l_f2, r_f2, so c % 2 is the leg) and the run [s_c, e_c] of equal flags of c around t
 * (SwingTrajectoryPlanner::threadSaftyGetStartStopTime on the stored schedule: the phase of t, an event time belonging to the earlier
 * phase, clamped to n_events - 1; [t, t] without a plan or with a one-phase schedule), P = e_c - s_c and Fz = force[6 (c % 2) + 2] of
 * the last observer output:
 *   flag[c] = Fz > threshold   if !cmd[c] && t - s_c > swing_fraction P     (a swing foot late in its phase)
 *   flag[c] = Fz > threshold   if  cmd[c] && t - s_c < stance_fraction P    (a stance foot early in its phase)
 *   flag[c] = cmd[c]           otherwise.
 * Order of one estimated tick of an instance with a record: (1) the schedule's flags at the previous observation's time, as without the
 * setting; (2) the rule above at that time on the stored observer output; (3) the filter on the detected flags (the odometry fusion too);
 * (4) the observer on the filter's estimated rbd with the stored effort and dt = period, its output stored; (5) after the plant step the
 * tick's applied torque (what HB_CHANNEL_TORQUE records) is stored as the next tick's effort. The detected flags reach the filter only:
 * the planner, MPC and WBC read the schedule's flags, as the reference's do. */
typedef struct {                 /* one robot's contact detection                                                                   */
  double cutoff_frequency;       /* the observer's [rad/s], > 0 as hb_contact_force_estimate_batch takes it (cutoffFrequency: 250) */
  double threshold;              /* F_z above which a foot counts as loaded [N], finite (contactForceEsimation.contactThreshold: 75) */
  double swing_fraction;         /* share of a swing phase after which the force decides, in [0, 1] (0.75)                         */
  double stance_fraction;        /* share of a stance phase before which the force decides, in [0, 1] (0.25)                        */
} hb_contact_detection;          /* 32 B */
#define HB_SETTING_CONTACT_DETECTION 20   /* hb_contact_detection for hb_rollout_set_contact_detection (hb_check_setting_records)         */
/* host only: task's contactForceEsimation cutoff and threshold (task NULL: 250 and 75, hb_parse_task_info's defaults), fractions 0.75 and
 * 0.25 (StateEstimateBase.cpp:215-221). -1 for a NULL out. */
int hb_default_contact_detection(const hb_task_info* task /*nullable*/, hb_contact_detection* out);
/* Contact detection of the context's estimated episodes: record i acts on instance i of hb_rollout_estimated_batch_dev; instances at or
 * beyond B, hb_rollout_batch_dev and every other entry point run without it. The contract of a per-robot episode setting (above): -1 also
 * for a record outside its documented range, -4 for B > max_batch, a rejected call keeps the previous setting. Per-instance context state:
 * the observer's filtered momentum, its last output (16, 50 each before the first: StateEstimateBase.cpp:61-62), the effort (10) and the
 * flags the filter last used (4). Every call that is not rejected clears that state (B == 0 included), so a restore comes after it; an
 * episode call with tick0 == 0 clears it too. The state is part of a snapshot row while a setting is made, adding 344 bytes to
 * hb_episode_state_bytes; unset, the row keeps its size. While a setting is made, each estimated tick runs one more launch (the observer). */
int hb_rollout_set_contact_detection(hb_ctx* ctx, int B, const hb_contact_detection* records);
/* The detection rule alone, as the episode's step (2) runs it: for each instance i, flags[i] (B x 4, in: the schedule's, out: detected)
 * at time t on the schedule of est[i] (has_plan, n_events, event_times, modes) and the observer output est_force[i] (B x 16) with
 * records[i]; records NULL leaves the flags unchanged. hb_contact_state_estimate_async takes device pointers (records on the host), and
 * hb_contact_state_estimate host pointers. -1: B < 0, a NULL pointer other than records, a record the setter rejects; -4: B > max_batch. */
int hb_contact_state_estimate_async(hb_ctx* ctx, int B, double t, const hb_estimation_state* est, const double* est_force,
                                    const hb_contact_detection* records /*nullable*/, uint8_t* flags);
int hb_contact_state_estimate(hb_ctx* ctx, int B, double t, const hb_estimation_state* est, const double* est_force,
                              const hb_contact_detection* records /*nullable*/, uint8_t* flags);
/* The detection state of instances 0 .. B-1 of the context (host pointers): est_force (B x 16, nullable), the last observer output, and
 * flags (B x 4, nullable), the flags the filter last used; an instance beyond the setting reads the cleared state (50 each, flags 0).
 * -1: B < 0 or no setting made since the context was created; -4: B > max_batch. */
int hb_rollout_contact_estimates(hb_ctx* ctx, int B, double* est_force /*nullable*/, uint8_t* flags /*nullable*/);
/* The rule on the host, the body the kernels run (host only, no context, no GPU): phase_times (B x 4 x 2, nullable) receives [s_c, e_c];
 * flags as hb_contact_state_estimate. -1 as there, without the capacity. */
int hb_contact_state_host(int B, double t, const hb_estimation_state* est, const double* est_force, const hb_contact_detection* records /*nullable*/,
                          uint8_t* flags, double* phase_times /*nullable*/);

/* One estimator update per instance (StateEstimateBase::updateJointStates / updateImu, StateEstimateBase.cpp:73-106, then
 * KalmanFilterEstimate::update): quat = (x, y, z, w); contact_flag: B x 4 (0 = the filter distrusts that foot, x100 noise);
 * rbd_out: B x 32 measured rbd state [zyx, p, q_j, omega_world, v, qd_j]. zyxOffset_ is taken as zero. The odometry fusion
 * (updateFromTopic) is a call of its own, hb_estimator_fuse_odometry_async, applied after this one. Instance i measures its feet heights
 * on the context's estimator map i (hb_estimator_set_maps) when it has one, and on state[i].feet_heights otherwise. */
int hb_estimator_update_batch_dev(hb_ctx* ctx, int B, const hb_kf_params* params, double dt, hb_kf_state* state, const double* quat,
                                  const double* ang_vel_local, const double* lin_acc_local, const double* joint_pos,
                                  const double* joint_vel, const uint8_t* contact_flag, double* rbd_out);
/* StateEstimateBase::estContactForce (legged_estimation/src/StateEstimateBase.cpp:130-206): momentum-observer disturbance torque and the
 * least-norm 6-D wrench at the toe frame of each foot. cutoff_frequency = contactForceEsimation.cutoffFrequency (task.info:349, 250);
 * dt > 1 is replaced by 0.002 as in the reference. rbd: measured state (B x 32), tau_cmd: last commanded joint torques (B x 10).
 * est_contact_force (B x 16) = [wrench_left(6), wrench_right(6), |F_l|, |F_r|, |W_l|, |W_r|]; disturbance_torque (B x 16, nullable). */
int hb_contact_force_estimate_batch_dev(hb_ctx* ctx, int B, double cutoff_frequency, double dt, hb_observer_state* state, const double* rbd,
                                        const double* tau_cmd, double* est_contact_force, double* disturbance_torque /*nullable*/);
/* LeggedHWSim::writeSim (legged_gazebo/src/LeggedHWSim.cpp:166-192): command (B x 10 x 5 as written by hb_joint_command_batch) delayed by up to
 * `delay` seconds (legged_gazebo/config/default.yaml:2, 0.009), PD + feed-forward evaluated with the current joint state -> tau (B x 10) */
int hb_actuation_batch_dev(hb_ctx* ctx, int B, double delay, const double* time /*B*/, hb_actuation_state* state, const double* command,
                           const double* rbd, double* tau);
/* one control period of the batched plant: rbd (B x 32, [zyx, p, q_j, omega_world, v, qd_j]) advanced in place under the joint torques tau
 * (B x 10); contact_force (B x 12) and contact_flag (B x 4) of the last substep are optional outputs */
int hb_sim_step_batch_dev(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, double* contact_force /*nullable*/,
                          uint8_t* contact_flag /*nullable*/);
/* The 500 Hz half of LeggedController::update between two MPC solves (LeggedController.cpp:154-184): evaluatePolicy of the RESIDENT solution at
 * the absolute time t_now[i], WeightedWbc (with the previous-solution fallback), torque law. Outputs the desired state / input / mode too
 * (inputs of hb_joint_command_batch). */
int hb_resident_wbc_batch_dev(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode /*nullable*/, double* x_des,
                              double* u_des, int32_t* mode_out, double* wbc_sol, double* torque /*nullable*/, int32_t* wbc_status /*nullable*/);
/* n_ticks ticks of B closed-loop episodes (LeggedController::update on the batched plant). On a tick with (tick0 + k) % mpc_every == 0 an MPC
 * cycle runs first: plan inputs built on the device from rbd (x0 = hb_rbd_to_centroidal, t0 = t, cmd_vel of the command segment in force,
 * horizon = time_to_target = horizon_N * dt or, for event_nodes contexts, the time horizon, prev_event = min(t, gait_start) - 0.5, IK
 * joint references), device planner, resident cycle without its WBC (cold start iff tick0 == 0). Every tick then runs
 * hb_resident_wbc_batch's policy + WeightedWbc at t (the adopted policy's for instances with an MPC latency, hb_rollout_set_mpc_latencies),
 * the joint command law (loaded, walking branch), the actuation model, saturation to
 * +-torque_limit (each robot's own delay and limits when hb_rollout_set_hardware has set records) and one plant step (with the tick's push wrench when hb_rollout_set_pushes has set schedules, on the instance's plant
 * when hb_rollout_set_plant_variations has set variations, on its ground when hb_rollout_set_terrains has set terrains). Failure checks run on the state entering each tick (finite, |roll| <= pi/2, base height) and on the
 * emergency stop the joint command raises; from its first failure on an instance is held (rbd put back to its last finite state after
 * every plant step; a non-finite state entering the first tick of a call is replaced by the nominal standing pose) and its outputs no
 * longer count in stats. rbd (B x 32), act, estop (B) and stats are device memory, in/out. cmd (B) is a host array, validated and copied
 * to the context once per call; p is read on the host. log (device, nullable): rbd at the start of every log_every-th tick of the call,
 * B x ceil(n_ticks / log_every) x 32. Asynchronous: launches only, on the context's stream; per-call scratch is allocated at max_batch by
 * the first call and freed by hb_destroy. */
int hb_rollout_batch_dev(hb_ctx* ctx, int B, int64_t tick0, int n_ticks, const hb_rollout_params* p, const hb_rollout_command* cmd, double* rbd,
                         hb_actuation_state* act, uint8_t* estop, hb_rollout_stats* stats, double* log /*nullable*/);
/* The sensors of the simulated robot (LeggedHWSim::readSim, legged_gazebo/src/LeggedHWSim.cpp:116-130, and the joint encoders) read from the
 * true rbd at absolute tick `tick`, in the inputs hb_estimator_update_batch takes: quat (B x 4, x y z w) of the ZYX angles after noise on
 * the angles; ang_vel_local (B x 3) = R' omega_world; lin_acc_local (B x 3) = R' (a_world + (0, 0, 9.81)) with a_world = (v - base_vel_prev)
 * / accel_dt, or 0 on an unprimed instance; joint_pos / joint_vel (B x 10) = q_j, qd_j; each plus sigma x its Philox normals. est (B) is
 * read for noise_stream / base_vel_prev / primed and gets base_vel_prev = v, primed = 1. Device pointers, asynchronous. */
int hb_sim_read_sensors_batch_dev(hb_ctx* ctx, int B, const hb_sensor_noise* noise, int64_t tick, double accel_dt, const double* rbd,
                                  hb_estimation_state* est, double* quat, double* ang_vel_local, double* lin_acc_local, double* joint_pos,
                                  double* joint_vel);
/* hb_rollout_batch_dev with the controllers on the estimated state. Every tick, after the start-of-tick checks: sensors from the true rbd
 * (hb_sim_read_sensors_batch_dev, accel_dt = p->sim.dt) and the filter's contact flags from the stored mode schedule at (tick - 1) * period
 * (all 1 before the first plan), hb_estimator_update at dt = period, yaw_obs += the shortest angular distance to the filter's yaw, est_stats
 * and est_log. On MPC ticks the plan inputs come from the estimated rbd with x0[9] = yaw_obs, the planner and the cycle see the estimate,
 * and the schedule of the new plan is copied into est. The policy, the WeightedWbc and the joint command law see the estimated rbd;
 * actuation, saturation, the plant and the failure checks the true one. est (B) is in/out; est_stats (B, nullable) in/out; est_log
 * (nullable) the estimated rbd in log's layout. Arguments are checked before any launch (sigmas finite and >= 0). With odometry set
 * (hb_rollout_set_odometry), the sensor read also reads each camera and the filter fuses the messages due on the tick. With a hardware
 * setting (hb_rollout_set_hardware), each robot's actuation, saturation and sensors run on its record. The filter measures each robot's
 * feet heights on its estimator map (hb_estimator_set_maps) when it has one, as hb_estimator_update_batch_dev does. */
int hb_rollout_estimated_batch_dev(hb_ctx* ctx, int B, int64_t tick0, int n_ticks, const hb_rollout_params* p, const hb_estimation_params* ep,
                                   const hb_rollout_command* cmd, double* rbd, hb_actuation_state* act, uint8_t* estop, hb_rollout_stats* stats,
                                   hb_estimation_state* est, hb_estimation_stats* est_stats /*nullable*/, double* log /*nullable*/,
                                   double* est_log /*nullable*/);
/* ---- recorded channels: what the controllers did and what the plant felt on every logged tick of both episode calls ----
 * A channel is one device buffer set on the context with hb_rollout_set_channel: B x rows x width elements of the channel's type,
 * instance-major as log. Row r of an episode call holds tick r * log_every of that call (the same row as log, so the state log[:, r] and
 * the action torque[:, r] are a pair), written after the tick's plant step from what the tick computed. A call with log_every == 0
 * records nothing; a NULL log does not stop the recording. Rows of an instance after its fail_tick hold what the kernels computed for
 * the held state (hb_rollout_stats says from which tick on). hb_rollout_estimated_batch_dev writes every set channel,
 * hb_rollout_batch_dev every one but HB_CHANNEL_SENSORS, which it leaves untouched. Instances at or beyond the call's B and rows at or
 * beyond its ceil(n_ticks / log_every) are not written. A call with log_every > 0 is rejected (-1, nothing enqueued) when a set channel
 * has fewer than B instances or fewer than ceil(n_ticks / log_every) rows. With no channel set, or log_every == 0, an episode launches
 * exactly what it launches without this feature; otherwise it adds one launch per recorded tick. */
#define HB_CHANNEL_TORQUE 0          /* double x 10: applied torques after saturation (what the plant step receives, before a variation's motor_strength;
                                        with a motor bridge, the mean over the tick's substeps of the motor's clipped torque) */
#define HB_CHANNEL_JOINT_COMMAND 1   /* double x 50: the joint command law's output per joint (pos_des, vel_des, kp, kd, ff), before the actuation delay */
#define HB_CHANNEL_X_DES 2           /* double x 22: the policy's desired state at t (adopted policy with a latency) */
#define HB_CHANNEL_U_DES 3           /* double x 22 */
#define HB_CHANNEL_WBC_SOLUTION 4    /* double x 38: [qdd, F, tau] after the fallback, weighted or hierarchical */
#define HB_CHANNEL_MODE 5            /* int32 x 1: the contact mode the WBC used */
#define HB_CHANNEL_CONTACT_FORCE 6   /* double x 12: the plant's world-frame force at each contact point in the tick's last substep */
#define HB_CHANNEL_CONTACT_FLAG 7    /* uint8 x 4: that normal force > 0 */
#define HB_CHANNEL_SENSORS 8         /* double x 30: quat (x y z w), ang_vel_local, lin_acc_local, joint_pos, joint_vel as the filter read them (estimated episodes only) */
#define HB_CHANNEL_STATUS 9          /* int32 x 3: wbc status; the MPC cycle's info.status and plan status on an MPC tick, -1 on other ticks */
#define HB_CHANNELS 10
/* Sets channel `channel` of the context's episodes to buffer (device memory, B x rows x the channel's width). B == 0 clears it (buffer may
 * be NULL). -1: an unknown channel, B < 0, rows < 0, or a NULL buffer with B > 0; -4: B > max_batch. A rejected call keeps the previous
 * channel. The call only stores the pointer: the caller keeps the buffer valid until the last episode call that writes it has completed. */
int hb_rollout_set_channel(hb_ctx* ctx, int32_t channel, int B, int rows, void* buffer /*nullable with B == 0*/);
int hb_rbd_to_centroidal_batch_dev(hb_ctx* ctx, int B, const double* rbd, double* x);
int hb_reference_expand_batch_dev(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* x_ref, double* swing_ref,
                                  int32_t* mode);
/* world positions of the four contact frames at the configuration of x (InverseKinematics::computeFootPos,
 * legged_interface/src/foot_planner/InverseKinematics.cpp:253-267) */
int hb_contact_positions_batch_dev(hb_ctx* ctx, int B, const double* x, double* pos /*B x 12*/);
/* probe used by the parity tests: the shipping node linearisation (lin_half of K0) expanded to full tiles: f (22), A = df/dx and
 * Bm = df/du (22 x 22), ee = [pos(12), vel(12), dpos/dx (12 x 22), dvel/dx (12 x 22), dvel/du (12 x 22)] */
int hb_probe_flow_map_dev(hb_ctx* ctx, int B, const double* x, const double* u, double* f, double* A, double* Bm, double* ee);

/* ---- host-pointer (synchronous) entry points: H2D copy, device call, D2H copy ---- */
int hb_wbc_qp_batch(hb_ctx* ctx, int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA,
                    const double* ubA, double* x, int32_t* status, int32_t* iters);
int hb_wbc_solve_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                       const uint8_t* stance_mode, double* sol, int32_t* status);
int hb_wbc_assemble_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                          const uint8_t* stance_mode /*nullable*/, double* H, double* g, double* A, double* lbA, double* ubA, int32_t* m_rows);
int hb_hoqp_solve_batch(hb_ctx* ctx, int B, const hb_hoqp_problem* problems, double* x, double* slack /*nullable*/, int32_t* status /*nullable*/);
int hb_hierarchical_wbc_solve_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, double* sol,
                                    int32_t* status /*nullable*/);
/* the three tasks HierarchicalWbc::update builds, one hb_hoqp_problem per instance; for inspection / parity tests */
int hb_hierarchical_wbc_tasks_batch(hb_ctx* ctx, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                                    hb_hoqp_problem* problems);
int hb_mpc_cold_start_batch(hb_ctx* ctx, int B, const double* x0, const int32_t* mode, double* x_traj, double* u_traj);
int hb_mpc_solve_batch(hb_ctx* ctx, int B, const double* x0, const double* x_ref, const double* swing_ref, const int32_t* mode,
                       double* x_traj, double* u_traj, hb_solve_info* info);
int hb_control_step_batch(hb_ctx* ctx, int B, double t_rel, const double* x0, const double* x_ref, const double* swing_ref,
                          const int32_t* mode, const double* rbd, double* x_traj, double* u_traj, hb_solve_info* info,
                          double* wbc_sol, double* torque, int32_t* wbc_status);
int hb_joint_command_batch(hb_ctx* ctx, int B, const hb_pd_gains* gains, double period, const double* x_des, const double* u_des,
                           const double* wbc_sol, const int32_t* mode_cmd, const double* rbd, const uint8_t* loaded, uint8_t* estop,
                           double* command, double* output_torque);
/* Host-pointer resident cycle. Only the USED entries of the fixed-capacity hb_reference structs cross PCIe. If `refs` points into page-locked
 * memory (cudaHostAlloc / cudaHostRegister; the whole array refs[0..B) must lie inside that allocation) the device gathers and validates the
 * entries itself and the call does no per-instance host work; a pageable array is validated and packed on the host first. Malformed structs
 * (counts beyond the capacities, unordered times, an empty target list, modes outside 0..3) return -1 on both paths. */
int hb_resident_cycle_batch(hb_ctx* ctx, int B, int cold_start, double t_rel, const double* t0, const double* x0, const hb_reference* refs,
                            const double* rbd, hb_solve_info* info, double* wbc_sol, double* torque, int32_t* wbc_status);
int hb_resident_read_batch(hb_ctx* ctx, int B, double* t0 /*nullable*/, double* x_traj /*nullable*/, double* u_traj /*nullable*/);
/* Restores a snapshot taken with hb_resident_read_batch (+ hb_resident_read_grid_batch): the next warm cycle shifts it exactly as if this
 * context had produced it (checkpoint / resume, migration of instances between contexts or GPUs). mode (B x (N+1), nullable) = node modes of
 * the solution, needed by hb_resident_wbc_batch until the next cycle; node_times / n_intervals are required by event_nodes contexts only. */
int hb_resident_write_batch(hb_ctx* ctx, int B, const double* t0, const double* x_traj, const double* u_traj, const int32_t* mode /*nullable*/,
                            const double* node_times /*nullable*/, const int32_t* n_intervals /*nullable*/);
/* node times / interval counts of the resident solution (contexts created with event_nodes = 1) */
int hb_resident_read_grid_batch(hb_ctx* ctx, int B, double* node_times, int32_t* n_intervals);
int hb_time_grid_batch(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* node_times, int32_t* n_intervals, int32_t* status /*nullable*/);
int hb_reference_expand_grid_batch(hb_ctx* ctx, int B, const double* node_times, const hb_reference* refs, double* x_ref, double* swing_ref, int32_t* mode);
int hb_mpc_solve_grid_batch(hb_ctx* ctx, int B, const double* x0, const double* node_times, const int32_t* n_intervals, const double* x_ref,
                            const double* swing_ref, const int32_t* mode, double* x_traj, double* u_traj, hb_solve_info* info);
/* hb_plan_references on the device, host pointers in and out (parity checks of the device planner against the host planner) */
int hb_plan_references_gpu(hb_ctx* ctx, int B, const hb_plan_input* in, double* latest_stance, hb_reference* out, int32_t* status /*nullable*/);
/* The whole cycle from the plan inputs: computeFootPos at x0 + planner (P1, P3, P4, P5) + hb_resident_cycle_batch, all on the device.
 * in[i].feet_pos is ignored (computed from in[i].x0); the planner's latest-stance state is resident (zeroed by cold_start, like
 * SwingTrajectoryPlanner's latestStanceposition_). Per instance 352 B + rbd go in, info / wbc_sol / torque / statuses come out.
 * plan_status[i] != 0: the planner rejected the instance (an all-stance reference at the current pose was used instead). */
int hb_resident_plan_cycle_batch(hb_ctx* ctx, int B, int cold_start, double t_rel, const hb_plan_input* in, const double* rbd,
                                 hb_solve_info* info, double* wbc_sol, double* torque, int32_t* wbc_status, int32_t* plan_status);
int hb_estimator_update_batch(hb_ctx* ctx, int B, const hb_kf_params* params, double dt, hb_kf_state* state, const double* quat,
                              const double* ang_vel_local, const double* lin_acc_local, const double* joint_pos, const double* joint_vel,
                              const uint8_t* contact_flag, double* rbd_out);
/* hb_sim_read_sensors_batch_dev with host pointers (est in/out) */
int hb_sim_read_sensors(hb_ctx* ctx, int B, const hb_sensor_noise* noise, int64_t tick, double accel_dt, const double* rbd, hb_estimation_state* est,
                        double* quat, double* ang_vel_local, double* lin_acc_local, double* joint_pos, double* joint_vel);
int hb_contact_force_estimate_batch(hb_ctx* ctx, int B, double cutoff_frequency, double dt, hb_observer_state* state, const double* rbd,
                                    const double* tau_cmd, double* est_contact_force, double* disturbance_torque /*nullable*/);
int hb_actuation_batch(hb_ctx* ctx, int B, double delay, const double* time, hb_actuation_state* state, const double* command, const double* rbd,
                       double* tau);
/* ---- the simulated hardware outside the episodes (simulated hardware, above): the episode's actuation and sensor read with explicit
 * records, so that an episode with hb_rollout_set_hardware can be written as a loop of public calls ----
 * hw (B, nullable): the record of each robot, validated as by hb_rollout_set_hardware (-1). hb_actuation_hw runs robot i's actuation with
 * hw[i].actuation_delay in place of delay (the limits are the caller's clip); hb_sim_read_sensors_hw reads robot i's sensors with hw[i]'s
 * offsets and sigmas in place of noise's sigmas. NULL hw is exactly hb_actuation_batch / hb_sim_read_sensors, which are these calls with
 * hw = NULL. Host pointers, synchronous; the context's hardware setting is not read. */
int hb_actuation_hw(hb_ctx* ctx, int B, double delay, const hb_hardware_setting* hw /*nullable*/, const double* time, hb_actuation_state* state,
                    const double* command, const double* rbd, double* tau);
int hb_sim_read_sensors_hw(hb_ctx* ctx, int B, const hb_sensor_noise* noise, const hb_hardware_setting* hw /*nullable*/, int64_t tick,
                           double accel_dt, const double* rbd, hb_estimation_state* est, double* quat, double* ang_vel_local, double* lin_acc_local,
                           double* joint_pos, double* joint_vel);
/* ---- the motor bridge outside the episodes (motor bridge, above): the episode's actuation, plant step and sensor read with explicit
 * records, so that an episode with hb_rollout_set_motor_bridge can be written as a loop of public calls ----
 * bridge (B, nullable): the record of every robot of the call, validated as by hb_rollout_set_motor_bridge (-1). Host pointers,
 * synchronous; the context's settings are not read.
 * hb_actuation_bridge: hb_actuation_hw, and with bridge, robot i's oldest entry is encoded on bridge[i] and written to motor_cmd (B x 10 x
 * 5: pos_m, vel_m, kp_m, kd_m, ff_m) in place of a torque to tau. Without bridge, tau is required and motor_cmd is not written (nullable);
 * with it, motor_cmd is required and tau is not written (nullable). hb_actuation_hw and hb_actuation_batch are it with bridge = NULL. */
int hb_actuation_bridge(hb_ctx* ctx, int B, double delay, const hb_hardware_setting* hw /*nullable*/, const hb_motor_bridge* bridge /*nullable*/,
                        const double* time, hb_actuation_state* state, const double* command, const double* rbd, double* tau /*nullable with bridge*/,
                        double* motor_cmd /*nullable without bridge*/);
/* hb_sim_step_terrain, and with bridge, each robot's joints run the motor PD on motor_cmd (B x 10 x 5, hb_actuation_bridge's) on every
 * substep, clipped to limits (B x 10, > 0); tau is then not read (nullable) and applied (B x 10, nullable) receives the mean over the
 * substeps of the clipped torque. Without bridge, tau is required and motor_cmd, limits and applied are not read or written.
 * hb_sim_step_terrain is it with bridge, motor_cmd, limits and applied NULL. */
int hb_sim_step_bridge(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau /*nullable with bridge*/,
                       const double* wrench /*nullable*/, const hb_plant_variation* v /*nullable*/, const hb_terrain* t /*nullable*/,
                       const hb_motor_bridge* bridge /*nullable*/, const double* motor_cmd, const double* limits, double* applied /*nullable*/,
                       double* contact_force /*nullable*/, uint8_t* contact_flag /*nullable*/);
/* hb_sim_step_bridge on each robot's own bodies: links (B, nullable) = the bodies of every robot of the call (link variations, above),
 * validated as by hb_rollout_set_link_variations (-1). hb_sim_step_bridge is it with links = NULL. */
int hb_sim_step_links(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau /*nullable with bridge*/,
                      const double* wrench /*nullable*/, const hb_plant_variation* v /*nullable*/, const hb_terrain* t /*nullable*/,
                      const hb_motor_bridge* bridge /*nullable*/, const double* motor_cmd, const double* limits, double* applied /*nullable*/,
                      const hb_link_variation* links /*nullable*/, double* contact_force /*nullable*/, uint8_t* contact_flag /*nullable*/);
/* hb_sim_step_links with each robot's joint model: joints (B, nullable) = the joints of every robot of the call (joint models, above),
 * validated as by hb_rollout_set_joint_models, and against params by the stability rule (-1 for either). This is the one host-pointer
 * plant step; hb_sim_step_links is it with joints = NULL. */
int hb_sim_step_joints(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau /*nullable with bridge*/,
                       const double* wrench /*nullable*/, const hb_plant_variation* v /*nullable*/, const hb_terrain* t /*nullable*/,
                       const hb_motor_bridge* bridge /*nullable*/, const double* motor_cmd, const double* limits, double* applied /*nullable*/,
                       const hb_link_variation* links /*nullable*/, const hb_joint_model* joints /*nullable*/, double* contact_force /*nullable*/,
                       uint8_t* contact_flag /*nullable*/);
/* hb_sim_read_sensors_hw, and with bridge, each robot's joint readings pass its encoders (steps (3) to (5) of the motor bridge, above)
 * after the offsets and the noise. hb_sim_read_sensors_hw is it with bridge = NULL. */
int hb_sim_read_sensors_bridge(hb_ctx* ctx, int B, const hb_sensor_noise* noise, const hb_hardware_setting* hw /*nullable*/,
                               const hb_motor_bridge* bridge /*nullable*/, int64_t tick, double accel_dt, const double* rbd, hb_estimation_state* est,
                               double* quat, double* ang_vel_local, double* lin_acc_local, double* joint_pos, double* joint_vel);
int hb_sim_step_batch(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, double* contact_force /*nullable*/,
                      uint8_t* contact_flag /*nullable*/);
/* hb_sim_step_batch with an external world wrench on each robot's base: wrench (B x 6) = force [N] at the base frame origin, then a couple
 * [N m], both in the world frame and constant over the step (generalised forces as for pushed episodes, above). NULL wrench is exactly
 * hb_sim_step_batch. */
int hb_sim_step_wrench(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, const double* wrench /*nullable*/,
                       double* contact_force /*nullable*/, uint8_t* contact_flag /*nullable*/);
/* hb_sim_step_wrench on varied plants: v (B, nullable) = the plant of each robot (varied plants, above), validated as by
 * hb_rollout_set_plant_variations (-1). NULL v is exactly hb_sim_step_wrench. */
int hb_sim_step_varied(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, const double* wrench /*nullable*/,
                       const hb_plant_variation* v /*nullable*/, double* contact_force /*nullable*/, uint8_t* contact_flag /*nullable*/);
/* hb_sim_step_varied on terrains: t (B, nullable) = the ground under each robot (terrain, above), validated as by hb_rollout_set_terrains
 * (-1). NULL t is exactly hb_sim_step_varied. hb_sim_step_batch, hb_sim_step_wrench and hb_sim_step_varied are it with the arguments
 * they lack passed as NULL, and it is hb_sim_step_bridge (the motor bridge, above) without a bridge. */
int hb_sim_step_terrain(hb_ctx* ctx, int B, const hb_sim_params* params, double* rbd, const double* tau, const double* wrench /*nullable*/,
                        const hb_plant_variation* v /*nullable*/, const hb_terrain* t /*nullable*/, double* contact_force /*nullable*/,
                        uint8_t* contact_flag /*nullable*/);
int hb_resident_wbc_batch(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode /*nullable*/, double* x_des, double* u_des,
                          int32_t* mode_out, double* wbc_sol, double* torque /*nullable*/, int32_t* wbc_status /*nullable*/);

/* ---- the MRT split outside the episodes: the adopted policy (MPC latency, above) through public calls ----
 * hb_policy_update: MPC_MRT_Interface::updatePolicy of instances 0 .. B-1, each with update[i] != 0 (update NULL: every one) copying the
 * resident solution into its adopted policy. -1 also when a flagged instance holds no resident solution. Synchronous. */
int hb_policy_update(hb_ctx* ctx, int B, const uint8_t* update /*nullable*/);
/* hb_resident_wbc_batch on the adopted policy: evaluatePolicy of each instance's adopted policy at t_now[i], the controller's WBC, torque
 * law. It is the same WBC as hb_resident_wbc_batch and shares its per-instance previous-solution fallback. -1 when an instance of the batch
 * has never adopted a policy. hb_policy_wbc takes host pointers (synchronous), hb_policy_wbc_async device pointers (asynchronous, on the
 * context's stream). */
int hb_policy_wbc(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode /*nullable*/, double* x_des, double* u_des,
                  int32_t* mode_out, double* wbc_sol, double* torque /*nullable*/, int32_t* wbc_status /*nullable*/);
int hb_policy_wbc_async(hb_ctx* ctx, int B, const double* t_now, const double* rbd, const uint8_t* stance_mode /*nullable*/, double* x_des,
                        double* u_des, int32_t* mode_out, double* wbc_sol, double* torque /*nullable*/, int32_t* wbc_status /*nullable*/);

/* ---- odometry outside the episodes: the camera read and the fusion of the estimated episodes (odometry, above) through public calls ----
 * hb_sim_read_odometry: the camera read of instances 0 .. B-1 at absolute tick `tick` on the context's odometry setting and camera state
 * (history and bias, updated), from the true rbd (B x 32); noise gives the seed, est (B) the noise streams (read only). has_msg[i] (B) = 1
 * when a message is due, with pos (B x 3) its position; 0 and pos = 0 otherwise, and for instances without a camera. -1 also for a tick
 * outside 0 .. 2^32 - 1.
 * hb_estimator_fuse_odometry: the fusion on the filter state hb_estimator_update_batch advanced (state, in/out) and the estimated rbd it
 * wrote (rbd, B x 32, in/out): instances with has_msg[i] != 0 take pos[i]; contact_flag (B x 4) as given to the filter, foot_radius from
 * params. An instance with has_msg[i] == 0 is left bit for bit as it is. Both give bit for bit what the estimated episode computes.
 * The plain names take host pointers (synchronous), the _async names device pointers (asynchronous, on the context's stream). */
int hb_sim_read_odometry(hb_ctx* ctx, int B, const hb_sensor_noise* noise, int64_t tick, const double* rbd, const hb_estimation_state* est,
                         double* pos, uint8_t* has_msg);
int hb_sim_read_odometry_async(hb_ctx* ctx, int B, const hb_sensor_noise* noise, int64_t tick, const double* rbd, const hb_estimation_state* est,
                               double* pos, uint8_t* has_msg);
int hb_estimator_fuse_odometry(hb_ctx* ctx, int B, const hb_kf_params* params, hb_kf_state* state, const double* pos, const uint8_t* has_msg,
                               const uint8_t* contact_flag, double* rbd);
int hb_estimator_fuse_odometry_async(hb_ctx* ctx, int B, const hb_kf_params* params, hb_kf_state* state, const double* pos, const uint8_t* has_msg,
                                     const uint8_t* contact_flag, double* rbd);

/* ---- episode snapshots: each robot's whole closed-loop state in one device row (checkpoint, resume, fork) ----
 * The episode calls continue across calls because part of an episode's state stays on the context between them. A snapshot row holds all
 * of that state for one instance, so that an episode can stop and continue in another context or process, and so that many instances can
 * start from one instance's exact mid-episode state (a fork).
 * In a row: every per-instance buffer an episode call reads from an earlier call: the resident MPC solution (the warm start), the
 * WeightedWbc fallback's previous solution, the planner's latest stance positions, the captured goal index and target, the adopted policy
 * of the MRT split and the tracking camera's history and bias. Not in a row: the caller's buffers (rbd, act, estop, stats and, in estimated
 * episodes, est and est_stats), which the caller saves itself, and configuration: the per-robot settings, the WBC settings and
 * formulation, loaded task settings and recorded channels.
 * Row layout (treated as opaque; hb_episode_state_bytes gives its size): a header of four int64 (horizon_N, event_nodes, the row's size in
 * bytes, HB_EPISODE_HAS_* flags), then these segments, each padded to a multiple of 8 bytes: the resident solution (t0 double; x_traj
 * (N+1) x 22 double; u_traj N x 22 double; on event-node contexts node_times (N+1) double; node modes (N+1) int32; on event-node contexts
 * n_intervals int32, each of these padded), the fallback's previous solution (38 double), the stance positions (12 double), the captured
 * goal index (int32, -1: none), the captured target (hb_target), the adopted policy (as the resident solution) and the camera state
 * ((HB_ODOM_MAX_DELAY + 1) x 3 double history, 3 double bias), and only on a context with a teleop setting the publisher state (4 double
 * filtered command, int32 1 + the goal last seen, int32 padding; teleoperation, above), so that rows of a context without one keep their
 * size. A segment whose buffer the context never allocated (no goals set, no odometry set, no policy adopted) saves as its cleared value:
 * goal index -1 (the source of the captured target: a goal's index, HB_MAX_GOALS for a teleop message), zeros elsewhere.
 * hb_episode_save_async writes row i (device memory, B rows) from instance src[i] of the context (src NULL: instance i), flags from the
 * context's bookkeeping. Asynchronous on the context's stream: src (host) is consumed when the call returns.
 * hb_episode_restore sets instance i of the context from row src[i] of the n_rows rows (src NULL: row i). It reads the rows' headers back
 * with one small synchronous copy before anything changes, and returns when the rows are written: a setting-like call, not a per-tick one.
 * After it, instances [0, B) hold the rows' solution, fallback solution and adopted policy as their flags say, so that a warm episode call
 * (tick0 > 0) passes its entry checks exactly when the rows would have passed them in the context that saved them. A restore writes the
 * goal and camera state whether or not goals or odometry are set, allocating their buffers as their setting calls do; hb_rollout_set_goals,
 * hb_rollout_set_odometry and hb_rollout_set_teleop clear that state, so a restore must come after them.
 * Return codes: -1 for a null context, B < 0, NULL rows with B > 0, a src entry outside [0, max_batch) (save) or [0, n_rows) (restore), a
 * B > n_rows restore with src NULL, and on restore a row whose fingerprint (horizon_N, event_nodes, size) differs from this context's, a row
 * without HB_EPISODE_HAS_SOLUTION, or fallback flags that would leave instances with a previous WBC solution that are not a prefix
 * [0, k) of the context; -4 for B > max_batch. B == 0 does nothing. A rejected call changes nothing and launches nothing. Each call is one
 * launch; without them an episode launches exactly what it launches without this feature. */
#define HB_EPISODE_HEADER_BYTES 32
#define HB_EPISODE_HAS_SOLUTION 1      /* the instance holds a resident MPC solution                                         */
#define HB_EPISODE_HAS_FALLBACK 2      /* the WeightedWbc fallback holds a previous solution                                 */
#define HB_EPISODE_HAS_POLICY 4        /* the instance has adopted a policy (MPC latency)                                    */
/* bytes of one instance's row for this context's configuration; -1 for a null context */
int64_t hb_episode_state_bytes(const hb_ctx* ctx);
int hb_episode_save_async(hb_ctx* ctx, int B, const int32_t* src /*host, nullable*/, void* rows /*device, B rows*/);
int hb_episode_restore(hb_ctx* ctx, int B, const int32_t* src /*host, nullable*/, int n_rows, const void* rows /*device, n_rows rows*/);
int hb_rbd_to_centroidal_batch(hb_ctx* ctx, int B, const double* rbd, double* x);
int hb_reference_expand_batch(hb_ctx* ctx, int B, const double* t0, const hb_reference* refs, double* x_ref, double* swing_ref,
                              int32_t* mode);
int hb_probe_flow_map(hb_ctx* ctx, int B, const double* x, const double* u, double* f, double* A, double* Bm, double* ee);
int hb_contact_positions_batch(hb_ctx* ctx, int B, const double* x, double* pos /*B x 12*/);

/* ---- host-only reference preprocessing (no GPU work): gait tiling, swing-foot planner, cmd_vel target ----
 * replaces GaitSchedule::{insert,tile}ModeSequenceTemplate (legged_interface/src/gait/GaitSchedule.cpp:57-161),
 * SwingTrajectoryPlanner::update (src/foot_planner/SwingTrajectoryPlanner.cpp:164-286), cmdVelToTargetTrajectories
 * (legged_controllers/src/TargetTrajectoriesPublisher.cpp:102-130) and calculateJointRef + InverseKinematics::computeIK
 * (src/SwitchedModelReferenceManager.cpp:251-300, src/foot_planner/InverseKinematics.cpp:20-231). latest_stance (B x 12) is the planner's state, in/out.
 * Returns 0, or -1 on misuse, or -5 when a schedule does not define the take-off / touch-down of a swing phase (the reference
 * throws there, SwingTrajectoryPlanner.cpp:421-458) or exceeds the capacity of hb_reference.
 * Instances are spread over std::thread::hardware_concurrency() host threads (hb_plan_set_threads overrides the count). */
int hb_plan_references(int B, const hb_plan_input* in, double* latest_stance, hb_reference* out);
/* hb_plan_references with an explicit target per instance: targets (B, nullable) replaces cmdVelToTargetTrajectories for every instance,
 * everything else unchanged (the swing planner still reads cmd_vel as its body velocity command; with joint_ik the target is resampled and
 * its joints filled by IK). NULL is hb_plan_references. -1 also for a record that hb_plan_set_targets rejects. */
int hb_plan_references_targets(int B, const hb_plan_input* in, const hb_target* targets, double* latest_stance, hb_reference* out);
/* hb_plan_references_targets with planner settings per instance: settings (B, nullable) replaces the compiled-in templates and swing
 * settings for every instance (hb_planner_settings). NULL settings, and hb_default_planner_settings records, give
 * hb_plan_references_targets bit for bit. -1 also for a record that is not valid. */
int hb_plan_references_settings(int B, const hb_plan_input* in, const hb_target* targets /*nullable*/, const hb_planner_settings* settings /*nullable*/,
                                double* latest_stance, hb_reference* out);
/* hb_plan_references_settings on height maps (height maps, above): maps (B, nullable), instance i plans on maps[i]. NULL maps is
 * hb_plan_references_settings, and all-zero maps give it bit for bit. -1 also for a map hb_plan_set_maps rejects. */
int hb_plan_references_maps(int B, const hb_plan_input* in, const hb_target* targets /*nullable*/, const hb_planner_settings* settings /*nullable*/,
                            const hb_terrain* maps /*nullable*/, double* latest_stance, hb_reference* out);
/* goalToTargetTrajectories (TargetTrajectoriesPublisher.cpp:83-100, with estimateTimeToTarget :29-38 and
 * targetPoseToTargetTrajectories :41-62) for the observation (t[i], x[i]) and goal[i] = (x, y, yaw), host only. With p = x[6:12] and
 * z' = p[2] + clamp(HB_COM_HEIGHT - p[2], -0.04, 0.04): sample 0 = (t, [0 (6), p[0], p[1], z', p[3], 0, 0, default joints]), sample 1 =
 * (t + T, [0 (6), goal x, goal y, z', goal yaw, 0, 0, default joints]) with T = max(|goal yaw - p[3]| / HB_TARGET_ROTATION_VELOCITY,
 * sqrt(dx^2 + dy^2) / HB_TARGET_DISPLACEMENT_VELOCITY), each square rounded before the sum. The yaw difference is not wrapped, as in the
 * reference: the goal yaw is absolute in the unwrapped convention of x[9]. T == 0 gives the single sample 1 at time t (n = 1) where the
 * reference would publish two samples at the same time. -1 for a NULL pointer, B < 0 or a non-finite t, x[6:10] or goal. */
int hb_goal_to_target(int B, const double* t, const double* x /*B x 22*/, const double* goal /*B x 3*/, hb_target* out);
/* hb_goal_to_target on height maps (B, nullable; height maps, above): the body heights of instance i's target are taken above maps[i].
 * NULL is hb_goal_to_target; -1 also for a map hb_plan_set_maps rejects. */
int hb_goal_to_target_maps(int B, const double* t, const double* x /*B x 22*/, const double* goal /*B x 3*/, const hb_terrain* maps /*nullable*/,
                           hb_target* out);
/* cmdVelToTargetTrajectories (TargetTrajectoriesPublisher.cpp:102-130) for the observation (t[i], x[i]) and cmd_vel[i] = (vx, vy, vz, yaw
 * rate), host only: the two-sample target the planner builds from cmd_vel with time_to_target = horizon (hb_plan_references with joint_ik
 * = 0 carries it bit for bit), the unused samples zero. The teleop messages' target (teleoperation, above). -1 for a NULL pointer, B < 0, a
 * non-finite t, horizon, x[6:12] or cmd_vel. */
int hb_cmd_vel_to_target(int B, const double* t, double horizon, const double* x /*B x 22*/, const double* cmd_vel /*B x 4*/, hb_target* out);
/* hb_cmd_vel_to_target on height maps (B, nullable; height maps, above): the body heights of instance i's target are taken above maps[i].
 * NULL is hb_cmd_vel_to_target; -1 also for a map hb_plan_set_maps rejects. */
int hb_cmd_vel_to_target_maps(int B, const double* t, double horizon, const double* x /*B x 22*/, const double* cmd_vel /*B x 4*/,
                              const hb_terrain* maps /*nullable*/, hb_target* out);
/* Host threads used by hb_plan_references (process-wide); 0 = hardware_concurrency. The result does not depend on the count. */
int hb_plan_set_threads(int n_threads);
/* speed-based gait selection (calculateVelAbs + walkGait / trotGait, src/SwitchedModelReferenceManager.cpp:185-249): updates the
 * 50-sample moving average of 0.5*(command + target) speed of every instance and applies the thresholds stance <= 0.02 < (no change)
 * <= 0.03 < trot < 0.4 <= level 3. gait_type: 0 walk (automatic), 2 trot (forced). level[i] = gait level in force after the call,
 * insert[i] = 1 when a new template is inserted on this call. */
int hb_gait_select(int B, hb_gait_selector* state, const int32_t* gait_type, const double* cmd_vel /*B x 4*/,
                   const double* target_state0 /*B x 22*/, int32_t* level, int32_t* insert);

/* ---- (e) multi-GPU shards (SURVEY 8e; replaces nothing in the reference, which runs one robot per process): one process + one hb_ctx
 * per GPU, instances split in contiguous blocks, no collective on the data path. The only exchange is the gather of per-instance
 * output rows (the 80-byte torque rows of the control step), by NCCL all-gather on the shard's own stream behind an event on the
 * context's stream, so it overlaps the next step's kernels. NCCL is resolved at run time (the libnccl.so.2 already in the process, else
 * the system one); a single-GPU caller never loads it. Return code -6: NCCL missing or a collective failed (hb_shard_last_error). */
#define HB_SHARD_ID_BYTES 128
typedef struct hb_shard hb_shard;
/* contiguous block [begin, begin + count) of `rank`; block sizes differ by at most one */
int hb_shard_partition(int total, int world, int rank, int* begin, int* count);
/* stable permutation that groups instances with the same mode sequence (mode: B x nodes), so that the warps of a wave run the same
 * swing-contact specialisation: sorted[i] = original[perm[i]]; inverse (nullable): inverse[perm[i]] = i */
int hb_shard_sort_by_schedule(int B, int nodes, const int32_t* mode, int32_t* perm, int32_t* inverse);
/* rank 0 draws the communicator id (HB_SHARD_ID_BYTES bytes); the caller hands the bytes to the other ranks out of band (MPI, a file, a socket) */
int hb_shard_unique_id(void* id);
/* collective over all ranks; total_instances = instances of the whole job, max_row_doubles = widest row ever gathered. world == 1: id may be NULL */
int hb_shard_create(hb_ctx* ctx, const void* id, int world, int rank, int total_instances, int max_row_doubles, hb_shard** out);
int hb_shard_destroy(hb_shard* shard);
int hb_shard_block(const hb_shard* shard, int* begin, int* count);
/* rows_dev: count x row_doubles of this rank's block (device). inverse_dev (nullable, device): undo a schedule sort first
 * (row i of the block = rows_dev[inverse_dev[i]]). *gathered_dev: total_instances x row_doubles in instance order on EVERY rank, complete
 * after hb_shard_wait; double buffered, valid until the second next call. Asynchronous: ordered behind the context's stream. */
int hb_shard_gather_dev(hb_shard* shard, int row_doubles, const double* rows_dev, const int32_t* inverse_dev, const double** gathered_dev);
/* the context's stream waits for the last gather; block_host != 0 also blocks the calling thread until it has landed */
int hb_shard_wait(hb_shard* shard, int block_host);
const char* hb_shard_last_error(const hb_shard* shard);

#ifdef __cplusplus
}
#endif
#endif
