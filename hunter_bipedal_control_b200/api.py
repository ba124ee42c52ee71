"""ctypes binding of libhunter_b200.so (C ABI in include/hunter_b200.h) and host-side mirrors of the reference operators.

The product path has no CPU fallback: if the CUDA library is missing or no H100 is visible, every entry point raises.

Mirrors of the reference interface for this path (same names / argument meaning / error behaviour):
  * ``WeightedWbc.update(stateDesired, inputDesired, rbdStateMeasured, mode, period)``  -- legged_wbc/include/legged_wbc/WbcBase.h:43-44,
    legged_wbc/src/WeightedWbc.cpp:18-66 (returns the 38-vector [qdd, F, tau]; on solver failure prints and re-uses the last solution).
  * ``SqpMpc.advance / evaluatePolicy``  -- the calls legged_controllers/src/LeggedController.cpp:144-156,406 makes through MPC_MRT_Interface.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libhunter_b200.so")
_lib = None

NX, NU, NQ, NJ, NWBC = 22, 22, 16, 10, 38
HB_MAX_EVENTS, HB_MAX_TARGETS, HB_MAX_SEGMENTS = 32, 16, 24
HB_MAX_HORIZON = 512       # longest horizon_N hb_create accepts
# hb_check_setting_records' kinds: the record type of each per-robot setting call
HB_SETTING_PUSHES, HB_SETTING_PLANT_VARIATIONS, HB_SETTING_TERRAINS, HB_SETTING_GOALS, HB_SETTING_ODOMETRY = 0, 1, 2, 3, 4
HB_SETTING_CONTROLLERS, HB_SETTING_HARDWARE, HB_SETTING_PLANNER, HB_SETTING_TARGETS, HB_SETTING_LATENCIES = 5, 6, 7, 8, 9
# The recorded channels of the episodes (hb_rollout_set_channel, HB_CHANNEL_*): name -> (index, element type, elements per row)
CHANNELS = {"torque": (0, np.float64, 10), "joint_command": (1, np.float64, 50), "x_des": (2, np.float64, 22), "u_des": (3, np.float64, 22),
            "wbc_solution": (4, np.float64, 38), "mode": (5, np.int32, 1), "contact_force": (6, np.float64, 12), "contact_flag": (7, np.uint8, 4),
            "sensors": (8, np.float64, 30), "status": (9, np.int32, 3)}
# episode snapshot rows (hb_episode_save_async): the header's size and its flags
HB_EPISODE_HEADER_BYTES, HB_EPISODE_HAS_SOLUTION, HB_EPISODE_HAS_FALLBACK, HB_EPISODE_HAS_POLICY = 32, 1, 2, 4

EXPORTED_SYMBOLS = [
    "hb_shard_partition", "hb_shard_sort_by_schedule", "hb_shard_unique_id", "hb_shard_create", "hb_shard_destroy", "hb_shard_block", "hb_shard_gather_dev", "hb_shard_wait", "hb_shard_last_error",
    "hb_default_config", "hb_create", "hb_destroy", "hb_sync", "hb_strerror", "hb_last_cuda_error", "hb_launch_count", "hb_last_reference_upload_bytes", "hb_stream", "hb_profile_enable", "hb_profile_read",
    "hb_wbc_qp_batch_dev", "hb_wbc_qp_rows_batch_dev", "hb_wbc_assemble_batch_dev", "hb_wbc_assemble_batch", "hb_wbc_solve_batch_dev", "hb_mpc_cold_start_batch_dev", "hb_mpc_solve_batch_dev",
    "hb_policy_eval_batch_dev", "hb_control_step_batch_dev", "hb_rbd_to_centroidal_batch_dev", "hb_reference_expand_batch_dev",
    "hb_probe_flow_map_dev", "hb_contact_positions_batch_dev", "hb_contact_positions_batch", "hb_plan_references", "hb_plan_set_threads", "hb_gait_select", "hb_resident_cycle_batch_dev", "hb_resident_cycle_batch", "hb_resident_read_batch", "hb_plan_references_batch_dev",
    "hb_plan_references_gpu", "hb_resident_plan_cycle_batch", "hb_default_kf_params", "hb_kf_reset", "hb_estimator_update_batch_dev",
    "hb_estimator_update_batch", "hb_default_pd_gains", "hb_joint_command_batch_dev", "hb_joint_command_batch",
    "hb_wbc_qp_batch", "hb_wbc_solve_batch", "hb_mpc_cold_start_batch", "hb_mpc_solve_batch", "hb_control_step_batch",
    "hb_rbd_to_centroidal_batch", "hb_reference_expand_batch", "hb_probe_flow_map",
    "hb_observer_reset", "hb_contact_force_estimate_batch_dev", "hb_contact_force_estimate_batch",
    "hb_default_wbc_settings", "hb_parse_task_info", "hb_wbc_get_settings", "hb_wbc_set_settings", "hb_wbc_set_kp_kd", "hb_load_task_info",
    "hb_wbc_set_formulation", "hb_wbc_get_formulation",
    "hb_hoqp_solve_batch_dev", "hb_hierarchical_wbc_solve_batch_dev", "hb_hoqp_solve_batch", "hb_hierarchical_wbc_solve_batch", "hb_hierarchical_wbc_tasks_batch",
    "hb_default_sim_params", "hb_actuation_reset", "hb_actuation_batch_dev", "hb_actuation_batch", "hb_sim_step_batch_dev", "hb_sim_step_batch",
    "hb_resident_wbc_batch_dev", "hb_resident_wbc_batch",
    "hb_time_grid_batch_dev", "hb_reference_expand_grid_batch_dev", "hb_mpc_solve_grid_batch_dev", "hb_policy_eval_grid_batch_dev",
    "hb_time_grid_batch", "hb_reference_expand_grid_batch", "hb_mpc_solve_grid_batch", "hb_resident_read_grid_batch", "hb_resident_write_batch",
    "hb_default_rollout_params", "hb_rollout_batch_dev", "hb_rollout_set_pushes", "hb_sim_step_wrench",
    "hb_default_plant_variation", "hb_rollout_set_plant_variations", "hb_sim_step_varied", "hb_rollout_set_terrains", "hb_sim_step_terrain",
    "hb_default_estimation_params", "hb_estimation_reset", "hb_sim_read_sensors_batch_dev", "hb_sim_read_sensors", "hb_rollout_estimated_batch_dev",
    "hb_plan_references_targets", "hb_goal_to_target", "hb_plan_set_targets", "hb_rollout_set_goals",
    "hb_rollout_set_mpc_latencies", "hb_policy_update", "hb_policy_wbc", "hb_policy_wbc_async",
    "hb_rollout_set_odometry", "hb_sim_read_odometry", "hb_sim_read_odometry_async", "hb_estimator_fuse_odometry", "hb_estimator_fuse_odometry_async",
    "hb_rollout_set_controller_settings",
    "hb_default_hardware_setting", "hb_rollout_set_hardware", "hb_actuation_hw", "hb_sim_read_sensors_hw",
    "hb_default_motor_bridge", "hb_rollout_set_motor_bridge", "hb_motor_bridge_encode", "hb_motor_bridge_feedback", "hb_actuation_bridge",
    "hb_sim_step_bridge", "hb_sim_read_sensors_bridge",
    "hb_default_link_variation", "hb_rollout_set_link_variations", "hb_sim_step_links",
    "hb_default_joint_model", "hb_rollout_set_joint_models", "hb_sim_step_joints",
    "hb_default_teleop_setting", "hb_rollout_set_teleop", "hb_cmd_vel_to_target",
    "hb_default_planner_settings", "hb_parse_planner_settings", "hb_plan_references_settings", "hb_plan_set_settings",
    "hb_plan_set_maps", "hb_plan_references_maps", "hb_goal_to_target_maps", "hb_cmd_vel_to_target_maps", "hb_estimator_set_maps",
    "hb_mpc_set_maps", "hb_wbc_set_maps", "hb_mpc_set_cone_maps",
    "hb_default_contact_detection", "hb_rollout_set_contact_detection", "hb_contact_state_estimate_async", "hb_contact_state_estimate",
    "hb_rollout_contact_estimates", "hb_contact_state_host",
    "hb_check_setting_records", "hb_rollout_set_channel",
    "hb_episode_state_bytes", "hb_episode_save_async", "hb_episode_restore",
]


class HbConfig(C.Structure):
    _fields_ = [("horizon_N", C.c_int32), ("dt", C.c_double), ("max_batch", C.c_int32), ("wbc_rho", C.c_double),
                ("qp_max_iter", C.c_int32), ("line_search_max_trials", C.c_int32), ("time_horizon", C.c_double), ("event_nodes", C.c_int32), ("e2e_chunks", C.c_int32)]


class HbSolveInfo(C.Structure):
    _fields_ = [("alpha", C.c_double), ("merit0", C.c_double), ("merit1", C.c_double), ("viol0", C.c_double), ("viol1", C.c_double),
                ("armijo", C.c_double), ("status", C.c_int32), ("n_trials", C.c_int32)]


INFO_DTYPE = np.dtype(HbSolveInfo)


class HbReference(C.Structure):
    _fields_ = [("n_events", C.c_int32), ("event_times", C.c_double * HB_MAX_EVENTS), ("modes", C.c_int32 * (HB_MAX_EVENTS + 1)),
                ("n_targets", C.c_int32), ("target_times", C.c_double * HB_MAX_TARGETS), ("target_states", (C.c_double * 22) * HB_MAX_TARGETS),
                ("n_segments", (C.c_int32 * 3) * 4), ("segments", (((C.c_double * 6) * HB_MAX_SEGMENTS) * 3) * 4)]


class HbPlanInput(C.Structure):
    _fields_ = [("t0", C.c_double), ("horizon", C.c_double), ("time_to_target", C.c_double), ("gait_start", C.c_double), ("prev_event", C.c_double),
                ("x0", C.c_double * 22), ("cmd_vel", C.c_double * 4), ("feet_pos", C.c_double * 12), ("gait", C.c_int32), ("joint_ik", C.c_int32)]


class HbTarget(C.Structure):
    _fields_ = [("n", C.c_int32), ("time", C.c_double * HB_MAX_TARGETS), ("state", (C.c_double * 22) * HB_MAX_TARGETS)]


def make_targets(times, states):
    """ctypes array of HbTarget (plan_references(targets=...), Context.set_plan_targets): instance i has the samples (times[i][k],
    states[i][k]), k < n_i. times: B sequences of strictly ascending absolute times (1..HB_MAX_TARGETS each); states: B sequences of
    22-vectors of the same lengths."""
    B = len(times)
    out = (HbTarget * B)()
    v = np.ctypeslib.as_array(out)
    for i in range(B):
        t, x = _f64(times[i]).reshape(-1), _f64(states[i]).reshape(-1, 22)
        n = len(t)
        if not 1 <= n <= HB_MAX_TARGETS or x.shape[0] != n:
            raise ValueError("targets: 1..%d samples with one state each expected, got %d times and %d states" % (HB_MAX_TARGETS, n, x.shape[0]))
        v["n"][i] = n; v["time"][i, :n] = t; v["state"][i, :n] = x
    return out


def reference_target(ref):
    """The target trajectory an HbReference carries (its target samples) as an HbTarget."""
    n = ref.n_targets
    return make_targets([np.array(ref.target_times[:n])], [np.array([ref.target_states[k][:] for k in range(n)])])[0]


def _maps_of(maps, B, what):
    """The height maps argument of a host planner call: None, or B HbTerrain (make_terrains)."""
    if maps is not None and len(maps) != B:
        raise ValueError("%s: %d height maps for %d instances" % (what, len(maps), B))
    return maps


def cmd_vel_to_target(t, horizon, x, cmd_vel, maps=None):
    """cmdVelToTargetTrajectories (hb_cmd_vel_to_target) for a batch: the two-sample target the planner builds from cmd_vel (vx, vy, vz, yaw
    rate) at time t on the observation x with time_to_target = horizon. t (B,) or a scalar, x (B, 22), cmd_vel (B, 4) or (4,). maps: B
    HbTerrain (make_terrains), the height map of each instance (hb_cmd_vel_to_target_maps). Returns a ctypes array of B HbTarget."""
    x = _f64(x).reshape(-1, NX); B = x.shape[0]
    t = _f64(np.broadcast_to(_f64(t), (B,))); cmd = _f64(np.broadcast_to(_f64(cmd_vel), (B, 4)))
    out = (HbTarget * B)()
    _check(load_library().hb_cmd_vel_to_target_maps(B, _ptr(t), C.c_double(horizon), _ptr(x), _ptr(cmd), _maps_of(maps, B, "cmd_vel_to_target"), out),
           "hb_cmd_vel_to_target_maps")
    return out


def goal_to_target(t, x, goal, maps=None):
    """goalToTargetTrajectories (hb_goal_to_target) for a batch: t (B,) or a scalar, x (B, 22), goal (B, 3) = (x, y, yaw) or (3,). maps: B
    HbTerrain (make_terrains), the height map of each instance (hb_goal_to_target_maps). Returns a ctypes array of B HbTarget."""
    x = _f64(x).reshape(-1, NX); B = x.shape[0]
    t = _f64(np.broadcast_to(_f64(t), (B,))); goal = _f64(np.broadcast_to(_f64(goal), (B, 3)))
    out = (HbTarget * B)()
    _check(load_library().hb_goal_to_target_maps(B, _ptr(t), _ptr(x), _ptr(goal), _maps_of(maps, B, "goal_to_target"), out), "hb_goal_to_target_maps")
    return out


HB_GAIT_MAX_PHASES = 8
MODE_NAMES = {"FLY": 0, "R": 1, "L": 2, "STANCE": 3}      # gait.info's mode names (string2ModeNumber)
SWING_FIELDS = ("swing_height", "swing_time_scale", "next_stance_z", "feet_bias_x1", "feet_bias_x2", "feet_bias_y", "feet_bias_z")


class HbGaitTemplate(C.Structure):
    _fields_ = [("n_phase", C.c_int32), ("modes", C.c_int32 * HB_GAIT_MAX_PHASES), ("switching_times", C.c_double * (HB_GAIT_MAX_PHASES + 1))]


class HbPlannerSettings(C.Structure):
    _fields_ = [("gait", HbGaitTemplate * 4)] + [(k, C.c_double) for k in SWING_FIELDS]


def gait_template(modes, switching_times):
    """HbGaitTemplate of a ModeSequenceTemplate: modes (names FLY / R / L / STANCE or ids 0..3) and their n + 1 switching times, [0] = 0.
    Raises ValueError for an unknown mode name, counts that do not match or more than HB_GAIT_MAX_PHASES phases; the library checks the
    times (hb_plan_set_settings)."""
    m = [MODE_NAMES[x] if isinstance(x, str) else int(x) for x in modes]
    t = [float(x) for x in switching_times]
    if not 1 <= len(m) <= HB_GAIT_MAX_PHASES or len(t) != len(m) + 1:
        raise ValueError("gait template: 1..%d modes and one more switching time expected, got %d and %d" % (HB_GAIT_MAX_PHASES, len(m), len(t)))
    g = HbGaitTemplate()
    g.n_phase = len(m)
    g.modes[:len(m)] = m
    g.switching_times[:len(t)] = t
    return g


def default_planner_settings():
    """hb_default_planner_settings: gait.info's four templates and task.info's swing_trajectory_config, the compiled-in planner values."""
    s = HbPlannerSettings()
    _check(load_library().hb_default_planner_settings(C.byref(s)), "hb_default_planner_settings")
    return s


def parse_planner_settings(task_info, gait_info):
    """hb_parse_planner_settings: swing_trajectory_config of a task.info file and the templates of a gait.info file in its list order (host
    only); absent keys and templates keep the defaults."""
    s = HbPlannerSettings()
    _check(load_library().hb_parse_planner_settings(str(task_info).encode(), str(gait_info).encode(), C.byref(s)), "hb_parse_planner_settings")
    return s


def _is_template(v):
    """A single template: an HbGaitTemplate or a (modes, switching_times) pair whose modes are names or ids."""
    if isinstance(v, HbGaitTemplate):
        return True
    return len(v) == 2 and all(isinstance(m, str) or np.ndim(m) == 0 for m in v[0])


def make_planner_settings(B, base=None, gaits=None, **fields):
    """ctypes array of B HbPlannerSettings (Context.set_planner_settings, plan_references(settings=...)): each robot's gait templates and
    swing settings. base (HbPlannerSettings) is every record's start, default default_planner_settings(). gaits maps a gait (name of
    GAIT_IDS or id) to a template, an HbGaitTemplate or (modes, switching_times) as gait_template takes, for every robot, or to a list of B
    such templates, one per robot. The swing fields (SWING_FIELDS) can be given by name, as a scalar or a (B,) array. Raises ValueError for
    an unknown name, a malformed template or a shape that does not broadcast."""
    base = default_planner_settings() if base is None else base
    out = (HbPlannerSettings * B)()
    v = np.ctypeslib.as_array(out)
    v[:] = np.frombuffer(bytes(base), dtype=v.dtype)[0]
    for name, value in fields.items():
        if name not in SWING_FIELDS:
            raise ValueError("planner settings: unknown field %r" % name)
        try:
            v[name] = np.broadcast_to(_f64(value), (B,))
        except ValueError as e:
            raise ValueError("planner settings: %s: (B,) or a scalar expected: %s" % (name, e))
    for gait, tmpl in (gaits or {}).items():
        g = GAIT_IDS[gait] if isinstance(gait, str) else int(gait)
        if not 0 <= g <= 3:
            raise ValueError("planner settings: gait %r outside 0..3" % (gait,))
        per = [tmpl] * B if _is_template(tmpl) else list(tmpl)
        if len(per) != B:
            raise ValueError("planner settings: gait %r: one template or %d expected, got %d" % (gait, B, len(per)))
        for i, t in enumerate(per):
            out[i].gait[g] = t if isinstance(t, HbGaitTemplate) else gait_template(*t)
    return out


class HbPdGains(C.Structure):
    _fields_ = [(k, C.c_double) for k in ("kp_position", "kd_position", "kp_big_stance", "kp_big_swing", "kd_big", "kp_small_stance",
                                          "kp_small_swing", "kd_small", "kd_feet")]


def default_pd_gains():
    g = HbPdGains()
    _check(load_library().hb_default_pd_gains(C.byref(g)), "hb_default_pd_gains")
    return g


class HbKfState(C.Structure):
    _fields_ = [("x_hat", C.c_double * 18), ("P", C.c_double * 324), ("feet_heights", C.c_double * 4)]


class HbKfParams(C.Structure):
    _fields_ = [(k, C.c_double) for k in ("foot_radius", "imu_process_noise_position", "imu_process_noise_velocity", "foot_process_noise_position",
                                          "foot_sensor_noise_position", "foot_sensor_noise_velocity", "foot_height_sensor_noise")]


class HbWbcSettings(C.Structure):
    _fields_ = [("torque_limits", C.c_double * 5)] + [(k, C.c_double) for k in (
        "friction_coefficient", "swing_kp", "swing_kd", "base_accel_kp", "base_accel_kd", "base_height_kp", "base_height_kd", "base_angular_kp",
        "base_angular_kd", "weight_swing_leg", "weight_base_accel", "weight_contact_force")]

    def as_array(self):
        return np.frombuffer(bytes(self), dtype=np.float64).copy()


class HbTaskInfo(C.Structure):
    _fields_ = [("wbc", HbWbcSettings), ("kalman", C.c_double * 7), ("contact_force_cutoff_frequency", C.c_double), ("contact_threshold", C.c_double),
                ("sqp_dt", C.c_double), ("sqp_iteration", C.c_int32), ("mpc_time_horizon", C.c_double), ("mpc_cold_start", C.c_int32), ("found", C.c_int32)]


def parse_task_info(path):
    """hb_parse_task_info: the WBC / estimator / discretisation settings of a task.info file (host only)."""
    ti = HbTaskInfo()
    _check(load_library().hb_parse_task_info(str(path).encode(), C.byref(ti)), "hb_parse_task_info")
    return ti


class HbContactDetection(C.Structure):
    SETTING_KIND = 20        # HB_SETTING_CONTACT_DETECTION, the record's kind for hb_check_setting_records
    _fields_ = [("cutoff_frequency", C.c_double), ("threshold", C.c_double), ("swing_fraction", C.c_double), ("stance_fraction", C.c_double)]


def default_contact_detection(task=None):
    """hb_default_contact_detection: the observer's cutoff and the contact threshold of task (an HbTaskInfo, or the path of a task.info
    file; None: 250 and 75), with the reference's fractions 0.75 and 0.25."""
    if task is not None and not isinstance(task, HbTaskInfo):
        task = parse_task_info(task)
    r = HbContactDetection()
    _check(load_library().hb_default_contact_detection(None if task is None else C.byref(task), C.byref(r)), "hb_default_contact_detection")
    return r


def make_contact_detection_settings(B, base=None, **fields):
    """ctypes array of B HbContactDetection (Context.set_contact_detection): each robot's contact detection in rollout_estimated. base
    (HbContactDetection, default default_contact_detection()) is the base of every record; any field can be given by name as a scalar or a
    (B,) array. Raises ValueError for an unknown name, a shape that does not broadcast, and a record the setter rejects, naming the first."""
    base = default_contact_detection() if base is None else base
    out = (HbContactDetection * B)()
    v = np.ctypeslib.as_array(out)
    v[:] = np.frombuffer(bytes(base), dtype=v.dtype)[0]
    for name, value in fields.items():
        if name not in v.dtype.names:
            raise ValueError("contact detection: unknown field %r" % name)
        try:
            v[name] = np.broadcast_to(_f64(value), (B,))
        except ValueError as e:
            raise ValueError("contact detection: %s: (B,) or a scalar expected: %s" % (name, e))
    return _check_records(HbContactDetection.SETTING_KIND, out, "contact_detection")


def _contact_records(records, B, what):
    """records (None, a ctypes array or a sequence of B HbContactDetection) as a ctypes array or None, or ValueError."""
    if records is None:
        return None
    if len(records) != B:
        raise ValueError("%s: %d records for %d instances" % (what, len(records), B))
    return records if isinstance(records, C.Array) else (HbContactDetection * B)(*records)


def contact_state_host(t, est, est_force, records, flags):
    """The contact detection rule on the host (hb_contact_state_host): est (ctypes array of B HbEstimationState, the stored schedules),
    est_force [B,16] (the observer's output), records (B HbContactDetection, or None: flags unchanged) and the schedule's flags [B,4] at
    time t. Returns (the detected flags [B,4] uint8, the phase times [B,4,2]: start and stop of each contact's run around t)."""
    B = len(est)
    force = _f64(est_force).reshape(B, 16)
    fl = np.ascontiguousarray(flags, dtype=np.uint8).reshape(B, 4).copy()
    times = np.zeros((B, 4, 2))
    _check(load_library().hb_contact_state_host(B, C.c_double(t), est, _ptr(force), _contact_records(records, B, "contact_state_host"), _ptr(fl),
                                                _ptr(times)), "hb_contact_state_host")
    return fl, times


HB_ACT_CAPACITY = 16
HB_WBC_WEIGHTED, HB_WBC_HIERARCHICAL = 0, 1
WBC_FORMULATIONS = {"weighted": HB_WBC_WEIGHTED, "hierarchical": HB_WBC_HIERARCHICAL}
HB_HOQP_MAX_LEVELS, HB_HOQP_N, HB_HOQP_MAX_EQ, HB_HOQP_MAX_IN, HB_HOQP_MAX_STACKED = 3, 38, 32, 40, 80


class HbHoqpProblem(C.Structure):
    _fields_ = [("n", C.c_int32), ("levels", C.c_int32), ("ma", C.c_int32 * HB_HOQP_MAX_LEVELS), ("md", C.c_int32 * HB_HOQP_MAX_LEVELS),
                ("a", ((C.c_double * HB_HOQP_N) * HB_HOQP_MAX_EQ) * HB_HOQP_MAX_LEVELS), ("b", (C.c_double * HB_HOQP_MAX_EQ) * HB_HOQP_MAX_LEVELS),
                ("d", ((C.c_double * HB_HOQP_N) * HB_HOQP_MAX_IN) * HB_HOQP_MAX_LEVELS), ("f", (C.c_double * HB_HOQP_MAX_IN) * HB_HOQP_MAX_LEVELS)]


def make_hoqp_problems(hierarchies):
    """hierarchies: list (one per instance) of lists of tasks (a, b, d, f) by decreasing priority -> ctypes array of HbHoqpProblem."""
    pbs = (HbHoqpProblem * len(hierarchies))()
    for pb, levels in zip(np.ctypeslib.as_array(pbs), hierarchies):
        pb["levels"] = len(levels)
        for l, (a, b, d, f) in enumerate(levels):
            a, d = _task_matrix(a), _task_matrix(d)
            pb["ma"][l], pb["md"][l] = len(a), len(d)
            pb["n"] = max(pb["n"], a.shape[1], d.shape[1])
            if len(a):
                pb["a"][l, :len(a), :a.shape[1]] = a; pb["b"][l, :len(a)] = b[:len(a)]
            if len(d):
                pb["d"][l, :len(d), :d.shape[1]] = d; pb["f"][l, :len(d)] = f[:len(d)]
    return pbs


def _task_matrix(m):
    """a or d of a task as a float matrix; None or an empty matrix has no rows and no columns."""
    m = np.zeros((0, 0)) if m is None else np.atleast_2d(np.asarray(m, dtype=float))
    return m if m.size else np.zeros((0, 0))


def hoqp_tasks(pb):
    """HbHoqpProblem -> list of (a, b, d, f) numpy tasks."""
    p = np.ctypeslib.as_array(pb)
    n, levels = int(p["n"]), int(p["levels"])
    return [(p["a"][l, :ma, :n].copy(), p["b"][l, :ma].copy(), p["d"][l, :md, :n].copy(), p["f"][l, :md].copy())
            for l, (ma, md) in enumerate(zip(p["ma"][:levels], p["md"][:levels]))]


class HbActuationState(C.Structure):
    _fields_ = [("count", C.c_int32), ("head", C.c_int32), ("stamp", C.c_double * HB_ACT_CAPACITY), ("cmd", (C.c_double * 50) * HB_ACT_CAPACITY)]


class HbSimParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("substeps", C.c_int32), ("ground_height", C.c_double), ("ground_stiffness", C.c_double), ("ground_damping", C.c_double),
                ("tangential_damping", C.c_double), ("friction_mu", C.c_double), ("joint_armature", C.c_double), ("joint_damping", C.c_double)]


def make_channels(B, rows, names=None, device="cuda"):
    """Zeroed buffers for Context.set_channels: {name: torch tensor (B, rows, width) of the channel's type} for each name of `names`
    (default: every channel of CHANNELS). rows = ceil(n_ticks / log_every) records an episode call of n_ticks ticks."""
    import torch
    names = list(CHANNELS) if names is None else list(names)
    for n in names:
        if n not in CHANNELS:
            raise ValueError("unknown channel %r (one of %s)" % (n, ", ".join(CHANNELS)))
    return {n: torch.zeros((B, rows, CHANNELS[n][2]), dtype=getattr(torch, np.dtype(CHANNELS[n][1]).name), device=device) for n in names}


def default_sim_params():
    p = HbSimParams()
    _check(load_library().hb_default_sim_params(C.byref(p)), "hb_default_sim_params")
    return p


def actuation_states(B):
    st = (HbActuationState * B)()
    _check(load_library().hb_actuation_reset(B, st), "hb_actuation_reset")
    return st


HB_ROLLOUT_MAX_CMDS = 8
ROLLOUT_FAIL = {"estop": 1, "orientation": 2, "height": 4, "nonfinite": 8}     # hb_rollout_stats.fail_reason bits


class HbRolloutCommand(C.Structure):
    _fields_ = [("gait", C.c_int32), ("gait_start", C.c_double), ("n_cmd", C.c_int32), ("cmd_time", C.c_double * HB_ROLLOUT_MAX_CMDS),
                ("cmd_vel", (C.c_double * 4) * HB_ROLLOUT_MAX_CMDS)]


class HbRolloutParams(C.Structure):
    _fields_ = [("period", C.c_double), ("mpc_every", C.c_int32), ("actuation_delay", C.c_double), ("sim", HbSimParams), ("gains", HbPdGains),
                ("torque_limit", C.c_double * 10), ("min_base_height", C.c_double), ("log_every", C.c_int32)]


class HbRolloutStats(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("fail_tick", "fail_reason", "mpc_bad", "wbc_fallbacks", "plan_rejects")] + [("max_abs_torque", C.c_double)]


ROLLOUT_STATS_DTYPE = np.dtype(HbRolloutStats)


def default_rollout_params():
    p = HbRolloutParams()
    _check(load_library().hb_default_rollout_params(C.byref(p)), "hb_default_rollout_params")
    return p


def rollout_stats(B):
    """Stats of B fresh episodes: zeros, fail_tick = -1."""
    st = np.zeros(B, dtype=ROLLOUT_STATS_DTYPE)
    st["fail_tick"] = -1
    return st


def make_rollout_commands(gait, gait_start, cmd_times, cmd_vels):
    """ctypes array of HbRolloutCommand. cmd_vels: [n, 4] (one schedule for the batch) or [B, n, 4]; cmd_times: [n] or [B, n], ascending;
    gait (name or id) and gait_start: one for the batch or one per instance. cmd_vels[.., j, :] holds from cmd_times[.., j] on."""
    vel = _f64(cmd_vels)
    tim = _f64(cmd_times)
    sizes = [vel.shape[0] if vel.ndim == 3 else 1, tim.shape[0] if tim.ndim == 2 else 1, np.size(gait_start)]
    if not isinstance(gait, str) and np.ndim(gait) > 0:
        sizes.append(len(gait))
    B = max(sizes)
    n = vel.shape[-2]
    if not 1 <= n <= HB_ROLLOUT_MAX_CMDS or tim.shape[-1] != n:
        raise ValueError("cmd_times / cmd_vels: 1..%d segments of the same count expected" % HB_ROLLOUT_MAX_CMDS)
    vel = np.broadcast_to(vel, (B, n, 4)); tim = np.broadcast_to(tim, (B, n))
    gids = _gait_ids(gait, B); start = np.broadcast_to(_f64(gait_start), (B,))
    cmds = (HbRolloutCommand * B)()
    v = np.ctypeslib.as_array(cmds)
    v["gait"] = gids; v["gait_start"] = start; v["n_cmd"] = n
    v["cmd_time"][:, :n] = tim; v["cmd_vel"][:, :n] = vel
    return cmds


HB_MAX_PUSHES = 4


class HbPushSchedule(C.Structure):
    _fields_ = [("n_push", C.c_int32), ("t_start", C.c_double * HB_MAX_PUSHES), ("duration", C.c_double * HB_MAX_PUSHES),
                ("force", (C.c_double * 3) * HB_MAX_PUSHES), ("torque", (C.c_double * 3) * HB_MAX_PUSHES)]


def make_push_schedules(B, t_start, duration, force, torque=None):
    """ctypes array of B HbPushSchedule (Context.set_pushes). Push j of instance i acts on the plant steps of the ticks with
    t_start[i, j] <= t < t_start[i, j] + duration[i, j]: a world force[i, j] [N] at the base origin plus a world couple torque[i, j] [N m]
    (None: zero). t_start / duration: (B, n), (n,) or scalars; force / torque: (B, n, 3), (n, 3) or (3,); n <= HB_MAX_PUSHES. Raises
    ValueError for a shape that does not broadcast and for a record hb_rollout_set_pushes rejects (its own check)."""
    tim, dur, frc = _f64(t_start), _f64(duration), _f64(force)
    trq = np.zeros(3) if torque is None else _f64(torque)
    dims = [a.shape[-1] for a in (tim, dur) if a.ndim >= 1] + [a.shape[-2] for a in (frc, trq) if a.ndim >= 2]
    n = max(dims) if dims else 1
    if not 0 <= n <= HB_MAX_PUSHES:
        raise ValueError("push schedules: at most %d pushes per instance, got %d" % (HB_MAX_PUSHES, n))
    try:
        tim = np.broadcast_to(tim, (B, n)); dur = np.broadcast_to(dur, (B, n))
        frc = np.broadcast_to(frc, (B, n, 3)); trq = np.broadcast_to(trq, (B, n, 3))
    except ValueError as e:
        raise ValueError("push schedules: t_start / duration (B, n), force / torque (B, n, 3) expected: %s" % e)
    out = (HbPushSchedule * B)()
    v = np.ctypeslib.as_array(out)
    v["n_push"] = n
    v["t_start"][:, :n] = tim; v["duration"][:, :n] = dur; v["force"][:, :n] = frc; v["torque"][:, :n] = trq
    return _check_records(HB_SETTING_PUSHES, out, "pushes")


class HbPlantVariation(C.Structure):
    _fields_ = [("payload_mass", C.c_double), ("payload_com", C.c_double * 3), ("payload_inertia", C.c_double * 9), ("friction_scale", C.c_double),
                ("stiffness_scale", C.c_double), ("damping_scale", C.c_double), ("motor_strength", C.c_double * NJ)]


def default_plant_variation():
    """hb_default_plant_variation: the nominal plant (no payload, every scale 1)."""
    v = HbPlantVariation()
    _check(load_library().hb_default_plant_variation(C.byref(v)), "hb_default_plant_variation")
    return v


def make_plant_variations(B, payload_mass=0.0, payload_com=(0.0, 0.0, 0.0), payload_inertia=None, friction_scale=1.0, stiffness_scale=1.0,
                          damping_scale=1.0, motor_strength=1.0):
    """ctypes array of B HbPlantVariation (Context.set_plant_variations, Context.sim_step). Instance i carries a payload of payload_mass[i]
    [kg] with its CoM at payload_com[i] (base frame, from the base origin) and inertia payload_inertia[i] (3 x 3 about the CoM, base frame;
    None: zero), on ground of friction_scale[i] * mu, stiffness_scale[i] * k and damping_scale[i] * d, with motor_strength[i, j] scaling the
    torque of joint j. Scalars and per-instance arrays broadcast: masses and scales () or (B,), payload_com (3,) or (B, 3), payload_inertia
    (3, 3) or (B, 3, 3), motor_strength (), (10,) or (B, 10) (per instance only: (B, 1)). Raises ValueError for a
    shape that does not broadcast and for a record hb_rollout_set_plant_variations rejects (its own check). The defaults give the nominal
    plant."""
    try:
        m = np.broadcast_to(_f64(payload_mass), (B,)); c = np.broadcast_to(_f64(payload_com), (B, 3))
        I = np.broadcast_to(np.zeros((3, 3)) if payload_inertia is None else _f64(payload_inertia), (B, 3, 3))
        fs, ks, ds = (np.broadcast_to(_f64(x), (B,)) for x in (friction_scale, stiffness_scale, damping_scale))
        ms = np.broadcast_to(_f64(motor_strength), (B, NJ))
    except ValueError as e:
        raise ValueError("plant variations: masses / scales (B,), payload_com (B, 3), payload_inertia (B, 3, 3), motor_strength (B, 10) expected: %s"
                         % e)
    out = (HbPlantVariation * B)()
    v = np.ctypeslib.as_array(out)
    v["payload_mass"] = m; v["payload_com"] = c; v["payload_inertia"] = I.reshape(B, 9)
    v["friction_scale"] = fs; v["stiffness_scale"] = ks; v["damping_scale"] = ds; v["motor_strength"] = ms
    return _check_records(HB_SETTING_PLANT_VARIATIONS, out, "plant_variations")


NBODY = 11             # the model's bodies: 0 base (+imu), 1-5 leg_l1..l5, 6-10 leg_r1..r5 (l5, r5 with their toe and heel)


class HbLinkVariation(C.Structure):
    SETTING_KIND = 13        # HB_SETTING_LINK_VARIATIONS, the record's kind for hb_check_setting_records
    _fields_ = [("mass_scale", C.c_double * NBODY), ("com_shift", (C.c_double * 3) * NBODY), ("inertia_scale", C.c_double * NBODY)]


def default_link_variation():
    """hb_default_link_variation: the nominal bodies (every scale 1, every shift 0)."""
    r = HbLinkVariation()
    _check(load_library().hb_default_link_variation(C.byref(r)), "hb_default_link_variation")
    return r


def make_link_variations(B, mass_scale=1.0, com_shift=0.0, inertia_scale=1.0):
    """ctypes array of B HbLinkVariation (Context.set_link_variations, Context.sim_step): body b of robot i has mass mass_scale[i, b] m_b,
    CoM c_b + com_shift[i, b] (body frame [m]) and inertia inertia_scale[i, b] I_b about it. Scalars and arrays broadcast over robot x body:
    the scales (), (11,) or (B, 11) (per robot only: (B, 1)), com_shift (), (3,), (11, 3) or (B, 11, 3). Raises ValueError for a shape that
    does not broadcast and for a record hb_rollout_set_link_variations rejects (its own check). The defaults give the nominal bodies."""
    try:
        ms = np.broadcast_to(_f64(mass_scale), (B, NBODY)); cs = np.broadcast_to(_f64(com_shift), (B, NBODY, 3))
        js = np.broadcast_to(_f64(inertia_scale), (B, NBODY))
    except ValueError as e:
        raise ValueError("link variations: mass_scale / inertia_scale (B, 11), com_shift (B, 11, 3) expected: %s" % e)
    out = (HbLinkVariation * B)()
    v = np.ctypeslib.as_array(out)
    v["mass_scale"] = ms; v["com_shift"] = cs; v["inertia_scale"] = js
    return _check_records(HbLinkVariation.SETTING_KIND, out, "link_variations")


class HbJointModel(C.Structure):
    SETTING_KIND = 21        # HB_SETTING_JOINT_MODELS, the record's kind for hb_check_setting_records
    _fields_ = [("friction_loss", C.c_double * NJ), ("friction_velocity", C.c_double), ("lower", C.c_double * NJ), ("upper", C.c_double * NJ),
                ("stop_stiffness", C.c_double), ("stop_damping", C.c_double)]


def default_joint_model():
    """hb_default_joint_model: the reference's joints (friction loss 0.2 N m, range stops at HB_JOINT_LOWER / HB_JOINT_UPPER) with
    v_s = 0.01 rad/s and the stop gains of MuJoCo's default solref and solimp."""
    r = HbJointModel()
    _check(load_library().hb_default_joint_model(C.byref(r)), "hb_default_joint_model")
    return r


def make_joint_models(B, friction_loss=None, friction_velocity=None, lower=None, upper=None, stop_stiffness=None, stop_damping=None):
    """ctypes array of B HbJointModel (Context.set_joint_models, Context.sim_step): each robot's friction loss f [N m] and regularisation
    velocity v_s [rad/s], its stop range [lower, upper] [rad] (+-inf: no stop on that side) and the stop's gains k [1/s^2], b [1/s]. A
    field not given is default_joint_model()'s. Per-joint fields broadcast from (), (10,) or (B, 10) (per robot only: (B, 1)), the others
    from () or (B,). Raises ValueError for a shape that does not broadcast and for a record hb_rollout_set_joint_models rejects (its own
    check); the stability rule against the plant's params is checked by the plant step and the episode calls."""
    d = np.ctypeslib.as_array(default_joint_model())
    fields = dict(friction_loss=friction_loss, friction_velocity=friction_velocity, lower=lower, upper=upper, stop_stiffness=stop_stiffness,
                  stop_damping=stop_damping)
    out = (HbJointModel * B)()
    v = np.ctypeslib.as_array(out)
    for name, x in fields.items():
        shape = (B,) + d[name].shape
        try:
            v[name] = np.broadcast_to(d[name] if x is None else _f64(x), shape)
        except ValueError as e:
            raise ValueError("joint models: %s %s expected: %s" % (name, shape, e))
    return _check_records(HbJointModel.SETTING_KIND, out, "joint_models")


HB_TERRAIN_MAX = 64


HEIGHT_MAPS_SETTING_KIND = 14     # HB_SETTING_HEIGHT_MAPS: HbTerrain records as planner height maps (Context.set_height_maps), for hb_check_setting_records
ESTIMATOR_MAPS_SETTING_KIND = 15  # HB_SETTING_ESTIMATOR_MAPS: HbTerrain records as estimator maps (Context.set_estimator_maps), for hb_check_setting_records
MPC_MAPS_SETTING_KIND = 17        # HB_SETTING_MPC_MAPS: HbTerrain records as MPC maps (Context.set_mpc_maps), for hb_check_setting_records
WBC_MAPS_SETTING_KIND = 18        # HB_SETTING_WBC_MAPS: HbTerrain records as WBC maps (Context.set_wbc_maps), for hb_check_setting_records
MPC_CONE_MAPS_SETTING_KIND = 19   # HB_SETTING_MPC_CONE_MAPS: HbTerrain records as MPC cone maps (Context.set_mpc_cone_maps), for hb_check_setting_records


class HbTerrain(C.Structure):
    _fields_ = [("nx", C.c_int32), ("ny", C.c_int32), ("origin", C.c_double * 2), ("spacing", C.c_double),
                ("height", (C.c_double * HB_TERRAIN_MAX) * HB_TERRAIN_MAX)]


def make_terrains(B, heights, spacing, origin=(0.0, 0.0)):
    """ctypes array of B HbTerrain (Context.set_terrains, Context.sim_step). Instance i stands on the height field heights[i] (ny x nx,
    2..HB_TERRAIN_MAX each): heights[i][j, k] is the ground z at world (origin[i][0] + k spacing[i], origin[i][1] + j spacing[i]),
    interpolated bilinearly between the samples and continued flat beyond the grid's edges. heights (ny, nx) or (B, ny, nx), spacing () or
    (B,), origin (2,) or (B, 2). Raises ValueError for a shape that does not broadcast and for a record hb_rollout_set_terrains rejects
    (its own check)."""
    h = _f64(heights)
    if h.ndim not in (2, 3):
        raise ValueError("terrains: heights (ny, nx) or (B, ny, nx) expected, got shape %s" % (h.shape,))
    ny, nx = h.shape[-2:]
    if not (2 <= nx <= HB_TERRAIN_MAX and 2 <= ny <= HB_TERRAIN_MAX):
        raise ValueError("terrains: 2..%d samples along x and y, got %d x %d" % (HB_TERRAIN_MAX, ny, nx))
    try:
        h = np.broadcast_to(h, (B, ny, nx)); s = np.broadcast_to(_f64(spacing), (B,)); o = np.broadcast_to(_f64(origin), (B, 2))
    except ValueError as e:
        raise ValueError("terrains: heights (B, ny, nx), spacing (B,), origin (B, 2) expected: %s" % e)
    out = (HbTerrain * B)()
    v = np.ctypeslib.as_array(out)
    v["nx"] = nx; v["ny"] = ny; v["origin"] = o; v["spacing"] = s
    v["height"][:, :ny, :nx] = h
    return _check_records(HB_SETTING_TERRAINS, out, "terrains")


HB_MAX_GOALS = 8


class HbGoalSchedule(C.Structure):
    _fields_ = [("n_goal", C.c_int32), ("time", C.c_double * HB_MAX_GOALS), ("goal", (C.c_double * 3) * HB_MAX_GOALS)]


def make_goal_schedules(B, times, goals):
    """ctypes array of B HbGoalSchedule (Context.set_goals). Goal j of instance i, the world pose goals[i, j] = (x, y, yaw), comes into
    force on the first MPC tick with t >= times[i, j]. times: (B, n), (n,) or a scalar, ascending; goals: (B, n, 3), (n, 3) or (3,);
    n <= HB_MAX_GOALS (n = 0: no goals). Raises ValueError for a shape that does not broadcast and for a record hb_rollout_set_goals
    rejects (its own check)."""
    tim, gol = _f64(times), _f64(goals)
    dims = [tim.shape[-1]] if tim.ndim >= 1 else []
    dims += [gol.shape[-2]] if gol.ndim >= 2 else []
    n = max(dims) if dims else 1
    if not 0 <= n <= HB_MAX_GOALS:
        raise ValueError("goal schedules: at most %d goals per instance, got %d" % (HB_MAX_GOALS, n))
    try:
        tim = np.broadcast_to(tim, (B, n)); gol = np.broadcast_to(gol, (B, n, 3))
    except ValueError as e:
        raise ValueError("goal schedules: times (B, n), goals (B, n, 3) expected: %s" % e)
    out = (HbGoalSchedule * B)()
    v = np.ctypeslib.as_array(out)
    v["n_goal"] = n
    v["time"][:, :n] = tim; v["goal"][:, :n] = gol
    return _check_records(HB_SETTING_GOALS, out, "goals")


class HbObserverState(C.Structure):
    _fields_ = [("p_filtered", C.c_double * 16)]


def observer_states(B):
    """Freshly reset momentum-observer states (pSCgZinvlast_ = 0)."""
    st = (HbObserverState * B)()
    _check(load_library().hb_observer_reset(B, st), "hb_observer_reset")
    return st


def default_kf_params():
    p = HbKfParams()
    _check(load_library().hb_default_kf_params(C.byref(p)), "hb_default_kf_params")
    return p


def kf_states(B):
    """Freshly reset filter states (x_hat = 0, P = 100 I)."""
    st = (HbKfState * B)()
    _check(load_library().hb_kf_reset(B, st), "hb_kf_reset")
    return st


class HbSensorNoise(C.Structure):
    _fields_ = [("seed", C.c_uint64)] + [(k, C.c_double) for k in ("orientation", "angular_velocity", "linear_acceleration", "joint_position",
                                                                   "joint_velocity")]


class HbEstimationParams(C.Structure):
    _fields_ = [("kf", HbKfParams), ("noise", HbSensorNoise)]


class HbEstimationState(C.Structure):
    _fields_ = [("kf", HbKfState), ("noise_stream", C.c_uint64), ("base_vel_prev", C.c_double * 3), ("primed", C.c_int32), ("yaw_obs", C.c_double),
                ("has_plan", C.c_int32), ("n_events", C.c_int32), ("event_times", C.c_double * HB_MAX_EVENTS), ("modes", C.c_int32 * (HB_MAX_EVENTS + 1))]


class HbEstimationStats(C.Structure):
    _fields_ = [(k, C.c_double) for k in ("max_vel_err", "max_height_err", "sum_sq_vel_err", "sum_sq_height_err")] + [("count", C.c_int32)]


ESTIMATION_STATS_DTYPE = np.dtype(HbEstimationStats)


def default_estimation_params():
    """Default filter (hb_default_kf_params), no sensor noise, seed 0."""
    p = HbEstimationParams()
    _check(load_library().hb_default_estimation_params(C.byref(p)), "hb_default_estimation_params")
    return p


def estimation_states(B, first_stream=0):
    """Fresh estimation states (filter reset, noise stream first_stream + i, unprimed accelerometer, no plan, yaw_obs = 0)."""
    st = (HbEstimationState * B)()
    _check(load_library().hb_estimation_reset(B, C.c_uint64(first_stream), st), "hb_estimation_reset")
    return st


def estimation_stats(B):
    """Estimation stats of B fresh episodes: zeros."""
    return np.zeros(B, dtype=ESTIMATION_STATS_DTYPE)


class HbControllerSetting(C.Structure):
    _fields_ = [("wbc", HbWbcSettings), ("gains", HbPdGains)]


def make_controller_settings(B, wbc=None, gains=None, **fields):
    """ctypes array of B HbControllerSetting (Context.set_controller_settings): each robot's WBC settings and joint PD gains in the episodes.
    wbc (HbWbcSettings) and gains (HbPdGains) are the base of every record, default hb_default_wbc_settings and default_pd_gains(). Any field
    of either struct can be given by name, as a scalar or a (B,) array; torque_limits as (5,) or (B, 5). Raises ValueError for an unknown
    name or a shape that does not broadcast."""
    lib = load_library()
    if wbc is None:
        wbc = HbWbcSettings()
        _check(lib.hb_default_wbc_settings(C.byref(wbc)), "hb_default_wbc_settings")
    gains = default_pd_gains() if gains is None else gains
    out = (HbControllerSetting * B)()
    v = np.ctypeslib.as_array(out)
    v["wbc"] = np.frombuffer(bytes(wbc), dtype=v.dtype["wbc"])[0]
    v["gains"] = np.frombuffer(bytes(gains), dtype=v.dtype["gains"])[0]
    for name, value in fields.items():
        part = "wbc" if name in v.dtype["wbc"].names else "gains" if name in v.dtype["gains"].names else None
        if part is None:
            raise ValueError("controller settings: unknown field %r" % name)
        shape = (B, 5) if name == "torque_limits" else (B,)
        try:
            v[part][name] = np.broadcast_to(_f64(value), shape)
        except ValueError as e:
            raise ValueError("controller settings: %s: %s expected: %s" % (name, "(5,) or (B, 5)" if shape[1:] else "(B,) or a scalar", e))
    return out


class HbHardwareSetting(C.Structure):
    _fields_ = [("actuation_delay", C.c_double), ("torque_limit", C.c_double * NJ)] + \
        [(k, C.c_double) for k in ("sigma_orientation", "sigma_angular_velocity", "sigma_linear_acceleration", "sigma_joint_position",
                                   "sigma_joint_velocity")] + \
        [(k, C.c_double * 3) for k in ("orientation_offset", "gyro_bias", "accel_bias")] + [("encoder_offset", C.c_double * NJ)]


def default_hardware_setting():
    """hb_default_hardware_setting: the default episode's actuation delay and torque limits, no sensor noise, no offsets."""
    s = HbHardwareSetting()
    _check(load_library().hb_default_hardware_setting(C.byref(s)), "hb_default_hardware_setting")
    return s


def make_hardware_settings(B, base=None, **fields):
    """ctypes array of B HbHardwareSetting (Context.set_hardware): each robot's simulated hardware in the episodes. base (HbHardwareSetting,
    default default_hardware_setting()) is the base of every record. Any field can be given by name, as a scalar or a (B,) array;
    torque_limit and encoder_offset as (10,) or (B, 10), orientation_offset, gyro_bias and accel_bias as (3,) or (B, 3). Raises ValueError
    for an unknown name or a shape that does not broadcast; the ranges are checked by the setter."""
    base = default_hardware_setting() if base is None else base
    out = (HbHardwareSetting * B)()
    v = np.ctypeslib.as_array(out)
    v[:] = np.frombuffer(bytes(base), dtype=v.dtype)[0]
    for name, value in fields.items():
        if name not in v.dtype.names:
            raise ValueError("hardware settings: unknown field %r" % name)
        shape = (B,) + v.dtype[name].shape
        try:
            v[name] = np.broadcast_to(_f64(value), shape)
        except ValueError as e:
            raise ValueError("hardware settings: %s: %s expected: %s" % (name, "(%d,) or (B, %d)" % (shape[1], shape[1]) if shape[1:] else "(B,) or a scalar", e))
    return out


class HbMotorBridge(C.Structure):
    SETTING_KIND = 11        # HB_SETTING_MOTOR_BRIDGE, the record's kind for hb_check_setting_records
    _fields_ = [("command_scale", C.c_double * NJ), ("direction", C.c_int32 * NJ), ("zero", C.c_double * NJ)] + \
        [(k, C.c_double * NJ) for k in ("kp_max", "kd_max", "pos_max", "vel_max", "ff_max")] + [("quantise", C.c_int32)]


def default_motor_bridge():
    """hb_default_motor_bridge: the real Hunter's joint path (legged_bridge_hw): the 0.7 command scale on joints 0, 1, 5, 6, its motor
    directions, zero offsets 0, the protocol ranges of each joint's X or D motor, and the protocol's quantisation."""
    r = HbMotorBridge()
    _check(load_library().hb_default_motor_bridge(C.byref(r)), "hb_default_motor_bridge")
    return r


def make_motor_bridges(B, base=None, **fields):
    """ctypes array of B HbMotorBridge (Context.set_motor_bridge): each robot's joint path through the motor driver in the episodes. base
    (HbMotorBridge, default default_motor_bridge()) is the base of every record. Any field can be given by name: quantise as a scalar or
    a (B,) array, the others as a scalar, (10,) or (B, 10). Raises ValueError for an unknown name, a shape that does not broadcast, a
    direction or quantise that is not an integer, and a record hb_rollout_set_motor_bridge rejects."""
    base = default_motor_bridge() if base is None else base
    out = (HbMotorBridge * B)()
    v = np.ctypeslib.as_array(out)
    v[:] = np.frombuffer(bytes(base), dtype=v.dtype)[0]
    for name, value in fields.items():
        if name not in v.dtype.names:
            raise ValueError("motor bridges: unknown field %r" % name)
        shape = (B,) + v.dtype[name].shape
        try:
            x = np.broadcast_to(np.asarray(value, dtype=np.float64), shape)
        except ValueError as e:
            raise ValueError("motor bridges: %s: %s expected: %s" % (name, "(10,) or (B, 10)" if shape[1:] else "(B,) or a scalar", e))
        if v.dtype[name].base.kind == "i" and not (np.isfinite(x).all() and (x == np.rint(x)).all() and (np.abs(x) < 2 ** 31).all()):
            raise ValueError("motor bridges: %s: int32 integers expected" % name)
        v[name] = x
    return _check_records(HbMotorBridge.SETTING_KIND, out, "motor_bridge")


def _bridge_records(bridge, B, what):
    """bridge (a ctypes array or a sequence of B HbMotorBridge) as a ctypes array (None stays None), or ValueError."""
    if bridge is None:
        return None
    if len(bridge) != B:
        raise ValueError("%s: %d motor bridges for %d robots" % (what, len(bridge), B))
    return bridge if isinstance(bridge, C.Array) else (HbMotorBridge * B)(*bridge)


def bridge_encode(bridge, command):
    """The motor bridge's command codec on the host (hb_motor_bridge_encode): command [B,10,5] (joint frame: pos_des, vel_des, kp, kd, ff)
    -> the decoded motor command [B,10,5] (motor frame: pos, vel, kp, kd, ff) of the records bridge (B HbMotorBridge)."""
    command = _f64(command).reshape(-1, NJ, 5)
    B = command.shape[0]
    out = np.zeros((B, NJ, 5))
    _check(load_library().hb_motor_bridge_encode(B, _bridge_records(bridge, B, "bridge_encode"), _ptr(command), _ptr(out)), "hb_motor_bridge_encode")
    return out


def bridge_feedback(bridge, q, qd):
    """The motor bridge's encoders on the host (hb_motor_bridge_feedback): joint readings q, qd [B,10] -> what the driver reports back in
    the joint frame, (q_out, qd_out)."""
    q, qd = _f64(q).reshape(-1, NJ), _f64(qd).reshape(-1, NJ)
    B = q.shape[0]
    q_out, qd_out = np.zeros((B, NJ)), np.zeros((B, NJ))
    _check(load_library().hb_motor_bridge_feedback(B, _bridge_records(bridge, B, "bridge_feedback"), _ptr(q), _ptr(qd), _ptr(q_out), _ptr(qd_out)),
           "hb_motor_bridge_feedback")
    return q_out, qd_out


HB_MAX_TELEOP_WINDOWS = 4
TELEOP_ALWAYS = 2 ** 31 - 1      # an off_tick that never comes (INT32_MAX)


class HbTeleopSetting(C.Structure):
    SETTING_KIND = 12        # HB_SETTING_TELEOP, the record's kind for hb_check_setting_records
    _fields_ = [("period_ticks", C.c_int32), ("n_window", C.c_int32), ("on_tick", C.c_int32 * HB_MAX_TELEOP_WINDOWS),
                ("off_tick", C.c_int32 * HB_MAX_TELEOP_WINDOWS), ("change_limit", C.c_double * 3)]


HbTeleop = HbTeleopSetting


def default_teleop_setting():
    """hb_default_teleop_setting: the reference's joystick and publisher: a message every 50 ticks (10 Hz), the deadman held from tick 0
    on, the change per message limited to 0.1 m/s, 0.05 m/s and 0.3 rad/s."""
    r = HbTeleopSetting()
    _check(load_library().hb_default_teleop_setting(C.byref(r)), "hb_default_teleop_setting")
    return r


def make_teleop_settings(B, period_ticks=50, windows=((0, TELEOP_ALWAYS),), change_limit=(0.1, 0.05, 0.3)):
    """ctypes array of B HbTeleopSetting (Context.set_teleop): each robot's joystick and target publisher in the episodes. period_ticks:
    (B,) or a scalar; windows: the absolute ticks [on, off) the deadman is held, (n, 2) for every robot, (B, n, 2), or a sequence of B
    (n_i, 2) sequences, n <= HB_MAX_TELEOP_WINDOWS (n = 0: no message ever); change_limit: the per-message change of vx, vy and yaw rate,
    (3,) or (B, 3) (inf: no limit). Raises ValueError for a shape that does not broadcast, a tick that is not an int32 integer and a record
    hb_rollout_set_teleop rejects (its own check)."""
    def ticks(a, shape, what):
        x = np.asarray(a, dtype=np.float64)
        try:
            x = np.broadcast_to(x, shape)
        except ValueError as e:
            raise ValueError("teleop settings: %s: %s expected: %s" % (what, shape, e))
        if not (np.isfinite(x).all() and (x == np.rint(x)).all() and (np.abs(x) < 2 ** 31).all()):
            raise ValueError("teleop settings: %s: int32 integers expected" % what)
        return x.astype(np.int32)
    w = None
    try:
        w = np.asarray(windows, dtype=np.float64)
    except ValueError:
        pass
    shape_error = ValueError("teleop settings: windows: (n, 2), (B, n, 2) or B sequences of (n_i, 2) expected")
    if w is not None and w.size == 0:                   # no window: no message ever
        per = [np.zeros((0, 2))] * B
    elif w is not None and w.ndim == 2 and w.shape[1] == 2:
        per = [w] * B
    elif w is not None and w.ndim == 3 and w.shape[0] == B and w.shape[2] == 2:
        per = list(w)
    elif w is None and len(windows) == B:
        per = [np.asarray(x, dtype=np.float64).reshape(-1, 2) for x in windows]
    else:
        raise shape_error
    if any(len(x) > HB_MAX_TELEOP_WINDOWS for x in per):
        raise ValueError("teleop settings: at most %d windows per robot" % HB_MAX_TELEOP_WINDOWS)
    out = (HbTeleopSetting * B)()
    v = np.ctypeslib.as_array(out)
    v["period_ticks"] = ticks(period_ticks, (B,), "period_ticks")
    for i, x in enumerate(per):
        x = ticks(x, x.shape, "windows")
        v["n_window"][i] = len(x)
        v["on_tick"][i, :len(x)] = x[:, 0]; v["off_tick"][i, :len(x)] = x[:, 1]
    try:
        v["change_limit"] = np.broadcast_to(_f64(change_limit), (B, 3))
    except ValueError as e:
        raise ValueError("teleop settings: change_limit: (3,) or (B, 3) expected: %s" % e)
    return _check_records(HbTeleopSetting.SETTING_KIND, out, "teleop")


HB_ODOM_MAX_DELAY = 15


class HbOdometrySetting(C.Structure):
    _fields_ = [("period_ticks", C.c_int32), ("delay_ticks", C.c_int32), ("sigma_position", C.c_double), ("sigma_drift", C.c_double)]


def make_odometry_settings(B, period_ticks, delay_ticks=0, sigma_position=0.0, sigma_drift=0.0):
    """ctypes array of B HbOdometrySetting (Context.set_odometry): the tracking camera of each robot of the estimated episodes, a message
    every period_ticks ticks (0: no camera) carrying the base position of delay_ticks ticks earlier (0..HB_ODOM_MAX_DELAY), with white noise
    sigma_position [m] and a bias whose random-walk increment per message is sigma_drift [m]. Each argument: (B,) or a scalar. Raises
    ValueError for a shape that does not broadcast, a tick count that is not an int32 integer and a record hb_rollout_set_odometry rejects
    (its own check)."""
    try:
        per, dly = (np.broadcast_to(np.asarray(a), (B,)) for a in (period_ticks, delay_ticks))
        sp, sd = (np.broadcast_to(_f64(a), (B,)) for a in (sigma_position, sigma_drift))
    except ValueError as e:
        raise ValueError("odometry settings: (B,) or scalars expected: %s" % e)
    out = (HbOdometrySetting * B)()
    v = np.ctypeslib.as_array(out)
    with np.errstate(invalid="ignore"):                 # a NaN or out-of-range tick count casts to garbage, rejected below
        v["period_ticks"] = per; v["delay_ticks"] = dly
    if not (np.array_equal(v["period_ticks"], per) and np.array_equal(v["delay_ticks"], dly)):
        raise ValueError("odometry settings: period_ticks and delay_ticks must be int32 integers")
    v["sigma_position"] = sp; v["sigma_drift"] = sd
    return _check_records(HB_SETTING_ODOMETRY, out, "odometry")


class HbGaitSelector(C.Structure):
    _fields_ = [("history", C.c_double * 50), ("vel_avg", C.c_double), ("head", C.c_int32), ("count", C.c_int32), ("gait_level", C.c_int32),
                ("reserved", C.c_int32)]


class GaitSelector:
    """Batch of speed-based gait selectors (SwitchedModelReferenceManager::calculateVelAbs + walkGait / trotGait)."""

    def __init__(self, B, gait_level=-1):
        self.B = B
        self.state = (HbGaitSelector * B)()
        np.ctypeslib.as_array(self.state)["gait_level"] = gait_level

    def update(self, cmd_vel, target_state0, gait_type=0):
        lib = load_library()
        cmd_vel = _f64(np.broadcast_to(_f64(cmd_vel), (self.B, 4))); ts = _f64(target_state0).reshape(self.B, 22)
        gt = np.ascontiguousarray(np.broadcast_to(np.asarray(gait_type, dtype=np.int32), (self.B,)))
        level = np.zeros(self.B, dtype=np.int32); insert = np.zeros(self.B, dtype=np.int32)
        _check(lib.hb_gait_select(self.B, self.state, _ptr(gt), _ptr(cmd_vel), _ptr(ts), _ptr(level), _ptr(insert)), "hb_gait_select")
        return level, insert

    @property
    def vel_avg(self):
        return np.ctypeslib.as_array(self.state)["vel_avg"].copy()


GAIT_IDS = {"stance": 0, "trot": 1, "standing_trot": 2, "flying_trot": 3}


def _gait_ids(gait, B):
    """Gait name (one for the batch) or any sequence / ndarray of names or ids (one per instance) -> int ids [B]."""
    if isinstance(gait, str):
        return [GAIT_IDS[gait]] * B
    if np.ndim(gait) == 0:
        return [int(gait)] * B
    ids = [GAIT_IDS[g] if isinstance(g, str) else int(g) for g in list(gait)]
    if len(ids) != B:
        raise ValueError("gait: expected one name or %d per-instance entries, got %d" % (B, len(ids)))
    return ids


def make_plan_inputs(t0, horizon, x0, cmd_vel, feet_pos, gait, gait_start, prev_event=None, time_to_target=None, joint_ik=True):
    """ctypes array of HbPlanInput for a batch (feet_pos may be None when the device computes it)."""
    x0 = _f64(x0); B = x0.shape[0]
    gids = _gait_ids(gait, B)
    cmd_vel = np.broadcast_to(_f64(cmd_vel), (B, 4))
    feet_pos = np.zeros((B, 12)) if feet_pos is None else _f64(feet_pos).reshape(B, 12)
    t0 = np.broadcast_to(_f64(t0), (B,)); gait_start = np.broadcast_to(_f64(gait_start), (B,))
    ins = (HbPlanInput * B)()
    v = np.ctypeslib.as_array(ins)
    v["t0"] = t0; v["horizon"] = horizon; v["time_to_target"] = horizon if time_to_target is None else time_to_target
    v["gait_start"] = gait_start; v["prev_event"] = (np.minimum(t0, gait_start) - 0.5) if prev_event is None else prev_event
    v["gait"] = gids
    v["joint_ik"] = 1 if joint_ik else 0
    v["x0"] = x0.reshape(B, 22); v["cmd_vel"] = cmd_vel; v["feet_pos"] = feet_pos
    return ins


def plan_set_threads(n):
    """Host threads of plan_references (0 = all); hb_plan_set_threads."""
    _check(load_library().hb_plan_set_threads(int(n)), "hb_plan_set_threads")


def plan_references(t0, horizon, x0, cmd_vel, feet_pos, gait, gait_start, prev_event=None, time_to_target=None, latest_stance=None, joint_ik=True,
                    targets=None, settings=None, maps=None):
    """Host-side reference planner (hb_plan_references): returns (ctypes array of HbReference, latest_stance[B,12]). targets: B HbTarget
    (make_targets, goal_to_target) planned on instead of the cmd_vel targets (hb_plan_references_targets); cmd_vel still drives the swing
    planner. settings: B HbPlannerSettings (make_planner_settings) in place of the compiled-in templates and swing settings
    (hb_plan_references_settings). maps: B HbTerrain (make_terrains), the height map each instance plans on (hb_plan_references_maps)."""
    lib = load_library()
    ins = make_plan_inputs(t0, horizon, x0, cmd_vel, feet_pos, gait, gait_start, prev_event, time_to_target, joint_ik)
    B = len(ins)
    if targets is not None and len(targets) != B:
        raise ValueError("plan_references: %d targets for %d instances" % (len(targets), B))
    if settings is not None and len(settings) != B:
        raise ValueError("plan_references: %d planner settings for %d instances" % (len(settings), B))
    ls = np.zeros((B, 12)) if latest_stance is None else _f64(latest_stance).copy()
    refs = (HbReference * B)()
    if maps is not None:
        _check(lib.hb_plan_references_maps(B, ins, targets, settings, _maps_of(maps, B, "plan_references"), _ptr(ls), refs), "hb_plan_references_maps")
    elif settings is None:
        _check(lib.hb_plan_references_targets(B, ins, targets, _ptr(ls), refs), "hb_plan_references_targets")
    else:
        _check(lib.hb_plan_references_settings(B, ins, targets, settings, _ptr(ls), refs), "hb_plan_references_settings")
    return refs, ls


class HunterB200Error(RuntimeError):
    pass


def load_library():
    """Load libhunter_b200.so. Raises if the CUDA extension has not been built (no CPU fallback exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise HunterB200Error("libhunter_b200.so is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                                  "(the product path has no CPU fallback)")
        _lib = C.CDLL(_LIB_PATH)
        _lib.hb_strerror.restype = C.c_char_p
        _lib.hb_last_cuda_error.restype = C.c_char_p
        _lib.hb_launch_count.restype = C.c_int64
        _lib.hb_last_reference_upload_bytes.restype = C.c_int64
        _lib.hb_episode_state_bytes.restype = C.c_int64
        _lib.hb_stream.restype = C.c_void_p
        _lib.hb_shard_last_error.restype = C.c_char_p
    return _lib


def _check(rc, what, ctx=None):
    if rc != 0:
        extra = ""
        if rc == -2 and ctx is not None:
            extra = ": " + load_library().hb_last_cuda_error(ctx).decode()
        raise HunterB200Error("%s failed: %s (%d)%s" % (what, load_library().hb_strerror(rc).decode(), rc, extra))


def _ptr(a):
    """Pointer of a numpy array (host) or of a torch tensor (host or cuda)."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return C.c_void_p(a.ctypes.data)
    return C.c_void_p(a.data_ptr())


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _check_records(kind, records, setting):
    """records, or ValueError naming the first that hb_rollout_set_<setting> rejects (hb_check_setting_records, its own check)."""
    bad = C.c_int32()
    if load_library().hb_check_setting_records(kind, len(records), records, C.byref(bad)) != 0:
        raise ValueError("%s: record %d is rejected by hb_rollout_set_%s" % (setting, bad.value, setting))
    return records


def reseed(est, first_stream):
    """Gives record i of the estimation states est (a tensor of B hb_estimation_state, as rollout_estimated takes) noise stream
    first_stream + i, in place; returns est. Forked estimated copies share their source's stream, so without this their sensor and camera
    noise stays identical. The noise an instance draws on absolute tick a is Philox4x32-10 under the key hb_sensor_noise.seed at the counter
    (block, a, noise_stream) and depends on nothing else, so a copy reseeded at the fork tick draws from then on exactly what an instance
    that had that stream from the start draws on those ticks."""
    import torch
    size, off = C.sizeof(HbEstimationState), HbEstimationState.noise_stream.offset
    rec = est.view(-1, size)
    streams = np.uint64(first_stream) + np.arange(rec.shape[0], dtype=np.uint64)
    rec[:, off:off + 8] = torch.from_numpy(streams.view(np.uint8).reshape(-1, 8)).to(est.device)
    return est


def _episode_index(src, B, n, what):
    """src as a list of B ints in [0, n) (None: 0 .. B-1), or ValueError."""
    idx = list(range(B)) if src is None else [int(i) for i in src]
    if len(idx) != B or not all(0 <= i < n for i in idx):
        raise ValueError("%s: %d instances from %s of %d" % (what, B, "0 .. B-1" if src is None else "src %s" % idx, n))
    return idx


def _gather(idx, rbd, act, estop, stats, est=None, est_stats=None):
    """Copies of instances idx of an episode's caller buffers: [rbd, act, estop, stats] and, with est, [est, est_stats]."""
    import torch
    t = torch.tensor(idx, dtype=torch.long, device=rbd.device)

    def take(x, size):
        return x.view(-1, size)[t].reshape(-1).clone()
    out = [rbd[t].clone(), take(act, C.sizeof(HbActuationState)), estop[t].clone(), np.asarray(stats)[idx].copy()]
    if est is not None:
        out += [take(est, C.sizeof(HbEstimationState)), np.asarray(est_stats)[idx].copy()]
    return out


class EpisodeSnapshot:
    """Episodes saved mid-way (Context.save_episodes): `rows`, the context state of each instance (a uint8 tensor (n, row bytes) on the
    device, hb_episode_save_async), and clones of the caller's buffers of the same instances: rbd (n, 32), act (n hb_actuation_state
    bytes), estop (n), stats (ROLLOUT_STATS_DTYPE), and for estimated episodes est (n hb_estimation_state bytes) and est_stats
    (ESTIMATION_STATS_DTYPE), None otherwise. Context.restore_episodes continues them, in this or another context of the same
    configuration; save / load keep them in an .npz file."""
    _TENSORS = ("rows", "rbd", "act", "estop", "est")

    def __init__(self, rows, rbd, act, estop, stats, est=None, est_stats=None):
        n = rows.shape[0]
        stats = np.asarray(stats, dtype=ROLLOUT_STATS_DTYPE)
        ok = (rows.dim() == 2 and tuple(rbd.shape) == (n, 32) and act.numel() == n * C.sizeof(HbActuationState) and tuple(estop.shape) == (n,)
              and stats.shape == (n,) and (est is None) == (est_stats is None))
        if ok and est is not None:
            est_stats = np.asarray(est_stats, dtype=ESTIMATION_STATS_DTYPE)
            ok = est.numel() == n * C.sizeof(HbEstimationState) and est_stats.shape == (n,)
        if not ok:
            raise ValueError("EpisodeSnapshot: the rows and the caller's buffers must hold the same instances (estimated: est and est_stats both)")
        self.rows, self.rbd, self.act, self.estop, self.stats, self.est, self.est_stats = rows, rbd, act, estop, stats, est, est_stats

    def __len__(self):
        return self.rows.shape[0]

    @property
    def estimated(self):
        return self.est is not None

    def save(self, path):
        """Writes the snapshot to the .npz file `path`."""
        arrays = {k: getattr(self, k).cpu().numpy() for k in self._TENSORS if getattr(self, k) is not None}
        arrays["stats"] = self.stats
        if self.estimated:
            arrays["est_stats"] = self.est_stats
        np.savez(path, **arrays)

    @classmethod
    def load(cls, path, device="cuda"):
        """The snapshot save wrote to `path`, its tensors on `device`."""
        import torch
        with np.load(path) as f:
            t = {k: torch.from_numpy(f[k]).to(device) for k in cls._TENSORS if k in f}
            return cls(t["rows"], t["rbd"], t["act"], t["estop"], f["stats"], t.get("est"), f["est_stats"] if "est_stats" in f else None)


def _check_hardware(what, hardware, B):
    if hardware is not None and len(hardware) != B:
        raise ValueError("%s: %d hardware settings for %d robots" % (what, len(hardware), B))


class Context:
    """Owner of one hb_ctx (one GPU, one stream). Single-owner: use it from one thread at a time."""

    def __init__(self, horizon_N=100, dt=0.01, max_batch=1024, device=0, wbc_rho=1e-8, qp_max_iter=40, line_search_max_trials=14, time_horizon=0.0,
                 event_nodes=False, e2e_chunks=0):
        lib = load_library()
        cfg = HbConfig()
        _check(lib.hb_default_config(C.byref(cfg)), "hb_default_config")
        cfg.horizon_N, cfg.dt, cfg.max_batch, cfg.wbc_rho = horizon_N, dt, max_batch, wbc_rho
        cfg.qp_max_iter, cfg.line_search_max_trials = qp_max_iter, line_search_max_trials
        cfg.time_horizon, cfg.event_nodes, cfg.e2e_chunks = float(time_horizon), 1 if event_nodes else 0, int(e2e_chunks)
        self.cfg = cfg
        self.N, self.dt, self.max_batch, self.device = horizon_N, dt, max_batch, device
        self._h = C.c_void_p()
        _check(lib.hb_create(C.byref(cfg), C.c_int(device), C.byref(self._h)), "hb_create")
        self._lib = lib

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.hb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        _check(self._lib.hb_sync(self._h), "hb_sync")

    # ------------------------------------------------------------------ run-time WBC settings (WbcBase::loadTasksSetting / setKpKd)
    def wbc_settings(self):
        s = HbWbcSettings()
        _check(self._lib.hb_wbc_get_settings(self._h, C.byref(s)), "hb_wbc_get_settings")
        return s

    def set_wbc_settings(self, s):
        _check(self._lib.hb_wbc_set_settings(self._h, C.byref(s)), "hb_wbc_set_settings")

    def set_kp_kd(self, swing_kp, swing_kd):
        _check(self._lib.hb_wbc_set_kp_kd(self._h, C.c_double(swing_kp), C.c_double(swing_kd)), "hb_wbc_set_kp_kd")

    def load_task_info(self, path):
        _check(self._lib.hb_load_task_info(self._h, str(path).encode()), "hb_load_task_info")

    def set_wbc_formulation(self, name):
        """The controller's WBC for every entry point that runs it: "weighted" (WeightedWbc, the default) or "hierarchical" (HierarchicalWbc)."""
        if name not in WBC_FORMULATIONS:
            raise ValueError("unknown WBC formulation %r (one of %s)" % (name, ", ".join(WBC_FORMULATIONS)))
        _check(self._lib.hb_wbc_set_formulation(self._h, C.c_int32(WBC_FORMULATIONS[name])), "hb_wbc_set_formulation")

    def wbc_formulation(self):
        f = C.c_int32()
        _check(self._lib.hb_wbc_get_formulation(self._h, C.byref(f)), "hb_wbc_get_formulation")
        return {v: k for k, v in WBC_FORMULATIONS.items()}[f.value]

    @property
    def launch_count(self):
        return int(self._lib.hb_launch_count(self._h))

    def profile_enable(self, on=True):
        _check(self._lib.hb_profile_enable(self._h, int(on)), "hb_profile_enable", self._h)

    def profile_read(self):
        ms = np.zeros(7); cnt = np.zeros(7, dtype=np.int64)
        _check(self._lib.hb_profile_read(self._h, _ptr(ms), _ptr(cnt)), "hb_profile_read", self._h)
        names = ["mpc_riccati", "mpc_forward_linesearch", "wbc_assemble", "qp_ipm", "other", "mpc_linearise", "mpc_lq_project"]
        return {n: dict(ms=float(m), launches=int(c)) for n, m, c in zip(names, ms, cnt)}

    @property
    def last_reference_upload_bytes(self):
        return int(self._lib.hb_last_reference_upload_bytes(self._h))

    @property
    def stream_handle(self):
        return int(self._lib.hb_stream(self._h) or 0)

    # ------------------------------------------------------------------ host-pointer calls (numpy in / numpy out)
    def wbc_qp(self, H, g, A, lbA, ubA):
        H, g, A, lbA, ubA = map(_f64, (H, g, A, lbA, ubA))
        B, n = g.shape
        m = lbA.shape[1]
        x = np.zeros((B, n)); st = np.zeros(B, dtype=np.int32); it = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_wbc_qp_batch(self._h, B, n, m, _ptr(H), _ptr(g), _ptr(A), _ptr(lbA), _ptr(ubA), _ptr(x), _ptr(st), _ptr(it)), "hb_wbc_qp_batch", self._h)
        return x, st, it

    def wbc_solve(self, x_des, u_des, rbd, mode, stance_mode=None):
        x_des, u_des, rbd = map(_f64, (x_des, u_des, rbd))
        B = x_des.shape[0]
        mode = np.ascontiguousarray(mode, dtype=np.int32)
        sm = None if stance_mode is None else np.ascontiguousarray(stance_mode, dtype=np.uint8)
        sol = np.zeros((B, NWBC)); st = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_wbc_solve_batch(self._h, B, _ptr(x_des), _ptr(u_des), _ptr(rbd), _ptr(mode), _ptr(sm), _ptr(sol), _ptr(st)), "hb_wbc_solve_batch", self._h)
        return sol, st

    def wbc_assemble(self, x_des, u_des, rbd, mode, stance_mode=None):
        """WeightedWbc's QP in the layout handed to qpOASES: returns (H [B,38,38], g [B,38], A [B,60,38], lbA, ubA [B,60], m_rows [B])."""
        x_des, u_des, rbd = map(_f64, (x_des, u_des, rbd))
        B = x_des.shape[0]
        mode = np.ascontiguousarray(mode, dtype=np.int32)
        sm = None if stance_mode is None else np.ascontiguousarray(stance_mode, dtype=np.uint8)
        H = np.zeros((B, NWBC, NWBC)); g = np.zeros((B, NWBC)); A = np.zeros((B, 60, NWBC)); lb = np.zeros((B, 60)); ub = np.zeros((B, 60))
        m = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_wbc_assemble_batch(self._h, B, _ptr(x_des), _ptr(u_des), _ptr(rbd), _ptr(mode), _ptr(sm), _ptr(H), _ptr(g), _ptr(A), _ptr(lb),
                                               _ptr(ub), _ptr(m)), "hb_wbc_assemble_batch", self._h)
        return H, g, A, lb, ub, m

    def hoqp_solve(self, problems):
        """legged::HoQp cascade for a batch (ctypes array of HbHoqpProblem): returns (x [B,38], stacked slack [B,80], status [B])."""
        B = len(problems)
        x = np.zeros((B, HB_HOQP_N)); sl = np.zeros((B, HB_HOQP_MAX_STACKED)); st = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_hoqp_solve_batch(self._h, B, problems, _ptr(x), _ptr(sl), _ptr(st)), "hb_hoqp_solve_batch", self._h)
        return x, sl, st

    def hierarchical_wbc_tasks(self, x_des, u_des, rbd, mode):
        x_des, u_des, rbd = map(_f64, (x_des, u_des, rbd)); B = x_des.shape[0]
        mode = np.ascontiguousarray(mode, dtype=np.int32)
        pbs = (HbHoqpProblem * B)()
        _check(self._lib.hb_hierarchical_wbc_tasks_batch(self._h, B, _ptr(x_des), _ptr(u_des), _ptr(rbd), _ptr(mode), pbs), "hb_hierarchical_wbc_tasks_batch", self._h)
        return pbs

    def hierarchical_wbc_solve(self, x_des, u_des, rbd, mode):
        """legged::HierarchicalWbc::update for a batch: returns (sol [B,38] = [qdd, F, tau], status [B])."""
        x_des, u_des, rbd = map(_f64, (x_des, u_des, rbd)); B = x_des.shape[0]
        mode = np.ascontiguousarray(mode, dtype=np.int32)
        sol = np.zeros((B, NWBC)); st = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_hierarchical_wbc_solve_batch(self._h, B, _ptr(x_des), _ptr(u_des), _ptr(rbd), _ptr(mode), _ptr(sol), _ptr(st)),
               "hb_hierarchical_wbc_solve_batch", self._h)
        return sol, st

    def mpc_cold_start(self, x0, mode):
        x0 = _f64(x0); B = x0.shape[0]
        mode = np.ascontiguousarray(mode, dtype=np.int32)
        xt = np.zeros((B, self.N + 1, NX)); ut = np.zeros((B, self.N, NU))
        _check(self._lib.hb_mpc_cold_start_batch(self._h, B, _ptr(x0), _ptr(mode), _ptr(xt), _ptr(ut)), "hb_mpc_cold_start_batch", self._h)
        return xt, ut

    def mpc_solve(self, x0, x_ref, swing, mode, xt, ut):
        x0, x_ref, swing = map(_f64, (x0, x_ref, swing))
        B = x0.shape[0]
        mode = np.ascontiguousarray(mode, dtype=np.int32)
        xt = _f64(xt).copy(); ut = _f64(ut).copy()
        info = np.zeros(B, dtype=INFO_DTYPE)
        _check(self._lib.hb_mpc_solve_batch(self._h, B, _ptr(x0), _ptr(x_ref), _ptr(swing), _ptr(mode), _ptr(xt), _ptr(ut), _ptr(info)), "hb_mpc_solve_batch", self._h)
        return xt, ut, info

    def time_grid(self, t0, refs):
        """Event-node time discretisation (row S1): returns (node_times [B, N+1], n_intervals [B], status [B])."""
        t0 = _f64(t0); B = t0.shape[0]
        tk = np.zeros((B, self.N + 1)); nn = np.zeros(B, dtype=np.int32); st = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_time_grid_batch(self._h, B, _ptr(t0), C.cast(refs, C.c_void_p), _ptr(tk), _ptr(nn), _ptr(st)), "hb_time_grid_batch", self._h)
        return tk, nn, st

    def reference_expand_grid(self, node_times, refs):
        tk = _f64(node_times); B = tk.shape[0]
        x_ref = np.zeros((B, self.N + 1, NX)); swing = np.zeros((B, self.N + 1, 24)); mode = np.zeros((B, self.N + 1), dtype=np.int32)
        _check(self._lib.hb_reference_expand_grid_batch(self._h, B, _ptr(tk), C.cast(refs, C.c_void_p), _ptr(x_ref), _ptr(swing), _ptr(mode)),
               "hb_reference_expand_grid_batch", self._h)
        return x_ref, swing, mode

    def mpc_solve_grid(self, x0, node_times, n_intervals, x_ref, swing, mode, xt, ut):
        x0, tk, x_ref, swing = map(_f64, (x0, node_times, x_ref, swing))
        B = x0.shape[0]
        nn = np.ascontiguousarray(n_intervals, dtype=np.int32); mode = np.ascontiguousarray(mode, dtype=np.int32)
        xt = _f64(xt).copy(); ut = _f64(ut).copy()
        info = np.zeros(B, dtype=INFO_DTYPE)
        _check(self._lib.hb_mpc_solve_grid_batch(self._h, B, _ptr(x0), _ptr(tk), _ptr(nn), _ptr(x_ref), _ptr(swing), _ptr(mode), _ptr(xt), _ptr(ut), _ptr(info)),
               "hb_mpc_solve_grid_batch", self._h)
        return xt, ut, info

    def resident_write(self, t0, xt, ut, mode=None, node_times=None, n_intervals=None):
        """Restore a resident-solution snapshot (hb_resident_write_batch)."""
        t0, xt, ut = _f64(t0), _f64(xt), _f64(ut); B = t0.shape[0]
        md = None if mode is None else np.ascontiguousarray(mode, dtype=np.int32)
        tk = None if node_times is None else _f64(node_times); nn = None if n_intervals is None else np.ascontiguousarray(n_intervals, dtype=np.int32)
        _check(self._lib.hb_resident_write_batch(self._h, B, _ptr(t0), _ptr(xt), _ptr(ut), _ptr(md), _ptr(tk), _ptr(nn)), "hb_resident_write_batch", self._h)

    def resident_read_grid(self, B):
        tk = np.zeros((B, self.N + 1)); nn = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_resident_read_grid_batch(self._h, B, _ptr(tk), _ptr(nn)), "hb_resident_read_grid_batch", self._h)
        return tk, nn

    def control_step(self, t_rel, x0, x_ref, swing, mode, rbd, xt, ut):
        x0, x_ref, swing, rbd = map(_f64, (x0, x_ref, swing, rbd))
        B = x0.shape[0]
        mode = np.ascontiguousarray(mode, dtype=np.int32)
        xt = _f64(xt).copy(); ut = _f64(ut).copy()
        info = np.zeros(B, dtype=INFO_DTYPE)
        sol = np.zeros((B, NWBC)); tau = np.zeros((B, NJ)); st = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_control_step_batch(self._h, B, C.c_double(t_rel), _ptr(x0), _ptr(x_ref), _ptr(swing), _ptr(mode), _ptr(rbd), _ptr(xt), _ptr(ut),
                                               _ptr(info), _ptr(sol), _ptr(tau), _ptr(st)), "hb_control_step_batch", self._h)
        return xt, ut, info, sol, tau, st

    def resident_cycle(self, cold_start, t_rel, t0, x0, refs, rbd):
        """Resident closed-loop cycle (hb_resident_cycle_batch); refs: ctypes array of HbReference. Returns (info, sol, torque, status)."""
        t0, x0, rbd = _f64(t0), _f64(x0), _f64(rbd); B = x0.shape[0]
        info = np.zeros(B, dtype=INFO_DTYPE); sol = np.zeros((B, NWBC)); tau = np.zeros((B, NJ)); st = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_resident_cycle_batch(self._h, B, 1 if cold_start else 0, C.c_double(t_rel), _ptr(t0), _ptr(x0), C.cast(refs, C.c_void_p),
                                                 _ptr(rbd), _ptr(info), _ptr(sol), _ptr(tau), _ptr(st)), "hb_resident_cycle_batch", self._h)
        return info, sol, tau, st

    def resident_read(self, B):
        t0 = np.zeros(B); xt = np.zeros((B, self.N + 1, NX)); ut = np.zeros((B, self.N, NU))
        _check(self._lib.hb_resident_read_batch(self._h, B, _ptr(t0), _ptr(xt), _ptr(ut)), "hb_resident_read_batch", self._h)
        return t0, xt, ut

    def plan_references_gpu(self, ins, latest_stance=None):
        """Device planner with host pointers: returns (refs, latest_stance, status)."""
        B = len(ins)
        ls = np.zeros((B, 12)) if latest_stance is None else _f64(latest_stance).copy()
        refs = (HbReference * B)(); st = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_plan_references_gpu(self._h, B, ins, _ptr(ls), refs, _ptr(st)), "hb_plan_references_gpu", self._h)
        return refs, ls, st

    def resident_plan_cycle(self, cold_start, t_rel, ins, rbd):
        """Whole cycle from plan inputs (hb_resident_plan_cycle_batch). Returns (info, sol, torque, wbc_status, plan_status)."""
        rbd = _f64(rbd); B = len(ins)
        info = np.zeros(B, dtype=INFO_DTYPE); sol = np.zeros((B, NWBC)); tau = np.zeros((B, NJ)); st = np.zeros(B, dtype=np.int32); ps = np.zeros(B, dtype=np.int32)
        _check(self._lib.hb_resident_plan_cycle_batch(self._h, B, 1 if cold_start else 0, C.c_double(t_rel), ins, _ptr(rbd), _ptr(info), _ptr(sol), _ptr(tau),
                                                      _ptr(st), _ptr(ps)), "hb_resident_plan_cycle_batch", self._h)
        return info, sol, tau, st, ps

    def estimator_update(self, dt, state, quat, ang_vel_local, lin_acc_local, joint_pos, joint_vel, contact_flag, params=None):
        """KalmanFilterEstimate::update for a batch; `state` (ctypes array of HbKfState) is updated in place. Instance i measures its feet
        heights on this context's estimator map i (set_estimator_maps) when it has one, on state[i].feet_heights otherwise. Returns rbd [B,32]."""
        quat, ang_vel_local, lin_acc_local, joint_pos, joint_vel = map(_f64, (quat, ang_vel_local, lin_acc_local, joint_pos, joint_vel))
        B = quat.shape[0]
        flags = np.ascontiguousarray(contact_flag, dtype=np.uint8).reshape(B, 4)
        params = params or default_kf_params()
        rbd = np.zeros((B, 32))
        _check(self._lib.hb_estimator_update_batch(self._h, B, C.byref(params), C.c_double(dt), state, _ptr(quat), _ptr(ang_vel_local), _ptr(lin_acc_local),
                                                   _ptr(joint_pos), _ptr(joint_vel), _ptr(flags), _ptr(rbd)), "hb_estimator_update_batch", self._h)
        return rbd

    def read_sensors(self, rbd, est, tick, noise=None, accel_dt=0.002, hardware=None, bridge=None):
        """Sensors of the simulated robot at absolute tick `tick` from the true rbd [B,32] (hb_sim_read_sensors_bridge); `est` (ctypes array
        of HbEstimationState) gives the noise streams and the accelerometer's previous velocity and is updated in place. noise: HbSensorNoise
        (None: exact). hardware: B HbHardwareSetting (make_hardware_settings), each robot's sensor offsets and sigmas in place of noise's
        sigmas; bridge: B HbMotorBridge (make_motor_bridges), each robot's joint encoders; None reads as hb_sim_read_sensors. Returns
        (quat [B,4], ang_vel_local [B,3], lin_acc_local [B,3], joint_pos [B,10], joint_vel [B,10])."""
        rbd = _f64(rbd); B = rbd.shape[0]
        noise = noise or HbSensorNoise()
        _check_hardware("read_sensors", hardware, B)
        bridge = _bridge_records(bridge, B, "read_sensors")
        quat = np.zeros((B, 4)); w = np.zeros((B, 3)); a = np.zeros((B, 3)); jp = np.zeros((B, NJ)); jv = np.zeros((B, NJ))
        _check(self._lib.hb_sim_read_sensors_bridge(self._h, B, C.byref(noise), hardware, bridge, C.c_int64(tick), C.c_double(accel_dt), _ptr(rbd), est,
                                                    _ptr(quat), _ptr(w), _ptr(a), _ptr(jp), _ptr(jv)), "hb_sim_read_sensors_bridge", self._h)
        return quat, w, a, jp, jv

    def actuation(self, time, state, command, rbd, delay=0.009, hardware=None, bridge=None):
        """LeggedHWSim::writeSim: delayed hybrid joint command -> applied joint torques [B,10]; `state` (ctypes array of HbActuationState) in place.
        hardware: B HbHardwareSetting (make_hardware_settings), each robot's actuation_delay in place of delay. bridge: B HbMotorBridge
        (make_motor_bridges): each robot's applied entry is encoded instead, and the decoded motor commands [B,10,5] (pos, vel, kp, kd, ff,
        motor frame) are returned in place of the torques, for sim_step(bridge=...) (hb_actuation_bridge)."""
        command, rbd = _f64(command), _f64(rbd); B = rbd.shape[0]
        time = _f64(np.broadcast_to(_f64(time), (B,)))
        _check_hardware("actuation", hardware, B)
        bridge = _bridge_records(bridge, B, "actuation")
        tau = np.zeros((B, NJ)) if bridge is None else None
        mcmd = None if bridge is None else np.zeros((B, NJ, 5))
        _check(self._lib.hb_actuation_bridge(self._h, B, C.c_double(delay), hardware, bridge, _ptr(time), state, _ptr(command), _ptr(rbd), _ptr(tau),
                                             _ptr(mcmd)), "hb_actuation_bridge", self._h)
        return tau if bridge is None else mcmd

    def sim_step(self, rbd, tau, params=None, wrench=None, variation=None, terrain=None, bridge=None, limits=None, links=None, joints=None):
        """One control period of the batched rigid-body plant: returns (rbd_next [B,32], contact_force [B,12], contact_flag [B,4]).
        wrench [B,6]: an external world force at the base origin, then a world couple, held over the period. variation: B HbPlantVariation
        (make_plant_variations), the plant of each robot. terrain: B HbTerrain (make_terrains), the ground under each robot. bridge: B
        HbMotorBridge (make_motor_bridges): tau is then the decoded motor commands [B,10,5] of actuation(bridge=...), whose motor PD runs on
        every substep, clipped to limits ([10] or [B,10]), and the mean clipped torque [B,10] is returned fourth. links: B
        HbLinkVariation (make_link_variations), the bodies of each robot. joints: B HbJointModel (make_joint_models), the range stops and
        friction loss of each robot's joints. Every step is hb_sim_step_joints; without any of the six it is the plain plant step of
        hb_sim_step_batch."""
        rbd = _f64(rbd).copy(); tau = _f64(tau); B = rbd.shape[0]
        params = params or default_sim_params()
        cf = np.zeros((B, 12)); fl = np.zeros((B, 4), dtype=np.uint8)
        w = None if wrench is None else _f64(wrench).reshape(B, 6)
        if variation is not None and len(variation) != B:
            raise ValueError("sim_step: %d plant variations for %d robots" % (len(variation), B))
        if terrain is not None and len(terrain) != B:
            raise ValueError("sim_step: %d terrains for %d robots" % (len(terrain), B))
        if links is not None and len(links) != B:
            raise ValueError("sim_step: %d link variations for %d robots" % (len(links), B))
        if joints is not None and len(joints) != B:
            raise ValueError("sim_step: %d joint models for %d robots" % (len(joints), B))
        bridge = _bridge_records(bridge, B, "sim_step")
        mcmd, lim, applied = None, None, None
        if bridge is not None:
            mcmd, tau = tau.reshape(B, NJ, 5), None
            lim = _f64(np.broadcast_to(_f64(limits), (B, NJ)))
            applied = np.zeros((B, NJ))
        _check(self._lib.hb_sim_step_joints(self._h, B, C.byref(params), _ptr(rbd), _ptr(tau), _ptr(w), variation, terrain, bridge, _ptr(mcmd), _ptr(lim),
                                            _ptr(applied), links, joints, _ptr(cf), _ptr(fl)), "hb_sim_step_joints", self._h)
        return (rbd, cf, fl) if bridge is None else (rbd, cf, fl, applied)

    def _set_instances(self, symbol, items):
        """One per-robot episode setting (hb_rollout_set_*): items[i] for instance i, None clears the setting."""
        n = 0 if items is None else len(items)
        _check(getattr(self._lib, symbol)(self._h, n, items), symbol, self._h)

    def set_terrains(self, terrains):
        """Terrains of this context's episodes (hb_rollout_set_terrains): terrains[i] (make_terrains) is the ground under instance i of every
        later rollout / rollout_estimated call, for the plant and the base-height check; instances beyond len(terrains) stand on the flat
        ground of params.sim.ground_height; None clears them."""
        self._set_instances("hb_rollout_set_terrains", terrains)

    def set_plant_variations(self, variations):
        """Plant variations of this context's episodes (hb_rollout_set_plant_variations): variations[i] (make_plant_variations) is the plant
        of instance i of every later rollout / rollout_estimated call, instances beyond len(variations) run the nominal plant; None clears
        them."""
        self._set_instances("hb_rollout_set_plant_variations", variations)

    def set_link_variations(self, variations):
        """Link variations of this context's episodes (hb_rollout_set_link_variations): variations[i] (make_link_variations) is the
        masses, CoMs and inertias of the bodies of instance i's plant in every later rollout / rollout_estimated call; instances beyond
        len(variations) run the nominal bodies; None clears them. The controllers are not told about it, and no other call reads it."""
        self._set_instances("hb_rollout_set_link_variations", variations)

    def set_joint_models(self, models):
        """Joint models of this context's episodes (hb_rollout_set_joint_models): models[i] (make_joint_models) gives the joints of instance
        i's plant range stops and friction loss in every later rollout / rollout_estimated call; instances beyond len(models) run without
        them; None clears them. The controllers are not told about it, and no other call reads it. An episode call whose params.sim break
        the models' stability rule, h (joint_damping + f_j / v_s) <= joint_armature, raises before it runs."""
        self._set_instances("hb_rollout_set_joint_models", models)

    def set_pushes(self, schedules):
        """Push schedules of this context's episodes (hb_rollout_set_pushes): schedules[i] (make_push_schedules) acts on instance i of every
        later rollout / rollout_estimated call, instances beyond len(schedules) are not pushed; None clears them."""
        self._set_instances("hb_rollout_set_pushes", schedules)

    def set_goals(self, schedules):
        """Goal schedules of this context's episodes (hb_rollout_set_goals): schedules[i] (make_goal_schedules) sends instance i of every
        later rollout / rollout_estimated call to its goal poses, each converted once into a target (goal_to_target) on the MPC tick it comes
        into force; instances beyond len(schedules) follow their cmd_vel; None clears them. Every call forgets the captured goals."""
        self._set_instances("hb_rollout_set_goals", schedules)

    def set_mpc_latencies(self, ticks):
        """MPC latencies of this context's episodes (hb_rollout_set_mpc_latencies): instance i of every later rollout / rollout_estimated
        call tracks the solution of an MPC cycle from ticks[i] ticks after the cycle (0 <= ticks[i] <= mpc_every; 0: from the cycle's own
        tick), instances beyond len(ticks) run with latency 0; None clears them."""
        if ticks is not None:
            ticks = (C.c_int32 * len(ticks))(*[int(getattr(d, "value", d)) for d in ticks])      # ints, or c_int32 records
        self._set_instances("hb_rollout_set_mpc_latencies", ticks)

    def policy_update(self, B, update=None):
        """MPC_MRT_Interface::updatePolicy of instances 0 .. B-1 (hb_policy_update): each with update[i] (None: every one) adopts the
        resident solution as the policy policy_wbc evaluates."""
        up = None if update is None else np.ascontiguousarray(update, dtype=np.uint8)
        if up is not None and up.shape != (B,):
            raise ValueError("policy_update: %d update flags for %d instances" % (up.size, B))
        _check(self._lib.hb_policy_update(self._h, int(B), _ptr(up)), "hb_policy_update", self._h)

    def policy_wbc(self, t_now, rbd, stance_mode=None):
        """resident_wbc on each instance's adopted policy (hb_policy_wbc): returns (x_des, u_des, mode, sol, torque, status)."""
        return self._wbc("hb_policy_wbc", t_now, rbd, stance_mode)

    def set_odometry(self, settings):
        """Tracking cameras of this context's estimated episodes (hb_rollout_set_odometry): settings[i] (make_odometry_settings) is the
        camera of instance i of every later rollout_estimated call, whose messages the filter fuses (updateFromTopic); instances beyond
        len(settings) have none; None clears them. Every call clears the cameras' history and bias."""
        self._set_instances("hb_rollout_set_odometry", settings)

    def set_controller_settings(self, settings):
        """Controller settings of this context's episodes (hb_rollout_set_controller_settings): settings[i] (make_controller_settings) is the
        WBC settings and joint PD gains of instance i of every later rollout / rollout_estimated call, in place of the context's WBC settings
        and params.gains; instances beyond len(settings) run those; None clears them. No other call reads them."""
        self._set_instances("hb_rollout_set_controller_settings", settings)

    def set_hardware(self, settings):
        """Simulated hardware of this context's episodes (hb_rollout_set_hardware): settings[i] (make_hardware_settings) is the actuation
        delay and torque limits of instance i of every later rollout / rollout_estimated call, and in rollout_estimated its sensor sigmas
        and offsets, in place of params' and est_params.noise's values; instances beyond len(settings) run those; None clears them. The
        controllers are not told about it, and no other call reads it."""
        self._set_instances("hb_rollout_set_hardware", settings)

    def set_motor_bridge(self, bridges):
        """Motor bridges of this context's episodes (hb_rollout_set_motor_bridge): bridges[i] (make_motor_bridges) is the joint path of
        instance i of every later rollout / rollout_estimated call through the real robot's motor driver: scaled, quantised commands, the
        motor's PD on every plant substep and, in rollout_estimated, quantised encoders; instances beyond len(bridges) run the simulated
        hardware's torque law; None clears them. The controllers are not told about it, and no other call reads it."""
        self._set_instances("hb_rollout_set_motor_bridge", bridges)

    def set_teleop(self, settings):
        """Teleoperation of this context's episodes (hb_rollout_set_teleop): settings[i] (make_teleop_settings) is the joystick and target
        publisher of instance i of every later rollout / rollout_estimated call: rate-limited cmd_vel messages at the teleop rate while the
        deadman is held, each converted once into a target (cmd_vel_to_target), the filtered command as the planner's cmd_vel; instances
        beyond len(settings) follow their cmd_vel segments directly; None clears them. Every call clears the publishers and the captured
        targets. An episode call rejects a record whose period or window starts are not multiples of its mpc_every."""
        self._set_instances("hb_rollout_set_teleop", settings)

    def set_channels(self, channels):
        """Recorded channels of this context's episodes (hb_rollout_set_channel): channels maps names of CHANNELS to contiguous cuda
        tensors (B, rows, width) of the channel's type (make_channels); every later rollout / rollout_estimated call with log_every > 0
        writes tick r * log_every of the call to row r of each (the sensors only in rollout_estimated). The channels not named are cleared;
        None clears all. The context keeps the tensors until they are replaced or cleared. A call with a set channel of fewer than its B
        instances or fewer than its rows is rejected. On an error every channel is cleared."""
        import torch
        channels = dict(channels or {})
        for name, t in channels.items():
            if name not in CHANNELS:
                raise ValueError("unknown channel %r (one of %s)" % (name, ", ".join(CHANNELS)))
            _, dtype, width = CHANNELS[name]
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == getattr(torch, np.dtype(dtype).name) and t.dim() == 3
                    and t.shape[2] == width and t.is_contiguous()):
                raise ValueError("channel %s: a contiguous cuda %s tensor (B, rows, %d) is needed" % (name, np.dtype(dtype).name, width))
        self._channels = {}
        try:
            for name, (c, _, _) in CHANNELS.items():
                t = channels.get(name)
                args = (0, 0, None) if t is None else (t.shape[0], t.shape[1], _ptr(t))
                _check(self._lib.hb_rollout_set_channel(self._h, c, *args), "hb_rollout_set_channel", self._h)
        except HunterB200Error:
            for c, _, _ in CHANNELS.values():
                self._lib.hb_rollout_set_channel(self._h, c, 0, 0, None)
            raise
        self._channels = channels

    def read_odometry(self, rbd, est, tick, noise=None):
        """The tracking cameras at absolute tick `tick` from the true rbd [B,32] (hb_sim_read_odometry), on this context's odometry setting
        and camera state (advanced); `est` (ctypes array of HbEstimationState) gives the noise streams, noise (HbSensorNoise, None: seed 0)
        the seed. Returns (pos [B,3], has_msg [B]): the message of each instance with one due, zeros for the others."""
        rbd = _f64(rbd); B = rbd.shape[0]
        noise = noise or HbSensorNoise()
        pos = np.zeros((B, 3)); has = np.zeros(B, dtype=np.uint8)
        _check(self._lib.hb_sim_read_odometry(self._h, B, C.byref(noise), C.c_int64(tick), _ptr(rbd), est, _ptr(pos), _ptr(has)),
               "hb_sim_read_odometry", self._h)
        return pos, has

    def fuse_odometry(self, state, pos, has_msg, contact_flag, rbd, params=None):
        """updateFromTopic after estimator_update (hb_estimator_fuse_odometry): each instance with has_msg[i] takes the message pos[i];
        `state` (ctypes array of HbKfState) is updated in place. rbd: the estimated rbd [B,32] estimator_update returned. Returns the fused rbd."""
        rbd = _f64(rbd).copy(); B = rbd.shape[0]
        pos = _f64(pos).reshape(B, 3)
        has = np.ascontiguousarray(has_msg, dtype=np.uint8).reshape(B)
        flags = np.ascontiguousarray(contact_flag, dtype=np.uint8).reshape(B, 4)
        params = params or default_kf_params()
        _check(self._lib.hb_estimator_fuse_odometry(self._h, B, C.byref(params), state, _ptr(pos), _ptr(has), _ptr(flags), _ptr(rbd)),
               "hb_estimator_fuse_odometry", self._h)
        return rbd

    def set_plan_targets(self, targets):
        """Explicit planner targets of this context (hb_plan_set_targets): targets[i] (make_targets, goal_to_target) replaces the cmd_vel
        target of instance i in plan_references_gpu and resident_plan_cycle (not in the episodes); None clears them."""
        self._set_instances("hb_plan_set_targets", targets)

    def set_planner_settings(self, settings):
        """Planner settings of this context (hb_plan_set_settings): settings[i] (make_planner_settings) gives the gait templates and swing
        settings of instance i in every device planner path -- plan_references_gpu, resident_plan_cycle, rollout and rollout_estimated --
        instances beyond len(settings) plan with the compiled-in ones; None clears them."""
        self._set_instances("hb_plan_set_settings", settings)

    def set_height_maps(self, maps):
        """Height maps of this context (hb_plan_set_maps): maps[i] (make_terrains) is the ground the planner of instance i is told about in
        every device planner path -- plan_references_gpu, resident_plan_cycle, rollout and rollout_estimated, their goal and teleop targets
        included -- measured from the flat ground the planner otherwise assumes (a terrain H under a plant at sim.ground_height g is the map
        H - g); instances beyond len(maps) plan without one; None clears them."""
        self._set_instances("hb_plan_set_maps", maps)

    def set_estimator_maps(self, maps):
        """Estimator maps of this context (hb_estimator_set_maps): maps[i] (make_terrains) is the ground the Kalman filter of instance i
        measures its feet heights on, in estimator_update and rollout_estimated, in place of its feet_heights; measured from the flat ground
        the filter otherwise assumes, as height maps are (a terrain H under a plant at sim.ground_height g is the map H - g). Instances
        beyond len(maps) run the filter without one; None clears them."""
        self._set_instances("hb_estimator_set_maps", maps)

    def set_mpc_maps(self, maps):
        """MPC maps of this context (hb_mpc_set_maps): maps[i] (make_terrains) is the ground the MPC of instance i holds its stance feet on,
        in every MPC path (mpc_solve, control_step, the resident cycles, rollout and rollout_estimated): the stance z row pulls each stance
        contact to 0.02 + h at its swing reference's (x, y). Measured from the flat ground the MPC otherwise assumes, as height maps are.
        Instances beyond len(maps) solve without one; None clears them."""
        self._set_instances("hb_mpc_set_maps", maps)

    def set_wbc_maps(self, maps):
        """WBC maps of this context (hb_wbc_set_maps): maps[i] (make_terrains) is the ground the WBC of instance i stands its friction
        pyramids on, in every WBC path (wbc_solve, wbc_assemble, the hierarchical solve and tasks, control_step, the resident cycles,
        resident_wbc, policy_wbc, rollout and rollout_estimated): each stance contact's pyramid is about the map's normal at its measured
        position. Instances beyond len(maps) keep the flat pyramids; None clears them."""
        self._set_instances("hb_wbc_set_maps", maps)

    def set_mpc_cone_maps(self, maps):
        """MPC cone maps of this context (hb_mpc_set_cone_maps): maps[i] (make_terrains) is the ground the MPC of instance i stands its
        friction cones on, in every MPC path (those of set_mpc_maps): each stance contact's cone bounds its force in the map's surface frame
        at its swing reference's (x, y). A setting of its own, apart from set_mpc_maps. Instances beyond len(maps) keep the cones about
        world z; None clears them."""
        self._set_instances("hb_mpc_set_cone_maps", maps)

    def set_contact_detection(self, records):
        """Contact detection of this context's estimated episodes (hb_rollout_set_contact_detection): records[i]
        (make_contact_detection_settings) makes instance i of every later rollout_estimated call run the momentum observer on each tick and
        hand its Kalman filter the flags of estContactState instead of the schedule's; instances beyond len(records), rollout and every
        other call run without it; None clears it. Every call clears the detection state (observer, effort, flags)."""
        self._set_instances("hb_rollout_set_contact_detection", records)

    def contact_state_estimate(self, t, est, est_force, records, flags):
        """The detection rule on the device (hb_contact_state_estimate): est (ctypes array of B HbEstimationState), est_force [B,16],
        records (B HbContactDetection, or None: flags unchanged) and the schedule's flags [B,4] at time t. Returns the detected flags [B,4]."""
        B = len(est)
        force = _f64(est_force).reshape(B, 16)
        fl = np.ascontiguousarray(flags, dtype=np.uint8).reshape(B, 4).copy()
        _check(self._lib.hb_contact_state_estimate(self._h, B, C.c_double(t), est, _ptr(force), _contact_records(records, B, "contact_state_estimate"),
                                                   _ptr(fl)), "hb_contact_state_estimate", self._h)
        return fl

    def contact_estimates(self, B):
        """The detection state of instances 0 .. B-1 (hb_rollout_contact_estimates): (the last observer output [B,16], the flags the filter
        last used [B,4])."""
        force = np.zeros((B, 16)); fl = np.zeros((B, 4), dtype=np.uint8)
        _check(self._lib.hb_rollout_contact_estimates(self._h, B, _ptr(force), _ptr(fl)), "hb_rollout_contact_estimates", self._h)
        return force, fl

    def resident_wbc(self, t_now, rbd, stance_mode=None):
        """Policy of the resident solution at absolute time t_now + WeightedWbc: returns (x_des, u_des, mode, sol, torque, status)."""
        return self._wbc("hb_resident_wbc_batch", t_now, rbd, stance_mode)

    def _wbc(self, symbol, t_now, rbd, stance_mode):
        """The body of resident_wbc and policy_wbc, which differ only in the policy they evaluate."""
        rbd = _f64(rbd); B = rbd.shape[0]
        t_now = _f64(np.broadcast_to(_f64(t_now), (B,)))
        sm = None if stance_mode is None else np.ascontiguousarray(stance_mode, dtype=np.uint8)
        xd = np.zeros((B, NX)); ud = np.zeros((B, NU)); md = np.zeros(B, dtype=np.int32); sol = np.zeros((B, NWBC)); tau = np.zeros((B, NJ)); st = np.zeros(B, dtype=np.int32)
        _check(getattr(self._lib, symbol)(self._h, B, _ptr(t_now), _ptr(rbd), _ptr(sm), _ptr(xd), _ptr(ud), _ptr(md), _ptr(sol), _ptr(tau), _ptr(st)),
               symbol, self._h)
        return xd, ud, md, sol, tau, st

    def contact_force_estimate(self, dt, state, rbd, tau_cmd, cutoff_frequency=250.0):
        """StateEstimateBase::estContactForce for a batch; `state` (ctypes array of HbObserverState) is updated in place.
        Returns (est_contact_force [B,16], disturbance_torque [B,16])."""
        rbd, tau_cmd = _f64(rbd), _f64(tau_cmd); B = rbd.shape[0]
        est = np.zeros((B, 16)); dist = np.zeros((B, 16))
        _check(self._lib.hb_contact_force_estimate_batch(self._h, B, C.c_double(cutoff_frequency), C.c_double(dt), state, _ptr(rbd), _ptr(tau_cmd), _ptr(est),
                                                         _ptr(dist)), "hb_contact_force_estimate_batch", self._h)
        return est, dist

    def joint_command(self, period, x_des, u_des, wbc_sol, mode_cmd, rbd, loaded=None, estop=None, gains=None):
        """Joint command law (LeggedController.cpp:186-257): returns (command [B,10,5], output_torque [B,10], estop [B])."""
        x_des, u_des, wbc_sol, rbd = _f64(x_des), _f64(u_des), _f64(wbc_sol), _f64(rbd); B = x_des.shape[0]
        mode_cmd = np.ascontiguousarray(mode_cmd, dtype=np.int32)
        gains = gains or default_pd_gains()
        ld = None if loaded is None else np.ascontiguousarray(loaded, dtype=np.uint8)
        es = np.zeros(B, dtype=np.uint8) if estop is None else np.ascontiguousarray(estop, dtype=np.uint8).copy()
        cmd = np.zeros((B, NJ, 5)); tau = np.zeros((B, NJ))
        _check(self._lib.hb_joint_command_batch(self._h, B, C.byref(gains), C.c_double(period), _ptr(x_des), _ptr(u_des), _ptr(wbc_sol), _ptr(mode_cmd),
                                                _ptr(rbd), None if ld is None else _ptr(ld), _ptr(es), _ptr(cmd), _ptr(tau)),
               "hb_joint_command_batch", self._h)
        return cmd, tau, es

    def rbd_to_centroidal(self, rbd):
        rbd = _f64(rbd); B = rbd.shape[0]
        x = np.zeros((B, NX))
        _check(self._lib.hb_rbd_to_centroidal_batch(self._h, B, _ptr(rbd), _ptr(x)), "hb_rbd_to_centroidal_batch", self._h)
        return x

    def reference_expand(self, t0, refs):
        """refs: ctypes array of HbReference (len B)."""
        t0 = _f64(t0); B = t0.shape[0]
        x_ref = np.zeros((B, self.N + 1, NX)); swing = np.zeros((B, self.N + 1, 24)); mode = np.zeros((B, self.N + 1), dtype=np.int32)
        _check(self._lib.hb_reference_expand_batch(self._h, B, _ptr(t0), C.cast(refs, C.c_void_p), _ptr(x_ref), _ptr(swing), _ptr(mode)), "hb_reference_expand_batch", self._h)
        return x_ref, swing, mode

    def contact_positions(self, x):
        x = _f64(x); B = x.shape[0]
        pos = np.zeros((B, 12))
        _check(self._lib.hb_contact_positions_batch(self._h, B, _ptr(x), _ptr(pos)), "hb_contact_positions_batch", self._h)
        return pos

    def probe_flow_map(self, x, u):
        x, u = _f64(x), _f64(u); B = x.shape[0]
        f = np.zeros((B, NX)); A = np.zeros((B, NX, NX)); Bm = np.zeros((B, NX, NU)); ee = np.zeros((B, 24 + 36 * NX))
        _check(self._lib.hb_probe_flow_map(self._h, B, _ptr(x), _ptr(u), _ptr(f), _ptr(A), _ptr(Bm), _ptr(ee)), "hb_probe_flow_map", self._h)
        out = dict(f=f, A=A, B=Bm, epos=ee[:, :12], evel=ee[:, 12:24], dpos_dx=ee[:, 24:24 + 264].reshape(B, 12, NX),
                   dvel_dx=ee[:, 24 + 264:24 + 528].reshape(B, 12, NX), dvel_du=ee[:, 24 + 528:].reshape(B, 12, NX))
        return out

    # ------------------------------------------------------------------ device-pointer calls (torch cuda tensors, asynchronous)
    def mpc_solve_dev(self, x0, x_ref, swing, mode, xt, ut, info=None):
        B = x0.shape[0]
        _check(self._lib.hb_mpc_solve_batch_dev(self._h, B, _ptr(x0), _ptr(x_ref), _ptr(swing), _ptr(mode), _ptr(xt), _ptr(ut), _ptr(info)), "hb_mpc_solve_batch_dev", self._h)

    def mpc_cold_start_dev(self, x0, mode, xt, ut):
        _check(self._lib.hb_mpc_cold_start_batch_dev(self._h, x0.shape[0], _ptr(x0), _ptr(mode), _ptr(xt), _ptr(ut)), "hb_mpc_cold_start_batch_dev", self._h)

    def wbc_solve_dev(self, x_des, u_des, rbd, mode, stance_mode, sol, status=None):
        _check(self._lib.hb_wbc_solve_batch_dev(self._h, x_des.shape[0], _ptr(x_des), _ptr(u_des), _ptr(rbd), _ptr(mode), _ptr(stance_mode), _ptr(sol), _ptr(status)),
               "hb_wbc_solve_batch_dev", self._h)

    def wbc_qp_dev(self, n, m, H, g, A, lbA, ubA, x, status=None, iters=None):
        _check(self._lib.hb_wbc_qp_batch_dev(self._h, g.shape[0], n, m, _ptr(H), _ptr(g), _ptr(A), _ptr(lbA), _ptr(ubA), _ptr(x), _ptr(status), _ptr(iters)),
               "hb_wbc_qp_batch_dev", self._h)

    def resident_cycle_dev(self, cold_start, t_rel, t0, x0, refs_dev_ptr, rbd, info, sol, tau, status=None):
        _check(self._lib.hb_resident_cycle_batch_dev(self._h, x0.shape[0], 1 if cold_start else 0, C.c_double(t_rel), _ptr(t0), _ptr(x0), C.c_void_p(refs_dev_ptr),
                                                     _ptr(rbd), _ptr(info), _ptr(sol), _ptr(tau), _ptr(status)), "hb_resident_cycle_batch_dev", self._h)

    def rollout(self, rbd, commands, n_ticks, tick0=0, params=None, act=None, estop=None, stats=None, log_every=0):
        """n_ticks ticks of closed-loop episodes on the device (hb_rollout_batch_dev). rbd: cuda float64 tensor [B, 32], advanced in place;
        commands: ctypes array of HbRolloutCommand (make_rollout_commands); act: cuda uint8 tensor of B hb_actuation_state (None: fresh, in
        place); estop: cuda uint8 tensor [B] (None: zeros, in place); stats: ROLLOUT_STATS_DTYPE array (None: rollout_stats(B)).
        Returns (rbd, act, estop, stats, log): stats as a new structured array, log a cuda tensor [B, ceil(n_ticks / log_every), 32] or None.
        Waits for the episode to finish (the stats are read back)."""
        return self._episodes(rbd, commands, n_ticks, tick0, params, act, estop, stats, log_every)

    def rollout_estimated(self, rbd, commands, n_ticks, tick0=0, params=None, est_params=None, est=None, act=None, estop=None, stats=None, est_stats=None,
                          log_every=0):
        """rollout() with the controllers on the Kalman filter's estimate from noisy sensors (hb_rollout_estimated_batch_dev). est_params:
        HbEstimationParams (None: default_estimation_params(), no noise); est: cuda uint8 tensor of B hb_estimation_state (None: fresh
        estimation_states(B), in place); est_stats: ESTIMATION_STATS_DTYPE array (None: zeros). Returns rollout()'s tuple followed by
        (est, est_stats, est_log): est_log the estimated rbd in log's layout, or None."""
        return self._episodes(rbd, commands, n_ticks, tick0, params, act, estop, stats, log_every, True, est_params, est, est_stats)

    def _episodes(self, rbd, commands, n_ticks, tick0, params, act, estop, stats, log_every, estimated=False, est_params=None, est=None, est_stats=None):
        """The body of rollout() and, with estimated = True, of rollout_estimated()."""
        import torch
        B = rbd.shape[0]
        dev = rbd.device
        params = params or default_rollout_params()
        params.log_every = int(log_every)
        if act is None:
            act = torch.zeros(B * C.sizeof(HbActuationState), dtype=torch.uint8, device=dev)
        if estop is None:
            estop = torch.zeros(B, dtype=torch.uint8, device=dev)

        def records(a, dtype):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype).view(np.uint8).copy()).to(dev)

        def new_log():
            return torch.zeros((B, -(-n_ticks // log_every), 32), dtype=torch.float64, device=dev) if log_every > 0 else None

        d_st = records(rollout_stats(B) if stats is None else stats, ROLLOUT_STATS_DTYPE)
        log = new_log()
        if estimated:
            est_params = est_params or default_estimation_params()
            if est is None:
                est = torch.from_numpy(np.frombuffer(bytes(estimation_states(B)), dtype=np.uint8).copy()).to(dev)
            d_es = records(estimation_stats(B) if est_stats is None else est_stats, ESTIMATION_STATS_DTYPE)
            est_log = new_log()
        torch.cuda.current_stream(dev).synchronize()          # the context's stream does not order itself after torch's
        head = (self._h, B, C.c_int64(tick0), int(n_ticks), C.byref(params))
        if estimated:
            _check(self._lib.hb_rollout_estimated_batch_dev(*head, C.byref(est_params), commands, _ptr(rbd), _ptr(act), _ptr(estop), _ptr(d_st), _ptr(est),
                                                            _ptr(d_es), _ptr(log), _ptr(est_log)), "hb_rollout_estimated_batch_dev", self._h)
        else:
            _check(self._lib.hb_rollout_batch_dev(*head, commands, _ptr(rbd), _ptr(act), _ptr(estop), _ptr(d_st), _ptr(log)), "hb_rollout_batch_dev", self._h)
        self.sync()
        out = (rbd, act, estop, d_st.cpu().numpy().view(ROLLOUT_STATS_DTYPE), log)
        return out + (est, d_es.cpu().numpy().view(ESTIMATION_STATS_DTYPE), est_log) if estimated else out

    # ------------------------------------------------------------------ episode snapshots (hb_episode_save_async / hb_episode_restore)
    @property
    def episode_state_bytes(self):
        """Bytes of one instance's snapshot row on this context (hb_episode_state_bytes)."""
        return int(self._lib.hb_episode_state_bytes(self._h))

    def save_episodes(self, B, rbd, act, estop, stats, est=None, est_stats=None, src=None):
        """Snapshot of B episodes between two rollout / rollout_estimated calls: instance src[i] (None: i) of this context and of the caller's
        buffers (rollout's tuple; est and est_stats for estimated episodes) becomes instance i of the returned EpisodeSnapshot."""
        import torch
        idx = _episode_index(src, B, rbd.shape[0], "save_episodes")
        if (est is None) != (est_stats is None):
            raise ValueError("save_episodes: est and est_stats go together")
        dev = rbd.device
        rows = torch.empty((B, self.episode_state_bytes), dtype=torch.uint8, device=dev)
        torch.cuda.current_stream(dev).synchronize()          # the context's stream does not order itself after torch's
        _check(self._lib.hb_episode_save_async(self._h, B, (C.c_int32 * B)(*idx), _ptr(rows)), "hb_episode_save_async", self._h)
        self.sync()
        out = [rows] + _gather(idx, rbd, act, estop, stats, est, est_stats)
        return EpisodeSnapshot(*out)

    def restore_episodes(self, snapshot, src=None):
        """Instance i of this context from instance src[i] (None: i) of the EpisodeSnapshot, for B = len(src) (None: every instance).
        Returns fresh buffers of the B instances to continue them with: (rbd, act, estop, stats) for rollout, followed by (est, est_stats)
        for rollout_estimated, with tick0 the tick the episodes were saved at. Set goals and odometry before: both clear what this restores."""
        import torch
        n = len(snapshot)
        B = n if src is None else len(src)
        idx = _episode_index(src, B, n, "restore_episodes")
        if snapshot.rows.shape[1] != self.episode_state_bytes:
            raise ValueError("restore_episodes: rows of %d bytes, this context's hold %d" % (snapshot.rows.shape[1], self.episode_state_bytes))
        rows = snapshot.rows.contiguous()
        torch.cuda.current_stream(rows.device).synchronize()
        _check(self._lib.hb_episode_restore(self._h, B, (C.c_int32 * B)(*idx), n, _ptr(rows)), "hb_episode_restore", self._h)
        return tuple(_gather(idx, snapshot.rbd, snapshot.act, snapshot.estop, snapshot.stats, snapshot.est, snapshot.est_stats))

    def control_step_dev(self, t_rel, x0, x_ref, swing, mode, rbd, xt, ut, info, sol, tau, status=None):
        _check(self._lib.hb_control_step_batch_dev(self._h, x0.shape[0], C.c_double(t_rel), _ptr(x0), _ptr(x_ref), _ptr(swing), _ptr(mode), _ptr(rbd), _ptr(xt),
                                                   _ptr(ut), _ptr(info), _ptr(sol), _ptr(tau), _ptr(status)), "hb_control_step_batch_dev", self._h)


# ---------------------------------------------------------------------------------------------------------------------
# Host-side mirrors of the reference operators (single-robot use, B = 1), for drop-in style tests.
class HierarchicalWbc:
    """Mirror of legged::HierarchicalWbc (legged_wbc/include/legged_wbc/HierarchicalWbc.h, src/HierarchicalWbc.cpp:18-31)."""

    def __init__(self, ctx=None):
        self._ctx = ctx or Context(max_batch=1)

    def update(self, stateDesired, inputDesired, rbdStateMeasured, mode, period):
        sol, st = self._ctx.hierarchical_wbc_solve(np.asarray(stateDesired)[None], np.asarray(inputDesired)[None], np.asarray(rbdStateMeasured)[None], [int(mode)])
        if st[0] != 0:
            raise HunterB200Error("[HierarchicalWbc] a level of the hierarchy did not solve (status %d)" % st[0])
        return sol[0]


class WeightedWbc:
    """Mirror of legged::WeightedWbc (legged_wbc/include/legged_wbc/WeightedWbc.h, WbcBase.h:41-76)."""

    def __init__(self, ctx=None):
        self._ctx = ctx or Context(max_batch=1)
        self._stance_mode = True      # WbcBase default until setStanceMode(false) (LeggedController.cpp:161-173)
        self._last = None

    def loadTasksSetting(self, taskFile=None, verbose=False):
        """WbcBase::loadTasksSetting + WeightedWbc::loadTasksSetting (WbcBase.cpp:352-411, WeightedWbc.cpp:96-111): torque limits, friction
        coefficient, task gains and weights from the task file; without a file the shipped values stay in force."""
        if taskFile is not None:
            self._ctx.load_task_info(taskFile)
        if verbose:
            s = self._ctx.wbc_settings()
            print(" #### WBC settings:", {k: (list(getattr(s, k)) if k == "torque_limits" else getattr(s, k)) for k, _ in s._fields_})

    def setKpKd(self, swingKp, swingKd):
        self._ctx.set_kp_kd(swingKp, swingKd)

    def setStanceMode(self, flag):
        self._stance_mode = bool(flag)

    def getContactForceSize(self):
        return 12

    def update(self, stateDesired, inputDesired, rbdStateMeasured, mode, period):
        sol, st = self._ctx.wbc_solve(np.asarray(stateDesired)[None], np.asarray(inputDesired)[None], np.asarray(rbdStateMeasured)[None],
                                      [int(mode)], [1 if self._stance_mode else 0])
        x = sol[0]
        if st[0] != 0:
            print("ERROR: WeightWBC Not Solved!!!")          # WeightedWbc.cpp:57-62
            if self._last is not None:
                x = self._last
        self._last = x.copy()
        return x


class SqpMpc:
    """Mirror of the MPC_MRT_Interface calls the controller makes (LeggedController.cpp:144-156,406) on a batch of 1."""

    def __init__(self, ctx=None, horizon_N=100, dt=0.01):
        self._ctx = ctx or Context(horizon_N=horizon_N, dt=dt, max_batch=1)
        self._xt = None
        self._ut = None
        self._mode = None

    def reset(self):
        self._xt = self._ut = None

    def advance(self, x0, x_ref, swing, mode):
        """One SQP iteration warm-started from the previous solution (mpc.coldStart false, task.info:146)."""
        x0 = np.asarray(x0, dtype=np.float64)[None]
        mode = np.asarray(mode, dtype=np.int32)[None]
        if self._xt is None:
            self._xt, self._ut = self._ctx.mpc_cold_start(x0, mode)
        xt, ut, info = self._ctx.mpc_solve(x0, np.asarray(x_ref)[None], np.asarray(swing)[None], mode, self._xt, self._ut)
        if info["status"][0] != 0:      # a failed iteration must not poison the next warm start: the previous solution stays
            raise HunterB200Error("[SqpMpc] numerical failure in the SQP iteration")   # the reference's MPC thread stops the controller (LeggedController.cpp:413-418)
        self._xt, self._ut, self._mode = xt, ut, mode
        return info[0]

    def evaluatePolicy(self, t_rel):
        s = min(max(t_rel / self._ctx.dt, 0.0), float(self._ctx.N))
        k = min(int(np.floor(s)), self._ctx.N - 1)
        al = s - k
        x = (1 - al) * self._xt[0, k] + al * self._xt[0, k + 1]
        k1 = min(k + 1, self._ctx.N - 1)
        u = (1 - al) * self._ut[0, k] + al * self._ut[0, k1]
        return x, u, int(self._mode[0, k])
