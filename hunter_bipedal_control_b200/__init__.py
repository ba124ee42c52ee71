"""hunter_bipedal_control_b200 -- H100-native batched NMPC + WBC solve path for the Hunter biped (one hot path, not a port).

Only what the path needs: ``csrc/`` (sm_90a CUDA kernels + the C ABI of include/hunter_b200.h) and ``api`` (ctypes binding and
host-side mirrors of the reference's WbcBase / MPC_MRT_Interface calls). No CPU fallback exists.
"""
from .api import (HbWbcSettings, HbTaskInfo, parse_task_info, Context, WeightedWbc, HierarchicalWbc, HbHoqpProblem, make_hoqp_problems, hoqp_tasks, SqpMpc, HbReference, HbSolveInfo, HbConfig, HunterB200Error, load_library, EXPORTED_SYMBOLS,
                  NX, NU, NQ, NJ, NWBC, INFO_DTYPE, HbPlanInput, plan_references, plan_set_threads, make_plan_inputs, GAIT_IDS, GaitSelector, HbPdGains, default_pd_gains, HbKfState, HbKfParams, default_kf_params, kf_states, HbObserverState, observer_states, HbActuationState, HbSimParams, default_sim_params, actuation_states,
                  HbRolloutCommand, HbRolloutParams, HbRolloutStats, ROLLOUT_STATS_DTYPE, ROLLOUT_FAIL, default_rollout_params, rollout_stats, make_rollout_commands,
                  HB_MAX_PUSHES, HbPushSchedule, make_push_schedules, HbPlantVariation, default_plant_variation, make_plant_variations, HB_TERRAIN_MAX, HbTerrain, make_terrains, HbSensorNoise, HbEstimationParams, HbEstimationState, HbEstimationStats, ESTIMATION_STATS_DTYPE, default_estimation_params, estimation_states, estimation_stats,
                  HbTarget, make_targets, reference_target, goal_to_target, HB_MAX_GOALS, HbGoalSchedule, make_goal_schedules,
                  HB_ODOM_MAX_DELAY, HbOdometrySetting, make_odometry_settings, HbControllerSetting, make_controller_settings,
                  HbHardwareSetting, default_hardware_setting, make_hardware_settings,
                  HbMotorBridge, default_motor_bridge, make_motor_bridges, bridge_encode, bridge_feedback,
                  NBODY, HbLinkVariation, default_link_variation, make_link_variations, HbJointModel, default_joint_model, make_joint_models,
                  HB_MAX_TELEOP_WINDOWS, TELEOP_ALWAYS, HbTeleop, HbTeleopSetting, default_teleop_setting, make_teleop_settings, cmd_vel_to_target,
                  HB_GAIT_MAX_PHASES, HbGaitTemplate, HbPlannerSettings, gait_template, default_planner_settings, parse_planner_settings, make_planner_settings,
                  CHANNELS, make_channels, EpisodeSnapshot, reseed,
                  HbContactDetection, default_contact_detection, make_contact_detection_settings, contact_state_host)

__all__ = ["HbWbcSettings", "HbTaskInfo", "parse_task_info", "Context", "WeightedWbc", "HierarchicalWbc", "HbHoqpProblem", "make_hoqp_problems", "hoqp_tasks", "SqpMpc", "HbReference", "HbSolveInfo", "HbConfig", "HunterB200Error", "load_library",
           "EXPORTED_SYMBOLS", "NX", "NU", "NQ", "NJ", "NWBC", "INFO_DTYPE", "HbPlanInput", "plan_references", "plan_set_threads", "make_plan_inputs", "GAIT_IDS", "GaitSelector", "HbPdGains", "default_pd_gains", "HbKfState", "HbKfParams", "default_kf_params", "kf_states", "HbObserverState", "observer_states", "HbActuationState", "HbSimParams", "default_sim_params", "actuation_states",
           "HbRolloutCommand", "HbRolloutParams", "HbRolloutStats", "ROLLOUT_STATS_DTYPE", "ROLLOUT_FAIL", "default_rollout_params", "rollout_stats", "make_rollout_commands",
           "HB_MAX_PUSHES", "HbPushSchedule", "make_push_schedules", "HbPlantVariation", "default_plant_variation", "make_plant_variations", "HB_TERRAIN_MAX", "HbTerrain", "make_terrains", "HbSensorNoise", "HbEstimationParams", "HbEstimationState", "HbEstimationStats", "ESTIMATION_STATS_DTYPE", "default_estimation_params", "estimation_states", "estimation_stats",
           "HbTarget", "make_targets", "reference_target", "goal_to_target", "HB_MAX_GOALS", "HbGoalSchedule", "make_goal_schedules",
           "HB_ODOM_MAX_DELAY", "HbOdometrySetting", "make_odometry_settings", "HbControllerSetting", "make_controller_settings",
           "HbHardwareSetting", "default_hardware_setting", "make_hardware_settings",
           "HbMotorBridge", "default_motor_bridge", "make_motor_bridges", "bridge_encode", "bridge_feedback",
           "NBODY", "HbLinkVariation", "default_link_variation", "make_link_variations", "HbJointModel", "default_joint_model", "make_joint_models",
           "HB_MAX_TELEOP_WINDOWS", "TELEOP_ALWAYS", "HbTeleop", "HbTeleopSetting", "default_teleop_setting", "make_teleop_settings", "cmd_vel_to_target",
           "HB_GAIT_MAX_PHASES", "HbGaitTemplate", "HbPlannerSettings", "gait_template", "default_planner_settings", "parse_planner_settings", "make_planner_settings",
           "CHANNELS", "make_channels", "EpisodeSnapshot", "reseed",
           "HbContactDetection", "default_contact_detection", "make_contact_detection_settings", "contact_state_host"]
