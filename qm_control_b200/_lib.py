"""ctypes binding of libqmb200.so (C ABI: include/qmb200.h).  Fails loudly when the library is missing."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.environ.get("QMB200_LIB", os.path.join(HERE, "libqmb200.so"))   # override only selects another build of the same library
ASSETS = os.path.join(ROOT, "assets")

NX, NU, RBD, CMD, TARGET, EMAX, KMAX = 30, 30, 55, 54, 37, 32, 4
GAIT_CAP, GAIT_MAXM = 64, 16   # QMB200_GAIT_CAP, QMB200_GAIT_MAXM
TARGET_CMD_VEL, TARGET_EE_CMD_VEL, TARGET_EE_GOAL = 0, 1, 2   # QMB200_TARGET_*: the target front-end's kinds (-1 in a per-robot kind: a held goal)
EE_FRAME_WORLD, EE_FRAME_HEADING = 0, 1   # QMB200_EE_FRAME_*: the frame a robot's end-effector targets are stated in (DESIGN.md §4.19)
TARGET_EE_PATH, TARGET_EE_PATH_FOLLOW = 3, 4   # QMB200_TARGET_EE_PATH(_FOLLOW): start / follow an end-effector path (DESIGN.md §4.20)
EE_PATH_MAX, EE_PATH_STATE = 32, 12   # QMB200_EE_PATH_MAX waypoints per path; QMB200_EE_PATH_STATE doubles of a robot's path state row
ST_OVERFLOW = 0x2      # QMB200_ST_OVERFLOW: a WBC overflow
ST_COMMAND = 0x20000   # QMB200_ST_COMMAND: a rejected qmb200_gait_dev_command row
ST_RESTORE = 0x40000   # QMB200_ST_RESTORE: a qmb200_robot_state_load source row outside [0, B)
ST_SPAWN = 0x80000     # QMB200_ST_SPAWN: a rejected qmb200_spawn_place row

dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int32)


class QmbError(RuntimeError):
    pass


class Config(C.Structure):
    _fields_ = [("task_file", C.c_char_p), ("urdf_file", C.c_char_p), ("reference_file", C.c_char_p), ("wbc_gains_file", C.c_char_p),
                ("batch", C.c_int32), ("device", C.c_int32), ("time_horizon", C.c_double), ("dt", C.c_double), ("max_nodes", C.c_int32), ("wbc_variant", C.c_int32)]


class WbcGains(C.Structure):
    """qmb200_wbc_gains (WbcBase::dynamicCallback, qm_wbc/cfg/wbcWigeht.cfg:7-47)."""
    _fields_ = [(n, C.c_double) for n in ("kp_swing", "kd_swing", "base_height_kp", "base_height_kd", "kp_base_linear", "kd_base_linear", "kp_base_angular", "kd_base_angular")] + \
               [("kp_arm_joint", C.c_double * 6), ("kd_arm_joint", C.c_double * 6), ("kp_ee_linear", C.c_double * 3), ("kd_ee_linear", C.c_double * 3), ("kp_ee_angular", C.c_double * 3), ("kd_ee_angular", C.c_double * 3)]


class SimParams(C.Structure):
    """qmb200_sim_params: the plant's contact and joint constants (include/qmb200.h, DESIGN.md §4.6)."""
    _fields_ = [(n, C.c_double) for n in ("ground_height", "foot_radius", "stiffness", "damping", "tangential_damping", "friction_mu")] + \
               [("joint_damping", C.c_double * 18), ("substeps_per_ms", C.c_int32)]


class PayloadEstParams(C.Structure):
    """qmb200_payload_est_params: the online payload estimator's constants (include/qmb200.h, DESIGN.md §4.6)."""
    _fields_ = [(n, C.c_double) for n in ("forgetting", "p0_mass", "p0_first_moment", "p0_inertia", "trace_max", "mass_min", "mass_max", "offset_max")]


SENSORS = 46   # QMB200_SENSORS


class SensorParams(C.Structure):
    """qmb200_sensor_params: the noise of the plant's IMU and encoder readings (include/qmb200.h, DESIGN.md §4.6)."""
    _fields_ = [("seed", C.c_uint64)] + [(n, C.c_double) for n in ("sigma_orientation", "sigma_gyro", "sigma_accel", "sigma_joint_pos", "sigma_joint_vel")]


class StateEstParams(C.Structure):
    """qmb200_state_est_params: the base state estimator's constants (include/qmb200.h, DESIGN.md §4.6)."""
    _fields_ = [(n, C.c_double) for n in ("process_base_pos", "process_base_vel", "process_foot", "meas_foot_pos", "meas_foot_vel", "meas_foot_height", "swing_scale",
                                          "foot_height", "p0_base_pos", "p0_base_vel", "p0_foot")]


class AttitudeParams(C.Structure):
    """qmb200_attitude_params: the attitude filter's constants (include/qmb200.h, DESIGN.md §4.6)."""
    _fields_ = [(n, C.c_double) for n in ("process_attitude", "process_gyro_bias", "meas_orientation", "p0_attitude", "p0_gyro_bias")]


class SlipParams(C.Structure):
    """qmb200_slip_params: the slip detector's thresholds (include/qmb200.h, DESIGN.md §4.6)."""
    _fields_ = [("gate", C.c_double), ("release", C.c_double), ("meas_slip", C.c_double), ("hold", C.c_int32)]


# the sensor reading's columns (qmb200_sim_read_sensors) and the state estimator's state x (qmb200_state_est_get)
SENSOR_LAYOUT = ("quat_x", "quat_y", "quat_z", "quat_w", "gyro_x", "gyro_y", "gyro_z", "accel_x", "accel_y", "accel_z") + \
                tuple("joint_pos_%d" % j for j in range(18)) + tuple("joint_vel_%d" % j for j in range(18))
STATE_EST_LAYOUT = ("p_x", "p_y", "p_z", "v_x", "v_y", "v_z") + tuple("foot_%s_%s" % (f, a) for f in ("LF", "RF", "LH", "RH") for a in "xyz")
# the reference sensor noise of qm_gazebo/config/default.yaml:3-8 (covariances 0.0012, 0.0004, 0.01 of orientation, angular velocity, linear acceleration)
SENSOR_NOISE_REFERENCE = dict(sigma_orientation=0.0012 ** 0.5, sigma_gyro=0.0004 ** 0.5, sigma_accel=0.01 ** 0.5)

# the payload estimator's parameter vector theta: the load's inertial parameters in the end-effector frame about its origin (include/qmb200.h)
THETA_LAYOUT = ("m", "mc_x", "mc_y", "mc_z", "I_xx", "I_xy", "I_xz", "I_yy", "I_yz", "I_zz")

# per-robot plant variation (include/qmb200.h: qmb200_sim_set_robot_params, qmb200_sim_step_ext): the column layouts of payload[B][8] and wrench[B][12]
PAYLOAD_LAYOUT = ("m_ee", "o_ee_x", "o_ee_y", "o_ee_z", "m_base", "o_base_x", "o_base_y", "o_base_z")
# the controller's model payload (qmb200_set_model_payload) has PAYLOAD_LAYOUT too; per robot it yields SRBD_LAYOUT (qmb200_debug_srbd_constants)
SRBD_LAYOUT = ("m",) + tuple("I_nom_%d%d" % (i, j) for i in range(3) for j in range(3)) + tuple("I_nom_inv_%d%d" % (i, j) for i in range(3) for j in range(3)) + \
              ("c_nom_x", "c_nom_y", "c_nom_z", "pad0", "pad1")
# per-robot controller tuning (qmb200_set_robot_tuning): field -> (offset, width) in a row of TUNING doubles; the WBC gains in WbcGains order
TUNING_LAYOUT = {}
for _n, _w in [("friction_mu", 1), ("wbc_friction", 1), ("mu_ee_pos", 1), ("mu_ee_ori", 1), ("mu_final_ee_pos", 1), ("mu_final_ee_ori", 1)] + \
              [(_f, getattr(_t, "_length_", 1)) for _f, _t in WbcGains._fields_] + [("kp_arm_wbc", 1), ("kd_arm_wbc", 1)]:
    TUNING_LAYOUT[_n] = (sum(w for _, w in TUNING_LAYOUT.values()), _w)
TUNING = sum(w for _, w in TUNING_LAYOUT.values())   # QMB200_TUNING
del _n, _w
WRENCH_LAYOUT = ("f_base_x", "f_base_y", "f_base_z", "n_base_x", "n_base_y", "n_base_z", "f_ee_x", "f_ee_y", "f_ee_z", "n_ee_x", "n_ee_y", "n_ee_z")
# one episode's plant draw (qmb200_episode_*): the columns of a row of EPISODE doubles, and the link bits of qmb200_episode_sample(_dev)
EPISODE_LAYOUT = ("friction_mu",) + PAYLOAD_LAYOUT + ("push_t_on", "push_duration") + WRENCH_LAYOUT + ("cmd_vel_x", "cmd_vel_y", "cmd_vel_z", "cmd_yaw_rate")
EPISODE = len(EPISODE_LAYOUT)   # QMB200_EPISODE
EPISODE_MODEL_PAYLOAD, EPISODE_MPC_FRICTION, EPISODE_WBC_FRICTION = 1, 2, 4   # QMB200_EPISODE_*
# one episode's spawn (qmb200_spawn_*): the columns of a row of SPAWN doubles, and the link bit of qmb200_spawn_sample(_dev)
SPAWN_LAYOUT = ("tile", "dx", "dy", "yaw")
SPAWN = len(SPAWN_LAYOUT)   # QMB200_SPAWN
SPAWN_GROUND_MAP = 1        # QMB200_SPAWN_GROUND_MAP
# one closed episode's metrics (qmb200_metrics_*): the columns of a row of METRICS doubles, and the width of the accumulator row of an open episode
METRICS_LAYOUT = ("duration", "end", "status", "distance", "path_length", "min_height", "max_tilt", "vel_err_rms", "yaw_rate_err_rms", "ee_pos_err_rms",
                  "ee_pos_err_max", "ee_ori_err_rms", "energy", "torque_rms", "slip", "touchdowns", "est_pos_err_rms", "est_vel_err_rms")
METRICS = len(METRICS_LAYOUT)   # QMB200_METRICS
METRICS_ACC = 32                # QMB200_METRICS_ACC
# one episode's command timeline (qmb200_timeline_*): the columns of a ranges row of TIMELINE doubles, and of a drawn slot of TIMELINE_CMD doubles
TIMELINE_LAYOUT = ("t_first", "gap", "p_gait", "gait_set", "w_none", "w_cmd_vel", "w_ee_cmd_vel", "w_ee_goal", "cmd_vel_x", "cmd_vel_y", "cmd_vel_z", "cmd_yaw_rate",
                   "ee_vx", "ee_vy", "ee_vz", "ee_x", "ee_y", "ee_z", "ee_qx", "ee_qy", "ee_qz", "ee_qw")
TIMELINE = len(TIMELINE_LAYOUT)   # QMB200_TIMELINE
TIMELINE_CMD_LAYOUT = ("t", "tmpl", "cmd_vel_x", "cmd_vel_y", "cmd_vel_z", "cmd_yaw_rate", "ee_kind") + tuple("ee_%d" % i for i in range(7))
TIMELINE_CMD = len(TIMELINE_CMD_LAYOUT)   # QMB200_TIMELINE_CMD
# one episode's end-effector path (qmb200_ee_path_*): the columns of a ranges row of EE_PATH_RANGES doubles; a drawn path is a row of the path table
# (qmb200_set_ee_paths): EE_PATH_MAX waypoints of (tau, x, y, z, qx, qy, qz, qw), zeros past its n_way
EE_PATH_RANGES_LAYOUT = ("n_way", "tau_first", "gap", "x", "y", "z", "yaw", "qx", "qy", "qz", "qw")
EE_PATH_RANGES = len(EE_PATH_RANGES_LAYOUT)   # QMB200_EE_PATH_RANGES
# a robot's curriculum (qmb200_curriculum_*): the columns of its row of CURRICULUM doubles and of its state of CURRICULUM_STATE int32, the kinds a
# curriculum attaches to, and a rule's condition ops and roles by their codes
CURRICULUM_LAYOUT = ("start_level", "up_after", "down_after", "threshold_0", "threshold_1", "threshold_2", "threshold_3")
CURRICULUM = len(CURRICULUM_LAYOUT)   # QMB200_CURRICULUM
CURRICULUM_STATE_LAYOUT = ("level", "pass_run", "fail_run", "n_updates")
CURRICULUM_STATE = len(CURRICULUM_STATE_LAYOUT)   # QMB200_CURRICULUM_STATE
CURRICULUM_MAX_COND = 4   # QMB200_CURRICULUM_MAX_COND
CURRICULUM_KINDS = ("episode", "spawn", "timeline", "ee_path")   # QMB200_CURRICULUM_EPISODE, _SPAWN, _TIMELINE, _EE_PATH
CURRICULUM_OPS = (">=", "<=")         # QMB200_CURRICULUM_GE, _LE
CURRICULUM_ROLES = ("pass", "fail")   # QMB200_CURRICULUM_PASS, _FAIL


class CurriculumRule(C.Structure):
    """qmb200_curriculum_rule: the level count and up to CURRICULUM_MAX_COND conditions on a closed episode's metrics row (include/qmb200.h)."""
    _fields_ = [("n_levels", C.c_int32), ("n_cond", C.c_int32), ("column", C.c_int32 * 4), ("op", C.c_int32 * 4), ("role", C.c_int32 * 4)]


# the blocks of a robot-state snapshot (qmb200_robot_state_*), block i being bit i of RobotStateDesc.blocks
ROBOT_STATE_BLOCKS = ("state_est", "attitude", "slip", "payload_est", "model_payload", "model_srbd", "gait", "gait_cursor", "mpc_n_nodes", "mpc_t", "mpc_event",
                      "mpc_x", "mpc_u", "wbc_input_last", "hw_ring_cmd", "hw_ring_stamp", "hw_ring_state", "gait_pending", "plant_mu", "plant_payload",
                      "robot_terrain", "ground_map", "tuning", "timeline_t", "timeline_tmpl", "timeline_vel", "timeline_ee_kind", "timeline_ee",
                      "mpc_n_events", "mpc_event_times", "mpc_modes", "mpc_status", "ee_frame")


class RobotStateDesc(C.Structure):
    """qmb200_robot_state_desc: what a robot-state snapshot holds (include/qmb200.h, DESIGN.md §4.17)."""
    _fields_ = [("batch", C.c_int32), ("n_blocks", C.c_int32), ("bytes", C.c_int64), ("blocks", C.c_uint64), ("gen", C.c_uint64 * len(ROBOT_STATE_BLOCKS))]


# every function include/qmb200.h declares, in header order: name -> (restype, argtypes).  Every pointer is c_void_p (numpy / torch addresses, byref,
# None), except the file-name strings and the config struct; int and int32_t are c_int32.  The CPU test-suite checks each slot against the header.
P, I32, I64, D, S, CFG = C.c_void_p, C.c_int32, C.c_int64, C.c_double, C.c_char_p, C.POINTER(Config)
PROTOTYPES = {
    "qmb200_create": (I32, [CFG, P]),
    "qmb200_destroy": (None, [P]),
    "qmb200_last_error": (S, [P]),
    "qmb200_get_dims": (I32, [P] * 5),
    "qmb200_get_model_info": (I32, [P] * 6),
    "qmb200_get_joint_name": (I32, [P, I32, P, I32]),
    "qmb200_wbc_update": (I32, [P] * 9),
    "qmb200_wbc_update_dev": (I32, [P] * 10),
    "qmb200_wbc_set_input_last": (I32, [P] * 2),
    "qmb200_wbc_get_input_last": (I32, [P] * 2),
    "qmb200_wbc_get_gains": (I32, [P] * 2),
    "qmb200_wbc_set_gains": (I32, [P] * 2),
    "qmb200_wbc_get_diagnostics": (I32, [P] * 2),
    "qmb200_wbc_set_iteration_caps": (I32, [P, I32, I32]),
    "qmb200_mpc_solve": (I32, [P] * 16),
    "qmb200_mpc_solve_dev": (I32, [P] * 10),
    "qmb200_mpc_set_iterations": (I32, [P, I32, D]),
    "qmb200_mpc_reset": (I32, [P]),
    "qmb200_mpc_set_solution": (I32, [P] * 6),
    "qmb200_mpc_get_solution": (I32, [P] * 8),
    "qmb200_policy_eval": (I32, [P] * 5),
    "qmb200_policy_eval_dev": (I32, [P] * 6),
    "qmb200_tick": (I32, [P] * 14),
    "qmb200_tick_dev": (I32, [P] * 15),
    "qmb200_centroidal_state_from_rbd": (I32, [P, I32, P, P]),
    "qmb200_set_model_payload": (I32, [P] * 2),
    "qmb200_get_model_payload": (I32, [P] * 3),
    "qmb200_set_robot_tuning": (I32, [P] * 2),
    "qmb200_get_robot_tuning": (I32, [P] * 3),
    "qmb200_get_handle_tuning": (I32, [P] * 2),
    "qmb200_payload_est_get_params": (I32, [P] * 2),
    "qmb200_payload_est_set_params": (I32, [P] * 2),
    "qmb200_payload_est_reset": (I32, [P] * 2),
    "qmb200_payload_est_step": (I32, [P, D] + [P] * 3),
    "qmb200_payload_est_step_dev": (I32, [P, D] + [P] * 4),
    "qmb200_payload_est_commit_dev": (I32, [P] * 2),
    "qmb200_payload_est_get": (I32, [P] * 4),
    "qmb200_payload_est_stop": (I32, [P]),
    "qmb200_get_model_payload_dev": (I32, [P] * 3),
    "qmb200_gait_schedule": (I32, [S, S, D, D, D, P, P]),
    "qmb200_gait_create": (I32, [S, S, P]),
    "qmb200_gait_destroy": (None, [P]),
    "qmb200_gait_insert_template": (I32, [P, S, S, D, D]),
    "qmb200_gait_get_mode_schedule": (I32, [P, D, D, P, P]),
    "qmb200_gait_dev_set_templates": (I32, [P, S, P, I32]),
    "qmb200_gait_dev_reset": (I32, [P] * 3),
    "qmb200_gait_dev_set_commands": (I32, [P, I32] + [P] * 3),
    "qmb200_gait_dev_set_commands_ee": (I32, [P, I32] + [P] * 5),
    "qmb200_gait_dev_step": (I32, [P] * 9),
    "qmb200_gait_dev_step_dev": (I32, [P] * 10),
    "qmb200_gait_dev_step_ee": (I32, [P] * 10),
    "qmb200_gait_dev_step_ee_dev": (I32, [P] * 11),
    "qmb200_gait_dev_get": (I32, [P] * 6),
    "qmb200_gait_dev_get_commands": (I32, [P] * 7),
    "qmb200_gait_dev_command": (I32, [P] * 7),
    "qmb200_gait_dev_command_dev": (I32, [P] * 8),
    "qmb200_gait_dev_get_pending": (I32, [P] * 6),
    "qmb200_gait_dev_stop": (I32, [P]),
    "qmb200_observation_update": (I32, [P] * 5),
    "qmb200_observation_update_dev": (I32, [P] * 6),
    "qmb200_target_trajectories": (I32, [P, I32] + [P] * 8),
    "qmb200_target_trajectories_dev": (I32, [P, I32] + [P] * 9),
    "qmb200_target_trajectories_per_robot": (I32, [P] * 10),
    "qmb200_target_trajectories_per_robot_dev": (I32, [P] * 11),
    "qmb200_initial_ee_target": (None, [P]),
    "qmb200_set_ee_frame": (I32, [P] * 2),
    "qmb200_get_ee_frame": (I32, [P] * 3),
    "qmb200_set_ee_paths": (I32, [P, I32, P, P]),
    "qmb200_get_ee_paths": (I32, [P] * 4),
    "qmb200_target_trajectories_path": (I32, [P] * 11),
    "qmb200_target_trajectories_path_dev": (I32, [P] * 12),
    "qmb200_control_law": (I32, [P] * 10),
    "qmb200_control_law_dev": (I32, [P] * 11),
    "qmb200_set_arm_gains": (I32, [P, D, D]),
    "qmb200_hw_write": (I32, [P] * 8),
    "qmb200_hw_write_dev": (I32, [P] * 9),
    "qmb200_hw_set_delay": (I32, [P, D]),
    "qmb200_sim_get_params": (I32, [P] * 2),
    "qmb200_sim_set_params": (I32, [P] * 2),
    "qmb200_sim_step": (I32, [P, D] + [P] * 6),
    "qmb200_sim_step_dev": (I32, [P, D] + [P] * 7),
    "qmb200_sim_set_robot_params": (I32, [P] * 3),
    "qmb200_sim_get_robot_params": (I32, [P] * 4),
    "qmb200_sim_step_ext": (I32, [P, D] + [P] * 7),
    "qmb200_sim_step_ext_dev": (I32, [P, D] + [P] * 8),
    "qmb200_sim_set_terrain": (I32, [P, I32, I32, I32, D, P]),
    "qmb200_sim_get_terrain": (I32, [P] * 6),
    "qmb200_sim_set_robot_terrain": (I32, [P] * 3),
    "qmb200_sim_get_robot_terrain": (I32, [P] * 4),
    "qmb200_sim_standing_state": (I32, [P, I32, P, P, P]),
    "qmb200_sim_get_sensor_params": (I32, [P] * 2),
    "qmb200_sim_set_sensor_params": (I32, [P] * 2),
    "qmb200_sim_read_sensors": (I32, [P, D, I64] + [P] * 4),
    "qmb200_sim_read_sensors_dev": (I32, [P, D, I64] + [P] * 5),
    "qmb200_state_est_get_params": (I32, [P] * 2),
    "qmb200_state_est_set_params": (I32, [P] * 2),
    "qmb200_state_est_reset": (I32, [P] * 2),
    "qmb200_state_est_step": (I32, [P, D] + [P] * 4),
    "qmb200_state_est_step_dev": (I32, [P, D] + [P] * 5),
    "qmb200_state_est_get": (I32, [P] * 4),
    "qmb200_state_est_stop": (I32, [P]),
    "qmb200_state_est_set_ground": (I32, [P] * 3),
    "qmb200_state_est_get_ground": (I32, [P] * 4),
    "qmb200_attitude_get_params": (I32, [P] * 2),
    "qmb200_attitude_set_params": (I32, [P] * 2),
    "qmb200_attitude_reset": (I32, [P]),
    "qmb200_attitude_step": (I32, [P, D] + [P] * 2),
    "qmb200_attitude_step_dev": (I32, [P, D] + [P] * 3),
    "qmb200_attitude_get": (I32, [P] * 5),
    "qmb200_attitude_stop": (I32, [P]),
    "qmb200_slip_get_params": (I32, [P] * 2),
    "qmb200_slip_set_params": (I32, [P] * 2),
    "qmb200_slip_reset": (I32, [P]),
    "qmb200_slip_step": (I32, [P, D] + [P] * 5),
    "qmb200_slip_step_dev": (I32, [P, D] + [P] * 6),
    "qmb200_slip_get": (I32, [P] * 4),
    "qmb200_slip_stop": (I32, [P]),
    "qmb200_robot_image_save": (I32, [P]),
    "qmb200_robot_image_clear": (I32, [P]),
    "qmb200_robot_image_restore": (I32, [P] * 2),
    "qmb200_robot_image_restore_dev": (I32, [P] * 3),
    "qmb200_robot_state_bytes": (I64, [P]),
    "qmb200_robot_state_save_dev": (I32, [P, P, I64, P, P]),
    "qmb200_robot_state_load_dev": (I32, [P] * 7),
    "qmb200_robot_state_load": (I32, [P] * 6),
    "qmb200_fall_detect": (I32, [P, P, D, D, P, P]),
    "qmb200_fall_detect_dev": (I32, [P, P, D, D, P, P, P]),
    "qmb200_episode_set_ranges": (I32, [P, P, P, I64]),
    "qmb200_episode_get_ranges": (I32, [P] * 5),
    "qmb200_episode_sample": (I32, [P, P, P, I32, P]),
    "qmb200_episode_sample_dev": (I32, [P, P, P, I32, P, P]),
    "qmb200_episode_draw": (I32, [P, I32, P, P, P]),
    "qmb200_spawn_set_ranges": (I32, [P, P, P, I64]),
    "qmb200_spawn_get_ranges": (I32, [P] * 5),
    "qmb200_spawn_sample": (I32, [P, P, P, I32] + [P] * 8),
    "qmb200_spawn_sample_dev": (I32, [P, P, P, I32] + [P] * 9),
    "qmb200_spawn_place": (I32, [P, P, P, P, I32] + [P] * 8),
    "qmb200_spawn_place_dev": (I32, [P, P, P, P, I32] + [P] * 9),
    "qmb200_spawn_here": (I32, [P] * 6),
    "qmb200_spawn_here_dev": (I32, [P] * 7),
    "qmb200_spawn_draw": (I32, [P, I32, P, P, P]),
    "qmb200_metrics_step": (I32, [P, D] + [P] * 12),
    "qmb200_metrics_step_dev": (I32, [P, D] + [P] * 13),
    "qmb200_metrics_close": (I32, [P] * 4 + [I32] + [P] * 3),
    "qmb200_metrics_close_dev": (I32, [P] * 4 + [I32] + [P] * 4),
    "qmb200_timeline_set_ranges": (I32, [P, I32, P, P, I64]),
    "qmb200_timeline_get_ranges": (I32, [P] * 6),
    "qmb200_timeline_sample": (I32, [P] * 4),
    "qmb200_timeline_sample_dev": (I32, [P] * 5),
    "qmb200_timeline_draw": (I32, [P, I32, P, P, P]),
    "qmb200_ee_path_set_ranges": (I32, [P, P, P, I64]),
    "qmb200_ee_path_get_ranges": (I32, [P] * 5),
    "qmb200_ee_path_sample": (I32, [P] * 4),
    "qmb200_ee_path_sample_dev": (I32, [P] * 5),
    "qmb200_ee_path_draw": (I32, [P, I32] + [P] * 4),
    "qmb200_curriculum_set": (I32, [P] * 3),
    "qmb200_curriculum_attach": (I32, [P, I32, P, P]),
    "qmb200_curriculum_update": (I32, [P] * 5 + [I32] + [P] * 2),
    "qmb200_curriculum_update_dev": (I32, [P] * 5 + [I32] + [P] * 3),
    "qmb200_curriculum_get": (I32, [P] * 3),
    "qmb200_curriculum_draw": (I32, [P, I32, I32] + [P] * 4),
    "qmb200_update": (I32, [P] * 10),
    "qmb200_update_dev": (I32, [P] * 11),
    "qmb200_set_pipeline": (I32, [P, I32]),
    "qmb200_set_profiling": (I32, [P, I32]),
    "qmb200_collect_kernel_times": (I32, [P]),
    "qmb200_get_kernel_times": (I32, [P] * 2),
    "qmb200_get_flow_kernel_time": (I32, [P] * 2),
    "qmb200_measure_fp64_peak": (I32, [P] * 2),
    "qmb200_debug_get_step": (I32, [P] * 4),
    "qmb200_mpc_set_solver": (I32, [P, I32]),
    "qmb200_mpc_get_solver": (I32, [P] * 6),
    "qmb200_comm_get_unique_id": (I32, [P]),
    "qmb200_comm_init": (I32, [P, I32, I32, P]),
    "qmb200_comm_destroy": (I32, [P]),
    "qmb200_comm_info": (I32, [P] * 4),
    "qmb200_allgather_torque": (I32, [P] * 6),
    "qmb200_gait_bin_permutation": (I32, [I32] + [P] * 5),
    "qmb200_debug_model_blob": (I64, [CFG, P, I64]),
    "qmb200_debug_srbd_constants": (I32, [CFG, I32, P, P]),
    "qmb200_launch_count": (I64, [P]),
    "qmb200_stream": (P, [P]),
}
SYMBOLS = list(PROTOTYPES)

_lib = None


def load_library():
    """Load libqmb200.so; raise (never fall back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise QmbError("libqmb200.so not built (%s): run `python -c 'import __graft_entry__ as g; g.build()'` — there is no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)   # AttributeError when the build lacks a declared symbol
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def asset(name):
    return os.path.join(ASSETS, name)
