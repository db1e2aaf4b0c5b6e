"""ctypes binding of libqmb200.so (C ABI: include/qmb200.h).  Fails loudly when the library is missing."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.environ.get("QMB200_LIB", os.path.join(HERE, "libqmb200.so"))   # override only selects another build of the same library
ASSETS = os.path.join(ROOT, "assets")

NX, NU, RBD, CMD, TARGET, EMAX, KMAX = 30, 30, 55, 54, 37, 32, 4

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


# the payload estimator's parameter vector theta: the load's inertial parameters in the end-effector frame about its origin (include/qmb200.h)
THETA_LAYOUT = ("m", "mc_x", "mc_y", "mc_z", "I_xx", "I_xy", "I_xz", "I_yy", "I_yz", "I_zz")

# per-robot plant variation (include/qmb200.h: qmb200_sim_set_robot_params, qmb200_sim_step_ext): the column layouts of payload[B][8] and wrench[B][12]
PAYLOAD_LAYOUT = ("m_ee", "o_ee_x", "o_ee_y", "o_ee_z", "m_base", "o_base_x", "o_base_y", "o_base_z")
# the controller's model payload (qmb200_set_model_payload) has PAYLOAD_LAYOUT too; per robot it yields SRBD_LAYOUT (qmb200_debug_srbd_constants)
SRBD_LAYOUT = ("m",) + tuple("I_nom_%d%d" % (i, j) for i in range(3) for j in range(3)) + tuple("I_nom_inv_%d%d" % (i, j) for i in range(3) for j in range(3)) + \
              ("c_nom_x", "c_nom_y", "c_nom_z", "pad0", "pad1")
WRENCH_LAYOUT = ("f_base_x", "f_base_y", "f_base_z", "n_base_x", "n_base_y", "n_base_z", "f_ee_x", "f_ee_y", "f_ee_z", "n_ee_x", "n_ee_y", "n_ee_z")


# every symbol include/qmb200.h declares (checked by the CPU test-suite)
SYMBOLS = ["qmb200_create", "qmb200_destroy", "qmb200_last_error", "qmb200_get_dims", "qmb200_get_model_info", "qmb200_get_joint_name",
           "qmb200_wbc_update", "qmb200_wbc_update_dev", "qmb200_wbc_set_input_last", "qmb200_wbc_get_input_last", "qmb200_wbc_get_gains", "qmb200_wbc_set_gains", "qmb200_wbc_get_diagnostics", "qmb200_wbc_set_iteration_caps",
           "qmb200_mpc_solve", "qmb200_mpc_solve_dev", "qmb200_mpc_set_iterations", "qmb200_mpc_set_solver", "qmb200_mpc_get_solver", "qmb200_mpc_reset", "qmb200_mpc_set_solution", "qmb200_mpc_get_solution",
           "qmb200_policy_eval", "qmb200_policy_eval_dev", "qmb200_tick", "qmb200_tick_dev", "qmb200_centroidal_state_from_rbd",
           "qmb200_gait_schedule", "qmb200_launch_count", "qmb200_stream", "qmb200_debug_get_step",
           "qmb200_gait_create", "qmb200_gait_destroy", "qmb200_gait_insert_template", "qmb200_gait_get_mode_schedule",
           "qmb200_observation_update", "qmb200_observation_update_dev", "qmb200_target_trajectories", "qmb200_target_trajectories_dev", "qmb200_initial_ee_target",
           "qmb200_control_law", "qmb200_control_law_dev", "qmb200_set_arm_gains", "qmb200_hw_write", "qmb200_hw_write_dev", "qmb200_hw_set_delay", "qmb200_update", "qmb200_update_dev",
           "qmb200_debug_model_blob", "qmb200_comm_get_unique_id", "qmb200_comm_init", "qmb200_comm_destroy", "qmb200_comm_info", "qmb200_allgather_torque", "qmb200_gait_bin_permutation", "qmb200_set_pipeline", "qmb200_set_profiling", "qmb200_collect_kernel_times", "qmb200_get_kernel_times", "qmb200_get_flow_kernel_time", "qmb200_measure_fp64_peak",
           "qmb200_sim_get_params", "qmb200_sim_set_params", "qmb200_sim_step", "qmb200_sim_step_dev", "qmb200_sim_standing_state",
           "qmb200_sim_set_robot_params", "qmb200_sim_get_robot_params", "qmb200_sim_step_ext", "qmb200_sim_step_ext_dev",
           "qmb200_sim_set_terrain", "qmb200_sim_get_terrain", "qmb200_sim_set_robot_terrain", "qmb200_sim_get_robot_terrain",
           "qmb200_set_model_payload", "qmb200_get_model_payload", "qmb200_debug_srbd_constants",
           "qmb200_payload_est_get_params", "qmb200_payload_est_set_params", "qmb200_payload_est_reset", "qmb200_payload_est_step", "qmb200_payload_est_step_dev",
           "qmb200_payload_est_commit_dev", "qmb200_payload_est_get", "qmb200_payload_est_stop", "qmb200_get_model_payload_dev"]

_lib = None


def load_library():
    """Load libqmb200.so; raise (never fall back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise QmbError("libqmb200.so not built (%s): run `python -c 'import __graft_entry__ as g; g.build()'` — there is no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.qmb200_last_error.restype = C.c_char_p
    lib.qmb200_last_error.argtypes = [C.c_void_p]
    lib.qmb200_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
    lib.qmb200_destroy.argtypes = [C.c_void_p]
    lib.qmb200_destroy.restype = None
    lib.qmb200_debug_model_blob.restype = C.c_int64
    lib.qmb200_debug_model_blob.argtypes = [C.POINTER(Config), C.c_void_p, C.c_int64]
    lib.qmb200_launch_count.restype = C.c_int64
    lib.qmb200_launch_count.argtypes = [C.c_void_p]
    lib.qmb200_stream.restype = C.c_void_p
    lib.qmb200_stream.argtypes = [C.c_void_p]
    lib.qmb200_set_arm_gains.argtypes = [C.c_void_p, C.c_double, C.c_double]
    lib.qmb200_hw_set_delay.argtypes = [C.c_void_p, C.c_double]
    lib.qmb200_mpc_set_iterations.argtypes = [C.c_void_p, C.c_int32, C.c_double]
    lib.qmb200_initial_ee_target.restype = None
    lib.qmb200_sim_step.argtypes = [C.c_void_p, C.c_double] + [C.c_void_p] * 6
    lib.qmb200_sim_step_dev.argtypes = [C.c_void_p, C.c_double] + [C.c_void_p] * 7
    lib.qmb200_sim_step_ext.argtypes = [C.c_void_p, C.c_double] + [C.c_void_p] * 7
    lib.qmb200_sim_step_ext_dev.argtypes = [C.c_void_p, C.c_double] + [C.c_void_p] * 8
    lib.qmb200_sim_set_robot_params.argtypes = [C.c_void_p] * 3
    lib.qmb200_sim_get_robot_params.argtypes = [C.c_void_p] * 4
    lib.qmb200_sim_set_terrain.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_void_p]
    lib.qmb200_sim_get_terrain.argtypes = [C.c_void_p] * 6
    lib.qmb200_sim_set_robot_terrain.argtypes = [C.c_void_p] * 3
    lib.qmb200_sim_get_robot_terrain.argtypes = [C.c_void_p] * 4
    lib.qmb200_set_model_payload.argtypes = [C.c_void_p] * 2
    lib.qmb200_get_model_payload.argtypes = [C.c_void_p] * 3
    lib.qmb200_debug_srbd_constants.argtypes = [C.POINTER(Config), C.c_int32, C.c_void_p, C.c_void_p]
    lib.qmb200_payload_est_get_params.argtypes = [C.c_void_p, C.POINTER(PayloadEstParams)]
    lib.qmb200_payload_est_set_params.argtypes = [C.c_void_p, C.POINTER(PayloadEstParams)]
    lib.qmb200_payload_est_reset.argtypes = [C.c_void_p] * 2
    lib.qmb200_payload_est_step.argtypes = [C.c_void_p, C.c_double] + [C.c_void_p] * 3
    lib.qmb200_payload_est_step_dev.argtypes = [C.c_void_p, C.c_double] + [C.c_void_p] * 4
    lib.qmb200_payload_est_commit_dev.argtypes = [C.c_void_p] * 2
    lib.qmb200_payload_est_get.argtypes = [C.c_void_p] * 4
    lib.qmb200_payload_est_stop.argtypes = [C.c_void_p]
    lib.qmb200_get_model_payload_dev.argtypes = [C.c_void_p] * 3
    lib.qmb200_sim_standing_state.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.qmb200_gait_destroy.restype = None
    lib.qmb200_gait_destroy.argtypes = [C.c_void_p]
    lib.qmb200_gait_insert_template.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_double, C.c_double]
    lib.qmb200_gait_get_mode_schedule.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
    for name in SYMBOLS:
        getattr(lib, name)
    _lib = lib
    return lib


def asset(name):
    return os.path.join(ASSETS, name)
