"""Python mirror of qm::QMInterface (qm_interface/include/qm_interface/QMInterface.h:31-54) and the solver handle.

QMInterface only records the three files the reference constructor takes and raises the same way on missing files
(QMInterface.cpp:45,53,61); ``Solver`` owns one ``qmb200_handle`` (one per GPU) and exposes the C-ABI calls on numpy
(host) or torch-cuda (device) buffers.
"""
import ctypes as C
import os

import numpy as np

from . import _lib
from ._lib import NX, NU, RBD, CMD, TARGET, EMAX, KMAX, Config, QmbError


class QMInterface:
    def __init__(self, taskFile=None, urdfFile=None, referenceFile=None, wbcGainsFile=None):
        self.taskFile = taskFile or _lib.asset("qm_task.info")
        self.urdfFile = urdfFile or _lib.asset("qm_robot.urdf")
        self.referenceFile = referenceFile or _lib.asset("qm_reference.info")
        self.gaitFile = _lib.asset("qm_gait.info")
        self.wbcGainsFile = wbcGainsFile
        for what, path in (("Task file", self.taskFile), ("URDF file", self.urdfFile), ("targetCommand file", self.referenceFile)):
            if not os.path.exists(path):
                raise ValueError("[QMInterface] %s not found: %s" % (what, path))


def _f64(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if shape is not None and tuple(a.shape) != tuple(shape):
        raise ValueError("expected shape %s, got %s" % (shape, a.shape))
    return a


def _i32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.int32)
    if shape is not None and tuple(a.shape) != tuple(shape):
        raise ValueError("expected shape %s, got %s" % (shape, a.shape))
    return a


def _p(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return C.c_void_p(a.ctypes.data)
    return C.c_void_p(a.data_ptr())   # torch tensor (device pointer)


class Solver:
    """One qmb200_handle: batched MPC + WBC for `batch` robots on CUDA device `device`."""

    def __init__(self, interface=None, batch=1, device=0, time_horizon=0.0, dt=0.0, max_nodes=0, wbc_variant=0):
        self.lib = _lib.load_library()
        self.interface = interface or QMInterface()
        cfg = Config(self.interface.taskFile.encode(), self.interface.urdfFile.encode(), self.interface.referenceFile.encode(),
                     self.interface.wbcGainsFile.encode() if self.interface.wbcGainsFile else None, batch, device, time_horizon, dt, max_nodes, wbc_variant)
        self._cfg = cfg
        h = C.c_void_p()
        rc = self.lib.qmb200_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise QmbError("qmb200_create failed (%d): %s" % (rc, self.lib.qmb200_last_error(None).decode()))
        self.h = h
        b, n, e, k = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        self.lib.qmb200_get_dims(self.h, C.byref(b), C.byref(n), C.byref(e), C.byref(k))
        self.batch, self.nmax, self.emax, self.kmax = b.value, n.value, e.value, k.value
        mass, hor, dtt = C.c_double(), C.c_double(), C.c_double()
        self.initial_state = np.zeros(NX); self.default_joint_state = np.zeros(18)
        self.lib.qmb200_get_model_info(self.h, C.byref(mass), _p(self.initial_state), _p(self.default_joint_state), C.byref(hor), C.byref(dtt))
        self.robot_mass, self.time_horizon, self.dt = mass.value, hor.value, dtt.value

    def close(self):
        if getattr(self, "h", None):
            self.lib.qmb200_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _call(self, name, *args):
        """qmb200_<name>(h, *args); a non-zero return code raises QmbError with the handle's last error."""
        rc = getattr(self.lib, "qmb200_" + name)(self.h, *args)
        if rc != 0:
            raise QmbError("qmb200_%s failed (%d): %s" % (name, rc, self.lib.qmb200_last_error(self.h).decode()))

    @property
    def launch_count(self):
        return int(self.lib.qmb200_launch_count(self.h))

    @property
    def stream(self):
        return self.lib.qmb200_stream(self.h)

    def joint_names(self):
        out = []
        for j in range(18):
            buf = C.create_string_buffer(64); self.lib.qmb200_get_joint_name(self.h, j, buf, 64); out.append(buf.value.decode())
        return out

    # ---------------- WBC ----------------
    def wbc_update(self, x_des, u_des, rbd, mode, period, time):
        B = self.batch
        x_des = _f64(x_des, (B, NX)); u_des = _f64(u_des, (B, NU)); rbd = _f64(rbd, (B, RBD)); mode = _i32(mode, (B,)); period = _f64(period, (B,)); time = _f64(time, (B,))
        cmd = np.empty((B, CMD)); status = np.empty(B, dtype=np.int32)
        self._call("wbc_update", _p(x_des), _p(u_des), _p(rbd), _p(mode), _p(period), _p(time), _p(cmd), _p(status))
        return cmd, status

    def wbc_update_dev(self, x_des, u_des, rbd, mode, period, time, cmd, status, stream=None):
        self._call("wbc_update_dev", _p(x_des), _p(u_des), _p(rbd), _p(mode), _p(period), _p(time), _p(cmd), _p(status), stream)

    def wbc_get_gains(self):
        """→ dict of the task-formulator PD gains (WbcBase::dynamicCallback fields)."""
        g = _lib.WbcGains(); self._call("wbc_get_gains", C.byref(g))
        return {n: (list(getattr(g, n)) if hasattr(getattr(g, n), "__len__") else getattr(g, n)) for n, _ in _lib.WbcGains._fields_}

    def wbc_set_gains(self, **gains):
        """Dynamic reconfigure of the WBC gains: keyword per field of qmb200_wbc_gains; unspecified fields keep their value."""
        g = _lib.WbcGains(); self._call("wbc_get_gains", C.byref(g))
        for k, v in gains.items():
            cur = getattr(g, k)
            if hasattr(cur, "__len__"):
                for i, x in enumerate(v):
                    cur[i] = float(x)
            else:
                setattr(g, k, float(v))
        self._call("wbc_set_gains", C.byref(g))

    def wbc_set_input_last(self, input_last=None):
        self._call("wbc_set_input_last", _p(_f64(input_last, (self.batch, NU))) if input_last is not None else None)

    def wbc_get_diagnostics(self):
        """→ dict(level0_passes, level1_iterations, level2_iterations, working_set) of the last WBC update, per robot."""
        d = np.zeros(self.batch, dtype=np.int32); self._call("wbc_get_diagnostics", _p(d))
        return dict(level0_passes=d & 0xFF, level1_iterations=(d >> 8) & 0xFF, level2_iterations=(d >> 16) & 0xFF, working_set=(d >> 24) & 0xFF)

    def wbc_set_iteration_caps(self, level0_passes=0, active_set_iterations=0):
        self._call("wbc_set_iteration_caps", int(level0_passes), int(active_set_iterations))

    def wbc_get_input_last(self):
        out = np.empty((self.batch, NU)); self._call("wbc_get_input_last", _p(out)); return out

    # ---------------- MPC ----------------
    def _prob(self, prob):
        B = self.batch
        return [_f64(prob["t0"], (B,)), _f64(prob["x0"], (B, NX)), _i32(prob["n_events"], (B,)), _f64(prob["event_times"], (B, EMAX)), _i32(prob["modes"], (B, EMAX + 1)),
                _i32(prob["n_target"], (B,)), _f64(prob["target_times"], (B, KMAX)), _f64(prob["target_states"], (B, KMAX, TARGET))]

    def mpc_solve(self, prob):
        B, N = self.batch, self.nmax; a = self._prob(prob)
        out = dict(n_nodes=np.zeros(B, dtype=np.int32), t=np.zeros((B, N)), event=np.zeros((B, N), dtype=np.int32), x=np.zeros((B, N, NX)), u=np.zeros((B, N, NU)),
                   status=np.zeros(B, dtype=np.int32), step_info=np.zeros((B, 4)))
        self._call("mpc_solve", *[_p(v) for v in a], _p(out["n_nodes"]), _p(out["t"]), _p(out["event"]), _p(out["x"]), _p(out["u"]), _p(out["status"]), _p(out["step_info"]))
        return out

    def mpc_solve_dev(self, prob_dev, stream=None):
        keys = ("t0", "x0", "n_events", "event_times", "modes", "n_target", "target_times", "target_states")
        self._call("mpc_solve_dev", *[_p(prob_dev[k]) for k in keys], stream)

    SOLVERS = {"sqp": 0, "ipm": 1, "ddp": 2}

    def mpc_set_solver(self, solver):
        """'sqp' (SqpMpc, what QMController runs), 'ipm' (ipm{} block) or 'ddp' (ddp{} block, discrete-time form): include/qmb200.h."""
        self._call("mpc_set_solver", self.SOLVERS[solver] if isinstance(solver, str) else int(solver))

    def mpc_get_solver(self):
        s, it = C.c_int32(), C.c_int32(); dt, gx, gn = C.c_double(), C.c_double(), C.c_double()
        self.lib.qmb200_mpc_get_solver(self.h, C.byref(s), C.byref(it), C.byref(dt), C.byref(gx), C.byref(gn))
        return dict(solver=s.value, iterations=it.value, delta_tol=dt.value, g_max=gx.value, g_min=gn.value)

    def mpc_set_iterations(self, sqp_iterations=0, cost_tol=0.0):
        """sqp.sqpIteration / costTol (SqpSolver::runImpl loop bound and checkConvergence tolerance)."""
        self._call("mpc_set_iterations", int(sqp_iterations), float(cost_tol))

    def mpc_reset(self):
        self._call("mpc_reset")

    def mpc_set_solution(self, sol):
        B, N = self.batch, self.nmax
        self._call("mpc_set_solution", _p(_i32(sol["n_nodes"], (B,))), _p(_f64(sol["t"], (B, N))), _p(_i32(sol["event"], (B, N))), _p(_f64(sol["x"], (B, N, NX))), _p(_f64(sol["u"], (B, N, NU))))

    def mpc_get_solution(self):
        B, N = self.batch, self.nmax
        out = dict(n_nodes=np.zeros(B, dtype=np.int32), t=np.zeros((B, N)), event=np.zeros((B, N), dtype=np.int32), x=np.zeros((B, N, NX)), u=np.zeros((B, N, NU)),
                   status=np.zeros(B, dtype=np.int32), step_info=np.zeros((B, 4)))
        self._call("mpc_get_solution", _p(out["n_nodes"]), _p(out["t"]), _p(out["event"]), _p(out["x"]), _p(out["u"]), _p(out["status"]), _p(out["step_info"]))
        return out

    def policy_eval(self, t):
        B = self.batch; t = _f64(t, (B,)); xd = np.empty((B, NX)); ud = np.empty((B, NU)); mode = np.empty(B, dtype=np.int32)
        self._call("policy_eval", _p(t), _p(xd), _p(ud), _p(mode))
        return xd, ud, mode

    def tick(self, prob, t_eval, rbd, period):
        B = self.batch; a = self._prob(prob); t_eval = _f64(t_eval, (B,)); rbd = _f64(rbd, (B, RBD)); period = _f64(period, (B,))
        cmd = np.empty((B, CMD)); status = np.empty(B, dtype=np.int32)
        self._call("tick", *[_p(v) for v in a], _p(t_eval), _p(rbd), _p(period), _p(cmd), _p(status))
        return cmd, status

    def tick_dev(self, prob_dev, t_eval, rbd, period, cmd, status, stream=None):
        keys = ("t0", "x0", "n_events", "event_times", "modes", "n_target", "target_times", "target_states")
        self._call("tick_dev", *[_p(prob_dev[k]) for k in keys], _p(t_eval), _p(rbd), _p(period), _p(cmd), _p(status), stream)

    # ---------------- multi-GPU (include/qmb200.h: one NCCL all-gather of the torque rows per tick, driven from the C++ host) ----------------
    def comm_unique_id(self):
        """rank 0: the 128-byte ncclUniqueId to ship to the other ranks."""
        buf = C.create_string_buffer(128)
        if self.lib.qmb200_comm_get_unique_id(buf) != 0:
            raise QmbError("qmb200_comm_get_unique_id: %s" % self.lib.qmb200_last_error(None).decode())
        return buf.raw

    def comm_init(self, nranks, rank, unique_id):
        self._call("comm_init", int(nranks), int(rank), C.c_char_p(bytes(unique_id)))

    def comm_info(self):
        n, r, v = C.c_int32(), C.c_int32(), C.c_int32(); self.lib.qmb200_comm_info(self.h, C.byref(n), C.byref(r), C.byref(v)); return n.value, r.value, v.value

    def allgather_torque(self, cmd_dev, torque_all_dev, perm_dev=None, stream=None):
        """torque_all[r * B + i] = cmd[i, 36:54] of rank r (original robot order when perm_dev is given); device tensors."""
        self._call("allgather_torque", None, _p(cmd_dev), _p(perm_dev), _p(torque_all_dev), stream)

    def gait_bin_permutation(self, prob):
        """Host: perm[p] = original index of the robot at position p after sorting by contact phase (qmb200_gait_bin_permutation)."""
        n = len(prob["t0"]); perm = np.zeros(n, dtype=np.int32)
        rc = self.lib.qmb200_gait_bin_permutation(n, _p(_f64(prob["t0"])), _p(_i32(prob["n_events"])), _p(_f64(prob["event_times"])), _p(_i32(prob["modes"])), _p(perm))
        if rc != 0:
            raise QmbError("qmb200_gait_bin_permutation failed")
        return perm

    def set_pipeline(self, chunks):
        """Number of robot ranges the tick runs as concurrent stream chains (include/qmb200.h: qmb200_set_pipeline)."""
        self._call("set_pipeline", int(chunks))

    def set_profiling(self, on=True):
        self._call("set_profiling", 1 if on else 0)

    def collect_kernel_times(self):
        self.lib.qmb200_collect_kernel_times(self.h)

    def kernel_times(self):
        ms = np.zeros(6); self._call("get_kernel_times", _p(ms))
        d = dict(zip(("setup", "lq", "riccati", "linesearch", "policy_eval", "wbc"), ms.tolist()))
        v = C.c_double(); self._call("get_flow_kernel_time", C.byref(v)); d["lq_flow"] = v.value   # part of "lq"
        return d

    def measure_fp64_peak(self):
        v = C.c_double(); self._call("measure_fp64_peak", C.byref(v)); return v.value

    def debug_get_step(self):
        B, N = self.batch, self.nmax; dx = np.zeros((B, N, NX)); du = np.zeros((B, N, NU)); robot = np.zeros((B, 8))
        self._call("debug_get_step", _p(dx), _p(du), _p(robot)); return dx, du, robot

    # ---------------- controller side (SURVEY §8f): observation, targets, control law, plant law, QMController::update ----------------
    def observation_update(self, rbd, period, t_obs, x_obs):
        """QMController::updateStateEstimation tail (QMController.cpp:236-243) → (t_obs, x_obs) advanced."""
        B = self.batch; rbd = _f64(rbd, (B, RBD)); period = _f64(period, (B,)); t = _f64(t_obs, (B,)).copy(); x = _f64(x_obs, (B, NX)).copy()
        self._call("observation_update", _p(rbd), _p(period), _p(t), _p(x)); return t, x

    def target_trajectories(self, kind, cmd, t_obs, x_obs, ee_state, last_ee_target, target=None):
        """QmTargetTrajectoriesPublisher_node.cpp:44-208 → (n_target, target_times, target_states, last_ee_target).  kind: one kind for every robot, or
        an int32 [B] array of per-robot kinds (qmb200_target_trajectories_per_robot), where -1 leaves the robot's target and last_ee_target as they are:
        target = (n_target [B], target_times [B, KMAX], target_states [B, KMAX, TARGET]) gives the target in force (default zeros)."""
        B = self.batch; c = np.zeros((B, 7)); cmd = np.asarray(cmd, dtype=np.float64).reshape(B, -1); c[:, :cmd.shape[1]] = cmd
        t = _f64(t_obs, (B,)); x = _f64(x_obs, (B, NX)); ee = _f64(ee_state, (B, 7)); le = _f64(last_ee_target, (B, 7)).copy()
        nt = np.zeros(B, dtype=np.int32); tt = np.zeros((B, KMAX)); ts = np.zeros((B, KMAX, TARGET))
        if np.ndim(kind) == 0:
            self._call("target_trajectories", int(kind), _p(c), _p(t), _p(x), _p(ee), _p(le), _p(nt), _p(tt), _p(ts)); return nt, tt, ts, le
        if target is not None:
            nt, tt, ts = _i32(target[0], (B,)).copy(), _f64(target[1], (B, KMAX)).copy(), _f64(target[2], (B, KMAX, TARGET)).copy()
        self._call("target_trajectories_per_robot", _p(_i32(kind, (B,))), _p(c), _p(t), _p(x), _p(ee), _p(le), _p(nt), _p(tt), _p(ts)); return nt, tt, ts, le

    def initial_ee_target(self):
        v = np.zeros(7); self.lib.qmb200_initial_ee_target(_p(v)); return np.tile(v, (self.batch, 1))

    def set_arm_gains(self, kp, kd):
        self._call("set_arm_gains", float(kp), float(kd))

    def control_law(self, x_des, u_des, wbc_cmd, t_obs, x_obs, joint_cmd, arm_pos_cmd, last_time):
        """SafetyChecker + updateControlLaw (QMController.cpp:159-190 / 427-445) → (joint_cmd, arm_pos_cmd, last_time, status)."""
        B = self.batch; jc = _f64(joint_cmd, (B, 18, 5)).copy(); ap = _f64(arm_pos_cmd, (B, 6)).copy(); lt = _f64(last_time, (B,)).copy(); st = np.zeros(B, dtype=np.int32)
        self._call("control_law", _p(_f64(x_des, (B, NX))), _p(_f64(u_des, (B, NU))), _p(_f64(wbc_cmd, (B, CMD))), _p(_f64(t_obs, (B,))), _p(_f64(x_obs, (B, NX))),
                   _p(jc), _p(ap), _p(lt), _p(st)); return jc, ap, lt, st

    def hw_set_delay(self, delay):
        self._call("hw_set_delay", float(delay))

    def hw_write(self, time, period, joint_cmd, joint_pos, joint_vel):
        """QMHWSim::writeSim (QMHWSim.cpp:98-116) → (effort[B,18], status)."""
        B = self.batch; eff = np.zeros((B, 18)); st = np.zeros(B, dtype=np.int32)
        self._call("hw_write", _p(_f64(time, (B,))), _p(_f64(period, (B,))), _p(_f64(joint_cmd, (B, 18, 5))), _p(_f64(joint_pos, (B, 18))), _p(_f64(joint_vel, (B, 18))), _p(eff), _p(st))
        return eff, st

    def update(self, rbd, period, t_obs, x_obs, joint_cmd, arm_pos_cmd, last_time):
        """QMController::update (QMController.cpp:128-175) on the stored policy → (t_obs, x_obs, joint_cmd, arm_pos_cmd, last_time, cmd[B,54], status)."""
        B = self.batch; t = _f64(t_obs, (B,)).copy(); x = _f64(x_obs, (B, NX)).copy(); jc = _f64(joint_cmd, (B, 18, 5)).copy(); ap = _f64(arm_pos_cmd, (B, 6)).copy(); lt = _f64(last_time, (B,)).copy()
        cmd = np.zeros((B, CMD)); st = np.zeros(B, dtype=np.int32)
        self._call("update", _p(_f64(rbd, (B, RBD))), _p(_f64(period, (B,))), _p(t), _p(x), _p(jc), _p(ap), _p(lt), _p(cmd), _p(st))
        return t, x, jc, ap, lt, cmd, st

    # device-pointer variants of the controller side (torch-cuda tensors, no synchronisation)
    def target_trajectories_dev(self, kind, cmd, t_obs, x_obs, ee_state, last_ee_target, n_target, target_times, target_states, stream=None):
        """kind: one kind for every robot, or an int32 [B] device tensor of per-robot kinds (qmb200_target_trajectories_per_robot_dev; a robot whose
        kind lies outside [0, 2], -1 for a held goal, is left untouched)."""
        if not hasattr(kind, "data_ptr"):
            self._call("target_trajectories_dev", int(kind), _p(cmd), _p(t_obs), _p(x_obs), _p(ee_state), _p(last_ee_target), _p(n_target), _p(target_times), _p(target_states), stream)
        else:
            self._call("target_trajectories_per_robot_dev", _p(kind), _p(cmd), _p(t_obs), _p(x_obs), _p(ee_state), _p(last_ee_target), _p(n_target), _p(target_times),
                       _p(target_states), stream)

    def update_dev(self, rbd, period, t_obs, x_obs, joint_cmd, arm_pos_cmd, last_time, cmd, status, stream=None):
        self._call("update_dev", _p(rbd), _p(period), _p(t_obs), _p(x_obs), _p(joint_cmd), _p(arm_pos_cmd), _p(last_time), _p(cmd), _p(status), stream)

    def hw_write_dev(self, time, period, joint_cmd, joint_pos, joint_vel, effort, status, stream=None):
        self._call("hw_write_dev", _p(time), _p(period), _p(joint_cmd), _p(joint_pos), _p(joint_vel), _p(effort), _p(status), stream)

    # ---------------- plant (include/qmb200.h: Gazebo's physics step behind QMHWSim + readSim's contact flags) ----------------
    def sim_get_params(self):
        """→ dict of qmb200_sim_params (joint_damping as a list of 18)."""
        p = _lib.SimParams(); self._call("sim_get_params", C.byref(p))
        return {n: (list(getattr(p, n)) if n == "joint_damping" else getattr(p, n)) for n, _ in _lib.SimParams._fields_}

    def sim_set_params(self, **params):
        """Keyword per field of qmb200_sim_params; unspecified fields keep their value."""
        p = _lib.SimParams(); self._call("sim_get_params", C.byref(p))
        for k, v in params.items():
            if k == "joint_damping":
                for i, x in enumerate(v):
                    p.joint_damping[i] = float(x)
            elif k == "substeps_per_ms":
                p.substeps_per_ms = int(v)
            else:
                setattr(p, k, float(v))
        self._call("sim_set_params", C.byref(p))

    def sim_step(self, duration, effort, q, v, wrench=None):
        """One physics step of every robot (effort held for `duration` s) → (q, v, rbd[B,55], contact[B], status[B]).
        wrench: optional [B, 12] external wrenches held over the step (layout _lib.WRENCH_LAYOUT, include/qmb200.h: qmb200_sim_step_ext)."""
        B = self.batch; q = _f64(q, (B, 24)).copy(); v = _f64(v, (B, 24)).copy(); rbd = np.zeros((B, RBD)); contact = np.zeros(B, dtype=np.int32); st = np.zeros(B, dtype=np.int32)
        if wrench is None:
            self._call("sim_step", float(duration), _p(_f64(effort, (B, 18))), _p(q), _p(v), _p(rbd), _p(contact), _p(st))
        else:
            self._call("sim_step_ext", float(duration), _p(_f64(effort, (B, 18))), _p(_f64(wrench, (B, 12))), _p(q), _p(v), _p(rbd), _p(contact), _p(st))
        return q, v, rbd, contact, st

    def sim_step_dev(self, duration, effort, q, v, rbd, contact, status, stream=None, wrench=None):
        """Device-pointer variant: q, v updated in place; no synchronisation.  wrench: optional [B, 12] device tensor."""
        if wrench is None:
            self._call("sim_step_dev", float(duration), _p(effort), _p(q), _p(v), _p(rbd), _p(contact), _p(status), stream)
        else:
            self._call("sim_step_ext_dev", float(duration), _p(effort), _p(wrench), _p(q), _p(v), _p(rbd), _p(contact), _p(status), stream)

    def sim_set_robot_params(self, friction_mu=None, payload=None):
        """Per-robot plant variation kept in the handle: friction_mu [B] (a scalar is broadcast), payload [B, 8] (layout _lib.PAYLOAD_LAYOUT).
        None clears that override.  The controller does not know about the payload.  Synchronous."""
        B = self.batch
        mu = None if friction_mu is None else _f64(np.broadcast_to(np.asarray(friction_mu, dtype=np.float64), (B,)), (B,))
        pl = None if payload is None else _f64(payload, (B, 8))
        self._call("sim_set_robot_params", _p(mu), _p(pl))

    def sim_get_robot_params(self):
        """→ dict(friction_mu [B] or None, payload [B, 8] or None): None where that override is not set."""
        B = self.batch; mu = np.zeros(B); pl = np.zeros((B, 8)); mask = C.c_int32()
        self._call("sim_get_robot_params", _p(mu), _p(pl), C.byref(mask))
        return dict(friction_mu=mu if mask.value & 1 else None, payload=pl if mask.value & 2 else None)

    def set_model_payload(self, payload=None):
        """The controller's model payload [B, 8] (layout _lib.PAYLOAD_LAYOUT): what the MPC and the WBC believe each robot carries, as if its URDF had a
        fixed link with the point mass at o_ee in the end-effector frame and one at o_base in the base frame.  Independent of the plant's
        sim_set_robot_params.  None clears it.  Synchronous."""
        pl = None if payload is None else _f64(payload, (self.batch, 8))
        self._call("set_model_payload", _p(pl))

    def get_model_payload(self):
        """→ the model payload [B, 8], or None when none is set."""
        pl = np.zeros((self.batch, 8)); is_set = C.c_int32()
        self._call("get_model_payload", _p(pl), C.byref(is_set))
        return pl if is_set.value else None

    def set_robot_tuning(self, tuning=None):
        """Per-robot controller parameters (_lib.TUNING_LAYOUT): the MPC friction cone, the WBC friction pyramid, the end-effector weights, the WBC gains and
        the control law's arm gains.  tuning: dict field -> scalar or [B] ([k] or [B, k] for the vector gains); fields not named take the handle's current
        values (get_handle_tuning).  While rows are set they replace the handle's values for every robot.  None clears them.  Synchronous."""
        rows = None if tuning is None else self.robot_tuning_rows(tuning)   # held until the library has copied it
        self._call("set_robot_tuning", _p(rows))

    def robot_tuning_rows(self, tuning):
        """The rows [B, TUNING] that set_robot_tuning(tuning) stores: the handle's current values with the named fields replaced.  Raises ValueError on an
        unknown field or a value of the wrong shape; the values themselves are checked by the library."""
        B = self.batch; rows = np.repeat(self.get_handle_tuning()[None, :], B, axis=0)
        for k, v in tuning.items():
            if k not in _lib.TUNING_LAYOUT:
                raise ValueError("robot tuning: unknown field %r (one of %s)" % (k, ", ".join(_lib.TUNING_LAYOUT)))
            off, w = _lib.TUNING_LAYOUT[k]; a = np.asarray(v, dtype=np.float64)
            ok = a.shape in ((), (B, w)) or a.shape == ((B,) if w == 1 else (w,))
            if not ok:
                raise ValueError("robot tuning: %s must be a scalar, %s, got shape %s" % (k, "[%d]" % B if w == 1 else "[%d] or [%d, %d]" % (w, B, w), a.shape))
            rows[:, off:off + w] = a.reshape(B, 1) if w == 1 and a.shape == (B,) else a   # a vector field's [k] is per axis, also when B == k
        return rows

    def get_handle_tuning(self):
        """→ the handle's own values as one tuning row [TUNING]: what every robot uses while no rows are set."""
        row = np.zeros(_lib.TUNING); self._call("get_handle_tuning", _p(row)); return row

    def get_robot_tuning(self):
        """→ dict field -> [B] ([B, k] for the vector gains) of the stored rows, or None when none are set."""
        rows = np.zeros((self.batch, _lib.TUNING)); is_set = C.c_int32()
        self._call("get_robot_tuning", _p(rows), C.byref(is_set))
        if not is_set.value:
            return None
        return {k: rows[:, off] if w == 1 else rows[:, off:off + w] for k, (off, w) in _lib.TUNING_LAYOUT.items()}

    # ---------------- online payload estimate (include/qmb200.h: qmb200_payload_est_*; DESIGN.md §4.6) ----------------
    def payload_est_get_params(self):
        """→ dict of qmb200_payload_est_params."""
        p = _lib.PayloadEstParams(); self._call("payload_est_get_params", C.byref(p))
        return {n: getattr(p, n) for n, _ in _lib.PayloadEstParams._fields_}

    def payload_est_set_params(self, **params):
        """Keyword per field of qmb200_payload_est_params; unspecified fields keep their value."""
        p = _lib.PayloadEstParams(); self._call("payload_est_get_params", C.byref(p))
        names = [n for n, _ in _lib.PayloadEstParams._fields_]
        for k, v in params.items():
            if k not in names:
                raise ValueError("payload_est_set_params: unknown parameter %r (one of %s)" % (k, ", ".join(names)))
            setattr(p, k, float(v))
        self._call("payload_est_set_params", C.byref(p))

    def payload_est_reset(self, prior=None):
        """(Re)start the estimator of every robot from prior [B, 8] (layout _lib.PAYLOAD_LAYOUT; None: the current model payload, zeros when none is set).
        Sets the model payload to prior.  Synchronous."""
        pl = None if prior is None else _f64(prior, (self.batch, 8))
        self._call("payload_est_reset", _p(pl))

    def payload_est_step(self, dt, effort, rbd):
        """One RLS update per robot from the measurement rbd [B, 55] and the effort [B, 18] held over the dt s that ended at it → status [B]."""
        B = self.batch; st = np.zeros(B, dtype=np.int32)
        self._call("payload_est_step", float(dt), _p(_f64(effort, (B, 18))), _p(_f64(rbd, (B, RBD))), _p(st))
        return st

    def payload_est_step_dev(self, dt, effort, rbd, status, stream=None):
        """Device-pointer variant: status [B] int32 written; no synchronisation."""
        self._call("payload_est_step_dev", float(dt), _p(effort), _p(rbd), _p(status), stream)

    def payload_est_commit_dev(self, stream=None):
        """The estimate → the end-effector half of every robot's model payload and its SRBD constants, in stream order; no synchronisation."""
        self._call("payload_est_commit_dev", stream)

    def payload_est_get(self):
        """→ dict(theta [B, 10] (layout _lib.THETA_LAYOUT), p_diag [B, 10], samples [B]).  Synchronous."""
        B = self.batch; th = np.zeros((B, 10)); pd = np.zeros((B, 10)); n = np.zeros(B, dtype=np.int32)
        self._call("payload_est_get", _p(th), _p(pd), _p(n))
        return dict(theta=th, p_diag=pd, samples=n)

    def payload_est_stop(self):
        """Release the estimator state; the model payload keeps its last committed rows."""
        self._call("payload_est_stop")

    def get_model_payload_dev(self, out, stream=None):
        """Copy the model payload rows the kernels read into the device tensor out [B, 8] in stream order (no synchronisation)."""
        self._call("get_model_payload_dev", _p(out), stream)

    def sim_set_terrain(self, tiles=None, cell=None):
        """Heightfield tile library of the plant: tiles [T, ny, nx] absolute world z (m) on nodes `cell` m apart (qm_control_b200.terrain builds them).
        None clears the library and every robot's terrain.  Synchronous."""
        if tiles is None:
            self._call("sim_set_terrain", 0, 0, 0, 0.0, None); return
        t = _f64(tiles)
        if t.ndim != 3:
            raise ValueError("expected tiles of shape [T, ny, nx], got %s" % (t.shape,))
        self._call("sim_set_terrain", t.shape[0], t.shape[2], t.shape[1], float(cell), _p(t))

    def sim_get_terrain(self):
        """→ dict(tiles [T, ny, nx], cell), or None when no library is set."""
        n, nx, ny, cell = C.c_int32(), C.c_int32(), C.c_int32(), C.c_double()
        self._call("sim_get_terrain", C.byref(n), C.byref(nx), C.byref(ny), C.byref(cell), None)
        if n.value == 0:
            return None
        t = np.zeros((n.value, ny.value, nx.value))
        self._call("sim_get_terrain", None, None, None, None, _p(t))
        return dict(tiles=t, cell=cell.value)

    def sim_set_robot_terrain(self, tile=None, origin=None):
        """Per-robot terrain: tile [B] (-1: the flat plane; a scalar is broadcast) with its node (0, 0) at world origin [B, 2] (default zeros).
        None clears it.  Synchronous."""
        B = self.batch
        if tile is None:
            self._call("sim_set_robot_terrain", None, None); return
        t = _i32(np.broadcast_to(np.asarray(tile), (B,)), (B,))
        o = _f64(np.zeros((B, 2)) if origin is None else np.broadcast_to(np.asarray(origin, dtype=np.float64), (B, 2)), (B, 2))
        self._call("sim_set_robot_terrain", _p(t), _p(o))

    def sim_get_robot_terrain(self):
        """→ dict(tile [B], origin [B, 2]), or None when no robot terrain is set."""
        t = np.zeros(self.batch, dtype=np.int32); o = np.zeros((self.batch, 2)); is_set = C.c_int32()
        self._call("sim_get_robot_terrain", _p(t), _p(o), C.byref(is_set))
        return dict(tile=t, origin=o) if is_set.value else None

    def sim_standing_state(self, xy_yaw):
        """Nominal standing configuration at the given base (x, y, yaw) rows → (q[n,24], v[n,24]).  With robot terrain set there is one row per robot,
        each standing on its own ground."""
        xy = _f64(xy_yaw).reshape(-1, 3); n = xy.shape[0]; q = np.zeros((n, 24)); v = np.zeros((n, 24))
        self._call("sim_standing_state", n, _p(xy), _p(q), _p(v))
        return q, v

    # ---------------- sensors and base state estimate (include/qmb200.h: qmb200_sim_read_sensors, qmb200_state_est_*; DESIGN.md §4.6) ----------------
    def sim_get_sensor_params(self):
        """→ dict of qmb200_sensor_params (seed an int, the sigmas floats)."""
        p = _lib.SensorParams(); self._call("sim_get_sensor_params", C.byref(p))
        return {n: getattr(p, n) for n, _ in _lib.SensorParams._fields_}

    def sim_set_sensor_params(self, **params):
        """Keyword per field of qmb200_sensor_params; unspecified fields keep their value."""
        p = _lib.SensorParams(); self._call("sim_get_sensor_params", C.byref(p))
        names = [n for n, _ in _lib.SensorParams._fields_]
        for k, v in params.items():
            if k not in names:
                raise ValueError("sim_set_sensor_params: unknown parameter %r (one of %s)" % (k, ", ".join(names)))
            setattr(p, k, int(v) if k == "seed" else float(v))
        self._call("sim_set_sensor_params", C.byref(p))

    def sim_read_sensors(self, dt, sample, q, v, v_prev):
        """IMU and encoder readings of the plant state (q, v) [B, 24] after a step of dt s that started at v_prev → sensors [B, 46] (_lib.SENSOR_LAYOUT)."""
        B = self.batch; out = np.zeros((B, _lib.SENSORS)); q, v, v_prev = _f64(q, (B, 24)), _f64(v, (B, 24)), _f64(v_prev, (B, 24))   # held until the call returns
        self._call("sim_read_sensors", float(dt), int(sample), _p(q), _p(v), _p(v_prev), _p(out))
        return out

    def sim_read_sensors_dev(self, dt, sample, q, v, v_prev, sensors, stream=None):
        """Device-pointer variant: sensors [B, 46] written; no synchronisation."""
        self._call("sim_read_sensors_dev", float(dt), int(sample), _p(q), _p(v), _p(v_prev), _p(sensors), stream)

    def state_est_get_params(self):
        """→ dict of qmb200_state_est_params."""
        p = _lib.StateEstParams(); self._call("state_est_get_params", C.byref(p))
        return {n: getattr(p, n) for n, _ in _lib.StateEstParams._fields_}

    def state_est_set_params(self, **params):
        """Keyword per field of qmb200_state_est_params; unspecified fields keep their value."""
        p = _lib.StateEstParams(); self._call("state_est_get_params", C.byref(p))
        names = [n for n, _ in _lib.StateEstParams._fields_]
        for k, v in params.items():
            if k not in names:
                raise ValueError("state_est_set_params: unknown parameter %r (one of %s)" % (k, ", ".join(names)))
            setattr(p, k, float(v))
        self._call("state_est_set_params", C.byref(p))

    def state_est_reset(self, base_pos):
        """(Re)start the base state estimator of every robot at base_pos [B, 3], at rest, P = diag(p0).  Synchronous."""
        base_pos = _f64(base_pos, (self.batch, 3))   # a copy of a strided view must live until the call returns
        self._call("state_est_reset", _p(base_pos))

    def state_est_step(self, dt, sensors, contact, rbd_est=None):
        """One filter call per robot from sensors [B, 46] and the contact mask [B] → (rbd_est [B, 55], status [B]).  rbd_est: what a robot with a
        non-finite input keeps (default zeros)."""
        B = self.batch; out = np.zeros((B, RBD)) if rbd_est is None else _f64(rbd_est, (B, RBD)).copy(); st = np.zeros(B, dtype=np.int32)
        sensors, contact = _f64(sensors, (B, _lib.SENSORS)), _i32(contact, (B,))   # held until the call returns
        self._call("state_est_step", float(dt), _p(sensors), _p(contact), _p(out), _p(st))
        return out, st

    def state_est_step_dev(self, dt, sensors, contact, rbd_est, status, stream=None):
        """Device-pointer variant: rbd_est [B, 55] and status [B] int32 written; no synchronisation."""
        self._call("state_est_step_dev", float(dt), _p(sensors), _p(contact), _p(rbd_est), _p(status), stream)

    def state_est_get(self):
        """→ dict(x [B, 18] (layout _lib.STATE_EST_LAYOUT), p_diag [B, 18], samples [B]).  Synchronous."""
        B = self.batch; x = np.zeros((B, 18)); pd = np.zeros((B, 18)); n = np.zeros(B, dtype=np.int32)
        self._call("state_est_get", _p(x), _p(pd), _p(n))
        return dict(x=x, p_diag=pd, samples=n)

    def state_est_stop(self):
        """Release the estimator state."""
        self._call("state_est_stop")

    def state_est_set_ground(self, tile=None, origin=None):
        """The estimator's ground map on the plant's tile library: tile [B] (-1: the plane; a scalar is broadcast) with its node (0, 0) at world
        origin [B, 2] (default zeros), held apart from the plant's robot terrain.  None clears it.  It survives state_est_reset and state_est_stop.
        Synchronous."""
        B = self.batch
        if tile is None:
            self._call("state_est_set_ground", None, None); return
        t = _i32(np.broadcast_to(np.asarray(tile), (B,)), (B,))
        o = _f64(np.zeros((B, 2)) if origin is None else np.broadcast_to(np.asarray(origin, dtype=np.float64), (B, 2)), (B, 2))
        self._call("state_est_set_ground", _p(t), _p(o))

    def state_est_get_ground(self):
        """→ dict(tile [B], origin [B, 2]), or None when no ground map is set."""
        t = np.zeros(self.batch, dtype=np.int32); o = np.zeros((self.batch, 2)); is_set = C.c_int32()
        self._call("state_est_get_ground", _p(t), _p(o), C.byref(is_set))
        return dict(tile=t, origin=o) if is_set.value else None

    # ---------------- attitude filter (include/qmb200.h: qmb200_attitude_*; DESIGN.md §4.6) ----------------
    def attitude_get_params(self):
        """→ dict of qmb200_attitude_params."""
        p = _lib.AttitudeParams(); self._call("attitude_get_params", C.byref(p))
        return {n: getattr(p, n) for n, _ in _lib.AttitudeParams._fields_}

    def attitude_set_params(self, **params):
        """Keyword per field of qmb200_attitude_params; unspecified fields keep their value."""
        p = _lib.AttitudeParams(); self._call("attitude_get_params", C.byref(p))
        names = [n for n, _ in _lib.AttitudeParams._fields_]
        for k, v in params.items():
            if k not in names:
                raise ValueError("attitude_set_params: unknown parameter %r (one of %s)" % (k, ", ".join(names)))
            setattr(p, k, float(v))
        self._call("attitude_set_params", C.byref(p))

    def attitude_reset(self):
        """(Re)start the attitude filter of every robot: b_hat = 0, P = diag(p0); the next call takes its reading.  Synchronous."""
        self._call("attitude_reset")

    def attitude_step(self, dt, sensors):
        """One filter call per robot on sensors [B, 46] → (sensors [B, 46] with the filtered quaternion and the bias-corrected gyro, status [B]).  The
        input is not modified."""
        B = self.batch; out = _f64(sensors, (B, _lib.SENSORS)).copy(); st = np.zeros(B, dtype=np.int32)
        self._call("attitude_step", float(dt), _p(out), _p(st))
        return out, st

    def attitude_step_dev(self, dt, sensors, status, stream=None):
        """Device-pointer variant: sensors [B, 46] rewritten in place, status [B] int32 written; no synchronisation."""
        self._call("attitude_step_dev", float(dt), _p(sensors), _p(status), stream)

    def attitude_get(self):
        """→ dict(quat [B, 4] (xyzw as stored), gyro_bias [B, 3], p_diag [B, 6], samples [B]).  Synchronous."""
        B = self.batch; qt = np.zeros((B, 4)); bias = np.zeros((B, 3)); pd = np.zeros((B, 6)); n = np.zeros(B, dtype=np.int32)
        self._call("attitude_get", _p(qt), _p(bias), _p(pd), _p(n))
        return dict(quat=qt, gyro_bias=bias, p_diag=pd, samples=n)

    def attitude_stop(self):
        """Release the filter state."""
        self._call("attitude_stop")

    # ---------------- slip detector (include/qmb200.h: qmb200_slip_*; DESIGN.md §4.6) ----------------
    def slip_get_params(self):
        """→ dict of qmb200_slip_params."""
        p = _lib.SlipParams(); self._call("slip_get_params", C.byref(p))
        return {n: getattr(p, n) for n, _ in _lib.SlipParams._fields_}

    def slip_set_params(self, **params):
        """Keyword per field of qmb200_slip_params; unspecified fields keep their value."""
        p = _lib.SlipParams(); self._call("slip_get_params", C.byref(p))
        names = [n for n, _ in _lib.SlipParams._fields_]
        for k, v in params.items():
            if k not in names:
                raise ValueError("slip_set_params: unknown parameter %r (one of %s)" % (k, ", ".join(names)))
            if k == "hold" and v != int(v):
                raise ValueError("slip_set_params: hold must be a whole number of calls, got %r" % (v,))
            setattr(p, k, int(v) if k == "hold" else float(v))
        self._call("slip_set_params", C.byref(p))

    def slip_reset(self):
        """(Re)start the slip detector of every robot: no foot slipping, counters zero.  Synchronous."""
        self._call("slip_reset")

    def slip_step(self, dt, sensors, contact):
        """One detector call per robot from sensors [B, 46] and the contact mask [B] → (stance [B], slip [B], status [B]); stance is the mask to pass to
        state_est_step.  Needs the state estimator running."""
        B = self.batch; stance = np.zeros(B, dtype=np.int32); slip = np.zeros(B, dtype=np.int32); st = np.zeros(B, dtype=np.int32)
        sensors, contact = _f64(sensors, (B, _lib.SENSORS)), _i32(contact, (B,))   # held until the call returns
        self._call("slip_step", float(dt), _p(sensors), _p(contact), _p(stance), _p(slip), _p(st))
        return stance, slip, st

    def slip_step_dev(self, dt, sensors, contact, stance, slip, status, stream=None):
        """Device-pointer variant: stance [B], slip [B] and status [B] int32 written; no synchronisation."""
        self._call("slip_step_dev", float(dt), _p(sensors), _p(contact), _p(stance), _p(slip), _p(status), stream)

    def slip_get(self):
        """→ dict(mask [B], hold [B, 4] (calls below release while slipping), onsets [B, 4]).  Synchronous."""
        B = self.batch; m = np.zeros(B, dtype=np.int32); hold = np.zeros((B, 4), dtype=np.int32); on = np.zeros((B, 4), dtype=np.int32)
        self._call("slip_get", _p(m), _p(hold), _p(on))
        return dict(mask=m, hold=hold, onsets=on)

    def slip_stop(self):
        """Release the detector state."""
        self._call("slip_stop")

    # ---------------- per-robot restart (include/qmb200.h: qmb200_robot_image_*, qmb200_fall_detect; DESIGN.md §4.10) ----------------
    def robot_image_save(self):
        """Save the start image: the per-robot rows of every component running now (state estimator, attitude filter, slip detector, payload
        estimator, model payload rows, device gait schedule and its cursors).  Replaces any previous image.  Synchronous."""
        self._call("robot_image_save")

    def robot_image_restore(self, mask):
        """Host variant of robot_image_restore_dev: mask [B] (nonzero: restart the robot)."""
        mask = _i32(np.broadcast_to(np.asarray(mask), (self.batch,)), (self.batch,))
        self._call("robot_image_restore", _p(mask))

    def robot_image_restore_dev(self, mask, stream=None):
        """For every robot with mask[b] != 0 (int32 [B] device tensor): its imaged rows return to the image, its MPC warm starts, WBC last input and
        hw_write FIFO go back to the cold start; one launch, no synchronisation.  Fails when the image no longer matches the running components."""
        self._call("robot_image_restore_dev", _p(mask), stream)

    def robot_image_clear(self):
        """Free the start image."""
        self._call("robot_image_clear")

    def fall_detect(self, rbd, count, z_min=0.3, tilt_max=0.3):
        """Host variant of fall_detect_dev: rbd [B, 55], count [B] → (count [B] updated, fallen [B])."""
        B = self.batch; rbd = _f64(rbd, (B, RBD)); count = _i32(count, (B,)).copy(); fallen = np.zeros(B, dtype=np.int32)
        self._call("fall_detect", _p(rbd), float(z_min), float(tilt_max), _p(count), _p(fallen))
        return count, fallen

    def fall_detect_dev(self, rbd, count, fallen, z_min=0.3, tilt_max=0.3, stream=None):
        """The sweeps' fall rule on the plant's rbd [B, 55]: fallen [B] int32 = non-finite base rows, height above the plant's ground under the base
        <= z_min, or |pitch|, |roll| >= tilt_max; count [B] int32 grows by one per fallen call and drops to 0 otherwise.  No synchronisation."""
        self._call("fall_detect_dev", _p(rbd), float(z_min), float(tilt_max), _p(count), _p(fallen), stream)

    # ---------------- per-episode draws: the ranges' set / get / draw path of qmb200_episode_* and qmb200_spawn_* (kind "episode" or "spawn") ----------------
    def _ranges_set(self, kind, width, lo, hi, seed):
        if lo is None and hi is None:
            self._call(kind + "_set_ranges", None, None, 0); return
        shape = (self.batch, width); lo = _f64(lo, shape); hi = _f64(hi, shape)
        s = int(seed) & 0xFFFFFFFFFFFFFFFF
        self._call(kind + "_set_ranges", _p(lo), _p(hi), s - (1 << 64) if s >> 63 else s)

    def _ranges_get(self, kind, width):
        lo = np.zeros((self.batch, width)); hi = np.zeros_like(lo); seed = C.c_int64(); is_set = C.c_int32()
        self._call(kind + "_get_ranges", _p(lo), _p(hi), C.byref(seed), C.byref(is_set))
        return dict(lo=lo, hi=hi, seed=seed.value & 0xFFFFFFFFFFFFFFFF) if is_set.value else None

    def _ranges_draw(self, kind, width, robot, episode):
        robot = _i32(np.ravel(robot)); episode = _i32(np.ravel(episode), robot.shape); rows = np.zeros((len(robot), width))
        self._call(kind + "_draw", len(robot), _p(robot), _p(episode), _p(rows))
        return rows

    # ---------------- per-episode plant draws (include/qmb200.h: qmb200_episode_*; DESIGN.md §4.11) ----------------
    def episode_set_ranges(self, lo=None, hi=None, seed=0):
        """Per-robot ranges lo, hi [B, EPISODE] (columns _lib.EPISODE_LAYOUT) and a 64-bit seed of the per-episode draws; None clears them.  Makes sure
        the plant's robot params are set (at the values in force where they were not).  Synchronous."""
        self._ranges_set("episode", _lib.EPISODE, lo, hi, seed)

    def episode_get_ranges(self):
        """→ dict(lo [B, EPISODE], hi [B, EPISODE], seed) of the stored ranges, or None when none are set."""
        return self._ranges_get("episode", _lib.EPISODE)

    def episode_sample(self, mask, episode, link=0, rows=None):
        """Host variant of episode_sample_dev: mask [B], episode [B] → rows [B, EPISODE] (rows of unmasked robots as given, zeros by default)."""
        B = self.batch; rows = np.zeros((B, _lib.EPISODE)) if rows is None else _f64(rows, (B, _lib.EPISODE)).copy()
        mask = _i32(np.broadcast_to(np.asarray(mask), (B,)), (B,)); episode = _i32(np.broadcast_to(np.asarray(episode), (B,)), (B,))
        self._call("episode_sample", _p(mask), _p(episode), int(link), _p(rows))
        return rows

    def episode_sample_dev(self, mask, episode, rows, link=0, stream=None):
        """Every robot with mask[b] != 0 (int32 [B] device tensor) draws episode[b]'s row (int32 [B]) into rows [B, EPISODE] (float64 device tensor) and
        the plant's robot params; link (_lib.EPISODE_* bits) also writes the model payload and the tuning rows' friction coefficients.  One launch, no
        synchronisation."""
        self._call("episode_sample_dev", _p(mask), _p(episode), int(link), _p(rows), stream)

    def episode_draw(self, robot, episode):
        """Host only: robot [n] (in [0, B)), episode [n] → the rows [n, EPISODE] the sampler draws for them on the stored ranges and seed."""
        return self._ranges_draw("episode", _lib.EPISODE, robot, episode)

    # ---------------- per-episode spawns (include/qmb200.h: qmb200_spawn_*; DESIGN.md §4.12) ----------------
    def spawn_set_ranges(self, lo=None, hi=None, seed=0):
        """Per-robot ranges lo, hi [B, SPAWN] (columns _lib.SPAWN_LAYOUT) and a 64-bit seed of the per-episode spawns; None clears them.  The offsets
        count from the plant's robot terrain origins in force; with a tile bound >= 0 the robot terrain rows are made to exist.  Synchronous."""
        self._ranges_set("spawn", _lib.SPAWN, lo, hi, seed)

    def spawn_get_ranges(self):
        """→ dict(lo [B, SPAWN], hi [B, SPAWN], seed) of the stored ranges, or None when none are set."""
        return self._ranges_get("spawn", _lib.SPAWN)

    def spawn_sample(self, mask, episode, q, v, rbd, contact, x_obs, last_ee, rbd_est=None, link=0, rows=None):
        """Host variant of spawn_sample_dev on copies of the arrays → dict(rows [B, SPAWN], q, v, rbd, contact, x_obs, last_ee[, rbd_est]); unmasked
        robots keep what was given (rows: zeros by default)."""
        B = self.batch
        out = dict(rows=np.zeros((B, _lib.SPAWN)) if rows is None else _f64(rows, (B, _lib.SPAWN)).copy(), q=_f64(q, (B, 24)).copy(), v=_f64(v, (B, 24)).copy(),
                   rbd=_f64(rbd, (B, RBD)).copy(), contact=_i32(contact, (B,)).copy(), x_obs=_f64(x_obs, (B, NX)).copy(), last_ee=_f64(last_ee, (B, 7)).copy())
        if rbd_est is not None:
            out["rbd_est"] = _f64(rbd_est, (B, RBD)).copy()
        mask = _i32(np.broadcast_to(np.asarray(mask), (B,)), (B,)); episode = _i32(np.broadcast_to(np.asarray(episode), (B,)), (B,))
        self._call("spawn_sample", _p(mask), _p(episode), int(link), *(_p(out[k]) for k in ("rows", "q", "v", "rbd", "contact", "x_obs", "last_ee")), _p(out.get("rbd_est")))
        return out

    def spawn_sample_dev(self, mask, episode, rows, q, v, rbd, contact, x_obs, last_ee, rbd_est=None, link=0, stream=None):
        """Every robot with mask[b] != 0 (int32 [B] device tensor) draws episode[b]'s spawn row (int32 [B]) into rows [B, SPAWN] and stands there: the
        plant's robot terrain row (and with link _lib.SPAWN_GROUND_MAP the estimator's ground map), q, v, rbd, contact, x_obs, last_ee turned with the
        base, rbd_est when given, and the reset rows of the running estimators (float64 / int32 device tensors).  One launch, no synchronisation."""
        self._call("spawn_sample_dev", _p(mask), _p(episode), int(link), _p(rows), _p(q), _p(v), _p(rbd), _p(contact), _p(x_obs), _p(last_ee), _p(rbd_est), stream)

    def spawn_draw(self, robot, episode):
        """Host only: robot [n] (in [0, B)), episode [n] → the spawn rows [n, SPAWN] the sampler draws for them on the stored ranges and seed."""
        return self._ranges_draw("spawn", _lib.SPAWN, robot, episode)

    # ---------------- device gait schedule (include/qmb200.h: qmb200_gait_dev_*; DESIGN.md §4.7) ----------------
    def gait_dev_set_templates(self, names=None, gait_file=None):
        """Load the template table: names (default: every template of the gait file, in the order of its list) → the names, a template's id being its
        index.  Fails while the schedule runs."""
        gait_file = gait_file or self.interface.gaitFile
        names = list(gait_template_names(gait_file) if names is None else names)
        arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
        self._call("gait_dev_set_templates", gait_file.encode(), C.cast(arr, C.c_void_p), len(names))
        self.gait_templates = names
        return names

    def gait_template_ids(self, names):
        """Template names → int32 ids in the loaded table; ValueError on a name the table lacks."""
        table = getattr(self, "gait_templates", None) or []
        unknown = sorted({n for n in names if n not in table})
        if unknown:
            raise ValueError("unknown gait template(s) %s (loaded: %s)" % (", ".join(unknown), ", ".join(table)))
        return np.array([table.index(n) for n in names], dtype=np.int32)

    def gait_dev_reset(self, tmpl, t_start):
        """(Re)start every robot's schedule: stance until t_start [B], then template tmpl [B] (ids or names).  Clears the command timeline.  Synchronous."""
        B = self.batch; tmpl = list(tmpl)
        ids = self.gait_template_ids(tmpl) if any(isinstance(n, str) for n in tmpl) else _i32(tmpl, (B,))
        ids, t_start = _i32(ids, (B,)), _f64(np.broadcast_to(np.asarray(t_start, dtype=np.float64), (B,)))
        self._call("gait_dev_reset", _p(ids), _p(t_start))

    def gait_dev_set_commands(self, t, tmpl, cmd_vel, ee_kind=None, ee_cmd=None):
        """The command timeline: t [B, C] (sorted per robot, +inf pads), tmpl [B, C] (ids, -1: none), cmd_vel [B, C, 4] (NaN rows: none), and optionally
        end-effector commands (DESIGN.md §4.8): ee_kind [B, C] (-1: none, 1: ee_cmd_vel, 2: goal) with ee_cmd [B, C, 7] (ee_cmd_vel: vx, vy, vz, the rest
        ignored; goal: position, quaternion xyzw; world frame).  Every cursor goes back to 0.  Synchronous."""
        B = self.batch; t = _f64(t); n = t.shape[1] if t.ndim == 2 else -1
        t = _f64(t, (B, n)); tmpl = _i32(tmpl, (B, n)); cmd_vel = _f64(cmd_vel, (B, n, 4))
        if ee_kind is None and ee_cmd is None:
            self._call("gait_dev_set_commands", n, _p(t), _p(tmpl), _p(cmd_vel))
            return
        if ee_kind is None or ee_cmd is None:
            raise ValueError("gait_dev_set_commands: ee_kind and ee_cmd go together")
        ee_kind = _i32(ee_kind, (B, n)); ee_cmd = _f64(ee_cmd, (B, n, 7))
        self._call("gait_dev_set_commands_ee", n, _p(t), _p(tmpl), _p(cmd_vel), _p(ee_kind), _p(ee_cmd))

    def gait_dev_step(self, t_obs, prob, cmd, target_kind=None):
        """Host variant of gait_dev_step_dev: prob's n_events / event_times / modes and cmd [B, 7] are updated in place (numpy) → (tmpl [B], mode [B],
        status [B]).  target_kind: an int32 [B] numpy array that receives each robot's target kind for this tick (qmb200_gait_dev_step_ee)."""
        B = self.batch; t_obs = _f64(t_obs, (B,)); tm = np.zeros(B, dtype=np.int32); md = np.zeros(B, dtype=np.int32); st = np.zeros(B, dtype=np.int32)
        for k, a in (("n_events", (B,)), ("event_times", (B, EMAX)), ("modes", (B, EMAX + 1))):
            prob[k] = (_i32 if k != "event_times" else _f64)(prob[k], a)
        if target_kind is None:
            self._call("gait_dev_step", _p(t_obs), _p(prob["n_events"]), _p(prob["event_times"]), _p(prob["modes"]), _p(cmd), _p(tm), _p(md), _p(st))
        else:
            if not (isinstance(target_kind, np.ndarray) and target_kind.dtype == np.int32 and target_kind.shape == (B,) and target_kind.flags.c_contiguous):
                raise ValueError("gait_dev_step: target_kind must be a contiguous int32 numpy array of shape (%d,)" % B)
            self._call("gait_dev_step_ee", _p(t_obs), _p(prob["n_events"]), _p(prob["event_times"]), _p(prob["modes"]), _p(cmd), _p(tm), _p(md), _p(st), _p(target_kind))
        return tm, md, st

    def gait_dev_step_dev(self, t_obs, prob, cmd, tmpl, mode, status, stream=None, target_kind=None):
        """One step per robot at t_obs [B] on the device problem rows of prob (n_events, event_times, modes) and cmd [B, 7]; tmpl, mode (or None) and
        status [B] int32 written; target_kind (an int32 [B] device tensor or None) receives each robot's target kind for this tick, the kind
        target_trajectories_dev takes (qmb200_gait_dev_step_ee_dev); no synchronisation."""
        if target_kind is None:
            self._call("gait_dev_step_dev", _p(t_obs), _p(prob["n_events"]), _p(prob["event_times"]), _p(prob["modes"]), _p(cmd), _p(tmpl), _p(mode), _p(status), stream)
        else:
            self._call("gait_dev_step_ee_dev", _p(t_obs), _p(prob["n_events"]), _p(prob["event_times"]), _p(prob["modes"]), _p(cmd), _p(tmpl), _p(mode), _p(status),
                       _p(target_kind), stream)

    def gait_dev_get(self):
        """→ dict(n_events [B], event_times [B, GAIT_CAP], modes [B, GAIT_CAP + 1], tmpl [B], cursor [B]).  Synchronous."""
        B, cap = self.batch, _lib.GAIT_CAP
        n = np.zeros(B, dtype=np.int32); ev = np.zeros((B, cap)); md = np.zeros((B, cap + 1), dtype=np.int32); tm = np.zeros(B, dtype=np.int32); cur = np.zeros(B, dtype=np.int32)
        self._call("gait_dev_get", _p(n), _p(ev), _p(md), _p(tm), _p(cur))
        return dict(n_events=n, event_times=ev, modes=md, tmpl=tm, cursor=cur)

    def gait_dev_stop(self):
        """Release the schedules and the timeline (the template table stays)."""
        self._call("gait_dev_stop")

    # ---------------- utilities ----------------
    def centroidal_state_from_rbd(self, rbd):
        rbd = _f64(rbd); n = rbd.shape[0]; x = np.empty((n, NX))
        self._call("centroidal_state_from_rbd", n, _p(rbd), _p(x)); return x


def gait_schedule(gait_name, t_start, lo, hi, gait_file=None):
    """GaitSchedule tiling of a gait.info template → (event_times[EMAX], mode_sequence[EMAX+1], n_events)."""
    lib = _lib.load_library(); ev = np.zeros(EMAX); md = np.full(EMAX + 1, 15, dtype=np.int32)
    n = lib.qmb200_gait_schedule((gait_file or _lib.asset("qm_gait.info")).encode(), gait_name.encode(), float(t_start), float(lo), float(hi), _p(ev), _p(md))
    if n < 0:
        raise QmbError("qmb200_gait_schedule failed: " + lib.qmb200_last_error(None).decode())
    return ev, md, n


def gait_template_names(gait_file=None):
    """The template names of a gait.info file, in the order of its `list` block."""
    import re
    txt = open(gait_file or _lib.asset("qm_gait.info")).read()
    m = re.search(r"(?m)^list\s*\{(.*?)^\}", txt, re.S)
    if m is None:
        raise ValueError("no list block in %s" % gait_file)
    return [n for _, n in sorted((int(i), n) for i, n in re.findall(r"\[(\d+)\]\s+(\S+)", m.group(1)))]


class GaitSchedule:
    """ocs2::legged_robot::GaitSchedule as QMInterface::loadGaitSchedule builds it (QMInterface.cpp:455-480): stateful host object, one per robot."""

    def __init__(self, interface=None):
        self.lib = _lib.load_library(); self.interface = interface or QMInterface(); g = C.c_void_p()
        if self.lib.qmb200_gait_create(self.interface.taskFile.encode(), self.interface.referenceFile.encode(), C.byref(g)) != 0:
            raise QmbError("qmb200_gait_create failed: " + self.lib.qmb200_last_error(None).decode())
        self.g = g

    def __del__(self):
        try:
            self.lib.qmb200_gait_destroy(self.g)
        except Exception:
            pass

    def insertModeSequenceTemplate(self, gait_name, startTime, finalTime, gait_file=None):
        if self.lib.qmb200_gait_insert_template(self.g, (gait_file or self.interface.gaitFile).encode(), gait_name.encode(), float(startTime), float(finalTime)) != 0:
            raise QmbError("qmb200_gait_insert_template failed: " + self.lib.qmb200_last_error(None).decode())

    def getModeSchedule(self, lowerBoundTime, upperBoundTime):
        ev = np.zeros(EMAX); md = np.full(EMAX + 1, 15, dtype=np.int32)
        n = self.lib.qmb200_gait_get_mode_schedule(self.g, float(lowerBoundTime), float(upperBoundTime), _p(ev), _p(md))
        if n < 0:
            raise QmbError("qmb200_gait_get_mode_schedule failed: " + self.lib.qmb200_last_error(None).decode())
        return ev, md, n
