"""CPU rehearsal of qm_control_b200.closed_loop.run for one robot — TEST INFRASTRUCTURE ONLY.

The oracle's restatements of the controller (target publisher, SQP MPC, evaluatePolicy, WBC, control law, QMHWSim::writeSim) drive the plant
twin (tests/sim_twin.cpp) at the rates of closed_loop.run: MPC every 10 ms, QMController::update every WBC period, writeSim + physics step every 1 ms.
With a recorder (tests/_loop_replay.Record) every call is recorded in the format of tests/_loop_replay.record, with a batch of one robot."""
import numpy as np

from _oracle import EMAX, KMAX, HwSimOracle, TargetOracle
from _sim_twin import SimTwin


def standing_state(oracle, twin, x=0.0, y=0.0, yaw=0.0):
    """qmb200_sim_standing_state restated: defaultJointState, feet sunk by m g / (4 k) below the plane (mean over the feet)."""
    mi = oracle.model_info(); q = mi["q_nominal"].copy(); q[0], q[1], q[3] = x, y, yaw
    r = oracle.rbd(q, np.zeros(24)); p = twin.params
    q[2] = p["ground_height"] + p["foot_radius"] - mi["mass"] * 9.81 / (4 * p["stiffness"]) - float(np.mean(r["foot_pos"][:, 2] - q[2]))
    return q, np.zeros(24)


def _sol(s, nmax):
    """an oracle solution (or None: none stored yet) as the handle's stored solution of one robot; status NO_STEP where the line search took no step"""
    if s is None:
        return dict(n_nodes=np.zeros(1, dtype=np.int32), t=np.zeros((1, nmax)), event=np.zeros((1, nmax), dtype=np.int32), x=np.zeros((1, nmax, 30)), u=np.zeros((1, nmax, 30)),
                    status=np.zeros(1, dtype=np.int32), step_info=np.zeros((1, 4)))
    d = s["dbg"][0]
    return dict(n_nodes=s["n_nodes"].copy(), t=s["t"].copy(), event=s["event"].copy(), x=s["x"].copy(), u=s["u"].copy(), status=np.array([16 if d[0] == 0 else 0], dtype=np.int32),
                step_info=np.array([[d[0], d[4], d[5], d[6]]]))


def run(oracle, duration=0.2, cmd_vel=(0.0, 0.0, 0.0, 0.0), wbc_period_ms=2, t_start=10.0, nmax=88, delay=0.009, mode_schedule=None, recorder=None):
    twin = SimTwin(); tgt = TargetOracle(); hw = HwSimOracle(delay)
    add = recorder.add if recorder is not None else (lambda stage, inp, out: None)
    if recorder is not None:
        recorder.meta.update(friction_mu=None, payload=None, model_payload=None, terrain=None)
    a1 = lambda v: np.array([v], dtype=np.float64)

    def step(duration, effort, q, v):
        q1, v1, rbd, contact, st = twin.step(duration, effort, q, v)
        add("sim", dict(duration=duration, effort=effort[None].copy(), q=q[None].copy(), v=v[None].copy(), wrench=None),
            dict(q=q1[None], v=v1[None], rbd=rbd[None], contact=np.array([contact], dtype=np.int32), status=np.array([st], dtype=np.int32)))
        return q1, v1, rbd, contact, st

    q, v = standing_state(oracle, twin)
    q, v, rbd, contact, st = step(1e-6, np.zeros(18), q, v)
    per = wbc_period_ms * 1e-3; t_obs = t_start - per
    x_obs = oracle.centroidal_state_from_rbd(rbd)
    ev, md, ne = mode_schedule if mode_schedule is not None else (np.zeros(EMAX), np.full(EMAX + 1, 15, dtype=np.int32), 0)
    joint_cmd = np.zeros((18, 5)); arm_pos = np.zeros(6); last_time = t_obs; input_last = np.zeros(30)
    last_ee = np.array([0.52, 0.09, 0.44, 0.5, -0.5, 0.5, -0.5]); cmd = np.zeros(7); cmd[:4] = cmd_vel
    sol = None; rec = []; status = 0

    def solve():
        nonlocal last_ee, sol
        times, states, le = tgt.target(0, cmd, t_obs, x_obs, rbd[48:55], last_ee)
        tt = np.zeros((1, KMAX)); tt[0, :2] = times; ts = np.zeros((1, KMAX, 37)); ts[0, :2] = states
        add("targets", dict(kind=0, cmd=cmd[None].copy(), t_obs=a1(t_obs), x_obs=x_obs[None].copy(), ee_state=rbd[None, 48:55].copy(), last_ee_target=last_ee[None].copy()),
            dict(n_target=np.array([2], dtype=np.int32), target_times=tt, target_states=ts, last_ee_target=le[None]))
        last_ee = le
        prob = dict(t0=np.array([t_obs]), x0=x_obs[None], n_events=np.array([ne], dtype=np.int32), event_times=ev[None], modes=md[None], n_target=np.array([2], dtype=np.int32),
                    target_times=tt, target_states=ts)
        before = sol
        sol = oracle.mpc_solve_batch(prob, nmax, prev=sol, want_dbg=recorder is not None)
        if recorder is not None:
            add("mpc", dict(prob={k: np.array(v) for k, v in prob.items()}, before=_sol(before, nmax)), dict(after=_sol(sol, nmax)))

    solve()
    n_ms = int(round(duration * 1e3))
    for k in range(n_ms):
        if k % 10 == 0 and k > 0:
            solve()
        if k % wbc_period_ms == 0:
            inp = dict(rbd=rbd[None].copy(), period=a1(per), t_obs=a1(t_obs), x_obs=x_obs[None].copy(), joint_cmd=joint_cmd[None].copy(), arm_pos_cmd=arm_pos[None].copy(),
                       last_time=a1(last_time), input_last=input_last[None].copy())
            t_obs, x_obs = oracle.observation_update(rbd, per, t_obs, x_obs)
            n = int(sol["n_nodes"][0])
            x_des, u_des, mode = oracle.evaluate_policy(sol["t"][0, :n], sol["event"][0, :n], sol["x"][0, :n], sol["u"][0, :n], ev[:ne], md[:ne + 1], t_obs)
            wcmd, input_last, _ = oracle.wbc_update(x_des, u_des, rbd, mode, per, t_obs, input_last)
            joint_cmd, arm_pos, last_time, safe = oracle.control_law(0, 0.0, 0.5, x_des, u_des, wcmd, t_obs, x_obs, joint_cmd, arm_pos, last_time)
            status |= 0 if safe else 0x10000
            add("update", inp, dict(t_obs=a1(t_obs), x_obs=x_obs[None].copy(), joint_cmd=joint_cmd[None].copy(), arm_pos_cmd=arm_pos[None].copy(), last_time=a1(last_time),
                                    cmd=wcmd[None].copy(), status=np.array([0 if safe else 0x10000], dtype=np.int32), input_last=input_last[None].copy()))
        time = t_start + k * 1e-3
        effort = hw.write(time, 1e-3, joint_cmd, q[6:], v[6:])
        add("hw_write", dict(time=a1(time), period=a1(1e-3), joint_cmd=joint_cmd[None].copy(), joint_pos=q[None, 6:].copy(), joint_vel=v[None, 6:].copy()),
            dict(effort=effort[None].copy(), status=np.zeros(1, dtype=np.int32)))
        q, v, rbd, contact, st = step(1e-3, effort, q, v)
        status |= st
        if (k + 1) % 10 == 0:
            rec.append(np.r_[rbd[3:6], rbd[0:3], rbd[48:55]])
    return dict(rec=np.array(rec), status=status, contact=contact, q=q, v=v)
