"""Call-by-call replay of a closed-loop run against the oracle and the plant twin — TEST INFRASTRUCTURE ONLY.

`record(solver, fn)` runs fn() (a qm_control_b200.closed_loop.run on `solver`) with the five device calls of the loop wrapped on the solver instance:
every wrapper synchronises the device, copies its arguments to the host, calls the library, synchronises and copies what the call wrote.  Around the
MPC solve it also keeps the stored solution before and after (mpc_get_solution), around the update the WBC's last input (wbc_get_input_last).
tests/_closed_loop_cpu.run fills the same Record from its oracle restatements.

The replay_* functions restate every recorded call of one stage from that call's own recorded inputs, which are the device's outputs of the stage
before: every comparison is one call deep, nothing accumulates and the tolerances of tests/_parity.py apply.  Each raises AssertionError at the
first mismatch and returns its worst errors and coverage counts."""
import inspect
import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from _oracle import TASK, HwSimOracle, TargetOracle
from _parity import CMD_BLOCKS, MPC_TOL, PLANT_TOL, Q_BLOCKS, RBD_BLOCKS, WBC_TOL, block_errors, cmd_errors, traj_errors
from _sim_twin_terrain import robot_terrain

NOT_PD, NO_STEP, SAFETY = 8, 16, 0x10000
NEAR = 1e-9           # relative distance of a line-search acceptance test from its threshold that round-off can cross


class Record:
    """meta: friction_mu [B] or None, payload [B, 8] or None (the plant's), model_payload [B, 8] or None, terrain dict(tiles [T, ny, nx] or None, cell or
    None, tile [B], origin [B, 2]) or None (the plant's ground); calls: (stage, inputs, outputs) in call order."""

    def __init__(self):
        self.meta = {}; self.calls = []

    def add(self, stage, inp, out):
        self.calls.append((stage, inp, out))

    def of(self, stage):
        return [(i, o) for s, i, o in self.calls if s == stage]


# wrapped method -> (stage, inputs, outputs): argument names of qm_control_b200.interface.Solver
WRAPPED = {"target_trajectories_dev": ("targets", ("kind", "cmd", "t_obs", "x_obs", "ee_state", "last_ee_target"), ("n_target", "target_times", "target_states", "last_ee_target")),
           "mpc_solve_dev": ("mpc", ("prob_dev",), ()),
           "update_dev": ("update", ("rbd", "period", "t_obs", "x_obs", "joint_cmd", "arm_pos_cmd", "last_time"), ("t_obs", "x_obs", "joint_cmd", "arm_pos_cmd", "last_time", "cmd", "status")),
           "hw_write_dev": ("hw_write", ("time", "period", "joint_cmd", "joint_pos", "joint_vel"), ("effort", "status")),
           "sim_step_dev": ("sim", ("duration", "effort", "q", "v", "wrench"), ("q", "v", "rbd", "contact", "status"))}


def _host(a):
    if a is None or isinstance(a, (int, float)):
        return a
    if isinstance(a, dict):
        return {k: _host(v) for k, v in a.items()}
    return a.detach().cpu().numpy().copy()


def record(solver, fn):
    """→ (fn(), Record).  The wrappers are instance attributes of `solver`, removed again when fn returns or raises."""
    import torch
    rec = Record()

    def wrap(name, stage, ins, outs):
        orig = getattr(solver, name); sig = inspect.signature(orig)

        def call(*args, **kw):
            a = sig.bind(*args, **kw); a.apply_defaults(); a = a.arguments
            torch.cuda.synchronize()
            if not rec.meta:
                p = solver.sim_get_robot_params(); rec.meta.update(friction_mu=p["friction_mu"], payload=p["payload"], model_payload=solver.get_model_payload())
                lib, robot = solver.sim_get_terrain(), solver.sim_get_robot_terrain()
                rec.meta["terrain"] = None if robot is None else dict(tiles=None if lib is None else lib["tiles"], cell=None if lib is None else lib["cell"], **robot)
            inp = {("prob" if k == "prob_dev" else k): _host(a[k]) for k in ins}
            if stage == "mpc":
                inp["before"] = solver.mpc_get_solution()
            if stage == "update":
                inp["input_last"] = solver.wbc_get_input_last()
            orig(*args, **kw)
            torch.cuda.synchronize()
            out = {k: _host(a[k]) for k in outs}
            if stage == "mpc":
                out["after"] = solver.mpc_get_solution()
            if stage == "update":
                out["input_last"] = solver.wbc_get_input_last()
            rec.add(stage, inp, out)
        return call

    try:
        for name, (stage, ins, outs) in WRAPPED.items():
            setattr(solver, name, wrap(name, stage, ins, outs))
        return fn(), rec
    finally:
        for name in WRAPPED:
            solver.__dict__.pop(name, None)


def _robot(d, b):
    return {k: v[b:b + 1] for k, v in d.items()}


# ---------------- targets ----------------
def replay_targets(rec):
    to = TargetOracle(); worst = 0.0; n = 0
    for i, (inp, out) in enumerate(rec.of("targets")):
        B = len(inp["t_obs"])
        assert np.all(out["n_target"] == 2) and np.all(out["target_times"][:, 2:] == 0) and np.all(out["target_states"][:, 2:] == 0), i
        for b in range(B):
            times, states, le = to.target(int(inp["kind"]), inp["cmd"][b], inp["t_obs"][b], inp["x_obs"][b], inp["ee_state"][b], inp["last_ee_target"][b])
            e = max(np.max(np.abs(out["target_times"][b, :2] - times)), np.max(np.abs(out["target_states"][b, :2] - states)))
            assert e <= 1e-12, ("targets call %d robot %d: %.3e" % (i, b, e))
            np.testing.assert_array_equal(out["last_ee_target"][b], le, err_msg="targets call %d robot %d: last EE target" % (i, b))
            worst = max(worst, e); n += 1
    return dict(worst=worst, replayed=n)


# ---------------- MPC ----------------
def _sqp_settings(task=TASK):
    body = re.search(r"(?m)^sqp\s*\n\{(.*?)^\}", open(task).read(), re.S).group(1)
    val = lambda k, d: float(re.search(r"(?m)^\s*%s\s+(\S+)" % k, body).group(1)) if re.search(r"(?m)^\s*%s\s" % k, body) else d
    return dict(g_max=val("g_max", 1e-2), g_min=val("g_min", 1e-6), gamma_c=1e-6, armijo_factor=1e-4, alpha_decay=0.5)   # gamma_c, armijo: ocs2 defaults (oracle/src/mpc.h)


def acceptance_margin(dbg, s):
    """Smallest relative distance of any test of the filter line search's last trial (oracle/src/mpc.cpp takeStep) from its threshold, from the
    oracle's debug row [alpha, base cost, base dyn SSE, base eq SSE, step cost, step dyn SSE, step eq SSE, armijo, trials, ...]."""
    alpha = dbg[0] if dbg[0] > 0 else s["alpha_decay"] ** (int(dbg[8]) - 1)
    bc, sc = dbg[1], dbg[4]; bv = np.sqrt(dbg[2] + dbg[3]); sv = np.sqrt(dbg[5] + dbg[6]); am = alpha * dbg[7]
    rel = lambda a, b: abs(a - b) / max(abs(a), abs(b), 1e-300)
    m = [rel(sv, s["g_max"])]
    if sv > s["g_max"]:
        m.append(rel(sv, (1 - s["gamma_c"]) * bv))
    elif sv < s["g_min"] and bv < s["g_min"] and am < 0.0:
        m += [rel(sv, s["g_min"]), rel(bv, s["g_min"]), abs(sc - bc - s["armijo_factor"] * am) / max(abs(bc), 1e-300)]
    else:
        m += [rel(sv, s["g_min"]), rel(bv, s["g_min"]), abs(sc - (bc - s["gamma_c"] * bv)) / max(abs(bc), 1e-300), rel(sv, (1 - s["gamma_c"]) * bv)]
    return min(m)


def replay_mpc(rec, oracles, nthreads=None):
    """Every solve of every robot on oracles[b] with the device's stored solution before the call as warm start: status, step size identical,
    trajectories at MPC_TOL per block.  A robot whose last line-search trial lies within NEAR of a threshold is reported; it may disagree on the step
    only then, and at most one per run."""
    ticks = rec.of("mpc"); B = len(ticks[0][0]["prob"]["t0"]); s = _sqp_settings()
    jobs = [(i, b) for i in range(len(ticks)) for b in range(B)]

    def one(job):
        i, b = job; inp = ticks[i][0]
        try:
            return oracles[b].mpc_solve_batch(_robot(inp["prob"], b), inp["before"]["x"].shape[1], prev=_robot(inp["before"], b), nthreads=1), None
        except RuntimeError as e:
            return None, str(e)
    with ThreadPoolExecutor(nthreads or os.cpu_count() or 1) as ex:   # the oracle's error string is thread-local; ctypes drops the GIL for the call
        res = list(ex.map(one, jobs))
    worst = {}; near = []; excused = []; no_step = 0; raised = 0; warm = 0
    for (i, b), (ref, err) in zip(jobs, res):
        after = ticks[i][1]["after"]; st = int(after["status"][b]); alpha = after["step_info"][b, 0]
        warm += int(ticks[i][0]["before"]["n_nodes"][b] >= 2)
        if ref is None:
            assert st & NOT_PD and st & NO_STEP, "mpc tick %d robot %d: the oracle raised (%s), the device status is %#x" % (i, b, err, st)
            raised += 1; continue
        d = ref["dbg"][0]; margin = acceptance_margin(d, s)
        if margin < NEAR:
            near.append((i, b, margin))
        want = NO_STEP if d[0] == 0 else 0
        if st != want or alpha != d[0]:
            assert margin < NEAR, "mpc tick %d robot %d: status %#x step %r, oracle %#x step %r (acceptance margin %.2e)" % (i, b, st, alpha, want, d[0], margin)
            excused.append((i, b, margin)); continue
        no_step += int(st == NO_STEP)
        lv = traj_errors(after, ref, b, 0)
        bad = {k: v for k, v in lv.items() if not v < MPC_TOL}
        assert not bad, "mpc tick %d robot %d (status %#x): per-block relative error above %.1e: %s" % (i, b, st, MPC_TOL, bad)
        for k, v in lv.items():
            worst[k] = max(worst.get(k, 0.0), v)
    for i, b, m in near:
        print("mpc tick %d robot %d: line-search acceptance within %.2e of its threshold%s" % (i, b, m, " (step differs)" if (i, b, m) in excused else ""))
    assert len(near) <= 1, "more than one robot at a line-search threshold within round-off: %s" % near
    return dict(worst=worst, replayed=len(jobs) - raised - len(excused), excused=len(excused), warm=warm, no_step=no_step, raised=raised, near=near, ticks=len(ticks))


def replay_invariant(rec):
    """The stored solution after solve k is the one before solve k + 1: nothing between two solves (update_dev) writes it."""
    ticks = rec.of("mpc")
    for k in range(len(ticks) - 1):
        a = ticks[k][1]["after"]; b = ticks[k + 1][0]["before"]
        for key in a:
            np.testing.assert_array_equal(a[key], b[key], err_msg="stored solution %s changed between solve %d and solve %d" % (key, k, k + 1))
    return len(ticks) - 1


# ---------------- update: observation → evaluatePolicy → WBC → control law ----------------
def _policy(oracle, after, prob, b, t):
    n = int(after["n_nodes"][b]); ne = int(prob["n_events"][b])
    return oracle.evaluate_policy(after["t"][b, :n], after["event"][b, :n], after["x"][b, :n], after["u"][b, :n], prob["event_times"][b, :ne], prob["modes"][b, :ne + 1], t)


def _certified(oracle, inp, b, x_des, u_des, mode, t, cmd_dev, cmd_ref):
    """The oracle's cascade fails its own KKT certificate (DESIGN.md §5) and the device's passes it (tests/test_contact_modes_gpu.py)."""
    import test_wbc_twin_cpu as tw
    from test_contact_modes_gpu import _level_certificate
    args = (oracle, tw._gains(), 0, t, x_des, u_des, inp["rbd"][b], mode, inp["period"][b], inp["input_last"][b])
    orc = _level_certificate(*args, cmd_ref[:36])
    return not orc["ok"] and _level_certificate(*args, cmd_dev[:36])["ok"]


def replay_update(rec, oracles):
    """observation_update (t exact, x at 1e-12), evaluatePolicy on the device's current solution and schedule, WbcBase::update with the recorded
    input_last (WBC_TOL per block), control law on the device's cmd54 (joint commands to 1e-10 where they come from the policy, exact elsewhere)."""
    worst = dict(x_obs=0.0, policy=0.0, **{k: 0.0 for k in CMD_BLOCKS}); n = 0; swing = 0; certified = 0; yaw_max = np.zeros(0)
    sol = None; u = 0
    for stage, inp, out in rec.calls:
        if stage == "mpc":
            sol = (out["after"], inp["prob"]); continue
        if stage != "update":
            continue
        after, prob = sol; B = len(inp["t_obs"])
        if not len(yaw_max):
            yaw_max = np.zeros(B)
        for b in range(B):
            o = oracles[b]; tag = "update %d robot %d" % (u, b)
            t, x = o.observation_update(inp["rbd"][b], inp["period"][b], inp["t_obs"][b], inp["x_obs"][b])
            assert out["t_obs"][b] == t, (tag, out["t_obs"][b], t)
            ex = float(np.max(np.abs(out["x_obs"][b] - x))); assert ex <= 1e-12, (tag, "x_obs", ex)
            yaw_max[b] = max(yaw_max[b], abs(out["x_obs"][b, 9]))
            t = out["t_obs"][b]; x = out["x_obs"][b]
            xd, ud, mode = _policy(o, after, prob, b, t); swing += int(mode != 15)
            ep = float(np.max(np.abs(out["input_last"][b] - ud))); assert ep <= 1e-10, (tag, "WBC input_last after the update vs the policy input", ep)
            cmd, il, _ = o.wbc_update(xd, ud, inp["rbd"][b], mode, inp["period"][b], t, inp["input_last"][b])
            lv = cmd_errors(out["cmd"][b], cmd)
            if not all(v < WBC_TOL for v in lv.values()):
                assert _certified(o, inp, b, xd, ud, mode, t, out["cmd"][b], cmd), "%s (mode %d): per-block relative error above %.1e: %s" % (tag, mode, WBC_TOL, lv)
                certified += 1
            else:
                for k, v in lv.items():
                    worst[k] = max(worst[k], v)
            jc, ap, lt, safe = o.control_law(0, 0.0, 0.5, xd, ud, out["cmd"][b], t, x, inp["joint_cmd"][b], inp["arm_pos_cmd"][b], inp["last_time"][b])
            jd = out["joint_cmd"][b]
            e = float(np.max(np.abs(jd[:, :2] - jc[:, :2]))); assert e <= 1e-10, (tag, "joint position / velocity commands", e)
            np.testing.assert_array_equal(jd[:, 2:], jc[:, 2:], err_msg=tag + ": joint gains / torques")
            np.testing.assert_array_equal(out["arm_pos_cmd"][b], ap, err_msg=tag); assert out["last_time"][b] == lt, tag
            assert (out["status"][b] & SAFETY != 0) == (not safe) and out["status"][b] & 0xFF == 0, (tag, hex(int(out["status"][b])))
            worst["x_obs"] = max(worst["x_obs"], ex); worst["policy"] = max(worst["policy"], ep, e); n += 1
        u += 1
    return dict(worst=worst, replayed=n, updates=u, swing=swing, certified=certified, yaw_max=yaw_max)


# ---------------- QMHWSim::writeSim ----------------
def replay_hw_write(rec, delay):
    sims = None; n = 0
    for i, (inp, out) in enumerate(rec.of("hw_write")):
        B = len(inp["time"]); sims = sims or [HwSimOracle(delay) for _ in range(B)]
        assert np.all(out["status"] == 0), (i, out["status"])
        for b in range(B):
            eff = sims[b].write(inp["time"][b], inp["period"][b], inp["joint_cmd"][b], inp["joint_pos"][b], inp["joint_vel"][b])
            np.testing.assert_array_equal(out["effort"][b], eff, err_msg="hw_write call %d robot %d" % (i, b))
            n += 1
    return dict(replayed=n)


# ---------------- plant ----------------
def replay_plant(rec, twin, every=1):
    """Every `every`-th plant step of every robot on the twin (a tests/_sim_twin_terrain.SimTwinTerrain) with the robot's friction, payload, wrench and
    ground of that step, at PLANT_TOL per block; contact mask and status exact."""
    mu, pl, ter = rec.meta.get("friction_mu"), rec.meta.get("payload"), rec.meta.get("terrain"); worst = {}; n = 0; pushed = 0
    for i, (inp, out) in enumerate(rec.of("sim")):
        if i % every:
            continue
        B = len(inp["q"]); w = inp["wrench"]
        for b in range(B):
            wb = None if w is None else w[b]; pushed += int(wb is not None and np.any(wb != 0))
            q, v, rbd, c, st = twin.step_ext(inp["duration"], inp["effort"][b], inp["q"][b], inp["v"][b], None if mu is None else mu[b], None if pl is None else pl[b], wb,
                                             terrain=robot_terrain(ter, b))
            assert out["contact"][b] == c and out["status"][b] == st, ("plant step %d robot %d" % (i, b), out["contact"][b], c, out["status"][b], st)
            for name, a, r, blocks in (("q", out["q"][b], q, Q_BLOCKS), ("v", out["v"][b], v, Q_BLOCKS), ("rbd", out["rbd"][b], rbd, RBD_BLOCKS)):
                err = block_errors(a, r, blocks)
                assert max(err.values()) < PLANT_TOL, ("plant step %d robot %d" % (i, b), name, err)
                for k, e in err.items():
                    worst[name + ":" + k] = max(worst.get(name + ":" + k, 0.0), e)
            n += 1
    return dict(worst=worst, replayed=n, pushed=pushed)
