"""End-effector commands on the GPU: the per-robot target call against the oracle's target front-end, the device step against the host-compiled core
(tests/gait_host_ee.cpp) bit for bit, a closed loop's target calls replayed on the oracle, the byte-identity of a timeline without end-effector
commands, and closed loops that reach goals standing and walking and follow an ee_cmd_vel stream.  Every run starts at yaw 0: the base target of both
end-effector commands is the hand's target minus (0.52, 0.09) in the world frame (DESIGN.md §4.8)."""
import numpy as np
import pytest

import qm_control_b200 as q
from qm_control_b200 import closed_loop
from qm_control_b200._lib import EMAX, KMAX, TARGET
from _gait_protocol import NAMES
from _oracle import TargetOracle
from test_ee_commands_cpu import Core, ee_timelines, geh, unit_quat  # noqa: F401  (geh: the host core's fixture)

pytestmark = pytest.mark.gpu
T_START = closed_loop.T_START
EE0 = np.array([0.52, 0.09, 0.44, 0.5, -0.5, 0.5, -0.5])   # qmb200_initial_ee_target


def quat_mul(a, b):
    """Hamilton product of xyzw quaternions (rows)"""
    ax, ay, az, aw = np.moveaxis(a, -1, 0); bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw,
                     aw * bw - ax * bx - ay * by - az * bz], -1)


def axis_angle(axis, angle):
    axis = axis / np.linalg.norm(axis, axis=-1, keepdims=True)
    return np.concatenate([axis * np.sin(angle / 2)[..., None], np.cos(angle / 2)[..., None]], -1)


def ori_err_deg(qa, qb):
    return np.degrees(2.0 * np.arccos(np.clip(np.abs(np.sum(qa * qb, axis=-1)), 0.0, 1.0)))


def _inputs(rng, B):
    """plausible target-call inputs: bases near the origin at small attitude, end effectors near their default pose, cmd rows whose 3:7 is a unit quaternion"""
    x = np.zeros((B, 30)); x[:, 6:9] = rng.uniform(-0.5, 0.5, (B, 3)); x[:, 8] += 0.45; x[:, 9] = rng.uniform(-3, 3, B); x[:, 10:12] = rng.uniform(-0.1, 0.1, (B, 2))
    ee = np.tile(EE0, (B, 1)); ee[:, :3] += rng.uniform(-0.2, 0.2, (B, 3)); ee[:, 3:] = quat_mul(axis_angle(rng.normal(size=(B, 3)), rng.uniform(0, 0.4, B)), ee[:, 3:])
    cmd = np.zeros((B, 7)); cmd[:, :3] = EE0[:3] + rng.uniform(-0.3, 0.3, (B, 3)); cmd[:, 3:] = np.array([unit_quat(rng) for _ in range(B)])
    le = np.tile(EE0, (B, 1)); le[:, :3] += rng.uniform(-0.15, 0.15, (B, 3))
    return cmd, T_START + rng.uniform(0, 5, B), x, ee, le


def test_per_robot_target_call_matches_the_oracle():
    """256 robots, kinds drawn from {-1, 0, 1, 2}: each robot's target and last_ee_target as the oracle's for its kind (1e-12, last_ee_target exact);
    a held robot's (-1) rows byte-unchanged; uniform kinds byte-identical to the scalar entry point, host and device."""
    import torch
    rng = np.random.default_rng(3); B = 256; s = q.Solver(batch=B); to = TargetOracle()
    cmd, t, x, ee, le = _inputs(rng, B)
    kinds = rng.integers(-1, 3, B).astype(np.int32)
    prior = (rng.integers(1, 4, B).astype(np.int32), rng.normal(size=(B, KMAX)), rng.normal(size=(B, KMAX, TARGET)))
    nt, tt, ts, le2 = s.target_trajectories(kinds, cmd, t, x, ee, le, target=prior)
    worst = 0.0
    for b in range(B):
        if kinds[b] < 0:
            assert nt[b] == prior[0][b] and tt[b].tobytes() == prior[1][b].tobytes() and ts[b].tobytes() == prior[2][b].tobytes() and le2[b].tobytes() == le[b].tobytes(), b
            continue
        times, states, le_ref = to.target(int(kinds[b]), cmd[b], t[b], x[b], ee[b], le[b])
        e = max(np.max(np.abs(tt[b, :2] - times)), np.max(np.abs(ts[b, :2] - states)))
        assert e <= 1e-12 and nt[b] == 2 and np.all(tt[b, 2:] == 0) and np.all(ts[b, 2:] == 0), (b, kinds[b], e)
        np.testing.assert_array_equal(le2[b], le_ref, err_msg="robot %d: last EE target" % b); worst = max(worst, e)
    print("worst %.2e over %d robots, %d held" % (worst, np.sum(kinds >= 0), np.sum(kinds < 0)))
    dev = torch.device("cuda", 0); T = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=dev)
    for k in (0, 1, 2):
        want = s.target_trajectories(k, cmd, t, x, ee, le)
        got = s.target_trajectories(np.full(B, k, dtype=np.int32), cmd, t, x, ee, le)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(want, got)), k
        outs = []
        for kind in (k, T(np.full(B, k, dtype=np.int32))):
            o = [T(le), torch.zeros(B, dtype=torch.int32, device=dev), torch.zeros((B, KMAX), dtype=torch.float64, device=dev),
                 torch.zeros((B, KMAX, TARGET), dtype=torch.float64, device=dev)]
            torch.cuda.synchronize(); s.target_trajectories_dev(kind, T(cmd), T(t), T(x), T(ee), *o); torch.cuda.synchronize(); outs.append([a.cpu().numpy() for a in o])
        assert all(a.tobytes() == b.tobytes() for a, b in zip(*outs)) and outs[0][3].tobytes() == want[2].tobytes(), k
    with pytest.raises(q.QmbError, match="outside"):
        s.target_trajectories(np.full(B, 3, dtype=np.int32), cmd, t, x, ee, le)
    s.close()


class Device:
    """the handle's device schedule behind the interface of test_ee_commands_cpu.Core, through the host-pointer step with target_kind"""

    def __init__(self, solver):
        self.s = solver; B = solver.batch; solver.gait_dev_set_templates()
        self.n_events = np.zeros(B, dtype=np.int32); self.ev = np.zeros((B, EMAX)); self.md = np.full((B, EMAX + 1), 15, dtype=np.int32); self.cmd = np.zeros((B, 7))

    def step(self, t_obs):
        kind = np.zeros(self.s.batch, dtype=np.int32)
        tm, mode, st = self.s.gait_dev_step(t_obs, dict(n_events=self.n_events, event_times=self.ev, modes=self.md), self.cmd, target_kind=kind)
        return tm, mode, st, kind


def test_device_step_matches_the_host_core(geh):
    """256 robots, 500 ticks, random timelines of gait, cmd_vel, ee_cmd_vel and goal rows: windows, cmd rows, templates, modes, status and target kinds
    bit for bit against the host-compiled core; the sources and cursors at the end as well."""
    rng = np.random.default_rng(13); B = 256; s = q.Solver(batch=B)
    gait0 = [NAMES[b % len(NAMES)] for b in range(B)]; t_start = T_START + rng.uniform(0.0, 1.0, size=B)
    t, tmpl, vel, kind, ee = ee_timelines(rng, B, t_start, 30, 5.0)
    dev, host = Device(s), Core(geh, B)
    s.gait_dev_reset(gait0, t_start); s.gait_dev_set_commands(t, tmpl, vel, ee_kind=kind, ee_cmd=ee)
    host.reset(gait0, t_start); host.set_commands(t, tmpl, vel, kind, ee)
    t_obs = t_start - 0.002; seen = np.zeros(4, dtype=np.int64)
    for i in range(500):
        tt = t_obs.copy()
        if i == 30:
            tt[7] = np.nan
        a, b = dev.step(tt), host.step(tt)
        for x, y, what in zip(a, b, ("tmpl", "mode", "status", "target_kind")):
            assert x.tobytes() == y.tobytes(), (i, what)
        for what in ("n_events", "ev", "md", "cmd"):
            assert getattr(dev, what).tobytes() == getattr(host, what).tobytes(), (i, what)
        seen += np.bincount(a[3] + 1, minlength=4); t_obs = t_obs + 0.01
    g = s.gait_dev_get(); src, cur = host.get(); assert np.array_equal(g["cursor"], cur)
    print("target kinds -1/0/1/2 seen %s times" % seen.tolist())
    assert np.all(seen > 100)
    s.gait_dev_stop(); s.close()


def test_entry_points_validate_end_effector_rows():
    s = q.Solver(batch=2); s.gait_dev_set_templates(["stance", "trot"]); s.gait_dev_reset(["stance", "trot"], 10.0)
    t = [[0.0], [0.0]]; tm = [[-1], [-1]]; nan4 = np.full((2, 1, 4), np.nan)
    goal = np.tile(EE0, (2, 1, 1))
    for vel, kind, ee, match in ((nan4, [[3], [-1]], goal, "ee_kind"), (np.zeros((2, 1, 4)), [[2], [-1]], goal, "both"),
                                 (nan4, [[1], [-1]], np.full((2, 1, 7), np.nan), "finite"), (nan4, [[2], [-1]], goal * [1, 1, 1, 1, 1, 1, 1.001], "unit norm")):
        with pytest.raises(q.QmbError, match=match):
            s.gait_dev_set_commands(t, tm, vel, ee_kind=kind, ee_cmd=ee)
    ok = goal.copy(); ok[1, 0] = [0.1, 0.0, 0.0] + [np.nan] * 4   # an ee_cmd_vel row ignores its columns 3:7
    s.gait_dev_set_commands(t, tm, nan4, ee_kind=[[2], [1]], ee_cmd=ok)
    s.gait_dev_stop(); s.close()


def _record_targets(solver, fn):
    """→ (fn(), calls): every target_trajectories_dev of the run with its inputs, the target rows before and after, on the host"""
    import torch
    calls = []; orig = solver.target_trajectories_dev
    H = lambda a: a.detach().cpu().numpy().copy() if hasattr(a, "detach") else a

    def call(kind, cmd, t_obs, x_obs, ee_state, last_ee_target, n_target, target_times, target_states, stream=None):
        torch.cuda.synchronize()
        inp = dict(kind=H(kind), cmd=H(cmd), t_obs=H(t_obs), x_obs=H(x_obs), ee_state=H(ee_state), last_ee_target=H(last_ee_target), n_target=H(n_target),
                   target_times=H(target_times), target_states=H(target_states))
        orig(kind, cmd, t_obs, x_obs, ee_state, last_ee_target, n_target, target_times, target_states, stream)
        torch.cuda.synchronize()
        calls.append((inp, dict(last_ee_target=H(last_ee_target), n_target=H(n_target), target_times=H(target_times), target_states=H(target_states))))
    solver.target_trajectories_dev = call
    try:
        return fn(), calls
    finally:
        del solver.target_trajectories_dev


def _mixed(B, rng):
    """1 s, stance: cmd_vel, ee_cmd_vel and goal rows at least 20 ms apart, in a random order per robot, goals within 0.1 m of the default pose"""
    C = 6
    t = np.array([np.sort(rng.choice(np.arange(0.0, 0.95, 0.02), size=C, replace=False)) for _ in range(B)])
    what = rng.integers(0, 3, (B, C)); what[:, 0] = 2; what[:, 3] = 2   # at least two goals per robot
    vel = np.full((B, C, 4), np.nan); goal = np.full((B, C, 7), np.nan); eev = np.full((B, C, 3), np.nan)
    vel[what == 0] = [0.0, 0.0, 0.0, 0.0]
    eev[what == 1] = rng.uniform(-0.05, 0.05, (np.sum(what == 1), 3))
    n = np.sum(what == 2); goal[what == 2] = np.c_[EE0[:3] + rng.uniform(-0.1, 0.1, (n, 3)), quat_mul(axis_angle(rng.normal(size=(n, 3)), rng.uniform(0, 0.2, n)), np.tile(EE0[3:], (n, 1)))]
    return dict(t=t, gait=np.full((B, C), None, dtype=object), cmd_vel=vel, ee_goal=goal, ee_cmd_vel=eev), what


def test_loop_replays_every_target_call_on_the_oracle():
    """16 robots at the origin, 1 s of stance with mixed rows: every target call replayed on the oracle with its recorded inputs (1e-12, last_ee_target
    exact) for the robots whose kind is not -1; held robots' rows unchanged by the call; each goal row published exactly once, by the first step at or
    after its time; the record's target_kind and ee_target are the calls'."""
    rng = np.random.default_rng(21); B = 16; s = q.Solver(batch=B)
    commands, what = _mixed(B, rng)
    r, calls = _record_targets(s, lambda: closed_loop.run(s, duration=1.0, gait="stance", commands=commands))
    to = TargetOracle(); worst = 0.0; n = 0; held = 0
    assert len(calls) == len(r["t"])
    for i, (inp, out) in enumerate(calls):
        kind = inp["kind"]; np.testing.assert_array_equal(kind, r["target_kind"][i])
        np.testing.assert_array_equal(out["target_states"][:, 1, 30:37], r["ee_target"][i])
        for b in range(B):
            if kind[b] < 0:
                assert all(inp[k][b].tobytes() == out[k][b].tobytes() for k in out), (i, b); held += 1; continue
            times, states, le = to.target(int(kind[b]), inp["cmd"][b], inp["t_obs"][b], inp["x_obs"][b], inp["ee_state"][b], inp["last_ee_target"][b])
            e = max(np.max(np.abs(out["target_times"][b, :2] - times)), np.max(np.abs(out["target_states"][b, :2] - states)))
            assert e <= 1e-12, (i, b, e)
            np.testing.assert_array_equal(out["last_ee_target"][b], le, err_msg="call %d robot %d" % (i, b)); worst = max(worst, e); n += 1
    t_obs = np.array([c[0]["t_obs"][0] for c in calls])
    for b in range(B):
        due = [T_START + tc for tc, w in zip(commands["t"][b], what[b]) if w == 2 and T_START + tc <= t_obs[-1]]
        pub = np.flatnonzero(r["target_kind"][:, b] == 2)
        assert len(pub) == len(due) and all(t_obs[p] >= d and (p == 0 or t_obs[p - 1] < d) for p, d in zip(pub, due)), (b, pub, due)
    print("replayed %d robot calls (worst %.2e), %d held" % (n, worst, held))
    assert held > 0 and n > 0
    s.close()


def _same(a, b, keys=("base", "ee", "status", "q", "v", "target_kind", "ee_target")):
    return {k: a[k].tobytes() == b[k].tobytes() for k in keys}


def test_empty_end_effector_arrays_leave_the_run_byte_identical():
    """64 robots, 1 s of trot with gait / cmd_vel rows: the run with all-NaN ee_goal and ee_cmd_vel arrays equals the run without them, byte for byte."""
    B = 64; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]; cmd = (0.2, 0.0, 0.0, 0.0)
    commands = dict(t=np.tile([0.0, 0.3, 0.61], (B, 1)), gait=np.tile(np.array([None, "pace", None], dtype=object), (B, 1)), cmd_vel=np.tile([[np.nan] * 4, cmd, cmd], (B, 1, 1)))
    runs = []
    for extra in ({}, dict(ee_goal=np.full((B, 3, 7), np.nan), ee_cmd_vel=np.full((B, 3, 3), np.nan))):
        s.mpc_reset(); s.wbc_set_input_last(None)
        runs.append(closed_loop.run(s, duration=1.0, gait="trot", cmd_vel=cmd, xy_yaw=xy, commands=dict(commands, **extra)))
    print(_same(*runs))
    assert all(_same(*runs).values()) and np.all(runs[0]["target_kind"] == 0)
    s.close()


def _start_ee(s, xy):
    r = closed_loop.run(s, duration=0.01, gait="stance", xy_yaw=xy); s.mpc_reset(); s.wbc_set_input_last(None)
    return r["start_ee"]


def _reach(r, goal, tail=10):
    """→ (position error [B] m, orientation error [B] deg) of the end effector against goal over the last `tail` records (the worst)"""
    ee = r["ee"][-tail:]
    return np.max(np.linalg.norm(ee[:, :, :3] - goal[None, :, :3], axis=2), axis=0), np.max(ori_err_deg(ee[:, :, 3:], goal[None, :, 3:]), axis=0)


def _up(r):
    base = r["base"]
    return np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3)


# Bounds from the first H100 run with margin; the values observed are in DESIGN.md §8 (stance: worst 0.039 m / 10.5 deg, median 0.011 m / 4.8 deg;
# walking: worst 0.003 m / 0.7 deg; ee_cmd_vel: 0.0246 m of the 0.05 m commanded).
STANCE_POS_M, STANCE_ORI_DEG, STANCE_POS_M_P50, STANCE_ORI_DEG_P50 = 0.06, 15.0, 0.02, 8.0
WALK_POS_M, WALK_ORI_DEG = 0.01, 3.0


def test_stance_reach():
    """64 robots standing at yaw 0, one goal each at 0.2 s within +-0.1 m and up to 15 deg of the start pose.  The goal's reach time is at most
    max(0.17 m / 0.3 m/s, 0.26 rad / 0.1 rad/s) = 2.6 s (targetDisplacementVelocity, targetRotationVelocity); 5 s leave over 2 s to settle.
    Everyone stays up with no status bit; the pose errors over the last 0.1 s stay under the bounds (they are not small: reaching up or down and
    turning the hand leave centimetres and degrees, DESIGN.md §8)."""
    rng = np.random.default_rng(31); B = 64; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    ee0 = _start_ee(s, xy)
    goal = ee0.copy(); goal[:, :3] += rng.uniform(-0.1, 0.1, (B, 3))
    goal[:, 3:] = quat_mul(axis_angle(rng.normal(size=(B, 3)), np.radians(rng.uniform(0, 15, B))), ee0[:, 3:])
    r = closed_loop.run(s, duration=5.0, gait="stance", xy_yaw=xy, commands=dict(t=np.full((B, 1), 0.2), gait=np.full((B, 1), None, dtype=object), ee_goal=goal[:, None]))
    pe, oe = _reach(r, goal)
    print("stance reach: position error p50 %.4f max %.4f m, orientation p50 %.2f max %.2f deg, status %s, up %d / %d" % (
        np.median(pe), pe.max(), np.median(oe), oe.max(), np.unique(r["status"]), _up(r).sum(), B))
    assert np.sum(r["target_kind"] == 2) == B and np.all(r["target_kind"][-1] == -1)
    assert np.all(_up(r)) and np.all(r["status"] == 0)
    assert pe.max() < STANCE_POS_M and oe.max() < STANCE_ORI_DEG and np.median(pe) < STANCE_POS_M_P50 and np.median(oe) < STANCE_ORI_DEG_P50
    s.close()


def test_walk_to_reach():
    """64 robots trotting at yaw 0, one goal each at 0.2 s 0.3-0.5 m ahead of the start pose (reach time at most 1.7 s), stance commanded at 2.5 s
    (in force from 3.5 s), 5 s in all: everyone up with no status bit, final pose errors under the bounds."""
    rng = np.random.default_rng(41); B = 64; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    ee0 = _start_ee(s, xy)
    goal = ee0.copy(); goal[:, 0] += rng.uniform(0.3, 0.5, B)
    nan7 = np.full((B, 7), np.nan)
    commands = dict(t=np.tile([0.2, 2.5], (B, 1)), gait=np.tile(np.array([None, "stance"], dtype=object), (B, 1)), ee_goal=np.stack([goal, nan7], 1))
    r = closed_loop.run(s, duration=5.0, gait="trot", xy_yaw=xy, commands=commands)
    pe, oe = _reach(r, goal); moved = r["base"][-1, :, 0] - r["start_base"][:, 0]
    print("walk to reach: base moved %.3f..%.3f m, position error p50 %.4f max %.4f m, orientation p50 %.2f max %.2f deg, status %s, up %d / %d" % (
        moved.min(), moved.max(), np.median(pe), pe.max(), np.median(oe), oe.max(), np.unique(r["status"]), _up(r).sum(), B))
    assert np.all(_up(r)) and np.all(r["status"] == 0)
    assert pe.max() < WALK_POS_M and oe.max() < WALK_ORI_DEG
    s.close()


def test_ee_cmd_vel_stream():
    """64 robots standing at yaw 0: ee_cmd_vel (0.05, 0, 0) from 0.2 s, zeros from 1.2 s, 3 s in all.  Every target call from 0.2 s on takes kind 1,
    whose target leads the hand by v * timeHorizon and keeps last_ee_target's height and orientation.  The hand moves in x by about half the
    commanded 0.05 m (the MPC trails the moving target; 0.0246 m on the first H100 run), its height stays near the target's and the target's height
    never changes."""
    B = 64; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    commands = dict(t=np.tile([0.2, 1.2], (B, 1)), gait=np.full((B, 2), None, dtype=object), ee_cmd_vel=np.tile([[0.05, 0.0, 0.0], [0.0, 0.0, 0.0]], (B, 1, 1)))
    r = closed_loop.run(s, duration=3.0, gait="stance", xy_yaw=xy, commands=commands)
    t_obs = r["t"] - 0.012
    on = t_obs >= T_START + 0.2 - 1e-9
    assert np.all(r["target_kind"][on] == 1) and np.all(r["target_kind"][~on] == 0)
    dx = r["ee"][-1, :, 0] - r["start_ee"][:, 0]; dz = np.abs(r["ee"][-1, :, 2] - r["ee_target"][-1, :, 2]); tz = np.ptp(r["ee_target"][on][:, :, 2], axis=0)
    print("ee_cmd_vel: moved %.4f..%.4f m in x, |z - target z| at the end %.4f m at most, target z spread %.2e, status %s" % (dx.min(), dx.max(), dz.max(), tz.max(),
                                                                                                                           np.unique(r["status"])))
    assert np.all(_up(r)) and np.all(r["status"] == 0)
    assert np.all(tz == 0.0) and dz.max() < 0.02 and 0.015 < dx.min() and dx.max() < 0.06
    s.close()
