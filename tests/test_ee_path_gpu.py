"""End-effector paths on the GPU (DESIGN.md §4.20): the device target call against the host build over several ticks of mixed kinds in both frames,
runs without path robots byte-identical to the per-robot call, the gait step with path rows against the statement, and a closed loop of standing
robots tracing a square: no status bits or falls, a lower hand error against the path than the same waypoints sent as successive goals, a rewind that
replays byte for byte, a branch that continues its source's path and a respawn that returns to the cmd_vel stream; the device command check of path
indices against the table in force, the table check on the handle's own MPC horizon, and a 1 s path loop replayed call by call on the host build and
the oracle."""
import numpy as np
import pytest

import qm_control_b200 as q
from qm_control_b200 import _lib, closed_loop
from test_ee_path_cpu import FOLLOW, START, _gait_statement, host, host_target, robots, table  # noqa: F401  (host: the host build's fixture)
from test_ee_frame_cpu import h_to_world, robots as frame_robots

pytestmark = pytest.mark.gpu
KMAX, TD = _lib.KMAX, _lib.TARGET

# Bounds of the square (4 waypoints 0.75 s apart, 10 cm side, from the standing hand) traced by 256 standing robots, set from the first H100 run
# (NVIDIA H100 80GB HBM3, 700 W) with margin: 11.9 / 11.1 mm as a path and 24.4 / 29.1 mm as goals, world / heading frame (DESIGN.md §8)
SQUARE_RMS_PATH_M = 0.016      # hand position RMS against p(t) between the first and the last waypoint, every robot of a frame
SQUARE_RATIO = 0.65            # path RMS / goal-timeline RMS


def _dev(a, dtype=None):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype or torch.float64, device="cuda")


def _host(*a):
    return [x.cpu().numpy() for x in a]


def test_device_target_call_equals_the_host_build_over_ticks(host):
    """4096 robots, kinds mixed per tick (path start, follow, out-of-table, goal, held, both streams) in both frames: the device call equals the host
    build to 1e-12 (the device's sincos is not the host's) tick after tick on the carried rows; without path robots it is byte-identical to the
    per-robot call."""
    import torch
    B = 4096; s = q.Solver(batch=B); n_way, way = table(40, 51)
    s.set_ee_paths([(way[p, :n_way[p], 0], way[p, :n_way[p], 1:]) for p in range(len(n_way))])
    got_t = s.get_ee_paths()
    assert len(got_t) == 40 and all(np.array_equal(got_t[p][0], way[p, :n_way[p], 0]) for p in range(40))
    kind, frame, cmd, t, x, ee, le, ps = robots(B, 52, n_way, way)
    fk, _, fcmd, _, _, _, _ = frame_robots(B, 53)
    s.set_ee_frame(frame)
    rng = np.random.default_rng(54)
    dev = dict(le=_dev(le), ps=_dev(ps), nt=_dev(np.full(B, -7), torch.int32), tt=_dev(np.full((B, KMAX), np.nan)), ts=_dev(np.full((B, KMAX, TD), np.nan)))
    hst = dict(le=le.copy(), ps=ps.copy(), nt=np.full(B, -7, dtype=np.int32), tt=np.full((B, KMAX), np.nan), ts=np.full((B, KMAX, TD), np.nan))
    for tick in range(6):
        k = np.where(rng.uniform(size=B) < 0.6, np.where(rng.uniform(size=B) < 0.2, START, FOLLOW), fk).astype(np.int32)
        c = np.where((k >= 3)[:, None], cmd, fcmd); tk = t + 0.4 * tick
        s.target_trajectories_dev(_dev(k, torch.int32), _dev(c), _dev(tk), _dev(x), _dev(ee), dev["le"], dev["nt"], dev["tt"], dev["ts"], path_state=dev["ps"])
        torch.cuda.synchronize()
        h = host_target(host, k, frame, c, tk, x, ee, hst["le"], hst["ps"], n_way, way)
        hst["le"], hst["ps"] = h[3], h[4]; w = h[0] != -7
        hst["nt"][w], hst["tt"][w], hst["ts"][w] = h[0][w], h[1][w], h[2][w]
        d = dict(zip(dev, _host(*dev.values())))
        assert np.array_equal(d["nt"], hst["nt"]), tick
        for key in ("le", "ps", "tt", "ts"):
            np.testing.assert_allclose(d[key], hst[key], rtol=0, atol=1e-12, err_msg="%s tick %d" % (key, tick))
        assert np.count_nonzero(d["nt"] == 4) > 100 and np.count_nonzero((k == FOLLOW) & (h[0] == -7)) > 100
    # without path robots: byte-identical to qmb200_target_trajectories_per_robot_dev
    outs = []
    for path_state in (None, _dev(ps)):
        o = [_dev(le), _dev(np.full(B, -7), torch.int32), _dev(np.full((B, KMAX), np.nan)), _dev(np.full((B, KMAX, TD), np.nan))]
        kw = {} if path_state is None else dict(path_state=path_state)
        s.target_trajectories_dev(_dev(fk, torch.int32), _dev(fcmd), _dev(t), _dev(x), _dev(ee), *o, **kw)
        torch.cuda.synchronize(); outs.append(_host(*o))
    for a, b in zip(*outs):
        assert a.tobytes() == b.tobytes()
    with pytest.raises(_lib.QmbError, match="path 0, waypoint 1: its gap to waypoint 0 is under T/2"):
        s.set_ee_paths([(np.array([0.5, 0.9]), np.tile([0, 0, 0, 0, 0, 0, 1.0], (2, 1)))])
    assert len(s.get_ee_paths()) == 40   # the refused table wrote nothing
    s.set_ee_paths(None); assert s.get_ee_paths() is None
    s.close()


def test_the_gait_step_with_path_rows_equals_the_statement():
    """64 robots, a timeline of path, goal and ee_cmd_vel rows: the device step's target kinds and cmd rows equal the statement tick by tick; a path row
    is refused while no table holds its index."""
    B, n_cmd, n_ticks = 64, 6, 60; s = q.Solver(batch=B); rng = np.random.default_rng(61)
    s.gait_dev_set_templates(["stance"]); t_start = 10.0
    s.gait_dev_reset(np.zeros(B, dtype=np.int32), np.full(B, t_start))
    t = t_start + 0.01 * np.arange(n_ticks)
    t_cmd = np.sort(rng.uniform(t_start - 0.05, t_start + 0.7, (B, n_cmd)), axis=1)
    kind = rng.choice([-1, 1, 2, 3], (B, n_cmd)).astype(np.int32)
    ee = np.zeros((B, n_cmd, 7)); ee[..., :3] = rng.uniform(-1, 1, (B, n_cmd, 3)); ee[..., 3:] = [0, 0, 0, 1.0]; ee[kind == 3, 0] = rng.integers(0, 3, int((kind == 3).sum()))
    args = (t_cmd, np.full((B, n_cmd), -1, dtype=np.int32), np.full((B, n_cmd, 4), np.nan))
    with pytest.raises(_lib.QmbError, match=r"ee_kind\[\d+\]\[\d+\] is QMB200_TARGET_EE_PATH, but no path table is set"):
        s.gait_dev_set_commands(*args, ee_kind=kind, ee_cmd=ee)
    s.set_ee_paths([(np.array([0.5 * (p + 1)]), np.array([[0.6, 0.1, 0.4, 0, 0, 0, 1.0]])) for p in range(2)])
    with pytest.raises(_lib.QmbError, match=r"ee path\[\d+\]\[\d+\] is not an index of the path table \(2 paths"):
        s.gait_dev_set_commands(*args, ee_kind=kind, ee_cmd=ee)
    s.set_ee_paths([(np.array([0.5 * (p + 1)]), np.array([[0.6, 0.1, 0.4, 0, 0, 0, 1.0]])) for p in range(3)])
    s.gait_dev_set_commands(*args, ee_kind=kind, ee_cmd=ee)
    prob = dict(n_events=np.zeros(B, dtype=np.int32), event_times=np.zeros((B, _lib.EMAX)), modes=np.zeros((B, _lib.EMAX + 1), dtype=np.int32))
    cmd = np.zeros((B, 7)); tk = np.zeros(B, dtype=np.int32); got_k, got_c = [], []
    for k in range(n_ticks):
        _, _, st = s.gait_dev_step(np.full(B, t[k]), prob, cmd, target_kind=tk)
        assert np.all(st == 0)
        got_k.append(tk.copy()); got_c.append(cmd.copy())
    none = np.zeros((n_ticks, B), dtype=np.int32)
    rc, rk, _ = _gait_statement(t, t_cmd, kind, ee, none, none, np.zeros((n_ticks, B, 7)))
    assert np.array_equal(np.array(got_k), rk) and np.array_equal(np.array(got_c), rc)
    assert np.count_nonzero(rk == START) > 20 and np.count_nonzero(rk == FOLLOW) > 200
    s.close()


def test_the_device_command_checks_path_indices_against_the_table_in_force():
    """gait_command_kernel: with no table every path row is refused; with three paths only the integer indices 0-2 without a cmd_vel are taken; a
    table shrunk to one path refuses index 2 again"""
    B = 8; s = q.Solver(batch=B); s.gait_dev_set_templates(["stance"]); s.gait_dev_reset(np.zeros(B, dtype=np.int32), np.full(B, 10.0))
    ee = np.zeros((B, 7)); ee[:, 0] = [0, 2, 3, 1.5, -1.0, np.nan, 1, 0]; ee[:, 6] = 1.0
    vel = np.full((B, 4), np.nan); vel[7] = 0.0   # robot 7: a path row that also carries a cmd_vel
    args = (np.ones(B, dtype=np.int32), np.full(B, -1, dtype=np.int32), vel, np.full(B, START, dtype=np.int32), ee)
    assert np.all(s.gait_dev_command(*args) == _lib.ST_COMMAND) and not np.any(s.gait_dev_get_pending()["set"])
    one = (np.array([0.5]), np.array([[0.6, 0.1, 0.4, 0, 0, 0, 1.0]]))
    s.set_ee_paths([one] * 3)
    st = s.gait_dev_command(*args); p = s.gait_dev_get_pending()
    assert (st != 0).tolist() == [False, False, True, True, True, True, False, True] and np.all(st[st != 0] == _lib.ST_COMMAND)
    assert p["set"].tolist() == [1, 1, 0, 0, 0, 0, 1, 0] and p["ee"][[0, 1, 6], 0].tolist() == [0, 2, 1] and np.all(p["ee_kind"][[0, 1, 6]] == START)
    s.set_ee_paths([one])
    assert (s.gait_dev_command(*args) != 0).tolist() == [False, True, True, True, True, True, True, True]
    s.close()


def test_the_table_check_takes_the_handles_mpc_horizon():
    """a handle made with a 0.6 s horizon takes waypoints 0.4 s apart (T/2 = 0.3 s), which the task file's 1 s horizon would refuse, and refuses 0.25 s;
    closed_loop's check agrees on the same T"""
    s = q.Solver(batch=2, time_horizon=0.6); assert s.time_horizon == 0.6
    way = lambda gap: [(np.array([0.5, 0.5 + gap]), np.tile([0.6, 0.1, 0.4, 0, 0, 0, 1.0], (2, 1)))]
    s.set_ee_paths(way(0.4)); assert len(s.get_ee_paths()) == 1 and len(closed_loop._ee_paths_spec(s.time_horizon, way(0.4))) == 1
    with pytest.raises(_lib.QmbError, match="its gap to waypoint 0 is under T/2 = 0.300000 s"):
        s.set_ee_paths(way(0.25))
    with pytest.raises(ValueError, match="at least time_horizon / 2 = 0.3 s apart"):
        closed_loop._ee_paths_spec(s.time_horizon, way(0.25))
    s.close()


def test_a_path_loop_replays_call_by_call_on_the_host_build_and_the_oracle(host):
    """1 s of 16 standing robots, frames mixed (heading robots at yaws across +-3 rad), 14 of them starting a 5 cm square path at 0.1 s (waypoints
    0.5 s apart, so every target holds 3 or 4 knots), with every loop call recorded (tests/_loop_replay.py, its target call recording the path rows
    too): each target call restated by the host build from its recorded inputs gives the recorded outputs to 1e-12, and every MPC solve of a tick
    with 3-4 knot targets equals the oracle's at the suite's tolerance (replay_mpc, warm-started from the device's stored solution)."""
    from unittest import mock
    import _loop_replay as R
    from _oracle import Oracle
    B = 16; s = q.Solver(batch=B); frame = (np.arange(B) % 2).astype(np.int32)
    xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.where(frame == 1, np.linspace(-3, 3, B), 0.0)]
    hand = _standing_hand(s, xy, "world", 0.1)
    tau = np.array([0.125, 0.625, 1.125, 1.625]); off = np.array([[0.05, 0, 0], [0.05, 0.05, 0], [0, 0.05, 0], [0, 0, 0]])
    paths = [(tau, np.c_[hand[:3] + off + (np.r_[xy[b, :2], 0.0] if frame[b] == 0 else 0.0), np.tile(hand[3:7], (4, 1))]) for b in range(B)]
    n_way = np.full(B, 4, dtype=np.int32); way = np.zeros((B, _lib.EE_PATH_MAX, 8)); way[:, :4, 0] = tau; way[:, :4, 1:] = [p[1] for p in paths]
    ids = np.where(np.arange(B) < 14, np.arange(B), -1)[:, None]
    tg = R.WRAPPED["target_trajectories_dev"]   # the target call's path rows, and its in-out target rows as they were before the call
    wrapped = dict(R.WRAPPED, target_trajectories_dev=("targets", tg[1] + ("path_state", "n_target", "target_times", "target_states"), tg[2] + ("path_state",)))
    s.mpc_reset(); s.wbc_set_input_last(None)
    with mock.patch.object(R, "WRAPPED", wrapped):
        res, rec = R.record(s, lambda: closed_loop.run(s, duration=1.0, gait="stance", xy_yaw=xy, ee_frame=frame, ee_paths=paths,
                                                       commands=dict(t=np.full((B, 1), 0.1), gait=[[None]] * B, ee_path=ids)))
    assert np.all(res["status"] == 0) and np.all(res["base"][:, :, 2] > 0.3)
    calls = rec.of("targets"); worst = 0.0; kinds = set()
    for i, (inp, out) in enumerate(calls):
        kind = np.broadcast_to(np.asarray(inp["kind"], dtype=np.int32), (B,))
        nt, tt, ts, le, ps = host_target(host, kind, frame, inp["cmd"], inp["t_obs"], inp["x_obs"], inp["ee_state"], inp["last_ee_target"], inp["path_state"],
                                         n_way, way)
        kept = nt == -7   # a robot the call leaves untouched keeps its target
        nt[kept], tt[kept], ts[kept] = inp["n_target"][kept], inp["target_times"][kept], inp["target_states"][kept]
        assert np.array_equal(nt, out["n_target"]), i
        for a, b in ((tt, out["target_times"]), (ts, out["target_states"]), (le, out["last_ee_target"]), (ps, out["path_state"])):
            e = float(np.max(np.abs(a - b))); worst = max(worst, e)
            assert e <= 1e-12, (i, e)
        kinds |= set(kind.tolist())
    assert len(calls) == 100 and {0, START, FOLLOW} <= kinds
    sub = R.Record(); sub.calls = [c for c in rec.calls if c[0] == "mpc" and np.any(c[1]["prob"]["n_target"] >= 3)]
    nk = np.concatenate([c[1]["prob"]["n_target"] for c in sub.calls])
    assert len(sub.calls) >= 85 and np.count_nonzero(nk == 4) >= 500 and np.count_nonzero(nk == 3) >= 250
    m = R.replay_mpc(sub, [Oracle()] * B)
    print("path loop replay: %d target calls (worst %.1e), %d ticks with 3-4 knots, %d robot-solves replayed (%d with 4 knots, %d with 3; %d warm, %d "
          "without a step, %d near a line-search threshold): %s" % (len(calls), worst, m["ticks"], m["replayed"], np.count_nonzero(nk == 4),
                                                                   np.count_nonzero(nk == 3), m["warm"], m["no_step"], len(m["near"]),
                                                                   ", ".join("%s %.1e" % kv for kv in m["worst"].items())))
    s.close()


def _square(B, frame, xy, hand, gap=0.75):
    """per robot one path: the corners of a 10 cm square from the standing hand (hand [7]: its pose relative to the base at yaw 0), waypoints gap s
    apart, the hand's orientation held (world frame: about the robot's base)"""
    corners = hand[:3] + np.array([[0.1, 0, 0], [0.1, 0.1, 0], [0, 0.1, 0], [0, 0, 0]])
    tau = gap * np.arange(1, 5); qd = np.tile(hand[3:7], (4, 1))
    return [(tau, np.c_[corners + (np.r_[xy[b, :2], 0.0] if frame == "world" else 0.0), qd]) for b in range(B)]


def _standing_hand(s, xy, frame, t_first):
    """robot 0's hand pose relative to its base (yaw 0) after t_first s of the stance the square starts from: the path's start pose"""
    s.mpc_reset(); s.wbc_set_input_last(None)
    r = closed_loop.run(s, duration=t_first, gait="stance", xy_yaw=xy, ee_frame=frame)
    e, b = r["ee"][-1, 0], r["base"][-1, 0]
    return np.r_[e[0] - b[0], e[1] - b[1], e[2:7]]


def _path_at(paths, ps, t):
    """the hand position of p(t) [T, B, 3] in the world at the record times t [T] from the first waypoint on (a position lerp between waypoints), for
    paths started as the path state rows ps [B, PS] say, in the paths' own coordinates"""
    out = np.zeros((len(t), len(paths), 3))
    for b, (tau, pose) in enumerate(paths):
        for c in range(3):
            out[:, b, c] = np.interp(t, ps[b, 1] + tau, pose[:, c])
    return out


def _trace(s, B, frame, goals, t_first=0.5, duration=4.0):
    """B standing robots at 2 m spacing trace the square from t_first: as a path, or (goals) as successive goals at the waypoint times → (record,
    p(t) [T, B, 3] against the hand, the path start t0 [B])"""
    xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]; paths = _square(B, frame, xy, _standing_hand(s, xy, frame, t_first))
    if goals:   # goal i at the start of its segment: t_first, then each earlier waypoint's time
        cmds = dict(t=t_first + np.r_[0.0, paths[0][0][:3]][None, :].repeat(B, 0), gait=[[None] * 4] * B,
                    ee_goal=np.stack([p[1] for p in paths]))
        kw = dict(commands=cmds)
    else:
        kw = dict(commands=dict(t=np.full((B, 1), t_first), gait=[[None]] * B, ee_path=np.arange(B)[:, None]), ee_paths=paths)
    s.mpc_reset(); s.wbc_set_input_last(None)
    with closed_loop.Session(s, duration, gait="stance", xy_yaw=xy, ee_frame=frame, **kw) as ss:
        rec = ss.step(ss.windows); ss.stream.synchronize()
        rec = {k: (v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in rec.items()}
        ps = None if goals else ss.path_state.cpu().numpy()
        ss.finish()
    return rec, paths, ps


@pytest.mark.parametrize("frame", ["world", "heading"])
def test_standing_robots_trace_a_square_closer_as_a_path_than_as_goals(frame):
    B = 256; s = q.Solver(batch=B)
    res = {}; ps = None
    for goals in (False, True):   # both measured against the path run's schedule and start heading
        rec, paths, p = _trace(s, B, frame, goals)
        ps = p if p is not None else ps
        assert np.all(rec["status"] == 0), np.unique(rec["status"])
        assert np.all(rec["base"][:, :, 2] > 0.3)
        assert np.all(ps[:, 0] == np.arange(B))
        w = (rec["t"][:, None] >= ps[None, :, 1] + paths[0][0][0]) & (rec["t"][:, None] <= ps[None, :, 1] + paths[0][0][-1])
        ref = _path_at(paths, ps, rec["t"])
        if frame == "heading":
            ref = np.stack([h_to_world(ps[:, 2], ps[:, 3], ps[:, 4], np.c_[r, np.tile([0, 0, 0, 1.0], (B, 1))])[:, :3] for r in ref])
        err = np.linalg.norm(rec["ee"][..., :3] - ref, axis=-1)
        rms = float(np.sqrt(np.mean(err[w] ** 2)))
        res[goals] = (rms, err[w])
    print("square %s: hand RMS against p(t) %.4f m as a path, %.4f m as goals; p50 / p95 as a path %.4f / %.4f m"
          % (frame, res[False][0], res[True][0], *np.percentile(res[False][1], [50, 95])))
    assert res[False][0] < SQUARE_RMS_PATH_M and res[False][0] < SQUARE_RATIO * res[True][0]
    s.close()


def test_a_rewind_mid_path_replays_a_branch_continues_and_a_respawn_returns_to_cmd_vel():
    import torch
    B = 8; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    paths = _square(B, "heading", xy, np.r_[0.52, 0.09, 0.44, 0.5, -0.5, 0.5, -0.5])[:1]
    cmds = dict(t=np.full((B, 1), 0.3), gait=[[None]] * B, ee_path=np.zeros((B, 1), dtype=np.int64))
    with closed_loop.Session(s, 2.0, gait="stance", xy_yaw=xy, ee_frame="heading", ee_paths=paths, commands=cmds) as ss:
        host = lambda rec: (ss.stream.synchronize(), {k: v.cpu().numpy() for k, v in rec.items() if hasattr(v, "cpu")})[1]
        ss.step(100); snap = ss.snapshot()   # 0.7 s into the path
        a = host(ss.step(30))
        ss.restore(snap)
        b = host(ss.step(30))
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
        assert np.all(a["target_kind"] == FOLLOW)
        pi = [i for i, r in enumerate(ss.rows) if r is ss.path_state][0]
        ss.restore(snap, mask=torch.tensor([0, 1] + [0] * (B - 2), dtype=torch.int32, device="cuda"), source=torch.zeros(B, dtype=torch.int32, device="cuda"))
        ss.stream.synchronize()
        assert ss.path_state[1].cpu().numpy().tobytes() == snap.rows[pi][0].cpu().numpy().tobytes()   # the branch continues robot 0's path
        c = host(ss.step(10))
        assert np.all(c["target_kind"][:, 1] == FOLLOW)
        ss.finish()
    s.close()
    s = q.Solver(batch=B)   # a respawn returns the robot to its start: the cmd_vel stream, no path
    with closed_loop.Session(s, 1.0, gait="stance", steer=True, xy_yaw=xy, ee_frame="heading", ee_paths=paths, respawn=dict(every=0.5)) as ss:
        ss.step(4); ss.command(np.ones(B, dtype=np.int32), ee_path=np.zeros(B, dtype=np.int32))
        rec = {k: (v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in ss.step(ss.windows - 4).items()}
        ss.finish()
    k = rec["target_kind"]   # windows 4.. of the run: the path starts at window 4's tick, the restart at the 0.5 s boundary (window 50)
    assert np.all(k[0] == START) and np.all(k[1:46] == FOLLOW) and np.all(k[46:] == 0), k[:, 0]
    s.close()
