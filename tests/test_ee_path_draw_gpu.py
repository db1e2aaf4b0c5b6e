"""Per-episode end-effector paths on the GPU (DESIGN.md §4.21): the sampler against the host rebuild (table rows, record rows and pending slots) with
its refusals, a drawn-path run byte-identical to the same paths given as a table and path commands, a respawning run whose every path starts on its
episode's first tick and whose target calls the host build restates, flat and moving curricula, and a rewind and a branch mid-path."""
import numpy as np
import pytest

import qm_control_b200 as q
from qm_control_b200 import _lib, closed_loop
from qm_control_b200.interface import gait_template_names
from test_ee_path_cpu import FOLLOW, START, host, host_target  # noqa: F401  (host: the host build's fixture)

pytestmark = pytest.mark.gpu
PMAX, W = _lib.EE_PATH_MAX, _lib.EE_PATH_RANGES
PR = {n: i for i, n in enumerate(_lib.EE_PATH_RANGES_LAYOUT)}
NAN = np.array([0x7FF8000000000000], dtype=np.uint64).view(np.float64)[0]


def _dev(a, dtype=None):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype or torch.float64, device="cuda")


def _ranges(rng, B, T):
    lo = np.zeros((B, W)); hi = np.zeros_like(lo)
    n = rng.integers(1, PMAX + 1, B); lo[:, PR["n_way"]] = hi[:, PR["n_way"]] = n
    lo[:, PR["tau_first"]] = 0.1; hi[:, PR["tau_first"]] = rng.choice([0.1, 0.6], B)
    lo[:, PR["gap"]] = 0.5 * T; hi[:, PR["gap"]] = 0.5 * T + rng.choice([0.0, 0.4], B)
    for c in ("x", "y", "z"):
        lo[:, PR[c]] = rng.uniform(-0.2, 0.2, B); hi[:, PR[c]] = lo[:, PR[c]] + rng.choice([0.0, 0.1], B)
    lo[:, PR["yaw"]] = -np.pi; hi[:, PR["yaw"]] = rng.choice([-np.pi, 0.0, np.pi], B)
    q_ = rng.normal(size=(B, 4)); q_ /= np.linalg.norm(q_, axis=1, keepdims=True); lo[:, 7:] = hi[:, 7:] = q_
    return lo, hi


def test_the_sampler_equals_the_host_rebuild_and_refusals_write_nothing(host):
    """4096 robots, random masks and episodes, 5 user paths in front: the record rows equal ee_path_draw byte for byte up to n_way, and so
    does every waypoint of the table rows, read through follow target calls (world robots: the knots are the waypoints' own bytes); the pending slots
    are the bytes qmb200_gait_dev_command writes for the same start rows, unmasked robots keep every byte, and each refusal writes nothing"""
    import torch
    B = 4096; s = q.Solver(batch=B); T = s.time_horizon; rng = np.random.default_rng(5); P = 5
    user = [(np.array([0.3, 0.3 + T]), np.tile([0.5, 0.1, 0.4, 0, 0, 0, 1.0], (2, 1))) for _ in range(P)]
    s.set_ee_paths(user)
    lo, hi = _ranges(rng, B, T)
    rows = _dev(np.full((B, PMAX, 8), 7.0)); mask = _dev(np.zeros(B), torch.int32); ep = _dev(np.zeros(B), torch.int32)
    with pytest.raises(q.QmbError, match="no ranges are set"):
        s.ee_path_sample_dev(mask, ep, rows)
    s.ee_path_set_ranges(lo, hi, seed=2 ** 64 - 5)
    with pytest.raises(q.QmbError, match="ee path ranges are set"):
        s.set_ee_paths(user[:2])
    assert len(s.get_ee_paths()) == P
    with pytest.raises(q.QmbError, match="device gait schedule is not running"):
        s.ee_path_sample_dev(mask, ep, rows)
    torch.cuda.synchronize(); assert np.all(rows.cpu().numpy() == 7.0)
    names = gait_template_names(); s.gait_dev_set_templates(names); s.gait_dev_reset(np.zeros(B, dtype=np.int32), np.zeros(B))
    m = (rng.uniform(size=B) < 0.6).astype(np.int32); e = rng.integers(0, 1 << 31, B).astype(np.int32)
    s.ee_path_sample_dev(_dev(m, torch.int32), _dev(e, torch.int32), rows); torch.cuda.synchronize()
    got = rows.cpu().numpy(); b = np.nonzero(m)[0]
    n_way, way = s.ee_path_draw(b, e[b])
    assert np.array_equal(n_way, lo[b, 0].astype(np.int32)) and np.all(got[m == 0] == 7.0)
    past = np.arange(PMAX)[None, :] >= n_way[:, None]   # the waypoints past n_way are not written
    assert got[b][~past].tobytes() == way[~past].tobytes() and np.all(got[b][past] == 7.0)
    pend = s.gait_dev_get_pending()
    assert np.all(pend["set"][m == 0] == 0) and np.all(pend["set"][b] == 1)
    # the table rows, every waypoint: following row P + b from t0 = 0 at t = tau_{j-1} (0 for j = 0), a world robot's knots 1..3 are waypoints j..j+2
    # of the row, tau and pose bytes unchanged, and n_target = 1 + min(n_way - j, 3) gives the row's n_way
    x = np.zeros((B, _lib.NX)); ee = np.tile([0.5, 0.1, 0.4, 0, 0, 0, 1.0], (B, 1)); cmd = np.zeros((B, 7))
    ps0 = np.zeros((B, _lib.EE_PATH_STATE)); ps0[:, 0] = P + np.arange(B); ps0[:, 5:] = ee
    seen = np.zeros((len(b), PMAX), dtype=bool)
    for j in range(0, PMAX, 3):
        on = n_way > j
        kind = np.full(B, -1, dtype=np.int32); kind[b[on]] = FOLLOW
        t = np.zeros(B); t[b[on]] = way[on, j - 1, 0] if j else 0.0
        nt, tt, ts, _, _ = s.target_trajectories_path(kind, cmd, t, x, ee, ee.copy(), ps0)
        k = np.minimum(n_way - j, 3)
        assert np.array_equal(nt[b[on]], 1 + k[on]), j
        for i in range(min(3, PMAX - j)):
            w = on & (k > i)
            assert tt[b[w], 1 + i].tobytes() == way[w, j + i, 0].tobytes() and ts[b[w], 1 + i, 30:37].tobytes() == way[w, j + i, 1:8].tobytes(), (j, i)
            seen[w, j + i] = True
    assert np.array_equal(seen, ~past)
    # a stopped schedule has no pending slots: refused, nothing written
    s.gait_dev_stop()
    with pytest.raises(q.QmbError, match="device gait schedule is not running"):
        s.ee_path_sample_dev(_dev(m, torch.int32), _dev(e + 1, torch.int32), rows)
    torch.cuda.synchronize(); assert rows.cpu().numpy().tobytes() == got.tobytes()
    # the pending slots are what the command writes for (tmpl -1, quiet NaN cmd_vel, path start of row P + b): with the same rows as a table
    s.ee_path_set_ranges(None)
    s.set_ee_paths(user + [(np.array([0.5]), np.array([[0, 0, 0, 0, 0, 0, 1.0]]))] * B)
    s.gait_dev_reset(np.zeros(B, dtype=np.int32), np.zeros(B))
    ee_cmd = np.zeros((B, 7)); ee_cmd[:, 0] = P + np.arange(B)
    st = s.gait_dev_command(m, np.full(B, -1), np.full((B, 4), NAN), np.full(B, _lib.TARGET_EE_PATH), ee_cmd)
    assert np.all(st == 0)
    want = s.gait_dev_get_pending()
    for key in pend:
        assert pend[key].tobytes() == want[key].tobytes(), key
    s.close()


def _hand(s, B):
    """the standing hand's pose relative to its base at yaw 0"""
    s.mpc_reset(); s.wbc_set_input_last(None)
    r = closed_loop.run(s, duration=0.1, gait="stance", xy_yaw=np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)], ee_frame="heading")
    return np.r_[r["ee"][-1, 0, :3] - np.r_[r["base"][-1, 0, :2], 0.0], r["ee"][-1, 0, 3:7]]


def _draw_spec(hand, n=4, seed=11, box=0.05):
    return dict(seed=seed, n=n, tau_first=(0.2, 0.3), gap=(0.5, 0.7), x=(hand[0] - box, hand[0] + box), y=(hand[1] - box, hand[1] + box),
                z=(hand[2] - box, hand[2] + box), yaw=(-0.3, 0.3), quat=hand[3:7])


def _np(rec):
    return {k: (v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in rec.items()}


def test_a_drawn_path_run_is_byte_identical_to_the_same_paths_given():
    """64 standing heading robots at mixed yaws, 1 s: the run with ee_path_draw equals the run given its ee_path_params as the table and a path
    command due by the first tick (the blocking first solve, one WBC period before the start), in every recorded output"""
    B = 64; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.linspace(-3.0, 3.0, B)]
    spec = _draw_spec(_hand(s, B))
    out = {}
    for given in (False, True):
        s.mpc_reset(); s.wbc_set_input_last(None)
        kw = dict(ee_path_draw=spec) if not given else dict(ee_paths=[(w[:, 0], w[:, 1:]) for w in out[False]["ee_path_params"][:, 0]],
                                                           commands=dict(t=np.full((B, 1), -1.0), gait=[[None]] * B, ee_path=np.arange(B)[:, None]))
        with closed_loop.Session(s, 1.0, gait="stance", xy_yaw=xy, ee_frame="heading", **kw) as ss:
            rec = ss.step(ss.windows); ss.stream.synchronize(); rec = _np(rec); ps = ss.path_state.cpu().numpy(); end = ss.finish()
        out[given] = dict(rec, ps=ps, **end)
    a, b = out[False], out[True]
    assert np.all(a["status"] == 0) and np.all(a["target_kind"][0] == START) and np.all(a["target_kind"][1:] == FOLLOW)
    for k in a:
        if k in ("ee_path_params", "ps", "gait_templates", "metrics_layout"):
            continue
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k
    assert np.array_equal(a["ps"][:, 0], np.arange(B)) and a["ps"][:, 1:].tobytes() == b["ps"][:, 1:].tobytes()
    s.close()


def test_a_respawning_run_starts_every_path_on_its_episodes_first_tick_and_replays_on_the_host_build(host):
    """32 robots, 0.5 s episodes with a timeline on: each episode's path starts on its first tick (t0 the episode's start, index P + b), and every
    target call restated by the host build from its recorded inputs, on the table rows of each robot's episode, gives the recorded outputs to 1e-12"""
    from unittest import mock
    import _loop_replay as R
    B = 32; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    spec = _draw_spec(_hand(s, B), n=3)
    tl = dict(seed=4, n=2, t_first=(0.05, 0.2), gap=(0.1, 0.2), weights=dict(none=1.0, cmd_vel=1.0), cmd_vel_x=(0.0, 0.1))
    user = [(np.array([0.4]), np.array([[0.5, 0.1, 0.4, 0.5, -0.5, 0.5, -0.5]]))] * 3; P = len(user)
    tg = R.WRAPPED["target_trajectories_dev"]
    wrapped = dict(R.WRAPPED, target_trajectories_dev=("targets", tg[1] + ("path_state", "n_target", "target_times", "target_states"), tg[2] + ("path_state",)))
    s.mpc_reset(); s.wbc_set_input_last(None)
    with mock.patch.object(R, "WRAPPED", wrapped):
        res, rec = R.record(s, lambda: closed_loop.run(s, duration=1.5, gait="stance", xy_yaw=xy, ee_frame="heading", ee_paths=user, ee_path_draw=spec,
                                                       timeline=tl, respawn=dict(every=0.5)))
    calls = rec.of("targets"); frame = np.ones(B, dtype=np.int32); prm = res["ee_path_params"]   # the run's ranges are gone: its rebuilt draws
    episode = np.full(B, -1); starts = 0; worst = 0.0
    for i, (inp, out) in enumerate(calls):
        kind = np.asarray(inp["kind"], dtype=np.int32); st = kind == START
        episode += st; starts += int(st.sum())
        assert np.all(episode >= 0), i   # the first tick starts every robot's first path
        tn, tw = np.r_[[len(t) for t, _ in user], np.full(B, 3)].astype(np.int32), np.zeros((P + B, PMAX, 8))
        for p, (t, pose) in enumerate(user):
            tw[p, :len(t), 0] = t; tw[p, :len(t), 1:] = pose
        tw[P:, :3] = prm[np.arange(B), episode]
        nt, tt, ts, le, ps = host_target(host, kind, frame, inp["cmd"], inp["t_obs"], inp["x_obs"], inp["ee_state"], inp["last_ee_target"], inp["path_state"], tn, tw)
        kept = nt == -7
        nt[kept], tt[kept], ts[kept] = inp["n_target"][kept], inp["target_times"][kept], inp["target_states"][kept]
        assert np.array_equal(nt, out["n_target"]), i
        for a, b in ((tt, out["target_times"]), (ts, out["target_states"]), (le, out["last_ee_target"]), (ps, out["path_state"])):
            e = float(np.max(np.abs(a - b))); worst = max(worst, e)
            assert e <= 1e-12, (i, e)
        if np.any(st):
            assert np.array_equal(out["path_state"][st, 0], P + np.nonzero(st)[0]) and np.all(out["path_state"][st, 1] == inp["t_obs"][st])
            assert np.all(inp["t_obs"][st] == calls[0][0]["t_obs"][0])   # the episode's first tick, on its own clock
    assert starts >= 3 * B and np.all(episode == res["episode"][-1])
    assert prm.shape[:2] == (B, int(res["episode"].max()) + 1) and prm.shape[2:] == (3, 8)
    print("respawning path replay: %d target calls, %d path starts, worst %.1e" % (len(calls), starts, worst))
    s.close()


def _curriculum_run(s, B, xy, spec, cur, seen=None):
    """a 1 s run of standing heading robots with 0.2 s episodes; seen (a list): every device draw as (mask, episode, rows) read right after the call"""
    import torch
    s.mpc_reset(); s.wbc_set_input_last(None)
    if seen is not None:
        f = s.ee_path_sample_dev

        def call(mask, episode, rows, stream=None):
            f(mask, episode, rows, stream); torch.cuda.synchronize()
            seen.append((mask.cpu().numpy().copy(), episode.cpu().numpy().copy(), rows.cpu().numpy().copy()))
        s.ee_path_sample_dev = call
    try:
        return closed_loop.run(s, duration=1.0, gait="stance", xy_yaw=xy, ee_frame="heading", ee_path_draw=spec, respawn=dict(every=0.2), curriculum=cur)
    finally:
        if seen is not None:
            del s.ee_path_sample_dev


def test_a_flat_curriculum_changes_nothing_and_a_moving_one_draws_at_each_episodes_level():
    """A flat curriculum (top = base) leaves every output byte-identical.  With a moving one, the levels the device update writes into the ranges are
    the ones the device sampler draws from: every row the sampler drew (recorded right after each call) equals ee_path_params, the host's rebuild at
    the episode's level, byte for byte, and rows drawn above level 0 differ from the level-0 rebuild."""
    B = 16; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    spec = _draw_spec(_hand(s, B), n=2)
    a = _curriculum_run(s, B, xy, spec, None)
    flat = {k: spec[k] for k in ("x", "y", "z", "tau_first", "gap", "yaw")}
    b = _curriculum_run(s, B, xy, spec, dict(levels=4, start=1, ee_path_draw=flat))
    for k in a:
        if k in ("gait_templates", "metrics_layout"):
            continue
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k
    top = dict(x=(spec["x"][0] - 0.05, spec["x"][1] + 0.05), gap=(0.6, 0.9))
    seen = []
    c = _curriculum_run(s, B, xy, spec, dict(levels=3, start=np.arange(B) % 3, up_after=1, ee_path_draw=top), seen)
    el, prm = c["episode_level"], c["ee_path_params"]; had = el >= 0
    assert np.all(np.isnan(prm[~had])) and not np.any(np.isnan(prm[had]))
    drawn = np.zeros(el.shape, dtype=bool); above = 0
    for mask, idx, rows in seen:
        for r in np.nonzero(mask)[0]:
            e = idx[r]; assert not drawn[r, e]; drawn[r, e] = True
            assert rows[r, :2].tobytes() == prm[r, e].tobytes(), (r, e, el[r, e])
            above += int(el[r, e] > 0)
    assert np.array_equal(drawn, had) and above >= B and len(np.unique(el[had])) == 3
    # above level 0 the device ranges moved: the same (robot, episode) drawn from the base box differs
    s.ee_path_set_ranges(*closed_loop._ee_path_box(closed_loop._ee_path_draw_spec(B, s.time_horizon, spec), B), spec["seed"])
    up = np.argwhere(had & (el > 0)); _, base = s.ee_path_draw(up[:, 0], up[:, 1])
    assert np.all(np.any(base[:, :2, :2] != prm[up[:, 0], up[:, 1], :, :2], axis=(1, 2)))
    s.ee_path_set_ranges(None)
    s.close()


def test_a_rewind_mid_path_replays_and_a_branch_follows_its_sources_path():
    import torch
    B = 8; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    spec = _draw_spec(_hand(s, B))
    s.mpc_reset(); s.wbc_set_input_last(None)
    with closed_loop.Session(s, 2.0, gait="stance", xy_yaw=xy, ee_frame="heading", ee_path_draw=spec) as ss:
        host_rec = lambda rec: (ss.stream.synchronize(), {k: v.cpu().numpy() for k, v in rec.items() if hasattr(v, "cpu")})[1]
        ss.step(60); snap = ss.snapshot()   # 0.6 s into the path
        a = host_rec(ss.step(40))
        ss.restore(snap)
        b = host_rec(ss.step(40))
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
        assert np.all(a["target_kind"] == FOLLOW)
        pi = [i for i, r in enumerate(ss.rows) if r is ss.path_state][0]
        ss.restore(snap, mask=torch.tensor([0, 1] + [0] * (B - 2), dtype=torch.int32, device="cuda"), source=torch.zeros(B, dtype=torch.int32, device="cuda"))
        ss.stream.synchronize()
        assert ss.path_state[1].cpu().numpy().tobytes() == snap.rows[pi][0].cpu().numpy().tobytes() and ss.path_state[1, 0].item() == 0.0
        c = host_rec(ss.step(10))
        assert np.all(c["target_kind"][:, 1] == FOLLOW) and np.all(c["status"] == 0)
        ss.finish()
    s.close()
