"""Per-episode command timelines inside the GPU closed loop (closed_loop.run(timeline=...), DESIGN.md §4.14): the device sampler is the host draw bit for
bit and writes nothing else; a drawn timeline runs as the same timeline given as commands; every respawned episode follows the gait protocol on its
own drawn rows; the draw composes with randomize, spawn and metrics."""
import numpy as np
import pytest

from qm_control_b200 import _lib
from qm_control_b200 import terrain as T
from _gait_protocol import NAMES, T as HORIZON, host_robot

pytestmark = pytest.mark.gpu

TL = {n: i for i, n in enumerate(_lib.TIMELINE_LAYOUT)}


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


def _ranges(rng, B, n_tmpl, ee=True):
    lo = np.zeros((B, _lib.TIMELINE)); lo[:, TL["t_first"]] = 10.0 + rng.uniform(0.0, 0.2, B); lo[:, TL["gap"]] = 0.05
    lo[:, TL["p_gait"]] = rng.choice([0.0, 0.5, 1.0], B); lo[:, TL["gait_set"]] = rng.integers(1, 1 << n_tmpl, B)
    lo[:, 4:8] = [1.0, 1.0, 1.0 if ee else 0.0, 1.0 if ee else 0.0]; lo[:, 8:18] = rng.uniform(-0.5, 0.5, (B, 10)); lo[:, TL["ee_qw"]] = 1.0
    hi = lo.copy(); hi[:, TL["t_first"]] += 0.3; hi[:, TL["gap"]] += 0.2; hi[:, 8:18] += rng.uniform(0.0, 0.3, (B, 10)); lo[::6, 8:18] = hi[::6, 8:18] = -0.0
    return lo, hi


def _stepped_timeline(s, rng, B, n, ee=True):
    """start every robot's schedule and load a timeline of n random commands whose first k[b] are due, then one host step: cursors at k"""
    s.gait_dev_set_templates(); ids = rng.integers(0, len(NAMES), B).astype(np.int32); s.gait_dev_reset(ids, np.full(B, 10.0))
    k = rng.integers(0, n + 1, B); t = np.where(np.arange(n)[None] < k[:, None], 9.0, np.inf)
    vel = np.where(rng.random((B, n, 1)) < 0.5, rng.uniform(-0.3, 0.3, (B, n, 4)), np.nan)
    kw = dict(ee_kind=np.full((B, n), -1, dtype=np.int32), ee_cmd=np.zeros((B, n, 7))) if ee else {}
    s.gait_dev_set_commands(t, rng.integers(-1, len(NAMES), (B, n)).astype(np.int32), vel, **kw)
    prob = dict(n_events=np.zeros(B, dtype=np.int32), event_times=np.zeros((B, _lib.EMAX)), modes=np.full((B, _lib.EMAX + 1), 15, dtype=np.int32))
    s.gait_dev_step(np.full(B, 10.0), prob, np.zeros((B, 7)))
    assert np.array_equal(s.gait_dev_get()["cursor"], k)
    return k


def _same(a, b):
    return all(a[key].tobytes() == b[key].tobytes() for key in a)


def test_sampler_is_the_host_draw_and_writes_nothing_else():
    import torch
    rng = np.random.default_rng(1); B, n = 4096, 5; s = _solver(B)
    try:
        k = _stepped_timeline(s, rng, B, n)
        lo, hi = _ranges(rng, B, len(NAMES)); seed = 2 ** 64 - 7
        mask = (rng.random(B) < 0.6).astype(np.int32); episode = rng.integers(-3, 1 << 30, B).astype(np.int32)
        sentinel = torch.full((B, n, _lib.TIMELINE_CMD), 7.25, dtype=torch.float64, device="cuda:0")
        before = s.gait_dev_get_commands()

        def refused(match):
            with pytest.raises(_lib.QmbError, match=match):
                s.timeline_sample_dev(torch.as_tensor(mask, device="cuda:0"), torch.as_tensor(episode, device="cuda:0"), sentinel)
            torch.cuda.synchronize()
            assert torch.all(sentinel == 7.25) and _same(s.gait_dev_get_commands(), before) and np.array_equal(s.gait_dev_get()["cursor"], k)
        refused("no ranges")
        s.timeline_set_ranges(n + 1, lo, hi, seed); refused("holds 5 commands per robot, the ranges draw 6")
        bad = lo.copy(); bad[17, TL["gait_set"]] = float(1 << len(NAMES)); s.timeline_set_ranges(n, bad, np.where(np.arange(22) == TL["gait_set"], bad, hi), seed)
        refused("at or above the template table's %d templates" % len(NAMES))
        with pytest.raises(_lib.QmbError, match="w_none of robot 0: must be fixed"):
            s.timeline_set_ranges(n, lo, np.where(np.arange(22) == TL["w_none"], lo + 1.0, hi), seed)
        assert s.timeline_get_ranges()["lo"].tobytes() == bad.tobytes()   # a rejection keeps the stored ranges
        s.timeline_set_ranges(n, lo, hi, seed)
        d_mask, d_ep = torch.as_tensor(mask, device="cuda:0"), torch.as_tensor(episode, device="cuda:0")
        s.timeline_sample_dev(d_mask, d_ep, sentinel); torch.cuda.synchronize()
        rows = sentinel.cpu().numpy(); m = mask.astype(bool); want = s.timeline_draw(np.arange(B)[m], episode[m])
        assert rows[m].tobytes() == want.tobytes() and np.all(rows[~m] == 7.25)
        got = s.gait_dev_get_commands()
        assert got["t"][m].tobytes() == want[..., 0].tobytes() and np.array_equal(got["tmpl"][m], want[..., 1].astype(np.int32))
        assert got["cmd_vel"][m].tobytes() == want[..., 2:6].tobytes() and np.array_equal(got["ee_kind"][m], want[..., 6].astype(np.int32))
        assert got["ee_cmd"][m].tobytes() == want[..., 7:].tobytes()
        for key in got:
            assert got[key][~m].tobytes() == before[key][~m].tobytes(), key
        assert np.array_equal(s.gait_dev_get()["cursor"], np.where(m, 0, k))
        kinds = want[..., 6]; assert np.any(kinds == 1) and np.any(kinds == 2) and np.any(np.isnan(want[..., 2])) and np.any(want[..., 1] >= 0)
        assert s.timeline_sample(mask, episode, rows=np.full((B, n, 14), 7.25)).tobytes() == rows.tobytes()   # the staged host variant
        # a timeline without end-effector rows refuses end-effector weights; the schedule must run
        s.gait_dev_set_commands(np.full((B, n), np.inf), np.full((B, n), -1, dtype=np.int32), np.full((B, n, 4), np.nan))
        before = s.gait_dev_get_commands(); k = np.zeros(B, dtype=int); sentinel.fill_(7.25)
        refused("no end-effector rows")
        s.gait_dev_stop()
        with pytest.raises(_lib.QmbError, match="not running"):
            s.timeline_sample_dev(d_mask, d_ep, sentinel)
        torch.cuda.synchronize(); assert torch.all(sentinel == 7.25)
        s.timeline_set_ranges(None); assert s.timeline_get_ranges() is None
    finally:
        s.close()


def _goal_spec(s, B):
    ee0 = s.initial_ee_target()[0]; q = ee0[3:7] / np.linalg.norm(ee0[3:7])
    return dict(seed=11, n=4, t_first=(0.05, 0.3), gap=(0.1, 0.3), p_gait=0.7, gaits=["trot", "standing_trot", "pace", "static_walk"],
                weights=dict(none=0.5, cmd_vel=1.0, ee_goal=1.0), cmd_vel_x=(-0.2, 0.3), cmd_yaw_rate=(-0.3, 0.3),
                ee_x=(ee0[0] - 0.05, ee0[0] + 0.05), ee_y=(ee0[1] - 0.05, ee0[1] + 0.05), ee_z=(ee0[2] - 0.05, ee0[2] + 0.05), ee_quat=q)


def test_a_drawn_timeline_runs_as_the_same_commands():
    from qm_control_b200 import closed_loop
    B = 64; s = _solver(B)
    try:
        s.mpc_reset(); s.wbc_set_input_last(None)   # both runs start cold
        a = closed_loop.run(s, duration=1.0, gait="trot", timeline=_goal_spec(s, B)); s.mpc_reset(); s.wbc_set_input_last(None)
        tp = a["timeline_params"][:, 0]; assert tp.shape == (B, 4, 14)
        kind = tp[..., 6]; assert np.any(kind == 2) and np.any(~np.isnan(tp[..., 2])) and np.any(tp[..., 1] >= 0)
        goal = np.where((kind == 2)[..., None], tp[..., 7:14], np.nan)
        commands = dict(t=tp[..., 0], gait=np.array([[None if g < 0 else NAMES[int(g)] for g in r] for r in tp[..., 1]], dtype=object), cmd_vel=tp[..., 2:6], ee_goal=goal)
        b = closed_loop.run(s, duration=1.0, gait="trot", commands=commands)
        assert set(a) - {"timeline_params"} == set(b)
        for key in b:
            if isinstance(b[key], np.ndarray):
                assert a[key].tobytes() == b[key].tobytes(), key
            else:
                assert a[key] == b[key], key
        assert s.timeline_get_ranges() is None
    finally:
        s.close()


def test_every_respawned_episode_follows_the_protocol_on_its_rows():
    """Episodes of 1.6 s, long enough for drawn gaits to take effect (a slot applied at t inserts its gait at t + the horizon, after the transition
    stance), with cmd_vel and ee_cmd_vel slots, so that the target kind switches between streams"""
    from qm_control_b200 import closed_loop
    B = 32; s = _solver(B); t_start = 10.0
    try:
        spec = dict(seed=3, n=6, t_first=(-0.05, 0.3), gap=(0.0, 0.3), p_gait=0.6, gaits=["trot", "pace", "static_walk", "standing_trot"],
                    weights=dict(none=1.0, cmd_vel=1.0, ee_cmd_vel=1.0), cmd_vel_x=(0.0, 0.3), ee_vx=(-0.03, 0.03), ee_vy=(-0.03, 0.03), ee_vz=(-0.02, 0.02))
        out = closed_loop.run(s, duration=3.2, gait="trot", t_start=t_start, respawn=dict(every=1.6), timeline=spec)
        ep, tp = out["episode"], out["timeline_params"]; E = int(ep.max()) + 1
        assert E >= 2 and tp.shape[:2] == (B, E)
        assert np.any(tp[:, 1:, :, :2] != tp[:, :1, :, :2])   # later episodes draw other rows
        gait0 = NAMES.index("trot"); drawn_modes = []
        for b in range(B):
            for e in range(E):
                ticks = np.nonzero(ep[:, b] == e)[0]
                rows = tp[b, e]; t_cmd = t_start + rows[:, 0]; g = host_robot("trot", t_start)
                active, cur, src, t, first_insert = gait0, 0, _lib.TARGET_CMD_VEL, t_start - 0.002, np.inf
                for i in ticks:
                    applied = -1
                    while cur < len(rows) and t_cmd[cur] <= t:
                        if rows[cur, 1] >= 0:
                            g.insertModeSequenceTemplate(NAMES[int(rows[cur, 1])], t + HORIZON, HORIZON); active = int(rows[cur, 1])
                            first_insert = min(first_insert, t + HORIZON)
                        if not np.isnan(rows[cur, 2]):
                            applied = _lib.TARGET_CMD_VEL
                        if rows[cur, 6] == _lib.TARGET_EE_CMD_VEL:
                            applied = _lib.TARGET_EE_CMD_VEL
                        cur += 1
                    ev, md, n = g.getModeSchedule(t - HORIZON, t + 2 * HORIZON)
                    src = applied if applied >= 0 else src
                    mode = md[int(np.searchsorted(ev[:n], t, side="left"))]
                    assert out["gait"][i, b] == active and out["mode"][i, b] == mode, (b, e, i)
                    assert out["target_kind"][i, b] == src, (b, e, i)
                    if t > first_insert:
                        drawn_modes.append(mode)
                    for _ in range(5):
                        t = t + 0.002
        # drawn gaits drove the schedule: windows after an insertion took effect, with modes a trot never has (pace, static_walk)
        assert len(drawn_modes) > 1000 and set(drawn_modes) - {6, 9, 15}
        assert np.any(out["target_kind"] == _lib.TARGET_EE_CMD_VEL) and np.any(out["target_kind"] == _lib.TARGET_CMD_VEL)
    finally:
        s.close()


def test_timeline_composes_with_randomize_spawn_and_metrics():
    from qm_control_b200 import closed_loop
    B = 24; s = _solver(B); xy = np.zeros((B, 3))
    try:
        kw = dict(duration=0.6, gait="trot", xy_yaw=xy, respawn=dict(every=0.2), randomize=dict(seed=4, cmd_vel_x=(0.0, 0.3), friction_mu=(0.5, 0.9)),
                  terrain=dict(tiles=np.stack([T.ramp(8.0), T.stairs(0.05, 0.25), T.rough(0.02, seed=4, flat_radius=0.2)]), cell=T.CELL,
                               tile=np.arange(B) % 4 - 1, origin=T.centred_origin(xy[:, :2])),
                  spawn=dict(seed=5, tile=(-1, 2), dx=(-0.1, 0.1), yaw=(0.2, 0.2)),
                  timeline=dict(seed=6, n=3, t_first=(0.0, 0.1), gap=(0.02, 0.06), p_gait=0.5, gaits=["trot", "pace"], weights=dict(none=1.0, cmd_vel=1.0),
                                cmd_vel_y=(-0.1, 0.1)))
        a = closed_loop.run(s, **kw)
        b = closed_loop.run(s, metrics=True, **kw)
        ep = a["episode"]; had = np.zeros((B, int(ep.max()) + 1), dtype=bool); had[np.broadcast_to(np.arange(B), ep.shape), ep] = True
        for key in ("episode_params", "spawn_params", "timeline_params"):
            covered = ~np.isnan(a[key].reshape(B, had.shape[1], -1)).all(-1)
            assert np.array_equal(covered, had), key
        assert set(b) - set(a) == {"episode_metrics", "metrics_layout"}
        for key in a:
            if isinstance(a[key], np.ndarray):
                assert a[key].tobytes() == b[key].tobytes(), key
    finally:
        s.close()
