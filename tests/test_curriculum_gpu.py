"""Per-robot curricula inside the GPU closed loop (closed_loop.run(curriculum=...), DESIGN.md §4.15): the device update is the host core byte for byte
and writes nothing else; a flat curriculum changes no output of a run; the samplers draw the rows the run rebuilds at each episode's level; the levels
follow the rule; a restore leaves the state; the run leaves the ranges, robot terrain rows and curriculum as it found them."""
import numpy as np
import pytest

import _curriculum_twin as tw
from qm_control_b200 import _lib
from qm_control_b200 import terrain as T

pytestmark = pytest.mark.gpu

TL = {n: i for i, n in enumerate(_lib.TIMELINE_LAYOUT)}
WIDTH = dict(episode=_lib.EPISODE, spawn=_lib.SPAWN, timeline=_lib.TIMELINE)


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


def _boxes(rng, B):
    """valid base and top boxes of every kind whose every level passes the kind's check: both ends positive friction, no tiles, fixed timeline columns"""
    out = {}
    lo = np.zeros((B, _lib.EPISODE)); lo[:, 0] = rng.uniform(0.3, 0.6, B); lo[:, 11:14] = rng.uniform(-50, 0, (B, 3)); lo[::9, 13] = -0.0
    hi = lo.copy(); hi[:, 0] += 0.3; hi[:, 11:14] += rng.uniform(0, 50, (B, 3)); tlo = lo.copy(); thi = hi.copy(); thi[:, 11:14] += rng.uniform(0, 200, (B, 3))
    tlo[:, 0] = rng.uniform(0.1, 0.3, B); thi[::5] = hi[::5]; tlo[::5] = lo[::5]
    out["episode"] = (lo, hi, tlo, thi)
    lo = np.zeros((B, _lib.SPAWN)); lo[:, 0] = -1.0; lo[:, 1:3] = rng.uniform(-0.2, 0.0, (B, 2)); lo[:, 3] = -0.1; hi = lo.copy(); hi[:, 1:4] += 0.2
    tlo = lo.copy(); thi = hi.copy(); thi[:, 3] = 2.5; tlo[:, 3] = -2.5; thi[:, 1] += rng.uniform(0, 1, B)
    out["spawn"] = (lo, hi, tlo, thi)
    lo = np.zeros((B, _lib.TIMELINE)); lo[:, TL["t_first"]] = 10.0; lo[:, TL["gap"]] = 0.1; lo[:, TL["gait_set"]] = 3.0; lo[:, TL["w_none"]] = 1.0; lo[:, TL["ee_qw"]] = 1.0
    hi = lo.copy(); hi[:, TL["t_first"]] += 0.2; hi[:, TL["cmd_vel_x"]] = 0.2
    tlo = lo.copy(); thi = hi.copy(); tlo[:, TL["p_gait"]] = thi[:, TL["p_gait"]] = 1.0; tlo[:, TL["w_cmd_vel"]] = thi[:, TL["w_cmd_vel"]] = 2.0; thi[:, TL["cmd_vel_x"]] = 0.8
    out["timeline"] = (lo, hi, tlo, thi)
    return out


def _ranges(s):
    r = {k: getattr(s, k + "_get_ranges")() for k in WIDTH}
    return {k: (v["lo"].tobytes(), v["hi"].tobytes()) for k, v in r.items() if v is not None}


@pytest.mark.parametrize("kinds", [("episode",), ("spawn",), ("timeline",), ("episode", "spawn", "timeline")])
def test_update_is_the_host_core_and_writes_nothing_else(kinds):
    import torch
    rng = np.random.default_rng(len(kinds) * 10 + len(kinds[0])); B, E, L = 4096, 5, 9; s = _solver(B); dev = "cuda:0"
    try:
        boxes = _boxes(rng, B)
        for k in kinds:
            lo, hi, _, _ = boxes[k]
            s.timeline_set_ranges(3, lo, hi, 5) if k == "timeline" else getattr(s, k + "_set_ranges")(lo, hi, 5)
        conditions = [("distance", ">=", "pass"), ("max_tilt", "<=", "pass"), ("slip", ">=", "fail")]
        rows = np.zeros((B, _lib.CURRICULUM)); rows[:, 0] = rng.integers(0, L, B); rows[:, 1] = rng.integers(1, 4, B); rows[:, 2] = rng.integers(1, 4, B)
        rows[:, 3:6] = rng.choice([0.0, 0.5, 1.0], (B, 3))
        level = np.zeros(B, dtype=np.int32); status = np.zeros(B, dtype=np.int32)

        def refused(match, *args):
            before = (s.curriculum_get(), _ranges(s))
            with pytest.raises(_lib.QmbError, match=match):
                s._call(*args)
            torch.cuda.synchronize(); after = (s.curriculum_get(), _ranges(s))
            assert (before[0] is None and after[0] is None or before[0].tobytes() == after[0].tobytes()) and before[1] == after[1]
        d = {k: torch.as_tensor(np.ones(B, dtype=np.int32), device=dev) for k in ("mask", "end", "episode", "level", "status")}
        m_dev = torch.zeros((B, E, _lib.METRICS), dtype=torch.float64, device=dev)
        p = lambda t: None if t is None else __import__("ctypes").c_void_p(t.data_ptr())
        args = lambda rows_, n: ("curriculum_update_dev", p(d["mask"]), p(d["end"]), p(d["episode"]), p(rows_), n, p(d["level"]), p(d["status"]), None)
        refused("no curriculum is set", *args(m_dev, E))
        s.curriculum_set(L, rows, conditions)
        refused("no kind is attached", *args(m_dev, E))
        for k in kinds:
            s.curriculum_attach(k, *boxes[k][2:])
        refused("the rule has conditions, and rows is NULL", *args(None, E))
        refused("n_episodes must be >= 1", *args(m_dev, 0))
        with pytest.raises(_lib.QmbError, match="ranges are attached already"):
            s.curriculum_attach(kinds[0], *boxes[kinds[0]][2:])
        with pytest.raises(_lib.QmbError, match="a curriculum is attached to these ranges"):
            s.timeline_set_ranges(3, *boxes["timeline"][:2]) if kinds[0] == "timeline" else getattr(s, kinds[0] + "_set_ranges")(*boxes[kinds[0]][:2])
        for rnd in range(4):   # random states from earlier rounds, then one round checked against the host core
            mask = (rng.random(B) < 0.6).astype(np.int32); end = rng.choice([0, 1, 2, 2, 3], B).astype(np.int32)
            episode = rng.integers(-1, E + 1, B).astype(np.int32)
            metrics = rng.choice([0.0, 0.5, 1.0, np.nan, 2.0], (B, E, _lib.METRICS))
            st0, r0 = s.curriculum_get(), {k: getattr(s, k + "_get_ranges")() for k in kinds}
            for name, a in (("mask", mask), ("end", end), ("episode", episode)):
                d[name].copy_(torch.as_tensor(a))
            lv0 = rng.integers(-5, 0, B).astype(np.int32); st_in = rng.integers(0, 4, B).astype(np.int32)
            d["level"].copy_(torch.as_tensor(lv0)); d["status"].copy_(torch.as_tensor(st_in)); m_dev.copy_(torch.as_tensor(metrics))
            s.curriculum_update_dev(d["mask"], d["end"], d["episode"], m_dev, d["level"], d["status"]); torch.cuda.synchronize()
            st1 = s.curriculum_get(); lv1 = d["level"].cpu().numpy(); sts1 = d["status"].cpu().numpy()
            for b in range(B):
                upd = mask[b] and end[b] in (1, 2); ovf = upd and not 0 <= episode[b] < E
                want = tw.step(st0[b], rows[b], end[b], metrics[b, episode[b]] if upd and not ovf else None, L,
                               [(_lib.METRICS_LAYOUT.index(c), o, r) for c, o, r in conditions]) if upd and not ovf else st0[b].tolist()
                assert st1[b].tolist() == want, (rnd, b)
                assert lv1[b] == (want[0] if upd and not ovf else lv0[b]) and sts1[b] == st_in[b] | (2 if ovf else 0), (rnd, b)
            moved = mask.astype(bool) & np.isin(end, (1, 2)) & (episode >= 0) & (episode < E)
            for k in kinds:
                r1 = getattr(s, k + "_get_ranges")(); base_lo, base_hi, top_lo, top_hi = boxes[k]; rc = 0 if k == "spawn" else -1
                want_lo = np.where(moved[:, None], tw.box(base_lo, top_lo, st1[:, 0], L, rc), r0[k]["lo"])
                want_hi = np.where(moved[:, None], tw.box(base_hi, top_hi, st1[:, 0], L, rc), r0[k]["hi"])
                assert r1["lo"].tobytes() == want_lo.tobytes() and r1["hi"].tobytes() == want_hi.tobytes(), (rnd, k)
                assert r1["lo"][~moved].tobytes() == r0[k]["lo"][~moved].tobytes()
        assert len(set(st1[:, 0])) > 3 and st1[:, 3].max() >= 3
        end = np.where(end == 3, 0, end).astype(np.int32)   # the host variant refuses a masked end outside {0, 1, 2} as a whole
        host = s.curriculum_update(mask, end, episode, lv0, st_in, rows=metrics)   # the staged host variant: the next round, as the device runs it
        st2 = s.curriculum_get(); lv = np.where(mask.astype(bool) & np.isin(end, (1, 2)) & (episode >= 0) & (episode < E), st2[:, 0], lv0)
        assert np.array_equal(host["level"], lv)
        # a restore of the start image leaves the state and the ranges
        s.robot_image_save(); before = (s.curriculum_get().tobytes(), _ranges(s))
        s.robot_image_restore(np.ones(B, dtype=np.int32))
        assert (s.curriculum_get().tobytes(), _ranges(s)) == before
        s.robot_image_clear()
        # the draw at a level is the kind's draw on the box of that level; a clear puts the base boxes back
        k = kinds[-1]; rb = rng.integers(0, B, 64); re_ = rng.integers(0, 50, 64); rl = rng.integers(0, L, 64)
        got = s.curriculum_draw(k, rb, re_, rl)
        s.curriculum_set(None); assert s.curriculum_get() is None
        for kk in kinds:
            lo, hi = getattr(s, kk + "_get_ranges")()["lo"], getattr(s, kk + "_get_ranges")()["hi"]
            assert lo.tobytes() == boxes[kk][0].tobytes() and hi.tobytes() == boxes[kk][1].tobytes(), kk
        base_lo, base_hi, top_lo, top_hi = boxes[k]; rc = 0 if k == "spawn" else -1
        for lv in np.unique(rl):
            sel = rl == lv
            blo = boxes[k][0].copy(); bhi = boxes[k][1].copy()
            blo[rb[sel]] = tw.box(base_lo[rb[sel]], top_lo[rb[sel]], lv, L, rc); bhi[rb[sel]] = tw.box(base_hi[rb[sel]], top_hi[rb[sel]], lv, L, rc)
            s.timeline_set_ranges(3, blo, bhi, 5) if k == "timeline" else getattr(s, k + "_set_ranges")(blo, bhi, 5)
            assert getattr(s, k + "_draw")(rb[sel], re_[sel]).tobytes() == got[sel].tobytes(), lv
    finally:
        s.close()


def _run_kw(B, xy):
    return dict(duration=0.6, gait="trot", xy_yaw=xy, respawn=dict(every=0.1), metrics=True, randomize=dict(seed=4, cmd_vel_x=(0.0, 0.3), friction_mu=(0.5, 0.9)),
                terrain=dict(tiles=np.stack([T.ramp(8.0), T.stairs(0.05, 0.25), T.rough(0.02, seed=4, flat_radius=0.2)]), cell=T.CELL,
                             tile=np.arange(B) % 4 - 1, origin=T.centred_origin(xy[:, :2])),
                spawn=dict(seed=5, tile=(-1, 1), dx=(-0.1, 0.1), yaw=(0.2, 0.2)),
                timeline=dict(seed=6, n=3, t_first=(0.0, 0.1), gap=(0.02, 0.06), p_gait=0.5, gaits=["trot", "pace"], weights=dict(none=1.0, cmd_vel=1.0),
                              cmd_vel_y=(-0.1, 0.1)))


def test_a_flat_curriculum_changes_no_output():
    from qm_control_b200 import closed_loop
    B = 24; s = _solver(B); xy = np.zeros((B, 3))
    try:
        kw = _run_kw(B, xy)
        a = closed_loop.run(s, **kw)
        flat = dict(levels=4, start=np.arange(B) % 4, when=[("duration", ">=", 0.05, "pass")],
                    randomize=dict(friction_mu=(0.5, 0.9)), spawn=dict(tile=(-1, 1)), timeline=dict(p_gait=0.5, cmd_vel_y=(-0.1, 0.1)))
        b = closed_loop.run(s, curriculum=flat, **kw)
        assert set(b) - set(a) == {"curriculum_level", "episode_level", "curriculum_state"}
        for key in a:
            if isinstance(a[key], np.ndarray):
                assert a[key].tobytes() == b[key].tobytes(), key
            else:
                assert a[key] == b[key], key
        assert b["curriculum_state"][:, 3].min() >= 4 and np.any(b["curriculum_state"][:, 0] != np.arange(B) % 4)   # the levels moved
    finally:
        s.close()


def test_a_curriculum_run_draws_at_its_levels_follows_the_rule_and_restores_what_it_found():
    import torch
    from qm_control_b200 import closed_loop
    B = 32; s = _solver(B); xy = np.zeros((B, 3)); L = 5
    try:
        kw = _run_kw(B, xy); kw.update(duration=2.0, respawn=dict(every=0.2, hold=0.1))
        # what the run must leave: earlier ranges of every kind, robot terrain rows, no curriculum
        prev = _boxes(np.random.default_rng(3), B)
        s.episode_set_ranges(*prev["episode"][:2], seed=1); s.timeline_set_ranges(2, *prev["timeline"][:2], seed=2)
        s.sim_set_terrain(kw["terrain"]["tiles"][:2], T.CELL); s.sim_set_robot_terrain(np.zeros(B), np.zeros((B, 2)))
        s.spawn_set_ranges(*prev["spawn"][:2], seed=3)
        found = (_ranges(s), s.sim_get_robot_terrain()["tile"].tobytes(), s.sim_get_robot_terrain()["origin"].tobytes(), s.curriculum_get())
        cur = dict(levels=L, start=np.arange(B) % L, up_after=np.where(np.arange(B) % 2, 1, 2), down_after=1,
                   when=[("distance", ">=", 0.02, "pass"), ("max_tilt", ">=", 0.05, "fail")],
                   randomize=dict(friction_mu=(0.2, 0.9), cmd_vel_x=(0.0, 0.6)), spawn=dict(tile=(-1, 2), dx=(-0.3, 0.3)),
                   timeline=dict(p_gait=1.0, gap=(0.0, 0.03), weights=dict(none=0.2, cmd_vel=2.0)))
        seen = {k: [] for k in ("episode", "spawn", "timeline")}

        def wrap(kind, name, at):
            f = getattr(s, name)

            def call(*args, **kw_):
                f(*args, **kw_); torch.cuda.synchronize()
                seen[kind].append((args[0].cpu().numpy().copy(), args[1].cpu().numpy().copy(), args[at].cpu().numpy().copy()))
            return call
        s.episode_sample_dev = wrap("episode", "episode_sample_dev", 2); s.spawn_sample_dev = wrap("spawn", "spawn_sample_dev", 2)
        s.timeline_sample_dev = wrap("timeline", "timeline_sample_dev", 2)
        try:
            out = closed_loop.run(s, curriculum=cur, **kw)
        finally:
            for name in ("episode_sample_dev", "spawn_sample_dev", "timeline_sample_dev"):
                delattr(s, name)
        assert (_ranges(s), s.sim_get_robot_terrain()["tile"].tobytes(), s.sim_get_robot_terrain()["origin"].tobytes(), s.curriculum_get()) == found
        ep, el, M = out["episode"], out["episode_level"], out["episode_metrics"]; E = el.shape[1]
        assert E >= 8 and np.all((el >= 0) == ~np.isnan(M[..., 0]))
        # the rows the samplers drew are the rebuilt *_params at each episode's level
        for kind, calls in seen.items():
            P = out[kind + "_params"]; n = 0
            for mask, idx, rows in calls:
                for b in np.nonzero(mask)[0]:
                    r = rows[b].copy()
                    if kind == "timeline":
                        r[:, 0] -= 10.0
                    assert r.tobytes() == P[b, idx[b]].tobytes(), (kind, b, idx[b]); n += 1
            assert n == np.sum(el >= 0), kind
        # the levels follow the rule from each robot's start
        conditions = [(_lib.METRICS_LAYOUT.index(c), o, r) for c, o, _, r in cur["when"]]
        for b in range(B):
            row = [b % L, 1 if b % 2 else 2, 1, 0.02, 0.05, 0.0, 0.0]; state = [b % L, 0, 0, 0]
            assert el[b, 0] == b % L
            for e in range(E - 1):
                if el[b, e + 1] < 0:
                    break
                state = tw.step(state, row, int(M[b, e, 1]), M[b, e], L, conditions)
                assert el[b, e + 1] == state[0], (b, e)
            assert out["curriculum_state"][b].tolist() == state, b
        lv = out["curriculum_level"]; assert np.array_equal(lv, el[np.arange(B)[None], ep])
        steps = np.diff(np.where(el >= 0, el, -1), axis=1)[(el[:, 1:] >= 0)]
        assert len(np.unique(el[el >= 0])) >= 3 and np.any(steps > 0) and np.any(steps < 0)   # levels went up and down
    finally:
        s.close()
