"""Restarts where robots fell and restarts a Session requests, inside the GPU closed loop (DESIGN.md §4.18): a placed row stands a robot exactly as
the sampler stands it on that row; the "here" row keeps the tile point and heading across the restore; requests at every boundary are the every rule
byte for byte; a request's end reaches the metrics row and the curriculum, and the fall rule's end wins."""
import numpy as np
import pytest

from qm_control_b200 import _lib, closed_loop
from qm_control_b200 import terrain as T

pytestmark = pytest.mark.gpu

SB = 4096
MT = {n: i for i, n in enumerate(_lib.METRICS_LAYOUT)}


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


def _library():
    return np.stack([T.ramp(10.0), T.stairs(0.06, 0.25), T.rough(0.02, seed=4, flat_radius=0.2)])


def _setup(h, tile0, origin0):
    h.sim_set_terrain(_library(), T.CELL); h.sim_set_robot_terrain(tile0, origin0); h.state_est_set_ground(tile0, origin0)
    h.state_est_reset(np.zeros((len(tile0), 3))); h.attitude_reset(); h.slip_reset()


def _inputs(s, rng, B):
    q, _ = s.sim_standing_state(np.c_[rng.uniform(-0.2, 0.2, (B, 2)), rng.uniform(-np.pi, np.pi, B)])
    return dict(q=q, v=rng.standard_normal((B, 24)), rbd=rng.standard_normal((B, _lib.RBD)), contact=rng.integers(0, 16, B).astype(np.int32),
                x_obs=rng.standard_normal((B, _lib.NX)), last_ee=np.c_[rng.standard_normal((B, 3)), np.tile([0.0, 0.0, 0.0, 1.0], (B, 1))],
                rbd_est=rng.standard_normal((B, _lib.RBD)))


def _rows_state(s):
    ter, gm = s.sim_get_robot_terrain(), s.state_est_get_ground()
    return dict(tile=ter["tile"], origin=ter["origin"], gm_tile=gm["tile"], gm_origin=gm["origin"], se=s.state_est_get(), at=s.attitude_get(), sl=s.slip_get())


def _flat(d):
    out = {}
    for k, v in d.items():
        if isinstance(v, dict):
            out.update({k + "." + kk: np.asarray(vv) for kk, vv in v.items()})
        else:
            out[k] = np.asarray(v)
    return out


def test_place_is_the_sampler_on_that_row_and_rejected_rows_write_nothing():
    rng = np.random.default_rng(11); s = _solver(SB); p = _solver(SB)
    try:
        tile0 = rng.integers(-1, 3, SB); origin0 = T.centred_origin(np.zeros((SB, 2)))
        for h in (s, p):
            _setup(h, tile0, origin0)
        rows = np.c_[rng.integers(-1, 3, SB), rng.uniform(-0.4, 0.4, (SB, 2)), rng.uniform(-np.pi, np.pi, SB)]
        rows[::7, 3] = np.pi; rows[1::7, 3] = -np.pi
        inp = _inputs(s, rng, SB); mask = (rng.random(SB) < 0.7).astype(np.int32); episode = rng.integers(0, 1000, SB).astype(np.int32)
        s.spawn_set_ranges(rows, rows, 7)   # lo = hi: the sampler's row is the given row itself
        a = s.spawn_sample(mask, episode, link=_lib.SPAWN_GROUND_MAP, **inp)
        b = p.spawn_place(mask, rows, origin0, link=_lib.SPAWN_GROUND_MAP, **inp)
        m = mask != 0
        assert a["rows"][m].tobytes() == rows[m].tobytes() and np.all(b["status"] == 0)
        for k in ("q", "v", "rbd", "contact", "x_obs", "last_ee", "rbd_est"):
            assert a[k].tobytes() == b[k].tobytes(), k
            assert b[k][~m].tobytes() == np.asarray(inp[k])[~m].tobytes(), k   # unmasked robots byte-unchanged
        ra, rb = _flat(_rows_state(s)), _flat(_rows_state(p))
        for k in ra:
            assert ra[k].tobytes() == rb[k].tobytes(), k

        # rejected rows: every class writes nothing and sets ST_SPAWN; the rest of the mask is placed
        bad = rows.copy(); cls = np.arange(SB) % 8
        bad[cls == 1, 0] = 0.5; bad[cls == 2, 0] = 3.0; bad[cls == 3, 0] = -2.0; bad[cls == 4, 1] = np.nan; bad[cls == 5, 2] = np.inf; bad[cls == 6, 3] = 3.2
        bad[cls == 7, 3] = np.nan
        before = _flat(_rows_state(p))
        c = p.spawn_place(np.ones(SB, np.int32), bad, origin0, link=_lib.SPAWN_GROUND_MAP, **inp)
        rej = cls != 0
        np.testing.assert_array_equal(c["status"], np.where(rej, _lib.ST_SPAWN, 0))
        for k in ("q", "v", "rbd", "contact", "x_obs", "last_ee", "rbd_est"):
            assert c[k][rej].tobytes() == np.asarray(inp[k])[rej].tobytes(), k
        after = _flat(_rows_state(p))
        for k in ("tile", "origin", "gm_tile", "gm_origin"):
            assert after[k][rej].tobytes() == before[k][rej].tobytes(), k
        # a tile >= 0 without robot terrain rows is rejected too
        p.state_est_set_ground(None); p.sim_set_robot_terrain(None)
        d = p.spawn_place(np.ones(SB, np.int32), rows, origin0, **inp)
        np.testing.assert_array_equal(d["status"], np.where(rows[:, 0] >= 0, _lib.ST_SPAWN, 0))
        with pytest.raises(_lib.QmbError, match="ground-map link needs"):
            p.spawn_place(mask, rows, origin0, link=_lib.SPAWN_GROUND_MAP, **inp)
        with pytest.raises(_lib.QmbError, match="unknown link bits"):
            p.spawn_place(mask, rows, origin0, link=4, **inp)
    finally:
        s.close(); p.close()


def test_here_then_place_keeps_the_tile_point_and_the_heading():
    import torch
    rng = np.random.default_rng(12); B = SB; s = _solver(B)
    try:
        tile0 = rng.integers(-1, 3, B); origin0 = T.centred_origin(np.zeros((B, 2)))
        _setup(s, tile0, origin0)
        start = np.c_[rng.uniform(-0.2, 0.2, (B, 2)), rng.uniform(-np.pi, np.pi, B)]
        q_start, _ = s.sim_standing_state(start)
        o_now = origin0 + rng.uniform(-0.3, 0.3, (B, 2)); s.sim_set_robot_terrain(tile0, o_now); s.state_est_set_ground(tile0, o_now)   # an earlier place
        rbd = rng.standard_normal((B, _lib.RBD)); rbd[:, 3:5] = start[:, :2] + rng.uniform(-0.5, 0.5, (B, 2)); rbd[:, 0] = rng.uniform(-9.0, 9.0, B)
        rbd[:4, 0] = [np.pi, -np.pi, 3 * np.pi, -7.0]
        mask = (rng.random(B) < 0.8).astype(np.int32); m = mask != 0
        rows_h = s.spawn_here(mask, rbd, q_start, origin0)
        dev = torch.device("cuda:0"); t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)
        rows_d = t(np.zeros((B, 4)))
        s.spawn_here_dev(t(mask, torch.int32), t(rbd), t(q_start), t(origin0), rows_d); torch.cuda.synchronize()
        assert rows_d.cpu().numpy().tobytes() == rows_h.tobytes()
        assert np.all(rows_h[~m] == 0.0) and np.all(np.abs(rows_h[m, 3]) <= np.pi)
        inp = _inputs(s, rng, B); inp["q"] = q_start
        out = s.spawn_place(mask, rows_h, origin0, link=_lib.SPAWN_GROUND_MAP, **inp)
        assert np.all(out["status"] == 0)
        ter = s.sim_get_robot_terrain()
        np.testing.assert_array_equal(ter["tile"][m], tile0[m])
        np.testing.assert_allclose(out["q"][m, 0:2] - ter["origin"][m], rbd[m, 3:5] - o_now[m], rtol=0, atol=1e-12)   # the same tile point
        np.testing.assert_array_equal(out["q"][m, 0:2], q_start[m, 0:2])
        np.testing.assert_allclose(np.exp(1j * out["q"][m, 3]), np.exp(1j * rbd[m, 0]), rtol=0, atol=1e-12)   # the same heading
        qh, _ = s.sim_standing_state(np.c_[q_start[:, 0:2], rows_h[:, 3]])   # on the new terrain rows
        np.testing.assert_allclose(out["q"][m], qh[m], rtol=0, atol=1e-12)
    finally:
        s.close()


RUN = dict(gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), metrics=True)


def _keys(out):
    return {k: np.asarray(v) for k, v in out.items() if not isinstance(v, (list, tuple))}


def _session(s, duration, at_window, mask_fn=None, end=2, at=None, respawn=None, **kw):
    import torch
    recs = []
    with closed_loop.Session(s, duration, **dict(RUN, respawn=respawn or dict(on_fall=False, on_request=True), **kw)) as ss:
        for i in range(ss.windows):
            if i > 0 and i % at_window == 0:
                ss.respawn(torch.ones(s.batch, dtype=torch.int32, device=ss.device) if mask_fn is None else mask_fn(ss), end=end, at=at)
            recs.append(ss.step(1))
        end_keys = ss.finish()
    rec = {k: np.concatenate([r[k] if isinstance(r[k], np.ndarray) else r[k].cpu().numpy() for r in recs]) for k in recs[0]}
    rec.update(end_keys)
    return rec


def test_requests_at_every_boundary_are_the_every_rule_byte_for_byte():
    B = 64; s = _solver(B)
    try:
        want = closed_loop.run(s, 0.3, **dict(RUN, respawn=dict(on_fall=False, every=0.1)))
        got = _session(s, 0.3, 10)
        assert set(_keys(want)) == set(_keys(got))
        for k, v in _keys(want).items():
            assert v.tobytes() == _keys(got)[k].tobytes(), k
    finally:
        s.close()


def test_a_random_request_changes_only_the_requested_robots_and_here_keeps_the_tile_point():
    import torch
    B = 64; s = _solver(B); rng = np.random.default_rng(3)
    try:
        tiles = np.stack([T.stairs(0.04, 0.25), T.rough(0.02, seed=4, flat_radius=0.2)])
        ter = dict(tiles=tiles, cell=T.CELL, tile=rng.integers(0, 2, B), origin=T.centred_origin(np.zeros((B, 2))))
        mask = (rng.random(B) < 0.5).astype(np.int32); m = mask != 0
        plain = _session(s, 0.3, 1000, terrain=ter)
        start = _session(s, 0.3, 15, mask_fn=lambda ss: torch.as_tensor(mask, device=ss.device), at="start", terrain=ter)
        here = _session(s, 0.3, 15, mask_fn=lambda ss: torch.as_tensor(mask, device=ss.device), at="here", terrain=ter)
        for k in ("base", "ee", "status"):   # unmasked robots are the session without requests; every robot's first episode too
            assert start[k][:, ~m].tobytes() == plain[k][:, ~m].tobytes() and here[k][:, ~m].tobytes() == plain[k][:, ~m].tobytes(), k
            assert here[k][:15].tobytes() == plain[k][:15].tobytes() and start[k][:15].tobytes() == plain[k][:15].tobytes(), k
        n = 15   # noise-free, a robot back at its start repeats its first episode for the common length
        assert start["base"][15:15 + n, m].tobytes() == plain["base"][:n, m].tobytes()
        np.testing.assert_array_equal(here["episode"][15:, m], 1); np.testing.assert_array_equal(here["episode"][15:, ~m], 0)
        # the first record of the placed episode lies over the point it left, in tile coordinates (10 ms of walking apart)
        sp = here["spawn_params"]; origin0 = ter["origin"]
        left = here["base"][14, m, 0:2] - (origin0[m] - sp[m, 0, 1:3]); placed = here["base"][15, m, 0:2] - (origin0[m] - sp[m, 1, 1:3])
        assert np.all(np.linalg.norm(placed - left, axis=1) < 0.02)
        np.testing.assert_array_equal(sp[m, 1, 0], ter["tile"][m]); assert np.all(np.isnan(sp[~m, 1]))
        assert np.all(np.abs(np.angle(np.exp(1j * (here["base"][15, m, 3] - here["base"][14, m, 3])))) < 0.05)
        assert not np.any(here["status"] & _lib.ST_SPAWN)
    finally:
        s.close()


def test_a_requests_end_reaches_the_metrics_and_the_curriculum_and_the_fall_rule_wins():
    import torch
    B = 32; s = _solver(B)
    try:
        end = torch.tensor(np.where(np.arange(B) % 2 == 0, 1, 2), dtype=torch.int32)
        cur = dict(levels=3, start=1, randomize=dict(friction_mu=(0.6, 0.6)))
        out = _session(s, 0.1, 5, end=end, respawn=dict(on_fall=False, every=10.0, on_request=True), randomize=dict(friction_mu=(0.8, 0.8)), curriculum=cur)
        np.testing.assert_array_equal(out["episode_metrics"][:, 0, MT["end"]], end.numpy())
        np.testing.assert_array_equal(out["episode_level"][:, 1], np.where(end.numpy() == 1, 0, 2))   # end 1 steps down, end 2 (passing) steps up
        # z_min above any base: every robot falls in every window and restarts at every boundary, the request's among them
        fell = _session(s, 0.1, 5, end=2, respawn=dict(on_fall=True, hold=0.01, z_min=5.0, on_request=True))
        ends = fell["episode_metrics"][:, :, MT["end"]]
        assert ends.shape[1] == 10 and np.all(ends[:, :-1] == 1) and np.all(ends[:, -1] == 0)
    finally:
        s.close()


def test_a_respawn_run_here_on_stairs_stands_every_restart_over_its_fall_point():
    B = 64; s = _solver(B); rng = np.random.default_rng(8)
    try:
        ter = dict(tiles=np.stack([T.stairs(0.04, 0.25)]), cell=T.CELL, tile=np.zeros(B), origin=T.centred_origin(np.zeros((B, 2))))
        rs = dict(on_fall=True, hold=0.15, z_min=5.0)   # z_min above any base: every robot "falls" and restarts every 150 ms
        here = closed_loop.run(s, 0.5, **dict(RUN, terrain=ter, respawn=dict(rs, at="here")))
        start = closed_loop.run(s, 0.5, **dict(RUN, terrain=ter, respawn=dict(rs, at="start")))
        ep = here["episode"]; sp = here["spawn_params"]; o0 = ter["origin"]
        first = np.argmax(ep > 0, axis=0); restarted = ep[-1] > 0
        assert restarted.all() and np.all(np.isfinite(sp[:, :ep[-1].min() + 1]))
        for b in np.nonzero(restarted)[0]:
            i = first[b]; e = ep[i, b]
            left = here["base"][i - 1, b, 0:2] - (o0[b] - sp[b, e - 1, 1:3]); placed = here["base"][i, b, 0:2] - (o0[b] - sp[b, e, 1:3])
            assert np.linalg.norm(placed - left) < 0.02, b
        for k in ("base", "ee", "status", "episode", "fallen"):   # until a robot's first restart both runs are one
            for b in range(B):
                n = first[b] if restarted[b] else len(ep)
                assert here[k][:n, b].tobytes() == start[k][:n, b].tobytes(), (k, b)
    finally:
        s.close()
