"""Per-episode spawns inside the GPU closed loop (closed_loop.run(spawn=...), DESIGN.md §4.12): the device sampler is the host draw bit for bit, stands
each robot where the host would, writes the reset rows the resets write and nothing for unmasked robots; every spawned episode is the first episode
of a run fixed at its rows; yaw-only spawns stand; the previous terrain rows and ground map are back after a run."""
import numpy as np
import pytest

from qm_control_b200 import _lib
from qm_control_b200 import terrain as T

pytestmark = pytest.mark.gpu

SP = {n: i for i, n in enumerate(_lib.SPAWN_LAYOUT)}
EP = {n: i for i, n in enumerate(_lib.EPISODE_LAYOUT)}
REC = ("base", "ee", "status")


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


def _library():
    return np.stack([T.ramp(10.0), T.stairs(0.06, 0.25), T.rough(0.02, seed=4, flat_radius=0.2)])


# ---------------- 1: the sampler ----------------
SB = 4096


def _inputs(s, rng, B):
    xy = np.c_[rng.uniform(-0.2, 0.2, (B, 2)), rng.uniform(-np.pi, np.pi, B)]
    q, v = s.sim_standing_state(xy)
    return dict(q=q, v=rng.standard_normal((B, 24)), rbd=rng.standard_normal((B, _lib.RBD)), contact=rng.integers(0, 16, B).astype(np.int32),
                x_obs=rng.standard_normal((B, _lib.NX)), last_ee=np.c_[rng.standard_normal((B, 3)), np.tile([0.0, 0.0, 0.0, 1.0], (B, 1))],
                rbd_est=rng.standard_normal((B, _lib.RBD)))


def _rows_state(s):
    return dict(ter=s.sim_get_robot_terrain(), gm=s.state_est_get_ground(), se=s.state_est_get(), at=s.attitude_get(), sl=s.slip_get())


def test_sample_is_the_host_draw_and_stands_every_robot_where_the_host_would():
    rng = np.random.default_rng(5); s = _solver(SB); ref = _solver(SB)
    try:
        tiles = _library(); s.sim_set_terrain(tiles, T.CELL); ref.sim_set_terrain(tiles, T.CELL)
        tile0 = rng.integers(-1, 3, SB); origin0 = T.centred_origin(np.zeros((SB, 2)))
        for h in (s, ref):
            h.sim_set_robot_terrain(tile0, origin0); h.state_est_set_ground(tile0, origin0)
            h.state_est_reset(np.zeros((SB, 3))); h.attitude_reset(); h.slip_reset()
        lo = np.tile([-1.0, -0.4, -0.3, -np.pi], (SB, 1)); hi = np.tile([2.0, 0.4, 0.3, np.pi], (SB, 1)); lo[::5] = hi[::5]; seed = 2 ** 64 - 99
        inp = _inputs(s, rng, SB); mask = (rng.random(SB) < 0.7).astype(np.int32); episode = rng.integers(0, 1000, SB).astype(np.int32)
        # refusals write nothing
        with pytest.raises(_lib.QmbError, match="no ranges"):
            s.spawn_sample(mask, episode, **inp)
        l2 = lo.copy(); l2[9, SP["tile"]] = 3.0
        with pytest.raises(_lib.QmbError, match="tile of robot 9"):
            s.spawn_set_ranges(l2, np.maximum(hi, l2), seed)
        assert s.spawn_get_ranges() is None
        s.spawn_set_ranges(lo, hi, seed)
        before = _rows_state(s)
        s.sim_set_robot_terrain(None)
        with pytest.raises(_lib.QmbError, match="cleared since"):
            s.spawn_sample(mask, episode, **inp)
        s.sim_set_robot_terrain(tile0, origin0); s.state_est_set_ground(None)
        with pytest.raises(_lib.QmbError, match="ground-map link needs"):
            s.spawn_sample(mask, episode, link=_lib.SPAWN_GROUND_MAP, **inp)
        s.state_est_set_ground(tile0, origin0)
        after = _rows_state(s)
        for k in ("ter", "gm"):
            for f in before[k]:
                assert before[k][f].tobytes() == after[k][f].tobytes(), (k, f)
        for k in ("se", "at", "sl"):
            for f in before[k]:
                assert np.asarray(before[k][f]).tobytes() == np.asarray(after[k][f]).tobytes(), (k, f)

        out = s.spawn_sample(mask, episode, link=_lib.SPAWN_GROUND_MAP, **inp)
        m = mask != 0; u = ~m
        rows = s.spawn_draw(np.arange(SB), episode)
        assert out["rows"][m].tobytes() == rows[m].tobytes() and np.all(out["rows"][u] == 0.0)
        ter = s.sim_get_robot_terrain(); gm = s.state_est_get_ground()   # the getters wait for the device
        np.testing.assert_array_equal(ter["tile"][m], rows[m, 0]); np.testing.assert_array_equal(ter["tile"][u], tile0[u])
        want = origin0 - rows[:, 1:3]
        assert ter["origin"][m].tobytes() == want[m].tobytes() and ter["origin"][u].tobytes() == origin0[u].tobytes()
        assert gm["tile"].tobytes() == ter["tile"].tobytes() and gm["origin"].tobytes() == ter["origin"].tobytes()
        # q: the host's standing pose on the drawn rows (qmb200_sim_standing_state reads them), bit for bit on the plane
        xy = np.c_[inp["q"][:, 0:2], np.where(m, rows[:, 3], inp["q"][:, 3])]
        qh, _ = s.sim_standing_state(xy)
        plane = m & (rows[:, 0] < 0)
        assert plane.sum() > 500 and out["q"][plane].tobytes() == qh[plane].tobytes()
        np.testing.assert_allclose(out["q"][m], qh[m], rtol=0, atol=1e-12)
        assert np.ptp(out["q"][m & (rows[:, 0] == 0), 4]) > 0.1   # the ramp tilts the robots
        assert np.all(out["v"][m] == 0.0)
        # the deepest foot sits at the static penetration: the rbd's base and joints, and the contact flags of the feet it presses in
        r = out["rbd"]
        np.testing.assert_array_equal(r[m][:, 3:6], out["q"][m][:, 0:3]); np.testing.assert_array_equal(r[m][:, 0:3], out["q"][m][:, 3:6])
        np.testing.assert_array_equal(r[m][:, 6:24], out["q"][m][:, 6:24]); assert np.all(r[m][:, 24:48] == 0.0)
        assert np.all(out["contact"][m] != 0)
        np.testing.assert_allclose(s.centroidal_state_from_rbd(r)[m], out["x_obs"][m], rtol=0, atol=1e-12)
        assert out["rbd_est"][m].tobytes() == r[m].tobytes()
        # the held end-effector target turned about the base by the yaw change
        dy = rows[:, 3] - inp["q"][:, 3]; c, sn = np.cos(dy), np.sin(dy); e0 = inp["last_ee"]; rel = e0[:, :2] - inp["q"][:, :2]
        turned = inp["q"][:, :2] + np.c_[c * rel[:, 0] - sn * rel[:, 1], sn * rel[:, 0] + c * rel[:, 1]]
        np.testing.assert_allclose(out["last_ee"][m][:, :2], turned[m], rtol=0, atol=1e-12); np.testing.assert_array_equal(out["last_ee"][m][:, 2], e0[m][:, 2])
        np.testing.assert_allclose(out["last_ee"][m][:, 5], np.sin(0.5 * dy[m]), rtol=0, atol=1e-12)
        # unmasked robots are byte-unchanged in every row
        for k in ("q", "v", "rbd", "contact", "x_obs", "last_ee", "rbd_est"):
            assert out[k][u].tobytes() == np.asarray(inp[k])[u].tobytes(), k
        # the reset rows: byte-equal to what the resets write at the new base positions, unmasked rows as they were
        base = np.where(m[:, None], out["q"][:, 0:3], 0.0)
        ref.state_est_reset(base); ref.attitude_reset(); ref.slip_reset()
        got, exp = _rows_state(s), _rows_state(ref)
        for k in ("se", "at", "sl"):
            for f in got[k]:
                assert np.asarray(got[k][f]).tobytes() == np.asarray(exp[k][f]).tobytes(), (k, f)
    finally:
        s.close(); ref.close()


# ---------------- 2: every spawned episode is the first episode of a run fixed at its rows ----------------
NB, EVERY_S, EPISODES = 16, 0.2, 3
RANDOMIZE = dict(seed=77, friction_mu=(0.4, 1.0), m_ee=(0.0, 1.5), cmd_vel_x=(0.0, 0.3))
SPAWN = dict(seed=31, tile=(-1, 2), dx=(-0.1, 0.1), dy=(-0.1, 0.1), yaw=(-np.pi, np.pi))


def _case(case):
    xy = np.zeros((NB, 3)); xy[:, 0] = 5.0 * np.arange(NB)
    kw = dict(gait="trot", xy_yaw=xy, terrain=dict(tiles=_library(), cell=T.CELL, tile=np.arange(NB) % 4 - 1, origin=T.centred_origin(xy[:, :2])))
    if case == "estimate":
        kw.update(state_estimator=True, attitude_filter=True, slip_detector=True, ground_map=True)
    if case == "commands":
        kw.update(gait="stance", commands=dict(t=np.full((NB, 1), 0.05), gait=np.full((NB, 1), "trot", dtype=object)))
    return kw


@pytest.mark.parametrize("case", ["truth", "estimate", "commands"])
def test_every_episode_is_the_first_episode_of_a_run_fixed_at_its_rows(case):
    from qm_control_b200 import closed_loop
    kw = _case(case); n = int(round(EVERY_S * 100))
    s = _solver(NB)
    try:
        r = closed_loop.run(s, duration=EVERY_S * EPISODES, respawn=dict(on_fall=False, every=EVERY_S), randomize=RANDOMIZE, spawn=SPAWN, **kw)
        assert s.sim_get_robot_terrain() is None and s.state_est_get_ground() is None and s.spawn_get_ranges() is None
    finally:
        s.close()
    P, S = r["episode_params"], r["spawn_params"]
    assert S.shape == (NB, EPISODES, _lib.SPAWN) and np.all(np.isin(S[:, :, 0], [-1, 0, 1, 2]))
    assert len(np.unique(S[:, :, 0])) == 4 and np.all(S[:, 1, 3] != S[:, 0, 3])
    for e in range(EPISODES):
        fixed = {f: (P[:, e, EP[f]], P[:, e, EP[f]]) for f in RANDOMIZE if f != "seed"}
        sfix = {f: (S[:, e, SP[f]], S[:, e, SP[f]]) for f in SPAWN if f != "seed"}
        s = _solver(NB)
        try:
            ref = closed_loop.run(s, duration=EVERY_S, respawn=dict(on_fall=False, every=EVERY_S), randomize=dict(seed=5, **fixed), spawn=dict(seed=6, **sfix), **kw)
        finally:
            s.close()
        assert ref["spawn_params"][:, 0].tobytes() == S[:, e].tobytes()
        for k in REC + (("base_est",) if case == "estimate" else ()):
            assert r[k][e * n:(e + 1) * n].tobytes() == ref[k][:n].tobytes(), "%s episode %d" % (k, e)


# ---------------- 3: yaw-only spawns on flat ground stand ----------------
def test_yaw_only_spawns_stand_and_hold_the_end_effector_turned_with_the_base():
    from qm_control_b200 import closed_loop
    B = 64; xy = np.zeros((B, 3)); xy[:, 0] = 3.0 * np.arange(B)
    yaw = np.where(np.arange(B) % 2 == 0, 0.0, np.linspace(-np.pi, np.pi, B))   # even robots at yaw 0: the same run's reference
    s = _solver(B)
    try:
        r = closed_loop.run(s, duration=1.0, gait="stance", xy_yaw=xy, spawn=dict(yaw=(yaw, yaw)))
    finally:
        s.close()
    z = r["base"][:, :, 2]; roll_pitch = np.abs(r["base"][:, :, 4:6]).max(axis=(0, 2))
    assert np.all(z.min(axis=0) > 0.3) and np.all(roll_pitch < 0.3), "no robot falls"
    # the end effector stays near its spawn pose turned with the base: its offset from the base in the yawed frame
    rel = r["ee"][:, :, :2] - r["base"][:, :, 0:2]; c, sn = np.cos(yaw), np.sin(yaw)
    local = np.stack([c * rel[..., 0] + sn * rel[..., 1], -sn * rel[..., 0] + c * rel[..., 1]], -1)   # the offset in the spawned heading's frame
    drift = np.linalg.norm(local[-1] - local[0], axis=-1); d0 = drift[0::2]; d1 = drift[1::2]
    assert np.abs(local[0, 1::2] - local[0, 0:1]).max() < 0.01   # every heading starts with the yaw-0 robots' offset, turned
    print("end-effector offset drift after 1 s: yaw 0 max %.4f m, spawned yaws max %.4f m" % (d0.max(), d1.max()))
    # the first H100 run gave 0.0316 m for both groups: the bound sits 10 % above it, and the spawned headings drift as the yaw-0 robots do
    assert d1.max() < 0.035 and d0.max() < 0.035 and abs(d1.max() - d0.max()) < 0.002


# ---------------- 4: the refusals that need a changed library or a bad link, and the restore of earlier rows ----------------
def test_a_shrunk_library_and_an_unknown_link_are_refused_writing_nothing():
    B = 64; rng = np.random.default_rng(9); s = _solver(B)
    try:
        tiles = _library(); s.sim_set_terrain(tiles, T.CELL)
        tile0 = rng.integers(-1, 2, B); origin0 = T.centred_origin(np.zeros((B, 2)))
        s.sim_set_robot_terrain(tile0, origin0)
        s.spawn_set_ranges(np.tile([-1.0, -0.1, -0.1, -1.0], (B, 1)), np.tile([2.0, 0.1, 0.1, 1.0], (B, 1)), 3)
        inp = _inputs(s, rng, B); mask = np.ones(B, dtype=np.int32); episode = np.zeros(B, dtype=np.int32)
        ter = s.sim_get_robot_terrain()
        with pytest.raises(_lib.QmbError, match="unknown link bits 2"):
            s.spawn_sample(mask, episode, link=2, **inp)
        s.sim_set_terrain(tiles[:2], T.CELL)   # every robot row is on tile <= 1: the library may shrink, below the ranges' tile bound 2
        with pytest.raises(_lib.QmbError, match="fewer tiles than the ranges draw from"):
            s.spawn_sample(mask, episode, **inp)
        after = s.sim_get_robot_terrain()
        assert after["tile"].tobytes() == ter["tile"].tobytes() and after["origin"].tobytes() == ter["origin"].tobytes()
        s.sim_set_terrain(tiles, T.CELL)
        out = s.spawn_sample(mask, episode, **inp)   # the same library again: the ranges are good
        assert np.all(out["rows"][:, 0] <= 2) and np.any(out["rows"][:, 0] == 2)
    finally:
        s.close()


def test_earlier_terrain_rows_ground_map_and_ranges_are_back_after_a_run():
    from qm_control_b200 import closed_loop
    B = 8; xy = np.zeros((B, 3)); xy[:, 0] = 5.0 * np.arange(B); s = _solver(B)
    try:
        lib0 = np.stack([T.flat(), T.ramp(5.0)]); s.sim_set_terrain(lib0, T.CELL)
        t0 = np.arange(B) % 3 - 1; o0 = T.centred_origin(xy[:, :2]) + 0.125
        s.sim_set_robot_terrain(t0, o0); s.state_est_set_ground(t0[::-1].copy(), o0 - 0.5)
        lo0 = np.tile([0.0, -0.2, 0.0, -0.5], (B, 1)); hi0 = np.tile([1.0, 0.2, 0.0, 0.5], (B, 1)); s.spawn_set_ranges(lo0, hi0, 17)
        before = (s.sim_get_terrain(), s.sim_get_robot_terrain(), s.state_est_get_ground(), s.spawn_get_ranges())
        ter = dict(tiles=_library(), cell=T.CELL, tile=np.arange(B) % 4 - 1, origin=T.centred_origin(xy[:, :2]))
        r = closed_loop.run(s, duration=0.1, gait="trot", xy_yaw=xy, terrain=ter, state_estimator=True, ground_map=True, spawn=dict(seed=2, tile=(0, 2), dx=(-0.2, 0.0), yaw=(-3.0, 3.0)))
        assert np.all(r["spawn_params"][:, 0, 0] >= 0)
        after = (s.sim_get_terrain(), s.sim_get_robot_terrain(), s.state_est_get_ground(), s.spawn_get_ranges())
        for a, b in zip(before, after):
            assert a.keys() == b.keys()
            for k in a:
                assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k
        # the earlier ranges draw from the earlier origins again: a spawn on the earlier library lands where one before the run would
        inp = _inputs(s, np.random.default_rng(1), B); out = s.spawn_sample(np.ones(B, dtype=np.int32), np.zeros(B, dtype=np.int32), **inp)
        got = s.sim_get_robot_terrain()
        assert got["origin"].tobytes() == (o0 - out["rows"][:, 1:3]).tobytes()
    finally:
        s.close()
