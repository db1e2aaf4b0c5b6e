"""The state estimator's ground map on the device (qmb200_state_est_set_ground, closed_loop.run(ground_map=...)), 64 robots.

The entry points and their interplay with the plant's tile library; a recorded noisy trot replayed through state_est_step with no map, an all -1 map
and a constant tile at ground_height, byte for byte; the raised-map identity; the map kernel call by call against the twin (tests/_ground_est_twin.py)
on a mixed library; and closed loops on terrain with the controller reading the estimate."""
import numpy as np
import pytest

from qm_control_b200 import _lib
from qm_control_b200 import terrain as TR

pytestmark = pytest.mark.gpu

NL = 64


def _solver(batch=NL):
    import qm_control_b200 as q
    return q.Solver(batch=batch, device=0)


def _wrap(a):
    return (a + np.pi) % (2 * np.pi) - np.pi


def _upright(r, ter):
    base = r["base"]; ground = TR.height(ter["tiles"], ter["cell"], ter["tile"][None], ter["origin"][None], base[:, :, :2])
    return np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2] - ground, axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3)


def _mixed(B=NL):
    """a 10 deg ramp, 6 cm stairs and 1 cm rough ground, each under its share of the robots from the start on, plus the flat plane on tile -1"""
    tiles = np.stack([TR.ramp(10.0), TR.stairs(0.06, 0.3, start=0.1), TR.rough(0.01, seed=7)])
    tile = np.arange(B) % 4 - 1
    return dict(tiles=tiles, cell=TR.CELL, tile=tile.astype(np.int32), origin=TR.centred_origin(np.zeros((B, 2))))


def _record(s, **kw):
    """closed_loop.run with every estimator call recorded → [(dt, sensors, contact, rbd_est, status, state_est_get)]"""
    import torch
    from qm_control_b200 import closed_loop
    rec = []; orig = s.state_est_step_dev

    def wrapped(dt, sensors, contact, rbd_est, status, stream=None):
        sn, c = sensors.clone(), contact.clone()
        orig(dt, sensors, contact, rbd_est, status, stream)
        torch.cuda.synchronize()
        rec.append((dt, sn.cpu().numpy(), c.cpu().numpy(), rbd_est.cpu().numpy(), status.cpu().numpy(), s.state_est_get()))
    s.state_est_step_dev = wrapped
    try:
        r = closed_loop.run(s, **kw)
    finally:
        del s.state_est_step_dev
    return r, rec


def _replay(s, base_pos, rec):
    """the recorded calls through the host entry point → [(x, p_diag, rbd_est, status)]"""
    s.state_est_reset(base_pos); out = []
    for dt, sens, contact, _, _, _ in rec:
        rbd, st = s.state_est_step(dt, sens, contact); g = s.state_est_get()
        out.append((g["x"], g["p_diag"], rbd, st))
    return out


def test_ground_map_entry_points():
    s = _solver(batch=4)
    try:
        assert s.state_est_get_ground() is None
        s.state_est_set_ground(-1); g = s.state_est_get_ground()   # no library: only the plane
        assert np.array_equal(g["tile"], [-1] * 4) and np.array_equal(g["origin"], np.zeros((4, 2)))
        with pytest.raises(_lib.QmbError, match="tile must be -1 or a tile of the library"):
            s.state_est_set_ground([0, -1, -1, -1])
        tiles = np.stack([TR.flat(1.0), TR.ramp(5.0, size=1.0), TR.rough(0.01, size=1.0)])
        s.sim_set_terrain(tiles, TR.CELL)
        tile = np.array([2, -1, 0, 1], dtype=np.int32); origin = np.arange(8.0).reshape(4, 2)
        s.state_est_set_ground(tile, origin); g = s.state_est_get_ground()
        assert np.array_equal(g["tile"], tile) and np.array_equal(g["origin"], origin)
        assert s.sim_get_robot_terrain() is None   # the plant's rows are its own
        for bad in (dict(tile=[3, 0, 0, 0], origin=origin), dict(tile=[-2, 0, 0, 0], origin=origin), dict(tile=tile, origin=np.full((4, 2), np.nan)),
                    dict(tile=tile, origin=np.full((4, 2), np.inf))):
            with pytest.raises(_lib.QmbError, match="qmb200_state_est_set_ground"):
                s.state_est_set_ground(**bad)
            g = s.state_est_get_ground(); assert np.array_equal(g["tile"], tile) and np.array_equal(g["origin"], origin)   # unchanged
        # a handle setting: the filter's reset and stop leave it
        s.state_est_reset(np.zeros((4, 3))); s.state_est_stop()
        assert np.array_equal(s.state_est_get_ground()["tile"], tile)
        # the library may not lose a tile the map references; clearing it clears the map with the robots' terrain
        with pytest.raises(_lib.QmbError, match="ground map references a tile"):
            s.sim_set_terrain(tiles[:2], TR.CELL)
        assert s.sim_get_terrain()["tiles"].shape[0] == 3
        s.sim_set_terrain(tiles[::-1], TR.CELL * 2)   # as many tiles: accepted, the map keeps its rows
        assert np.array_equal(s.state_est_get_ground()["tile"], tile)
        s.sim_set_robot_terrain(tile, origin)
        s.sim_set_terrain(None)
        assert s.state_est_get_ground() is None and s.sim_get_robot_terrain() is None
        s.sim_set_terrain(tiles, TR.CELL); s.state_est_set_ground(1); s.state_est_set_ground(None)
        assert s.state_est_get_ground() is None
    finally:
        s.close()


@pytest.fixture(scope="module")
def trot_record():
    """a 0.3 s trot of 64 robots on the plane with the reference sensor noise and the attitude filter: the recorded estimator calls"""
    s = _solver(); rng = np.random.default_rng(4); xy = np.c_[rng.uniform(-1, 1, (NL, 2)), rng.uniform(-np.pi, np.pi, NL)]
    try:
        _, rec = _record(s, duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, state_estimator=True, sensor_noise="reference", attitude_filter=True)
    finally:
        s.close()
    assert len(rec) == 301
    return rec


def test_plane_maps_are_bit_identical(trot_record):
    """No map, an all -1 map and a constant tile at the plant's ground_height: x, diag P, rbd_est and status byte-identical over every call"""
    rec = trot_record; s = _solver(); base = rec[0][5]["x"][:, 0:3]
    try:
        for gh in (0.0, 0.04):
            s.sim_set_params(ground_height=gh); s.state_est_set_params(foot_height=gh + 0.0265 - s.robot_mass * 9.81 / 4e6)
            s.sim_set_terrain(None); want = _replay(s, base + [0, 0, gh], rec)
            s.state_est_set_ground(-1); minus = _replay(s, base + [0, 0, gh], rec)
            s.sim_set_terrain(np.full((1,) + TR.flat().shape, gh), TR.CELL); s.state_est_set_ground(0, TR.centred_origin(np.zeros((NL, 2))))
            const = _replay(s, base + [0, 0, gh], rec)
            for k, (w, a, b) in enumerate(zip(want, minus, const)):
                for i in range(4):
                    assert w[i].tobytes() == a[i].tobytes() == b[i].tobytes(), (gh, k, i)
    finally:
        s.close()


def test_raised_map_shifts_z_by_the_rise():
    """A ramp stream replayed with the map on the ramp and on the ramp raised by 0.25 m (the reset raised with it): the five z components of x move by
    the rise, everything else stays (1e-12)"""
    ter = dict(tiles=TR.ramp(10.0)[None], cell=TR.CELL, tile=np.zeros(NL, dtype=np.int32), origin=TR.centred_origin(np.zeros((NL, 2))))
    s = _solver(); rise = 0.25
    try:
        _, rec = _record(s, duration=0.2, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), terrain=ter, state_estimator=True, sensor_noise="reference",
                         attitude_filter=True, ground_map=True)
        base = rec[0][5]["x"][:, 0:3]
        s.sim_set_terrain(np.concatenate([ter["tiles"], ter["tiles"] + rise]), TR.CELL)
        s.state_est_set_ground(0, ter["origin"]); a = _replay(s, base, rec)
        s.state_est_set_ground(1, ter["origin"]); b = _replay(s, base + [0, 0, rise], rec)
    finally:
        s.close()
    z = np.zeros(18, dtype=bool); z[[2, 8, 11, 14, 17]] = True; worst = 0.0
    for (xa, pa, _, sa), (xb, pb, _, sb) in zip(a, b):
        d = xb - xa
        worst = max(worst, np.max(np.abs(d[:, z] - rise)), np.max(np.abs(d[:, ~z])))
        np.testing.assert_allclose(pb, pa, rtol=1e-9, atol=1e-18)
        assert np.array_equal(sa, sb)
    print("raised map on the device: worst deviation from the pure shift %.1e m" % worst)
    assert worst < 1e-12


def test_map_kernel_equals_the_twin():
    """0.3 s trot on a mixed library (10 deg ramp, 6 cm stairs, 1 cm rough, the plane) with the reference sensor noise, the attitude filter and a perfect
    map: every call's x and diag P per robot at 1e-10 relative, rbd_est at 1e-9, status bits identical"""
    import _ground_est_twin as G
    from _sim_twin_terrain import robot_terrain
    ter = _mixed(); s = _solver()
    try:
        _, rec = _record(s, duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), terrain=ter, state_estimator=True, sensor_noise="reference",
                         attitude_filter=True, ground_map=True)
        params = s.state_est_get_params(); gh = s.sim_get_params()["ground_height"]
    finally:
        s.close()
    assert len(rec) == 301
    twins = [G.GroundEstTwin(params, robot_terrain(ter, b), gh) for b in range(NL)]
    states = [twins[b].reset(rec[0][5]["x"][b, 0:3]) for b in range(NL)]
    worst = np.zeros(3)
    for k, (dt, sens, contact, rbd_est, status, got) in enumerate(rec):
        for b in range(NL):
            rbd, code = twins[b].step(states[b], dt, sens[b], int(contact[b]))
            assert code == status[b], (k, b, code, status[b])
            x, pd = states[b]["x"], np.diag(states[b]["P"])
            ex = np.max(np.abs(got["x"][b] - x)) / max(np.max(np.abs(x)), 1e-2); ep = np.max(np.abs(got["p_diag"][b] - pd)) / np.max(np.abs(pd))
            d = rbd_est[b] - rbd; d[0:3] = _wrap(d[0:3])
            if rbd[54] * rbd_est[b, 54] < 0:
                d[51:55] = rbd_est[b, 51:55] + rbd[51:55]
            er = np.max(np.abs(d))
            worst = np.maximum(worst, [ex, ep, er])
            assert ex < 1e-10 and ep < 1e-10 and er < 1e-9, (k, b, ex, ep, er)
    print("map kernel vs twin over 301 calls x %d robots: x %.1e, diag P %.1e (worst relative), rbd_est %.1e" % (NL, *worst))


def _loop(ter, **kw):
    """closed_loop.run of a 1 s trot at 0.3 m/s on ter with an error watch on |z_hat - z| and |v_hat - v| (per-robot maxima over every estimator call)"""
    import torch
    from qm_control_b200 import closed_loop
    s = _solver(); box = {}
    orig_sim, orig_est = s.sim_step_dev, s.state_est_step_dev

    def sim(duration, effort, q, v, rbd, contact, status, stream=None, wrench=None):
        box["rbd"] = rbd; orig_sim(duration, effort, q, v, rbd, contact, status, stream, wrench=wrench)

    def est(dt, sensors, contact, rbd_est, status, stream=None):
        orig_est(dt, sensors, contact, rbd_est, status, stream)
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            e = torch.stack([(rbd_est[:, 5] - box["rbd"][:, 5]).abs(), (rbd_est[:, 27:30] - box["rbd"][:, 27:30]).norm(dim=1)], 1)
            box["max"] = e if "max" not in box else torch.maximum(box["max"], e)
    if kw.get("state_estimator"):
        s.sim_step_dev, s.state_est_step_dev = sim, est
    try:
        r = closed_loop.run(s, duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), terrain=ter, **kw)
        assert s.state_est_get_ground() is None and s.sim_get_terrain() is None   # restored
        if "max" in box:
            torch.cuda.synchronize(); r["watch"] = box["max"].cpu().numpy()
        return r
    finally:
        s.close()


def test_closed_loop_on_terrain_with_the_map():
    """64 robots, 1 s trot at 0.3 m/s over flat ground, a 10 deg ramp, 3 cm stairs and 1 cm rough ground (from 0.2 m ahead of the start), reference
    sensor noise, attitude filter, perfect map: no robot falls that stays up on the true state, |z_hat - z| and |v_hat - v| stay bounded; with an
    all -1 map the ramp robots' |z_hat - z| grows to the order of the ground's rise under their feet"""
    tiles = np.stack([TR.ramp(10.0, start=0.2), TR.stairs(0.03, 0.3, start=0.2), TR.rough(0.01, seed=7, flat_radius=0.2)])
    tile = (np.arange(NL) % 4 - 1).astype(np.int32); ter = dict(tiles=tiles, cell=TR.CELL, tile=tile, origin=TR.centred_origin(np.zeros((NL, 2))))
    est = dict(state_estimator=True, sensor_noise="reference", attitude_filter=True)
    truth = _loop(ter)
    mapped = _loop(ter, ground_map=True, **est)
    blind = _loop(ter, ground_map=dict(tile=np.full(NL, -1, dtype=np.int32), origin=ter["origin"]), **est)
    up_t, up_m = _upright(truth, ter), _upright(mapped, ter)
    names = ["flat", "ramp 10 deg", "stairs 3 cm", "rough 1 cm"]; ramp = tile == 0
    ahead = mapped["base"][-1, :, :2] + [0.3, 0.0]   # about where the front feet stand at the end
    rise = TR.height(tiles, TR.CELL, tile, ter["origin"], ahead)
    for t in range(-1, 3):
        sel = tile == t
        print("%-12s up on the truth %2d/%2d, on the mapped estimate %2d/%2d; |z_hat - z| max p50 / max %.2e / %.2e m, |v_hat - v| max p50 / max %.3f / %.3f m/s;"
              " all -1 map: |z_hat - z| max p50 %.2e m, |v_hat - v| max p50 %.3f m/s; ground 0.3 m ahead of the base at the end p50 %.3f m" % (
                  names[t + 1], up_t[sel].sum(), sel.sum(), up_m[sel].sum(), sel.sum(), np.median(mapped["watch"][sel, 0]), mapped["watch"][sel, 0].max(),
                  np.median(mapped["watch"][sel, 1]), mapped["watch"][sel, 1].max(), np.median(blind["watch"][sel, 0]), np.median(blind["watch"][sel, 1]),
                  np.median(rise[sel])))
    assert np.all(up_m[up_t]), np.nonzero(up_t & ~up_m)
    for t, (zb, vb) in BOUNDS.items():
        sel = up_t & (tile == t)
        assert mapped["watch"][sel, 0].max() < zb and mapped["watch"][sel, 1].max() < vb, (names[t + 1], mapped["watch"][sel].max(axis=0))
    # without the map the ramp's rise shows in z_hat: centimetres, a sizeable share of the rise under the front feet (measured 22 mm against 48 mm),
    # where the mapped estimate stays within millimetres
    assert np.median(blind["watch"][ramp, 0]) > max(0.01, 0.3 * np.median(rise[ramp]), 10.0 * np.median(mapped["watch"][ramp, 0]))


# per tile (-1: flat) the bounds on max |z_hat - z| (m) and max |v_hat - v| (m/s) over the run: about twice the worst robot of the first measurement on an
# H100 80GB HBM3 (flat 1.0 mm / 0.040 m/s, ramp 1.8 mm / 0.051, stairs 0.6 mm / 0.044, rough 12.6 mm / 0.686, DESIGN.md §8)
BOUNDS = {-1: (0.004, 0.1), 0: (0.004, 0.1), 1: (0.004, 0.1), 2: (0.025, 1.2)}


def test_closed_loop_ground_map_needs_the_estimator_and_terrain():
    from qm_control_b200 import closed_loop
    s = _solver(batch=4)
    try:
        ter = dict(tiles=TR.ramp(5.0, start=0.35)[None], cell=TR.CELL, tile=np.zeros(4, dtype=np.int32), origin=TR.centred_origin(np.zeros((4, 2))))
        with pytest.raises(ValueError, match="ground_map"):
            closed_loop.run(s, duration=0.01, state_estimator=True, terrain=ter)
        for kw in (dict(ground_map=True), dict(ground_map=True, terrain=ter), dict(ground_map=True, state_estimator=True), dict(state_estimator=True, terrain=ter, ground_map="yes")):
            with pytest.raises(ValueError, match="ground_map"):
                closed_loop.run(s, duration=0.01, **kw)
        assert s.state_est_get_ground() is None and s.sim_get_terrain() is None
    finally:
        s.close()
