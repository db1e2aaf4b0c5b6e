"""Heightfield terrain under the feet on the device (qmb200_sim_set_terrain, qmb200_sim_set_robot_terrain, the terrain-aware standing state and
closed_loop.run(terrain=...)) against the CPU terrain twin (tests/sim_twin_terrain.cpp), bit-identity of neutral terrain, invariances, known answers
of sliding and sticking on a ramp, and the closed loop on a ramp on an H100."""
import ctypes as C

import numpy as np
import pytest

import _loop_replay as R
from _oracle import Oracle
from _parity import PLANT_TOL, Q_BLOCKS, RBD_BLOCKS, block_errors
from _sim_twin import DEFAULTS
from _sim_twin_terrain import SimTwinTerrain
from qm_control_b200 import terrain as T
from test_sim_variation_gpu import _states, _variation

pytestmark = pytest.mark.gpu

B = 256                  # the state groups of test_sim_gpu.py / test_sim_variation_gpu.py
SIZE, CELL = 4.0, 0.02


@pytest.fixture(scope="module")
def solver():
    import qm_control_b200 as q
    s = q.Solver(batch=B, device=0)
    yield s
    s.close()


@pytest.fixture(scope="module")
def twin():
    return SimTwinTerrain()


def _clear(s):
    s.sim_set_terrain(None)
    assert s.sim_get_terrain() is None and s.sim_get_robot_terrain() is None


def _front_foot_x(oracle):
    mi = oracle.model_info(); q = mi["q_nominal"].copy()
    return float(oracle.rbd(q, np.zeros(24))["foot_pos"][0, 0] - q[0])


def _library(oracle):
    """10 deg ramp along x; 15 deg ramp along the diagonal; a 5 cm step edge under the front feet; rough ground with sigma 2 cm"""
    return np.stack([T.ramp(10.0), T.ramp(15.0, 45.0), T.stairs(0.05, 10.0, start=_front_foot_x(oracle) - 0.005), T.rough(0.02, seed=9)])


def _on_terrain(solver, oracle, twin, tiles, tile, seed=5):
    """the perturbed state groups moved onto each robot's ground: the offsets of test_sim_variation_gpu's states (all but the lifted group 1 mm lower)
    from the flat standing state, applied to the terrain standing state of robot b (tile[b], its tile centred under its base)"""
    q, v, eff = _states(oracle, twin); q[32:, 2] -= 0.001   # all groups but the lifted one 1 mm lower: most robots touch their ground
    flat, _ = solver.sim_standing_state(np.c_[q[:, :2], q[:, 3]])
    origin = T.centred_origin(q[:, :2])
    solver.sim_set_terrain(tiles, CELL); solver.sim_set_robot_terrain(tile, origin)
    on, _ = solver.sim_standing_state(np.c_[q[:, :2], q[:, 3]])
    q[:, 2] += on[:, 2] - flat[:, 2]; q[:, 4:6] += on[:, 4:6]
    return q, v, eff, dict(tiles=tiles, cell=CELL, tile=np.asarray(tile), origin=origin)


def _compare(got, ref, tag):
    qg, vg, rg, cg, sg = got; qt, vt, rt, ct, st = ref
    assert np.all(sg == 0) and np.all(st == 0), tag
    np.testing.assert_array_equal(cg, ct, err_msg=tag)
    worst = {}
    for name, a, b, blocks in (("q", qg, qt, Q_BLOCKS), ("v", vg, vt, Q_BLOCKS), ("rbd", rg, rt, RBD_BLOCKS)):
        err = block_errors(a, b, blocks); worst[name] = max(err.values())
        assert worst[name] < PLANT_TOL, (tag, name, err)
    return worst


# ---------------- 1. set / get ----------------
def test_terrain_round_trip_and_validation(solver, oracle):
    from qm_control_b200 import QmbError
    lib = solver.lib; h = solver.h
    _clear(solver)
    tiles = _library(oracle); tile = np.arange(B) % 5 - 1; origin = np.random.default_rng(1).uniform(-3, 3, (B, 2))
    try:
        solver.sim_set_terrain(tiles, CELL); solver.sim_set_robot_terrain(tile, origin)
        got = solver.sim_get_terrain(); np.testing.assert_array_equal(got["tiles"], tiles); assert got["cell"] == CELL
        rt = solver.sim_get_robot_terrain(); np.testing.assert_array_equal(rt["tile"], tile); np.testing.assert_array_equal(rt["origin"], origin)

        def unchanged():
            g = solver.sim_get_terrain(); np.testing.assert_array_equal(g["tiles"], tiles); assert g["cell"] == CELL
            r = solver.sim_get_robot_terrain(); np.testing.assert_array_equal(r["tile"], tile); np.testing.assert_array_equal(r["origin"], origin)
        small = tiles[:2]
        bad_lib = [(tiles, 0.0), (tiles, -0.1), (tiles, np.nan), (tiles, np.inf), (np.where(np.arange(tiles.size).reshape(tiles.shape) == 77, np.nan, tiles), CELL),
                   (np.where(np.arange(tiles.size).reshape(tiles.shape) == 5, np.inf, tiles), CELL), (tiles[:, :1, :], CELL), (tiles[:, :, :1], CELL),
                   (small, CELL)]                                                   # fewer tiles than robot 4 references
        for t, c in bad_lib:
            with pytest.raises(QmbError):
                solver.sim_set_terrain(t, c)
            unchanged()
        one = np.zeros(4)
        for args in ((0, 2, 2, CELL), (-1, 2, 2, CELL), (1 << 30, 1 << 16, 1 << 16, CELL), (1 << 30, 1 << 30, 1 << 30, CELL)):   # n_tiles < 1; byte count overflows
            assert lib.qmb200_sim_set_terrain(h, *args, one.ctypes.data_as(C.c_void_p)) != 0, args
            unchanged()
        for bt, bo in ((np.where(np.arange(B) == 3, 4, tile), origin), (np.where(np.arange(B) == 3, -2, tile), origin),
                       (tile, np.where(np.arange(2 * B).reshape(B, 2) == 9, np.nan, origin)), (tile, np.where(np.arange(2 * B).reshape(B, 2) == 8, -np.inf, origin))):
            with pytest.raises(QmbError):
                solver.sim_set_robot_terrain(bt, bo)
            unchanged()
        assert lib.qmb200_sim_set_robot_terrain(h, tile.astype(np.int32).ctypes.data_as(C.c_void_p), None) != 0; unchanged()   # null origin
        # a library with more tiles is accepted with the robots on it; clearing the library clears the robots' terrain
        solver.sim_set_terrain(np.concatenate([tiles, tiles[:1]]), CELL); solver.sim_set_robot_terrain(np.full(B, 4), origin)
        assert solver.sim_get_robot_terrain()["tile"][0] == 4
        solver.sim_set_terrain(None)
        assert solver.sim_get_terrain() is None and solver.sim_get_robot_terrain() is None
        with pytest.raises(QmbError):   # no library: only tile -1
            solver.sim_set_robot_terrain(np.zeros(B), origin)
        solver.sim_set_robot_terrain(-1, origin); assert np.all(solver.sim_get_robot_terrain()["tile"] == -1)
        solver.sim_set_robot_terrain(None); assert solver.sim_get_robot_terrain() is None
    finally:
        _clear(solver)


# ---------------- 2. neutral terrain ----------------
def test_neutral_terrain_is_bit_identical(solver, oracle, twin):
    q, v, eff = _states(oracle, twin)
    plain = solver.sim_step(1e-3, eff, q, v)
    try:
        solver.sim_set_terrain(_library(oracle), CELL); solver.sim_set_robot_terrain(-1, np.random.default_rng(2).uniform(-2, 2, (B, 2)))
        minus1 = solver.sim_step(1e-3, eff, q, v)
        solver.sim_set_robot_terrain(None); lib_only = solver.sim_step(1e-3, eff, q, v)
    finally:
        _clear(solver)
    for a, b, c in zip(plain, minus1, lib_only):
        np.testing.assert_array_equal(a, b); np.testing.assert_array_equal(a, c)


@pytest.mark.parametrize("g", [0.0, 0.05])
def test_constant_tile_is_the_plane(solver, oracle, twin, g):
    q, v, eff = _states(oracle, twin); q[:, 2] += g
    try:
        solver.sim_set_params(ground_height=g); plane = solver.sim_step(1e-3, eff, q, v)
        solver.sim_set_params(ground_height=0.0)
        tiles = np.full((2,) + T.flat().shape, g); tiles[1] += 0.3   # a second tile nobody stands on
        solver.sim_set_terrain(tiles, CELL); solver.sim_set_robot_terrain(0, T.centred_origin(q[:, :2]) + np.random.default_rng(3).uniform(-3, 3, (B, 2)))
        tile = solver.sim_step(1e-3, eff, q, v)
    finally:
        solver.sim_set_params(ground_height=DEFAULTS["ground_height"]); _clear(solver)
    assert np.count_nonzero(plane[3]) >= 32
    for a, b in zip(plane, tile):
        np.testing.assert_array_equal(a, b)


# ---------------- 3. against the twin ----------------
@pytest.mark.parametrize("varied", [False, True])
def test_step_on_terrain_matches_the_twin(solver, oracle, twin, varied):
    tiles = _library(oracle); tile = np.arange(B) % 4
    try:
        q, v, eff, ter = _on_terrain(solver, oracle, twin, tiles, tile)
        mu, pl, wr = (_variation("mu")[0], _variation("payload")[1], _variation("wrench")[2]) if varied else (None, None, None)
        solver.sim_set_robot_params(friction_mu=mu, payload=pl)
        got = solver.sim_step(1e-3, eff, q, v, wrench=wr)
        solver.sim_set_robot_params(); solver.sim_set_robot_terrain(None)
        flat = solver.sim_step(1e-3, eff, q, v)   # the terrain changes the step
    finally:
        solver.sim_set_robot_params(); _clear(solver)
    ref = twin.step_batch_ext(1e-3, eff, q, v, mu=mu, payload=pl, wrench=wr, terrain=ter)
    touching = [np.count_nonzero(got[3][tile == t]) for t in range(4)]
    for t in range(4):
        rows = tile == t
        w = _compare(tuple(a[rows] for a in got), tuple(a[rows] for a in ref), "tile %d varied %s" % (t, varied))
        print("tile %d%s: %d robots in contact, worst per-block rel err q %.1e v %.1e rbd %.1e" % (t, " + mu, payload, wrench" if varied else "", np.count_nonzero(got[3][rows]),
                                                                                              w["q"], w["v"], w["rbd"]))
    assert min(touching) > 0 and sum(touching) >= 32, touching
    assert np.max(np.abs(flat[1] - got[1])) > 1e-3


# ---------------- 4. batch position ----------------
def test_batch_order_with_mixed_tiles(solver, oracle, twin):
    tiles = _library(oracle); tile = np.arange(B) % 5 - 1; perm = np.random.default_rng(7).permutation(B)
    try:
        q, v, eff, ter = _on_terrain(solver, oracle, twin, tiles, tile)
        origin = ter["origin"] + np.random.default_rng(8).uniform(-0.01, 0.01, (B, 2))
        solver.sim_set_robot_terrain(tile, origin); a = solver.sim_step(1e-3, eff, q, v)
        solver.sim_set_robot_terrain(tile[perm], origin[perm]); b = solver.sim_step(1e-3, eff[perm], q[perm], v[perm])
    finally:
        _clear(solver)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x[perm], y)


# ---------------- 5. rotation ----------------
KP = np.r_[[2000.0] * 12, [200.0] * 6]; KD = np.r_[[20.0] * 12, [2.0] * 6]   # PD hold of defaultJointState (leg / arm joints)


def _pd_run(s, q, v, n_ms):
    """hold the joints at defaultJointState by hw_write PD (zero delay) for n_ms plant steps of 1 ms → q, v, rbd, contact after each step"""
    Bn = len(q); jc = np.zeros((Bn, 18, 5)); jc[:, :, 0] = s.default_joint_state; jc[:, :, 2] = KP; jc[:, :, 3] = KD
    s.hw_set_delay(0.0); out = []
    for k in range(n_ms):
        eff, st = s.hw_write(np.full(Bn, (k + 1) * 1e-3), np.full(Bn, 1e-3), jc, q[:, 6:], v[:, 6:])
        assert np.all(st == 0)
        q, v, rbd, c, sst = s.sim_step(1e-3, eff, q, v)
        assert np.all(sst == 0), k
        out.append((q, v, rbd, c))
    return out


def _rotate_back(q, v, rbd, centre, psi):
    """state of a robot rotated by yaw psi about the vertical through `centre`, mapped back into the unrotated frame"""
    c, s = np.cos(-psi), np.sin(-psi); Rz = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    q = q.copy(); v = v.copy(); rbd = rbd.copy()
    q[:3] = Rz @ (q[:3] - centre); v[:3] = Rz @ v[:3]; q[3] -= psi
    rbd[3:6] = q[:3]; rbd[0] -= psi; rbd[24:27] = Rz @ rbd[24:27]; rbd[27:30] = Rz @ rbd[27:30]; rbd[48:51] = Rz @ (rbd[48:51] - centre)
    x, y, z, w = rbd[51:55]; hz = np.array([0.0, 0.0, np.sin(-psi / 2), np.cos(-psi / 2)])   # q_z(-psi) (x) q
    rbd[51:55] = [hz[3] * x - hz[2] * y, hz[3] * y + hz[2] * x, hz[3] * z + hz[2] * w, hz[3] * w - hz[2] * z]
    if rbd[54] < 0:
        rbd[51:55] *= -1
    return q, v, rbd


def _rotation_errors(on_ramp, n_ms):
    """a robot at yaw 0 and its copy rotated by pi/2 about the vertical through its tile's centre, PD-held for n_ms: on_ramp, the first on a 10 deg
    ramp along x and the copy on the same ramp along y; else both on the plane → per-block relative error in the rotated frame after each 1 ms step"""
    import qm_control_b200 as qm
    s = qm.Solver(batch=2, device=0)
    try:
        rx = T.ramp(10.0); tiles = np.stack([rx, rx.T])                       # rx.T: the ramp along y, node for node
        centre = np.array([[1.0, -2.0, 0.0], [-3.0, 0.5, 0.0]]); psi = np.pi / 2
        s.sim_set_terrain(tiles, CELL); s.sim_set_robot_terrain([0, 1] if on_ramp else [-1, -1], T.centred_origin(centre[:, :2]))
        q, v = s.sim_standing_state(np.c_[centre[:, :2], [0.0, psi]])
        assert abs(q[1, 4] - q[0, 4]) < 1e-12 and abs(q[1, 5] - q[0, 5]) < 1e-12 and abs(q[1, 2] - q[0, 2]) < 1e-12
        v[0, :3] = [0.05, 0.02, -0.1]; c, sn = np.cos(psi), np.sin(psi); v[1, :3] = [c * 0.05 - sn * 0.02, sn * 0.05 + c * 0.02, -0.1]
        v[:, 6:] = np.random.default_rng(4).uniform(-0.2, 0.2, 18)
        runs = _pd_run(s, q, v, n_ms)
    finally:
        s.close()
    errs = []
    for k, (qk, vk, rk, ck) in enumerate(runs):
        a = (qk[0].copy(), vk[0].copy(), rk[0].copy()); a[0][:3] -= centre[0]; a[2][3:6] = a[0][:3]; a[2][48:51] -= centre[0]
        if a[2][54] < 0:
            a[2][51:55] *= -1
        b = _rotate_back(qk[1], vk[1], rk[1], centre[1], psi)
        errs.append(max(max(block_errors(x, y, bl).values()) for x, y, bl in zip(a, b, (Q_BLOCKS, Q_BLOCKS, RBD_BLOCKS))))
        assert ck[0] == ck[1], k
    return np.array(errs)


def test_rotation_invariance_after_one_step():
    """a ramp along x under a robot at yaw 0 and the same ramp along y under a robot at yaw pi/2 agree in the rotated frame after one 1 ms step"""
    ramp = _rotation_errors(True, 100); plane = _rotation_errors(False, 100)
    at = lambda e: " / ".join("%.1e" % e[k - 1] for k in (1, 10, 30, 50, 60, 70, 80, 100))
    print("rotation invariance, per-block rel err after 1 / 10 / 30 / 50 / 60 / 70 / 80 / 100 ms of PD hold: ramp %s; the plane, same robots %s" % (at(ramp), at(plane)))
    assert ramp[0] < 1e-8 and plane[0] < 1e-8


@pytest.mark.xfail(strict=True, reason="measured on H100: the rotated pair agrees to 1e-12 after 1 ms and to 6e-8 after 60 ms of PD hold on the ramp, "
                   "then the difference grows to 4e-6 at 70 ms and 1.6e-4 by 100 ms. The same pair on flat ground grows alike (8e-8 at 60 ms, 5e-6 at "
                   "70 ms, 1.2e-5 at 100 ms): round-off amplified by the held robot's dynamics, not the terrain. "
                   "test_rotation_invariance_after_one_step prints both curves.")
def test_rotation_invariance_over_100_ms_within_1e_6():
    assert np.max(_rotation_errors(True, 100)) < 1e-6


# ---------------- 6. slide and stick ----------------
@pytest.mark.parametrize("mu", [0.1, 0.6])
def test_slide_and_stick_on_a_15_degree_ramp(mu):
    import qm_control_b200 as qm
    s = qm.Solver(batch=1, device=0)
    try:
        th = np.radians(15.0); m = s.robot_mass
        s.sim_set_params(friction_mu=mu); s.sim_set_terrain(T.ramp(15.0)[None], CELL); s.sim_set_robot_terrain([0], T.centred_origin(np.zeros((1, 2))))
        q, v = s.sim_standing_state(np.zeros((1, 3)))
        n_ms = 400 if mu < 0.3 else 1000
        runs = _pd_run(s, q, v, n_ms)
        down = np.array([-np.cos(th), 0.0, -np.sin(th)])
        vd = np.array([r[1][0, :3] @ down for r in runs]); t = np.arange(1, n_ms + 1) * 1e-3
        if mu < 0.3:
            w = (t > 0.1) & (t <= 0.4); acc = np.polyfit(t[w], vd[w], 1)[0]; want = 9.81 * (np.sin(th) - mu * np.cos(th))
            print("slide, mu %.1f: downhill acceleration over 0.1-0.4 s %.4f m/s^2, g (sin - mu cos) %.4f" % (mu, acc, want))
            assert abs(acc - want) < 0.05 * want
        else:
            creep = m * 9.81 * np.sin(th) / (4 * DEFAULTS["tangential_damping"]); w = t > 0.5
            print("stick, mu %.1f: mean downhill speed over 0.5-1 s %.4f m/s, creep m g sin / (4 gamma) %.4f" % (mu, np.mean(vd[w]), creep))
            assert np.mean(vd[w]) < 1.5 * creep and runs[-1][3][0] == 15
    finally:
        s.close()


# ---------------- 7. standing state ----------------
def test_standing_state_on_a_ramp_and_a_constant_tile(solver, oracle):
    th, phi = np.radians(12.0), np.radians(30.0)
    xy_yaw = np.c_[np.random.default_rng(6).uniform(-2, 2, (B, 2)), np.random.default_rng(7).uniform(-np.pi, np.pi, B)]
    m = oracle.model_info()["mass"]; delta0 = m * 9.81 / (4 * DEFAULTS["stiffness"]); r = DEFAULTS["foot_radius"]
    try:
        flat, _ = solver.sim_standing_state(xy_yaw)
        tiles = np.stack([T.ramp(12.0, 30.0), np.full(T.flat().shape, 0.0)])
        origin = T.centred_origin(xy_yaw[:, :2]); tile = np.arange(B) % 2
        solver.sim_set_terrain(tiles, CELL); solver.sim_set_robot_terrain(tile, origin)
        with pytest.raises(Exception):
            solver.sim_standing_state(xy_yaw[:3])            # one row per robot
        q, v = solver.sim_standing_state(xy_yaw)
    finally:
        _clear(solver)
    assert np.all(v == 0)
    n = np.array([-np.tan(th) * np.cos(phi), -np.tan(th) * np.sin(phi), 1.0]); n /= np.linalg.norm(n)
    worst = 0.0
    for b in np.nonzero(tile == 0)[0]:
        fp = oracle.rbd(q[b], np.zeros(24))["foot_pos"]
        H, gx, gy = T.height(tiles, CELL, 0, origin[b], fp[:, :2], gradient=True); s = np.sqrt(1 + gx ** 2 + gy ** 2)
        pen = (H - (fp[:, 2] - r * s)) / s
        worst = max(worst, float(np.max(np.abs(pen - delta0))))
        cy, sy = np.cos(q[b, 3]), np.sin(q[b, 3]); cp, sp, cr, sr = np.cos(q[b, 4]), np.sin(q[b, 4]), np.cos(q[b, 5]), np.sin(q[b, 5])
        zb = np.array([cy * sp * cr + sy * sr, sy * sp * cr - cy * sr, cp * cr])    # base z axis of R = Rz Ry Rx
        assert np.linalg.norm(zb - n) < 1e-9, (b, zb, n)
    print("standing on a 12 deg ramp: worst |penetration - m g / 4k| %.1e m" % worst)
    assert worst < 1e-6
    const = tile == 1
    assert np.max(np.abs(q[const] - flat[const])) < 1e-12


# ---------------- 8. NaN row ----------------
def test_nan_row_on_a_tile_is_isolated(solver, oracle, twin):
    tiles = _library(oracle); tile = np.arange(B) % 4
    try:
        q, v, eff, ter = _on_terrain(solver, oracle, twin, tiles, tile)
        good = solver.sim_step(1e-3, eff, q, v)
        qn = q.copy(); qn[37, :3] = np.nan; qn[90, 0] = np.inf
        bad = solver.sim_step(1e-3, eff, qn, v)
    finally:
        _clear(solver)
    st = bad[4]; assert st[37] & 4 and st[90] & 4
    keep = np.ones(B, bool); keep[[37, 90]] = False
    for a, b in zip(good, bad):
        np.testing.assert_array_equal(a[keep], b[keep])


# ---------------- 9. closed loop ----------------
_STANCE = {}


def _stance_on_ramp():
    """stance for 1 s on a 5 deg ramp with mu 0.6, 8 robots at yaws spread over the circle (run once per module)"""
    import qm_control_b200 as qm
    from qm_control_b200 import closed_loop
    if not _STANCE:
        n = 8; s = qm.Solver(batch=n, device=0)
        try:
            xy = np.zeros((n, 3)); xy[:, 0] = 2.0 * np.arange(n); xy[:, 2] = np.linspace(-np.pi, np.pi, n, endpoint=False)
            ter = dict(tiles=T.ramp(5.0)[None], cell=CELL, tile=np.zeros(n, dtype=np.int32), origin=T.centred_origin(xy[:, :2]))
            r = closed_loop.run(s, duration=1.0, gait="stance", xy_yaw=xy, friction_mu=0.6, terrain=ter)
            _STANCE.update(r=r, yaw=xy[:, 2], restored=s.sim_get_terrain() is None and s.sim_get_robot_terrain() is None)
        finally:
            s.close()
    r = _STANCE["r"]
    drift = np.max(np.linalg.norm(r["base"][:, :, :3] - r["start_base"][None, :, :3], axis=2), axis=0)
    return r, drift, int(np.bitwise_or.reduce(r["status"].ravel()))


def test_closed_loop_stance_on_a_5_degree_ramp():
    r, drift, st = _stance_on_ramp()
    print("stance on a 5 deg ramp, 1 s: max base drift per robot (yaw %s) %s mm, status OR %#x, contact at the end %s" % (
        np.array2string(_STANCE["yaw"], precision=2), np.array2string(drift * 1e3, precision=1), st, r["contact"]))
    assert _STANCE["restored"] and st == 0


@pytest.mark.xfail(strict=True, reason="measured on H100: no status bits and all four feet in contact at the end, but the base drifts 17-150 mm within "
                   "1 s of stance depending on the robot's yaw on the slope; the controller does not see the terrain (its base-height and attitude "
                   "targets are those of flat ground).")
def test_closed_loop_stance_on_a_5_degree_ramp_drifts_under_2cm():
    r, drift, st = _stance_on_ramp()
    assert st == 0 and np.max(drift) < 0.02 and np.all(r["contact"] == 15)


def test_closed_loop_on_a_ramp_replays_call_by_call():
    import qm_control_b200 as qm
    from qm_control_b200 import closed_loop
    n = 6; s = qm.Solver(batch=n, device=0)
    try:
        xy = np.zeros((n, 3)); xy[:, 0] = 2.0 * np.arange(n)
        tiles = np.stack([T.ramp(8.0, 0.0, start=0.3), T.ramp(6.0, 90.0)]); tile = np.arange(n) % 2
        ter = dict(tiles=tiles, cell=CELL, tile=tile, origin=T.centred_origin(xy[:, :2]))
        res, rec = R.record(s, lambda: closed_loop.run(s, duration=0.1, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, terrain=ter))
    finally:
        s.close()
    np.testing.assert_array_equal(rec.meta["terrain"]["tile"], tile); np.testing.assert_array_equal(rec.meta["terrain"]["tiles"], tiles)
    oracles = [Oracle()] * n
    tg = R.replay_targets(rec); mpc = R.replay_mpc(rec, oracles); up = R.replay_update(rec, oracles); hw = R.replay_hw_write(rec, 0.009)
    pl = R.replay_plant(rec, SimTwinTerrain())
    print("ramp closed loop replay: plant %d robot-steps, worst %s; mpc %d robot-solves; update %d; hw_write %d; targets %d" % (
        pl["replayed"], {k: "%.1e" % e for k, e in pl["worst"].items()}, mpc["replayed"], up["replayed"], hw["replayed"], tg["replayed"]))
    assert pl["replayed"] == 101 * n and hw["replayed"] == 100 * n and up["replayed"] == 50 * n and mpc["replayed"] + mpc["excused"] == 10 * n
