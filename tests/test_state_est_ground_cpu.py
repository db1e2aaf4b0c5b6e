"""The state estimator's ground map on the host, no GPU (tests/_ground_est_twin.py): the foot-height row's Jacobian against central differences, the
plant's contact law against the row's measured value at standing states on a ramp and on rough ground, two identities of the map rows, and the
gradient columns at work on a ramp."""
import numpy as np
import pytest

import _ground_est_twin as G
import _state_est_twin as T
from _sim_twin_terrain import SimTwinTerrain
from qm_control_b200 import terrain as TR

CELL = 0.02
SIZE = 2.0


@pytest.fixture(scope="module")
def twin():
    return SimTwinTerrain()


def _map(tile, tiles=None):
    """one robot's map with the tile's centre node at the world origin"""
    return dict(tiles=tile[None] if tiles is None else tiles, cell=CELL, tile=0, origin=TR.centred_origin(np.zeros(2), SIZE, CELL))


def _standing(oracle, twin, ter):
    """qmb200_sim_standing_state on one robot's terrain restated with the oracle's feet and the terrain twin's ground: the base tilted onto the plane
    fitted through the ground under the feet (8 fixed-point rounds), the deepest foot at the static penetration"""
    mi = oracle.model_info(); p = twin.params; q = mi["q_nominal"].copy(); q[2:6] = 0.0
    delta0 = mi["mass"] * 9.81 / (4.0 * p["stiffness"])
    for _ in range(8):
        pf = oracle.rbd(q, np.zeros(24))["foot_pos"]
        H = np.array([twin.ground(ter, *pf[f, :2])[0] for f in range(4)])
        bx, by = np.linalg.lstsq(pf[:, :2] - pf[:, :2].mean(0), H - H.mean(), rcond=None)[0]
        n = np.array([-bx, -by, 1.0]) / np.sqrt(1.0 + bx * bx + by * by)
        q[4] = np.arctan2(n[0], n[2]); q[5] = np.arcsin(-n[1])   # yaw 0: base z = (s_p c_r, -s_r, c_p c_r)
    pf = oracle.rbd(q, np.zeros(24))["foot_pos"]; z = -np.inf
    for f in range(4):
        H, gx, gy = twin.ground(ter, *pf[f, :2])
        z = max(z, H - pf[f, 2] + (p["foot_radius"] - delta0) * np.sqrt(1.0 + gx * gx + gy * gy))
    q[2] = z
    return q, delta0


def _stance(oracle, twin, ter, ms):
    """the terrain twin from its standing state with the joints held by a PD law, 1 ms steps → (q0, delta0, [(q, v, v_prev, contact)])"""
    q, delta0 = _standing(oracle, twin, ter); q0 = q.copy(); v = np.zeros(24); qn = q[6:].copy()
    kp = np.r_[np.full(12, 300.0), np.full(6, 20.0)]; kd = np.r_[np.full(12, 6.0), np.full(6, 0.3)]
    out = []
    for _ in range(ms):
        q1, v1, _, c, st = twin.step_ext(1e-3, kp * (qn - q[6:]) - kd * v[6:], q, v, terrain=ter)
        assert st == 0
        out.append((q1, v1, v, c)); q, v = q1, v1
    return q0, delta0, out


def _replay(f, base_pos, stream):
    """the filter f from base_pos over a stream of plant steps, noise-free readings → the state dict after every call"""
    s = f.reset(base_pos); out = []
    for k, (q, v, v_prev, c) in enumerate(stream):
        _, code = f.step(s, 1e-3, T.read_sensors(q, v, v_prev, 1e-3, k, 0, T.NOISE_OFF), c)
        assert code == 0, k
        out.append(dict(x=s["x"].copy(), P=s["P"].copy()))
    return out


@pytest.mark.parametrize("kind", ["ramp", "rough", "step edge"])
def test_row_jacobian_is_minus_the_gradient(oracle, kind):
    """h_f(x) = p_f,z - H(p_f,x, p_f,y): central differences over the foot's xyz equal [-gx, -gy, 1] of the twin's lookup, at points strictly inside
    cells (the bilinear gradient is continuous there)"""
    tile = {"ramp": TR.ramp(10.0, 30.0, size=SIZE, cell=CELL), "rough": TR.rough(0.02, seed=5, size=SIZE, cell=CELL),
            "step edge": TR.stairs(0.06, 0.3, start=0.1, size=SIZE, cell=CELL)}[kind]
    f = G.GroundEstTwin(T.default_params(oracle.model_info()["mass"]), _map(tile), oracle=oracle)
    rng = np.random.default_rng(2); eps = 1e-7
    pts = [np.r_[(np.floor(rng.uniform(-0.5, 0.5, 2) / CELL) + rng.uniform(0.1, 0.9, 2)) * CELL, 0.02] for _ in range(60)]
    if kind == "step edge":   # the two cells around the node 0.1 m ahead of the centre, one of which is the one-cell-wide edge
        pts = [np.r_[0.08 + (k % 2 + rng.uniform(0.1, 0.9)) * CELL, rng.uniform(-0.3, 0.3), 0.02] for k in range(60)]
    h = lambda p: p[2] - f.ground(p[0], p[1])[0]
    steep = 0.0
    for p in pts:
        _, gx, gy = f.ground(p[0], p[1])
        d = np.array([(h(p + eps * e) - h(p - eps * e)) / (2 * eps) for e in np.eye(3)])
        np.testing.assert_allclose(d, [-gx, -gy, 1.0], rtol=0, atol=1e-7 * max(1.0, abs(gx), abs(gy)))
        C, _ = f.rows(np.r_[np.zeros(6), np.tile(p, 4)])
        assert np.array_equal(C[24, 6:9], [-gx, -gy, 1.0])
        steep = max(steep, np.hypot(gx, gy))
    assert steep > {"ramp": 0.17, "rough": 0.05, "step edge": 2.9}[kind]   # the cells sampled do slope (a 6 cm rise over a 2 cm cell: 3)


@pytest.mark.parametrize("kind", ["ramp", "rough"])
def test_plant_law_meets_the_row(oracle, twin, kind):
    """After 100 ms standing on a 12 deg ramp and on 1 cm rough ground, held by a PD law on the joints: per foot p_z - H = s c to within twice the
    static penetration m g / (4 k), the spread the loads of the four feet can give it; the plane's row misses by centimetres"""
    tile = TR.ramp(12.0, size=SIZE, cell=CELL) if kind == "ramp" else TR.rough(0.01, seed=3, size=SIZE, cell=CELL)
    ter = _map(tile); fh = T.default_params(oracle.model_info()["mass"])["foot_height"]
    _, delta0, stream = _stance(oracle, twin, ter, 100)
    q, v, _, c = stream[-1]
    assert c == 15
    pf = oracle.rbd(q, v)["foot_pos"]
    res = G.height_residual(pf, ter, fh); plane = pf[:, 2] - fh
    print("%s: map row residual %s m (static penetration %.1e m), plane row residual %s m" % (kind, np.array2string(res, precision=6), delta0, np.array2string(plane, precision=4)))
    assert np.max(np.abs(res)) < 2.0 * delta0 * 1.03
    assert np.max(np.abs(plane)) > 0.01


@pytest.fixture(scope="module")
def ramp_stream(oracle, twin):
    ter = _map(TR.ramp(10.0, size=SIZE, cell=CELL))
    q0, _, stream = _stance(oracle, twin, ter, 150)
    return ter, q0, stream


def test_constant_tile_at_ground_height_is_the_plane_twin(oracle, ramp_stream):
    """A map of tile -1 or of a constant tile at ground_height gives the plane twin's x and P exactly, call by call, on a stream whose legs move"""
    _, q0, stream = ramp_stream
    prm = T.default_params(oracle.model_info()["mass"])
    want = _replay(T.StateEstTwin(prm, oracle), q0[0:3], stream[:60])
    for ter in (_map(TR.flat(SIZE, CELL)), dict(_map(TR.flat(SIZE, CELL)), tile=-1)):
        got = _replay(G.GroundEstTwin(prm, ter, oracle=oracle), q0[0:3], stream[:60])
        for a, b in zip(got, want):
            assert np.array_equal(a["x"], b["x"]) and np.array_equal(a["P"], b["P"])


def test_raised_map_shifts_z_by_the_rise(oracle, ramp_stream):
    """The map and the reset raised by 0.25 m: p_z and the four foot z of x move by exactly that (1e-12), every other component of x and all of P stay"""
    ter, q0, stream = ramp_stream
    prm = T.default_params(oracle.model_info()["mass"]); rise = 0.25
    a = _replay(G.GroundEstTwin(prm, ter, oracle=oracle), q0[0:3], stream)
    b = _replay(G.GroundEstTwin(prm, dict(ter, tiles=ter["tiles"] + rise), oracle=oracle), q0[0:3] + [0, 0, rise], stream)
    z = np.zeros(18, dtype=bool); z[[2, 8, 11, 14, 17]] = True
    worst = 0.0
    for u, w in zip(a, b):
        d = w["x"] - u["x"]
        worst = max(worst, np.max(np.abs(d[z] - rise)), np.max(np.abs(d[~z])))
        np.testing.assert_allclose(w["P"], u["P"], rtol=1e-9, atol=1e-18)
    print("raised map: worst deviation from the pure shift %.1e m" % worst)
    assert worst < 1e-12


class _ZOnlyTwin(G.GroundEstTwin):
    """the map's measured values with the plane's C: a height row without the gradient columns"""

    def rows(self, x):
        return self.C.copy(), super().rows(x)[1]


def test_gradient_columns_correct_x_on_a_ramp(oracle, twin, ramp_stream):
    """A 3 cm start error in x under 150 ms of a stance stream of the terrain twin.  On a 10 deg ramp along x the height rows see only the error's
    component along the ramp's normal: the filter removes it (the base error ends within 0.3 mm of the slope), and the -gx columns let it do so partly
    in x, by about 30 mm sin^2(10 deg) = 0.9 mm, where a z-only row moves z alone.  The part along the slope is not observable from foot heights and
    stays, as the whole error does on a flat tile."""
    ter, q0, stream = ramp_stream
    prm = T.default_params(oracle.model_info()["mass"]); err = np.array([0.03, 0.0, 0.0]); th = np.radians(10.0)
    flat = _map(TR.flat(SIZE, CELL)); fq0, _, fstream = _stance(oracle, twin, flat, len(stream))
    end = {}
    for tag, cls, t, s0, st in (("ramp", G.GroundEstTwin, ter, q0, stream), ("ramp, z-only row", _ZOnlyTwin, ter, q0, stream),
                                ("flat", G.GroundEstTwin, flat, fq0, fstream)):
        out = _replay(cls(prm, t, oracle=oracle), s0[0:3] + err, st)
        end[tag] = out[-1]["x"][0:3] - st[-1][0][0:3]
        print("%s: base error after %d ms (x, y, z) %s mm (start 30 mm in x)" % (tag, len(stream), np.array2string(end[tag] * 1e3, precision=2)))
    normal = np.array([-np.sin(th), 0.0, np.cos(th)])
    assert abs(end["flat"][0] - 0.03) < 1e-3 and abs(end["flat"][2]) < 1e-4
    assert abs(end["ramp"] @ normal) < 3e-4
    assert end["ramp, z-only row"][0] - end["ramp"][0] > 0.6e-3   # measured 0.87 mm
