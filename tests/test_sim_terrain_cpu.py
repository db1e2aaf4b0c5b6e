"""Heightfield terrain of the plant on the CPU: the terrain twin (tests/sim_twin_terrain.cpp) against the plane law of tests/sim_twin_ext.cpp, the
direction of its contact force on a ramp, its ground lookup against qm_control_b200.terrain.height and finite differences, and the NaN-safe clamp of that
helper."""
import numpy as np
import pytest

import _closed_loop_cpu
from _sim_twin_ext import SimTwinExt
from _sim_twin_terrain import SimTwinTerrain
from qm_control_b200 import terrain as T

CELL = 0.05


@pytest.fixture(scope="module")
def twin():
    return SimTwinTerrain()


def _states(oracle, twin, n=48, seed=3):
    """standing states perturbed into contact, sliding, landing and lifted feet, with random efforts"""
    rng = np.random.default_rng(seed); q0, _ = _closed_loop_cpu.standing_state(oracle, twin); lim = oracle.model_info()["effort"]
    q = np.tile(q0, (n, 1)); v = np.zeros((n, 24))
    q[:, 6:] += rng.uniform(-0.01, 0.01, (n, 18)); q[:, 3] = rng.uniform(-np.pi, np.pi, n); q[:, 4:6] = rng.uniform(-0.004, 0.004, (n, 2)); q[:, :2] = rng.uniform(-0.5, 0.5, (n, 2))
    q[:, 2] += rng.uniform(-0.002, 0.001, n); v[:, 6:] = rng.uniform(-0.1, 0.1, (n, 18)); v[:, :3] = rng.uniform(-0.5, 0.5, (n, 3))
    v[n // 4:n // 2, 2] = -0.3; q[-4:, 2] += 0.05
    return q, v, rng.uniform(-0.3, 0.3, (n, 18)) * lim


@pytest.mark.parametrize("g", [0.0, 0.05])
def test_constant_tile_is_the_plane_law_bit_for_bit(oracle, twin, g):
    q, v, eff = _states(oracle, twin); q[:, 2] += g
    plane = SimTwinExt(ground_height=g)   # the plane law
    tiles = np.full((1,) + T.grid(2.0, CELL)[0].shape, g)
    origin = T.centred_origin(np.zeros(2), 2.0, CELL)
    touching = 0
    for b in range(len(q)):
        ter = dict(tiles=tiles, cell=CELL, tile=0, origin=origin)
        a = twin.step_ext(2e-3, eff[b], q[b], v[b], terrain=ter); p = plane.step_ext(2e-3, eff[b], q[b], v[b])
        for x, y in zip(a, p):
            np.testing.assert_array_equal(x, y)
        qa = twin.accel_ext(eff[b], q[b], v[b], terrain=ter); qp = plane.accel_ext(eff[b], q[b], v[b])
        for x, y in zip(qa, qp):
            np.testing.assert_array_equal(x, y)
        touching += int(qa[2] != 0)
    assert touching >= len(q) // 2


def test_force_on_a_ramp_at_rest_is_along_the_normal(oracle, twin):
    th = np.radians(10.0); tiles = T.ramp(10.0, size=2.0, cell=CELL)[None]; ter = dict(tiles=tiles, cell=CELL, tile=0, origin=T.centred_origin(np.zeros(2), 2.0, CELL))
    q, _ = _closed_loop_cpu.standing_state(oracle, twin); n = np.array([-np.sin(th), 0.0, np.cos(th)])
    for dz in (0.0, -0.01, -0.03):
        qq = q.copy(); qq[2] += dz
        _, F, mask = twin.accel_ext(np.zeros(18), qq, np.zeros(24), terrain=ter)
        on = [f for f in range(4) if mask & (8 >> f)]
        assert on, dz
        for f in on:
            assert np.linalg.norm(np.cross(F[f], n)) <= 1e-12 * np.linalg.norm(F[f]) and F[f] @ n > 0, (dz, f, F[f])


def test_twin_lookup_matches_the_numpy_helper_and_finite_differences(twin):
    tiles = np.stack([T.rough(0.02, seed=4, corr=0.1, size=1.0, cell=CELL), T.ramp(15.0, 45.0, size=1.0, cell=CELL), T.stairs(0.05, 0.3, start=0.1, size=1.0, cell=CELL)])
    rng = np.random.default_rng(11); origin = np.array([-0.4, 0.3]); ext = (tiles.shape[2] - 1) * CELL
    xy = origin + rng.uniform(-0.3, ext + 0.3, (400, 2))   # inside the tile and beyond each border
    for t in range(len(tiles)):
        ter = dict(tiles=tiles, cell=CELL, tile=t, origin=origin)
        H, gx, gy = T.height(tiles, CELL, np.full(len(xy), t), origin, xy, gradient=True)
        for k, (x, y) in enumerate(xy):
            got = twin.ground(ter, x, y)
            np.testing.assert_allclose(got, (H[k], gx[k], gy[k]), rtol=0, atol=1e-12)
        # strictly inside cells, central differences of the bilinear height equal its gradient up to the cross term's O(eps) share
        u = rng.uniform(0.1, 0.9, (200, 2)) * CELL + CELL * rng.integers(0, tiles.shape[1] - 1, (200, 2)); p = origin + u; eps = 1e-6
        Hx = (T.height(tiles, CELL, t, origin, p + [eps, 0]) - T.height(tiles, CELL, t, origin, p - [eps, 0])) / (2 * eps)
        Hy = (T.height(tiles, CELL, t, origin, p + [0, eps]) - T.height(tiles, CELL, t, origin, p - [0, eps])) / (2 * eps)
        for k in range(len(p)):
            _, tgx, tgy = twin.ground(ter, *p[k])
            assert abs(tgx - Hx[k]) <= 1e-6 * max(1.0, abs(tgx)) and abs(tgy - Hy[k]) <= 1e-6 * max(1.0, abs(tgy)), (t, k, tgx, Hx[k], tgy, Hy[k])


def test_numpy_helper_clamp_is_nan_safe():
    tiles = T.rough(0.05, seed=2, size=1.0, cell=CELL)[None]
    for xy in ([np.nan, 0.2], [0.2, np.nan], [np.nan, np.nan], [np.inf, -np.inf], [-np.inf, np.nan]):
        H, gx, gy = T.height(tiles, CELL, 0, [0.0, 0.0], np.array(xy), gradient=True)
        assert np.isfinite(H) and tiles.min() <= H <= tiles.max(), xy
        for g, c in ((gx, xy[0]), (gy, xy[1])):
            assert g == 0.0 or np.isfinite(c), (xy, gx, gy)
    H = T.height(tiles, CELL, [-1, 0], [0.0, 0.0], np.array([[np.nan, np.nan]] * 2), ground=0.3)
    assert H[0] == 0.3 and np.isfinite(H[1])
    # outside the tile: the border value, zero gradient across the clamped axis
    H, gx, gy = T.height(tiles, CELL, 0, [0.0, 0.0], np.array([-5.0, 0.5]), gradient=True)
    assert H == T.height(tiles, CELL, 0, [0.0, 0.0], np.array([0.0, 0.5])) and gx == 0.0
