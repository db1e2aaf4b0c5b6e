"""Heightfield terrain for the plant (Solver.sim_set_terrain / Solver.sim_set_robot_terrain, include/qmb200.h: qmb200_sim_set_terrain) and the
numpy restatement of the plant's ground lookup.

A tile is an array [ny, nx] of absolute heights (world z, m) on nodes `cell` m apart; node (i, j) of robot b's tile lies at world origin[b] +
(i cell, j cell).  The builders share one square grid whose centre node sits at local (0, 0), and they keep the ground at z = 0 around that centre, so
a robot placed over it (centred_origin) starts on the ground its controller expects: the controller's base-height target is absolute (comHeight,
QmTargetTrajectoriesPublisher_node.cpp:87) and it does not see the terrain.  Builders return one tile; stack them (np.stack) into a library, and add
them to combine features (a ramp with steps on it).
"""
import numpy as np

SIZE = 4.0    # tile edge (m)
CELL = 0.02   # node spacing (m)


def grid(size=SIZE, cell=CELL):
    """Local node coordinates (X, Y), each [ny, nx], with the centre node at (0, 0)."""
    n = int(round(size / cell)) + 1
    c = (np.arange(n) - (n - 1) // 2) * cell
    return np.meshgrid(c, c)


def centred_origin(xy, size=SIZE, cell=CELL):
    """World origin (node (0, 0)) of a tile whose centre node lies at world xy [..., 2]."""
    n = int(round(size / cell)) + 1
    return np.asarray(xy, dtype=np.float64) - (n - 1) // 2 * cell


def _along(direction_deg, size, cell):
    X, Y = grid(size, cell); a = np.radians(direction_deg)
    return X * np.cos(a) + Y * np.sin(a)


def flat(size=SIZE, cell=CELL):
    return np.zeros_like(grid(size, cell)[0])


def ramp(angle_deg, direction_deg=0.0, start=None, size=SIZE, cell=CELL):
    """A slope of `angle_deg` rising along `direction_deg` (from +x towards +y).  start None: one plane through z = 0 at the centre; else flat (z = 0)
    up to `start` m from the centre along the direction, rising beyond."""
    d = _along(direction_deg, size, cell); t = np.tan(np.radians(angle_deg))
    return t * d if start is None else t * np.maximum(d - start, 0.0)


def stairs(rise, run, start=0.35, direction_deg=0.0, size=SIZE, cell=CELL):
    """Steps of height `rise` every `run` m along `direction_deg`, the first edge `start` m from the centre; flat (z = 0) before it.  A negative rise
    goes down.  The ground is bilinear between nodes, so an edge is a slope one cell wide."""
    d = _along(direction_deg, size, cell)
    return rise * np.where(d >= start, np.floor((d - start) / run) + 1.0, 0.0)


def rough(sigma, seed=0, corr=0.1, flat_radius=0.0, size=SIZE, cell=CELL):
    """Seeded rough ground: normal node heights smoothed over `corr` m (a box filter in x and y) and scaled to standard deviation `sigma` m; zero within
    `flat_radius` m of the centre."""
    X, Y = grid(size, cell); h = np.random.default_rng(seed).standard_normal(X.shape)
    k = max(1, int(round(corr / cell)))
    if k > 1:
        box = np.ones(k) / k
        h = np.apply_along_axis(np.convolve, 0, h, box, mode="same"); h = np.apply_along_axis(np.convolve, 1, h, box, mode="same")
    h *= sigma / np.std(h)
    h[np.hypot(X, Y) <= flat_radius] = 0.0
    return h


def height(tiles, cell, tile, origin, xy, ground=0.0, gradient=False):
    """Ground height under world points xy [..., 2] of robots on `tile` [...] (-1: the plane z = ground) with origins [..., 2]: the plant's lookup
    (bilinear in the cell, the border height outside the tile with zero gradient across the clamped axis).  gradient: also return (gx, gy)."""
    xy = np.asarray(xy, dtype=np.float64); origin = np.asarray(origin, dtype=np.float64)
    tile = np.asarray(tile); shape = np.broadcast_shapes(xy.shape[:-1], origin.shape[:-1], tile.shape)
    x, y = np.broadcast_to(xy[..., 0], shape), np.broadcast_to(xy[..., 1], shape)
    ox, oy = np.broadcast_to(origin[..., 0], shape), np.broadcast_to(origin[..., 1], shape); t = np.broadcast_to(tile, shape).astype(np.int64)
    H = np.full(shape, float(ground)); gx = np.zeros(shape); gy = np.zeros(shape)
    on = t >= 0
    if tiles is not None and np.any(on):
        tiles = np.asarray(tiles, dtype=np.float64); ny, nx = tiles.shape[1:]
        ur, vr = (x[on] - ox[on]) / cell, (y[on] - oy[on]) / cell
        u = np.fmin(np.fmax(ur, 0.0), nx - 1.0); v = np.fmin(np.fmax(vr, 0.0), ny - 1.0)   # fmin / fmax: a NaN coordinate lands inside the tile
        i = np.minimum(np.floor(u).astype(np.int64), nx - 2); j = np.minimum(np.floor(v).astype(np.int64), ny - 2)
        fx, fy = u - i, v - j; tt = t[on]
        h00, h10, h01, h11 = tiles[tt, j, i], tiles[tt, j, i + 1], tiles[tt, j + 1, i], tiles[tt, j + 1, i + 1]
        hxy = h11 - h10 - h01 + h00
        H[on] = h00 + fx * (h10 - h00) + fy * (h01 - h00) + fx * fy * hxy
        gx[on] = np.where(ur == u, ((h10 - h00) + fy * hxy) / cell, 0.0); gy[on] = np.where(vr == v, ((h01 - h00) + fx * hxy) / cell, 0.0)
    return (H, gx, gy) if gradient else H
