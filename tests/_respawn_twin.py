"""numpy statement of the fall rule of qmb200_fall_detect (include/qmb200.h) — TEST INFRASTRUCTURE ONLY."""
import numpy as np

from qm_control_b200 import terrain as T


def fall_flags(rbd, terrain=None, z_min=0.3, tilt_max=0.3, ground=0.0):
    """rbd [..., B, 55] (plant truth) → fallen [..., B] bool: a non-finite base row (zyx, p), p_z - H(p_x, p_y) <= z_min with H the robot's ground
    (terrain: dict(tiles, cell, tile [B], origin [B, 2]) or None for the plane z = ground), or |pitch| or |roll| >= tilt_max."""
    rbd = np.asarray(rbd, dtype=np.float64); base = rbd[..., 0:6]
    finite = np.all(np.isfinite(base), axis=-1)
    xy = np.where(finite[..., None], base[..., 3:5], 0.0)
    H = np.full(finite.shape, float(ground)) if terrain is None else T.height(terrain["tiles"], terrain["cell"], terrain["tile"], terrain["origin"], xy, ground=ground)
    with np.errstate(invalid="ignore"):
        up = finite & (base[..., 5] - H > z_min) & (np.abs(base[..., 1]) < tilt_max) & (np.abs(base[..., 2]) < tilt_max)
    return ~up


def fall_counts(flags):
    """flags [ticks, B] of consecutive calls → the detector's count after each call [ticks, B] (one more per fallen call, 0 otherwise)."""
    flags = np.asarray(flags, dtype=bool); out = np.zeros(flags.shape, dtype=np.int32); c = np.zeros(flags.shape[1:], dtype=np.int32)
    for i, f in enumerate(flags):
        c = np.where(f, c + 1, 0); out[i] = c
    return out
