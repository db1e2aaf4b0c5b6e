"""numpy statement of the per-episode draw of qmb200_episode_* (include/qmb200.h, DESIGN.md §4.11) — TEST INFRASTRUCTURE ONLY."""
from fractions import Fraction

import numpy as np

from _state_est_twin import _mix

DOMAIN = np.uint64(0x6a09e667f3bcc909)   # episode_api.cuh's EPISODE_DOMAIN


def _u64(a):
    """the C cast to uint64_t (negative integers taken mod 2^64)"""
    a = np.asarray(a)
    return a.astype(np.uint64) if a.dtype == np.uint64 else a.astype(np.int64).astype(np.uint64)


def uniform(seed, robot, episode, channel):
    """u in (0, 1) of (seed, robot, episode, channel) (numpy broadcasting): the four words hashed in turn, the 53 high bits of one more hash, plus a half"""
    h = _mix(_mix(_mix(_mix(_u64(seed) ^ DOMAIN) ^ _u64(robot)) ^ _u64(episode)) ^ _u64(channel))
    return ((_mix(h) >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53


def fma(a, b, c):
    """a * b + c rounded once (to nearest, ties to even): exact rationals, then Python's correctly rounded int division"""
    a, b, c = np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), np.asarray(c, dtype=np.float64))
    return np.array([float(Fraction(x) * Fraction(y) + Fraction(z)) for x, y, z in zip(a.ravel(), b.ravel(), c.ravel())]).reshape(a.shape)


def rows(lo, hi, seed, robot, episode):
    """lo, hi [n, C], seed / robot / episode [n] → the rows [n, C]: column c is fma(u(seed, robot, episode, c), hi - lo, lo), and lo itself where hi == lo"""
    lo = np.asarray(lo, dtype=np.float64); hi = np.asarray(hi, dtype=np.float64)
    u = uniform(np.asarray(seed)[:, None], np.asarray(robot)[:, None], np.asarray(episode)[:, None], np.arange(lo.shape[1])[None, :])
    return np.where(hi == lo, lo, fma(u, hi - lo, lo))
