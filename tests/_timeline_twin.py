"""numpy statement of the per-episode command timeline draw of qmb200_timeline_* (include/qmb200.h, DESIGN.md §4.14) — TEST INFRASTRUCTURE ONLY."""
import numpy as np

import _episode_twin as ep

DOMAIN = np.uint64(0x3c6ef372fe94f82b)   # timeline_api.cuh's TIMELINE_DOMAIN
NAN = np.array([0x7FF8000000000000], dtype=np.uint64).view(np.float64)[0]
EE_CMD_VEL, EE_GOAL = 1, 2               # QMB200_TARGET_EE_*


def rows(lo, hi, seed, robot, episode, n):
    """lo, hi [m, 22], seed / robot / episode [m] → the slots [m, n, 14]: t, tmpl, cmd_vel[4], ee_kind, ee[7]"""
    lo = np.asarray(lo, dtype=np.float64); hi = np.asarray(hi, dtype=np.float64); m = len(lo)
    seed, robot, episode = (np.asarray(a) for a in (seed, robot, episode))

    def u(ch):
        return ep.uniform(seed, robot, episode, np.full(m, ch), DOMAIN)

    def box(c, ch, where=None):   # fixed: lo itself; box: fma(u, hi - lo, lo); only where `where` (the rest stays 0)
        out = lo[:, c].copy() if where is None else np.where(where, lo[:, c], 0.0)
        d = hi[:, c] != lo[:, c] if where is None else (hi[:, c] != lo[:, c]) & where
        if np.any(d):
            out[d] = ep.fma(u(ch)[d], (hi[:, c] - lo[:, c])[d], lo[:, c][d])
        return out
    mask = lo[:, 3].astype(np.uint64)
    bits = [[i for i in range(32) if (int(x) >> i) & 1] for x in mask]
    pc = np.array([len(b) for b in bits], dtype=np.float64)
    w = lo[:, 4:8]; run = np.stack([w[:, 0], w[:, 0] + w[:, 1], w[:, 0] + w[:, 1] + w[:, 2], w[:, 0] + w[:, 1] + w[:, 2] + w[:, 3]], axis=1)
    last = np.array([max([k for k in range(4) if r[k] > 0.0] or [0]) for r in w])
    out = np.zeros((m, n, 14)); t = None
    for j in range(n):
        ch = 16 * j
        t = box(0, 0) if j == 0 else t + box(1, ch)
        out[:, j, 0] = t
        gate = u(ch + 1) < lo[:, 2]
        k = np.minimum(np.floor(u(ch + 2) * pc), pc - 1)
        out[:, j, 1] = [bits[i][int(k[i])] if gate[i] else -1 for i in range(m)]
        x = u(ch + 3) * run[:, 3]
        above = run > x[:, None]
        kind = np.where(above.any(1), above.argmax(1), last)
        cv = kind == 1
        for i in range(4):
            out[:, j, 2 + i] = np.where(cv, box(8 + i, ch + 4 + i, cv), NAN)
        out[:, j, 6] = np.select([kind == 2, kind == 3], [EE_CMD_VEL, EE_GOAL], -1)
        for i in range(3):
            out[:, j, 7 + i] = np.where(kind == 2, box(12 + i, ch + 8 + i, kind == 2), np.where(kind == 3, box(15 + i, ch + 11 + i, kind == 3), 0.0))
        for i in range(4):
            out[:, j, 10 + i] = np.where(kind == 3, lo[:, 18 + i], 0.0)
    return out
