"""numpy statement of the per-robot curriculum of qmb200_curriculum_* (include/qmb200.h, DESIGN.md §4.15) — TEST INFRASTRUCTURE ONLY."""
import numpy as np

import _episode_twin as ep

METRICS = 18


def box(base, top, level, n_levels, round_col=-1):
    """base, top [m, W], level [m] → the box [m, W] at each level: base at 0, top at n_levels - 1, base between them where base == top, else
    fma(level / (n_levels - 1), top - base, base), floor(x + 0.5) in the rounded column"""
    base = np.asarray(base, dtype=np.float64); top = np.asarray(top, dtype=np.float64); lv = np.broadcast_to(np.asarray(level), base.shape[:1])[:, None]
    f = np.broadcast_to(lv.astype(np.float64) / np.float64(n_levels - 1), base.shape)
    mid = (lv > 0) & (lv < n_levels - 1) & (base != top)
    out = np.where(lv <= 0, base, top).copy()
    out[(lv > 0) & (lv < n_levels - 1) & (base == top)] = base[(lv > 0) & (lv < n_levels - 1) & (base == top)]
    if np.any(mid):
        x = ep.fma(f[mid], (top - base)[mid], base[mid])
        if round_col >= 0:
            x = np.where(np.nonzero(mid)[1] == round_col, np.floor(x + 0.5), x)
        out[mid] = x
    return out


def step(state, row, end, metrics, n_levels, conditions):
    """one update of one robot: state [level, pass_run, fail_run, n_updates], row [start, up_after, down_after, thr0..3], end, the closed episode's metrics
    row [18] (read only with conditions), conditions [(column index, op ">=" / "<=", role "pass" / "fail")] → the new state"""
    level, passes, fails, n = (int(x) for x in state)
    if end not in (1, 2):
        return [level, passes, fails, n]
    holds = [(metrics[c] >= row[3 + i]) if op == ">=" else (metrics[c] <= row[3 + i]) for i, (c, op, _) in enumerate(conditions)]
    failed = end == 1 or any(h for h, (_, _, role) in zip(holds, conditions) if role == "fail")
    passed = not failed and end == 2 and all(h for h, (_, _, role) in zip(holds, conditions) if role == "pass")
    n += 1
    if passed:
        passes, fails = passes + 1, 0
        if passes >= row[1]:
            level, passes = min(level + 1, n_levels - 1), 0
    elif failed:
        passes, fails = 0, fails + 1
        if fails >= row[2]:
            level, fails = max(level - 1, 0), 0
    return [level, passes, fails, n]
