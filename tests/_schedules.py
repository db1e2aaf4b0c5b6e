"""Mode schedules beyond the three gaits of synthetic.make_batch, for the contact-mode and time-grid tests.

Every gait of assets/qm_gait.info, hand-built schedules that reach the masks no gait uses (a bound on the fore/hind pairs, single-foot
stances, all 16 masks in a row), a helper that puts a schedule into one robot of a make_batch dict, the oracle robot by robot (it raises for
the whole batch when one robot raises), and the equality-row count of every node of a grid."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from qm_control_b200 import _lib, synthetic
from qm_control_b200._lib import EMAX

GAIT_FILE = _lib.asset("qm_gait.info")
ALL_GAITS = ("stance", "trot", "standing_trot", "flying_trot", "pace", "standing_pace", "dynamic_walk", "static_walk", "amble", "lindyhop", "skipping", "pawup")
WEAK_EPS = 1e-6          # ocs2 weakEpsilon: the interval start / end shift at event nodes


def _check(e, m):
    if len(e) > EMAX:
        raise ValueError("schedule window needs more than EMAX events")
    return np.asarray(e, dtype=np.float64), np.asarray(m, dtype=np.int32)


def gait_schedule(name, t0, phase, horizon=1.0):
    """GaitSchedule tiling of gait `name` as make_batch does it: the template starts `phase` of a cycle before t0 - 2 horizon and the
    window is [t0 - horizon, t0 + 2 horizon] → (event_times, modes) with len(modes) = len(event_times) + 1."""
    times, modes = synthetic._gait_template(GAIT_FILE, name); dur = times[-1]
    e, m = synthetic.tile_schedule(times, modes, t0 - 2.0 * horizon - phase * dur, t0 - horizon, t0 + 2.0 * horizon)
    return _check(e, m)


def _tiled(phases, t0, horizon, phase=0.0):
    """A template of (mode, duration) phases tiled over [t0 - 0.25, t0 + horizon + 0.25]: short phases need a tighter window than the gaits."""
    times = np.r_[0.0, np.cumsum([d for _, d in phases])]; modes = [m for m, _ in phases]
    e, m = synthetic.tile_schedule(times, modes, t0 - 0.25 - phase * times[-1], t0 - 0.25, t0 + horizon + 0.25)
    return _check(e, m)


def bound(t0, horizon=1.0, phase=0.0):
    """fore pair / hind pair (masks 12 and 3) in 0.3 s phases."""
    return _tiled([(12, 0.3), (3, 0.3)], t0, horizon, phase)


def single_foot(mask, t0, horizon=1.0, phase=0.0):
    """mask (one foot down: 8, 4, 2, 1; or 0) between stance phases, 0.2 s each."""
    return _tiled([(mask, 0.2), (15, 0.2)], t0, horizon, phase)


def all_masks(t0, horizon=1.0, phase=0.0):
    """masks 0, 1, ..., 15 in 80 ms phases."""
    return _tiled([(m, 0.08) for m in range(16)], t0, horizon, phase)


def with_schedule(prob, b, events, modes):
    """Overwrite robot b's mode schedule in a make_batch dict (in place); every other input stays as make_batch made it."""
    events = np.asarray(events, dtype=np.float64); modes = np.asarray(modes, dtype=np.int32); ne = len(events)
    assert len(modes) == ne + 1 and ne <= EMAX
    prob["event_times"][b] = 0.0; prob["event_times"][b, :ne] = events
    prob["modes"][b] = 15; prob["modes"][b, :ne + 1] = modes; prob["n_events"][b] = ne
    return prob


def _robot(d, b):
    return {k: v[b:b + 1] for k, v in d.items()}


def oracle_per_robot(oracle, prob, nmax, prev=None, nthreads=8):
    """The oracle robot by robot → list of (result, None) or (None, error string); a result is the one-robot dict of mpc_solve_batch."""
    B = len(prob["t0"])

    def one(b):
        try:
            return oracle.mpc_solve_batch(_robot(prob, b), nmax, prev=None if prev is None else _robot(prev, b), nthreads=1), None
        except RuntimeError as e:
            return None, str(e)
    with ThreadPoolExecutor(nthreads) as ex:          # the oracle's error string is thread-local; ctypes drops the GIL for the call
        return list(ex.map(one, range(B)))


def mode_at(events, modes, t):
    return int(modes[int(np.searchsorted(events, t, side="left"))])


def ndep(mode):
    """Equality rows of a node in `mode`: 3 per stance foot (zero velocity), 4 per swing foot (zero force + normal velocity)."""
    return sum(3 if (mode >> (3 - f)) & 1 else 4 for f in range(4))


def mode_rows(events, modes, t, event, n):
    """For every interval k < n - 1 of a grid (t, event): the equality-row count of its mode; -1 at pre-event nodes (no input there)."""
    rows = np.full(n - 1, -1, dtype=np.int32)
    for k in range(n - 1):
        if event[k] != 1:
            rows[k] = ndep(mode_at(events, modes, t[k] + (WEAK_EPS if event[k] == 2 else 0.0)))
    return rows


def grid_has_nonpositive_interval(t, event, n):
    """getIntervalDuration <= 0 anywhere on the grid, with the interval_start / interval_end shifts of the event nodes."""
    for k in range(n - 1):
        if event[k] == 1:
            continue
        ts = t[k] + (WEAK_EPS if event[k] == 2 else 0.0); te = t[k + 1] - (WEAK_EPS if event[k + 1] == 1 else 0.0)
        if not te - ts > 0.0:
            return True
    return False
