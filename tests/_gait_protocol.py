"""The GaitSchedule protocol driven on two sides — TEST INFRASTRUCTURE ONLY: random command timelines, one host qmb200_gait object per robot, and a
tick-by-tick comparison of a device-schedule implementation's windows, command rows, active templates and modes against those objects."""
import numpy as np

from qm_control_b200 import _lib
from qm_control_b200.interface import GaitSchedule, gait_template_names

GAIT_FILE = _lib.asset("qm_gait.info")
NAMES = gait_template_names(GAIT_FILE)
T = 1.0                       # mpc.timeHorizon (task.info)
ST_OVERFLOW, ST_NAN = 2, 4


def host_robot(gait, t_start):
    """qmb200_gait_create followed by qmb200_gait_insert_template(gait, t_start, T): the reset's definition"""
    g = GaitSchedule(); g.insertModeSequenceTemplate(gait, t_start, T, gait_file=GAIT_FILE)
    return g


def host_window(g, t):
    """→ (event_times [EMAX], modes [EMAX + 1], n) of getModeSchedule(t - T, t + 2T), or None where the host returns -2"""
    try:
        return g.getModeSchedule(t - T, t + 2 * T)
    except _lib.QmbError as e:
        assert "more than EMAX" in str(e)
        return None


def timeline(rng, n, t_end):
    """n commands in [0, t_end) with the gaps the protocol must survive: 1 ms, the same tick, inside a transition stance, long"""
    gaps = rng.choice([0.001, 0.0, 0.004, 0.05, 0.08, 1.0 + rng.uniform(0.0, 0.1), rng.uniform(0.2, 3.0)], size=n)
    t = rng.uniform(0.0, 0.5) + np.cumsum(gaps)
    t = t[t < t_end]
    gait = [NAMES[i] if i < len(NAMES) else None for i in rng.integers(0, len(NAMES) + 3, size=len(t))]
    for k in range(1, len(t)):   # the same gait twice
        if rng.uniform() < 0.15:
            gait[k] = gait[k - 1]
    vel = np.where(rng.uniform(size=(len(t), 1)) < 0.5, rng.uniform(-0.5, 0.5, size=(len(t), 4)), np.nan)
    return t, gait, vel


def drive(core, gait0, t_start, timelines, ticks, dt=0.01, nan_ticks=()):
    """Drive `core` (the host-compiled core or the device, both with reset / set_commands / step and the rows n_events, ev, md, cmd) and the host
    objects tick by tick; every window, command row, active template and mode must agree.  A robot is followed until its
    first overflow (where the host's object and the core's untouched schedule part ways).  → overflow tick per robot (-1: none), windows compared"""
    B = len(gait0); core.reset(gait0, t_start)
    C_ = max(len(tl[0]) for tl in timelines)
    t = np.full((B, C_), np.inf); tmpl = np.full((B, C_), -1, dtype=np.int32); vel = np.full((B, C_, 4), np.nan)
    for b, (tc, g, v) in enumerate(timelines):
        t[b, :len(tc)] = t_start[b] + tc; tmpl[b, :len(tc)] = [-1 if n is None else NAMES.index(n) for n in g]; vel[b, :len(tc)] = v
    core.set_commands(t, tmpl, vel)
    host = [host_robot(gait0[b], t_start[b]) for b in range(B)]
    active = [NAMES.index(g) for g in gait0]; cursor = [0] * B; cmd = np.zeros((B, 4)); over = np.full(B, -1); compared = 0
    t_obs = np.asarray(t_start, dtype=np.float64) - 0.002
    for i in range(ticks):
        tt = t_obs.copy()
        for b in nan_ticks and [b for b, k in nan_ticks if k == i]:
            tt[b] = np.nan
        tm, mode, st = core.step(tt)
        for b in range(B):
            if over[b] >= 0:
                continue
            if np.isnan(tt[b]):
                assert st[b] == ST_NAN; continue
            while cursor[b] < C_ and t[b, cursor[b]] <= tt[b]:
                if tmpl[b, cursor[b]] >= 0:
                    host[b].insertModeSequenceTemplate(NAMES[tmpl[b, cursor[b]]], tt[b] + T, T, gait_file=GAIT_FILE); active[b] = tmpl[b, cursor[b]]
                if not np.isnan(vel[b, cursor[b], 0]):
                    cmd[b] = vel[b, cursor[b]]
                cursor[b] += 1
            w = host_window(host[b], tt[b])
            if w is None:
                assert st[b] == ST_OVERFLOW, (b, i); over[b] = i; continue
            ev, md, n = w
            assert st[b] == 0 and core.n_events[b] == n, (b, i, st[b], core.n_events[b], n)
            assert core.ev[b].tobytes() == ev.tobytes(), (b, i)      # bit for bit, zeros past the count
            assert np.array_equal(core.md[b], md), (b, i)
            assert core.cmd[b, :4].tobytes() == cmd[b].tobytes() and tm[b] == active[b], (b, i)
            lb = int(np.searchsorted(ev[:n], tt[b], side="left")); assert mode[b] == md[lb]
            compared += 1
        t_obs = t_obs + dt
    return over, compared
