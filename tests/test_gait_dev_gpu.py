"""The device gait schedule on the GPU: gait_step_kernel against one host qmb200_gait object per robot (random per-robot timelines, every window, command
row and status bit for bit), the entry points' validation, and closed loops: a timeline that changes nothing leaves the run byte-identical, a
stance → trot → stance switch, and a run past the length the host tiling allowed."""
import numpy as np
import pytest

import qm_control_b200 as q
from qm_control_b200 import _lib, closed_loop
from _gait_protocol import NAMES, drive, timeline

pytestmark = pytest.mark.gpu
T_START = closed_loop.T_START


class Device:
    """the handle's device schedule behind the interface tests/_gait_protocol.drive expects, through the host-pointer step"""

    def __init__(self, solver):
        self.s = solver; B = solver.batch; solver.gait_dev_set_templates()
        self.n_events = np.zeros(B, dtype=np.int32); self.ev = np.zeros((B, _lib.EMAX)); self.md = np.full((B, _lib.EMAX + 1), 15, dtype=np.int32)
        self.cmd = np.zeros((B, 7))

    def reset(self, gait, t_start):
        self.s.gait_dev_reset(gait, t_start)

    def set_commands(self, t, tmpl, vel):
        self.s.gait_dev_set_commands(t, tmpl, vel)

    def step(self, t_obs):
        return self.s.gait_dev_step(t_obs, dict(n_events=self.n_events, event_times=self.ev, modes=self.md), self.cmd)


def test_kernel_matches_the_host_objects():
    """256 robots, 500 ticks, random per-robot timelines over every template (1 ms gaps, same-tick pairs, switches inside a transition stance, the same
    gait twice, into and out of stance)."""
    rng = np.random.default_rng(11); B = 256; s = q.Solver(batch=B)
    gait0 = [NAMES[b % len(NAMES)] for b in range(B)]; t_start = T_START + rng.uniform(0.0, 1.0, size=B)
    timelines = [timeline(rng, 20, 5.0) for _ in range(B)]
    dev = Device(s)
    over, compared = drive(dev, gait0, t_start, timelines, 500, nan_ticks=[(7, 30)])
    print("%d windows compared bit for bit, overflow on %d robots" % (compared, (over >= 0).sum()))
    assert compared > 0.9 * B * 500
    g = s.gait_dev_get(); assert np.all(g["n_events"][over < 0] == dev.n_events[over < 0])
    s.gait_dev_stop(); s.close()


def test_skipping_overflow_on_the_device():
    """The two-switch skipping case of the CPU suite overflows on the device on exactly the host's ticks."""
    phases = np.arange(0.0, 1.2, 0.01); B = len(phases); s = q.Solver(batch=B)
    timelines = [(np.array([2.0 + p, 2.15 + p]), ["skipping"] * 2, np.full((2, 4), np.nan)) for p in phases]
    over, _ = drive(Device(s), ["skipping"] * B, np.full(B, T_START), timelines, 400)
    assert (over >= 0).any()
    s.close()


def test_entry_points_validate():
    s = q.Solver(batch=2)
    with pytest.raises(q.QmbError, match="not running"):
        s.gait_dev_get()
    with pytest.raises(q.QmbError, match="no template table"):
        s._call("gait_dev_reset", _lib.P(np.zeros(2, dtype=np.int32).ctypes.data), _lib.P(np.zeros(2).ctypes.data))
    with pytest.raises(q.QmbError):
        s.gait_dev_set_templates(["trot", "gallop"])
    s.gait_dev_set_templates(["stance", "trot"])
    with pytest.raises(q.QmbError, match="template"):
        s.gait_dev_reset(np.array([0, 2], dtype=np.int32), [10.0, 10.0])
    s.gait_dev_reset(["stance", "trot"], 10.0)
    with pytest.raises(q.QmbError, match="running"):
        s.gait_dev_set_templates(["trot"])
    for t, tm, vel, match in (([[0.5, 0.4], [0.0, 0.0]], [[-1, -1]] * 2, np.full((2, 2, 4), np.nan), "sorted"),
                              ([[0.0], [0.0]], [[2], [-1]], np.full((2, 1, 4), np.nan), "template"),
                              ([[0.0], [0.0]], [[1], [-1]], [[[0.1, np.nan, 0, 0]], [[np.nan] * 4]], "cmd_vel")):
        with pytest.raises(q.QmbError, match=match):
            s.gait_dev_set_commands(t, tm, vel)
    g = s.gait_dev_get(); assert list(g["tmpl"]) == [0, 1] and list(g["cursor"]) == [0, 0]
    s.gait_dev_stop(); s.gait_dev_stop()
    with pytest.raises(q.QmbError, match="not running"):
        s.gait_dev_step(np.zeros(2), dict(n_events=np.zeros(2), event_times=np.zeros((2, _lib.EMAX)), modes=np.zeros((2, _lib.EMAX + 1))), np.zeros((2, 7)))
    s.close()


def _same(a, b, keys=("base", "ee", "status", "q", "v")):
    return {k: a[k].tobytes() == b[k].tobytes() for k in keys}


@pytest.mark.parametrize("mixed", [False, True])
def test_a_timeline_that_changes_nothing_leaves_the_run_byte_identical(mixed):
    """64 robots for 1 s, on trot or on every template but stance and pawup: commands that re-send the run's cmd_vel or nothing at all give the run
    without commands byte for byte (the window's event times come from the same recurrence from t_start, and the MPC reads the schedule only through
    lower_bound, the grid in [t0, tf] and the swing enclosure).  Not for stance (the loop passes no events for it without commands) nor pawup: its LF
    foot never touches down, so that swing phase is closed only by the final stance of the tiling, which the host puts after the run's end and the
    rolled window after t_obs + 2T; the swing reference then differs (on every other template and foot the enclosures agree over the 1 s)."""
    B = 64; s = q.Solver(batch=B)
    mix = [n for n in NAMES if n not in ("stance", "pawup")]
    gait = [mix[b % len(mix)] for b in range(B)] if mixed else "trot"
    cmd = (0.2, 0.0, 0.0, 0.0); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    commands = dict(t=np.tile([0.0, 0.3, 0.61], (B, 1)), gait=np.full((B, 3), None, dtype=object), cmd_vel=np.tile([[np.nan] * 4, cmd, cmd], (B, 1, 1)))
    runs = []
    for kw in ({}, {}, dict(commands=commands)):   # every run from a cold MPC and WBC state: a run leaves its warm start behind
        s.mpc_reset(); s.wbc_set_input_last(None)
        runs.append(closed_loop.run(s, duration=1.0, gait=gait, cmd_vel=cmd, xy_yaw=xy, **kw))
    ref, again, got = runs
    print("repeat:", _same(ref, again), "commands:", _same(ref, got))
    assert all(_same(ref, again).values()) and all(_same(ref, got).values())
    assert np.all(got["gait"] == np.array([NAMES.index(g) for g in ([gait] * B if isinstance(gait, str) else gait)])[None, :])
    s.close()


def test_stance_trot_stance():
    """64 robots, 4 s: stance, trot at 0.3 m/s from 0.5 s, stance (cmd_vel 0) from 2.0 s.  Each command takes effect T later (inserted at t_obs + T).
    Everyone stays up with no status bit; the planned mode is stance until the trot starts, alternates LF_RH / RF_LH during it and is stance again
    from the transition stance inserted at t_cmd + T on; each base moves during the trot and stops after it."""
    B = 64; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    commands = dict(t=np.tile([0.5, 2.0], (B, 1)), gait=np.tile(np.array(["trot", "stance"], dtype=object), (B, 1)),
                    cmd_vel=np.tile([[0.3, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0]], (B, 1, 1)))
    r = closed_loop.run(s, duration=4.0, gait="stance", xy_yaw=xy, commands=commands)
    t_obs = r["t"] - 0.012                                    # the t_obs of each record's gait step (the tick that opens the record's window)
    z = r["base"][:, :, 2]; print("min z %.3f, status %s" % (z.min(), np.unique(r["status"])))
    assert np.all(r["status"] == 0) and z.min() > 0.3
    i1, i2 = np.argmax(t_obs >= T_START + 0.5), np.argmax(t_obs >= T_START + 2.0)   # the steps that applied the commands
    on, off = t_obs[i1] + 1.0, t_obs[i2] + 1.0               # stance → trot needs no transition stance; trot → stance inserts it at off
    md, eps = r["mode"], 1e-9
    assert np.all(md[t_obs < on - eps] == 15) and np.all(md[t_obs > off + eps] == 15)
    assert set(np.unique(md[(t_obs > on + eps) & (t_obs < off - eps)])) == {6, 9}
    assert np.all(r["gait"][:i1] == NAMES.index("stance")) and np.all(r["gait"][i1:i2] == NAMES.index("trot")) and np.all(r["gait"][i2:] == NAMES.index("stance"))
    x = r["base"][:, :, 0]; a, b, c = np.argmax(t_obs > on), np.argmax(t_obs > off), np.argmax(t_obs > off + 0.5)
    moved, after = x[b] - x[a], np.abs(x[-1] - x[c])
    print("moved during the trot %.3f..%.3f m, in the last 0.5 s %.4f m at most" % (moved.min(), moved.max(), after.max()))
    assert moved.min() > 0.05 and after.max() < 0.03
    s.close()


def test_runs_past_the_old_length_limit():
    """64 robots, 10.5 s: stance for 1 s, then trot.  Without commands this run's host schedule does not fit QMB200_EMAX events."""
    B = 64; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    with pytest.raises((ValueError, q.QmbError)):
        closed_loop.run(s, duration=10.5, gait="trot", xy_yaw=xy)
    commands = dict(t=np.full((B, 1), 1.0), gait=np.full((B, 1), "trot", dtype=object), cmd_vel=np.tile([0.3, 0.0, 0.0, 0.0], (B, 1, 1)))
    r = closed_loop.run(s, duration=10.5, gait="stance", xy_yaw=xy, commands=commands)
    print("min z %.3f, status %s" % (r["base"][:, :, 2].min(), np.unique(r["status"])))
    assert np.all(r["status"] == 0) and r["base"][:, :, 2].min() > 0.3
    s.close()
