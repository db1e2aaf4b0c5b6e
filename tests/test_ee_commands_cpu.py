"""End-effector commands on the device command timeline, on the host, no GPU: the gait schedule's core (qm_control_b200/csrc/kernels/gait_api.cuh,
compiled with g++ by tests/gait_host_ee.cpp, the very step function gait_step_kernel runs) against a small Python statement of the target-source
protocol (DESIGN.md §4.8) on random timelines, bit for bit; and closed_loop.run's calls with end-effector commands on a fake Solver."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from _oracle import REFERENCE, TASK
from _gait_protocol import GAIT_FILE, NAMES, ST_NAN, ST_OVERFLOW, T, timeline
from qm_control_b200 import closed_loop
from qm_control_b200._lib import EMAX
from test_gait_dev_cpu import B, _calls, _fake_solver

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
CMD_VEL, EE_CMD_VEL, EE_GOAL, HELD = 0, 1, 2, -1


@pytest.fixture(scope="module")
def geh(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("gait_host_ee") / "libgaithostee.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include",
                           "-I" + CSRC, "-o", lib_path, os.path.join(ROOT, "tests", "gait_host_ee.cpp"), os.path.join(CSRC, "host", "qm_config.cpp")])
    lib = C.CDLL(lib_path); lib.geh_create.restype = C.c_void_p
    lib.geh_create.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_double]
    lib.geh_destroy.argtypes = [C.c_void_p]; lib.geh_reset.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double]
    lib.geh_set_commands.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5; lib.geh_step.argtypes = [C.c_void_p] * 10; lib.geh_get.argtypes = [C.c_void_p] * 3
    return lib


class Core:
    """B robots of the host-compiled core with the table of every qm_gait.info template; cmd rows start at zero"""

    def __init__(self, lib, B_):
        self.lib, self.B = lib, B_
        arr = (C.c_char_p * len(NAMES))(*[n.encode() for n in NAMES])
        self.h = lib.geh_create(TASK.encode(), REFERENCE.encode(), GAIT_FILE.encode(), C.cast(arr, C.c_void_p), len(NAMES), B_, T); assert self.h
        self.n_events = np.zeros(B_, dtype=np.int32); self.ev = np.zeros((B_, EMAX)); self.md = np.full((B_, EMAX + 1), 15, dtype=np.int32); self.cmd = np.zeros((B_, 7))

    def __del__(self):
        self.lib.geh_destroy(C.c_void_p(self.h))

    def reset(self, gait, t_start):
        for b in range(self.B):
            assert self.lib.geh_reset(C.c_void_p(self.h), b, NAMES.index(gait[b]), float(t_start[b])) == 0

    def set_commands(self, t, tmpl, vel, ee_kind=None, ee=None):
        self._cmd = [np.ascontiguousarray(t, dtype=np.float64), np.ascontiguousarray(tmpl, dtype=np.int32), np.ascontiguousarray(vel, dtype=np.float64),
                     None if ee_kind is None else np.ascontiguousarray(ee_kind, dtype=np.int32), None if ee is None else np.ascontiguousarray(ee, dtype=np.float64)]
        self.lib.geh_set_commands(C.c_void_p(self.h), self._cmd[0].shape[1], *[None if a is None else a.ctypes.data for a in self._cmd])

    def step(self, t_obs):
        t_obs = np.ascontiguousarray(t_obs, dtype=np.float64); tm, mode, st, kind = (np.zeros(self.B, dtype=np.int32) for _ in range(4))
        self.lib.geh_step(C.c_void_p(self.h), *[a.ctypes.data for a in (t_obs, self.n_events, self.ev, self.md, self.cmd, tm, mode, st, kind)])
        return tm, mode, st, kind

    def get(self):
        src, cur = np.zeros(self.B, dtype=np.int32), np.zeros(self.B, dtype=np.int32)
        self.lib.geh_get(C.c_void_p(self.h), src.ctypes.data, cur.ctypes.data)
        return src, cur


def unit_quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def ee_timelines(rng, B_, t_start, n, t_end):
    """Per robot the gait / cmd_vel rows of _gait_protocol.timeline; a row without cmd_vel becomes a goal (35 %), an ee_cmd_vel (35 %) or stays
    without a target command.  ee_cmd_vel rows carry NaN in their ignored columns 3:7.  → (t [B, C] +inf padded, tmpl, vel [B, C, 4], ee_kind, ee [B, C, 7])"""
    tls = [timeline(rng, n, t_end) for _ in range(B_)]; C_ = max(len(tl[0]) for tl in tls)
    t = np.full((B_, C_), np.inf); tmpl = np.full((B_, C_), -1, dtype=np.int32); vel = np.full((B_, C_, 4), np.nan)
    kind = np.full((B_, C_), -1, dtype=np.int32); ee = np.full((B_, C_, 7), np.nan)
    for b, (tc, g, v) in enumerate(tls):
        t[b, :len(tc)] = t_start[b] + tc; tmpl[b, :len(tc)] = [-1 if x is None else NAMES.index(x) for x in g]; vel[b, :len(tc)] = v
        for c in range(len(tc)):
            if not np.isnan(v[c, 0]):
                continue
            u = rng.uniform()
            if u < 0.35:
                kind[b, c] = EE_GOAL; ee[b, c, :3] = [0.52, 0.09, 0.44] + rng.uniform(-0.2, 0.2, 3); ee[b, c, 3:] = unit_quat(rng)
            elif u < 0.7:
                kind[b, c] = EE_CMD_VEL; ee[b, c, :3] = rng.uniform(-0.1, 0.1, 3)
    return t, tmpl, vel, kind, ee


class Statement:
    """The protocol's table in Python: per robot the source, the cursor and the target front-end's cmd row.  A step whose status is not 0 changes
    nothing and reports the source's kind; otherwise the due rows apply in order (a cmd_vel row writes cmd[0:4], an ee_cmd_vel row cmd[0:3], a goal
    cmd[0:7]) and the last target command sets the source; a goal applied by this step is published (kind 2), a goal source is held (-1)."""

    def __init__(self, t, vel, kind, ee):
        self.t, self.vel, self.kind, self.ee = t, vel, kind, ee; B_ = t.shape[0]
        self.src = np.zeros(B_, dtype=np.int32); self.cur = np.zeros(B_, dtype=np.int32); self.cmd = np.zeros((B_, 7))

    def step(self, t_obs, status):
        out = np.zeros(len(t_obs), dtype=np.int32)
        for b, tb in enumerate(t_obs):
            applied = -1
            if status[b] == 0:
                while self.cur[b] < self.t.shape[1] and self.t[b, self.cur[b]] <= tb:
                    c = self.cur[b]
                    if not np.isnan(self.vel[b, c, 0]):
                        self.cmd[b, :4] = self.vel[b, c]; applied = CMD_VEL
                    if self.kind[b, c] >= 0:
                        m = 7 if self.kind[b, c] == EE_GOAL else 3
                        self.cmd[b, :m] = self.ee[b, c, :m]; applied = self.kind[b, c]
                    self.cur[b] += 1
                if applied >= 0:
                    self.src[b] = applied
            out[b] = EE_GOAL if applied == EE_GOAL else HELD if self.src[b] == EE_GOAL else self.src[b]
        return out


def _drive(geh, B_, gait0, t_start, tl, ticks, nan_ticks=()):
    """Three cores in lock step: with the end-effector rows, with the same timeline and no end-effector arrays, and with end-effector arrays that
    hold no command.  → (kinds seen, overflowing steps, windows compared)"""
    t, tmpl, vel, kind, ee = tl
    cores = [Core(geh, B_) for _ in range(3)]
    for core, ek in zip(cores, ((kind, ee), (None, None), (np.full_like(kind, -1), np.full_like(ee, np.nan)))):
        core.reset(gait0, t_start); core.set_commands(t, tmpl, vel, *ek)
    ref = Statement(t, vel, kind, ee); seen = {}; overflow = 0; compared = 0
    t_obs = np.asarray(t_start, dtype=np.float64) - 0.002
    for i in range(ticks):
        tt = t_obs.copy()
        for b in [b for b, k in nan_ticks if k == i]:
            tt[b] = np.nan
        (tm, mode, st, k), plain, empty = (c.step(tt) for c in cores)
        assert np.array_equal(st, plain[2]) and np.array_equal(tm, plain[0]) and np.array_equal(mode, plain[1]), i
        for other, out in ((cores[1], plain), (cores[2], empty)):
            assert other.n_events.tobytes() == cores[0].n_events.tobytes() and other.ev.tobytes() == cores[0].ev.tobytes(), i   # windows unchanged
            assert other.md.tobytes() == cores[0].md.tobytes(), i
        assert np.all(plain[3] == CMD_VEL) and empty[3].tobytes() == plain[3].tobytes() and cores[2].cmd.tobytes() == cores[1].cmd.tobytes(), i
        want = ref.step(tt, st)
        src, cur = cores[0].get()
        np.testing.assert_array_equal(k, want, err_msg="target_kind, tick %d" % i)
        np.testing.assert_array_equal(src, ref.src, err_msg="source, tick %d" % i); np.testing.assert_array_equal(cur, ref.cur, err_msg="cursor, tick %d" % i)
        assert cores[0].cmd.tobytes() == ref.cmd.tobytes(), (i, np.flatnonzero(np.any(cores[0].cmd != ref.cmd, axis=1)))   # bit for bit
        assert set(np.unique(st)) <= {0, ST_NAN, ST_OVERFLOW}
        for v in k:
            seen[int(v)] = seen.get(int(v), 0) + 1
        overflow += int(np.sum(st == ST_OVERFLOW)); compared += int(np.sum(st == 0))
        t_obs = t_obs + 0.01
    return seen, overflow, compared


def test_core_follows_the_protocol_on_random_timelines(geh):
    """24 robots over every template, 1000 ticks (10 s), random timelines of gait, cmd_vel, ee_cmd_vel and goal rows (1 ms gaps, same-tick groups,
    long gaps), with NaN ticks: cmd rows, target kinds, sources and cursors bit for bit against the statement; windows, templates, modes and status
    identical to the run without end-effector arrays and to the run with arrays that hold no command."""
    rng = np.random.default_rng(5); B_ = 24
    gait0 = [NAMES[b % len(NAMES)] for b in range(B_)]; t_start = 10.0 + rng.uniform(0.0, 1.0, size=B_)
    seen, overflow, compared = _drive(geh, B_, gait0, t_start, ee_timelines(rng, B_, t_start, 60, 10.0), 1000, nan_ticks=[(3, 17), (5, 400), (9, 401)])
    print("target kinds seen %s, %d overflowing steps, %d steps compared" % (seen, overflow, compared))
    assert all(seen.get(k, 0) > 200 for k in (HELD, CMD_VEL, EE_CMD_VEL)) and seen.get(EE_GOAL, 0) > 30 and compared > 0.9 * B_ * 1000


def test_failed_steps_leave_source_and_cmd_untouched(geh):
    """Skipping robots with two skipping → skipping switches 0.15 s apart (they overflow on some phases) and, from 1 s on, a row every 10 ms that
    alternates between a goal and an ee_cmd_vel command, each with other values: on every step that overflows, the robot keeps its source, cursor
    and cmd row and reports that source's kind (the rows due then wait for a later step); a NaN step on it does the same.  Every goal row is
    published exactly once on robots whose steps never failed."""
    phases = np.arange(0.0, 1.2, 0.01); B_ = len(phases); core = Core(geh, B_); core.reset(["skipping"] * B_, np.full(B_, 10.0))
    n_ee = 300; t_ee = 11.0 + 0.01 * np.arange(n_ee) + 0.005
    t = np.sort(np.c_[np.tile(t_ee, (B_, 1)), 12.0 + phases, 12.15 + phases], axis=1); C_ = t.shape[1]
    tmpl = np.where(t == (12.0 + phases)[:, None], NAMES.index("skipping"), -1); tmpl[t == (12.15 + phases)[:, None]] = NAMES.index("skipping")
    tmpl = tmpl.astype(np.int32); vel = np.full((B_, C_, 4), np.nan); kind = np.full((B_, C_), -1, dtype=np.int32); ee = np.full((B_, C_, 7), np.nan)
    for b in range(B_):
        for j, c in enumerate(np.flatnonzero(tmpl[b] < 0)):
            kind[b, c] = EE_GOAL if j % 2 == 0 else EE_CMD_VEL
            ee[b, c, :3] = [0.5 + 1e-4 * j, 0.09, 0.44]
            if j % 2 == 0:
                ee[b, c, 3:] = [0.5, -0.5, 0.5, -0.5]
    core.set_commands(t, tmpl, vel, kind, ee)
    tt = np.full(B_, 9.998); hit = due = 0; published = np.zeros((B_, C_), dtype=bool); failed = np.zeros(B_, dtype=bool)
    for i in range(500):
        src0, cur0 = core.get(); cmd0 = core.cmd.copy()
        tm, mode, st, k = core.step(tt); src, cur = core.get()
        for b in np.flatnonzero(st == ST_OVERFLOW):
            want = HELD if src0[b] == EE_GOAL else src0[b]
            assert src[b] == src0[b] and cur[b] == cur0[b] and k[b] == want and core.cmd[b].tobytes() == cmd0[b].tobytes(), (i, b)
            hit += 1; due += int(cur0[b] < C_ and t[b, cur0[b]] <= tt[b])
            t2 = tt.copy(); t2[b] = np.nan; c1 = core.cmd.copy()
            _, _, st2, k2 = core.step(t2); src2, cur2 = core.get()
            assert st2[b] == ST_NAN and src2[b] == src0[b] and cur2[b] == cur[b] and k2[b] == want and core.cmd[b].tobytes() == c1[b].tobytes()
            break   # the extra step moved the other robots on; leave the rest of this tick's overflows to later ticks
        failed |= st != 0
        for b in np.flatnonzero((st == 0) & (k == EE_GOAL)):
            c = max(j for j in range(cur0[b], cur[b]) if kind[b, j] >= 0)   # the step's last target command
            assert kind[b, c] == EE_GOAL and not published[b, c] and core.cmd[b].tobytes() == ee[b, c].tobytes(), (i, b)
            published[b, c] = True
        tt = tt + 0.01
    print("overflow on %d of %d phases (%d checked, %d with a row due), goals published %d" % (failed.sum(), B_, hit, due, published.sum()))
    ok = ~failed
    assert hit > 0 and due > 0 and np.all(published[ok] == (kind[ok] == EE_GOAL))


# ---- closed_loop.run on a fake Solver, tensors on the CPU (tests/test_gait_dev_cpu.py's) ----
GOAL = [0.6, 0.1, 0.45, 0.5, -0.5, 0.5, -0.5]


def test_loop_calls_with_end_effector_commands():
    """The calls are those of a run with commands; the timeline goes to Solver.gait_dev_set_commands with ee_kind / ee_cmd; every gait step's
    target_kind buffer is the kind the following target call takes, and the record gains target_kind and ee_target."""
    nan = [np.nan] * 7
    cmds = dict(t=[[0.005, 0.5, 0.6], [0.0, 0.0, 0.3]], gait=[["pace", None, None], [None, None, "stance"]],
                cmd_vel=[[[np.nan] * 4, [np.nan] * 4, [0.1, 0, 0, 0]], [[np.nan] * 4] * 3],
                ee_goal=[[GOAL, nan, nan], [nan, GOAL, nan]], ee_cmd_vel=[[[np.nan] * 3, [0.05, 0.0, 0.0], [np.nan] * 3], [[np.nan] * 3, [np.nan] * 3, [0, 0, 0.01]]])
    s, calls, r = _calls(commands=cmds)
    _, plain, _ = _calls(commands=dict(t=cmds["t"], gait=cmds["gait"]))
    assert calls == plain
    t, tm, vel = s.gait_dev_set_commands.call_args[0]; kw = s.gait_dev_set_commands.call_args[1]
    np.testing.assert_array_equal(kw["ee_kind"], [[EE_GOAL, EE_CMD_VEL, -1], [-1, EE_GOAL, EE_CMD_VEL]])
    np.testing.assert_array_equal(kw["ee_cmd"][0, 0], GOAL); np.testing.assert_array_equal(kw["ee_cmd"][1, 1], GOAL)
    np.testing.assert_array_equal(kw["ee_cmd"][0, 1, :3], [0.05, 0.0, 0.0]); np.testing.assert_array_equal(kw["ee_cmd"][1, 2, :3], [0, 0, 0.01])
    assert vel[0, 2, 0] == 0.1 and np.isnan(vel[1]).all()
    for st, tc in zip(s.gait_dev_step_dev.call_args_list, s.target_trajectories_dev.call_args_list):
        assert st[1]["target_kind"] is tc[0][0] and st[0][2] is tc[0][1] and st[0][0] is tc[0][2]
    assert r["target_kind"].shape == (2, B) and r["target_kind"].dtype == np.int32 and r["ee_target"].shape == (2, B, 7)


def test_loop_without_end_effector_keys_sets_a_plain_timeline():
    """commands without ee_goal / ee_cmd_vel load the timeline without end-effector arrays; the target calls still take the steps' kinds."""
    s, calls, r = _calls(commands=dict(t=[[0.0], [0.0]], gait=[[None], [None]], cmd_vel=[[[0.2, 0, 0, 0]], [[np.nan] * 4]]))
    assert s.gait_dev_set_commands.call_args[1] == {}
    assert all(tc[0][0] is st[1]["target_kind"] for st, tc in zip(s.gait_dev_step_dev.call_args_list, s.target_trajectories_dev.call_args_list))


@pytest.mark.parametrize("extra, match", [
    (dict(ee_goal=np.zeros((B, 1, 6))), "shape"),
    (dict(ee_cmd_vel=np.zeros((B, 2, 3))), "shape"),
    (dict(ee_goal=[[[0.6, np.nan, 0.4, 0.5, -0.5, 0.5, -0.5]], [[np.nan] * 7]]), "finite or all NaN"),
    (dict(ee_cmd_vel=[[[np.inf, 0, 0]], [[np.nan] * 3]]), "finite or all NaN"),
    (dict(ee_goal=[[[0.6, 0.1, 0.4, 0.5, -0.5, 0.5, -0.5 + 1e-6]], [[np.nan] * 7]]), "unit norm"),
    (dict(ee_goal=[[GOAL], [[np.nan] * 7]], ee_cmd_vel=[[[0.1, 0, 0]], [[np.nan] * 3]]), "at most one"),
    (dict(ee_goal=[[GOAL], [[np.nan] * 7]], cmd_vel=[[[0.1, 0, 0, 0]], [[np.nan] * 4]]), "at most one"),
    (dict(ee_target=[[GOAL], [GOAL]]), "dict"),
])
def test_loop_rejects_bad_end_effector_commands(extra, match):
    s = _fake_solver()
    with pytest.raises(ValueError, match=match):
        closed_loop.run(s, duration=0.01, commands=dict(t=[[0.0], [0.1]], gait=[[None], [None]], **extra))
    assert s.mock_calls == []


def test_unit_quaternions_within_the_tolerance_pass():
    goal = np.array(GOAL); goal[3:] *= 1.0 + 4e-10
    s, calls, r = _calls(commands=dict(t=[[0.0], [0.0]], gait=[[None], [None]], ee_goal=[[goal], [GOAL]]))
    assert s.gait_dev_set_commands.call_args[1]["ee_kind"].tolist() == [[EE_GOAL], [EE_GOAL]]
