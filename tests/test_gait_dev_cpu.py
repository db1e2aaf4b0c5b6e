"""The device gait schedule on the host, no GPU: its core (qm_control_b200/csrc/kernels/gait_api.cuh, compiled with g++ by tests/gait_host.cpp, the very
step function gait_step_kernel runs) against one host qmb200_gait object per robot driven through the same protocol (random timelines over all twelve
templates, every window bit for bit, overflow exactly where the host returns -2), and closed_loop.run's calls with and without commands on a fake
Solver."""
import contextlib
import ctypes as C
import os
import subprocess
import types
from unittest import mock

import numpy as np
import pytest

from _oracle import REFERENCE, TASK
from qm_control_b200 import _lib
from qm_control_b200._lib import EMAX
from qm_control_b200.interface import GaitSchedule
from _gait_protocol import GAIT_FILE, NAMES, ST_NAN, ST_OVERFLOW, T, drive, timeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")


@pytest.fixture(scope="module")
def gsh(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("gait_host") / "libgaithost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include",
                           "-I" + CSRC, "-o", lib_path, os.path.join(ROOT, "tests", "gait_host.cpp"), os.path.join(CSRC, "host", "qm_config.cpp")])
    lib = C.CDLL(lib_path); lib.gsh_create.restype = C.c_void_p
    lib.gsh_create.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_double]
    lib.gsh_destroy.argtypes = [C.c_void_p]; lib.gsh_reset.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double]
    lib.gsh_set_commands.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 3; lib.gsh_step.argtypes = [C.c_void_p] * 9
    return lib


class Core:
    """B robots of the host-compiled core with the table of every qm_gait.info template"""

    def __init__(self, lib, B):
        self.lib, self.B = lib, B
        arr = (C.c_char_p * len(NAMES))(*[n.encode() for n in NAMES])
        self.h = lib.gsh_create(TASK.encode(), REFERENCE.encode(), GAIT_FILE.encode(), C.cast(arr, C.c_void_p), len(NAMES), B, T); assert self.h
        self.n_events = np.zeros(B, dtype=np.int32); self.ev = np.zeros((B, EMAX)); self.md = np.full((B, EMAX + 1), 15, dtype=np.int32); self.cmd = np.zeros((B, 7))

    def __del__(self):
        self.lib.gsh_destroy(C.c_void_p(self.h))

    def reset(self, gait, t_start):
        for b in range(self.B):
            assert self.lib.gsh_reset(C.c_void_p(self.h), b, NAMES.index(gait[b]), float(t_start[b])) == 0

    def set_commands(self, t, tmpl, vel):
        self._cmd = [np.ascontiguousarray(t, dtype=np.float64), np.ascontiguousarray(tmpl, dtype=np.int32), np.ascontiguousarray(vel, dtype=np.float64)]
        self.lib.gsh_set_commands(C.c_void_p(self.h), self._cmd[0].shape[1], *[a.ctypes.data for a in self._cmd])

    def step(self, t_obs):
        t_obs = np.ascontiguousarray(t_obs, dtype=np.float64); tm, mode, st = (np.zeros(self.B, dtype=np.int32) for _ in range(3))
        self.lib.gsh_step(C.c_void_p(self.h), *[a.ctypes.data for a in (t_obs, self.n_events, self.ev, self.md, self.cmd, tm, mode, st)])
        return tm, mode, st


def test_core_matches_the_host_objects_on_random_protocols(gsh):
    """24 robots over every template, 1000 ticks of 10 ms each (10 s), random timelines of gait and cmd_vel commands."""
    rng = np.random.default_rng(7); B = 24
    gait0 = [NAMES[b % len(NAMES)] for b in range(B)]; t_start = 10.0 + rng.uniform(0.0, 1.0, size=B)
    timelines = [timeline(rng, 40, 10.0) for _ in range(B)]
    over, compared = drive(Core(gsh, B), gait0, t_start, timelines, 1000, nan_ticks=[(3, 17), (5, 400)])
    n_cmd = sum(len(tl[0]) for tl in timelines)
    print("%d windows compared bit for bit, %d commands, overflow on %d robots at ticks %s" % (compared, n_cmd, (over >= 0).sum(), over[over >= 0]))
    assert compared > 0.9 * B * 1000


def test_core_long_run_without_commands_keeps_rolling(gsh):
    """6000 ticks (60 s) of each template without a command: the window never overflows and equals the host's."""
    over, compared = drive(Core(gsh, len(NAMES)), NAMES, np.full(len(NAMES), 10.0), [(np.zeros(0), [], np.zeros((0, 4)))] * len(NAMES), 6000)
    assert np.all(over < 0) and compared == 6000 * len(NAMES)


def test_skipping_through_a_transition_overflows_where_the_host_does(gsh):
    """A skipping robot holds up to 29 events in steady state and one switch through a transition stance reaches 31 at most (searched over every pair
    and 10 ms phase).  Two skipping → skipping switches 0.15 s apart, at every 10 ms phase of the 1.2 s cycle, reach 33 on some phases: the core
    overflows exactly on the ticks where the host returns -2."""
    phases = np.arange(0.0, 1.2, 0.01); B = len(phases)
    timelines = [(np.array([2.0 + p, 2.15 + p]), ["skipping"] * 2, np.full((2, 4), np.nan)) for p in phases]
    over, compared = drive(Core(gsh, B), ["skipping"] * B, np.full(B, 10.0), timelines, 500)
    print("overflow on %d of %d phases" % ((over >= 0).sum(), B))
    assert (over >= 0).any()


def test_overflow_and_nan_leave_everything_as_it_was(gsh):
    """A step that overflows or reads a non-finite t_obs writes nothing: rows, command row and the schedule stay, and the due commands are applied by a
    later step."""
    phases = np.arange(0.0, 1.2, 0.01); B = len(phases)
    core = Core(gsh, B); core.reset(["skipping"] * B, np.full(B, 10.0))
    core.set_commands(10.0 + np.c_[2.0 + phases, 2.15 + phases], np.full((B, 2), NAMES.index("skipping")), np.tile([0.1, 0.0, 0.0, 0.0], (B, 2, 1)))
    t = np.full(B, 9.998)
    for i in range(500):
        before = (core.n_events.copy(), core.ev.copy(), core.md.copy(), core.cmd.copy())
        tm, mode, st = core.step(t)
        hit = np.flatnonzero(st == ST_OVERFLOW)
        if len(hit):
            b = hit[0]
            assert core.n_events[b] == before[0][b] and core.ev[b].tobytes() == before[1][b].tobytes() and np.array_equal(core.md[b], before[2][b])
            assert core.cmd[b].tobytes() == before[3][b].tobytes()   # nor the cmd_vel of the overflowing step's command
            tt = t.copy(); tt[b] = np.inf; n0 = core.n_events.copy(); e0 = core.ev.copy()
            tm, mode, st = core.step(tt)
            assert st[b] == ST_NAN and core.n_events[b] == n0[b] and core.ev[b].tobytes() == e0[b].tobytes()
            return
        t = t + 0.01
    pytest.fail("no overflow")


# ---- closed_loop.run on a fake Solver, tensors on the CPU ----
B = 2


class _FakeStream:
    cuda_stream = 0

    def __init__(self, device=None):
        pass

    def synchronize(self):
        pass


def _fake_solver():
    names = ["sim_standing_state", "sim_step_dev", "centroidal_state_from_rbd", "initial_ee_target", "hw_set_delay", "target_trajectories_dev", "mpc_solve_dev",
             "update_dev", "hw_write_dev", "gait_dev_set_templates", "gait_dev_reset", "gait_dev_set_commands", "gait_dev_step_dev", "gait_dev_stop"]
    s = mock.Mock(spec=names, batch=B, time_horizon=1.0, _cfg=types.SimpleNamespace(device=0))
    q0 = np.zeros((B, 24)); q0[:, 2] = 0.45
    s.sim_standing_state.return_value = (q0, np.zeros((B, 24)))
    s.centroidal_state_from_rbd.side_effect = lambda rbd: np.zeros((B, _lib.NX))
    s.initial_ee_target.return_value = np.zeros((B, 7))
    return s


def _calls(**kw):
    import torch
    from qm_control_b200 import closed_loop
    s = _fake_solver()
    with mock.patch.object(torch.cuda, "Stream", _FakeStream), mock.patch.object(torch.cuda, "stream", lambda st: contextlib.nullcontext()):
        r = closed_loop.run(s, **dict(dict(duration=0.02, torch_device="cpu", gait="trot"), **kw))
    return s, [c[0] for c in s.mock_calls], r


def _parent_calls():
    """the calls closed_loop.run issues without commands, for a 20 ms run (WBC every 2 ms)"""
    out = ["sim_standing_state", "sim_step_dev", "centroidal_state_from_rbd", "initial_ee_target", "hw_set_delay", "target_trajectories_dev", "mpc_solve_dev"]
    for k in range(20):
        out += (["target_trajectories_dev", "mpc_solve_dev"] if k == 10 else []) + (["update_dev"] if k % 2 == 0 else []) + ["hw_write_dev", "sim_step_dev"]
    return out


def test_loop_calls_without_commands_are_unchanged():
    s, calls, r = _calls()
    assert calls == _parent_calls() and "gait" not in r and "mode" not in r


def test_loop_calls_with_commands():
    cmds = dict(t=[[0.005, 0.5], [0.0, 0.0]], gait=[["pace", None], [None, "stance"]], cmd_vel=[[[0.2, 0, 0, 0], [np.nan] * 4], [[np.nan] * 4, [np.nan] * 4]])
    s, calls, r = _calls(commands=cmds)
    want = ["gait_dev_set_templates"]
    for c in _parent_calls():
        if c == "hw_set_delay":
            want += ["gait_dev_reset", "gait_dev_set_commands"]
        if c == "target_trajectories_dev":
            want.append("gait_dev_step_dev")
        want.append(c)
    assert calls == want + ["gait_dev_stop"]
    assert s.gait_dev_set_templates.call_args[0][0] == NAMES
    tmpl, t0 = s.gait_dev_reset.call_args[0]; assert list(tmpl) == [NAMES.index("trot")] * 2 and np.all(t0 == 10.0)
    t, tm, vel = s.gait_dev_set_commands.call_args[0]
    np.testing.assert_array_equal(t, 10.0 + np.array(cmds["t"])); assert tm.tolist() == [[NAMES.index("pace"), -1], [-1, NAMES.index("stance")]]
    assert vel[0, 0, 0] == 0.2 and np.isnan(vel[1]).all()
    tg = s.target_trajectories_dev.call_args_list
    for st, tc in zip(s.gait_dev_step_dev.call_args_list, tg):
        assert st[0][2] is tc[0][1] and st[0][0] is tc[0][2]   # the step writes the cmd rows the targets read, at the same t_obs
    assert st[0][1]["modes"] is s.mpc_solve_dev.call_args[0][0]["modes"]
    assert r["gait"].shape == (2, B) and r["mode"].shape == (2, B) and r["gait_templates"] == NAMES


def test_loop_runs_past_the_host_tiling_limit_with_commands():
    """A 9 s trot needs more than EMAX events in the host's one window for the run; with commands the loop rolls the window and runs."""
    from qm_control_b200 import closed_loop
    with pytest.raises((ValueError, _lib.QmbError), match="more than"):
        closed_loop._schedules("trot", B, 10.0, 9.998, 10.0 + 9.0 + 2.0)
    s, calls, r = _calls(commands=dict(t=np.zeros((B, 0)), gait=np.zeros((B, 0), dtype=object)), duration=9.0)
    assert calls.count("gait_dev_step_dev") == calls.count("target_trajectories_dev") == 900 and r["gait"].shape == (900, B)


@pytest.mark.parametrize("commands, match", [
    (dict(t=[[0.0]], gait=[["trot"]]), "shape"),
    (dict(t=[[0.0], [0.1]], gait=[["trot"], ["gallop"]]), "unknown gait"),
    (dict(t=[[0.5, 0.4], [0.0, 0.1]], gait=[["trot", None], [None, None]]), "sorted"),
    (dict(t=[[0.0], [np.nan]], gait=[[None], [None]]), "sorted"),
    (dict(t=[[0.0], [0.1]], gait=[[None], [None]], cmd_vel=[[[0.1, np.nan, 0, 0]], [[np.nan] * 4]]), "cmd_vel"),
    (dict(t=[[0.0], [0.1]], gait=[[None], [None]], vel=1), "dict"),
    ([0.0], "dict"),
])
def test_loop_rejects_bad_commands(commands, match):
    from qm_control_b200 import closed_loop
    s = _fake_solver()
    with pytest.raises(ValueError, match=match):
        closed_loop.run(s, duration=0.01, commands=commands)
    with pytest.raises(ValueError, match="unknown gait"):
        closed_loop.run(s, duration=0.01, gait="gallop", commands=dict(t=np.zeros((B, 0)), gait=np.zeros((B, 0), dtype=object)))
    assert s.mock_calls == []


def test_template_names_follow_the_gait_file():
    assert NAMES[:4] == ["stance", "trot", "standing_trot", "flying_trot"] and len(NAMES) == 12
    for n in NAMES:
        g = GaitSchedule(); g.insertModeSequenceTemplate(n, 10.0, T, gait_file=GAIT_FILE)   # every listed name is a template of the file
