"""The stepped closed loop and its command channel on the host, no GPU (DESIGN.md §4.16): the gait core with a pending command slot (compiled with
g++ by tests/gait_host_session.cpp, the very functions gait_step_kernel and gait_command_kernel run) against the same row on the timeline, byte for
byte; the device check of a command row against a numpy statement of it; closed_loop.Session's spec errors and calls on a fake Solver; the bindings and
the command kernel's resources."""
import contextlib
import ctypes as C
import os
import re
import shutil
import subprocess
from unittest import mock

import numpy as np
import pytest

from _oracle import REFERENCE, TASK
from _gait_protocol import GAIT_FILE, NAMES, ST_OVERFLOW
from test_ee_commands_cpu import ee_timelines, unit_quat
from test_gait_dev_cpu import B, _FakeStream, _fake_solver
from qm_control_b200 import _lib, closed_loop
from qm_control_b200._lib import EMAX

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
ST_COMMAND = 0x20000
NAMES_ABI = ("qmb200_gait_dev_command", "qmb200_gait_dev_command_dev", "qmb200_gait_dev_get_pending")


@pytest.fixture(scope="module")
def gsh(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("gait_host_session") / "libgaithostsession.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include",
                           "-I" + CSRC, "-o", lib_path, os.path.join(ROOT, "tests", "gait_host_session.cpp"), os.path.join(CSRC, "host", "qm_config.cpp")])
    lib = C.CDLL(lib_path); lib.gsh_create.restype = C.c_void_p
    lib.gsh_create.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_double]
    lib.gsh_destroy.argtypes = [C.c_void_p]; lib.gsh_reset.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double]
    lib.gsh_set_commands.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5; lib.gsh_command.argtypes = [C.c_void_p] * 7
    lib.gsh_step.argtypes = [C.c_void_p] * 8 + [C.c_int]; lib.gsh_get.argtypes = [C.c_void_p] * 4
    lib.gsh_check.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p]
    return lib


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


class Core:
    """B robots of the host-compiled core with the table of every qm_gait.info template, horizon T; MPC rows and cmd start at zero"""

    def __init__(self, lib, B_, T):
        self.lib, self.B = lib, B_
        arr = (C.c_char_p * len(NAMES))(*[n.encode() for n in NAMES])
        self.h = lib.gsh_create(TASK.encode(), REFERENCE.encode(), GAIT_FILE.encode(), C.cast(arr, C.c_void_p), len(NAMES), B_, T); assert self.h
        self.n_events = np.zeros(B_, dtype=np.int32); self.ev = np.zeros((B_, EMAX)); self.md = np.full((B_, EMAX + 1), 15, dtype=np.int32); self.cmd = np.zeros((B_, 7))

    def __del__(self):
        self.lib.gsh_destroy(C.c_void_p(self.h))

    def reset(self, tmpl, t_start):
        for b in range(self.B):
            assert self.lib.gsh_reset(C.c_void_p(self.h), b, int(tmpl[b]), float(t_start[b])) == 0

    def set_commands(self, t, tmpl, vel, kind, ee):
        self._cmd = [_c(t, np.float64), _c(tmpl, np.int32), _c(vel, np.float64), _c(kind, np.int32), _c(ee, np.float64)]
        self.lib.gsh_set_commands(C.c_void_p(self.h), self._cmd[0].shape[1], *[a.ctypes.data for a in self._cmd])

    def command(self, mask, tmpl, vel, kind, ee):
        rows = [_c(mask, np.int32), _c(tmpl, np.int32), _c(vel, np.float64), _c(kind, np.int32), _c(ee, np.float64)]; st = np.zeros(self.B, dtype=np.int32)
        self.lib.gsh_command(C.c_void_p(self.h), *[a.ctypes.data for a in rows], st.ctypes.data)
        return st

    def step(self, t_obs, with_pending=1):
        t_obs = _c(t_obs, np.float64); kind, st = np.zeros(self.B, dtype=np.int32), np.zeros(self.B, dtype=np.int32)
        self.lib.gsh_step(C.c_void_p(self.h), *[a.ctypes.data for a in (t_obs, self.n_events, self.ev, self.md, self.cmd, kind, st)], with_pending)
        return kind, st

    def get(self):
        robots = np.zeros((self.B, self.lib.gsh_robot_bytes()), dtype=np.uint8); cur, pend = np.zeros(self.B, dtype=np.int32), np.zeros(self.B, dtype=np.int32)
        self.lib.gsh_get(C.c_void_p(self.h), robots.ctypes.data, cur.ctypes.data, pend.ctypes.data)
        return robots, cur, pend

    def rows(self):
        return self.n_events.tobytes() + self.ev.tobytes() + self.md.tobytes() + self.cmd.tobytes()


def _random_rows(rng, B_):
    """one valid command row per robot: a template (40 %), and none, a cmd_vel, an ee_cmd_vel or a goal → (tmpl, vel [B, 4], kind, ee [B, 7])"""
    tmpl = np.where(rng.uniform(size=B_) < 0.4, rng.integers(0, len(NAMES), B_), -1).astype(np.int32)
    vel = np.full((B_, 4), np.nan); kind = np.full(B_, -1, dtype=np.int32); ee = np.zeros((B_, 7))
    for b, u in enumerate(rng.uniform(size=B_)):
        if u < 0.3:
            vel[b] = rng.uniform(-0.5, 0.5, 4)
        elif u < 0.55:
            kind[b] = 1; ee[b, :3] = rng.uniform(-0.1, 0.1, 3)
        elif u < 0.8:
            kind[b] = 2; ee[b, :3] = [0.52, 0.09, 0.44] + rng.uniform(-0.2, 0.2, 3); ee[b, 3:] = unit_quat(rng)
    return tmpl, vel, kind, ee


def _insert(tl, pos, t_row, row):
    """the timeline tl with row (tmpl, vel, kind, ee per robot) inserted at column pos[b] with time t_row[b]"""
    t, tmpl, vel, kind, ee = tl; B_, C_ = t.shape
    out = [np.zeros((B_, C_ + 1) + a.shape[2:], dtype=a.dtype) for a in tl]
    for b in range(B_):
        p = pos[b]
        for o, a, r in zip(out, tl, (t_row[b],) + tuple(x[b] for x in row)):
            o[b, :p] = a[b, :p]; o[b, p] = r; o[b, p + 1:] = a[b, p:]
    return out


@pytest.mark.parametrize("seed,T", [(1, 1.0), (2, 1.0), (3, 2.5), (4, 4.0)])
def test_a_pending_row_equals_the_same_row_last_on_the_timeline(gsh, seed, T):
    """Two cores from the same reset and timeline: A gets the row as a command, B the same row inserted on its timeline right after the rows due at the
    step's t.  Up to and including that step they agree byte for byte (robot, MPC rows, cmd, target kind; B's cursor one further when the step
    succeeds).  Long horizons make the window overflow, where A's slot stays set.  Before the step A gets another command, which the second replaces."""
    rng = np.random.default_rng(seed); B_ = 64
    t_start = 10.0 + rng.uniform(0.0, 0.3, B_); gait0 = rng.integers(0, len(NAMES), B_)
    tl = ee_timelines(rng, B_, t_start, 12, 4.0)
    ticks = int(rng.integers(1, 150)); t_obs = [t_start - 0.002 + 0.01 * i for i in range(ticks + 1)]
    t_cmd = t_obs[ticks]
    row = _random_rows(rng, B_); pos = (tl[0] <= t_cmd[:, None]).sum(1)
    a, b = Core(gsh, B_, T), Core(gsh, B_, T)
    a.reset(gait0, t_start); b.reset(gait0, t_start)
    a.set_commands(*tl); b.set_commands(*_insert(tl, pos, t_cmd, row))
    failed = np.zeros(B_, dtype=bool)
    for i in range(ticks):
        ka, sa = a.step(t_obs[i]); kb, sb = b.step(t_obs[i])
        assert ka.tobytes() == kb.tobytes() and sa.tobytes() == sb.tobytes() and a.rows() == b.rows(), i
        failed |= sa != 0
    mask = (rng.uniform(size=B_) < 0.8).astype(np.int32)
    first = _random_rows(rng, B_)
    assert not a.command(mask, *first).any()
    assert not a.command(mask, *row).any()   # replaces the first
    b2 = Core(gsh, B_, T); b2.reset(gait0, t_start); b2.set_commands(*tl)   # unmasked robots: the timeline without the row
    for i in range(ticks):
        b2.step(t_obs[i])
    _, _, pend = a.get(); np.testing.assert_array_equal(pend, mask)
    ka, sa = a.step(t_cmd); kb, sb = b.step(t_cmd); kc, sc = b2.step(t_cmd)
    ra, ca, pa = a.get(); rb, cb, _ = b.get(); rc, cc, _ = b2.get()
    m = mask.astype(bool) & ~failed   # a robot that overflowed earlier has B's row at an earlier place in its due rows
    np.testing.assert_array_equal(sa[m], sb[m]); np.testing.assert_array_equal(ka[m], kb[m])
    assert ra[m].tobytes() == rb[m].tobytes()
    np.testing.assert_array_equal(ca[m] + (sa[m] == 0), cb[m])
    for x, y in ((a.n_events, b.n_events), (a.ev, b.ev), (a.md, b.md), (a.cmd, b.cmd)):
        assert x[m].tobytes() == y[m].tobytes()
    np.testing.assert_array_equal(pa[m], (sa[m] != 0).astype(np.int32))   # cleared on success, still set after a failed step
    um = ~mask.astype(bool)
    assert ra[um].tobytes() == rc[um].tobytes() and np.array_equal(ca[um], cc[um]) and np.array_equal(sa[um], sc[um]) and not pa[um].any()
    assert a.n_events[um].tobytes() == b2.n_events[um].tobytes() and a.cmd[um].tobytes() == b2.cmd[um].tobytes()
    if T >= 2.5:
        assert np.any(sa[m] == ST_OVERFLOW), "no overflow case"
    assert np.any(sa[m] == 0)


def test_without_a_pending_row_the_step_is_the_step_before(gsh):
    rng = np.random.default_rng(9); B_ = 48
    t_start = 10.0 + rng.uniform(0.0, 0.3, B_); gait0 = rng.integers(0, len(NAMES), B_); tl = ee_timelines(rng, B_, t_start, 10, 3.0)
    a, b = Core(gsh, B_, 1.0), Core(gsh, B_, 1.0)
    for c in (a, b):
        c.reset(gait0, t_start); c.set_commands(*tl)
    for i in range(300):
        t = t_start - 0.002 + 0.01 * i
        assert a.step(t, 1)[0].tobytes() + a.rows() == b.step(t, 0)[0].tobytes() + b.rows()
    assert a.get()[0].tobytes() == b.get()[0].tobytes()


def _statement(tmpl, vel, kind, ee, nt):
    """the command rule in numpy: QMB200_ST_COMMAND where a row breaks one of qmb200_gait_dev_set_commands_ee's rules, else 0"""
    none = np.isnan(vel[:, 0])
    bad = (tmpl < -1) | (tmpl >= nt) | np.where(none, ~np.isnan(vel).all(1), ~np.isfinite(vel).all(1))
    ee_on = kind != -1
    goal = kind == 2
    bad |= ee_on & ~np.isin(kind, [1, 2])
    bad |= ee_on & np.isin(kind, [1, 2]) & ~none
    m = np.where(goal[:, None], np.ones(7, bool), np.arange(7) < 3)
    bad |= np.isin(kind, [1, 2]) & none & ~np.all(np.isfinite(ee) | ~m, axis=1)
    with np.errstate(invalid="ignore"):
        qn = np.sqrt(np.sum(ee[:, 3:7] ** 2, axis=1))
        bad |= goal & none & np.all(np.isfinite(ee), axis=1) & ~(np.abs(qn - 1.0) <= 1e-9)
    return np.where(bad, ST_COMMAND, 0).astype(np.int32)


def test_the_device_check_equals_its_numpy_statement(gsh):
    rng = np.random.default_rng(5); m = 20000; nt = len(NAMES)
    tmpl, vel, kind, ee = _random_rows(rng, m)
    case = rng.integers(0, 12, m)   # 0 and 1: valid; the rest break one rule
    tmpl[case == 2] = rng.choice([-2, nt, nt + 5, -(1 << 30)], np.sum(case == 2))
    vel[case == 3] = rng.uniform(-1, 1, (np.sum(case == 3), 4)); vel[case == 3, rng.integers(0, 4)] = np.nan            # partly NaN
    vel[case == 4] = np.inf
    kind[case == 5] = rng.choice([0, 3, -7], np.sum(case == 5))
    r6 = case == 6; kind[r6] = 1; ee[r6, :3] = 0.1; ee[r6, rng.integers(0, 3)] = rng.choice([np.nan, np.inf])
    r7 = case == 7; kind[r7] = 2; ee[r7] = [0.5, 0, 0.4, 0, 0, 0, 1]; ee[r7, rng.integers(0, 7)] = np.nan
    r8 = case == 8; kind[r8] = 2; ee[r8] = [0.5, 0, 0.4, 0, 0, 0, 1]; ee[r8, 6] = 1.0 + rng.choice([2e-9, -2e-9, 0.5], np.sum(r8))
    r9 = case == 9; kind[r9] = rng.choice([1, 2], np.sum(r9)); ee[r9] = [0.5, 0, 0.4, 0, 0, 0, 1]; vel[r9] = 0.1   # both
    r10 = case == 10; vel[r10] = np.nan; kind[r10] = 1; ee[r10, :3] = 0.1; ee[r10, 3:] = np.nan                                        # ignored columns of ee_cmd_vel
    r11 = case == 11; vel[r11] = np.nan; kind[r11] = 2; ee[r11] = [0.5, 0, 0.4, 0, 0, 0, 1.0 + 5e-10]                                   # inside 1e-9
    out = np.zeros(m, dtype=np.int32)
    rows = [_c(tmpl, np.int32), _c(vel, np.float64), _c(kind, np.int32), _c(ee, np.float64)]
    gsh.gsh_check(m, *[a.ctypes.data for a in rows], nt, out.ctypes.data)
    np.testing.assert_array_equal(out, _statement(tmpl, vel, kind, ee, nt))
    assert np.all(out[case >= 2] == np.where(np.isin(case[case >= 2], [10, 11]), 0, ST_COMMAND))
    assert np.all(out[case < 2] == 0)


# ---------------------------------------------------------------------------------------------------------------------- closed_loop.Session on a fake Solver
@contextlib.contextmanager
def _cpu_torch():
    import torch
    with mock.patch.object(torch.cuda, "Stream", _FakeStream), mock.patch.object(torch.cuda, "stream", lambda st: contextlib.nullcontext()):
        yield


def _solver():
    s = _fake_solver()
    s.gait_dev_command_dev = mock.Mock()
    return s


@pytest.mark.parametrize("kw,match", [
    (dict(respawn=dict(hold=0.015)), "multiple of 10 ms"), (dict(commands=dict(t=np.zeros((3, 1)), gait=[[None]] * 3)), "commands t must have shape"),
    (dict(steer=True, gait="gallop"), "unknown gait name"), (dict(metrics=1), "metrics must be None or True")])
def test_session_spec_errors_raise_before_any_solver_call(kw, match):
    s = _solver()
    with pytest.raises(ValueError, match=match):
        closed_loop.Session(s, 0.02, **kw)
    assert s.mock_calls == []
    with pytest.raises(TypeError, match="no_such_option"):
        closed_loop.Session(s, 0.02, no_such_option=1)
    assert s.mock_calls == []


def test_command_spec_errors_raise_before_any_solver_call():
    s = _solver()
    plain = closed_loop.Session(s, 0.02, gait="trot")
    with pytest.raises(ValueError, match="needs the device gait schedule"):
        plain.command(np.ones(B))
    steer = closed_loop.Session(s, 0.02, gait="trot", steer=True)
    for kw, match in ((dict(mask=np.ones(B + 1)), "mask must have shape"), (dict(mask=np.ones(B), cmd_vel=np.zeros((B, 3))), r"cmd_vel must have shape \(2, 4\)"),
                      (dict(mask=np.ones(B), ee_goal=np.zeros(7)), "ee_goal must have shape"), (dict(mask=np.ones(B), gait=np.zeros((B, 1))), "gait must have shape"),
                      (dict(mask=np.ones(B)), "not open")):
        with pytest.raises(ValueError, match=match):
            steer.command(**kw)
    yaw = closed_loop.Session(s, 0.02, gait="trot", steer=True, spawn=dict(yaw=(-0.5, 0.5)))
    with pytest.raises(ValueError, match="drawn spawn yaw"):
        yaw.command(np.ones(B), ee_cmd_vel=np.zeros((B, 3)))
    with pytest.raises(ValueError, match="not open"):
        steer.step()
    assert s.mock_calls == []


def _session_calls(chunks, duration=0.05, commands_at=(), **kw):
    s = _solver()
    with _cpu_torch():
        with closed_loop.Session(s, duration, **dict(dict(torch_device="cpu", gait="trot"), **kw)) as ss:
            recs = []
            for i, n in enumerate(chunks):
                if i in commands_at:
                    ss.command(np.ones(B, dtype=np.int32), cmd_vel=np.full((B, 4), 0.1))
                recs.append(ss.step(n))
            with pytest.raises(ValueError, match="exceed"):
                ss.step(1)
            end = ss.finish()
    return [c[0] for c in s.mock_calls], recs, end


def test_chunked_sessions_make_the_calls_of_run():
    import test_gait_dev_cpu
    _, want, _ = test_gait_dev_cpu._calls(duration=0.05, commands=dict(t=[[0.0], [0.0]], gait=[[None], [None]]))
    for chunks in ((5,), (1, 3, 1), (1, 1, 1, 1, 1), (2, 3)):
        calls, recs, end = _session_calls(chunks, commands=dict(t=[[0.0], [0.0]], gait=[[None], [None]]))
        assert calls == want, chunks
        assert [len(r["t"]) for r in recs] == list(chunks) and [tuple(r["gait"].shape) for r in recs] == [(n, B) for n in chunks]
        np.testing.assert_allclose(np.concatenate([r["t"] for r in recs]), 10.0 + 0.01 * np.arange(1, 6))
        assert set(end) >= {"q", "v", "contact", "start_base", "start_ee", "gait_templates"}


def test_a_command_is_one_call_before_the_tick_it_feeds():
    calls, _, _ = _session_calls((2, 3), steer=True, commands_at=(1,))
    i = calls.index("gait_dev_command_dev")
    assert calls.count("gait_dev_command_dev") == 1 and calls[i + 1:i + 4] == ["gait_dev_step_dev", "target_trajectories_dev", "mpc_solve_dev"]
    assert calls[:i].count("mpc_solve_dev") == 2 and calls.index("gait_dev_set_commands") < i   # after windows 0 and 1's ticks; steer loads a timeline
    s = _solver()
    with _cpu_torch():
        with closed_loop.Session(s, 0.02, torch_device="cpu", gait="trot", steer=True):
            pass
    t = s.gait_dev_set_commands.call_args[0][0]
    assert t.shape == (B, 0)   # steer: an empty timeline


def test_entry_points_are_bound_declared_and_the_status_bit_is_free():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES_ABI:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name
    assert "#define QMB200_ST_COMMAND 0x20000" in h and _lib.ST_COMMAND == ST_COMMAND
    bits = {int(v, 0) for k, v in re.findall(r"#define (QMB200_ST_\w+) (0x[0-9a-fA-F]+|\d+)", h) if k != "QMB200_ST_COMMAND"}
    assert ST_COMMAND not in bits and ST_COMMAND > max(bits) and ST_COMMAND >= 1 << 16 + 1   # above QMB200_ST_SAFETY and the MPC flags (bits 8..15)
    api = open(os.path.join(CSRC, "kernels", "respawn_api.cuh")).read()
    assert int(re.search(r"RESTORE_MAX_SEGS = (\d+)", api).group(1)) >= 8 + 5   # every imaged block and the cold-start blocks with the pending rows


def test_command_kernel_compiles_for_sm90a_without_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    obj = str(tmp_path / "gait.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "kernels", "gait_kernel.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    m = re.search(r"Function properties for (\w*gait_command_kernel\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert m and m.groups()[1:] == ("0", "0", "0"), r.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if os.path.exists(cuobjdump):
        sass = subprocess.run([cuobjdump, "-sass", "-fun", m.group(1), obj], capture_output=True, text=True, check=True).stdout
        assert "gait_command_kernel" in sass and not re.search(r"\b(LDL|STL)\b", sass)
