"""Per-episode end-effector paths on the host, no GPU (DESIGN.md §4.21): the draw core compiled with g++ (tests/ee_path_draw_host.cpp) against an
independent numpy statement, every drawn row against the path table's check, the independence of its columns, the range check and the curriculum's
level checks of the kind, closed_loop.run(ee_path_draw=...) validation, refusals and calls on a fake Solver, the bindings and the sampler's resources."""
import contextlib
import ctypes as C
import os
import re
import shutil
import subprocess
import types
from unittest import mock

import numpy as np
import pytest

import _episode_twin as ep
from test_ee_frame_cpu import _resources
from test_gait_dev_cpu import B, _FakeStream, _fake_solver, _parent_calls
from qm_control_b200 import _lib, closed_loop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
PR = {n: i for i, n in enumerate(_lib.EE_PATH_RANGES_LAYOUT)}
PMAX, W = _lib.EE_PATH_MAX, _lib.EE_PATH_RANGES
NAMES = ("qmb200_ee_path_set_ranges", "qmb200_ee_path_get_ranges", "qmb200_ee_path_sample", "qmb200_ee_path_sample_dev", "qmb200_ee_path_draw")

# ---------------------------------------------------------------------------------------------------------------------- the numpy statement
DOMAIN = np.uint64(0xa54ff53a5f1d36f1)   # ee_path_draw_api.cuh's EE_PATH_DOMAIN
SIN = [1 / 51090942171709440000, -1 / 121645100408832000, 1 / 355687428096000, -1 / 1307674368000, 1 / 6227020800, -1 / 39916800, 1 / 362880, -1 / 5040,
       1 / 120, -1 / 6]
COS = [-1 / 1124000727777607680000, 1 / 2432902008176640000, -1 / 6402373705728000, 1 / 20922789888000, -1 / 87178291200, 1 / 479001600, -1 / 3628800,
       1 / 40320, -1 / 720, 1 / 24, -1 / 2]


def sincos(h):
    """sine and cosine of h in [-pi/2, pi/2]: the Taylor polynomials to h^21 / h^22 in Horner form, every product and sum rounded once"""
    z = h * h; p = np.full_like(h, SIN[0]); q = np.full_like(h, COS[0])
    for c in SIN[1:]:
        p = p * z + c
    for c in COS[1:]:
        q = q * z + c
    return h + (h * z) * p, 1.0 + z * q


def after(t, g):
    """t + g, rounded up where the nearest rounding falls short of the exact sum"""
    s = t + g; v = s - t; e = (t - (s - v)) + (g - v)
    return np.where(e > 0.0, np.nextafter(s, np.inf), s)


def draw(lo, hi, seed, robot, episode):
    """lo, hi [m, 11], seed / robot / episode [m] → (n_way [m], way [m, 32, 8]): waypoint i's time on channel 8 i (tau_first, then the previous time plus
    gap, rounded up where it falls short), its position on 8 i + 1..3, its quaternion Rz(yaw) quat with yaw on 8 i + 4; a box column fma(u, hi - lo, lo), a fixed one lo itself"""
    lo = np.asarray(lo, dtype=np.float64); hi = np.asarray(hi, dtype=np.float64); m = len(lo)
    n = lo[:, 0].astype(int); way = np.zeros((m, PMAX, 8)); t = np.zeros(m)
    for i in range(PMAX):
        act = i < n

        def box(c, ch):
            out = lo[:, c].copy(); d = (hi[:, c] != lo[:, c]) & act
            if np.any(d):
                out[d] = ep.fma(ep.uniform(seed, robot, episode, np.full(m, ch), DOMAIN)[d], (hi[:, c] - lo[:, c])[d], lo[:, c][d])
            return out
        tau = box(1, 8 * i) if i == 0 else after(t, box(2, 8 * i))
        sh, ch = sincos(0.5 * box(6, 8 * i + 4))
        qx, qy, qz, qw = (lo[:, 7 + k] for k in range(4))
        w = np.stack([tau, box(3, 8 * i + 1), box(4, 8 * i + 2), box(5, 8 * i + 3), ch * qx - sh * qy, ch * qy + sh * qx, ch * qz + sh * qw, ch * qw - sh * qz], 1)
        way[act, i] = w[act]; t = np.where(act, tau, t)
    return n, way


# ---------------------------------------------------------------------------------------------------------------------- the host build
@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("ee_path_draw") / "libeepathdrawhost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include",
                           "-I" + CSRC, "-o", lib_path, os.path.join(ROOT, "tests", "ee_path_draw_host.cpp")])
    lib = C.CDLL(lib_path)
    lib.epd_rows.argtypes = [C.c_int] + [C.c_void_p] * 7
    lib.epd_ranges_error.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_char_p, C.c_int]
    lib.epd_paths_error.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_char_p, C.c_int]
    lib.epd_attach_error.argtypes = [C.c_int, C.c_int, C.c_double] + [C.c_void_p] * 4 + [C.c_char_p, C.c_int]
    return lib


def _c(a, dtype=np.float64):
    return np.ascontiguousarray(a, dtype=dtype)


def _rows(core, lo, hi, seed, robot, episode):
    m = len(lo); lo, hi = _c(lo), _c(hi); seed, robot, episode = (_c(a, np.uint64) for a in (seed, robot, episode))
    n_way = np.zeros(m, dtype=np.int32); way = np.zeros((m, PMAX, 8))
    core.epd_rows(m, seed.ctypes.data, robot.ctypes.data, episode.ctypes.data, lo.ctypes.data, hi.ctypes.data, n_way.ctypes.data, way.ctypes.data)
    return n_way, way


def _ranges(rng, m, n, T=1.0):
    """valid ranges covering the corners: fixed columns holding -0.0, zero-width boxes, yaw boxes and fixed yaws at +-pi, gaps at exactly T/2"""
    lo = np.zeros((m, W)); hi = np.zeros_like(lo)
    lo[:, PR["n_way"]] = hi[:, PR["n_way"]] = n
    lo[:, PR["tau_first"]] = rng.choice([0.05, rng.uniform(0.01, 1.0)], m); hi[:, PR["tau_first"]] = lo[:, PR["tau_first"]] + rng.choice([0.0, 0.5], m)
    lo[:, PR["gap"]] = rng.choice([0.5 * T, rng.uniform(0.5 * T, 2.0)], m); hi[:, PR["gap"]] = lo[:, PR["gap"]] + rng.choice([0.0, 0.7], m)
    for c in ("x", "y", "z"):
        lo[:, PR[c]] = rng.uniform(-1.0, 1.0, m); fixed = rng.uniform(size=m) < 0.4
        hi[:, PR[c]] = np.where(fixed, lo[:, PR[c]], lo[:, PR[c]] + rng.uniform(0.0, 1.0, m))
        z = fixed & (rng.uniform(size=m) < 0.3); lo[z, PR[c]] = hi[z, PR[c]] = -0.0
    kind = rng.integers(0, 5, m)   # a box, the full circle, fixed +pi, fixed -pi, fixed -0.0
    a = rng.uniform(-np.pi, np.pi, (m, 2)); a.sort(1)
    lo[:, PR["yaw"]] = np.select([kind == 0, kind == 1, kind == 2, kind == 3], [a[:, 0], -np.pi, np.pi, -np.pi], -0.0)
    hi[:, PR["yaw"]] = np.select([kind == 0, kind == 1, kind == 2, kind == 3], [a[:, 1], np.pi, np.pi, -np.pi], -0.0)
    q = rng.normal(size=(m, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True); q[::7] = [-0.0, 0.0, -0.0, 1.0]; q[1::7] = [0.5, -0.5, 0.5, -0.5]
    lo[:, 7:11] = hi[:, 7:11] = q
    return lo, hi


def _keys(rng, m):
    seed = rng.integers(0, 2 ** 63, m, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, m, dtype=np.uint64)
    return seed, rng.integers(0, 1 << 20, m).astype(np.uint64)


@pytest.mark.parametrize("n", [1, 4, 32])
def test_core_equals_the_numpy_statement_bit_for_bit(core, n):
    rng = np.random.default_rng(200 + n); m = 3000
    lo, hi = _ranges(rng, m, n); seed, robot = _keys(rng, m)
    for episode in (np.zeros(m, dtype=np.uint64), rng.integers(0, 1 << 31, m).astype(np.uint64), np.full(m, 2 ** 64 - 1, dtype=np.uint64)):
        n_way, way = _rows(core, lo, hi, seed, robot, episode)
        n_tw, way_tw = draw(lo, hi, seed, robot, episode)
        assert np.array_equal(n_way, n_tw) and way.tobytes() == way_tw.tobytes()   # byte for byte: -0.0 included


def test_the_polynomial_sines_are_the_library_sines_within_an_ulp_or_two():
    h = np.linspace(-np.pi / 2, np.pi / 2, 100_001)
    s, c = sincos(h)
    assert np.max(np.abs(s - np.sin(h))) <= 4.5e-16 and np.max(np.abs(c - np.cos(h))) <= 4.5e-16


@pytest.mark.parametrize("T", [1.0, 0.6])
def test_every_drawn_row_passes_the_path_table_check(core, T):
    rng = np.random.default_rng(7); msg = C.create_string_buffer(256)
    for n in (1, 2, 5, 32):
        lo, hi = _ranges(rng, 500, n, T); seed, robot = _keys(rng, 500)
        assert _check(core, lo, hi, T) == (0, "")
        n_way, way = _rows(core, lo, hi, seed, robot, rng.integers(0, 1 << 31, 500).astype(np.uint64))
        rc = core.epd_paths_error(len(n_way), _c(n_way, np.int32).ctypes.data, _c(way).ctypes.data, T, msg, 256)
        assert rc == 0, msg.value.decode()
        assert np.all(way[:, n:] == 0.0) and np.all(np.diff(way[:, :n, 0], axis=1) >= 0.5 * T)


def test_changing_one_box_leaves_every_other_column(core):
    rng = np.random.default_rng(8); m = 400; n = 6
    lo, hi = _ranges(rng, m, n); seed, robot = _keys(rng, m); episode = rng.integers(0, 1 << 31, m).astype(np.uint64)
    _, a = _rows(core, lo, hi, seed, robot, episode)
    for c, cols in (("x", [1]), ("y", [2]), ("z", [3]), ("yaw", [4, 5, 6, 7]), ("gap", [0]), ("tau_first", [0])):
        l2, h2 = lo.copy(), hi.copy(); h2[:, PR[c]] = h2[:, PR[c]] + 0.25 if c != "yaw" else np.minimum(h2[:, PR[c]] + 0.25, np.pi)
        _, b = _rows(core, l2, h2, seed, robot, episode)
        other = [k for k in range(8) if k not in cols]
        assert a[:, :, other].tobytes() == b[:, :, other].tobytes(), c
        assert not np.array_equal(a[:, :n, cols], b[:, :n, cols]), c


def _check(core, lo, hi, T=1.0):
    msg = C.create_string_buffer(256); rc = core.epd_ranges_error(len(lo), _c(lo).ctypes.data, _c(hi).ctypes.data, T, msg, 256)
    return rc, msg.value.decode()


def _valid(Bn=4):
    lo = np.zeros((Bn, W)); lo[:, PR["n_way"]] = 3; lo[:, PR["tau_first"]] = 0.2; lo[:, PR["gap"]] = 0.6; lo[:, PR["qw"]] = 1.0
    hi = lo.copy(); hi[:, PR["tau_first"]] = 0.4; hi[:, PR["gap"]] = 1.0; hi[:, PR["x"]] = 0.1; hi[:, PR["yaw"]] = 1.0
    return lo, hi


@pytest.mark.parametrize("field,lo_v,hi_v,why", [
    ("x", np.nan, 0.0, "bounds must be finite"), ("y", 0.5, 0.1, "lo must be <= hi"), ("z", -1e308, 1e308, "hi - lo must be finite"),
    ("n_way", 3.0, 4.0, "must be fixed (lo == hi)"), ("n_way", 0.0, 0.0, "must be an integer in [1, QMB200_EE_PATH_MAX (32)]"),
    ("n_way", 33.0, 33.0, "must be an integer in [1, QMB200_EE_PATH_MAX (32)]"), ("n_way", 2.5, 2.5, "must be an integer in [1, QMB200_EE_PATH_MAX (32)]"),
    ("tau_first", 0.0, 0.3, "lo must be > 0 (seconds after the path starts)"), ("gap", 0.49, 1.0, "lo must be >= T/2 = 0.500000 s"),
    ("yaw", -3.2, 0.0, "bounds must lie in [-pi, pi]"), ("yaw", 0.0, 3.2, "bounds must lie in [-pi, pi]"), ("qw", 1.0, 0.9, "lo must be <= hi"),
    ("qx", 0.0, 0.1, "must be fixed (lo == hi)"),
])
def test_each_range_rule_names_the_field_and_the_robot(core, field, lo_v, hi_v, why):
    lo, hi = _valid(); assert _check(core, lo, hi) == (0, "")
    lo[2, PR[field]] = lo_v; hi[2, PR[field]] = hi_v
    assert _check(core, lo, hi) == (1, "qmb200_ee_path_set_ranges: %s of robot 2: %s" % (field, why))


def test_the_quaternion_rule_names_the_robot(core):
    lo, hi = _valid(); lo[3, PR["qw"]] = hi[3, PR["qw"]] = 1.0 + 2e-9
    assert _check(core, lo, hi) == (1, "qmb200_ee_path_set_ranges: quat of robot 3: must have unit norm (within 1e-9)")
    lo[3, PR["qw"]] = hi[3, PR["qw"]] = 1.0 + 5e-10
    assert _check(core, lo, hi) == (0, "")
    lo[3, PR["yaw"]] = -np.pi; hi[3, PR["yaw"]] = np.pi; lo[1, PR["gap"]] = 0.5
    assert _check(core, lo, hi) == (0, "")


def test_the_last_drawn_time_is_bounded_so_that_every_drawn_row_stays_finite(core):
    lo, hi = _valid(); lo[:, PR["n_way"]] = hi[:, PR["n_way"]] = 32; hi[:, PR["tau_first"]] = 0.4
    hi[1, PR["gap"]] = 1e299   # 0.4 + 31e299 > 1e300: the later waypoint times could overflow
    assert _check(core, lo, hi) == (1, "qmb200_ee_path_set_ranges: gap of robot 1: tau_first hi + (n_way - 1) gap hi must be <= 1e300 s")
    hi[1, PR["gap"]] = 3.2e298   # 0.4 + 31 * 3.2e298 = 9.92e299: accepted, and every row it draws is finite and passes the table check
    assert _check(core, lo, hi) == (0, "")
    m = 400; lo, hi = np.repeat(lo[1:2], m, 0), np.repeat(hi[1:2], m, 0); rng = np.random.default_rng(9); seed, robot = _keys(rng, m)
    n_way, way = _rows(core, lo, hi, seed, robot, rng.integers(0, 1 << 31, m).astype(np.uint64))
    msg = C.create_string_buffer(256)
    assert np.all(np.isfinite(way)) and core.epd_paths_error(m, _c(n_way, np.int32).ctypes.data, _c(way).ctypes.data, 1.0, msg, 256) == 0, msg.value.decode()
    assert np.max(way[:, -1, 0]) > 1e299


def _attach(core, L, base_lo, base_hi, top_lo, top_hi, T=1.0):
    a = [_c(x) for x in (base_lo, base_hi, top_lo, top_hi)]; msg = C.create_string_buffer(256)
    rc = core.epd_attach_error(L, len(a[0]), T, *(x.ctypes.data for x in a), msg, 256)
    return rc, msg.value.decode()


def test_the_curriculum_checks_every_level_and_both_ends(core):
    lo, hi = _valid()
    top_lo, top_hi = lo.copy(), hi.copy(); top_hi[:, PR["x"]] = 0.5; top_lo[:, PR["gap"]] = 0.8; top_hi[:, PR["yaw"]] = np.pi
    assert _attach(core, 5, lo, hi, top_lo, top_hi) == (0, "")
    t = top_lo.copy(); t[1, PR["n_way"]] = 4.0; th = top_hi.copy(); th[1, PR["n_way"]] = 4.0
    assert _attach(core, 5, lo, hi, t, th) == (1, "ee_path n_way of robot 1: must be equal in the base and top boxes")
    t = top_lo.copy(); t[2, PR["qz"]] = 1e-3
    assert _attach(core, 5, lo, hi, t, top_hi) == (1, "ee_path qz of robot 2: must be equal in the base and top boxes")
    # gap lo 0.6 → 0.3: level 2 of 5 (0.45) is the first under T/2
    t = top_lo.copy(); t[0, PR["gap"]] = 0.3
    assert _attach(core, 5, lo, hi, t, top_hi) == (1, "ee_path level 2: gap of robot 0: lo must be >= T/2 = 0.500000 s")
    th = top_hi.copy(); th[3, PR["yaw"]] = 4.0   # yaw hi 1 → 4: level 3 of 4 (4.0) leaves [-pi, pi]
    assert _attach(core, 4, lo, hi, top_lo, th) == (1, "ee_path level 3: yaw of robot 3: bounds must lie in [-pi, pi]")


# ---------------------------------------------------------------------------------------------------------------------- closed_loop
DRAW = dict(seed=3, n=4, tau_first=(0.3, 0.5), gap=(0.6, 0.8), x=(0.4, 0.6), y=(-0.1, 0.1), z=(0.35, 0.45), yaw=(-0.5, 0.5), quat=(0.5, -0.5, 0.5, -0.5))


@pytest.mark.parametrize("bad,match", [
    ([1], "ee_path_draw must be None or dict"), (dict(DRAW, foo=1), "ee_path_draw must be None or dict"), (dict(DRAW, n=0), r"n must be an integer in \[1, 32\]"),
    (dict(DRAW, n=33), "n must be"), (dict(DRAW, n=2.0), "n must be"), ({k: v for k, v in DRAW.items() if k != "gap"}, r"needs gap=\(lo, hi\)"),
    ({k: v for k, v in DRAW.items() if k != "x"}, r"needs x=\(lo, hi\)"), (dict(DRAW, tau_first=(0.0, 0.5)), "tau_first lo must be > 0"),
    (dict(DRAW, gap=(0.4, 0.8)), "gap lo must be >= time_horizon / 2 = 0.5 s"), (dict(DRAW, yaw=(-4.0, 0.0)), r"yaw bounds must lie in \[-pi, pi\]"),
    (dict(DRAW, x=(0.6, 0.4)), "finite with lo <= hi"), (dict(DRAW, x=(np.zeros(3), 1.0)), "scalars or"), (dict(DRAW, seed=-1), "seed must be"),
    (dict(DRAW, quat=(0, 0, 0, 2.0)), "unit norm"), (dict(DRAW, n=32, gap=(0.6, 1e299)), r"tau_first hi \+ \(n - 1\) gap hi must be <= 1e300"), ({k: v for k, v in DRAW.items() if k != "quat"}, r"quat must be \[4\]"), (dict(DRAW, quat=np.ones((3, 4)) / 2), "quat must be"),
])
def test_a_malformed_ee_path_draw_raises_before_any_solver_call(bad, match):
    s = _fake_solver()
    with pytest.raises(ValueError, match=match):
        closed_loop.run(s, duration=0.02, ee_path_draw=bad)
    assert s.mock_calls == []


def test_drawn_paths_share_the_end_effector_refusals():
    s = types.SimpleNamespace(batch=B, time_horizon=1.0)
    with pytest.raises(ValueError, match="drawn spawn yaw cannot go with ee_path commands to world-frame robots"):
        closed_loop.run(s, duration=0.02, ee_path_draw=DRAW, spawn=dict(yaw=(-1.0, 1.0)))
    with pytest.raises(ValueError, match="at=\"here\" cannot go with ee_path commands to world-frame robots"):
        closed_loop.run(s, duration=0.02, ee_path_draw=DRAW, respawn=dict(every=0.01, at="here"))
    for kw in (dict(spawn=dict(yaw=(-1.0, 1.0))), dict(respawn=dict(every=0.01, at="here"))):   # heading-frame robots pass the spec checks
        with pytest.raises(AttributeError):
            closed_loop.run(s, duration=0.02, ee_path_draw=DRAW, ee_frame="heading", **kw)


def test_a_curriculum_top_box_for_the_paths_is_checked():
    s = _fake_solver(); run = dict(respawn=dict(every=0.2), ee_path_draw=DRAW)
    for top, match in ((dict(n=5), "top box's fields"), (dict(seed=1), "top box's fields"), (dict(quat=(0, 0, 0, 1.0)), "quat must equal the run's"),
                       (dict(gap=(0.1, 0.8)), "gap lo must be >= time_horizon / 2"), (dict(x=(0.7, 0.6)), "finite with lo <= hi")):
        with pytest.raises(ValueError, match=match):
            closed_loop.run(s, duration=0.02, curriculum=dict(levels=3, ee_path_draw=top), **run)
    with pytest.raises(ValueError, match="needs the run's own ee_path_draw"):
        closed_loop.run(s, duration=0.02, respawn=dict(every=0.2), curriculum=dict(levels=3, ee_path_draw=dict(x=(0, 1))))
    assert s.mock_calls == []


def _run_calls(**kw):
    import torch
    s = _fake_solver(); log = []
    for name in ("get_ee_paths", "set_ee_paths", "timeline_get_ranges", "timeline_set_ranges", "timeline_sample_dev", "ee_path_get_ranges", "ee_path_set_ranges",
                 "ee_path_sample_dev", "curriculum_draw"):
        setattr(s, name, mock.Mock())
    s.get_ee_paths.return_value = None; s.timeline_get_ranges.return_value = None; s.ee_path_get_ranges.return_value = None
    with mock.patch.object(torch.cuda, "Stream", _FakeStream), mock.patch.object(torch.cuda, "stream", lambda st: contextlib.nullcontext()):
        closed_loop.run(s, **dict(dict(duration=0.02, torch_device="cpu", gait="trot"), **kw))
    return s, [c[0] for c in s.mock_calls]


def test_the_draw_is_the_last_of_the_episodes_beginning_and_the_ranges_are_cleared_before_the_table(monkeypatch):
    monkeypatch.setattr(closed_loop.Session, "finish", lambda self: {})
    tl = dict(n=2, t_first=(0.0, 0.1), gap=(0.1, 0.2))
    s, calls = _run_calls(ee_path_draw=DRAW, timeline=tl, ee_paths=[(np.array([0.5, 1.2]), np.tile([0.5, 0.1, 0.4, 0.5, -0.5, 0.5, -0.5], (2, 1)))])
    first = calls.index("target_trajectories_dev")
    assert calls[:first].count("ee_path_sample_dev") == 1 and calls.index("timeline_sample_dev") < calls.index("ee_path_sample_dev") < first
    assert calls.index("gait_dev_reset") < calls.index("ee_path_sample_dev") and calls.count("ee_path_sample_dev") == 1
    assert calls.index("set_ee_paths") < calls.index("ee_path_get_ranges") < calls.index("ee_path_set_ranges")   # the table first, then the ranges
    tail = calls[calls.index("gait_dev_stop"):]
    assert tail == ["gait_dev_stop", "ee_path_set_ranges", "timeline_set_ranges", "set_ee_paths"]   # cleared, then the table restored
    (lo, hi, seed), _ = s.ee_path_set_ranges.call_args_list[0]
    assert seed == 3 and lo.shape == (B, W) and np.all(lo[:, PR["n_way"]] == 4) and np.all(hi[:, PR["n_way"]] == 4)
    assert np.all(lo[:, PR["gap"]] == 0.6) and np.all(hi[:, PR["yaw"]] == 0.5) and np.all(lo[:, 7:] == [0.5, -0.5, 0.5, -0.5]) and np.all(lo[:, 7:] == hi[:, 7:])
    assert s.ee_path_set_ranges.call_args_list[1][0] == (None,)
    mask, idx = s.ee_path_sample_dev.call_args[0][:2]
    assert mask.tolist() == [1] * B and idx.tolist() == [0] * B and tuple(s.ee_path_sample_dev.call_args[0][2].shape) == (B, PMAX, 8)
    # the path rows go to every target call
    assert all(c.kwargs.get("path_state") is not None for c in s.target_trajectories_dev.call_args_list)


def test_without_ee_path_draw_the_calls_are_the_parents():
    _, calls = _run_calls()
    assert calls == _parent_calls()


def test_bindings_and_header_agree():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name
    assert "#define QMB200_EE_PATH_RANGES %d" % W in h and W == 11 and len(_lib.EE_PATH_RANGES_LAYOUT) == W
    assert "#define QMB200_CURRICULUM_EE_PATH 3" in h and _lib.CURRICULUM_KINDS.index("ee_path") == 3
    assert "#define QMB200_STATE_BLOCKS 33" in h   # no snapshot block: the drawn rows are library rows, the robot's path row is the loop's
    api = open(os.path.join(CSRC, "kernels", "ee_path_draw_api.cuh")).read()
    assert "0x%016xull" % int(DOMAIN) in api
    others = [re.search(r"_DOMAIN = (0x[0-9a-f]+)ull", open(os.path.join(CSRC, "kernels", f)).read()).group(1) for f in ("episode_api.cuh", "spawn_api.cuh", "timeline_api.cuh")]
    assert "0x%016x" % int(DOMAIN) not in others


def test_the_sampler_and_the_curriculum_update_compile_for_sm90a_without_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    for src, kernel in (("ee_path_draw_kernel.cu", "ee_path_sample_kernel"), ("curriculum_kernel.cu", "curriculum_update_kernel")):
        obj, err = _resources(nvcc, src, tmp_path)
        m = re.search(r"Function properties for (\w*%s\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads" % kernel, err)
        assert m and m.groups()[1:] == ("0", "0", "0"), err
        if os.path.exists(cuobjdump):
            sass = subprocess.run([cuobjdump, "-sass", "-fun", m.group(1), obj], capture_output=True, text=True, check=True).stdout
            assert kernel in sass and not re.search(r"\b(LDL|STL)\b", sass)
