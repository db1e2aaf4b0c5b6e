"""Per-episode command timelines on the host, no GPU (DESIGN.md §4.14): the draw core compiled with g++ (tests/timeline_host.cpp) against its numpy
statement (tests/_timeline_twin.py), the distribution of its choices, the range check, closed_loop.run(timeline=...) validation and its ranges on a fake
Solver, the bindings and the sampler's resources."""
import ctypes as C
import os
import re
import shutil
import subprocess
import types
from unittest import mock

import numpy as np
import pytest

import _timeline_twin as tw
from qm_control_b200 import _lib, closed_loop
from qm_control_b200.interface import gait_template_names

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
TL = {n: i for i, n in enumerate(_lib.TIMELINE_LAYOUT)}
NAMES = ("qmb200_timeline_set_ranges", "qmb200_timeline_get_ranges", "qmb200_timeline_sample", "qmb200_timeline_sample_dev", "qmb200_timeline_draw",
         "qmb200_gait_dev_get_commands")


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("timeline") / "libtimelinehost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-I" + CSRC,
                           "-o", lib_path, os.path.join(ROOT, "tests", "timeline_host.cpp")])
    return C.CDLL(lib_path)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _rows(core, lo, hi, seed, robot, episode, n):
    m = len(lo); lo = np.ascontiguousarray(lo, dtype=np.float64); hi = np.ascontiguousarray(hi, dtype=np.float64)
    seed, robot, episode = (np.ascontiguousarray(a, dtype=np.uint64) for a in (seed, robot, episode))
    out = np.zeros((m, n, _lib.TIMELINE_CMD)); core.tl_rows(C.c_int(m), C.c_int(n), _ptr(seed), _ptr(robot), _ptr(episode), _ptr(lo), _ptr(hi), _ptr(out))
    return out


def _ranges(rng, m):
    """valid ranges covering the corners: fixed columns holding -0.0, p_gait 0 and 1, single-bit and 12-bit masks, zero weights"""
    lo = np.zeros((m, _lib.TIMELINE)); hi = np.zeros_like(lo)
    lo[:, TL["t_first"]] = rng.uniform(5.0, 10.0, m); hi[:, TL["t_first"]] = lo[:, TL["t_first"]] + rng.choice([0.0, 0.5], m)
    lo[:, TL["gap"]] = rng.choice([0.0, 0.01, 0.2], m); hi[:, TL["gap"]] = lo[:, TL["gap"]] + rng.choice([0.0, 0.3], m)
    p = rng.choice([0.0, 1.0, 0.5, rng.uniform()], m); lo[:, TL["p_gait"]] = hi[:, TL["p_gait"]] = p
    mask = np.where(rng.uniform(size=m) < 0.3, 1 << rng.integers(0, 32, m), np.where(rng.uniform(size=m) < 0.5, 0xFFF, rng.integers(1, 1 << 32, m)))
    lo[:, TL["gait_set"]] = hi[:, TL["gait_set"]] = mask.astype(np.float64)
    w = rng.uniform(0.0, 2.0, (m, 4)) * (rng.uniform(size=(m, 4)) < 0.7); w[w.sum(1) == 0, 1] = 1.0
    lo[:, 4:8] = hi[:, 4:8] = w
    for c in range(8, 18):
        lo[:, c] = rng.uniform(-1.0, 1.0, m); fixed = rng.uniform(size=m) < 0.4
        hi[:, c] = np.where(fixed, lo[:, c], lo[:, c] + rng.uniform(0.0, 1.0, m))
        z = fixed & (rng.uniform(size=m) < 0.3); lo[z, c] = hi[z, c] = -0.0
    q = rng.normal(size=(m, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True); q[::7] = [-0.0, 0.0, -0.0, 1.0]
    lo[:, 18:22] = hi[:, 18:22] = q
    return lo, hi


def _keys(rng, m):
    seed = rng.integers(0, 2 ** 63, m, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, m, dtype=np.uint64)
    return seed, rng.integers(0, 1 << 20, m).astype(np.uint64), rng.integers(0, 1 << 31, m).astype(np.uint64)


@pytest.mark.parametrize("n", [1, 4, 16])
def test_core_equals_the_numpy_statement_bit_for_bit(core, n):
    rng = np.random.default_rng(100 + n); m = 3000
    lo, hi = _ranges(rng, m); seed, robot, _ = _keys(rng, m)
    for episode in (np.zeros(m, dtype=np.uint64), rng.integers(0, 1 << 31, m).astype(np.uint64), np.full(m, 2 ** 64 - 1, dtype=np.uint64)):
        got = _rows(core, lo, hi, seed, robot, episode, n)
        assert got.tobytes() == tw.rows(lo, hi, seed, robot, episode, n).tobytes()   # byte for byte: NaN bits and -0.0 included


def test_times_sorted_choices_masked_and_frequencies_as_weighted(core):
    rng = np.random.default_rng(3); m, n = 4000, 16
    lo, hi = _ranges(rng, m); seed, robot, episode = _keys(rng, m)
    r = _rows(core, lo, hi, seed, robot, episode, n)
    assert np.all(np.diff(r[:, :, 0], axis=1) >= 0.0)
    tmpl = r[:, :, 1].astype(int); mask = lo[:, TL["gait_set"]].astype(np.int64)
    assert np.all((tmpl == -1) | ((mask[:, None] >> np.maximum(tmpl, 0)) & 1 == 1))
    p = lo[:, TL["p_gait"]]; assert np.all(tmpl[p == 0.0] == -1) and np.all(tmpl[p == 1.0] >= 0)
    kind = np.select([~np.isnan(r[:, :, 2]), r[:, :, 6] == 1, r[:, :, 6] == 2], [1, 2, 3], 0)
    w = lo[:, 4:8]; assert np.all(np.take_along_axis(w, kind, axis=1) > 0.0)
    # one robot's ranges, 20000 draws (robots): each kind and each template at its weight's frequency within 5 sigma
    N = 20000; lo1 = np.tile(lo[0], (N, 1)); lo1[:, TL["p_gait"]] = 0.4; lo1[:, TL["gait_set"]] = 0b101101; lo1[:, 4:8] = [1.0, 0.0, 2.0, 5.0]; hi1 = lo1.copy()
    r = _rows(core, lo1, hi1, np.full(N, 9), np.arange(N), np.zeros(N), 1)[:, 0]
    kind = np.select([~np.isnan(r[:, 2]), r[:, 6] == 1, r[:, 6] == 2], [1, 2, 3], 0)
    for k, pk in enumerate(np.array([1.0, 0.0, 2.0, 5.0]) / 8.0):
        assert abs(np.mean(kind == k) - pk) <= 5 * np.sqrt(pk * (1 - pk) / N) + 1e-12, k
    t = r[:, 1].astype(int); assert abs(np.mean(t >= 0) - 0.4) <= 5 * np.sqrt(0.24 / N)
    for b in (0, 2, 3, 5):
        assert abs(np.mean(t[t >= 0] == b) - 0.25) <= 5 * np.sqrt(0.1875 / np.sum(t >= 0)), b
    assert set(np.unique(t)) == {-1, 0, 2, 3, 5}


def test_changing_one_weight_leaves_every_other_column(core):
    rng = np.random.default_rng(8); m = 500; lo, hi = _ranges(rng, m); lo[:, 4:8] = hi[:, 4:8] = 1.0; seed, robot, episode = _keys(rng, m)
    a = _rows(core, lo, hi, seed, robot, episode, 6); lo[:, 4] = hi[:, 4] = 1.5
    b = _rows(core, lo, hi, seed, robot, episode, 6)
    assert a[:, :, :2].tobytes() == b[:, :, :2].tobytes()   # times and templates
    same = np.select([~np.isnan(a[:, :, 2]), a[:, :, 6] == 1, a[:, :, 6] == 2], [1, 2, 3], 0) == np.select([~np.isnan(b[:, :, 2]), b[:, :, 6] == 1, b[:, :, 6] == 2], [1, 2, 3], 0)
    assert np.all(np.where(same[..., None], a[:, :, 2:] == b[:, :, 2:], True) | (np.isnan(a[:, :, 2:]) & np.isnan(b[:, :, 2:])))


def _check(core, lo, hi):
    msg = C.create_string_buffer(256); rc = core.tl_ranges_error(C.c_int(len(lo)), _ptr(np.ascontiguousarray(lo)), _ptr(np.ascontiguousarray(hi)), msg, 256)
    return rc, msg.value.decode()


def _valid(B=5):
    lo = np.zeros((B, _lib.TIMELINE)); lo[:, TL["t_first"]] = 10.0; lo[:, TL["w_none"]] = 1.0; lo[:, TL["ee_qw"]] = 1.0
    hi = lo.copy(); hi[:, TL["t_first"]] = 11.0; hi[:, TL["gap"]] = 0.5; hi[:, TL["cmd_vel_x"]] = 0.5
    return lo, hi


@pytest.mark.parametrize("field,lo_v,hi_v,why", [
    ("t_first", np.nan, 0.0, "bounds must be finite"), ("ee_x", 0.2, 0.1, "lo must be <= hi"), ("cmd_vel_y", -1.5e308, 1.5e308, "hi - lo must be finite"),
    ("gap", -0.01, 0.1, "lo must be >= 0"), ("p_gait", 0.1, 0.2, "must be fixed (lo == hi)"), ("gait_set", 1.0, 3.0, "must be fixed (lo == hi)"),
    ("w_cmd_vel", 0.0, 1.0, "must be fixed (lo == hi)"), ("ee_qx", 0.0, 0.1, "must be fixed (lo == hi)"), ("p_gait", 1.5, 1.5, "must lie in [0, 1]"),
    ("p_gait", -0.1, -0.1, "must lie in [0, 1]"), ("gait_set", 2.5, 2.5, "must be an integer in [0, 2^32)"), ("gait_set", 2.0 ** 32, 2.0 ** 32, "must be an integer in [0, 2^32)"),
    ("gait_set", -1.0, -1.0, "must be an integer in [0, 2^32)"), ("w_ee_goal", -1.0, -1.0, "must be >= 0")])
def test_range_check_names_the_field_and_the_robot(core, field, lo_v, hi_v, why):
    lo, hi = _valid()
    assert _check(core, lo, hi) == (0, "")
    lo[3, TL[field]] = lo_v; hi[3, TL[field]] = hi_v
    assert _check(core, lo, hi) == (1, "qmb200_timeline_set_ranges: %s of robot 3: %s" % (field, why))


@pytest.mark.parametrize("edit,why", [
    (dict(p_gait=0.5), "gait_set of robot 2: must be non-zero when p_gait > 0"), (dict(w_none=0.0), "weights of robot 2: must have a positive sum"),
    (dict(ee_qw=1.0 + 2e-9), "ee_quat of robot 2: must have unit norm (within 1e-9)"), (dict(ee_qw=0.0), "ee_quat of robot 2: must have unit norm (within 1e-9)")])
def test_row_rules_name_the_robot(core, edit, why):
    lo, hi = _valid()
    for k, v in edit.items():
        lo[2, TL[k]] = hi[2, TL[k]] = v
    assert _check(core, lo, hi) == (1, "qmb200_timeline_set_ranges: " + why)
    lo[2, TL["gait_set"]] = hi[2, TL["gait_set"]] = 2.0 ** 32 - 1; lo[2, TL["w_none"]] = hi[2, TL["w_none"]] = 1.0; lo[2, 18:22] = hi[2, 18:22] = [0.0, 0.0, 0.0, 1.0]
    assert _check(core, lo, hi) == (0, "")


# ---------------------------------------------------------------------------------------------------------------------------- closed_loop.run(timeline=...)
GOOD = dict(n=3, t_first=(0.1, 0.2), gap=(0.1, 0.3))


@pytest.mark.parametrize("bad,match", [
    ([0.1], "timeline must be None or dict"), (dict(GOOD, n=0), "n must be an integer >= 1"), (dict(GOOD, n=2.0), "n must be an integer"),
    (dict(n=3, gap=(0.1, 0.2)), "needs t_first"), (dict(GOOD, seed=-1), "seed must be an integer"), (dict(GOOD, foo=(0, 1)), "unknown timeline field 'foo'"),
    (dict(GOOD, cmd_vel_x=(1.0, 0.0)), "finite with lo <= hi"), (dict(GOOD, cmd_vel_x=0.5), "must be a pair"), (dict(GOOD, gap=(-0.1, 0.1)), "gap lo must be >= 0"),
    (dict(GOOD, ee_x=(np.zeros(3), 1.0)), "scalars or"), (dict(GOOD, p_gait=1.5, gaits=["trot"]), "p_gait must lie in"),
    (dict(GOOD, p_gait=0.5, gaits=["trot", "gallop"]), "unknown gait name"), (dict(GOOD, p_gait=0.5), "at least one gait"),
    (dict(GOOD, weights=dict(none=0.0)), "positive sum"), (dict(GOOD, weights=dict(cmd_vel=-1.0, none=2.0)), ">= 0"),
    (dict(GOOD, weights=dict(walk=1.0)), "weights must be dict"), (dict(GOOD, weights=dict(ee_cmd_vel=1.0)), "ee_cmd_vel needs ee_vx"),
    (dict(GOOD, weights=dict(ee_goal=1.0), ee_x=(0, 1), ee_y=(0, 1), ee_z=(0, 1)), "ee_goal needs ee_quat"),
    (dict(GOOD, weights=dict(ee_goal=1.0), ee_x=(0, 1), ee_y=(0, 1), ee_z=(0, 1), ee_quat=(0, 0, 0, 2.0)), "unit norm"),
    (dict(GOOD, p_gait=np.full(3, 0.5), gaits=["trot"]), r"scalar or \[4\]"),
    (dict(GOOD, weights=dict(ee_goal=1.0), ee_x=(0, 1), ee_y=(0, 1), ee_z=(0, 1), ee_quat=1.0), r"ee_quat must be \[4\] or \[4, 4\]")])
def test_closed_loop_rejects_a_malformed_timeline_before_any_solver_call(bad, match):
    s = mock.Mock(batch=4)
    with pytest.raises(ValueError, match=match):
        closed_loop.run(s, duration=0.02, gait="trot", timeline=bad)
    assert s.mock_calls == []


def test_closed_loop_rejects_conflicts_before_any_solver_call():
    s = mock.Mock(batch=4)
    with pytest.raises(ValueError, match="timeline and commands"):
        closed_loop.run(s, duration=0.02, timeline=GOOD, commands=dict(t=np.zeros((4, 1)), gait=[[None]] * 4))
    with pytest.raises(ValueError, match="unknown gait name"):
        closed_loop.run(s, duration=0.02, gait="gallop", timeline=GOOD)
    ee = dict(GOOD, weights=dict(ee_cmd_vel=1.0), ee_vx=(0, 0.1), ee_vy=(0, 0), ee_vz=(0, 0))
    with pytest.raises(ValueError, match="drawn spawn yaw"):
        closed_loop.run(s, duration=0.02, timeline=ee, spawn=dict(yaw=(-0.5, 0.5)))
    assert s.mock_calls == []
    closed_loop._spawn_spec(4, dict(yaw=(0.3, 0.3)), None, None, closed_loop._timeline_spec(4, "stance", ee, None)["gd"])   # a fixed yaw is fine


class _Stop(Exception):
    pass


def test_ranges_hold_the_fixed_columns_and_the_previous_ranges_come_back():
    B = 4; prev = dict(n=2, lo=np.ones((B, 22)), hi=np.ones((B, 22)), seed=5); st = dict(ranges=prev, told=None)

    def set_ranges(n=None, lo=None, hi=None, seed=0):
        if lo is not None and st["told"] is None:
            st["told"] = (n, lo.copy(), hi.copy(), seed); raise _Stop
        st["ranges"] = None if lo is None else dict(n=n, lo=lo, hi=hi, seed=seed)
    impl = dict(timeline_get_ranges=lambda: st["ranges"], timeline_set_ranges=set_ranges, gait_dev_set_templates=lambda names: names, gait_dev_stop=lambda: None)
    s = mock.Mock(spec=list(impl), batch=B, _cfg=types.SimpleNamespace(device=0))
    for name, f in impl.items():
        getattr(s, name).side_effect = f
    cmd = np.array([[0.1, 0.2, 0.0, 0.3]] * B); gaits = [["trot"], ["pace", "trot"], ["static_walk"], ["trot"]]
    spec = dict(seed=7, n=5, t_first=(0.1, [0.2, 0.3, 0.4, 0.5]), gap=(0.2, 0.2), p_gait=[0.0, 0.5, 1.0, 1.0], gaits=gaits, weights=dict(none=1.0, ee_goal=[0, 1, 2, 0]),
                cmd_vel_y=(-0.4, 0.4), ee_x=(0.5, 0.6), ee_y=(0.0, 0.0), ee_z=(0.3, 0.4), ee_quat=(0.0, 0.0, 0.0, 1.0))
    with pytest.raises(_Stop):
        closed_loop.run(s, duration=0.02, gait="trot", cmd_vel=cmd, t_start=10.0, timeline=spec)
    n, lo, hi, seed = st["told"]; ids = {nm: i for i, nm in enumerate(gait_template_names())}
    assert n == 5 and seed == 7
    np.testing.assert_array_equal(lo[:, TL["t_first"]], 10.1); np.testing.assert_array_equal(hi[:, TL["t_first"]], 10.0 + np.array([0.2, 0.3, 0.4, 0.5]))
    np.testing.assert_array_equal(lo[:, TL["gait_set"]], [sum(1 << ids[x] for x in g) for g in gaits]); np.testing.assert_array_equal(lo[:, TL["p_gait"]], [0.0, 0.5, 1.0, 1.0])
    np.testing.assert_array_equal(lo[:, 4:8], [[1, 0, 0, 0], [1, 0, 0, 1], [1, 0, 0, 2], [1, 0, 0, 0]])
    np.testing.assert_array_equal(lo[:, TL["cmd_vel_x"]], 0.1); np.testing.assert_array_equal(hi[:, TL["cmd_vel_y"]], 0.4); np.testing.assert_array_equal(lo[:, TL["cmd_yaw_rate"]], 0.3)
    np.testing.assert_array_equal(lo[:, TL["ee_qw"]], 1.0); np.testing.assert_array_equal(hi[:, TL["ee_z"]], 0.4); np.testing.assert_array_equal(lo[:, TL["ee_vx"]:TL["ee_vz"] + 1], 0.0)
    fixed = [c for c in range(22) if c not in (TL["t_first"], TL["cmd_vel_y"], TL["ee_x"], TL["ee_z"])]
    np.testing.assert_array_equal(lo[:, fixed], hi[:, fixed])
    assert st["ranges"]["seed"] == 5 and st["ranges"]["n"] == 2   # the previous ranges are back


def test_entry_points_are_bound_and_declared():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name
    assert "#define QMB200_TIMELINE 22" in h and len(_lib.TIMELINE_LAYOUT) == _lib.TIMELINE == 22
    assert "#define QMB200_TIMELINE_CMD 14" in h and len(_lib.TIMELINE_CMD_LAYOUT) == _lib.TIMELINE_CMD == 14
    # distinct from the plant draws' (episode_api.cuh), the spawns' (spawn_api.cuh) and the sensor noise's (state_est_api.cuh)
    assert tw.DOMAIN not in (np.uint64(0x6a09e667f3bcc909), np.uint64(0xbb67ae8584caa73b), np.uint64(0x9e3779b97f4a7c15))
    for f, c in (("episode_api.cuh", "0x6a09e667f3bcc909"), ("spawn_api.cuh", "0xbb67ae8584caa73b"), ("state_est_api.cuh", "0x9e3779b97f4a7c15"),
                 ("timeline_api.cuh", "%#x" % int(tw.DOMAIN))):
        assert c in open(os.path.join(CSRC, "kernels", f)).read(), f


def test_sampler_compiles_for_sm90a_without_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    obj = str(tmp_path / "timeline.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "kernels", "timeline_kernel.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    assert any("timeline_sample_kernel" in k for k in kernels), r.stderr
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == len(kernels) and all(f == ("0", "0", "0") for f in frames), r.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if os.path.exists(cuobjdump):
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
        assert not re.search(r"\b(LDL|STL)\b", sass)
