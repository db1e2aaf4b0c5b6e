"""End-effector paths on the host, no GPU (DESIGN.md §4.20): the target front-end's path branch compiled with g++ (tests/ee_path_host.cpp, the function
ctrl_target_kernel runs) against an independent numpy statement on 1e5 robots; its agreement with the goal kind on the start tick, with the world frame
at the origin, and its equivariance; the table's check; the gait core's path rows against a Python statement; the bindings and the kernels' resources;
closed_loop's ee_paths / ee_path spec, refusals and calls on a fake Solver."""
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
from scipy.spatial.transform import Rotation

from test_ee_frame_cpu import COM_HEIGHT, DISP_VEL, QJ, ROT_VEL, T_TARGET, h_from_world, h_to_world, _resources
from test_gait_dev_cpu import B, _FakeStream, _fake_solver, _parent_calls
from qm_control_b200 import _lib, closed_loop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
NX, KMAX, TD, PMAX, PS = _lib.NX, _lib.KMAX, _lib.TARGET, _lib.EE_PATH_MAX, _lib.EE_PATH_STATE
START, FOLLOW = _lib.TARGET_EE_PATH, _lib.TARGET_EE_PATH_FOLLOW
OFFSET = np.array([0.52, 0.09])


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("ee_path") / "libeepathhost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include",
                           "-I" + CSRC, "-o", lib_path, os.path.join(ROOT, "tests", "ee_path_host.cpp")])
    lib = C.CDLL(lib_path)
    lib.eep_target.argtypes = [C.c_int] + [C.c_void_p] * 10 + [C.c_int] + [C.c_void_p] * 5
    lib.eep_paths_error.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_char_p, C.c_int]
    lib.eep_check.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_void_p]
    lib.eep_steps.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 12
    assert (lib.eep_kmax(), lib.eep_target_dim(), lib.eep_path_max(), lib.eep_path_state()) == (KMAX, TD, PMAX, PS)
    return lib


def _c(a, dtype=np.float64):
    return np.ascontiguousarray(a, dtype=dtype)


def host_target(lib, kind, frame, cmd, t, x, ee, le, ps, n_way, way, fill=np.nan):
    """the host build on n robots → (n_target [n], tt [n, KMAX], ts [n, KMAX, TD], le [n, 7], ps [n, PS]); untouched rows keep `fill` (n_target -7)"""
    n = len(kind); prm = _c([COM_HEIGHT, DISP_VEL, ROT_VEL, T_TARGET])
    le, ps = _c(le).copy(), _c(ps).copy(); nt = np.full(n, -7, dtype=np.int32); tt = np.full((n, KMAX), fill); ts = np.full((n, KMAX, TD), fill)
    kind, frame, cmd, t, x, ee, n_way, way = _c(kind, np.int32), _c(frame, np.int32), _c(cmd), _c(t), _c(x), _c(ee), _c(n_way, np.int32), _c(way)
    lib.eep_target(n, prm.ctypes.data, _c(QJ).ctypes.data, kind.ctypes.data, frame.ctypes.data, cmd.ctypes.data, t.ctypes.data, x.ctypes.data, ee.ctypes.data,
                   le.ctypes.data, ps.ctypes.data, len(n_way), n_way.ctypes.data, way.ctypes.data, nt.ctypes.data, tt.ctypes.data, ts.ctypes.data)
    return nt, tt, ts, le, ps


# ---------------------------------------------------------------------------------------------------------------------- the numpy statement
def slerp(a, l, r):
    """poses at weight a [n] between poses l and r [n, 7]: a l + (1 - a) r and the Eigen slerp of the MPC's target interpolation; a == 1 gives l"""
    o = np.empty_like(l); o[:, :3] = a[:, None] * l[:, :3] + (1.0 - a[:, None]) * r[:, :3]
    ql, qr = l[:, 3:], r[:, 3:]; tq = 1.0 - a; d = np.sum(ql * qr, axis=1); ad = np.abs(d)
    lin = ad >= 1.0 - 2.220446049250313e-16
    th = np.arccos(np.minimum(ad, 1.0)); st = np.where(lin, 1.0, np.sin(th))
    s0 = np.where(lin, 1.0 - tq, np.sin((1.0 - tq) * th) / st); s1 = np.where(lin, tq, np.sin(tq * th) / st)
    s1 = np.where(d < 0.0, -s1, s1)
    o[:, 3:] = s0[:, None] * ql + s1[:, None] * qr
    return np.where((a == 1.0)[:, None], l, o)


def statement(kind, frame, cmd, t, x, ee, le, ps, n_way, way):
    """the path rule (DESIGN.md §4.20) for robots of kind START / FOLLOW → (written [n] bool, nt [n], tt [n, KMAX], ts [n, KMAX, TD], le, ps)"""
    n = len(t); le, ps = le.copy(), ps.copy(); hd = frame == 1; P = len(n_way)
    fi = np.where(kind == START, cmd[:, 0], ps[:, 0])
    valid = (fi >= 0) & (fi < P) & (np.floor(fi) == fi)
    p = np.where(valid, fi, 0).astype(int); nw = n_way[p]
    st = valid & (kind == START)
    ps[st] = np.c_[np.full(st.sum(), fi[st]), t[st], x[st][:, [6, 7, 9]], ee[st]]
    psi = x[:, 9]; c, s = np.cos(psi), np.sin(psi)
    off = np.where(hd[:, None], np.c_[c * 0.52 - s * 0.09, s * 0.52 + c * 0.09], OFFSET)
    W = way[p]                                                            # [n, PMAX, 8]
    def world(k):                                                         # waypoint k [n] of each robot's path in the world
        w = W[np.arange(n), np.clip(k, 0, PMAX - 1), 1:]
        return np.where(hd[:, None], h_to_world(ps[:, 2], ps[:, 3], ps[:, 4], w), w)
    g = world(nw - 1)                                                     # the final waypoint, a goal published on the start tick
    gl = np.where(hd[:, None], h_from_world(g[:, 0] - off[:, 0], g[:, 1] - off[:, 1], psi, g), g)
    le[st] = gl[st]
    t0 = ps[:, 1]
    after = (t0[:, None] + W[:, :, 0] > t[:, None]) & (np.arange(PMAX)[None, :] < nw[:, None])
    j = np.argmax(after, axis=1); live = valid & after.any(axis=1)
    tr = t0 + W[np.arange(n), j, 0]; tl = np.where(j == 0, t0, t0 + W[np.arange(n), np.maximum(j - 1, 0), 0])
    left = np.where((j == 0)[:, None], ps[:, 5:12], world(j - 1))
    a = np.minimum((tr - t) / np.where(tr > tl, tr - tl, 1.0), 1.0)
    e0 = slerp(a, left, world(j))
    m = np.minimum(nw - j, KMAX - 1)
    nt = 1 + m; tt = np.zeros((n, KMAX)); ts = np.zeros((n, KMAX, TD)); tt[:, 0] = t
    ts[:, 0, 6], ts[:, 0, 7] = x[:, 6], x[:, 7]; ts[:, 0, 30:37] = e0
    for k in range(1, KMAX):
        wk = world(j + k - 1)
        tt[:, k] = t0 + W[np.arange(n), np.clip(j + k - 1, 0, PMAX - 1), 0]
        ts[:, k, 6:8] = wk[:, :2] - off; ts[:, k, 30:37] = wk
    for k in range(KMAX):
        ts[:, k, 8] = COM_HEIGHT; ts[:, k, 9] = psi; ts[:, k, 12:30] = QJ
        out = k > m
        tt[out, k] = 0.0; ts[out, k] = 0.0
    return live, nt, tt, ts, le, ps


def table(P, seed, T=T_TARGET):
    """P random paths: 1 to 8 waypoints, first time in (0, 1], gaps in [T/2, 1.5 T], positions within 1 m, random orientations"""
    rng = np.random.default_rng(seed)
    n_way = rng.integers(1, 9, P).astype(np.int32); way = np.zeros((P, PMAX, 8))
    for p in range(P):
        k = n_way[p]
        way[p, :k, 0] = np.cumsum(np.r_[rng.uniform(0.05, 1.0), rng.uniform(0.5 * T, 1.5 * T, k - 1)])
        way[p, :k, 1:4] = rng.uniform(-1, 1, (k, 3)); way[p, :k, 4:8] = Rotation.random(k, random_state=seed + p).as_quat()
    return n_way, way


def robots(n, seed, n_way, way, origin=False):
    """n random path robots: kind START / FOLLOW, frame {0, 1}, indices mostly in the table (some outside or not integers), t before, inside and after
    each path, bases within ±20 m at unwrapped yaws within ±50 rad; origin: current and start bases at (0, 0, yaw 0)"""
    rng = np.random.default_rng(seed); P = len(n_way)
    kind = np.where(rng.uniform(size=n) < 0.3, START, FOLLOW).astype(np.int32); frame = rng.integers(0, 2, n).astype(np.int32)
    x = rng.uniform(-0.3, 0.3, (n, NX)); x[:, 6:8] = rng.uniform(-20, 20, (n, 2)); x[:, 8] = rng.uniform(0.3, 0.5, n); x[:, 9] = rng.uniform(-50, 50, n)
    ee = np.c_[x[:, 6:8] + rng.uniform(-1, 1, (n, 2)), rng.uniform(0.2, 0.7, n), Rotation.random(n, random_state=seed).as_quat()]
    le = np.c_[rng.uniform(0.3, 0.7, (n, 3)), Rotation.random(n, random_state=seed + 1).as_quat()]
    idx = rng.integers(0, P, n).astype(np.float64)
    bad = rng.uniform(size=n); idx[bad < 0.02] = -1.0; idx[(bad >= 0.02) & (bad < 0.04)] = P; idx[(bad >= 0.04) & (bad < 0.05)] += 0.5
    t0 = rng.uniform(0.0, 10.0, n)
    ps = np.c_[idx, t0, x[:, 6:8] + rng.uniform(-2, 2, (n, 2)), x[:, 9] + rng.uniform(-3, 3, n), ee[:, :3] + rng.uniform(-0.3, 0.3, (n, 3)),
               Rotation.random(n, random_state=seed + 2).as_quat()]
    span = way[np.clip(idx, 0, P - 1).astype(int), np.maximum(n_way[np.clip(idx, 0, P - 1).astype(int)] - 1, 0), 0]
    t = t0 + rng.uniform(-0.5, 1.0, n) * (span + 0.5)
    cmd = np.zeros((n, 7)); cmd[:, 0] = idx; cmd[:, 1:] = rng.uniform(-1, 1, (n, 6))   # ee[1:7] of a path row are not read
    st = kind == START
    t[st] = rng.uniform(0.0, 10.0, int(st.sum()))
    if origin:
        x[:, 6:8] = 0.0; x[:, 9] = 0.0; ps[:, 2:5] = 0.0
    return kind, frame, cmd, t, x, ee, le, ps


# ---------------------------------------------------------------------------------------------------------------------- the host build
def test_the_host_build_equals_the_path_rule_on_1e5_robots(host):
    n_way, way = table(40, 3)
    kind, frame, cmd, t, x, ee, le, ps = robots(100_000, 5, n_way, way)
    nt, tt, ts, le_out, ps_out = host_target(host, kind, frame, cmd, t, x, ee, le, ps, n_way, way)
    live, rn, rt, rs, rl, rp = statement(kind, frame, cmd, t, x, ee, le, ps, n_way, way)
    dead = ~live
    assert np.all(nt[dead] == -7) and np.all(np.isnan(tt[dead])) and np.all(np.isnan(ts[dead]))
    assert np.array_equal(nt[live], rn[live])
    np.testing.assert_allclose(tt[live], rt[live], rtol=0, atol=1e-12)
    np.testing.assert_allclose(ts[live], rs[live], rtol=0, atol=1e-12)
    np.testing.assert_allclose(le_out, rl, rtol=0, atol=1e-12)
    np.testing.assert_allclose(ps_out, rp, rtol=0, atol=0)
    # the draw covers every case, in both frames: starts, follows before / inside / after the path, 1 to 3 waypoint knots, indices outside the table
    st = kind == START; fi = np.where(st, cmd[:, 0], ps[:, 0]); outside = ~((fi >= 0) & (fi < len(n_way)) & (np.floor(fi) == fi))
    for f in (0, 1):
        for m in (st & live, ~st & live & (t < ps[:, 1]), ~st & ~live & ~outside, outside, live & (nt == 2), live & (nt == 3), live & (nt == 4)):
            assert np.count_nonzero(m & (frame == f)) > 200
    assert np.array_equal(le_out[outside], le[outside]) and np.array_equal(ps_out[outside], ps[outside])
    assert np.array_equal(le_out[~st], le[~st])   # a follow never moves the hold


def test_on_its_start_tick_a_one_waypoint_path_publishes_the_goal_bit_for_bit(host):
    n = 4000; rng = np.random.default_rng(8)
    _, frame, _, _, x, ee, le, ps = robots(n, 9, *table(4, 1))
    t = rng.uniform(20.0, 30.0, n)
    goal = np.c_[np.where(frame[:, None] == 1, rng.uniform(0.2, 0.8, (n, 3)), ee[:, :3] + rng.uniform(-0.5, 0.5, (n, 3))), Rotation.random(n, random_state=4).as_quat()]
    g = host_target(host, np.full(n, 2), frame, goal, t, x, ee, le, ps, [1], np.zeros((1, PMAX, 8)))
    tau = g[1][:, 1] - t
    assert np.array_equal(t + tau, g[1][:, 1])   # Sterbenz: the reach time's difference is exact
    way = np.zeros((n, PMAX, 8)); way[:, 0, 0] = tau; way[:, 0, 1:] = goal
    cmd = np.zeros((n, 7)); cmd[:, 0] = np.arange(n)
    p = host_target(host, np.full(n, START), frame, cmd, t, x, ee, le, ps, np.ones(n), way)
    for a, b in zip(g[:4], p[:4]):
        assert a.tobytes() == b.tobytes()
    assert np.array_equal(p[4][:, 0], np.arange(n)) and np.array_equal(p[4][:, 1], t) and np.array_equal(p[4][:, 5:12], ee)


def test_at_the_origin_a_heading_robot_is_a_world_robot_bit_for_bit(host):
    n_way, way = table(40, 13)
    kind, _, cmd, t, x, ee, le, ps = robots(20_000, 14, n_way, way, origin=True)
    n = len(t)
    w = host_target(host, kind, np.zeros(n), cmd, t, x, ee, le, ps, n_way, way); h = host_target(host, kind, np.ones(n), cmd, t, x, ee, le, ps, n_way, way)
    for a, b in zip(w[:3] + w[4:], h[:3] + h[4:]):
        assert a.tobytes() == b.tobytes()
    f = kind == FOLLOW   # a start's hold is the final waypoint in the world for a world robot, in the base target's frame for a heading robot
    assert w[3][f].tobytes() == h[3][f].tobytes()


def _apply(px, py, psi, ts):
    """the base pose P = (px, py, psi) [n] applied to target states ts [n, K, TD] stated at the origin"""
    out = ts.copy(); c, s = np.cos(psi)[:, None], np.sin(psi)[:, None]
    out[..., 6] = c * ts[..., 6] - s * ts[..., 7] + px[:, None]; out[..., 7] = s * ts[..., 6] + c * ts[..., 7] + py[:, None]; out[..., 9] = ts[..., 9] + psi[:, None]
    for k in range(ts.shape[1]):
        out[:, k, 30:37] = h_to_world(px, py, psi, ts[:, k, 30:37])
    return out


def test_the_path_rule_is_equivariant(host):
    n_way, way = table(40, 21)
    kind, _, cmd, t, x, ee, le, ps = robots(20_000, 22, n_way, way, origin=True)
    n = len(t); frame = np.ones(n, dtype=np.int32); x[:, 10:12] = 0.0
    rng = np.random.default_rng(23); px, py, psi = rng.uniform(-20, 20, n), rng.uniform(-20, 20, n), rng.uniform(-50, 50, n)
    xp = x.copy(); xp[:, 6] = px; xp[:, 7] = py; xp[:, 9] = psi
    psp = ps.copy(); psp[:, 2] = px; psp[:, 3] = py; psp[:, 4] = psi; psp[:, 5:12] = h_to_world(px, py, psi, ps[:, 5:12])
    o = host_target(host, kind, frame, cmd, t, x, ee, le, ps, n_way, way, fill=0.0)
    p = host_target(host, kind, frame, cmd, t, xp, h_to_world(px, py, psi, ee), le, psp, n_way, way, fill=0.0)
    assert np.array_equal(o[0], p[0])
    np.testing.assert_allclose(p[1], o[1], rtol=0, atol=1e-12)
    live = o[0] > 0; K = np.arange(KMAX)[None, :] < o[0][:, None]
    np.testing.assert_allclose(np.where(K[live][..., None], p[2][live], 0.0), np.where(K[live][..., None], _apply(px[live], py[live], psi[live], o[2][live]), 0.0),
                               rtol=0, atol=1e-12)
    np.testing.assert_allclose(p[3], o[3], rtol=0, atol=1e-12)   # the hold is body-relative
    np.testing.assert_allclose(p[4][:, 5:12], h_to_world(px, py, psi, o[4][:, 5:12]), rtol=0, atol=1e-12)


def _check(host, n_way, way, T=T_TARGET):
    buf = C.create_string_buffer(512)
    n = host.eep_paths_error(len(n_way), _c(n_way, np.int32).ctypes.data, _c(way).ctypes.data, T, buf, 512)
    return buf.value.decode() if n else ""


def test_the_table_check_names_the_path_and_the_waypoint(host):
    n_way, way = table(3, 31)
    assert _check(host, n_way, way) == "" and _check(host, [], np.zeros((0, PMAX, 8))) == ""
    cases = []
    for rule, edit, want in (
            ("non-finite", lambda w, n: w.__setitem__((2, 1, 3), np.nan), "path 2, waypoint 1: value 3 is not finite"),
            ("too few", lambda w, n: n.__setitem__(1, 0), "path 1 has 0 waypoints, not 1 to QMB200_EE_PATH_MAX (32)"),
            ("too many", lambda w, n: n.__setitem__(0, PMAX + 1), "path 0 has 33 waypoints"),
            ("tau_0 <= 0", lambda w, n: w.__setitem__((1, 0, 0), 0.0), "path 1, waypoint 0: its time must be > 0"),
            ("not increasing", lambda w, n: w.__setitem__((2, 1, 0), w[2, 0, 0]), "path 2, waypoint 1: its time is not after waypoint 0's"),
            ("gap", lambda w, n: w.__setitem__((2, 1, 0), w[2, 0, 0] + 0.49 * T_TARGET), "path 2, waypoint 1: its gap to waypoint 0 is under T/2"),
            ("quaternion", lambda w, n: w.__setitem__((0, 0, slice(4, 8)), w[0, 0, 4:8] * (1.0 + 3e-9)), "path 0, waypoint 0: its quaternion must have unit norm")):
        n2, w2 = n_way.copy(), way.copy(); n2[:] = [2, 3, 2]
        for p in range(3):
            w2[p, :3, 0] = [0.2, 0.8, 1.4]
        edit(w2, n2)
        msg = _check(host, n2, w2)
        assert msg.startswith("qmb200_set_ee_paths: " + want), (rule, msg)
        cases.append(rule)
    assert len(cases) == 7
    w3 = way.copy(); w3[0, 0, 4:8] = [0, 0, 0, 1.0 + 0.9e-9]; n3 = n_way.copy()
    assert _check(host, n3, w3) == ""   # within 1e-9 of 1


# ---------------------------------------------------------------------------------------------------------------------- the gait core
def test_the_command_check_takes_path_rows_only_with_a_table(host):
    rows = [(3, [2.0]), (3, [0.0]), (3, [4.0]), (3, [1.5]), (3, [-1.0]), (3, [np.nan]), (0, [0.0]), (-7, [0.0]), (-2, [0.0]), (1, [0.1, 0.0, 0.0]), (-1, [])]
    n = len(rows); kind = np.array([k for k, _ in rows], dtype=np.int32); ee = np.zeros((n, 7))
    for i, (_, v) in enumerate(rows):
        ee[i, :len(v)] = v
    tmpl = np.full(n, -1, dtype=np.int32); vel = np.full((n, 4), np.nan)
    def check(n_paths, v=vel):
        out = np.zeros(n, dtype=np.int32)
        host.eep_check(n, tmpl.ctypes.data, _c(v).ctypes.data, kind.ctypes.data, ee.ctypes.data, 1, n_paths, out.ctypes.data)
        return (out != 0).tolist()
    R = True
    assert check(-1) == [R, R, R, R, R, R, R, R, R, False, False]   # no table (the check's default): every path row, and kinds 0, -7, -2 rejected
    assert check(0) == check(-1)
    assert check(4) == [False, False, R, R, R, R, R, R, R, False, False]
    assert check(4, np.zeros((n, 4)))[:2] == [R, R]   # a path row with a cmd_vel


def _gait_statement(t, t_cmd, kind, ee, pend_set, pend_kind, pend_ee):
    """the sources, target kinds and cmd rows of path / goal / ee_cmd_vel rows and pending rows (DESIGN.md §4.8, §4.20), one robot at a time"""
    Bn, n_ticks = t_cmd.shape[0], len(t)
    cmd, tk, src = np.zeros((n_ticks, Bn, 7)), np.zeros((n_ticks, Bn), dtype=np.int32), np.zeros((n_ticks, Bn), dtype=np.int32)
    for b in range(Bn):
        row, s, cur, pend = np.zeros(7), 0, 0, None
        for k in range(n_ticks):
            if pend_set[k, b]:
                pend = (pend_kind[k, b], pend_ee[k, b])
            due = []
            while cur < t_cmd.shape[1] and t_cmd[b, cur] <= t[k]:
                due.append((kind[b, cur], ee[b, cur])); cur += 1
            if pend is not None:
                due.append(pend); pend = None
            applied = -1
            for kd, e in due:
                if kd < 0:
                    continue
                m = {1: 3, 2: 7, 3: 1}[kd]; row[:m] = e[:m]; applied = kd
            if applied >= 0:
                s = applied
            tk[k, b] = applied if applied in (2, 3) else (-1 if s == 2 else 4 if s == 3 else s)
            cmd[k, b], src[k, b] = row, s
    return cmd, tk, src


def test_the_gait_core_applies_path_rows_as_the_statement(host):
    rng = np.random.default_rng(41); Bn, n_cmd, n_ticks = 64, 6, 60
    t = 0.5 + 0.01 * np.arange(n_ticks)
    t_cmd = np.sort(rng.uniform(0.45, 1.2, (Bn, n_cmd)), axis=1)
    kind = rng.choice([-1, 1, 2, 3], (Bn, n_cmd)).astype(np.int32)
    ee = np.zeros((Bn, n_cmd, 7)); ee[..., :3] = rng.uniform(-1, 1, (Bn, n_cmd, 3)); ee[..., 3:] = [0, 0, 0, 1.0]
    ee[kind == 3, 0] = rng.integers(0, 5, int((kind == 3).sum()))
    vel = np.full((Bn, n_cmd, 4), np.nan)
    pend_set = (rng.uniform(size=(n_ticks, Bn)) < 0.05).astype(np.int32); pend_kind = rng.choice([1, 2, 3], (n_ticks, Bn)).astype(np.int32)
    pend_ee = np.zeros((n_ticks, Bn, 7)); pend_ee[..., :3] = rng.uniform(-1, 1, (n_ticks, Bn, 3)); pend_ee[..., 3:] = [0, 0, 0, 1.0]
    pend_ee[pend_kind == 3, 0] = rng.integers(0, 5, int((pend_kind == 3).sum()))
    cmd = np.zeros((n_ticks, Bn, 7)); tk, src, st = (np.zeros((n_ticks, Bn), dtype=np.int32) for _ in range(3))
    host.eep_steps(Bn, n_ticks, _c(t).ctypes.data, n_cmd, _c(t_cmd).ctypes.data, _c(kind, np.int32).ctypes.data, _c(ee).ctypes.data, _c(vel).ctypes.data,
                   pend_set.ctypes.data, pend_kind.ctypes.data, _c(pend_ee).ctypes.data, _c(np.full((n_ticks, Bn, 4), np.nan)).ctypes.data, cmd.ctypes.data,
                   tk.ctypes.data, src.ctypes.data, st.ctypes.data)
    assert np.all(st == 0)
    rc, rk, rs = _gait_statement(t, t_cmd, kind, ee, pend_set, pend_kind, pend_ee)
    assert np.array_equal(tk, rk) and np.array_equal(src, rs) and np.array_equal(cmd, rc)
    assert np.count_nonzero(tk == START) > 50 and np.count_nonzero(tk == FOLLOW) > 500   # both path kinds occur


# ---------------------------------------------------------------------------------------------------------------------- bindings, resources
def test_bindings_and_header_agree():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name, value in (("QMB200_TARGET_EE_PATH", START), ("QMB200_TARGET_EE_PATH_FOLLOW", FOLLOW), ("QMB200_EE_PATH_MAX", PMAX), ("QMB200_EE_PATH_STATE", PS)):
        assert re.search(r"#define %s %d\b" % (name, value), h), name
    assert (START, FOLLOW, PMAX, PS) == (3, 4, 32, 12)
    P, I32 = C.c_void_p, C.c_int32
    assert _lib.PROTOTYPES["qmb200_set_ee_paths"] == (I32, [P, I32, P, P]) and _lib.PROTOTYPES["qmb200_get_ee_paths"] == (I32, [P] * 4)
    assert _lib.PROTOTYPES["qmb200_target_trajectories_path"] == (I32, [P] * 11) and _lib.PROTOTYPES["qmb200_target_trajectories_path_dev"] == (I32, [P] * 12)
    for f in ("qmb200_set_ee_paths", "qmb200_get_ee_paths", "qmb200_target_trajectories_path", "qmb200_target_trajectories_path_dev"):
        assert re.search(r"int %s\(" % f, h), f
    assert int(re.search(r"#define QMB200_STATE_BLOCKS (\d+)", h).group(1)) == 33   # no snapshot block: the path rows are the loop's own


def test_the_target_and_gait_kernels_compile_for_sm90a_without_spills(tmp_path):
    """ctrl_target_kernel keeps the parent's one 40-byte frame (the world-frame cmd_vel rotation's sincos slow path); the path branch adds none.  The
    gait step keeps its 840-byte frame (the working copy of a robot's schedule) and the command kernel none."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    for src, kernels in (("ctrl_kernels.cu", (("ctrl_target_kernel", "40"),)), ("gait_kernel.cu", (("gait_step_kernel", "840"), ("gait_command_kernel", "0")))):
        _, err = _resources(nvcc, src, tmp_path)
        for kernel, frame in kernels:
            m = re.search(r"Function properties for (\w*%s\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads" % kernel, err)
            assert m and m.groups()[1:] == (frame, "0", "0"), err


# ---------------------------------------------------------------------------------------------------------------------- closed_loop
SQUARE = [(np.array([0.5, 1.0, 1.5, 2.0]), np.array([[0.62, 0.09, 0.44, 0.5, -0.5, 0.5, -0.5], [0.62, 0.19, 0.44, 0.5, -0.5, 0.5, -0.5],
                                                      [0.52, 0.19, 0.44, 0.5, -0.5, 0.5, -0.5], [0.52, 0.09, 0.44, 0.5, -0.5, 0.5, -0.5]]))]


def _path_commands(n=B, path=0):
    return dict(t=np.zeros((n, 1)), gait=[[None]] * n, ee_path=np.full((n, 1), path))


@pytest.mark.parametrize("ee_paths, match", [
    ("square", "ee_paths must be"), ([], "ee_paths must be"), ([(np.array([0.5]),)], r"ee_paths\[0\] must be a pair"),
    ([(np.array([0.5, 1.0]), np.zeros((2, 6)))], r"ee_paths\[0\] must be \(t \[n\], pose \[n, 7\]\)"),
    ([(np.arange(1, 34) * 1.0, np.tile([0, 0, 0, 0, 0, 0, 1.0], (33, 1)))], "1 <= n <= 32"),
    ([(np.array([0.0]), np.array([[0, 0, 0, 0, 0, 0, 1.0]]))], "must be > 0 and strictly increasing"),
    ([(np.array([0.5, 0.5]), np.tile([0, 0, 0, 0, 0, 0, 1.0], (2, 1)))], "strictly increasing"),
    ([(np.array([0.5, 0.9]), np.tile([0, 0, 0, 0, 0, 0, 1.0], (2, 1)))], "at least time_horizon / 2"),
    ([(np.array([0.5]), np.array([[0, 0, np.nan, 0, 0, 0, 1.0]]))], "must be finite"),
    ([(np.array([0.5]), np.array([[0, 0, 0, 0, 0, 0, 1.1]]))], "unit norm")])
def test_a_malformed_ee_paths_raises_before_any_solver_call(ee_paths, match):
    s = _fake_solver()
    with pytest.raises(ValueError, match=match):
        closed_loop.run(s, duration=0.02, ee_paths=ee_paths)
    with pytest.raises(ValueError, match=match):
        closed_loop.Session(s, 0.02, ee_paths=ee_paths)
    assert s.mock_calls == []


def test_malformed_ee_path_commands_raise_before_any_solver_call():
    s = _fake_solver()
    for kw, match in ((dict(commands=_path_commands()), r"ids must lie in \[-1, 0\)"), (dict(commands=_path_commands(path=1), ee_paths=SQUARE), r"in \[-1, 1\)"),
                      (dict(commands=dict(_path_commands(), ee_path=np.full((B, 1), 0.0)), ee_paths=SQUARE), "integer path ids"),
                      (dict(commands=dict(_path_commands(), ee_path=np.full((B, 2), 0)), ee_paths=SQUARE), "integer path ids"),
                      (dict(commands=dict(_path_commands(), ee_path=np.full((B, 1), -2)), ee_paths=SQUARE), "integer path ids"),
                      (dict(commands=dict(_path_commands(), ee_cmd_vel=np.full((B, 1, 3), 0.1)), ee_paths=SQUARE), "at most one of cmd_vel, ee_goal, ee_cmd_vel and ee_path")):
        with pytest.raises(ValueError, match=match):
            closed_loop.run(s, duration=0.02, **kw)
    assert s.mock_calls == []


def test_path_commands_to_world_robots_share_the_refusals_and_are_named_in_them():
    s = types.SimpleNamespace(batch=B, time_horizon=1.0); yaw = dict(yaw=(-np.pi, np.pi))
    with pytest.raises(ValueError, match="drawn spawn yaw cannot go with ee_path commands to world-frame robots"):
        closed_loop.run(s, duration=0.02, commands=_path_commands(), ee_paths=SQUARE, spawn=yaw)
    with pytest.raises(ValueError, match="at=\"here\" cannot go with ee_path commands to world-frame robots"):
        closed_loop.run(s, duration=0.02, commands=_path_commands(), ee_paths=SQUARE, respawn=dict(at="here", every=0.1))
    mixed = dict(t=np.zeros((B, 2)), gait=[[None, None]] * B, ee_path=np.array([[0, -1]] * B), ee_goal=np.full((B, 2, 7), np.nan))
    mixed["ee_goal"][:, 1] = [0.5, 0.0, 0.5, 0.0, 0.0, 0.0, 1.0]
    with pytest.raises(ValueError, match="drawn spawn yaw cannot go with ee_goal / ee_cmd_vel / ee_path commands to world-frame robots"):
        closed_loop.run(s, duration=0.02, commands=mixed, ee_paths=SQUARE, spawn=yaw)
    only_goal = dict(mixed, ee_path=np.array([[-1, -1]] + [[0, -1]] * (B - 1)))   # robot 0: a goal only; the others: a path and a goal
    with pytest.raises(ValueError, match="drawn spawn yaw cannot go with ee_goal / ee_cmd_vel commands to world-frame robots"):   # robot 0 draws, the rest is fixed
        closed_loop.run(s, duration=0.02, commands=only_goal, ee_paths=SQUARE, spawn=dict(yaw=(np.array([-1.0] + [0.2] * (B - 1)), np.array([1.0] + [0.2] * (B - 1)))))
    closed_loop._run_specs(s, False, dict(closed_loop.RUN_DEFAULTS, commands=_path_commands(), ee_paths=SQUARE, spawn=yaw, ee_frame="heading"))   # lifted
    solver = _fake_solver()
    for name in ("robot_image_save", "robot_image_restore_dev", "robot_image_clear", "fall_detect_dev", "spawn_here_dev", "spawn_place_dev"):
        setattr(solver, name, mock.Mock())
    here = closed_loop.Session(solver, 0.03, gait="trot", steer=True, respawn=dict(every=0.01, at="here"), ee_paths=SQUARE)
    with pytest.raises(ValueError, match="Session.command: ee_path to world-frame robots cannot go with a drawn spawn yaw or a restart \"here\""):
        here.command(np.ones(B), ee_path=np.zeros(B, dtype=np.int32))
    with pytest.raises(ValueError, match="Session.command: ee_goal / ee_cmd_vel / ee_path to world-frame robots cannot go"):
        here.command(np.ones(B), ee_path=np.zeros(B, dtype=np.int32), ee_cmd_vel=np.zeros((B, 3)))
    plain = closed_loop.Session(solver, 0.03, gait="trot", steer=True)
    with pytest.raises(ValueError, match="ee_path needs the session's ee_paths"):
        plain.command(np.ones(B), ee_path=np.zeros(B, dtype=np.int32))
    hd = closed_loop.Session(solver, 0.03, gait="trot", steer=True, ee_paths=SQUARE)
    with pytest.raises(ValueError, match="integer path ids"):
        hd.command(np.ones(B), ee_path=np.zeros(B))
    with pytest.raises(ValueError, match="ee_path must have shape"):
        hd.command(np.ones(B), ee_path=np.zeros(B + 1, dtype=np.int32))
    assert solver.mock_calls == []


def test_a_path_call_needs_per_robot_kinds():
    from qm_control_b200.interface import Solver
    fake = types.SimpleNamespace(_call=mock.Mock())
    with pytest.raises(ValueError, match="path_state needs per-robot kinds"):
        Solver.target_trajectories_dev(fake, 0, None, None, None, None, None, None, None, None, path_state=np.zeros((B, PS)))
    assert fake._call.mock_calls == []


def test_the_spec_check_uses_the_handles_horizon():
    """closed_loop's T/2 rule takes the solver's MPC horizon, the T qmb200_set_ee_paths checks against"""
    short = [(np.array([0.5, 0.9]), np.tile([0, 0, 0, 0, 0, 0, 1.0], (2, 1)))]
    assert len(closed_loop._ee_paths_spec(0.6, short)) == 1
    with pytest.raises(ValueError, match="at least time_horizon / 2 = 0.5 s apart"):
        closed_loop._ee_paths_spec(1.0, short)
    src = open(os.path.join(CSRC, "capi_ctrl.inc")).read()
    assert "ee_paths_error(n, n_way, way, h->hm.dev.time_horizon)" in src   # the horizon qmb200_get_model_info (Solver.time_horizon) reports


def _run_calls(**kw):
    import torch
    s = _fake_solver()
    s.get_ee_paths = mock.Mock(return_value=None); s.set_ee_paths = mock.Mock()
    with mock.patch.object(torch.cuda, "Stream", _FakeStream), mock.patch.object(torch.cuda, "stream", lambda st: contextlib.nullcontext()):
        closed_loop.run(s, **dict(dict(duration=0.02, torch_device="cpu", gait="trot"), **kw))
    return s, [c[0] for c in s.mock_calls]


def test_without_ee_paths_the_calls_are_the_parents_and_with_them_the_table_is_set_and_restored():
    _, calls = _run_calls()
    assert calls == _parent_calls()
    s, calls = _run_calls(ee_paths=SQUARE)
    assert calls == ["get_ee_paths", "set_ee_paths"] + _parent_calls() + ["set_ee_paths"]
    assert s.set_ee_paths.call_args_list[1][0][0] is None
    t, pose = s.set_ee_paths.call_args_list[0][0][0][0]
    assert np.array_equal(t, SQUARE[0][0]) and np.array_equal(pose, SQUARE[0][1])
    s, calls = _run_calls(ee_paths=SQUARE, commands=_path_commands())   # the target call takes the loop's path rows
    tcalls = [c for c in s.mock_calls if c[0] == "target_trajectories_dev"]
    assert tcalls and all(c[2]["path_state"].shape == (B, PS) for c in tcalls)
    assert [c[0] for c in s.mock_calls if c[0] == "gait_dev_set_commands"] and s.gait_dev_set_commands.call_args[1]["ee_kind"].tolist() == [[START]] * B
