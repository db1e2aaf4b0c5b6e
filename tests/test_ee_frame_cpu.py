"""End-effector targets in the robot's heading frame on the host, no GPU (DESIGN.md §4.19): the target front-end's per-robot body compiled with g++
(tests/ee_frame_host.cpp, the function ctrl_target_kernel runs) against a numpy statement of the heading rule and, in the world frame, against the
oracle; its equivariance and its agreement with upstream at the origin; the spawn's hold rule and the setter's check; the bindings, the snapshot block
and the kernels' resources; closed_loop's ee_frame spec, the refusals it lifts per robot and the calls it adds on a fake Solver."""
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

from _oracle import TargetOracle
from test_gait_dev_cpu import B, _FakeStream, _fake_solver, _parent_calls
from qm_control_b200 import _lib, closed_loop, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
NX, KMAX, TD = _lib.NX, _lib.KMAX, _lib.TARGET
COM_HEIGHT, DISP_VEL, ROT_VEL, T_TARGET = 0.4, 0.3, 0.1, 1.0   # reference.info:1-4, task.info mpc.timeHorizon
QJ = synthetic._info_vector(_lib.asset("qm_reference.info"), "defaultJointState", 18)
RI = Rotation.from_quat([0.5, -0.5, 0.5, -0.5])   # Eigen (w, x, y, z) = (-0.5, 0.5, -0.5, 0.5)
OFFSET = np.array([0.52, 0.09])


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("ee_frame") / "libeeframehost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include",
                           "-I" + CSRC, "-o", lib_path, os.path.join(ROOT, "tests", "ee_frame_host.cpp")])
    lib = C.CDLL(lib_path)
    lib.eef_target.argtypes = [C.c_int] + [C.c_void_p] * 12
    lib.eef_spawn_hold.argtypes = [C.c_int] + [C.c_void_p] * 5
    lib.eef_frame_error.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    assert lib.eef_kmax() == KMAX and lib.eef_target_dim() == TD
    return lib


def _c(a, dtype=np.float64):
    return np.ascontiguousarray(a, dtype=dtype)


def host_target(lib, kind, frame, cmd, t, x, ee, le, fill=np.nan):
    """the host build on n robots → (n_target [n], tt [n, KMAX], ts [n, KMAX, TD], le [n, 7]); untouched rows keep `fill` (n_target -7)"""
    n = len(kind); prm = _c([COM_HEIGHT, DISP_VEL, ROT_VEL, T_TARGET])
    le = _c(le).copy(); nt = np.full(n, -7, dtype=np.int32); tt = np.full((n, KMAX), fill); ts = np.full((n, KMAX, TD), fill)
    kind, frame, cmd, t, x, ee = _c(kind, np.int32), _c(frame, np.int32), _c(cmd), _c(t), _c(x), _c(ee)
    lib.eef_target(n, prm.ctypes.data, _c(QJ).ctypes.data, kind.ctypes.data, frame.ctypes.data, cmd.ctypes.data, t.ctypes.data, x.ctypes.data,
                   ee.ctypes.data, le.ctypes.data, nt.ctypes.data, tt.ctypes.data, ts.ctypes.data)
    return nt, tt, ts, le


# ---------------------------------------------------------------------------------------------------------------------- the numpy statement
def h_to_world(x, y, psi, p):
    """pose p [n, 7] (position, quaternion xyzw) in the heading frame of bases (x, y, psi) [n] → the world: Rz(psi) p + (x, y, 0), q_z(psi) q"""
    c, s, ch, sh = np.cos(psi), np.sin(psi), np.cos(0.5 * psi), np.sin(0.5 * psi)
    qx, qy, qzz, qw = p[:, 3], p[:, 4], p[:, 5], p[:, 6]
    q = np.stack([ch * qx - sh * qy, ch * qy + sh * qx, ch * qzz + sh * qw, ch * qw - sh * qzz], -1)
    return np.c_[c * p[:, 0] - s * p[:, 1] + x, s * p[:, 0] + c * p[:, 1] + y, p[:, 2], q]


def h_from_world(x, y, psi, p):
    """pose p [n, 7] in the world → the heading frame of bases (x, y, psi)"""
    return h_to_world(np.zeros_like(psi), np.zeros_like(psi), -psi, np.c_[p[:, 0] - x, p[:, 1] - y, p[:, 2:7]])


def h_from_world_pos(x, y, psi, p):
    c, s = np.cos(psi), np.sin(psi); dx, dy = p[:, 0] - x, p[:, 1] - y
    return np.c_[c * dx + s * dy, c * dy - s * dx, p[:, 2]]


def statement(kind, frame, cmd, t, x, ee, le):
    """the target front-end's rule (DESIGN.md §4.19) for robots of one kind in [0, 2] → (tt [n, 2], ts [n, 2, TD], le [n, 7]); frame 1: heading"""
    n = len(t); le = le.copy(); base = x[:, 6:12].copy(); hd = frame == 1
    px, py, psi = np.where(hd, base[:, 0], 0.0), np.where(hd, base[:, 1], 0.0), np.where(hd, base[:, 3], 0.0)
    Hw = lambda p, X=px, Y=py, P=psi: np.where(hd[:, None], h_to_world(X, Y, P, p), p)
    vel = np.zeros((n, 3)); bt = base.copy(); bt[:, 2] = COM_HEIGHT; bt[:, 4:6] = 0.0
    rot_off = lambda: np.where(hd[:, None], np.c_[np.cos(psi) * 0.52 - np.sin(psi) * 0.09, np.sin(psi) * 0.52 + np.cos(psi) * 0.09], OFFSET)
    if kind == 0:
        vel = Rotation.from_euler("ZYX", base[:, 3:6]).apply(cmd[:, :3])
        bt[:, 0] = base[:, 0] + vel[:, 0] * T_TARGET; bt[:, 1] = base[:, 1] + vel[:, 1] * T_TARGET; bt[:, 3] = base[:, 3] + cmd[:, 3] * T_TARGET
        reset = np.linalg.norm(Hw(le)[:, :3] - ee[:, :3], axis=1) > 0.1
        le[:, :3] = np.where(reset[:, None], np.where(hd[:, None], h_from_world_pos(px, py, psi, ee), ee[:, :3]), le[:, :3])
        ec = Hw(le); et = np.where(hd[:, None], h_to_world(bt[:, 0], bt[:, 1], bt[:, 3], le), le); tr = t + T_TARGET
    elif kind == 1:
        v = (Rotation.from_quat(ee[:, 3:7]) * RI.inv()).apply(cmd[:, :3])
        et = np.c_[ee[:, 0] + v[:, 0] * T_TARGET, ee[:, 1] + v[:, 1] * T_TARGET, Hw(le)[:, 2:7]]; ec = ee.copy()
        bt[:, 0:2] = et[:, 0:2] - rot_off(); tr = t + T_TARGET
    else:
        g = Hw(cmd[:, :7]); et = g; ec = ee.copy(); bt[:, 0:2] = g[:, 0:2] - rot_off()
        qc, qt = ee[:, 3:7], g[:, 3:7]
        dq = qc[:, 3:4] * qt[:, :3] - qt[:, 3:4] * qc[:, :3] + np.cross(qc[:, :3], qt[:, :3])
        tr = t + np.maximum(np.linalg.norm(dq, axis=1) / ROT_VEL, np.linalg.norm(g[:, :3] - ee[:, :3], axis=1) / DISP_VEL)
        le = np.where(hd[:, None], h_from_world(bt[:, 0], bt[:, 1], psi, g), g)
    bc = base.copy(); bc[:, 2] = COM_HEIGHT; bc[:, 4:6] = 0.0
    djs = np.broadcast_to(QJ, (n, 18)); z = np.zeros((n, 3))
    ts = np.stack([np.c_[vel, z, bc, djs, ec], np.c_[vel, z, bt, djs, et]], 1)
    return np.c_[t, tr], ts, le


def robots(n, seed, origin=False):
    """n random robots: kind [-1, 2], frame {0, 1}, unwrapped yaw in ±50 rad, bases within ±20 m; origin: bases at (0, 0, yaw 0)"""
    rng = np.random.default_rng(seed)
    kind = rng.integers(-1, 3, n).astype(np.int32); frame = rng.integers(0, 2, n).astype(np.int32)
    x = rng.uniform(-0.3, 0.3, (n, NX)); x[:, 6:8] = rng.uniform(-20, 20, (n, 2)); x[:, 8] = rng.uniform(0.3, 0.5, n); x[:, 9] = rng.uniform(-50, 50, n)
    if origin:
        x[:, 6:8] = 0.0; x[:, 9] = 0.0
    ee = np.c_[x[:, 6:8] + rng.uniform(-1, 1, (n, 2)), rng.uniform(0.2, 0.7, n), Rotation.random(n, random_state=seed).as_quat()]
    hold = np.c_[rng.uniform(0.3, 0.7, (n, 2)), rng.uniform(0.2, 0.7, n), Rotation.random(n, random_state=seed + 1).as_quat()]
    le = np.where(frame[:, None] == 1, hold, np.c_[ee[:, :3] + rng.uniform(-0.12, 0.12, (n, 3)), hold[:, 3:7]])
    cmd = rng.uniform(-0.5, 0.5, (n, 7)); g = kind == 2
    cmd[g, 3:7] = Rotation.random(int(g.sum()), random_state=seed + 2).as_quat()
    cmd[g, 0:3] = np.where(frame[g, None] == 1, rng.uniform(0.2, 0.8, (int(g.sum()), 3)), ee[g, :3] + rng.uniform(-0.5, 0.5, (int(g.sum()), 3)))
    t = rng.uniform(0.0, 10.0, n)
    return kind, frame, cmd, t, x, ee, le


def _away_from_the_reset_edge(frame, cmd, x, ee, le):
    """robots whose cmd_vel hold is not within 1e-9 m of the 0.1 m reset distance (where rounding may take either side)"""
    base = x[:, 6:12]; hd = frame == 1
    w = np.where(hd[:, None], h_to_world(base[:, 0], base[:, 1], base[:, 3], le), le)
    return np.abs(np.linalg.norm(w[:, :3] - ee[:, :3], axis=1) - 0.1) > 1e-9


# ---------------------------------------------------------------------------------------------------------------------- the host build
def test_the_host_build_equals_the_heading_rule_on_1e5_robots(host):
    kind, frame, cmd, t, x, ee, le = robots(100_000, 11)
    nt, tt, ts, le_out = host_target(host, kind, frame, cmd, t, x, ee, le)
    held = (kind < 0)
    assert np.all(nt[held] == -7) and np.all(np.isnan(tt[held])) and np.all(np.isnan(ts[held])) and np.array_equal(le_out[held], le[held])
    for k in (0, 1, 2):
        m = (kind == k) & _away_from_the_reset_edge(frame, cmd, x, ee, le) if k == 0 else kind == k
        rt, rs, rl = statement(k, frame[m], cmd[m], t[m], x[m], ee[m], le[m])
        assert np.all(nt[m] == 2) and np.all(tt[m][:, 2:] == 0.0) and np.all(ts[m][:, 2:] == 0.0)
        np.testing.assert_allclose(tt[m][:, :2], rt, rtol=0, atol=1e-12, err_msg="kind %d times" % k)
        np.testing.assert_allclose(ts[m][:, :2], rs, rtol=0, atol=1e-12, err_msg="kind %d states" % k)
        np.testing.assert_allclose(le_out[m], rl, rtol=0, atol=1e-12, err_msg="kind %d hold" % k)
        for f in (0, 1):   # both frames took part
            assert np.count_nonzero(frame[m] == f) > 1000


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_the_world_frame_equals_the_oracle(host, kind):
    _, _, cmd, t, x, ee, le = robots(300, 20 + kind)
    n = len(t); frame = np.zeros(n, dtype=np.int32); k = np.full(n, kind, dtype=np.int32)
    if kind == 2:
        cmd[:, 3:7] = Rotation.random(n, random_state=7).as_quat()
    nt, tt, ts, le_out = host_target(host, k, frame, cmd, t, x, ee, le)
    to = TargetOracle()
    for i in range(n):
        rt, rs, rl = to.target(kind, cmd[i], t[i], x[i], ee[i], le[i])
        assert nt[i] == 2
        np.testing.assert_allclose(tt[i, :2], rt, rtol=0, atol=1e-12); np.testing.assert_allclose(ts[i, :2], rs, rtol=0, atol=1e-12)
        np.testing.assert_allclose(le_out[i], rl, rtol=0, atol=1e-12)


def test_at_the_origin_the_heading_frame_is_upstream_bit_for_bit(host):
    kind, _, cmd, t, x, ee, le = robots(20_000, 31, origin=True)
    kind = np.where(kind < 0, 2, kind).astype(np.int32); cmd[kind == 0] = 0.0   # kind 0 with zero cmd_vel: the base target is the base
    n = len(t); le = np.c_[ee[:, :3] + np.random.default_rng(3).uniform(-0.12, 0.12, (n, 3)), le[:, 3:7]]
    w = host_target(host, kind, np.zeros(n), cmd, t, x, ee, le); h = host_target(host, kind, np.ones(n), cmd, t, x, ee, le)
    for a, b in zip(w[:3], h[:3]):
        assert a.tobytes() == b.tobytes()
    m = kind != 2   # a goal's hold is the goal in the world for a world robot, in the base target's frame for a heading robot
    assert w[3][m].tobytes() == h[3][m].tobytes()


def _pose(px, py, psi, ts):
    """the pose P = (px, py, psi) [n] applied to target states ts [n, 2, TD] stated at the origin"""
    out = ts.copy(); c, s = np.cos(psi)[:, None], np.sin(psi)[:, None]
    out[..., 0] = c * ts[..., 0] - s * ts[..., 1]; out[..., 1] = s * ts[..., 0] + c * ts[..., 1]   # the cmd_vel knot velocity
    out[..., 6] = c * ts[..., 6] - s * ts[..., 7] + px[:, None]; out[..., 7] = s * ts[..., 6] + c * ts[..., 7] + py[:, None]; out[..., 9] = ts[..., 9] + psi[:, None]
    for k in range(2):
        out[:, k, 30:37] = h_to_world(px, py, psi, ts[:, k, 30:37])
    return out


def test_the_heading_rule_is_equivariant(host):
    kind, _, cmd, t, x, ee, le = robots(20_000, 41, origin=True)
    n = len(t); frame = np.ones(n, dtype=np.int32); kind = np.where(kind < 0, 0, kind).astype(np.int32); x[:, 10:12] = 0.0   # pitch, roll: not the frame's
    rng = np.random.default_rng(42); px, py, psi = rng.uniform(-20, 20, n), rng.uniform(-20, 20, n), rng.uniform(-50, 50, n)
    xp = x.copy(); xp[:, 6] = px; xp[:, 7] = py; xp[:, 9] = psi
    eep = h_to_world(px, py, psi, ee)
    keep = _away_from_the_reset_edge(frame, cmd, x, ee, le)
    o = host_target(host, kind, frame, cmd, t, x, ee, le); p = host_target(host, kind, frame, cmd, t, xp, eep, le)
    np.testing.assert_allclose(p[1][keep], o[1][keep], rtol=0, atol=1e-12)
    np.testing.assert_allclose(p[2][keep][:, :2], _pose(px[keep], py[keep], psi[keep], o[2][keep][:, :2]), rtol=0, atol=1e-12)
    np.testing.assert_allclose(p[3][keep], o[3][keep], rtol=0, atol=1e-12)   # the hold is body-relative


def test_a_spawn_turns_a_world_hold_and_leaves_a_heading_hold(host):
    n = 4096; rng = np.random.default_rng(5)
    e0 = np.c_[rng.uniform(-2, 2, (n, 3)), Rotation.random(n, random_state=5).as_quat()]; xy = rng.uniform(-2, 2, (n, 2))
    yaw0, yaw = rng.uniform(-np.pi, np.pi, n), rng.uniform(-np.pi, np.pi, n); yaw[:8] = yaw0[:8]   # some robots keep their heading
    heading = (np.arange(n) % 2).astype(np.int32)
    e = _c(e0).copy()
    host.eef_spawn_hold(n, e.ctypes.data, _c(xy).ctypes.data, _c(yaw0).ctypes.data, _c(yaw).ctypes.data, heading.ctypes.data)
    hd = heading == 1
    assert e[hd].tobytes() == e0[hd].tobytes() and e[:8].tobytes() == e0[:8].tobytes()
    d = yaw - yaw0; w = ~hd
    want = h_to_world(xy[:, 0], xy[:, 1], d, np.c_[e0[:, 0] - xy[:, 0], e0[:, 1] - xy[:, 1], e0[:, 2:7]])
    np.testing.assert_allclose(e[w & (d != 0)], want[w & (d != 0)], rtol=0, atol=1e-12)


def test_the_setter_accepts_world_and_heading_only(host):
    buf = C.create_string_buffer(256)
    assert host.eef_frame_error(_c([0, 1, 1, 0], np.int32).ctypes.data, 4, buf, 256) == 0
    for rows, robot in (([0, 2, 1], 1), ([1, 1, -1], 2), ([7], 0)):
        assert host.eef_frame_error(_c(rows, np.int32).ctypes.data, len(rows), buf, 256) > 0
        msg = buf.value.decode()
        assert msg.startswith("qmb200_set_ee_frame: frame of robot %d is %d" % (robot, rows[robot])) and "QMB200_EE_FRAME_HEADING" in msg


# ---------------------------------------------------------------------------------------------------------------------- bindings, snapshot block, resources
def test_bindings_header_and_snapshot_block_agree():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    assert re.search(r"int qmb200_set_ee_frame\(qmb200_handle\* h, const int32_t\* frame", h) and re.search(r"int qmb200_get_ee_frame\(", h)
    assert _lib.PROTOTYPES["qmb200_set_ee_frame"] == (C.c_int32, [C.c_void_p] * 2) and _lib.PROTOTYPES["qmb200_get_ee_frame"] == (C.c_int32, [C.c_void_p] * 3)
    assert "#define QMB200_EE_FRAME_WORLD 0" in h and "#define QMB200_EE_FRAME_HEADING 1" in h and (_lib.EE_FRAME_WORLD, _lib.EE_FRAME_HEADING) == (0, 1)
    n = int(re.search(r"#define QMB200_STATE_BLOCKS (\d+)", h).group(1))
    assert n == 33 and _lib.ROBOT_STATE_BLOCKS[-1] == "ee_frame" and len(_lib.RobotStateDesc._fields_[-1][1]()) == n
    names = re.search(r"kStateName\[QMB200_STATE_BLOCKS\] = \{(.*?)\};", open(os.path.join(CSRC, "capi_respawn.inc")).read(), re.S).group(1)
    assert re.findall(r'"[^"]+"', names)[-1] == '"end-effector frame rows"'
    api = open(os.path.join(CSRC, "kernels", "respawn_api.cuh")).read()
    assert int(re.search(r"RESTORE_MAX_SEGS = (\d+)", api).group(1)) >= n


def _resources(nvcc, src, tmp_path):
    obj = str(tmp_path / (os.path.basename(src) + ".o"))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", "-x", "cu",
                        os.path.join(CSRC, "kernels", src), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return obj, r.stderr


def test_the_target_and_spawn_kernels_compile_for_sm90a_without_spills(tmp_path):
    """The spawn kernels keep no stack frame and no local memory.  The target kernel's one frame is the parent's: the 40 bytes of the Payne-Hanek slow
    path of the sincos in the world-frame cmd_vel rotation (rot_zyx, kept bit for bit), taken for angles beyond 2^31 rad only; the heading branch's
    spawn_sincos adds none."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    for src, kernels, frame in (("spawn_kernel.cu", ("spawn_sample_kernel", "spawn_place_kernel", "spawn_here_kernel"), "0"), ("ctrl_kernels.cu", ("ctrl_target_kernel",), "40")):
        obj, err = _resources(nvcc, src, tmp_path)
        for kernel in kernels:
            m = re.search(r"Function properties for (\w*%s\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads" % kernel, err)
            assert m and m.groups()[1:] == (frame, "0", "0"), err
            if frame == "0" and os.path.exists(cuobjdump):
                sass = subprocess.run([cuobjdump, "-sass", "-fun", m.group(1), obj], capture_output=True, text=True, check=True).stdout
                assert kernel in sass and not re.search(r"\b(LDL|STL)\b", sass)


# ---------------------------------------------------------------------------------------------------------------------- closed_loop
@pytest.mark.parametrize("ee_frame", ["body", "Heading", 1, 0.5, [0, 1, 1], np.array([0.0, 1.0]), np.array([0, 2]), np.array([[0, 1]]), [-1, 0]])
def test_a_malformed_ee_frame_raises_before_any_solver_call(ee_frame):
    s = mock.Mock(batch=B)   # B = 2 robots
    with pytest.raises(ValueError, match="ee_frame must be"):
        closed_loop.run(s, duration=0.02, ee_frame=ee_frame)
    with pytest.raises(ValueError, match="ee_frame must be"):
        closed_loop.Session(s, 0.02, ee_frame=ee_frame)
    assert s.mock_calls == []


def _goal_commands(n=4):
    goal = np.full((n, 1, 7), np.nan); goal[:, 0] = [0.5, 0.0, 0.5, 0.0, 0.0, 0.0, 1.0]
    return dict(t=np.zeros((n, 1)), gait=[[None]] * n, ee_goal=goal)


def test_the_refusals_hold_for_world_robots_only():
    s = types.SimpleNamespace(batch=4); cmds = _goal_commands()
    yaw = dict(yaw=(-np.pi, np.pi))
    closed_loop._run_specs(s, False, dict(closed_loop.RUN_DEFAULTS, commands=cmds, spawn=yaw, ee_frame="heading"))   # lifted
    closed_loop._run_specs(s, False, dict(closed_loop.RUN_DEFAULTS, commands=cmds, respawn=dict(at="here", every=0.1), ee_frame="heading"))
    tl = dict(seed=0, n=2, t_first=(0.1, 0.2), gap=(0.1, 0.2), weights=dict(ee_goal=1.0), ee_x=(0.4, 0.6), ee_y=(-0.1, 0.1), ee_z=(0.3, 0.5),
              ee_quat=(0.0, 0.0, 0.0, 1.0))
    closed_loop._run_specs(s, False, dict(closed_loop.RUN_DEFAULTS, timeline=tl, spawn=yaw, ee_frame="heading"))
    mixed = np.array([1, 1, 0, 1])
    with pytest.raises(ValueError, match="drawn spawn yaw cannot go with ee_goal / ee_cmd_vel commands to world-frame robots"):
        closed_loop.run(s, duration=0.02, commands=cmds, spawn=yaw, ee_frame=mixed)
    with pytest.raises(ValueError, match="at=\"here\" cannot go with ee_goal / ee_cmd_vel commands to world-frame robots"):
        closed_loop.run(s, duration=0.02, commands=cmds, respawn=dict(at="here", every=0.1), ee_frame=mixed)
    with pytest.raises(ValueError, match="drawn spawn yaw"):
        closed_loop.run(s, duration=0.02, timeline=tl, spawn=yaw, ee_frame=mixed)
    # per robot: the world robot 2 may draw a yaw when it gets no end-effector command, or keep a fixed one while it gets them
    few = _goal_commands(); few["ee_goal"][2] = np.nan
    closed_loop._run_specs(s, False, dict(closed_loop.RUN_DEFAULTS, commands=few, spawn=yaw, ee_frame=mixed))
    closed_loop._run_specs(s, False, dict(closed_loop.RUN_DEFAULTS, commands=cmds, spawn=dict(yaw=(np.array([-1, -1, 0.2, -1.0]), np.array([1, 1, 0.2, 1.0]))),
                                          ee_frame=mixed))
    with pytest.raises(ValueError, match="drawn spawn yaw"):   # a drawn yaw itself still cannot go with a restart "here"
        closed_loop.run(s, duration=0.02, spawn=yaw, respawn=dict(at="here", every=0.1), ee_frame="heading")


def test_session_commands_and_requests_are_refused_per_world_robot():
    s = _fake_solver()
    for name in ("robot_image_save", "robot_image_restore_dev", "robot_image_clear", "fall_detect_dev", "spawn_here_dev", "spawn_place_dev"):
        setattr(s, name, mock.Mock())
    goal = np.zeros((B, 7)); goal[:, 6] = 1.0
    here = closed_loop.Session(s, 0.03, gait="trot", steer=True, respawn=dict(every=0.01, at="here"), ee_frame=np.array([1, 0]))
    with pytest.raises(ValueError, match="to world-frame robots cannot go with a drawn spawn yaw or a restart \"here\""):
        here.command(np.ones(B), ee_goal=goal)
    with pytest.raises(ValueError, match="not open"):   # robot 0 alone is a heading robot: accepted up to the open check
        here.command(np.array([1, 0]), ee_goal=goal)
    hd = closed_loop.Session(s, 0.03, gait="trot", steer=True, respawn=dict(every=0.01, at="here"), ee_frame="heading")
    with pytest.raises(ValueError, match="not open"):
        hd.command(np.ones(B), ee_goal=goal)
    req = closed_loop.Session(s, 0.03, gait="trot", respawn=dict(every=0.01, on_request=True), ee_frame="heading",
                              commands=dict(t=np.zeros((B, 1)), gait=[[None]] * B, ee_cmd_vel=np.full((B, 1, 3), 0.1)))
    with pytest.raises(ValueError, match="not open"):
        req.respawn(np.ones(B), at="here")
    world = closed_loop.Session(s, 0.03, gait="trot", respawn=dict(every=0.01, on_request=True), ee_frame=np.array([1, 0]),
                                commands=dict(t=np.zeros((B, 1)), gait=[[None]] * B, ee_cmd_vel=np.full((B, 1, 3), 0.1)))
    with pytest.raises(ValueError, match="cannot go with ee_goal / ee_cmd_vel commands to world-frame robots"):
        world.respawn(np.ones(B), at="here")
    assert s.mock_calls == []


def _run_calls(**kw):
    import torch
    s = _fake_solver()
    s.get_ee_frame = mock.Mock(return_value=None); s.set_ee_frame = mock.Mock()
    with mock.patch.object(torch.cuda, "Stream", _FakeStream), mock.patch.object(torch.cuda, "stream", lambda st: contextlib.nullcontext()):
        closed_loop.run(s, **dict(dict(duration=0.02, torch_device="cpu", gait="trot"), **kw))
    return s, [c[0] for c in s.mock_calls]


def test_without_ee_frame_the_calls_are_the_parents_and_with_it_the_rows_are_set_and_restored():
    _, calls = _run_calls()
    assert calls == _parent_calls()
    _, world = _run_calls(ee_frame="world")
    assert world == _parent_calls()
    s, calls = _run_calls(ee_frame="heading")
    assert calls == ["get_ee_frame", "set_ee_frame"] + _parent_calls() + ["set_ee_frame"]
    assert s.set_ee_frame.call_args_list[0][0][0].tolist() == [1] * B and s.set_ee_frame.call_args_list[1][0][0] is None
    s, _ = _run_calls(ee_frame=np.array([0, 1]))
    assert s.set_ee_frame.call_args_list[0][0][0].tolist() == [0, 1] and s.set_ee_frame.call_args_list[0][0][0].dtype == np.int32
