"""Restarts that stand robots where they are, and restarts a Session requests, on the host, no GPU (DESIGN.md §4.18): the "here" row and the place
check compiled with g++ (tests/spawn_place_host.cpp, the functions spawn_here_kernel and spawn_place_kernel run) against numpy statements, the spec
errors of respawn at / on_request and Session.respawn, the calls they add on a fake Solver, the bindings and the kernels' resources."""
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

from test_gait_dev_cpu import B, _FakeStream, _fake_solver
from qm_control_b200 import _lib, closed_loop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
PI, TWO_PI = 3.141592653589793, 6.283185307179586
ST_SPAWN = 0x80000
NAMES = ("qmb200_spawn_place", "qmb200_spawn_place_dev", "qmb200_spawn_here", "qmb200_spawn_here_dev")


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("spawn_place") / "libspawnplacehost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include",
                           "-I" + CSRC, "-o", lib_path, os.path.join(ROOT, "tests", "spawn_place_host.cpp")])
    lib = C.CDLL(lib_path)
    lib.sph_here.argtypes = [C.c_int] + [C.c_void_p] * 6
    lib.sph_place_ok.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def wrap_statement(y):
    with np.errstate(invalid="ignore"):
        w = np.minimum(np.maximum(y - TWO_PI * np.floor((y + PI) / TWO_PI), -PI), PI)
        return np.where((np.abs(y) <= PI) | ~np.isfinite(y), y, w)


def here_statement(rbd, q_start, origin, ter, has):
    """numpy statement of spawn_here_row: tile, (x - x_start) + (origin - o_now), the same in y, the wrapped yaw; o_now = origin without rows"""
    ox = np.where(has, ter[:, 1], origin[:, 0]); oy = np.where(has, ter[:, 2], origin[:, 1])
    return np.stack([np.where(has, ter[:, 0], -1.0), (rbd[:, 3] - q_start[:, 0]) + (origin[:, 0] - ox), (rbd[:, 4] - q_start[:, 1]) + (origin[:, 1] - oy),
                     wrap_statement(rbd[:, 0])], axis=1)


def place_ok_statement(rows, n_tiles, rows_set):
    t, dx, dy, yaw = rows.T
    with np.errstate(invalid="ignore"):
        return ((np.floor(t) == t) & (t >= -1) & (t < n_tiles) & ((t < 0) | rows_set) & np.isfinite(dx) & np.isfinite(dy) & (yaw >= -PI) & (yaw <= PI)).astype(np.int32)


def _here(core, rbd, q_start, origin, ter, has):
    n = len(rbd); rows = np.zeros((n, _lib.SPAWN)); a = [_c(rbd, np.float64), _c(q_start, np.float64), _c(origin, np.float64), _c(ter, np.float64), _c(has, np.int32)]
    core.sph_here(n, *[x.ctypes.data for x in a], rows.ctypes.data)
    return rows


def test_here_row_equals_the_numpy_statement_bit_for_bit(core):
    rng = np.random.default_rng(5); n = 100_000
    rbd = rng.normal(size=(n, _lib.RBD)) * 3.0; q_start = rng.normal(size=(n, 24)); origin = rng.normal(size=(n, 2)) * 5.0
    ter = np.c_[rng.integers(-1, 3, n), rng.normal(size=(n, 2)) * 5.0]; has = rng.integers(0, 2, n)
    yaw = rng.uniform(-40.0, 40.0, n)   # many turns, and the edges of the wrap
    edges = np.array([PI, -PI, np.nextafter(PI, 4.0), np.nextafter(-PI, -4.0), 3 * PI, -3 * PI, TWO_PI, -TWO_PI, 0.0, -0.0, 1e6, -1e6, np.inf, -np.inf, np.nan])
    yaw[:len(edges)] = edges; rbd[:, 0] = yaw
    got = _here(core, rbd, q_start, origin, ter, has); want = here_statement(rbd, q_start, origin, ter, has.astype(bool))
    assert got.tobytes() == want.tobytes()
    fin = np.isfinite(yaw)
    assert np.all(np.abs(got[fin, 3]) <= PI) and np.allclose(np.sin(got[fin, 3]), np.sin(yaw[fin]), atol=1e-9) and np.allclose(np.cos(got[fin, 3]), np.cos(yaw[fin]), atol=1e-9)
    np.testing.assert_array_equal(got[has == 0, 0], -1.0)   # the plane: only the heading matters, dx, dy hold the travel
    np.testing.assert_array_equal(got[has == 0, 1], rbd[has == 0, 3] - q_start[has == 0, 0])
    # placed at x_start with the tile's origin origin - (dx, dy), the base stands on the tile point it stood on
    o_new = origin - got[:, 1:3]; h = has == 1
    np.testing.assert_allclose(q_start[h, :2] - o_new[h], rbd[h, 3:5] - ter[h, 1:3], rtol=0, atol=1e-12)


def test_place_check_equals_the_numpy_statement_on_every_rejection_class(core):
    rng = np.random.default_rng(6); n_tiles = 3
    good = np.c_[rng.integers(-1, n_tiles, 64), rng.normal(size=(64, 2)), rng.uniform(-PI, PI, 64)]
    classes = dict(tile_fraction=(0, 0.5), tile_below=(0, -2.0), tile_above=(0, float(n_tiles)), tile_nan=(0, np.nan), tile_inf=(0, np.inf), tile_ninf=(0, -np.inf),
                   dx_nan=(1, np.nan), dx_inf=(1, np.inf), dy_nan=(2, np.nan), dy_ninf=(2, -np.inf), yaw_above=(3, np.nextafter(PI, 4.0)), yaw_below=(3, -3.2),
                   yaw_nan=(3, np.nan))
    rows, rows_set, bad = [good, good.copy()], [np.ones(64, np.int32), np.zeros(64, np.int32)], [np.zeros(64, bool), good[:, 0] >= 0]   # a tile without rows
    for c, v in classes.values():
        r = good.copy(); r[:, c] = v; rows.append(r); rows_set.append(np.ones(64, np.int32)); bad.append(np.ones(64, bool))
    edge = good.copy(); edge[:8, 3] = PI; edge[8:16, 3] = -PI; edge[16:24, 0] = n_tiles - 1; edge[24:32, 0] = -1.0
    rows.append(edge); rows_set.append(np.ones(64, np.int32)); bad.append(np.zeros(64, bool))
    rows, rows_set, bad = np.concatenate(rows), np.concatenate(rows_set), np.concatenate(bad)
    ok = np.zeros(len(rows), np.int32)
    core.sph_place_ok(len(rows), _c(rows, np.float64).ctypes.data, n_tiles, _c(rows_set, np.int32).ctypes.data, ok.ctypes.data)
    np.testing.assert_array_equal(ok, place_ok_statement(rows, n_tiles, rows_set.astype(bool)))
    np.testing.assert_array_equal(ok, (~bad).astype(np.int32))


# ---------------------------------------------------------------------------------------------------------------------- spec errors
TER = dict(tiles=np.zeros((3, 5, 5)), cell=0.5, tile=np.array([0, 1, 2, -1]), origin=np.zeros((4, 2)))


@pytest.mark.parametrize("kw,match", [
    (dict(respawn=dict(at="there")), "respawn at must be"), (dict(respawn=dict(at=1)), "respawn at must be"),
    (dict(respawn=dict(on_request="yes")), "on_request must be True or False"), (dict(respawn=dict(every=0.1, on_request=True)), "on_request needs a Session"),
    (dict(respawn=dict(on_fall=False)), "needs on_fall, every or on_request"),
    (dict(respawn=dict(at="here", every=0.1), spawn=dict(yaw=(-0.5, 0.5))), "at=\"here\" cannot go with a drawn spawn yaw"),
    (dict(respawn=dict(at="here", every=0.1), terrain=TER, state_estimator=True, ground_map=dict(tile=np.zeros(4), origin=np.zeros((4, 2)))),
     "at=\"here\" cannot go with a ground_map dict"),
])
def test_closed_loop_rejects_a_malformed_restart_before_any_solver_call(kw, match):
    with pytest.raises(ValueError, match=match):
        closed_loop.run(None, duration=0.02, **kw)


def test_here_is_refused_beside_a_curriculum_spawn_and_end_effector_commands():
    s = types.SimpleNamespace(batch=4)
    cur = dict(levels=2, spawn=dict(dx=(0.0, 0.5)))
    with pytest.raises(ValueError, match="cannot go with a curriculum attached to the spawn"):
        closed_loop.run(s, duration=0.02, terrain=TER, respawn=dict(at="here", every=0.1), spawn=dict(dx=(0.0, 0.1)), curriculum=cur)
    goal = np.full((4, 1, 7), np.nan); goal[:, 0] = [0.5, 0.0, 0.5, 0.0, 0.0, 0.0, 1.0]
    with pytest.raises(ValueError, match="cannot go with ee_goal / ee_cmd_vel"):
        closed_loop.run(s, duration=0.02, respawn=dict(at="here", every=0.1), commands=dict(t=np.zeros((4, 1)), gait=[[None]] * 4, ee_goal=goal))
    closed_loop._run_specs(s, False, dict(closed_loop.RUN_DEFAULTS, respawn=dict(at="here", every=0.1), spawn=dict(yaw=(0.5, 0.5))))   # a fixed yaw is fine


# ---------------------------------------------------------------------------------------------------------------------- closed_loop.Session on a fake Solver
@contextlib.contextmanager
def _cpu_torch():
    import torch
    with mock.patch.object(torch.cuda, "Stream", _FakeStream), mock.patch.object(torch.cuda, "stream", lambda st: contextlib.nullcontext()):
        yield


def _solver():
    s = _fake_solver()
    for name in ("robot_image_save", "robot_image_restore_dev", "robot_image_clear", "fall_detect_dev", "spawn_here_dev", "spawn_place_dev"):
        setattr(s, name, mock.Mock())
    s.sim_get_robot_terrain = mock.Mock(return_value=None)
    return s


def test_session_respawn_errors_raise_before_any_write():
    import torch
    s = _solver()
    plain = closed_loop.Session(s, 0.03, gait="trot", respawn=dict(every=0.01))
    with pytest.raises(ValueError, match="needs respawn=dict"):
        plain.respawn(np.ones(B))
    ss = closed_loop.Session(s, 0.03, gait="trot", respawn=dict(on_fall=False, on_request=True))   # a request alone may restart robots
    for kw, match in ((dict(mask=np.ones(B + 1)), "mask must have shape"), (dict(mask=np.ones(B), end=3), "end must be 1"), (dict(mask=np.ones(B), end=0), "end must be 1"),
                      (dict(mask=np.ones(B), end=[1, 2, 2]), "end must be 1 or 2, a scalar"), (dict(mask=np.ones(B), end=np.array([1, 3])), "end must be 1"),
                      (dict(mask=np.ones(B), end=torch.tensor([2, 4])), "end must be 1"), (dict(mask=np.ones(B), end=True), "end must be"),
                      (dict(mask=np.ones(B), at="there"), "at must be None"), (dict(mask=np.ones(B), at=np.zeros((B, 3))), "at rows must have shape"),
                      (dict(mask=np.ones(B)), "not open")):
        with pytest.raises(ValueError, match=match):
            ss.respawn(**kw)
    ee = closed_loop.Session(s, 0.03, gait="trot", respawn=dict(every=0.01, on_request=True),
                             commands=dict(t=np.zeros((B, 1)), gait=[[None]] * B, ee_cmd_vel=np.full((B, 1, 3), 0.1)))
    with pytest.raises(ValueError, match="cannot go with ee_goal"):
        ee.respawn(np.ones(B), at="here")
    assert s.mock_calls == []
    here = closed_loop.Session(s, 0.03, gait="trot", steer=True, respawn=dict(every=0.01, at="here"))
    with pytest.raises(ValueError, match="restart \"here\""):
        here.command(np.ones(B), ee_cmd_vel=np.zeros((B, 3)))
    assert s.mock_calls == []


def _calls(requests=(), windows=(1, 1, 1), **respawn):
    s = _solver()
    with _cpu_torch():
        with closed_loop.Session(s, 0.01 * sum(windows), torch_device="cpu", gait="trot", respawn=respawn) as ss:
            for i, n in enumerate(windows):
                for (at_i, kw) in requests:
                    if at_i == i:
                        ss.respawn(**kw)
                ss.step(n)
            end = ss.finish()
    return s, [c[0] for c in s.mock_calls], end


def test_without_the_new_keys_no_place_call_is_made():
    _, calls, end = _calls(every=0.01)
    _, same, _ = _calls(every=0.01, at="start", on_request=False)
    assert calls == same and not {"spawn_here_dev", "spawn_place_dev", "sim_get_robot_terrain"} & set(calls) and "spawn_params" not in end


def test_here_adds_here_restore_place_at_every_boundary():
    _, start, _ = _calls(every=0.01)
    s, here, end = _calls(every=0.01, at="here")
    want = []
    for c in start:   # after the start's restore the run's start origins are read; every later restore is framed by here and place
        want += ["spawn_here_dev", c, "spawn_place_dev"] if c == "robot_image_restore_dev" and want.count("mpc_solve_dev") else [c]
        want += ["sim_get_robot_terrain"] if c == "robot_image_restore_dev" and not want.count("mpc_solve_dev") else []
    assert here == want and here.count("spawn_place_dev") == 2   # the boundaries of windows 1 and 2
    args = s.spawn_here_dev.call_args[0]; pargs = s.spawn_place_dev.call_args[0]
    assert args[4] is pargs[1] and args[3] is pargs[2]   # the rows here writes are the rows place reads, from the same origins
    sp = end["spawn_params"]   # the record: episode 0 the start's row, then the rows place accepted (the fake leaves them zero, its status 0)
    assert sp.shape == (B, 3, _lib.SPAWN) and np.all(sp[:, 0] == [-1.0, 0.0, 0.0, 0.0]) and np.all(sp[:, 1:] == 0.0)


def test_a_request_adds_exactly_here_restore_place_at_its_boundary():
    _, base, _ = _calls(on_fall=False, on_request=True)
    s, calls, _ = _calls(requests=[(1, dict(mask=np.array([0, 1]), end=1, at="here"))], on_fall=False, on_request=True)
    i = [k for k, c in enumerate(base) if c == "robot_image_restore_dev"][1]   # the start's restore, then window 1's boundary
    assert calls == base[:i] + ["spawn_here_dev", "robot_image_restore_dev", "spawn_place_dev"] + base[i + 1:]
    assert s.spawn_here_dev.call_args[0][0].tolist() == [0, 1] and s.spawn_place_dev.call_args[0][0].tolist() == [0, 1]
    _, start_req, _ = _calls(requests=[(1, dict(mask=np.array([1, 0]), at="start"))], on_fall=False, on_request=True)
    assert start_req == base   # a request to the start is the restore every boundary already issues


def test_entry_points_are_bound_declared_and_the_status_bit_is_free():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name
    assert len(_lib.PROTOTYPES["qmb200_spawn_place"][1]) == 13 and len(_lib.PROTOTYPES["qmb200_spawn_place_dev"][1]) == 14
    assert len(_lib.PROTOTYPES["qmb200_spawn_here"][1]) == 6 and len(_lib.PROTOTYPES["qmb200_spawn_here_dev"][1]) == 7
    assert "#define QMB200_ST_SPAWN (QMB200_ST_RESTORE << 1)" in h and _lib.ST_SPAWN == ST_SPAWN == _lib.ST_RESTORE << 1
    bits = [int(v, 0) for k, v in re.findall(r"#define (QMB200_ST_\w+) (0x[0-9a-fA-F]+|\d+)", h)] + [_lib.ST_RESTORE]
    assert ST_SPAWN not in bits and ST_SPAWN > max(bits)


def test_place_and_here_kernels_compile_for_sm90a_without_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    obj = str(tmp_path / "spawn.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "kernels", "spawn_kernel.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    for kernel in ("spawn_place_kernel", "spawn_here_kernel"):
        m = re.search(r"Function properties for (\w*%s\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads" % kernel, r.stderr)
        assert m and m.groups()[1:] == ("0", "0", "0"), r.stderr
        if os.path.exists(cuobjdump):
            sass = subprocess.run([cuobjdump, "-sass", "-fun", m.group(1), obj], capture_output=True, text=True, check=True).stdout
            assert kernel in sass and not re.search(r"\b(LDL|STL)\b", sass)
