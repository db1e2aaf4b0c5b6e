"""Per-episode spawns on the host, no GPU (DESIGN.md §4.12): the draw core compiled with g++ (tests/spawn_host.cpp) against its numpy statement, its
distribution and its keys, the range check, the ported standing pose against the host's standing_on_terrain, closed_loop.run(spawn=...) validation and
its ranges on a fake Solver, the bindings and the kernel's resources."""
import ctypes as C
import os
import re
import shutil
import subprocess
import types
from unittest import mock

import numpy as np
import pytest
from scipy import stats

import _episode_twin as etw
from _oracle import GAINS, REFERENCE, TASK, URDF
from _state_est_twin import _mix
from qm_control_b200 import _lib, closed_loop, terrain

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
SP = {n: i for i, n in enumerate(_lib.SPAWN_LAYOUT)}
NAMES = ("qmb200_spawn_set_ranges", "qmb200_spawn_get_ranges", "qmb200_spawn_sample", "qmb200_spawn_sample_dev", "qmb200_spawn_draw")
DOMAIN = np.uint64(0xbb67ae8584caa73b)   # spawn_api.cuh's SPAWN_DOMAIN


def twin_uniform(seed, robot, episode, column):
    """u in (0, 1) of (seed, robot, episode, column): the four words hashed in turn (the spawn domain), the 53 high bits of one more hash, plus a half"""
    u = etw._u64
    h = _mix(_mix(_mix(_mix(u(seed) ^ DOMAIN) ^ u(robot)) ^ u(episode)) ^ u(column))
    return ((_mix(h) >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53


def twin_rows(lo, hi, seed, robot, episode):
    """lo, hi [n, 4], keys [n] → rows [n, 4]: lo where hi == lo; the tile lo + min(floor(u (hi - lo + 1)), hi - lo); else fma(u, hi - lo, lo)"""
    lo = np.asarray(lo, dtype=np.float64); hi = np.asarray(hi, dtype=np.float64); d = hi - lo
    u = twin_uniform(np.asarray(seed)[:, None], np.asarray(robot)[:, None], np.asarray(episode)[:, None], np.arange(_lib.SPAWN)[None, :])
    out = etw.fma(u, d, lo)
    out[:, 0] = lo[:, 0] + np.minimum(np.floor(u[:, 0] * (d[:, 0] + 1.0)), d[:, 0])
    return np.where(hi == lo, lo, out)


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    d = tmp_path_factory.mktemp("spawn")
    # the host's standing_on_terrain, its text as capi_sim.inc has it, compiled beside the port
    src = open(os.path.join(CSRC, "capi_sim.inc")).read()
    m = re.search(r"^void standing_on_terrain\(.*?^}\n", src, re.S | re.M); assert m, "capi_sim.inc has standing_on_terrain"
    (d / "host_standing.inc").write_text(m.group(0))
    lib_path = str(d / "libspawnhost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-I" + CSRC,
                           "-DHOST_STANDING=\"%s\"" % (d / "host_standing.inc"), "-o", lib_path, os.path.join(ROOT, "tests", "spawn_host.cpp"),
                           os.path.join(CSRC, "host", "qm_config.cpp")])
    lib = C.CDLL(lib_path); lib.sp_create.restype = C.c_void_p
    return lib


@pytest.fixture(scope="module")
def model(core):
    h = core.sp_create(TASK.encode(), URDF.encode(), REFERENCE.encode(), GAINS.encode()); assert h
    yield C.c_void_p(h)
    core.sp_destroy(C.c_void_p(h))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _rows(core, lo, hi, seed, robot, episode):
    n = len(seed); lo = np.ascontiguousarray(lo, dtype=np.float64); hi = np.ascontiguousarray(hi, dtype=np.float64)
    seed, robot, episode = (np.ascontiguousarray(a, dtype=np.uint64) for a in (seed, robot, episode))
    out = np.zeros((n, _lib.SPAWN)); core.sp_rows(C.c_int(n), _ptr(seed), _ptr(robot), _ptr(episode), _ptr(lo), _ptr(hi), _ptr(out))
    return out


def _keys(rng, n):
    seed = rng.integers(0, 2 ** 63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    robot = rng.integers(0, 1 << 20, n).astype(np.uint64); episode = rng.integers(-2, 1 << 31, n).astype(np.int64).astype(np.uint64)
    return seed, robot, episode


def _ranges(rng, n, n_tiles=6):
    lo = np.zeros((n, 4)); hi = np.zeros((n, 4))
    lo[:, 0] = rng.integers(-1, n_tiles, n); hi[:, 0] = np.minimum(lo[:, 0] + rng.integers(0, n_tiles, n), n_tiles - 1)
    for c in (1, 2):
        lo[:, c] = rng.uniform(-2.0, 2.0, n) * 10.0 ** rng.integers(-3, 2, n); hi[:, c] = lo[:, c] + rng.uniform(0.0, 2.0, n)
    lo[:, 3] = rng.uniform(-np.pi, 0.0, n); hi[:, 3] = rng.uniform(0.0, np.pi, n)
    return lo, hi


def test_core_equals_the_numpy_statement_bit_for_bit(core):
    rng = np.random.default_rng(21); n = 120_000
    seed, robot, episode = _keys(rng, n); col = rng.integers(0, _lib.SPAWN, n).astype(np.int32)
    u = np.zeros(n); core.sp_uniform(C.c_int(n), _ptr(seed), _ptr(robot), _ptr(episode), _ptr(col), _ptr(u))
    np.testing.assert_array_equal(u, twin_uniform(seed, robot, episode, col))
    assert np.all(u > 0.0) and np.all(u < 1.0)
    m = 30_000; seed, robot, episode = _keys(rng, m); lo, hi = _ranges(rng, m)   # 120000 values
    got = _rows(core, lo, hi, seed, robot, episode)
    np.testing.assert_array_equal(got, twin_rows(lo, hi, seed, robot, episode))
    assert np.all(got >= lo) and np.all(got <= hi) and np.all(np.floor(got[:, 0]) == got[:, 0])
    wide = hi[:, 0] - lo[:, 0] >= 2   # the integer draw reaches both ends of its range
    assert np.any(got[wide, 0] == lo[wide, 0]) and np.any(got[wide, 0] == hi[wide, 0])


def test_fixed_columns_are_lo_byte_for_byte(core):
    rng = np.random.default_rng(3); m = 2000; seed, robot, episode = _keys(rng, m); lo, _ = _ranges(rng, m)
    lo[:4, 1] = [-0.0, 0.0, 1e-300, -5.0]; lo[:4, 3] = [-0.0, np.pi, -np.pi, 0.25]; lo[:4, 0] = [-1.0, 0.0, 5.0, 2.0]
    got = _rows(core, lo, lo.copy(), seed, robot, episode)
    assert got.tobytes() == lo.tobytes()   # -0.0 stays -0.0
    assert got.tobytes() == twin_rows(lo, lo.copy(), seed, robot, episode).tobytes()


def test_each_column_is_uniform(core):
    """chi-square on the tile over [-1, 4], Kolmogorov-Smirnov on dx, dy and yaw, over 20000 episodes of one robot and 20000 robots of one episode"""
    n = 20000; lo = np.tile([-1.0, -0.5, 0.2, -np.pi], (n, 1)); hi = np.tile([4.0, 0.5, 0.7, np.pi], (n, 1))
    for seed, robot, episode in ((np.full(n, 7), np.full(n, 3), np.arange(n)), (np.full(n, 2 ** 63 + 9), np.arange(n), np.zeros(n))):
        r = _rows(core, lo, hi, seed, robot, episode)
        counts = np.bincount(r[:, 0].astype(int) + 1, minlength=6); assert len(counts) == 6
        assert stats.chisquare(counts).pvalue > 1e-4, counts
        for c, (a, b) in ((1, (-0.5, 0.5)), (2, (0.2, 0.7)), (3, (-np.pi, np.pi))):
            assert stats.kstest(r[:, c], "uniform", args=(a, b - a)).pvalue > 1e-4, c


def test_seed_robot_and_episode_each_change_every_column(core):
    lo, hi = np.array([[-1.0, 0.0, 0.0, -np.pi]]), np.array([[1e6, 1.0, 1.0, np.pi]])
    base = _rows(core, lo, hi, [7], [3], [2])
    for key in (([8], [3], [2]), ([7], [4], [2]), ([7], [3], [3])):
        assert np.all(_rows(core, lo, hi, *key) != base), key


def _check(core, lo, hi, n_tiles):
    msg = C.create_string_buffer(256)
    rc = core.sp_ranges_error(C.c_int(len(lo)), _ptr(np.ascontiguousarray(lo)), _ptr(np.ascontiguousarray(hi)), C.c_int(n_tiles), msg, 256)
    return rc, msg.value.decode()


@pytest.mark.parametrize("field,lo_v,hi_v,why", [
    ("dx", np.nan, 0.0, "bounds must be finite"), ("dy", 0.0, np.inf, "bounds must be finite"), ("yaw", 0.2, 0.1, "lo must be <= hi"),
    ("dx", -1.5e308, 1.5e308, "hi - lo must be finite"), ("tile", 0.5, 1.0, "bounds must be integers"), ("tile", 0.0, 1.5, "bounds must be integers"),
    ("tile", -2.0, 0.0, "bounds must lie in [-1, 3), the tiles of the library in force"), ("tile", 0.0, 3.0, "bounds must lie in [-1, 3), the tiles of the library in force"),
    ("yaw", -3.2, 0.0, "bounds must lie in [-pi, pi]"), ("yaw", 0.0, 3.15, "bounds must lie in [-pi, pi]"), ("tile", np.inf, np.inf, "bounds must be finite")])
def test_range_check_names_the_field_and_the_robot(core, field, lo_v, hi_v, why):
    B = 5; lo = np.tile([-1.0, -0.1, -0.1, -np.pi], (B, 1)); hi = np.tile([2.0, 0.1, 0.1, np.pi], (B, 1))
    assert _check(core, lo, hi, 3) == (0, "")
    lo[3, SP[field]] = lo_v; hi[3, SP[field]] = hi_v
    assert _check(core, lo, hi, 3) == (1, "qmb200_spawn_set_ranges: %s of robot 3: %s" % (field, why))


def test_without_a_library_only_the_plane_is_a_tile(core):
    lo = np.array([[-1.0, 0.0, 0.0, 0.0]]); hi = lo.copy()
    assert _check(core, lo, hi, 0) == (0, "")
    hi[0, 0] = 0.0
    assert _check(core, lo, hi, 0)[1].endswith("tile of robot 0: bounds must lie in [-1, 0), the tiles of the library in force")


# ------------------------------------------------------------------------------------------------------------------------------ the standing pose
def _library():
    return np.stack([terrain.ramp(10.0), terrain.stairs(0.06, 0.25), terrain.rough(0.02, seed=3), terrain.ramp(8.0, direction_deg=60.0) + terrain.stairs(-0.05, 0.3)])


def test_every_chain_is_a_serial_chain_off_the_base(core, model):
    assert core.sp_chains_serial(model) == 1


def test_port_equals_the_host_standing_on_terrain(core, model):
    """ramp, stairs, rough and combined tiles, seeded offsets and yaws: z, pitch and roll within 1e-12 m / rad of the host's standing_on_terrain"""
    tiles = _library(); ny, nx = tiles.shape[1:]; rng = np.random.default_rng(8); n = 400
    tile = rng.integers(0, len(tiles), n); origin = terrain.centred_origin(np.zeros(2)) - rng.uniform(-1.2, 1.2, (n, 2))
    rows = np.c_[tile, origin].astype(np.float64); xy_yaw = np.c_[rng.uniform(-0.3, 0.3, (n, 2)), rng.uniform(-np.pi, np.pi, n)]
    radius, delta0 = 0.0265, 0.0
    for delta0 in (0.0, 1e-4):
        port = np.zeros((n, 3)); host = np.zeros((n, 3))
        core.sp_standing(model, _ptr(np.ascontiguousarray(tiles)), C.c_int(nx), C.c_int(ny), C.c_double(terrain.CELL), C.c_int(n), _ptr(rows), _ptr(xy_yaw),
                         C.c_double(radius), C.c_double(delta0), _ptr(port), _ptr(host))
        assert np.all(np.isfinite(port))
        np.testing.assert_allclose(port, host, rtol=0, atol=1e-12)
        assert np.ptp(port[:, 1]) > 0.1 and np.ptp(port[:, 0]) > 0.05   # the tiles tilt and lift the robots


def test_port_kinematics_equal_the_host_kinematics(core, model):
    rng = np.random.default_rng(2)
    for _ in range(50):
        base = np.r_[rng.uniform(-2, 2, 2), rng.uniform(0.3, 0.6), rng.uniform(-np.pi, np.pi), rng.uniform(-0.3, 0.3, 2)]
        ee, feet, eh, fh = np.zeros(7), np.zeros(12), np.zeros(7), np.zeros(12)
        core.sp_kinematics(model, _ptr(base), _ptr(ee), _ptr(feet), _ptr(eh), _ptr(fh))
        np.testing.assert_allclose(ee, eh, rtol=0, atol=1e-12); np.testing.assert_allclose(feet, fh, rtol=0, atol=1e-12)


# --------------------------------------------------------------------------------------------------------------------------- closed_loop.run(spawn=...)
TER = dict(tiles=np.zeros((3, 5, 5)), cell=0.5, tile=np.array([0, 1, 2, -1]), origin=np.zeros((4, 2)))


@pytest.mark.parametrize("kw,match", [
    (dict(spawn=[0.1]), "spawn must be None or dict"), (dict(spawn=dict(seed=-1)), "spawn seed must be an integer"), (dict(spawn=dict(seed=True)), "spawn seed"),
    (dict(spawn=dict(x=(0.0, 1.0))), "unknown spawn field 'x'"), (dict(spawn=dict(yaw=0.5)), "must be a pair"), (dict(spawn=dict(yaw=("a", 1.0))), "must be a pair"),
    (dict(spawn=dict(yaw=(np.zeros((2, 2)), 1.0))), "scalars or"), (dict(spawn=dict(yaw=(1.0, 0.0))), "finite with lo <= hi"),
    (dict(spawn=dict(yaw=(-4.0, 0.0))), r"yaw bounds must lie in \[-pi, pi\]"), (dict(spawn=dict(tile=(-1, 0))), "spawn tile needs terrain"),
    (dict(spawn=dict(dx=(0.0, 0.2), dy=(0.0, 0.1))), "spawn dx, dy needs terrain"), (dict(spawn=dict(tile=(0, 3)), terrain=TER), r"integers in \[-1, 3\)"),
    (dict(spawn=dict(tile=(-2, 0)), terrain=TER), "integers in"), (dict(spawn=dict(tile=(0.5, 1)), terrain=TER), "integers in"),
    (dict(spawn=dict(dx=(0.0, 0.2)), terrain=TER, state_estimator=True, ground_map=dict(tile=np.zeros(4), origin=np.zeros((4, 2)))), "ground_map dict cannot go"),
])
def test_closed_loop_rejects_a_malformed_spawn_before_any_solver_call(kw, match):
    with pytest.raises(ValueError, match=match):
        closed_loop.run(None, duration=0.02, **kw)


def test_a_drawn_yaw_is_refused_beside_end_effector_commands():
    goal = np.full((4, 1, 7), np.nan); goal[:, 0] = [0.5, 0.0, 0.5, 0.0, 0.0, 0.0, 1.0]
    commands = dict(t=np.zeros((4, 1)), gait=[[None]] * 4, ee_goal=goal)
    s = types.SimpleNamespace(batch=4)
    with pytest.raises(ValueError, match="drawn spawn yaw cannot go with ee_goal"):
        closed_loop.run(s, duration=0.02, commands=commands, spawn=dict(yaw=(-1.0, 1.0)))
    gd = closed_loop._gait_commands(4, "stance", commands)
    closed_loop._spawn_spec(4, dict(yaw=(0.5, 0.5)), None, None, gd)   # a fixed yaw is fine


class _Stop(Exception):
    pass


B = 4


def _fake(robot_terrain=None, prev_ranges=None):
    """→ (solver, state): get / set semantics of the calls a spawning run makes before its loop; spawn_set_ranges with ranges stops the run there"""
    st = dict(lib=None, robot_terrain=robot_terrain, ranges=prev_ranges, told=None)

    def set_ranges(lo=None, hi=None, seed=0):
        if lo is not None and st["told"] is None:
            st["told"] = (lo.copy(), hi.copy(), seed); raise _Stop
        st["ranges"] = None if lo is None else dict(lo=lo, hi=hi, seed=seed)

    def set_robot_terrain(tile=None, origin=None):
        st["robot_terrain"] = None if tile is None else dict(tile=np.asarray(tile), origin=np.asarray(origin))
    impl = dict(spawn_get_ranges=lambda: st["ranges"], spawn_set_ranges=set_ranges, sim_get_robot_terrain=lambda: st["robot_terrain"],
                sim_set_robot_terrain=set_robot_terrain, sim_get_terrain=lambda: st["lib"], sim_set_terrain=lambda tiles=None, cell=None: st.update(lib=None if tiles is None else dict(tiles=tiles, cell=cell)))
    solver = mock.Mock(spec=list(impl), batch=B, _cfg=types.SimpleNamespace(device=0))
    for name, f in impl.items():
        getattr(solver, name).side_effect = f
    return solver, st


def test_columns_not_named_are_fixed_at_the_runs_values_and_everything_is_restored():
    prev = dict(lo=np.ones((B, 4)), hi=np.full((B, 4), 2.0), seed=5)
    s, st = _fake(prev_ranges=prev)
    xy = np.c_[np.zeros((B, 2)), [0.1, -0.2, 0.3, 0.0]]
    with pytest.raises(_Stop):
        closed_loop.run(s, duration=0.02, xy_yaw=xy, terrain=TER, spawn=dict(seed=9, dx=(-0.1, [0.2, 0.3, 0.4, 0.5]), tile=(0, 2)))
    lo, hi, seed = st["told"]
    assert seed == 9
    np.testing.assert_array_equal(lo[:, SP["dx"]], -0.1); np.testing.assert_array_equal(hi[:, SP["dx"]], [0.2, 0.3, 0.4, 0.5])
    np.testing.assert_array_equal(lo[:, SP["tile"]], 0); np.testing.assert_array_equal(hi[:, SP["tile"]], 2)
    np.testing.assert_array_equal(lo[:, [SP["dy"], SP["yaw"]]], hi[:, [SP["dy"], SP["yaw"]]])
    np.testing.assert_array_equal(lo[:, SP["dy"]], 0.0); np.testing.assert_array_equal(lo[:, SP["yaw"]], xy[:, 2])
    assert st["ranges"]["seed"] == 5 and np.all(st["ranges"]["lo"] == 1.0)   # the previous ranges are back
    assert st["robot_terrain"] is None and st["lib"] is None                   # and the previous terrain


def test_earlier_ranges_come_back_after_the_earlier_terrain_and_an_unnamed_yaw_is_wrapped():
    prev = dict(lo=np.zeros((B, 4)), hi=np.zeros((B, 4)), seed=5)
    s, st = _fake(prev_ranges=prev)
    xy = np.c_[np.zeros((B, 2)), [4.0, -4.0, np.pi, -np.pi]]
    with pytest.raises(_Stop):
        closed_loop.run(s, duration=0.02, xy_yaw=xy, terrain=TER, spawn=dict(dx=(0.0, 0.1)))
    lo, hi, _ = st["told"]
    np.testing.assert_array_equal(lo[:, SP["yaw"]], [4.0 - 2 * np.pi, 2 * np.pi - 4.0, np.pi, -np.pi]); np.testing.assert_array_equal(hi[:, SP["yaw"]], lo[:, SP["yaw"]])
    names = [c[0] for c in s.mock_calls]
    assert names[-1] == "spawn_set_ranges" and "sim_set_terrain" in names[:-1]   # the earlier ranges are set again once the earlier terrain is back


@pytest.mark.parametrize("robot_terrain,want", [(None, -1), (dict(tile=np.array([1, 0, -1, 2]), origin=np.zeros((B, 2))), [1, 0, -1, 2])])
def test_a_fixed_tile_is_the_robots_terrain_row(robot_terrain, want):
    s, st = _fake(robot_terrain=robot_terrain)
    with pytest.raises(_Stop):
        closed_loop.run(s, duration=0.02, spawn=dict(yaw=(-np.pi, np.pi)))
    lo, hi, _ = st["told"]
    np.testing.assert_array_equal(lo[:, SP["tile"]], want); np.testing.assert_array_equal(hi[:, SP["tile"]], want)
    np.testing.assert_array_equal(hi[:, SP["yaw"]], np.pi); assert st["ranges"] is None


def test_without_spawn_the_loop_makes_no_spawn_call():
    s, _ = _fake()
    with pytest.raises(ValueError, match="cmd_vel must have shape"):
        closed_loop.run(s, duration=0.01, cmd_vel=np.zeros(3))
    assert s.mock_calls == []


def test_entry_points_are_bound_and_declared():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name
    assert "#define QMB200_SPAWN 4" in h and _lib.SPAWN_LAYOUT == ("tile", "dx", "dy", "yaw") and _lib.SPAWN == 4
    assert re.search(r"#define QMB200_SPAWN_GROUND_MAP %d\b" % _lib.SPAWN_GROUND_MAP, h)
    assert len(_lib.PROTOTYPES["qmb200_spawn_sample"][1]) == 12 and len(_lib.PROTOTYPES["qmb200_spawn_sample_dev"][1]) == 13


def test_spawn_kernel_compiles_for_sm90a_without_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    obj = str(tmp_path / "spawn.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "kernels", "spawn_kernel.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    assert any("spawn_sample_kernel" in k for k in kernels), r.stderr
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == len(kernels) and all(f == ("0", "0", "0") for f in frames), r.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if os.path.exists(cuobjdump):
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
        assert not re.search(r"\b(LDL|STL)\b", sass)
