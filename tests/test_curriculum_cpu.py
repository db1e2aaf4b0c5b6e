"""Per-robot curricula on the host, no GPU (DESIGN.md §4.15): the box and update core compiled with g++ (tests/curriculum_host.cpp) against its numpy
statement (tests/_curriculum_twin.py), the validation of the rule, the rows and every attached level, closed_loop.run(curriculum=...) validation and its
calls on a fake Solver, the bindings and the update kernel's resources."""
import ctypes as C
import os
import re
import shutil
import subprocess
import types
from unittest import mock

import numpy as np
import pytest

import _curriculum_twin as tw
from qm_control_b200 import _lib, closed_loop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
NAMES = ("qmb200_curriculum_set", "qmb200_curriculum_attach", "qmb200_curriculum_update", "qmb200_curriculum_update_dev", "qmb200_curriculum_get",
         "qmb200_curriculum_draw")
MT = {n: i for i, n in enumerate(_lib.METRICS_LAYOUT)}
TL = {n: i for i, n in enumerate(_lib.TIMELINE_LAYOUT)}


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("curriculum") / "libcurriculumhost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-I" + CSRC,
                           "-o", lib_path, os.path.join(ROOT, "tests", "curriculum_host.cpp")])
    return C.CDLL(lib_path)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _box(core, base, top, level, n_levels, round_col=-1):
    base = np.ascontiguousarray(base, dtype=np.float64); top = np.ascontiguousarray(top, dtype=np.float64); level = np.ascontiguousarray(level, dtype=np.int32)
    out = np.zeros_like(base)
    core.cu_box(C.c_int(len(base)), C.c_int(base.shape[1]), C.c_int(round_col), C.c_int(n_levels), _ptr(level), _ptr(base), _ptr(top), _ptr(out))
    return out


@pytest.mark.parametrize("n_levels", [2, 3, 17, 256])
def test_box_at_every_level_equals_the_numpy_statement_byte_for_byte(core, n_levels):
    rng = np.random.default_rng(n_levels); m = 40 if n_levels == 256 else 160; W = 6
    base = rng.uniform(-2.0, 2.0, (m, W)); top = base + rng.uniform(-3.0, 3.0, (m, W))
    base[::5, 1] = -0.0; top[::7, 2] = -0.0; top[1::9, 3] = 1e300; base[2::11, 3] = -1e300   # -0.0 at one end, wide spans
    base[:, 0] = rng.integers(-1, 4, m); top[:, 0] = rng.integers(-1, 9, m)            # an integer (tile) column
    eq = np.zeros((m, W), dtype=bool); eq[:, 4:] = rng.uniform(size=(m, 2)) < 0.3; top[eq] = base[eq]   # equal columns
    z = np.zeros((m, W), dtype=bool); z[:, 4:] = ~eq[:, 4:] & (rng.uniform(size=(m, 2)) < 0.2); base[z] = top[z] = -0.0   # -0.0 at both ends
    for level in range(n_levels):
        lv = np.full(m, level)
        for rc in (-1, 0):
            got = _box(core, base, top, lv, n_levels, rc)
            assert got.tobytes() == tw.box(base, top, lv, n_levels, rc).tobytes(), (level, rc)
        if level == 0:
            assert got.tobytes() == base.tobytes()
        if level == n_levels - 1:
            assert got.tobytes() == top.tobytes()
        assert got[eq].tobytes() == base[eq].tobytes() and np.all(np.signbit(got[z]))
        assert np.all(np.floor(got[:, 0]) == got[:, 0])


def test_tile_rounds_half_up_on_both_sides_of_one_half(core):
    # tile 0 → 3 over 7 levels: x = 0.5 l exactly, so the odd levels sit on .5 and round up; 0 → -1 rounds -0.5 up to 0
    base = np.zeros((4, 4)); top = np.zeros((4, 4)); top[0, 0] = 3.0; top[1, 0] = -1.0; base[2, 0] = 1.0; top[2, 0] = 2.0; top[3, 0] = 1.0
    got = np.array([_box(core, base, top, np.full(4, lv), 7, 0)[:, 0] for lv in range(7)])
    np.testing.assert_array_equal(got[:, 0], [0, 1, 1, 2, 2, 3, 3])
    np.testing.assert_array_equal(got[1:6, 1], [0, 0, 0, -1, -1])   # x = -l / 6: -1/6, -1/3 round to 0; -1/2 rounds up to 0; -2/3, -5/6 to -1
    np.testing.assert_array_equal(got[:, 2], [1, 1, 1, 2, 2, 2, 2])
    assert got[3, 2] == 2.0 and got[2, 2] == 1.0   # 1.5 rounds up; 1.333 down
    assert np.all(got[:, 3] == np.floor(np.arange(7) / 6.0 + 0.5)) and got[3, 3] == 1.0


def _stream(core, n_levels, conditions, row, end, metrics, state):
    cols = np.array([c for c, _, _ in conditions] + [0] * 4, dtype=np.int32)[:4]
    ops = np.array([_lib.CURRICULUM_OPS.index(o) for _, o, _ in conditions] + [0] * 4, dtype=np.int32)[:4]
    roles = np.array([_lib.CURRICULUM_ROLES.index(r) for _, _, r in conditions] + [0] * 4, dtype=np.int32)[:4]
    row = np.ascontiguousarray(row, dtype=np.float64); end = np.ascontiguousarray(end, dtype=np.int32); metrics = np.ascontiguousarray(metrics, dtype=np.float64)
    st = np.ascontiguousarray(state, dtype=np.int32).copy(); out = np.zeros((len(end), 4), dtype=np.int32)
    core.cu_stream(C.c_int(n_levels), C.c_int(len(conditions)), _ptr(cols), _ptr(ops), _ptr(roles), _ptr(row), C.c_int(len(end)), _ptr(end), _ptr(metrics), _ptr(st), _ptr(out))
    return out


def test_rule_streams_equal_a_plain_statement_of_the_rule(core):
    rng = np.random.default_rng(7); covered = set()
    for trial in range(400):
        L = int(rng.choice([2, 3, 5, 12])); nc = int(rng.integers(0, 5))
        conditions = [(int(rng.integers(0, 18)), str(rng.choice([">=", "<="])), str(rng.choice(["pass", "fail"]))) for _ in range(nc)]
        thr = rng.choice([0.0, 0.5, 1.0], 4)
        row = np.r_[rng.integers(0, L), rng.integers(1, 4), rng.integers(1, 4), thr]
        k = 60; end = rng.choice([0, 1, 2, 2, 2, 3, -1], k)
        metrics = rng.choice([0.0, 0.5, 1.0, np.nan, 0.25, 2.0], (k, 18))   # exact thresholds and NaN
        for i, (c, _, _) in enumerate(conditions):   # values exactly at the threshold
            metrics[rng.uniform(size=k) < 0.3, c] = thr[i]
        state = np.array([row[0], 0, 0, 0]); got = _stream(core, L, conditions, row, end, metrics, state)
        want = state.tolist()
        for j in range(k):
            want = tw.step(want, row, end[j], metrics[j], L, conditions)
            assert got[j].tolist() == want, (trial, j)
            covered |= {("top", want[0] == L - 1), ("bottom", want[0] == 0)}
        covered.add(("moved", got[-1, 3] > 0))
    assert covered >= {("top", True), ("bottom", True), ("moved", True)}


def test_up_after_and_down_after_count_runs_and_clamp(core):
    row = [1, 2, 3, 0, 0, 0, 0]; m = np.zeros((12, 18))
    got = _stream(core, 3, [], row, [2, 2, 2, 2, 2, 1, 2, 1, 1, 1, 0, 1], m, [1, 0, 0, 0])
    assert got[:, 0].tolist() == [1, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1]
    assert got[:, 1].tolist() == [1, 0, 1, 0, 1, 0, 1, 0, 0, 0, 0, 0] and got[:, 2].tolist() == [0, 0, 0, 0, 0, 1, 0, 1, 2, 0, 0, 1]
    assert got[:, 3].tolist() == [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 10, 11]   # end 0 counts nothing


def _err(core, rows, n_levels=4, conditions=((0, 0, 0),)):
    c = np.array([x[0] for x in conditions] + [0] * 4, dtype=np.int32)[:4]; o = np.array([x[1] for x in conditions] + [0] * 4, dtype=np.int32)[:4]
    r = np.array([x[2] for x in conditions] + [0] * 4, dtype=np.int32)[:4]; rows = np.ascontiguousarray(rows, dtype=np.float64)
    msg = C.create_string_buffer(256)
    rc = core.cu_error(C.c_int(n_levels), C.c_int(len(conditions)), _ptr(c), _ptr(o), _ptr(r), C.c_int(len(rows)), _ptr(rows), msg, 256)
    return rc, msg.value.decode()


@pytest.mark.parametrize("col,v,why", [(0, 4.0, "start_level of robot 2: must be an integer in [0, 4)"), (0, 1.5, "start_level of robot 2: must be an integer in [0, 4)"),
                                       (0, -1.0, "start_level of robot 2: must be an integer in [0, 4)"), (1, 0.0, "up_after of robot 2: must be an integer in [1, 2^31)"),
                                       (2, 2.5, "down_after of robot 2: must be an integer in [1, 2^31)"), (2, np.inf, "down_after of robot 2: must be an integer in [1, 2^31)"),
                                       (5, np.nan, "threshold[2] of robot 2: must be finite")])
def test_row_check_names_the_field_and_the_robot(core, col, v, why):
    rows = np.tile([0.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.0], (4, 1))
    assert _err(core, rows) == (0, "")
    rows[2, col] = v
    assert _err(core, rows) == (1, why)


@pytest.mark.parametrize("n_levels,conditions,why", [(1, [], "rule n_levels must be >= 2"), (3, [(0, 0, 0)] * 5, "rule n_cond must lie in [0, 4]"),
                                                     (3, [(0, 0, 0), (18, 0, 0)], "rule column[1] must be a metrics column in [0, 18)"),
                                                     (3, [(3, 2, 0)], "rule op[0] must be QMB200_CURRICULUM_GE or QMB200_CURRICULUM_LE"),
                                                     (3, [(3, 1, -1)], "rule role[0] must be QMB200_CURRICULUM_PASS or QMB200_CURRICULUM_FAIL")])
def test_rule_check_names_the_field(core, n_levels, conditions, why):
    assert _err(core, np.tile([0.0, 1.0, 1.0, 0, 0, 0, 0], (2, 1)), n_levels, conditions) == (1, why)


def _attach_err(core, kind, base_lo, base_hi, top_lo, top_hi, n_levels, n_tiles=3):
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (base_lo, base_hi, top_lo, top_hi)]; msg = C.create_string_buffer(256)
    rc = core.cu_attach_error(C.c_int(kind), C.c_int(n_tiles), C.c_int(n_levels), C.c_int(len(a[0])), *(_ptr(x) for x in a), msg, 256)
    return rc, msg.value.decode()


def test_every_level_is_checked_and_the_first_failure_named(core):
    B = 3; lo = np.zeros((B, _lib.EPISODE)); lo[:, 0] = 0.8; hi = lo.copy(); hi[:, 0] = 1.0
    assert _attach_err(core, 0, lo, hi, lo, hi, 5) == (0, "")
    # friction lo 0.8 → -0.2: level 4 of 5 (exactly 0.0 at f = 0.8) is the first with lo <= 0
    tlo = lo.copy(); tlo[1, 0] = -0.2; thi = hi.copy()
    assert _attach_err(core, 0, lo, hi, tlo, thi, 6) == (1, "episode level 4: friction_mu of robot 1: lo must be > 0")
    # an interior level fails while both ends pass: lo and hi cross between them (lo 0 → 2, hi 3 → 1: lo > hi from f > 3/4)
    slo = np.zeros((B, 4)); shi = np.zeros((B, 4)); slo[:, 0] = shi[:, 0] = -1.0; slo[2, 1] = 0.0; shi[2, 1] = 3.0
    tlo, thi = slo.copy(), shi.copy(); tlo[2, 1] = 2.0; thi[2, 1] = 1.0
    r = _attach_err(core, 1, slo, shi, tlo, thi, 9)
    assert r == (1, "spawn level 7: dx of robot 2: lo must be <= hi"), r
    tlo, thi = slo.copy(), shi.copy(); thi[0, 0] = 3.0   # a tile beyond the library: hi -1 + 4 l / 3 rounds to 0, 2, then 3
    assert _attach_err(core, 1, slo, shi, tlo, thi, 4) == (1, "spawn level 3: tile of robot 0: bounds must lie in [-1, 3), the tiles of the library in force")
    tl = np.zeros((B, _lib.TIMELINE)); tl[:, TL["w_none"]] = 1.0; tl[:, TL["ee_qw"]] = 1.0; tl[:, TL["gait_set"]] = 5.0
    top = tl.copy(); top[1, TL["gait_set"]] = 4.0
    assert _attach_err(core, 2, tl, tl, top, top, 3) == (1, "timeline gait_set of robot 1: must be equal in the base and top boxes")
    top = tl.copy(); top[2, TL["ee_qz"]] = 1e-3
    assert _attach_err(core, 2, tl, tl, top, top, 3) == (1, "timeline ee_qz of robot 2: must be equal in the base and top boxes")
    top = tl.copy(); top[:, TL["w_none"]] = 0.0; top[:, TL["w_cmd_vel"]] = 2.0; top[0, TL["p_gait"]] = 0.5   # p_gait and weights may move
    assert _attach_err(core, 2, tl, tl, top, top, 3) == (0, "")


# ------------------------------------------------------------------------------------------------------------------------ closed_loop.run(curriculum=...)
RUN = dict(respawn=dict(every=0.2), randomize=dict(friction_mu=(0.5, 0.9)))
TOP = dict(friction_mu=(0.2, 0.9))


@pytest.mark.parametrize("bad,kw,match", [
    ([3], RUN, "curriculum must be None or dict"), (dict(levels=3, randomize=TOP, foo=1), RUN, "curriculum must be None or dict"),
    (dict(levels=3, randomize=TOP), dict(randomize=RUN["randomize"]), "needs respawn"),
    (dict(levels=3, randomize=TOP), dict(respawn=dict(hold=0.1), randomize=RUN["randomize"]), "needs respawn every"),
    (dict(levels=1, randomize=TOP), RUN, "levels must be an integer >= 2"), (dict(levels=3.0, randomize=TOP), RUN, "levels must be an integer"),
    (dict(levels=3, start=3, randomize=TOP), RUN, r"start must be an integer in \[0, 3\)"), (dict(levels=3, start=[0, 1], randomize=TOP), RUN, "start must be"),
    (dict(levels=3, up_after=0, randomize=TOP), RUN, "up_after must be"), (dict(levels=3, down_after=1.5, randomize=TOP), RUN, "down_after must be"),
    (dict(levels=3, when=[("distance", ">=", 1.0, "pass")], randomize=TOP), RUN, "when needs metrics=True"),
    (dict(levels=3), RUN, "at least one of"), (dict(levels=3, spawn=dict(yaw=(0, 1))), RUN, "curriculum spawn needs the run's own spawn"),
    (dict(levels=3, randomize=dict(seed=3, **TOP)), RUN, "top box's fields"), (dict(levels=3, randomize=dict(mu=(0, 1))), RUN, "unknown randomize field 'mu'"),
    (dict(levels=3, randomize=dict(friction_mu=(0.9, 0.2))), RUN, "finite with lo <= hi"), (dict(levels=3, randomize=dict(friction_mu=(0.0, 0.2))), RUN, "lo must be > 0"),
    (dict(levels=3, randomize=dict(friction_mu=(np.zeros(3), 1.0))), RUN, "scalars or"),
])
def test_closed_loop_rejects_a_malformed_curriculum_before_any_solver_call(bad, kw, match):
    s = mock.Mock(batch=4)
    with pytest.raises(ValueError, match=match):
        closed_loop.run(s, duration=0.02, curriculum=bad, **kw)
    assert s.mock_calls == []


@pytest.mark.parametrize("when,match", [([("dist", ">=", 1.0, "pass")], "unknown curriculum column 'dist'"), ([("distance", ">", 1.0, "pass")], "op must be one of"),
                                        ([("distance", ">=", 1.0, "win")], "role one of"), ([("distance", ">=", np.nan, "pass")], "must be a finite scalar"),
                                        ([("distance", ">=", 1.0)], r"\(column, op, threshold, role\)"), ([("distance", ">=", 1.0, "pass")] * 5, "at most 4")])
def test_closed_loop_rejects_malformed_conditions(when, match):
    s = mock.Mock(batch=4)
    with pytest.raises(ValueError, match=match):
        closed_loop.run(s, duration=0.02, metrics=True, curriculum=dict(levels=3, when=when, randomize=TOP), **RUN)
    assert s.mock_calls == []


def test_closed_loop_rejects_a_timeline_top_that_moves_its_gaits_or_quaternion():
    s = mock.Mock(batch=4); base = dict(n=2, t_first=(0.0, 0.1), gap=(0.1, 0.2), p_gait=0.5, gaits=["trot"])
    for top, match in ((dict(gaits=["pace"]), "gaits"), (dict(weights=dict(ee_goal=1.0), ee_x=(0, 1), ee_y=(0, 1), ee_z=(0, 1), ee_quat=(0, 0, 1.0, 0)), "ee_quat"),
                       (dict(n=3), "top box's fields"), (dict(gap=(-1.0, 0.0)), "gap lo must be >= 0")):
        with pytest.raises(ValueError, match=match):
            closed_loop.run(s, duration=0.02, respawn=dict(every=0.2), timeline=base, curriculum=dict(levels=3, timeline=top))
    ee = dict(weights=dict(none=1.0, ee_cmd_vel=1.0), ee_vx=(0, 0.1), ee_vy=(0, 0), ee_vz=(0, 0))
    with pytest.raises(ValueError, match="drawn spawn yaw"):   # the top box's end-effector commands meet the run's own drawn yaw
        closed_loop.run(s, duration=0.02, respawn=dict(every=0.2), timeline=base, spawn=dict(yaw=(-0.5, 0.5)), curriculum=dict(levels=3, timeline=ee))
    assert s.mock_calls == []


class _Stop(Exception):
    pass


def test_the_run_sets_the_curriculum_attaches_the_top_boxes_and_clears_it_first():
    """On a fake Solver: the run's ranges are level 0, the top box differs only in the named columns, the rule and rows are the spec's, and the
    curriculum is cleared before the scopes restore the previous ranges"""
    B = 4; log = []; st = dict(ranges=None)
    impl = dict(sim_get_robot_params=lambda: dict(friction_mu=None, payload=None), sim_set_robot_params=lambda **kw: log.append(("robot_params", kw)),
                sim_get_params=lambda: dict(friction_mu=0.7), episode_get_ranges=lambda: st["ranges"],
                episode_set_ranges=lambda lo=None, hi=None, seed=0: log.append(("episode_set_ranges", lo, hi, seed)),
                curriculum_set=lambda *a: log.append(("curriculum_set",) + a), robot_image_clear=lambda: log.append(("robot_image_clear",)),
                curriculum_attach=lambda *a: (log.append(("curriculum_attach",) + a), (_ for _ in ()).throw(_Stop)))
    s = mock.Mock(spec=list(impl), batch=B, _cfg=types.SimpleNamespace(device=0))
    for name, f in impl.items():
        getattr(s, name).side_effect = f
    cur = dict(levels=12, start=[0, 1, 2, 11], up_after=2, down_after=[1, 1, 3, 1], when=[("distance", ">=", [0.1, 0.2, 0.3, 0.4], "pass"), ("max_tilt", "<=", 0.5, "fail")],
               randomize=dict(f_base_x=(0.0, 255.0)))
    with pytest.raises(_Stop):
        closed_loop.run(s, duration=0.02, cmd_vel=(0.2, 0, 0, 0), metrics=True, respawn=dict(every=0.2), randomize=dict(seed=9, friction_mu=(0.5, 0.9)), curriculum=cur)
    names = [e[0] for e in log]
    assert names[names.index("episode_set_ranges"):] == ["episode_set_ranges", "curriculum_set", "curriculum_attach", "robot_image_clear", "curriculum_set",
                                                         "episode_set_ranges", "robot_params"]
    _, lo, hi, seed = log[names.index("episode_set_ranges")]
    _, L, rows, conditions = log[names.index("curriculum_set")]
    _, kind, tlo, thi = log[names.index("curriculum_attach")]
    EP = {n: i for i, n in enumerate(_lib.EPISODE_LAYOUT)}
    assert seed == 9 and L == 12 and kind == "episode" and conditions == [("distance", ">=", "pass"), ("max_tilt", "<=", "fail")]
    np.testing.assert_array_equal(rows, np.c_[[0, 1, 2, 11], np.full(4, 2), [1, 1, 3, 1], [0.1, 0.2, 0.3, 0.4], np.full(4, 0.5), np.zeros((4, 2))])
    assert lo[:, EP["f_base_x"]].tolist() == [0] * 4 and thi[:, EP["f_base_x"]].tolist() == [255.0] * 4 and tlo[:, EP["f_base_x"]].tolist() == [0] * 4
    other = [c for c in range(_lib.EPISODE) if c != EP["f_base_x"]]
    assert tlo[:, other].tobytes() == lo[:, other].tobytes() and thi[:, other].tobytes() == hi[:, other].tobytes()
    assert log[names.index("curriculum_set") + 3] == ("curriculum_set",)   # cleared, then the previous ranges (none) restored
    assert log[names.index("curriculum_set") + 4][1:] == (None, None, 0)


def test_entry_points_are_bound_and_declared():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name
    assert "#define QMB200_CURRICULUM 7" in h and len(_lib.CURRICULUM_LAYOUT) == _lib.CURRICULUM == 7
    assert "#define QMB200_CURRICULUM_STATE 4" in h and len(_lib.CURRICULUM_STATE_LAYOUT) == _lib.CURRICULUM_STATE == 4
    for i, k in enumerate(_lib.CURRICULUM_KINDS):
        assert "#define QMB200_CURRICULUM_%s %d" % (k.upper(), i) in h
    assert C.sizeof(_lib.CurriculumRule) == 4 * 14


def test_update_kernel_compiles_for_sm90a_without_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    obj = str(tmp_path / "curriculum.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "kernels", "curriculum_kernel.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    assert any("curriculum_update_kernel" in k for k in kernels), r.stderr
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == len(kernels) and all(f == ("0", "0", "0") for f in frames), r.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if os.path.exists(cuobjdump):
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
        assert not re.search(r"\b(LDL|STL)\b", sass)
