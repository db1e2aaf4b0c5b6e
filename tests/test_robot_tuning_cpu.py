"""Per-robot controller tuning on the host, no GPU: the row layout of the header, the bindings and the kernels' Tuning block; the node evaluator's cost
value with a row (tests/tuning_host.cpp) against the oracle built from a task.info edited to that row; closed_loop.run(tuning=...) on a fake Solver."""
import ctypes as C
import os
import re
import subprocess
import types
from unittest import mock

import numpy as np
import pytest

from _oracle import GAINS, REFERENCE, ROOT, TASK, URDF, Oracle, _d, _i, f64, i32
from _tuning import L, edited_files
from qm_control_b200 import _lib, closed_loop, synthetic

CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "tuning_host.cpp")
LIB = os.path.join(ROOT, "tests", "_build", "libtuninghost.so")
B = 4
# a row far from the handle's values in every field the cost reads (friction below the task file's 0.3, other end-effector weights)
ROW = np.r_[0.15, 0.6, 500.0, 3000.0, 8000.0, 250.0, np.arange(32) + 10.0, 7.0, 2.5]


def test_header_row_layout_matches_the_bindings_and_the_kernels():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    assert int(re.search(r"#define QMB200_TUNING (\d+)", h).group(1)) == _lib.TUNING == 40
    assert [k for k in L][:6] == ["friction_mu", "wbc_friction", "mu_ee_pos", "mu_ee_ori", "mu_final_ee_pos", "mu_final_ee_ori"]
    assert list(L)[6:20] == [n for n, _ in _lib.WbcGains._fields_] and L["kp_arm_joint"] == (14, 6) and L["kd_ee_angular"] == (35, 3)
    assert L["kp_arm_wbc"] == (38, 1) and L["kd_arm_wbc"] == (39, 1)
    assert C.sizeof(_lib.WbcGains) == 32 * 8
    dc = open(os.path.join(CSRC, "kernels", "dev_common.cuh")).read()
    assert "constexpr int TUNING_MODEL = 38, TUNING_DBL = 40, TUNING_ARM_KP = 38, TUNING_ARM_KD = 39;" in dc
    assert re.search(r"static_assert\(sizeof\(Tuning\) == TUNING_MODEL \* 8", dc)
    for name in ("qmb200_set_robot_tuning", "qmb200_get_robot_tuning", "qmb200_get_handle_tuning"):
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h)


@pytest.fixture(scope="module")
def tun():
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-I" + CSRC, "-o", LIB, SRC,
                           os.path.join(CSRC, "host", "qm_config.cpp")])
    lib = C.CDLL(LIB); lib.tun_create.restype = C.c_void_p; lib.tun_cost.restype = C.c_double
    hs = []

    def create(task=TASK, gains=GAINS):
        h = lib.tun_create(task.encode(), URDF.encode(), REFERENCE.encode(), gains.encode()); assert h; hs.append(h); return C.c_void_p(h)
    yield lib, create
    for h in hs:
        lib.tun_destroy(C.c_void_p(h))


def _cost(lib, h, row, et, md, tt, ts, t, x, u, terminal):
    return lib.tun_cost(h, None if row is None else _d(f64(row)), C.c_int(len(et)), _d(f64(et)), _i(i32(md)), C.c_int(len(tt)), _d(f64(tt)), _d(f64(ts)), C.c_double(float(t)),
                        _d(f64(x)), _d(f64(u)), C.c_int(terminal))


def test_cost_value_with_a_row_equals_the_oracle_on_the_edited_task_file(tun, tmp_path):
    """Along an oracle solution: cost_value with ROW on the file's model equals the oracle built from task.info edited to ROW (1e-11 relative) and,
    bit for bit, cost_value without a row on a model parsed from the edited files."""
    lib, create = tun
    task, gains = edited_files(tmp_path, ROW, "row")
    base, edited = create(), create(task, gains)
    o = Oracle(task=task); o.mpc_set(dt=0.015, horizon=1.0)
    prob, _ = synthetic.make_batch(np.array([2]), config=5)
    sol = o.mpc_solve_batch(prob, 100, nthreads=1); n = int(sol["n_nodes"][0]); t = sol["t"][0, :n]; ev = sol["event"][0, :n]
    ne = int(prob["n_events"][0]); et = prob["event_times"][0, :ne]; md = prob["modes"][0, :ne + 1]; nk = int(prob["n_target"][0]); tt = prob["target_times"][0, :nk]; ts = prob["target_states"][0, :nk]
    checked = 0; differs = 0
    for k in range(0, n - 1, 4):
        if ev[k] == 1:
            continue
        tk = t[k] + (1e-6 if ev[k] == 2 else 0.0); x = sol["x"][0, k]; u = sol["u"][0, k]
        fo, _, _, _ = o.stage_probe(et, md, tt, ts, tk, x, u, want_grad=False)
        c = _cost(lib, base, ROW, et, md, tt, ts, tk, x, u, 0)
        assert abs(c - fo) <= 1e-11 * max(1.0, abs(fo)), (k, c, fo)
        assert c == _cost(lib, edited, None, et, md, tt, ts, tk, x, u, 0)
        differs += c != _cost(lib, base, None, et, md, tt, ts, tk, x, u, 0); checked += 1
    assert checked >= 10 and differs == checked   # the row changes every node's cost: the comparison is not vacuous
    x = sol["x"][0, n - 1]; c = _cost(lib, base, ROW, et, md, tt, ts, t[n - 1], x, np.zeros(30), 1)   # the final cost reads the final weights
    assert c == _cost(lib, edited, None, et, md, tt, ts, t[n - 1], x, np.zeros(30), 1) != _cost(lib, base, None, et, md, tt, ts, t[n - 1], x, np.zeros(30), 1)


def test_the_handle_row_through_the_pointer_is_the_model_bit_for_bit(tun):
    """A row holding the model's own values gives the cost of no row, bit for bit"""
    lib, create = tun
    h = create(); row = np.zeros(40)
    vals = dict(friction_mu=0.3, wbc_friction=0.3, mu_ee_pos=2000.0, mu_ee_ori=1000.0, mu_final_ee_pos=2000.0, mu_final_ee_ori=1000.0)   # qm_task.info
    for k, v in vals.items():
        row[L[k][0]] = v
    prob, _ = synthetic.make_batch(np.array([1]), config=4)
    rng = np.random.default_rng(2); ne = int(prob["n_events"][0]); nk = int(prob["n_target"][0])
    args = (prob["event_times"][0, :ne], prob["modes"][0, :ne + 1], prob["target_times"][0, :nk], prob["target_states"][0, :nk])
    for j in range(20):
        t = float(prob["t0"][0]) + 0.05 * j; x = prob["x0"][0] + rng.uniform(-0.05, 0.05, 30); u = np.r_[np.tile([3.0, -2.0, 70.0], 4), rng.uniform(-0.2, 0.2, 18)]
        for term in (0, 1):
            assert _cost(lib, h, row, *args, t, x, u, term) == _cost(lib, h, None, *args, t, x, u, term)


# ---------------------------------------------------------------------------------------------------------------------------- closed_loop.run(tuning=...)
HANDLE_ROW = np.arange(40, dtype=np.float64) + 1.0


def _fake(rows=None, robot_mu=None, plant_mu=0.6):
    """→ (solver, state): set / get semantics of Solver.set_robot_tuning / get_robot_tuning; solver.mock_calls logs every call in order."""
    st = dict(rows=rows, robot_params=dict(friction_mu=robot_mu, payload=None))

    def set_tuning(tuning=None):
        if tuning is None:
            st["rows"] = None; return
        r = np.repeat(HANDLE_ROW[None], B, axis=0)
        for k, v in tuning.items():
            off, w = L[k]; a = np.asarray(v, dtype=np.float64); r[:, off:off + w] = a.reshape(B, 1) if w == 1 and a.shape == (B,) else a
        st["rows"] = r

    def get_tuning():
        return None if st["rows"] is None else {k: st["rows"][:, off] if w == 1 else st["rows"][:, off:off + w] for k, (off, w) in L.items()}
    impl = dict(set_robot_tuning=set_tuning, get_robot_tuning=get_tuning, sim_get_robot_params=lambda: st["robot_params"],
                sim_set_robot_params=lambda friction_mu=None, payload=None: st.update(robot_params=dict(friction_mu=friction_mu, payload=payload)),
                sim_get_params=lambda: dict(friction_mu=plant_mu))
    solver = mock.Mock(spec=list(impl), batch=B, _cfg=types.SimpleNamespace(device=0))
    for name, f in impl.items():
        getattr(solver, name).side_effect = f
    return solver, st


@pytest.mark.parametrize("tuning,match", [
    ([0.3], "tuning must be a dict"),
    (dict(no_such_field=1.0), "unknown tuning field 'no_such_field'"),
    (dict(friction_mu=0.0), "friction_mu must be finite and > 0"),
    (dict(wbc_friction=[0.3, -0.1, 0.3, 0.3]), "wbc_friction must be finite and > 0"),
    (dict(mu_ee_pos=np.nan), "mu_ee_pos must be finite and >= 0"),
    (dict(kd_arm_wbc=-0.5), "kd_arm_wbc must be finite and >= 0"),
    (dict(kp_ee_linear=np.ones(4)), r"kp_ee_linear must be a scalar, \[3\] or \[4, 3\]"),
    (dict(kp_swing=np.ones(3)), r"kp_swing must be a scalar, \[4\]"),
    (dict(mu_ee_ori="plant"), "mu_ee_ori must be numbers, got 'plant'"),
    (dict(friction_mu="told"), "friction_mu must be numbers or \"plant\""),
])
def test_malformed_tuning_raises_before_any_solver_call(tuning, match):
    s, _ = _fake()
    with pytest.raises(ValueError, match=match):
        closed_loop.run(s, duration=0.01, tuning=tuning)
    assert s.mock_calls == []


@pytest.mark.parametrize("prev", [None, np.full((B, 40), 2.0)])
def test_previous_rows_are_restored_when_the_run_fails(prev):
    s, st = _fake(rows=None if prev is None else prev.copy())
    with pytest.raises(ValueError, match="cmd_vel must have shape"):
        closed_loop.run(s, duration=0.01, cmd_vel=np.zeros(3), tuning=dict(mu_ee_pos=[1.0, 2.0, 3.0, 4.0], kp_ee_linear=[1.0, 2.0, 3.0]))
    assert [c[0] for c in s.mock_calls] == ["get_robot_tuning", "set_robot_tuning", "set_robot_tuning"]
    told = s.mock_calls[1][1][0]; np.testing.assert_array_equal(told["mu_ee_pos"], [1.0, 2.0, 3.0, 4.0]); np.testing.assert_array_equal(told["kp_ee_linear"], [1.0, 2.0, 3.0])
    if prev is None:
        assert st["rows"] is None
    else:
        np.testing.assert_array_equal(st["rows"], prev)


@pytest.mark.parametrize("run_mu,robot_mu,want", [(np.array([0.15, 0.2, 0.25, 0.3]), np.full(B, 0.9), [0.15, 0.2, 0.25, 0.3]),   # this run's friction_mu
                                                  (0.4, None, [0.4] * B),
                                                  (None, np.array([0.5, 0.6, 0.7, 0.8]), [0.5, 0.6, 0.7, 0.8]),                       # the handle's robot params
                                                  (None, None, [0.6] * B)])                                                            # the plant params
def test_plant_resolves_to_the_runs_friction(run_mu, robot_mu, want):
    s, _ = _fake(robot_mu=robot_mu)
    with pytest.raises(ValueError, match="cmd_vel must have shape"):
        closed_loop.run(s, duration=0.01, cmd_vel=np.zeros(3), friction_mu=run_mu, tuning=dict(friction_mu="plant", wbc_friction="plant", kd_arm_wbc=0.7))
    told = [c for c in s.mock_calls if c[0] == "set_robot_tuning"][0][1][0]
    np.testing.assert_array_equal(told["friction_mu"], want); np.testing.assert_array_equal(told["wbc_friction"], want); assert told["kd_arm_wbc"] == 0.7


def test_without_tuning_the_loop_makes_no_tuning_call():
    s, _ = _fake()
    with pytest.raises(ValueError, match="cmd_vel must have shape"):
        closed_loop.run(s, duration=0.01, cmd_vel=np.zeros(3))
    assert s.mock_calls == []


@pytest.mark.parametrize("B_,field_,w", [(3, "kp_ee_linear", 3), (6, "kd_arm_joint", 6)])
def test_a_vector_gain_of_k_values_is_per_axis_also_when_the_batch_has_k_robots(B_, field_, w):
    """Solver.robot_tuning_rows with B == k: [k] is the per-axis form, the same for every robot; [B, k] is per robot"""
    from qm_control_b200.interface import Solver
    handle = np.arange(40, dtype=np.float64) + 1.0
    fake = types.SimpleNamespace(batch=B_, get_handle_tuning=lambda: handle.copy())
    off = L[field_][0]; per_axis = np.arange(w) + 100.0
    rows = Solver.robot_tuning_rows(fake, {field_: per_axis, "friction_mu": np.arange(B_) + 0.5})
    np.testing.assert_array_equal(rows[:, off:off + w], np.repeat(per_axis[None], B_, axis=0))
    np.testing.assert_array_equal(rows[:, L["friction_mu"][0]], np.arange(B_) + 0.5)
    per_robot = np.arange(B_ * w, dtype=np.float64).reshape(B_, w)
    np.testing.assert_array_equal(Solver.robot_tuning_rows(fake, {field_: per_robot})[:, off:off + w], per_robot)
    others = [i for i in range(40) if not off <= i < off + w]
    np.testing.assert_array_equal(Solver.robot_tuning_rows(fake, {field_: per_robot})[:, others], np.repeat(handle[None, others], B_, axis=0))
