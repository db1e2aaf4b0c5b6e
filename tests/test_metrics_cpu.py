"""Per-episode metrics on the host, no GPU (DESIGN.md §4.13): the per-robot core compiled with g++ (tests/metrics_host.cpp) against the numpy statement
of the column table (tests/_metrics_twin.py) on random step / close sequences, closed_loop.run(metrics=...) validation and its episode bound on a fake
Solver, the bindings and the kernels' resources."""
import ctypes as C
import os
import re
import shutil
import subprocess
from unittest import mock

import numpy as np
import pytest

import _metrics_twin as mtw
from _oracle import GAINS, REFERENCE, TASK, URDF, Oracle
from qm_control_b200 import _lib, closed_loop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
NAMES = ("qmb200_metrics_step", "qmb200_metrics_step_dev", "qmb200_metrics_close", "qmb200_metrics_close_dev")
ACC, METRICS = _lib.METRICS_ACC, _lib.METRICS


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("metrics") / "libmetricshost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-I" + CSRC,
                           "-o", lib_path, os.path.join(ROOT, "tests", "metrics_host.cpp"), os.path.join(CSRC, "host", "qm_config.cpp")])
    lib = C.CDLL(lib_path); lib.mt_create.restype = C.c_void_p
    return lib


@pytest.fixture(scope="module")
def model(core):
    h = core.mt_create(TASK.encode(), URDF.encode(), REFERENCE.encode(), GAINS.encode()); assert h
    yield C.c_void_p(h)
    core.mt_destroy(C.c_void_p(h))


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _step(core, model, tiles, cell, rows, ground_height, dt, inp, acc):
    a = acc.copy(); B = len(a); ny, nx = (0, 0) if tiles is None else tiles.shape[1:]
    core.mt_step(model, _ptr(tiles), C.c_int(nx), C.c_int(ny), C.c_double(cell or 0.0), _ptr(rows), C.c_double(ground_height), C.c_int(B), C.c_double(dt),
                 *(_ptr(inp[k]) for k in ("rbd", "contact", "effort", "cmd", "kind", "n_target", "target_times", "target_states", "time", "status", "rbd_est")),
                 _ptr(a))
    return a


def _close(core, mask, end, episode, acc, out, status):
    a, o, s = acc.copy(), out.copy(), status.copy()
    core.mt_close(C.c_int(len(a)), _ptr(mask), _ptr(end), _ptr(episode), C.c_int(o.shape[1]), _ptr(a), _ptr(o), _ptr(s))
    return a, o, s


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _inputs(rng, oracle, B, prev_rbd):
    """one step's random inputs of B robots: a pose that moves from the previous one (so the displacement terms see steps of a few cm), contact masks,
    targets of 0..5 knots with times before, between and after the sample's time, quaternion pairs on both sides of the sign flip and near each other,
    kinds -1..2 or NULL, an estimate or NULL"""
    q0 = oracle.model_info()["q_nominal"]
    r = prev_rbd.copy()
    r[:, 3:5] += rng.normal(0.0, 0.02, (B, 2)); r[:, 5] = rng.uniform(0.15, 0.6, B)
    r[:, 0] = rng.uniform(-np.pi, np.pi, B); r[:, 1:3] = rng.uniform(-0.6, 0.6, (B, 2))
    r[:, 6:24] = q0[6:] + rng.uniform(-0.4, 0.4, (B, 18)); r[:, 24:48] = rng.normal(0.0, 1.0, (B, 24))
    r[:, 48:51] = r[:, 3:6] + rng.uniform(-0.6, 0.6, (B, 3)); r[:, 51:55] = _unit(rng.normal(size=(B, 4)))
    n = rng.integers(0, 6, B).astype(np.int32)
    gaps = rng.uniform(1e-3, 0.3, (B, _lib.KMAX)); tt = 10.0 + np.cumsum(gaps, axis=1)
    ts = rng.normal(0.0, 0.5, (B, _lib.KMAX, _lib.TARGET)); ts[:, :, 33:37] = _unit(rng.normal(size=(B, _lib.KMAX, 4)))
    near = rng.random(B) < 0.2   # next knot's quaternion within ~1e-9 of the first, or its negation: the slerp's blend branch and its sign
    ts[near, 1, 33:37] = ts[near, 0, 33:37] * rng.choice([-1.0, 1.0], (near.sum(), 1)) + rng.normal(0.0, 1e-10, (near.sum(), 4))
    time = tt[:, 0] + rng.uniform(-0.2, 1.2, B) * (tt[:, -1] - tt[:, 0]) - 1e-3
    at = rng.random(B) < 0.1; time[at] = tt[at, 1] - 1e-3   # samples exactly on a knot
    status = rng.integers(-2 ** 31, 2 ** 31, B).astype(np.int32) * (rng.random(B) < 0.3)
    kind = None if rng.random() < 0.3 else rng.integers(-1, 3, B).astype(np.int32)
    est = None if rng.random() < 0.4 else r + rng.normal(0.0, 0.01, r.shape)
    return dict(rbd=r, contact=rng.integers(0, 16, B).astype(np.int32), effort=rng.normal(0.0, 20.0, (B, 18)), cmd=rng.normal(0.0, 0.5, (B, 7)), kind=kind,
                n_target=n, target_times=tt, target_states=ts, time=time, status=status.astype(np.int32), rbd_est=est)


def _assert_close(got, want, what):
    assert got.shape == want.shape
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    err = np.abs(got[~nan] - want[~nan]) / np.maximum(np.abs(want[~nan]), 1.0)
    assert err.size == 0 or err.max() <= 1e-12, (what, err.max())


def test_core_equals_the_numpy_statement_on_random_sequences(core, model):
    """3000 robots through 6 rounds of a step of every robot (a random terrain row per robot and round, some on the plane) and a close of a random subset
    (random ends, some invalid; episode indices inside and outside the out rows; some accumulators still empty)"""
    oracle = Oracle(); rng = np.random.default_rng(11); B, E = 3000, 4
    tiles = rng.uniform(-0.1, 0.1, (3, 10, 12)); cell = 0.1; ground_height = 0.02
    twin = mtw.MetricsTwin(oracle, tiles, cell, ground_height)
    acc_g = np.zeros((B, ACC)); acc_w = acc_g.copy(); out_g = np.full((B, E, METRICS), np.nan); out_w = out_g.copy()
    st_g = np.zeros(B, dtype=np.int32); st_w = st_g.copy()
    rbd = np.zeros((B, 55)); seen = dict(changed_row=False, empty_closed=False, overflow=False, refused=False, cmd_none=False)
    rows = np.c_[rng.integers(-1, 3, B), rng.uniform(-0.5, 0.0, (B, 2))].astype(np.float64)
    for rnd in range(6):
        skip = rng.random(B) < 0.15   # robots without a sample this round: they keep an empty or older accumulator
        inp = _inputs(rng, oracle, B, rbd); rbd = inp["rbd"]
        new_rows = rows.copy(); move = rng.random(B) < 0.5
        new_rows[move, 0] = rng.integers(-1, 3, move.sum()); new_rows[move, 1:] = rng.uniform(-0.5, 0.0, (move.sum(), 2))
        seen["changed_row"] |= bool(np.any(new_rows[:, 0] != rows[:, 0])); rows = new_rows
        dt = float(rng.choice([1e-3, 2.5e-4]))
        g = _step(core, model, tiles, cell, rows, ground_height, dt, inp, acc_g)
        w = twin.step(acc_w, dt, **inp, terrain_rows=rows)
        acc_g = np.where(skip[:, None], acc_g, g); acc_w = np.where(skip[:, None], acc_w, w)
        _assert_close(acc_g, acc_w, "accumulators after step %d" % rnd)
        seen["cmd_none"] |= bool(np.any((acc_w[:, mtw.N] > 0) & (acc_w[:, mtw.N_CMD] == 0)))
        mask = (rng.random(B) < 0.4).astype(np.int32); end = rng.integers(-1, 4, B).astype(np.int32); episode = rng.integers(-1, E + 1, B).astype(np.int32)
        seen["empty_closed"] |= bool(np.any(mask.astype(bool) & (acc_w[:, mtw.N] == 0) & (end >= 0) & (end <= 2)))
        seen["overflow"] |= bool(np.any(mask.astype(bool) & ((episode < 0) | (episode >= E)) & (end >= 0) & (end <= 2)))
        seen["refused"] |= bool(np.any(mask.astype(bool) & ((end < 0) | (end > 2))))
        acc_g, out_g, st_g = _close(core, mask, end, episode, acc_g, out_g, st_g)
        acc_w, out_w, st_w = mtw.close(mask, end, episode, acc_w, out_w, st_w)
        _assert_close(acc_g, acc_w, "accumulators after close %d" % rnd); _assert_close(out_g, out_w, "rows after close %d" % rnd)
        np.testing.assert_array_equal(st_g, st_w)
    assert all(seen.values()), seen
    filled = ~np.isnan(out_w[..., 0])
    assert filled.sum() > 1000 and np.any(np.isnan(out_w[filled][:, 7])) and np.any(out_w[filled][:, 15] > 0) and np.any(out_w[filled][:, 14] > 0)


def test_one_sample_episodes_and_one_knot_targets(core, model):
    """a single sample: distance 0, path 0, slip 0, no touchdowns; a one-knot target is its knot at any time; status words OR bit for bit"""
    oracle = Oracle(); rng = np.random.default_rng(5); B = 16
    inp = _inputs(rng, oracle, B, np.zeros((B, 55))); inp["n_target"][:] = 1; inp["rbd_est"] = None; inp["kind"] = None
    inp["status"] = np.array([0, 1, -1, 2 ** 30] * 4, dtype=np.int32)
    acc = _step(core, model, None, None, None, 0.0, 1e-3, inp, np.zeros((B, ACC)))
    _, out, _ = _close(core, np.ones(B, np.int32), np.zeros(B, np.int32), np.zeros(B, np.int32), acc, np.full((B, 1, METRICS), np.nan), np.zeros(B, np.int32))
    row = out[:, 0]
    np.testing.assert_array_equal(row[:, [0, 1, 3, 4, 14, 15]], np.tile([1e-3, 0, 0, 0, 0, 0], (B, 1)))
    np.testing.assert_array_equal(row[:, 2], (inp["status"].astype(np.int64) & 0xFFFFFFFF).astype(np.float64))
    pe = np.linalg.norm(inp["rbd"][:, 48:51] - inp["target_states"][:, 0, 30:33], axis=1)
    np.testing.assert_allclose(row[:, 9], pe, rtol=1e-14); np.testing.assert_array_equal(row[:, 9], row[:, 10])
    assert np.all(np.isnan(row[:, 16:18]))


# --------------------------------------------------------------------------------------------------------------------------- closed_loop.run(metrics=...)
@pytest.mark.parametrize("value", [False, 1, "yes", dict(), [True]])
def test_closed_loop_rejects_anything_but_true_before_any_solver_call(value):
    s = mock.Mock(spec=[], batch=4)
    with pytest.raises(ValueError, match="metrics must be None or True"):
        closed_loop.run(s, duration=0.02, metrics=value)
    assert s.mock_calls == []


@pytest.mark.parametrize("respawn,ticks,want", [
    (None, 30, 1), (True, 30, 3), (dict(hold=0.05), 30, 6), (dict(every=0.2), 30, 3), (dict(every=0.05, hold=0.2), 31, 7),
    (dict(on_fall=False, every=0.1), 30, 3), (dict(on_fall=False, every=0.1), 31, 4), (dict(hold=0.01), 1, 1), (dict(hold=0.01), 5, 5)])
def test_episode_rows_bound_the_episodes_a_spec_allows(respawn, ticks, want):
    """every episode but the last lasts at least min(hold, every) windows and a robot restarts only at a window boundary before the last window's end"""
    rs = None if respawn is None else closed_loop._respawn_spec(respawn)
    assert closed_loop._metrics_episodes(ticks, rs) == want


def test_entry_points_are_bound_and_declared():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name
    assert "#define QMB200_METRICS 18" in h and "#define QMB200_METRICS_ACC 32" in h and _lib.METRICS == 18 and _lib.METRICS_ACC == 32
    assert _lib.METRICS_LAYOUT[:3] == ("duration", "end", "status") and _lib.METRICS_LAYOUT[-2:] == ("est_pos_err_rms", "est_vel_err_rms")
    for i, name in enumerate(_lib.METRICS_LAYOUT):   # the header's column table names the columns in the same order
        assert re.search(r"\*\s+%d\s+%s\s" % (i, name), h), name
    assert len(_lib.PROTOTYPES["qmb200_metrics_step"][1]) == 14 and len(_lib.PROTOTYPES["qmb200_metrics_step_dev"][1]) == 15
    assert len(_lib.PROTOTYPES["qmb200_metrics_close"][1]) == 8 and len(_lib.PROTOTYPES["qmb200_metrics_close_dev"][1]) == 9


def test_metrics_kernels_compile_for_sm90a_without_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    obj = str(tmp_path / "metrics.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "kernels", "metrics_kernel.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    assert any("metrics_step_kernel" in k for k in kernels) and any("metrics_close_kernel" in k for k in kernels), r.stderr
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == len(kernels) and all(f == ("0", "0", "0") for f in frames), r.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if os.path.exists(cuobjdump):
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
        assert not re.search(r"\b(LDL|STL)\b", sass)
