"""The online payload estimator on the host, no GPU: the arm-row regressor against the plant twin's dynamics, the RLS restatement on exact data, the
parameter struct's layout, and the SRBD payload fold the host and the commit kernel share (qmb200_debug_srbd_constants) against a numpy restatement."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from qm_control_b200 import _lib
from _payload_est_twin import PayloadEstTwin, point_mass_theta
from _sim_twin_ext import SimTwinExt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def twin():
    return PayloadEstTwin()


@pytest.fixture(scope="module")
def plant():
    return SimTwinExt()


def _djs():
    from _oracle import REFERENCE
    txt = open(REFERENCE).read()
    import re
    block = txt[txt.index("defaultJointState"):]
    return np.array([float(m) for m in re.findall(r"\(\d+,0\)\s+([-\d.eE+]+)", block)[:18]])


def _random_state(rng, z):
    q = np.r_[rng.uniform(-0.2, 0.2, 2), z, rng.uniform(-3.0, 3.0), rng.uniform(-0.15, 0.15, 2), _djs() + rng.uniform(-0.3, 0.3, 18)]
    v = np.r_[rng.uniform(-0.5, 0.5, 3), rng.uniform(-1.0, 1.0, 3), rng.uniform(-2.0, 2.0, 18)]
    return q, v


def _rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-12)


def test_regressor_identity_on_the_plant_dynamics(twin, plant):
    """With an EE point mass, a base payload and a base wrench in the plant, the nominal arm residual y_a equals Phi(q, v, qdd) theta_true at the plant's
    acceleration, feet in and out of contact, efforts inside and beyond the limits; an EE wrench breaks the identity (the documented limitation)."""
    rng = np.random.default_rng(7); masks = set()
    for k in range(24):
        q, v = _random_state(rng, z=0.42 if k % 2 else 0.8)
        m, o = rng.uniform(0.2, 2.5), rng.uniform(-0.1, 0.1, 3)
        payload = np.r_[m, o, rng.uniform(0.5, 4.0), rng.uniform(-0.2, 0.2, 3)]
        wrench = np.r_[rng.uniform(-60, 60, 6), np.zeros(6)]
        effort = rng.uniform(-120, 120, 18)
        qdd, _, mask = plant.accel_ext(effort, q, v, payload=payload, wrench=wrench); masks.add(mask != 0)
        y, Phi = twin.residual_and_regressor(q, v, qdd, effort)
        assert _rel(Phi @ point_mass_theta(m, o), y) < 1e-9, k
        ee_push = wrench.copy(); ee_push[6:9] = (0.0, 0.0, 30.0)
        qdd_p, _, _ = plant.accel_ext(effort, q, v, payload=payload, wrench=ee_push)
        y_p, Phi_p = twin.residual_and_regressor(q, v, qdd_p, effort)
        assert _rel(Phi_p @ point_mass_theta(m, o), y_p) > 1e-3, k
    assert masks == {True, False}, "both contact cases must occur"


def test_rls_with_unit_forgetting_recovers_theta_on_exact_data(twin, plant):
    """lambda = 1, a wide prior and exact accelerations over random excitation: theta_true to 1e-8 (a full inertia tensor, not only a point mass)."""
    rng = np.random.default_rng(11)
    est = PayloadEstTwin(forgetting=1.0, p0_mass=1e8, p0_first_moment=1e8, p0_inertia=1e8, trace_max=1e12)
    theta_true = point_mass_theta(1.3, [0.02, -0.04, 0.06]) + np.r_[0, 0, 0, 0, 0.01, 0.002, -0.001, 0.02, 0.003, 0.015]
    s = est.reset(np.zeros(8))
    for k in range(200):
        q, v = _random_state(rng, z=0.8)
        qdd = rng.uniform(-20, 20, 24)
        _, Phi = twin.residual_and_regressor(q, v, qdd, np.zeros(18))
        assert est.rls(s, Phi @ theta_true, Phi) == 0
    assert np.max(np.abs(s["theta"] - theta_true)) < 1e-8 * np.max(np.abs(theta_true)), s["theta"] - theta_true


def test_static_pose_recovers_mass_and_horizontal_first_moment(twin):
    """One static pose (v = 0, qdd = 0), default parameters: gravity alone excites m and the horizontal components of m c; theta does not move along the
    unexcited directions (m c along gravity, the inertia) and P's trace stays within trace_max."""
    est = PayloadEstTwin(); rng = np.random.default_rng(5)
    q, _ = _random_state(rng, z=0.8); v = np.zeros(24)
    theta_true = point_mass_theta(1.7, [0.03, 0.05, -0.02])
    _, Phi = twin.residual_and_regressor(q, v, np.zeros(24), np.zeros(18))
    s = est.reset(np.zeros(8)); th0 = s["theta"].copy()
    for _ in range(3000):
        assert est.rls(s, Phi @ theta_true, Phi) == 0
        assert np.trace(s["P"]) <= est.params["trace_max"] * (1 + 1e-12)
    d = twin.rbd(q, v); g_local = d["R"].T @ np.array([0.0, 0.0, 1.0])
    assert abs(s["theta"][0] - 1.7) < 1e-5   # the prior's pull decays as the forgetting discounts it: 2.7e-6 kg left after 3 s of samples
    horiz = lambda h: h - (h @ g_local) * g_local
    assert np.max(np.abs(horiz(s["theta"][1:4]) - horiz(theta_true[1:4]))) < 1e-5
    assert abs((s["theta"][1:4] - th0[1:4]) @ g_local) < 1e-9 and np.max(np.abs(s["theta"][4:] - th0[4:])) < 1e-9


def test_params_layout_matches_the_header(tmp_path):
    fields = [n for n, _ in _lib.PayloadEstParams._fields_]
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "qmb200.h"', 'int main(void) {', '  printf("%zu\\n", sizeof(qmb200_payload_est_params));']
    body += ['  printf("%%zu\\n", offsetof(qmb200_payload_est_params, %s));' % f for f in fields] + ['  return 0; }']
    src = tmp_path / "layout.c"; src.write_text("\n".join(body) + "\n"); exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert out[0] == C.sizeof(_lib.PayloadEstParams) and out[1:] == [getattr(_lib.PayloadEstParams, f).offset for f in fields]
    assert fields == ["forgetting", "p0_mass", "p0_first_moment", "p0_inertia", "trace_max", "mass_min", "mass_max", "offset_max"]
    assert len(_lib.THETA_LAYOUT) == 10


def _cfg():
    return _lib.Config(_lib.asset("qm_task.info").encode(), _lib.asset("qm_robot.urdf").encode(), _lib.asset("qm_reference.info").encode(), None, 1, 0, 0.0, 0.0, 0, 0)


def _srbd(rows):
    lib = _lib.load_library(); cfg = _cfg()
    pl = None if rows is None else np.ascontiguousarray(rows, dtype=np.float64).reshape(-1, 8)
    n = 1 if pl is None else len(pl); out = np.full((n, 24), np.nan)
    assert lib.qmb200_debug_srbd_constants(C.byref(cfg), n, None if pl is None else pl.ctypes.data, out.ctypes.data) == 0
    return out


def fold_numpy(nominal, R_ee, p_ee, row):
    """the point masses of row added to the nominal SRBD block by the parallel-axis theorem; the EE frame at (R_ee, p_ee), the base frame at the origin, level"""
    m, I, c = nominal[0], nominal[1:10].reshape(3, 3), -nominal[19:22]
    for mp, pos in ((row[0], p_ee + R_ee @ row[1:4]), (row[4], row[5:8])):
        if mp == 0.0:
            continue
        mt = m + mp; cn = (m * c + mp * pos) / mt
        par = lambda mm, d: mm * (d @ d * np.eye(3) - np.outer(d, d))
        I = I + par(m, c - cn) + par(mp, pos - cn); m, c = mt, cn
    return np.r_[m, I.ravel(), np.linalg.inv(I).ravel(), -c, 0.0, 0.0]


def test_shared_fold_equals_a_numpy_restatement(twin):
    """The host's SRBD constants of random payload rows (the function the commit kernel runs) equal the parallel-axis fold in numpy at 1e-14 per block,
    with the end-effector frame at defaultJointState from the oracle's kinematics; zero masses give the nominal block bit for bit."""
    rng = np.random.default_rng(2)
    rows = np.c_[rng.uniform(0, 3, 40), rng.uniform(-0.3, 0.3, (40, 3)), rng.uniform(0, 5, 40), rng.uniform(-0.3, 0.3, (40, 3))]
    rows[::4, 0] = 0.0; rows[::3, 4] = 0.0
    got = _srbd(rows); nominal = _srbd(None)[0]
    d = twin.rbd(np.r_[np.zeros(6), _djs()], np.zeros(24))
    for row, g in zip(rows, got):
        ref = fold_numpy(nominal, d["R"], d["pos"], row)
        for sl in (slice(0, 1), slice(1, 10), slice(10, 19), slice(19, 22)):
            assert np.max(np.abs(g[sl] - ref[sl])) <= 1e-14 * np.max(np.abs(ref[sl])), (row, sl)
    zero = _srbd(np.c_[np.zeros((3, 1)), rng.uniform(-1, 1, (3, 3)), np.zeros((3, 1)), rng.uniform(-1, 1, (3, 3))])
    assert all(z.tobytes() == nominal.tobytes() for z in zero)
