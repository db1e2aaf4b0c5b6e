"""Plant step without a GPU: physics pins on the CPU twin (tests/sim_twin.cpp), the qmb200_sim_params layout and defaults, and a closed-loop
rehearsal of qm_control_b200.closed_loop on the oracle's controller restatements."""
import ctypes as C
import os
import xml.etree.ElementTree as ET

import numpy as np
import pytest

import _closed_loop_cpu
from _oracle import ROOT
from _sim_twin import DEFAULTS, SimTwin
from qm_control_b200 import _lib

FIXTURE_URDF = os.path.join(ROOT, "tests", "fixtures", "ref_inputs", "robot.urdf")
G = 9.81


@pytest.fixture(scope="module")
def twin():
    return SimTwin()


def test_params_struct_layout_matches_the_header():
    hdr = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    body = hdr[hdr.index("typedef struct {\n  double ground_height;"):hdr.index("} qmb200_sim_params;")]
    names = [l.split()[1].rstrip(";").split("[")[0] for l in body.splitlines()[1:] if l.strip() and not l.strip().startswith("/*")]
    assert names == [n for n, _ in _lib.SimParams._fields_]
    assert _lib.SimParams.joint_damping.offset == 48 and _lib.SimParams.substeps_per_ms.offset == 48 + 18 * 8
    assert C.sizeof(_lib.SimParams) == 200


def test_defaults_are_what_the_reference_urdf_says():
    root = ET.parse(FIXTURE_URDF).getroot()
    for foot in ("LF_FOOT", "RF_FOOT", "LH_FOOT", "RH_FOOT"):
        link = [l for l in root.findall("link") if l.get("name") == foot][0]
        assert float(link.find("collision/geometry/sphere").get("radius")) == DEFAULTS["foot_radius"]
        gz = [g for g in root.findall("gazebo") if g.get("reference") == foot][0]
        assert float(gz.find("mu1").text) == DEFAULTS["friction_mu"] and float(gz.find("mu2").text) == DEFAULTS["friction_mu"]
    damping = {j.get("name"): float(j.find("dynamics").get("damping")) for j in root.findall("joint") if j.find("dynamics") is not None and j.get("type") != "fixed"}
    legs = [n for n in damping if n[:2] in ("LF", "LH", "RF", "RH")]; arm = [n for n in damping if n not in legs]
    assert len(legs) == 12 and len(arm) == 6
    assert {damping[n] for n in legs} == {DEFAULTS["joint_damping"][0]} and {damping[n] for n in arm} == {DEFAULTS["joint_damping"][12]}


def _momentum(oracle, q, v):
    r = oracle.rbd(q, v); return r["Ag"] @ v, r


def test_free_fall_momentum(oracle):
    """No contact, effort or damping: d(linear momentum)/dt = -m g e_z, angular momentum about the COM conserved, both to O(h)."""
    m = oracle.model_info()["mass"]; rng = np.random.default_rng(5)
    q = oracle.model_info()["q_nominal"] + np.r_[0, 0, 5.0, rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.3, 0.3, 18)]
    v = np.r_[rng.uniform(-0.5, 0.5, 6), rng.uniform(-1, 1, 18)]
    h0, _ = _momentum(oracle, q, v); T = 0.05; errs = []
    for spm in (2, 4):
        tw = SimTwin(ground_height=-100.0, joint_damping=[0.0] * 18, substeps_per_ms=spm)
        q1, v1, _, contact, st = tw.step(T, np.zeros(18), q, v); assert contact == 0 and st == 0
        h1, _ = _momentum(oracle, q1, v1)
        lin = (h1[:3] - h0[:3]) / T - np.array([0, 0, -m * G]); ang = h1[3:] - h0[3:]
        errs.append((np.linalg.norm(lin) / (m * G), np.linalg.norm(ang) / max(1.0, np.linalg.norm(h0[3:]))))
    assert errs[1][0] < 2e-3 and errs[1][1] < 2e-3, errs
    assert errs[1][0] < 0.6 * errs[0][0] and errs[1][1] < 0.6 * errs[0][1], errs   # first order in h


def test_power_balance_over_one_small_step(oracle):
    """Delta(T + V) over one step h equals h qdot^T (S^T tau + J^T F - D qdot) to O(h^2): sliding feet, damping and effort all active."""
    mi = oracle.model_info(); tw = SimTwin(); rng = np.random.default_rng(8)
    q, v = _closed_loop_cpu.standing_state(oracle, tw); q[2] -= 0.002
    v = np.r_[0.3, -0.2, -0.05, rng.uniform(-0.2, 0.2, 3), rng.uniform(-0.5, 0.5, 18)]
    tau = rng.uniform(-5, 5, 18)

    def energy(q, v):
        r = oracle.rbd(q, v); return 0.5 * v @ r["M"] @ v + mi["mass"] * G * r["com"][2]

    _, F, mask = tw.accel(tau, q, v); assert mask == 15
    r = oracle.rbd(q, v); D = np.array(tw.params["joint_damping"])
    power = v[6:] @ (tau - D * v[6:]) + sum(r["foot_vel"][f] @ F[f] for f in range(4))
    errs = []
    for h in (4e-6, 2e-6):
        q1, v1, _, _, st = SimTwin(substeps_per_ms=int(round(1e-3 / h))).step(h, tau, q, v); assert st == 0
        errs.append(abs(energy(q1, v1) - energy(q, v) - h * power))
    assert errs[0] < 1e-3 * h * abs(power) * 1e3 and errs[1] < 0.35 * errs[0], (errs, power)   # O(h^2): halving h quarters the error


def test_standing_state_is_at_rest(oracle, twin):
    """At the standing state the feet carry m g in total, each m g / 4, at rest.  With gravity-compensating joint torques no net force acts on the
    base and the joint rows balance; what remains is the base moment of the COM's horizontal offset from the feet's centre (about 5 cm: the arm),
    which equal foot loads cannot cancel and the controller's contact-force distribution takes up."""
    mi = oracle.model_info(); q, v = _closed_loop_cpu.standing_state(oracle, twin, 0.3, -0.2, 0.7)
    r = oracle.rbd(q, v)
    _, F, mask = twin.accel(np.zeros(18), q, v); assert mask == 15
    np.testing.assert_allclose(F[:, 2], mi["mass"] * G / 4, rtol=1e-9); assert np.sum(F[:, 2]) == pytest.approx(mi["mass"] * G, rel=1e-12)
    np.testing.assert_allclose(F[:, :2], 0.0, atol=0)
    Q = r["Jfoot"].T @ F.reshape(12) - r["nle"]; tau = -Q[6:]
    qdd, _, _ = twin.accel(tau, q, v)
    r1 = oracle.rbd(q, v); Q1 = r1["M"] @ qdd
    assert np.max(np.abs(Q1[:3])) < 1e-9 * mi["mass"] * G                                  # no net force on the base
    np.testing.assert_allclose(Q1[6:], 0.0, atol=1e-9 * mi["mass"] * G)                     # joint rows balanced
    com_off = r["com"][:2] - np.mean(r["foot_pos"][:, :2], axis=0)
    n_base = np.linalg.solve(r["Jbase"][3:, 3:6].T, Q1[3:6])                               # euler-rate rows -> world moment
    np.testing.assert_allclose(n_base[:2], mi["mass"] * G * np.array([-com_off[1], com_off[0]]), rtol=0.05, atol=0.05)   # m g e_z x offset


def test_closed_loop_rehearsal_stance_keeps_the_robot_up(oracle):
    """One robot, stance, 0.2 s: the oracle's controller restatements at the rates of closed_loop.run drive the twin; the robot stays up."""
    r = _closed_loop_cpu.run(oracle, duration=0.2)
    q0, _ = _closed_loop_cpu.standing_state(oracle, SimTwin())
    base = r["rec"][:, :6]
    assert r["status"] == 0 and r["contact"] == 15
    assert np.max(np.abs(base[:, 2] - q0[2])) < 0.01, base[:, 2]
    assert np.max(np.abs(base[:, 4])) < 0.05 and np.max(np.abs(base[:, 5])) < 0.05, base[:, 3:6]
