"""Per-robot plant variation without a GPU: payload and external-wrench physics on the CPU twin with variation (tests/sim_twin_ext.cpp), the
payload / wrench layouts of include/qmb200.h against the binding, and a closed-loop rehearsal with a payload the controller does not know about."""
import os
import re

import numpy as np

import _closed_loop_cpu
from _oracle import ROOT
from _sim_twin import SimTwin
from _sim_twin_ext import SimTwinExt
from qm_control_b200 import _lib

G = 9.81
PL = {n: i for i, n in enumerate(_lib.PAYLOAD_LAYOUT)}
WR = {n: i for i, n in enumerate(_lib.WRENCH_LAYOUT)}


def _payload(m_ee=0.0, o_ee=(0, 0, 0), m_base=0.0, o_base=(0, 0, 0)):
    p = np.zeros(8); p[PL["m_ee"]] = m_ee; p[PL["m_base"]] = m_base
    for k, x in zip("xyz", o_ee):
        p[PL["o_ee_" + k]] = x
    for k, x in zip("xyz", o_base):
        p[PL["o_base_" + k]] = x
    return p


def _wrench(f_base=(0, 0, 0), n_base=(0, 0, 0), f_ee=(0, 0, 0), n_ee=(0, 0, 0)):
    w = np.zeros(12)
    for name, vec in (("f_base", f_base), ("n_base", n_base), ("f_ee", f_ee), ("n_ee", n_ee)):
        for k, x in zip("xyz", vec):
            w[WR[name + "_" + k]] = x
    return w


def _rot_zyx(z, y, x):
    cz, sz, cy, sy, cx, sx = np.cos(z), np.sin(z), np.cos(y), np.sin(y), np.cos(x), np.sin(x)
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]); Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]); Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    return Rz @ Ry @ Rx


def _point(oracle, q, frame, o):
    """world position of the point o (frame coordinates) fixed to the end-effector frame or to the base, from the oracle's forward kinematics"""
    if frame == "ee":
        r = oracle.rbd(q, np.zeros(24)); return r["ee_pos"] + r["ee_rot"] @ o
    return q[:3] + _rot_zyx(*q[3:6]) @ o


def _random_q(oracle, rng, z=0.45):
    q = oracle.model_info()["q_nominal"] + np.r_[rng.uniform(-0.5, 0.5, 2), z, rng.uniform(-0.4, 0.4, 3), rng.uniform(-0.3, 0.3, 18)]
    return q


def test_header_layouts_match_the_binding():
    hdr = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for sym in ("qmb200_sim_set_robot_params", "qmb200_sim_get_robot_params", "qmb200_sim_step_ext", "qmb200_sim_step_ext_dev"):
        assert re.search(r"\bint %s\(" % sym, hdr), sym
        assert sym in _lib.SYMBOLS, sym
    for name, layout in (("payload[B][8]", _lib.PAYLOAD_LAYOUT), ("wrench[B][12]", _lib.WRENCH_LAYOUT)):
        m = re.search(re.escape(name) + r"\s+layout: \[([^\]]*)\]", hdr); assert m, name
        assert tuple(s.strip() for s in m.group(1).split(",")) == layout, (name, m.group(1))
    # the kernel's own layout comment says the same
    src = open(os.path.join(ROOT, "qm_control_b200", "csrc", "kernels", "sim_kernel.cu")).read()
    assert "payload[B][8]    [m_ee, o_ee(3), m_base, o_base(3)]" in src and "wrench[B][12]    [f_base, n_base, f_ee, n_ee]" in src


def test_payload_gravity_is_the_point_jacobian_transpose(oracle):
    """At v = 0: nle(payload) - nle(none) = J_p^T (m_p g e_z), J_p a central difference of the payload point's world position."""
    tw = SimTwinExt(); rng = np.random.default_rng(11); eps = 1e-6
    for trial in range(4):
        q = _random_q(oracle, rng); v = np.zeros(24)
        base = tw.rbd_ext(q, v)["nle"]
        for frame in ("ee", "base"):
            m = rng.uniform(0.5, 3.0); o = rng.uniform(-0.1, 0.1, 3)
            p = _payload(m_ee=m, o_ee=o) if frame == "ee" else _payload(m_base=m, o_base=o)
            dn = tw.rbd_ext(q, v, p)["nle"] - base
            J = np.zeros((3, 24))
            for c in range(24):
                dq = np.zeros(24); dq[c] = eps
                J[:, c] = (_point(oracle, q + dq, frame, o) - _point(oracle, q - dq, frame, o)) / (2 * eps)
            np.testing.assert_allclose(dn, J.T @ np.array([0, 0, m * G]), rtol=0, atol=1e-6 * m * G, err_msg="%s payload, trial %d" % (frame, trial))


def test_momentum_balance_in_flight_with_payloads_and_wrenches(oracle):
    """Feet clear of the ground, zero effort and damping, both payloads and both wrenches set: from the twin's qdd, the linear momentum rate is
    (m + m_ee + m_base)(-g e_z) + f_base + f_ee and the angular momentum rate about the COM is sum (p_i - c) x f_i + n_i."""
    tw = SimTwinExt(ground_height=-100.0, joint_damping=[0.0] * 18); rng = np.random.default_rng(12); m0 = oracle.model_info()["mass"]
    for trial in range(3):
        q = _random_q(oracle, rng, z=3.0); v = np.r_[rng.uniform(-0.5, 0.5, 6), rng.uniform(-1, 1, 18)]
        pl = _payload(rng.uniform(0.5, 3), rng.uniform(-0.1, 0.1, 3), rng.uniform(0.5, 3), rng.uniform(-0.1, 0.1, 3))
        fb, nb, fe, ne = (rng.uniform(-40, 40, 3) for _ in range(4))
        qdd, F, mask = tw.accel_ext(np.zeros(18), q, v, payload=pl, wrench=_wrench(fb, nb, fe, ne)); assert mask == 0 and np.all(F == 0)
        r = tw.rbd_ext(q, v, pl)
        assert abs(r["mass"] - (m0 + pl[PL["m_ee"]] + pl[PL["m_base"]])) < 1e-12 * m0
        hdot = r["Ag"] @ qdd + r["dAg_v"]
        lin = r["mass"] * np.array([0, 0, -G]) + fb + fe
        p_ee = oracle.rbd(q, v)["ee_pos"]; c = r["com"]
        ang = np.cross(q[:3] - c, fb) + nb + np.cross(p_ee - c, fe) + ne
        np.testing.assert_allclose(hdot[:3], lin, rtol=0, atol=1e-9 * r["mass"] * G)
        np.testing.assert_allclose(hdot[3:], ang, rtol=0, atol=1e-9 * r["mass"] * G)


def test_neutral_variation_is_the_plain_twin(oracle):
    """The shared mu, zero payloads and a zero wrench reproduce the plain twin step (tests/sim_twin.cpp) bit for bit."""
    tw = SimTwinExt(); q, v = _closed_loop_cpu.standing_state(oracle, tw); q[2] -= 0.001
    v = np.r_[0.3, -0.2, -0.05, np.zeros(21)]; eff = np.random.default_rng(3).uniform(-5, 5, 18)
    a = tw.step(1e-3, eff, q, v); b = tw.step_ext(1e-3, eff, q, v, mu=tw.params["friction_mu"], payload=np.zeros(8), wrench=np.zeros(12))
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_closed_loop_rehearsal_stance_with_an_ee_payload(oracle, monkeypatch):
    """One robot, stance, 0.2 s, a 1 kg payload in the gripper that the controller does not know about: the rehearsal of test_sim_cpu.py with its
    plant twin carrying the payload stays up with no status bit."""
    payload = _payload(m_ee=1.0)

    class PayloadTwin(SimTwinExt):
        def step(self, duration, effort, q, v):
            return self.step_ext(duration, effort, q, v, payload=payload)
    monkeypatch.setattr(_closed_loop_cpu, "SimTwin", PayloadTwin)
    r = _closed_loop_cpu.run(oracle, duration=0.2)
    q0, _ = _closed_loop_cpu.standing_state(oracle, SimTwin())
    base = r["rec"][:, :6]
    assert r["status"] == 0 and r["contact"] == 15
    assert np.max(np.abs(base[:, 2] - q0[2])) < 0.01, base[:, 2]
    assert np.max(np.abs(base[:, 4])) < 0.05 and np.max(np.abs(base[:, 5])) < 0.05, base[:, 3:6]
