"""HierarchicalMpcWbc (qm_wbc/src/HierarchicalMpcWbc.cpp:18-34) in the oracle: KKT certificates of the literal level problems and an exact re-solve.

task1 = height + base angular + base linear + 100 swing, task2 = contact force; the six arm accelerations carry no task.  The cascade optimum is nevertheless
unique: the floating-base rows couple the arm accelerations to the contact forces through M[base, arm] (condition ~3e3), level 2 spends them - up to the arm
TORQUE LIMITS, which become active (working sets of 7-19 rows, arm accelerations of 1e4 rad/s^2) - on pulling F towards the MPC's forces.  The literal HoQp
iterate (normal-equation Hessian in fullPivLu-kernel coordinates) carries 1e-6..1e-4 of noise on such a problem; the oracle therefore refines every level >= 1 on
the active set its QP identified (HoQp::polish in oracle/src/wbc.cpp) and is pinned here, solver-independently:
  * every level satisfies the KKT conditions of HoQp.cpp:53-124 with NNLS multipliers to 1e-9,
  * the final point equals the equality-constrained least-squares solution on its active set, re-solved with numpy's SVD, to 1e-8,
  * the 12 leg torques QMMpcController consumes (QMController.cpp:427-431) follow from it by updateCmd."""
import numpy as np

import test_wbc_twin_cpu as tw
from qm_control_b200 import synthetic


def _exact(A, b, E, e):
    U, s, Vt = np.linalg.svd(E, full_matrices=True); k = int((s > s.max() * 1e-12).sum())
    xp = Vt[:k].T @ ((U[:, :k].T @ e) / s[:k]); N = Vt[k:].T
    return xp if N.shape[1] == 0 else xp + N @ np.linalg.lstsq(A @ N, b - A @ xp, rcond=1e-13)[0]


def assert_variant_levels(oracle, g, x_des, u_des, rbd, mode, period, il, tag=None):
    """HierarchicalMpcWbc levels of the oracle for one robot at t = 12: KKT points to 1e-9, the final point equal to the exact re-solve on its active set,
    the torques by updateCmd → (torques, final level)."""
    dbg = oracle.wbc_debug(x_des, u_des, rbd, int(mode), period, 12.0, input_last=il, variant=1)
    (A0, b0, D0, f0), (A1, b1), (A2, b2), M = tw._tasks(oracle, dbg, u_des, int(mode), 12.0, g)
    A1v = np.r_[A1[:4], A2[12:14], A1[10:]]; b1v = np.r_[b1[:4], b2[12:14], b1[10:]]; A2v = A2[:12]; b2v = b2[:12]      # HierarchicalMpcWbc.cpp:23-28 (A1[10:]: the swing rows)
    x0, x1, x2 = dbg["levels"]; v0 = np.maximum(0.0, D0 @ x0 - f0); fcap = f0 + v0
    for lvl, (x, xprev, A, bb, Aeq) in enumerate(((x1, x0, A1v, b1v, A0), (x2, x1, A2v, b2v, np.r_[A0, A1v])), start=1):
        assert np.max(np.abs(Aeq @ (x - xprev))) < 1e-8 * (1.0 + np.max(np.abs(Aeq @ xprev))), (tag, lvl)
        viol = D0 @ x - fcap; assert viol.max() < 1e-8, (tag, lvl, viol.max())
        act = viol > -1e-7 * (1.0 + np.abs(fcap)); r = tw._certificate(A.T @ (A @ x - bb), Aeq, D0[act]); assert r < 1e-9, (tag, lvl, r)
    xs = _exact(A2v, b2v, np.r_[A0, A1v, D0[act]], np.r_[A0 @ x0, A1v @ x1, fcap[act]])
    assert np.max(np.abs(xs - x2) / np.maximum(1.0, np.abs(xs))) < 1e-8, (tag, np.max(np.abs(xs - x2) / np.maximum(1.0, np.abs(xs))))
    tau = M["M"][6:] @ x2[:24] - M["Jfoot"].T[6:] @ x2[24:] + M["nle"][6:]
    cmd = oracle.wbc_update_batch(x_des[None], u_des[None], rbd[None], [int(mode)], [period], [12.0], il[None], variant=1)[0][0]   # (the batch entry does not raise when the literal QP stalls in the free arm directions)
    np.testing.assert_allclose(cmd[36:], tau, rtol=1e-10, atol=1e-9)
    return tau, x2


def test_mpc_variant_levels_are_kkt_points_and_match_an_exact_resolve(oracle):
    g = tw._gains(); ids = np.arange(12); prob, wbc = synthetic.make_batch(ids, config=3)
    x_des, u_des, mode = synthetic.nominal_wbc_inputs(prob, oracle.model_info()["mass"])
    u_des = u_des + synthetic.uniform(77, ids, 1, 30, -1.0, 1.0) * np.r_[np.full(12, 5.0), np.full(18, 0.2)]
    il = u_des + synthetic.uniform(78, ids, 2, 30, -0.002, 0.002); saturated = 0
    for b in range(len(ids)):
        tau, x2 = assert_variant_levels(oracle, g, x_des[b], u_des[b], wbc["rbd"][b], mode[b], wbc["period"][b], il[b], tag=b)
        lim = oracle.model_info()["effort"][12:]; saturated += int(np.sum(np.abs(np.abs(tau[12:]) - lim) < 1e-6))
        assert np.max(np.abs(x2[18:24])) > 1e3                                                             # the untasked arm accelerations really are that large
    assert saturated >= len(ids)                                                                          # arm torque limits active: at least one per robot on average
