"""Independent optimality certificate for the oracle's whole-body controller.

The task formulators of qm_wbc/src/WbcBase.cpp:228-546 and the stack of HierarchicalWbc.cpp:18-44 are reference-OWNED code: they are
transliterated here in numpy (rotations through scipy, the Euler-rate acceleration term by finite differences) on top of the rigid-body
quantities that tests/test_oracle_cpu.py pins independently.  HoQp's level problems (HoQp.cpp:53-124) are convex QPs, so a point is optimal
iff it is feasible and its gradient is a combination of the active constraint normals with non-negative inequality multipliers: the test
finds those multipliers by non-negative least squares for each of the three levels of the oracle's solution.  No QP solver is shared with the
oracle (it uses a primal active set), so this pins the cascade result for the literal reference formulation."""
import numpy as np
import pytest
from scipy.optimize import nnls
from scipy.spatial.transform import Rotation

from _oracle import GAINS
from qm_control_b200 import synthetic

NQ, NDEC = 24, 36


def _gains():
    vals = {}
    for line in open(GAINS):
        parts = line.split()
        if len(parts) == 2:
            try:
                vals[parts[0]] = float(parts[1])
            except ValueError:
                pass
    return vals


def _T(e):   # getMappingFromEulerAnglesZyxDerivativeToGlobalAngularVelocity [ocs2]: columns = axes of z, y', x''
    z, y = e[0], e[1]
    return np.array([[0.0, -np.sin(z), np.cos(y) * np.cos(z)], [0.0, np.cos(z), np.cos(y) * np.sin(z)], [1.0, 0.0, -np.sin(y)]])


def _rot(e):
    return Rotation.from_euler("ZYX", e).as_matrix()


def _rot_err(Rl, Rr):   # rotationErrorInWorld(lhs, rhs): rotation vector of lhs * rhs^T
    return Rotation.from_matrix(Rl @ Rr.T).as_rotvec()


def _tasks(oracle, dbg, u_des, mode, time, g, mu=0.3):
    """WbcBase formulators → (A0, b0, D0, f0), (A1, b1), (A2, b2) exactly as HierarchicalWbc::update stacks them; mu: the friction pyramid's coefficient."""
    qm, vm, qd, vd, bacc = dbg["q_meas"], dbg["v_meas"], dbg["q_des"], dbg["v_des"], dbg["base_acc"]
    M = oracle.rbd(qm, vm); D = oracle.rbd(qd, vd); info = oracle.model_info()
    flags = [(mode >> (3 - f)) & 1 for f in range(4)]; nc = sum(flags)
    Mm, h, J, dJ = M["M"], M["nle"], M["Jfoot"], M["dJfoot"]
    # --- task0
    a_eom = np.c_[Mm[:6], -J.T[:6]]; b_eom = -h[:6]                                                        # formulateFloatingBaseEomTask
    lim = np.r_[np.tile(info["effort"][:3], 4), info["effort"][12:]]
    d_tau = np.r_[np.c_[Mm[6:], -J.T[6:]], np.c_[-Mm[6:], J.T[6:]]]; f_tau = np.r_[lim - h[6:], lim + h[6:]]   # formulateTorqueLimitsTask
    a_nc = np.zeros((3 * nc, NDEC)); b_nc = np.zeros(3 * nc); j = 0                                       # formulateNoContactMotionTask
    for i in range(4):
        if flags[i]:
            a_nc[3 * j:3 * j + 3, :NQ] = J[3 * i:3 * i + 3]; b_nc[3 * j:3 * j + 3] = -dJ[3 * i:3 * i + 3] @ vm; j += 1
    a_fr = np.zeros((3 * (4 - nc), NDEC)); j = 0                                                            # formulateFrictionConeTask
    for i in range(4):
        if not flags[i]:
            a_fr[3 * j:3 * j + 3, NQ + 3 * i:NQ + 3 * i + 3] = np.eye(3); j += 1
    pyr = np.array([[0, 0, -1], [1, 0, -mu], [-1, 0, -mu], [0, 1, -mu], [0, -1, -mu]], dtype=float)
    d_fr = np.zeros((5 * nc + 3 * (4 - nc), NDEC)); j = 0
    for i in range(4):
        if flags[i]:
            d_fr[5 * j:5 * j + 5, NQ + 3 * i:NQ + 3 * i + 3] = pyr; j += 1
    A0 = np.r_[a_eom, a_nc, a_fr]; b0 = np.r_[b_eom, b_nc, np.zeros(len(a_fr))]; D0 = np.r_[d_tau, d_fr]; f0 = np.r_[f_tau, np.zeros(len(d_fr))]
    # --- task1 (time >= 10) / taskInit
    if time < 10:                                                                                          # formulateArmJointNomalTrackingTask
        A1 = np.zeros((6, NDEC)); A1[:, NQ - 6:NQ] = np.eye(6)
        kp = np.array([g["kp_arm_joint_%d" % (i + 1)] for i in range(6)]); kd = np.array([g["kd_arm_joint_%d" % (i + 1)] for i in range(6)])
        b1 = kp * (qd[NQ - 6:] - qm[NQ - 6:]) + kd * (vd[NQ - 6:] - vm[NQ - 6:])
    else:
        a_h = np.zeros((1, NDEC)); a_h[0, 2] = 1.0                                                         # formulateBaseHeightMotionTask
        b_h = [bacc[2] + g["baseHeightKp"] * (qd[2] - qm[2]) + g["baseHeightKd"] * (vd[2] - vm[2])]
        e_m = qm[3:6]; Tm = _T(e_m)                                                                        # formulateBaseAngularMotionTask
        a_w = np.zeros((3, NDEC)); a_w[:, :NQ] = M["Jbase"][3:6]
        w_m = Tm @ vm[3:6]; w_d = Tm @ vd[3:6]; err = _rot_err(_rot(qd[3:6]), _rot(e_m))
        hfd = 1e-6; Tdot_ed = (_T(e_m + hfd * vd[3:6]) - _T(e_m - hfd * vd[3:6])) / (2 * hfd) @ vd[3:6]    # d/dt T along the desired Euler rates
        acc_d = Tm @ bacc[3:6] + Tdot_ed                                                                   # getGlobalAngularAccelerationFromEulerAnglesZyxDerivatives
        b_w = acc_d + g["kp_base_angular"] * err + g["kd_base_angular"] * (w_d - w_m) - M["dJbase"][3:6] @ vm
        a_el = np.zeros((3, NDEC)); a_el[:, :NQ] = M["Jee"][:3]                                             # formulateEeLinearMotionTrackingTask
        kpl = np.array([g["kp_ee_linear_%s" % a] for a in "xyz"]); kdl = np.array([g["kd_ee_linear_%s" % a] for a in "xyz"])
        b_el = kpl * (D["ee_pos"] - M["ee_pos"]) + kdl * (D["Jee"][:3] @ vd - M["Jee"][:3] @ vm) - M["dJee"][:3] @ vm
        a_ea = np.zeros((3, NDEC)); a_ea[:, :NQ] = M["Jee"][3:6]; a_ea[:, 3:6] = 0.0                         # formulateEeAngularMotionTrackingTask
        kpa = np.array([g["kp_ee_angular_%s" % a] for a in "xyz"]); kda = np.array([g["kd_ee_angular_%s" % a] for a in "xyz"])
        dj_tmp = M["dJee"][3:6].copy(); dj_tmp[:, 3:6] = 0.0
        b_ea = kpa * _rot_err(D["ee_rot"], M["ee_rot"]) + kda * (-(M["Jee"][3:6] @ vm)) - dj_tmp @ vm
        a_sw = np.zeros((3 * (4 - nc), NDEC)); b_sw = np.zeros(3 * (4 - nc)); j = 0                         # formulateSwingLegTask * 100
        for i in range(4):
            if not flags[i]:
                acc = g["kp_swing"] * (D["foot_pos"][i] - M["foot_pos"][i]) + g["kd_swing"] * (D["foot_vel"][i] - M["foot_vel"][i])
                a_sw[3 * j:3 * j + 3, :NQ] = J[3 * i:3 * i + 3]; b_sw[3 * j:3 * j + 3] = acc - dJ[3 * i:3 * i + 3] @ vm; j += 1
        A1 = np.r_[a_h, a_w, a_el, a_ea, 100.0 * a_sw]; b1 = np.r_[b_h, b_w, b_el, b_ea, 100.0 * b_sw]
    # --- task2
    a_f = np.zeros((12, NDEC)); a_f[:, NQ:] = np.eye(12)                                                    # formulateContactForceTask
    a_bl = np.zeros((2, NDEC)); a_bl[:, :2] = np.eye(2)                                                     # formulateBaseLinearMotionTask
    b_bl = bacc[:2] + g["kp_base_linear"] * (qd[:2] - qm[:2]) + g["kd_base_linear"] * (vd[:2] - vm[:2])
    A2 = np.r_[a_f, a_bl]; b2 = np.r_[u_des[:12], b_bl]
    return (A0, b0, D0, f0), (A1, b1), (A2, b2), M


def _certificate(g, A_eq, D_act):
    """min over (mu free, lam >= 0) of |g + A_eq^T mu + D_act^T lam| (free multipliers split into two non-negative parts → Lawson-Hanson NNLS);
    returns the residual relative to |g|."""
    cols = np.c_[A_eq.T, -A_eq.T, D_act.T] if len(D_act) else np.c_[A_eq.T, -A_eq.T]
    if cols.shape[1] == 0:
        return np.linalg.norm(g) / (1.0 + np.linalg.norm(g))
    scale = np.maximum(np.linalg.norm(cols, axis=0), 1e-300)          # column scaling only rescales the multipliers
    sol, rnorm = nnls(cols / scale, -g, maxiter=20000)
    return rnorm / (1.0 + np.linalg.norm(g))


def assert_levels_are_kkt_points(oracle, g, x_des, u_des, rbd, mode, period, time, il, tag=None, mu=0.3):
    """The three HoQp levels of the oracle's WBC (variant 0) for one robot: level 0 stationary, levels 1 and 2 in the null space of the
    higher-priority tasks, feasible for their inequalities and KKT points with NNLS multipliers; the command follows by updateCmd."""
    dbg = oracle.wbc_debug(x_des, u_des, rbd, int(mode), period, time, input_last=il)
    (A0, b0, D0, f0), (A1, b1), (A2, b2), M = _tasks(oracle, dbg, u_des, int(mode), time, g, mu)
    x0, x1, x2 = dbg["levels"]
    # level 0: smooth problem (slack eliminated): A0'(A0 x - b0) + D0' (D0 x - f0)_+ = 0
    v0 = np.maximum(0.0, D0 @ x0 - f0); g0 = A0.T @ (A0 @ x0 - b0) + D0.T @ v0
    assert np.linalg.norm(g0) / (1.0 + np.linalg.norm(A0.T @ b0)) < 1e-7, (tag, "level 0 stationarity", np.linalg.norm(g0))
    fcap = f0 + v0
    for lvl, (x, xprev, A, bb, Aeq) in enumerate(((x1, x0, A1, b1, A0), (x2, x1, A2, b2, np.r_[A0, A1])), start=1):
        assert np.max(np.abs(Aeq @ (x - xprev))) < 1e-6 * (1.0 + np.max(np.abs(Aeq @ xprev))), (tag, lvl, "left the null space of the higher-priority tasks")
        viol = D0 @ x - fcap; assert viol.max() < 1e-6, (tag, lvl, "violates a higher-priority inequality", viol.max())
        active = viol > -1e-7
        r = _certificate(A.T @ (A @ x - bb), Aeq, D0[active]); assert r < 1e-6, (tag, lvl, "KKT residual", r)
    # updateCmd (WbcBase.cpp:548-563)
    cmd, _, _ = oracle.wbc_update(x_des, u_des, rbd, int(mode), period, time, input_last=il)
    np.testing.assert_allclose(cmd[:36], x2, rtol=0, atol=1e-12)
    np.testing.assert_allclose(cmd[36:], M["M"][6:] @ x2[:NQ] - M["Jfoot"].T[6:] @ x2[NQ:] + M["nle"][6:], rtol=1e-10, atol=1e-9)


@pytest.mark.parametrize("config,time", [(3, 12.0), (4, 12.0), (5, 12.0), (3, 3.0)])
def test_oracle_wbc_levels_satisfy_hoqp_kkt(oracle, config, time):
    g = _gains(); ids = np.arange(6); prob, wbc = synthetic.make_batch(ids, config=config)
    x_des, u_des, mode = synthetic.nominal_wbc_inputs(prob, oracle.model_info()["mass"])
    u_des = u_des + synthetic.uniform(77, ids, 1, 30, -1.0, 1.0) * np.r_[np.full(12, 5.0), np.full(18, 0.2)]
    il = synthetic.uniform(78, ids, 2, 30, -0.1, 0.1)
    for b in range(len(ids)):
        for f in range(4):
            if not (mode[b] >> (3 - f)) & 1:
                u_des[b, 3 * f:3 * f + 3] = 0.0
        assert_levels_are_kkt_points(oracle, g, x_des[b], u_des[b], wbc["rbd"][b], mode[b], wbc["period"][b], time, il[b], tag=b)
