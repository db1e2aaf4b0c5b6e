"""Independent certificates for the oracle's MPC tick.

(1) The SQP step (dx, du) the oracle gets from constraint projection + Riccati recursion must be THE solution of the equality-constrained QP that
    setupQuadraticSubproblem defines (HPIPM solves that QP exactly in the reference): feasibility of the linearised dynamics and equality rows, and
    stationarity with multipliers recovered by plain least squares in a backward pass - no projection, no Riccati, nothing shared with the oracle's solver.
(2) The derivative blocks of that QP against central finite differences of the oracle's own value functions: cost gradient (tracking + end-effector +
    barriers + friction cone), equality-constraint Jacobians C, D.  (The dynamics Jacobians are covered in tests/test_oracle_cpu.py.)"""
import numpy as np
import pytest

from qm_control_b200 import synthetic

NMAX = 88


def assert_kkt_point(qp):
    """Feasibility and stationarity of the oracle's SQP step on the QP `qp` (oracle.mpc_qp) → the set of equality-row counts met."""
    N = qp["n_nodes"] - 1; dx, du = qp["dx"], qp["du"]
    assert np.allclose(dx[0], 0.0)                                                      # cold start: the first node already sits on the measured state
    worst_feas = 0.0; ngs = set()
    for k in range(N):
        worst_feas = max(worst_feas, np.max(np.abs(qp["A"][k] @ dx[k] + qp["B"][k] @ du[k] + qp["b"][k] - dx[k + 1])))
        if not qp["is_event"][k]:
            ng = qp["ng"][k]; ngs.add(int(ng))
            worst_feas = max(worst_feas, np.max(np.abs(qp["C"][k, :ng] @ dx[k] + qp["D"][k, :ng] @ du[k] + qp["e"][k, :ng])))
        else:
            assert np.all(du[k] == 0.0)
    assert worst_feas < 1e-9 * (1.0 + np.max(np.abs(dx)) + np.max(np.abs(du))), worst_feas
    lam = qp["QN"] @ dx[N] + qp["qN"]; worst = 0.0
    for k in range(N - 1, -1, -1):
        if qp["is_event"][k]:
            continue                                                                    # jump map x+ = x: lam_k = lam_{k+1}, no input, no cost
        ng = qp["ng"][k]; Ck, Dk = qp["C"][k, :ng], qp["D"][k, :ng]
        gu = qp["R"][k] @ du[k] + qp["P"][k] @ dx[k] + qp["r"][k] + qp["B"][k].T @ lam
        nu = np.linalg.lstsq(Dk.T, -gu, rcond=None)[0]                                  # D has full row rank: the multipliers are unique
        worst = max(worst, np.linalg.norm(gu + Dk.T @ nu) / (1.0 + np.linalg.norm(gu)))
        lam = qp["Q"][k] @ dx[k] + qp["P"][k].T @ du[k] + qp["q"][k] + qp["A"][k].T @ lam + Ck.T @ nu
    assert worst < 1e-8, worst
    return ngs


@pytest.mark.parametrize("robot", [0, 1, 2, 5])          # stance, trot, flying trot, flying trot at another phase
def test_sqp_step_is_the_kkt_point_of_the_qp(oracle, robot):
    oracle.mpc_set(dt=0.015, horizon=1.0); prob, _ = synthetic.make_batch(np.array([robot]), config=5)
    qp = oracle.mpc_qp(prob, NMAX); assert qp["n_nodes"] - 1 >= 67
    assert assert_kkt_point(qp) <= {12, 14, 16}


def test_cost_gradient_and_constraint_jacobians_by_finite_differences(oracle):
    oracle.mpc_set(dt=0.015, horizon=1.0); prob, _ = synthetic.make_batch(np.array([2]), config=5)      # flying trot: swing and stance legs, normal-velocity rows
    qp = oracle.mpc_qp(prob, NMAX); sol = oracle.mpc_solve_batch(prob, NMAX, nthreads=1); n = int(sol["n_nodes"][0]); ev = sol["event"][0, :n]
    checked = 0
    for k in range(2, n - 2, 9):
        if ev[k] != 0 or ev[k + 1] != 0 or qp["is_event"][k]:
            continue
        assert_node_derivatives(oracle, prob, qp, sol, k)
        checked += 1
    assert checked >= 5


def assert_node_derivatives(oracle, prob, qp, sol, k):
    """Cost gradient and the equality-constraint Jacobians C, D of node k (no event at k or k + 1) against central differences of the oracle's stage
    functions, at the node's cold-start guess → the node's mode."""
    n = int(sol["n_nodes"][0]); t = sol["t"][0, :n]
    ne = int(prob["n_events"][0]); et = prob["event_times"][0, :ne]; md = prob["modes"][0, :ne + 1]; tt = prob["target_times"][0, :2]; ts = prob["target_states"][0, :2]
    mass = oracle.model_info()["mass"]; x = prob["x0"][0].copy()
    dt = t[k + 1] - t[k]; mode = md[int(np.searchsorted(et, t[k], side="left"))]; flags = [(mode >> (3 - f)) & 1 for f in range(4)]; nc = sum(flags)
    u = np.zeros(30)                                                                                   # the cold-start guess of node k (QMInitializer): state held, weight compensation
    for f in range(4):
        if flags[f]:
            u[3 * f + 2] = mass * 9.81 / nc
    f0, q, r, g0 = oracle.stage_probe(et, md, tt, ts, t[k], x, u)
    np.testing.assert_allclose(dt * q, qp["q"][k], rtol=1e-10, atol=1e-10); np.testing.assert_allclose(dt * r, qp["r"][k], rtol=1e-10, atol=1e-10)   # the probe sees the node the QP was built at
    np.testing.assert_allclose(g0, qp["e"][k, :len(g0)], rtol=0, atol=1e-12); ng = len(g0)
    h = 1e-6; fd_q = np.zeros(30); fd_r = np.zeros(30); fd_C = np.zeros((ng, 30)); fd_D = np.zeros((ng, 30))
    for i in range(30):
        d = np.zeros(30); d[i] = h
        fp, _, _, gp = oracle.stage_probe(et, md, tt, ts, t[k], x + d, u, want_grad=False); fm, _, _, gm = oracle.stage_probe(et, md, tt, ts, t[k], x - d, u, want_grad=False)
        fd_q[i] = (fp - fm) / (2 * h); fd_C[:, i] = (gp - gm) / (2 * h)
        fp, _, _, gp = oracle.stage_probe(et, md, tt, ts, t[k], x, u + d, want_grad=False); fm, _, _, gm = oracle.stage_probe(et, md, tt, ts, t[k], x, u - d, want_grad=False)
        fd_r[i] = (fp - fm) / (2 * h); fd_D[:, i] = (gp - gm) / (2 * h)
    scale = max(1.0, np.max(np.abs(q)), np.max(np.abs(r)))
    assert np.max(np.abs(fd_q - q)) < 2e-6 * scale and np.max(np.abs(fd_r - r)) < 2e-6 * scale, (k, np.max(np.abs(fd_q - q)), np.max(np.abs(fd_r - r)))
    assert np.max(np.abs(fd_C - qp["C"][k, :ng])) < 1e-6 * (1.0 + np.max(np.abs(qp["C"][k]))) and np.max(np.abs(fd_D - qp["D"][k, :ng])) < 1e-6 * (1.0 + np.max(np.abs(qp["D"][k])))
    return mode


def test_discrete_dynamics_sensitivities_by_finite_differences(oracle):
    """A_d, B_d and the defect b of the multiple-shooting nodes against central differences of a numpy RK2 (Heun, DESIGN.md section 2) step built from the
    oracle's continuous flow map only - pins the sensitivity integrator independently of the dual-number propagation the oracle uses."""
    oracle.mpc_set(dt=0.015, horizon=1.0); prob, _ = synthetic.make_batch(np.array([1]), config=5)      # trot
    qp = oracle.mpc_qp(prob, NMAX); sol = oracle.mpc_solve_batch(prob, NMAX, nthreads=1); n = int(sol["n_nodes"][0]); t = sol["t"][0, :n]; ev = sol["event"][0, :n]
    ne = int(prob["n_events"][0]); et = prob["event_times"][0, :ne]; md = prob["modes"][0, :ne + 1]; mass = oracle.model_info()["mass"]; x = prob["x0"][0].copy()

    def step(xx, uu, dt):
        k1 = oracle.flow_map(xx, uu)[0]; k2 = oracle.flow_map(xx + dt * k1, uu)[0]; return xx + 0.5 * dt * (k1 + k2)

    checked = 0
    for k in range(3, n - 2, 13):
        if ev[k] != 0 or ev[k + 1] != 0 or qp["is_event"][k]:
            continue
        dt = t[k + 1] - t[k]; mode = md[int(np.searchsorted(et, t[k], side="left"))]; flags = [(mode >> (3 - f)) & 1 for f in range(4)]; u = np.zeros(30)
        for f in range(4):
            if flags[f]:
                u[3 * f + 2] = mass * 9.81 / sum(flags)
        np.testing.assert_allclose(step(x, u, dt) - x, qp["b"][k], rtol=0, atol=1e-12)                      # defect against the held state of the cold start
        h = 1e-6; A = np.zeros((30, 30)); B = np.zeros((30, 30))
        for i in range(30):
            d = np.zeros(30); d[i] = h
            A[:, i] = (step(x + d, u, dt) - step(x - d, u, dt)) / (2 * h); B[:, i] = (step(x, u + d, dt) - step(x, u - d, dt)) / (2 * h)
        assert np.max(np.abs(A - qp["A"][k])) < 1e-7 and np.max(np.abs(B - qp["B"][k])) < 1e-7, (k, np.max(np.abs(A - qp["A"][k])), np.max(np.abs(B - qp["B"][k])))
        checked += 1
    assert checked >= 4
