"""Plant step on the device (qmb200_sim_step, kernels/sim_kernel.cu) against the CPU twin (tests/sim_twin.cpp), and the closed loop of
qm_control_b200.closed_loop on an H100."""
import numpy as np
import pytest

import _closed_loop_cpu
from _parity import PLANT_TOL, Q_BLOCKS, RBD_BLOCKS, block_errors
from _sim_twin import DEFAULTS, SimTwin

pytestmark = pytest.mark.gpu

B = 256


@pytest.fixture(scope="module")
def solver():
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0)


@pytest.fixture(scope="module")
def twin():
    return SimTwin()


def _states(oracle, twin):
    """B synthetic states in 8 groups of 32: feet above, touching and below the ground, sliding (friction saturated) and sticking feet; zero,
    random and out-of-limit efforts."""
    rng = np.random.default_rng(2024); eff_lim = oracle.model_info()["effort"]
    q0, _ = _closed_loop_cpu.standing_state(oracle, twin)
    q = np.tile(q0, (B, 1)); v = np.zeros((B, 24)); eff = np.zeros((B, 18))
    q[:, 6:] += rng.uniform(-0.01, 0.01, (B, 18)); q[:, 3] = rng.uniform(-np.pi, np.pi, B); q[:, 4:6] = rng.uniform(-0.004, 0.004, (B, 2)); q[:, :2] = rng.uniform(-1, 1, (B, 2))
    v[:, 6:] = rng.uniform(-0.1, 0.1, (B, 18)); v[:, 3:6] = rng.uniform(-0.05, 0.05, (B, 3))
    g = np.arange(B) // 32
    q[g == 0, 2] += 0.08                                                        # feet above the ground
    q[g == 1, 2] += rng.uniform(0.0, 0.001, 32)                                 # touching
    q[g == 2, 2] -= rng.uniform(0.0005, 0.002, 32)                               # below
    v[g == 3, 0:2] = rng.uniform(-0.8, 0.8, (32, 2)); q[g == 3, 2] -= 0.001     # sliding: |v_t| well above mu F_n / gamma
    v[g == 4, 0:2] = rng.uniform(-1e-3, 1e-3, (32, 2))                          # sticking: viscous branch
    v[g == 5, 2] = -0.3                                                          # landing
    eff[g == 6] = rng.uniform(-1, 1, (32, 18)) * eff_lim
    eff[g == 7] = rng.uniform(-2.5, 2.5, (32, 18)) * eff_lim                    # beyond the limits: clipped
    eff[(g >= 1) & (g <= 5)] = rng.uniform(-0.2, 0.2, (160, 18)) * eff_lim
    return q, v, eff


def test_params_defaults_and_validation(solver):
    from qm_control_b200 import QmbError
    p = solver.sim_get_params()
    assert p == DEFAULTS
    for bad in (dict(stiffness=0.0), dict(damping=float("nan")), dict(foot_radius=-1.0), dict(substeps_per_ms=0), dict(joint_damping=[-1.0] * 18), dict(ground_height=float("inf"))):
        with pytest.raises(QmbError):
            solver.sim_set_params(**bad)
    assert solver.sim_get_params() == DEFAULTS


def test_sim_step_matches_the_twin(solver, twin, oracle):
    q, v, eff = _states(oracle, twin)
    qg, vg, rg, cg, sg = solver.sim_step(1e-3, eff, q, v)
    qt, vt, rt, ct, st = twin.step_batch(1e-3, eff, q, v)
    assert np.all(sg == 0) and np.all(st == 0)
    np.testing.assert_array_equal(cg, ct)
    g = np.arange(B) // 32
    assert np.all(ct[g == 0] == 0) and np.count_nonzero(ct) >= B // 8 and len(set(ct.tolist())) >= 5, ct   # a foot pushed in deep rebounds within the 1 ms
    for name, a, b, blocks in (("q", qg, qt, Q_BLOCKS), ("v", vg, vt, Q_BLOCKS), ("rbd", rg, rt, RBD_BLOCKS)):
        err = block_errors(a, b, blocks)
        assert max(err.values()) < PLANT_TOL, (name, err)


def test_batch_position_invariance(solver, twin, oracle):
    q, v, eff = _states(oracle, twin); perm = np.random.default_rng(7).permutation(B)
    a = solver.sim_step(1e-3, eff, q, v); b = solver.sim_step(1e-3, eff[perm], q[perm], v[perm])
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x[perm], y)


def test_rbd_round_trip_to_the_centroidal_state(solver, twin, oracle):
    q, v, eff = _states(oracle, twin)
    qg, vg, rg, _, _ = solver.sim_step(1e-3, eff, q, v)
    x = solver.centroidal_state_from_rbd(rg)
    for b in range(0, B, 7):
        xo = oracle.centroidal_state_from_rbd(twin.measure(qg[b], vg[b]))   # the oracle's centroidal state at the device's (q, v)
        np.testing.assert_allclose(x[b], xo, rtol=0, atol=1e-8 * max(1.0, np.max(np.abs(xo))))


@pytest.fixture(scope="module")
def loop_solver():
    import qm_control_b200 as q
    return q.Solver(batch=64, device=0)


def test_closed_loop_stance_stands(loop_solver):
    from qm_control_b200 import closed_loop
    r = closed_loop.run(loop_solver, duration=1.0, gait="stance")
    base, ee, b0 = r["base"], r["ee"], r["start_base"]
    print("stance: max |dz| %.4f m, max |roll|,|pitch| %.4f rad, max xy drift %.4f m, max EE dev %.4f m, status OR %#x, contact %s" % (
        np.max(np.abs(base[:, :, 2] - b0[None, :, 2])), np.max(np.abs(base[:, :, 4:6])), np.max(np.linalg.norm(base[:, :, :2] - b0[None, :, :2], axis=2)),
        np.max(np.linalg.norm(ee[:, :, :3] - r["start_ee"][None, :, :3], axis=2)), int(np.bitwise_or.reduce(r["status"].ravel())), np.unique(r["contact"])))
    assert np.all(r["status"] == 0)
    assert np.max(np.abs(base[:, :, 2] - b0[None, :, 2])) < 0.01
    assert np.max(np.abs(base[:, :, 4:6])) < 0.05
    assert np.max(np.linalg.norm(ee[:, :, :3] - r["start_ee"][None, :, :3], axis=2)) < 0.01
    assert np.all(r["contact"] == 15)


@pytest.mark.xfail(strict=True, reason="measured on H100: the base drifts 3.3 cm backwards in 1 s of stance. cmdVelToTargetTrajectories anchors every target "
                   "at the current base pose, so nothing pulls the base back to where it started; the drift comes from the start transient (the robot rises "
                   "from the standing state's 0.389 m to comHeight 0.4 m with the arm's COM 5 cm ahead of the feet). DESIGN.md section 8.")
def test_closed_loop_stance_base_xy_drift_below_2cm(loop_solver):
    from qm_control_b200 import closed_loop
    r = closed_loop.run(loop_solver, duration=1.0, gait="stance")
    assert np.max(np.linalg.norm(r["base"][:, :, :2] - r["start_base"][None, :, :2], axis=2)) < 0.02


def test_closed_loop_trot_does_not_fall(loop_solver):
    from qm_control_b200 import closed_loop
    r = closed_loop.run(loop_solver, duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0))
    base = r["base"]
    print("trot: min base z %.4f m, max |roll|,|pitch| %.4f rad, mean distance %.4f m, status OR %#x" % (
        np.min(base[:, :, 2]), np.max(np.abs(base[:, :, 4:6])), np.mean(np.linalg.norm(base[-1, :, :2] - r["start_base"][:, :2], axis=1)), int(np.bitwise_or.reduce(r["status"].ravel()))))
    assert np.all(np.isfinite(base)) and np.all((r["status"] & 4) == 0)
    assert np.min(base[:, :, 2]) > 0.3
    assert np.max(np.abs(base[:, :, 4:6])) < 0.3
