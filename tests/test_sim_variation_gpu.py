"""Per-robot plant variation on the device (qmb200_sim_set_robot_params, qmb200_sim_step_ext, closed_loop.run's per-robot inputs) against the CPU
twin with variation (tests/sim_twin_ext.cpp), bit-identity of neutral variation, and closed-loop robustness sweeps on an H100."""
import numpy as np
import pytest

import _closed_loop_cpu
from _parity import PLANT_TOL, Q_BLOCKS, RBD_BLOCKS, block_errors
from _sim_twin import DEFAULTS
from _sim_twin_ext import SimTwinExt
from qm_control_b200 import _lib

pytestmark = pytest.mark.gpu

B = 256
PL = {n: i for i, n in enumerate(_lib.PAYLOAD_LAYOUT)}
WR = {n: i for i, n in enumerate(_lib.WRENCH_LAYOUT)}


@pytest.fixture(scope="module")
def solver():
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0)


@pytest.fixture(scope="module")
def twin():
    return SimTwinExt()


def _states(oracle, twin):
    """the state groups of test_sim_gpu.py: 8 groups of 32 (feet above, touching, below, sliding, sticking, landing; random and clipped efforts)"""
    rng = np.random.default_rng(2024); eff_lim = oracle.model_info()["effort"]
    q0, _ = _closed_loop_cpu.standing_state(oracle, twin)
    q = np.tile(q0, (B, 1)); v = np.zeros((B, 24)); eff = np.zeros((B, 18))
    q[:, 6:] += rng.uniform(-0.01, 0.01, (B, 18)); q[:, 3] = rng.uniform(-np.pi, np.pi, B); q[:, 4:6] = rng.uniform(-0.004, 0.004, (B, 2)); q[:, :2] = rng.uniform(-1, 1, (B, 2))
    v[:, 6:] = rng.uniform(-0.1, 0.1, (B, 18)); v[:, 3:6] = rng.uniform(-0.05, 0.05, (B, 3))
    g = np.arange(B) // 32
    q[g == 0, 2] += 0.08
    q[g == 1, 2] += rng.uniform(0.0, 0.001, 32)
    q[g == 2, 2] -= rng.uniform(0.0005, 0.002, 32)
    v[g == 3, 0:2] = rng.uniform(-0.8, 0.8, (32, 2)); q[g == 3, 2] -= 0.001
    v[g == 4, 0:2] = rng.uniform(-1e-3, 1e-3, (32, 2))
    v[g == 5, 2] = -0.3
    eff[g == 6] = rng.uniform(-1, 1, (32, 18)) * eff_lim
    eff[g == 7] = rng.uniform(-2.5, 2.5, (32, 18)) * eff_lim
    eff[(g >= 1) & (g <= 5)] = rng.uniform(-0.2, 0.2, (160, 18)) * eff_lim
    return q, v, eff


def _variation(kind, n=B, seed=5):
    """(mu[n], payload[n, 8], wrench[n, 12]) of one kind of variation; None where that kind leaves the input unset"""
    rng = np.random.default_rng(seed)
    if kind == "mu":
        return rng.uniform(0.1, 1.2, n), None, None
    if kind == "payload":
        p = np.zeros((n, 8)); p[:, PL["m_ee"]] = rng.uniform(0, 3, n); p[:, PL["m_base"]] = rng.uniform(0, 3, n)
        for k in "xyz":
            p[:, PL["o_ee_" + k]] = rng.uniform(-0.1, 0.1, n); p[:, PL["o_base_" + k]] = rng.uniform(-0.1, 0.1, n)
        return None, p, None
    w = np.zeros((n, 12)); w[:, :] = np.c_[rng.uniform(-60, 60, (n, 3)), rng.uniform(-8, 8, (n, 3)), rng.uniform(-30, 30, (n, 3)), rng.uniform(-3, 3, (n, 3))]
    w[rng.random(n) < 0.25] = 0.0
    w[rng.random(n) < 0.25, :6] = 0.0
    w[rng.random(n) < 0.25, 6:] = 0.0
    return None, None, w


def _set(solver, mu, payload):
    solver.sim_set_robot_params(friction_mu=mu, payload=payload)


@pytest.mark.parametrize("kind", ["mu", "payload", "wrench"])
def test_step_ext_matches_the_twin(solver, twin, oracle, kind):
    q, v, eff = _states(oracle, twin); mu, pl, wr = _variation(kind)
    try:
        _set(solver, mu, pl)
        qg, vg, rg, cg, sg = solver.sim_step(1e-3, eff, q, v, wrench=wr)
    finally:
        _set(solver, None, None)
    qt, vt, rt, ct, st = twin.step_batch_ext(1e-3, eff, q, v, mu=mu, payload=pl, wrench=wr)
    assert np.all(sg == 0) and np.all(st == 0)
    np.testing.assert_array_equal(cg, ct)
    for name, a, b, blocks in (("q", qg, qt, Q_BLOCKS), ("v", vg, vt, Q_BLOCKS), ("rbd", rg, rt, RBD_BLOCKS)):
        err = block_errors(a, b, blocks)
        assert max(err.values()) < PLANT_TOL, (kind, name, err)
    qp, vp, _, _, _ = solver.sim_step(1e-3, eff, q, v)   # the variation changes the step
    assert np.max(np.abs(vp - vg)) > 1e-6


def test_neutral_variation_is_bit_identical(solver, twin, oracle):
    import qm_control_b200 as qm
    q, v, eff = _states(oracle, twin)
    plain = solver.sim_step(1e-3, eff, q, v)
    try:
        _set(solver, np.full(B, DEFAULTS["friction_mu"]), np.zeros((B, 8)))
        assert solver.sim_get_robot_params()["payload"] is not None
        neutral = solver.sim_step(1e-3, eff, q, v, wrench=np.zeros((B, 12)))
    finally:
        _set(solver, None, None)
    cleared = solver.sim_step(1e-3, eff, q, v)
    fresh = qm.Solver(batch=B, device=0).sim_step(1e-3, eff, q, v)
    for a, b, c, d in zip(plain, neutral, cleared, fresh):
        np.testing.assert_array_equal(a, b); np.testing.assert_array_equal(c, d); np.testing.assert_array_equal(a, d)


def test_batch_order_with_per_robot_inputs(solver, twin, oracle):
    q, v, eff = _states(oracle, twin); perm = np.random.default_rng(7).permutation(B)
    mu, _, _ = _variation("mu"); _, pl, _ = _variation("payload"); _, _, wr = _variation("wrench")
    try:
        _set(solver, mu, pl); a = solver.sim_step(1e-3, eff, q, v, wrench=wr)
        _set(solver, mu[perm], pl[perm]); b = solver.sim_step(1e-3, eff[perm], q[perm], v[perm], wrench=wr[perm])
    finally:
        _set(solver, None, None)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x[perm], y)


def test_robot_params_validation_and_round_trip(solver):
    from qm_control_b200 import QmbError
    assert solver.sim_get_robot_params() == dict(friction_mu=None, payload=None)
    mu, pl, _ = _variation("mu")[0], _variation("payload")[1], None
    try:
        _set(solver, mu, pl)
        for bad_mu, bad_pl in ((np.r_[0.0, mu[1:]], pl), (np.r_[-1.0, mu[1:]], pl), (np.r_[np.nan, mu[1:]], pl), (mu, np.where(np.arange(8) == PL["m_ee"], -1.0, pl)),
                               (mu, np.where(np.arange(8) == PL["m_base"], -0.5, pl)), (mu, np.where(np.arange(8) == PL["o_ee_y"], np.inf, pl)),
                               (mu, np.where(np.arange(8) == PL["o_base_z"], np.nan, pl)), (np.full(B, np.inf), None)):
            with pytest.raises(QmbError):
                _set(solver, bad_mu, bad_pl)
            got = solver.sim_get_robot_params()
            np.testing.assert_array_equal(got["friction_mu"], mu); np.testing.assert_array_equal(got["payload"], pl)
        _set(solver, None, pl); got = solver.sim_get_robot_params(); assert got["friction_mu"] is None; np.testing.assert_array_equal(got["payload"], pl)
        _set(solver, 0.4, None); got = solver.sim_get_robot_params(); assert got["payload"] is None; np.testing.assert_array_equal(got["friction_mu"], np.full(B, 0.4))
    finally:
        _set(solver, None, None)
    assert solver.sim_get_robot_params() == dict(friction_mu=None, payload=None)


# ---------------- closed loop ----------------
NL = 64
FALL = dict(min_z=0.3, max_roll_pitch=0.3)   # test_sim_gpu.py's trot bounds


@pytest.fixture(scope="module")
def loop_solver():
    import qm_control_b200 as q
    return q.Solver(batch=NL, device=0)


def _run(**kw):
    """closed_loop.run on a fresh handle: the MPC's warm start and the WBC's last input live in the handle, so runs on one handle differ"""
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    s = q.Solver(batch=NL, device=0)
    try:
        return closed_loop.run(s, **kw)
    finally:
        s.close()


def _same_record(a, b, rows=slice(None)):
    for k in ("base", "ee", "status"):
        np.testing.assert_array_equal(a[k][:, rows], b[k][:, rows], err_msg=k)
    for k in ("contact", "q", "v", "start_base", "start_ee"):
        np.testing.assert_array_equal(a[k][rows], b[k][rows], err_msg=k)
    np.testing.assert_array_equal(a["t"], b["t"])


def _upright(r):
    base = r["base"]
    return np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > FALL["min_z"]) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < FALL["max_roll_pitch"]) & \
        np.all((r["status"] & 4) == 0, axis=0)


def test_closed_loop_neutral_inputs_are_bit_identical():
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    plain = _run(duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0))
    s = q.Solver(batch=NL, device=0)
    try:
        neutral = closed_loop.run(s, duration=0.3, gait=["trot"] * NL, cmd_vel=np.tile([0.3, 0.0, 0.0, 0.0], (NL, 1)), friction_mu=0.6, payload=np.zeros((NL, 8)),
                                  pushes=(np.full(NL, 0.1), np.full(NL, 0.1), np.zeros((NL, 12))))
        assert s.sim_get_robot_params() == dict(friction_mu=None, payload=None)   # restored
    finally:
        s.close()
    _same_record(plain, neutral)


def test_closed_loop_mixed_batch_matches_uniform_runs(loop_solver):
    """64 robots with per-robot cmd_vel, stance / trot and payloads: each robot's record equals its record in a uniform run of its configuration."""
    from qm_control_b200 import closed_loop
    configs = [("stance", (0.0, 0.0, 0.0, 0.0), (0.0, 0.0)), ("trot", (0.3, 0.0, 0.0, 0.0), (1.0, 0.0)), ("trot", (0.2, 0.1, 0.0, 0.0), (0.0, 2.0)),
               ("stance", (0.0, 0.0, 0.0, 0.2), (2.0, 1.0))]
    which = np.arange(NL) % len(configs)

    def inputs(rows):
        pl = np.zeros((len(rows), 8)); pl[:, PL["m_ee"]] = [configs[c][2][0] for c in rows]; pl[:, PL["m_base"]] = [configs[c][2][1] for c in rows]
        return [configs[c][0] for c in rows], np.array([configs[c][1] for c in rows]), pl
    gait, cmd, pl = inputs(which)
    mixed = _run(duration=0.3, gait=gait, cmd_vel=cmd, payload=pl)
    for c in range(len(configs)):
        g, cm, p = inputs(np.full(NL, c))
        uni = _run(duration=0.3, gait=g[0], cmd_vel=cm[0], payload=p)
        rows = np.nonzero(which == c)[0]
        for k in ("base", "ee", "status"):
            np.testing.assert_array_equal(mixed[k][:, rows], uni[k][:, rows], err_msg="config %d %s" % (c, k))
        for k in ("contact", "q", "v"):
            np.testing.assert_array_equal(mixed[k][rows], uni[k][rows], err_msg="config %d %s" % (c, k))


def test_closed_loop_restores_robot_params_on_error(loop_solver):
    from qm_control_b200 import closed_loop
    loop_solver.sim_set_robot_params(friction_mu=0.5)
    try:
        with pytest.raises(ValueError):
            closed_loop.run(loop_solver, duration=0.01, cmd_vel=np.zeros(3), payload=np.zeros((NL, 8)))
        got = loop_solver.sim_get_robot_params()
        np.testing.assert_array_equal(got["friction_mu"], np.full(NL, 0.5)); assert got["payload"] is None
    finally:
        loop_solver.sim_set_robot_params()


def _stance_ee_payload_run():
    m = np.linspace(0.0, 2.0, NL); pl = np.zeros((NL, 8)); pl[:, PL["m_ee"]] = m
    return m, _run(duration=1.0, gait="stance", payload=pl)


def test_closed_loop_stance_ee_payload_sweep():
    """Stance, 1 s, EE payload 0-2 kg the controller does not know about: every robot stays up and the end effector droops more with more load
    while the controller catches the load (the first 0.1 s)."""
    m, r = _stance_ee_payload_run()
    dz = r["ee"][:, :, 2] - r["start_ee"][None, :, 2]
    droop = np.max(-dz[:10], axis=0)
    print("stance EE payload: droop in the first 0.1 s at 0 / 1 / 2 kg %.2f / %.2f / %.2f mm, EE z - start at 1 s %.2f / %.2f / %.2f mm; max |dz| base %.4f m; status OR %#x" % (
        droop[0] * 1e3, droop[NL // 2] * 1e3, droop[-1] * 1e3, dz[-1, 0] * 1e3, dz[-1, NL // 2] * 1e3, dz[-1, -1] * 1e3,
        np.max(np.abs(r["base"][:, :, 2] - r["start_base"][None, :, 2])), int(np.bitwise_or.reduce(r["status"].ravel()))))
    assert np.all(_upright(r)) and np.all(r["contact"] == 15) and np.all(r["status"] == 0)
    assert droop[-1] > droop[0] + 0.005


@pytest.mark.xfail(strict=True, reason="measured on H100: with 1-2 kg in the gripper the end effector first droops (16 mm at 2 kg after 0.1 s) and then climbs 29-63 mm "
                   "above its start within 1 s of stance. Neither the MPC model nor the WBC knows the payload, so the arm is driven by a model without it; "
                   "the EE target itself stays at the initial pose (it is re-anchored only beyond 0.1 m). DESIGN.md section 8.")
def test_closed_loop_stance_ee_holds_its_pose_within_2cm_under_2kg():
    _, r = _stance_ee_payload_run()
    assert np.max(np.abs(r["ee"][:, :, 2] - r["start_ee"][None, :, 2])) < 0.02


def test_closed_loop_trot_lateral_push_sweep(loop_solver):
    """Trot at 0.3 m/s, a lateral (+y) base push of 0-300 N for 0.1 s from t = 0.3 s: the pushed base moves in the direction of the push."""
    from qm_control_b200 import closed_loop
    F = np.linspace(0.0, 300.0, NL); w = np.zeros((NL, 12)); w[:, WR["f_base_y"]] = F
    r = _run(duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), pushes=(np.full(NL, 0.3), np.full(NL, 0.1), w))
    up = _upright(r); dy = r["base"][:, :, 1] - r["start_base"][None, :, 1]
    i_push = np.searchsorted(r["t"] - 10.0, 0.45)   # 50 ms after the push ends
    shift = dy[i_push] - dy[i_push, 0]
    print("trot lateral push: largest recovered %.0f N (%d/%d up), y shift at 0.45 s: %s mm" % (np.max(F[up]) if up.any() else -1, int(up.sum()), NL,
                                                                                                 np.array2string(shift[::8] * 1e3, precision=1)))
    assert up[0] and np.all(up[F <= 50.0])
    assert np.all(shift[1:][up[1:]] > 0.0)


def test_closed_loop_trot_friction_sweep(loop_solver):
    """Trot at 0.3 m/s on floors with mu from 0.15 (below the controller's friction cone, 0.3) to 1.0."""
    from qm_control_b200 import closed_loop
    mu = np.linspace(0.15, 1.0, NL)
    r = _run(duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), friction_mu=mu)
    up = _upright(r); dist = np.linalg.norm(r["base"][-1, :, :2] - r["start_base"][:, :2], axis=1)
    print("trot friction sweep: lowest mu up %.3f, all up above %.3f, fallen %d/%d, distance at mu %.2f / %.2f: %.3f / %.3f m" % (
        np.min(mu[up]) if up.any() else -1, np.max(mu[~up]) if (~up).any() else mu[0], int((~up).sum()), NL, mu[0], mu[-1], dist[0], dist[-1]))
    assert np.all(up[mu >= 0.3])
