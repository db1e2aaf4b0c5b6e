"""The online payload estimator on the device (qmb200_payload_est_*, closed_loop.run(payload_estimator=...)), 64 robots.

The step kernel is replayed call by call on the CPU twin (tests/_payload_est_twin.py) from a recorded closed loop; the commit is checked against the host's
SRBD constants and against a fresh handle told the committed rows; then closed loops with an unknown end-effector payload in stance and trot."""
import numpy as np
import pytest

from _parity import MPC_TOL, TICK_TOL, assert_cmd, assert_traj
from qm_control_b200 import _lib

pytestmark = pytest.mark.gpu

NL = 64
PL = {n: i for i, n in enumerate(_lib.PAYLOAD_LAYOUT)}


def _solver(batch=NL):
    import qm_control_b200 as q
    return q.Solver(batch=batch, device=0)


def _ee_payload(m):
    pl = np.zeros((len(m), 8)); pl[:, PL["m_ee"]] = m
    return pl


def _upright(r):
    base = r["base"]
    return np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3)


def test_params_defaults_and_validation():
    s = _solver(batch=2)
    try:
        from _payload_est_twin import DEFAULTS
        assert s.payload_est_get_params() == DEFAULTS
        for bad in (dict(forgetting=0.0), dict(forgetting=1.5), dict(p0_mass=0.0), dict(p0_inertia=-1.0), dict(trace_max=np.nan), dict(mass_min=2.0, mass_max=1.0),
                    dict(offset_max=np.inf)):
            with pytest.raises(_lib.QmbError):
                s.payload_est_set_params(**bad)
            assert s.payload_est_get_params() == DEFAULTS
        s.payload_est_set_params(forgetting=1.0); assert s.payload_est_get_params()["forgetting"] == 1.0
        for call in (lambda: s.payload_est_commit_dev(), lambda: s.payload_est_get(), lambda: s.payload_est_step(1e-3, np.zeros((2, 18)), np.zeros((2, 55)))):
            with pytest.raises(_lib.QmbError, match="not running"):
                call()
    finally:
        s.close()


def test_step_kernel_equals_the_twin_on_closed_loop_data():
    """0.3 s trot, 0-2 kg EE payloads in the plant, the estimator from a zero prior: every call's theta and diag P per robot at 1e-10 relative, status
    bits identical."""
    import torch
    from qm_control_b200 import closed_loop
    from _payload_est_twin import PayloadEstTwin
    s = _solver(); rec = []
    orig = s.payload_est_step_dev

    def wrapped(dt, effort, rbd, status, stream=None):
        e, r = effort.clone(), rbd.clone()
        orig(dt, effort, rbd, status, stream)
        torch.cuda.current_stream().synchronize(); torch.cuda.synchronize()
        rec.append((dt, e.cpu().numpy(), r.cpu().numpy(), status.cpu().numpy(), s.payload_est_get()))
    s.payload_est_step_dev = wrapped
    try:
        m = np.linspace(0.0, 2.0, NL)
        closed_loop.run(s, duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), payload=_ee_payload(m), model_payload=np.zeros((NL, 8)), payload_estimator=True)
    finally:
        del s.payload_est_step_dev
        s.close()
    assert len(rec) == 300
    twin = PayloadEstTwin(); states = [twin.reset(np.zeros(8)) for _ in range(NL)]
    worst = np.zeros(2)
    for k, (dt, effort, rbd, status, got) in enumerate(rec):
        for b in range(NL):
            code = twin.step(states[b], dt, effort[b], rbd[b])
            assert code == status[b], (k, b, code, status[b])
            th, pd = states[b]["theta"], np.diag(states[b]["P"])
            et = np.max(np.abs(got["theta"][b] - th)) / max(np.max(np.abs(th)), 1e-2); ep = np.max(np.abs(got["p_diag"][b] - pd)) / np.max(np.abs(pd))
            worst = np.maximum(worst, [et, ep])
            assert et < 1e-10 and ep < 1e-10, (k, b, et, ep)
        assert np.all(got["samples"] == k + 1)
    print("payload estimator vs twin over 300 calls x %d robots: theta %.1e, diag P %.1e (worst relative)" % (NL, worst[0], worst[1]))


def test_commit_writes_the_host_fold_and_keeps_the_base_half():
    """After steps on standing data: the committed rows are the twin's commit of theta, base halves bit for bit, and the SRBD constants the kernels read
    (through qmb200_centroidal_state_from_rbd, which reads them back) equal a handle told the committed rows; a zero estimate is the nominal model bit for bit."""
    from _payload_est_twin import PayloadEstTwin
    rng = np.random.default_rng(4)
    prior = np.c_[rng.uniform(0, 2, NL), rng.uniform(-0.05, 0.05, (NL, 3)), rng.uniform(0, 4, NL), rng.uniform(-0.2, 0.2, (NL, 3))]
    prior[::4, 0] = 0.0; prior[::4, 1:4] = 0.0
    s = _solver(); ref = _solver(); nom = _solver()
    try:
        s.payload_est_reset(prior)
        xy = np.c_[rng.uniform(-1, 1, (NL, 2)), rng.uniform(-3, 3, NL)]; qs, vs = s.sim_standing_state(xy)
        effort = np.zeros((NL, 18))
        qq, vv, rbd, _, _ = s.sim_step(1e-3, effort, qs, vs)
        assert np.all(s.payload_est_step(1e-3, effort, rbd) == 0)
        still = np.arange(NL) % 4 == 0
        eff = np.where(still[:, None], 0.0, rng.uniform(-20, 20, (NL, 18)))
        for _ in range(5):
            qq, vv, rbd2, _, _ = s.sim_step(1e-3, eff, qq, vv)
            s.payload_est_step(1e-3, eff, rbd2)
        got = s.payload_est_get()
        s.payload_est_commit_dev(); rows = s.get_model_payload()
        twin = PayloadEstTwin()
        want = np.array([twin.commit(got["theta"][b], prior[b]) for b in range(NL)])
        np.testing.assert_array_equal(rows[:, 4:], prior[:, 4:])
        np.testing.assert_allclose(rows, want, rtol=1e-15, atol=1e-15)
        ref.set_model_payload(rows)
        x_est, x_ref = s.centroidal_state_from_rbd(rbd2), ref.centroidal_state_from_rbd(rbd2)
        assert np.max(np.abs(x_est - x_ref)) <= 1e-14 * max(1.0, np.max(np.abs(x_ref)))
        zero = (rows[:, 0] == 0.0) & (rows[:, 4] == 0.0)
        if np.any(zero):
            x_nom = nom.centroidal_state_from_rbd(rbd2)
            assert x_est[zero].tobytes() == x_nom[zero].tobytes()
        s.payload_est_stop(); np.testing.assert_array_equal(s.get_model_payload(), rows)   # the last committed rows stay
        with pytest.raises(_lib.QmbError, match="not running"):
            s.payload_est_get()
    finally:
        for h in (s, ref, nom):
            h.close()


def test_mpc_and_wbc_after_a_commit_equal_a_handle_told_the_rows():
    from qm_control_b200 import synthetic
    rng = np.random.default_rng(9)
    prob, wbc = synthetic.make_batch(np.arange(NL), config=5)
    s = _solver(); ref = _solver()
    try:
        prior = _ee_payload(rng.uniform(0.2, 2.0, NL)); prior[:, 1:4] = rng.uniform(-0.05, 0.05, (NL, 3))
        s.payload_est_reset(prior); s.payload_est_commit_dev(); rows = s.get_model_payload()
        ref.set_model_payload(rows)
        for h in (s, ref):
            h.mpc_reset(); h.wbc_set_input_last(None)
        assert_traj(s.mpc_solve(prob), ref.mpc_solve(prob), MPC_TOL, tag="mpc after commit")
        x_des = prob["x0"]; u_des = np.zeros((NL, 30)); u_des[:, 2:12:3] = 80.0; mode = np.full(NL, 15, dtype=np.int32)
        c1, s1 = s.wbc_update(x_des, u_des, wbc["rbd"], mode, wbc["period"], wbc["time"])
        c2, s2 = ref.wbc_update(x_des, u_des, wbc["rbd"], mode, wbc["period"], wbc["time"])
        assert_cmd(c1, c2, TICK_TOL, tag="wbc after commit"); np.testing.assert_array_equal(s1, s2)
    finally:
        s.close(); ref.close()


def _loop(**kw):
    from qm_control_b200 import closed_loop
    s = _solver()
    try:
        prev = s.payload_est_get_params()
        r = closed_loop.run(s, **kw)
        assert s.get_model_payload() is None and s.payload_est_get_params() == prev   # restored
        return r
    finally:
        s.close()


_STANCE = {}


def _stance():
    if not _STANCE:
        m = np.linspace(0.0, 2.0, NL)
        _STANCE.update(m=m, est=_loop(duration=1.0, gait="stance", payload=_ee_payload(m), payload_estimator=True),
                       unknown=_loop(duration=1.0, gait="stance", payload=_ee_payload(m)))
    return _STANCE["m"], _STANCE["est"], _STANCE["unknown"]


def test_closed_loop_stance_estimates_the_payload():
    m, est, unknown = _stance()
    m_hat = est["payload_est"][-1, :, 0]; err = np.abs(m_hat - m)
    dz = lambda r, t0=0: np.max(np.abs(r["ee"][t0:, :, 2] - r["start_ee"][None, :, 2]), axis=0)
    print("stance, estimator: |m_hat - m| p50 %.4f max %.4f kg; EE max |dz| over the last 0.5 s %.1f mm; max |dz| at 2 kg: estimate %.1f mm, not told %.1f mm" % (
        np.median(err), err.max(), dz(est, 50).max() * 1e3, dz(est)[-1] * 1e3, dz(unknown)[-1] * 1e3))
    assert np.all(_upright(est)) and np.all(est["contact"] == 15) and np.all(est["status"] == 0)
    assert np.all(err <= np.maximum(0.05, 0.05 * m))
    assert dz(est, 50).max() < 0.02
    heavy = m >= 1.0
    assert np.all(dz(est)[heavy] < dz(unknown)[heavy])


def test_closed_loop_trot_estimates_the_payload():
    m = np.linspace(0.0, 2.0, NL)
    r = _loop(duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), payload=_ee_payload(m), payload_estimator=True)
    err = np.abs(r["payload_est"][-1, :, 0] - m)
    print("trot, estimator: %d/%d up, |m_hat - m| p50 %.4f max %.4f kg" % (int(_upright(r).sum()), NL, np.median(err), err.max()))
    assert np.all(_upright(r))
    assert np.all(err <= np.maximum(0.1, 0.15 * m))


def test_closed_loop_without_a_payload_estimates_none():
    r = _loop(duration=1.0, gait="stance", payload_estimator=True)
    print("stance, no payload: max m_hat %.4f kg" % r["payload_est"][:, :, 0].max())
    assert np.all(r["payload_est"][:, :, 0] <= 0.05)


def test_closed_loop_restores_the_model_payload_and_params_on_error():
    from qm_control_b200 import closed_loop
    s = _solver()
    try:
        prev = np.zeros((NL, 8)); prev[:, PL["m_ee"]] = 0.25; s.set_model_payload(prev); params = s.payload_est_get_params()
        for bad in ("yes", 1, [0.9]):
            with pytest.raises(ValueError):
                closed_loop.run(s, duration=0.01, payload_estimator=bad)
        with pytest.raises(ValueError):   # fails inside the run, after the estimator has started
            closed_loop.run(s, duration=0.01, cmd_vel=np.zeros(3), payload_estimator=dict(forgetting=0.99))
        with pytest.raises(ValueError):
            closed_loop.run(s, duration=0.01, payload_estimator=dict(no_such_parameter=1.0))
        np.testing.assert_array_equal(s.get_model_payload(), prev); assert s.payload_est_get_params() == params
        with pytest.raises(_lib.QmbError, match="not running"):
            s.payload_est_get()
    finally:
        s.close()
