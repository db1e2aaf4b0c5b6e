"""The attitude filter on the device (qmb200_attitude_*, closed_loop.run(attitude_filter=...)), 64 robots.

The kernel is checked call by call against the numpy twin (tests/_attitude_twin.py) on a recorded trotting closed loop with the reference sensor
noise; then closed loops in which the controller reads the base state estimate built on the filtered orientation."""
import numpy as np
import pytest

from qm_control_b200 import _lib

pytestmark = pytest.mark.gpu

NL = 64


def _solver(batch=NL):
    import qm_control_b200 as q
    return q.Solver(batch=batch, device=0)


def _upright(r):
    base = r["base"]
    return np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3)


def _rows(rng, n, B):
    """n sensor readings of B robots: random unit quaternions (either sign) and rates; the other columns random"""
    out = rng.normal(size=(n, B, _lib.SENSORS)); out[:, :, 0:4] /= np.linalg.norm(out[:, :, 0:4], axis=2, keepdims=True)
    return out


def test_params_defaults_and_validation():
    import _attitude_twin as A
    s = _solver(batch=2)
    try:
        assert s.attitude_get_params() == A.default_params()
        for bad in (dict(process_attitude=-1e-3), dict(meas_orientation=0.0), dict(p0_gyro_bias=np.nan), dict(process_gyro_bias=np.inf), dict(p0_attitude=-1.0)):
            with pytest.raises(_lib.QmbError):
                s.attitude_set_params(**bad)
            assert s.attitude_get_params() == A.default_params()
        with pytest.raises(ValueError):
            s.attitude_set_params(no_such_parameter=1.0)
        for call in (lambda: s.attitude_get(), lambda: s.attitude_step(1e-3, np.zeros((2, _lib.SENSORS)))):
            with pytest.raises(_lib.QmbError, match="not running"):
                call()
        s.attitude_stop()   # stopping a filter that is not running is a no-op
        # the host variant: robot 1's non-finite gyro leaves its row as passed; robot 0 takes its normalised reading
        s.attitude_reset()
        rows = _rows(np.random.default_rng(2), 1, 2)[0]; rows[0, 0:4] *= 3.0; rows[1, 5] = np.nan
        out, st = s.attitude_step(1e-3, rows)
        assert st.tolist() == [0, A.ST_NAN]
        assert np.array_equal(out[1], rows[1], equal_nan=True) and out[0, 4:].tobytes() == rows[0, 4:].tobytes()
        want = rows[0, 0:4] / np.linalg.norm(rows[0, 0:4]); want = -want if want[3] < 0 else want
        np.testing.assert_allclose(out[0, 0:4], want, rtol=0, atol=1e-15)
        got = s.attitude_get(); assert got["samples"].tolist() == [1, 0]
        with pytest.raises(_lib.QmbError):
            s.attitude_step(0.0, rows)
        s.attitude_stop(); s.attitude_stop()
    finally:
        s.close()


def test_step_kernel_equals_the_twin_on_closed_loop_data():
    """0.3 s trot with the estimator, the attitude filter and the reference sensor noise on: every call's q_hat and output row per robot at 1e-12,
    b_hat and diag P at 1e-10 relative, status identical, the call count k + 1."""
    import torch
    import _attitude_twin as A
    from qm_control_b200 import closed_loop
    s = _solver(); rec = []
    orig = s.attitude_step_dev

    def wrapped(dt, sensors, status, stream=None):
        sn = sensors.clone()
        orig(dt, sensors, status, stream)
        torch.cuda.synchronize()
        rec.append((dt, sn.cpu().numpy(), sensors.cpu().numpy(), status.cpu().numpy(), s.attitude_get()))
    s.attitude_step_dev = wrapped
    rng = np.random.default_rng(6); xy = np.c_[rng.uniform(-1, 1, (NL, 2)), rng.uniform(-np.pi, np.pi, NL)]
    try:
        closed_loop.run(s, duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, state_estimator=True, attitude_filter=True, sensor_noise="reference")
        params = s.attitude_get_params()
    finally:
        del s.attitude_step_dev
        s.close()
    assert len(rec) == 301
    twin = A.AttitudeTwin(params); states = [twin.reset() for _ in range(NL)]
    worst = np.zeros(4)
    for k, (dt, sn, out, status, got) in enumerate(rec):
        for b in range(NL):
            row, code = twin.step(states[b], dt, sn[b])
            assert code == status[b], (k, b, code, status[b])
            st = states[b]
            eq = np.max(np.abs(got["quat"][b] - st["q"])); er = np.max(np.abs(out[b] - row))
            eb = np.max(np.abs(got["gyro_bias"][b] - st["b"])) / max(np.max(np.abs(st["b"])), 1e-6)
            pd = np.diag(st["P"]); ep = np.max(np.abs(got["p_diag"][b] - pd)) / np.max(np.abs(pd))
            worst = np.maximum(worst, [eq, er, eb, ep])
            assert eq < 1e-12 and er < 1e-12 and eb < 1e-10 and ep < 1e-10, (k, b, eq, er, eb, ep)
        assert np.all(got["samples"] == k + 1)
    print("attitude filter vs twin over 301 calls x %d robots: q_hat %.1e, row %.1e, b_hat %.1e, diag P %.1e (relative)" % (NL, *worst))


def test_one_robot_handle_matches_robot_0():
    rows = _rows(np.random.default_rng(3), 30, NL)
    s, one = _solver(), _solver(batch=1)
    try:
        s.attitude_reset(); one.attitude_reset()
        for k in range(len(rows)):
            a, _ = s.attitude_step(1e-3, rows[k]); b, _ = one.attitude_step(1e-3, rows[k][:1])
            assert a[:1].tobytes() == b.tobytes(), k
        ga, gb = s.attitude_get(), one.attitude_get()
        assert all(ga[key][:1].tobytes() == gb[key].tobytes() for key in ga)
    finally:
        s.close(); one.close()


def _loop(settle=100, **kw):
    """closed_loop.run on a fresh handle, with the running maxima per robot of the wrapped zyx error of rbd_est against the plant's rbd over the
    estimator calls from the settle-th on, r["ori_err"] [B] (the first calls rest on a few readings, each off by the reading's noise)"""
    import torch
    from qm_control_b200 import closed_loop
    s = _solver(); box = {"calls": 0}
    orig_sim, orig_est = s.sim_step_dev, s.state_est_step_dev

    def sim(duration, effort, q, v, rbd, contact, status, stream=None, wrench=None):
        box["rbd"] = rbd; orig_sim(duration, effort, q, v, rbd, contact, status, stream, wrench=wrench)

    def est(dt, sensors, contact, rbd_est, status, stream=None):
        orig_est(dt, sensors, contact, rbd_est, status, stream)
        box["calls"] += 1
        if box["calls"] <= settle:
            return
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            e = torch.remainder(rbd_est[:, 0:3] - box["rbd"][:, 0:3] + np.pi, 2 * np.pi).sub_(np.pi).abs().amax(dim=1)
            box["err"] = e if "err" not in box else torch.maximum(box["err"], e)
    s.sim_step_dev, s.state_est_step_dev = sim, est
    try:
        prev = (s.state_est_get_params(), s.sim_get_sensor_params(), s.attitude_get_params())
        r = closed_loop.run(s, **kw)
        assert (s.state_est_get_params(), s.sim_get_sensor_params(), s.attitude_get_params()) == prev   # restored
        torch.cuda.synchronize(); r["ori_err"] = box["err"].cpu().numpy()
        return r
    finally:
        s.close()


def _report(tag, r):
    dz = np.abs(r["base_est"][:, :, 2] - r["base"][:, :, 2])
    bits = np.bitwise_or.reduce(r["status"], axis=0)
    print("%s: %d/%d up, %d with status bits (OR 0x%x), wrapped zyx error of rbd_est after 0.1 s p50 / max %.2e / %.2e rad, max |z_hat - z| %.2e m" % (
        tag, int(_upright(r).sum()), NL, int(np.count_nonzero(bits)), int(np.bitwise_or.reduce(bits)), np.median(r["ori_err"]), r["ori_err"].max(), dz.max()))


def test_closed_loop_trot_with_reference_noise():
    """The point of the filter: a 1 s trot at 0.3 m/s on the estimate under the reference IMU noise keeps every robot upright, and the controller's
    orientation stays within the measured bound of the plant's.  The same run without the filter is printed beside it, not asserted on.  Some robots
    raise QMB200_ST_OVERFLOW: their random start yaws put the world-fixed end-effector target behind them (DESIGN.md §8), as on the true state."""
    rng = np.random.default_rng(8); xy = np.c_[rng.uniform(-1, 1, (NL, 2)), rng.uniform(-np.pi, np.pi, NL)]
    kw = dict(duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, state_estimator=True, sensor_noise="reference")
    r = _loop(attitude_filter=True, **kw)
    _report("trot, reference noise, with the attitude filter", r)
    _report("trot, reference noise, without it", _loop(**kw))
    assert np.all(_upright(r))
    assert r["ori_err"].max() < 0.015   # measured p50 / max 5.9e-3 / 1.1e-2 rad after 0.1 s; 0.13 / 0.15 rad without the filter


def test_closed_loop_stance_noise_free_with_the_filter():
    r = _loop(duration=1.0, gait="stance", state_estimator=True, attitude_filter=True)
    _report("stance, noise-free, with the attitude filter", r)
    assert np.all(_upright(r)) and np.all(r["status"] == 0) and np.all(r["contact"] == 15)


def test_closed_loop_rejects_a_misplaced_filter():
    from qm_control_b200 import closed_loop
    s = _solver()
    try:
        prev = s.attitude_get_params()
        for kw in (dict(attitude_filter=True), dict(state_estimator=True, attitude_filter="yes"), dict(state_estimator=True, attitude_filter=dict(no_such_parameter=1.0))):
            with pytest.raises(ValueError):
                closed_loop.run(s, duration=0.01, **kw)
        assert s.attitude_get_params() == prev
        closed_loop.run(s, duration=0.01, state_estimator=True, attitude_filter=dict(meas_orientation=2e-3))
        assert s.attitude_get_params() == prev
        with pytest.raises(_lib.QmbError, match="not running"):
            s.attitude_get()
    finally:
        s.close()
