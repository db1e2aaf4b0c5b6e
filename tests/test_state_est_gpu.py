"""The sensor model and the base state estimator on the device (qmb200_sim_read_sensors, qmb200_state_est_*, closed_loop.run(state_estimator=...)),
64 robots.

The sensor kernel is checked against the numpy twin (tests/_state_est_twin.py) on recorded plant states, the filter kernel call by call on a recorded
trotting closed loop with the reference sensor noise; then closed loops in which the controller reads only the estimate."""
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


def _wrap(a):
    return (a + np.pi) % (2 * np.pi) - np.pi


def test_params_defaults_and_validation():
    import _state_est_twin as T
    s = _solver(batch=2)
    try:
        assert s.sim_get_sensor_params() == T.NOISE_OFF
        assert s.state_est_get_params() == T.default_params(s.robot_mass)
        for bad in (dict(sigma_gyro=-1.0), dict(sigma_accel=np.nan), dict(sigma_orientation=np.inf)):
            with pytest.raises(_lib.QmbError):
                s.sim_set_sensor_params(**bad)
            assert s.sim_get_sensor_params() == T.NOISE_OFF
        for bad in (dict(process_base_pos=-1e-3), dict(meas_foot_vel=np.nan), dict(swing_scale=-2.0), dict(foot_height=np.inf), dict(p0_foot=np.inf)):
            with pytest.raises(_lib.QmbError):
                s.state_est_set_params(**bad)
            assert s.state_est_get_params() == T.default_params(s.robot_mass)
        s.sim_set_sensor_params(seed=2 ** 64 - 1, **_lib.SENSOR_NOISE_REFERENCE)
        assert s.sim_get_sensor_params() == dict(T.NOISE_OFF, seed=2 ** 64 - 1, **_lib.SENSOR_NOISE_REFERENCE)
        s.state_est_set_params(foot_height=-0.5); assert s.state_est_get_params()["foot_height"] == -0.5
        for call in (lambda: s.state_est_get(), lambda: s.state_est_step(1e-3, np.zeros((2, 46)), np.zeros(2))):
            with pytest.raises(_lib.QmbError, match="not running"):
                call()
        with pytest.raises(_lib.QmbError):
            s.state_est_reset(np.full((2, 3), np.nan))
        s.state_est_stop()   # stopping a filter that is not running is a no-op
    finally:
        s.close()


@pytest.mark.parametrize("noise", ["off", "reference"])
def test_sensor_kernel_equals_the_twin(noise):
    """Plant states of 64 robots at random yaw after random-effort steps: every reading at 1e-12, the draws those of each robot's own index."""
    import _state_est_twin as T
    s = _solver(); rng = np.random.default_rng(1)
    try:
        p = dict(T.NOISE_OFF) if noise == "off" else dict(T.NOISE_OFF, seed=99, sigma_joint_pos=1e-3, sigma_joint_vel=2e-2, **_lib.SENSOR_NOISE_REFERENCE)
        s.sim_set_sensor_params(**p)
        q, v = s.sim_standing_state(np.c_[rng.uniform(-1, 1, (NL, 2)), rng.uniform(-np.pi, np.pi, NL)])
        worst = 0.0
        for k in range(5):
            v_prev = v
            q1, v1, _, _, _ = s.sim_step(1e-3, rng.uniform(-40, 40, (NL, 18)), q, v)
            got = s.sim_read_sensors(1e-3, k, q1, v1, v)
            for b in range(NL):
                want = T.read_sensors(q1[b], v1[b], v[b], 1e-3, k, b, p)
                if want[3] * got[b, 3] < 0:   # q and -q are one rotation: compare the rotation
                    want[0:4] = -want[0:4]
                worst = max(worst, np.max(np.abs(got[b] - want)))
            q, v = q1, v1
        print("sensor kernel vs twin (%s): %.1e" % (noise, worst))
        assert worst < 1e-12
        one = _solver(batch=1)   # robot 0 alone draws what robot 0 of the batch draws
        try:
            one.sim_set_sensor_params(**p)
            assert one.sim_read_sensors(1e-3, 4, q[:1], v[:1], v_prev[:1]).tobytes() == s.sim_read_sensors(1e-3, 4, q, v, v_prev)[:1].tobytes()
        finally:
            one.close()
    finally:
        s.close()


def test_step_kernel_equals_the_twin_on_closed_loop_data():
    """0.3 s trot with the estimator and the reference sensor noise on: every call's x and diag P per robot at 1e-10 relative, rbd_est at 1e-9, status
    bits identical."""
    import torch
    import _state_est_twin as T
    from qm_control_b200 import closed_loop
    s = _solver(); rec = []
    orig = s.state_est_step_dev

    def wrapped(dt, sensors, contact, rbd_est, status, stream=None):
        sn, c = sensors.clone(), contact.clone()
        orig(dt, sensors, contact, rbd_est, status, stream)
        torch.cuda.synchronize()
        rec.append((dt, sn.cpu().numpy(), c.cpu().numpy(), rbd_est.cpu().numpy(), status.cpu().numpy(), s.state_est_get()))
    s.state_est_step_dev = wrapped
    rng = np.random.default_rng(6); xy = np.c_[rng.uniform(-1, 1, (NL, 2)), rng.uniform(-np.pi, np.pi, NL)]
    try:
        closed_loop.run(s, duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, state_estimator=True, sensor_noise="reference")
        params = s.state_est_get_params()
    finally:
        del s.state_est_step_dev
        s.close()
    assert len(rec) == 301
    twin = T.StateEstTwin(params); states = [twin.reset(rec[0][5]["x"][b, 0:3]) for b in range(NL)]
    worst = np.zeros(3)
    for k, (dt, sens, contact, rbd_est, status, got) in enumerate(rec):
        for b in range(NL):
            rbd, code = twin.step(states[b], dt, sens[b], int(contact[b]))
            assert code == status[b], (k, b, code, status[b])
            x, pd = states[b]["x"], np.diag(states[b]["P"])
            ex = np.max(np.abs(got["x"][b] - x)) / max(np.max(np.abs(x)), 1e-2); ep = np.max(np.abs(got["p_diag"][b] - pd)) / np.max(np.abs(pd))
            d = rbd_est[b] - rbd; d[0:3] = _wrap(d[0:3])
            if rbd[54] * rbd_est[b, 54] < 0:
                d[51:55] = rbd_est[b, 51:55] + rbd[51:55]
            er = np.max(np.abs(d))
            worst = np.maximum(worst, [ex, ep, er])
            assert ex < 1e-10 and ep < 1e-10 and er < 1e-9, (k, b, ex, ep, er)
        assert np.all(got["samples"] == k + 1)
    print("state estimator vs twin over 301 calls x %d robots: x %.1e, diag P %.1e (worst relative), rbd_est %.1e" % (NL, *worst))


def _loop(watch=False, **kw):
    """closed_loop.run on a fresh handle; with watch, the running maxima over every estimator call of |rbd_est - rbd| on the orientation (wrapped),
    joints, w_world and joint rates, and of |v_hat - v|"""
    import torch
    from qm_control_b200 import closed_loop
    s = _solver(); box = {}
    if watch:
        orig_sim, orig_est = s.sim_step_dev, s.state_est_step_dev

        def sim(duration, effort, q, v, rbd, contact, status, stream=None, wrench=None):
            box["rbd"] = rbd; orig_sim(duration, effort, q, v, rbd, contact, status, stream, wrench=wrench)

        def est(dt, sensors, contact, rbd_est, status, stream=None):
            orig_est(dt, sensors, contact, rbd_est, status, stream)
            with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
                d = (rbd_est - box["rbd"]).abs(); d[:, 0:3] = torch.remainder(rbd_est[:, 0:3] - box["rbd"][:, 0:3] + np.pi, 2 * np.pi).sub_(np.pi).abs()
                err = torch.stack([torch.cat([d[:, 0:3], d[:, 6:27], d[:, 30:48]], 1).max(), d[:, 27:30].max()])
                box["err"] = err if "err" not in box else torch.maximum(box["err"], err)
        s.sim_step_dev, s.state_est_step_dev = sim, est
    try:
        prev = (s.state_est_get_params(), s.sim_get_sensor_params())
        r = closed_loop.run(s, **kw)
        assert (s.state_est_get_params(), s.sim_get_sensor_params()) == prev   # restored
        if watch:
            torch.cuda.synchronize(); r["watch"] = box["err"].cpu().numpy()
        return r
    finally:
        s.close()


def _report(tag, r):
    dz = np.abs(r["base_est"][:, :, 2] - r["base"][:, :, 2]); dxy = np.linalg.norm(r["base_est"][-1, :, 0:2] - r["base"][-1, :, 0:2], axis=1)
    print("%s: %d/%d up, max |z_hat - z| %.2e m, max |v_hat - v| %.2e m/s, xy drift at the end p50 / max %.2e / %.2e m, rbd_est vs rbd %.1e" % (
        tag, int(_upright(r).sum()), NL, dz.max(), r["watch"][1], np.median(dxy), dxy.max(), r["watch"][0]))
    return dz.max(), r["watch"][1]


def test_closed_loop_stance_on_the_estimate():
    r = _loop(watch=True, duration=1.0, gait="stance", state_estimator=True)
    dz, dv = _report("stance, noise-free estimate", r)
    assert np.all(_upright(r)) and np.all(r["status"] == 0) and np.all(r["contact"] == 15)
    assert r["watch"][0] < 1e-12
    assert dz < 2e-4 and dv < 0.012


def test_closed_loop_trot_through_yaw_pi_on_the_estimate():
    """Trot at 0.3 m/s turning at -1 rad/s from yaw -pi + 0.2: the plant's yaw passes -pi, the estimate's yaw wraps to +pi and the observation unwraps it.
    The turn runs towards -pi: the loop's end-effector orientation target is fixed in the world (the target front-end keeps the first one), so near
    yaw +-pi the arm holds its end effector almost half a turn from its natural pose and pulls the base back; turning the other way from +pi - 0.1 the
    controller on the true state never reaches pi and raises QMB200_ST_OVERFLOW on some robots (DESIGN.md §8)."""
    xy = np.c_[np.zeros((NL, 2)), np.full(NL, -np.pi + 0.2)]
    r = _loop(watch=True, duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, -1.0), xy_yaw=xy, state_estimator=True)
    dz, dv = _report("trot through yaw -pi, noise-free estimate", r)
    past = r["base"][:, :, 3] < -np.pi
    assert np.all(past.any(axis=0)), "the yaw must pass -pi"
    assert np.all(r["base_est"][:, :, 3][past] > 0.0)   # the estimate reports the wrapped yaw there
    assert np.all(_upright(r)) and np.all(r["status"] == 0)
    assert r["watch"][0] < 1e-12
    assert dz < 5e-4 and dv < 0.08


def test_closed_loop_with_both_estimators():
    pl = np.zeros((NL, 8)); pl[:, 0] = 1.0
    r = _loop(duration=1.0, gait="stance", payload=pl, payload_estimator=True, state_estimator=True)
    print("stance, 1 kg EE payload, payload and state estimators: %d/%d up, m_hat p50 %.3f kg" % (int(_upright(r).sum()), NL, np.median(r["payload_est"][-1, :, 0])))
    assert all(np.all(np.isfinite(r[k])) for k in ("base", "base_est", "ee", "payload_est"))
    assert np.all(_upright(r))


def test_closed_loop_rejects_what_the_estimator_cannot_do():
    from qm_control_b200 import closed_loop
    from qm_control_b200 import terrain as T
    s = _solver()
    try:
        prev = (s.state_est_get_params(), s.sim_get_sensor_params())
        ter = dict(tiles=T.ramp(5.0, start=0.35)[None], cell=T.CELL, tile=np.zeros(NL, dtype=np.int32), origin=T.centred_origin(np.zeros((NL, 2))))
        for kw in (dict(state_estimator=True, terrain=ter), dict(state_estimator="yes"), dict(sensor_noise="reference"),
                   dict(state_estimator=True, sensor_noise="loud"), dict(state_estimator=dict(no_such_parameter=1.0))):
            with pytest.raises(ValueError):
                closed_loop.run(s, duration=0.01, **kw)
        assert (s.state_est_get_params(), s.sim_get_sensor_params()) == prev and s.sim_get_terrain() is None
        with pytest.raises(_lib.QmbError, match="not running"):
            s.state_est_get()
    finally:
        s.close()
