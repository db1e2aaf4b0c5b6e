"""The slip detector on the device (qmb200_slip_*, closed_loop.run(slip_detector=...)), 64 robots.

The kernel is checked call by call against the numpy twin (tests/_slip_twin.py, on the state estimator's twin) on a recorded noisy trotting closed
loop on low-friction floors; then closed loops in which the estimator reads the detector's trusted stance mask."""
import numpy as np
import pytest

from qm_control_b200 import _lib

pytestmark = pytest.mark.gpu

NL = 64
MU = np.linspace(0.15, 0.6, NL)


def _solver(batch=NL):
    import qm_control_b200 as q
    return q.Solver(batch=batch, device=0)


def _upright(r):
    base = r["base"]
    return np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3)


def test_params_defaults_and_validation():
    import _slip_twin as S
    s = _solver(batch=2)
    try:
        assert s.slip_get_params() == S.default_params()
        for bad in (dict(gate=0.0), dict(gate=np.nan), dict(release=0.0), dict(release=20.0), dict(release=np.inf), dict(meas_slip=-1e-3),
                    dict(meas_slip=np.nan), dict(hold=-1)):
            with pytest.raises(_lib.QmbError):
                s.slip_set_params(**bad)
            assert s.slip_get_params() == S.default_params()
        for bad in (dict(no_such_parameter=1.0), dict(hold=2.5)):
            with pytest.raises(ValueError):
                s.slip_set_params(**bad)
        s.slip_set_params(release=16.27, hold=0); s.slip_set_params(**S.default_params())
        rows = np.zeros((2, _lib.SENSORS)); rows[:, 3] = 1.0; contact = np.array([15, 9], dtype=np.int32)
        for call in (lambda: s.slip_get(), lambda: s.slip_step(1e-3, rows, contact)):
            with pytest.raises(_lib.QmbError, match="slip detector is not running"):
                call()
        s.slip_stop()   # stopping a detector that is not running is a no-op
        s.slip_reset()
        with pytest.raises(_lib.QmbError, match="state estimator is not running"):
            s.slip_step(1e-3, rows, contact)
        s.state_est_reset(np.zeros((2, 3)))
        # before the estimator's first call the mask passes through; a non-finite row passes it through with QMB200_ST_NAN
        bad = rows.copy(); bad[1, 40] = np.nan
        stance, slip, st = s.slip_step(1e-3, bad, contact)
        assert stance.tolist() == [15, 9] and slip.tolist() == [0, 0] and st.tolist() == [0, S.ST_NAN]
        with pytest.raises(_lib.QmbError):
            s.slip_step(0.0, rows, contact)
        got = s.slip_get(); assert got["mask"].tolist() == [0, 0] and not got["hold"].any() and not got["onsets"].any()
        s.slip_stop(); s.slip_stop(); s.state_est_stop()
    finally:
        s.close()


def test_step_kernel_equals_the_twin_on_closed_loop_data():
    """0.3 s trot at 0.3 m/s on floors of mu 0.15-0.6 with the reference sensor noise, the attitude filter, the detector and the estimator: every call's
    stance and slip masks, status, and the stored mask, hold counters and onsets per robot equal the twin's, except at calls where some foot's d^2
    lies within 1e-9 relative of gate or release (counted and printed; the twin then takes the device's state)."""
    import torch
    import _slip_twin as S
    import _state_est_twin as T
    from qm_control_b200 import closed_loop
    s = _solver(); rec = []; orig = s.slip_step_dev

    def wrapped(dt, sensors, contact, stance, slip, status, stream=None):
        orig(dt, sensors, contact, stance, slip, status, stream)
        torch.cuda.synchronize()
        rec.append((dt, sensors.cpu().numpy(), contact.cpu().numpy(), stance.cpu().numpy(), slip.cpu().numpy(), status.cpu().numpy(), s.slip_get()))
    s.slip_step_dev = wrapped
    rng = np.random.default_rng(6); xy = np.c_[rng.uniform(-1, 1, (NL, 2)), rng.uniform(-np.pi, np.pi, NL)]
    try:
        closed_loop.run(s, duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, friction_mu=MU, state_estimator=True, attitude_filter=True,
                        slip_detector=True, sensor_noise="reference")
        se_params, sl_params = s.state_est_get_params(), s.slip_get_params()
        q0, _ = s.sim_standing_state(xy)
    finally:
        del s.slip_step_dev
        s.close()
    assert len(rec) == 301
    se = T.StateEstTwin(se_params); sl = S.SlipTwin(se, sl_params)
    st = [se.reset(q0[b, 0:3]) for b in range(NL)]; ss = [sl.reset() for _ in range(NL)]
    near, flagged = set(), np.zeros(NL, dtype=bool)
    for k, (dt, sn, contact, stance, slip, status, got) in enumerate(rec):
        for b in range(NL):
            t_stance, t_slip, t_code, d2 = sl.step(ss[b], st[b], dt, sn[b], contact[b])
            if sl.near_threshold(d2, contact[b]):
                near.add(k); ss[b] = dict(mask=int(got["mask"][b]), hold=got["hold"][b].astype(int), onsets=got["onsets"][b].astype(int))
            else:
                assert (t_stance, t_slip, t_code) == (stance[b], slip[b], status[b]), (k, b, t_stance, stance[b], t_slip, slip[b], t_code, status[b])
                assert ss[b]["mask"] == got["mask"][b] and np.array_equal(ss[b]["hold"], got["hold"][b]) and np.array_equal(ss[b]["onsets"], got["onsets"][b]), (k, b)
            se.step(st[b], dt, sn[b], stance[b])
            flagged[b] |= slip[b] != 0
    onsets = rec[-1][6]["onsets"]
    print("slip detector vs twin over %d calls x %d robots: %d call(s) with a d^2 within 1e-9 of a threshold; %d robots flagged, %d onsets in all" % (
        len(rec), NL, len(near), flagged.sum(), onsets.sum()))


def _loop(**kw):
    """closed_loop.run on a fresh handle with the running maxima per robot of |v_hat - v| over the estimator calls, r["v_err"] [B]"""
    import torch
    from qm_control_b200 import closed_loop
    s = _solver(); box = {}
    orig_sim, orig_est = s.sim_step_dev, s.state_est_step_dev

    def sim(duration, effort, q, v, rbd, contact, status, stream=None, wrench=None):
        box["rbd"] = rbd; orig_sim(duration, effort, q, v, rbd, contact, status, stream, wrench=wrench)

    def est(dt, sensors, contact, rbd_est, status, stream=None):
        orig_est(dt, sensors, contact, rbd_est, status, stream)
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            e = (rbd_est[:, 27:30] - box["rbd"][:, 27:30]).norm(dim=1)
            box["err"] = e if "err" not in box else torch.maximum(box["err"], e)
    s.sim_step_dev, s.state_est_step_dev = sim, est
    try:
        prev = (s.state_est_get_params(), s.sim_get_sensor_params(), s.slip_get_params())
        r = closed_loop.run(s, **kw)
        assert (s.state_est_get_params(), s.sim_get_sensor_params(), s.slip_get_params()) == prev   # restored
        with pytest.raises(_lib.QmbError, match="not running"):
            s.slip_get()
        torch.cuda.synchronize(); r["v_err"] = box["err"].cpu().numpy()
        return r
    finally:
        s.close()


def test_closed_loop_stance_noise_free():
    """A noise-free stance: no foot is flagged, no status bit, and the estimate is bit-identical to the run without the detector."""
    kw = dict(duration=1.0, gait="stance", state_estimator=True)
    r, raw = _loop(slip_detector=True, **kw), _loop(**kw)
    assert np.all(_upright(r)) and np.all(r["status"] == 0) and not r["slip"].any()
    assert r["base_est"].tobytes() == raw["base_est"].tobytes() and r["base"].tobytes() == raw["base"].tobytes()


def test_closed_loop_low_friction_trot():
    """A 1 s trot at 0.3 m/s on floors of mu 0.15-0.6 with the reference IMU noise and the attitude filter, with and without the detector: every output
    is finite, and no more robots fall with the detector than without it.  Fallen, xy drift of the estimate, |v_hat - v| and flagged robots per mu bin
    are printed (DESIGN.md §8)."""
    rng = np.random.default_rng(8); xy = np.c_[rng.uniform(-1, 1, (NL, 2)), np.zeros(NL)]
    kw = dict(duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, friction_mu=MU, state_estimator=True, attitude_filter=True, sensor_noise="reference")
    runs = {"with": _loop(slip_detector=True, **kw), "without": _loop(**kw)}
    for tag, r in runs.items():
        assert all(np.all(np.isfinite(r[k])) for k in ("base", "base_est", "ee", "q", "v")), tag
        fallen = ~_upright(r); drift = np.linalg.norm(r["base_est"][-1, :, 0:2] - r["base"][-1, :, 0:2], axis=1)
        flagged = r["slip"].any(axis=0) if "slip" in r else np.zeros(NL, dtype=bool)
        bins = [slice(i * NL // 4, (i + 1) * NL // 4) for i in range(4)]
        print("%s the detector: %d/%d fallen, xy drift p50 / p95 %.1f / %.1f mm, |v_hat - v| max p50 / p95 %.3f / %.3f m/s, %d robots flagged; per mu bin %s: "
              "fallen %s, flagged %s" % (tag, fallen.sum(), NL, 1e3 * np.median(drift), 1e3 * np.percentile(drift, 95), np.median(r["v_err"]), np.percentile(r["v_err"], 95),
                                         flagged.sum(), ["%.2f-%.2f" % (MU[b][0], MU[b][-1]) for b in bins], [int(fallen[b].sum()) for b in bins], [int(flagged[b].sum()) for b in bins]))
    assert (~_upright(runs["with"])).sum() <= (~_upright(runs["without"])).sum()


def test_one_robot_handle_matches_robot_0():
    """The same rows on a 64-robot handle and a one-robot handle: robot 0's outputs and state are identical."""
    rng = np.random.default_rng(3)
    s, one = _solver(), _solver(batch=1)
    try:
        for h in (s, one):
            h.state_est_reset(np.zeros((h.batch, 3))); h.slip_reset()
        q = np.zeros(24); q[2] = 0.45; v = np.zeros(24)
        for k in range(30):
            rows = np.tile(np.r_[0.0, 0.0, 0.0, 1.0, rng.normal(size=42) * 0.3], (NL, 1)); rows[:, 7:10] += [0.0, 0.0, 9.81]
            contact = np.full(NL, 15, dtype=np.int32)
            a = s.slip_step(1e-3, rows, contact); b = one.slip_step(1e-3, rows[:1], contact[:1])
            assert all(x[:1].tobytes() == y.tobytes() for x, y in zip(a, b)), k
            s.state_est_step(1e-3, rows, a[0]); one.state_est_step(1e-3, rows[:1], b[0])
        ga, gb = s.slip_get(), one.slip_get()
        assert all(ga[key][:1].tobytes() == gb[key].tobytes() for key in ga)
        assert ga["onsets"].any()   # random joint rates slide the feet: the test exercises the flags
    finally:
        s.close(); one.close()
