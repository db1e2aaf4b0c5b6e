"""Per-episode metrics inside the GPU closed loop (closed_loop.run(metrics=True), DESIGN.md §4.13): every recorded metrics call equals the numpy
statement on its own inputs, every other output is byte-identical with and without metrics, the rows agree with the 10 ms record, episodes that repeat
bit for bit score bit for bit alike, and the entry points write only what they say."""
import numpy as np
import pytest

import _metrics_twin as mtw
from _oracle import Oracle
from qm_control_b200 import _lib
from qm_control_b200 import terrain as T
from test_respawn_gpu import _replay_case

pytestmark = pytest.mark.gpu

COL = {n: i for i, n in enumerate(_lib.METRICS_LAYOUT)}
WR = {n: i for i, n in enumerate(_lib.WRENCH_LAYOUT)}


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


def _np(a):
    return None if a is None else a.detach().cpu().numpy().copy()


# ---------------- 1 + 3: one call deep, and the rows against the record ----------------
CB, HOLD_S, EVERY_S, TILT_MAX = 32, 0.01, 0.1, 0.1


def _deep_setup():
    """32 robots trotting on randomized cmd_vel with the state estimator; every other robot is pushed sideways and rolled from each episode's start, and
    a tilt of 0.1 rad at a window's end counts as a fall, so that pushed robots restart on the fall rule and the others at the every limit"""
    xy = np.zeros((CB, 3)); xy[:, 0] = 2.0 * (np.arange(CB) % 8); xy[:, 1] = 2.0 * (np.arange(CB) // 8)
    w = np.zeros((CB, 12)); w[::2, WR["f_base_y"]] = 350.0; w[::2, WR["n_base_x"]] = 60.0
    return dict(duration=0.3, gait="trot", xy_yaw=xy, pushes=(np.zeros(CB), np.full(CB, 0.08), w), state_estimator=True,
                respawn=dict(hold=HOLD_S, every=EVERY_S, tilt_max=TILT_MAX), randomize=dict(seed=4, cmd_vel_x=(0.0, 0.4), cmd_yaw_rate=(-0.3, 0.3)))


@pytest.fixture(scope="module")
def deep():
    from qm_control_b200 import closed_loop
    s = _solver(CB); calls = []
    step, close = s.metrics_step_dev, s.metrics_close_dev

    def rec_step(dt, rbd, contact, effort, cmd, n_target, target_times, target_states, time, status, acc, kind=None, rbd_est=None, stream=None):
        c = dict(kind="step", dt=dt, rbd=_np(rbd), contact=_np(contact), effort=_np(effort), cmd=_np(cmd), n_target=_np(n_target), target_times=_np(target_times),
                 target_states=_np(target_states), time=_np(time), status=_np(status), kind_rows=_np(kind), rbd_est=_np(rbd_est), acc_in=_np(acc))
        step(dt, rbd, contact, effort, cmd, n_target, target_times, target_states, time, status, acc, kind=kind, rbd_est=rbd_est, stream=stream)
        c["acc_out"] = _np(acc); calls.append(c)

    def rec_close(mask, end, episode, acc, out, status, stream=None):
        c = dict(kind="close", mask=_np(mask), end=_np(end), episode=_np(episode), acc_in=_np(acc), out_in=_np(out), status_in=_np(status))
        close(mask, end, episode, acc, out, status, stream)
        c.update(acc_out=_np(acc), out_out=_np(out), status_out=_np(status)); calls.append(c)
    s.metrics_step_dev, s.metrics_close_dev = rec_step, rec_close
    try:
        r = closed_loop.run(s, metrics=True, **_deep_setup())
        ground = s.sim_get_params()["ground_height"]
    finally:
        s.close()
    return r, calls, ground


def test_every_metrics_call_is_the_numpy_statement_of_its_own_inputs(deep):
    r, calls, ground = deep
    twin = mtw.MetricsTwin(Oracle(), ground_height=ground)
    steps = [c for c in calls if c["kind"] == "step"]; closes = [c for c in calls if c["kind"] == "close"]
    assert len(steps) == 300 and len(closes) >= 3
    for i, c in enumerate(steps):
        want = twin.step(c["acc_in"], c["dt"], c["rbd"], c["contact"], c["effort"], c["cmd"], c["n_target"], c["target_times"], c["target_states"], c["time"],
                         c["status"], kind=c["kind_rows"], rbd_est=c["rbd_est"])
        np.testing.assert_allclose(c["acc_out"], want, rtol=1e-10, atol=1e-10, err_msg="step %d" % i)
    for i, c in enumerate(closes):
        acc, out, st = mtw.close(c["mask"], c["end"], c["episode"], c["acc_in"], c["out_in"], c["status_in"])
        np.testing.assert_allclose(c["out_out"], out, rtol=1e-10, atol=1e-10, err_msg="close %d" % i)
        np.testing.assert_array_equal(c["acc_out"], acc); np.testing.assert_array_equal(c["status_out"], st)
    assert all(c["kind_rows"] is None and c["rbd_est"] is not None for c in steps)


def test_rows_agree_with_the_record(deep):
    r = deep[0]; M, ep, fallen, st, base = r["episode_metrics"], r["episode"], r["fallen"], r["status"], r["base"]
    assert r["metrics_layout"] == _lib.METRICS_LAYOUT and M.shape == (CB, int(ep.max()) + 1, _lib.METRICS)
    hold = int(round(HOLD_S * 100)); ends = []
    for b in range(CB):
        for e in range(M.shape[1]):
            w = np.flatnonzero(ep[:, b] == e); row = M[b, e]
            if len(w) == 0:
                assert np.all(np.isnan(row)); continue
            assert int(round(row[COL["duration"]] / 1e-3)) == 10 * len(w), (b, e)      # one sample per plant step of the episode's windows
            assert row[COL["status"]] == float(np.bitwise_or.reduce(st[w, b].astype(np.int64) & 0xFFFFFFFF)), (b, e)
            last = e == ep[-1, b]
            fell = not last and len(w) >= hold and np.all(fallen[w[-hold:], b])
            ends.append(row[COL["end"]]); assert row[COL["end"]] == (0 if last else 1 if fell else 2), (b, e)
            tilt = np.max(np.maximum(np.abs(base[w, b, 4]), np.abs(base[w, b, 5])))
            assert row[COL["max_tilt"]] >= tilt and row[COL["min_height"]] <= np.min(base[w, b, 2])
            assert row[COL["touchdowns"]] >= 0 and row[COL["energy"]] > 0 and np.isfinite(row[COL["est_pos_err_rms"]])
    assert 1 in ends and 2 in ends and 0 in ends, "the pushes toppled no robot"


# ---------------- 2 + 5: every other output is byte-identical; one episode without respawn ----------------
RB = 12


def _case(case):
    xy = np.zeros((RB, 3)); xy[:, 0] = 3.0 * np.arange(RB)
    kw = dict(duration=0.2, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.1), xy_yaw=xy)
    if case == "estimate":
        kw.update(state_estimator=True, attitude_filter=True, slip_detector=True, sensor_noise="reference")
    if case == "commands":
        goal = np.full((RB, 2, 7), np.nan); goal[:, 1] = np.c_[xy[:, 0] + 0.52, xy[:, 1] + 0.09, np.full(RB, 0.49), np.tile([0.5, -0.5, 0.5, -0.5], (RB, 1))]
        kw.update(gait="stance", commands=dict(t=np.tile([0.03, 0.1], (RB, 1)), gait=np.tile(np.array(["trot", None], dtype=object), (RB, 1)), ee_goal=goal))
    if case == "episodes":
        tiles = np.stack([T.ramp(8.0), T.stairs(0.04, 0.3), T.rough(0.015, seed=2)])
        kw.update(terrain=dict(tiles=tiles, cell=T.CELL, tile=np.arange(RB) % 3, origin=T.centred_origin(xy[:, :2])), state_estimator=True, ground_map=True,
                  respawn=dict(every=0.05), randomize=dict(seed=9, friction_mu=(0.3, 0.9), cmd_vel_x=(0.0, 0.4)),
                  spawn=dict(seed=2, tile=(-1, 2), dx=(-0.2, 0.2), yaw=(-np.pi, np.pi)))
    return kw


@pytest.mark.parametrize("case", ["truth", "estimate", "commands", "episodes"])
def test_every_other_output_is_byte_identical_with_and_without_metrics(case):
    from qm_control_b200 import closed_loop
    runs = []
    for m in (None, True):
        s = _solver(RB)
        try:
            runs.append(closed_loop.run(s, metrics=m, **_case(case)))
        finally:
            s.close()
    plain, scored = runs
    assert set(scored) - set(plain) == {"episode_metrics", "metrics_layout"}
    for k, v in plain.items():
        if isinstance(v, np.ndarray):
            assert v.dtype == scored[k].dtype and v.tobytes() == scored[k].tobytes(), k
        else:
            assert v == scored[k], k
    M = scored["episode_metrics"]
    if case == "episodes":
        assert M.shape[1] == 4 and np.all(M[:, :3, COL["end"]] == 2) and np.all(M[:, 3, COL["end"]] == 0)
        assert np.all(np.isfinite(M[..., COL["min_height"]])) and np.all(np.isfinite(M[..., COL["est_vel_err_rms"]]))
    else:   # no respawn: one episode over the whole run, closed by its end
        assert M.shape == (RB, 1, _lib.METRICS)
        np.testing.assert_array_equal(np.round(M[:, 0, COL["duration"]] / 1e-3), 200); np.testing.assert_array_equal(M[:, 0, COL["end"]], 0)
        if case == "truth":
            assert np.all(M[:, 0, COL["vel_err_rms"]] < 0.3) and np.all(np.isnan(M[:, 0, COL["est_pos_err_rms"]])) and np.all(M[:, 0, COL["touchdowns"]] > 0)
        if case == "commands":   # cmd_vel samples until the goal is published at 0.1 s
            assert np.all(np.isfinite(M[:, 0, COL["vel_err_rms"]]))


# ---------------- 4: episodes that repeat score alike ----------------
@pytest.mark.parametrize("case", ["truth", "estimate"])
def test_repeating_episodes_have_bit_identical_rows(case):
    from qm_control_b200 import closed_loop
    kw, skw = _replay_case(case)
    s = _solver(16, **skw)
    try:
        r = closed_loop.run(s, metrics=True, **kw)
    finally:
        s.close()
    M = r["episode_metrics"]; assert M.shape[1] == 3
    np.testing.assert_array_equal(M[:, :, COL["end"]], np.tile([2, 2, 0], (16, 1)))
    keep = [i for i in range(_lib.METRICS) if i != COL["end"]]
    for e in (1, 2):
        assert M[:, e, keep].tobytes() == M[:, 0, keep].tobytes(), "episode %d" % e
    assert np.all(M[:, :, COL["path_length"]] > 0) and not np.any(np.isnan(M[:, :, COL["ee_pos_err_rms"]]))


# ---------------- 6: the entry points ----------------
def test_close_writes_masked_robots_only_and_refusals_write_nothing():
    import torch
    B, E = 8, 3; s = _solver(B); rng = np.random.default_rng(3); dev = torch.device("cuda:0")
    try:
        acc0 = np.abs(rng.normal(size=(B, _lib.METRICS_ACC))); acc0[:, 0] = rng.integers(0, 4, B); acc0[:, [19, 29]] = 1.0; acc0[:, 2] = 5.0
        out0 = rng.normal(size=(B, E, _lib.METRICS)); st0 = rng.integers(0, 4, B).astype(np.int32)
        mask = np.array([1, 0, 1, 1, 0, 1, 1, 0], dtype=np.int32); end = np.array([0, 1, 2, 3, 0, 1, 2, 0], dtype=np.int32)
        episode = np.array([0, 1, 2, 0, 1, 3, -1, 2], dtype=np.int32)
        t = lambda a: torch.as_tensor(a, device=dev)
        acc, out, st = t(acc0.copy()), t(out0.copy()), t(st0.copy())
        s.metrics_close_dev(t(mask), t(end), t(episode), acc, out, st); torch.cuda.synchronize()
        wa, wo, ws = mtw.close(mask, end, episode, acc0, out0, st0)
        np.testing.assert_array_equal(_np(acc), wa); np.testing.assert_allclose(_np(out), wo, rtol=1e-15); np.testing.assert_array_equal(_np(st), ws)
        quiet = (mask == 0) | (end == 3)   # unmasked, and the masked robot with an end outside {0, 1, 2}
        assert _np(acc)[quiet].tobytes() == acc0[quiet].tobytes() and _np(out)[quiet].tobytes() == out0[quiet].tobytes() and np.all(_np(st)[quiet] == st0[quiet])
        assert np.all(_np(st)[[5, 6]] & 2) and np.all(_np(acc)[[5, 6]] == 0)   # episode 3 and -1: no row, the overflow bit, reopened
        host = s.metrics_close(mask, np.where(end == 3, 0, end), episode, acc0, out0, st0)   # the host variant is the same launch
        np.testing.assert_array_equal(host["out"][~quiet], _np(out)[~quiet])
        with pytest.raises(_lib.QmbError, match="end of robot 3 must be 0, 1 or 2"):
            s.metrics_close(mask, end, episode, acc0, out0, st0)
        # refusals: nothing written
        a2, o2, s2 = t(acc0.copy()), t(out0.copy()), t(st0.copy())
        for bad in (lambda: s.metrics_close_dev(None, t(end), t(episode), a2, o2, s2), lambda: s.metrics_close_dev(t(mask), t(end), t(episode), a2, o2[:, :0], s2)):
            with pytest.raises(_lib.QmbError):
                bad()
        z = torch.zeros((B, _lib.RBD), dtype=torch.float64, device=dev); zi = torch.zeros(B, dtype=torch.int32, device=dev)
        args = (z, zi, torch.zeros((B, 18), dtype=torch.float64, device=dev), torch.zeros((B, 7), dtype=torch.float64, device=dev), zi,
                torch.zeros((B, _lib.KMAX), dtype=torch.float64, device=dev), torch.zeros((B, _lib.KMAX, _lib.TARGET), dtype=torch.float64, device=dev),
                torch.zeros(B, dtype=torch.float64, device=dev), zi, a2)
        for dt in (0.0, -1e-3, np.nan, np.inf):
            with pytest.raises(_lib.QmbError, match="dt must be finite and > 0"):
                s.metrics_step_dev(dt, *args)
        with pytest.raises(_lib.QmbError, match="null buffer"):
            s.metrics_step_dev(1e-3, None, *args[1:])
        torch.cuda.synchronize()
        assert _np(a2).tobytes() == acc0.tobytes() and _np(o2).tobytes() == out0.tobytes() and _np(s2).tobytes() == st0.tobytes()
        # the host step is the device step
        s.metrics_step_dev(1e-3, *args); torch.cuda.synchronize()
        host = s.metrics_step(1e-3, *(_np(a) for a in args[:-1]), acc0)
        assert host.tobytes() == _np(a2).tobytes()
    finally:
        s.close()
