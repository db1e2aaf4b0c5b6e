"""The slip detector on the host, no GPU (tests/_slip_twin.py with the state estimator's twin): no flag on noise-free and noisy stance feet of the CPU
rehearsal, an injected single-foot slide flagged, released and kept out of the estimate, the estimate unchanged when nothing is flagged, the
parameter struct's layout against include/qmb200.h, and closed_loop.run's calls with and without the detector on a fake Solver."""
import contextlib
import ctypes as C
import os
import subprocess
import types
from unittest import mock

import numpy as np
import pytest

import _attitude_twin as A
import _closed_loop_cpu
import _loop_replay as R
import _slip_twin as S
import _state_est_twin as T
from _oracle import Oracle
from qm_control_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOISE = dict(T.NOISE_OFF, seed=5, **_lib.SENSOR_NOISE_REFERENCE)
SETTLE = 50            # calls of start transient (the estimator's velocity settles from rest; d^2 up to 11 on the trot's first 40 calls)
FOOT, K0, N, SPEED = 0, 100, 50, 0.5   # the injected slide: foot LF, from call 100, 50 calls of 1 ms at 0.5 m/s along world x


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@pytest.fixture(scope="module")
def rehearsals(oracle):
    """the plant steps of 0.2 s of the CPU rehearsal (floor mu 0.6): {"trot": trot at 0.3 m/s, "stance": standing} → [(dt, q, v, v_prev, contact)]"""
    from qm_control_b200.interface import gait_schedule
    out = {}
    for tag, sched, cmd in (("trot", gait_schedule("trot", 10.0, 9.998, 12.2), (0.3, 0.0, 0.0, 0.0)), ("stance", None, (0.0, 0.0, 0.0, 0.0))):
        rec = R.Record()
        _closed_loop_cpu.run(oracle, duration=0.2, cmd_vel=cmd, t_start=10.0, mode_schedule=sched, recorder=rec)
        out[tag] = [(i["duration"], o["q"][0], o["v"][0], i["v"][0], int(o["contact"][0])) for i, o in rec.of("sim")]
    return out


def _rows(steps, noise, slide=None):
    """the sensor rows of plant steps (sample k - 1 for step k, the loop's numbering); slide = (oracle, foot, k0, n, u): from call k0 for n calls the
    encoders of the foot's leg read the joint motion of the foot sliding at world velocity u, integrated, so positions and rates agree; the leg keeps
    the displacement afterwards"""
    rows, dq = [], np.zeros(18)
    for k, (dt, q, v, v_prev, _) in enumerate(steps):
        s = T.read_sensors(q, v, v_prev, dt, k - 1, 0, noise)
        if slide is not None and slide[2] <= k < slide[2] + slide[3]:
            oracle, f, u = slide[0], slide[1], slide[4]
            e = T.zyx_from_rot(T.rot_from_quat(s[0:4]))
            J = oracle.rbd(np.r_[0.0, 0.0, 0.0, e, s[10:28] + dq], np.zeros(24))["Jfoot"][3 * f:3 * f + 3, 6:24]   # world axes, per joint rate
            cols = np.flatnonzero(np.any(J != 0.0, axis=0)); assert len(cols) == 3, cols
            rate = np.zeros(18); rate[cols] = np.linalg.solve(J[:, cols], u)
            dq = dq + dt * rate; s[28:46] += rate
        s[10:28] += dq
        rows.append(s)
    return rows


def _chain(oracle, steps, rows, detector=True, attitude=False, params=None):
    """[attitude filter →] slip detector → estimator twins on the rows → dict(slip [n, 4] flags, contact [n, 4] flags, rbd [n, 55], v_err [n])"""
    se = T.StateEstTwin(T.default_params(oracle.model_info()["mass"]), oracle); sl = S.SlipTwin(se, params); f = A.AttitudeTwin()
    st, ss, sa = se.reset(steps[0][1][0:3]), sl.reset(), f.reset()
    out = dict(slip=[], contact=[], rbd=[], v_err=[])
    for (dt, q, v, v_prev, contact), row in zip(steps, rows):
        if attitude:
            row, code = f.step(sa, dt, row); assert code == 0
        stance, slip, code = contact, 0, 0
        if detector:
            stance, slip, code, _ = sl.step(ss, st, dt, row, contact); assert code == 0
            assert stance == contact & ~slip and slip & ~contact == 0
        rbd, code = se.step(st, dt, row, stance); assert code == 0
        out["slip"].append(S.stance_flags(slip)); out["contact"].append(S.stance_flags(contact)); out["rbd"].append(rbd)
        out["v_err"].append(np.linalg.norm(rbd[27:30] - v[0:3]))
    return {k: np.array(a) for k, a in out.items()}


def test_stance_feet_are_not_flagged(oracle, rehearsals):
    """Noise-free, and with the reference IMU noise behind the attitude filter: after the start transient no stance foot of the rehearsal's stance
    and trot (floor mu 0.6) is flagged.  DESIGN.md §4.6 bounds the flagged fraction of stance samples at 1 %; measured 0 on all four streams."""
    for tag, steps in rehearsals.items():
        for noise, att in ((T.NOISE_OFF, False), (NOISE, True)):
            r = _chain(oracle, steps, _rows(steps, noise), attitude=att)
            inc = r["contact"][SETTLE:]; frac = r["slip"][SETTLE:][inc].mean()
            print("%s, %s: %d stance samples after the transient, flagged fraction %.4f" % (tag, "reference noise + attitude filter" if att else "noise-free", inc.sum(), frac))
            assert frac < 0.01 and inc.sum() > 300


def test_injected_slide_is_flagged_released_and_kept_out_of_the_estimate(oracle, rehearsals):
    """One stance foot's encoders read a 0.5 m/s slide for 50 ms: the foot is flagged within 3 calls and no other foot is; it is trusted again within
    hold + 3 calls after the slide ends; over the slide the estimator's |v_hat - v| is lower with the detector than without it."""
    steps = rehearsals["trot"]
    assert all(S.stance_flags(c)[FOOT] for *_, c in steps[K0 - 10:K0 + N + 20])   # the foot stays in contact over the window
    hold = S.default_params()["hold"]
    for noise, att in ((T.NOISE_OFF, False), (NOISE, True)):
        rows = _rows(steps, noise, slide=(oracle, FOOT, K0, N, np.array([SPEED, 0.0, 0.0])))
        with_det, without = _chain(oracle, steps, rows, attitude=att), _chain(oracle, steps, rows, detector=False, attitude=att)
        fl = with_det["slip"]; on = np.flatnonzero(fl[:, FOOT])
        onset, last = on[on >= K0].min() - K0, on.max() - (K0 + N - 1)
        e_det, e_raw = with_det["v_err"][K0:K0 + N].max(), without["v_err"][K0:K0 + N].max()
        print("%s: flagged %d call(s) after the slide starts, last flagged %d call(s) after it ends (hold %d); max |v_hat - v| over the slide %.3f m/s with "
              "the detector, %.3f m/s without" % ("reference noise + attitude filter" if att else "noise-free", onset, last, hold, e_det, e_raw))
        assert onset <= 3 and on.min() >= K0 and np.all(fl[K0 + 3:K0 + N, FOOT])
        assert 0 < last <= hold + 3
        assert not fl[SETTLE:, [f for f in range(4) if f != FOOT]].any()
        assert e_det < 0.5 * e_raw   # measured 0.014 against 0.213 m/s noise-free


def test_estimate_is_unchanged_when_no_foot_is_flagged(oracle, rehearsals):
    """With no foot flagged the estimator's outputs on the trusted mask are bit-identical to those on the plant's mask."""
    for steps in rehearsals.values():
        rows = _rows(steps, T.NOISE_OFF)
        a, b = _chain(oracle, steps, rows), _chain(oracle, steps, rows, detector=False)
        assert not a["slip"].any() and a["rbd"].tobytes() == b["rbd"].tobytes()


def test_first_call_and_non_finite_rows_pass_the_mask_through(oracle, rehearsals):
    se = T.StateEstTwin(T.default_params(oracle.model_info()["mass"]), oracle); sl = S.SlipTwin(se)
    dt, q, v, v_prev, contact = rehearsals["trot"][0]; row = T.read_sensors(q, v, v_prev, dt, -1, 0, T.NOISE_OFF)
    st, ss = se.reset(q[0:3]), sl.reset(); ss["mask"] = 8
    assert sl.step(ss, st, dt, row, 15)[:3] == (15, 0, 0) and ss["mask"] == 8   # the estimator has had no call
    se.step(st, dt, row, 15); bad = row.copy(); bad[30] = np.nan
    assert sl.step(ss, st, dt, bad, 15)[:3] == (15, 0, T.ST_NAN) and ss["mask"] == 8


def _offsets(tmp_path, struct, fields):
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "qmb200.h"', 'int main(void) {', '  printf("%%zu\\n", sizeof(%s));' % struct]
    body += ['  printf("%%zu\\n", offsetof(%s, %s));' % (struct, f) for f in fields] + ['  return 0; }']
    src = tmp_path / ("%s.c" % struct); src.write_text("\n".join(body) + "\n"); exe = tmp_path / struct
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    return [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]


def test_params_layout_matches_the_header(tmp_path):
    fields = [n for n, _ in _lib.SlipParams._fields_]
    out = _offsets(tmp_path, "qmb200_slip_params", fields)
    assert out[0] == C.sizeof(_lib.SlipParams) and out[1:] == [getattr(_lib.SlipParams, f).offset for f in fields]
    assert list(S.default_params()) == fields


# ---- closed_loop.run on a fake Solver, tensors on the CPU ----
B = 2


class _FakeStream:
    cuda_stream = 0

    def __init__(self, device=None):
        pass

    def synchronize(self):
        pass


def _fake_solver():
    params = dict(state_est_get_params={}, sim_get_sensor_params={}, attitude_get_params={}, slip_get_params={})
    names = ["sim_standing_state", "sim_step_dev", "sim_read_sensors_dev", "state_est_reset", "state_est_step_dev", "state_est_stop", "state_est_set_params",
             "sim_set_sensor_params", "attitude_reset", "attitude_step_dev", "attitude_stop", "attitude_set_params", "slip_reset", "slip_step_dev",
             "slip_stop", "slip_set_params", "centroidal_state_from_rbd", "initial_ee_target", "hw_set_delay", "target_trajectories_dev", "mpc_solve_dev",
             "update_dev", "hw_write_dev"] + list(params)
    s = mock.Mock(spec=names, batch=B, time_horizon=1.0, _cfg=types.SimpleNamespace(device=0))
    for n, v in params.items():
        getattr(s, n).return_value = v
    q0 = np.zeros((B, 24)); q0[:, 2] = 0.45
    s.sim_standing_state.return_value = (q0, np.zeros((B, 24)))
    s.centroidal_state_from_rbd.side_effect = lambda rbd: np.zeros((B, _lib.NX))
    s.initial_ee_target.return_value = np.zeros((B, 7))
    return s


def _calls(**kw):
    import torch
    from qm_control_b200 import closed_loop
    s = _fake_solver()
    with mock.patch.object(torch.cuda, "Stream", _FakeStream), mock.patch.object(torch.cuda, "stream", lambda st: contextlib.nullcontext()):
        r = closed_loop.run(s, duration=0.02, torch_device="cpu", state_estimator=True, **kw)
    return s, [c[0] for c in s.mock_calls], r


def _parent_calls(att):
    """the calls closed_loop.run issued before the slip detector existed, for a 20 ms run with the estimator (WBC every 2 ms)"""
    meas = ["sim_read_sensors_dev"] + (["attitude_step_dev"] if att else []) + ["state_est_step_dev"]
    out = ["state_est_get_params", "sim_get_sensor_params"] + (["attitude_get_params"] if att else [])
    out += ["sim_standing_state", "sim_step_dev", "sim_read_sensors_dev", "state_est_reset"] + (["attitude_reset", "attitude_step_dev"] if att else [])
    out += ["state_est_step_dev", "centroidal_state_from_rbd", "initial_ee_target", "hw_set_delay", "target_trajectories_dev", "mpc_solve_dev"]
    for k in range(20):
        out += (["target_trajectories_dev", "mpc_solve_dev"] if k == 10 else []) + (["update_dev"] if k % 2 == 0 else []) + ["hw_write_dev", "sim_step_dev"] + meas
    out += (["attitude_stop", "attitude_set_params"] if att else []) + ["state_est_stop", "sim_set_sensor_params", "state_est_set_params"]
    return out


@pytest.mark.parametrize("att", [False, True])
def test_loop_calls_without_the_detector_are_unchanged(att):
    s, calls, r = _calls(**({"attitude_filter": True} if att else {}))
    assert calls == _parent_calls(att) and "slip" not in r
    contact = s.sim_step_dev.call_args_list[0][0][5]
    assert all(c[0][2] is contact for c in s.state_est_step_dev.call_args_list)   # the estimator reads the plant's contact mask


@pytest.mark.parametrize("att", [False, True])
def test_loop_calls_with_the_detector(att):
    s, calls, r = _calls(slip_detector=dict(hold=3), **({"attitude_filter": True} if att else {}))
    # the parent's calls, with the detector's set-up, a detector step before every estimator step and its clean-up
    want, first_cleanup = [], "attitude_stop" if att else "state_est_stop"   # the scopes close in reverse: the detector's first
    for c in _parent_calls(att):
        if c == "sim_standing_state":
            want += ["slip_get_params", "slip_set_params"]
        if c == "state_est_step_dev":
            want += (["slip_reset"] if "slip_reset" not in want else []) + ["slip_step_dev"]
        if c == first_cleanup:
            want += ["slip_stop", "slip_set_params"]
        want.append(c)
    assert calls == want
    assert s.slip_set_params.call_args_list[0][1] == dict(hold=3)
    contact = s.sim_step_dev.call_args_list[0][0][5]
    for d, e in zip(s.slip_step_dev.call_args_list, s.state_est_step_dev.call_args_list):
        assert d[0][2] is contact and e[0][2] is d[0][3]   # the estimator reads the detector's stance mask
    assert r["slip"].shape == (2, B)


def test_loop_rejects_a_misplaced_detector():
    from qm_control_b200 import closed_loop
    s = _fake_solver()
    for kw in (dict(slip_detector=True), dict(slip_detector={}, sensor_noise=None), dict(state_estimator=True, slip_detector="yes")):
        with pytest.raises(ValueError, match="slip_detector"):
            closed_loop.run(s, duration=0.01, **kw)
    assert s.mock_calls == []
