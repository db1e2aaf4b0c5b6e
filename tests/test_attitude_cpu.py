"""The attitude filter on the host, no GPU (tests/_attitude_twin.py): noise-free tracking on plant-twin trajectories and on the CPU rehearsal of a
trotting closed loop, the reference IMU noise on a synthetic rocking rotation, an injected gyro bias, the filter's invariances, its benefit to the
base state estimator on the rehearsal, and the parameter struct's layout against include/qmb200.h."""
import ctypes as C
import copy
import os
import subprocess

import numpy as np
import pytest

import _attitude_twin as A
import _closed_loop_cpu
import _loop_replay as R
import _state_est_twin as T
from _oracle import Oracle
from _sim_twin import SimTwin
from qm_control_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOISE = dict(T.NOISE_OFF, seed=5, **_lib.SENSOR_NOISE_REFERENCE)
BIAS = np.array([0.05, -0.03, 0.02])


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@pytest.fixture(scope="module")
def rehearsal(oracle):
    """the plant steps of a 0.2 s trot at 0.3 m/s of the CPU rehearsal: [(duration, q, v, v_prev, contact)]"""
    from qm_control_b200.interface import gait_schedule
    rec = R.Record(); sched = gait_schedule("trot", 10.0, 9.998, 12.2)
    _closed_loop_cpu.run(oracle, duration=0.2, cmd_vel=(0.3, 0.0, 0.0, 0.0), t_start=10.0, mode_schedule=sched, recorder=rec)
    return [(i["duration"], o["q"][0], o["v"][0], i["v"][0], int(o["contact"][0])) for i, o in rec.of("sim")]


def _twin_trajectory(oracle, steps=40, seed=3):
    """plant-twin steps of 1 ms from the standing state with random efforts: [(dt, q, v, v_prev)]"""
    twin = SimTwin(); rng = np.random.default_rng(seed)
    q, v = _closed_loop_cpu.standing_state(oracle, twin, yaw=2.5)
    out = []
    for _ in range(steps):
        q1, v1, _, _, _ = twin.step(1e-3, rng.uniform(-30, 30, 18), q, v)
        out.append((1e-3, q1, v1, v)); q, v = q1, v1
    return out


def _rocking(seconds=3.0, yaw0=2.9, yaw_rate=0.4, dt=1e-3):
    """a synthetic base rotation: a slow turn under a 2.5 Hz rocking in pitch (0.1 rad) and roll (0.08 rad): [(dt, q, v, v_prev)]"""
    out, w = [], 2 * np.pi * 2.5
    for k in range(int(round(seconds / dt))):
        t = (k + 1) * dt
        e = [yaw0 + yaw_rate * t, 0.1 * np.sin(w * t), 0.08 * np.sin(w * t + 1.0)]
        ed = [yaw_rate, 0.1 * w * np.cos(w * t), 0.08 * w * np.cos(w * t + 1.0)]
        q = np.r_[0.0, 0.0, 0.45, e, np.zeros(18)]; v = np.r_[0.0, 0.0, 0.0, ed, np.zeros(18)]
        out.append((dt, q, v, v))
    return out


def _run(steps, noise, bias=np.zeros(3), params=None, check_p=False):
    """the twin on the readings of plant states [(dt, q, v, v_prev)] (sample k - 1 for step k, the loop's numbering) → (angle errors of the raw reading
    and of the filtered one against the plant [n], the final state)"""
    f = A.AttitudeTwin(params); s = f.reset(); raw, filt = [], []
    for k, (dt, q, v, v_prev) in enumerate(steps):
        sens = T.read_sensors(q, v, v_prev, dt, k - 1, 0, noise); sens[4:7] += bias
        out, code = f.step(s, dt, sens)
        assert code == 0, k
        if check_p:
            P = s["P"]; assert np.array_equal(P, P.T) and np.linalg.eigvalsh(P).min() > 0, k
        qt = T.quat_from_rot(T.rot_zyx(q[3:6]))
        raw.append(A.angle_between(qt, sens[0:4])); filt.append(A.angle_between(qt, out[0:4]))
    return np.array(raw), np.array(filt), s


def test_noise_free_readings_track_the_plant(oracle, rehearsal):
    """Noise off: the filtered orientation stays within a bound of the plant's.  The gyro reading ends the step, so each prediction lags the plant's
    rotation by about half a step's worth (|w| dt / 2 once the filter has settled); that lag, not rounding, sets the bound."""
    _, e_twin, _ = _run(_twin_trajectory(oracle), T.NOISE_OFF)
    _, e_reh, _ = _run([(dt, q, v, vp) for dt, q, v, vp, _ in rehearsal], T.NOISE_OFF)
    _, e_rock, _ = _run(_rocking(1.0), T.NOISE_OFF)
    print("noise-free orientation error, max: random-effort twin steps %.2e rad, rehearsal trot %.2e rad, rocking rotation %.2e rad" % (
        e_twin.max(), e_reh.max(), e_rock.max()))
    assert e_twin.max() < 1e-3 and e_reh.max() < 2e-4 and e_rock.max() < 1.2e-3   # measured 6.9e-4, 1.2e-4, 9.4e-4


def test_reference_noise_is_filtered():
    """The reference IMU noise on 3 s of the rocking rotation: the filtered orientation's RMS error over the second half is far below the reading's."""
    raw, filt, _ = _run(_rocking(3.0), NOISE)
    h = len(raw) // 2; rms = lambda a: float(np.sqrt(np.mean(a[h:] ** 2)))
    print("reference noise, rocking rotation, RMS over the second half: reading %.4f rad, filtered %.4f rad (%.1fx)" % (rms(raw), rms(filt), rms(raw) / rms(filt)))
    assert rms(raw) / rms(filt) > 14.0   # measured 0.0594 -> 0.0038 rad, 15.8x


def test_gyro_bias_is_learned():
    """A constant gyro bias added to the noisy gyro columns: b_hat within 5 mrad/s of it after 3 s; P symmetric positive definite throughout."""
    raw, filt, s = _run(_rocking(3.0), NOISE, bias=BIAS, check_p=True)
    h = len(raw) // 2; rms = lambda a: float(np.sqrt(np.mean(a[h:] ** 2)))
    err = np.linalg.norm(s["b"] - BIAS)
    print("gyro bias %s: |b_hat - b| %.2e rad/s after 3 s, filtered RMS %.4f rad" % (BIAS, err, rms(filt)))
    assert err < 5e-3


def test_invariances():
    f = A.AttitudeTwin(); steps = _rocking(0.3); rng = np.random.default_rng(4)
    # q_m and -q_m: bit-identical rows
    a, b = f.reset(), f.reset()
    for k, (dt, q, v, vp) in enumerate(steps):
        sens = T.read_sensors(q, v, vp, dt, k, 0, NOISE); flip = sens.copy()
        if rng.random() < 0.5:
            flip[0:4] = -flip[0:4]
        oa, _ = f.step(a, dt, sens); ob, _ = f.step(b, dt, flip)
        assert oa.tobytes() == ob.tobytes(), k
    # a yaw carried through +-pi: q_hat never changes sign, moves in small steps once settled (the first calls weigh single readings) and stays on the
    # plant, while the reading's w changes sign
    s = f.reset(); prev = None; worst = 0.0; crossed = False; w_signs = set()
    for k, (dt, q, v, vp) in enumerate(_rocking(0.6, yaw0=np.pi - 0.2, yaw_rate=1.0)):
        sens = T.read_sensors(q, v, vp, dt, k, 0, NOISE); out, _ = f.step(s, dt, sens)
        crossed = crossed or q[3] > np.pi; w_signs.add(bool(T.quat_from_rot(T.rot_zyx(q[3:6]))[3] >= 0))
        if prev is not None:
            assert np.dot(prev, s["q"]) > 0.0 and (k < 100 or A.angle_between(prev, s["q"]) < 5e-3), k
        if k >= 100:
            worst = max(worst, A.angle_between(T.quat_from_rot(T.rot_zyx(q[3:6])), out[0:4]))
        prev = s["q"].copy()
    print("yaw through pi: worst orientation error after 0.1 s %.2e rad" % worst)
    assert crossed and len(w_signs) == 2 and worst < 0.01, worst
    # the first call returns the normalised reading and leaves the other columns as they are
    s = f.reset(); sens = T.read_sensors(*steps[0][1:], 1e-3, 0, 0, NOISE); sens[0:4] *= -2.0
    out, code = f.step(s, 1e-3, sens)
    want = -0.5 * sens[0:4] / np.linalg.norm(0.5 * sens[0:4]); want = -want if want[3] < 0 else want
    assert code == 0 and s["n"] == 1 and np.allclose(out[0:4], want, rtol=0, atol=1e-16) and out[4:].tobytes() == sens[4:].tobytes()
    # a non-finite quaternion or gyro: ST_NAN, row and state untouched; a non-finite accelerometer is not read
    for col in (2, 5):
        bad = sens.copy(); bad[col] = np.nan; before = copy.deepcopy(s); keep = bad.copy()
        out, code = f.step(s, 1e-3, bad)
        assert out is None and code == T.ST_NAN and np.array_equal(bad, keep, equal_nan=True)
        assert all(np.array_equal(s[k], before[k]) for k in s)
    bad = sens.copy(); bad[8] = np.inf
    out, code = f.step(s, 1e-3, bad)
    assert code == 0 and out[8] == np.inf and s["n"] == 2


def test_filter_helps_the_state_estimator_on_the_rehearsal(oracle, rehearsal):
    """The reference IMU noise on the rehearsal's plant states, the base state estimator (its twin, default parameters) on the raw readings and on the
    attitude filter's rows: the filtered chain estimates z and the base velocity better.  The velocity gains less: in 0.2 s the filter has not settled
    far below the reading, and the velocity also carries the accelerometer's noise."""
    f = A.AttitudeTwin(); se = T.StateEstTwin(T.default_params(oracle.model_info()["mass"]), oracle)
    s_at = f.reset(); s_raw, s_flt = se.reset(rehearsal[0][1][0:3]), se.reset(rehearsal[0][1][0:3])
    err = {"raw": [], "filtered": []}
    for k, (dt, q, v, v_prev, contact) in enumerate(rehearsal):
        sens = T.read_sensors(q, v, v_prev, dt, k - 1, 0, NOISE)
        row, code = f.step(s_at, dt, sens); assert code == 0
        for tag, st, y in (("raw", s_raw, sens), ("filtered", s_flt, row)):
            rbd, code = se.step(st, dt, y, contact); assert code == 0
            err[tag].append([abs(rbd[5] - q[2]), np.linalg.norm(rbd[27:30] - v[0:3])])
    raw, flt = np.array(err["raw"]), np.array(err["filtered"])
    h = len(raw) // 2; rms = lambda a: np.sqrt(np.mean(a[h:] ** 2, axis=0))
    print("rehearsal with reference noise, RMS over the second half: |z_hat - z| raw %.2e m, filtered %.2e m; |v_hat - v| raw %.3f m/s, filtered %.3f m/s" % (
        rms(raw)[0], rms(flt)[0], rms(raw)[1], rms(flt)[1]))
    ratio = rms(raw) / rms(flt)
    assert ratio[0] > 3.0 and ratio[1] > 1.25, ratio   # measured 3.7x on z (0.66 -> 0.18 mm), 1.4x on v (18 -> 13 mm/s)


def _offsets(tmp_path, struct, fields):
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "qmb200.h"', 'int main(void) {', '  printf("%%zu\\n", sizeof(%s));' % struct]
    body += ['  printf("%%zu\\n", offsetof(%s, %s));' % (struct, f) for f in fields] + ['  return 0; }']
    src = tmp_path / ("%s.c" % struct); src.write_text("\n".join(body) + "\n"); exe = tmp_path / struct
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    return [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]


def test_params_layout_matches_the_header(tmp_path):
    fields = [n for n, _ in _lib.AttitudeParams._fields_]
    out = _offsets(tmp_path, "qmb200_attitude_params", fields)
    assert out[0] == C.sizeof(_lib.AttitudeParams) and out[1:] == [getattr(_lib.AttitudeParams, f).offset for f in fields]
    assert list(A.default_params()) == fields
