"""The sensor model and the base state estimator on the host, no GPU: the sensor identities on plant-twin trajectories, free fall, the noise generator,
the filter on the CPU rehearsal of a trotting closed loop, and the parameter structs' layouts against include/qmb200.h."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _closed_loop_cpu
import _loop_replay as R
import _state_est_twin as T
from _oracle import Oracle
from _sim_twin import SimTwin
from qm_control_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def _wrap(a):
    return (a + np.pi) % (2 * np.pi) - np.pi


def _trajectory(oracle, steps=40, seed=3):
    """plant-twin steps of 1 ms from the standing state with random efforts: [(q, v, v_prev, rbd)]"""
    twin = SimTwin(); rng = np.random.default_rng(seed)
    q, v = _closed_loop_cpu.standing_state(oracle, twin, yaw=2.5)
    out = []
    for _ in range(steps):
        q1, v1, rbd, _, _ = twin.step(1e-3, rng.uniform(-30, 30, 18), q, v)
        out.append((q1, v1, v, rbd)); q, v = q1, v1
    return out


def test_sensor_identities_on_the_plant_twin(oracle):
    """Noise off: gyro = R^T w_world of the twin's rbd, the quaternion gives back the plant's zyx, accel = R^T (dv/dt - g), the encoders are q, v."""
    for q, v, v_prev, rbd in _trajectory(oracle):
        s = T.read_sensors(q, v, v_prev, 1e-3, 0, 0, T.NOISE_OFF)
        R = T.rot_zyx(rbd[0:3])
        np.testing.assert_allclose(s[4:7], R.T @ rbd[24:27], rtol=0, atol=1e-13)
        e = T.zyx_from_rot(T.rot_from_quat(s[0:4]))
        assert np.max(np.abs(_wrap(e - rbd[0:3]))) < 1e-15 * 4, e - rbd[0:3]
        np.testing.assert_allclose(s[7:10], R.T @ ((rbd[27:30] - v_prev[0:3]) / 1e-3 - T.G), rtol=0, atol=1e-9)
        assert s[10:28].tobytes() == rbd[6:24].tobytes() and s[28:46].tobytes() == rbd[30:48].tobytes()


def test_free_fall_reads_zero_specific_force(oracle):
    """A robot dropped from 1 m above the plane with zero effort: no foot touches and the accelerometer reads 0 to 1e-9 in every step."""
    twin = SimTwin()
    q, v = _closed_loop_cpu.standing_state(oracle, twin, yaw=0.7); q[2] += 1.0
    for _ in range(50):
        q1, v1, rbd, contact, st = twin.step(1e-3, np.zeros(18), q, v)
        assert contact == 0 and st == 0
        s = T.read_sensors(q1, v1, v, 1e-3, 0, 0, T.NOISE_OFF)
        assert np.max(np.abs(s[7:10])) < 1e-9, s[7:10]
        q, v = q1, v1
    assert v[2] < -0.4   # it did fall


def test_noise_generator():
    """Deterministic in (seed, robot, sample, channel); independent of the batch; N(0, 1) over 1e5 draws; another seed gives other draws."""
    n = 100000; k = np.arange(n)
    a = T.normal(7, k % 64, k // 64, k % 45); b = T.normal(7, k % 64, k // 64, k % 45)
    assert a.tobytes() == b.tobytes()
    assert abs(a.mean()) < 4 / np.sqrt(n) and abs(a.std() - 1.0) < 4 / np.sqrt(2 * n)
    assert np.mean(T.normal(8, k % 64, k // 64, k % 45) == a) < 1e-3
    # robot 5's reading in a batch of 1 and in a batch of 64: the same function of its index, whatever else is drawn
    p = dict(T.NOISE_OFF, seed=123, sigma_orientation=0.03, sigma_gyro=0.02, sigma_accel=0.1, sigma_joint_pos=1e-3, sigma_joint_vel=1e-2)
    q = np.r_[0, 0, 0.45, 0.3, 0.05, -0.02, np.zeros(18)]; v = np.r_[np.zeros(3), 0.1, 0.0, 0.0, np.zeros(18)]
    alone = T.read_sensors(q, v, v, 1e-3, 9, 5, p)
    batch = [T.read_sensors(q, v, v, 1e-3, 9, r, p) for r in range(64)]
    assert batch[5].tobytes() == alone.tobytes() and not np.array_equal(batch[4], alone)
    ch = np.arange(45)
    assert np.array_equal(T.normal(123, 5, 9, ch), T.normal(123, np.full(45, 5), np.full(45, 9), ch))
    assert np.all(np.isfinite(T.normal(0, 0, -1, ch)))   # the reading of the start (sample -1)


@pytest.fixture(scope="module")
def rehearsal(oracle):
    """the plant steps of a 0.2 s trot at 0.3 m/s of the CPU rehearsal: [(duration, q, v, v_prev, contact)]"""
    from qm_control_b200.interface import gait_schedule
    rec = R.Record(); sched = gait_schedule("trot", 10.0, 9.998, 12.2)
    _closed_loop_cpu.run(oracle, duration=0.2, cmd_vel=(0.3, 0.0, 0.0, 0.0), t_start=10.0, mode_schedule=sched, recorder=rec)
    return [(i["duration"], o["q"][0], o["v"][0], i["v"][0], int(o["contact"][0])) for i, o in rec.of("sim")]


def test_filter_tracks_the_rehearsal(oracle, rehearsal):
    """Noise off, default parameters (the model's mass from the oracle): P stays symmetric positive definite, z and v track the plant, the xy variance
    grows (unobservable) while the z and velocity variances stay bounded."""
    f = T.StateEstTwin(T.default_params(oracle.model_info()["mass"]), oracle)
    s = f.reset(rehearsal[0][1][0:3]); dz, dv, pd = [], [], []
    modes = set()
    for k, (dt, q, v, v_prev, contact) in enumerate(rehearsal):
        sens = T.read_sensors(q, v, v_prev, dt, k - 1, 0, T.NOISE_OFF)
        rbd, code = f.step(s, dt, sens, contact)
        assert code == 0, k
        P = s["P"]; assert np.array_equal(P, P.T) and np.linalg.eigvalsh(P).min() > 0, k
        dz.append(abs(rbd[5] - q[2])); dv.append(np.max(np.abs(rbd[27:30] - v[0:3]))); pd.append(np.diag(P).copy()); modes.add(contact)
    dz, dv, pd = np.array(dz), np.array(dv), np.array(pd)
    print("rehearsal, 0.2 s trot: max |z_hat - z| %.2e m, max |v_hat - v| %.2e m/s, diag P xy %.1e -> %.1e, z %.1e, v %.1e" % (
        dz.max(), dv.max(), pd[1, 0], pd[-1, 0], pd[-1, 2], pd[-1, 3:6].max()))
    assert len(modes) > 1, "the trot must change contacts"
    assert dz.max() < 2e-3 and dv[50:].max() < 0.05
    assert pd[-1, 0] > 1.5 * pd[1, 0] and pd[-1, 1] > 1.5 * pd[1, 1]
    assert pd[:, 2].max() < 1e-5 and pd[:, 3:6].max() < 1e-3


def _offsets(tmp_path, struct, fields):
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "qmb200.h"', 'int main(void) {', '  printf("%%zu %%d\\n", sizeof(%s), QMB200_SENSORS);' % struct]
    body += ['  printf("%%zu\\n", offsetof(%s, %s));' % (struct, f) for f in fields] + ['  return 0; }']
    src = tmp_path / ("%s.c" % struct); src.write_text("\n".join(body) + "\n"); exe = tmp_path / struct
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    return [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]


@pytest.mark.parametrize("struct, mirror", [("qmb200_sensor_params", _lib.SensorParams), ("qmb200_state_est_params", _lib.StateEstParams)])
def test_params_layout_matches_the_header(tmp_path, struct, mirror):
    fields = [n for n, _ in mirror._fields_]
    out = _offsets(tmp_path, struct, fields)
    assert out[0] == C.sizeof(mirror) and out[1] == _lib.SENSORS == len(_lib.SENSOR_LAYOUT) and out[2:] == [getattr(mirror, f).offset for f in fields]
    assert len(_lib.STATE_EST_LAYOUT) == 18
