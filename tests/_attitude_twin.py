"""CPU twin of the attitude filter (qm_control_b200/csrc/kernels/attitude_kernel.cu) — TEST INFRASTRUCTURE ONLY.

The filter of one robot in dense 6x6 matrices with numpy.linalg.solve, where the kernel keeps P as a packed triangle in registers, forms F P F^T from
F's blocks and inverts the 3x3 S by its adjugate.  Rotations come from tests/_state_est_twin.py."""
import numpy as np

from _state_est_twin import ST_NAN, rot_from_quat

NX = 6


def default_params():
    """qmb200_attitude_params defaults (include/qmb200.h, DESIGN.md §4.6)"""
    return dict(process_attitude=4e-7, process_gyro_bias=1e-8, meas_orientation=1.2e-3, p0_attitude=1.2e-3, p0_gyro_bias=1e-4)


# ---- unit quaternions, xyzw ----
def qmul(a, b):
    return np.array([a[3] * b[0] + b[3] * a[0] + (a[1] * b[2] - a[2] * b[1]), a[3] * b[1] + b[3] * a[1] + (a[2] * b[0] - a[0] * b[2]),
                     a[3] * b[2] + b[3] * a[2] + (a[0] * b[1] - a[1] * b[0]), a[3] * b[3] - (a[0] * b[0] + a[1] * b[1] + a[2] * b[2])])


def qconj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def qexp(v):
    """[v sin(|v|/2) / |v|, cos(|v|/2)]"""
    th = np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    if th == 0.0:
        return np.array([0.0, 0.0, 0.0, 1.0])
    f = np.sin(0.5 * th) / th
    return np.array([v[0] * f, v[1] * f, v[2] * f, np.cos(0.5 * th)])


def qlog(q):
    """v 2 atan2(|v|, w) / |v| (q with w >= 0)"""
    n = np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2])
    return q[0:3] * (2.0 * np.arctan2(n, q[3]) / n if n > 0.0 else 0.0)


def angle_between(qa, qb):
    """the angle of the rotation from qa to qb (either sign of either), rad"""
    d = qmul(qconj(qa), qb)
    return 2.0 * np.arctan2(np.linalg.norm(d[0:3]), abs(d[3]))


class AttitudeTwin:
    """The filter of one robot per state dict (reset → step ...), as attitude_step_kernel."""

    def __init__(self, params=None):
        self.p = dict(default_params() if params is None else params)

    def reset(self):
        p = self.p
        return dict(q=np.array([0.0, 0.0, 0.0, 1.0]), b=np.zeros(3), P=np.diag([p["p0_attitude"]] * 3 + [p["p0_gyro_bias"]] * 3), n=0)

    def step(self, s, dt, sensors):
        """one kernel call on the state dict s (updated in place) → (the rewritten sensor row [46], or None for a non-finite input, status)"""
        sensors = np.asarray(sensors, dtype=np.float64); qm, gy = sensors[0:4], sensors[4:7]
        if not (np.all(np.isfinite(qm)) and np.all(np.isfinite(gy))):
            return None, ST_NAN
        p = self.p; code = 0
        if s["n"] == 0:
            s["q"] = qm / np.sqrt(np.sum(qm * qm))
        else:
            dq = qexp((gy - s["b"]) * dt); qp = qmul(s["q"], dq)
            F = np.eye(NX); F[0:3, 0:3] = rot_from_quat(dq).T; F[0:3, 3:6] = -dt * np.eye(3)
            P = F @ s["P"] @ F.T + dt * np.diag([p["process_attitude"]] * 3 + [p["process_gyro_bias"]] * 3)
            dm = qmul(qconj(qp), qm)
            if dm[3] < 0.0:
                dm = -dm
            r = qlog(dm)
            S = P[0:3, 0:3] + p["meas_orientation"] * np.eye(3)
            K = np.linalg.solve(S, P[0:3, :]).T   # P H^T S^-1, S symmetric
            dx = K @ r
            qn = qmul(qp, qexp(dx[0:3])); qn = qn / np.sqrt(np.sum(qn * qn))
            bn = s["b"] + dx[3:6]
            Pn = P - K @ P[0:3, :]; Pn = 0.5 * (Pn + Pn.T)
            if np.all(np.isfinite(qn)) and np.all(np.isfinite(bn)) and np.all(np.isfinite(Pn)):
                s["q"], s["b"], s["P"] = qn, bn, Pn
            else:
                code = ST_NAN
        s["n"] += 1
        out = sensors.copy(); q = s["q"]
        out[0:4] = -q if q[3] < 0.0 else q
        out[4:7] = gy - s["b"]
        return out, code
