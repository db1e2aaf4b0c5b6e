"""CPU twin of the sensor model and the base state estimator (qm_control_b200/csrc/kernels/state_est_kernel.cu) — TEST INFRASTRUCTURE ONLY.

The sensor model and the noise generator are restated in numpy.  The filter takes the legs' kinematics from the oracle's model (orc_rbd at the base
origin: forward-mode differentiation of the frame positions, not the kernel's spatial-vector pass) and is written in dense matrices with
numpy.linalg.solve, where the kernel gathers C P C^T from blocks of P by index and factors it with the warp Cholesky."""
import numpy as np

from _oracle import Oracle

ST_NAN, ST_NOT_PD = 4, 8
G = np.array([0.0, 0.0, -9.81])
NX, NY = 18, 28


def default_params(robot_mass, ground_height=0.0, foot_radius=0.0265, stiffness=1e6):
    """qmb200_state_est_params defaults (include/qmb200.h, DESIGN.md §4.6); foot_height from the default plant params and the model's mass"""
    return dict(process_base_pos=1e-4, process_base_vel=1e-2, process_foot=1e-4, meas_foot_pos=1e-6, meas_foot_vel=1e-2, meas_foot_height=1e-4, swing_scale=1e4,
                foot_height=ground_height + foot_radius - robot_mass * 9.81 / (4.0 * stiffness), p0_base_pos=1e-6, p0_base_vel=1e-4, p0_foot=1e-6)


# ---- the noise generator: splitmix64's finaliser over (seed, robot, sample, channel), Box-Muller ----
def _mix(z):
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
    return z ^ (z >> np.uint64(31))


def normal(seed, robot, sample, channel):
    """N(0, 1) draws, a pure function of the four integers (numpy broadcasting; sample may be negative: it is taken mod 2^64)"""
    def u(a):   # the C cast to uint64_t
        a = np.asarray(a)
        return a.astype(np.uint64) if a.dtype == np.uint64 else a.astype(np.int64).astype(np.uint64)
    h = _mix(_mix(_mix(_mix(u(seed) ^ np.uint64(0x9e3779b97f4a7c15)) ^ u(robot)) ^ u(sample)) ^ u(channel))
    u1 = ((_mix(h) >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    u2 = ((_mix(h ^ np.uint64(0xd1b54a32d192ed03)) >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(6.283185307179586 * u2)


# ---- rotations ----
def rot_zyx(e):
    z, y, x = e; cz, sz, cy, sy, cx, sx = np.cos(z), np.sin(z), np.cos(y), np.sin(y), np.cos(x), np.sin(x)
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1.0]]); Ry = np.array([[cy, 0, sy], [0, 1.0, 0], [-sy, 0, cy]]); Rx = np.array([[1.0, 0, 0], [0, cx, -sx], [0, sx, cx]])
    return Rz @ Ry @ Rx


def euler_rate_map(e):
    z, y = e[0], e[1]
    return np.array([[0.0, -np.sin(z), np.cos(y) * np.cos(z)], [0.0, np.cos(z), np.cos(y) * np.sin(z)], [1.0, 0.0, -np.sin(y)]])


def quat_from_rot(m):
    """xyzw, Shepperd's method with the largest-pivot choice of Eigen"""
    t = np.trace(m)
    if t > 0:
        s = np.sqrt(t + 1.0); w = 0.5 * s; s = 0.5 / s
        return np.array([(m[2, 1] - m[1, 2]) * s, (m[0, 2] - m[2, 0]) * s, (m[1, 0] - m[0, 1]) * s, w])
    i = int(np.argmax(np.diag(m))); j, k = (i + 1) % 3, (i + 2) % 3
    s = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0); o = np.zeros(4); o[i] = 0.5 * s; s = 0.5 / s
    o[3] = (m[k, j] - m[j, k]) * s; o[j] = (m[j, i] + m[i, j]) * s; o[k] = (m[k, i] + m[i, k]) * s
    return o


def rot_from_quat(qt):
    x, y, z, w = np.asarray(qt) / np.linalg.norm(qt)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def zyx_from_rot(R):
    return np.array([np.arctan2(R[1, 0], R[0, 0]), np.arcsin(np.clip(-R[2, 0], -1.0, 1.0)), np.arctan2(R[2, 1], R[2, 2])])


def expm_so3(n):
    th = np.linalg.norm(n)
    if th == 0.0:
        return np.eye(3)
    K = np.array([[0, -n[2], n[1]], [n[2], 0, -n[0]], [-n[1], n[0], 0]]) / th
    return np.eye(3) + np.sin(th) * K + (1.0 - np.cos(th)) * K @ K


# ---- the sensor model ----
def read_sensors(q, v, v_prev, dt, sample, robot, params):
    """qmb200_sim_read_sensors of one robot: [quat xyzw, gyro, accel, joint pos, joint vel]; params: qmb200_sensor_params as a dict"""
    p = params; R = rot_zyx(q[3:6]); om = euler_rate_map(q[3:6]) @ v[3:6]
    nz = lambda ch, sigma: sigma * normal(p["seed"], robot, sample, ch) if sigma > 0 else 0.0
    gyro = R.T @ om + np.array([nz(3 + i, p["sigma_gyro"]) for i in range(3)])
    accel = R.T @ ((v[0:3] - v_prev[0:3]) / dt - G) + np.array([nz(6 + i, p["sigma_accel"]) for i in range(3)])
    if p["sigma_orientation"] > 0:
        R = R @ expm_so3(np.array([nz(i, p["sigma_orientation"]) for i in range(3)]))
    return np.r_[quat_from_rot(R), gyro, accel, q[6:24] + np.array([nz(9 + j, p["sigma_joint_pos"]) for j in range(18)]),
                 v[6:24] + np.array([nz(27 + j, p["sigma_joint_vel"]) for j in range(18)])]


NOISE_OFF = dict(seed=0, sigma_orientation=0.0, sigma_gyro=0.0, sigma_accel=0.0, sigma_joint_pos=0.0, sigma_joint_vel=0.0)


def _measurement_matrix():
    C = np.zeros((NY, NX))
    for i in range(4):
        for k in range(3):
            C[3 * i + k, k] = 1.0; C[3 * i + k, 6 + 3 * i + k] = -1.0   # p - p_foot_i
            C[12 + 3 * i + k, 3 + k] = 1.0                              # v
        C[24 + i, 6 + 3 * i + 2] = 1.0                                  # p_foot_i,z
    return C


class StateEstTwin:
    """The filter of one robot per state dict (reset → step ...), as state_est_step_kernel."""

    C = _measurement_matrix()

    def __init__(self, params, oracle=None):
        self.p = dict(params); self.oracle = oracle or Oracle()

    def reset(self, base_pos):
        p = self.p
        return dict(x=np.r_[base_pos, np.zeros(15)], P=np.diag([p["p0_base_pos"]] * 3 + [p["p0_base_vel"]] * 3 + [p["p0_foot"]] * 12), n=0)

    def legs(self, sensors):
        """attitude and leg kinematics of one reading → (zyx, w_world, a_world, r[4, 3], rd[4, 3], ee_pos_rel, ee_rot)"""
        R = rot_from_quat(sensors[0:4]); e = zyx_from_rot(R); om = R @ sensors[4:7]; a = R @ sensors[7:10] + G
        ed = np.linalg.solve(euler_rate_map(e), om)
        o = self.oracle.rbd(np.r_[0.0, 0.0, 0.0, e, sensors[10:28]], np.r_[0.0, 0.0, 0.0, ed, sensors[28:46]])
        return e, om, a, o["foot_pos"], o["foot_vel"], o["ee_pos"], o["ee_rot"]

    def step(self, s, dt, sensors, contact):
        """one kernel call on the state dict s (updated in place) → (rbd_est [55] or None for a non-finite input, status)"""
        if not np.all(np.isfinite(sensors)):
            return None, ST_NAN
        p = self.p; e, om, a, r, rd, ee_p, ee_R = self.legs(sensors)
        stance = np.array([(contact >> (3 - i)) & 1 for i in range(4)], dtype=bool)
        code = 0
        if s["n"] == 0:
            s["x"] = s["x"].copy(); s["x"][6:] = (s["x"][0:3] + r).ravel()
        else:
            A = np.eye(NX); A[0:3, 3:6] = dt * np.eye(3)
            q = np.r_[[p["process_base_pos"]] * 3, [p["process_base_vel"]] * 3, np.repeat(np.where(stance, 1.0, p["swing_scale"]) * p["process_foot"], 3)]
            x = A @ s["x"] + np.r_[0.5 * dt * dt * a, dt * a, np.zeros(12)]
            P = A @ s["P"] @ A.T + dt * np.diag(q)
            y = np.r_[-r.ravel(), -rd.ravel(), np.full(4, p["foot_height"])]
            sc = np.where(stance, 1.0, p["swing_scale"])
            Rm = np.diag(np.r_[np.repeat(sc, 3) * p["meas_foot_pos"], np.repeat(sc, 3) * p["meas_foot_vel"], sc * p["meas_foot_height"]])
            S = self.C @ P @ self.C.T + Rm
            if np.any(np.linalg.eigvalsh(S) <= 0):
                code = ST_NOT_PD
            else:
                K = np.linalg.solve(S, self.C @ P).T
                x_new = x + K @ (y - self.C @ x)
                P_new = P - K @ self.C @ P; P_new = 0.5 * (P_new + P_new.T)
                if np.all(np.isfinite(x_new)) and np.all(np.isfinite(P_new)):
                    s["x"], s["P"] = x_new, P_new
                else:
                    code = ST_NAN
        s["n"] += 1
        x = s["x"]
        rbd = np.r_[e, x[0:3], sensors[10:28], om, x[3:6], sensors[28:46], x[0:3] + ee_p, quat_from_rot(ee_R)]
        return rbd, code
