"""numpy statement of the per-episode metrics (include/qmb200.h: qmb200_metrics_*; DESIGN.md §4.13) — TEST INFRASTRUCTURE ONLY.

It follows the header's column table and accumulator layout call by call: step() adds one sample of every robot to a copy of the accumulator rows, close()
closes the masked robots' episodes.  Nothing comes from the product's kinematics or interpolation: the foot frames are the oracle's (Oracle.rbd), the
ground is a bilinear lookup written here, the target's end-effector pose is a linear interpolation and a slerp written here, the angle comes from a
Hamilton product."""
import numpy as np

RBD, KMAX, TARGET, METRICS, ACC = 55, 4, 37, 18, 32
ST_OVERFLOW, CMD_VEL = 2, 0
# accumulator columns (include/qmb200.h)
N, DUR, STATUS, X0, Y0, X, Y, FEET, CONTACT, PATH, MIN_H, MAX_TILT, N_CMD, VEL_SQ, YAW_SQ, EE_SQ, EE_MAX, ORI_SQ, ENERGY, TAU_SQ, SLIP, TOUCH, N_EST, \
    EST_P, EST_V = 0, 1, 2, 3, 4, 5, 6, 7, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31


def ground(tiles, cell, row, ground_height, x, y):
    """the plant's ground height at world (x, y) under terrain row [tile, ox, oy] (None or tile -1: the plane): bilinear inside the tile, the border outside"""
    if row is None or int(row[0]) < 0:
        return ground_height
    h = tiles[int(row[0])]; ny, nx = h.shape
    u = min(max((x - row[1]) / cell, 0.0), nx - 1.0); v = min(max((y - row[2]) / cell, 0.0), ny - 1.0)
    i = min(int(np.floor(u)), nx - 2); j = min(int(np.floor(v)), ny - 2); fx = u - i; fy = v - j
    return (1 - fx) * (1 - fy) * h[j, i] + fx * (1 - fy) * h[j, i + 1] + (1 - fx) * fy * h[j + 1, i] + fx * fy * h[j + 1, i + 1]


def slerp(q0, q1, s):
    """Eigen's Quaternion::slerp from q0 towards q1 by the fraction s (the shorter arc; the linear blend when the two nearly coincide)"""
    d = float(np.dot(q0, q1))
    if abs(d) >= 1.0 - np.finfo(float).eps:
        w0, w1 = 1.0 - s, s
    else:
        th = np.arccos(abs(d)); w0, w1 = np.sin((1.0 - s) * th) / np.sin(th), np.sin(s * th) / np.sin(th)
    return w0 * q0 + (w1 if d >= 0 else -w1) * q1


def target_ee(n, times, states, t):
    """the end-effector pose (p [3], q xyzw [4]) of a target of n knots (clamped to [1, KMAX]) at time t: t held within the knots' times, then between
    knots t_i < t <= t_i+1 (t_0 <= t on the first) the blend from knot i towards knot i+1 by (t - t_i) / (t_i+1 - t_i)"""
    n = min(max(int(n), 1), KMAX); p = states[:n, 30:33]; q = states[:n, 33:37]
    if n == 1:
        return p[0].copy(), q[0].copy()
    t = min(max(t, times[0]), times[n - 1])
    i = min(max(int(np.searchsorted(times[:n], t, side="left")) - 1, 0), n - 2)
    s = (t - times[i]) / (times[i + 1] - times[i])
    return (1.0 - s) * p[i] + s * p[i + 1], slerp(q[i], q[i + 1], s)


def qmul(a, b):
    """Hamilton product of quaternions a, b in xyzw order"""
    av, aw, bv, bw = a[:3], a[3], b[:3], b[3]
    return np.r_[aw * bv + bw * av + np.cross(av, bv), aw * bw - av @ bv]


class MetricsTwin:
    """oracle: an Oracle (tests/_oracle.py) for the foot frames; tiles [T, ny, nx], cell: the plant's tile library (None: none)"""

    def __init__(self, oracle, tiles=None, cell=None, ground_height=0.0):
        self.oracle, self.tiles, self.cell, self.ground_height = oracle, tiles, cell, float(ground_height)

    def feet(self, r):
        q = np.r_[r[3:6], r[0:3], r[6:24]]
        return self.oracle.rbd(q, np.zeros(24))["foot_pos"]

    def sample(self, a, dt, r, contact, tau, cmd, cmd_vel, n, times, states, t, status, est, row):
        """one robot's accumulator row a [ACC] after one sample → the new row"""
        a = a.copy(); first = a[N] == 0
        a[N] += 1; a[DUR] += dt; a[STATUS] = float(int(a[STATUS]) | (int(status) & 0xFFFFFFFF))
        h = r[5] - ground(self.tiles, self.cell, row, self.ground_height, r[3], r[4]); tilt = max(abs(r[1]), abs(r[2]))
        if first:
            a[X0:Y0 + 1] = r[3:5]; a[MIN_H] = h; a[MAX_TILT] = tilt
        else:
            a[PATH] += np.hypot(r[3] - a[X], r[4] - a[Y]); a[MIN_H] = np.fmin(a[MIN_H], h); a[MAX_TILT] = np.fmax(a[MAX_TILT], tilt)
        a[X:Y + 1] = r[3:5]
        feet = self.feet(r)[:, :2]; prev, now = int(a[CONTACT]), int(contact) & 15
        bit = lambda m, f: (m >> (3 - f)) & 1   # foot f (contact order LF, RF, LH, RH) is bit 3 - f
        if not first:
            last = a[FEET:FEET + 8].reshape(4, 2)
            a[SLIP] += sum(np.hypot(*(feet[f] - last[f])) for f in range(4) if bit(prev, f) and bit(now, f))
            a[TOUCH] += bin(now & ~prev & 15).count("1")
        a[FEET:FEET + 8] = feet.ravel(); a[CONTACT] = now
        if cmd_vel:
            a[N_CMD] += 1; a[VEL_SQ] += (r[27] - states[0, 0]) ** 2 + (r[28] - states[0, 1]) ** 2; a[YAW_SQ] += (r[26] - cmd[3]) ** 2
        p, q = target_ee(n, times, states, t)
        e = np.linalg.norm(r[48:51] - p); a[EE_SQ] += e * e; a[EE_MAX] = e if first else np.fmax(a[EE_MAX], e)
        rel = qmul(np.r_[-q[:3], q[3]], r[51:55]); ang = 2.0 * np.arctan2(np.linalg.norm(rel[:3]), abs(rel[3])); a[ORI_SQ] += ang * ang
        a[ENERGY] += np.sum(np.abs(tau * r[30:48])) * dt; a[TAU_SQ] += np.sum(tau * tau) / 18.0
        if est is not None:
            a[N_EST] += 1; a[EST_P] += np.sum((est[3:6] - r[3:6]) ** 2); a[EST_V] += np.sum((est[27:30] - r[27:30]) ** 2)
        return a

    def step(self, acc, dt, rbd, contact, effort, cmd, n_target, target_times, target_states, time, status, kind=None, rbd_est=None, terrain_rows=None):
        """qmb200_metrics_step on copies: every robot's sample at time + dt → the accumulator rows [B, ACC]"""
        out = np.array(acc, dtype=np.float64, copy=True)
        for b in range(len(out)):
            out[b] = self.sample(out[b], dt, rbd[b], contact[b], effort[b], cmd[b], kind is None or kind[b] == CMD_VEL, n_target[b], target_times[b],
                                 target_states[b], time[b] + dt, status[b], None if rbd_est is None else rbd_est[b],
                                 None if terrain_rows is None else terrain_rows[b])
        return out


def finish(a, end):
    """the row [METRICS] of an accumulator row"""
    n, nc, ne = a[N], a[N_CMD], a[N_EST]
    rms = lambda s, c: np.sqrt(s / c) if c > 0 else np.nan
    some = lambda v: v if n > 0 else np.nan
    return np.array([a[DUR], end, a[STATUS], some(np.hypot(a[X] - a[X0], a[Y] - a[Y0])), a[PATH], some(a[MIN_H]), some(a[MAX_TILT]), rms(a[VEL_SQ], nc),
                     rms(a[YAW_SQ], nc), rms(a[EE_SQ], n), some(a[EE_MAX]), rms(a[ORI_SQ], n), a[ENERGY], rms(a[TAU_SQ], n), a[SLIP], a[TOUCH],
                     rms(a[EST_P], ne), rms(a[EST_V], ne)])


def close(mask, end, episode, acc, out, status):
    """qmb200_metrics_close's device semantics on copies → (acc, out [B, E, METRICS], status)"""
    acc = np.array(acc, dtype=np.float64, copy=True); out = np.array(out, dtype=np.float64, copy=True); status = np.array(status, dtype=np.int32, copy=True)
    for b in np.nonzero(mask)[0]:
        if not 0 <= end[b] <= 2:
            continue
        if 0 <= episode[b] < out.shape[1]:
            out[b, episode[b]] = finish(acc[b], end[b])
        else:
            status[b] |= ST_OVERFLOW
        acc[b] = 0.0
    return acc, out, status
