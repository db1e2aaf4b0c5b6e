"""WBC inputs where the inequalities of the HoQp cascade bind, shared by tests/test_wbc_inequalities_cpu.py and tests/test_wbc_inequalities_gpu.py.

Every regime starts from the config-3 stance batch of synthetic.make_batch and changes what it is about:
  fast       the measured base and joint velocities x20 (base up to 2 m/s and 2 rad/s, joints up to 4 rad/s), every contact mask.  The contact rows'
             bias accelerations then ask for forces and torques outside the pyramids and limits: up to 11 violated rows at the minimum-norm
             level-0 point and 14 at a later pass, more than the 6 that fit beside the 18 task rows in a buffer of 24;
  edge       desired tangential forces at 1.5 mu Fz, with the robot's own pyramid coefficient mu in {0.15, 0.3, 0.6};
  apex       one stance foot whose desired normal force is 0 or negative (touchdown, lift-off): its five pyramid rows all meet at F = 0 and are
             linearly dependent;
  saturated  arm joints 1.2 rad from their targets (the end-effector task at kp 2500 asks for more than the arm's effort limits) and swing legs
             0.4 rad from theirs;
  init_*     fast, edge and apex at t = 3 s: HierarchicalWbc's arm joint tracking branch (t < 10).
A level 0 that needs slack (optimal v* > 0) was searched for with the oracle on the fast states at up to x40 and not found: the contact rows can always be
met inside the limits for this model, so there is no such regime."""
import os

import numpy as np

from _tuning import _set_block_key
from qm_control_b200 import _lib, synthetic

REGIMES = ("fast", "edge", "apex", "saturated", "init_fast", "init_edge", "init_apex")
FAST_SCALE = 20.0
MUS = (0.15, 0.3, 0.6)


def _flags(mode):
    return [(int(mode) >> (3 - f)) & 1 for f in range(4)]


def _base(n, seed_offset, mass):
    ids = np.arange(seed_offset, seed_offset + n); prob, wbc = synthetic.make_batch(ids, config=3)
    x_des = prob["x0"].copy(); rbd = wbc["rbd"].copy()
    u_des = synthetic.uniform(77, ids, 1, 30, -1.0, 1.0) * np.r_[np.full(12, 5.0), np.full(18, 0.2)]
    il = synthetic.uniform(78, ids, 2, 30, -0.1, 0.1)
    return ids, x_des, u_des, rbd, wbc["period"].copy(), il


def _weight(u_des, mode, mass, skip=()):
    for b in range(len(mode)):
        fl = _flags(mode[b]); feet = [f for f in range(4) if fl[f] and f not in skip]
        for f in range(4):
            if not fl[f]:
                u_des[b, 3 * f:3 * f + 3] = 0.0
            elif f in feet:
                u_des[b, 3 * f + 2] += mass * 9.81 / len(feet)


def regime(name, mass):
    """→ dict(x_des, u_des, rbd, mode, period, time, input_last, wbc_friction) for one regime's robots"""
    kind = name[5:] if name.startswith("init_") else name; time = 3.0 if name.startswith("init_") else 12.0
    off = 1000 * (1 + REGIMES.index(name))
    if kind == "fast":
        n = 48; ids, x_des, u_des, rbd, period, il = _base(n, off, mass)
        mode = (np.arange(n) % 16).astype(np.int32); rbd[:, 24:48] *= FAST_SCALE; _weight(u_des, mode, mass); mu = np.full(n, 0.3)
    elif kind == "edge":
        n = 24; ids, x_des, u_des, rbd, period, il = _base(n, off, mass)
        mode = np.array([(15, 14, 7, 11, 13, 15)[i % 6] for i in range(n)], dtype=np.int32)
        mu = np.array([MUS[i % 3] for i in range(n)]); u_des[:, :12] = 0.0; _weight(u_des, mode, mass)
        th = synthetic.uniform(79, ids, 3, 4, -np.pi, np.pi)
        for b in range(n):
            for f in range(4):
                if _flags(mode[b])[f]:
                    ft = 1.5 * mu[b] * u_des[b, 3 * f + 2]; u_des[b, 3 * f] = ft * np.cos(th[b, f]); u_des[b, 3 * f + 1] = ft * np.sin(th[b, f])
    elif kind == "apex":
        n = 16; ids, x_des, u_des, rbd, period, il = _base(n, off, mass)
        mode = np.array([(15, 15, 14, 7)[i % 4] for i in range(n)], dtype=np.int32); mu = np.full(n, 0.3); u_des[:, :12] = 0.0
        for b in range(n):
            fl = _flags(mode[b]); apex = [f for f in range(4) if fl[f]][b % 3]
            _weight(u_des[b:b + 1], mode[b:b + 1], mass, skip=(apex,))
            u_des[b, 3 * apex + 2] = (0.0, -20.0)[(b // 3) % 2]                          # touchdown: 0; lift-off pull: negative
    elif kind == "saturated":
        n = 16; ids, x_des, u_des, rbd, period, il = _base(n, off, mass)
        mode = np.array([(15, 6, 9, 14, 7, 15, 11, 13)[i % 8] for i in range(n)], dtype=np.int32); mu = np.full(n, 0.3); _weight(u_des, mode, mass)
        sgn = np.where(synthetic.uniform(80, ids, 4, 18, -1.0, 1.0) > 0, 1.0, -1.0)
        x_des[:, 24:30] = rbd[:, 18:24] + 1.2 * sgn[:, 12:]                              # arm targets far from the measured arm
        x_des[:, 12:24] = rbd[:, 6:18] + 0.4 * sgn[:, :12]                               # leg targets far from the measured legs (swing error)
    else:
        raise ValueError(name)
    return dict(x_des=x_des, u_des=u_des, rbd=rbd, mode=mode, period=period, time=np.full(len(mode), time), input_last=il, wbc_friction=mu)


def batch(mass, names=REGIMES):
    """every regime in one batch → (dict of stacked inputs, regime name per robot)"""
    parts = [regime(n, mass) for n in names]
    out = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    return out, np.concatenate([[n] * len(p["mode"]) for n, p in zip(names, parts)])


class Oracles:
    """one CPU oracle per pyramid coefficient: task.info with frictionConeTask.frictionCoefficient edited to mu"""
    def __init__(self, directory):
        self.dir = str(directory); self.by_mu = {}

    def __call__(self, mu):
        from _oracle import Oracle
        mu = float(mu)
        if mu not in self.by_mu:
            text = _set_block_key(open(_lib.asset("qm_task.info")).read(), "frictionConeTask", "frictionCoefficient", mu)
            path = os.path.join(self.dir, "task_mu_%g.info" % mu); open(path, "w").write(text)
            self.by_mu[mu] = Oracle(task=path)
        return self.by_mu[mu]

    def wbc_update(self, r, variant=0):
        """the oracle's commands for a regime dict, robot by robot on the oracle of its mu"""
        B = len(r["mode"]); cmd = np.zeros((B, 54))
        for mu in np.unique(r["wbc_friction"]):
            sel = np.nonzero(r["wbc_friction"] == mu)[0]
            cmd[sel], _ = self(mu).wbc_update_batch(r["x_des"][sel], r["u_des"][sel], r["rbd"][sel], r["mode"][sel], r["period"][sel], r["time"][sel],
                                                    r["input_last"][sel], variant=variant, nthreads=8)
        return cmd


def level0_passes(A0, b0, D0, f0, cap=30):
    """numpy statement of the kernel's level-0 rule: minimum-norm least squares on the task rows plus the violated set V, V updated to the strictly
    violated rows plus the rows of V on their boundary, until V repeats → (x0, list of |V| per pass, number of violated rows at the minimum-norm point,
    list of the rank of each pass's rows)"""
    nin = len(D0); V = np.zeros(nin, dtype=bool); sizes = []; ranks = []
    for _ in range(cap):
        sizes.append(int(V.sum()))
        A = np.r_[A0, D0[V]]; b = np.r_[b0, f0[V]]
        x, _, rank, _ = np.linalg.lstsq(A, b, rcond=1e-11); ranks.append(int(rank))
        val = D0 @ x - f0; sc = 1e-9 * (1.0 + np.abs(f0))
        nV = (val > sc) | (V & (val >= -sc))
        if np.array_equal(nV, V):
            break
        V = nV
    return x, sizes, sizes[1] if len(sizes) > 1 else 0, ranks
