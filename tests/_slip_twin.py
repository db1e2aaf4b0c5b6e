"""CPU twin of the slip detector (slip_step_kernel, qm_control_b200/csrc/kernels/state_est_kernel.cu) — TEST INFRASTRUCTURE ONLY.

The test of one robot on the estimator twin's state dict (tests/_state_est_twin.py): the legs from StateEstTwin.legs, the 3x3 system solved with
numpy.linalg.solve where the kernel inverts it by its adjugate."""
import numpy as np

from _state_est_twin import ST_NAN  # noqa: F401 (re-exported for the tests)


def default_params():
    """qmb200_slip_params defaults (include/qmb200.h, DESIGN.md §4.6)"""
    return dict(gate=16.27, release=7.81, meas_slip=2.5e-3, hold=5)


def stance_flags(mask):
    """contact bit order: foot f at bit 3 - f"""
    return np.array([(int(mask) >> (3 - f)) & 1 for f in range(4)], dtype=bool)


def to_mask(flags):
    return int(sum(1 << (3 - f) for f in range(4) if flags[f]))


class SlipTwin:
    """The detector of one robot per state dict (reset → step ...), as slip_step_kernel; se: the estimator twin (StateEstTwin) whose legs and
    process_base_vel it uses."""

    def __init__(self, se, params=None):
        self.se = se; self.p = dict(default_params() if params is None else params)

    def reset(self):
        return dict(mask=0, hold=np.zeros(4, dtype=int), onsets=np.zeros(4, dtype=int))

    def d2(self, se_state, dt, sensors):
        """d^2 of every foot (in contact or not) against the prior of the estimator state se_state → [4]"""
        _, _, a, _, rd, _, _ = self.se.legs(sensors)
        v = se_state["x"][3:6] + a * dt
        S = se_state["P"][3:6, 3:6] + (dt * self.se.p["process_base_vel"] + self.p["meas_slip"]) * np.eye(3)
        u = v[None, :] + rd
        return np.einsum("fi,fi->f", u, np.linalg.solve(S, u.T).T)

    def step(self, s, se_state, dt, sensors, contact):
        """one kernel call on the state dict s (updated in place) → (stance, slip, status, d2 [4] or None where the contact mask passed through)"""
        if not np.all(np.isfinite(sensors)):
            return int(contact), 0, ST_NAN, None
        if se_state["n"] == 0:
            return int(contact), 0, 0, None
        d2 = self.d2(se_state, dt, sensors); p = self.p
        inc = stance_flags(contact); sl = stance_flags(s["mask"])
        if np.any(inc & ~np.isfinite(d2)):
            return int(contact), 0, ST_NAN, d2
        for f in range(4):
            if not inc[f]:
                sl[f] = False; s["hold"][f] = 0
            elif sl[f]:
                if d2[f] < p["release"]:
                    s["hold"][f] += 1
                    if s["hold"][f] >= p["hold"]:
                        sl[f] = False; s["hold"][f] = 0
                else:
                    s["hold"][f] = 0
            elif d2[f] > p["gate"]:
                sl[f] = True; s["hold"][f] = 0; s["onsets"][f] += 1
        s["mask"] = to_mask(sl)
        return int(contact) & ~s["mask"], s["mask"], 0, d2

    def near_threshold(self, d2, contact, rel=1e-9):
        """True when some foot in contact has d^2 within rel of gate or release: the kernel's rounding may then decide the other way"""
        if d2 is None:
            return False
        inc = stance_flags(contact)
        return bool(np.any(inc & ((np.abs(d2 - self.p["gate"]) <= rel * self.p["gate"]) | (np.abs(d2 - self.p["release"]) <= rel * self.p["release"]))))
