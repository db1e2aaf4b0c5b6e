"""ctypes binding of the CPU twin of the plant step (tests/sim_twin.cpp) — TEST INFRASTRUCTURE ONLY.

The twin is compiled on first use into a temporary directory, together with the oracle's model code (oracle/src/model.cpp)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from _oracle import REFERENCE, ROOT, TASK, URDF, _d, f64

SRC = os.path.join(ROOT, "tests", "sim_twin.cpp")
ORACLE_SRC = os.path.join(ROOT, "oracle", "src")
_lib = None

# qmb200_sim_params defaults (include/qmb200.h, DESIGN.md §4.6)
DEFAULTS = dict(ground_height=0.0, foot_radius=0.0265, stiffness=1e6, damping=1e3, tangential_damping=1e3, friction_mu=0.6,
                joint_damping=[0.05] * 12 + [0.0] * 6, substeps_per_ms=4)


def load():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="qmb_sim_twin_"), "libsimtwin.so")
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-variable", "-I" + ORACLE_SRC, "-o", out, SRC, os.path.join(ORACLE_SRC, "model.cpp")])
        lib = C.CDLL(out)
        lib.twin_create.restype = C.c_void_p
        lib.twin_destroy.argtypes = [C.c_void_p]
        lib.twin_accel.argtypes = [C.c_void_p] + [C.c_void_p] * 7
        lib.twin_step.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double] + [C.c_void_p] * 6
        _lib = lib
    return _lib


def _params(p):
    return f64(np.r_[p["ground_height"], p["foot_radius"], p["stiffness"], p["damping"], p["tangential_damping"], p["friction_mu"], p["joint_damping"]])


class SimTwin:
    def __init__(self, **params):
        self.lib = load()
        self.h = C.c_void_p(self.lib.twin_create(URDF.encode(), TASK.encode(), REFERENCE.encode()))
        assert self.h.value, "sim twin: model load failed"
        self.params = dict(DEFAULTS); self.params.update(params)

    def __del__(self):
        try:
            self.lib.twin_destroy(self.h)
        except Exception:
            pass

    def substeps(self, duration):
        """equal substeps no longer than 1 ms / substeps_per_ms (as qmb200_sim_step_dev)"""
        n = max(1, int(np.ceil(duration * 1e3 * self.params["substeps_per_ms"] - 1e-9)))
        return n, duration / n

    def step(self, duration, effort, q, v):
        """one robot → (q, v, rbd[55], contact, status)"""
        n, h = self.substeps(duration); q = f64(q).copy(); v = f64(v).copy(); rbd = np.zeros(55); c = C.c_int(); s = C.c_int(); p = _params(self.params)
        self.lib.twin_step(self.h, _d(p), n, h, _d(f64(effort)), _d(q), _d(v), _d(rbd), C.byref(c), C.byref(s))
        return q, v, rbd, c.value, s.value

    def measure(self, q, v):
        """the measured state rbd[55] at (q, v) (no substep)"""
        q = f64(q).copy(); v = f64(v).copy(); rbd = np.zeros(55); c = C.c_int(); s = C.c_int(); p = _params(self.params)
        self.lib.twin_step(self.h, _d(p), 0, 0.0, _d(np.zeros(18)), _d(q), _d(v), _d(rbd), C.byref(c), C.byref(s))
        return rbd

    def step_batch(self, duration, effort, q, v):
        out = [self.step(duration, effort[b], q[b], v[b]) for b in range(len(q))]
        return (np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out]), np.array([o[3] for o in out], dtype=np.int32),
                np.array([o[4] for o in out], dtype=np.int32))

    def accel(self, effort, q, v):
        """right-hand side of one substep → (qdd[24], F[4,3] contact forces, contact mask)"""
        qdd = np.zeros(24); F = np.zeros(12); m = C.c_int(); p = _params(self.params)
        rc = self.lib.twin_accel(self.h, _d(p), _d(f64(effort)), _d(f64(q)), _d(f64(v)), _d(qdd), _d(F), C.byref(m))
        assert rc == 0, "sim twin: mass matrix not positive definite"
        return qdd, F.reshape(4, 3), m.value
