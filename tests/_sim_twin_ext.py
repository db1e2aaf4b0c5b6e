"""ctypes binding of the CPU twin of the plant step with per-robot variation (tests/sim_twin_ext.cpp) — TEST INFRASTRUCTURE ONLY.

SimTwinExt is the plain twin (tests/_sim_twin.py) plus the variation entry points: friction mu (a scalar per robot), payload [8] and wrench [12] in the
layouts of qmb200_sim_set_robot_params / qmb200_sim_step_ext.  The library is compiled on first use into a temporary directory, together with the
oracle's model code (oracle/src/model.cpp)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from _oracle import REFERENCE, ROOT, TASK, URDF, _d, f64
from _sim_twin import ORACLE_SRC, SimTwin, _params

SRC = os.path.join(ROOT, "tests", "sim_twin_ext.cpp")
_lib = None


def load():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="qmb_sim_twin_ext_"), "libsimtwinext.so")
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-variable", "-I" + ORACLE_SRC, "-o", out, SRC, os.path.join(ORACLE_SRC, "model.cpp")])
        lib = C.CDLL(out)
        lib.twin_ext_create.restype = C.c_void_p
        lib.twin_ext_destroy.argtypes = [C.c_void_p]
        lib.twin_accel_ext.argtypes = [C.c_void_p] * 10
        lib.twin_step_ext.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_double] + [C.c_void_p] * 6
        lib.twin_rbd_ext.argtypes = [C.c_void_p] * 10
        _lib = lib
    return _lib


def _opt(a, n):
    return None if a is None else f64(a).reshape(n)


def _ptr(a):
    return None if a is None else _d(a)


class SimTwinExt(SimTwin):
    def __init__(self, **params):
        super().__init__(**params)
        self.xlib = load()
        self.xh = C.c_void_p(self.xlib.twin_ext_create(URDF.encode(), TASK.encode(), REFERENCE.encode()))
        assert self.xh.value, "sim twin (ext): model load failed"

    def __del__(self):
        try:
            self.xlib.twin_ext_destroy(self.xh)
        except Exception:
            pass
        super().__del__()

    def _row(self, mu):
        p = dict(self.params)
        if mu is not None:
            p["friction_mu"] = float(mu)
        return _params(p)

    def step_ext(self, duration, effort, q, v, mu=None, payload=None, wrench=None):
        """one robot with its own friction, payload and wrench → (q, v, rbd[55], contact, status)"""
        n, h = self.substeps(duration); q = f64(q).copy(); v = f64(v).copy(); rbd = np.zeros(55); c = C.c_int(); s = C.c_int()
        p = self._row(mu); pl = _opt(payload, 8); wr = _opt(wrench, 12)
        self.xlib.twin_step_ext(self.xh, _d(p), _ptr(pl), _ptr(wr), n, h, _d(f64(effort)), _d(q), _d(v), _d(rbd), C.byref(c), C.byref(s))
        return q, v, rbd, c.value, s.value

    def step_batch_ext(self, duration, effort, q, v, mu=None, payload=None, wrench=None):
        """per-robot arrays: mu [B], payload [B, 8], wrench [B, 12] (each optional)"""
        pick = lambda a, b: None if a is None else a[b]
        out = [self.step_ext(duration, effort[b], q[b], v[b], pick(mu, b), pick(payload, b), pick(wrench, b)) for b in range(len(q))]
        return (np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out]), np.array([o[3] for o in out], dtype=np.int32),
                np.array([o[4] for o in out], dtype=np.int32))

    def accel_ext(self, effort, q, v, mu=None, payload=None, wrench=None):
        """right-hand side of one substep with the variation → (qdd[24], F[4,3], contact mask)"""
        qdd = np.zeros(24); F = np.zeros(12); m = C.c_int(); p = self._row(mu); pl = _opt(payload, 8); wr = _opt(wrench, 12)
        rc = self.xlib.twin_accel_ext(self.xh, _d(p), _ptr(pl), _ptr(wr), _d(f64(effort)), _d(f64(q)), _d(f64(v)), _d(qdd), _d(F), C.byref(m))
        assert rc == 0, "sim twin: mass matrix not positive definite"
        return qdd, F.reshape(4, 3), m.value

    def rbd_ext(self, q, v, payload=None):
        """rigid-body quantities of the robot with its payload → dict(M, nle, Ag (about the COM), dAg_v, com, mass)"""
        o = dict(M=np.zeros((24, 24)), nle=np.zeros(24), Ag=np.zeros((6, 24)), dAg_v=np.zeros(6), com=np.zeros(3)); mass = C.c_double(); pl = _opt(payload, 8)
        self.xlib.twin_rbd_ext(self.xh, _ptr(pl), _d(f64(q)), _d(f64(v)), *[_d(o[k]) for k in ("M", "nle", "Ag", "dAg_v", "com")], C.byref(mass))
        o["mass"] = mass.value
        return o
