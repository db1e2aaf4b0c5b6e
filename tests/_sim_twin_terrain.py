"""ctypes binding of the CPU twin of the plant step on heightfield terrain (tests/sim_twin_terrain.cpp) — TEST INFRASTRUCTURE ONLY.

SimTwinTerrain is the twin with per-robot variation (tests/_sim_twin_ext.py) whose step_ext / step_batch_ext / accel_ext also take
terrain = dict(tiles [T, ny, nx], cell, tile, origin) as Solver.sim_set_terrain / sim_set_robot_terrain take them: tile a scalar and origin [2] for one
robot, tile [B] and origin [B, 2] in the batch call; None or tile -1 is the params' plane (tests/sim_twin_ext.cpp's plane law).  The library is
compiled on first use into a temporary directory, together with the oracle's model code (oracle/src/model.cpp)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from _oracle import REFERENCE, ROOT, TASK, URDF, _d, f64
from _sim_twin import ORACLE_SRC
from _sim_twin_ext import SimTwinExt, _opt, _ptr

SRC = os.path.join(ROOT, "tests", "sim_twin_terrain.cpp")
_lib = None


def load():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="qmb_sim_twin_terrain_"), "libsimtwinterrain.so")
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-variable", "-I" + ORACLE_SRC, "-I" + os.path.dirname(SRC), "-o", out, SRC,
                               os.path.join(ORACLE_SRC, "model.cpp")])
        lib = C.CDLL(out)
        lib.twin_ext_create.restype = C.c_void_p
        lib.twin_ext_destroy.argtypes = [C.c_void_p]
        tile = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double]
        lib.twin_accel_terrain.argtypes = [C.c_void_p] * 4 + tile + [C.c_void_p] * 6
        lib.twin_step_terrain.argtypes = [C.c_void_p] * 4 + tile + [C.c_int, C.c_double] + [C.c_void_p] * 6
        lib.twin_ground.argtypes = tile + [C.c_double, C.c_double] + [C.c_void_p] * 3
        _lib = lib
    return _lib


def _on_tile(terrain):
    """one robot's terrain → (C arguments of its tile, the tile array they point into), or None on the plane"""
    if terrain is None or int(terrain["tile"]) < 0:
        return None
    t = f64(terrain["tiles"][int(terrain["tile"])]).copy(); o = np.asarray(terrain["origin"], dtype=np.float64)
    return (_d(t), t.shape[1], t.shape[0], float(terrain["cell"]), float(o[0]), float(o[1])), t


def robot_terrain(terrain, b):
    """robot b's terrain out of a batch terrain (tile [B], origin [B, 2]); None stays None"""
    return None if terrain is None else dict(tiles=terrain["tiles"], cell=terrain["cell"], tile=np.asarray(terrain["tile"])[b], origin=np.asarray(terrain["origin"])[b])


class SimTwinTerrain(SimTwinExt):
    def __init__(self, **params):
        super().__init__(**params)
        self.tlib = load()
        self.th = C.c_void_p(self.tlib.twin_ext_create(URDF.encode(), TASK.encode(), REFERENCE.encode()))
        assert self.th.value, "sim twin (terrain): model load failed"

    def __del__(self):
        try:
            self.tlib.twin_ext_destroy(self.th)
        except Exception:
            pass
        super().__del__()

    def step_ext(self, duration, effort, q, v, mu=None, payload=None, wrench=None, terrain=None):
        """one robot with its own friction, payload, wrench and terrain → (q, v, rbd[55], contact, status)"""
        tile = _on_tile(terrain)
        if tile is None:
            return super().step_ext(duration, effort, q, v, mu, payload, wrench)
        n, h = self.substeps(duration); q = f64(q).copy(); v = f64(v).copy(); rbd = np.zeros(55); c = C.c_int(); s = C.c_int()
        p = self._row(mu); pl = _opt(payload, 8); wr = _opt(wrench, 12)
        self.tlib.twin_step_terrain(self.th, _d(p), _ptr(pl), _ptr(wr), *tile[0], n, h, _d(f64(effort)), _d(q), _d(v), _d(rbd), C.byref(c), C.byref(s))
        return q, v, rbd, c.value, s.value

    def step_batch_ext(self, duration, effort, q, v, mu=None, payload=None, wrench=None, terrain=None):
        """per-robot arrays: mu [B], payload [B, 8], wrench [B, 12], terrain with tile [B] and origin [B, 2] (each optional)"""
        pick = lambda a, b: None if a is None else a[b]
        out = [self.step_ext(duration, effort[b], q[b], v[b], pick(mu, b), pick(payload, b), pick(wrench, b), robot_terrain(terrain, b)) for b in range(len(q))]
        return (np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out]), np.array([o[3] for o in out], dtype=np.int32),
                np.array([o[4] for o in out], dtype=np.int32))

    def accel_ext(self, effort, q, v, mu=None, payload=None, wrench=None, terrain=None):
        """right-hand side of one substep with the variation and terrain → (qdd[24], F[4,3], contact mask)"""
        tile = _on_tile(terrain)
        if tile is None:
            return super().accel_ext(effort, q, v, mu, payload, wrench)
        qdd = np.zeros(24); F = np.zeros(12); m = C.c_int(); p = self._row(mu); pl = _opt(payload, 8); wr = _opt(wrench, 12)
        rc = self.tlib.twin_accel_terrain(self.th, _d(p), _ptr(pl), _ptr(wr), *tile[0], _d(f64(effort)), _d(f64(q)), _d(f64(v)), _d(qdd), _d(F), C.byref(m))
        assert rc == 0, "sim twin: mass matrix not positive definite"
        return qdd, F.reshape(4, 3), m.value

    def ground(self, terrain, x, y):
        """the twin's height and gradient (H, gx, gy) of one robot's tile at world (x, y)"""
        tile = _on_tile(terrain); H, gx, gy = C.c_double(), C.c_double(), C.c_double()
        self.tlib.twin_ground(*tile[0], float(x), float(y), C.byref(H), C.byref(gx), C.byref(gy))
        return H.value, gx.value, gy.value
