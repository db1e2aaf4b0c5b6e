"""CPU twin of the online payload estimator (qm_control_b200/csrc/kernels/payload_est_kernel.cu) — TEST INFRASTRUCTURE ONLY.

The nominal M, nle, end-effector Jacobian, twist and bias acceleration come from the oracle's model (tests/payload_est_twin.cpp, compiled on first use into
a temporary directory with oracle/src/model.cpp); the regressor, the RLS update and the commit are restated here in numpy, in full matrices:
    y   = M[a, :] qdd + nle[a] - sat(tau)_a                                        (the six arm rows a of the nominal model)
    Phi = -(J_v,a^T R Y_f + J_w,a^T R Y_n)                                        (Newton-Euler of the load in the end-effector frame, about its origin)
with the frame's linear and angular acceleration a = J_v qdd + dJ_v v, dw = J_w qdd + dJ_w v and a - g = a + 9.81 z."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from _oracle import REFERENCE, ROOT, TASK, URDF, _d, f64
from _sim_twin import ORACLE_SRC

SRC = os.path.join(ROOT, "tests", "payload_est_twin.cpp")
ARM = slice(18, 24)
ST_NAN, ST_NOT_PD = 4, 8
_lib = None

# qmb200_payload_est_params defaults (include/qmb200.h, DESIGN.md §4.6)
DEFAULTS = dict(forgetting=0.999, p0_mass=25.0, p0_first_moment=0.25, p0_inertia=0.0025, trace_max=30.0, mass_min=0.02, mass_max=10.0, offset_max=0.3)


def load():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="qmb_payload_est_twin_"), "libpayloadesttwin.so")
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-variable", "-I" + ORACLE_SRC, "-o", out, SRC, os.path.join(ORACLE_SRC, "model.cpp")])
        lib = C.CDLL(out)
        lib.twin_est_create.restype = C.c_void_p
        lib.twin_est_destroy.argtypes = [C.c_void_p]
        lib.twin_est_rbd.argtypes = [C.c_void_p] * 12
        _lib = lib
    return _lib


def skew(x):
    return np.array([[0.0, -x[2], x[1]], [x[2], 0.0, -x[0]], [-x[1], x[0], 0.0]])


def inertia_map(u):
    """L(u) with I u = L(u) [xx, xy, xz, yy, yz, zz]"""
    return np.array([[u[0], u[1], u[2], 0, 0, 0], [0, u[0], 0, u[1], u[2], 0], [0, 0, u[0], 0, u[1], u[2]]], dtype=float)


def point_mass_theta(m, o):
    """theta of a point mass m at offset o in the end-effector frame"""
    o = np.asarray(o, dtype=float); I = m * (o @ o * np.eye(3) - np.outer(o, o))
    return np.r_[m, m * o, I[0, 0], I[0, 1], I[0, 2], I[1, 1], I[1, 2], I[2, 2]]


def rbd_to_qv(rbd):
    """the measurement rbd[55] → (q, v with euler rates), as the WBC's measured pass reads it"""
    rbd = np.asarray(rbd, dtype=float); q = np.r_[rbd[3:6], rbd[0:3], rbd[6:24]]
    z, y = q[3], q[4]
    T = np.array([[0.0, -np.sin(z), np.cos(y) * np.cos(z)], [0.0, np.cos(z), np.cos(y) * np.sin(z)], [1.0, 0.0, -np.sin(y)]])
    v = np.r_[rbd[27:30], np.linalg.solve(T, rbd[24:27]), rbd[30:48]]
    return q, v


class PayloadEstTwin:
    def __init__(self, **params):
        self.lib = load()
        self.h = C.c_void_p(self.lib.twin_est_create(URDF.encode(), TASK.encode(), REFERENCE.encode()))
        assert self.h.value, "payload estimator twin: model load failed"
        self.params = dict(DEFAULTS); self.params.update(params)

    def __del__(self):
        try:
            self.lib.twin_est_destroy(self.h)
        except Exception:
            pass

    def rbd(self, q, v):
        """nominal model at (q, v) → dict(M, nle, J (6x24: linear, angular), dJv, pos, R, vel, w, effort)"""
        o = dict(M=np.zeros((24, 24)), nle=np.zeros(24), J=np.zeros((6, 24)), dJv=np.zeros(6), pos=np.zeros(3), R=np.zeros((3, 3)), vel=np.zeros(3), w=np.zeros(3), effort=np.zeros(18))
        self.lib.twin_est_rbd(self.h, _d(f64(q)), _d(f64(v)), *[_d(o[k]) for k in ("M", "nle", "J", "dJv", "pos", "R", "vel", "w", "effort")])
        return o

    def residual_and_regressor(self, q, v, qdd, effort):
        """(y [6], Phi [6, 10]) of the nominal arm rows at (q, v) with acceleration qdd and the effort held"""
        d = self.rbd(q, v); qdd = np.asarray(qdd, dtype=float)
        tau = np.clip(np.asarray(effort, dtype=float), -d["effort"], d["effort"])
        y = d["M"][ARM] @ qdd + d["nle"][ARM] - tau[12:18]
        acc = d["J"] @ qdd + d["dJv"]; R = d["R"]
        w, dw, a = R.T @ d["w"], R.T @ acc[3:6], R.T @ (acc[0:3] + np.array([0.0, 0.0, 9.81]))
        Yf = np.zeros((3, 10)); Yn = np.zeros((3, 10))
        Yf[:, 0] = a; Yf[:, 1:4] = skew(dw) + skew(w) @ skew(w)
        Yn[:, 1:4] = -skew(a); Yn[:, 4:10] = inertia_map(dw) + skew(w) @ inertia_map(w)
        Phi = -(d["J"][0:3, ARM].T @ R @ Yf + d["J"][3:6, ARM].T @ R @ Yn)
        return y, Phi

    # ---- the estimator state of one robot and its RLS step, as the kernel's ----
    def reset(self, prior_row):
        p = self.params; P = np.diag(np.r_[p["p0_mass"], [p["p0_first_moment"]] * 3, [p["p0_inertia"]] * 6])
        return dict(theta=point_mass_theta(prior_row[0], prior_row[1:4]), P=P, q=np.zeros(24), v=np.zeros(24), n=0)

    def step(self, s, dt, effort, rbd):
        """one call of payload_est_step_kernel on the state dict s (updated in place) → status"""
        q, v = rbd_to_qv(rbd)
        if not (np.all(np.isfinite(q)) and np.all(np.isfinite(v)) and np.all(np.isfinite(effort))):
            return ST_NAN
        if s["n"] == 0:
            s.update(q=q, v=v, n=1); return 0
        dq = q - s["q"]; dq[3:6] -= 2 * np.pi * np.rint(dq[3:6] / (2 * np.pi))
        qm, vm, qdd = s["q"] + 0.5 * dq, 0.5 * (v + s["v"]), (v - s["v"]) / dt
        y, Phi = self.residual_and_regressor(qm, vm, qdd, effort)
        code = self.rls(s, y, Phi)
        s.update(q=q, v=v, n=s["n"] + 1)
        return code

    def rls(self, s, y, Phi):
        lam = self.params["forgetting"]; P, th = s["P"], s["theta"]
        G = P @ Phi.T; S = lam * np.eye(6) + Phi @ G
        try:
            L = np.linalg.cholesky(S)
        except np.linalg.LinAlgError:
            return ST_NOT_PD
        K = np.linalg.solve(L.T, np.linalg.solve(L, G.T)).T
        th_new = th + K @ (y - Phi @ th)
        KG = K @ G.T; P_new = (P - 0.5 * (KG + KG.T)) / lam
        tr = np.trace(P_new)
        if tr > self.params["trace_max"]:
            P_new *= self.params["trace_max"] / tr
        if not (np.all(np.isfinite(th_new)) and np.all(np.isfinite(P_new))):
            return ST_NAN
        s.update(theta=th_new, P=P_new)
        return 0

    def commit(self, theta, row):
        """theta → the model payload row [8] (end-effector half replaced, base half kept)"""
        p = self.params; m0 = theta[0]; m = min(max(m0, 0.0), p["mass_max"]); o = np.zeros(3)
        if m0 >= p["mass_min"]:
            o = theta[1:4] / m0; n = np.linalg.norm(o)
            if n > p["offset_max"]:
                o = o * (p["offset_max"] / n)
        return np.r_[m, o, row[4:8]]
