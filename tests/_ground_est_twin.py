"""CPU twin of the state estimator's ground map (qmb200_state_est_set_ground, state_est_kernel.cu's map instantiation) — TEST INFRASTRUCTURE ONLY.

GroundEstTwin is the plane twin (tests/_state_est_twin.py) whose four foot-height rows follow one robot's mapped ground: the rows of C are built dense,
+1 at p_f,z and -gx_f, -gy_f at p_f,x, p_f,y, and H, g come from the terrain twin's own interpolation (SimTwinTerrain.ground, tests/sim_twin_terrain.cpp),
not from the product's lookup.  The innovation of foot f is foot_height + (H_f - ground_height) + (s_f - 1) c - p_f,z with c = foot_height -
ground_height, so a zero gradient and H_f = ground_height give the plane twin's numbers."""
import numpy as np

from _sim_twin_terrain import SimTwinTerrain
from _state_est_twin import NX, ST_NAN, ST_NOT_PD, StateEstTwin, quat_from_rot

_SIM = None


def _sim():
    global _SIM
    if _SIM is None:
        _SIM = SimTwinTerrain()
    return _SIM


class GroundEstTwin(StateEstTwin):
    """terrain: one robot's map, dict(tiles [T, ny, nx], cell, tile, origin [2]) (tile -1 or None: the plane z = ground_height)."""

    def __init__(self, params, terrain, ground_height=0.0, oracle=None):
        super().__init__(params, oracle); self.terrain = terrain; self.ground_height = float(ground_height)

    def ground(self, x, y):
        """(H, gx, gy) of the map at world (x, y)"""
        if self.terrain is None or int(self.terrain["tile"]) < 0:
            return self.ground_height, 0.0, 0.0
        return _sim().ground(self.terrain, x, y)

    def rows(self, x):
        """the dense C and the height rows' y_f - H_f part (foot_height + (H - ground_height) + (s - 1) c) at the predicted state x"""
        p = self.p; C = self.C.copy(); yh = np.zeros(4); c = p["foot_height"] - self.ground_height
        for f in range(4):
            H, gx, gy = self.ground(x[6 + 3 * f], x[7 + 3 * f]); s = np.sqrt(1.0 + gx * gx + gy * gy)
            C[24 + f, 6 + 3 * f] -= gx; C[24 + f, 7 + 3 * f] -= gy
            yh[f] = p["foot_height"] + (H - self.ground_height) + (s - 1.0) * c
        return C, yh

    def step(self, s, dt, sensors, contact):
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
            C, yh = self.rows(x)
            inn = np.r_[-r.ravel(), -rd.ravel(), np.full(4, p["foot_height"])] - self.C @ x
            inn[24:] = yh - x[8::3]
            sc = np.where(stance, 1.0, p["swing_scale"])
            Rm = np.diag(np.r_[np.repeat(sc, 3) * p["meas_foot_pos"], np.repeat(sc, 3) * p["meas_foot_vel"], sc * p["meas_foot_height"]])
            S = C @ P @ C.T + Rm
            if np.any(np.linalg.eigvalsh(S) <= 0):
                code = ST_NOT_PD
            else:
                K = np.linalg.solve(S, C @ P).T
                x_new = x + K @ inn
                P_new = P - K @ C @ P; P_new = 0.5 * (P_new + P_new.T)
                if np.all(np.isfinite(x_new)) and np.all(np.isfinite(P_new)):
                    s["x"], s["P"] = x_new, P_new
                else:
                    code = ST_NAN
        s["n"] += 1
        x = s["x"]
        rbd = np.r_[e, x[0:3], sensors[10:28], om, x[3:6], sensors[28:46], x[0:3] + ee_p, quat_from_rot(ee_R)]
        return rbd, code


def height_residual(q_foot, terrain, foot_height, ground_height=0.0):
    """h_f - s_f c of world foot-centre points q_foot [4, 3] on one robot's map: 0 where the map row is met exactly"""
    t = GroundEstTwin.__new__(GroundEstTwin); t.terrain = terrain; t.ground_height = float(ground_height)
    out = np.zeros(len(q_foot))
    for f, (x, y, z) in enumerate(q_foot):
        H, gx, gy = t.ground(x, y)
        out[f] = z - H - np.sqrt(1.0 + gx * gx + gy * gy) * (foot_height - ground_height)
    return out
