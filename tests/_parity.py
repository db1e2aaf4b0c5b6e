"""Parity metrics shared by the GPU tests.

The contract (BASELINE.json north_star) is 1e-5 relative on the optimal trajectories and on the WBC vector.  A single
max-norm over a whole trajectory hides small blocks behind large ones (67-134 N contact forces next to O(0.1) joint
velocities; 80 Nm torques next to accelerations), so every comparison here is PER BLOCK of like quantities:

    err(block) = max |cuda - oracle| / max(floor(block), max |oracle block|)

`floor` is the natural magnitude of the block in this model (SURVEY.md 8d synthetic ranges) - it only keeps the ratio
meaningful when a block is numerically zero (swing-leg forces, a base at rest).  The ASSERTED tolerances sit three decades
below the contract (the CUDA path and the oracle agree to ~1e-11 on one SQP step), so a
regression of the kernels' accuracy by more than ~100x fails the suite long before the contract is in danger."""
import json
import os

import numpy as np

CONTRACT = 1e-5          # north_star tolerance
MPC_TOL = 1e-8           # asserted: one SQP iteration (LQ + projection + Riccati + line search), per block
WBC_TOL = 1e-8           # asserted: one WbcBase::update on identical inputs, per block
MPCWBC_TOL = 1e-8        # asserted: HierarchicalMpcWbc (arm torque limits active, arm accelerations of 1e4 rad/s^2 behind a 3e3-conditioned 6x6 block); both sides are KKT
                         # points to 1e-11 once the oracle refines its levels on the active set, observed agreement ~1e-11
TICK_TOL = 1e-6          # asserted: MPC -> evaluatePolicy -> WBC chain (the WBC's PD laws multiply the MPC's ~1e-11 by gains up to 6000: still a decade below the contract)
PLANT_TOL = 1e-8         # asserted: one plant step against the CPU plant twin, per block of q, v and the measurement rbd

# name -> (lo, hi, floor)
X_BLOCKS = {"h_lin/m": (0, 3, 0.1), "h_ang/m": (3, 6, 0.05), "base_pos": (6, 9, 0.1), "base_zyx": (9, 12, 0.1), "leg_q": (12, 24, 0.1), "arm_q": (24, 30, 0.1)}
U_BLOCKS = {"force": (0, 12, 10.0), "leg_qd": (12, 24, 0.1), "arm_qd": (24, 30, 0.1)}
CMD_BLOCKS = {"base_lin_acc": (0, 3, 1.0), "base_ang_acc": (3, 6, 1.0), "leg_acc": (6, 18, 1.0), "arm_acc": (18, 24, 1.0), "force": (24, 36, 10.0), "leg_torque": (36, 48, 1.0), "arm_torque": (48, 54, 1.0)}
Q_BLOCKS = {"pos": (0, 3, 1.0), "euler": (3, 6, 1.0), "joints": (6, 24, 1.0)}                    # the plant's q [24] and v [24]
RBD_BLOCKS = {"euler": (0, 3, 1.0), "pos": (3, 6, 1.0), "joints": (6, 24, 1.0), "w": (24, 27, 1.0), "v_lin": (27, 30, 1.0), "joint_vel": (30, 48, 1.0), "ee_pos": (48, 51, 1.0),
              "ee_quat": (51, 55, 1.0)}                                                            # the plant's measurement rbd [55]

_LOG = os.environ.get("QMB_PARITY_LOG")


def _log(tag, levels):
    if _LOG:
        with open(_LOG, "a") as f:
            f.write(json.dumps({"test": tag, "levels": {k: float(v) for k, v in levels.items()}}) + "\n")


def block_errors(out, ref, blocks):
    """out, ref: [..., D] arrays; → {block: err} with the per-block relative error defined above (max over the leading axes)."""
    out = np.asarray(out); ref = np.asarray(ref); res = {}
    for name, (lo, hi, floor) in blocks.items():
        d = np.max(np.abs(out[..., lo:hi] - ref[..., lo:hi])) if out.size else 0.0
        s = max(floor, float(np.max(np.abs(ref[..., lo:hi]))) if ref.size else floor)
        res[name] = float(d) / s
    return res


def traj_errors(out, ref, b_out=None, b_ref=None):
    """Per-block errors of the trajectories of one robot pair (or, with b_* None, of every robot: worst block error over the batch).
    Also checks the grid: node count, node times (1e-12) and event annotations."""
    pairs = [(b_out, b_ref)] if b_out is not None else [(b, b) for b in range(len(ref["n_nodes"]))]
    worst = {}
    for bo, br in pairs:
        n = int(ref["n_nodes"][br]); assert int(out["n_nodes"][bo]) == n, (bo, int(out["n_nodes"][bo]), n)
        if "t" in out and "t" in ref:
            np.testing.assert_allclose(out["t"][bo, :n], ref["t"][br, :n], rtol=0, atol=1e-12); np.testing.assert_array_equal(out["event"][bo, :n], ref["event"][br, :n])
        ex = block_errors(out["x"][bo, :n], ref["x"][br, :n], X_BLOCKS)
        k = np.nonzero(ref["event"][br, :n - 1] != 1)[0]
        eu = block_errors(out["u"][bo, k], ref["u"][br, k], U_BLOCKS)
        for name, v in list(ex.items()) + [("u:" + kk, vv) for kk, vv in eu.items()]:
            worst[name] = max(worst.get(name, 0.0), v)
    return worst


def assert_traj(out, ref, tol=MPC_TOL, tag="mpc", b_out=None, b_ref=None):
    lv = traj_errors(out, ref, b_out, b_ref); _log(tag, lv)
    bad = {k: v for k, v in lv.items() if not v < tol}
    assert not bad, "%s: per-block relative error above %.1e: %s" % (tag, tol, bad)
    return lv


def cmd_errors(cmd, ref, blocks=None):
    """cmd, ref: [B, 54] (or [54]) - per robot and per block, worst robot reported."""
    cmd = np.atleast_2d(cmd); ref = np.atleast_2d(ref); res = {}
    for name, (lo, hi, floor) in (blocks or CMD_BLOCKS).items():
        d = np.max(np.abs(cmd[:, lo:hi] - ref[:, lo:hi]), axis=1); s = np.maximum(floor, np.max(np.abs(ref[:, lo:hi]), axis=1))
        res[name] = float(np.max(d / s)) if len(d) else 0.0
    return res


def assert_cmd(cmd, ref, tol=WBC_TOL, tag="wbc", blocks=None):
    lv = cmd_errors(cmd, ref, blocks); _log(tag, lv)
    bad = {k: v for k, v in lv.items() if not v < tol}
    assert not bad, "%s: per-block relative error above %.1e: %s" % (tag, tol, bad)
    return lv
