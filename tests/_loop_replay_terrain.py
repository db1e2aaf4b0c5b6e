"""Call-by-call replay of a closed-loop run on heightfield terrain — TEST INFRASTRUCTURE ONLY.

tests/_loop_replay.py records the loop's device calls and restates each stage; its plant stage knows friction, payload and wrench.  Here
`record(solver, fn)` records the same way and also keeps the plant's ground as the run sets it (Solver.sim_get_terrain + sim_get_robot_terrain at
the first plant step) in rec.meta["terrain"] = dict(tiles, cell, tile [B], origin [B, 2]) or None, and `replay_plant` restates every plant step on the
terrain twin (tests/sim_twin_terrain.cpp) with that ground.  The other stages replay with tests/_loop_replay.py unchanged."""
import functools

import numpy as np

import _loop_replay as R
from _sim_twin_terrain import robot_terrain


def record(solver, fn):
    """→ (fn(), Record) as _loop_replay.record, with rec.meta["terrain"]"""
    seen = {}
    orig = solver.sim_step_dev

    @functools.wraps(orig)
    def sim_step_dev(*args, **kw):
        if not seen:
            lib, robot = solver.sim_get_terrain(), solver.sim_get_robot_terrain()
            seen["terrain"] = None if robot is None else dict(tiles=None if lib is None else lib["tiles"], cell=None if lib is None else lib["cell"], **robot)
        return orig(*args, **kw)
    solver.sim_step_dev = sim_step_dev   # _loop_replay.record wraps this one and removes the instance attribute again when fn returns
    try:
        res, rec = R.record(solver, fn)
    finally:
        solver.__dict__.pop("sim_step_dev", None)
    rec.meta["terrain"] = seen.get("terrain")
    return res, rec


def replay_plant(rec, twin, every=1):
    """_loop_replay.replay_plant on the recorded terrain: every `every`-th plant step of every robot on the twin (a SimTwinTerrain) with the robot's
    friction, payload, wrench and ground of that step, at PLANT_TOL per block; contact mask and status exact."""
    mu, pl, ter = rec.meta.get("friction_mu"), rec.meta.get("payload"), rec.meta.get("terrain"); worst = {}; n = 0; pushed = 0
    for i, (inp, out) in enumerate(rec.of("sim")):
        if i % every:
            continue
        B = len(inp["q"]); w = inp["wrench"]
        for b in range(B):
            wb = None if w is None else w[b]; pushed += int(wb is not None and np.any(wb != 0))
            q, v, rbd, c, st = twin.step_ext(inp["duration"], inp["effort"][b], inp["q"][b], inp["v"][b], None if mu is None else mu[b], None if pl is None else pl[b], wb,
                                             terrain=robot_terrain(ter, b))
            assert out["contact"][b] == c and out["status"][b] == st, ("plant step %d robot %d" % (i, b), out["contact"][b], c, out["status"][b], st)
            for name, a, r, blocks in (("q", out["q"][b], q, R.Q_BLOCKS), ("v", out["v"][b], v, R.Q_BLOCKS), ("rbd", out["rbd"][b], rbd, R.RBD_BLOCKS)):
                err = R._rel(a, r, blocks)
                assert max(err.values()) < R.PLANT_TOL, ("plant step %d robot %d" % (i, b), name, err)
                for k, e in err.items():
                    worst[name + ":" + k] = max(worst.get(name + ":" + k, 0.0), e)
            n += 1
    return dict(worst=worst, replayed=n, pushed=pushed)
