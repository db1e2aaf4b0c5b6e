"""The GPU closed loop (qm_control_b200.closed_loop.run) replayed call by call against the oracle and the plant twin (tests/_loop_replay.py).

The parity tests of the controller kernels take their inputs from synthetic.make_batch and hand the warm start over with mpc_set_solution.  Here the
inputs are the states the loop visits: the device's own warm-start chain over 30 solves, x0 from the observation update with its yaw unwrapped past
pi, targets re-anchored at every tick, the WBC at plant states with swing feet, slipping feet and payloads, evaluatePolicy 0-8 ms into each solution,
and the hw_write FIFO and plant pushes in their real order, all on a torch side stream.  Every call is restated from its own recorded inputs, so
every comparison is one call deep at the usual tolerances."""
import os
import time

import numpy as np
import pytest

import _loop_replay as R
from _oracle import Oracle
from _payload_urdf import edited_urdf
from _sim_twin_terrain import SimTwinTerrain
from qm_control_b200 import _lib

pytestmark = pytest.mark.gpu

G = 6                        # robots per condition
B = 5 * G                    # 30: not a multiple of 8
DURATION = 0.3
PL = {n: i for i, n in enumerate(_lib.PAYLOAD_LAYOUT)}
WR = {n: i for i, n in enumerate(_lib.WRENCH_LAYOUT)}
TURN = slice(G, 2 * G)


def _conditions():
    """trot at 0.3 m/s; trot turning at +-0.8 rad/s from yaw +-3.10; stance pushed sideways with 150 N for 0.1 s; trot with 1.5 kg in the gripper,
    the controller told; the same payload untold on a floor with mu 0.35."""
    grp = np.arange(B) // G
    gait = ["stance" if g == 2 else "trot" for g in grp]
    cmd = np.zeros((B, 4)); cmd[np.isin(grp, (0, 3, 4)), 0] = 0.3
    sign = np.where(np.arange(G) % 2 == 0, 1.0, -1.0); cmd[TURN, 3] = 0.8 * sign
    xy_yaw = np.zeros((B, 3)); xy_yaw[:, 0] = 0.5 * np.arange(B); xy_yaw[TURN, 2] = 3.10 * sign
    w = np.zeros((B, 12)); w[grp == 2, WR["f_base_y"]] = 150.0
    pushes = (np.full(B, 0.1), np.where(grp == 2, 0.1, 0.0), w)
    payload = np.zeros((B, 8)); payload[grp >= 3, PL["m_ee"]] = 1.5; payload[grp >= 3, PL["o_ee_x"]] = 0.02; payload[grp >= 3, PL["o_ee_z"]] = 0.04
    model = np.where((grp == 3)[:, None], payload, 0.0)
    mu = np.where(grp == 4, 0.35, 0.6)
    return dict(duration=DURATION, gait=gait, cmd_vel=cmd, xy_yaw=xy_yaw, pushes=pushes, payload=payload, friction_mu=mu, model_payload=model)


def _fresh_run(record):
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    s = q.Solver(batch=B, device=0)
    try:
        if record:
            return R.record(s, lambda: closed_loop.run(s, **_conditions()))
        return closed_loop.run(s, **_conditions()), None
    finally:
        s.close()


def test_closed_loop_replays_call_by_call(tmp_path):
    t0 = time.time()
    res, rec = _fresh_run(record=True)
    plain, _ = _fresh_run(record=False)
    for k in ("base", "ee", "status", "contact", "q", "v"):           # recording does not perturb the run
        np.testing.assert_array_equal(res[k], plain[k], err_msg=k)
    t_run = time.time() - t0

    cond = _conditions(); grp = np.arange(B) // G
    np.testing.assert_array_equal(rec.meta["payload"], cond["payload"]); np.testing.assert_array_equal(rec.meta["friction_mu"], cond["friction_mu"])
    np.testing.assert_array_equal(rec.meta["model_payload"], cond["model_payload"])
    nominal = Oracle(); told = Oracle(urdf=edited_urdf(tmp_path, cond["payload"][3 * G]))
    oracles = [told if g == 3 else nominal for g in grp]
    n_solves, n_updates = int(round(DURATION * 100)), int(round(DURATION * 500))

    stages = dict(targets=lambda: R.replay_targets(rec), mpc=lambda: R.replay_mpc(rec, oracles), invariant=lambda: R.replay_invariant(rec),
                  update=lambda: R.replay_update(rec, oracles), hw_write=lambda: R.replay_hw_write(rec, 0.009), plant=lambda: R.replay_plant(rec, SimTwinTerrain()))
    out = {}; failed = {}; secs = {}
    for name, replay in stages.items():          # every stage runs and reports before the first failure is raised
        t1 = time.time()
        try:
            out[name] = replay()
        except AssertionError as e:
            failed[name] = str(e)[:3000]
        secs[name] = time.time() - t1

    fmt = lambda d: ", ".join("%s %.1e" % (k, v) for k, v in d.items())
    print("\nclosed-loop replay, %d robots, %.1f s: run twice %.1f s; replay %s (%d threads)" % (B, DURATION, t_run, ", ".join("%s %.1f s" % kv for kv in secs.items()),
                                                                                            os.cpu_count() or 1))
    tg, mpc, inv, up, hw, pl = (out.get(k) for k in stages)
    if tg:
        print("  targets   worst %.1e over %d robot-calls" % (tg["worst"], tg["replayed"]))
    if mpc:
        print("  mpc       %d robot-solves replayed (%d warm, %d without a step, %d raised, %d near a line-search threshold): %s" % (
            mpc["replayed"], mpc["warm"], mpc["no_step"], mpc["raised"], len(mpc["near"]), fmt(mpc["worst"])))
    if up:
        print("  update    %d robot-updates (%d in swing, %d certified by KKT), max |yaw| turning group %.4f: %s" % (
            up["replayed"], up["swing"], up["certified"], float(np.max(up["yaw_max"][TURN])), fmt(up["worst"])))
    if hw:
        print("  hw_write  %d robot-calls bit-exact" % hw["replayed"])
    if pl:
        print("  plant     %d robot-steps (%d pushed): %s" % (pl["replayed"], pl["pushed"], fmt(pl["worst"])))
    for name, msg in failed.items():
        print("  FAILED %s: %s" % (name, msg))
    assert not failed, sorted(failed)

    assert mpc["ticks"] == n_solves and mpc["replayed"] + mpc["excused"] == n_solves * B and mpc["raised"] == 0
    assert mpc["warm"] == (n_solves - 1) * B and inv == n_solves - 1
    assert tg["replayed"] == n_solves * B
    assert up["updates"] == n_updates and up["replayed"] == n_updates * B
    assert hw["replayed"] == int(round(DURATION * 1e3)) * B and pl["replayed"] == (int(round(DURATION * 1e3)) + 1) * B
    assert up["swing"] > 0 and pl["pushed"] == 100 * G
    assert np.all(up["yaw_max"][TURN] > np.pi), up["yaw_max"][TURN]
