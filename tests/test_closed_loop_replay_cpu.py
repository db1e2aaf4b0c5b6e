"""The call-by-call replay of tests/_loop_replay.py on the CPU rehearsal of the closed loop (tests/_closed_loop_cpu.py): replaying the rehearsal's
own record reproduces it exactly, and a record whose warm start, WBC input_last or observation clock is taken from one call too early fails the MPC,
WBC and observation comparison respectively, so the replay of a GPU run would catch an off-by-one in the device's buffers."""
import copy

import numpy as np
import pytest

import _closed_loop_cpu
import _loop_replay as R
from _oracle import Oracle
from _sim_twin_terrain import SimTwinTerrain

T_START, DURATION = 10.0, 0.1


@pytest.fixture(scope="module")
def rehearsal():
    """one robot trotting at 0.3 m/s for 0.1 s: 10 solves, 50 updates, 101 plant steps"""
    from qm_control_b200.interface import gait_schedule
    oracle = Oracle(); rec = R.Record()
    sched = gait_schedule("trot", T_START, T_START - 0.002, T_START + DURATION + 2.0)
    _closed_loop_cpu.run(oracle, duration=DURATION, cmd_vel=(0.3, 0.0, 0.0, 0.0), t_start=T_START, mode_schedule=sched, recorder=rec)
    return oracle, rec


def test_replay_reproduces_the_rehearsal_exactly(rehearsal):
    oracle, rec = rehearsal
    assert [len(rec.of(s)) for s in ("targets", "mpc", "update", "hw_write", "sim")] == [10, 10, 50, 100, 101]
    tg = R.replay_targets(rec); assert tg["worst"] == 0.0 and tg["replayed"] == 10
    mpc = R.replay_mpc(rec, [oracle])
    assert mpc["replayed"] == 10 and mpc["warm"] == 9 and mpc["raised"] == 0 and not mpc["near"]
    assert all(v == 0.0 for v in mpc["worst"].values()), mpc["worst"]
    assert R.replay_invariant(rec) == 9
    up = R.replay_update(rec, [oracle])
    assert up["replayed"] == 50 and up["swing"] > 0 and up["certified"] == 0
    assert all(v == 0.0 for v in up["worst"].values()), up["worst"]
    assert R.replay_hw_write(rec, 0.009)["replayed"] == 100
    pl = R.replay_plant(rec, SimTwinTerrain())
    assert pl["replayed"] == 101 and pl["pushed"] == 0 and all(v == 0.0 for v in pl["worst"].values()), pl


def _one_call_early(rec, stage, key):
    """a copy of the record where every call of `stage` but the first reads inputs[key] of the call before it"""
    out = R.Record(); out.meta = dict(rec.meta); prev = None
    for s, inp, o in rec.calls:
        if s == stage:
            cur = inp[key]; inp = dict(inp)
            if prev is not None:
                inp[key] = copy.deepcopy(prev)
            prev = cur
        out.add(s, inp, o)
    return out


@pytest.mark.parametrize("stage,key,replay,match", [
    ("mpc", "before", lambda rec, o: R.replay_mpc(rec, [o]), r"mpc tick 1 robot 0"),
    ("update", "input_last", lambda rec, o: R.replay_update(rec, [o]), r"update 1 robot 0 \(mode \d+\): per-block relative error"),
    ("update", "t_obs", lambda rec, o: R.replay_update(rec, [o]), r"update 1 robot 0"),
])
def test_replay_catches_an_input_one_call_early(rehearsal, stage, key, replay, match):
    oracle, rec = rehearsal
    bad = _one_call_early(rec, stage, key)
    second = lambda r: r.of(stage)[1][0][key]["x"] if key == "before" else r.of(stage)[1][0][key]
    assert not np.array_equal(second(bad), second(rec))
    with pytest.raises(AssertionError, match=match):
        replay(bad, oracle)
