"""Robot-state snapshots on the GPU (DESIGN.md §4.17), sensor noise off: a robot rewound to a snapshot replays its records bit for bit in every
configuration of the loop, a branched robot follows its source bit for bit, the library's refusals write nothing, and a torch planner steers robots by
predictive sampling on branched copies of them without synchronising."""
import numpy as np
import pytest

from qm_control_b200 import _lib
from qm_control_b200 import terrain as TR

pytestmark = pytest.mark.gpu

GETTERS = ("mpc_get_solution", "wbc_get_input_last", "sim_get_robot_params", "sim_get_robot_terrain", "get_model_payload", "get_robot_tuning", "payload_est_get",
           "state_est_get", "state_est_get_ground", "attitude_get", "slip_get", "gait_dev_get", "gait_dev_get_commands", "gait_dev_get_pending")


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


def _flat(x):
    """a getter's result as a list of (dtype, shape, bytes)"""
    if x is None:
        return [None]
    if isinstance(x, dict):
        return [k for key in sorted(x) for k in [key] + _flat(x[key])]
    if isinstance(x, (tuple, list)):
        return [k for v in x for k in _flat(v)]
    a = np.asarray(x)
    return [(a.dtype.str, a.shape, a.tobytes())]


def _getters(s):
    out = {}
    for g in GETTERS:
        try:
            out[g] = _flat(getattr(s, g)())
        except _lib.QmbError:   # the component does not run
            out[g] = ["not running"]
    return out


def _host(ss, rec):
    """a chunk's records on the host, once the session's stream has written them"""
    ss.stream.synchronize()
    return {k: v if isinstance(v, np.ndarray) else v.cpu().numpy() for k, v in rec.items()}


def _assert_same(a, b, what):
    assert set(a) == set(b), what
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), (what, k)


def _terrain(B):
    return dict(tiles=np.stack([TR.ramp(8.0), TR.stairs(0.05, 0.25), TR.rough(0.01, seed=7)]), cell=TR.CELL, tile=(np.arange(B) % 4 - 1).astype(np.int32),
                origin=TR.centred_origin(np.zeros((B, 2))))


def _commands(B):
    """a gait switch to pace for even robots at 0.05 s, an end-effector goal for every third robot at 0.12 s, a cmd_vel step for the rest at 0.2 s"""
    t = np.tile([0.05, 0.12, 0.2], (B, 1)); g = [["pace" if b % 2 == 0 else None, None, None] for b in range(B)]
    vel = np.full((B, 3, 4), np.nan); goal = np.full((B, 3, 7), np.nan)
    for b in range(B):
        if b % 3 == 0:
            goal[b, 1] = [0.55, 0.05 * (b % 2), 0.45, 0.0, 0.0, 0.0, 1.0]
        vel[b, 2] = [0.2, 0.0, 0.0, 0.1 * (b % 3 - 1)]
    return dict(t=t, gait=g, cmd_vel=vel, ee_goal=goal)


def _configs(B):
    rng = np.random.default_rng(3)
    pushes = (np.full(B, 0.1), np.full(B, 0.1), np.c_[rng.uniform(-30, 30, (B, 3)), np.zeros((B, 9))])   # on across the snapshot's window 15
    return dict(
        truth=(dict(), dict(gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.1), pushes=pushes, payload_estimator=True, model_payload="plant",
                            payload=np.c_[np.full(B, 0.3), np.zeros((B, 7))], terrain=_terrain(B), commands=_commands(B), metrics=True,
                            friction_mu=np.linspace(0.5, 0.9, B))),
        estimators=(dict(), dict(gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), terrain=_terrain(B), state_estimator=True, attitude_filter=True, slip_detector=True,
                                 ground_map=True, metrics=True)),
        mpc_wbc=(dict(wbc_variant=1), dict(gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.1))),
        sqp=(dict(), dict(gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.0), steer=True)),
        ipm=(dict(), dict(gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.0), steer=True)),
        ddp=(dict(), dict(gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.0), steer=True)))


@pytest.mark.parametrize("name", ["truth", "estimators", "mpc_wbc", "sqp", "ipm", "ddp"])
def test_rewind_equals_replay(name):
    """snapshot at window w, n windows, every robot restored from itself, the same n windows again: every record, the final state, the metrics
    accumulator and the library getters are the same bits"""
    import torch
    from qm_control_b200 import closed_loop
    B = 8; w, n = 15, 20; skw, kw = _configs(B)[name]; s = _solver(B, **skw)
    if name in ("sqp", "ipm", "ddp"):
        s.mpc_set_solver(name)
    try:
        with closed_loop.Session(s, 0.01 * (w + 2 * n), **kw) as ss:
            ss.step(w)
            if "commands" in kw:   # a command pending at the snapshot, applied by the tick after it
                ss.command(torch.ones(B, dtype=torch.int32, device=ss.device), cmd_vel=torch.full((B, 4), 0.15, dtype=torch.float64, device=ss.device))
            snap = ss.snapshot()
            runs = []
            for i in range(2):
                if i:
                    ss.restore(snap)
                rec = _host(ss, ss.step(n))
                runs.append((rec, [a.cpu().numpy() for a in ss.rows], _getters(s)))
            ss.finish()
    finally:
        s.close()
    (ra, rows_a, ga), (rb, rows_b, gb) = runs
    np.testing.assert_allclose(rb["t"] - ra["t"], 0.01 * n)   # the record times are the session's: n windows later
    _assert_same({k: v for k, v in ra.items() if k != "t"}, {k: v for k, v in rb.items() if k != "t"}, name)
    assert len(rows_a) == len(rows_b) and all(x.tobytes() == y.tobytes() for x, y in zip(rows_a, rows_b)), name
    for g in GETTERS:
        assert ga[g] == gb[g], (name, g)
    assert not np.any(ra["status"] & _lib.ST_RESTORE)
    print("rewind %s: %d records of %d robots, %d loop rows, %d library bytes per robot" % (name, n, B, len(rows_a), snap.desc.bytes))


def test_branch_equals_source():
    """restored robots follow robot source[b] of the same session run without the restore, byte for byte; unmasked robots follow themselves; the
    getters show the source's rows"""
    import torch
    from qm_control_b200 import closed_loop
    B = 12; w, n = 10, 25; rng = np.random.default_rng(8)
    tuning = dict(kp_swing=np.linspace(300.0, 400.0, B))
    kw = dict(gait="trot", cmd_vel=np.c_[np.linspace(0.0, 0.3, B), np.zeros((B, 2)), np.linspace(-0.2, 0.2, B)], friction_mu=np.linspace(0.4, 0.9, B),
              model_payload=np.c_[np.linspace(0.0, 0.5, B), np.zeros((B, 7))], tuning=tuning, terrain=_terrain(B), metrics=True,
              pushes=(np.full(B, 0.05), np.full(B, 0.2), np.c_[rng.uniform(-20, 20, (B, 3)), np.zeros((B, 9))]))
    perm = rng.permutation(B).astype(np.int32); many = rng.integers(0, 3, B).astype(np.int32)
    mask = np.ones(B, dtype=np.int32); mask[[1, 5]] = 0
    handles = [_solver(B) for _ in range(3)]   # one handle per session: a second session would warm-start from the first one's MPC solution
    try:
        with closed_loop.Session(handles[0], 0.01 * (w + n), **kw) as ss:   # the reference: no restore
            ss.step(w); want = _host(ss, ss.step(n)); ss.finish()
        for s, source in zip(handles[1:], (perm, many)):
            with closed_loop.Session(s, 0.01 * (w + n), **kw) as ss:
                ss.step(w); snap = ss.snapshot()
                ss.restore(snap, mask=torch.as_tensor(mask, device=ss.device), source=torch.as_tensor(source, device=ss.device))
                ss.stream.synchronize()
                src = np.where(mask != 0, source, np.arange(B))
                fr = s.sim_get_robot_params()["friction_mu"]; pl = s.get_model_payload(); tn = s.get_robot_tuning()
                got = _host(ss, ss.step(n)); ss.finish()
            for k in want:
                if k == "t":
                    continue
                assert got[k].tobytes() == want[k][:, src].tobytes(), k
            np.testing.assert_array_equal(fr, np.asarray(kw["friction_mu"])[src])
            np.testing.assert_array_equal(pl, kw["model_payload"][src])
            np.testing.assert_array_equal(tn["kp_swing"], tuning["kp_swing"][src])
    finally:
        for s in handles:
            s.close()


@pytest.mark.parametrize("name", ["gaits", "commands"])
def test_a_branch_at_window_zero_equals_source(name):
    """a snapshot of window 0 is taken after that window's blocking MPC tick: restored at once, robots of other gaits (and, with commands, other target
    kinds at that tick) follow their sources byte for byte through the window's updates, records, metrics and end state"""
    import torch
    from qm_control_b200 import closed_loop
    B = 12; n = 20; rng = np.random.default_rng(21)
    gaits = [["trot", "pace", "stance", "static_walk"][b % 4] for b in range(B)]
    kw = dict(gait=gaits, cmd_vel=np.c_[np.linspace(0.0, 0.3, B), np.zeros((B, 2)), np.linspace(-0.2, 0.2, B)], friction_mu=np.linspace(0.4, 0.9, B),
              metrics=True, payload_estimator=True, model_payload="plant", payload=np.c_[np.linspace(0.0, 0.4, B), np.zeros((B, 7))])
    if name == "commands":   # an end-effector goal due at the first tick for every third robot: target kinds differ within window 0
        goal = np.full((B, 1, 7), np.nan); goal[::3, 0] = [0.55, 0.0, 0.45, 0.0, 0.0, 0.0, 1.0]
        kw["commands"] = dict(t=np.full((B, 1), -0.005), gait=[[None]] * B, ee_goal=goal)
    source = rng.permutation(B).astype(np.int32); source[:3] = [1, 2, 1]   # a permutation of most robots, and many-to-one
    mask = np.ones(B, dtype=np.int32); mask[[4, 9]] = 0
    handles = [_solver(B) for _ in range(2)]
    try:
        with closed_loop.Session(handles[0], 0.01 * n, **kw) as ss:
            want = _host(ss, ss.step(n)); end_want = ss.finish()
        with closed_loop.Session(handles[1], 0.01 * n, **kw) as ss:
            snap = ss.snapshot()
            ss.restore(snap, mask=torch.as_tensor(mask, device=ss.device), source=torch.as_tensor(source, device=ss.device))
            got = _host(ss, ss.step(n)); end_got = ss.finish()
    finally:
        for s in handles:
            s.close()
    src = np.where(mask != 0, source, np.arange(B))
    if name == "commands":
        assert len(np.unique(want["target_kind"][0])) >= 2 and not np.array_equal(want["target_kind"][0], want["target_kind"][0, src])
    assert len({gaits[b] for b in src}) == 4 and any(gaits[b] != gaits[src[b]] for b in range(B))
    for k in want:
        if k != "t":
            assert got[k].tobytes() == want[k][:, src].tobytes(), k
    for k in ("q", "v", "contact", "episode_metrics"):
        assert end_got[k].tobytes() == end_want[k][src].tobytes(), k


def test_refusals_write_nothing_and_a_bad_source_leaves_its_robot():
    import torch
    from qm_control_b200 import closed_loop
    B = 16
    s = _solver(B)
    try:
        with closed_loop.Session(s, 0.3, gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.0), payload_estimator=True, steer=True) as ss:
            ss.step(5)
            dev = ss.device

            def save():
                buf = torch.empty(B * s.robot_state_bytes(), dtype=torch.uint8, device=dev)
                desc = s.robot_state_save_dev(buf, ss._s); ss.stream.synchronize()
                return buf, desc

            def unchanged(call, match):
                before, _ = save()
                with pytest.raises((_lib.QmbError, ValueError), match=match):
                    call()
                after, _ = save()
                assert torch.equal(before, after)

            old, old_desc = save()
            ss.step(5)
            ones = torch.ones(B, dtype=torch.int32, device=dev)
            # a component reset between save and load
            s.payload_est_reset()
            unchanged(lambda: s.robot_state_load_dev(old, old_desc, ones, stream=ss._s), "payload estimator was reset")
            unchanged(lambda: ss.restore(closed_loop.Snapshot(ss, old, old_desc, [a.clone() for a in ss.rows], torch.zeros(B, dtype=torch.int64, device=dev), 50)),
                      "library refuses")
            # a settings array set for the first time
            cur, cur_desc = save()
            s.set_robot_tuning(dict(kp_swing=350.0))
            unchanged(lambda: s.robot_state_load_dev(cur, cur_desc, ones, stream=ss._s), "tuning rows exists now but was not saved")
            s.set_robot_tuning(None)
            # a short buffer, for the save and for the load
            cur, cur_desc = save()
            unchanged(lambda: s.robot_state_save_dev(cur[:-4], ss._s), "buffer holds")
            unchanged(lambda: s.robot_state_load_dev(cur[:-4], cur_desc, ones, stream=ss._s), "buffer holds")
            # out-of-range sources: those robots untouched with ST_RESTORE, the others restored from their sources
            ss.step(5); now, _ = save()
            source = torch.as_tensor(np.r_[np.arange(B - 4)[::-1], [-1, B, B + 3, -(1 << 31)]].astype(np.int32), device=dev)
            status = torch.full((B,), 7, dtype=torch.int32, device=dev)
            s.robot_state_load_dev(cur, cur_desc, ones, source, status, stream=ss._s); got, _ = save()
            s.robot_state_load_dev(now, cur_desc, ones, stream=ss._s)   # back to now, then only the valid robots
            valid = torch.as_tensor(np.r_[np.ones(B - 4), np.zeros(4)].astype(np.int32), device=dev)
            s.robot_state_load_dev(cur, cur_desc, valid, source, stream=ss._s); want, _ = save()
            assert torch.equal(got, want) and not torch.equal(got, now)
            assert status.cpu().tolist() == [0] * (B - 4) + [_lib.ST_RESTORE] * 4
            # the host twin
            st = s.robot_state_load(cur, cur_desc, np.ones(B), source.cpu().numpy())
            assert st.tolist() == [0] * (B - 4) + [_lib.ST_RESTORE] * 4
            # a session restore with a bad source puts ST_RESTORE into the next window's record
            snap = ss.snapshot(); ss.step(2)
            ss.restore(snap, source=source)
            rec = _host(ss, ss.step(1))
            assert np.all((rec["status"][0, B - 4:] & _lib.ST_RESTORE) != 0) and not np.any(rec["status"][0, :B - 4] & _lib.ST_RESTORE)
            ss.finish()
    finally:
        s.close()


DEMO_BOUND = 0.05   # rad, the heading bound of the session's heading controller test (tests/test_session_gpu.py), fixed before the run


def test_predictive_sampling_on_branches_steers_the_leaders():
    """16 leaders, each branched onto 15 candidates with a grid of yaw rates; after 0.3 s every robot rewinds, each leader takes its best candidate's
    rate for 0.1 s, and again: all in torch on the session's stream, no synchronisation until the end"""
    import torch
    from qm_control_b200 import closed_loop
    L, K = 16, 15; B = L * (K + 1); look, act, cycles = 30, 10, 40
    rates = torch.linspace(-0.6, 0.6, K, dtype=torch.float64)
    goal_h = np.random.default_rng(12).uniform(-1.0, 1.0, L)
    s = _solver(B)
    try:
        with closed_loop.Session(s, 0.01 * (1 + cycles * (look + act)), steer=True, gait="trot", cmd_vel=(0.25, 0.0, 0.0, 0.0)) as ss:
            dev = ss.device
            ss.step(1)   # snapshots from window 1 on: each is taken before its window's MPC tick
            with torch.cuda.stream(ss.stream):
                lead = torch.arange(B, device=dev) // (K + 1) * (K + 1)   # robot b's leader (a leader is its own)
                is_lead = (torch.arange(B, device=dev) % (K + 1) == 0)
                cand = (~is_lead).to(torch.int32); everyone = torch.ones(B, dtype=torch.int32, device=dev)
                goal = torch.as_tensor(goal_h, device=dev).repeat_interleave(K + 1)
                rates = rates.to(dev)   # once: a host-to-device copy inside the cycles would synchronise
                grid = torch.cat([torch.zeros(1, dtype=torch.float64, device=dev), rates]).repeat(L)
                vel = torch.zeros((B, 4), dtype=torch.float64, device=dev); vel[:, 0] = 0.25
            for _ in range(cycles):
                snap = ss.snapshot()
                with torch.cuda.stream(ss.stream):
                    ss.restore(snap, mask=cand, source=lead.to(torch.int32))
                    vel[:, 3] = grid; ss.command(cand, cmd_vel=vel)
                ss.step(look)
                with torch.cuda.stream(ss.stream):
                    err = (torch.remainder(goal - ss.state["q"][:, 3] + np.pi, 2.0 * np.pi) - np.pi).abs().view(L, K + 1)[:, 1:]
                    best = rates[err.argmin(1)].repeat_interleave(K + 1)
                    ss.restore(snap)
                    vel[:, 3] = best; ss.command(everyone, cmd_vel=vel)
                rec = ss.step(act)
            end = ss.finish()
    finally:
        s.close()
    err = np.abs(np.remainder(goal_h - end["q"][::K + 1, 3] + np.pi, 2 * np.pi) - np.pi)
    status = rec["status"].cpu().numpy()
    print("predictive sampling, %d leaders x %d candidates, %d cycles: final heading error max %.4f rad, mean %.4f rad, start max %.3f rad"
          % (L, K, cycles, err.max(), err.mean(), np.abs(goal_h).max()))
    assert not np.any(status & (_lib.ST_COMMAND | _lib.ST_RESTORE))
    assert err.max() < DEMO_BOUND
