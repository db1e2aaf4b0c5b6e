"""End-effector targets in the robot's heading frame on the GPU (DESIGN.md §4.19): the device target call against the host build, world-frame rows
byte-identical to no rows, a turning trot through +-pi with the hand held on the body, stance and walking reaches at spread headings, drawn spawn yaws
and restarts with end-effector goals, and snapshots that carry the frame."""
import numpy as np
import pytest

import qm_control_b200 as q
from qm_control_b200 import _lib, closed_loop
from test_ee_commands_gpu import (STANCE_ORI_DEG, STANCE_ORI_DEG_P50, STANCE_POS_M, STANCE_POS_M_P50, WALK_ORI_DEG, WALK_POS_M, _start_ee, _up, axis_angle,
                                  ori_err_deg, quat_mul)
from test_ee_frame_cpu import h_from_world, h_to_world, host, host_target, robots  # noqa: F401  (host: the host build's fixture)
from test_session_gpu import _same

pytestmark = pytest.mark.gpu
KMAX, TD = _lib.KMAX, _lib.TARGET


def _dev(a, dtype=None):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype or torch.float64, device="cuda")


def test_device_target_call_equals_the_host_build(host):
    """4096 robots of every kind (-1 held) and both frames at unwrapped yaws up to +-50 rad: the device call equals the host build to 1e-12 (the device's
    sincospi is not the host's sin); world robots are byte-identical to the call without rows and with all-world rows; held robots are untouched."""
    import torch
    B = 4096; s = q.Solver(batch=B)
    kind, frame, cmd, t, x, ee, le = robots(B, 61)

    def call(rows):
        s.set_ee_frame(rows)
        out = [_dev(le), _dev(np.full(B, -7), torch.int32), _dev(np.full((B, KMAX), np.nan)), _dev(np.full((B, KMAX, TD), np.nan))]
        torch.cuda.synchronize()
        s.target_trajectories_dev(_dev(kind, torch.int32), _dev(cmd), _dev(t), _dev(x), _dev(ee), *out)
        torch.cuda.synchronize()
        le_o, nt, tt, ts = (a.cpu().numpy() for a in out)
        return nt, tt, ts, le_o
    got, none, world = call(frame), call(None), call(np.zeros(B))
    assert s.get_ee_frame() is not None and np.all(s.get_ee_frame() == 0)
    s.set_ee_frame(None); assert s.get_ee_frame() is None
    want = host_target(host, kind, frame, cmd, t, x, ee, le)
    held, w = kind < 0, frame == 0
    assert np.all(got[0][held] == -7) and np.all(np.isnan(got[2][held])) and got[3][held].tobytes() == le[held].tobytes()
    for a, b, c in zip(got, none, world):
        assert a[w].tobytes() == b[w].tobytes() == c[w].tobytes() and b.tobytes() == c.tobytes()
    assert np.array_equal(got[0], want[0])
    for a, b in zip(got[1:], want[1:]):
        np.testing.assert_allclose(a[~held], b[~held], rtol=0, atol=1e-12)
    with pytest.raises(_lib.QmbError, match="frame of robot 3 is 2"):
        s.set_ee_frame(np.r_[0, 1, 0, 2, np.zeros(B - 4)].astype(np.int32))
    assert s.get_ee_frame() is None   # the refused rows wrote nothing
    s.close()


def test_a_loop_with_all_world_rows_is_byte_identical_to_one_without():
    B = 16; s = q.Solver(batch=B); xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.linspace(-3, 3, B)]
    runs = []
    for kw in ({}, dict(ee_frame=np.zeros(B, dtype=np.int32))):
        s.mpc_reset(); s.wbc_set_input_last(None)
        runs.append(closed_loop.run(s, duration=0.3, gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.5), xy_yaw=xy, **kw))
    _same(*runs); assert s.get_ee_frame() is None
    s.close()


def test_a_heading_frame_robot_turns_through_pi():
    """DESIGN.md §8's first failing turn: 16 robots trotting 0.3 m/s at +0.5 rad/s from pi - 0.1 (+-1 mrad), 4 s, stepped window by window.  In the
    world frame no robot reaches pi; in the heading frame every robot stays up with no status bit and passes pi, its hand stays within the 0.1 m
    re-anchor distance of its current hold, and that hold (in H) moves by no more than the one re-anchor at the start.  The turn at +1 rad/s, where the
    hold ratchets across the body, is a measured finding in DESIGN.md §4.19."""
    B = 16; s = q.Solver(batch=B)
    xy = np.c_[np.arange(B) * 3.0, np.zeros(B), np.pi - 0.1 + np.linspace(-1e-3, 1e-3, B)]
    with closed_loop.Session(s, 4.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.5), xy_yaw=xy, ee_frame="heading") as ss:
        yaws, st, d_hand, le0 = [], np.zeros(B, dtype=np.int64), np.zeros(B), None
        for _ in range(ss.windows):
            rec = ss.step(1); ss.stream.synchronize()
            base = rec["base"][0].cpu().numpy(); ee = rec["ee"][0].cpu().numpy(); le = ss.last_ee.cpu().numpy(); st |= rec["status"][0].cpu().numpy()
            le0 = le.copy() if le0 is None else le0
            hand = h_from_world(base[:, 0], base[:, 1], base[:, 3], ee)
            d_hand = np.maximum(d_hand, np.linalg.norm(hand[:, :3] - le[:, :3], axis=1)); yaws.append(base[:, 3])
        ss.finish()
    yaw = np.unwrap(np.array(yaws), axis=0); moved = np.linalg.norm(le[:, :3] - le0[:, :3], axis=1)
    print("heading frame at +0.5 rad/s from pi - 0.1: final yaw %.2f..%.2f, status bits %s, hand to hold worst %.4f m, hold moved %.4f m" % (
        yaw[-1].min(), yaw[-1].max(), np.unique(st), d_hand.max(), moved.max()))
    assert np.all(st == 0) and np.all(np.abs(base[:, 2]) > 0.3) and np.all(yaw[-1] > np.pi + 1.0)
    assert d_hand.max() < 0.11 and moved.max() < 0.11
    s.close()


def _spread(B):
    return np.c_[np.arange(B) * 2.0, np.zeros(B), -np.pi + 2 * np.pi * np.arange(B) / B]


def _published(r):
    """each robot's goal as its target call published it in the world (the record whose target kind is 2)"""
    i = np.argmax(r["target_kind"] == 2, axis=0)
    assert np.all(np.sum(r["target_kind"] == 2, axis=0) == 1)
    return r["ee_target"][i, np.arange(r["ee_target"].shape[1])]


def _bins(yaw, err, name):
    edges = np.linspace(-np.pi, np.pi, 9)
    med = [np.median(err[(yaw >= a) & (yaw < b)]) for a, b in zip(edges[:-1], edges[1:])]
    print("%s median per 45-deg heading bin: %s" % (name, " ".join("%.4f" % m for m in med)))


def test_stance_reach_at_any_heading():
    """test_ee_commands_gpu's stance reach with the goals stated in the heading frame and 64 start yaws over [-pi, pi): the same bounds."""
    rng = np.random.default_rng(31); B = 64; s = q.Solver(batch=B); xy = _spread(B)
    ee0 = _start_ee(s, xy)
    ee0_h = h_from_world(xy[:, 0], xy[:, 1], xy[:, 2], ee0)
    goal = ee0_h.copy(); goal[:, :3] += rng.uniform(-0.1, 0.1, (B, 3))
    goal[:, 3:] = quat_mul(axis_angle(rng.normal(size=(B, 3)), np.radians(rng.uniform(0, 15, B))), ee0_h[:, 3:])
    r = closed_loop.run(s, duration=5.0, gait="stance", xy_yaw=xy, ee_frame="heading",
                        commands=dict(t=np.full((B, 1), 0.2), gait=np.full((B, 1), None, dtype=object), ee_goal=goal[:, None]))
    gw = _published(r); ee = r["ee"][-10:]
    pe = np.max(np.linalg.norm(ee[:, :, :3] - gw[None, :, :3], axis=2), axis=0); oe = np.max(ori_err_deg(ee[:, :, 3:], gw[None, :, 3:]), axis=0)
    print("stance reach at spread headings: position p50 %.4f max %.4f m, orientation p50 %.2f max %.2f deg, status %s, up %d / %d" % (
        np.median(pe), pe.max(), np.median(oe), oe.max(), np.unique(r["status"]), _up(r).sum(), B))
    _bins(xy[:, 2], pe, "stance position error (m)"); _bins(xy[:, 2], oe, "stance orientation error (deg)")
    assert np.all(_up(r)) and np.all(r["status"] == 0)
    assert pe.max() < STANCE_POS_M and oe.max() < STANCE_ORI_DEG and np.median(pe) < STANCE_POS_M_P50 and np.median(oe) < STANCE_ORI_DEG_P50
    s.close()


def test_walk_to_reach_at_any_heading():
    """test_ee_commands_gpu's walk to reach with the goals 0.3-0.5 m ahead along each robot's own heading, 64 start yaws over [-pi, pi)."""
    rng = np.random.default_rng(41); B = 64; s = q.Solver(batch=B); xy = _spread(B)
    ee0 = _start_ee(s, xy)
    goal = h_from_world(xy[:, 0], xy[:, 1], xy[:, 2], ee0); goal[:, 0] += rng.uniform(0.3, 0.5, B)
    nan7 = np.full((B, 7), np.nan)
    commands = dict(t=np.tile([0.2, 2.5], (B, 1)), gait=np.tile(np.array([None, "stance"], dtype=object), (B, 1)), ee_goal=np.stack([goal, nan7], 1))
    r = closed_loop.run(s, duration=5.0, gait="trot", xy_yaw=xy, commands=commands, ee_frame="heading")
    gw = _published(r); ee = r["ee"][-10:]
    pe = np.max(np.linalg.norm(ee[:, :, :3] - gw[None, :, :3], axis=2), axis=0); oe = np.max(ori_err_deg(ee[:, :, 3:], gw[None, :, 3:]), axis=0)
    print("walk to reach at spread headings: position p50 %.4f max %.4f m, orientation p50 %.2f max %.2f deg, status %s, up %d / %d" % (
        np.median(pe), pe.max(), np.median(oe), oe.max(), np.unique(r["status"]), _up(r).sum(), B))
    _bins(xy[:, 2], pe, "walk position error (m)"); _bins(xy[:, 2], oe, "walk orientation error (deg)")
    assert np.all(_up(r)) and np.all(r["status"] == 0)
    assert pe.max() < WALK_POS_M and oe.max() < WALK_ORI_DEG
    s.close()


def test_drawn_yaws_and_restarts_go_with_end_effector_goals():
    """A drawn spawn yaw, a restart every 1 s and an ee_goal timeline, in the heading frame, stepped window by window: every published goal is
    H(observation at its tick) applied to one of the robot's drawn slots, to 1e-9.  A Session restarting "here" takes command(ee_goal=...)."""
    import torch
    B = 16; s = q.Solver(batch=B); TL = {n: i for i, n in enumerate(_lib.TIMELINE_CMD_LAYOUT)}
    tl = dict(seed=3, n=3, t_first=(0.1, 0.2), gap=(0.2, 0.3), weights=dict(none=0.2, ee_goal=1.0), ee_x=(0.45, 0.6), ee_y=(-0.05, 0.15),
              ee_z=(0.35, 0.5), ee_quat=(0.5, -0.5, 0.5, -0.5))
    xy = np.c_[np.arange(B) * 3.0, np.zeros(B), np.zeros(B)]
    found = 0
    with closed_loop.Session(s, 3.0, gait="stance", xy_yaw=xy, spawn=dict(seed=5, yaw=(-np.pi, np.pi)), respawn=dict(every=1.0), timeline=tl,
                             ee_frame="heading") as ss:
        obs, kinds, targets, episodes = [], [], [], []
        for _ in range(ss.windows):
            st = ss.state; ss.stream.synchronize()
            obs.append(st["x_obs"].cpu().numpy().copy()); episodes.append(st["episode"].cpu().numpy().copy())
            rec = ss.step(1); ss.stream.synchronize()
            kinds.append(rec["target_kind"][0].cpu().numpy()); targets.append(rec["ee_target"][0].cpu().numpy())
        ep_after = [e for e in episodes[1:]] + [episodes[-1]]
        end = ss.finish()
    slots = end["timeline_params"]   # [B, E, n, TIMELINE_CMD], goals in the heading frame
    for i, (x, k, tg, e0, e1) in enumerate(zip(obs, kinds, targets, episodes, ep_after)):
        for b in np.nonzero((k == 2) & (e0 == e1))[0]:   # a restart at this boundary writes a new observation before the tick
            c = h_from_world(x[b:b + 1, 6], x[b:b + 1, 7], x[b:b + 1, 9], tg[b:b + 1])[0]
            rows = slots[b, e0[b]][:, TL["ee_0"]:TL["ee_0"] + 7]
            assert np.min(np.max(np.abs(rows - c), axis=1)) < 1e-9, (i, b, c, rows)
            found += 1
    print("published goals checked: %d, spawn yaws %s" % (found, np.round(end["spawn_params"][:, :, 3][:4], 2)))
    assert found >= B and np.ptp(end["spawn_params"][:, 0, 3]) > 1.0
    with closed_loop.Session(s, 0.05, gait="stance", xy_yaw=xy, steer=True, respawn=dict(every=0.02, at="here"), ee_frame="heading") as ss:
        ss.step(1)
        goal = np.tile([0.55, 0.05, 0.45, 0.5, -0.5, 0.5, -0.5], (B, 1))
        ss.command(torch.ones(B, dtype=torch.int32, device="cuda"), ee_goal=goal)   # accepted: a world session refuses it
        st_x = ss.state["x_obs"].clone(); ss.stream.synchronize()   # the observation the next tick publishes from
        rec = ss.step(1); ss.stream.synchronize()   # the records are enqueued on the session's stream
        kinds = rec["target_kind"].cpu().numpy(); tgt = rec["ee_target"][0].cpu().numpy(); x = st_x.cpu().numpy()
        assert np.all(kinds == 2), kinds   # the accepted goal is published by the tick that opens the step
        np.testing.assert_allclose(tgt, h_to_world(x[:, 6], x[:, 7], x[:, 9], goal), rtol=0, atol=1e-9)
        ss.finish()
    s.close()


def test_snapshots_replay_and_branches_carry_the_frame():
    """Mixed frames, trotting and turning: a rewind replays byte for byte; a heading robot branched onto a world robot takes its frame and hold."""
    import torch
    B = 8; s = q.Solver(batch=B); frame = np.array([1, 0] * 4, dtype=np.int32)
    xy = np.c_[np.arange(B) * 3.0, np.zeros(B), np.linspace(-2, 2, B)]
    with closed_loop.Session(s, 0.4, gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.6), xy_yaw=xy, ee_frame=frame) as ss:
        host = lambda rec: (ss.stream.synchronize(), {k: v.cpu().numpy() for k, v in rec.items() if hasattr(v, "cpu")})[1]   # records are enqueued on ss.stream
        ss.step(5); snap = ss.snapshot()
        a = host(ss.step(10))
        ss.restore(snap)
        b = host(ss.step(10))
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
        li = [i for i, r in enumerate(ss.rows) if r is ss.last_ee][0]
        ss.restore(snap, mask=torch.tensor([0, 1] + [0] * (B - 2), dtype=torch.int32, device="cuda"),
                   source=torch.tensor([0] * B, dtype=torch.int32, device="cuda"))
        ss.stream.synchronize()
        assert s.get_ee_frame().tolist() == [1, 1] + frame[2:].tolist()   # the branched robot shows its source's frame
        assert ss.last_ee[1].cpu().numpy().tobytes() == snap.rows[li][0].cpu().numpy().tobytes()
        ss.step(5); ss.finish()
    assert s.get_ee_frame() is None
    s.close()


def test_a_heading_turn_replays_call_by_call_on_the_host_build(host):
    """0.3 s of 16 robots trotting at +1 rad/s from yaws near +-pi, frames mixed, with every target call recorded (tests/_loop_replay.py): each call
    restated by the host build from its recorded inputs gives the recorded outputs to 1e-12."""
    import _loop_replay as R
    B = 16; s = q.Solver(batch=B); frame = (np.arange(B) % 4 != 0).astype(np.int32)
    xy = np.c_[np.arange(B) * 3.0, np.zeros(B), np.pi - 0.05 + 0.1 * np.arange(B) / B]
    _, rec = R.record(s, lambda: closed_loop.run(s, duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 1.0), xy_yaw=xy, ee_frame=frame))
    calls = rec.of("targets"); worst = 0.0; crossed = False
    for i, (inp, out) in enumerate(calls):
        kind = np.broadcast_to(np.asarray(inp["kind"], dtype=np.int32), (B,))
        nt, tt, ts, le = host_target(host, kind, frame, inp["cmd"], inp["t_obs"], inp["x_obs"], inp["ee_state"], inp["last_ee_target"])
        assert np.array_equal(nt, out["n_target"]), i
        for a, b in ((tt, out["target_times"]), (ts, out["target_states"]), (le, out["last_ee_target"])):
            e = np.max(np.abs(a - b)); worst = max(worst, e)
            assert e <= 1e-12, (i, e)
        crossed |= bool(np.any(np.abs(inp["x_obs"][:, 9]) > np.pi))
    print("replayed %d target calls of %d robots, worst %.2e, unwrapped yaw past pi: %s" % (len(calls), B, worst, crossed))
    assert len(calls) == 30 and crossed
    s.close()
