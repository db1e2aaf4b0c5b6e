"""Per-robot restart inside the GPU closed loop (closed_loop.run(respawn=...), DESIGN.md §4.10): robots that never respawn are untouched, every
episode of a noise-free run repeats the first bit for bit, a restore writes exactly the image rows of the masked robots, the device fall detector is
the numpy rule, and the loop's calls still replay on the oracle and the plant twin after cold restarts."""
import numpy as np
import pytest

import _loop_replay as R
from _oracle import Oracle
from _respawn_twin import fall_counts, fall_flags
from _sim_twin_terrain import SimTwinTerrain
from qm_control_b200 import _lib
from qm_control_b200 import terrain as T

pytestmark = pytest.mark.gpu

PL = {n: i for i, n in enumerate(_lib.PAYLOAD_LAYOUT)}
WR = {n: i for i, n in enumerate(_lib.WRENCH_LAYOUT)}
REC = ("base", "ee", "status")


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


def _rbd(base):
    """record rows (x, y, z, yaw, pitch, roll) → rbd rows with zyx and p where the plant writes them"""
    r = np.zeros(base.shape[:-1] + (_lib.RBD,)); r[..., 0:3] = base[..., 3:6]; r[..., 3:6] = base[..., 0:3]
    return r


# ---------------- 1 + 4: independence, replay after a fall, the detector ----------------
FB = 64
FALL_S = 1.5


def _fall_setup():
    """16 robots each: trot at 0.3 m/s; trot on mu 0.15 with 2 kg in the gripper and a 180 N lateral push from 0.3 s for 0.1 s; trot blind onto 9 cm
    stairs; trot again"""
    grp = np.arange(FB) // 16
    xy = np.zeros((FB, 3)); xy[:, 0] = 2.0 * (np.arange(FB) % 8); xy[:, 1] = 2.0 * (np.arange(FB) // 8)
    payload = np.zeros((FB, 8)); payload[grp == 1, PL["m_ee"]] = 2.0
    w = np.zeros((FB, 12)); w[grp == 1, WR["f_base_y"]] = 180.0
    ter = dict(tiles=np.stack([T.stairs(0.09, 0.3, start=0.35)]), cell=T.CELL, tile=np.where(grp == 2, 0, -1), origin=T.centred_origin(xy[:, :2]))
    return dict(duration=FALL_S, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, friction_mu=np.where(grp == 1, 0.15, 0.6), payload=payload,
                pushes=(np.full(FB, 0.3), np.full(FB, 0.1), w), terrain=ter)


@pytest.fixture(scope="module")
def fall_runs():
    from qm_control_b200 import closed_loop
    out = {}
    for tag, extra in (("plain", {}), ("respawn", dict(respawn=dict(hold=0.05)))):
        s = _solver(FB)
        try:
            out[tag] = closed_loop.run(s, **_fall_setup(), **extra)
        finally:
            s.close()
    return out


def test_robots_that_never_respawn_are_bit_identical(fall_runs):
    plain, r = fall_runs["plain"], fall_runs["respawn"]
    ep = r["episode"]; stay = ep[-1] == 0
    assert np.any(r["fallen"]) and np.any(ep[-1] > 0), "no robot fell and respawned"
    assert np.any(stay) and np.sum(~stay) >= 4, (int(np.sum(stay)), int(np.sum(~stay)))
    for k in REC:
        np.testing.assert_array_equal(r[k][:, stay], plain[k][:, stay], err_msg=k)
    for k in ("contact", "q", "v"):
        np.testing.assert_array_equal(r[k][stay], plain[k][stay], err_msg=k)
    # a respawned robot's first episode is the plain run's until the window after its restart was decided
    for b in np.flatnonzero(~stay):
        n0 = int(np.argmax(ep[:, b] > 0))
        for k in REC:
            np.testing.assert_array_equal(r[k][:n0, b], plain[k][:n0, b], err_msg="%s robot %d" % (k, b))


def test_later_episodes_repeat_the_first_after_a_fall(fall_runs):
    r = fall_runs["respawn"]; ep = r["episode"]; checked = 0
    for b in np.flatnonzero(ep[-1] > 0):
        len0 = int(np.sum(ep[:, b] == 0))
        for e in range(1, ep[-1, b] + 1):
            rows = np.flatnonzero(ep[:, b] == e); n = min(len(rows), len0)
            assert np.all(np.diff(rows) == 1)
            for k in REC:
                np.testing.assert_array_equal(r[k][rows[:n], b], r[k][:n, b], err_msg="%s robot %d episode %d" % (k, b, e))
            checked += n
    assert checked > 0


def test_device_detector_is_the_numpy_rule(fall_runs):
    r = fall_runs["respawn"]; ter = _fall_setup()["terrain"]
    flags = fall_flags(_rbd(r["base"]), ter)
    np.testing.assert_array_equal(r["fallen"].astype(bool), flags)                  # in the loop, on the plant's rbd
    assert np.any(flags[:, ter["tile"] == 0]) and np.any(flags[:, ter["tile"] == -1])
    s = _solver(FB)
    try:
        s.sim_set_terrain(ter["tiles"], ter["cell"]); s.sim_set_robot_terrain(ter["tile"], ter["origin"])
        count = np.zeros(FB, dtype=np.int32); counts = fall_counts(flags)
        for i, row in enumerate(_rbd(r["base"])):
            count, fallen = s.fall_detect(row, count)
            np.testing.assert_array_equal(fallen.astype(bool), flags[i], err_msg="tick %d" % i)
            np.testing.assert_array_equal(count, counts[i], err_msg="tick %d" % i)
        nan = _rbd(r["base"][0]); nan[3, 5] = np.nan; nan[4, 1] = np.inf
        _, fallen = s.fall_detect(nan, np.zeros(FB, dtype=np.int32))
        assert fallen[3] == 1 and fallen[4] == 1
        for bad in (dict(z_min=np.nan), dict(tilt_max=0.0), dict(tilt_max=np.inf)):
            with pytest.raises(_lib.QmbError):
                s.fall_detect(nan, np.zeros(FB, dtype=np.int32), **bad)
    finally:
        s.close()


# ---------------- 2: exact replay of every episode ----------------
EB = 16
EVERY_S, EPISODES = 0.2, 3


def _replay_case(case):
    xy = np.zeros((EB, 3)); xy[:, 0] = 2.0 * np.arange(EB)
    tiles = np.stack([T.ramp(5.0, start=0.35), T.stairs(0.03, 0.3, start=0.35)])
    ter = dict(tiles=tiles, cell=T.CELL, tile=np.arange(EB) % 3 - 1, origin=T.centred_origin(xy[:, :2]))
    kw = dict(duration=EVERY_S * EPISODES, xy_yaw=xy, respawn=dict(on_fall=False, every=EVERY_S))
    if case == "truth":
        w = np.zeros((EB, 12)); w[:, WR["f_base_y"]] = 60.0
        payload = np.zeros((EB, 8)); payload[::2, PL["m_ee"]] = 1.0
        goal = np.full((EB, 2, 7), np.nan); goal[:, 1] = np.c_[xy[:, 0] + 0.52, xy[:, 1] + 0.09, np.full(EB, 0.49), np.tile([0.5, -0.5, 0.5, -0.5], (EB, 1))]
        commands = dict(t=np.tile([0.05, 0.1], (EB, 1)), gait=np.tile(np.array(["trot", None], dtype=object), (EB, 1)), ee_goal=goal)
        return dict(kw, gait="stance", pushes=(np.full(EB, 0.03), np.full(EB, 0.05), w), payload=payload, payload_estimator=True, commands=commands, terrain=ter), {}
    if case == "estimate":
        return dict(kw, gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.0), state_estimator=True, attitude_filter=True, slip_detector=True, terrain=ter, ground_map=True), {}
    return dict(kw, gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.0)), dict(wbc_variant=1)


@pytest.mark.parametrize("case", ["truth", "estimate", "mpc_wbc_variant"])
def test_every_episode_repeats_the_first_bit_for_bit(case):
    from qm_control_b200 import closed_loop
    kw, skw = _replay_case(case)
    s = _solver(EB, **skw)
    try:
        r = closed_loop.run(s, **kw)
    finally:
        s.close()
    n = int(round(EVERY_S * 100))
    np.testing.assert_array_equal(r["episode"], np.repeat(np.arange(EPISODES), n)[:, None] * np.ones((1, EB), dtype=np.int32))
    keys = REC + (("gait", "mode", "target_kind", "ee_target", "payload_est") if case == "truth" else ("base_est", "slip") if case == "estimate" else ())
    for k in keys:
        for e in range(1, EPISODES):
            np.testing.assert_array_equal(r[k][e * n:(e + 1) * n], r[k][:n], err_msg="%s episode %d" % (k, e))
    assert not np.any(r["fallen"]) and np.all(r["status"] & 0xFF == 0)
    if case == "truth":
        assert np.any(r["target_kind"] == _lib.TARGET_EE_GOAL) and len(np.unique(r["gait"])) > 1
        assert np.any(r["payload_est"][n - 1, ::2, 0] > 0.2)


# ---------------- 3: what a restore writes ----------------
def _getters(s):
    se, at, sl, pe, gd = s.state_est_get(), s.attitude_get(), s.slip_get(), s.payload_est_get(), s.gait_dev_get()
    out = {"se_" + k: v for k, v in se.items()}
    out.update({"at_" + k: v for k, v in at.items()}); out.update({"sl_" + k: v for k, v in sl.items()}); out.update({"pe_" + k: v for k, v in pe.items()})
    out.update({"gd_" + k: v for k, v in gd.items()}); out["model"] = s.get_model_payload()
    out["n_nodes"] = s.mpc_get_solution()["n_nodes"]; out["input_last"] = s.wbc_get_input_last()
    return out


def test_restore_writes_the_image_rows_of_masked_robots_only():
    import torch
    from qm_control_b200 import closed_loop
    B = 32; rng = np.random.default_rng(7); s = _solver(B); snaps = {}; calls = []
    orig_save, orig_restore = s.robot_image_save, s.robot_image_restore_dev

    def save():
        orig_save(); snaps["image"] = _getters(s)

    def restore(mask, stream=None):
        calls.append(1)
        if len(calls) != 6:
            return orig_restore(mask, stream)
        mask.copy_(torch.as_tensor(rng.integers(0, 2, B), dtype=torch.int32, device=mask.device))   # the loop restores its own rows with it too
        torch.cuda.synchronize(); snaps["mask"] = mask.cpu().numpy().astype(bool); snaps["before"] = _getters(s)
        orig_restore(mask, stream); torch.cuda.synchronize(); snaps["after"] = _getters(s)
    s.robot_image_save, s.robot_image_restore_dev = save, restore
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * np.arange(B)
    try:
        closed_loop.run(s, duration=0.1, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), xy_yaw=xy, state_estimator=True, sensor_noise="reference", attitude_filter=True,
                        slip_detector=True, payload_estimator=True, commands=dict(t=np.full((B, 1), 0.02), gait=np.full((B, 1), "trot", dtype=object)),
                        respawn=dict(on_fall=False, every=1.0))
    finally:
        s.close()
    m, img, bef, aft = snaps["mask"], snaps["image"], snaps["before"], snaps["after"]
    assert 0 < m.sum() < B
    for k in img:
        if k in ("n_nodes", "input_last"):
            assert np.all(aft[k][m] == 0), k
        else:
            np.testing.assert_array_equal(aft[k][m], img[k][m], err_msg=k)
        np.testing.assert_array_equal(aft[k][~m], bef[k][~m], err_msg=k)
    for k in ("se_samples", "at_samples", "pe_samples", "se_x", "at_quat", "n_nodes", "input_last"):   # the restore had something to change
        assert np.any(bef[k][m] != aft[k][m]), k


def test_restore_refuses_a_stale_image_and_writes_nothing():
    B = 8; s = _solver(B); rng = np.random.default_rng(3)
    try:
        q0, v0 = s.sim_standing_state(np.zeros((B, 3)))
        with pytest.raises(_lib.QmbError, match="no start image"):
            s.robot_image_restore(np.ones(B, dtype=np.int32))
        s.state_est_reset(q0[:, 0:3]); s.attitude_reset(); s.robot_image_save()
        s.attitude_step(1e-3, s.sim_read_sensors(1e-3, 0, q0, v0, v0))   # the filter now differs from its image
        il = rng.standard_normal((B, _lib.NU)); s.wbc_set_input_last(il); at = s.attitude_get()
        s.state_est_stop()
        with pytest.raises(_lib.QmbError, match="state estimator"):
            s.robot_image_restore(np.ones(B, dtype=np.int32))
        s.state_est_reset(q0[:, 0:3])   # a reset leaves the image stale too
        with pytest.raises(_lib.QmbError, match="state estimator"):
            s.robot_image_restore(np.ones(B, dtype=np.int32))
        for k, v in s.attitude_get().items():
            np.testing.assert_array_equal(v, at[k], err_msg=k)
        np.testing.assert_array_equal(s.wbc_get_input_last(), il)
        s.robot_image_save(); s.slip_reset()
        with pytest.raises(_lib.QmbError, match="slip detector runs but was not imaged"):
            s.robot_image_restore(np.ones(B, dtype=np.int32))
        s.slip_stop(); s.robot_image_restore(np.arange(B) % 2)
        np.testing.assert_array_equal(s.wbc_get_input_last()[1::2], 0.0); np.testing.assert_array_equal(s.wbc_get_input_last()[0::2], il[0::2])
        s.robot_image_clear(); s.robot_image_clear()
        with pytest.raises(_lib.QmbError, match="no start image"):
            s.robot_image_restore(np.ones(B, dtype=np.int32))
    finally:
        s.close()


# ---------------- 5: the replay harness across cold restarts ----------------
def test_respawn_run_replays_call_by_call():
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    B = 30; grp = np.arange(B) // 10
    xy = np.zeros((B, 3)); xy[:, 0] = 0.5 * np.arange(B)
    w = np.zeros((B, 12)); w[grp == 2, WR["f_base_y"]] = 150.0
    kw = dict(duration=0.3, gait=["stance" if g == 2 else "trot" for g in grp], cmd_vel=np.where((grp == 1)[:, None], [0.3, 0.0, 0.0, 0.0], 0.0), xy_yaw=xy,
              pushes=(np.full(B, 0.03), np.full(B, 0.05), w), respawn=dict(hold=0.02, every=0.1))
    s = q.Solver(batch=B, device=0)
    try:
        res, rec = R.record(s, lambda: closed_loop.run(s, **kw))
    finally:
        s.close()
    assert res["episode"][-1].min() == 2
    oracles = [Oracle()] * B
    out = dict(targets=R.replay_targets(rec), mpc=R.replay_mpc(rec, oracles), update=R.replay_update(rec, oracles), plant=R.replay_plant(rec, SimTwinTerrain(), every=3))
    cold = sum(int(np.sum(i["before"]["n_nodes"] < 2)) for i, _ in rec.of("mpc"))
    assert cold >= 3 * B, cold                          # the first solve and one after each restart
    assert out["mpc"]["replayed"] >= 0.9 * len(rec.of("mpc")) * B and out["update"]["replayed"] == 150 * B and out["plant"]["pushed"] > 0, out
