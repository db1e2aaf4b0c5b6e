"""Per-episode plant draws inside the GPU closed loop (closed_loop.run(randomize=...), DESIGN.md §4.11): the device sampler is the host draw bit for bit
and writes only what its mask and links say, a spec that names no field changes nothing, and every drawn episode is the first episode of a run fixed
at its row."""
import numpy as np
import pytest

import _episode_twin as tw
from qm_control_b200 import _lib
from qm_control_b200 import terrain as T

pytestmark = pytest.mark.gpu

EP = {n: i for i, n in enumerate(_lib.EPISODE_LAYOUT)}
REC = ("base", "ee", "status")


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


def _random_ranges(rng, B):
    lo = rng.uniform(-1.0, 1.0, (B, _lib.EPISODE)); hi = lo + rng.uniform(0.0, 1.0, (B, _lib.EPISODE))
    for f in ("friction_mu", "m_ee", "m_base", "push_t_on", "push_duration"):
        lo[:, EP[f]] = rng.uniform(0.1, 0.5, B); hi[:, EP[f]] = lo[:, EP[f]] + rng.uniform(0.0, 2.0, B)
    lo[::7] = hi[::7]   # some robots fixed
    return lo, hi


def _state(s):
    rp = s.sim_get_robot_params(); tn = s.get_robot_tuning()
    return dict(mu=rp["friction_mu"], payload=rp["payload"], model=s.get_model_payload(), ranges=s.episode_get_ranges(),
                tuning=None if tn is None else np.c_[tn["friction_mu"], tn["wbc_friction"], tn["mu_ee_pos"]])


def _same(a, b):
    for k in a:
        if isinstance(a[k], dict):
            _same(a[k], b[k])
        elif a[k] is None:
            assert b[k] is None, k
        else:
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


# ---------------- 1: the sampler ----------------
SB = 4096


def test_sample_dev_is_the_host_draw_and_writes_what_its_mask_and_links_say():
    import torch
    rng = np.random.default_rng(21); s = _solver(SB); ref = _solver(SB)
    try:
        lo, hi = _random_ranges(rng, SB); seed = 2 ** 64 - 12345
        for bad in (dict(f=EP["friction_mu"], lo=0.0), dict(f=EP["o_ee_x"], lo=2.0), dict(f=EP["push_duration"], lo=-0.1)):
            l2 = lo.copy(); l2[9, bad["f"]] = bad["lo"]
            with pytest.raises(_lib.QmbError, match="%s of robot 9" % _lib.EPISODE_LAYOUT[bad["f"]]):
                s.episode_set_ranges(l2, hi, seed)
            assert s.episode_get_ranges() is None and s.sim_get_robot_params()["friction_mu"] is None   # nothing stored, no rows made
        with pytest.raises(_lib.QmbError, match="no ranges"):
            s.episode_sample(np.ones(SB), np.zeros(SB))
        s.episode_set_ranges(lo, hi, seed)
        got = s.episode_get_ranges(); assert got["seed"] == seed and got["lo"].tobytes() == lo.tobytes() and got["hi"].tobytes() == hi.tobytes()
        rp = s.sim_get_robot_params(); np.testing.assert_array_equal(rp["friction_mu"], s.sim_get_params()["friction_mu"]); np.testing.assert_array_equal(rp["payload"], 0.0)
        with pytest.raises(_lib.QmbError, match="hi - lo must be finite"):
            l2 = lo.copy(); h2 = hi.copy(); l2[3, EP["f_ee_x"]] = -1.5e308; h2[3, EP["f_ee_x"]] = 1.5e308; s.episode_set_ranges(l2, h2, 1)
        assert s.episode_get_ranges()["lo"].tobytes() == lo.tobytes() and s.episode_get_ranges()["seed"] == seed   # the stored ranges stay
        model0 = np.c_[rng.uniform(0, 1, (SB, 4)), rng.uniform(0, 1, (SB, 4))] * [1, 0.1, 0.1, 0.1, 1, 0.1, 0.1, 0.1]
        qs, vs = s.sim_standing_state(np.zeros((SB, 3))); _, _, rbd, _, _ = s.sim_step(1e-3, np.zeros((SB, 18)), qs, vs)
        dev = torch.device("cuda:0")
        rows = torch.full((SB, _lib.EPISODE), np.nan, dtype=torch.float64, device=dev)
        # refusals write nothing
        mask = torch.ones(SB, dtype=torch.int32, device=dev); ep = torch.zeros_like(mask)
        before = _state(s)
        for link, match in ((_lib.EPISODE_MODEL_PAYLOAD, "needs a model payload"), (_lib.EPISODE_MPC_FRICTION, "need tuning rows"), (8, "unknown link bits")):
            with pytest.raises(_lib.QmbError, match=match):
                s.episode_sample_dev(mask, ep, rows, link)
        s.set_model_payload(model0); s.payload_est_reset()
        with pytest.raises(_lib.QmbError, match="payload estimator runs"):
            s.episode_sample_dev(mask, ep, rows, _lib.EPISODE_MODEL_PAYLOAD)
        s.payload_est_stop(); s.set_model_payload(model0)
        torch.cuda.synchronize(); assert torch.all(torch.isnan(rows))
        after = _state(s); before["model"] = model0; _same(before, after)
        s.set_robot_tuning(dict(friction_mu=0.3, wbc_friction=0.4))
        for link in (0, _lib.EPISODE_MODEL_PAYLOAD, _lib.EPISODE_MPC_FRICTION, _lib.EPISODE_WBC_FRICTION, 7):
            prev = _state(s); prev_rows = rows.cpu().numpy()
            m = rng.integers(0, 2, SB).astype(np.int32); e = rng.integers(0, 1 << 31, SB).astype(np.int32)
            s.episode_sample_dev(torch.as_tensor(m, device=dev), torch.as_tensor(e, device=dev), rows, link)
            now = _state(s); r = rows.cpu().numpy(); on = m != 0
            want = s.episode_draw(np.flatnonzero(on), e[on])
            assert r[on].tobytes() == want.tobytes(), link
            assert r[~on].tobytes() == prev_rows[~on].tobytes()
            assert now["mu"][on].tobytes() == want[:, 0].tobytes() and now["payload"][on].tobytes() == want[:, 1:9].tobytes()
            assert now["mu"][~on].tobytes() == prev["mu"][~on].tobytes() and now["payload"][~on].tobytes() == prev["payload"][~on].tobytes()
            model_want = prev["model"].copy()
            if link & _lib.EPISODE_MODEL_PAYLOAD:
                model_want[on] = want[:, 1:9]
            assert now["model"].tobytes() == model_want.tobytes(), link
            tn_want = prev["tuning"].copy()
            if link & _lib.EPISODE_MPC_FRICTION:
                tn_want[on, 0] = want[:, 0]
            if link & _lib.EPISODE_WBC_FRICTION:
                tn_want[on, 1] = want[:, 0]
            assert now["tuning"].tobytes() == tn_want.tobytes(), link
            if link & 1:   # the SRBD rows the kernels read are the host's fold of the drawn rows (as test_commit_writes_the_host_fold_and_keeps_the_base_half)
                ref.set_model_payload(now["model"])
                x, x_ref = s.centroidal_state_from_rbd(rbd), ref.centroidal_state_from_rbd(rbd)
                assert np.max(np.abs(x - x_ref)) <= 1e-14 * max(1.0, np.max(np.abs(x_ref)))
        # the host twin of the draw
        b = np.arange(0, SB, 97); e = np.arange(len(b)) * 1000003 % (1 << 31)
        np.testing.assert_array_equal(s.episode_draw(b, e), tw.rows(lo[b], hi[b], np.full(len(b), seed, dtype=np.uint64), b, e))
        s.episode_set_ranges(None)
        assert s.episode_get_ranges() is None
        with pytest.raises(_lib.QmbError, match="no ranges"):
            s.episode_draw([0], [0])
    finally:
        s.close(); ref.close()


def test_a_handle_with_ranges_tears_down_cleanly_and_keeps_fixed_columns_byte_for_byte():
    """The range buffers belong to the handle's allocations and are freed once: after a handle with ranges is closed, a fresh handle's checked device
    calls succeed.  A fixed column of -0.0 is drawn as -0.0 on the device, as on the host."""
    import torch
    B = 64; dev = torch.device("cuda:0")
    for _ in range(2):
        s = _solver(B)
        try:
            lo = np.zeros((B, _lib.EPISODE)); lo[:, EP["friction_mu"]] = 0.5; hi = lo.copy(); hi[:, EP["cmd_vel_x"]] = 0.4
            lo[:, EP["f_base_y"]] = hi[:, EP["f_base_y"]] = -0.0
            s.episode_set_ranges(lo, hi, 3)
            rows = torch.zeros((B, _lib.EPISODE), dtype=torch.float64, device=dev); mask = torch.ones(B, dtype=torch.int32, device=dev)
            s.episode_sample_dev(mask, torch.zeros_like(mask), rows, 0); torch.cuda.synchronize()
            r = rows.cpu().numpy()
            assert r.tobytes() == s.episode_draw(np.arange(B), np.zeros(B)).tobytes() and np.all(np.signbit(r[:, EP["f_base_y"]]))
        finally:
            s.close()
    s = _solver(B)
    try:   # a fresh handle after the teardowns: its checked _dev entry points report no stale error
        q0, v0 = s.sim_standing_state(np.zeros((B, 3)))
        q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev); rbd = torch.zeros((B, _lib.RBD), dtype=torch.float64, device=dev)
        contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
        s.sim_step_dev(1e-3, torch.zeros((B, 18), dtype=torch.float64, device=dev), q, v, rbd, contact, st)
        s.fall_detect_dev(rbd, torch.zeros_like(contact), torch.zeros_like(contact)); torch.cuda.synchronize()
        assert np.all(st.cpu().numpy() == 0)
    finally:
        s.close()


# ---------------- 2: a spec that names no field ----------------
NB = 16


def _base_kw(xy):
    return dict(duration=0.4, gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.1), xy_yaw=xy)


@pytest.mark.parametrize("case", ["truth", "truth_respawn", "estimate", "estimate_respawn"])
def test_a_spec_that_names_no_field_changes_nothing(case):
    from qm_control_b200 import closed_loop
    xy = np.zeros((NB, 3)); xy[:, 0] = 2.0 * np.arange(NB)
    kw = _base_kw(xy)
    if case.startswith("estimate"):
        kw.update(state_estimator=True, attitude_filter=True, slip_detector=True)
    if case.endswith("respawn"):
        kw.update(respawn=dict(on_fall=False, every=0.2))
    out = {}
    for tag, extra in (("plain", {}), ("named_none", dict(randomize=dict(seed=3)))):
        s = _solver(NB)
        try:
            before = _state(s)
            out[tag] = closed_loop.run(s, **kw, **extra)
            _same(before, _state(s))
        finally:
            s.close()
    for k in REC + ("q", "v"):
        assert out["plain"][k].tobytes() == out["named_none"][k].tobytes(), k
    p = out["named_none"]["episode_params"]; assert p.shape == (NB, 2 if case.endswith("respawn") else 1, _lib.EPISODE)
    np.testing.assert_array_equal(p[:, :, EP["cmd_vel_x"]], 0.2); np.testing.assert_array_equal(p[:, :, EP["friction_mu"]], 0.6)


# ---------------- 3: every drawn episode is the first episode of a run fixed at its row ----------------
EVERY_S, EPISODES = 0.2, 3
RANGES = dict(seed=77, friction_mu=(0.3, 1.0), m_ee=(0.0, 2.0), m_base=(0.0, 3.0), push_t_on=(0.02, 0.1), push_duration=(0.02, 0.06), f_base_y=(-100.0, 100.0),
              cmd_vel_x=(0.0, 0.4), cmd_yaw_rate=(-0.3, 0.3))


def _exact_case(case):
    xy = np.zeros((NB, 3)); xy[:, 0] = 2.0 * np.arange(NB)
    kw = dict(gait="trot", xy_yaw=xy)
    if case == "linked":
        kw.update(model_payload="plant", tuning=dict(friction_mu="plant"))
    if case == "commands_terrain":
        tiles = np.stack([T.ramp(5.0, start=0.35), T.stairs(0.03, 0.3, start=0.35)])
        kw.update(gait="stance", terrain=dict(tiles=tiles, cell=T.CELL, tile=np.arange(NB) % 3 - 1, origin=T.centred_origin(xy[:, :2])),
                  commands=dict(t=np.full((NB, 1), 0.05), gait=np.full((NB, 1), "trot", dtype=object)))
    return kw


@pytest.mark.parametrize("case", ["plain", "linked", "commands_terrain"])
def test_every_episode_is_the_first_episode_of_a_run_fixed_at_its_row(case):
    from qm_control_b200 import closed_loop
    kw = _exact_case(case); n = int(round(EVERY_S * 100)); told = []
    s = _solver(NB)
    try:
        before = _state(s); orig = s.episode_set_ranges

        def set_ranges(lo=None, hi=None, seed=0):
            if lo is not None:
                told.append((lo.copy(), hi.copy(), seed))
            orig(lo, hi, seed)
        s.episode_set_ranges = set_ranges
        r = closed_loop.run(s, duration=EVERY_S * EPISODES, respawn=dict(on_fall=False, every=EVERY_S), randomize=RANGES, **kw)
        s.episode_set_ranges = orig
        _same(before, _state(s))   # ranges, robot params, model payload and tuning rows are back
    finally:
        s.close()
    np.testing.assert_array_equal(r["episode"], np.repeat(np.arange(EPISODES), n)[:, None] * np.ones((1, NB), dtype=np.int32))
    lo, hi, seed = told[0]; P = r["episode_params"]
    assert P.shape == (NB, EPISODES, _lib.EPISODE)
    for e in range(EPISODES):
        np.testing.assert_array_equal(P[:, e], tw.rows(lo, hi, np.full(NB, seed, dtype=np.uint64), np.arange(NB), np.full(NB, e)))
    assert np.all(P[:, 1] != P[:, 0], axis=0)[[EP[f] for f in RANGES if f != "seed"]].all()
    for e in range(EPISODES):
        row = P[:, e]; fixed = {f: (row[:, EP[f]], row[:, EP[f]]) for f in RANGES if f != "seed"}
        s = _solver(NB)
        try:
            ref = closed_loop.run(s, duration=EVERY_S, respawn=dict(on_fall=False, every=EVERY_S), randomize=dict(seed=5, **fixed), **kw)
        finally:
            s.close()
        np.testing.assert_array_equal(ref["episode_params"][:, 0], row)
        for k in REC:
            assert r[k][e * n:(e + 1) * n].tobytes() == ref[k][:n].tobytes(), "%s episode %d" % (k, e)
