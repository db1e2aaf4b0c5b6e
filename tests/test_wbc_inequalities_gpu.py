"""The CUDA WBC where its inequalities bind: every regime of tests/_wbc_regimes.py in one batch of 192 + 3 robots (no multiple of 8, so the regimes mix inside the
eight-warp CTAs), each robot with its own friction pyramid, on both hierarchies.

Asserted: no WBC status bit; every robot's result is the cascade optimum by the level-by-level KKT certificate (tests/test_contact_modes_gpu.py) with the
robot's mu and level 0's optimal slack; agreement with the oracle where the oracle passes the same certificate (per block where the optimum is unique, in
the level objectives where it is only unique in them); an exact re-solve of every level on the GPU result's active set; the level-0 and working-set
paths reached; robots whose level 0 needs more rows than it holds flagged; bit-identical rows under a permutation; and a full tick on fast-moving states against the oracle."""
import numpy as np
import pytest

import _wbc_regimes as R
import test_wbc_twin_cpu as tw
from _parity import CMD_BLOCKS, MPCWBC_TOL, TICK_TOL, WBC_TOL, assert_cmd
from test_contact_modes_gpu import _level_certificate
from test_wbc_mpc_variant_cpu import _exact

pytestmark = pytest.mark.gpu
EXTRA = 3                      # robots of the fast regime appended again: 195 robots


@pytest.fixture(scope="module")
def oracles(tmp_path_factory):
    return R.Oracles(tmp_path_factory.mktemp("wbc_mu"))


def _inputs(mass):
    r, names = R.batch(mass)
    r = {k: np.concatenate([v, v[:EXTRA]]) for k, v in r.items()}; names = np.concatenate([names, names[:EXTRA]])
    assert len(names) % 8
    return r, names


def _run(r, variant, perm=None):
    import qm_control_b200 as q
    B = len(r["mode"]); s = q.Solver(batch=B, wbc_variant=variant)
    try:
        idx = np.arange(B) if perm is None else perm
        s.set_robot_tuning(dict(wbc_friction=r["wbc_friction"][idx])); s.wbc_set_input_last(r["input_last"][idx])
        cmd, st = s.wbc_update(r["x_des"][idx], r["u_des"][idx], r["rbd"][idx], r["mode"][idx], r["period"][idx], r["time"][idx])
        return cmd, st, s.wbc_get_diagnostics()
    finally:
        s.close()


@pytest.mark.parametrize("variant", [0, 1])
def test_every_regime_is_the_cascade_optimum_and_matches_the_oracle(oracles, variant):
    mass = oracles(0.3).model_info()["mass"]; r, names = _inputs(mass); B = len(names); g = tw._gains()
    cmd, st, diag = _run(r, variant)
    bad = np.nonzero(st & 0xFF)[0]
    assert len(bad) == 0, "WBC status bits: " + ", ".join("robot %d (%s) 0x%x" % (b, names[b], st[b]) for b in bad)
    ref = oracles.wbc_update(r, variant)
    blocks = dict(CMD_BLOCKS)
    if variant == 1:
        blocks["arm_acc"] = (18, 24, 1e3)          # the untasked arm accelerations of HierarchicalMpcWbc (tests/test_wbc_gpu.py)
    compared = 0; off = []
    for b in range(B):
        m = int(r["mode"][b]); mu = r["wbc_friction"][b]; orc = oracles(mu)
        args = (orc, g, variant, r["time"][b], r["x_des"][b], r["u_des"][b], r["rbd"][b], m, r["period"][b], r["input_last"][b])
        gpu = _level_certificate(*args, cmd[b, :36], mu=mu)
        assert gpu["ok"], ("GPU result is not the cascade optimum", variant, b, names[b], m, gpu)
        orc_c = _level_certificate(*args, ref[b, :36], mu=mu)
        if not orc_c["ok"]:
            off.append(b); continue
        compared += 1
        if variant == 1 or r["time"][b] >= 10.0 or m == 15:     # unique optimum (tests/test_contact_modes_gpu.py::test_wbc_on_all_16_masks)
            assert_cmd(cmd[b:b + 1], ref[b:b + 1], MPCWBC_TOL if variant else WBC_TOL, tag="wbc inequalities variant %d robot %d (%s)" % (variant, b, names[b]), blocks=blocks)
        else:
            for lvl in ("obj1", "obj2"):
                assert abs(gpu[lvl] - orc_c[lvl]) <= 1e-8 * (1.0 + abs(orc_c[lvl])), (variant, b, names[b], lvl, gpu[lvl], orc_c[lvl])
    print("variant %d: %d robots compared with the oracle, oracle off the certificate on %s" % (variant, compared, [(b, names[b]) for b in off]))
    # the oracle's HierarchicalMpcWbc cascade leaves a level-0 inequality on some robots (DESIGN.md §5): measured 154 of 195 certified, 193 for HierarchicalWbc
    assert compared >= (150 if variant else B - 8), off
    # the paths the regimes are for
    for name in R.REGIMES:
        sel = names == name
        print("variant %d %-10s level-0 passes max %d, level-1 / level-2 iterations max %d / %d, working set max %d" % (
            variant, name, diag["level0_passes"][sel].max(), diag["level1_iterations"][sel].max(), diag["level2_iterations"][sel].max(), diag["working_set"][sel].max()))
    assert np.any(diag["level0_passes"][names == "fast"] >= 3)       # a violated set, then its repeat
    for name in ("edge", "apex", "saturated"):
        assert np.any(diag["working_set"][names == name] > 0), name
    assert np.all(diag["level1_iterations"] < 80) and np.all(diag["level2_iterations"] < 80) and np.all(diag["level0_passes"] < 30)   # inside the default caps


@pytest.mark.parametrize("variant", [0, 1])
def test_exact_resolve_level_by_level(oracles, variant):
    """Every fourth robot, level by level against equality-constrained least squares re-solved with numpy's SVD (tests/test_wbc_mpc_variant_cpu.py): level 0
    by the numpy statement of the kernel's level-0 rule, levels 1 and 2 on the active set of the GPU result with the levels above held at their values.
    The optimal residuals A_p x of every level are unique, so they are compared for both hierarchies; HierarchicalMpcWbc's optimum is unique, so there the
    whole final point is compared as well."""
    mass = oracles(0.3).model_info()["mass"]; r, names = _inputs(mass); g = tw._gains()
    cmd, st, _ = _run(r, variant); assert np.all((st & 0xFF) == 0)
    rel = lambda a, b: np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)))
    worst = np.zeros(4)
    for b in range(0, len(names), 4):
        m = int(r["mode"][b]); mu = r["wbc_friction"][b]; orc = oracles(mu); t = r["time"][b]
        dbg = orc.wbc_debug(r["x_des"][b], r["u_des"][b], r["rbd"][b], m, r["period"][b], t, input_last=r["input_last"][b], variant=variant)
        (A0, b0, D0, f0), (A1, b1), (A2, b2), _ = tw._tasks(orc, dbg, r["u_des"][b], m, t if variant == 0 else 12.0, g, mu)   # HierarchicalMpcWbc has no init branch
        if variant == 1:
            A1, b1, A2, b2 = np.r_[A1[:4], A2[12:14], A1[10:]], np.r_[b1[:4], b2[12:14], b1[10:]], A2[:12], b2[:12]
        x = cmd[b, :36]; x0 = R.level0_passes(A0, b0, D0, f0)[0]; fcap = f0 + np.maximum(0.0, D0 @ x0 - f0)
        act = D0 @ x - fcap > -1e-7 * (1.0 + np.abs(fcap))          # the active rows of the certificate
        x1 = _exact(A1, b1, np.r_[A0, D0[act]], np.r_[A0 @ x0, fcap[act]])
        x2 = _exact(A2, b2, np.r_[A0, A1, D0[act]], np.r_[A0 @ x0, A1 @ x, fcap[act]])
        errs = [rel(A0 @ x, A0 @ x0), rel(A1 @ x, A1 @ x1), rel(A2 @ x, A2 @ x2), rel(x, x2) if variant == 1 else 0.0]
        worst = np.maximum(worst, errs)
        assert max(errs) < 1e-8, (variant, b, names[b], errs)
    print("exact re-solve variant %d: worst relative difference of A0 x, A1 x, A2 x, x: %s" % (variant, worst))


def test_permuted_batch_gives_bit_identical_rows(oracles):
    mass = oracles(0.3).model_info()["mass"]; r, names = _inputs(mass)
    perm = np.random.default_rng(5).permutation(len(names))
    for variant in (0, 1):
        a, sa, _ = _run(r, variant); p, sp, _ = _run(r, variant, perm)
        np.testing.assert_array_equal(a[perm], p); np.testing.assert_array_equal(sa[perm], sp)


def test_tick_on_fast_moving_states(oracles):
    """MPC -> policy -> WBC on the trot batch with the measured velocities x20, against oracle.tick_batch: the whole chain on fast-moving states, with a
    violated set at level 0.  Whether a robot's level 0 needs more than 24 rows here is not asserted: the desired states come from the MPC."""
    import qm_control_b200 as q
    from qm_control_b200 import synthetic
    B = 37; prob, wbc = synthetic.make_batch(np.arange(B), config=4); rbd = wbc["rbd"].copy(); rbd[:, 24:48] *= R.FAST_SCALE
    s = q.Solver(batch=B, dt=0.015); o = oracles(0.3); o.mpc_set(dt=0.015, horizon=1.0)
    try:
        t_eval = prob["t0"] + 0.002
        cmd, st = s.tick(prob, t_eval, rbd, wbc["period"])
        assert np.all((st & 0xFF) == 0), np.unique(st)
        assert np.any(s.wbc_get_diagnostics()["level0_passes"] >= 3)   # a violated set, then its repeat
        ref = o.tick_batch(prob, s.nmax, t_eval, rbd, wbc["period"], np.zeros((B, 30)), nthreads=8)
        assert_cmd(cmd, ref["cmd"], TICK_TOL, tag="tick on fast-moving states")
    finally:
        s.close()


def test_a_robot_whose_level_0_needs_more_rows_is_flagged(oracles):
    """The stance batch (config 3) with the measured velocities x20: by the numpy statement of the kernel's level-0 rule one robot of 48 reaches a violated set
    of more than 14 rows (18 + 14 = 32 rows, the level-0 capacity, DESIGN.md §4.1).  Exactly those robots come out with QMB200_ST_OVERFLOW; every other robot
    has no status bit and is the cascade optimum."""
    import qm_control_b200 as q
    from qm_control_b200 import synthetic
    B = 48; ids = np.arange(B); g = tw._gains(); o = oracles(0.3); mass = o.model_info()["mass"]
    prob, wbc = synthetic.make_batch(ids, config=3); x_des, u_des, mode = synthetic.nominal_wbc_inputs(prob, mass)
    u_des = u_des + synthetic.uniform(77, ids, 1, 30, -1.0, 1.0) * np.r_[np.full(12, 5.0), np.full(18, 0.2)]
    rbd = wbc["rbd"].copy(); rbd[:, 24:48] *= R.FAST_SCALE; il = synthetic.uniform(78, ids, 2, 30, -0.1, 0.1); tarr = np.full(B, 12.0)
    need = np.zeros(B, dtype=int)
    for b in range(B):
        dbg = o.wbc_debug(x_des[b], u_des[b], rbd[b], int(mode[b]), wbc["period"][b], 12.0, input_last=il[b])
        (A0, b0, D0, f0), _, _, _ = tw._tasks(o, dbg, u_des[b], int(mode[b]), 12.0, g)
        need[b] = max(R.level0_passes(A0, b0, D0, f0)[1])
    assert (need > 14).sum() >= 1, need
    s = q.Solver(batch=B)
    try:
        s.wbc_set_input_last(il); cmd, st = s.wbc_update(x_des, u_des, rbd, mode, wbc["period"], tarr)
    finally:
        s.close()
    np.testing.assert_array_equal(st & 0xFF, np.where(need > 14, 2, 0), err_msg=str(need))
    for b in np.nonzero(need <= 14)[0]:
        c = _level_certificate(o, g, 0, 12.0, x_des[b], u_des[b], rbd[b], mode[b], wbc["period"][b], il[b], cmd[b, :36])
        assert c["ok"], (b, need[b], c)
