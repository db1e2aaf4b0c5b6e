"""The CUDA MPC, WBC and tick against the oracle on every contact mode: all twelve gaits of assets/qm_gait.info, a bound (12/3), single-foot stances and a
schedule through all 16 masks.  One and three feet down give nodes with 15 and 13 equality rows, so 15 and 17 free inputs: an odd input count puts the arm's
projected columns of the Riccati kernel on an odd column (they straddle a tensor-core fragment pair) and the identity padding of H on an odd row.  Tolerances
are those of tests/_parity.py; the step size must be identical."""
import numpy as np
import pytest

import _schedules as S
from _parity import CMD_BLOCKS, MPC_TOL, MPCWBC_TOL, TICK_TOL, WBC_TOL, assert_cmd, assert_traj
import test_wbc_twin_cpu as tw
from test_mpc_gpu import _check

pytestmark = pytest.mark.gpu
T0 = 12.0


def _schedules(t0=T0, horizon=1.0):
    """five phases of every gait, the bound, the four single-foot stances and all 16 masks: 66 robots (no multiple of 4, 8 or 16)."""
    out = []
    for g in S.ALL_GAITS:
        for j in range(5):
            out.append((g, S.gait_schedule(g, t0, (j + 0.37) / 5.0, horizon)))
    out.append(("bound", S.bound(t0, horizon, 0.31)))
    for m in (8, 4, 2, 1):
        out.append(("single_foot_%d" % m, S.single_foot(m, t0, horizon, 0.23)))
    out.append(("all_masks", S.all_masks(t0, horizon, 0.17)))
    return out


def _batch(names=None):
    sch = [s for s in _schedules() if names is None or s[0] in names]
    B = len(sch); prob, wbc = synthetic_batch(B)
    for b, (_, (e, m)) in enumerate(sch):
        S.with_schedule(prob, b, e, m)
    return [n for n, _ in sch], prob, wbc


def synthetic_batch(B):
    from qm_control_b200 import synthetic
    return synthetic.make_batch(np.arange(B), config=4)


def _advance(oracle, prob, prev):
    """next tick: t0 + 10 ms, x0 on the oracle's own policy (the same for both sides)."""
    prob = dict(prob); prob["t0"] = prob["t0"] + 0.01; x0 = np.zeros_like(prob["x0"])
    for b in range(len(x0)):
        n = prev["n_nodes"][b]; ne = prob["n_events"][b]
        x0[b], _, _ = oracle.evaluate_policy(prev["t"][b, :n], prev["event"][b, :n], prev["x"][b, :n], prev["u"][b, :n], prob["event_times"][b, :ne], prob["modes"][b, :ne + 1], prob["t0"][b])
    prob["x0"] = x0
    return prob


def _two_ticks(oracle, solver, prob, ticks=2):
    prev = None; res = []
    for tick in range(ticks):
        if tick:
            prob = _advance(oracle, prob, prev)
        out = solver.mpc_solve(prob); ref = oracle.mpc_solve_batch(prob, solver.nmax, prev=prev, nthreads=8)
        res.append((out, ref)); prev = ref; solver.mpc_set_solution(ref)   # the oracle's solution is both sides' warm start
    return prob, res


def _rows(prob, ref):
    rows = set()
    for b in range(len(prob["t0"])):
        n = int(ref["n_nodes"][b]); ne = prob["n_events"][b]
        rows |= set(S.mode_rows(prob["event_times"][b, :ne], prob["modes"][b], ref["t"][b], ref["event"][b], n).tolist())
    return rows


@pytest.mark.parametrize("dt", [0.015, 0.01])
def test_sqp_on_every_contact_mode(oracle, dt):
    import qm_control_b200 as q
    names, prob, _ = _batch(); B = len(names); assert B % 4
    solver = q.Solver(batch=B, dt=dt, max_nodes=96 if dt == 0.015 else 0); oracle.mpc_set(dt=dt, horizon=1.0)   # all_masks needs 89 nodes at dt 0.015, one more than the default
    _, res = _two_ticks(oracle, solver, prob)
    assert {13, 15} <= _rows(prob, res[0][1])
    _check(res, "contact modes dt %g" % dt)


def test_three_sqp_iterations_with_one_and_three_feet_down(oracle):
    import qm_control_b200 as q
    names, prob, _ = _batch({"dynamic_walk", "static_walk", "pawup", "single_foot_8", "single_foot_4", "single_foot_2", "single_foot_1"}); B = len(names)
    solver = q.Solver(batch=B, dt=0.015); oracle.mpc_set(dt=0.015, horizon=1.0)
    try:
        solver.mpc_set_iterations(3); oracle.mpc_set_sqp(3)
        out = solver.mpc_solve(prob); ref = oracle.mpc_solve_batch(prob, solver.nmax, nthreads=8)
        assert {13, 15} <= _rows(prob, ref)
        assert np.all((out["status"] & ~(16 | 32)) == 0), np.unique(out["status"])
        np.testing.assert_array_equal((out["status"] & 32) != 0, ref["dbg"][:, 9] < 3)
        np.testing.assert_array_equal(out["step_info"][:, 0], ref["dbg"][:, 0])
        assert_traj(out, ref, 10 * MPC_TOL, tag="contact modes, 3 sqp iterations")
    finally:
        oracle.mpc_set_sqp(1)


def _solver_variant(oracle, name, B):
    import qm_control_b200 as q
    from test_solver_variants_gpu import _block
    names, prob, _ = _batch(); prob = {k: v[-B:] for k, v in prob.items()}     # the last B robots: the walks, pawup, the bound, the single-foot stances and all masks
    s = q.Solver(batch=B, dt=0.015, max_nodes=96); s.mpc_set_solver(name); oracle.mpc_set(dt=0.015, horizon=1.0)
    if name == "ipm":
        ipm = _block("ipm"); oracle.mpc_set_solver(solver=1, iterations=int(ipm["ipmIteration"]), delta_tol=ipm["deltaTol"], g_max=ipm["g_max"], g_min=ipm["g_min"])
    else:
        ddp = _block("ddp"); oracle.mpc_set_solver(solver=2, iterations=int(ddp["maxNumIterations"]), ddp_penalty=ddp["constraintPenaltyInitialValue"], ddp_min_step=1e-2, ddp_max_step=1.0)
    try:
        _, res = _two_ticks(oracle, s, prob)
    finally:
        sq = _block("sqp"); oracle.mpc_set_solver(solver=0, iterations=1, delta_tol=sq["deltaTol"], g_max=sq["g_max"], g_min=sq["g_min"])
    return names[-B:], prob, res


def test_ipm_on_every_contact_mode(oracle):
    names, prob, res = _solver_variant(oracle, "ipm", 66)
    assert {13, 15} <= _rows(prob, res[0][1])
    for tick, (out, ref) in enumerate(res):
        assert np.all((out["status"] & ~16) == 0), np.unique(out["status"])
        np.testing.assert_array_equal(out["step_info"][:, 0], ref["dbg"][:, 0])
        assert_traj(out, ref, MPC_TOL, tag="contact modes ipm tick %d" % tick)
        acc = ref["dbg"][:, 0] > 0
        np.testing.assert_allclose(out["step_info"][acc, 1], ref["dbg"][acc, 4], rtol=1e-6, atol=1e-8)   # cost after the step


DDP_NOT_PD = 33    # single_foot_4: its first DDP step is rejected on both sides (alpha 0)
DDP_GAP = 5e-8     # robots whose step is rejected (alpha 0 on both sides): measured 2.6e-8 in the base angles of the kept rollout; pinned so a regression fails


def test_ddp_on_every_contact_mode(oracle):
    """37 robots: the 16-robot trial CTAs of the rollout kernel end on a partial CTA.  Status and step length exactly; the robots that take a step at MPC_TOL,
    with their cost and the descent of the merit; the robots whose step both sides reject at DDP_GAP."""
    names, prob, res = _solver_variant(oracle, "ddp", 37)
    assert {13, 15} <= _rows(prob, res[0][1])
    assert names[DDP_NOT_PD] == "single_foot_4" and res[0][1]["dbg"][DDP_NOT_PD, 0] == 0.0
    for tick, (out, ref) in enumerate(res):
        keep = np.arange(len(names)) if tick == 0 else np.delete(np.arange(len(names)), DDP_NOT_PD)
        if tick == 1:   # open finding, pinned: the oracle takes the second tick of this robot from its rejected first step, the kernels flag NOT_PD | NO_STEP
            assert out["status"][DDP_NOT_PD] == 8 | 16 and out["step_info"][DDP_NOT_PD, 0] == 0.0, (out["status"][DDP_NOT_PD], ref["dbg"][DDP_NOT_PD])
        out = {k: v[keep] for k, v in out.items()}; ref = {k: v[keep] for k, v in ref.items()}
        assert np.all((out["status"] & ~16) == 0), np.unique(out["status"])
        np.testing.assert_array_equal(out["step_info"][:, 0], ref["dbg"][:, 0])
        acc = ref["dbg"][:, 0] > 0; assert acc.sum() >= len(acc) // 2, acc
        for b in range(len(acc)):                 # a robot without an accepted step keeps the nominal rollout of its guess, which amplifies last-bit differences
            tol = MPC_TOL if acc[b] else DDP_GAP
            assert_traj(out, ref, tol, tag="contact modes ddp tick %d robot %d (step %s)" % (tick, b, "taken" if acc[b] else "rejected"), b_out=b, b_ref=b)
        np.testing.assert_allclose(out["step_info"][acc, 1], ref["dbg"][acc, 4], rtol=1e-8, atol=1e-9)
        merit0 = ref["dbg"][:, 1] + 20.0 * np.sqrt(ref["dbg"][:, 3]); merit = out["step_info"][:, 1] + 20.0 * np.sqrt(out["step_info"][:, 3])
        assert np.all(merit[acc] < merit0[acc]), (merit, merit0)


@pytest.mark.parametrize("variant,time", [(0, 12.0), (0, 3.0), (1, 12.0), (1, 3.0)])
def test_wbc_on_all_16_masks(oracle, variant, time):
    """149 robots, mask = id % 16: a CTA of eight warps mixes contact counts."""
    import qm_control_b200 as q
    from qm_control_b200 import synthetic
    B = 149; ids = np.arange(B); solver = q.Solver(batch=B, wbc_variant=variant)
    prob, wbc = synthetic.make_batch(ids, config=3)
    mode = (ids % 16).astype(np.int32); u_des = np.zeros((B, 30))
    for b in range(B):
        nc = bin(int(mode[b])).count("1")
        for f in range(4):
            if (mode[b] >> (3 - f)) & 1:
                u_des[b, 3 * f + 2] = solver.robot_mass * 9.81 / nc
    u_des = u_des + synthetic.uniform(77, ids, 1, 30, -1.0, 1.0) * np.r_[np.full(12, 5.0), np.full(18, 0.2)]
    for b in range(B):
        for f in range(4):
            if not (mode[b] >> (3 - f)) & 1:
                u_des[b, 3 * f:3 * f + 3] = 0.0
    il = synthetic.uniform(78, ids, 2, 30, -0.1, 0.1); tarr = np.full(B, time); x_des = prob["x0"].copy()
    solver.wbc_set_input_last(il)
    cmd, status = solver.wbc_update(x_des, u_des, wbc["rbd"], mode, wbc["period"], tarr)
    ref, _ = oracle.wbc_update_batch(x_des, u_des, wbc["rbd"], mode, wbc["period"], tarr, il, variant=variant, nthreads=8)
    assert np.all(status == 0), np.unique(status)
    np.testing.assert_array_equal(solver.wbc_get_input_last(), u_des)
    blocks = dict(CMD_BLOCKS)
    if variant == 1:
        blocks["arm_acc"] = (18, 24, 1e3)          # the untasked arm accelerations of HierarchicalMpcWbc (tests/test_wbc_gpu.py)
    g = tw._gains(); compared = 0; oracle_off = []
    for m in range(16):
        sel = mode == m
        if variant == 0 and time >= 10 or m == 15:
            assert_cmd(cmd[sel], ref[sel], MPCWBC_TOL if variant else WBC_TOL, tag="wbc variant %d t=%g mask %d" % (variant, time, m), blocks=blocks)
            continue
        # With a swing foot the GPU result is certified level by level against the literal HoQp problems (tests/test_wbc_twin_cpu.py), robot by robot.  Where the
        # oracle's own result passes the same certificate, the level optima agree; in HierarchicalMpcWbc the optimum is unique (levels 1 and 2 leave no free
        # direction: the arm accelerations follow from the stance forces through M[base, arm]), so the commands agree per block as well.  The init branch leaves a
        # swing leg's accelerations untasked: there only the optimal level values are unique.
        for b in np.nonzero(sel)[0]:
            args = (oracle, g, variant, time, x_des[b], u_des[b], wbc["rbd"][b], m, wbc["period"][b], il[b])
            gpu = _level_certificate(*args, cmd[b, :36]); orc = _level_certificate(*args, ref[b, :36])
            assert gpu["ok"], ("GPU result is not the cascade optimum", variant, time, m, b, gpu)
            if not orc["ok"]:
                oracle_off.append(b); continue
            for lvl in ("obj1", "obj2"):
                assert abs(gpu[lvl] - orc[lvl]) <= 1e-8 * (1.0 + abs(orc[lvl])), (variant, time, m, b, lvl, gpu[lvl], orc[lvl])
            if variant == 1:
                assert_cmd(cmd[b], ref[b], MPCWBC_TOL, tag="wbc variant 1 mask %d robot %d" % (m, b), blocks=blocks)
            compared += 1
    assert compared >= 60 or (variant == 0 and time >= 10), (compared, oracle_off)          # the oracle is certified on most swing-foot robots (tests/test_contact_modes_cpu.py lists where it is not)


def _level_certificate(oracle, g, variant, time, x_des, u_des, rbd, mode, period, il, x, mu=0.3):
    """KKT certificate of a WBC result x against the literal level problems of one robot → dict(ok, e0, viol, r1, r2, obj1, obj2).
    e0: distance of A0 x from the level-0 optimum A0 x0 (unique), viol: worst violation of a level-0 inequality (slack included), r1 / r2: NNLS KKT residuals
    of levels 1 and 2 at x, obj1 / obj2: the level objectives.  mu: the robot's friction pyramid (the oracle's task file must hold the same)."""
    dbg = oracle.wbc_debug(x_des, u_des, rbd, int(mode), period, time, input_last=il, variant=variant)
    (A0, b0, D0, f0), (A1, b1), (A2, b2), _ = tw._tasks(oracle, dbg, u_des, int(mode), time if variant == 0 else 12.0, g, mu)   # HierarchicalMpcWbc has no init branch
    if variant == 1:                                                    # HierarchicalMpcWbc.cpp:23-28: height + base angular + base linear + 100 swing, then the forces
        A1, b1, A2, b2 = np.r_[A1[:4], A2[12:14], A1[10:]], np.r_[b1[:4], b2[12:14], b1[10:]], A2[:12], b2[:12]
    x0 = dbg["levels"][0]; fcap = f0 + np.maximum(0.0, D0 @ x0 - f0)
    viol = D0 @ x - fcap; act = viol > -1e-7 * (1.0 + np.abs(fcap))
    e0 = np.max(np.abs(A0 @ (x - x0))) / (1.0 + np.max(np.abs(A0 @ x0)))
    r1 = tw._certificate(A1.T @ (A1 @ x - b1), A0, D0[act]); r2 = tw._certificate(A2.T @ (A2 @ x - b2), np.r_[A0, A1], D0[act])
    ok = e0 < 1e-8 and viol.max() < 1e-8 and r1 < 1e-7 and r2 < 1e-7
    return dict(ok=bool(ok), e0=e0, viol=viol.max(), r1=r1, r2=r2, obj1=float(np.sum((A1 @ x - b1) ** 2)), obj2=float(np.sum((A2 @ x - b2) ** 2)))


def _t_in_phase(prob, b, feet):
    """midpoint of the first phase inside (t0, t0 + 0.6) with `feet` feet down, clipped to that window; None when there is none."""
    ne = prob["n_events"][b]; ev = prob["event_times"][b, :ne]; md = prob["modes"][b]; t0 = prob["t0"][b]
    for i in range(ne + 1):
        lo = ev[i - 1] if i else -np.inf; hi = ev[i] if i < ne else np.inf
        a, z = max(lo, t0), min(hi, t0 + 0.6)
        if z - a > 2e-3 and bin(int(md[i])).count("1") == feet:
            return 0.5 * (a + z)
    return None


def _eval_times(prob):
    """per robot: a time inside a three-foot phase for even robots, a one-foot phase for odd ones (falling back to the other, then to t0 + 2 ms)."""
    out = np.zeros(len(prob["t0"]))
    for b in range(len(out)):
        pref = (3, 1) if b % 2 == 0 else (1, 3)
        t = _t_in_phase(prob, b, pref[0]) or _t_in_phase(prob, b, pref[1])
        out[b] = prob["t0"][b] + 0.002 if t is None else t
    return out


def _subset():
    return _batch({"dynamic_walk", "static_walk", "pawup", "single_foot_8", "single_foot_2", "all_masks", "bound"})


def test_policy_eval_in_one_and_three_foot_phases(oracle):
    import qm_control_b200 as q
    names, prob, _ = _subset(); B = len(names); solver = q.Solver(batch=B, dt=0.015, max_nodes=96); oracle.mpc_set(dt=0.015, horizon=1.0)
    solver.mpc_solve(prob)                                                     # the handle keeps the mode schedule policy_eval reads the mode from
    ref = oracle.mpc_solve_batch(prob, solver.nmax, nthreads=8); solver.mpc_set_solution(ref)
    tq = _eval_times(prob); xd, ud, mode = solver.policy_eval(tq); feet = set()
    for b in range(B):
        n = ref["n_nodes"][b]; ne = prob["n_events"][b]
        x, u, m = oracle.evaluate_policy(ref["t"][b, :n], ref["event"][b, :n], ref["x"][b, :n], ref["u"][b, :n], prob["event_times"][b, :ne], prob["modes"][b, :ne + 1], tq[b])
        np.testing.assert_allclose(xd[b], x, rtol=0, atol=1e-12); np.testing.assert_allclose(ud[b], u, rtol=0, atol=1e-10); assert mode[b] == m, (b, mode[b], m)
        feet.add(bin(int(m)).count("1"))
    assert {1, 3} <= feet


def test_tick_chain_in_one_and_three_foot_phases(oracle):
    import qm_control_b200 as q
    names, prob, wbc = _subset(); B = len(names); solver = q.Solver(batch=B, dt=0.015, max_nodes=96); oracle.mpc_set(dt=0.015, horizon=1.0)
    t_eval = _eval_times(prob)
    cmd, status = solver.tick(prob, t_eval, wbc["rbd"], wbc["period"])
    assert np.all((status & ~(16 << 8)) == 0), np.unique(status)
    ref = oracle.mpc_solve_batch(prob, solver.nmax, nthreads=8); feet = set()
    for b in range(B):
        n = ref["n_nodes"][b]; ne = prob["n_events"][b]
        x, u, m = oracle.evaluate_policy(ref["t"][b, :n], ref["event"][b, :n], ref["x"][b, :n], ref["u"][b, :n], prob["event_times"][b, :ne], prob["modes"][b, :ne + 1], t_eval[b])
        c, _, _ = oracle.wbc_update(x, u, wbc["rbd"][b], m, wbc["period"][b], t_eval[b], input_last=np.zeros(30))
        assert_cmd(cmd[b], c, TICK_TOL, tag="contact-mode tick robot %d (%s, mode %d)" % (b, names[b], m)); feet.add(bin(int(m)).count("1"))
    assert {1, 3} <= feet
