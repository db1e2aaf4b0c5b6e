"""The MPC kernels past their node-count capacity thresholds, up to the handle's node limit, against the oracle.

A long enough grid changes what three kernels do (the constants below, recomputed from the kernels' formulas in tests/test_node_capacity_cpu.py):
  K1 mpc_setup_kernel      stages 4 warps x round16(48 nmax + 320) B of grid in dynamic shared memory: from nmax = K1_OPT_IN past the 48 KB default, on the
                           200 KB opt-in of mpc_configure_device; mpc_alloc refuses a handle past NODE_LIMIT nodes
  K3 mpc_riccati_kernel    caches the node types of n <= RIC_NTYPE nodes in shared memory; a longer robot reads every node type from its stage record
  K4 mpc_linesearch_kernel covers the nodes in passes of LS_THREADS threads: three or more passes from n = 2 LS_THREADS + 1
and the DDP trial kernel walks every CTA's robots in lock step up to the longest one.  None of these paths faults when it is wrong: it computes something else.
So: padding a handle changes no bit, the node limit is exact, long grids (T = 1 s, dt down to 1 ms) match the oracle at the tolerances of tests/_parity.py,
and a long robot gives the same bits alone and among neighbours of other lengths."""
import numpy as np
import pytest

import _schedules as S
from _parity import MPC_TOL, TICK_TOL, assert_cmd, assert_traj
from test_contact_modes_gpu import _advance, _rows, _two_ticks
from test_mpc_gpu import _check

pytestmark = pytest.mark.gpu
T0, H, DT = 12.0, 1.0, 0.015
K1_OPT_IN = 250        # first nmax whose K1 staging needs more than 48 KB of shared memory
RIC_NTYPE = 512        # the longest grid whose node types K3 keeps in shared memory
NODE_LIMIT = 1060      # the largest max_nodes a handle accepts
LS_THREADS = 128       # nodes per K4 pass
DDP_RPC = 16           # robots per CTA of the DDP trial kernel (seven step lengths 1 ... 1/64 on a pitch of 8 lanes: 128 / 8, capped at 16)
MAX_NODES = (0, K1_OPT_IN - 1, K1_OPT_IN, RIC_NTYPE, RIC_NTYPE + 1, NODE_LIMIT)   # 0: the default padding (88 nodes at dt 0.015)
# T stays at 1 s: the grids are long through dt alone.  (a) ~260 nodes: three K4 passes; (b) one stance robot without events at exactly RIC_NTYPE nodes next to
# robots with events at more; (c) ~1000 nodes inside the default padding ceil(T / dt) + 21 = 1021
GRIDS = {"a": 0.0039, "b": 0.00196, "c": 0.001}
FLAT = 9               # the stance robot without events of the long batch: n = ceil(T / dt) + 1


def _cat(a, b):
    return {k: np.concatenate([a[k], b[k]]) for k in a}


def _base():
    """config 5 (stance / trot / flying trot by id) and config 4 (trot): B = 9."""
    from qm_control_b200 import synthetic
    p5, w5 = synthetic.make_batch(np.arange(6), config=5, t0=T0); p4, w4 = synthetic.make_batch(np.arange(3), config=4, t0=T0)
    return list(synthetic.GAITS) * 2 + ["trot"] * 3, _cat(p5, p4), _cat(w5, w4)


def long_batch():
    """the base batch, a stance robot without events (robot FLAT) and a one-foot stance (15 free inputs): B = 11."""
    from qm_control_b200 import synthetic
    names, prob, wbc = _base(); p, w = synthetic.make_batch(np.arange(9, 11), config=4, t0=T0)
    S.with_schedule(p, 0, [], [15]); S.with_schedule(p, 1, *S.single_foot(2, T0, H, 0.23))
    return names + ["stance_flat", "single_foot_2"], _cat(prob, p), _cat(wbc, w)


def default_nmax(dt):
    return int(np.ceil(H / dt - 1e-9)) + 21


def assert_grid(case, names, n, nmax):
    """what grid `case` claims, on node counts n [B] (the CUDA path's or the oracle's) of long_batch at GRIDS[case] on a handle of nmax nodes."""
    n = np.asarray(n); assert nmax == default_nmax(GRIDS[case]) and n.max() <= nmax, (case, n, nmax)
    if case == "a":
        assert nmax >= K1_OPT_IN and 2 * LS_THREADS < n.min() and n.max() < 280, n                       # every robot takes three K4 passes
    elif case == "b":
        others = np.delete(n, FLAT)
        assert names[FLAT] == "stance_flat" and n[FLAT] == RIC_NTYPE and others.min() > RIC_NTYPE, n      # both K3 paths in one launch
        assert n[names.index("single_foot_2")] > RIC_NTYPE and n[names.index("trot")] > RIC_NTYPE, n
    else:
        assert 990 <= n.min() and n.max() <= nmax, n


def _same(a, b, robots=None, keys=("status", "step_info")):
    """bit equality of two solutions on the first n nodes of every robot (status, step info and cmd where given)"""
    robots = range(len(b["n_nodes"])) if robots is None else robots
    for r in robots:
        n = int(b["n_nodes"][r]); assert int(a["n_nodes"][r]) == n, (r, a["n_nodes"][r], n)
        for k in ("t", "event", "x", "u"):
            assert np.array_equal(a[k][r, :n], b[k][r, :n]), (r, k)
        for k in keys:
            assert np.array_equal(a[k][r], b[k][r]), (r, k)


@pytest.mark.parametrize("solver_name", ["sqp", "ddp"])
def test_padding_changes_nothing(oracle, solver_name):
    """The same batch on handles of 88 (default) to NODE_LIMIT nodes, two solves, the second from each handle's own stored solution: K1 interpolates out of a
    padded previous grid.  Every output is bit-identical to the default handle's."""
    import qm_control_b200 as q
    _, prob, _ = _base(); B = len(prob["t0"])
    ref = None; prob2 = None
    for m in MAX_NODES:
        s = q.Solver(batch=B, dt=DT, max_nodes=m); s.mpc_set_solver(solver_name)
        assert s.nmax == (m if m else default_nmax(DT)), (m, s.nmax)
        first = s.mpc_solve(prob)
        if ref is None:
            assert s.nmax < K1_OPT_IN - 1 and np.all((first["status"] & ~16) == 0) and np.any(first["step_info"][:, 0] > 0), first["status"]
            prob2 = _advance(oracle, prob, first)
        second = s.mpc_solve(prob2); stored = s.mpc_get_solution(); s.close()
        if ref is None:
            ref = (first, second); continue
        for tick, (got, want) in enumerate(zip((first, second, stored), ref + (ref[1],))):
            try:
                _same(got, want)
            except AssertionError as e:
                raise AssertionError("max_nodes %d, %s, tick %d: %s" % (m, solver_name, min(tick, 1), e)) from None


def test_padded_tick_changes_nothing(oracle):
    """qmb200_tick (one chain and two robot ranges) on the padded handles: commands, status and the stored solution of two ticks equal the default handle's."""
    import qm_control_b200 as q
    _, prob, wbc = _base(); B = len(prob["t0"]); ref = None; prob2 = None
    for m in MAX_NODES:
        for chunks in (1, 2):
            s = q.Solver(batch=B, dt=DT, max_nodes=m); s.set_pipeline(chunks); res = []
            for tick in range(2):
                if tick and prob2 is None:
                    prob2 = _advance(oracle, prob, res[0])                    # from the default handle's first tick, the same for every handle
                p = prob2 if tick else prob
                cmd, st = s.tick(p, p["t0"] + 0.002, wbc["rbd"], wbc["period"])
                sol = s.mpc_get_solution(); sol["cmd"] = cmd; sol["tick_status"] = st; res.append(sol)
            s.close()
            if ref is None:
                assert np.all((res[0]["tick_status"] & ~(16 << 8)) == 0), res[0]["tick_status"]
                ref = res; continue
            for tick in range(2):
                try:
                    _same(res[tick], ref[tick], keys=("status", "step_info", "cmd", "tick_status"))
                except AssertionError as e:
                    raise AssertionError("max_nodes %d, %d chains, tick %d: %s" % (m, chunks, tick, e)) from None


def test_node_limit_at_creation():
    """max_nodes = NODE_LIMIT + 1, or a horizon and dt whose default padding exceeds NODE_LIMIT, fail at creation; the largest default grid that fits
    creates, and a handle created after the refusals solves as before."""
    import qm_control_b200 as q
    _, prob, _ = _base(); B = len(prob["t0"])
    s = q.Solver(batch=B, dt=DT); ref = s.mpc_solve(prob); s.close()
    with pytest.raises(q.QmbError, match="max_nodes too large"):
        q.Solver(batch=B, dt=DT, max_nodes=NODE_LIMIT + 1)
    with pytest.raises(q.QmbError, match="max_nodes too large"):
        q.Solver(batch=B, dt=H / (NODE_LIMIT - 20))                       # ceil(T / dt) + 21 = NODE_LIMIT + 1
    edge = q.Solver(batch=B, dt=H / (NODE_LIMIT - 21)); assert edge.nmax == NODE_LIMIT; edge.close()
    after = q.Solver(batch=B, dt=DT); _same(after.mpc_solve(prob), ref)


def _long(case):
    import qm_control_b200 as q
    names, prob, wbc = long_batch(); dt = GRIDS[case]
    return names, prob, wbc, q.Solver(batch=len(names), dt=dt)


@pytest.fixture
def long_grid(oracle):
    """sets the oracle's grid for one case and puts the default grid back"""
    def use(case):
        oracle.mpc_set(dt=GRIDS[case], horizon=H)
        return _long(case)
    yield use
    oracle.mpc_set(dt=DT, horizon=H)


@pytest.mark.parametrize("case", sorted(GRIDS))
def test_long_grid_sqp(oracle, long_grid, case):
    names, prob, _, solver = long_grid(case)
    _, res = _two_ticks(oracle, solver, prob)
    for out, _ in res:
        assert_grid(case, names, out["n_nodes"], solver.nmax)
    assert 15 in _rows(prob, res[0][1])                                    # the one-foot stance: an odd input count on a long grid
    _check(res, "long grid %s dt %g" % (case, GRIDS[case]))


def test_three_sqp_iterations_across_the_type_cache(oracle, long_grid):
    names, prob, _, solver = long_grid("b")
    try:
        solver.mpc_set_iterations(3); oracle.mpc_set_sqp(3)
        out = solver.mpc_solve(prob); ref = oracle.mpc_solve_batch(prob, solver.nmax, nthreads=8)
        assert_grid("b", names, out["n_nodes"], solver.nmax)
        assert np.all((out["status"] & ~(16 | 32)) == 0), np.unique(out["status"])
        np.testing.assert_array_equal((out["status"] & 32) != 0, ref["dbg"][:, 9] < 3)
        np.testing.assert_array_equal(out["step_info"][:, 0], ref["dbg"][:, 0])
        assert_traj(out, ref, 10 * MPC_TOL, tag="long grid b, 3 sqp iterations")
    finally:
        oracle.mpc_set_sqp(1)


def _ddp(oracle, solver):
    from test_solver_variants_gpu import _block
    ddp = _block("ddp"); solver.mpc_set_solver("ddp")
    oracle.mpc_set_solver(solver=2, iterations=int(ddp["maxNumIterations"]), ddp_penalty=ddp["constraintPenaltyInitialValue"], ddp_min_step=ddp["minStepLength"], ddp_max_step=ddp["maxStepLength"])


def _sqp(oracle):
    from test_solver_variants_gpu import _block
    sq = _block("sqp"); oracle.mpc_set_solver(solver=0, iterations=1, delta_tol=sq["deltaTol"], g_max=sq["g_max"], g_min=sq["g_min"])


def test_ddp_on_a_long_grid(oracle, long_grid):
    """the trial kernel's CTA holds robots of 512 and more nodes; rules of test_ddp_on_every_contact_mode"""
    names, prob, _, solver = long_grid("b")
    try:
        _ddp(oracle, solver); _, res = _two_ticks(oracle, solver, prob)
    finally:
        _sqp(oracle)
    n = res[0][0]["n_nodes"]; assert_grid("b", names, n, solver.nmax)
    assert len(n) <= DDP_RPC and len(set(n.tolist())) >= 5, n                     # one trial CTA, walked in lock step to its longest robot
    for tick, (out, ref) in enumerate(res):
        assert np.all((out["status"] & ~16) == 0), np.unique(out["status"])
        np.testing.assert_array_equal(out["step_info"][:, 0], ref["dbg"][:, 0])
        acc = ref["dbg"][:, 0] > 0; assert acc.sum() >= len(acc) // 2, acc
        for b in np.nonzero(acc)[0]:
            assert_traj(out, ref, MPC_TOL, tag="long grid ddp tick %d robot %d" % (tick, b), b_out=b, b_ref=b)
        np.testing.assert_allclose(out["step_info"][acc, 1], ref["dbg"][acc, 4], rtol=1e-8, atol=1e-9)
        merit0 = ref["dbg"][:, 1] + 20.0 * np.sqrt(ref["dbg"][:, 3]); merit = out["step_info"][:, 1] + 20.0 * np.sqrt(out["step_info"][:, 3])
        assert np.all(merit[acc] < merit0[acc]), (merit, merit0)


def test_policy_eval_on_a_thousand_nodes(oracle, long_grid):
    """every node time, every event time and 1e-9 either side of it"""
    names, prob, _, solver = long_grid("c"); B = len(names)
    solver.mpc_solve(prob)                                                     # the handle keeps the mode schedule policy_eval reads the mode from
    ref = oracle.mpc_solve_batch(prob, solver.nmax, nthreads=8); solver.mpc_set_solution(ref)
    assert_grid("c", names, ref["n_nodes"], solver.nmax)
    queries = []
    for b in range(B):
        n = int(ref["n_nodes"][b]); ev = prob["event_times"][b, :prob["n_events"][b]]; ev = ev[(ev >= T0) & (ev <= T0 + H)]
        queries.append(list(ref["t"][b, :n]) + [te + d for te in ev for d in (0.0, -1e-9, 1e-9)])
    assert min(len(qs) for qs in queries) > 1000
    for i in range(max(len(qs) for qs in queries)):
        tq = np.array([qs[i % len(qs)] for qs in queries])
        xd, ud, mode = solver.policy_eval(tq)
        for b in range(B):
            n = ref["n_nodes"][b]; ne = prob["n_events"][b]
            x, u, m = oracle.evaluate_policy(ref["t"][b, :n], ref["event"][b, :n], ref["x"][b, :n], ref["u"][b, :n], prob["event_times"][b, :ne], prob["modes"][b, :ne + 1], tq[b])
            np.testing.assert_allclose(xd[b], x, rtol=0, atol=1e-12, err_msg="%s t=%r" % (names[b], tq[b]))
            np.testing.assert_allclose(ud[b], u, rtol=0, atol=1e-10, err_msg="%s t=%r" % (names[b], tq[b])); assert mode[b] == m, (names[b], tq[b])


def test_tick_across_the_type_cache(oracle, long_grid):
    names, prob, wbc, solver = long_grid("b"); B = len(names)
    t_eval = prob["t0"] + 0.0123
    cmd, status = solver.tick(prob, t_eval, wbc["rbd"], wbc["period"])
    assert np.all((status & ~(16 << 8)) == 0), np.unique(status)
    ref = oracle.tick_batch(prob, solver.nmax, t_eval, wbc["rbd"], wbc["period"], np.zeros((B, 30)), nthreads=8)
    sol = solver.mpc_get_solution(); assert_grid("b", names, sol["n_nodes"], solver.nmax)
    assert_cmd(cmd, ref["cmd"], TICK_TOL, tag="long grid b tick")
    assert_traj(sol, ref, MPC_TOL, tag="long grid b tick trajectories")


@pytest.mark.parametrize("solver_name", ["sqp", "ddp"])
def test_long_robots_do_not_see_their_neighbours(solver_name):
    """every robot of grid (b) alone on a one-robot handle gives the bits it gives in the mixed batch: K3 picks its node-type path per CTA, the DDP trial
    CTA walks to its longest robot"""
    import qm_control_b200 as q
    names, prob, _, solver = _long("b"); solver.mpc_set_solver(solver_name)
    mixed = solver.mpc_solve(prob); assert_grid("b", names, mixed["n_nodes"], solver.nmax); solver.close()
    one = q.Solver(batch=1, dt=GRIDS["b"]); one.mpc_set_solver(solver_name); assert one.nmax == solver.nmax
    for b in range(len(names)):
        one.mpc_reset(); alone = one.mpc_solve({k: v[b:b + 1] for k, v in prob.items()})
        _same(alone, {k: v[b:b + 1] for k, v in mixed.items()})
