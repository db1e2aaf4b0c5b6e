"""The MPC's time grid (timeDiscretizationWithEvents in the setup kernel) against the oracle at its corners: an event on a grid node or within dt_min of one
(the node is merged), events at t0 and t0 + T, two events closer than dt_min, no event inside the horizon, the node limit; other t0, horizons and dt; 1, 3 and 4
target knots; a warm start across an event; policy_eval at node, event and out-of-horizon times.  A robot the oracle cannot solve must carry the status the
oracle's exception names, and must not disturb its neighbours."""
import numpy as np
import pytest

import _schedules as S
from _parity import MPC_TOL, assert_traj
from test_contact_modes_gpu import _two_ticks
from test_mpc_gpu import _check

pytestmark = pytest.mark.gpu
T0, DT, H, P = 12.0, 0.015, 1.0, 0.35
OVERFLOW, NOT_PD, NO_STEP, NEG_DT = 2, 8, 16, 64


def _node(k, t0=T0, dt=DT):
    t = t0
    for _ in range(k):       # the grid accumulates dt node by node
        t = t + dt
    return t


def _around(te, before=2, after=6, m0=9):
    """trot-like 9/6 schedule with an event at te and phases of P around it."""
    ev = [te + P * i for i in range(-before, after)]
    return ev, [15] + [m0 if i % 2 == 0 else 15 - m0 for i in range(len(ev) - 1)] + [15]


def _placed():
    tn = _node(20); tf = T0 + H; cases = {}
    for d in (0.0, 5e-9, -5e-9, 1.5e-8, -1.5e-8, 2e-6, -2e-6):
        cases["node 20 %+g" % d] = _around(tn + d)
    cases["at t0"] = _around(T0, before=1); cases["t0 + 5e-9"] = _around(T0 + 5e-9, before=1)
    cases["at tf"] = _around(tf, before=3, after=2); cases["tf - 5e-9"] = _around(tf - 5e-9, before=3, after=2)
    for gap in (0.005, 5e-9):
        cases["pair %g apart" % gap] = ([tn - 0.7, tn - 0.35, tn, tn + gap, tn + 0.35, tn + 0.7, tn + 1.05], [15, 6, 9, 15, 6, 9, 6, 15])
    cases["all before t0"] = ([T0 - 0.7, T0 - 0.35], [15, 9, 15]); cases["all after tf"] = ([tf + 0.1, tf + 0.45], [15, 9, 15])
    cases["no events, stance"] = ([], [15]); cases["no events, mask 7"] = ([], [7])
    return cases


def _batch(cases):
    from qm_control_b200 import synthetic
    names = list(cases); prob, wbc = synthetic.make_batch(np.arange(len(names)), config=4)
    for b, n in enumerate(names):
        S.with_schedule(prob, b, *cases[n])
    return names, prob, wbc


def _same(a, b, robots):
    for k in ("n_nodes", "t", "event", "x", "u", "status", "step_info"):
        assert np.array_equal(a[k][robots], b[k][robots]), k


def test_placed_events(oracle):
    import qm_control_b200 as q
    cases = _placed(); names, prob, _ = _batch(cases); B = len(names)
    solver = q.Solver(batch=B, dt=DT); oracle.mpc_set(dt=DT, horizon=H)
    out = solver.mpc_solve(prob); res = S.oracle_per_robot(oracle, prob, solver.nmax)
    good = [b for b, (r, _) in enumerate(res) if r is not None]; kinds = set()
    for b, (r, err) in enumerate(res):
        st = int(out["status"][b]); tag = "%s: status %#x" % (names[b], st)
        if r is not None:
            assert st & ~NO_STEP == 0, tag
            assert out["step_info"][b, 0] == r["dbg"][0, 0], tag
            assert_traj(out, r, MPC_TOL, tag="grid " + names[b], b_out=b, b_ref=0); kinds.add("solved")
        elif "not positive definite" in err:
            n = int(out["n_nodes"][b])
            assert st & (NOT_PD | NO_STEP) == NOT_PD | NO_STEP and st & ~(NOT_PD | NO_STEP | NEG_DT) == 0, tag
            assert bool(st & NEG_DT) == S.grid_has_nonpositive_interval(out["t"][b], out["event"][b], n), tag
            assert out["step_info"][b, 0] == 0.0, tag
            assert np.all(np.isfinite(out["x"][b, :n])) and np.all(np.isfinite(out["u"][b, :n])), tag; kinds.add("not_pd")
        else:
            assert "not enclosed" in err, err
            assert st & OVERFLOW, tag; kinds.add("overflow")
    assert kinds == {"solved", "not_pd", "overflow"}, kinds
    # the failing robots' schedules replaced by a plain trot: every well-formed robot is bit-identical
    plain = {k: v.copy() for k, v in prob.items()}
    for b, (r, _) in enumerate(res):
        if r is None:
            S.with_schedule(plain, b, *_around(_node(20) + 0.0123))
    _same(out, q.Solver(batch=B, dt=DT).mpc_solve(plain), good)


LONG_GAP = 3e-7    # measured 1.5e-7 (leg joint velocities) at a 2 s horizon, dt 0.01 and 0.015 alike; horizons up to 1.5 s agree below 1e-10


@pytest.mark.parametrize("t0,horizon,dt", [(0.0, 1.0, 0.015), (3.141, 1.0, 0.015), (1000.0037, 1.0, 0.015), (T0, 0.6, 0.015), (T0, 1.5, 0.015), (T0, 1.0, 0.007), (T0, 2.0, 0.01)])
def test_other_start_times_horizons_and_steps(oracle, t0, horizon, dt):
    """At a 2 s horizon the trajectories differ by up to LONG_GAP per block (cause not yet found); everything else is exact there too, and the CUDA step of a
    cold start is certified as the KKT point of the oracle's QP."""
    import qm_control_b200 as q
    from qm_control_b200 import synthetic
    import test_mpc_twin_cpu as mt
    B = 6; prob, _ = synthetic.make_batch(np.arange(B), config=4, t0=t0, horizon=horizon)
    S.with_schedule(prob, B - 1, *S.single_foot(2, t0, horizon, 0.23))                      # one foot down: an odd input count on every grid
    solver = q.Solver(batch=B, dt=dt, time_horizon=horizon); oracle.mpc_set(dt=dt, horizon=horizon)
    try:
        _, res = _two_ticks(oracle, solver, prob)
        if horizon > 1.5:
            cold = q.Solver(batch=B, dt=dt, time_horizon=horizon); cold.mpc_solve(prob); dx, du, _ = cold.debug_get_step()
            for b in (0, B - 1):
                qp = oracle.mpc_qp({k: v[b:b + 1] for k, v in prob.items()}, solver.nmax, max_k=solver.nmax); n = qp["n_nodes"]
                qp["dx"][:n] = dx[b, :n]; qp["du"][:n - 1] = np.where(qp["is_event"][:n - 1, None] != 0, 0.0, du[b, :n - 1])   # the jump map has no input
                mt.assert_kkt_point(qp)
    finally:
        oracle.mpc_set(dt=0.015, horizon=1.0)
    assert res[0][1]["t"][0, 0] == t0 and abs(res[0][1]["t"][0, res[0][1]["n_nodes"][0] - 1] - (t0 + horizon)) < 1e-9
    if horizon <= 1.5:
        _check(res, "grid t0=%g T=%g dt=%g" % (t0, horizon, dt))
        return
    for tick, (out, ref) in enumerate(res):
        assert np.all((out["status"] & ~NO_STEP) == 0), np.unique(out["status"])
        np.testing.assert_array_equal(out["step_info"][:, 0], ref["dbg"][:, 0])
        np.testing.assert_allclose(out["step_info"][:, 1], ref["dbg"][:, 4], rtol=1e-6, atol=1e-8)
        assert_traj(out, ref, LONG_GAP, tag="grid T=%g tick %d" % (horizon, tick))            # grid (node count, times, events) exact inside


def test_target_knot_counts(oracle):
    """1, 3 and 4 knots, before t0, inside the horizon and ending before tf: the interpolation holds the first and the last knot."""
    import qm_control_b200 as q
    from qm_control_b200 import synthetic
    B = 6; prob, _ = synthetic.make_batch(np.arange(B), config=5); t0 = T0
    layouts = [[t0 - 0.1], [t0 - 0.2, t0 + 0.3, t0 + 0.6], [t0 - 0.05, t0 + 0.1, t0 + 0.5, t0 + 0.8], [t0 + 0.2], [t0, t0 + 0.25, t0 + 0.45], [t0 + 0.1, t0 + 0.2, t0 + 0.3, t0 + 0.4]]
    a, z = prob["target_states"][:, 0].copy(), prob["target_states"][:, 1].copy()
    for b, knots in enumerate(layouts):
        k = len(knots); prob["n_target"][b] = k; prob["target_times"][b] = 0.0; prob["target_times"][b, :k] = knots
        for i in range(k):
            w = (i + 1) / (k + 1); prob["target_states"][b, i] = (1 - w) * a[b] + w * z[b]
            prob["target_states"][b, i, 8] += 0.02 * (i % 2)       # a non-monotone base height through the knots
    solver = q.Solver(batch=B, dt=DT); oracle.mpc_set(dt=DT, horizon=H)
    _, res = _two_ticks(oracle, solver, prob)
    _check(res, "target knots")


def test_warm_start_across_an_event(oracle):
    """an event at t0 + 5 ms: the second tick (t0 + 10 ms) starts in the new mode from the previous solution."""
    import qm_control_b200 as q
    from qm_control_b200 import synthetic
    B = 5; prob, _ = synthetic.make_batch(np.arange(B), config=4)
    for b, m0 in enumerate((9, 6, 7, 8, 14)):
        ev = [T0 + 0.005 + P * i for i in range(-2, 6)]
        md = [15] + [m0 if i % 2 == 0 else 15 for i in range(len(ev) - 1)] + [15]  # stance until the event at t0 + 5 ms, m0 after it
        S.with_schedule(prob, b, ev, md)
    solver = q.Solver(batch=B, dt=DT); oracle.mpc_set(dt=DT, horizon=H)
    _, res = _two_ticks(oracle, solver, prob)
    _check(res, "warm start across an event")


def _fast_trot(t0=T0):
    """40 ms phases: 30 events, more nodes than the default handle holds at dt 0.015."""
    ev = [t0 - 0.02 + 0.04 * i for i in range(30)]
    return ev, [15] + [9 if i % 2 == 0 else 6 for i in range(29)] + [15]


def test_node_limit(oracle):
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import synthetic
    B = 5; F = 2; prob, wbc = synthetic.make_batch(np.arange(B), config=4); S.with_schedule(prob, F, *_fast_trot())
    oracle.mpc_set(dt=DT, horizon=H)
    (r, err), = S.oracle_per_robot(oracle, {k: v[F:F + 1] for k, v in prob.items()}, 400); assert err is None
    n = int(r["n_nodes"][0]); default = q.Solver(batch=B, dt=DT); assert n > default.nmax
    exact = q.Solver(batch=B, dt=DT, max_nodes=n); out = exact.mpc_solve(prob); ref = oracle.mpc_solve_batch(prob, n, nthreads=8)
    assert np.all((out["status"] & ~NO_STEP) == 0); np.testing.assert_array_equal(out["step_info"][:, 0], ref["dbg"][:, 0]); assert_traj(out, ref, MPC_TOL, tag="node limit exact")
    plain = {k: v.copy() for k, v in prob.items()}; S.with_schedule(plain, F, *_around(T0 + 0.0123))
    others = [b for b in range(B) if b != F]; keys = ("t0", "x0", "n_events", "event_times", "modes", "n_target", "target_times", "target_states"); dev = torch.device("cuda", 0)
    for solver in (q.Solver(batch=B, dt=DT, max_nodes=n - 1), default):
        got = solver.mpc_solve(prob); base = q.Solver(batch=B, dt=DT, max_nodes=solver.nmax).mpc_solve(plain)
        assert got["status"][F] & OVERFLOW and np.all((got["status"][others] & ~NO_STEP) == 0), got["status"]
        _same(got, base, others)
        solver.mpc_reset(); solver.mpc_solve_dev({k: torch.from_numpy(np.ascontiguousarray(prob[k])).to(dev) for k in keys}); torch.cuda.synchronize()
        sol = solver.mpc_get_solution(); assert sol["status"][F] & OVERFLOW; _same(sol, base, others)
        solver.mpc_reset(); cmd, st = solver.tick(prob, prob["t0"] + 0.002, wbc["rbd"], wbc["period"])
        assert (st[F] >> 8) & OVERFLOW and np.all((st[others] & ~(NO_STEP << 8)) == 0), [hex(int(v)) for v in st]
        cmd_plain, st_plain = q.Solver(batch=B, dt=DT, max_nodes=solver.nmax).tick(plain, plain["t0"] + 0.002, wbc["rbd"], wbc["period"])
        assert np.array_equal(cmd[others], cmd_plain[others]) and np.array_equal(st[others], st_plain[others])
        _same(solver.mpc_get_solution(), q.Solver(batch=B, dt=DT, max_nodes=solver.nmax).mpc_solve(plain), others)


def test_policy_eval_at_edge_times(oracle):
    import qm_control_b200 as q
    cases = {k: v for k, v in _placed().items() if k in ("node 20 +0", "node 20 +2e-06", "at t0", "pair 0.005 apart")}
    names, prob, _ = _batch(cases); B = len(names); solver = q.Solver(batch=B, dt=DT); oracle.mpc_set(dt=DT, horizon=H)
    solver.mpc_solve(prob)                                                     # the handle keeps the mode schedule policy_eval reads the mode from
    ref = oracle.mpc_solve_batch(prob, solver.nmax, nthreads=8); solver.mpc_set_solution(ref)
    queries = [[] for _ in range(B)]
    for b in range(B):
        n = int(ref["n_nodes"][b]); t = ref["t"][b, :n]; e = ref["event"][b, :n]; ne = prob["n_events"][b]; ev = prob["event_times"][b, :ne]
        qs = [T0 - 1e-3, t[-1], t[-1] + 0.05] + list(t)
        for te in ev:
            qs += [te, te - 1e-9, te + 1e-9]
        qs += [0.5 * (t[k] + t[k + 1]) for k in range(n - 1) if e[k] == 1]      # pre/post-event node pair
        queries[b] = qs
    L = max(len(qs) for qs in queries)
    for i in range(L):
        tq = np.array([queries[b][i % len(queries[b])] for b in range(B)])
        xd, ud, mode = solver.policy_eval(tq)
        for b in range(B):
            n = ref["n_nodes"][b]; ne = prob["n_events"][b]
            x, u, m = oracle.evaluate_policy(ref["t"][b, :n], ref["event"][b, :n], ref["x"][b, :n], ref["u"][b, :n], prob["event_times"][b, :ne], prob["modes"][b, :ne + 1], tq[b])
            np.testing.assert_allclose(xd[b], x, rtol=0, atol=1e-12, err_msg="%s t=%r" % (names[b], tq[b]))
            np.testing.assert_allclose(ud[b], u, rtol=0, atol=1e-10, err_msg="%s t=%r" % (names[b], tq[b])); assert mode[b] == m, (names[b], tq[b])
