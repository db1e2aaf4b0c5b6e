"""The oracle on the contact modes the three gaits of make_batch never produce: one and three feet down (15 and 13 equality rows per node), the lateral
and fore/hind pairs, every one of the 16 masks.  The certificates of tests/test_mpc_twin_cpu.py, tests/test_wbc_twin_cpu.py and
tests/test_wbc_mpc_variant_cpu.py, run on those modes, so the GPU comparisons of tests/test_contact_modes_gpu.py rest on a pinned reference."""
import numpy as np
import pytest

import _schedules as S
import test_mpc_twin_cpu as mt
import test_wbc_mpc_variant_cpu as mv
import test_wbc_twin_cpu as tw
from qm_control_b200 import synthetic

NMAX = 128
SCHEDULES = {"dynamic_walk": lambda t0: S.gait_schedule("dynamic_walk", t0, 0.37), "static_walk": lambda t0: S.gait_schedule("static_walk", t0, 0.57),
             "pawup": lambda t0: S.gait_schedule("pawup", t0, 0.17), "single_foot_8": lambda t0: S.single_foot(8, t0, phase=0.23),
             "single_foot_1": lambda t0: S.single_foot(1, t0, phase=0.61), "all_masks": lambda t0: S.all_masks(t0, phase=0.17)}


def _prob(name, robot=1):
    prob, wbc = synthetic.make_batch(np.array([robot]), config=4)
    return S.with_schedule(prob, 0, *SCHEDULES[name](prob["t0"][0])), wbc


@pytest.mark.parametrize("name", list(SCHEDULES))
def test_sqp_step_is_the_kkt_point_on_every_contact_mode(oracle, name):
    oracle.mpc_set(dt=0.015, horizon=1.0); prob, _ = _prob(name)
    qp = oracle.mpc_qp(prob, NMAX); assert qp["n_nodes"] - 1 >= 67
    assert mt.assert_kkt_point(qp) - {12, 14, 16}                                       # every schedule reaches a row count the three gaits of make_batch never do


def test_the_schedules_reach_every_row_count(oracle):
    """the certified schedules together give nodes with 12, 13, 14, 15 and 16 equality rows."""
    oracle.mpc_set(dt=0.015, horizon=1.0); rows = set()
    for name in SCHEDULES:
        qp = oracle.mpc_qp(_prob(name)[0], NMAX); N = qp["n_nodes"] - 1
        rows |= set(qp["ng"][:N][qp["is_event"][:N] == 0].tolist())
    assert rows == {12, 13, 14, 15, 16}, sorted(rows)


@pytest.mark.parametrize("feet", [1, 3])
def test_derivatives_by_finite_differences_with_one_and_three_feet_down(oracle, feet):
    oracle.mpc_set(dt=0.015, horizon=1.0); prob, _ = _prob("single_foot_8" if feet == 1 else "dynamic_walk")
    qp = oracle.mpc_qp(prob, NMAX); sol = oracle.mpc_solve_batch(prob, NMAX, nthreads=1); n = int(sol["n_nodes"][0]); ev = sol["event"][0, :n]
    et = prob["event_times"][0, :prob["n_events"][0]]; md = prob["modes"][0]; checked = 0
    for k in range(2, n - 2):
        if ev[k] != 0 or ev[k + 1] != 0 or qp["is_event"][k] or bin(S.mode_at(et, md, sol["t"][0, k])).count("1") != feet:
            continue
        mode = mt.assert_node_derivatives(oracle, prob, qp, sol, k)
        assert qp["ng"][k] == S.ndep(mode) == 16 - feet
        checked += 1
        if checked == 2:
            break
    assert checked == 2


def _wbc_inputs(masks, mass, seed_ids):
    """config-3 robots with their contact mask replaced: weight-compensating forces on the stance feet, perturbed, zero on the swing feet."""
    prob, wbc = synthetic.make_batch(seed_ids, config=3)
    u = np.zeros((len(masks), 30))
    for b, m in enumerate(masks):
        nc = bin(m).count("1")
        for f in range(4):
            if (m >> (3 - f)) & 1:
                u[b, 3 * f + 2] = mass * 9.81 / nc
    u = u + synthetic.uniform(77, seed_ids, 1, 30, -1.0, 1.0) * np.r_[np.full(12, 5.0), np.full(18, 0.2)]
    for b, m in enumerate(masks):
        for f in range(4):
            if not (m >> (3 - f)) & 1:
                u[b, 3 * f:3 * f + 3] = 0.0
    return prob["x0"].copy(), u, np.asarray(masks, dtype=np.int32), wbc


# The oracle's HoQp cascade is not a certified optimum everywhere on the new modes; those cases stay here as strict xfails so a change of either side shows:
#   init branch (t < 10) with swing feet: mask 0 hits the oracle's QP iteration cap, masks 1 and 12 leave level 2 outside a level-0 inequality;
#   HierarchicalMpcWbc with masks 4, 2, 7, 11, 13, 14: level 1 is not a KKT point of its level problem (NNLS residual 0.06 .. 6e3).
# The CUDA results on these robots pass the certificate (tests/test_contact_modes_gpu.py::test_wbc_on_all_16_masks): the oracle is the side that is off.
UNCERTIFIED_INIT = {0, 1, 12}
UNCERTIFIED_VARIANT1 = {4, 2, 7, 11, 13, 14}


def _maybe_xfail(mask, bad, why):
    return pytest.param(mask, marks=pytest.mark.xfail(strict=True, reason=why)) if mask in bad else mask


@pytest.mark.parametrize("mask", range(16))
def test_wbc_levels_are_kkt_points_on_all_16_masks(oracle, mask):
    g = tw._gains(); ids = np.arange(16); x_des, u_des, mode, wbc = _wbc_inputs(list(range(16)), oracle.model_info()["mass"], ids)
    il = synthetic.uniform(78, ids, 2, 30, -0.1, 0.1)
    tw.assert_levels_are_kkt_points(oracle, g, x_des[mask], u_des[mask], wbc["rbd"][mask], mode[mask], wbc["period"][mask], 12.0, il[mask], tag=("mask", mask))


@pytest.mark.parametrize("mask", [_maybe_xfail(m, UNCERTIFIED_INIT, "oracle's init-branch cascade not certified with swing feet") for m in range(16)])
def test_wbc_init_branch_levels_are_kkt_points_on_all_16_masks(oracle, mask):
    g = tw._gains(); ids = np.arange(16); x_des, u_des, mode, wbc = _wbc_inputs(list(range(16)), oracle.model_info()["mass"], ids)
    il = synthetic.uniform(78, ids, 2, 30, -0.1, 0.1)
    tw.assert_levels_are_kkt_points(oracle, g, x_des[mask], u_des[mask], wbc["rbd"][mask], mode[mask], wbc["period"][mask], 3.0, il[mask], tag=("mask", mask))


VARIANT1_MASKS = [8, 4, 2, 1, 7, 11, 13, 14]


@pytest.mark.parametrize("mask", [_maybe_xfail(m, UNCERTIFIED_VARIANT1, "oracle's HierarchicalMpcWbc level 1 not a KKT point") for m in VARIANT1_MASKS])
def test_wbc_mpc_variant_levels_with_one_and_three_feet_down(oracle, mask):
    ids = np.arange(len(VARIANT1_MASKS)); g = tw._gains(); b = VARIANT1_MASKS.index(mask)
    x_des, u_des, mode, wbc = _wbc_inputs(VARIANT1_MASKS, oracle.model_info()["mass"], ids)
    il = u_des + synthetic.uniform(78, ids, 2, 30, -0.002, 0.002)
    mv.assert_variant_levels(oracle, g, x_des[b], u_des[b], wbc["rbd"][b], mode[b], wbc["period"][b], il[b], tag=("mask", mask))
