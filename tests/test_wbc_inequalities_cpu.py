"""The WBC regimes of tests/_wbc_regimes.py reach what they are meant to reach, and the oracle's cascade is certified on them.

The regimes put the HoQp inequalities where they bind (fast-moving states, friction pyramids at their edges and apex, saturated torques).  Checked on the
CPU: the fast states violate more than six level-0 rows at the minimum-norm level-0 point (more than fit beside the 18 task rows in 24), the edge and apex
states end with active pyramid rows, the saturated states with torques at their limits; and the oracle's three levels are KKT points of the literal level
problems (tests/test_wbc_twin_cpu.py) with the robot's own friction coefficient."""
import numpy as np
import pytest

import _wbc_regimes as R
import test_wbc_twin_cpu as tw

LEVEL0_ROWS = 14        # violated rows the kernel's level 0 holds beside its 18 task rows (MAXR0 = 32 in wbc_kernel.cu)
ORACLE_OFF = {"init_fast": {3, 24}}   # robots whose oracle result misses the level-1 certificate (the arm-tracking branch leaves a swing leg untasked)


@pytest.fixture(scope="module")
def oracles(tmp_path_factory):
    return R.Oracles(tmp_path_factory.mktemp("wbc_mu"))


def _robots(oracles, name):
    """per robot of the regime: (inputs, level-0 tasks, oracle levels, level-0 emulation)"""
    g = tw._gains(); r = R.regime(name, oracles(0.3).model_info()["mass"]); out = []
    for b in range(len(r["mode"])):
        orc = oracles(r["wbc_friction"][b]); m = int(r["mode"][b])
        dbg = orc.wbc_debug(r["x_des"][b], r["u_des"][b], r["rbd"][b], m, r["period"][b], r["time"][b], input_last=r["input_last"][b])
        (A0, b0, D0, f0), _, _, M = tw._tasks(orc, dbg, r["u_des"][b], m, r["time"][b], g, r["wbc_friction"][b])
        out.append(dict(A0=A0, b0=b0, D0=D0, f0=f0, M=M, levels=dbg["levels"], emu=R.level0_passes(A0, b0, D0, f0), nc=bin(m).count("1")))
    return r, out


@pytest.mark.parametrize("name", R.REGIMES)
def test_regime_reaches_its_inequalities(oracles, name):
    r, robots = _robots(oracles, name)
    B = len(robots)
    first = np.array([x["emu"][2] for x in robots]); largest = np.array([max(x["emu"][1]) for x in robots])
    vstar = np.array([np.max(np.maximum(0.0, x["D0"] @ x["levels"][0] - x["f0"])) for x in robots])
    assert np.all(vstar < 1e-8), vstar.max()                      # level 0 is feasible: no regime needs slack for this model
    assert np.all(largest <= LEVEL0_ROWS), largest                 # every violated set fits the kernel's level 0
    final = []
    for x in robots:
        x2 = x["levels"][2]; fcap = x["f0"] + np.maximum(0.0, x["D0"] @ x["levels"][0] - x["f0"]); viol = x["D0"] @ x2 - fcap
        act = viol > -1e-7 * (1.0 + np.abs(fcap)); pyr = act[36:36 + 5 * x["nc"]].reshape(x["nc"], 5) if x["nc"] else np.zeros((0, 5), bool)
        final.append((int(act[:36].sum()), int(pyr.sum()), int(pyr.all(axis=1).sum())))
    final = np.array(final)
    print("%s: %d robots, violated rows at the minimum-norm point max %d (%d robots > 6), largest set %d, active torque / pyramid rows %s / %s, apex feet %d"
          % (name, B, first.max(), (first > 6).sum(), largest.max(), final[:, 0].max(), final[:, 1].max(), final[:, 2].sum()))
    kind = name[5:] if name.startswith("init_") else name
    if name == "fast":
        assert (first > 6).sum() >= 3 and largest.max() > 6          # more than the six rows that fit beside the task rows in a buffer of 24
        big = [(18 + n, k) for x in robots for n, k in zip(x["emu"][1], x["emu"][3]) if 18 + n > 24]
        assert any(k < n and k <= 27 for n, k in big), big             # a rank-deficient pass of more than 24 rows that forms its Gram (KG0 = 27)
        assert any(k < n and k > 27 for n, k in big), big              # one that solves on its independent rows and checks the dependent ones
    if kind in ("edge", "apex"):
        assert np.all(final[:, 1] > 0)                                # every robot ends with an active pyramid row
    if kind == "apex":
        assert final[:, 2].sum() >= B // 2                            # at least half the robots hold a foot at the apex, all five rows active
    if kind == "saturated":
        assert np.all(final[:, 0] > 0)                                # every robot ends with a torque at its limit


@pytest.mark.parametrize("name", R.REGIMES)
def test_oracle_passes_the_certificate(oracles, name):
    g = tw._gains(); r = R.regime(name, oracles(0.3).model_info()["mass"]); off = set()
    for b in range(len(r["mode"])):
        try:
            tw.assert_levels_are_kkt_points(oracles(r["wbc_friction"][b]), g, r["x_des"][b], r["u_des"][b], r["rbd"][b], r["mode"][b], r["period"][b],
                                            r["time"][b], r["input_last"][b], tag=(name, b), mu=r["wbc_friction"][b])
        except AssertionError:
            off.add(b)
    assert off == ORACLE_OFF.get(name, set()), sorted(off)


def test_twin_friction_coefficient_reaches_the_pyramid(oracles):
    """_tasks(mu=...) builds the pyramid of that coefficient: rows [Fx - mu Fz, -Fx - mu Fz, Fy - mu Fz, -Fy - mu Fz] after -Fz"""
    r = R.regime("edge", oracles(0.3).model_info()["mass"]); g = tw._gains(); orc = oracles(0.3)
    dbg = orc.wbc_debug(r["x_des"][0], r["u_des"][0], r["rbd"][0], int(r["mode"][0]), r["period"][0], 12.0, input_last=r["input_last"][0])
    for mu in R.MUS:
        D0 = tw._tasks(orc, dbg, r["u_des"][0], int(r["mode"][0]), 12.0, g, mu)[0][2]
        np.testing.assert_array_equal(D0[36:41, 24:27], [[0, 0, -1], [1, 0, -mu], [-1, 0, -mu], [0, 1, -mu], [0, -1, -mu]])
