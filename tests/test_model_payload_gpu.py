"""The controller's model payload on the device (qmb200_set_model_payload, closed_loop.run(model_payload=...)).

Specification: a robot whose model payload is p computes what a handle built from the edited URDF (tests/_payload_urdf.py: the point masses as
extra fixed links) computes for it.  Every entry point is compared with such handles on the same robots' inputs, per block at 1e-8; one sample
also goes against the oracle on the edited URDF.  Then bit-identity of a zero payload and of a permuted batch, and closed-loop runs on an H100."""
import numpy as np
import pytest

from _parity import MPC_TOL, TICK_TOL, X_BLOCKS, assert_cmd, assert_traj, block_errors
from _payload_urdf import edited_urdf
from qm_control_b200 import _lib

pytestmark = pytest.mark.gpu

TOL = 1e-8
PL = {n: i for i, n in enumerate(_lib.PAYLOAD_LAYOUT)}
VALUES = [[1.5, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0],             # EE only
          [2.0, 0.03, -0.02, 0.05, 0.0, 0.0, 0.0, 0.0],          # EE with an offset
          [0.0, 0.0, 0.0, 0.0, 4.0, 0.12, -0.05, 0.09],          # base only, offset
          [0.7, -0.01, 0.04, 0.02, 5.0, -0.2, 0.1, 0.06]]        # both
PER = 8
B = PER * len(VALUES)
DT = 0.015


def _payload_rows():
    return np.repeat(np.array(VALUES), PER, axis=0)   # robots [v * PER, (v + 1) * PER) carry VALUES[v]


def _rows(v):
    return np.arange(v * PER, (v + 1) * PER)


def _inputs(config=5):
    from qm_control_b200 import synthetic
    prob, wbc = synthetic.make_batch(np.arange(B), config=config)
    return prob, wbc


def _solver(urdf=None, wbc_variant=0, batch=B):
    import qm_control_b200 as q
    return q.Solver(interface=q.QMInterface(urdfFile=urdf), batch=batch, device=0, dt=DT, wbc_variant=wbc_variant)


@pytest.fixture(scope="module")
def urdfs(tmp_path_factory):
    d = tmp_path_factory.mktemp("payload_urdf")
    return [edited_urdf(d, v, name="robot_payload_%d.urdf" % i) for i, v in enumerate(VALUES)]


@pytest.fixture(scope="module")
def handles(urdfs):
    """(told, refs) per WBC variant: one handle with the per-robot model payload, one handle per edited URDF"""
    out = {}
    for variant in (0, 1):
        told = _solver(wbc_variant=variant); told.set_model_payload(_payload_rows())
        out[variant] = (told, [_solver(u, wbc_variant=variant) for u in urdfs])
    return out


def _fresh(*solvers):
    for s in solvers:
        s.mpc_reset(); s.wbc_set_input_last(None)


def _x_close(a, b, tag):
    lv = block_errors(a, b, X_BLOCKS); bad = {k: v for k, v in lv.items() if not v < TOL}
    assert not bad, "%s: %s" % (tag, bad)


@pytest.mark.parametrize("solver_name", ["sqp", "ipm", "ddp"])
def test_mpc_solve_equals_the_edited_urdf(handles, solver_name):
    """Solutions and status words per robot.  A DDP robot whose step fails (QMB200 MPC flags NOT_PD | NO_STEP, alpha 0) keeps the nominal
    single-shooting rollout of its initial guess; on these cold-started synthetic problems that rollout diverges (merit 5e4-1e6), and it amplifies the
    last-bit differences of the SRBD constants to ~1e-5 in the base angles (measured on H100; the inputs agree to 1e-16).  For those robots the
    inputs are compared; every robot with a step, the whole trajectory."""
    prob, _ = _inputs()
    told, refs = handles[0]
    try:
        for s in [told] + refs:
            s.mpc_set_solver(solver_name)
        _fresh(told, *refs)
        got = told.mpc_solve(prob)
        for v, ref in enumerate(refs):
            want = ref.mpc_solve(prob); rows = _rows(v)
            np.testing.assert_array_equal(got["status"][rows], want["status"][rows])
            failed = (got["status"][rows] & 8) != 0   # MST_NOT_PD: no step was taken
            for b in rows[failed]:
                n = int(got["n_nodes"][b]); assert n == want["n_nodes"][b] and got["step_info"][b, 0] == want["step_info"][b, 0] == 0.0
                np.testing.assert_allclose(got["u"][b, :n], want["u"][b, :n], rtol=0, atol=TOL * max(10.0, np.max(np.abs(want["u"][b, :n]))))
            ok = rows[~failed]
            sub = lambda d: {k: d[k][ok] for k in ("n_nodes", "t", "event", "x", "u")}
            assert_traj(sub(got), sub(want), TOL, tag="model payload %s value %d" % (solver_name, v))
    finally:
        for s in [told] + refs:
            s.mpc_set_solver("sqp")


@pytest.mark.parametrize("variant", [0, 1])
def test_wbc_update_equals_the_edited_urdf(handles, variant):
    """All 54 outputs of WbcBase::update (both variants) on random desired states / inputs around the synthetic states."""
    prob, wbc = _inputs()
    told, refs = handles[variant]
    rng = np.random.default_rng(7 + variant)
    x_des = prob["x0"] + rng.uniform(-0.01, 0.01, (B, 30)); u_des = np.zeros((B, 30)); u_des[:, 2:12:3] = 80.0; u_des[:, 12:] = rng.uniform(-0.1, 0.1, (B, 18))
    mode = np.full(B, 15, dtype=np.int32); mode[1::2] = 9   # stance and a trot phase (LF + RH)
    _fresh(told, *refs)
    cmd, st = told.wbc_update(x_des, u_des, wbc["rbd"], mode, wbc["period"], wbc["time"])
    for v, ref in enumerate(refs):
        c, s = ref.wbc_update(x_des, u_des, wbc["rbd"], mode, wbc["period"], wbc["time"]); rows = _rows(v)
        assert_cmd(cmd[rows], c[rows], TOL, tag="model payload wbc variant %d value %d" % (variant, v))
        np.testing.assert_array_equal(st[rows], s[rows])


def test_update_equals_the_edited_urdf(handles):
    """observation -> evaluatePolicy -> WBC -> control law on the stored policy of one solve"""
    prob, wbc = _inputs()
    told, refs = handles[0]
    _fresh(told, *refs)
    told.mpc_solve(prob)
    t_obs = prob["t0"].copy(); x_obs = prob["x0"].copy(); jc = np.zeros((B, 18, 5)); ap = np.zeros((B, 6)); lt = prob["t0"].copy()
    got = told.update(wbc["rbd"], wbc["period"], t_obs, x_obs, jc, ap, lt)
    for v, ref in enumerate(refs):
        ref.mpc_solve(prob); want = ref.update(wbc["rbd"], wbc["period"], t_obs, x_obs, jc, ap, lt); rows = _rows(v)
        _x_close(got[1][rows], want[1][rows], "observation value %d" % v)
        assert_cmd(got[5][rows], want[5][rows], TOL, tag="model payload update value %d" % v)
        jg, jw = got[2][rows], want[2][rows]
        assert np.max(np.abs(jg - jw)) <= TOL * max(1.0, np.max(np.abs(jw))), "joint commands value %d" % v
        np.testing.assert_array_equal(got[6][rows], want[6][rows])


@pytest.mark.parametrize("chunks", [1, 2])
def test_tick_equals_the_edited_urdf(handles, chunks):
    prob, wbc = _inputs()
    told, refs = handles[0]
    t_eval = prob["t0"] + 0.002
    try:
        told.set_pipeline(chunks); _fresh(told, *refs)
        cmd, st = told.tick(prob, t_eval, wbc["rbd"], wbc["period"]); sol = told.mpc_get_solution()
        for v, ref in enumerate(refs):
            c, s = ref.tick(prob, t_eval, wbc["rbd"], wbc["period"]); rows = _rows(v)
            assert_cmd(cmd[rows], c[rows], TOL, tag="model payload tick chunks %d value %d" % (chunks, v))
            np.testing.assert_array_equal(st[rows], s[rows])
            sub = lambda d: {k: d[k][rows] for k in ("n_nodes", "t", "event", "x", "u")}
            assert_traj(sub(sol), sub(ref.mpc_get_solution()), TOL, tag="model payload tick traj value %d" % v)
    finally:
        told.set_pipeline(1)


def test_centroidal_state_from_rbd_equals_the_edited_urdf(handles):
    _, wbc = _inputs()
    told, refs = handles[0]
    x = told.centroidal_state_from_rbd(wbc["rbd"])
    for v, ref in enumerate(refs):
        rows = _rows(v); _x_close(x[rows], ref.centroidal_state_from_rbd(wbc["rbd"])[rows], "centroidal_state_from_rbd value %d" % v)
    from qm_control_b200 import QmbError
    with pytest.raises(QmbError, match="n must equal the batch size"):
        told.centroidal_state_from_rbd(wbc["rbd"][:3])


def test_tick_sample_against_the_oracle_on_the_edited_urdf(handles, urdfs):
    """The robots of the 'both' payload value against the oracle built from their edited URDF (the CPU reference of the whole tick)."""
    from _oracle import Oracle
    prob, wbc = _inputs()
    told, _ = handles[0]
    v = 3; rows = _rows(v); t_eval = prob["t0"] + 0.002
    _fresh(told)
    cmd, st = told.tick(prob, t_eval, wbc["rbd"], wbc["period"]); sol = told.mpc_get_solution()
    o = Oracle(urdf=urdfs[v]); o.mpc_set(dt=DT, horizon=1.0)
    sub = {k: np.asarray(a)[rows] for k, a in prob.items()}
    ref = o.tick_batch(sub, told.nmax, t_eval[rows], wbc["rbd"][rows], wbc["period"][rows], np.zeros((PER, 30)), nthreads=4)
    assert_cmd(cmd[rows], ref["cmd"], TICK_TOL, tag="model payload tick vs oracle")
    assert_traj({k: sol[k][rows] for k in ("n_nodes", "t", "event", "x", "u")}, ref, MPC_TOL, tag="model payload traj vs oracle")


def test_zero_model_payload_is_bit_identical_to_none():
    prob, wbc = _inputs(); t_eval = prob["t0"] + 0.002
    a = _solver(); b = _solver()
    try:
        b.set_model_payload(np.zeros((B, 8)))
        assert b.get_model_payload() is not None and a.get_model_payload() is None
        for chunks in (1, 2):
            for s in (a, b):
                s.set_pipeline(chunks); _fresh(s)
            ca, sa = a.tick(prob, t_eval, wbc["rbd"], wbc["period"]); cb, sb = b.tick(prob, t_eval, wbc["rbd"], wbc["period"])
            np.testing.assert_array_equal(ca, cb); np.testing.assert_array_equal(sa, sb)
            for k, val in a.mpc_get_solution().items():
                np.testing.assert_array_equal(val, b.mpc_get_solution()[k], err_msg=k)
    finally:
        a.close(); b.close()


def test_permuted_batch_is_bit_identical():
    prob, wbc = _inputs(); t_eval = prob["t0"] + 0.002
    perm = np.random.default_rng(3).permutation(B); pl = _payload_rows()
    a = _solver(); b = _solver()
    try:
        a.set_model_payload(pl); b.set_model_payload(pl[perm])
        ca, sa = a.tick(prob, t_eval, wbc["rbd"], wbc["period"])
        cb, sb = b.tick({k: np.asarray(val)[perm] for k, val in prob.items()}, t_eval[perm], wbc["rbd"][perm], wbc["period"][perm])
        np.testing.assert_array_equal(ca[perm], cb); np.testing.assert_array_equal(sa[perm], sb)
        xa = a.centroidal_state_from_rbd(wbc["rbd"]); xb = b.centroidal_state_from_rbd(wbc["rbd"][perm])
        np.testing.assert_array_equal(xa[perm], xb)
    finally:
        a.close(); b.close()


def test_validation_and_round_trip():
    s = _solver(batch=4)
    try:
        assert s.get_model_payload() is None
        pl = np.zeros((4, 8)); pl[:, PL["m_ee"]] = [0.0, 0.5, 1.0, 2.0]; pl[2, PL["o_base_z"]] = 0.1
        s.set_model_payload(pl); np.testing.assert_array_equal(s.get_model_payload(), pl)
        from qm_control_b200 import QmbError
        for bad, msg in ((np.nan, "payload must be finite"), (-1.0, "payload masses must be >= 0")):
            b = pl.copy(); b[1, PL["m_base"]] = bad
            with pytest.raises(QmbError, match=msg):
                s.set_model_payload(b)
            np.testing.assert_array_equal(s.get_model_payload(), pl)   # unchanged on rejection
        assert s.sim_get_robot_params()["payload"] is None   # independent of the plant's payload
        s.set_model_payload(None); assert s.get_model_payload() is None
    finally:
        s.close()


# ---------------- closed loop ----------------
NL = 64


def _run(**kw):
    """closed_loop.run on a fresh handle (the MPC's warm start and the WBC's last input live in the handle)"""
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    s = q.Solver(batch=NL, device=0)
    try:
        r = closed_loop.run(s, **kw)
        assert s.get_model_payload() is None and s.sim_get_robot_params()["payload"] is None   # restored
        return r
    finally:
        s.close()


def _upright(r):
    base = r["base"]
    return np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3) & \
        np.all((r["status"] & 4) == 0, axis=0)


def test_closed_loop_zero_model_payload_is_bit_identical():
    plain = _run(duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0))
    zero = _run(duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), model_payload=np.zeros((NL, 8)))
    for k in ("base", "ee", "status", "contact", "q", "v", "start_base", "start_ee"):
        np.testing.assert_array_equal(plain[k], zero[k], err_msg=k)


def test_closed_loop_restores_model_payload_on_error():
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    s = q.Solver(batch=NL, device=0)
    try:
        prev = np.zeros((NL, 8)); prev[:, PL["m_ee"]] = 0.25; s.set_model_payload(prev)
        with pytest.raises(ValueError):
            closed_loop.run(s, duration=0.01, cmd_vel=np.zeros(3), model_payload="plant")
        np.testing.assert_array_equal(s.get_model_payload(), prev)
        with pytest.raises(ValueError):
            closed_loop.run(s, duration=0.01, model_payload="estimate")
        np.testing.assert_array_equal(s.get_model_payload(), prev)
    finally:
        s.close()


_STANCE = {}


def _stance_runs():
    """Stance, 1 s, EE payload 0-2 kg in the plant: the controller not told, and told (model_payload='plant')"""
    if not _STANCE:
        m = np.linspace(0.0, 2.0, NL); pl = np.zeros((NL, 8)); pl[:, PL["m_ee"]] = m
        _STANCE.update(m=m, unknown=_run(duration=1.0, gait="stance", payload=pl), told=_run(duration=1.0, gait="stance", payload=pl, model_payload="plant"))
    return _STANCE["m"], _STANCE["unknown"], _STANCE["told"]


def test_closed_loop_stance_told_payload_reduces_the_ee_excursion():
    m, unknown, told = _stance_runs()
    dz = lambda r: np.max(np.abs(r["ee"][:, :, 2] - r["start_ee"][None, :, 2]), axis=0)
    du, dt = dz(unknown), dz(told); heavy = m >= 1.0
    print("stance EE payload, max |dz| at 0 / 1 / 2 kg: not told %.1f / %.1f / %.1f mm, told %.1f / %.1f / %.1f mm; told max over >= 1 kg %.1f mm" % (
        du[0] * 1e3, du[NL // 2] * 1e3, du[-1] * 1e3, dt[0] * 1e3, dt[NL // 2] * 1e3, dt[-1] * 1e3, np.max(dt[heavy]) * 1e3))
    assert np.all(_upright(told)) and np.all(told["contact"] == 15) and np.all(told["status"] == 0)
    assert np.all(dt[heavy] < du[heavy])


def test_closed_loop_stance_told_ee_holds_its_pose_within_2cm_under_2kg():
    _, _, told = _stance_runs()
    assert np.max(np.abs(told["ee"][:, :, 2] - told["start_ee"][None, :, 2])) < 0.02


def test_closed_loop_trot_with_a_wrong_payload_estimate_stays_up():
    """The controller is told 1 kg, the gripper carries 2 kg."""
    plant = np.zeros((NL, 8)); plant[:, PL["m_ee"]] = 2.0; model = np.zeros((NL, 8)); model[:, PL["m_ee"]] = 1.0
    r = _run(duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), payload=plant, model_payload=model)
    up = _upright(r); dist = np.linalg.norm(r["base"][-1, :, :2] - r["start_base"][:, :2], axis=1)
    print("trot, plant 2 kg / model 1 kg: %d/%d up, base distance p50 %.3f m" % (int(up.sum()), NL, float(np.median(dist))))
    assert np.all(up)
