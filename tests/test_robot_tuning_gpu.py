"""Per-robot controller tuning on the device (qmb200_set_robot_tuning, closed_loop.run(tuning=...)).

Specification: a robot whose tuning row is r computes what a handle built from task.info and a gains file edited to r (tests/_tuning.py), with r's arm
gains set through qmb200_set_arm_gains, computes for it.  Only the source of each value changes, so the comparison is bit for bit.  Then neutral rows
against no rows, a permuted batch, a sample against the oracle, the told friction pyramid, the entry points and a closed-loop run."""
import numpy as np
import pytest

from _parity import MPC_TOL, TICK_TOL, assert_cmd, assert_traj
from _tuning import L, distinct_rows, edited_files, field

pytestmark = pytest.mark.gpu

NV, PER = 8, 8
B = NV * PER
DT = 0.015
TRAJ = ("n_nodes", "t", "event", "x", "u", "status", "step_info")


def _solver(task=None, gains=None, wbc_variant=0, batch=B):
    import qm_control_b200 as q
    return q.Solver(interface=q.QMInterface(taskFile=task, wbcGainsFile=gains), batch=batch, device=0, dt=DT, wbc_variant=wbc_variant)


def _inputs(config=5):
    from qm_control_b200 import synthetic
    return synthetic.make_batch(np.arange(B), config=config)


def _rows(v):
    return np.arange(v * PER, (v + 1) * PER)


def _fresh(*solvers):
    for s in solvers:
        s.mpc_reset(); s.wbc_set_input_last(None)


@pytest.fixture(scope="module")
def values():
    s = _solver(batch=1)
    try:
        return distinct_rows(s.get_handle_tuning(), NV)
    finally:
        s.close()


@pytest.fixture(scope="module")
def files(values, tmp_path_factory):
    d = tmp_path_factory.mktemp("tuning")
    return [edited_files(d, r, str(v)) for v, r in enumerate(values)]


@pytest.fixture(scope="module")
def handles(values, files):
    """(told, refs) per WBC variant: one handle with the per-robot rows, one handle per edited file pair holding that row as its own values"""
    out = {}
    for variant in (0, 1):
        told = _solver(wbc_variant=variant); told.set_robot_tuning({k: np.repeat(values[:, off:off + w], PER, axis=0).reshape(B, w) if w > 1 else np.repeat(values[:, off], PER)
                                                                     for k, (off, w) in L.items()})
        refs = []
        for r, (task, gains) in zip(values, files):
            s = _solver(task, gains, wbc_variant=variant); s.set_arm_gains(field(r, "kp_arm_wbc"), field(r, "kd_arm_wbc")); refs.append(s)
        out[variant] = (told, refs)
    yield out
    for told, refs in out.values():
        for s in [told] + refs:
            s.close()


def _same(a, b, keys, rows, tag):
    for k in keys:
        np.testing.assert_array_equal(np.asarray(a[k])[rows], np.asarray(b[k])[rows], err_msg="%s: %s" % (tag, k))


def test_rows_are_stored_per_robot(handles, values):
    told, refs = handles[0]
    got = told.get_robot_tuning()
    for v, ref in enumerate(refs):
        np.testing.assert_array_equal(ref.get_handle_tuning(), values[v])   # the edited files hold the row
        for k, (off, w) in L.items():
            np.testing.assert_array_equal(np.asarray(got[k])[_rows(v)].reshape(PER, w), np.repeat(values[v:v + 1, off:off + w], PER, axis=0))


@pytest.mark.parametrize("solver_name", ["sqp", "ipm", "ddp"])
def test_mpc_solve_equals_the_edited_handle_bit_for_bit(handles, solver_name):
    prob, _ = _inputs()
    told, refs = handles[0]
    try:
        for s in [told] + refs:
            s.mpc_set_solver(solver_name)
        _fresh(told, *refs)
        got = told.mpc_solve(prob)
        for v, ref in enumerate(refs):
            _same(got, ref.mpc_solve(prob), TRAJ, _rows(v), "%s value %d" % (solver_name, v))
    finally:
        for s in [told] + refs:
            s.mpc_set_solver("sqp")


@pytest.mark.parametrize("variant", [0, 1])
def test_wbc_update_equals_the_edited_handle_bit_for_bit(handles, variant):
    prob, wbc = _inputs()
    told, refs = handles[variant]
    rng = np.random.default_rng(7 + variant)
    x_des = prob["x0"] + rng.uniform(-0.01, 0.01, (B, 30)); u_des = np.zeros((B, 30)); u_des[:, 2:12:3] = 80.0; u_des[:, 0:12:3] = 15.0; u_des[:, 12:] = rng.uniform(-0.1, 0.1, (B, 18))
    mode = np.full(B, 15, dtype=np.int32); mode[1::2] = 9
    for time in (wbc["time"], wbc["time"] + 12.0):   # before and after the 10 s arm-tracking phase of HierarchicalWbc
        _fresh(told, *refs)
        cmd, st = told.wbc_update(x_des, u_des, wbc["rbd"], mode, wbc["period"], time)
        for v, ref in enumerate(refs):
            c, s = ref.wbc_update(x_des, u_des, wbc["rbd"], mode, wbc["period"], time); rows = _rows(v)
            np.testing.assert_array_equal(cmd[rows], c[rows], err_msg="variant %d value %d" % (variant, v)); np.testing.assert_array_equal(st[rows], s[rows])


def test_update_equals_the_edited_handle_bit_for_bit(handles):
    """observation -> evaluatePolicy -> WBC -> control law (the row's arm gains in the joint commands)"""
    prob, wbc = _inputs()
    told, refs = handles[0]
    _fresh(told, *refs)
    told.mpc_solve(prob)
    t_obs = prob["t0"].copy(); x_obs = prob["x0"].copy(); jc = np.zeros((B, 18, 5)); ap = np.zeros((B, 6)); lt = prob["t0"].copy()
    got = told.update(wbc["rbd"], wbc["period"], t_obs, x_obs, jc, ap, lt)
    for v, ref in enumerate(refs):
        ref.mpc_solve(prob); want = ref.update(wbc["rbd"], wbc["period"], t_obs, x_obs, jc, ap, lt); rows = _rows(v)
        for i in range(len(got)):
            np.testing.assert_array_equal(got[i][rows], want[i][rows], err_msg="output %d value %d" % (i, v))
        assert np.all(got[2][rows][:, 12:, 3] == field(_value_row(told, v), "kd_arm_wbc"))   # the row's arm gain reached the joint commands


def _value_row(told, v):
    t = told.get_robot_tuning(); b = v * PER
    return np.concatenate([np.atleast_1d(np.asarray(t[k])[b]) for k in L])


@pytest.mark.parametrize("chunks", [1, 2])
def test_tick_equals_the_edited_handle_bit_for_bit(handles, chunks):
    prob, wbc = _inputs()
    told, refs = handles[0]
    t_eval = prob["t0"] + 0.002
    try:
        told.set_pipeline(chunks); _fresh(told, *refs)
        cmd, st = told.tick(prob, t_eval, wbc["rbd"], wbc["period"]); sol = told.mpc_get_solution()
        for v, ref in enumerate(refs):
            c, s = ref.tick(prob, t_eval, wbc["rbd"], wbc["period"]); rows = _rows(v)
            np.testing.assert_array_equal(cmd[rows], c[rows]); np.testing.assert_array_equal(st[rows], s[rows])
            _same(sol, ref.mpc_get_solution(), TRAJ, rows, "tick chunks %d value %d" % (chunks, v))
    finally:
        told.set_pipeline(1)


def test_tick_sample_against_the_oracle_on_the_edited_files(handles, files):
    from _oracle import Oracle
    prob, wbc = _inputs()
    told, _ = handles[0]
    t_eval = prob["t0"] + 0.002
    _fresh(told)
    cmd, _ = told.tick(prob, t_eval, wbc["rbd"], wbc["period"]); sol = told.mpc_get_solution()
    for v in (1, 6):
        rows = _rows(v); task, gains = files[v]
        o = Oracle(task=task, gains=gains); o.mpc_set(dt=DT, horizon=1.0)
        sub = {k: np.asarray(a)[rows] for k, a in prob.items()}
        ref = o.tick_batch(sub, told.nmax, t_eval[rows], wbc["rbd"][rows], wbc["period"][rows], np.zeros((PER, 30)), nthreads=4)
        assert_cmd(cmd[rows], ref["cmd"], TICK_TOL, tag="tuning tick vs oracle value %d" % v)
        assert_traj({k: sol[k][rows] for k in ("n_nodes", "t", "event", "x", "u")}, ref, MPC_TOL, tag="tuning traj vs oracle value %d" % v)


def test_neutral_rows_are_bit_identical_to_no_rows_and_a_permuted_batch_follows_its_rows(values):
    prob, wbc = _inputs(); t_eval = prob["t0"] + 0.002
    a, b, c = _solver(), _solver(), _solver()
    perm = np.random.default_rng(3).permutation(B); rows = np.repeat(values, PER, axis=0)
    as_dict = lambda r: {k: r[:, off] if w == 1 else r[:, off:off + w] for k, (off, w) in L.items()}
    try:
        b.set_robot_tuning(as_dict(np.repeat(b.get_handle_tuning()[None], B, axis=0)))
        for chunks in (1, 2):
            for s in (a, b):
                s.set_pipeline(chunks); _fresh(s)
            ca, sa = a.tick(prob, t_eval, wbc["rbd"], wbc["period"]); cb, sb = b.tick(prob, t_eval, wbc["rbd"], wbc["period"])
            np.testing.assert_array_equal(ca, cb); np.testing.assert_array_equal(sa, sb)
            for k, val in a.mpc_get_solution().items():
                np.testing.assert_array_equal(val, b.mpc_get_solution()[k], err_msg=k)
        b.set_robot_tuning(as_dict(rows)); c.set_robot_tuning(as_dict(rows[perm])); _fresh(b)
        cb, sb = b.tick(prob, t_eval, wbc["rbd"], wbc["period"])
        cc, sc = c.tick({k: np.asarray(val)[perm] for k, val in prob.items()}, t_eval[perm], wbc["rbd"][perm], wbc["period"][perm])
        np.testing.assert_array_equal(cb[perm], cc); np.testing.assert_array_equal(sb[perm], sc)
    finally:
        a.close(); b.close(); c.close()


def test_told_friction_pyramid_is_enforced():
    """wbc_friction 0.15 / 0.3 / 0.6 on stance states whose desired forces push 30 % sideways: every robot comes out without a WBC status bit, every foot
    force lies in its own pyramid |Fx|, |Fy| <= mu_b Fz (to 1e-9 of the force scale), and at 0.15 the pyramid binds on some foot, so the check is not vacuous."""
    prob, wbc = _inputs(); mus = np.array([0.15, 0.3, 0.6])[np.arange(B) % 3]
    s = _solver()
    try:
        s.set_robot_tuning(dict(wbc_friction=mus))
        rng = np.random.default_rng(11)
        u_des = np.zeros((B, 30)); u_des[:, 2:12:3] = 80.0; u_des[:, 0:12:3] = rng.uniform(-24.0, 24.0, (B, 4)); u_des[:, 1:12:3] = rng.uniform(-24.0, 24.0, (B, 4))
        cmd, st = s.wbc_update(prob["x0"], u_des, wbc["rbd"], np.full(B, 15, dtype=np.int32), wbc["period"], wbc["time"] + 12.0)
        F = cmd[:, 24:36].reshape(B, 4, 3); scale = np.max(np.abs(F), axis=(1, 2))
        ok = (st & 0xFF) == 0; assert np.all(ok), np.unique(st)
        excess = np.maximum(np.abs(F[:, :, 0]), np.abs(F[:, :, 1])) - mus[:, None] * F[:, :, 2]
        assert np.all(excess[ok] <= 1e-9 * scale[ok, None]), np.max(excess[ok] / scale[ok, None])
        low = ok & (mus == 0.15); assert np.any(excess[low] >= -1e-9 * scale[low, None])   # a pyramid row is active
    finally:
        s.close()


def test_entry_points_validate_clear_and_follow_the_handle():
    from qm_control_b200 import QmbError
    s = _solver(batch=4)
    try:
        assert s.get_robot_tuning() is None
        h = s.get_handle_tuning(); assert field(h, "friction_mu") == 0.3 and field(h, "kd_arm_wbc") == 0.5
        rows = np.zeros((4, 40)); s.lib.qmb200_get_robot_tuning(s.h, rows.ctypes.data, None); np.testing.assert_array_equal(rows, np.repeat(h[None], 4, axis=0))
        s.set_robot_tuning(dict(friction_mu=[0.2, 0.3, 0.4, 0.5], kp_ee_linear=[1.0, 2.0, 3.0]))
        good = s.get_robot_tuning(); np.testing.assert_array_equal(good["friction_mu"], [0.2, 0.3, 0.4, 0.5]); np.testing.assert_array_equal(good["kp_ee_linear"][2], [1.0, 2.0, 3.0])
        for kw, msg in ((dict(wbc_friction=[0.3, 0.0, 0.3, 0.3]), "wbc_friction of robot 1 must be > 0"), (dict(mu_ee_ori=np.nan), "mu_ee_ori of robot 0 must be finite"),
                        (dict(kd_ee_angular=[[0, 0, 0]] * 3 + [[0, 0, -1.0]]), r"kd_ee_angular\[2\] of robot 3 must be >= 0"), (dict(kp_arm_wbc=-1.0), "kp_arm_wbc of robot 0 must be >= 0")):
            with pytest.raises(QmbError, match=msg):
                s.set_robot_tuning(kw)
            assert msg.split(" of ")[0].replace("\\", "") in s.lib.qmb200_last_error(s.h).decode()
            after = s.get_robot_tuning()
            for k in L:
                np.testing.assert_array_equal(after[k], good[k])   # unchanged on rejection
        s.set_robot_tuning(None); assert s.get_robot_tuning() is None
        s.wbc_set_gains(kp_swing=123.0); s.set_arm_gains(1.5, 0.25)
        h2 = s.get_handle_tuning(); assert field(h2, "kp_swing") == 123.0 and field(h2, "kp_arm_wbc") == 1.5 and field(h2, "kd_arm_wbc") == 0.25
        s.lib.qmb200_get_robot_tuning(s.h, rows.ctypes.data, None); np.testing.assert_array_equal(rows, np.repeat(h2[None], 4, axis=0))
    finally:
        s.close()


# ---------------- closed loop ----------------
NL = 64


def _run(**kw):
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    s = q.Solver(batch=NL, device=0)
    try:
        r = closed_loop.run(s, **kw)
        assert s.get_robot_tuning() is None   # restored
        return r
    finally:
        s.close()


def test_closed_loop_neutral_rows_are_bit_identical():
    import qm_control_b200 as q
    s = q.Solver(batch=1, device=0); h = s.get_handle_tuning(); s.close()
    neutral = {k: h[off] if w == 1 else h[off:off + w] for k, (off, w) in L.items()}
    plain = _run(duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0))
    told = _run(duration=0.3, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), tuning=neutral)
    for k in ("base", "ee", "status", "contact", "q", "v"):
        np.testing.assert_array_equal(plain[k], told[k], err_msg=k)


def test_closed_loop_told_the_plant_friction():
    """64 robots trotting at 0.3 m/s on floors of mu 0.15-0.3 with the MPC cone and the WBC pyramid told each robot's floor.  Asserted: the record is
    finite and the rows are restored; the fall counts against the untold run are reported in DESIGN.md §8."""
    mu = np.linspace(0.15, 0.3, NL)
    kw = dict(duration=1.0, gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), friction_mu=mu)
    told = _run(tuning=dict(friction_mu="plant", wbc_friction="plant"), **kw)
    untold = _run(**kw)
    for r in (told, untold):
        assert np.all(np.isfinite(r["base"])) and np.all(np.isfinite(r["q"]))
    fallen = lambda r: int(np.sum(np.min(r["base"][:, :, 2], axis=0) < 0.3))
    print("closed loop mu 0.15-0.3: fallen told %d untold %d of %d" % (fallen(told), fallen(untold), NL))
