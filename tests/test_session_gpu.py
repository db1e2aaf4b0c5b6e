"""The stepped closed loop on the GPU (closed_loop.Session, DESIGN.md §4.16): stepping in uneven chunks gives run's outputs and solver calls byte for
byte; commands from device tensors give what the same rows on a commands timeline give, and a respawn drops them; the command kernel equals the host
rule on a large batch and its refusals write nothing; a torch heading controller on the session's stream steers trotting robots to their goals."""
import numpy as np
import pytest

from qm_control_b200 import _lib
from qm_control_b200 import terrain as TR
from test_session_cpu import _statement

pytestmark = pytest.mark.gpu


def _solver(B, **kw):
    import qm_control_b200 as q
    return q.Solver(batch=B, device=0, **kw)


class _Recorder:
    """the solver with every public method call's name logged in order"""

    def __init__(self, s):
        self._s, self.calls = s, []

    def __getattr__(self, name):
        a = getattr(self._s, name)
        if name.startswith("_") or not callable(a):
            return a

        def call(*args, **kw):
            self.calls.append(name)
            return a(*args, **kw)
        return call


def _same(a, b):
    assert set(a) == set(b)
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k
        else:
            assert a[k] == b[k], k


def _stepped(s, duration, chunks, on_boundary=None, **kw):
    """a Session stepped in chunks (the last one takes the rest) → run's outputs; on_boundary(session, windows done) before each chunk"""
    from qm_control_b200 import closed_loop
    with closed_loop.Session(s, duration, **kw) as ss:
        recs, done = [], 0
        for n in list(chunks) + [ss.windows - sum(chunks)]:
            if on_boundary is not None:
                on_boundary(ss, done)
            recs.append(ss.step(n)); done += n
        end = ss.finish()
    out = {k: np.concatenate([r[k] if isinstance(r[k], np.ndarray) else r[k].cpu().numpy() for r in recs]) for k in recs[0]}
    out.update(end)
    return out


def _configs(B):
    xy = np.zeros((B, 3)); xy[:, 0] = np.arange(B) * 0.0
    mixed = dict(tiles=np.stack([TR.ramp(8.0), TR.stairs(0.05, 0.25), TR.rough(0.01, seed=7)]), cell=TR.CELL, tile=(np.arange(B) % 4 - 1).astype(np.int32),
                 origin=TR.centred_origin(xy[:, :2]))
    return dict(
        truth=dict(gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.1)),
        estimators=dict(gait="trot", cmd_vel=(0.3, 0.0, 0.0, 0.0), terrain=mixed, state_estimator=True, sensor_noise="reference", attitude_filter=True,
                        slip_detector=True, ground_map=True),
        episodes=dict(gait="trot", xy_yaw=xy, respawn=dict(every=0.1), metrics=True, terrain=mixed,
                      randomize=dict(seed=4, cmd_vel_x=(0.0, 0.3), friction_mu=(0.5, 0.9)), spawn=dict(seed=5, tile=(-1, 1), dx=(-0.1, 0.1), yaw=(0.2, 0.2)),
                      timeline=dict(seed=6, n=3, t_first=(0.0, 0.1), gap=(0.02, 0.06), p_gait=0.5, gaits=["trot", "pace"], weights=dict(none=1.0, cmd_vel=1.0)),
                      curriculum=dict(levels=3, randomize=dict(friction_mu=(0.3, 0.9)), timeline=dict(p_gait=1.0))))


@pytest.mark.parametrize("name", ["truth", "estimators", "episodes"])
def test_chunking_is_invisible(name):
    from qm_control_b200 import closed_loop
    B = 16; kw = _configs(B)[name]
    s, s2 = _solver(B), _solver(B)   # one handle each: without respawn a second loop would warm-start from the first one's MPC solution
    try:
        a = _Recorder(s); want = closed_loop.run(a, duration=0.4, **kw)
        b = _Recorder(s2); got = _stepped(b, 0.4, (1, 3, 7), **kw)
    finally:
        s.close(); s2.close()
    _same(want, got)
    assert a.calls == b.calls and len(a.calls) > 1000


def _inject(rng, B, names):
    """random command rows for a random mask: a gait switch, a cmd_vel step, an end-effector goal or an ee_cmd_vel, NaN rows for none.  The gaits are
    ones whose 3 s window stays within QMB200_EMAX events: a step that overflows keeps its slot, and a later command would replace the row a timeline
    still holds."""
    mask = (rng.uniform(size=B) < 0.4).astype(np.int32)
    gait = np.where(rng.uniform(size=B) < 0.3, rng.choice([names.index(n) for n in ("stance", "trot", "pace")], B), -1).astype(np.int32)
    vel = np.full((B, 4), np.nan); goal = np.full((B, 7), np.nan); eev = np.full((B, 3), np.nan)
    for b, u in enumerate(rng.uniform(size=B)):
        if u < 0.35:
            vel[b] = [rng.uniform(-0.2, 0.4), rng.uniform(-0.1, 0.1), 0.0, rng.uniform(-0.3, 0.3)]
        elif u < 0.6:
            q = rng.normal(size=4) * [0.1, 0.1, 0.1, 1.0]; goal[b, :3] = [0.52, 0.09, 0.44] + rng.uniform(-0.1, 0.1, 3); goal[b, 3:] = q / np.linalg.norm(q)
        elif u < 0.8:
            eev[b] = rng.uniform(-0.05, 0.05, 3)
    return mask, gait, vel, goal, eev


def _as_timeline(B, names, shots, base=None):
    """run's commands for the injected rows [(window, rows)], each at 7 ms before its tick's t_obs (strictly after the previous tick's), after base's;
    padded with empty rows due after the run's end"""
    per = [[] for _ in range(B)]
    if base is not None:
        for b in range(B):
            for c in range(base["t"].shape[1]):
                per[b].append((base["t"][b, c], base["gait"][b][c], base["cmd_vel"][b, c], np.full(7, np.nan), np.full(3, np.nan)))
    for w, (mask, gait, vel, goal, eev) in shots:
        for b in np.flatnonzero(mask):
            per[b].append((0.01 * w - 0.007, None if gait[b] < 0 else names[gait[b]], vel[b], goal[b], eev[b]))
    C = max(1, max(len(p) for p in per))
    t = np.full((B, C), 100.0); g = [[None] * C for _ in range(B)]; v = np.full((B, C, 4), np.nan); eg = np.full((B, C, 7), np.nan); ev = np.full((B, C, 3), np.nan)
    for b, rows in enumerate(per):
        rows.sort(key=lambda r: r[0])   # stable: a base row at the injected row's time stays before it
        for c, (tt, gg, vv, gl, ee) in enumerate(rows):
            t[b, c] = tt; g[b][c] = gg; v[b, c] = vv; eg[b, c] = gl; ev[b, c] = ee
    return dict(t=t, gait=g, cmd_vel=v, ee_goal=eg, ee_cmd_vel=ev)


@pytest.mark.parametrize("on_base", [False, True])
def test_commands_equal_the_same_rows_on_a_timeline(on_base):
    import torch
    from qm_control_b200 import closed_loop
    B = 64; s, s2 = _solver(B), _solver(B); rng = np.random.default_rng(11 + on_base); names = closed_loop.gait_template_names()
    windows = sorted(rng.choice(np.arange(1, 100), 9, replace=False)); shots = [(int(w), _inject(rng, B, names)) for w in windows]
    base = None
    if on_base:   # 1.5 ms after the previous tick: before an injected row of the same window
        tb = np.sort(rng.choice(np.arange(1, 100), (B, 3)), axis=1) * 0.01 - 0.0085
        base = dict(t=tb, gait=[[rng.choice(["trot", "pace", None]) for _ in range(3)] for _ in range(B)],
                    cmd_vel=np.where(rng.uniform(size=(B, 3, 1)) < 0.5, rng.uniform(-0.2, 0.3, (B, 3, 4)), np.nan))
    kw = dict(gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.0))

    def inject(ss, done):
        for w, rows in shots:
            if w == done:
                dev = [torch.as_tensor(a, device="cuda:0") for a in rows]
                ss.command(dev[0], gait=dev[1], cmd_vel=dev[2], ee_goal=dev[3], ee_cmd_vel=dev[4])
    try:
        want = closed_loop.run(s, duration=1.0, commands=_as_timeline(B, names, shots, base), **kw)
        chunks = [windows[0]] + list(np.diff(windows))
        got = _stepped(s2, 1.0, chunks, on_boundary=inject, **(dict(commands=base) if on_base else dict(steer=True)), **kw)
    finally:
        s.close(); s2.close()
    _same(want, got)
    print("injected rows: target kinds %s, gaits %s" % (np.unique(got["target_kind"]).tolist(), np.unique(got["gait"]).tolist()))
    assert np.all((got["status"] & _lib.ST_COMMAND) == 0)
    assert {1, 2} <= set(np.unique(got["target_kind"]).tolist()) and len(np.unique(got["gait"])) >= 2   # the rows did act


def test_a_command_for_a_robot_that_respawns_at_that_boundary_is_dropped():
    import torch
    B = 32; s = _solver(B); kw = dict(gait="trot", steer=True, respawn=dict(every=0.1), cmd_vel=(0.2, 0.0, 0.0, 0.0))
    mask = np.zeros(B, dtype=np.int32); mask[::3] = 1

    def inject(ss, done):
        if done == 10:   # every robot's first episode ends at this boundary
            ss.command(torch.as_tensor(mask, device="cuda:0"), gait=torch.full((B,), 1, dtype=torch.int32, device="cuda:0"),
                       cmd_vel=torch.full((B, 4), 0.5, dtype=torch.float64, device="cuda:0"))
    try:
        want = _stepped(s, 0.3, (10,), **kw)
        got = _stepped(s, 0.3, (10,), on_boundary=inject, **kw)
    finally:
        s.close()
    _same(want, got)


def test_command_kernel_is_the_host_rule_on_a_large_batch_and_refusals_write_nothing():
    import torch
    from test_session_cpu import _random_rows
    B = 4096; s = _solver(B); rng = np.random.default_rng(2)
    try:
        names = s.gait_dev_set_templates(); nt = len(names); s.gait_dev_reset(np.zeros(B, dtype=np.int32), np.full(B, 10.0))
        empty = s.gait_dev_get_pending(); assert not empty["set"].any()
        first = _random_rows(rng, B); ones = np.ones(B, dtype=np.int32)
        assert not s.gait_dev_command(ones, *first).any()
        before = s.gait_dev_get_pending()
        tmpl, vel, kind, ee = _random_rows(rng, B)
        bad = rng.integers(0, 6, B)
        tmpl[bad == 1] = nt; vel[bad == 2, 1] = np.nan; vel[bad == 2, 0] = 0.1; kind[bad == 3] = 5
        kind[bad == 4] = 2; vel[bad == 4] = np.nan; ee[bad == 4] = [0.5, 0, 0.4, 0, 0, 0.1, 1.0]
        kind[bad == 5] = 1; vel[bad == 5] = np.nan; ee[bad == 5, 1] = np.inf
        mask = (rng.uniform(size=B) < 0.7).astype(np.int32)
        d = lambda a: torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")
        status = torch.full((B,), -1, dtype=torch.int32, device="cuda:0")
        s.gait_dev_command_dev(d(mask), d(tmpl), d(vel), d(kind), d(ee), status)
        got = s.gait_dev_get_pending(); st = status.cpu().numpy()
        want_st = np.where(mask == 1, _statement(tmpl, vel, kind, ee, nt), 0)
        np.testing.assert_array_equal(st, want_st)
        acc = (mask == 1) & (want_st == 0)
        assert np.any(acc) and np.any(want_st != 0)
        for k, rows in (("tmpl", tmpl), ("cmd_vel", vel), ("ee_kind", kind), ("ee", ee)):
            assert got[k][acc].tobytes() == np.ascontiguousarray(rows, dtype=got[k].dtype)[acc].tobytes(), k
            assert got[k][~acc].tobytes() == before[k][~acc].tobytes(), k   # unmasked and rejected robots: byte-unchanged
        assert np.all(got["set"] == 1)
        # refusals: a NULL buffer, then a stopped schedule; nothing is written
        st0 = status.clone(); rc = s.lib.qmb200_gait_dev_command_dev(s.h, None, None, None, None, None, None, None)
        assert rc != 0 and "null buffer" in s.lib.qmb200_last_error(s.h).decode()
        assert all(s.gait_dev_get_pending()[k].tobytes() == got[k].tobytes() for k in got)
        s.gait_dev_stop()
        with pytest.raises(_lib.QmbError, match="not running"):
            s.gait_dev_command_dev(d(mask), d(tmpl), d(vel), d(kind), d(ee), status)
        torch.cuda.synchronize(); assert status.cpu().numpy().tobytes() == st0.cpu().numpy().tobytes()
        # a reset empties every slot
        s.gait_dev_reset(np.zeros(B, dtype=np.int32), np.full(B, 10.0)); assert not s.gait_dev_get_pending()["set"].any()
    finally:
        s.close()


HEADING_BOUND = 0.05   # rad; measured 0.0253 max, 0.0104 mean on one H100 80GB HBM3 at 700 W (DESIGN.md §4.16)


def heading_controller(state, goal, vx=0.25, gain=2.0, rate_max=0.6):
    """a torch heading controller on the session's tensors: cmd_vel = (vx, 0, 0, clamp(gain * wrap(goal - yaw))) from the plant's yaw q[:, 3]"""
    import torch
    err = torch.remainder(goal - state["q"][:, 3] + np.pi, 2.0 * np.pi) - np.pi
    vel = torch.zeros((len(goal), 4), dtype=torch.float64, device=goal.device)
    vel[:, 0] = vx; vel[:, 3] = torch.clamp(gain * err, -rate_max, rate_max)
    return vel


def test_a_torch_heading_controller_steers_trotting_robots_to_their_goals():
    import torch
    from qm_control_b200 import closed_loop
    B = 256; s = _solver(B); rng = np.random.default_rng(4)
    goal_h = rng.uniform(-1.2, 1.2, B)
    try:
        with closed_loop.Session(s, 4.0, steer=True, gait="trot") as ss:
            with torch.cuda.stream(ss.stream):
                goal = torch.as_tensor(goal_h, device=ss.device); ones = torch.ones(B, dtype=torch.int32, device=ss.device)
            for _ in range(ss.windows):
                with torch.cuda.stream(ss.stream):
                    ss.command(ones, cmd_vel=heading_controller(ss.state, goal))
                rec = ss.step(1)
            end = ss.finish()
    finally:
        s.close()
    err = np.abs(np.remainder(goal_h - end["q"][:, 3] + np.pi, 2 * np.pi) - np.pi)
    status = rec["status"].cpu().numpy()
    print("heading controller, %d trotting robots, 4 s: final heading error max %.4f rad, mean %.4f rad, start max %.3f rad"
          % (B, err.max(), err.mean(), np.abs(goal_h).max()))
    assert np.all((status & _lib.ST_COMMAND) == 0)
    assert err.max() < HEADING_BOUND
