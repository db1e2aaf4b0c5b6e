"""A host-pointer entry point is its `_dev` twin with the caller's arrays staged on the handle's stream.

For each of the ten host-pointer entry points, the host call on one handle and the `_dev` call on an identically created and prepared twin
(warm start, WBC input_last, hw-write delay ring, robot params and model payload) give bit-identical outputs, in-out arrays included.  Every
`_dev` output starts as NaN (int32: -1), so an element the kernels leave unwritten shows up.  The stateless entry points leave no trace in the
tick chain, and the argument errors keep their return codes and texts."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

B = 37
IN, INOUT, OUT = "in", "inout", "out"


def _solver(variant=0):
    import qm_control_b200 as q
    return q.Solver(batch=B, dt=0.015, wbc_variant=variant)


def _inputs(seed=0):
    from qm_control_b200 import synthetic
    prob, wbc = synthetic.make_batch(np.arange(B), config=4)
    return prob, wbc, np.random.default_rng(seed)


def _robot_params(rng):
    mu = rng.uniform(0.4, 0.9, B)
    payload = np.c_[rng.uniform(0, 1.5, B), rng.uniform(-0.05, 0.05, (B, 3)), rng.uniform(0, 2.0, B), rng.uniform(-0.1, 0.1, (B, 3))]
    return mu, payload


def _prepare(s, prob, wbc, variation=True):
    """The handle state the entry points read: a warm start, input_last, a filled hw-write ring and (optionally) robot params and a model payload."""
    from qm_control_b200 import synthetic
    rng = np.random.default_rng(100)
    s.mpc_solve(prob)
    _, u, _ = synthetic.nominal_wbc_inputs(prob, s.robot_mass)
    s.wbc_set_input_last(u + rng.normal(size=u.shape) * 1e-2)
    s.hw_set_delay(0.004)
    for k in range(3):
        s.hw_write(np.full(B, 0.001 * (k + 2)), np.full(B, 0.001), rng.normal(size=(B, 18, 5)), rng.normal(size=(B, 18)), rng.normal(size=(B, 18)))
    if variation:
        mu, payload = _robot_params(rng)
        s.sim_set_robot_params(friction_mu=mu, payload=payload)
        s.set_model_payload(payload)


def _cases():
    """name → (wbc variant, f(prob, wbc, rng, solver) → (scalar arguments, [(role, array)]))."""
    from qm_control_b200 import synthetic

    def wbc_update(prob, wbc, rng, s):
        x, u, mode = synthetic.nominal_wbc_inputs(prob, s.robot_mass)
        return [], [(IN, x), (IN, u), (IN, wbc["rbd"]), (IN, mode.astype(np.int32)), (IN, wbc["period"]), (IN, wbc["time"] + 0.002),
                    (OUT, np.zeros((B, 54))), (OUT, np.zeros(B, np.int32))]

    def policy_eval(prob, wbc, rng, s):
        return [], [(IN, prob["t0"] + rng.uniform(0, 0.6, B)), (OUT, np.zeros((B, 30))), (OUT, np.zeros((B, 30))), (OUT, np.zeros(B, np.int32))]

    def tick(prob, wbc, rng, s):
        return [], [(IN, prob[k]) for k in ("t0", "x0", "n_events", "event_times", "modes", "n_target", "target_times", "target_states")] + \
               [(IN, prob["t0"] + 0.002), (IN, wbc["rbd"]), (IN, wbc["period"]), (OUT, np.zeros((B, 54))), (OUT, np.zeros(B, np.int32))]

    def observation_update(prob, wbc, rng, s):
        return [], [(IN, wbc["rbd"]), (IN, wbc["period"]), (INOUT, prob["t0"]), (INOUT, prob["x0"] + rng.normal(size=(B, 30)) * 1e-3)]

    def target_trajectories(prob, wbc, rng, s):
        ee = np.c_[rng.uniform(-1, 1, (B, 3)), rng.normal(size=(B, 4))]; ee[:, 3:] /= np.linalg.norm(ee[:, 3:], axis=1, keepdims=True)
        last = ee + rng.uniform(-0.12, 0.12, (B, 7))
        return [C.c_int32(0)], [(IN, rng.uniform(-0.5, 0.5, (B, 7))), (IN, prob["t0"]), (IN, prob["x0"]), (IN, ee), (INOUT, last),
                                (OUT, np.zeros(B, np.int32)), (OUT, np.zeros((B, 4))), (OUT, np.zeros((B, 4, 37)))]

    def control_law(prob, wbc, rng, s):
        t = rng.uniform(9.0, 11.0, B)
        return [], [(IN, rng.normal(size=(B, 30))), (IN, rng.normal(size=(B, 30))), (IN, rng.normal(size=(B, 54))), (IN, t), (IN, rng.normal(size=(B, 30))),
                    (INOUT, rng.normal(size=(B, 18, 5))), (INOUT, rng.normal(size=(B, 6))), (INOUT, t - rng.uniform(0.0, 0.02, B)), (OUT, np.zeros(B, np.int32))]

    def hw_write(prob, wbc, rng, s):
        return [], [(IN, np.full(B, 0.005)), (IN, np.full(B, 0.001)), (IN, rng.normal(size=(B, 18, 5))), (IN, rng.normal(size=(B, 18))), (IN, rng.normal(size=(B, 18))),
                    (OUT, np.zeros((B, 18))), (OUT, np.zeros(B, np.int32))]

    def update(prob, wbc, rng, s):
        return [], [(IN, wbc["rbd"]), (IN, wbc["period"]), (INOUT, prob["t0"]), (INOUT, prob["x0"]), (INOUT, rng.normal(size=(B, 18, 5))), (INOUT, rng.normal(size=(B, 6))),
                    (INOUT, prob["t0"] - 0.02), (OUT, np.zeros((B, 54))), (OUT, np.zeros(B, np.int32))]

    def _plant(rng, s, wrench):
        q, v = s.sim_standing_state(np.c_[rng.uniform(-1, 1, (B, 2)), rng.uniform(-np.pi, np.pi, B)])
        v = v + rng.normal(size=v.shape) * 1e-2
        arrays = [(IN, rng.normal(size=(B, 18)))] + ([(IN, rng.normal(size=(B, 12)) * 5.0)] if wrench else []) + \
                 [(INOUT, q), (INOUT, v), (OUT, np.zeros((B, 55))), (OUT, np.zeros(B, np.int32)), (OUT, np.zeros(B, np.int32))]
        return [0.002], arrays

    return {"wbc_update": (0, wbc_update), "policy_eval": (0, policy_eval), "tick": (0, tick), "observation_update": (0, observation_update),
            "target_trajectories": (0, target_trajectories), "control_law": (1, control_law), "hw_write": (0, hw_write), "update": (1, update),
            "sim_step_ext": (0, lambda p, w, r, s: _plant(r, s, True)), "sim_step": (0, lambda p, w, r, s: _plant(r, s, False))}


def _ptr(a):
    return C.c_void_p(a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr())


def _call_host(s, name, scalars, arrays):
    """→ the in-out and out arrays after qmb200_<name> with host arrays."""
    host = [np.ascontiguousarray(a, dtype=a.dtype).copy() for _, a in arrays]
    rc = getattr(s.lib, "qmb200_" + name)(s.h, *scalars, *[_ptr(a) for a in host])
    assert rc == 0, s.lib.qmb200_last_error(s.h).decode()
    return [a for (role, _), a in zip(arrays, host) if role != IN]


def _nan_like(a):
    import torch
    return torch.full((a.nbytes,), 0xFF, dtype=torch.uint8, device="cuda").view(torch.float64 if a.dtype == np.float64 else torch.int32).reshape(a.shape)


def _call_dev(s, name, scalars, arrays):
    """→ the in-out and out arrays after qmb200_<name>_dev with device arrays; every out array starts as all-ones bytes (NaN, int32 -1)."""
    import torch
    dev = [_nan_like(a) if role == OUT else torch.from_numpy(np.ascontiguousarray(a).copy()).cuda() for role, a in arrays]
    torch.cuda.synchronize()
    rc = getattr(s.lib, "qmb200_" + name + "_dev")(s.h, *scalars, *[_ptr(a) for a in dev], None)
    assert rc == 0, s.lib.qmb200_last_error(s.h).decode()
    torch.cuda.synchronize()
    return [a.cpu().numpy() for (role, _), a in zip(arrays, dev) if role != IN]


def _assert_bits(a, b, tag):
    assert a.shape == b.shape and a.dtype == b.dtype, tag
    diff = a.view(np.uint8).reshape(a.shape[0], -1) != b.view(np.uint8).reshape(b.shape[0], -1)
    assert not diff.any(), "%s: %d robots differ" % (tag, int(diff.any(axis=1).sum()))


@pytest.mark.parametrize("name", list(_cases()))
def test_host_call_is_its_dev_twin(name):
    variant, make = _cases()[name]
    prob, wbc, _ = _inputs()
    host, dev = _solver(variant), _solver(variant)
    for s in (host, dev):
        _prepare(s, prob, wbc)
    scalars, arrays = make(prob, wbc, np.random.default_rng(7), host)
    got_h = _call_host(host, name, scalars, arrays)
    got_d = _call_dev(dev, name, scalars, arrays)
    written = [role for role, _ in arrays if role != IN]
    for i, (a, b) in enumerate(zip(got_h, got_d)):
        if written[i] == OUT and b.dtype == np.float64:
            assert np.isfinite(b).all(), "%s: output %d not written in full by the kernels" % (name, i)
        elif written[i] == OUT:
            assert (b != -1).all(), "%s: output %d not written in full by the kernels" % (name, i)
        _assert_bits(a, b, "%s output %d" % (name, i))
    # the handle state both calls leave behind is the same too
    _assert_bits(host.wbc_get_input_last(), dev.wbc_get_input_last(), name + " input_last")
    sh, sd = host.mpc_get_solution(), dev.mpc_get_solution()
    for k in sh:
        _assert_bits(sh[k], sd[k], name + " solution " + k)


def _device_problem(prob):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in prob.items()}


def _tick_dev(s, pd, t_eval, rbd, period):
    import torch
    cmd = torch.zeros((B, 54), dtype=torch.float64, device="cuda"); st = torch.zeros(B, dtype=torch.int32, device="cuda")
    s.tick_dev(pd, t_eval, rbd, period, cmd, st); torch.cuda.synchronize()
    return cmd.cpu().numpy(), st.cpu().numpy()


@pytest.mark.parametrize("name", ["policy_eval", "observation_update", "target_trajectories", "control_law", "sim_step_ext"])
def test_stateless_host_call_leaves_the_tick_alone(name):
    """A host call between two ticks changes nothing the second tick computes."""
    import torch
    variant, make = _cases()[name]
    prob, wbc, _ = _inputs()
    plain, probed = _solver(variant), _solver(variant)
    for s in (plain, probed):
        _prepare(s, prob, wbc, variation=False)
    pd = _device_problem(prob); te = torch.from_numpy(prob["t0"] + 0.002).cuda()
    rbd = torch.from_numpy(wbc["rbd"]).cuda(); period = torch.from_numpy(wbc["period"]).cuda()
    first = [_tick_dev(s, pd, te, rbd, period) for s in (plain, probed)]
    scalars, arrays = make(prob, wbc, np.random.default_rng(7), probed)
    _call_host(probed, name, scalars, arrays)
    second = [_tick_dev(s, pd, te, rbd, period) for s in (plain, probed)]
    for (a, b), tag in ((first, "first"), (second, "second")):
        _assert_bits(a[0], b[0], name + " " + tag + " tick cmd"); _assert_bits(a[1], b[1], name + " " + tag + " tick status")


# the texts the host entry points give for a NULL output
NULL_OUTPUT_ERRORS = {"wbc_update": "qmb200_wbc_update: null buffer", "policy_eval": "qmb200_policy_eval: null buffer", "tick": "qmb200_tick: null buffer",
                      "observation_update": "qmb200_observation_update: null buffer", "target_trajectories": "qmb200_target_trajectories: null buffer",
                      "control_law": "qmb200_control_law: null buffer", "hw_write": "qmb200_hw_write: null buffer", "update": "qmb200_update: null buffer",
                      "sim_step_ext": "qmb200_sim_step_ext: null buffer", "sim_step": "qmb200_sim_step: null buffer"}


def test_argument_errors():
    prob, wbc, rng = _inputs()
    s = _solver()
    for name, (_, make) in _cases().items():
        scalars, arrays = make(prob, wbc, np.random.default_rng(7), s)
        ptrs = [_ptr(np.ascontiguousarray(a)) for _, a in arrays]; ptrs[-1] = None
        assert getattr(s.lib, "qmb200_" + name)(s.h, *scalars, *ptrs) == -1, name
        assert s.lib.qmb200_last_error(s.h).decode() == NULL_OUTPUT_ERRORS[name]
    _, arrays = _cases()["tick"][1](prob, wbc, rng, s)
    for key, idx, bad, text in (("n_events", 2, 40, "qmb200_tick: n_events[5] = 40 outside [0, QMB200_EMAX]"), ("n_target", 5, 0, "qmb200_tick: n_target[5] = 0 outside [1, QMB200_KMAX]")):
        host = [np.ascontiguousarray(a).copy() for _, a in arrays]; host[idx][5] = bad
        assert s.lib.qmb200_tick(s.h, *[_ptr(a) for a in host]) == -1, key
        assert s.lib.qmb200_last_error(s.h).decode() == text
    # a rejected payload leaves the stored robot params and model payload as they were
    mu, payload = _robot_params(rng)
    s.sim_set_robot_params(friction_mu=mu, payload=payload); s.set_model_payload(payload)
    bad = payload.copy(); bad[3, 4] = -1.0
    assert s.lib.qmb200_sim_set_robot_params(s.h, None, _ptr(bad)) == -1
    assert s.lib.qmb200_last_error(s.h).decode() == "qmb200_sim_set_robot_params: payload masses must be >= 0"
    bad[3, 4] = np.nan
    assert s.lib.qmb200_set_model_payload(s.h, _ptr(bad)) == -1
    assert s.lib.qmb200_last_error(s.h).decode() == "qmb200_set_model_payload: payload must be finite"
    bad_mu = mu.copy(); bad_mu[0] = 0.0
    assert s.lib.qmb200_sim_set_robot_params(s.h, _ptr(bad_mu), None) == -1
    assert s.lib.qmb200_last_error(s.h).decode() == "qmb200_sim_set_robot_params: friction_mu must be finite and > 0"
    got = s.sim_get_robot_params()
    np.testing.assert_array_equal(got["friction_mu"], mu); np.testing.assert_array_equal(got["payload"], payload)
    np.testing.assert_array_equal(s.get_model_payload(), payload)
