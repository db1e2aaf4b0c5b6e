"""closed_loop.run's per-run overrides (terrain, model payload, payload estimator, plant robot params) on a fake Solver that keeps the handle's state in
a dict and logs every call: the overrides are set in that order and restored in reverse on every error path, and the handle ends as it started.
No GPU: closed_loop._run rejects a cmd_vel of the wrong shape before it touches the device."""
import types
from unittest import mock

import numpy as np
import pytest

from qm_control_b200 import closed_loop

B = 4
TERRAIN = dict(tiles=np.zeros((2, 3, 3)), cell=0.02, tile=np.array([1, 0, 1, 0]), origin=np.zeros((B, 2)))
TERRAIN_SET = ["sim_get_terrain", "sim_get_robot_terrain", "sim_set_robot_terrain", "sim_set_terrain", "sim_set_robot_terrain"]
TERRAIN_RESTORE = ["sim_set_robot_terrain", "sim_set_terrain", "sim_set_robot_terrain"]   # robot terrain cleared first, then the library, then the robots


def _fake():
    """→ (solver, state): the setters have the semantics of qm_control_b200.interface.Solver's; solver.mock_calls logs every call in order."""
    st = dict(terrain=dict(tiles=np.full((1, 3, 3), 0.1), cell=0.5), robot_terrain=dict(tile=np.array([0, -1, 0, -1]), origin=np.ones((B, 2))),
              robot_params=dict(friction_mu=np.full(B, 0.5), payload=None), model_payload=np.full((B, 8), 0.25), est_params=dict(forgetting=0.999), est_running=False)

    def set_terrain(tiles=None, cell=None):
        st["terrain"] = None if tiles is None else dict(tiles=tiles, cell=cell)
        if tiles is None:   # clearing the library clears the robots' terrain
            st["robot_terrain"] = None

    def set_est_params(**params):
        for k in params:
            if k not in st["est_params"]:
                raise ValueError("payload_est_set_params: unknown parameter %r" % (k,))
        st["est_params"] = dict(st["est_params"], **params)

    impl = dict(sim_get_terrain=lambda: st["terrain"], sim_set_terrain=set_terrain, sim_get_robot_terrain=lambda: st["robot_terrain"],
                sim_set_robot_terrain=lambda tile=None, origin=None: st.update(robot_terrain=None if tile is None else dict(tile=tile, origin=origin)),
                sim_get_robot_params=lambda: st["robot_params"], sim_set_robot_params=lambda friction_mu=None, payload=None: st.update(robot_params=dict(friction_mu=friction_mu, payload=payload)),
                get_model_payload=lambda: st["model_payload"], set_model_payload=lambda payload=None: st.update(model_payload=payload),
                payload_est_get_params=lambda: st["est_params"], payload_est_set_params=set_est_params, payload_est_stop=lambda: st.update(est_running=False),
                payload_est_reset=lambda: st.update(model_payload=np.zeros((B, 8)) if st["model_payload"] is None else st["model_payload"], est_running=True))
    solver = mock.Mock(spec=list(impl), batch=B, _cfg=types.SimpleNamespace(device=0))
    for name, f in impl.items():
        getattr(solver, name).side_effect = f
    return solver, st


def test_every_override_is_restored_in_reverse_when_the_run_fails():
    s, st = _fake(); before = dict(st)
    payload = np.zeros((B, 8)); payload[:, 0] = 1.5
    with pytest.raises(ValueError, match="cmd_vel must have shape"):
        closed_loop.run(s, duration=0.01, cmd_vel=np.zeros(3), terrain=TERRAIN, payload=payload, friction_mu=0.3, model_payload="plant", payload_estimator=dict(forgetting=0.99))
    np.testing.assert_equal(st, before)
    assert [c[0] for c in s.mock_calls] == TERRAIN_SET + [
        "get_model_payload", "set_model_payload",                                                  # "plant": this run's payload
        "get_model_payload", "payload_est_get_params", "payload_est_set_params", "payload_est_reset",
        "sim_get_robot_params", "sim_set_robot_params",
        "sim_set_robot_params",                                                                    # _run raised: the reverse order from here
        "payload_est_stop", "set_model_payload", "payload_est_set_params",
        "set_model_payload"] + TERRAIN_RESTORE
    assert s.mock_calls[6][1][0] is payload and s.mock_calls[9][2] == dict(forgetting=0.99)
    assert s.mock_calls[12][2]["friction_mu"] == 0.3 and s.mock_calls[12][2]["payload"] is payload


def test_a_failing_estimator_setup_restores_the_outer_overrides():
    s, st = _fake(); before = dict(st)
    with pytest.raises(ValueError, match="unknown parameter 'no_such_parameter'"):
        closed_loop.run(s, duration=0.01, terrain=TERRAIN, friction_mu=0.3, model_payload=np.ones((B, 8)), payload_estimator=dict(no_such_parameter=1.0))
    np.testing.assert_equal(st, before)
    assert [c[0] for c in s.mock_calls] == TERRAIN_SET + [
        "get_model_payload", "set_model_payload",
        "get_model_payload", "payload_est_get_params", "payload_est_set_params",                   # raises: the plant's robot params are never touched
        "payload_est_stop", "set_model_payload", "payload_est_set_params",
        "set_model_payload"] + TERRAIN_RESTORE
