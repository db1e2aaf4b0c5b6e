"""Per-episode plant draws on the host, no GPU (DESIGN.md §4.11): the draw core compiled with g++ (tests/episode_host.cpp) against its numpy statement,
its distribution and its keys, the range check, closed_loop.run(randomize=...) validation and its ranges on a fake Solver, the bindings and the kernel's
resources."""
import ctypes as C
import os
import re
import shutil
import subprocess
import types
from unittest import mock

import numpy as np
import pytest
from scipy import stats

import _episode_twin as tw
from qm_control_b200 import _lib, closed_loop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
EP = {n: i for i, n in enumerate(_lib.EPISODE_LAYOUT)}
NAMES = ("qmb200_episode_set_ranges", "qmb200_episode_get_ranges", "qmb200_episode_sample", "qmb200_episode_sample_dev", "qmb200_episode_draw")


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("episode") / "libepisodehost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-I" + CSRC,
                           "-o", lib_path, os.path.join(ROOT, "tests", "episode_host.cpp")])
    return C.CDLL(lib_path)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _u(core, seed, robot, episode, channel):
    seed, robot, episode = (np.ascontiguousarray(a, dtype=np.uint64) for a in (seed, robot, episode)); channel = np.ascontiguousarray(channel, dtype=np.int32)
    out = np.zeros(len(seed)); core.ep_uniform(C.c_int(len(seed)), _ptr(seed), _ptr(robot), _ptr(episode), _ptr(channel), _ptr(out))
    return out


def _rows(core, lo, hi, seed, robot, episode):
    n = len(seed); lo = np.ascontiguousarray(lo, dtype=np.float64); hi = np.ascontiguousarray(hi, dtype=np.float64)
    seed, robot, episode = (np.ascontiguousarray(a, dtype=np.uint64) for a in (seed, robot, episode))
    out = np.zeros((n, _lib.EPISODE)); core.ep_rows(C.c_int(n), _ptr(seed), _ptr(robot), _ptr(episode), _ptr(lo), _ptr(hi), _ptr(out))
    return out


def _keys(rng, n):
    seed = rng.integers(0, 2 ** 63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)   # every bit of a uint64
    robot = rng.integers(0, 1 << 20, n).astype(np.uint64); episode = (rng.integers(-2, 1 << 31, n).astype(np.int64)).astype(np.uint64)   # the kernel's int32 cast
    return seed, robot, episode


def _ranges(rng, n):
    scale = 10.0 ** rng.integers(-3, 4, (n, _lib.EPISODE))
    lo = rng.uniform(-1.0, 1.0, (n, _lib.EPISODE)) * scale; hi = lo + rng.uniform(0.0, 2.0, (n, _lib.EPISODE)) * scale
    return lo, hi


def test_core_equals_the_numpy_statement_bit_for_bit(core):
    rng = np.random.default_rng(11); n = 120_000
    seed, robot, episode = _keys(rng, n); channel = rng.integers(0, _lib.EPISODE, n)
    u = _u(core, seed, robot, episode, channel)
    np.testing.assert_array_equal(u, tw.uniform(seed, robot, episode, channel))
    assert np.all(u > 0.0) and np.all(u < 1.0)
    m = 4000; seed, robot, episode = _keys(rng, m); lo, hi = _ranges(rng, m)   # 108000 values
    got = _rows(core, lo, hi, seed, robot, episode)
    np.testing.assert_array_equal(got, tw.rows(lo, hi, seed, robot, episode))
    uu = tw.uniform(seed[:, None], robot[:, None], episode[:, None], np.arange(_lib.EPISODE)[None])
    assert np.sum(got != uu * (hi - lo) + lo) > 100, "the single rounding shows: the core computes the fma, not u * d + lo"
    assert np.all(got >= lo) and np.all(got <= hi)


def test_equal_bounds_draw_lo_exactly(core):
    rng = np.random.default_rng(5); m = 2000; seed, robot, episode = _keys(rng, m); lo, _ = _ranges(rng, m)
    lo[:6] = np.array([np.nextafter(0.0, 1.0), 1e300, -1e-300, 0.6, 0.0, -0.0])[:, None]
    assert _rows(core, lo, lo, seed, robot, episode).tobytes() == lo.tobytes()   # byte for byte: -0.0 stays -0.0
    got = _rows(core, lo, lo.copy(), seed, robot, episode); assert got.tobytes() == tw.rows(lo, lo.copy(), seed, robot, episode).tobytes()


def test_each_channel_is_uniform(core):
    """Kolmogorov-Smirnov per channel over 20000 episodes of one robot on [0, 1], and over 20000 robots of one episode"""
    n = 20000; lo, hi = np.zeros((n, _lib.EPISODE)), np.ones((n, _lib.EPISODE))
    for seed, robot, episode in ((np.full(n, 7), np.full(n, 3), np.arange(n)), (np.full(n, 2 ** 63 + 9), np.arange(n), np.zeros(n))):
        r = _rows(core, lo, hi, seed, robot, episode)
        p = [stats.kstest(r[:, c], "uniform").pvalue for c in range(_lib.EPISODE)]
        assert min(p) > 1e-4, p
    c = np.corrcoef(r.T); assert np.max(np.abs(c - np.eye(_lib.EPISODE))) < 0.05   # channels are not correlated


def test_seed_robot_and_episode_each_change_every_column(core):
    lo, hi = np.zeros((1, _lib.EPISODE)), np.ones((1, _lib.EPISODE))
    base = _rows(core, lo, hi, [7], [3], [2])
    for key in (([8], [3], [2]), ([7], [4], [2]), ([7], [3], [3])):
        assert np.all(_rows(core, lo, hi, *key) != base), key


def _check(core, lo, hi):
    msg = C.create_string_buffer(256); rc = core.ep_ranges_error(C.c_int(len(lo)), _ptr(np.ascontiguousarray(lo)), _ptr(np.ascontiguousarray(hi)), msg, 256)
    return rc, msg.value.decode()


@pytest.mark.parametrize("field,lo_v,hi_v,why", [
    ("cmd_vel_x", np.nan, 0.0, "bounds must be finite"), ("f_ee_z", 0.0, np.inf, "bounds must be finite"), ("o_ee_y", 0.2, 0.1, "lo must be <= hi"),
    ("f_base_x", -1.5e308, 1.5e308, "hi - lo must be finite"), ("friction_mu", 0.0, 1.0, "lo must be > 0"), ("friction_mu", -0.1, 1.0, "lo must be > 0"),
    ("m_ee", -1e-9, 1.0, "lo must be >= 0"), ("m_base", -1.0, 1.0, "lo must be >= 0"), ("push_t_on", -0.01, 0.3, "lo must be >= 0"),
    ("push_duration", -0.1, 0.1, "lo must be >= 0")])
def test_range_check_names_the_field_and_the_robot(core, field, lo_v, hi_v, why):
    B = 5; lo = np.zeros((B, _lib.EPISODE)); lo[:, EP["friction_mu"]] = 0.5; hi = lo + 1.0
    assert _check(core, lo, hi) == (0, "")
    lo[3, EP[field]] = lo_v; hi[3, EP[field]] = hi_v
    assert _check(core, lo, hi) == (1, "qmb200_episode_set_ranges: %s of robot 3: %s" % (field, why))


def test_negative_bounds_of_signed_fields_are_accepted(core):
    lo = np.full((2, _lib.EPISODE), -2.0); hi = np.full_like(lo, -1.0)
    for f in ("friction_mu", "m_ee", "m_base", "push_t_on", "push_duration"):
        lo[:, EP[f]] = 0.1; hi[:, EP[f]] = 0.2
    assert _check(core, lo, hi) == (0, "")


# ---------------------------------------------------------------------------------------------------------------------------- closed_loop.run(randomize=...)
@pytest.mark.parametrize("bad,match", [
    ([0.1, 0.2], "randomize must be None or dict"), (dict(seed=-1), "seed must be an integer"), (dict(seed=1.5), "seed must be an integer"),
    (dict(seed=True), "seed must be an integer"), (dict(seed=2 ** 64), "seed must be an integer"), (dict(mu=(0.1, 0.2)), "unknown randomize field 'mu'"),
    (dict(friction_mu=0.5), "must be a pair"), (dict(friction_mu=(0.1, 0.2, 0.3)), "must be a pair"), (dict(friction_mu="ab"), "must be a pair"),
    (dict(friction_mu=("0.1", 0.2)), "must be a pair"), (dict(f_base_x=(np.zeros((2, 2)), 1.0)), "scalars or"), (dict(f_base_x=(np.zeros(3), np.ones(4))), "scalars or"),
    (dict(f_base_x=(1.0, 0.0)), "finite with lo <= hi"), (dict(cmd_vel_x=(np.nan, 0.0)), "finite with lo <= hi"),
    (dict(cmd_vel_x=(-1e308, 1e308)), "finite with lo <= hi"), (dict(friction_mu=(0.0, 1.0)), "friction_mu lo must be > 0"),
    (dict(m_ee=(-0.5, 1.0)), "m_ee lo must be >= 0"), (dict(push_t_on=([0.1, -0.1], 0.5)), "push_t_on lo must be >= 0"), (dict(push_duration=(-0.1, 0.1)), "push_duration lo")])
def test_closed_loop_rejects_a_malformed_randomize_before_any_solver_call(bad, match):
    with pytest.raises(ValueError, match=match):
        closed_loop.run(None, duration=0.02, randomize=bad)   # no solver: the rejection comes first


def test_closed_loop_rejects_a_linked_payload_draw_beside_the_payload_estimator():
    with pytest.raises(ValueError, match="payload_estimator"):
        closed_loop.run(None, duration=0.02, model_payload="plant", payload_estimator=True, randomize=dict(m_ee=(0.0, 2.0)))
    closed_loop._randomize_spec(4, dict(m_ee=(0.0, 2.0)))   # alone, or with a fixed payload beside the estimator, the spec is fine


def test_bounds_of_another_batch_are_rejected():
    with pytest.raises(ValueError, match=r"scalars or \[4\]"):
        closed_loop._randomize_spec(4, dict(m_ee=(np.zeros(3), 1.0)))
    assert closed_loop._randomize_spec(4, dict(seed=np.uint64(2 ** 64 - 1), m_ee=(np.zeros(4), 1.0)))["seed"] == 2 ** 64 - 1


class _Stop(Exception):
    pass


B = 4


def _fake(robot_mu=None, robot_payload=None, prev_ranges=None, model=None, tuning=None):
    """→ (solver, state): get / set semantics of the calls a randomized run makes before its loop; episode_set_ranges with ranges stops the run there"""
    st = dict(robot_params=dict(friction_mu=robot_mu, payload=robot_payload), ranges=prev_ranges, model=model, tuning=tuning, told=None)

    def set_ranges(lo=None, hi=None, seed=0):
        if lo is not None and st["told"] is None:
            st["told"] = (lo.copy(), hi.copy(), seed); raise _Stop
        st["ranges"] = None if lo is None else dict(lo=lo, hi=hi, seed=seed)
    impl = dict(sim_get_robot_params=lambda: dict(st["robot_params"]), sim_get_params=lambda: dict(friction_mu=0.6),
                sim_set_robot_params=lambda friction_mu=None, payload=None: st.update(robot_params=dict(friction_mu=friction_mu, payload=payload)),
                episode_get_ranges=lambda: st["ranges"], episode_set_ranges=set_ranges, get_model_payload=lambda: st["model"],
                set_model_payload=lambda p=None: st.update(model=p), get_robot_tuning=lambda: st["tuning"], set_robot_tuning=lambda t=None: st.update(tuning=t))
    solver = mock.Mock(spec=list(impl), batch=B, _cfg=types.SimpleNamespace(device=0))
    for name, f in impl.items():
        getattr(solver, name).side_effect = f
    return solver, st


def test_fields_not_named_are_fixed_at_the_runs_values_and_everything_is_restored():
    prev = dict(lo=np.ones((B, 27)), hi=np.full((B, 27), 2.0), seed=5)
    s, st = _fake(robot_mu=np.array([0.5, 0.6, 0.7, 0.8]), prev_ranges=prev)
    w = np.arange(B * 12, dtype=np.float64).reshape(B, 12); cmd = np.array([[0.1, 0.2, 0.0, 0.3]] * B)
    with pytest.raises(_Stop):
        closed_loop.run(s, duration=0.02, cmd_vel=cmd, pushes=(np.full(B, 0.2), np.full(B, 0.1), w), payload=np.full((B, 8), 0.25),
                        randomize=dict(seed=9, friction_mu=(0.15, [1.0, 0.9, 0.8, 0.7]), f_base_y=(-180.0, 180.0)))
    lo, hi, seed = st["told"]
    assert seed == 9
    np.testing.assert_array_equal(lo[:, EP["friction_mu"]], 0.15); np.testing.assert_array_equal(hi[:, EP["friction_mu"]], [1.0, 0.9, 0.8, 0.7])
    np.testing.assert_array_equal(lo[:, EP["f_base_y"]], -180.0); np.testing.assert_array_equal(hi[:, EP["f_base_y"]], 180.0)
    fixed = [c for c in range(27) if c not in (EP["friction_mu"], EP["f_base_y"])]
    np.testing.assert_array_equal(lo[:, fixed], hi[:, fixed])
    np.testing.assert_array_equal(lo[:, 1:9], 0.25); np.testing.assert_array_equal(lo[:, EP["push_t_on"]], 0.2); np.testing.assert_array_equal(lo[:, EP["push_duration"]], 0.1)
    np.testing.assert_array_equal(np.delete(lo[:, 11:23], 1, axis=1), np.delete(w, 1, axis=1)); np.testing.assert_array_equal(lo[:, 23:27], cmd)
    assert st["ranges"] is prev or (st["ranges"]["seed"] == 5 and np.all(st["ranges"]["lo"] == 1.0))   # the previous ranges are back
    np.testing.assert_array_equal(st["robot_params"]["friction_mu"], [0.5, 0.6, 0.7, 0.8]); assert st["robot_params"]["payload"] is None


@pytest.mark.parametrize("robot_mu,want", [(None, 0.6), (np.array([0.3, 0.4, 0.5, 0.6]), [0.3, 0.4, 0.5, 0.6])])
def test_fixed_friction_and_payload_fall_back_to_the_handle(robot_mu, want):
    s, st = _fake(robot_mu=robot_mu)
    with pytest.raises(_Stop):
        closed_loop.run(s, duration=0.02, randomize=dict(cmd_vel_x=(0.0, 0.5)))
    lo, hi, seed = st["told"]
    assert seed == 0
    np.testing.assert_array_equal(lo[:, 0], want); np.testing.assert_array_equal(lo[:, 1:23], 0.0); np.testing.assert_array_equal(hi[:, EP["cmd_vel_x"]], 0.5)
    assert st["ranges"] is None and st["robot_params"]["friction_mu"] is robot_mu


def test_without_randomize_the_loop_makes_no_episode_call():
    s, _ = _fake()
    with pytest.raises(ValueError, match="cmd_vel must have shape"):
        closed_loop.run(s, duration=0.01, cmd_vel=np.zeros(3))
    assert s.mock_calls == []


def test_entry_points_are_bound_and_declared():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name
    assert "#define QMB200_EPISODE 27" in h and len(_lib.EPISODE_LAYOUT) == _lib.EPISODE == 27
    assert _lib.EPISODE_LAYOUT[EP["push_t_on"]:EP["push_t_on"] + 2] == ("push_t_on", "push_duration") and _lib.EPISODE_LAYOUT[EP["f_base_x"]:EP["f_base_x"] + 12] == _lib.WRENCH_LAYOUT
    for name, v in (("MODEL_PAYLOAD", _lib.EPISODE_MODEL_PAYLOAD), ("MPC_FRICTION", _lib.EPISODE_MPC_FRICTION), ("WBC_FRICTION", _lib.EPISODE_WBC_FRICTION)):
        assert re.search(r"#define QMB200_EPISODE_%s %d\b" % (name, v), h), name


def test_episode_kernel_compiles_for_sm90a_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(CSRC, "kernels", "episode_kernel.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "episode.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    assert any("episode_sample_kernel" in k for k in kernels), r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == len(kernels) and all(sp == ("0", "0") for sp in spills), r.stderr
