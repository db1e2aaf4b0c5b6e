"""CPU checks of the per-robot restart (DESIGN.md §4.10): the fall rule's numpy statement against the sweeps' expression, the closed loop's respawn
option validation, the bound entry points and the new kernels' resources."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from _respawn_twin import fall_counts, fall_flags
from qm_control_b200 import _lib, closed_loop
from qm_control_b200 import terrain as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("qmb200_robot_image_save", "qmb200_robot_image_clear", "qmb200_robot_image_restore", "qmb200_robot_image_restore_dev", "qmb200_fall_detect",
         "qmb200_fall_detect_dev")


def _sweep_fallen(base, ground=0.0):
    """tools/bench_closedloop.py's rule over a run's record base [ticks, B, 6] = (x, y, z, yaw, pitch, roll)"""
    return ~(np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2] - ground, axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3))


def _rbd(base):
    """record rows (x, y, z, yaw, pitch, roll) → rbd rows [.., 55] with zyx and p where the plant writes them"""
    r = np.zeros(base.shape[:-1] + (55,)); r[..., 0:3] = base[..., 3:6]; r[..., 3:6] = base[..., 0:3]; r[..., 6:] = 0.25
    return r


def _crafted(B=64, ticks=5, seed=3):
    rng = np.random.default_rng(seed)
    base = np.zeros((ticks, B, 6)); base[..., 0:2] = rng.uniform(-0.5, 1.5, (ticks, B, 2)); base[..., 2] = rng.uniform(0.2, 0.6, (ticks, B))
    base[..., 3] = rng.uniform(-3, 3, (ticks, B)); base[..., 4:6] = rng.uniform(-0.4, 0.4, (ticks, B, 2))
    base[:, 0:8] = [0.0, 0.0, 0.5, 0.0, 0.0, 0.0]             # upright on every tick
    base[2, 1, 2] = 0.3; base[2, 2, 4] = 0.3; base[2, 3, 5] = -0.3  # on each threshold: fallen
    base[3, 4, 2] = np.nextafter(0.3, 1.0); base[3, 5, 4] = np.nextafter(0.3, 0.0); base[3, 6, 5] = -np.nextafter(0.3, 0.0)   # just inside: upright
    base[1, 7, 0] = np.nan; base[4, 7, 4] = np.inf             # non-finite rows
    return base


def test_fall_rule_matches_the_sweeps_expression_on_the_plane():
    base = _crafted()
    flags = fall_flags(_rbd(base))
    np.testing.assert_array_equal(flags.any(axis=0), _sweep_fallen(base))
    assert not flags[:, 0].any() and flags[2, 1] and flags[2, 2] and flags[2, 3] and not flags[3, 4:7].any() and flags[1, 7] and flags[4, 7]


def test_fall_rule_matches_the_sweeps_expression_on_a_terrain_tile():
    base = _crafted(seed=5); B = base.shape[1]
    tiles = np.stack([T.flat(), T.ramp(10.0, start=0.35) + T.stairs(0.09, 0.3, start=0.35), T.stairs(0.06, 0.3, start=0.35)])
    ter = dict(tiles=tiles, cell=T.CELL, tile=np.arange(B) % 4 - 1, origin=T.centred_origin(np.zeros((B, 2))))
    ground = T.height(ter["tiles"], ter["cell"], ter["tile"][None], ter["origin"][None], np.nan_to_num(base[:, :, :2]))
    base[2, 9, 2] = ground[2, 9] + 0.3   # on the threshold above the tile
    flags = fall_flags(_rbd(base), ter)
    np.testing.assert_array_equal(flags.any(axis=0), _sweep_fallen(base, ground))
    assert flags[2, 9] and np.any(flags != fall_flags(_rbd(base))), "the terrain changes some verdict"


def test_fall_counts_grow_per_fallen_call_and_drop_to_zero():
    f = np.array([[0, 1], [1, 1], [1, 0], [0, 1]], dtype=bool)
    np.testing.assert_array_equal(fall_counts(f), [[0, 1], [1, 2], [2, 0], [0, 1]])


@pytest.mark.parametrize("bad", [{"bogus": 1}, "yes", 1, {"hold": 0.015}, {"hold": 0.0}, {"hold": -0.01}, {"every": 0.205}, {"every": 0.0},
                                 {"hold": "0.1"}, {"z_min": np.nan}, {"tilt_max": 0.0}, {"tilt_max": np.inf}, {"on_fall": 1}, {"on_fall": False}])
def test_closed_loop_rejects_a_malformed_respawn_before_any_solver_call(bad):
    with pytest.raises(ValueError, match="respawn"):
        closed_loop.run(None, duration=0.02, respawn=bad)   # no solver: the rejection comes first


def test_respawn_spec_in_windows():
    assert closed_loop._respawn_spec(True) == dict(on_fall=True, hold_windows=10, z_min=0.3, tilt_max=0.3, every_ms=None)
    assert closed_loop._respawn_spec(dict(on_fall=False, every=0.2, hold=0.05)) == dict(on_fall=False, hold_windows=5, z_min=0.3, tilt_max=0.3, every_ms=200)


def test_entry_points_are_bound_and_declared():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES:
        assert name in _lib.PROTOTYPES and re.search(r"int %s\(" % name, h), name


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "qm_control_b200", "csrc", "kernels", "respawn_kernel.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "respawn.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    assert any("image_restore_kernel" in k for k in kernels) and any("fall_detect_kernel" in k for k in kernels), r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == len(kernels) and all(s == ("0", "0") for s in spills), r.stderr
