"""Robot-state snapshots on the host, no GPU (DESIGN.md §4.17): the masked row gather of image_restore_kernel (compiled with g++ by
tests/restore_host.cpp, the very functions the kernel runs) against a numpy statement, and with an identity source against the start image's restore
rule; the bindings and the descriptor's layout; the gather kernel's resources; closed_loop.Session's snapshot refusals and calls on a fake Solver."""
import contextlib
import ctypes as C
import os
import re
import shutil
import subprocess
from unittest import mock

import numpy as np
import pytest

from test_gait_dev_cpu import B, _FakeStream, _fake_solver, _parent_calls
from qm_control_b200 import _lib, closed_loop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "qm_control_b200", "csrc")
ST_RESTORE = 0x40000
NAMES_ABI = ("qmb200_robot_state_bytes", "qmb200_robot_state_save_dev", "qmb200_robot_state_load_dev", "qmb200_robot_state_load")


@pytest.fixture(scope="module")
def rh(tmp_path_factory):
    lib_path = str(tmp_path_factory.mktemp("restore_host") / "librestorehost.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include",
                           "-I" + CSRC, "-o", lib_path, os.path.join(ROOT, "tests", "restore_host.cpp")])
    lib = C.CDLL(lib_path)
    lib.rh_gather.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _gather(rh, dst, src, mask, row, status=True):
    """rh_gather on copies of dst (list of uint32 [B, words]) → (the written tables, status [B] or None)"""
    out = [np.ascontiguousarray(d, dtype=np.uint32).copy() for d in dst]; srcs = [None if s is None else np.ascontiguousarray(s, dtype=np.uint32) for s in src]
    n = len(out); Bn = out[0].shape[0]
    dp = (C.c_void_p * n)(*[a.ctypes.data for a in out]); sp = (C.c_void_p * n)(*[None if a is None else a.ctypes.data for a in srcs])
    words = np.array([a.shape[1] for a in out], dtype=np.int32)
    m = None if mask is None else np.ascontiguousarray(mask, dtype=np.int32); r = None if row is None else np.ascontiguousarray(row, dtype=np.int32)
    st = np.full(Bn, -7, dtype=np.int32) if status else None
    assert rh.rh_gather(n, dp, sp, words.ctypes.data, Bn, None if m is None else m.ctypes.data, None if r is None else r.ctypes.data,
                        None if st is None else st.ctypes.data) == 0
    return out, st


def _statement(dst, src, mask, row):
    """the gather in numpy: robot b with mask[b] (None: every robot) and source r = row[b] (None: b) in [0, B) takes src[r] (zeros for a NULL src)"""
    Bn = dst[0].shape[0]; m = np.ones(Bn, bool) if mask is None else np.asarray(mask) != 0
    r = np.arange(Bn) if row is None else np.asarray(row, dtype=np.int64)
    ok = m & (r >= 0) & (r < Bn); rc = np.clip(r, 0, Bn - 1)
    out = []
    for d, s in zip(dst, src):
        take = np.zeros_like(d) if s is None else s[rc]
        out.append(np.where(ok[:, None], take, d).astype(np.uint32))
    return out, np.where(m & ~ok, ST_RESTORE, 0).astype(np.int32)


def _tables(rng, Bn, n):
    words = rng.integers(1, 40, n); words[0] = 1
    dst = [rng.integers(0, 1 << 32, (Bn, w), dtype=np.uint64).astype(np.uint32) for w in words]
    src = [None if rng.uniform() < 0.2 else rng.integers(0, 1 << 32, (Bn, w), dtype=np.uint64).astype(np.uint32) for w in words]
    return dst, src


@pytest.mark.parametrize("seed", range(6))
def test_the_gather_equals_its_numpy_statement(rh, seed):
    rng = np.random.default_rng(seed); Bn = int(rng.integers(1, 70)); n = int(rng.integers(1, 29))
    dst, src = _tables(rng, Bn, n)
    for mask in (None, (rng.uniform(size=Bn) < 0.6).astype(np.int32), rng.integers(-3, 3, Bn)):
        perm = rng.permutation(Bn); many = rng.integers(0, Bn, Bn)
        bad = many.copy(); sel = rng.uniform(size=Bn) < 0.3; bad[sel] = rng.choice([-1, Bn, Bn + 7, -(1 << 31), (1 << 31) - 1], sel.sum())
        for row in (None, perm, many, bad):
            got, st = _gather(rh, dst, src, mask, row)
            want, wst = _statement(dst, src, mask, row)
            assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want)), (mask, row)
            np.testing.assert_array_equal(st, wst)
    assert np.any(wst == ST_RESTORE) or Bn < 4


def test_an_identity_source_is_the_start_image_restore_byte_for_byte(rh):
    """NULL row and row = b write what the restore wrote before it had a source index: mask[b] ? (src ? src[b] : 0) : untouched"""
    rng = np.random.default_rng(11)
    for Bn, n in ((1, 1), (5, 13), (64, 28), (257, 7)):
        dst, src = _tables(rng, Bn, n); mask = (rng.uniform(size=Bn) < 0.5).astype(np.int32)
        before = [np.where(mask[:, None] != 0, np.zeros_like(d) if s is None else s, d) for d, s in zip(dst, src)]
        a, sa = _gather(rh, dst, src, mask, None); b, sb = _gather(rh, dst, src, mask, np.arange(Bn))
        assert [x.tobytes() for x in a] == [x.tobytes() for x in before] == [x.tobytes() for x in b]
        assert not sa.any() and not sb.any()
        c, _ = _gather(rh, dst, src, None, None)   # a save: every robot from its own row
        assert [x.tobytes() for x in c] == [(np.zeros_like(d) if s is None else s).tobytes() for d, s in zip(dst, src)]


def test_entry_points_are_bound_declared_and_the_status_bit_is_free():
    h = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    for name in NAMES_ABI:
        assert name in _lib.PROTOTYPES and re.search(r"\b%s\(" % name, h), name
    assert _lib.PROTOTYPES["qmb200_robot_state_bytes"][0] is C.c_int64
    assert "#define QMB200_ST_RESTORE (QMB200_ST_COMMAND << 1)" in h and _lib.ST_RESTORE == ST_RESTORE == _lib.ST_COMMAND << 1
    bits = [int(v, 0) for k, v in re.findall(r"#define (QMB200_ST_\w+) (0x[0-9a-fA-F]+|\d+)", h)]
    assert ST_RESTORE not in bits and ST_RESTORE > max(bits)
    n = int(re.search(r"#define QMB200_STATE_BLOCKS (\d+)", h).group(1))
    assert len(_lib.ROBOT_STATE_BLOCKS) == n == len(set(_lib.ROBOT_STATE_BLOCKS)) and n <= 64
    api = open(os.path.join(CSRC, "kernels", "respawn_api.cuh")).read()
    assert int(re.search(r"RESTORE_MAX_SEGS = (\d+)", api).group(1)) >= n
    names = re.search(r"kStateName\[QMB200_STATE_BLOCKS\] = \{(.*?)\};", open(os.path.join(CSRC, "capi_respawn.inc")).read(), re.S).group(1)
    assert len(re.findall(r'"[^"]+"', names)) == n


def test_descriptor_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in _lib.RobotStateDesc._fields_]
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "qmb200.h"', 'int main(void) {', '  printf("%zu\\n", sizeof(qmb200_robot_state_desc));']
    body += ['  printf("%%zu\\n", offsetof(qmb200_robot_state_desc, %s));' % f for f in fields] + ['  return 0; }']
    src = tmp_path / "desc.c"; src.write_text("\n".join(body) + "\n"); exe = tmp_path / "desc"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert out[0] == C.sizeof(_lib.RobotStateDesc) and out[1:] == [getattr(_lib.RobotStateDesc, f).offset for f in fields]


def test_the_gather_kernel_compiles_for_sm90a_without_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    obj = str(tmp_path / "respawn.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "kernels", "respawn_kernel.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    m = re.search(r"Function properties for (\w*image_restore_kernel\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert m and m.groups()[1:] == ("0", "0", "0"), r.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if os.path.exists(cuobjdump):
        sass = subprocess.run([cuobjdump, "-sass", "-fun", m.group(1), obj], capture_output=True, text=True, check=True).stdout
        assert "image_restore_kernel" in sass and not re.search(r"\b(LDL|STL)\b", sass)


# ---------------------------------------------------------------------------------------------------------------------- closed_loop.Session on a fake Solver
@contextlib.contextmanager
def _cpu_torch():
    import torch
    with mock.patch.object(torch.cuda, "Stream", _FakeStream), mock.patch.object(torch.cuda, "stream", lambda st: contextlib.nullcontext()):
        yield


def _solver():
    s = _fake_solver()
    s.robot_state_bytes = mock.Mock(return_value=24)
    s.robot_state_save_dev = mock.Mock(side_effect=lambda buf, stream: _lib.RobotStateDesc(batch=B, bytes=24))
    s.robot_state_load_dev = mock.Mock()
    return s


@pytest.mark.parametrize("kw", [dict(respawn=True), dict(randomize=dict(friction_mu=(0.5, 1.0))), dict(spawn=dict(yaw=(-0.5, 0.5))),
                                dict(timeline=dict(n=2, t_first=(0.1, 0.2), gap=(0.1, 0.2))),
                                dict(respawn=dict(every=0.01), curriculum=dict(levels=2, randomize=dict(friction_mu=(0.5, 1.0))), randomize=dict(friction_mu=(0.5, 0.5)))])
def test_snapshots_refuse_per_episode_sessions_before_any_solver_call(kw):
    s = _solver()
    ss = closed_loop.Session(s, 0.02, gait="trot", **kw)
    for call in (ss.snapshot, lambda: ss.restore(None)):
        with pytest.raises(ValueError, match="snapshots cannot go with"):
            call()
    assert s.mock_calls == []


def test_restore_refusals_raise_before_any_write():
    import torch
    s = _solver()
    with _cpu_torch():
        plain = closed_loop.Session(s, 0.05, torch_device="cpu", gait="trot")
        with pytest.raises(ValueError, match="not open"):
            plain.snapshot()
        with closed_loop.Session(s, 0.05, torch_device="cpu", gait="trot") as a, \
                closed_loop.Session(s, 0.05, torch_device="cpu", gait="trot") as b:
            a.step(1); b.step(1)
            snap_a = a.snapshot(); n = len(s.mock_calls)
            q = a.q.clone()
            with pytest.raises(ValueError, match="another session"):
                b.restore(snap_a)
            with pytest.raises(ValueError, match=r"source must have shape \(2,\)"):
                a.restore(snap_a, source=np.zeros(3))
            s.robot_state_load_dev.side_effect = _lib.QmbError("qmb200_robot_state_load_dev failed (-1): the state estimator was reset")
            with pytest.raises(ValueError, match="library refuses the snapshot.*state estimator"):
                a.restore(snap_a)
            assert [c[0] for c in s.mock_calls[n:]] == ["robot_state_load_dev"] and torch.equal(a.q, q) and a.k0 is None
            s.robot_state_load_dev.side_effect = None
            a.step(1)
            with pytest.raises(ValueError, match="window 0"):
                a.restore(closed_loop.Snapshot(a, snap_a.buf, snap_a.desc, snap_a.rows, snap_a.k0, 0))
            a.finish()
            with pytest.raises(ValueError, match="not open"):
                a.restore(snap_a)


def test_a_session_without_snapshots_makes_the_calls_of_before():
    s = _solver()
    with _cpu_torch():
        with closed_loop.Session(s, 0.02, torch_device="cpu", gait="trot") as ss:
            ss.step(1); ss.step(1); ss.finish()
    assert [c[0] for c in s.mock_calls] == _parent_calls()


def test_a_snapshot_and_a_restore_are_one_call_each_at_the_boundary():
    import torch
    s = _solver()
    with _cpu_torch():
        with closed_loop.Session(s, 0.02, torch_device="cpu", gait="trot", pushes=(np.zeros(B), np.full(B, 0.004), np.ones((B, 12)))) as ss:
            ss.step(1)
            snap = ss.snapshot()
            assert snap.window == 1 and len(snap.rows) == len(ss.rows) == len(ss.own) + 4 and snap.buf.numel() == 24 * B   # the push rows and acc_st
            ss.restore(snap, mask=np.array([1, 1]), source=np.array([1, 5]))
            assert ss.k0.tolist() == [0, 0]   # robot 1's source lies outside [0, B): its clock stays
            ss.step(1); ss.finish()
    calls = [c[0] for c in s.mock_calls]
    want = _parent_calls(); i = want.index("target_trajectories_dev", want.index("mpc_solve_dev") + 1)
    assert calls == want[:i] + ["robot_state_bytes", "robot_state_save_dev", "robot_state_load_dev"] + want[i:]
    args = s.robot_state_load_dev.call_args[0]
    assert args[0] is snap.buf and args[1] is snap.desc and args[2].tolist() == [1, 1] and args[3].tolist() == [1, 5]
    assert isinstance(args[4], torch.Tensor) and args[4].shape == (B,)
