"""CPU checks of the product's host side: the C-ABI library loads and exports every symbol include/qmb200.h declares,
fails loudly without a GPU (no CPU fallback), host utilities (gait tiling, observation conversion inputs) and the
synthetic-batch generator."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import qm_control_b200 as q
from qm_control_b200 import _lib, synthetic
from qm_control_b200.interface import gait_schedule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _c_kind(decl):
    """Kind of a C type, with or without a parameter name: ptr / str (const char*) / int32 / int64 / double / void."""
    if "*" in decl:
        return "str" if re.fullmatch(r"const\s+char\s*\*\s*\w*", decl) else "ptr"
    return {"int": "int32", "int32_t": "int32", "int64_t": "int64", "double": "double", "void": "void"}[decl.replace("const ", "").split()[0]]


def _ctypes_kind(t):
    if t is None:
        return "void"
    if t is C.c_char_p:
        return "str"
    if t is C.c_void_p or issubclass(t, C._Pointer):
        return "ptr"
    return {C.c_int32: "int32", C.c_int64: "int64", C.c_double: "double"}[t]


def _header_prototypes():
    """name → (return kind, [argument kinds]) of every function include/qmb200.h declares, in header order."""
    hdr = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    code = re.sub(r"^\s*#.*$", "", re.sub(r"/\*.*?\*/|//[^\n]*", "", hdr, flags=re.S), flags=re.M)
    protos = {}
    for ret, name, params in re.findall(r"([\w\s*]+?)\b(qmb200_\w+)\s*\(([^()]*)\)\s*;", code):
        params = [p.strip() for p in params.split(",")] if params.strip() not in ("", "void") else []
        assert name not in protos, name
        protos[name] = (_c_kind(ret.strip()), [_c_kind(p) for p in params])
    assert set(protos) == set(re.findall(r"\b(qmb200_[a-z_0-9]+)\s*\(", hdr)), "a declaration the prototype parser missed"
    return protos


def test_library_exports_every_declared_symbol():
    """The binding's prototype table has every function of include/qmb200.h, in header order, with the same return and argument kinds."""
    declared = _header_prototypes()
    assert len(declared) >= 24
    assert list(_lib.PROTOTYPES) == list(declared) and _lib.SYMBOLS == list(declared)
    for name, (ret, args) in declared.items():
        restype, argtypes = _lib.PROTOTYPES[name]
        assert (_ctypes_kind(restype), [_ctypes_kind(t) for t in argtypes]) == (ret, args), name
    lib = q.load_library()
    for name, (restype, argtypes) in _lib.PROTOTYPES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == list(argtypes), name


def test_create_fails_loudly_without_gpu_or_files():
    import torch
    lib = q.load_library()
    with pytest.raises(ValueError):
        q.QMInterface(taskFile="/nonexistent/task.info")   # QMInterface.cpp:45: invalid_argument on a missing file
    if not torch.cuda.is_available():
        with pytest.raises(q.QmbError) as e:
            q.Solver(batch=2)
        assert "no CPU fallback" in str(e.value)
    cfg = _lib.Config(b"/nonexistent/task.info", _lib.asset("qm_robot.urdf").encode(), _lib.asset("qm_reference.info").encode(), None, 1, 0, 0.0, 0.0, 0, 0)
    h = C.c_void_p()
    assert lib.qmb200_create(C.byref(cfg), C.byref(h)) == -2 and b"not found" in lib.qmb200_last_error(None)
    assert lib.qmb200_create(None, C.byref(h)) == -1


def test_gait_schedule_tiling_matches_python_twin():
    """GaitSchedule::getModeSchedule tiling: C++ host helper vs the numpy generator used for the synthetic batches."""
    for gait in ("stance", "trot", "flying_trot"):
        times, modes = synthetic._gait_template(_lib.asset("qm_gait.info"), gait)
        ev, md, n = gait_schedule(gait, 10.3, 11.0, 14.0)
        e2, m2 = synthetic.tile_schedule(times, modes, 10.3, 11.0, 14.0)
        assert n == len(e2) and md[0] == 15 and md[n] == 15
        np.testing.assert_allclose(ev[:n], e2, atol=1e-12); np.testing.assert_array_equal(md[:n + 1], m2)
    ev, md, n = gait_schedule("trot", 0.0, -1.0, 1.0)
    np.testing.assert_allclose(np.diff(ev[:n]), 0.35); assert list(md[1:3]) == [9, 6]   # LF_RH then RF_LH (gait.info:30-43)


def test_synthetic_batches_are_shard_invariant_and_deterministic():
    full, wf = synthetic.make_batch(np.arange(24), config=5)
    part, wp = synthetic.make_batch(np.arange(8, 16), config=5)
    for k in full:
        np.testing.assert_array_equal(full[k][8:16], part[k])
    np.testing.assert_array_equal(wf["rbd"][8:16], wp["rbd"])
    again, _ = synthetic.make_batch(np.arange(24), config=5)
    np.testing.assert_array_equal(full["x0"], again["x0"])
    assert set(np.unique(full["modes"])) <= {0, 6, 9, 15}
    u = synthetic.uniform(1, np.arange(4000), 3, 8, -1.0, 1.0); assert abs(u.mean()) < 0.02 and abs(u.std() - 1 / np.sqrt(3)) < 0.02


def test_shard_ranges_cover_the_batch():
    from qm_control_b200.parallel import shard_range
    for total, world in ((8192, 8), (10, 4), (7, 8), (1, 1)):
        spans = [shard_range(total, r, world) for r in range(world)]
        assert spans[0][0] == 0 and spans[-1][1] == total and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


class _GaitTwin:
    """List-based restatement of GaitSchedule [upstream, recalled] used to cross-check the C++ host object."""

    def __init__(self):
        self.ev = [0.5]; self.md = [15, 15]; self.tmpl = ([0.0, 1.0], [15]); self.pts = 0.1   # reference.info:27-52, task.info:9

    def tile(self, start, final):
        times, modes = self.tmpl; self.ev.append(start)
        while self.ev[-1] < final:
            for i, m in enumerate(modes):
                self.md.append(m); self.ev.append(self.ev[-1] + (times[i + 1] - times[i]))
        self.md.append(15)

    def insert(self, tmpl, start, final):
        self.tmpl = tmpl; idx = int(np.searchsorted(self.ev, start, side="left"))
        if idx < len(self.ev):
            del self.ev[idx:]; del self.md[idx + 1:]
        stance = 0.0 if self.md[-1] == 15 else self.pts
        if stance > 0:
            self.ev.append(start); self.md.append(15)
        self.tile(start + stance, final)

    def get(self, lo, hi):
        idx = int(np.searchsorted(self.ev, lo, side="left"))
        if idx > 0:
            del self.ev[:idx - 1]; del self.md[:idx - 1]; self.md[0] = 15
        start = self.ev[-1]; self.ev.pop(); self.md.pop(); self.tile(start, hi)
        return list(self.ev), list(self.md)


def test_stateful_gait_schedule_follows_the_controller_protocol():
    """MPC ticks ask for [t0 - T, tf + T] (SwitchedModelReferenceManager::modifyReferences); gait commands arrive through
    GaitReceiver::preSolverRun → insertModeSequenceTemplate(template, finalTime, timeHorizon)."""
    from qm_control_b200.interface import GaitSchedule
    gs = GaitSchedule(); tw = _GaitTwin(); T = 1.0
    tmpl = {g: synthetic._gait_template(_lib.asset("qm_gait.info"), g) for g in ("trot", "flying_trot", "stance")}
    t0 = 0.0
    for tick in range(400):
        t0 = 0.01 * tick
        if tick == 50:
            gs.insertModeSequenceTemplate("trot", t0 + T, T); tw.insert((list(tmpl["trot"][0]), tmpl["trot"][1]), t0 + T, T)
        if tick == 200:
            gs.insertModeSequenceTemplate("flying_trot", t0 + T, T); tw.insert((list(tmpl["flying_trot"][0]), tmpl["flying_trot"][1]), t0 + T, T)
        ev, md, n = gs.getModeSchedule(t0 - T, t0 + 2 * T); ev_t, md_t = tw.get(t0 - T, t0 + 2 * T)
        assert n == len(ev_t); np.testing.assert_allclose(ev[:n], ev_t, rtol=0, atol=1e-12); assert list(md[:n + 1]) == md_t
        assert md[0] == 15 and md[n] == 15 and np.all(np.diff(ev[:n]) > 0) and ev[n - 1] >= t0 + 2 * T
        if tick == 49:
            assert set(md[:n + 1]) == {15}                              # standing until the first gait command
        if tick == 120:                                                 # trot since t = 1.5: LF_RH / RF_LH alternate every 0.35 s
            k = int(np.searchsorted(ev[:n], 1.5 + 1e-9)); assert list(md[k:k + 4]) == [9, 6, 9, 6]; np.testing.assert_allclose(np.diff(ev[k - 1:k + 3]), 0.35)
        if tick == 300:                                                 # the switch trot → flying trot passes through phaseTransitionStanceTime of stance
            k = int(np.searchsorted(ev[:n], 3.0 - 1e-9)); assert md[k + 1] == 15 and abs(ev[k + 1] - ev[k] - 0.1) < 1e-12


def test_header_is_plain_c_and_struct_layouts_match_the_python_binding(tmp_path):
    """include/qmb200.h must compile as C (the boundary a cgo / JNI / C++ maintainer binds) and the ctypes mirrors of its structs must have
    the same size and field offsets."""
    import subprocess
    src = tmp_path / "layout.c"
    fields_cfg = [n for n, _ in _lib.Config._fields_]; fields_g = [n for n, _ in _lib.WbcGains._fields_]
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "qmb200.h"', 'int main(void) {', '  printf("%zu\\n", sizeof(qmb200_config));']
    body += ['  printf("%%zu\\n", offsetof(qmb200_config, %s));' % f for f in fields_cfg]
    body += ['  printf("%zu\\n", sizeof(qmb200_wbc_gains));'] + ['  printf("%%zu\\n", offsetof(qmb200_wbc_gains, %s));' % f for f in fields_g]
    body += ['  printf("%d %d %d %d %d %d %d\\n", QMB200_NX, QMB200_NU, QMB200_RBD, QMB200_CMD, QMB200_TARGET, QMB200_EMAX, QMB200_KMAX);', '  return 0; }']
    src.write_text("\n".join(body) + "\n"); exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)], text=True).split("\n")
    it = iter(out)
    assert int(next(it)) == C.sizeof(_lib.Config)
    for f in fields_cfg:
        assert int(next(it)) == getattr(_lib.Config, f).offset, f
    assert int(next(it)) == C.sizeof(_lib.WbcGains)
    for f in fields_g:
        assert int(next(it)) == getattr(_lib.WbcGains, f).offset, f
    assert [int(v) for v in next(it).split()] == [_lib.NX, _lib.NU, _lib.RBD, _lib.CMD, _lib.TARGET, _lib.EMAX, _lib.KMAX]
