"""The controller's model payload on the host, no GPU: the per-robot SRBD constants of qmb200_set_model_payload (qmb200_debug_srbd_constants) against
two independent derivations of the same constants from the edited URDF (tests/_payload_urdf.py): the product's own parser (qmb200_debug_model_blob)
and the oracle's (tests/_oracle.py model_info).  Also the header / binding layouts and the validation messages."""
import ctypes as C
import hashlib
import os
import re

import numpy as np
import pytest

from qm_control_b200 import _lib
from _payload_urdf import edited_urdf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROBOT_MASS = 27.371574   # sum of the URDF's link masses (test_oracle_cpu.py)
NS = 22                  # the SRBD constants proper: m, I_nom(9), I_nom_inv(9), c_nom(3); then two zeros of padding

PAYLOADS = {
    "ee": [1.5, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0],
    "ee_offset": [2.0, 0.03, -0.02, 0.05, 0.0, 0.0, 0.0, 0.0],
    "base": [0.0, 0.0, 0.0, 0.0, 3.0, 0.0, 0.0, 0.0],
    "base_offset": [0.0, 0.0, 0.0, 0.0, 4.0, 0.12, -0.05, 0.09],
    "both": [0.7, -0.01, 0.04, 0.02, 5.0, -0.2, 0.1, 0.06],
}


def _cfg(urdf=None):
    return _lib.Config(_lib.asset("qm_task.info").encode(), (urdf or _lib.asset("qm_robot.urdf")).encode(), _lib.asset("qm_reference.info").encode(), None, 1, 0, 0.0, 0.0, 0, 0)


def _srbd(payload, urdf=None):
    lib = _lib.load_library(); cfg = _cfg(urdf)
    pl = None if payload is None else np.ascontiguousarray(payload, dtype=np.float64).reshape(-1, 8)
    n = 1 if pl is None else pl.shape[0]; out = np.full((n, len(_lib.SRBD_LAYOUT)), np.nan)
    rc = lib.qmb200_debug_srbd_constants(C.byref(cfg), n, None if pl is None else pl.ctypes.data, out.ctypes.data)
    assert rc == 0, lib.qmb200_last_error(None).decode()
    return out


def _blob(urdf=None):
    lib = _lib.load_library(); cfg = _cfg(urdf)
    n = lib.qmb200_debug_model_blob(C.byref(cfg), None, 0); assert n > 0, lib.qmb200_last_error(None).decode()
    buf = (C.c_ubyte * n)(); assert lib.qmb200_debug_model_blob(C.byref(cfg), buf, n) == n
    return bytes(buf)


@pytest.fixture(scope="module")
def srbd_offset():
    """Byte offset of DevModel's SRBD fields (total_mass, I_nom, I_nom_inv, c_nom) in the model blob: where the nominal block's 176 bytes occur, once."""
    nominal = _srbd(None)[0, :NS].tobytes(); blob = _blob()
    off = blob.find(nominal)
    assert off >= 0 and blob.find(nominal, off + 1) < 0 and off % 8 == 0
    return off


def _blob_srbd(urdf, off):
    return np.frombuffer(_blob(urdf), dtype=np.float64, count=NS, offset=off)


def _close(a, b, tol=1e-12):
    """per block of like quantities (m, I_nom, I_nom_inv, c_nom), relative to the block's largest entry"""
    for name, sl in (("m", slice(0, 1)), ("I_nom", slice(1, 10)), ("I_nom_inv", slice(10, 19)), ("c_nom", slice(19, 22))):
        scale = max(np.max(np.abs(b[sl])), 1e-3)
        assert np.max(np.abs(a[sl] - b[sl])) <= tol * scale, (name, a[sl], b[sl])


def test_zero_payload_is_the_model_bit_for_bit(srbd_offset):
    """No payload and all-zero payload rows give DevModel's own SRBD fields bit for bit, padded with two zeros."""
    blob = np.frombuffer(_blob(), dtype=np.float64, count=NS, offset=srbd_offset)
    for rows in (_srbd(None), _srbd(np.zeros((3, 8))), _srbd([[0.0, 0.3, -0.2, 0.1, 0.0, 0.5, 0.5, -0.5]])):   # offsets of a zero mass do not matter
        for r in rows:
            assert r[:NS].tobytes() == blob.tobytes() and np.all(r[NS:] == 0.0)
    assert blob[0] == pytest.approx(ROBOT_MASS, abs=1e-9)


@pytest.mark.parametrize("name", sorted(PAYLOADS))
def test_constants_equal_the_edited_urdf_model(tmp_path, srbd_offset, name):
    """The constants of a payload row equal the product parser's constants for the URDF with the payload links, to 1e-12 per block."""
    pl = PAYLOADS[name]
    got = _srbd([pl])[0]
    ref = _blob_srbd(edited_urdf(tmp_path, pl), srbd_offset)
    _close(got[:NS], ref)
    assert got[0] == pytest.approx(ROBOT_MASS + pl[0] + pl[4], abs=1e-9)
    assert np.all(got[NS:] == 0.0)
    np.testing.assert_allclose(got[1:10].reshape(3, 3) @ got[10:19].reshape(3, 3), np.eye(3), atol=1e-12)


def test_rows_are_independent():
    """Several payloads in one call: row b depends on payload row b only."""
    rows = np.array([PAYLOADS[n] for n in sorted(PAYLOADS)] + [[0.0] * 8])
    together = _srbd(rows)
    for b, row in enumerate(rows):
        assert together[b].tobytes() == _srbd([row])[0].tobytes()


@pytest.mark.parametrize("name", sorted(PAYLOADS))
def test_constants_equal_the_oracle_on_the_edited_urdf(tmp_path, name):
    """A second, independent derivation: the oracle's model of the edited URDF (its own URDF parser and composite-body fold)."""
    from _oracle import Oracle
    pl = PAYLOADS[name]
    got = _srbd([pl])[0]
    info = Oracle(urdf=edited_urdf(tmp_path, pl)).model_info()
    assert info["mass"] == pytest.approx(ROBOT_MASS + pl[0] + pl[4], abs=1e-9)
    assert got[0] == pytest.approx(info["mass"], rel=1e-12)
    ref = np.concatenate([[info["mass"]], info["inertia_nominal"].ravel(), np.linalg.inv(info["inertia_nominal"]).ravel(), info["com_to_base"]])
    _close(got[:NS], ref)


def test_payload_changes_the_constants(tmp_path):
    """Sanity of the comparison itself: a 2 kg EE payload moves the composite by far more than the tolerances above."""
    nominal = _srbd(None)[0]; ee = _srbd([PAYLOADS["ee_offset"]])[0]
    assert ee[0] - nominal[0] == pytest.approx(2.0, abs=1e-12)
    assert np.max(np.abs(ee[19:22] - nominal[19:22])) > 1e-2 and np.max(np.abs(ee[1:10] - nominal[1:10])) > 1e-2


def test_edited_urdf_lives_in_the_temp_dir(tmp_path):
    """The helper writes under the given directory only; assets/ and the md5-pinned fixtures stay as they are."""
    watched = [os.path.join(ROOT, "assets", f) for f in sorted(os.listdir(os.path.join(ROOT, "assets")))]
    ref_dir = os.path.join(ROOT, "tests", "fixtures", "ref_inputs")
    watched += [os.path.join(ref_dir, f) for f in sorted(os.listdir(ref_dir))]
    before = {p: hashlib.md5(open(p, "rb").read()).hexdigest() for p in watched}
    path = edited_urdf(tmp_path, PAYLOADS["both"])
    assert os.path.dirname(path) == str(tmp_path) and "payload_ee" in open(path).read() and "payload_base" in open(path).read()
    assert {p: hashlib.md5(open(p, "rb").read()).hexdigest() for p in watched} == before


def test_validation_messages():
    lib = _lib.load_library(); cfg = _cfg(); out = np.zeros((1, 24))
    for bad, msg in (([np.nan, 0, 0, 0, 0, 0, 0, 0], "payload must be finite"), ([0, 0, 0, np.inf, 0, 0, 0, 0], "payload must be finite"),
                     ([-1.0, 0, 0, 0, 0, 0, 0, 0], "payload masses must be >= 0"), ([0, 0, 0, 0, -0.5, 0, 0, 0], "payload masses must be >= 0")):
        pl = np.array([bad], dtype=np.float64)
        assert lib.qmb200_debug_srbd_constants(C.byref(cfg), 1, pl.ctypes.data, out.ctypes.data) == -1
        assert lib.qmb200_last_error(None).decode() == "qmb200_debug_srbd_constants: " + msg
    assert lib.qmb200_debug_srbd_constants(C.byref(cfg), -1, None, out.ctypes.data) == -1
    src = open(os.path.join(ROOT, "qm_control_b200", "csrc", "capi.cu")).read()
    assert '"qmb200_set_model_payload"' in src   # the setter shares the validation (payload_error) under its own name


def test_header_and_binding_layouts():
    hdr = open(os.path.join(ROOT, "include", "qmb200.h")).read()
    assert re.search(r"#define QMB200_SRBD 24\b", hdr) and len(_lib.SRBD_LAYOUT) == 24 and _lib.SRBD_LAYOUT[0] == "m" and _lib.SRBD_LAYOUT[19:22] == ("c_nom_x", "c_nom_y", "c_nom_z")
    for sym, args in (("qmb200_set_model_payload", r"qmb200_handle\* h, const double\* payload /\*\[B\]\[8\] or NULL\*/"),
                      ("qmb200_get_model_payload", r"const qmb200_handle\* h, double\* payload /\*\[B\]\[8\]\*/, int32_t\* is_set"),
                      ("qmb200_debug_srbd_constants", r"const qmb200_config\* cfg, int32_t n, const double\* payload /\*\[n\]\[8\] or NULL\*/, double\* out /\*\[n\]\[QMB200_SRBD\]\*/")):
        assert re.search(r"int %s\(%s\);" % (sym, args), hdr), sym
        assert sym in _lib.SYMBOLS
    assert "[m_ee, o_ee_x, o_ee_y, o_ee_z, m_base, o_base_x, o_base_y, o_base_z]" in hdr and _lib.PAYLOAD_LAYOUT[0] == "m_ee" and _lib.PAYLOAD_LAYOUT[4] == "m_base"
    lib = _lib.load_library()
    for sym in ("qmb200_set_model_payload", "qmb200_get_model_payload", "qmb200_debug_srbd_constants"):
        assert getattr(lib, sym).argtypes is not None
