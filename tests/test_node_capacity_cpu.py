"""Premises of tests/test_node_capacity_gpu.py, on the oracle alone: the capacity thresholds it states follow from the kernels' formulas, and every grid it
runs has the node counts its case claims, with every robot solvable and no non-positive interval on any grid."""
import math
import os
import re

import numpy as np
import pytest

import _schedules as S
import test_node_capacity_gpu as cap
from qm_control_b200._lib import EMAX

KERNELS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "qm_control_b200", "csrc", "kernels", "mpc_kernels.cu")


def _src():
    with open(KERNELS) as f:
        return f.read()


def _const(src, name):
    m = re.search(r"\b%s = (\d+)" % name, src); assert m, name
    return int(m.group(1))


def test_thresholds_follow_from_the_kernels():
    """K1 (mpc_kernels.cu:38-45): every warp of the setup kernel stages, per node, the previous and the new node time (8 + 8 B), the node's event (4 B), a
    SetupIdx {int iu, ix; double au, ax} (24 B) and a flag (4 B), plus EMAX event times and 64 B of modes: 48 nmax + 320 B, rounded up to 16 B, times
    SETUP_WARPS = 4 warps per CTA (the launch at :1181).  Past 48 KB the launch needs the 200 KB opt-in of mpc_configure_device (:1167); mpc_alloc (:1157)
    refuses more than 200 KB.  So the opt-in is first used at nmax = 250 (4 x 12320 B > 49152 B) and the last accepted nmax is 1060 (4 x 51200 B = 200 KB).
    K3 (:509, :614-617): node types live in shared memory for n <= RIC_NTYPE = 512; from n = 513 every node_type(k) reads SI_TYPE from the stage record.
    K4 (:866, :885): one CTA of 32 LS_WARPS = 128 threads walks k = tid, tid + 128, ... <= N = n - 1: ceil(n / 128) passes, three from n = 257."""
    src = _src()
    assert "struct SetupIdx { int iu, ix; double au, ax; };" in src
    assert "(size_t)nmax * (8 + 8 + 4 + sizeof(SetupIdx) + 4) + 8 * EMAX + 64" in src
    assert "SETUP_WARPS * ((setup_smem_per_warp(nmax) + 15) & ~(size_t)15) > 200 * 1024" in src
    assert "cudaFuncSetAttribute(mpc_setup_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)" in src
    warps = _const(src, "SETUP_WARPS")
    setup = lambda nmax: warps * (((nmax * (8 + 8 + 4 + 24 + 4) + 8 * EMAX + 64) + 15) // 16 * 16)
    opt_in = next(m for m in range(1, 4096) if setup(m) > 48 * 1024)
    limit = max(m for m in range(1, 4096) if setup(m) <= 200 * 1024)
    assert (opt_in, limit) == (cap.K1_OPT_IN, cap.NODE_LIMIT), (opt_in, limit)
    assert "const bool types_in_smem = n <= RIC_NTYPE;" in src and _const(src, "RIC_NTYPE") == cap.RIC_NTYPE
    assert "for (int k = tid; k <= N; k += 32 * LS_WARPS)" in src and 32 * _const(src, "LS_WARPS") == cap.LS_THREADS
    assert next(n for n in range(1, 4096) if math.ceil(n / cap.LS_THREADS) >= 3) == 2 * cap.LS_THREADS + 1
    # the DDP trial CTA: ddp.lineSearch steps 1, 1/2, ... >= 1/100 (capi_mpc.inc), lanes padded to a power of two, RO_RPC_MAX robots at most
    assert "constexpr int RO_RPC_MAX = 16;" in src and "RO_THREADS = 128" in src
    trials = sum(1 for j in range(32) if 0.5 ** j >= 1e-2); pitch = 1 << (trials - 1).bit_length()
    assert min(128 // pitch, 16) == cap.DDP_RPC, (trials, pitch)


@pytest.mark.parametrize("case", sorted(cap.GRIDS))
def test_grids_have_the_claimed_node_counts(oracle, case):
    names, prob, _ = cap.long_batch(); dt = cap.GRIDS[case]; nmax = cap.default_nmax(dt)
    oracle.mpc_set(dt=dt, horizon=cap.H)
    try:
        res = S.oracle_per_robot(oracle, prob, nmax)
    finally:
        oracle.mpc_set(dt=cap.DT, horizon=cap.H)
    errors = {names[b]: err for b, (_, err) in enumerate(res) if err is not None}
    assert not errors, errors
    n = np.array([int(r["n_nodes"][0]) for r, _ in res])
    cap.assert_grid(case, names, n, nmax)
    for b, (r, _) in enumerate(res):
        assert not S.grid_has_nonpositive_interval(r["t"][0], r["event"][0], n[b]), (case, names[b])


def test_the_padding_batch_is_solvable(oracle):
    names, prob, _ = cap._base(); assert len(names) % 4
    res = S.oracle_per_robot(oracle, prob, cap.default_nmax(cap.DT))
    assert all(err is None for _, err in res), [err for _, err in res]
