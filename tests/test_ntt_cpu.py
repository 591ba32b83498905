"""The transform probe (tests/devprobe/ntt_probe.cu) compiles for sm_90a, and the host side of the product's transforms
(csrc/ntt.cuh) that it exposes is right at every size 2^1 .. 2^28: the pass plan keeps its contract, and the root and coset tables
hold the powers the model (tests/quotient_model.py) computes with pow()."""
import functools
import os
import sys

import numpy as np
import pytest

import quotient_model as qm

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

TILE_LOG = 11
R_INV = pow(1 << 256, qm.P - 2, qm.P)
SIZES = range(1, qm.TWO_ADICITY + 1)


def _has_nvcc():
    import probe
    return probe.nvcc() is not None


@pytest.fixture(scope="module")
def ntt():
    if not _has_nvcc():
        pytest.skip("nvcc not available")
    import ntt
    return ntt


def _plain(limbs):
    """(k, 8) uint32 limbs of x R mod p, the form the tables are stored in -> object array of x"""
    import probe
    return np.array([v * R_INV % qm.P for v in probe.from_limbs(limbs)], dtype=object)


def _pows(vals):
    return np.array(list(vals), dtype=object)


def test_probe_compiles_for_sm90a(ntt, tmp_path):
    import ctypes
    so = ntt.build(out_dir=str(tmp_path))
    assert os.path.getsize(so) > 0
    L = ctypes.CDLL(so)
    for sym in ntt.SYMBOLS:
        assert hasattr(L, sym)


def test_plan_at_every_size(ntt):
    """stages sum to L; no pass exceeds the tile; every pass but the contiguous last one has at most T - 2 = 9 stages (global runs of
    >= 4 entries); as few passes as that allows; the passes before the last are balanced and the last is the largest"""
    for L in SIZES:
        T = min(L, TILE_LOG)
        k = ntt.plan(L)
        P = len(k)
        assert sum(k) == L and all(1 <= s <= T for s in k), (L, k)
        assert L <= T + (P - 1) * (T - 2), (L, k)
        assert P == 1 or L > T + (P - 2) * (T - 2), (L, k)                 # no fewer passes would do
        if P > 1:
            assert max(k[:-1]) <= T - 2, (L, k)
            assert max(k[:-1]) - min(k[:-1]) <= 1 and k[:-1] == sorted(k[:-1]), (L, k)
            assert k[-1] >= max(k[:-1]), (L, k)
            assert k[-1] - min(k) <= 1 or min(k[:-1]) == T - 2, (L, k)      # balanced unless the cap moved stages to the last
    pinned = {1: [1], 8: [8], 11: [11], 12: [6, 6], 13: [6, 7], 18: [9, 9], 19: [9, 10], 20: [9, 11], 21: [7, 7, 7],
              22: [7, 7, 8], 25: [8, 8, 9], 28: [9, 9, 10]}
    assert {L: ntt.plan(L) for L in pinned} == pinned


@functools.lru_cache(maxsize=None)
def _root_tables():
    w11 = qm.root(11)
    w11_inv = pow(w11, qm.P - 2, qm.P)
    return {"w_lo": _pows(pow(qm.W28, t, qm.P) for t in range(1 << 14)),
            "w_hi": _pows(pow(qm.W28, t << 14, qm.P) for t in range(1 << 14)),
            "loc": _pows(pow(w11, t, qm.P) for t in range(1 << 10)),
            "loc_inv": _pows(pow(w11_inv, t, qm.P) for t in range(1 << 10))}


def test_tables_at_every_size(ntt):
    """w28^t, w28^(2^14 t), w_11^(+-t) and the coset pair g^t, g^(2^g_log t) / n (g = w_(L+1), or 25 at L = 28), as stored"""
    want = _root_tables()
    for L in SIZES:
        got, g_log = ntt.tables(L)
        for name, w in want.items():
            if L == 1:
                assert (_plain(got[name]) == w).all(), name
            else:                                                           # the same for every domain
                assert np.array_equal(got[name], first[name]), (L, name)
        if L == 1:
            first = got
        n, g = 1 << L, qm.shift(L)
        assert len(got["g_lo"]) == 1 << g_log and len(got["g_lo"]) * len(got["g_hi"]) == n, (L, g_log)
        n_inv = pow(n, qm.P - 2, qm.P)
        assert (_plain(got["g_lo"]) == _pows(pow(g, t, qm.P) for t in range(1 << g_log))).all(), L
        assert (_plain(got["g_hi"]) == _pows(pow(g, t << g_log, qm.P) * n_inv % qm.P for t in range(n >> g_log))).all(), L
