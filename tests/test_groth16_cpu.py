"""The G2 model (tests/g2_model.py), the test-only trusted setup (tests/groth16_model.py) on the oracle's witnesses of several gadget
circuits in both witness forms, and the host side of pob_msm_g2 / pob_groth16_prove: scratch sizes, declarations, no CPU path."""
import ctypes
import os
import random
import zlib

import numpy as np
import pytest

import g1_model as gm
import g2_model as g2m
import groth16_model as g16
import quotient_model as qm
from helpers import suite
from r1cs_reader import R1cs, witness_ints

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q = g2m.Q
# gadget circuits with 0, 1, 2, 5 and 32 public outputs; the domain of each is at most 2^11
SUITES = ["test_poseidon_2", "test_divide", "test_mask", "test_selector", "test_num_2_bits_safe_32", "test_is_in_range",
          "test_assert_less_than", "test_rlp_integer_1"]


# ---- F_q2 and G2 ---------------------------------------------------------------------------------------------------------------
def test_fq2_field_laws():
    rng = random.Random(21)
    el = lambda: (rng.randrange(Q), rng.randrange(Q))
    for _ in range(50):
        a, b, c = el(), el(), el()
        assert g2m.mul2(a, b) == g2m.mul2(b, a)
        assert g2m.mul2(g2m.mul2(a, b), c) == g2m.mul2(a, g2m.mul2(b, c))
        assert g2m.mul2(a, g2m.add2(b, c)) == g2m.add2(g2m.mul2(a, b), g2m.mul2(a, c))
        assert g2m.mul2(a, g2m.ONE) == a and g2m.add2(a, g2m.neg2(a)) == g2m.ZERO
        assert g2m.mul2(a, g2m.inv2(a)) == g2m.ONE
        # the device forms: Karatsuba and complex squaring give the same products
        v0, v1 = a[0] * b[0] % Q, a[1] * b[1] % Q
        assert ((v0 - v1) % Q, ((a[0] + a[1]) * (b[0] + b[1]) - v0 - v1) % Q) == g2m.mul2(a, b)
        assert ((a[0] + a[1]) * (a[0] - a[1]) % Q, 2 * a[0] * a[1] % Q) == g2m.mul2(a, a)
    assert g2m.mul2((0, 1), (0, 1)) == (Q - 1, 0)                      # u^2 = -1
    for a in ((0, 5), (7, 0), (1, Q - 1)):                              # elements with a zero half, and edges
        assert g2m.mul2(a, g2m.inv2(a)) == g2m.ONE


def test_twist_constants():
    assert g2m.mul2(g2m.B2, (9, 1)) == (3, 0)                            # b' = 3 / (9 + u)
    assert g2m.on_curve(g2m.G)
    assert g2m.mul(g2m.R_ORDER, g2m.G, reduce=False) is g2m.INF      # [r] G2 = O
    assert g2m.mul(g2m.R_ORDER - 1, g2m.G) == g2m.neg(g2m.G)
    rng = random.Random(22)
    for _ in range(3):
        a, b = rng.randrange(1, g2m.R_ORDER), rng.randrange(1, g2m.R_ORDER)
        pa = g2m.mul(a, g2m.G)
        assert g2m.on_curve(pa) and g2m.mul(b, pa) == g2m.mul(a * b, g2m.G)
        assert g2m.add(pa, g2m.mul(b, g2m.G)) == g2m.mul(a + b, g2m.G)
    assert g2m.add(g2m.G, g2m.neg(g2m.G)) is g2m.INF
    assert g2m.add(g2m.G, g2m.G) == g2m.mul(2, g2m.G)
    assert g2m.msm([g2m.G, g2m.mul(3, g2m.G), g2m.INF], [5, 7, 9]) == g2m.mul(26, g2m.G)


def test_encoding_order():
    p = g2m.mul(12345, g2m.G)
    enc = g2m.encode_points([p, g2m.INF])
    assert enc.shape == (2, 16) and not enc[1].any()
    coords = [sum(int(enc[0][4 * k + i]) << (64 * i) for i in range(4)) for k in range(4)]
    assert [gm.from_mont(c) for c in coords] == [p[0][0], p[0][1], p[1][0], p[1][1]]
    canon = g2m.encode_points([p], mont=False)
    assert g2m.decode_point(canon[0]) == p and g2m.decode_point([0] * 16) is g2m.INF


# ---- the trapdoor setup on real circuits -----------------------------------------------------------------------------------------
def _circuit(name, opt, tmp_path):
    """(R1cs, W) of the suite's first accepted case in the given form, from the oracle's --O0 witness through the file's labels"""
    import pob_b200
    from oracle import oracle
    s = suite(name)
    f = str(tmp_path / ("%s_%d.r1cs" % (name, opt)))
    pob_b200.write_r1cs(s["main"], f, opt=opt)
    R = R1cs(f)
    case = next(c for c in s["cases"] if c["expected"] is not None)
    w = oracle.run(s["main"], case["input"])
    try:
        assert w.ok
        W = witness_ints(w.limbs[R.labels.astype(np.int64)])
    finally:
        w.free()
    return R, W


def _quotient(R, W):
    A, B, C = R.products(W)
    return qm.quotient(A, B, C, W[:R.n_pub_out + R.n_pub_in + 1], R.m)


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
@pytest.mark.parametrize("name", SUITES)
def test_trapdoor_model(name, opt, tmp_path):
    R, W = _circuit(name, opt, tmp_path)
    assert len(R.failing_rows(W)) == 0
    rng = random.Random(zlib.crc32(name.encode()) + opt)
    toxic = [rng.randrange(1, qm.P) for _ in range(5)]
    S = g16.Setup(R, *toxic)
    np_ = S.n_pub
    q = _quotient(R, W)
    assert len(q) == S.n and S.h_keys.shape == (S.n,) and S.c_keys.shape == (S.n_vars - np_ - 1,)
    for r, s in [(0, 0)] + [(rng.randrange(1 << 256), rng.randrange(1 << 256)) for _ in range(3)]:
        a, b, c = S.proof_scalars(W, q, r, s)
        assert S.verify(a, b, c, W[:np_ + 1]), (r, s)
    # a changed private entry that some row reads (its quotient recomputed, as the prover would) fails
    used = sorted(set(int(x) for x in R.wire) - set(range(np_ + 1)))
    rng.shuffle(used)
    for j in used:
        Wt = W.copy()
        Wt[j] = (Wt[j] + 1) % qm.P
        if len(R.failing_rows(Wt)) > 0:
            break
    else:
        raise AssertionError("no private entry that a row reads")
    a, b, c = S.proof_scalars(Wt, _quotient(R, Wt), 0, 0)
    assert not S.verify(a, b, c, Wt[:np_ + 1])
    # one changed q_k fails
    qt = q.copy()
    k = rng.randrange(len(q))
    qt[k] = (qt[k] + 1) % qm.P
    a, b, c = S.proof_scalars(W, qt, 5, 7)
    assert not S.verify(a, b, c, W[:np_ + 1])
    # a wrong public input fails
    a, b, c = S.proof_scalars(W, q, 0, 0)
    wp = W[:np_ + 1].copy()
    wp[0] = 2
    assert not S.verify(a, b, c, wp)


# ---- host side of the library ------------------------------------------------------------------------------------------------------
def test_g2_work_bytes():
    """at least the grouped list (4 n) and the G1 scratch; monotone from n = 2^8 (below, the step from c = 4 to c = 5 drops 13 window
    sums, 3.3 KB, while the buckets grow by less)"""
    import pob_b200
    prev = 0
    for lg in range(0, 29):
        for n in ((1 << lg), (1 << lg) + 1, 3 << max(lg - 1, 0)):
            assert pob_b200.msm_g2_work_bytes(n) >= max(4 * n, pob_b200.msm_g1_work_bytes(n))
        b = pob_b200.msm_g2_work_bytes(1 << lg)
        assert lg <= 8 or b >= prev
        prev = b
    for bad, code in ((0, -1), ((1 << 31) + 1, -5)):
        with pytest.raises(pob_b200.PobError) as e:
            pob_b200.msm_g2_work_bytes(bad)
        assert e.value.code == code


def test_proof_json_shape():
    import pob_b200
    p = pob_b200.Proof((1, 2), ((3, 4), (5, 6)), None)
    j = p.to_json()
    assert j["protocol"] == "groth16" and j["curve"] == "bn128"
    assert j["pi_a"] == ["1", "2", "1"] and j["pi_b"] == [["3", "4"], ["5", "6"], ["1", "0"]] and j["pi_c"] == ["0", "1", "0"]
    assert pob_b200.public_json([7, qm.P + 1]) == ["7", "1"]
    limbs = [0] * 32
    limbs[0], limbs[4], limbs[8], limbs[12], limbs[16], limbs[20] = 1, 2, 3, 4, 5, 6
    assert pob_b200.proof_from_limbs(limbs) == pob_b200.Proof((1, 2), ((3, 4), (5, 6)), None)


def test_declared_and_no_cpu_path():
    import pob_b200
    hdr = open(os.path.join(ROOT, "include", "pob_b200.h")).read()
    for decl in ("int pob_msm_g2_work_bytes(uint64_t n, uint64_t *bytes);",
                 "int pob_msm_g2(int device, const void *bases, const void *scalars, uint64_t n,",
                 "int pob_groth16_work_bytes(pob_handle *h, uint64_t *bytes);",
                 "int pob_groth16_prove(pob_handle *h, uint32_t index, const pob_groth16_key *key,",
                 "} pob_groth16_key;"):
        assert decl in hdr, decl
    L = pob_b200.lib()
    assert L.pob_groth16_work_bytes(None, None) == -1
    assert L.pob_groth16_prove(None, 0, None, None, None, None, None, 0, None) == -1
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is visible")
    except ImportError:
        pass
    n = 4
    w = ctypes.c_uint64(0)
    assert L.pob_msm_g2_work_bytes(n, ctypes.byref(w)) == 0
    # well-formed, disjoint, aligned (never dereferenced) addresses: the call gets as far as looking for the device
    rc = L.pob_msm_g2(0, 1 << 20, 2 << 20, n, 3 << 20, 4 << 20, w.value, None)
    assert rc == -2 and b"device" in L.pob_last_error()
