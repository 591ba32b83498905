"""The quotient model (tests/quotient_model.py) on the CPU: its roots and shift, its transforms, and the identity that the GPU tests
use at every size -- h(r) (r^n - 1) = A^(r) B^(r) - C^(r), with h through q_i / (g^n - 1) on the coset -- on the oracle's reduced
Spend(31) witness with rows from the written `.r1cs`."""
import random

import numpy as np

import quotient_model as qm
from helpers import suite
from r1cs_reader import R1cs, witness_ints


def test_roots_and_shift():
    assert qm.W28 == 19103219067921713944291392827692070036145651957329286315305642004821462161904
    assert (qm.P - 1) % (1 << 28) == 0 and qm.T % 2 == 1
    assert pow(5, (qm.P - 1) // 2, qm.P) == qm.P - 1                 # 5 is a non-residue
    assert all(pow(k, (qm.P - 1) // 2, qm.P) == 1 for k in (2, 3, 4))   # and the smallest one >= 2
    assert pow(qm.W28, 1 << 27, qm.P) == qm.P - 1                     # w28 has order exactly 2^28
    for log_n in (1, 10, 18, 22, 25, 27):
        g = qm.shift(log_n)
        assert pow(g, 1 << log_n, qm.P) == qm.P - 1
    g28 = qm.shift(28)
    assert g28 == 25 and pow(g28, 1 << 28, qm.P) not in (1, qm.P - 1)
    assert [qm.domain_log(m, 1) for m in (215962292, 21508380, 2605281, 261862)] == [28, 25, 22, 18]


def test_ntt_round_trip():
    rng = random.Random(10)
    x = np.array([rng.randrange(qm.P) for _ in range(1 << 10)], dtype=object)
    assert (qm.intt(qm.ntt(x)) == x).all()
    y = qm.ntt(x)                                                     # and ntt is the evaluation at w^i
    w = qm.root(10)
    for i in (0, 1, 517, 1023):
        assert y[i] == sum(int(c) * pow(w, i * j, qm.P) for j, c in enumerate(x)) % qm.P


def _spend_o1(tmp_path):
    """the reduced Spend(31) rows' A.w, B.w, C.w on the oracle's witness, and w[0 .. n_pub]"""
    import pob_b200
    from oracle import oracle
    f = str(tmp_path / "spend_o1.r1cs")
    pob_b200.write_r1cs("Spend(31)", f, opt=1)
    R = R1cs(f)
    w = oracle.run("Spend(31)", suite("test_spend")["cases"][0]["input"])
    try:
        W = witness_ints(w.limbs[R.labels.astype(np.int64)])
    finally:
        w.free()
    A, B, C = R.products(W)
    return R, A, B, C, W[:R.n_pub_out + R.n_pub_in + 1]


def _sides(q, log_n, r, vecs):
    """(h(r) (r^n - 1), A^(r) B^(r) - C^(r)) with A^(r), B^(r), C^(r) over the given rows only"""
    n = 1 << log_n
    g = qm.shift(log_n)
    h = qm.bary(q, g, log_n, r) * pow(pow(g, n, qm.P) - 1, qm.P - 2, qm.P) % qm.P
    a, b, c = (qm.bary(v, 1, log_n, r) for v in vecs)
    return h * (pow(r, n, qm.P) - 1) % qm.P, (a * b - c) % qm.P


def test_model_quotient_on_reduced_spend(tmp_path):
    R, A, B, C, w_pub = _spend_o1(tmp_path)
    assert ((A * B - C) % qm.P == 0).all()
    m = R.m
    q = qm.quotient(A, B, C, w_pub, m)
    log_n = qm.domain_log(m, len(w_pub) - 1)
    assert log_n == 18 and len(q) == 1 << 18
    nz = m + len(w_pub)
    _, vecs = qm.rows(A, B, C, w_pub, m)
    rows = [v[:nz] for v in vecs]
    rng = random.Random(262144)
    for _ in range(2):
        r = rng.randrange(qm.P)
        lhs, rhs = _sides(q, log_n, r, rows)
        assert lhs == rhs
    i = rng.randrange(len(q))                                         # one changed entry breaks it
    q[i] = (q[i] + 1) % qm.P
    lhs, rhs = _sides(q, log_n, rng.randrange(qm.P), rows)
    assert lhs != rhs
