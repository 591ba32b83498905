"""Single operations of the device tower and pairing (csrc/fq12_hd.h, csrc/pairing.cuh) through the test-only probe
(tests/devprobe/pairing_probe.cu), each compared exactly with the model (tests/pairing_model.py): F_q6 and F_q12 products, squares
and inverses on edge operands (0, 1, q - 1, a zero half) and random ones, conjugation and the Frobenius maps, cyclotomic squaring on
cyclotomic-subgroup elements, the sparse line product, the final exponentiation alone, the Miller loop alone (its value raised to
(q^12 - 1) / r by the model's pow is the model's pairing) and the subgroup check [r]Q = O."""
import os
import random
import sys

import pytest

import g1_model as gm
import g2_model as g2m
import pairing_model as pm

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

pytestmark = pytest.mark.gpu

Q, R = pm.Q, pm.R_ORDER


def _operands(rng, k=6):
    """edge operands, then k random ones"""
    r = lambda: pm.random12(rng)
    qm1 = pm.from_coeffs([Q - 1] * 12)
    return [pm.ZERO, pm.ONE, qm1, (r()[0], pm.Z6), (pm.Z6, r()[1]), (qm1[0], pm.Z6), (pm.from_fq2((0, 1))[0], r()[1])] + \
           [r() for _ in range(k)]


def _six(a):
    return (a[0], pm.Z6)


def test_fq6_ops():
    import pairing
    rng = random.Random(61)
    a = _operands(rng)
    b = list(reversed(_operands(rng)))
    assert pairing.elem(pairing.FQ6_MUL, a, b) == [_six((pm.mul6(x[0], y[0]), None)) for x, y in zip(a, b)]
    assert pairing.elem(pairing.FQ6_SQR, a) == [_six((pm.mul6(x[0], x[0]), None)) for x in a]
    want = [_six((pm.Z6 if x[0] == pm.Z6 else pm.inv6(x[0]), None)) for x in a]          # 1 / 0 gives 0
    assert pairing.elem(pairing.FQ6_INV, a) == want


def test_fq12_ops():
    import pairing
    rng = random.Random(62)
    a = _operands(rng)
    b = list(reversed(_operands(rng)))
    assert pairing.elem(pairing.FQ12_MUL, a, b) == [pm.mul12(x, y) for x, y in zip(a, b)]
    assert pairing.elem(pairing.FQ12_SQR, a) == [pm.sqr12(x) for x in a]
    assert pairing.elem(pairing.FQ12_INV, a) == [pm.ZERO if x == pm.ZERO else pm.inv12(x) for x in a]
    assert pairing.elem(pairing.FQ12_CONJ, a) == [pm.conj12(x) for x in a]


def test_frobenius():
    import pairing
    rng = random.Random(63)
    a = _operands(rng, k=2)
    for op, k in ((pairing.FROB1, 1), (pairing.FROB2, 2), (pairing.FROB3, 3)):
        assert pairing.elem(op, a) == [pm.frob(x, k) for x in a], k


def _cyclotomic(x):
    """x^((q^6 - 1)(q^2 + 1)), in the cyclotomic subgroup"""
    f = pm.mul12(pm.conj12(x), pm.inv12(x))
    return pm.mul12(pm.frob(f, 2), f)


def test_cyclotomic_squaring():
    import pairing
    rng = random.Random(64)
    a = [pm.ONE] + [_cyclotomic(pm.random12(rng)) for _ in range(4)]
    assert pairing.elem(pairing.CYC_SQR, a) == [pm.sqr12(x) for x in a]


def test_sparse_line_product():
    import pairing
    rng = random.Random(65)
    a = _operands(rng)
    e2 = lambda: (rng.randrange(Q), rng.randrange(Q))
    lines = [(e2(), e2(), e2()) for _ in a]
    lines[1] = ((0, 0), e2(), (0, 0))
    lines[2] = ((Q - 1, Q - 1), (Q - 1, Q - 1), (Q - 1, Q - 1))
    b = [((c0, c3, c4), pm.Z6) for c0, c3, c4 in lines]                           # the probe reads the line from b.c0
    want = [pm.mul12(x, ((c0, pm.Z2, pm.Z2), (c3, c4, pm.Z2))) for x, (c0, c3, c4) in zip(a, lines)]
    assert pairing.elem(pairing.MUL_034, a, b) == want


def test_final_exponentiation_alone():
    import pairing
    rng = random.Random(66)
    a = [pm.ONE, pm.ZERO, pm.random12(rng), pm.random12(rng)]
    assert pairing.elem(pairing.FINAL_EXP, a) == [pm.final_exp(x) for x in a]


def test_miller_loop_alone_and_subgroup():
    import pairing
    rng = random.Random(67)
    outside = pm.twist_point_outside_g2(68)
    g1s = [gm.G, gm.mul(rng.randrange(1, R), gm.G), None, gm.G, gm.G]
    g2s = [g2m.G, g2m.mul(rng.randrange(1, R), g2m.G), g2m.G, None, outside]
    f, in_g2 = pairing.miller(g1s, g2s)
    for p, q, v in zip(g1s[:4], g2s[:4], f[:4]):
        assert pm.final_exp(v) == pm.pairing(p, q)
    assert f[2] == pm.ONE and f[3] == pm.ONE                                    # O on either side: 1, before the exponentiation too
    assert in_g2 == [True, True, True, True, False]
    assert g2m.mul(R, outside, reduce=False) is not None
