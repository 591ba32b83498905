"""The G1 model (tests/g1_model.py), the modulus-parameterised Montgomery product run with q, and the host side of pob_msm_g1:
scratch sizes, declarations, and no CPU path."""
import ctypes
import os
import random

import pytest

import g1_model as gm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_generator_order_and_group_law():
    assert gm.on_curve(gm.G)
    assert gm.mul(gm.R_ORDER, gm.G) is gm.INF
    assert gm.from_jac(gm.jac_add(gm.to_jac(gm.G), gm.to_jac(gm.neg(gm.G)))) is gm.INF
    assert gm.add(gm.G, gm.neg(gm.G)) is gm.INF
    assert gm.add(gm.INF, gm.G) == gm.G and gm.add(gm.G, gm.INF) == gm.G
    assert gm.add(gm.G, gm.G) == gm.from_jac(gm.jac_dbl(gm.to_jac(gm.G))) == gm.mul(2, gm.G)
    rng = random.Random(1)
    for _ in range(4):
        a, b = rng.randrange(gm.R_ORDER), rng.randrange(gm.R_ORDER)
        pa = gm.mul(a, gm.G)
        assert gm.on_curve(pa) and gm.mul(b, pa) == gm.mul(a * b, gm.G)
        assert gm.add(pa, gm.mul(b, gm.G)) == gm.mul(a + b, gm.G)
    assert gm.mul(gm.R_ORDER + 5, gm.G) == gm.mul(5, gm.G)          # [s]P = [s mod r]P


def test_naive_msm_and_encoding():
    rng = random.Random(2)
    ts = [rng.randrange(gm.R_ORDER) for _ in range(5)]
    ss = [rng.randrange(1 << 256) for _ in range(5)]
    pts = [gm.mul(t, gm.G) for t in ts]
    assert gm.msm(pts, ss) == gm.mul(sum(t * s for t, s in zip(ts, ss)), gm.G)
    assert gm.msm(pts + [gm.INF], ss + [7]) == gm.msm(pts, ss)
    enc = gm.encode_bases(pts + [gm.INF])
    assert enc.shape == (6, 8) and not enc[5].any()
    x = sum(int(enc[0][i]) << (64 * i) for i in range(4))
    assert gm.from_mont(x) == pts[0][0] and gm.to_mont(gm.from_mont(x)) == x
    limbs = [(pts[0][k] >> (64 * i)) & ((1 << 64) - 1) for k in (0, 1) for i in range(4)]
    assert gm.decode_point(limbs) == pts[0] and gm.decode_point([0] * 8) is gm.INF


def test_even_odd_montgomery_product_with_q():
    """fr_hd.h's mont_mul<M> is one implementation for Fr and F_q: its limb model, bounds asserted, with q"""
    rng = random.Random(3)
    rinv = pow(1 << 256, -1, gm.Q)
    vals = [0, 1, 2, gm.Q - 1, gm.Q - 2, 1 << 253, gm.M32, (1 << 224) - 1] + [rng.randrange(gm.Q) for _ in range(1500)]
    for i, a in enumerate(vals):
        b = vals[(i * 7 + 3) % len(vals)]
        assert gm.mont_limb_model(a, b, gm.Q) == a * b * rinv % gm.Q
    for _ in range(300):
        a, b = rng.randrange(gm.Q), rng.randrange(1 << 256)
        assert gm.mont_limb_model(a, b, gm.Q) == a * b * rinv % gm.Q


def test_work_bytes_bound():
    import pob_b200
    prev = 0
    for lg in range(0, 29):
        for n in ((1 << lg), (1 << lg) + 1, 3 << max(lg - 1, 0)):
            b = pob_b200.msm_g1_work_bytes(n)
            assert b >= 4 * n
            if n >= 1 << 18:
                assert b <= 64 * n, (n, b)
        b = pob_b200.msm_g1_work_bytes(1 << lg)
        assert b >= prev
        prev = b
    for n in (21454051, 215907954):                                    # the main shape's witnesses
        assert pob_b200.msm_g1_work_bytes(n) <= 64 * n
    with pytest.raises(pob_b200.PobError) as e:
        pob_b200.msm_g1_work_bytes(0)
    assert e.value.code == -1
    with pytest.raises(pob_b200.PobError) as e:
        pob_b200.msm_g1_work_bytes((1 << 31) + 1)
    assert e.value.code == -5


def test_declared_and_no_cpu_path():
    import pob_b200
    hdr = open(os.path.join(ROOT, "include", "pob_b200.h")).read()
    assert "int pob_msm_g1_work_bytes(uint64_t n, uint64_t *bytes);" in hdr
    assert "int pob_msm_g1(int device, const void *bases, const void *scalars, uint64_t n," in hdr
    L = pob_b200.lib()
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is visible")
    except ImportError:
        pass
    n = 4
    w = ctypes.c_uint64(0)
    assert L.pob_msm_g1_work_bytes(n, ctypes.byref(w)) == 0
    # well-formed, disjoint, aligned (never dereferenced) addresses: the call gets as far as looking for the device
    rc = L.pob_msm_g1(0, 1 << 20, 2 << 20, n, 3 << 20, 4 << 20, w.value, None)
    assert rc == -2 and b"device" in L.pob_last_error()
