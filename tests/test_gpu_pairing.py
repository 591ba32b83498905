"""pob_bn254_pairing against the pairing model (tests/pairing_model.py): exact values on the generators and random pairs, O on either
side, bilinearity over 1000 random (a, b) checked on the GPU alone, e([r-1]P, Q) e(P, Q) = 1, and the consumer-stream call."""
import os
import random
import sys

import pytest

import g1_model as gm
import g2_model as g2m
import pairing_model as pm
from r1cs_reader import limbs_of
from test_gpu_msm import _dev

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

pytestmark = pytest.mark.gpu

R = pm.R_ORDER


def _pair_dev(g1, g2, stream=None):
    """pob_bn254_pairing over device tensors of key-form points; the (n, 48) uint64 output"""
    import torch
    import pob_b200
    n = g1.shape[0]
    out = torch.empty((n, 48), dtype=torch.uint64, device=g1.device)
    torch.cuda.synchronize()
    handle = None if stream is None else stream.cuda_stream
    rc = pob_b200.lib().pob_bn254_pairing(g1.device.index, g1.data_ptr(), g2.data_ptr(), n, out.data_ptr(), handle)
    assert rc == 0, pob_b200.lib().pob_last_error()
    if stream is not None:
        stream.synchronize()
    return out


def _values(out):
    import torch
    raw = out.view(torch.int64).cpu().numpy().tobytes()
    return [tuple(int.from_bytes(raw[384 * i + 32 * k:384 * i + 32 * k + 32], "little") for k in range(12)) for i in range(out.shape[0])]


def test_exact_against_model():
    import pob_b200
    rng = random.Random(41)
    g1s = [gm.G] + [gm.mul(rng.randrange(1, R), gm.G) for _ in range(3)]
    g2s = [g2m.G] + [g2m.mul(rng.randrange(1, R), g2m.G) for _ in range(3)]
    got = pob_b200.pairing(g1s, g2s)
    for p, q, e in zip(g1s, g2s, got):
        assert e == pm.coeffs(pm.pairing(p, q))


def test_infinity_gives_one():
    import pob_b200
    one = pm.coeffs(pm.ONE)
    assert pob_b200.pairing([None, gm.G, None], [g2m.G, None, None]) == [one] * 3


def test_bilinearity_on_the_gpu():
    """e([a]G1, [b]G2) = e([ab]G1, G2) = e(G1, [ab]G2) for 1000 random (a, b), every value computed on the GPU"""
    import torch
    import g2
    rng = random.Random(42)
    n = 1000
    a = [rng.randrange(1, R) for _ in range(n)]
    b = [rng.randrange(1, R) for _ in range(n)]
    ab = [x * y % R for x, y in zip(a, b)]
    sc = lambda v: _dev(limbs_of(v, R))
    ones = [1] * n
    e1 = _pair_dev(g2.fixed_base(1, sc(a)), g2.fixed_base(2, sc(b)))
    e2 = _pair_dev(g2.fixed_base(1, sc(ab)), g2.fixed_base(2, sc(ones)))
    e3 = _pair_dev(g2.fixed_base(1, sc(ones)), g2.fixed_base(2, sc(ab)))
    assert torch.equal(e1.view(torch.int64), e2.view(torch.int64)) and torch.equal(e1.view(torch.int64), e3.view(torch.int64))
    assert len(set(_values(e1[:50]))) == 50
    assert _values(e3[:1])[0] == pm.coeffs(pm.pairing(gm.mul(ab[0], gm.G), g2m.G))


def test_inverse_and_stream():
    import torch
    import pob_b200
    rng = random.Random(43)
    p, q = gm.mul(rng.randrange(1, R), gm.G), g2m.mul(rng.randrange(1, R), g2m.G)
    e_inv, e = pob_b200.pairing([gm.mul(R - 1, p), p], [q, q])
    assert pm.mul12(pm.from_coeffs(e_inv), pm.from_coeffs(e)) == pm.ONE
    g1 = _dev(gm.encode_bases([p, gm.G] * 8))
    g2 = _dev(g2m.encode_points([q, g2m.G] * 8))
    sync = _pair_dev(g1, g2)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(10 ** 7)
    asyn = _pair_dev(g1, g2, st)
    assert torch.equal(sync.view(torch.int64), asyn.view(torch.int64))
    assert _values(sync[:1])[0] == e


def test_argument_errors():
    import torch
    import pob_b200
    L = pob_b200.lib()
    g1 = torch.zeros((2, 8), dtype=torch.uint64, device="cuda")
    g2 = torch.zeros((2, 16), dtype=torch.uint64, device="cuda")
    out = torch.full((2, 48), 7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for args in ((0, g2.data_ptr(), 2, out.data_ptr()), (g1.data_ptr(), 0, 2, out.data_ptr()), (g1.data_ptr(), g2.data_ptr(), 2, 0),
                 (g1.data_ptr(), g2.data_ptr(), 0, out.data_ptr()), (g1.data_ptr() + 8, g2.data_ptr(), 2, out.data_ptr()),
                 (g1.data_ptr(), g2.data_ptr(), 2, g2.data_ptr())):
        assert L.pob_bn254_pairing(0, *args, None) == -1, args
    torch.cuda.synchronize()
    assert (out == 7).all()
