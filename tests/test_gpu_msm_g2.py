"""The BN254 G2 multi-exponentiation on the GPU (pob_msm_g2) against tests/g2_model.py, and the device F_q2 / G2 arithmetic behind it.

Small cases compare with the model exactly, on distinct bases P_i = [t_i]G2 (t_i known), so the answer is [sum t_i s_i]G2.  Large
cases tile K = 1024 model points P_k = [t_k]G2 up to n: then sum_i [s_i] P_i = [sum_k t_k S_k]G2 with S_k = sum_{i = k mod K} s_i, the
class sums of tests/test_gpu_msm.py.  One changed scalar must change every large result."""
import os
import random
import sys

import numpy as np
import pytest

import g1_model as gm
import g2_model as g2m
from test_gpu_msm import MAIN_SHAPE, SPECIAL, TILE, _class_sums, _dev, _random_scalars, _witness_tensor

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

pytestmark = pytest.mark.gpu

Q = g2m.Q
RINV = pow(1 << 256, -1, Q)
_TILE_T = []


def _chain(n, rng):
    """n distinct model points [t0 + i d]G2 by successive additions, and their t_i"""
    t0, d = rng.randrange(1, g2m.R_ORDER), rng.randrange(1, g2m.R_ORDER)
    P, D, pts = g2m.mul(t0, g2m.G), g2m.mul(d, g2m.G), []
    for _ in range(n):
        pts.append(P)
        P = g2m.add(P, D)
    return pts, [(t0 + i * d) % g2m.R_ORDER for i in range(n)]


def _tile():
    if not _TILE_T:
        pts, ts = _chain(TILE, random.Random(2048))
        _TILE_T.extend([_dev(g2m.encode_points(pts)), ts])
    return _TILE_T[0], _TILE_T[1]


def _tiled_bases(n):
    import torch
    B, _ = _tile()
    return B.view(torch.int64).repeat((n + TILE - 1) // TILE, 1)[:n].contiguous().view(torch.uint64)


def _tiled_want(s):
    _, ts = _tile()
    return g2m.mul(sum(t * v for t, v in zip(ts, _class_sums(s))) % g2m.R_ORDER, g2m.G)


def _check_tiled(bases, s, flip_at):
    """the MSM of (bases, s) equals the tiled model; flipping bit 0 of s[flip_at] changes it (s is restored)"""
    import torch
    import pob_b200
    want = _tiled_want(s)
    assert pob_b200.msm_g2(bases, s) == want
    v = s.view(torch.int64)
    old = v[flip_at, 0].clone()
    v[flip_at, 0] ^= 1
    try:
        changed = pob_b200.msm_g2(bases, s)
        assert changed != want and changed == _tiled_want(s)
    finally:
        v[flip_at, 0] = old


# ---- 1. arithmetic, element by element ---------------------------------------------------------------------------------------
def test_fq2_elements():
    import g2
    rng = random.Random(31)
    edge = [0, 1, Q - 1, gm.to_mont(1), Q - 2, 1 << 253]
    halves = [(x, 0) for x in edge] + [(0, x) for x in edge] + [(x, y) for x in edge[:3] for y in edge[:3]]
    a = [h for h in halves for _ in halves] + [(rng.randrange(Q), rng.randrange(Q)) for _ in range(1000)]
    b = [h for _ in halves for h in halves] + [(rng.randrange(Q), rng.randrange(Q)) for _ in range(1000)]
    mont = lambda v: g2m.scale2(v, RINV)                                # the device product of raw limbs: a b / R
    assert g2.elem(g2.MUL, a, b) == [mont(g2m.mul2(x, y)) for x, y in zip(a, b)]
    assert g2.elem(g2.SQR, a) == [mont(g2m.mul2(x, x)) for x in a]
    assert g2.elem(g2.ADD, a, b) == [g2m.add2(x, y) for x, y in zip(a, b)]
    assert g2.elem(g2.SUB, a, b) == [g2m.sub2(x, y) for x, y in zip(a, b)]
    assert g2.elem(g2.NEG, a) == [g2m.neg2(x) for x in a]
    to_m = lambda v: (gm.to_mont(v[0]), gm.to_mont(v[1]))
    from_m = lambda v: (gm.from_mont(v[0]), gm.from_mont(v[1]))
    inv_in = a[:400]
    assert g2.elem(g2.INV, inv_in) == [to_m(g2m.inv2(from_m(x))) if x != (0, 0) else (0, 0) for x in inv_in]


def test_point_formulas():
    import g2
    rng = random.Random(32)
    P = [g2m.mul(rng.randrange(1, g2m.R_ORDER), g2m.G) for _ in range(12)] + [g2m.G]
    O = g2m.INF
    a, b = [], []
    for p in P:
        q = P[rng.randrange(len(P))]
        for x, y in ((p, q), (p, p), (p, g2m.neg(p)), (O, p), (p, O), (O, O)):
            a.append(x)
            b.append(y)
    dbl = lambda x: g2m.add(x, x)
    for op, f in ((g2.G2_ADD, g2m.add), (g2.G2_ADD_AFF, g2m.add),
                  (g2.G2_DBL, lambda x, y: dbl(x)), (g2.G2_DBL_AFF, lambda x, y: dbl(x)),
                  (g2.G2_ADD_Z, lambda x, y: g2m.add(dbl(x), dbl(y))), (g2.G2_ADD_AFF_Z, lambda x, y: g2m.add(dbl(x), y)),
                  (g2.G2_ADD_ZZ, lambda x, y: g2m.add(g2m.mul(3, x), g2m.mul(3, y)))):
        assert g2.point(op, a, b) == [f(x, y) for x, y in zip(a, b)], op
    two = [dbl(p) for p in P]
    assert g2.point(g2.G2_ADD_AFF_Z, P, two) == [g2m.mul(4, p) for p in P]     # the mixed addition's doubling branch, Z != 1
    assert g2.point(g2.G2_ADD_AFF_Z, P, [g2m.neg(t) for t in two]) == [O] * len(P)
    ks = [0, 1, 2, 3, 0xffffffff] + [rng.randrange(1 << 32) for _ in range(len(a) - 5)]
    assert g2.point(g2.G2_MUL_U32, a, b, ks) == [g2m.mul(k, x) if x is not O else O for k, x in zip(ks, a)]


def test_fixed_base_keys():
    """the test probe's batched [k_i]G, which builds the trapdoor keys of tests/test_gpu_groth16.py, on edge and random scalars"""
    import g2
    rng = random.Random(33)
    ks = SPECIAL + [rng.randrange(1 << 256) for _ in range(64)]
    s = _dev(gm.encode_scalars(ks))
    p1 = g2.fixed_base(1, s).cpu().numpy()
    p2 = g2.fixed_base(2, s).cpu().numpy()
    assert (gm.encode_bases([gm.mul(k, gm.G) for k in ks]) == p1).all()
    assert (g2m.encode_points([g2m.mul(k, g2m.G) for k in ks]) == p2).all()


# ---- 2. exact small MSMs -----------------------------------------------------------------------------------------------------
def _exact(pts, ts, ss):
    import pob_b200
    want = g2m.mul(sum(t * s for t, s in zip(ts, ss)) % g2m.R_ORDER, g2m.G)
    got = pob_b200.msm_g2(_dev(g2m.encode_points(pts)), _dev(gm.encode_scalars(ss)))
    assert got == want, (len(pts), got, want)


@pytest.mark.parametrize("n", [1, 2, 3, 31, 33, 256, 1000, 4096])
def test_exact_small(n):
    rng = random.Random(n)
    pts, ts = _chain(n, rng)
    kinds = [lambda: rng.randrange(1 << 256)] + [lambda v=v: v for v in SPECIAL]
    _exact(pts, ts, [kinds[rng.randrange(len(kinds))]() for _ in range(n)])
    _exact(pts, ts, [rng.randrange(1 << 256) for _ in range(n)])
    for v in SPECIAL:
        _exact(pts, ts, [v] * n)


def test_exact_special_cases():
    import pob_b200
    rng = random.Random(6)
    pts, ts = _chain(1000, rng)
    assert pob_b200.msm_g2(_dev(g2m.encode_points(pts)), _dev(gm.encode_scalars([0] * 1000))) is None
    inf_pts = [g2m.INF if i % 3 == 0 else p for i, p in enumerate(pts)]
    inf_ts = [0 if i % 3 == 0 else t for i, t in enumerate(ts)]
    _exact(inf_pts, inf_ts, [rng.randrange(1 << 256) for _ in range(1000)])
    _exact([g2m.INF] * 33, [0] * 33, [rng.randrange(1 << 256) for _ in range(33)])
    for n in (1000, 4096):
        _exact([pts[0]] * n, [ts[0]] * n, [rng.randrange(1 << 256)] * n)
        _exact([pts[0]] * n, [ts[0]] * n, [1] * n)
    alt = [pts[i // 2] if i % 2 == 0 else g2m.neg(pts[i // 2]) for i in range(1000)]
    alt_t = [ts[i // 2] if i % 2 == 0 else g2m.R_ORDER - ts[i // 2] for i in range(1000)]
    s = [rng.randrange(1 << 256) for _ in range(500)]
    assert pob_b200.msm_g2(_dev(g2m.encode_points(alt)), _dev(gm.encode_scalars([v for v in s for _ in (0, 1)]))) is None
    _exact(alt, alt_t, [rng.randrange(1 << 256) for _ in range(1000)])


@pytest.mark.parametrize("c", range(4, 17))
def test_every_window_size(c):
    """the window rule is G1's (csrc/msm.cuh msm_window_bits): n = 2^(c + 3) + 1 has window c"""
    import torch
    n = (1 << (c + 3)) + 1
    s = _random_scalars(n, seed=100 + c)
    rng = random.Random(c)
    pos = torch.tensor([rng.randrange(n) for _ in SPECIAL], device="cuda")
    s.view(torch.int64)[pos] = _dev(gm.encode_scalars(SPECIAL)).view(torch.int64)
    _check_tiled(_tiled_bases(n), s, rng.randrange(n))


# ---- 3. exact large MSMs -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [20, 24])
def test_large_random(log_n):
    n = 1 << log_n
    _check_tiled(_tiled_bases(n), _random_scalars(n, seed=200 + log_n), n // 5)


def test_skewed_witness_like():
    """96 % of the entries 0 or 1, the rest random, at 2^24"""
    import torch
    n = 1 << 24
    s = _random_scalars(n, seed=196)
    g = torch.Generator(device="cuda")
    g.manual_seed(197)
    small = torch.rand(n, device="cuda", generator=g) < 0.96
    bits = torch.randint(0, 2, (n,), device="cuda", generator=g)
    v = s.view(torch.int64)
    v[small] = 0
    v[small, 0] = bits[small]
    _check_tiled(_tiled_bases(n), s, 54321)


def _witness_case(c, rng):
    import torch
    w = _witness_tensor(c.witness_device_ptr(0), c.n_signals)
    bases = _tiled_bases(c.n_signals)
    _check_tiled(bases, w, rng.randrange(c.n_signals))
    del bases
    torch.cuda.empty_cache()


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
def test_spend_witness(opt):
    import pob_b200
    from helpers import suite
    c = pob_b200.Circuit("Spend(31)", max_slots=1, opt=opt)
    try:
        assert c.run([suite("test_spend")["cases"][0]["input"]]).status[0] == 0
        _witness_case(c, random.Random(131 + opt))
    finally:
        c.close()


@pytest.mark.parametrize("opt,n_signals", [(1, 21454051), (0, 215907954)], ids=["O1", "O0"])
def test_main_shape(opt, n_signals):
    """main_proof_of_burn's witness, both forms; --O0 puts 27.6 GB of G2 bases next to one slot"""
    import pob_b200
    from pob_b200 import synth
    packed = synth.pack_instances(synth.make_batch(1, MAIN_SHAPE, seed=4242), MAIN_SHAPE)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1, opt=opt)
    try:
        assert c.run_packed(packed).status[0] == 0 and c.n_signals == n_signals
        _witness_case(c, random.Random(25 + opt))
    finally:
        c.close()


# ---- 4. the consumer stream ---------------------------------------------------------------------------------------------------
def test_consumer_stream_equals_the_synchronous_call():
    """on a non-blocking stream that sleeps first, with the scratch and out allocated on it: the same point as without a stream"""
    import torch
    import pob_b200
    n = 100003
    bases, s = _tiled_bases(n), _random_scalars(n, seed=7)
    want = pob_b200.msm_g2(bases, s)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(10 ** 8)
    out = pob_b200.msm_g2(bases, s, stream=st)
    st.synchronize()
    assert g2m.decode_point(out.cpu().tolist()) == want == _tiled_want(s)


# ---- 5. errors -----------------------------------------------------------------------------------------------------------------
def test_errors_before_anything_runs():
    import torch
    import pob_b200
    L = pob_b200.lib()
    n = 256
    need = pob_b200.msm_g2_work_bytes(n)
    bases, s = _tiled_bases(n), _random_scalars(n, seed=1)
    out = torch.zeros(16, dtype=torch.uint64, device="cuda")
    work = torch.zeros(need + 128, dtype=torch.uint8, device="cuda")
    B, S, O, W = bases.data_ptr(), s.data_ptr(), out.data_ptr(), work.data_ptr()
    torch.cuda.synchronize()
    cases = [(B, S, n, O, W, need), (None, S, n, O, W, need), (B, None, n, O, W, need), (B, S, n, None, W, need), (B, S, n, O, None, need),
             (B, S, 0, O, W, need), (B + 8, S, n, O, W, need), (B, S + 8, n, O, W, need), (B, S, n, O + 8, W, need), (B, S, n, O, W + 8, need),
             (B, S, n, O, W, need - 1), (B, S, n, W + 16, W, need), (B, S, n, B + 128 * (n - 1), W, need), (B, S, n, O, B, need),
             (B, S, n, O, S, need)]
    for k, (b, sc, nn, o, w, wb) in enumerate(cases):
        rc = L.pob_msm_g2(0, b, sc, nn, o, w, wb, None)
        assert rc == (0 if k == 0 else -1), (k, rc, L.pob_last_error())
        if k == 0:
            want = g2m.decode_point(out.cpu().tolist())
            out.zero_()
            work.fill_(0xA5)
            torch.cuda.synchronize()
    assert not out.view(torch.int64).any() and (work == 0xA5).all()   # nothing ran after the first call
    assert want == _tiled_want(s)
    assert L.pob_msm_g2(0, B, S, (1 << 31) + 1, O, W, need, None) == -5
