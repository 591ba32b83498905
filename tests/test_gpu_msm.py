"""The BN254 G1 multi-exponentiation on the GPU (pob_msm_g1) against tests/g1_model.py.

Small cases compare with the model exactly, on distinct bases P_i = [t_i]G (t_i known), so the answer is [sum t_i s_i]G.  Large
cases tile K = 1024 model points P_k = [t_k]G up to n: then sum_i [s_i] P_i = [sum_k t_k S_k]G with S_k = sum_{i = k mod K} s_i,
and the class sums come from exact torch integer reductions over the scalars' 32-bit halves (each half-sum < 2^60 up to 2^28
entries), independently of the library.  One changed scalar must change every large result."""
import os
import random
import sys

import numpy as np
import pytest

import g1_model as gm

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

pytestmark = pytest.mark.gpu

MAIN_SHAPE = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)
TILE = 1024
SPECIAL = [0, 1, 2, gm.R_ORDER - 1, gm.R_ORDER, gm.R_ORDER + 1, (1 << 256) - 1]
_TILE_T = []


def _dev(arr):
    import torch
    return torch.from_numpy(arr.view(np.int64)).cuda().view(torch.uint64)


def _chain(n, rng):
    """n distinct model points [t0 + i d]G by successive additions, and their t_i"""
    t0, d = rng.randrange(1, gm.R_ORDER), rng.randrange(1, gm.R_ORDER)
    P, D, pts = gm.mul(t0, gm.G), gm.mul(d, gm.G), []
    for _ in range(n):
        pts.append(P)
        P = gm.add(P, D)
    return pts, [(t0 + i * d) % gm.R_ORDER for i in range(n)]


def _tile():
    """K model points P_k = [t_k]G as a (K, 8) device tensor, and t"""
    if not _TILE_T:
        pts, ts = _chain(TILE, random.Random(1024))
        _TILE_T.extend([_dev(gm.encode_bases(pts)), ts])
    return _TILE_T[0], _TILE_T[1]


def _tiled_bases(n):
    import torch
    B, _ = _tile()
    return B.view(torch.int64).repeat((n + TILE - 1) // TILE, 1)[:n].contiguous().view(torch.uint64)


def _class_sums(s):
    """S_k = sum_{i = k mod K} s_i as exact ints, from an (n, 4) uint64 CUDA tensor"""
    import torch
    n = s.shape[0]
    halves = s.view(torch.int32).view(n, 8)
    pad = (-n) % TILE
    S = [0] * TILE
    for h in range(8):
        col = halves[:, h].to(torch.int64) & 0xffffffff
        if pad:
            col = torch.cat([col, torch.zeros(pad, dtype=torch.int64, device=col.device)])
        sums = col.view(-1, TILE).sum(0).cpu().tolist()
        for k in range(TILE):
            S[k] += sums[k] << (32 * h)
    return S


def _tiled_want(s):
    _, ts = _tile()
    return gm.mul(sum(t * v for t, v in zip(ts, _class_sums(s))) % gm.R_ORDER, gm.G)


def _check_tiled(bases, s, flip_at):
    """the MSM of (bases, s) equals the tiled model; flipping bit 0 of s[flip_at] changes it (s is restored)"""
    import torch
    import pob_b200
    want = _tiled_want(s)
    assert pob_b200.msm_g1(bases, s) == want
    v = s.view(torch.int64)
    old = v[flip_at, 0].clone()
    v[flip_at, 0] ^= 1
    try:
        changed = pob_b200.msm_g1(bases, s)
    finally:
        v[flip_at, 0] = old
    assert changed != want and changed == _tiled_want(_flipped(s, flip_at))


def _flipped(s, i):
    import torch
    t = s.clone()
    t.view(torch.int64)[i, 0] ^= 1
    return t


class _View:
    """a (n, 4) uint64 device tensor over memory the library owns (a resident witness), without a copy"""
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n, 4), "typestr": "<i8", "data": (ptr, False), "version": 3}


def _witness_tensor(ptr, n):
    import torch
    return torch.as_tensor(_View(ptr, n), device="cuda").view(torch.uint64)


def _random_scalars(n, seed):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return torch.randint(-(1 << 63), (1 << 63) - 1, (n, 4), dtype=torch.int64, device="cuda", generator=g).view(torch.uint64)


# ---- 1. arithmetic, element by element ---------------------------------------------------------------------------------------
def test_fq_elements():
    import fq
    rng = random.Random(11)
    edge = [0, 1, 2, gm.Q - 1, gm.Q - 2, 1 << 253, (1 << 253) - 1, gm.M32, (1 << 64) - 1, gm.to_mont(1)]
    a = edge * len(edge) + [rng.randrange(gm.Q) for _ in range(2000)]
    b = [e for e in edge for _ in edge] + [rng.randrange(gm.Q) for _ in range(2000)]
    rinv = pow(1 << 256, -1, gm.Q)
    assert fq.elem(fq.MUL, a, b) == [x * y * rinv % gm.Q for x, y in zip(a, b)]
    assert fq.elem(fq.ADD, a, b) == [(x + y) % gm.Q for x, y in zip(a, b)]
    assert fq.elem(fq.SUB, a, b) == [(x - y) % gm.Q for x, y in zip(a, b)]
    assert fq.elem(fq.NEG, a) == [(-x) % gm.Q for x in a]
    assert fq.elem(fq.TO_MONT, a) == [gm.to_mont(x) for x in a]
    assert fq.elem(fq.FROM_MONT, a) == [gm.from_mont(x) for x in a]
    inv_in = [x for x in a[:300]]
    assert fq.elem(fq.INV, inv_in) == [gm.to_mont(pow(gm.from_mont(x), -1, gm.Q)) if x else 0 for x in inv_in]


def test_point_formulas():
    import fq
    rng = random.Random(12)
    P = [gm.mul(rng.randrange(1, gm.R_ORDER), gm.G) for _ in range(24)] + [gm.G]
    O = gm.INF
    a, b = [], []
    for p in P:
        q = P[rng.randrange(len(P))]
        for x, y in ((p, q), (p, p), (p, gm.neg(p)), (O, p), (p, O), (O, O)):
            a.append(x)
            b.append(y)
    for op, f in ((fq.G1_ADD, lambda x, y: gm.add(x, y)),
                  (fq.G1_ADD_AFF, lambda x, y: gm.add(x, y)),
                  (fq.G1_DBL, lambda x, y: gm.add(x, x)),
                  (fq.G1_DBL_AFF, lambda x, y: gm.add(x, x)),
                  (fq.G1_ADD_Z, lambda x, y: gm.add(gm.add(x, x), gm.add(y, y))),
                  (fq.G1_ADD_AFF_Z, lambda x, y: gm.add(gm.add(x, x), y))):
        assert fq.point(op, a, b) == [f(x, y) for x, y in zip(a, b)], op
    # 2a + b with b = 2a (the mixed addition's doubling branch with Z != 1) and b = -2a
    two = [gm.add(p, p) for p in P]
    assert fq.point(fq.G1_ADD_AFF_Z, P, two) == [gm.mul(4, p) for p in P]
    assert fq.point(fq.G1_ADD_AFF_Z, P, [gm.neg(t) for t in two]) == [O] * len(P)
    ks = [0, 1, 2, 3, 0xffffffff] + [rng.randrange(1 << 32) for _ in range(len(a) - 5)]
    assert fq.point(fq.G1_MUL_U32, a, b, ks) == [gm.mul(k, x) if x is not O else O for k, x in zip(ks, a)]


# ---- 2. exact small MSMs -----------------------------------------------------------------------------------------------------
def _exact(pts, ts, ss):
    import pob_b200
    want = gm.mul(sum(t * s for t, s in zip(ts, ss)) % gm.R_ORDER, gm.G)
    got = pob_b200.msm_g1(_dev(gm.encode_bases(pts)), _dev(gm.encode_scalars(ss)))
    assert got == want, (len(pts), got, want)


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 255, 256, 1000, 4096])
def test_exact_small(n):
    rng = random.Random(n)
    pts, ts = _chain(n, rng)
    kinds = [lambda: rng.randrange(1 << 256)] + [lambda v=v: v for v in SPECIAL]
    ss = [kinds[rng.randrange(len(kinds))]() for _ in range(n)]
    _exact(pts, ts, ss)
    _exact(pts, ts, [rng.randrange(1 << 256) for _ in range(n)])
    for v in SPECIAL:
        _exact(pts, ts, [v] * n)


def test_exact_special_cases():
    import pob_b200
    rng = random.Random(5)
    pts, ts = _chain(1000, rng)
    assert pob_b200.msm_g1(_dev(gm.encode_bases(pts)), _dev(gm.encode_scalars([0] * 1000))) is None
    # some bases are infinity: they contribute nothing
    inf_pts = [gm.INF if i % 3 == 0 else p for i, p in enumerate(pts)]
    inf_ts = [0 if i % 3 == 0 else t for i, t in enumerate(ts)]
    _exact(inf_pts, inf_ts, [rng.randrange(1 << 256) for _ in range(1000)])
    _exact([gm.INF] * 33, [0] * 33, [rng.randrange(1 << 256) for _ in range(33)])
    # every base equal, every scalar equal: one deep bucket per window that doubles inside its sum
    for n in (1000, 4096):
        _exact([pts[0]] * n, [ts[0]] * n, [rng.randrange(1 << 256)] * n)
        _exact([pts[0]] * n, [ts[0]] * n, [1] * n)
    # P and -P alternating
    alt = [pts[i // 2] if i % 2 == 0 else gm.neg(pts[i // 2]) for i in range(1000)]
    alt_t = [ts[i // 2] if i % 2 == 0 else gm.R_ORDER - ts[i // 2] for i in range(1000)]
    s = [rng.randrange(1 << 256) for _ in range(500)]
    assert pob_b200.msm_g1(_dev(gm.encode_bases(alt)), _dev(gm.encode_scalars([v for v in s for _ in (0, 1)]))) is None
    _exact(alt, alt_t, [rng.randrange(1 << 256) for _ in range(1000)])


@pytest.mark.parametrize("c", range(4, 17))
def test_every_window_size(c):
    """pob_msm_g1 picks c = clamp(floor(log2 n) - 3, 4, 16) (csrc/msm.cuh msm_window_bits): n = 2^(c + 3) + 1 has window c"""
    import torch
    n = (1 << (c + 3)) + 1
    s = _random_scalars(n, seed=c)
    rng = random.Random(c)
    pos = torch.tensor([rng.randrange(n) for _ in SPECIAL], device="cuda")
    s.view(torch.int64)[pos] = _dev(gm.encode_scalars(SPECIAL)).view(torch.int64)
    _check_tiled(_tiled_bases(n), s, rng.randrange(n))


# ---- 3. exact large MSMs -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [20, 24])
def test_large_random(log_n):
    n = 1 << log_n
    _check_tiled(_tiled_bases(n), _random_scalars(n, seed=log_n), n // 3)


def test_skewed_witness_like():
    """96 % of the entries 0 or 1 (like a KeccakfRound-dominated witness), the rest random, at 2^24"""
    import torch
    n = 1 << 24
    s = _random_scalars(n, seed=96)
    g = torch.Generator(device="cuda")
    g.manual_seed(97)
    small = torch.rand(n, device="cuda", generator=g) < 0.96
    bits = torch.randint(0, 2, (n,), device="cuda", generator=g)
    v = s.view(torch.int64)
    v[small] = 0
    v[small, 0] = bits[small]
    _check_tiled(_tiled_bases(n), s, 12345)


def _witness_case(c, index, rng):
    """the witness MSM of resident instance `index` (A / B1 shape: all n_signals entries), with the tiled bases"""
    import torch
    ptr = c.witness_device_ptr(index)
    w = _witness_tensor(ptr, c.n_signals)
    bases = _tiled_bases(c.n_signals)
    _check_tiled(bases, w, rng.randrange(c.n_signals))
    del bases
    torch.cuda.empty_cache()


def _quotient_case(c, index, rng):
    """the H MSM over the quotient of instance `index`, reusing the quotient's work as the MSM's scratch"""
    import torch
    import pob_b200
    n = 1 << c.r1cs_domain()
    work = torch.empty((2 * n, 4), dtype=torch.uint64, device="cuda")
    q = c.r1cs_quotient(index, work=work)
    bases = _tiled_bases(n)
    want = _tiled_want(q)
    assert pob_b200.msm_g1(bases, q, work=work) == want
    i = rng.randrange(n)
    q.view(torch.int64)[i, 0] ^= 1
    assert pob_b200.msm_g1(bases, q, work=work) not in (want, None)
    del q, work, bases
    torch.cuda.empty_cache()


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
def test_spend_witness_and_quotient(opt):
    import pob_b200
    from helpers import suite
    c = pob_b200.Circuit("Spend(31)", max_slots=2, opt=opt)
    try:
        assert c.run([suite("test_spend")["cases"][0]["input"]]).status[0] == 0
        rng = random.Random(31 + opt)
        _witness_case(c, 0, rng)
        _quotient_case(c, 0, rng)
    finally:
        c.close()


def test_main_shape_reduced():
    """main_proof_of_burn, reduced witness (21,454,051 entries) and its 2^25 quotient"""
    import pob_b200
    from pob_b200 import synth
    packed = synth.pack_instances(synth.make_batch(1, MAIN_SHAPE, seed=4242), MAIN_SHAPE)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1, opt=1)
    try:
        assert c.run_packed(packed).status[0] == 0 and c.n_signals == 21454051
        rng = random.Random(25)
        _witness_case(c, 0, rng)
        _quotient_case(c, 0, rng)
    finally:
        c.close()


def test_main_shape_o0():
    """main_proof_of_burn, --O0 witness (215,907,954 entries) and its 2^28 quotient, one resident witness"""
    import pob_b200
    from pob_b200 import synth
    packed = synth.pack_instances(synth.make_batch(1, MAIN_SHAPE, seed=4242), MAIN_SHAPE)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1)
    try:
        assert c.run_packed(packed).status[0] == 0 and c.n_signals == 215907954
        rng = random.Random(28)
        _witness_case(c, 0, rng)
        _quotient_case(c, 0, rng)
    finally:
        c.close()


# ---- 5. the hand-off -------------------------------------------------------------------------------------------------------
def test_handoff_on_a_consumer_stream():
    """submit / acquire(stream) / quotient / witness MSM / H MSM on the quotient's work / release(stream), on a non-blocking stream
    that sleeps before each MSM: every result equals the synchronous calls on the same instance, so no slot was reused before the
    MSMs read it"""
    import torch
    import pob_b200
    from test_gpu_shapes import _spend_inputs
    inputs = _spend_inputs(4, seed=2718)
    c = pob_b200.Circuit("Spend(31)", max_slots=2, opt=1)
    try:
        n = 1 << c.r1cs_domain()
        wb, hb = _tiled_bases(c.n_signals), _tiled_bases(n)
        want = []
        for inp in inputs:
            assert c.run([inp]).status[0] == 0
            w = _witness_tensor(c.witness_device_ptr(0), c.n_signals)
            want.append((pob_b200.msm_g1(wb, w), pob_b200.msm_g1(hb, c.r1cs_quotient(0))))
        assert len(set(want)) == 4
        st = torch.cuda.Stream()
        got = []
        c.submit(c.pack(inputs))
        while True:
            r = c.acquire(st.cuda_stream)
            if r is None:
                break
            idx, ptr = r
            with torch.cuda.stream(st):
                work = torch.empty((2 * n, 4), dtype=torch.uint64, device="cuda")
            q = c.r1cs_quotient(idx, stream=st, work=work)
            with torch.cuda.stream(st):
                torch.cuda._sleep(10 ** 8)
            a = pob_b200.msm_g1(wb, (ptr, c.n_signals), stream=st)
            h = pob_b200.msm_g1(hb, q, stream=st, work=work)
            c.release(idx, st.cuda_stream)
            got.append((idx, a, h))
        assert (c.finish().status == 0).all()
        st.synchronize()
        for idx, a, h in got:
            assert (gm.decode_point(a.cpu().tolist()), gm.decode_point(h.cpu().tolist())) == want[idx]
    finally:
        c.close()


# ---- 6. errors ---------------------------------------------------------------------------------------------------------------
def test_errors_before_anything_runs():
    import ctypes
    import torch
    import pob_b200
    L = pob_b200.lib()
    n = 256
    need = pob_b200.msm_g1_work_bytes(n)
    bases, s = _tiled_bases(n), _random_scalars(n, seed=1)
    out = torch.zeros(8, dtype=torch.uint64, device="cuda")
    work = torch.zeros(need + 64, dtype=torch.uint8, device="cuda")
    B, S, O, W = bases.data_ptr(), s.data_ptr(), out.data_ptr(), work.data_ptr()
    torch.cuda.synchronize()
    cases = [(B, S, n, O, W, need), (None, S, n, O, W, need), (B, None, n, O, W, need), (B, S, n, None, W, need), (B, S, n, O, None, need),
             (B, S, 0, O, W, need), (B + 8, S, n, O, W, need), (B, S + 8, n, O, W, need), (B, S, n, O + 8, W, need), (B, S, n, O, W + 8, need),
             (B, S, n, O, W, need - 1), (B, S, n, W + 16, W, need), (B, S, n, B + 64, W, need), (B, S, n, O, B, need), (B, S, n, O, S, need)]
    for k, (b, sc, nn, o, w, wb) in enumerate(cases):
        rc = L.pob_msm_g1(0, b, sc, nn, o, w, wb, None)
        assert rc == (0 if k == 0 else -1), (k, rc, L.pob_last_error())
        if k == 0:
            want = gm.decode_point(out.cpu().tolist())
            out.zero_()
            work.fill_(0xA5)
            torch.cuda.synchronize()
    assert not out.view(torch.int64).any() and (work == 0xA5).all()   # nothing ran after the first call
    assert want == _tiled_want(s)
    assert L.pob_msm_g1(0, B, S, (1 << 31) + 1, O, W, need, None) == -5
