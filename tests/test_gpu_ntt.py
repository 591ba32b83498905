"""The product's BN254 transforms (csrc/ntt.cuh) at every size 2^1 .. 2^28, through the test-only probe tests/devprobe/ntt_probe.cu,
against the definition (tests/quotient_model.py).

The inverse leaves position j holding coefficient k = rev_L(j) times g^k (g the coset shift, 1/n included); the forward takes
bit-reversed coefficients to the values at w^i.  Up to 2^16 every entry of random and structured vectors equals the Python model
(inverse, forward and the quotient sequence).  At every size, closed forms are checked on every entry up to 2^20 and above that on
2^16 random entries plus the first and last entry of every tile and pass block: a constant, impulses at natural and bit-reversed
positions, and the alternating vector.  Above 2^16, random vectors generated on the device must come back as the same polynomial
(barycentric evaluation on the device at two points), and the quotient must equal A.B - C of separately transformed copies."""
import os
import random
import sys

import numpy as np
import pytest

import quotient_model as qm
from r1cs_reader import witness_ints

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

pytestmark = pytest.mark.gpu

P = qm.P
TILE_LOG = 11
M64 = (1 << 64) - 1
EXACT_MAX, FULL_CLOSED_MAX, FULL_QUOTIENT_MAX = 16, 20, 22


def _to_dev(vals):
    import torch
    v = np.asarray(vals, dtype=object)
    limbs = np.stack([((v >> (64 * k)) & M64).astype(np.uint64) for k in range(4)], axis=1)
    return torch.from_numpy(np.ascontiguousarray(limbs).view(np.int64)).cuda()


def _ints(t, idx=None):
    """entries (all, or the rows idx) of an (n, 4) int64 CUDA tensor of limbs as Python ints"""
    import torch
    if idx is not None:
        t = t[torch.from_numpy(idx).cuda()]
    return witness_ints(t.cpu().numpy().view(np.uint64))


def _rev(idx, L):
    idx = np.asarray(idx, dtype=np.int64)
    out = np.zeros_like(idx)
    for b in range(L):
        out |= ((idx >> b) & 1) << (L - 1 - b)
    return out


class _Pow:
    """x^e for int64 arrays e in [0, 2^bits), from two tables of the model's powers"""
    def __init__(self, x, bits):
        self.h = (bits + 1) // 2
        self.lo = qm.powers(x, 1 << self.h)
        self.hi = qm.powers(pow(x, 1 << self.h, P), 1 << (bits - self.h))

    def __call__(self, e):
        e = np.asarray(e, dtype=np.int64)
        return self.lo[e & ((1 << self.h) - 1)] * self.hi[e >> self.h] % P


def _sample(ntt, L, rng):
    """None (every entry) up to 2^20; above, 2^16 random positions and the first and last entry of every tile and every block of
    every pass of the plan"""
    if L <= FULL_CLOSED_MAX:
        return None
    n = 1 << L
    T = min(L, TILE_LOG)
    idx = [rng.integers(0, n, 1 << 16, dtype=np.int64), np.array([0, n - 1], dtype=np.int64)]
    blk = L
    tiles = np.arange(n >> T, dtype=np.int64)
    for k in ntt.plan(L):
        log_s, log_c = blk - k, T - k
        for u, i in ((tiles << log_c, 0), (((tiles + 1) << log_c) - 1, (1 << k) - 1)):
            idx.append(((u >> log_s) << blk) + (u & ((1 << log_s) - 1)) + (i << log_s))
        blocks = np.arange(n >> blk, dtype=np.int64)
        idx += [blocks << blk, ((blocks + 1) << blk) - 1]
        blk -= k
    return np.unique(np.concatenate(idx))


def _check(got, want, what):
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, "%s: %d entries differ, first at %s" % (what, len(bad), bad[:8])


@pytest.fixture(scope="module")
def ntt():
    import ntt
    return ntt


# ---- exact, every entry against the model --------------------------------------------------------------------------------------
def _vectors(L, rng):
    n = 1 << L
    return {"random": [rng.randrange(P) for _ in range(n)],
            "p-1": [P - 1] * n,
            "mixed": [rng.choice((0, 1, P - 1, P - 2, rng.randrange(P))) for _ in range(n)]}


@pytest.mark.parametrize("L", range(1, EXACT_MAX + 1))
def test_exact(ntt, L):
    """every entry of inverse, forward and the quotient sequence equals the Python model"""
    n = 1 << L
    rng = random.Random(1000 + L)
    rev = qm._bitrev(n)
    gk = qm.powers(qm.shift(L), n)
    for name, x in _vectors(L, rng).items():
        t = _to_dev(x)
        ntt.inverse(L, t)
        _check(_ints(t), (qm.intt(x) * gk % P)[rev], "inverse of %s at 2^%d" % (name, L))
        t = _to_dev(x)
        ntt.forward(L, t)
        _check(_ints(t), qm.ntt(np.asarray(x, dtype=object)[rev]), "forward of %s at 2^%d" % (name, L))
    vs = _vectors(L, rng)
    a, b, c = vs["random"], vs["mixed"], [rng.randrange(P) for _ in range(n)]
    ta, tb, tc = (_to_dev(v) for v in (a, b, c))
    ntt.quotient(L, ta, tb, tc)
    A, B, C = (qm.ntt(qm.intt(v) * gk % P) for v in (a, b, c))
    _check(_ints(ta), (A * B - C) % P, "quotient at 2^%d" % L)


# ---- closed forms at every size ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", range(1, qm.TWO_ADICITY + 1))
def test_closed_forms(ntt, L):
    import torch
    n = 1 << L
    rng = np.random.default_rng(2000 + L)
    idx = _sample(ntt, L, rng)
    pos = np.arange(n, dtype=np.int64) if idx is None else idx
    k = _rev(pos, L)                                       # coefficient held at each checked position after the inverse
    w, g = _Pow(qm.root(L), L), _Pow(qm.shift(L), L)
    n_inv = pow(n, P - 2, P)
    zero = np.zeros(len(pos), dtype=object)
    p1, one = _to_dev([P - 1]), _to_dev([1])
    x = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    try:
        # the constant p - 1: the single coefficient p - 1 at k = 0, and p - 1 everywhere again
        x.copy_(p1.expand(n, 4))
        ntt.inverse(L, x)
        want = zero.copy()
        want[pos == 0] = P - 1
        _check(_ints(x, idx), want, "inverse of p-1 at 2^%d" % L)
        ntt.forward(L, x)
        _check(_ints(x, idx), np.full(len(pos), P - 1, dtype=object), "p-1 round trip at 2^%d" % L)

        # an impulse at natural position j: coefficients w^(-jk) / n times g^k
        j = int(rng.integers(1, n)) if n > 2 else 1
        x.zero_()
        x[j] = one[0]
        ntt.inverse(L, x)
        _check(_ints(x, idx), w((-j * k) % n) * n_inv % P * g(k) % P, "inverse of e_%d at 2^%d" % (j, L))

        # an impulse at bit-reversed position rev(k0), forward: the values w^(i k0)
        k0 = int(rng.integers(1, n)) if n > 2 else 1
        x.zero_()
        x[int(_rev([k0], L)[0])] = one[0]
        ntt.forward(L, x)
        _check(_ints(x, idx), w((pos * k0) % n), "forward of coefficient %d at 2^%d" % (k0, L))

        # (-1)^i: the single coefficient 1 at k = n/2 (held at position 1), then g^(n/2) (-1)^i
        x.view(n // 2, 8)[:, :4] = one[0]
        x.view(n // 2, 8)[:, 4:] = p1[0]
        ntt.inverse(L, x)
        gh = pow(qm.shift(L), n // 2, P)
        want = zero.copy()
        want[pos == 1] = gh
        _check(_ints(x, idx), want, "inverse of (-1)^i at 2^%d" % L)
        ntt.forward(L, x)
        want = np.full(len(pos), P - gh, dtype=object)
        want[pos % 2 == 0] = gh
        _check(_ints(x, idx), want, "(-1)^i round trip at 2^%d" % L)
    finally:
        del x
        torch.cuda.empty_cache()


# ---- dense random vectors above 2^16 -------------------------------------------------------------------------------------------
def _random_dev(n, gen):
    """n canonical entries with random limbs, the top limb below p's"""
    import torch
    x = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    x.random_(-2 ** 63, 2 ** 63 - 1, generator=gen)
    x[:, 3].random_(0, P >> 192, generator=gen)
    return x


def _points(rng, L):
    n = 1 << L
    pts = []
    while len(pts) < 2:
        r = rng.randrange(P)
        if pow(r, n, P) not in (1, pow(qm.shift(L), n, P)):
            pts.append(r)
    return pts


def _bary(t, shift, L, r):
    import torch
    import bary
    torch.cuda.synchronize()
    return bary.evaluate(t.data_ptr(), t.shape[0], shift, qm.root(L), L, r)


@pytest.mark.parametrize("L", range(EXACT_MAX + 1, qm.TWO_ADICITY + 1))
def test_random_round_trip(ntt, L):
    """forward(inverse(x)) holds the values of x's polynomial on the coset: the same polynomial at two random points"""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(3000 + L)
    x0 = _random_dev(1 << L, gen)
    x = x0.clone()
    try:
        ntt.inverse(L, x)
        ntt.forward(L, x)
        for r in _points(random.Random(L), L):
            assert _bary(x, qm.shift(L), L, r) == _bary(x0, 1, L, r), "2^%d at r = %d" % (L, r)
    finally:
        del x, x0
        torch.cuda.empty_cache()


@pytest.mark.parametrize("L", range(EXACT_MAX + 1, qm.TWO_ADICITY))
def test_random_quotient(ntt, L):
    """the quotient sequence equals y_A y_B - y_C of copies transformed one by one: every entry up to 2^22, sampled above"""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(4000 + L)
    a, b, c = (_random_dev(1 << L, gen) for _ in range(3))
    ys = [v.clone() for v in (a, b, c)]
    try:
        for y in ys:
            ntt.inverse(L, y)
            ntt.forward(L, y)
        ntt.quotient(L, a, b, c)
        idx = None
        if L > FULL_QUOTIENT_MAX:
            rng = np.random.default_rng(L)
            idx = np.unique(np.concatenate([rng.integers(0, 1 << L, 1 << 16, dtype=np.int64), _sample(ntt, L, rng)]))
        ya, yb, yc = (_ints(y, idx) for y in ys)
        _check(_ints(a, idx), (ya * yb - yc) % P, "quotient at 2^%d" % L)
    finally:
        del a, b, c, ys
        torch.cuda.empty_cache()
