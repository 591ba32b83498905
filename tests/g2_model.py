"""Big-integer model of BN254 G2, written from the definitions alone: F_q2 = F_q[u] / (u^2 + 1) with elements (c0, c1) = c0 + c1 u,
the twist y^2 = x^3 + b' with b' = 3 / (9 + u), its generator and its order-r subgroup; affine addition with every special case,
scalar multiplication, a naive multi-exponentiation, and the 128-byte (x.c0, x.c1, y.c0, y.c1) encoding pob_msm_g2 reads (Montgomery
form) and writes (canonical), all-zero = infinity.  Builds on tests/g1_model.py for F_q.  None is used by the library."""
import g1_model as gm

Q = gm.Q
R_ORDER = gm.R_ORDER
INF = None
ZERO, ONE = (0, 0), (1, 0)
B2 = (19485874751759354771024239261021720505790618469301721065564631296452457478373,
      266929791119991161246907387137283842545076965332900288569378510910307636690)
G = ((10857046999023057135944570762232829481370756359578518086990519993285655852781,
      11559732032986387107991004021392285783925812861821192530917403151452391805634),
     (8495653923123431417604973247489272438418190587263600148770280649306958101930,
      4082367875863433681332203403145435568316851327593401208105741076214120093531))


def add2(a, b):
    return ((a[0] + b[0]) % Q, (a[1] + b[1]) % Q)


def sub2(a, b):
    return ((a[0] - b[0]) % Q, (a[1] - b[1]) % Q)


def neg2(a):
    return ((-a[0]) % Q, (-a[1]) % Q)


def mul2(a, b):
    """schoolbook: (a0 + a1 u)(b0 + b1 u) = a0 b0 - a1 b1 + (a0 b1 + a1 b0) u"""
    return ((a[0] * b[0] - a[1] * b[1]) % Q, (a[0] * b[1] + a[1] * b[0]) % Q)


def inv2(a):
    """1 / (c0 + c1 u) = (c0 - c1 u) / (c0^2 + c1^2)"""
    t = pow((a[0] * a[0] + a[1] * a[1]) % Q, -1, Q)
    return (a[0] * t % Q, (-a[1]) * t % Q)


def scale2(a, k):
    return (a[0] * k % Q, a[1] * k % Q)


def on_curve(p):
    if p is INF:
        return True
    x, y = p
    return sub2(mul2(y, y), add2(mul2(mul2(x, x), x), B2)) == ZERO


def neg(p):
    return INF if p is INF else (p[0], neg2(p[1]))


def add(p, q):
    """affine addition with every special case: O + P, P + P, P + (-P)"""
    if p is INF:
        return q
    if q is INF:
        return p
    (x1, y1), (x2, y2) = p, q
    if x1 == x2:
        if add2(y1, y2) == ZERO:
            return INF
        lam = mul2(scale2(mul2(x1, x1), 3), inv2(scale2(y1, 2)))
    else:
        lam = mul2(sub2(y2, y1), inv2(sub2(x2, x1)))
    x3 = sub2(sub2(mul2(lam, lam), x1), x2)
    return (x3, sub2(mul2(lam, sub2(x1, x3)), y1))


def mul(k, p, reduce=True):
    """[k]P by double-and-add; k is taken mod r unless reduce=False (for the order check [r]G = O)"""
    if reduce:
        k %= R_ORDER
    acc = INF
    for bit in bin(k)[2:] if k else "":
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, p)
    return acc


def msm(points, scalars):
    acc = INF
    for p, s in zip(points, scalars):
        acc = add(acc, mul(s, p))
    return acc


def _enc(v, mont):
    return (gm.to_mont(v) if mont else v).to_bytes(32, "little")


def encode_points(points, mont=True):
    """(n, 16) uint64 array: per point x.c0, x.c1, y.c0, y.c1 as 32-byte LE F_q elements (Montgomery form unless mont=False),
    infinity all-zero"""
    import numpy as np
    raw = b"".join((0).to_bytes(128, "little") if p is INF else
                   b"".join(_enc(v, mont) for v in (p[0][0], p[0][1], p[1][0], p[1][1])) for p in points)
    return np.frombuffer(raw, dtype=np.uint64).reshape(len(points), 16).copy()


def decode_point(limbs):
    """16 uint64 limbs (canonical x.c0, x.c1, y.c0, y.c1) -> affine point, all-zero -> infinity"""
    v = [int(x) & ((1 << 64) - 1) for x in limbs]
    c = [sum(v[4 * k + i] << (64 * i) for i in range(4)) for k in range(4)]
    return INF if not any(c) else ((c[0], c[1]), (c[2], c[3]))
