"""Big-integer model of BN254 G1, written from the curve definition alone (y^2 = x^3 + 3 over F_q, generator (1, 2), prime order
r, cofactor 1): F_q and its Montgomery form, affine and Jacobian addition and doubling, scalar multiplication, a naive
multi-exponentiation, the 64-byte (x, y) encoding pob_msm_g1 reads and writes ((0, 0) = infinity), and the even/odd CIOS
Montgomery product of csrc/fr_hd.h for any modulus below 2^254.  None is used by the library."""
Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
R_ORDER = 21888242871839275222246405745257275088548364400416034343698204186575808495617
B = 3
G = (1, 2)
R = 1 << 256
M32 = (1 << 32) - 1
INF = None                                            # the point at infinity, affine


def to_mont(x):
    return x * R % Q


def from_mont(x):
    return x * pow(R, -1, Q) % Q


def on_curve(p):
    return p is INF or (p[1] * p[1] - p[0] ** 3 - B) % Q == 0


def neg(p):
    return INF if p is INF else (p[0], (-p[1]) % Q)


def add(p, q):
    """affine addition with every special case: O + P, P + P, P + (-P)"""
    if p is INF:
        return q
    if q is INF:
        return p
    (x1, y1), (x2, y2) = p, q
    if x1 == x2:
        if (y1 + y2) % Q == 0:
            return INF
        lam = 3 * x1 * x1 * pow(2 * y1, -1, Q) % Q
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, Q) % Q
    x3 = (lam * lam - x1 - x2) % Q
    return (x3, (lam * (x1 - x3) - y1) % Q)


def jac_dbl(p):
    """Jacobian (X, Y, Z), x = X / Z^2, y = Y / Z^3; Z = 0 is O (a = 0: dbl-2009-l)"""
    X, Y, Z = p
    if Z == 0 or Y == 0:
        return (1, 1, 0)
    A, Bq = X * X % Q, Y * Y % Q
    C = Bq * Bq % Q
    D = 2 * ((X + Bq) ** 2 - A - C) % Q
    E = 3 * A % Q
    X3 = (E * E - 2 * D) % Q
    return (X3, (E * (D - X3) - 8 * C) % Q, 2 * Y * Z % Q)


def jac_add(p, q):
    """Jacobian addition (add-2007-bl), falling back to doubling for P + P and to O for P + (-P)"""
    X1, Y1, Z1 = p
    X2, Y2, Z2 = q
    if Z1 == 0:
        return q
    if Z2 == 0:
        return p
    Z1Z1, Z2Z2 = Z1 * Z1 % Q, Z2 * Z2 % Q
    U1, U2 = X1 * Z2Z2 % Q, X2 * Z1Z1 % Q
    S1, S2 = Y1 * Z2 * Z2Z2 % Q, Y2 * Z1 * Z1Z1 % Q
    if U1 == U2:
        return jac_dbl(p) if S1 == S2 else (1, 1, 0)
    H, rr = (U2 - U1) % Q, 2 * (S2 - S1) % Q
    I = 4 * H * H % Q
    J, V = H * I % Q, U1 * I % Q
    X3 = (rr * rr - J - 2 * V) % Q
    return (X3, (rr * (V - X3) - 2 * S1 * J) % Q, ((Z1 + Z2) ** 2 - Z1Z1 - Z2Z2) * H % Q)


def to_jac(p):
    return (1, 1, 0) if p is INF else (p[0], p[1], 1)


def from_jac(p):
    X, Y, Z = p
    if Z == 0:
        return INF
    zi = pow(Z, -1, Q)
    return (X * zi * zi % Q, Y * zi ** 3 % Q)


def mul(k, p):
    """[k]P by double-and-add over Jacobian coordinates; any integer k (reduced mod r)"""
    k %= R_ORDER
    acc = (1, 1, 0)
    base = to_jac(p)
    for bit in bin(k)[2:] if k else "":
        acc = jac_dbl(acc)
        if bit == "1":
            acc = jac_add(acc, base)
    return from_jac(acc)


def msm(points, scalars):
    """naive sum_i [s_i] P_i with affine additions"""
    acc = INF
    for p, s in zip(points, scalars):
        acc = add(acc, mul(s, p))
    return acc


def encode_bases(points):
    """(n, 8) uint64 array: per point x then y as 32-byte LE Montgomery-form F_q elements, infinity as (0, 0)"""
    import numpy as np
    raw = b"".join((0).to_bytes(64, "little") if p is INF else to_mont(p[0]).to_bytes(32, "little") + to_mont(p[1]).to_bytes(32, "little")
                   for p in points)
    return np.frombuffer(raw, dtype=np.uint64).reshape(len(points), 8).copy()


def encode_scalars(values):
    import numpy as np
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in values), dtype=np.uint64).reshape(len(values), 4).copy()


def decode_point(limbs):
    """8 uint64 limbs (x canonical, then y) -> affine point, (0, 0) -> infinity"""
    v = [int(x) & ((1 << 64) - 1) for x in limbs]
    x, y = (sum(v[4 * k + i] << (64 * i) for i in range(4)) for k in (0, 1))
    return INF if x == 0 and y == 0 else (x, y)


class _Chain:                                         # a PTX carry chain (add.cc / addc.cc / mad.lo.cc / madc.hi.cc)
    def __init__(self):
        self.c = 0

    def add(self, x, y, cin):
        s = x + y + (self.c if cin else 0)
        self.c = s >> 32
        return s & M32


def _row(T, src, w, ch, first_cin):
    cin = first_cin
    for k in range(4):
        T[2 * k] = ch.add(T[2 * k], (src[k] * w) & M32, cin)
        cin = True
        T[2 * k + 1] = ch.add(T[2 * k + 1], (src[k] * w) >> 32, True)


def mont_limb_model(a, b, mod):
    """fr_hd.h's device mont_mul<M> (two accumulators E / O, one carry chain per row, the shift a renaming) for modulus `mod`,
    limb by limb, with its bounds asserted (no O row carries out, E needs 9 limbs, result < 2 mod).  Returns a b 2^-256 mod `mod`."""
    n0 = (-pow(mod, -1, 1 << 32)) % (1 << 32)
    pl = [(mod >> (32 * i)) & M32 for i in range(8)]
    al = [(a >> (32 * i)) & M32 for i in range(8)]
    bl = [(b >> (32 * i)) & M32 for i in range(8)]
    E, O, x = [0] * 9, [0] * 8, 0
    for i in range(8):
        ch = _Chain()
        E[0] = ch.add(E[0], x, False)
        _row(O, al[1::2], bl[i], ch, True)
        assert ch.c == 0
        ch = _Chain()
        _row(E, al[0::2], bl[i], ch, False)
        E[8] = ch.add(E[8], 0, True)
        m = (E[0] * n0) & M32
        ch = _Chain()
        _row(O, pl[1::2], m, ch, False)
        assert ch.c == 0
        ch = _Chain()
        _row(E, pl[0::2], m, ch, False)
        E[8] = ch.add(E[8], 0, True)
        assert ch.c == 0 and E[0] == 0
        x, E, O = E[1], O[:] + [0], E[2:9] + [0]
    ch = _Chain()
    r = [ch.add(E[0], x, False)] + [0] * 7
    for k in range(1, 8):
        r[k] = ch.add(E[k], O[k - 1], True)
    assert ch.c == 0 and O[7] == 0 and E[8] == 0
    v = sum(r[k] << (32 * k) for k in range(8))
    assert v < 2 * mod
    return v - mod if v >= mod else v
