"""Big-integer model of the BN254 optimal ate pairing, written from the definitions alone, for the tests of csrc/fq12_hd.h,
csrc/pairing.cuh and pob_groth16_verify.  None is used by the library.

Tower: F_q2 = F_q[u] / (u^2 + 1) (tests/g2_model.py), F_q6 = F_q2[v] / (v^3 - xi) with xi = 9 + u, F_q12 = F_q6[w] / (w^2 - v).  An
F_q6 element is a 3-tuple of F_q2 pairs, an F_q12 element a 2-tuple of F_q6 (c0 + c1 w).  As a check of the tower, every element
also has a flat form: 12 F_q coefficients of 1, w, .., w^11 modulo w^12 - 18 w^6 + 82 (w^6 = xi, so u = w^6 - 9).

Pairing: G2 points live on the twist y^2 = x^3 + 3 / xi; the untwisting map (x, y) -> (x w^2, y w^3) sends them to y^2 = x^3 + 3
over F_q12, where this model runs an AFFINE Miller loop (chord-and-tangent lines, a vertical line when a sum is O) over the plain
binary digits of 6x + 2, adds the lines at pi(Q) and -pi^2(Q) (pi the q-power Frobenius of the untwisted point), and raises the
product to (q^12 - 1) / r with pow.  The device uses projective coordinates on the twist, signed digits and a chain for the
exponent, so the two agree only in the final value, which is what the definition fixes."""
import random

import g1_model as gm
import g2_model as g2m

Q = gm.Q
R_ORDER = gm.R_ORDER
X = 4965661367192848881                                # the BN parameter: q = 36x^4 + 36x^3 + 24x^2 + 6x + 1
ATE = 6 * X + 2
FINAL_EXP = (Q ** 12 - 1) // R_ORDER
XI = (9, 1)

Z2, O2 = (0, 0), (1, 0)
add2, sub2, mul2, neg2, inv2 = g2m.add2, g2m.sub2, g2m.mul2, g2m.neg2, g2m.inv2


def conj2(a):
    return (a[0], (-a[1]) % Q)


# ---- F_q6 ---------------------------------------------------------------------------------------------------------------------
Z6, O6 = (Z2, Z2, Z2), (O2, Z2, Z2)


def add6(a, b):
    return tuple(add2(x, y) for x, y in zip(a, b))


def sub6(a, b):
    return tuple(sub2(x, y) for x, y in zip(a, b))


def neg6(a):
    return tuple(neg2(x) for x in a)


def mul6(a, b):
    """schoolbook, v^3 = xi"""
    c = [Z2] * 5
    for i in range(3):
        for j in range(3):
            c[i + j] = add2(c[i + j], mul2(a[i], b[j]))
    return (add2(c[0], mul2(XI, c[3])), add2(c[1], mul2(XI, c[4])), c[2])


def mul_v(a):
    """a v"""
    return (mul2(XI, a[2]), a[0], a[1])


def inv6(a):
    """by the norm to F_q2: 1 / a = a^q a^(q^2) / N(a), written out as the adjugate of multiplication by a"""
    a0, a1, a2 = a
    t0 = sub2(mul2(a0, a0), mul2(XI, mul2(a1, a2)))
    t1 = sub2(mul2(XI, mul2(a2, a2)), mul2(a0, a1))
    t2 = sub2(mul2(a1, a1), mul2(a0, a2))
    d = inv2(add2(mul2(a0, t0), mul2(XI, add2(mul2(a2, t1), mul2(a1, t2)))))
    return (mul2(t0, d), mul2(t1, d), mul2(t2, d))


# ---- F_q12 --------------------------------------------------------------------------------------------------------------------
ONE = (O6, Z6)
ZERO = (Z6, Z6)


def add12(a, b):
    return (add6(a[0], b[0]), add6(a[1], b[1]))


def sub12(a, b):
    return (sub6(a[0], b[0]), sub6(a[1], b[1]))


def mul12(a, b):
    """(a0 + a1 w)(b0 + b1 w) = a0 b0 + a1 b1 v + (a0 b1 + a1 b0) w"""
    return (add6(mul6(a[0], b[0]), mul_v(mul6(a[1], b[1]))), add6(mul6(a[0], b[1]), mul6(a[1], b[0])))


def sqr12(a):
    return mul12(a, a)


def conj12(a):
    """a^(q^6): w -> -w"""
    return (a[0], neg6(a[1]))


def inv12(a):
    """1 / (a0 + a1 w) = (a0 - a1 w) / (a0^2 - a1^2 v)"""
    d = inv6(sub6(mul6(a[0], a[0]), mul_v(mul6(a[1], a[1]))))
    return (mul6(a[0], d), neg6(mul6(a[1], d)))


def pow12(a, e):
    r = ONE
    for bit in bin(e)[2:] if e else "":
        r = sqr12(r)
        if bit == "1":
            r = mul12(r, a)
    return r


def from_fq(c):
    return (((c % Q, 0), Z2, Z2), Z6)


def from_fq2(c):
    return ((c, Z2, Z2), Z6)


W = (Z6, O6)                                            # w


def coeffs(a):
    """the 12 canonical F_q values in the order of the device's (and vk_alphabeta_12's) nesting: c0.c0.c0, c0.c0.c1, .., c1.c2.c1"""
    return tuple(v for h in a for e in h for v in e)


def from_coeffs(v):
    v = list(v)
    e = [(v[2 * k], v[2 * k + 1]) for k in range(6)]
    return ((e[0], e[1], e[2]), (e[3], e[4], e[5]))


# basis index k of w^k: c0.cj is w^(2j), c1.cj is w^(2j + 1)
def to_flat(a):
    """12 coefficients of 1, w, .., w^11 modulo w^12 - 18 w^6 + 82 (c0 + c1 u -> c0 - 9 c1 + c1 w^6)"""
    f = [0] * 12
    for half in range(2):
        for j in range(3):
            c0, c1 = a[half][j]
            k = 2 * j + half
            f[k] = (f[k] + c0 - 9 * c1) % Q
            f[k + 6] = (f[k + 6] + c1) % Q
    return f


def flat_mul(a, b):
    c = [0] * 23
    for i in range(12):
        for j in range(12):
            c[i + j] += a[i] * b[j]
    for k in range(22, 11, -1):                         # w^k = 18 w^(k-6) - 82 w^(k-12)
        c[k - 6] += 18 * c[k]
        c[k - 12] -= 82 * c[k]
    return [x % Q for x in c[:12]]


def frob(a, k=1):
    """a^(q^k) by pow: the definition the device's constants are checked against"""
    return pow12(a, Q ** k)


def frob_const(k, j):
    """gamma_{k,j} = xi^(j (q^k - 1) / 6): (c w^j)^(q^k) = c^(q^k) gamma_{k,j} w^j"""
    e = j * (Q ** k - 1) // 6
    r, b = O2, XI
    while e:
        if e & 1:
            r = mul2(r, b)
        b = mul2(b, b)
        e >>= 1
    return r


def random12(rng):
    return from_coeffs([rng.randrange(Q) for _ in range(12)])


# ---- points over F_q12 and the Miller loop ----------------------------------------------------------------------------------
def untwist(p):
    """twist point ((x0, x1), (y0, y1)) -> (x w^2, y w^3) on y^2 = x^3 + 3 over F_q12; None = O"""
    if p is None:
        return None
    x, y = p
    w2 = mul12(W, W)
    return (mul12(from_fq2(x), w2), mul12(from_fq2(y), mul12(w2, W)))


def _line(t, s, p):
    """the line through t and s (the tangent when t = s, the vertical when t = -s) at p = (x, y), and t + s; all affine over F_q12"""
    (x1, y1), (x2, y2) = t, s
    xp, yp = p
    if x1 == x2 and add12(y1, y2) == ZERO:
        return sub12(xp, x1), None
    if x1 == x2:
        lam = mul12(mul12(from_fq(3), sqr12(x1)), inv12(add12(y1, y1)))
    else:
        lam = mul12(sub12(y2, y1), inv12(sub12(x2, x1)))
    x3 = sub12(sub12(sqr12(lam), x1), x2)
    y3 = sub12(mul12(lam, sub12(x1, x3)), y1)
    return sub12(sub12(yp, y1), mul12(lam, sub12(xp, x1))), (x3, y3)


def miller(p, q_tw):
    """f_{6x+2,Q}(P) l_{[6x+2]Q, pi(Q)}(P) l_{[6x+2]Q + pi(Q), -pi^2(Q)}(P): P in G1 (affine ints), Q on the twist.  O on either side: 1"""
    if p is None or q_tw is None:
        return ONE
    pp = (from_fq(p[0]), from_fq(p[1]))
    qq = untwist(q_tw)
    f, t = ONE, qq
    for bit in bin(ATE)[3:]:
        l, t = _line(t, t, pp)
        f = mul12(sqr12(f), l)
        if bit == "1":
            l, t = _line(t, qq, pp)
            f = mul12(f, l)
    q1 = (frob(qq[0]), frob(qq[1]))
    q2 = (frob(q1[0]), neg12(frob(q1[1])))
    l, t = _line(t, q1, pp)
    f = mul12(f, l)
    l, _ = _line(t, q2, pp)
    return mul12(f, l)


def neg12(a):
    return (neg6(a[0]), neg6(a[1]))


def final_exp(f):
    return pow12(f, FINAL_EXP)


def pairing(p, q_tw):
    return final_exp(miller(p, q_tw))


def multi_pairing(pairs):
    f = ONE
    for p, q_tw in pairs:
        f = mul12(f, miller(p, q_tw))
    return final_exp(f)


# ---- Groth16 ------------------------------------------------------------------------------------------------------------------
def verify(vk, proof, publics):
    """e(-A, B) e(vk_x, gamma2) e(C, delta2) e(alpha1, beta2) == 1 with vk_x = IC_0 + sum_j pub_j IC_j.  vk: dict of model points
    alpha1, beta2, gamma2, delta2, ic (a list); proof: (A, B, C).  False for a public input >= r, as on-chain verifiers refuse it."""
    if any(not 0 <= s < R_ORDER for s in publics):
        return False
    a, b, c = proof
    vk_x = vk["ic"][0]
    for s, pt in zip(publics, vk["ic"][1:]):
        vk_x = gm.add(vk_x, gm.mul(s, pt))
    return multi_pairing([(gm.neg(a), b), (vk_x, vk["gamma2"]), (c, vk["delta2"]), (vk["alpha1"], vk["beta2"])]) == ONE


# ---- twist points outside G2 --------------------------------------------------------------------------------------------------
def sqrt2(a):
    """a square root in F_q2 (q = 3 mod 4), or None"""
    a1 = _pow2(a, (Q - 3) // 4)
    alpha = mul2(mul2(a1, a1), a)
    x0 = mul2(a1, a)
    if alpha == ((Q - 1), 0):
        x = mul2((0, 1), x0)
    else:
        x = mul2(_pow2(add2(O2, alpha), (Q - 1) // 2), x0)
    return x if mul2(x, x) == (a[0] % Q, a[1] % Q) else None


def _pow2(a, e):
    r = O2
    while e:
        if e & 1:
            r = mul2(r, a)
        a = mul2(a, a)
        e >>= 1
    return r


def twist_point_outside_g2(seed):
    """a point on the twist whose order is not r: a random x with x^3 + b' a square in F_q2 ([r]P != O is asserted)"""
    rng = random.Random(seed)
    while True:
        x = (rng.randrange(Q), rng.randrange(Q))
        y = sqrt2(add2(mul2(mul2(x, x), x), g2m.B2))
        if y is not None:
            p = (x, y)
            assert g2m.on_curve(p) and g2m.mul(R_ORDER, p, reduce=False) is not None
            return p
