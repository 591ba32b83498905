"""The Groth16 quotient evaluations (pob_b200.h: pob_r1cs_quotient, DESIGN.md §5) written from their definition with Python
integers and numpy object arrays, and nothing of the library.

p - 1 = 2^28 t; w28 = 5^t (5 is the smallest quadratic non-residue); w_k = w28^(2^(28-k)).  The domain of a system with m rows and
n_pub public signals is n = 2^log_n >= m + n_pub + 1 with omega = w_log_n; the coset shift is g = w_(log_n + 1) for log_n < 28 and 25
at log_n = 28.  q[i] = A^(g w^i) B^(g w^i) - C^(g w^i), where A^ interpolates the rows' A.w followed by the public rows (a = w[s]).
"""
import numpy as np

P = 21888242871839275222246405745257275088548364400416034343698204186575808495617
TWO_ADICITY = 28
NQR = 5
T = (P - 1) >> TWO_ADICITY
W28 = pow(NQR, T, P)


def root(k):
    """w_k, a primitive 2^k-th root of unity"""
    assert 0 <= k <= TWO_ADICITY
    return pow(W28, 1 << (TWO_ADICITY - k), P)


def shift(log_n):
    """the coset shift of a 2^log_n domain"""
    return root(log_n + 1) if log_n < TWO_ADICITY else NQR * NQR


def domain_log(m, n_pub):
    log_n = 0
    while (1 << log_n) < m + n_pub + 1:
        log_n += 1
    return log_n


def powers(x, n):
    """[1, x, ..., x^(n-1)] mod P as an object array, by doubling"""
    out = np.array([1], dtype=object)
    while len(out) < n:
        out = np.concatenate((out, out * pow(x, len(out), P) % P))
    return out[:n]


def _bitrev(n):
    bits = n.bit_length() - 1
    idx = np.arange(n)
    rev = np.zeros(n, dtype=np.int64)
    for b in range(bits):
        rev |= ((idx >> b) & 1) << (bits - 1 - b)
    return rev


def _dft(x, w):
    """sum_j x_j w^(ij) for every i (len(x) a power of two, w of that order): radix-2 decimation in time"""
    n = len(x)
    a = np.asarray(x, dtype=object)[_bitrev(n)]
    h = 1
    while h < n:
        tw = powers(pow(w, n // (2 * h), P), h)
        a = a.reshape(-1, 2 * h)
        u, v = a[:, :h], a[:, h:] * tw % P
        a = np.concatenate(((u + v) % P, (u - v) % P), axis=1)
        h *= 2
    return a.reshape(-1)


def ntt(coef):
    """values at w^i of the polynomial with these coefficients"""
    n = len(coef)
    return _dft(coef, root(n.bit_length() - 1))


def intt(vals):
    """coefficients of the polynomial of degree < n through (w^i, vals[i])"""
    n = len(vals)
    return _dft(vals, pow(root(n.bit_length() - 1), P - 2, P)) * pow(n, P - 2, P) % P


def rows(a, b, c, w_pub, m):
    """the three row vectors of length n: the m products, then the public rows (a = w[s]), then zeros"""
    n_pub = len(w_pub) - 1
    log_n = domain_log(m, n_pub)
    n = 1 << log_n
    out = []
    for v, pub in ((a, w_pub), (b, None), (c, None)):
        x = np.zeros(n, dtype=object)
        x[:m] = np.asarray(v, dtype=object)[:m] % P
        if pub is not None:
            x[m:m + len(pub)] = np.asarray(pub, dtype=object) % P
        out.append(x)
    return log_n, out


def quotient(a, b, c, w_pub, m):
    """q (object array of length n): a, b, c are the rows' A.w, B.w, C.w; w_pub = w[0 .. n_pub]"""
    log_n, vecs = rows(a, b, c, w_pub, m)
    n = 1 << log_n
    gk = powers(shift(log_n), n)
    A, B, C = (ntt(intt(v) * gk % P) for v in vecs)
    return (A * B - C) % P


def bary(values, shift_, log_n, r, first=0):
    """sum_i values[i] L_(first + i)(r): the polynomial of degree < n = 2^log_n that takes values[i] at shift_ w^(first + i) (and 0 at
    the points not given), evaluated at r, which is not one of the points.  L_i(r) = (r^n - s^n) x_i / (n s^n (r - x_i)) with
    x_i = s w^i; the sum of the fractions v_i x_i / (r - x_i) is folded pairwise and inverted once: O(len(values))."""
    n = 1 << log_n
    v = np.asarray(values, dtype=object) % P
    k = len(v)
    if k == 0:
        return 0
    x = powers(root(log_n), k) * (shift_ * pow(root(log_n), first, P) % P) % P
    num, den = v * x % P, (r - x) % P
    while len(num) > 1:
        if len(num) & 1:
            num, den = np.append(num, 0), np.append(den, 1)
        n0, n1, d0, d1 = num[0::2], num[1::2], den[0::2], den[1::2]
        num, den = (n0 * d1 + n1 * d0) % P, d0 * d1 % P
    sn = pow(shift_, n, P)
    return (pow(r, n, P) - sn) * num[0] % P * pow(n * sn % P * den[0] % P, P - 2, P) % P


def identity_holds(q, log_n, r, a_r, b_r, c_r):
    """h(r) (r^n - 1) == A^(r) B^(r) - C^(r), with h through q_i / (g^n - 1) on the coset"""
    n = 1 << log_n
    g = shift(log_n)
    h = bary(q, g, log_n, r) * pow(pow(g, n, P) - 1, P - 2, P) % P
    return h * (pow(r, n, P) - 1) % P == (a_r * b_r - c_r) % P
