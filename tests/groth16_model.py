"""A test-only Groth16 trusted setup whose trapdoor the tests know, written from the definitions with Python integers and numpy object
arrays, and nothing of the library.

Circuit: an iden3 `.r1cs` (tests/r1cs_reader.py) with m rows, n_pub public signals and the quotient's domain n = 2^log_n
(tests/quotient_model.py).  The rows' A, B, C are interpolated on the domain, followed by the public rows m + s (s = 0 .. n_pub) with
a = w[s], as pob_r1cs_quotient does, so wire i has the polynomials u_i, v_i, w_i with

    u_i(x) = sum_rows A[row][i] L_row(x) + [i <= n_pub] L_(m + i)(x),   v_i, w_i likewise from B and C (no public rows),

L_k the Lagrange basis of the domain.  From the toxic waste (tau, alpha, beta, gamma, delta) the key's discrete logarithms are

    alpha1 = alpha, beta1 = beta2 = beta, delta1 = delta2 = delta, A_i = u_i(tau), B1_i = B2_i = v_i(tau),
    C_i = (beta u_i(tau) + alpha v_i(tau) + w_i(tau)) / delta for i > n_pub,
    H_k = L^coset_k(tau) (tau^n - 1) / ((g^n - 1) delta),

L^coset_k the Lagrange basis of the coset g w^k.  Then sum_k q_k H_k = h(tau) z(tau) / delta for the library's q, since
q_k / (g^n - 1) = h(g w^k) (quotient_model.identity_holds).  A proof with blinding r, s has the discrete logarithms

    a = alpha + sum_i w_i u_i + r delta,  b = beta + sum_i w_i v_i + s delta,
    c = sum_{i > n_pub} w_i C_i + sum_k q_k H_k + s a + r b - r s delta,

and, by bilinearity, the pairing check e(A, B) = e(alpha, beta) e(IC, gamma) e(C, delta) is exactly the equation in Fr

    a b = alpha beta + sum_{i <= n_pub} w_i (beta u_i + alpha v_i + w_i)(tau) + c delta       (verify)

so no pairing code is needed.  gamma cancels from it (the IC points are that sum over gamma, times gamma)."""
import numpy as np

import quotient_model as qm

P = qm.P


def batch_inverse(vals):
    """1 / v for every v (none zero) with one modular inversion"""
    n = len(vals)
    pre = [1] * (n + 1)
    for i, v in enumerate(vals):
        pre[i + 1] = pre[i] * int(v) % P
    inv = pow(pre[n], P - 2, P)
    out = [0] * n
    for i in range(n - 1, -1, -1):
        out[i] = inv * pre[i] % P
        inv = inv * int(vals[i]) % P
    return np.array(out, dtype=object)


def lagrange_at(shift_, log_n, x):
    """L_k(x) for k = 0 .. n - 1, the Lagrange basis of the points shift_ w^k, at x (not one of them):
    L_k(x) = (x^n - s^n) x_k / (n s^n (x - x_k))"""
    n = 1 << log_n
    xs = qm.powers(qm.root(log_n), n) * shift_ % P
    sn = pow(shift_, n, P)
    scale = (pow(x, n, P) - sn) * pow(n * sn % P, P - 2, P) % P
    return xs * batch_inverse((x - xs) % P) % P * scale % P


def _scatter(n, idx, vals):
    """out[j] = sum of vals[t] with idx[t] = j"""
    out = np.zeros(n, dtype=object)
    if len(idx) == 0:
        return out
    order = np.argsort(idx, kind="stable")
    idx_s, v_s = idx[order], vals[order]
    uniq, starts = np.unique(idx_s, return_index=True)
    out[uniq] = np.add.reduceat(v_s, starts) % P
    return out


class Setup:
    """the trapdoor key of a `.r1cs` (an R1cs) for toxic waste (tau, alpha, beta, gamma, delta), as discrete logarithms"""

    def __init__(self, R, tau, alpha, beta, gamma, delta):
        self.R = R
        self.tau, self.alpha, self.beta, self.gamma, self.delta = tau, alpha, beta, gamma, delta
        self.m, self.n_pub, self.n_vars = R.m, R.n_pub_out + R.n_pub_in, R.n_wires
        self.log_n = qm.domain_log(self.m, self.n_pub)
        n = self.n = 1 << self.log_n
        L = lagrange_at(1, self.log_n, tau)
        row, which = R.term_lc // 3, R.term_lc % 3
        uvw = []
        for j in range(3):
            sel = which == j
            uvw.append(_scatter(self.n_vars, R.wire[sel], R.coef[sel] * L[row[sel]]))
        u, v, w = uvw
        u[:self.n_pub + 1] = (u[:self.n_pub + 1] + L[self.m:self.m + self.n_pub + 1]) % P
        self.u, self.v, self.w = u, v, w
        di = pow(delta, P - 2, P)
        self.ic = (beta * u + alpha * v + w) % P                       # beta u_i + alpha v_i + w_i
        self.a_keys, self.b_keys = u, v
        self.c_keys = self.ic[self.n_pub + 1:] * di % P
        g = qm.shift(self.log_n)
        zt = (pow(tau, n, P) - 1) % P
        self.h_keys = lagrange_at(g, self.log_n, tau) * (zt * pow((pow(g, n, P) - 1) * delta % P, P - 2, P) % P) % P

    def proof_scalars(self, W, q, r, s):
        """(a, b, c) of the proof of witness W (ints per wire) with quotient q (n ints) and blinding r, s"""
        W = np.asarray(W, dtype=object) % P
        q = np.asarray(q, dtype=object) % P
        r, s = r % P, s % P
        a = (self.alpha + int((W * self.u % P).sum()) + r * self.delta) % P
        b = (self.beta + int((W * self.v % P).sum()) + s * self.delta) % P
        c = (int((W[self.n_pub + 1:] * self.c_keys % P).sum()) + int((q * self.h_keys % P).sum()) + s * a + r * b - r * s % P * self.delta) % P
        return a, b, c

    def verify(self, a, b, c, w_pub):
        """the Groth16 equation in Fr over the discrete logarithms: w_pub = w[0 .. n_pub]"""
        pub = int((np.asarray(w_pub, dtype=object) % P * self.ic[:self.n_pub + 1] % P).sum())
        return a * b % P == (self.alpha * self.beta + pub + c * self.delta) % P
