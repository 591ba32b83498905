// fq2_hd.h -- F_q2 = F_q[u] / (u^2 + 1) and BN254 G2 for the G2 multi-exponentiation (msm.cuh: pob_msm_g2) and the proof
// (pob_groth16_prove).
//
// An element is c0 + c1 u with c0, c1 in F_q, both in Montgomery form like Fq.  Products: Karatsuba (3 fq_mul), squares: the
// complex-squaring form (a0 + a1)(a0 - a1) + 2 a0 a1 u (2 fq_mul), 1 / (c0 + c1 u) = (c0 - c1 u) / (c0^2 + c1^2) (one fq_inv).
//
// G2: the sextic twist y^2 = x^3 + b' over F_q2, b' = 3 / (9 + u), with a subgroup of prime order r (its cofactor is not 1).  The
// point formulas of fq_hd.h are templates over the field; with the overloads below they are G2's.
#pragma once
#include "fq_hd.h"

namespace pob {

struct Fq2 { Fq c0, c1; };

POB_HD Fq2 fq2_zero() { Fq2 r; r.c0 = r.c1 = fq_zero(); return r; }
POB_HD Fq2 fq2_one() { Fq2 r; r.c0 = fq_one(); r.c1 = fq_zero(); return r; }
POB_HD bool fq2_is_zero(const Fq2 &a) { return fq_is_zero(a.c0) && fq_is_zero(a.c1); }
POB_HD Fq2 fq2_add(const Fq2 &a, const Fq2 &b) { Fq2 r; r.c0 = fq_add(a.c0, b.c0); r.c1 = fq_add(a.c1, b.c1); return r; }
POB_HD Fq2 fq2_sub(const Fq2 &a, const Fq2 &b) { Fq2 r; r.c0 = fq_sub(a.c0, b.c0); r.c1 = fq_sub(a.c1, b.c1); return r; }
POB_HD Fq2 fq2_neg(const Fq2 &a) { Fq2 r; r.c0 = fq_neg(a.c0); r.c1 = fq_neg(a.c1); return r; }
// (a0 + a1 u)(b0 + b1 u) = a0 b0 - a1 b1 + ((a0 + a1)(b0 + b1) - a0 b0 - a1 b1) u
POB_HD Fq2 fq2_mul(const Fq2 &a, const Fq2 &b) {
    const Fq v0 = fq_mul(a.c0, b.c0), v1 = fq_mul(a.c1, b.c1);
    Fq2 r;
    r.c0 = fq_sub(v0, v1);
    r.c1 = fq_sub(fq_sub(fq_mul(fq_add(a.c0, a.c1), fq_add(b.c0, b.c1)), v0), v1);
    return r;
}
POB_HD Fq2 fq2_sqr(const Fq2 &a) {
    const Fq t = fq_mul(a.c0, a.c1);
    Fq2 r;
    r.c0 = fq_mul(fq_add(a.c0, a.c1), fq_sub(a.c0, a.c1));
    r.c1 = fq_add(t, t);
    return r;
}
// 0 gives 0
POB_HD Fq2 fq2_inv(const Fq2 &a) {
    const Fq t = fq_inv(fq_add(fq_sqr(a.c0), fq_sqr(a.c1)));
    Fq2 r;
    r.c0 = fq_mul(a.c0, t);
    r.c1 = fq_neg(fq_mul(a.c1, t));
    return r;
}
POB_HD Fq2 fq2_to_mont(const Fq2 &a) { Fq2 r; r.c0 = fq_to_mont(a.c0); r.c1 = fq_to_mont(a.c1); return r; }
POB_HD Fq2 fq2_from_mont(const Fq2 &a) { Fq2 r; r.c0 = fq_from_mont(a.c0); r.c1 = fq_from_mont(a.c1); return r; }

// the field interface of the point formulas (fq_hd.h)
POB_HD Fq2 f_add(const Fq2 &a, const Fq2 &b) { return fq2_add(a, b); }
POB_HD Fq2 f_sub(const Fq2 &a, const Fq2 &b) { return fq2_sub(a, b); }
POB_HD Fq2 f_mul(const Fq2 &a, const Fq2 &b) { return fq2_mul(a, b); }
POB_HD Fq2 f_sqr(const Fq2 &a) { return fq2_sqr(a); }
POB_HD Fq2 f_neg(const Fq2 &a) { return fq2_neg(a); }
POB_HD Fq2 f_inv(const Fq2 &a) { return fq2_inv(a); }
POB_HD Fq2 f_to_mont(const Fq2 &a) { return fq2_to_mont(a); }
POB_HD Fq2 f_from_mont(const Fq2 &a) { return fq2_from_mont(a); }
POB_HD bool f_is_zero(const Fq2 &a) { return fq2_is_zero(a); }
POB_HD void f_set_zero(Fq2 &a) { a = fq2_zero(); }
POB_HD void f_set_one(Fq2 &a) { a = fq2_one(); }

// helpers of the pairing's tower (fq12_hd.h)
POB_HD Fq2 fq2_conj(const Fq2 &a) { Fq2 r; r.c0 = a.c0; r.c1 = fq_neg(a.c1); return r; }          // a^q, the Frobenius of F_q2
POB_HD Fq2 fq2_mul_fq(const Fq2 &a, const Fq &k) { Fq2 r; r.c0 = fq_mul(a.c0, k); r.c1 = fq_mul(a.c1, k); return r; }
// a xi with xi = 9 + u: (9 a0 - a1) + (9 a1 + a0) u, by additions
POB_HD Fq2 fq2_mul_xi(const Fq2 &a) {
    const Fq2 a2 = fq2_add(a, a), a4 = fq2_add(a2, a2), a8 = fq2_add(a4, a4), a9 = fq2_add(a8, a);
    Fq2 r; r.c0 = fq_sub(a9.c0, a.c1); r.c1 = fq_add(a9.c1, a.c0); return r;
}

typedef Aff<Fq2> G2Aff;      // 128 bytes: x.c0, x.c1, y.c0, y.c1
typedef Xyzz<Fq2> G2Xyzz;

}  // namespace pob
