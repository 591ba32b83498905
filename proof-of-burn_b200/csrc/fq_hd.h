// fq_hd.h -- BN254 base field F_q, and the point arithmetic of the multi-exponentiations (msm.cuh: pob_msm_g1, pob_msm_g2).
//
// F_q reuses the modulus-parameterised operations of fr_hd.h (mod_add, mod_sub, mont_mul: the even/odd CIOS product on the
// device), instantiated with q = 0x30644e72...fd47 < 2^254.  Elements stay in Montgomery form (x R mod q, R = 2^256) throughout;
// only the final affine conversion leaves it.
//
// G1: y^2 = x^3 + 3 over F_q, prime order r (= the Fr modulus), cofactor 1, so no point but O has y = 0.  Points in flight are
// XYZZ ("extended Jacobian") coordinates: (X, Y, ZZ, ZZZ) stands for x = X / ZZ, y = Y / ZZZ with ZZ^3 = ZZZ^2; ZZ = 0 is O.
// Affine inputs use (0, 0) for O (it is not on the curve).  Formulas: Bernstein-Lange's explicit-formulas database, g1p/xyzz
// (a = 0): mixed addition madd-2008-s (8 M + 2 S), addition add-2008-s (12 M + 2 S), doubling dbl-2008-s-1 (6 M + 3 S) and its
// affine form mdbl-2008-s-1 (4 M + 3 S).  Each addition handles P + P (it doubles), P + (-P) (O) and O on either side itself.
// The formulas never use b, so they are templates over the field (F_q for G1, F_q2 for G2, fq2_hd.h); g1_* name the F_q ones.
#pragma once
#include "fr_hd.h"

namespace pob {

struct Fq { uint32_t l[8]; };          // little-endian 32-bit limbs, Montgomery form unless a function says otherwise

struct FqMod {
    static POB_HD uint32_t limb(int i) {
        constexpr uint32_t Q[8] = {0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return Q[i];
    }
    static constexpr uint32_t n0 = 0xe4866389u;                       // -q^-1 mod 2^32
};
POB_HD uint32_t fq_r2_limb(int i) {                                    // R^2 mod q
    constexpr uint32_t R2[8] = {0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u, 0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u};
    return R2[i];
}
POB_HD uint32_t fq_one_limb(int i) {                                   // R mod q: 1 in Montgomery form
    constexpr uint32_t ONE[8] = {0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
    return ONE[i];
}

POB_HD Fq fq_zero() { Fq r; for (int i = 0; i < 8; i++) r.l[i] = 0; return r; }
POB_HD Fq fq_one() { Fq r; for (int i = 0; i < 8; i++) r.l[i] = fq_one_limb(i); return r; }
POB_HD bool fq_is_zero(const Fq &a) { uint32_t o = 0; for (int i = 0; i < 8; i++) o |= a.l[i]; return o == 0; }
POB_HD Fq fq_add(const Fq &a, const Fq &b) { return mod_add<FqMod>(a, b); }
POB_HD Fq fq_sub(const Fq &a, const Fq &b) { return mod_sub<FqMod>(a, b); }
POB_HD Fq fq_mul(const Fq &a, const Fq &b) { return mont_mul<FqMod>(a, b); }          // Montgomery product a b / R
POB_HD Fq fq_sqr(const Fq &a) { return mont_mul<FqMod>(a, a); }
POB_HD Fq fq_neg(const Fq &a) { return mod_sub<FqMod>(fq_zero(), a); }
POB_HD Fq fq_to_mont(const Fq &a) { Fq r2; for (int i = 0; i < 8; i++) r2.l[i] = fq_r2_limb(i); return fq_mul(a, r2); }
POB_HD Fq fq_from_mont(const Fq &a) { Fq one = fq_zero(); one.l[0] = 1; return fq_mul(a, one); }
// a^-1 (Montgomery form in and out) by Fermat, a^(q-2): one per multi-exponentiation, so the ladder's 254 squarings do not matter.
// a = 0 gives 0.
POB_HD Fq fq_inv(const Fq &a) {
    Fq e = mod_value<FqMod, Fq>(); e.l[0] -= 2;                       // q - 2 (q's lowest limb is > 2)
    Fq r = fq_one();
    for (int i = 253; i >= 0; i--) {
        r = fq_sqr(r);
        if ((e.l[i >> 5] >> (i & 31)) & 1u) r = fq_mul(r, a);
    }
    return r;
}

// the field interface of the point formulas below, which are written once for any F with these overloads: F_q here, F_q2 in
// fq2_hd.h (the G2 twist has a = 0 too, and no formula uses b)
POB_HD Fq f_add(const Fq &a, const Fq &b) { return fq_add(a, b); }
POB_HD Fq f_sub(const Fq &a, const Fq &b) { return fq_sub(a, b); }
POB_HD Fq f_mul(const Fq &a, const Fq &b) { return fq_mul(a, b); }
POB_HD Fq f_sqr(const Fq &a) { return fq_sqr(a); }
POB_HD Fq f_neg(const Fq &a) { return fq_neg(a); }
POB_HD Fq f_inv(const Fq &a) { return fq_inv(a); }
POB_HD Fq f_to_mont(const Fq &a) { return fq_to_mont(a); }
POB_HD Fq f_from_mont(const Fq &a) { return fq_from_mont(a); }
POB_HD bool f_is_zero(const Fq &a) { return fq_is_zero(a); }
POB_HD void f_set_zero(Fq &a) { a = fq_zero(); }
POB_HD void f_set_one(Fq &a) { a = fq_one(); }

template <class F> struct Aff { F x, y; };              // (0, 0) = O
template <class F> struct Xyzz { F x, y, zz, zzz; };    // zz = 0: O
typedef Aff<Fq> G1Aff;
typedef Xyzz<Fq> G1Xyzz;

template <class F> POB_HD Xyzz<F> pt_inf() { Xyzz<F> r; f_set_zero(r.x); r.y = r.zz = r.zzz = r.x; return r; }
template <class F> POB_HD bool pt_is_inf(const Xyzz<F> &p) { return f_is_zero(p.zz); }
template <class F> POB_HD bool pt_aff_is_inf(const Aff<F> &a) { return f_is_zero(a.x) && f_is_zero(a.y); }
template <class F> POB_HD Xyzz<F> pt_from_aff(const Aff<F> &a) {
    if (pt_aff_is_inf(a)) return pt_inf<F>();
    Xyzz<F> r; r.x = a.x; r.y = a.y; f_set_one(r.zz); r.zzz = r.zz; return r;
}
template <class F> POB_HD Aff<F> pt_aff_neg(const Aff<F> &a) { Aff<F> r; r.x = a.x; r.y = f_neg(a.y); return r; }

// [2]P, dbl-2008-s-1.  Y = 0 (not on the curve, or O) gives ZZ = 0, i.e. O.
template <class F> POB_HD Xyzz<F> pt_dbl(const Xyzz<F> &p) {
    const F u = f_add(p.y, p.y), v = f_sqr(u), w = f_mul(u, v), s = f_mul(p.x, v);
    const F x2 = f_sqr(p.x), m = f_add(f_add(x2, x2), x2);
    Xyzz<F> r;
    r.x = f_sub(f_sub(f_sqr(m), s), s);
    r.y = f_sub(f_mul(m, f_sub(s, r.x)), f_mul(w, p.y));
    r.zz = f_mul(v, p.zz);
    r.zzz = f_mul(w, p.zzz);
    return r;
}
// [2]A for an affine A != O, mdbl-2008-s-1
template <class F> POB_HD Xyzz<F> pt_dbl_aff(const Aff<F> &a) {
    const F u = f_add(a.y, a.y), v = f_sqr(u), w = f_mul(u, v), s = f_mul(a.x, v);
    const F x2 = f_sqr(a.x), m = f_add(f_add(x2, x2), x2);
    Xyzz<F> r;
    r.x = f_sub(f_sub(f_sqr(m), s), s);
    r.y = f_sub(f_mul(m, f_sub(s, r.x)), f_mul(w, a.y));
    r.zz = v;
    r.zzz = w;
    return r;
}
// P + A, madd-2008-s
template <class F> POB_HD Xyzz<F> pt_add_aff(const Xyzz<F> &p, const Aff<F> &a) {
    if (pt_aff_is_inf(a)) return p;
    if (pt_is_inf(p)) return pt_from_aff(a);
    const F pp_ = f_sub(f_mul(a.x, p.zz), p.x), rr = f_sub(f_mul(a.y, p.zzz), p.y);
    if (f_is_zero(pp_)) return f_is_zero(rr) ? pt_dbl_aff(a) : pt_inf<F>();
    const F pp = f_sqr(pp_), ppp = f_mul(pp_, pp), q = f_mul(p.x, pp);
    Xyzz<F> r;
    r.x = f_sub(f_sub(f_sub(f_sqr(rr), ppp), q), q);
    r.y = f_sub(f_mul(rr, f_sub(q, r.x)), f_mul(p.y, ppp));
    r.zz = f_mul(p.zz, pp);
    r.zzz = f_mul(p.zzz, ppp);
    return r;
}
// P + Q, add-2008-s
template <class F> POB_HD Xyzz<F> pt_add(const Xyzz<F> &p, const Xyzz<F> &o) {
    if (pt_is_inf(o)) return p;
    if (pt_is_inf(p)) return o;
    const F u1 = f_mul(p.x, o.zz), s1 = f_mul(p.y, o.zzz);
    const F pp_ = f_sub(f_mul(o.x, p.zz), u1), rr = f_sub(f_mul(o.y, p.zzz), s1);
    if (f_is_zero(pp_)) return f_is_zero(rr) ? pt_dbl(p) : pt_inf<F>();
    const F pp = f_sqr(pp_), ppp = f_mul(pp_, pp), q = f_mul(u1, pp);
    Xyzz<F> r;
    r.x = f_sub(f_sub(f_sub(f_sqr(rr), ppp), q), q);
    r.y = f_sub(f_mul(rr, f_sub(q, r.x)), f_mul(s1, ppp));
    r.zz = f_mul(f_mul(p.zz, o.zz), pp);
    r.zzz = f_mul(f_mul(p.zzz, o.zzz), ppp);
    return r;
}
// [k]P for k < 2^32, double-and-add from the top bit
template <class F> POB_HD Xyzz<F> pt_mul_u32(const Xyzz<F> &p, uint32_t k) {
    Xyzz<F> acc = pt_inf<F>();
    for (int i = 31; i >= 0; i--) {
        if (!pt_is_inf(acc)) acc = pt_dbl(acc);
        if ((k >> i) & 1u) acc = pt_add(acc, p);
    }
    return acc;
}
// [k]P for a 256-bit k (8 LE 32-bit limbs), double-and-add from the top bit: the proof's blinding terms and the test probe's keys
template <class F> POB_HD Xyzz<F> pt_mul_u256(const Xyzz<F> &p, const uint32_t *k) {
    Xyzz<F> acc = pt_inf<F>();
    for (int i = 255; i >= 0; i--) {
        if (!pt_is_inf(acc)) acc = pt_dbl(acc);
        if ((k[i >> 5] >> (i & 31)) & 1u) acc = pt_add(acc, p);
    }
    return acc;
}
// affine x, y in CANONICAL form (out of Montgomery form); O gives (0, 0).  One inversion: 1/Z = ZZ / ZZZ.
template <class F> POB_HD Aff<F> pt_to_affine_canonical(const Xyzz<F> &p) {
    Aff<F> a;
    if (pt_is_inf(p)) { f_set_zero(a.x); a.y = a.x; return a; }
    const F izzz = f_inv(p.zzz), iz = f_mul(p.zz, izzz);
    a.x = f_from_mont(f_mul(p.x, f_sqr(iz)));
    a.y = f_from_mont(f_mul(p.y, izzz));
    return a;
}

// the G1 names of the formulas
POB_HD G1Xyzz g1_inf() { return pt_inf<Fq>(); }
POB_HD bool g1_is_inf(const G1Xyzz &p) { return pt_is_inf(p); }
POB_HD bool g1_aff_is_inf(const G1Aff &a) { return pt_aff_is_inf(a); }
POB_HD G1Xyzz g1_from_aff(const G1Aff &a) { return pt_from_aff(a); }
POB_HD G1Aff g1_aff_neg(const G1Aff &a) { return pt_aff_neg(a); }
POB_HD G1Xyzz g1_dbl(const G1Xyzz &p) { return pt_dbl(p); }
POB_HD G1Xyzz g1_dbl_aff(const G1Aff &a) { return pt_dbl_aff(a); }
POB_HD G1Xyzz g1_add_aff(const G1Xyzz &p, const G1Aff &a) { return pt_add_aff(p, a); }
POB_HD G1Xyzz g1_add(const G1Xyzz &p, const G1Xyzz &o) { return pt_add(p, o); }
POB_HD G1Xyzz g1_mul_u32(const G1Xyzz &p, uint32_t k) { return pt_mul_u32(p, k); }
POB_HD G1Aff g1_to_affine_canonical(const G1Xyzz &p) { return pt_to_affine_canonical(p); }

}  // namespace pob
