// fq_hd.h -- BN254 base field F_q and G1 point arithmetic for the multi-exponentiation (msm.cuh, pob_msm_g1).
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

struct G1Aff { Fq x, y; };              // (0, 0) = O
struct G1Xyzz { Fq x, y, zz, zzz; };    // zz = 0: O

POB_HD G1Xyzz g1_inf() { G1Xyzz r; r.x = r.y = r.zz = r.zzz = fq_zero(); return r; }
POB_HD bool g1_is_inf(const G1Xyzz &p) { return fq_is_zero(p.zz); }
POB_HD bool g1_aff_is_inf(const G1Aff &a) { return fq_is_zero(a.x) && fq_is_zero(a.y); }
POB_HD G1Xyzz g1_from_aff(const G1Aff &a) {
    if (g1_aff_is_inf(a)) return g1_inf();
    G1Xyzz r; r.x = a.x; r.y = a.y; r.zz = r.zzz = fq_one(); return r;
}
POB_HD G1Aff g1_aff_neg(const G1Aff &a) { G1Aff r; r.x = a.x; r.y = fq_neg(a.y); return r; }

// [2]P, dbl-2008-s-1.  Y = 0 (not on the curve, or O) gives ZZ = 0, i.e. O.
POB_HD G1Xyzz g1_dbl(const G1Xyzz &p) {
    const Fq u = fq_add(p.y, p.y), v = fq_sqr(u), w = fq_mul(u, v), s = fq_mul(p.x, v);
    const Fq x2 = fq_sqr(p.x), m = fq_add(fq_add(x2, x2), x2);
    G1Xyzz r;
    r.x = fq_sub(fq_sub(fq_sqr(m), s), s);
    r.y = fq_sub(fq_mul(m, fq_sub(s, r.x)), fq_mul(w, p.y));
    r.zz = fq_mul(v, p.zz);
    r.zzz = fq_mul(w, p.zzz);
    return r;
}
// [2]A for an affine A != O, mdbl-2008-s-1
POB_HD G1Xyzz g1_dbl_aff(const G1Aff &a) {
    const Fq u = fq_add(a.y, a.y), v = fq_sqr(u), w = fq_mul(u, v), s = fq_mul(a.x, v);
    const Fq x2 = fq_sqr(a.x), m = fq_add(fq_add(x2, x2), x2);
    G1Xyzz r;
    r.x = fq_sub(fq_sub(fq_sqr(m), s), s);
    r.y = fq_sub(fq_mul(m, fq_sub(s, r.x)), fq_mul(w, a.y));
    r.zz = v;
    r.zzz = w;
    return r;
}
// P + A, madd-2008-s
POB_HD G1Xyzz g1_add_aff(const G1Xyzz &p, const G1Aff &a) {
    if (g1_aff_is_inf(a)) return p;
    if (g1_is_inf(p)) return g1_from_aff(a);
    const Fq pp_ = fq_sub(fq_mul(a.x, p.zz), p.x), rr = fq_sub(fq_mul(a.y, p.zzz), p.y);
    if (fq_is_zero(pp_)) return fq_is_zero(rr) ? g1_dbl_aff(a) : g1_inf();
    const Fq pp = fq_sqr(pp_), ppp = fq_mul(pp_, pp), q = fq_mul(p.x, pp);
    G1Xyzz r;
    r.x = fq_sub(fq_sub(fq_sub(fq_sqr(rr), ppp), q), q);
    r.y = fq_sub(fq_mul(rr, fq_sub(q, r.x)), fq_mul(p.y, ppp));
    r.zz = fq_mul(p.zz, pp);
    r.zzz = fq_mul(p.zzz, ppp);
    return r;
}
// P + Q, add-2008-s
POB_HD G1Xyzz g1_add(const G1Xyzz &p, const G1Xyzz &o) {
    if (g1_is_inf(o)) return p;
    if (g1_is_inf(p)) return o;
    const Fq u1 = fq_mul(p.x, o.zz), s1 = fq_mul(p.y, o.zzz);
    const Fq pp_ = fq_sub(fq_mul(o.x, p.zz), u1), rr = fq_sub(fq_mul(o.y, p.zzz), s1);
    if (fq_is_zero(pp_)) return fq_is_zero(rr) ? g1_dbl(p) : g1_inf();
    const Fq pp = fq_sqr(pp_), ppp = fq_mul(pp_, pp), q = fq_mul(u1, pp);
    G1Xyzz r;
    r.x = fq_sub(fq_sub(fq_sub(fq_sqr(rr), ppp), q), q);
    r.y = fq_sub(fq_mul(rr, fq_sub(q, r.x)), fq_mul(s1, ppp));
    r.zz = fq_mul(fq_mul(p.zz, o.zz), pp);
    r.zzz = fq_mul(fq_mul(p.zzz, o.zzz), ppp);
    return r;
}
// [k]P for k < 2^32, double-and-add from the top bit
POB_HD G1Xyzz g1_mul_u32(const G1Xyzz &p, uint32_t k) {
    G1Xyzz acc = g1_inf();
    for (int i = 31; i >= 0; i--) {
        if (!g1_is_inf(acc)) acc = g1_dbl(acc);
        if ((k >> i) & 1u) acc = g1_add(acc, p);
    }
    return acc;
}
// affine x, y in CANONICAL form (out of Montgomery form); O gives (0, 0).  One inversion: 1/Z = ZZ / ZZZ.
POB_HD G1Aff g1_to_affine_canonical(const G1Xyzz &p) {
    G1Aff a;
    if (g1_is_inf(p)) { a.x = a.y = fq_zero(); return a; }
    const Fq izzz = fq_inv(p.zzz), iz = fq_mul(p.zz, izzz);
    a.x = fq_from_mont(fq_mul(p.x, fq_sqr(iz)));
    a.y = fq_from_mont(fq_mul(p.y, izzz));
    return a;
}

}  // namespace pob
