// fq12_hd.h -- the pairing's extension tower over F_q2 (fq2_hd.h), for pairing.cuh (pob_bn254_pairing, pob_groth16_verify).
//
//   F_q6  = F_q2[v] / (v^3 - xi), xi = 9 + u        an element is c0 + c1 v + c2 v^2
//   F_q12 = F_q6[w] / (w^2 - v)                     an element is c0 + c1 w
// so w^6 = xi, and the F_q2 coefficient of w^k sits at c(k & 1).c(k >> 1).  That nesting, c0.c0.c0, c0.c0.c1, c0.c1.c0, ..,
// c1.c2.c1, is the order of snarkjs's vk_alphabeta_12 as far as known here.  Every F_q value is in Montgomery form.
//
// Products are Karatsuba at both levels (F_q6: 6 F_q2 products, F_q12: 3 F_q6 products); 1 / a goes down the tower to one fq_inv.
// The Frobenius maps use (c w^k)^(q^j) = c^(q^j) gamma_{j,k} w^k with gamma_{j,k} = xi^(k (q^j - 1) / 6): the literals below, each
// pinned by tests/pairing_model.py.  fq12_cyc_sqr is Granger-Scott's squaring, valid only in the cyclotomic subgroup (the values
// left by the easy part of the final exponentiation, f^((q^6 - 1)(q^2 + 1))).
//
// The F_q12 values are 384 bytes, so the heavy operations are out-of-line functions (__noinline__): one copy of each in the
// binary, operands passed through local memory.
#pragma once
#include "fq2_hd.h"

#define POB_DNI __device__ __noinline__
#define POB_DFI __device__ __forceinline__

namespace pob {

struct Fq6 { Fq2 c0, c1, c2; };
struct Fq12 { Fq6 c0, c1; };

// gamma_{j,k} for j = 1, 2, 3 and k = 1 .. 5: [j - 1][k - 1][c0 / c1][limb], Montgomery form
__constant__ uint32_t FQ12_FROB[3][5][2][8] = {
    {{{0x33144907u, 0xaf9ba696u, 0x87afb78au, 0xca6b1d73u, 0xf08a2087u, 0x11bded5eu, 0x1a1f3a7cu, 0x02f34d75u},
      {0x4c492d72u, 0xa222ae23u, 0x565de15bu, 0xd00f02a4u, 0x53dfc926u, 0xdc2ff3a2u, 0xb3899551u, 0x10a75716u}},
     {{0x4563ab30u, 0xb5773b10u, 0xa9aa6454u, 0x347f91c8u, 0x242e0991u, 0x7a007127u, 0x118214ecu, 0x1956bcd8u},
      {0xa0aa4757u, 0x6e849f1eu, 0x89f89141u, 0xaa1c7b6du, 0xfae0ca3au, 0xb6e713cdu, 0x4e82ebc3u, 0x26694fbbu}},
     {{0x2936b629u, 0xe4bbdd0cu, 0xe133bacbu, 0xbb30f162u, 0xf9645366u, 0x31a9d1b6u, 0xa500f8ddu, 0x253570beu},
      {0x5ffe77c7u, 0xa1d77ce4u, 0x7826d1dbu, 0x07affd11u, 0xbb7edc6bu, 0x6d16bd27u, 0x85defeccu, 0x2c872002u}},
     {{0x843abe92u, 0x7361d77fu, 0x273411fbu, 0xa5bb2bd3u, 0x4b3e2399u, 0x9c941f31u, 0xbb9fd3ecu, 0x15df9cddu},
      {0x4bd8c949u, 0x5dddfd15u, 0xa4445b60u, 0x62cb29a5u, 0x0c7dd2b9u, 0x37bc870au, 0x3171f0fdu, 0x24830a9du}},
     {{0x41690fe7u, 0xc970692fu, 0x27694b0bu, 0xe2403421u, 0x83c459e8u, 0x32bee66bu, 0x0ab08841u, 0x12aabcedu},
      {0x40aebfa9u, 0x0d485d23u, 0xab2fcc57u, 0x05193418u, 0x8a4910f5u, 0xd3b0a40bu, 0x35d2925au, 0x2f21ebb5u}}},
    {{{0x00fa1bf2u, 0xca8d8005u, 0x68b39769u, 0xf0c5d614u, 0xad0d4418u, 0x0e201271u, 0xbad856e6u, 0x04290f65u}, {0}},
     {{0x13e80b9cu, 0x3350c88eu, 0xdb5e56b9u, 0x7dce557cu, 0xb615564au, 0x6001b4b8u, 0x020217e0u, 0x2682e617u}, {0}},
     {{0x12edefaau, 0x68c34889u, 0x72aabf4fu, 0x8d087f68u, 0x09081231u, 0x51e1a247u, 0x4729c0fau, 0x2259d6b1u}, {0}},
     {{0xd782e155u, 0x71930c11u, 0xffbe3323u, 0xa6bb947cu, 0xd4741444u, 0xaa303344u, 0x26594943u, 0x2c3b3f0du}, {0}},
     {{0xc494f1abu, 0x08cfc388u, 0x8d1373d4u, 0x19b31514u, 0xcb6c0213u, 0x584e90fdu, 0xdf2f8849u, 0x09e1685bu}, {0}}},
    {{{0x4e46d97du, 0x36531618u, 0xd4c96d9fu, 0x0af7129eu, 0xca1009b5u, 0x659da72fu, 0x83a20d23u, 0x08116d89u},
      {0xc39c1939u, 0xb1df4af7u, 0x8a73bf7fu, 0x3d9f0287u, 0x8caf0ae0u, 0x9b222092u, 0xeff054a6u, 0x26684515u}},
     {{0x16ad6badu, 0xc9af22f7u, 0x4aa662b2u, 0xb311782au, 0xe248c7f4u, 0x19eeaf64u, 0xe3439f82u, 0x20273e77u},
      {0xf7ce93acu, 0xacc02860u, 0x7ba76b4cu, 0x3933d581u, 0x446c8467u, 0x69e6188bu, 0x4417cc55u, 0x0a46036du}},
     {{0xaf46471eu, 0x5764af0au, 0x873e0fc1u, 0xdc50792eu, 0x881d04f6u, 0x86a673ffu, 0x3c30a74cu, 0x0b2eddb4u},
      {0x787e8580u, 0x9a490f32u, 0xf04af8b1u, 0x8fd16d7fu, 0xc6027bf2u, 0x4b39888eu, 0x5b52a15du, 0x03dd2e70u}},
     {{0x7b6762dfu, 0x448a93a5u, 0x28fdeadfu, 0xbfd62df5u, 0x0e9bd47au, 0xd858f5d0u, 0x3476ec58u, 0x06b03d4du},
      {0xbcc936d1u, 0x2b19daf4u, 0x56f4299fu, 0xa1a54e7au, 0x5adeaef1u, 0xb533eee0u, 0x84dda0b2u, 0x170c812bu}},
     {{0x75cf559fu, 0xe0bc4b22u, 0xc154e60fu, 0xc238b945u, 0x929a7d5eu, 0x803982a5u, 0xf7e4a37eu, 0x15ce052du},
      {0xbf3799a7u, 0x2d28efbdu, 0x1ad60773u, 0x9b097e3cu, 0xaf4a535bu, 0x982d4113u, 0xe3056063u, 0x24e18991u}}}};

POB_DFI Fq2 fq12_frob_const(int j, int k) {
    Fq2 r;
    for (int i = 0; i < 8; i++) { r.c0.l[i] = FQ12_FROB[j - 1][k - 1][0][i]; r.c1.l[i] = FQ12_FROB[j - 1][k - 1][1][i]; }
    return r;
}

// ---- F_q6 ----------------------------------------------------------------------------------------------------------------------
POB_DFI Fq6 fq6_zero() { Fq6 r; r.c0 = r.c1 = r.c2 = fq2_zero(); return r; }
POB_DFI Fq6 fq6_one() { Fq6 r = fq6_zero(); r.c0 = fq2_one(); return r; }
POB_DFI bool fq6_is_zero(const Fq6 &a) { return fq2_is_zero(a.c0) && fq2_is_zero(a.c1) && fq2_is_zero(a.c2); }
POB_DFI Fq6 fq6_add(const Fq6 &a, const Fq6 &b) { Fq6 r; r.c0 = fq2_add(a.c0, b.c0); r.c1 = fq2_add(a.c1, b.c1); r.c2 = fq2_add(a.c2, b.c2); return r; }
POB_DFI Fq6 fq6_sub(const Fq6 &a, const Fq6 &b) { Fq6 r; r.c0 = fq2_sub(a.c0, b.c0); r.c1 = fq2_sub(a.c1, b.c1); r.c2 = fq2_sub(a.c2, b.c2); return r; }
POB_DFI Fq6 fq6_neg(const Fq6 &a) { Fq6 r; r.c0 = fq2_neg(a.c0); r.c1 = fq2_neg(a.c1); r.c2 = fq2_neg(a.c2); return r; }
POB_DFI Fq6 fq6_mul_v(const Fq6 &a) { Fq6 r; r.c0 = fq2_mul_xi(a.c2); r.c1 = a.c0; r.c2 = a.c1; return r; }     // a v

// Karatsuba: v_i = a_i b_i, c0 = v0 + xi ((a1 + a2)(b1 + b2) - v1 - v2), c1 = (a0 + a1)(b0 + b1) - v0 - v1 + xi v2,
// c2 = (a0 + a2)(b0 + b2) - v0 - v2 + v1
POB_DNI Fq6 fq6_mul(const Fq6 &a, const Fq6 &b) {
    const Fq2 v0 = fq2_mul(a.c0, b.c0), v1 = fq2_mul(a.c1, b.c1), v2 = fq2_mul(a.c2, b.c2);
    Fq6 r;
    r.c0 = fq2_add(v0, fq2_mul_xi(fq2_sub(fq2_sub(fq2_mul(fq2_add(a.c1, a.c2), fq2_add(b.c1, b.c2)), v1), v2)));
    r.c1 = fq2_add(fq2_sub(fq2_sub(fq2_mul(fq2_add(a.c0, a.c1), fq2_add(b.c0, b.c1)), v0), v1), fq2_mul_xi(v2));
    r.c2 = fq2_add(fq2_sub(fq2_sub(fq2_mul(fq2_add(a.c0, a.c2), fq2_add(b.c0, b.c2)), v0), v2), v1);
    return r;
}
POB_DFI Fq6 fq6_sqr(const Fq6 &a) { return fq6_mul(a, a); }
// a (b0 + b1 v): the sparse product of the line functions
POB_DNI Fq6 fq6_mul_01(const Fq6 &a, const Fq2 &b0, const Fq2 &b1) {
    const Fq2 v0 = fq2_mul(a.c0, b0), v1 = fq2_mul(a.c1, b1);
    Fq6 r;
    r.c0 = fq2_add(v0, fq2_mul_xi(fq2_mul(a.c2, b1)));
    r.c1 = fq2_sub(fq2_sub(fq2_mul(fq2_add(a.c0, a.c1), fq2_add(b0, b1)), v0), v1);
    r.c2 = fq2_add(fq2_mul(a.c2, b0), v1);
    return r;
}
POB_DFI Fq6 fq6_mul_fq2(const Fq6 &a, const Fq2 &b) { Fq6 r; r.c0 = fq2_mul(a.c0, b); r.c1 = fq2_mul(a.c1, b); r.c2 = fq2_mul(a.c2, b); return r; }
// 1 / a: the adjugate t over the norm d = a0 t0 + xi (a2 t1 + a1 t2) in F_q2; 0 gives 0
POB_DNI Fq6 fq6_inv(const Fq6 &a) {
    const Fq2 t0 = fq2_sub(fq2_sqr(a.c0), fq2_mul_xi(fq2_mul(a.c1, a.c2)));
    const Fq2 t1 = fq2_sub(fq2_mul_xi(fq2_sqr(a.c2)), fq2_mul(a.c0, a.c1));
    const Fq2 t2 = fq2_sub(fq2_sqr(a.c1), fq2_mul(a.c0, a.c2));
    const Fq2 d = fq2_inv(fq2_add(fq2_mul(a.c0, t0), fq2_mul_xi(fq2_add(fq2_mul(a.c2, t1), fq2_mul(a.c1, t2)))));
    Fq6 r; r.c0 = fq2_mul(t0, d); r.c1 = fq2_mul(t1, d); r.c2 = fq2_mul(t2, d);
    return r;
}

// ---- F_q12 ---------------------------------------------------------------------------------------------------------------------
POB_DFI Fq12 fq12_one() { Fq12 r; r.c0 = fq6_one(); r.c1 = fq6_zero(); return r; }
POB_DFI bool fq12_is_one(const Fq12 &a) {
    const Fq one = fq_one();
    bool ok = fq6_is_zero(a.c1) && fq_is_zero(a.c0.c0.c1) && fq2_is_zero(a.c0.c1) && fq2_is_zero(a.c0.c2);
    for (int i = 0; i < 8; i++) ok = ok && a.c0.c0.c0.l[i] == one.l[i];
    return ok;
}
POB_DFI Fq12 fq12_conj(const Fq12 &a) { Fq12 r; r.c0 = a.c0; r.c1 = fq6_neg(a.c1); return r; }     // a^(q^6)
// (a0 + a1 w)(b0 + b1 w) = a0 b0 + a1 b1 v + ((a0 + a1)(b0 + b1) - a0 b0 - a1 b1) w
POB_DNI Fq12 fq12_mul(const Fq12 &a, const Fq12 &b) {
    const Fq6 v0 = fq6_mul(a.c0, b.c0), v1 = fq6_mul(a.c1, b.c1);
    Fq12 r;
    r.c1 = fq6_sub(fq6_sub(fq6_mul(fq6_add(a.c0, a.c1), fq6_add(b.c0, b.c1)), v0), v1);
    r.c0 = fq6_add(v0, fq6_mul_v(v1));
    return r;
}
// (a0 + a1 w)^2 = (a0 + a1)(a0 + a1 v) - t - t v + 2 t w, t = a0 a1
POB_DNI Fq12 fq12_sqr(const Fq12 &a) {
    const Fq6 t = fq6_mul(a.c0, a.c1);
    Fq12 r;
    r.c0 = fq6_sub(fq6_sub(fq6_mul(fq6_add(a.c0, a.c1), fq6_add(a.c0, fq6_mul_v(a.c1))), t), fq6_mul_v(t));
    r.c1 = fq6_add(t, t);
    return r;
}
// 1 / (a0 + a1 w) = (a0 - a1 w) / (a0^2 - a1^2 v); 0 gives 0
POB_DNI Fq12 fq12_inv(const Fq12 &a) {
    const Fq6 d = fq6_inv(fq6_sub(fq6_sqr(a.c0), fq6_mul_v(fq6_sqr(a.c1))));
    Fq12 r; r.c0 = fq6_mul(a.c0, d); r.c1 = fq6_neg(fq6_mul(a.c1, d));
    return r;
}
// a^(q^j), j = 1, 2, 3: conjugate each coefficient when j is odd, then scale the coefficient of w^k by gamma_{j,k}
POB_DNI Fq12 fq12_frob(const Fq12 &a, int j) {
    Fq2 c[6] = {a.c0.c0, a.c1.c0, a.c0.c1, a.c1.c1, a.c0.c2, a.c1.c2};   // the coefficient of w^k
    for (int k = 0; k < 6; k++) {
        if (j & 1) c[k] = fq2_conj(c[k]);
        if (k) c[k] = fq2_mul(c[k], fq12_frob_const(j, k));
    }
    Fq12 r;
    r.c0.c0 = c[0]; r.c1.c0 = c[1]; r.c0.c1 = c[2]; r.c1.c1 = c[3]; r.c0.c2 = c[4]; r.c1.c2 = c[5];
    return r;
}
// a (c0 + c3 w + c4 v w), the line functions' shape (pairing.cuh): c0 in F_q2 at w^0, c3 at w^1, c4 at w^3
POB_DNI Fq12 fq12_mul_034(const Fq12 &a, const Fq2 &c0, const Fq2 &c3, const Fq2 &c4) {
    const Fq6 t0 = fq6_mul_fq2(a.c0, c0), t1 = fq6_mul_01(a.c1, c3, c4);
    Fq12 r;
    r.c1 = fq6_sub(fq6_sub(fq6_mul_01(fq6_add(a.c0, a.c1), fq2_add(c0, c3), c4), t0), t1);
    r.c0 = fq6_add(t0, fq6_mul_v(t1));
    return r;
}
// a^2 for a in the cyclotomic subgroup (a^(q^6 + 1)(q^2 + 1)-th powers, i.e. after the easy part): Granger-Scott, 9 F_q2 squares
POB_DNI Fq12 fq12_cyc_sqr(const Fq12 &x) {
    const Fq2 t0a = fq2_sqr(x.c1.c1), t1 = fq2_sqr(x.c0.c0);
    const Fq2 t6 = fq2_sub(fq2_sub(fq2_sqr(fq2_add(x.c1.c1, x.c0.c0)), t0a), t1);            // 2 x11 x00
    const Fq2 t2a = fq2_sqr(x.c0.c2), t3 = fq2_sqr(x.c1.c0);
    const Fq2 t7 = fq2_sub(fq2_sub(fq2_sqr(fq2_add(x.c0.c2, x.c1.c0)), t2a), t3);            // 2 x02 x10
    const Fq2 t4a = fq2_sqr(x.c1.c2), t5 = fq2_sqr(x.c0.c1);
    const Fq2 t8 = fq2_mul_xi(fq2_sub(fq2_sub(fq2_sqr(fq2_add(x.c1.c2, x.c0.c1)), t4a), t5));  // 2 x12 x01 xi
    const Fq2 t0 = fq2_add(fq2_mul_xi(t0a), t1), t2 = fq2_add(fq2_mul_xi(t2a), t3), t4 = fq2_add(fq2_mul_xi(t4a), t5);
    auto dbl = [](const Fq2 &a) { return fq2_add(a, a); };
    Fq12 z;
    z.c0.c0 = fq2_add(dbl(fq2_sub(t0, x.c0.c0)), t0);
    z.c0.c1 = fq2_add(dbl(fq2_sub(t2, x.c0.c1)), t2);
    z.c0.c2 = fq2_add(dbl(fq2_sub(t4, x.c0.c2)), t4);
    z.c1.c0 = fq2_add(dbl(fq2_add(t8, x.c1.c0)), t8);
    z.c1.c1 = fq2_add(dbl(fq2_add(t6, x.c1.c1)), t6);
    z.c1.c2 = fq2_add(dbl(fq2_add(t7, x.c1.c2)), t7);
    return z;
}

}  // namespace pob
