// fr_hd.h -- BN254-Fr arithmetic for the witness VM: 8 x 32-bit limbs, column-wise Montgomery multiply.
//
// Every signal of the proof-of-burn circuits is an element of this field (reference: the implicit field
// ops under every `<==` -- circomlib/circuits/gates.circom:26,34,42, comparators.circom:30-33,
// poseidon.circom:12-15; prime in tests/poseidon.py:1-3).  The reference's own implementation is the
// fr.asm/fr.cpp the circom toolchain emits (not in the tree); this is an independent implementation.
//
// The functions are __host__ __device__ on purpose: the device build is the product; the host build is
// used only by the compile-time constant folder of the layout compiler and by the test-only emulator
// under tests/emu/ that lets the VM programs be checked against the oracle on a machine without a GPU.
// Device code uses 32-bit limbs with 64-bit accumulators (IMAD.WIDE on sm_90a).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define POB_HD __host__ __device__ __forceinline__
#else
#define POB_HD inline
#endif

namespace pob {

struct Fr { uint32_t l[8]; };   // canonical value in [0,p), little-endian limbs == 32-byte .wtns entry

#define POB_P_LIMBS {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u}
// R^2 mod p with R = 2^256 (Montgomery conversion factor)
#define POB_R2_LIMBS {0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u, 0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u}
#define POB_N0 0xefffffffu      // -p^-1 mod 2^32

POB_HD uint32_t fr_p_limb(int i) {
    constexpr uint32_t P[8] = POB_P_LIMBS;
    return P[i];
}
POB_HD uint32_t fr_r2_limb(int i) {
    constexpr uint32_t R2[8] = POB_R2_LIMBS;
    return R2[i];
}

// The modulus-dependent operations below (geq_mod, mod_add, mod_sub, mont_mul) are templates over a modulus M -- M::limb(i), its
// 32-bit limbs, and M::n0 = -M^-1 mod 2^32 -- and an element type T of eight 32-bit limbs `l`.  Their bounds hold for any odd
// modulus below 2^254.  Fr is the instance FrMod; fq_hd.h adds F_q, the base field of BN254 G1 (the multi-exponentiation).
struct FrMod {
    static POB_HD uint32_t limb(int i) { return fr_p_limb(i); }
    static constexpr uint32_t n0 = POB_N0;
};

POB_HD Fr fr_zero() { Fr r; for (int i = 0; i < 8; i++) r.l[i] = 0; return r; }
POB_HD Fr fr_from_u64(uint64_t v) { Fr r = fr_zero(); r.l[0] = (uint32_t)v; r.l[1] = (uint32_t)(v >> 32); return r; }
POB_HD bool fr_is_zero(const Fr &a) { uint32_t o = 0; for (int i = 0; i < 8; i++) o |= a.l[i]; return o == 0; }
POB_HD bool fr_eq(const Fr &a, const Fr &b) { uint32_t o = 0; for (int i = 0; i < 8; i++) o |= a.l[i] ^ b.l[i]; return o == 0; }
POB_HD bool fr_fits64(const Fr &a) { uint32_t o = 0; for (int i = 2; i < 8; i++) o |= a.l[i]; return o == 0; }
POB_HD uint64_t fr_lo64(const Fr &a) { return (uint64_t)a.l[0] | ((uint64_t)a.l[1] << 32); }
// a >= M ?
template <class M, class T> POB_HD bool geq_mod(const T &a) {
#ifdef __CUDA_ARCH__
    uint32_t br;                                                       // borrow of a - M
    asm("sub.cc.u32 %0, %1, %9;\n\tsubc.cc.u32 %0, %2, %10;\n\tsubc.cc.u32 %0, %3, %11;\n\tsubc.cc.u32 %0, %4, %12;\n\t"
        "subc.cc.u32 %0, %5, %13;\n\tsubc.cc.u32 %0, %6, %14;\n\tsubc.cc.u32 %0, %7, %15;\n\tsubc.cc.u32 %0, %8, %16;\n\t"
        "subc.u32 %0, 0, 0;"
        : "=&r"(br)
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(M::limb(0)), "r"(M::limb(1)), "r"(M::limb(2)), "r"(M::limb(3)), "r"(M::limb(4)), "r"(M::limb(5)), "r"(M::limb(6)), "r"(M::limb(7)));
    return br == 0;
#else
    for (int i = 7; i >= 0; i--) { uint32_t p = M::limb(i); if (a.l[i] > p) return true; if (a.l[i] < p) return false; }
    return true;
#endif
}
POB_HD bool fr_geq_p(const Fr &a) { return geq_mod<FrMod>(a); }
// r = a + b / a - b mod 2^256, returning the carry / borrow.  On the device one carry chain (add.cc / addc.cc): the portable form
// costs four instructions per limb.
template <class T> POB_HD uint32_t raw_add(T &r, const T &a, const T &b) {
#ifdef __CUDA_ARCH__
    uint32_t c;
    asm("add.cc.u32 %0, %9, %17;\n\taddc.cc.u32 %1, %10, %18;\n\taddc.cc.u32 %2, %11, %19;\n\taddc.cc.u32 %3, %12, %20;\n\t"
        "addc.cc.u32 %4, %13, %21;\n\taddc.cc.u32 %5, %14, %22;\n\taddc.cc.u32 %6, %15, %23;\n\taddc.cc.u32 %7, %16, %24;\n\t"
        "addc.u32 %8, 0, 0;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7]), "=r"(c)
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
    return c;
#else
    uint64_t c = 0;
    for (int i = 0; i < 8; i++) { c += (uint64_t)a.l[i] + b.l[i]; r.l[i] = (uint32_t)c; c >>= 32; }
    return (uint32_t)c;
#endif
}
template <class T> POB_HD uint32_t raw_sub(T &r, const T &a, const T &b) {
#ifdef __CUDA_ARCH__
    uint32_t br;
    asm("sub.cc.u32 %0, %9, %17;\n\tsubc.cc.u32 %1, %10, %18;\n\tsubc.cc.u32 %2, %11, %19;\n\tsubc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, %21;\n\tsubc.cc.u32 %5, %14, %22;\n\tsubc.cc.u32 %6, %15, %23;\n\tsubc.cc.u32 %7, %16, %24;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7]), "=r"(br)
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
    return br & 1u;
#else
    uint64_t br = 0;
    for (int i = 0; i < 8; i++) { uint64_t d = (uint64_t)a.l[i] - b.l[i] - br; r.l[i] = (uint32_t)d; br = (d >> 32) & 1; }
    return (uint32_t)br;
#endif
}
POB_HD uint32_t fr_raw_add(Fr &r, const Fr &a, const Fr &b) { return raw_add(r, a, b); }
POB_HD uint32_t fr_raw_sub(Fr &r, const Fr &a, const Fr &b) { return raw_sub(r, a, b); }
template <class M, class T> POB_HD T mod_value() { T r; for (int i = 0; i < 8; i++) r.l[i] = M::limb(i); return r; }
POB_HD Fr fr_p() { return mod_value<FrMod, Fr>(); }
template <class M, class T> POB_HD T mod_add(const T &a, const T &b) {
#ifdef __CUDA_ARCH__
    T r, t; raw_add(r, a, b);                                          // a, b < M < 2^254: no carry out
    const uint32_t keep = 0u - raw_sub(t, r, mod_value<M, T>());      // all-ones: r < M
#pragma unroll
    for (int i = 0; i < 8; i++) t.l[i] ^= (t.l[i] ^ r.l[i]) & keep;
    return t;
#else
    T r; uint32_t c = raw_add(r, a, b);
    if (c || geq_mod<M>(r)) { T t; raw_sub(t, r, mod_value<M, T>()); return t; }
    return r;
#endif
}
template <class M, class T> POB_HD T mod_sub(const T &a, const T &b) {
#ifdef __CUDA_ARCH__
    T r, t; const uint32_t wrap = 0u - raw_sub(r, a, b);              // all-ones: a < b
    raw_add(t, r, mod_value<M, T>());
#pragma unroll
    for (int i = 0; i < 8; i++) r.l[i] ^= (r.l[i] ^ t.l[i]) & wrap;
    return r;
#else
    T r; if (raw_sub(r, a, b)) { T t; raw_add(t, r, mod_value<M, T>()); return t; }
    return r;
#endif
}
POB_HD Fr fr_add(const Fr &a, const Fr &b) { return mod_add<FrMod>(a, b); }
POB_HD Fr fr_sub(const Fr &a, const Fr &b) { return mod_sub<FrMod>(a, b); }
POB_HD Fr fr_neg(const Fr &a) { if (fr_is_zero(a)) return a; Fr t; fr_raw_sub(t, fr_p(), a); return t; }

// Montgomery product a*b*2^-256 mod M.  Result < M (one conditional subtraction); a < M, b < 2^256.
// Portable form (host, emulator, `make portable`): column-wise (product scanning) -- the 64 limb products of the 512-bit product
// are mutually independent (each column keeps a split lo/hi accumulator, so no carry chain links them), and the reduction needs
// only the 8-step chain m_k = column_k * n0'.  On the device it compiles to 620 instructions (130 IMAD.WIDE + 354 adds).
#if defined(__CUDA_ARCH__) && !defined(POB_PORTABLE_MONT)
// Device form: CIOS over two accumulators, E (limb k at weight 2^32k) and O (limb k at weight 2^32(k+1)), so that every 32x32
// product lands on an aligned limb PAIR: ptxas fuses each `mad(c).lo.cc / madc.hi.cc` pair into one IMAD.WIDE.U32(.X) with
// carry-in/out predicates -- 128 multiply-adds and ~70 other instructions per product instead of ~620 (the portable form below
// splits every product into halves to keep its column sums inside 64 bits).  Per word b_i: E += a_even*b_i, O += a_odd*b_i,
// m = E0*n0', E += p_even*m, O += p_odd*m, then t >>= 32 (E' = O, O' = E >> 64, E'[0] += E[1]) -- a renaming in unrolled code.
// Bounds (a < M < 2^254, b < 2^256): t < 2^288 before the shift, so E needs 9 limbs, O 8, and no O row carries out.  The algorithm
// (same chains, same renaming) is checked against big-integer arithmetic by tests/test_host.py::test_even_odd_montgomery_model,
// and with the F_q modulus by tests/test_msm_cpu.py.
#define POB_ROW(T, s0, s1, s2, s3, w)                                                                                              \
    "mad.lo.cc.u32 %0, %" s0 ", %" w ", %0;\n\tmadc.hi.cc.u32 %1, %" s0 ", %" w ", %1;\n\t"                                         \
    "madc.lo.cc.u32 %2, %" s1 ", %" w ", %2;\n\tmadc.hi.cc.u32 %3, %" s1 ", %" w ", %3;\n\t"                                        \
    "madc.lo.cc.u32 %4, %" s2 ", %" w ", %4;\n\tmadc.hi.cc.u32 %5, %" s2 ", %" w ", %5;\n\t"                                        \
    "madc.lo.cc.u32 %6, %" s3 ", %" w ", %6;\n\tmadc.hi.cc.u32 %7, %" s3 ", %" w ", %7;\n\t"
__device__ __forceinline__ void mont_row_e(uint32_t *T, uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3, uint32_t w) {   // T[0..7] += s*w, carry into T[8]
    asm(POB_ROW(T, "9", "10", "11", "12", "13") "addc.u32 %8, %8, 0;"
        : "+r"(T[0]), "+r"(T[1]), "+r"(T[2]), "+r"(T[3]), "+r"(T[4]), "+r"(T[5]), "+r"(T[6]), "+r"(T[7]), "+r"(T[8])
        : "r"(s0), "r"(s1), "r"(s2), "r"(s3), "r"(w));
}
__device__ __forceinline__ void mont_row_o(uint32_t *T, uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3, uint32_t w) {   // T[0..7] += s*w (never carries out)
    uint32_t unused = 0;
    asm(POB_ROW(T, "9", "10", "11", "12", "13") "addc.u32 %8, %8, 0;"
        : "+r"(T[0]), "+r"(T[1]), "+r"(T[2]), "+r"(T[3]), "+r"(T[4]), "+r"(T[5]), "+r"(T[6]), "+r"(T[7]), "+r"(unused)
        : "r"(s0), "r"(s1), "r"(s2), "r"(s3), "r"(w));
}
// e0 += x, the carry of that limb (weight 2^32 = O's first limb) enters the row T[0..7] += s*w
__device__ __forceinline__ void mont_row_o_carry(uint32_t &e0, uint32_t x, uint32_t *T, uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3, uint32_t w) {
    asm("add.cc.u32 %8, %8, %14;\n\t"
        "madc.lo.cc.u32 %0, %9, %13, %0;\n\tmadc.hi.cc.u32 %1, %9, %13, %1;\n\t"
        "madc.lo.cc.u32 %2, %10, %13, %2;\n\tmadc.hi.cc.u32 %3, %10, %13, %3;\n\t"
        "madc.lo.cc.u32 %4, %11, %13, %4;\n\tmadc.hi.cc.u32 %5, %11, %13, %5;\n\t"
        "madc.lo.cc.u32 %6, %12, %13, %6;\n\tmadc.hi.u32 %7, %12, %13, %7;"
        : "+r"(T[0]), "+r"(T[1]), "+r"(T[2]), "+r"(T[3]), "+r"(T[4]), "+r"(T[5]), "+r"(T[6]), "+r"(T[7]), "+r"(e0)
        : "r"(s0), "r"(s1), "r"(s2), "r"(s3), "r"(w), "r"(x));
}
template <class M, class T> __device__ __forceinline__ T mont_mul(const T &a, const T &b) {
    uint32_t E[9], O[9], x = 0;
#pragma unroll
    for (int k = 0; k < 9; k++) E[k] = O[k] = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const uint32_t bi = b.l[i];
        mont_row_o_carry(E[0], x, O, a.l[1], a.l[3], a.l[5], a.l[7], bi);
        mont_row_e(E, a.l[0], a.l[2], a.l[4], a.l[6], bi);
        const uint32_t m = E[0] * M::n0;
        mont_row_o(O, M::limb(1), M::limb(3), M::limb(5), M::limb(7), m);
        mont_row_e(E, M::limb(0), M::limb(2), M::limb(4), M::limb(6), m);                    // E[0] is 0 now
        x = E[1];
        uint32_t N[9];
#pragma unroll
        for (int k = 0; k < 7; k++) N[k] = E[k + 2];
        N[7] = 0; N[8] = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) E[k] = O[k];
        E[8] = 0;
#pragma unroll
        for (int k = 0; k < 9; k++) O[k] = N[k];
    }
    T r;
    asm("add.cc.u32 %0, %8, %16;\n\taddc.cc.u32 %1, %9, %17;\n\taddc.cc.u32 %2, %10, %18;\n\taddc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\taddc.cc.u32 %5, %13, %21;\n\taddc.cc.u32 %6, %14, %22;\n\taddc.u32 %7, %15, %23;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7])
        : "r"(E[0]), "r"(E[1]), "r"(E[2]), "r"(E[3]), "r"(E[4]), "r"(E[5]), "r"(E[6]), "r"(E[7]),
          "r"(x), "r"(O[0]), "r"(O[1]), "r"(O[2]), "r"(O[3]), "r"(O[4]), "r"(O[5]), "r"(O[6]));
    if (geq_mod<M>(r)) { T sub; raw_sub(sub, r, mod_value<M, T>()); return sub; }                     // r < 2M
    return r;
}
#undef POB_ROW
#else
template <class M, class T> POB_HD T mont_mul(const T &a, const T &b) {
    uint32_t X[16];
    uint64_t c = 0;
#pragma unroll
    for (int k = 0; k < 15; k++) {                       // X = a * b
        uint64_t lo = c, hi = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int jj = k - i;
            if (jj >= 0 && jj < 8) { const uint64_t p = (uint64_t)a.l[i] * b.l[jj]; lo += (uint32_t)p; hi += p >> 32; }
        }
        X[k] = (uint32_t)lo; c = (lo >> 32) + hi;
    }
    X[15] = (uint32_t)c;
    uint32_t m[8];
    c = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {                        // low half: choose m_k so that column k becomes 0 mod 2^32
        uint64_t lo = c + X[k], hi = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) if (i < k) { const uint64_t p = (uint64_t)m[i] * M::limb(k - i); lo += (uint32_t)p; hi += p >> 32; }
        m[k] = (uint32_t)lo * M::n0;
        const uint64_t p0 = (uint64_t)m[k] * M::limb(0); lo += (uint32_t)p0; hi += p0 >> 32;
        c = (lo >> 32) + hi;
    }
    T r;
#pragma unroll
    for (int k = 8; k < 16; k++) {                       // high half: the result limbs
        uint64_t lo = c + X[k], hi = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) { const int jj = k - i; if (jj >= 1 && jj < 8) { const uint64_t p = (uint64_t)m[i] * M::limb(jj); lo += (uint32_t)p; hi += p >> 32; } }
        r.l[k - 8] = (uint32_t)lo; c = (lo >> 32) + hi;
    }
    if (c || geq_mod<M>(r)) { T sub; raw_sub(sub, r, mod_value<M, T>()); return sub; }
    return r;
}
#endif
POB_HD Fr fr_mont(const Fr &a, const Fr &b) { return mont_mul<FrMod>(a, b); }
POB_HD Fr fr_r2() { Fr r; for (int i = 0; i < 8; i++) r.l[i] = fr_r2_limb(i); return r; }
POB_HD Fr fr_to_mont(const Fr &a) { return fr_mont(a, fr_r2()); }
POB_HD Fr fr_from_mont(const Fr &a) { Fr one = fr_from_u64(1); return fr_mont(a, one); }
// canonical * canonical -> canonical.  Small operands (the overwhelmingly common case: bits, bytes,
// lengths) take a plain 64x64 product, which is < 2^128 < p and needs no reduction.
POB_HD Fr fr_mul(const Fr &a, const Fr &b) {
    if (fr_fits64(a) && fr_fits64(b)) {
        uint64_t x = fr_lo64(a), y = fr_lo64(b);
        uint64_t x0 = (uint32_t)x, x1 = x >> 32, y0 = (uint32_t)y, y1 = y >> 32;
        uint64_t p00 = x0 * y0, p01 = x0 * y1, p10 = x1 * y0, p11 = x1 * y1;
        uint64_t mid = (p00 >> 32) + (uint32_t)p01 + (uint32_t)p10;
        uint64_t hi = p11 + (p01 >> 32) + (p10 >> 32) + (mid >> 32);
        Fr r = fr_zero();
        r.l[0] = (uint32_t)p00; r.l[1] = (uint32_t)mid; r.l[2] = (uint32_t)hi; r.l[3] = (uint32_t)(hi >> 32);
        return r;
    }
    return fr_mont(fr_mont(a, b), fr_r2());
}
POB_HD int fr_bit(const Fr &a, unsigned i) { return (int)((a.l[i >> 5] >> (i & 31)) & 1u); }
// a^-1 by Fermat (a != 0), Montgomery ladder over the fixed exponent p-2
POB_HD Fr fr_inv(const Fr &a) {
    Fr am = fr_to_mont(a);
    Fr r = fr_to_mont(fr_from_u64(1));
    Fr e; { Fr two = fr_from_u64(2); fr_raw_sub(e, fr_p(), two); }
    for (int i = 253; i >= 0; i--) {
        r = fr_mont(r, r);
        if (fr_bit(e, (unsigned)i)) r = fr_mont(r, am);
    }
    return fr_from_mont(r);
}
// a^-1 by the binary extended Euclidean algorithm (a != 0): ~2*254 shift/subtract steps on 8 limbs, roughly an
// order of magnitude fewer instructions than the Fermat ladder; used by the witness VM for IsZero's inverse hints
POB_HD bool fr_geq(const Fr &a, const Fr &b) {
    for (int i = 7; i >= 0; i--) { if (a.l[i] > b.l[i]) return true; if (a.l[i] < b.l[i]) return false; }
    return true;
}
POB_HD void fr_shr1(Fr &a) {
#pragma unroll
    for (int i = 0; i < 7; i++) a.l[i] = (a.l[i] >> 1) | (a.l[i + 1] << 31);
    a.l[7] >>= 1;
}
POB_HD void fr_half_mod(Fr &x) {            // x/2 mod p for x in [0,p): (x + p)/2 when x is odd; x + p < 2^255 fits
    if (x.l[0] & 1u) { Fr t; fr_raw_add(t, x, fr_p()); x = t; }
    fr_shr1(x);
}
POB_HD Fr fr_inv_eea(const Fr &a) {
    Fr u = a, v = fr_p(), x1 = fr_from_u64(1), x2 = fr_zero();
    const Fr one = fr_from_u64(1);
    while (!fr_eq(u, one) && !fr_eq(v, one)) {
        while (!(u.l[0] & 1u)) { fr_shr1(u); fr_half_mod(x1); }
        while (!(v.l[0] & 1u)) { fr_shr1(v); fr_half_mod(x2); }
        if (fr_geq(u, v)) { Fr t; fr_raw_sub(t, u, v); u = t; x1 = fr_sub(x1, x2); }
        else { Fr t; fr_raw_sub(t, v, u); v = t; x2 = fr_sub(x2, x1); }
    }
    return fr_eq(u, one) ? x1 : x2;
}
// value < 2^n ?  (n <= 256)
POB_HD bool fr_lt_pow2(const Fr &a, unsigned n) {
    uint32_t bad = 0;
#pragma unroll
    for (unsigned i = 0; i < 8; i++) {
        unsigned lo = 32 * i;
        if (lo >= n) bad |= a.l[i];
        else if (lo + 32 > n) bad |= a.l[i] >> (n - lo);
    }
    return bad == 0;
}
// integer quotient / remainder of canonical representatives by a divisor that fits 32 bits (the circuits
// only divide by compile-time constants 136, 4 and 2: utils/keccak.circom:420, rlp/...leaf.circom:60)
POB_HD void fr_divmod_u32(const Fr &a, uint32_t d, Fr &q, Fr &r) {
    uint64_t rem = 0; q = fr_zero();
    for (int i = 7; i >= 0; i--) { uint64_t cur = (rem << 32) | a.l[i]; q.l[i] = (uint32_t)(cur / d); rem = cur % d; }
    r = fr_from_u64(rem);
}
// general 256/256 schoolbook (shift-subtract); rare path (divisor is a signal, e.g. the Divide(16) gadget suite)
POB_HD void fr_divmod(const Fr &a, const Fr &b, Fr &q, Fr &r) {
    if (fr_fits64(b) && (fr_lo64(b) >> 32) == 0) { fr_divmod_u32(a, b.l[0], q, r); return; }
    q = fr_zero(); r = fr_zero();
    for (int i = 255; i >= 0; i--) {
        uint32_t c = 0;
        for (int k = 0; k < 8; k++) { uint32_t n = (r.l[k] << 1) | c; c = r.l[k] >> 31; r.l[k] = n; }
        r.l[0] |= (uint32_t)fr_bit(a, (unsigned)i);
        Fr t; if (!fr_raw_sub(t, r, b)) { r = t; q.l[i >> 5] |= 1u << (i & 31); }
    }
}

}  // namespace pob
