// pairing.cuh -- the optimal ate pairing of BN254 (pob_bn254_pairing) and Groth16 verification (pob_groth16_verify), DESIGN.md §5
// "Verification".
//
// e(P, Q) = f^((q^12 - 1) / r), f = f_{6x+2,Q}(P) l_{T,pi(Q)}(P) l_{T + pi(Q),-pi^2(Q)}(P), x = 4965661367192848881, T = [6x+2]Q.
// Q lives on the twist y^2 = x^3 + 3 / xi (fq2_hd.h); the untwisting map is (x, y) -> (x w^2, y w^3).
//   Miller loop.  6x + 2 in non-adjacent form (66 digits, 21 non-zero below the top one).  T stays on the twist in homogeneous
//     projective coordinates (X : Y : Z), so no step inverts.  Doubling and addition are the formulas of Costello-Lange-Naehrig /
//     Aranha et al. for a D-type twist: each step returns its line l = c0 yP + c1 xP w + c2 v w, scaled by an F_q2 factor that the
//     final exponentiation removes, and multiplies f by it with the sparse fq12_mul_034.  The k pairs of a multi-pairing share
//     f's squarings.  A pair with O on either side is skipped: it contributes 1.
//   pi(Q) = (conj(x) gamma_{1,2}, conj(y) gamma_{1,3}), -pi^2(Q) = (x gamma_{2,2}, y): the Frobenius of the untwisted point, on the
//     twist.
//   Final exponentiation.  Easy part f^((q^6 - 1)(q^2 + 1)): conjugate over f, then a q^2 Frobenius.  Hard part: exactly
//     (q^4 - q^2 + 1) / r = l0 + l1 q + l2 q^2 + q^3 with l0 = -36x^3 - 30x^2 - 18x - 2, l1 = -36x^3 - 18x^2 - 12x + 1,
//     l2 = 6x^2 + 1 (an identity in x, checked by tests/test_pairing_cpu.py), from a = f^x, b = a^x, c = b^x by cyclotomic squarings,
//     with conjugation as the inverse.  The result is therefore the pairing itself, not a power of it.
// G2 membership is the definition, [r]Q = O (one 256-bit scalar multiplication).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fq12_hd.h"

using namespace pob;

namespace {

enum { PAIR_LINES = 88 };                                     // 65 doublings, 21 additions, pi(Q), -pi^2(Q)
// the digits of 6x + 2 below its top one (index 65): bit i of POS / NEG = digit i is +1 / -1; digit 64 is 0
constexpr uint64_t PAIR_NAF_POS = 0x2002004200804028ull, PAIR_NAF_NEG = 0x82889008420a0480ull;
constexpr uint64_t PAIR_X = 0x44e992b44a6909f1ull;           // x

struct G2Proj { Fq2 x, y, z; };
struct PairLine { Fq2 c0, c1, c2; };                          // the line before its scaling by yP (c0) and xP (c1): 192 bytes

__device__ __forceinline__ Fq pair_fq_const(const uint32_t (&v)[8]) { Fq r; for (int i = 0; i < 8; i++) r.l[i] = v[i]; return r; }
__device__ __forceinline__ Fq2 pair_b2() {                   // b' = 3 / (9 + u), Montgomery form
    constexpr uint32_t C0[8] = {0x77b802a8u, 0x3bf938e3u, 0x3633535du, 0x020b1b27u, 0x49755260u, 0x26b7edf0u, 0x4384a86du, 0x2514c632u};
    constexpr uint32_t C1[8] = {0xd1dcff67u, 0x38e7ecccu, 0x93ce0d3eu, 0x65f0b37du, 0x22ac00aau, 0xd749d0ddu, 0x4a688d4du, 0x0141b9ceu};
    Fq2 r; r.c0 = pair_fq_const(C0); r.c1 = pair_fq_const(C1); return r;
}
__device__ __forceinline__ Fq pair_two_inv() {               // 1 / 2, Montgomery form
    constexpr uint32_t V[8] = {0x4f060572u, 0x87bee7d2u, 0x2f1c6ae5u, 0xd0fd2addu, 0xfcfd4f44u, 0x8f5f7492u, 0x3d9cbfacu, 0x1f37631au};
    return pair_fq_const(V);
}

// ---- Miller loop --------------------------------------------------------------------------------------------------------------
// T = 2T and the tangent at T: a = XY/2, b = Y^2, c = Z^2, e = 3 b' c, f = 3e, g = (b + f)/2, h = 2YZ;
// X' = a (b - f), Y' = g^2 - 3 e^2, Z' = b h; line (-h, 3 X^2, e - b)
__device__ __noinline__ PairLine pair_dbl_step(G2Proj &t) {
    const Fq hf = pair_two_inv();
    const Fq2 a = fq2_mul_fq(fq2_mul(t.x, t.y), hf), b = fq2_sqr(t.y), c = fq2_sqr(t.z);
    const Fq2 e = fq2_mul(pair_b2(), fq2_add(fq2_add(c, c), c)), f = fq2_add(fq2_add(e, e), e);
    const Fq2 g = fq2_mul_fq(fq2_add(b, f), hf);
    const Fq2 h = fq2_sub(fq2_sqr(fq2_add(t.y, t.z)), fq2_add(b, c));
    const Fq2 j = fq2_sqr(t.x), e2 = fq2_sqr(e);
    PairLine l;
    l.c0 = fq2_neg(h);
    l.c1 = fq2_add(fq2_add(j, j), j);
    l.c2 = fq2_sub(e, b);
    t.x = fq2_mul(a, fq2_sub(b, f));
    t.y = fq2_sub(fq2_sqr(g), fq2_add(fq2_add(e2, e2), e2));
    t.z = fq2_mul(b, h);
    return l;
}
// T = T + Q (Q affine) and the line through them: theta = Y - qy Z, lambda = X - qx Z; line (lambda, -theta, theta qx - lambda qy)
__device__ __noinline__ PairLine pair_add_step(G2Proj &t, const G2Aff &q) {
    const Fq2 th = fq2_sub(t.y, fq2_mul(q.y, t.z)), la = fq2_sub(t.x, fq2_mul(q.x, t.z));
    const Fq2 c = fq2_sqr(th), d = fq2_sqr(la), e = fq2_mul(la, d), f = fq2_mul(t.z, c), g = fq2_mul(t.x, d);
    const Fq2 h = fq2_sub(fq2_add(e, f), fq2_add(g, g));
    PairLine l;
    l.c0 = la;
    l.c1 = fq2_neg(th);
    l.c2 = fq2_sub(fq2_mul(th, q.x), fq2_mul(la, q.y));
    t.x = fq2_mul(la, h);
    t.y = fq2_sub(fq2_mul(th, fq2_sub(g, h)), fq2_mul(e, t.y));
    t.z = fq2_mul(t.z, e);
    return l;
}
__device__ __forceinline__ G2Aff pair_pi(const G2Aff &q) {     // pi(Q)
    G2Aff r; r.x = fq2_mul(fq2_conj(q.x), fq12_frob_const(1, 2)); r.y = fq2_mul(fq2_conj(q.y), fq12_frob_const(1, 3)); return r;
}
__device__ __forceinline__ G2Aff pair_neg_pi2(const G2Aff &q) { // -pi^2(Q); gamma_{2,3} = -1
    G2Aff r; r.x = fq2_mul(q.x, fq12_frob_const(2, 2)); r.y = q.y; return r;
}
__device__ __forceinline__ void pair_ell(Fq12 &f, const PairLine &l, const G1Aff &p) {
    f = fq12_mul_034(f, fq2_mul_fq(l.c0, p.y), fq2_mul_fq(l.c1, p.x), l.c2);
}
__device__ __forceinline__ int pair_digit(int i) {
    return i >= 64 ? 0 : ((PAIR_NAF_POS >> i) & 1) ? 1 : ((PAIR_NAF_NEG >> i) & 1) ? -1 : 0;
}

// The line sequence of one Q, in the Miller loop's order, into out[PAIR_LINES]: the fixed G2 points of a verification key.
__device__ void pair_lines(const G2Aff &q, PairLine *out) {
    G2Proj t; t.x = q.x; t.y = q.y; t.z = fq2_one();
    const G2Aff nq = pt_aff_neg(q);
    int k = 0;
#pragma unroll 1
    for (int i = 64; i >= 0; i--) {
        out[k++] = pair_dbl_step(t);
        const int d = pair_digit(i);
        if (d) out[k++] = pair_add_step(t, d > 0 ? q : nq);
    }
    out[k++] = pair_add_step(t, pair_pi(q));
    out[k++] = pair_add_step(t, pair_neg_pi2(q));
}

// The product of k <= 3 Miller loops sharing the squarings of f.  Pair j: P p[j] (affine, Montgomery) and either precomputed lines
// pre[j] (pair_lines) or, when pre[j] is null, the lines of q[j] computed on the way.  skip[j]: the pair contributes 1.
__device__ __noinline__ Fq12 pair_miller(const G1Aff *p, const G2Aff *q, const PairLine *const *pre, const bool *skip, int k) {
    G2Proj t[3];
    G2Aff nq[3];
    for (int j = 0; j < k; j++) { t[j].x = q[j].x; t[j].y = q[j].y; t[j].z = fq2_one(); nq[j] = pt_aff_neg(q[j]); }
    Fq12 f = fq12_one();
    int li = 0;
#pragma unroll 1
    for (int i = 64; i >= 0; i--) {
        if (i != 64) f = fq12_sqr(f);
        for (int j = 0; j < k; j++)
            if (!skip[j]) pair_ell(f, pre[j] ? pre[j][li] : pair_dbl_step(t[j]), p[j]);
        li++;
        const int d = pair_digit(i);
        if (d) {
            for (int j = 0; j < k; j++)
                if (!skip[j]) pair_ell(f, pre[j] ? pre[j][li] : pair_add_step(t[j], d > 0 ? q[j] : nq[j]), p[j]);
            li++;
        }
    }
    for (int j = 0; j < k; j++)
        if (!skip[j]) pair_ell(f, pre[j] ? pre[j][li] : pair_add_step(t[j], pair_pi(q[j])), p[j]);
    li++;
    for (int j = 0; j < k; j++)
        if (!skip[j]) pair_ell(f, pre[j] ? pre[j][li] : pair_add_step(t[j], pair_neg_pi2(q[j])), p[j]);
    return f;
}

// ---- final exponentiation -----------------------------------------------------------------------------------------------------
// a^e in the cyclotomic subgroup, square-and-multiply from the top bit of e
__device__ __noinline__ Fq12 pair_cyc_pow(const Fq12 &a, uint64_t e) {
    Fq12 r = a;
    const int top = 63 - __clzll(e);
#pragma unroll 1
    for (int i = top - 1; i >= 0; i--) {
        r = fq12_cyc_sqr(r);
        if ((e >> i) & 1) r = fq12_mul(r, a);
    }
    return r;
}
// f^((q^12 - 1) / r), exactly; 0 gives 0
__device__ __noinline__ Fq12 pair_final_exp(const Fq12 &f0) {
    Fq12 f = fq12_mul(fq12_conj(f0), fq12_inv(f0));                    // f^(q^6 - 1)
    f = fq12_mul(fq12_frob(f, 2), f);                                   // ^(q^2 + 1)
    const Fq12 a = pair_cyc_pow(f, PAIR_X), b = pair_cyc_pow(a, PAIR_X), c = pair_cyc_pow(b, PAIR_X);
    const Fq12 c36 = pair_cyc_pow(c, 36), b6 = pair_cyc_pow(b, 6);
    const Fq12 b18 = pair_cyc_pow(b6, 3), a6 = pair_cyc_pow(a, 6);
    const Fq12 a12 = fq12_cyc_sqr(a6), a18 = fq12_mul(a12, a6);
    const Fq12 c36b18 = fq12_mul(c36, b18);
    const Fq12 l0 = fq12_conj(fq12_mul(fq12_mul(c36b18, fq12_cyc_sqr(b6)), fq12_mul(a18, fq12_cyc_sqr(f))));   // f^l0
    const Fq12 l1 = fq12_mul(fq12_conj(fq12_mul(c36b18, a12)), f);                                            // f^l1
    const Fq12 l2 = fq12_mul(b6, f);                                                                          // f^l2
    return fq12_mul(fq12_mul(l0, fq12_frob(l1, 1)), fq12_mul(fq12_frob(l2, 2), fq12_frob(f, 3)));
}

// ---- points -------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool pair_lt_q(const Fq &a) { return !geq_mod<FqMod>(a); }
__device__ __forceinline__ bool pair_lt_q(const Fq2 &a) { return pair_lt_q(a.c0) && pair_lt_q(a.c1); }
// affine Montgomery-form point on y^2 = x^3 + b, or (0, 0)
__device__ __forceinline__ bool pair_on_g1(const G1Aff &a) {
    if (pt_aff_is_inf(a)) return true;
    const Fq three = fq_to_mont(Fq{{3, 0, 0, 0, 0, 0, 0, 0}});
    return fq_is_zero(fq_sub(fq_sqr(a.y), fq_add(fq_mul(fq_sqr(a.x), a.x), three)));
}
__device__ __forceinline__ bool pair_on_twist(const G2Aff &a) {
    if (pt_aff_is_inf(a)) return true;
    return fq2_is_zero(fq2_sub(fq2_sqr(a.y), fq2_add(fq2_mul(fq2_sqr(a.x), a.x), pair_b2())));
}
// [r]Q = O, for Q on the twist (O is in the subgroup)
__device__ __noinline__ bool pair_in_g2(const G2Aff &q) {
    const Fr r = fr_p();
    return pt_is_inf(pt_mul_u256(pt_from_aff(q), r.l));
}

__device__ __forceinline__ Fq pair_ld_fq(const uint4 *p) {
    const uint4 a = p[0], b = p[1];
    Fq r; r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}
__device__ __forceinline__ void pair_st_fq(uint4 *p, const Fq &a) {
    p[0] = make_uint4(a.l[0], a.l[1], a.l[2], a.l[3]); p[1] = make_uint4(a.l[4], a.l[5], a.l[6], a.l[7]);
}
__device__ __forceinline__ G1Aff pair_ld_g1(const uint4 *p) { G1Aff a; a.x = pair_ld_fq(p); a.y = pair_ld_fq(p + 2); return a; }
__device__ __forceinline__ G2Aff pair_ld_g2(const uint4 *p) {
    G2Aff a; a.x.c0 = pair_ld_fq(p); a.x.c1 = pair_ld_fq(p + 2); a.y.c0 = pair_ld_fq(p + 4); a.y.c1 = pair_ld_fq(p + 6); return a;
}
__device__ __forceinline__ G1Aff pair_g1_to_mont(const G1Aff &a) { G1Aff r; r.x = fq_to_mont(a.x); r.y = fq_to_mont(a.y); return r; }
__device__ __forceinline__ G2Aff pair_g2_to_mont(const G2Aff &a) { G2Aff r; r.x = fq2_to_mont(a.x); r.y = fq2_to_mont(a.y); return r; }

// ---- pob_bn254_pairing ----------------------------------------------------------------------------------------------------------
// one pair per thread: g1 (64 B) and g2 (128 B) Montgomery-form affine points in, 12 canonical F_q values out (384 B)
__global__ void __launch_bounds__(128) k_bn254_pairing(const uint4 *g1, const uint4 *g2, uint64_t n, uint4 *out) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const G1Aff p = pair_ld_g1(g1 + 4 * i);
        const G2Aff q = pair_ld_g2(g2 + 8 * i);
        const bool skip = pt_aff_is_inf(p) || pt_aff_is_inf(q);
        const PairLine *pre = nullptr;
        const Fq12 e = pair_final_exp(pair_miller(&p, &q, &pre, &skip, 1));
        const Fq *v = &e.c0.c0.c0;                                       // Fq12 is 12 consecutive Fq in the output order
        for (int k = 0; k < 12; k++) pair_st_fq(out + 24 * i + 2 * k, fq_from_mont(v[k]));
    }
}

// ---- pob_groth16_verify ---------------------------------------------------------------------------------------------------------
enum { VERIFY_OK = 0, VERIFY_FAIL = 1, VERIFY_BAD_POINT = 2, VERIFY_BAD_SUBGROUP = 3, VERIFY_BAD_PUBLIC = 4, VERIFY_BAD_KEY = 5 };
enum { VERIFY_PREP_THREADS = 128 };

// byte offsets into the caller's work buffer
struct VerifyLayout { uint64_t flags, m_ab, gamma_lines, delta_lines, bytes; };
__host__ __device__ __forceinline__ VerifyLayout verify_layout() {
    VerifyLayout L;
    L.flags = 0;                                                         // one word per preparation thread: the key is bad
    L.m_ab = 4 * VERIFY_PREP_THREADS;                                    // f_{alpha1,beta2}, before the final exponentiation
    L.gamma_lines = L.m_ab + 512;
    L.delta_lines = L.gamma_lines + PAIR_LINES * sizeof(PairLine);
    L.bytes = L.delta_lines + PAIR_LINES * sizeof(PairLine);
    return L;
}

struct VerifyKeyDev {
    uint32_t n_pub;
    const uint4 *alpha1, *beta2, *gamma2, *delta2, *ic;                  // Montgomery form, as in a .zkey
};

// The once-per-call preparation, one block of VERIFY_PREP_THREADS: every thread checks a share of the IC points; one lane of each
// warp does one of the long single-thread jobs, so that they run side by side (warp 0: alpha1, beta2 and f_{alpha1,beta2}; warp 1:
// beta2's subgroup; warps 2 and 3: gamma2 and delta2, their subgroups and their lines).
__global__ void __launch_bounds__(VERIFY_PREP_THREADS) k_verify_prepare(VerifyKeyDev vk, uint8_t *work) {
    const VerifyLayout L = verify_layout();
    const uint32_t t = threadIdx.x;
    bool bad = false;
    for (uint32_t i = t; i <= vk.n_pub; i += VERIFY_PREP_THREADS) {
        const G1Aff a = pair_ld_g1(vk.ic + 4 * i);
        bad |= !(pair_lt_q(a.x) && pair_lt_q(a.y) && pair_on_g1(a));
    }
    if (t == 0) {
        const G1Aff a = pair_ld_g1(vk.alpha1);
        const G2Aff b = pair_ld_g2(vk.beta2);
        const bool ok = pair_lt_q(a.x) && pair_lt_q(a.y) && pair_on_g1(a) && pair_lt_q(b.x) && pair_lt_q(b.y) && pair_on_twist(b);
        bad |= !ok;
        const bool skip = pt_aff_is_inf(a) || pt_aff_is_inf(b);
        const PairLine *pre = nullptr;
        *(Fq12 *)(work + L.m_ab) = ok ? pair_miller(&a, &b, &pre, &skip, 1) : fq12_one();
    } else if (t == 32) {
        bad |= !pair_in_g2(pair_ld_g2(vk.beta2));
    } else if (t == 64 || t == 96) {
        const G2Aff q = pair_ld_g2(t == 64 ? vk.gamma2 : vk.delta2);
        const bool ok = pair_lt_q(q.x) && pair_lt_q(q.y) && !pt_aff_is_inf(q) && pair_on_twist(q) && pair_in_g2(q);
        bad |= !ok;
        if (ok) pair_lines(q, (PairLine *)(work + (t == 64 ? L.gamma_lines : L.delta_lines)));
    }
    ((uint32_t *)(work + L.flags))[t] = bad;
}

struct VerifyArgs {
    VerifyKeyDev vk;
    const uint4 *proofs;      // n x 256 B: A, B, C canonical affine, all-zero = O
    const uint4 *publics;     // n x n_pub x 32 B canonical
    uint64_t n;
    uint32_t *status;
    const uint8_t *work;
};

// one proof per thread: the checks of A, B, C and the public inputs, vk_x, the three-pair Miller product times f_{alpha1,beta2},
// the final exponentiation, the comparison with 1
__global__ void __launch_bounds__(128) k_groth16_verify(VerifyArgs v) {
    const VerifyLayout L = verify_layout();
    bool key_bad = false;
    for (int t = 0; t < VERIFY_PREP_THREADS; t++) key_bad |= ((const uint32_t *)(v.work + L.flags))[t] != 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < v.n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (key_bad) { v.status[i] = VERIFY_BAD_KEY; continue; }
        const uint4 *pr = v.proofs + 16 * i;
        G1Aff a = pair_ld_g1(pr), c = pair_ld_g1(pr + 12);
        G2Aff b = pair_ld_g2(pr + 4);
        if (!(pair_lt_q(a.x) && pair_lt_q(a.y) && pair_lt_q(b.x) && pair_lt_q(b.y) && pair_lt_q(c.x) && pair_lt_q(c.y))) {
            v.status[i] = VERIFY_BAD_POINT; continue;
        }
        a = pair_g1_to_mont(a); b = pair_g2_to_mont(b); c = pair_g1_to_mont(c);
        if (!(pair_on_g1(a) && pair_on_twist(b) && pair_on_g1(c))) { v.status[i] = VERIFY_BAD_POINT; continue; }
        bool pub_ok = true;
        for (uint32_t j = 0; j < v.vk.n_pub; j++) pub_ok = pub_ok && !fr_geq_p(*(const Fr *)(v.publics + 2 * ((uint64_t)i * v.vk.n_pub + j)));
        if (!pub_ok) { v.status[i] = VERIFY_BAD_PUBLIC; continue; }
        if (!pair_in_g2(b)) { v.status[i] = VERIFY_BAD_SUBGROUP; continue; }
        G1Xyzz x = pt_from_aff(pair_ld_g1(v.vk.ic));
#pragma unroll 1
        for (uint32_t j = 0; j < v.vk.n_pub; j++) {
            const Fr s = *(const Fr *)(v.publics + 2 * ((uint64_t)i * v.vk.n_pub + j));
            x = pt_add(x, pt_mul_u256(pt_from_aff(pair_ld_g1(v.vk.ic + 4 * (j + 1))), s.l));
        }
        G1Aff p[3];
        p[0] = pt_aff_neg(a);
        p[1] = pair_g1_to_mont(pt_to_affine_canonical(x));
        p[2] = c;
        G2Aff q[3];
        q[0] = b;
        q[1] = q[2] = b;                                                 // unused: their lines are precomputed
        const PairLine *pre[3] = {nullptr, (const PairLine *)(v.work + L.gamma_lines), (const PairLine *)(v.work + L.delta_lines)};
        const bool skip[3] = {pt_aff_is_inf(a) || pt_aff_is_inf(b), pt_aff_is_inf(p[1]), pt_aff_is_inf(c)};
        const Fq12 f = fq12_mul(pair_miller(p, q, pre, skip, 3), *(const Fq12 *)(v.work + L.m_ab));
        v.status[i] = fq12_is_one(pair_final_exp(f)) ? VERIFY_OK : VERIFY_FAIL;
    }
}

}  // namespace
