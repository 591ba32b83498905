// groth16.cuh -- the last step of pob_groth16_prove (DESIGN.md §5): the blinding terms and the additions of alpha, beta and delta
// around the five multi-exponentiations (msm.cuh), and the scratch layout of the whole proof.
//
//   A  = alpha1 + MSM(A)  + [r] delta1
//   B1 = beta1  + MSM(B1) + [s] delta1,  B = beta2 + MSM(B2) + [s] delta2
//   C  = MSM(C) + MSM(H) + [s] A + [r] B1 - [r s] delta1
// r and s arrive by value (any 256-bit integers, taken mod r).  One thread: four G1 and one G2 256-bit scalar multiplications and
// three inversions, small next to the multi-exponentiations.
#pragma once
#include "msm.cuh"

namespace {

struct Groth16Assemble {
    const uint4 *alpha1, *beta1, *delta1, *beta2, *delta2;    // key points: affine, Montgomery form
    const uint4 *h, *a, *b1, *c, *b2;                          // the MSM results: affine, canonical
    uint32_t r[8], s[8];                                       // blinding scalars, LE
    uint4 *proof;                                              // A (4 uint4), B (8), C (4): affine, canonical
};

template <class F> __device__ __forceinline__ Aff<F> g16_ld(const uint4 *p, bool canonical) {
    Aff<F> a; msm_ld(p, a.x); msm_ld(p + MsmCurve<F>::FIELD_U4, a.y);
    if (canonical) { a.x = f_to_mont(a.x); a.y = f_to_mont(a.y); }    // (0, 0) stays (0, 0)
    return a;
}
template <class F> __device__ __forceinline__ void g16_st(uint4 *p, const Xyzz<F> &P) {
    const Aff<F> a = pt_to_affine_canonical(P);
    msm_st(p, a.x); msm_st(p + MsmCurve<F>::FIELD_U4, a.y);
}
__device__ __forceinline__ Fr g16_mod_r(const uint32_t *v) {
    Fr s; for (int i = 0; i < 8; i++) s.l[i] = v[i];
#pragma unroll 1
    for (int k = 0; k < 5; k++) {                                      // 2^256 < 6 r
        if (!fr_geq_p(s)) break;
        Fr t; fr_raw_sub(t, s, fr_p()); s = t;
    }
    return s;
}

__global__ void k_groth16_assemble(Groth16Assemble g) {
    const Fr r = g16_mod_r(g.r), s = g16_mod_r(g.s), rs = fr_mul(r, s);
    const G1Xyzz d1 = pt_from_aff(g16_ld<Fq>(g.delta1, false));
    G1Xyzz A = pt_add_aff(pt_from_aff(g16_ld<Fq>(g.alpha1, false)), g16_ld<Fq>(g.a, true));
    A = pt_add(A, pt_mul_u256(d1, r.l));
    G1Xyzz B1 = pt_add_aff(pt_from_aff(g16_ld<Fq>(g.beta1, false)), g16_ld<Fq>(g.b1, true));
    B1 = pt_add(B1, pt_mul_u256(d1, s.l));
    G2Xyzz B = pt_add_aff(pt_from_aff(g16_ld<Fq2>(g.beta2, false)), g16_ld<Fq2>(g.b2, true));
    B = pt_add(B, pt_mul_u256(pt_from_aff(g16_ld<Fq2>(g.delta2, false)), s.l));
    G1Xyzz C = pt_add_aff(pt_from_aff(g16_ld<Fq>(g.c, true)), g16_ld<Fq>(g.h, true));
    C = pt_add(C, pt_mul_u256(A, s.l));
    C = pt_add(C, pt_mul_u256(B1, r.l));
    C = pt_add(C, pt_mul_u256(pt_from_aff(pt_aff_neg(g16_ld<Fq>(g.delta1, false))), rs.l));
    g16_st(g.proof, A);
    g16_st(g.proof + 4, B);
    g16_st(g.proof + 12, C);
}

// byte offsets into the caller's work buffer of one proof over a domain of n = 2^log_n points and n_vars witness entries
struct Groth16Layout {
    uint64_t q, scratch, h, a, b1, c, b2, bytes;
};
static Groth16Layout groth16_layout(uint64_t n, uint64_t n_vars, uint64_t n_pub) {
    Groth16Layout L;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t o = at; at += (bytes + 255) & ~255ull; return o; };
    uint64_t s = std::max<uint64_t>(64 * n, msm_layout<MsmG1>(n).bytes);                   // the quotient's work, then the H MSM's
    s = std::max(s, msm_layout<MsmG1>(n_vars).bytes);                                       // A and B1
    if (n_vars > n_pub + 1) s = std::max(s, msm_layout<MsmG1>(n_vars - n_pub - 1).bytes);   // C
    s = std::max(s, msm_layout<MsmG2>(n_vars).bytes);                                       // B2
    L.q = take(32 * n);
    L.scratch = take(s);
    L.h = take(64); L.a = take(64); L.b1 = take(64); L.c = take(64); L.b2 = take(128);
    L.bytes = at;
    return L;
}

}  // namespace
