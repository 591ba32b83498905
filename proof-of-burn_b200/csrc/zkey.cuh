// zkey.cuh -- the GPU check of a snarkjs `.zkey` against the circuit (pob_zkey_load, pob_b200.cu).
//
// Coefficients (Schwartz-Zippel).  x_j (one per wire) and rho_c (one per domain row) are pseudo-random canonical elements < 2^253,
// derived from the caller's seed by zk_rand.  For M = A, B:
//   coefficient side  S_M = sum over the section-4 entries (M, c, s, v) of mont(mont(v, x_s), rho_c)        (k_zkey_coefs)
//   row side          T_M = sum over rows c of mont((M x)_c, rho_c), (M x)_c from k_r1cs_products over x  (k_zkey_rows)
// mont(a, b) = a b / R.  With v = k R^2 (the encoding snarkjs uses), mont(mont(v, x), rho) = k x rho, so S_M = sum rho_c x_s k, and
// T_M = (sum rho_c (M x)_c) / R: the matrices agree iff S_M = mont(T_M, R^2).  With v = k (canonical), S_M = (sum rho_c x_s k) / R^2,
// which is mont(T_M, 1) when the matrices agree.  Field sums are exact, so the per-block partial sums (one slot per block, added to
// launch after launch on one stream) and their final reduction give the same value in any order.
// Points.  Every coordinate < q, and y^2 = x^3 + b (G1: b = 3; G2: b' = 3 / (9 + u)) with x, y read in Montgomery form, or (0, 0).
// The same test with x, y read as canonical elements is counted too, as a diagnosis of the encoding.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fq2_hd.h"

using namespace pob;

namespace {

enum { ZK_THREADS = 256 };

// counters of one pob_zkey_load call, in device memory
struct ZkeyCounters {
    unsigned long long points_bad, points_bad_canonical, out_of_range, first_bad;   // first_bad: section << 40 | index, ~0 = none
    uint32_t match, match_canonical;                                                // written by k_zkey_final
};

// splitmix64's finaliser
__device__ __forceinline__ uint64_t zk_mix(uint64_t z) {
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
// element `i` of stream `tag` (0: x, 1: rho), uniform below 2^253 < r
__device__ __forceinline__ Fr zk_rand(uint64_t seed, uint32_t tag, uint64_t i) {
    const uint64_t h = zk_mix(seed ^ zk_mix(2 * i + tag));
    Fr r;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint64_t v = zk_mix(h + 0x632be59bd9b4e019ull * (uint64_t)(k + 1));
        if (k == 3) v &= (1ull << 61) - 1;
        r.l[2 * k] = (uint32_t)v; r.l[2 * k + 1] = (uint32_t)(v >> 32);
    }
    return r;
}
__device__ __forceinline__ Fr zk_load(const uint4 *p, uint64_t i) {
    const uint4 a = p[2 * i], b = p[2 * i + 1];
    Fr r; r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}

// the two sums of a block, added to its slot acc[2 blockIdx + m]
__device__ void zk_block_add(Fr s0, Fr s1, Fr *acc) {
    __shared__ Fr sh[2][ZK_THREADS];
    sh[0][threadIdx.x] = s0; sh[1][threadIdx.x] = s1;
    __syncthreads();
    for (uint32_t w = ZK_THREADS / 2; w; w >>= 1) {
        if (threadIdx.x < w) {
            sh[0][threadIdx.x] = fr_add(sh[0][threadIdx.x], sh[0][threadIdx.x + w]);
            sh[1][threadIdx.x] = fr_add(sh[1][threadIdx.x], sh[1][threadIdx.x + w]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        acc[2 * blockIdx.x] = fr_add(acc[2 * blockIdx.x], sh[0][0]);
        acc[2 * blockIdx.x + 1] = fr_add(acc[2 * blockIdx.x + 1], sh[1][0]);
    }
}

__global__ void __launch_bounds__(256) k_zkey_fill_x(uint4 *x, uint64_t n, uint64_t seed) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const Fr v = zk_rand(seed, 0, i);
        x[2 * i] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
        x[2 * i + 1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
    }
}

// section-4 entries (44 B each, 4-byte aligned) against x and rho.  An entry whose matrix, constraint or signal is out of range is
// counted and skipped before any of its fields is used as an index.
__global__ void __launch_bounds__(ZK_THREADS) k_zkey_coefs(const uint32_t *ent, uint64_t n, const uint4 *x, uint64_t n_vars, uint64_t domain,
                                                            uint64_t seed, Fr *acc, ZkeyCounters *ctr) {
    Fr s0 = fr_zero(), s1 = fr_zero();
    unsigned long long bad = 0;
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t *p = ent + 11 * e;
        const uint32_t m = p[0], c = p[1], s = p[2];
        if (m > 1 || c >= domain || s >= n_vars) { bad++; continue; }
        Fr v;
#pragma unroll
        for (int k = 0; k < 8; k++) v.l[k] = p[3 + k];
        for (int k = 0; k < 5 && fr_geq_p(v); k++) { Fr t; fr_raw_sub(t, v, fr_p()); v = t; }   // 2^256 < 6 r
        const Fr t = fr_mont(fr_mont(v, zk_load(x, s)), zk_rand(seed, 1, c));
        if (m == 0) s0 = fr_add(s0, t); else s1 = fr_add(s1, t);
    }
    if (bad) atomicAdd(&ctr->out_of_range, bad);
    zk_block_add(s0, s1, acc);
}

// rows [first, first + n) of the row side: a[k], b[k] = (A x), (B x) of row first + k (b may be null)
__global__ void __launch_bounds__(ZK_THREADS) k_zkey_rows(const uint4 *a, const uint4 *b, uint64_t first, uint64_t n, uint64_t seed, Fr *acc) {
    Fr s0 = fr_zero(), s1 = fr_zero();
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
        const Fr rho = zk_rand(seed, 1, first + k);
        s0 = fr_add(s0, fr_mont(zk_load(a, k), rho));
        if (b) s1 = fr_add(s1, fr_mont(zk_load(b, k), rho));
    }
    zk_block_add(s0, s1, acc);
}

// one block: S_M and T_M from the n_slots block slots of each side, compared under both readings
__global__ void __launch_bounds__(ZK_THREADS) k_zkey_final(const Fr *coef_acc, const Fr *row_acc, uint32_t n_slots, ZkeyCounters *ctr) {
    __shared__ Fr sh[4][ZK_THREADS];
    Fr v[4] = {fr_zero(), fr_zero(), fr_zero(), fr_zero()};
    for (uint32_t i = threadIdx.x; i < n_slots; i += ZK_THREADS)
        for (int m = 0; m < 2; m++) { v[m] = fr_add(v[m], coef_acc[2 * i + m]); v[2 + m] = fr_add(v[2 + m], row_acc[2 * i + m]); }
    for (int j = 0; j < 4; j++) sh[j][threadIdx.x] = v[j];
    __syncthreads();
    for (uint32_t w = ZK_THREADS / 2; w; w >>= 1) {
        if (threadIdx.x < w) for (int j = 0; j < 4; j++) sh[j][threadIdx.x] = fr_add(sh[j][threadIdx.x], sh[j][threadIdx.x + w]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        uint32_t match = 0, canon = 0;
        for (int m = 0; m < 2; m++) {
            if (fr_eq(sh[m][0], fr_mont(sh[2 + m][0], fr_r2()))) match |= 1u << m;
            if (fr_eq(sh[m][0], fr_from_mont(sh[2 + m][0]))) canon |= 1u << m;
        }
        ctr->match = match; ctr->match_canonical = canon;
    }
}

__device__ __forceinline__ bool zk_lt_q(const Fq &a) { return !geq_mod<FqMod>(a); }
__device__ __forceinline__ Fq zk_fq(const uint4 *p, uint64_t i) {     // element i (32 B) of a point array
    const uint4 a = p[2 * i], b = p[2 * i + 1];
    Fq r; r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}
template <class F> __device__ __forceinline__ bool zk_on_curve(const F &x, const F &y, const F &b) {
    return f_is_zero(f_sub(f_sqr(y), f_add(f_mul(f_sqr(x), x), b)));
}
__device__ __forceinline__ void zk_point(const uint4 *p, uint64_t i, const Fq &b, bool &ok, bool &ok_canonical) {
    const Fq x = zk_fq(p, 2 * i), y = zk_fq(p, 2 * i + 1);
    const bool inf = fq_is_zero(x) && fq_is_zero(y), range = zk_lt_q(x) && zk_lt_q(y);
    ok = inf || (range && zk_on_curve(x, y, b));
    ok_canonical = inf || (range && zk_on_curve(fq_to_mont(x), fq_to_mont(y), b));
}
__device__ __forceinline__ void zk_point(const uint4 *p, uint64_t i, const Fq2 &b, bool &ok, bool &ok_canonical) {
    Fq2 x, y;
    x.c0 = zk_fq(p, 4 * i); x.c1 = zk_fq(p, 4 * i + 1); y.c0 = zk_fq(p, 4 * i + 2); y.c1 = zk_fq(p, 4 * i + 3);
    const bool inf = fq2_is_zero(x) && fq2_is_zero(y);
    const bool range = zk_lt_q(x.c0) && zk_lt_q(x.c1) && zk_lt_q(y.c0) && zk_lt_q(y.c1);
    ok = inf || (range && zk_on_curve(x, y, b));
    ok_canonical = inf || (range && zk_on_curve(fq2_to_mont(x), fq2_to_mont(y), b));
}

// points [0, n) of section `section`, whose first one has index idx0 there; F = Fq (G1, 64 B) or Fq2 (G2, 128 B); b in Montgomery form
template <class F>
__global__ void __launch_bounds__(ZK_THREADS) k_zkey_points(const uint4 *pts, uint64_t n, uint32_t section, uint64_t idx0, F b, ZkeyCounters *ctr) {
    unsigned long long bad = 0, bad_c = 0, first = ~0ull;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        bool ok, ok_c;
        zk_point(pts, i, b, ok, ok_c);
        if (!ok) { bad++; first = min(first, ((unsigned long long)section << 40) | (idx0 + i)); }
        if (!ok_c) bad_c++;
    }
    if (bad) { atomicAdd(&ctr->points_bad, bad); atomicMin(&ctr->first_bad, first); }
    if (bad_c) atomicAdd(&ctr->points_bad_canonical, bad_c);
}

}  // namespace
