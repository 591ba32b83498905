// ntt.cuh -- BN254-Fr number-theoretic transforms for the Groth16 quotient (pob_r1cs_quotient, DESIGN.md §5).
//
//   k_ntt_inv  one pass of the inverse transform: decimation in frequency, natural order in, bit-reversed order out.  The last
//              pass multiplies the entry at bit-reversed position j (coefficient k = rev(j)) by g^k / n: the coset shift.
//   k_ntt_fwd  one pass of the forward transform: decimation in time, bit-reversed order in, natural order out.  The last pass of
//              the third vector can write A.B - C instead of its own values (the quotient evaluations).
//
// Data stay canonical; every constant (roots, g^k / n) is stored in Montgomery form, so fr_mont(x, c R) = x c is canonical too.
// A transform of 2^L entries runs in ceil-balanced passes (ntt_plan).  One pass cuts its blocks of N = s * 2^k entries into
// sub-transforms of 2^k entries at stride s (entries r + s i, i < 2^k); a CTA loads 2^T / 2^k of them with neighbouring r into
// shared memory, so a warp reads runs of 2^(T-k) consecutive entries, runs the k radix-2 stages there and writes them back.  For
// the inverse, a pass is the local transform followed by the inter-pass twiddle w_N^-(r rev(i)); the forward pass is its exact
// inverse up to the factor 2^k: the twiddle w_N^(r rev(i)), then the local transform.  Global memory is read and written in
// 16-byte halves, one per lane of a lane pair, so a warp's accesses cover whole 32-byte sectors (DESIGN.md §2.3).
//
// Roots: w28 = 5^((p-1) / 2^28) generates the 2^28-th roots; w_k = w28^(2^(28-k)).  Any power w28^E (E < 2^28) is the product of
// two table entries, lo[E mod 2^14] * hi[E >> 14] (512 KiB each); the local stages use w_11^t (t < 1024, 32 KiB, and its inverse).
// The coset factors g^k / n come from a second pair of tables sized for the handle's n (1 MiB at n = 2^28).  Nothing is n/2 long.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "fr_hd.h"

using namespace pob;

namespace {

const uint32_t NTT_MAX_LOG = 28;          // 2^28 | p - 1
const uint32_t NTT_TILE_LOG = 11;         // entries per CTA: 2^11 x 32 B = 64 KiB of shared memory
const uint32_t NTT_THREADS = 256;
const uint32_t NTT_TW_LOG = 14;           // w28 powers: lo / hi tables of 2^14 entries

struct NttTables {                        // device pointers, Montgomery form
    const Fr *w_lo, *w_hi;                // w28^t, w28^(t 2^14)
    const Fr *loc, *loc_inv;              // w_11^t, w_11^-t, t < 1024
    const Fr *g_lo, *g_hi;                // g^t, g^(t 2^g_log) / n
    uint32_t g_log;
};
struct NttPass {
    uint4 *x;                             // the vector, n entries as 2 x uint4 each, transformed in place
    uint32_t log_n, log_blk, log_k, log_tile;     // transform, block N = s 2^k, stages of this pass, entries per CTA
    uint32_t last;                        // inverse: apply g^rev(j) / n; forward with q != null: write q = A.B - C
    const uint4 *a, *b; uint4 *q;         // forward last pass of the C vector: A, B (canonical, natural order) and the output
    NttTables t;
};

__device__ __forceinline__ uint32_t ntt_rev(uint32_t x, uint32_t bits) { return bits ? __brev(x) >> (32 - bits) : 0u; }
__device__ __forceinline__ Fr ldg_fr(const Fr *p) {
    const uint4 lo = __ldg((const uint4 *)p), hi = __ldg((const uint4 *)p + 1);
    Fr r; r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w; r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
    return r;
}
// w28^E * R, E < 2^28
__device__ __forceinline__ Fr ntt_w28(const NttTables &t, uint32_t e) {
    return fr_mont(ldg_fr(t.w_lo + (e & ((1u << NTT_TW_LOG) - 1))), ldg_fr(t.w_hi + (e >> NTT_TW_LOG)));
}
// global entry of tile entry e = (row i, column c) of CTA `tile`: sub-transform u = tile 2^(T-k) + c, block u >> log s, r = u mod s
__device__ __forceinline__ uint64_t ntt_index(const NttPass &p, uint32_t tile, uint32_t e, uint32_t &r, uint32_t &i) {
    const uint32_t log_c = p.log_tile - p.log_k, log_s = p.log_blk - p.log_k;
    const uint64_t u = ((uint64_t)tile << log_c) | (e & ((1u << log_c) - 1));
    i = e >> log_c; r = (uint32_t)(u & ((1ull << log_s) - 1));
    return ((u >> log_s) << p.log_blk) + r + ((uint64_t)i << log_s);
}
__device__ __forceinline__ void ntt_load(const NttPass &p, uint4 *sm) {
    const uint32_t halves = 2u << p.log_tile;
    for (uint32_t hh = threadIdx.x; hh < halves; hh += blockDim.x) {
        uint32_t r, i;
        sm[hh] = p.x[2 * ntt_index(p, blockIdx.x, hh >> 1, r, i) + (hh & 1)];
    }
}
__device__ __forceinline__ void ntt_store(const NttPass &p, const uint4 *sm, uint4 *dst) {
    const uint32_t halves = 2u << p.log_tile;
    for (uint32_t hh = threadIdx.x; hh < halves; hh += blockDim.x) {
        uint32_t r, i;
        dst[2 * ntt_index(p, blockIdx.x, hh >> 1, r, i) + (hh & 1)] = sm[hh];
    }
}
// the inter-pass twiddle exponent of tile entry e as a power of w28: (r rev_k(i)) N-th roots
__device__ __forceinline__ uint32_t ntt_tw_exp(const NttPass &p, uint32_t r, uint32_t i) {
    return (uint32_t)(((uint64_t)r * ntt_rev(i, p.log_k)) << (NTT_MAX_LOG - p.log_blk)) & ((1u << NTT_MAX_LOG) - 1);
}

__global__ void __launch_bounds__(NTT_THREADS) k_ntt_inv(const NttPass p) {
    extern __shared__ uint4 sm[];
    Fr *S = (Fr *)sm;
    const uint32_t log_c = p.log_tile - p.log_k, pairs = 1u << (p.log_tile - 1);
    ntt_load(p, sm);
    __syncthreads();
    for (int q = (int)p.log_k - 1; q >= 0; q--) {                        // half size 2^q: (u, v) -> (u + v, (u - v) w_(q+1)^-j)
        for (uint32_t b = threadIdx.x; b < pairs; b += blockDim.x) {
            const uint32_t c = b & ((1u << log_c) - 1), k = b >> log_c, j = k & ((1u << q) - 1);
            const uint32_t i0 = ((k >> q) << (q + 1)) | j;
            const uint32_t e0 = (i0 << log_c) | c, e1 = ((i0 + (1u << q)) << log_c) | c;
            const Fr u = S[e0], v = S[e1];
            S[e0] = fr_add(u, v);
            const Fr d = fr_sub(u, v);
            S[e1] = j ? fr_mont(d, ldg_fr(p.t.loc_inv + (j << (10 - q)))) : d;
        }
        __syncthreads();
    }
    const bool twiddle = p.log_blk > p.log_k;
    if (twiddle || p.last) {
        for (uint32_t e = threadIdx.x; e < (1u << p.log_tile); e += blockDim.x) {
            uint32_t r, i;
            const uint64_t g = ntt_index(p, blockIdx.x, e, r, i);
            Fr f;
            if (p.last) {                                                  // coefficient rev(g) times g^rev(g) / n
                const uint32_t k = ntt_rev((uint32_t)g, p.log_n);
                f = fr_mont(ldg_fr(p.t.g_lo + (k & ((1u << p.t.g_log) - 1))), ldg_fr(p.t.g_hi + (k >> p.t.g_log)));
            } else {
                const uint32_t ex = ntt_tw_exp(p, r, i);
                if (!ex) continue;
                f = ntt_w28(p.t, (1u << NTT_MAX_LOG) - ex);
            }
            S[e] = fr_mont(S[e], f);
        }
        __syncthreads();
    }
    ntt_store(p, sm, p.x);
}

__global__ void __launch_bounds__(NTT_THREADS) k_ntt_fwd(const NttPass p) {
    extern __shared__ uint4 sm[];
    Fr *S = (Fr *)sm;
    const uint32_t log_c = p.log_tile - p.log_k, pairs = 1u << (p.log_tile - 1);
    ntt_load(p, sm);
    __syncthreads();
    if (p.log_blk > p.log_k) {
        for (uint32_t e = threadIdx.x; e < (1u << p.log_tile); e += blockDim.x) {
            uint32_t r, i;
            ntt_index(p, blockIdx.x, e, r, i);
            const uint32_t ex = ntt_tw_exp(p, r, i);
            if (ex) S[e] = fr_mont(S[e], ntt_w28(p.t, ex));
        }
        __syncthreads();
    }
    for (uint32_t q = 0; q < p.log_k; q++) {                            // half size 2^q: (u, v) -> (u + v w_(q+1)^j, u - v w_(q+1)^j)
        for (uint32_t b = threadIdx.x; b < pairs; b += blockDim.x) {
            const uint32_t c = b & ((1u << log_c) - 1), k = b >> log_c, j = k & ((1u << q) - 1);
            const uint32_t i0 = ((k >> q) << (q + 1)) | j;
            const uint32_t e0 = (i0 << log_c) | c, e1 = ((i0 + (1u << q)) << log_c) | c;
            const Fr u = S[e0], v = j ? fr_mont(S[e1], ldg_fr(p.t.loc + (j << (10 - q)))) : S[e1];
            S[e0] = fr_add(u, v);
            S[e1] = fr_sub(u, v);
        }
        __syncthreads();
    }
    if (p.q) {                                                            // q = A.B - C: (A B R^-1) R^2 R^-1 = A B
        const Fr r2 = fr_r2();
        for (uint32_t e = threadIdx.x; e < (1u << p.log_tile); e += blockDim.x) {
            uint32_t r, i;
            const uint64_t g = ntt_index(p, blockIdx.x, e, r, i);
            const Fr A = ((const Fr *)p.a)[g], B = ((const Fr *)p.b)[g];     // plain loads: q may be A's own buffer
            S[e] = fr_sub(fr_mont(fr_mont(A, B), r2), S[e]);
        }
        __syncthreads();
        ntt_store(p, sm, p.q);
    } else {
        ntt_store(p, sm, p.x);
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------------------
// stages per pass of a 2^L transform with 2^T-entry tiles, in the order of the inverse transform (the forward one runs them in
// reverse): as few passes as keep every pass but the contiguous last one at <= T - 2 stages (runs of >= 4 entries = 128 bytes),
// balanced, the largest last.  A balanced pass above T - 2 (only 10 + 10 at L = 20 for T = 11) gives its excess to the last pass,
// which still has at most T stages because the pass count allows it.
static std::vector<uint32_t> ntt_plan(uint32_t L, uint32_t T) {
    uint32_t q = 0;
    while (L > T + q * (T - 2)) q++;
    const uint32_t P = q + 1;
    std::vector<uint32_t> k(P, L / P);
    for (uint32_t i = 0; i < L % P; i++) k[P - 1 - i]++;
    for (uint32_t i = 0; i + 1 < P; i++)
        if (k[i] > T - 2) { k[P - 1] += k[i] - (T - 2); k[i] = T - 2; }
    return k;
}

static Fr fr_pow_m(Fr base_m, const Fr &e) {                              // Montgomery form in and out
    Fr r = fr_to_mont(fr_from_u64(1));
    for (int i = 255; i >= 0; i--) { r = fr_mont(r, r); if (fr_bit(e, (unsigned)i)) r = fr_mont(r, base_m); }
    return r;
}
// w28 = 5^((p - 1) >> 28), Montgomery form
static Fr ntt_w28_host() {
    Fr e = fr_p(); e.l[0] -= 1;                                            // p - 1 (p is odd)
    for (int k = 0; k < 28; k++) fr_shr1(e);
    return fr_pow_m(fr_to_mont(fr_from_u64(5)), e);
}
static void ntt_powers(std::vector<Fr> &out, size_t count, const Fr &step_m, const Fr &first_m) {
    out.resize(count);
    Fr cur = first_m;
    for (size_t i = 0; i < count; i++) { out[i] = cur; cur = fr_mont(cur, step_m); }
}
// the coset shift of a 2^L domain, Montgomery form: w_(L+1) (so g^n = -1) for L < 28; 25 (snarkjs's Fr.shift = nqr^2) at L = 28
static Fr ntt_shift_host(uint32_t L) {
    if (L >= NTT_MAX_LOG) return fr_to_mont(fr_from_u64(25));
    Fr g = ntt_w28_host();
    for (uint32_t k = L + 1; k < NTT_MAX_LOG; k++) g = fr_mont(g, g);
    return g;
}

// the tables of NttTables for a 2^L domain, on the host, Montgomery form
struct NttHostTables {
    std::vector<Fr> w_lo, w_hi, loc, loc_inv, g_lo, g_hi;
    uint32_t g_log;
};
static NttHostTables ntt_host_tables(uint32_t L) {
    NttHostTables H;
    const Fr one = fr_to_mont(fr_from_u64(1)), w28 = ntt_w28_host();
    Fr w14 = w28, w11 = w28;
    for (uint32_t k = 0; k < NTT_TW_LOG; k++) w14 = fr_mont(w14, w14);
    for (uint32_t k = 0; k < NTT_MAX_LOG - NTT_TILE_LOG; k++) w11 = fr_mont(w11, w11);
    ntt_powers(H.w_lo, 1u << NTT_TW_LOG, w28, one);
    ntt_powers(H.w_hi, 1u << (NTT_MAX_LOG - NTT_TW_LOG), w14, one);
    ntt_powers(H.loc, 1u << (NTT_TILE_LOG - 1), w11, one);
    ntt_powers(H.loc_inv, 1u << (NTT_TILE_LOG - 1), fr_to_mont(fr_inv(fr_from_mont(w11))), one);
    const Fr g = ntt_shift_host(L);
    Fr gs = g;
    H.g_log = (L + 1) / 2;
    for (uint32_t k = 0; k < H.g_log; k++) gs = fr_mont(gs, gs);
    ntt_powers(H.g_lo, 1ull << H.g_log, g, one);
    ntt_powers(H.g_hi, 1ull << (L - H.g_log), gs, fr_to_mont(fr_inv(fr_from_u64(1ull << L))));   // g^(t 2^g_log) / n
    return H;
}

// once per process and device, before the first launch: both kernels use 32 << NTT_TILE_LOG bytes of dynamic shared memory
static cudaError_t ntt_init_kernels() {
    const int smem = 32 << NTT_TILE_LOG;
    cudaError_t e = cudaFuncSetAttribute(k_ntt_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_ntt_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    return e;
}

// enqueue the inverse transform of the 2^L entries at x (2 uint4 each) with 2^T-entry tiles, natural order in, bit-reversed
// order out; its last pass multiplies coefficient k by g^k / n
static cudaError_t ntt_inverse_coset(uint4 *x, uint32_t L, uint32_t T, const NttTables &t, cudaStream_t st) {
    const std::vector<uint32_t> k = ntt_plan(L, T);
    const uint32_t P = (uint32_t)k.size(), grid = (uint32_t)((1ull << L) >> T), smem = 32u << T;
    uint32_t blk = L;
    for (uint32_t i = 0; i < P; i++) {
        const NttPass p{x, L, blk, k[i], T, i + 1 == P, nullptr, nullptr, nullptr, t};
        k_ntt_inv<<<grid, NTT_THREADS, smem, st>>>(p);
        blk -= k[i];
    }
    return cudaGetLastError();
}

// enqueue the forward transform of x, bit-reversed order in, natural order out; with q set, its last pass writes q = A.B - x's
// values instead of them (A, B canonical, natural order; q may be a)
static cudaError_t ntt_forward(uint4 *x, uint32_t L, uint32_t T, const NttTables &t, cudaStream_t st,
                               const uint4 *a = nullptr, const uint4 *b = nullptr, uint4 *q = nullptr) {
    const std::vector<uint32_t> k = ntt_plan(L, T);
    const uint32_t P = (uint32_t)k.size(), grid = (uint32_t)((1ull << L) >> T), smem = 32u << T;
    uint32_t blk = 0;
    for (uint32_t i = P; i-- > 0;) {
        blk += k[i];
        NttPass p{x, L, blk, k[i], T, 0, nullptr, nullptr, nullptr, t};
        if (q && i == 0) { p.last = 1; p.a = a; p.b = b; p.q = q; }
        k_ntt_fwd<<<grid, NTT_THREADS, smem, st>>>(p);
    }
    return cudaGetLastError();
}

}  // namespace
