// msm.cuh -- BN254 multi-exponentiation sum_i [s_i] P_i over G1 (pob_msm_g1) or G2 (pob_msm_g2), DESIGN.md §5: Pippenger with
// signed c-bit digits.  One pipeline for both groups: the kernels that carry points are templates over a curve trait (MsmCurve<F>,
// F = Fq or Fq2: point types, formulas, loads and stores); k_msm_digits and k_msm_scan see only scalars and are shared.
//
// Per window j (one after another, so that the scratch holds one window's grouping):
//   k_msm_digits<false>  signed digit d of every scalar (s mod r first); a histogram of |d| - 1 (the bucket).  d = 0 writes nothing.
//   k_msm_scan           bucket offsets (one CTA; also resets the counts to the offsets, as the scatter's cursors).
//   k_msm_digits<true>   the same digits again, each nonzero one written as (point index | sign << 31) at its bucket's cursor:
//                        a counting sort, so the list is grouped by bucket.  Warp-aggregated atomics: lanes with equal buckets
//                        take one atomic between them (a 0/1 witness puts almost every entry into bucket 0 of window 0).
//   k_msm_sum<Bases>     bucket sums as a segmented reduction over the grouped list, cut into T equal chunks that ignore bucket
//                        boundaries.  A bucket that starts and ends inside one chunk is complete there and is written directly;
//                        the first and last segments of every chunk go out as (bucket, partial sum) pairs -- in bucket order,
//                        so the same kernel (k_msm_sum<Partials>, 32 pairs per thread) reduces them again, until one thread
//                        takes the last <= 64 pairs.  A bucket that holds every point is thus summed by all T threads, then by
//                        T / 16, ..., not by one.
//   k_msm_reduce         sum_b (b + 1) B_b over the window's buckets: G threads take 16 buckets each (running sums from the top,
//                        then + lo * segment sum), and the G partials go through the k_msm_sum<Partials> cascade into W_j.
// Then k_msm_final: Horner over the windows (c doublings each) and one conversion to canonical affine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include "fq2_hd.h"

using namespace pob;

namespace {

const uint32_t MSM_THREADS = 128;
const uint32_t MSM_SCALAR_BITS = 255;     // signed digits of s < r < 2^254 need one bit above r's 254 (the last carry)
const uint32_t MSM_PAIRS = 32;            // partial sums a thread takes in the second and later levels of the cascade
const uint32_t MSM_FINAL = 64;            // the last level: one thread takes what is left
const uint32_t MSM_SEG = 16;              // buckets per thread of the bucket reduction
const uint32_t MSM_NONE = 0xffffffffu;    // key of an empty partial (sorts last, names no bucket)
const uint64_t MSM_MAX_N = 1ull << 31;    // a grouped entry is a 31-bit point index and a sign bit

// window size c (bits per digit) for n points: log2(n) - 3, within [4, 16].  A window costs n additions into its 2^(c-1) buckets
// plus about 2 * 2^(c-1) for their reduction; 255 / c windows.  16 keeps one window's buckets at 4 MiB.
static uint32_t msm_window_bits(uint64_t n) {
    uint32_t lg = 0;
    while (lg < 63 && (2ull << lg) <= n) lg++;
    return std::min<uint32_t>(16, std::max<uint32_t>(4, lg > 3 ? lg - 3 : 0));
}
// chunks (threads) of the first bucket-sum level: about 16 grouped entries per thread for n <= 2^20, then at most 2^16 threads
static uint32_t msm_chunks(uint64_t n) { return (uint32_t)std::min<uint64_t>(1u << 16, std::max<uint64_t>(32, n / 16)); }

// a curve of the multi-exponentiation: points over F (G1: Fq, G2: Fq2), the formulas of fq_hd.h, and loads / stores of F as uint4s
template <class F> struct MsmCurve {
    typedef F Field;
    typedef Aff<F> Affine;
    typedef Xyzz<F> Point;
    static const uint32_t FIELD_U4 = sizeof(F) / 16;                  // uint4s per element: 2 (Fq) or 4 (Fq2)
    static const uint32_t AFF_BYTES = 2 * sizeof(F);                   // one affine base / output point
};
typedef MsmCurve<Fq> MsmG1;
typedef MsmCurve<Fq2> MsmG2;

struct MsmLayout {                        // byte offsets into the caller's work buffer
    uint32_t c, windows, buckets, chunks, seg_threads;
    uint64_t idx, cnt, offs, bkt, keys_a, pts_a, keys_b, pts_b, win, bytes;
};
template <class C> static MsmLayout msm_layout(uint64_t n) {
    typedef typename C::Point Pt;
    MsmLayout L;
    L.c = msm_window_bits(n);
    L.windows = (MSM_SCALAR_BITS + L.c - 1) / L.c;
    L.buckets = 1u << (L.c - 1);
    L.chunks = msm_chunks(n);
    L.seg_threads = (L.buckets + MSM_SEG - 1) / MSM_SEG;
    const uint64_t pa = std::max<uint64_t>(2ull * L.chunks, L.seg_threads);
    const uint64_t pb = 2 * ((pa + MSM_PAIRS - 1) / MSM_PAIRS);
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t o = at; at += (bytes + 255) & ~255ull; return o; };
    L.idx = take(4 * n);
    L.cnt = take(4ull * (L.buckets + 1));
    L.offs = take(4ull * (L.buckets + 1));
    L.bkt = take(sizeof(Pt) * (uint64_t)L.buckets);
    L.keys_a = take(4 * pa);
    L.pts_a = take(sizeof(Pt) * pa);
    L.keys_b = take(4 * pb);
    L.pts_b = take(sizeof(Pt) * pb);
    L.win = take(sizeof(Pt) * (uint64_t)L.windows);
    L.bytes = at;
    return L;
}

__device__ __forceinline__ Fq msm_ld_fq(const uint4 *p) {
    const uint4 lo = __ldg(p), hi = __ldg(p + 1);
    Fq r; r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w; r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
    return r;
}
__device__ __forceinline__ void msm_st_fq(uint4 *p, const Fq &a) {
    p[0] = make_uint4(a.l[0], a.l[1], a.l[2], a.l[3]);
    p[1] = make_uint4(a.l[4], a.l[5], a.l[6], a.l[7]);
}
__device__ __forceinline__ void msm_ld(const uint4 *p, Fq &r) { r = msm_ld_fq(p); }
__device__ __forceinline__ void msm_ld(const uint4 *p, Fq2 &r) { r.c0 = msm_ld_fq(p); r.c1 = msm_ld_fq(p + 2); }
__device__ __forceinline__ void msm_st(uint4 *p, const Fq &a) { msm_st_fq(p, a); }
__device__ __forceinline__ void msm_st(uint4 *p, const Fq2 &a) { msm_st_fq(p, a.c0); msm_st_fq(p + 2, a.c1); }
template <class F> __device__ __forceinline__ Xyzz<F> msm_ld_xyzz(const Xyzz<F> *p) {
    const uint4 *q = (const uint4 *)p;
    const uint32_t u = MsmCurve<F>::FIELD_U4;
    Xyzz<F> r; msm_ld(q, r.x); msm_ld(q + u, r.y); msm_ld(q + 2 * u, r.zz); msm_ld(q + 3 * u, r.zzz);
    return r;
}
template <class F> __device__ __forceinline__ void msm_st_xyzz(Xyzz<F> *p, const Xyzz<F> &a) {
    uint4 *q = (uint4 *)p;
    const uint32_t u = MsmCurve<F>::FIELD_U4;
    msm_st(q, a.x); msm_st(q + u, a.y); msm_st(q + 2 * u, a.zz); msm_st(q + 3 * u, a.zzz);
}

// signed digit of window j of s mod r: s = sum_j d_j 2^(c j), d_j in (-2^(c-1), 2^(c-1)]
__device__ __forceinline__ int32_t msm_digit(const uint4 *scalar, uint32_t c, uint32_t j) {
    const uint4 lo = __ldg(scalar), hi = __ldg(scalar + 1);
    Fr s; s.l[0] = lo.x; s.l[1] = lo.y; s.l[2] = lo.z; s.l[3] = lo.w; s.l[4] = hi.x; s.l[5] = hi.y; s.l[6] = hi.z; s.l[7] = hi.w;
#pragma unroll 1
    for (int k = 0; k < 5; k++) {                                      // 2^256 < 6 r
        if (!fr_geq_p(s)) break;
        Fr t; fr_raw_sub(t, s, fr_p()); s = t;
    }
    const uint32_t mask = (1u << c) - 1, half = 1u << (c - 1);
    uint32_t carry = 0;
    int32_t d = 0;
#pragma unroll 1
    for (uint32_t w = 0; w <= j; w++) {
        const uint32_t v = (s.l[0] & mask) + carry;
        carry = v > half;
        d = (int32_t)v - (carry ? (int32_t)(1u << c) : 0);
#pragma unroll
        for (int k = 0; k < 7; k++) s.l[k] = (s.l[k] >> c) | (s.l[k + 1] << (32 - c));
        s.l[7] >>= c;
    }
    return d;
}

// kScatter = false: cnt[bucket] += 1 per nonzero digit.  true: idx[cnt[bucket]++] = point | sign << 31
template <bool kScatter>
__global__ void __launch_bounds__(256) k_msm_digits(const uint4 *scalars, uint64_t n, uint32_t c, uint32_t j, uint32_t *cnt, uint32_t *idx) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {   // warp-uniform trip count
        const uint64_t i = base + lane;
        int32_t d = i < n ? msm_digit(scalars + 2 * i, c, j) : 0;
        const uint32_t has = __ballot_sync(0xffffffffu, d != 0);
        if (d != 0) {
            const uint32_t key = (uint32_t)(d < 0 ? -d : d) - 1;
            const uint32_t peers = __match_any_sync(has, key);
            const uint32_t leader = __ffs(peers) - 1;
            uint32_t at = 0;
            if (lane == leader) at = atomicAdd(cnt + key, (uint32_t)__popc(peers));
            at = __shfl_sync(peers, at, leader) + __popc(peers & ((1u << lane) - 1));
            if (kScatter) idx[at] = (uint32_t)i | (d < 0 ? 0x80000000u : 0u);
        }
    }
}

// one CTA of 1024 threads: offs[b] = sum_{b' < b} cnt[b'] for b <= K, and cnt[b] = offs[b] (the scatter's cursors)
__global__ void __launch_bounds__(1024) k_msm_scan(uint32_t *cnt, uint32_t K, uint32_t *offs) {
    __shared__ uint32_t part[1024];
    const uint32_t per = (K + 1023) / 1024, lo = threadIdx.x * per, hi = min(lo + per, K);
    uint32_t s = 0;
    for (uint32_t b = lo; b < hi; b++) s += cnt[b];
    part[threadIdx.x] = s;
    __syncthreads();
    for (uint32_t d = 1; d < 1024; d <<= 1) {                         // inclusive scan (Hillis-Steele)
        const uint32_t v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = part[threadIdx.x] - s;
    for (uint32_t b = lo; b < hi; b++) { const uint32_t v = cnt[b]; offs[b] = run; cnt[b] = run; run += v; }
    if (threadIdx.x == 1023) offs[K] = part[1023];
}

// the entries of the first bucket-sum level: the grouped list of one window, keys from the bucket offsets
template <class C> struct MsmBases {
    typedef C Curve;
    const uint32_t *offs, *idx;
    const uint4 *bases;                                                // n affine points, 2 FIELD_U4 uint4s each
    uint32_t K;
    __device__ uint32_t count() const { return offs[K]; }
    __device__ uint32_t first_key(uint32_t p) const {                  // the bucket b with offs[b] <= p < offs[b + 1]
        uint32_t lo = 0, hi = K;                                       // offs[lo] <= p < offs[hi]
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) / 2; if (offs[mid] <= p) lo = mid; else hi = mid; }
        return lo;
    }
    __device__ uint32_t next_key(uint32_t b, uint32_t p) const { while (offs[b + 1] <= p) b++; return b; }
    __device__ void add(typename C::Point &acc, uint32_t p) const {
        const uint32_t e = __ldg(idx + p);
        const uint4 *q = bases + 2 * C::FIELD_U4 * (uint64_t)(e & 0x7fffffffu);
        typename C::Affine a; msm_ld(q, a.x); msm_ld(q + C::FIELD_U4, a.y);
        if (e >> 31) a = pt_aff_neg(a);
        acc = pt_add_aff(acc, a);
    }
};
// the entries of a later level: (key, partial sum) pairs, keys ascending, MSM_NONE last
template <class C> struct MsmPartials {
    typedef C Curve;
    const uint32_t *keys;
    const typename C::Point *pts;
    uint32_t m;
    __device__ uint32_t count() const { return m; }
    __device__ uint32_t first_key(uint32_t p) const { return keys[p]; }
    __device__ uint32_t next_key(uint32_t, uint32_t p) const { return keys[p]; }
    __device__ void add(typename C::Point &acc, uint32_t p) const { acc = pt_add(acc, msm_ld_xyzz(pts + p)); }
};

// one level of the segmented reduction: T threads, thread t takes entries [t L, (t + 1) L), L = ceil(count / T).  A segment
// (run of one key) that neither starts nor ends the chunk is a whole bucket: out[key] = its sum.  The first segment goes to pair
// 2t, the last to pair 2t + 1 (pair 2t + 1 is (key, O) when the chunk has one segment, both are (MSM_NONE, O) when it is empty).
// With pkey == nullptr (the last level, T = 1) every segment is written to out.  Keys >= nb are not written.
template <class Src>
__global__ void __launch_bounds__(MSM_THREADS) k_msm_sum(Src src, uint32_t T, uint32_t nb, typename Src::Curve::Point *out, uint32_t *pkey,
                                                        typename Src::Curve::Point *ppt) {
    typedef typename Src::Curve::Field F;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint32_t m = src.count(), L = (uint32_t)(((uint64_t)m + T - 1) / T);
    const uint32_t start = (uint32_t)min((uint64_t)t * L, (uint64_t)m), end = (uint32_t)min((uint64_t)start + L, (uint64_t)m);
    if (start >= end) {
        if (pkey) { pkey[2 * t] = pkey[2 * t + 1] = MSM_NONE; msm_st_xyzz(ppt + 2 * t, pt_inf<F>()); msm_st_xyzz(ppt + 2 * t + 1, pt_inf<F>()); }
        return;
    }
    uint32_t b = src.first_key(start);
    bool first = true;
    Xyzz<F> acc = pt_inf<F>();
    for (uint32_t p = start; p < end; p++) {
        const uint32_t k = src.next_key(b, p);
        if (k != b) {
            if (first && pkey) { pkey[2 * t] = b; msm_st_xyzz(ppt + 2 * t, acc); }
            else if (b < nb) msm_st_xyzz(out + b, acc);
            first = false; b = k; acc = pt_inf<F>();
        }
        src.add(acc, p);
    }
    if (!pkey) { if (b < nb) msm_st_xyzz(out + b, acc); return; }
    if (first) { pkey[2 * t] = b; msm_st_xyzz(ppt + 2 * t, acc); acc = pt_inf<F>(); }
    pkey[2 * t + 1] = b; msm_st_xyzz(ppt + 2 * t + 1, acc);
}

// thread g: sum_{b in [lo, lo + S)} (b + 1) B_b = sum (b - lo + 1) B_b (running sums from the top) + lo * sum B_b, as pair (0, .)
template <class C>
__global__ void __launch_bounds__(MSM_THREADS) k_msm_reduce(const typename C::Point *bkt, uint32_t K, uint32_t G, uint32_t *pkey, typename C::Point *ppt) {
    typedef typename C::Field F;
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const uint32_t lo = g * MSM_SEG, hi = min(lo + MSM_SEG, K);
    Xyzz<F> run = pt_inf<F>(), acc = pt_inf<F>();
    for (uint32_t b = hi; b-- > lo;) { run = pt_add(run, msm_ld_xyzz(bkt + b)); acc = pt_add(acc, run); }
    pkey[g] = 0;
    msm_st_xyzz(ppt + g, pt_add(acc, pt_mul_u32(run, lo)));
}

// sum_j 2^(c j) W_j, then canonical affine x, y into out (C::AFF_BYTES: 64 bytes for G1, 128 for G2)
template <class C>
__global__ void k_msm_final(const typename C::Point *win, uint32_t W, uint32_t c, uint4 *out) {
    typedef typename C::Field F;
    Xyzz<F> acc = pt_inf<F>();
    for (uint32_t j = W; j-- > 0;) {
        if (!pt_is_inf(acc)) for (uint32_t k = 0; k < c; k++) acc = pt_dbl(acc);
        acc = pt_add(acc, msm_ld_xyzz(win + j));
    }
    const Aff<F> a = pt_to_affine_canonical(acc);
    msm_st(out, a.x); msm_st(out + C::FIELD_U4, a.y);
}

// reduce m (key, sum) pairs at (ka, pa) into out[key < nb], ping-ponging with (kb, pb)
template <class C>
static void msm_cascade(uint32_t m, uint32_t nb, typename C::Point *out, uint32_t *ka, typename C::Point *pa, uint32_t *kb, typename C::Point *pb,
                        cudaStream_t st) {
    while (m > MSM_FINAL) {
        const uint32_t T = (m + MSM_PAIRS - 1) / MSM_PAIRS;
        k_msm_sum<MsmPartials<C>><<<(T + MSM_THREADS - 1) / MSM_THREADS, MSM_THREADS, 0, st>>>(MsmPartials<C>{ka, pa, m}, T, nb, out, kb, pb);
        std::swap(ka, kb); std::swap(pa, pb);
        m = 2 * T;
    }
    k_msm_sum<MsmPartials<C>><<<1, 1, 0, st>>>(MsmPartials<C>{ka, pa, m}, 1, nb, out, nullptr, nullptr);
}

// enqueue the whole multi-exponentiation on st; work holds msm_layout<C>(n).bytes, out C::AFF_BYTES
template <class C>
static cudaError_t msm_enqueue(const uint4 *bases, const uint4 *scalars, uint64_t n, uint4 *out, uint8_t *work, uint32_t n_sms, cudaStream_t st) {
    typedef typename C::Point Pt;
    const MsmLayout L = msm_layout<C>(n);
    uint32_t *idx = (uint32_t *)(work + L.idx), *cnt = (uint32_t *)(work + L.cnt), *offs = (uint32_t *)(work + L.offs);
    uint32_t *ka = (uint32_t *)(work + L.keys_a), *kb = (uint32_t *)(work + L.keys_b);
    Pt *bkt = (Pt *)(work + L.bkt), *pa = (Pt *)(work + L.pts_a), *pb = (Pt *)(work + L.pts_b), *win = (Pt *)(work + L.win);
    const unsigned dgrid = (unsigned)std::min<uint64_t>((n + 255) / 256, 16ull * n_sms);
    const unsigned sgrid = (L.chunks + MSM_THREADS - 1) / MSM_THREADS;
    for (uint32_t j = 0; j < L.windows; j++) {
        cudaError_t e = cudaMemsetAsync(cnt, 0, 4ull * (L.buckets + 1), st);
        if (e == cudaSuccess) e = cudaMemsetAsync(bkt, 0, sizeof(Pt) * (uint64_t)L.buckets, st);     // O everywhere
        if (e != cudaSuccess) return e;
        k_msm_digits<false><<<dgrid, 256, 0, st>>>(scalars, n, L.c, j, cnt, nullptr);
        k_msm_scan<<<1, 1024, 0, st>>>(cnt, L.buckets, offs);
        k_msm_digits<true><<<dgrid, 256, 0, st>>>(scalars, n, L.c, j, cnt, idx);
        k_msm_sum<MsmBases<C>><<<sgrid, MSM_THREADS, 0, st>>>(MsmBases<C>{offs, idx, bases, L.buckets}, L.chunks, L.buckets, bkt, ka, pa);
        msm_cascade<C>(2 * L.chunks, L.buckets, bkt, ka, pa, kb, pb, st);
        k_msm_reduce<C><<<(L.seg_threads + MSM_THREADS - 1) / MSM_THREADS, MSM_THREADS, 0, st>>>(bkt, L.buckets, L.seg_threads, ka, pa);
        msm_cascade<C>(L.seg_threads, 1, win + j, ka, pa, kb, pb, st);
    }
    k_msm_final<C><<<1, 1, 0, st>>>(win, L.windows, L.c, out);
    return cudaGetLastError();
}

}  // namespace
