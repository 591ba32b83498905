// kernels.cuh -- device code (sm_90a) of the batched witness generator; included by pob_b200.cu only.
//
//   k_eval    one thread-block cluster (1, 2, 4 or 8 CTAs) per proof instance: runs the levelised witness program over the
//             instance store, levels separated by a cluster barrier.  Thread ops: BN254-Fr FMA / IsZero / inverse / div-mod /
//             byte packing / constraint checks (vm_exec.h; field arithmetic in fr_hd.h: inline-PTX Montgomery product, carry-chain
//             add / sub; two 128-bit accesses per value slot).  Warp ops: one Keccak absorb per warp, state lane l held by
//             thread l, Theta column parities / D, RhoPi lane walk and Chi neighbours exchanged with warp shuffles; every
//             intermediate lane word the bit-level circuit exposes (utils/keccak.circom:58-297) is written to the store
//             (238 words per round).  Poseidon permutations, one warp each, cut into POS_SEGMENTS segments over consecutive levels
//             (state element j in Montgomery form on lane j, Mix/MixS via shuffles; round constants and MDS matrices staged in
//             shared memory by TMA).  Prefix sums by warp scan.  IsZero inverse hints: table lookups in their level for small
//             inputs; the ones that need a field inversion are batch-inverted (one inversion per worker thread) by a state machine
//             that advances INV_STEPS iterations per level.
//   k_expand_round / k_expand_codes  the HBM-bound kernels: materialise every witness entry as a 32-byte little-endian
//             field element, one 16-byte half per thread and 128-bit store (STG.E.128), so that a warp's store covers 512
//             contiguous bytes.  Algorithmic bytes = 32 * n_signals per instance (6.909 GB for main_proof_of_burn).
//             KeccakfRound blocks (95.8 %) are driven by 8-byte group descriptors and the round's lane words, everything
//             else by one 32-bit code per entry; both kernels stage their tables in shared memory with TMA bulk copies
//             (cp.async.bulk + mbarrier).
//   k_check_eq / k_check_kc / k_check_r1  every constraint of the circuit evaluated against a resident witness (cons_check.h).
//   k_check_rounds  layout-independent check of every KeccakfRound block (textbook round on its in/out signals).
//   k_r1cs_products  A.w, B.w, C.w of a window of `.r1cs` rows (r1cs.h row plan) against a resident witness, for a GPU prover.
//   k_digest  64-bit digest of a materialised witness (parity tests at full size; the built-in on-GPU consumer).
//   k_pow_grind  proof-of-work burn-key search (the step before the path): one candidate key per thread.
#pragma once
#include <cuda_runtime.h>
#include "vm_exec.h"
#include "cons_check.h"

using namespace pob;

namespace {

// Keccak tables in constant memory: a constexpr array inside a device function is rebuilt on the thread's stack at every use
// (ptxas: 26 STL.128 + 3 dependent LDL per Keccak round), which tripled the latency of an absorb.
__constant__ uint64_t c_keccak_rc[24] = {
    0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808AULL, 0x8000000080008000ULL, 0x000000000000808BULL,
    0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008AULL, 0x0000000000000088ULL,
    0x0000000080008009ULL, 0x000000008000000AULL, 0x000000008000808BULL, 0x800000000000008BULL, 0x8000000000008089ULL,
    0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800AULL, 0x800000008000000AULL,
    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};                        // keccak.circom:253-262
__constant__ int c_keccak_rot[25] = {1, 10, 7, 11, 17, 18, 3, 5, 16, 8, 21, 24, 4, 15, 23, 19, 13, 12, 2, 20, 14, 22, 9, 6, 1};     // RhoPi lane walk, keccak.circom:195
__constant__ int c_keccak_inv_rot[25] = {0, 23, 17, 5, 11, 6, 22, 1, 8, 21, 0, 2, 16, 15, 19, 12, 7, 3, 4, 14, 18, 9, 20, 13, 10};  // i such that rot[i + 1] == L  (L = 1..24)

// One Absorb (utils/keccak.circom:304-323) by one warp; lane l < 25 owns state lane l.
__device__ void absorb_warp(uint64_t *W, const AbsorbOp op) {
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const bool act = lane < 25;
    const int l = act ? lane : 0;
    uint64_t st = (act && op.s_idx != NONE_IDX) ? W[op.s_idx + l] : 0ull;
    if (lane < 17) st ^= W[op.blk_idx + lane];
    if (act) W[op.out_idx + l] = st;
    const int col = l % 5;
    // lane constants of the round (hoisted: nothing below the loop header depends on memory except the round constant)
    const int i = lane < 24 ? lane : 0;
    const int rot_src = c_keccak_rot[i], shl = keccak_shl(i), rot_dst = c_keccak_inv_rot[l], cb_src = chi_b(l), cc_src = chi_c(l);
#pragma unroll 1
    for (int r = 0; r < 24; r++) {
        const uint64_t rc = c_keccak_rc[r];
        uint64_t *B = W + op.out_idx + RW * r;
        // Theta: Xor5 chain of my column (all lanes of a column compute it redundantly; lanes 0..4 store it)
        uint64_t v0 = __shfl_sync(FULL, st, col), v1 = __shfl_sync(FULL, st, col + 5), v2 = __shfl_sync(FULL, st, col + 10),
                 v3 = __shfl_sync(FULL, st, col + 15), v4 = __shfl_sync(FULL, st, col + 20);
        uint64_t x0 = v0 ^ v1, x1 = x0 ^ v2, x2 = x1 ^ v3, c = x2 ^ v4;
        if (lane < 5) { B[rw_x5(lane, 0)] = x0; B[rw_x5(lane, 1)] = x1; B[rw_x5(lane, 2)] = x2; B[rw_x5(lane, 3)] = c; }
        // D(i) = c[(i+4)%5] ^ rotl(c[(i+1)%5], 1)
        uint64_t ca = __shfl_sync(FULL, c, (col + 1) % 5), cb = __shfl_sync(FULL, c, (col + 4) % 5);
        uint64_t s0 = ca << 1, s1 = ca >> 63, so = s0 | s1, d = cb ^ so;
        if (lane < 5) { B[rw_dd(lane, 0)] = s0; B[rw_dd(lane, 1)] = s1; B[rw_dd(lane, 2)] = so; B[rw_dd(lane, 3)] = d; }
        uint64_t th = st ^ d;
        if (act) B[rw_th(l)] = th;
        // RhoPi: lane i < 24 performs step i on theta[rot[i]], the result belongs to lane rot[i+1]
        uint64_t a = __shfl_sync(FULL, th, rot_src);
        uint64_t a0 = a >> (64 - shl), a1 = a << shl, ro = a0 | a1;
        if (lane < 24) { B[rw_rp(lane, 0)] = a0; B[rw_rp(lane, 1)] = a1; B[rw_rp(lane, 2)] = ro; }
        uint64_t rp = __shfl_sync(FULL, ro, rot_dst);
        if (lane == 0) rp = th;
        // Chi
        uint64_t vb = __shfl_sync(FULL, rp, cb_src), vc = __shfl_sync(FULL, rp, cc_src);
        uint64_t nb = ~vb, bc = nb & vc, ch = rp ^ bc;
        if (act) { B[rw_ch(l, 0)] = nb; B[rw_ch(l, 1)] = bc; B[rw_ch(l, 2)] = ch; }
        // Iota
        if (lane == 0) { B[RW_RC] = rc; ch ^= rc; }
        if (act) B[rw_out(l)] = ch;
        st = ch;
    }
}

// ---- one Poseidon permutation by one warp (circomlib/circuits/poseidon.circom:67-196) ---------------------------
// Lane j < t owns state element j in Montgomery form; Mix / MixS exchange elements with warp shuffles; every
// intermediate signal is converted back to canonical form and written to its slot (layout: program.h PosLayout).
__device__ __forceinline__ Fr shfl_fr(const Fr &v, int src) {
    Fr r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.l[i] = __shfl_sync(0xffffffffu, v.l[i], src);
    return r;
}
__device__ void poseidon_warp(const VmCtx &x, const PoseidonOp op, const Fr *pk) {
    const int lane = threadIdx.x & 31;
    const uint32_t t = op.t; const PosLayout L = pos_layout(t);
    const bool act = (uint32_t)lane < t; const uint32_t j = act ? (uint32_t)lane : 0u;
    const Fr *K = pk + op.koff;
    uint64_t *V = x.U + x.val_base + 4ull * op.base;
    const uint32_t Q = pos_steps(L);
    // values are parked in their slots in MONTGOMERY form until the end of the segment that wrote them (nothing but Poseidon segments
    // reads them before the last segment is through): no conversion sits on the dependency chain of the 65 rounds
    auto put = [&](uint32_t off, const Fr &m) { if (act) vm_store_val(V + 4ull * off, m); };
    Fr s;
    uint32_t q = op.q0;
    if (q == 0) { s = fr_add(fr_to_mont(vm_load(x, x.aux[op.in_aux + j])), K[L.kC + j]); put(j, s); q = 1; }     // step 0: ark[0]
    else {                                                                                                          // state after the previous segment;
        uint64_t *ps = V + 4ull * (pos_state_off(L, q - 1) + j);                                                    // its slots are the one thing that
        s = vm_load_val(ps); if (act) vm_store_val(ps, fr_from_mont(s));                                            // segment left in Montgomery form
    }
    auto full = [&](uint32_t F, uint32_t coff, uint32_t moff) {
        Fr x2 = fr_mont(s, s), x4 = fr_mont(x2, x2), x5 = fr_mont(x4, s);
        put(F + 3 * j, x2); put(F + 3 * j + 1, x4); put(F + 3 * j + 2, x5);
        Fr y = fr_add(x5, K[L.kC + coff + j]); put(F + 3 * t + j, y);
        Fr acc = fr_zero();
        for (uint32_t k = 0; k < t; k++) { Fr yk = shfl_fr(y, (int)k); acc = fr_add(acc, fr_mont(K[moff + k * t + j], yk)); }
        put(F + 4 * t + j, acc); s = acc;
    };
#pragma unroll 1
    for (; q < op.q1 && q < Q - 1; q++) {
        if (q <= 4) { const uint32_t f = q - 1; full(L.F1 + 5 * t * f, (f + 1) * t, f == 3 ? L.kP : L.kM); }
        else if (q < 5 + L.rp) {
            const uint32_t r = q - 5, B = L.PB + r * (4 + t), so = (2 * t - 1) * r;
            Fr x2 = fr_mont(s, s), x4 = fr_mont(x2, x2), x5 = fr_mont(x4, s);                // meaningful on lane 0 only
            Fr z0 = fr_add(x5, K[L.kC + 5 * t + r]);
            if (lane == 0) { vm_store_val(V + 4ull * B, x2); vm_store_val(V + 4ull * (B + 1), x4); vm_store_val(V + 4ull * (B + 2), x5); vm_store_val(V + 4ull * (B + 3), z0); }
            z0 = shfl_fr(z0, 0);
            const Fr in = (lane == 0) ? z0 : s;
            Fr prod = fr_mont(K[L.kS + so + j], in);                                          // S[so + i] * in[i]
            Fr o0 = fr_zero();
            for (uint32_t k = 0; k < t; k++) o0 = fr_add(o0, shfl_fr(prod, (int)k));
            Fr oj = fr_add(s, fr_mont(z0, K[L.kS + so + t + (j ? j : 1) - 1]));                // lanes 1..t-1
            s = (lane == 0) ? o0 : oj;
            put(B + 4 + j, s);
        } else { const uint32_t f = q - 5 - L.rp; full(L.SB + 5 * t * f, 5 * t + L.rp + f * t, L.kM); }
    }
    if (op.q1 == Q) {                                                                          // last step
        Fr x2 = fr_mont(s, s), x4 = fr_mont(x2, x2), x5 = fr_mont(x4, s);
        put(L.LB + 3 * j, x2); put(L.LB + 3 * j + 1, x4); put(L.LB + 3 * j + 2, x5);
        Fr prod = fr_mont(K[L.kM + j * t], x5), out = fr_zero();
        for (uint32_t k = 0; k < t; k++) out = fr_add(out, shfl_fr(prod, (int)k));
        if (lane == 0) vm_store_val(V + 4ull * (L.LB + 3 * t), out);
    }
    // every segment converts what it wrote (all 32 lanes: Montgomery -> canonical, in place) except the state the next segment resumes from
    __syncwarp();
    const uint32_t keep = op.q1 < Q ? pos_state_off(L, op.q1 - 1) : L.total;
    for (uint32_t i = pos_step_begin(L, op.q0) + (uint32_t)lane; i < pos_step_begin(L, op.q1); i += 32) {
        if (i >= keep && i < keep + t) continue;
        uint64_t *p = V + 4ull * i;
        vm_store_val(p, fr_from_mont(vm_load_val(p)));
    }
}

// ---- prefix sum with every partial sum a signal (substring_check.circom:47-49, :95) by one warp -----------------
__device__ void psum_warp(const VmCtx &x, const PsumOp op) {
    const uint32_t lane = threadIdx.x & 31, per = (op.n + 31) / 32;
    const uint32_t lo = min(op.n, lane * per), hi = min(op.n, lo + per);
    Fr acc = fr_zero();
    for (uint32_t k = lo; k < hi; k++) acc = fr_add(acc, vm_load(x, x.aux[op.aux0 + k]));
    Fr incl = acc;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        Fr o;
#pragma unroll
        for (int i = 0; i < 8; i++) o.l[i] = __shfl_up_sync(0xffffffffu, incl.l[i], off);
        if ((int)lane >= off) incl = fr_add(incl, o);
    }
    Fr run = fr_add(vm_load(x, op.x0), fr_sub(incl, acc));            // x0 + sum of all earlier lanes
    uint64_t *V = x.U + x.val_base + 4ull * op.dst;
    for (uint32_t k = lo; k < hi; k++) { run = fr_add(run, vm_load(x, x.aux[op.aux0 + k])); vm_store_val(V + 4ull * k, run); }
}

struct EvalArgs {
    const Op *ops; const AbsorbOp *absorbs; const PoseidonOp *poseidons; const Fr *pos_konst; const PsumOp *psums;
    const Level *levels; uint32_t n_levels, inv_begin, ginv_begin, inv_end;
    const Code *aux; const Fr *konst; const Fr *invtab;
    const Code *out_codes; uint32_t n_outputs, n_inputs, val_base;
    uint64_t *stores; uint64_t store_stride;     // u64 units
    const uint64_t *inputs;                       // chunk base: instance j at inputs + j * n_inputs * 4
    uint32_t *status; uint64_t *outputs;          // chunk base
    long long *prof;                              // tuning only: per-level clock64 stamps of instance 0 (or null)
    uint32_t pos_konst_bytes, levels_bytes;       // sizes of the two TMA-staged tables (multiples of 16 bytes)
    uint32_t prefetch;                            // 1: fetch the next op record / prefetch its operand lines while the current op runs
    uint32_t ginv_level;                          // first level at which every deferred inverse has its input (n_levels: none before the end)
};

// deferred IsZero inverses (comparators.circom:30): vm_exec.h vm_ginv_start / inv_chain_steps / vm_ginv_finish.  INV_WORKERS threads per
// CTA (its last 8 warps: warp ops are dealt from warp 0 upwards) run one inversion each, INV_STEPS iterations of it per level.  The
// iterations are issue-bound: with every thread a worker (half as many products to unwind per worker) the levels that carry them
// take longer.
static const uint32_t INV_WORKERS = 256, INV_STEPS = 64;
// parked state: word-major ([33 words][workers]) so that a warp's loads and stores are conflict-free
static const uint32_t INV_PARK_WORDS = 33;
__device__ __forceinline__ void inv_park(uint32_t *s, uint32_t nw, uint32_t t, const InvChain &c) {
#pragma unroll
    for (int k = 0; k < 8; k++) { s[(k) * nw + t] = c.u.l[k]; s[(8 + k) * nw + t] = c.v.l[k]; s[(16 + k) * nw + t] = c.r.l[k]; s[(24 + k) * nw + t] = c.s.l[k]; }
    s[32 * nw + t] = c.k;
}
__device__ __forceinline__ InvChain inv_unpark(const uint32_t *s, uint32_t nw, uint32_t t) {
    InvChain c;
#pragma unroll
    for (int k = 0; k < 8; k++) { c.u.l[k] = s[(k) * nw + t]; c.v.l[k] = s[(8 + k) * nw + t]; c.r.l[k] = s[(16 + k) * nw + t]; c.s.l[k] = s[(24 + k) * nw + t]; }
    c.k = s[32 * nw + t];
    return c;
}

// ---- TMA (bulk async copy engine) and cluster primitives ---------------------------------------------------------------
// cp.async.bulk global -> shared with mbarrier completion (SASS: UBLKCP.S.G + SYNCS.ARRIVE.TRANS64); the copies are issued by
// one thread and land while the CTA does other work.  Addresses and sizes must be multiples of 16 bytes.
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile("{\n.reg .pred P1;\nLAB_WAIT:\nmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n@P1 bra DONE;\nbra LAB_WAIT;\nDONE:\n}"
                 ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
// all threads of all CTAs of the cluster; release/acquire at cluster scope orders the global-memory store traffic of a level
// before the loads of the next one
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__device__ __forceinline__ Op ldg_op(const Op *p) { const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p)); return Op{v.x, v.y, v.z, v.w}; }
__device__ __forceinline__ void prefetch_code(const VmCtx &x, Code c) {
    const uint32_t k = code_kind(c), p = code_payload(c);
    const void *q = (k == K_VAL) ? (const void *)(x.U + x.val_base + 4ull * p) : (k == K_BIT) ? (const void *)(x.U + (p >> 6)) : nullptr;
    if (q) asm volatile("prefetch.global.L1 [%0];" ::"l"(q));
}
__device__ __forceinline__ void prefetch_operands(const VmCtx &x, const Op &o) {
    const uint32_t opc = op_opc(o);
    if (opc == OP_PACK8 || opc == OP_SELSUM) { if (opc == OP_SELSUM) prefetch_code(x, o.a); return; }   // their operand lists live in aux[]
    prefetch_code(x, o.a);
    if (opc == OP_FMA || opc == OP_CHK_EQ || opc == OP_DIV || opc == OP_MOD) prefetch_code(x, o.b);
    if (opc == OP_FMA) prefetch_code(x, o.c);
}

// k_eval: one thread-block CLUSTER per proof instance (cluster size C = 1, 2, 4 or 8 CTAs of THREADS threads; C = 1 is a plain
// CTA).  The levelised program is spread over all C*THREADS threads / all warps of the cluster, levels are separated by a
// cluster barrier; the instance store lives in global memory (L2-resident).  Poseidon round / MDS constants (C, S, M, P of
// circomlib/circuits/poseidon_constants.circom, Montgomery form) and the level table are staged in shared memory by TMA.
template <int THREADS>
// Register cap 104 for the 512-thread shape: 512 x 104 leaves 12 K registers of the SM, enough for one k_expand_round CTA (256 x 32) to
// stay resident next to a k_eval CTA.  Without the cap the SM belongs to k_eval alone: the kernel runs faster and the batch slower.
__global__ void __maxnreg__(THREADS == 1024 ? 64 : 104) k_eval(const EvalArgs a) {
    extern __shared__ __align__(128) uint8_t dyn_smem[];
    const uint32_t C = cluster_nctarank(), rank = cluster_ctarank();
    const uint32_t inst = blockIdx.x / C, tid = threadIdx.x;
    const uint32_t gt = rank * THREADS + tid, GT = C * THREADS;
    uint64_t *U = a.stores + (uint64_t)inst * a.store_stride;
    __shared__ uint32_t s_status;
    __shared__ __align__(8) uint64_t s_bar;
    Fr *s_pk = reinterpret_cast<Fr *>(dyn_smem);
    Level *s_levels = reinterpret_cast<Level *>(dyn_smem + a.pos_konst_bytes);
    uint32_t *s_inv = reinterpret_cast<uint32_t *>(dyn_smem + a.pos_konst_bytes + a.levels_bytes);     // INV_WORKERS parked chains
    const bool inv_worker = tid + INV_WORKERS >= THREADS;
    const uint32_t wt = tid - (THREADS - INV_WORKERS), wid = rank * INV_WORKERS + wt, NWK = C * INV_WORKERS;
    bool inv_running = false;                     // this worker has an inversion in progress (state parked in s_inv)
    if (tid == 0) { s_status = STATUS_OK; mbar_init(&s_bar, 1); if (rank == 0) a.status[inst] = STATUS_OK; }
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(&s_bar, a.pos_konst_bytes + a.levels_bytes);
        tma_load_1d(s_pk, a.pos_konst, a.pos_konst_bytes, &s_bar);
        tma_load_1d(s_levels, a.levels, a.levels_bytes, &s_bar);
    }
    const uint64_t *in = a.inputs + (uint64_t)inst * a.n_inputs * 4;
    // inputs -> first value slots, reduced mod p like the circom loader does (a caller may hand over limbs >= p)
    for (uint32_t i = gt; i < a.n_inputs; i += GT) {
        Fr v = vm_load_val(in + 4ull * i);
        while (fr_geq_p(v)) { Fr t; fr_raw_sub(t, v, fr_p()); v = t; }
        vm_store_val(U + a.val_base + 4ull * i, v);
    }
    mbar_wait(&s_bar, 0);
    cluster_sync_all();
    VmCtx x{U, a.val_base, a.konst, a.aux, a.invtab, &s_status};
    // warp ops are dealt round-robin over the CTAs of the cluster (the 17 absorbs of a level land on 8 SMs, not on one)
    const uint32_t gwarp = (tid >> 5) * C + rank, nwarp = GT >> 5;
    for (uint32_t lv = 0; lv < a.n_levels; lv++) {
        if (a.prof && inst == 0 && gt == 0) a.prof[lv] = clock64();
        const Level L = s_levels[lv];
        // thread ops of one level are mutually independent: the next op record is fetched, and the cache lines of its operands
        // are requested (prefetch.global.L1), while the current op executes -- two of the three dependent memory latencies
        // of an op (record -> operand -> result) overlap with the previous op
        {
            uint32_t i = L.t_begin + gt;
            Op nxt = i < L.t_end ? ldg_op(a.ops + i) : Op{0, 0, 0, 0};
            for (; i < L.t_end; i += GT) {
                const Op cur = nxt;
                if (i + GT < L.t_end) { nxt = ldg_op(a.ops + i + GT); if (a.prefetch) prefetch_operands(x, nxt); }
                vm_exec_op(x, cur);
            }
        }
        // warp ops: Poseidons take the first warps (long), Keccak absorbs the next ones
        for (uint32_t q = L.p_begin + gwarp; q < L.p_end; q += nwarp) poseidon_warp(x, a.poseidons[q], s_pk);
        { const uint32_t np = (L.p_end - L.p_begin) % nwarp, wv = (gwarp + nwarp - np) % nwarp;
          for (uint32_t w = L.w_begin + wv; w < L.w_end; w += nwarp) absorb_warp(U, a.absorbs[w]);
          const uint32_t nw2 = (np + (L.w_end - L.w_begin)) % nwarp, sv = (gwarp + nwarp - nw2) % nwarp;
          for (uint32_t q = L.s_begin + sv; q < L.s_end; q += nwarp) psum_warp(x, a.psums[q]); }
        if (inv_worker) {
            if (lv == a.ginv_level) {                                               // deferred inverses: start
                InvChain c;
                if (vm_ginv_start(x, a.ops, a.ginv_begin, a.inv_end, wid, NWK, c)) { inv_park(s_inv, INV_WORKERS, wt, c); inv_running = true; }
            } else if (inv_running) {                                               // step; unwind as soon as the inverse is there
                InvChain c = inv_unpark(s_inv, INV_WORKERS, wt);
                if (inv_chain_steps(c, INV_STEPS)) { vm_ginv_finish(x, a.ops, a.ginv_begin, a.inv_end, wid, NWK, inv_chain_result(c)); inv_running = false; }
                else inv_park(s_inv, INV_WORKERS, wt, c);
            }
        }
        cluster_sync_all();
    }
    if (a.prof && inst == 0 && gt == 0) a.prof[a.n_levels] = clock64();
    // finish the deferred inverses (or do all of it when their inputs only became ready in the last level)
    if (inv_worker) {
        if (a.ginv_level >= a.n_levels) vm_inv_batch(x, a.ops, a.ginv_begin, a.inv_end, wid, NWK);
        else if (inv_running) {
            InvChain c = inv_unpark(s_inv, INV_WORKERS, wt);
            while (!inv_chain_steps(c, 64)) { }
            vm_ginv_finish(x, a.ops, a.ginv_begin, a.inv_end, wid, NWK, inv_chain_result(c));
        }
    }
    if (a.prof && inst == 0) { cluster_sync_all(); if (gt == 0) { a.prof[a.n_levels + 1] = clock64(); a.prof[a.n_levels + 2] = clock64(); } }
    __syncthreads();
    if (tid == 0 && s_status != STATUS_OK) atomicMin(a.status + inst, s_status);
    cluster_sync_all();
    if (gt == 0 && atomicAdd(a.status + inst, 0u) == STATUS_OK) a.status[inst] = 0u;
    for (uint32_t i = gt; i < a.n_outputs; i += GT) {
        uint64_t v[4]; vm_expand(a.out_codes[i], U, 0, a.val_base, a.konst, v);
        uint64_t *o = a.outputs + ((uint64_t)inst * a.n_outputs + i) * 4;
        o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[3];
    }
}

// Half a 32-byte entry as one 128-bit store (STG.E.128; sm_90 has no 256-bit store).  No "memory" clobber on purpose: the
// compiler must be free to hoist the next entries' loads above it so that several loads are in flight per thread (the
// witness is written, never read, here).
__device__ __forceinline__ void st128(uint64_t *p, uint64_t a, uint64_t b) { asm volatile("st.global.v2.b64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b)); }

struct ExpandArgs {
    const Tile *tiles; const Code *codes; const Fr *konst; const uint2 *round_desc;
    const uint64_t *stores; uint64_t store_stride; uint32_t val_base;   // store of chunk-local instance 0
    uint64_t *const *wit;                         // per materialised instance of the group: witness slot base
    const uint32_t *inst;                         // per materialised instance of the group: instance index within the batch
    const uint32_t *status;                       // per instance of the batch; a rejected instance contributes no witness
    uint32_t chunk_first;                         // batch index of the chunk's first instance (store = inst - chunk_first)
    uint32_t tile0;                               // first tile of this launch (k_expand_codes)
};

// k_expand_round: grid = (KeccakfRound tiles, instances in the group) -- 95.8 % of the witness.  One CTA streams one
// tile (<= 4096 entries = 128 KiB in the O0 layout) with one 128-bit store per half entry.  The source of every entry
// follows from an 8-byte descriptor per 64 entries and a lane word of the round; the tile's <= 130 descriptors and the round's 263 words are
// staged in shared memory by two TMA bulk copies, so the streaming loop touches no global memory but the witness itself.
constexpr int ROUND_THREADS = 256;
__global__ void __launch_bounds__(ROUND_THREADS) k_expand_round(const ExpandArgs a) {
    const uint32_t gi = a.inst[blockIdx.y];
    if (a.status[gi] != 0) return;                // reference: a failed assert leaves no witness (tests/test.py:65-68)
    const Tile t = a.tiles[blockIdx.x];
    const uint64_t *Ub = a.stores + (uint64_t)(gi - a.chunk_first) * a.store_stride + t.ubase;
    uint64_t *W = a.wit[blockIdx.y] + t.dst * 4;
    __shared__ __align__(16) uint2 sD[MAX_TILE_SIGNALS / 64];
    __shared__ __align__(16) uint64_t sWraw[ROUND_WORDS_SPAN + 3];
    __shared__ __align__(8) uint64_t s_bar;
    // the tile's descriptors and the round's lane words arrive by TMA: two bulk copies issued by one thread, completion on an
    // mbarrier.  The word window starts at the 16-byte boundary at or below the round base (the base is only 8-byte aligned).
    const uint32_t odd = (uint32_t)((reinterpret_cast<uintptr_t>(Ub) >> 3) & 1u);
    const uint32_t nd = (t.n + 63) >> 6, d_bytes = ((nd + 1) & ~1u) * 8u, w_bytes = (ROUND_WORDS_SPAN + 3) / 2 * 16u;
    if (threadIdx.x == 0) mbar_init(&s_bar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&s_bar, d_bytes + w_bytes);
        tma_load_1d(sD, a.round_desc + (t.code_off >> 6), d_bytes, &s_bar);
        tma_load_1d(sWraw, Ub - odd, w_bytes, &s_bar);
    }
    mbar_wait(&s_bar, 0);
    const uint64_t *sW = sWraw + odd;
    // one 16-byte half u of the tile per thread and store (entry u / 2; the upper half of an entry is zero): a warp's store
    // covers 512 contiguous bytes.  Two 128-bit stores of the same thread per entry would leave every store instruction
    // half of each 32-byte sector it touches, twice the L2 write requests for the same bytes.
#pragma unroll 8
    for (uint32_t u = threadIdx.x; u < 2 * t.n; u += ROUND_THREADS) {
        const uint32_t k = u >> 1;
        const uint2 d = sD[k >> 6];
        const uint32_t tt = k & 63, mode = d.y >> 16;
        uint32_t w = d.x & 0xffffu, b = tt;
        if (mode) {                          // phase (mode-1) of a gate block [out_i, a_i, b_i]_i
            const uint32_t sidx = (mode - 1) * 64 + tt, g = sidx / 3, m = sidx - 3 * g;
            b = g; w = (m == 0) ? (d.x & 0xffffu) : (m == 1) ? (d.x >> 16) : (d.y & 0xffffu);
        }
        const uint64_t v = (u & 1u) ? 0ull : (sW[w] >> b) & 1ull;
        st128(W + 2ull * u, v, 0);
    }
}

// k_expand_codes: grid = (instances in the group, code tiles) -- INSTANCE-major, so that a tile's code stream is fetched
// from DRAM once and served from L2 to the other witnesses of the group.  One 32-bit code per entry.  The tile's code stream
// (<= 32 KiB, contiguous) is brought into shared memory by ONE TMA bulk copy, so the first of the two dependent memory hops of
// an entry (code -> store word / value -> witness) costs a shared-memory read; the gathers of UG half entries per thread are
// then in flight together, ahead of the stores.  Launched with unused dynamic shared memory so that three CTAs are resident
// per SM (pob_b200.cu codes_dyn_smem).
__global__ void __launch_bounds__(256, 3) k_expand_codes(const ExpandArgs a) {
    constexpr int UG = 4;
    const uint32_t gi = a.inst[blockIdx.x];
    if (a.status[gi] != 0) return;
    const Tile t = a.tiles[a.tile0 + blockIdx.y];
    const uint64_t *U = a.stores + (uint64_t)(gi - a.chunk_first) * a.store_stride;
    uint64_t *W = a.wit[blockIdx.x] + t.dst * 4;
    const uint64_t *Ub = U + t.ubase;
    __shared__ __align__(16) Code sC[TILE_SIGNALS + 4];
    __shared__ __align__(8) uint64_t s_bar;
    const uint32_t off4 = t.code_off & 3u, bytes = (((t.n + off4) * 4u) + 15u) & ~15u;     // TMA wants 16-byte aligned source and size
    if (threadIdx.x == 0) mbar_init(&s_bar, 1);
    __syncthreads();
    if (threadIdx.x == 0) { mbar_expect_tx(&s_bar, bytes); tma_load_1d(sC, a.codes + (t.code_off - off4), bytes, &s_bar); }
    mbar_wait(&s_bar, 0);
    const Code *c = sC + off4;
    // one 16-byte half u of the tile per thread and store, as in k_expand_round: entry u / 2, half h = u & 1 (the same for every
    // u of a thread).  Lanes 2j and 2j+1 read the same code word (a shared-memory broadcast); a warp's stores cover 512
    // contiguous bytes, and a value slot or constant (32-byte aligned) is gathered by a lane pair as one whole sector, one
    // 128-bit load per lane.  A 0/1 bit or a small constant has a zero upper half: that lane stores zeros and gathers nothing.
    const uint32_t n2 = 2 * t.n, h = threadIdx.x & 1u;
    for (uint32_t base = threadIdx.x; base < n2; base += 256 * UG) {
        uint64_t v[UG][2];
#pragma unroll
        for (int j = 0; j < UG; j++) {
            const uint32_t u = base + 256 * j;
            const Code cd = u < n2 ? c[u >> 1] : 0u;
            const uint32_t kind = code_kind(cd), p = code_payload(cd);
            v[j][0] = v[j][1] = 0;
            if (kind == K_VAL || kind == K_KONST) {
                const uint64_t *s = (kind == K_VAL) ? U + a.val_base + 4ull * p : reinterpret_cast<const uint64_t *>(a.konst + p);
                const ulonglong2 q = reinterpret_cast<const ulonglong2 *>(s)[h];
                v[j][0] = q.x; v[j][1] = q.y;
            } else if (!h) v[j][0] = (kind == K_BIT) ? (Ub[p >> 6] >> (p & 63)) & 1ull : p;
        }
#pragma unroll
        for (int j = 0; j < UG; j++) { const uint32_t u = base + 256 * j; if (u < n2) st128(W + 2ull * u, v[j][0], v[j][1]); }
    }
}

// digest = sum_i mix(i, limbs) mod 2^64 -- must equal oracle/pob_oracle.c:pob_oracle_digest
__global__ void __launch_bounds__(256) k_digest(const uint64_t *wit, uint64_t n_signals, unsigned long long *out, const uint32_t *status) {
    if (status && *status != 0) return;           // rejected instance: no witness, digest stays 0
    uint64_t acc = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_signals; i += (uint64_t)gridDim.x * blockDim.x) {
        const ulonglong4 v = *reinterpret_cast<const ulonglong4 *>(wit + 4 * i);
        uint64_t h = (i + 1) * 0x9E3779B97F4A7C15ULL;
        h ^= v.x * 0xBF58476D1CE4E5B9ULL + v.y * 0x94D049BB133111EBULL + v.z * 0xD6E8FEB86659FD93ULL + v.w * 0xA0761D6478BD642FULL;
        h ^= h >> 29; h *= 0xBF58476D1CE4E5B9ULL; h ^= h >> 32;
        acc += h;
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    __shared__ uint64_t part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) { uint64_t s = 0; for (int w = 0; w < 8; w++) s += part[w]; atomicAdd(out, (unsigned long long)s); }
}

// ---- proof-of-work burn-key grinder (reference tests/main.py:47-56; circuits/utils/proof_of_work.circom:54-81) ----
// One candidate key per thread: a single-block keccak256 of key|reveal|extra|"EIP-7503" held in 25 registers.
struct GrindArgs { uint64_t start[4], lanes_tail[9]; uint64_t first, count; uint32_t zero_bytes; unsigned long long *hit; };
__device__ __forceinline__ uint64_t bswap64(uint64_t x) { return __byte_perm((uint32_t)(x >> 32), 0, 0x0123) | ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32); }
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int n) { return (x << n) | (x >> (64 - n)); }
__global__ void __launch_bounds__(256) k_pow_grind(const GrindArgs a) {
    const uint64_t idx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.count) return;
    // key = start + first + idx (256-bit add)
    uint64_t k0 = a.start[0], k1 = a.start[1], k2 = a.start[2], k3 = a.start[3];
    const uint64_t add = a.first + idx;
    k0 += add; if (k0 < add) { if (++k1 == 0) { if (++k2 == 0) ++k3; } }
    uint64_t s[25];
    s[0] = bswap64(k3); s[1] = bswap64(k2); s[2] = bswap64(k1); s[3] = bswap64(k0);      // 32-byte big-endian key
#pragma unroll
    for (int i = 0; i < 9; i++) s[4 + i] = a.lanes_tail[i];                                // reveal | extra | "EIP-7503"
    s[13] = 0x01; s[14] = 0; s[15] = 0; s[16] = 0x8000000000000000ull;                     // 0x01 ... 0x80 padding of a 104-byte message
#pragma unroll
    for (int i = 17; i < 25; i++) s[i] = 0;
#pragma unroll 1
    for (int r = 0; r < 24; r++) {
        uint64_t c[5], d[5], b[25];
#pragma unroll
        for (int x = 0; x < 5; x++) c[x] = s[x] ^ s[x + 5] ^ s[x + 10] ^ s[x + 15] ^ s[x + 20];
#pragma unroll
        for (int x = 0; x < 5; x++) d[x] = c[(x + 4) % 5] ^ rotl64(c[(x + 1) % 5], 1);
#pragma unroll
        for (int i = 0; i < 25; i++) s[i] ^= d[i % 5];
        b[0] = s[0];
#pragma unroll
        for (int i = 0; i < 24; i++) b[keccak_rot(i + 1)] = rotl64(s[keccak_rot(i)], keccak_shl(i));
#pragma unroll
        for (int i = 0; i < 25; i++) s[i] = b[i] ^ (~b[chi_b(i)] & b[chi_c(i)]);
        s[0] ^= c_keccak_rc[r];
    }
    const uint64_t mask = a.zero_bytes >= 8 ? ~0ull : ((1ull << (8 * a.zero_bytes)) - 1);
    if ((s[0] & mask) == 0) atomicMin(a.hit, (unsigned long long)idx);
}

// ---- self-check: every KeccakfRound block of a materialised witness satisfies out == KeccakRound_r(in) -------------
// One warp per block.  Lane l < 25 assembles lane word l of `in` (witness entries base+1600+64l .. +63) and of `out`
// (base+64l ..) from the 32-byte entries, lane 0 gathers the 25 input words and runs one textbook round.
__global__ void __launch_bounds__(256) k_check_rounds(const uint64_t *wit, const uint64_t *block_base, uint32_t n_blocks, unsigned long long *n_bad) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= n_blocks) return;
    const uint64_t base = block_base[warp];
    const int r = (int)(warp % 24);                       // round blocks are emitted 24 per Keccakf, in order
    uint64_t win = 0, wout = 0; bool bad = false;
    if (lane < 25) {
        for (uint32_t k = 0; k < 64; k++) {
            const ulonglong4 a = *reinterpret_cast<const ulonglong4 *>(wit + 4 * (base + 1600 + 64 * lane + k));
            const ulonglong4 b = *reinterpret_cast<const ulonglong4 *>(wit + 4 * (base + 64 * lane + k));
            bad |= (a.x > 1) | (b.x > 1) | ((a.y | a.z | a.w | b.y | b.z | b.w) != 0);
            win |= (a.x & 1ull) << k; wout |= (b.x & 1ull) << k;
        }
    }
    uint64_t s[25], o[25];
#pragma unroll
    for (int i = 0; i < 25; i++) { s[i] = __shfl_sync(0xffffffffu, win, i); o[i] = __shfl_sync(0xffffffffu, wout, i); }
    bad = __any_sync(0xffffffffu, bad);
    if (lane == 0) {
        uint64_t c[5], d[5], b[25];
#pragma unroll
        for (int x = 0; x < 5; x++) c[x] = s[x] ^ s[x + 5] ^ s[x + 10] ^ s[x + 15] ^ s[x + 20];
#pragma unroll
        for (int x = 0; x < 5; x++) d[x] = c[(x + 4) % 5] ^ rotl64(c[(x + 1) % 5], 1);
#pragma unroll
        for (int i = 0; i < 25; i++) s[i] ^= d[i % 5];
        b[0] = s[0];
#pragma unroll
        for (int i = 0; i < 24; i++) b[keccak_rot(i + 1)] = rotl64(s[keccak_rot(i)], keccak_shl(i));
#pragma unroll
        for (int i = 0; i < 25; i++) s[i] = b[i] ^ (~b[chi_b(i)] & b[chi_c(i)]);
        s[0] ^= c_keccak_rc[r];
#pragma unroll
        for (int i = 0; i < 25; i++) bad |= (s[i] != o[i]);
        if (bad) atomicAdd(n_bad, 1ull);
    }
}


// ---- full constraint self-check (SURVEY.md 8(f) rank 4): every `<==` / `===` of the circuit against a resident witness ----
// One thread per record; the shared KeccakfRound set is replayed for every round block (grid = records x blocks).
// rep[0] = failing circuit constraints, rep[1] = failing hint records, rep[2] = smallest failing record id.
struct CheckArgs {
    ConsView V; const Fr *konst; const uint64_t *wit;
    const uint64_t *bases; uint32_t n_blocks;       // null / 0: the flat set (absolute indices)
    uint64_t id0;                                   // record id of (block 0, first eq record) of this set
    unsigned long long *rep;
};
__device__ __forceinline__ void check_fail(const CheckArgs &a, uint64_t id, bool hint) {
    atomicAdd(a.rep + (hint ? 1 : 0), 1ull); atomicMin(a.rep + 2, (unsigned long long)id);
}
__global__ void __launch_bounds__(256) k_check_eq(const CheckArgs a) {
    const uint64_t per = a.V.n_eq, total = per * (a.bases ? a.n_blocks : 1u);
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t blk = t / per, r = t - blk * per, base = a.bases ? a.bases[blk] : 0;
        if (!cons_eq_ok(a.wit, base, a.V.eq[2 * r], a.V.eq[2 * r + 1])) check_fail(a, a.id0 + blk * a.V.n_records() + r, false);
    }
}
__global__ void __launch_bounds__(256) k_check_kc(const CheckArgs a) {
    const uint64_t per = a.V.n_kc, total = per * (a.bases ? a.n_blocks : 1u);
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t blk = t / per, r = t - blk * per, base = a.bases ? a.bases[blk] : 0;
        if (!cons_kc_ok(a.wit, base, a.V.kc[r], a.konst, c_keccak_rc[blk % 24])) check_fail(a, a.id0 + blk * a.V.n_records() + a.V.n_eq + r, false);
    }
}
__global__ void __launch_bounds__(256) k_check_r1(const CheckArgs a) {
    const uint64_t per = a.V.n_r1, total = per * (a.bases ? a.n_blocks : 1u);
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t blk = t / per, r = t - blk * per, base = a.bases ? a.bases[blk] : 0;
        const ConsR1 rec = a.V.r1[r];
        if (!cons_r1_ok(a.wit, base, rec, a.V.terms, a.konst)) check_fail(a, a.id0 + blk * a.V.n_records() + a.V.n_eq + a.V.n_kc + r, r1_hint(rec));
    }
}

// ---- .r1cs row products (r1cs.h): out[k] = A.w, B.w, C.w of row first + k, 32-byte canonical little-endian ------------------
// Row k of the plan is decoded into (set, block, kind, local record): the flat set's eq / kc / r1 records first, then the round
// set once per block.  A LANE PAIR owns a row: both lanes evaluate it (the same loads, merged in the warp's request) and lane h
// stores 16-byte half h of each product, so that a warp's store covers 16 rows = 512 contiguous bytes per vector -- one thread
// writing a whole 32-byte entry as two 128-bit stores is the pattern that halved the expand kernels' rate (DESIGN.md §2.3).
struct R1csArgs {
    ConsView flat, round; const Fr *konst; const uint64_t *wit;
    const uint64_t *bases;                          // first witness index of every round block (n_blocks of them)
    uint64_t first, n;                              // rows [first, first + n)
    uint4 *a, *b, *c;                               // n entries each, or null (not computed)
};
__device__ __forceinline__ void st_half(uint4 *out, uint64_t k, uint32_t h, const Fr &v) {
    out[2 * k + h] = h ? make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]) : make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);   // no dynamic index: Fr stays in registers
}
__global__ void __launch_bounds__(256) k_r1cs_products(const R1csArgs a) {
    const uint32_t h = threadIdx.x & 1u;
    const uint64_t nf = a.flat.n_records(), per = a.round.n_records();
    const bool want_ab = a.a || a.b;
    const Fr w0 = cons_load(a.wit, 0, 0);                                   // constants are multiples of w[0], as in the file
    for (uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 1; k < a.n; k += ((uint64_t)gridDim.x * blockDim.x) >> 1) {
        uint64_t r = a.first + k, base = 0, rc = 0;
        const bool in_round = r >= nf;
        if (in_round) { const uint64_t q = r - nf, blk = q / per; r = q - blk * per; base = a.bases[blk]; rc = c_keccak_rc[blk % 24]; }
        const ConsView V = in_round ? a.round : a.flat;
        Fr A = fr_zero(), B = fr_zero(), C;
        if (r < V.n_eq) {                                                   // C = w[a] - w[b]
            C = fr_sub(cons_load(a.wit, base, V.eq[2 * r], w0), cons_load(a.wit, base, V.eq[2 * r + 1], w0));
        } else if (r < V.n_eq + V.n_kc) {                                   // C = w[a] - k w0
            const ConsTerm t = V.kc[r - V.n_eq];
            C = fr_sub(cons_load(a.wit, base, t.idx, w0), fr_mul(cons_coef_value(t.coef, a.konst, rc), w0));
        } else {
            const ConsR1 rec = V.r1[r - V.n_eq - V.n_kc];
            const ConsTerm *t = V.terms + rec.off;
            C = a.c ? cons_lc(a.wit, base, t + rec.na + rec.nb, r1_nc(rec), a.konst, w0) : fr_zero();
            if (want_ab && rec.na) { A = cons_lc(a.wit, base, t, rec.na, a.konst, w0); B = cons_lc(a.wit, base, t + rec.na, rec.nb, a.konst, w0); }
        }
        if (a.a) st_half(a.a, k, h, A);
        if (a.b) st_half(a.b, k, h, B);
        if (a.c) st_half(a.c, k, h, C);
    }
}

}  // namespace
