// store_probe.cu -- how fast one SM-side store form writes a witness-sized buffer, compressible or not.
//   Two ~6 GiB buffers made like the library's witness slots (cuMemCreate, COMP_GENERIC and COMP_NONE), three data patterns
//   (the KeccakfRound pattern: 32-byte entries whose byte 0 is a pseudo-random 0/1 and the rest zero; all zeros; random
//   32-byte entries), three store forms:
//     (a) stg       one 16-byte half entry per lane (STG.E.128), one 256 KiB tile per CTA -- k_expand_round's form
//     (b) bulk      the lanes fill a shared-memory ring of NB chunks of S KiB; one thread writes each chunk with
//                   cp.async.bulk.global.shared::cta (UBLKCP.G.S)
//     (c) bulk+ef   (b) with an L2::cache_hint evict_first policy on the bulk store
//   CTAs per SM are set through dynamic shared memory, as the library does.  Timing: CUDA events over whole-buffer passes in
//   windows of >= 0.5 s; every configuration is timed in each of 5 rounds (arms alternate), median / min / max reported.
//   nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -O3 -o tools/probes/store_probe tools/probes/store_probe.cu \
//        -L/usr/local/cuda/lib64/stubs -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)
#define CD(x) do { CUresult e_ = (x); if (e_ != CUDA_SUCCESS) { fprintf(stderr, "%s:%d CUresult %d\n", __FILE__, __LINE__, (int)e_); exit(1); } } while (0)

static constexpr uint32_t T = 256;                     // threads per CTA, as k_expand_round
static constexpr uint32_t TILE_BYTES = 256u << 10;     // one CTA writes one tile (8192 entries), as k_expand_round
static constexpr uint32_t TILE_HALVES = TILE_BYTES / 16;

enum Pattern { ROUND = 0, ZEROS = 1, RANDOM = 2 };
static const char *pat_name[] = {"round", "zeros", "random"};

__device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x;
}
// 16-byte half g of the buffer (entry g / 2)
__device__ __forceinline__ void half_value(int pat, uint32_t g, uint64_t &a, uint64_t &b) {
    if (pat == ROUND) { a = (g & 1u) ? 0ull : (uint64_t)(mix32(g >> 1) & 1u); b = 0; }
    else if (pat == ZEROS) { a = 0; b = 0; }
    else { a = ((uint64_t)mix32(4 * g) << 32) | mix32(4 * g + 1); b = ((uint64_t)mix32(4 * g + 2) << 32) | mix32(4 * g + 3); }
}

// (a) one 128-bit store per half entry, a warp's store covers 512 contiguous bytes
__global__ void __launch_bounds__(T) k_stg(uint64_t *buf, int pat) {
    const uint32_t g0 = blockIdx.x * TILE_HALVES;
    uint64_t *W = buf + 2ull * g0;
#pragma unroll 8
    for (uint32_t u = threadIdx.x; u < TILE_HALVES; u += T) {
        uint64_t a, b; half_value(pat, g0 + u, a, b);
        asm volatile("st.global.v2.b64 [%0], {%1, %2};" ::"l"(W + 2ull * u), "l"(a), "l"(b));
    }
}

// (b) / (c) a ring of nb chunks of chunk bytes in dynamic shared memory.  Per chunk c: fill buffer c % nb, make the
// generic-proxy writes visible to the async proxy, barrier, one thread issues the bulk store and commits it.  Before the
// barrier of chunk c that thread waits until at most nb - 2 bulk stores still read shared memory, so the store of chunk
// c + 1 - nb has left buffer (c + 1) % nb before anyone refills it after the barrier: one barrier per chunk.
template <bool HINT>
__global__ void __launch_bounds__(T) k_bulk(uint64_t *buf, int pat, uint32_t chunk, uint32_t nb) {
    extern __shared__ __align__(128) uint64_t ring[];
    const uint32_t g0 = blockIdx.x * TILE_HALVES, ch = chunk / 16, nchunks = TILE_BYTES / chunk;
    uint64_t *W = buf + 2ull * g0;
    uint64_t pol = 0;
    if (HINT) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    for (uint32_t c = 0; c < nchunks; c++) {
        uint64_t *S = ring + 2ull * ch * (c % nb);
#pragma unroll 4
        for (uint32_t u = threadIdx.x; u < ch; u += T) {
            uint64_t a, b; half_value(pat, g0 + c * ch + u, a, b);
            *reinterpret_cast<ulonglong2 *>(S + 2ull * u) = make_ulonglong2(a, b);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (threadIdx.x == 0) {
            if (nb == 2) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            else if (nb == 3) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            else asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t s = (uint32_t)__cvta_generic_to_shared(S);
            uint64_t *dst = W + 2ull * ch * c;
            if (HINT) asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst), "r"(s), "r"(chunk), "l"(pol) : "memory");
            else asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(s), "r"(chunk) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

struct Cfg {
    int arm;               // 0 stg, 1 bulk, 2 bulk + evict_first
    uint32_t chunk_kb, nb, ctas_per_sm;
    int pat, mem;          // mem: 0 compressible, 1 not
    std::vector<double> tbs;
    std::string name() const {
        char s[96];
        if (arm == 0) snprintf(s, sizeof s, "(a) stg            %u CTA/SM", ctas_per_sm);
        else snprintf(s, sizeof s, "(%c) bulk%s S=%2u KiB NB=%u %u CTA/SM", arm == 1 ? 'b' : 'c', arm == 2 ? "+ef" : "   ", chunk_kb, nb, ctas_per_sm);
        return s;
    }
};

static uint32_t dyn_smem(const Cfg &c) {
    // 2 CTAs/SM: 91 KiB, k_expand_round's total today (85 KiB dynamic + its static tables); 1 CTA/SM: 120 KiB or the ring
    const uint32_t ring = c.arm ? c.chunk_kb * c.nb * 1024u : 0u;
    return std::max(ring, (c.ctas_per_sm == 2 ? 91u : 120u) * 1024u);
}

static void launch(const Cfg &c, uint64_t *buf, uint32_t ntiles) {
    const uint32_t sm = dyn_smem(c);
    if (c.arm == 0) k_stg<<<ntiles, T, sm>>>(buf, c.pat);
    else if (c.arm == 1) k_bulk<false><<<ntiles, T, sm>>>(buf, c.pat, c.chunk_kb * 1024u, c.nb);
    else k_bulk<true><<<ntiles, T, sm>>>(buf, c.pat, c.chunk_kb * 1024u, c.nb);
}

static uint32_t occupancy(const Cfg &c) {
    int n = 0;
    if (c.arm == 0) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_stg, T, dyn_smem(c)));
    else if (c.arm == 1) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_bulk<false>, T, dyn_smem(c)));
    else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_bulk<true>, T, dyn_smem(c)));
    return (uint32_t)n;
}

static uint64_t *make_buffer(size_t bytes, bool comp, int dev) {
    CUmemAllocationProp p{};
    p.type = CU_MEM_ALLOCATION_TYPE_PINNED; p.location.type = CU_MEM_LOCATION_TYPE_DEVICE; p.location.id = dev;
    p.allocFlags.compressionType = comp ? CU_MEM_ALLOCATION_COMP_GENERIC : CU_MEM_ALLOCATION_COMP_NONE;
    size_t gran = 0; CD(cuMemGetAllocationGranularity(&gran, &p, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    bytes = (bytes + gran - 1) / gran * gran;
    CUmemGenericAllocationHandle h; CD(cuMemCreate(&h, bytes, &p, 0));
    CUdeviceptr va; CD(cuMemAddressReserve(&va, bytes, gran, 0, 0)); CD(cuMemMap(va, bytes, 0, h, 0));
    CUmemAccessDesc acc{}; acc.location = p.location; acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE; CD(cuMemSetAccess(va, bytes, &acc, 1));
    CUmemAllocationProp got{}; CD(cuMemGetAllocationPropertiesFromHandle(&got, h));
    printf("buffer %s: %.2f GB, asked %s, granted %s\n", comp ? "A" : "B", bytes / 1e9, comp ? "COMP_GENERIC" : "COMP_NONE",
           got.allocFlags.compressionType == CU_MEM_ALLOCATION_COMP_GENERIC ? "COMP_GENERIC" : "COMP_NONE");
    return reinterpret_cast<uint64_t *>(va);
}

static void gpu_state(const char *when) {
    FILE *f = popen("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu --format=csv,noheader", "r");
    char line[256] = {0};
    if (f) { if (!fgets(line, sizeof line, f)) line[0] = 0; pclose(f); }
    printf("%s: %s", when, line[0] ? line : "nvidia-smi not available\n");
}

int main() {
    const double window_s = 0.5;
    const int rounds = 5;
    int dev = 0; CK(cudaSetDevice(dev)); CK(cudaFree(0));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, dev));
    printf("%s, %d SMs\n", prop.name, prop.multiProcessorCount);
    gpu_state("before");
    CK(cudaFuncSetAttribute(k_stg, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    CK(cudaFuncSetAttribute(k_bulk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    CK(cudaFuncSetAttribute(k_bulk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    const size_t bytes = 6ull << 30;                    // ~ one main-shape witness (6.91 GB)
    const uint32_t ntiles = (uint32_t)(bytes / TILE_BYTES);
    uint64_t *bufs[2] = {make_buffer(bytes, true, dev), make_buffer(bytes, false, dev)};
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));

    auto run = [&](std::vector<Cfg> &cfgs) {
        std::vector<int> passes(cfgs.size());
        for (size_t i = 0; i < cfgs.size(); i++) {       // warm-up and calibration: passes per window
            uint64_t *b = bufs[cfgs[i].mem];
            launch(cfgs[i], b, ntiles); CK(cudaGetLastError());
            CK(cudaEventRecord(e0)); for (int p = 0; p < 3; p++) launch(cfgs[i], b, ntiles); CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1)); float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
            passes[i] = std::max(1, (int)(window_s * 1e3 / (ms / 3) + 0.999));
        }
        for (int r = 0; r < rounds; r++)
            for (size_t i = 0; i < cfgs.size(); i++) {
                uint64_t *b = bufs[cfgs[i].mem];
                CK(cudaEventRecord(e0)); for (int p = 0; p < passes[i]; p++) launch(cfgs[i], b, ntiles); CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1)); float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
                cfgs[i].tbs.push_back((double)ntiles * TILE_BYTES * passes[i] / (ms * 1e-3) / 1e12);
            }
        for (Cfg &c : cfgs) std::sort(c.tbs.begin(), c.tbs.end());
    };
    auto med = [](const Cfg &c) { return c.tbs[c.tbs.size() / 2]; };
    auto print = [&](const std::vector<Cfg> &cfgs) {
        for (const Cfg &c : cfgs)
            printf("  %-8s %-14s %-38s occ %u  TB/s median %.3f  [%.3f, %.3f]\n", pat_name[c.pat], c.mem ? "COMP_NONE" : "COMP_GENERIC",
                   c.name().c_str(), occupancy(c), med(c), c.tbs.front(), c.tbs.back());
    };

    // 1. the sweep: round pattern on compressible memory
    std::vector<Cfg> sweep;
    for (uint32_t cps : {2u, 1u}) sweep.push_back(Cfg{0, 0, 0, cps, ROUND, 0, {}});
    for (int arm : {1, 2})
        for (uint32_t cps : {2u, 1u})
            for (uint32_t kb : {4u, 8u, 16u, 32u})
                for (uint32_t nb : {2u, 3u, 4u}) {
                    Cfg c{arm, kb, nb, cps, ROUND, 0, {}};
                    if (dyn_smem(c) <= (cps == 2 ? 91u : 160u) * 1024u) sweep.push_back(c);
                }
    printf("\nsweep: round pattern, compressible buffer, %d rounds of >= %.1f s windows, whole-buffer passes of %.2f GB\n",
           rounds, window_s, (double)ntiles * TILE_BYTES / 1e9);
    run(sweep);
    print(sweep);
    const Cfg *best[3] = {nullptr, nullptr, nullptr};
    for (const Cfg &c : sweep) if (c.ctas_per_sm == 2 || c.arm) if (!best[c.arm] || med(c) > med(*best[c.arm])) best[c.arm] = &c;
    const Cfg a2 = sweep[0];
    for (int arm = 1; arm <= 2; arm++)
        printf("best %s: median %+.1f %% against (a) 2 CTA/SM; ranges %s\n", best[arm]->name().c_str(), 100.0 * (med(*best[arm]) / med(a2) - 1),
               best[arm]->tbs.front() > a2.tbs.back() ? "disjoint" : "overlap");

    // 2. the other patterns and the uncompressed buffer: (a) and the best (b) and (c)
    std::vector<Cfg> rest;
    for (int mem : {0, 1})
        for (int pat : {ROUND, ZEROS, RANDOM}) {
            if (mem == 0 && pat == ROUND) continue;
            for (int arm = 0; arm <= 2; arm++) { Cfg c = *best[arm]; c.pat = pat; c.mem = mem; c.tbs.clear(); if (arm == 0) c = Cfg{0, 0, 0, 2, pat, mem, {}}; rest.push_back(c); }
        }
    printf("\nother patterns and memory: (a) at 2 CTA/SM and the best (b), (c) of the sweep\n");
    run(rest);
    print(rest);
    gpu_state("after");
    return 0;
}
