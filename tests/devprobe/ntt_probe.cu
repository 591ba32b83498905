// tests/devprobe/ntt_probe.cu -- TEST-ONLY front-end of the product's BN254 transforms (csrc/ntt.cuh), for tests/test_ntt_cpu.py
// and tests/test_gpu_ntt.py.
//
// pob_r1cs_quotient reaches the transforms only at the domain sizes of the circuits it is given; this file runs the same pass
// plan (ntt_plan), host tables (ntt_host_tables) and launch functions (ntt_inverse_coset, ntt_forward) at any 2^L, L <= 28, on
// caller vectors.  Nothing here is part of the product: libpob_b200.so never contains or calls this file.  Built by
// tests/devprobe/ntt.py.
//
// The host entry points need no GPU.  The device entry points take DEVICE pointers to caller vectors of 2^L canonical 32-byte
// entries (16-byte aligned), upload the tables, launch, synchronise, free everything and return the cudaError_t.  No state
// survives a call.
#include <algorithm>
#include <cstring>
#include "ntt.cuh"

namespace {

struct DevTables {
    NttTables t{};
    std::vector<void *> allocs;
    cudaError_t err = cudaSuccess;
    const Fr *up(const std::vector<Fr> &v) {
        void *d = nullptr;
        if (err == cudaSuccess) err = cudaMalloc(&d, v.size() * sizeof(Fr));
        if (err == cudaSuccess) { allocs.push_back(d); err = cudaMemcpy(d, v.data(), v.size() * sizeof(Fr), cudaMemcpyHostToDevice); }
        return (const Fr *)d;
    }
    explicit DevTables(uint32_t L) {
        const NttHostTables H = ntt_host_tables(L);
        t.w_lo = up(H.w_lo); t.w_hi = up(H.w_hi); t.loc = up(H.loc); t.loc_inv = up(H.loc_inv);
        t.g_lo = up(H.g_lo); t.g_hi = up(H.g_hi); t.g_log = H.g_log;
        if (err == cudaSuccess) err = ntt_init_kernels();
    }
    ~DevTables() { for (void *p : allocs) cudaFree(p); }
};

// 0: inverse of x, 1: forward of x, 2: the quotient sequence on (x, b, c)
int run(int what, uint32_t L, void *x, void *b, void *c) {
    if (L < 1 || L > NTT_MAX_LOG) return (int)cudaErrorInvalidValue;
    DevTables D(L);
    const uint32_t T = std::min(L, NTT_TILE_LOG);
    cudaError_t err = D.err;
    uint4 *va = (uint4 *)x, *vb = (uint4 *)b, *vc = (uint4 *)c;
    if (err == cudaSuccess && what == 0) err = ntt_inverse_coset(va, L, T, D.t, 0);
    if (err == cudaSuccess && what == 1) err = ntt_forward(va, L, T, D.t, 0);
    if (what == 2)                                    // pob_r1cs_quotient's per-vector sequence, q over a
        for (uint4 *v : {va, vb, vc}) {
            if (err == cudaSuccess) err = ntt_inverse_coset(v, L, T, D.t, 0);
            if (err == cudaSuccess) err = v == vc ? ntt_forward(v, L, T, D.t, 0, va, vb, va) : ntt_forward(v, L, T, D.t, 0);
        }
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    return (int)err;
}

}  // namespace

extern "C" {

// ntt_plan(L, min(L, 11)) into stages[0..return value)
uint32_t ntt_probe_plan(uint32_t L, uint32_t *stages) {
    const std::vector<uint32_t> k = ntt_plan(L, std::min(L, NTT_TILE_LOG));
    for (size_t i = 0; i < k.size(); i++) stages[i] = k[i];
    return (uint32_t)k.size();
}
// the six tables of a 2^L domain as stored (Montgomery form), concatenated in the order w_lo, w_hi, loc, loc_inv, g_lo, g_hi;
// sizes[6] receives their entry counts and sizes[6] = g_log.  out == NULL only fills sizes.
void ntt_probe_tables(uint32_t L, uint64_t *sizes, uint32_t *out) {
    const NttHostTables H = ntt_host_tables(L);
    uint64_t at = 0, k = 0;
    for (const std::vector<Fr> *v : {&H.w_lo, &H.w_hi, &H.loc, &H.loc_inv, &H.g_lo, &H.g_hi}) {
        sizes[k++] = v->size();
        if (out) memcpy(out + 8 * at, v->data(), v->size() * sizeof(Fr));
        at += v->size();
    }
    sizes[6] = H.g_log;
}

int ntt_probe_inverse(uint32_t L, void *x) { return run(0, L, x, nullptr, nullptr); }
int ntt_probe_forward(uint32_t L, void *x) { return run(1, L, x, nullptr, nullptr); }
int ntt_probe_quotient(uint32_t L, void *a, void *b, void *c) { return run(2, L, a, b, c); }

}  // extern "C"
