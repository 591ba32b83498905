// tests/devprobe/g2_probe.cu -- TEST-ONLY front-end of the device F_q2 and G2 arithmetic (csrc/fq2_hd.h, and the point formulas of
// csrc/fq_hd.h over F_q2) behind pob_msm_g2 and pob_groth16_prove, for tests/test_gpu_msm_g2.py and tests/test_gpu_groth16.py.
// Nothing here is part of the product: libpob_b200.so never contains or calls this file.  Built by tests/devprobe/g2.py.
//
// g2_probe_elem / g2_probe_point take HOST arrays, run one device thread per element, copy the results back and return the
// cudaError_t.  g2_probe_fixed_base works on DEVICE arrays: the batched [k_i]G the tests build trapdoor proving keys with.
#include <cuda_runtime.h>
#include <cstring>
#include "fq2_hd.h"

using namespace pob;

namespace {

enum { FQ2_MUL = 0, FQ2_SQR = 1, FQ2_ADD = 2, FQ2_SUB = 3, FQ2_NEG = 4, FQ2_INV = 5 };
// point ops on affine Montgomery-form inputs a, b (O = all-zero); every result leaves through pt_to_affine_canonical
enum { G2_ADD = 0, G2_ADD_AFF = 1, G2_DBL = 2, G2_DBL_AFF = 3, G2_ADD_Z = 4, G2_ADD_AFF_Z = 5, G2_MUL_U32 = 6, G2_ADD_ZZ = 7 };

__global__ void k_fq2_elem(int op, const Fq2 *a, const Fq2 *b, Fq2 *out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fq2 r;
    switch (op) {
        case FQ2_MUL: r = fq2_mul(a[i], b[i]); break;
        case FQ2_SQR: r = fq2_sqr(a[i]); break;
        case FQ2_ADD: r = fq2_add(a[i], b[i]); break;
        case FQ2_SUB: r = fq2_sub(a[i], b[i]); break;
        case FQ2_NEG: r = fq2_neg(a[i]); break;
        default: r = fq2_inv(a[i]); break;
    }
    out[i] = r;
}

__global__ void k_g2_point(int op, const G2Aff *a, const G2Aff *b, const uint32_t *k, G2Aff *out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G2Xyzz pa = pt_from_aff(a[i]), pb = pt_from_aff(b[i]);
    G2Xyzz r;
    switch (op) {
        case G2_ADD: r = pt_add(pa, pb); break;
        case G2_ADD_AFF: r = pt_add_aff(pa, b[i]); break;
        case G2_DBL: r = pt_dbl(pa); break;
        case G2_DBL_AFF: r = pt_aff_is_inf(a[i]) ? pt_inf<Fq2>() : pt_dbl_aff(a[i]); break;
        case G2_ADD_Z: r = pt_add(pt_dbl(pa), pt_dbl(pb)); break;                  // 2a + 2b, both with Z != 1 (unless O)
        case G2_ADD_AFF_Z: r = pt_add_aff(pt_dbl(pa), b[i]); break;                // 2a + b
        case G2_MUL_U32: r = pt_mul_u32(pa, k[i]); break;
        default: r = pt_add(pt_mul_u32(pa, 3), pt_mul_u32(pb, 3)); break;          // 3a + 3b: Z != 1 on both sides, also for a = b
    }
    out[i] = pt_to_affine_canonical(r);
}

// out[i] = [k_i] G in the key form (affine, Montgomery, O = all-zero); k_i are 32-byte LE integers
template <class F>
__global__ void k_fixed_base(Aff<F> g, const uint4 *k, uint64_t n, Aff<F> *out) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4 lo = k[2 * i], hi = k[2 * i + 1];
        const uint32_t s[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
        Aff<F> a = pt_to_affine_canonical(pt_mul_u256(pt_from_aff(g), s));
        a.x = f_to_mont(a.x); a.y = f_to_mont(a.y);
        out[i] = a;
    }
}

template <class T>
int run(uint32_t n, const T *a, const T *b, const uint32_t *k, T *out, void (*launch)(const T *, const T *, const uint32_t *, T *)) {
    T *da = nullptr, *db = nullptr, *dout = nullptr;
    uint32_t *dk = nullptr;
    const size_t bytes = sizeof(T) * n;
    cudaError_t e = cudaMalloc(&da, bytes);
    if (e == cudaSuccess) e = cudaMalloc(&db, bytes);
    if (e == cudaSuccess) e = cudaMalloc(&dout, bytes);
    if (e == cudaSuccess) e = cudaMalloc(&dk, 4ull * n);
    if (e == cudaSuccess) e = cudaMemcpy(da, a, bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && b) e = cudaMemcpy(db, b, bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && k) e = cudaMemcpy(dk, k, 4ull * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) { launch(da, db, dk, dout); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, bytes, cudaMemcpyDeviceToHost);
    cudaFree(da); cudaFree(db); cudaFree(dout); cudaFree(dk);
    return (int)e;
}

int g_op;
uint32_t g_n;

}  // namespace

extern "C" {

// out[i] = op(a[i], b[i]) over F_q2, 16 x uint32 per element (c0 then c1; b may be NULL for unary ops)
int g2_probe_elem(int op, const uint32_t *a, const uint32_t *b, uint32_t *out, uint32_t n) {
    g_op = op; g_n = n;
    return run<Fq2>(n, (const Fq2 *)a, (const Fq2 *)b, nullptr, (Fq2 *)out, [](const Fq2 *x, const Fq2 *y, const uint32_t *, Fq2 *o) {
        k_fq2_elem<<<(g_n + 127) / 128, 128>>>(g_op, x, y ? y : x, o, g_n);
    });
}

// out[i] = canonical affine of op(a[i], b[i]) (32 x uint32 per point); k[i] is the scalar of G2_MUL_U32
int g2_probe_point(int op, const uint32_t *a, const uint32_t *b, const uint32_t *k, uint32_t *out, uint32_t n) {
    g_op = op; g_n = n;
    return run<G2Aff>(n, (const G2Aff *)a, (const G2Aff *)b, k, (G2Aff *)out, [](const G2Aff *x, const G2Aff *y, const uint32_t *kk, G2Aff *o) {
        k_g2_point<<<(g_n + 127) / 128, 128>>>(g_op, x, y, kk, o, g_n);
    });
}

// device arrays: out[i] = [k[i]] G over G1 (g2 == 0; g: 16 uint32, out: 64 B per point) or G2 (g2 != 0; g: 32 uint32, out: 128 B),
// g on the host in Montgomery form; waits for the result
int g2_probe_fixed_base(int g2, const uint32_t *g, const void *k, uint64_t n, void *out) {
    const unsigned grid = (unsigned)((n + 127) / 128 < 8192 ? (n + 127) / 128 : 8192);
    if (n == 0) return 0;
    if (g2) { G2Aff G; memcpy(&G, g, sizeof G); k_fixed_base<Fq2><<<grid, 128>>>(G, (const uint4 *)k, n, (G2Aff *)out); }
    else { G1Aff G; memcpy(&G, g, sizeof G); k_fixed_base<Fq><<<grid, 128>>>(G, (const uint4 *)k, n, (G1Aff *)out); }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

}  // extern "C"
