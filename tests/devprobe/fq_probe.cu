// tests/devprobe/fq_probe.cu -- TEST-ONLY front-end of the device F_q and G1 arithmetic (csrc/fq_hd.h) behind pob_msm_g1, for
// tests/test_gpu_msm.py.  Nothing here is part of the product: libpob_b200.so never contains or calls this file.  Built by
// tests/devprobe/fq.py.
//
// Both entry points take HOST arrays, run one device thread per element, copy the results back and return the cudaError_t.
#include <cuda_runtime.h>
#include "fq_hd.h"

using namespace pob;

namespace {

enum { FQ_MUL = 0, FQ_ADD = 1, FQ_SUB = 2, FQ_INV = 3, FQ_TO_MONT = 4, FQ_FROM_MONT = 5, FQ_NEG = 6 };
// point ops on affine Montgomery-form inputs a, b (O = (0, 0)); every result leaves through g1_to_affine_canonical
enum { G1_ADD = 0, G1_ADD_AFF = 1, G1_DBL = 2, G1_DBL_AFF = 3, G1_ADD_Z = 4, G1_ADD_AFF_Z = 5, G1_MUL_U32 = 6 };

__global__ void k_fq_elem(int op, const Fq *a, const Fq *b, Fq *out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fq r;
    switch (op) {
        case FQ_MUL: r = fq_mul(a[i], b[i]); break;
        case FQ_ADD: r = fq_add(a[i], b[i]); break;
        case FQ_SUB: r = fq_sub(a[i], b[i]); break;
        case FQ_INV: r = fq_inv(a[i]); break;
        case FQ_TO_MONT: r = fq_to_mont(a[i]); break;
        case FQ_FROM_MONT: r = fq_from_mont(a[i]); break;
        default: r = fq_neg(a[i]); break;
    }
    out[i] = r;
}

__global__ void k_g1_point(int op, const G1Aff *a, const G1Aff *b, const uint32_t *k, G1Aff *out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G1Xyzz pa = g1_from_aff(a[i]), pb = g1_from_aff(b[i]);
    G1Xyzz r;
    switch (op) {
        case G1_ADD: r = g1_add(pa, pb); break;
        case G1_ADD_AFF: r = g1_add_aff(pa, b[i]); break;
        case G1_DBL: r = g1_dbl(pa); break;
        case G1_DBL_AFF: r = g1_aff_is_inf(a[i]) ? g1_inf() : g1_dbl_aff(a[i]); break;
        case G1_ADD_Z: r = g1_add(g1_dbl(pa), g1_dbl(pb)); break;                 // 2a + 2b, both with Z != 1
        case G1_ADD_AFF_Z: r = g1_add_aff(g1_dbl(pa), b[i]); break;               // 2a + b
        default: r = g1_mul_u32(pa, k[i]); break;
    }
    out[i] = g1_to_affine_canonical(r);
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

// out[i] = op(a[i], b[i]) over F_q, 8 x uint32 per element (b may be NULL for unary ops)
int fq_probe_elem(int op, const uint32_t *a, const uint32_t *b, uint32_t *out, uint32_t n) {
    g_op = op; g_n = n;
    return run<Fq>(n, (const Fq *)a, (const Fq *)b, nullptr, (Fq *)out, [](const Fq *x, const Fq *y, const uint32_t *, Fq *o) {
        k_fq_elem<<<(g_n + 127) / 128, 128>>>(g_op, x, y ? y : x, o, g_n);
    });
}

// out[i] = canonical affine of op(a[i], b[i]) (16 x uint32 per point: x then y); k[i] is the scalar of G1_MUL_U32
int fq_probe_point(int op, const uint32_t *a, const uint32_t *b, const uint32_t *k, uint32_t *out, uint32_t n) {
    g_op = op; g_n = n;
    return run<G1Aff>(n, (const G1Aff *)a, (const G1Aff *)b, k, (G1Aff *)out, [](const G1Aff *x, const G1Aff *y, const uint32_t *kk, G1Aff *o) {
        k_g1_point<<<(g_n + 127) / 128, 128>>>(g_op, x, y, kk, o, g_n);
    });
}

}  // extern "C"
