// tests/devprobe/pairing_probe.cu -- TEST-ONLY front-end of the device tower and pairing (csrc/fq12_hd.h, csrc/pairing.cuh) behind
// pob_bn254_pairing and pob_groth16_verify, for tests/test_gpu_pairing_probe.py: single operations on caller-chosen operands, so that
// a wrong pairing shows which part is wrong.  Nothing here is part of the product: libpob_b200.so never contains or calls this file.
// Built by tests/devprobe/pairing.py.
//
// Both functions take HOST arrays (raw limbs: Montgomery form is the caller's business), run one device thread per element, copy the
// results back and return the cudaError_t.
#include <cuda_runtime.h>
#include "pairing.cuh"

namespace {

enum {
    P_FQ6_MUL = 0, P_FQ6_SQR, P_FQ6_INV, P_FQ12_MUL, P_FQ12_SQR, P_FQ12_INV, P_FQ12_CONJ, P_FROB1, P_FROB2, P_FROB3, P_CYC_SQR,
    P_MUL_034, P_FINAL_EXP
};

// out[i] = op(a[i], b[i]); the F_q6 ops use the c0 halves (the c1 half of the result is 0); P_MUL_034 takes its line (c0, c3, c4)
// from b[i].c0.c0, b[i].c0.c1, b[i].c0.c2
__global__ void k_probe_elem(int op, const Fq12 *a, const Fq12 *b, Fq12 *out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fq12 x = a[i], y = b[i];
    Fq12 r;
    r.c1 = fq6_zero();
    switch (op) {
        case P_FQ6_MUL: r.c0 = fq6_mul(x.c0, y.c0); break;
        case P_FQ6_SQR: r.c0 = fq6_sqr(x.c0); break;
        case P_FQ6_INV: r.c0 = fq6_inv(x.c0); break;
        case P_FQ12_MUL: r = fq12_mul(x, y); break;
        case P_FQ12_SQR: r = fq12_sqr(x); break;
        case P_FQ12_INV: r = fq12_inv(x); break;
        case P_FQ12_CONJ: r = fq12_conj(x); break;
        case P_FROB1: r = fq12_frob(x, 1); break;
        case P_FROB2: r = fq12_frob(x, 2); break;
        case P_FROB3: r = fq12_frob(x, 3); break;
        case P_CYC_SQR: r = fq12_cyc_sqr(x); break;
        case P_MUL_034: r = fq12_mul_034(x, y.c0.c0, y.c0.c1, y.c0.c2); break;
        default: r = pair_final_exp(x); break;
    }
    out[i] = r;
}

// the Miller loop alone (O on either side: 1) and the subgroup check [r]Q = O of each pair
__global__ void k_probe_miller(const G1Aff *p, const G2Aff *q, Fq12 *out, uint32_t *in_g2, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G1Aff pp = p[i];
    const G2Aff qq = q[i];
    const bool skip = pt_aff_is_inf(pp) || pt_aff_is_inf(qq);
    const PairLine *pre = nullptr;
    out[i] = pair_miller(&pp, &qq, &pre, &skip, 1);
    in_g2[i] = pair_in_g2(qq);
}

template <class T> cudaError_t up(T **d, const void *h, size_t bytes) {
    cudaError_t e = cudaMalloc(d, bytes);
    if (e == cudaSuccess && h) e = cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice);
    return e;
}

}  // namespace

extern "C" {

// a, b, out: n x 96 uint32 (12 F_q elements in the order c0.c0.c0, c0.c0.c1, .., c1.c2.c1)
int pairing_probe_elem(int op, const uint32_t *a, const uint32_t *b, uint32_t *out, uint32_t n) {
    Fq12 *da = nullptr, *db = nullptr, *dout = nullptr;
    const size_t bytes = sizeof(Fq12) * n;
    cudaError_t e = up(&da, a, bytes);
    if (e == cudaSuccess) e = up(&db, b ? b : a, bytes);
    if (e == cudaSuccess) e = up(&dout, nullptr, bytes);
    if (e == cudaSuccess) { k_probe_elem<<<(n + 63) / 64, 64>>>(op, da, db, dout, n); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, bytes, cudaMemcpyDeviceToHost);
    cudaFree(da); cudaFree(db); cudaFree(dout);
    return (int)e;
}

// p: n x 16 uint32 (G1, Montgomery), q: n x 32 uint32 (G2, Montgomery), out: n x 96 uint32, in_g2: n uint32
int pairing_probe_miller(const uint32_t *p, const uint32_t *q, uint32_t *out, uint32_t *in_g2, uint32_t n) {
    G1Aff *dp = nullptr; G2Aff *dq = nullptr; Fq12 *dout = nullptr; uint32_t *dg = nullptr;
    cudaError_t e = up(&dp, p, sizeof(G1Aff) * n);
    if (e == cudaSuccess) e = up(&dq, q, sizeof(G2Aff) * n);
    if (e == cudaSuccess) e = up(&dout, nullptr, sizeof(Fq12) * n);
    if (e == cudaSuccess) e = up(&dg, nullptr, 4ull * n);
    if (e == cudaSuccess) { k_probe_miller<<<(n + 63) / 64, 64>>>(dp, dq, dout, dg, n); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, sizeof(Fq12) * n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(in_g2, dg, 4ull * n, cudaMemcpyDeviceToHost);
    cudaFree(dp); cudaFree(dq); cudaFree(dout); cudaFree(dg);
    return (int)e;
}

}  // extern "C"
