// verify.cu -- host side of pob_bn254_pairing and pob_groth16_verify (include/pob_b200.h); the kernels live in pairing.cuh.  A
// translation unit of its own, so that the tower's constant table and the pairing code leave every other kernel's binary unchanged.
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <initializer_list>
#include <string>
#include "../../include/pob_b200.h"
#include "pairing.cuh"

// pob_last_error's message store lives in pob_b200.cu
void pob_set_error(const std::string &msg);

namespace {

int fail(int code, const std::string &msg) { pob_set_error(msg); return code; }
bool misaligned(std::initializer_list<const void *> bufs, uintptr_t a) {
    for (const void *p : bufs) if ((uintptr_t)p % a) return true;
    return false;
}
bool overlap(const void *a, uint64_t na, const void *b, uint64_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return na && nb && x < y + nb && y < x + na;
}
int set_device(const char *who, int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return fail(POB_E_NO_DEVICE, std::string(who) + ": no such CUDA device");
    if (cudaError_t e = cudaSetDevice(device)) return fail(POB_E_CUDA, std::string(who) + ": " + cudaGetErrorString(e));
    return POB_OK;
}
// a grid of `threads`-thread blocks covering n, at most 2^20 blocks (the kernels stride)
unsigned grid_for(uint64_t n, unsigned threads) { return (unsigned)std::min<uint64_t>((n + threads - 1) / threads, 1u << 20); }
int finish(const char *who, void *consumer_stream) {
    cudaError_t e = cudaGetLastError();
    if (!e && !consumer_stream) e = cudaStreamSynchronize(nullptr);
    return e ? fail(POB_E_CUDA, std::string(who) + ": " + cudaGetErrorString(e)) : POB_OK;
}

// one thread per pair or proof, 128 threads per block: the only shape measured (DESIGN.md §5 "Verification"), not yet chosen
// against others
constexpr unsigned PAIR_THREADS = 128;

}  // namespace

extern "C" {

int pob_bn254_pairing(int device, const void *g1, const void *g2, uint64_t n, void *out, void *consumer_stream) {
    const char *who = "pob_bn254_pairing";
    if (!g1 || !g2 || !out || n == 0) return fail(POB_E_BAD_ARG, std::string(who) + ": null argument or n == 0");
    if (misaligned({g1, g2, out}, 16)) return fail(POB_E_BAD_ARG, std::string(who) + ": g1, g2 and out must be 16-byte aligned");
    if (n > (1ull << 40)) return fail(POB_E_RANGE, std::string(who) + ": n exceeds 2^40");
    if (overlap(out, 384 * n, g1, 64 * n) || overlap(out, 384 * n, g2, 128 * n)) return fail(POB_E_BAD_ARG, std::string(who) + ": out overlaps g1 or g2");
    if (int rc = set_device(who, device)) return rc;
    const cudaStream_t st = (cudaStream_t)consumer_stream;
    k_bn254_pairing<<<grid_for(n, PAIR_THREADS), PAIR_THREADS, 0, st>>>((const uint4 *)g1, (const uint4 *)g2, n, (uint4 *)out);
    return finish(who, consumer_stream);
}

int pob_groth16_verify_work_bytes(uint32_t n_pub, uint64_t n, uint64_t *bytes) {
    (void)n_pub; (void)n;                                                // the layout does not depend on them
    if (!bytes) return fail(POB_E_BAD_ARG, "pob_groth16_verify_work_bytes: null argument");
    *bytes = verify_layout().bytes;
    return POB_OK;
}

int pob_groth16_verify(int device, const pob_groth16_vk *vk, const void *proofs, const void *publics, uint64_t n, uint32_t *status,
                       void *work, uint64_t work_bytes, void *consumer_stream) {
    const char *who = "pob_groth16_verify";
    const std::string w(who);
    if (!vk || !proofs || !status || !work || n == 0) return fail(POB_E_BAD_ARG, w + ": null argument or n == 0");
    if (!vk->alpha1 || !vk->beta2 || !vk->gamma2 || !vk->delta2 || !vk->ic) return fail(POB_E_BAD_ARG, w + ": null key pointer");
    if (vk->n_pub && !publics) return fail(POB_E_BAD_ARG, w + ": publics is null with n_pub > 0");
    if (misaligned({vk->alpha1, vk->beta2, vk->gamma2, vk->delta2, vk->ic, proofs, publics, work}, 16) || misaligned({status}, 4))
        return fail(POB_E_BAD_ARG, w + ": key points, proofs, publics and work must be 16-byte aligned, status 4-byte");
    if (n > (1ull << 40)) return fail(POB_E_RANGE, w + ": n exceeds 2^40");
    const VerifyLayout L = verify_layout();
    if (work_bytes < L.bytes) return fail(POB_E_BAD_ARG, w + ": work is shorter than pob_groth16_verify_work_bytes = " + std::to_string(L.bytes));
    const uint64_t pub_bytes = publics ? 32ull * vk->n_pub * n : 0;
    // the inputs: proofs, publics and the key's five point ranges; status and work are written, so neither may touch any of them
    // or each other
    const struct { const void *p; uint64_t bytes; } in[] = {{proofs, 256 * n}, {publics, pub_bytes}, {vk->alpha1, 64}, {vk->beta2, 128},
                                                            {vk->gamma2, 128}, {vk->delta2, 128}, {vk->ic, 64ull * (vk->n_pub + 1)}};
    for (const auto &x : in) {
        if (overlap(status, 4 * n, x.p, x.bytes)) return fail(POB_E_BAD_ARG, w + ": status overlaps proofs, publics or a key point");
        if (overlap(work, L.bytes, x.p, x.bytes)) return fail(POB_E_BAD_ARG, w + ": work overlaps proofs, publics or a key point");
    }
    if (overlap(status, 4 * n, work, L.bytes)) return fail(POB_E_BAD_ARG, w + ": status overlaps work");
    if (int rc = set_device(who, device)) return rc;
    const cudaStream_t st = (cudaStream_t)consumer_stream;
    const VerifyKeyDev k{vk->n_pub, (const uint4 *)vk->alpha1, (const uint4 *)vk->beta2, (const uint4 *)vk->gamma2, (const uint4 *)vk->delta2,
                         (const uint4 *)vk->ic};
    k_verify_prepare<<<1, VERIFY_PREP_THREADS, 0, st>>>(k, (uint8_t *)work);
    const VerifyArgs a{k, (const uint4 *)proofs, (const uint4 *)publics, n, status, (const uint8_t *)work};
    k_groth16_verify<<<grid_for(n, PAIR_THREADS), PAIR_THREADS, 0, st>>>(a);
    return finish(who, consumer_stream);
}

}  // extern "C"
