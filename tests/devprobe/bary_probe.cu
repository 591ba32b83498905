// tests/devprobe/bary_probe.cu -- TEST-ONLY barycentric evaluator of a device vector, for tests/test_gpu_quotient.py.
//
// Evaluates the polynomial through a vector that lives in device memory at one point, straight from the barycentric formula (no
// transform), on the device instantiation of csrc/fr_hd.h.  Vectors of the main shape (2^25 and 2^28 entries) are too long to
// evaluate in Python; tests/test_gpu_quotient.py checks this evaluator against the Python one (tests/quotient_model.py) on 2^22
// vectors before it relies on it.  Nothing here is part of the product: libpob_b200.so never contains or calls this file.
// Built by tests/devprobe/bary.py.
//
// The entry point takes a device vector and host scalars (8 x uint32 little-endian limbs, the Fr layout), allocates, launches,
// synchronises, copies the result out, frees and returns the cudaError_t.  No state survives a call.
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "fr_hd.h"

using namespace pob;

namespace {

const uint32_t THREADS = 256, CTAS = 1024;

// The polynomial of degree < n that takes v[i] at x_(first+i) = s w^(first+i) (0 at the points not given) is, at r,
// (r^n - s^n) / (n s^n) * sum_i v[i] x_i / (r - x_i).  Every thread folds its terms into one fraction num / den (num canonical, den
// in Montgomery form: N/D + a/d = (N d + a D) / (D d)); the CTA folds its threads' fractions, and k_bary_final folds the CTAs' and
// divides once.
__device__ __forceinline__ void bary_fold(Fr &N, Fr &D, const Fr &n, const Fr &d) { N = fr_add(fr_mont(N, d), fr_mont(n, D)); D = fr_mont(D, d); }
__device__ Fr pow_m(Fr b, uint64_t e) {                       // Montgomery form in and out
    Fr r = fr_to_mont(fr_from_u64(1));
    for (; e; e >>= 1) { if (e & 1) r = fr_mont(r, b); b = fr_mont(b, b); }
    return r;
}
__global__ void k_bary(const Fr *v, uint64_t first, uint64_t count, Fr s, Fr w, Fr r, Fr *fn, Fr *fd) {
    __shared__ Fr sn[THREADS], sd[THREADS];
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (uint64_t)gridDim.x * blockDim.x;
    const Fr wm = fr_to_mont(w), rm = fr_to_mont(r), step = pow_m(wm, stride);
    Fr x = fr_mont(pow_m(wm, first + t), fr_to_mont(s));        // x_i R
    Fr N = fr_zero(), D = fr_to_mont(fr_from_u64(1));
    for (uint64_t i = t; i < count; i += stride) {
        bary_fold(N, D, fr_mont(v[i], x), fr_sub(rm, x));
        x = fr_mont(x, step);
    }
    sn[threadIdx.x] = N; sd[threadIdx.x] = D;
    __syncthreads();
    for (uint32_t h = blockDim.x / 2; h; h >>= 1) {
        if (threadIdx.x < h) { Fr a = sn[threadIdx.x], b = sd[threadIdx.x]; bary_fold(a, b, sn[threadIdx.x + h], sd[threadIdx.x + h]); sn[threadIdx.x] = a; sd[threadIdx.x] = b; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { fn[blockIdx.x] = sn[0]; fd[blockIdx.x] = sd[0]; }
}
__global__ void k_bary_final(const Fr *fn, const Fr *fd, uint32_t parts, Fr s, Fr r, uint32_t log_n, Fr *out) {
    Fr N = fr_zero(), D = fr_to_mont(fr_from_u64(1));
    for (uint32_t i = 0; i < parts; i++) bary_fold(N, D, fn[i], fd[i]);
    const Fr sum = fr_mul(N, fr_inv(fr_from_mont(D)));
    const Fr rn = fr_from_mont(pow_m(fr_to_mont(r), 1ull << log_n)), sn = fr_from_mont(pow_m(fr_to_mont(s), 1ull << log_n));
    const Fr den = fr_mul(fr_from_u64(1ull << log_n), sn);
    *out = fr_mul(fr_mul(sum, fr_sub(rn, sn)), fr_inv(den));
}

Fr host_fr(const uint32_t *l) { Fr f; for (int i = 0; i < 8; i++) f.l[i] = l[i]; return f; }

}  // namespace

extern "C" {

// sum_i values[i] L_(first+i)(r) over the points s w^j of a 2^log_n domain (w its generator).  `values` is a DEVICE array of count
// canonical entries (a tensor of the caller); s, w, r and the result are host limbs.
int bary_probe_eval(const void *values, uint64_t first, uint64_t count, const uint32_t *s, const uint32_t *w, const uint32_t *r,
                    uint32_t log_n, uint32_t *result) {
    std::vector<void *> allocs;
    Fr *fn = nullptr, *fd = nullptr, *out = nullptr;
    cudaError_t err = cudaMalloc(&fn, CTAS * sizeof(Fr));
    if (fn) allocs.push_back(fn);
    if (err == cudaSuccess) { err = cudaMalloc(&fd, CTAS * sizeof(Fr)); if (fd) allocs.push_back(fd); }
    if (err == cudaSuccess) { err = cudaMalloc(&out, sizeof(Fr)); if (out) allocs.push_back(out); }
    if (err == cudaSuccess) {
        k_bary<<<CTAS, THREADS>>>((const Fr *)values, first, count, host_fr(s), host_fr(w), host_fr(r), fn, fd);
        err = cudaGetLastError();
    }
    if (err == cudaSuccess) { k_bary_final<<<1, 1>>>(fn, fd, CTAS, host_fr(s), host_fr(r), log_n, out); err = cudaGetLastError(); }
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    if (err == cudaSuccess) err = cudaMemcpy(result, out, sizeof(Fr), cudaMemcpyDeviceToHost);
    for (void *p : allocs) cudaFree(p);
    return (int)err;
}

}  // extern "C"
