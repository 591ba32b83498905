// cons_check.h -- evaluation of the circuit's constraint records (program.h: ConsSet) against a materialised witness.
//
// __host__ __device__: the device instantiation is the on-GPU self-check (kernels.cuh: k_check_*, C-ABI pob_selfcheck);
// the host instantiation is used only by the test-only emulator (tests/emu/) to validate the constraint emitter against
// oracle witnesses on a machine without a GPU.
#pragma once
#include "program.h"
#include "vm_exec.h"

namespace pob {

static const uint32_t CONS_ONE = 0xffffffffu;        // "the constant 1" inside the block-relative KeccakfRound set

struct ConsView {                                    // one ConsSet in device (or host) memory
    const uint32_t *eq; uint64_t n_eq;               // pairs
    const ConsTerm *kc; uint64_t n_kc;
    const ConsR1 *r1; uint64_t n_r1;
    const ConsTerm *terms;
    POB_HD uint64_t n_records() const { return n_eq + n_kc + n_r1; }
};

// CONS_ONE is the constant wire w[0]: `one` is its value, 1 on every witness the circuit accepts (the .r1cs products pass the
// witness's own w[0], so that they stay the rows' linear forms on any witness)
POB_HD Fr cons_load(const uint64_t *wit, uint64_t base, uint32_t idx, const Fr &one = fr_from_u64(1)) {
    if (idx == CONS_ONE) return one;
    return vm_load_val(wit + 4ull * (base + idx));
}
POB_HD bool cons_eq_ok(const uint64_t *wit, uint64_t base, uint32_t a, uint32_t b) {
    const uint64_t *p = wit + 4ull * (base + a), *q = wit + 4ull * (base + b);
    return ((p[0] ^ q[0]) | (p[1] ^ q[1]) | (p[2] ^ q[2]) | (p[3] ^ q[3])) == 0;
}
// the constant a coefficient code stands for (rc = Keccak round constant of the enclosing round block)
POB_HD Fr cons_coef_value(uint32_t c, const Fr *konst, uint64_t rc) {
    const uint32_t k = cc_kind(c), p = cc_payload(c);
    if (k == CC_POS) return fr_from_u64(p);
    if (k == CC_NEG) return fr_neg(fr_from_u64(p));
    if (k == CC_KONST) return konst[p];
    return fr_from_u64((rc >> (p & 63)) & 1ull);
}
POB_HD bool cons_kc_ok(const uint64_t *wit, uint64_t base, const ConsTerm t, const Fr *konst, uint64_t rc) {
    return fr_eq(cons_load(wit, base, t.idx), cons_coef_value(t.coef, konst, rc));
}
POB_HD Fr cons_lc(const uint64_t *wit, uint64_t base, const ConsTerm *t, uint32_t n, const Fr *konst, const Fr &one = fr_from_u64(1)) {
    Fr acc = fr_zero();
    for (uint32_t i = 0; i < n; i++) {
        const Fr v = cons_load(wit, base, t[i].idx, one);
        const uint32_t k = cc_kind(t[i].coef), p = cc_payload(t[i].coef);
        if (k == CC_POS) acc = fr_add(acc, p == 1 ? v : fr_mul(v, fr_from_u64(p)));
        else if (k == CC_NEG) acc = fr_sub(acc, p == 1 ? v : fr_mul(v, fr_from_u64(p)));
        else acc = fr_add(acc, fr_mul(v, konst[p]));
    }
    return acc;
}
// (sum A) * (sum B) == (sum C); a record without A terms is linear: 0 == sum C
POB_HD bool cons_r1_ok(const uint64_t *wit, uint64_t base, const ConsR1 r, const ConsTerm *terms, const Fr *konst) {
    const ConsTerm *t = terms + r.off;
    const Fr C = cons_lc(wit, base, t + r.na + r.nb, r1_nc(r), konst);
    if (r.na == 0) return fr_is_zero(C);
    const Fr A = cons_lc(wit, base, t, r.na, konst), B = cons_lc(wit, base, t + r.na, r.nb, konst);
    return fr_eq(fr_mul(A, B), C);
}

}  // namespace pob
