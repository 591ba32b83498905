// r1cs.cpp -- the iden3 `.r1cs` writer (binary format version 1) over a row plan (r1cs.h).
//
// File: "r1cs", u32 version = 1, u32 nSections = 3, then sections 1, 2, 3, each as u32 type, u64 byte size, content; all
// integers little-endian.  1 header: u32 fieldDefSize = 32, p (32 bytes LE), u32 nWires, nPubOut, nPubIn, nPrvIn, u64 nLabels,
// u32 mConstraints.  2 constraints: A, B, C of every row, each u32 nTerms then nTerms x (u32 wireId, 32-byte canonical LE
// coefficient); a row means A*B - C = 0.  3 wire-to-label map: nWires x u64.  Every size is known from the plan before the
// first byte, so the file is streamed through one buffer and never held in memory (a main-shape --O0 file is tens of GB).
#include "r1cs.h"
#include <cstdio>
#include <cstring>

namespace pob {
namespace {

struct Out {
    FILE *f = nullptr; std::string path; std::vector<char> buf; size_t used = 0; uint64_t total = 0;
    explicit Out(const std::string &p) : path(p), buf(16u << 20) {
        f = fopen(p.c_str(), "wb");
        if (!f) throw R1csIoError("cannot open " + p);
    }
    ~Out() { if (f) fclose(f); }
    void flush() { if (used && fwrite(buf.data(), 1, used, f) != used) throw R1csIoError("short write to " + path); total += used; used = 0; }
    void put(const void *p, size_t n) { if (used + n > buf.size()) flush(); memcpy(buf.data() + used, p, n); used += n; }
    void u32(uint32_t v) { put(&v, 4); }
    void u64(uint64_t v) { put(&v, 8); }
    void fr(const Fr &v) { put(v.l, 32); }                       // limbs are little-endian u32: the 32-byte LE form
    void term(uint64_t wire, const Fr &c) { u32((uint32_t)wire); fr(c); }
    uint64_t close() {
        flush();
        const int rc = fclose(f); f = nullptr;
        if (rc != 0) throw R1csIoError("short write to " + path);
        return total;
    }
};

// rows of one set of the plan (block base `base` and round constant rc; base 0 for the flat set)
void write_set(Out &o, const ConsSet &S, const std::vector<Fr> &konst, uint64_t base, uint64_t rc) {
    auto wire = [&](uint32_t idx) -> uint64_t { return idx == CONS_ONE ? 0 : base + idx; };
    const Fr one = fr_from_u64(1), minus_one = fr_neg(one);
    for (size_t i = 0; i + 1 < S.eq.size(); i += 2) {                 // C = w[a] - w[b]
        const uint64_t a = wire(S.eq[i]), b = wire(S.eq[i + 1]);
        o.u32(0); o.u32(0); o.u32(2);
        if (a < b) { o.term(a, one); o.term(b, minus_one); } else { o.term(b, minus_one); o.term(a, one); }
    }
    for (const ConsTerm &t : S.kc) {                                  // C = w[a] - k w0
        const uint64_t a = wire(t.idx);
        const Fr k = cons_coef_value(t.coef, konst.data(), rc);
        o.u32(0); o.u32(0);
        if (a == 0) { o.u32(1); o.term(0, fr_sub(one, k)); }
        else if (fr_is_zero(k)) { o.u32(1); o.term(a, one); }
        else { o.u32(2); o.term(0, fr_neg(k)); o.term(a, one); }
    }
    for (const ConsR1 &r : S.r1) {                                    // stored normalised: A, B (empty when A is), C
        const ConsTerm *t = S.terms.data() + r.off;
        for (uint32_t n : {(uint32_t)r.na, (uint32_t)r.nb, r1_nc(r)}) {
            o.u32(n);
            for (uint32_t i = 0; i < n; i++, t++) o.term(wire(t->idx), cons_coef_value(t->coef, konst.data(), 0));
        }
    }
}

}  // namespace

uint64_t write_r1cs(const RowPlan &R, const std::string &path) {
    const uint64_t rows = R.n_rows();
    if (R.n_wires > 0xffffffffull || rows > 0xffffffffull) throw std::runtime_error("pob: the system exceeds the 32-bit counts of the .r1cs header");
    Out o(path);
    o.put("r1cs", 4); o.u32(1); o.u32(3);
    o.u32(1); o.u64(64);
    o.u32(32); o.fr(fr_p());
    o.u32((uint32_t)R.n_wires); o.u32(R.n_outputs); o.u32(0); o.u32(R.n_inputs);   // no main declares public inputs
    o.u64(R.n_labels); o.u32((uint32_t)rows);
    o.u32(2); o.u64(12 * rows + 36 * R.n_terms);
    write_set(o, R.flat, R.konst, 0, 0);
    for (size_t b = 0; b < R.bases.size(); b++) write_set(o, R.round, R.konst, R.bases[b], keccak_rc((int)(b % 24)));
    o.u32(3); o.u64(8 * R.n_wires);
    for (uint64_t k = 0; k < R.n_wires; k++) o.u64(R.opt_level ? R.witness_map[k] : k);
    const uint64_t n = o.close();
    if (n != R.file_bytes()) throw std::runtime_error("pob: internal: .r1cs size " + std::to_string(n) + " differs from the plan's " + std::to_string(R.file_bytes()));
    return n;
}

}  // namespace pob
