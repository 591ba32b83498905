// compiler.cpp -- layout compiler for the proof-of-burn circuits (see compiler.h / program.h).
//
// One C++ function per circom template of the include closure of circuits/main_proof_of_burn.circom:27 and
// circuits/main_spend.circom:6.  Each function (i) reserves the component's own signals in circom's --O0
// order [outputs; inputs; intermediates], (ii) instantiates its sub-components in the order circom numbers
// them, (iii) records for every signal a 32-bit CODE saying where its value comes from, emitting VM ops for
// the values that actually have to be computed.  Copies (`a <== b`) cost nothing at run time: both signals
// get the same code.  Keccak lanes are 64-bit store words whose 64 bit-signals are BIT codes.
//
// Numbering rules: SURVEY.md Appendix C.  R3 default = completion order (circom >= 2.1 instantiates a
// sub-component when its last input is assigned); `hcreate` flips Num2Bits_strict and MultiAND(n>=3).
#include "compiler.h"
#include <sys/mman.h>
#include <algorithm>
#include <array>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <unordered_map>
#include "poseidon_constants_data.h"
#include "r1cs.h"
#include "vm_exec.h"

namespace pob {
namespace {

struct Blk { uint64_t sig; size_t pos; };          // first own signal: witness index and flat-code position
struct Lane { uint32_t w; };                       // lane word index in the store; NONE_IDX = constant zero lane

static const Code ZERO = 0, ONE = 1;

struct KeyHash {
    size_t operator()(const std::array<uint32_t, 4> &k) const {
        uint64_t h = 0x9E3779B97F4A7C15ULL;
        for (uint32_t v : k) { h ^= v; h *= 0xBF58476D1CE4E5B9ULL; h ^= h >> 29; }
        return (size_t)h;
    }
};
struct FrHash {
    size_t operator()(const std::array<uint32_t, 8> &k) const {
        uint64_t h = 0x9E3779B97F4A7C15ULL;
        for (uint32_t v : k) { h ^= v; h *= 0x94D049BB133111EBULL; h ^= h >> 31; }
        return (size_t)h;
    }
};

// linear combination over witness indices (index 0 = the constant 1), used only by the constraint emitter
struct LC {
    std::vector<std::pair<uint64_t, Fr>> t;
    static Fr I(int64_t v) { return v >= 0 ? fr_from_u64((uint64_t)v) : fr_neg(fr_from_u64((uint64_t)(-v))); }
    LC &s(uint64_t idx, int64_t c = 1) { t.push_back({idx, I(c)}); return *this; }
    LC &sf(uint64_t idx, const Fr &c) { t.push_back({idx, c}); return *this; }
    LC &k(int64_t c) { return s(0, c); }
    LC &kf(const Fr &c) { return sf(0, c); }
};

// constraint sink: one for the flat part (absolute witness indices), one for the shared KeccakfRound set (relative)
struct ConsSink {
    ConsSet *S = nullptr; std::vector<Fr> *konst = nullptr;
    std::unordered_map<std::array<uint32_t, 8>, uint32_t, FrHash> *kix = nullptr;
    uint32_t coef(const Fr &c) const {
        if (fr_fits64(c) && fr_lo64(c) < (1u << 30)) return (CC_POS << 30) | (uint32_t)fr_lo64(c);
        Fr n = fr_neg(c);
        if (fr_fits64(n) && fr_lo64(n) < (1u << 30)) return (CC_NEG << 30) | (uint32_t)fr_lo64(n);
        std::array<uint32_t, 8> key; memcpy(key.data(), c.l, 32);
        auto it = kix->find(key);
        uint32_t ix;
        if (it != kix->end()) ix = it->second; else { ix = (uint32_t)konst->size(); konst->push_back(c); kix->emplace(key, ix); }
        return (CC_KONST << 30) | ix;
    }
    void eq(uint64_t a, uint64_t b) { S->eq.push_back((uint32_t)a); S->eq.push_back((uint32_t)b); }
    void kc(uint64_t a, const Fr &v) { S->kc.push_back(ConsTerm{(uint32_t)a, coef(v)}); }
    void kc_raw(uint64_t a, uint32_t c) { S->kc.push_back(ConsTerm{(uint32_t)a, c}); }
    void r1(const LC &A, const LC &B, const LC &C, bool hint = false) {
        if (A.t.size() > 255 || B.t.size() > 255 || C.t.size() > 32767) throw std::runtime_error("pob: internal: constraint with too many terms in one combination");
        S->r1.push_back(ConsR1{(uint32_t)S->terms.size(), (uint16_t)(C.t.size() | (hint ? 0x8000u : 0u)), (uint8_t)A.t.size(), (uint8_t)B.t.size()});
        for (const LC *L : {&A, &B, &C}) for (auto &q : L->t) S->terms.push_back(ConsTerm{(uint32_t)q.first, coef(q.second)});
    }
};

class Builder {
  public:
    bool hcreate, dry;                 // dry: first pass, only counts lane words
    // ---- constraint emission (statement by statement from the circom sources; no-ops unless cs.S is set) ----
    ConsSink cs;
    bool want_cs() const { return cs.S != nullptr; }
    void q_eq(uint64_t a, uint64_t b) { if (cs.S) cs.eq(a, b); }                                 // `a <== b`, both signals
    void q_eqn(uint64_t a, uint64_t b, size_t n, size_t sa = 1, size_t sb = 1) { if (cs.S) for (size_t i = 0; i < n; i++) cs.eq(a + i * sa, b + i * sb); }
    void q_const(uint64_t a, uint64_t v) { if (cs.S) cs.kc(a, fr_from_u64(v)); }                 // `a <== 5`
    void q_constf(uint64_t a, const Fr &v) { if (cs.S) cs.kc(a, v); }
    void q_r1(const LC &A, const LC &Bq, const LC &C) { if (cs.S) cs.r1(A, Bq, C); }             // A * B == C
    void q_lin(const LC &C) { if (cs.S) cs.r1(LC(), LC(), C); }                                  // C == 0
    void q_mul(uint64_t a, uint64_t b, uint64_t c) { if (cs.S) cs.r1(LC().s(a), LC().s(b), LC().s(c)); }   // s[a]*s[b] == s[c]
    void q_hint(const LC &A, const LC &Bq, const LC &C) { if (cs.S) cs.r1(A, Bq, C, true); }     // pins a `<--` value the circuit leaves free
    uint32_t val_base;
    // flat codes (pointer-stable arena)
    Code *flat = nullptr; size_t flat_n = 0, flat_cap = (size_t)1 << 30;
    uint64_t nsig = 0;
    struct Seg { uint64_t dst; size_t pos; uint64_t n; bool round; uint32_t ubase; };
    std::vector<Seg> segs;
    // store
    uint32_t n_words = 0, n_vals = 0;
    std::vector<uint32_t> lvlW, lvlV;
    // program
    struct OpRec { Op op; uint32_t level; };
    std::vector<OpRec> ops;
    struct PsumRec { PsumOp op; uint32_t level; };
    std::vector<PsumRec> psums;
    std::vector<uint8_t> inv_generic;   // per value slot: 1 = an IsZero inverse whose input is expected to be a large value
    struct PosRec { PoseidonOp op; uint32_t level; };
    std::vector<PosRec> poseidons;
    std::vector<Fr> pos_konst; uint32_t pos_koff[6] = {~0u, ~0u, ~0u, ~0u, ~0u, ~0u};
    struct AbsRec { AbsorbOp op; uint32_t level; };
    std::vector<AbsRec> absorbs;
    std::vector<Code> aux;
    std::vector<Fr> konsts;
    std::unordered_map<std::array<uint32_t, 8>, uint32_t, FrHash> konst_ix;
    std::unordered_map<std::array<uint32_t, 4>, Code, KeyHash> cse;
    std::unordered_map<std::array<uint32_t, 4>, size_t, KeyHash> chk_ix;
    uint64_t n_round_blocks = 0;
    Code MINUS1;

    Builder(bool hc, bool dry_, uint32_t vb) : hcreate(hc), dry(dry_), val_base(vb) {
        flat = (Code *)mmap(nullptr, flat_cap * sizeof(Code), PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (flat == MAP_FAILED) throw std::runtime_error("pob: cannot reserve code arena");
        Fr m1; Fr one = fr_from_u64(1); fr_raw_sub(m1, fr_p(), one);
        MINUS1 = konst(m1);                             // must be konst index 0: vm_exec.h keys its negate fast path on it
        if (MINUS1 != c_konst(0)) throw std::runtime_error("pob: internal: MINUS1 must be the first table constant");
        Blk b = alloc(1); flat[b.pos] = ONE;            // witness[0] = 1
    }
    ~Builder() { if (flat && flat != MAP_FAILED) munmap(flat, flat_cap * sizeof(Code)); }

    // ---- signals ----
    // component list for the order-pinning kit (tools/diff_sym.py): every sub-component's own signals are one alloc()
    struct Comp { uint64_t sig; uint64_t n; const char *tmpl; };
    std::vector<Comp> *comps = nullptr;
    Blk alloc(size_t n, const char *tmpl = nullptr) {
        if (comps && tmpl) comps->push_back(Comp{nsig, n, tmpl});
        if (segs.empty() || segs.back().round) segs.push_back({nsig, flat_n, 0, false, 0});
        if (flat_n + n > flat_cap) throw std::runtime_error("pob: code arena exhausted");
        Blk b{nsig, flat_n};
        segs.back().n += n; flat_n += n; nsig += n;
        return b;
    }
    std::vector<uint64_t> round_sigs;  // first signal of every KeccakfRound block, in emission order
    void round_block(uint32_t ubase) {
        if (comps) comps->push_back(Comp{nsig, ROUND_SIGNALS, "KeccakfRound*"});       // expanded from the shared walk by the writer
        round_sigs.push_back(nsig);
        segs.push_back({nsig, 0, ROUND_SIGNALS, true, ubase});
        nsig += ROUND_SIGNALS; n_round_blocks++;
    }
    inline Code &at(size_t pos) { return flat[pos]; }
    void copy(size_t dst, const Code *src, size_t n) { memcpy(flat + dst, src, n * sizeof(Code)); }

    // ---- store ----
    uint32_t new_words(uint32_t n, uint32_t level) {
        uint32_t w = n_words; n_words += n;
        if (!dry && (uint64_t)n_words > val_base) throw std::runtime_error("pob: lane-word region overflow");
        lvlW.resize(n_words, level);
        return w;
    }
    uint32_t new_val(uint32_t level) { lvlV.push_back(level); return n_vals++; }
    uint32_t val_u64(uint32_t slot) const { return val_base + 4u * slot; }
    Code bit_of_val(uint32_t slot, uint32_t bit) const {
        uint32_t idx = val_u64(slot) + bit / 64;
        if (!dry && idx >= MAX_STORE_U64) throw std::runtime_error("pob: instance store exceeds 128 MiB (code range)");
        return c_bit(idx & (MAX_STORE_U64 - 1), bit % 64);
    }
    Code lane_bit(Lane l, uint32_t k) const { return l.w == NONE_IDX ? ZERO : c_bit(l.w, k); }
    void set_lane(size_t pos, Lane l) { for (uint32_t k = 0; k < 64; k++) flat[pos + k] = lane_bit(l, k); }

    uint32_t level_of(Code c) const {
        uint32_t k = code_kind(c), p = code_payload(c);
        if (k == K_VAL) return lvlV[p];
        if (k == K_BIT) { uint32_t idx = p >> 6; if (dry) return 0; return idx < val_base ? lvlW[idx] : lvlV[(idx - val_base) / 4]; }
        return 0;
    }

    // ---- constants ----
    Code konst(const Fr &v) {
        if (fr_fits64(v) && fr_lo64(v) < (1u << 30)) return c_const((uint32_t)fr_lo64(v));
        std::array<uint32_t, 8> k; memcpy(k.data(), v.l, 32);
        auto it = konst_ix.find(k);
        if (it != konst_ix.end()) return c_konst(it->second);
        uint32_t ix = (uint32_t)konsts.size(); konsts.push_back(v); konst_ix.emplace(k, ix);
        return c_konst(ix);
    }
    Code konst_u64(uint64_t v) { return konst(fr_from_u64(v)); }
    Code pow2(unsigned n) {                         // 2^n mod p
        Fr r = fr_from_u64(1); for (unsigned i = 0; i < n; i++) r = fr_add(r, r); return konst(r);
    }
    bool const_val(Code c, Fr &out) const {
        uint32_t k = code_kind(c);
        if (k == K_CONST) { out = fr_from_u64(code_payload(c)); return true; }
        if (k == K_KONST) { out = konsts[code_payload(c)]; return true; }
        return false;
    }
    bool is_zero(Code c) const { return c == ZERO; }

    // ---- value ops ----
    Code emit_val(uint32_t opc, Code a, Code b, Code c, uint32_t level) {
        std::array<uint32_t, 4> key{opc, a, b, c};
        auto it = cse.find(key);
        if (it != cse.end()) return it->second;
        uint32_t slot = new_val(level);
        if (slot >= (1u << 26)) throw std::runtime_error("pob: too many value slots");
        ops.push_back({Op{(opc << 26) | slot, a, b, c}, level});
        Code r = c_val(slot); cse.emplace(key, r); return r;
    }
    Code fma(Code a, Code b, Code c) {              // a*b + c
        Fr fa, fb, fc; bool ka = const_val(a, fa), kb = const_val(b, fb), kc = const_val(c, fc);
        if (ka && kb && kc) return konst(fr_add(fr_mul(fa, fb), fc));
        if ((ka && fr_is_zero(fa)) || (kb && fr_is_zero(fb))) return c;
        if (ka && kb) { a = konst(fr_mul(fa, fb)); b = ONE; fa = fr_mul(fa, fb); fb = fr_from_u64(1); }
        if (kc && fr_is_zero(fc)) {
            if (ka && fr_eq(fa, fr_from_u64(1))) return b;
            if (kb && fr_eq(fb, fr_from_u64(1))) return a;
        }
        if (ka && !kb) { std::swap(a, b); std::swap(ka, kb); std::swap(fa, fb); }   // keep the constant factor in `b` (VM fast paths)
        uint32_t lv = 1 + std::max(level_of(a), std::max(level_of(b), level_of(c)));
        return emit_val(OP_FMA, a, b, c, lv);
    }
    Code add(Code a, Code b) { return fma(a, ONE, b); }
    Code sub(Code a, Code b) { return fma(b, MINUS1, a); }
    Code mul(Code a, Code b) { return fma(a, b, ZERO); }
    Code not1(Code a) { return fma(a, MINUS1, ONE); }           // 1 - a
    Code isz(Code a) {
        Fr fa; if (const_val(a, fa)) return fr_is_zero(fa) ? ONE : ZERO;
        return emit_val(OP_ISZ, a, 0, 0, 1 + level_of(a));
    }
    Code inv(Code a, bool likely_large = false) {
        Fr fa; if (const_val(a, fa)) return fr_is_zero(fa) ? ZERO : konst(fr_inv(fa));
        Code r = emit_val(OP_INV, a, 0, 0, 1 + level_of(a));
        if (likely_large) { inv_generic.resize(n_vals, 0); inv_generic[code_payload(r)] = 1; }
        return r;
    }
    // (a > k) on canonical integers == prod_{j<=k} (1 - IsEqual(j, a))
    Code gtc(Code a, uint32_t k) {
        Fr fa; if (const_val(a, fa)) return (!fr_fits64(fa) || fr_lo64(fa) > k) ? ONE : ZERO;
        return emit_val(OP_GTC, a, k, 0, 1 + level_of(a));
    }
    // sum_{j<=i} IsEqual(sel, j) * vals[j]  for every i < n, as n independent ops over one shared operand list
    void selsum(Code sel, const Code *vals, size_t n, Code *out) {
        uint32_t lv = level_of(sel);
        for (size_t i = 0; i < n; i++) lv = std::max(lv, level_of(vals[i]));
        uint32_t a0 = (uint32_t)aux.size();
        aux.insert(aux.end(), vals, vals + n);
        for (size_t i = 0; i < n; i++) {
            uint32_t slot = new_val(lv + 1);
            ops.push_back({Op{(OP_SELSUM << 26) | slot, sel, a0, (uint32_t)i}, lv + 1});
            out[i] = c_val(slot);
        }
    }
    // V[k] = x0 + sum_{i<=k} terms[i], every partial sum a signal: one warp-level prefix-sum op
    void prefix_sum(Code x0, const Code *terms, size_t n, Code *out) {
        uint32_t lv = level_of(x0);
        for (size_t i = 0; i < n; i++) lv = std::max(lv, level_of(terms[i]));
        uint32_t a0 = (uint32_t)aux.size(); aux.insert(aux.end(), terms, terms + n);
        uint32_t first = n_vals;
        for (size_t i = 0; i < n; i++) { uint32_t slot = new_val(lv + 1); out[i] = c_val(slot); }
        psums.push_back({PsumOp{a0, (uint32_t)n, first, x0}, lv + 1});
    }
    // balanced sum of terms that are `var` accumulations in the circuit (only the total is a signal)
    Code sum_tree(std::vector<Code> v) {
        if (v.empty()) return ZERO;
        while (v.size() > 1) {
            std::vector<Code> nx; nx.reserve((v.size() + 1) / 2);
            for (size_t i = 0; i + 1 < v.size(); i += 2) nx.push_back(add(v[i], v[i + 1]));
            if (v.size() & 1) nx.push_back(v.back());
            v.swap(nx);
        }
        return v[0];
    }
    Code divmod(bool want_mod, Code a, Code b, uint64_t base) {
        uint32_t lv = 1 + std::max(level_of(a), level_of(b));
        return emit_val(want_mod ? OP_MOD : OP_DIV, a, b, (uint32_t)base, lv);
    }
    // ---- constraint checks ----
    void emit_chk(uint32_t opc, Code a, uint32_t b, uint64_t base, uint32_t level) {
        std::array<uint32_t, 4> key{opc, a, b, 0};
        auto it = chk_ix.find(key);
        if (it != chk_ix.end()) { Op &o = ops[it->second].op; if ((uint32_t)base < o.c) o.c = (uint32_t)base; return; }
        chk_ix.emplace(key, ops.size());
        ops.push_back({Op{opc << 26, a, b, (uint32_t)base}, level});
    }
    void chk_eq(Code a, Code b, uint64_t base) {
        Fr fa, fb;
        if (a == b) return;
        if (const_val(a, fa) && const_val(b, fb) && fr_eq(fa, fb)) return;
        emit_chk(OP_CHK_EQ, a, b, base, 1 + std::max(level_of(a), level_of(b)));
    }
    void chk_range(Code a, unsigned nbits, uint64_t base) {
        if (nbits >= 254) return;                    // every canonical value is < 2^254
        Fr fa;
        if (const_val(a, fa)) { if (!fr_lt_pow2(fa, nbits)) emit_chk(OP_CHK_EQ, ONE, ZERO, base, 1); return; }
        if (code_kind(a) == K_BIT && nbits >= 1) return;
        emit_chk(OP_CHK_RANGE, a, nbits, base, 1 + level_of(a));
    }
    // ---- lane ops ----
    uint32_t pack8_words(const Code *bytes, uint32_t nwords) {   // bytes[8*nwords] -> nwords consecutive lane words
        uint32_t lv = 0;
        for (uint32_t i = 0; i < 8 * nwords; i++) lv = std::max(lv, level_of(bytes[i]));
        uint32_t w0 = new_words(nwords, lv + 1);
        for (uint32_t w = 0; w < nwords; w++) {
            uint32_t a0 = (uint32_t)aux.size();
            for (int k = 0; k < 8; k++) aux.push_back(bytes[8 * w + k]);
            uint32_t l = 0; for (int k = 0; k < 8; k++) l = std::max(l, level_of(bytes[8 * w + k]));
            lvlW[w0 + w] = l + 1;
            ops.push_back({Op{(OP_PACK8 << 26) | (w0 + w), a0, 0, 0}, l + 1});
        }
        return w0;
    }
    // one Poseidon permutation as a warp op: returns the first slot of its value block (layout: program.h)
    uint32_t poseidon(uint32_t t, const Code *in) {
        if (t < 3 || t > 5) throw std::runtime_error("pob: Poseidon width outside this circuit's closure (t = 3, 4, 5)");
        const PosLayout L = pos_layout(t);
        if (pos_koff[t] == ~0u) {                       // C, S, M, P of this width, converted to Montgomery form once
            pos_koff[t] = (uint32_t)pos_konst.size();
            const uint64_t (*tabs[4])[4] = {t == 3 ? POSEIDON_C_T3 : t == 4 ? POSEIDON_C_T4 : POSEIDON_C_T5,
                                            t == 3 ? POSEIDON_S_T3 : t == 4 ? POSEIDON_S_T4 : POSEIDON_S_T5,
                                            t == 3 ? POSEIDON_M_T3 : t == 4 ? POSEIDON_M_T4 : POSEIDON_M_T5,
                                            t == 3 ? POSEIDON_P_T3 : t == 4 ? POSEIDON_P_T4 : POSEIDON_P_T5};
            const uint32_t cnt[4] = {t * 8 + L.rp, L.rp * (2 * t - 1), t * t, t * t};
            for (int k = 0; k < 4; k++) for (uint32_t i = 0; i < cnt[k]; i++) { Fr f; memcpy(f.l, tabs[k][i], 32); pos_konst.push_back(fr_to_mont(f)); }
        }
        uint32_t lv = 0; for (uint32_t j = 0; j < t; j++) lv = std::max(lv, level_of(in[j]));
        uint32_t a0 = (uint32_t)aux.size(); aux.insert(aux.end(), in, in + t);
        uint32_t base = n_vals;
        const uint32_t Q = pos_steps(L), Kseg = POS_SEGMENTS;
        for (uint32_t i = 0; i < L.total; i++) new_val(lv + Kseg);              // consumers see the block after the last segment
        for (uint32_t k = 0; k < Kseg; k++) poseidons.push_back({PoseidonOp{t, a0, base, pos_koff[t], k * Q / Kseg, (k + 1) * Q / Kseg}, lv + 1 + k});
        return base;
    }
    // one Absorb: returns base word of its ABSORB_WORDS block
    uint32_t absorb(uint32_t s_idx, uint32_t blk_idx) {
        uint32_t lv = 0;
        if (s_idx != NONE_IDX) for (int l = 0; l < 25; l++) lv = std::max(lv, dry ? 0u : lvlW[s_idx + l]);
        for (int l = 0; l < 17; l++) lv = std::max(lv, dry ? 0u : lvlW[blk_idx + l]);
        uint32_t out = new_words(ABSORB_WORDS, lv + 1);
        absorbs.push_back({AbsorbOp{s_idx, blk_idx, out, 0}, lv + 1});
        return out;
    }
};

// ---- constraint-emitter helpers -------------------------------------------------------------------------------
static Fr pow2_fr(unsigned n) { Fr r = fr_from_u64(1); for (unsigned i = 0; i < n; i++) r = fr_add(r, r); return r; }

// ============================================================================================================
// circomlib/circuits/gates.circom
// ============================================================================================================
// AND :29-35 (own: out, a, b).  Scalar XOR/OR only occur inside the Keccak lane arrays (handled as lanes).
static Blk T_AND(Builder &B, Code a, Code b) {
    Blk o = B.alloc(3, "AND"); B.at(o.pos + 1) = a; B.at(o.pos + 2) = b; B.at(o.pos) = B.mul(a, b);
    B.q_mul(o.sig + 1, o.sig + 2, o.sig);                                         // out <== a*b            gates.circom:34
    return o;
}
// MultiAND(n) :68-96
static Blk T_MultiAND(Builder &B, int n, const Code *in) {
    Blk o = B.alloc(1 + (size_t)n, "MultiAND"); B.copy(o.pos + 1, in, (size_t)n);
    if (n == 1) { B.at(o.pos) = in[0]; B.q_eq(o.sig, o.sig + 1); }                // out <== in[0]          :76
    else if (n == 2) {
        Blk a = T_AND(B, in[0], in[1]); B.at(o.pos) = B.at(a.pos);
        B.q_eq(a.sig + 1, o.sig + 1); B.q_eq(a.sig + 2, o.sig + 2); B.q_eq(o.sig, a.sig);   // :79-81
    } else {
        int n1 = n / 2, n2 = n - n / 2;
        Blk a2, x0, x1;
        if (B.hcreate) {
            a2 = B.alloc(3, "AND");
            x0 = T_MultiAND(B, n1, in); x1 = T_MultiAND(B, n2, in + n1);
            Code u = B.at(x0.pos), v = B.at(x1.pos);
            B.at(a2.pos + 1) = u; B.at(a2.pos + 2) = v; B.at(a2.pos) = B.mul(u, v); B.at(o.pos) = B.at(a2.pos);
            B.q_mul(a2.sig + 1, a2.sig + 2, a2.sig);
        } else {
            x0 = T_MultiAND(B, n1, in); x1 = T_MultiAND(B, n2, in + n1);
            a2 = T_AND(B, B.at(x0.pos), B.at(x1.pos)); B.at(o.pos) = B.at(a2.pos);
        }
        B.q_eqn(x0.sig + 1, o.sig + 1, (size_t)n1); B.q_eqn(x1.sig + 1, o.sig + 1 + (size_t)n1, (size_t)n2);   // :90-91
        B.q_eq(a2.sig + 1, x0.sig); B.q_eq(a2.sig + 2, x1.sig); B.q_eq(o.sig, a2.sig);                           // :92-94
    }
    return o;
}

// ============================================================================================================
// circomlib/circuits/bitify.circom, aliascheck.circom, compconstant.circom
// ============================================================================================================
// bit i of a value code
static Code bit_of(Builder &B, Code in, unsigned i) {
    Fr f;
    if (B.const_val(in, f)) return i < 256 ? c_const((uint32_t)fr_bit(f, i)) : ZERO;
    if (code_kind(in) == K_BIT) return i == 0 ? in : ZERO;
    return B.bit_of_val(code_payload(in), i);
}
// Num2Bits(n) :25-39  own: out[n], in
static Blk T_Num2Bits(Builder &B, int n, Code in) {
    Blk o = B.alloc((size_t)n + 1, "Num2Bits");
    for (int i = 0; i < n; i++) B.at(o.pos + (size_t)i) = bit_of(B, in, (unsigned)i);
    B.at(o.pos + (size_t)n) = in;
    B.chk_range(in, (unsigned)n, o.sig);
    if (B.want_cs()) {
        LC sum; Fr e2 = fr_from_u64(1);
        for (int i = 0; i < n; i++) {
            const uint64_t oi = o.sig + (uint64_t)i;
            B.q_r1(LC().s(oi), LC().s(oi).k(-1), LC());                          // out[i] * (out[i] - 1) === 0   bitify.circom:33
            sum.sf(oi, e2); e2 = fr_add(e2, e2);
        }
        sum.s(o.sig + (uint64_t)n, -1); B.q_lin(sum);                             // lc1 === in                     :38
    }
    return o;
}
// Bits2Num(n) :55-67  own: out, in[n]
static Blk T_Bits2Num(Builder &B, int n, const Code *in) {
    Blk o = B.alloc((size_t)n + 1, "Bits2Num"); B.copy(o.pos + 1, in, (size_t)n);
    std::vector<Code> terms; for (int i = 0; i < n; i++) terms.push_back(B.mul(in[i], B.pow2((unsigned)i)));
    B.at(o.pos) = B.sum_tree(terms);
    if (B.want_cs()) {
        LC sum; Fr e2 = fr_from_u64(1);
        for (int i = 0; i < n; i++) { sum.sf(o.sig + 1 + (uint64_t)i, e2); e2 = fr_add(e2, e2); }
        sum.s(o.sig, -1); B.q_lin(sum);                                           // lc1 ==> out                    bitify.circom:66
    }
    return o;
}
// CompConstant(ct) :25-73 with ct = p-1  own: out, in[254], parts[127], sout ; child Num2Bits(135)
static Blk T_CompConstant(Builder &B, const Fr &ct, const Code *in) {
    Blk o = B.alloc(1 + 254 + 127 + 1, "CompConstant"); B.copy(o.pos + 1, in, 254);
    size_t parts = o.pos + 255;
    Fr one = fr_from_u64(1);
    Fr b; { Fr t = fr_from_u64(1); for (int i = 0; i < 128; i++) t = fr_add(t, t); b = fr_sub(t, one); }
    Fr a = one, e = one;
    std::vector<Code> terms;
    LC sum;
    for (int i = 0; i < 127; i++) {
        int clsb = fr_bit(ct, (unsigned)(2 * i)), cmsb = fr_bit(ct, (unsigned)(2 * i + 1));
        Code slsb = in[2 * i], smsb = in[2 * i + 1], ml = B.mul(smsb, slsb), p;
        Code kb = B.konst(b), ka = B.konst(a), nkb = B.konst(fr_neg(b)), nka = B.konst(fr_neg(a));
        if (!cmsb && !clsb)      p = B.fma(slsb, kb, B.fma(smsb, kb, B.fma(ml, nkb, ZERO)));
        else if (!cmsb && clsb)  p = B.fma(smsb, nka, B.fma(smsb, kb, B.fma(slsb, nka, B.fma(ml, ka, ka))));
        else if (cmsb && !clsb)  p = B.fma(smsb, nka, B.fma(ml, kb, ka));
        else                     p = B.fma(ml, nka, ka);
        B.at(parts + (size_t)i) = p; terms.push_back(p);
        if (B.want_cs()) {                                                        // compconstant.circom:51-58, as (k*smsb) * slsb == linear
            const uint64_t L = o.sig + 1 + 2 * (uint64_t)i, M = L + 1, Pq = o.sig + 255 + (uint64_t)i;
            const Fr na = fr_neg(a), nb_ = fr_neg(b);
            if (!cmsb && !clsb)      B.q_r1(LC().sf(M, b), LC().s(L), LC().sf(M, b).sf(L, b).s(Pq, -1));            // p = -b*m*l + b*m + b*l
            else if (!cmsb && clsb)  B.q_r1(LC().sf(M, a), LC().s(L), LC().s(Pq).sf(L, a).sf(M, nb_).sf(M, a).kf(na)); // p = a*m*l - a*l + b*m - a*m + a
            else if (cmsb && !clsb)  B.q_r1(LC().sf(M, b), LC().s(L), LC().s(Pq).sf(M, a).kf(na));                  // p = b*m*l - a*m + a
            else                     B.q_r1(LC().sf(M, a), LC().s(L), LC().kf(a).s(Pq, -1));                         // p = -a*m*l + a
            sum.s(Pq);
        }
        b = fr_sub(b, e); a = fr_add(a, e); e = fr_add(e, e);
    }
    Code sumc = B.sum_tree(terms);
    B.at(o.pos + 255 + 127) = sumc;
    Blk nb = T_Num2Bits(B, 135, sumc);
    B.at(o.pos) = B.at(nb.pos + 127);
    if (B.want_cs()) {
        sum.s(o.sig + 255 + 127, -1); B.q_lin(sum);                               // sout <== sum                   :65
        B.q_eq(nb.sig + 135, o.sig + 255 + 127);                                  // num2bits.in <== sout           :69
        B.q_eq(o.sig, nb.sig + 127);                                              // out <== num2bits.out[127]      :71
    }
    return o;
}
// AliasCheck :24-32  own: in[254]
static Blk T_AliasCheck(Builder &B, const Code *in) {
    Blk o = B.alloc(254, "AliasCheck"); B.copy(o.pos, in, 254);
    Fr m1; Fr one = fr_from_u64(1); fr_raw_sub(m1, fr_p(), one);
    Blk cc = T_CompConstant(B, m1, in);
    B.chk_eq(B.at(cc.pos), ZERO, o.sig);
    B.q_eqn(cc.sig + 1, o.sig, 254);                                              // in[i] ==> compConstant.in[i]   aliascheck.circom:29
    B.q_const(cc.sig, 0);                                                         // compConstant.out === 0         :31
    return o;
}
// Num2Bits_strict :41-53  own: out[254], in
static Blk T_Num2Bits_strict(Builder &B, Code in) {
    Blk o = B.alloc(255, "Num2Bits_strict"); B.at(o.pos + 254) = in;
    Blk nb, ac;
    if (B.hcreate) {
        std::vector<Code> bits(254); for (int i = 0; i < 254; i++) bits[i] = bit_of(B, in, (unsigned)i);
        ac = T_AliasCheck(B, bits.data());
        nb = T_Num2Bits(B, 254, in); B.copy(o.pos, &B.at(nb.pos), 254);
    } else {
        nb = T_Num2Bits(B, 254, in); B.copy(o.pos, &B.at(nb.pos), 254);
        ac = T_AliasCheck(B, &B.at(nb.pos));
    }
    B.q_eq(nb.sig + 254, o.sig + 254);                                            // in ==> n2b.in                  bitify.circom:48
    B.q_eqn(o.sig, nb.sig, 254); B.q_eqn(ac.sig, nb.sig, 254);                    // n2b.out[i] ==> out[i], aliasCheck.in[i]   :50-51
    return o;
}

// ============================================================================================================
// circomlib/circuits/comparators.circom, mux1.circom
// ============================================================================================================
// IsZero :24-35  own: out, in, inv
static Blk T_IsZero(Builder &B, Code in, bool likely_large = false) {
    Blk o = B.alloc(3, "IsZero"); B.at(o.pos + 1) = in; B.at(o.pos + 2) = B.inv(in, likely_large); B.at(o.pos) = B.isz(in);
    if (B.want_cs()) {
        B.q_r1(LC().s(o.sig + 1), LC().s(o.sig + 2), LC().k(1).s(o.sig, -1));     // out <== -in*inv + 1            comparators.circom:32
        B.q_r1(LC().s(o.sig + 1), LC().s(o.sig), LC());                           // in*out === 0                   :33
        B.q_hint(LC().s(o.sig + 2), LC().s(o.sig), LC());                         // inv <-- in != 0 ? 1/in : 0     :30 (inv is free when in == 0)
    }
    return o;
}
// IsEqual :37-46  own: out, in[2] ; isz.in = in[1] - in[0]
static Blk T_IsEqual(Builder &B, Code in0, Code in1, bool likely_large = false) {
    Blk o = B.alloc(3, "IsEqual"); B.at(o.pos + 1) = in0; B.at(o.pos + 2) = in1;
    Blk z = T_IsZero(B, B.sub(in1, in0), likely_large); B.at(o.pos) = B.at(z.pos);
    B.q_lin(LC().s(z.sig + 1).s(o.sig + 2, -1).s(o.sig + 1));                     // in[1] - in[0] ==> isz.in       comparators.circom:43
    B.q_eq(o.sig, z.sig);                                                         // isz.out ==> out                :45
    return o;
}
// LessThan(n) :89-100
static Blk T_LessThan(Builder &B, int n, Code in0, Code in1) {
    Blk o = B.alloc(3, "LessThan"); B.at(o.pos + 1) = in0; B.at(o.pos + 2) = in1;
    Blk nb = T_Num2Bits(B, n + 1, B.sub(B.add(in0, B.pow2((unsigned)n)), in1));
    B.at(o.pos) = B.not1(B.at(nb.pos + (size_t)n));
    if (B.want_cs()) {
        B.q_lin(LC().s(nb.sig + (uint64_t)n + 1).s(o.sig + 1, -1).kf(fr_neg(pow2_fr((unsigned)n))).s(o.sig + 2));   // n2b.in <== in[0] + (1<<n) - in[1]   :96
        B.q_lin(LC().s(o.sig).k(-1).s(nb.sig + (uint64_t)n));                     // out <== 1 - n2b.out[n]         :98
    }
    return o;
}
// LessEqThan(n) :105-115
static Blk T_LessEqThan(Builder &B, int n, Code in0, Code in1) {
    Blk o = B.alloc(3, "LessEqThan"); B.at(o.pos + 1) = in0; B.at(o.pos + 2) = in1;
    Blk lt = T_LessThan(B, n, in0, B.add(in1, ONE)); B.at(o.pos) = B.at(lt.pos);
    B.q_eq(lt.sig + 1, o.sig + 1); B.q_lin(LC().s(lt.sig + 2).s(o.sig + 2, -1).k(-1)); B.q_eq(o.sig, lt.sig);   // comparators.circom:111-113
    return o;
}
// GreaterEqThan(n) :131-141
static Blk T_GreaterEqThan(Builder &B, int n, Code in0, Code in1) {
    Blk o = B.alloc(3, "GreaterEqThan"); B.at(o.pos + 1) = in0; B.at(o.pos + 2) = in1;
    Blk lt = T_LessThan(B, n, in1, B.add(in0, ONE)); B.at(o.pos) = B.at(lt.pos);
    B.q_eq(lt.sig + 1, o.sig + 2); B.q_lin(LC().s(lt.sig + 2).s(o.sig + 1, -1).k(-1)); B.q_eq(o.sig, lt.sig);   // comparators.circom:137-139
    return o;
}
// Mux1 :34-48 + MultiMux1(1) :21-32
static Blk T_Mux1(Builder &B, Code c0, Code c1, Code s) {
    Blk o = B.alloc(4, "Mux1"); B.at(o.pos + 1) = c0; B.at(o.pos + 2) = c1; B.at(o.pos + 3) = s;
    Blk m = B.alloc(4, "MultiMux1"); B.at(m.pos + 1) = c0; B.at(m.pos + 2) = c1; B.at(m.pos + 3) = s;
    B.at(m.pos) = B.fma(B.sub(c1, c0), s, c0);
    B.at(o.pos) = B.at(m.pos);
    if (B.want_cs()) {
        B.q_r1(LC().s(m.sig + 2).s(m.sig + 1, -1), LC().s(m.sig + 3), LC().s(m.sig).s(m.sig + 1, -1));   // out[i] <== (c[i][1] - c[i][0])*s + c[i][0]   mux1.circom:29
        B.q_eqn(m.sig + 1, o.sig + 1, 2); B.q_eq(m.sig + 3, o.sig + 3); B.q_eq(o.sig, m.sig);             // :43-47
    }
    return o;
}

// ============================================================================================================
// circomlib/circuits/poseidon.circom
// ============================================================================================================
// PoseidonEx(nInputs,1) :67-196  own: out[1], inputs[n], initialState.  The arithmetic is one warp op (Builder::poseidon);
// here only the circom numbering of its ~1100 signals is laid out over the op's value block.
static Blk T_PoseidonEx(Builder &B, int nInputs, const Code *inputs, Code initialState) {
    const uint32_t t = (uint32_t)nInputs + 1; const PosLayout L = pos_layout(t);
    Blk o = B.alloc(2 + (size_t)nInputs, "PoseidonEx"); B.copy(o.pos + 1, inputs, (size_t)nInputs); B.at(o.pos + 1 + (size_t)nInputs) = initialState;
    Code st[8], cur[8];
    st[0] = initialState; for (uint32_t j = 1; j < t; j++) st[j] = inputs[j - 1];
    const uint32_t base = B.poseidon(t, st);
    auto V = [&](uint32_t off) { return c_val(base + off); };
    // constraint side: canonical constant tables and the witness index of the signal carrying state element j
    const bool cs = B.want_cs();
    const uint64_t (*TC)[4] = t == 3 ? POSEIDON_C_T3 : t == 4 ? POSEIDON_C_T4 : POSEIDON_C_T5;
    const uint64_t (*TS)[4] = t == 3 ? POSEIDON_S_T3 : t == 4 ? POSEIDON_S_T4 : POSEIDON_S_T5;
    const uint64_t (*TM)[4] = t == 3 ? POSEIDON_M_T3 : t == 4 ? POSEIDON_M_T4 : POSEIDON_M_T5;
    const uint64_t (*TP)[4] = t == 3 ? POSEIDON_P_T3 : t == 4 ? POSEIDON_P_T4 : POSEIDON_P_T5;
    auto F = [](const uint64_t (*tab)[4], uint32_t i) { Fr f; memcpy(f.l, tab[i], 32); return f; };
    uint64_t cidx[8];
    {   // ark[0]  (Ark :18-25  own: out[t], in[t])
        Blk a = B.alloc(2 * t, "Ark");
        for (uint32_t j = 0; j < t; j++) {
            B.at(a.pos + j) = V(j); B.at(a.pos + t + j) = st[j]; cur[j] = V(j);
            if (cs) {
                B.q_eq(a.sig + t + j, j ? o.sig + 1 + (j - 1) : o.sig + 1 + (uint64_t)nInputs);      // ark[0].in[j] <== inputs[j-1] | initialState   :84-90
                B.q_lin(LC().s(a.sig + j).s(a.sig + t + j, -1).kf(fr_neg(F(TC, j))));                // out[i] <== in[i] + C[i + r]                    :23
            }
            cidx[j] = a.sig + j;
        }
    }
    auto sigma = [&](Code in, uint32_t off, uint64_t src) -> uint64_t {   // Sigma :5-16  own: out, in, in2, in4
        Blk s = B.alloc(4, "Sigma"); B.at(s.pos) = V(off + 2); B.at(s.pos + 1) = in; B.at(s.pos + 2) = V(off); B.at(s.pos + 3) = V(off + 1);
        if (cs) {
            B.q_eq(s.sig + 1, src);                                               // sigma.in <== previous layer's out
            B.q_mul(s.sig + 1, s.sig + 1, s.sig + 2); B.q_mul(s.sig + 2, s.sig + 2, s.sig + 3); B.q_mul(s.sig + 3, s.sig + 1, s.sig);   // :12-15
        }
        return s.sig;
    };
    auto full = [&](uint32_t Fo, uint32_t coff, const uint64_t (*MT)[4]) {   // t x Sigma, Ark :18-25, Mix :27-39
        uint64_t so[8];
        for (uint32_t j = 0; j < t; j++) so[j] = sigma(cur[j], Fo + 3 * j, cidx[j]);
        Blk a = B.alloc(2 * t, "Ark"); for (uint32_t j = 0; j < t; j++) { B.at(a.pos + j) = V(Fo + 3 * t + j); B.at(a.pos + t + j) = V(Fo + 3 * j + 2); }
        Blk m = B.alloc(2 * t, "Mix"); for (uint32_t j = 0; j < t; j++) { B.at(m.pos + j) = V(Fo + 4 * t + j); B.at(m.pos + t + j) = V(Fo + 3 * t + j); cur[j] = V(Fo + 4 * t + j); }
        if (cs) for (uint32_t j = 0; j < t; j++) {
            B.q_eq(a.sig + t + j, so[j]);                                         // ark.in[j] <== sigmaF[..][j].out
            B.q_lin(LC().s(a.sig + j).s(a.sig + t + j, -1).kf(fr_neg(F(TC, coff + j))));
            B.q_eq(m.sig + t + j, a.sig + j);                                     // mix.in[j] <== ark.out[j]
            LC l; l.s(m.sig + j, -1); for (uint32_t k = 0; k < t; k++) l.sf(m.sig + t + k, F(MT, k * t + j)); B.q_lin(l);   // out[i] <== sum_j M[j][i]*in[j]   :36
        }
        for (uint32_t j = 0; j < t; j++) cidx[j] = m.sig + j;
    };
    for (uint32_t f = 0; f < 4; f++) full(L.F1 + 5 * t * f, (f + 1) * t, f == 3 ? TP : TM);              // :101-136 (the 4th mixes with P)
    for (uint32_t r = 0; r < L.rp; r++) {                                            // :138-160
        const uint32_t Bs = L.PB + r * (4 + t);
        const uint64_t so = sigma(cur[0], Bs, cidx[0]);
        Blk m = B.alloc(2 * t, "MixS");                                              // MixS :52-65  own: out[t], in[t]
        for (uint32_t j = 0; j < t; j++) { B.at(m.pos + j) = V(Bs + 4 + j); B.at(m.pos + t + j) = j == 0 ? V(Bs + 3) : cur[j]; }
        for (uint32_t j = 0; j < t; j++) cur[j] = V(Bs + 4 + j);
        if (cs) {
            const uint32_t sb = (2 * t - 1) * r;
            B.q_lin(LC().s(m.sig + t).s(so, -1).kf(fr_neg(F(TC, 5 * t + r))));    // mixS.in[0] <== sigmaP.out + C[(nRoundsF\2+1)*t + r]   :149
            for (uint32_t j = 1; j < t; j++) B.q_eq(m.sig + t + j, cidx[j]);      // mixS.in[j] <== previous out[j]                        :151-155
            LC l; l.s(m.sig, -1); for (uint32_t i = 0; i < t; i++) l.sf(m.sig + t + i, F(TS, sb + i)); B.q_lin(l);        // out[0] <== lc       :60
            for (uint32_t i = 1; i < t; i++) B.q_lin(LC().s(m.sig + i, -1).s(m.sig + t + i).sf(m.sig + t, F(TS, sb + t + i - 1)));   // :62
        }
        for (uint32_t j = 0; j < t; j++) cidx[j] = m.sig + j;
    }
    for (uint32_t f = 0; f < 3; f++) full(L.SB + 5 * t * f, 5 * t + L.rp + f * t, TM);                  // :162-182
    uint64_t so[8];
    for (uint32_t j = 0; j < t; j++) so[j] = sigma(cur[j], L.LB + 3 * j, cidx[j]);  // :184-187
    Blk ml = B.alloc(1 + t, "MixLast");                                                         // MixLast :41-50  own: out, in[t]
    B.at(ml.pos) = V(L.LB + 3 * t); for (uint32_t j = 0; j < t; j++) B.at(ml.pos + 1 + j) = V(L.LB + 3 * j + 2);
    B.at(o.pos) = V(L.LB + 3 * t);
    if (cs) {
        LC l; l.s(ml.sig, -1);
        for (uint32_t j = 0; j < t; j++) { B.q_eq(ml.sig + 1 + j, so[j]); l.sf(ml.sig + 1 + j, F(TM, j * t)); }
        B.q_lin(l);                                                               // out <== sum_j M[j][s]*in[j], s = 0   :49
        B.q_eq(o.sig, ml.sig);                                                    // out[i] <== mixLast[i].out            :194
    }
    return o;
}
// Poseidon(n) :198-208
static Blk T_Poseidon(Builder &B, int n, const Code *inputs) {
    Blk o = B.alloc(1 + (size_t)n, "Poseidon"); B.copy(o.pos + 1, inputs, (size_t)n);
    Blk e = T_PoseidonEx(B, n, inputs, ZERO); B.at(o.pos) = B.at(e.pos);
    B.q_const(e.sig + 1 + (uint64_t)n, 0); B.q_eqn(e.sig + 1, o.sig + 1, (size_t)n); B.q_eq(o.sig, e.sig);   // poseidon.circom:203-207
    return o;
}

// ============================================================================================================
// circuits/utils/assert.circom
// ============================================================================================================
// AssertBits(B) :13-18  own: in, bits[B]
static Blk T_AssertBits(Builder &B, int nb_, Code in) {
    Blk o = B.alloc(1 + (size_t)nb_, "AssertBits"); B.at(o.pos) = in;
    Blk nb = T_Num2Bits(B, nb_, in); B.copy(o.pos + 1, &B.at(nb.pos), (size_t)nb_);
    B.q_eq(nb.sig + (uint64_t)nb_, o.sig); B.q_eqn(o.sig + 1, nb.sig, (size_t)nb_);   // signal bits[B] <== Num2Bits(B)(in)   assert.circom:17
    return o;
}
// AssertByteString(N) :26-31
static Blk T_AssertByteString(Builder &B, int N, const Code *in) {
    Blk o = B.alloc((size_t)N, "AssertByteString"); B.copy(o.pos, in, (size_t)N);
    for (int i = 0; i < N; i++) { Blk a = T_AssertBits(B, 8, in[i]); B.q_eq(a.sig, o.sig + (uint64_t)i); }   // AssertBits(8)(in[i])   assert.circom:29
    return o;
}
// AssertLessThan :40-47 / AssertLessEqThan :56-63 / AssertGreaterEqThan :72-79  own: a, b, out
static Blk T_AssertCmp(Builder &B, int kind, int nb, Code a, Code b) {
    Blk o = B.alloc(3, kind == 0 ? "AssertLessThan" : kind == 1 ? "AssertLessEqThan" : "AssertGreaterEqThan"); B.at(o.pos) = a; B.at(o.pos + 1) = b;
    Blk ba = T_AssertBits(B, nb, a), bb = T_AssertBits(B, nb, b);
    Blk r = kind == 0 ? T_LessThan(B, nb, a, b) : kind == 1 ? T_LessEqThan(B, nb, a, b) : T_GreaterEqThan(B, nb, a, b);
    B.at(o.pos + 2) = B.at(r.pos);
    B.chk_eq(B.at(r.pos), ONE, o.sig);
    B.q_eq(ba.sig, o.sig); B.q_eq(bb.sig, o.sig + 1);                             // AssertBits(B)(a); AssertBits(B)(b)      assert.circom:43-44
    B.q_eq(r.sig + 1, o.sig); B.q_eq(r.sig + 2, o.sig + 1); B.q_eq(o.sig + 2, r.sig);   // signal out <== LessThan(B)([a, b])   :45
    B.q_const(o.sig + 2, 1);                                                      // out === 1                                :46
    return o;
}
static Blk T_AssertLessThan(Builder &B, int nb, Code a, Code b) { return T_AssertCmp(B, 0, nb, a, b); }
static Blk T_AssertLessEqThan(Builder &B, int nb, Code a, Code b) { return T_AssertCmp(B, 1, nb, a, b); }
static Blk T_AssertGreaterEqThan(Builder &B, int nb, Code a, Code b) { return T_AssertCmp(B, 2, nb, a, b); }

// ============================================================================================================
// circuits/utils/array.circom
// ============================================================================================================
// Filter(N) :26-40  own: out[N], in, isEq[N]
static Blk T_Filter(Builder &B, int N, Code in) {
    size_t n = (size_t)N; Blk o = B.alloc(2 * n + 1, "Filter"); B.at(o.pos + n) = in;
    for (size_t i = 0; i < n; i++) {
        Blk e = T_IsEqual(B, c_const((uint32_t)i), in);
        Code eq = B.at(e.pos); B.at(o.pos + n + 1 + i) = eq;
        B.at(o.pos + i) = B.gtc(in, (uint32_t)i);      // prod_{j<=i} (1 - isEq[j]) == (in > i)
        if (B.want_cs()) {
            const uint64_t isEq = o.sig + n + 1 + i;
            B.q_const(e.sig + 1, i); B.q_eq(e.sig + 2, o.sig + n); B.q_eq(isEq, e.sig);       // isEq[i] <== IsEqual()([i, in])          array.circom:32
            if (i > 0) B.q_r1(LC().s(o.sig + i - 1), LC().k(1).s(isEq, -1), LC().s(o.sig + i));   // out[i] <== out[i-1] * (1 - isEq[i])   :34
            else B.q_lin(LC().s(o.sig).k(-1).s(isEq));                                        // out[0] <== 1 - isEq[0]                 :37
        }
    }
    return o;
}
// Fit(M,N) :47-57  own: out[N], in[M]
static Blk T_Fit(Builder &B, int M, int N, const Code *in) {
    Blk o = B.alloc((size_t)N + (size_t)M, "Fit"); B.copy(o.pos + (size_t)N, in, (size_t)M);
    for (int i = 0; i < N; i++) {
        B.at(o.pos + (size_t)i) = i < M ? in[i] : ZERO;
        if (i < M) B.q_eq(o.sig + (uint64_t)i, o.sig + (uint64_t)N + (uint64_t)i); else B.q_const(o.sig + (uint64_t)i, 0);   // array.circom:52-55
    }
    return o;
}
// Flatten(M,N) :64-72 / Reshape(M,N) :79-87: identity on row-major data  own: out[n], in[n]
static Blk T_CopyArray(Builder &B, size_t n, const Code *in) {
    Blk o = B.alloc(2 * n, "Flatten/Reshape"); B.copy(o.pos, in, n); B.copy(o.pos + n, in, n);
    B.q_eqn(o.sig, o.sig + n, n);                                                 // out[i*N + j] <== in[i][j]   array.circom:69 / :84
    return o;
}
// Reverse(N) :94-99
static Blk T_Reverse(Builder &B, int N, const Code *in) {
    size_t n = (size_t)N; Blk o = B.alloc(2 * n, "Reverse"); B.copy(o.pos + n, in, n);
    for (size_t i = 0; i < n; i++) { B.at(o.pos + i) = in[n - 1 - i]; B.q_eq(o.sig + i, o.sig + n + (n - 1 - i)); }   // out[i] <== in[N-1-i]   array.circom:97
    return o;
}

// ============================================================================================================
// circuits/utils/convert.circom
// ============================================================================================================
// LittleEndianBytes2Num(N) :12-26  own: out, in[N]
static Blk T_LittleEndianBytes2Num(Builder &B, int N, const Code *in) {
    Blk o = B.alloc(1 + (size_t)N, "LittleEndianBytes2Num"); B.copy(o.pos + 1, in, (size_t)N);
    Blk abs_ = T_AssertByteString(B, N, in);
    std::vector<Code> terms; for (int i = 0; i < N; i++) terms.push_back(B.mul(in[i], B.pow2((unsigned)(8 * i))));
    B.at(o.pos) = B.sum_tree(terms);
    if (B.want_cs()) {
        B.q_eqn(abs_.sig, o.sig + 1, (size_t)N);                                  // AssertByteString(N)(in)   convert.circom:19
        LC l; l.s(o.sig, -1); for (int i = 0; i < N; i++) l.sf(o.sig + 1 + (uint64_t)i, pow2_fr((unsigned)(8 * i))); B.q_lin(l);   // out <== lc   :25
    }
    return o;
}
// BigEndianBytes2Num(N) :33-39  own: out, in[N], inReversed[N]
static Blk T_BigEndianBytes2Num(Builder &B, int N, const Code *in) {
    size_t n = (size_t)N; Blk o = B.alloc(1 + 2 * n, "BigEndianBytes2Num"); B.copy(o.pos + 1, in, n);
    Blk r = T_Reverse(B, N, in); B.copy(o.pos + 1 + n, &B.at(r.pos), n);
    Blk l = T_LittleEndianBytes2Num(B, N, &B.at(r.pos)); B.at(o.pos) = B.at(l.pos);
    B.q_eqn(r.sig + n, o.sig + 1, n); B.q_eqn(o.sig + 1 + n, r.sig, n);           // signal inReversed[N] <== Reverse(N)(in)             convert.circom:37
    B.q_eqn(l.sig + 1, o.sig + 1 + n, n); B.q_eq(o.sig, l.sig);                   // out <== LittleEndianBytes2Num(N)(inReversed)        :38
    return o;
}
// Num2BitsSafe(N) :46-56
static Blk T_Num2BitsSafe(Builder &B, int N, Code in) {
    size_t n = (size_t)N;
    if (N >= 254) {
        Blk o = B.alloc(n + 1 + 254, "Num2BitsSafe"); B.at(o.pos + n) = in;
        Blk st = T_Num2Bits_strict(B, in); B.copy(o.pos + n + 1, &B.at(st.pos), 254);
        Blk f = T_Fit(B, 254, N, &B.at(st.pos)); B.copy(o.pos, &B.at(f.pos), n);
        B.q_eq(st.sig + 254, o.sig + n); B.q_eqn(o.sig + n + 1, st.sig, 254);     // signal bitsStrict[254] <== Num2Bits_strict()(in)   convert.circom:51
        B.q_eqn(f.sig + n, o.sig + n + 1, 254); B.q_eqn(o.sig, f.sig, n);         // out <== Fit(254, N)(bitsStrict)                    :52
        return o;
    }
    Blk o = B.alloc(n + 1, "Num2BitsSafe"); B.at(o.pos + n) = in;
    Blk nb = T_Num2Bits(B, N, in); B.copy(o.pos, &B.at(nb.pos), n);
    B.q_eq(nb.sig + n, o.sig + n); B.q_eqn(o.sig, nb.sig, n);                     // out <== Num2Bits(N)(in)                            :54
    return o;
}
// Num2LittleEndianBytes(N) :69-82  own: out[N], in, bits[8N], byteArrays[N][8]
static Blk T_Num2LittleEndianBytes(Builder &B, int N, Code in) {
    size_t n = (size_t)N; Blk o = B.alloc(n + 1 + 16 * n, "Num2LittleEndianBytes"); B.at(o.pos + n) = in;
    Blk b = T_Num2BitsSafe(B, 8 * N, in); B.copy(o.pos + n + 1, &B.at(b.pos), 8 * n);
    Blk r = T_CopyArray(B, 8 * n, &B.at(b.pos)); B.copy(o.pos + n + 1 + 8 * n, &B.at(r.pos), 8 * n);
    B.q_eq(b.sig + 8 * n, o.sig + n); B.q_eqn(o.sig + n + 1, b.sig, 8 * n);       // signal bits[N*8] <== Num2BitsSafe(N*8)(in)          convert.circom:77
    B.q_eqn(r.sig + 8 * n, o.sig + n + 1, 8 * n); B.q_eqn(o.sig + n + 1 + 8 * n, r.sig, 8 * n);   // signal byteArrays[N][8] <== Reshape(N, 8)(bits)   :78
    for (size_t i = 0; i < n; i++) {
        Blk bn = T_Bits2Num(B, 8, &B.at(r.pos + 8 * i)); B.at(o.pos + i) = B.at(bn.pos);
        B.q_eqn(bn.sig + 1, o.sig + n + 1 + 8 * n + 8 * i, 8); B.q_eq(o.sig + i, bn.sig);   // out[i] <== Bits2Num(8)(byteArrays[i])   :80
    }
    return o;
}
// Num2BigEndianBytes(N) :90-96  own: out[N], in, littleEndian[N]
static Blk T_Num2BigEndianBytes(Builder &B, int N, Code in) {
    size_t n = (size_t)N; Blk o = B.alloc(2 * n + 1, "Num2BigEndianBytes"); B.at(o.pos + n) = in;
    Blk le = T_Num2LittleEndianBytes(B, N, in); B.copy(o.pos + n + 1, &B.at(le.pos), n);
    Blk rv = T_Reverse(B, N, &B.at(le.pos)); B.copy(o.pos, &B.at(rv.pos), n);
    B.q_eq(le.sig + n, o.sig + n); B.q_eqn(o.sig + n + 1, le.sig, n);             // signal littleEndian[N] <== Num2LittleEndianBytes(N)(in)   convert.circom:94
    B.q_eqn(rv.sig + n, o.sig + n + 1, n); B.q_eqn(o.sig, rv.sig, n);             // out <== Reverse(N)(littleEndian)                          :95
    return o;
}
// Bytes2Nibbles(N) :103-125  own: out[2N], in[N], inDecomposed[N][8]
static Blk T_Bytes2Nibbles(Builder &B, int N, const Code *in) {
    size_t n = (size_t)N; Blk o = B.alloc(11 * n, "Bytes2Nibbles"); B.copy(o.pos + 2 * n, in, n);
    for (size_t i = 0; i < n; i++) {
        Blk nb = T_Num2Bits(B, 8, in[i]); B.copy(o.pos + 3 * n + 8 * i, &B.at(nb.pos), 8);
        Code lo = ZERO, hi = ZERO;
        for (unsigned j = 0; j < 4; j++) {
            lo = B.fma(B.at(nb.pos + j), B.pow2(j), lo);
            hi = B.fma(B.at(nb.pos + j + 4), B.pow2(j), hi);
        }
        B.at(o.pos + 2 * i) = hi; B.at(o.pos + 2 * i + 1) = lo;
        if (B.want_cs()) {
            const uint64_t dec = o.sig + 3 * n + 8 * i;
            B.q_eq(nb.sig + 8, o.sig + 2 * n + i); B.q_eqn(dec, nb.sig, 8);       // inDecomposed[i] <== Num2Bits(8)(in[i])   convert.circom:110
            LC h, l; h.s(o.sig + 2 * i, -1); l.s(o.sig + 2 * i + 1, -1);
            for (unsigned j = 0; j < 4; j++) { l.s(dec + j, 1 << j); h.s(dec + j + 4, 1 << j); }
            B.q_lin(h); B.q_lin(l);                                               // out[2i] <== higher; out[2i+1] <== lower  :122-123
        }
    }
    return o;
}
// Nibbles2Bytes(n) :132-141  own: bytes[n], nibbles[2n]
static Blk T_Nibbles2Bytes(Builder &B, int n_, const Code *nib) {
    size_t n = (size_t)n_; Blk o = B.alloc(3 * n, "Nibbles2Bytes"); B.copy(o.pos + n, nib, 2 * n);
    for (size_t i = 0; i < n; i++) {
        Blk a0 = T_AssertBits(B, 4, nib[2 * i]), a1 = T_AssertBits(B, 4, nib[2 * i + 1]);
        B.at(o.pos + i) = B.fma(nib[2 * i], c_const(16), nib[2 * i + 1]);
        B.q_eq(a0.sig, o.sig + n + 2 * i); B.q_eq(a1.sig, o.sig + n + 2 * i + 1);                      // AssertBits(4)(nibbles[2i]), (nibbles[2i+1])   convert.circom:136-137
        B.q_lin(LC().s(o.sig + i, -1).s(o.sig + n + 2 * i, 16).s(o.sig + n + 2 * i + 1));             // bytes[i] <== nibbles[2i]*16 + nibbles[2i+1]   :138
    }
    return o;
}

// ============================================================================================================
// circuits/utils/divide.circom
// ============================================================================================================
// Divide(N) :17-33  own: out, rem, a, b
static Blk T_Divide(Builder &B, int N, Code a, Code b) {
    Blk o = B.alloc(4, "Divide");
    Code q, r; Fr fa, fb;
    if (B.const_val(a, fa) && B.const_val(b, fb) && !fr_is_zero(fb)) { Fr fq, fr_; fr_divmod(fa, fb, fq, fr_); q = B.konst(fq); r = B.konst(fr_); }
    else { q = B.divmod(false, a, b, o.sig); r = B.divmod(true, a, b, o.sig); }
    B.at(o.pos) = q; B.at(o.pos + 1) = r; B.at(o.pos + 2) = a; B.at(o.pos + 3) = b;
    Blk lt = T_AssertLessThan(B, N, r, b);
    Blk le = T_AssertLessEqThan(B, N, q, a);
    B.chk_eq(B.fma(q, b, r), a, o.sig);
    B.q_eq(lt.sig, o.sig + 1); B.q_eq(lt.sig + 1, o.sig + 3);                     // AssertLessThan(N)(rem, b)     divide.circom:27
    B.q_eq(le.sig, o.sig); B.q_eq(le.sig + 1, o.sig + 2);                         // AssertLessEqThan(N)(out, a)   :30
    B.q_r1(LC().s(o.sig), LC().s(o.sig + 3), LC().s(o.sig + 2).s(o.sig + 1, -1)); // out * b + rem === a           :32
    return o;
}

// ============================================================================================================
// circuits/utils/selector.circom
// ============================================================================================================
// Selector(n) :21-46  own: out, vals[n], select, isEq[n], sum[n+1]
static Blk T_Selector(Builder &B, int n_, const Code *vals, Code select) {
    size_t n = (size_t)n_; Blk o = B.alloc(1 + n + 1 + n + n + 1, "Selector");
    B.copy(o.pos + 1, vals, n); B.at(o.pos + 1 + n) = select;
    size_t isEq = o.pos + 2 + n, sum = isEq + n;
    const uint64_t qSel = o.sig + 1 + n, qEq = o.sig + 2 + n, qSum = qEq + n;
    B.at(sum) = ZERO; B.q_const(qSum, 0);                                         // sum[0] <== 0                            selector.circom:30
    LC all;
    for (size_t i = 0; i < n; i++) {
        Blk e = T_IsEqual(B, select, c_const((uint32_t)i)); B.at(isEq + i) = B.at(e.pos);
        if (B.want_cs()) {
            B.q_eq(e.sig + 1, qSel); B.q_const(e.sig + 2, i); B.q_eq(qEq + i, e.sig);                 // isEq[i] <== IsEqual()([select, i])      :33
            B.q_r1(LC().s(qEq + i), LC().s(o.sig + 1 + i), LC().s(qSum + i + 1).s(qSum + i, -1));    // sum[i+1] <== sum[i] + isEq[i]*vals[i]   :39
            all.s(qEq + i);
        }
    }
    B.selsum(select, vals, n, &B.at(sum + 1));          // sum[i+1] = sum_{j<=i} isEq[j]*vals[j]
    B.chk_eq(B.gtc(select, (uint32_t)(n - 1)), ZERO, o.sig);   // sumIsEq === 1  <=>  select in [0, n)
    if (B.want_cs()) { all.k(-1); B.q_lin(all); B.q_eq(o.sig, qSum + n); }        // sumIsEq === 1 ; out <== sum[n]           :43-45
    B.at(o.pos) = B.at(sum + n); return o;
}
// SelectorArray1D(n,p) :62-77 / SelectorArray2D(n,p,q) :91-110  own: out[cols], arrays[n][cols], select, arraysT[cols][n]
static Blk T_SelectorArray(Builder &B, int n_, size_t cols, const Code *arrays, Code select) {
    size_t n = (size_t)n_; Blk o = B.alloc(cols + n * cols + 1 + cols * n, "SelectorArray1D/2D");
    B.copy(o.pos + cols, arrays, n * cols); B.at(o.pos + cols + n * cols) = select;
    size_t T = o.pos + cols + n * cols + 1;
    const uint64_t qArr = o.sig + cols, qSel = o.sig + cols + n * cols, qT = qSel + 1;
    for (size_t i = 0; i < n; i++) for (size_t j = 0; j < cols; j++) { B.at(T + j * n + i) = arrays[i * cols + j]; B.q_eq(qT + j * n + i, qArr + i * cols + j); }   // arraysT[j][i] <== arrays[i][j]   :69 / :101
    for (size_t j = 0; j < cols; j++) {
        Blk s = T_Selector(B, n_, &B.at(T + j * n), select); B.at(o.pos + j) = B.at(s.pos);
        B.q_eqn(s.sig + 1, qT + j * n, n); B.q_eq(s.sig + 1 + n, qSel); B.q_eq(o.sig + j, s.sig);   // out[i] <== Selector(n)(arraysT[i], select)   :75 / :107
    }
    return o;
}

// ============================================================================================================
// circuits/utils/shift.circom, concat.circom
// ============================================================================================================
// ShiftLeft(n) :17-36  own: out[n], in[n], count, isEq[n][n], temp[n][n]
static Blk T_ShiftLeft(Builder &B, int n_, const Code *in, Code count) {
    size_t n = (size_t)n_; Blk o = B.alloc(2 * n + 1 + 2 * n * n, "ShiftLeft");
    B.copy(o.pos + n, in, n); B.at(o.pos + 2 * n) = count;
    size_t isEq = o.pos + 2 * n + 1, temp = isEq + n * n;
    const uint64_t qIn = o.sig + n, qCnt = o.sig + 2 * n, qEq = qCnt + 1, qTmp = qEq + n * n;
    Blk al = T_AssertLessEqThan(B, 16, count, c_const((uint32_t)n));
    B.q_eq(al.sig, qCnt); B.q_const(al.sig + 1, n);                               // AssertLessEqThan(16)(count, n)          shift.circom:22
    for (size_t i = 0; i < n; i++) {
        std::vector<Code> terms;
        LC row;
        for (size_t j = 0; j < n; j++) {
            Blk e = T_IsEqual(B, c_const((uint32_t)i), B.sub(c_const((uint32_t)j), count));
            Code eq = B.at(e.pos); B.at(isEq + i * n + j) = eq;
            Code tv = B.mul(eq, in[j]); B.at(temp + i * n + j) = tv; terms.push_back(tv);
            if (B.want_cs()) {
                B.q_const(e.sig + 1, i); B.q_lin(LC().s(e.sig + 2).k(-(int64_t)j).s(qCnt)); B.q_eq(qEq + i * n + j, e.sig);   // isEq[i][j] <== IsEqual()([i, j - count])   :29
                B.q_mul(qEq + i * n + j, qIn + j, qTmp + i * n + j);                                                             // temp[i][j] <== isEq[i][j] * in[j]          :30
                row.s(qTmp + i * n + j);
            }
        }
        B.at(o.pos + i) = B.sum_tree(terms);
        if (B.want_cs()) { row.s(o.sig + i, -1); B.q_lin(row); }                  // out[i] <== outVars[i]                   :33
    }
    return o;
}
// ShiftRight(n,maxShift) :51-75  own: out[n+ms], in[n], count, isEq[ms+1], temps[ms+1][n]
static Blk T_ShiftRight(Builder &B, int n_, int ms_, const Code *in, Code count) {
    size_t n = (size_t)n_, ms = (size_t)ms_; Blk o = B.alloc(n + ms + n + 1 + ms + 1 + (ms + 1) * n, "ShiftRight");
    B.copy(o.pos + n + ms, in, n); B.at(o.pos + 2 * n + ms) = count;
    size_t isEq = o.pos + 2 * n + ms + 1, temps = isEq + ms + 1;
    const uint64_t qIn = o.sig + n + ms, qCnt = o.sig + 2 * n + ms, qEq = qCnt + 1, qTmp = qEq + ms + 1;
    Blk al = T_AssertLessEqThan(B, 16, count, c_const((uint32_t)ms));
    B.q_eq(al.sig, qCnt); B.q_const(al.sig + 1, ms);                              // AssertLessEqThan(16)(count, maxShift)   shift.circom:56
    std::vector<std::vector<Code>> acc(n + ms);
    std::vector<LC> rows(B.want_cs() ? n + ms : 0);
    for (size_t i = 0; i <= ms; i++) {
        Blk e = T_IsEqual(B, c_const((uint32_t)i), count); Code eq = B.at(e.pos); B.at(isEq + i) = eq;
        B.q_const(e.sig + 1, i); B.q_eq(e.sig + 2, qCnt); B.q_eq(qEq + i, e.sig);                                // isEq[i] <== IsEqual()([i, count])       :64
        for (size_t j = 0; j < n; j++) {
            Code tv = B.mul(eq, in[j]); B.at(temps + i * n + j) = tv; acc[i + j].push_back(tv);
            if (B.want_cs()) { B.q_mul(qEq + i, qIn + j, qTmp + i * n + j); rows[i + j].s(qTmp + i * n + j); }   // temps[i][j] <== isEq[i] * in[j]         :66
        }
    }
    for (size_t k = 0; k < n + ms; k++) {
        B.at(o.pos + k) = B.sum_tree(acc[k]);
        if (B.want_cs()) { rows[k].s(o.sig + k, -1); B.q_lin(rows[k]); }          // out[i] <== outVars[i]                   :72
    }
    return o;
}
// Mask(n) :18-30  own: out[n], in[n], count, filter[n]
static Blk T_Mask(Builder &B, int n_, const Code *in, Code count) {
    size_t n = (size_t)n_; Blk o = B.alloc(3 * n + 1, "Mask"); B.copy(o.pos + n, in, n); B.at(o.pos + 2 * n) = count;
    Blk f = T_Filter(B, n_, count); B.copy(o.pos + 2 * n + 1, &B.at(f.pos), n);
    B.q_eq(f.sig + n, o.sig + 2 * n); B.q_eqn(o.sig + 2 * n + 1, f.sig, n);       // signal filter[n] <== Filter(n)(count)   concat.circom:24
    for (size_t i = 0; i < n; i++) { B.at(o.pos + i) = B.mul(in[i], B.at(f.pos + i)); B.q_mul(o.sig + n + i, o.sig + 2 * n + 1 + i, o.sig + i); }   // out[i] <== in[i] * filter[i]   :27
    return o;
}
// Concat(A,B) :47-84  own: out[A+B], outLen, a[A], aLen, b[B], bLen, maskedA[A], maskedB[B], shiftedB[A+B]
static Blk T_Concat(Builder &B, int A, int Bn, const Code *a, Code aLen, const Code *b, Code bLen) {
    size_t NA = (size_t)A, NB = (size_t)Bn, T = NA + NB;
    Blk o = B.alloc(T + 1 + NA + 1 + NB + 1 + NA + NB + T, "Concat");
    size_t ia = o.pos + T + 1, iaL = ia + NA, ib = iaL + 1, ibL = ib + NB, mA = ibL + 1, mB = mA + NA, sB = mB + NB;
    const uint64_t d = o.sig - o.pos;                                             // flat position -> witness index inside this block
    B.copy(ia, a, NA); B.at(iaL) = aLen; B.copy(ib, b, NB); B.at(ibL) = bLen;
    Blk la = T_AssertLessEqThan(B, 16, aLen, c_const((uint32_t)A));
    Blk lb = T_AssertLessEqThan(B, 16, bLen, c_const((uint32_t)Bn));
    Blk ma = T_Mask(B, A, a, aLen); B.copy(mA, &B.at(ma.pos), NA);
    Blk mb = T_Mask(B, Bn, b, bLen); B.copy(mB, &B.at(mb.pos), NB);
    Blk sh = T_ShiftRight(B, Bn, A, &B.at(mb.pos), aLen); B.copy(sB, &B.at(sh.pos), T);
    for (size_t i = 0; i < T; i++) B.at(o.pos + i) = i < NA ? B.add(B.at(ma.pos + i), B.at(sh.pos + i)) : B.at(sh.pos + i);
    B.at(o.pos + T) = B.add(aLen, bLen);
    if (B.want_cs()) {
        B.q_eq(la.sig, d + iaL); B.q_const(la.sig + 1, NA); B.q_eq(lb.sig, d + ibL); B.q_const(lb.sig + 1, NB);      // AssertLessEqThan(16)(aLen, maxLenA), (bLen, maxLenB)   concat.circom:67-68
        B.q_eqn(ma.sig + NA, d + ia, NA); B.q_eq(ma.sig + 2 * NA, d + iaL); B.q_eqn(d + mA, ma.sig, NA);              // maskedA <== Mask(maxLenA)(a, aLen)                     :70
        B.q_eqn(mb.sig + NB, d + ib, NB); B.q_eq(mb.sig + 2 * NB, d + ibL); B.q_eqn(d + mB, mb.sig, NB);              // maskedB <== Mask(maxLenB)(b, bLen)                     :71
        B.q_eqn(sh.sig + T, d + mB, NB); B.q_eq(sh.sig + T + NB, d + iaL); B.q_eqn(d + sB, sh.sig, T);                // shiftedB <== ShiftRight(maxLenB, maxLenA)(maskedB, aLen)   :73
        for (size_t i = 0; i < T; i++) {
            if (i < NA) B.q_lin(LC().s(o.sig + i, -1).s(d + mA + i).s(d + sB + i));                                   // out[i] <== maskedA[i] + shiftedB[i]                    :77
            else B.q_eq(o.sig + i, d + sB + i);                                                                       // out[i] <== shiftedB[i]                                 :79
        }
        B.q_lin(LC().s(o.sig + T, -1).s(d + iaL).s(d + ibL));                                                         // outLen <== aLen + bLen                                 :83
    }
    return o;
}

// ============================================================================================================
// circuits/utils/substring_check.circom
// ============================================================================================================
// SubstringCheck(maxMainLen, subLen) :24-100
static Blk T_SubstringCheck(Builder &B, int maxMainLen, int subLen, const Code *mainInput, Code mainLen, const Code *subInput) {
    size_t MM = (size_t)maxMainLen, SL = (size_t)subLen, Kn = MM - SL + 1;
    Blk o = B.alloc(1 + MM + 1 + SL + 1 + (MM + 1) + Kn + Kn + (Kn + 1) + (Kn + 1) + 1, "SubstringCheck");
    size_t iMain = o.pos + 1, iLen = iMain + MM, iSub = iLen + 1, subNum = iSub + SL, Mo = subNum + 1,
           exists = Mo + MM + 1, isLast = exists + Kn, allowed = isLast + Kn, sums = allowed + Kn + 1, dne = sums + Kn + 1;
    const uint64_t d = o.sig - o.pos;
    const bool cs = B.want_cs();
    B.copy(iMain, mainInput, MM); B.at(iLen) = mainLen; B.copy(iSub, subInput, SL);
    Blk as = T_AssertByteString(B, subLen, subInput);
    Blk am = T_AssertByteString(B, maxMainLen, mainInput);
    Blk l1 = T_AssertLessEqThan(B, 16, mainLen, c_const((uint32_t)MM));
    Blk l2 = T_AssertLessEqThan(B, 16, c_const((uint32_t)SL), mainLen);
    Blk sn = T_LittleEndianBytes2Num(B, subLen, subInput); Code subN = B.at(sn.pos); B.at(subNum) = subN;
    if (cs) {
        B.q_eqn(as.sig, d + iSub, SL); B.q_eqn(am.sig, d + iMain, MM);                                    // AssertByteString(subLen)(subInput), (maxMainLen)(mainInput)   substring_check.circom:33-34
        B.q_eq(l1.sig, d + iLen); B.q_const(l1.sig + 1, MM); B.q_const(l2.sig, SL); B.q_eq(l2.sig + 1, d + iLen);   // :36-37
        B.q_eqn(sn.sig + 1, d + iSub, SL); B.q_eq(d + subNum, sn.sig);                                    // subInputNum <== LittleEndianBytes2Num(subLen)(subInput)     :40
        B.q_const(d + Mo, 0); B.q_const(d + allowed, 1); B.q_const(d + sums, 0);                          // M[0] <== 0; allowed[0] <== 1; sums[0] <== 0                 :46, :61, :65
    }
    B.at(Mo) = ZERO;
    Fr pw = fr_from_u64(1), c256 = fr_from_u64(256);
    {   // M[i+1] = mainInput[i]*256^i + M[i]
        std::vector<Code> terms(MM);
        for (size_t i = 0; i < MM; i++) {
            terms[i] = B.mul(mainInput[i], B.konst(pw));
            if (cs) B.q_lin(LC().s(d + Mo + i + 1, -1).sf(d + iMain + i, pw).s(d + Mo + i));              // M[i+1] <== mainInput[i]*(256**i) + M[i]                     :48
            pw = fr_mul(pw, c256);
        }
        B.prefix_sum(ZERO, terms.data(), MM, &B.at(Mo + 1));
    }
    B.at(allowed) = ONE; B.at(sums) = ZERO;
    pw = fr_from_u64(1);
    Code lastIdx = B.add(B.sub(mainLen, c_const((uint32_t)SL)), ONE);
    std::vector<Code> sterms(Kn);
    for (size_t i = 0; i < Kn; i++) {
        Blk e1 = T_IsEqual(B, c_const((uint32_t)i), lastIdx); B.at(isLast + i) = B.at(e1.pos);
        B.at(allowed + i + 1) = B.gtc(lastIdx, (uint32_t)i);       // allowed[i]*(1 - isLastIndex[i]) == (lastIdx > i)
        Blk e2 = T_IsEqual(B, B.mul(subN, B.konst(pw)), B.sub(B.at(Mo + i + SL), B.at(Mo + i)), /*likely_large=*/true);
        Code ex = B.at(e2.pos); B.at(exists + i) = ex;
        sterms[i] = B.mul(B.at(allowed + i + 1), ex);
        if (cs) {
            B.q_const(e1.sig + 1, i); B.q_lin(LC().s(e1.sig + 2).s(d + iLen, -1).k((int64_t)SL - 1)); B.q_eq(d + isLast + i, e1.sig);   // isLastIndex[i] <== IsEqual()([i, mainLen - subLen + 1])   :72
            B.q_r1(LC().s(d + allowed + i), LC().k(1).s(d + isLast + i, -1), LC().s(d + allowed + i + 1));                               // allowed[i+1] <== allowed[i] * (1 - isLastIndex[i])         :75
            B.q_lin(LC().s(e2.sig + 1).sf(d + subNum, fr_neg(pw))); B.q_lin(LC().s(e2.sig + 2).s(d + Mo + i + SL, -1).s(d + Mo + i));
            B.q_eq(d + exists + i, e2.sig);                                                                                               // exists[i] <== IsEqual()([subInputNum*(256**i), M[i+subLen] - M[i]])   :91
            B.q_r1(LC().s(d + allowed + i + 1), LC().s(d + exists + i), LC().s(d + sums + i + 1).s(d + sums + i, -1));                   // sums[i+1] <== sums[i] + allowed[i+1]*exists[i]             :95
        }
        pw = fr_mul(pw, c256);
    }
    B.prefix_sum(ZERO, sterms.data(), Kn, &B.at(sums + 1));   // sums[i+1] = sums[i] + allowed[i+1]*exists[i]
    Blk z = T_IsZero(B, B.at(sums + Kn)); B.at(dne) = B.at(z.pos);
    B.at(o.pos) = B.not1(B.at(z.pos));
    if (cs) {
        B.q_eq(z.sig + 1, d + sums + Kn); B.q_eq(d + dne, z.sig);                 // doesNotExist <== IsZero()(sums[maxMainLen - subLen + 1])   :98
        B.q_lin(LC().s(o.sig).k(-1).s(d + dne));                                  // out <== 1 - doesNotExist                                    :99
    }
    return o;
}

// ============================================================================================================
// circuits/utils/keccak.circom -- lane level.  A lane is a store word; its 64 signals are BIT codes.
// The emitters below write codes sequentially through a cursor because inside the Keccak sub-circuit every
// lane word index is known from the layout alone.
// ============================================================================================================
struct LaneSink {
    Code *p;
    uint32_t base;                       // added to every lane word (0 when emitting the shared relative table)
    void lane(Lane l) { for (uint32_t k = 0; k < 64; k++) *p++ = (l.w == NONE_IDX) ? ZERO : c_bit(base + l.w, k); }
    // XorArray/OrArray/AndArray(64) :77-128 -- own out,a,b then 64 gates [out,a,b]   (384 signals)
    void gate_array(Lane out, Lane a, Lane b) {
        lane(out); lane(a); lane(b);
        for (uint32_t k = 0; k < 64; k++) {
            *p++ = (out.w == NONE_IDX) ? ZERO : c_bit(base + out.w, k);
            *p++ = (a.w == NONE_IDX) ? ZERO : c_bit(base + a.w, k);
            *p++ = (b.w == NONE_IDX) ? ZERO : c_bit(base + b.w, k);
        }
    }
    void unary(Lane out, Lane in) { lane(out); lane(in); }   // ShL/ShR :19-51, NotArray :92-98  (128 signals)
};
// KeccakfRound(r) :290-297 relative to the round base (see program.h for the word map)
static void emit_round(LaneSink &S) {
    auto W = [](uint32_t w) { return Lane{w}; };
    Lane in[25], th[25], rp[25], ch[25], out[25];
    for (int l = 0; l < 25; l++) { in[l] = W((uint32_t)l); th[l] = W(rw_th(l)); ch[l] = W(rw_ch(l, 2)); out[l] = W(rw_out(l)); }
    rp[0] = th[0];
    for (int i = 0; i < 24; i++) rp[keccak_rot(i + 1)] = W(rw_rp(i, 2));
    // own: out, in, theta, rhopi, chi
    for (int l = 0; l < 25; l++) S.lane(out[l]);
    for (int l = 0; l < 25; l++) S.lane(in[l]);
    for (int l = 0; l < 25; l++) S.lane(th[l]);
    for (int l = 0; l < 25; l++) S.lane(rp[l]);
    for (int l = 0; l < 25; l++) S.lane(ch[l]);
    // Theta :151-170  own: out, in, c[5], d[5]
    for (int l = 0; l < 25; l++) S.lane(th[l]);
    for (int l = 0; l < 25; l++) S.lane(in[l]);
    for (int i = 0; i < 5; i++) S.lane(W(rw_x5(i, 3)));
    for (int i = 0; i < 5; i++) S.lane(W(rw_dd(i, 3)));
    for (int i = 0; i < 5; i++) {        // Xor5(64) :58-70  own: out,a,b,c,d,e,xor_ab,xor_abc,xor_abcd
        S.lane(W(rw_x5(i, 3)));
        for (int j = 0; j < 5; j++) S.lane(in[5 * j + i]);
        S.lane(W(rw_x5(i, 0))); S.lane(W(rw_x5(i, 1))); S.lane(W(rw_x5(i, 2)));
        S.gate_array(W(rw_x5(i, 0)), in[i], in[5 + i]);
        S.gate_array(W(rw_x5(i, 1)), W(rw_x5(i, 0)), in[10 + i]);
        S.gate_array(W(rw_x5(i, 2)), W(rw_x5(i, 1)), in[15 + i]);
        S.gate_array(W(rw_x5(i, 3)), W(rw_x5(i, 2)), in[20 + i]);
    }
    for (int i = 0; i < 5; i++) {        // D :135-144  own: out,a,b,aux0,aux1,aux2
        Lane a = W(rw_x5((i + 1) % 5, 3)), b = W(rw_x5((i + 4) % 5, 3));
        S.lane(W(rw_dd(i, 3))); S.lane(a); S.lane(b); S.lane(W(rw_dd(i, 0))); S.lane(W(rw_dd(i, 1))); S.lane(W(rw_dd(i, 2)));
        S.unary(W(rw_dd(i, 0)), a);                                   // ShL(64,1)
        S.unary(W(rw_dd(i, 1)), a);                                   // ShR(64,63)
        S.gate_array(W(rw_dd(i, 2)), W(rw_dd(i, 0)), W(rw_dd(i, 1)));   // OrArray
        S.gate_array(W(rw_dd(i, 3)), b, W(rw_dd(i, 2)));                // XorArray(b, aux2)
    }
    for (int i = 0; i < 5; i++) for (int j = 0; j < 5; j++) S.gate_array(th[i + 5 * j], in[i + 5 * j], W(rw_dd(i, 3)));
    // RhoPi :191-204  own: out, in
    for (int l = 0; l < 25; l++) S.lane(rp[l]);
    for (int l = 0; l < 25; l++) S.lane(th[l]);
    for (int i = 0; i < 24; i++) {       // stepRhoPi :177-184  own: out,a,aux0,aux1
        Lane a = th[keccak_rot(i)];
        S.lane(W(rw_rp(i, 2))); S.lane(a); S.lane(W(rw_rp(i, 0))); S.lane(W(rw_rp(i, 1)));
        S.unary(W(rw_rp(i, 0)), a);                                   // ShR(64,shr)
        S.unary(W(rw_rp(i, 1)), a);                                   // ShL(64,shl)
        S.gate_array(W(rw_rp(i, 2)), W(rw_rp(i, 0)), W(rw_rp(i, 1)));
    }
    // Chi :228-241  own: out, in
    for (int l = 0; l < 25; l++) S.lane(ch[l]);
    for (int l = 0; l < 25; l++) S.lane(rp[l]);
    for (int l = 0; l < 25; l++) {       // stepChi :212-221  own: out,a,b,c,bXor,bc
        Lane a = rp[l], b = rp[chi_b(l)], c = rp[chi_c(l)];
        S.lane(ch[l]); S.lane(a); S.lane(b); S.lane(c); S.lane(W(rw_ch(l, 0))); S.lane(W(rw_ch(l, 1)));
        S.unary(W(rw_ch(l, 0)), b);                                   // NotArray
        S.gate_array(W(rw_ch(l, 1)), W(rw_ch(l, 0)), c);              // AndArray
        S.gate_array(ch[l], a, W(rw_ch(l, 1)));                       // XorArray
    }
    // Iota(r) :273-283  own: out, in, roundConstants
    for (int l = 0; l < 25; l++) S.lane(out[l]);
    for (int l = 0; l < 25; l++) S.lane(ch[l]);
    S.lane(W(RW_RC));
    S.lane(W(RW_RC));                                                 // RoundConstants(r) :248-266  own: out[64]
    S.gate_array(out[0], ch[0], W(RW_RC));
}

// The constraint system of one KeccakfRound(r) block (keccak.circom:290-297 and everything below it), over signal indices
// RELATIVE to the block's first signal.  Same traversal order as emit_round; REL_ONE stands for the constant 1.
static const uint64_t REL_ONE = 0xffffffffull;
struct RelComp { uint32_t off, n; const char *tmpl; };
struct RoundCons {
    ConsSink &S; uint32_t cur = 0;
    std::vector<RelComp> *comps = nullptr;
    void comp(uint32_t off, uint32_t n, const char *t) { if (comps) comps->push_back(RelComp{off, n, t}); }
    uint32_t take(uint32_t n) { uint32_t o = cur; cur += n; return o; }
    void eqn(uint32_t a, uint32_t b, uint32_t n) { for (uint32_t k = 0; k < n; k++) S.eq(a + k, b + k); }
    void eq64(uint32_t a, uint32_t b) { eqn(a, b, 64); }
    // XorArray :77-86 / OrArray :104-113 / AndArray :120-129 (64): own out, a, b, then 64 gates [out, a, b]
    uint32_t gate_array(int kind, uint32_t srcA, uint32_t srcB) {
        const uint32_t o = take(64), a = take(64), b = take(64);
        comp(o, 192, kind == 0 ? "XorArray" : kind == 1 ? "OrArray" : "AndArray");
        eq64(a, srcA); eq64(b, srcB);
        for (uint32_t k = 0; k < 64; k++) {
            const uint32_t g = take(3);
            comp(g, 3, kind == 0 ? "XOR" : kind == 1 ? "OR" : "AND");
            S.eq(g + 1, a + k); S.eq(g + 2, b + k);
            if (kind == 0) S.r1(LC().s(g + 1, 2), LC().s(g + 2), LC().s(g + 1).s(g + 2).s(g, -1));       // XOR: out <== a + b - 2*a*b   gates.circom:26
            else if (kind == 1) S.r1(LC().s(g + 1), LC().s(g + 2), LC().s(g + 1).s(g + 2).s(g, -1));     // OR : out <== a + b - a*b     gates.circom:42
            else S.r1(LC().s(g + 1), LC().s(g + 2), LC().s(g));                                           // AND: out <== a*b             gates.circom:34
            S.eq(o + k, g);
        }
        return o;
    }
    uint32_t shl(uint32_t src, uint32_t r) {         // ShL(64, r) :40-51  own: out, in
        const uint32_t o = take(64), in = take(64); eq64(in, src); comp(o, 128, "ShL");
        for (uint32_t i = 0; i < 64; i++) { if (i < r) S.kc(o + i, fr_zero()); else S.eq(o + i, in + i - r); }
        return o;
    }
    uint32_t shr(uint32_t src, uint32_t r) {         // ShR(64, r) :19-30
        const uint32_t o = take(64), in = take(64); eq64(in, src); comp(o, 128, "ShR");
        for (uint32_t i = 0; i < 64; i++) { if (i + r >= 64) S.kc(o + i, fr_zero()); else S.eq(o + i, in + i + r); }
        return o;
    }
    uint32_t notarr(uint32_t src) {                  // NotArray(64) :92-98  own: out, a ; out[i] <== 1 - a[i]
        const uint32_t o = take(64), a = take(64); eq64(a, src); comp(o, 128, "NotArray");
        for (uint32_t i = 0; i < 64; i++) S.r1(LC(), LC(), LC().s(o + i).s(a + i).s(REL_ONE, -1));
        return o;
    }
    void round() {
        const uint32_t r_out = take(1600), r_in = take(1600), r_theta = take(1600), r_rhopi = take(1600), r_chi = take(1600);
        comp(r_out, 8000, "KeccakfRound");
        {   // signal theta[25][64] <== Theta()(in)   :293 ; Theta :151-170  own: out, in, c[5], d[5]
            const uint32_t t_out = take(1600), t_in = take(1600), t_c = take(320), t_d = take(320);
            comp(t_out, 3840, "Theta");
            eqn(t_in, r_in, 1600);
            for (uint32_t i = 0; i < 5; i++) {          // c[i] <== Xor5(64)(in[i], in[5+i], in[10+i], in[15+i], in[20+i])   :157 ; Xor5 :58-70
                const uint32_t x_out = take(64); uint32_t x_in[5]; for (int j = 0; j < 5; j++) x_in[j] = take(64);
                const uint32_t x_ab = take(64), x_abc = take(64), x_abcd = take(64);
                comp(x_out, 576, "Xor5");
                for (uint32_t j = 0; j < 5; j++) eq64(x_in[j], t_in + 64 * (5 * j + i));
                eq64(x_ab, gate_array(0, x_in[0], x_in[1])); eq64(x_abc, gate_array(0, x_ab, x_in[2]));
                eq64(x_abcd, gate_array(0, x_abc, x_in[3])); eq64(x_out, gate_array(0, x_abcd, x_in[4]));
                eq64(t_c + 64 * i, x_out);
            }
            for (uint32_t i = 0; i < 5; i++) {          // d[i] <== D()(c[(i+1)%5], c[(i+4)%5])   :162 ; D :135-144  own: out, a, b, aux0, aux1, aux2
                const uint32_t d_out = take(64), d_a = take(64), d_b = take(64), d_0 = take(64), d_1 = take(64), d_2 = take(64);
                comp(d_out, 384, "D");
                eq64(d_a, t_c + 64 * ((i + 1) % 5)); eq64(d_b, t_c + 64 * ((i + 4) % 5));
                eq64(d_0, shl(d_a, 1)); eq64(d_1, shr(d_a, 63));
                eq64(d_2, gate_array(1, d_0, d_1)); eq64(d_out, gate_array(0, d_b, d_2));
                eq64(t_d + 64 * i, d_out);
            }
            for (uint32_t i = 0; i < 5; i++) for (uint32_t j = 0; j < 5; j++)                 // out[i + j*5] <== XorArray(64)(in[i + j*5], d[i])   :167
                eq64(t_out + 64 * (i + 5 * j), gate_array(0, t_in + 64 * (i + 5 * j), t_d + 64 * i));
            eqn(r_theta, t_out, 1600);
        }
        {   // signal rhopi <== RhoPi()(theta)   :294 ; RhoPi :191-204  own: out, in
            const uint32_t p_out = take(1600), p_in = take(1600);
            comp(p_out, 3200, "RhoPi");
            eqn(p_in, r_theta, 1600);
            eq64(p_out, p_in);                                                        // out[0] <== in[0]   :197
            for (int i = 0; i < 24; i++) {              // out[rot[i+1]] <== stepRhoPi(shl, 64 - shl)(in[rot[i]])   :202 ; stepRhoPi :177-184  own: out, a, aux0, aux1
                const uint32_t sh = (uint32_t)keccak_shl(i);
                const uint32_t s_out = take(64), s_a = take(64), s_0 = take(64), s_1 = take(64);
                comp(s_out, 256, "stepRhoPi");
                eq64(s_a, p_in + 64 * (uint32_t)keccak_rot(i));
                eq64(s_0, shr(s_a, 64 - sh)); eq64(s_1, shl(s_a, sh));
                eq64(s_out, gate_array(1, s_0, s_1));
                eq64(p_out + 64 * (uint32_t)keccak_rot(i + 1), s_out);
            }
            eqn(r_rhopi, p_out, 1600);
        }
        {   // signal chi <== Chi()(rhopi)   :295 ; Chi :228-241  own: out, in
            const uint32_t c_out = take(1600), c_in = take(1600);
            comp(c_out, 3200, "Chi");
            eqn(c_in, r_rhopi, 1600);
            for (int i = 0; i < 25; i++) {              // out[i] <== stepChi()(in[i], in[..], in[..])   :233-239 ; stepChi :212-221  own: out, a, b, c, bXor, bc
                const uint32_t s_out = take(64), s_a = take(64), s_b = take(64), s_c = take(64), s_bx = take(64), s_bc = take(64);
                comp(s_out, 384, "stepChi");
                eq64(s_a, c_in + 64 * (uint32_t)i); eq64(s_b, c_in + 64 * (uint32_t)chi_b(i)); eq64(s_c, c_in + 64 * (uint32_t)chi_c(i));
                eq64(s_bx, notarr(s_b)); eq64(s_bc, gate_array(2, s_bx, s_c)); eq64(s_out, gate_array(0, s_a, s_bc));
                eq64(c_out + 64 * (uint32_t)i, s_out);
            }
            eqn(r_chi, c_out, 1600);
        }
        {   // out <== Iota(r)(chi)   :296 ; Iota :273-283  own: out, in, roundConstants ; RoundConstants(r) :248-266  own: out[64]
            const uint32_t i_out = take(1600), i_in = take(1600), i_rc = take(64);
            comp(i_out, 3264, "Iota");
            eqn(i_in, r_chi, 1600);
            const uint32_t rc = take(64);
            comp(rc, 64, "RoundConstants");
            for (uint32_t k = 0; k < 64; k++) S.kc_raw(rc + k, (CC_RCBIT << 30) | k);   // out[i] <== (rc[r] >> i) & 1   :264
            eq64(i_rc, rc);
            eq64(i_out, gate_array(0, i_in, i_rc));                                   // out[0] <== XorArray(64)(in[0], roundConstants)   :279
            eqn(i_out + 64, i_in + 64, 1536);                                         // out[i] <== in[i], i >= 1                          :281
            eqn(r_out, i_out, 1600);
        }
    }
};

// Absorb :304-323  (s: previous state words or NONE_IDX; blk: 17 block words).  Returns the state-out word base.
static uint32_t T_Absorb(Builder &B, uint32_t s_idx, uint32_t blk_idx, Blk *own) {
    uint32_t A = B.absorb(s_idx, blk_idx), out_w = A + RW * 24;
    Blk o = B.alloc(1600 + 1600 + 1088 + 1600, "Absorb"); if (own) *own = o;
    LaneSink S{&B.at(o.pos), 0};
    for (uint32_t l = 0; l < 25; l++) S.lane(Lane{out_w + l});
    for (uint32_t l = 0; l < 25; l++) S.lane(Lane{s_idx == NONE_IDX ? NONE_IDX : s_idx + l});
    for (uint32_t l = 0; l < 17; l++) S.lane(Lane{blk_idx + l});
    for (uint32_t l = 0; l < 25; l++) S.lane(Lane{A + l});
    const uint64_t qS = o.sig + 1600, qBlk = o.sig + 3200, qAux = o.sig + 4288;
    for (uint32_t l = 0; l < 17; l++) {                               // XorArray(64)(s[i], block[i])
        if (B.comps) { B.comps->push_back(Builder::Comp{B.nsig, 192, "XorArray"}); for (uint32_t k = 0; k < 64; k++) B.comps->push_back(Builder::Comp{B.nsig + 192 + 3 * k, 3, "XOR"}); }
        Blk x = B.alloc(384); LaneSink X{&B.at(x.pos), 0};
        X.gate_array(Lane{A + l}, Lane{s_idx == NONE_IDX ? NONE_IDX : s_idx + l}, Lane{blk_idx + l});
        if (B.want_cs()) {                                            // aux[i] <== XorArray(64)(s[i], block[i])   keccak.circom:316
            B.q_eqn(x.sig + 64, qS + 64 * l, 64); B.q_eqn(x.sig + 128, qBlk + 64 * l, 64); B.q_eqn(qAux + 64 * l, x.sig, 64);
            for (uint32_t k = 0; k < 64; k++) {
                const uint64_t g = x.sig + 192 + 3 * k;
                B.q_eq(g + 1, x.sig + 64 + k); B.q_eq(g + 2, x.sig + 128 + k);
                B.q_r1(LC().s(g + 1, 2), LC().s(g + 2), LC().s(g + 1).s(g + 2).s(g, -1));     // XOR   gates.circom:26
                B.q_eq(x.sig + k, g);
            }
        }
    }
    B.q_eqn(qAux + 64 * 17, qS + 64 * 17, 64 * 8);                    // aux[i] <== s[i], i >= 17                    :318
    // Keccakf :356-367  own: out, in, midRound[25][25][64]
    Blk k = B.alloc(1600 + 1600 + 25 * 1600, "Keccakf"); LaneSink Kf{&B.at(k.pos), 0};
    for (uint32_t l = 0; l < 25; l++) Kf.lane(Lane{out_w + l});
    for (uint32_t l = 0; l < 25; l++) Kf.lane(Lane{A + l});
    for (uint32_t r = 0; r <= 24; r++) for (uint32_t l = 0; l < 25; l++) Kf.lane(Lane{A + RW * r + l});
    B.q_eqn(k.sig + 1600, qAux, 1600); B.q_eqn(o.sig, k.sig, 1600);   // out <== Keccakf()(aux)                      :322
    B.q_eqn(k.sig + 3200, k.sig + 1600, 1600);                        // midRound[0] <== in                          :361
    for (uint32_t r = 0; r < 24; r++) {
        const uint64_t rb = B.nsig;
        B.round_block(A + RW * r);
        B.q_eqn(rb + 1600, k.sig + 3200 + 1600 * (uint64_t)r, 1600);  // midRound[i+1] <== KeccakfRound(i)(midRound[i])   :363
        B.q_eqn(k.sig + 3200 + 1600 * (uint64_t)(r + 1), rb, 1600);
    }
    B.q_eqn(k.sig, k.sig + 3200 + 1600 * 24, 1600);                   // out <== midRound[24]                        :366
    return out_w;
}
// Final(n) :330-349 and Keccak(n) :374-385 ; in_words: n*17 block words ; returns Keccak's own block
static Blk T_Keccak(Builder &B, int n_, uint32_t in_words, Code blocks) {
    size_t n = (size_t)n_;
    Blk ko = B.alloc(256 + n * 1088 + 1 + 1600, "Keccak");                      // Keccak own: out[256], in, blocks, finalState
    { LaneSink S{&B.at(ko.pos + 256), 0}; for (uint32_t w = 0; w < n * 17; w++) S.lane(Lane{in_words + w}); }
    B.at(ko.pos + 256 + n * 1088) = blocks;
    Blk fo = B.alloc(1600 + n * 1088 + 1 + (n + 1) * 1600, "Final");           // Final own: out, in, blocks, s[n+1]
    { LaneSink S{&B.at(fo.pos + 1600), 0}; for (uint32_t w = 0; w < n * 17; w++) S.lane(Lane{in_words + w}); }
    B.at(fo.pos + 1600 + n * 1088) = blocks;
    size_t s = fo.pos + 1600 + n * 1088 + 1;
    const uint64_t qS = fo.sig + 1600 + n * 1088 + 1, qFin = ko.sig + 256 + n * 1088 + 1;
    for (size_t i = 0; i < 1600; i++) { B.at(s + i) = ZERO; B.q_const(qS + i, 0); }   // s[0][i][j] <== 0            keccak.circom:339
    uint32_t st = NONE_IDX;
    for (size_t b = 0; b < n; b++) {
        Blk ab;
        st = T_Absorb(B, st, in_words + 17 * (uint32_t)b, &ab);
        LaneSink S{&B.at(s + 1600 * (b + 1)), 0}; for (uint32_t l = 0; l < 25; l++) S.lane(Lane{st + l});
        B.q_eqn(ab.sig + 1600, qS + 1600 * b, 1600); B.q_eqn(ab.sig + 3200, fo.sig + 1600 + 1088 * b, 1088);   // s[b+1] <== Absorb()(s[b], in[b])   :344
        B.q_eqn(qS + 1600 * (b + 1), ab.sig, 1600);
    }
    Blk sel = T_SelectorArray(B, n_ + 1, 1600, &B.at(s), blocks);
    B.copy(fo.pos, &B.at(sel.pos), 1600);
    B.copy(ko.pos + 256 + n * 1088 + 1, &B.at(fo.pos), 1600);
    B.copy(ko.pos, &B.at(fo.pos), 256);
    if (B.want_cs()) {
        B.q_eqn(sel.sig + 1600, qS, (n + 1) * 1600); B.q_eq(sel.sig + 1600 + (n + 1) * 1600, fo.sig + 1600 + n * 1088);   // out <== SelectorArray2D(nBlocksIn+1, 25, 64)(s, blocks)   :348
        B.q_eqn(fo.sig, sel.sig, 1600);
        B.q_eqn(fo.sig + 1600, ko.sig + 256, n * 1088); B.q_eq(fo.sig + 1600 + n * 1088, ko.sig + 256 + n * 1088);        // finalState <== Final(nBlocksIn)(in, blocks)               :379
        B.q_eqn(qFin, fo.sig, 1600);
        B.q_eqn(ko.sig, qFin, 256);                                                                                        // out[i] <== finalState[i \ 64][i % 64]                    :383
    }
    return ko;
}
// Pad(maxBlocks, blockSize) :412-446  own: out[B], numBlocks, in[B], inLen, div, rem, filter[B+1], isEq[B], isLast[B]
static Blk T_Pad(Builder &B, int maxBlocks, int blockSize, const Code *in, Code inLen) {
    size_t Bn = (size_t)maxBlocks * (size_t)blockSize; Blk o = B.alloc(Bn + 1 + Bn + 1 + 2 + (Bn + 1) + Bn + Bn, "Pad");
    size_t numBlocks = o.pos + Bn, iIn = numBlocks + 1, iLen = iIn + Bn, div = iLen + 1, rem = div + 1,
           filter = rem + 1, isEq = filter + Bn + 1, isLast = isEq + Bn;
    const uint64_t d = o.sig - o.pos; const bool cs = B.want_cs();
    B.copy(iIn, in, Bn); B.at(iLen) = inLen;
    Blk dv = T_Divide(B, 16, inLen, c_const((uint32_t)blockSize)); B.at(div) = B.at(dv.pos); B.at(rem) = B.at(dv.pos + 1);
    Code nbk = B.add(B.at(div), ONE); B.at(numBlocks) = nbk;
    Blk al = T_AssertLessEqThan(B, 16, nbk, c_const((uint32_t)maxBlocks));
    B.at(filter) = ONE;
    if (cs) {
        B.q_eq(dv.sig + 2, d + iLen); B.q_const(dv.sig + 3, (uint64_t)blockSize); B.q_eq(d + div, dv.sig); B.q_eq(d + rem, dv.sig + 1);   // signal (div, rem) <== Divide(16)(inLen, blockSize)   keccak.circom:420
        B.q_lin(LC().s(d + numBlocks, -1).s(d + div).k(1));                                                                              // numBlocks <== div + 1                                :421
        B.q_eq(al.sig, d + numBlocks); B.q_const(al.sig + 1, (uint64_t)maxBlocks);                                                       // AssertLessEqThan(16)(numBlocks, maxBlocks)           :423
        B.q_const(d + filter, 1);                                                                                                        // filter[0] <== 1                                      :428
    }
    for (size_t i = 0; i < Bn; i++) {
        Blk e = T_IsEqual(B, c_const((uint32_t)i), inLen); Code eq = B.at(e.pos); B.at(isEq + i) = eq;
        B.at(filter + i + 1) = B.gtc(inLen, (uint32_t)i);          // filter[i]*(1 - isEq[i]) == (inLen > i)
        if (cs) {
            B.q_const(e.sig + 1, i); B.q_eq(e.sig + 2, d + iLen); B.q_eq(d + isEq + i, e.sig);                         // isEq[i] <== IsEqual()([i, inLen])               :431
            B.q_r1(LC().s(d + filter + i), LC().k(1).s(d + isEq + i, -1), LC().s(d + filter + i + 1));                // filter[i+1] <== filter[i] * (1 - isEq[i])       :432
        }
    }
    Code lastPos = B.sub(B.mul(nbk, c_const((uint32_t)blockSize)), ONE);
    for (size_t i = 0; i < Bn; i++) {
        Blk e = T_IsEqual(B, c_const((uint32_t)i), lastPos); Code l = B.at(e.pos); B.at(isLast + i) = l;
        B.at(o.pos + i) = B.fma(l, c_const(0x80), B.fma(in[i], B.at(filter + i + 1), B.at(isEq + i)));
        if (cs) {
            B.q_const(e.sig + 1, i); B.q_lin(LC().s(e.sig + 2).s(d + numBlocks, -(int64_t)blockSize).k(1)); B.q_eq(d + isLast + i, e.sig);   // isLast[i] <== IsEqual()([i, numBlocks*blockSize - 1])   :437
            B.q_r1(LC().s(d + iIn + i), LC().s(d + filter + i + 1), LC().s(o.sig + i).s(d + isEq + i, -1).s(d + isLast + i, -0x80));        // out[i] <== in[i]*filter[i+1] + 0x01*isEq[i] + 0x80*isLast[i]   :444
        }
    }
    return o;
}
// KeccakBytes(maxBlocks) :454-489
static Blk T_KeccakBytes(Builder &B, int maxBlocks, const Code *in, Code inLen) {
    size_t Bn = (size_t)maxBlocks * 136;
    Blk o = B.alloc(32 + Bn + 1 + Bn + 1 + 24 * Bn + 256 + 256, "KeccakBytes");
    size_t iIn = o.pos + 32, iLen = iIn + Bn, padded = iLen + 1, numBlocks = padded + Bn, inBitsArray = numBlocks + 1,
           inBits = inBitsArray + 8 * Bn, inBlocks = inBits + 8 * Bn, outBits = inBlocks + 8 * Bn, outBytes = outBits + 256;
    const uint64_t d = o.sig - o.pos; const bool cs = B.want_cs();
    B.copy(iIn, in, Bn); B.at(iLen) = inLen;
    Blk al = T_AssertLessThan(B, 16, inLen, c_const((uint32_t)Bn));
    Blk p = T_Pad(B, maxBlocks, 136, in, inLen); B.copy(padded, &B.at(p.pos), Bn); B.at(numBlocks) = B.at(p.pos + Bn);
    if (cs) {
        B.q_eq(al.sig, d + iLen); B.q_const(al.sig + 1, Bn);                                                         // AssertLessThan(16)(inLen, maxBlocks*136)          keccak.circom:460
        B.q_eqn(p.sig + Bn + 1, d + iIn, Bn); B.q_eq(p.sig + 2 * Bn + 1, d + iLen);                                  // (padded, numBlocks) <== Pad(maxBlocks, 136)(in, inLen)   :463-465
        B.q_eqn(d + padded, p.sig, Bn); B.q_eq(d + numBlocks, p.sig + Bn);
    }
    uint32_t words = B.pack8_words(&B.at(padded), (uint32_t)(Bn / 8));         // bytes -> 17 lanes per block
    for (size_t i = 0; i < Bn; i++) {                                          // Num2Bits(8)(padded[i])
        Blk nb = B.alloc(9, "Num2Bits");
        for (uint32_t k = 0; k < 8; k++) B.at(nb.pos + k) = c_bit(words + (uint32_t)(i / 8), 8 * (uint32_t)(i % 8) + k);
        B.at(nb.pos + 8) = B.at(padded + i);
        B.chk_range(B.at(padded + i), 8, nb.sig);
        B.copy(inBitsArray + 8 * i, &B.at(nb.pos), 8);
        if (cs) {
            LC sum;
            for (uint32_t k = 0; k < 8; k++) { B.q_r1(LC().s(nb.sig + k), LC().s(nb.sig + k).k(-1), LC()); sum.s(nb.sig + k, 1 << k); }   // Num2Bits(8)   bitify.circom:33, :38
            sum.s(nb.sig + 8, -1); B.q_lin(sum);
            B.q_eq(nb.sig + 8, d + padded + i); B.q_eqn(d + inBitsArray + 8 * i, nb.sig, 8);                         // inBitsArray[i] <== Num2Bits(8)(padded[i])         :470
        }
    }
    Blk fl = T_CopyArray(B, 8 * Bn, &B.at(inBitsArray)); B.copy(inBits, &B.at(fl.pos), 8 * Bn);   // Flatten
    B.copy(inBlocks, &B.at(inBits), 8 * Bn);
    Blk k = T_Keccak(B, maxBlocks, words, B.at(numBlocks)); B.copy(outBits, &B.at(k.pos), 256);
    Blk rs = T_CopyArray(B, 256, &B.at(outBits)); B.copy(outBytes, &B.at(rs.pos), 256);           // Reshape
    if (cs) {
        B.q_eqn(fl.sig + 8 * Bn, d + inBitsArray, 8 * Bn); B.q_eqn(d + inBits, fl.sig, 8 * Bn);                      // inBits <== Flatten(maxBlocks*136, 8)(inBitsArray)   :472
        B.q_eqn(d + inBlocks, d + inBits, 8 * Bn);                                                                   // inBlocks[i][j][k] <== inBits[i*17*64 + j*64 + k]    :479
        B.q_eqn(k.sig + 256, d + inBlocks, 8 * Bn); B.q_eq(k.sig + 256 + 8 * Bn, d + numBlocks); B.q_eqn(d + outBits, k.sig, 256);   // outBits <== Keccak(maxBlocks)(inBlocks, numBlocks)   :484
        B.q_eqn(rs.sig + 256, d + outBits, 256); B.q_eqn(d + outBytes, rs.sig, 256);                                 // outBytes <== Reshape(32, 8)(outBits)                :485
    }
    for (size_t i = 0; i < 32; i++) {
        Blk bn = T_Bits2Num(B, 8, &B.at(outBytes + 8 * i)); B.at(o.pos + i) = B.at(bn.pos);
        B.q_eqn(bn.sig + 1, d + outBytes + 8 * i, 8); B.q_eq(o.sig + i, bn.sig);                                     // out[i] <== Bits2Num(8)(outBytes[i])                 :487
    }
    return o;
}

// ============================================================================================================
// circuits/utils/public_commitment.circom, constants.circom, burn_address.circom, proof_of_work.circom
// ============================================================================================================
// PublicCommitment(N) :18-42  own: out, in[N][32], flattenIn, block, hash[32], reducedHash[31]
static Blk T_PublicCommitment(Builder &B, int N, const Code *in) {
    size_t n32 = (size_t)N * 32; int nb = (N * 32) / 136 + ((N * 32) % 136 != 0); size_t blk = (size_t)nb * 136;
    Blk o = B.alloc(1 + n32 + n32 + blk + 32 + 31, "PublicCommitment");
    size_t iIn = o.pos + 1, flat = iIn + n32, block = flat + n32, hash = block + blk, red = hash + 32;
    const uint64_t d = o.sig - o.pos;
    B.copy(iIn, in, n32);
    for (int i = 0; i < N; i++) { Blk a = T_AssertByteString(B, 32, in + 32 * i); B.q_eqn(a.sig, d + iIn + 32 * (size_t)i, 32); }   // AssertByteString(32)(in[i])   public_commitment.circom:24
    Blk f = T_CopyArray(B, n32, in); B.copy(flat, &B.at(f.pos), n32);
    Blk ft = T_Fit(B, (int)n32, (int)blk, &B.at(flat)); B.copy(block, &B.at(ft.pos), blk);
    Blk k = T_KeccakBytes(B, nb, &B.at(block), c_const((uint32_t)n32)); B.copy(hash, &B.at(k.pos), 32);
    Blk f2 = T_Fit(B, 32, 31, &B.at(hash)); B.copy(red, &B.at(f2.pos), 31);
    Blk be = T_BigEndianBytes2Num(B, 31, &B.at(red)); B.at(o.pos) = B.at(be.pos);
    if (B.want_cs()) {
        B.q_eqn(f.sig + n32, d + iIn, n32); B.q_eqn(d + flat, f.sig, n32);                                   // flattenIn <== Flatten(N, 32)(in)                   :33
        B.q_eqn(ft.sig + blk, d + flat, n32); B.q_eqn(d + block, ft.sig, blk);                               // block <== Fit(N*32, numBlocks*136)(flattenIn)      :34
        B.q_eqn(k.sig + 32, d + block, blk); B.q_const(k.sig + 32 + blk, n32); B.q_eqn(d + hash, k.sig, 32); // hash <== KeccakBytes(numBlocks)(block, N*32)        :36
        B.q_eqn(f2.sig + 31, d + hash, 32); B.q_eqn(d + red, f2.sig, 31);                                    // reducedHash <== Fit(32, 31)(hash)                  :39
        B.q_eqn(be.sig + 1, d + red, 31); B.q_eq(o.sig, be.sig);                                             // out <== BigEndianBytes2Num(31)(reducedHash)        :41
    }
    return o;
}
// constants.circom :3-15
static Code POSEIDON_PREFIX(Builder &B, int add) {
    // keccak("EIP-7503") mod p = 5265656504298861414514317065875120428884240036965045859626767452974705356670
    Fr r; const uint32_t l[8] = {0x3d892f7eu, 0xf0363f98u, 0x980a6b46u, 0xd115b780u, 0xcd46cec2u, 0x007d2482u, 0xee7876b8u, 0x0ba44186u};
    memcpy(r.l, l, 32);
    return B.konst(fr_add(r, fr_from_u64((uint64_t)add)));
}
// BurnAddress :47-58  own: addressBytes[20], burnKey, revealAmount, burnExtraCommitment, hash, hashBytes[32]
static Blk T_BurnAddress(Builder &B, Code burnKey, Code revealAmount, Code bec) {
    Blk o = B.alloc(20 + 3 + 1 + 32, "BurnAddress");
    B.at(o.pos + 20) = burnKey; B.at(o.pos + 21) = revealAmount; B.at(o.pos + 22) = bec;
    Code ins[4] = {POSEIDON_PREFIX(B, 0), burnKey, revealAmount, bec};
    Blk p = T_Poseidon(B, 4, ins); B.at(o.pos + 23) = B.at(p.pos);
    Blk b = T_Num2BigEndianBytes(B, 32, B.at(p.pos)); B.copy(o.pos + 24, &B.at(b.pos), 32);
    Blk f = T_Fit(B, 32, 20, &B.at(o.pos + 24)); B.copy(o.pos, &B.at(f.pos), 20);
    if (B.want_cs()) {
        Fr pre; B.const_val(ins[0], pre);
        B.q_constf(p.sig + 1, pre); B.q_eqn(p.sig + 2, o.sig + 20, 3); B.q_eq(o.sig + 23, p.sig);            // hash <== Poseidon(4)([PREFIX, burnKey, revealAmount, burnExtraCommitment])   burn_address.circom:55
        B.q_eq(b.sig + 32, o.sig + 23); B.q_eqn(o.sig + 24, b.sig, 32);                                      // hashBytes <== Num2BigEndianBytes(32)(hash)                                   :56
        B.q_eqn(f.sig + 20, o.sig + 24, 32); B.q_eqn(o.sig, f.sig, 20);                                      // addressBytes <== Fit(32, 20)(hashBytes)                                      :57
    }
    return o;
}
// BurnAddressHash :67-83  own: addressHashNibbles[64], 3 inputs, addressBytes[20], addressBytesBlock[136], addressHash[32]
static Blk T_BurnAddressHash(Builder &B, Code burnKey, Code revealAmount, Code bec) {
    Blk o = B.alloc(64 + 3 + 20 + 136 + 32, "BurnAddressHash");
    B.at(o.pos + 64) = burnKey; B.at(o.pos + 65) = revealAmount; B.at(o.pos + 66) = bec;
    Blk a = T_BurnAddress(B, burnKey, revealAmount, bec); B.copy(o.pos + 67, &B.at(a.pos), 20);
    Blk f = T_Fit(B, 20, 136, &B.at(o.pos + 67)); B.copy(o.pos + 87, &B.at(f.pos), 136);
    Blk k = T_KeccakBytes(B, 1, &B.at(o.pos + 87), c_const(20)); B.copy(o.pos + 223, &B.at(k.pos), 32);
    Blk nb = T_Bytes2Nibbles(B, 32, &B.at(o.pos + 223)); B.copy(o.pos, &B.at(nb.pos), 64);
    if (B.want_cs()) {
        B.q_eqn(a.sig + 20, o.sig + 64, 3); B.q_eqn(o.sig + 67, a.sig, 20);                                  // addressBytes <== BurnAddress()(...)                         burn_address.circom:77
        B.q_eqn(f.sig + 136, o.sig + 67, 20); B.q_eqn(o.sig + 87, f.sig, 136);                               // addressBytesBlock <== Fit(20, 136)(addressBytes)            :78
        B.q_eqn(k.sig + 32, o.sig + 87, 136); B.q_const(k.sig + 32 + 136, 20); B.q_eqn(o.sig + 223, k.sig, 32);   // addressHash <== KeccakBytes(1)(addressBytesBlock, 20)  :79
        B.q_eqn(nb.sig + 64, o.sig + 223, 32); B.q_eqn(o.sig, nb.sig, 64);                                   // addressHashNibbles <== Bytes2Nibbles(32)(addressHash)       :82
    }
    return o;
}
// EIP7503 :11-21
static Blk T_EIP7503(Builder &B) {
    static const uint8_t s[8] = {69, 73, 80, 45, 55, 53, 48, 51};
    Blk o = B.alloc(8, "EIP7503");
    for (int i = 0; i < 8; i++) { B.at(o.pos + (size_t)i) = c_const(s[i]); B.q_const(o.sig + (uint64_t)i, s[i]); }   // out[i] <== 'EIP-7503'[i]   proof_of_work.circom:13-20
    return o;
}
// ConcatFixed4(A,B,C,D) :28-48  own: out[A+B+C+D], a, b, c, d
static Blk T_ConcatFixed4(Builder &B, int A, int Bn, int C, int D, const Code *a, const Code *b, const Code *c, const Code *d) {
    size_t T = (size_t)(A + Bn + C + D); Blk o = B.alloc(2 * T, "ConcatFixed4");
    B.copy(o.pos, a, (size_t)A); B.copy(o.pos + (size_t)A, b, (size_t)Bn); B.copy(o.pos + (size_t)(A + Bn), c, (size_t)C);
    B.copy(o.pos + (size_t)(A + Bn + C), d, (size_t)D);
    B.copy(o.pos + T, &B.at(o.pos), T);
    B.q_eqn(o.sig, o.sig + T, T);                                                 // out[i] <== a[i]; out[i+A] <== b[i]; ...   proof_of_work.circom:36-47
    return o;
}
// ProofOfWorkChecker :54-81
static Blk T_ProofOfWorkChecker(Builder &B, Code burnKey, Code revealAmount, Code bec, Code minimumZeroBytes) {
    Blk o = B.alloc(4 + 96 + 8 + 104 + 136 + 32 + 32, "ProofOfWorkChecker");
    size_t bk = o.pos + 4, ra = bk + 32, be = ra + 32, eip = be + 32, hin = eip + 8, blk = hin + 104, kec = blk + 136, sbz = kec + 32;
    const uint64_t d = o.sig - o.pos; const bool cs = B.want_cs();
    B.at(o.pos) = burnKey; B.at(o.pos + 1) = revealAmount; B.at(o.pos + 2) = bec; B.at(o.pos + 3) = minimumZeroBytes;
    Blk x = T_Num2BigEndianBytes(B, 32, burnKey); B.copy(bk, &B.at(x.pos), 32);
    if (cs) { B.q_eq(x.sig + 32, o.sig); B.q_eqn(d + bk, x.sig, 32); }                                        // burnKeyBytes <== Num2BigEndianBytes(32)(burnKey)   proof_of_work.circom:61
    x = T_Num2BigEndianBytes(B, 32, revealAmount); B.copy(ra, &B.at(x.pos), 32);
    if (cs) { B.q_eq(x.sig + 32, o.sig + 1); B.q_eqn(d + ra, x.sig, 32); }                                    // :62
    x = T_Num2BigEndianBytes(B, 32, bec); B.copy(be, &B.at(x.pos), 32);
    if (cs) { B.q_eq(x.sig + 32, o.sig + 2); B.q_eqn(d + be, x.sig, 32); }                                    // :63
    x = T_EIP7503(B); B.copy(eip, &B.at(x.pos), 8);
    B.q_eqn(d + eip, x.sig, 8);                                                                               // eip7503 <== EIP7503()()                            :64
    x = T_ConcatFixed4(B, 32, 32, 32, 8, &B.at(bk), &B.at(ra), &B.at(be), &B.at(eip)); B.copy(hin, &B.at(x.pos), 104);
    if (cs) { B.q_eqn(x.sig + 104, d + bk, 104); B.q_eqn(d + hin, x.sig, 104); }                              // hasherInput <== ConcatFixed4(32, 32, 32, 8)(...)   :68 (the four inputs are adjacent own signals)
    x = T_Fit(B, 104, 136, &B.at(hin)); B.copy(blk, &B.at(x.pos), 136);
    if (cs) { B.q_eqn(x.sig + 136, d + hin, 104); B.q_eqn(d + blk, x.sig, 136); }                             // burnKeyBlock <== Fit(hasherInputLen, 136)(hasherInput)   :73
    x = T_KeccakBytes(B, 1, &B.at(blk), c_const(104)); B.copy(kec, &B.at(x.pos), 32);
    if (cs) { B.q_eqn(x.sig + 32, d + blk, 136); B.q_const(x.sig + 32 + 136, 104); B.q_eqn(d + kec, x.sig, 32); }   // burnKeyKeccak <== KeccakBytes(1)(burnKeyBlock, hasherInputLen)   :74
    x = T_Filter(B, 32, minimumZeroBytes); B.copy(sbz, &B.at(x.pos), 32);
    if (cs) { B.q_eq(x.sig + 32, o.sig + 3); B.q_eqn(d + sbz, x.sig, 32); }                                   // shouldBeZero <== Filter(32)(minimumZeroBytes)      :77
    for (size_t i = 0; i < 32; i++) {
        B.chk_eq(B.mul(B.at(kec + i), B.at(sbz + i)), ZERO, o.sig);
        B.q_r1(LC().s(d + kec + i), LC().s(d + sbz + i), LC());                                               // burnKeyKeccak[i] * shouldBeZero[i] === 0           :79
    }
    return o;
}

// ============================================================================================================
// circuits/utils/rlp/*.circom
// ============================================================================================================
// CountBytes(N) integer.circom:16-49  own: len, bytes[N], isZero[N], stillZero[N]
static Blk T_CountBytes(Builder &B, int N, const Code *bytes) {
    size_t n = (size_t)N; Blk o = B.alloc(1 + 3 * n, "CountBytes"); B.copy(o.pos + 1, bytes, n);
    for (size_t i = 0; i < n; i++) {
        Blk z = T_IsZero(B, bytes[i]); B.at(o.pos + 1 + n + i) = B.at(z.pos);
        B.q_eq(z.sig + 1, o.sig + 1 + i); B.q_eq(o.sig + 1 + n + i, z.sig);       // isZero[i] <== IsZero()(bytes[i])              integer.circom:24
    }
    std::vector<Code> terms;
    LC sum;
    for (size_t i = 0; i < n; i++) {
        Code sz = i == 0 ? B.at(o.pos + 1 + n) : B.mul(B.at(o.pos + 1 + n + i), B.at(o.pos + 1 + 2 * n + i - 1));
        B.at(o.pos + 1 + 2 * n + i) = sz; terms.push_back(sz);
        if (B.want_cs()) {
            if (i == 0) B.q_eq(o.sig + 1 + 2 * n, o.sig + 1 + n);                 // stillZero[0] <== isZero[0]                    :32
            else B.q_mul(o.sig + 1 + n + i, o.sig + 1 + 2 * n + i - 1, o.sig + 1 + 2 * n + i);   // stillZero[i] <== isZero[i] * stillZero[i-1]   :34
            sum.s(o.sig + 1 + 2 * n + i);
        }
    }
    B.at(o.pos) = B.sub(c_const((uint32_t)n), B.sum_tree(terms));
    if (B.want_cs()) { sum.s(o.sig).k(-(int64_t)n); B.q_lin(sum); }               // len <== N - leadingZeros                      :47
    return o;
}
// RlpInteger(N) integer.circom:67-110
static Blk T_RlpInteger(Builder &B, int N, Code in) {
    size_t n = (size_t)N; Blk o = B.alloc(n + 1 + 1 + 1 + n + 1 + n + 3, "RlpInteger");
    size_t outLen = o.pos + n + 1, iIn = outLen + 1, bytes = iIn + 1, length = bytes + n, bigEndian = length + 1,
           isSingle = bigEndian + n, isZero = isSingle + 1, first = isZero + 1;
    const uint64_t d = o.sig - o.pos; const bool cs = B.want_cs();
    B.at(iIn) = in;
    Blk x = T_Num2BigEndianBytes(B, N, in); B.copy(bytes, &B.at(x.pos), n);
    if (cs) { B.q_eq(x.sig + n, d + iIn); B.q_eqn(d + bytes, x.sig, n); }                                     // bytes <== Num2BigEndianBytes(N)(in)               integer.circom:77
    x = T_CountBytes(B, N, &B.at(bytes)); Code len = B.at(x.pos); B.at(length) = len;
    if (cs) { B.q_eqn(x.sig + 1, d + bytes, n); B.q_eq(d + length, x.sig); }                                  // length <== CountBytes(N)(bytes)                   :80
    x = T_ShiftLeft(B, N, &B.at(bytes), B.sub(c_const((uint32_t)n), len)); B.copy(bigEndian, &B.at(x.pos), n);
    if (cs) { B.q_eqn(x.sig + n, d + bytes, n); B.q_lin(LC().s(x.sig + 2 * n).k(-(int64_t)n).s(d + length)); B.q_eqn(d + bigEndian, x.sig, n); }   // bigEndian <== ShiftLeft(N)(bytes, N - length)   :83
    x = T_LessThan(B, N * 8, in, c_const(128)); Code single = B.at(x.pos); B.at(isSingle) = single;
    if (cs) { B.q_eq(x.sig + 1, d + iIn); B.q_const(x.sig + 2, 128); B.q_eq(d + isSingle, x.sig); }           // isSingleByte <== LessThan(N*8)([in, 128])         :86
    x = T_IsZero(B, in, /*likely_large=*/true); Code iz = B.at(x.pos); B.at(isZero) = iz;      // in = a balance: not a table-sized value
    if (cs) { B.q_eq(x.sig + 1, d + iIn); B.q_eq(d + isZero, x.sig); }                                        // isZero <== IsZero()(in)                           :89
    x = T_Mux1(B, B.add(c_const(0x80), len), in, single); B.at(first) = B.at(x.pos);
    if (cs) { B.q_lin(LC().s(x.sig + 1).k(-0x80).s(d + length, -1)); B.q_eq(x.sig + 2, d + iIn); B.q_eq(x.sig + 3, d + isSingle); B.q_eq(d + first, x.sig); }   // firstRlpByte <== Mux1()([0x80 + length, in], isSingleByte)   :95
    B.at(o.pos) = B.fma(iz, c_const(0x80), B.at(first));
    Code ns = B.not1(single);
    for (size_t i = 1; i < n + 1; i++) B.at(o.pos + i) = B.mul(ns, B.at(bigEndian + i - 1));
    B.at(outLen) = B.add(B.add(ns, len), iz);
    if (cs) {
        B.q_lin(LC().s(o.sig, -1).s(d + first).s(d + isZero, 0x80));                                          // out[0] <== firstRlpByte + isZero * 0x80           :98
        for (size_t i = 1; i < n + 1; i++) B.q_r1(LC().k(1).s(d + isSingle, -1), LC().s(d + bigEndian + i - 1), LC().s(o.sig + i));   // out[i] <== (1 - isSingleByte) * bigEndian[i-1]   :103
        B.q_lin(LC().s(d + outLen, -1).k(1).s(d + isSingle, -1).s(d + length).s(d + isZero));                 // outLen <== (1 - isSingleByte) + length + isZero   :109
    }
    return o;
}
// RlpEmptyAccount(maxBalanceBytes) empty_account.circom:20-134
static const uint8_t STORAGE_CODE_RLP[66] = {
    160, 86, 232, 31, 23, 27, 204, 85, 166, 255, 131, 69, 230, 146, 192, 248, 110, 91, 72, 224, 27, 153, 108, 173, 192, 1, 98, 47, 181, 227, 99, 180, 33,
    160, 197, 210, 70, 1, 134, 247, 35, 60, 146, 126, 125, 178, 220, 199, 3, 192, 229, 0, 182, 83, 202, 130, 39, 59, 123, 250, 216, 4, 93, 133, 164, 112};
static Blk T_RlpEmptyAccount(Builder &B, int mbb, Code balance) {
    size_t m = (size_t)mbb, OL = 4 + m + 66; Blk o = B.alloc(OL + 1 + 1 + (4 + m) + 1 + (m + 1) + 1 + 1 + 66, "RlpEmptyAccount");
    size_t outLen = o.pos + OL, iBal = outLen + 1, pre = iBal + 1, preLen = pre + 4 + m, balRlp = preLen + 1,
           balRlpLen = balRlp + m + 1, nabLen = balRlpLen + 1, sc = nabLen + 1;
    const uint64_t d = o.sig - o.pos; const bool cs = B.want_cs();
    B.at(iBal) = balance;
    B.at(pre + 2) = c_const(0x80);
    Blk r = T_RlpInteger(B, mbb, balance); B.copy(balRlp, &B.at(r.pos), m + 1); B.at(balRlpLen) = B.at(r.pos + m + 1);
    for (size_t i = 0; i < m + 1; i++) B.at(pre + 3 + i) = B.at(balRlp + i);
    B.at(nabLen) = B.add(ONE, B.at(balRlpLen));
    B.at(preLen) = B.add(c_const(2), B.at(nabLen));
    for (size_t i = 0; i < 66; i++) B.at(sc + i) = c_const(STORAGE_CODE_RLP[i]);
    B.at(pre) = c_const(0xf8);
    B.at(pre + 1) = B.add(B.at(nabLen), c_const(66));
    Blk cc = T_Concat(B, 4 + mbb, 66, &B.at(pre), B.at(preLen), &B.at(sc), c_const(66));
    B.copy(o.pos, &B.at(cc.pos), OL); B.at(outLen) = B.at(cc.pos + OL);
    if (cs) {
        const size_t A = 4 + m;
        B.q_const(d + pre + 2, 0x80);                                                                         // prefixedNonceAndBalanceRlp[2] <== 0x80            empty_account.circom:32
        B.q_eq(r.sig + m + 2, d + iBal); B.q_eqn(d + balRlp, r.sig, m + 1); B.q_eq(d + balRlpLen, r.sig + m + 1);   // (balanceRlp, balanceRlpLen) <== RlpInteger(maxBalanceBytes)(balance)   :35
        B.q_eqn(d + pre + 3, d + balRlp, m + 1);                                                              // prefixedNonceAndBalanceRlp[i+3] <== balanceRlp[i] :37
        B.q_lin(LC().s(d + nabLen, -1).k(1).s(d + balRlpLen));                                                // nonceAndBalanceRlpLen <== 1 + balanceRlpLen       :41
        B.q_lin(LC().s(d + preLen, -1).k(2).s(d + nabLen));                                                   // prefixedNonceAndBalanceRlpLen <== 2 + ...         :42
        for (size_t i = 0; i < 66; i++) B.q_const(d + sc + i, STORAGE_CODE_RLP[i]);                           // storageAndCodeHashRlp[i] <== ...                  :48-115
        B.q_const(d + pre, 0xf8);                                                                             // prefixedNonceAndBalanceRlp[0] <== 0xf7 + 1        :117
        B.q_lin(LC().s(d + pre + 1, -1).s(d + nabLen).k(66));                                                 // prefixedNonceAndBalanceRlp[1] <== nonceAndBalanceRlpLen + 66   :118
        B.q_eqn(cc.sig + OL + 1, d + pre, A); B.q_eq(cc.sig + OL + 1 + A, d + preLen);                        // concat.a, concat.aLen                             :122-123
        B.q_eqn(cc.sig + OL + 1 + A + 1, d + sc, 66); B.q_const(cc.sig + OL + 1 + A + 1 + 66, 66);            // concat.b, concat.bLen                             :124-125
        B.q_eqn(o.sig, cc.sig, OL); B.q_eq(d + outLen, cc.sig + OL);                                          // out <== concat.out; outLen <== concat.outLen      :127-128
    }
    return o;
}
// TruncatedAddressHash(addressHashBytes) merkle_patricia_trie_leaf.circom:50-90 (`temp` :76 never assigned => 0)
static Blk T_TruncatedAddressHash(Builder &B, int ahb, const Code *nibbles, Code nibLen) {
    size_t a = (size_t)ahb; Blk o = B.alloc((a + 1) + 1 + 2 * a + 1 + 2 + 2 * a + (2 * a + 2) + (2 * a - 1), "TruncatedAddressHash");
    size_t outLen = o.pos + a + 1, iNib = outLen + 1, iLen = iNib + 2 * a, div = iLen + 1, rem = div + 1, shifted = rem + 1,
           outNib = shifted + 2 * a, temp = outNib + 2 * a + 2;
    const uint64_t d = o.sig - o.pos; const bool cs = B.want_cs();
    B.copy(iNib, nibbles, 2 * a); B.at(iLen) = nibLen;
    for (size_t i = 0; i < 2 * a - 1; i++) { B.at(temp + i) = ZERO; if (cs) B.q_hint(LC(), LC(), LC().s(d + temp + i)); }   // `signal temp[...]` is never assigned (:76): the calculator leaves 0
    Blk al = T_AssertLessEqThan(B, 7, nibLen, c_const((uint32_t)(2 * a)));
    Blk dv = T_Divide(B, 7, nibLen, c_const(2)); B.at(div) = B.at(dv.pos); Code rm = B.at(dv.pos + 1); B.at(rem) = rm;
    Blk s = T_ShiftLeft(B, 2 * ahb, nibbles, B.sub(c_const((uint32_t)(2 * a)), nibLen)); B.copy(shifted, &B.at(s.pos), 2 * a);
    B.at(outNib) = B.add(c_const(2), rm);
    B.at(outNib + 1) = B.mul(rm, B.at(shifted));
    if (cs) {
        B.q_eq(al.sig, d + iLen); B.q_const(al.sig + 1, 2 * a);                                               // AssertLessEqThan(7)(addressHashNibblesLen, 2*addressHashBytes)   merkle_patricia_trie_leaf.circom:59
        B.q_eq(dv.sig + 2, d + iLen); B.q_const(dv.sig + 3, 2); B.q_eq(d + div, dv.sig); B.q_eq(d + rem, dv.sig + 1);   // (div, rem) <== Divide(7)(addressHashNibblesLen, 2)    :62
        B.q_eqn(s.sig + 2 * a, d + iNib, 2 * a); B.q_lin(LC().s(s.sig + 4 * a).k(-(int64_t)(2 * a)).s(d + iLen)); B.q_eqn(d + shifted, s.sig, 2 * a);   // shifted <== ShiftLeft(2a)(nibbles, 2a - len)   :65-66
        B.q_lin(LC().s(d + outNib, -1).k(2).s(d + rem));                                                      // outNibbles[0] <== 2 + rem                          :73
        B.q_mul(d + rem, d + shifted, d + outNib + 1);                                                        // outNibbles[1] <== rem * shifted[0]                 :74
    }
    for (size_t i = 0; i < 2 * a; i++) {
        if (i < 2 * a - 1) {
            Blk m = T_Mux1(B, B.at(shifted + i), B.at(shifted + i + 1), rm); B.at(outNib + i + 2) = B.at(m.pos);
            if (cs) { B.q_eq(m.sig + 1, d + shifted + i); B.q_eq(m.sig + 2, d + shifted + i + 1); B.q_eq(m.sig + 3, d + rem); B.q_eq(d + outNib + i + 2, m.sig); }   // outNibbles[i+2] <== Mux1()([shifted[i], shifted[i+1]], rem)   :80
        } else {
            B.at(outNib + i + 2) = B.mul(B.not1(rm), B.at(shifted + i));
            B.q_r1(LC().k(1).s(d + rem, -1), LC().s(d + shifted + i), LC().s(d + outNib + i + 2));            // outNibbles[i+2] <== (1 - rem) * shifted[i]         :82
        }
    }
    Blk nb = T_Nibbles2Bytes(B, ahb + 1, &B.at(outNib)); B.copy(o.pos, &B.at(nb.pos), a + 1);
    B.at(outLen) = B.add(ONE, B.at(div));
    if (cs) {
        B.q_eqn(nb.sig + a + 1, d + outNib, 2 * a + 2); B.q_eqn(o.sig, nb.sig, a + 1);                        // out <== Nibbles2Bytes(addressHashBytes + 1)(outNibbles)   :87
        B.q_lin(LC().s(d + outLen, -1).k(1).s(d + div));                                                      // outLen <== 1 + div                                 :89
    }
    return o;
}
// RlpMerklePatriciaTrieLeaf(maxAddressHashBytes, maxBalanceBytes) :102-189
static Blk T_RlpMerklePatriciaTrieLeaf(Builder &B, int mahb, int mbb, const Code *nibbles, Code nibLen, Code balance) {
    size_t mrea = 4 + (size_t)mbb + 66, mvr = 2 + mrea, mkl = 1 + (size_t)mahb, mkr = 1 + mkl, mpk = 2 + mkr, MO = mpk + mvr;
    Blk o = B.alloc(MO + 1 + 2 * (size_t)mahb + 1 + 1 + mkl + 1 + mrea + 1 + mpk + 1 + mvr + 1, "RlpMerklePatriciaTrieLeaf");
    size_t outLen = o.pos + MO, iNib = outLen + 1, iLen = iNib + 2 * (size_t)mahb, iBal = iLen + 1, key = iBal + 1, keyLen = key + mkl,
           rea = keyLen + 1, reaLen = rea + mrea, pk = reaLen + 1, pkLen = pk + mpk, vr = pkLen + 1, vrLen = vr + mvr;
    const uint64_t d = o.sig - o.pos; const bool cs = B.want_cs();
    B.copy(iNib, nibbles, 2 * (size_t)mahb); B.at(iLen) = nibLen; B.at(iBal) = balance;
    Blk t = T_TruncatedAddressHash(B, mahb, nibbles, nibLen); B.copy(key, &B.at(t.pos), mkl); Code kl = B.at(t.pos + mkl); B.at(keyLen) = kl;
    Blk ag = T_AssertGreaterEqThan(B, 16, kl, c_const(2));
    Blk e = T_RlpEmptyAccount(B, mbb, balance); B.copy(rea, &B.at(e.pos), mrea); Code rl = B.at(e.pos + mrea); B.at(reaLen) = rl;
    B.at(vr) = c_const(0xb8); B.at(vr + 1) = rl;
    for (size_t i = 0; i < mrea; i++) B.at(vr + i + 2) = B.at(rea + i);
    Code vl = B.add(c_const(2), rl); B.at(vrLen) = vl;
    B.at(pk) = c_const(0xf8);
    B.at(pk + 1) = B.add(B.add(kl, ONE), vl);
    B.at(pk + 2) = B.add(c_const(0x80), kl);
    for (size_t i = 0; i < mkl; i++) B.at(pk + i + 3) = B.at(key + i);
    B.at(pkLen) = B.add(c_const(3), kl);
    Blk cc = T_Concat(B, (int)mpk, (int)mvr, &B.at(pk), B.at(pkLen), &B.at(vr), vl);
    B.copy(o.pos, &B.at(cc.pos), MO); B.at(outLen) = B.at(cc.pos + MO);
    if (cs) {
        const size_t ah2 = 2 * (size_t)mahb;
        B.q_eqn(t.sig + mkl + 1, d + iNib, ah2); B.q_eq(t.sig + mkl + 1 + ah2, d + iLen);                     // (key, keyLen) <== TruncatedAddressHash(maxAddressHashBytes)(addressHashNibbles, addressHashNibblesLen)   merkle_patricia_trie_leaf.circom:148
        B.q_eqn(d + key, t.sig, mkl); B.q_eq(d + keyLen, t.sig + mkl);
        B.q_eq(ag.sig, d + keyLen); B.q_const(ag.sig + 1, 2);                                                 // AssertGreaterEqThan(16)(keyLen, 2)                 :150
        B.q_eq(e.sig + mrea + 1, d + iBal); B.q_eqn(d + rea, e.sig, mrea); B.q_eq(d + reaLen, e.sig + mrea);  // (rlpEmptyAccount, len) <== RlpEmptyAccount(maxBalanceBytes)(balance)   :153-155
        B.q_const(d + vr, 0xb8); B.q_eq(d + vr + 1, d + reaLen); B.q_eqn(d + vr + 2, d + rea, mrea);          // valueRlp[0], [1], [i+2]                            :164-168
        B.q_lin(LC().s(d + vrLen, -1).k(2).s(d + reaLen));                                                    // valueRlpLen <== 2 + rlpEmptyAccountLen             :170
        B.q_const(d + pk, 0xf8);                                                                              // prefixedKeyRlp[0] <== 0xf7 + 1                     :173
        B.q_lin(LC().s(d + pk + 1, -1).s(d + keyLen).k(1).s(d + vrLen));                                      // prefixedKeyRlp[1] <== (keyLen + 1) + valueRlpLen   :174
        B.q_lin(LC().s(d + pk + 2, -1).k(0x80).s(d + keyLen));                                                // prefixedKeyRlp[2] <== 0x80 + keyLen                :175
        B.q_eqn(d + pk + 3, d + key, mkl);                                                                    // prefixedKeyRlp[i+3] <== key[i]                     :177
        B.q_lin(LC().s(d + pkLen, -1).k(3).s(d + keyLen));                                                    // prefixedKeyRlpLen <== 3 + keyLen                   :179
        B.q_eqn(cc.sig + MO + 1, d + pk, mpk); B.q_eq(cc.sig + MO + 1 + mpk, d + pkLen);                      // (out, outLen) <== Concat(...)(a <== prefixedKeyRlp, aLen <== ..., b <== valueRlp, bLen <== ...)   :182-187
        B.q_eqn(cc.sig + MO + 1 + mpk + 1, d + vr, mvr); B.q_eq(cc.sig + MO + 1 + mpk + 1 + mvr, d + vrLen);
        B.q_eqn(o.sig, cc.sig, MO); B.q_eq(d + outLen, cc.sig + MO);
    }
    return o;
}
// IsInRange(B) :196-207  own: out, lower, value, upper, lowerLteValue, valueLteUpper
static Blk T_IsInRange(Builder &B, int nb, Code lower, Code value, Code upper) {
    Blk o = B.alloc(6, "IsInRange"); B.at(o.pos + 1) = lower; B.at(o.pos + 2) = value; B.at(o.pos + 3) = upper;
    Blk b1 = T_AssertBits(B, nb, lower), b2 = T_AssertBits(B, nb, value), b3 = T_AssertBits(B, nb, upper);
    Blk a = T_LessEqThan(B, nb, lower, value); B.at(o.pos + 4) = B.at(a.pos);
    Blk b = T_LessEqThan(B, nb, value, upper); B.at(o.pos + 5) = B.at(b.pos);
    B.at(o.pos) = B.mul(B.at(a.pos), B.at(b.pos));
    if (B.want_cs()) {
        B.q_eq(b1.sig, o.sig + 1); B.q_eq(b2.sig, o.sig + 2); B.q_eq(b3.sig, o.sig + 3);                      // AssertBits(B)(lower), (value), (upper)             merkle_patricia_trie_leaf.circom:201-203
        B.q_eq(a.sig + 1, o.sig + 1); B.q_eq(a.sig + 2, o.sig + 2); B.q_eq(o.sig + 4, a.sig);                 // lowerLteValue <== LessEqThan(B)([lower, value])    :204
        B.q_eq(b.sig + 1, o.sig + 2); B.q_eq(b.sig + 2, o.sig + 3); B.q_eq(o.sig + 5, b.sig);                 // valueLteUpper <== LessEqThan(B)([value, upper])    :205
        B.q_mul(o.sig + 4, o.sig + 5, o.sig);                                                                 // out <== lowerLteValue * valueLteUpper              :206
    }
    return o;
}
// LeafDetector(N) :247-294
static Blk T_LeafDetector(Builder &B, int N, const Code *layer, Code layerLen) {
    size_t n = (size_t)N; Blk o = B.alloc(1 + n + 1 + 16, "LeafDetector");
    B.copy(o.pos + 1, layer, n); B.at(o.pos + 1 + n) = layerLen;
    size_t v = o.pos + 2 + n;
    const uint64_t qL = o.sig + 1, qLen = o.sig + 1 + n, qv = o.sig + 2 + n; const bool cs = B.want_cs();
    Blk al = T_AssertLessEqThan(B, 16, layerLen, c_const((uint32_t)n));
    if (cs) { B.q_eq(al.sig, qLen); B.q_const(al.sig + 1, n); }                                               // AssertLessEqThan(16)(layerLen, N)                  merkle_patricia_trie_leaf.circom:253
    Blk x = T_IsEqual(B, layer[0], c_const(0xf8)); B.at(v + 0) = B.at(x.pos);                              // leafPrefixIsF8
    if (cs) { B.q_eq(x.sig + 1, qL); B.q_const(x.sig + 2, 0xf8); B.q_eq(qv + 0, x.sig); }                     // :256
    Code totalLength = layer[1]; B.at(v + 1) = totalLength; B.q_eq(qv + 1, qL + 1);                          // totalLength <== layer[1]   :258
    x = T_IsEqual(B, B.add(totalLength, c_const(2)), layerLen); B.at(v + 2) = B.at(x.pos);                 // isConsistentWithLayerLen
    if (cs) { B.q_lin(LC().s(x.sig + 1).s(qv + 1, -1).k(-2)); B.q_eq(x.sig + 2, qLen); B.q_eq(qv + 2, x.sig); }   // :259
    Code keyPrefix = layer[2]; B.at(v + 3) = keyPrefix; B.q_eq(qv + 3, qL + 2);                              // keyPrefix <== layer[2]     :261
    x = T_LessEqThan(B, 16, keyPrefix, c_const(0xb7)); B.at(v + 4) = B.at(x.pos);                          // keyPrefixIsValid
    if (cs) { B.q_eq(x.sig + 1, qv + 3); B.q_const(x.sig + 2, 0xb7); B.q_eq(qv + 4, x.sig); }                 // :262
    x = T_IsInRange(B, 16, c_const(0x81), keyPrefix, c_const(0xb7)); Code multi = B.at(x.pos); B.at(v + 5) = multi;
    if (cs) { B.q_const(x.sig + 1, 0x81); B.q_eq(x.sig + 2, qv + 3); B.q_const(x.sig + 3, 0xb7); B.q_eq(qv + 5, x.sig); }   // keyIsMultiByte <== IsInRange(16)(0x81, keyPrefix, 0xb7)   :267
    Code extra = B.mul(multi, B.sub(keyPrefix, c_const(0x80))); B.at(v + 6) = extra;
    B.q_r1(LC().s(qv + 5), LC().s(qv + 3).k(-0x80), LC().s(qv + 6));                                          // keyExtraLen <== keyIsMultiByte * (keyPrefix - 0x80)   :268
    Code keyLen = B.add(ONE, extra); B.at(v + 7) = keyLen;
    B.q_lin(LC().s(qv + 7, -1).k(1).s(qv + 6));                                                               // keyLen <== 1 + keyExtraLen                        :269
    Code base = B.add(c_const(2), keyLen);
    auto sel = [&](int off, size_t dst) {                   // Selector(N)(layer, 2 + keyLen + off)          :272, :275, :278, :281
        Blk sx = T_Selector(B, N, layer, off ? B.add(base, c_const((uint32_t)off)) : base);
        B.at(v + dst) = B.at(sx.pos);
        if (cs) { B.q_eqn(sx.sig + 1, qL, n); B.q_lin(LC().s(sx.sig + 1 + n).k(-(2 + off)).s(qv + 7, -1)); B.q_eq(qv + dst, sx.sig); }
        return B.at(sx.pos);
    };
    Code vwp = sel(0, 8);
    x = T_IsEqual(B, vwp, c_const(0xb8)); B.at(v + 9) = B.at(x.pos);
    if (cs) { B.q_eq(x.sig + 1, qv + 8); B.q_const(x.sig + 2, 0xb8); B.q_eq(qv + 9, x.sig); }                 // valueWrapperPrefixIsB8     :273
    Code vwl = sel(1, 10);
    Code vp = sel(2, 11);
    x = T_IsEqual(B, vp, c_const(0xf8)); B.at(v + 12) = B.at(x.pos);
    if (cs) { B.q_eq(x.sig + 1, qv + 11); B.q_const(x.sig + 2, 0xf8); B.q_eq(qv + 12, x.sig); }               // valuePrefixIsF8            :279
    Code vlen = sel(3, 13);
    x = T_IsEqual(B, vwl, B.add(vlen, c_const(2))); B.at(v + 14) = B.at(x.pos);
    if (cs) { B.q_eq(x.sig + 1, qv + 10); B.q_lin(LC().s(x.sig + 2).s(qv + 13, -1).k(-2)); B.q_eq(qv + 14, x.sig); }   // isValueWrapperLenConsistent   :284
    x = T_IsEqual(B, B.add(B.add(keyLen, vlen), c_const(6)), layerLen); B.at(v + 15) = B.at(x.pos);
    if (cs) { B.q_lin(LC().s(x.sig + 1).s(qv + 7, -1).s(qv + 13, -1).k(-6)); B.q_eq(x.sig + 2, qLen); B.q_eq(qv + 15, x.sig); }   // isKeyValueLenEqualWithLayerLen   :287
    Code ands[7] = {B.at(v + 0), B.at(v + 2), B.at(v + 4), B.at(v + 9), B.at(v + 14), B.at(v + 12), B.at(v + 15)};
    x = T_MultiAND(B, 7, ands);
    B.at(o.pos) = B.at(x.pos);
    if (cs) {
        static const int order[7] = {0, 2, 4, 9, 14, 12, 15};
        for (int k = 0; k < 7; k++) B.q_eq(x.sig + 1 + (uint64_t)k, qv + (uint64_t)order[k]);
        B.q_eq(o.sig, x.sig);                                                                                 // isLeaf <== MultiAND(7)([...])                     :289-293
    }
    return o;
}

// ============================================================================================================
// circuits/spend.circom, circuits/proof_of_burn.circom
// ============================================================================================================
// Spend(maxAmountBytes) :32-53
static Blk T_Spend(Builder &B, int mab, Code burnKey, Code balance, Code withdrawn, Code extra) {
    Blk o = B.alloc(1 + 4 + 2 + 128, "Spend");
    B.at(o.pos + 1) = burnKey; B.at(o.pos + 2) = balance; B.at(o.pos + 3) = withdrawn; B.at(o.pos + 4) = extra;
    size_t coin = o.pos + 5, rem = o.pos + 6, by = o.pos + 7;
    const bool cs = B.want_cs();
    Blk ag = T_AssertGreaterEqThan(B, mab * 8, balance, withdrawn);
    if (cs) { B.q_eq(ag.sig, o.sig + 2); B.q_eq(ag.sig + 1, o.sig + 3); }                                     // AssertGreaterEqThan(maxAmountBytes*8)(balance, withdrawnBalance)   spend.circom:41
    Code i1[3] = {POSEIDON_PREFIX(B, 2), burnKey, balance};
    Fr pre; B.const_val(i1[0], pre);
    Blk p = T_Poseidon(B, 3, i1); B.at(coin) = B.at(p.pos);
    if (cs) { B.q_constf(p.sig + 1, pre); B.q_eq(p.sig + 2, o.sig + 1); B.q_eq(p.sig + 3, o.sig + 2); B.q_eq(o.sig + 5, p.sig); }   // coin <== Poseidon(3)([PREFIX, burnKey, balance])   :43
    Code i2[3] = {POSEIDON_PREFIX(B, 2), burnKey, B.sub(balance, withdrawn)};
    p = T_Poseidon(B, 3, i2); B.at(rem) = B.at(p.pos);
    if (cs) { B.q_constf(p.sig + 1, pre); B.q_eq(p.sig + 2, o.sig + 1); B.q_lin(LC().s(p.sig + 3).s(o.sig + 2, -1).s(o.sig + 3)); B.q_eq(o.sig + 6, p.sig); }   // remainingCoin <== Poseidon(3)([PREFIX, burnKey, balance - withdrawnBalance])   :44
    const uint64_t src[4] = {o.sig + 5, o.sig + 3, o.sig + 6, o.sig + 4};
    const Code srcc[4] = {B.at(coin), withdrawn, B.at(rem), extra};
    for (int k = 0; k < 4; k++) {                                                                             // coinBytes / withdrawnBalanceBytes / remainingCoinBytes / extraCommmitmentBytes   :46-49
        Blk x = T_Num2BigEndianBytes(B, 32, srcc[k]); B.copy(by + 32 * (size_t)k, &B.at(x.pos), 32);
        if (cs) { B.q_eq(x.sig + 32, src[k]); B.q_eqn(o.sig + 7 + 32 * (uint64_t)k, x.sig, 32); }
    }
    Blk x = T_PublicCommitment(B, 4, &B.at(by)); B.at(o.pos) = B.at(x.pos);
    if (cs) { B.q_eqn(x.sig + 1, o.sig + 7, 128); B.q_eq(o.sig, x.sig); }                                     // commitment <== PublicCommitment(4)([...])         :51
    return o;
}
struct PobParams { int maxNumLayers, maxNodeBlocks, maxHeaderBlocks, minLeafAddressNibbles, amountBytes, powMinimumZeroBytes; Fr maxIntendedBalance, maxActualBalance; };
// ProofOfBurn(...) :34-212
static Blk T_ProofOfBurn(Builder &B, const PobParams &P, const Code *in) {
    size_t L = (size_t)P.maxNumLayers, NB = (size_t)P.maxNodeBlocks * 136, HB = (size_t)P.maxHeaderBlocks * 136;
    size_t nIn = 6 + L * NB + L + 1 + HB + 3;
    size_t nMid = 2 + 64 + 32 + 32 + 5 * 32 + NB + 1 + L + (L - 1) + L * 32 + L * 31 + L + 1 + 139 + 1;
    Blk o = B.alloc(1 + nIn + nMid, "ProofOfBurn");
    B.copy(o.pos + 1, in, nIn);
    const Code *I = &B.at(o.pos + 1);
    Code burnKey = I[0], actualBalance = I[1], intendedBalance = I[2], revealAmount = I[3], bec = I[4], numLeafNib = I[5];
    const Code *layers = I + 6, *layerLens = layers + L * NB;
    Code numLayers = layerLens[L];
    const Code *blockHeader = layerLens + L + 1;
    Code blockHeaderLen = blockHeader[HB], relax = blockHeader[HB + 1], proofExtra = blockHeader[HB + 2];
    size_t remainingCoin = o.pos + 1 + nIn, nullifier = remainingCoin + 1, addrNib = nullifier + 1, blockRoot = addrNib + 64, stateRoot = blockRoot + 32,
           nullB = stateRoot + 32, remB = nullB + 32, revB = remB + 32, becB = revB + 32, ecB = becB + 32, lastLayer = ecB + 32,
           lastLayerLen = lastLayer + NB, layerExists = lastLayerLen + 1, subChk = layerExists + L, layerKec = subChk + (L - 1),
           redKec = layerKec + L * 32, isLeaf = redKec + L * 31, isLastLeaf = isLeaf + L, leaf = isLastLeaf + 1, leafLen = leaf + 139;
    // constraint side: witness indices of the inputs (circuits/proof_of_burn.circom:43-72) and of the intermediates above
    const bool cs = B.want_cs();
    const uint64_t d = o.sig - o.pos, qI = o.sig + 1, qBurnKey = qI, qActual = qI + 1, qIntended = qI + 2, qReveal = qI + 3, qBec = qI + 4, qNumNib = qI + 5,
                   qLayers = qI + 6, qLens = qLayers + L * NB, qNumLayers = qLens + L, qHeader = qNumLayers + 1, qHeaderLen = qHeader + HB, qRelax = qHeaderLen + 1, qExtra = qRelax + 1;
    int ab8 = P.amountBytes * 8;
    Blk x = T_AssertLessEqThan(B, ab8, intendedBalance, B.konst(P.maxIntendedBalance));
    if (cs) { B.q_eq(x.sig, qIntended); B.q_constf(x.sig + 1, P.maxIntendedBalance); }                        // AssertLessEqThan(amountBytes*8)(intendedBalance, maxIntendedBalance)   proof_of_burn.circom:84
    x = T_AssertLessEqThan(B, ab8, actualBalance, B.konst(P.maxActualBalance));
    if (cs) { B.q_eq(x.sig, qActual); B.q_constf(x.sig + 1, P.maxActualBalance); }                            // (actualBalance, maxActualBalance)                  :85
    x = T_AssertLessEqThan(B, ab8, intendedBalance, actualBalance);
    if (cs) { B.q_eq(x.sig, qIntended); B.q_eq(x.sig + 1, qActual); }                                         // (intendedBalance, actualBalance)                   :86
    Code relax2 = B.mul(relax, c_const(2)), minNib = c_const((uint32_t)P.minLeafAddressNibbles);
    x = T_AssertLessEqThan(B, 16, relax2, minNib);
    if (cs) { B.q_lin(LC().s(x.sig).s(qRelax, -2)); B.q_const(x.sig + 1, (uint64_t)P.minLeafAddressNibbles); }   // AssertLessEqThan(16)(byteSecurityRelax*2, minLeafAddressNibbles)   :89
    x = T_AssertGreaterEqThan(B, 16, numLeafNib, B.sub(minNib, relax2));
    if (cs) { B.q_eq(x.sig, qNumNib); B.q_lin(LC().s(x.sig + 1).k(-(int64_t)P.minLeafAddressNibbles).s(qRelax, 2)); }   // AssertGreaterEqThan(16)(numLeafAddressNibbles, min - relax*2)   :90
    x = T_AssertBits(B, ab8, revealAmount);
    B.q_eq(x.sig, qReveal);                                                                                   // AssertBits(amountBytes*8)(revealAmount)            :93
    x = T_AssertLessEqThan(B, ab8, revealAmount, intendedBalance);
    if (cs) { B.q_eq(x.sig, qReveal); B.q_eq(x.sig + 1, qIntended); }                                         // AssertLessEqThan(..)(revealAmount, intendedBalance)   :97
    for (size_t i = 0; i < L; i++) {
        x = T_AssertLessThan(B, 16, layerLens[i], c_const((uint32_t)(NB * 8)));
        if (cs) { B.q_eq(x.sig, qLens + i); B.q_const(x.sig + 1, NB * 8); }                                   // AssertLessThan(16)(layerLens[i], maxNodeBlocks*136*8)   :101
        x = T_AssertByteString(B, (int)NB, layers + i * NB);
        B.q_eqn(x.sig, qLayers + i * NB, NB);                                                                 // AssertByteString(maxNodeBlocks*136)(layers[i])     :102
    }
    x = T_AssertLessThan(B, 16, blockHeaderLen, c_const((uint32_t)(HB * 8)));
    if (cs) { B.q_eq(x.sig, qHeaderLen); B.q_const(x.sig + 1, HB * 8); }                                      // :105
    x = T_AssertByteString(B, (int)HB, blockHeader);
    B.q_eqn(x.sig, qHeader, HB);                                                                              // :106
    Code p3[3] = {POSEIDON_PREFIX(B, 2), burnKey, B.sub(intendedBalance, revealAmount)};
    x = T_Poseidon(B, 3, p3); B.at(remainingCoin) = B.at(x.pos);
    if (cs) { Fr pre; B.const_val(p3[0], pre); B.q_constf(x.sig + 1, pre); B.q_eq(x.sig + 2, qBurnKey); B.q_lin(LC().s(x.sig + 3).s(qIntended, -1).s(qReveal)); B.q_eq(d + remainingCoin, x.sig); }   // remainingCoin <== Poseidon(3)([COIN_PREFIX, burnKey, intendedBalance - revealAmount])   :113
    Code p2[2] = {POSEIDON_PREFIX(B, 1), burnKey};
    x = T_Poseidon(B, 2, p2); B.at(nullifier) = B.at(x.pos);
    if (cs) { Fr pre; B.const_val(p2[0], pre); B.q_constf(x.sig + 1, pre); B.q_eq(x.sig + 2, qBurnKey); B.q_eq(d + nullifier, x.sig); }   // nullifier <== Poseidon(2)([NULLIFIER_PREFIX, burnKey])   :116
    x = T_BurnAddressHash(B, burnKey, revealAmount, bec); B.copy(addrNib, &B.at(x.pos), 64);
    if (cs) { B.q_eq(x.sig + 64, qBurnKey); B.q_eq(x.sig + 65, qReveal); B.q_eq(x.sig + 66, qBec); B.q_eqn(d + addrNib, x.sig, 64); }     // addressHashNibbles <== BurnAddressHash()(...)   :119
    x = T_KeccakBytes(B, P.maxHeaderBlocks, blockHeader, blockHeaderLen); B.copy(blockRoot, &B.at(x.pos), 32);
    if (cs) { B.q_eqn(x.sig + 32, qHeader, HB); B.q_eq(x.sig + 32 + HB, qHeaderLen); B.q_eqn(d + blockRoot, x.sig, 32); }                 // blockRoot <== KeccakBytes(maxHeaderBlocks)(blockHeader, blockHeaderLen)   :122
    for (size_t i = 0; i < 32; i++) B.at(stateRoot + i) = blockHeader[91 + i];
    B.q_eqn(d + stateRoot, qHeader + 91, 32);                                                                 // stateRoot[i] <== blockHeader[91 + i]               :128
    {
        const size_t dst[5] = {nullB, remB, revB, becB, ecB};
        const uint64_t src[5] = {d + nullifier, d + remainingCoin, qReveal, qBec, qExtra};
        const Code srcc[5] = {B.at(nullifier), B.at(remainingCoin), revealAmount, bec, proofExtra};
        for (int k = 0; k < 5; k++) {                                                                         // nullifierBytes ... extraCommitmentBytes <== Num2BigEndianBytes(32)(..)   :131-135
            x = T_Num2BigEndianBytes(B, 32, srcc[k]); B.copy(dst[k], &B.at(x.pos), 32);
            if (cs) { B.q_eq(x.sig + 32, src[k]); B.q_eqn(d + dst[k], x.sig, 32); }
        }
    }
    {
        std::vector<Code> six(192);
        memcpy(&six[0], &B.at(blockRoot), 128); memcpy(&six[32], &B.at(nullB), 128); memcpy(&six[64], &B.at(remB), 128);
        memcpy(&six[96], &B.at(revB), 128); memcpy(&six[128], &B.at(becB), 128); memcpy(&six[160], &B.at(ecB), 128);
        x = T_PublicCommitment(B, 6, six.data()); B.at(o.pos) = B.at(x.pos);
        if (cs) { B.q_eqn(x.sig + 1, d + blockRoot, 32); B.q_eqn(x.sig + 33, d + nullB, 160); B.q_eq(o.sig, x.sig); }   // commitment <== PublicCommitment(6)([...])   :136-138
    }
    Code selLast = B.sub(numLayers, ONE);
    x = T_SelectorArray(B, P.maxNumLayers, NB, layers, selLast); B.copy(lastLayer, &B.at(x.pos), NB);
    if (cs) { B.q_eqn(x.sig + NB, qLayers, L * NB); B.q_lin(LC().s(x.sig + NB + L * NB).s(qNumLayers, -1).k(1)); B.q_eqn(d + lastLayer, x.sig, NB); }   // lastLayer <== SelectorArray1D(maxNumLayers, NB)(layers, numLayers - 1)   :141-142
    x = T_Selector(B, P.maxNumLayers, layerLens, selLast); B.at(lastLayerLen) = B.at(x.pos);
    if (cs) { B.q_eqn(x.sig + 1, qLens, L); B.q_lin(LC().s(x.sig + 1 + L).s(qNumLayers, -1).k(1)); B.q_eq(d + lastLayerLen, x.sig); }                  // lastLayerLen <== Selector(maxNumLayers)(layerLens, numLayers - 1)   :143
    x = T_Filter(B, P.maxNumLayers, numLayers); B.copy(layerExists, &B.at(x.pos), L);
    if (cs) { B.q_eq(x.sig + L, qNumLayers); B.q_eqn(d + layerExists, x.sig, L); }                            // layerExists <== Filter(maxNumLayers)(numLayers)    :146
    Code numLeaves = ZERO;
    LC leaves;
    for (size_t i = 0; i < L; i++) {
        x = T_LeafDetector(B, (int)NB, layers + i * NB, layerLens[i]); Code lf = B.at(x.pos); B.at(isLeaf + i) = lf;
        if (cs) { B.q_eqn(x.sig + 1, qLayers + i * NB, NB); B.q_eq(x.sig + 1 + NB, qLens + i); B.q_eq(d + isLeaf + i, x.sig); leaves.s(d + isLeaf + i); }   // isLeaf[i] <== LeafDetector(NB)(layers[i], layerLens[i])   :159
        numLeaves = B.add(numLeaves, lf);
        x = T_KeccakBytes(B, P.maxNodeBlocks, layers + i * NB, layerLens[i]); B.copy(layerKec + 32 * i, &B.at(x.pos), 32);
        if (cs) { B.q_eqn(x.sig + 32, qLayers + i * NB, NB); B.q_eq(x.sig + 32 + NB, qLens + i); B.q_eqn(d + layerKec + 32 * i, x.sig, 32); }              // layerKeccaks[i] <== KeccakBytes(maxNodeBlocks)(layers[i], layerLens[i])   :163
        x = T_Fit(B, 32, 31, &B.at(layerKec + 32 * i)); B.copy(redKec + 31 * i, &B.at(x.pos), 31);
        if (cs) { B.q_eqn(x.sig + 31, d + layerKec + 32 * i, 32); B.q_eqn(d + redKec + 31 * i, x.sig, 31); }                                              // reducedLayerKeccaks[i] <== Fit(32, 31)(layerKeccaks[i])   :164
        if (i > 0) {
            x = T_SubstringCheck(B, (int)NB, 31, layers + (i - 1) * NB, layerLens[i - 1], &B.at(redKec + 31 * i));
            Code sc = B.at(x.pos);
            B.at(subChk + i - 1) = sc;
            B.chk_eq(B.mul(B.not1(sc), B.at(layerExists + i)), ZERO, o.sig);
            if (cs) {
                B.q_eqn(x.sig + 1, qLayers + (i - 1) * NB, NB); B.q_eq(x.sig + 1 + NB, qLens + i - 1); B.q_eqn(x.sig + 2 + NB, d + redKec + 31 * i, 31);   // substringCheckers[i-1] <== SubstringCheck(NB, 31)(subInput, mainLen, mainInput)   :171-175
                B.q_eq(d + subChk + i - 1, x.sig);
                B.q_r1(LC().k(1).s(d + subChk + i - 1, -1), LC().s(d + layerExists + i), LC());               // (1 - substringCheckers[i-1]) * layerExists[i] === 0   :180
            }
        }
    }
    B.chk_eq(numLeaves, ONE, o.sig);
    if (cs) { leaves.k(-1); B.q_lin(leaves); }                                                                // numDetectedLeaves === 1                            :186
    x = T_LeafDetector(B, (int)NB, &B.at(lastLayer), B.at(lastLayerLen)); B.at(isLastLeaf) = B.at(x.pos);
    if (cs) { B.q_eqn(x.sig + 1, d + lastLayer, NB); B.q_eq(x.sig + 1 + NB, d + lastLayerLen); B.q_eq(d + isLastLeaf, x.sig); B.q_const(d + isLastLeaf, 1); }   // isLastLayerLeaf <== LeafDetector(..)(lastLayer, lastLayerLen); === 1   :187-188
    B.chk_eq(B.at(isLastLeaf), ONE, o.sig);
    for (size_t i = 0; i < 32; i++) B.chk_eq(B.at(layerKec + i), B.at(stateRoot + i), o.sig);
    B.q_eqn(d + layerKec, d + stateRoot, 32);                                                                 // layerKeccaks[0][i] === stateRoot[i]                :192
    x = T_RlpMerklePatriciaTrieLeaf(B, 32, P.amountBytes, &B.at(addrNib), numLeafNib, actualBalance);
    B.copy(leaf, &B.at(x.pos), 139); B.at(leafLen) = B.at(x.pos + 139);
    if (cs) {
        B.q_eqn(x.sig + 140, d + addrNib, 64); B.q_eq(x.sig + 204, qNumNib); B.q_eq(x.sig + 205, qActual);    // (leaf, leafLen) <== RlpMerklePatriciaTrieLeaf(32, amountBytes)(addressHashNibbles, numLeafAddressNibbles, actualBalance)   :198-200
        B.q_eqn(d + leaf, x.sig, 139); B.q_eq(d + leafLen, x.sig + 139);
        B.q_eqn(d + leaf, d + lastLayer, 139); B.q_eq(d + leafLen, d + lastLayerLen);                         // leaf[i] === lastLayer[i]; leafLen === lastLayerLen   :204, :206
    }
    for (size_t i = 0; i < 139; i++) B.chk_eq(B.at(leaf + i), B.at(lastLayer + i), o.sig);
    B.chk_eq(B.at(leafLen), B.at(lastLayerLen), o.sig);
    x = T_ProofOfWorkChecker(B, burnKey, revealAmount, bec, B.add(c_const((uint32_t)P.powMinimumZeroBytes), relax));
    if (cs) { B.q_eq(x.sig, qBurnKey); B.q_eq(x.sig + 1, qReveal); B.q_eq(x.sig + 2, qBec); B.q_lin(LC().s(x.sig + 3).k(-(int64_t)P.powMinimumZeroBytes).s(qRelax, -1)); }   // ProofOfWorkChecker()(burnKey, revealAmount, burnExtraCommitment, powMinimumZeroBytes + byteSecurityRelax)   :211
    return o;
}

// ============================================================================================================
// main dispatch
// ============================================================================================================
struct MainInfo { const char *name; int nparams; const char *schema; };
static const MainInfo MAINS[] = {
    {"Spend", 1, "burnKey,balance,withdrawnBalance,extraCommitment"},
    {"ProofOfBurn", 8, "burnKey,actualBalance,intendedBalance,revealAmount,burnExtraCommitment,numLeafAddressNibbles,layers[p0][p1*136],layerLens[p0],numLayers,blockHeader[p2*136],blockHeaderLen,byteSecurityRelax,_proofExtraCommitment"},
    {"EIP7503", 0, ""}, {"ConcatFixed4", 4, "a[p0],b[p1],c[p2],d[p3]"},
    {"ProofOfWorkChecker", 0, "burnKey,revealAmount,burnExtraCommitment,minimumZeroBytes"},
    {"PublicCommitment", 1, "in[p0][32]"}, {"Poseidon", 1, "inputs[p0]"}, {"Divide", 1, "a,b"},
    {"SubstringCheck", 2, "mainInput[p0],mainLen,subInput[p1]"}, {"ShiftLeft", 1, "in[p0],count"},
    {"ShiftRight", 2, "in[p0],count"}, {"Mask", 1, "in[p0],count"}, {"Concat", 2, "a[p0],aLen,b[p1],bLen"},
    {"Selector", 1, "vals[p0],select"}, {"SelectorArray1D", 2, "arrays[p0][p1],select"},
    {"SelectorArray2D", 3, "arrays[p0][p1][p2],select"}, {"BigEndianBytes2Num", 1, "in[p0]"},
    {"LittleEndianBytes2Num", 1, "in[p0]"}, {"Bytes2Nibbles", 1, "in[p0]"}, {"Num2BigEndianBytes", 1, "in"},
    {"Num2LittleEndianBytes", 1, "in"}, {"Nibbles2Bytes", 1, "nibbles[2*p0]"}, {"Num2BitsSafe", 1, "in"},
    {"Pad", 2, "in[p0*p1],inLen"}, {"KeccakBytes", 1, "in[p0*136],inLen"},
    {"BurnAddress", 0, "burnKey,revealAmount,burnExtraCommitment"}, {"BurnAddressHash", 0, "burnKey,revealAmount,burnExtraCommitment"},
    {"AssertBits", 1, "in"}, {"AssertByteString", 1, "in[p0]"}, {"AssertLessThan", 1, "a,b"}, {"AssertLessEqThan", 1, "a,b"},
    {"AssertGreaterEqThan", 1, "a,b"}, {"Filter", 1, "in"}, {"Fit", 2, "in[p0]"}, {"Reverse", 1, "in[p0]"},
    {"Flatten", 2, "in[p0][p1]"}, {"Reshape", 2, "in[p0*p1]"}, {"RlpInteger", 1, "in"}, {"CountBytes", 1, "bytes[p0]"},
    {"RlpEmptyAccount", 1, "balance"}, {"TruncatedAddressHash", 1, "addressHashNibbles[2*p0],addressHashNibblesLen"},
    {"IsInRange", 1, "lower,value,upper"}, {"LeafDetector", 1, "layer[p0],layerLen"},
    {"RlpMerklePatriciaTrieLeaf", 2, "addressHashNibbles[2*p0],addressHashNibblesLen,balance"},
    {nullptr, 0, nullptr}};

static int PI(const std::vector<Fr> &p, size_t i) {
    if (i >= p.size()) throw std::runtime_error("pob: missing template parameter");
    return (int)p[i].l[0];
}
// number of scalar inputs of a main, from its schema
static size_t count_inputs(const char *schema, const std::vector<Fr> &p) {
    size_t total = 0; const char *s = schema;
    while (*s) {
        while (*s && *s != '[' && *s != ',') s++;
        size_t n = 1;
        while (*s == '[') {
            s++; size_t term = 1, acc = 0; bool have = false;       // expression: factors joined by '*'
            while (*s && *s != ']') {
                if (*s == 'p') { s++; term *= (size_t)PI(p, (size_t)(*s - '0')); s++; have = true; }
                else if (*s >= '0' && *s <= '9') { size_t v = 0; while (*s >= '0' && *s <= '9') v = v * 10 + (size_t)(*s++ - '0'); term *= v; have = true; }
                else if (*s == '*') s++;
                else throw std::runtime_error("pob: bad schema expression");
            }
            if (have) acc = term;
            n *= acc; if (*s == ']') s++;
        }
        total += n;
        if (*s == ',') s++;
    }
    return total;
}

static uint32_t run_main(Builder &B, const std::string &name, const std::vector<Fr> &p, const Code *in) {
    auto IS = [&](const char *s) { return name == s; };
    if (IS("Spend")) { T_Spend(B, PI(p, 0), in[0], in[1], in[2], in[3]); return 1; }
    if (IS("ProofOfBurn")) {
        if (p.size() < 8) throw std::runtime_error("pob: ProofOfBurn needs 8 parameters");
        PobParams P{PI(p, 0), PI(p, 1), PI(p, 2), PI(p, 3), PI(p, 4), PI(p, 5), p[6], p[7]};
        // proof_of_burn.circom:195-204 hard-codes maxLeafLen = 139 = the output length of RlpMerklePatriciaTrieLeaf(32, 31)
        // (108 + amountBytes) and compares 139 bytes of lastLayer: any other amountBytes, or layers shorter than 139
        // bytes, do not compile in the reference either
        if (P.maxNumLayers < 1 || P.maxNodeBlocks < 1 || P.maxHeaderBlocks < 1 || P.amountBytes != 31 || (size_t)P.maxNodeBlocks * 136 < 139 ||
            (size_t)P.maxHeaderBlocks * 136 < 123)
            throw std::runtime_error("pob: unsupported ProofOfBurn shape (needs amountBytes == 31, maxNodeBlocks*136 >= 139, maxHeaderBlocks*136 >= 123)");
        T_ProofOfBurn(B, P, in); return 1;
    }
    if (IS("EIP7503")) { T_EIP7503(B); return 8; }
    if (IS("ConcatFixed4")) { int A = PI(p, 0), Bn = PI(p, 1), C = PI(p, 2), D = PI(p, 3); T_ConcatFixed4(B, A, Bn, C, D, in, in + A, in + A + Bn, in + A + Bn + C); return (uint32_t)(A + Bn + C + D); }
    if (IS("ProofOfWorkChecker")) { T_ProofOfWorkChecker(B, in[0], in[1], in[2], in[3]); return 0; }
    if (IS("PublicCommitment")) { T_PublicCommitment(B, PI(p, 0), in); return 1; }
    if (IS("Poseidon")) { T_Poseidon(B, PI(p, 0), in); return 1; }
    if (IS("Divide")) { T_Divide(B, PI(p, 0), in[0], in[1]); return 2; }
    if (IS("SubstringCheck")) { int mm = PI(p, 0); T_SubstringCheck(B, mm, PI(p, 1), in, in[mm], in + mm + 1); return 1; }
    if (IS("ShiftLeft")) { int n = PI(p, 0); T_ShiftLeft(B, n, in, in[n]); return (uint32_t)n; }
    if (IS("ShiftRight")) { int n = PI(p, 0), ms = PI(p, 1); T_ShiftRight(B, n, ms, in, in[n]); return (uint32_t)(n + ms); }
    if (IS("Mask")) { int n = PI(p, 0); T_Mask(B, n, in, in[n]); return (uint32_t)n; }
    if (IS("Concat")) { int A = PI(p, 0), Bn = PI(p, 1); T_Concat(B, A, Bn, in, in[A], in + A + 1, in[A + 1 + Bn]); return (uint32_t)(A + Bn + 1); }
    if (IS("Selector")) { int n = PI(p, 0); T_Selector(B, n, in, in[n]); return 1; }
    if (IS("SelectorArray1D")) { int n = PI(p, 0), q = PI(p, 1); T_SelectorArray(B, n, (size_t)q, in, in[n * q]); return (uint32_t)q; }
    if (IS("SelectorArray2D")) { int n = PI(p, 0), q = PI(p, 1) * PI(p, 2); T_SelectorArray(B, n, (size_t)q, in, in[n * q]); return (uint32_t)q; }
    if (IS("BigEndianBytes2Num")) { T_BigEndianBytes2Num(B, PI(p, 0), in); return 1; }
    if (IS("LittleEndianBytes2Num")) { T_LittleEndianBytes2Num(B, PI(p, 0), in); return 1; }
    if (IS("Bytes2Nibbles")) { T_Bytes2Nibbles(B, PI(p, 0), in); return (uint32_t)(2 * PI(p, 0)); }
    if (IS("Num2BigEndianBytes")) { T_Num2BigEndianBytes(B, PI(p, 0), in[0]); return (uint32_t)PI(p, 0); }
    if (IS("Num2LittleEndianBytes")) { T_Num2LittleEndianBytes(B, PI(p, 0), in[0]); return (uint32_t)PI(p, 0); }
    if (IS("Nibbles2Bytes")) { T_Nibbles2Bytes(B, PI(p, 0), in); return (uint32_t)PI(p, 0); }
    if (IS("Num2BitsSafe")) { T_Num2BitsSafe(B, PI(p, 0), in[0]); return (uint32_t)PI(p, 0); }
    if (IS("Pad")) { int Bn = PI(p, 0) * PI(p, 1); T_Pad(B, PI(p, 0), PI(p, 1), in, in[Bn]); return (uint32_t)(Bn + 1); }
    if (IS("KeccakBytes")) { int Bn = PI(p, 0) * 136; T_KeccakBytes(B, PI(p, 0), in, in[Bn]); return 32; }
    if (IS("BurnAddress")) { T_BurnAddress(B, in[0], in[1], in[2]); return 20; }
    if (IS("BurnAddressHash")) { T_BurnAddressHash(B, in[0], in[1], in[2]); return 64; }
    if (IS("AssertBits")) { T_AssertBits(B, PI(p, 0), in[0]); return 0; }
    if (IS("AssertByteString")) { T_AssertByteString(B, PI(p, 0), in); return 0; }
    if (IS("AssertLessThan")) { T_AssertLessThan(B, PI(p, 0), in[0], in[1]); return 0; }
    if (IS("AssertLessEqThan")) { T_AssertLessEqThan(B, PI(p, 0), in[0], in[1]); return 0; }
    if (IS("AssertGreaterEqThan")) { T_AssertGreaterEqThan(B, PI(p, 0), in[0], in[1]); return 0; }
    if (IS("Filter")) { T_Filter(B, PI(p, 0), in[0]); return (uint32_t)PI(p, 0); }
    if (IS("Fit")) { T_Fit(B, PI(p, 0), PI(p, 1), in); return (uint32_t)PI(p, 1); }
    if (IS("Reverse")) { T_Reverse(B, PI(p, 0), in); return (uint32_t)PI(p, 0); }
    if (IS("Flatten") || IS("Reshape")) { size_t n = (size_t)PI(p, 0) * (size_t)PI(p, 1); T_CopyArray(B, n, in); return (uint32_t)n; }
    if (IS("RlpInteger")) { T_RlpInteger(B, PI(p, 0), in[0]); return (uint32_t)(PI(p, 0) + 2); }
    if (IS("CountBytes")) { T_CountBytes(B, PI(p, 0), in); return 1; }
    if (IS("RlpEmptyAccount")) { T_RlpEmptyAccount(B, PI(p, 0), in[0]); return (uint32_t)(4 + PI(p, 0) + 66 + 1); }
    if (IS("TruncatedAddressHash")) { int a = PI(p, 0); T_TruncatedAddressHash(B, a, in, in[2 * a]); return (uint32_t)(a + 2); }
    if (IS("IsInRange")) { T_IsInRange(B, PI(p, 0), in[0], in[1], in[2]); return 1; }
    if (IS("LeafDetector")) { int n = PI(p, 0); T_LeafDetector(B, n, in, in[n]); return 1; }
    if (IS("RlpMerklePatriciaTrieLeaf")) {
        int a = PI(p, 0), b = PI(p, 1); T_RlpMerklePatriciaTrieLeaf(B, a, b, in, in[2 * a], in[2 * a + 1]);
        return (uint32_t)((4 + a) + (2 + 4 + b + 66) + 1);
    }
    throw std::runtime_error("pob: unknown main template '" + name + "'");
}

struct BuildOut { uint32_t n_words; };

static void build(Builder &B, const std::string &name, const std::vector<Fr> &params, size_t n_in, uint32_t *n_out) {
    std::vector<Code> in(n_in ? n_in : 1);
    for (size_t i = 0; i < n_in; i++) { uint32_t s = B.new_val(0); in[i] = c_val(s); }
    *n_out = run_main(B, name, params, in.data());
}

}  // namespace

const char *main_input_schema(const std::string &main_name, int *nparams) {
    for (const MainInfo *m = MAINS; m->name; m++)
        if (main_name == m->name) { if (nparams) *nparams = m->nparams; return m->schema; }
    return nullptr;
}

// 64-signal group descriptors of a table of BIT codes relative to a round's word base (program.h: Program::round_desc);
// throws when a group is neither a lane nor a phase of a gate array (the derivation doubles as a check of the table)
static std::vector<uint64_t> derive_round_desc(const Code *codes, uint32_t n) {
    if (n % 64) throw std::runtime_error("pob: internal: round table size is not a multiple of 64");
    std::vector<uint64_t> desc(n / 64);
    for (uint32_t g = 0; g < n / 64; g++) {
        const Code *c = codes + 64 * g;
        auto W = [&](int j) { return (code_payload(c[j]) >> 6); };
        auto Bt = [&](int j) { return (code_payload(c[j]) & 63u); };
        bool ok = true, lane = true;
        for (int j = 0; j < 64; j++) { if (code_kind(c[j]) != K_BIT) ok = false; if (W(j) != W(0) || Bt(j) != (uint32_t)j) lane = false; }
        uint64_t d = 0;
        if (ok && lane) d = (uint64_t)W(0);
        else if (ok) {
            bool found = false;
            for (uint32_t f = 0; f < 3 && !found; f++) {
                uint32_t w[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}; bool m = true;
                for (uint32_t j = 0; j < 64 && m; j++) {
                    uint32_t sidx = 64 * f + j, gi = sidx / 3, mem = sidx % 3;
                    if (Bt((int)j) != gi) m = false;
                    else if (w[mem] == 0xffffffffu) w[mem] = W((int)j);
                    else if (w[mem] != W((int)j)) m = false;
                }
                if (m) { d = (uint64_t)w[0] | ((uint64_t)w[1] << 16) | ((uint64_t)w[2] << 32) | ((uint64_t)(1 + f) << 48); found = true; }
            }
            ok = found;
        }
        // k_expand_round indexes its shared-memory word table with all three descriptor words
        if (!ok || (d & 0xffff) >= ROUND_WORDS_SPAN || ((d >> 48) && (((d >> 16) & 0xffff) >= ROUND_WORDS_SPAN || ((d >> 32) & 0xffff) >= ROUND_WORDS_SPAN)))
            throw std::runtime_error("pob: internal: round table group does not fit a descriptor");
        desc[g] = d;
    }
    return desc;
}

// ---- `--O1`-style reduction (SURVEY.md 8(f) rank 2) --------------------------------------------------------------------
// circom's default simplifier (the reference deploys through it: .github/workflows/circuitscan.yml:29,36) removes signals
// tied by `signal = signal` and `signal = constant` constraints.  Here: union-find over the eq records of the constraint
// system (the shared KeccakfRound set is resolved once and stamped into every round block), a class is "constant" when one
// of its members has a kc record; a signal stays iff it is a main input / output, or the lowest-numbered member of a
// non-constant class.  Which member circom keeps, and whether it also folds constraints that BECOME linear after the
// substitution, is not pinned by anything in the reference (no circom here): parity of the reduced ORDER is unpinned; every
// retained value equals the --O0 witness through witness_map (tested).
struct Reduction { std::vector<uint32_t> round_keep; std::vector<uint8_t> keep_flat; uint64_t n_kept = 0; };
static uint32_t uf_find(std::vector<uint32_t> &p, uint32_t x) { while (p[x] != x) { p[x] = p[p[x]]; x = p[x]; } return x; }
static void uf_union(std::vector<uint32_t> &p, uint32_t a, uint32_t b) { a = uf_find(p, a); b = uf_find(p, b); if (a == b) return; if (a < b) p[b] = a; else p[a] = b; }

// equality classes of the N --O0 signals under the eq records of a compiled constraint system (the representative of a class is its
// lowest-numbered member), and which classes are constant (a member has a kc record; witness[0]'s class always is)
struct EqClasses {
    std::vector<uint32_t> parent; std::vector<uint8_t> is_const_root;
    uint32_t root(uint32_t s) { return uf_find(parent, s); }
};
static EqClasses eq_classes(const Program &P, uint64_t N) {
    EqClasses E;
    std::vector<uint32_t> &parent = E.parent; std::vector<uint8_t> &is_const_root = E.is_const_root;
    // the shared round set, resolved once: relative representative (lowest index) and constness per relative signal
    std::vector<uint32_t> rp(ROUND_SIGNALS); for (uint32_t i = 0; i < ROUND_SIGNALS; i++) rp[i] = i;
    for (size_t i = 0; i + 1 < P.cons_round.eq.size(); i += 2) uf_union(rp, P.cons_round.eq[i], P.cons_round.eq[i + 1]);
    std::vector<uint8_t> rconst(ROUND_SIGNALS, 0);
    for (const ConsTerm &t : P.cons_round.kc) rconst[uf_find(rp, t.idx)] = 1;
    parent.resize(N); is_const_root.assign(N, 0);
    for (uint64_t i = 0; i < N; i++) parent[i] = (uint32_t)i;
    for (uint64_t base : P.round_block_sig) for (uint32_t i = 0; i < ROUND_SIGNALS; i++) { const uint32_t r = uf_find(rp, i); parent[base + i] = (uint32_t)(base + r); if (r == i && rconst[i]) is_const_root[base + i] = 1; }
    for (size_t i = 0; i + 1 < P.cons_flat.eq.size(); i += 2) {
        uint32_t a = uf_find(parent, P.cons_flat.eq[i]), b2 = uf_find(parent, P.cons_flat.eq[i + 1]);
        if (a == b2) continue;
        const uint8_t c = is_const_root[a] | is_const_root[b2];
        if (a < b2) { parent[b2] = a; is_const_root[a] = c; } else { parent[a] = b2; is_const_root[b2] = c; }
    }
    for (const ConsTerm &t : P.cons_flat.kc) is_const_root[uf_find(parent, t.idx)] = 1;
    is_const_root[uf_find(parent, 0)] = 1;                                    // witness[0] itself is kept as main I/O
    return E;
}

Program compile_circuit(const std::string &main_name, const std::vector<Fr> &params, bool hcreate, bool want_constraints, int opt_level) {
    if (opt_level < 0 || opt_level > 1) throw std::runtime_error("pob: opt_level must be 0 (--O0) or 1 (signal=signal / signal=constant elimination)");
    const bool user_wants_constraints = want_constraints;
    if (opt_level) want_constraints = true;
    int np = 0; const char *schema = main_input_schema(main_name, &np);
    if (!schema) throw std::runtime_error("pob: unknown main template '" + main_name + "'");
    if ((int)params.size() < np) throw std::runtime_error("pob: too few template parameters for " + main_name);
    size_t n_in = count_inputs(schema, params);
    uint32_t n_out = 0;
    uint32_t n_words;
    { Builder dry(hcreate, true, 0); build(dry, main_name, params, n_in, &n_out); n_words = dry.n_words; }
    uint32_t val_base = (n_words + 3u) & ~3u;
    Builder B(hcreate, false, val_base);
    Program P;
    std::unordered_map<std::array<uint32_t, 8>, uint32_t, FrHash> cons_kix;
    if (want_constraints) {
        B.cs.S = &P.cons_flat; B.cs.konst = &P.cons_konst; B.cs.kix = &cons_kix;
        B.q_const(0, 1);                                                          // witness[0] is the constant 1
    }
    build(B, main_name, params, n_in, &n_out);
    if (want_constraints) {
        ConsSink rs; rs.S = &P.cons_round; rs.konst = &P.cons_konst; rs.kix = &cons_kix;
        RoundCons rc{rs}; rc.round();
        if (rc.cur != ROUND_SIGNALS) throw std::runtime_error("pob: internal: KeccakfRound constraint walk covers " + std::to_string(rc.cur) + " signals");
        P.round_block_sig = B.round_sigs; P.has_constraints = true;
        if (P.cons_konst.empty()) P.cons_konst.push_back(fr_zero());
    }

    P.main_name = main_name; P.params = params; P.hcreate = hcreate;
    P.n_signals = B.nsig; P.n_outputs = n_out; P.n_inputs = (uint32_t)n_in; P.input_schema = schema;
    P.n_words = B.n_words; P.val_base = val_base; P.n_vals = B.n_vals;
    if (P.store_u64() >= MAX_STORE_U64) throw std::runtime_error("pob: instance store exceeds the 128 MiB code range");
    P.aux = B.aux; P.konst = B.konsts;
    if (P.konst.empty()) P.konst.push_back(fr_zero());
    if (P.aux.empty()) P.aux.push_back(0);
    // ---- levelise ----
    // OP_INV results (the `inv` hint signal of IsZero) are consumed by no other op.  The ones whose input is a small value (the
    // overwhelming majority: differences of indices, bytes, lengths) are ordinary thread ops of their level -- a table lookup.  The
    // ones expected to need a real field inversion (`likely_large`: SubstringCheck's exists[], RlpInteger's IsZero(balance)) are
    // DEFERRED: batch-inverted with Montgomery's trick, one inversion per worker thread, and that inversion is spread over the
    // levels that follow the one where their inputs are ready (kernels.cuh: k_eval) instead of sitting at the end of the kernel.
    std::vector<uint8_t> is_inv_slot(B.n_vals, 0);
    B.inv_generic.resize(B.n_vals, 0);
    auto deferred = [&](const Op &o) { return op_opc(o) == OP_INV && B.inv_generic[op_dst(o)] != 0; };
    size_t n_inv = 0; uint32_t ginv_ready = 0;
    for (auto &o : B.ops) if (op_opc(o.op) == OP_INV) { is_inv_slot[op_dst(o.op)] = 1; if (deferred(o.op)) { n_inv++; ginv_ready = std::max(ginv_ready, o.level); } }
    auto uses_inv = [&](Code c) { return code_kind(c) == K_VAL && is_inv_slot[code_payload(c)]; };
    for (auto &o : B.ops) {
        uint32_t opc = op_opc(o.op);
        bool bad = false;
        if (opc == OP_FMA) bad = uses_inv(o.op.a) || uses_inv(o.op.b) || uses_inv(o.op.c);
        else if (opc == OP_CHK_EQ || opc == OP_DIV || opc == OP_MOD) bad = uses_inv(o.op.a) || uses_inv(o.op.b);
        else if (opc != OP_PACK8) bad = uses_inv(o.op.a);
        if (bad) throw std::runtime_error("pob: internal: an IsZero inverse is consumed by another op");
    }
    for (Code c : B.aux) if (uses_inv(c)) throw std::runtime_error("pob: internal: an IsZero inverse is consumed by an operand list");
    uint32_t max_level = 0;
    for (auto &o : B.ops) if (!deferred(o.op)) max_level = std::max(max_level, o.level);
    for (auto &a : B.absorbs) max_level = std::max(max_level, a.level);
    for (auto &q : B.poseidons) max_level = std::max(max_level, q.level);
    for (auto &q : B.psums) max_level = std::max(max_level, q.level);
    std::vector<uint32_t> scount(max_level + 2, 0), sstart(max_level + 2, 0);
    for (auto &q : B.psums) scount[q.level]++;
    for (uint32_t l = 1; l <= max_level + 1; l++) sstart[l] = sstart[l - 1] + scount[l - 1];
    P.psums.resize(B.psums.size());
    { std::vector<uint32_t> sp = sstart; for (auto &q : B.psums) P.psums[sp[q.level]++] = q.op; }
    for (auto &q : B.psums) if (uses_inv(q.op.x0)) throw std::runtime_error("pob: internal: an IsZero inverse feeds a prefix sum");
    std::vector<uint32_t> pcount(max_level + 2, 0), pstart(max_level + 2, 0);
    for (auto &q : B.poseidons) pcount[q.level]++;
    for (uint32_t l = 1; l <= max_level + 1; l++) pstart[l] = pstart[l - 1] + pcount[l - 1];
    P.poseidons.resize(B.poseidons.size());
    { std::vector<uint32_t> pp = pstart; for (auto &q : B.poseidons) P.poseidons[pp[q.level]++] = q.op; }
    P.pos_konst = B.pos_konst; if (P.pos_konst.empty()) P.pos_konst.push_back(fr_zero());
    for (auto &q : B.poseidons) for (uint32_t j = 0; j < q.op.t; j++) if (uses_inv(B.aux[q.op.in_aux + j])) throw std::runtime_error("pob: internal: an IsZero inverse feeds a Poseidon");
    std::vector<uint32_t> tcount(max_level + 2, 0), wcount(max_level + 2, 0);
    for (auto &o : B.ops) if (!deferred(o.op)) tcount[o.level]++;
    for (auto &a : B.absorbs) wcount[a.level]++;
    std::vector<uint32_t> tstart(max_level + 2, 0), wstart(max_level + 2, 0);
    for (uint32_t l = 1; l <= max_level + 1; l++) { tstart[l] = tstart[l - 1] + tcount[l - 1]; wstart[l] = wstart[l - 1] + wcount[l - 1]; }
    P.ops.resize(B.ops.size()); P.absorbs.resize(B.absorbs.size());
    P.inv_begin = (uint32_t)(B.ops.size() - n_inv); P.inv_end = (uint32_t)B.ops.size();
    P.ginv_begin = P.inv_begin;                              // (the table-sized group is no longer deferred)
    { std::vector<uint32_t> tp = tstart, wp = wstart; uint32_t gp = P.ginv_begin;
      for (auto &o : B.ops) {
          if (deferred(o.op)) P.ops[gp++] = o.op;
          else P.ops[tp[o.level]++] = o.op;
      }
      for (auto &a : B.absorbs) P.absorbs[wp[a.level]++] = a.op; }
    // inside a level: long sequential ops first, then grouped by opcode / operand class so that the 32 lanes of a
    // warp run the same case of the interpreter switch (and the same fast or slow multiplication path)
    auto op_key = [](const Op &o) -> uint32_t {
        uint32_t opc = op_opc(o);
        uint32_t k = (opc + 2) << 4;
        if (opc == OP_FMA) k |= (o.b == c_const(1)) ? 0u : (o.b == c_konst(0)) ? 1u : (code_kind(o.b) == K_KONST) ? 3u : 2u;
        return k;
    };
    for (uint32_t l = 1; l <= max_level; l++) {
        if (tcount[l] == 0 && wcount[l] == 0 && pcount[l] == 0 && scount[l] == 0) continue;
        std::stable_sort(P.ops.begin() + tstart[l], P.ops.begin() + tstart[l] + tcount[l], [&](const Op &x, const Op &y) { return op_key(x) < op_key(y); });
        if (n_inv && l >= ginv_ready && P.ginv_level == 0xffffffffu) P.ginv_level = (uint32_t)P.levels.size();   // first level that starts with every deferred input ready
        P.levels.push_back(Level{tstart[l], tstart[l] + tcount[l], wstart[l], wstart[l] + wcount[l], pstart[l], pstart[l] + pcount[l], sstart[l], sstart[l] + scount[l]});
    }
    if (P.ginv_level == 0xffffffffu) P.ginv_level = (uint32_t)P.levels.size();
    // ---- renumber the value slots in execution order ----
    // Slot numbers are labels; after levelising and sorting they are scattered.  Renumbered in (level, op order) the 32 lanes of a
    // warp store 32 consecutive slots (one 1 KB run instead of 32 scattered sectors) and next-level operand loads fall into the
    // same lines.  Inputs keep slots [0, n_in); Poseidon / prefix-sum blocks move as blocks; the deferred inverses come last.
    {
        const uint32_t NV = B.n_vals;
        std::vector<uint32_t> remap(NV, 0xffffffffu);
        uint32_t next = 0;
        for (uint32_t i = 0; i < (uint32_t)n_in; i++) remap[i] = next++;
        auto has_dst = [](uint32_t opc) { return opc == OP_FMA || opc == OP_ISZ || opc == OP_INV || opc == OP_DIV || opc == OP_MOD || opc == OP_GTC || opc == OP_SELSUM; };
        auto take = [&](uint32_t old, uint32_t n) { for (uint32_t k = 0; k < n; k++) { if (remap[old + k] != 0xffffffffu) throw std::runtime_error("pob: internal: value slot defined twice"); remap[old + k] = next++; } };
        for (const Level &L : P.levels) {
            for (uint32_t i = L.t_begin; i < L.t_end; i++) if (has_dst(op_opc(P.ops[i]))) take(op_dst(P.ops[i]), 1);
            for (uint32_t q = L.p_begin; q < L.p_end; q++) if (P.poseidons[q].q0 == 0) take(P.poseidons[q].base, pos_layout(P.poseidons[q].t).total);
            for (uint32_t q = L.s_begin; q < L.s_end; q++) take(P.psums[q].dst, P.psums[q].n);
        }
        for (uint32_t i = P.inv_begin; i < P.inv_end; i++) take(op_dst(P.ops[i]), 1);
        if (next != NV) throw std::runtime_error("pob: internal: slot renumbering covers " + std::to_string(next) + " of " + std::to_string(NV) + " slots");
        auto rc = [&](Code c) -> Code {
            const uint32_t k = code_kind(c), pl = code_payload(c);
            if (k == K_VAL) return c_val(remap[pl]);
            if (k == K_BIT) {
                const uint32_t idx = pl >> 6;
                if (idx >= val_base) { const uint32_t slot = (idx - val_base) / 4, limb = (idx - val_base) % 4; return c_bit(val_base + 4 * remap[slot] + limb, pl & 63u); }
            }
            return c;
        };
        for (Op &o : P.ops) {
            const uint32_t opc = op_opc(o);
            if (has_dst(opc)) o.opc_dst = (opc << 26) | remap[op_dst(o)];
            if (opc == OP_PACK8) continue;                       // a = raw aux offset
            o.a = rc(o.a);
            if (opc == OP_FMA || opc == OP_CHK_EQ || opc == OP_DIV || opc == OP_MOD) o.b = rc(o.b);
            if (opc == OP_FMA) o.c = rc(o.c);
        }
        for (Code &c : P.aux) c = rc(c);
        for (PsumOp &q : P.psums) { q.dst = remap[q.dst]; q.x0 = rc(q.x0); }
        for (PoseidonOp &q : P.poseidons) q.base = remap[q.base];
        for (size_t i = 0; i < B.flat_n; i++) B.flat[i] = rc(B.flat[i]);
    }
    // ---- reduced witness: which signals stay ----
    std::vector<uint32_t> round_keep;            // retained relative indices inside a KeccakfRound block (same for every block)
    if (opt_level) {
        const uint64_t N = B.nsig;
        EqClasses E = eq_classes(P, N);
        const uint64_t n_io = 1ull + n_out + n_in;
        auto kept = [&](uint64_t s) { if (s < n_io) return true; const uint32_t r = E.root((uint32_t)s); return r == s && !E.is_const_root[r]; };
        // inside a round block the retained set must be the same for all blocks (it is: in/out tie to the enclosing Keccakf's
        // lower-numbered midRound signals, everything else is block-internal); verified below while the map is built
        if (!B.round_sigs.empty()) { const uint64_t b0 = B.round_sigs[0]; for (uint32_t i = 0; i < ROUND_SIGNALS; i++) if (kept(b0 + i)) round_keep.push_back(i); }
        P.witness_map.reserve(N / 8);
        for (auto &sg : B.segs) {
            if (sg.round) {
                size_t k = 0;
                for (uint32_t i = 0; i < ROUND_SIGNALS; i++) {
                    const bool kp = kept(sg.dst + i);
                    const bool want = k < round_keep.size() && round_keep[k] == i;
                    if (kp != want) throw std::runtime_error("pob: internal: KeccakfRound blocks do not reduce uniformly");
                    if (kp) { P.witness_map.push_back((uint32_t)(sg.dst + i)); k++; }
                }
            } else for (uint64_t i = 0; i < sg.n; i++) if (kept(sg.dst + i)) P.witness_map.push_back((uint32_t)(sg.dst + i));
        }
    }
    // ---- codes + tiles ----
    P.codes.resize(ROUND_SIGNALS);
    { LaneSink S{P.codes.data(), 0}; emit_round(S);
      if ((size_t)(S.p - P.codes.data()) != ROUND_SIGNALS) throw std::runtime_error("pob: internal: round table size mismatch"); }
    P.round_desc = derive_round_desc(P.codes.data(), ROUND_SIGNALS);
    P.n_round_blocks = B.n_round_blocks; P.n_flat_signals = B.flat_n; P.n_signals_o0 = B.nsig; P.opt_level = opt_level;
    if (opt_level) {
        // reduced program: codes = [retained entries of the shared round table | retained flat codes]; every tile goes
        // through the generic code path (k_expand_codes), round blocks as tiles over the shared table with their own ubase
        std::vector<Code> rt(round_keep.size()); for (size_t k = 0; k < round_keep.size(); k++) rt[k] = P.codes[round_keep[k]];
        P.codes = rt;
        const uint32_t RT = (uint32_t)round_keep.size();
        // what stays of a round block are whole 64-signal lanes (the `out` of every gate of a gate array, the NotArray outputs):
        // the descriptor-driven k_expand_round applies to the reduced blocks too
        bool fast_round = true;
        try { P.round_desc = derive_round_desc(rt.data(), RT); } catch (const std::exception &) { fast_round = false; P.round_desc.assign(1, 0); }
        if (P.round_desc.empty()) P.round_desc.assign(1, 0);
        P.out_code_off = RT + 1;
        uint64_t dst = 0; size_t mp = 0;
        const uint32_t ts = TILE_SIGNALS;
        for (auto &sg : B.segs) {
            if (sg.round) {
                const uint32_t rts = (fast_round && RT <= MAX_TILE_SIGNALS) ? RT : ts;      // one CTA streams what is left of a round block (266 KB)
                for (uint32_t done = 0; done < RT; done += rts) { Tile t; t.dst = dst + done; t.n = std::min(rts, RT - done); t.code_off = done; t.ubase = sg.ubase; t.pad = fast_round ? 1 : 0; P.tiles.push_back(t); }
                dst += RT; mp += RT;
            } else {
                const size_t first = P.codes.size();
                while (mp < P.witness_map.size() && P.witness_map[mp] < sg.dst + sg.n) { P.codes.push_back(B.flat[sg.pos + (P.witness_map[mp] - sg.dst)]); mp++; }
                const uint64_t n = P.codes.size() - first;
                for (uint64_t done = 0; done < n; done += ts) { Tile t; t.dst = dst + done; t.n = (uint32_t)std::min<uint64_t>(ts, n - done); t.code_off = (uint32_t)(first + done); t.ubase = 0; t.pad = 0; P.tiles.push_back(t); }
                dst += n;
            }
        }
        if (dst != P.witness_map.size() || mp != P.witness_map.size()) throw std::runtime_error("pob: internal: reduced layout does not add up");
        P.n_signals = dst;
        if (!user_wants_constraints) { P.cons_flat = ConsSet(); P.cons_round = ConsSet(); P.has_constraints = false; }
        std::stable_sort(P.tiles.begin(), P.tiles.end(), [](const Tile &a, const Tile &b) { return a.pad > b.pad; });
        return P;
    }
    P.codes.insert(P.codes.end(), B.flat, B.flat + B.flat_n);
    uint32_t tile_signals = LAYOUT_TILE_SIGNALS;
#ifdef POB_TUNING
    if (const char *v = getenv("POB_TILE_SIGNALS")) { uint32_t t = (uint32_t)atoi(v); if (t >= 128 && t <= TILE_SIGNALS && t % 128 == 0) tile_signals = t; }   // 128: the TMA copy of a tile's descriptors needs 16-byte alignment
#endif
    for (auto &s : B.segs) {
        uint64_t done = 0;
        while (done < s.n) {
            uint32_t n = (uint32_t)std::min<uint64_t>(tile_signals, s.n - done);
            Tile t; t.dst = s.dst + done; t.n = n; t.pad = 0;
            if (s.round) { t.code_off = (uint32_t)done; t.ubase = s.ubase; t.pad = 1; }
            else { t.code_off = (uint32_t)(ROUND_SIGNALS + s.pos + done); t.ubase = 0; }
            P.tiles.push_back(t); done += n;
        }
    }
    // Tile order is free (every tile carries its own destination).  KeccakfRound tiles only read L1-resident tables, the
    // other tiles read their code stream and store values through L2/DRAM; interleaving those reads with the write
    // stream costs DRAM efficiency, so all round tiles go first, the rest last.
    std::stable_sort(P.tiles.begin(), P.tiles.end(), [](const Tile &a, const Tile &b) { return a.pad > b.pad; });
    return P;
}

// ---- the .r1cs row plan (r1cs.h) -----------------------------------------------------------------------------------------
// A combination as (sort key, coefficient): key = wire, except in the block-relative round set, where CONS_ONE (wire 0) is key 0
// and relative signal i is key i + 1, so that ascending keys are ascending absolute wires in every block.
static uint64_t lc_key(uint32_t idx, bool rel) { return idx == CONS_ONE ? 0 : rel ? (uint64_t)idx + 1 : idx; }
static uint64_t lc_idx(uint64_t key, bool rel) { return !rel ? key : key == 0 ? CONS_ONE : key - 1; }
static LC lc_of(const ConsTerm *t, uint32_t n, const std::vector<Fr> &konst, bool rel) {
    LC L; for (uint32_t i = 0; i < n; i++) L.sf(lc_key(t[i].idx, rel), cons_coef_value(t[i].coef, konst.data(), 0)); return L;
}
// merge by key, drop zero coefficients, sort ascending
static void lc_normalize(LC &L) {
    std::sort(L.t.begin(), L.t.end(), [](const std::pair<uint64_t, Fr> &x, const std::pair<uint64_t, Fr> &y) { return x.first < y.first; });
    size_t o = 0;
    for (size_t i = 0; i < L.t.size();) {
        std::pair<uint64_t, Fr> m = L.t[i++];
        while (i < L.t.size() && L.t[i].first == m.first) m.second = fr_add(m.second, L.t[i++].second);
        if (!fr_is_zero(m.second)) L.t[o++] = m;
    }
    L.t.resize(o);
}
static void lc_unkey(LC &L, bool rel) { for (auto &q : L.t) q.first = lc_idx(q.first, rel); }
// one r1 row of the plan: normalised, B emptied when A is, left out when A and C are empty (returns false then)
static bool plan_r1(ConsSink &S, LC &A, LC &Bq, LC &C, bool rel) {
    lc_normalize(A); lc_normalize(Bq); lc_normalize(C);
    if (A.t.empty()) Bq.t.clear();
    if (A.t.empty() && C.t.empty()) return false;
    lc_unkey(A, rel); lc_unkey(Bq, rel); lc_unkey(C, rel);
    S.r1(A, Bq, C);
    return true;
}

// --O0 rows of one ConsSet: eq with a == b, kc `w0 == 1` and all-empty r1 records dropped, hints dropped, r1 combinations normalised
static void plan_o0_set(const ConsSet &in, ConsSink &S, bool rel) {
    const std::vector<Fr> &konst = *S.konst;
    for (size_t i = 0; i + 1 < in.eq.size(); i += 2) if (in.eq[i] != in.eq[i + 1]) S.eq(in.eq[i], in.eq[i + 1]);
    for (const ConsTerm &t : in.kc) {
        const bool on_one = t.idx == CONS_ONE || (!rel && t.idx == 0);
        if (on_one && cc_kind(t.coef) != CC_RCBIT && fr_eq(cons_coef_value(t.coef, konst.data(), 0), fr_from_u64(1))) continue;   // 1 w0 - 1 w0
        S.kc_raw(t.idx, t.coef);
    }
    for (const ConsR1 &r : in.r1) {
        if (r1_hint(r)) continue;
        const ConsTerm *t = in.terms.data() + r.off;
        LC A = lc_of(t, r.na, konst, rel), Bq = lc_of(t + r.na, r.nb, konst, rel), C = lc_of(t + r.na + r.nb, r1_nc(r), konst, rel);
        plan_r1(S, A, Bq, C, rel);
    }
}

// terms of the rows of one set in block round r (kc rows: C = w[a] - k w0 has 1 or 2 terms; eq rows 2)
static uint64_t plan_set_terms(const ConsSet &S, const std::vector<Fr> &konst, bool rel, uint64_t rc) {
    uint64_t n = S.eq.size();
    for (const ConsTerm &t : S.kc) {
        const bool on_one = t.idx == CONS_ONE || (!rel && t.idx == 0);
        n += (on_one || fr_is_zero(cons_coef_value(t.coef, konst.data(), rc))) ? 1 : 2;
    }
    for (const ConsR1 &r : S.r1) n += r.na + r.nb + r1_nc(r);
    return n;
}

RowPlan build_row_plan(const std::string &main_name, const std::vector<Fr> &params, bool hcreate, int opt_level) {
    Program P = compile_circuit(main_name, params, hcreate, true, opt_level);
    RowPlan R;
    R.opt_level = opt_level; R.n_wires = P.n_signals; R.n_labels = P.n_signals_o0; R.n_outputs = P.n_outputs; R.n_inputs = P.n_inputs;
    R.konst = P.cons_konst;
    std::unordered_map<std::array<uint32_t, 8>, uint32_t, FrHash> kix;         // the emitter's constant dedupe, seeded with its table
    for (size_t i = 0; i < R.konst.size(); i++) { std::array<uint32_t, 8> key; memcpy(key.data(), R.konst[i].l, 32); kix.emplace(key, (uint32_t)i); }
    ConsSink fs; fs.S = &R.flat; fs.konst = &R.konst; fs.kix = &kix;
    if (!opt_level) {
        ConsSink rs; rs.S = &R.round; rs.konst = &R.konst; rs.kix = &kix;
        plan_o0_set(P.cons_flat, fs, false);
        plan_o0_set(P.cons_round, rs, true);
        R.bases = P.round_block_sig;
        R.n_terms = plan_set_terms(R.flat, R.konst, false, 0);
        uint64_t per_round[24];
        for (int r = 0; r < 24; r++) per_round[r] = plan_set_terms(R.round, R.konst, true, keccak_rc(r));
        for (size_t b = 0; b < R.bases.size(); b++) R.n_terms += per_round[b % 24];
        uint64_t nl_flat = 0, nl_round = 0;
        for (const ConsR1 &r : R.flat.r1) nl_flat += r.na != 0;
        for (const ConsR1 &r : R.round.r1) nl_round += r.na != 0;
        R.n_nonlinear = nl_flat + R.bases.size() * nl_round;
        return R;
    }
    // --O1: substitute the equality classes of the reduction into the --O0 rows, in the same order.  A term on a signal moves to its
    // class representative (kept, so it has a reduced wire) or, in a constant class, becomes coef * value on wire 0; eq and kc
    // records thereby become empty.  A main input / output that is not its class's representative keeps one row, s - rep (or
    // s - k w0), at its first eq / kc record, so that its own wire stays constrained.
    const uint64_t N = P.n_signals_o0, n_io = 1ull + P.n_outputs + P.n_inputs;
    EqClasses E = eq_classes(P, N);
    std::vector<uint32_t> red(N, NONE_IDX);
    for (size_t k = 0; k < P.witness_map.size(); k++) red[P.witness_map[k]] = (uint32_t)k;
    std::unordered_map<uint32_t, Fr> cval;                                     // value of every constant class, by representative
    auto set_val = [&](uint32_t s, const Fr &v) {
        const uint32_t r = E.root(s);
        auto it = cval.find(r);
        if (it == cval.end()) cval.emplace(r, v);
        else if (!fr_eq(it->second, v)) throw std::runtime_error("pob: internal: two constants disagree in one equality class (signal " + std::to_string(s) + ")");
    };
    set_val(0, fr_from_u64(1));
    for (const ConsTerm &t : P.cons_flat.kc) set_val(t.idx, cons_coef_value(t.coef, P.cons_konst.data(), 0));
    for (size_t b = 0; b < P.round_block_sig.size(); b++)
        for (const ConsTerm &t : P.cons_round.kc) set_val((uint32_t)(P.round_block_sig[b] + t.idx), cons_coef_value(t.coef, P.cons_konst.data(), keccak_rc((int)(b % 24))));
    auto subst = [&](LC &L, uint32_t s, const Fr &c) {
        const uint32_t r = E.root(s);
        if (E.is_const_root[r]) {
            auto it = cval.find(r);
            if (it == cval.end()) throw std::runtime_error("pob: internal: constant class without a value");
            L.sf(0, fr_mul(c, it->second));
        } else {
            if (red[r] == NONE_IDX) throw std::runtime_error("pob: internal: class representative is not a reduced-witness entry");
            L.sf(red[r], c);
        }
    };
    auto subst_lc = [&](const ConsTerm *t, uint32_t n, uint64_t base) {
        LC L;
        for (uint32_t i = 0; i < n; i++) {
            const Fr c = cons_coef_value(t[i].coef, P.cons_konst.data(), 0);
            if (t[i].idx == CONS_ONE) L.sf(0, c); else subst(L, (uint32_t)(base + t[i].idx), c);
        }
        return L;
    };
    std::vector<uint8_t> io_done(n_io, 0);
    auto io_row = [&](uint32_t s) {
        if (s == 0 || s >= n_io || io_done[s]) return;
        io_done[s] = 1;
        const uint32_t r = E.root(s);
        if (r == s && !E.is_const_root[r]) return;                              // its own representative: terms already land on it
        LC A, Bq, C; C.sf(red[s], fr_from_u64(1)); subst(C, s, fr_neg(fr_from_u64(1)));
        plan_r1(fs, A, Bq, C, false);
    };
    for (size_t i = 0; i + 1 < P.cons_flat.eq.size(); i += 2) { io_row(P.cons_flat.eq[i]); io_row(P.cons_flat.eq[i + 1]); }
    for (const ConsTerm &t : P.cons_flat.kc) io_row(t.idx);
    auto r1_rows = [&](const ConsSet &S, uint64_t base) {
        for (const ConsR1 &r : S.r1) {
            if (r1_hint(r)) continue;
            const ConsTerm *t = S.terms.data() + r.off;
            LC A = subst_lc(t, r.na, base), Bq = subst_lc(t + r.na, r.nb, base), C = subst_lc(t + r.na + r.nb, r1_nc(r), base);
            plan_r1(fs, A, Bq, C, false);
        }
    };
    r1_rows(P.cons_flat, 0);
    for (uint64_t base : P.round_block_sig) r1_rows(P.cons_round, base);
    R.witness_map = std::move(P.witness_map);
    R.n_terms = plan_set_terms(R.flat, R.konst, false, 0);
    for (const ConsR1 &r : R.flat.r1) R.n_nonlinear += r.na != 0;
    return R;
}

uint64_t RowPlan::file_bytes() const {
    // magic, version, nSections; 3 section headers; header content; per row 3 term counts, per term wire + coefficient; labels
    return 12 + 3 * 12 + 64 + 12 * n_rows() + 36 * n_terms + 8 * n_wires;
}

// Component list of a circuit shape in numbering order: one line `first_signal,n_own_signals,template` per component instance
// (KeccakfRound blocks expanded from the shared walk).  tools/diff_sym.py compares it with the component structure of a real
// circom `.sym` (SURVEY.md Appendix C: the only way to pin the ORDER the reference leaves unpinned).
uint64_t write_components(const std::string &main_name, const std::vector<Fr> &params, bool hcreate, const std::string &path) {
    int np = 0; const char *schema = main_input_schema(main_name, &np);
    if (!schema) throw std::runtime_error("pob: unknown main template '" + main_name + "'");
    if ((int)params.size() < np) throw std::runtime_error("pob: too few template parameters for " + main_name);
    size_t n_in = count_inputs(schema, params);
    uint32_t n_out = 0, n_words;
    { Builder dry(hcreate, true, 0); build(dry, main_name, params, n_in, &n_out); n_words = dry.n_words; }
    Builder B(hcreate, false, (n_words + 3u) & ~3u);
    std::vector<Builder::Comp> comps; B.comps = &comps;
    build(B, main_name, params, n_in, &n_out);
    ConsSet dummy; std::vector<Fr> dk; std::unordered_map<std::array<uint32_t, 8>, uint32_t, FrHash> dix;
    ConsSink rs; rs.S = &dummy; rs.konst = &dk; rs.kix = &dix;
    std::vector<RelComp> rel; RoundCons rc{rs}; rc.comps = &rel; rc.round();
    FILE *f = fopen(path.c_str(), "w");
    if (!f) throw std::runtime_error("pob: cannot open " + path);
    fprintf(f, "# pob_b200 component list: %s hcreate=%d n_signals=%llu\n# first_signal,n_own_signals,template\n", main_name.c_str(), hcreate ? 1 : 0, (unsigned long long)B.nsig);
    uint64_t n = 0;
    for (const Builder::Comp &c : comps) {
        if (c.n == ROUND_SIGNALS && strcmp(c.tmpl, "KeccakfRound*") == 0) { for (const RelComp &r : rel) { fprintf(f, "%llu,%u,%s\n", (unsigned long long)(c.sig + r.off), r.n, r.tmpl); n++; } }
        else { fprintf(f, "%llu,%llu,%s\n", (unsigned long long)c.sig, (unsigned long long)c.n, c.tmpl); n++; }
    }
    if (fclose(f) != 0) throw std::runtime_error("pob: short write to " + path);
    return n;
}

std::vector<Fr> build_inverse_table() {
    const uint32_t N = 1u << 16;
    std::vector<Fr> inv(N), pre(N);
    Fr acc = fr_from_u64(1);
    for (uint32_t i = 1; i < N; i++) { pre[i] = acc; acc = fr_mul(acc, fr_from_u64(i)); }
    Fr ai = fr_inv(acc);
    for (uint32_t i = N - 1; i >= 1; i--) { inv[i] = fr_mul(ai, pre[i]); ai = fr_mul(ai, fr_from_u64(i)); }
    inv[0] = fr_zero();
    return inv;
}

}  // namespace pob
