// program.h -- the compiled witness program: what the layout compiler (compiler.cpp, host, once per
// circuit shape) hands to the GPU kernels (kernels.cu, once per proof instance).
//
// Design ("evaluate small, materialise big").  A circom --O0 witness for main_proof_of_burn is 215.9 M field
// elements (6.9 GB) but only ~0.6 M of them are distinct computed values; the rest are copies, constants and
// single bits of 64-bit Keccak lane words.  So one instance is processed in two stages:
//   1. EVAL  -- a levelised straight-line program over a compact per-instance STORE (u64 words):
//        lane-word region  W[0 .. n_words)          Keccak lanes, packed input blocks
//        value region      V[slot] = 4 x u64         canonical BN254-Fr values (inputs first)
//      thread ops (FMA over Fr, IsZero, inverse, integer div/mod, byte packing, constraint checks) and
//      warp ops (one Keccak absorb = block XOR + 24 rounds, emitting every intermediate lane word).
//   2. EXPAND -- every witness entry is described by one 32-bit operand CODE (constant, bit of a store word,
//      store value, table constant); the expand kernel turns codes into 32-byte little-endian field
//      elements and streams them to HBM.  All 2016 KeccakfRound blocks (102,656 signals each, 95.8 % of the
//      witness) share ONE code table, addressed relative to the round's word base.
#pragma once
#include <stdint.h>
#include <string>
#include <vector>
#include "fr_hd.h"

namespace pob {

// ---- operand / witness codes --------------------------------------------------------------------------------
typedef uint32_t Code;
enum : uint32_t { K_CONST = 0, K_BIT = 1, K_VAL = 2, K_KONST = 3 };
POB_HD uint32_t code_kind(Code c) { return c >> 30; }
POB_HD uint32_t code_payload(Code c) { return c & 0x3fffffffu; }
POB_HD Code c_const(uint32_t v) { return v; }                                    // v < 2^30
POB_HD Code c_bit(uint32_t u64idx, uint32_t bit) { return (1u << 30) | (u64idx << 6) | bit; }   // u64idx < 2^24
POB_HD Code c_val(uint32_t slot) { return (2u << 30) | slot; }
POB_HD Code c_konst(uint32_t idx) { return (3u << 30) | idx; }
static const uint32_t MAX_STORE_U64 = 1u << 24;                                  // 128 MiB per instance store

// ---- thread ops ---------------------------------------------------------------------------------------------
enum Opc : uint32_t {
    OP_FMA = 1,        // V[dst] = a*b + c
    OP_ISZ = 2,        // V[dst] = (a == 0)                       comparators.circom:24-35 (out)
    OP_INV = 3,        // V[dst] = a != 0 ? 1/a : 0               comparators.circom:30 (hint)
    OP_DIV = 4,        // V[dst] = a \ b   (integer)              utils/divide.circom:23 ; c = raw component base
    OP_MOD = 5,        // V[dst] = a % b   (integer)              utils/divide.circom:24
    OP_PACK8 = 6,      // W[dst] = sum_k (aux[a+k] & 0xff) << 8k  utils/keccak.circom:467-482 (bytes -> lane)
    OP_CHK_EQ = 7,     // a == b else fail(c)                     any `===`
    OP_CHK_RANGE = 8,  // a < 2^b else fail(c)                    bitify.circom:38 (Num2Bits sum check)
    // closed forms of the circuits' one-hot prefix patterns (identical values, no dependency chain):
    OP_GTC = 9,        // V[dst] = (a > b) as canonical integers, b raw u32.  prod_{j<=i}(1 - IsEqual(j, a)) == (a > i):
                       //   utils/keccak.circom:427-433 (Pad filter), array.circom:26-40 (Filter), substring_check.circom:87-88
    OP_SELSUM = 10,    // V[dst] = (a <= c) ? aux[b + a] : 0, b/c raw.  sum_{j<=c} IsEqual(a, j)*vals[j]: selector.circom:31-41
};
struct Op { uint32_t opc_dst; Code a, b, c; };                    // opc in the top 6 bits, dst in the low 26
POB_HD uint32_t op_opc(const Op &o) { return o.opc_dst >> 26; }
POB_HD uint32_t op_dst(const Op &o) { return o.opc_dst & 0x3ffffffu; }

// ---- warp op: one Absorb (utils/keccak.circom:304-323) = 17-lane XOR + Keccakf (24 KeccakfRound) -------------
// Word layout written at W[out .. out + ABSORB_WORDS):
//   out + 0..24                       aux[25]  (= s ^ block on the 17 rate lanes)
//   round r base  rb = out + RW*r     rb+0..24 is the round INPUT (aux, or the previous round's OUT)
//     rb + X5(i,k)  i<5,k<4   Xor5 chain of column i: xor_ab, xor_abc, xor_abcd, c[i]       keccak.circom:58-70
//     rb + DD(i,k)  i<5,k<4   D: c<<1, c>>63, or, d[i]                                        :135-144
//     rb + TH(l)    l<25      Theta out                                                       :151-170
//     rb + RP(i,k)  i<24,k<3  stepRhoPi i: a>>shr, a<<shl, or                                 :177-204
//     rb + CH(l,k)  l<25,k<3  stepChi of lane l: ~b, ~b&c, a^(~b&c)                           :212-241
//     rb + RCW                round-constant word                                             :248-266
//     rb + OUT(l)   l<25      Iota out = round output                                         :273-283
static const uint32_t NONE_IDX = 0xffffffffu;
struct AbsorbOp { uint32_t s_idx, blk_idx, out_idx, pad; };       // s_idx == NONE_IDX: all-zero state
enum : uint32_t { RW = 238, RW_X5 = 25, RW_DD = 45, RW_TH = 65, RW_RP = 90, RW_CH = 162, RW_RC = 237, RW_OUT = 238,
                  ROUND_WORDS_SPAN = 263, ABSORB_WORDS = 25 + 24 * 238, ROUND_SIGNALS = 102656 };
POB_HD uint32_t rw_x5(int i, int k) { return RW_X5 + 4 * i + k; }
POB_HD uint32_t rw_dd(int i, int k) { return RW_DD + 4 * i + k; }
POB_HD uint32_t rw_th(int l) { return RW_TH + l; }
POB_HD uint32_t rw_rp(int i, int k) { return RW_RP + 3 * i + k; }
POB_HD uint32_t rw_ch(int l, int k) { return RW_CH + 3 * l + k; }
POB_HD uint32_t rw_out(int l) { return RW_OUT + l; }

// ---- warp op: one Poseidon permutation (circomlib/circuits/poseidon.circom:67-196, optimised schedule) ----------
// Lane j < t owns state element j (Montgomery form); every intermediate signal the circuit exposes is written, in
// canonical form, to a block of value slots laid out in computation order:
//   0 .. t-1                         ark[0].out
//   F1 + 5t*f, f = 0..3              first-half full round f: sigma j -> (in2, in4, out) at +3j ; ark.out at +3t ; mix.out at +4t
//   PB + (4+t)*r, r = 0..RP-1        partial round r: sigma (in2, in4, out), mixS.in[0] (= out + C), mixS.out[t]
//   SB + 5t*f, f = 0..2              second-half full rounds (same shape)
//   LB                               last sigmas (3t), then mixLast.out
// One permutation is cut into POS_SEGMENTS warp ops of consecutive "steps" (step 0 = ark[0]; 1..4 first-half full rounds; then the RP
// partial rounds; 3 second-half full rounds; the last step = final sigmas + mixLast), scheduled in consecutive
// levels: nothing but the last segment's result is consumed, so a 65-round dependency chain (~0.7 M cycles on one warp) no longer
// holds up a whole level while every other warp of the cluster idles -- it proceeds alongside 16 levels of other work.  Between
// segments the state is re-read from the value block (parked there in Montgomery form anyway).
struct PoseidonOp { uint32_t t, in_aux, base, koff, q0, q1; };  // inputs: aux[in_aux .. +t) = initialState, inputs[]; steps [q0, q1)
static const uint32_t POS_SEGMENTS = 16;
struct PosLayout { uint32_t t, rp, F1, PB, SB, LB, total, kC, kS, kM, kP, ktotal; };
POB_HD PosLayout pos_layout(uint32_t t) {
    PosLayout L; L.t = t; L.rp = (t == 3) ? 57u : (t == 4) ? 56u : 60u;
    L.F1 = t; L.PB = 21 * t; L.SB = L.PB + L.rp * (4 + t); L.LB = L.SB + 15 * t; L.total = L.LB + 3 * t + 1;
    L.kC = 0; L.kS = t * 8 + L.rp; L.kM = L.kS + L.rp * (2 * t - 1); L.kP = L.kM + t * t; L.ktotal = L.kP + t * t;
    return L;
}
POB_HD uint32_t pos_steps(const PosLayout &L) { return L.rp + 9; }
// offset (in the value block) of state element 0 after step q (q < steps - 1)
POB_HD uint32_t pos_state_off(const PosLayout &L, uint32_t q) {
    if (q == 0) return 0;
    if (q <= 4) return L.F1 + 5 * L.t * (q - 1) + 4 * L.t;
    if (q < 5 + L.rp) return L.PB + (q - 5) * (4 + L.t) + 4;
    return L.SB + 5 * L.t * (q - 5 - L.rp) + 4 * L.t;
}

// first offset (in the value block) written by step q; step q writes [pos_step_begin(q), pos_step_begin(q + 1))
POB_HD uint32_t pos_step_begin(const PosLayout &L, uint32_t q) {
    if (q == 0) return 0;
    if (q <= 4) return L.F1 + 5 * L.t * (q - 1);
    if (q < 5 + L.rp) return L.PB + (q - 5) * (4 + L.t);
    if (q < L.rp + 8) return L.SB + 5 * L.t * (q - 5 - L.rp);
    return q == L.rp + 8 ? L.LB : L.total;
}

// ---- warp op: prefix sum whose every partial sum is a signal (substring_check.circom:47-49 M[], :95 sums[]) -------
//   V[dst + k] = x0 + sum_{i <= k} aux[aux0 + i]      (k < n); lanes own contiguous ranges, totals combined by a warp scan
struct PsumOp { uint32_t aux0, n, dst; Code x0; };

struct Level { uint32_t t_begin, t_end, w_begin, w_end, p_begin, p_end, s_begin, s_end; };

// ---- expand tiles: a contiguous run of witness entries and where its codes live -------------------------------
struct Tile { uint64_t dst; uint32_t n, code_off, ubase, pad; };  // BIT codes are relative to ubase; pad = 1: round tile (all BIT)
static const uint32_t TILE_SIGNALS = 8192;
// entries per tile of the O0 layout (128 KiB of witness).  Resident k_expand_round CTAs write neighbouring tiles, so smaller
// tiles keep the write front narrower: 4096 made the round tiles 4 % faster than 8192 on compressible slots (DESIGN.md §2.3)
static const uint32_t LAYOUT_TILE_SIGNALS = 4096;
static const uint32_t MAX_TILE_SIGNALS = 32768;  // upper bound for the POB_TILE_SIGNALS tuning knob

// ---- constraint system of the circuit (SURVEY.md 8(f) rank 4: on-GPU self-check; rank 2: reduced witness map) -------
// Written from the circom sources statement by statement (every `<==` / `===` of the include closure), over WITNESS
// INDICES -- independent of the codes/ops that produce the witness values.  Three record kinds:
//   eq   : s[a] == s[b]                                       (`x <== y` between two signals -- the vast majority)
//   kc   : s[a] == constant                                   (`x <== 5`, RoundConstants bits)
//   r1   : (sum A_i s_i) * (sum B_i s_i) == (sum C_i s_i)     (everything else; no A/B terms: a linear constraint)
// Index 0 is witness[0] = 1 (constant terms), as in an .r1cs.  `hint` records are not constraints of the circuit: they
// pin signals the circuit itself leaves free (`inv <-- in != 0 ? 1/in : 0`, comparators.circom:30; the unassigned
// `temp[]` of merkle_patricia_trie_leaf.circom:76) to the values the reference calculator writes.
// Coefficients: top two bits 0 = +small (30 bits), 1 = -small, 2 = index into Program::cons_konst, 3 = bit k of the
// Keccak round constant of the block's round (only in the shared KeccakfRound set).
struct ConsTerm { uint32_t idx, coef; };
enum : uint32_t { CC_POS = 0, CC_NEG = 1, CC_KONST = 2, CC_RCBIT = 3 };
POB_HD uint32_t cc_kind(uint32_t c) { return c >> 30; }
POB_HD uint32_t cc_payload(uint32_t c) { return c & 0x3fffffffu; }
struct ConsR1 { uint32_t off; uint16_t nc_hint; uint8_t na, nb; };   // terms[off .. off+na) = A, then B, then C (nc = low 15 bits; bit 15 = hint)
POB_HD uint32_t r1_nc(const ConsR1 &r) { return r.nc_hint & 0x7fffu; }
POB_HD bool r1_hint(const ConsR1 &r) { return (r.nc_hint >> 15) != 0; }
struct ConsSet {
    std::vector<uint32_t> eq;          // 2 per record
    std::vector<ConsTerm> kc;          // s[idx] == coef
    std::vector<ConsR1> r1;
    std::vector<ConsTerm> terms;
    uint64_t n_records() const { return eq.size() / 2 + kc.size() + r1.size(); }
};

struct Program {
    // identity
    std::string main_name;
    std::vector<Fr> params;
    bool hcreate = false;
    // witness shape
    uint64_t n_signals = 0;        // including witness[0] = 1
    uint32_t n_outputs = 0, n_inputs = 0;
    std::string input_schema;      // "name[d0][d1],name2,..." in declaration order
    // store shape
    uint32_t n_words = 0;          // lane-word region size (u64)
    uint32_t val_base = 0;         // u64 index of V[0] (multiple of 4)
    uint32_t n_vals = 0;           // value slots (inputs are slots 0..n_inputs-1)
    uint64_t store_u64() const { return (uint64_t)val_base + 4ull * n_vals; }
    // eval program
    std::vector<Op> ops;           // [0, inv_begin) sorted by level, then the deferred OP_INV ops
    uint32_t inv_begin = 0, ginv_begin = 0, inv_end = 0;   // [ginv_begin, inv_end): the DEFERRED IsZero inverses (expected to need a real
                                   // inversion): batch-inverted per worker thread; inv_begin == ginv_begin (kept for the emulator)
    uint32_t ginv_level = 0xffffffffu;   // index of the first level that starts with all their inputs ready (== levels.size(): none)
    std::vector<AbsorbOp> absorbs; // sorted by level
    std::vector<PoseidonOp> poseidons;   // sorted by level
    std::vector<PsumOp> psums;     // sorted by level
    std::vector<Fr> pos_konst;     // Poseidon C,S,M,P tables per width, MONTGOMERY form (PoseidonOp::koff)
    std::vector<Level> levels;
    std::vector<Code> aux;         // PACK8 operand lists
    std::vector<Fr> konst;         // big constants
    // expand program
    std::vector<Code> codes;       // [0, ROUND_SIGNALS) = shared KeccakfRound table, then flat codes
    std::vector<Tile> tiles;
    // compact form of the shared KeccakfRound table: one 8-byte descriptor per 64 consecutive signals
    //   bits 0-15 w0, 16-31 w1, 32-47 w2 (lane words relative to the round base), 48-63 mode:
    //   mode 0: a lane -- signal t is bit t of w0;  mode 1+f: 64-signal phase f of a 192-signal gate block
    //   [out_i, a_i, b_i]_i -- signal s = 64 f + t is bit s/3 of w_{s%3}
    std::vector<uint64_t> round_desc;
    // constraint system (only when compiled with want_constraints): flat part over absolute witness indices, the shared
    // KeccakfRound set over indices relative to a round block's first signal; round_block_sig[i] = first signal of block i
    // (blocks are emitted 24 per Keccakf, in round order: round = i % 24)
    bool has_constraints = false;
    ConsSet cons_flat, cons_round;
    std::vector<Fr> cons_konst;
    std::vector<uint64_t> round_block_sig;
    // reduced (`--O1`-style) witness: opt_level 1 drops every signal that a `signal = signal` or `signal = constant`
    // constraint of the circuit ties to an earlier signal / a constant (main inputs and outputs always stay); the
    // retained signals keep their --O0 order.  n_signals / codes / tiles then describe the REDUCED vector;
    // n_signals_o0 is the full count and witness_map[k] the --O0 index of reduced entry k (SURVEY.md 8(f) rank 2).
    int opt_level = 0;
    uint64_t n_signals_o0 = 0;
    std::vector<uint32_t> witness_map;
    uint32_t out_code_off = ROUND_SIGNALS + 1;   // position in `codes` of the code of witness[1] (the first output)
    // statistics
    uint64_t n_round_blocks = 0, n_flat_signals = 0;
};

}  // namespace pob
