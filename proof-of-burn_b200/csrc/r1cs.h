// r1cs.h -- the R1CS rows of a circuit shape in `.r1cs` order (the row plan), and the iden3 `.r1cs` writer.
//
// The row plan is the one place that fixes the row order; the file writer (r1cs.cpp) and the GPU (pob_r1cs_check,
// k_r1cs_products) both consume it.  It keeps the self-check's flat-set + round-set + block-bases form, so row k is record k of
//   flat.eq, flat.kc, flat.r1, then for every round block b (in round_block_sig order) round.eq, round.kc, round.r1
// with record ids == row indices: hint records and records whose three linear combinations are empty after merging are left out.
// Row form:  eq (a, b): A = B = 0, C = w[a] - w[b];  kc (a, k): A = B = 0, C = w[a] - k w0 (CC_RCBIT: the bit of round b % 24);
//            r1: A, B, C as stored, B empty when A is.  Inside a combination terms are merged by wire, zero coefficients dropped,
//            and sorted by ascending wire (CONS_ONE = wire 0 first).
// --O1 plan: wires are reduced-witness indices; every row is an r1 record of `flat` (absolute indices, no round set), see
// build_row_plan in compiler.cpp.
#pragma once
#include <stdexcept>
#include <string>
#include <vector>
#include "cons_check.h"

namespace pob {

struct RowPlan {
    int opt_level = 0;
    uint64_t n_wires = 0, n_labels = 0;           // nWires (== witness entries of the form), nLabels (== --O0 signals)
    uint32_t n_outputs = 0, n_inputs = 0;
    ConsSet flat, round;
    std::vector<uint64_t> bases;                  // first --O0 signal of every round block (empty in the --O1 plan)
    std::vector<Fr> konst;                        // CC_KONST coefficients
    std::vector<uint32_t> witness_map;            // --O1: label (--O0 signal id) of every wire
    uint64_t n_nonlinear = 0, n_terms = 0;        // rows with a non-empty A; A + B + C terms over all rows
    uint64_t n_rows() const { return flat.n_records() + bases.size() * round.n_records(); }
    uint64_t file_bytes() const;                  // size of the `.r1cs` the writer produces
};

// compile the circuit with its constraint system and derive its rows; opt_level 1 = the reduced (POB_CREATE_O1) witness
RowPlan build_row_plan(const std::string &main_name, const std::vector<Fr> &params, bool hcreate, int opt_level);

struct R1csIoError : std::runtime_error { using std::runtime_error::runtime_error; };
// stream the iden3 `.r1cs` (version 1: header, constraints, wire-to-label map) to path through a buffer, never holding the file in
// memory; throws R1csIoError when the file cannot be opened or a write comes up short.  Returns the bytes written (== file_bytes()).
uint64_t write_r1cs(const RowPlan &plan, const std::string &path);

}  // namespace pob
