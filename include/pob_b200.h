/* pob_b200.h -- C ABI of the H100-native batched witness generator for worm-privacy/proof-of-burn.
 *
 * Drop-in boundary.  The reference has no library interface for this path: witness generation is the
 * process CLI the circom toolchain emits, `./<circuit> input.json witness.wtns`
 * (reference Makefile:5-6, tests/test.py:60-63), with the circuit identity fixed at compile time by
 * `component main = ...` (circuits/main_proof_of_burn.circom:27, circuits/main_spend.circom:6).  The entry
 * points below are what an FFI for that path binds: fix a circuit shape once (pob_create == `circom -c` +
 * `make`), then push batches of inputs through it (pob_run_batch == N runs of `./<circuit>`), and read back
 * per-instance accept/reject + output signals, optionally a full `.wtns`.  Plain pointers and sizes only.
 *
 * Field elements cross the ABI as 4 x uint64 little-endian limbs, canonical (< p, non-Montgomery): the same
 * 32-byte form the .wtns file stores.  JSON parsing (the schema tests/main.py:160-178 emits) lives in the
 * Python host (proof-of-burn_b200/pob_b200), which flattens inputs in declaration order
 * (circuits/proof_of_burn.circom:43-72, circuits/spend.circom:33-36).
 *
 * Errors: every function returns 0 on success and a negative POB_E_* code otherwise; pob_last_error()
 * returns a message for the calling thread.  There is NO CPU fallback: without a CUDA device pob_create
 * fails with POB_E_NO_DEVICE.  A failed circuit constraint is not an API error: it is reported per
 * instance in status[] (reference: any failed `===` aborts the calculator, tests/test.py:65-68).
 */
#ifndef POB_B200_H
#define POB_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct pob_handle pob_handle;

enum {
    POB_OK = 0,
    POB_E_BAD_ARG = -1,       /* null pointer, unknown template, wrong parameter count, n == 0 ... */
    POB_E_NO_DEVICE = -2,     /* no CUDA device / device index out of range */
    POB_E_CUDA = -3,          /* a CUDA runtime call failed (message in pob_last_error) */
    POB_E_NO_MEMORY = -4,     /* not even one witness slot fits in free HBM */
    POB_E_RANGE = -5,         /* instance index not resident / offset out of range */
    POB_E_IO = -6,            /* file write failed */
    POB_E_COMPILE = -7,       /* the layout compiler rejected the circuit shape */
    POB_E_REJECTED = -8,      /* the instance failed a circuit constraint: it has no witness (reference tests/test.py:65-68) */
    POB_E_BUSY = -9,          /* every witness slot is held by the consumer: release one first / a batch is in flight */
    POB_E_KEY = -10,          /* a .zkey is malformed, does not fit the circuit, or fails its check (pob_zkey_info / pob_zkey_load) */
    POB_DONE = 1              /* pob_acquire: no further witness in this batch (not an error) */
};

/* flags for pob_run_batch */
enum {
    POB_RUN_EXPAND = 1u,          /* materialise every instance's full witness vector in its HBM slot */
    POB_RUN_DIGEST = 2u,          /* also compute a 64-bit digest of each materialised witness (reads it back once) */
    POB_RUN_INPUTS_STAGED = 4u,   /* ignore `inputs`, use the device-resident batch set by pob_stage_inputs */
    POB_RUN_DISCARD = 8u          /* generation-only run: with n > n_slots earlier witnesses are overwritten UNREAD by later
                                     ones (throughput measurement of the path itself).  Without this flag, a digest or a
                                     retain list, pob_run_batch refuses n > n_slots: use pob_submit/pob_acquire/pob_release. */
};

typedef struct {
    uint64_t n_signals;        /* witness entries incl. witness[0] = 1 (== nWitness in the .wtns header) */
    uint32_t n_outputs;        /* main output signals = witness[1 .. n_outputs] */
    uint32_t n_inputs;         /* scalar input signals in declaration order */
    uint64_t witness_bytes;    /* 32 * n_signals */
    uint64_t wtns_file_bytes;  /* 76 + 32 * n_signals */
    uint64_t store_bytes;      /* compact per-instance evaluation store */
    uint64_t n_ops;            /* thread ops per instance */
    uint32_t n_absorbs;        /* Keccak absorbs (= Keccak-f permutations) per instance */
    uint32_t n_levels;         /* dependency levels of the eval program */
    uint32_t n_tiles;          /* expand tiles per instance */
    uint32_t n_slots;          /* witness slots resident in HBM (0 when no device handle) */
    uint32_t chunk;            /* instances evaluated per eval launch */
    uint32_t expand_group;     /* instances materialised per expand launch (<= n_slots) */
    uint32_t opt_level;        /* 0 = circom --O0 witness (every signal), 1 = reduced witness (POB_CREATE_O1) */
    uint64_t n_signals_o0;     /* witness entries of the --O0 layout (== n_signals when opt_level == 0) */
    uint32_t n_compressed_slots; /* of the n_slots, those the driver made compressible memory (Compute Data Compression) */
} pob_desc;

/* `hcreate` argument of pob_create / pob_layout_info / pob_constraint_info: bit 0 = creation-order sub-component numbering
 * (SURVEY.md App. C R3), POB_CREATE_O1 = produce the REDUCED witness the circom simplifier's `--O1` level implies (the reference
 * deploys through circom's default simplifier: .github/workflows/circuitscan.yml:29,36; its Makefile builds --O0): every signal
 * tied to an earlier signal or to a constant by a `signal = signal` / `signal = constant` constraint is dropped, main inputs and
 * outputs always stay, the rest keeps its --O0 order.  main_proof_of_burn: 215,907,954 -> see pob_desc.n_signals.  Which member
 * of an equality class circom itself keeps is not pinned by the reference: the reduced ORDER is "parity unpinned" like the
 * --O0 order; every retained value equals the --O0 witness through pob_witness_map (tested). */
enum { POB_CREATE_HCREATE = 1, POB_CREATE_O1 = 0x100 };

/* replaces: `circom -c <main>.circom --O0 && make` (reference Makefile:2-3, tests/test.py:32,55).
 * main_name/params = the `component main = Name(p0, p1, ...)` expression; params are nparams x 4 limbs.
 * hcreate: 0 = completion-order sub-component numbering (default), 1 = creation order (SURVEY.md App. C R3).
 * max_slots: upper bound on resident witness slots (0 = as many as fit in 80 % of free HBM). */
int pob_create(const char *main_name, const uint64_t *params, int nparams, int hcreate, int device,
               uint32_t max_slots, pob_handle **out);
void pob_destroy(pob_handle *h);

/* host-only: run the layout compiler and report the shape; needs no GPU (used by the CPU test-suite) */
int pob_layout_info(const char *main_name, const uint64_t *params, int nparams, int hcreate, pob_desc *out);
/* input schema "name[d0][d1],name2,..." with dims as expressions over p0..p7; NULL if unknown template */
const char *pob_input_schema(const char *main_name, int *nparams);

/* host-only, order-pinning kit (the reference pins no witness ORDER: it holds no .sym / .wtns; SURVEY.md Appendix C).  Writes
 * one line `first_signal,n_own_signals,template` per component instance of the --O0 layout, in numbering order, for
 * tools/diff_sym.py to compare with the `.sym` of a real `circom --O0 --sym` build.  *n_components receives the line count. */
int pob_write_components(const char *main_name, const uint64_t *params, int nparams, int hcreate, const char *path, uint64_t *n_components);

int pob_describe(const pob_handle *h, pob_desc *out);
/* reduced witness only: map[k] = --O0 signal index of reduced witness entry k (n_signals entries) */
int pob_witness_map(const pob_handle *h, uint32_t *map);

/* pinned host memory for the caller's input / output arrays (so H2D/D2H inside pob_run_batch are async DMA) */
void *pob_alloc_pinned(uint64_t bytes);
void pob_free_pinned(void *p);

/* copy a batch of inputs (n x n_inputs x 4 limbs) to HBM once; later runs with POB_RUN_INPUTS_STAGED reuse it */
int pob_stage_inputs(pob_handle *h, const uint64_t *inputs, uint32_t n);

/* replaces: n runs of `./<circuit> input.json witness.wtns` (reference Makefile:5-6, tests/test.py:60-63).
 * inputs : n x n_inputs x 4 limbs (host; pinned preferred), flattened in declaration order.
 * status : n x uint32 out; 0 = every constraint holds, else 1 + witness index of the first signal of the
 *          lowest-numbered component that owns a failing constraint.
 * outputs: n x n_outputs x 4 limbs out (may be NULL).
 * digests: n x uint64 out, only with POB_RUN_DIGEST (may be NULL otherwise); 0 for a rejected instance.
 * A rejected instance (status != 0) contributes NO witness: its slot is not written and every accessor below
 * answers POB_E_REJECTED for it (the reference calculator aborts without a usable witness, tests/test.py:65-68).
 * With POB_RUN_EXPAND instance i lives in slot i % n_slots.  n > n_slots is only accepted together with
 * POB_RUN_DIGEST (every witness is consumed by the digest kernel before its slot is reused) or POB_RUN_DISCARD;
 * afterwards the last n_slots instances are resident. */
int pob_run_batch(pob_handle *h, const uint64_t *inputs, uint32_t n, uint32_t flags,
                  uint32_t *status, uint64_t *outputs, uint64_t *digests);
/* the same, but only the instances retain[0..n_retain) (strictly ascending, n_retain <= n_slots) are materialised:
 * all n instances are evaluated (status, outputs), the retained ones stay resident, the others cost no HBM traffic
 * (SURVEY.md 8(b) "which indices to retain"). */
int pob_run_batch_retain(pob_handle *h, const uint64_t *inputs, uint32_t n, uint32_t flags,
                         const uint32_t *retain, uint32_t n_retain,
                         uint32_t *status, uint64_t *outputs, uint64_t *digests);

/* ---- consumer-paced hand-off (SURVEY.md 8(f) rank 1): no witness is ever overwritten unread ----------------------
 * The reference's contract is one run -> one witness.wtns the prover reads (Makefile:5-6).  Here the consumer (an
 * on-GPU prover stage, an exporter) takes the witnesses of a batch one by one, in instance order, and hands each
 * slot back when it is done; generation stalls -- on the GPU, stream-ordered -- while all slots are held.
 *   pob_submit   start a batch (POB_RUN_EXPAND implied); returns at once, work is queued as slots allow.
 *   pob_acquire  next instance: POB_OK (*index, *dptr = its resident witness), POB_E_REJECTED (*index set, no witness,
 *                nothing to release), POB_DONE (batch exhausted), POB_E_BUSY (release a slot first).
 *                consumer_stream == NULL: returns when the witness is complete in HBM (host wait);
 *                else (a cudaStream_t): returns at once and makes that stream wait for the witness on the GPU.
 *   pob_release  the consumer is done with instance `index`; consumer_stream (or NULL = already finished on the
 *                host) orders the reuse of the slot after the consumer's queued work -- also when the reuse comes
 *                from a later pob_submit / pob_run_batch / pob_export_batch on this handle.
 *   pob_finish   drain the batch (instances never acquired are generated and dropped), return status/outputs/digests.
 *                A witness still held counts as released on the stream it was acquired on: its slot is reused only
 *                after that stream's queued work, so that stream must stay valid until pob_finish returns (a witness
 *                acquired with NULL is taken as read already).
 * The host accessors below (pob_copy_witness, pob_write_wtns, pob_witness_device_ptr, the self-checks, and the row
 * products / quotient with a NULL stream) wait on the host for a held witness that was acquired on a stream and is
 * still being generated; given a stream, pob_r1cs_products / pob_r1cs_quotient make that stream wait for it instead.
 * One batch at a time per handle; the last n_slots non-released instances stay resident after pob_finish. */
int pob_submit(pob_handle *h, const uint64_t *inputs, uint32_t n, uint32_t flags);
int pob_acquire(pob_handle *h, uint32_t *index, void **dptr, void *consumer_stream);
int pob_release(pob_handle *h, uint32_t index, void *consumer_stream);
int pob_finish(pob_handle *h, uint32_t *status, uint64_t *outputs, uint64_t *digests);

/* replaces: n runs of `./<circuit> input_i.json witness_i.wtns` INCLUDING the files: every accepted instance is
 * exported through the consumer-paced path above -- D2H over several copy streams into a pinned staging ring, a writer
 * thread per batch doing the file I/O -- so generation, PCIe transfer and disk writes overlap and no witness is dropped.
 * paths: n entries; NULL entry (or paths == NULL) = transfer to host memory only (PCIe line-rate measurement). */
typedef struct {
    uint64_t witnesses;        /* exported instances */
    uint64_t bytes;            /* .wtns bytes moved to the host */
    float total_ms;            /* wall time of the call */
    float d2h_gbs;             /* bytes / total time */
} pob_export_stats;
int pob_export_batch(pob_handle *h, const uint64_t *inputs, uint32_t n, uint32_t flags, const char *const *paths,
                     uint32_t *status, uint64_t *outputs, pob_export_stats *stats);

/* device timings of the last pob_run_batch (CUDA events on the library's own streams), and kernel count */
typedef struct {
    float total_ms;          /* first H2D / first kernel -> last kernel of the batch */
    float expand_ms;         /* sum of expand-kernel durations */
    float eval_ms;           /* sum of eval-kernel durations */
    uint32_t expand_launches, eval_launches, other_launches;
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t eval_clusters;  /* bit C set: some eval launch of the batch ran C CTAs (a thread-block cluster) per instance */
} pob_timing;
int pob_last_timing(const pob_handle *h, pob_timing *out);

/* replaces: the `witness.wtns` the calculator writes (layout: SURVEY.md Appendix B).  `index` is the
 * instance index within the last batch; it must still be resident. */
int pob_copy_witness(pob_handle *h, uint32_t index, uint64_t first_signal, uint64_t n_signals, uint64_t *dst_host);
int pob_write_wtns(pob_handle *h, uint32_t index, const char *path);
/* device pointer of a resident witness (for an on-GPU consumer such as a prover's first stage) */
int pob_witness_device_ptr(pob_handle *h, uint32_t index, void **dptr);

/* ---- on-GPU self-check of a resident witness (SURVEY.md 8(f) rank 4, Keccak part) -----------------------------------
 * Independent of the layout tables that produced the witness: for every KeccakfRound component (95.8 % of the entries)
 * the kernel reads the component's own `in[25][64]` and `out[25][64]` signals straight from the witness (positions fixed
 * by circuits/utils/keccak.circom:290-297: out first, then in), recomputes one textbook Keccak-f round (theta, rho-pi,
 * chi, iota with the round index the block has inside its Keccakf) and compares; it also checks that all 3200 entries
 * are 0 or 1.  *n_blocks = blocks examined, *n_bad = blocks that fail. */
int pob_selfcheck_keccak(pob_handle *h, uint32_t index, uint64_t *n_blocks, uint64_t *n_bad);

/* ---- full constraint self-check (SURVEY.md 8(f) rank 4) ------------------------------------------------------------------
 * Evaluates EVERY constraint of the circuit against resident witness `index`, on the GPU.  The constraint system is written
 * from the circom sources statement by statement -- every `<==` and `===` of the include closure: the gate equations of
 * circuits/utils/keccak.circom:58-297 (out = a + b - 2ab, ...), circomlib/circuits/poseidon.circom:5-65 (Sigma, Ark, Mix,
 * MixS, MixLast), bitify.circom:33,38 (Num2Bits bits and sum), comparators.circom:32-33 (IsZero), selector.circom:33-45,
 * substring_check.circom:46-99, ... -- over witness INDICES, independently of the program that produced the values.  It
 * reads 100 % of the witness entries.  `hint` records additionally pin the signals the circuit itself leaves free
 * (`inv <-- in != 0 ? 1/in : 0`; the never-assigned temp[] of merkle_patricia_trie_leaf.circom:76) to the values the
 * reference calculator writes.  The first call compiles and uploads the constraint system (seconds for the main shape). */
typedef struct {
    uint64_t n_constraints;     /* circuit constraints evaluated (the shared KeccakfRound set counted once per round block) */
    uint64_t n_nonlinear;       /* of those, A*B = C records with a non-empty A (an .r1cs would call them non-linear) */
    uint64_t n_hints;           /* hint records evaluated */
    uint64_t n_failed;          /* failing circuit constraints */
    uint64_t n_hint_failed;     /* failing hint records */
    uint64_t first_failed;      /* smallest failing record id, UINT64_MAX when everything holds */
    uint64_t signals_read;      /* distinct witness entries referenced by at least one record (== n_signals) */
    float ms;                   /* device time of the check */
} pob_check_report;
int pob_selfcheck(pob_handle *h, uint32_t index, pob_check_report *out);
/* host-only: compile the constraint system of a circuit shape and report its size (no GPU needed) */
int pob_constraint_info(const char *main_name, const uint64_t *params, int nparams, int hcreate, pob_check_report *out);

/* ---- the circuit as an R1CS: the `.r1cs` a prover is set up from, and its rows on the GPU ---------------------------------
 * replaces: the `.r1cs` of `circom --r1cs`.  The rows are the constraint system above in record order -- flat eq, kc, r1 records,
 * then those of the shared KeccakfRound set for every round block -- without the hint records (not constraints of the circuit)
 * and without records whose A, B and C are all empty after merging (the `witness[0] == 1` record).  eq (a, b) is the row
 * 0 * 0 = w[a] - w[b], kc (a, k) is 0 * 0 = w[a] - k w0, an A*B = C record keeps its combinations (B empty when A is); inside a
 * combination terms are merged by wire, zero coefficients dropped, wires ascending.  With POB_CREATE_O1 the wires are the
 * reduced witness entries: every term moves to its equality class's representative or, in a constant class, to wire 0 times the
 * constant; the eq / kc rows vanish, except one row `s - representative` (or `s - k w0`) for each main input / output that is not
 * its class's representative.  The file and the reduced witness agree on the wire order by construction, whatever order circom
 * itself would choose.  n_wires..n_labels are the header fields of the file. */
typedef struct {
    uint64_t n_wires;          /* == pob_desc.n_signals for the same flags */
    uint32_t n_pub_out;        /* n_outputs */
    uint32_t n_pub_in;         /* 0: no main declares public inputs */
    uint32_t n_prv_in;         /* n_inputs */
    uint64_t n_labels;         /* n_signals_o0 (section 3 maps wire -> --O0 signal id: identity for --O0, pob_witness_map for O1) */
    uint64_t n_constraints;    /* rows (mConstraints) */
    uint64_t n_nonlinear;      /* rows with a non-empty A */
    uint64_t n_terms;          /* A + B + C terms over all rows */
    uint64_t file_bytes;       /* size of the .r1cs */
} pob_r1cs_desc;
/* host-only: write the iden3 binary `.r1cs` (version 1; coefficients canonical 32-byte LE, as circom writes them) of a circuit
 * shape; hcreate as in pob_layout_info (bit 0, POB_CREATE_O1).  The file is streamed, never held in memory (a main-shape --O0
 * file is tens of GB).  path == NULL: count only, write nothing.  A failed open or short write is POB_E_IO. */
int pob_write_r1cs(const char *main_name, const uint64_t *params, int nparams, int hcreate, const char *path, pob_r1cs_desc *out);
/* every .r1cs row of the handle's form (O0 or O1) against resident witness `index`; record ids in the report are row indices;
 * n_hints / n_hint_failed are 0, signals_read = wires referenced.  The first call builds and uploads the row plan. */
int pob_r1cs_check(pob_handle *h, uint32_t index, pob_check_report *out);
/* the first stage of a GPU Groth16 prover: rows [first_row, first_row + n_rows) of the .r1cs, a[k], b[k], c[k] = A.w, B.w, C.w of
 * row first_row + k as 32-byte canonical LE field elements (a row's constants multiply w[0], as in the file, so these are the rows'
 * linear forms on any witness), into caller device buffers (any may be NULL: not computed), each
 * 16-byte aligned (else POB_E_BAD_ARG, before anything is enqueued).
 * consumer_stream NULL: returns when done; else (a cudaStream_t) enqueued on that stream, which the caller has ordered after the
 * witness (pob_acquire on it, or a finished pob_run_batch).  first_row + n_rows beyond the row count: POB_E_RANGE. */
int pob_r1cs_products(pob_handle *h, uint32_t index, uint64_t first_row, uint64_t n_rows, void *a, void *b, void *c, void *consumer_stream);

/* ---- the second stage: the Groth16 quotient evaluations (the scalars of the prover's H multi-exponentiation) --------------
 * Follows snarkjs `groth16 prove` as far as it is known; the match with snarkjs / rapidsnark is unverified (INTEGRATION.md §3(e)).
 * Field BN254 Fr, p - 1 = 2^28 t.  w28 = 5^t (5: the smallest quadratic non-residue), w_k = w28^(2^(28-k)).
 * m = .r1cs rows of the handle's form, n_pub = n_pub_out + n_pub_in (= n_outputs).  Domain: n = 2^log_n, the smallest power of two
 * >= m + n_pub + 1, omega = w_log_n; log_n > 28 is POB_E_RANGE.  Row vectors of length n: rows [0, m) are A.w, B.w, C.w as
 * pob_r1cs_products returns them; row m + s (s = 0 .. n_pub) has a = w[s], b = c = 0; every other row is 0.  A^, B^, C^ are the
 * polynomials of degree < n with A^(omega^k) = a_k.  Coset shift g = w_(log_n + 1) (g^n = -1) when log_n < 28, g = 25 (nqr^2) when
 * log_n = 28.  Output q[i] = A^(g omega^i) B^(g omega^i) - C^(g omega^i), i = 0 .. n - 1, natural order, canonical 32-byte LE.
 * snarkjs derives C on the domain as A o B; both agree on a witness that satisfies the rows. */
/* log_n of the handle's domain (builds the row plan on first use, like pob_r1cs_check) */
int pob_r1cs_domain(pob_handle *h, uint32_t *log_n);
/* q[0..n) of resident witness `index` into `out` (n x 32 B); `work` is caller scratch of 2 n x 32 B, not overlapping out (else
 * POB_E_BAD_ARG, as is a null out or work, or one that is not 16-byte aligned).  consumer_stream: as pob_r1cs_products (NULL = return when done; else enqueued, no host
 * wait, nothing allocated).  The first call builds the root and coset tables (at most 2 MB), freed by pob_destroy. */
int pob_r1cs_quotient(pob_handle *h, uint32_t index, void *out, void *work, void *consumer_stream);

/* ---- the third stage: BN254 G1 multi-exponentiation (the prover's A, B1, C and H MSMs) ---------------------------------------
 * out = sum_i [s_i] P_i over BN254 G1 (y^2 = x^3 + 3 over F_q, q = 0x30644e72...fd47, cofactor 1).
 * bases  : n affine points, 64 B each: x then y, each a 32-byte LE element of F_q in MONTGOMERY form (R = 2^256), the form a
 *          snarkjs .zkey stores its G1 sections in (as far as known here; not checked against a real .zkey).  (0, 0) = infinity.
 *          Bases are not checked to be on the curve.
 * scalars: n x 32 B LE integers, e.g. the resident witness (from pob_acquire) or q from pob_r1cs_quotient.  Any 256-bit
 *          value is allowed; since every point has order r, [s]P = [s mod r]P.
 * out    : one point, 64 B, x then y as CANONICAL 32-byte LE F_q elements; (0, 0) = infinity.  Device memory.
 * work   : caller scratch of at least pob_msm_g1_work_bytes(n) bytes, not overlapping bases, scalars or out; at most 64 n bytes
 *          for n >= 2^18 (the size of pob_r1cs_quotient's work, so the H MSM can reuse it).
 * consumer_stream: NULL = return when done; else (a cudaStream_t) enqueued with no host wait and nothing allocated.
 * n == 0, a null or non-16-byte-aligned pointer, a short or overlapping work, out overlapping bases or scalars: POB_E_BAD_ARG
 * before anything is enqueued.  n > 2^31: POB_E_RANGE.  No such device: POB_E_NO_DEVICE.
 * A Groth16 prover calls it four times: A over (A bases, w, n_signals), B1 likewise, C over (C bases, w + 32 (n_outputs + 1),
 * n_signals - n_outputs - 1), H over (H bases, q, 2^log_n) (INTEGRATION.md §3(e)). */
int pob_msm_g1_work_bytes(uint64_t n, uint64_t *bytes);          /* host-only, no GPU needed */
int pob_msm_g1(int device, const void *bases, const void *scalars, uint64_t n,
               void *out, void *work, uint64_t work_bytes, void *consumer_stream);

/* ---- the fourth stage: BN254 G2 multi-exponentiation (the prover's B MSM) -------------------------------------------------------
 * out = sum_i [s_i] P_i over BN254 G2: the twist y^2 = x^3 + 3 / (9 + u) over F_q2 = F_q[u] / (u^2 + 1), whose points of order r
 * form a subgroup (the cofactor is not 1).  The same Pippenger pipeline as pob_msm_g1, over F_q2.
 * bases  : n affine points, 128 B each: x.c0, x.c1, y.c0, y.c1 (x = x.c0 + x.c1 u), each a 32-byte LE element of F_q in MONTGOMERY
 *          form, as the G1 bases (the form of a snarkjs .zkey's G2 sections as far as known here; not checked against a real .zkey).
 *          All-zero = infinity.  Bases must lie in the order-r subgroup: this is NOT checked, and [s]P = [s mod r]P holds only there.
 * scalars: n x 32 B LE integers, any 256-bit value (taken mod r).
 * out    : one point, 128 B in the same order, CANONICAL F_q elements; all-zero = infinity.  Device memory.
 * work   : caller scratch of at least pob_msm_g2_work_bytes(n) bytes, not overlapping bases, scalars or out.
 * consumer_stream, argument checks and error codes: as pob_msm_g1. */
int pob_msm_g2_work_bytes(uint64_t n, uint64_t *bytes);          /* host-only, no GPU needed */
int pob_msm_g2(int device, const void *bases, const void *scalars, uint64_t n,
               void *out, void *work, uint64_t work_bytes, void *consumer_stream);

/* ---- the proof: Groth16 over BN254 from a resident witness and a proving key in device memory --------------------------------
 * snarkjs's convention, which pob_r1cs_quotient follows: n_vars = pob_desc.n_signals of the handle's form, n_pub = n_outputs, the
 * domain n = 2^log_n of pob_r1cs_domain.  w = resident witness `index`, q = its quotient (pob_r1cs_quotient).  The key is a set of
 * device pointers to its sections (no .zkey is read here); every point is affine, Montgomery form, (0, 0) = infinity:
 *   A  = alpha1 + sum_i w_i A_i  + [r] delta1
 *   B  = beta2  + sum_i w_i B2_i + [s] delta2,   B1 = beta1 + sum_i w_i B1_i + [s] delta1
 *   C  = sum_{i > n_pub} w_i C_i + sum_k q_k H_k + [s] A + [r] B1 - [r s] delta1
 * r and s are any 256-bit values, taken mod r.  For zero knowledge they must be uniformly random and secret: that is the caller's
 * job, this function draws no random numbers (r = s = 0 is accepted).  proof: 256 bytes of device memory, all canonical affine:
 * A (64 B, x then y), B (128 B, x.c0, x.c1, y.c0, y.c1), C (64 B).
 * The call enqueues on consumer_stream, with no host wait, nothing allocated and no host memory read after it returns (r and s go to
 * the kernel by value): the quotient into `work`, the H MSM over it, the A, B1, C and B2 MSMs over the witness, one assembly kernel.
 * Witness readiness and consumer_stream (NULL = return when done) are as pob_r1cs_quotient's, and so are the index errors.  A null
 * argument, counts that differ from the handle's, a null or non-16-byte-aligned key pointer, proof or work, work shorter than
 * pob_groth16_work_bytes, or a proof overlapping work: POB_E_BAD_ARG, before anything is enqueued. */
typedef struct {
    uint64_t n_vars;                       /* must equal the handle's n_signals  (else POB_E_BAD_ARG) */
    uint32_t n_pub;                        /* must equal n_outputs               (else POB_E_BAD_ARG) */
    uint32_t log_n;                        /* must equal pob_r1cs_domain         (else POB_E_BAD_ARG) */
    const void *alpha1, *beta1, *delta1;   /* one G1 point each, 64 B, Montgomery, as pob_msm_g1 bases  */
    const void *beta2, *delta2;            /* one G2 point each, 128 B, Montgomery, as pob_msm_g2 bases */
    const void *a, *b1;                    /* n_vars G1 points                                           */
    const void *b2;                        /* n_vars G2 points                                           */
    const void *c;                         /* n_vars - n_pub - 1 G1 points, wires n_pub + 1 ..           */
    const void *h;                         /* 2^log_n G1 points, paired with q[k] of pob_r1cs_quotient   */
} pob_groth16_key;
/* bytes of `work` a proof on this handle needs: q (32 n), then the largest of the quotient's 64 n and the MSM scratches, then the
 * five MSM results (builds the row plan on first use, like pob_r1cs_domain) */
int pob_groth16_work_bytes(pob_handle *h, uint64_t *bytes);
int pob_groth16_prove(pob_handle *h, uint32_t index, const pob_groth16_key *key,
                      const uint64_t r[4], const uint64_t s[4],
                      void *proof, void *work, uint64_t work_bytes, void *consumer_stream);

/* ---- the proving key from a snarkjs .zkey ----------------------------------------------------------------------------------------
 * The format as far as known here (not checked against a file written by snarkjs; DESIGN.md §5 "Key loading").  Integers are little
 * endian.  "zkey", u32 version (1), u32 n_sections, then per section u32 id, u64 size, size bytes, in any order.  Ids 1..9 appear
 * exactly once each; id 10 (contributions) and unknown ids are skipped.
 *   1: u32 protocol (1 = Groth16)
 *   2: u32 n8q (32), q, u32 n8r (32), r, u32 nVars, u32 nPublic, u32 domainSize, alpha1 G1, beta1 G1, beta2 G2, gamma2 G2, delta1 G1,
 *      delta2 G2 (660 bytes)
 *   3: nPublic + 1 G1 points (IC: checked, not returned)
 *   4: u32 nCoefs, then nCoefs x 44 B: u32 matrix (0 = A, 1 = B), u32 constraint, u32 signal, value = c R^2 mod r (R = 2^256).
 *      snarkjs appends the A entries (m + s, s, 1) for s = 0 .. nPublic: the public rows of pob_r1cs_quotient.  No C matrix.
 *   5: A, nVars G1   6: B1, nVars G1   7: B2, nVars G2   8: C, nVars - nPublic - 1 G1   9: H, domainSize G1
 * Points are affine, 64 B (G1) or 128 B (G2), Montgomery form, (0, 0) = infinity: the form of pob_msm_g1 / pob_msm_g2, so sections 5-9
 * land in device memory byte for byte. */
typedef struct {
    uint64_t n_vars;           /* nVars   (== pob_desc.n_signals of a handle the key fits) */
    uint32_t n_pub;            /* nPublic (== n_outputs) */
    uint32_t log_n;            /* log2 domainSize (== pob_r1cs_domain) */
    uint64_t n_coefs;          /* section-4 entries, the public rows included */
    uint64_t file_bytes;
    uint64_t a_bytes, b1_bytes, b2_bytes, c_bytes, h_bytes;   /* device bytes of pob_groth16_key.a, .b1, .b2, .c, .h */
    uint64_t key_bytes;        /* those five plus alpha1, beta1, delta1 (64 B each) and beta2, delta2 (128 B each) */
} pob_zkey_desc;
/* host-only, no GPU needed: parse the header and the section table and validate the structure (magic, version, protocol, n8q / n8r,
 * both moduli, one each of sections 1-9, every section size against nVars, nPublic, domainSize and nCoefs, domainSize a power of two
 * <= 2^28).  A file that cannot be read or ends early: POB_E_IO; any structural error: POB_E_KEY; pob_last_error names it. */
int pob_zkey_info(const char *path, pob_zkey_desc *out);

typedef struct {
    uint32_t coef_match;            /* bit 0: matrix A of section 4 equals the handle's .r1cs A rows plus the public rows, bit 1: B equals
                                       B; values read as c R^2 mod r */
    uint32_t coef_match_canonical;  /* the same bits with the values read as canonical elements (diagnosis of the encoding) */
    uint64_t coef_out_of_range;     /* entries with matrix > 1, constraint >= domainSize or signal >= nVars (counted, never used) */
    uint64_t points_checked;        /* points of sections 2, 3 and 5-9 */
    uint64_t points_bad;            /* a coordinate >= q, or off the curve read in Montgomery form */
    uint64_t points_bad_canonical;  /* the same with the coordinates read as canonical elements */
    uint32_t first_bad_section;     /* section of the first bad point (smallest section, then index); 0 = none */
    uint32_t reserved;
    uint64_t first_bad_index;       /* its index in the section (section 2: 0 alpha1, 1 beta1, 2 beta2, 3 gamma2, 4 delta1, 5 delta2) */
    float read_ms;                  /* host time in file reads (reader thread) */
    float copy_ms;                  /* device time of the host-to-device copies */
    float check_ms;                 /* device time of the check kernels (both sides of the coefficient check, the point checks) */
    float total_ms;                 /* wall time of the call */
    uint64_t bytes_read;
    uint64_t device_scratch_bytes;  /* peak device memory the call allocated itself (freed before it returns) */
} pob_zkey_report;
/* Fill the caller's key buffers from a .zkey and check the key against the handle's circuit on the GPU.  dst: a pob_groth16_key whose
 * n_vars / n_pub / log_n are the handle's and whose pointers are device buffers of the sizes pob_zkey_info gives (16-byte aligned);
 * after success it is ready for pob_groth16_prove.  A key whose nVars, nPublic or domainSize differ from the handle's n_signals,
 * n_outputs or pob_r1cs_domain is refused before any transfer (POB_E_KEY).  The file streams through a ring of pinned staging buffers
 * of at most staging_bytes in all (0 = 256 MiB; at least 512), read by a host thread while earlier chunks are copied and checked; it is
 * never held in host memory whole.  A setup call: it waits on the host, and allocates and frees device scratch (reported).
 * The check: with pseudo-random x_j per wire and rho_c per domain row derived from `seed` on the device, for M = A, B
 *   sum over section-4 entries (M, c, s, v) of rho_c x_s c   ==   sum_c rho_c (M x)_c   (k_r1cs_products over x, + the public rows for A),
 * equal for equal matrices and, except with probability about 2 / r, different for any other; every point of sections 2, 3, 5-9 has
 * coordinates < q and lies on y^2 = x^3 + 3 (G1) or the twist (G2) read in Montgomery form, or is (0, 0).  Not checked: the G2 subgroup.
 * A failure of either part is POB_E_KEY with rep filled in (rep may be NULL). */
int pob_zkey_load(pob_handle *h, const char *path, uint64_t seed, uint64_t staging_bytes, const pob_groth16_key *dst, pob_zkey_report *rep);

/* the verification key of a .zkey (host-only, no GPU needed): alpha1 | beta2 | gamma2 | delta2 | IC copied byte for byte from sections 2
 * and 3, 448 + 64 (n_pub + 1) bytes, Montgomery form as in the file; *n_pub = nPublic.  The file is validated exactly as pob_zkey_info
 * does (same errors).  out_bytes shorter than the key: POB_E_BAD_ARG (with *n_pub set, so a caller can size out and call again). */
int pob_zkey_vk(const char *path, void *out, uint64_t out_bytes, uint32_t *n_pub);

/* ---- verification: the BN254 optimal ate pairing and Groth16 verdicts --------------------------------------------------------------
 * e(P, Q) = f^((q^12 - 1) / r), the optimal ate pairing of BN254 (x = 4965661367192848881): the Miller loop over 6x + 2 and the lines
 * at pi(Q) and -pi^2(Q), then the final exponentiation to exactly (q^12 - 1) / r (DESIGN.md §5 "Verification").  Values of F_q12 are
 * 12 F_q elements in the nesting F_q12 = F_q6[w] / (w^2 - v), F_q6 = F_q2[v] / (v^3 - (9 + u)): c0.c0.c0, c0.c0.c1, c0.c1.c0, ..,
 * c1.c2.c1, each a 32-byte LE CANONICAL element (the order of snarkjs's vk_alphabeta_12 as far as known here; not checked against
 * snarkjs).  O on either side gives 1.
 * pob_bn254_pairing: out[i] = e(g1[i], g2[i]), i < n.  g1: n x 64 B points as pob_msm_g1 bases, g2: n x 128 B as pob_msm_g2 bases
 * (Montgomery form, all-zero = O), out: n x 384 B, all device memory.  The inputs are NOT checked to lie on their curves or in G1 / G2;
 * outside them the value is not a pairing.  consumer_stream: NULL = return when done; else enqueued with no host wait and nothing
 * allocated.  n == 0, a null or non-16-byte-aligned pointer, or out overlapping an input: POB_E_BAD_ARG before anything is enqueued. */
int pob_bn254_pairing(int device, const void *g1, const void *g2, uint64_t n, void *out, void *consumer_stream);

/* Groth16 verification, one verdict per proof: proof i is valid iff
 *   e(-A_i, B_i) e(vk_x, gamma2) e(C_i, delta2) e(alpha1, beta2) == 1,   vk_x = IC_0 + sum_j pub_ij IC_j.
 * vk     : device pointers, Montgomery form, affine, (0, 0) = O, as in a .zkey (pob_zkey_vk gives them in one buffer).
 * proofs : n x 256 B, exactly what pob_groth16_prove writes: A (64 B), B (128 B), C (64 B), canonical affine, all-zero = O.
 * publics: n x n_pub x 32 B canonical LE values; may be NULL when n_pub == 0.
 * status : n x uint32 of device memory, one of POB_VERIFY_* below.  The checks run in this order and the first failure is reported:
 *          a proof coordinate >= q or a point off its curve (BAD_POINT), a public input >= r (BAD_PUBLIC: never reduced, as on-chain
 *          verifiers refuse it), B outside the order-r subgroup ([r]B != O: BAD_SUBGROUP), the equation (FAIL).  A = O or B = O is
 *          not refused: its pairing is 1 and the equation decides.  A malformed key gives BAD_KEY to every proof of the call: a
 *          coordinate >= q, a point off its curve, beta2, gamma2 or delta2 outside the subgroup, or gamma2 or delta2 = O.
 * work   : caller scratch of pob_groth16_verify_work_bytes: the key's check flags, f_{alpha1,beta2} before its final exponentiation,
 *          and the precomputed lines of gamma2 and delta2.
 * consumer_stream: as pob_msm_g1 (NULL = return when done; else stream-ordered, no host wait, nothing allocated).
 * A null pointer (publics only when n_pub > 0), a pointer that is not 16-byte aligned (status: 4-byte), a short work, n == 0, or
 * status or work overlapping proofs, publics, a key point or each other: POB_E_BAD_ARG before anything is enqueued. */
enum {
    POB_VERIFY_OK = 0,              /* valid */
    POB_VERIFY_FAIL = 1,            /* the pairing equation fails */
    POB_VERIFY_BAD_POINT = 2,       /* a proof coordinate >= q, or a point off its curve */
    POB_VERIFY_BAD_SUBGROUP = 3,    /* B outside the order-r subgroup */
    POB_VERIFY_BAD_PUBLIC = 4,      /* a public input >= r */
    POB_VERIFY_BAD_KEY = 5          /* the verification key is malformed (every proof of the call) */
};
typedef struct {
    uint32_t n_pub;
    const void *alpha1, *beta2, *gamma2, *delta2;  /* device, Montgomery, as in a .zkey: 64, 128, 128, 128 B */
    const void *ic;                                 /* (n_pub + 1) G1 points, 64 B each */
} pob_groth16_vk;
int pob_groth16_verify_work_bytes(uint32_t n_pub, uint64_t n, uint64_t *bytes);   /* host-only, no GPU needed */
int pob_groth16_verify(int device, const pob_groth16_vk *vk, const void *proofs, const void *publics, uint64_t n,
                       uint32_t *status, void *work, uint64_t work_bytes, void *consumer_stream);

/* ---- the step just before the path (SURVEY.md 8(f) rank 3) ------------------------------------------------------
 * replaces: find_burn_key() of the reference input generator (tests/main.py:47-56): starting at start_key, find the
 * first burnKey >= start_key whose keccak256(burnKey[32 BE] | revealAmount[32 BE] | burnExtraCommitment[32 BE] |
 * "EIP-7503") begins with `zero_bytes` zero bytes (circuits/utils/proof_of_work.circom:54-81).  Searches at most
 * max_tries consecutive keys on the GPU; *tries receives the number of keys up to and including the hit.
 * Returns POB_E_RANGE when no key in the window satisfies the check. */
int pob_pow_grind(int device, const uint64_t start_key[4], const uint64_t reveal_amount[4], const uint64_t burn_extra_commitment[4],
                  uint32_t zero_bytes, uint64_t max_tries, uint64_t found_key[4], uint64_t *tries);

const char *pob_last_error(void);
const char *pob_version(void);

#ifdef __cplusplus
}
#endif
#endif
