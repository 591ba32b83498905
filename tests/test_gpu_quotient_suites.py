"""pob_r1cs_products and pob_r1cs_quotient on every gadget circuit of the golden suites (all but the ProofOfBurn test shape), in both
witness forms, on the first accepted case of each suite; then on adversarial witnesses written over the resident one.

Rows: the device products equal the written `.r1cs` evaluated in Python (tests/r1cs_reader.py) on every row of every system of at
most 1 M rows; the eight --O0 Keccak-family systems (2.6 - 5.1 M rows) instead pass pob_r1cs_check.  Quotient: up to 2^16 points it
equals the model (tests/quotient_model.py) entry for entry; larger domains satisfy h(r) (r^n - 1) = A^(r) B^(r) - C^(r) at two
points through the device evaluator (test_gpu_quotient._main_identity).  A changed q_i fails either check.  Neither kernel needs a
satisfying witness, so an all-(p - 1) witness drives every combination through its largest sums."""
import ctypes
import random

import numpy as np
import pytest

import quotient_model as qm
from helpers import gold, _cudart, cuda_poke
from r1cs_reader import R1cs, witness_ints
from test_gpu_quotient import _main_identity

pytestmark = pytest.mark.gpu

P = qm.P
M64 = (1 << 64) - 1
SUITES = [s for s in gold() if s["suite"] != "test_proof_of_burn"]
FILE_ROWS_MAX = 1 << 20                 # products checked against the file up to here; pob_r1cs_check above
EXACT_LOG_MAX = 16                      # q equals the model entry for entry up to here; the identity above
ADVERSARIAL = [("test_poseidon_4", 0), ("test_num_2_bits_safe_256", 0), ("test_rlp_empty_account_3", 1),
               ("test_leaf_detector_2", 0)]


def _limbs(vals):
    v = np.asarray(vals, dtype=object)
    return np.ascontiguousarray(np.stack([((v >> (64 * k)) & M64).astype(np.uint64) for k in range(4)], axis=1))


def _write_witness(dptr, vals):
    """overwrite a whole resident witness (32 bytes per entry at device pointer dptr) with one cudaMemcpy"""
    limbs = _limbs(vals)
    rc = _cudart().cudaMemcpy(ctypes.c_void_p(dptr), ctypes.c_void_p(limbs.ctypes.data), ctypes.c_size_t(limbs.nbytes), ctypes.c_int(1))
    assert rc == 0, "cudaMemcpy H2D failed: %d" % rc


def _ints(t):
    return witness_ints(t.cpu().numpy())


def _accepted(s, opt):
    import pob_b200
    case = next(c for c in s["cases"] if c["expected"] is not None)
    c = pob_b200.Circuit(s["main"], max_slots=1, opt=opt)
    res = c.run([case["input"]])
    assert res.status[0] == 0, "%s: the expected case is rejected" % s["suite"]
    return c


def _products_equal_the_file(c, R, W):
    want = R.products(W)
    for g, w, v in zip(c.r1cs_products(0), want, "ABC"):
        got = _ints(g)
        assert (got == w).all(), "%s rows %s differ" % (v, np.nonzero(got != w)[0][:10])
    return want


def _quotient_equals_the_model(c, R, W, log_n):
    A, B, C = R.products(W)
    q = c.r1cs_quotient(0)
    assert q.shape == (1 << log_n, 4)
    got = _ints(q)
    want = qm.quotient(A, B, C, W[:R.n_pub_out + R.n_pub_in + 1], R.m)
    assert (got == want).all(), "entries %s differ" % np.nonzero(got != want)[0][:10]
    return q, got, want


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
@pytest.mark.parametrize("s", SUITES, ids=[s["suite"] for s in SUITES])
def test_quotient_and_products(s, opt, tmp_path):
    import pob_b200
    d = pob_b200.write_r1cs(s["main"], None, opt=opt)                  # counts only: the writer's header without the file
    small = d["n_constraints"] <= FILE_ROWS_MAX
    R = None
    if small:
        f = str(tmp_path / "c.r1cs")
        pob_b200.write_r1cs(s["main"], f, opt=opt)
        R = R1cs(f)
        assert (R.m, R.n_pub_out, R.n_pub_in) == (d["n_constraints"], d["n_pub_out"], 0)
    c = _accepted(s, opt)
    try:
        log_n = c.r1cs_domain()
        assert log_n == qm.domain_log(d["n_constraints"], d["n_pub_out"])
        if small:
            W = witness_ints(c.witness(0))
            _products_equal_the_file(c, R, W)
        else:
            rep = c.r1cs_check(0)
            assert rep["n_constraints"] == d["n_constraints"] and rep["n_failed"] == 0
        if log_n <= EXACT_LOG_MAX:
            q, got, want = _quotient_equals_the_model(c, R, W, log_n)
            i = random.Random(log_n).randrange(1 << log_n)
            cuda_poke(q.data_ptr(), i, (int(got[i]) + 1) % P)
            after = _ints(q)
            assert np.nonzero(after != want)[0].tolist() == [i]
        else:
            _main_identity(c, 0, log_n, random.Random(1000 * log_n + opt))
    finally:
        c.close()


@pytest.mark.parametrize("name,opt", ADVERSARIAL, ids=["%s-O%d" % a for a in ADVERSARIAL])
def test_adversarial_witnesses(name, opt, tmp_path):
    """witnesses that satisfy nothing, w[0] included: every entry p - 1; uniform random canonical entries; the accepted witness with
    a few entries set to 0 and p - 1.  The products equal the file's, and q the model's, on each."""
    import pob_b200
    s = next(x for x in SUITES if x["suite"] == name)
    f = str(tmp_path / "c.r1cs")
    pob_b200.write_r1cs(s["main"], f, opt=opt)
    R = R1cs(f)
    c = _accepted(s, opt)
    try:
        log_n = c.r1cs_domain()
        assert log_n <= 15
        real = witness_ints(c.witness(0))
        n = len(real)
        rng = random.Random(n)
        mixed = real.copy()
        for k in rng.sample(range(n), min(n, 16)):
            mixed[k] = rng.choice((0, P - 1))
        mixed[0] = P - 1
        dptr = c.witness_device_ptr(0)
        for what, W in (("p-1", np.full(n, P - 1, dtype=object)),
                        ("random", np.array([rng.randrange(P) for _ in range(n)], dtype=object)),
                        ("mixed", mixed)):
            _write_witness(dptr, W)
            assert (witness_ints(c.witness(0)) == W).all()
            if what != "mixed":
                assert len(R.failing_rows(W)) > 0, what                      # the rows do not hold: nothing relies on them
            _products_equal_the_file(c, R, W)
            _quotient_equals_the_model(c, R, W, log_n)
    finally:
        c.close()


def test_misaligned_and_foreign_buffers_are_rejected():
    """both entry points access caller buffers as uint4: a buffer 8 bytes into an allocation is POB_E_BAD_ARG before anything is
    enqueued; r1cs_quotient() also refuses out / work on another device than the handle's"""
    import torch
    import pob_b200
    s = next(x for x in SUITES if x["suite"] == "test_poseidon_2")
    c = _accepted(s, 0)
    try:
        n = 1 << c.r1cs_domain()
        out = torch.empty((n + 1, 4), dtype=torch.uint64, device="cuda")
        work = torch.empty((2 * n + 1, 4), dtype=torch.uint64, device="cuda")
        L = pob_b200.lib()
        o, w = out.data_ptr(), work.data_ptr()
        assert L.pob_r1cs_quotient(c._h, 0, o + 8, w, None) == -1
        assert L.pob_r1cs_quotient(c._h, 0, o, w + 8, None) == -1
        for args in ((o + 8, None, None), (None, o + 8, None), (None, None, o + 8), (o, w, o + 40)):
            assert L.pob_r1cs_products(c._h, 0, 0, 1, *args, None) == -1
        with pytest.raises(pob_b200.PobError) as e:
            c.r1cs_quotient(0, out=out.view(-1)[1:4 * n + 1])
        assert e.value.code == -1
        assert torch.equal(c.r1cs_quotient(0, out=out[:n], work=work[:2 * n]), c.r1cs_quotient(0))   # aligned: accepted
        if torch.cuda.device_count() > 1:
            other = torch.empty((n, 4), dtype=torch.uint64, device="cuda:1")
            with pytest.raises(ValueError):
                c.r1cs_quotient(0, out=other)
    finally:
        c.close()
