"""The `.r1cs` rows on the GPU: pob_r1cs_products against products computed in Python from the written `.r1cs`
(tests/r1cs_reader.py) and the resident witness, its windows and argument checks, pob_r1cs_check on Spend(31) and the main shape
in both witness forms, and the products enqueued on a consumer stream inside the consumer-paced hand-off."""
import numpy as np
import pytest

from helpers import suite, cuda_poke
from r1cs_reader import R1cs, witness_ints

pytestmark = pytest.mark.gpu

ROUND_BLOCK_ROWS = 89216 + 1920 + 9920      # eq + kc + r1 records of one KeccakfRound block (none is a hint or trivial)


def _ints(t):
    return witness_ints(t.cpu().numpy())


def _spend(opt, tmp_path, max_slots=2):
    import pob_b200
    s = suite("test_spend")
    c = pob_b200.Circuit("Spend(31)", max_slots=max_slots, opt=opt)
    res = c.run([s["cases"][0]["input"], s["cases"][1]["input"]])
    assert res.status[0] == 0 and res.status[1] != 0
    f = str(tmp_path / ("spend_o%d.r1cs" % opt))
    pob_b200.write_r1cs("Spend(31)", f, opt=opt)
    return c, R1cs(f)


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
def test_products_equal_the_file(opt, tmp_path):
    """every row's A.w, B.w, C.w on the GPU equals, value for value, the products of the written .r1cs with the witness; A*B = C"""
    import pob_b200
    c, R = _spend(opt, tmp_path)
    try:
        W = witness_ints(c.witness(0))
        A, B, C = R.products(W)
        ga, gb, gc = c.r1cs_products(0)
        assert ga.shape == (R.m, 4)
        vals = [_ints(t) for t in (ga, gb, gc)]
        for g, want in zip(vals, (A, B, C)):
            assert (g < pob_b200.P).all(), "non-canonical output"
            assert (g == want).all(), "rows %s differ" % np.nonzero(g != want)[0][:10]
        assert ((vals[0] * vals[1] - vals[2]) % pob_b200.P == 0).all()
        rep = c.r1cs_check(0)
        assert rep["n_constraints"] == R.m and rep["n_failed"] == 0 and rep["n_hints"] == 0 and rep["first_failed"] == 2 ** 64 - 1
        assert rep["n_nonlinear"] == int((R.lc_n[0::3] > 0).sum())
        assert rep["signals_read"] == len(np.unique(R.wire))
    finally:
        c.close()


def test_windows_and_argument_checks(tmp_path):
    import pob_b200
    c, R = _spend(0, tmp_path)
    try:
        full = [_ints(t) for t in c.r1cs_products(0)]
        nf = R.m - 24 * ROUND_BLOCK_ROWS                       # Spend(31): one Keccakf = 24 round blocks after the flat rows
        assert nf > 0
        starts = [0, nf - 3, nf + ROUND_BLOCK_ROWS - 5, nf + 23 * ROUND_BLOCK_ROWS - 1, R.m - 7, R.m - 1]
        for first in starts:
            for count in (1, 7, 10):
                count = min(count, R.m - first)
                got = c.r1cs_products(0, first, count)
                for g, want in zip(got, full):
                    assert (_ints(g) == want[first:first + count]).all(), (first, count)
        for b in range(24):                                    # both ends of every round block
            for first in (nf + b * ROUND_BLOCK_ROWS - 1, nf + (b + 1) * ROUND_BLOCK_ROWS - 1):
                got = c.r1cs_products(0, first, 2 if first + 2 <= R.m else 1)
                assert all((_ints(g) == w[first:first + g.shape[0]]).all() for g, w in zip(got, full))
        a, b, cc = c.r1cs_products(0, R.m, 0)
        assert a.shape == (0, 4)
        only_c = c.r1cs_products(0, 5, 100, vectors="c")
        assert only_c[0] is None and only_c[1] is None and (_ints(only_c[2]) == full[2][5:105]).all()
        with pytest.raises(pob_b200.PobError) as e:
            c.r1cs_products(0, R.m, 1)
        assert e.value.code == pob_b200.E_RANGE
        with pytest.raises(pob_b200.PobError) as e:
            c.r1cs_products(0, R.m - 1, 2)
        assert e.value.code == pob_b200.E_RANGE
        with pytest.raises(pob_b200.PobError) as e:
            c.r1cs_products(1, 0, 1)
        assert e.value.code == pob_b200.E_REJECTED
        with pytest.raises(pob_b200.PobError) as e:
            c.r1cs_check(1)
        assert e.value.code == pob_b200.E_REJECTED
    finally:
        c.close()


def test_first_failed_is_the_row_the_file_finds(tmp_path):
    """O0 Spend(31): after a poke, pob_r1cs_check's first_failed is the lowest row of the file that fails on the poked witness"""
    import pob_b200
    c, R = _spend(0, tmp_path)
    try:
        W = witness_ints(c.witness(0))
        ptr, rows = R.rows_of_wire()
        dptr = c.witness_device_ptr(0)
        rng = np.random.default_rng(99)
        for k in [int(v) for v in rng.choice(np.arange(1, R.n_wires), size=40, replace=False)]:
            old = W[k]
            W[k] = (old + 1) % R.p
            bad = [int(r) for r in np.unique(rows[ptr[k]:ptr[k + 1]]) if not R.row_ok(int(r), W)]
            cuda_poke(dptr, k, W[k])
            rep = c.r1cs_check(0)
            cuda_poke(dptr, k, old)
            W[k] = old
            assert rep["n_failed"] == len(bad)
            assert rep["first_failed"] == (min(bad) if bad else 2 ** 64 - 1), k
        assert c.r1cs_check(0)["n_failed"] == 0
    finally:
        c.close()


def test_products_on_a_consumer_stream():
    """inside submit / acquire(stream) / release(stream), products enqueued on the consumer stream without a host wait equal those of
    the synchronous call"""
    import torch
    import pob_b200
    s = suite("test_spend")
    inputs = [s["cases"][0]["input"]] * 4
    c = pob_b200.Circuit("Spend(31)", max_slots=2, opt=1)
    try:
        packed = c.pack(inputs)
        res = c.run_packed(packed[:1])
        assert res.status[0] == 0
        want = [t.clone() for t in c.r1cs_products(0)]
        n = want[0].shape[0]
        st = torch.cuda.Stream()
        got = []
        c.submit(packed)
        while True:
            r = c.acquire(st.cuda_stream)
            if r is None:
                break
            idx, dptr = r
            assert dptr is not None
            got.append(c.r1cs_products(idx, 0, n, stream=st))
            c.release(idx, st.cuda_stream)
        fin = c.finish()
        assert (fin.status == 0).all() and len(got) == 4
        st.synchronize()
        for g in got:
            for x, y in zip(g, want):
                assert torch.equal(x.cpu(), y.cpu())
    finally:
        c.close()


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
def test_r1cs_check_main_shape(opt):
    """main_proof_of_burn, two synthetic instances: every row holds; for the reduced form 150 pokes are noticed, except entries the
    circuit leaves free and only a hint pins (the same --O0 entry then fails a hint record of pob_selfcheck and no constraint)"""
    import pob_b200
    from pob_b200 import synth
    shape = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)
    packed = synth.pack_instances(synth.make_batch(2, shape, seed=4242), shape)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=2, opt=opt)
    missed = []
    try:
        res = c.run_packed(packed)
        assert (res.status == 0).all()
        for i in (0, 1):
            r = c.r1cs_check(i)
            assert r["n_failed"] == 0 and r["n_hints"] == 0
            assert (r["n_constraints"], r["n_nonlinear"]) == ((215962292, 17910859) if opt == 0 else (21508380, 16142845))
        if opt == 0:
            return
        wmap = c.witness_map()
        dptr = c.witness_device_ptr(0)
        rng = np.random.default_rng(150)
        for k in [int(v) for v in rng.integers(1, c.n_signals, 150)]:
            old = pob_b200.from_limbs(c.witness(0, k, 1)[0])
            cuda_poke(dptr, k, (old + 1) % pob_b200.P)
            r = c.r1cs_check(0)
            cuda_poke(dptr, k, old)
            if r["n_failed"] == 0:
                missed.append(k)
        assert c.r1cs_check(0)["n_failed"] == 0
    finally:
        c.close()
    if missed:
        c0 = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1)
        try:
            assert c0.run_packed(packed[:1]).status[0] == 0
            dptr = c0.witness_device_ptr(0)
            for k in missed:
                i = int(wmap[k])
                old = pob_b200.from_limbs(c0.witness(0, i, 1)[0])
                cuda_poke(dptr, i, (old + 1) % pob_b200.P)
                r = c0.selfcheck(0)
                cuda_poke(dptr, i, old)
                assert r["n_failed"] == 0 and r["n_hint_failed"] > 0, "reduced entry %d (--O0 %d) is pinned by nothing" % (k, i)
        finally:
            c0.close()
