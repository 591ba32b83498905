"""The Groth16 quotient on the GPU (pob_r1cs_quotient) against its definition (tests/quotient_model.py).

Reduced Spend(31) (n = 2^18): q equals the Python model entry for entry.  Every larger size is checked through one identity at random
points r: with h the polynomial through q_i / (g^n - 1) on the coset, h(r) (r^n - 1) = A^(r) B^(r) - C^(r).  Every q_i enters h(r)
with a nonzero weight, so one point checks the whole vector -- its order, omega, g and the 1/n scaling -- up to 2n/p.  Spend(31)
--O0 (2^22) is evaluated in Python; the main shape (2^25 reduced, 2^28 --O0 with the shift 25) by the barycentric evaluator of
tests/devprobe/bary_probe.cu over the device vectors, which is first checked against the Python one.  A changed q_i breaks the
identity at every size."""
import os
import random
import sys

import numpy as np
import pytest

import quotient_model as qm
from helpers import suite, cuda_poke
from r1cs_reader import R1cs, witness_ints

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

pytestmark = pytest.mark.gpu

MAIN_SHAPE = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)


def _ints(t):
    return witness_ints(t.cpu().numpy())


def dev_bary(t, shift, log_n, r, first=0):
    """qm.bary over the rows of a (k, 4) uint64 CUDA tensor, evaluated on the GPU by tests/devprobe/bary_probe.cu"""
    import torch
    import bary
    assert t.is_contiguous() and t.shape[1] == 4
    torch.cuda.synchronize()
    return bary.evaluate(t.data_ptr(), t.shape[0], shift, qm.root(log_n), log_n, r, first=first)


def _point(rng, log_n):
    r = rng.randrange(qm.P)
    n = 1 << log_n
    assert pow(r, n, qm.P) not in (1, pow(qm.shift(log_n), n, qm.P))      # off the domain and the coset
    return r


def _h_side(h_at_r, log_n, r):
    """h(r) (r^n - 1) from sum_i q_i L_i(r) on the coset"""
    n = 1 << log_n
    g = qm.shift(log_n)
    return h_at_r * pow(pow(g, n, qm.P) - 1, qm.P - 2, qm.P) % qm.P * (pow(r, n, qm.P) - 1) % qm.P


def _spend(opt, tmp_path, max_slots=2):
    import pob_b200
    s = suite("test_spend")
    c = pob_b200.Circuit("Spend(31)", max_slots=max_slots, opt=opt)
    res = c.run([s["cases"][0]["input"], s["cases"][1]["input"]])
    assert res.status[0] == 0 and res.status[1] != 0
    f = str(tmp_path / ("spend_o%d.r1cs" % opt))
    pob_b200.write_r1cs("Spend(31)", f, opt=opt)
    R = R1cs(f)
    W = witness_ints(c.witness(0))
    return c, R, R.products(W), W[:R.n_pub_out + R.n_pub_in + 1]


def test_reduced_spend_equals_the_model(tmp_path):
    """n = 2^18: every q_i equals the model's; the identity holds, and fails after one device entry is changed"""
    import pob_b200
    c, R, (A, B, C), w_pub = _spend(1, tmp_path)
    try:
        assert c.r1cs_domain() == 18
        q = c.r1cs_quotient(0)
        assert q.shape == (1 << 18, 4)
        got = _ints(q)
        want = qm.quotient(A, B, C, w_pub, R.m)
        assert (got == want).all(), "entries %s differ" % np.nonzero(got != want)[0][:10]
        rng = random.Random(18)
        r = _point(rng, 18)
        _, vecs = qm.rows(A, B, C, w_pub, R.m)
        a, b, cc = (qm.bary(v[:R.m + len(w_pub)], 1, 18, r) for v in vecs)
        assert _h_side(qm.bary(got, qm.shift(18), 18, r), 18, r) == (a * b - cc) % qm.P
        i = rng.randrange(1 << 18)
        cuda_poke(q.data_ptr(), i, (int(got[i]) + 1) % qm.P)
        assert _h_side(dev_bary(q, qm.shift(18), 18, r), 18, r) != (a * b - cc) % qm.P
        assert c.r1cs_quotient(0).equal(c.r1cs_quotient(0))                 # deterministic, and `out` is fully rewritten
    finally:
        c.close()


def test_errors(tmp_path):
    import torch
    import pob_b200
    c, R, _, _ = _spend(1, tmp_path)
    try:
        n = 1 << c.r1cs_domain()
        out = torch.empty((n, 4), dtype=torch.uint64, device="cuda")
        work = torch.empty((2 * n, 4), dtype=torch.uint64, device="cuda")
        L = pob_b200.lib()
        assert L.pob_r1cs_quotient(c._h, 0, None, work.data_ptr(), None) == -1
        assert L.pob_r1cs_quotient(c._h, 0, out.data_ptr(), None, None) == -1
        assert L.pob_r1cs_quotient(c._h, 0, work.data_ptr() + 32 * n, work.data_ptr(), None) == -1     # out inside work
        with pytest.raises(pob_b200.PobError) as e:
            c.r1cs_quotient(1)
        assert e.value.code == pob_b200.E_REJECTED
        with pytest.raises(pob_b200.PobError) as e:
            c.r1cs_quotient(2)
        assert e.value.code == pob_b200.E_RANGE
        with pytest.raises(ValueError):
            c.r1cs_quotient(0, out=out[:n - 1])
        assert torch.equal(c.r1cs_quotient(0, out=out, work=work), c.r1cs_quotient(0))
    finally:
        c.close()


def test_spend_o0_identity(tmp_path):
    """n = 2^22, evaluated in Python at two points; the probe's evaluator agrees with the Python one on these vectors"""
    c, R, (A, B, C), w_pub = _spend(0, tmp_path)
    try:
        assert c.r1cs_domain() == 22
        q = c.r1cs_quotient(0)
        got = _ints(q)
        ga = c.r1cs_products(0, vectors="a")[0]
        _, vecs = qm.rows(A, B, C, w_pub, R.m)
        rows = [v[:R.m + len(w_pub)] for v in vecs]
        rng = random.Random(22)
        g = qm.shift(22)
        for k in range(2):
            r = _point(rng, 22)
            hq = qm.bary(got, g, 22, r)
            a, b, cc = (qm.bary(v, 1, 22, r) for v in rows)
            assert _h_side(hq, 22, r) == (a * b - cc) % qm.P
            if k == 0:                                                       # the device evaluator, before the main shape relies on it
                assert dev_bary(q, g, 22, r) == hq
                assert dev_bary(ga, 1, 22, r) == qm.bary(A, 1, 22, r)
                assert dev_bary(ga[1000:], 1, 22, r, first=1000) == qm.bary(A[1000:], 1, 22, r, first=1000)
        i = rng.randrange(1 << 22)
        cuda_poke(q.data_ptr(), i, (int(got[i]) + 1) % qm.P)
        assert _h_side(dev_bary(q, g, 22, r), 22, r) != (a * b - cc) % qm.P
    finally:
        c.close()


def _main_identity(c, index, log_n, rng):
    """the identity at two points, every side evaluated on the device; then a changed q_i must break it"""
    import pob_b200
    q = c.r1cs_quotient(index)
    assert q.shape == (1 << log_n, 4)
    rows = c._r1cs_rows if getattr(c, "_r1cs_rows", None) else c.r1cs_check(index)["n_constraints"]
    c._r1cs_rows = rows
    n_pub = c.n_outputs
    w_pub = [pob_b200.from_limbs(x) for x in c.witness(index, 0, n_pub + 1)]
    g = qm.shift(log_n)
    pts = [_point(rng, log_n) for _ in range(2)]
    sides = {r: [] for r in pts}
    for v in "abc":
        t = c.r1cs_products(index, vectors=v)["abc".index(v)]
        for r in pts:
            x = dev_bary(t, 1, log_n, r)
            if v == "a":
                x = (x + qm.bary(w_pub, 1, log_n, r, first=rows)) % qm.P
            sides[r].append(x)
        del t
    for r in pts:
        a, b, cc = sides[r]
        assert _h_side(dev_bary(q, g, log_n, r), log_n, r) == (a * b - cc) % qm.P, "identity fails at instance %d" % index
    i = rng.randrange(1 << log_n)
    old = pob_b200.from_limbs(q[i].cpu().numpy())
    cuda_poke(q.data_ptr(), i, (old + 1) % qm.P)
    r = pts[0]
    a, b, cc = sides[r]
    assert _h_side(dev_bary(q, g, log_n, r), log_n, r) != (a * b - cc) % qm.P


def test_main_shape_reduced():
    """main_proof_of_burn, reduced witness (2^25), two synthetic instances"""
    import pob_b200
    from pob_b200 import synth
    packed = synth.pack_instances(synth.make_batch(2, MAIN_SHAPE, seed=4242), MAIN_SHAPE)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=2, opt=1)
    try:
        assert (c.run_packed(packed).status == 0).all()
        assert c.r1cs_domain() == 25
        rng = random.Random(25)
        for i in (0, 1):
            _main_identity(c, i, 25, rng)
    finally:
        c.close()


def test_main_shape_o0():
    """main_proof_of_burn, --O0 witness: log_n = 28, the only domain with the shift 25; one resident witness at a time"""
    import torch
    import pob_b200
    from pob_b200 import synth
    packed = synth.pack_instances(synth.make_batch(2, MAIN_SHAPE, seed=4242), MAIN_SHAPE)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1)
    try:
        assert c.r1cs_domain() == 28
        rng = random.Random(28)
        for k in (0, 1):
            assert c.run_packed(packed[k:k + 1]).status[0] == 0
            _main_identity(c, 0, 28, rng)
            torch.cuda.empty_cache()
    finally:
        c.close()


def test_quotient_on_a_consumer_stream():
    """inside submit / acquire(stream) / release(stream), the quotient enqueued on the consumer stream without a host wait equals
    the synchronous call"""
    import torch
    import pob_b200
    s = suite("test_spend")
    inputs = [s["cases"][0]["input"]] * 4
    c = pob_b200.Circuit("Spend(31)", max_slots=2, opt=1)
    try:
        packed = c.pack(inputs)
        assert c.run_packed(packed[:1]).status[0] == 0
        want = c.r1cs_quotient(0).clone()
        st = torch.cuda.Stream()
        got = []
        c.submit(packed)
        while True:
            r = c.acquire(st.cuda_stream)
            if r is None:
                break
            idx, dptr = r
            assert dptr is not None
            got.append(c.r1cs_quotient(idx, stream=st))
            c.release(idx, st.cuda_stream)
        fin = c.finish()
        assert (fin.status == 0).all() and len(got) == 4
        st.synchronize()
        for g in got:
            assert torch.equal(g.cpu(), want.cpu())
    finally:
        c.close()
