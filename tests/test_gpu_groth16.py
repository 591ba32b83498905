"""Groth16 proofs on the GPU (pob_groth16_prove) checked exactly, with no pairing: the key comes from a test-only trusted setup whose
trapdoor the test knows (tests/groth16_model.py), built on the GPU by the test probe's fixed-base [k_i]G (tests/devprobe/g2_probe.cu).
Each proof point must equal [a]G1, [b]G2, [c]G1 for the scalars the model predicts, and those scalars must satisfy the Groth16
equation in Fr, which is the pairing check by bilinearity.  A tampered witness must still give the predicted proof, and fail the
equation.  On the main shape the key is tiled from 1024 points of known discrete logarithm (not a valid key), and the prediction
comes from class sums of w and q (tests/test_gpu_msm.py)."""
import os
import random
import sys
import zlib

import numpy as np
import pytest

import g1_model as gm
import g2_model as g2m
import groth16_model as g16
import quotient_model as qm
from helpers import cuda_poke, suite
from r1cs_reader import R1cs, limbs_of, witness_ints
from test_gpu_msm import MAIN_SHAPE, TILE, _class_sums, _dev, _witness_tensor

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

pytestmark = pytest.mark.gpu

P = qm.P
SUITES = ["test_poseidon_2", "test_divide", "test_mask", "test_selector", "test_num_2_bits_safe_32", "test_is_in_range",
          "test_assert_less_than", "test_rlp_integer_1"]


def _scalars(vals):
    return _dev(limbs_of(vals, P))


def _key(S):
    """the Groth16Key of a groth16_model.Setup, on the GPU"""
    import g2
    import pob_b200
    g1 = lambda v: g2.fixed_base(1, _scalars(v))
    g2p = lambda v: g2.fixed_base(2, _scalars(v))
    return pob_b200.Groth16Key(alpha1=g1([S.alpha]), beta1=g1([S.beta]), delta1=g1([S.delta]), beta2=g2p([S.beta]), delta2=g2p([S.delta]),
                               a=g1(S.a_keys), b1=g1(S.b_keys), b2=g2p(S.b_keys), c=g1(S.c_keys), h=g1(S.h_keys))


def _expect(S, W, q, r, s, proof):
    """the proof equals the model's prediction; returns whether the prediction satisfies the Groth16 equation"""
    a, b, c = S.proof_scalars(W, q, r, s)
    assert proof.a == gm.mul(a, gm.G), "A"
    assert proof.b == g2m.mul(b, g2m.G), "B"
    assert proof.c == gm.mul(c, gm.G), "C"
    return S.verify(a, b, c, W[:S.n_pub + 1])


def _setup(c, main, opt, tmp_path):
    import pob_b200
    f = str(tmp_path / "c.r1cs")
    pob_b200.write_r1cs(main, f, opt=opt)
    R = R1cs(f)
    rng = random.Random(zlib.crc32(main.encode()) + opt)
    S = g16.Setup(R, *[rng.randrange(1, P) for _ in range(5)])
    assert (S.n_vars, S.n_pub, S.log_n) == (c.n_signals, c.n_outputs, c.r1cs_domain())
    return R, S, rng


def _prove_and_tamper(c, R, S, rng, exact_q):
    """proofs with r = s = 0 and random r, s satisfy the equation; after one private witness entry is overwritten the proof still
    equals the prediction (q from pob_r1cs_quotient) and fails it"""
    key = _key(S)
    W = witness_ints(c.witness(0))
    q = qm.quotient(*R.products(W), W[:S.n_pub + 1], R.m) if exact_q else witness_ints(c.r1cs_quotient(0).cpu().numpy())
    for r, s in ((0, 0), (rng.randrange(1 << 256), rng.randrange(1 << 256)), (rng.randrange(P), P - 1)):
        assert _expect(S, W, q, r, s, c.groth16_prove(0, key, r=r, s=s)), (r, s)
    used = sorted(set(int(x) for x in R.wire) - set(range(S.n_pub + 1)))
    rng.shuffle(used)
    for j in used:
        Wt = W.copy()
        Wt[j] = (Wt[j] + 1) % P
        if len(R.failing_rows(Wt)) > 0:
            break
    cuda_poke(c.witness_device_ptr(0), j, Wt[j])
    assert (witness_ints(c.witness(0)) == Wt).all()
    qt = witness_ints(c.r1cs_quotient(0).cpu().numpy())
    r, s = rng.randrange(P), rng.randrange(P)
    assert not _expect(S, Wt, qt, r, s, c.groth16_prove(0, key, r=r, s=s))


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
@pytest.mark.parametrize("name", SUITES)
def test_gadget_proofs(name, opt, tmp_path):
    import pob_b200
    s = suite(name)
    c = pob_b200.Circuit(s["main"], max_slots=1, opt=opt)
    try:
        assert c.run([next(x for x in s["cases"] if x["expected"] is not None)["input"]]).status[0] == 0
        R, S, rng = _setup(c, s["main"], opt, tmp_path)
        _prove_and_tamper(c, R, S, rng, exact_q=True)
    finally:
        c.close()


def test_spend_reduced(tmp_path):
    """Spend(31), reduced witness: 259,945 wires over a 2^18 domain"""
    import pob_b200
    c = pob_b200.Circuit("Spend(31)", max_slots=1, opt=1)
    try:
        assert c.run([suite("test_spend")["cases"][0]["input"]]).status[0] == 0
        R, S, rng = _setup(c, "Spend(31)", 1, tmp_path)
        assert S.log_n == 18
        _prove_and_tamper(c, R, S, rng, exact_q=False)
    finally:
        c.close()


# ---- tiled keys of known discrete logarithms -----------------------------------------------------------------------------------
_TILES = {}


def _tile(group):
    """TILE points [t_k]G of the group and their t_k"""
    import g2
    if group not in _TILES:
        rng = random.Random(4096 + group)
        ts = [rng.randrange(1, P) for _ in range(TILE)]
        _TILES[group] = (g2.fixed_base(group, _scalars(ts)), ts)
    return _TILES[group]


def _tiled(group, n):
    import torch
    B, _ = _tile(group)
    return B.view(torch.int64).repeat((n + TILE - 1) // TILE, 1)[:n].contiguous().view(torch.uint64)


def _tiled_key(c, consts):
    """a key whose points are tiled: alpha, beta, delta from consts, every section a repetition of _tile"""
    import g2
    import pob_b200
    nv, npub, n = c.n_signals, c.n_outputs, 1 << c.r1cs_domain()
    al, be, de = consts
    one = lambda grp, v: g2.fixed_base(grp, _scalars([v]))
    a = _tiled(1, nv)
    return pob_b200.Groth16Key(alpha1=one(1, al), beta1=one(1, be), delta1=one(1, de), beta2=one(2, be), delta2=one(2, de),
                               a=a, b1=a, b2=_tiled(2, nv), c=_tiled(1, nv - npub - 1), h=_tiled(1, n))


def _tiled_prediction(c, consts, w, q, r, s):
    """(A, B, C) of a tiled-key proof, from class sums of w (an (n_vars, 4) tensor) and q"""
    import pob_b200
    al, be, de = consts
    t1, t2 = _tile(1)[1], _tile(2)[1]
    dot = lambda ts, S: sum(t * v for t, v in zip(ts, S)) % P
    Sw = _class_sums(w)
    sa, sb1, sb2 = dot(t1, Sw), dot(t1, Sw), dot(t2, Sw)
    sc, sh = dot(t1, _class_sums(w[c.n_outputs + 1:].contiguous())), dot(t1, _class_sums(q))
    r, s = r % P, s % P
    a = (al + sa + r * de) % P
    b1 = (be + sb1 + s * de) % P
    b = (be + sb2 + s * de) % P
    cc = (sc + sh + s * a + r * b1 - r * s * de) % P
    return pob_b200.Proof(gm.mul(a, gm.G), g2m.mul(b, g2m.G), gm.mul(cc, gm.G))


def test_main_shape_reduced():
    """main_proof_of_burn, reduced witness (21,454,051 wires, 2^25 domain): sizes and the work layout at scale"""
    import torch
    import pob_b200
    from pob_b200 import synth
    packed = synth.pack_instances(synth.make_batch(1, MAIN_SHAPE, seed=4242), MAIN_SHAPE)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1, opt=1)
    try:
        assert c.run_packed(packed).status[0] == 0 and c.n_signals == 21454051 and c.r1cs_domain() == 25
        rng = random.Random(2525)
        consts = [rng.randrange(1, P) for _ in range(3)]
        key = _tiled_key(c, consts)
        work = torch.empty(c.groth16_work_bytes(), dtype=torch.uint8, device="cuda")
        r, s = rng.randrange(P), rng.randrange(P)
        got = c.groth16_prove(0, key, r=r, s=s, work=work)
        w = _witness_tensor(c.witness_device_ptr(0), c.n_signals)
        q = c.r1cs_quotient(0)
        assert got == _tiled_prediction(c, consts, w, q, r, s)
        del key, work, q
        torch.cuda.empty_cache()
    finally:
        c.close()


def test_handoff_on_a_consumer_stream():
    """acquire(stream) / prove / release(stream) on a non-blocking stream with a sleep queued before each proof: every proof equals
    the synchronous one of the same witness, for four distinct witnesses"""
    import torch
    import pob_b200
    from test_gpu_shapes import _spend_inputs
    inputs = _spend_inputs(4, seed=31415)
    c = pob_b200.Circuit("Spend(31)", max_slots=2, opt=1)
    try:
        rng = random.Random(77)
        consts = [rng.randrange(1, P) for _ in range(3)]
        key = _tiled_key(c, consts)
        r, s = rng.randrange(P), rng.randrange(P)
        want = []
        for inp in inputs:
            assert c.run([inp]).status[0] == 0
            want.append(c.groth16_prove(0, key, r=r, s=s))
            w = _witness_tensor(c.witness_device_ptr(0), c.n_signals)
            assert want[-1] == _tiled_prediction(c, consts, w, c.r1cs_quotient(0), r, s)
        assert len(set(want)) == 4
        st = torch.cuda.Stream()
        got = []
        c.submit(c.pack(inputs))
        while True:
            a = c.acquire(st.cuda_stream)
            if a is None:
                break
            idx, _ = a
            with torch.cuda.stream(st):
                torch.cuda._sleep(10 ** 8)
            out = c.groth16_prove(idx, key, r=r, s=s, stream=st)
            c.release(idx, st.cuda_stream)
            got.append((idx, out))
        assert (c.finish().status == 0).all()
        st.synchronize()
        assert sorted(i for i, _ in got) == [0, 1, 2, 3]
        for idx, out in got:
            assert pob_b200.proof_from_limbs(out.cpu().tolist()) == want[idx]
    finally:
        c.close()


def test_errors_before_anything_runs(tmp_path):
    import ctypes
    import torch
    import pob_b200
    s = suite("test_poseidon_2")
    c = pob_b200.Circuit(s["main"], max_slots=1, opt=1)
    try:
        assert c.run([s["cases"][0]["input"]]).status[0] == 0
        R, S, rng = _setup(c, s["main"], 1, tmp_path)
        key = _key(S)
        need = c.groth16_work_bytes()
        work = torch.zeros(need + 512, dtype=torch.uint8, device="cuda")
        proof = torch.zeros(64, dtype=torch.uint64, device="cuda")
        L = pob_b200.lib()
        rl = np.zeros(4, dtype=np.uint64)
        base = dict(n_vars=c.n_signals, n_pub=c.n_outputs, log_n=c.r1cs_domain(), **{f: getattr(key, f).data_ptr() for f in key._fields})

        def call(kc=None, pr=None, wk=None, wb=None, index=0, r=rl.ctypes.data, k=None):
            d = dict(base, **(k or {}))
            kc = pob_b200.Groth16KeyC(d["n_vars"], d["n_pub"], d["log_n"], *[d[f] for f in key._fields]) if kc is None else kc
            return L.pob_groth16_prove(c._h, index, ctypes.byref(kc) if kc is not False else None, r, rl.ctypes.data,
                                       proof.data_ptr() if pr is None else pr, work.data_ptr() if wk is None else wk,
                                       need if wb is None else wb, None)
        assert call() == 0
        torch.cuda.synchronize()
        want = proof.clone()
        proof.zero_()
        work.fill_(0xA5)
        torch.cuda.synchronize()
        W0, P0 = work.data_ptr(), proof.data_ptr()
        bad = [dict(k={"n_vars": c.n_signals + 1}), dict(k={"n_pub": c.n_outputs + 1}), dict(k={"log_n": c.r1cs_domain() + 1}),
               dict(kc=False), dict(r=None), dict(pr=0), dict(wk=0), dict(wb=need - 1), dict(pr=W0 + 256), dict(pr=W0 + need - 16),
               dict(pr=P0 + 8), dict(wk=W0 + 8)]
        bad += [dict(k={f: 0}) for f in key._fields] + [dict(k={f: getattr(key, f).data_ptr() + 8}) for f in key._fields]
        for k, b in enumerate(bad):
            rc = call(**b)
            assert rc == -1, (k, b, rc, L.pob_last_error())
        torch.cuda.synchronize()
        assert not proof.view(torch.int64).any() and (work == 0xA5).all()   # nothing ran
        assert call(index=1) == pob_b200.E_RANGE
        assert call() == 0
        torch.cuda.synchronize()
        assert torch.equal(proof, want)
        W = witness_ints(c.witness(0))
        q = qm.quotient(*R.products(W), W[:S.n_pub + 1], R.m)
        assert _expect(S, W, q, 0, 0, pob_b200.proof_from_limbs(want.cpu().tolist()[:32]))
    finally:
        c.close()
