"""pob_groth16_verify: proofs pob_groth16_prove writes on trapdoor keys (tests/groth16_model.py) verify as the device buffers they are,
each rejection has its own status, batches of simulated proofs with invalid ones at known positions get every status right in order,
the acquire -> prove -> verify -> release hand-off equals the synchronous result, bad arguments are refused before anything runs, and
the CLI exports a verification key and verifies with it."""
import ctypes
import json
import os
import random
import sys

import numpy as np
import pytest

import g1_model as gm
import g2_model as g2m
import pairing_model as pm
from helpers import cuda_poke, suite
from r1cs_reader import limbs_of, witness_ints
from test_gpu_groth16 import SUITES, _key, _scalars, _setup
from test_gpu_msm import _dev

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devprobe"))

pytestmark = pytest.mark.gpu

Q, R = pm.Q, pm.R_ORDER
OK, FAIL, BAD_POINT, BAD_SUBGROUP, BAD_PUBLIC, BAD_KEY = range(6)


def _vk(S):
    """the DeviceVerificationKey of a groth16_model.Setup: IC_i = [(beta u_i + alpha v_i + w_i) / gamma] G1"""
    import g2
    import pob_b200
    gi = pow(S.gamma, -1, R)
    g1 = lambda v: g2.fixed_base(1, _scalars(v))
    g2p = lambda v: g2.fixed_base(2, _scalars(v))
    return pob_b200.DeviceVerificationKey(S.n_pub, g1([S.alpha]), g2p([S.beta]), g2p([S.gamma]), g2p([S.delta]),
                                          g1([int(v) * gi % R for v in S.ic[:S.n_pub + 1]]))


def _pub_tensor(vals):
    return _dev(limbs_of(vals, 1 << 256)) if vals else None


def _verify(vk, proofs, pubs):
    import pob_b200
    return list(pob_b200.groth16_verify(vk, proofs, pubs if isinstance(pubs, list) or pubs is None else pubs))


def _prove_verify_tamper(c, R1, S, rng):
    import torch
    import pob_b200
    key, vk = _key(S), _vk(S)
    W = witness_ints(c.witness(0))
    pub = _pub_tensor([int(v) for v in W[1:S.n_pub + 1]])
    out = torch.empty(32, dtype=torch.uint64, device="cuda")
    for r, s in ((0, 0), (rng.randrange(R), rng.randrange(R))):
        c.groth16_prove(0, key, r=r, s=s, out=out)
        assert _verify(vk, out, pub) == [OK], (r, s)
    used = sorted(set(int(x) for x in R1.wire) - set(range(S.n_pub + 1)))
    rng.shuffle(used)
    for j in used:
        Wt = W.copy()
        Wt[j] = (Wt[j] + 1) % R
        if len(R1.failing_rows(Wt)) > 0:
            break
    cuda_poke(c.witness_device_ptr(0), j, Wt[j])
    c.groth16_prove(0, key, out=out)
    assert _verify(vk, out, pub) == [FAIL]


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
@pytest.mark.parametrize("name", SUITES)
def test_real_proofs_verify(name, opt, tmp_path):
    import pob_b200
    s = suite(name)
    c = pob_b200.Circuit(s["main"], max_slots=1, opt=opt)
    try:
        assert c.run([next(x for x in s["cases"] if x["expected"] is not None)["input"]]).status[0] == 0
        R1, S, rng = _setup(c, s["main"], opt, tmp_path)
        _prove_verify_tamper(c, R1, S, rng)
    finally:
        c.close()


def test_spend_reduced_verifies(tmp_path):
    import pob_b200
    c = pob_b200.Circuit("Spend(31)", max_slots=1, opt=1)
    try:
        assert c.run([suite("test_spend")["cases"][0]["input"]]).status[0] == 0
        R1, S, rng = _setup(c, "Spend(31)", 1, tmp_path)
        _prove_verify_tamper(c, R1, S, rng)
    finally:
        c.close()


# ---- simulated proofs: a b = alpha beta + gamma (k_0 + sum_j pub_j k_j) + c delta, IC_j = [k_j] G1 ----------------------------------
class Sim:
    def __init__(self, n_pub, seed):
        import g2
        import pob_b200
        self.rng = random.Random(seed)
        self.n_pub = n_pub
        self.alpha, self.beta, self.gamma, self.delta = (self.rng.randrange(1, R) for _ in range(4))
        self.k = [self.rng.randrange(1, R) for _ in range(n_pub + 1)]
        g1 = lambda v: g2.fixed_base(1, _scalars(v))
        g2p = lambda v: g2.fixed_base(2, _scalars(v))
        self.vk = pob_b200.DeviceVerificationKey(n_pub, g1([self.alpha]), g2p([self.beta]), g2p([self.gamma]), g2p([self.delta]), g1(self.k))

    def scalars(self, n):
        di = pow(self.delta, -1, R)
        a = [self.rng.randrange(1, R) for _ in range(n)]
        b = [self.rng.randrange(1, R) for _ in range(n)]
        pubs = [[self.rng.randrange(R) for _ in range(self.n_pub)] for _ in range(n)]
        c = [(x * y - self.alpha * self.beta - self.gamma * (self.k[0] + sum(p * k for p, k in zip(ps, self.k[1:])))) * di % R
             for x, y, ps in zip(a, b, pubs)]
        return a, b, c, pubs

    def proofs(self, a, b, c):
        """(n, 32) uint64 CUDA tensor of canonical proofs [a]G1, [b]G2, [c]G1"""
        import torch
        import g2
        A, B, C = (g2.fixed_base(g, _scalars(v)).view(torch.int64) for g, v in ((1, a), (2, b), (1, c)))
        raw = torch.cat([A, B, C], dim=1).cpu().numpy().view(np.uint64)
        return _dev(_canonical(raw))

    def full_vk(self):
        import pob_b200
        return pob_b200.VerificationKey(gm.mul(self.alpha, gm.G), g2m.mul(self.beta, g2m.G), g2m.mul(self.gamma, g2m.G),
                                        g2m.mul(self.delta, g2m.G), [gm.mul(k, gm.G) for k in self.k])


def _canonical(mont):
    """Montgomery-form limbs -> canonical, element by element (4 limbs each)"""
    ri = pow(1 << 256, -1, Q)
    v = mont.reshape(-1, 4)
    ints = [int(a) | int(b) << 64 | int(c) << 128 | int(d) << 192 for a, b, c, d in v.tolist()]
    return limbs_of([x * ri % Q for x in ints], Q).reshape(mont.shape)


def _set_fq(t, row, word, value):
    """overwrite the F_q element at uint64 offset word of proof row with value (t: the int64 view of the proofs)"""
    import torch
    t[row, word:word + 4] = _dev(limbs_of([value], 1 << 256)).view(torch.int64)[0]


def _get_fq(t, row, word):
    v = t[row, word:word + 4].cpu().numpy().view(np.uint64)
    return sum(int(x) << (64 * k) for k, x in enumerate(v))


def test_each_rejection():
    import torch
    import pob_b200
    sim = Sim(2, 51)
    a, b, c, pubs = sim.scalars(12)
    P = sim.proofs(a, b, c).view(torch.int64)
    out_g2 = pm.twist_point_outside_g2(52)
    exp = [OK] * 12
    pubs[1][0] = (pubs[1][0] + 1) % R; exp[1] = FAIL                      # wrong public input
    pubs[2][1] = pubs[2][1] + R; exp[2] = BAD_PUBLIC                      # public input >= r
    P[3, 0:8], P[3, 24:32] = P[3, 24:32].clone(), P[3, 0:8].clone(); exp[3] = FAIL     # A and C swapped
    P[4, 0:8] = 0; exp[4] = FAIL                                          # A = O
    _set_fq(P, 5, 0, _get_fq(P, 5, 0) + Q); exp[5] = BAD_POINT            # a coordinate >= q
    _set_fq(P, 6, 28, (_get_fq(P, 6, 28) + 1) % Q); exp[6] = BAD_POINT    # C off its curve
    _set_fq(P, 7, 12, (_get_fq(P, 7, 12) + 1) % Q); exp[7] = BAD_POINT    # B off its curve
    for k, v in enumerate((out_g2[0][0], out_g2[0][1], out_g2[1][0], out_g2[1][1])):
        _set_fq(P, 8, 8 + 4 * k, v)
    exp[8] = BAD_SUBGROUP                                                 # B on the twist, outside G2
    P[9, 8:24] = 0; exp[9] = FAIL                                         # B = O
    _set_fq(P, 10, 28, Q - 1); exp[10] = BAD_POINT                        # y = q - 1: off the curve
    P = P.view(torch.uint64)
    assert _verify(sim.vk, P, _pub_tensor([x for p in pubs for x in p])) == exp
    # the same verdicts through the int interface
    vk_int = sim.full_vk()
    limbs = P.view(torch.int64).cpu().numpy().view(np.uint64)
    proofs = [pob_b200.proof_from_limbs(limbs[i].tolist()) for i in range(12)]
    assert list(pob_b200.groth16_verify(vk_int, proofs, pubs)) == exp
    # a malformed key: every proof gets BAD_KEY
    bad = sim.vk._replace(gamma2=sim.vk.gamma2.clone())
    bad.gamma2.view(torch.int64)[0, 1] ^= 1 << 17                         # a flipped bit in gamma2
    assert _verify(bad, P, _pub_tensor([x for p in pubs for x in p])) == [BAD_KEY] * 12
    bad = sim.vk._replace(beta2=_dev(g2m.encode_points([out_g2])))        # beta2 outside G2
    assert _verify(bad, P, _pub_tensor([x for p in pubs for x in p])) == [BAD_KEY] * 12
    bad = sim.vk._replace(delta2=torch.zeros((1, 16), dtype=torch.int64, device="cuda").view(torch.uint64))   # delta2 = O
    assert _verify(bad, P, _pub_tensor([x for p in pubs for x in p])) == [BAD_KEY] * 12


@pytest.mark.parametrize("n", [1, 2, 1000, 1 << 17])
def test_batches(n):
    """distinct valid simulated proofs mixed with invalid ones at known positions; every status in order"""
    import torch
    sim = Sim(1 if n != 1000 else 3, 60 + n)
    a, b, c, pubs = sim.scalars(n)
    rng = random.Random(n)
    exp = [OK] * n
    bad = set(rng.sample(range(n), min(n - 1, max(1, n // 50)))) if n > 1 else set()
    for i in bad:
        kind = rng.randrange(3)
        if kind == 0:
            c[i] = (c[i] + 1) % R; exp[i] = FAIL
        elif kind == 1:
            pubs[i][0] += R; exp[i] = BAD_PUBLIC
        else:
            a[i] = 0; exp[i] = FAIL                                       # A = O
    P = sim.proofs(a, b, c)
    st = _verify(sim.vk, P, _pub_tensor([x for p in pubs for x in p]))
    assert st == exp
    if n == 1:
        c[0] = (c[0] + 5) % R
        assert _verify(sim.vk, sim.proofs(a, b, c), _pub_tensor(pubs[0])) == [FAIL]


def test_handoff_prove_verify(tmp_path):
    """acquire -> prove -> verify -> release on a non-blocking stream with a sleep before each proof, over four witnesses"""
    import torch
    import pob_b200
    s = suite("test_poseidon_2")
    inputs = [x["input"] for x in s["cases"] if x["expected"] is not None][:4]
    assert len(inputs) == 4
    c = pob_b200.Circuit(s["main"], max_slots=2, opt=1)
    try:
        assert c.run([inputs[0]]).status[0] == 0
        R1, S, rng = _setup(c, s["main"], 1, tmp_path)
        key, vk = _key(S), _vk(S)
        r, sb = rng.randrange(R), rng.randrange(R)
        pubs, want = [], []
        for inp in inputs:
            res = c.run([inp])
            assert res.status[0] == 0
            pubs.append([int(v) % R for v in res.outputs[0]])
            want.append(c.groth16_prove(0, key, r=r, s=sb))
        wst = list(pob_b200.groth16_verify(vk, want, pubs))
        assert wst == [OK] * 4
        st = torch.cuda.Stream()
        c.submit(c.pack(inputs))
        got = []
        while True:
            a = c.acquire(st.cuda_stream)
            if a is None:
                break
            idx, _ = a
            with torch.cuda.stream(st):
                torch.cuda._sleep(10 ** 8)
            out = c.groth16_prove(idx, key, r=r, s=sb, stream=st)
            status = pob_b200.groth16_verify(vk, out, _pub_tensor(pubs[idx]), stream=st)
            c.release(idx, st.cuda_stream)
            got.append((idx, out, status))
        assert (c.finish().status == 0).all()
        st.synchronize()
        assert sorted(i for i, _, _ in got) == [0, 1, 2, 3]
        for idx, out, status in got:
            assert pob_b200.proof_from_limbs(out.cpu().tolist()) == want[idx]
            assert int(status[0]) == wst[idx]
    finally:
        c.close()


def test_argument_errors():
    import torch
    import pob_b200
    sim = Sim(1, 70)
    a, b, c, pubs = sim.scalars(4)
    P = sim.proofs(a, b, c)
    pub = _pub_tensor([x for p in pubs for x in p])
    need = pob_b200.groth16_verify_work_bytes(1, 4)
    work = torch.zeros(need + 256, dtype=torch.uint8, device="cuda")
    status = torch.full((8,), 9, dtype=torch.int32, device="cuda")
    L = pob_b200.lib()
    vk = sim.vk
    base = dict(n_pub=1, alpha1=vk.alpha1.data_ptr(), beta2=vk.beta2.data_ptr(), gamma2=vk.gamma2.data_ptr(), delta2=vk.delta2.data_ptr(),
                ic=vk.ic.data_ptr())
    torch.cuda.synchronize()

    def call(kc=None, k=None, pr=None, pu=None, n=4, stt=None, wk=None, wb=None):
        d = dict(base, **(k or {}))
        kc = pob_b200.Groth16VkC(d["n_pub"], d["alpha1"], d["beta2"], d["gamma2"], d["delta2"], d["ic"]) if kc is None else kc
        return L.pob_groth16_verify(0, ctypes.byref(kc) if kc is not False else None, P.data_ptr() if pr is None else pr,
                                    pub.data_ptr() if pu is None else pu, n, status.data_ptr() if stt is None else stt,
                                    work.data_ptr() if wk is None else wk, need if wb is None else wb, None)
    W0, S0 = work.data_ptr(), status.data_ptr()
    bad = [dict(kc=False), dict(pr=0), dict(stt=0), dict(wk=0), dict(n=0), dict(wb=need - 1), dict(pr=P.data_ptr() + 8),
           dict(pu=pub.data_ptr() + 8), dict(wk=W0 + 8), dict(stt=S0 + 2), dict(stt=P.data_ptr() + 64), dict(stt=pub.data_ptr()),
           dict(stt=W0 + 128), dict(wk=P.data_ptr()), dict(stt=vk.ic.data_ptr() + 64), dict(stt=vk.gamma2.data_ptr()),
           dict(wk=vk.ic.data_ptr()), dict(wk=vk.alpha1.data_ptr() - need + 16)]
    bad += [dict(k={f: 0}) for f in ("alpha1", "beta2", "gamma2", "delta2", "ic")]
    bad += [dict(k={f: base[f] + 8}) for f in ("alpha1", "beta2", "gamma2", "delta2", "ic")]
    for j, b_ in enumerate(bad):
        assert call(**b_) == -1, (j, b_, L.pob_last_error())
    assert L.pob_groth16_verify(0, ctypes.byref(pob_b200.Groth16VkC(1, *[base[f] for f in ("alpha1", "beta2", "gamma2", "delta2", "ic")])),
                                P.data_ptr(), None, 4, S0, W0, need, None) == -1     # publics NULL with n_pub > 0
    torch.cuda.synchronize()
    assert (status == 9).all() and not work.any()                         # nothing ran
    assert call() == 0
    assert status[:4].tolist() == [OK] * 4


# ---- the CLI and the exported key -----------------------------------------------------------------------------------------------------
def test_cli_export_and_verify(tmp_path, capsys):
    import secrets
    import pob_b200
    from test_gpu_zkey import _zkey
    s = suite("test_poseidon_2")
    c = pob_b200.Circuit(s["main"], max_slots=1, opt=1)
    try:
        assert c.run([s["cases"][0]["input"]]).status[0] == 0
        R1, S, rng = _setup(c, s["main"], 1, tmp_path)
        Z = _zkey(S, R1)
    finally:
        c.close()
    zk = str(tmp_path / "k.zkey")
    Z.write(zk)
    inp, pj, uj, vkj = (str(tmp_path / f) for f in ("in.json", "proof.json", "public.json", "vk.json"))
    json.dump(s["cases"][0]["input"], open(inp, "w"))
    assert pob_b200.main([s["main"], "--prove", zk, inp, pj, uj, "--O1"]) == 0
    assert pob_b200.main(["--export-vk", zk, vkj]) == 0
    vk = json.load(open(vkj))
    assert vk["nPublic"] == S.n_pub and len(vk["IC"]) == S.n_pub + 1 and vk["protocol"] == "groth16"
    want = pm.pairing(gm.mul(S.alpha, gm.G), g2m.mul(S.beta, g2m.G))
    ab = vk["vk_alphabeta_12"]
    assert tuple(int(ab[h][j][k]) for h in range(2) for j in range(3) for k in range(2)) == pm.coeffs(want)
    capsys.readouterr()
    assert pob_b200.main(["--verify", vkj, uj, pj]) == 0
    assert capsys.readouterr().out.strip().endswith("OK")
    pub = json.load(open(uj))
    bad = str(tmp_path / "public_bad.json")
    json.dump([str((int(pub[0]) + 1) % R)] + pub[1:], open(bad, "w"))
    assert pob_b200.main(["--verify", vkj, uj, pj, bad, pj]) == 1
    lines = capsys.readouterr().out.strip().splitlines()
    assert lines[-2].endswith("OK") and lines[-1].endswith("FAIL")


def test_stream_with_int_key_and_host_inputs():
    """a VerificationKey of ints and host lists with a stream held back by a sleep: the key and the inputs go to the device on that
    stream, so the verdicts are right when the stream reaches them, and nothing the call allocated is reused before"""
    import torch
    import pob_b200
    sim = Sim(2, 80)
    a, b, c, pubs = sim.scalars(6)
    P = sim.proofs(a, b, c)
    limbs = P.view(torch.int64).cpu().numpy().view(np.uint64)
    proofs = [pob_b200.proof_from_limbs(limbs[i].tolist()) for i in range(6)]
    pubs[4][1] = (pubs[4][1] + 1) % R
    want = [OK, OK, OK, OK, FAIL, OK]
    vk = sim.full_vk()
    assert list(pob_b200.groth16_verify(vk, proofs, pubs)) == want
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(10 ** 8)
    status = pob_b200.groth16_verify(vk, proofs, pubs, stream=st)
    junk = [torch.full((1 << 16,), -1, dtype=torch.int64, device="cuda") for _ in range(8)]   # reuse freed blocks on the default stream
    torch.cuda.synchronize()
    assert status.tolist() == want
    del junk


def test_python_argument_checks():
    import torch
    import pob_b200
    sim = Sim(1, 81)
    a, b, c, pubs = sim.scalars(4)
    P = sim.proofs(a, b, c)
    pub = _pub_tensor([x for p in pubs for x in p])
    short = torch.zeros(3, dtype=torch.int32, device="cuda")
    wide = torch.zeros(4, dtype=torch.int64, device="cuda")
    for kw in (dict(status=short), dict(status=wide), dict(status=torch.zeros(4, dtype=torch.int32)),
               dict(work=torch.zeros(16, dtype=torch.uint8, device="cuda"))):
        with pytest.raises(ValueError):
            pob_b200.groth16_verify(sim.vk, P, pub, **kw)
    with pytest.raises(ValueError):
        pob_b200.groth16_verify(sim.vk._replace(ic=sim.vk.ic[:1]), P, pub)                    # IC shorter than n_pub + 1 points
    with pytest.raises(ValueError):
        pob_b200.groth16_verify(sim.vk._replace(gamma2=sim.vk.gamma2.cpu()), P, pub)          # a key point not on the device
    assert list(pob_b200.groth16_verify(sim.vk, P, pub, status=torch.zeros(8, dtype=torch.int32, device="cuda"))) == [OK] * 4
