"""The pairing model (tests/pairing_model.py) without a GPU: the tower against flat F_q[w] / (w^12 - 18 w^6 + 82) arithmetic, every
literal of csrc/fq12_hd.h and csrc/pairing.cuh against its definition, the exponent chain, bilinearity, the model verifier on
trapdoor proofs of gadget circuits, the JSON forms of Proof and VerificationKey, pob_zkey_vk on written keys, and the new CLI forms'
argument matching."""
import json
import os
import random
import re
import zlib

import pytest

import g1_model as gm
import g2_model as g2m
import groth16_model as g16
import pairing_model as pm
import zkey_writer as zw
from helpers import suite
from test_groth16_cpu import _circuit, _quotient

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "proof-of-burn_b200", "csrc")
Q, R = pm.Q, pm.R_ORDER


# ---- the tower ------------------------------------------------------------------------------------------------------------------
def test_tower_against_flat_arithmetic():
    rng = random.Random(31)
    edge = [pm.ZERO, pm.ONE, pm.from_coeffs([Q - 1] * 12), (pm.random12(rng)[0], pm.Z6), (pm.Z6, pm.random12(rng)[1])]
    vals = edge + [pm.random12(rng) for _ in range(8)]
    for a in vals:
        for b in vals[:6]:
            assert pm.to_flat(pm.mul12(a, b)) == pm.flat_mul(pm.to_flat(a), pm.to_flat(b))
            assert pm.to_flat(pm.add12(a, b)) == [(x + y) % Q for x, y in zip(pm.to_flat(a), pm.to_flat(b))]
        if a != pm.ZERO:
            assert pm.mul12(a, pm.inv12(a)) == pm.ONE
        if a[0] != pm.Z6:
            assert pm.mul6(a[0], pm.inv6(a[0])) == pm.O6
    w = pm.to_flat(pm.W)
    assert w == [0, 1] + [0] * 10
    w6 = pm.to_flat(pm.pow12(pm.W, 6))
    assert w6 == pm.to_flat(pm.from_fq2(pm.XI))                       # w^6 = xi
    assert pm.to_flat(pm.from_fq2((0, 1))) == [Q - 9] + [0] * 5 + [1] + [0] * 5      # u = w^6 - 9
    a, b = pm.random12(rng), pm.random12(rng)
    assert pm.mul12(pm.mul12(a, b), pm.inv12(b)) == a
    assert pm.coeffs(pm.from_coeffs(range(12))) == tuple(range(12))


def test_frobenius_and_conjugation():
    rng = random.Random(32)
    a = pm.random12(rng)
    for k in (1, 2, 3):
        f = pm.frob(a, k)
        for half in range(2):
            for j in range(3):
                c = a[half][j] if k % 2 == 0 else pm.conj2(a[half][j])
                assert f[half][j] == pm.mul2(c, pm.frob_const(k, 2 * j + half))
    assert pm.frob(a, 6) == pm.conj12(a)
    for j in range(6):                                                # gamma_{2,j} lies in F_q; gamma_{2,3} = -1
        assert pm.frob_const(2, j)[1] == 0
    assert pm.frob_const(2, 3) == (Q - 1, 0)


def _literals(text, name):
    body = re.search(name + r"[^=]*=\s*\{(.*?)\};", text, re.S).group(1)
    return [int(v, 16) for v in re.findall(r"0x([0-9a-f]+)u", body)]


def _fq_of(limbs):
    return gm.from_mont(sum(v << (32 * i) for i, v in enumerate(limbs)))


def test_device_literals():
    """every constant of the device tower and pairing, against its definition"""
    text = open(os.path.join(CSRC, "fq12_hd.h")).read()
    body = re.search(r"FQ12_FROB\[3\]\[5\]\[2\]\[8\] = \{(.*?)\};", text, re.S).group(1)
    groups = re.findall(r"\{(0x[^{}]*|0)\}", body)
    assert len(groups) == 30
    for n, g in enumerate(groups):
        vals = [int(v, 16) for v in re.findall(r"0x([0-9a-f]+)u", g)] or [0] * 8
        j, k, c = n // 10 + 1, (n // 2) % 5 + 1, n % 2
        assert _fq_of(vals) == pm.frob_const(j, k)[c], (j, k, c)
    ptext = open(os.path.join(CSRC, "pairing.cuh")).read()
    b2 = re.search(r"pair_b2\(\) \{.*?C0\[8\] = \{(.*?)\};.*?C1\[8\] = \{(.*?)\};", ptext, re.S)
    assert tuple(_fq_of([int(v, 16) for v in re.findall(r"0x([0-9a-f]+)u", b2.group(k))]) for k in (1, 2)) == g2m.B2
    half = re.search(r"pair_two_inv\(\) \{.*?V\[8\] = \{(.*?)\};", ptext, re.S).group(1)
    assert _fq_of([int(v, 16) for v in re.findall(r"0x([0-9a-f]+)u", half)]) * 2 % Q == 1
    pos, neg = (int(v, 16) for v in re.search(r"PAIR_NAF_POS = 0x([0-9a-f]+)ull, PAIR_NAF_NEG = 0x([0-9a-f]+)ull", ptext).groups())
    assert int(re.search(r"PAIR_X = 0x([0-9a-f]+)ull", ptext).group(1), 16) == pm.X
    digits = [((pos >> i) & 1) - ((neg >> i) & 1) for i in range(64)]
    assert pos & neg == 0 and sum(d << i for i, d in enumerate(digits)) + (1 << 65) == pm.ATE     # digit 64 is 0, digit 65 is 1
    assert all(not (digits[i] and digits[i + 1]) for i in range(63))                              # non-adjacent
    assert int(re.search(r"PAIR_LINES = (\d+)", ptext).group(1)) == 65 + sum(1 for d in digits if d) + 2


def test_final_exponent_chain():
    """the hard part of the device's final exponentiation is exactly (q^4 - q^2 + 1) / r, not a multiple of it"""
    x = pm.X
    assert Q == 36 * x ** 4 + 36 * x ** 3 + 24 * x ** 2 + 6 * x + 1 and R == 36 * x ** 4 + 36 * x ** 3 + 18 * x ** 2 + 6 * x + 1
    l0, l1, l2 = -36 * x ** 3 - 30 * x ** 2 - 18 * x - 2, -36 * x ** 3 - 18 * x ** 2 - 12 * x + 1, 6 * x ** 2 + 1
    assert (Q ** 4 - Q ** 2 + 1) % R == 0
    assert l0 + l1 * Q + l2 * Q ** 2 + Q ** 3 == (Q ** 4 - Q ** 2 + 1) // R
    assert (Q ** 6 - 1) * (Q ** 2 + 1) * ((Q ** 4 - Q ** 2 + 1) // R) == pm.FINAL_EXP


# ---- the pairing ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def e_gen():
    return pm.pairing(gm.G, g2m.G)


def test_pairing_order_and_bilinearity(e_gen):
    assert e_gen != pm.ONE
    assert pm.pow12(e_gen, R) == pm.ONE
    rng = random.Random(33)
    for _ in range(2):
        a, b = rng.randrange(1, R), rng.randrange(1, R)
        assert pm.pairing(gm.mul(a, gm.G), g2m.mul(b, g2m.G)) == pm.pow12(e_gen, a * b % R)
    assert pm.pairing(None, g2m.G) == pm.ONE and pm.pairing(gm.G, None) == pm.ONE
    assert pm.multi_pairing([(gm.G, g2m.G), (gm.neg(gm.G), g2m.G)]) == pm.ONE


def test_point_outside_g2():
    p = pm.twist_point_outside_g2(34)
    assert g2m.on_curve(p) and g2m.mul(R, p, reduce=False) is not None


# ---- the model verifier on trapdoor proofs ---------------------------------------------------------------------------------------
def trapdoor_vk(S):
    """the verification key of a groth16_model.Setup as model points: IC_i = [(beta u_i + alpha v_i + w_i) / gamma] G1"""
    gi = pow(S.gamma, -1, R)
    return {"alpha1": gm.mul(S.alpha, gm.G), "beta2": g2m.mul(S.beta, g2m.G), "gamma2": g2m.mul(S.gamma, g2m.G),
            "delta2": g2m.mul(S.delta, g2m.G), "ic": [gm.mul(int(v) * gi, gm.G) for v in S.ic[:S.n_pub + 1]]}


@pytest.mark.parametrize("name", ["test_divide", "test_mask"])
def test_model_verifier(name, tmp_path):
    R1, W = _circuit(name, 1, tmp_path)
    rng = random.Random(zlib.crc32(name.encode()))
    S = g16.Setup(R1, *[rng.randrange(1, R) for _ in range(5)])
    assert S.n_pub >= 1
    vk = trapdoor_vk(S)
    q = _quotient(R1, W)
    a, b, c = S.proof_scalars(W, q, rng.randrange(R), rng.randrange(R))
    proof = (gm.mul(a, gm.G), g2m.mul(b, g2m.G), gm.mul(c, gm.G))
    pub = [int(v) for v in W[1:S.n_pub + 1]]
    assert pm.verify(vk, proof, pub)
    Wt = W.copy()                                                      # a tampered private witness entry
    j = next(j for j in range(S.n_pub + 1, len(W)) if len(R1.failing_rows(_bump(W, j))) > 0)
    Wt[j] = (Wt[j] + 1) % R
    at, bt, ct = S.proof_scalars(Wt, _quotient(R1, Wt), 0, 0)
    assert not pm.verify(vk, (gm.mul(at, gm.G), g2m.mul(bt, g2m.G), gm.mul(ct, gm.G)), pub)
    assert not pm.verify(vk, proof, [(pub[0] + 1) % R] + pub[1:])     # a wrong public input
    assert not pm.verify(vk, (proof[2], proof[1], proof[0]), pub)     # A and C swapped
    assert not pm.verify(vk, proof, [pub[0] + R] + pub[1:])           # a public input >= r is refused, not reduced


def _bump(W, j):
    Wt = W.copy()
    Wt[j] = (Wt[j] + 1) % R
    return Wt


# ---- JSON -------------------------------------------------------------------------------------------------------------------------
def test_json_round_trips():
    import pob_b200
    p = pob_b200.Proof(gm.mul(5, gm.G), g2m.mul(6, g2m.G), None)
    d = json.loads(json.dumps(p.to_json()))
    assert pob_b200.Proof.from_json(d) == p
    inf = pob_b200.Proof(None, None, gm.G)
    assert pob_b200.Proof.from_json(inf.to_json()) == inf
    for bad in (dict(d, pi_a=[d["pi_a"][0], d["pi_a"][1], "2"]), dict(d, pi_b=d["pi_b"][:2] + [["0", "1"]]),
                dict(d, pi_c=["0", "0", "0"]), dict(d, pi_b=[["0", "0"], ["0", "0"], ["0", "0"]])):
        with pytest.raises(ValueError):
            pob_b200.Proof.from_json(bad)
    vk = pob_b200.VerificationKey(gm.mul(3, gm.G), g2m.mul(4, g2m.G), g2m.mul(7, g2m.G), g2m.mul(8, g2m.G), [gm.G, None, gm.mul(9, gm.G)])
    d = {"protocol": "groth16", "curve": "bn128", "nPublic": 2, "vk_alpha_1": pob_b200._g1_json(vk.alpha1),
         "vk_beta_2": pob_b200._g2_json(vk.beta2), "vk_gamma_2": pob_b200._g2_json(vk.gamma2), "vk_delta_2": pob_b200._g2_json(vk.delta2),
         "vk_alphabeta_12": [[["1", "2"]] * 3] * 2, "IC": [pob_b200._g1_json(p) for p in vk.ic]}
    assert pob_b200.VerificationKey.from_json(json.loads(json.dumps(d))) == vk      # vk_alphabeta_12 is not trusted: ignored
    assert vk.n_pub == 2
    with pytest.raises(ValueError):
        pob_b200.VerificationKey.from_json(dict(d, nPublic=3))
    # a coordinate outside [0, q) is refused, never reduced into a valid key
    x, y = vk.ic[0]
    for bad in (dict(d, IC=[[str(x + Q), str(y), "1"]] + d["IC"][1:]), dict(d, vk_alpha_1=[str(x), str(-y), "1"]),
                dict(d, vk_delta_2=[[d["vk_delta_2"][0][0], str(Q)], d["vk_delta_2"][1], ["1", "0"]])):
        with pytest.raises(ValueError):
            pob_b200.VerificationKey.from_json(bad)
    with pytest.raises(ValueError):
        vk._replace(ic=[(x + Q, y)] + vk.ic[1:]).to_device()


# ---- pob_zkey_vk ------------------------------------------------------------------------------------------------------------------
def _vk_zkey(n_pub, seed):
    """a structurally valid .zkey with distinct, recognisable section-2 and section-3 bytes (points need not be on a curve here)"""
    rng = random.Random(seed)
    nv, dom = n_pub + 3, 8
    sec2 = {k: bytes(rng.randrange(256) for _ in range(zw.SEC2_SIZES[k])) for k in zw.SEC2_POINTS}
    ic = bytes(rng.randrange(256) for _ in range(64 * (n_pub + 1)))
    pts = {5: bytes(64 * nv), 6: bytes(64 * nv), 7: bytes(128 * nv), 8: bytes(64 * (nv - n_pub - 1)), 9: bytes(64 * dom)}
    return zw.Zkey(nv, n_pub, dom, sec2, ic, _no_entries(), pts)


def _no_entries():
    import numpy as np
    return np.zeros(0, dtype=zw.ENTRY)


def _zkey_vk(path, out_bytes):
    import ctypes
    import pob_b200
    buf = ctypes.create_string_buffer(max(out_bytes, 1))
    n = ctypes.c_uint32(0)
    rc = pob_b200.lib().pob_zkey_vk(os.fsencode(path), buf, out_bytes, ctypes.byref(n))
    return rc, buf.raw[:out_bytes], n.value


@pytest.mark.parametrize("n_pub", [0, 1, 5])
def test_zkey_vk_bytes(n_pub, tmp_path):
    Z = _vk_zkey(n_pub, n_pub)
    want = Z.sec2["alpha1"] + Z.sec2["beta2"] + Z.sec2["gamma2"] + Z.sec2["delta2"] + Z.ic
    for order in ([1, 2, 3, 4, 5, 6, 7, 8, 9], [9, 3, 7, 1, 8, 2, 6, 4, 5]):
        Z.order = order
        p = str(tmp_path / ("k%d.zkey" % order[0]))
        Z.write(p)
        rc, raw, n = _zkey_vk(p, len(want))
        assert (rc, raw, n) == (0, want, n_pub)
        rc, _, n = _zkey_vk(p, len(want) - 1)                          # a short out: refused, n_pub reported
        assert (rc, n) == (-1, n_pub)


def _set(**kw):
    def f(Z):
        for k, v in kw.items():
            setattr(Z, k, v)
    return f


@pytest.mark.parametrize("case", [
    ("magic", _set(magic=b"zkez"), -10), ("version", _set(version=2), -10), ("protocol", _set(protocol=2), -10),
    ("q", _set(q=zw.Q_MOD + 2), -10), ("r", _set(r=zw.R_MOD + 2), -10), ("n8q", _set(n8q=48), -10),
    ("missing3", _set(order=[1, 2, 4, 5, 6, 7, 8, 9]), -10), ("twice3", _set(order=[1, 2, 3, 3, 4, 5, 6, 7, 8, 9]), -10),
    ("size3", _set(size_delta={3: 64}), -10), ("domain", _set(domain=6), -10), ("truncated", _set(truncate=100), -6)],
    ids=lambda c: c[0])
def test_zkey_vk_refuses_what_zkey_info_refuses(case, tmp_path):
    import pob_b200
    Z = _vk_zkey(1, 7)
    case[1](Z)
    p = str(tmp_path / "bad.zkey")
    Z.write(p)
    with pytest.raises(pob_b200.PobError) as e:
        pob_b200.zkey_info(p)
    rc, _, _ = _zkey_vk(p, 4096)
    assert rc == case[2] == e.value.code
    with pytest.raises(pob_b200.PobError):
        pob_b200.VerificationKey.from_zkey(p)


def test_verification_key_from_zkey(tmp_path):
    import pob_b200
    pts = {"alpha1": gm.mul(3, gm.G), "beta1": gm.mul(4, gm.G), "beta2": g2m.mul(5, g2m.G), "gamma2": g2m.mul(6, g2m.G),
           "delta1": gm.mul(7, gm.G), "delta2": g2m.mul(8, g2m.G)}
    enc = lambda p: (g2m.encode_points([p]) if isinstance(p[0], tuple) else gm.encode_bases([p])).tobytes()
    ic = [gm.mul(11, gm.G), None]
    Z = _vk_zkey(1, 9)
    Z.sec2 = {k: enc(v) for k, v in pts.items()}
    Z.ic = gm.encode_bases(ic).tobytes()
    p = str(tmp_path / "k.zkey")
    Z.write(p)
    vk = pob_b200.VerificationKey.from_zkey(p)
    assert vk == pob_b200.VerificationKey(pts["alpha1"], pts["beta2"], pts["gamma2"], pts["delta2"], ic)


# ---- the CLI ------------------------------------------------------------------------------------------------------------------------
def test_cli_forms(tmp_path, capsys):
    """the new forms are matched before the legacy 3-argument form; malformed ones fall through to the usage message (exit 2); the
    existing forms keep their meaning"""
    import pob_b200
    assert pob_b200.main(["--verify", "vk.json", "public.json"]) == 2                     # a public.json without its proof.json
    assert pob_b200.main(["--export-vk", "key.zkey"]) == 2
    with pytest.raises(pob_b200.PobError):                                                # matched: reads the (missing) key file
        pob_b200.main(["--export-vk", str(tmp_path / "missing.zkey"), str(tmp_path / "vk.json")])
    assert not os.path.exists(tmp_path / "vk.json")
    with pytest.raises(FileNotFoundError):                                                # matched: reads the (missing) vk file
        pob_b200.main(["--verify", str(tmp_path / "vk.json"), "p.json", "q.json"])
    out = str(tmp_path / "c.r1cs")                                                        # an old form, unchanged
    assert pob_b200.main([suite("test_divide")["main"], "--r1cs", out, "--O1"]) == 0
    assert os.path.getsize(out) > 0
    capsys.readouterr()
