"""pob_zkey_load on the GPU: keys written by tests/zkey_writer.py from the test-only trusted setup (tests/groth16_model.py) or from tiled
points, loaded through a staging ring whose buffers cut entries and points, byte-compared with the file, checked, and proved from.
Every corruption of the coefficients or the points must be found, and named in the report."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import g1_model as gm
import g2_model as g2m
import quotient_model as qm
import zkey_writer as zw
from helpers import suite
from r1cs_reader import witness_ints
from test_gpu_groth16 import SUITES, _expect, _key, _scalars, _setup, _tile

pytestmark = pytest.mark.gpu

P = qm.P
HERE = os.path.dirname(os.path.abspath(__file__))
ODD_STAGING = 4 * 1237                  # 1237-byte buffers: not a multiple of 44, 64 or 128


def _b(t):
    return t.cpu().numpy().tobytes()


def _zkey(S, R):
    """the Zkey of a groth16_model.Setup, points from the GPU probe"""
    import g2
    key = _key(S)
    gi = pow(S.gamma, P - 2, P)
    ic = g2.fixed_base(1, _scalars([int(v) * gi % P for v in S.ic[:S.n_pub + 1]]))
    sec2 = {"alpha1": _b(key.alpha1), "beta1": _b(key.beta1), "beta2": _b(key.beta2), "delta1": _b(key.delta1), "delta2": _b(key.delta2),
            "gamma2": _b(g2.fixed_base(2, _scalars([S.gamma])))}
    pts = {5: _b(key.a), 6: _b(key.b1), 7: _b(key.b2), 8: _b(key.c), 9: _b(key.h)}
    return zw.Zkey(S.n_vars, S.n_pub, S.n, sec2, _b(ic), zw.entries_from_r1cs(R), pts)


def _clean(rep, n_points):
    assert rep["coef_match"] == 3 and rep["coef_out_of_range"] == 0, rep
    assert rep["points_bad"] == 0 and rep["first_bad_section"] == 0 and rep["points_checked"] == n_points, rep


def _n_points(Z):
    return 6 + Z.n_pub + 1 + 3 * Z.n_vars + (Z.n_vars - Z.n_pub - 1) + Z.domain


def _same_bytes(key, path):
    s2 = zw.read_section(path, 2)[84:]
    for t, off, n in ((key.alpha1, 0, 64), (key.beta1, 64, 64), (key.beta2, 128, 128), (key.delta1, 384, 64), (key.delta2, 448, 128)):
        assert _b(t) == s2[off:off + n]
    for sid, t in ((5, key.a), (6, key.b1), (7, key.b2), (8, key.c), (9, key.h)):
        assert _b(t) == zw.read_section(path, sid), sid


def _exact(c, R, S, rng, path, staging):
    key, rep = c.load_zkey(path, seed=rng.randrange(1 << 64), staging_bytes=staging)
    _clean(rep, 6 + S.n_pub + 1 + 3 * S.n_vars + (S.n_vars - S.n_pub - 1) + S.n)
    _same_bytes(key, path)
    W = witness_ints(c.witness(0))
    q = witness_ints(c.r1cs_quotient(0).cpu().numpy())
    r, s = rng.randrange(P), rng.randrange(P)
    assert _expect(S, W, q, r, s, c.groth16_prove(0, key, r=r, s=s))
    return rep


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
@pytest.mark.parametrize("name", SUITES)
def test_exact_load(name, opt, tmp_path):
    import pob_b200
    s = suite(name)
    c = pob_b200.Circuit(s["main"], max_slots=1, opt=opt)
    try:
        assert c.run([next(x for x in s["cases"] if x["expected"] is not None)["input"]]).status[0] == 0
        R, S, rng = _setup(c, s["main"], opt, tmp_path)
        Z = _zkey(S, R)
        Z.order = [9, 4, 2, 7, (10, b"\1" * 9), 1, 5, 3, 8, 6]
        path = str(tmp_path / "k.zkey")
        Z.write(path)
        _exact(c, R, S, rng, path, ODD_STAGING)
    finally:
        c.close()


def test_exact_load_spend_reduced(tmp_path):
    import pob_b200
    c = pob_b200.Circuit("Spend(31)", max_slots=1, opt=1)
    try:
        assert c.run([suite("test_spend")["cases"][0]["input"]]).status[0] == 0
        R, S, rng = _setup(c, "Spend(31)", 1, tmp_path)
        assert S.log_n == 18
        path = str(tmp_path / "k.zkey")
        _zkey(S, R).write(path)
        rep = _exact(c, R, S, rng, path, 4 * ((1 << 20) + 13))
        assert rep["bytes_read"] == pob_b200.zkey_info(path)["file_bytes"] - 12 - 9 * 12 - 4
    finally:
        c.close()


_MULTI = r"""
import json, resource, sys
sys.path[:0] = %r
import torch, pob_b200
from helpers import suite
from test_gpu_groth16 import _tiled_prediction
from test_gpu_msm import _witness_tensor
path, consts, r, s = sys.argv[1], json.loads(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
c = pob_b200.Circuit("Spend(31)", max_slots=1, opt=0)
assert c.run([suite("test_spend")["cases"][0]["input"]]).status[0] == 0
c.r1cs_domain()
torch.cuda.synchronize()
before = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
key, rep = c.load_zkey(path, staging_bytes=64 << 20)
grew = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss - before
got = c.groth16_prove(0, key, r=r, s=s)
w = _witness_tensor(c.witness_device_ptr(0), c.n_signals)
want = _tiled_prediction(c, consts, w, c.r1cs_quotient(0), r, s)
print(json.dumps({"rep": rep, "rss_growth_kib": grew, "same": got == want}))
"""


def test_multi_chunk_spend_o0(tmp_path):
    """Spend(31) --O0 (2,603,360 wires, 2^22 domain): real coefficients, tiled points, 16 MiB staging buffers; host RSS of the loading
    process grows by far less than the file"""
    import g2
    import pob_b200
    from r1cs_reader import R1cs
    f = str(tmp_path / "c.r1cs")
    pob_b200.write_r1cs("Spend(31)", f, opt=0)
    R = R1cs(f)
    nv, npub, dom = R.n_wires, R.n_pub_out, 1 << qm.domain_log(R.m, R.n_pub_out)
    assert dom == 1 << 22
    rng = random.Random(2222)
    consts = [rng.randrange(1, P) for _ in range(3)]
    one = lambda grp, v: _b(g2.fixed_base(grp, _scalars([v])))
    t1, t2 = _b(_tile(1)[0]), _b(_tile(2)[0])
    sec2 = {"alpha1": one(1, consts[0]), "beta1": one(1, consts[1]), "beta2": one(2, consts[1]), "gamma2": one(2, 5),
            "delta1": one(1, consts[2]), "delta2": one(2, consts[2])}
    Z = zw.Zkey(nv, npub, dom, sec2, t1[:64 * (npub + 1)], zw.entries_from_r1cs(R),
                {5: zw.Tiled(t1, nv, 64), 6: zw.Tiled(t1, nv, 64), 7: zw.Tiled(t2, nv, 128), 8: zw.Tiled(t1, nv - npub - 1, 64), 9: zw.Tiled(t1, dom, 64)})
    del R
    path = str(tmp_path / "k.zkey")
    size = Z.write(path)
    r, s = rng.randrange(P), rng.randrange(P)
    code = _MULTI % ([HERE, os.path.join(os.path.dirname(HERE), "proof-of-burn_b200")],)
    out = subprocess.run([sys.executable, "-c", code, path, json.dumps(consts), str(r), str(s)], capture_output=True, text=True, cwd=HERE)
    assert out.returncode == 0, out.stderr[-3000:]
    res = json.loads(out.stdout.strip().splitlines()[-1])
    _clean(res["rep"], 6 + npub + 1 + 3 * nv + (nv - npub - 1) + dom)
    assert res["same"]
    assert res["rss_growth_kib"] * 1024 < size / 8, (res["rss_growth_kib"], size)


# ---- corruptions, on one small circuit -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small(tmp_path_factory):
    import pob_b200
    s = suite("test_poseidon_2")
    c = pob_b200.Circuit(s["main"], max_slots=1, opt=1)
    assert c.run([s["cases"][0]["input"]]).status[0] == 0
    d = tmp_path_factory.mktemp("zk")
    R, S, rng = _setup(c, s["main"], 1, d)
    Z = _zkey(S, R)
    yield c, R, S, Z, d
    c.close()


def _load(c, Z, d, name="k.zkey"):
    """(report, None) of a key that loads, or (report, error) of one that is refused"""
    import pob_b200
    path = str(d / name)
    Z.write(path)
    try:
        _, rep = c.load_zkey(path, seed=987654321, staging_bytes=ODD_STAGING)
        return rep, None
    except pob_b200.ZkeyError as e:
        return e.report, e


def _with_entries(Z, e):
    import copy
    Y = copy.copy(Z)
    Y.entries = e
    return Y


def _rows_of(Z, matrix):
    e = Z.entries
    return np.unique(e["constraint"][e["matrix"] == matrix])


def test_good_key_and_harmless_changes(small):
    c, R, S, Z, d = small
    rep, err = _load(c, Z, d)
    assert err is None
    _clean(rep, _n_points(Z))
    rng = np.random.default_rng(5)
    rep, err = _load(c, _with_entries(Z, Z.entries[rng.permutation(len(Z.entries))]), d)          # entry order does not matter
    assert err is None and rep["coef_match"] == 3
    e = Z.entries.copy()                                                                       # one coefficient split in two
    i = int(np.nonzero(e["matrix"] == 1)[0][0])
    v = int(witness_ints(e["value"][i:i + 1])[0])
    part = 123456789123456789
    e["value"][i] = zw.limbs([(v - part) % P])[0]
    extra = e[i:i + 1].copy()
    extra["value"][0] = zw.limbs([part])[0]
    rep, err = _load(c, _with_entries(Z, np.concatenate([e, extra])), d)
    assert err is None and rep["coef_match"] == 3


def _mismatch(c, Z, d, e, cleared):
    rep, err = _load(c, _with_entries(Z, e), d)
    assert err is not None and err.code == -10, rep
    assert rep["coef_match"] == 3 & ~cleared, rep
    assert rep["points_bad"] == 0 and rep["coef_out_of_range"] == 0
    assert "matrix " + "AB"[cleared.bit_length() - 1] in str(err)


def test_coefficient_mismatches(small):
    c, R, S, Z, d = small
    E = Z.entries
    ia, ib = int(np.nonzero(E["matrix"] == 0)[0][3]), int(np.nonzero(E["matrix"] == 1)[0][2])
    e = E.copy(); e["value"][ia, 0] ^= np.uint64(1 << 40); _mismatch(c, Z, d, e, 1)                       # one value changed
    e = E.copy(); e["signal"][ib] = (e["signal"][ib] + 1) % S.n_vars; _mismatch(c, Z, d, e, 2)             # signal moved
    e = E.copy(); e["constraint"][ia] = (e["constraint"][ia] + 1) % R.m; _mismatch(c, Z, d, e, 1)          # constraint moved
    _mismatch(c, Z, d, np.delete(E, ib), 2)                                                                # one entry dropped
    _mismatch(c, Z, d, np.concatenate([E, E[ia:ia + 1]]), 1)                                               # one entry duplicated
    _mismatch(c, Z, d, E[:len(E) - S.n_pub - 1], 1)                                                        # public rows left out
    ra = _rows_of(Z, 0)                                                                                    # two rows swapped
    r1, r2 = int(ra[0]), int(ra[-1])
    e = E.copy()
    c1, c2 = e["constraint"] == r1, e["constraint"] == r2
    e["constraint"][c1], e["constraint"][c2] = r2, r1
    rep, err = _load(c, _with_entries(Z, e), d)
    assert err is not None and not rep["coef_match"] & 1, rep


def test_canonical_values_are_diagnosed(small):
    c, R, S, Z, d = small
    rep, err = _load(c, _with_entries(Z, zw.entries_from_r1cs(R, canonical=True)), d)
    assert err is not None and rep["coef_match"] == 0 and rep["coef_match_canonical"] == 3, rep
    assert "canonical" in str(err)


def test_key_of_the_other_form_is_refused_on_its_header(small, tmp_path):
    import pob_b200
    s = suite("test_poseidon_2")
    c0 = pob_b200.Circuit(s["main"], max_slots=1, opt=0)
    try:
        c, R, S, Z, d = small
        path = str(tmp_path / "o1.zkey")
        Z.write(path)
        with pytest.raises(pob_b200.ZkeyError) as e:
            c0.load_zkey(path)
        assert e.value.report is None and "nVars" in str(e.value)
    finally:
        c0.close()


def test_out_of_range_entries(small):
    c, R, S, Z, d = small
    bad = Z.entries[:5].copy()
    bad["matrix"][0] = 2
    bad["constraint"][1] = S.n
    bad["signal"][2] = S.n_vars
    bad["matrix"][3] = 0xFFFFFFFF
    bad["signal"][4] = 0xFFFFFFFF
    rep, err = _load(c, _with_entries(Z, np.concatenate([Z.entries, bad])), d)
    assert err is not None and rep["coef_out_of_range"] == 5 and rep["coef_match"] == 3, rep
    assert "out of range" in str(err)


def _flip(buf, pos, bit=3):
    b = bytearray(buf)
    b[pos] ^= 1 << bit
    return bytes(b)


@pytest.mark.parametrize("sid", [2, 3, 5, 6, 7, 8, 9])
def test_point_bit_flip(small, sid):
    import copy
    c, R, S, Z, d = small
    Y = copy.copy(Z)
    Y.sec2, Y.points = dict(Z.sec2), dict(Z.points)
    if sid == 2:
        Y.sec2["gamma2"] = _flip(Z.sec2["gamma2"], 100)
        idx = 3
    elif sid == 3:
        idx = S.n_pub
        Y.ic = _flip(Z.ic, 64 * idx + 5)
    else:
        pb = 128 if sid == 7 else 64
        n = len(Z.points[sid]) // pb
        idx = n // 2
        Y.points[sid] = _flip(Z.points[sid], pb * idx + pb - 20)
    rep, err = _load(c, Y, d)
    assert err is not None and rep["points_bad"] == 1, rep
    assert (rep["first_bad_section"], rep["first_bad_index"]) == (sid, idx), rep
    assert rep["coef_match"] == 3


def test_coordinate_not_below_q(small):
    import copy
    c, R, S, Z, d = small
    Y = copy.copy(Z)
    Y.points = dict(Z.points)
    a = np.frombuffer(Z.points[5], dtype=np.uint64).reshape(-1, 8).copy()
    i = int(np.nonzero(a.any(axis=1))[0][1])
    x = int(witness_ints(a[i:i + 1, :4])[0])
    a[i, :4] = zw.limbs([x + gm.Q])[0]
    Y.points[5] = a.tobytes()
    rep, err = _load(c, Y, d)
    assert err is not None and rep["points_bad"] == 1 and (rep["first_bad_section"], rep["first_bad_index"]) == (5, i), rep


def _canonical(buf):
    a = np.frombuffer(buf, dtype=np.uint64).reshape(-1, 4)
    return zw.limbs([gm.from_mont(int(v)) for v in witness_ints(a)]).tobytes()


def test_canonical_points_are_diagnosed(small):
    import copy
    c, R, S, Z, d = small
    Y = copy.copy(Z)
    Y.sec2 = {k: _canonical(v) for k, v in Z.sec2.items()}
    Y.ic = _canonical(Z.ic)
    Y.points = {k: _canonical(v) for k, v in Z.points.items()}
    rep, err = _load(c, Y, d)
    n_inf = sum(int((~np.frombuffer(v, dtype=np.uint64).reshape(-1, 8 if k != 7 else 16).any(axis=1)).sum()) for k, v in Z.points.items())
    assert err is not None and rep["points_bad"] == rep["points_checked"] - n_inf and rep["points_bad_canonical"] == 0, rep
    assert "canonical" in str(err)


# ---- the command line ------------------------------------------------------------------------------------------------------------
def test_cli(small, tmp_path, monkeypatch, capsys):
    import secrets
    import pob_b200
    c, R, S, Z, d = small
    s = suite("test_poseidon_2")
    good, bad = str(tmp_path / "good.zkey"), str(tmp_path / "bad.zkey")
    Z.write(good)
    e = Z.entries.copy()
    e["value"][0, 1] ^= np.uint64(1)
    _with_entries(Z, e).write(bad)
    assert pob_b200.main([s["main"], "--check-zkey", good, "--O1"]) == 0
    assert json.loads(capsys.readouterr().out.strip().splitlines()[-1])["ok"]
    assert pob_b200.main([s["main"], "--check-zkey", bad, "--O1"]) == 1
    assert not json.loads(capsys.readouterr().out.strip().splitlines()[-1])["ok"]
    case = s["cases"][0]
    inp = str(tmp_path / "in.json")
    json.dump(case["input"], open(inp, "w"))
    rs = [31337, 4242]
    monkeypatch.setattr(secrets, "randbelow", lambda n: rs.pop(0) % n)
    pj, uj = str(tmp_path / "proof.json"), str(tmp_path / "public.json")
    assert pob_b200.main([s["main"], "--prove", good, inp, pj, uj, "--O1"]) == 0
    res = c.run([case["input"]])
    W = witness_ints(c.witness(0))
    q = qm.quotient(*R.products(W), W[:S.n_pub + 1], R.m)
    a, b, cc = S.proof_scalars(W, q, 31337, 4242)
    want = pob_b200.Proof(gm.mul(a, gm.G), g2m.mul(b, g2m.G), gm.mul(cc, gm.G))
    assert json.load(open(pj)) == want.to_json()
    assert json.load(open(uj)) == pob_b200.public_json(res.outputs[0])
    rejected = next((x for x in s["cases"] if x["expected"] is None), None)
    if rejected is not None:
        json.dump(rejected["input"], open(inp, "w"))
        os.remove(pj)
        assert pob_b200.main([s["main"], "--prove", good, inp, pj, uj, "--O1"]) == 1
        assert not os.path.exists(pj)
    json.dump(case["input"], open(inp, "w"))
    assert pob_b200.main([s["main"], "--prove", bad, inp, pj + ".2", uj, "--O1"]) == 1
    assert not os.path.exists(pj + ".2")
