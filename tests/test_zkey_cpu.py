"""pob_zkey_info without a GPU: the header of a written `.zkey` (tests/zkey_writer.py), and each structural defect refused with
POB_E_KEY or POB_E_IO and a message that names it.  The points are placeholders: the header reader does not look at them."""
import pytest

import quotient_model as qm
from helpers import suite
from r1cs_reader import R1cs
import zkey_writer as zw

E_IO, E_KEY = -6, -10


@pytest.fixture(scope="module")
def base(tmp_path_factory):
    import pob_b200
    main = suite("test_poseidon_2")["main"]
    f = str(tmp_path_factory.mktemp("zk") / "c.r1cs")
    pob_b200.write_r1cs(main, f, opt=1)
    return R1cs(f)


def _key(R):
    n_pub = R.n_pub_out + R.n_pub_in
    dom = 1 << qm.domain_log(R.m, n_pub)
    nv = R.n_wires
    sec2 = {k: bytes(zw.SEC2_SIZES[k]) for k in zw.SEC2_POINTS}
    pts = {5: bytes(64 * nv), 6: bytes(64 * nv), 7: bytes(128 * nv), 8: bytes(64 * (nv - n_pub - 1)), 9: bytes(64 * dom)}
    return zw.Zkey(nv, n_pub, dom, sec2, bytes(64 * (n_pub + 1)), zw.entries_from_r1cs(R), pts)


def _info(Z, tmp_path, name="k.zkey"):
    import pob_b200
    p = str(tmp_path / name)
    Z.write(p)
    return pob_b200.zkey_info(p)


def _refused(Z, tmp_path, code, words):
    import pob_b200
    p = str(tmp_path / "bad.zkey")
    Z.write(p)
    with pytest.raises(pob_b200.PobError) as e:
        pob_b200.zkey_info(p)
    assert e.value.code == code, str(e.value)
    for w in words:
        assert w in str(e.value), (w, str(e.value))


def test_header(base, tmp_path):
    Z = _key(base)
    d = _info(Z, tmp_path)
    nv, npub = base.n_wires, base.n_pub_out + base.n_pub_in
    assert (d["n_vars"], d["n_pub"], d["log_n"]) == (nv, npub, qm.domain_log(base.m, npub))
    assert d["n_coefs"] == len(Z.entries) == int((base.term_lc % 3 < 2).sum()) + npub + 1
    assert d["a_bytes"] == d["b1_bytes"] == 64 * nv and d["b2_bytes"] == 128 * nv
    assert d["c_bytes"] == 64 * (nv - npub - 1) and d["h_bytes"] == 64 << d["log_n"]
    assert d["key_bytes"] == d["a_bytes"] + d["b1_bytes"] + d["b2_bytes"] + d["c_bytes"] + d["h_bytes"] + 448
    assert d["file_bytes"] == (tmp_path / "k.zkey").stat().st_size


def test_section_order_and_unknown_sections(base, tmp_path):
    want = _info(_key(base), tmp_path, "a.zkey")
    Z = _key(base)
    Z.order = [9, (10, b"contributions"), 4, 7, 1, 3, (77, bytes(100)), 8, 2, 6, 5]
    got = _info(Z, tmp_path, "b.zkey")
    assert {k: v for k, v in got.items() if k != "file_bytes"} == {k: v for k, v in want.items() if k != "file_bytes"}
    assert got["file_bytes"] == want["file_bytes"] + 2 * 12 + 13 + 100


def _set(**kw):
    def f(Z):
        for k, v in kw.items():
            setattr(Z, k, v)
    return f


CASES = {
    "magic": (_set(magic=b"zkex"), E_KEY, ["magic"]),
    "version": (_set(version=2), E_KEY, ["version"]),
    "protocol": (_set(protocol=2), E_KEY, ["protocol", "Groth16"]),
    "q": (_set(q=zw.Q_MOD + 2), E_KEY, ["q is not"]),
    "r": (_set(r=zw.R_MOD - 2), E_KEY, ["r is not"]),
    "n8q": (_set(n8q=48), E_KEY, ["n8q"]),
    "n8r": (_set(n8r=48), E_KEY, ["n8r"]),
    "domain_not_pow2": (lambda Z: setattr(Z, "domain", Z.domain + 1), E_KEY, ["domainSize"]),
}
for _sid in range(1, 10):
    CASES["missing_%d" % _sid] = (lambda Z, s=_sid: setattr(Z, "order", [x for x in Z.order if x != s]), E_KEY, ["section %d is missing" % _sid])
    CASES["twice_%d" % _sid] = (lambda Z, s=_sid: setattr(Z, "order", Z.order + [s]), E_KEY, ["section %d appears twice" % _sid])
for _sid in range(1, 10):
    # the section is one point / entry / word longer than the header implies
    _unit = {1: 4, 2: 4, 3: 64, 4: 44, 5: 64, 6: 64, 7: 128, 8: 64, 9: 64}[_sid]
    CASES["size_%d" % _sid] = (lambda Z, s=_sid, u=_unit: (setattr(Z, "order", [x for x in Z.order if x != s] + [(s, Z._content(s)[0] * b"\0" + bytes(u))])),
                               E_KEY, ["section %d has" % _sid])
CASES["n_coefs"] = (_set(n_coefs=3), E_KEY, ["section 4 has", "nCoefs"])
CASES["n_vars"] = (lambda Z: setattr(Z, "n_vars", Z.n_vars + 1), E_KEY, ["section 5 has", "nVars"])


@pytest.mark.parametrize("case", sorted(CASES))
def test_structural_errors(base, tmp_path, case):
    mutate, code, words = CASES[case]
    Z = _key(base)
    mutate(Z)
    _refused(Z, tmp_path, code, words)


@pytest.mark.parametrize("sid", range(1, 10))
def test_truncated_inside_each_section(base, tmp_path, sid):
    Z = _key(base)
    p = str(tmp_path / "whole.zkey")
    Z.write(p)
    off, size = zw.sections(p)[sid]
    Z.truncate = off + size // 2
    _refused(Z, tmp_path, E_IO, ["ends early", "section %d" % sid])


def test_truncated_header(base, tmp_path):
    Z = _key(base)
    Z.truncate = 7
    _refused(Z, tmp_path, E_IO, ["ends early"])
    Z.truncate = 20
    _refused(Z, tmp_path, E_IO, ["ends early"])
