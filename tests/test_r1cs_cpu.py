"""The `.r1cs` writer (pob_write_r1cs) on the CPU, read back with an independent Python reader (tests/r1cs_reader.py) and checked
against ORACLE witnesses: header, sorted and zero-free combinations, A*B = C on every row, the wire-to-label map, for the --O0 and
the reduced (--O1) witness form."""
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import gold, suite
from r1cs_reader import R1cs, witness_ints

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = [s for s in gold() if s["suite"] != "test_proof_of_burn"]


def _write(tmp_path, main, opt, hcreate=False):
    import pob_b200
    f = str(tmp_path / ("o%d_h%d.r1cs" % (opt, int(hcreate))))
    d = pob_b200.write_r1cs(main, f, hcreate=hcreate, opt=opt)
    return d, R1cs(f), f


@pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])
@pytest.mark.parametrize("s", SMALL, ids=[s["suite"] for s in SMALL])
def test_r1cs_holds_on_the_oracle_witness(s, opt, tmp_path):
    import pob_b200
    from oracle import oracle
    d, R, f = _write(tmp_path, s["main"], opt)
    L = pob_b200.layout_info(s["main"], opt=opt)
    assert d["file_bytes"] == os.path.getsize(f) == R.size
    assert R.version == 1 and R.section_order == [1, 2, 3] and R.p == pob_b200.P
    assert (R.n_wires, R.n_pub_out, R.n_pub_in, R.n_prv_in, R.n_labels) == (L["n_signals"], L["n_outputs"], 0, L["n_inputs"], L["n_signals_o0"])
    assert (R.m, R.n_terms) == (d["n_constraints"], d["n_terms"]) and d["n_wires"] == R.n_wires
    assert d["n_nonlinear"] == int((R.lc_n[0::3] > 0).sum())
    assert R.lc_sorted_unique_nonzero()
    assert not ((R.lc_n[0::3] == 0) & (R.lc_n[1::3] > 0)).any(), "B is written empty when A is"
    assert not ((R.lc_n[0::3] == 0) & (R.lc_n[2::3] == 0)).any(), "a row with A and C empty"
    if opt == 0:
        ci = pob_b200.constraint_info(s["main"])
        # the witness[0] == 1 record is the only trivial one
        assert d["n_constraints"] == ci["n_constraints"] - 1 and d["n_nonlinear"] == ci["n_nonlinear"]
        assert np.array_equal(R.labels, np.arange(R.n_wires, dtype=np.uint64))
        wmap = None
    else:
        import emu
        name, params = oracle.parse_main(s["main"])
        pl = oracle.to_limbs(params) if params else np.zeros((1, 4), dtype=np.uint64)
        wmap = emu.EmuProgram(name, pl, len(params), opt=1).witness_map()[0]
        assert np.array_equal(R.labels, wmap.astype(np.uint64))
    done = 0
    for case in s["cases"]:
        if case["expected"] is None:
            continue
        w = oracle.run(s["main"], case["input"])
        try:
            W = witness_ints(w.limbs if wmap is None else w.limbs[wmap])
            n = w.n_signals
        finally:
            w.free()
        bad = R.failing_rows(W)
        assert len(bad) == 0, "%s: rows %s fail" % (s["suite"], bad[:10])
        done += 1
        if n > 1_000_000 and done >= 2:
            break
    assert done


def test_main_shape_counts():
    """main_proof_of_burn without writing the file: the --O0 system is the constraint system less the witness[0] record; the reduced
    system's sizes are pinned (DESIGN.md §5)"""
    import pob_b200
    d0 = pob_b200.write_r1cs(pob_b200.MAIN_PROOF_OF_BURN)
    assert (d0["n_wires"], d0["n_labels"], d0["n_constraints"], d0["n_nonlinear"]) == (215907954, 215907954, 215962293 - 1, 17910859)
    assert (d0["n_pub_out"], d0["n_pub_in"], d0["n_prv_in"]) == (1, 0, 10906)
    assert (d0["n_terms"], d0["file_bytes"]) == (477377583, 21504404236)
    d1 = pob_b200.write_r1cs(pob_b200.MAIN_PROOF_OF_BURN, opt=1)
    assert (d1["n_wires"], d1["n_labels"], d1["n_constraints"], d1["n_nonlinear"]) == (21454051, 215907954, 21508380, 16142845)
    assert (d1["n_terms"], d1["file_bytes"]) == (82752621, 3408827436)


def test_reduced_spend_notices_a_changed_entry(tmp_path):
    """O1 Spend(31): +1 on 2,000 random reduced entries, one at a time, breaks some row -- except entries the circuit leaves free and
    only a hint pins: such an entry, poked in the --O0 witness, fails a hint record and no constraint of the --O0 system"""
    import emu
    from oracle import oracle
    s = suite("test_spend")
    d, R, f = _write(tmp_path, "Spend(31)", 1)
    w = oracle.run("Spend(31)", s["cases"][0]["input"])
    W0 = w.limbs.copy()
    w.free()
    wmap = R.labels.astype(np.int64)
    W = witness_ints(W0[wmap])
    assert len(R.failing_rows(W)) == 0
    ptr, rows = R.rows_of_wire()
    rng = np.random.default_rng(2031)
    missed = []
    for k in rng.choice(np.arange(1, R.n_wires), size=2000, replace=False):
        k = int(k)
        old = W[k]
        W[k] = (old + 1) % R.p
        if all(R.row_ok(int(r), W) for r in np.unique(rows[ptr[k]:ptr[k + 1]])):
            missed.append(k)
        W[k] = old
    name, params = oracle.parse_main("Spend(31)")
    pl = oracle.to_limbs(params)
    for k in missed:
        i = int(wmap[k])
        P0 = W0.copy()
        P0[i] = oracle.to_limbs([(oracle.from_limbs(W0[i]) + 1) % oracle.P])[0]
        r = emu.check_constraints(name, pl, len(params), P0)
        assert r["n_failed"] == 0 and r["n_hint_failed"] > 0, "reduced entry %d (--O0 %d) is pinned by nothing" % (k, i)
    assert len(missed) < 100, len(missed)


def test_r1cs_follows_the_numbering_policy(tmp_path):
    """the hcreate system accepts the oracle's hcreate witness, the default system rejects it"""
    from oracle import oracle
    s = suite("test_num_2_bits_safe_256")
    w = oracle.run(s["main"], s["cases"][0]["input"], hcreate=True)
    try:
        W = witness_ints(w.limbs)
    finally:
        w.free()
    _, same, _ = _write(tmp_path, s["main"], 0, hcreate=True)
    assert len(same.failing_rows(W)) == 0
    _, other, _ = _write(tmp_path, s["main"], 0, hcreate=False)
    assert len(other.failing_rows(W)) > 0


def test_cli_writes_the_same_bytes(tmp_path):
    import pob_b200
    for opt in (0, 1):
        f = str(tmp_path / ("api%d.r1cs" % opt))
        pob_b200.write_r1cs("Poseidon(3)", f, opt=opt)
        g = str(tmp_path / ("cli%d.r1cs" % opt))
        env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "proof-of-burn_b200"), ROOT]))
        subprocess.check_call([sys.executable, "-m", "pob_b200", "Poseidon(3)", "--r1cs", g] + (["--O1"] if opt else []), env=env, cwd=str(tmp_path))
        assert open(f, "rb").read() == open(g, "rb").read()


def test_write_errors_are_io_errors(tmp_path):
    import pob_b200
    with pytest.raises(pob_b200.PobError) as e:
        pob_b200.write_r1cs("Poseidon(2)", str(tmp_path / "no" / "such" / "dir.r1cs"))
    assert e.value.code == -6
