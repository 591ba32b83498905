"""Time the `.zkey` path on the main shape's reduced form: write a proving key into DIR (the real section-4 coefficients of the circuit's
`.r1cs`, tiled points as in tests/test_gpu_groth16.py: not a valid key, but one the check passes), then time pob_zkey_info, the load
(GB/s of the file), its check, and one proof from the loaded key.  The file is read right after it was written, so it comes from the
page cache: these numbers are the loader's, not a disk's (dropping the cache is not done here).  Prints one JSON line (and writes it to
--out), with the card name and power limit read in the same run.

    python tools/zkey_bench.py DIR [--reps 2] [--keep] [--out zkey_bench.json]
"""
import argparse
import json
import mmap
import os
import random
import struct
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "proof-of-burn_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]


def ab_entries(path, n_pub):
    """the section-4 entries of a `.r1cs`: every A and B term in row order, then the public rows; one pass over the file"""
    import zkey_writer as zw
    f = open(path, "rb")
    mm = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
    pos, secs = 12, {}
    for _ in range(struct.unpack_from("<I", mm, 8)[0]):
        typ, size = struct.unpack_from("<IQ", mm, pos)
        secs[typ] = (pos + 12, size)
        pos += 12 + size
    h = secs[1][0]
    m = struct.unpack_from("<I", mm, h + 60)[0]
    starts, counts, rows, mats = [], [], [], []
    q = secs[2][0]
    u32 = struct.Struct("<I").unpack_from
    for row in range(m):
        for j in range(3):
            n = u32(mm, q)[0]
            if j < 2 and n:
                starts.append(q + 4); counts.append(n); rows.append(row); mats.append(j)
            q += 4 + 36 * n
    counts = np.array(counts, dtype=np.int64)
    first = np.repeat(np.cumsum(counts) - counts, counts)
    offs = np.repeat(np.array(starts, dtype=np.int64), counts) + 36 * (np.arange(int(counts.sum()), dtype=np.int64) - first)
    rows, mats = np.repeat(np.array(rows, dtype=np.uint32), counts), np.repeat(np.array(mats, dtype=np.uint32), counts)
    buf = np.frombuffer(mm, dtype=np.uint8)
    e = np.zeros(len(offs) + n_pub + 1, dtype=zw.ENTRY)
    k = len(offs)
    e["matrix"][:k], e["constraint"][:k] = mats, rows
    e["signal"][:k] = buf[offs[:, None] + np.arange(4)].copy().view("<u4").ravel()
    raw = buf[offs[:, None] + 4 + np.arange(32)].copy().view("<u8").reshape(k, 4)
    uniq, inv = np.unique(raw, axis=0, return_inverse=True)
    vals = [int(a) | int(b) << 64 | int(c) << 128 | int(d) << 192 for a, b, c, d in uniq]
    e["value"][:k] = zw.encode_values(vals)[inv.ravel()]
    e["constraint"][k:] = m + np.arange(n_pub + 1)
    e["signal"][k:] = np.arange(n_pub + 1)
    e["value"][k:] = zw.encode_values([1] * (n_pub + 1))
    del buf
    return e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--keep", action="store_true", help="leave the key file in DIR")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import pob_b200
    import zkey_writer as zw
    from pob_b200 import synth
    from r1cs_bench import card
    from test_gpu_groth16 import _scalars, _tile
    from test_gpu_msm import MAIN_SHAPE
    import g2
    os.makedirs(a.dir, exist_ok=True)
    r1cs, path = os.path.join(a.dir, "main_o1.r1cs"), os.path.join(a.dir, "main_o1.zkey")
    t0 = time.time()
    pob_b200.write_r1cs(pob_b200.MAIN_PROOF_OF_BURN, r1cs, opt=1)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1, opt=1)
    nv, npub, dom = c.n_signals, c.n_outputs, 1 << c.r1cs_domain()
    ent = ab_entries(r1cs, npub)
    os.remove(r1cs)
    rng = random.Random(2525)
    consts = [rng.randrange(1, pob_b200.P) for _ in range(3)]
    b = lambda t: t.cpu().numpy().tobytes()
    one = lambda grp, v: b(g2.fixed_base(grp, _scalars([v])))
    t1, t2 = b(_tile(1)[0]), b(_tile(2)[0])
    sec2 = {"alpha1": one(1, consts[0]), "beta1": one(1, consts[1]), "beta2": one(2, consts[1]), "gamma2": one(2, 5),
            "delta1": one(1, consts[2]), "delta2": one(2, consts[2])}
    Z = zw.Zkey(nv, npub, dom, sec2, t1[:64 * (npub + 1)], ent, {5: zw.Tiled(t1, nv, 64), 6: zw.Tiled(t1, nv, 64), 7: zw.Tiled(t2, nv, 128),
                                                             8: zw.Tiled(t1, nv - npub - 1, 64), 9: zw.Tiled(t1, dom, 64)})
    size = Z.write(path)
    del Z, ent
    write_s = time.time() - t0
    packed = synth.pack_instances(synth.make_batch(1, MAIN_SHAPE, seed=4242), MAIN_SHAPE)
    assert c.run_packed(packed).status[0] == 0
    res = {"file_bytes": size, "n_vars": nv, "log_n": c.r1cs_domain(), "write_s": write_s, "page_cache": True}
    ti = time.perf_counter()
    info = pob_b200.zkey_info(path)
    res["info_ms"] = (time.perf_counter() - ti) * 1e3
    res["n_coefs"] = info["n_coefs"]
    loads = []
    for _ in range(a.reps):
        key = None
        torch.cuda.empty_cache()
        key, rep = c.load_zkey(path)
        loads.append(rep)
    best = min(loads, key=lambda r: r["total_ms"])
    assert best["coef_match"] == 3 and best["points_bad"] == 0, best
    res.update(load_ms=best["total_ms"], load_gbs=size / best["total_ms"] / 1e6, read_ms=best["read_ms"], copy_ms=best["copy_ms"],
               check_ms=best["check_ms"], device_scratch_bytes=best["device_scratch_bytes"], loads_ms=[r["total_ms"] for r in loads])
    work = torch.empty(c.groth16_work_bytes(), dtype=torch.uint8, device="cuda")
    times = []
    for _ in range(a.reps + 1):
        torch.cuda.synchronize()
        tp = time.perf_counter()
        c.groth16_prove(0, key, r=1, s=2, work=work)
        times.append((time.perf_counter() - tp) * 1e3)
    res["prove_ms"], res["prove_ms_all"] = min(times[1:]), times[1:]
    c.close()
    if not a.keep:
        os.remove(path)
    line = json.dumps({"card": card(), "results": res})
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
