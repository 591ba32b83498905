"""Time pob_msm_g2 (the BN254 G2 multi-exponentiation) and pob_groth16_prove: G2 MSMs on uniform random 256-bit scalars at n = 2^20 ...
2^26 and on the witness of main_proof_of_burn in both forms (21,454,051 reduced and 215,907,954 --O0 scalars, one synthetic instance);
then whole proofs of the reduced witness with a tiled key, and the per-stage split from calling the stages one by one on the same
stream: quotient, H, A, B1, C, B2.  The assembly (blinding and additions) is the whole proof less the sum of the stages.  Bases and
key points are 1024 distinct points tiled up to n (the time does not depend on which points they are; a tiled key is not a valid
key).  Best of --reps after a warm-up, CUDA events on one stream.  Prints one JSON line (and writes it to --out), with the card name
and power limit read in the same run.

    python tools/prove_bench.py [--reps 3] [--max-log 26] [--out prove_bench.json]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "proof-of-burn_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from msm_bench import random_scalars, tile_bases, timed  # noqa: E402


def tile_g2(n):
    import torch
    import g2_model as g2m
    pts, P = [], g2m.G
    for _ in range(1024):
        pts.append(P)
        P = g2m.add(P, g2m.G)
    B = torch.from_numpy(g2m.encode_points(pts).view("int64")).cuda()
    return B.repeat((n + 1023) // 1024, 1)[:n].contiguous().view(torch.uint64)


def msm_call(group, bases, s_ptr, n, out, work, sp):
    import pob_b200
    f = pob_b200.lib().pob_msm_g2 if group == 2 else pob_b200.lib().pob_msm_g1
    wb = work.numel() * work.element_size()
    return lambda: pob_b200._check(f(0, bases.data_ptr(), s_ptr, n, out.data_ptr(), work.data_ptr(), wb, sp))


def run_g2(label, bases, s_ptr, n, reps):
    import torch
    import pob_b200
    st = torch.cuda.Stream()
    need = pob_b200.msm_g2_work_bytes(n)
    work = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(16, dtype=torch.uint64, device="cuda")
    ms, all_ms = timed(st, msm_call(2, bases, s_ptr, n, out, work, ctypes.c_void_p(st.cuda_stream)), reps)
    r = {"case": label, "n": n, "ms": ms, "ms_all": all_ms, "points_per_s": n / ms * 1e3, "work_bytes": need}
    print(json.dumps(r), file=sys.stderr)
    return r


def prove_stages(c, reps):
    """the whole proof of resident witness 0 with a tiled key, and each stage alone"""
    import torch
    import pob_b200
    nv, npub, L = c.n_signals, c.n_outputs, c.r1cs_domain()
    n = 1 << L
    a, h, b2 = tile_bases(nv), tile_bases(n), tile_g2(nv)
    cc = a[npub + 1:]
    key = pob_b200.Groth16Key(alpha1=a[:1], beta1=a[1:2], delta1=a[2:3], beta2=b2[:1], delta2=b2[1:2], a=a, b1=a, b2=b2, c=cc, h=h)
    need = c.groth16_work_bytes()
    work = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(32, dtype=torch.uint64, device="cuda")
    st = torch.cuda.Stream()
    sp = ctypes.c_void_p(st.cuda_stream)
    w = c.witness_device_ptr(0)
    res = {"case": "prove_reduced", "n_vars": nv, "log_n": L, "work_bytes": need}
    res["ms"], res["ms_all"] = timed(st, lambda: c.groth16_prove(0, key, r=12345, s=67890, stream=st, out=out, work=work), reps)
    qbuf = work[:32 * n].view(torch.uint64).view(n, 4)
    scratch = work[32 * n:]                                   # the library's layout: q, then the scratch (pob_groth16_work_bytes)
    o1, o2 = out[:8], out[:16]
    stages = {
        "quotient": lambda: c.r1cs_quotient(0, stream=st, out=qbuf, work=scratch[:64 * n].view(torch.uint64).view(2 * n, 4)),
        "H": msm_call(1, h, qbuf.data_ptr(), n, o1, scratch, sp),
        "A": msm_call(1, a, w, nv, o1, scratch, sp),
        "B1": msm_call(1, a, w, nv, o1, scratch, sp),
        "C": msm_call(1, cc, w + 32 * (npub + 1), nv - npub - 1, o1, scratch, sp),
        "B2": msm_call(2, b2, w, nv, o2, scratch, sp),
    }
    res["stages_ms"] = {k: timed(st, f, reps)[0] for k, f in stages.items()}
    res["stages_ms"]["assembly_and_rest"] = res["ms"] - sum(res["stages_ms"].values())
    print(json.dumps(res), file=sys.stderr)
    return res


def main():
    import torch
    import pob_b200
    from pob_b200 import synth
    from r1cs_bench import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-log", type=int, default=26)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = []
    for lg in range(20, a.max_log + 1, 2):
        n = 1 << lg
        b, s = tile_g2(n), random_scalars(n, lg)
        res.append(run_g2("g2_random_2^%d" % lg, b, s.data_ptr(), n, a.reps))
        del b, s
        torch.cuda.empty_cache()
    shape = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)
    for opt in (1, 0):
        c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1, opt=opt)
        try:
            assert c.run_packed(synth.pack_instances(synth.make_batch(1, shape, seed=2718), shape)).status[0] == 0
            b = tile_g2(c.n_signals)
            res.append(run_g2("g2_witness_%s" % ("reduced" if opt else "O0"), b, c.witness_device_ptr(0), c.n_signals, a.reps))
            del b
            torch.cuda.empty_cache()
            if opt:
                res.append(prove_stages(c, a.reps))
                torch.cuda.empty_cache()
        finally:
            c.close()
    line = json.dumps({"card": card(), "results": res})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
