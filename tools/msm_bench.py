"""Time pob_msm_g1 (the BN254 G1 multi-exponentiation): uniform random 256-bit scalars at n = 2^20 ... 2^28, a witness-like vector at
2^24 (96 % of the entries 0 or 1, the rest random), the witness MSM of main_proof_of_burn in both forms (21,454,051 reduced and
215,907,954 --O0 scalars, one synthetic instance) and the H MSM over its quotient (2^25 reduced, 2^28 --O0, reusing the quotient's
work).  Bases are 1024 distinct curve points tiled up to n (the time does not depend on which points they are).  Best of --reps
after a warm-up, CUDA events on one stream.  Prints one JSON line (and writes it to --out), with the card name and power limit read
in the same run.

    python tools/msm_bench.py [--reps 2] [--max-log 28] [--out msm_bench.json]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "proof-of-burn_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]


def tile_bases(n):
    import torch
    import g1_model as gm
    pts, P = [], gm.G
    for _ in range(1024):
        pts.append(P)
        P = gm.add(P, gm.G)
    B = torch.from_numpy(gm.encode_bases(pts).view("int64")).cuda()
    return B.repeat((n + 1023) // 1024, 1)[:n].contiguous().view(torch.uint64)


def timed(st, fn, reps):
    import torch
    times = []
    for _ in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        fn()
        e1.record(st)
        st.synchronize()
        times.append(e0.elapsed_time(e1))
    return min(times[1:]), times[1:]


def run(label, bases, s_ptr, n, reps, work=None):
    import torch
    import pob_b200
    st = torch.cuda.Stream()
    need = pob_b200.msm_g1_work_bytes(n)
    if work is None:
        work = torch.empty(need, dtype=torch.uint8, device="cuda")
    wbytes = work.numel() * work.element_size()
    out = torch.empty(8, dtype=torch.uint64, device="cuda")
    lib, sp = pob_b200.lib(), ctypes.c_void_p(st.cuda_stream)
    ms, all_ms = timed(st, lambda: pob_b200._check(lib.pob_msm_g1(0, bases.data_ptr(), s_ptr, n, out.data_ptr(), work.data_ptr(), wbytes, sp)), reps)
    r = {"case": label, "n": n, "ms": ms, "ms_all": all_ms, "points_per_s": n / ms * 1e3, "work_bytes": need}
    print(json.dumps(r), file=sys.stderr)
    return r


def random_scalars(n, seed):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return torch.randint(-(1 << 63), (1 << 63) - 1, (n, 4), dtype=torch.int64, device="cuda", generator=g)


def main():
    import torch
    import pob_b200
    from pob_b200 import synth
    from r1cs_bench import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--max-log", type=int, default=28)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = []
    for lg in range(20, a.max_log + 1, 2):
        n = 1 << lg
        b, s = tile_bases(n), random_scalars(n, lg)
        res.append(run("random_2^%d" % lg, b, s.data_ptr(), n, a.reps))
        if lg == 24:
            small = torch.rand(n, device="cuda") < 0.96
            bits = torch.randint(0, 2, (n,), device="cuda")
            s[small] = 0
            s[small, 0] = bits[small]
            res.append(run("witness_like_2^24", b, s.data_ptr(), n, a.reps))
        del b, s
        torch.cuda.empty_cache()
    shape = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)
    for opt in (1, 0):
        c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1, opt=opt)
        try:
            assert c.run_packed(synth.pack_instances(synth.make_batch(1, shape, seed=2718), shape)).status[0] == 0
            n = c.n_signals
            b = tile_bases(n)
            res.append(run("witness_%s" % ("reduced" if opt else "O0"), b, c.witness_device_ptr(0), n, a.reps))
            del b
            torch.cuda.empty_cache()
            L = c.r1cs_domain()
            work = torch.empty((2 << L, 4), dtype=torch.uint64, device="cuda")
            q = c.r1cs_quotient(0, work=work)
            b = tile_bases(1 << L)
            res.append(run("H_2^%d" % L, b, q.data_ptr(), 1 << L, a.reps, work=work))
            del b, q, work
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
