"""Time pob_r1cs_quotient for main_proof_of_burn, --O0 (n = 2^28, max_slots=1) and reduced (n = 2^25) witness, on one synthetic
instance: the whole quotient and its products step alone (k_r1cs_products over every row), best of --reps after a warm-up, with CUDA
events on one stream.  Reports the global-memory bytes the passes move (from the pass count, against 3.35 TB/s) and the Montgomery
products per second (counted from n and log_n).  Prints one JSON line (and writes it to --out), with the card name and power limit
read in the same run.

    python tools/quotient_bench.py [--reps 3] [--out quotient_bench.json]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "proof-of-burn_b200"), os.path.join(ROOT, "tools")]

HBM_TBS = 3.35          # H100 SXM 80 GB peak DRAM bandwidth
TILE_LOG = 11           # ntt.cuh: NTT_TILE_LOG


def ntt_plan(L, T):
    """stages per pass (ntt.cuh: ntt_plan)"""
    q = 0
    while L > T + q * (T - 2):
        q += 1
    P = q + 1
    k = [L // P] * P
    for i in range(L % P):
        k[P - 1 - i] += 1
    return k


def model(m, n_pub, L):
    """bytes and Montgomery products of one quotient (DESIGN.md §5).  Per pass every entry is read and written once (64 B); the
    fused last pass also reads A and B.  The products step writes 3 m entries (its witness reads are not counted) and the fills the
    rest of the three vectors.  Products: L n per vector for the butterflies of both transforms (every butterfly counted, also those
    whose twiddle is 1), 2 per entry for every inter-pass twiddle (table product + apply) and for the coset factor, 2 per entry for
    A.B."""
    n = 1 << L
    P = len(ntt_plan(L, min(L, TILE_LOG)))
    ntt_bytes = 3 * 2 * P * 64 * n + 64 * n
    fill_bytes = 32 * 3 * n
    monts = 3 * (L * n + 2 * 2 * n * (P - 1) + 2 * n) + 2 * n
    return {"log_n": L, "n": n, "passes_per_transform": P, "stages": ntt_plan(L, min(L, TILE_LOG)), "ntt_bytes": ntt_bytes,
            "fill_bytes": fill_bytes, "mont_products": monts, "rows": m, "n_pub": n_pub}


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


def bench(opt, reps):
    import torch
    import pob_b200
    from pob_b200 import synth
    shape = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1, opt=opt)
    try:
        assert c.run_packed(synth.pack_instances(synth.make_batch(1, shape, seed=2718), shape)).status[0] == 0
        rows = c.r1cs_check(0)["n_constraints"]
        L = c.r1cs_domain()
        n = 1 << L
        out = torch.empty((n, 4), dtype=torch.uint64, device="cuda")
        work = torch.empty((2 * n, 4), dtype=torch.uint64, device="cuda")
        st = torch.cuda.Stream()
        lib, h = pob_b200.lib(), c._h
        sp = ctypes.c_void_p(st.cuda_stream)
        q_ms, q_all = timed(st, lambda: pob_b200._check(lib.pob_r1cs_quotient(h, 0, out.data_ptr(), work.data_ptr(), sp)), reps)
        p_ms, p_all = timed(st, lambda: pob_b200._check(lib.pob_r1cs_products(h, 0, 0, rows, out.data_ptr(), work.data_ptr(),
                                                                               work.data_ptr() + 32 * n, sp)), reps)
        M = model(rows, c.n_outputs, L)
        ntt_ms = q_ms - p_ms
        M.update({"opt": opt, "quotient_ms": q_ms, "quotient_ms_all": q_all, "products_ms": p_ms, "products_ms_all": p_all,
                  "ntt_ms": ntt_ms, "ntt_tbs": M["ntt_bytes"] / ntt_ms / 1e9, "ntt_bytes_fraction_of_peak": M["ntt_bytes"] / ntt_ms / 1e9 / HBM_TBS,
                  "mont_per_s": M["mont_products"] / ntt_ms * 1e3, "buffer_bytes": 3 * 32 * n})
        return M
    finally:
        c.close()


def main():
    from r1cs_bench import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card(), "results": [bench(opt, a.reps) for opt in (0, 1)]}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
