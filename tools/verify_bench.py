"""Time the verification path: pob_bn254_pairing at n = 1 and 2^16, and pob_groth16_verify of n = 1, 2^10, 2^14 and 2^17 proofs at
n_pub = 1 and at the main shape's n_pub.  Proofs are valid simulated ones (a trapdoor key, c solved from a and b), 1024 distinct ones
tiled to n; every status is checked to be 0.  Best of --reps after a warm-up, CUDA events around each call.  Prints one JSON line (and
writes it to --out), with the card name and power limit read in the same run.

    python tools/verify_bench.py [--reps 3] [--out verify_bench.json]
"""
import argparse
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "proof-of-burn_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests"),
                os.path.join(ROOT, "tests", "devprobe")]

DISTINCT = 1024


def timed(fn, reps):
    import torch
    fn()                                                                  # warm-up
    torch.cuda.synchronize()
    best = None
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        best = ms if best is None else min(best, ms)
    return best


def tile(t, n):
    import torch
    v = t.view(torch.int64)
    return v.repeat((n + v.shape[0] - 1) // v.shape[0], 1)[:n].contiguous().view(torch.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import pob_b200
    import g2
    from r1cs_bench import card
    from test_gpu_groth16_verify import Sim
    from test_gpu_msm import _dev
    from r1cs_reader import limbs_of
    R = pob_b200.R_ORDER
    res = {"card": card(), "reps": a.reps}
    L = pob_b200.lib()
    st = torch.cuda.current_stream().cuda_stream

    # the pairing
    rng = random.Random(1)
    sc = lambda v: _dev(limbs_of(v, R))
    g1s = g2.fixed_base(1, sc([rng.randrange(1, R) for _ in range(DISTINCT)]))
    g2s = g2.fixed_base(2, sc([rng.randrange(1, R) for _ in range(DISTINCT)]))
    res["pairing_ms"] = {}
    for n in (1, 1 << 16):
        p, q = tile(g1s, n), tile(g2s, n)
        out = torch.empty((n, 48), dtype=torch.uint64, device="cuda")
        f = lambda: pob_b200._check(L.pob_bn254_pairing(0, p.data_ptr(), q.data_ptr(), n, out.data_ptr(), st))
        res["pairing_ms"][str(n)] = timed(f, a.reps)

    # verification
    main_pub = pob_b200.layout_info(pob_b200.MAIN_PROOF_OF_BURN)["n_outputs"]
    res["main_shape_n_pub"] = main_pub
    res["verify_ms"] = {}
    for n_pub in sorted({1, main_pub}):
        sim = Sim(n_pub, 7 + n_pub)
        x, y, z, pubs = sim.scalars(DISTINCT)
        proofs = sim.proofs(x, y, z)
        pub = _dev(limbs_of([v for p in pubs for v in p], 1 << 256)).view(DISTINCT, 4 * n_pub)
        vk = sim.vk
        kc = pob_b200.Groth16VkC(n_pub, *[t.data_ptr() for t in (vk.alpha1, vk.beta2, vk.gamma2, vk.delta2, vk.ic)])
        work = torch.empty(pob_b200.groth16_verify_work_bytes(n_pub, 1), dtype=torch.uint8, device="cuda")
        for n in (1, 1 << 10, 1 << 14, 1 << 17):
            P, U = tile(proofs, n), tile(pub, n)
            status = torch.full((n,), 9, dtype=torch.int32, device="cuda")
            import ctypes
            f = lambda: pob_b200._check(L.pob_groth16_verify(0, ctypes.byref(kc), P.data_ptr(), U.data_ptr(), n, status.data_ptr(),
                                                             work.data_ptr(), work.numel(), st))
            ms = timed(f, a.reps)
            assert int((status != 0).sum()) == 0, "a valid proof was rejected"
            res["verify_ms"]["n_pub=%d n=%d" % (n_pub, n)] = ms
            res["verify_ms"]["n_pub=%d n=%d per_proof_us" % (n_pub, n)] = 1000 * ms / n
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
