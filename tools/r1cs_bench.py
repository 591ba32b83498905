"""Time the `.r1cs` rows on the GPU for main_proof_of_burn, --O0 and reduced (--O1) witness: pob_r1cs_products over every row in
windows that fit a fixed buffer, the bytes/s it writes, and pob_r1cs_check next to pob_selfcheck.  Prints one JSON line (and
writes it to --out), with the card name and power limit read in the same run.

    python tools/r1cs_bench.py [--window-rows 16777216] [--reps 3] [--out r1cs_bench.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "proof-of-burn_b200")]


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"], out["max_sm_clock_mhz"] = float(q[0]), float(q[1])
    except Exception as e:          # the number is still reported, without the card's limit
        out["power_limit_w"] = "unavailable: %s" % e
    return out


def bench(opt, window, reps):
    import torch
    import pob_b200
    from pob_b200 import synth
    shape = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1, opt=opt)
    try:
        res = c.run_packed(synth.pack_instances(synth.make_batch(1, shape, seed=2718), shape))
        assert res.status[0] == 0
        chk = c.r1cs_check(0)                                  # builds and uploads the row plan
        rows = chk["n_constraints"]
        chk_ms = min(c.r1cs_check(0)["ms"] for _ in range(reps))
        self_ms = min(c.selfcheck(0)["ms"] for _ in range(reps)) if opt == 0 else None
        bufs = [torch.empty((window, 4), dtype=torch.uint64, device="cuda") for _ in range(3)]
        st = torch.cuda.Stream()
        L = pob_b200.lib()
        times = []
        for _ in range(reps + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for first in range(0, rows, window):
                n = min(window, rows - first)
                pob_b200._check(L.pob_r1cs_products(c._h, 0, first, n, bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(),
                                                    ctypes.c_void_p(st.cuda_stream)))
            e1.record(st)
            st.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = min(times[1:])
        return {"opt": opt, "rows": rows, "n_nonlinear": chk["n_nonlinear"], "window_rows": window, "buffer_bytes": 3 * 32 * window,
                "products_ms": ms, "products_ms_all": times[1:], "written_bytes": 96 * rows, "written_gbs": 96 * rows / ms / 1e6,
                "r1cs_check_ms": chk_ms, "selfcheck_ms": self_ms, "witness_entries": c.n_signals}
    finally:
        c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-rows", type=int, default=1 << 24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card(), "results": [bench(opt, a.window_rows, a.reps) for opt in (0, 1)]}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
