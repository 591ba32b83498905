#!/usr/bin/env python3
"""Can k_eval CTAs share SMs with the two resident k_expand_round CTAs?  (TUNING build.)  The round kernel caps itself at two CTAs
per SM with unused dynamic shared memory; with 85 KiB each there is no room left for an eval CTA (53 KiB of TMA-staged tables), with
<= 80 KiB there is (2 x 86 + 53 < 227 KiB; registers: 2 x 256 x 32 + 512 x 96 = 64 K).  Prints generation throughput of a staged
512-instance batch for several (shared-memory cap, eval shape) pairs."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "proof-of-burn_b200"))
import numpy as np
import pob_b200
from pob_b200 import synth

pob_b200.LIB_PATH = os.path.join(ROOT, "proof-of-burn_b200", "pob_b200", "libpob_b200_tuning.so")
shape = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)
packed = synth.pack_instances(synth.make_batch(512, shape, seed=5), shape)
ref = None
# (expand smem cap KB, eval threads, eval cluster)
CASES = [(85, 512, 0), (85, 512, 2), (85, 1024, 1)]
for smem_kb, threads, cluster in CASES:
    os.environ.update({"POB_EXPAND_SMEM_KB": str(smem_kb), "POB_EVAL_THREADS": str(threads), "POB_EVAL_CLUSTER": str(cluster)})
    try:
        c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN)
        c.stage(packed)
        c.run_packed(None, n=512, staged=True, discard=True)
        t = [c.run_packed(None, n=512, staged=True, discard=True).timing for _ in range(2)]
        best = min(t, key=lambda q: q["total_ms"])
        dg = c.run_packed(packed[:3], digest=True)
        if ref is None:
            ref = dg.digests.copy()
        print(json.dumps({"expand_smem_kb": smem_kb, "eval_threads": threads, "eval_cluster": cluster, "wit_s": round(512 / (best["total_ms"] / 1e3), 1),
                          "expand_gbs": round(32.0 * c.n_signals * 512 / (best["expand_ms"] / 1e3) / 1e9, 1), "eval_ms_per_launch": round(best["eval_ms"] / best["eval_launches"], 2),
                          "digests_ok": bool(np.array_equal(dg.digests, ref))}), flush=True)
        c.close()
    except Exception as e:
        print(json.dumps({"expand_smem_kb": smem_kb, "eval_threads": threads, "eval_cluster": cluster, "error": str(e)}), flush=True)
