#!/usr/bin/env python3
"""Does the code-tile kernel (4.1 % of the bytes, gathers from the instance stores) hide next to the round kernel (bandwidth-
bound) when both run at the same time on two streams?  (TUNING build: POB_CODES_OVERLAP = 0 after it, 1 next to it / round kernel
launched first, 2 next to it / code kernel launched first; POB_EXPAND_SMEM_KB = the round kernel's shared-memory cap, which decides
how many code CTAs fit beside its two resident CTAs.)  Staged 512-instance batch of the main shape, digests compared."""
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
CASES = [(0, 85), (1, 85), (2, 85), (1, 72), (2, 72), (1, 64), (0, 85)]
if len(sys.argv) > 1:
    CASES = [tuple(int(v) for v in a.split(",")) for a in sys.argv[1:]]
for overlap, smem_kb in CASES:
    os.environ.update({"POB_CODES_OVERLAP": str(overlap), "POB_EXPAND_SMEM_KB": str(smem_kb)})
    try:
        c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN)
        c.stage(packed)
        c.run_packed(None, n=512, staged=True, discard=True)
        t = [c.run_packed(None, n=512, staged=True, discard=True).timing for _ in range(3)]
        best = min(t, key=lambda q: q["total_ms"])
        dg = c.run_packed(packed[:3], digest=True)
        if ref is None:
            ref = dg.digests.copy()
        print(json.dumps({"codes_overlap": overlap, "expand_smem_kb": smem_kb, "wit_s": round(512 / (best["total_ms"] / 1e3), 1),
                          "expand_gbs": round(32.0 * c.n_signals * 512 / (best["expand_ms"] / 1e3) / 1e9, 1),
                          "digests_ok": bool(np.array_equal(dg.digests, ref))}), flush=True)
        c.close()
    except Exception as e:
        print(json.dumps({"codes_overlap": overlap, "expand_smem_kb": smem_kb, "error": str(e)}), flush=True)
