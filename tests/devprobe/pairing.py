"""ctypes front-end of the TEST-ONLY tower and pairing probe (tests/devprobe/pairing_probe.cu): single operations of csrc/fq12_hd.h
and csrc/pairing.cuh on caller-chosen operands, in and out as the model's canonical values (tests/pairing_model.py)."""
import ctypes, os, subprocess, tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "..", "proof-of-burn_b200", "csrc")
_LIB = None
(FQ6_MUL, FQ6_SQR, FQ6_INV, FQ12_MUL, FQ12_SQR, FQ12_INV, FQ12_CONJ, FROB1, FROB2, FROB3, CYC_SQR, MUL_034,
 FINAL_EXP) = range(13)


def build(out_dir=None):
    """compile the probe for sm_90a when it is missing or older than its sources; returns the .so path.  Falls back to a temporary
    directory when the tree is not writable."""
    from probe import nvcc
    srcs = [os.path.join(_HERE, "pairing_probe.cu")] + [os.path.join(_CSRC, f) for f in ("pairing.cuh", "fq12_hd.h", "fq2_hd.h", "fq_hd.h", "fr_hd.h")]
    so = os.path.join(out_dir or _HERE, "libpairing_probe.so")
    if os.path.exists(so) and all(os.path.getmtime(s) <= os.path.getmtime(so) for s in srcs):
        return so
    if not os.access(os.path.dirname(so), os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix="pairing_probe_"), "libpairing_probe.so")
    nv = nvcc()
    if nv is None:
        raise RuntimeError("nvcc not found: the pairing probe cannot be built")
    subprocess.check_call([nv, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                           "-I", _CSRC, "-o", so, srcs[0], "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        vp, u32, ci = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int
        L.pairing_probe_elem.restype = ci
        L.pairing_probe_elem.argtypes = [ci, vp, vp, vp, u32]
        L.pairing_probe_miller.restype = ci
        L.pairing_probe_miller.argtypes = [vp, vp, vp, vp, u32]
        _LIB = L
    return _LIB


def _enc(vals):
    """model F_q12 values -> (n, 96) uint32, Montgomery form"""
    import g1_model as gm
    import pairing_model as pm
    raw = b"".join(gm.to_mont(c).to_bytes(32, "little") for v in vals for c in pm.coeffs(v))
    return np.frombuffer(raw, dtype=np.uint32).reshape(len(vals), 96).copy()


def _dec(arr):
    import g1_model as gm
    import pairing_model as pm
    raw = arr.tobytes()
    return [pm.from_coeffs(gm.from_mont(int.from_bytes(raw[384 * i + 32 * k:384 * i + 32 * k + 32], "little")) for k in range(12))
            for i in range(arr.shape[0])]


def elem(op, a, b=None):
    """[op(a_i, b_i)] as model F_q12 values (F_q6 ops: on and into the c0 halves)"""
    A = _enc(a)
    B = _enc(b) if b is not None else None
    out = np.zeros_like(A)
    rc = lib().pairing_probe_elem(op, A.ctypes.data, None if B is None else B.ctypes.data, out.ctypes.data, len(a))
    if rc:
        raise RuntimeError("pairing_probe_elem: CUDA error %d" % rc)
    return _dec(out)


def miller(g1s, g2s):
    """([f_i], [in_g2_i]): the device Miller loop of each pair (its value before the final exponentiation) and [r]Q = O"""
    import g1_model as gm
    import g2_model as g2m
    P = np.ascontiguousarray(gm.encode_bases(g1s).view(np.uint32))
    Q = np.ascontiguousarray(g2m.encode_points(g2s).view(np.uint32))
    out = np.zeros((len(g1s), 96), dtype=np.uint32)
    flag = np.zeros(len(g1s), dtype=np.uint32)
    rc = lib().pairing_probe_miller(P.ctypes.data, Q.ctypes.data, out.ctypes.data, flag.ctypes.data, len(g1s))
    if rc:
        raise RuntimeError("pairing_probe_miller: CUDA error %d" % rc)
    return _dec(out), [bool(x) for x in flag]
