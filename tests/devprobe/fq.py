"""ctypes front-end of the TEST-ONLY F_q / G1 probe (tests/devprobe/fq_probe.cu): the device arithmetic of csrc/fq_hd.h on
caller-chosen operands, as Python ints."""
import ctypes, os, subprocess, tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "..", "proof-of-burn_b200", "csrc")
_LIB = None
MUL, ADD, SUB, INV, TO_MONT, FROM_MONT, NEG = range(7)
G1_ADD, G1_ADD_AFF, G1_DBL, G1_DBL_AFF, G1_ADD_Z, G1_ADD_AFF_Z, G1_MUL_U32 = range(7)


def build(out_dir=None):
    """compile the probe for sm_90a when it is missing or older than its sources; returns the .so path.  Falls back to a temporary
    directory when the tree is not writable."""
    from probe import nvcc
    srcs = [os.path.join(_HERE, "fq_probe.cu")] + [os.path.join(_CSRC, f) for f in ("fq_hd.h", "fr_hd.h")]
    so = os.path.join(out_dir or _HERE, "libfq_probe.so")
    if os.path.exists(so) and all(os.path.getmtime(s) <= os.path.getmtime(so) for s in srcs):
        return so
    if not os.access(os.path.dirname(so), os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix="fq_probe_"), "libfq_probe.so")
    nv = nvcc()
    if nv is None:
        raise RuntimeError("nvcc not found: the F_q probe cannot be built")
    subprocess.check_call([nv, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                           "-I", _CSRC, "-o", so, srcs[0], "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        vp, u32, ci = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int
        L.fq_probe_elem.restype = ci
        L.fq_probe_elem.argtypes = [ci, vp, vp, vp, u32]
        L.fq_probe_point.restype = ci
        L.fq_probe_point.argtypes = [ci, vp, vp, vp, vp, u32]
        _LIB = L
    return _LIB


def _limbs(vals, words):
    return np.frombuffer(b"".join(int(v).to_bytes(4 * words, "little") for v in vals), dtype=np.uint32).reshape(len(vals), words).copy()


def _ints(arr, words):
    return [int.from_bytes(row.tobytes(), "little") for row in arr.reshape(-1, words)]


def elem(op, a, b=None):
    """[op(a_i, b_i)] over F_q as ints (raw limbs in and out: Montgomery form is the caller's business)"""
    A = _limbs(a, 8)
    B = _limbs(b, 8) if b is not None else None
    out = np.zeros_like(A)
    rc = lib().fq_probe_elem(op, A.ctypes.data, None if B is None else B.ctypes.data, out.ctypes.data, len(a))
    if rc:
        raise RuntimeError("fq_probe_elem: CUDA error %d" % rc)
    return _ints(out, 8)


def point(op, a, b, k=None):
    """canonical affine results of a point op; a, b lists of model points (None = infinity), given to the device in Montgomery form"""
    import g1_model as gm
    enc = lambda pts: np.ascontiguousarray(gm.encode_bases(pts).view(np.uint32))
    A, B = enc(a), enc(b)
    K = np.array(k if k is not None else [0] * len(a), dtype=np.uint32)
    out = np.zeros_like(A)
    rc = lib().fq_probe_point(op, A.ctypes.data, B.ctypes.data, K.ctypes.data, out.ctypes.data, len(a))
    if rc:
        raise RuntimeError("fq_probe_point: CUDA error %d" % rc)
    return [gm.decode_point(row) for row in out.view(np.uint64).reshape(-1, 8)]
