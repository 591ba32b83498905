"""ctypes front-end of the TEST-ONLY F_q2 / G2 probe (tests/devprobe/g2_probe.cu): the device arithmetic of csrc/fq2_hd.h on
caller-chosen operands, as Python ints, and the batched fixed-base [k_i]G over G1 and G2 that builds trapdoor proving keys."""
import ctypes, os, subprocess, tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "..", "proof-of-burn_b200", "csrc")
_LIB = None
MUL, SQR, ADD, SUB, NEG, INV = range(6)
G2_ADD, G2_ADD_AFF, G2_DBL, G2_DBL_AFF, G2_ADD_Z, G2_ADD_AFF_Z, G2_MUL_U32, G2_ADD_ZZ = range(8)


def build(out_dir=None):
    """compile the probe for sm_90a when it is missing or older than its sources; returns the .so path.  Falls back to a temporary
    directory when the tree is not writable."""
    from probe import nvcc
    srcs = [os.path.join(_HERE, "g2_probe.cu")] + [os.path.join(_CSRC, f) for f in ("fq2_hd.h", "fq_hd.h", "fr_hd.h")]
    so = os.path.join(out_dir or _HERE, "libg2_probe.so")
    if os.path.exists(so) and all(os.path.getmtime(s) <= os.path.getmtime(so) for s in srcs):
        return so
    if not os.access(os.path.dirname(so), os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix="g2_probe_"), "libg2_probe.so")
    nv = nvcc()
    if nv is None:
        raise RuntimeError("nvcc not found: the G2 probe cannot be built")
    subprocess.check_call([nv, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                           "-I", _CSRC, "-o", so, srcs[0], "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        vp, u32, ci = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int
        L.g2_probe_elem.restype = ci
        L.g2_probe_elem.argtypes = [ci, vp, vp, vp, u32]
        L.g2_probe_point.restype = ci
        L.g2_probe_point.argtypes = [ci, vp, vp, vp, vp, u32]
        L.g2_probe_fixed_base.restype = ci
        L.g2_probe_fixed_base.argtypes = [ci, vp, vp, ctypes.c_uint64, vp]
        _LIB = L
    return _LIB


def _limbs(vals):
    """F_q2 elements (c0, c1) -> (n, 16) uint32, raw (Montgomery form is the caller's business)"""
    return np.frombuffer(b"".join(int(c).to_bytes(32, "little") for v in vals for c in v), dtype=np.uint32).reshape(len(vals), 16).copy()


def elem(op, a, b=None):
    """[op(a_i, b_i)] over F_q2 as (c0, c1) int pairs, raw limbs in and out"""
    A = _limbs(a)
    B = _limbs(b) if b is not None else None
    out = np.zeros_like(A)
    rc = lib().g2_probe_elem(op, A.ctypes.data, None if B is None else B.ctypes.data, out.ctypes.data, len(a))
    if rc:
        raise RuntimeError("g2_probe_elem: CUDA error %d" % rc)
    raw = out.tobytes()
    return [(int.from_bytes(raw[64 * i:64 * i + 32], "little"), int.from_bytes(raw[64 * i + 32:64 * i + 64], "little")) for i in range(len(a))]


def point(op, a, b, k=None):
    """canonical affine results of a G2 point op; a, b lists of model points (None = infinity), given in Montgomery form"""
    import g2_model as g2m
    enc = lambda pts: np.ascontiguousarray(g2m.encode_points(pts).view(np.uint32))
    A, B = enc(a), enc(b)
    K = np.array(k if k is not None else [0] * len(a), dtype=np.uint32)
    out = np.zeros_like(A)
    rc = lib().g2_probe_point(op, A.ctypes.data, B.ctypes.data, K.ctypes.data, out.ctypes.data, len(a))
    if rc:
        raise RuntimeError("g2_probe_point: CUDA error %d" % rc)
    return [g2m.decode_point(row) for row in out.view(np.uint64).reshape(-1, 16)]


def fixed_base(group, scalars):
    """[k_i]G on the GPU for an (n, 4) uint64 CUDA tensor of scalars k_i: an (n, 8) (group 1) or (n, 16) (group 2) uint64 CUDA tensor
    of key-form points (affine, Montgomery), G the group's generator"""
    import torch
    import g1_model as gm
    import g2_model as g2m
    n = scalars.shape[0]
    assert scalars.is_cuda and scalars.is_contiguous() and scalars.shape[1] == 4
    g = np.ascontiguousarray((g2m.encode_points([g2m.G]) if group == 2 else gm.encode_bases([gm.G])).view(np.uint32))
    out = torch.empty((n, 16 if group == 2 else 8), dtype=torch.uint64, device=scalars.device)
    torch.cuda.synchronize()
    rc = lib().g2_probe_fixed_base(1 if group == 2 else 0, g.ctypes.data, scalars.data_ptr(), n, out.data_ptr())
    if rc:
        raise RuntimeError("g2_probe_fixed_base: CUDA error %d" % rc)
    return out
