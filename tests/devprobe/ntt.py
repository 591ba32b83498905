"""ctypes front-end of the TEST-ONLY transform probe (tests/devprobe/ntt_probe.cu): the product's own pass plan, host tables and
transform launches of csrc/ntt.cuh at any 2^L, L <= 28.  plan() and tables() run on the host; inverse(), forward() and
quotient() transform caller CUDA tensors in place."""
import ctypes, os, subprocess, tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "..", "proof-of-burn_b200", "csrc")
_LIB = None
TABLES = ("w_lo", "w_hi", "loc", "loc_inv", "g_lo", "g_hi")
SYMBOLS = ("ntt_probe_plan", "ntt_probe_tables", "ntt_probe_inverse", "ntt_probe_forward", "ntt_probe_quotient")


def build(out_dir=None):
    """compile the probe for sm_90a when it is missing or older than its sources; returns the .so path.  Falls back to a temporary
    directory when the tree is not writable."""
    from probe import nvcc
    srcs = [os.path.join(_HERE, "ntt_probe.cu")] + [os.path.join(_CSRC, f) for f in ("ntt.cuh", "fr_hd.h")]
    so = os.path.join(out_dir or _HERE, "libntt_probe.so")
    if os.path.exists(so) and all(os.path.getmtime(s) <= os.path.getmtime(so) for s in srcs):
        return so
    if not os.access(os.path.dirname(so), os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix="ntt_probe_"), "libntt_probe.so")
    nv = nvcc()
    if nv is None:
        raise RuntimeError("nvcc not found: the transform probe cannot be built")
    subprocess.check_call([nv, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                           "-I", _CSRC, "-o", so, srcs[0], "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        vp, u32 = ctypes.c_void_p, ctypes.c_uint32
        L.ntt_probe_plan.restype = u32
        L.ntt_probe_plan.argtypes = [u32, vp]
        L.ntt_probe_tables.restype = None
        L.ntt_probe_tables.argtypes = [u32, vp, vp]
        for f, n in (("ntt_probe_inverse", 1), ("ntt_probe_forward", 1), ("ntt_probe_quotient", 3)):
            getattr(L, f).restype = ctypes.c_int
            getattr(L, f).argtypes = [u32] + [vp] * n
        _LIB = L
    return _LIB


def plan(L):
    """stages per pass of a 2^L transform, in the order of the inverse transform: ntt_plan(L, min(L, 11))"""
    out = (ctypes.c_uint32 * 32)()
    return list(out[:lib().ntt_probe_plan(L, out)])


def tables(L):
    """({name: (k, 8) uint32 limbs, Montgomery form, as stored}, g_log) of a 2^L domain"""
    sizes = np.zeros(7, dtype=np.uint64)
    lib().ntt_probe_tables(L, sizes.ctypes.data, None)
    flat = np.zeros((int(sizes[:6].sum()), 8), dtype=np.uint32)
    lib().ntt_probe_tables(L, sizes.ctypes.data, flat.ctypes.data)
    out, at = {}, 0
    for name, k in zip(TABLES, sizes[:6]):
        out[name] = flat[at:at + int(k)]
        at += int(k)
    return out, int(sizes[6])


def _vec(L, t):
    import torch
    assert t.is_cuda and t.dtype in (torch.uint64, torch.int64) and t.is_contiguous() and tuple(t.shape) == (1 << L, 4)
    assert t.data_ptr() % 16 == 0
    return t.data_ptr()


def _ok(rc, what):
    if rc != 0:
        raise RuntimeError("%s: CUDA error %d" % (what, rc))


def inverse(L, x):
    """x ((2^L, 4) canonical limbs on the GPU) in place: position j gets coefficient k = rev_L(j) times g^k (g = the coset shift)"""
    import torch
    torch.cuda.synchronize()
    _ok(lib().ntt_probe_inverse(L, _vec(L, x)), "ntt_probe_inverse")


def forward(L, x):
    """x in place: bit-reversed coefficients in, their values at w^i out"""
    import torch
    torch.cuda.synchronize()
    _ok(lib().ntt_probe_forward(L, _vec(L, x)), "ntt_probe_forward")


def quotient(L, a, b, c):
    """pob_r1cs_quotient's transform sequence on three row vectors: q = A.B - C on the coset, written over a; b and c are left
    transformed"""
    import torch
    torch.cuda.synchronize()
    _ok(lib().ntt_probe_quotient(L, _vec(L, a), _vec(L, b), _vec(L, c)), "ntt_probe_quotient")
