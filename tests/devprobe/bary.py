"""ctypes front-end of the TEST-ONLY barycentric evaluator (tests/devprobe/bary_probe.cu): the polynomial through a device vector,
evaluated at one point on the GPU from the formula alone.  Used by tests/test_gpu_quotient.py for vectors too long for Python."""
import ctypes, os, subprocess, tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "..", "..", "proof-of-burn_b200", "csrc")
_LIB = None


def build(out_dir=None):
    """compile the evaluator for sm_90a when it is missing or older than its sources; returns the .so path.  Falls back to a
    temporary directory when the tree is not writable."""
    from probe import nvcc
    srcs = [os.path.join(_HERE, "bary_probe.cu"), os.path.join(_CSRC, "fr_hd.h")]
    so = os.path.join(out_dir or _HERE, "libbary_probe.so")
    if os.path.exists(so) and all(os.path.getmtime(s) <= os.path.getmtime(so) for s in srcs):
        return so
    if not os.access(os.path.dirname(so), os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix="bary_probe_"), "libbary_probe.so")
    nv = nvcc()
    if nv is None:
        raise RuntimeError("nvcc not found: the barycentric probe cannot be built")
    subprocess.check_call([nv, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                           "-I", _CSRC, "-o", so, srcs[0], "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        L.bary_probe_eval.restype = ctypes.c_int
        L.bary_probe_eval.argtypes = [vp, u64, u64, vp, vp, vp, u32, vp]
        _LIB = L
    return _LIB


def _limbs8(v):
    return (ctypes.c_uint32 * 8)(*[(int(v) >> (32 * i)) & 0xFFFFFFFF for i in range(8)])


def evaluate(ptr, count, shift, omega, log_n, r, first=0):
    """sum_i v_i L_(first+i)(r) over the points shift omega^j of a 2^log_n domain, v = `count` canonical 32-byte entries at device
    pointer `ptr` (the caller orders the writes of v before this call)"""
    res = (ctypes.c_uint32 * 8)()
    rc = lib().bary_probe_eval(ptr, first, count, _limbs8(shift), _limbs8(omega), _limbs8(r), log_n, res)
    if rc != 0:
        raise RuntimeError("bary_probe_eval: CUDA error %d" % rc)
    return int.from_bytes(bytes(res), "little")
