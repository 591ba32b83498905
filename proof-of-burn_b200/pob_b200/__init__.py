"""pob_b200 -- Python host of the H100-native batched witness generator (ctypes over libpob_b200.so).

Mirrors the reference's interface for this path: the process CLI the circom toolchain emits,
`./<circuit> input.json witness.wtns` (reference Makefile:5-6, tests/test.py:60-63), with the input-JSON
schema tests/main.py:160-178 writes (keys = the main template's `signal input` names, values JSON ints or
decimal strings, nested arrays, scalars possibly wrapped in 1-element arrays).

    from pob_b200 import Circuit
    c = Circuit("ProofOfBurn(16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)")       # == circom -c + make
    res = c.run([input_dict, ...])                                              # == N x ./main input.json w.wtns
    res.status[i] == 0, res.outputs[i] -> [commitment]; c.write_wtns(i, "witness.wtns")

All witness computation happens in hand-written CUDA (csrc/pob_b200.cu).  There is no CPU fallback: if the
extension is missing or no GPU is visible, construction fails loudly.
"""
import collections
import ctypes
import json
import os
import re

import numpy as np

P = 21888242871839275222246405745257275088548364400416034343698204186575808495617
R_ORDER = P                                       # BN254's group order r is the scalar field's modulus
Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583   # BN254's base field modulus
_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpob_b200.so")

RUN_EXPAND, RUN_DIGEST, RUN_INPUTS_STAGED, RUN_DISCARD = 1, 2, 4, 8
CREATE_HCREATE, CREATE_O1 = 1, 0x100
E_RANGE, E_REJECTED, E_BUSY, E_KEY, DONE = -5, -8, -9, -10, 1
VERIFY_STATUS = ("OK", "FAIL", "BAD_POINT", "BAD_SUBGROUP", "BAD_PUBLIC", "BAD_KEY")    # pob_b200.h: POB_VERIFY_*, by value
MAIN_PROOF_OF_BURN = "ProofOfBurn(16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)"   # circuits/main_proof_of_burn.circom:27
MAIN_SPEND = "Spend(31)"                                                       # circuits/main_spend.circom:6
TEST_PROOF_OF_BURN = "ProofOfBurn(4, 4, 5, 20, 31, 2, 10 ** 18, 10 ** 19)"     # tests/testcases/proof_of_burn.py:53


class PobError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("pob_b200 error %d: %s" % (code, msg))
        self.code = code


class Desc(ctypes.Structure):
    _fields_ = [("n_signals", ctypes.c_uint64), ("n_outputs", ctypes.c_uint32), ("n_inputs", ctypes.c_uint32),
                ("witness_bytes", ctypes.c_uint64), ("wtns_file_bytes", ctypes.c_uint64), ("store_bytes", ctypes.c_uint64),
                ("n_ops", ctypes.c_uint64), ("n_absorbs", ctypes.c_uint32), ("n_levels", ctypes.c_uint32),
                ("n_tiles", ctypes.c_uint32), ("n_slots", ctypes.c_uint32), ("chunk", ctypes.c_uint32), ("expand_group", ctypes.c_uint32),
                ("opt_level", ctypes.c_uint32), ("n_signals_o0", ctypes.c_uint64), ("n_compressed_slots", ctypes.c_uint32)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class Timing(ctypes.Structure):
    _fields_ = [("total_ms", ctypes.c_float), ("expand_ms", ctypes.c_float), ("eval_ms", ctypes.c_float),
                ("expand_launches", ctypes.c_uint32), ("eval_launches", ctypes.c_uint32), ("other_launches", ctypes.c_uint32),
                ("h2d_bytes", ctypes.c_uint64), ("d2h_bytes", ctypes.c_uint64),
                ("eval_clusters", ctypes.c_uint32)]     # bit C: some eval launch ran C CTAs per instance

    def as_dict(self):
        return {k: (float(getattr(self, k)) if k.endswith("_ms") else int(getattr(self, k))) for k, _ in self._fields_}


class ExportStats(ctypes.Structure):
    _fields_ = [("witnesses", ctypes.c_uint64), ("bytes", ctypes.c_uint64), ("total_ms", ctypes.c_float), ("d2h_gbs", ctypes.c_float)]

    def as_dict(self):
        return {"witnesses": int(self.witnesses), "bytes": int(self.bytes), "total_ms": float(self.total_ms), "d2h_gbs": float(self.d2h_gbs)}


class CheckReport(ctypes.Structure):
    _fields_ = [("n_constraints", ctypes.c_uint64), ("n_nonlinear", ctypes.c_uint64), ("n_hints", ctypes.c_uint64), ("n_failed", ctypes.c_uint64),
                ("n_hint_failed", ctypes.c_uint64), ("first_failed", ctypes.c_uint64), ("signals_read", ctypes.c_uint64), ("ms", ctypes.c_float)]

    def as_dict(self):
        return {k: (float(getattr(self, k)) if k == "ms" else int(getattr(self, k))) for k, _ in self._fields_}


class R1csDesc(ctypes.Structure):
    _fields_ = [("n_wires", ctypes.c_uint64), ("n_pub_out", ctypes.c_uint32), ("n_pub_in", ctypes.c_uint32), ("n_prv_in", ctypes.c_uint32),
                ("n_labels", ctypes.c_uint64), ("n_constraints", ctypes.c_uint64), ("n_nonlinear", ctypes.c_uint64), ("n_terms", ctypes.c_uint64),
                ("file_bytes", ctypes.c_uint64)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class Groth16KeyC(ctypes.Structure):
    """pob_b200.h: pob_groth16_key"""
    _fields_ = [("n_vars", ctypes.c_uint64), ("n_pub", ctypes.c_uint32), ("log_n", ctypes.c_uint32)] + \
        [(f, ctypes.c_void_p) for f in ("alpha1", "beta1", "delta1", "beta2", "delta2", "a", "b1", "b2", "c", "h")]


class Groth16Key(collections.namedtuple("Groth16Key", "alpha1 beta1 delta1 beta2 delta2 a b1 b2 c h")):
    """A Groth16 proving key as CUDA tensors (pob_b200.h: pob_groth16_key): G1 points are (k, 8) uint64 tensors and G2 points (k, 16),
    affine, Montgomery-form F_q limbs as msm_g1 / msm_g2 take them.  alpha1, beta1, delta1: one G1 point each; beta2, delta2: one G2
    point each; a, b1: n_signals G1 points; b2: n_signals G2 points; c: n_signals - n_outputs - 1 G1 points (wires n_outputs + 1 ..);
    h: 2^r1cs_domain() G1 points, paired with the quotient's q[k]."""


class ZkeyDesc(ctypes.Structure):
    """pob_b200.h: pob_zkey_desc"""
    _fields_ = [("n_vars", ctypes.c_uint64), ("n_pub", ctypes.c_uint32), ("log_n", ctypes.c_uint32), ("n_coefs", ctypes.c_uint64),
                ("file_bytes", ctypes.c_uint64), ("a_bytes", ctypes.c_uint64), ("b1_bytes", ctypes.c_uint64), ("b2_bytes", ctypes.c_uint64),
                ("c_bytes", ctypes.c_uint64), ("h_bytes", ctypes.c_uint64), ("key_bytes", ctypes.c_uint64)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class ZkeyReport(ctypes.Structure):
    """pob_b200.h: pob_zkey_report"""
    _fields_ = [("coef_match", ctypes.c_uint32), ("coef_match_canonical", ctypes.c_uint32), ("coef_out_of_range", ctypes.c_uint64),
                ("points_checked", ctypes.c_uint64), ("points_bad", ctypes.c_uint64), ("points_bad_canonical", ctypes.c_uint64),
                ("first_bad_section", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("first_bad_index", ctypes.c_uint64),
                ("read_ms", ctypes.c_float), ("copy_ms", ctypes.c_float), ("check_ms", ctypes.c_float), ("total_ms", ctypes.c_float),
                ("bytes_read", ctypes.c_uint64), ("device_scratch_bytes", ctypes.c_uint64)]

    def as_dict(self):
        return {k: (float(getattr(self, k)) if k.endswith("_ms") else int(getattr(self, k))) for k, _ in self._fields_ if k != "reserved"}


class Groth16VkC(ctypes.Structure):
    """pob_b200.h: pob_groth16_vk"""
    _fields_ = [("n_pub", ctypes.c_uint32)] + [(f, ctypes.c_void_p) for f in ("alpha1", "beta2", "gamma2", "delta2", "ic")]


class ZkeyError(PobError):
    """a .zkey that does not fit the circuit (POB_E_KEY); .report is the check's report (a dict), None when it was refused on its header"""

    def __init__(self, code, msg, report=None):
        super().__init__(code, msg)
        self.report = report


class Proof(collections.namedtuple("Proof", "a b c")):
    """A Groth16 proof as ints: a and c are G1 points (x, y), b a G2 point ((x0, x1), (y0, y1)) with x = x0 + x1 u; None = infinity."""

    def to_json(self):
        """the proof.json dictionary of snarkjs (pi_a, pi_b, pi_c as projective decimal strings with z = 1, pi_b coordinates as
        [c0, c1]).  The shape follows snarkjs as far as it is known here; it has not been checked against snarkjs."""
        return {"pi_a": _g1_json(self.a), "pi_b": _g2_json(self.b), "pi_c": _g1_json(self.c), "protocol": "groth16", "curve": "bn128"}

    @classmethod
    def from_json(cls, d):
        """the inverse of to_json: z = 1, or the infinity encodings to_json writes; anything else raises ValueError"""
        return cls(_g1_from_json(d["pi_a"]), _g2_from_json(d["pi_b"]), _g1_from_json(d["pi_c"]))


def _g1_json(p):
    return ["0", "1", "0"] if p is None else [str(p[0]), str(p[1]), "1"]


def _g2_json(p):
    if p is None:
        return [["0", "0"], ["1", "0"], ["0", "0"]]
    return [[str(p[0][0]), str(p[0][1])], [str(p[1][0]), str(p[1][1])], ["1", "0"]]


def _g1_from_json(v):
    v = [str(x) for x in v]
    if v == ["0", "1", "0"]:
        return None
    if len(v) != 3 or v[2] != "1":
        raise ValueError("a G1 point must be [x, y, 1] or [0, 1, 0] (infinity): %r" % (v,))
    return (int(v[0]), int(v[1]))


def _g2_from_json(v):
    v = [[str(x) for x in c] for c in v]
    if v == [["0", "0"], ["1", "0"], ["0", "0"]]:
        return None
    if len(v) != 3 or any(len(c) != 2 for c in v) or v[2] != ["1", "0"]:
        raise ValueError("a G2 point must be [[x0, x1], [y0, y1], [1, 0]] or [[0, 0], [1, 0], [0, 0]] (infinity): %r" % (v,))
    return ((int(v[0][0]), int(v[0][1])), (int(v[1][0]), int(v[1][1])))


def public_json(outputs):
    """the public signals of a proof (snarkjs public.json: decimal strings), from the circuit's outputs (BatchResult.outputs[i])"""
    return [str(int(v) % P) for v in outputs]


_LIB = None


def lib():
    """Load the CUDA extension.  Fails loudly when it has not been built (python __graft_entry__.py build)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("pob_b200: %s is missing -- build it with `make -C proof-of-burn_b200/csrc` "
                              "(there is no CPU fallback)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        vp, u32, u64, ci = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int
        L.pob_create.restype = ci
        L.pob_create.argtypes = [ctypes.c_char_p, vp, ci, ci, ci, u32, ctypes.POINTER(vp)]
        L.pob_destroy.argtypes = [vp]
        L.pob_layout_info.restype = ci
        L.pob_layout_info.argtypes = [ctypes.c_char_p, vp, ci, ci, ctypes.POINTER(Desc)]
        L.pob_input_schema.restype = ctypes.c_char_p
        L.pob_input_schema.argtypes = [ctypes.c_char_p, ctypes.POINTER(ci)]
        L.pob_describe.restype = ci
        L.pob_describe.argtypes = [vp, ctypes.POINTER(Desc)]
        L.pob_alloc_pinned.restype = vp
        L.pob_alloc_pinned.argtypes = [u64]
        L.pob_free_pinned.argtypes = [vp]
        L.pob_stage_inputs.restype = ci
        L.pob_stage_inputs.argtypes = [vp, vp, u32]
        L.pob_run_batch.restype = ci
        L.pob_run_batch.argtypes = [vp, vp, u32, u32, vp, vp, vp]
        L.pob_last_timing.restype = ci
        L.pob_last_timing.argtypes = [vp, ctypes.POINTER(Timing)]
        L.pob_copy_witness.restype = ci
        L.pob_copy_witness.argtypes = [vp, u32, u64, u64, vp]
        L.pob_write_wtns.restype = ci
        L.pob_write_wtns.argtypes = [vp, u32, ctypes.c_char_p]
        L.pob_witness_device_ptr.restype = ci
        L.pob_witness_device_ptr.argtypes = [vp, u32, ctypes.POINTER(vp)]
        L.pob_selfcheck_keccak.restype = ci
        L.pob_selfcheck_keccak.argtypes = [vp, u32, ctypes.POINTER(u64), ctypes.POINTER(u64)]
        L.pob_selfcheck.restype = ci
        L.pob_selfcheck.argtypes = [vp, u32, ctypes.POINTER(CheckReport)]
        L.pob_constraint_info.restype = ci
        L.pob_constraint_info.argtypes = [ctypes.c_char_p, vp, ci, ci, ctypes.POINTER(CheckReport)]
        L.pob_write_components.restype = ci
        L.pob_write_components.argtypes = [ctypes.c_char_p, vp, ci, ci, ctypes.c_char_p, ctypes.POINTER(u64)]
        L.pob_witness_map.restype = ci
        L.pob_witness_map.argtypes = [vp, vp]
        L.pob_run_batch_retain.restype = ci
        L.pob_run_batch_retain.argtypes = [vp, vp, u32, u32, vp, u32, vp, vp, vp]
        L.pob_submit.restype = ci
        L.pob_submit.argtypes = [vp, vp, u32, u32]
        L.pob_acquire.restype = ci
        L.pob_acquire.argtypes = [vp, ctypes.POINTER(u32), ctypes.POINTER(vp), vp]
        L.pob_release.restype = ci
        L.pob_release.argtypes = [vp, u32, vp]
        L.pob_finish.restype = ci
        L.pob_finish.argtypes = [vp, vp, vp, vp]
        L.pob_export_batch.restype = ci
        L.pob_export_batch.argtypes = [vp, vp, u32, u32, vp, vp, vp, ctypes.POINTER(ExportStats)]
        L.pob_write_r1cs.restype = ci
        L.pob_write_r1cs.argtypes = [ctypes.c_char_p, vp, ci, ci, ctypes.c_char_p, ctypes.POINTER(R1csDesc)]
        L.pob_r1cs_check.restype = ci
        L.pob_r1cs_check.argtypes = [vp, u32, ctypes.POINTER(CheckReport)]
        L.pob_r1cs_products.restype = ci
        L.pob_r1cs_products.argtypes = [vp, u32, u64, u64, vp, vp, vp, vp]
        L.pob_r1cs_domain.restype = ci
        L.pob_r1cs_domain.argtypes = [vp, ctypes.POINTER(u32)]
        L.pob_r1cs_quotient.restype = ci
        L.pob_r1cs_quotient.argtypes = [vp, u32, vp, vp, vp]
        L.pob_msm_g1_work_bytes.restype = ci
        L.pob_msm_g1_work_bytes.argtypes = [u64, ctypes.POINTER(u64)]
        L.pob_msm_g1.restype = ci
        L.pob_msm_g1.argtypes = [ci, vp, vp, u64, vp, vp, u64, vp]
        L.pob_msm_g2_work_bytes.restype = ci
        L.pob_msm_g2_work_bytes.argtypes = [u64, ctypes.POINTER(u64)]
        L.pob_msm_g2.restype = ci
        L.pob_msm_g2.argtypes = [ci, vp, vp, u64, vp, vp, u64, vp]
        L.pob_groth16_work_bytes.restype = ci
        L.pob_groth16_work_bytes.argtypes = [vp, ctypes.POINTER(u64)]
        L.pob_groth16_prove.restype = ci
        L.pob_groth16_prove.argtypes = [vp, u32, ctypes.POINTER(Groth16KeyC), vp, vp, vp, vp, u64, vp]
        L.pob_zkey_info.restype = ci
        L.pob_zkey_info.argtypes = [ctypes.c_char_p, ctypes.POINTER(ZkeyDesc)]
        L.pob_zkey_load.restype = ci
        L.pob_zkey_load.argtypes = [vp, ctypes.c_char_p, u64, u64, ctypes.POINTER(Groth16KeyC), ctypes.POINTER(ZkeyReport)]
        L.pob_zkey_vk.restype = ci
        L.pob_zkey_vk.argtypes = [ctypes.c_char_p, vp, u64, ctypes.POINTER(u32)]
        L.pob_bn254_pairing.restype = ci
        L.pob_bn254_pairing.argtypes = [ci, vp, vp, u64, vp, vp]
        L.pob_groth16_verify_work_bytes.restype = ci
        L.pob_groth16_verify_work_bytes.argtypes = [u32, u64, ctypes.POINTER(u64)]
        L.pob_groth16_verify.restype = ci
        L.pob_groth16_verify.argtypes = [ci, ctypes.POINTER(Groth16VkC), vp, vp, u64, vp, vp, u64, vp]
        L.pob_pow_grind.restype = ci
        L.pob_pow_grind.argtypes = [ci, vp, vp, vp, u32, u64, vp, ctypes.POINTER(u64)]
        L.pob_last_error.restype = ctypes.c_char_p
        L.pob_version.restype = ctypes.c_char_p
        _LIB = L
    return _LIB


def _check(rc):
    if rc != 0:
        raise PobError(rc, lib().pob_last_error().decode())


# ---- field / schema helpers --------------------------------------------------------------------------------
def eval_int_expr(text, env=None):
    """Template parameters and schema dimensions are tiny integer expressions (`10 ** 19`, `p1*136`, `2*p0`): evaluate
    them with a whitelisted AST walk -- integers, names from `env`, + - * // ** and unary minus; nothing else."""
    import ast
    import operator
    ops = {ast.Add: operator.add, ast.Sub: operator.sub, ast.Mult: operator.mul, ast.FloorDiv: operator.floordiv, ast.Pow: operator.pow}

    def ev(n):
        if isinstance(n, ast.Expression):
            return ev(n.body)
        if isinstance(n, ast.Constant) and isinstance(n.value, int) and not isinstance(n.value, bool):
            return n.value
        if isinstance(n, ast.Name) and env is not None and n.id in env:
            return int(env[n.id])
        if isinstance(n, ast.UnaryOp) and isinstance(n.op, ast.USub):
            return -ev(n.operand)
        if isinstance(n, ast.BinOp) and type(n.op) in ops:
            a, b = ev(n.left), ev(n.right)
            if isinstance(n.op, ast.Pow) and (b < 0 or b > 4096 or abs(a) > 1 << 64):
                raise ValueError("exponent out of range in %r" % text)
            return ops[type(n.op)](a, b)
        raise ValueError("unsupported expression %r" % text)
    return int(ev(ast.parse(text.strip(), mode="eval")))


def parse_int(v):
    """one input value: JSON int, decimal string, or 0x-prefixed hex string (some circom loaders accept it)"""
    if isinstance(v, str):
        t = v.strip()
        return int(t, 16) if t.lower().startswith(("0x", "-0x")) else int(t)
    return int(v)


def parse_main(expr):
    """'ProofOfBurn(4, 4, 5, 20, 31, 2, 10 ** 18, 10 ** 19)' -> ('ProofOfBurn', [4, 4, 5, 20, 31, 2, 10**18, 10**19])"""
    m = re.match(r"\s*(\w+)\s*(?:\((.*)\))?\s*;?\s*$", expr, re.S)
    if not m:
        raise ValueError("cannot parse main expression %r" % expr)
    args = (m.group(2) or "").strip()
    return m.group(1), ([eval_int_expr(a) for a in args.split(",")] if args else [])


def to_limbs(vals):
    """ints of any sign/size (reduced mod p like the circom loader) -> (n, 4) uint64 little-endian limbs"""
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        v = int(v) % P
        if v >> 64:
            for k in range(4):
                out[i, k] = (v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF
        else:
            out[i, 0] = v
    return out


def from_limbs(row):
    return int(row[0]) | (int(row[1]) << 64) | (int(row[2]) << 128) | (int(row[3]) << 192)


def input_schema(name, params):
    """[(input name, [dims])] in declaration order, from the library (single source of truth)."""
    n = ctypes.c_int(0)
    s = lib().pob_input_schema(name.encode(), ctypes.byref(n))
    if s is None:
        raise PobError(-1, "unknown main template %r" % name)
    if len(params) < n.value:
        raise PobError(-1, "%s needs %d template parameters" % (name, n.value))
    env = {"p%d" % i: v for i, v in enumerate(params)}
    out = []
    for item in [x for x in s.decode().split(",") if x]:
        m = re.match(r"(\w+)((?:\[[^\]]+\])*)$", item)
        out.append((m.group(1), [eval_int_expr(d, env) for d in re.findall(r"\[([^\]]+)\]", m.group(2))]))
    return out


def _flatten(v, out):
    if isinstance(v, (list, tuple)):
        for e in v:
            _flatten(e, out)
    else:
        out.append(parse_int(v))


def flatten_input(schema, inp):
    """One input JSON object -> flat list of ints in declaration order.  Element counts must match the circuit
    exactly, as with the circom loader; unknown keys are ignored, missing keys are an error."""
    flat = []
    for name, dims in schema:
        if name not in inp:
            raise KeyError("input signal %r missing" % name)
        vals = []
        _flatten(inp[name], vals)
        want = int(np.prod(dims)) if dims else 1
        if len(vals) != want:
            raise ValueError("input %s: circuit expects %d values, got %d" % (name, want, len(vals)))
        flat.extend(vals)
    return flat


def layout_info(main_expr, hcreate=False, opt=0):
    """Shape of a circuit's witness program; runs the host-side layout compiler only (no GPU needed)."""
    name, params = parse_main(main_expr)
    pl = to_limbs(params) if params else np.zeros((1, 4), dtype=np.uint64)
    d = Desc()
    _check(lib().pob_layout_info(name.encode(), pl.ctypes.data, len(params), (CREATE_HCREATE if hcreate else 0) | (CREATE_O1 if opt else 0), ctypes.byref(d)))
    return d.as_dict()


def constraint_info(main_expr, hcreate=False):
    """size of a circuit shape's constraint system (host only): constraints, non-linear ones, hint records, signals covered"""
    name, params = parse_main(main_expr)
    pl = to_limbs(params) if params else np.zeros((1, 4), dtype=np.uint64)
    r = CheckReport()
    _check(lib().pob_constraint_info(name.encode(), pl.ctypes.data, len(params), int(hcreate), ctypes.byref(r)))
    return r.as_dict()


def write_components(main_expr, path, hcreate=False):
    """order-pinning kit: component list (`first_signal,n_own_signals,template` per line) of the --O0 layout; see tools/diff_sym.py"""
    name, params = parse_main(main_expr)
    pl = to_limbs(params) if params else np.zeros((1, 4), dtype=np.uint64)
    n = ctypes.c_uint64(0)
    _check(lib().pob_write_components(name.encode(), pl.ctypes.data, len(params), CREATE_HCREATE if hcreate else 0, os.fsencode(path), ctypes.byref(n)))
    return int(n.value)


def write_r1cs(main_expr, path=None, hcreate=False, opt=0):
    """the circuit's iden3 `.r1cs` (pob_b200.h: pob_write_r1cs), over the --O0 witness or, with opt=1, the reduced one; its wire
    order is the order of the witness this library writes.  path=None: sizes only.  Returns the header counts and file_bytes."""
    name, params = parse_main(main_expr)
    pl = to_limbs(params) if params else np.zeros((1, 4), dtype=np.uint64)
    d = R1csDesc()
    _check(lib().pob_write_r1cs(name.encode(), pl.ctypes.data, len(params), (CREATE_HCREATE if hcreate else 0) | (CREATE_O1 if opt else 0),
                                None if path is None else os.fsencode(path), ctypes.byref(d)))
    return d.as_dict()


def zkey_info(path):
    """header of a snarkjs `.zkey` (pob_zkey_info; host only, no GPU): n_vars, n_pub, log_n, n_coefs, file_bytes and the device bytes
    of each key section.  A malformed file raises ZkeyError (E_KEY) or PobError (-6, I/O)."""
    d = ZkeyDesc()
    rc = lib().pob_zkey_info(os.fsencode(path), ctypes.byref(d))
    if rc == E_KEY:
        raise ZkeyError(rc, lib().pob_last_error().decode())
    _check(rc)
    return d.as_dict()


class PinnedArray:
    """numpy view over cudaMallocHost memory (so H2D copies inside run() are asynchronous DMA)."""

    def __init__(self, shape, dtype):
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self.ptr = lib().pob_alloc_pinned(max(1, self.nbytes))
        if not self.ptr:
            raise PobError(-3, "pob_alloc_pinned failed")
        buf = (ctypes.c_uint8 * max(1, self.nbytes)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def free(self):
        if self.ptr:
            self.array = None
            lib().pob_free_pinned(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class BatchResult:
    def __init__(self, status, outputs, digests, timing):
        self.status, self.outputs_limbs, self.digests, self.timing = status, outputs, digests, timing

    @property
    def n_ok(self):
        return int((self.status == 0).sum())

    @property
    def outputs(self):
        return [[from_limbs(r) for r in inst] for inst in self.outputs_limbs]


class Circuit:
    """One compiled circuit shape bound to one GPU (== the executable `circom -c ... && make` produces)."""

    def __init__(self, main_expr, device=0, hcreate=False, max_slots=0, opt=0):
        """opt=1: the reduced (`--O1`-style) witness (pob_b200.h: POB_CREATE_O1); witness_map() gives the --O0 index of each entry"""
        self.main_expr, self.device = main_expr, int(device)
        self.name, self.params = parse_main(main_expr)
        self.schema = input_schema(self.name, self.params)
        pl = to_limbs(self.params) if self.params else np.zeros((1, 4), dtype=np.uint64)
        h = ctypes.c_void_p()
        _check(lib().pob_create(self.name.encode(), pl.ctypes.data, len(self.params), (CREATE_HCREATE if hcreate else 0) | (CREATE_O1 if opt else 0),
                                int(device), int(max_slots), ctypes.byref(h)))
        self._h = h
        d = Desc()
        _check(lib().pob_describe(self._h, ctypes.byref(d)))
        self.desc = d.as_dict()
        self.n_signals, self.n_inputs, self.n_outputs = self.desc["n_signals"], self.desc["n_inputs"], self.desc["n_outputs"]

    def close(self):
        if getattr(self, "_h", None):
            lib().pob_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- inputs ----
    def pack(self, inputs, pinned=False):
        """list of input JSON objects (or one) -> (n, n_inputs, 4) uint64 array"""
        if isinstance(inputs, dict):
            inputs = [inputs]
        n = len(inputs)
        shape = (n, max(1, self.n_inputs), 4)
        holder = PinnedArray(shape, np.uint64) if pinned else None
        arr = holder.array if pinned else np.zeros(shape, dtype=np.uint64)
        for i, inp in enumerate(inputs):
            arr[i, : self.n_inputs] = to_limbs(flatten_input(self.schema, inp))
        return (arr, holder) if pinned else arr

    def stage(self, packed):
        packed = np.ascontiguousarray(packed, dtype=np.uint64)
        _check(lib().pob_stage_inputs(self._h, packed.ctypes.data, packed.shape[0]))

    # ---- run ----
    def _inputs_ptr(self, packed, n, staged):
        if staged:
            assert n is not None
            return None, n, None
        packed = np.ascontiguousarray(packed, dtype=np.uint64)
        return packed.ctypes.data, (packed.shape[0] if n is None else n), packed

    def run_packed(self, packed, n=None, expand=True, digest=False, staged=False, discard=False, retain=None):
        """One synchronous batch (pob_run_batch / pob_run_batch_retain).  With expand and n > n_slots the library wants
        to know what happens to the witnesses: digest=True (each one is consumed by the on-GPU digest), discard=True
        (generation-only measurement), retain=[indices] (only those are materialised) -- or use submit()/acquire()."""
        ptr, n, keep = self._inputs_ptr(packed, n, staged)
        flags = (RUN_EXPAND if expand else 0) | (RUN_DIGEST if digest else 0) | (RUN_INPUTS_STAGED if staged else 0) | (RUN_DISCARD if discard else 0)
        status = np.zeros(n, dtype=np.uint32)
        outputs = np.zeros((n, max(1, self.n_outputs), 4), dtype=np.uint64)
        digests = np.zeros(n, dtype=np.uint64)
        if retain is None:
            _check(lib().pob_run_batch(self._h, ptr, n, flags, status.ctypes.data, outputs.ctypes.data, digests.ctypes.data if digest else None))
        else:
            r = np.ascontiguousarray(retain, dtype=np.uint32)
            _check(lib().pob_run_batch_retain(self._h, ptr, n, flags, r.ctypes.data if len(r) else None, len(r), status.ctypes.data, outputs.ctypes.data,
                                              digests.ctypes.data if digest else None))
        return BatchResult(status, outputs[:, : self.n_outputs], digests if digest else None, self.last_timing())

    def run(self, inputs, expand=True, digest=False, discard=False, retain=None):
        return self.run_packed(self.pack(inputs), expand=expand, digest=digest, discard=discard, retain=retain)

    def last_timing(self):
        t = Timing()
        _check(lib().pob_last_timing(self._h, ctypes.byref(t)))
        return t.as_dict()

    # ---- consumer-paced hand-off (pob_submit / pob_acquire / pob_release / pob_finish) ----
    def submit(self, packed, n=None, staged=False, digest=False):
        ptr, n, keep = self._inputs_ptr(packed, n, staged)
        self._inflight = (keep, n, digest)                   # the input buffer must outlive the batch
        _check(lib().pob_submit(self._h, ptr, n, (RUN_DIGEST if digest else 0) | (RUN_INPUTS_STAGED if staged else 0)))

    def acquire(self, stream=None):
        """next witness of the submitted batch: (index, device pointer) ; (index, None) for a rejected instance ;
        None when the batch is exhausted.  Raises PobError(E_BUSY) when every slot is held."""
        idx, dptr = ctypes.c_uint32(0), ctypes.c_void_p()
        rc = lib().pob_acquire(self._h, ctypes.byref(idx), ctypes.byref(dptr), stream)
        if rc == DONE:
            return None
        if rc == E_REJECTED:
            return int(idx.value), None
        _check(rc)
        return int(idx.value), dptr.value

    def release(self, index, stream=None):
        _check(lib().pob_release(self._h, index, stream))

    def finish(self):
        keep, n, digest = self._inflight
        status = np.zeros(n, dtype=np.uint32)
        outputs = np.zeros((n, max(1, self.n_outputs), 4), dtype=np.uint64)
        digests = np.zeros(n, dtype=np.uint64)
        _check(lib().pob_finish(self._h, status.ctypes.data, outputs.ctypes.data, digests.ctypes.data if digest else None))
        self._inflight = None
        return BatchResult(status, outputs[:, : self.n_outputs], digests if digest else None, self.last_timing())

    def export_batch(self, packed, paths=None, n=None, staged=False):
        """== n runs of `./<circuit> input_i.json paths[i]` (reference Makefile:5-6): every accepted instance is exported
        while later ones are generated; paths=None (or a None entry) moves the .wtns image to host memory only.
        Returns (BatchResult, export stats)."""
        ptr, n, keep = self._inputs_ptr(packed, n, staged)
        arr = None
        if paths is not None:
            assert len(paths) == n
            arr = (ctypes.c_char_p * n)(*[None if q is None else os.fsencode(q) for q in paths])
        status = np.zeros(n, dtype=np.uint32)
        outputs = np.zeros((n, max(1, self.n_outputs), 4), dtype=np.uint64)
        st = ExportStats()
        _check(lib().pob_export_batch(self._h, ptr, n, RUN_INPUTS_STAGED if staged else 0, arr, status.ctypes.data, outputs.ctypes.data, ctypes.byref(st)))
        return BatchResult(status, outputs[:, : self.n_outputs], None, self.last_timing()), st.as_dict()

    # ---- witness access ----
    def witness(self, index, first=0, count=None):
        count = self.n_signals - first if count is None else count
        out = np.zeros((count, 4), dtype=np.uint64)
        _check(lib().pob_copy_witness(self._h, index, first, count, out.ctypes.data))
        return out

    def write_wtns(self, index, path):
        _check(lib().pob_write_wtns(self._h, index, os.fsencode(path)))

    def selfcheck_keccak(self, index):
        """on-GPU check that every KeccakfRound block of resident witness `index` satisfies out == KeccakRound(in);
        returns (blocks examined, blocks failing)"""
        nb, bad = ctypes.c_uint64(0), ctypes.c_uint64(0)
        _check(lib().pob_selfcheck_keccak(self._h, index, ctypes.byref(nb), ctypes.byref(bad)))
        return int(nb.value), int(bad.value)

    def selfcheck(self, index):
        """on-GPU evaluation of EVERY constraint of the circuit (all `<==` / `===` of the circom sources) against resident
        witness `index`; returns the report dict (n_constraints, n_failed, n_hint_failed, first_failed, signals_read, ms)"""
        r = CheckReport()
        _check(lib().pob_selfcheck(self._h, index, ctypes.byref(r)))
        return r.as_dict()

    def r1cs_check(self, index):
        """on-GPU evaluation of every `.r1cs` row of this handle's form (--O0 or reduced) against resident witness `index`;
        report as selfcheck(), with first_failed a row index"""
        r = CheckReport()
        _check(lib().pob_r1cs_check(self._h, index, ctypes.byref(r)))
        return r.as_dict()

    def r1cs_products(self, index, first=0, count=None, stream=None, vectors="abc"):
        """A.w, B.w, C.w of `.r1cs` rows [first, first + count) of resident witness `index`, computed on the GPU: a tuple of torch
        uint64 CUDA tensors of shape (count, 4), the little-endian limbs of canonical field elements (None for a vector not in
        `vectors`).  stream: a torch.cuda.Stream (or a raw cudaStream_t) ordered after the witness (e.g. by acquire(stream)); the
        tensors are allocated and the work is enqueued on it without a host wait; None returns when done."""
        import torch
        if count is None:
            if getattr(self, "_r1cs_rows", None) is None:
                self._r1cs_rows = self.r1cs_check(index)["n_constraints"]
            count = self._r1cs_rows - first
        dev = torch.device("cuda", self.device)
        handle = None if stream is None else getattr(stream, "cuda_stream", stream)
        with torch.cuda.stream(torch.cuda.ExternalStream(handle, device=dev) if handle else torch.cuda.current_stream(dev)):
            out = [torch.empty((count, 4), dtype=torch.uint64, device=dev) if v in vectors else None for v in "abc"]
        ptr = [None if t is None else t.data_ptr() for t in out]
        _check(lib().pob_r1cs_products(self._h, index, first, count, ptr[0], ptr[1], ptr[2], handle))
        return tuple(out)

    def r1cs_domain(self):
        """log2 of the quotient's domain size n: the smallest power of two >= rows + public signals + 1 (pob_r1cs_domain)"""
        v = ctypes.c_uint32(0)
        _check(lib().pob_r1cs_domain(self._h, ctypes.byref(v)))
        return int(v.value)

    def r1cs_quotient(self, index, stream=None, out=None, work=None):
        """the Groth16 quotient evaluations of resident witness `index` on the GPU (pob_b200.h: pob_r1cs_quotient): a torch uint64
        CUDA tensor of shape (n, 4), q[i] = A^(g w^i) B^(g w^i) - C^(g w^i) as the limbs of canonical field elements.  out (n x 32 B)
        and work (2 n x 32 B of scratch) are allocated on `stream` unless given; stream as in r1cs_products."""
        import torch
        n = 1 << self.r1cs_domain()
        dev = torch.device("cuda", self.device)
        handle = None if stream is None else getattr(stream, "cuda_stream", stream)
        with torch.cuda.stream(torch.cuda.ExternalStream(handle, device=dev) if handle else torch.cuda.current_stream(dev)):
            if out is None:
                out = torch.empty((n, 4), dtype=torch.uint64, device=dev)
            if work is None:
                work = torch.empty((2 * n, 4), dtype=torch.uint64, device=dev)
        for t, need, what in ((out, 32 * n, "out"), (work, 64 * n, "work")):
            if not t.is_cuda or t.device != dev or not t.is_contiguous() or t.numel() * t.element_size() < need:
                raise ValueError("r1cs_quotient: %s must be a contiguous tensor on %s of at least %d bytes" % (what, dev, need))
        _check(lib().pob_r1cs_quotient(self._h, index, out.data_ptr(), work.data_ptr(), handle))
        return out

    def groth16_work_bytes(self):
        """bytes of scratch groth16_prove needs on this circuit (pob_groth16_work_bytes)"""
        v = ctypes.c_uint64(0)
        _check(lib().pob_groth16_work_bytes(self._h, ctypes.byref(v)))
        return int(v.value)

    def groth16_prove(self, index, key, r=None, s=None, stream=None, out=None, work=None):
        """a Groth16 proof of resident witness `index` on the GPU (pob_b200.h: pob_groth16_prove) with a Groth16Key.  r and s are the
        blinding scalars; each defaults to secrets.randbelow(R_ORDER), as zero knowledge needs.  Returns a Proof of ints; with a stream
        (torch.cuda.Stream or raw cudaStream_t) the work and any out / work tensor it allocates are enqueued on it, and the (32,) uint64
        out tensor (A: 8 limbs, B: 16, C: 8, canonical) is returned unsynchronised."""
        import secrets
        import torch
        r = secrets.randbelow(R_ORDER) if r is None else int(r)
        s = secrets.randbelow(R_ORDER) if s is None else int(s)
        dev = torch.device("cuda", self.device)
        handle = None if stream is None else getattr(stream, "cuda_stream", stream)
        need = self.groth16_work_bytes()
        with torch.cuda.stream(torch.cuda.ExternalStream(handle, device=dev) if handle else torch.cuda.current_stream(dev)):
            if out is None:
                out = torch.empty(32, dtype=torch.uint64, device=dev)
            if work is None:
                work = torch.empty(need, dtype=torch.uint8, device=dev)
        for t, what in [(out, "out"), (work, "work")] + [(v, "key." + f) for f, v in zip(key._fields, key)]:
            if not t.is_cuda or t.device != dev or not t.is_contiguous():
                raise ValueError("groth16_prove: %s must be a contiguous tensor on %s" % (what, dev))
        if out.numel() * out.element_size() < 256:
            raise ValueError("groth16_prove: out must hold 256 bytes")
        kc = Groth16KeyC(self.n_signals, self.n_outputs, self.r1cs_domain(), *[v.data_ptr() for v in key])
        rl, sl = to_limbs([r % (1 << 256)]), to_limbs([s % (1 << 256)])
        _check(lib().pob_groth16_prove(self._h, index, ctypes.byref(kc), rl.ctypes.data, sl.ctypes.data, out.data_ptr(), work.data_ptr(),
                                       work.numel() * work.element_size(), handle))
        if handle:
            return out
        return proof_from_limbs(out.cpu().tolist())

    def load_zkey(self, path, seed=None, staging_bytes=0):
        """the Groth16Key of a snarkjs `.zkey` (pob_zkey_load): the key tensors are allocated on this circuit's device and filled from
        the file, which is checked against the circuit on the GPU on the way.  seed: of the coefficient check's random combination,
        secrets.randbits(64) by default.  staging_bytes: pinned staging ring (0 = the library's default).  Returns (Groth16Key, report
        dict); a key that does not fit raises ZkeyError with .report."""
        import secrets
        import torch
        info = zkey_info(path)
        seed = secrets.randbits(64) if seed is None else int(seed)
        dev = torch.device("cuda", self.device)
        n1 = lambda b, w: torch.empty((max(1, b // (8 * w)), w), dtype=torch.uint64, device=dev)    # a section of no points: one unused row
        key = Groth16Key(alpha1=n1(64, 8), beta1=n1(64, 8), delta1=n1(64, 8), beta2=n1(128, 16), delta2=n1(128, 16), a=n1(info["a_bytes"], 8),
                         b1=n1(info["b1_bytes"], 8), b2=n1(info["b2_bytes"], 16), c=n1(info["c_bytes"], 8), h=n1(info["h_bytes"], 8))
        torch.cuda.synchronize(dev)
        kc = Groth16KeyC(self.n_signals, self.n_outputs, self.r1cs_domain(), *[v.data_ptr() for v in key])
        rep = ZkeyReport()
        rc = lib().pob_zkey_load(self._h, os.fsencode(path), seed & ((1 << 64) - 1), int(staging_bytes), ctypes.byref(kc), ctypes.byref(rep))
        if rc == E_KEY:
            checked = rep.points_checked > 0
            raise ZkeyError(rc, lib().pob_last_error().decode(), rep.as_dict() if checked else None)
        _check(rc)
        return key, rep.as_dict()

    def witness_map(self):
        m = np.zeros(self.n_signals, dtype=np.uint32)
        _check(lib().pob_witness_map(self._h, m.ctypes.data))
        return m

    def witness_device_ptr(self, index):
        p = ctypes.c_void_p()
        _check(lib().pob_witness_device_ptr(self._h, index, ctypes.byref(p)))
        return p.value


def pow_grind(start_key, reveal_amount, burn_extra_commitment, zero_bytes=2, max_tries=1 << 32, device=0):
    """GPU replacement of the reference's find_burn_key (tests/main.py:47-56): first burnKey >= start_key whose
    keccak(burnKey | revealAmount | burnExtraCommitment | "EIP-7503") starts with `zero_bytes` zero bytes.
    Returns (burn_key, tries)."""
    a, b, c = (to_limbs([v]) for v in (start_key, reveal_amount, burn_extra_commitment))
    out = np.zeros((1, 4), dtype=np.uint64)
    tries = ctypes.c_uint64(0)
    _check(lib().pob_pow_grind(int(device), a.ctypes.data, b.ctypes.data, c.ctypes.data, int(zero_bytes), int(max_tries), out.ctypes.data, ctypes.byref(tries)))
    return from_limbs(out[0]), int(tries.value)


def msm_g1_work_bytes(n):
    """bytes of scratch pob_msm_g1 needs for n points (host only, no GPU); at most 64 n for n >= 2^18"""
    v = ctypes.c_uint64(0)
    _check(lib().pob_msm_g1_work_bytes(int(n), ctypes.byref(v)))
    return int(v.value)


def msm_g1(bases, scalars, stream=None, out=None, work=None, device=None):
    """sum_i [s_i] P_i over BN254 G1 on the GPU (pob_b200.h: pob_msm_g1).  bases: (n, 8) uint64 CUDA tensor, per point x then y as
    Montgomery-form F_q limbs, (0, 0) = infinity.  scalars: (n, 4) uint64 CUDA tensor of 256-bit LE integers, or (device pointer, n)
    for memory the caller owns, such as a resident witness (Circuit.acquire / witness_device_ptr).  Returns (x, y) as canonical
    ints, or None for infinity.  With a stream (torch.cuda.Stream or raw cudaStream_t) the work and any out / work tensor it has
    to allocate are enqueued on it, and the (8,) uint64 out tensor (x limbs, then y limbs) is returned unsynchronised."""
    import torch
    if isinstance(scalars, tuple):
        s_ptr, n = int(scalars[0]), int(scalars[1])
    else:
        if scalars.dim() != 2 or scalars.shape[1] != 4 or scalars.dtype not in (torch.uint64, torch.int64) or not scalars.is_contiguous():
            raise ValueError("msm_g1: scalars must be a contiguous (n, 4) uint64 tensor")
        s_ptr, n = scalars.data_ptr(), scalars.shape[0]
    if bases.dim() != 2 or bases.shape[1] != 8 or bases.shape[0] != n or bases.dtype not in (torch.uint64, torch.int64) or not bases.is_contiguous():
        raise ValueError("msm_g1: bases must be a contiguous (n, 8) uint64 tensor with n = %d" % n)
    dev = bases.device if device is None else torch.device("cuda", device)
    handle = None if stream is None else getattr(stream, "cuda_stream", stream)
    with torch.cuda.stream(torch.cuda.ExternalStream(handle, device=dev) if handle else torch.cuda.current_stream(dev)):
        if out is None:
            out = torch.empty(8, dtype=torch.uint64, device=dev)
        if work is None:
            work = torch.empty(msm_g1_work_bytes(n), dtype=torch.uint8, device=dev)
    for t, what in ((bases, "bases"), (out, "out"), (work, "work")):
        if not t.is_cuda or t.device != dev or not t.is_contiguous():
            raise ValueError("msm_g1: %s must be a contiguous tensor on %s" % (what, dev))
    _check(lib().pob_msm_g1(dev.index, bases.data_ptr(), s_ptr, n, out.data_ptr(), work.data_ptr(),
                            work.numel() * work.element_size(), handle))
    if handle:
        return out
    v = [int(x) & ((1 << 64) - 1) for x in out.cpu().tolist()]
    x, y = (sum(v[4 * k + i] << (64 * i) for i in range(4)) for k in (0, 1))
    return None if x == 0 and y == 0 else (x, y)


def _point(limbs, coords):
    v = [int(x) & ((1 << 64) - 1) for x in limbs]
    c = [sum(v[4 * k + i] << (64 * i) for i in range(4)) for k in range(coords)]
    return c if any(c) else None


def proof_from_limbs(limbs):
    """Proof of ints from the 32 uint64 limbs pob_groth16_prove writes"""
    a, b, c = _point(limbs[0:8], 2), _point(limbs[8:24], 4), _point(limbs[24:32], 2)
    return Proof(None if a is None else tuple(a), None if b is None else ((b[0], b[1]), (b[2], b[3])), None if c is None else tuple(c))


def msm_g2_work_bytes(n):
    """bytes of scratch pob_msm_g2 needs for n points (host only, no GPU)"""
    v = ctypes.c_uint64(0)
    _check(lib().pob_msm_g2_work_bytes(int(n), ctypes.byref(v)))
    return int(v.value)


def msm_g2(bases, scalars, stream=None, out=None, work=None, device=None):
    """sum_i [s_i] P_i over BN254 G2 on the GPU (pob_b200.h: pob_msm_g2).  bases: (n, 16) uint64 CUDA tensor, per point x.c0, x.c1,
    y.c0, y.c1 as Montgomery-form F_q limbs, all-zero = infinity; points of the order-r subgroup (not checked).  scalars as msm_g1.
    Returns ((x0, x1), (y0, y1)) as canonical ints, or None for infinity; with a stream the (16,) uint64 out tensor, unsynchronised."""
    import torch
    if isinstance(scalars, tuple):
        s_ptr, n = int(scalars[0]), int(scalars[1])
    else:
        if scalars.dim() != 2 or scalars.shape[1] != 4 or scalars.dtype not in (torch.uint64, torch.int64) or not scalars.is_contiguous():
            raise ValueError("msm_g2: scalars must be a contiguous (n, 4) uint64 tensor")
        s_ptr, n = scalars.data_ptr(), scalars.shape[0]
    if bases.dim() != 2 or bases.shape[1] != 16 or bases.shape[0] != n or bases.dtype not in (torch.uint64, torch.int64) or not bases.is_contiguous():
        raise ValueError("msm_g2: bases must be a contiguous (n, 16) uint64 tensor with n = %d" % n)
    dev = bases.device if device is None else torch.device("cuda", device)
    handle = None if stream is None else getattr(stream, "cuda_stream", stream)
    with torch.cuda.stream(torch.cuda.ExternalStream(handle, device=dev) if handle else torch.cuda.current_stream(dev)):
        if out is None:
            out = torch.empty(16, dtype=torch.uint64, device=dev)
        if work is None:
            work = torch.empty(msm_g2_work_bytes(n), dtype=torch.uint8, device=dev)
    for t, what in ((bases, "bases"), (out, "out"), (work, "work")):
        if not t.is_cuda or t.device != dev or not t.is_contiguous():
            raise ValueError("msm_g2: %s must be a contiguous tensor on %s" % (what, dev))
    _check(lib().pob_msm_g2(dev.index, bases.data_ptr(), s_ptr, n, out.data_ptr(), work.data_ptr(),
                            work.numel() * work.element_size(), handle))
    if handle:
        return out
    c = _point(out.cpu().tolist(), 4)
    return None if c is None else ((c[0], c[1]), (c[2], c[3]))


# ---- verification (pob_bn254_pairing, pob_groth16_verify) -----------------------------------------------------------------------
_RM = 1 << 256


def _fq_bytes(v, mont):
    """32 LE bytes of an F_q coordinate: its Montgomery form (v must be canonical, 0 <= v < q: a key's point is never reduced), or
    v itself unchanged (a proof's coordinate, which the device range-checks)"""
    v = int(v)
    if mont and not 0 <= v < Q:
        raise ValueError("a key coordinate must lie in [0, q): %d" % v)
    return (v * _RM % Q if mont else v).to_bytes(32, "little")


def _enc_g1(p, mont):
    return bytes(64) if p is None else _fq_bytes(p[0], mont) + _fq_bytes(p[1], mont)


def _enc_g2(p, mont):
    return bytes(128) if p is None else b"".join(_fq_bytes(v, mont) for v in (p[0][0], p[0][1], p[1][0], p[1][1]))


def _u64(raw, width):
    return np.frombuffer(raw, dtype=np.uint64).reshape(-1, width).copy()


def _to_dev(arr, dev):
    """a uint64 numpy array as a uint64 CUDA tensor, copied on the current stream from a pinned staging buffer (no host wait; the
    caching host allocator keeps the buffer until the copy is done)"""
    import torch
    return torch.from_numpy(arr.view(np.int64)).pin_memory().to(dev, non_blocking=True).view(torch.uint64)


def _dec_fq(raw, mont):
    v = int.from_bytes(raw, "little")
    return v * pow(_RM, -1, Q) % Q if mont else v


def _dec_g1(raw, mont):
    return None if not any(raw) else (_dec_fq(raw[:32], mont), _dec_fq(raw[32:64], mont))


def _dec_g2(raw, mont):
    if not any(raw):
        return None
    c = [_dec_fq(raw[32 * k:32 * k + 32], mont) for k in range(4)]
    return ((c[0], c[1]), (c[2], c[3]))


def _stream_ctx(dev, handle):
    import torch
    return torch.cuda.stream(torch.cuda.ExternalStream(handle, device=dev) if handle else torch.cuda.current_stream(dev))


def pairing(g1_points, g2_points, device=0):
    """[e(P_i, Q_i)] on the GPU (pob_bn254_pairing): P_i G1 points (x, y), Q_i G2 points ((x0, x1), (y0, y1)), canonical ints, None =
    infinity; not checked to lie in G1 / G2.  Each value is a 12-tuple of ints in vk_alphabeta_12's nesting (c0.c0.c0, c0.c0.c1, ..)."""
    import torch
    n = len(g1_points)
    if n == 0 or len(g2_points) != n:
        raise ValueError("pairing: need equally many (>= 1) G1 and G2 points")
    dev = torch.device("cuda", device)
    a = _to_dev(_u64(b"".join(_enc_g1(p, True) for p in g1_points), 8), dev)
    b = _to_dev(_u64(b"".join(_enc_g2(p, True) for p in g2_points), 16), dev)
    out = torch.empty((n, 48), dtype=torch.uint64, device=dev)
    torch.cuda.synchronize(dev)
    _check(lib().pob_bn254_pairing(dev.index, a.data_ptr(), b.data_ptr(), n, out.data_ptr(), None))
    raw = out.view(torch.int64).cpu().numpy().tobytes()
    return [tuple(int.from_bytes(raw[384 * i + 32 * k:384 * i + 32 * k + 32], "little") for k in range(12)) for i in range(n)]


class DeviceVerificationKey(collections.namedtuple("DeviceVerificationKey", "n_pub alpha1 beta2 gamma2 delta2 ic")):
    """A verification key as CUDA tensors (pob_b200.h: pob_groth16_vk): alpha1 (1, 8), beta2, gamma2, delta2 (1, 16) and ic
    (n_pub + 1, 8) uint64, affine Montgomery form as in a .zkey."""


class VerificationKey(collections.namedtuple("VerificationKey", "alpha1 beta2 gamma2 delta2 ic")):
    """A Groth16 verification key of ints: alpha1 and the IC points (a list of n_pub + 1) are G1 points (x, y), beta2, gamma2 and
    delta2 G2 points ((x0, x1), (y0, y1)); None = infinity."""

    @property
    def n_pub(self):
        return len(self.ic) - 1

    @classmethod
    def from_zkey(cls, path):
        """sections 2 and 3 of a snarkjs `.zkey` (pob_zkey_vk; host only, no GPU).  A malformed file raises ZkeyError or PobError."""
        n_pub = ctypes.c_uint32(0)
        rc = lib().pob_zkey_vk(os.fsencode(path), ctypes.create_string_buffer(1), 1, ctypes.byref(n_pub))   # short: sizes the key
        if rc == E_KEY:
            raise ZkeyError(rc, lib().pob_last_error().decode())
        if rc != -1:
            _check(rc)
        buf = ctypes.create_string_buffer(448 + 64 * (n_pub.value + 1))
        rc = lib().pob_zkey_vk(os.fsencode(path), buf, len(buf), ctypes.byref(n_pub))
        if rc == E_KEY:
            raise ZkeyError(rc, lib().pob_last_error().decode())
        _check(rc)
        raw = buf.raw
        ic = [_dec_g1(raw[448 + 64 * k:512 + 64 * k], True) for k in range(n_pub.value + 1)]
        return cls(_dec_g1(raw[:64], True), _dec_g2(raw[64:192], True), _dec_g2(raw[192:320], True), _dec_g2(raw[320:448], True), ic)

    @classmethod
    def from_json(cls, d):
        """from snarkjs's verification_key.json shape (to_json); vk_alphabeta_12 is ignored (verification recomputes it)"""
        if d.get("protocol", "groth16") != "groth16" or d.get("curve", "bn128") != "bn128":
            raise ValueError("not a Groth16 BN254 verification key")
        ic = [_g1_from_json(p) for p in d["IC"]]
        if "nPublic" in d and int(d["nPublic"]) != len(ic) - 1:
            raise ValueError("nPublic is %s but IC has %d points" % (d["nPublic"], len(ic)))
        vk = cls(_g1_from_json(d["vk_alpha_1"]), _g2_from_json(d["vk_beta_2"]), _g2_from_json(d["vk_gamma_2"]),
                 _g2_from_json(d["vk_delta_2"]), ic)
        for p in [vk.alpha1] + list(vk.ic):
            if p is not None and not all(0 <= v < Q for v in p):
                raise ValueError("a G1 coordinate of the key is not in [0, q): %r" % (p,))
        for p in (vk.beta2, vk.gamma2, vk.delta2):
            if p is not None and not all(0 <= v < Q for c in p for v in c):
                raise ValueError("a G2 coordinate of the key is not in [0, q): %r" % (p,))
        return vk

    def to_json(self, device=0):
        """snarkjs's verification_key.json dictionary, as far as its shape is known here; vk_alphabeta_12 = e(alpha1, beta2) from
        pob_bn254_pairing, nested [[[c000, c001], [c010, c011], [c020, c021]], [[c100, ..], ..]]"""
        e = pairing([self.alpha1], [self.beta2], device=device)[0]
        ab = [[[str(e[6 * h + 2 * j]), str(e[6 * h + 2 * j + 1])] for j in range(3)] for h in range(2)]
        return {"protocol": "groth16", "curve": "bn128", "nPublic": self.n_pub, "vk_alpha_1": _g1_json(self.alpha1),
                "vk_beta_2": _g2_json(self.beta2), "vk_gamma_2": _g2_json(self.gamma2), "vk_delta_2": _g2_json(self.delta2),
                "vk_alphabeta_12": ab, "IC": [_g1_json(p) for p in self.ic]}

    def to_device(self, device=0):
        """the DeviceVerificationKey of this key on cuda:device"""
        import torch
        dev = torch.device("cuda", device)
        raw = [(_enc_g1(self.alpha1, True), 8), (_enc_g2(self.beta2, True), 16), (_enc_g2(self.gamma2, True), 16),
               (_enc_g2(self.delta2, True), 16), (b"".join(_enc_g1(p, True) for p in self.ic), 8)]      # every coordinate checked first
        return DeviceVerificationKey(self.n_pub, *[_to_dev(_u64(r, w), dev) for r, w in raw])


def groth16_verify_work_bytes(n_pub, n):
    """bytes of scratch pob_groth16_verify needs (host only, no GPU)"""
    v = ctypes.c_uint64(0)
    _check(lib().pob_groth16_verify_work_bytes(int(n_pub), int(n), ctypes.byref(v)))
    return int(v.value)


def groth16_verify(vk, proofs, publics, device=0, stream=None, status=None, work=None):
    """Groth16 verdicts on the GPU (pob_groth16_verify), one per proof: 0 valid, else a VERIFY_STATUS code.
    vk: VerificationKey or DeviceVerificationKey.  proofs: a list of Proof, or a CUDA uint64 tensor of (32,) or (n, 32) limbs as
    Circuit.groth16_prove's out.  publics: a list of n lists of n_pub ints (values >= r are passed through unreduced and refused), or
    a CUDA uint64 tensor of n x n_pub x 4 limbs.  status: an optional CUDA int32 / uint32 tensor of >= n elements; work: an optional
    CUDA tensor of >= groth16_verify_work_bytes bytes.  Returns a numpy uint32 array; with a stream (torch.cuda.Stream or raw
    cudaStream_t) everything, the key's and the host inputs' transfers included (through pinned staging buffers), is enqueued on it
    with no host wait, and the (n,) status tensor is returned unsynchronised."""
    import torch
    handle = None if stream is None else getattr(stream, "cuda_stream", stream)
    if isinstance(proofs, torch.Tensor):
        dev = proofs.device
        if not proofs.is_cuda or not proofs.is_contiguous() or proofs.numel() % 32 or proofs.element_size() != 8:
            raise ValueError("groth16_verify: proofs must be a contiguous CUDA uint64 tensor of n x 32 limbs")
        n = proofs.numel() // 32
    else:
        dev = torch.device("cuda", device)
        n = len(proofs)
    if n == 0:
        raise ValueError("groth16_verify: no proofs")
    n_pub = vk.n_pub
    with _stream_ctx(dev, handle):                  # every temporary is allocated on the stream that uses it
        if isinstance(vk, VerificationKey):
            vk = vk.to_device(dev.index)
        if not isinstance(proofs, torch.Tensor):
            raw = b"".join(_enc_g1(p.a, False) + _enc_g2(p.b, False) + _enc_g1(p.c, False) for p in proofs)
            proofs = _to_dev(_u64(raw, 32), dev)
        pub_t = None
        if isinstance(publics, torch.Tensor):
            if publics.device != dev or not publics.is_contiguous() or publics.numel() != 4 * n_pub * n or publics.element_size() != 8:
                raise ValueError("groth16_verify: publics must be a contiguous CUDA uint64 tensor of n x n_pub x 4 limbs")
            pub_t = publics
        elif n_pub:
            if len(publics) != n or any(len(v) != n_pub for v in publics):
                raise ValueError("groth16_verify: need n_pub = %d public inputs for each of %d proofs" % (n_pub, n))
            if any(not 0 <= int(x) < 1 << 256 for v in publics for x in v):
                raise ValueError("groth16_verify: a public input must be a 256-bit unsigned integer")
            pub_t = _to_dev(_u64(b"".join(int(x).to_bytes(32, "little") for v in publics for x in v), 4), dev)
        if status is None:
            status = torch.empty(n, dtype=torch.int32, device=dev)
        if work is None:
            work = torch.empty(groth16_verify_work_bytes(n_pub, n), dtype=torch.uint8, device=dev)
    key_bytes = {"alpha1": 64, "beta2": 128, "gamma2": 128, "delta2": 128, "ic": 64 * (n_pub + 1)}
    for t, what, need in [(status, "status", 4 * n), (work, "work", groth16_verify_work_bytes(n_pub, n))] + \
            [(getattr(vk, f), "vk." + f, b) for f, b in key_bytes.items()]:
        if not isinstance(t, torch.Tensor) or t.device != dev or not t.is_contiguous() or t.numel() * t.element_size() < need:
            raise ValueError("groth16_verify: %s must be a contiguous tensor on %s of at least %d bytes" % (what, dev, need))
    if status.element_size() != 4:
        raise ValueError("groth16_verify: status must hold 32-bit elements")
    kc = Groth16VkC(n_pub, *[t.data_ptr() for t in (vk.alpha1, vk.beta2, vk.gamma2, vk.delta2, vk.ic)])
    if handle is None:
        torch.cuda.synchronize(dev)
    _check(lib().pob_groth16_verify(dev.index, ctypes.byref(kc), proofs.data_ptr(), None if pub_t is None else pub_t.data_ptr(), n,
                                    status.data_ptr(), work.data_ptr(), work.numel() * work.element_size(), handle))
    if handle:
        return status
    return status[:n].cpu().numpy().astype(np.uint32)


def repad_pob_input(inp, max_layers, node_blocks, header_blocks):
    """Re-pad a ProofOfBurn input JSON to a circuit shape: unused layers are zero with length 256 (the convention of
    reference tests/main.py:148-150), the header is zero-extended.  The reference generator still pads to the (4,.,5)
    test shape (tests/main.py:8-11) although main_proof_of_burn.circom:27 needs (16,4,16)."""
    out = dict(inp)
    nb, hb = node_blocks * 136, header_blocks * 136
    layers = [list(l)[:nb] + [0] * (nb - len(l)) for l in inp["layers"]]
    lens = list(inp["layerLens"])
    while len(layers) < max_layers:
        layers.append([0] * nb)
        lens.append(256)
    out["layers"], out["layerLens"] = layers[:max_layers], lens[:max_layers]
    hdr = list(inp["blockHeader"])
    out["blockHeader"] = hdr[:hb] + [0] * (hb - len(hdr))
    return out


CIRCUIT_ALIASES = {"main_proof_of_burn": MAIN_PROOF_OF_BURN, "main_spend": MAIN_SPEND}


def main(argv=None):
    """CLI shim with the reference calculator's argv: `python -m pob_b200 <circuit> input.json witness.wtns`
    (reference Makefile:5-6); <circuit> is main_proof_of_burn, main_spend or a `Template(params)` expression.
    Batch form: `python -m pob_b200 <circuit> --batch in1.json in2.json ... --out DIR` evaluates all inputs in one
    pob_run_batch and writes DIR/<name>.wtns for every accepted instance.
    R1CS form: `python -m pob_b200 <circuit> --r1cs out.r1cs [--O1]` writes the circuit's `.r1cs` (host only, no GPU) in the wire
    order of the --O0 witness, or of the reduced one with --O1.
    Key check: `python -m pob_b200 <circuit> --check-zkey key.zkey [--O1]` loads a snarkjs `.zkey` and checks it against the circuit on
    the GPU (Circuit.load_zkey); prints the report, exit code 1 when the key does not fit.
    Proof: `python -m pob_b200 <circuit> --prove key.zkey input.json proof.json public.json [--O1]` generates the witness, loads and
    checks the key, proves on the GPU and writes snarkjs-shaped proof.json and public.json; a rejected input or a key that does not
    fit exits 1 and writes no proof.
    Verification key: `python -m pob_b200 --export-vk key.zkey verification_key.json` writes snarkjs's verification_key.json shape
    from the .zkey (vk_alphabeta_12 computed on the GPU).
    Verification: `python -m pob_b200 --verify verification_key.json public.json proof.json [public2.json proof2.json ...]` (snarkjs's
    argument order) verifies every pair in one GPU call, prints one line per pair (OK or the status's name) and exits 0 only when
    every proof is valid, else 1."""
    import sys
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) == 3 and argv[0] == "--export-vk":
        vk = VerificationKey.from_zkey(argv[1])
        with open(argv[2], "w") as f:
            json.dump(vk.to_json(), f, indent=1)
        return 0
    if len(argv) >= 4 and len(argv) % 2 == 0 and argv[0] == "--verify":
        with open(argv[1]) as f:
            try:
                vk = VerificationKey.from_json(json.load(f))
            except ValueError as e:
                print("%s: %s" % (argv[1], e), file=sys.stderr)
                return 1
        pairs = [(argv[k], argv[k + 1]) for k in range(2, len(argv), 2)]
        publics, proofs = [], []
        for pub_path, proof_path in pairs:
            with open(pub_path) as f:
                publics.append([int(v) for v in json.load(f)])
            with open(proof_path) as f:
                proofs.append(Proof.from_json(json.load(f)))
        if any(len(p) != vk.n_pub for p in publics):
            print("a public.json does not hold nPublic = %d values" % vk.n_pub, file=sys.stderr)
            return 1
        status = groth16_verify(vk, proofs, publics)
        for (pub_path, proof_path), s in zip(pairs, status):
            print("%s %s: %s" % (pub_path, proof_path, VERIFY_STATUS[int(s)]))
        return 0 if all(int(s) == 0 for s in status) else 1
    if len(argv) in (3, 4) and argv[1] == "--check-zkey" and argv[3:] in ([], ["--O1"]):
        c = Circuit(CIRCUIT_ALIASES.get(argv[0], argv[0]), max_slots=1, opt=1 if argv[3:] else 0)
        try:
            _, rep = c.load_zkey(argv[2])
            print(json.dumps(dict(rep, ok=True)))
            return 0
        except ZkeyError as e:
            print(json.dumps(dict(e.report or {}, ok=False)))
            print(str(e), file=sys.stderr)
            return 1
        finally:
            c.close()
    if len(argv) in (6, 7) and argv[1] == "--prove" and argv[6:] in ([], ["--O1"]):
        key_path, input_path, proof_path, public_path = argv[2:6]
        c = Circuit(CIRCUIT_ALIASES.get(argv[0], argv[0]), max_slots=1, opt=1 if argv[6:] else 0)
        try:
            res = c.run([json.load(open(input_path))])
            if res.status[0] != 0:
                print("Error: constraint failed in the component at witness index %d" % (int(res.status[0]) - 1), file=sys.stderr)
                return 1
            try:
                key, _ = c.load_zkey(key_path)
            except ZkeyError as e:
                print(str(e), file=sys.stderr)
                return 1
            proof = c.groth16_prove(0, key)
            with open(proof_path, "w") as f:
                json.dump(proof.to_json(), f)
            with open(public_path, "w") as f:
                json.dump(public_json(res.outputs[0]), f)
            return 0
        finally:
            c.close()
    if len(argv) in (3, 4) and argv[1] == "--r1cs" and argv[3:] in ([], ["--O1"]):
        d = write_r1cs(CIRCUIT_ALIASES.get(argv[0], argv[0]), argv[2], opt=1 if argv[3:] else 0)
        print("%s: %d wires, %d constraints (%d non-linear), %d bytes" % (argv[2], d["n_wires"], d["n_constraints"], d["n_nonlinear"], d["file_bytes"]))
        return 0
    if len(argv) >= 4 and argv[1] == "--batch" and "--out" in argv:
        k = argv.index("--out")
        files, outdir = argv[2:k], argv[k + 1]
        os.makedirs(outdir, exist_ok=True)
        c = Circuit(CIRCUIT_ALIASES.get(argv[0], argv[0]))
        paths = [os.path.join(outdir, os.path.splitext(os.path.basename(f))[0] + ".wtns") for f in files]
        res, _ = c.export_batch(c.pack([json.load(open(f)) for f in files]), paths)     # consumer-paced: any number of inputs
        rc = 0
        for i, f in enumerate(files):
            if res.status[i] != 0:
                print("%s: constraint failed in the component at witness index %d" % (f, int(res.status[i]) - 1), file=sys.stderr)
                rc = 1
        return rc
    if len(argv) != 3 or argv[0] in ("--export-vk", "--verify"):
        print("usage: python -m pob_b200 <main_proof_of_burn|main_spend|Template(params)> input.json witness.wtns\n"
              "       python -m pob_b200 <circuit> --batch in1.json in2.json ... --out DIR\n"
              "       python -m pob_b200 <circuit> --r1cs out.r1cs [--O1]\n"
              "       python -m pob_b200 <circuit> --check-zkey key.zkey [--O1]\n"
              "       python -m pob_b200 <circuit> --prove key.zkey input.json proof.json public.json [--O1]\n"
              "       python -m pob_b200 --export-vk key.zkey verification_key.json\n"
              "       python -m pob_b200 --verify verification_key.json public.json proof.json [public2.json proof2.json ...]", file=sys.stderr)
        return 2
    c = Circuit(CIRCUIT_ALIASES.get(argv[0], argv[0]), max_slots=1)
    res = c.run([json.load(open(argv[1]))])
    if res.status[0] != 0:
        print("Error: constraint failed in the component at witness index %d" % (int(res.status[0]) - 1), file=sys.stderr)
        return 1
    c.write_wtns(0, argv[2])
    return 0
