"""Witness slots are compressible memory (Compute Data Compression) wherever the device supports it: pob_desc reports how
many of the slots the driver made compressible, and a witness in such a slot is bit-exact."""
import ctypes

import pytest

from helpers import pob_fixture, repad_pob

pytestmark = pytest.mark.gpu

CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED = 107     # cuda.h


def device_supports_compression(device=0):
    """asked of the driver directly, independently of the library under test"""
    cu = ctypes.CDLL("libcuda.so.1")
    dev, v = ctypes.c_int(), ctypes.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(ctypes.byref(dev), device) == 0
    assert cu.cuDeviceGetAttribute(ctypes.byref(v), CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, dev) == 0
    return v.value != 0


def test_main_shape_witness_in_a_compressed_slot_is_the_oracles():
    import pob_b200
    from oracle import oracle
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=1)
    try:
        d = c.desc
        assert d["n_slots"] == 1 and d["n_compressed_slots"] <= d["n_slots"]
        if not device_supports_compression():
            return
        assert d["n_compressed_slots"] == 1, "the device supports compression but the driver granted none"
        inp = repad_pob(pob_fixture(), 16, 4, 16)
        res = c.run([inp], expand=True, digest=True)
        w = oracle.run(pob_b200.MAIN_PROOF_OF_BURN, inp)
        try:
            assert w.ok and res.status[0] == 0
            assert int(res.digests[0]) == w.digest(), "witness digest in a compressed slot differs from the oracle"
        finally:
            w.free()
    finally:
        c.close()
