"""The consumer-paced hand-off against slow on-GPU consumers: every witness distinct, every read checked against its own oracle
witness.

The consumer works on torch.cuda.Streams (non-blocking, like the library's own streams) and spins with torch.cuda._sleep before it
reads, so that a read the library does not order after the right expansion -- or an expansion not ordered after the consumer's
reads -- sees another instance's witness.  Each sleep is followed by an event; where the race window matters a test asserts that
the event has not completed yet, so a host step that outlasted the sleep fails the test instead of letting it pass vacuously.
A consumer read is a device-to-device copy of the whole slot on the consumer stream (or the `.r1cs` row products / the quotient
enqueued there).  Every test synchronises its streams before it closes the handle."""
import ctypes

import numpy as np
import pytest

import quotient_model as qm
from helpers import _cudart
from r1cs_reader import R1cs, witness_ints
from test_gpu_shapes import _spend_inputs

pytestmark = pytest.mark.gpu

SPEND = "Spend(31)"
SLEEP = 10 ** 9                     # torch.cuda._sleep cycles: about 0.5 s at the H100's clock
MAIN_SHAPE = (16, 4, 16, 50, 31, 2, 10 ** 19, 10 ** 20)
REJECTED = 3                        # the pool's one instance with withdrawnBalance > balance
OPTS = pytest.mark.parametrize("opt", [0, 1], ids=["O0", "O1"])

_POOL = []
_ORACLE = {}


def _pool():
    """16 distinct Spend(31) inputs; instance 3 is rejected, the others are accepted"""
    if not _POOL:
        _POOL.extend(_spend_inputs(16, seed=7503, rejected=(REJECTED,)))
    return _POOL


def _oracle(inp):
    from oracle import oracle
    key = tuple(sorted(inp.items()))
    if key not in _ORACLE:
        w = oracle.run(SPEND, inp)
        assert w.ok
        _ORACLE[key] = w
    return _ORACLE[key]


def _want(inp, m):
    """the oracle witness of `inp` in the handle's form (m = witness_map() of a reduced handle, None for --O0)"""
    w = _oracle(inp)
    return w.limbs if m is None else w.limbs[m]


@pytest.fixture(scope="module", autouse=True)
def _free_oracle_witnesses():
    yield
    for w in _ORACLE.values():
        w.free()
    _ORACLE.clear()


@pytest.fixture(autouse=True)
def _return_cached_device_memory():
    """the consumer buffers and quotients go back to the device, so later handles find the free memory they would without them"""
    yield
    import torch
    torch.cuda.empty_cache()


def _handle(opt, max_slots=2):
    import pob_b200
    c = pob_b200.Circuit(SPEND, max_slots=max_slots, opt=opt)
    return c, (c.witness_map() if opt else None)


def _buffers(c, n):
    import torch
    bufs = [torch.empty((c.n_signals, 4), dtype=torch.uint64, device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    return bufs


def _sleep(st, cycles=SLEEP):
    """spin on stream st; returns an event that completes when the spin is over"""
    import torch
    with torch.cuda.stream(st):
        torch.cuda._sleep(cycles)
    ev = torch.cuda.Event()
    ev.record(st)
    return ev


def _copy(st, dst, dptr):
    """the consumer's read: the whole slot at dptr into the torch buffer dst, enqueued on st"""
    nbytes = dst.numel() * dst.element_size()
    rc = _cudart().cudaMemcpyAsync(ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(dptr), ctypes.c_size_t(nbytes), ctypes.c_int(3),
                                   ctypes.c_void_p(st.cuda_stream))
    assert rc == 0, "cudaMemcpyAsync failed: %d" % rc


def _open(ev, what):
    assert not ev.query(), "the consumer's sleep ended before %s: the window under test was closed" % what


def _same(buf, want, what):
    got = buf.cpu().numpy()
    diff = np.nonzero((got != want).any(axis=1))[0]
    assert len(diff) == 0, "%s: %d entries differ from the oracle, first %d" % (what, len(diff), diff[0])


def _sync(*streams):
    for s in streams:
        s.synchronize()


@OPTS
@pytest.mark.parametrize("n_streams", [1, 2], ids=["one_stream", "two_streams"])
def test_slow_consumer_within_a_batch(opt, n_streams):
    """8 instances through 2 slots; each witness is read after a sleep and released on the consumer stream, so the expansion of
    the instance two places later must wait for the read.  With two streams that alternate and sleep 0.5 s and 0.1 s, releases
    complete out of order and a slot passes between the streams."""
    import torch
    inps = _pool()[:8]
    c, m = _handle(opt)
    streams = [torch.cuda.Stream() for _ in range(n_streams)]
    sleeps = [SLEEP, SLEEP // 5][:n_streams]
    try:
        bufs = _buffers(c, len(inps))
        c.submit(c.pack(inps))
        seen, taken = [], 0
        while True:
            st = streams[taken % n_streams]
            r = c.acquire(st.cuda_stream)
            if r is None:
                break
            idx, dptr = r
            seen.append(idx)
            if dptr is None:
                assert idx == REJECTED
                continue
            ev = _sleep(st, sleeps[taken % n_streams])
            _copy(st, bufs[idx], dptr)
            c.release(idx, st.cuda_stream)
            _open(ev, "the release of instance %d was queued" % idx)
            taken += 1
        fin = c.finish()
        assert seen == list(range(8)) and taken == 7
        assert [i for i in range(8) if fin.status[i] != 0] == [REJECTED]
        _sync(*streams)
        for i in range(8):
            if i != REJECTED:
                _same(bufs[i], _want(inps[i], m), "instance %d" % i)
    finally:
        _sync(*streams)
        c.close()


@OPTS
def test_consumer_stream_waits_for_the_witness(opt):
    """instance 2 reuses instance 0's slot, whose release on stream a is still behind a sleep: acquire(2) on stream b returns at
    once, and a copy enqueued on b right away must still see instance 2's witness, not instance 0's"""
    import torch
    inps = _pool()[8:12]
    c, m = _handle(opt)
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        bufs = _buffers(c, 2)
        c.submit(c.pack(inps))
        i0, p0 = c.acquire(a.cuda_stream)
        _copy(a, bufs[0], p0)
        ev = _sleep(a)
        c.release(i0, a.cuda_stream)
        i1, _ = c.acquire(b.cuda_stream)
        c.release(i1, b.cuda_stream)
        i2, p2 = c.acquire(b.cuda_stream)
        _copy(b, bufs[1], p2)
        _open(ev, "the copy of instance 2 was enqueued")
        assert (i0, i1, i2) == (0, 1, 2) and p2 == p0
        c.release(i2, b.cuda_stream)
        assert c.finish().n_ok == 4
        _sync(a, b)
        _same(bufs[0], _want(inps[0], m), "instance 0")
        _same(bufs[1], _want(inps[2], m), "instance 2")
    finally:
        _sync(a, b)
        c.close()


@OPTS
@pytest.mark.parametrize("via", ["run", "submit"])
def test_release_orders_the_next_batch(opt, via):
    """batch A's last two witnesses are read behind a sleep and released on the consumer stream; pob_finish returns, and batch B
    (n = n_slots, other inputs) starts on the same handle while the consumer still sleeps: B must not expand into the slots before
    the consumer's reads"""
    import torch
    A, B = _pool()[8:11], _pool()[11:13]
    c, m = _handle(opt)
    st = torch.cuda.Stream()
    try:
        bufs = _buffers(c, len(A))
        c.submit(c.pack(A))
        ev = None
        while True:
            r = c.acquire(st.cuda_stream)
            if r is None:
                break
            idx, dptr = r
            if idx == len(A) - 2:
                ev = _sleep(st)
            _copy(st, bufs[idx], dptr)
            c.release(idx, st.cuda_stream)
        assert c.finish().n_ok == len(A)
        packed = c.pack(B)
        _open(ev, "batch B started")
        if via == "run":
            assert (c.run_packed(packed).status == 0).all()
            for i in range(len(B)):
                assert np.array_equal(c.witness(i), _want(B[i], m)), "batch B instance %d" % i
        else:
            c.submit(packed)
            seen = []
            while True:
                r = c.acquire()
                if r is None:
                    break
                idx, dptr = r
                assert np.array_equal(c.witness(idx), _want(B[idx], m)), "batch B instance %d" % idx
                c.release(idx)
                seen.append(idx)
            assert seen == [0, 1] and c.finish().n_ok == len(B)
        st.synchronize()
        for i in range(len(A)):
            _same(bufs[i], _want(A[i], m), "batch A instance %d" % i)
    finally:
        _sync(st)
        c.close()


@OPTS
def test_finish_waits_for_a_held_witness(opt):
    """instance 1 is acquired on a stream, read there after a sleep and never released; pob_finish generates instances 2-4 while
    the read is still queued, and instance 3 goes to instance 1's slot"""
    import torch
    inps = _pool()[8:13]
    c, m = _handle(opt)
    st = torch.cuda.Stream()
    try:
        bufs = _buffers(c, 1)
        c.submit(c.pack(inps))
        i0, _ = c.acquire(st.cuda_stream)
        c.release(i0, st.cuda_stream)
        i1, p1 = c.acquire(st.cuda_stream)
        assert (i0, i1) == (0, 1)
        ev = _sleep(st)
        _copy(st, bufs[0], p1)
        _open(ev, "pob_finish was called")
        assert c.finish().n_ok == len(inps)
        st.synchronize()
        _same(bufs[0], _want(inps[1], m), "held instance 1")
    finally:
        _sync(st)
        c.close()


@OPTS
@pytest.mark.parametrize("accessor", ["witness", "write_wtns", "r1cs_products", "r1cs_products_other_stream"])
def test_host_reads_of_a_stream_acquired_witness(opt, accessor, tmp_path):
    """Instance 0 is released on stream a behind a sleep, instance 1 is rejected, instance 2 is acquired and released, and instance
    3 -- in instance 1's slot, expanded on the library's stream after instance 2, which reuses instance 0's slot -- is acquired on
    stream b, which returns at once.  While its expansion still waits for the sleep, one accessor is called and must read
    instance 3's witness: witness(), write_wtns(), r1cs_products() with no stream, or r1cs_products() on a third stream that did
    not acquire."""
    import torch
    import pob_b200
    inps = _pool()[REJECTED - 1:REJECTED + 4]
    c, m = _handle(opt)
    a, b, other = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    path = str(tmp_path / "w.wtns")
    R = None
    try:
        # first use of the exporter, the row plan and the allocator's blocks on `other`, outside the window
        assert c.run_packed(c.pack(inps[:1])).status[0] == 0
        if accessor == "write_wtns":
            c.write_wtns(0, path)
        elif accessor.startswith("r1cs_products"):
            f = str(tmp_path / "spend.r1cs")
            pob_b200.write_r1cs(SPEND, f, opt=opt)
            R = R1cs(f)
            c.r1cs_products(0, 0, R.m, stream=other if accessor.endswith("other_stream") else None)
        torch.cuda.synchronize()
        c.submit(c.pack(inps))
        i0, _ = c.acquire(a.cuda_stream)
        ev = _sleep(a)
        c.release(i0, a.cuda_stream)
        assert c.acquire(b.cuda_stream) == (1, None)
        i2, _ = c.acquire(b.cuda_stream)
        c.release(i2)
        i3, p3 = c.acquire(b.cuda_stream)
        assert (i0, i2, i3) == (0, 2, 3) and p3 is not None
        _open(ev, "%s(3) was called" % accessor)
        if accessor == "witness":
            got = c.witness(3)
        elif accessor == "write_wtns":
            c.write_wtns(3, path)
        else:
            got = c.r1cs_products(3, 0, R.m, stream=other if accessor.endswith("other_stream") else None)
            other.synchronize()
        c.release(3)
        assert c.finish().n_ok == len(inps) - 1
        want = _want(inps[3], m)
        if accessor == "witness":
            diff = np.nonzero((got != want).any(axis=1))[0]
            assert len(diff) == 0, "witness(3): %d entries differ from the oracle, first %d" % (len(diff), diff[0])
        elif accessor == "write_wtns":
            assert open(path, "rb").read() == _wtns_image(inps[3], m, tmp_path), "write_wtns(3) differs from the oracle's .wtns"
        else:
            for g, w, v in zip(got, R.products(witness_ints(want)), "abc"):
                bad = np.nonzero(witness_ints(g.cpu().numpy()) != w)[0]
                assert len(bad) == 0, "%s(3): %d rows of %s.w differ, first %d" % (accessor, len(bad), v, bad[0])
    finally:
        _sync(a, b, other)
        c.close()


def _wtns_image(inp, m, tmp_path):
    """the oracle's .wtns of `inp`; for a reduced handle the same file over the reduced entries (n_signals at bytes 60..64, the
    witness section's size at 68..76)"""
    ref = str(tmp_path / "oracle.wtns")
    _oracle(inp).write_wtns(ref)
    raw = open(ref, "rb").read()
    if m is None:
        return raw
    n = len(m)
    hdr = bytearray(raw[:76])
    assert int.from_bytes(hdr[60:64], "little") == _oracle(inp).n_signals
    hdr[60:64] = n.to_bytes(4, "little")
    hdr[68:76] = (32 * n).to_bytes(8, "little")
    return bytes(hdr) + np.ascontiguousarray(_want(inp, m)).tobytes()


def test_main_shape_reduced_quotient_on_a_consumer_stream():
    """the real consumer: 4 distinct synthetic main-shape instances through 2 slots, the quotient of each computed on the consumer
    stream with no host wait; each equals the same instance's quotient computed afterwards by the synchronous call"""
    import torch
    import pob_b200
    from pob_b200 import synth
    packed = synth.pack_instances(synth.make_batch(4, MAIN_SHAPE, seed=7503), MAIN_SHAPE)
    c = pob_b200.Circuit(pob_b200.MAIN_PROOF_OF_BURN, max_slots=2, opt=1)
    st = torch.cuda.Stream()
    try:
        got = {}
        c.submit(packed)
        while True:
            r = c.acquire(st.cuda_stream)
            if r is None:
                break
            idx, dptr = r
            assert dptr is not None
            got[idx] = c.r1cs_quotient(idx, stream=st)
            c.release(idx, st.cuda_stream)
        assert (c.finish().status == 0).all() and sorted(got) == [0, 1, 2, 3]
        st.synchronize()
        assert not torch.equal(got[0], got[1])
        for k in (0, 2):
            assert (c.run_packed(packed[k:k + 2]).status == 0).all()
            for i in (k, k + 1):
                assert torch.equal(c.r1cs_quotient(i - k), got[i]), "instance %d" % i
    finally:
        _sync(st)
        c.close()


def test_first_quotient_on_a_consumer_stream(tmp_path):
    """On a fresh handle the first r1cs_quotient runs on a consumer stream, right after the row plan and the transform tables are
    uploaded: it equals the model.  The uploads are ordered before the stream's first kernel by a synchronisation at their end;
    this test cannot make such a copy late, so it checks the value only."""
    import torch
    import pob_b200
    inp = _pool()[8]
    c, m = _handle(1)
    st = torch.cuda.Stream()
    try:
        c.submit(c.pack([inp]))
        idx, dptr = c.acquire(st.cuda_stream)
        assert idx == 0 and dptr is not None
        q = c.r1cs_quotient(idx, stream=st)
        c.release(idx, st.cuda_stream)
        assert c.finish().n_ok == 1
        st.synchronize()
        f = str(tmp_path / "spend_o1.r1cs")
        pob_b200.write_r1cs(SPEND, f, opt=1)
        R = R1cs(f)
        W = witness_ints(_want(inp, m))
        A, B, C = R.products(W)
        want = qm.quotient(A, B, C, W[:R.n_pub_out + R.n_pub_in + 1], R.m)
        got = witness_ints(q.cpu().numpy())
        assert (got == want).all(), "entries %s differ" % np.nonzero(got != want)[0][:10]
    finally:
        _sync(st)
        c.close()
