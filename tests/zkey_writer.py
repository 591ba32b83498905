"""A test-only writer of snarkjs Groth16 `.zkey` files in the format pob_b200.h describes (as far as known here), written from that
description alone.  A Zkey holds the header fields, the section-2 and section-3 points, the section-4 entries (a numpy structured array)
and a source per point section 5-9; write() streams it, so a key larger than memory can be written from tiled points.  Every field is
a plain attribute, so a test corrupts a key by changing one before it writes: the magic, a modulus, an entry, the section order, a
section's declared size, a dropped or repeated section, a truncation.

Integers little endian.  "zkey", u32 version, u32 n_sections, then per section u32 id, u64 size, content.  Section 4 values are
c R^2 mod r (R = 2^256)."""
import struct

import numpy as np

R_MOD = 21888242871839275222246405745257275088548364400416034343698204186575808495617
Q_MOD = 21888242871839275222246405745257275088696311157297823662689037894645226208583
MONT = (1 << 256) % R_MOD
ENTRY = np.dtype([("matrix", "<u4"), ("constraint", "<u4"), ("signal", "<u4"), ("value", "<u8", (4,))])
SEC2_POINTS = ("alpha1", "beta1", "beta2", "gamma2", "delta1", "delta2")
SEC2_SIZES = {"alpha1": 64, "beta1": 64, "beta2": 128, "gamma2": 128, "delta1": 64, "delta2": 128}
CHUNK = 1 << 24


def limbs(vals):
    """ints -> (n, 4) uint64 limbs (each value < 2^256)"""
    vals = [int(v) for v in vals]
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(4):
            out[i, k] = (v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF
    return out


def encode_values(vals, canonical=False):
    """coefficients (ints mod r) -> (n, 4) uint64 limbs of c R^2 mod r, or of c itself with canonical=True"""
    cache = {}
    out = []
    for v in vals:
        v = int(v) % R_MOD
        if v not in cache:
            cache[v] = v if canonical else v * MONT * MONT % R_MOD
        out.append(cache[v])
    return limbs(out)


def entries_from_r1cs(R, domain_rows=None, canonical=False, public_rows=True):
    """the section-4 entries of a `.r1cs` (tests/r1cs_reader.R1cs): every A and B term in row order, then snarkjs's public rows
    (constraint m + s, signal s, value 1) for s = 0 .. n_pub"""
    row, which = R.term_lc // 3, R.term_lc % 3
    sel = which < 2
    n_pub = R.n_pub_out + R.n_pub_in
    extra = n_pub + 1 if public_rows else 0
    e = np.zeros(int(sel.sum()) + extra, dtype=ENTRY)
    k = int(sel.sum())
    e["matrix"][:k] = which[sel]
    e["constraint"][:k] = row[sel]
    e["signal"][:k] = R.wire[sel]
    e["value"][:k] = encode_values(R.coef[sel], canonical)
    if extra:
        e["constraint"][k:] = R.m + np.arange(extra)
        e["signal"][k:] = np.arange(extra)
        e["value"][k:] = encode_values([1] * extra, canonical)
    return e


class Tiled:
    """a point section of `count` points repeating `tile` (bytes of whole points), streamed"""

    def __init__(self, tile, count, point_bytes):
        self.tile, self.count, self.pb = bytes(tile), int(count), int(point_bytes)

    @property
    def nbytes(self):
        return self.count * self.pb

    def chunks(self):
        per = len(self.tile) // self.pb
        reps = max(1, CHUNK // len(self.tile))
        block = self.tile * reps
        left = self.count
        while left:
            n = min(left, per * reps)
            yield block[:n * self.pb]
            left -= n


def _nbytes(src):
    return src.nbytes if isinstance(src, Tiled) else len(memoryview(src).cast("B"))


def _chunks(src):
    if isinstance(src, Tiled):
        yield from src.chunks()
    else:
        mv = memoryview(src).cast("B")
        for o in range(0, len(mv), CHUNK):
            yield mv[o:o + CHUNK]


class Zkey:
    def __init__(self, n_vars, n_pub, domain, sec2, ic, entries, points):
        """sec2: {name: bytes} for the six points of section 2; ic: bytes of n_pub + 1 G1 points; entries: ENTRY array;
        points: {5: a, 6: b1, 7: b2, 8: c, 9: h}, each bytes, a numpy array or a Tiled"""
        self.magic, self.version, self.protocol = b"zkey", 1, 1
        self.n8q, self.q, self.n8r, self.r = 32, Q_MOD, 32, R_MOD
        self.n_vars, self.n_pub, self.domain = n_vars, n_pub, domain
        self.sec2, self.ic, self.entries, self.points = dict(sec2), ic, entries, dict(points)
        self.n_coefs = None                                  # None: len(entries)
        self.order = [1, 2, 3, 4, 5, 6, 7, 8, 9]             # ids in file order; a (id, bytes) item is an extra section
        self.size_delta = {}                                 # id -> bytes added to the declared size (content unchanged)
        self.truncate = None                                 # total file bytes to keep

    def section2(self):
        head = struct.pack("<I", self.n8q) + self.q.to_bytes(32, "little") + struct.pack("<I", self.n8r) + self.r.to_bytes(32, "little")
        head += struct.pack("<III", self.n_vars, self.n_pub, self.domain)
        return head + b"".join(bytes(self.sec2[k]) for k in SEC2_POINTS)

    def _content(self, sid):
        """(size, chunk iterator) of section sid"""
        if sid == 1:
            b = struct.pack("<I", self.protocol)
        elif sid == 2:
            b = self.section2()
        elif sid == 3:
            b = bytes(self.ic)
        elif sid == 4:
            n = len(self.entries) if self.n_coefs is None else self.n_coefs
            ent = np.ascontiguousarray(self.entries)
            size = 4 + ent.nbytes

            def it():
                yield struct.pack("<I", n)
                yield from _chunks(ent.view(np.uint8))
            return size, it()
        else:
            src = self.points[sid]
            return _nbytes(src), _chunks(src)
        return len(b), iter([b])

    def write(self, path):
        """streams the file; returns its size"""
        written = 0
        with open(path, "wb") as f:
            def put(b):
                nonlocal written
                b = bytes(b)
                if self.truncate is not None:
                    b = b[:max(0, self.truncate - written)]
                f.write(b)
                written += len(b)
            put(self.magic + struct.pack("<II", self.version, len(self.order)))
            for item in self.order:
                if isinstance(item, tuple):
                    sid, body = item
                    size, it = len(body), iter([body])
                else:
                    sid = item
                    size, it = self._content(sid)
                put(struct.pack("<IQ", sid, size + self.size_delta.get(sid, 0)))
                for ch in it:
                    put(ch)
                    if self.truncate is not None and written >= self.truncate:
                        return written
        return written


def sections(path):
    """{id: (content offset, size)} of a .zkey's section table (the last occurrence of an id)"""
    out = {}
    with open(path, "rb") as f:
        hd = f.read(12)
        pos = 12
        for _ in range(struct.unpack_from("<I", hd, 8)[0]):
            f.seek(pos)
            sid, size = struct.unpack("<IQ", f.read(12))
            out[sid] = (pos + 12, size)
            pos += 12 + size
    return out


def read_section(path, sid):
    off, size = sections(path)[sid]
    with open(path, "rb") as f:
        f.seek(off)
        return f.read(size)
