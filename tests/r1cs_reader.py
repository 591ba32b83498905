"""An independent reader of iden3 `.r1cs` files (binary format version 1), written from the format alone, for the tests.

Layout: "r1cs", u32 version, u32 nSections, then sections (u32 type, u64 size, content), integers little-endian.  Section 1:
u32 fieldDefSize, p, u32 nWires, nPubOut, nPubIn, nPrvIn, u64 nLabels, u32 mConstraints.  Section 2: per row A, B, C, each u32 nTerms
then nTerms x (u32 wire, fieldDefSize-byte LE coefficient); a row means A*B - C = 0.  Section 3: nWires x u64 labels.
Evaluation uses Python integers (numpy object arrays), nothing of the library."""
import struct

import numpy as np


class R1cs:
    def __init__(self, path):
        raw = open(path, "rb").read()
        self.size = len(raw)
        assert raw[:4] == b"r1cs", "bad magic"
        self.version, nsec = struct.unpack_from("<II", raw, 4)
        pos, secs = 12, {}
        for _ in range(nsec):
            typ, size = struct.unpack_from("<IQ", raw, pos)
            pos += 12
            secs[typ] = (pos, size)
            pos += size
        assert pos == len(raw), "sections do not cover the file"
        self.section_order = list(secs)
        h, hs = secs[1]
        fs = struct.unpack_from("<I", raw, h)[0]
        assert fs == 32 and hs == 4 + fs + 16 + 8 + 4
        self.p = int.from_bytes(raw[h + 4:h + 36], "little")
        self.n_wires, self.n_pub_out, self.n_pub_in, self.n_prv_in = struct.unpack_from("<IIII", raw, h + 36)
        self.n_labels = struct.unpack_from("<Q", raw, h + 52)[0]
        self.m = struct.unpack_from("<I", raw, h + 60)[0]
        # section 2: walk the combination headers, then gather every term at once
        c0, csize = secs[2]
        lc_off = np.zeros(3 * self.m, dtype=np.int64)
        lc_n = np.zeros(3 * self.m, dtype=np.int64)
        q = c0
        for i in range(3 * self.m):
            n = int.from_bytes(raw[q:q + 4], "little")
            lc_off[i], lc_n[i] = q + 4, n
            q += 4 + 36 * n
        assert q == c0 + csize, "constraint section size"
        self.lc_n = lc_n
        self.lc_start = np.concatenate(([0], np.cumsum(lc_n)[:-1])).astype(np.int64)
        T = int(lc_n.sum())
        self.n_terms = T
        self.term_lc = np.repeat(np.arange(3 * self.m, dtype=np.int64), lc_n)
        toff = np.repeat(lc_off, lc_n) + 36 * (np.arange(T, dtype=np.int64) - np.repeat(self.lc_start, lc_n))
        buf = np.frombuffer(raw, dtype=np.uint8)
        tb = buf[toff[:, None] + np.arange(36)]
        self.wire = np.ascontiguousarray(tb[:, :4]).view("<u4").ravel().astype(np.int64)
        limbs = np.ascontiguousarray(tb[:, 4:]).view("<u8").reshape(T, 4)
        self.coef_zero = ~limbs.any(axis=1)
        lo = limbs.astype(object)
        self.coef = lo[:, 0] + (lo[:, 1] << 64) + (lo[:, 2] << 128) + (lo[:, 3] << 192)
        l0, ls = secs[3]
        assert ls == 8 * self.n_wires
        self.labels = np.frombuffer(raw, dtype="<u8", count=self.n_wires, offset=l0)

    def lc_sorted_unique_nonzero(self):
        same = self.term_lc[1:] == self.term_lc[:-1]
        return bool((self.wire[1:][same] > self.wire[:-1][same]).all()) and not self.coef_zero.any() and bool((self.coef < self.p).all())

    def products(self, w):
        """w: object array (or list) of Python ints, one per wire -> (A.w, B.w, C.w) per row as object arrays"""
        w = np.asarray(w, dtype=object)
        prod = self.coef * w[self.wire]
        sums = np.zeros(3 * self.m, dtype=object)
        nz = self.lc_n > 0
        if self.n_terms:
            sums[nz] = np.add.reduceat(prod, self.lc_start[nz])
        sums = sums % self.p
        return sums[0::3], sums[1::3], sums[2::3]

    def failing_rows(self, w):
        A, B, C = self.products(w)
        return np.nonzero((A * B - C) % self.p != 0)[0]

    def rows_of_wire(self):
        """CSR index wire -> rows that reference it"""
        order = np.argsort(self.wire, kind="stable")
        rows = (self.term_lc // 3)[order]
        ptr = np.searchsorted(self.wire[order], np.arange(self.n_wires + 1))
        return ptr, rows

    def row_ok(self, r, w):
        vals = []
        for j in range(3):
            i = 3 * r + j
            s, n = int(self.lc_start[i]), int(self.lc_n[i])
            vals.append(sum(int(self.coef[t]) * int(w[int(self.wire[t])]) for t in range(s, s + n)) % self.p)
        return (vals[0] * vals[1] - vals[2]) % self.p == 0


def witness_ints(limbs):
    """(n, 4) uint64 limbs -> object array of Python ints"""
    lo = np.asarray(limbs).astype(object)
    return lo[:, 0] + (lo[:, 1] << 64) + (lo[:, 2] << 128) + (lo[:, 3] << 192)


def limbs_of(vals, p):
    """iterable of ints -> (n, 4) uint64 limbs of v mod p"""
    vals = [int(v) % p for v in vals]
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(4):
            out[i, k] = (v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF
    return out
