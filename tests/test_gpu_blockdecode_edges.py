"""Column-block read path at its edges: LZ4 block decode (csrc/lz4.cu, MO_XCALL_LZ4_DECODE) on blocks written sequence by sequence
(tests/lz4_blocks.py) against their decoded-bytes model and the oracle decoder, and vector unmarshal (csrc/vecdecode.cu,
MO_XCALL_VECTOR_UNMARSHAL) against a restatement of Vector.UnmarshalBinary.

The LZ4 blocks aim at the decode kernel's own branches: source window refills inside lengths and offsets, ring versus global matches on
both sides of the ring size, overlapping matches with periods below the warp width, the conditional sync after a match, and more blocks
than resident warps so that warps decode a second block after another one's bytes went through their ring and window."""
import ctypes
import re
import struct

import numpy as np
import pytest

import lz4_blocks as L
from matrixone_b200 import capi, ops
from matrixone_b200.ops import VectorView
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, marshal_vector, xcall
from test_lz4_blocks import oracle_decode

pytestmark = pytest.mark.gpu

FILL = 0xA7              # what the output buffers hold before a call: a byte the kernel must never leave behind
RESIDENT_WARPS = 132 * 64   # an H100's resident warps at most: block indices above this are decoded in a later grid-stride step


def _upload(buf, off, arr):
    arr = np.ascontiguousarray(arr)
    if arr.nbytes:
        capi.check(buf.lib.MoB200_Upload(buf.ptr + off, arr.ctypes.data, arr.nbytes), buf.lib)


def _bad_block(msg):
    m = re.search(r"block (\d+) ", msg)
    assert m, msg
    return int(m.group(1))


class Lz4Call:
    """blocks placed by the test: source block i at a chosen misalignment mod 16, its output at an unaligned offset with a gap behind it"""

    def __init__(self, blocks, dls, mis):
        so, do, self.desc = 0, 0, np.zeros((len(blocks), 4), np.int64)
        for i, (b, dl) in enumerate(zip(blocks, dls)):
            so = (so + 15) // 16 * 16 + mis[i] % 16
            do = (do + 15) // 16 * 16 + (5 * i + 3) % 16
            self.desc[i] = (so, len(b), do, dl)
            so += len(b); do += dl + 9
        self.src = np.zeros(so + 16, np.uint8)
        for i, b in enumerate(blocks):
            self.src[self.desc[i, 0]:self.desc[i, 0] + len(b)] = np.frombuffer(b, np.uint8)
        self.dbytes, self.dofs = do + 16, self.desc[:, 2].copy()
        self.dsrc, self.ddesc = DeviceBuffer.from_numpy(self.src), DeviceBuffer.from_numpy(self.desc.reshape(-1))
        self.ddst = DeviceBuffer.from_numpy(np.full(self.dbytes, FILL, np.uint8))

    def run(self):
        return xcall(capi.XCALL_LZ4_DECODE, [Vector(data_ptr=self.ddst.ptr, data_nbytes=self.dbytes, length=1),
                                            Vector(data_ptr=self.dsrc.ptr, data_nbytes=self.src.nbytes, length=1),
                                            Vector(data_ptr=self.ddesc.ptr, data_nbytes=self.desc.nbytes, length=1)],
                     len(self.desc), raise_on_error=False)

    def drop(self, i):
        """block i becomes the empty block (no source, no output)"""
        self.desc[i] = 0
        _upload(self.ddesc, 32 * i, self.desc[i])

    def check(self, wants, names, gaps=True):
        """every block's output equals its expected bytes (None: not checked), and (gaps) nothing else in the output buffer was written"""
        got = self.ddst.to_numpy(np.uint8, self.dbytes)
        exp = np.full(self.dbytes, FILL, np.uint8)
        care = np.full(self.dbytes, gaps)
        for i, w in enumerate(wants):
            if w is not None:
                exp[self.dofs[i]:self.dofs[i] + len(w)] = np.frombuffer(w, np.uint8)
                care[self.dofs[i]:self.dofs[i] + len(w)] = True
        wrong = care & (got != exp)
        if wrong.any():
            first = int(np.argmax(wrong))
            i = int(np.searchsorted(self.dofs, first, side="right")) - 1
            pytest.fail("output byte %d (block %d %s, byte %d) is %d, expected %d" % (first, i, names[i], first - self.dofs[i], got[first], exp[first]))

    def free(self):
        for b in (self.dsrc, self.ddesc, self.ddst):
            b.free()


def _decode_exactly(entries):
    """entries = [(name, block bytes, expected bytes, source misalignment)]: one call, every output byte checked"""
    call = Lz4Call([e[1] for e in entries], [len(e[2]) for e in entries], [e[3] for e in entries])
    rc, msg = call.run()
    assert rc == 0, msg
    call.check([e[2] for e in entries], [e[0] for e in entries])
    call.free()


# ------------------------------------------------------------------------------------------------------------- LZ4 exactness
def test_lz4_edge_and_random_blocks_decode_to_the_model(gpu):
    """every edge-table block at source misalignments 0..15 and 3000 random edge blocks (the corpus test_lz4_blocks.py shows reaches every
    branch of the kernel), the empty block in both spellings, at unaligned output offsets, in one call"""
    entries = [(name, L.encode(s, t), L.model(s, t), m) for name, s, t, m in L.placed_corpus()]
    entries += [("no_source_bytes", b"", b"", 0), ("empty_block", b"\x00", b"", 7), ("empty_block_aligned", b"\x00", b"", 0)]
    assert any(len(e[2]) > 65536 for e in entries if e[0] == "offset_65535_last")
    _decode_exactly(entries)


def test_lz4_more_blocks_than_resident_warps(gpu):
    """20,000 blocks, most of them tiny.  Far, overlapping-far and ring-overlap blocks sit above RESIDENT_WARPS, so the warp that decodes
    them has decoded another block into its ring and window first."""
    rng = np.random.default_rng(3)
    table = L.edge_table()
    heavy = ["far_edge_off3", "far_off4097", "far_overlap_long_off17", "ring_overlap_off5", "ring_edge_off31", "sync_boundary_off31",
             "offset_65535_overlapping", "literal_wraps_ring", "window_walk_500", "nc_ends_in_long_match"]
    entries = []
    for i in range(20000):
        if i >= RESIDENT_WARPS and i % 613 == 0 or i % 4999 == 17:
            name = heavy[(i // 613) % len(heavy)]
            s, t = table[name]
        else:
            name = "tiny_%d" % i
            lit = L.random_bytes(rng, int(rng.integers(1, 40)))
            s = [(lit, int(rng.integers(1, len(lit) + 1)), int(rng.integers(4, 60)))] if rng.random() < 0.7 else []
            t = L.random_bytes(rng, int(rng.integers(0, 20)))
        entries.append((name, L.encode(s, t), L.model(s, t), i % 16))
    assert sum(1 for i, e in enumerate(entries) if i > RESIDENT_WARPS and not e[0].startswith("tiny")) >= 10
    _decode_exactly(entries)


# ------------------------------------------------------------------------------------------------------------- accept / reject
ACCEPT_SET = ["literals_only_1", "literals_only_15_ext_0", "nibble15_ext0_both", "ext_255_then_0", "ext_255_255_then_0",
              "ring_overlap_off1", "ring_overlap_off3", "ring_overlap_off31", "ring_overlap_off32", "ring_overlap_off33",
              "ring_edge_off5", "ring_edge_off64", "far_edge_off3", "far_edge_off17", "far_edge_off65", "far_overlap_long_off1",
              "far_overlap_long_off7", "sync_boundary_off31", "sync_past_boundary_off100", "window_walk_490", "window_walk_500",
              "window_walk_505", "window_walk_510", "nc_ends_in_match", "nc_ends_in_long_match", "nc_match_in_last_5",
              "nc_match_starts_late", "ring_edge_off4092_len4", "far_edge_off4091_len6", "sync_past_boundary_off31"]


def _mutants(name, seqs, tail):
    blk, dl = L.encode(seqs, tail), len(L.model(seqs, tail))
    out = [("%s cut to %d bytes" % (name, k), blk[:k], dl) for k in range(len(blk))]
    for p in L.parse(blk)[2]:
        for v in sorted({0, 255, (blk[p] + 1) & 255, (blk[p] - 1) & 255} - {blk[p]}):
            out.append(("%s byte %d = %d" % (name, p, v), blk[:p] + bytes([v]) + blk[p + 1:], dl))
    out += [("%s dl + 1" % name, blk, dl + 1)] + ([("%s dl - 1" % name, blk, dl - 1)] if dl else [])
    return out


def test_lz4_accepts_exactly_the_blocks_the_oracle_accepts_and_names_the_lowest_bad_one(gpu):
    """Truncations, token / extension / offset bytes set to 0, 255 and +-1, and decoded sizes off by one, of 30 edge blocks, all in one
    call.  The call fails while an oracle-rejected block is in it and names the lowest one; that block is then emptied and the call
    repeated, so every rejected block is named in turn.  The last call succeeds and the accepted mutants decode to the oracle's bytes."""
    table = L.edge_table()
    muts = [m for name in ACCEPT_SET for m in _mutants(name, *table[name])]
    order = np.random.default_rng(5).permutation(len(muts))
    muts = [muts[i] for i in order]
    verdict = [oracle_decode(b, dl) for _, b, dl in muts]
    wants = [out if n == dl else None for (_, _, dl), (n, out) in zip(muts, verdict)]
    bad = [i for i, w in enumerate(wants) if w is None]
    assert len(muts) > RESIDENT_WARPS and min(bad) < RESIDENT_WARPS < max(bad)
    assert len(bad) < len(muts)
    call = Lz4Call([m[1] for m in muts], [m[2] for m in muts], [i for i in range(len(muts))])
    for expect in bad:
        rc, msg = call.run()
        assert rc != 0, "the call succeeded with oracle-rejected block %d (%s) in it" % (expect, muts[expect][0])
        got = _bad_block(msg)
        assert got == expect, "named block %d (%s, oracle: %s), the lowest oracle-rejected one is %d (%s)" % (
            got, muts[got][0], "accepts" if wants[got] is not None else "rejects", expect, muts[expect][0])
        call.drop(got)
    rc, msg = call.run()
    assert rc == 0, msg
    call.check(wants, [m[0] for m in muts], gaps=False)
    call.free()


# ------------------------------------------------------------------------------------------------------------- vector unmarshal
def go_unmarshal(b):
    """Vector.UnmarshalBinary (vector.go:766-814) with Bitmap.Unmarshal (bitmap.go:419-431), restated over a buffer of exactly the marshalled
    bytes: a dict of the fields and sections, or None where the Go code panics (a slice bound past the bytes, a bitmap size that is negative
    as an int or not a multiple of 8)."""
    n = len(b)

    def cut(lo, k):
        if lo + k > n:
            raise IndexError
        return b[lo:lo + k]

    u32 = lambda lo: struct.unpack("<I", cut(lo, 4))[0]
    try:
        typ = cut(1, 16)
        v = dict(vclass=cut(0, 1)[0], oid=typ[0], size=struct.unpack("<i", typ[4:8])[0], width=struct.unpack("<i", typ[8:12])[0],
                 scale=struct.unpack("<i", typ[12:16])[0], length=u32(17), count=0, words=b"")
        o = 25
        v["data"] = cut(o, u32(21)); o += len(v["data"])
        v["area"] = cut(o + 4, u32(o)); o += 4 + len(v["area"])
        nsp_len = u32(o); o += 4
        if nsp_len:
            nsp = cut(o, nsp_len); o += nsp_len
            if nsp_len < 24:
                raise IndexError
            v["count"] = struct.unpack("<q", nsp[:8])[0]
            size = struct.unpack("<Q", nsp[16:24])[0]
            if size >= 1 << 63 or 24 + size > nsp_len or size % 8:
                raise IndexError
            v["words"] = nsp[24:24 + size]
        v["sorted"] = cut(o, 1)[0]
        return v
    except IndexError:
        return None


def blob(data=b"", area=b"", length=None, nsp=None, vclass=0, oid=capi.T_UINT8, size=1, width=3, scale=-2, sorted_flag=0, trailer=b""):
    """marshalled bytes with every section given explicitly (nsp = the bitmap bytes, b"" for none)"""
    length = len(data) if length is None else length
    nsp = b"" if nsp is None else nsp
    return (bytes([vclass, oid, 0, 0, 0]) + struct.pack("<iiiII", size, width, scale, length, len(data)) + data +
            struct.pack("<I", len(area)) + area + struct.pack("<I", len(nsp)) + nsp + bytes([sorted_flag]) + trailer)


def bitmap(words, count=None, nbits=None, size=None):
    w = np.asarray(words, np.uint64).tobytes()
    count = sum(bin(int(x)).count("1") for x in words) if count is None else count
    return struct.pack("<qQQ", count, len(words) * 64 if nbits is None else nbits, len(w) if size is None else size) + w


class Unmarshal:
    """reusable device buffers for many MO_XCALL_VECTOR_UNMARSHAL calls"""
    CAP = 2_600_000

    def __init__(self):
        self.src = DeviceBuffer(2 * self.CAP + 64)          # a header, data and area of up to CAP bytes each
        self.data, self.area, self.nulls = DeviceBuffer(self.CAP + 64), DeviceBuffer(self.CAP + 64), DeviceBuffer(8 * 4096)
        self.fill = np.full(self.CAP + 64, FILL, np.uint8)

    def run(self, b, mis=None, data_cap=None, area_cap=None, nulls_cap=None, want_nulls=True):
        """mis = source misalignment in device memory, None: host source.  Returns (rc, message, view, data, area, nulls words)"""
        ref = go_unmarshal(b)
        if ref is None:   # room for whatever the header claims, so that only the parse can fail the call
            ref = dict(data=bytes(len(b)), area=bytes(len(b)), length=struct.unpack("<I", b[17:21])[0] if len(b) >= 21 else 0)
        data_cap = len(ref["data"]) + 16 if data_cap is None else data_cap
        area_cap = len(ref["area"]) + 16 if area_cap is None else area_cap
        want = (ref["length"] + 63) // 64
        nulls_cap = want + 2 if nulls_cap is None else nulls_cap
        arr = np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
        if mis is None:
            srcv = Vector(data_ptr=arr.ctypes.data, data_nbytes=len(b), length=1)
        else:
            _upload(self.src, mis, arr[:len(b)])
            srcv = Vector(data_ptr=self.src.ptr + mis, data_nbytes=len(b), length=1)
        _upload(self.data, 0, self.fill[:data_cap + 16])
        _upload(self.area, 0, self.fill[:area_cap + 16])
        _upload(self.nulls, 0, self.fill[:8 * (nulls_cap + 2)])
        view = np.zeros(ctypes.sizeof(VectorView), np.uint8)
        rc, msg = xcall(capi.XCALL_VECTOR_UNMARSHAL, [
            Vector(data=view, length=1), Vector(data_ptr=self.data.ptr, data_nbytes=data_cap, length=1),
            Vector(data_ptr=self.area.ptr, data_nbytes=area_cap, length=1),
            Vector(data_ptr=self.nulls.ptr, data_nbytes=8 * nulls_cap, length=1) if want_nulls else Vector(length=0), srcv], 1, raise_on_error=False)
        return (rc, msg, VectorView.from_buffer_copy(view.tobytes()), self.data.to_numpy(np.uint8, data_cap + 16),
                self.area.to_numpy(np.uint8, area_cap + 16), self.nulls.to_numpy(np.uint8, 8 * (nulls_cap + 2)))

    def check(self, b, mis=None, want_nulls=True, **caps):
        """the call succeeds exactly when the restatement accepts the bytes, and then every field and section matches it"""
        ref = go_unmarshal(b)
        rc, msg, view, data, area, nulls = self.run(b, mis, want_nulls=want_nulls, **caps)
        where = "%d bytes at %s" % (len(b), "host" if mis is None else "misalignment %d" % mis)
        if ref is None:
            assert rc != 0 and "malformed" in msg, "malformed bytes accepted: %s (%s)" % (where, msg)
            return
        assert rc == 0, "%s: %s" % (where, msg)
        got = (view.vclass, view.oid, view.size, view.width, view.scale, view.length, view.data_len, view.area_len, view.null_count,
               view.nulls_words, view.sorted, view.bad)
        want_words = (ref["length"] + 63) // 64
        assert got == (ref["vclass"], ref["oid"], ref["size"], ref["width"], ref["scale"], ref["length"], len(ref["data"]),
                       len(ref["area"]), ref["count"], want_words, ref["sorted"], 0), where
        for name, out, sec in (("data", data, ref["data"]), ("area", area, ref["area"])):
            assert out[:len(sec)].tobytes() == sec, "%s section differs: %s" % (name, where)
            assert (out[len(sec):] == FILL).all(), "written past the %s section: %s" % (name, where)
        words = (ref["words"] + bytes(8 * want_words))[:8 * want_words]
        if want_nulls:
            assert nulls[:len(words)].tobytes() == words, "nulls differ: " + where
            assert (nulls[len(words):] == FILL).all(), "written past the null words: " + where
        else:
            assert (nulls == FILL).all(), where

    def free(self):
        for x in (self.src, self.data, self.area, self.nulls):
            x.free()


@pytest.fixture(scope="module")
def um(gpu):
    u = Unmarshal()
    yield u
    u.free()


SECTION_LENGTHS = list(range(18)) + [63, 64, 65, 8191, 8192, 8193]
PLACEMENTS = list(range(16)) + [None]


def test_unmarshal_section_lengths_at_every_source_alignment(um):
    rng = np.random.default_rng(11)
    for ln in SECTION_LENGTHS:
        d, a = L.random_bytes(rng, ln), L.random_bytes(rng, ln)
        fixed = blob(d, oid=capi.T_UINT8, length=ln)
        varlena = blob(d, a, length=ln // 3, oid=61, size=24, sorted_flag=1)
        for mis in PLACEMENTS:
            um.check(fixed, mis)
            um.check(varlena, mis)


def test_unmarshal_a_column_past_one_grid_stride(um):
    """data and area of 2.5 MB: more 8-byte words than the copy kernel's grid has threads, so its grid-stride loop runs"""
    rng = np.random.default_rng(12)
    d, a = L.random_bytes(rng, 2_500_003), L.random_bytes(rng, 2_400_005)
    b = blob(d, a, length=2_500_003 // 24, oid=61, size=24)
    for mis in (0, 1, 7, 8, 13, None):
        um.check(b, mis, want_nulls=False)


def test_unmarshal_null_bitmaps(um):
    """bitmaps of exactly (length + 63) / 64 words, fewer (the rest reads as not NULL), more (cut), an empty one, and no nulls wanted"""
    rng = np.random.default_rng(13)
    for length in (1, 63, 64, 65, 8193):
        want = (length + 63) // 64
        d = L.random_bytes(rng, 8 * length)
        mask = rng.random(length) < 0.3
        mask[-1] = True
        words = bitmap_from_bools(mask)
        for w in (words, words[:want - 1], np.concatenate([words, rng.integers(0, 2 ** 63, 3).astype(np.uint64)]), []):
            b = blob(d, length=length, oid=capi.T_INT64, size=8, nsp=bitmap(list(w), nbits=length))
            for mis in (0, 3, None):
                um.check(b, mis)
            um.check(b, 5, want_nulls=False)
        um.check(blob(d, length=length, oid=capi.T_INT64, size=8), 2)               # no bitmap: no row is NULL


def test_unmarshal_constant_vectors_sorted_flag_and_trailing_bytes(um):
    const = blob(struct.pack("<q", -42), length=1000, vclass=1, oid=capi.T_INT64, size=8)
    const_null = blob(b"", length=1000, vclass=1, oid=capi.T_INT64, size=8, nsp=bitmap([1], nbits=1))
    sorted_col = blob(np.arange(300, dtype=np.int64).tobytes(), length=300, oid=capi.T_INT64, size=8, sorted_flag=1)
    for b in (const, const_null, sorted_col):
        for trailer in (b"", b"\x01", b"\xff" * 13):
            for mis in (0, 9, None):
                um.check(b + trailer, mis)
    v = go_unmarshal(const_null)
    assert v["vclass"] == 1 and v["data"] == b"" and v["words"] == struct.pack("<Q", 1)


def _valid_blobs():
    rng = np.random.default_rng(14)
    return [blob(L.random_bytes(rng, 40), L.random_bytes(rng, 9), length=5, nsp=bitmap([0b10110])),
            blob(L.random_bytes(rng, 17), length=17, sorted_flag=1),
            blob(b"", length=0),
            blob(struct.pack("<q", 7), length=64, vclass=1, oid=capi.T_INT64, size=8, nsp=bitmap([1, 0])),
            blob(L.random_bytes(rng, 24), length=65, nsp=bitmap([3, 1 << 63, 5], nbits=130))]


def _corruptions(b):
    """the same bytes with dataLen / areaLen / nspLen and the bitmap's size field rewritten"""
    dl = struct.unpack("<I", b[21:25])[0]
    ao = 25 + dl
    al = struct.unpack("<I", b[ao:ao + 4])[0]
    no = ao + 4 + al
    nl = struct.unpack("<I", b[no:no + 4])[0]
    put = lambda o, fmt, v: b[:o] + struct.pack(fmt, v) + b[o + struct.calcsize(fmt):]
    out = []
    for v in (0, 1, dl - 1, dl + 1, dl + 4, len(b), len(b) - 25, 0xFFFFFFFF, 0x80000000):
        out.append(put(21, "<I", v & 0xFFFFFFFF))
    for v in (0, 1, al + 1, al - 1, al + 5, len(b) - ao - 4, len(b) - ao - 5, 0xFFFFFFFF):
        out.append(put(ao, "<I", v & 0xFFFFFFFF))
    for v in list(range(1, 24)) + [nl + 1, nl - 1, nl + 8, nl - 8, 0xFFFFFFFF]:
        out.append(put(no, "<I", v & 0xFFFFFFFF))
    if nl >= 24:
        so = no + 4 + 16
        size = struct.unpack("<Q", b[so:so + 8])[0]
        for v in (0, 1, 7, size - 1, size + 1, size - 8, size + 8, nl - 24, nl - 23, 2 ** 63, 2 ** 64 - 8, 2 ** 64 - 16, 2 ** 64 - 24):
            out.append(put(so, "<Q", v % 2 ** 64))
    return out


def test_unmarshal_fails_exactly_when_the_bytes_are_malformed(um):
    """every prefix of valid vectors and their length fields rewritten (including a bitmap size near 2**64, which must not wrap around
    the bound check): the call fails exactly when the restatement of the Go decoder panics, and otherwise decodes like it"""
    seen = {True: 0, False: 0}
    for i, b in enumerate(_valid_blobs()):
        assert go_unmarshal(b) is not None
        cases = [b[:k] for k in range(len(b))] + _corruptions(b)
        for j, c in enumerate(cases):
            seen[go_unmarshal(c) is None] += 1
            um.check(c, None if j % 5 == 4 else (i + j) % 16)
    assert seen[True] > 300 and seen[False] > 10


def test_unmarshal_output_capacities(um):
    b = blob(np.arange(200, dtype=np.uint8).tobytes(), b"xyz" * 11, length=130, nsp=bitmap([1, 2, 4]))
    assert um.run(b, 0, data_cap=200, area_cap=33, nulls_cap=3)[0] == 0
    um.check(b, 0, data_cap=200, area_cap=33, nulls_cap=3)
    for caps in (dict(data_cap=199, area_cap=33, nulls_cap=3), dict(data_cap=200, area_cap=32, nulls_cap=3),
                 dict(data_cap=200, area_cap=33, nulls_cap=2)):
        rc, msg = um.run(b, 0, **caps)[:2]
        assert rc != 0 and "too small" in msg, caps
    assert um.run(b, 0, data_cap=200, area_cap=33, nulls_cap=0, want_nulls=False)[0] == 0


# ------------------------------------------------------------------------------------------------------------- end to end
def test_far_and_overlapping_far_matches_through_unmarshal_to_sum(gpu):
    """an int64 column whose block repeats a stretch from 5.6 KB back (a far match) and a constant run of 1000 values (an overlapping match
    of period 8 longer than the ring): LZ4 decode, unmarshal, AGG_SUM over the non-NULL rows equals numpy's sum"""
    rng = np.random.default_rng(15)
    a = rng.integers(-10 ** 9, 10 ** 9, 700)
    col = np.concatenate([a, a[:300], np.full(1000, 7), rng.integers(-10 ** 9, 10 ** 9, 100)]).astype(np.int64)
    null = rng.random(len(col)) < 0.1
    raw = marshal_vector(capi.T_INT64, col, len(col), nulls=bitmap_from_bools(null))
    seqs = [(raw[:25 + 5600], 5600, 2400), (raw[25 + 8000:25 + 8008], 8, 7992)]
    tail = raw[25 + 16000:]
    assert L.model(seqs, tail) == raw
    assert {"match_far", "match_far_overlap"} <= L.classify(seqs, 5, tail)
    call = Lz4Call([L.encode(seqs, tail)], [len(raw)], [5])
    rc, msg = call.run()
    assert rc == 0, msg
    call.check([raw], ["column"])
    n = len(col)
    data, nulls = DeviceBuffer(8 * n), DeviceBuffer(8 * ((n + 63) // 64))
    view = ops.vector_unmarshal_device(call.ddst.view(len(raw) + 16, int(call.desc[0, 2])), len(raw), data, None, nulls)
    assert view.length == n and view.data_len == 8 * n and view.null_count == int(null.sum())
    res, rn = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    xcall(capi.XCALL_AGG(capi.AGG_SUM, capi.T_INT64), [Vector(data=res, nulls=rn, length=1),
                                                        Vector(data_ptr=data.ptr, data_nbytes=8 * n, nulls_ptr=nulls.ptr, length=n)], n)
    assert res[0] == int(col[~null].sum())
    for x in (data, nulls):
        x.free()
    call.free()
