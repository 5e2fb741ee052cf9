"""Varlena vector columns laid out row by row for the row-wise distance and normalize_l2 edge tests, and per-row references.

Each row of a built column chooses its own length (0 included), whether it is stored inline in its 24-byte cell (at most 23 bytes)
or in the area, its offset mod 16 in the area, and whether its cell points at the bytes of an earlier row (as after a Shuffle of a
varlena column).  Area bytes no row owns hold FILL, so a kernel that reads past a row or at a wrong offset sees huge values.

The references are the oracle's restatements of the Go loops, called one row at a time: og_distance_rows_* with n = 1 and stride 0,
og_moarray_cossim_* and og_normalize_l2_*."""
import numpy as np

import oracle_lib as O
from matrixone_b200.vector import DeviceBuffer

FILL = 0x7F                 # area padding: every float32 / float64 made of these bytes is ~3.4e38 / ~1.4e306
INLINE_MAX = 23

# og_distance_rows kinds (metric/types.go MetricType) and the cosine similarity of moarray, which has no kind there
L2, IP, COSDIST, L1, L2SQ = 0, 1, 2, 3, 4
COSSIM = "cossim"
KINDS = (L2, L2SQ, IP, COSDIST, COSSIM, L1)


class Column:
    """cells uint8[24 * n] and area uint8[] of a varlena column built from rows[i] (a 1-D array of dtype) with, per row:
      store[i]  "i" inline (the row must fit in 23 bytes) or "a" area (any length, 0 and short rows included);
      pad[i]    the row's offset mod 16 in the area (area rows only);
      dup[i]    j < i: the cell is a copy of row j's cell (the row's own array and store are ignored), None: the row has its own bytes.
    kind[i] is what the row became: "inline", "area" or "dup"."""

    def __init__(self, rows, dtype, store=None, pad=None, dup=None, tail=16):
        n = len(rows)
        self.dtype = np.dtype(dtype)
        store = store or ["i" if len(r) * self.dtype.itemsize <= INLINE_MAX else "a" for r in rows]
        pad = pad if pad is not None else [0] * n
        dup = dup or [None] * n
        cells = np.zeros((n, 24), np.uint8)
        chunks, off = [], 0
        self.kind, self.offset = [], [None] * n
        self.rows = []
        for i in range(n):
            if dup[i] is not None:
                j = dup[i]
                assert j < i
                cells[i] = cells[j]
                self.rows.append(self.rows[j])
                self.offset[i] = self.offset[j]
                self.kind.append("dup")
                continue
            b = np.ascontiguousarray(rows[i], self.dtype).view(np.uint8).reshape(-1)
            self.rows.append(np.ascontiguousarray(rows[i], self.dtype))
            if store[i] == "i":
                assert b.size <= INLINE_MAX, (i, b.size)
                cells[i, 0] = b.size
                cells[i, 1:1 + b.size] = b
                self.kind.append("inline")
                continue
            gap = (pad[i] - off) % 16
            chunks.append(np.full(gap, FILL, np.uint8))
            off += gap
            u32 = cells[i].view(np.uint32)
            u32[0], u32[1], u32[2] = 0xFFFFFFFF, off, b.size
            chunks.append(b)
            self.offset[i] = off
            off += b.size
            self.kind.append("area")
        chunks.append(np.full(tail, FILL, np.uint8))
        self.cells = cells.reshape(-1)
        self.area = np.concatenate(chunks)
        self.n = n

    def __len__(self):
        return self.n

    def stores(self):
        """the store[] of this layout for a rebuild with other rows; a duplicated row then gets bytes of its own in the area"""
        return ["i" if k == "inline" else "a" for k in self.kind]

    def device(self, k):
        """(cells, area) as DeviceBuffers, the area a view that starts k bytes past a 256-aligned allocation; the view keeps its owner
        (free it with area.owner.free())"""
        cells = DeviceBuffer.from_numpy(self.cells)
        owner = DeviceBuffer.from_numpy(np.concatenate([np.full(k, FILL, np.uint8), self.area]))
        return cells, owner.view(self.area.nbytes, k)


def decode(cells, area, i, dtype):
    """row i of a varlena column by the cell rules of varlena_ref (csrc/common.cuh): bs[0] <= 23 inline, else u32[1] = offset and
    u32[2] = length; None when the cell points outside the area"""
    c = np.asarray(cells[24 * i:24 * i + 24], np.uint8)
    if c[0] <= INLINE_MAX:
        return c[1:1 + c[0]].copy().view(dtype)
    off, ln = int(c.view(np.uint32)[1]), int(c.view(np.uint32)[2])
    if off + ln > len(area):
        return None
    return np.asarray(area[off:off + ln], np.uint8).copy().view(dtype)


def row_distance(kind, p, q):
    """the Go value of one row: (float64 result, error) with error True where moarray.CosineSimilarity fails on a zero vector"""
    p, q = np.ascontiguousarray(p), np.ascontiguousarray(q)
    assert p.dtype == q.dtype and p.shape == q.shape
    f32 = p.dtype == np.float32
    if kind == COSSIM:
        err = np.zeros(1, np.int32)
        fn = O.go().og_moarray_cossim_f32 if f32 else O.go().og_moarray_cossim_f64
        v = fn(O.p(p), O.p(q), p.size, O.p(err))
        return float(v), bool(err[0])
    out = np.zeros(1)
    fn = O.go().og_distance_rows_f32 if f32 else O.go().og_distance_rows_f64
    fn(kind, O.p(out), O.p(p), 0, O.p(q), 0, p.size, 1, None)
    return float(out[0]), False


def matrix_distance(kind, a, b, rnulls=None):
    """one og_distance_rows call over a dense matrix (b: one row = a const operand, stride 0)"""
    out = np.zeros(a.shape[0])
    fn = O.go().og_distance_rows_f32 if a.dtype == np.float32 else O.go().og_distance_rows_f64
    fn(kind, O.p(out), O.p(a), a.shape[1], O.p(b), 0 if b.shape[0] == 1 else b.shape[1], a.shape[1], a.shape[0], O.p(rnulls))
    return out


def normalize(v):
    """og_normalize_l2 of one row; None for an empty row ("cannot normalize empty vector")"""
    v = np.ascontiguousarray(v)
    out = np.empty_like(v)
    fn = O.go().og_normalize_l2_f32 if v.dtype == np.float32 else O.go().og_normalize_l2_f64
    return None if fn(O.p(v), O.p(out), v.size) else out


def same(got, want):
    """elementwise: equal bits, or NaN on both sides (x86 and the device make different NaN payloads)"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape
    ut = np.uint32 if got.dtype == np.float32 else np.uint64
    return (got.view(ut) == want.view(ut)) | (np.isnan(got) & np.isnan(want))


# ---- the columns the edge tests run on ---------------------------------------------------------------------------------------------
def slice_elems(dtype):
    """elements of one 128-byte ring slice"""
    return 128 // np.dtype(dtype).itemsize


def ragged_lengths(dtype):
    """row lengths around the 4- and 8-element chunks and around every slice boundary up to 6 slices, then 9 to 12 slices"""
    eps = slice_elems(dtype)
    ls = [0, 1, 2, 3, 4, 5, 7, 8, 9, 12, 15, 16, 17]
    for k in range(1, 7):
        ls += [k * eps - 1, k * eps, k * eps + 1]
    return ls + [10 * eps - 1, 10 * eps + 4, 12 * eps + 11]


def slices(n, dtype, chunk):
    """whole ring slices of a row of n elements whose Go loop takes `chunk` elements at a time (nsl in godist.cuh)"""
    return (n // chunk) * chunk // slice_elems(dtype)


def _store(rng, nbytes):
    return "i" if nbytes <= INLINE_MAX and rng.random() < 0.6 else "a"


def ragged_pair(dtype, seed, nrows=96, special=False):
    """(x, q): two per-row columns whose row i has the same length on both sides, lengths from ragged_lengths shuffled so that every
    warp mixes slice counts, empty, inline and area rows; x row i sits at offset i mod 16 in its area and q row i at 5 i + 3 mod 16;
    rows 50, 81 and 90 repeat the cells of rows 7, 33 and 50.  special: some rows get special values (_specials)"""
    rng = np.random.default_rng(seed)
    it = np.dtype(dtype).itemsize
    base = ragged_lengths(dtype)
    lens = (base * (nrows // len(base) + 1))[:nrows]
    rng.shuffle(lens)
    lens[:3] = [0, 0, 3]            # an empty inline row, an empty area row and a short area row head the first warp
    xs = [rng.standard_normal(ln).astype(dtype) for ln in lens]
    qs = [rng.standard_normal(ln).astype(dtype) for ln in lens]
    sx = [_store(rng, ln * it) for ln in lens]
    sq = [_store(rng, ln * it) for ln in lens]
    sx[0] = sq[0] = "i"
    sx[1] = sq[1] = sx[2] = sq[2] = "a"
    dup = [None] * nrows
    for i, j in ((50, 7), (81, 33), (90, 50)):
        if i < nrows:
            dup[i] = j
    if special:
        _specials(xs, qs, dtype, rng)
    x = Column(xs, dtype, sx, [i % 16 for i in range(nrows)], dup)
    q = Column(qs, dtype, sq, [(5 * i + 3) % 16 for i in range(nrows)], dup)
    return x, q


def _specials(xs, qs, dtype, rng):
    """by row i mod 12: NaN, +Inf, -Inf or -0.0 at chunk-edge, slice-edge and last (tail) positions; subnormal rows; all -0.0 rows;
    exactly parallel, anti-parallel and identical rows; (float32) rows whose squares and products overflow the float32 accumulator
    (3.4e38) but not a float64 one"""
    tiny = np.finfo(dtype).smallest_subnormal
    special = (np.nan, np.inf, -np.inf, -0.0)
    eps = slice_elems(dtype)
    for i in range(len(xs)):
        n = xs[i].size
        if n == 0:
            continue
        r = i % 12
        if r < 4:
            for pos in (3, 4, 7, 8, eps - 1, eps, n - 1):
                if pos < n and rng.random() < 0.5:
                    (xs if i % 2 else qs)[i][pos] = special[r]
        elif r == 4:
            xs[i] = (rng.integers(-50, 50, n) * tiny).astype(dtype)
            qs[i] = (rng.integers(-50, 50, n) * tiny).astype(dtype)
        elif r == 5:
            xs[i][:] = -0.0
            qs[i][:] = -0.0
        elif r == 6:
            qs[i] = xs[i] * 2
        elif r == 7:
            qs[i] = xs[i] * -4
        elif r == 8:
            qs[i] = xs[i].copy()
        elif r == 9 and dtype == np.float32:
            xs[i] = (xs[i] * 3e19).astype(dtype)
            qs[i] = xs[i] * -0.5


def uniform_column(dtype, seed, n, dim, pads):
    """n rows of dim elements, row i at offset pads[i % len(pads)] mod 16 in the area"""
    rng = np.random.default_rng(seed)
    rows = [rng.standard_normal(dim).astype(dtype) for _ in range(n)]
    return Column(rows, dtype, pad=[pads[i % len(pads)] for i in range(n)])


def normalize_column(dtype, seed, nrows=160):
    """normalize_l2 input: ragged lengths >= 1, inline rows (float64 up to 2 elements), area rows at every offset mod 16, zero rows
    (one of them -0.0), rows of special values, duplicated cells"""
    rng = np.random.default_rng(seed)
    it = np.dtype(dtype).itemsize
    base = [n for n in ragged_lengths(dtype) if n > 0]
    lens = (base * (nrows // len(base) + 1))[:nrows]
    rng.shuffle(lens)
    rows = [(rng.standard_normal(ln) * rng.choice([1e-3, 1.0, 1e3])).astype(dtype) for ln in lens]
    rows[4][:] = 0
    rows[9][:] = -0.0
    tiny = np.finfo(dtype).smallest_subnormal
    rows[13] = (rng.integers(-9, 9, lens[13]) * tiny).astype(dtype)
    rows[13][0] = tiny
    rows[17][-1] = np.inf
    rows[21][0] = np.nan
    store = [_store(rng, ln * it) for ln in lens]
    dup = [None] * nrows
    for i, j in ((40, 3), (41, 3), (100, 60), (150, 140)):
        if i < nrows:
            dup[i] = j
    return Column(rows, dtype, store, [(3 * i + 1) % 16 for i in range(nrows)], dup)
