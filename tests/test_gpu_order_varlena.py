"""MO_XCALL_ORDER_SELS over string keys (CHAR, VARCHAR, TEXT, BLOB ...: 24-byte cells + area) and the small fixed-width types BIT, YEAR,
ENUM and UUID.  Values compare as Go's bytes.Compare; the order is total (ties by row id, then row index), so every result is compared
exactly with the host restatement (order_varlena_reference: Python's bytes < is bytes.Compare), and the reference's own .result orders of the TPC-H
queries that end in a string ORDER BY must come out of the device."""
import numpy as np
import pytest

import golden_tables as G
import order_varlena_reference as R
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, bitmap_to_bools, varlena_bytes_column, varlena_char1_column, xcall

pytestmark = pytest.mark.gpu

FLAGS = [0, R.DESC, R.NULLS_FIRST, R.NULLS_LAST, R.DESC | R.NULLS_FIRST, R.DESC | R.NULLS_LAST]
VARLENA = [capi.T_CHAR, capi.T_VARCHAR, capi.T_BINARY, capi.T_VARBINARY, capi.T_BLOB, capi.T_TEXT, capi.T_DATALINK]


def _order(cols, masks, flags, types, n, limit=None, row_ids=None):
    nulls = [bitmap_from_bools(m) if m is not None else None for m in masks]
    return ops.order_sels(cols, nulls, flags, limit=limit, row_ids=row_ids, types=types, length=n)


def _want(cols, masks, flags, n, limit=None, row_ids=None):
    w = R.order_lexsort(cols, masks, flags, n, row_ids=row_ids)
    return w if limit is None or limit < 0 else w[:limit]


def _values(rng, n, lengths, alphabet=b"ab\x00\xff", prefix=b""):
    """n values with lengths drawn from `lengths` over a small alphabet (many equal values and prefixes of each other)"""
    al = np.frombuffer(alphabet, np.uint8)
    ls = rng.choice(np.asarray(lengths), n)
    return [prefix + al[rng.integers(0, len(al), int(k))].tobytes() for k in ls]


def _lengths_around_words():
    return sorted(set(list(range(0, 41)) + [63, 64, 65] + [8 * k + d for k in range(1, 9) for d in (-1, 0, 1)]))


@pytest.mark.parametrize("flag", FLAGS)
@pytest.mark.parametrize("nullable", [False, True])
def test_lengths_and_flags(gpu, flag, nullable):
    n = 20_000
    rng = np.random.default_rng(flag * 2 + nullable)
    v = _values(rng, n, _lengths_around_words())
    m = (rng.random(n) < 0.15) if nullable else None
    assert (_order([v], [m], [flag], [capi.T_VARCHAR], n) == _want([v], [m], [flag], n)).all()


@pytest.mark.parametrize("T", VARLENA)
def test_every_varlena_type(gpu, T):
    n = 3000
    rng = np.random.default_rng(T)
    v = _values(rng, n, [0, 1, 5, 22, 23, 24, 25, 40], alphabet=bytes(range(256)))
    assert (_order([v], [None], [0], [T], n) == _want([v], [None], [0], n)).all()


@pytest.mark.parametrize("L", [1000, 65_535])
@pytest.mark.parametrize("flag", [0, R.DESC])
def test_long_values(gpu, L, flag):
    """long values: 1000 equal bytes then one differing byte, prefixes of each other, and the longest supported value"""
    rng = np.random.default_rng(L + flag)
    base = bytes(rng.integers(0, 256, L - 1, dtype=np.uint8))
    v = [base + bytes([b]) for b in (0, 1, 255, 7, 0)] + [base, base[:-1], base[:500], b""]
    v += [base[:k] + b"\xff" for k in (0, 10, 998)]
    v *= 3
    n = len(v)
    assert (_order([v], [None], [flag], [capi.T_TEXT], n) == _want([v], [None], [flag], n)).all()


def test_prefixes_and_embedded_bytes(gpu):
    v = [b"a", b"", b"a\x00", b"a\x01", b"a\xff", b"\xff", b"\x00", b"\x00\x00", b"b", b"a\x00\x00", b"\xff\xff", b"ab", b"a"]
    v += [b"x" * 1000 + b"\x00", b"x" * 1000 + b"\x01", b"x" * 1000, b"x" * 999 + b"\xff", b"x" * 1001]
    n = len(v)
    for flag in FLAGS:
        got = _order([v], [None], [flag], [capi.T_VARBINARY], n)
        assert (got == _want([v], [None], [flag], n)).all()
    assert [v[i] for i in _order([v], [None], [0], [capi.T_VARBINARY], n)] == sorted(v)
    for v in ([b"same value"] * 5000, [b"same value"] * 2500 + [b"same valud"] + [b"same value"] * 2500, [b""] * 100):
        n = len(v)
        assert (_order([v], [None], [0], [capi.T_VARCHAR], n) == _want([v], [None], [0], n)).all()


@pytest.mark.parametrize("flag", FLAGS)
def test_all_null_const_and_garbage_cells(gpu, flag):
    n = 5000
    rng = np.random.default_rng(flag)
    v = _values(rng, n, [3, 30, 300])
    cells, area = varlena_bytes_column(v)
    m = rng.random(n) < 0.3
    bad = cells.copy().reshape(n, 24)
    u32 = bad.view(np.uint32)
    u32[m, 0] = 0xFFFFFFFF                       # NULL rows: cells that point far outside the area are never read
    u32[m, 1] = 0xFFFFFF00
    u32[m, 2] = 0x7FFFFFFF
    got = _order([(bad.reshape(-1), area)], [m], [flag], [capi.T_VARCHAR], n)
    assert (got == _want([v], [m], [flag], n)).all()
    assert (_order([v], [np.ones(n, bool)], [flag], [capi.T_VARCHAR], n) == np.arange(n)).all()
    assert (_order([[v[0]]], [None], [flag], [capi.T_VARCHAR], n) == np.arange(n)).all()
    assert (_order([[b"x" * 40]], [np.ones(1, bool)], [flag], [capi.T_VARCHAR], n) == np.arange(n)).all()
    second = rng.integers(0, 50, n).astype(np.int64)
    for first, fm in (([v[0]], None), ([v[0]], np.ones(1, bool)), ([v[0]] * n, None)):
        got = _order([first, second], [fm, None], [flag, 0], [capi.T_VARCHAR, capi.T_INT64], n)
        assert (got == R.order_lexsort([second], [None], [0], n)).all()


@pytest.mark.parametrize("nkeys", [2, 3, 5, 8])
@pytest.mark.parametrize("rids", ["none", "shuffled", "duplicates"])
@pytest.mark.parametrize("pos", [0, 1, 2])
def test_mixed_keys_and_row_ids(gpu, nkeys, rids, pos):
    n = 30_000
    rng = np.random.default_rng(nkeys * 100 + len(rids) * 10 + pos)
    kinds = ["varlena", "int64", "decimal64", "date"]
    cols, types = [], []
    for k in range(nkeys):
        kind = kinds[(k + pos) % 4]
        if kind == "varlena":
            cols.append(_values(rng, n, [0, 1, 7, 8, 9, 23, 24, 30], alphabet=b"ab"))
            types.append([capi.T_VARCHAR, capi.T_CHAR, capi.T_TEXT][k % 3])
        elif kind == "int64":
            cols.append(rng.integers(-3, 3, n).astype(np.int64)); types.append(capi.T_INT64)
        elif kind == "decimal64":
            cols.append(rng.integers(-2, 2, n).astype(np.int64) * 10**12); types.append(capi.T_DECIMAL64)
        else:
            cols.append(rng.integers(0, 3, n).astype(np.int32)); types.append(capi.T_DATE)
    masks = [(rng.random(n) < 0.2) if k % 2 else None for k in range(nkeys)]
    flags = [FLAGS[(k * 5 + nkeys) % 6] for k in range(nkeys)]
    row_ids = None if rids == "none" else (rng.permutation(n).astype(np.int64) * 3 - 7 if rids == "shuffled" else rng.integers(0, n // 10, n).astype(np.int64))
    got = _order(cols, masks, flags, types, n, row_ids=row_ids)
    assert (got == _want(cols, masks, flags, n, row_ids=row_ids)).all()
    if rids != "none":
        assert (got[:2000] == R.order_reference(cols, masks, flags, n, row_ids=row_ids)[:2000]).all()


def _customer_cells(ids):
    """VARCHAR(25) 'Customer#%09d' names, every cell inline (18 bytes)"""
    n = len(ids)
    cells = np.zeros((n, 24), np.uint8)
    cells[:, 0] = 18
    cells[:, 1:10] = np.frombuffer(b"Customer#", np.uint8)
    digits = np.asarray(ids, np.int64)
    for j in range(9):
        cells[:, 18 - j] = 48 + digits % 10
        digits = digits // 10
    return cells.reshape(-1)


def test_ten_million_customer_names(gpu):
    n = 10_000_000
    rng = np.random.default_rng(7)
    ids = rng.permutation(n) + 1
    ids[rng.random(n) < 0.01] = 42                       # some duplicates
    cells = _customer_cells(ids)
    got = _order([(cells, None)], [None], [0], [capi.T_VARCHAR], n)
    assert (got == np.argsort(ids, kind="stable")).all()
    top = _order([(cells, None)], [None], [R.DESC], [capi.T_VARCHAR], n, limit=100)
    assert (top == np.argsort(-ids, kind="stable")[:100]).all()


@pytest.mark.parametrize("case", ["words", "skewed", "long_common_prefix"])
def test_realistic_data(gpu, case):
    n = 1_000_000
    rng = np.random.default_rng(len(case))
    if case == "words":
        syll = [b"al", b"be", b"ca", b"do", b"er", b"fi", b"go", b"ha", b"it", b"jo", b"ke", b"lu", b" ", b"x", b"qu"]
        k = rng.integers(1, 12, n)
        pick = rng.integers(0, len(syll), (n, 12))
        v = [b"".join(syll[j] for j in pick[i, :k[i]]) for i in range(n)]
    elif case == "skewed":
        pool = _values(rng, 2000, list(range(1, 60)), alphabet=b"abcdefgh")
        v = [pool[min(int(z), 1999)] for z in rng.zipf(1.3, n)]
    else:
        pre = b"P" * 37
        v = [pre + x for x in _values(rng, n, [0, 3, 8, 20], alphabet=b"xyz")]
    m = rng.random(n) < 0.05
    for flag in (0, R.DESC | R.NULLS_FIRST):
        want = _want([v], [m], [flag], n)
        assert (_order([v], [m], [flag], [capi.T_TEXT], n) == want).all()
        for limit in (1, 100, 10_000):
            assert (_order([v], [m], [flag], [capi.T_TEXT], n, limit=limit) == want[:limit]).all()


@pytest.mark.parametrize("case", ["ties_at_limit", "constant_prefix"])
def test_top(gpu, case):
    n = 2 ** 20 + 3
    rng = np.random.default_rng(len(case))
    if case == "ties_at_limit":
        v = _values(rng, n, [1, 2], alphabet=b"abc")        # 12 distinct values: ~10^5 rows tied at every boundary
    else:
        v = [b"Customer#00000" + x for x in _values(rng, n, [4], alphabet=b"0123456789")]
    second = rng.integers(0, 5, n).astype(np.int16)
    flags = [0, R.DESC]
    full = _want([v, second], [None, None], flags, n)
    assert (_order([v, second], [None, None], flags, [capi.T_CHAR, capi.T_INT16], n) == full).all()
    for limit in (0, 1, 10, 1000, 100_000, n - 1, n + 5):
        got = _order([v, second], [None, None], flags, [capi.T_CHAR, capi.T_INT16], n, limit=limit)
        assert (got == full[:limit]).all(), limit


def _shuffle_varlena(cells, nulls_mask, s):
    """SHUFFLE(24) of a varlena column: the cells (they keep pointing into the source area) and the nulls"""
    c24 = np.ascontiguousarray(cells).view(np.dtype((np.void, 24)))
    if nulls_mask is None:
        return ops.shuffle(c24, s).view(np.uint8).reshape(-1), None
    d, dn = ops.shuffle(c24, s, src_nulls=bitmap_from_bools(nulls_mask), want_nulls=True)
    return d.view(np.uint8).reshape(-1), bitmap_to_bools(dn, len(s))


def _union(parts):
    """Vector.UnionBatch of varlena columns: cells concatenated, non-inline offsets rebased into the concatenated areas"""
    cells, areas, base = [], [], 0
    for c, a in parts:
        c = c.reshape(-1, 24).copy()
        big = c[:, 0] > 23
        c.view(np.uint32)[big, 1] += np.uint32(base)
        cells.append(c.reshape(-1))
        areas.append(a)
        base += len(a)
    return np.concatenate(cells), np.concatenate(areas)


@pytest.mark.parametrize("limit", [None, 100, 5000])
def test_merge_of_shards_equals_whole_table(gpu, limit):
    n = 200_000
    rng = np.random.default_rng(5 if limit is None else limit)
    v = _values(rng, n, [2, 10, 23, 24, 40, 70], alphabet=b"abcd")
    d = rng.integers(0, 30, n).astype(np.int32)
    mv, md = rng.random(n) < 0.1, rng.random(n) < 0.05
    flags, types = [R.DESC | R.NULLS_LAST, 0], [capi.T_VARCHAR, capi.T_DATE]
    whole = _order([v, d], [mv, md], flags, types, n, limit=limit)
    assert (whole == _want([v, d], [mv, md], flags, n, limit=limit)).all()
    parts, pm, pd, pdm, rids = [], [], [], [], []
    for r0, r1 in [(0, 70_000), (70_000, 70_001), (70_001, 150_000), (150_000, n)]:
        cells, area = varlena_bytes_column(v[r0:r1])
        s = _order([(cells, area), d[r0:r1]], [mv[r0:r1], md[r0:r1]], flags, types, r1 - r0, limit=limit)
        sc, sm = _shuffle_varlena(cells, mv[r0:r1], s)
        parts.append((sc, area)); pm.append(sm)
        dd, ddn = ops.shuffle(d[r0:r1], s, src_nulls=bitmap_from_bools(md[r0:r1]), want_nulls=True)
        pd.append(dd); pdm.append(bitmap_to_bools(ddn, len(s)))
        rids.append(r0 + s)
    rid = np.concatenate(rids)
    sel = _order([_union(parts), np.concatenate(pd)], [np.concatenate(pm), np.concatenate(pdm)], flags, types, len(rid), limit=limit, row_ids=rid)
    assert (rid[sel] == whole).all()


def test_streaming_top_over_8192_row_batches(gpu):
    n, limit = 100_000, 777
    rng = np.random.default_rng(8192)
    v = _values(rng, n, [5, 30], alphabet=b"abc")
    m = rng.random(n) < 0.1
    keep_cells, keep_area, keep_m, keep_rid = np.zeros(0, np.uint8), np.zeros(0, np.uint8), m[:0], np.zeros(0, np.int64)
    for b0 in range(0, n, 8192):
        b1 = min(n, b0 + 8192)
        cells, area = _union([(keep_cells, keep_area), varlena_bytes_column(v[b0:b1])])
        mm = np.concatenate([keep_m, m[b0:b1]])
        rid = np.concatenate([keep_rid, np.arange(b0, b1)])
        s = _order([(cells, area)], [mm], [R.DESC], [capi.T_VARCHAR], len(rid), limit=limit, row_ids=rid)
        keep_cells, _ = _shuffle_varlena(cells, None, s)
        keep_area, keep_m, keep_rid = area, mm[s], rid[s]
    assert (keep_rid == _want([v], [m], [R.DESC], n, limit=limit)).all()


def test_order_then_shuffle_varlena_payload(gpu):
    n = 100_000
    rng = np.random.default_rng(9)
    key = _values(rng, n, [1, 3, 30], alphabet=b"ab")
    pay = _values(rng, n, [0, 5, 23, 24, 100])
    pm = rng.random(n) < 0.2
    s = _order([key], [None], [R.DESC], [capi.T_VARCHAR], n)
    want = _want([key], [None], [R.DESC], n)
    assert (s == want).all()
    cells, area = varlena_bytes_column(pay)
    dc, dm = _shuffle_varlena(cells, pm, s)
    assert (dm == pm[want]).all()
    c = dc.reshape(n, 24)
    for i in range(0, n, 97):
        if c[i, 0] <= 23:
            got = c[i, 1:1 + c[i, 0]].tobytes()
        else:
            off, ln = c[i].view(np.uint32)[1:3]
            got = area[off:off + ln].tobytes()
        assert got == pay[want[i]]


def test_host_and_device_forms_agree(gpu):
    n = 2_000_000
    rng = np.random.default_rng(11)
    v = _values(rng, n, [3, 12, 30, 60], alphabet=b"abcdef")
    b = rng.integers(0, 1000, n).astype(np.int64)
    m = rng.random(n) < 0.1
    flags, types = [R.NULLS_FIRST, R.DESC], [capi.T_VARCHAR, capi.T_INT64]
    cells, area = varlena_bytes_column(v)
    host = _order([(cells, area), b], [m, None], flags, types, n)
    assert (host == _want([v, b], [m, None], flags, n)).all()
    dc, da, db, dm = DeviceBuffer.from_numpy(cells), DeviceBuffer.from_numpy(area), DeviceBuffer.from_numpy(b), DeviceBuffer.from_numpy(bitmap_from_bools(m))
    out = DeviceBuffer(8 * n)
    lib = capi.load_library()
    for limit in (None, 1000):
        nout = n if limit is None else limit
        ops.order_sels_device([(dc, da), db], [dm, None], types, flags, n, out.ptr, limit=limit)
        lib.MoB200_Sync()
        assert (out.to_numpy(np.int64, nout) == host[:nout]).all()
    for x in (dc, da, db, dm, out):
        x.free()


def test_bad_cells_are_rejected_with_the_lowest_row(gpu):
    n = 100
    v = [b"%03d-" % i * 10 for i in range(n)]              # 50-byte values: every cell points into the area
    cells, area = varlena_bytes_column(v)
    sels = np.zeros(n, np.int64)

    def call(cells, area, nulls=None, T=capi.T_VARCHAR):
        vecs = [Vector(data=sels, length=n), ops._params_vec(ops._order_params([T], [0], -1, False)),
                Vector(data=cells, area=area, nulls=nulls, length=n)]
        return xcall(capi.XCALL_ORDER_SELS, vecs, n, raise_on_error=False)

    assert call(cells, area)[0] == 0 and (sels == _want([v], [None], [0], n)).all()
    c = cells.reshape(n, 24).copy()
    c.view(np.uint32)[40, 1] = len(area)                  # offset past the area
    c.view(np.uint32)[17, 2] = 51                          # length past the area (the last value) -- lower row
    c.view(np.uint32)[17, 1] = len(area) - 50
    rc, msg = call(c.reshape(-1), area)
    assert rc == capi.RC_INVALID_ARGUMENT and "key 0 row 17" in msg, msg
    nulls = bitmap_from_bools(np.arange(n) == 17)
    rc, msg = call(c.reshape(-1), area, nulls=nulls)
    assert rc == capi.RC_INVALID_ARGUMENT and "key 0 row 40" in msg, msg
    rc, msg = call(cells, None)                            # non-inline cells without an area
    assert rc == capi.RC_INVALID_ARGUMENT and "key 0 row 0" in msg, msg
    big, barea = varlena_bytes_column([b"x" * (capi.ORDER_MAX_VARLENA + 1)] + v[1:])
    rc, msg = call(big, barea)
    assert rc == capi.RC_INVALID_ARGUMENT and msg
    rc, _ = call(cells[:24 * 50], area)                    # short cells
    assert rc == capi.RC_INVALID_ARGUMENT
    # the cell rule's edges: a value that ends at the area's end is good, one whose end wraps 32 bits is not
    e = cells.reshape(n, 24).copy()
    e.view(np.uint32)[17, 1], e.view(np.uint32)[17, 2] = len(area) - len(v[-1]), len(v[-1])
    assert call(e.reshape(-1), area)[0] == 0 and (sels == _want([v[:17] + [v[-1]] + v[18:]], [None], [0], n)).all()
    e.view(np.uint32)[5, 1], e.view(np.uint32)[5, 2] = 0xFFFFFFF0, 0x20
    rc, msg = call(e.reshape(-1), area)
    assert rc == capi.RC_INVALID_ARGUMENT and "key 0 row 5" in msg, msg
    # device cells 8-byte but not 16-byte aligned, and 1-byte misaligned
    for off in (8, 1):
        buf = DeviceBuffer(c.nbytes + 16)
        dv = buf.view(c.nbytes, off)
        capi.check(buf.lib.MoB200_Upload(dv.ptr, c.ctypes.data, c.nbytes), buf.lib)
        vecs = [Vector(data=sels, length=n), ops._params_vec(ops._order_params([capi.T_VARCHAR], [0], -1, False)),
                Vector(data_ptr=dv.ptr, data_nbytes=c.nbytes, area=area, length=n)]
        rc, msg = xcall(capi.XCALL_ORDER_SELS, vecs, n, raise_on_error=False)
        assert rc == capi.RC_INVALID_ARGUMENT and "key 0 row 17" in msg, (off, msg)
        capi.check(buf.lib.MoB200_Upload(dv.ptr, cells.ctypes.data, cells.nbytes), buf.lib)
        assert xcall(capi.XCALL_ORDER_SELS, vecs, n, raise_on_error=False)[0] == 0 and (sels == _want([v], [None], [0], n)).all()
        buf.free()
    # one cell: a const key at len 2, a one-row column at len 1 -- both read cell 0
    for m in (1, 2):
        out = np.full(m, -1, np.int64)
        for cell, rc_want in ((cells[:24], 0), (c.reshape(-1)[17 * 24:18 * 24], capi.RC_INVALID_ARGUMENT)):
            vecs = [Vector(data=out, length=m), ops._params_vec(ops._order_params([capi.T_VARCHAR], [0], -1, False)),
                    Vector(data=cell.copy(), area=area, length=m)]
            rc, msg = xcall(capi.XCALL_ORDER_SELS, vecs, m, raise_on_error=False)
            assert rc == rc_want and (rc == 0 or "key 0 row 0" in msg), (m, msg)
            assert rc or list(out) == list(range(m))


@pytest.mark.parametrize("T", [capi.T_BIT, capi.T_YEAR, capi.T_ENUM, capi.T_UUID])
@pytest.mark.parametrize("flag", FLAGS)
def test_small_fixed_width_types(gpu, T, flag):
    n = 5000
    rng = np.random.default_rng(T * 10 + flag)
    m = rng.random(n) < 0.15
    if T == capi.T_UUID:                                   # CompareUuid: the 16 bytes byte by byte
        u = rng.integers(0, 3, (n, 16)).astype(np.uint8)
        u[rng.random(n) < 0.3] = rng.integers(0, 256, 16, dtype=np.uint8)
        u[:, 8:] = rng.integers(0, 256, (n, 8), dtype=np.uint8) * (rng.random((n, 1)) < 0.5)
        got = _order([u], [m], [flag], [T], n)
        ref = [bytes(r) for r in u]
        assert (got == _want([ref], [m], [flag], n)).all()
        return
    if T == capi.T_BIT:
        c = rng.integers(0, np.iinfo(np.uint64).max, n, dtype=np.uint64, endpoint=True)
        c[rng.random(n) < 0.3] = 5
    elif T == capi.T_YEAR:
        c = rng.integers(-32768, 32767, n, endpoint=True).astype(np.int16)
        c[rng.random(n) < 0.5] = rng.integers(1990, 2030, 1)[0]
    else:
        c = rng.integers(0, 65535, n, endpoint=True).astype(np.uint16)
        c[rng.random(n) < 0.5] = 3
    assert (_order([c], [m], [flag], [T], n) == _want([c], [m], [flag], n)).all()


def test_fixed_width_launch_count(gpu):
    """a call with only fixed-width keys runs the sort it ran before string keys existed: per 64-bit word one histogram, one plan and
    eight scatter kernels, then the sels"""
    n = 1 << 20
    rng = np.random.default_rng(1)
    a, b = rng.integers(-100, 100, n).astype(np.int64), rng.standard_normal(n)
    lib = capi.load_library()
    c0 = lib.MoB200_KernelLaunchCount()
    got = _order([a, b], [None, None], [0, R.DESC], [capi.T_INT64, capi.T_FLOAT64], n)
    assert lib.MoB200_KernelLaunchCount() - c0 == 2 * 10 + 1
    assert (got == _want([a, b], [None, None], [0, R.DESC], n)).all()


# ---- the reference's own results ----------------------------------------------------------------------------------------------------------
_TYPE = {"CHAR(10)": capi.T_CHAR, "CHAR(25)": capi.T_CHAR, "VARCHAR(25)": capi.T_VARCHAR, "VARCHAR(1)": capi.T_VARCHAR,
         "DECIMAL(15,2)": capi.T_DECIMAL64, "INTEGER": capi.T_INT32, "BIGINT": capi.T_INT64}


@pytest.mark.parametrize("q", ["q16", "q2", "q20", "q21", "q1"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_reference_result_orders(gpu, q, seed):
    keys, flags, tnames, limit, rows = R.golden_order_query(q)
    n = len(rows)
    perm = np.random.default_rng(seed).permutation(n)
    shuffled = [[k[i] for i in perm] if isinstance(k, list) else k[perm] for k in keys]
    got = _order(shuffled, [None] * len(keys), flags, [_TYPE[t] for t in tnames], n, limit=limit)
    want = R.key_tuples(keys, [None] * len(keys), n)
    have = R.key_tuples(shuffled, [None] * len(keys), n)
    assert [have[i] for i in got] == want[:len(got)]
    if len(set(want)) == n:
        assert [rows[perm[i]] for i in got] == rows[:len(got)]


def test_q1_group_order_over_lineitem_varlena(gpu):
    """ORDER BY l_returnflag, l_linestatus over the VARCHAR(1) cells of the reference's lineitem: the groups come out in q1.result's order"""
    cols, _, _ = G.tpch_fixture()
    n = len(cols["returnflag"])
    rf, ls = varlena_char1_column(cols["returnflag"]), varlena_char1_column(cols["linestatus"])
    s = _order([(rf, None), (ls, None)], [None, None], [0, 0], [capi.T_VARCHAR, capi.T_VARCHAR], n)
    pairs = [(chr(cols["returnflag"][i]), chr(cols["linestatus"][i])) for i in s]
    groups = [p for j, p in enumerate(pairs) if j == 0 or p != pairs[j - 1]]
    assert groups == [(r[0], r[1]) for r in R.golden_order_query("q1")[4]]
    assert (s == np.lexsort((cols["linestatus"], cols["returnflag"]))).all()
