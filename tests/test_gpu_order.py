"""MO_XCALL_ORDER_SELS on the GPU: ORDER BY and ORDER BY ... LIMIT as sels.  The order is total (ties by row id, then row index), so
every result is compared exactly with the host restatement (order_reference.order_lexsort, itself checked against the compare.New
comparator in test_oracle_order.py); Top results equal the first `limit` rows of the order; merged shard results equal the whole-table
call; the restated reference Top operator agrees on the output key sequence."""
import time

import numpy as np
import pytest

import golden_tables as G
import order_reference as R
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, bitmap_to_bools, xcall

pytestmark = pytest.mark.gpu

FLAGS = [0, R.DESC, R.NULLS_FIRST, R.NULLS_LAST, R.DESC | R.NULLS_FIRST, R.DESC | R.NULLS_LAST]
I64, U64 = np.iinfo(np.int64), np.iinfo(np.uint64)


def _col(T, rng, n):
    """n values of type T with the edge values of the type mixed in"""
    if T in (capi.T_FLOAT32, capi.T_FLOAT64):
        dt = np.float32 if T == capi.T_FLOAT32 else np.float64
        fi = np.finfo(dt)
        edge = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, fi.tiny / 4, -fi.tiny / 4, fi.tiny, fi.max, -fi.max, 1.0, -1.0], dtype=dt)
        c = (rng.standard_normal(n) * 10).astype(dt)
        m = rng.random(n) < 0.3
        c[m] = rng.choice(edge, int(m.sum()))
        return c
    if T == capi.T_DECIMAL128:
        big = [0, 1, -1, (1 << 64) - 1, 1 << 64, (1 << 64) + 1, -(1 << 64), -(1 << 64) - 1, -(1 << 64) + 1, (1 << 127) - 1, -(1 << 127)]
        vals = [int(x) for x in rng.integers(-10**6, 10**6, n)]
        for i in np.flatnonzero(rng.random(n) < 0.4):
            vals[i] = big[rng.integers(0, len(big))] + int(rng.integers(-2, 3)) * int(i % 2)
        vals = [max(min(v, (1 << 127) - 1), -(1 << 127)) for v in vals]
        out = np.zeros((n, 2), dtype=np.uint64)
        out[:, 0] = [v & (U64.max) for v in vals]
        out[:, 1] = [(v >> 64) & U64.max for v in vals]
        return out
    dt = np.dtype(capi.NP_OF_T.get(T, np.int64))
    if T == capi.T_BOOL:
        return rng.integers(0, 2, n).astype(np.uint8)
    info = np.iinfo(dt)
    c = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
    small = rng.random(n) < 0.3
    c[small] = rng.integers(-3 if info.min < 0 else 0, 3, int(small.sum())).astype(dt)
    m = rng.random(n) < 0.1
    c[m] = rng.choice(np.array([info.min, info.max, 0], dtype=dt), int(m.sum()))
    return c


ALL_TYPES = [capi.T_BOOL, capi.T_INT8, capi.T_INT16, capi.T_INT32, capi.T_INT64, capi.T_UINT8, capi.T_UINT16, capi.T_UINT32, capi.T_UINT64,
             capi.T_FLOAT32, capi.T_FLOAT64, capi.T_DATE, capi.T_TIME, capi.T_DATETIME, capi.T_TIMESTAMP, capi.T_DECIMAL64, capi.T_DECIMAL128]


def _order(cols, masks, flags, types, n, limit=None, row_ids=None):
    nulls = [bitmap_from_bools(m) if m is not None else None for m in masks]
    return ops.order_sels(cols, nulls, flags, limit=limit, row_ids=row_ids, types=types, length=n)


@pytest.mark.parametrize("T", ALL_TYPES)
@pytest.mark.parametrize("flag", FLAGS)
@pytest.mark.parametrize("nullable", [False, True])
def test_every_key_type(gpu, T, flag, nullable):
    n = 5000
    rng = np.random.default_rng(T * 100 + flag * 2 + nullable)
    c = _col(T, rng, n)
    m = (rng.random(n) < 0.15) if nullable else None
    got = _order([c], [m], [flag], [T], n)
    assert (got == R.order_lexsort([c], [m], [flag], n)).all()


@pytest.mark.parametrize("T", [capi.T_INT32, capi.T_FLOAT64, capi.T_DECIMAL128])
@pytest.mark.parametrize("flag", FLAGS)
def test_all_null_constant_and_const_keys(gpu, T, flag):
    """every digit skipped: an all-NULL column, a constant column, 1-element const keys (NULL and not); the order is then by row"""
    n = 4097
    rng = np.random.default_rng(T + flag)
    c = _col(T, rng, n)
    const = np.repeat(c[:1], n, axis=0)
    assert (_order([c], [np.ones(n, bool)], [flag], [T], n) == np.arange(n)).all()
    assert (_order([const], [None], [flag], [T], n) == np.arange(n)).all()
    assert (_order([c[:1]], [None], [flag], [T], n) == np.arange(n)).all()
    assert (_order([c[:1]], [np.ones(1, bool)], [flag], [T], n) == np.arange(n)).all()
    second = rng.integers(0, 50, n).astype(np.int64)
    for first, fm in ((c[:1], None), (c[:1], np.ones(1, bool)), (const, None)):
        got = _order([first, second], [fm, None], [flag, 0], [T, capi.T_INT64], n)
        assert (got == R.order_lexsort([second], [None], [0], n)).all()


@pytest.mark.parametrize("nkeys", [2, 3, 5, 8])
@pytest.mark.parametrize("rids", ["none", "shuffled", "duplicates"])
def test_multi_key_and_row_ids(gpu, nkeys, rids):
    n = 30_000
    rng = np.random.default_rng(nkeys * 10 + len(rids))
    types = [ALL_TYPES[(3 * k + nkeys) % len(ALL_TYPES)] for k in range(nkeys)]
    cols = [_col(T, rng, n) for T in types]
    for k, T in enumerate(types):   # few distinct values, so the later keys and the row ids decide
        if T != capi.T_DECIMAL128:
            cols[k] = cols[k][rng.integers(0, 4, n)]
    masks = [(rng.random(n) < 0.2) if k % 2 else None for k in range(nkeys)]
    flags = [FLAGS[(k * 5 + nkeys) % 6] for k in range(nkeys)]
    row_ids = None if rids == "none" else (rng.permutation(n).astype(np.int64) * 3 - 7 if rids == "shuffled" else rng.integers(0, n // 10, n).astype(np.int64))
    got = _order(cols, masks, flags, types, n, row_ids=row_ids)
    assert (got == R.order_lexsort(cols, masks, flags, n, row_ids=row_ids)).all()
    if n <= 30_000 and rids != "none":
        assert (got[:3000] == R.order_reference(cols, masks, flags, n, row_ids=row_ids)[:3000]).all()


@pytest.mark.parametrize("n", [0, 1, 2, 4095, 4096, 4097, 2 ** 20 + 3])
def test_sizes(gpu, n):
    rng = np.random.default_rng(n)
    c = rng.integers(-1000, 1000, n).astype(np.int64)
    m = rng.random(n) < 0.05
    f = rng.standard_normal(n)
    for cols, masks, flags, types in (([c], [None], [0], [capi.T_INT64]), ([f, c], [m, None], [R.DESC, 0], [capi.T_FLOAT64, capi.T_INT64])):
        got = _order(cols, masks, flags, types, n)
        assert got.shape == (n,) and (got == R.order_lexsort(cols, masks, flags, n)).all()


def test_fifty_million_rows(gpu):
    n = 50_000_000
    rng = np.random.default_rng(50)
    c = rng.integers(I64.min, I64.max, n, dtype=np.int64)
    got = _order([c], [None], [0], [capi.T_INT64], n)
    assert (got == np.argsort(c, kind="stable")).all()
    top = _order([c], [None], [R.DESC], [capi.T_INT64], n, limit=1000)
    assert (top == np.argsort(~(c.view(np.uint64) ^ np.uint64(1 << 63)), kind="stable")[:1000]).all()   # DESC = ascending NOT of the image


@pytest.mark.parametrize("case", ["uniform", "ties", "constant_first"])
def test_top_equals_prefix_of_order(gpu, case):
    n = 2 ** 20 + 3
    rng = np.random.default_rng(len(case))
    if case == "uniform":
        cols, types = [rng.standard_normal(n), rng.integers(0, 10, n).astype(np.int32)], [capi.T_FLOAT64, capi.T_INT32]
    elif case == "ties":           # 10^6 rows tied at the boundary
        k = rng.integers(0, 1000, n).astype(np.int64)
        k[rng.permutation(n)[:1_000_000]] = 500
        cols, types = [k, rng.integers(0, 3, n).astype(np.int8)], [capi.T_INT64, capi.T_INT8]
    else:
        cols, types = [np.full(n, 7, np.int64), rng.integers(-10**9, 10**9, n).astype(np.int64)], [capi.T_INT64, capi.T_INT64]
    masks = [rng.random(n) < 0.01, None]
    flags = [R.NULLS_LAST, R.DESC]
    full = _order(cols, masks, flags, types, n)
    assert (full == R.order_lexsort(cols, masks, flags, n)).all()
    for limit in (0, 1, 10, 10_000, n - 1, n, n + 5):
        got = _order(cols, masks, flags, types, n, limit=limit)
        assert (got == full[:limit]).all(), limit


def _shard_merge(cols, masks, flags, types, n, limit, bounds):
    """per block range: the range's sels, SHUFFLE of its keys and nulls, global row ids base + sels; then one call over the concatenation"""
    kcols, kmasks, rids = [[] for _ in cols], [[] for _ in cols], []
    for r0, r1 in bounds:
        s = _order([c[r0:r1] for c in cols], [m[r0:r1] if m is not None else None for m in masks], flags, types, r1 - r0, limit=limit)
        for k, (c, m) in enumerate(zip(cols, masks)):
            part = c[r0:r1]
            if part.ndim == 2:
                kcols[k].append(ops.shuffle(np.ascontiguousarray(part).view(np.dtype((np.void, 16))).reshape(-1), s).view(np.uint64).reshape(-1, 2))
                kmasks[k].append(None if m is None else m[r0:r1][s])
            elif m is None:
                kcols[k].append(ops.shuffle(part, s))
                kmasks[k].append(None)
            else:
                d, dn = ops.shuffle(part, s, src_nulls=bitmap_from_bools(m[r0:r1]), want_nulls=True)
                kcols[k].append(d)
                kmasks[k].append(bitmap_to_bools(dn, len(s)))
        rids.append(r0 + s)
    mc = [np.concatenate(p) for p in kcols]
    mm = [None if m is None else np.concatenate(p) for m, p in zip(masks, kmasks)]
    rid = np.concatenate(rids)
    sel = _order(mc, mm, flags, types, len(rid), limit=limit, row_ids=rid)
    return rid[sel]


@pytest.mark.parametrize("limit", [None, 100, 5000])
def test_merge_of_block_ranges_equals_whole_table(gpu, limit):
    n = 200_000
    rng = np.random.default_rng(3 if limit is None else limit)
    cols = [rng.integers(0, 50, n).astype(np.int32), rng.standard_normal(n).round(1), _col(capi.T_DECIMAL128, rng, n)]
    types = [capi.T_DATE, capi.T_FLOAT64, capi.T_DECIMAL128]
    masks = [rng.random(n) < 0.1, None, rng.random(n) < 0.05]
    flags = [R.DESC, R.NULLS_FIRST, 0]
    whole = _order(cols, masks, flags, types, n, limit=limit)
    bounds = [(0, 70_000), (70_000, 70_001), (70_001, 150_000), (150_000, n)]
    assert (_shard_merge(cols, masks, flags, types, n, limit, bounds) == whole).all()


def test_streaming_top_over_8192_row_batches(gpu):
    """top.go's per-batch Call: the rows kept so far plus the next batch, with their row ids, in one call"""
    n, limit = 100_000, 777
    rng = np.random.default_rng(8192)
    c = rng.integers(0, 300, n).astype(np.int16)
    f = rng.random(n).astype(np.float32)
    m = rng.random(n) < 0.1
    flags, types = [R.DESC, 0], [capi.T_INT16, capi.T_FLOAT32]
    keep_c, keep_f, keep_m, keep_rid = c[:0], f[:0], m[:0], np.zeros(0, np.int64)
    for b0 in range(0, n, 8192):
        b1 = min(n, b0 + 8192)
        cc, ff, mm = np.concatenate([keep_c, c[b0:b1]]), np.concatenate([keep_f, f[b0:b1]]), np.concatenate([keep_m, m[b0:b1]])
        rid = np.concatenate([keep_rid, np.arange(b0, b1)])
        s = _order([cc, ff], [mm, None], flags, types, len(rid), limit=limit, row_ids=rid)
        keep_c, keep_f, keep_m, keep_rid = cc[s], ff[s], mm[s], rid[s]
    assert (keep_rid == _order([c, f], [m, None], flags, types, n, limit=limit)).all()


def test_order_then_shuffle_payload(gpu):
    n = 100_000
    rng = np.random.default_rng(9)
    key = rng.integers(0, 1000, n).astype(np.int64)
    km = rng.random(n) < 0.1
    pay = rng.standard_normal(n)
    pm = rng.random(n) < 0.2
    s = _order([key], [km], [R.DESC | R.NULLS_LAST], [capi.T_INT64], n)
    d, dn = ops.shuffle(pay, s, src_nulls=bitmap_from_bools(pm), want_nulls=True)
    want = R.order_lexsort([key], [km], [R.DESC | R.NULLS_LAST], n)
    assert (d == pay[want]).all() and (bitmap_to_bools(dn, n) == pm[want]).all()


def test_lineitem_fixture(gpu):
    """ORDER BY l_returnflag, l_linestatus, l_shipdate DESC, l_extendedprice and LIMIT 100 over the reference's 6005-row lineitem"""
    cols, ints, _ = G.tpch_fixture()
    n = len(cols["shipdate"])
    keys = [cols["returnflag"], cols["linestatus"], cols["shipdate"], ints["extendedprice_cents"]]
    types = [capi.T_UINT8, capi.T_UINT8, capi.T_DATE, capi.T_DECIMAL64]
    flags = [0, 0, R.DESC, 0]
    s = _order(keys, [None] * 4, flags, types, n)
    want = R.order_reference(keys, [None] * 4, flags, n)
    assert (s == want).all()
    assert (ops.shuffle(cols["quantity"], s) == cols["quantity"][want]).all()
    assert (_order(keys, [None] * 4, flags, types, n, limit=100) == want[:100]).all()


@pytest.mark.parametrize("limit", [1, 50, 20_000])
def test_against_reference_top_operator(gpu, limit):
    n = 20_000
    rng = np.random.default_rng(limit)
    cols = [rng.integers(0, 20, n).astype(np.int64), rng.integers(0, 5, n).astype(np.float64) / 4, rng.integers(0, 9, n).astype(np.uint16)]
    masks = [rng.random(n) < 0.1, None, rng.random(n) < 0.3]
    flags = [0, R.DESC, R.DESC | R.NULLS_FIRST]
    keys = R.key_tuples(cols, masks, n)
    s = _order(cols, masks, flags, [capi.T_INT64, capi.T_FLOAT64, capi.T_UINT16], n, limit=limit)
    top = R.top_reference(keys, list(range(n)), flags, limit)
    assert [keys[i] for i in s] == [k for k, _ in top]


def test_host_and_device_forms_agree_and_device_form_only_enqueues(gpu):
    n = 4_000_000
    rng = np.random.default_rng(11)
    a = rng.integers(0, 1 << 20, n).astype(np.int64)
    b = rng.standard_normal(n)
    m = rng.random(n) < 0.1
    flags, types = [R.NULLS_FIRST, R.DESC], [capi.T_INT64, capi.T_FLOAT64]
    host = _order([a, b], [m, None], flags, types, n)
    da, db, dm = DeviceBuffer.from_numpy(a), DeviceBuffer.from_numpy(b), DeviceBuffer.from_numpy(bitmap_from_bools(m))
    out = DeviceBuffer(8 * n)
    lib = capi.load_library()
    for limit in (None, 1000):
        nout = n if limit is None else limit
        ops.order_sels_device([da, db], [dm, None], types, flags, n, out.ptr, limit=limit)
        lib.MoB200_Sync()
        assert (out.to_numpy(np.int64, nout) == host[:nout]).all()
    enq, synced = [], []
    for _ in range(3):
        t0 = time.perf_counter()
        ops.order_sels_device([da, db], [dm, None], types, flags, n, out.ptr)
        enq.append(time.perf_counter() - t0)
        lib.MoB200_Sync()
        synced.append(time.perf_counter() - t0)
    assert min(enq) < 0.5 * min(synced), (enq, synced)
    for x in (da, db, dm, out):
        x.free()


def test_malformed_arguments(gpu):
    n = 100
    c = np.arange(n, dtype=np.int64)
    sels = np.zeros(n, np.int64)

    def call(params, cols, sels_buf=sels, length=n):
        vecs = [Vector(data=sels_buf, length=len(sels_buf)), ops._params_vec(params)] + cols
        return xcall(capi.XCALL_ORDER_SELS, vecs, length, raise_on_error=False)

    def params(types, flags=None, limit=-1, rid=0):
        return ops._order_params(types, flags or [0] * len(types), limit, rid)

    good = Vector(data=c, length=n)
    assert call(params([capi.T_INT64]), [good])[0] == 0 and (sels == np.arange(n)).all()
    cases = {
        "no keys": (params([]), [good]),
        "nine keys": (params([capi.T_INT64] * 9), [good] * 9),
        "varchar key": (params([61]), [good]),
        "decimal256 key": (params([34]), [good]),
        "short key column": (params([capi.T_INT64]), [Vector(data=c[:50], length=50)]),
        "short row ids": (params([capi.T_INT64], rid=1), [good, Vector(data=c[:10], length=10)]),
    }
    for name, (p, cols) in cases.items():
        rc, msg = call(p, cols)
        assert rc == capi.RC_INVALID_ARGUMENT and msg, name
    assert call(params([capi.T_INT64]), [good], sels_buf=np.zeros(10, np.int64))[0] == capi.RC_INVALID_ARGUMENT
    assert call(params([capi.T_INT64], limit=10), [good], sels_buf=np.zeros(10, np.int64))[0] == 0
    assert call(params([capi.T_INT64]), [good], length=1 << 32)[0] == capi.RC_INVALID_ARGUMENT
    short = np.zeros(4, np.uint8)
    assert xcall(capi.XCALL_ORDER_SELS, [Vector(data=sels, length=n), Vector(data=short, length=1, const=True), good], n, raise_on_error=False)[0] == capi.RC_INVALID_ARGUMENT
