"""MO_XCALL_GO_IN / MO_XCALL_GO_NOT_IN on the device against in_reference.py (operator_in.go restated): every supported type, lists on both
sides of the shared-memory table budget, duplicates and NULL elements, column NULLs, const and const NULL columns and lists, skipped rows,
float +-0 and NaN, 16-byte values that differ only in the high word, strings inline and in the area; and, through the operand harness of
test_gpu_go_operands.py, host and device forms, launch counts, the enqueue-only form, the bitmap tail and the refusals."""
import ctypes as C

import numpy as np
import pytest

import cell_edges as E
import in_reference as R
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, bitmap_from_bools, bitmap_to_bools, varlena_bytes_column
from test_gpu_go_operands import ONE_NULL, Arg, call, rand_bits, result_nulls, words

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu


def ints(dt, lo, hi):
    return lambda rng, k: rng.integers(lo, hi, k).astype(dt)


def floats(dt):
    def make(rng, k):
        v = (rng.integers(-20, 20, k) / 4).astype(dt)
        special = np.array([0.0, -0.0, np.nan, np.inf, -np.inf], dt)
        pick = rng.random(k) < 0.2
        v[pick] = special[rng.integers(0, special.size, int(pick.sum()))]
        return v
    return make


def wide(rng, k):
    """16-byte rows: low words from a small range, high words 0 or 1, so equal low words differ only in the high word"""
    v = np.zeros((k, 2), np.uint64)
    v[:, 0] = rng.integers(0, 12, k).astype(np.uint64)
    v[:, 1] = rng.integers(0, 2, k).astype(np.uint64)
    return v


VOCAB = [b"", b"a", b"ab", b"abc", b"ab\x00", b"\x00", b"FOB", b"TRUCK", b"x" * 23, b"x" * 24, b"x" * 24 + b"y", b"pre" * 10 + b"1",
         b"pre" * 10 + b"2", b"\xe4\xb8\xad\xe6\x96\x87", b"MAIL", b"z" * 300]


def strs(rng, k):
    return [VOCAB[i] for i in rng.integers(0, len(VOCAB), k)]


FIXED = {capi.T_BOOL: ints(np.uint8, 0, 2), capi.T_INT8: ints(np.int8, -128, 128), capi.T_UINT8: ints(np.uint8, 0, 256),
         capi.T_INT16: ints(np.int16, -40, 40), capi.T_UINT16: ints(np.uint16, 65500, 65536), capi.T_YEAR: ints(np.int16, 1990, 2030),
         capi.T_INT32: ints(np.int32, -50, 50), capi.T_UINT32: ints(np.uint32, 0, 80), capi.T_DATE: ints(np.int32, 738000, 738100),
         capi.T_INT64: ints(np.int64, -3, 60), capi.T_UINT64: lambda r, k: (np.uint64(2 ** 64 - 40) + r.integers(0, 40, k).astype(np.uint64)),
         capi.T_TIME: ints(np.int64, 0, 90), capi.T_DATETIME: ints(np.int64, -5, 70), capi.T_TIMESTAMP: ints(np.int64, 10 ** 15, 10 ** 15 + 70),
         capi.T_DECIMAL64: ints(np.int64, -30, 30), capi.T_FLOAT32: floats(np.float32), capi.T_FLOAT64: floats(np.float64),
         capi.T_DECIMAL128: wide, capi.T_UUID: wide}
STRINGS = [capi.T_CHAR, capi.T_VARCHAR, capi.T_TEXT, capi.T_BLOB, capi.T_BINARY, capi.T_VARBINARY]
ALL_TYPES = list(FIXED) + STRINGS


def make(T, rng, k):
    return strs(rng, k) if T in STRINGS else FIXED[T](rng, k)


def rows_of(x):
    return list(x) if isinstance(x, list) else [x[i] for i in range(len(x))]


def check(T, col, vals, negate, cn=None, vn=None, skip=None, length=None):
    n = length if length is not None else len(col)
    got, gn = ops.go_in(T, col, vals, negate=negate, col_nulls=None if cn is None else bitmap_from_bools(cn),
                        values_nulls=None if vn is None else bitmap_from_bools(vn),
                        rnulls=None if skip is None else bitmap_from_bools(skip), length=n)
    c = rows_of(col)
    if len(c) == 1 and n > 1:                                     # a const column
        c, cn = c * n, None if cn is None else np.repeat(cn, n)
    ref, rn = R.evaluate(c, cn, rows_of(vals), vn, negate=negate, skip=skip)
    assert (gn == np.array(rn)).all()
    live = ~np.array(rn)
    assert (got[live] == np.array([ref[i] for i in np.flatnonzero(live)], bool)).all()
    return got, gn


@pytest.mark.parametrize("negate", [False, True])
@pytest.mark.parametrize("T", ALL_TYPES)
def test_every_type_against_the_reference(gpu, T, negate):
    rng = np.random.default_rng(T * 2 + negate)
    n = 1000
    for m in (0, 1, 2, 8, 300):
        col = make(T, rng, n)
        vals = make(T, rng, m)
        if m >= 2:                                                # duplicates
            vals = rows_of(vals)
            vals[-1] = vals[0]
            vals = vals if T in STRINGS else np.array(vals)
        cn = rng.random(n) < 0.1
        vn = rng.random(m) < 0.2
        skip = rng.random(n) < 0.1
        check(T, col, vals, negate, cn, vn, skip)


@pytest.mark.parametrize("T", [capi.T_INT32, capi.T_INT64, capi.T_FLOAT64, capi.T_DECIMAL128, capi.T_VARCHAR])
def test_lists_past_the_shared_memory_budget(gpu, T):
    """10^5 values: the table is read from global memory; the column also holds values outside the list"""
    rng = np.random.default_rng(T)
    m, n = 100_000, 50_000
    if T in STRINGS:
        vals = [b"v%07d" % i + (b"-long-suffix-past-inline" if i % 3 == 0 else b"") for i in range(m)]
        col = [vals[i] if i < m else b"miss%d" % i for i in rng.integers(0, 2 * m, n)]
    elif T == capi.T_DECIMAL128:
        vals = np.stack([np.arange(m, dtype=np.uint64), np.arange(m, dtype=np.uint64) % 2], axis=1)
        col = np.stack([rng.integers(0, 2 * m, n).astype(np.uint64), rng.integers(0, 2, n).astype(np.uint64)], axis=1)
    else:
        dt = {capi.T_INT32: np.int32, capi.T_INT64: np.int64, capi.T_FLOAT64: np.float64}[T]
        vals = (rng.permutation(4 * m)[:m] - 2 * m).astype(dt)
        col = rng.integers(-2 * m, 2 * m, n).astype(dt)
    for negate in (False, True):
        check(T, col, vals, negate, cn=rng.random(n) < 0.05, vn=rng.random(m) < 0.01)


@pytest.mark.parametrize("T", [capi.T_INT16, capi.T_FLOAT32, capi.T_UUID, capi.T_CHAR])
def test_const_and_const_null_columns_and_lists(gpu, T):
    rng = np.random.default_rng(5)
    n = 777
    vals = make(T, rng, 8)
    one = make(T, rng, 1)
    for negate in (False, True):
        check(T, one, vals, negate, length=n)                                        # const column
        got, gn = check(T, one, vals, negate, cn=np.array([True]), length=n)         # const NULL column: every row NULL
        assert gn.all()
        check(T, make(T, rng, n), one, negate)                                       # const list
        got, gn = check(T, make(T, rng, n), one, negate, vn=np.array([True]))        # const NULL list: the empty set
        assert (got[~gn] == negate).all()
        check(T, make(T, rng, n), vals, negate, vn=np.ones(8, bool))                 # all-NULL list
        check(T, make(T, rng, 1), vals, negate, length=1)                            # len == 1: a one-row column
        check(T, make(T, rng, 1), vals, negate, cn=np.array([True]), length=1)


def test_float_signed_zero_and_nan(gpu):
    for dt, T in ((np.float32, capi.T_FLOAT32), (np.float64, capi.T_FLOAT64)):
        col = np.array([0.0, -0.0, np.nan, 1.0, -np.nan, 2.0] * 20, dt)
        for vals in (np.array([-0.0, np.nan], dt), np.array([0.0], dt), np.array([np.nan, 1.0], dt)):
            for negate in (False, True):
                got, _ = check(T, col, vals, negate)
                nan = np.isnan(col)
                assert (got[nan] == negate).all()                                     # a NaN row is never found
                if 0.0 in vals:
                    assert (got[col == 0] != negate).all()                            # +0 and -0 are one key


def test_wide_values_differ_in_the_high_word(gpu):
    col = np.array([[5, 0], [5, 1], [5, 2 ** 63], [6, 0]], np.uint64)
    vals = np.array([[5, 1]], np.uint64)
    for T in (capi.T_DECIMAL128, capi.T_UUID):
        got, _ = check(T, np.tile(col, (50, 1)), np.repeat(vals, 3, axis=0), False)
        assert got.reshape(50, 4).tolist() == [[False, True, False, False]] * 50


def test_strings_compare_bytes(gpu):
    col = [b"", b"ab", b"ab ", b"AB", b"ab\x00", b"x" * 23, b"x" * 24, b"pre" * 10 + b"1", b"pre" * 10 + b"3"] * 11
    vals = [b"", b"ab", b"ab\x00", b"x" * 24, b"pre" * 10 + b"1", b"pre" * 10 + b"2"]
    got, _ = check(capi.T_VARCHAR, col, vals, False)
    assert got[:9].tolist() == [True, True, False, False, True, False, True, True, False]


@pytest.mark.parametrize("T,dt", [(capi.T_INT32, np.int32), (capi.T_INT64, np.int64)])
def test_ten_million_rows_device_form(gpu, T, dt):
    n = 10_000_037                                               # not a multiple of 64
    rng = np.random.default_rng(3)
    col = rng.integers(0, 1000, n).astype(dt)
    cn = rng.random(n) < 0.01
    skip = rng.random(n) < 0.01
    for m in (8, 2000):
        vals = rng.choice(1000, m // 8 if m > 1000 else m, replace=False).astype(dt)
        vals = np.resize(vals, m)
        for negate in (False, True):
            d_col, d_vals = DeviceBuffer.from_numpy(col), DeviceBuffer.from_numpy(vals)
            d_cn = DeviceBuffer.from_numpy(bitmap_from_bools(cn))
            d_out = DeviceBuffer(n)
            d_rn = DeviceBuffer.from_numpy(bitmap_from_bools(skip))
            ops.go_in_device(T, d_col, d_vals, m, n, d_out, d_rn, negate=negate, col_nulls=d_cn)
            got = d_out.to_numpy(np.uint8, n).astype(bool)
            gn = bitmap_to_bools(d_rn.to_numpy(np.uint64), n)
            for b in (d_col, d_vals, d_cn, d_out, d_rn):
                b.free()
            assert (gn == (cn | skip)).all()
            want = np.isin(col, vals) != negate
            assert (got[~gn] == want[~gn]).all()


# ---- the operand harness: host form == device form, launches, enqueue-only, the bitmap tail, refusals
N = 1000


def params(m):
    return Arg(np.array([m], np.int64))


def in_args(T, shape, m, rng):
    """shape: v column, c const, n const NULL; the list has NULL elements"""
    n = 1 if shape == "len1" else N
    if T in STRINGS:
        def data(k):
            return varlena_bytes_column(strs(rng, k))
    else:
        def data(k):
            return make(T, rng, k), None
    k = 1 if shape in ("c", "n") else n
    d, area = data(k)
    nulls = ONE_NULL if shape == "n" else (np.zeros(1, np.uint64) if shape == "c" else rand_bits(rng, n, 0.1))
    col = Arg(d, nulls, area)
    ld, larea = data(max(m, 1))
    lst = Arg(ld, rand_bits(rng, max(m, 1), 0.2), larea)
    return [Arg(np.full(n, 0x5a, np.uint8), result_nulls(rng, n)), col, lst, params(m)], n


HARNESS = [(T, shape, m) for T in (capi.T_INT32, capi.T_INT8, capi.T_FLOAT64, capi.T_DECIMAL128, capi.T_VARCHAR)
           for shape in ("v", "c", "n", "len1") for m in (0, 3, 3000)]


@pytest.mark.parametrize("T,shape,m", HARNESS)
def test_host_and_device_forms_agree(gpu, T, shape, m):
    rng = np.random.default_rng(T + m)
    args, n = in_args(T, shape, m, rng)
    for fid in (capi.XCALL_GO_IN(T), capi.XCALL_GO_NOT_IN(T)):
        rc_h, msg_h, k_h, _, host = call(gpu, fid, args, n, device=False)
        rc_d, msg_d, k_d, _, dev = call(gpu, fid, args, n, device=True)
        assert rc_h == rc_d == 0, (msg_h, msg_d)
        host_empty = m == 0 or bitmap_to_bools(args[2].slots["pnulls"].view(np.uint64), m).all()
        assert (k_h, k_d) == (1 if host_empty else 2, 2 if m else 1), (k_h, k_d)
        assert host == dev
        rn = np.frombuffer(host[(0, "pnulls")], np.uint64)
        if n & 63:
            assert rn[-1] >> np.uint64(n & 63) == 0, "bits past len are cleared"
        if shape == "n":
            assert (bitmap_to_bools(rn, n)).all()


@pytest.fixture
def stream(gpu):
    s = torch.cuda.Stream()
    capi.check(gpu.MoB200_SetStream(C.c_void_p(s.cuda_stream)), gpu)
    yield s
    capi.check(gpu.MoB200_SetStream(None), gpu)


@pytest.mark.parametrize("T", [capi.T_INT32, capi.T_UINT64, capi.T_FLOAT32, capi.T_UUID])
@pytest.mark.parametrize("shape", ["v", "n"])
def test_fixed_width_only_enqueues_on_device_operands(gpu, stream, T, shape):
    rng = np.random.default_rng(11)
    args, n = in_args(T, shape, 40, rng)
    rc, msg, _, idle, dev = call(gpu, capi.XCALL_GO_IN(T), args, n, device=True, stream=stream, host_args=(3,))
    assert rc == 0, msg
    assert not idle, "the all-device call waited for its stream"
    rc, msg, _, idle, host = call(gpu, capi.XCALL_GO_IN(T), args, n, device=False, stream=stream)
    assert rc == 0 and idle, msg
    assert host == dev


@pytest.mark.parametrize("T", [capi.T_INT64, capi.T_DECIMAL128, capi.T_VARCHAR])
def test_all_null_host_list_skips_the_build(gpu, T):
    """a host list whose elements are all NULL is the empty set without a build; a device one runs the build, which inserts nothing"""
    rng = np.random.default_rng(4)
    args, n = in_args(T, "v", 70, rng)
    args[2].slots["pnulls"] = np.full(words(70), ~np.uint64(0), np.uint64)
    for fid, negate in ((capi.XCALL_GO_IN(T), 0), (capi.XCALL_GO_NOT_IN(T), 1)):
        rc_h, msg_h, k_h, _, host = call(gpu, fid, args, n, device=False)
        rc_d, msg_d, k_d, _, dev = call(gpu, fid, args, n, device=True)
        assert rc_h == rc_d == 0 and (k_h, k_d) == (1, 2), (msg_h, msg_d, k_h, k_d)
        assert host == dev
        rn = bitmap_to_bools(np.frombuffer(host[(0, "pnulls")], np.uint64), n)
        assert (np.frombuffer(host[(0, "pdata")], np.uint8)[~rn] == negate).all()


def refused(gpu, fid, args, n, match):
    for device in (False, True):
        rc, msg, k, _, _ = call(gpu, fid, args, n, device)
        assert rc == capi.RC_INVALID_ARGUMENT and k == 0, msg
        assert match in msg, msg


@pytest.mark.parametrize("T", [capi.T_INT64, capi.T_VARCHAR])
def test_refusals(gpu, T):
    rng = np.random.default_rng(2)
    args, n = in_args(T, "v", 10, rng)
    what = "go in"
    refused(gpu, capi.XCALL_GO_IN(T), args[:3] + [params(-1)], n, what + ": nvalues -1 outside")
    refused(gpu, capi.XCALL_GO_IN(T), args[:3] + [params(2 ** 31)], n, what + ": nvalues 2147483648 outside")
    refused(gpu, capi.XCALL_GO_IN(T), args[:3] + [params(11)], n, what + ": operand 2 holds")
    refused(gpu, capi.XCALL_GO_IN(T), args[:3] + [Arg()], n, what + ": params missing")
    refused(gpu, capi.XCALL_GO_NOT_IN(T), args[:3] + [Arg()], n, "go not in: params missing")
    for bad in (capi.T_BIT, capi.T_ENUM, capi.T_DATALINK, 34):
        refused(gpu, capi.XCALL_GO_IN(bad), args, n, "go in: unsupported type %d" % bad)
    assert ops.go_in(T, make(T, rng, 0), make(T, rng, 3), length=0)[0].size == 0


def _bad(values, rows):
    cells, area = varlena_bytes_column(values)
    c = cells.reshape(-1, 24).copy()
    for r in rows:
        u32 = c[r].view(np.uint32)
        u32[0], u32[1], u32[2] = 0xFFFFFFFF, area.size, 5
    return c.reshape(-1), area


def test_bad_cells_are_named(gpu):
    n, m = 300, 50
    col = [b"y" * 30] * n
    vals = [b"x" * 30] * m
    cn = np.zeros(n, bool); cn[7] = True
    vn = np.zeros(m, bool); vn[4] = True
    for negate in (False, True):
        with pytest.raises(capi.MoError, match="go %sin: operand 1 row 19" % ("not " if negate else "")):
            ops.go_in(capi.T_VARCHAR, _bad(col, [7, 19, 200]), vals, negate, col_nulls=bitmap_from_bools(cn))
        with pytest.raises(capi.MoError, match="operand 2 row 9"):
            ops.go_in(capi.T_TEXT, col, _bad(vals, [4, 9, 30]), negate, values_nulls=bitmap_from_bools(vn))
    skip = np.zeros(n, bool); skip[[7, 19, 200]] = True                    # skipped rows are not read
    got, gn = ops.go_in(capi.T_VARCHAR, _bad(col, [7, 19, 200]), vals, rnulls=bitmap_from_bools(skip))
    assert (gn == skip).all() and not got[~skip].any()
    # device column cells 8-byte but not 16-byte aligned (three 8-byte loads) and 1-byte misaligned (byte loads); a value that ends at the
    # area's end is good, one a byte past it or whose end wraps 32 bits is not
    col = [b"%03d" % (i % 70) * 10 for i in range(n)]
    vals = [b"%03d" % i * 10 for i in range(0, 100, 2)]
    want, _ = ops.go_in(capi.T_VARCHAR, col, vals)
    want[5] = want[-1]
    cells, area = E.edges(col, 5, None, None)
    lc, la = varlena_bytes_column(vals)
    dlc, dla, darea = DeviceBuffer.from_numpy(lc), DeviceBuffer.from_numpy(la), DeviceBuffer.from_numpy(area)
    for shift in E.SHIFTS:
        for c, bad_row in ((cells, None), (E.edges(col, 5, 19, 40)[0], 19), (E.edges(col, 5, None, 23)[0], 23)):
            owner, dc = E.on_device(c, shift)
            out, outn = DeviceBuffer(n), DeviceBuffer.from_numpy(np.zeros((n + 63) // 64, np.uint64))
            if bad_row is None:
                ops.go_in_device(capi.T_VARCHAR, (dc, darea), (dlc, dla), m, n, out, outn)
                assert (out.to_numpy(np.uint8).astype(bool) == want).all(), shift
            else:
                with pytest.raises(capi.MoError, match="operand 1 row %d" % bad_row):
                    ops.go_in_device(capi.T_VARCHAR, (dc, darea), (dlc, dla), m, n, out, outn)
            for x in (owner, out, outn):
                x.free()
    for x in (dlc, dla, darea):
        x.free()
