"""MO_XCALL_GO_CASE, MO_XCALL_GO_COALESCE and MO_XCALL_GO_CASE_SELECT on the device against case_reference.py, byte for byte: every
type, 1, 2, 16 and 1024 WHENs with and without ELSE, const, const NULL and all-NULL operands, one row and a ragged last bitmap word,
skipped rows, values passed through as bytes (float -0 and NaN payloads), strings inline, at 23 / 24 bytes, with zero bytes and long, the
area capacity protocol, bad cells chosen and not chosen, host form == device form, launch counts, the enqueue-only form, the refusals, a
grid-stride run past 10^7 rows, and the short-circuit a CASE needs around a failing branch."""
import ctypes as C

import numpy as np
import pytest

import case_reference as R
import cell_edges as E
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, bitmap_to_bools, varlena_bytes_column, xcall
from test_gpu_go_operands import ONE_NULL, Arg, call, rand_bits, words

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

N = 1000
FIXED = sorted(ops.CASE_WIDTH)
STRINGS = list(ops.CASE_STR_TYPES)
VOCAB = [b"", b"a", b"ab\x00c", b"\x00", b"x" * 23, b"y" * 24, b"z" * 25, b"long value " * 4, b"\xe4\xb8\xad", b"q" * 300]


def rows_bytes(data, width, k):
    b = np.ascontiguousarray(data).view(np.uint8).reshape(-1).tobytes()
    return [b[i * width:(i + 1) * width] for i in range(k)]


def operand(rng, T, kind, n, cond=False):
    """(Arg, per-row values with None for NULL).  kind: v column (10% NULL), c const, n const NULL, a all-NULL column"""
    k = 1 if kind in "cn" else n
    if cond:
        data, vals, area = rng.integers(0, 2, k).astype(np.uint8), None, None
        vals = [bool(x) for x in data]
    elif T in STRINGS:
        vals = [VOCAB[i] for i in rng.integers(0, len(VOCAB), k)]
        data, area = varlena_bytes_column(vals)
    else:
        w = ops.CASE_WIDTH[T]
        data, area = rng.integers(0, 256, k * w).astype(np.uint8), None
        vals = rows_bytes(data, w, k)
    if kind == "n":
        nulls = ONE_NULL
    elif kind == "c":
        nulls = np.zeros(1, np.uint64)
    elif kind == "a":
        nulls = bitmap_from_bools(np.ones(n, bool))
    else:
        nulls = rand_bits(rng, n, 0.1)
    isnull = bitmap_to_bools(nulls, k)
    return Arg(data, nulls, area), [None if isnull[i] else v for i, v in enumerate(vals)]


def result_arg(rng, T, n, cap=0):
    """a result with random bytes (skipped rows must keep them) and about 10% of its rows skipped, ones past len"""
    skip = rng.random(n) < 0.1
    rn = bitmap_from_bools(skip)
    if n & 63:
        rn[-1] |= np.uint64(~((1 << (n & 63)) - 1) & 0xffffffffffffffff)
    w = 24 if T in STRINGS else ops.CASE_WIDTH[T]
    prior = rng.integers(0, 256, n * w).astype(np.uint8)
    return Arg(prior, rn, np.full(cap, 0xee, np.uint8) if cap else None), skip, prior.tobytes()


def case_call(rng, T, nsel, has_else, n, coalesce=False, kinds="vcna", cap=None):
    """the arguments of one call and what the reference says it leaves: (args, expected {slot: bytes} without the area, expected area)"""
    ops_, conds, values = [], [], []
    pick = lambda: kinds[rng.integers(0, len(kinds))]   # noqa: E731
    for j in range(nsel):
        if not coalesce:
            a, v = operand(rng, T, pick(), n, cond=True)
            ops_.append(a); conds.append(v)
        a, v = operand(rng, T, pick(), n)
        ops_.append(a); values.append(v)
    else_rows = None
    if has_else:
        a, else_rows = operand(rng, T, pick(), n)
        ops_.append(a)
    strs = T in STRINGS
    res, skip, prior = result_arg(rng, T, n)
    out = R.coalesce(values, n, skip) if coalesce else R.case_fn(conds, values, else_rows, n, skip)
    if strs:
        cells, area = R.str_bytes(out, prior)
        res = Arg(prior, res.slots["pnulls"].view(np.uint64), np.zeros(len(area) if cap is None else cap, np.uint8))
    else:
        cells, area = R.fixed_bytes(out, ops.CASE_WIDTH[T], prior), b""
    prm = Arg(np.frombuffer(bytes(capi.CaseParams(nsel, has_else, 0)), np.uint8))
    want_nulls = bitmap_from_bools(R.nulls_of(out)).tobytes()
    return [res, prm] + ops_, {(0, "pdata"): cells, (0, "pnulls"): want_nulls}, area


def fid_of(T, coalesce):
    return capi.XCALL_GO_COALESCE(T) if coalesce else capi.XCALL_GO_CASE(T)


def check_call(gpu, T, nsel, has_else, n, seed, coalesce=False, kinds="vcna"):
    rng = np.random.default_rng(seed)
    args, want, area = case_call(rng, T, nsel, has_else, n, coalesce, kinds)
    got = {}
    for device in (False, True):
        rc, msg, launches, _, out = call(gpu, fid_of(T, coalesce), args, n, device=device)
        assert rc == 0, msg
        assert launches == (3 if T in STRINGS else 1)
        for k, v in want.items():
            assert out[k] == v, (device, k)
        if T in STRINGS:
            assert np.frombuffer(out[(1, "pdata")], np.int64)[1] == len(area)
            if area:
                assert out[(0, "parea")] == area
        got[device] = out
    assert got[False] == got[True], "host and device forms leave the same bytes"


@pytest.mark.parametrize("has_else", [0, 1])
@pytest.mark.parametrize("nsel", [1, 2, 16])
@pytest.mark.parametrize("T", FIXED + STRINGS)
def test_case_every_type(gpu, T, nsel, has_else):
    check_call(gpu, T, nsel, has_else, N, seed=T * 100 + nsel * 2 + has_else)
    check_call(gpu, T, nsel, has_else, 1, seed=T + nsel, kinds="vc")     # len == 1: one-element operands are columns


@pytest.mark.parametrize("nsel", [1, 2, 16])
@pytest.mark.parametrize("T", FIXED + STRINGS)
def test_coalesce_every_type(gpu, T, nsel):
    check_call(gpu, T, nsel, 0, N, seed=T * 7 + nsel, coalesce=True)


@pytest.mark.parametrize("has_else", [0, 1])
@pytest.mark.parametrize("T", [capi.T_INT64, capi.T_DECIMAL128, capi.T_BOOL, capi.T_VARCHAR])
def test_a_thousand_whens(gpu, T, has_else):
    check_call(gpu, T, capi.CASE_MAX_WHENS, has_else, 200, seed=T + has_else, kinds="vcn")
    check_call(gpu, T, capi.CASE_MAX_WHENS, 0, 200, seed=T + 5, coalesce=True, kinds="vn")


def test_const_null_operands_only_matter_where_chosen(gpu):
    n = 130
    c1 = (np.arange(n) % 3 == 0).astype(np.uint8)
    x = np.arange(n, dtype=np.int64)
    # WHEN <const NULL> THEN x  WHEN c1 THEN <const NULL>  ELSE x: the const NULL condition never matches, the const NULL value nulls c1's rows
    v, nl = ops.go_case(capi.T_INT64, [(np.array([1], np.uint8), ONE_NULL), (c1, None)], [(x, None), (np.array([7], np.int64), ONE_NULL)],
                        (x, None))
    assert (nl == c1.astype(bool)).all()
    assert (v[~nl] == x[~nl]).all() and (v[nl] == 0).all()
    v, nl = ops.go_coalesce(capi.T_INT64, [(np.array([5], np.int64), ONE_NULL), (x, bitmap_from_bools(c1.astype(bool))), (np.array([9], np.int64), None)])
    assert not nl.any() and (v == np.where(c1 == 1, 9, x)).all()


@pytest.mark.parametrize("T,dt", [(capi.T_FLOAT64, np.float64), (capi.T_FLOAT32, np.float32)])
def test_float_values_pass_as_bytes(gpu, T, dt):
    bits = np.dtype(dt).itemsize * 8
    ut = np.uint64 if bits == 64 else np.uint32
    special = np.array([0.0, -0.0, np.inf, -np.inf], dt).view(ut).tolist() + [int(0x7ff8dead00000001 if bits == 64 else 0x7fc0beef),
                                                                           int(0xfff0000000000001 if bits == 64 else 0xff800001)]
    a = np.array(special * 20, ut)
    b = a[::-1].copy()
    c = (np.arange(a.size) % 2).astype(np.uint8)
    v, nl = ops.go_iff(T, (c, None), (a.view(dt), None), (b.view(dt), None))
    assert not nl.any()
    assert (v.view(ut) == np.where(c == 1, a, b)).all()


def test_strings_at_their_edges(gpu):
    vals = [b"", b"x" * 23, b"y" * 24, b"a\x00b", b"\x00" * 30, b"p" * 40]
    n = len(vals) * 11
    col = [vals[i % len(vals)] for i in range(n)]
    c = (np.arange(n) % 2).astype(np.uint8)
    long_const = [b"L" * 40]
    cells, area, nl = ops.go_iff(capi.T_VARCHAR, (c, None), (col, None), (long_const, None))
    want = [col[i] if c[i] else long_const[0] for i in range(n)]
    wc, wa = R.str_bytes(want, bytes(24 * n))
    assert cells.tobytes() == wc and area.tobytes() == wa and not nl.any()
    # a long const chosen by every row: len * 40 bytes, more than any operand's area
    cells, area, _ = ops.go_case(capi.T_TEXT, [(np.array([1], np.uint8), None)], [(long_const, None)], None, length=1000)
    assert area.nbytes == 40 * 1000
    assert cells.tobytes() == R.str_bytes(long_const * 1000, bytes(24 * 1000))[0]


@pytest.mark.parametrize("device", [False, True])
def test_area_capacity_protocol(gpu, device):
    rng = np.random.default_rng(5)
    args, want, area = case_call(rng, capi.T_VARCHAR, 3, 1, N, kinds="vc", cap=0)
    assert len(area) > 100
    short = 57
    args[0] = Arg(args[0].slots["pdata"], args[0].slots["pnulls"].view(np.uint64), np.full(short, 0xee, np.uint8))
    rc, msg, launches, _, out = call(gpu, capi.XCALL_GO_CASE(capi.T_VARCHAR), args, N, device=device)
    assert rc == capi.RC_OUT_OF_RANGE, msg
    assert launches == 2, "the write is not launched"
    assert np.frombuffer(out[(1, "pdata")], np.int64)[1] == len(area)
    for s in ("pdata", "pnulls", "parea"):
        assert out[(0, s)] == args[0].slots[s].tobytes(), "the result is unchanged"
    args[0] = Arg(args[0].slots["pdata"], args[0].slots["pnulls"].view(np.uint64), np.zeros(len(area), np.uint8))
    rc, msg, launches, _, out = call(gpu, capi.XCALL_GO_CASE(capi.T_VARCHAR), args, N, device=device)
    assert rc == 0 and launches == 3, msg
    assert out[(0, "pdata")] == want[(0, "pdata")] and out[(0, "pnulls")] == want[(0, "pnulls")] and out[(0, "parea")] == area


@pytest.mark.parametrize("device", [False, True])
def test_bad_cells_only_where_chosen(gpu, device):
    n = 300
    vals = [b"v" * 30] * n
    cells, area = varlena_bytes_column(vals)
    bad = cells.copy().reshape(n, 24)
    bad.view(np.uint32)[:, 1] = 10 ** 6                     # every cell points past the area
    c = np.zeros(n, np.uint8)
    c[[77, 150]] = 1
    res = Arg(np.zeros(24 * n, np.uint8), np.zeros(words(n), np.uint64), np.zeros(40 * n, np.uint8))
    prm = Arg(np.frombuffer(bytes(capi.CaseParams(1, 1, 0)), np.uint8))
    args = [res, prm, Arg(c), Arg(bad.reshape(-1), None, area), Arg(cells, None, area)]
    rc, msg, _, _, out = call(gpu, capi.XCALL_GO_CASE(capi.T_VARCHAR), args, n, device=device)
    assert rc == capi.RC_INVALID_ARGUMENT and "operand 3 row 77" in msg, msg
    assert out[(0, "pdata")] == bytes(24 * n)
    args[2] = Arg(np.zeros(n, np.uint8))                       # the bad THEN is never chosen: never read
    rc, msg, _, _, out = call(gpu, capi.XCALL_GO_CASE(capi.T_VARCHAR), args, n, device=device)
    assert rc == 0, msg
    assert out[(0, "pdata")] == R.str_bytes(vals, bytes(24 * n))[0]
    if not device:
        return
    # THEN cells on the device 8-byte but not 16-byte aligned (three 8-byte loads) and 1-byte misaligned (byte loads); a value that ends
    # at the area's end is good, one a byte past it or whose end wraps 32 bits is not
    vals = [b"%03d" % i * 10 for i in range(n)]
    c = (np.arange(n) % 3 == 0).astype(np.uint8)
    ec, ea = E.edges(vals, 6, None, None)
    els, elsa = varlena_bytes_column([b"else value longer than the inline cell"])

    def case(then_ptr):
        r, rn, rarea = np.zeros(24 * n, np.uint8), np.zeros(words(n), np.uint64), np.zeros(40 * n, np.uint8)
        prm = np.frombuffer(bytes(capi.CaseParams(1, 1, 0)), np.uint8).copy()
        vecs = [Vector(data=r, nulls=rn, area=rarea, length=n), Vector(data=prm), Vector(data=c, length=n),
                Vector(data=ec if then_ptr is None else None, data_ptr=then_ptr, data_nbytes=ec.nbytes, area=ea, length=n),
                Vector(data=els, area=elsa, length=n)]
        rc, msg = xcall(capi.XCALL_GO_CASE(capi.T_VARCHAR), vecs, n, raise_on_error=False)
        return rc, msg, r.tobytes() + rarea.tobytes()

    rc, msg, want = case(None)
    assert rc == 0, msg
    for shift in E.SHIFTS:
        for cells, bad_row in ((ec, None), (E.edges(vals, 6, 9, 30)[0], 9), (E.edges(vals, 6, None, 12)[0], 12)):
            owner, dc = E.on_device(cells, shift)
            rc, msg, got = case(dc.ptr)
            owner.free()
            if bad_row is None:
                assert rc == 0 and got == want, (shift, msg)
            else:
                assert rc == capi.RC_INVALID_ARGUMENT and "operand 3 row %d" % bad_row in msg, (shift, msg)


def test_ten_million_rows(gpu):
    n = 10_000_037
    rng = np.random.default_rng(9)
    x = rng.integers(-10 ** 12, 10 ** 12, n)
    y = rng.integers(-10 ** 12, 10 ** 12, n)
    c1, c2 = (rng.random(n) < 0.3).astype(np.uint8), (rng.random(n) < 0.5).astype(np.uint8)
    yn = rng.random(n) < 0.05
    skip = rng.random(n) < 0.01
    bufs = [DeviceBuffer.from_numpy(a) for a in (c1, x, c2, y, bitmap_from_bools(yn), np.array([42], np.int64))]
    d_out, d_rn = DeviceBuffer(8 * n), DeviceBuffer.from_numpy(bitmap_from_bools(skip))
    ops.go_case_device(capi.T_INT64, [(bufs[0], None), (bufs[2], None)], [(bufs[1], None), (bufs[3], bufs[4])], (bufs[5], None), n, d_out, d_rn)
    got, gn = d_out.to_numpy(np.int64, n), bitmap_to_bools(d_rn.to_numpy(np.uint64), n)
    for b in bufs + [d_out, d_rn]:
        b.free()
    want = np.where(c1 == 1, x, np.where(c2 == 1, y, 42))
    wn = skip | ((c1 == 0) & (c2 == 1) & yn)
    assert (gn == wn).all()
    live = ~gn
    assert (got[live] == want[live]).all()
    assert (got[~skip & gn] == 0).all()


def test_ten_million_string_rows(gpu):
    n = 10_000_037
    rng = np.random.default_rng(10)
    vocab = [b"short", b"s" * 23, b"forty bytes of a value, more than inline", b"w" * 24]
    ia, ib = rng.integers(0, 4, n), rng.integers(0, 4, n)
    c = (rng.random(n) < 0.5).astype(np.uint8)
    vc, va = varlena_bytes_column(vocab)
    canon = vc.reshape(4, 24)
    def col(idx):                                  # every row's cell points at the vocabulary's one area
        return canon[idx].reshape(-1)
    d = [DeviceBuffer.from_numpy(a) for a in (c, col(ia), col(ib), va)]
    long_len = np.array([0, 0, 40, 24])
    need = int(np.where(c == 1, long_len[ia], long_len[ib]).sum())
    d_out, d_rn, d_area = DeviceBuffer(24 * n), DeviceBuffer.from_numpy(np.zeros(words(n), np.uint64)), DeviceBuffer(need)
    rc, area_len = ops.go_case_device(capi.T_VARCHAR, [(d[0], None)], [((d[1], d[3]), None)], ((d[2], d[3]), None), n, d_out, d_rn, d_area)
    assert rc == 0 and area_len == need
    cells = d_out.to_numpy(np.uint8, 24 * n).reshape(n, 24)
    area = d_area.to_numpy(np.uint8, need)
    for b in d + [d_out, d_rn, d_area]:
        b.free()
    idx = np.where(c == 1, ia, ib)
    lens = np.array([5, 23, 40, 24])[idx]
    long_ = lens > 23
    assert (cells[~long_] == canon[idx[~long_]]).all()
    ll = np.where(long_, lens, 0)
    offs = np.cumsum(ll) - ll
    u32 = cells.view(np.uint32)
    assert (u32[long_, 0] == 0xffffffff).all() and (u32[long_, 1] == offs[long_]).all() and (u32[long_, 2] == lens[long_]).all()
    for i in rng.choice(np.flatnonzero(long_), 2000, replace=False):
        assert area[offs[i]:offs[i] + lens[i]].tobytes() == vocab[idx[i]]


# ---- CASE_SELECT
def test_case_select_matches_eval_case(gpu):
    rng = np.random.default_rng(2)
    n = 777
    select = rng.random(n) < 0.8
    rem = bitmap_from_bools(~select)
    conds = []
    for kind in ("v", "v", "c", "n"):
        a, rows = operand(rng, None, kind, n, cond=True)
        conds.append((a, R.expand(rows, n)))
    when_lists, then_lists, else_list = R.case_select_lists(list(select), [r for _, r in conds])
    for j, (a, _) in enumerate(conds):
        assert (bitmap_to_bools(rem, n) == ~np.array(when_lists[j])).all()
        then, rem = ops.case_select(rem, a.slots["pdata"], None if a.slots["pnulls"] is None else a.slots["pnulls"].view(np.uint64), n)
        assert (bitmap_to_bools(then, n) == ~np.array(then_lists[j])).all()
        assert then[-1] >> np.uint64(n & 63) == np.uint64((1 << (64 - (n & 63))) - 1), "bits past len are set in the prefill"
    assert (bitmap_to_bools(rem, n) == ~np.array(else_list)).all()


@pytest.fixture
def stream(gpu):
    s = torch.cuda.Stream()
    capi.check(gpu.MoB200_SetStream(C.c_void_p(s.cuda_stream)), gpu)
    yield s
    capi.check(gpu.MoB200_SetStream(None), gpu)


@pytest.mark.parametrize("T", [capi.T_INT64, capi.T_DECIMAL128, capi.T_INT8])
def test_fixed_width_and_select_only_enqueue(gpu, stream, T):
    rng = np.random.default_rng(T)
    args, want, _ = case_call(rng, T, 2, 1, N)
    rc, msg, launches, idle, out = call(gpu, capi.XCALL_GO_CASE(T), args, N, device=True, stream=stream, host_args=(1,))
    assert rc == 0 and launches == 1, msg
    assert not idle, "the all-device call waited for its stream"
    assert out[(0, "pdata")] == want[(0, "pdata")]
    sel = [Arg(np.zeros(words(N), np.uint64)), Arg(rand_bits(rng, N, 0.3)), Arg(rng.integers(0, 2, N).astype(np.uint8), rand_bits(rng, N, 0.1))]
    rc, msg, launches, idle, dev = call(gpu, capi.XCALL_GO_CASE_SELECT, sel, N, device=True, stream=stream)
    assert rc == 0 and launches == 1 and not idle, msg
    rc, msg, launches, idle, host = call(gpu, capi.XCALL_GO_CASE_SELECT, sel, N, device=False, stream=stream)
    assert rc == 0 and idle and host == dev, msg


# ---- refusals
def refusal_args(T, n=N, nsel=1, has_else=1):
    rng = np.random.default_rng(0)
    return case_call(rng, T, nsel, has_else, n, kinds="v")[0]


@pytest.mark.parametrize("T", [capi.T_INT32, capi.T_VARCHAR])
def test_refusals(gpu, T):
    fid = capi.XCALL_GO_CASE(T)

    def refused(args, text, f=fid, n=N):
        for device in (False, True):
            rc, msg, _, _, _ = call(gpu, f, args, n, device=device)
            assert rc == capi.RC_INVALID_ARGUMENT and text in msg, (device, msg)

    for bad_t in (capi.T_BINARY, capi.T_VARBINARY, capi.T_YEAR, 90):
        refused(refusal_args(T), "unsupported type", f=capi.XCALL_GO_CASE(bad_t))
    for nsel, he, text in ((0, 1, "n 0"), (1025, 0, "n 1025"), (1, 2, "has_else 2")):
        a = refusal_args(T)
        a[1] = Arg(np.frombuffer(bytes(capi.CaseParams(nsel, he, 0)), np.uint8))
        refused(a, text)
    a = refusal_args(T, has_else=0)
    a[1] = Arg(np.frombuffer(bytes(capi.CaseParams(1, 1, 0)), np.uint8))
    refused(a, "has_else 1", f=capi.XCALL_GO_COALESCE(T))
    a = refusal_args(T)
    a[3].slots["pdata"] = a[3].slots["pdata"][:-1]
    refused(a, "operand 3 holds")
    a = refusal_args(T)
    a[0].slots["pdata"] = a[0].slots["pdata"][:-1]
    refused(a, "the result holds")
    a = refusal_args(T)
    a[0].slots["pnulls"] = None
    refused(a, "no null bitmap")
    a = refusal_args(T)
    a[1].slots["pdata"] = None
    refused(a, "params missing")


# ---- the short-circuit: CASE WHEN d <> 0 THEN x / d ELSE 0 END with division by zero an error
def test_short_circuit_around_a_failing_division(gpu):
    rng = np.random.default_rng(4)
    n = 1000
    x = rng.integers(-10 ** 6, 10 ** 6, n).astype(np.int64)
    d = rng.integers(-5, 5, n).astype(np.int64)
    first_zero = int(np.flatnonzero(d == 0)[0])
    rem = np.zeros(words(n), np.uint64)                     # selectList: every row
    cond = (d != 0).astype(np.uint8)                         # the WHEN, evaluated under rem
    then, rem = ops.case_select(rem, cond, None, n)
    rc, q, qn, err_row, msg = ops.dec_div(64, x, d, 2, 2, n, rnulls=then, div0_error=True)
    assert rc == 0, msg
    zero = np.zeros((1, 2), np.uint64)
    vals, nl = ops.go_case(capi.T_DECIMAL128, [(cond, None)], [(q, qn)], (zero, None))
    assert not nl.any()
    assert (vals[d == 0] == 0).all()
    assert (vals[d != 0] == q[d != 0]).all()
    rc, _, _, err_row, msg = ops.dec_div(64, x, d, 2, 2, n, div0_error=True)
    assert rc == capi.RC_DIVISION_BY_ZERO and err_row == first_zero, msg


def test_const_bad_cell_names_the_row_that_chose_it(gpu):
    n = 300
    good_cells, good_area = varlena_bytes_column([b"g" * 30] * n)
    bad_cells, bad_area = varlena_bytes_column([b"b" * 30])
    bad_cells = bad_cells.copy()
    bad_cells.view(np.uint32)[1] = 10 ** 6                     # the const THEN points past its area
    c = np.zeros(n, np.uint8)
    c[[123, 200]] = 1
    res = Arg(np.zeros(24 * n, np.uint8), np.zeros(words(n), np.uint64), np.zeros(30 * n, np.uint8))
    prm = Arg(np.frombuffer(bytes(capi.CaseParams(1, 1, 0)), np.uint8))
    args = [res, prm, Arg(c), Arg(bad_cells, None, bad_area), Arg(good_cells, None, good_area)]
    for device in (False, True):
        rc, msg, _, _, _ = call(gpu, capi.XCALL_GO_CASE(capi.T_VARCHAR), args, n, device=device)
        assert rc == capi.RC_INVALID_ARGUMENT and "operand 3 row 123:" in msg, msg


@pytest.mark.parametrize("T", [capi.T_INT64, capi.T_DECIMAL128])
def test_a_thousand_whens_only_enqueue(gpu, stream, T):
    """2049 operand descriptors (82 KB) go up with the call, and it still returns before its stream has run"""
    rng = np.random.default_rng(T + 1)
    args, want, _ = case_call(rng, T, capi.CASE_MAX_WHENS, 1, N, kinds="vcn")
    rc, msg, launches, idle, out = call(gpu, capi.XCALL_GO_CASE(T), args, N, device=True, stream=stream, host_args=(1,))
    assert rc == 0 and launches == 1, msg
    assert not idle, "the all-device call waited for its stream"
    assert out[(0, "pdata")] == want[(0, "pdata")] and out[(0, "pnulls")] == want[(0, "pnulls")]
