"""Row-wise distances (csrc/distance.cu, the row_batch ring of csrc/godist.cuh) and normalize_l2 at their edges, against the oracle's
restatement of the Go loops row by row (rowdist_columns.py).

One lane owns one row and a warp stages 32 rows through a cp.async ring (3 stages with two per-row operands, 5 with a const side),
so the cases aim at what differs between the lanes of one warp: slice counts (nsl) from 0 to 12 side by side, empty, inline and area
rows, every offset mod 16 on each operand, duplicated cells, NULL rows and error rows.  Uniform columns put the last slice on both
sides of each ring wrap, and n above three grid-strides of resident warps (the grid is capped at 2 CTAs of 128 threads per SM) makes
warps take several batches.

Go ids and normalize_l2 are compared bit for bit (signed zeros included), any NaN standing for any NaN: x86 and the device make
different NaN payloads.  Reference ids 0..3 are compared with the reference C at 1e-5 (it accumulates in double under -ffast-math)."""
import ctypes as C

import numpy as np
import pytest

import cell_edges as E
import oracle_lib as O
import rowdist_columns as R
from matrixone_b200 import capi
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, varlena_bytes_column, varlena_column_from_matrix, xcall

pytestmark = pytest.mark.gpu

SENT = -1234.5          # what result rows hold before a call: NULL rows must keep it
OFILL = 0xEE            # what the normalize_l2 result area holds before a call
DTYPES = [np.float32, np.float64]
KIND_NAMES = {R.L2: "l2", R.L2SQ: "l2sq", R.IP: "ip", R.COSDIST: "cosdist", R.COSSIM: "cossim", R.L1: "l1"}
FID = {np.float32: {R.L2: capi.XCALL_GO_L2_F32, R.L2SQ: capi.XCALL_GO_L2SQ_F32, R.IP: capi.XCALL_GO_IP_F32,
                    R.COSDIST: capi.XCALL_GO_COSDIST_F32, R.COSSIM: capi.XCALL_GO_COSSIM_F32, R.L1: capi.XCALL_GO_L1_F32},
       np.float64: {R.L2: capi.XCALL_GO_L2_F64, R.L2SQ: capi.XCALL_GO_L2SQ_F64, R.IP: capi.XCALL_GO_IP_F64,
                    R.COSDIST: capi.XCALL_GO_COSDIST_F64, R.COSSIM: capi.XCALL_GO_COSSIM_F64, R.L1: capi.XCALL_GO_L1_F64}}
NORM_FID = {np.float32: capi.XCALL_GO_NORMALIZE_L2_F32, np.float64: capi.XCALL_GO_NORMALIZE_L2_F64}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nulls_mask(n, nulls):
    return np.zeros(n, bool) if nulls is None else np.asarray(nulls, bool)


def _want(kind, x, q, n, nulls=None):
    """per row: the Go value of f(x_i, q_i) (a one-row column is a const operand), SENT on NULL rows; and the rows whose evaluation
    fails (cosine similarity of a zero vector)"""
    null = _nulls_mask(n, nulls)
    want, err = np.full(n, SENT), np.zeros(n, bool)
    for i in range(n):
        if not null[i]:
            want[i], err[i] = R.row_distance(kind, x.rows[0 if x.n == 1 else i], q.rows[0 if q.n == 1 else i])
    return want, err


def _call_host(fid, x, q, n, nulls=None):
    res = np.full(n, SENT)
    rc, msg = xcall(fid, [Vector(data=res, nulls=None if nulls is None else bitmap_from_bools(nulls), length=n),
                          Vector(data=x.cells, area=x.area, length=n), Vector(data=q.cells, area=q.area, length=n)], n, raise_on_error=False)
    return rc, msg, res


def _call_device(fid, x, q, n, kx, kq, nulls=None):
    """every operand resident: cells, result and nulls in device buffers, each area a view kx / kq bytes past an aligned allocation"""
    xc, xa = x.device(kx)
    qc, qa = q.device(kq)
    dr = DeviceBuffer.from_numpy(np.full(n, SENT))
    dn = None if nulls is None else DeviceBuffer.from_numpy(bitmap_from_bools(nulls))
    rc, msg = xcall(fid, [Vector(data_ptr=dr.ptr, data_nbytes=8 * n, nulls_ptr=None if dn is None else dn.ptr, length=n),
                          Vector(data_ptr=xc.ptr, data_nbytes=xc.nbytes, area_ptr=xa.ptr, area_nbytes=xa.nbytes, length=n),
                          Vector(data_ptr=qc.ptr, data_nbytes=qc.nbytes, area_ptr=qa.ptr, area_nbytes=qa.nbytes, length=n)], n, raise_on_error=False)
    res = dr.to_numpy(np.float64, n)
    for b in (xc, xa.owner, qc, qa.owner, dr) + (() if dn is None else (dn,)):
        b.free()
    return rc, msg, res


def _check(got, want, what, x=None):
    ok = R.same(got, want)
    if not ok.all():
        bad = np.flatnonzero(~ok)[:8]
        lens = "" if x is None else " lens %s kinds %s" % ([x.rows[i].size if x.n > 1 else x.rows[0].size for i in bad],
                                                          [x.kind[i] if x.n > 1 else "const" for i in bad])
        pytest.fail("%s: %d rows differ, first %s: got %s want %s%s" % (what, (~ok).sum(), bad.tolist(), got[bad].tolist(), want[bad].tolist(), lens))


def _run_both(kind, dt, x, q, n, what, nulls=None, kx=5, kq=11):
    """host and device forms of one call against the per-row reference; rows whose evaluation fails are made NULL first"""
    want, err = _want(kind, x, q, n, nulls)
    if err.any():
        nulls = _nulls_mask(n, nulls) | err
        want[err] = SENT
    fid = FID[dt][kind]
    rc, msg, res = _call_host(fid, x, q, n, nulls)
    assert rc == 0, (what, msg)
    _check(res, want, "%s host" % what, x)
    rc, msg, res = _call_device(fid, x, q, n, kx, kq, nulls)
    assert rc == 0, (what, msg)
    _check(res, want, "%s device (area views +%d / +%d)" % (what, kx, kq), x)


# ---- 1. ragged rows in one warp, two per-row operands -------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", R.KINDS, ids=KIND_NAMES.get)
@pytest.mark.parametrize("dt", DTYPES)
def test_ragged_warp_two_per_row_operands(gpu, dt, kind):
    """neighbouring lanes with slice counts 0..12, empty / inline / area / duplicated rows, x and q at separately chosen offsets mod 16;
    the device form with the areas at every view offset 1..15"""
    x, q = R.ragged_pair(dt, 11)
    n = x.n
    want, err = _want(kind, x, q, n)
    assert not err.any()
    fid = FID[dt][kind]
    rc, msg, res = _call_host(fid, x, q, n)
    assert rc == 0, msg
    _check(res, want, "ragged host", x)
    for k in range(1, 16):
        rc, msg, res = _call_device(fid, x, q, n, k, (7 * k) % 16)
        assert rc == 0, msg
        _check(res, want, "ragged device (area views +%d / +%d)" % (k, (7 * k) % 16), x)


# ---- 2. uniform columns at the ring-wrap boundaries -----------------------------------------------------------------------------------
RING = {"two": 3, "const_second": 5, "const_first": 5, "both_const": 5}


@pytest.mark.parametrize("mode", list(RING))
@pytest.mark.parametrize("dt", DTYPES)
def test_ring_wrap(gpu, dt, mode):
    """maxsl = NST - 1, NST, NST + 1 and 2 NST for the 3-stage ring (two per-row operands) and the 5-stage ring (a const side: second,
    first = the operand swap, or both), with and without a tail past the last slice"""
    nst = RING[mode]
    eps = R.slice_elems(dt)
    n = 97
    for m in (nst - 1, nst, nst + 1, 2 * nst):
        for dim in (m * eps, m * eps + 9):
            for chunk in (8, 4):
                assert R.slices(dim, dt, chunk) == m
            pads = list(range(16))
            x = R.uniform_column(dt, dim, n, dim, pads)
            q = R.uniform_column(dt, dim + 1, n, dim, pads[::-1])
            c1 = R.uniform_column(dt, dim + 2, 1, dim, [m % 16])
            c2 = R.uniform_column(dt, dim + 3, 1, dim, [0])
            a, b = {"two": (x, q), "const_second": (x, c1), "const_first": (c1, q), "both_const": (c1, c2)}[mode]
            for kind in R.KINDS:
                _run_both(kind, dt, a, b, n, "%s maxsl %d dim %d %s" % (mode, m, dim, KIND_NAMES[kind]), kx=m % 16 or 1, kq=3)


# ---- 3. grid-stride and partial warps ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
def test_grid_stride_and_partial_warps(gpu, dt):
    """n above three times the resident rows (num SMs x 2 CTAs x 128), n % 32 != 0, rows at mixed offsets mod 16 (rows of 37 / 19
    elements back to back), NULL rows keeping SENT; then n in {1, 31, 32, 33} on the ragged columns"""
    n = 131_071
    assert n >= 3 * _sms() * 2 * 128
    dim = 37 if dt == np.float32 else 19
    rng = np.random.default_rng(7)
    a = rng.standard_normal((n, dim)).astype(dt)
    b = rng.standard_normal((n, dim)).astype(dt)
    a[77_777] = b[77_777]
    null = rng.random(n) < 0.1
    ac, aa = varlena_column_from_matrix(a)
    bc, ba = varlena_column_from_matrix(b)
    qc, qa = varlena_column_from_matrix(b[:1])
    for kind in (R.L2, R.L2SQ, R.IP, R.COSDIST, R.L1):
        for (cells, area, bm) in ((bc, ba, b), (qc, qa, b[:1])):
            want = R.matrix_distance(kind, a, bm, bitmap_from_bools(null))
            want[null] = SENT
            res = np.full(n, SENT)
            xcall(FID[dt][kind], [Vector(data=res, nulls=bitmap_from_bools(null), length=n), Vector(data=ac, area=aa, length=n),
                                  Vector(data=cells, area=area, length=n)], n)
            _check(res, want, "grid-stride %s%s" % (KIND_NAMES[kind], " const" if bm.shape[0] == 1 else ""))
    # cosine similarity: per-row reference, resident operands
    want = np.full(n, SENT)
    for i in np.flatnonzero(~null):
        want[i] = R.row_distance(R.COSSIM, a[i], b[i])[0]
    dac, daa, dbc, dba = (DeviceBuffer.from_numpy(v) for v in (ac, aa, bc, ba))
    dr, dn = DeviceBuffer.from_numpy(np.full(n, SENT)), DeviceBuffer.from_numpy(bitmap_from_bools(null))
    xcall(FID[dt][R.COSSIM], [Vector(data_ptr=dr.ptr, data_nbytes=8 * n, nulls_ptr=dn.ptr, length=n),
                              Vector(data_ptr=dac.ptr, data_nbytes=dac.nbytes, area_ptr=daa.ptr, area_nbytes=daa.nbytes, length=n),
                              Vector(data_ptr=dbc.ptr, data_nbytes=dbc.nbytes, area_ptr=dba.ptr, area_nbytes=dba.nbytes, length=n)], n)
    _check(dr.to_numpy(np.float64, n), want, "grid-stride cossim device")
    for buf in (dac, daa, dbc, dba, dr, dn):
        buf.free()
    x, q = R.ragged_pair(dt, 13)
    for m in (1, 31, 32, 33):
        xm = R.Column(x.rows[:m], dt, x.stores()[:m], list(range(m)))
        qm = R.Column(q.rows[:m], dt, None, [(3 * i) % 16 for i in range(m)])
        for kind in R.KINDS:
            _run_both(kind, dt, xm, qm, m, "n=%d %s" % (m, KIND_NAMES[kind]))


# ---- 4. NULL result rows -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
def test_null_rows_keep_their_result(gpu, dt):
    """NULL rows keep SENT in host and device forms, including NULL rows whose operands differ in length (they are never evaluated)
    and whole NULL warps"""
    x, q = R.ragged_pair(dt, 17)
    n = x.n
    rng = np.random.default_rng(17)
    null = rng.random(n) < 0.3
    null[64:96] = True
    # a NULL row whose operands differ in length: a dimension error if it were evaluated
    qrows = list(q.rows)
    j = next(i for i in range(n) if null[i] and x.kind[i] == "area" and q.kind[i] == "area")
    qrows[j] = np.concatenate([qrows[j], np.ones(1, dt)])
    q = R.Column(qrows, dt, q.stores(), [(5 * i + 3) % 16 for i in range(n)])
    for kind in R.KINDS:
        _run_both(kind, dt, x, q, n, "nulls %s" % KIND_NAMES[kind], nulls=null)


# ---- 5. special values ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", R.KINDS, ids=KIND_NAMES.get)
@pytest.mark.parametrize("dt", DTYPES)
def test_special_values(gpu, dt, kind):
    """NaN, +-Inf and -0.0 at chunk-edge, slice-edge and tail positions; subnormal operands (a build that flushes denormals fails
    here); all -0.0 rows (the inner product of zeros is -0.0); float32 rows whose accumulator overflows; exactly parallel and
    anti-parallel rows (the clamp and the float32 snap to +-1 of cosine similarity); const second operand with specials too"""
    x, q = R.ragged_pair(dt, 19, special=True)
    _run_both(kind, dt, x, q, x.n, "specials %s" % KIND_NAMES[kind])
    for i in (8, 20, 45):     # a const second operand holding special values, against rows of its length
        c = R.Column([q.rows[i]], dt, pad=[i % 16])
        same_len = [r for r in x.rows if r.size == c.rows[0].size] or [c.rows[0]]
        xr = R.Column(same_len * 3, dt, pad=[(3 * k + 1) % 16 for k in range(3 * len(same_len))])
        _run_both(kind, dt, xr, c, xr.n, "specials const %s row %d" % (KIND_NAMES[kind], i))


# ---- 6. reference ids 0..3 against the reference C --------------------------------------------------------------------------------------------
def _ref_call(ref, fid, x, q, n, nulls=None):
    res = np.full(n, SENT)
    v = [Vector(data=res, nulls=None if nulls is None else bitmap_from_bools(nulls), length=n),
         Vector(data=x.cells, area=x.area, length=n), Vector(data=q.cells, area=q.area, length=n)]
    args = (capi.XCallArgs * 3)(*(a.fill_raw_ptr_len() for a in v))
    err = (C.c_uint8 * 256)()
    assert ref.XCall(0, fid, err, C.cast(args, C.c_void_p), n) == 0
    return res


@pytest.mark.parametrize("dt,ids", [(np.float32, (capi.XCALL_L2DISTANCE_F32, capi.XCALL_L2DISTANCE_SQ_F32)),
                                    (np.float64, (capi.XCALL_L2DISTANCE_F64, capi.XCALL_L2DISTANCE_SQ_F64))])
def test_reference_ids_prefix_null_first_row_and_ragged(gpu, dt, ids):
    """the dim comes from the first cell of arg 1 (NULL or not, empty or not) and longer rows are read as their prefix; ragged, unaligned
    rows of arg 2 at least that long; NULL rows untouched"""
    ref = O.ref()
    if ref is None:
        pytest.skip("oracle/_ref missing")
    rng = np.random.default_rng(23)
    eps = R.slice_elems(dt)
    n = 100
    for dim0 in (0, 3, eps - 1, 2 * eps + 5, 5 * eps):
        lens = [dim0] + [dim0 + int(rng.integers(0, 2 * eps)) for _ in range(n - 1)]
        xs = [rng.standard_normal(ln).astype(dt) for ln in lens]
        qs = [rng.standard_normal(dim0 + int(rng.integers(0, 40))).astype(dt) for _ in range(n)]
        x = R.Column(xs, dt, pad=[(7 * i) % 16 for i in range(n)])
        q = R.Column(qs, dt, pad=[(3 * i + 2) % 16 for i in range(n)])
        c = R.Column([qs[0]], dt, pad=[9])
        for nulls in (None, np.arange(n) % 5 == 0):     # row 0 NULL: its cell still sets the dim
            for b in (q, c):
                for fid in ids:
                    want = _ref_call(ref, fid, x, b, n, nulls)
                    rc, msg, got = _call_host(fid, x, b, n, nulls)
                    assert rc == 0, msg
                    np.testing.assert_allclose(got, want, rtol=1e-5, atol=0, err_msg="dim0 %d" % dim0)
                    rc, msg, got = _call_device(fid, x, b, n, 13, 6, nulls)
                    assert rc == 0, msg
                    np.testing.assert_allclose(got, want, rtol=1e-5, atol=0, err_msg="dim0 %d device" % dim0)
                    if nulls is not None:
                        assert (got[nulls] == SENT).all()
                    if dim0 == 0:
                        assert (got[~_nulls_mask(n, nulls)] == 0.0).all()


# ---- 7. normalize_l2 -------------------------------------------------------------------------------------------------------------------------
def _normalize_call(dt, col, n, nulls=None, device=None):
    """(rc, msg, result cells, result area); device = (k_in, k_out): every buffer resident, the input area a view k_in bytes and the
    result area a view k_out bytes past aligned allocations"""
    nb = None if nulls is None else bitmap_from_bools(nulls)
    if device is None:
        oc, oa = np.full(24 * n, 0x55, np.uint8), np.full(col.area.nbytes, OFILL, np.uint8)
        rc, msg = xcall(NORM_FID[dt], [Vector(data=oc, area=oa, nulls=nb, length=n), Vector(data=col.cells, area=col.area, length=n)], n,
                        raise_on_error=False)
        return rc, msg, oc, oa
    ki, ko = device
    ic, ia = col.device(ki)
    doc = DeviceBuffer.from_numpy(np.full(24 * n, 0x55, np.uint8))
    downer = DeviceBuffer.from_numpy(np.full(col.area.nbytes + ko, OFILL, np.uint8))
    doa = downer.view(col.area.nbytes, ko)
    dn = None if nb is None else DeviceBuffer.from_numpy(nb)
    rc, msg = xcall(NORM_FID[dt], [Vector(data_ptr=doc.ptr, data_nbytes=doc.nbytes, area_ptr=doa.ptr, area_nbytes=doa.nbytes,
                                          nulls_ptr=None if dn is None else dn.ptr, length=n),
                                   Vector(data_ptr=ic.ptr, data_nbytes=ic.nbytes, area_ptr=ia.ptr, area_nbytes=ia.nbytes, length=n)], n,
                    raise_on_error=False)
    oc, oa = doc.to_numpy(np.uint8), downer.to_numpy(np.uint8)[ko:]
    for b in (ic, ia.owner, doc, downer) + (() if dn is None else (dn,)):
        b.free()
    return rc, msg, oc, oa


def _check_normalize(dt, col, n, oc, oa, nulls, what):
    """result cells mirror the input's (inline rows: length byte, normalized bytes, zeros; area rows: the input cell), NULL rows are
    empty inline cells, every live row decodes to og_normalize_l2 of its row, and result area bytes no live row owns keep OFILL"""
    null = _nulls_mask(n, nulls)
    const = col.n == 1 and n > 1
    owned = np.zeros(oa.nbytes, bool)
    for i in range(n):
        cell = oc[24 * i:24 * i + 24]
        if null[i]:
            assert not cell.any(), (what, i, "NULL row")
            continue
        r = 0 if const else i
        src = col.cells[24 * r:24 * r + 24]
        want = R.normalize(col.rows[r])
        got = R.decode(oc, oa, i, dt)
        assert got is not None and R.same(got, want).all(), (what, i, col.kind[r], col.rows[r].size, got, want)
        if src[0] <= R.INLINE_MAX:
            assert cell[0] == src[0] and not cell[1 + int(src[0]):].any(), (what, i)
        else:
            assert (cell == src).all(), (what, i)
            off = col.offset[r]
            owned[off:off + col.rows[r].nbytes] = True
    assert (oa[~owned] == OFILL).all(), (what, np.flatnonzero(oa[~owned] != OFILL)[:8])


@pytest.mark.parametrize("dt", DTYPES)
def test_normalize_mixed_columns(gpu, dt):
    """ragged rows, inline rows (float64: up to 2 elements), area rows at every offset mod 16, zero and -0.0 rows, subnormal, Inf and
    NaN rows, duplicated cells, NULL rows; host form, and device form with the input and result areas at different view offsets"""
    col = R.normalize_column(dt, 29)
    n = col.n
    null = np.random.default_rng(29).random(n) < 0.2
    null[[4, 9, 13, 17, 21, 3, 40]] = False
    null[41] = True                         # one of two duplicates of row 3 is NULL
    for nulls in (None, null):
        rc, msg, oc, oa = _normalize_call(dt, col, n, nulls)
        assert rc == 0, msg
        _check_normalize(dt, col, n, oc, oa, nulls, "host")
        for ki, ko in ((3, 3), (1, 12), (15, 0), (0, 7)):
            rc, msg, oc, oa = _normalize_call(dt, col, n, nulls, device=(ki, ko))
            assert rc == 0, msg
            _check_normalize(dt, col, n, oc, oa, nulls, "device +%d/+%d" % (ki, ko))


@pytest.mark.parametrize("dt", DTYPES)
def test_normalize_grid_stride_and_const(gpu, dt):
    """n above three grid-strides of resident rows, with NULL rows; a const input (one cell, len > 1) stored in the area and inline,
    with and without NULL rows, row 0 NULL included.

    Regression: the result area of a const input was written by row 0 only, so with row 0 NULL every other row's cell pointed at
    result bytes nobody wrote.  The first row that is not NULL writes it now."""
    rng = np.random.default_rng(31)
    n = 131_071
    eps = R.slice_elems(dt)
    lens = rng.integers(1, 3 * eps, n)
    mat = rng.standard_normal(int(lens.sum())).astype(dt)
    starts = np.cumsum(lens) - lens
    rows = [mat[s:s + ln] for s, ln in zip(starts, lens)]
    col = R.Column(rows, dt, pad=[int(v) for v in rng.integers(0, 16, n)])
    null = rng.random(n) < 0.1
    rc, msg, oc, oa = _normalize_call(dt, col, n, null, device=(9, 4))
    assert rc == 0, msg
    _check_normalize(dt, col, n, oc, oa, null, "grid-stride")
    for v, pad in ((rng.standard_normal(3 * eps + 5).astype(dt), 7), (np.array([0.5, -2.0], dt), None)):
        c = R.Column([v], dt, pad=[pad or 0])
        m = 1000
        for nulls in (None, np.arange(m) % 3 == 1, np.arange(m) % 3 == 0):
            for device in (None, (5, 2)):
                rc, msg, oc, oa = _normalize_call(dt, c, m, nulls, device)
                assert rc == 0, msg
                _check_normalize(dt, c, m, oc, oa, nulls, "const %s nulls %s" % (c.kind[0], None if nulls is None else int(np.argmax(~nulls))))


# ---- 8. error rows among valid rows of one warp --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
def test_error_rows_in_a_valid_warp(gpu, dt):
    """one bad row among valid ragged rows: operands of different lengths ("dimension"), a zero row under cosine similarity ("zero"),
    a cell whose offset + length passes the area (checked before any read); normalize_l2 of an empty row and of an out-of-area cell"""
    x, q = R.ragged_pair(dt, 37)
    n = x.n
    j = next(i for i in range(33, n) if x.kind[i] == "area" and q.kind[i] == "area" and x.rows[i].size > R.slice_elems(dt))
    qrows = list(q.rows)
    qrows[j] = qrows[j][:-1]
    store = q.stores()
    qd = R.Column(qrows, dt, store, [(5 * i + 3) % 16 for i in range(n)])
    for kind in R.KINDS:
        rc, msg, _ = _call_host(FID[dt][kind], x, qd, n)
        assert rc == capi.RC_INVALID_ARGUMENT and "dimension" in msg, (kind, rc, msg)
        rc, msg, _ = _call_device(FID[dt][kind], x, qd, n, 2, 9)
        assert rc == capi.RC_INVALID_ARGUMENT and "dimension" in msg, (kind, rc, msg)
    xz = list(x.rows)
    xz[j] = np.zeros_like(xz[j])
    xzc = R.Column(xz, dt, x.stores(), [i % 16 for i in range(n)])
    rc, msg, _ = _call_host(FID[dt][R.COSSIM], xzc, q, n)
    assert rc != 0 and "zero" in msg, msg
    rc, msg, res = _call_host(FID[dt][R.COSDIST], xzc, q, n)      # cosine distance of a zero row is 1, not an error
    assert rc == 0 and res[j] == 1.0, msg
    # a cell whose offset + length passes areaSz, among valid rows
    for col, other, swap in ((x, q, False), (q, x, True)):
        cells = col.cells.copy()
        u32 = cells.reshape(n, 24)[j].view(np.uint32)
        u32[1] = col.area.nbytes - int(u32[2]) + 4
        bad = R.Column.__new__(R.Column)
        bad.__dict__.update(col.__dict__)
        bad.cells = cells
        a, b = (other, bad) if swap else (bad, other)
        for kind in R.KINDS:
            rc, msg, _ = _call_host(FID[dt][kind], a, b, n)
            assert rc == capi.RC_INVALID_ARGUMENT and "outside" in msg, (kind, rc, msg)
            rc, msg, _ = _call_device(FID[dt][kind], a, b, n, 4, 12)
            assert rc == capi.RC_INVALID_ARGUMENT and "outside" in msg, (kind, rc, msg)
        if not swap:
            rc, msg, _, _ = _normalize_call(dt, bad, n)
            assert rc == capi.RC_INVALID_ARGUMENT and "outside" in msg, msg
    # normalize_l2: an empty row among valid ones
    col = R.normalize_column(dt, 41)
    rows = list(col.rows)
    rows[37] = rows[37][:0]
    ce = R.Column(rows, dt, col.stores(), [(3 * i + 1) % 16 for i in range(col.n)])
    rc, msg, _, _ = _normalize_call(dt, ce, ce.n)
    assert rc != 0 and "empty" in msg, msg
    # the cell edges: a vector that ends at the area's end is good; one that ends a byte past it, or whose end wraps 32 bits, is not
    m = 40
    rng = np.random.default_rng(3)
    rows = [rng.standard_normal(8).astype(dt) for _ in range(m)]
    vals = [r.tobytes() for r in rows]
    qc, qa = varlena_bytes_column([vals[0]])

    def l2(cells, area, n=m, nulls=None, dev=None):
        res = np.full(n, SENT)
        xv = Vector(data=cells, area=area, length=n) if dev is None else Vector(data_ptr=dev.ptr, data_nbytes=dev.nbytes, area=area, length=n)
        rc, msg = xcall(FID[dt][R.L2SQ], [Vector(data=res, nulls=None if nulls is None else bitmap_from_bools(nulls), length=n), xv,
                                          Vector(data=qc, area=qa, length=n)], n, raise_on_error=False)
        return rc, msg, res

    def norm(cells, area, n=m, dev=None):
        oc, oa = np.zeros(24 * n, np.uint8), np.zeros(max(area.nbytes if area is not None else 0, 1), np.uint8)
        xv = Vector(data=cells, area=area, length=n) if dev is None else Vector(data_ptr=dev.ptr, data_nbytes=dev.nbytes, area=area, length=n)
        return xcall(NORM_FID[dt], [Vector(data=oc, area=oa, length=n), xv], n, raise_on_error=False)

    cells, area = varlena_bytes_column(vals)
    rc, msg, base = l2(cells, area)
    assert rc == 0, msg
    rc, msg, res = l2(*E.edges(vals, 5, None, None))
    assert rc == 0 and res[5] == base[-1] and (np.delete(res, 5) == np.delete(base, 5)).all(), msg
    assert norm(*E.edges(vals, 5, None, None))[0] == 0
    for past, wrap in ((6, None), (None, 7)):
        for rc, msg in (l2(*E.edges(vals, None, past, wrap))[:2], norm(*E.edges(vals, None, past, wrap))):
            assert rc == capi.RC_INVALID_ARGUMENT and "outside" in msg, (past, wrap, msg)
    nl = np.isin(np.arange(m), [6, 7])                              # bad cells in NULL rows are never read
    rc, msg, res = l2(*E.edges(vals, None, 6, 7), nulls=nl)
    assert rc == 0 and (res[nl] == SENT).all() and (res[~nl] == base[~nl]).all(), msg
    for rc, msg in (l2(cells, None)[:2], norm(cells, None)):       # non-inline cells without an area
        assert rc == capi.RC_INVALID_ARGUMENT and "outside" in msg, msg
    e, ea = E.edges(vals, 0, 1, None)                               # one cell: a const at len 2, a one-row column at len 1
    for k in (1, 2):
        rc, msg, res = l2(e[:24], ea, n=k)
        assert rc == 0 and (res == base[-1]).all(), msg
        assert norm(e[:24], ea, n=k)[0] == 0
        for rc, msg in (l2(e[24:48], ea, n=k)[:2], norm(e[24:48], ea, n=k)):
            assert rc == capi.RC_INVALID_ARGUMENT and "outside" in msg, (k, msg)
    for shift in E.SHIFTS:                                          # device cells 8-byte but not 16-byte aligned, and 1-byte misaligned
        for c, ok in ((cells, True), (E.edges(vals, None, 6, None)[0], False)):
            owner, dc = E.on_device(c, shift)
            rc, msg, res = l2(None, area, dev=dc)
            nrc, nmsg = norm(None, area, dev=dc)
            owner.free()
            if ok:
                assert rc == 0 and (res == base).all() and nrc == 0, (shift, msg, nmsg)
            else:
                assert rc == nrc == capi.RC_INVALID_ARGUMENT and "outside" in msg and "outside" in nmsg, (shift, msg, nmsg)
