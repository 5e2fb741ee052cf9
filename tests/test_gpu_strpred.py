"""MO_XCALL_GO_COMPARE over the varlena types and MO_XCALL_GO_LIKE against the host restatement (tests/like_reference.py), exactly: every
row's null bit, and the value of every row that is not NULL.  Columns mix inline and non-inline values, empty values, embedded zero bytes,
multi-byte and invalid UTF-8 and 1 KB values; operands are const or columns, with NULLs, a const NULL and pre-set result null bits."""
import numpy as np
import pytest

from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, bitmap_to_bools, varlena_bytes_column, xcall

import cell_edges as E
import like_reference as L

pytestmark = pytest.mark.gpu

ALPHABET = [b"a", b"b", b"c", b"%", b"_", b"\\", b"\x00", b"\n", "é".encode(), "中".encode(), "\U0001F600".encode(), b"\xff",
            b"\xc3", b"\xed\xa0\x80", "�".encode()]


def rand_value(rng):
    k = rng.integers(0, 10)
    if k == 0:
        return b""
    if k == 1:                                       # a 1 KB TEXT value
        return bytes(rng.integers(0, 256, 1024, dtype=np.uint8))
    if k <= 3:                                       # around the inline limit (23 bytes)
        return b"".join(ALPHABET[j] for j in rng.integers(0, 3, rng.integers(20, 27)))
    if k == 4:
        return b"special pending " + b"x" * int(rng.integers(0, 200)) + b" requests accounts"
    return b"".join(ALPHABET[j] for j in rng.integers(0, len(ALPHABET), rng.integers(1, 12)))


def column(rng, n):
    return [rand_value(rng) for _ in range(n)]


def nulls(rng, n, p):
    return rng.random(n) < p


def check(got, gnulls, want, wnulls):
    assert list(gnulls) == list(wnulls)
    bad = [i for i, v in want.items() if bool(got[i]) != v]
    assert not bad, "rows %s differ" % bad[:10]


# every tier-A rule and quirk, and tier-B patterns with `_` next to multi-byte runes
CONST_PATTERNS = [b"", b"%", b"_", b"a", b"\xc3", b"abc", b"_bc", b"%bc", b"ab_", b"ab%", b"%b%", b"%b_", b"_b%", b"%%", b"%_", b"_%",
                  b"%pending%accounts%", b"%special%requests%", b"%a%%b%", b"%a\\b%c%", b"\\%", b"a\\_", b"ab\\", b"%\\%", b"\\%%",
                  b"%\\%%a%", b"_a_", b"%a_b%", "_é%".encode(), "%é_".encode(), "é_".encode(), "%中_%".encode(), b"a\xff_",
                  b"%\\_%", b"___", b"%\x00%", b"%\n%", b"x" * 30 + b"%", b"%" + b"x" * 40]


@pytest.mark.parametrize("pat", CONST_PATTERNS)
def test_like_const_pattern(pat):
    rng = np.random.default_rng(len(pat) * 7919 + sum(pat))
    n = 3000
    vals = column(rng, n)
    vn, skip = nulls(rng, n, 0.1), nulls(rng, n, 0.1)
    got, gn = ops.like(vals, pat, col_nulls=bitmap_from_bools(vn), rnulls=bitmap_from_bools(skip))
    want, wn = L.like_column(vals, [pat], True, vnulls=vn, skip=skip)
    check(got, gn, want, wn)


def test_like_column_pattern():
    rng = np.random.default_rng(1)
    n = 4000
    vals = column(rng, n)
    pats = [b"".join(ALPHABET[j] for j in rng.integers(0, len(ALPHABET), rng.integers(0, 6))) for _ in range(n)]
    for i in range(0, n, 3):                         # make matches likely: a pattern cut from its own value, with `_` on a rune
        v = vals[i].decode("utf-8", "replace")[:8]
        pats[i] = ("%" + v[1:3] + "_%").encode() if len(v) > 3 else b"%"
    vn, pn, skip = nulls(rng, n, 0.1), nulls(rng, n, 0.1), nulls(rng, n, 0.05)
    got, gn = ops.like(vals, pats, col_nulls=bitmap_from_bools(vn), pattern_nulls=bitmap_from_bools(pn), rnulls=bitmap_from_bools(skip))
    want, wn = L.like_column(vals, pats, False, vnulls=vn, pnulls=pn, skip=skip)
    check(got, gn, want, wn)
    assert 0 < sum(want.values()) < len(want)


def test_like_const_subject_column_pattern():
    rng = np.random.default_rng(2)
    n = 500
    pats = [b"".join(ALPHABET[j] for j in rng.integers(0, 6, rng.integers(0, 5))) for _ in range(n)]
    got, gn = ops.like(["aé%b".encode()], pats)
    want, wn = L.like_column(["aé%b".encode()] * n, pats, False)
    check(got, gn, want, wn)


def test_like_const_null_pattern_and_subject():
    rng = np.random.default_rng(3)
    n = 300
    vals = column(rng, n)
    got, gn = ops.like(vals, b"%a%", pattern_nulls=np.array([1], np.uint64))
    assert gn.all()
    got, gn = ops.like([b"abc"], [b"a%"] * n, col_nulls=np.array([1], np.uint64))
    assert gn.all()


STR_TYPES = [capi.T_CHAR, capi.T_VARCHAR, capi.T_BINARY, capi.T_VARBINARY, capi.T_BLOB, capi.T_TEXT, capi.T_DATALINK]


@pytest.mark.parametrize("T", STR_TYPES)
@pytest.mark.parametrize("op", range(6))
def test_compare(op, T):
    rng = np.random.default_rng(op * 100 + T)
    n = 2000
    a = column(rng, n)
    b = [a[i] if rng.random() < 0.3 else (a[i][:-1] if a[i] and rng.random() < 0.3 else rand_value(rng)) for i in range(n)]
    an, bn, skip = nulls(rng, n, 0.1), nulls(rng, n, 0.1), nulls(rng, n, 0.1)
    got, gn = ops.str_compare(op, T, a, b, a_nulls=bitmap_from_bools(an), b_nulls=bitmap_from_bools(bn), rnulls=bitmap_from_bools(skip))
    wn = an | bn | skip
    want = {i: L.compare(op, a[i], b[i]) for i in range(n) if not wn[i]}
    check(got, gn, want, wn)
    for cst, col in ((a[7], b), (b"abc\x00", a)):   # const on either side
        g1, n1 = ops.str_compare(op, T, [cst], col)
        check(g1, n1, {i: L.compare(op, cst, col[i]) for i in range(n)}, [False] * n)
        g2, n2 = ops.str_compare(op, T, col, [cst])
        check(g2, n2, {i: L.compare(op, col[i], cst) for i in range(n)}, [False] * n)
    g3, n3 = ops.str_compare(op, T, a, [b"x"], b_nulls=np.array([1], np.uint64))
    assert n3.all()


def test_fixed_width_compare_launches_unchanged():
    """fixed-width GO_COMPARE runs its own two kernels (null merge, compare) exactly as before; a string compare or LIKE is one kernel"""
    lib = capi.load_library()
    a = np.arange(1000, dtype=np.int64)
    for T, dt in ((capi.T_INT64, np.int64), (capi.T_INT32, np.int32), (capi.T_FLOAT64, np.float64)):
        x, y = a.astype(dt), a[::-1].astype(dt)
        r, rn = np.zeros(1000, np.uint8), np.zeros(16, np.uint64)
        c0 = lib.MoB200_KernelLaunchCount()
        xcall(capi.XCALL_GO_COMPARE(capi.CMP_LT, T), [Vector(data=r, nulls=rn, length=1000), Vector(data=x), Vector(data=y)], 1000)
        assert lib.MoB200_KernelLaunchCount() - c0 == 2
        assert (r.astype(bool) == (x < y)).all()
    vals = [b"a", b"bb" * 20]
    c0 = lib.MoB200_KernelLaunchCount()
    ops.str_compare(capi.CMP_EQ, capi.T_VARCHAR, vals, vals)
    ops.like(vals, b"%b%")
    assert lib.MoB200_KernelLaunchCount() - c0 == 2


def _dev_pair(values):
    cells, area = varlena_bytes_column(values)
    return DeviceBuffer.from_numpy(cells), (DeviceBuffer.from_numpy(area) if area.size else None)


@pytest.mark.parametrize("pat", [b"%pending%accounts%", b"%a_b%", b"ab%"])
def test_device_forms(pat):
    """resident operands: the result equals the host form's, and the call is one kernel launch.  With the const pattern in host memory the
    call's only synchronise is its status read-back; a device-resident const pattern is copied back first (its null word, its cell and, for
    a long pattern, its bytes), each copy a synchronise of its own, as a device parameter block is.  The synchronise count itself is not
    observable through the ABI and is not asserted here."""
    rng = np.random.default_rng(5)
    n = 5000
    vals = column(rng, n)
    vn, skip = nulls(rng, n, 0.1), nulls(rng, n, 0.1)
    want, wn = ops.like(vals, pat, col_nulls=bitmap_from_bools(vn), rnulls=bitmap_from_bools(skip))
    col = _dev_pair(vals)
    vnd = DeviceBuffer.from_numpy(bitmap_from_bools(vn))
    out, outn = DeviceBuffer(n), DeviceBuffer.from_numpy(bitmap_from_bools(skip))
    lib = capi.load_library()
    for p in (varlena_bytes_column([pat]), _dev_pair([pat])):
        c0 = lib.MoB200_KernelLaunchCount()
        ops.like_device(col, p, n, out, outn, col_nulls=vnd)
        assert lib.MoB200_KernelLaunchCount() - c0 == 1
        capi.check(lib.MoB200_Sync(), lib)
        gn = bitmap_to_bools(outn.to_numpy(np.uint64), n)
        assert (gn == wn).all()
        g = out.to_numpy(np.uint8).astype(bool)
        assert (g[~wn] == want[~wn]).all()
        outn = DeviceBuffer.from_numpy(bitmap_from_bools(skip))
    b = [v[::-1] for v in vals]
    wc, wcn = ops.str_compare(capi.CMP_GE, capi.T_TEXT, vals, b)
    out2, out2n = DeviceBuffer(n), DeviceBuffer.from_numpy(np.zeros((n + 63) // 64, np.uint64))
    ops.str_compare_device(capi.CMP_GE, capi.T_TEXT, col, _dev_pair(b), n, out2, out2n)
    capi.check(lib.MoB200_Sync(), lib)
    assert not bitmap_to_bools(out2n.to_numpy(np.uint64), n).any()
    assert (out2.to_numpy(np.uint8).astype(bool) == wc).all()


def _bad_cells(values, rows):
    cells, area = varlena_bytes_column(values)
    c = cells.reshape(-1, 24).copy()
    for r in rows:
        u32 = c[r].view(np.uint32)
        u32[0], u32[1], u32[2] = 0xFFFFFFFF, area.size, 5      # points past the end of the area
    return c.reshape(-1), area


def test_bad_cell_named_at_lowest_row():
    n = 200
    vals = [b"x" * 30] * n
    bad = _bad_cells(vals, [3, 17, 40])
    vn = np.zeros(n, bool); vn[3] = True                         # a NULL row's cell is never read
    with pytest.raises(capi.MoError, match="operand 1 row 17"):
        ops.like(bad, b"%x%", col_nulls=bitmap_from_bools(vn))
    with pytest.raises(capi.MoError, match="operand 2 row 17"):
        ops.str_compare(capi.CMP_EQ, capi.T_VARCHAR, vals, bad, a_nulls=bitmap_from_bools(vn))
    with pytest.raises(capi.MoError, match="operand 2 row 3"):
        ops.like(vals, bad)
    skip = np.zeros(n, bool); skip[[3, 17, 40]] = True            # skipped rows are not read either
    got, gn = ops.like(bad, b"%x%", rnulls=bitmap_from_bools(skip))
    assert (gn == skip).all() and got[~skip].all()
    # the cell rule's edges: a value that ends at the area's end is good, one whose end wraps 32 bits is not
    cells, area = varlena_bytes_column(vals)
    e = cells.reshape(n, 24).copy()
    u = e.view(np.uint32)
    u[17, 1], u[17, 2] = area.size - 30, 30
    got, _ = ops.str_compare(capi.CMP_EQ, capi.T_VARCHAR, vals, (e.reshape(-1), area))
    assert got.all()
    u[5, 1], u[5, 2] = 0xFFFFFFF0, 0x20
    with pytest.raises(capi.MoError, match="operand 2 row 5"):
        ops.str_compare(capi.CMP_EQ, capi.T_VARCHAR, vals, (e.reshape(-1), area))
    # a const pattern's cell, read on the host: ending at the area's end is good; a byte past it, a 32-bit wrap or no area is not
    pats = [b"%" + b"y" * 30 + b"%", b"%" + b"x" * 28 + b"%"]
    pe, pa = E.edges(pats, 0, 1, None)
    pw, pwa = E.edges(pats, None, None, 0)
    for k in (n, 1):                                              # a const at len n; at len 1 the one cell is a column
        got, _ = ops.like(vals[:k], (pe[:24], pa), length=k)
        assert got.all()
        for bad_pat in ((pe[24:48], pa), (pw[:24], pwa), (pe[:24], None)):
            with pytest.raises(capi.MoError, match="operand 2 row 0"):
                ops.like(vals[:k], bad_pat, length=k)
    got, gn = ops.like(vals, (pe[24:48], pa), pattern_nulls=np.array([1], np.uint64))   # a const NULL pattern's cell is never read
    assert gn.all()
    # device cells 8-byte but not 16-byte aligned (three 8-byte loads), and 1-byte misaligned (byte loads)
    b = [v[::-1] + b"!" for v in vals]
    want, _ = ops.str_compare(capi.CMP_LT, capi.T_TEXT, vals, b)
    bc, ba = varlena_bytes_column(b)
    dbc, dba, darea = DeviceBuffer.from_numpy(bc), DeviceBuffer.from_numpy(ba), DeviceBuffer.from_numpy(area)
    for shift in E.SHIFTS:
        for c, bad_row in ((cells, None), (E.edges(vals, None, 17, 40)[0], 17)):
            owner, dc = E.on_device(c, shift)
            out, outn = DeviceBuffer(n), DeviceBuffer.from_numpy(np.zeros((n + 63) // 64, np.uint64))
            if bad_row is None:
                ops.str_compare_device(capi.CMP_LT, capi.T_TEXT, (dc, darea), (dbc, dba), n, out, outn)
                assert (out.to_numpy(np.uint8).astype(bool) == want).all(), shift
            else:
                with pytest.raises(capi.MoError, match="operand 1 row 17"):
                    ops.str_compare_device(capi.CMP_LT, capi.T_TEXT, (dc, darea), (dbc, dba), n, out, outn)
            for x in (owner, out, outn):
                x.free()
    for x in (dbc, dba, darea):
        x.free()


def test_in_and_not_in_through_the_string_map():
    """IN / NOT IN over strings needs no entry point: PACK_STR_KEYS of the tuple -> STR_GROUP_IDS, then STR_JOIN_FIND of the column; a row is
    IN the tuple exactly when its id is not 0, and a NULL row keeps its bit in the pack's skip bitmap.  Restates opOperatorStrIn.operatorIn /
    operatorNotIn (operator_in.go:147-193): NULL -> NULL, else membership in the tuple's set (NOT IN: its negation)."""
    rng = np.random.default_rng(9)
    tuple_vals = list({rand_value(rng) for _ in range(40)}) + [b"", b"x" * 300]
    n = 3000
    col = [tuple_vals[rng.integers(0, len(tuple_vals))] if rng.random() < 0.4 else rand_value(rng) for _ in range(n)]
    cn = nulls(rng, n, 0.1)
    tb, to, _ = ops.pack_str_keys([tuple_vals], [capi.T_VARCHAR], has_null=False)
    m = ops.StrJoinMap(tb, to)
    kb, ko, skip = ops.pack_str_keys([col], [capi.T_VARCHAR], nulls=[bitmap_from_bools(cn)], has_null=False)
    vals = m.find(kb, ko, nulls=skip)
    m.release()
    got_null = bitmap_to_bools(skip, n)
    s = set(tuple_vals)
    assert (got_null == cn).all()
    for i in range(n):
        if not cn[i]:
            assert (vals[i] != 0) == (col[i] in s)          # IN; NOT IN is its negation with the same nulls


def test_one_row_batch_reads_the_pattern_as_a_column():
    """With len == 1 a 24-byte pattern operand cannot be told from a one-row column (Vector.FillRawPtrLen gives both the same dataSz), so
    GO_LIKE reads it as a column: rune level.  Go's likeFn asks IsConst() and applies optimizeRuleForLike; where the two tiers disagree a
    one-row batch with a const pattern differs from the reference, e.g. 'é' LIKE '_' (false there, one byte; true here, one rune).  With two
    or more rows the same pattern is const and byte level."""
    for v, pat in (("é".encode(), b"_"), (b"%", b"\\%"), ("xé".encode(), b"%\xc3_"), (b"xa\\bxc", b"%a\\b%c%")):
        assert L.like(v, pat, pat_const=True) != L.like(v, pat, pat_const=False)
        got, gn = ops.like([v], [pat], length=1)
        assert not gn[0] and bool(got[0]) == L.like(v, pat, pat_const=False)
        got, gn = ops.like([v, v], pat)
        assert not gn.any() and got.tolist() == [L.like(v, pat, pat_const=True)] * 2
