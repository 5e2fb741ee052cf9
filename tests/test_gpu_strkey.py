"""Byte-string keys on the device (PACK_STR_KEYS, STR_GROUP_IDS, STR_JOIN_FIND, JOIN_PROBE_GIDS) through the C-ABI, exactly against the
StrHashMap restatement (strkey_reference.py) and, for joins, the oracle's restatement of GroupSels.Finalize and the probe emission loop."""
import ctypes as C

import numpy as np
import pytest

import cell_edges as E
import oracle_lib as O
import strkey_reference as R
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, varlena_bytes_column, xcall

pytestmark = pytest.mark.gpu

FIXED = [(capi.T_BOOL, np.uint8), (capi.T_INT8, np.int8), (capi.T_INT16, np.int16), (capi.T_INT32, np.int32), (capi.T_INT64, np.int64),
         (capi.T_UINT8, np.uint8), (capi.T_UINT16, np.uint16), (capi.T_UINT32, np.uint32), (capi.T_UINT64, np.uint64), (capi.T_FLOAT32, np.float32),
         (capi.T_FLOAT64, np.float64), (capi.T_DATE, np.int32), (capi.T_TIME, np.int64), (capi.T_DATETIME, np.int64), (capi.T_TIMESTAMP, np.int64),
         (capi.T_DECIMAL64, np.int64), (capi.T_DECIMAL128, None), (capi.T_BIT, np.uint64), (capi.T_YEAR, np.int16), (capi.T_ENUM, np.uint16),
         (capi.T_UUID, None)]


@pytest.fixture(params=[0, 1, 4, 16], ids=lambda b: "hash_bits%d" % b)
def hash_bits(request, gpu):
    """strkey_hash_bits: 0 = the full hash; 1, 4, 16 make hash tags collide so that the byte compare decides"""
    assert gpu.MoB200_SetTuning(b"strkey_hash_bits", request.param) == 0
    yield request.param
    gpu.MoB200_SetTuning(b"strkey_hash_bits", 0)


def _values(rng, n, lens=(0, 1, 2, 7, 8, 22, 23, 24, 25, 40, 100)):
    out = []
    for i in range(n):
        ln = lens[rng.integers(len(lens))]
        v = bytes(rng.integers(0, 4, ln, dtype=np.uint8))          # many embedded zero bytes, many equal values
        out.append(v)
    return out


def _fixed(rng, T, dt, n):
    if dt is None:
        return rng.integers(0, 3, (n, 2), dtype=np.uint64)
    if np.dtype(dt).kind == "f":
        return rng.choice(np.array([-0.0, 0.0, 1.5, np.nan], dt), n)
    return rng.integers(0, 3, n).astype(dt)


def _nulls(rng, n, p):
    return rng.random(n) < p


def _pack_check(cols, types, nulls, has_null, n):
    got_b, got_o, skip = ops.pack_str_keys(cols, types, [bitmap_from_bools(x) if x is not None else None for x in nulls], has_null, length=n)
    keys = R.encode_keys(cols, types, nulls, has_null, n)
    want_b, want_o = R.flat(keys)
    assert (got_o == want_o).all()
    assert got_b.tobytes() == want_b.tobytes()
    if not has_null:
        assert (skip == bitmap_from_bools([k is None for k in keys])).all()
    return keys, got_b, got_o, skip


@pytest.mark.parametrize("has_null", [False, True])
def test_pack_every_type_both_null_modes(gpu, has_null):
    rng = np.random.default_rng(11 + has_null)
    n = 3000
    for chunk in range(0, len(FIXED), 6):
        part = FIXED[chunk:chunk + 6]
        cols = [_fixed(rng, T, dt, n) for T, dt in part] + [_values(rng, n)]
        types = [T for T, _ in part] + [(capi.T_VARCHAR, capi.T_TEXT, capi.T_CHAR, capi.T_BLOB)[chunk // 6]]
        nulls = [_nulls(rng, n, 0.1) for _ in cols]
        _pack_check(cols, types, nulls, has_null, n)


@pytest.mark.parametrize("has_null", [False, True])
def test_pack_const_columns_and_cell_forms(gpu, has_null):
    rng = np.random.default_rng(3)
    n = 500
    vals = [b"", b"\x00", b"x" * 23, b"y" * 24, b"\x00" * 30, b"z" * 65535] + _values(rng, n - 6)
    for ctypes_ in ([capi.T_BINARY, capi.T_VARBINARY], [capi.T_DATALINK, capi.T_TEXT]):
        cols = [np.array([42], np.int64), [b"const value longer than twenty-three"], vals, [b"short"]]
        types = [capi.T_INT64] + ctypes_ + [capi.T_VARCHAR]
        for const_null in (False, True):
            nulls = [[const_null], None, _nulls(rng, n, 0.2), [False]]
            _pack_check(cols, types, nulls, has_null, n)


def test_pack_errors(gpu):
    n = 10
    vals = [b"value %02d " % i * 4 for i in range(n)]          # 36 bytes: area cells
    prm = ops._params_vec(ops._strkey_params([capi.T_INT32, capi.T_VARCHAR], True))
    cells, area = varlena_bytes_column(vals)
    col0 = np.arange(n, dtype=np.int32)
    # capacity: MO_RC_OUT_OF_RANGE with offsets[len] = the bytes needed
    want_b, want_o = R.flat(R.encode_keys([col0, vals], [capi.T_INT32, capi.T_VARCHAR], None, True))
    out, off = np.zeros(5, np.uint8), np.zeros(n + 1, np.uint64)
    rc, msg = xcall(capi.XCALL_PACK_STR_KEYS, [Vector(data=out), Vector(data=off, length=n), prm, Vector(data=col0), Vector(data=cells, area=area, length=n)], n,
                    raise_on_error=False)
    assert rc == capi.RC_OUT_OF_RANGE and int(off[n]) == len(want_b)
    # a cell pointing outside its area: the column and its lowest bad row
    bad = cells.copy().reshape(n, 24)
    for r in (7, 9):
        bad[r].view(np.uint32)[1] = 10_000
    with pytest.raises(capi.MoError, match="column 1 row 7"):
        ops.pack_str_keys([col0, (bad.reshape(-1), area)], [capi.T_INT32, capi.T_VARCHAR])
    with pytest.raises(capi.MoError, match="column 0 has a 65536-byte value"):
        ops.pack_str_keys([[b"a", b"b" * 65536]], [capi.T_TEXT])
    with pytest.raises(capi.MoError, match="unsupported type"):
        ops.pack_str_keys([np.zeros(3, np.int64)], [999])
    # the cell edges: a value that ends at the area's end is good; one that ends a byte past it, or whose end wraps 32 bits, is not
    types = [capi.T_INT32, capi.T_VARCHAR]
    want = ops.pack_str_keys([col0, vals[:2] + [vals[-1]] + vals[3:]], types)
    got = ops.pack_str_keys([col0, E.edges(vals, 2, None, None)], types)
    assert got[0].tobytes() == want[0].tobytes() and (got[1] == want[1]).all()
    for past, wrap, row in ((5, None, 5), (None, 4, 4), (6, 3, 3)):
        with pytest.raises(capi.MoError, match="column 1 row %d" % row):
            ops.pack_str_keys([col0, E.edges(vals, None, past, wrap)], types)
    nm = bitmap_from_bools(np.isin(np.arange(n), [3, 6]))          # bad cells in NULL rows are never read
    got = ops.pack_str_keys([col0, E.edges(vals, None, 6, 3)], types, [None, nm])
    want = ops.pack_str_keys([col0, vals], types, [None, nm])
    assert got[0].tobytes() == want[0].tobytes()
    with pytest.raises(capi.MoError, match="column 1 row 0"):      # non-inline cells without an area
        ops.pack_str_keys([col0, (cells, None)], types)
    # one cell: a const column at len 2, a one-row column at len 1
    e, ea = E.edges(vals, 0, 1, None)
    for m in (1, 2):
        got = ops.pack_str_keys([(e[:24], ea)], [capi.T_VARCHAR], length=m)
        want = ops.pack_str_keys([[vals[-1]] * m], [capi.T_VARCHAR], length=m)
        assert got[0].tobytes() == want[0].tobytes() and (got[1] == want[1]).all()
        with pytest.raises(capi.MoError, match="column 0 row 0"):
            ops.pack_str_keys([(e[24:48], ea)], [capi.T_VARCHAR], length=m)
    # device cells 8-byte but not 16-byte aligned, and 1-byte misaligned
    want = ops.pack_str_keys([vals], [capi.T_VARCHAR])
    darea = DeviceBuffer.from_numpy(area)
    for shift in E.SHIFTS:
        for c, bad_row in ((cells, None), (E.edges(vals, None, 7, None)[0], 7)):
            owner, dc = E.on_device(c, shift)
            db, do = DeviceBuffer(4096), DeviceBuffer(8 * (n + 1))
            if bad_row is None:
                ops.pack_str_keys_device([(dc, darea)], None, [capi.T_VARCHAR], n, db, do)
                assert db.to_numpy(np.uint8)[:len(want[0])].tobytes() == want[0].tobytes(), shift
                assert (do.to_numpy(np.uint64, n + 1) == want[1]).all(), shift
            else:
                with pytest.raises(capi.MoError, match="column 0 row 7"):
                    ops.pack_str_keys_device([(dc, darea)], None, [capi.T_VARCHAR], n, db, do)
            for b in (owner, db, do):
                b.free()
    darea.free()


def _names(ids):
    return [b"Customer#%09d" % i for i in ids]


def _check_groups(tab, table, got, want):
    assert (got == want).all()
    wb, wo = R.table_bytes(table)
    g = int(tab.ngroups[0])
    assert g == len(table)
    assert (tab.offsets[:g + 1] == wo).all() and tab.bytes[:int(wo[-1])].tobytes() == wb.tobytes()


@pytest.mark.parametrize("ngroups", [1, 10, 1000, 100_000, 1_000_000])
def test_group_ids_customer_names(gpu, ngroups):
    rng = np.random.default_rng(ngroups)
    n = max(2 * ngroups, 1000)
    ids = rng.integers(0, ngroups, n)
    ids[:ngroups] = rng.permutation(ngroups)[:min(ngroups, n)]
    rng.shuffle(ids)
    vals = _names(ids)
    kb, ko, _ = ops.pack_str_keys([vals], [capi.T_VARCHAR])
    keys = [b"\x00\x12\x00" + v for v in vals]
    assert kb.tobytes() == b"".join(keys)
    table = {}
    want = R.insert(table, keys)
    tab = ops.StrGroupTable(16, 64)                     # grows on the capacity error
    got, first = tab.insert(kb, ko, first_rows=True)
    _check_groups(tab, table, got, want)
    assert (first == _first_rows(keys, table)).all()


def _first_rows(keys, table):
    first = {}
    for i, k in enumerate(keys):
        if k is not None:
            first.setdefault(k, i)
    return np.array([first[k] for k in sorted(table, key=table.get)], np.int64)


def test_group_ids_over_many_calls_equal_one_call(gpu, hash_bits):
    rng = np.random.default_rng(7)
    n = 20_000 if hash_bits in (0, 16) else 3000
    vals = _values(rng, n, lens=(0, 3, 23, 24, 30))
    nulls = _nulls(rng, n, 0.05)
    for has_null in (False, True):
        keys = R.encode_keys([vals, rng.integers(0, 2, n).astype(np.int16)], [capi.T_VARCHAR, capi.T_INT16], [nulls, None], has_null)
        kb, ko = R.flat(keys)
        skip = None if has_null else bitmap_from_bools([k is None for k in keys])
        table = {}
        want = R.insert(table, keys)
        one = ops.StrGroupTable(n, max(len(kb), 1))
        _check_groups(one, table, one.insert(kb, ko, skip), want)
        many = ops.StrGroupTable(4, 16)
        got, s = [], 0
        while s < n:
            e = min(n, s + int(rng.integers(1, 2000)))
            sub_o = ko[s:e + 1] - ko[s]
            sub_skip = None if has_null else bitmap_from_bools([k is None for k in keys[s:e]])
            got.append(many.insert(kb[int(ko[s]):int(ko[e])], sub_o, sub_skip))
            s = e
        _check_groups(many, table, np.concatenate(got), want)
        probe = R.encode_keys([_values(rng, 500, lens=(0, 3, 23)), np.zeros(1, np.int16)], [capi.T_VARCHAR, capi.T_INT16], None, has_null, 500)
        pb, po = R.flat(probe)
        jm = ops.StrJoinMap(kb, ko, skip, prepare=False)
        assert (jm.find(pb, po) == R.find(table, probe)).all()


def test_distinct_keys_and_nulls(gpu, hash_bits):
    f = np.array([-0.0, 0.0, np.nan, 0.0, -0.0, np.nan, np.nan], np.float64)
    f[6] = np.frombuffer(np.uint64(0x7ff8000000000001).tobytes(), np.float64)[0]
    cases = [([f], [capi.T_FLOAT64], None),
             ([[b"a", b"ab", b"a", b"ab"], [b"bc", b"c", b"bc", b"c"]], [capi.T_VARCHAR, capi.T_VARCHAR], None),
             ([np.array([5, 5, 6, 7, 6], np.int64), [b"k", b"k", b"k", b"k", b"k"]], [capi.T_INT64, capi.T_CHAR], [[True, False, True, False, True], None])]
    for cols, types, nulls in cases:
        for has_null in (False, True):
            keys, kb, ko, skip = _pack_check(cols, types, nulls or [None] * len(cols), has_null, len(cols[0]))
            table = {}
            want = R.insert(table, keys)
            tab = ops.StrGroupTable()
            _check_groups(tab, table, tab.insert(kb, ko, skip), want)
    assert len(set(R.encode_keys(cases[0][0], cases[0][1], None, True))) == 4


def test_table_full_leaves_the_table_untouched(gpu, hash_bits):
    keys = [b"k%d" % i for i in range(100)]
    kb, ko = R.flat(keys)
    tab = ops.StrGroupTable(200, 4096)
    tab.insert(kb[:int(ko[50])], ko[:51])
    more = [b"new%d" % i for i in range(100)]
    mb, mo = R.flat(more)
    for cap_groups, cap_bytes in ((120, 4096), (200, int(tab.offsets[50]) + 10)):
        groups = np.zeros(100, np.uint64)
        tb, to = tab.bytes[:cap_bytes].copy(), tab.offsets[:cap_groups + 1].copy()
        ng = tab.ngroups.copy()
        rc, msg = xcall(capi.XCALL_STR_GROUP_IDS, [Vector(data=groups), Vector(data=ng, length=1), Vector(data=tb), Vector(data=to), Vector(data=mb),
                                                   Vector(data=mo, length=100), Vector(length=0)], 100, raise_on_error=False)
        assert rc == capi.RC_INVALID_ARGUMENT and "need 150 groups and %d bytes" % (int(tab.offsets[50]) + len(mb)) in msg, msg
        assert int(ng[0]) == 50 and (to == tab.offsets[:cap_groups + 1]).all() and (tb == tab.bytes[:cap_bytes]).all()


def test_device_form(gpu, hash_bits):
    rng = np.random.default_rng(5)
    n, card = (50_000, 5000) if hash_bits in (0, 16) else (5000, 500)
    vals = _names(rng.integers(0, card, n))
    a = rng.integers(0, 3, n).astype(np.int64)
    nl = _nulls(rng, n, 0.01)
    keys = R.encode_keys([vals, a], [capi.T_VARCHAR, capi.T_INT64], [None, nl], True)
    wb, wo = R.flat(keys)
    cells, area = varlena_bytes_column(vals)
    dc, da, dcol, dn = DeviceBuffer.from_numpy(cells), DeviceBuffer.from_numpy(area), DeviceBuffer.from_numpy(a), DeviceBuffer.from_numpy(bitmap_from_bools(nl))
    db, do = DeviceBuffer(len(wb) + 100), DeviceBuffer(8 * (n + 1))
    ops.pack_str_keys_device([(dc, da), dcol], [None, dn], [capi.T_VARCHAR, capi.T_INT64], n, db, do)
    assert (do.to_numpy(np.uint64) == wo).all() and db.to_numpy(np.uint8)[:len(wb)].tobytes() == wb.tobytes()
    table = {}
    want = R.insert(table, keys)
    tbw, tow = R.table_bytes(table)
    dg, dng, dtb, dto, dfr = DeviceBuffer(8 * n), DeviceBuffer.from_numpy(np.zeros(1, np.int64)), DeviceBuffer(len(tbw) + 64), DeviceBuffer.from_numpy(np.zeros(n + 1, np.uint64)), DeviceBuffer(8 * n)
    ops.StrGroupTable().insert_device(db.view(len(wb)), do, n, dg, dng, dtb, dto, dfr)
    assert (dg.to_numpy(np.uint64) == want).all() and int(dng.to_numpy(np.int64)[0]) == len(table)
    assert (dto.to_numpy(np.uint64)[:len(table) + 1] == tow).all() and dtb.to_numpy(np.uint8)[:len(tbw)].tobytes() == tbw.tobytes()
    assert (dfr.to_numpy(np.int64)[:len(table)] == _first_rows(keys, table)).all()
    # STR_JOIN_FIND with device pointers only enqueues; prepared by the table offsets pointer or rebuilt
    dv = DeviceBuffer(8 * n)
    for prepared in (False, True):
        if prepared:
            capi.check(gpu.MoB200_StrJoinMapPrepare(C.c_void_p(dtb.ptr), C.c_void_p(dto.ptr), len(table)), gpu)
        gpu.MoB200_Memset(C.c_void_p(dv.ptr), 0xff, 8 * n)
        ops.str_join_find_device(dv, n, len(table), dtb.view(len(tbw)), dto, db.view(len(wb)), do)
        capi.check(gpu.MoB200_Sync(), gpu)
        assert (dv.to_numpy(np.uint64) == want).all()
    gpu.MoB200_JoinMapRelease(C.c_void_p(dto.ptr))


def test_device_table_with_host_ngroups_over_batches(gpu, hash_bits):
    """device key / table buffers with a host ngroups: every call must hand the new group count back, so batches continue the numbering"""
    rng = np.random.default_rng(9)
    n = 4000
    keys = [b"\x00" + bytes(v) for v in _values(rng, n, lens=(1, 5, 23, 30))]
    table = {}
    want = R.insert(table, keys)
    tbw, tow = R.table_bytes(table)
    ng = np.zeros(1, np.int64)
    dtb, dto = DeviceBuffer(len(tbw) + 64), DeviceBuffer.from_numpy(np.zeros(n + 1, np.uint64))
    got = []
    for s, e in ((0, 1700), (1700, n)):
        kb, ko = R.flat(keys[s:e])
        db, do, dg = DeviceBuffer.from_numpy(kb), DeviceBuffer.from_numpy(ko), DeviceBuffer(8 * (e - s))
        ops.StrGroupTable().insert_device(db, do, e - s, dg, ng, dtb, dto)
        assert int(ng[0]) == len(set(keys[:e]))
        got.append(dg.to_numpy(np.uint64))
    assert (np.concatenate(got) == want).all() and int(ng[0]) == len(table)
    assert (dto.to_numpy(np.uint64)[:len(table) + 1] == tow).all() and dtb.to_numpy(np.uint8)[:len(tbw)].tobytes() == tbw.tobytes()


def test_host_offsets_past_their_bytes_are_refused(gpu):
    kb, ko = R.flat([b"abc", b"defg"])
    bad = ko.copy(); bad[-1] = 100
    with pytest.raises(capi.MoError, match="key offsets end at 100"):
        ops.StrGroupTable().insert(kb, bad)
    jm = ops.StrJoinMap(kb, ko, prepare=False)
    with pytest.raises(capi.MoError, match="probe key offsets end past the key bytes"):
        jm.find(kb, bad)


def _oracle_pairs(ids, ng, vals, jt):
    nbuild, nprobe = len(ids), len(vals)
    offsets = np.zeros(ng + 2, np.int32); sels = np.zeros(max(nbuild, 1), np.int32)
    m = O.go().og_join_sels(O.p(ids), nbuild, ng, O.p(offsets), O.p(sels))
    unique = ng == nbuild
    cap = nprobe + 4 * nprobe + 4 * nbuild + 1024
    while True:
        op, ob = np.zeros(cap, np.int64), np.zeros(cap, np.int64)
        r = O.go().og_join_probe(O.p(vals), nprobe, None if unique else O.p(offsets), None if unique else O.p(sels), jt, O.p(op), O.p(ob), cap)
        if r <= cap:
            return offsets, sels[:m], op[:r], ob[:r]
        cap = r


@pytest.mark.parametrize("jt", [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI])
@pytest.mark.parametrize("shape", ["varchar", "int64_pair"])
def test_string_join_matches_the_oracle(gpu, jt, shape, hash_bits):
    rng = np.random.default_rng(jt * 10 + len(shape))
    nbuild, nprobe, card = (60_000, 80_000, 9000) if hash_bits in (0, 16) else (6000, 8000, 600)
    if shape == "varchar":
        pool = [bytes(v) for v in _values(rng, card, lens=(0, 5, 23, 24, 31))]
        bsel, psel = rng.integers(0, card, nbuild), rng.integers(0, 2 * card, nprobe)
        bcols, pcols = [[pool[i] for i in bsel]], [[pool[i] if i < card else b"absent%d" % i for i in psel]]
        types = [capi.T_VARCHAR]
    else:
        a, b = rng.integers(0, 100, card), rng.integers(0, 100, card)
        bsel, psel = rng.integers(0, card, nbuild), rng.integers(0, card, nprobe)
        bcols, pcols = [a[bsel], b[bsel]], [a[psel], b[psel] + (rng.random(nprobe) < 0.3) * 1000]
        types = [capi.T_INT64, capi.T_INT64]
    bnull, pnull = _nulls(rng, nbuild, 0.03), _nulls(rng, nprobe, 0.03)
    bkeys = R.encode_keys(bcols, types, [bnull] + [None] * (len(types) - 1), False)
    pkeys = R.encode_keys(pcols, types, [pnull] + [None] * (len(types) - 1), False)
    table = {}
    ids = R.insert(table, bkeys)
    vals = R.find(table, pkeys)
    offsets, sels, op, ob = _oracle_pairs(ids, len(table), vals, jt)
    bb, bo, bskip = ops.pack_str_keys(bcols, types, [bitmap_from_bools(bnull)] + [None] * (len(types) - 1), has_null=False)
    pb, po, pskip = ops.pack_str_keys(pcols, types, [bitmap_from_bools(pnull)] + [None] * (len(types) - 1), has_null=False)
    for prepare in (False, True):
        jm = ops.StrJoinMap(bb, bo, bskip, prepare=prepare)
        assert jm.ngroups == len(table) and not jm.hash_on_unique()
        assert (jm.offsets == offsets).all() and (jm.sels == sels).all()
        assert (jm.find(pb, po, pskip) == vals).all()
        gp, gb = jm.probe(pb, po, jt, pskip)
        assert (gp == op).all() and (gb == ob).all()
        jm.release()


@pytest.mark.parametrize("jt", [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI])
def test_probe_gids_equals_join_probe(gpu, jt):
    rng = np.random.default_rng(jt)
    for nbuild, card in ((5000, 5000), (50_000, 700)):
        pool = rng.integers(0, 1 << 62, card, dtype=np.uint64)
        build = rng.permutation(pool) if card == nbuild else pool[rng.integers(0, card, nbuild)]
        probe = np.where(rng.random(30_000) < 0.5, pool[rng.integers(0, card, 30_000)], np.uint64(7)).astype(np.uint64)
        pn = bitmap_from_bools(_nulls(rng, 30_000, 0.05))
        jm = ops.JoinMap(build, prepare=False)
        want_p, want_b = jm.probe(probe, jt, pn)
        got_p, got_b = ops.probe_gids(jm.find(probe, pn), jm.ngroups, jm.offsets, jm.sels, jt)
        assert got_p.tobytes() == want_p.tobytes() and got_b.tobytes() == want_b.tobytes()
        # the form on resident vectors gives the same pairs
        vals = jm.find(probe, pn)
        dp, dbld, dc = DeviceBuffer(8 * len(want_p)), DeviceBuffer(8 * len(want_p)), DeviceBuffer(8)
        ops.probe_gids_device(DeviceBuffer.from_numpy(vals), len(vals), jm.ngroups, DeviceBuffer.from_numpy(jm.offsets) if jm.offsets is not None else None,
                              DeviceBuffer.from_numpy(jm.sels) if jm.sels is not None else None, jt, dp, dbld, dc)
        assert int(dc.to_numpy(np.int64)[0]) == len(want_p)
        assert dp.to_numpy(np.int64).tobytes() == want_p.tobytes() and dbld.to_numpy(np.int64).tobytes() == want_b.tobytes()
    with pytest.raises(capi.MoError, match="exceeds the group count"):
        ops.probe_gids(np.array([1, 2, 9], np.uint64), 2, None, None, jt)
