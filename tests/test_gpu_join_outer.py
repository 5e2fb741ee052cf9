"""Right, full outer, right semi / anti and single hash joins on the device, each compared exactly with the host restatement of the
reference's probe loop, syncBitmap and finalize (join_outer_reference): pairs, matched bitmaps, finalize rows and SINGLE failures; plus SHUFFLE
with negative sels and a Q13-shaped right join end to end."""
import numpy as np
import pytest

import join_outer_reference as J
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, bitmap_to_bools, xcall

pytestmark = pytest.mark.gpu


def words_of(mask):
    return bitmap_from_bools(mask) if len(mask) else np.zeros(0, np.uint64)


def int_case(seed, nbuild, nprobe, card, unique=False, null_p=0.05):
    r = np.random.default_rng(seed)
    if unique:
        build = r.permutation(max(2 * nbuild, 2))[:nbuild].astype(np.uint64)
        bnull = np.zeros(nbuild, bool)
        probe = r.integers(0, max(3 * nbuild, 2), nprobe).astype(np.uint64)
    else:
        build = r.integers(0, card, nbuild).astype(np.uint64)
        bnull = r.random(nbuild) < null_p
        probe = r.integers(0, card + card // 4 + 1, nprobe).astype(np.uint64)
    return build, bnull, probe, r.random(nprobe) < null_p


def expected(build, bnull, probe, pnull, jt, matched=None):
    """(pairs, matched) from the restatement, or the SingleError it raises"""
    _, tk, off, sels = J.build_map(build, bnull)
    vals = J.find(tk, probe, pnull)
    m = np.zeros(len(build), bool) if matched is None else matched
    try:
        p, b = J.probe_fast(vals, off, sels, jt, m)
    except J.SingleError as e:
        return e, m
    return (p, b), m


def int_map(build, bnull, prepare=True):
    return ops.JoinMap(build, bitmap_from_bools(bnull) if bnull.any() else None, prepare=prepare)


def varchar_keys(keys, nulls):
    """keys as VARCHAR values (some longer than the 23 inline bytes), PACK_STR_KEYS'd: (bytes, offsets, skip)"""
    vals = [b"cust#%09d" % k + (b"-long-tail" * 2 if k % 3 == 0 else b"") for k in keys.tolist()]
    return ops.pack_str_keys([vals], [capi.T_VARCHAR], [bitmap_from_bools(nulls) if nulls.any() else None], has_null=False)


def probe_both(kind, build, bnull, probe, pnull, jt, matched, capacity=None):
    if kind == "int":
        jm = int_map(build, bnull)
        try:
            return jm.probe(probe, jt, bitmap_from_bools(pnull) if pnull.any() else None, capacity, matched), jm.hash_on_unique()
        finally:
            jm.release()
    bb, bo, bs = varchar_keys(build, bnull)
    pb, po, ps = varchar_keys(probe, pnull)
    jm = ops.StrJoinMap(bb, bo, bs)
    try:
        return jm.probe(pb, po, jt, ps, capacity, matched), jm.hash_on_unique()
    finally:
        jm.release()


def check_join(kind, build, bnull, probe, pnull, jt):
    want, wm = expected(build, bnull, probe, pnull, jt)
    matched = ops.matched_bitmap(len(build))
    if isinstance(want, J.SingleError):
        with pytest.raises(capi.MoError, match=J.SCALAR_SUBQUERY) as e:
            probe_both(kind, build, bnull, probe, pnull, jt, matched)
        row = want.probe_row if want.probe_row is not None else want.build_row
        assert e.value.rc == capi.RC_INTERNAL_ERROR and ("row %d)" % row) in str(e.value)
        return None
    (gp, gb), unique = probe_both(kind, build, bnull, probe, pnull, jt, matched)
    assert np.array_equal(gp, want[0]) and np.array_equal(gb, want[1])
    assert np.array_equal(bitmap_to_bools(matched, len(build)), wm)
    if jt in J.RIGHT_TYPES:
        assert np.array_equal(ops.join_build_rows(matched, len(build), jt), J.finalize(wm, jt))
    return unique


@pytest.mark.parametrize("jt", J.NEW_TYPES)
@pytest.mark.parametrize("shape", ["unique", "multi"])
@pytest.mark.parametrize("kind", ["int", "varchar"])
def test_every_type_matches_the_reference(gpu, kind, shape, jt):
    build, bnull, probe, pnull = int_case(jt * 7 + len(shape), 20_000, 50_000, 6000, unique=shape == "unique")
    unique = check_join(kind, build, bnull, probe, pnull, jt)
    assert unique in (None, shape == "unique")


@pytest.mark.parametrize("nbuild,nprobe,card,unique", [(1, 1, 1, False), (1, 1000, 1, False), (65, 1, 20, False), (1000, 1_000_000, 1000, False),
                                                       (3_000_000, 1_000_000, 0, True), (2_000_001, 1_000_000, 400_000, False)])
@pytest.mark.parametrize("jt", [capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_RIGHT_SEMI, capi.JOIN_RIGHT_ANTI])
def test_cardinalities(gpu, nbuild, nprobe, card, unique, jt):
    check_join("int", *int_case(nbuild + nprobe, nbuild, nprobe, card, unique), jt)


@pytest.mark.parametrize("jt", [capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_RIGHT_SEMI, capi.JOIN_RIGHT_ANTI, capi.JOIN_RIGHT_SINGLE])
def test_heavy_hitters_mark_by_warp(gpu, jt):
    """one group of 10^4 build rows and groups of 31, 32 and 33: marked by the whole warp (>= 32) or by its thread"""
    r = np.random.default_rng(jt)
    build = np.concatenate([np.full(10_000, 5), np.full(31, 6), np.full(32, 7), np.full(33, 8), r.integers(100, 5000, 20_000)]).astype(np.uint64)
    build = build[r.permutation(len(build))]
    bnull = r.random(len(build)) < 0.01
    probe = np.concatenate([np.array([5, 6, 7, 8, 9]), r.integers(100, 9000, 3000)]).astype(np.uint64)
    if jt == capi.JOIN_RIGHT_SINGLE:
        probe = np.array([5, 6, 7, 8, 9], np.uint64)                  # each heavy group once: no build row is matched twice
    check_join("int", build, bnull, probe, np.zeros(len(probe), bool), jt)


@pytest.mark.parametrize("jt", [capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_RIGHT_SINGLE])
def test_capacity_protocol_leaves_the_bitmap_alone(gpu, jt):
    build = np.arange(5000, dtype=np.uint64) // 2                       # two build rows per key
    probe = np.arange(0, 2500, 3, dtype=np.uint64)                      # each key once
    matched = ops.matched_bitmap(len(build))
    jm = int_map(build, np.zeros(5000, bool))
    with pytest.raises(capi.MoError) as e:
        jm.probe(probe, jt, capacity=10, matched=matched)
    assert e.value.rc == capi.RC_OUT_OF_RANGE and not matched.any()
    gp, gb = jm.probe(probe, jt, matched=matched)                       # repeated with the reported count: no false second match
    jm.release()
    (wp, wb), wm = expected(build, np.zeros(5000, bool), probe, np.zeros(len(probe), bool), jt)
    assert np.array_equal(gp, wp) and np.array_equal(gb, wb) and np.array_equal(bitmap_to_bools(matched, 5000), wm)


@pytest.mark.parametrize("nbatch", [1, 3, 17])
@pytest.mark.parametrize("jt", [capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_RIGHT_SEMI, capi.JOIN_RIGHT_SINGLE])
def test_one_bitmap_over_probe_batches(gpu, nbatch, jt):
    unique = jt == capi.JOIN_RIGHT_SINGLE
    build, bnull, probe, pnull = int_case(nbatch, 30_000, 0 if unique else 100_000, 8000, unique=unique)
    if unique:
        probe = np.random.default_rng(nbatch).permutation(60_000)[:25_000].astype(np.uint64)   # every build row matched at most once
        pnull = np.zeros(len(probe), bool)
    want, wm = expected(build, bnull, probe, pnull, jt)
    jm = int_map(build, bnull)
    matched = ops.matched_bitmap(len(build))
    cuts = np.linspace(0, len(probe), nbatch + 1).astype(int)
    gp, gb = [], []
    for a, z in zip(cuts[:-1], cuts[1:]):
        p, b = jm.probe(probe[a:z], jt, bitmap_from_bools(pnull[a:z]) if pnull[a:z].any() else None, matched=matched)
        gp.append(p + a); gb.append(b)
    jm.release()
    assert np.array_equal(np.concatenate(gp), want[0]) and np.array_equal(np.concatenate(gb), want[1])
    assert np.array_equal(bitmap_to_bools(matched, len(build)), wm)
    assert np.array_equal(ops.join_build_rows(matched, len(build), jt), J.finalize(wm, jt))


def test_left_single_names_the_lowest_offending_row(gpu):
    build = np.array([1, 2, 2, 3, 3, 4], np.uint64)
    probe = np.zeros(100_000, np.uint64) + 1
    probe[[70_000, 4321, 99_999]] = [2, 3, 2]
    jm = int_map(build, np.zeros(6, bool))
    with pytest.raises(capi.MoError, match=r"scalar subquery returns more than 1 row \(probe row 4321\)") as e:
        jm.probe(probe, capi.JOIN_SINGLE)
    assert e.value.rc == capi.RC_INTERNAL_ERROR
    gp, gb = jm.probe(np.array([1, 4, 9], np.uint64), capi.JOIN_SINGLE)
    assert gp.tolist() == [0, 1, 2] and gb.tolist() == [0, 5, -1]
    jm.release()


def test_right_single_fails_on_a_second_match(gpu):
    build = np.arange(1000, dtype=np.uint64)
    jm = int_map(build, np.zeros(1000, bool))
    single = capi.JOIN_RIGHT_SINGLE
    matched = ops.matched_bitmap(1000)
    with pytest.raises(capi.MoError, match=r"more than 1 row \(build row 17\)"):       # twice in one batch
        jm.probe(np.array([400, 17, 3, 17, 400], np.uint64), single, matched=matched)
    matched = ops.matched_bitmap(1000)
    jm.probe(np.array([5, 6], np.uint64), single, matched=matched)
    with pytest.raises(capi.MoError, match=r"more than 1 row \(build row 6\)"):        # in a later batch
        jm.probe(np.array([7, 6], np.uint64), single, matched=matched)
    wa, wb = ops.matched_bitmap(1000), ops.matched_bitmap(1000)             # two workers, each fine alone
    jm.probe(np.array([1, 2, 999], np.uint64), single, matched=wa)
    jm.probe(np.array([3, 999], np.uint64), single, matched=wb)
    with pytest.raises(capi.MoError, match=r"more than 1 row \(build row 999\)"):      # ... until their bitmaps merge
        ops.join_matched_merge([wa, wb], 1000, single)
    assert bitmap_to_bools(ops.join_matched_merge([wa, wb], 1000, capi.JOIN_RIGHT), 1000).nonzero()[0].tolist() == [1, 2, 3, 999]
    jm.release()


@pytest.mark.parametrize("n", [1, 2, 8])
@pytest.mark.parametrize("nbuild", [1, 63, 64, 65, 100_003])
def test_merge_and_build_rows(gpu, n, nbuild):
    r = np.random.default_rng(n * nbuild)
    masks = [r.random(nbuild) < 0.2 for _ in range(n)]
    for jt in J.RIGHT_TYPES:
        if jt == capi.JOIN_RIGHT_SINGLE and n > 1:
            continue
        want = J.sync_bitmap(masks, jt)
        got = ops.join_matched_merge([words_of(m) for m in masks], nbuild, jt)
        assert np.array_equal(bitmap_to_bools(got, nbuild), want)
        assert np.array_equal(ops.join_build_rows(got, nbuild, jt), J.finalize(want, jt))
    disjoint = [(np.arange(nbuild) % n) == k for k in range(n)]
    got = ops.join_matched_merge([words_of(m) for m in disjoint], nbuild, capi.JOIN_RIGHT_SINGLE)
    assert bitmap_to_bools(got, nbuild).all()


def test_bitmap_missing_short_or_past(gpu):
    jm = int_map(np.arange(200, dtype=np.uint64), np.zeros(200, bool))
    with pytest.raises(ValueError):
        jm.probe(np.arange(10, dtype=np.uint64), capi.JOIN_RIGHT)
    prm = np.array([capi.JOIN_RIGHT, 0], np.int32).view(np.uint8)
    base = [Vector(data=np.zeros(64, np.int64), length=64), Vector(data=np.zeros(64, np.int64), length=64), Vector(data=np.zeros(1, np.int64), length=1),
            Vector(data=prm, length=1), Vector(data=jm.table_keys, length=200), Vector(length=0), Vector(length=0),
            Vector(data=np.arange(10, dtype=np.uint64), length=10)]
    rc, msg = xcall(capi.XCALL_JOIN_PROBE, base + [Vector(length=0)], 10, raise_on_error=False)
    assert rc == capi.RC_INVALID_ARGUMENT and "matched bitmap" in msg
    rc, msg = xcall(capi.XCALL_JOIN_PROBE, base + [Vector(data=np.zeros(3, np.uint64), length=3)], 10, raise_on_error=False)
    assert rc == capi.RC_INVALID_ARGUMENT and "holds 192 rows" in msg
    jm.release()
    jm = int_map(np.arange(300, dtype=np.uint64) // 2, np.zeros(300, bool))   # with sels: a row past the bitmap is found on the device
    with pytest.raises(capi.MoError, match="build row 298 lies past the matched bitmap"):
        jm.probe(np.array([149], np.uint64), capi.JOIN_RIGHT_SEMI, matched=np.zeros(4, np.uint64))
    jm.release()
    matched = ops.matched_bitmap(2)                  # a group id above ngroups fails the call before it writes or marks anything
    with pytest.raises(capi.MoError, match="exceeds the group count"):
        ops.probe_gids(np.array([1, 2, 9], np.uint64), 2, None, None, capi.JOIN_RIGHT, matched=matched)
    assert not matched.any()


def test_device_pointers(gpu):
    """JOIN_PROBE_GIDS, JOIN_MATCHED_MERGE and JOIN_BUILD_ROWS on resident buffers give the host forms' results"""
    build, bnull, probe, pnull = int_case(3, 50_000, 200_000, 20_000)
    jm = int_map(build, bnull)
    vals = jm.find(probe, bitmap_from_bools(pnull))
    nb = len(build)
    words = (nb + 63) // 64
    halves = [(0, 120_000), (120_000, len(probe))]
    host_maps = []
    dev = {k: DeviceBuffer.from_numpy(v) for k, v in (("off", jm.offsets), ("sels", jm.sels))}
    dmaps = [DeviceBuffer.from_numpy(np.zeros(words, np.uint64)) for _ in halves]
    for (a, z), dm in zip(halves, dmaps):
        hm = ops.matched_bitmap(nb)
        hp, hb = ops.probe_gids(vals[a:z], jm.ngroups, jm.offsets, jm.sels, capi.JOIN_FULL, matched=hm)
        host_maps.append(hm)
        dv = DeviceBuffer.from_numpy(vals[a:z])
        op, ob, cnt = DeviceBuffer(8 * len(hp) + 8), DeviceBuffer(8 * len(hp) + 8), DeviceBuffer(8)
        ops.probe_gids_device(dv, z - a, jm.ngroups, dev["off"], dev["sels"], capi.JOIN_FULL, op, ob, cnt, dm)
        c = int(cnt.to_numpy(np.int64)[0])
        assert c == len(hp) and np.array_equal(op.to_numpy(np.int64, c), hp) and np.array_equal(ob.to_numpy(np.int64, c), hb)
        assert np.array_equal(dm.to_numpy(np.uint64), hm)
        for b in (dv, op, ob, cnt):
            b.free()
    merged = ops.join_matched_merge(host_maps, nb, capi.JOIN_FULL)
    ops.join_matched_merge_device(dmaps[0], dmaps, nb, capi.JOIN_FULL)          # in place into the first input
    rows = ops.join_build_rows(merged, nb, capi.JOIN_FULL)
    dsels, dcnt = DeviceBuffer(8 * nb), DeviceBuffer(8)
    ops.join_build_rows_device(dmaps[0], nb, capi.JOIN_FULL, dsels.ptr, dcnt.ptr)
    capi.check(gpu.MoB200_Sync(), gpu)
    assert np.array_equal(dmaps[0].to_numpy(np.uint64), merged)
    c = int(dcnt.to_numpy(np.int64)[0])
    assert np.array_equal(dsels.to_numpy(np.int64, c), rows)
    assert np.array_equal(rows, J.finalize(J.sync_bitmap([bitmap_to_bools(m, nb) for m in host_maps], capi.JOIN_FULL), capi.JOIN_FULL))
    for b in list(dev.values()) + dmaps + [dsels, dcnt]:
        b.free()
    jm.release()


# ---- the asynchronous form: merge (not RIGHT SINGLE) and build rows only enqueue with device pointers
from test_gpu_async_forms import Arg, Case, forms, run, stream  # noqa: E402,F401


def async_cases():
    r = np.random.default_rng(11)
    nb = 70_001
    w = (nb + 63) // 64
    maps = [words_of(r.random(nb) < 0.3) for _ in range(3)]
    prm = lambda jt: Arg(np.array([jt, 0], np.int32), host=True)   # noqa: E731
    merge = Case(capi.XCALL_JOIN_MATCHED_MERGE, [Arg(np.full(w, 7, np.uint64)), Arg(np.array([3], np.int32), host=True), prm(capi.JOIN_FULL)]
                 + [Arg(m) for m in maps], nb)
    rows = int((~bitmap_to_bools(maps[0], nb)).sum())
    build_rows = Case(capi.XCALL_JOIN_BUILD_ROWS, [Arg(np.full(rows, -1, np.int64)), Arg(np.full(1, -1, np.int64)), Arg(maps[0]), prm(capi.JOIN_RIGHT_ANTI)], nb)
    return {"merge": merge, "build_rows": build_rows}


@pytest.mark.parametrize("name", ["merge", "build_rows"])
def test_async_forms(gpu, stream, name):
    case = async_cases()[name]
    want = None
    for label, host in forms(case):
        rc, idle, out = run(gpu, case, host, stream)
        assert rc == 0, (label, capi.last_error(gpu))
        if host:
            assert idle, "%s: returned before its stream ran" % label
        else:
            assert not idle, "the all-device call waited for its stream"
        want = want or out
        for slot in want:
            assert out[slot] == want[slot], (label, slot)


# ---- SHUFFLE with negative sels: the NULL row of an outer join's missing side
@pytest.mark.parametrize("sz", [1, 2, 4, 8, 16, 24])
@pytest.mark.parametrize("src_nulls", [False, True])
def test_shuffle_negative_sels_gather_null_rows(gpu, sz, src_nulls):
    r = np.random.default_rng(sz)
    n, m = 10_000, 7_777
    src = r.integers(1, 256, (n, sz)).astype(np.uint8)
    if sz == 24:                                                       # varlena cells: inline values of 1..23 bytes
        src[:, 0] = r.integers(1, 24, n)
    snull = r.random(n) < 0.2 if src_nulls else np.zeros(n, bool)
    sels = r.integers(0, n, m).astype(np.int64)
    neg = r.random(m) < 0.3
    sels[neg] = -1
    want = np.where(neg[:, None], 0, src[np.maximum(sels, 0)]).astype(np.uint8)
    wnull = neg | (snull[np.maximum(sels, 0)] & ~neg)
    for with_dst_nulls in (True, False):
        dst = np.full((m, sz), 0xcd, np.uint8)
        dn = np.full((m + 63) // 64, 0xffff, np.uint64) if with_dst_nulls else None
        sv = Vector(data=src.reshape(-1), nulls=bitmap_from_bools(snull) if src_nulls else None, length=n)
        xcall(capi.XCALL_SHUFFLE(sz), [Vector(data=dst.reshape(-1), nulls=dn, length=m), sv, Vector(data=sels, length=m)], m)
        assert np.array_equal(dst, want)
        if with_dst_nulls:
            assert np.array_equal(dn, bitmap_from_bools(wnull))


# ---- Q13 shape: customer LEFT OUTER JOIN orders, run as a RIGHT join with customer as the build side
def test_q13_customer_left_outer_join_orders_as_a_right_join(gpu):
    """select c_count, count(*) from (select c_custkey, count(o_orderkey) c_count from customer left outer join orders on c_custkey = o_custkey
    group by c_custkey) group by c_count: GROUP_IDS + JOIN_SELS (JoinMap), JOIN_PROBE (RIGHT) over order batches, JOIN_BUILD_ROWS, SHUFFLE with -1
    for the orders side of unmatched customers, and a grouped COUNT(o_orderkey)"""
    r = np.random.default_rng(13)
    ncust, nord = 150_000, 1_500_000
    c_custkey = (r.permutation(ncust) + 1).astype(np.uint64)
    # about a third of the customers place no order (TPC-H: custkey % 3 == 0)
    buyers = c_custkey[c_custkey % 3 != 0]
    o_custkey = buyers[r.integers(0, len(buyers), nord)].astype(np.uint64)
    o_orderkey = (np.arange(nord, dtype=np.int64) * 4 + 1)
    jm = ops.JoinMap(c_custkey)
    assert jm.hash_on_unique()
    matched = ops.matched_bitmap(ncust)
    probe_rows, build_rows = [], []
    for a in range(0, nord, 400_000):                                  # order batches
        p, b = jm.probe(o_custkey[a:a + 400_000], capi.JOIN_RIGHT, matched=matched)
        probe_rows.append(p + a); build_rows.append(b)
    unmatched = ops.join_build_rows(matched, ncust, capi.JOIN_RIGHT)
    jm.release()
    o_sels = np.concatenate(probe_rows + [np.full(len(unmatched), -1, np.int64)])
    c_sels = np.concatenate(build_rows + [unmatched])
    okey, onull = ops.shuffle(o_orderkey, o_sels, want_nulls=True)
    ckey = ops.shuffle(c_custkey, c_sels)
    tab = ops.GroupTable(ncust)
    gids = tab.insert(ckey)
    ngroups = int(tab.ngroups[0])
    c_count = np.zeros(ngroups, np.int64)
    assert ops.group_agg(capi.AGG_COUNT, capi.T_INT64, c_count, None, None, gids, okey, onull, len(gids)) == 0
    got = dict(zip(*np.unique(c_count, return_counts=True)))
    per_cust = np.bincount(o_custkey.astype(np.int64), minlength=ncust + 1)[c_custkey.astype(np.int64)]
    want = dict(zip(*np.unique(per_cust, return_counts=True)))
    assert ngroups == ncust and got == want and want[0] == (c_custkey % 3 == 0).sum()
