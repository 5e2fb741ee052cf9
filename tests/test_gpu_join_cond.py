"""Hash joins with a non-equality condition on the device: JOIN_COND over the INNER candidate pairs of JOIN_PROBE / STR_JOIN_FIND +
JOIN_PROBE_GIDS, compared exactly with the host restatement of the reference's probe loop (join_cond_reference): pairs, order, matched bitmaps,
finalize rows, SINGLE failures and malformed candidates; plus TPC-H Q21's EXISTS / NOT EXISTS subqueries end to end on the reference's rows."""
import json
import os

import numpy as np
import pytest

import join_cond_reference as C
import join_outer_reference as J
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, bitmap_to_bools, xcall

pytestmark = pytest.mark.gpu

ALL_TYPES = tuple(J.FLAVOUR)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CMP_EQ, CMP_NE, CMP_GT = 0, 1, 2


def words_of(mask):
    return bitmap_from_bools(mask) if len(mask) else np.zeros(0, np.uint64)


def expected(cp, cb, cond, null, nprobe, jt, matched):
    try:
        return C.probe_fast(cp, cb, cond, null, nprobe, jt, matched)
    except J.SingleError as e:
        return e


def check(cp, cb, cond, null, nprobe, jt, nbuild, matched=None, wm=None):
    """JOIN_COND against the restatement; `matched` / `wm` carry a bitmap across batches.  Returns the pairs (None after a SINGLE failure)."""
    wm = np.zeros(nbuild, bool) if wm is None else wm
    matched = (ops.matched_bitmap(nbuild) if jt in J.RIGHT_TYPES else None) if matched is None else matched
    want = expected(cp, cb, cond, null, nprobe, jt, wm)
    cn = words_of(null) if null is not None and null.any() else None
    if isinstance(want, J.SingleError):
        with pytest.raises(capi.MoError, match=J.SCALAR_SUBQUERY) as e:
            ops.join_cond(cp, cb, cond, nprobe, jt, cn, matched=matched)
        row = want.probe_row if want.probe_row is not None else want.build_row
        assert e.value.rc == capi.RC_INTERNAL_ERROR and ("row %d)" % row) in str(e.value), (str(e.value), row)
        return None
    gp, gb = ops.join_cond(cp, cb, cond, nprobe, jt, cn, matched=matched)
    assert np.array_equal(gp, want[0]) and np.array_equal(gb, want[1]), jt
    if matched is not None:
        assert np.array_equal(bitmap_to_bools(matched, nbuild), wm)
    return gp, gb


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


def varchar_keys(keys, nulls):
    vals = [b"ord#%09d" % k + (b"-long-tail" * 2 if k % 3 == 0 else b"") for k in keys.tolist()]
    return ops.pack_str_keys([vals], [capi.T_VARCHAR], [bitmap_from_bools(nulls) if nulls.any() else None], has_null=False)


class Map:
    """the build side as a JoinMap (8-byte keys) or a StrJoinMap (VARCHAR keys); probe(..) = JOIN_PROBE or STR_JOIN_FIND + JOIN_PROBE_GIDS"""

    def __init__(self, kind, build, bnull):
        self.kind = kind
        if kind == "int":
            self.m = ops.JoinMap(build, bitmap_from_bools(bnull) if bnull.any() else None)
        else:
            bb, bo, bs = varchar_keys(build, bnull)
            self.m = ops.StrJoinMap(bb, bo, bs)

    def probe(self, keys, pnull, jt=capi.JOIN_INNER, matched=None):
        if self.kind == "int":
            return self.m.probe(keys, jt, bitmap_from_bools(pnull) if pnull.any() else None, matched=matched)
        pb, po, ps = varchar_keys(keys, pnull)
        return self.m.probe(pb, po, jt, ps, matched=matched)

    def release(self):
        self.m.release()


@pytest.mark.parametrize("jt", ALL_TYPES)
@pytest.mark.parametrize("shape", ["unique", "multi"])
@pytest.mark.parametrize("kind", ["int", "varchar"])
def test_every_type_matches_the_reference(gpu, kind, shape, jt):
    """pass rates 0, 1 %, 50 % and 100 %, with and without NULLs in the condition; the always-true condition equals JOIN_PROBE of the type"""
    build, bnull, probe, pnull = int_case(jt * 5 + len(shape), 20_000, 50_000, 6000, unique=shape == "unique")
    jm = Map(kind, build, bnull)
    try:
        cp, cb = jm.probe(probe, pnull)
        assert jm.m.hash_on_unique() == (shape == "unique") and len(cp) > 10_000
        r = np.random.default_rng(jt)
        for rate in (0.0, 0.01, 0.5, 1.0):
            cond = r.random(len(cp)) < rate
            for with_nulls in (False, True):
                null = (r.random(len(cp)) < 0.2) if with_nulls else None
                got = check(cp, cb, cond, null, len(probe), jt, len(build))
                if rate == 1.0 and not with_nulls:
                    matched = ops.matched_bitmap(len(build)) if jt in J.RIGHT_TYPES else None
                    try:
                        want = jm.probe(probe, pnull, jt, matched)
                    except capi.MoError:
                        assert got is None
                        continue
                    assert got is not None and got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    finally:
        jm.release()


@pytest.mark.parametrize("jt", ALL_TYPES)
def test_rows_without_candidates_and_empty_batches(gpu, jt):
    nb = 40
    # probe rows 0, 1 (start), 5..7 (middle) and 10, 11 (end) have no candidates
    cp = np.array([2, 2, 3, 4, 4, 4, 8, 9, 9], np.int64)
    cb = np.array([0, 7, 3, 1, 2, 39, 5, 6, 8], np.int64)
    for cond in (np.ones(9, bool), np.array([0, 1, 1, 0, 1, 0, 0, 1, 0], bool), np.zeros(9, bool)):
        check(cp, cb, cond, None, 12, jt, nb)
        check(cp, cb, cond, np.arange(9) % 4 == 1, 12, jt, nb)
    e = np.zeros(0, np.int64)
    for nprobe in (0, 1, 1000):                                       # npairs = 0; len = 0
        got = check(e, e, np.zeros(0, bool), None, nprobe, jt, nb)
        assert len(got[0]) == (nprobe if jt in (capi.JOIN_LEFT, capi.JOIN_ANTI, capi.JOIN_SINGLE, capi.JOIN_FULL) else 0)


@pytest.mark.parametrize("jt", ALL_TYPES)
@pytest.mark.parametrize("rate", [0.01, 0.5, 1.0])
def test_heavy_rows_and_warp_edges(gpu, jt, rate):
    """a probe row with 10^5 + 17 candidates and rows with exactly 31, 32 and 33: walked by the whole warp (>= 32) or by its thread"""
    r = np.random.default_rng(jt)
    build = np.concatenate([np.full(100_017, 5), np.full(31, 6), np.full(32, 7), np.full(33, 8), r.integers(100, 3000, 20_000)]).astype(np.uint64)
    build = build[r.permutation(len(build))]
    probe = np.concatenate([np.array([9, 5, 6, 7, 8]), r.integers(100, 6000, 3000), np.array([7, 6, 5])]).astype(np.uint64)
    jm = Map("int", build, np.zeros(len(build), bool))
    cp, cb = jm.probe(probe, np.zeros(len(probe), bool))
    jm.release()
    assert np.bincount(cp)[1:5].tolist() == [100_017, 31, 32, 33]
    cond = r.random(len(cp)) < rate
    if jt == capi.JOIN_SINGLE:                                        # the lowest probe row with two passing pairs is named
        assert check(cp, cb, cond, None, len(probe), jt, len(build)) is None
        cond[cp != 2] = False
        cond[cp == 2] = np.arange(31) == 17                           # ... and one passing pair out of 31 is fine
    check(cp, cb, cond, r.random(len(cp)) < 0.1, len(probe), jt, len(build))


@pytest.mark.parametrize("jt", [capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_RIGHT_SINGLE, capi.JOIN_INNER])
def test_capacity_protocol_leaves_the_bitmap_alone(gpu, jt):
    build = np.arange(5000, dtype=np.uint64) // 2
    probe = np.arange(0, 2500, 3, dtype=np.uint64)
    jm = Map("int", build, np.zeros(5000, bool))
    cp, cb = jm.probe(probe, np.zeros(len(probe), bool))
    jm.release()
    cond = (cb % 2 == 0) | (cp % 5 == 0)
    matched = ops.matched_bitmap(5000) if jt in J.RIGHT_TYPES else None
    with pytest.raises(capi.MoError, match="exceed the output capacity") as e:
        ops.join_cond(cp, cb, cond, len(probe), jt, capacity=10, matched=matched)
    assert e.value.rc == capi.RC_OUT_OF_RANGE and (matched is None or not matched.any())
    op, ob, cnt = np.zeros(10, np.int64), np.zeros(10, np.int64), np.zeros(1, np.int64)
    prm = np.array([jt, 0], np.int32).view(np.uint8)
    vecs = [Vector(data=op, length=10), Vector(data=ob, length=10), Vector(data=cnt, length=1), Vector(data=prm, length=1), Vector(data=cp, length=len(cp)),
            Vector(data=cb, length=len(cb)), Vector(data=cond.view(np.uint8), length=len(cp))] + ([Vector(data=matched, length=len(matched))] if matched is not None else [])
    rc, _ = xcall(capi.XCALL_JOIN_COND, vecs, len(probe), raise_on_error=False)
    want = expected(cp, cb, cond, None, len(probe), jt, np.zeros(5000, bool))
    assert rc == capi.RC_OUT_OF_RANGE and int(cnt[0]) == len(want[0]) and (matched is None or not matched.any())
    check(cp, cb, cond, None, len(probe), jt, 5000, matched)                # the repeat with room: no false second match


@pytest.mark.parametrize("nbatch", [1, 3, 17])
@pytest.mark.parametrize("jt", [capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_RIGHT_SEMI, capi.JOIN_RIGHT_ANTI, capi.JOIN_RIGHT_SINGLE])
def test_one_bitmap_over_probe_batches(gpu, nbatch, jt):
    """one bitmap over the batches, then JOIN_MATCHED_MERGE of two workers' bitmaps and JOIN_BUILD_ROWS"""
    single = jt == capi.JOIN_RIGHT_SINGLE
    build, bnull, probe, pnull = int_case(nbatch, 30_000, 100_000, 8000)
    if single:                                                        # every build row a candidate of at most one probe row
        probe = np.random.default_rng(nbatch).permutation(8000)[:6000].astype(np.uint64)
        build, bnull, pnull = np.arange(30_000, dtype=np.uint64), np.zeros(30_000, bool), np.zeros(6000, bool)
    jm = Map("int", build, bnull)
    nb = len(build)
    r = np.random.default_rng(nbatch + jt)
    shared, workers, wm = ops.matched_bitmap(nb), [ops.matched_bitmap(nb), ops.matched_bitmap(nb)], np.zeros(nb, bool)
    gp, gb, whole = [], [], []
    cuts = np.linspace(0, len(probe), nbatch + 1).astype(int)
    for i, (a, z) in enumerate(zip(cuts[:-1], cuts[1:])):
        cp, cb = jm.probe(probe[a:z], pnull[a:z])
        cond, null = r.random(len(cp)) < 0.4, r.random(len(cp)) < 0.1
        p, b = check(cp, cb, cond, null, z - a, jt, nb, shared, wm)
        ops.join_cond(cp, cb, cond, z - a, jt, words_of(null), matched=workers[i % 2])
        gp.append(p + a); gb.append(b); whole.append((cp + a, cb, cond, null))
    jm.release()
    cp, cb, cond, null = (np.concatenate([w[k] for w in whole]) for k in range(4))
    want = C.probe_fast(cp, cb, cond, null, len(probe), jt, np.zeros(nb, bool))
    assert np.array_equal(np.concatenate(gp), want[0]) and np.array_equal(np.concatenate(gb), want[1])
    merged = ops.join_matched_merge(workers, nb, jt)
    assert np.array_equal(merged, shared)
    assert np.array_equal(ops.join_build_rows(merged, nb, jt), J.finalize(wm, jt))


def test_left_single_fails_only_when_two_pairs_pass(gpu):
    cp = np.array([0, 0, 0, 1, 1, 3, 3, 3, 3], np.int64)
    cb = np.array([4, 5, 6, 1, 2, 7, 8, 9, 3], np.int64)
    cond = np.array([0, 1, 0, 1, 0, 0, 0, 1, 0], bool)                # at most one passing pair per row: fine
    p, b = ops.join_cond(cp, cb, cond, 5, capi.JOIN_SINGLE)
    assert p.tolist() == [0, 1, 2, 3, 4] and b.tolist() == [5, 1, -1, 9, -1]
    cond[[0, 8]] = True                                               # rows 0 and 3 now have two
    with pytest.raises(capi.MoError, match=r"more than 1 row \(probe row 0\)"):
        ops.join_cond(cp, cb, cond, 5, capi.JOIN_SINGLE)
    cond[0] = False
    with pytest.raises(capi.MoError, match=r"more than 1 row \(probe row 3\)"):
        ops.join_cond(cp, cb, cond, 5, capi.JOIN_SINGLE)


def test_right_single_fails_on_a_second_passing_match(gpu):
    single = capi.JOIN_RIGHT_SINGLE
    cp = np.array([0, 0, 1, 2, 2], np.int64)
    cb = np.array([17, 3, 17, 400, 3], np.int64)
    m = ops.matched_bitmap(1000)
    ops.join_cond(cp, cb, np.array([1, 0, 0, 1, 1], bool), 3, single, matched=m)            # 17 and 3 each pass once
    assert np.flatnonzero(bitmap_to_bools(m, 1000)).tolist() == [3, 17, 400]
    m = ops.matched_bitmap(1000)
    with pytest.raises(capi.MoError, match=r"more than 1 row \(build row 3\)"):                # twice in one batch
        ops.join_cond(cp, cb, np.array([1, 1, 1, 0, 1], bool), 3, single, matched=m)
    m = ops.matched_bitmap(1000)
    ops.join_cond(cp[:2], cb[:2], np.array([0, 1], bool), 1, single, matched=m)
    with pytest.raises(capi.MoError, match=r"more than 1 row \(build row 3\)"):                # in a later batch
        ops.join_cond(cp[3:] - 2, cb[3:], np.array([0, 1], bool), 1, single, matched=m)


def test_malformed_candidates(gpu):
    def rc_msg(cp, cb, nprobe, jt=capi.JOIN_INNER, matched=None, ncond=None):
        cp, cb = np.array(cp, np.int64), np.array(cb, np.int64)
        cond = np.ones(len(cp) if ncond is None else ncond, np.uint8)
        vecs = [Vector(data=np.zeros(64, np.int64), length=64), Vector(data=np.zeros(64, np.int64), length=64), Vector(data=np.zeros(1, np.int64), length=1),
                Vector(data=np.array([jt, 0], np.int32).view(np.uint8), length=1), Vector(data=cp, length=len(cp)), Vector(data=cb, length=len(cb)),
                Vector(data=cond, length=len(cond))] + ([Vector(data=matched, length=len(matched))] if matched is not None else [])
        return xcall(capi.XCALL_JOIN_COND, vecs, nprobe, raise_on_error=False)

    assert rc_msg([0, 1, 1, 2], [0, 1, 2, 3], 3) == (0, "")
    for cp, cb, nprobe, pos in (([0, 1, 1, 0, 2], [0] * 5, 3, 3),             # unsorted probe rows
                                ([0, 1, 5], [0] * 3, 3, 2),                    # a probe row >= len
                                ([0, 1, 1], [0, -1, 2], 3, 1),                 # a negative build row
                                ([-1, 0], [0, 0], 3, 0),                       # a negative probe row
                                ([0, 2, 1, 9], [0] * 4, 3, 2),                 # the lowest of two
                                ([0, 0], [1, 1], 0, 0)):                       # len = 0
        rc, msg = rc_msg(cp, cb, nprobe)
        assert rc == capi.RC_INVALID_ARGUMENT and ("candidate %d is malformed" % pos) in msg, (cp, msg)
    rc, msg = rc_msg([0, 1, 2], [0, 200, 3], 3, capi.JOIN_RIGHT, np.zeros(1, np.uint64))   # a build row past the bitmap
    assert rc == capi.RC_INVALID_ARGUMENT and "build row 200 lies past the matched bitmap" in msg
    rc, msg = rc_msg([0, 1, 2], [0, 1, 2], 3, capi.JOIN_RIGHT_SEMI, np.zeros(0, np.uint64))
    assert rc == capi.RC_INVALID_ARGUMENT and "matched bitmap" in msg
    rc, msg = rc_msg([0, 1, 2], [0, 1, 2], 3, ncond=2)                               # a short condition
    assert rc == capi.RC_INVALID_ARGUMENT and "buffers too small" in msg
    with pytest.raises(ValueError):
        ops.join_cond([0], [0], [True], 1, capi.JOIN_RIGHT)


@pytest.mark.parametrize("jt", [capi.JOIN_SEMI, capi.JOIN_FULL, capi.JOIN_RIGHT_ANTI])
def test_device_pointers(gpu, jt):
    """join_cond_device on resident candidates, condition, outputs and bitmap gives the host form's result"""
    build, bnull, probe, pnull = int_case(jt, 50_000, 200_000, 20_000)
    jm = Map("int", build, bnull)
    cp, cb = jm.probe(probe, pnull)
    jm.release()
    r = np.random.default_rng(jt)
    cond, null = r.random(len(cp)) < 0.3, r.random(len(cp)) < 0.1
    nb = len(build)
    hm = ops.matched_bitmap(nb)
    hp, hb = ops.join_cond(cp, cb, cond, len(probe), jt, words_of(null), matched=hm if jt in J.RIGHT_TYPES else None)
    dev = [DeviceBuffer.from_numpy(x) for x in (cp, cb, cond.view(np.uint8), words_of(null), np.zeros((nb + 63) // 64, np.uint64))]
    op, ob, cnt = DeviceBuffer(8 * len(hp) + 8), DeviceBuffer(8 * len(hp) + 8), DeviceBuffer(8)
    ops.join_cond_device(*dev[:4], len(cp), len(probe), jt, op, ob, cnt, dev[4] if jt in J.RIGHT_TYPES else None)
    c = int(cnt.to_numpy(np.int64)[0])
    assert c == len(hp) and np.array_equal(op.to_numpy(np.int64, c), hp) and np.array_equal(ob.to_numpy(np.int64, c), hb)
    if jt in J.RIGHT_TYPES:
        assert np.array_equal(dev[4].to_numpy(np.uint64), hm) and hm.any()
    small = DeviceBuffer(8)
    if len(hp) > 1:
        with pytest.raises(capi.MoError) as e:
            ops.join_cond_device(*dev[:4], len(cp), len(probe), jt, small, small, cnt, dev[4] if jt in J.RIGHT_TYPES else None)
        assert e.value.rc == capi.RC_OUT_OF_RANGE and int(cnt.to_numpy(np.int64)[0]) == len(hp)
    for b in dev + [op, ob, cnt, small]:
        b.free()


# ---- TPC-H Q21 on the reference's rows: the EXISTS / NOT EXISTS subqueries as SEMI / ANTI joins with l2.l_suppkey <> l1.l_suppkey
def q21_rows():
    d = json.load(open(os.path.join(GOLDEN, "tpch_q21.json")))
    assert d["counts"] == {"lineitem": 6005, "orders": 1500, "supplier": 10, "nation": 25}
    return d


def go_compare(op, T, a, b):
    """GO_COMPARE(op, T) of two columns (b may be a 1-element const): (bool, null words)"""
    n = len(a)
    out, on = np.zeros(n, np.uint8), np.zeros((n + 63) // 64, np.uint64)
    xcall(capi.XCALL_GO_COMPARE(op, T), [Vector(data=out, nulls=on, length=n), Vector(data=a, length=n), Vector(data=b, length=n)], n)
    return out, on


def subquery(kind, probe_keys, probe_supp, build_keys, build_supp, jt):
    """EXISTS / NOT EXISTS (select * from lineitem l2 where l2.l_orderkey = l1.l_orderkey and l2.l_suppkey <> l1.l_suppkey): INNER candidates,
    SHUFFLE of both l_suppkey sides, GO_COMPARE(<>), JOIN_COND; kind "left" = l1 probes (SEMI / ANTI), "right" = l1 is the build side
    (RIGHT_SEMI / RIGHT_ANTI and JOIN_BUILD_ROWS).  Returns the l1 rows that survive, ascending."""
    if kind == "left":
        jm = ops.JoinMap(build_keys)
        cp, cb = jm.probe(probe_keys)
        jm.release()
        ne, nn = go_compare(CMP_NE, capi.T_INT32, ops.shuffle(probe_supp, cp), ops.shuffle(build_supp, cb))
        p, b = ops.join_cond(cp, cb, ne.astype(bool), len(probe_keys), jt, nn)
        return p, len(cp)
    jm = ops.JoinMap(probe_keys)                                       # l1 is the build side
    cp, cb = jm.probe(build_keys)
    jm.release()
    ne, nn = go_compare(CMP_NE, capi.T_INT32, ops.shuffle(build_supp, cp), ops.shuffle(probe_supp, cb))
    matched = ops.matched_bitmap(len(probe_keys))
    p, _ = ops.join_cond(cp, cb, ne.astype(bool), len(build_keys), jt, nn, matched=matched)
    assert len(p) == 0
    return ops.join_build_rows(matched, len(probe_keys), jt), len(cp)


def test_q21_exists_and_not_exists_end_to_end(gpu):
    d = q21_rows()
    okey = np.array(d["l_orderkey"], np.int64)
    supp = np.array(d["l_suppkey"], np.int32)
    commit, receipt = np.array(d["l_commitdate"], np.int32), np.array(d["l_receiptdate"], np.int32)
    # l1: l_receiptdate > l_commitdate
    gt, gn = go_compare(CMP_GT, capi.T_DATE, receipt, commit)
    l1 = ops.filter_sels(gt, gn)
    assert len(l1) == 3752
    k1, s1 = ops.shuffle(okey, l1), ops.shuffle(supp, l1)
    # a nested loop over the rows, written from the SQL
    by_order = {}
    for i in range(len(okey)):
        by_order.setdefault(int(okey[i]), []).append(i)
    late = receipt > commit
    nested = [i for i in l1.tolist() if any(supp[j] != supp[i] for j in by_order[int(okey[i])])
              and not any(supp[j] != supp[i] and late[j] for j in by_order[int(okey[i])])]
    assert len(nested) == 307
    results = {}
    for kind, semi, anti in (("left", capi.JOIN_SEMI, capi.JOIN_ANTI), ("right", capi.JOIN_RIGHT_SEMI, capi.JOIN_RIGHT_ANTI)):
        ex, npairs = subquery(kind, k1, s1, okey.astype(np.uint64), supp, semi)      # EXISTS: l2 = every lineitem
        if kind == "left":
            assert npairs == 18788                                     # every lineitem of the same order, the row itself included
        kx, sx = ops.shuffle(k1, ex), ops.shuffle(s1, ex)
        nex, _ = subquery(kind, kx.astype(np.uint64), sx, k1.astype(np.uint64), s1, anti)   # NOT EXISTS: l3 = the late lineitems
        results[kind] = l1[ex[nex]]
    assert results["left"].tolist() == nested and results["right"].tolist() == nested
    # orders with o_orderstatus = 'F' (a 1-byte GO_COMPARE), then supplier and nation = 'BRAZIL' (its key selected on the host)
    status = np.frombuffer(d["o_orderstatus"].encode(), np.uint8).copy()
    fo, fn = go_compare(CMP_EQ, capi.T_UINT8, status, np.array([ord("F")], np.uint8))
    forders = np.array(d["o_orderkey"], np.int64)[ops.filter_sels(fo, fn)]
    surv = results["left"]
    om = ops.JoinMap(forders.astype(np.uint64))
    p_o, _ = om.probe(okey[surv].astype(np.uint64))
    om.release()
    rows = surv[p_o]
    sm = ops.JoinMap(np.array(d["s_suppkey"], np.uint64))
    p_s, b_s = sm.probe(supp[rows].astype(np.uint64))
    sm.release()
    assert len(p_s) == len(rows) == sum(1 for i in nested if okey[i] in set(forders.tolist()))
    # numwait per supplier before the nation filter: GROUP_IDS / GROUP_AGG COUNT, ORDER_SELS by numwait desc, s_name (as its key)
    tab = ops.GroupTable(16)
    gids = tab.insert(ops.shuffle(np.array(d["s_suppkey"], np.int64), b_s).astype(np.uint64))
    ng = int(tab.ngroups[0])
    numwait = np.zeros(ng, np.int64)
    assert ops.group_agg(capi.AGG_COUNT, capi.T_INT64, numwait, None, None, gids, np.zeros(len(gids), np.int64)) == 0
    order = ops.order_sels([numwait, tab.keys[:ng].astype(np.int64)], None, [capi.ORDER_DESC, 0])
    want = sorted(((-list(supp[rows]).count(s), int(s)) for s in set(supp[rows].tolist())))
    assert [(-int(numwait[g]), int(tab.keys[g])) for g in order] == want
    brazil = d["n_nationkey"][d["n_name"].index("BRAZIL")]
    nk = ops.shuffle(np.array(d["s_nationkey"], np.int32), b_s)
    bz, bn = go_compare(CMP_EQ, capi.T_INT32, nk, np.array([brazil], np.int32))
    final = ops.filter_sels(bz, bn)
    assert len(final) == 0 and d["q21_result"] == []                  # 03_QUERIES/q21.result is empty at this scale
