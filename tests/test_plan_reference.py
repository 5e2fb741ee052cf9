"""The plan operator's exact restatement (plan_reference.py) against the oracle, no GPU: the Q6 / Q1 shapes against og_q6 / og_q1, and small
plans against chains of the oracle's primitives (og_compare / og_between -> og_filter_sels -> og_group_ids -> og_count / og_minmax /
og_sum_float64).  This pins the reference independently of the kernel it judges."""
import numpy as np
import pytest

import oracle_lib as O
import plan_reference as R
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import bitmap_from_bools

Q1COLS = ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")


@pytest.mark.parametrize("n", [1, 257, 100_003])
def test_reference_q6_matches_oracle(n):
    cols = datagen.lineitem(10, 0, n)
    want, ns, _ = O.q6(cols, n, datagen.q6_params(), nthreads=1)
    p = ops.q6_plan()
    got = R.run(p.P, [cols["shipdate"], cols["discount"], cols["quantity"], cols["extendedprice"]], None, n)
    if ns == 0:
        assert got == []
        return
    assert len(got) == 1 and got[0]["rows"] == ns and got[0]["aggs"][0][1] == ns and got[0]["key"] == 0
    s, _, absum = got[0]["aggs"][0]
    assert abs(s - want) <= ns * R.U * absum


@pytest.mark.parametrize("n", [64, 100_003])
def test_reference_q1_matches_oracle(n):
    cols = datagen.lineitem(10, 0, n)
    want = O.q1(cols, n, datagen.Q1_CUTOFF)
    p = ops.q1_plan(datagen.Q1_CUTOFF, row_base=5)
    got = R.run(p.P, [cols[k] for k in Q1COLS], None, n)
    assert [(g["key"] & 0xff, g["key"] >> 8, g["rows"], g["first_row"] - 5) for g in got] == \
        [(w["returnflag"], w["linestatus"], w["count_order"], w["first_row"]) for w in want]
    for g, w in zip(got, want):
        for a, f in enumerate(("sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc")):
            v, c, absum = g["aggs"][a]
            assert c == w["count_order"] and abs(v - w[f]) <= (c * R.U * absum if a < 4 else 2 * R.U * (absum + abs(v))), f
        assert g["aggs"][7][:2] == (float(w["count_order"]), w["count_order"])


def _oracle_chain(n, conjuncts, keys, values):
    """rows kept by the oracle's filter, their 1-based first-seen group ids, and per value column (type, data, null words)
    COUNT / SUM / MIN / MAX states of the kept rows"""
    lib = O.go()
    keep = np.ones(n, bool)
    for make in conjuncts:
        r = np.zeros(n, np.uint8); rn = np.zeros(n // 64 + 2, np.uint64)
        make(r, rn)
        sels = np.zeros(n, np.int64)
        k = lib.og_filter_sels(O.p(r), O.p(rn), n, O.p(sels))
        m = np.zeros(n, bool); m[sels[:k]] = True
        keep &= m
    idx = np.flatnonzero(keep)
    ks = np.ascontiguousarray(keys[idx], np.uint64)
    groups = np.zeros(max(idx.size, 1), np.uint64); table = np.zeros(max(idx.size, 1), np.uint64)
    ng = lib.og_group_ids(O.p(ks), idx.size, O.p(groups), O.p(table), 0, max(idx.size, 1))
    out = []
    for T, data, words in values:
        d = np.ascontiguousarray(data[idx]); nw = bitmap_from_bools(R.null_mask(words, n)[idx]) if words is not None else None
        cnt = np.zeros(ng, np.int64); lib.og_count(0, O.p(nw), 0, O.p(groups), idx.size, O.p(cnt))
        sums = np.zeros(ng); sn = np.ones(ng, np.uint8)
        lib.og_sum_float64(T, O.p(d), O.p(nw), 0, O.p(groups), idx.size, O.p(sums), O.p(sn), None)
        mm = []
        for is_max in (0, 1):
            st = np.zeros(ng, d.dtype); isn = np.ones(ng, np.uint8)
            lib.og_minmax(is_max, T, O.p(d), O.p(nw), 0, O.p(groups), idx.size, O.p(st), O.p(isn))
            mm.append(st.astype(np.float64))
        out.append((cnt, sums, mm[0], mm[1]))
    star = np.zeros(ng, np.int64); lib.og_count(1, None, 0, O.p(groups), idx.size, O.p(star))
    first = [int(idx[np.flatnonzero(groups[:idx.size] == g + 1)[0]]) for g in range(ng)]
    return table[:ng], first, star, out


def _check_against_chain(got, table, first, star, states, row_base=0):
    assert [g["key"] for g in got] == [int(k) for k in table]
    assert [g["first_row"] for g in got] == [f + row_base for f in first]
    assert [g["rows"] for g in got] == list(star)
    for g, gr in enumerate(got):
        for v, (cnt, sums, mins, maxs) in enumerate(states):
            a = gr["aggs"][5 * v: 5 * v + 5]            # COUNT, SUM, MIN, MAX, AVG of value column v
            assert [x[1] for x in a] == [cnt[g]] * 5
            if cnt[g]:
                assert abs(a[1][0] - sums[g]) <= cnt[g] * R.U * a[1][2]
                assert a[2][0] == mins[g] and a[3][0] == maxs[g]
                assert abs(a[4][0] - sums[g] / cnt[g]) <= 2 * R.U * (a[4][2] + abs(a[4][0]))


def test_reference_int64_predicates_and_nullable_values_match_oracle_chain():
    """int64 >= 2^60 (the planner casts the constant to int64), float64 BETWEEN with a NULL-bearing column, an int32 key"""
    rng = np.random.default_rng(11)
    n = 6000
    y = (np.int64(2 ** 60) + rng.integers(-3, 4, n)).astype(np.int64)
    x = np.round(rng.standard_normal(n) * 8, 1)
    key = (rng.integers(0, 40, n) * 7 - 100).astype(np.int32)
    xw = bitmap_from_bools(rng.random(n) < 0.2)
    lib = O.go()
    c60 = np.array([2 ** 60], np.int64); lo = np.array([-6.0]); hi = np.array([9.5])
    conj = [lambda r, rn: lib.og_compare(3, capi.T_INT64, O.p(r), O.p(y), O.p(c60), n, 0, 1, None, None, O.p(rn)),
            lambda r, rn: lib.og_between(capi.T_FLOAT64, O.p(r), O.p(x), O.p(lo), O.p(hi), n, O.p(xw), O.p(rn))]
    table, first, star, states = _oracle_chain(n, conj, key.view(np.uint32).astype(np.uint64), [(capi.T_FLOAT64, x, xw)])
    p = ops.FusedPlan([capi.T_INT32, capi.T_FLOAT64, capi.T_INT64], row_base=1000)
    p.where(2, ">=", 2.0 ** 60).where(1, "between", -6.0, 9.5).group_by(0)
    for kind in (capi.AGG_COUNT, capi.AGG_SUM, capi.AGG_MIN, capi.AGG_MAX, capi.AGG_AVG):
        p.agg(kind, 1)
    got = R.run(p.P, [key, x, y], [None, xw, None], n)
    assert len(got) > 20
    _check_against_chain(got, table, first, star, states, row_base=1000)


def test_reference_unsigned_and_float32_match_oracle_chain():
    """uint64 > 2^63 (unsigned compare), two keys (int16, uint8) packed like fillKeys, float32 values widened exactly"""
    rng = np.random.default_rng(12)
    n = 5000
    u = (np.uint64(2 ** 63) + rng.integers(0, 3, n).astype(np.uint64) - np.uint64(1)).astype(np.uint64)
    k1 = rng.integers(-300, 300, n).astype(np.int16) // 50
    k2 = rng.integers(0, 3, n).astype(np.uint8) * 100
    f = (rng.standard_normal(n) * 3).astype(np.float32)
    fw = bitmap_from_bools(rng.random(n) < 0.1)
    lib = O.go()
    c63 = np.array([2 ** 63], np.uint64)
    conj = [lambda r, rn: lib.og_compare(2, capi.T_UINT64, O.p(r), O.p(u), O.p(c63), n, 0, 1, None, None, O.p(rn))]
    packed = k1.view(np.uint16).astype(np.uint64) | (k2.astype(np.uint64) << np.uint64(16))
    table, first, star, states = _oracle_chain(n, conj, packed, [(capi.T_FLOAT32, f, fw)])
    p = ops.FusedPlan([capi.T_UINT64, capi.T_INT16, capi.T_UINT8, capi.T_FLOAT32])
    p.where(0, ">", 2.0 ** 63).group_by(1, 2)
    for kind in (capi.AGG_COUNT, capi.AGG_SUM, capi.AGG_MIN, capi.AGG_MAX, capi.AGG_AVG):
        p.agg(kind, 3)
    got = R.run(p.P, [u, k1, k2, f], [None, None, None, fw], n)
    assert len(got) > 10 and sum(g["rows"] for g in got) == int((u > np.uint64(2 ** 63)).sum())
    _check_against_chain(got, table, first, star, states)


def test_reference_exact_integer_compare():
    """the comparisons the issue's repros need, against Python integers"""
    x = np.array([2 ** 60 - 1, 2 ** 60, 2 ** 60 + 1], np.int64)
    assert R.compare(x, R.GE, 2.0 ** 60).tolist() == [False, True, True]
    assert R.compare(np.array([2 ** 53, 2 ** 53 + 1], np.int64), R.EQ, 2.0 ** 53).tolist() == [True, False]
    assert R.compare(np.array([2 ** 63 + 1, 2 ** 63, 1], np.uint64), R.GT, 2.0 ** 63).tolist() == [True, False, False]
    big = np.array([-2 ** 63, -1, 0, 2 ** 63 - 1], np.int64)
    for op in range(6):
        for c in (2.0 ** 63, -2.0 ** 63, 2.0 ** 64, -2.5, 0.5, float("inf"), -float("inf"), float("nan")):
            # Python compares an int with a float exactly (and NaN by IEEE)
            want = [{0: v == c, 1: v != c, 2: v > c, 3: v >= c, 4: v < c, 5: v <= c}[op] for v in map(int, big)]
            assert R.compare(big, op, c).tolist() == want, (op, c)


def test_reference_keys_and_null_modes():
    """fillKeys layout: has_null_keys writes a marker byte per column; without it a NULL key row joins no group"""
    k8 = np.array([-1, 5, -1, 7], np.int8); k16 = np.array([300, -2, 300, 9], np.int16)
    nw = bitmap_from_bools(np.array([False, True, False, False]))
    p = ops.FusedPlan([capi.T_INT8, capi.T_INT16], has_null_keys=True).group_by(0, 1).agg(capi.AGG_COUNT, -1)
    got = R.run(p.P, [k8, k16], [nw, None], 4)
    assert [(g["key"], g["rows"]) for g in got] == [(0xff00 | (300 << 24), 2), (1 | (0xfffe << 16), 1), (0x0700 | (9 << 24), 1)]
    p = ops.FusedPlan([capi.T_INT8, capi.T_INT16]).group_by(0, 1).agg(capi.AGG_COUNT, -1)
    got = R.run(p.P, [k8, k16], [nw, None], 4)
    assert [(g["key"], g["rows"], g["first_row"]) for g in got] == [(0xff | (300 << 8), 2, 0), (7 | (9 << 8), 1, 3)]
