"""TPC-H Q14 end to end through the C ABI on the reference's lineitem and part rows (golden/tpch_q14.json), against
03_QUERIES/q14.result (promo_revenue 17.68284163936513):

    select 100.00 * sum(case when p_type like 'PROMO%' then l_extendedprice * (1 - l_discount) else 0 end)
           / sum(l_extendedprice * (1 - l_discount)) as promo_revenue
    from lineitem, part where l_partkey = p_partkey and l_shipdate >= date '1996-04-01' and l_shipdate < date '1996-04-01' + interval '1' month

l_extendedprice and l_discount are DECIMAL(15,2).  The pipeline: two DATE compares, MULTI_AND, FILTER_SELS; JOIN_PROBE to part and
SHUFFLE(24) of p_type; GO_LIKE 'PROMO%', then GO_CASE_SELECT, so the THEN branch is evaluated only on the rows its WHEN took;
DEC_ARITH 1 - l_discount (Decimal64, scale 2) and l_extendedprice * that (Decimal128, scale 4) -- once under THEN's prefill, once over
every row for the denominator; GO_CASE(DECIMAL128) with the const 0 ELSE at scale 4 (the planner's cast of 0 to the THEN's type); two
DEC_SUMs, each exact against a Fraction restatement.

The last step runs on the host, as one scalar step over the two sums.  100.00 * a is exact: DECIMAL(5,2) times the sum's Decimal128 at
scale 4 is a Decimal128 at scale 6.  The division is the float64 one: each side converted as Decimal128ToFloat64 does (the integer over
10^scale, correctly rounded), then divided.  Its 16-significant-digit form is q14.result's value.  The planner's decimal division
(list_operator.go: Decimal128 at scale min(12, scale1 + 6)) would print 17.682841639365 and does not match the file."""
import json
import os
from fractions import Fraction

import numpy as np
import pytest

from matrixone_b200 import capi, ops
from matrixone_b200.vector import Vector, bitmap_from_bools, bitmap_to_bools
from test_gpu_tpch_q12 import bool_call, days, logic, shuffle_cells, strs

pytestmark = pytest.mark.gpu


def signed128(v):
    lo, hi = int(v[0]), int(v[1])
    x = lo | (hi << 64)
    return x - (1 << 128) if x >> 127 else x


def test_q14_end_to_end(gpu):
    d = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tpch_q14.json")))
    assert d["counts"] == {"lineitem": 6005, "part": 200}
    n = d["counts"]["lineitem"]
    ship = np.array(d["l_shipdate"], np.int32)
    lo, hi = days("1996-04-01"), days("1996-05-01")
    conj = [bool_call(capi.XCALL_GO_COMPARE(capi.CMP_GE, capi.T_DATE), n, Vector(data=ship), Vector(data=np.array([lo], np.int32))),
            bool_call(capi.XCALL_GO_COMPARE(capi.CMP_LT, capi.T_DATE), n, Vector(data=ship), Vector(data=np.array([hi], np.int32)))]
    where, wn = logic(capi.XCALL_GO_MULTI_AND, n, conj)
    sels = ops.filter_sels(where, wn)
    assert sels.tolist() == [i for i in range(n) if lo <= ship[i] < hi]
    # l_partkey = p_partkey
    jm = ops.JoinMap(np.array(d["p_partkey"], np.uint64))
    probe, build = jm.probe(np.array(d["l_partkey"], np.uint64)[sels])
    jm.release()
    rows = sels[probe]
    m = len(rows)
    assert m == len(sels) == 62
    tcells, tarea = strs([t.encode() for t in d["p_type"]])
    ptype = (shuffle_cells(tcells, build), tarea)
    promo, promo_nulls = ops.like(ptype, b"PROMO%")
    assert not promo_nulls.any()
    assert promo.tolist() == [d["p_type"][b].startswith("PROMO") for b in build]
    # EvalCase's select lists: every joined row is selected, the WHEN takes the PROMO rows
    then, rem = ops.case_select(np.zeros((m + 63) // 64, np.uint64), promo.astype(np.uint8), None, m)
    assert (bitmap_to_bools(then, m) == ~promo).all() and (bitmap_to_bools(rem, m) == promo).all()
    price = np.array(d["l_extendedprice"], np.int64)[rows]
    disc = np.array(d["l_discount"], np.int64)[rows]
    one = np.array([100], np.int64)                                   # 1 at scale 2

    def revenue(rnulls):
        rc, one_minus, omn, _ = ops.dec_arith(1, 64, one, disc, 2, 2, m, rnulls=rnulls)
        assert rc == 0
        rc, rev, rvn, _ = ops.dec_arith(2, 64, price, one_minus, 2, 2, m, rnulls=omn)
        assert rc == 0
        return rev, rvn

    rev_then, rev_then_nulls = revenue(then)                          # THEN: only the rows the WHEN took
    rev_all, rev_all_nulls = revenue(None)                            # the denominator's argument: every row
    assert not bitmap_to_bools(rev_all_nulls, m).any()
    assert (bitmap_to_bools(rev_then_nulls, m) == ~promo).all()
    exact = [int(p) * (100 - int(q)) for p, q in zip(price, disc)]   # scale 4
    assert [signed128(v) for v in rev_all] == exact
    case_vals, case_nulls = ops.go_case(capi.T_DECIMAL128, [(promo.astype(np.uint8), None)], [(rev_then, rev_then_nulls)],
                                        (np.zeros((1, 2), np.uint64), None))
    assert not case_nulls.any()
    assert [signed128(v) for v in case_vals] == [e if p else 0 for e, p in zip(exact, promo)]
    sums = []
    for col, nulls in ((case_vals, bitmap_from_bools(case_nulls)), (rev_all, None)):
        acc, cnt = np.zeros((1, 2), np.uint64), np.zeros(1, np.int64)
        ops.dec_sum(128, np.ascontiguousarray(col, np.uint64), acc, cnt, None, nulls, m)
        assert int(cnt[0]) == m
        sums.append(signed128(acc[0]))
    a, b = sums
    assert Fraction(a, 10 ** 4) == sum(Fraction(e, 10 ** 4) for e, p in zip(exact, promo) if p)
    assert Fraction(b, 10 ** 4) == sum(Fraction(e, 10 ** 4) for e in exact)
    # host: 100.00 * a exact at scale 6, then the float64 division of the two Decimal128ToFloat64 values
    promo_revenue = (10000 * a / 10 ** 6) / (b / 10 ** 4)
    assert "%.16g" % promo_revenue == d["q14_result"] == "17.68284163936513"
    assert "%.12f" % Fraction(10000 * a * 10 ** 4, b * 10 ** 6) != d["q14_result"]
