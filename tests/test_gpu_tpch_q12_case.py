"""TPC-H Q12 with its real conditional sums, on the reference's lineitem and orders rows (golden/tpch_q12.json), against
03_QUERIES/q12.result (FOB 4 5, TRUCK 5 7):

    sum(case when o_orderpriority = '1-URGENT' or o_orderpriority = '2-HIGH' then 1 else 0 end) as high_line_count,
    sum(case when o_orderpriority <> '1-URGENT' and o_orderpriority <> '2-HIGH' then 1 else 0 end) as low_line_count

Through the C ABI: the WHERE clause, FILTER_SELS, JOIN_PROBE and SHUFFLE(24) as in test_gpu_tpch_q12.py; each WHEN is the literal
GO_COMPARE(CHAR) / MULTI_OR or MULTI_AND form, each CASE is GO_CASE(INT64) with the const THEN 1 and ELSE 0, and the group by sums
those INT64 columns with PACK_STR_KEYS / STR_GROUP_IDS / GROUP_AGG(SUM), the order by ORDER_SELS."""
import json
import os

import numpy as np
import pytest

from matrixone_b200 import capi, ops
from matrixone_b200.vector import Vector
from test_gpu_tpch_q12 import bool_call, const_str, days, logic, shuffle_cells, strs

pytestmark = pytest.mark.gpu


def test_q12_sums_of_case_end_to_end(gpu):
    d = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tpch_q12.json")))
    n = d["counts"]["lineitem"]
    ship, commit, receipt = (np.array(d[k], np.int32) for k in ("l_shipdate", "l_commitdate", "l_receiptdate"))
    mode_cells, mode_area = strs([m.encode() for m in d["l_shipmode"]])
    modes = Vector(data=mode_cells, area=mode_area, length=n)
    in_list, _ = strs([b"FOB", b"TRUCK"])
    conj = [bool_call(capi.XCALL_GO_IN(capi.T_CHAR), n, modes, Vector(data=in_list, length=2), Vector(data=np.array([2], np.int64)))]
    lt = capi.XCALL_GO_COMPARE(capi.CMP_LT, capi.T_DATE)
    conj.append(bool_call(lt, n, Vector(data=commit), Vector(data=receipt)))
    conj.append(bool_call(lt, n, Vector(data=ship), Vector(data=commit)))
    conj.append(bool_call(capi.XCALL_GO_COMPARE(capi.CMP_GE, capi.T_DATE), n, Vector(data=receipt),
                          Vector(data=np.array([days("1996-01-01")], np.int32))))
    conj.append(bool_call(lt, n, Vector(data=receipt), Vector(data=np.array([days("1997-01-01")], np.int32))))
    where, wn = logic(capi.XCALL_GO_MULTI_AND, n, conj)
    sels = ops.filter_sels(where, wn)
    jm = ops.JoinMap(np.array(d["o_orderkey"], np.uint64))
    probe, build = jm.probe(np.array(d["l_orderkey"], np.uint64)[sels])
    jm.release()
    m = len(probe)
    assert m == len(sels) == 21
    pcells, parea = strs([p.encode() for p in d["o_orderpriority"]])
    prio = Vector(data=shuffle_cells(pcells, build), area=parea, length=m)
    eq = [bool_call(capi.XCALL_GO_COMPARE(capi.CMP_EQ, capi.T_CHAR), m, prio, const_str(v)) for v in (b"1-URGENT", b"2-HIGH")]
    ne = [bool_call(capi.XCALL_GO_COMPARE(capi.CMP_NE, capi.T_CHAR), m, prio, const_str(v)) for v in (b"1-URGENT", b"2-HIGH")]
    cases = []
    for when, when_nulls in (logic(capi.XCALL_GO_MULTI_OR, m, eq), logic(capi.XCALL_GO_MULTI_AND, m, ne)):
        vals, nulls = ops.go_case(capi.T_INT64, [(when, when_nulls)], [(np.array([1], np.int64), None)], (np.array([0], np.int64), None))
        assert not nulls.any() and set(vals.tolist()) <= {0, 1}
        cases.append(vals.astype(np.int64))
    prio_rows = [d["o_orderpriority"][b] for b in build]
    assert cases[0].tolist() == [int(p in ("1-URGENT", "2-HIGH")) for p in prio_rows]
    assert (cases[0] + cases[1] == 1).all()
    smodes = strs([d["l_shipmode"][i].encode() for i in sels[probe]])
    kb, ko, _ = ops.pack_str_keys([smodes], [capi.T_CHAR])
    tab = ops.StrGroupTable()
    gids = tab.insert(kb, ko)
    ng = int(tab.ngroups[0])
    sums = []
    for col in cases:
        s = np.zeros(ng, np.int64)
        assert ops.group_agg(capi.AGG_SUM, capi.T_INT64, s, None, None, gids, col) == 0
        sums.append(s)
    first = [int(np.flatnonzero(gids == g + 1)[0]) for g in range(ng)]
    names = [d["l_shipmode"][sels[probe][i]] for i in first]
    order = ops.order_sels([[x.encode() for x in names]], None, [0], types=[capi.T_CHAR])
    got = [[names[g], int(sums[0][g]), int(sums[1][g])] for g in order]
    assert got == d["q12_result"] == [["FOB", 4, 5], ["TRUCK", 5, 7]]
