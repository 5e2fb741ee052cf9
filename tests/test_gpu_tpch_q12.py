"""TPC-H Q12 on the reference's lineitem and orders rows (golden/tpch_q12.json), against 03_QUERIES/q12.result (FOB 4 5, TRUCK 5 7):

    select l_shipmode, sum(case when o_orderpriority = '1-URGENT' or o_orderpriority = '2-HIGH' then 1 else 0 end) as high_line_count,
           sum(case when o_orderpriority <> '1-URGENT' and o_orderpriority <> '2-HIGH' then 1 else 0 end) as low_line_count
    from orders, lineitem
    where o_orderkey = l_orderkey and l_shipmode in ('FOB', 'TRUCK') and l_commitdate < l_receiptdate and l_shipdate < l_commitdate
          and l_receiptdate >= date '1996-01-01' and l_receiptdate < date '1996-01-01' + interval '1' year
    group by l_shipmode order by l_shipmode

Through the C ABI: GO_IN(CHAR) on l_shipmode, the four DATE compares, MULTI_AND, FILTER_SELS; JOIN_PROBE to orders; SHUFFLE(24) of
o_orderpriority.  CASE is not built, so each sum(case when p then 1 else 0 end) counts the rows where p holds, with p evaluated as
GO_IN(CHAR) / GO_NOT_IN(CHAR) of ('1-URGENT', '2-HIGH') -- checked equal to the literal `= OR =` / `<> AND <>` form built from GO_COMPARE
and MULTI_OR / MULTI_AND.  The group by runs PACK_STR_KEYS / STR_GROUP_IDS / GROUP_AGG(SUM), the order by ORDER_SELS."""
import datetime
import json
import os

import numpy as np
import pytest

from matrixone_b200 import capi, ops
from matrixone_b200.vector import Vector, bitmap_to_bools, varlena_bytes_column, xcall

pytestmark = pytest.mark.gpu


def days(s):
    return datetime.date.fromisoformat(s).toordinal() - datetime.date(1970, 1, 1).toordinal()


def bool_call(fid, n, *operands):
    """one GO-convention call with a bool result: (values uint8[n], null bitmap words)"""
    r = np.zeros(n, np.uint8)
    rn = np.zeros((n + 63) // 64, np.uint64)
    xcall(fid, [Vector(data=r, nulls=rn, length=n)] + list(operands), n)
    return r, rn


def strs(values):
    cells, area = varlena_bytes_column(values)
    return cells, (area if area.size else None)


def const_str(value):
    cells, area = strs([value])
    return Vector(data=cells, area=area, length=1)


def logic(fid, n, ops_):
    return bool_call(fid, n, Vector(data=np.array([len(ops_)], np.int32)), *[Vector(data=r, nulls=rn, length=n) for r, rn in ops_])


def shuffle_cells(cells, sels):
    m = len(sels)
    dst = np.zeros(24 * m, np.uint8)
    xcall(capi.XCALL_SHUFFLE(24), [Vector(data=dst, length=m), Vector(data=cells, length=len(cells) // 24),
                                   Vector(data=np.ascontiguousarray(sels, np.int64), length=m)], m)
    return dst


def test_q12_end_to_end(gpu):
    d = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tpch_q12.json")))
    assert d["counts"] == {"lineitem": 6005, "orders": 1500}
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
    want = [i for i in range(n) if d["l_shipmode"][i] in ("FOB", "TRUCK") and commit[i] < receipt[i] and ship[i] < commit[i]
            and days("1996-01-01") <= receipt[i] < days("1997-01-01")]
    assert sels.tolist() == want and len(want) == 21
    # o_orderkey = l_orderkey
    jm = ops.JoinMap(np.array(d["o_orderkey"], np.uint64))
    probe, build = jm.probe(np.array(d["l_orderkey"], np.uint64)[sels])
    jm.release()
    assert len(probe) == len(sels)
    m = len(probe)
    pcells, parea = strs([p.encode() for p in d["o_orderpriority"]])
    prio = Vector(data=shuffle_cells(pcells, build), area=parea, length=m)
    urgent, _ = strs([b"1-URGENT", b"2-HIGH"])
    lst = Vector(data=urgent, length=2)
    high, hn = bool_call(capi.XCALL_GO_IN(capi.T_CHAR), m, prio, lst, Vector(data=np.array([2], np.int64)))
    low, ln_ = bool_call(capi.XCALL_GO_NOT_IN(capi.T_CHAR), m, prio, lst, Vector(data=np.array([2], np.int64)))
    eq = [bool_call(capi.XCALL_GO_COMPARE(capi.CMP_EQ, capi.T_CHAR), m, prio, const_str(v)) for v in (b"1-URGENT", b"2-HIGH")]
    ne = [bool_call(capi.XCALL_GO_COMPARE(capi.CMP_NE, capi.T_CHAR), m, prio, const_str(v)) for v in (b"1-URGENT", b"2-HIGH")]
    high_lit, _ = logic(capi.XCALL_GO_MULTI_OR, m, eq)
    low_lit, _ = logic(capi.XCALL_GO_MULTI_AND, m, ne)
    assert not bitmap_to_bools(hn, m).any() and not bitmap_to_bools(ln_, m).any()
    assert (high == high_lit).all() and (low == low_lit).all() and (high != low).all()
    # group by l_shipmode: the key bytes, group ids, sum of the two 0 / 1 columns
    smodes = strs([d["l_shipmode"][i].encode() for i in sels[probe]])
    kb, ko, _ = ops.pack_str_keys([smodes], [capi.T_CHAR])
    tab = ops.StrGroupTable()
    gids = tab.insert(kb, ko)
    ng = int(tab.ngroups[0])
    sums = []
    for col in (high, low):
        s = np.zeros(ng, np.int64)
        assert ops.group_agg(capi.AGG_SUM, capi.T_INT64, s, None, None, gids, col.astype(np.int64)) == 0
        sums.append(s)
    first = [int(np.flatnonzero(gids == g + 1)[0]) for g in range(ng)]
    names = [d["l_shipmode"][sels[probe][i]] for i in first]
    order = ops.order_sels([[x.encode() for x in names]], None, [0], types=[capi.T_CHAR])
    got = [[names[g], int(sums[0][g]), int(sums[1][g])] for g in order]
    assert got == d["q12_result"] == [["FOB", 4, 5], ["TRUCK", 5, 7]]
