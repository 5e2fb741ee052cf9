"""TPC-H Q13 on the reference's customer and orders rows (golden/tpch_q13.json), against 03_QUERIES/q13.result row for row:

    select c_count, count(*) as custdist
    from (select c_custkey, count(o_orderkey) from customer left outer join orders
          on c_custkey = o_custkey and o_comment not like '%pending%accounts%' group by c_custkey) as c_orders (c_custkey, c_count)
    group by c_count order by custdist desc, c_count desc

The whole chain runs through the C-ABI: JOIN_PROBE(INNER) gives the candidate pairs of the equality key; SHUFFLE(24) gathers o_comment's
cells by the candidate build rows (they still point into o_comment's area); GO_LIKE evaluates the const multi-% pattern over them and
Logic_VecNot negates it (NOT LIKE); JOIN_COND(LEFT) turns the pairs and the condition into the LEFT join's rows; PACK_KEYS / GROUP_IDS /
GROUP_AGG(COUNT) run the two group-bys and ORDER_SELS the ORDER BY."""
import json
import os

import numpy as np
import pytest

from matrixone_b200 import capi, ops
from matrixone_b200.vector import Vector, varlena_bytes_column, xcall

import like_reference as L

pytestmark = pytest.mark.gpu

PATTERN = b"%pending%accounts%"


def q13_rows():
    d = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tpch_q13.json")))
    assert d["counts"] == {"customer": 150, "orders": 1500}
    return d


def shuffle_cells(cells, sels):
    """SHUFFLE(24) of varlena cells; the output cells point into the source column's area"""
    m = len(sels)
    dst = np.zeros(24 * m, np.uint8)
    xcall(capi.XCALL_SHUFFLE(24), [Vector(data=dst, length=m), Vector(data=cells, length=len(cells) // 24),
                                   Vector(data=np.ascontiguousarray(sels, np.int64), length=m)], m)
    return dst


def group_count(keys_col, col, col_nulls):
    """PACK_KEYS (one 8-byte-or-narrower column, raw value bytes) -> GROUP_IDS -> GROUP_AGG(COUNT, col): (group key values, counts)"""
    keys, _ = ops.pack_keys([keys_col], has_null=False)
    tab = ops.GroupTable(len(keys) + 1)
    gids = tab.insert(keys)
    ng = int(tab.ngroups[0])
    cnt = np.zeros(ng, np.int64)
    assert ops.group_agg(capi.AGG_COUNT, capi.T_INT64, cnt, None, None, gids, col, col_nulls) == 0
    return tab.keys[:ng].astype(np.int64), cnt


def test_q13_end_to_end(gpu):
    d = q13_rows()
    ckey = np.array(d["c_custkey"], np.int32)
    okey = np.array(d["o_orderkey"], np.int64)
    ocust = np.array(d["o_custkey"], np.int32)
    comments = [c.encode() for c in d["o_comment"]]
    cells, area = varlena_bytes_column(comments)
    # customer LEFT JOIN orders ON c_custkey = o_custkey AND <cond>: the INNER candidates of the key first
    jm = ops.JoinMap(ocust.astype(np.uint64))
    cp, cb = jm.probe(ckey.astype(np.uint64))
    jm.release()
    assert len(cp) == 1500                                           # every order's customer exists
    # o_comment NOT LIKE '%pending%accounts%' over the candidate pairs
    sc = shuffle_cells(cells, cb)
    like = np.zeros(len(cp), np.uint8)
    like_nulls = np.zeros((len(cp) + 63) // 64, np.uint64)
    xcall(capi.XCALL_GO_LIKE, [Vector(data=like, nulls=like_nulls, length=len(cp)), Vector(data=sc, area=area, length=len(cp)),
                               Vector(data=varlena_bytes_column([PATTERN])[0], length=1)], len(cp))
    assert not like_nulls.any()
    assert like.astype(bool).tolist() == [L.like(comments[b], PATTERN) for b in cb]
    assert L.optimize_rule(PATTERN) is not None                      # the multi-% chain of optimizeRuleForLike
    lib = capi.load_library()
    cond = np.zeros(len(cp), np.uint8)
    capi.check(lib.Logic_VecNot(cond.ctypes.data, like.ctypes.data, len(cp), like_nulls.ctypes.data, 0), lib)
    assert (cond == 1 - like).all() and 0 < int(like.sum()) < len(cp)
    p, b = ops.join_cond(cp, cb, cond.astype(bool), len(ckey), capi.JOIN_LEFT, like_nulls)
    # count(o_orderkey) group by c_custkey: the orders side of a row without a match is NULL (SHUFFLE with sel -1)
    ok, okn = ops.shuffle(okey, b, want_nulls=True)
    ck = ops.shuffle(ckey, p)
    cust, c_count = group_count(ck, ok, okn)
    assert len(cust) == 150
    # count(*) group by c_count, order by custdist desc, c_count desc
    c_counts, custdist = group_count(c_count, np.zeros(len(c_count), np.int64), None)
    order = ops.order_sels([custdist, c_counts], None, [capi.ORDER_DESC, capi.ORDER_DESC])
    got = [[int(c_counts[g]), int(custdist[g])] for g in order]
    assert got == d["q13_result"]
