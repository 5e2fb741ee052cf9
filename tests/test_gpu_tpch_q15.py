"""TPC-H Q15 end to end on the reference's lineitem and supplier rows (tests/golden/tpch_q15.json, row counts checked against the load's
10_select_count.result), through the C ABI on the DECIMAL(15,2) schema: the shipdate range as two DATE compares -> FILTER_SELS -> SHUFFLE;
l_extendedprice * (1 - l_discount) as DEC_ARITH sub and mul; GROUP_IDS on l_suppkey -> DEC_SUM; the max of total_revenue as ORDER_SELS
(DECIMAL128 descending, limit 1); total_revenue = max as GO_COMPARE(==, DECIMAL128); the join to supplier.  The result equals q15.result."""
import datetime
import json
import os

import numpy as np
import pytest

import oracle_lib as O
from matrixone_b200 import capi, ops
from matrixone_b200.vector import Vector, xcall

pytestmark = pytest.mark.gpu


def _days(y, m, d):
    return datetime.date(y, m, d).toordinal() - datetime.date(1970, 1, 1).toordinal()


def _date_cmp(op, col, const):
    n = len(col)
    r = np.zeros(n, dtype=np.uint8); rn = np.zeros((n + 63) // 64, dtype=np.uint64)
    xcall(capi.XCALL_GO_COMPARE(op, capi.T_DATE), [Vector(data=r, nulls=rn, length=n), Vector(data=col, length=n),
                                                   Vector(data=np.asarray([const], dtype=np.int32), length=n)], n)
    assert not rn.any()
    return r


def test_q15_end_to_end(gpu):
    d = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tpch_q15.json")))
    assert d["counts"] == {"lineitem": 6005, "supplier": 10}
    ship = np.asarray(d["l_shipdate"], dtype=np.int32)
    supp = np.asarray(d["l_suppkey"], dtype=np.int32)
    price = np.asarray(d["l_extendedprice"], dtype=np.int64)
    disc = np.asarray(d["l_discount"], dtype=np.int64)
    # l_shipdate >= date '1995-12-01' and l_shipdate < date '1995-12-01' + interval '3' month
    m = _date_cmp(capi.CMP_GE, ship, _days(1995, 12, 1)) & _date_cmp(capi.CMP_LT, ship, _days(1996, 3, 1))
    sels = ops.filter_sels(m)
    k = len(sels)
    assert k > 0
    p_, d_, s_ = ops.shuffle(price, sels), ops.shuffle(disc, sels), ops.shuffle(supp, sels)
    # l_extendedprice * (1 - l_discount): DECIMAL(15,2) * DECIMAL(16,2) -> Decimal128 at scale 4
    rc, one_minus, _, _ = ops.dec_arith(1, 64, np.asarray([1], dtype=np.int64), d_, 0, 2, k)
    assert rc == 0
    rc, rev, _, _ = ops.dec_arith(2, 64, p_, one_minus, 2, 2, k)
    assert rc == 0
    # group by l_suppkey: sum(...) as total_revenue
    keys, _ = ops.pack_keys([s_], has_null=False)
    tab = ops.GroupTable(k + 1)
    gids = tab.insert(keys)
    ng = int(tab.ngroups[0])
    total = np.zeros((ng, 2), dtype=np.uint64); cnt = np.zeros(ng, dtype=np.int64)
    ops.dec_sum(128, rev, total, cnt, gids, None, k)
    # select max(total_revenue) from q15_revenue0
    top = ops.order_sels([total], None, [capi.ORDER_DESC], limit=1)
    assert len(top) == 1
    mx = total[int(top[0]):int(top[0]) + 1].copy()
    # total_revenue = (max): DECIMAL128 compare, both at scale 4
    eq, eqn = ops.dec_compare(capi.CMP_EQ, 128, total, mx, 4, 4, ng)
    assert not eqn.any()
    win = ops.filter_sels(eq)
    # supplier join q15_revenue0 on s_suppkey = supplier_no, order by s_suppkey
    s_key = np.asarray(d["s_suppkey"], dtype=np.int64)
    jm = ops.JoinMap(s_key.astype(np.uint64))
    pr, br = jm.probe(tab.keys[:ng][win].astype(np.uint64))
    jm.release()
    totals = O.d128_to_int(total)
    rows = sorted([str(int(s_key[b])), d["s_name"][b], d["s_address"][b], d["s_phone"][b], O.decimal_str(totals[int(win[p])], 4)]
                  for p, b in zip(pr, br))
    assert rows == d["q15_result"]
    assert rows == [["1", "Supplier#000000001", " N kD4on9OM Ipw3,gf0JBoQDd7tgrzrddZ", "27-918-335-1736", "863528.2162"]]
