"""TPC-H Q16 on the reference's part, partsupp and supplier rows (golden/tpch_q16.json), against 03_QUERIES/q16.result row for row (41 rows):

    select p_brand, p_type, p_size, count(distinct ps_suppkey) as supplier_cnt
    from partsupp, part
    where p_partkey = ps_partkey and p_brand <> 'Brand#35' and p_type not like 'ECONOMY BURNISHED%'
          and p_size in (14, 7, 21, 24, 35, 33, 2, 20)
          and ps_suppkey not in (select s_suppkey from supplier where s_comment like '%Customer%Complaints%')
    group by p_brand, p_type, p_size order by supplier_cnt desc, p_brand, p_type, p_size

Through the C ABI: GO_COMPARE(!=, CHAR), GO_LIKE + Logic_VecNot, GO_IN(INT32), MULTI_AND and FILTER_SELS over part; GO_LIKE over supplier;
the NOT IN (subquery) as a JOIN_PROBE ANTI join, and also as GO_NOT_IN(INT32) with the subquery's rows as a device-resident list (empty at
this scale: nvalues == 0), which must keep the same rows; JOIN_PROBE to part; count(distinct ps_suppkey) as two PACK_STR_KEYS /
STR_GROUP_IDS passes and GROUP_AGG(COUNT); ORDER_SELS."""
import json
import os

import numpy as np
import pytest

from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_to_bools
from test_gpu_tpch_q12 import bool_call, const_str, logic, shuffle_cells, strs

pytestmark = pytest.mark.gpu

SIZES = [14, 7, 21, 24, 35, 33, 2, 20]


def test_q16_end_to_end(gpu):
    d = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tpch_q16.json")))
    assert d["counts"] == {"part": 200, "partsupp": 800, "supplier": 10}
    n = 200
    brand_cells, brand_area = strs([b.encode() for b in d["p_brand"]])
    type_cells, type_area = strs([t.encode() for t in d["p_type"]])
    size = np.array(d["p_size"], np.int32)
    b1 = bool_call(capi.XCALL_GO_COMPARE(capi.CMP_NE, capi.T_CHAR), n, Vector(data=brand_cells, area=brand_area, length=n), const_str(b"Brand#35"))
    like, like_n = bool_call(capi.XCALL_GO_LIKE, n, Vector(data=type_cells, area=type_area, length=n), const_str(b"ECONOMY BURNISHED%"))
    lib = capi.load_library()
    not_like = np.zeros(n, np.uint8)
    capi.check(lib.Logic_VecNot(not_like.ctypes.data, like.ctypes.data, n, like_n.ctypes.data, 0), lib)
    b3 = bool_call(capi.XCALL_GO_IN(capi.T_INT32), n, Vector(data=size), Vector(data=np.array(SIZES, np.int32)),
                   Vector(data=np.array([len(SIZES)], np.int64)))
    assert b3[0].astype(bool).tolist() == [s in SIZES for s in d["p_size"]]
    where, wn = logic(capi.XCALL_GO_MULTI_AND, n, [b1, (not_like, like_n), b3])
    psel = ops.filter_sels(where, wn)
    want = [i for i in range(n) if d["p_brand"][i] != "Brand#35" and not d["p_type"][i].startswith("ECONOMY BURNISHED") and d["p_size"][i] in SIZES]
    assert psel.tolist() == want and want
    # the subquery: s_suppkey where s_comment like '%Customer%Complaints%'
    ns = 10
    sc, sa = strs([c.encode() for c in d["s_comment"]])
    sl, sln = bool_call(capi.XCALL_GO_LIKE, ns, Vector(data=sc, area=sa, length=ns), const_str(b"%Customer%Complaints%"))
    ssel = ops.filter_sels(sl, sln)
    sub = ops.shuffle(np.array(d["s_suppkey"], np.int32), ssel)
    assert len(sub) == 0                                          # no supplier comment of this scale matches
    # ps_suppkey NOT IN (subquery): an ANTI join of partsupp against the subquery's rows
    ps_supp = np.array(d["ps_suppkey"], np.int32)
    nps = len(ps_supp)
    jm = ops.JoinMap(sub.astype(np.uint64))
    anti, _ = jm.probe(ps_supp.astype(np.uint64), capi.JOIN_ANTI)
    jm.release()
    # ... and as GO_NOT_IN(INT32) with the subquery's rows as a device-resident list: nvalues == 0, the empty set
    d_col, d_list = DeviceBuffer.from_numpy(ps_supp), DeviceBuffer.from_numpy(np.zeros(1, np.int32))
    d_out, d_rn = DeviceBuffer(nps), DeviceBuffer.from_numpy(np.zeros((nps + 63) // 64, np.uint64))
    ops.go_in_device(capi.T_INT32, d_col, d_list, len(sub), nps, d_out, d_rn, negate=True)
    keep = d_out.to_numpy(np.uint8, nps).astype(bool)
    assert not bitmap_to_bools(d_rn.to_numpy(np.uint64), nps).any()
    for b in (d_col, d_list, d_out, d_rn):
        b.free()
    assert keep.all() and np.flatnonzero(keep).tolist() == sorted(anti.tolist()) == list(range(nps))
    # p_partkey = ps_partkey over the kept partsupp rows and the selected parts
    jm = ops.JoinMap(np.array(d["p_partkey"], np.uint64)[psel])
    probe, build = jm.probe(np.array(d["ps_partkey"], np.uint64)[anti])
    jm.release()
    ps_rows, p_rows = anti[probe], psel[build]
    m = len(ps_rows)
    bcol = (shuffle_cells(brand_cells, p_rows), brand_area)
    tcol = (shuffle_cells(type_cells, p_rows), type_area)
    scol = ops.shuffle(size, p_rows)
    supp = ops.shuffle(ps_supp, ps_rows)
    types = [capi.T_CHAR, capi.T_VARCHAR, capi.T_INT32]
    # count(distinct ps_suppkey): pass 1 groups (p_brand, p_type, p_size, ps_suppkey); pass 2 groups the first row of each pass-1 group by
    # (p_brand, p_type, p_size) and counts them
    kb, ko, _ = ops.pack_str_keys([bcol, tcol, scol, supp], types + [capi.T_INT32])
    _, first = ops.StrGroupTable().insert(kb, ko, first_rows=True)
    kb, ko, _ = ops.pack_str_keys([(shuffle_cells(bcol[0], first), brand_area), (shuffle_cells(tcol[0], first), type_area),
                                   ops.shuffle(scol, first)], types)
    tab = ops.StrGroupTable()
    gids = tab.insert(kb, ko)
    ng = int(tab.ngroups[0])
    cnt = np.zeros(ng, np.int64)
    assert ops.group_agg(capi.AGG_COUNT, capi.T_INT64, cnt, None, None, gids, np.zeros(len(first), np.int64)) == 0
    g_first = np.array([int(np.flatnonzero(gids == g + 1)[0]) for g in range(ng)])
    rows = p_rows[first[g_first]]
    g_brand = [d["p_brand"][r].encode() for r in rows]
    g_type = [d["p_type"][r].encode() for r in rows]
    g_size = size[rows]
    order = ops.order_sels([cnt, g_brand, g_type, g_size], None, [capi.ORDER_DESC, 0, 0, 0],
                           types=[capi.T_INT64, capi.T_CHAR, capi.T_VARCHAR, capi.T_INT32])
    got = [[g_brand[g].decode(), g_type[g].decode(), int(g_size[g]), int(cnt[g])] for g in order]
    assert len(got) == 41 and got == d["q16_result"]
