"""Extract the columns TPC-H Q21 reads from the reference's TPC-H load scripts into tpch_q21.json (run once; the JSON is committed).

test/distributed/cases/benchmark/tpch/02_LOAD:
  03_insert_lineitem.sql  l_orderkey (BIGINT), l_suppkey (INT), l_commitdate, l_receiptdate (DATE, days since 1970-01-01).  LINEITEM's first
                          column is L_LINEITEM_ID (01_DDL/01_create_table.sql:77-83), so l_orderkey is the second value of each tuple and
                          l_suppkey the fourth.
  05_insert_orders.sql    o_orderkey, o_orderstatus
  09_insert_supplier.sql  s_suppkey, s_name, s_nationkey
  04_insert_nation.sql    n_nationkey, n_name
Row counts are checked against 10_select_count.result; the query's expected result is 03_QUERIES/q21.result."""
import datetime
import json
import os
import re

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
LOAD = "test/distributed/cases/benchmark/tpch/02_LOAD"
DATE = r'"(\d{4})-(\d\d)-(\d\d)"'


def _read(name):
    return open(os.path.join(REF, LOAD, name)).read()


def _days(y, m, d):
    return datetime.date(int(y), int(m), int(d)).toordinal() - datetime.date(1970, 1, 1).toordinal()


def _counts():
    """table -> count(*) from 10_select_count.result"""
    return {t: int(n) for t, n in re.findall(r"select count\(\*\) from (\w+);\ncount\(\*\)\n(\d+)", _read("10_select_count.result"))}


def _q21_result():
    """03_QUERIES/q21.result: the result rows below the header line 's_name<TAB>numwait'"""
    text = open(os.path.join(REF, "test/distributed/cases/benchmark/tpch/03_QUERIES/q21.result")).read()
    body = text.split("s_name\tnumwait\n", 1)[1]
    return [line.split("\t") for line in body.splitlines() if line.strip()]


def tpch_q21():
    # (id, orderkey, partkey, suppkey, linenumber, qty, price, disc, tax, "flag", "status", "shipdate", "commitdate", "receiptdate", ...)
    li = re.findall(r'^\((\d+),(\d+),(\d+),(\d+),(\d+),[^"]*"."\s*,\s*"."\s*,\s*' + DATE + ',' + DATE + ',' + DATE,
                    _read("03_insert_lineitem.sql"), re.M)
    orders = re.findall(r'^\((\d+),(\d+),"(.)",', _read("05_insert_orders.sql"), re.M)
    supplier = re.findall(r'^\((\d+),"([^"]*)","[^"]*",(\d+),', _read("09_insert_supplier.sql"), re.M)
    nation = re.findall(r'^\((\d+),"([^"]*)",(\d+),', _read("04_insert_nation.sql"), re.M)
    counts = _counts()
    assert (len(li), len(orders), len(supplier), len(nation)) == (counts["lineitem"], counts["orders"], counts["supplier"], counts["nation"]), \
        (len(li), len(orders), len(supplier), len(nation), counts)
    return {"_source": "%s: 03_insert_lineitem.sql, 05_insert_orders.sql, 09_insert_supplier.sql, 04_insert_nation.sql (row counts of "
                       "10_select_count.result); dates are days since 1970-01-01; expected result: 03_QUERIES/q21.result" % LOAD,
            "counts": {"lineitem": len(li), "orders": len(orders), "supplier": len(supplier), "nation": len(nation)},
            "l_orderkey": [int(r[1]) for r in li], "l_suppkey": [int(r[3]) for r in li],
            "l_commitdate": [_days(*r[8:11]) for r in li], "l_receiptdate": [_days(*r[11:14]) for r in li],
            "o_orderkey": [int(r[0]) for r in orders], "o_orderstatus": "".join(r[2] for r in orders),
            "s_suppkey": [int(r[0]) for r in supplier], "s_name": [r[1] for r in supplier], "s_nationkey": [int(r[2]) for r in supplier],
            "n_nationkey": [int(r[0]) for r in nation], "n_name": [r[1] for r in nation],
            "q21_result": _q21_result()}


if __name__ == "__main__":
    with open(os.path.join(OUT, "tpch_q21.json"), "w") as f:
        json.dump(tpch_q21(), f, separators=(",", ":"))
