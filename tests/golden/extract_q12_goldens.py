"""Extract the columns TPC-H Q12 reads from the reference's TPC-H load scripts into tpch_q12.json (run once; the JSON is committed).

test/distributed/cases/benchmark/tpch/02_LOAD:
  03_insert_lineitem.sql  l_orderkey (the second value: LINEITEM's first column is L_LINEITEM_ID), l_shipdate, l_commitdate, l_receiptdate
                          (DATE, days since 1970-01-01) and l_shipmode (CHAR(10))
  05_insert_orders.sql    o_orderkey, o_orderpriority (CHAR(15))
Row counts are checked against 10_select_count.result; the query's expected result is 03_QUERIES/q12.result."""
import datetime
import json
import os
import re

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
TPCH = "test/distributed/cases/benchmark/tpch"
LOAD = TPCH + "/02_LOAD"


def _read(name):
    return open(os.path.join(REF, LOAD, name)).read()


def tuples(name):
    """the value tuples of an insert script: each line '(v, v, ...),' or '...;' -- a value is a double-quoted string (no escapes in these
    files) or a number"""
    src = _read(name)
    assert "\\" not in src
    return [[s if n == "" else n for s, n in re.findall(r'"([^"]*)"|(-?[\d.]+)', ln)] for ln in src.splitlines() if ln.startswith("(")]


def counts():
    return {t: int(n) for t, n in re.findall(r"select count\(\*\) from (\w+);\ncount\(\*\)\n(\d+)", _read("10_select_count.result"))}


def days(s):
    return datetime.date.fromisoformat(s).toordinal() - datetime.date(1970, 1, 1).toordinal()


def result(q, header):
    body = open(os.path.join(REF, TPCH, "03_QUERIES", q)).read().split(header + "\n", 1)[1]
    return [line.split("\t") for line in body.splitlines() if line.strip()]


def tpch_q12():
    li, orders, c = tuples("03_insert_lineitem.sql"), tuples("05_insert_orders.sql"), counts()
    assert all(len(r) == 17 for r in li) and all(len(r) == 9 for r in orders)
    assert (len(li), len(orders)) == (c["lineitem"], c["orders"]), (len(li), len(orders), c)
    return {"_source": "%s: 03_insert_lineitem.sql, 05_insert_orders.sql (row counts of 10_select_count.result); expected result: "
                       "03_QUERIES/q12.result as [l_shipmode, high_line_count, low_line_count] rows" % LOAD,
            "counts": {"lineitem": len(li), "orders": len(orders)},
            "l_orderkey": [int(r[1]) for r in li], "l_shipdate": [days(r[11]) for r in li], "l_commitdate": [days(r[12]) for r in li],
            "l_receiptdate": [days(r[13]) for r in li], "l_shipmode": [r[15] for r in li],
            "o_orderkey": [int(r[0]) for r in orders], "o_orderpriority": [r[5] for r in orders],
            "q12_result": [[m, int(h), int(lo)] for m, h, lo in result("q12.result", "l_shipmode\thigh_line_count\tlow_line_count")]}


if __name__ == "__main__":
    with open(os.path.join(OUT, "tpch_q12.json"), "w") as f:
        json.dump(tpch_q12(), f)
