"""Extract the columns TPC-H Q13 reads from the reference's TPC-H load scripts into tpch_q13.json (run once; the JSON is committed).

test/distributed/cases/benchmark/tpch/02_LOAD:
  02_insert_customer.sql  c_custkey (the first value of each tuple)
  05_insert_orders.sql    o_orderkey, o_custkey, o_comment (VARCHAR(79), the last value; the file's comments hold no backslash or quote, so
                          the double-quoted literal is the value's bytes)
Row counts are checked against 10_select_count.result; the query's expected result is 03_QUERIES/q13.result."""
import json
import os
import re

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
TPCH = "test/distributed/cases/benchmark/tpch"
LOAD = TPCH + "/02_LOAD"


def _read(name):
    return open(os.path.join(REF, LOAD, name)).read()


def _counts():
    return {t: int(n) for t, n in re.findall(r"select count\(\*\) from (\w+);\ncount\(\*\)\n(\d+)", _read("10_select_count.result"))}


def _q13_result():
    """03_QUERIES/q13.result: the rows below the header line 'c_count<TAB>custdist'"""
    text = open(os.path.join(REF, TPCH, "03_QUERIES/q13.result")).read()
    body = text.split("c_count\tcustdist\n", 1)[1]
    return [[int(x) for x in line.split("\t")] for line in body.splitlines() if line.strip()]


def tpch_q13():
    customer = re.findall(r'^\((\d+),"', _read("02_insert_customer.sql"), re.M)
    src = _read("05_insert_orders.sql")
    assert "\\" not in src
    # (orderkey, custkey, "status", totalprice, "date", "priority", "clerk", shippriority, "comment")
    orders = re.findall(r'^\((\d+),(\d+),"[^"]*",[\d.]+,"[^"]*","[^"]*","[^"]*",\d+,"([^"]*)"\)[,;]$', src, re.M)
    counts = _counts()
    assert (len(customer), len(orders)) == (counts["customer"], counts["orders"]), (len(customer), len(orders), counts)
    return {"_source": "%s: 02_insert_customer.sql, 05_insert_orders.sql (row counts of 10_select_count.result); expected result: "
                       "03_QUERIES/q13.result as [c_count, custdist] rows" % LOAD,
            "counts": {"customer": len(customer), "orders": len(orders)},
            "c_custkey": [int(r) for r in customer],
            "o_orderkey": [int(r[0]) for r in orders], "o_custkey": [int(r[1]) for r in orders], "o_comment": [r[2] for r in orders],
            "q13_result": _q13_result()}


if __name__ == "__main__":
    with open(os.path.join(OUT, "tpch_q13.json"), "w") as f:
        json.dump(tpch_q13(), f)
