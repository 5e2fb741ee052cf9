"""Extract the columns TPC-H Q15 reads from the reference's TPC-H load scripts into tpch_q15.json (run once; the JSON is committed).

test/distributed/cases/benchmark/tpch/02_LOAD:
  03_insert_lineitem.sql  l_suppkey (INT), l_extendedprice, l_discount (DECIMAL(15,2), kept as their unscaled integers at scale 2) and
                          l_shipdate (DATE, days since 1970-01-01).  LINEITEM's first column is L_LINEITEM_ID (01_DDL/01_create_table.sql:77-83),
                          so l_suppkey is the fourth value of each tuple.
  09_insert_supplier.sql  s_suppkey, s_name, s_address, s_phone
Row counts are checked against 10_select_count.result; the query's expected result is 03_QUERIES/q15.result."""
import datetime
import json
import os
import re

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
LOAD = "test/distributed/cases/benchmark/tpch/02_LOAD"
DATE = r'"(\d{4})-(\d\d)-(\d\d)"'
DEC2 = r'(-?\d+)\.(\d\d)'


def _read(name):
    return open(os.path.join(REF, LOAD, name)).read()


def _days(y, m, d):
    return datetime.date(int(y), int(m), int(d)).toordinal() - datetime.date(1970, 1, 1).toordinal()


def _counts():
    """table -> count(*) from 10_select_count.result"""
    return {t: int(n) for t, n in re.findall(r"select count\(\*\) from (\w+);\ncount\(\*\)\n(\d+)", _read("10_select_count.result"))}


def _cents(whole, frac):
    return int(whole) * 100 + (-1 if whole.startswith("-") else 1) * int(frac)


def _q15_result():
    text = open(os.path.join(REF, "test/distributed/cases/benchmark/tpch/03_QUERIES/q15.result")).read()
    body = text.split("s_suppkey\ts_name\ts_address\ts_phone\ttotal_revenue\n", 1)[1]
    return [line.split("\t") for line in body.splitlines() if line.strip()]


def tpch_q15():
    # (id, orderkey, partkey, suppkey, linenumber, qty, price, disc, tax, "flag", "status", "shipdate", ...)
    li = re.findall(r'^\(\d+,\d+,\d+,(\d+),\d+,[^,]+,' + DEC2 + ',' + DEC2 + r',[^,]+,"."\s*,\s*"."\s*,\s*' + DATE, _read("03_insert_lineitem.sql"), re.M)
    supplier = re.findall(r'^\((\d+),"([^"]*)","([^"]*)",\d+,"([^"]*)",', _read("09_insert_supplier.sql"), re.M)
    counts = _counts()
    assert (len(li), len(supplier)) == (counts["lineitem"], counts["supplier"]), (len(li), len(supplier), counts)
    return {"_source": "%s: 03_insert_lineitem.sql, 09_insert_supplier.sql (row counts of 10_select_count.result); l_extendedprice and "
                       "l_discount are unscaled at scale 2; dates are days since 1970-01-01; expected result: 03_QUERIES/q15.result" % LOAD,
            "counts": {"lineitem": len(li), "supplier": len(supplier)},
            "l_suppkey": [int(r[0]) for r in li], "l_extendedprice": [_cents(r[1], r[2]) for r in li],
            "l_discount": [_cents(r[3], r[4]) for r in li], "l_shipdate": [_days(*r[5:8]) for r in li],
            "s_suppkey": [int(r[0]) for r in supplier], "s_name": [r[1] for r in supplier], "s_address": [r[2] for r in supplier],
            "s_phone": [r[3] for r in supplier], "q15_result": _q15_result()}


if __name__ == "__main__":
    with open(os.path.join(OUT, "tpch_q15.json"), "w") as f:
        json.dump(tpch_q15(), f, separators=(",", ":"))
