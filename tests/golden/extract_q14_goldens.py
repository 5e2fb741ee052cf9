"""Extract the columns TPC-H Q14 reads from the reference's TPC-H load scripts into tpch_q14.json (run once; the JSON is committed).

test/distributed/cases/benchmark/tpch/02_LOAD:
  03_insert_lineitem.sql  l_partkey, l_extendedprice and l_discount (DECIMAL(15,2), as integers at scale 2), l_shipdate (DATE, days since
                          1970-01-01)
  06_insert_part.sql      p_partkey, p_type (VARCHAR(25))
Row counts are checked against 10_select_count.result; the query's expected result is 03_QUERIES/q14.result, recorded as printed."""
import decimal
import json
import os

from extract_q12_goldens import LOAD, OUT, REF, TPCH, counts, days, tuples


def cents(s):
    v = decimal.Decimal(s) * 100
    assert v == v.to_integral_value(), s
    return int(v)


def tpch_q14():
    li, part, c = tuples("03_insert_lineitem.sql"), tuples("06_insert_part.sql"), counts()
    assert all(len(r) == 17 for r in li) and all(len(r) == 9 for r in part)
    assert (len(li), len(part)) == (c["lineitem"], c["part"]), (len(li), len(part), c)
    res = open(os.path.join(REF, TPCH, "03_QUERIES", "q14.result")).read().split("\npromo_revenue\n", 1)[1].split()
    assert len(res) == 1
    return {"_source": "%s: 03_insert_lineitem.sql, 06_insert_part.sql (row counts of 10_select_count.result); expected result: "
                       "03_QUERIES/q14.result's promo_revenue as printed" % LOAD,
            "counts": {"lineitem": len(li), "part": len(part)},
            "l_partkey": [int(r[2]) for r in li], "l_extendedprice": [cents(r[6]) for r in li], "l_discount": [cents(r[7]) for r in li],
            "l_shipdate": [days(r[11]) for r in li],
            "p_partkey": [int(r[0]) for r in part], "p_type": [r[4] for r in part],
            "q14_result": res[0]}


if __name__ == "__main__":
    with open(os.path.join(OUT, "tpch_q14.json"), "w") as f:
        json.dump(tpch_q14(), f)
