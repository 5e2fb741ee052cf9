"""Extract the columns TPC-H Q16 reads from the reference's TPC-H load scripts into tpch_q16.json (run once; the JSON is committed).

test/distributed/cases/benchmark/tpch/02_LOAD:
  06_insert_part.sql      p_partkey, p_brand (CHAR(10)), p_type (VARCHAR(25)), p_size
  07_insert_partsupp.sql  ps_partkey, ps_suppkey
  09_insert_supplier.sql  s_suppkey, s_comment (VARCHAR(101))
Row counts are checked against 10_select_count.result (200 / 800 / 10); the query's expected result is 03_QUERIES/q16.result (41 rows)."""
import json
import os

from extract_q12_goldens import LOAD, OUT, counts, result, tuples


def tpch_q16():
    part, ps, supp, c = tuples("06_insert_part.sql"), tuples("07_insert_partsupp.sql"), tuples("09_insert_supplier.sql"), counts()
    assert all(len(r) == 9 for r in part) and all(len(r) == 5 for r in ps) and all(len(r) == 7 for r in supp)
    assert (len(part), len(ps), len(supp)) == (c["part"], c["partsupp"], c["supplier"]) == (200, 800, 10), (len(part), len(ps), len(supp), c)
    res = [[b, t, int(s), int(n)] for b, t, s, n in result("q16.result", "p_brand\tp_type\tp_size\tsupplier_cnt")]
    assert len(res) == 41
    return {"_source": "%s: 06_insert_part.sql, 07_insert_partsupp.sql, 09_insert_supplier.sql (row counts of 10_select_count.result); "
                       "expected result: 03_QUERIES/q16.result as [p_brand, p_type, p_size, supplier_cnt] rows" % LOAD,
            "counts": {"part": len(part), "partsupp": len(ps), "supplier": len(supp)},
            "p_partkey": [int(r[0]) for r in part], "p_brand": [r[3] for r in part], "p_type": [r[4] for r in part],
            "p_size": [int(r[5]) for r in part],
            "ps_partkey": [int(r[0]) for r in ps], "ps_suppkey": [int(r[1]) for r in ps],
            "s_suppkey": [int(r[0]) for r in supp], "s_comment": [r[6] for r in supp],
            "q16_result": res}


if __name__ == "__main__":
    with open(os.path.join(OUT, "tpch_q16.json"), "w") as f:
        json.dump(tpch_q16(), f)
