"""Transcribe the ORDER BY results of the reference's TPC-H queries whose last stage sorts by string keys into tests/golden/order_kat.json
(data only; no test reads the reference tree).

Run in the build container (needs /root/reference):   python tests/golden/extract_order_goldens.py

Source: test/distributed/cases/benchmark/tpch/03_QUERIES/q{16,2,20,21,1}.result (tiny dataset): the result rows in the order the reference
printed them (tab-separated after the statement's closing ';'; q1 is space-separated), with each query's ORDER BY and LIMIT and the key
columns' types from 01_DDL/01_create_table.sql (CHAR / VARCHAR as bytes, DECIMAL(15,2) as cents, INTEGER / BIGINT as ints).
"""
import json
import os

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))

SPEC = {
    "q16": {"order_by": [["supplier_cnt", "desc"], ["p_brand", "asc"], ["p_type", "asc"], ["p_size", "asc"]], "limit": None,
            "types": {"p_brand": "CHAR(10)", "p_type": "VARCHAR(25)", "p_size": "INTEGER", "supplier_cnt": "BIGINT"}},
    "q2": {"order_by": [["s_acctbal", "desc"], ["n_name", "asc"], ["s_name", "asc"], ["p_partkey", "asc"]], "limit": 100,
           "types": {"s_acctbal": "DECIMAL(15,2)", "n_name": "CHAR(25)", "s_name": "CHAR(25)", "p_partkey": "INTEGER"}},
    "q20": {"order_by": [["s_name", "asc"]], "limit": None, "types": {"s_name": "CHAR(25)"}},
    "q21": {"order_by": [["numwait", "desc"], ["s_name", "asc"]], "limit": 100, "types": {"s_name": "CHAR(25)", "numwait": "BIGINT"}},
    "q1": {"order_by": [["l_returnflag", "asc"], ["l_linestatus", "asc"]], "limit": None,
           "types": {"l_returnflag": "VARCHAR(1)", "l_linestatus": "VARCHAR(1)"}},
}


def order_result_kats():
    base = os.path.join(REF, "test/distributed/cases/benchmark/tpch/03_QUERIES")
    out = {"_source": "test/distributed/cases/benchmark/tpch/03_QUERIES/q{16,2,20,21,1}.result (tiny dataset), key types of "
                      "01_DDL/01_create_table.sql"}
    for q, s in SPEC.items():
        lines = open(os.path.join(base, q + ".result")).read().rstrip("\n").split("\n")
        end = max(i for i, l in enumerate(lines) if l.strip() == ";")
        split = (lambda l: l.split()) if q == "q1" else (lambda l: l.split("\t"))
        cols = split(lines[end + 1])
        rows = [split(l) for l in lines[end + 2:] if l.strip()]
        assert all(len(r) == len(cols) for r in rows), q
        out[q] = dict(s, columns=cols, rows=rows)
    return out


def main():
    data = order_result_kats()
    with open(os.path.join(OUT, "order_kat.json"), "w") as f:
        json.dump(data, f, indent=0)
    print("order_kat", {k: len(v["rows"]) for k, v in data.items() if not k.startswith("_")})


if __name__ == "__main__":
    main()
