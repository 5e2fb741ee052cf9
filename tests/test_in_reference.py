"""in_reference.py against the reference's own IN / NOT IN results (golden/in_kat.json, from operator.result), and its rules at the edges
operator_in.go pins: NULL elements of the list, NULL rows, float +-0 and NaN."""
import json
import os

import numpy as np

import in_reference as R

KAT = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "in_kat.json")))
DTYPES = {"int32": np.int32, "float32": np.uint32, "date": np.int32, "datetime": np.int64}


def typed(col, vals):
    """the JSON's cast values of column `col` as the column's element type (float32 from its bits, varchar as bytes)"""
    t = KAT["columns"][col]
    if t == "varchar":
        return [bytes.fromhex(v) for v in vals]
    a = np.array(vals, dtype=DTYPES[t])
    return a.view(np.float32) if t == "float32" else a


def selected(stmt):
    """rows every IN / NOT IN of the WHERE clause holds for (the table has no NULLs)"""
    keep = np.ones(len(KAT["rows"]), bool)
    for c in stmt["where"]:
        k = "abcde".index(c["col"])
        col = typed(c["col"], [r["values"][k] for r in KAT["rows"]])
        got, nulls = R.evaluate(col, None, typed(c["col"], c["values"]), negate=c["negate"])
        assert not any(nulls)
        keep &= np.array(got, bool)
    return [r for r, k in zip(KAT["rows"], keep) if k]


def test_statements_match_the_reference_results():
    assert len(KAT["statements"]) == 9
    for s in KAT["statements"]:
        rows = selected(s)
        if s["sql"].startswith("select * "):
            got = [r["text"] for r in rows]
        else:                                              # sum(a) grouped by the one other output column, in its order
            g = 2 if ",c " in s["sql"] else 4
            sums = {}
            for r in rows:
                sums[r["text"][g]] = sums.get(r["text"][g], 0) + r["values"][0]
            got = sorted([[str(v), k] for k, v in sums.items()], key=lambda x: (int(x[0]), x[1]) if "suma" in s["sql"] else x[1])
        assert got == s["result"], s["sql"]


def test_go_map_equality_and_null_rules():
    f = np.float64
    col = [f(0.0), f(-0.0), f("nan"), f(1.5), f(2.0)]
    vals, vn = [f(-0.0), f("nan"), f(1.5), f(7.0)], [False, False, True, False]
    got, nulls = R.evaluate(col, [False, False, False, False, True], vals, vn)
    assert got == [True, True, False, False, None] and nulls == [False] * 4 + [True]
    got, _ = R.evaluate(col[:4], None, vals, vn, negate=True)
    assert got == [False, False, True, True]          # NaN NOT IN (...) is true; a NULL element nulls no row
    assert R.evaluate([np.int64(2)], None, [np.int64(1), np.int64(0)], [False, True], negate=True)[0] == [True]
    assert R.evaluate([b"ab", b"ab "], None, [b"ab"])[0] == [True, False]   # bytes: no trimming
    assert R.evaluate([np.int32(3)], None, [np.int32(3)], [True])[0] == [False]   # a const NULL list is the empty set
