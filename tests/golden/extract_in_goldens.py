"""Extract the IN / NOT IN cases of the reference's operator test into in_kat.json (run once; the JSON is committed).

test/distributed/cases/operator/operator.result:219-257: the table t2(a int, b varchar(5), c float, d date, e datetime), its four rows, and
the nine statements whose WHERE clause is a conjunction of `col [not] in (literals)`.  For each literal the planner's cast to the column's
type is recorded: INT as int32, VARCHAR as its bytes (hex), FLOAT as the float32 bits, DATE as types.Date (days since 0001-01-01, both
'YYYY-MM-DD' and 'YYYYMMDD' spellings) and DATETIME as types.Datetime (microseconds since 0001-01-01 00:00:00).  Each statement's result
rows are recorded as the file prints them."""
import datetime
import json
import os
import re
import struct

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
SRC = "test/distributed/cases/operator/operator.result"
FIRST, LAST = 219, 257
COLS = {"a": "int32", "b": "varchar", "c": "float32", "d": "date", "e": "datetime"}


def cast(col, lit):
    t = COLS[col]
    lit = lit.strip()
    if lit[0] in "'\"":
        lit = lit[1:-1]
    if t == "int32":
        return int(lit)
    if t == "varchar":
        return lit.encode().hex()
    if t == "float32":
        return struct.unpack("<I", struct.pack("<f", float(lit)))[0]
    if t == "date":
        d = datetime.datetime.strptime(lit, "%Y-%m-%d" if "-" in lit else "%Y%m%d").date()
        return d.toordinal() - 1
    dt = datetime.datetime.strptime(lit, "%Y-%m-%d %H:%M:%S")
    return ((dt.date().toordinal() - 1) * 86400 + dt.hour * 3600 + dt.minute * 60 + dt.second) * 1000000


def main():
    lines = open(os.path.join(REF, SRC)).read().splitlines()[FIRST - 1:LAST]
    assert lines[0] == "drop table if exists t2;" and lines[1].startswith("create table t2("), lines[:2]
    rows, stmts = [], []
    i = 2
    while i < len(lines):
        ln = lines[i]
        m = re.match(r"insert into t2 values\((.*)\);$", ln)
        if m:
            vals = [v.strip().strip("'") for v in m.group(1).split(",")]
            rows.append({"text": vals, "values": [cast(c, v) for c, v in zip("abcde", vals)]})
            i += 1
            continue
        assert ln.startswith("select "), ln
        conds = [{"col": c, "negate": bool(n.strip()), "values": [cast(c, v) for v in re.findall(r"'[^']*'|\"[^\"]*\"|[^,]+", lits)]}
                 for c, n, lits in re.findall(r"\b([a-e]) (not )?in \(([^)]*)\)", ln)]
        assert conds, ln
        i += 2                                            # the statement, then the header line of its result
        result = []
        while i < len(lines) and not lines[i].startswith(("select ", "drop ")):
            result.append([f.strip() for f in lines[i].replace("  𝄀", "").split("  ¦  ")])
            i += 1
        stmts.append({"sql": ln, "where": conds, "result": result})
        if lines[i - 1].startswith("drop "):
            break
    assert len(rows) == 4 and len(stmts) == 9, (len(rows), len(stmts))
    with open(os.path.join(OUT, "in_kat.json"), "w") as f:
        json.dump({"source": "%s:%d-%d" % (SRC, FIRST, LAST), "columns": COLS, "rows": rows, "statements": stmts}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
