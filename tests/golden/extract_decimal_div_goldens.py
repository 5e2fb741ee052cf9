"""Extract decimal division, AVG and comparison results from the reference's SQL test file into decimal_div_kat.json (run once; the JSON
is committed).

Source: test/distributed/cases/dtype/decimal.result.  The file is replayed statement by statement as far as these checks need: CREATE
TABLE gives each DECIMAL(p, s) column its scale, INSERT adds rows, DROP removes the table.  A statement is taken when it is one of
    select <x> / <y> from <t>;              x, y a DECIMAL column of t or a numeric literal
    select avg(<c>) from <t>;
    select * from <t> where <c> <op> <lit>; select count(*) from <t> where <c> <op> <lit>;     op one of = != <> > >= < <=
and every operand value is known exactly at its column's scale.  A table is no longer used once an INSERT into it gives a value with more
fractional digits than the column's scale, a value that is not a plain numeric literal, or an error, or once it is UPDATEd, DELETEd from,
ALTERed or TRUNCATEd.  Each skipped candidate statement is recorded with its reason.  The result scale of a division or an AVG is the last
number of the `[type,precision,scale]` header; a comparison is recorded as the number of rows the statement returns."""
import json
import os
import re
from decimal import Decimal

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
SRC = "test/distributed/cases/dtype/decimal.result"
NUM = re.compile(r"^[+-]?\d+(\.\d+)?$")
OPS = {"=": 0, "!=": 1, "<>": 1, ">": 2, ">=": 3, "<": 4, "<=": 5}
SQL_START = re.compile(r"^(select|insert|create|drop|update|delete|alter|truncate|use|set|show|prepare|execute|begin|commit|rollback|explain|with|desc|describe|start|deallocate|analyze)\b", re.I)


def _statements(lines):
    """(line number, sql text, result lines) in file order"""
    out, i = [], 0
    while i < len(lines):
        if not SQL_START.match(lines[i].strip()):
            i += 1
            continue
        start, sql = i + 1, lines[i].strip()
        while not sql.endswith(";") and i + 1 < len(lines):
            i += 1
            sql += " " + lines[i].strip()
        i += 1
        res = []
        while i < len(lines) and not SQL_START.match(lines[i].strip()):
            res.append(lines[i])
            i += 1
        out.append((start, sql, res))
    return out


def _split_top(s):
    parts, depth, cur = [], 0, ""
    for ch in s:
        if ch == "(":
            depth += 1
        elif ch == ")":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append(cur.strip())
            cur = ""
        else:
            cur += ch
    if cur.strip():
        parts.append(cur.strip())
    return parts


def _unscaled(lit, scale):
    """a numeric literal as its unscaled integer at `scale`, or None when it has more fractional digits"""
    if not NUM.match(lit):
        return None
    frac = lit.split(".")[1] if "." in lit else ""
    if len(frac) > scale:
        return None
    return int(Decimal(lit).scaleb(scale))


def _lit(lit):
    """a numeric literal operand: (unscaled, scale, precision)"""
    frac = lit.split(".")[1] if "." in lit else ""
    digits = len(lit.lstrip("+-").replace(".", "").lstrip("0")) or 1
    return int(Decimal(lit).scaleb(len(frac))), len(frac), max(digits, len(frac))


def _result(res):
    """(header scale, value strings) of a result block, or None for an error"""
    if not res or not res[0].startswith("➤"):
        return None
    m = re.search(r"\[(\d+),(\d+),(\d+)\]", res[0])
    vals = [line.split("  𝄀")[0].strip() for line in res[1:] if line.strip()]
    return (int(m.group(3)) if m else None), vals


def extract():
    lines = open(os.path.join(REF, SRC)).read().split("\n")
    tables, div, avg, cmp, skipped = {}, [], [], [], []
    for ln, sql, res in _statements(lines):
        low = sql.lower()
        m = re.match(r"create table (?:if not exists )?(\w+)\s*\((.*)\)\s*;$", sql, re.I)
        if m:
            cols, order = {}, []
            for part in _split_top(m.group(2)):
                w = part.split()
                if not w or w[0].lower() in ("primary", "key", "unique", "index", "constraint", "foreign"):
                    continue
                order.append(w[0].lower())
                dm = re.match(r"\w+\s+decimal\s*\(\s*(\d+)\s*(?:,\s*(\d+)\s*)?\)", part, re.I)
                if dm:
                    cols[w[0].lower()] = (int(dm.group(1)), int(dm.group(2) or 0))
            ok = _result(res) is None and not any(line.strip() for line in res)
            tables[m.group(1).lower()] = {"cols": cols, "order": order, "rows": [], "usable": ok, "why": "" if ok else "CREATE failed"}
            continue
        m = re.match(r"insert into (\w+)\s*(?:\(([^)]*)\))?\s*values\s*(.*);$", sql, re.I)
        if m and m.group(1).lower() in tables:
            t = tables[m.group(1).lower()]
            names = [c.strip().lower() for c in m.group(2).split(",")] if m.group(2) else t["order"]
            if any(line.strip() for line in res):
                t["usable"], t["why"] = False, "an INSERT failed (line %d)" % ln
                continue
            for tup in re.findall(r"\(([^()]*)\)", m.group(3)):
                vals = [v.strip() for v in _split_top(tup)]
                row = {}
                for c, v in zip(names, vals):
                    if c not in t["cols"]:
                        continue
                    if v.upper() == "NULL":
                        row[c] = None
                        continue
                    p, s = t["cols"][c]
                    u = _unscaled(v, s)
                    if u is None or abs(u) >= 10 ** p:
                        t["usable"], t["why"] = False, "value %s is not exact at DECIMAL(%d,%d) (line %d)" % (v, p, s, ln)
                    row[c] = u
                for c in t["cols"]:
                    row.setdefault(c, None)
                t["rows"].append(row)
            continue
        m = re.match(r"(?:update|delete from|alter table|truncate(?: table)?)\s+(\w+)", sql, re.I)
        if m and m.group(1).lower() in tables:
            tables[m.group(1).lower()]["usable"] = False
            tables[m.group(1).lower()]["why"] = "the table is modified (line %d)" % ln
            continue
        m = re.match(r"drop table (?:if exists )?(\w+)", sql, re.I)
        if m:
            tables.pop(m.group(1).lower(), None)
            continue
        if not low.startswith("select"):
            continue
        is_div = re.match(r"select\s+([\w.+-]+)\s*/\s*([\w.+-]+)\s+from\s+(\w+)\s*;$", sql, re.I)
        is_avg = re.match(r"select\s+avg\((\w+)\)\s+from\s+(\w+)\s*;$", sql, re.I)
        is_cmp = re.match(r"select\s+(\*|count\(\*\))\s+from\s+(\w+)\s+where\s+(\w+)\s*(<>|!=|>=|<=|=|>|<)\s*([+-]?[\d.]+)\s*;$", sql, re.I)
        candidate = re.search(r"/|avg\(|where\s+\w+\s*(<>|!=|>=|<=|=|>|<)", low)
        if not (is_div or is_avg or is_cmp):
            if candidate:
                skipped.append({"line": ln, "sql": sql, "reason": "not a single division, AVG or column-constant comparison over one table"})
            continue
        tname = (is_div.group(3) if is_div else is_avg.group(2) if is_avg else is_cmp.group(2)).lower()
        t = tables.get(tname)
        r = _result(res)
        if t is None or not t["usable"]:
            skipped.append({"line": ln, "sql": sql, "reason": "table %s: %s" % (tname, "unknown" if t is None else t["why"])})
            continue
        if r is None:
            skipped.append({"line": ln, "sql": sql, "reason": "the statement returns an error"})
            continue
        if is_div:
            ops = []
            for x in (is_div.group(1).lower(), is_div.group(2).lower()):
                if x in t["cols"]:
                    p, s = t["cols"][x]
                    ops.append({"col": x, "scale": s, "precision": p, "values": [row[x] for row in t["rows"]]})
                elif NUM.match(x):
                    u, s, p = _lit(x)
                    ops.append({"const": u, "scale": s, "precision": p})
                else:
                    ops = None
                    break
            if ops is None:
                skipped.append({"line": ln, "sql": sql, "reason": "an operand is neither a DECIMAL column nor a numeric literal"})
                continue
            div.append({"line": ln, "sql": sql, "a": ops[0], "b": ops[1], "result_scale": r[0], "result": r[1]})
        elif is_avg:
            c = is_avg.group(1).lower()
            if c not in t["cols"]:
                skipped.append({"line": ln, "sql": sql, "reason": "not a DECIMAL column"})
                continue
            p, s = t["cols"][c]
            avg.append({"line": ln, "sql": sql, "scale": s, "precision": p, "values": [row[c] for row in t["rows"]], "result_scale": r[0],
                        "result": r[1]})
        else:
            c = is_cmp.group(3).lower()
            if c not in t["cols"]:
                skipped.append({"line": ln, "sql": sql, "reason": "not a DECIMAL column"})
                continue
            p, s = t["cols"][c]
            u, ls, lp = _lit(is_cmp.group(5))
            rows = int(r[1][0]) if is_cmp.group(1) != "*" else len(r[1])
            cmp.append({"line": ln, "sql": sql, "op": OPS[is_cmp.group(4)], "scale": s, "precision": p, "values": [row[c] for row in t["rows"]],
                        "const": u, "const_scale": ls, "const_precision": lp, "rows": rows})
    return {"_source": SRC + ", replayed as tests/golden/extract_decimal_div_goldens.py describes", "div": div, "avg": avg, "compare": cmp,
            "skipped": skipped}


if __name__ == "__main__":
    with open(os.path.join(OUT, "decimal_div_kat.json"), "w") as f:
        json.dump(extract(), f, indent=1, ensure_ascii=False)
