"""Extract LIKE known answers from the reference into like_kat.json (run once; the JSON is committed).

  pkg/sql/plan/function/func_builtin_regexp_test.go  Test_BuiltIn_RegularMatchForLikeOp: {pat, str, expected} passed straight to
                                                     regularMatchForLikeOp -- the rune-level matcher ("tier": "regular").  The Go
                                                     string literals are unescaped with Go's rules (go_unquote).
  test/distributed/cases/operator/like_operator.result, function/func_like.result
                                                     every `SELECT <literal> [NOT] LIKE <literal> [AS name];` and the one value below its
                                                     header line.  Both operands are const, so likeFn applies optimizeRuleForLike first
                                                     ("tier": "like").  The literals are unescaped as the SQL scanner does (sql_unquote).
Values are stored as hex strings of their bytes."""
import json
import os
import re

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))

# a single- or double-quoted SQL string literal, doubled delimiters and backslash escapes included
SQL_LIT = r"""('(?:[^'\\]|\\.|'')*'|"(?:[^"\\]|\\.|"")*")"""
SELECT_LIKE = re.compile(r"^select\s+" + SQL_LIT + r"\s+(not\s+)?like\s+" + SQL_LIT + r"(?:\s+as\s+\w+)?\s*;\s*$", re.I)


def sql_unquote(lit):
    """Scanner.scanString + handleEscape (pkg/sql/parsers/dialect/mysql/scanner.go:519-540): a doubled delimiter is one delimiter;
    \\n \\0 \\b \\Z \\r \\t are control bytes; \\% and \\_ keep their backslash (LIKE sees the escape); any other \\x is x."""
    delim, body = lit[0:1], lit[1:-1]
    out, i = bytearray(), 0
    while i < len(body):
        c = body[i:i + 1]
        if c == delim and body[i + 1:i + 2] == delim:
            out += delim
            i += 2
            continue
        if c == b"\\" and i + 1 < len(body):
            x = body[i + 1:i + 2]
            if x in (b"%", b"_"):
                out += b"\\" + x
            else:
                out += {b"n": b"\n", b"0": b"\0", b"b": b"\b", b"Z": b"\x1a", b"r": b"\r", b"t": b"\t"}.get(x, x)
            i += 2
            continue
        out += c
        i += 1
    return bytes(out)


def go_unquote(lit):
    """a Go interpreted string literal's body: \\\\ \\" \\n \\t"""
    out, i = bytearray(), 0
    while i < len(lit):
        if lit[i:i + 1] == b"\\":
            out += {b"\\": b"\\", b'"': b'"', b"n": b"\n", b"t": b"\t"}[lit[i + 1:i + 2]]
            i += 2
        else:
            out += lit[i:i + 1]
            i += 1
    return bytes(out)


def regular_cases():
    path = "pkg/sql/plan/function/func_builtin_regexp_test.go"
    src = open(os.path.join(REF, path), "rb").read()
    body = src.split(b"func Test_BuiltIn_RegularMatchForLikeOp", 1)[1].split(b"\nfunc ", 1)[0]
    rows = re.findall(rb'\{pat: "((?:[^"\\]|\\.)*)", str: "((?:[^"\\]|\\.)*)", expected: (true|false)\}', body)
    assert rows, "no cases found"
    return [{"source": path, "tier": "regular", "pat": go_unquote(p).hex(), "str": go_unquote(s).hex(), "not": False,
             "expected": e == b"true"} for p, s, e in rows]


def sql_cases(rel):
    lines = open(os.path.join(REF, rel), "rb").read().split(b"\n")
    out = []
    for k, line in enumerate(lines):
        m = SELECT_LIKE.match(line.decode("utf-8", "surrogateescape"))
        if not m:
            continue
        value = lines[k + 2].strip()                     # the statement, its header line, then the value
        assert value in (b"0", b"1"), (rel, k + 1, value)
        enc = lambda t: t.encode("utf-8", "surrogateescape")
        out.append({"source": "%s:%d" % (rel, k + 1), "tier": "like", "str": sql_unquote(enc(m.group(1))).hex(),
                    "pat": sql_unquote(enc(m.group(3))).hex(), "not": m.group(2) is not None, "expected": value == b"1"})
    return out


def main():
    cases = regular_cases()
    for rel in ("test/distributed/cases/operator/like_operator.result", "test/distributed/cases/function/func_like.result"):
        cases += sql_cases(rel)
    with open(os.path.join(OUT, "like_kat.json"), "w") as f:
        json.dump({"_source": __doc__.splitlines()[0], "cases": cases}, f, indent=0)
    print(len(cases), "cases")


if __name__ == "__main__":
    main()
