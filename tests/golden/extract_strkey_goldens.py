"""Transcribe the reference's StrHashMap iterator test into tests/golden/strhashmap_kat.json (data only; no test reads the reference tree).

Run in the build container (needs /root/reference):   python tests/golden/extract_strkey_goldens.py

Source: pkg/common/hashmap/strhashmap_test.go TestIterator: three maps over Rows rows of six columns (int8, int16, int32, int64, decimal64,
char), row i holding i in every fixed-width column and strconv.Itoa(i) in the char column (newVectors); the third sets every even row NULL
in all six columns (newVectorsWithNull).  The ids Insert and then Find return are transcribed with the hasNull flag of each map.
"""
import json
import os
import re

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
SRC = "pkg/common/hashmap/strhashmap_test.go"


def strhashmap_kats():
    text = open(os.path.join(REF, SRC)).read()
    rows = int(re.search(r"\bRows\s*=\s*(\d+)", text).group(1))
    body = text[text.index("func TestIterator("):]
    body = body[:body.index("\nfunc ", 1)]
    assert "if j%2 == 0 {" in text[text.index("func newVectorsWithNull("):]        # the NULL pattern of newVectorsWithNull
    assert "strconv.Itoa(v)" in text[text.index("func newStringVector("):]         # the char column's values
    cases = []
    for block in body.split("m := mpool.MustNewZero()")[1:]:
        has_null = re.search(r"NewStrHashMap\((true|false)", block).group(1) == "true"
        types = re.findall(r"types\.New\(types\.T_(\w+), 0, 0\)", block)
        with_null = "newVectorsWithNull(" in block
        ids = [[int(x) for x in m.split(",")] for m in re.findall(r"require\.Equal\(t, \[\]uint64\{([\d, ]+)\}, vs\[:Rows\]\)", block)]
        assert len(ids) == 2, "Insert then Find"
        cases.append({"has_null": has_null, "types": types, "even_rows_null": with_null, "insert_ids": ids[0], "find_ids": ids[1]})
    return {"_source": SRC + " TestIterator: row i = i in every fixed-width column, strconv.Itoa(i) in the char column", "rows": rows, "cases": cases}


def main():
    data = strhashmap_kats()
    with open(os.path.join(OUT, "strhashmap_kat.json"), "w") as f:
        json.dump(data, f, indent=1)
    print("strhashmap_kat", len(data["cases"]), "cases of", data["rows"], "rows")


if __name__ == "__main__":
    main()
