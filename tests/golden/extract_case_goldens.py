"""Record the reference's own CASE and COALESCE tables into case_kat.json (run once; the JSON is committed).

  TestCoalesce (pkg/sql/plan/function/func_binary_test.go:338, cases from initCoalesceTestCase :273-336): the int64 and varchar cases; the
      vector-type cases are out of scope.
  Test_CaseWhen_WithNullAndStringComparison (pkg/sql/plan/function/operatorSet_test.go:435): strCaseFn over one WHEN and an ELSE.

Each case is written as its inputs (values + null flags, strings as hex) and its expected result; the Go source lines are checked to hold
exactly these literals, so a change in the reference's tables fails the extraction instead of drifting silently."""
import json
import os

REF = "/root/reference/pkg/sql/plan/function"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "case_kat.json")


def col(values, nulls):
    return {"values": [v.encode().hex() if isinstance(v, str) else v for v in values], "nulls": nulls}


CASES = [
    {"name": "TestCoalesce: test Coalesce int64", "fn": "coalesce", "type": "int64",
     "source": ("func_binary_test.go", ["[]int64{1, 4, 8, 16, 32, 0},", "[]bool{true, true, true, true, true, true}),"]),
     "inputs": [col([1, 4, 8, 16, 32, 0], [True] * 6), col([1, 4, 8, 16, 32, 0], [False] * 6)],
     "expect": col([1, 4, 8, 16, 32, 0], [False] * 6)},
    {"name": "TestCoalesce: test Coalesce varchar", "fn": "coalesce", "type": "varchar",
     "source": ("func_binary_test.go", ['[]string{"hello", "", "world"},', '[]bool{false, true, false}),', '[]string{"hello", "-", "world"},',
                                        '[]bool{true, false, true}),']),
     "inputs": [col(["hello", "", "world"], [False, True, False]), col(["hello", "-", "world"], [True, False, True])],
     "expect": col(["hello", "-", "world"], [False, False, False])},
    {"name": "Test_CaseWhen_WithNullAndStringComparison", "fn": "case", "type": "varchar",
     "source": ("operatorSet_test.go", ['[]bool{false}, []bool{false}),', '[]string{"true"}, []bool{false}),', '[]string{"false"}, []bool{false}),']),
     "inputs": [col([False], [False]), col(["true"], [False]), col(["false"], [False])],
     "expect": col(["false"], [False])},
]


def main():
    for c in CASES:
        f, lines = c.pop("source")
        text = open(os.path.join(REF, f)).read()
        for ln in lines:
            assert ln in text, (c["name"], ln)
    with open(OUT, "w") as fh:
        json.dump(CASES, fh, indent=1)
        fh.write("\n")


if __name__ == "__main__":
    main()
