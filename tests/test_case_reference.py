"""case_reference.py pinned to the reference's own tables (golden/case_kat.json: TestCoalesce's int64 and varchar cases and
Test_CaseWhen_WithNullAndStringComparison), IF == CASE with one WHEN and an ELSE over random inputs, EvalCase's select lists, and the
string layout against vector.varlena_bytes_column.  No GPU."""
import json
import os

import numpy as np
import pytest

import case_reference as R
from matrixone_b200.vector import varlena_bytes_column

KAT = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "case_kat.json")))


def rows(c, typ):
    vals = [bytes.fromhex(v) if typ == "varchar" and isinstance(v, str) else v for v in c["values"]]
    return [None if nl else v for v, nl in zip(vals, c["nulls"])]


@pytest.mark.parametrize("case", KAT, ids=[c["name"] for c in KAT])
def test_reference_tables(case):
    ins = [rows(c, case["type"]) for c in case["inputs"]]
    n = max(len(c) for c in ins)
    if case["fn"] == "coalesce":
        got = R.coalesce(ins, n)
    else:
        got = R.case_fn(ins[0:-1:2], ins[1:-1:2], ins[-1] if len(ins) % 2 else None, n)
    assert got == rows(case["expect"], case["type"])


def rand_col(rng, n, const=False):
    k = 1 if const else n
    return [None if rng.random() < 0.2 else int(rng.integers(0, 5)) for _ in range(k)]


def rand_cond(rng, n, const=False):
    k = 1 if const else n
    return [None if rng.random() < 0.2 else bool(rng.integers(0, 2)) for _ in range(k)]


@pytest.mark.parametrize("seed", range(20))
def test_iff_is_case_with_one_when_and_an_else(seed):
    rng = np.random.default_rng(seed)
    n = 50
    c, a, b = rand_cond(rng, n, seed % 3 == 0), rand_col(rng, n, seed % 4 == 0), rand_col(rng, n, seed % 5 == 0)
    skip = list(rng.random(n) < 0.1)
    assert R.iff_fn(c, a, b, n, skip) == R.case_fn([c], [a], b, n, skip)


@pytest.mark.parametrize("seed", range(10))
def test_case_over_its_select_lists(seed):
    """evaluating each branch only over its select list and then CASE over the results gives CASE over fully evaluated branches"""
    rng = np.random.default_rng(seed)
    n, m = 64, 4
    select = list(rng.random(n) < 0.8)
    conds = [rand_cond(rng, n) for _ in range(m)]
    vals = [rand_col(rng, n) for _ in range(m)]
    z = rand_col(rng, n)
    when_lists, then_lists, else_list = R.case_select_lists(select, conds)
    # a branch evaluated under its list: rows outside it are garbage (here 99) the CASE must never read
    masked_c = [[c[i] if wl[i] else True for i in range(n)] for c, wl in zip(conds, when_lists)]
    masked_v = [[v[i] if tl[i] else 99 for i in range(n)] for v, tl in zip(vals, then_lists)]
    masked_z = [z[i] if else_list[i] else 99 for i in range(n)]
    skip = [not s for s in select]
    want = R.case_fn(conds, vals, z, n, skip)
    # the device walks WHENs in order and stops at the first match, so an unselected row of WHEN j is never read: restate that walk
    got = []
    for i in range(n):
        if skip[i]:
            got.append(R.SKIP)
            continue
        for j in range(m):
            if masked_c[j][i] is not None and masked_c[j][i]:
                got.append(masked_v[j][i])
                break
        else:
            got.append(masked_z[i])
    assert got == want
    for j in range(m):
        took = then_lists[j]
        assert all(when_lists[j][i] for i in range(n) if took[i])
        assert not any(took[i] and then_lists[k][i] for k in range(j) for i in range(n))


def test_string_layout_is_varlena_bytes_column():
    vals = [b"", b"a" * 23, b"b" * 24, b"c\x00d", b"e" * 100]
    cells, area = R.str_bytes(vals, b"")
    c2, a2 = varlena_bytes_column(vals)
    assert cells == c2.tobytes() and area == a2.tobytes()
    cells, area = R.str_bytes([None, R.SKIP, b"x" * 30], bytes(24) + b"\x07" * 24 + bytes(24))
    assert cells[:24] == bytes(24) and cells[24:48] == b"\x07" * 24 and area == b"x" * 30
