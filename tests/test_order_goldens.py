"""The host restatement of ORDER BY over string keys (order_varlena_reference) against the reference's own output: the rows of
the TPC-H queries whose last stage orders by string keys (q16, q2, q20, q21, and q1's group order), shuffled, must come back in the order of
their .result files."""
import numpy as np
import pytest

import order_varlena_reference as R

QUERIES = ["q16", "q2", "q20", "q21", "q1"]


def _take(keys, perm):
    return [[k[i] for i in perm] if isinstance(k, list) else k[perm] for k in keys]


@pytest.mark.parametrize("q", QUERIES)
@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_restatement_reproduces_result_order(q, seed):
    keys, flags, _, limit, rows = R.golden_order_query(q)
    n = len(rows)
    perm = np.random.default_rng(seed).permutation(n)
    shuffled = _take(keys, perm)
    order = R.order_reference(shuffled, [None] * len(keys), flags, n, limit=limit)
    want = R.key_tuples(keys, [None] * len(keys), n)
    got = R.key_tuples(shuffled, [None] * len(keys), n)
    assert [got[i] for i in order] == want[:len(order)]
    if len(set(want)) == n:                       # distinct key tuples: the whole rows come back in the printed order
        assert [rows[perm[i]] for i in order] == rows[:len(order)]
    lex = R.order_lexsort(shuffled, [None] * len(keys), flags, n)
    assert (lex[:len(order)] == order).all()


def test_fixtures_hold_rows():
    """q16 and q1 carry the ordering evidence (q2 prints one row; q20 and q21 print none on the tiny dataset)"""
    assert len(R.golden_order_query("q16")[4]) == 41 and len(R.golden_order_query("q1")[4]) == 4
