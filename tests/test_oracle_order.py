"""The restated reference Top operator (container/heap over 8192-row batches) against an independent sorted() with the compare.New
comparator: on NaN-free inputs their output key sequences are equal (ties may carry different rows)."""
import numpy as np
import pytest

import order_reference as R

FLAGS = [0, R.DESC, R.NULLS_FIRST, R.NULLS_LAST, R.DESC | R.NULLS_FIRST, R.DESC | R.NULLS_LAST]


def _data(rng, n, nkeys, small):
    cols, nulls = [], []
    for k in range(nkeys):
        if k % 3 == 0:
            c = rng.integers(-5 if small else -10**12, 5 if small else 10**12, n).astype(np.int64)
        elif k % 3 == 1:
            c = rng.integers(0, 3, n).astype(np.float64) * 0.5 - 0.5
        else:
            c = rng.integers(0, 4 if small else 60000, n).astype(np.uint16)
        cols.append(c)
        nulls.append(rng.random(n) < 0.2 if k % 2 == 0 else None)
    return cols, nulls


@pytest.mark.parametrize("flag", FLAGS)
@pytest.mark.parametrize("limit", [0, 1, 37, 1000, 1001, 5000])
def test_top_matches_sorted_one_key(flag, limit):
    rng = np.random.default_rng(limit * 31 + flag)
    n = 1000
    cols, nulls = _data(rng, n, 1, small=limit % 2 == 1)
    keys = R.key_tuples(cols, nulls, n)
    got = R.top_reference(keys, list(range(n)), [flag], limit)
    want = R.order_reference(cols, nulls, [flag], n, limit=limit)
    assert len(got) == min(limit, n)
    assert [k for k, _ in got] == [keys[i] for i in want]


@pytest.mark.parametrize("nkeys", [2, 3, 5])
@pytest.mark.parametrize("limit", [1, 100, 20000, 25000])
def test_top_matches_sorted_multi_key_batches(nkeys, limit):
    """20000 rows arrive as three 8192-row batches"""
    rng = np.random.default_rng(nkeys * 7 + limit)
    n = 20000
    cols, nulls = _data(rng, n, nkeys, small=True)
    flags = [FLAGS[(i + nkeys) % len(FLAGS)] for i in range(nkeys)]
    keys = R.key_tuples(cols, nulls, n)
    got = R.top_reference(keys, list(range(n)), flags, limit)
    want = R.order_reference(cols, nulls, flags, n, limit=limit)
    assert [k for k, _ in got] == [keys[i] for i in want]


@pytest.mark.parametrize("flag", FLAGS)
def test_lexsort_matches_sorted(flag):
    """the large-size reference of the GPU tests is the same order as the comparator restatement"""
    rng = np.random.default_rng(flag)
    n = 3000
    cols, nulls = _data(rng, n, 3, small=True)
    cols.append(np.stack([rng.integers(0, 3, n).astype(np.uint64) << np.uint64(62), rng.integers(-1, 2, n).astype(np.int64).view(np.uint64)], axis=1))
    nulls.append(None)
    flags = [flag, FLAGS[(flag + 1) % 6], flag ^ R.DESC, flag]
    rid = rng.permutation(n)
    assert (R.order_lexsort(cols, nulls, flags, n, row_ids=rid) == R.order_reference(cols, nulls, flags, n, row_ids=rid)).all()
    assert (R.order_lexsort(cols, nulls, flags, n) == R.order_reference(cols, nulls, flags, n)).all()
