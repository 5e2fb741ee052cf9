"""Host restatement of ORDER BY over string keys, for the tests of MO_XCALL_ORDER_SELS with CHAR / VARCHAR / TEXT / BLOB ... keys.

A string key column is a list of bytes.  Go orders such values with bytes.Compare (sort.go varlenaLess / varlenaGreater,
compare/strcompare.go), which is Python's bytes <.  Every bytes column is replaced by its ranks in sorted(set(values)) -- equal values get
equal ranks and the ranks order as the values do -- and the fixed-width restatements of order_reference then apply unchanged:

  key_tuples, order_reference, order_lexsort   as in order_reference, with bytes columns ranked first
  golden_order_query                           the ORDER BY goldens of the reference's TPC-H queries (tests/golden/order_kat.json)
"""
import json
import os

import numpy as np

import order_reference as R

DESC, NULLS_FIRST, NULLS_LAST = R.DESC, R.NULLS_FIRST, R.NULLS_LAST


def bytes_ranks(values):
    """a string column (list of bytes) as int64 ranks in Python's bytes order, which is Go's bytes.Compare"""
    rank_of = {v: i for i, v in enumerate(sorted(set(values)))}
    return np.fromiter((rank_of[v] for v in values), dtype=np.int64, count=len(values))


def ranked(cols):
    return [bytes_ranks(c) if isinstance(c, list) else c for c in cols]


def key_tuples(cols, nulls, n):
    return R.key_tuples(ranked(cols), nulls, n)


def order_reference(cols, nulls, flags, n, row_ids=None, limit=None):
    return R.order_reference(ranked(cols), nulls, flags, n, row_ids=row_ids, limit=limit)


def order_lexsort(cols, nulls, flags, n, row_ids=None):
    return R.order_lexsort(ranked(cols), nulls, flags, n, row_ids=row_ids)


def golden_order_query(q):
    """(key columns, flags, type names, limit, result rows) of query q: CHAR / VARCHAR keys as lists of bytes, DECIMAL(15,2) as int64 cents,
    INTEGER as int32, BIGINT as int64 -- the key columns in ORDER BY order, rows as the reference printed them"""
    d = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "order_kat.json")))[q]
    rows, cols, keys, flags, types = d["rows"], d["columns"], [], [], []
    for name, direction in d["order_by"]:
        j, T = cols.index(name), d["types"][name]
        vals = [r[j] for r in rows]
        if T.startswith(("CHAR", "VARCHAR")):
            keys.append([v.encode() for v in vals])
        elif T.startswith("DECIMAL"):
            keys.append(np.asarray([round(float(v) * 100) for v in vals], dtype=np.int64))
        else:
            keys.append(np.asarray([int(v) for v in vals], dtype=np.int32 if T == "INTEGER" else np.int64))
        flags.append(DESC if direction == "desc" else 0)
        types.append(T)
    return keys, flags, types, d["limit"], rows
