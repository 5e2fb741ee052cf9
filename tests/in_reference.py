"""Host restatement of the reference's IN / NOT IN (pkg/sql/plan/function/operator_in.go), for the tests of MO_XCALL_GO_IN and
MO_XCALL_GO_NOT_IN.  Kept in step with:

  build_set(values, nulls)   op.init: Go's map[T]bool / map[string]bool of the tuple, its NULL elements skipped (a const NULL tuple: empty).
  member(s, v)               the map lookup: Go map equality -- the raw value for fixed-width types (+0.0 and -0.0 are one key, a NaN key is
                             never found; decimals and UUIDs are their bytes), the bytes for strings.
  evaluate(...)              operatorIn / operatorNotIn row by row: a NULL row is NULL, any other row `ok` (NOT IN: `!ok`) with a clear null
                             bit, so a NULL in the tuple never makes a row NULL.  Rows already NULL in the result on entry are skipped, the
                             project's GO convention for the selectList.
"""
import math

import numpy as np


def key(v):
    """the map key of one value (numpy scalar, Python number or bytes); None for a NaN, which a Go map never finds"""
    if isinstance(v, (bytes, bytearray)):
        return bytes(v)
    if isinstance(v, (float, np.floating)):
        if math.isnan(v):
            return None
        if v == 0:
            v = type(v)(0)
        return np.asarray(v).tobytes()
    if isinstance(v, np.ndarray):          # a 16-byte row (DECIMAL128, UUID)
        return v.tobytes()
    return np.asarray(v).tobytes()


def build_set(values, nulls=None):
    s = set()
    for i, v in enumerate(values):
        if nulls is not None and nulls[i]:
            continue
        k = key(v)
        if k is not None:
            s.add(k)
    return s


def member(s, v):
    k = key(v)
    return k is not None and k in s


def evaluate(col, col_nulls, values, values_nulls=None, negate=False, skip=None):
    """(result bool[n], nulls bool[n]) of col IN values (NOT IN: negate); col_nulls / skip: bool[n] or None.  Skipped rows stay NULL and
    their result is None (not written)."""
    s = build_set(values, values_nulls)
    n = len(col)
    out, nulls = [None] * n, [False] * n
    for i in range(n):
        if (skip is not None and skip[i]) or (col_nulls is not None and col_nulls[i]):
            nulls[i] = True
            continue
        out[i] = member(s, col[i]) != negate
    return out, nulls
