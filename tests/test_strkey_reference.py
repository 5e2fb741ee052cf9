"""The StrHashMap restatement (strkey_reference.py) against the reference's own iterator test (strhashmap_test.go TestIterator, transcribed
in tests/golden/strhashmap_kat.json), and the properties of its key format.  No GPU."""
import json
import os

import numpy as np

import strkey_reference as R
from matrixone_b200 import capi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "strhashmap_kat.json")
TYPES = {"int8": (capi.T_INT8, np.int8), "int16": (capi.T_INT16, np.int16), "int32": (capi.T_INT32, np.int32), "int64": (capi.T_INT64, np.int64),
         "decimal64": (capi.T_DECIMAL64, np.int64), "char": (capi.T_CHAR, None)}


def kat_columns(case, rows):
    """the test's vectors: row i = i (fixed width) or strconv.Itoa(i) (char); every even row NULL in every column when even_rows_null"""
    cols, types = [], []
    for name in case["types"]:
        T, dt = TYPES[name]
        cols.append([str(i).encode() for i in range(rows)] if dt is None else np.arange(rows, dtype=dt))
        types.append(T)
    nulls = [[i % 2 == 0 for i in range(rows)]] * len(cols) if case["even_rows_null"] else None
    return cols, types, nulls


def test_restatement_reproduces_the_reference_iterator_test():
    kat = json.load(open(GOLDEN))
    assert len(kat["cases"]) == 3
    for case in kat["cases"]:
        cols, types, nulls = kat_columns(case, kat["rows"])
        keys = R.encode_keys(cols, types, nulls, case["has_null"])
        table = {}
        assert R.insert(table, keys).tolist() == case["insert_ids"]
        assert R.find(table, keys).tolist() == case["find_ids"]


def test_key_format():
    # fixed width: marker + storage bytes; varlena: marker + uint16 LE length + bytes; NULL: 0x01 alone
    k = R.encode_keys([np.array([7], np.int16), [b"ab"]], [capi.T_INT16, capi.T_VARCHAR], [[False], [True]], True, n=1)
    assert k == [b"\x00\x07\x00\x01"]
    k = R.encode_keys([np.array([7], np.int16), [b"ab"]], [capi.T_INT16, capi.T_VARCHAR], None, False, n=1)
    assert k == [b"\x07\x00\x02\x00ab"]
    assert R.encode_keys([np.array([1, 2], np.int32)], [capi.T_INT32], [[False, True]], False) == [b"\x01\x00\x00\x00", None]


def test_distinct_rows_stay_distinct():
    # ("a", "bc") / ("ab", "c"), -0.0 / +0.0 and two NaN payloads are three pairs of different keys
    for has_null in (False, True):
        k = R.encode_keys([[b"a", b"ab"], [b"bc", b"c"]], [capi.T_VARCHAR, capi.T_VARCHAR], None, has_null)
        assert k[0] != k[1]
    f = np.array([-0.0, 0.0, np.nan, -np.nan], np.float64)
    f[3] = np.frombuffer(np.uint64(0x7ff8000000000001).tobytes(), np.float64)[0]
    k = R.encode_keys([f], [capi.T_FLOAT64], None, False)
    assert len(set(k)) == 4
    # a NULL key (has_null) is a group of its own; without has_null the row is skipped
    t = {}
    assert R.insert(t, R.encode_keys([np.array([5, 5, 6], np.int64)], [capi.T_INT64], [[True, False, True]], True)).tolist() == [1, 2, 1]
    t = {}
    assert R.insert(t, R.encode_keys([np.array([5, 5, 6], np.int64)], [capi.T_INT64], [[True, False, True]], False)).tolist() == [0, 1, 0]
