"""Restatement of the reference's StrHashMap (pkg/common/hashmap/strhashmap.go:92-385, iterator.go:62-108,
pkg/container/hashtable/string_hash_map.go:97-158) in plain Python: encodeHashKeys as bytes per row, and first-seen insert / find as a dict
over those bytes.  The reference keys its table by a 192-bit hash of the bytes; equal bytes are the same group here, which is its result
except on a hash collision.  Its zero padding of keys shorter than 16 bytes is left out: the column codes are self-delimiting."""
import struct

import numpy as np

from matrixone_b200 import capi


def encode_keys(cols, types, nulls=None, has_null=True, n=None):
    """cols: per column a numpy array (fixed width; DECIMAL128 / UUID as uint64[n, 2]) or, for a varlena type, a list of bytes; a column of one
    element is const.  nulls: per column a bool sequence (one element for a const column) or None.  Returns per row its key bytes, or None for
    a row that joins no group (a NULL without has_null)."""
    n = n if n is not None else max(len(c) for c in cols)
    nulls = nulls if nulls is not None else [None] * len(cols)
    out = []
    for i in range(n):
        key = bytearray()
        skip = False
        for c, T, nl in zip(cols, types, nulls):
            r = 0 if len(c) == 1 and n != 1 else i
            isnull = nl is not None and bool(nl[r])
            if has_null:
                key.append(1 if isnull else 0)
                if isnull:
                    continue
            elif isnull:
                skip = True
                break
            if T in capi.T_VARLENA:
                v = bytes(c[r])
                key += struct.pack("<H", len(v)) + v
            else:
                key += np.ascontiguousarray(c[r:r + 1]).tobytes()
        out.append(None if skip else bytes(key))
    return out


def insert(table, keys):
    """StrHashMap insert: 1-based ids in first-seen order, persisting in `table` (dict bytes -> id); 0 for a skipped row"""
    ids = np.zeros(len(keys), np.uint64)
    for i, k in enumerate(keys):
        if k is not None:
            ids[i] = table.setdefault(k, len(table) + 1)
    return ids


def find(table, keys):
    """strHashmapIterator.Find: the id, or 0 when the key is absent or the row is skipped"""
    return np.array([0 if k is None else table.get(k, 0) for k in keys], np.uint64)


def table_bytes(table):
    """the group table as STR_GROUP_IDS lays it out: (bytes, offsets uint64[ngroups + 1]) in id order"""
    keys = sorted(table, key=table.get)
    off = np.zeros(len(keys) + 1, np.uint64)
    off[1:] = np.cumsum([len(k) for k in keys]) if keys else []
    return np.frombuffer(b"".join(keys), np.uint8), off


def flat(keys):
    """rows' keys as PACK_STR_KEYS returns them: (bytes, offsets uint64[n + 1]); a skipped row has an empty key"""
    ks = [k or b"" for k in keys]
    off = np.zeros(len(ks) + 1, np.uint64)
    off[1:] = np.cumsum([len(k) for k in ks]) if ks else []
    return np.frombuffer(b"".join(ks), np.uint8), off
