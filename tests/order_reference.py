"""Host restatements of ORDER BY / Top for the tests of MO_XCALL_ORDER_SELS.

  compare_rows       compare.New(type, desc, nullsLast) per key, left to right (pkg/compare/compare.go:24-115,231-239, nullsCompare in
                     compare/types.go:57-80, GenericAscCompare / GenericDescCompare in container/types/compare.go:52-105)
  order_reference    sorted() with that comparator plus the row-id tie-break: the one total order the device computes
  order_lexsort      the same order through np.lexsort on the decoded values (large sizes)
  top_reference      the reference Top operator itself: processBatch (top.go:274-322) over 8192-row batches with Go's container/heap,
                     evalInMemory (top.go:434-452) popping into reversed order.  Its ties fall where the heap leaves them, so only its
                     output key sequence is comparable.
"""
import functools

import numpy as np

DESC, NULLS_FIRST, NULLS_LAST = 2, 4, 8


def nulls_last_of(flag):
    """order.go:143-150: neither NULLS flag -> nullsLast = desc"""
    if flag & NULLS_FIRST:
        return False
    if flag & NULLS_LAST:
        return True
    return bool(flag & DESC)


def _generic(x, y):
    if x == y:
        return 0
    if x < y:
        return -1
    return 1


def compare_rows(a, b, flags):
    """a, b: tuples of (is_null, value) per key.  Returns <0, 0, >0 as the reference's ctr.compare."""
    for (n0, x), (n1, y), f in zip(a, b, flags):
        nl = nulls_last_of(f)
        if n0 and n1:
            continue
        if n0 or n1:
            if n0:
                return 1 if nl else -1
            return -1 if nl else 1
        c = _generic(x, y)
        if f & DESC:
            c = -c
        if c:
            return c
    return 0


def key_tuples(cols, nulls, n):
    """cols: list of sequences (a 1-element sequence = const key); nulls: list of bool masks or None.  Python values: DECIMAL128 columns
    (uint64[n, 2]) become ints, floats lose the sign of zero (Go's == does not see it)."""
    out = []
    for i in range(n):
        row = []
        for c, m in zip(cols, nulls):
            r = 0 if len(c) == 1 else i
            isnull = bool(m[r]) if m is not None else False
            v = c[r]
            if isinstance(v, np.ndarray):
                v = int(np.int64(v[1])) * (1 << 64) + int(v[0])
            elif isinstance(v, (np.floating, float)):
                v = float(v) + 0.0
            else:
                v = int(v)
            row.append((isnull, None if isnull else v))
        out.append(tuple(row))
    return out


def order_reference(cols, nulls, flags, n, row_ids=None, limit=None):
    keys = key_tuples(cols, nulls, n)
    rid = list(range(n)) if row_ids is None else [int(x) for x in row_ids]

    def cmp(i, j):
        c = compare_rows(keys[i], keys[j], flags)
        if c:
            return c
        return _generic(rid[i], rid[j]) or _generic(i, j)

    order = sorted(range(n), key=functools.cmp_to_key(cmp))
    if limit is not None and 0 <= limit < n:
        order = order[:limit]
    return np.asarray(order, dtype=np.int64)


def _flip_desc(v, desc):
    return ~v if desc else v


def order_lexsort(cols, nulls, flags, n, row_ids=None):
    """np.lexsort over (per key: null rank, NaN flag, value image), then the row ids; lexsort is stable, so the row index breaks the rest"""
    planes = []
    for c, m, f in zip(cols, nulls, flags):
        c = np.asarray(c)
        if len(c) == 1 and n != 1:
            c = np.repeat(c, n, axis=0)
        desc, nl = bool(f & DESC), nulls_last_of(f)
        isnull = np.zeros(n, bool) if m is None else (np.repeat(m, n) if len(m) == 1 and n != 1 else np.asarray(m, bool))
        rank = np.where(isnull, 1 if nl else 0, 0 if nl else 1).astype(np.uint8)
        sign = np.uint64(1 << 63)
        if c.ndim == 2:
            hi = _flip_desc(c[:, 1].astype(np.uint64) ^ sign, desc)
            lo = _flip_desc(c[:, 0].astype(np.uint64), desc)
            vals = [np.where(isnull, 0, hi), np.where(isnull, 0, lo)]
        elif c.dtype.kind == "f":
            x = c.astype(np.float64)
            nan = np.isnan(x)
            x = np.where(nan | isnull, 0.0, x) + 0.0
            vals = [np.where(isnull, False, nan ^ desc), np.where(isnull, 0.0, -x if desc else x)]   # NaN above every number
        elif c.dtype.kind == "i":
            v = c.astype(np.int64).view(np.uint64) ^ sign
            vals = [np.where(isnull, np.uint64(0), _flip_desc(v, desc))]
        else:
            v = c.astype(np.uint64)
            vals = [np.where(isnull, np.uint64(0), _flip_desc(v, desc))]
        planes.append([rank] + vals)
    seq = [p for key in planes for p in key]          # most significant first
    if row_ids is not None:
        seq.append(np.asarray(row_ids, np.int64))
    return np.lexsort(tuple(reversed(seq))).astype(np.int64) if seq else np.arange(n, dtype=np.int64)


# ---- the reference Top operator, restated ---------------------------------------------------------------------------------------------------
class _TopHeap:
    """ctr of top.go: data slots (the batch ctr.bat holds) and ctr.sels, a heap whose Less is compare(...) > 0 (types.go:227-246)"""

    def __init__(self, flags):
        self.flags, self.data, self.sels = flags, [], []

    def less(self, i, j):
        return compare_rows(self.data[self.sels[i]][0], self.data[self.sels[j]][0], self.flags) > 0

    def swap(self, i, j):
        self.sels[i], self.sels[j] = self.sels[j], self.sels[i]

    # Go's container/heap (heap.go): up, down, Init, Fix, Pop
    def up(self, j):
        while True:
            i = int((j - 1) / 2)          # Go's integer division truncates toward zero: the parent of 0 is 0
            if i == j or not self.less(j, i):
                break
            self.swap(i, j)
            j = i

    def down(self, i0, n):
        i = i0
        while True:
            j1 = 2 * i + 1
            if j1 >= n or j1 < 0:
                break
            j = j1
            j2 = j1 + 1
            if j2 < n and self.less(j2, j1):
                j = j2
            if not self.less(j, i):
                break
            self.swap(i, j)
            i = j
        return i > i0

    def init(self):
        n = len(self.sels)
        for i in range(n // 2 - 1, -1, -1):
            self.down(i, n)

    def fix(self, i):
        if not self.down(i, len(self.sels)):
            self.up(i)

    def pop(self):
        n = len(self.sels) - 1
        self.swap(0, n)
        self.down(0, n)
        return self.sels.pop()


def top_reference(keys, payload, flags, limit, batch=8192):
    """keys: list of key tuples (key_tuples), payload: per row value carried along (cmp.Copy copies every column).  Rows arrive in
    `batch`-row batches.  Returns [(key tuple, payload)] in output order."""
    if limit == 0:
        return []
    h = _TopHeap(flags)
    for b0 in range(0, len(keys), batch):
        rows = list(range(b0, min(b0 + batch, len(keys))))
        fill = min(limit - len(h.sels), len(rows))                       # processBatch: fill the first `limit` rows
        for r in rows[:max(fill, 0)]:
            h.sels.append(len(h.data))
            h.data.append((keys[r], payload[r]))
            if len(h.sels) == limit:
                h.init()
        for r in rows[max(fill, 0):]:                                    # then replace the root on a strictly smaller row
            if compare_rows(keys[r], h.data[h.sels[0]][0], flags) < 0:
                h.data[h.sels[0]] = (keys[r], payload[r])
                h.fix(0)
    if len(h.sels) < limit:                                              # evalInMemory
        h.init()
    out = [None] * len(h.sels)
    for i in range(len(h.sels)):
        out[len(out) - 1 - i] = h.pop()
    return [h.data[s] for s in out]
