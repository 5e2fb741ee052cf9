"""Host restatement of the hash join's right-flavoured and single joins (test infrastructure): container.probe with the matched-row bitmap
(pkg/sql/colexec/hashjoin/join.go:383-628, NonEqCond == nil), syncBitmap (join.go:650-689) and finalize (join.go:691-727), over the ids of a
build-side JoinMap.  Join flavours are JoinType + IsRightJoin (types.go:317-381).

probe() is the reference's row loop; probe_fast() is the same result in numpy for the sizes the GPU tests use, and the CPU tests hold the two
equal.  Pairs are (probe row, build row | -1) in the reference's order: probe rows ascending, per probe row its sels ascending.  A SEMI probe row
is emitted as (row, -1) on both map paths: the result of a semi join has probe columns only."""
import numpy as np

from matrixone_b200 import capi

# (plan.Node_JoinType, IsRightJoin) of every MO_JOIN_* type; FULL OUTER always runs right-flavoured (compile.go sets IsRightJoin for Node_OUTER)
FLAVOUR = {
    capi.JOIN_INNER: ("INNER", False), capi.JOIN_LEFT: ("LEFT", False), capi.JOIN_SEMI: ("SEMI", False), capi.JOIN_ANTI: ("ANTI", False),
    capi.JOIN_SINGLE: ("SINGLE", False), capi.JOIN_RIGHT: ("RIGHT", True), capi.JOIN_FULL: ("OUTER", True),
    capi.JOIN_RIGHT_SEMI: ("SEMI", True), capi.JOIN_RIGHT_ANTI: ("ANTI", True), capi.JOIN_RIGHT_SINGLE: ("SINGLE", True),
}
RIGHT_TYPES = (capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_RIGHT_SEMI, capi.JOIN_RIGHT_ANTI, capi.JOIN_RIGHT_SINGLE)
NEW_TYPES = (capi.JOIN_SINGLE,) + RIGHT_TYPES
SCALAR_SUBQUERY = "scalar subquery returns more than 1 row"


class Checkers:
    """the HashJoin type checkers of types.go:317-382"""

    def __init__(self, join_type, is_right_join):
        self.t, self.right = join_type, is_right_join

    def IsInner(self): return self.t == "INNER"
    def IsLeftOuter(self): return self.t == "LEFT"
    def IsRightOuter(self): return self.t == "RIGHT"
    def IsFullOuter(self): return self.t == "OUTER"
    def IsSemi(self): return self.t == "SEMI"
    def IsLeftSemi(self): return not self.right and self.t == "SEMI"
    def IsRightSemi(self): return self.right and self.t == "SEMI"
    def IsAnti(self): return self.t == "ANTI"
    def IsLeftAnti(self): return not self.right and self.t == "ANTI"
    def IsRightAnti(self): return self.right and self.t == "ANTI"
    def IsSingle(self): return self.t == "SINGLE"
    def IsLeftSingle(self): return not self.right and self.t == "SINGLE"
    def IsRightSingle(self): return self.right and self.t == "SINGLE"
    def EmitUnmatchedProbe(self): return self.IsLeftOuter() or self.IsLeftSingle() or self.IsLeftAnti() or self.IsFullOuter()
    def EmitUnmatchedBuild(self): return self.right or self.IsFullOuter()


def checkers(join_type):
    return Checkers(*FLAVOUR[join_type])


class SingleError(Exception):
    """moerr internal error "scalar subquery returns more than 1 row"; probe_row / build_row = the row the device names"""

    def __init__(self, probe_row=None, build_row=None):
        super().__init__(SCALAR_SUBQUERY)
        self.probe_row, self.build_row = probe_row, build_row


# ---------------------------------------------------------------------------------------------- the build side's JoinMap
def build_map(keys, nulls=None):
    """IntHashMap insert + GroupSels (first-seen 1-based ids; a NULL key gets no group) -> (groups per row, table_keys, offsets, sels); offsets /
    sels None when the map keeps no sels (every row its own group, or no group at all: HashOnUnique)"""
    keys = np.asarray(keys, dtype=np.uint64)
    n = len(keys)
    live = np.ones(n, bool) if nulls is None else ~np.asarray(nulls, bool)
    rows = np.flatnonzero(live)
    uk, first, inv = np.unique(keys[rows], return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")             # ids in first-seen order
    rank = np.empty(len(uk), np.int64)
    rank[order] = np.arange(len(uk))
    groups = np.zeros(n, np.uint64)
    groups[rows] = rank[inv] + 1
    table_keys = uk[order]
    ngroups = len(uk)
    if ngroups == n or ngroups == 0:
        return groups, table_keys, None, None
    g = groups[rows].astype(np.int64) - 1
    sels = rows[np.argsort(g, kind="stable")].astype(np.int32)
    offsets = np.zeros(ngroups + 2, np.int32)
    offsets[1:ngroups + 1] = np.cumsum(np.bincount(g, minlength=ngroups))
    offsets[ngroups + 1] = offsets[ngroups]
    return groups, table_keys, offsets, sels


def find(table_keys, keys, nulls=None):
    """intHashMapIterator.Find: the 1-based group id of every probe key, 0 = absent or NULL"""
    keys = np.asarray(keys, dtype=np.uint64)
    vals = np.zeros(len(keys), np.uint64)
    if len(table_keys):
        order = np.argsort(table_keys)
        sk = table_keys[order]
        pos = np.minimum(np.searchsorted(sk, keys), len(sk) - 1)
        hit = sk[pos] == keys
        vals[hit] = order[pos[hit]] + 1
    if nulls is not None:
        vals[np.asarray(nulls, bool)] = 0
    return vals


# ---------------------------------------------------------------------------------------------- container.probe, syncBitmap, finalize
def probe(vals, offsets, sels, join_type, matched=None):
    """container.probe over Find's ids (join.go:416-560) for one probe batch; `matched` (numpy bool[nbuild], rightRowsMatched) is marked in
    place for the right-flavoured types.  The reference fails at the first offending row in row order; the error carries the row the device
    names: the lowest offending probe row (LEFT SINGLE), or the lowest build row this batch matches a second time (RIGHT SINGLE)."""
    h = checkers(join_type)
    out_p, out_b = [], []
    twice = []                                            # RIGHT SINGLE: build rows found marked already (join.go:462,541)
    unique = offsets is None                              # HashOnUnique (join.go:450-498)

    def mark(r):
        if h.IsSingle() and matched[r]:
            twice.append(r)
        matched[r] = True

    for row in range(len(vals)):
        v = int(vals[row])
        nm = 0 if v == 0 else (1 if unique else int(offsets[v] - offsets[v - 1]))
        if nm == 0:                                       # z == 0 || v == 0 (join.go:433-449)
            if h.EmitUnmatchedProbe():
                out_p.append(row); out_b.append(-1)       # appendOneNotMatch
            continue
        idx = v - 1
        if unique:
            if not h.IsRightSemi() and not h.IsAnti():   # appendOneMatch (join.go:452-458)
                out_p.append(row); out_b.append(-1 if h.IsLeftSemi() else idx)
            if h.right:                                   # join.go:461-467
                mark(idx)
            continue
        rsels = [int(x) for x in sels[offsets[idx]:offsets[idx + 1]]]   # GetSels (join.go:500-516)
        if h.IsLeftSingle():
            if len(rsels) > 1:
                raise SingleError(probe_row=row)
        elif h.IsLeftSemi():
            out_p.append(row); out_b.append(-1)
            continue
        elif h.IsLeftAnti():
            continue
        if h.right:                                       # psSelsForOneRow (join.go:539-547)
            for s in rsels:
                mark(s)
        if not h.IsRightSemi() and not h.IsAnti():       # join.go:549-566
            for s in rsels:
                out_p.append(row); out_b.append(s)
    if twice:
        raise SingleError(build_row=min(twice))
    return np.array(out_p, np.int64), np.array(out_b, np.int64)


def sync_bitmap(bitmaps, join_type):
    """syncBitmap (join.go:650-676) over the workers' bitmaps: their OR; RIGHT SINGLE fails when the summed counts exceed the OR's count, i.e.
    when a row is set in two of them (the error names the lowest such row).  Returns the OR, not yet negated."""
    acc = np.zeros_like(bitmaps[0], dtype=bool)
    cnt = 0
    twice = np.zeros_like(acc)
    for b in bitmaps:
        b = np.asarray(b, bool)
        cnt += int(b.sum())
        twice |= acc & b
        acc |= b
    if checkers(join_type).IsSingle() and cnt > int(acc.sum()):
        raise SingleError(build_row=int(np.flatnonzero(twice)[0]))
    return acc


def finalize(matched, join_type):
    """syncBitmap's Negate unless the join is a semi join (join.go:682-684), then finalize's iterator (join.go:686, 691-727): the build rows emitted
    with NULL probe-side columns, ascending"""
    m = np.asarray(matched, bool)
    return np.flatnonzero(m if checkers(join_type).IsSemi() else ~m).astype(np.int64)


def probe_fast(vals, offsets, sels, join_type, matched=None):
    """probe() in numpy: the same pairs, marks and errors"""
    h = checkers(join_type)
    vals = np.asarray(vals, np.int64)
    n = len(vals)
    if offsets is None:
        m = (vals > 0).astype(np.int64)
        start = np.maximum(vals - 1, 0)
    else:
        off = np.asarray(offsets, np.int64)
        m = np.where(vals > 0, off[vals] - off[np.maximum(vals - 1, 0)], 0)
        start = np.where(vals > 0, off[np.maximum(vals - 1, 0)], 0)
    if h.IsLeftSingle() and (m > 1).any():
        raise SingleError(probe_row=int(np.flatnonzero(m > 1)[0]))
    rows = np.repeat(np.arange(n, dtype=np.int64), m)
    k = np.arange(len(rows), dtype=np.int64) - np.repeat(np.cumsum(m) - m, m)
    pos = np.repeat(start, m) + k
    build = pos if offsets is None else np.asarray(sels, np.int64)[pos]
    if h.right:
        if h.IsSingle():
            hits = np.bincount(build, minlength=len(matched)) + matched.astype(np.int64) if len(build) else matched.astype(np.int64)
            bad = np.flatnonzero(hits > 1)
            matched[build] = True
            if len(bad):
                raise SingleError(build_row=int(bad[0]))
        matched[build] = True
    if h.IsRightSemi() or h.IsAnti():
        if h.IsLeftAnti():
            r = np.flatnonzero(m == 0)
            return r.astype(np.int64), np.full(len(r), -1, np.int64)
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    if h.IsLeftSemi():
        r = np.flatnonzero(m > 0)
        return r.astype(np.int64), np.full(len(r), -1, np.int64)
    if not h.EmitUnmatchedProbe():
        return rows, build
    # interleave the unmatched probe rows (row, -1) into row order
    c = np.maximum(m, 1)
    out_p = np.repeat(np.arange(n, dtype=np.int64), c)
    out_b = np.full(len(out_p), -1, np.int64)
    matched_slots = np.repeat(m > 0, c)
    out_b[matched_slots] = build
    return out_p, out_b
