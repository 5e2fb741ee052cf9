"""An exact restatement of the fused plan operator (MO_XCALL_PLAN, include/mo_b200.h) in plain numpy / Python, no GPU.

run(plan, cols, nulls, n) evaluates a mo_plan_t (FusedPlan.P) row by row in meaning, vectorised in form, and returns the groups in the
reference's first-seen order, in the format of FusedPlan.parse plus what a tolerance needs.  Semantics, after the reference:
  columns     loaded by type: INT8/16/32 and DATE sign-extended, BOOL and the unsigned types zero-extended, FLOAT32 widened exactly
  predicates  a conjunction (filter.go:125-141 keeps rows with !null && true); a NULL operand rejects the row.  The column value is
              compared with the float64 constant MATHEMATICALLY, which is what the reference computes once the planner has cast an
              integral constant to the column type (func_compare.go, operator_between.go:138-199: BETWEEN inclusive at both ends).
              A NaN constant follows IEEE like the reference's float compare: != is true, every other comparison false.
  program     float64, one IEEE round-to-nearest per node, no FMA (evalExpression.go:575-640 evaluates one node at a time); integer
              columns enter as float64(value); NULL propagates; x / 0 and x / -0.0 give NULL
  keys        the byte layout of fillKeys (pkg/common/hashmap/inthashmap.go:113-180): with has_null_keys every key column writes a
              marker byte then its value bytes, a NULL writes the marker 1 only; without it a row with a NULL key joins no group
              (zValues[i] = 0, inthashmap.go:171-180).  No keys: one group, present only if a row qualified.
  groups      rows, first_row (+ row_base) and key, numbered in first-seen order (og_group_ids, the observable Int64HashMap order)
  aggregates  COUNT(*) counts rows, COUNT(v) non-NULL values (count2.go); MIN / MAX skip NaN (an all-NaN group is NaN with count > 0),
              -0.0 equals 0.0; SUM is math.fsum (NaN if a NaN or both infinities occur, else the infinity present); AVG = sum / count
              (sumavg2.go:323-335); count 0 = NULL
"""
import math

import numpy as np

from matrixone_b200 import capi

DTYPE = {capi.T_BOOL: np.uint8, capi.T_INT8: np.int8, capi.T_INT16: np.int16, capi.T_INT32: np.int32, capi.T_INT64: np.int64,
         capi.T_UINT8: np.uint8, capi.T_UINT16: np.uint16, capi.T_UINT32: np.uint32, capi.T_UINT64: np.uint64,
         capi.T_FLOAT32: np.float32, capi.T_FLOAT64: np.float64,
         capi.T_DATE: np.int32, capi.T_TIME: np.int64, capi.T_DATETIME: np.int64, capi.T_TIMESTAMP: np.int64}
FLOAT_TYPES = (capi.T_FLOAT32, capi.T_FLOAT64)
EQ, NE, GT, GE, LT, LE, BETWEEN = range(7)
OPS_BY_NAME = capi.PLAN_CMP
U = 2.0 ** -52


def _int_cmp(x, op, t):
    """x (int64 / uint64 array) OP t for a Python int t of any size"""
    info = np.iinfo(x.dtype)
    if op == EQ:
        return x == x.dtype.type(t) if info.min <= t <= info.max else np.zeros(x.shape, bool)
    if op == GT:
        return np.ones(x.shape, bool) if t < info.min else np.zeros(x.shape, bool) if t >= info.max else x > x.dtype.type(t)
    if op == GE:
        return np.ones(x.shape, bool) if t <= info.min else np.zeros(x.shape, bool) if t > info.max else x >= x.dtype.type(t)
    if op == LT:
        return np.zeros(x.shape, bool) if t <= info.min else np.ones(x.shape, bool) if t > info.max else x < x.dtype.type(t)
    assert op == LE
    return np.zeros(x.shape, bool) if t < info.min else np.ones(x.shape, bool) if t >= info.max else x <= x.dtype.type(t)


def compare(x, op, c):
    """exact x OP c of an integer array with a float64 constant (x is an integer: x > c <=> x > floor(c), x >= c <=> x >= ceil(c), ...)"""
    if math.isnan(c):
        return np.full(x.shape, op == NE)
    if math.isinf(c):
        above = c > 0           # every integer is below +inf and above -inf
        return np.full(x.shape, {EQ: False, NE: True, GT: not above, GE: not above, LT: above, LE: above}[op])
    if op in (EQ, NE):
        eq = _int_cmp(x, EQ, int(c)) if c == math.floor(c) else np.zeros(x.shape, bool)
        return eq if op == EQ else ~eq
    if op in (GT, LE):
        return _int_cmp(x, op, math.floor(c))
    return _int_cmp(x, op, math.ceil(c))


def _float_cmp(x, op, c):
    with np.errstate(invalid="ignore"):
        return {EQ: x == c, NE: x != c, GT: x > c, GE: x >= c, LT: x < c, LE: x <= c}[op]


def predicate(T, col, op, lo, hi=0.0):
    """col OP lo (BETWEEN: lo <= col <= hi) for a column of type T, NULLs not considered"""
    if T in FLOAT_TYPES:
        x, cmp = np.asarray(col).astype(np.float64), _float_cmp
    else:
        x, cmp = np.asarray(col).astype(np.uint64 if T == capi.T_UINT64 else np.int64), compare
    if op == BETWEEN:
        return cmp(x, GE, lo) & cmp(x, LE, hi)
    return cmp(x, op, lo)


def null_mask(words, n):
    """nulls bitmap words (or None) -> bool[n]"""
    if words is None:
        return np.zeros(n, bool)
    bits = np.unpackbits(np.ascontiguousarray(words, dtype=np.uint64).view(np.uint8), bitorder="little")
    return bits[:n].astype(bool)


def run(P, cols, nulls, n):
    """P: mo_plan_t (FusedPlan.P); cols: numpy arrays of the declared types; nulls: per column bitmap words or None (or None).
    Returns [{key, first_row, rows, aggs: [(value, count, abs_sum), ...]}] in first-seen order; abs_sum = sum |x| for SUM / AVG."""
    nc = P.ncols
    types = [P.col_type[c] for c in range(nc)]
    raw = [np.ascontiguousarray(cols[c]).view(DTYPE[types[c]])[:n] for c in range(nc)]
    isnull = [null_mask(None if nulls is None else nulls[c], n) for c in range(nc)]

    # ---- filter
    sel = np.ones(n, bool)
    for q in range(P.npreds):
        pr = P.pred[q]
        sel &= predicate(types[pr.col], raw[pr.col], pr.op, pr.lo, pr.hi) & ~isnull[pr.col]

    # ---- program: value slots 0..ncols-1 are the columns, ncols + i instruction i
    vals = [raw[c].astype(np.float64) for c in range(nc)]
    vnull = list(isnull)
    with np.errstate(all="ignore"):
        for i in range(P.ninstr):
            ins = P.instr[i]
            if ins.op == capi.PLAN_OP_CONST:
                vals.append(np.full(n, ins.imm)); vnull.append(np.zeros(n, bool))
            elif ins.op == capi.PLAN_OP_COL:
                vals.append(vals[ins.a].copy()); vnull.append(vnull[ins.a].copy())
            else:
                a, b = vals[ins.a], vals[ins.b]
                nul = vnull[ins.a] | vnull[ins.b]
                if ins.op == capi.PLAN_OP_ADD:
                    v = a + b
                elif ins.op == capi.PLAN_OP_SUB:
                    v = a - b
                elif ins.op == capi.PLAN_OP_MUL:
                    v = a * b
                else:
                    z = b == 0.0
                    v = np.where(z, 0.0, a / np.where(z, 1.0, b))
                    nul = nul | z
                vals.append(v); vnull.append(nul)

    # ---- keys (fillKeys byte layout)
    keys = np.zeros(n, np.uint64)
    if not P.has_null_keys:
        shift = 0
        for k in range(P.nkeys):
            c = P.key_col[k]
            sz = raw[c].dtype.itemsize
            sel &= ~isnull[c]
            keys |= raw[c].view("u%d" % sz).astype(np.uint64) << np.uint64(8 * shift)
            shift += sz
    else:
        off = np.zeros(n, np.uint64)
        for k in range(P.nkeys):
            c = P.key_col[k]
            sz = raw[c].dtype.itemsize
            m = isnull[c]
            keys |= np.where(m, np.uint64(1) << (np.uint64(8) * off), np.uint64(0))
            b = raw[c].view("u%d" % sz).astype(np.uint64) << (np.uint64(8) * (off + np.uint64(1)))
            keys |= np.where(m, np.uint64(0), b)
            off += np.where(m, np.uint64(1), np.uint64(1 + sz))

    rows_idx = np.flatnonzero(sel)
    ks = keys[rows_idx]
    if ks.shape[0] == 0:
        return []
    uniq, first_idx, inv = np.unique(ks, return_index=True, return_inverse=True)
    order = np.argsort(first_idx, kind="stable")
    rank = np.empty_like(order); rank[order] = np.arange(order.shape[0])
    gid = rank[inv.reshape(-1)]
    ng = order.shape[0]
    rows = np.bincount(gid, minlength=ng)
    out_keys = uniq[order]
    first_rows = rows_idx[first_idx[order]] + P.row_base

    # ---- aggregates
    by_group = np.argsort(gid, kind="stable")
    starts = np.concatenate([[0], np.cumsum(rows)])
    aggs = []
    for a in range(P.naggs):
        kind, vs = P.agg[a].kind, P.agg[a].value
        if vs < 0:
            aggs.append((rows.astype(np.float64), rows, np.zeros(ng)))
            continue
        v = vals[vs][rows_idx]
        live = ~vnull[vs][rows_idx]
        cnt = np.bincount(gid[live], minlength=ng)
        if kind == capi.AGG_COUNT:
            aggs.append((cnt.astype(np.float64), cnt, np.zeros(ng)))
        elif kind in (capi.AGG_MIN, capi.AGG_MAX):
            num = live & ~np.isnan(v)
            res = np.full(ng, np.inf if kind == capi.AGG_MIN else -np.inf)
            (np.fmin if kind == capi.AGG_MIN else np.fmax).at(res, gid[num], v[num])
            res[np.bincount(gid[num], minlength=ng) == 0] = np.nan      # no number: NULL (count 0) or all NaN (count > 0)
            aggs.append((res, cnt, np.zeros(ng)))
        else:
            sums = _group_fsum(np.where(live, v, 0.0)[by_group], starts)
            with np.errstate(all="ignore"):
                absum = np.bincount(gid[live], weights=np.abs(v[live]), minlength=ng)
                res = sums if kind == capi.AGG_SUM else sums / np.maximum(cnt, 1)
            aggs.append((res, cnt, absum))
    return [{"key": int(out_keys[g]), "first_row": int(first_rows[g]), "rows": int(rows[g]),
             "aggs": [(float(aggs[a][0][g]), int(aggs[a][1][g]), float(aggs[a][2][g])) for a in range(P.naggs)]} for g in range(ng)]


def _group_fsum(v, starts):
    """exact (correctly rounded) per-group sums of v grouped by [starts[g], starts[g + 1]); IEEE rules for NaN and infinities"""
    ng = starts.shape[0] - 1
    out = np.zeros(ng)
    lst = v.tolist()
    for g in range(ng):
        part = lst[starts[g]:starts[g + 1]]
        try:
            out[g] = math.fsum(part)
        except (ValueError, OverflowError):
            pinf = any(x == math.inf for x in part)
            ninf = any(x == -math.inf for x in part)
            if any(x != x for x in part) or (pinf and ninf):
                out[g] = math.nan
            elif pinf or ninf:
                out[g] = math.inf if pinf else -math.inf
            else:                                   # the exact sum of finite values overflows
                out[g] = math.copysign(math.inf, sum(part))
    return out


def assert_matches(got, want, P, first_row_unknown=False):
    """got: FusedPlan.parse output, want: run().  Exact: group set and order, key, first_row, rows, every count, MIN and MAX (-0.0 == 0.0).
    SUM: |got - fsum| <= m 2^-52 sum|x| (m = count: holds for any summation order); AVG: that bound / m plus a rounding of each side."""
    assert len(got) == len(want), (len(got), len(want))
    if not want:
        return
    gk = np.array([g["key"] for g in got], np.uint64); wk = np.array([g["key"] for g in want], np.uint64)
    bad = np.flatnonzero(gk != wk)
    assert bad.size == 0, ("key", int(bad[0]), hex(int(gk[bad[0]])), hex(int(wk[bad[0]])))
    if not first_row_unknown:
        gf = np.array([g["first_row"] for g in got]); wf = np.array([g["first_row"] for g in want])
        bad = np.flatnonzero(gf != wf)
        assert bad.size == 0, ("first_row", int(bad[0]), int(gf[bad[0]]), int(wf[bad[0]]))
    gr = np.array([g["rows"] for g in got]); wr = np.array([g["rows"] for g in want])
    bad = np.flatnonzero(gr != wr)
    assert bad.size == 0, ("rows", int(bad[0]), int(gr[bad[0]]), int(wr[bad[0]]))
    for a in range(P.naggs):
        kind = P.agg[a].kind
        gv = np.array([g["aggs"][a][0] for g in got]); gc = np.array([g["aggs"][a][1] for g in got])
        wv = np.array([g["aggs"][a][0] for g in want]); wc = np.array([g["aggs"][a][1] for g in want])
        wa = np.array([g["aggs"][a][2] for g in want])
        bad = np.flatnonzero(gc != wc)
        assert bad.size == 0, ("count", a, kind, int(bad[0]), int(gc[bad[0]]), int(wc[bad[0]]))
        has = wc > 0
        if kind == capi.AGG_COUNT:
            ok = gv == wc
        elif kind in (capi.AGG_MIN, capi.AGG_MAX):
            ok = ~has | (gv == wv) | (np.isnan(gv) & np.isnan(wv))
        else:
            with np.errstate(all="ignore"):
                m = np.maximum(wc, 1)
                tol = m * U * wa if kind == capi.AGG_SUM else U * wa + U * np.abs(wv)
                fin = np.isfinite(wv)
                ok = ~has | np.where(fin, np.abs(gv - wv) <= tol, (gv == wv) | (np.isnan(gv) & np.isnan(wv)))
        bad = np.flatnonzero(~ok)
        assert bad.size == 0, ("value", a, kind, int(bad[0]), float(gv[bad[0]]), float(wv[bad[0]]), int(wc[bad[0]]))
