"""Host restatement of the hash join with a non-equality condition (test infrastructure): container.probe with NonEqCond != nil
(pkg/sql/colexec/hashjoin/join.go:383-628; HashOnUnique at 450-498, the sels path at 499-611), the condition given per candidate pair.

The candidate pairs of a probe batch are its INNER pairs (join_outer_reference.probe with JOIN_INNER): probe rows ascending, per row its sels
ascending.  cond[k] is the condition of candidate k: True, False or None (NULL); evalNonEqCondition (join.go:763-782) passes a pair only when the
result is true and not NULL.  probe() is the reference's row loop; probe_fast() is the same result in numpy over the candidate pairs (JOIN_COND's
arguments) for the sizes the GPU tests use, and the CPU tests hold the two equal.  Errors carry the row the device names, as in
join_outer_reference."""
import numpy as np

from join_outer_reference import SingleError, checkers

DEFAULT_BATCH_SIZE = 8192                                 # colexec.DefaultBatchSize: the result rows of one returned batch


def passes(c):
    return c is not None and bool(c)


def probe(vals, offsets, sels, join_type, cond, matched=None, batch_size=DEFAULT_BATCH_SIZE):
    """container.probe over Find's ids with a NonEqCond: the result pairs of one probe batch, over every result batch the loop returns.
    `matched` (numpy bool[nbuild], rightRowsMatched) is marked in place for the right-flavoured types."""
    h = checkers(join_type)
    unique = offsets is None
    out_p, out_b = [], []
    twice = []                                            # RIGHT SINGLE: build rows found marked already (join.go:481,574)
    res = 0                                               # resRowCnt of the result batch being filled

    def emit(row, b):
        nonlocal res
        out_p.append(row); out_b.append(b)
        res += 1

    def mark(r):
        if h.IsSingle() and matched[r]:
            twice.append(r)
        matched[r] = True

    k = 0                                                 # the candidate position of the row's first candidate
    for row in range(len(vals)):
        v = int(vals[row])
        if v == 0:                                        # z == 0 || v == 0 (join.go:433-449)
            if h.EmitUnmatchedProbe():
                emit(row, -1)                             # appendOneNotMatch
        elif unique:                                      # join.go:476-497
            idx = v - 1
            if passes(cond[k]):
                if not h.IsRightSemi() and not h.IsAnti():
                    emit(row, -1 if h.IsLeftSemi() else idx)
                if h.right:
                    mark(idx)
            elif h.EmitUnmatchedProbe():
                emit(row, -1)
            k += 1
        else:
            rsels = [int(x) for x in sels[offsets[v - 1]:offsets[v]]]   # GetSels; no filtering with a NonEqCond (join.go:500-516)
            left_matched = False                          # leftRowMatched
            j = 0
            while j < len(rsels):                         # psSelsForOneRow, processCount sels at a time (join.go:570-611)
                count = min(len(rsels) - j, batch_size - res)
                for jj in range(j, j + count):
                    s = rsels[jj]
                    if not passes(cond[k + jj]):
                        continue
                    if h.right:
                        mark(s)
                    elif h.IsSingle() and left_matched:
                        raise SingleError(probe_row=row)
                    left_matched = True
                    if not h.IsRightSemi() and not h.IsAnti():
                        emit(row, -1 if h.IsLeftSemi() else s)
                    if h.IsLeftSemi():                    # ctr.sels = nil; break
                        count = len(rsels) - j
                        break
                j += count
                if j == len(rsels) and not left_matched and h.EmitUnmatchedProbe():
                    emit(row, -1)
                if res >= batch_size:
                    res = 0                               # the batch is returned; the loop resumes where it stopped
            k += len(rsels)
            continue
        if res >= batch_size:
            res = 0
    if twice:
        raise SingleError(build_row=min(twice))
    return np.array(out_p, np.int64), np.array(out_b, np.int64)


def probe_fast(cand_probe, cand_build, cond, cond_null, nprobe, join_type, matched=None):
    """probe() in numpy over the candidate pairs: the same pairs, marks and errors.  cond / cond_null: bool per candidate (cond_null None = no
    NULLs)."""
    h = checkers(join_type)
    cp = np.asarray(cand_probe, np.int64)
    cb = np.asarray(cand_build, np.int64)
    f = np.asarray(cond, bool).copy()
    if cond_null is not None:
        f &= ~np.asarray(cond_null, bool)
    pp, pb = cp[f], cb[f]                                 # P(i) of every row, rows ascending, in candidate order
    pc = np.bincount(pp, minlength=nprobe) if len(pp) else np.zeros(nprobe, np.int64)
    if h.IsLeftSingle() and (pc > 1).any():
        raise SingleError(probe_row=int(np.flatnonzero(pc > 1)[0]))
    if h.right:
        if h.IsSingle():
            hits = matched.astype(np.int64) + (np.bincount(pb, minlength=len(matched)) if len(pb) else 0)
            matched[pb] = True
            bad = np.flatnonzero(hits > 1)
            if len(bad):
                raise SingleError(build_row=int(bad[0]))
        matched[pb] = True
    if h.IsRightSemi() or h.IsRightAnti():
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    if h.IsLeftSemi() or h.IsLeftAnti():
        r = np.flatnonzero(pc > 0 if h.IsLeftSemi() else pc == 0)
        return r.astype(np.int64), np.full(len(r), -1, np.int64)
    if not h.EmitUnmatchedProbe():
        return pp, pb
    c = np.maximum(pc, 1)                                 # (i, -1) for a row without a passing pair
    out_p = np.repeat(np.arange(nprobe, dtype=np.int64), c)
    out_b = np.full(len(out_p), -1, np.int64)
    out_b[np.repeat(pc > 0, c)] = pb
    return out_p, out_b
