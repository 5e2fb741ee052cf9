"""Case builders for the single-column aggregates (csrc/agg.cu, the H0 path) and the grouped ones (csrc/colops.cu, BatchFill).

agg_kernel reads a 16-byte aligned column as 128-bit vectors of V = 16 / sizeof(T) rows through three loops: an unrolled loop of
8 vectors per thread, a one-vector remainder loop and a scalar tail for the last n % V rows.  A column that is not 16-byte aligned
goes through the scalar loop whole.  The functions here restate launch_agg's sizing and the kernel's row-to-thread mapping, so
that the row counts in regions() can be shown (on the CPU) to run every path, and so that planted rows land on the thread and
CTA a case claims.  The builders make a wrong row mapping visible in an exact result: null rows hold a value no live row has,
and unique extremes sit where the mapping changes.

The functions take the element size in bytes and the SM count; nothing here needs a GPU.
"""
import numpy as np

KTHREADS = 256       # agg_kernel's CTA size
CTAS_PER_SM = 4      # launch_agg: grid = min(CTAS_PER_SM x SMs, ceil(n / (V x KTHREADS)))
UNROLL = 8           # vectors per thread per unrolled iteration


def vec_rows(itemsize):
    """V: rows per 128-bit load"""
    return 16 // itemsize


def grid_of(n, itemsize, sms):
    V = vec_rows(itemsize)
    work = -(-n // (V * KTHREADS))
    return max(1, min(CTAS_PER_SM * sms, work))


def loop_counts(n, itemsize, sms, vec=True):
    """{"unrolled", "remainder", "tail"}: iterations each path runs, summed over the grid's threads (a vector counts once per
    unrolled load), plus "grid", "nthreads" and "nvec"."""
    V = vec_rows(itemsize)
    grid = grid_of(n, itemsize, sms)
    nt = grid * KTHREADS
    nvec = n // V if vec else 0
    tid = np.arange(nt, dtype=np.int64)
    # unrolled: for (v = tid; v + 7 nt < nvec; v += 8 nt)
    u = np.maximum(0, -(-(nvec - (UNROLL - 1) * nt - tid) // (UNROLL * nt)))
    v = tid + UNROLL * nt * u
    rem = np.maximum(0, -(-(nvec - v) // nt))
    return {"unrolled": int(u.sum()) * UNROLL, "remainder": int(rem.sum()), "tail": n - nvec * V,
            "grid": grid, "nthreads": nt, "nvec": nvec}


def owner(row, n, itemsize, sms, vec=True):
    """(cta, thread in the CTA, path) of the thread that reads `row`; path is "unrolled", "remainder" or "tail" ("tail" for every
    row of a column that is not 16-byte aligned)"""
    V = vec_rows(itemsize)
    nt = grid_of(n, itemsize, sms) * KTHREADS
    nvec = n // V if vec else 0
    if row < nvec * V:
        vv = row // V
        tid = vv % nt
        u = max(0, -(-(nvec - (UNROLL - 1) * nt - tid) // (UNROLL * nt)))
        path = "unrolled" if (vv - tid) // nt < UNROLL * u else "remainder"
    else:
        tid = (row - nvec * V) % nt
        path = "tail"
    return tid // KTHREADS, tid % KTHREADS, path


def region_bases(itemsize, sms):
    """(label, vector count) of each loop region; regions() adds 0 .. V - 1 tail rows to each"""
    NT = CTAS_PER_SM * sms * KTHREADS
    return [("no vector", 0),                                     # n < V
            ("nvec < grid threads, one CTA", 100),
            ("nvec < grid threads, 6 CTAs", 5 * KTHREADS + 3),
            ("remainder loop only, 3+ strides", 3 * NT + 17),
            ("unrolled, remainder 0", UNROLL * NT),
            ("unrolled, remainder 1", UNROLL * NT + 1),
            ("unrolled, remainder nthreads - 1", UNROLL * NT + NT - 1),
            ("unrolled, remainder 7 nthreads - 1", UNROLL * NT + 7 * NT - 1)]


def regions(itemsize, sms):
    """[(n, label)] ascending: every region base plus 0 .. V - 1 scalar-tail rows (n = 0 excluded)"""
    V = vec_rows(itemsize)
    out = [(nvec * V + t, "%s + %d tail" % (label, t)) for label, nvec in region_bases(itemsize, sms) for t in range(V)]
    return sorted(o for o in out if o[0] > 0)


# ------------------------------------------------------------------------------------------------------------- data builders
def live_band(dt):
    """(lo, hi): the range live rows are drawn from; values past it (poison and planted extremes) fit the type on both sides"""
    dt = np.dtype(dt)
    if dt.kind == "f":
        return -1000, 1000
    info = np.iinfo(dt)
    if dt.itemsize == 1:
        return int(info.min) + 40, int(info.max) - 40
    if dt.kind == "u":
        return 1000, 1000 + 2 ** (min(8 * dt.itemsize, 40) - 2)
    return -2 ** (min(8 * dt.itemsize, 40) - 2), 2 ** (min(8 * dt.itemsize, 40) - 2)


def poison(dt):
    """(low, high) values for null rows: below and above every live and planted value (SUM: +-2^40 where the type holds it)"""
    dt = np.dtype(dt)
    if dt.kind == "f":
        return -2.0 ** 40, 2.0 ** 40
    info = np.iinfo(dt)
    if dt.itemsize == 8:
        return (0, 2 ** 63) if dt.kind == "u" else (-2 ** 40 - 7, 2 ** 40 + 7)
    return int(info.min), int(info.max)


def poisoned_column(dt, n, rng, null_frac=0.1, neg_zero=True):
    """n rows drawn from live_band, a nulls mask with null_frac of the rows and poison in every null row (alternately low and high).
    Float columns hold small integers, so every partial sum is exact and a float SUM must match the serial loop bit for bit; a
    quarter of their zeros are -0.0.  Returns (col, mask)."""
    dt = np.dtype(dt)
    lo, hi = live_band(dt)
    if dt.kind == "f":
        col = rng.integers(lo, hi, n, endpoint=True).astype(dt)
        if neg_zero:
            z = np.flatnonzero(col == 0)
            col[z[rng.random(len(z)) < 0.25]] = -0.0
    else:
        col = rng.integers(lo, hi, n, endpoint=True, dtype=np.int64 if dt.kind == "i" else np.uint64).astype(dt)
    mask = rng.random(n) < null_frac
    pl, ph = poison(dt)
    idx = np.flatnonzero(mask)
    col[idx[0::2]] = pl
    col[idx[1::2]] = ph
    return col, mask


def bitmap_with_tail_bits(mask, rng):
    """the nulls bitmap of mask, with random bits set past len in the last word (rows the call must not read)"""
    n = len(mask)
    words = np.zeros((n + 63) // 64, np.uint64)
    bits = np.packbits(np.asarray(mask, np.uint8), bitorder="little")
    words.view(np.uint8)[:len(bits)] = bits
    if n % 64:
        junk = np.uint64(int(rng.integers(0, 2 ** 63, dtype=np.int64)) << (n % 64) & (2 ** 64 - 1))
        words[-1] |= junk
    return words


def planted_rows(n, itemsize, sms, mask):
    """{name: row}: where a unique extreme is planted: the first and last row, row 64k + 63 (the last row of a nulls word, the
    middle one that exists), the first live row after a null row, and the first row of each loop path in use"""
    out = {"first": 0, "last": n - 1}
    if n > 64:
        k = (n // 64) // 2
        out["64k+63"] = 64 * k + 63
    after = np.flatnonzero(mask[:-1] & ~mask[1:])
    if len(after):
        out["after null"] = int(after[len(after) // 2]) + 1
    c = loop_counts(n, itemsize, sms)
    V, nt, nvec = vec_rows(itemsize), c["nthreads"], c["nvec"]
    if nvec >= UNROLL * nt:          # the last vector of the last thread's first unrolled iteration
        out["unrolled, last thread"] = (UNROLL * nt - 1) * V + V - 1
    if c["remainder"]:               # thread 0's first remainder vector
        u0 = max(0, -(-(nvec - (UNROLL - 1) * nt) // (UNROLL * nt)))
        out["remainder, thread 0"] = UNROLL * nt * u0 * V
    if c["tail"]:
        out["tail, last"] = n - 1
    return out


def plant_extreme(col, mask, row, is_max, value, rng=None):
    """make col[row] the unique extreme (value, past every live value) and put a more extreme value into a null row next to it.
    The caller guarantees row is live.  Returns the neighbour null row (or None)."""
    col[row] = value
    mask[row] = False
    nb = row + 1 if row + 1 < len(col) else row - 1
    if nb < 0 or nb == row:
        return None
    mask[nb] = True
    dt = col.dtype
    pl, ph = poison(dt)
    col[nb] = ph if is_max else pl
    return nb


def zero_tie_rows(n, itemsize, sms, kind):
    """(first_zero_row, other_zero_row) for a float column with n rows where the first zero in row order and the first zero in the
    kernel's thread / CTA order disagree: other_zero_row is read by a thread that comes before first_zero_row's thread.
      "lane":  the first zero at thread 5 of CTA 0's first vector, the other at thread 0's next stride or its scalar tail
      "cta":   the first zero in CTA 1, the other in CTA 0 (a later stride)
      "tail":  the first zero in a vector row, the other in the scalar tail on thread 0"""
    V = vec_rows(itemsize)
    c = loop_counts(n, itemsize, sms)
    nt = c["nthreads"]
    if kind == "lane":
        first = 5 * V + 1
        other = nt * V if c["nvec"] > nt else c["nvec"] * V
    elif kind == "cta":
        first = KTHREADS * V + 2
        other = nt * V
    else:
        first = 7 * V + V - 1
        other = c["nvec"] * V
    return first, other
