"""The aggregate case builders (agg_cases.py) against agg_kernel's sizing and row mapping, counted on the CPU: the row counts of
regions() run every loop path at the SM counts of the H100 SXM (132) and PCIe (114), and planted rows land where they are
claimed to, so the GPU tests built on them cannot pass without reaching the path they aim at."""
import numpy as np
import pytest

import agg_cases as A

SIZES = [1, 2, 4, 8]


def _brute_owner(n, itemsize, sms):
    """row -> (cta, thread, path) by walking agg_kernel's loops thread by thread (small n only)"""
    V = A.vec_rows(itemsize)
    nt = A.grid_of(n, itemsize, sms) * A.KTHREADS
    nvec = n // V
    out = {}
    for tid in range(nt):
        v = tid
        while v + (A.UNROLL - 1) * nt < nvec:
            for k in range(A.UNROLL):
                for j in range(V):
                    out[(v + k * nt) * V + j] = (tid, "unrolled")
            v += A.UNROLL * nt
        while v < nvec:
            for j in range(V):
                out[v * V + j] = (tid, "remainder")
            v += nt
        for i in range(nvec * V + tid, n, nt):
            out[i] = (tid, "tail")
    return out


@pytest.mark.parametrize("sms", [114, 132])
@pytest.mark.parametrize("itemsize", SIZES)
def test_regions_run_every_loop_path(itemsize, sms):
    V = A.vec_rows(itemsize)
    full = A.CTAS_PER_SM * sms
    seen = set()
    for n, label in A.regions(itemsize, sms):
        c = A.loop_counts(n, itemsize, sms)
        assert c["unrolled"] % A.UNROLL == 0
        # every row is read once: unrolled and remainder vectors cover nvec, the tail the rest
        assert c["unrolled"] + c["remainder"] == c["nvec"] and c["nvec"] * V + c["tail"] == n, label
        if c["nvec"] == 0:
            seen.add("no vector")
        if 0 < c["nvec"] < c["nthreads"]:
            seen.add("nvec < grid threads")
        if c["grid"] < full:
            seen.add("partial grid")
        if c["grid"] == full and c["unrolled"] == 0 and c["remainder"] >= 3 * c["nthreads"]:
            seen.add("remainder only, full grid, 3 strides")
        if c["unrolled"]:
            seen.add("unrolled")
            rem = c["nvec"] - A.UNROLL * c["nthreads"] * (c["nvec"] // (A.UNROLL * c["nthreads"]))
            seen.add("unrolled, remainder %s" % {0: "0", 1: "1", c["nthreads"] - 1: "nt-1", 7 * c["nthreads"] - 1: "7nt-1"}.get(rem, "other"))
            if c["tail"] == V - 1:
                seen.add("unrolled + tail V-1")
        if c["tail"]:
            seen.add("tail %d" % c["tail"])
    want = {"no vector", "nvec < grid threads", "partial grid", "remainder only, full grid, 3 strides", "unrolled",
            "unrolled, remainder 0", "unrolled, remainder 1", "unrolled, remainder nt-1", "unrolled, remainder 7nt-1"}
    want |= {"tail %d" % t for t in range(1, V)}
    if V > 1:
        want.add("unrolled + tail V-1")
    assert want <= seen, want - seen
    # the unrolled loop first runs at nvec = 8 x grid threads (132 SMs: 2.16 M rows of an 8-byte type, 17.3 M of a 1-byte type)
    if sms == 132:
        assert min(n for n, _ in A.regions(itemsize, sms) if A.loop_counts(n, itemsize, sms)["unrolled"]) == A.UNROLL * full * 256 * V


@pytest.mark.parametrize("itemsize", SIZES)
def test_owner_matches_a_walk_of_the_loops(itemsize):
    """owner() against a row-by-row walk of the kernel's loops, with 1 SM so the unrolled loop is reached at small n"""
    sms = 1
    V = A.vec_rows(itemsize)
    nt = A.CTAS_PER_SM * sms * A.KTHREADS
    for nvec in (0, 3, 300, 3 * nt + 5, 8 * nt, 8 * nt + 1, 9 * nt - 1, 15 * nt - 1):
        for t in sorted({0, 1, V - 1}):
            n = nvec * V + t
            if n == 0:
                continue
            walk = _brute_owner(n, itemsize, sms)
            assert sorted(walk) == list(range(n))
            rows = np.unique(np.r_[np.arange(0, n, max(1, n // 997)), n - 1, np.arange(max(0, n - 2 * V), n)])
            for r in rows:
                cta, th, path = A.owner(int(r), n, itemsize, sms)
                assert (cta * A.KTHREADS + th, path) == walk[int(r)], (n, r)
            c = A.loop_counts(n, itemsize, sms)
            assert c["unrolled"] * V == sum(1 for p in walk.values() if p[1] == "unrolled")
            assert c["remainder"] * V == sum(1 for p in walk.values() if p[1] == "remainder")


@pytest.mark.parametrize("sms", [114, 132])
@pytest.mark.parametrize("itemsize", SIZES)
def test_planted_rows_land_where_claimed(itemsize, sms):
    rng = np.random.default_rng(itemsize + sms)
    V = A.vec_rows(itemsize)
    for n, label in A.regions(itemsize, sms):
        if n % V not in (0, V - 1):
            continue
        mask = rng.random(n) < 0.1
        rows = A.planted_rows(n, itemsize, sms, mask)
        assert rows["first"] == 0 and rows["last"] == n - 1
        if "64k+63" in rows:
            assert rows["64k+63"] % 64 == 63 and rows["64k+63"] < n
        if "after null" in rows:
            assert mask[rows["after null"] - 1] and not mask[rows["after null"]]
        for name, path in (("unrolled, last thread", "unrolled"), ("remainder, thread 0", "remainder"), ("tail, last", "tail")):
            if name in rows:
                cta, th, p = A.owner(rows[name], n, itemsize, sms)
                assert p == path, (label, name)
                if name == "unrolled, last thread":
                    assert cta * A.KTHREADS + th == A.loop_counts(n, itemsize, sms)["nthreads"] - 1
                if name == "remainder, thread 0":
                    assert (cta, th) == (0, 0)
        c = A.loop_counts(n, itemsize, sms)
        assert ("unrolled, last thread" in rows) == (c["nvec"] >= A.UNROLL * c["nthreads"])
        assert ("remainder, thread 0" in rows) == (c["remainder"] > 0)
        if n > 100_000:
            continue
        # plant_extreme: the planted row is live, its neighbour null and more extreme
        col, m = A.poisoned_column(np.int32, n, rng)
        lo, hi = A.live_band(np.int32)
        r = rows["last"]
        nb = A.plant_extreme(col, m, r, False, lo - 1)
        assert not m[r] and col[r] == lo - 1 and col[~m].min() == lo - 1 and np.count_nonzero(col[~m] == lo - 1) == 1
        if nb is not None:
            assert m[nb] and col[nb] < col[r]


@pytest.mark.parametrize("sms", [114, 132])
@pytest.mark.parametrize("itemsize", [4, 8])
def test_zero_tie_rows_disagree_in_row_and_thread_order(itemsize, sms):
    """the first zero in row order is read by a later thread (or CTA) than another zero, so a reduction that breaks ties by thread
    order keeps the wrong zero"""
    V = A.vec_rows(itemsize)
    nt = A.CTAS_PER_SM * sms * A.KTHREADS
    for kind, n in (("lane", 3 * nt * V + 1), ("lane", 100 * V + 1), ("cta", 3 * nt * V), ("cta", 9 * nt * V + V - 1),
                    ("tail", 100 * V + 3), ("tail", 8 * nt * V + V - 1)):
        first, other = A.zero_tie_rows(n, itemsize, sms, kind)
        assert first < other < n, (kind, n)
        c1, t1, _ = A.owner(first, n, itemsize, sms)
        c2, t2, p2 = A.owner(other, n, itemsize, sms)
        assert (c2, t2) < (c1, t1), (kind, n)
        if kind == "cta":
            assert c2 < c1
        if kind == "tail":
            assert p2 == "tail"


def test_bitmap_tail_bits_and_poison():
    rng = np.random.default_rng(1)
    for n in (1, 63, 64, 65, 1000):
        mask = rng.random(n) < 0.3
        w = A.bitmap_with_tail_bits(mask, rng)
        bits = np.unpackbits(w.view(np.uint8), bitorder="little").astype(bool)
        assert np.array_equal(bits[:n], mask)
        if n % 64:
            assert len(w) == (n + 63) // 64
    for dt in (np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64):
        col, m = A.poisoned_column(dt, 10_000, rng)
        lo, hi = A.live_band(dt)
        live = col[~m]
        assert live.min() >= lo and live.max() <= hi
        pl, ph = A.poison(dt)
        assert pl < lo - 1 and ph > hi + 1        # poison stays past a planted extreme lo - 1 / hi + 1
        assert set(np.unique(col[m]).tolist()) <= {dt(pl), dt(ph)}
