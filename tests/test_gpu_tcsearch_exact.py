"""The tensor-core search (csrc/tcsearch.cu) returns the exact answer at the shapes, data and modes where its completeness
proof is weakest.  Every case forces the tensor-core path (search_mode 2), checks the result with
search_reference.check_exact_topk (Go-order oracle, bit-exact distances, lowest key in a tie, and an independent float64
check), and shows that the candidate pass did the work: it ran (get_tc_kused) and proved at least one query without the
exact kernel (get_tc_fallbacks < nq) -- unless the case exists to force fallbacks."""
import numpy as np
import pytest

import oracle_lib as O
import search_reference as S
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, xcall

pytestmark = pytest.mark.gpu

L2, IP, COS = capi.METRIC_L2, capi.METRIC_IP, capi.METRIC_COS
KNOBS = ("tc_pair", "tc_ladder", "tc_share", "tc_range_mb")


def _stat(gpu, name):
    return int(gpu.MoB200_SetTuning(name.encode(), 0))


def _with_knobs(gpu, knobs, fn):
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        for name in KNOBS:
            gpu.MoB200_SetTuning(name.encode(), int(knobs.get(name, 0)))
        return fn()
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
        for name in KNOBS:
            gpu.MoB200_SetTuning(name.encode(), 0)


def bf_search(gpu, ds, qs, k, metric=L2, key_base=0, prepared=True, device_io=False, **knobs):
    """brute-force search on the tensor-core path: (keys, dists, K columns of the candidate pass, fallbacks)"""
    nq, dim = qs.shape

    def run():
        idx = ops.BruteForceIndex(ds, dim, metric, key_base=key_base)
        try:
            if not prepared:   # the operand is split per call instead of once at load
                gpu.MoB200_SearchRelease(idx.buf.ptr)
                idx.prepared = False
            if device_io:      # queries in device memory, results left in device memory
                dq = DeviceBuffer.from_numpy(qs)
                kd, dd = DeviceBuffer(nq * k * 8), DeviceBuffer(nq * k * 8)
                try:
                    idx.search(dq, k, out=(kd.ptr, dd.ptr))
                    keys, dists = kd.to_numpy(np.int64), dd.to_numpy(np.float64)
                finally:
                    dq.free(); kd.free(); dd.free()
            else:
                keys, dists = idx.search(qs, k)
            return keys, dists, _stat(gpu, "get_tc_kused"), _stat(gpu, "get_tc_fallbacks")
        finally:
            idx.destroy()
    return _with_knobs(gpu, knobs, run)


def expected_kused(dim, k, ladder):
    """the first candidate pass multiplies the hi.hi columns (one-term level: ladder 2, k <= 16) or the whole K'"""
    return 64 * ((dim + 63) // 64) if ladder == 2 and k <= 16 else S.kprime(dim)


def did_the_work(kused, fallbacks, nq, dim, k, ladder):
    assert kused == expected_kused(dim, k, ladder), (kused, expected_kused(dim, k, ladder))
    assert 0 <= fallbacks < nq, (fallbacks, nq)


# ---- shape grid ----------------------------------------------------------------------------------------------------------
# (dim, n, nq, k, metric, knobs, prepared, device_io, key_base): every dim, n, nq and k value and every knob setting appears;
# tc_range_mb=1 at dim 1024 over 40,000 rows makes 79 row ranges (more than 64 merge lists per query)
GRID = [
    (16, 128, 1, 1, L2, dict(tc_pair=1, tc_ladder=1), True, False, 0),
    (17, 129, 127, 16, L2, dict(tc_ladder=2), False, False, 0),
    (33, 1023, 128, 16, IP, dict(tc_ladder=2, tc_share=1), True, True, 0),
    (100, 1024, 129, 17, L2, dict(tc_pair=2, tc_ladder=1), True, False, 0),
    (129, 20_001, 255, 32, COS, dict(tc_ladder=1), True, False, 0),
    (1024, 20_001, 256, 16, L2, dict(tc_pair=2, tc_ladder=2), False, False, 0),
    (1536, 1024, 257, 1, COS, dict(tc_pair=2, tc_ladder=2), True, True, 0),
    (3072, 1023, 1000, 16, L2, dict(tc_pair=1, tc_ladder=2, tc_share=1), True, False, 0),
    (4096, 20_001, 129, 16, IP, dict(tc_ladder=2), True, False, 0),
    (4096, 1024, 257, 32, L2, dict(tc_pair=2, tc_ladder=1), False, True, 0),
    (1024, 40_000, 257, 10, L2, dict(tc_ladder=2, tc_range_mb=1), True, False, 0),
    (100, 20_001, 1000, 16, L2, dict(tc_pair=2, tc_ladder=1, tc_share=1), True, False, 0),
    (33, 1024, 256, 32, IP, dict(tc_pair=2, tc_ladder=1), True, False, 0),
    (17, 20_001, 257, 17, COS, dict(tc_ladder=2, tc_share=1), False, False, 1 << 33),
    (129, 128, 255, 1, L2, dict(tc_pair=2, tc_ladder=2), True, True, 7),
    (16, 1023, 128, 16, L2, dict(tc_ladder=1), False, False, 1 << 40),
    (1536, 20_001, 127, 16, COS, dict(tc_ladder=2), True, False, 0),
]


@pytest.mark.parametrize("dim,n,nq,k,metric,knobs,prepared,device_io,key_base", GRID,
                         ids=["d%d-n%d-q%d-k%d-m%d-%s%s%s" % (g[0], g[1], g[2], g[3], g[4], "-".join("%s%d" % kv for kv in sorted(g[5].items())),
                                                            "" if g[6] else "-unprep", "-dev" if g[7] else "") for g in GRID])
def test_shape_grid_is_exact(gpu, dim, n, nq, k, metric, knobs, prepared, device_io, key_base):
    rng = np.random.default_rng(dim * 7 + n + nq + k)
    ds = rng.standard_normal((n, dim)).astype(np.float32)
    qs = rng.standard_normal((nq, dim)).astype(np.float32)
    qs[:min(3, nq)] = ds[[0, n // 2, n - 1][:min(3, nq)]]          # self matches
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, k, metric, key_base, prepared, device_io, **knobs)
    S.check_exact_topk(keys, dists, ds, qs, k, metric, key_base)
    did_the_work(kused, fallbacks, nq, dim, k, knobs.get("tc_ladder", 0))


# ---- adversarial data ------------------------------------------------------------------------------------------------------
def _bf16_down(u):
    """bf16 truncation of non-negative fp32 values: bf16-exact and never larger"""
    return (np.ascontiguousarray(u, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def _bf16_rows(rng, m, dim, norm2):
    """bf16-exact non-negative rows with |x|^2 <= norm2"""
    u = rng.random((m, dim)).astype(np.float32)
    u *= np.float32(np.sqrt(norm2)) / np.linalg.norm(u, axis=1, keepdims=True).astype(np.float32)
    return _bf16_down(u)


def hidden_neighbour_data(dim, n=1024, nadv=4, nplain=60, seed=0, per_step=1, ndecoy=20, frac=8):
    """bf16-exact non-negative rows where a truncating accumulator hides the nearest neighbour behind decoys.

    per_step=1: query h is S.lost_tail_rows(dim, h); its nearest row is an exact copy (distance 0), which a truncating fp32
    accumulator sees at 2 T units (T tail components, unit = TAIL^2 ~ 2^-23).  The decoys drop a = 4, 6, ..., 42 tail components
    (ndecoy=20; 4, 5, ..., 43 for 40): real distance a units, seen at 2 T - a.  The decoys seen closest fill the list of the
    copy's row range and push it out; the best of them sits 2 T - 24 units from that list's threshold -- more than the
    fixed-step bound (~145 units at |q|, |x| ~ 1) and less than the step-dependent one from dim 1536 on.
    per_step=16: sixteen TAIL16[frac] products (just under 1/frac ulp) per k16 step; the decoys drop 8, 16, ..., 160 of them, one
    per k16 block (dim >= 2592), each worth 1/frac ulp of distance.  The H100 truncates every such product away: the copy is seen
    at ~2 T 16/frac ulps and each decoy 1/frac ulp closer per dropped product, past a bound of one (frac=8) or three (frac=4)
    ulps a step; the bound prices 17.
    The other queries are plain rows of the dataset."""
    rng = np.random.default_rng(seed + dim)
    ds = _bf16_rows(rng, n, dim, 0.98)
    qs = np.empty((nadv + nplain, dim), dtype=np.float32)
    drops = [8 * (j + 1) for j in range(ndecoy)] if per_step == 16 else [4 + (40 // ndecoy) * j for j in range(ndecoy)]
    for h in range(nadv):
        q, tail = S.lost_tail_rows(dim, h, per_step, frac)
        qs[h] = q
        r0 = 128 * (2 * h + 1) + 10            # copy + decoys inside one 128-row tile, so inside one row range
        ds[r0] = q
        for j, a in enumerate(drops):
            x = q.copy(); x[tail[:a]] = 0.0
            ds[r0 + 1 + j] = x
    plain = rng.choice(np.arange(1024 + 10, n) if n > 1100 else np.arange(0, 128), nplain, replace=False)
    qs[nadv:] = ds[plain]
    return ds, qs


@pytest.mark.parametrize("no_share", [0, 1])     # tc_share=1 turns cross-unit threshold sharing off
@pytest.mark.parametrize("dim,per_step,frac", [(1536, 1, 8), (3072, 1, 8), (4096, 1, 8), (3072, 16, 8), (4096, 16, 8), (3072, 16, 4), (4096, 16, 4)])
def test_bf16_exact_rows_do_not_hide_the_nearest_neighbour(gpu, dim, per_step, frac, no_share):
    """the bound must price the accumulation of the pass that ran: a one-term pass over dim columns runs dim/16 k16 steps,
    and each of them may lose up to 17 ulps of its largest term"""
    ds, qs = hidden_neighbour_data(dim, n=2048, per_step=per_step, frac=frac)
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, 1, L2, tc_ladder=2, tc_share=no_share)
    S.check_exact_topk(keys, dists, ds, qs, 1, L2)
    assert dists.reshape(-1)[:4].tolist() == [0.0] * 4
    did_the_work(kused, fallbacks, qs.shape[0], dim, 1, 2)


def lo_aligned_hidden_neighbour_data(dim=64, n=4096, nadv=4, nplain=60, seed=1):
    """rows whose bf16 residual points along the row: q = h (1 + 2^-10) with h bf16-exact, so the one-term pass misses
    q.x - qh.xh ~ 2^-9 |q||x| in full, close to what the one-term bound allows.  The copy of q (distance 0) is seen ~2^-8 |q|^2
    away, twenty bf16-exact decoys (components lowered by 10 bf16 steps) only half as far off: the decoys fill the copy's list
    and a bound that is too small by a factor of 4 would prove the best decoy to be the nearest row."""
    rng = np.random.default_rng(seed + dim)
    ds = _bf16_down(rng.uniform(0.75, 1.0, (n, dim)))
    qs = np.empty((nadv + nplain, dim), dtype=np.float32)
    for h in range(nadv):
        hq = _bf16_down(rng.uniform(0.75, 1.0, dim))
        qs[h] = hq * np.float32(1 + 2.0 ** -10)
        r0 = 128 * (2 * h + 1) + 10
        ds[r0] = qs[h]
        for j in range(20):
            x = hq.copy(); x[:5 + 2 * j] -= np.float32(10 * 2.0 ** -8)
            ds[r0 + 1 + j] = x
    qs[nadv:] = ds[rng.choice(np.arange(1100, n), nplain, replace=False)]
    return ds, qs


def test_lo_aligned_rows_do_not_hide_the_nearest_neighbour(gpu):
    """the one-term bound is nearly tight here: the pass must not prove a decoy to be the nearest row"""
    ds, qs = lo_aligned_hidden_neighbour_data()
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, 1, L2, tc_ladder=2, tc_share=1)
    S.check_exact_topk(keys, dists, ds, qs, 1, L2)
    assert dists.reshape(-1)[:4].tolist() == [0.0] * 4
    did_the_work(kused, fallbacks, qs.shape[0], ds.shape[1], 1, 2)


@pytest.mark.parametrize("ladder", [1, 2])
def test_crowd_spread_over_row_ranges(gpu, ladder):
    """100 rows around one point, two or so per row range, each range's list otherwise far: more crowd rows than the merge
    re-scores, so the first unconsumed entry of a list (not its full-list threshold) is what bounds the rows left out"""
    rng = np.random.default_rng(17)
    n, dim, nq, k = 20_001, 64, 64, 10
    ds = rng.standard_normal((n, dim)).astype(np.float32)
    c = rng.standard_normal(dim)
    crowd = np.linspace(100, n - 100, 100).astype(np.int64)
    ds[crowd] = (c + 1e-3 * rng.standard_normal((100, dim))).astype(np.float32)
    qs = rng.standard_normal((nq, dim)).astype(np.float32)
    qs[0::2] = (c + 1e-3 * rng.standard_normal((nq // 2, dim))).astype(np.float32)
    qs[1::2] = ds[rng.choice(np.setdiff1d(np.arange(n), crowd), nq // 2, replace=False)]
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, k, L2, tc_ladder=ladder)
    S.check_exact_topk(keys, dists, ds, qs, k, L2)
    assert kused == expected_kused(dim, k, ladder) and 0 < fallbacks < nq, (kused, fallbacks)


def test_large_common_offset_defeats_the_proof(gpu):
    """|q|, |x| ~ 8000 with neighbour gaps ~ 1e-6 of that: tc_eps dwarfs the gaps, the proof fails, the exact kernel answers"""
    rng = np.random.default_rng(11)
    n, dim, nq, k = 4096, 64, 256, 8
    ds = (np.float32(1000.0) + np.float32(1e-3) * rng.standard_normal((n, dim))).astype(np.float32)
    qs = (np.float32(1000.0) + np.float32(1e-3) * rng.standard_normal((nq, dim))).astype(np.float32)
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, k, L2, tc_ladder=1)
    S.check_exact_topk(keys, dists, ds, qs, k, L2)
    assert kused == S.kprime(dim) and fallbacks > nq // 2, (kused, fallbacks)


@pytest.mark.parametrize("pair", [1, 2])
@pytest.mark.parametrize("ladder", [1, 2])
def test_duplicates_across_range_and_pair_boundaries_keep_key_order(gpu, pair, ladder):
    """seven copies of a row at 5, 127/128 (tile edge), 255/256, 1023/1024; queries at the CTA-pair seam (rows 127/128 and
    255/256 of the batch): a tie cut by the k-th place keeps the lowest keys, in order, under a large key_base"""
    rng = np.random.default_rng(12)
    n, dim, nq, k = 4096, 32, 300, 4
    ds = rng.standard_normal((n, dim)).astype(np.float32)
    dup = [5, 127, 128, 255, 256, 1023, 1024]
    ds[dup] = ds[5]
    qs = rng.standard_normal((nq, dim)).astype(np.float32)
    seam = [0, 127, 128, 255, 256, 299]
    qs[seam] = ds[5] + np.float32(1e-2) * rng.standard_normal((len(seam), dim)).astype(np.float32)
    base = (1 << 35) + 3
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, k, L2, key_base=base, tc_pair=pair, tc_ladder=ladder)
    S.check_exact_topk(keys, dists, ds, qs, k, L2, key_base=base)
    assert (keys.reshape(nq, k)[seam] == np.asarray(dup[:k]) + base).all()
    did_the_work(kused, fallbacks, nq, dim, k, ladder)


@pytest.mark.parametrize("pair", [1, 2])
def test_mirror_rows_tie_in_key_order(gpu, pair):
    """x and 2q - x (both exact in fp32) have bit-identical Go-order distances to q but different approximate ones, so the
    candidate pass may list them in either order: the result must still put the lower key first"""
    rng = np.random.default_rng(16)
    n, dim, nq, k = 4096, 48, 256, 6
    grid = lambda a: (np.floor(a * 2 ** 22) / 2 ** 22).astype(np.float32)      # multiples of 2^-22 in [1, 2): 2q - x is exact
    ds = grid(rng.uniform(1, 2, (n, dim)))
    qs = grid(rng.uniform(1.25, 1.75, (nq, dim)))
    perm = rng.permutation(n)[:6 * nq].reshape(nq, 6)
    for q in range(nq):
        rows = perm[q]
        for j, r in enumerate(rows[:3]):
            x = grid(qs[q] + (0.01 * (j + 1)) * rng.uniform(-1, 1, dim))
            ds[r], ds[rows[3 + j]] = x, 2 * qs[q] - x
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, k, L2, tc_pair=pair, tc_ladder=1)
    S.check_exact_topk(keys, dists, ds, qs, k, L2)
    d = dists.reshape(nq, k)
    assert (d[:, 0::2] == d[:, 1::2]).mean() > 0.9          # the mirror pairs did tie
    did_the_work(kused, fallbacks, nq, dim, k, 1)


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("scale", [1e-18, 1e18])
@pytest.mark.parametrize("ladder", [1, 2])
def test_tiny_and_huge_rows(gpu, scale, ladder, metric):
    """rows scaled by 1e-18 (|q|^2 |x|^2 underflows fp32) and by 1e18 (|q|^2 + |x|^2 near the fp32 limit), with planted
    near neighbours 1e-3 apart"""
    rng = np.random.default_rng(13)
    n, dim, nq, k = 4096, 64, 256, 8
    ds = rng.standard_normal((n, dim))
    qs = rng.standard_normal((nq, dim))
    for q in range(0, nq, 8):   # a run of neighbours at growing distance
        ds[q * 12:q * 12 + 12] = qs[q] + 0.05 * (1 + 1e-3 * np.arange(12))[:, None] * rng.standard_normal(dim) / 8
    ds = (ds * scale).astype(np.float32); qs = (qs * scale).astype(np.float32)
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, k, metric, tc_ladder=ladder)
    S.check_exact_topk(keys, dists, ds, qs, k, metric)
    did_the_work(kused, fallbacks, nq, dim, k, ladder)


@pytest.mark.parametrize("ladder", [1, 2])
def test_cosine_near_parallel_rows_of_very_different_lengths(gpu, ladder):
    rng = np.random.default_rng(14)
    n, dim, nq, k = 4096, 64, 64, 10
    ds = rng.standard_normal((n, dim)).astype(np.float32)
    v = rng.standard_normal(dim)
    lengths = 10.0 ** rng.uniform(-3, 3, 300)
    ds[1000:1300] = (lengths[:, None] * (v + 1e-4 * rng.standard_normal((300, dim)))).astype(np.float32)
    qs = rng.standard_normal((nq, dim)).astype(np.float32)
    qs[:nq // 2] = (v + 1e-4 * rng.standard_normal((nq // 2, dim))).astype(np.float32)
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, k, COS, tc_ladder=ladder)
    S.check_exact_topk(keys, dists, ds, qs, k, COS)
    did_the_work(kused, fallbacks, nq, dim, k, ladder)


@pytest.mark.parametrize("ladder", [1, 2])
def test_mixed_batch_scatters_fallbacks_to_their_own_queries(gpu, ladder):
    """every other query sits in a crowded cluster and fails the proof; the rest succeed: the exact kernel answers a strict,
    non-contiguous subset and each answer must land on its own query"""
    rng = np.random.default_rng(15)
    n, dim, nq, k = 8192, 64, 200, 10
    ds = rng.standard_normal((n, dim)).astype(np.float32)
    c = 4 * rng.standard_normal(dim)
    ds[3000:3600] = (c + 1e-4 * rng.standard_normal((600, dim))).astype(np.float32)
    qs = rng.standard_normal((nq, dim)).astype(np.float32)
    qs[1::2] = ds[rng.choice(3000, nq // 2, replace=False)]
    qs[0::2] = (c + 1e-4 * rng.standard_normal((nq // 2, dim))).astype(np.float32)
    keys, dists, kused, fallbacks = bf_search(gpu, ds, qs, k, L2, tc_ladder=ladder)
    S.check_exact_topk(keys, dists, ds, qs, k, L2)
    assert kused == expected_kused(dim, k, ladder) and 0 < fallbacks < nq, (kused, fallbacks)


# ---- IVF ------------------------------------------------------------------------------------------------------------------
def ivf_case(nlist, dim, sizes, nq, seed):
    """centroids, entries with list sizes `sizes` (-1: random), their assignment and queries next to random lists"""
    rng = np.random.default_rng(seed)
    centers = (4 * rng.standard_normal((nlist, dim))).astype(np.float32)
    sizes = [int(s) if s >= 0 else int(rng.integers(20, 400)) for s in sizes]
    assign = np.repeat(np.arange(nlist, dtype=np.int32), sizes)
    rng.shuffle(assign)
    data = (centers[assign] + rng.standard_normal((assign.size, dim))).astype(np.float32)
    ql = rng.integers(0, nlist, nq)
    qs = (centers[ql] + rng.standard_normal((nq, dim))).astype(np.float32)
    qs[:3] = data[[0, assign.size // 2, assign.size - 1]]
    return centers, data, assign, qs


def ivf_search(gpu, centers, data, assign, qs, k, nprobe, prepared=True, ladder=1, sqrt_out=False, **knobs):
    """IVF search on the tensor-core path: (keys, dists, stats) with stats = K columns of the list scan's first pass and of the
    centroid probe's pass (0: exact kernel), queries refined, queries that reached the exact kernel"""
    def run():
        idx = ops.IvfflatSearchIndex(data, assign, centers)
        try:
            if not prepared:
                gpu.MoB200_SearchRelease(idx.d_data.ptr)
                idx.prepared = False
            keys, dists = idx.search(qs, k, nprobe, sqrt_out)
            return keys, dists, {s: _stat(gpu, "get_tc_" + s) for s in ("kused", "probe_kused", "refined", "fallbacks")}
        finally:
            idx.destroy()
    return _with_knobs(gpu, dict(knobs, tc_ladder=ladder), run)


def ivf_check(centers, data, assign, qs, k, nprobe, keys, dists, sqrt_out=False):
    n, dim = data.shape
    nq, nlist = qs.shape[0], centers.shape[0]
    okeys = np.zeros(nq * k, dtype=np.int64); odists = np.zeros(nq * k)
    O.go().og_ivf_search_f32(O.p(data), O.p(assign), n, dim, O.p(centers), nlist, O.p(qs), nq, nprobe, k, 0, int(sqrt_out), 8,
                             O.p(okeys), O.p(odists))
    probes, _ = O.bruteforce(centers, qs, nprobe)
    probes = probes.reshape(nq, nprobe)
    allowed = [np.flatnonzero(np.isin(assign, probes[q])) for q in range(nq)]
    S.check_exact_topk(keys, dists, data, qs, k, L2, oracle=(okeys, odists), allowed=allowed, sqrt_out=sqrt_out)


@pytest.mark.parametrize("dim", [36, 72, 100])        # not a multiple of 8 (scalar split) / of 8 but not of 64 / neither
@pytest.mark.parametrize("ladder,prepared", [(1, True), (2, True), (2, False)])
def test_ivf_odd_dims_and_list_edges(gpu, dim, ladder, prepared):
    """lists of 3 (shorter than k), 128 and 129 rows next to random ones; nprobe 1 leaves some queries with fewer than k rows"""
    nlist, nq, k = 24, 300, 10
    sizes = [3, 128, 129] + [-1] * (nlist - 3)
    centers, data, assign, qs = ivf_case(nlist, dim, sizes, nq, seed=dim)
    qs[3:9] = centers[[0, 0, 1, 1, 2, 2]] + np.float32(0.5)
    for nprobe in (1, 3):
        keys, dists, st = ivf_search(gpu, centers, data, assign, qs, k, nprobe, prepared, ladder)
        ivf_check(centers, data, assign, qs, k, nprobe, keys, dists)
        assert st["kused"] == expected_kused(dim, k, ladder) and 0 <= st["fallbacks"] < nq, st
        assert st["probe_kused"] == 0, st      # 24 centroids: the probe runs on the exact kernel


def test_ivf_hi_only_pass_ignores_stale_scratch(gpu):
    """the one-term IVF pass reads whole 64-column k-blocks of the query operand; at dim 72 the columns past dim must be
    zero whatever an earlier call left in the scratch memory (here: a host dataset of 3e38 staged by a brute-force call)"""
    nlist, dim, nq, k, nprobe = 16, 72, 300, 10, 3
    centers, data, assign, qs = ivf_case(nlist, dim, [-1] * nlist, nq, seed=5)
    fill = np.full((60_000, dim), np.uint32(0x7F617F61), dtype=np.uint32).view(np.float32)   # every bf16 half ~3e38
    fk, fd = np.zeros(1, dtype=np.int64), np.zeros(1)
    p = ops._search_params(fill.shape[0], dim, 1, 1, L2)
    xcall(capi.XCALL_BRUTEFORCE_TOPK_F32, [Vector(data=fk, length=1), Vector(data=fd, length=1), Vector(data=fill.reshape(-1), length=fill.shape[0]),
                                           Vector(data=qs[:1].reshape(-1).copy(), length=1), ops._params_vec(p)], 1)
    keys, dists, st = ivf_search(gpu, centers, data, assign, qs, k, nprobe, True, 2)
    ivf_check(centers, data, assign, qs, k, nprobe, keys, dists)
    assert st["kused"] == 128 and st["refined"] <= nq // 10, st


@pytest.mark.parametrize("nprobe", [17, 32])
def test_ivf_wide_tensor_core_probe(gpu, nprobe):
    """nlist 1024 and nprobe 17-32: the centroid probe itself runs on the tensor cores in wide mode (k = nprobe > 16: the
    three-term pass over the whole K', get_tc_probe_kused)"""
    nlist, dim, nq, k = 1024, 64, 300, 10
    centers, data, assign, qs = ivf_case(nlist, dim, [24] * nlist, nq, seed=nprobe)
    keys, dists, st = ivf_search(gpu, centers, data, assign, qs, k, nprobe, True, 2, sqrt_out=True)
    ivf_check(centers, data, assign, qs, k, nprobe, keys, dists, sqrt_out=True)
    assert st["kused"] == expected_kused(dim, k, 2) and 0 <= st["fallbacks"] < nq, st
    assert st["probe_kused"] == S.kprime(dim), st


@pytest.mark.parametrize("prepared,no_share", [(True, 0), (True, 1), (False, 1)])
@pytest.mark.parametrize("dim", [1536, 3072])
def test_ivf_bf16_exact_rows_do_not_hide_the_nearest_neighbour(gpu, dim, prepared, no_share):
    """the IVF one-term pass prices its accumulation by its own k-blocks too (per-list bounds of the residual operands).
    List 0 has its centroid at the origin, so its residuals are the rows of hidden_neighbour_data; forty decoys fill the
    copy's list of 32 candidates.  List 1 lies far away.  nprobe 1, k 1."""
    ds0, qs = hidden_neighbour_data(dim, n=2048, ndecoy=40)
    rng = np.random.default_rng(dim)
    c1 = np.full(dim, 4.0 / np.sqrt(dim), dtype=np.float32)
    ds1 = c1 + np.float32(0.5) * _bf16_rows(rng, 256, dim, 0.98)
    data = np.concatenate([ds0, ds1]).astype(np.float32)
    assign = np.concatenate([np.zeros(len(ds0), np.int32), np.ones(len(ds1), np.int32)])
    centers = np.stack([np.zeros(dim, np.float32), c1])
    keys, dists, st = ivf_search(gpu, centers, data, assign, qs, 1, 1, prepared, 2, tc_share=no_share)
    ivf_check(centers, data, assign, qs, 1, 1, keys, dists)
    assert dists.reshape(-1)[:4].tolist() == [0.0] * 4
    assert st["kused"] == expected_kused(dim, 1, 2) and 0 <= st["fallbacks"] < qs.shape[0], st
