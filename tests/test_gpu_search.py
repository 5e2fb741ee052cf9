"""GPU parity: brute-force top-k, IVF-flat probe and top-k merge against the oracle restatement of
GoBruteForceIndex.Search / IvfflatSearchIndex.Search.  Distances bit-exact; keys equal wherever the oracle's distances
are not tied."""
import numpy as np
import pytest

import oracle_lib as O
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer

pytestmark = pytest.mark.gpu


def _check_topk(keys, dists, okeys, odists, nq, k):
    keys = keys.reshape(nq, k); dists = dists.reshape(nq, k); okeys = okeys.reshape(nq, k); odists = odists.reshape(nq, k)
    assert (dists == odists).all(), np.abs(dists - odists).max()          # bit-exact distances, ascending
    for q in range(nq):
        same = keys[q] == okeys[q]
        if not same.all():            # only allowed where distances tie
            for j in np.flatnonzero(~same):
                assert (odists[q] == odists[q][j]).sum() > 1, (q, j)


@pytest.mark.parametrize("n,dim,nq,k", [(1000, 16, 7, 1), (1000, 16, 7, 5), (1000, 16, 7, 50), (5000, 128, 130, 10),
                                        (777, 768, 65, 10), (3000, 100, 3, 64), (64, 8, 1, 10), (100, 30, 5, 3), (200, 7, 9, 4)])
@pytest.mark.parametrize("metric", [capi.METRIC_L2, capi.METRIC_IP, capi.METRIC_COS, capi.METRIC_L1])
def test_bruteforce_topk_matches_oracle(gpu, n, dim, nq, k, metric):
    rng = np.random.default_rng(n + dim + k)
    ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
    idx = ops.BruteForceIndex(ds, dim, metric)
    keys, dists = idx.search(qs, k)
    okeys, odists = O.bruteforce(ds, qs, k, metric)
    _check_topk(keys, dists, okeys, odists, nq, k)
    idx.destroy()


def test_self_match_exact_zero_and_front_padding(gpu):
    """brute_force_test.go:76-146 (key == i, distance == 0.0) and brute_force.go:319-331 (front padding with -1 / 0)"""
    ds = datagen.vectors_f32(20, 0, 10_000, 128)
    idx = ops.BruteForceIndex(ds, 128)
    keys, dists = idx.search(ds[:2000], 3)
    keys = keys.reshape(-1, 3); dists = dists.reshape(-1, 3)
    assert (keys[:, 0] == np.arange(2000)).all() and (dists[:, 0] == 0.0).all() and (np.diff(dists, axis=1) >= 0).all()
    idx.destroy()
    small = ops.BruteForceIndex(ds[:2], 128)
    keys, dists = small.search(ds[:1], 5)
    assert list(keys[:3]) == [-1, -1, -1] and list(dists[:3]) == [0.0, 0.0, 0.0] and keys[3] == 0 and dists[3] == 0.0
    assert small.search(ds[:1], 0)[0].size == 0
    with pytest.raises(capi.MoError):
        small.search(ds[:1], 65)           # beyond the fused kernel's k limit: loud error, no fallback
    small.destroy()


def test_ties_resolve_to_lower_row_id(gpu):
    ds = np.zeros((300, 8), dtype=np.float32); ds[:, 0] = np.arange(300) % 3      # many exact ties
    idx = ops.BruteForceIndex(ds, 8)
    keys, dists = idx.search(np.zeros((1, 8), dtype=np.float32), 10)
    assert list(keys) == [0, 3, 6, 9, 12, 15, 18, 21, 24, 27] and (dists == 0).all()
    okeys, odists = O.bruteforce(ds, np.zeros((1, 8), dtype=np.float32), 10)
    assert (odists == dists).all()
    idx.destroy()


def test_topk_merge_of_shards_equals_global(gpu):
    """dataset sharded by rows (the multi-GPU layout): per-shard top-k + merge == global top-k"""
    rng = np.random.default_rng(12)
    n, dim, nq, k = 6000, 64, 50, 10
    ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
    gk, gd = O.bruteforce(ds, qs, k)
    sk, sd = [], []
    for s in range(4):
        lo, hi = s * 1500, (s + 1) * 1500
        idx = ops.BruteForceIndex(ds[lo:hi], dim, key_base=lo)
        a, b = idx.search(qs, k)
        sk.append(a); sd.append(b); idx.destroy()
    mk, md = ops.topk_merge(np.stack(sk), np.stack(sd), nq, k)
    _check_topk(mk, md, gk, gd, nq, k)
    # a shard with fewer than k rows contributes front-padded lists; the merge must skip the padding
    idx = ops.BruteForceIndex(ds[:4], dim); a, b = idx.search(qs, k); idx.destroy()
    idx = ops.BruteForceIndex(ds[4:n], dim, key_base=4); c, d = idx.search(qs, k); idx.destroy()
    mk, md = ops.topk_merge(np.stack([a, c]), np.stack([b, d]), nq, k)
    _check_topk(mk, md, gk, gd, nq, k)


@pytest.mark.parametrize("metric,sqrt_out", [(capi.METRIC_L2, False), (capi.METRIC_L2, True), (capi.METRIC_IP, False), (capi.METRIC_COS, False)])
def test_ivf_probe_matches_oracle(gpu, metric, sqrt_out):
    nlist, dim, n, nq, k, nprobe = 64, 96, 20_000, 150, 10, 8
    centers = datagen.vectors_f32(30, 0, nlist, dim) * 4
    data = datagen.vectors_f32(31, 0, n, dim, centers, 1.0)
    qs = datagen.vectors_f32(32, 0, nq, dim, centers, 1.0)
    assign = np.zeros(n, dtype=np.int32)
    O.go().og_assign_centroids_f32(O.p(data), n, dim, O.p(centers), nlist, metric, O.p(assign))
    okeys = np.zeros(nq * k, dtype=np.int64); odists = np.zeros(nq * k)
    O.go().og_ivf_search_f32(O.p(data), O.p(assign), n, dim, O.p(centers), nlist, O.p(qs), nq, nprobe, k, metric, int(sqrt_out), 8, O.p(okeys), O.p(odists))
    idx = ops.IvfflatSearchIndex(data, assign, centers, metric)
    keys, dists = idx.search(qs, k, nprobe, sqrt_out)
    _check_topk(keys, dists, okeys, odists, nq, k)
    # nprobe == nlist degenerates to brute force
    keys, dists = idx.search(qs[:10], k, nlist, sqrt_out)
    bk, bd = O.bruteforce(data, qs[:10], k, metric)
    if sqrt_out:
        bd = np.sqrt(bd)
    _check_topk(keys, dists, bk, bd, 10, k)
    idx.destroy()


def test_ivf_empty_lists_and_small_index(gpu):
    dim = 16
    centers = np.eye(8, dim, dtype=np.float32) * 10
    centers[np.arange(8), (np.arange(8) + 1) % dim] = 0.37 * np.arange(8, dtype=np.float32)    # break centroid-distance ties
    data =np.repeat(centers[:2], 3, axis=0) + 0.01 * np.arange(6, dtype=np.float32)[:, None]      # only lists 0 and 1 have rows
    assign = np.asarray([0, 0, 0, 1, 1, 1], dtype=np.int32)
    idx = ops.IvfflatSearchIndex(data, assign, centers)
    qs = centers[[0, 5]]
    keys, dists = idx.search(qs, 4, 2)
    okeys = np.zeros(8, dtype=np.int64); odists = np.zeros(8)
    O.go().og_ivf_search_f32(O.p(data), O.p(assign), 6, dim, O.p(centers), 8, O.p(qs), 2, 2, 4, 0, 0, 1, O.p(okeys), O.p(odists))
    assert (dists == odists).all() and (keys == okeys).all()
    idx.destroy()


@pytest.mark.parametrize("n,dim,nq,k", [(20_000, 128, 300, 10), (9_000, 768, 257, 10), (5_000, 100, 130, 5), (70_000, 64, 1000, 16), (300, 32, 40, 3),
                                        (20_000, 96, 200, 32), (1_024, 64, 500, 25)])   # k > 16: the wide mode of centroid probes
@pytest.mark.parametrize("pair", [1, 2])   # 1: single-CTA units (128 queries), 2: CTA pairs (a cluster of two sharing the row tile, 256 queries)
@pytest.mark.parametrize("ladder", [1, 2])  # 1: three-term product only, 2: hi-only level first, then three-term for the unproven
def test_tensor_core_candidate_path_is_exact(gpu, n, dim, nq, k, pair, ladder):
    """tensor-core (wgmma) candidate generation + exact re-scoring + completeness proof (csrc/tcsearch.cu): the results must be the exact
    answer (bit-exact distances), and the tensor path itself must be doing the work (few proof failures -> few fallbacks)."""
    ds = datagen.vectors_f32(40, 0, n, dim); qs = datagen.vectors_f32(41, 0, nq, dim)
    qs[:7] = ds[[0, 5, n // 2, n - 1, 17, 100, 255]]          # self matches: exact distance 0
    okeys, odists = O.bruteforce(ds, qs, k)
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        gpu.MoB200_SetTuning(b"tc_pair", pair)
        gpu.MoB200_SetTuning(b"tc_ladder", ladder)
        idx = ops.BruteForceIndex(ds, dim)
        keys, dists = idx.search(qs, k)
        fallbacks = gpu.MoB200_SetTuning(b"get_tc_fallbacks", 0)
        idx.destroy()
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
        gpu.MoB200_SetTuning(b"tc_pair", 0)
        gpu.MoB200_SetTuning(b"tc_ladder", 0)
    _check_topk(keys, dists, okeys, odists, nq, k)
    assert dists.reshape(nq, k)[:7, 0].tolist() == [0.0] * 7
    assert 0 <= fallbacks <= max(2, nq // 20), fallbacks


def test_tensor_core_path_near_ties_fall_back_to_exact(gpu):
    """many exactly tied rows defeat the completeness proof: those queries are re-run on the exact kernel, results stay exact"""
    n, dim, nq, k = 4096, 64, 256, 10
    ds = np.zeros((n, dim), dtype=np.float32); ds[:, 0] = np.arange(n) % 7
    qs = np.zeros((nq, dim), dtype=np.float32); qs[:, 1] = np.arange(nq) % 3
    okeys, odists = O.bruteforce(ds, qs, k)
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        idx = ops.BruteForceIndex(ds, dim)
        keys, dists = idx.search(qs, k)
        fallbacks = gpu.MoB200_SetTuning(b"get_tc_fallbacks", 0)
        idx.destroy()
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
    assert (dists == odists).all() and fallbacks > 0


def test_tensor_core_path_non_finite_inputs_use_exact_kernel(gpu):
    n, dim, nq, k = 4096, 64, 256, 5
    ds = datagen.vectors_f32(42, 0, n, dim); qs = datagen.vectors_f32(43, 0, nq, dim)
    ds[77, 3] = np.inf
    okeys, odists = O.bruteforce(ds, qs, k)
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        idx = ops.BruteForceIndex(ds, dim)
        keys, dists = idx.search(qs, k)
        assert gpu.MoB200_SetTuning(b"get_tc_fallbacks", 0) == nq
        idx.destroy()
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
    _check_topk(keys, dists, okeys, odists, nq, k)


@pytest.mark.parametrize("sqrt_out", [False, True])
@pytest.mark.parametrize("nlist,dim,n,nq,k,nprobe", [(64, 96, 20_000, 150, 10, 8), (32, 768, 6_000, 300, 10, 32), (16, 100, 3_000, 64, 5, 3),
                                                    (1024, 64, 30_000, 300, 10, 32), (300, 64, 9_000, 200, 4, 9)])   # probe itself on the tensor cores
@pytest.mark.parametrize("ladder,prepared", [(1, True), (2, True), (2, False)])   # three-term only / one-term level first; operand split at load or per call
def test_ivf_tensor_core_scan_is_exact(gpu, nlist, dim, n, nq, k, nprobe, sqrt_out, ladder, prepared):
    """IVF list scan through the tcgen05 candidate kernel ((list, query-tile) units over gathered split operands): exact results"""
    centers = datagen.vectors_f32(30, 0, nlist, dim) * 4
    data = datagen.vectors_f32(31, 0, n, dim, centers, 1.0)
    qs = datagen.vectors_f32(32, 0, nq, dim, centers, 1.0)
    qs[:5] = data[[0, 7, n // 3, n - 1, 99]]
    assign = np.zeros(n, dtype=np.int32)
    O.go().og_assign_centroids_f32(O.p(data), n, dim, O.p(centers), nlist, 0, O.p(assign))
    okeys = np.zeros(nq * k, dtype=np.int64); odists = np.zeros(nq * k)
    O.go().og_ivf_search_f32(O.p(data), O.p(assign), n, dim, O.p(centers), nlist, O.p(qs), nq, nprobe, k, 0, int(sqrt_out), 8, O.p(okeys), O.p(odists))
    idx = ops.IvfflatSearchIndex(data, assign, centers)
    if not prepared:
        gpu.MoB200_SearchRelease(idx.d_data.ptr)
        idx.prepared = False
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        gpu.MoB200_SetTuning(b"tc_ladder", ladder)
        keys, dists = idx.search(qs, k, nprobe, sqrt_out)
        fallbacks = gpu.MoB200_SetTuning(b"get_tc_fallbacks", 0)
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
        gpu.MoB200_SetTuning(b"tc_ladder", 0)
        idx.destroy()
    _check_topk(keys, dists, okeys, odists, nq, k)
    assert dists.reshape(nq, k)[:5, 0].tolist() == [0.0] * 5
    assert 0 <= fallbacks <= max(3, nq // 10), fallbacks


@pytest.mark.gpu
def test_ivf_refine_pass_resolves_crowded_lists(gpu):
    """40 near-duplicates of the query inside one list: the whole-list pass keeps 16 candidates per (query, list) and cannot prove the
    top-k complete; the sub-range refine pass (still on the tensor cores) can, and the answer equals the oracle's"""
    nlist, dim, n, nq, k, nprobe = 4, 64, 8_000, 40, 16, 4
    centers = datagen.vectors_f32(40, 0, nlist, dim) * 4
    data = datagen.vectors_f32(41, 0, n, dim, centers, 1.0)
    rng = np.random.default_rng(5)
    base = data[123].copy()
    dup_rows = np.arange(200, 200 + 40 * 150, 150)
    data[dup_rows] = base + (rng.standard_normal((40, dim)) * 1e-4).astype(np.float32)
    qs = datagen.vectors_f32(42, 0, nq, dim, centers, 1.0)
    qs[0] = base
    assign = np.zeros(n, dtype=np.int32)
    O.go().og_assign_centroids_f32(O.p(data), n, dim, O.p(centers), nlist, 0, O.p(assign))
    okeys = np.zeros(nq * k, dtype=np.int64); odists = np.zeros(nq * k)
    O.go().og_ivf_search_f32(O.p(data), O.p(assign), n, dim, O.p(centers), nlist, O.p(qs), nq, nprobe, k, 0, 0, 8, O.p(okeys), O.p(odists))
    idx = ops.IvfflatSearchIndex(data, assign, centers)
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        keys, dists = idx.search(qs, k, nprobe, False)
        refined = gpu.MoB200_SetTuning(b"get_tc_refined", 0)
        fallbacks = gpu.MoB200_SetTuning(b"get_tc_fallbacks", 0)
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
        idx.destroy()
    _check_topk(keys, dists, okeys, odists, nq, k)
    assert refined >= 1, refined
    assert fallbacks <= refined


def test_search_statistics_describe_only_the_last_search(gpu):
    """get_tc_* after a brute-force search on the exact kernel describe that search, not the IVF search before it, whose centroid
    probe and list scan ran on the tensor cores"""
    nlist, dim, n, nq, k, nprobe = 300, 64, 9_000, 200, 4, 9
    centers = datagen.vectors_f32(30, 0, nlist, dim) * 4
    data = datagen.vectors_f32(31, 0, n, dim, centers, 1.0)
    qs = datagen.vectors_f32(32, 0, nq, dim, centers, 1.0)
    ivf = ops.IvfflatSearchIndex(data, np.arange(n) % nlist, centers)
    bf = ops.BruteForceIndex(data[:1000], dim)
    stats = lambda: tuple(gpu.MoB200_SetTuning(b"get_tc_" + s, 0) for s in (b"kused", b"probe_kused", b"refined", b"fallbacks"))
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        ivf.search(qs, k, nprobe)
        kused, probe_kused, refined, fallbacks = stats()
        assert kused > 0 and probe_kused > 0 and refined >= 0 and fallbacks >= 0, stats()
        gpu.MoB200_SetTuning(b"search_mode", 1)
        bf.search(qs, k)
        assert stats() == (0, 0, -1, -1)
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
        ivf.destroy(); bf.destroy()


@pytest.mark.gpu
def test_prepared_operand_is_dropped_when_the_dataset_is_overwritten(gpu):
    """MoB200_SearchPrepare caches the split operand of a resident dataset; a library write into that buffer (Upload) must
    invalidate it, so the next search sees the new rows"""
    n, dim, nq, k = 20_000, 64, 300, 5
    ds1 = datagen.vectors_f32(50, 0, n, dim); ds2 = datagen.vectors_f32(51, 0, n, dim)
    qs = datagen.vectors_f32(52, 0, nq, dim)
    idx = ops.BruteForceIndex(ds1, dim)
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        k1, d1 = idx.search(qs, k)
        ok1, od1 = O.bruteforce(ds1, qs, k)
        _check_topk(k1, d1, ok1, od1, nq, k)
        capi.check(gpu.MoB200_Upload(idx.buf.ptr, ds2.ctypes.data, ds2.nbytes), gpu)
        k2, d2 = idx.search(qs, k)
        ok2, od2 = O.bruteforce(ds2, qs, k)
        _check_topk(k2, d2, ok2, od2, nq, k)
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
        idx.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("n,dim,nq,k", [(20_000, 128, 300, 10), (9_000, 768, 257, 10), (70_000, 64, 1000, 16)])
@pytest.mark.parametrize("metric", [capi.METRIC_IP, capi.METRIC_COS])
@pytest.mark.parametrize("ladder", [1, 2])
def test_tensor_core_path_inner_product_and_cosine_are_exact(gpu, n, dim, nq, k, metric, ladder):
    """inner product (no norms in the epilogue) and cosine (operands normalised at split time: 1 - cos = |q^ - x^|^2 / 2) go through the
    same candidate kernel; re-scoring uses the Go-order inner product / cosine distance, so results equal the exact kernel's"""
    ds = datagen.vectors_f32(60, 0, n, dim); qs = datagen.vectors_f32(61, 0, nq, dim)
    ds[11] *= 3.0; ds[12] *= 0.25          # different lengths: inner product and cosine disagree about the order
    qs[:3] = ds[[0, 5, n // 2]]
    okeys, odists = O.bruteforce(ds, qs, k, metric)
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        gpu.MoB200_SetTuning(b"tc_ladder", ladder)
        idx = ops.BruteForceIndex(ds, dim, metric)
        keys, dists = idx.search(qs, k)
        fallbacks = gpu.MoB200_SetTuning(b"get_tc_fallbacks", 0)
        idx.destroy()
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
        gpu.MoB200_SetTuning(b"tc_ladder", 0)
    _check_topk(keys, dists, okeys, odists, nq, k)
    assert 0 <= fallbacks <= max(8, nq // 5), fallbacks


@pytest.mark.gpu
def test_tensor_core_cosine_with_a_zero_vector_uses_the_exact_kernel(gpu):
    n, dim, nq, k = 5_000, 64, 64, 4
    ds = datagen.vectors_f32(62, 0, n, dim); qs = datagen.vectors_f32(63, 0, nq, dim)
    ds[100] = 0.0                           # cosine distance to a zero vector is 1 by the Go rule; it cannot be normalised
    okeys, odists = O.bruteforce(ds, qs, k, capi.METRIC_COS)
    try:
        gpu.MoB200_SetTuning(b"search_mode", 2)
        idx = ops.BruteForceIndex(ds, dim, capi.METRIC_COS)
        keys, dists = idx.search(qs, k)
        assert gpu.MoB200_SetTuning(b"get_tc_fallbacks", 0) == nq
        idx.destroy()
    finally:
        gpu.MoB200_SetTuning(b"search_mode", 0)
    _check_topk(keys, dists, okeys, odists, nq, k)


@pytest.mark.parametrize("nlist,dim,n", [(64, 96, 20_000), (1024, 64, 70_000)])
def test_index_build_centroid_assignment_matches_productl2_oracle(gpu, nlist, dim, n):
    """IvfflatSearchIndex.build == Productl2.probeRun (pkg/sql/colexec/productl2/product_l2.go:317-407): every entry goes to its nearest
    centroid, brute-force Search(limit = 1).  The second shape (nlist >= 1024, >= 65536 entries per call) takes the tensor-core candidate
    pass + exact re-score; the first the exact kernel.  Equal only up to ties in the float64 distance."""
    centers = datagen.vectors_f32(40, 0, nlist, dim) * 4
    data = datagen.vectors_f32(41, 0, n, dim, centers, 1.0)
    want = np.zeros(n, dtype=np.int32)
    O.go().og_assign_centroids_f32(O.p(data), n, dim, O.p(centers), nlist, capi.METRIC_L2, O.p(want))
    dev = DeviceBuffer.from_numpy(data)
    idx = ops.IvfflatSearchIndex.build(dev, n, centers, capi.METRIC_L2, chunk=n)
    got = np.empty(n, dtype=np.int32)
    got[idx.row_ids] = np.repeat(np.arange(nlist, dtype=np.int32), np.diff(idx.offsets))
    bad = np.nonzero(got != want)[0]
    for i in bad:   # a differing assignment must be an exact tie
        d = ((data[i].astype(np.float64) - centers[[got[i], want[i]]].astype(np.float64)) ** 2).sum(axis=1)
        assert abs(d[0] - d[1]) <= 1e-6 * max(d[0], 1.0), (i, got[i], want[i], d)
    assert bad.size <= n // 1000
    idx.destroy(); dev.free()
