"""GPU parity of filtered search (MO_XCALL_BRUTEFORCE_TOPK_FILTERED_F32 / MO_XCALL_IVF_TOPK_FILTERED_F32): the answer is the
unfiltered search run over the admitted rows only, with the original keys.  The reference is the oracle's brute-force / IVF search
on the admitted subset (the IVF probes depend only on the centroids, so the subset has the same probes), subset ordinals mapped back
to keys; bloom admission comes from the reference's own bloom.c (oracle/_ref/libbloom_ref.so)."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as O
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer, Vector, xcall

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAXF32 = float(np.finfo(np.float32).max)
_vp, _u64, _u32, _sz = C.c_void_p, C.c_uint64, C.c_uint32, C.c_size_t


def _bloom_proto(lib):
    lib.bloomfilter_init_with_seed.restype = _vp; lib.bloomfilter_init_with_seed.argtypes = [_u64, _u32, _u64]
    lib.bloomfilter_free.restype = None; lib.bloomfilter_free.argtypes = [_vp]
    lib.bloomfilter_add_fixed.restype = None; lib.bloomfilter_add_fixed.argtypes = [_vp, _vp, _sz, _sz, _sz, _vp, _sz]
    lib.bloomfilter_test_fixed.restype = None; lib.bloomfilter_test_fixed.argtypes = [_vp, _vp, _sz, _sz, _sz, _vp, _sz, _vp]
    return lib


@pytest.fixture(scope="module")
def blooms(gpu):
    p = os.path.join(ROOT, "oracle", "_ref", "libbloom_ref.so")
    if not os.path.exists(p):
        pytest.skip("oracle/_ref/libbloom_ref.so not built")
    return _bloom_proto(capi.load_library()), _bloom_proto(C.CDLL(p))


@pytest.fixture(autouse=True)
def _knobs(gpu):
    yield
    for name in (b"search_mode", b"search_filter_path"):
        gpu.MoB200_SetTuning(name, 0)


def _set(gpu, mode, path):
    assert gpu.MoB200_SetTuning(b"search_mode", mode) == 0 and gpu.MoB200_SetTuning(b"search_filter_path", path) == 0


class Bloom:
    """the same small filter in the product and in the reference (about 4 bits per member: roughly one key in ten that is not a
    member passes too), so its false positives are part of the admitted set"""

    def __init__(self, blooms, members, k=3, seed=77):
        self.ours, self.ref = blooms
        nbits = max(64, 4 * len(members))
        self.a = self.ours.bloomfilter_init_with_seed(nbits, k, seed)
        self.b = self.ref.bloomfilter_init_with_seed(nbits, k, seed)
        self.add(members)

    def add(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        for lib, bf in ((self.ours, self.a), (self.ref, self.b)):
            lib.bloomfilter_add_fixed(bf, keys.ctypes.data, keys.nbytes, 8, keys.size, None, 0)

    def admits(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        r = np.zeros(keys.size, dtype=np.uint8)
        self.ref.bloomfilter_test_fixed(self.b, keys.ctypes.data, keys.nbytes, 8, keys.size, None, 0, r.ctypes.data)
        return r.astype(bool)

    def free(self):
        self.ours.bloomfilter_free(self.a); self.ref.bloomfilter_free(self.b)


def _bitmap(keys, nwords):
    w = np.zeros(nwords, dtype=np.uint64)
    keys = np.asarray(keys, dtype=np.int64)
    keys = keys[(keys >= 0) & (keys < 64 * nwords)]
    np.bitwise_or.at(w, keys >> 6, np.uint64(1) << (keys & 63).astype(np.uint64))
    return w


def _bitmap_admits(w, keys):
    keys = np.asarray(keys, dtype=np.int64)
    ok = (keys >= 0) & (keys < 64 * w.size)
    out = np.zeros(keys.size, dtype=bool)
    kk = keys[ok]
    out[ok] = ((w[kk >> 6] >> (kk & 63).astype(np.uint64)) & np.uint64(1)).astype(bool)
    return out


def _make_filter(kind, blooms, keys, rng, frac, eligible=None):
    """a filter over `keys` admitting about `frac` of them (members drawn from `eligible` only), and the admitted mask the reference
    derives from it"""
    pick = rng.random(keys.size) < frac
    members = keys[pick if eligible is None else pick & eligible]
    if kind == "bitmap":
        w = _bitmap(members, int(keys.max()) // 64 + 2)
        return w, _bitmap_admits(w, keys), None
    bl = Bloom(blooms, members)
    return bl.a, bl.admits(keys), bl


def _check(keys, dists, okeys, odists, nq, k):
    keys = keys.reshape(nq, k); dists = dists.reshape(nq, k); okeys = okeys.reshape(nq, k); odists = odists.reshape(nq, k)
    assert (dists == odists).all(), np.abs(dists - odists).max()
    for q in range(nq):
        for j in np.flatnonzero(keys[q] != okeys[q]):       # only where the distances tie
            assert (odists[q] == odists[q][j]).sum() > 1 and okeys[q][j] >= 0, (q, j)


def _ref_bf(ds, qs, k, metric, adm, key_base=0):
    rows = np.flatnonzero(adm)
    okeys, odists = O.bruteforce(np.ascontiguousarray(ds[rows]).reshape(-1, ds.shape[1]), qs, k, metric)
    okeys = np.where(okeys >= 0, rows[np.maximum(okeys, 0)] + key_base, -1)
    return okeys, odists


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("kind", ["bitmap", "bloom"])
@pytest.mark.parametrize("metric", [capi.METRIC_L2, capi.METRIC_L2SQ, capi.METRIC_IP, capi.METRIC_COS, capi.METRIC_L1])
def test_bruteforce_filtered_matches_subset(gpu, blooms, metric, kind, mode, path):
    _set(gpu, mode, path)
    for dim, k, prepared, frac in ((768, 10, True, 0.3), (100, 1, False, 0.6), (100, 64, True, 0.2), (96, 16, False, 0.05)):
        rng = np.random.default_rng(dim + k + metric)
        n, nq = 3000, 130
        ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
        key_base = 1000
        filt, adm, bl = _make_filter(kind, blooms, np.arange(n) + key_base, rng, frac)
        idx = ops.BruteForceIndex(ds, dim, metric, key_base=key_base)
        if not prepared and idx.prepared:
            gpu.MoB200_SearchRelease(idx.buf.ptr)
        keys, dists = idx.search(qs, k, filter=filt)
        assert gpu.MoB200_SetTuning(b"get_filter_admitted", 0) == adm.sum()
        assert gpu.MoB200_SetTuning(b"get_filter_compacted", 0) == (1 if path == 2 else 0)
        okeys, odists = _ref_bf(ds, qs, k, metric, adm, key_base)
        _check(keys, dists, okeys, odists, nq, k)
        idx.destroy()
        if bl:
            bl.free()


def _ivf_setup(dim, n=20_000, nlist=64, nq=150, seed=30):
    centers = datagen.vectors_f32(seed, 0, nlist, dim) * 4
    data = datagen.vectors_f32(seed + 1, 0, n, dim, centers, 1.0)
    qs = datagen.vectors_f32(seed + 2, 0, nq, dim, centers, 1.0)
    assign = np.zeros(n, dtype=np.int32)
    O.go().og_assign_centroids_f32(O.p(data), n, dim, O.p(centers), nlist, 0, O.p(assign))
    return centers, data, qs, assign


def _ref_ivf(data, assign, centers, qs, k, nprobe, metric, adm, sqrt_out=False):
    rows = np.flatnonzero(adm)
    sub = np.ascontiguousarray(data[rows]).reshape(-1, data.shape[1]); sa = np.ascontiguousarray(assign[rows])
    nq = qs.shape[0]
    okeys = np.zeros(nq * k, dtype=np.int64); odists = np.zeros(nq * k)
    O.go().og_ivf_search_f32(O.p(sub), O.p(sa), rows.size, data.shape[1], O.p(centers), centers.shape[0], O.p(qs), nq, nprobe, k, metric,
                             int(sqrt_out), 8, O.p(okeys), O.p(odists))
    return np.where(okeys >= 0, rows[np.maximum(okeys, 0)], -1), odists


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("kind", ["bitmap", "bloom"])
@pytest.mark.parametrize("dim,metric,k,sharded", [(96, capi.METRIC_L2, 10, False), (768, capi.METRIC_L2, 1, False),
                                                   (100, capi.METRIC_L2, 16, True), (96, capi.METRIC_COS, 10, False)])
def test_ivf_filtered_matches_subset(gpu, blooms, dim, metric, k, sharded, kind, mode, path):
    _set(gpu, mode, path)
    centers, data, qs, assign = _ivf_setup(dim)
    if sharded:                       # a list-sharded index: this shard holds the even lists only
        keep = assign % 2 == 0
        data, assign = np.ascontiguousarray(data[keep]), np.ascontiguousarray(assign[keep])
    rng = np.random.default_rng(dim + k)
    n = data.shape[0]
    # no member in every fifth list: with a bitmap those lists have no admitted row at all (a bloom filter lets a few through)
    filt, adm, bl = _make_filter(kind, blooms, np.arange(n), rng, 0.4, eligible=assign % 5 != 1)
    if kind == "bitmap":
        assert not adm[assign % 5 == 1].any()
    idx = ops.IvfflatSearchIndex(data, assign, centers, metric)
    for nprobe, sqrt_out in ((8, False), (3, True)):
        keys, dists = idx.search(qs, k, nprobe, sqrt_out, filter=filt)
        okeys, odists = _ref_ivf(data, assign, centers, qs, k, nprobe, metric, adm, sqrt_out)
        _check(keys, dists, okeys, odists, qs.shape[0], k)
    idx.destroy()
    if bl:
        bl.free()


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("mode", [1, 2])
def test_all_admitted_is_byte_identical_to_unfiltered(gpu, mode, path):
    _set(gpu, mode, path)
    rng = np.random.default_rng(5)
    n, dim, nq, k = 4000, 128, 300, 10
    ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
    idx = ops.BruteForceIndex(ds, dim, key_base=7)
    a = idx.search(qs, k)
    b = idx.search(qs, k, filter=np.full((n + 7) // 64 + 1, ~np.uint64(0), dtype=np.uint64))
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    idx.destroy()
    centers, data, qs, assign = _ivf_setup(96, n=10_000)
    ix = ops.IvfflatSearchIndex(data, assign, centers)
    a = ix.search(qs, k, 8)
    b = ix.search(qs, k, 8, filter=np.full(10_000 // 64 + 1, ~np.uint64(0), dtype=np.uint64))
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    ix.destroy()


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("mode", [1, 2])
def test_none_and_fewer_than_k_admitted(gpu, mode, path):
    _set(gpu, mode, path)
    rng = np.random.default_rng(9)
    n, dim, nq = 2048, 64, 200
    ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
    idx = ops.BruteForceIndex(ds, dim)
    none = np.zeros(n // 64, dtype=np.uint64)
    keys, dists = idx.search(qs, 1, filter=none)                  # k = 1, nothing admitted: brute_force.go:289-303
    assert (keys == -1).all() and (dists == MAXF32).all()
    keys, dists = idx.search(qs, 5, filter=none)
    assert (keys == -1).all() and (dists == 0).all()
    three = _bitmap([5, 700, 2047], n // 64)
    keys, dists = idx.search(qs, 5, filter=three)                 # front padding, then the three rows in order
    okeys, odists = _ref_bf(ds, qs, 5, capi.METRIC_L2, _bitmap_admits(three, np.arange(n)))
    k2 = keys.reshape(nq, 5)
    assert (k2[:, :2] == -1).all() and (dists.reshape(nq, 5)[:, :2] == 0).all()
    _check(keys, dists, okeys, odists, nq, 5)
    keys, dists = idx.search(qs, 1, filter=three)
    okeys, odists = _ref_bf(ds, qs, 1, capi.METRIC_L2, _bitmap_admits(three, np.arange(n)))
    _check(keys, dists, okeys, odists, nq, 1)
    idx.destroy()
    centers, data, qs, assign = _ivf_setup(96, n=10_000)
    ix = ops.IvfflatSearchIndex(data, assign, centers)
    keys, dists = ix.search(qs, 1, 8, filter=np.zeros(4, dtype=np.uint64))
    assert (keys == -1).all() and (dists == 0).all()           # IVF pads with distance 0
    few = _bitmap(np.arange(0, 10_000, 997), 10_000 // 64 + 1)
    keys, dists = ix.search(qs, 10, 8, filter=few)
    okeys, odists = _ref_ivf(data, assign, centers, qs, 10, 8, capi.METRIC_L2, _bitmap_admits(few, np.arange(10_000)))
    _check(keys, dists, okeys, odists, qs.shape[0], 10)
    ix.destroy()


@pytest.mark.parametrize("path", [1, 2])
def test_bitmap_length_and_pointer_kinds(gpu, path):
    _set(gpu, 0, path)
    rng = np.random.default_rng(11)
    n, dim, nq, k = 1000, 32, 20, 8
    ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
    idx = ops.BruteForceIndex(ds, dim)
    w = np.full(4, ~np.uint64(0), dtype=np.uint64)                  # keys 0..255 set; every key >= 256 is past the bitmap
    keys, dists = idx.search(qs, k, filter=w)
    assert keys.max() < 256
    okeys, odists = _ref_bf(ds, qs, k, capi.METRIC_L2, np.arange(n) < 256)
    _check(keys, dists, okeys, odists, nq, k)
    dw = DeviceBuffer.from_numpy(w)                                  # the same words as a device pointer
    dk, dd = idx.search(qs, k, filter=dw)
    assert dk.tobytes() == keys.tobytes() and dd.tobytes() == dists.tobytes()
    dw.free()
    keys, dists = idx.search(qs, k, filter=np.zeros(0, dtype=np.uint64))   # no words: nothing admitted
    assert (keys == -1).all()
    idx.destroy()


@pytest.mark.parametrize("path", [1, 2])
def test_bloom_bits_added_on_the_device_are_searched(gpu, blooms, path):
    _set(gpu, 0, path)
    rng = np.random.default_rng(12)
    n, dim, nq, k = 3000, 64, 40, 10
    ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
    idx = ops.BruteForceIndex(ds, dim)
    bl = Bloom(blooms, np.arange(0, n, 50))
    keys, dists = idx.search(qs, k, filter=bl.a)                     # the mirror exists from here on
    okeys, odists = _ref_bf(ds, qs, k, capi.METRIC_L2, bl.admits(np.arange(n)))
    _check(keys, dists, okeys, odists, nq, k)
    bl.add(np.arange(7, n, 13))                                      # bloomfilter_add_fixed writes the device mirror
    keys, dists = idx.search(qs, k, filter=bl.a)
    okeys, odists = _ref_bf(ds, qs, k, capi.METRIC_L2, bl.admits(np.arange(n)))
    _check(keys, dists, okeys, odists, nq, k)
    bl.free()
    idx.destroy()


def test_bruteforce_shards_merge_to_the_whole(gpu):
    rng = np.random.default_rng(13)
    n, dim, nq, k = 6000, 128, 300, 10
    ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
    w = _bitmap(np.flatnonzero(rng.random(n) < 0.3), n // 64 + 1)
    whole = ops.BruteForceIndex(ds, dim)
    gk, gd = whole.search(qs, k, filter=w)
    whole.destroy()
    a = ops.BruteForceIndex(ds[:2500], dim); ak, ad = a.search(qs, k, filter=w); a.destroy()
    b = ops.BruteForceIndex(ds[2500:], dim, key_base=2500); bk, bd = b.search(qs, k, filter=w); b.destroy()
    mk, md = ops.topk_merge(np.stack([ak, bk]), np.stack([ad, bd]), nq, k)
    assert mk.tobytes() == gk.tobytes() and md.tobytes() == gd.tobytes()


def test_auto_path_follows_the_admitted_count(gpu):
    _set(gpu, 0, 0)
    rng = np.random.default_rng(14)
    n, dim, nq, k = 20_000, 64, 256, 10
    ds = rng.standard_normal((n, dim)).astype(np.float32); qs = rng.standard_normal((nq, dim)).astype(np.float32)
    idx = ops.BruteForceIndex(ds, dim)
    idx.search(qs, k, filter=_bitmap(np.arange(0, n, 1000), n // 64 + 1))
    assert gpu.MoB200_SetTuning(b"get_filter_admitted", 0) == 20 and gpu.MoB200_SetTuning(b"get_filter_compacted", 0) == 1
    idx.search(qs, k, filter=np.full(n // 64 + 1, ~np.uint64(0), dtype=np.uint64))
    assert gpu.MoB200_SetTuning(b"get_filter_admitted", 0) == n and gpu.MoB200_SetTuning(b"get_filter_compacted", 0) == 0
    idx.search(qs, k)
    assert gpu.MoB200_SetTuning(b"get_filter_admitted", 0) == -1
    idx.destroy()
    centers, data, qs, assign = _ivf_setup(64, n=20_000)
    ix = ops.IvfflatSearchIndex(data, assign, centers)
    ix.search(qs, k, 8, filter=_bitmap(np.arange(0, 20_000, 100), 20_000 // 64 + 1))
    assert gpu.MoB200_SetTuning(b"get_filter_compacted", 0) == 1
    ix.search(qs, k, 8, filter=_bitmap(np.arange(20_000), 20_000 // 64 + 1))
    assert gpu.MoB200_SetTuning(b"get_filter_compacted", 0) == 0
    ix.destroy()


def test_malformed_descriptors_are_rejected(gpu):
    rng = np.random.default_rng(15)
    ds = rng.standard_normal((300, 16)).astype(np.float32); qs = rng.standard_normal((4, 16)).astype(np.float32)
    w = np.ones(8, dtype=np.uint64)
    dbuf = DeviceBuffer.from_numpy(ds)
    p = ops._search_params(300, 16, 4, 3, capi.METRIC_L2)
    keys = np.zeros(12, dtype=np.int64); dists = np.zeros(12)

    def run(desc_bytes):
        fv = Vector(data=np.frombuffer(desc_bytes, dtype=np.uint8).copy(), length=1, const=True)
        return xcall(capi.XCALL_BRUTEFORCE_TOPK_FILTERED_F32, [Vector(data=keys, length=4), Vector(data=dists, length=4),
                     Vector(data_ptr=dbuf.ptr, data_nbytes=dbuf.nbytes, length=300), Vector(data=qs.reshape(-1), length=4),
                     ops._params_vec(p), fv], 4, raise_on_error=False)[0]

    assert run(bytes(capi.SearchFilter(capi.SEARCH_FILTER_KEY_BITMAP, 0, w.ctypes.data, w.size))) == 0
    assert run(bytes(capi.SearchFilter(7, 0, w.ctypes.data, w.size))) == capi.RC_INVALID_ARGUMENT
    assert run(bytes(capi.SearchFilter(capi.SEARCH_FILTER_KEY_BLOOM, 0, None, 0))) == capi.RC_INVALID_ARGUMENT
    assert run(bytes(capi.SearchFilter(capi.SEARCH_FILTER_KEY_BITMAP, 0, None, 8))) == capi.RC_INVALID_ARGUMENT
    assert run(bytes(capi.SearchFilter(capi.SEARCH_FILTER_KEY_BITMAP, 0, w.ctypes.data, w.size))[:12]) == capi.RC_INVALID_ARGUMENT
    junk = np.zeros(64, dtype=np.uint8)                              # not a bloom filter (no magic)
    assert run(bytes(capi.SearchFilter(capi.SEARCH_FILTER_KEY_BLOOM, 0, junk.ctypes.data, 0))) == capi.RC_INVALID_ARGUMENT
    dbuf.free()
