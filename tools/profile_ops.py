"""Resident-column timings of the operator kernels that have no bench.py workload of their own (generic fused plan, filter->sels, Shrink,
first-seen group ids, grouped aggregates, decimal SUM): CUDA-event kernel time through MoB200_LastKernelMs, GB/s of ALGORITHMIC bytes.
    python tools/profile_ops.py [rows] > ops.json"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from matrixone_b200 import capi, datagen, ops  # noqa: E402
from matrixone_b200.vector import DeviceBuffer, Vector, xcall  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000_000
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    kms = C.c_float()
    out = {"rows": n}

    def timed(fn, reps=5):
        ts = []
        for _ in range(reps + 1):
            fn()
            capi.check(lib.MoB200_LastKernelMs(C.byref(kms)), lib)
            ts.append(kms.value)
        return float(np.median(ts[1:]))

    names = ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")
    size = {"shipdate": 4, "returnflag": 1, "linestatus": 1}
    bufs = {k: DeviceBuffer(size.get(k, 8) * n, lib) for k in names}
    capi.check(lib.MoB200_GenLineitem(10, 0, n, *[bufs[k].ptr for k in names]), lib)
    # ---- generic fused plan: Q6 and Q1 shapes, device-resident result
    lib.MoB200_SetTuning(b"plan_specialise", 0)      # time the generic interpreter (the recognised shapes would dispatch to the specialised kernels)
    p6 = ops.q6_plan(); r6 = DeviceBuffer(p6.result_bytes(4), lib)
    ms = timed(lambda: p6.run([bufs["shipdate"], bufs["discount"], bufs["quantity"], bufs["extendedprice"]], n, max_groups=4, out_ptr=r6.ptr))
    out["plan_q6"] = {"ms": ms, "gbs": 28.0 * n / ms / 1e6, "rows_per_s": n / ms * 1e3}
    p1 = ops.q1_plan(datagen.Q1_CUTOFF); r1 = DeviceBuffer(p1.result_bytes(16), lib)
    ms = timed(lambda: p1.run([bufs[k] for k in names], n, max_groups=16, out_ptr=r1.ptr))
    out["plan_q1"] = {"ms": ms, "gbs": 38.0 * n / ms / 1e6, "rows_per_s": n / ms * 1e3}
    lib.MoB200_SetTuning(b"plan_specialise", 1)
    ms = timed(lambda: p6.run([bufs["shipdate"], bufs["discount"], bufs["quantity"], bufs["extendedprice"]], n, max_groups=4, out_ptr=r6.ptr))
    out["plan_q6_recognised_shape"] = {"ms": ms, "gbs": 28.0 * n / ms / 1e6}
    ms = timed(lambda: p1.run([bufs[k] for k in names], n, max_groups=16, out_ptr=r1.ptr))
    out["plan_q1_recognised_shape"] = {"ms": ms, "gbs": 38.0 * n / ms / 1e6}
    if os.environ.get("MOB_PROFILE_ONLY") == "plan":
        print(json.dumps(out)); return
    spec6 = DeviceBuffer(16, lib)
    ms = timed(lambda: ops.q6_filter_sum_device(bufs["shipdate"], bufs["discount"], bufs["quantity"], bufs["extendedprice"], n, *datagen.q6_params(), out_ptr=spec6.ptr))
    out["q6_specialised"] = {"ms": ms, "gbs": 28.0 * n / ms / 1e6}
    # ---- compare -> sels -> Shrink on one column
    dr = DeviceBuffer(n, lib); drn = DeviceBuffer(((n + 63) // 64) * 8, lib)
    capi.check(lib.MoB200_Memset(drn.ptr, 0, drn.nbytes), lib)
    cut = np.asarray([datagen.DATE_1995_01_01], dtype=np.int32)
    cmpv = [Vector(data_ptr=dr.ptr, data_nbytes=n, nulls_ptr=drn.ptr, length=n), Vector(data_ptr=bufs["shipdate"].ptr, data_nbytes=4 * n, length=n), Vector(data=cut, length=n)]
    ms = timed(lambda: xcall(capi.XCALL_GO_COMPARE(4, capi.T_DATE), cmpv, n))
    out["go_compare_date_lt"] = {"ms": ms, "gbs": (5.0 + 0.125) * n / ms / 1e6}
    dsels = DeviceBuffer(8 * n, lib); dcnt = DeviceBuffer(8, lib)
    ms = timed(lambda: ops.filter_sels_device(dr, drn, n, dsels.ptr, dcnt.ptr))
    k = int(dcnt.to_numpy(np.int64)[0])
    out["filter_sels"] = {"ms": ms, "selected": k, "gbs": (1.125 * n + 8.0 * k) / ms / 1e6}
    dst = DeviceBuffer(8 * k, lib)
    shv = [Vector(data_ptr=dst.ptr, data_nbytes=8 * k, length=k), Vector(data_ptr=bufs["quantity"].ptr, data_nbytes=8 * n, length=n), Vector(data_ptr=dsels.ptr, data_nbytes=8 * k, length=k)]
    ms = timed(lambda: xcall(capi.XCALL_SHUFFLE(8), shv, k))
    out["shuffle_f64"] = {"ms": ms, "gbs": 24.0 * k / ms / 1e6}
    dsels.free(); dst.free(); dr.free(); drn.free()
    # ---- first-seen group ids + grouped SUM, low and high cardinality
    m = min(n, 100_000_000)
    for card in (4, 1_000_000):
        keys = DeviceBuffer(8 * m, lib); groups = DeviceBuffer(8 * m, lib)
        capi.check(lib.MoB200_GenInt64(7, 0, m, keys.ptr, None, 0), lib)
        # fold the 2^32 generator range down to `card` distinct keys with the Go modulo kernel (non-negative after + 2^31)
        kb = np.asarray([1 << 31], dtype=np.int64); kc = np.asarray([card], dtype=np.int64)
        rn = DeviceBuffer(((m + 63) // 64) * 8, lib); capi.check(lib.MoB200_Memset(rn.ptr, 0, rn.nbytes), lib)
        prm = np.zeros(2, dtype=np.int64); prm[1] = -1
        kv = lambda: Vector(data_ptr=keys.ptr, data_nbytes=8 * m, nulls_ptr=rn.ptr, length=m)
        xcall(capi.XCALL_GO_ARITH(0, capi.T_INT64), [kv(), Vector(data_ptr=keys.ptr, data_nbytes=8 * m, length=m), Vector(data=kb, length=m), Vector(data=prm.view(np.uint8), length=m)], m)
        xcall(capi.XCALL_GO_ARITH(4, capi.T_INT64), [kv(), Vector(data_ptr=keys.ptr, data_nbytes=8 * m, length=m), Vector(data=kc, length=m), Vector(data=prm.view(np.uint8), length=m)], m)
        cap = card + 64
        tkeys = DeviceBuffer(8 * cap, lib); ng = DeviceBuffer(8, lib)
        def gid():
            capi.check(lib.MoB200_Memset(ng.ptr, 0, 8), lib)
            ops.GroupTable(1).insert_device(keys, m, groups, ng, tkeys, cap)
        ms = timed(gid, reps=3)
        found = int(ng.to_numpy(np.int64)[0])
        out["group_ids_card_%d" % card] = {"ms_insert_kernel": ms, "rows": m, "groups": found, "rows_per_s_insert": m / ms * 1e3}
        state = DeviceBuffer(8 * found, lib); sn = DeviceBuffer(((found + 63) // 64) * 8, lib); cnt = DeviceBuffer(8 * found, lib)
        capi.check(lib.MoB200_Memset(state.ptr, 0, state.nbytes), lib); capi.check(lib.MoB200_Memset(sn.ptr, 0xff, sn.nbytes), lib); capi.check(lib.MoB200_Memset(cnt.ptr, 0, cnt.nbytes), lib)
        gv = [Vector(data_ptr=state.ptr, data_nbytes=8 * found, nulls_ptr=sn.ptr, length=found), Vector(data_ptr=cnt.ptr, data_nbytes=8 * found, length=found),
              Vector(data_ptr=groups.ptr, data_nbytes=8 * m, length=m), Vector(data_ptr=bufs["quantity"].ptr, data_nbytes=8 * m, length=m)]
        ms = timed(lambda: xcall(capi.XCALL_GROUP_AGG(capi.AGG_SUM, capi.T_FLOAT64), gv, m), reps=3)
        out["group_sum_f64_card_%d" % card] = {"ms": ms, "gbs": 16.0 * m / ms / 1e6, "rows_per_s": m / ms * 1e3}
        for b in (keys, groups, rn, tkeys, ng, state, sn, cnt):
            b.free()
    # ---- bloom filter probe (cgo/bloom.h entry points): build on 10 M keys, probe m int64 keys; the reference's own C next to it on one host core
    try:
        _vp, _sz, _u64, _u32 = C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint32
        def proto(l):
            l.bloomfilter_init_with_seed.restype = _vp; l.bloomfilter_init_with_seed.argtypes = [_u64, _u32, _u64]
            l.bloomfilter_add_fixed.restype = None; l.bloomfilter_add_fixed.argtypes = [_vp, _vp, _sz, _sz, _sz, _vp, _sz]
            l.bloomfilter_test_fixed.restype = None; l.bloomfilter_test_fixed.argtypes = [_vp, _vp, _sz, _sz, _sz, _vp, _sz, _vp]
            l.bloomfilter_free.restype = None; l.bloomfilter_free.argtypes = [_vp]
            return l
        proto(lib)
        nb, nk, kk = 10_000_000, min(n, 100_000_000), 3
        nbits = 1 << 27                                            # 16 MB filter, ~13 bits per key
        keys = DeviceBuffer(8 * nk, lib); res = DeviceBuffer(nk, lib)
        capi.check(lib.MoB200_GenInt64(11, 0, nk, keys.ptr, None, 0), lib)
        bf = lib.bloomfilter_init_with_seed(nbits, kk, 1)
        lib.bloomfilter_add_fixed(bf, keys.ptr, 8 * nb, 8, nb, None, 0)
        ms = timed(lambda: lib.bloomfilter_test_fixed(bf, keys.ptr, 8 * nk, 8, nk, None, 0, res.ptr), reps=3)
        out["bloom_test_fixed_i64"] = {"ms": ms, "keys": nk, "filter_mb": nbits / 8e6, "k": kk, "keys_per_s": nk / ms * 1e3, "gbs_stream": 9.0 * nk / ms / 1e6}
        ms = timed(lambda: lib.bloomfilter_add_fixed(bf, keys.ptr, 8 * nb, 8, nb, None, 0), reps=3)
        out["bloom_add_fixed_i64"] = {"ms": ms, "keys": nb, "keys_per_s": nb / ms * 1e3}
        hit = int(res.to_numpy(np.uint8).sum())
        out["bloom_test_fixed_i64"]["positives"] = hit
        # one 8192-row block from HOST pointers (the drop-in case), and the reference's C on the same block
        import time
        hk = keys.to_numpy(np.int64, 8192).copy(); hr = np.zeros(8192, np.uint8)
        def block(l, f):
            t0 = time.perf_counter()
            for _ in range(200):
                l.bloomfilter_test_fixed(f, hk.ctypes.data, hk.nbytes, 8, 8192, None, 0, hr.ctypes.data)
            return (time.perf_counter() - t0) / 200 * 1e6
        block(lib, bf)
        out["bloom_block_8192_host_us"] = block(lib, bf)
        refp = os.path.join(ROOT, "oracle", "_ref", "libbloom_ref.so")
        if os.path.exists(refp):
            ref = proto(C.CDLL(refp))
            hb = keys.to_numpy(np.int64, nb)
            rbf = ref.bloomfilter_init_with_seed(nbits, kk, 1)
            ref.bloomfilter_add_fixed(rbf, hb.ctypes.data, hb.nbytes, 8, nb, None, 0)
            out["bloom_block_8192_reference_c_us"] = block(ref, rbf)
            hres = np.zeros(nb, np.uint8)
            t0 = time.perf_counter()
            ref.bloomfilter_test_fixed(rbf, hb.ctypes.data, hb.nbytes, 8, nb, None, 0, hres.ctypes.data)
            out["bloom_reference_c_keys_per_s_one_core"] = nb / (time.perf_counter() - t0)
            ref.bloomfilter_free(rbf)
        lib.bloomfilter_free(bf); keys.free(); res.free()
    except Exception as e:   # keep the other numbers
        out["bloom_error"] = repr(e)
    # ---- LZ4 block decode: 16000 column blocks (8192 int64 rows each, ~2.5x compressible) in one call vs liblz4 on one host core
    try:
        import time
        import pyarrow as pa
        rng = np.random.default_rng(3)
        raws = [(rng.integers(0, 1000, 8192) + i).astype(np.int64).tobytes() for i in range(64)]
        comps = [pa.compress(r, codec="lz4_raw", asbytes=True) for r in raws]
        nblk = 16000                                              # a scan's worth: the decoder keeps one block per warp in flight, up to 48 per SM
        blocks = [comps[i % 64] for i in range(nblk)]
        src = np.frombuffer(b"".join(blocks), dtype=np.uint8)
        desc = np.zeros((nblk, 4), dtype=np.int64); so = 0
        for i, b in enumerate(blocks):
            desc[i] = (so, len(b), i * 65536, 65536); so += len(b)
        dsrc = DeviceBuffer.from_numpy(src); ddesc = DeviceBuffer.from_numpy(desc.reshape(-1)); ddst = DeviceBuffer(nblk * 65536, lib)
        vecs = [Vector(data_ptr=ddst.ptr, data_nbytes=nblk * 65536, length=nblk * 65536), Vector(data_ptr=dsrc.ptr, data_nbytes=src.nbytes, length=src.nbytes),
                Vector(data_ptr=ddesc.ptr, data_nbytes=desc.nbytes, length=4 * nblk)]
        ms = timed(lambda: xcall(capi.XCALL_LZ4_DECODE, vecs, nblk), reps=3)
        assert ddst.to_numpy(np.uint8, 65536).tobytes() == raws[0]
        t0 = time.perf_counter()
        for c in blocks[:400]:
            pa.decompress(c, decompressed_size=65536, codec="lz4_raw", asbytes=True)
        cpu_s = (time.perf_counter() - t0) / 400 * nblk
        out["lz4_decode"] = {"ms": ms, "blocks": nblk, "compressed_mb": src.nbytes / 1e6, "decoded_mb": nblk * 65536 / 1e6, "gbs_out": nblk * 65536 / ms / 1e6,
                             "liblz4_one_core_gbs_out": nblk * 65536 / cpu_s / 1e9}
        dsrc.free(); ddesc.free(); ddst.free()
    except Exception as e:
        out["lz4_error"] = repr(e)
    # ---- Elkan k-means (index build): 100 k x 128-d vectors, 256 clusters, <= 10 iterations; the oracle port (= the reference's loop) on one host core
    try:
        import time
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import oracle_lib as O
        kn, kd, kk = 100_000, 128, 256
        kv = datagen.vectors_f32(33, 0, kn, kd)
        kinit = kv[:: kn // kk][:kk].copy()
        krnd = np.random.default_rng(5).random(kd * kk * 4).astype(np.float32)
        ops.kmeans_elkan(kv[:2000], kinit[:8], 2, krnd)                       # warm-up
        t0 = time.perf_counter()
        gc, ga, gi = ops.kmeans_elkan(kv, kinit, 10, krnd)
        gpu_s = time.perf_counter() - t0
        oc = kinit.copy(); oa = np.zeros(kn, np.int64)
        t0 = time.perf_counter()
        oi = O.go().og_km_cluster_f32(O.p(kv), kn, kd, O.p(oc), kk, 10, O.p(krnd), len(krnd), O.p(oa))
        cpu_s = time.perf_counter() - t0
        out["kmeans_elkan"] = {"n": kn, "dim": kd, "k": kk, "iterations": gi, "gpu_s_host_pointers": gpu_s, "oracle_one_core_s": cpu_s,
                               "bit_equal": bool(gi == oi and (ga == oa).all() and gc.tobytes() == oc.tobytes())}
    except Exception as e:
        out["kmeans_error"] = repr(e)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
