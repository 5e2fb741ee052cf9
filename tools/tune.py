#!/usr/bin/env python
"""One-call kernel survey on a GPU: every hot kernel at a bench-like size, variants side by side.
Prints one JSON line per measurement (kernel-only CUDA-event time via MoB200_LastKernelMs, median of `reps`)."""
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from matrixone_b200 import capi, datagen, ops  # noqa: E402
from matrixone_b200.vector import DeviceBuffer, Vector, varlena_column_from_matrix, xcall  # noqa: E402

lib = None
PEAK = 6568.4
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass

# Q6 selectivity sweep: (name, (date_lo, date_hi, disc_lo, disc_hi, qty_hi))
Q6_SWEEP = (("q6", datagen.q6_params()),
            ("every_row_passes", (-2**31, 2**31 - 1, -np.inf, np.inf, np.inf)),
            ("discount_window_empty", (-2**31, 2**31 - 1, 1.0, 0.0, np.inf)),
            ("no_row_passes", (0, 0, -np.inf, np.inf, np.inf)))
Q6_GRAINS = (32, 64, 128)
Q6_VARIANTS = (0, 1)   # selective (default), dense


def q6_touched_bytes(shipdate, discount, quantity, params, grain):
    """Bytes the selective Q6 kernel must read when DRAM is fetched in aligned `grain`-byte blocks: all of shipdate; discount in the
    blocks holding a row inside the date range; quantity where a row also passed the discount test; price where a row passed all
    three.  The columns start on a `grain` boundary (device allocations are 256-byte aligned), and the slice must too."""
    date_lo, date_hi, disc_lo, disc_hi, qty_hi = params
    alive = (shipdate >= date_lo) & (shipdate < date_hi)

    def blocks(mask, width):
        per = grain // width
        m = np.zeros(-(-mask.size // per) * per, dtype=bool)
        m[:mask.size] = mask
        return int(m.reshape(-1, per).any(axis=1).sum()) * grain

    total = blocks(np.ones(shipdate.size, dtype=bool), 4) + blocks(alive, 8)
    alive &= (discount >= disc_lo) & (discount <= disc_hi)
    total += blocks(alive, 8)
    alive &= quantity < qty_hi
    return total + blocks(alive, 8)


def l2_fetch_granularity():
    """cudaLimitMaxL2FetchGranularity as the CUDA runtime reports it, or None.  Read only: the limit is process-wide, and a library
    embedded in a database must leave it to the host process."""
    for name in ("libcudart.so", "libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            rt = C.CDLL(name)
        except OSError:
            continue
        v = C.c_size_t(0)
        return v.value if rt.cudaDeviceGetLimit(C.byref(v), 5) == 0 else None   # 5 = cudaLimitMaxL2FetchGranularity
    return None


def kms():
    v = C.c_float()
    lib.MoB200_LastKernelMs(C.byref(v))
    return v.value


def timed(fn, reps=7, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        fn()
        ts.append(kms())
    return statistics.median(ts), min(ts)


def report(name, ms, best, nbytes=None, **kw):
    d = {"bench": name, "kernel_ms_median": round(ms, 4), "kernel_ms_min": round(best, 4)}
    if nbytes:
        d["GBps"] = round(nbytes / ms / 1e6, 1)
        d["frac_of_measured_hbm"] = round(nbytes / ms / 1e6 / PEAK, 3)
    d.update(kw)
    print(json.dumps(d), flush=True)


def q6_sweep(b, n):
    """selective (default) vs dense (q6_variant=1) Q6 kernel, timed alternately over parameter sets of falling selectivity, next to the
    bytes each set makes the selective kernel read (counted from the columns)"""
    print(json.dumps({"bench": "q6_env", "l2_fetch_granularity": l2_fetch_granularity()}), flush=True)
    chunk = 1 << 24
    for name, P in Q6_SWEEP:
        touched = dict.fromkeys(Q6_GRAINS, 0)
        for r0 in range(0, n, chunk):
            m = min(chunk, n - r0)
            sd = b["shipdate"].view(4 * m, 4 * r0).to_numpy(np.int32)
            di = b["discount"].view(8 * m, 8 * r0).to_numpy(np.float64)
            qt = b["quantity"].view(8 * m, 8 * r0).to_numpy(np.float64)
            for g in Q6_GRAINS:
                touched[g] += q6_touched_bytes(sd, di, qt, P, g)
        times = {var: [] for var in Q6_VARIANTS}
        results = {}
        for _ in range(5):
            for var in Q6_VARIANTS:
                lib.MoB200_SetTuning(b"q6_variant", var)
                ms, _best = timed(lambda: results.__setitem__(var, ops.q6_filter_sum(b["shipdate"], b["discount"], b["quantity"], b["extendedprice"], n, *P)), reps=3, warm=1)
                times[var].append(ms)
        lib.MoB200_SetTuning(b"q6_variant", 0)
        for var in Q6_VARIANTS:
            ms = statistics.median(times[var])
            report("q6_sweep", ms, min(times[var]), 28.0 * n, params=name, variant=var, rows=n, kernel_ms_range=[round(min(times[var]), 4), round(max(times[var]), 4)],
                   Grows_per_s=round(n / ms / 1e6, 2), qualifying_rows=results[var][1], same_as_dense=results[var][:2] == results[1][:2],
                   touched_bytes_per_row={g: round(touched[g] / n, 3) for g in Q6_GRAINS},
                   touched_GBps={g: round(touched[g] / ms / 1e6, 1) for g in Q6_GRAINS})


def main():
    global lib
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    which = set(sys.argv[1:]) or {"q6", "q1", "sum", "elem", "dist", "bf"}
    n = int(os.environ.get("TUNE_ROWS", 200_000_000))
    if which & {"q6", "q1"}:
        names = ["shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus"]
        size = {"shipdate": 4, "returnflag": 1, "linestatus": 1}
        b = {k: DeviceBuffer(size.get(k, 8) * n, lib) for k in names}
        capi.check(lib.MoB200_GenLineitem(10, 0, n, b["shipdate"].ptr, b["quantity"].ptr, b["extendedprice"].ptr, b["discount"].ptr,
                                          b["tax"].ptr, b["returnflag"].ptr, b["linestatus"].ptr), lib)
        if "q6" in which:
            q6_sweep(b, n)
        if "q1" in which:
            for var in (0, 1):   # kernel chosen from the input (TMA from 65,536 rows), register kernel
                lib.MoB200_SetTuning(b"q1_variant", var)
                ms, best = timed(lambda: ops.q1_group_agg(b["shipdate"], b["quantity"], b["extendedprice"], b["discount"], b["tax"],
                                                          b["returnflag"], b["linestatus"], n, datagen.Q1_CUTOFF))
                report("q1_packed_keys", ms, best, 38.0 * n, variant=var, rows=n, Grows_per_s=round(n / ms / 1e6, 2))
            lib.MoB200_SetTuning(b"q1_variant", 0)
        for x in b.values():
            x.free()
    if "sum" in which:
        for rows in (10_000_000, 400_000_000):
            dv = DeviceBuffer(8 * rows, lib); dn = DeviceBuffer(8 * ((rows + 63) // 64), lib)
            capi.check(lib.MoB200_GenInt64(1, 0, rows, dv.ptr, dn.ptr, 50), lib)
            ms, best = timed(lambda: ops.agg_sum(capi.T_INT64, dv, None, rows))
            report("sum_int64", ms, best, 8.0 * rows, rows=rows)
            ms, best = timed(lambda: ops.agg_sum(capi.T_INT64, dv, dn, rows))
            report("sum_int64_nulls", ms, best, 8.125 * rows, rows=rows)
            ms, best = timed(lambda: ops.agg_min(capi.T_INT64, dv, None, rows))
            report("min_int64", ms, best, 8.0 * rows, rows=rows)
            dv.free(); dn.free()
    if "elem" in which:
        rows = 200_000_000
        a = DeviceBuffer(8 * rows, lib); bb = DeviceBuffer(8 * rows, lib); r = DeviceBuffer(8 * rows, lib)
        capi.check(lib.MoB200_GenInt64(1, 0, rows, a.ptr, None, 0), lib)
        capi.check(lib.MoB200_GenInt64(2, 0, rows, bb.ptr, None, 0), lib)
        import time
        for name, fn, nb in (("SignedInt_VecAdd_i64", lambda: lib.SignedInt_VecAdd(r.ptr, a.ptr, bb.ptr, rows, None, 0, 8), 24.0 * rows),
                             ("Numeric_VecLt_i64", lambda: lib.Numeric_VecLt(r.ptr, a.ptr, bb.ptr, rows, None, 0, capi.T_INT64), 17.0 * rows)):
            fn(); fn()
            t0 = time.perf_counter()
            for _ in range(5):
                fn()
            ms = (time.perf_counter() - t0) / 5 * 1e3
            report(name, ms, ms, nb, rows=rows, timer="wall clock incl. sync")
        # the Go-convention ops (goelem.cu): result nulls in/out, first-offender status
        rn = DeviceBuffer(8 * ((rows + 63) // 64), lib)
        capi.check(lib.MoB200_Memset(rn.ptr, 0, rn.nbytes), lib)
        params = np.zeros(2, dtype=np.int64)
        for name, fid, nb, rsz in (("go_add_i64", capi.XCALL_GO_ARITH(0, capi.T_INT64), 24.125 * rows, 8), ("go_lt_i64", capi.XCALL_GO_COMPARE(4, capi.T_INT64), 17.125 * rows, 1)):
            args = [Vector(data_ptr=r.ptr, data_nbytes=rsz * rows, nulls_ptr=rn.ptr, length=rows), Vector(data_ptr=a.ptr, data_nbytes=8 * rows, length=rows),
                    Vector(data_ptr=bb.ptr, data_nbytes=8 * rows, length=rows), Vector(data=params.view(np.uint8), length=rows)]
            xcall(fid, args, rows); xcall(fid, args, rows)
            ks = []
            for _ in range(5):
                xcall(fid, args, rows); ks.append(kms())
            report(name, float(np.median(ks)), min(ks), nb, rows=rows)
        rn.free()
        for x in (a, bb, r):
            x.free()
    if "dist" in which:
        rows, dim = int(os.environ.get("TUNE_DIST_ROWS", "2000000")), 768
        mat = DeviceBuffer(4 * rows * dim, lib)
        capi.check(lib.MoB200_GenVectorsF32(20, 0, rows, dim, mat.ptr, None, 0, 1.0), lib)
        cells = np.zeros((rows, 6), dtype=np.uint32); cells[:, 0] = 0xFFFFFFFF
        cells[:, 1] = (np.arange(rows, dtype=np.uint64) * (dim * 4)).astype(np.uint32); cells[:, 2] = dim * 4
        dc = DeviceBuffer.from_numpy(cells.view(np.uint8).reshape(-1), lib)
        q = datagen.vectors_f32(21, 0, 1, dim)
        qc, qa = varlena_column_from_matrix(q)
        dr = DeviceBuffer(8 * rows, lib)
        import time
        for fid, nm in ((capi.XCALL_L2DISTANCE_SQ_F32, "xcall_l2sq_f32_const"), (capi.XCALL_GO_L2SQ_F32, "go_l2sq_f32_const"), (capi.XCALL_GO_COSDIST_F32, "go_cosdist_f32_const")):
            args = [Vector(data_ptr=dr.ptr, data_nbytes=8 * rows, length=rows),
                    Vector(data_ptr=dc.ptr, data_nbytes=dc.nbytes, area_ptr=mat.ptr, area_nbytes=mat.nbytes, length=rows),
                    Vector(data=qc, area=qa, length=rows, const=True)]
            xcall(fid, args, rows); xcall(fid, args, rows)
            t0 = time.perf_counter()
            ks = []
            for _ in range(5):
                xcall(fid, args, rows); ks.append(kms())
            ms = (time.perf_counter() - t0) / 5 * 1e3
            report(nm, float(np.median(ks)), min(ks), rows * (dim * 4 + 24 + 8.0), rows=rows, wall_ms_incl_sync=round(ms, 4))
        for x in (mat, dc, dr):
            x.free()
    if "bf" in which:
        dim = 768
        for rows, nq in ((200_000, 2048), (1_000_000, 1024), (1_000_000, 10_000)):
            ds = DeviceBuffer(4 * rows * dim, lib)
            capi.check(lib.MoB200_GenVectorsF32(20, 0, rows, dim, ds.ptr, None, 0, 1.0), lib)
            dq = DeviceBuffer(4 * nq * dim, lib)
            capi.check(lib.MoB200_GenVectorsF32(21, 0, nq, dim, dq.ptr, None, 0, 1.0), lib)
            idx = ops.BruteForceIndex(ds, dim, lib=lib)
            import time
            for mode, name in ((1, "exact"), (2, "tensor_core")):
                lib.MoB200_SetTuning(b"search_mode", mode)
                ms, best = timed(lambda: idx.search(dq, 10), reps=3, warm=1)
                t0 = time.perf_counter(); idx.search(dq, 10); wall = (time.perf_counter() - t0) * 1e3
                flop = (3.0 if mode == 1 else 2.0 * 3) * rows * nq * dim
                report("bruteforce_l2_top10_" + name, ms, best, None, rows=rows, queries=nq, kernel_qps=round(nq / ms * 1e3, 1), call_wall_ms=round(wall, 2),
                       call_qps=round(nq / wall * 1e3, 1), TFLOPs=round(flop / ms / 1e9, 2), fallbacks=lib.MoB200_SetTuning(b"get_tc_fallbacks", 0))
            lib.MoB200_SetTuning(b"search_mode", 0)
            ds.free(); dq.free()


if __name__ == "__main__":
    main()
