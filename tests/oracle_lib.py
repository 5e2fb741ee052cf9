"""ctypes access to the CPU oracle (TEST INFRASTRUCTURE): oracle/liboracle_go.so (C restatement of the Go loops) and,
when present, oracle/_ref/libmo_ref.so (the reference's own C compiled unchanged) and libusearch_ref.so.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference may import this module.
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import build as oracle_build  # noqa: E402

_vp, _u64, _i32, _i64, _f64 = C.c_void_p, C.c_uint64, C.c_int32, C.c_int64, C.c_double

_go = None
_ref = None
_usearch = None


def go():
    global _go
    if _go is None:
        path = oracle_build.build_oracle_go()
        lib = C.CDLL(path)
        lib.og_arith.restype = _i32
        lib.og_arith.argtypes = [_i32, _i32, _vp, _vp, _vp, _u64, _i32, _i32, _vp, _vp, _vp, _i32, _vp]
        lib.og_compare.restype = _i32
        lib.og_compare.argtypes = [_i32, _i32, _vp, _vp, _vp, _u64, _i32, _i32, _vp, _vp, _vp]
        lib.og_compare_f32_scale.restype = _i32
        lib.og_compare_f32_scale.argtypes = [_i32, _i32, _vp, _vp, _vp, _u64, _i32, _i32, _vp, _vp, _vp]
        lib.og_between.restype = _i32
        lib.og_between.argtypes = [_i32, _vp, _vp, _vp, _vp, _u64, _vp, _vp]
        lib.og_multi_logic.restype = _i32
        lib.og_multi_logic.argtypes = [_i32, _vp, _vp, _i32, _vp, _vp, _vp, _u64]
        lib.og_filter_sels.restype = _i64
        lib.og_filter_sels.argtypes = [_vp, _vp, _u64, _vp]
        lib.og_shuffle_fixed.restype = None
        lib.og_shuffle_fixed.argtypes = [_vp, _vp, _vp, _i64, _i32]
        lib.og_nulls_filter.restype = None
        lib.og_nulls_filter.argtypes = [_vp, _u64, _vp, _i64, _vp]
        for sfx in ("f32", "f64"):
            getattr(lib, "og_km_init_bounds_" + sfx).restype = None
            getattr(lib, "og_km_init_bounds_" + sfx).argtypes = [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _vp]
            getattr(lib, "og_km_centroid_dists_" + sfx).restype = None
            getattr(lib, "og_km_centroid_dists_" + sfx).argtypes = [_vp, _i64, _i64, _vp, _vp]
            getattr(lib, "og_km_assign_" + sfx).restype = _i64
            getattr(lib, "og_km_assign_" + sfx).argtypes = [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp]
            getattr(lib, "og_km_recalc_" + sfx).restype = _i32
            getattr(lib, "og_km_recalc_" + sfx).argtypes = [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _vp]
            getattr(lib, "og_km_update_bounds_" + sfx).restype = None
            getattr(lib, "og_km_update_bounds_" + sfx).argtypes = [_vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp]
            getattr(lib, "og_km_cluster_" + sfx).restype = _i64
            getattr(lib, "og_km_cluster_" + sfx).argtypes = [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _i64, _vp]
        lib.og_lz4_decode_block.restype = _i64
        lib.og_lz4_decode_block.argtypes = [_vp, _i64, _vp, _i64]
        lib.og_join_sels.restype = _i64
        lib.og_join_sels.argtypes = [_vp, _i64, _i64, _vp, _vp]
        lib.og_join_find.restype = None
        lib.og_join_find.argtypes = [_vp, _i64, _vp, _vp, _i64, _vp]
        lib.og_join_probe.restype = _i64
        lib.og_join_probe.argtypes = [_vp, _i64, _vp, _vp, _i32, _vp, _vp, _i64]
        lib.og_group_ids.restype = _i64
        lib.og_group_ids.argtypes = [_vp, _u64, _vp, _vp, _i64, _i64]
        lib.og_sum_int64.restype = _i32
        lib.og_sum_int64.argtypes = [_i32, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _vp, _vp]
        lib.og_sum_uint64.restype = _i32
        lib.og_sum_uint64.argtypes = [_i32, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _vp, _vp]
        lib.og_sum_float64.restype = _i32
        lib.og_sum_float64.argtypes = [_i32, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _vp]
        lib.og_count.restype = None
        lib.og_count.argtypes = [_i32, _vp, _u64, _vp, _u64, _vp]
        lib.og_minmax.restype = _i32
        lib.og_minmax.argtypes = [_i32, _i32, _vp, _vp, _u64, _vp, _u64, _vp, _vp]
        for sfx, ct in (("f32", C.c_float), ("f64", C.c_double)):
            for name in ("l2sq", "l2", "l1", "ip", "cosdist"):
                f = getattr(lib, "og_%s_%s" % (name, sfx))
                f.restype = ct
                f.argtypes = [_vp, _vp, _i64]
            f = getattr(lib, "og_cossim_%s" % sfx)
            f.restype = ct
            f.argtypes = [_vp, _vp, _i64, _vp]
            f = getattr(lib, "og_moarray_cossim_%s" % sfx)
            f.restype = _f64
            f.argtypes = [_vp, _vp, _i64, _vp]
            f = getattr(lib, "og_normalize_l2_%s" % sfx)
            f.restype = _i32
            f.argtypes = [_vp, _vp, _i64]
            f = getattr(lib, "og_distance_rows_%s" % sfx)
            f.restype = _i32
            f.argtypes = [_i32, _vp, _vp, _i64, _vp, _i64, _i64, _u64, _vp]
        lib.og_heap_topk_f32.restype = None
        lib.og_heap_topk_f32.argtypes = [_vp, _vp, _i64, _i32, _vp, _vp]
        lib.og_bruteforce_search.restype = _i32
        lib.og_bruteforce_search.argtypes = [_i32, _i32, _vp, _i64, _i64, _vp, _i64, _i32, _i32, _vp, _vp]
        lib.og_ivf_search_f32.restype = _i32
        lib.og_ivf_search_f32.argtypes = [_vp, _vp, _i64, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp]
        lib.og_assign_centroids_f32.restype = None
        lib.og_assign_centroids_f32.argtypes = [_vp, _i64, _i64, _vp, _i64, _i32, _vp]
        lib.og_q6.restype = _i32
        lib.og_q6.argtypes = [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _f64, _f64, _f64, _i32, _vp, _vp, _vp]
        lib.og_q1.restype = _i64
        lib.og_q1.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp]
        lib.og_sum_int64_mt.restype = _i32
        lib.og_sum_int64_mt.argtypes = [_vp, _vp, _i64, _i32, _vp, _vp]
        lib.og_gen_lineitem.restype = None
        lib.og_gen_lineitem.argtypes = [_u64, _u64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
        lib.og_gen_int64.restype = None
        lib.og_gen_int64.argtypes = [_u64, _u64, _i64, _i32, _vp]
        lib.og_gen_vectors_f32.restype = None
        lib.og_gen_vectors_f32.argtypes = [_u64, _u64, _i64, _i64, _i32, _vp, _vp, _i64, C.c_float, _vp]
        lib.og_d64_addsub.restype = _i32
        lib.og_d64_addsub.argtypes = [_i32, _vp, _vp, _vp, _u64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]
        lib.og_d64_mul.restype = _i32
        lib.og_d64_mul.argtypes = [_vp, _vp, _vp, _u64, _i32, _i32, _i32, _i32, _vp, _vp, _vp]
        lib.og_d128_addsub.restype = _i32
        lib.og_d128_addsub.argtypes = [_i32, _vp, _vp, _vp, _u64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]
        lib.og_d128_mul.restype = _i32
        lib.og_d128_mul.argtypes = [_vp, _vp, _vp, _u64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]
        lib.og_mul_result_scale.restype = _i32
        lib.og_mul_result_scale.argtypes = [_i32, _i32]
        lib.og_sum_d64.restype = None
        lib.og_sum_d64.argtypes = [_vp, _vp, _u64, _vp, _u64, _vp, _vp]
        lib.og_sum_d128.restype = None
        lib.og_sum_d128.argtypes = [_vp, _vp, _u64, _vp, _u64, _vp, _vp]
        lib.og_kahan_sum.restype = _f64
        lib.og_kahan_sum.argtypes = [_vp, _i64]
        _go = lib
    return _go


def ref():
    """the reference's C kernels compiled unchanged; None when neither /root/reference nor a prebuilt .so exists"""
    global _ref
    if _ref is None:
        path = oracle_build.build_mo_ref()
        if not path or not os.path.exists(path):
            return None
        lib = C.CDLL(path)
        ar = [_vp, _vp, _vp, _u64, _vp, _i32, _i32]
        for k in ("SignedInt", "UnsignedInt", "Float"):
            for op in ("Add", "Sub", "Mul", "Mod"):
                f = getattr(lib, "%s_Vec%s" % (k, op)); f.restype = _i32; f.argtypes = ar
        for n in ("Float_VecDiv", "Float_VecIntegerDiv"):
            f = getattr(lib, n); f.restype = _i32; f.argtypes = ar
        for op in ("Eq", "Ne", "Gt", "Ge", "Lt", "Le"):
            f = getattr(lib, "Numeric_Vec%s" % op); f.restype = _i32; f.argtypes = ar
        lib.Logic_VecAnd.restype = _i32; lib.Logic_VecAnd.argtypes = [_vp, _vp, _vp, _u64, _vp, _vp, _vp, _i32]
        lib.Logic_VecOr.restype = _i32; lib.Logic_VecOr.argtypes = [_vp, _vp, _vp, _u64, _vp, _vp, _vp, _i32]
        lib.Logic_VecXor.restype = _i32; lib.Logic_VecXor.argtypes = [_vp, _vp, _vp, _u64, _vp, _i32]
        lib.Logic_VecNot.restype = _i32; lib.Logic_VecNot.argtypes = [_vp, _vp, _u64, _vp, _i32]
        lib.Bitmap_Count.restype = _u64; lib.Bitmap_Count.argtypes = [_vp, _u64]
        lib.Bitmap_IsEmpty.restype = C.c_bool; lib.Bitmap_IsEmpty.argtypes = [_vp, _u64]
        lib.Bitmap_Contains.restype = C.c_bool; lib.Bitmap_Contains.argtypes = [_vp, _u64]
        lib.Bitmap_Add.restype = None; lib.Bitmap_Add.argtypes = [_vp, _u64]
        lib.Bitmap_Remove.restype = None; lib.Bitmap_Remove.argtypes = [_vp, _u64]
        for n in ("Bitmap_And", "Bitmap_Or"):
            f = getattr(lib, n); f.restype = None; f.argtypes = [_vp, _vp, _vp, _u64]
        lib.Bitmap_Not.restype = None; lib.Bitmap_Not.argtypes = [_vp, _vp, _u64]
        lib.XCall.restype = _i32; lib.XCall.argtypes = [_i64, _i64, _vp, _vp, _u64]
        _ref = lib
    return _ref


def usearch():
    global _usearch
    if _usearch is None:
        path = oracle_build.build_usearch_ref()
        if not path or not os.path.exists(path):
            return None
        lib = C.CDLL(path)
        # usearch_exact_search(dataset, n, stride, queries, q, stride, scalar_kind, dims, metric_kind, count, threads,
        #                      keys, keys_stride, distances, distances_stride, &error)   c/usearch.h:471-478
        lib.usearch_exact_search.restype = None
        lib.usearch_exact_search.argtypes = [_vp, C.c_size_t, C.c_size_t, _vp, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                             C.c_int, C.c_size_t, C.c_size_t, _vp, C.c_size_t, _vp, C.c_size_t, C.POINTER(C.c_char_p)]
        _usearch = lib
    return _usearch


def p(a):
    """pointer of a numpy array (or None)"""
    return None if a is None else a.ctypes.data


# ---- convenience wrappers used by several tests ---------------------------------------------------------------------
def bruteforce(dataset, queries, limit, metric=0, nthreads=8):
    ds = np.ascontiguousarray(dataset)
    qs = np.ascontiguousarray(queries)
    is64 = 1 if ds.dtype == np.float64 else 0
    nq = qs.shape[0]
    keys = np.zeros(nq * limit, dtype=np.int64)
    dists = np.zeros(nq * limit, dtype=np.float64)
    go().og_bruteforce_search(is64, metric, p(ds), ds.shape[0], ds.shape[1], p(qs), nq, limit, nthreads, p(keys), p(dists))
    return keys, dists


def q6(cols, n, params, nthreads=1):
    s = np.zeros(1, dtype=np.float64); nul = np.zeros(1, dtype=np.uint8); ns = np.zeros(1, dtype=np.int64)
    go().og_q6(p(cols["shipdate"]), p(cols["discount"]), p(cols["quantity"]), p(cols["extendedprice"]), n,
               params[0], params[1], params[2], params[3], params[4], nthreads, p(s), p(nul), p(ns))
    return float(s[0]), int(ns[0]), bool(nul[0])


def q1(cols, n, cutoff, nthreads=1):
    keys = np.zeros(64, dtype=np.uint64); sums = np.zeros(64 * 7, dtype=np.float64)
    cnts = np.zeros(64 * 4, dtype=np.int64); first = np.zeros(64, dtype=np.int64)
    ng = go().og_q1(p(cols["shipdate"]), p(cols["quantity"]), p(cols["extendedprice"]), p(cols["discount"]), p(cols["tax"]),
                    p(cols["returnflag"]), p(cols["linestatus"]), n, cutoff, nthreads, p(keys), p(sums), p(cnts), p(first))
    out = []
    for g in range(max(ng, 0)):
        s = sums[g * 7:(g + 1) * 7]; c = cnts[g * 4:(g + 1) * 4]
        out.append({"returnflag": int(keys[g]) & 0xff, "linestatus": (int(keys[g]) >> 8) & 0xff, "first_row": int(first[g]),
                    "sum_qty": s[0], "sum_base_price": s[1], "sum_disc_price": s[2], "sum_charge": s[3],
                    "avg_qty": s[4] / c[0], "avg_price": s[5] / c[1], "avg_disc": s[6] / c[2], "sum_disc": s[6], "count_order": int(c[3])})
    out.sort(key=lambda g: g["first_row"])
    return out


def gen_lineitem(seed, row0, n, nthreads=8, names=("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")):
    """lineitem columns for rows [row0, row0 + n): the C twin of MoB200_GenLineitem / datagen.lineitem, first-touched by the pool"""
    dts = {"shipdate": np.int32, "returnflag": np.uint8, "linestatus": np.uint8}
    cols = {k: np.empty(n, dtype=dts.get(k, np.float64)) for k in names}
    g = lambda k: p(cols[k]) if k in cols else None
    go().og_gen_lineitem(seed, row0, n, nthreads, g("shipdate"), g("quantity"), g("extendedprice"), g("discount"), g("tax"), g("returnflag"), g("linestatus"))
    return cols


def gen_int64(seed, row0, n, nthreads=8):
    out = np.empty(n, dtype=np.int64)
    go().og_gen_int64(seed, row0, n, nthreads, p(out))
    return out


def gen_vectors_f32(seed, row0, n, dim, nthreads=8, centers=None, sigma=1.0, want_components=False):
    out = np.empty((n, dim), dtype=np.float32)
    comp = np.empty(n, dtype=np.int32) if want_components else None
    c = None if centers is None else np.ascontiguousarray(centers, dtype=np.float32)
    go().og_gen_vectors_f32(seed, row0, n, dim, nthreads, p(out), p(c), 0 if c is None else c.shape[0], float(sigma), p(comp))
    return (out, comp) if want_components else out


def d128_to_int(arr):
    """uint64[n, 2] {lo, hi} two's-complement -> python ints"""
    a = np.asarray(arr, dtype=np.uint64).reshape(-1, 2)
    out = []
    for lo, hi in a:
        v = (int(hi) << 64) | int(lo)
        out.append(v - (1 << 128) if v >> 127 else v)
    return out


def int_to_d128(vals):
    out = np.zeros((len(vals), 2), dtype=np.uint64)
    for i, v in enumerate(vals):
        u = v & ((1 << 128) - 1)
        out[i, 0] = u & 0xFFFFFFFFFFFFFFFF
        out[i, 1] = u >> 64
    return out


def decimal_str(v, scale):
    """Decimal.Format: unscaled integer -> fixed-point text"""
    sign = "-" if v < 0 else ""
    s = str(abs(v)).rjust(scale + 1, "0")
    return sign + (s[:-scale] + "." + s[-scale:] if scale else s)
