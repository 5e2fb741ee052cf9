"""Filtered vector search: throughput of the masked scan, the compacted search and auto selection against the unfiltered search.

    python tools/filtered_search_bench.py [--rows 1000000] [--ivf-rows 2000000] [--queries 10000] [--runs 5] [--out FILE]

Brute force at the BASELINE config 4 shape (1 M x 768, 10 k queries, k = 10) and IVF-flat with the config 5 list structure (1024 lists,
nprobe 32) at the rows one GPU holds next to its prepared operand.  For every admitted fraction a bloom filter is built from a random key
subset; the forced masked path (search_filter_path 1), the forced compacted path (2), auto (0) and the unfiltered search are timed in the
same process, alternating, with CUDA events after a warm-up, median of --runs.  Every timed output is checked against an unfiltered
search of an index built from the admitted rows only (a sample of the queries).  The card's name and power limit are printed with the
numbers: a rate means nothing without them.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from matrixone_b200 import capi, ops  # noqa: E402
from matrixone_b200.vector import DeviceBuffer  # noqa: E402

FRACTIONS = [1.0, 0.5, 0.1, 0.01, 0.001, 0.0001]
PATHS = {"mask": 1, "compact": 2, "auto": 0}
CHECK_Q = 256


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still printed, marked as measured on an unknown card
        return "unknown (%s)" % e


class Bloom:
    def __init__(self, lib, keys, seed):
        lib.bloomfilter_init_with_seed.restype = C.c_void_p
        lib.bloomfilter_init_with_seed.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64]
        lib.bloomfilter_add_fixed.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t]
        lib.bloomfilter_test_fixed.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        lib.bloomfilter_free.argtypes = [C.c_void_p]
        self.lib = lib
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        self.h = lib.bloomfilter_init_with_seed(max(64, 16 * keys.size), 3, seed)
        lib.bloomfilter_add_fixed(self.h, keys.ctypes.data, keys.nbytes, 8, keys.size, None, 0)

    def admits(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        r = np.zeros(keys.size, dtype=np.uint8)
        self.lib.bloomfilter_test_fixed(self.h, keys.ctypes.data, keys.nbytes, 8, keys.size, None, 0, r.ctypes.data)
        return r.astype(bool)

    def free(self):
        self.lib.bloomfilter_free(self.h)


def once(lib, fn):
    """CUDA-event time of one call of fn() in milliseconds (the search returns its results to the host: it ends synchronised)"""
    capi.check(lib.MoB200_TimerStart(), lib)
    fn()
    t = C.c_float()
    capi.check(lib.MoB200_TimerStop(C.byref(t)), lib)
    return t.value


def same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--ivf-rows", type=int, default=2_000_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    dim, k, nlist, nprobe, nq = 768, 10, 1024, 32, a.queries
    report = {"card": card(), "dim": dim, "k": k, "queries": nq, "runs": a.runs, "results": []}
    print("card (name, power limit, max SM clock):", report["card"], flush=True)

    cent = DeviceBuffer(4 * nlist * dim, lib)
    capi.check(lib.MoB200_GenVectorsF32(30, 0, nlist, dim, cent.ptr, None, 0, 1.0), lib)
    hcent = cent.to_numpy(np.float32).reshape(nlist, dim) * np.float32(4.0)
    cent.free(); cent = DeviceBuffer.from_numpy(hcent, lib)
    dq = DeviceBuffer(4 * nq * dim, lib)
    capi.check(lib.MoB200_GenVectorsF32(32, 0, nq, dim, dq.ptr, cent.ptr, nlist, 1.0), lib)
    qs = dq.to_numpy(np.float32).reshape(nq, dim)
    qcheck = np.ascontiguousarray(qs[:CHECK_Q])

    for which in ("bruteforce", "ivf"):
        n = a.rows if which == "bruteforce" else a.ivf_rows
        data = DeviceBuffer(4 * n * dim, lib)
        capi.check(lib.MoB200_GenVectorsF32(31, 0, n, dim, data.ptr, cent.ptr, nlist, 1.0), lib)
        if which == "bruteforce":
            idx = ops.BruteForceIndex(data, dim, capi.METRIC_L2, lib=lib)
            keys_of_rows = np.arange(n, dtype=np.int64)
            search = lambda q, f=None: idx.search(q, k, filter=f)
        else:
            idx = ops.IvfflatSearchIndex.build(data, n, hcent, capi.METRIC_L2, lib)
            data.free()                       # the index holds its own list-ordered copy
            keys_of_rows = idx.row_ids        # primary key of every list-ordered entry
            search = lambda q, f=None: idx.search(q, k, nprobe, filter=f)
        search(dq)
        ms_unf = float(np.median([once(lib, lambda: search(dq)) for _ in range(a.runs)]))
        print("%s n=%d unfiltered: %.2f ms  %.0f qps" % (which, n, ms_unf, nq / ms_unf * 1e3), flush=True)
        rng = np.random.default_rng(7)
        for frac in FRACTIONS:
            members = np.flatnonzero(rng.random(n) < frac).astype(np.int64)
            bl = Bloom(lib, members, 1234)
            row = {"workload": which, "rows": n, "fraction": frac}
            outs = {}
            # alternate: every round times each path once, the unfiltered search included
            times = {p: [] for p in list(PATHS) + ["unfiltered"]}
            for p, v in PATHS.items():      # warm-up of every shape
                lib.MoB200_SetTuning(b"search_filter_path", v); search(dq, bl.h)
            search(dq)
            for _ in range(a.runs):
                for p, v in PATHS.items():
                    lib.MoB200_SetTuning(b"search_filter_path", v)
                    times[p].append(once(lib, lambda: search(dq, bl.h)))
                    if p == "auto":
                        row["auto_compacted"] = lib.MoB200_SetTuning(b"get_filter_compacted", 0)
                        row["admitted"] = lib.MoB200_SetTuning(b"get_filter_admitted", 0)
                times["unfiltered"].append(once(lib, lambda: search(dq)))
            for p, v in PATHS.items():
                lib.MoB200_SetTuning(b"search_filter_path", v)
                outs[p] = search(qcheck, bl.h)
            lib.MoB200_SetTuning(b"search_filter_path", 0)
            # subset check: an index of the admitted rows only, unfiltered; its ordinals mapped back to keys
            adm_keys = keys_of_rows[bl.admits(keys_of_rows)] if which == "ivf" else np.flatnonzero(bl.admits(keys_of_rows))
            if which == "bruteforce":
                rows = adm_keys
                sub = DeviceBuffer(4 * max(rows.size, 1) * dim, lib)
                if rows.size:
                    dr = DeviceBuffer.from_numpy(rows, lib)
                    capi.check(lib.MoB200_GatherRowsF32(sub.ptr, data.ptr, dr.ptr, rows.size, dim), lib); dr.free()
                sidx = ops.BruteForceIndex(sub.view(4 * rows.size * dim), dim, capi.METRIC_L2, lib=lib)
                sk, sd = sidx.search(qcheck, k)
                sk = np.where(sk >= 0, (rows if rows.size else np.zeros(1, dtype=np.int64))[np.maximum(sk, 0)], -1)
                sidx.destroy(); sub.free()
            else:
                adm = bl.admits(idx.row_ids)                         # list-ordered entries whose primary key is admitted
                pos = np.flatnonzero(adm)
                sub = DeviceBuffer(4 * max(pos.size, 1) * dim, lib)
                if pos.size:
                    dr = DeviceBuffer.from_numpy(pos.astype(np.int64), lib)
                    capi.check(lib.MoB200_GatherRowsF32(sub.ptr, idx.d_data.ptr, dr.ptr, pos.size, dim), lib); dr.free()
                lists = np.repeat(np.arange(nlist), np.diff(idx.offsets))[pos]
                sidx = ops.IvfflatSearchIndex(sub.view(4 * pos.size * dim), lists.astype(np.int32), hcent, capi.METRIC_L2, lib)
                sub.free()                                           # (the index keeps its own list-ordered copy)
                sk, sd = sidx.search(qcheck, k, nprobe)              # keys = positions in the subset (already in list order)
                ids = idx.row_ids[pos] if pos.size else np.zeros(1, dtype=np.int64)
                sk = np.where(sk >= 0, ids[np.maximum(sk, 0)], -1)
                sidx.destroy()
            ok = all(o[1].tobytes() == sd.tobytes() for o in outs.values()) and all(same(outs[p], outs["mask"]) for p in outs)
            keys_ok = all(np.array_equal(o[0], sk) for o in outs.values())
            row.update({p + "_ms": float(np.median(v)) for p, v in times.items()})
            row.update({p + "_qps": nq / float(np.median(v)) * 1e3 for p, v in times.items()})
            row["spread_ms"] = {p: [float(min(v)), float(max(v))] for p, v in times.items()}
            row["matches_subset_search"] = {"distances": bool(ok), "keys": bool(keys_ok)}
            report["results"].append(row)
            print(json.dumps(row), flush=True)
            bl.free()
        idx.destroy()
        data.free()
    dq.free(); cent.free()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
