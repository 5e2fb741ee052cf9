#!/usr/bin/env python
"""Joins with a non-equality condition (JOIN_COND) on resident columns, timed with CUDA events (medians of alternating runs).

    python tools/join_cond_bench.py [--rows 60000000] [--reps 5] [--parent-lib PATH] [--out FILE]

The workload is TPC-H Q21's EXISTS subquery shape, a self-join of lineitem-like rows on l_orderkey with l_suppkey <> l_suppkey: 6 * 10^7
rows, 1..7 rows per order key (uniform), probed against a prepared JoinMap of all of them in 10^6-row batches.  Every probe row has 1..7
candidates (5 on average), its own row among them.
  inner        JOIN_PROBE INNER over every batch (the candidate pairs)
  cond_*       JOIN_COND alone over every batch's candidates and condition (computed once, outside the timing): SEMI, ANTI, LEFT, and
               RIGHT + JOIN_BUILD_ROWS
  exists_chain INNER + SHUFFLE(4) of both l_suppkey sides + GO_COMPARE(<>) + JOIN_COND(SEMI) per batch, the count of each probe read back
--parent-lib loads a second build of libmo_b200.so (another commit) and times every arm with it too (parent_*), on the same buffers,
alternating with this build's.  Every call that reads a result count back does so, as a caller must.  Prints one JSON line: the card and its
power limit, then the arms."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from matrixone_b200 import capi, ops  # noqa: E402
from matrixone_b200.vector import Vector  # noqa: E402

CMP_NE = 1


def dv(t, length=1, nbytes=None, nulls=None):
    return Vector(data_ptr=t.data_ptr(), data_nbytes=t.numel() * t.element_size() if nbytes is None else nbytes, length=length,
                  nulls_ptr=nulls.data_ptr() if nulls is not None else None)


def prm(jt):
    return Vector(data=np.array([jt, 0], np.int32).view(np.uint8), length=1)


def call(lib, fid, vecs, n):
    arr = (capi.XCallArgs * len(vecs))()
    for i, v in enumerate(vecs):
        arr[i] = v.fill_raw_ptr_len()
    err = (C.c_uint8 * 256)()
    rc = lib.XCall(1, fid, err, C.cast(arr, C.c_void_p), n)
    if rc:
        raise RuntimeError("XCall 0x%x rc=%d %s" % (fid, rc, bytes(err[1:1 + err[0]]).decode(errors="replace")))


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def alternate(arms, reps):
    """arms: {name: fn}; one warm-up each, then reps rounds in alternating order; median ms per arm"""
    for fn in arms.values():
        fn()
    times = {k: [] for k in arms}
    for r in range(reps):
        for k in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            times[k].append(timed(arms[k]))
    return {k: statistics.median(v) for k, v in times.items()}, {k: [round(x, 3) for x in v] for k, v in times.items()}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def lineitem(n, seed=21):
    """l_orderkey (1..7 rows per key, rows grouped by order as lineitem is) and l_suppkey of n rows"""
    r = np.random.default_rng(seed)
    per = r.integers(1, 8, n // 2 + 8)                     # more orders than n rows need
    norders = int(np.searchsorted(np.cumsum(per), n)) + 1
    okey = np.repeat(np.arange(1, norders + 1, dtype=np.int64) * 4, per[:norders])[:n]
    supp = r.integers(1, 100_001, n).astype(np.int32)
    return okey, supp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=60_000_000)
    ap.add_argument("--batch", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("join_cond_bench: no CUDA device")
    stream = torch.cuda.Stream()               # one stream for the libraries and the events
    libs = {"this": capi.load_library()}
    if a.parent_lib:
        libs["parent"] = capi.load_library(a.parent_lib)
    for lib in libs.values():
        capi.check(lib.MoB200_Init(0), lib)
        capi.check(lib.MoB200_SetStream(C.c_void_p(stream.cuda_stream)), lib)
    n, batch = a.rows, a.batch
    nbatches = (n + batch - 1) // batch
    okey, supp = lineitem(n)
    jm = ops.JoinMap(okey.astype(np.uint64))   # GROUP_IDS + JOIN_SELS + MoB200_JoinMapPrepare
    if "parent" in libs:
        capi.check(libs["parent"].MoB200_JoinMapPrepare(jm.table_keys.ctypes.data, jm.ngroups), libs["parent"])
    rec = {"card": card(), "torch": torch.__version__, "rows": n, "batch": batch, "groups": jm.ngroups}
    with torch.cuda.stream(stream):
        dkey, dsupp = torch.from_numpy(okey).cuda(), torch.from_numpy(supp).cuda()
        doff, dsels = torch.from_numpy(jm.offsets).cuda(), torch.from_numpy(jm.sels).cuda()
        cap = 8 * batch
        op, ob, cnt = torch.empty(cap, dtype=torch.int64, device="cuda"), torch.empty(cap, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
        ro, rb = torch.empty(cap, dtype=torch.int64, device="cuda"), torch.empty(cap, dtype=torch.int64, device="cuda")
        s1, s2 = torch.empty(cap, dtype=torch.int32, device="cuda"), torch.empty(cap, dtype=torch.int32, device="cuda")
        cond, cnull = torch.empty(cap, dtype=torch.uint8, device="cuda"), torch.zeros(cap // 64 + 1, dtype=torch.int64, device="cuda")
        matched = torch.zeros((n + 63) // 64, dtype=torch.int64, device="cuda")
        fsels, fcnt = torch.empty(n, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
        table = Vector(data=jm.table_keys, length=jm.ngroups)

        def bounds(b):
            lo = b * batch
            return lo, min(n, lo + batch) - lo

        def inner(lib, b):
            lo, m = bounds(b)
            call(lib, capi.XCALL_JOIN_PROBE, [dv(op), dv(ob), dv(cnt), prm(capi.JOIN_INNER), table, dv(doff, jm.ngroups + 2), dv(dsels),
                                              Vector(data_ptr=dkey.data_ptr() + 8 * lo, data_nbytes=8 * m, length=m)], m)
            return int(cnt.item())

        def condition(lib, k, lo, m, po, bo):
            """l_suppkey of the batch's rows (po: batch rows) <> l_suppkey of the build rows (bo) into cond / cnull"""
            call(lib, capi.XCALL_SHUFFLE(4), [dv(s1, k, 4 * k), Vector(data_ptr=dsupp.data_ptr() + 4 * lo, data_nbytes=4 * m, length=m),
                                              Vector(data_ptr=po.data_ptr(), data_nbytes=8 * k, length=k)], k)
            call(lib, capi.XCALL_SHUFFLE(4), [dv(s2, k, 4 * k), dv(dsupp, n), Vector(data_ptr=bo.data_ptr(), data_nbytes=8 * k, length=k)], k)
            cnull[:(k + 63) // 64].zero_()
            call(lib, capi.XCALL_GO_COMPARE(CMP_NE, capi.T_INT32), [dv(cond, k, k, cnull), dv(s1, k, 4 * k), dv(s2, k, 4 * k)], k)

        def join_cond(lib, jt, m, k, po, bo, c, cn):
            vecs = [dv(ro), dv(rb), dv(cnt), prm(jt), dv(po, k, 8 * k), dv(bo, k, 8 * k), dv(c, k, k, cn)]
            call(lib, capi.XCALL_JOIN_COND, vecs + ([dv(matched)] if jt >= capi.JOIN_RIGHT else []), m)

        # every batch's candidates and condition, kept for the cond_* arms
        kept, npairs = [], 0
        for b in range(nbatches):
            lo, m = bounds(b)
            k = inner(libs["this"], b)
            condition(libs["this"], k, lo, m, op[:k], ob[:k])
            kept.append((m, k, op[:k].clone(), ob[:k].clone(), cond[:k].clone(), cnull[:(k + 63) // 64].clone()))
            npairs += k
        torch.cuda.synchronize()
        rec["candidate_pairs"] = npairs

        def run_inner(lib):
            def run():
                for b in range(nbatches):
                    inner(lib, b)
            return run

        def run_cond(lib, jt):
            def run():
                if jt >= capi.JOIN_RIGHT:
                    matched.zero_()
                for m, k, po, bo, c, cn in kept:
                    join_cond(lib, jt, m, k, po, bo, c, cn)
                if jt >= capi.JOIN_RIGHT:
                    call(lib, capi.XCALL_JOIN_BUILD_ROWS, [dv(fsels, n), dv(fcnt), dv(matched), prm(jt)], n)
            return run

        def run_chain(lib):
            def run():
                for b in range(nbatches):
                    lo, m = bounds(b)
                    k = inner(lib, b)
                    condition(lib, k, lo, m, op[:k], ob[:k])
                    join_cond(lib, capi.JOIN_SEMI, m, k, op[:k], ob[:k], cond, cnull)
            return run

        arms = {}
        for name, lib in libs.items():
            pre = "" if name == "this" else name + "_"
            arms.update({pre + "inner": run_inner(lib), pre + "cond_semi": run_cond(lib, capi.JOIN_SEMI), pre + "cond_anti": run_cond(lib, capi.JOIN_ANTI),
                         pre + "cond_left": run_cond(lib, capi.JOIN_LEFT), pre + "cond_right+build_rows": run_cond(lib, capi.JOIN_RIGHT),
                         pre + "exists_chain": run_chain(lib)})
        med, raw = alternate(arms, a.reps)
        rec["arms"] = {k: {"ms": round(ms, 3), "probe_rows_per_s": n / (ms / 1e3), "runs_ms": raw[k]} for k, ms in med.items()}
    if "parent" in libs:
        libs["parent"].MoB200_JoinMapRelease(jm.table_keys.ctypes.data)
    for lib in libs.values():
        lib.MoB200_SetStream(None)
    jm.release()
    line = json.dumps(rec)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
