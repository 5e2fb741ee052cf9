#!/usr/bin/env python
"""Right-flavoured hash joins and the NULL-row SHUFFLE on resident columns, timed with CUDA events (medians of alternating runs).

    python tools/join_outer_bench.py [--reps 5] [--parent-lib PATH] [--out FILE]

  probe_int   10^8 probe rows in 10^6-row JOIN_PROBE batches against a prepared 10^6-row unique map (about half the probe keys match):
              INNER; RIGHT + JOIN_BUILD_ROWS; RIGHT SEMI (a probe that emits nothing) + JOIN_BUILD_ROWS
  probe_str   10^7 probe rows of 16-byte string keys in 10^6-row batches: STR_JOIN_FIND + JOIN_PROBE_GIDS, INNER against RIGHT + finalize
  shuffle     SHUFFLE(8) and SHUFFLE(24) over 10^8 random sels (a tenth of them -1 in the `null_sels` rows), with a destination bitmap
--parent-lib loads a second build of libmo_b200.so (another commit) and times its probe arms (parent_*) and SHUFFLE (without -1 sels, which
it does not define) on the same buffers, alternating with this build's.  Every probe call reads its result count back, as a caller must.
Prints one JSON line per measurement and, first, the card and its power limit."""
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


def dv(t, length=1):
    return Vector(data_ptr=t.data_ptr(), data_nbytes=t.numel() * t.element_size(), length=length)


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


def adopt(lib, stream):
    capi.check(lib.MoB200_Init(0), lib)
    capi.check(lib.MoB200_SetStream(C.c_void_p(stream.cuda_stream)), lib)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def bench_probe_int(libs, reps, emit):
    nbuild, batch, nbatches = 1_000_000, 1_000_000, 100
    g = torch.Generator(device="cuda").manual_seed(1)
    build = torch.randperm(2 * nbuild, device="cuda", generator=g)[:nbuild].to(torch.int64)
    table_keys = build.cpu().numpy().view(np.uint64).copy()            # GROUP_IDS of distinct keys: group g + 1 is build row g
    keys = torch.randint(0, 2 * nbuild, (batch,), device="cuda", generator=g, dtype=torch.int64)
    words = (nbuild + 63) // 64
    matched = torch.zeros(words, dtype=torch.int64, device="cuda")
    cap = batch
    op, ob = torch.empty(cap, dtype=torch.int64, device="cuda"), torch.empty(cap, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    sels, scnt = torch.empty(nbuild, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    for lib in libs.values():
        capi.check(lib.MoB200_JoinMapPrepare(table_keys.ctypes.data, nbuild), lib)

    def probe(lib, jt):
        def run():
            if jt >= capi.JOIN_RIGHT:
                matched.zero_()
            for _ in range(nbatches):
                vecs = [dv(op), dv(ob), dv(cnt), prm(jt), Vector(data=table_keys, length=nbuild), Vector(length=0), Vector(length=0), dv(keys, batch)]
                call(lib, capi.XCALL_JOIN_PROBE, vecs + ([dv(matched)] if jt >= capi.JOIN_RIGHT else []), batch)
            if jt >= capi.JOIN_RIGHT:
                call(lib, capi.XCALL_JOIN_BUILD_ROWS, [dv(sels, nbuild), dv(scnt), dv(matched), prm(jt)], nbuild)
        return run

    arms = {}
    for name, lib in libs.items():
        pre = "" if name == "this" else name + "_"
        arms.update({pre + "inner": probe(lib, capi.JOIN_INNER), pre + "right+finalize": probe(lib, capi.JOIN_RIGHT),
                     pre + "right_semi+finalize": probe(lib, capi.JOIN_RIGHT_SEMI)})
    med, raw = alternate(arms, reps)
    rows = nbatches * batch
    for k, ms in med.items():
        emit({"bench": "probe_int", "arm": k, "build_rows": nbuild, "probe_rows": rows, "batch": batch, "ms": round(ms, 3),
              "probe_rows_per_s": rows / (ms / 1e3), "runs_ms": raw[k]})
    for lib in libs.values():
        lib.MoB200_JoinMapRelease(table_keys.ctypes.data)


def bench_probe_str(libs, reps, emit):
    nbuild, batch, nbatches = 1_000_000, 1_000_000, 10
    r = np.random.default_rng(2)
    bkeys = r.permutation(2 * nbuild)[:nbuild]
    pkeys = r.integers(0, 2 * nbuild, batch)
    bb = np.frombuffer(b"".join(b"key-%012d" % k for k in bkeys.tolist()), np.uint8)       # 16 bytes each
    pb = np.frombuffer(b"".join(b"key-%012d" % k for k in pkeys.tolist()), np.uint8)
    bo, po = np.arange(nbuild + 1, dtype=np.uint64) * 16, np.arange(batch + 1, dtype=np.uint64) * 16
    jm = ops.StrJoinMap(bb, bo)
    dpb, dpo = torch.from_numpy(pb.copy()).cuda(), torch.from_numpy(po.view(np.int64).copy()).cuda()
    dtb, dto = torch.from_numpy(jm.table_bytes.copy()).cuda(), torch.from_numpy(jm.table_offsets.view(np.int64).copy()).cuda()
    vals = torch.empty(batch, dtype=torch.int64, device="cuda")
    op, ob, cnt = torch.empty(batch, dtype=torch.int64, device="cuda"), torch.empty(batch, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    matched = torch.zeros((nbuild + 63) // 64, dtype=torch.int64, device="cuda")
    sels, scnt = torch.empty(nbuild, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    ng = Vector(data=np.array([jm.ngroups], np.int64), length=1)
    for lib in libs.values():
        capi.check(lib.MoB200_StrJoinMapPrepare(C.c_void_p(dtb.data_ptr()), C.c_void_p(dto.data_ptr()), jm.ngroups), lib)

    def probe(lib, jt):
        def run():
            if jt >= capi.JOIN_RIGHT:
                matched.zero_()
            for _ in range(nbatches):
                call(lib, capi.XCALL_STR_JOIN_FIND, [dv(vals, batch), ng, dv(dtb), dv(dto), dv(dpb), dv(dpo, batch)], batch)
                vecs = [dv(op), dv(ob), dv(cnt), prm(jt), ng, Vector(length=0), Vector(length=0), dv(vals, batch)]
                call(lib, capi.XCALL_JOIN_PROBE_GIDS, vecs + ([dv(matched)] if jt >= capi.JOIN_RIGHT else []), batch)
            if jt >= capi.JOIN_RIGHT:
                call(lib, capi.XCALL_JOIN_BUILD_ROWS, [dv(sels, nbuild), dv(scnt), dv(matched), prm(jt)], nbuild)
        return run

    arms = {}
    for name, lib in libs.items():
        pre = "" if name == "this" else name + "_"
        arms.update({pre + "inner": probe(lib, capi.JOIN_INNER), pre + "right+finalize": probe(lib, capi.JOIN_RIGHT)})
    med, raw = alternate(arms, reps)
    for k, ms in med.items():
        emit({"bench": "probe_str16", "arm": k, "build_rows": nbuild, "probe_rows": nbatches * batch, "ms": round(ms, 3),
              "probe_rows_per_s": nbatches * batch / (ms / 1e3), "runs_ms": raw[k]})
    for lib in libs.values():
        lib.MoB200_JoinMapRelease(C.c_void_p(dto.data_ptr()))
    jm.release()


def bench_shuffle(libs, reps, emit):
    n = 100_000_000
    g = torch.Generator(device="cuda").manual_seed(3)
    sels = torch.randint(0, n, (n,), device="cuda", generator=g, dtype=torch.int64)
    null_sels = sels.clone()
    null_sels[torch.rand(n, device="cuda", generator=g) < 0.1] = -1
    dn = torch.empty((n + 63) // 64, dtype=torch.int64, device="cuda")
    for sz in (8, 24):
        src = torch.empty(n * sz, dtype=torch.uint8, device="cuda").random_(generator=g)
        dst = torch.empty(n * sz, dtype=torch.uint8, device="cuda")
        sn = torch.zeros((n + 63) // 64, dtype=torch.int64, device="cuda")

        def shuffle(lib, s):
            return lambda: call(lib, capi.XCALL_SHUFFLE(sz), [Vector(data_ptr=dst.data_ptr(), data_nbytes=n * sz, nulls_ptr=dn.data_ptr(), length=n),
                                                               Vector(data_ptr=src.data_ptr(), data_nbytes=n * sz, nulls_ptr=sn.data_ptr(), length=n), dv(s, n)], n)
        arms = {"this": shuffle(libs["this"], sels), "this_null_sels": shuffle(libs["this"], null_sels)}
        if "parent" in libs:
            arms["parent"] = shuffle(libs["parent"], sels)
        med, raw = alternate(arms, reps)
        for k, ms in med.items():
            emit({"bench": "shuffle", "sz": sz, "arm": k, "sels": n, "ms": round(ms, 3),
                  "algorithmic_GB_per_s": n * (8 + 2 * sz) / (ms / 1e3) / 1e9, "runs_ms": raw[k]})
        del src, dst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default=None, choices=["probe_int", "probe_str", "shuffle"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("join_outer_bench: no CUDA device")
    # one stream for the libraries and the events: the default stream would hand each library back its own, which the events do not see
    stream = torch.cuda.Stream()
    libs = {"this": capi.load_library()}
    if a.parent_lib:
        libs["parent"] = capi.load_library(a.parent_lib)
    for lib in libs.values():
        adopt(lib, stream)
    out = open(a.out, "w") if a.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
    emit({"card": card(), "torch": torch.__version__})
    with torch.cuda.stream(stream):
        for name, fn in (("probe_int", bench_probe_int), ("probe_str", bench_probe_str), ("shuffle", bench_shuffle)):
            if a.only in (None, name):
                fn(libs, a.reps, emit)
    for lib in libs.values():
        lib.MoB200_SetStream(None)


if __name__ == "__main__":
    main()
