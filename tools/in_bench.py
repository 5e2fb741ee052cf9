#!/usr/bin/env python
"""IN / NOT IN on resident columns: MO_XCALL_GO_IN over INT32, INT64 and strings, one GPU, one process.

    python tools/in_bench.py [--rows N] [--runs R] [--out FILE]

Shapes over --rows rows (default 10^8): INT32 and INT64 with lists of m = 2, 8, 512 and 10^5 values (512 has its table in shared memory,
10^5 reads it from global memory, so both sides of the probe's budget are timed); CHAR values of up to 10 bytes, all inline, with m = 2 and
7 (Q12's l_shipmode IN ('FOB', 'TRUCK'), Q22's seven country codes); strings longer than 23 bytes (in the area) with m = 16.  About half of
the rows are in the list.  kernel_ms is the probe kernel (the library's CUDA events, MoB200_LastKernelMs); call_ms the whole call between
events on the library's stream, the set build included; build_ms the set-build kernel on its own, from a separate torch.profiler pass
(CUDA activities) over --runs calls per shape.  Medians of --runs runs after a warm-up of every shape.  Every shape's hit count is checked
against the count computed from the generated rows before anything is printed.  bytes = column + bool result + the result bitmap read and written
(+ the area bytes of the long strings), from the shapes; GB/s = bytes over kernel_ms next to the H100 SXM data-sheet HBM3 peak of 3.35 TB/s.
For m <= 16 the caller's alternative is timed on the same rows: m GO_COMPARE(==) calls and one MULTI_OR (alt_ms, between events).  The
card's name and power limit are read in the same call.  Strings are resident in chunks of 2^24 rows (32-bit area offsets), one call per chunk.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from matrixone_b200 import capi  # noqa: E402
from matrixone_b200.vector import Vector, varlena_bytes_column, xcall  # noqa: E402
from strpred_bench import Chunk, card  # noqa: E402

HBM_PEAK_BPS = 3.35e12
CHUNK = 1 << 24


def out_vecs(n, out, outn):
    return Vector(data_ptr=out.data_ptr(), data_nbytes=n, nulls_ptr=outn.data_ptr(), length=n)


class Fixed:
    def __init__(self, dt, n, m, g):
        self.T = capi.T_INT32 if dt == torch.int32 else capi.T_INT64
        self.w = 4 if dt == torch.int32 else 8
        self.n, self.m = n, m
        self.col = torch.randint(0, 2 * m, (n,), generator=g, device="cuda", dtype=dt)      # about half the rows hit
        self.vals = torch.randperm(2 * m, generator=g, device="cuda")[:m].to(dt)
        self.expected = int(torch.isin(self.col, self.vals).sum())
        self.out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        self.outn = torch.zeros((n + 63) // 64, dtype=torch.int64, device="cuda")
        self.bytes = n * (self.w + 1) + 2 * ((n + 63) // 64) * 8

    def calls(self, rows=None):
        n = rows or self.n
        return [(n, out_vecs(n, self.out, self.outn), Vector(data_ptr=self.col.data_ptr(), data_nbytes=self.w * n, length=n),
                 Vector(data_ptr=self.vals.data_ptr(), data_nbytes=self.w * self.m, length=self.m))]

    def compare(self, j, rows, res, resn):
        v = self.vals[j:j + 1]
        return xcall(capi.XCALL_GO_COMPARE(capi.CMP_EQ, self.T), [out_vecs(rows, res, resn), self.calls()[0][2],
                                                                   Vector(data_ptr=v.data_ptr(), data_nbytes=self.w, length=1)], rows)


class Strings:
    T = capi.T_CHAR

    def __init__(self, tmpl_in, tmpl_out, n, g):
        self.list = tmpl_in
        tmpl = tmpl_in + tmpl_out
        self.m = len(tmpl_in)
        self.chunks, left, self.expected = [], n, 0
        while left:
            k = min(CHUNK, left)
            idx = torch.randint(len(tmpl), (k,), generator=g, device="cuda")
            self.expected += int((idx < self.m).sum())
            self.chunks.append(Chunk(tmpl, idx))
            left -= k
        cells, area = varlena_bytes_column(tmpl_in)
        self.lcells = torch.from_numpy(cells).cuda()
        self.larea = torch.from_numpy(area).cuda() if area.size else None
        self.n = n
        self.bytes = sum(24 * c.n + c.area_read + c.n + 2 * ((c.n + 63) // 64) * 8 for c in self.chunks)

    def lvec(self):
        a = self.larea
        return Vector(data_ptr=self.lcells.data_ptr(), data_nbytes=24 * self.m, length=self.m, area_ptr=None if a is None else a.data_ptr(),
                      area_nbytes=0 if a is None else a.numel())

    def calls(self, rows=None):
        if rows:
            c = self.chunks[0]
            v = c.vec(); v.data_nbytes = 24 * rows; v.length = rows
            return [(rows, out_vecs(rows, c.out, c.outn), v, self.lvec())]
        return [(c.n, out_vecs(c.n, c.out, c.outn), c.vec(), self.lvec()) for c in self.chunks]


def build_ms(lib, shape, runs):
    """the set-build kernel's time per run of the shape (every chunk's build), the mean over `runs` runs, from torch.profiler's CUDA activities"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            run_in(lib, shape)
        torch.cuda.synchronize()
    ts = [e.time_range.elapsed_us() for e in prof.events() if "build" in e.name and ("go_in" in e.name or "in_str" in e.name)]
    if len(ts) != runs * len(shape.calls()):
        raise SystemExit("in_bench: the profiler saw %d build kernels, %d expected" % (len(ts), runs * len(shape.calls())))
    return sum(ts) / runs / 1e3


def timed(lib, fn):
    capi.check(lib.MoB200_TimerStart(), lib)
    kms = fn()
    tot = C.c_float()
    capi.check(lib.MoB200_TimerStop(C.byref(tot)), lib)
    return kms, tot.value


def run_in(lib, shape, rows=None):
    kms = 0.0
    for n, out, col, lst in shape.calls(rows):
        xcall(capi.XCALL_GO_IN(shape.T), [out, col, lst, Vector(data=np.array([shape.m], np.int64))], n, lib=lib)
        ms = C.c_float()
        capi.check(lib.MoB200_LastKernelMs(C.byref(ms)), lib)
        kms += ms.value
    return kms


def run_alt(lib, shape, scratch):
    """m GO_COMPARE(==) calls and one MULTI_OR over their results, per chunk"""
    for n, out, col, lst in shape.calls():
        ops_ = []
        for j in range(shape.m):
            res, resn = scratch[j]
            if isinstance(shape, Fixed):
                shape.compare(j, n, res, resn)
            else:
                cells, area = varlena_bytes_column([shape.list[j]])
                xcall(capi.XCALL_GO_COMPARE(capi.CMP_EQ, capi.T_CHAR), [out_vecs(n, res, resn), col,
                      Vector(data=cells, area=area if area.size else None, length=1)], n, lib=lib)
            ops_.append(Vector(data_ptr=res.data_ptr(), data_nbytes=n, nulls_ptr=resn.data_ptr(), length=n))
        xcall(capi.XCALL_GO_MULTI_OR, [out, Vector(data=np.array([shape.m], np.int32))] + ops_, n, lib=lib)
    return 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("in_bench: no CUDA device (the measurement needs the H100)")
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    name, power = card()
    g = torch.Generator(device="cuda").manual_seed(1)
    n = a.rows
    modes = [b"FOB", b"TRUCK", b"MAIL", b"SHIP", b"RAIL", b"AIR", b"REG AIR"]
    codes = [b"%d" % c for c in (13, 31, 23, 29, 30, 18, 17)]
    longs = [b"long-string-value-number-%04d-padded" % i for i in range(32)]
    shapes = {}
    for dt, tn in ((torch.int32, "INT32"), (torch.int64, "INT64")):
        for m in (2, 8, 512, 100_000):
            shapes["%s m=%d" % (tn, m)] = Fixed(dt, n, m, g)
    shapes["CHAR m=2 (Q12 l_shipmode)"] = Strings(modes[:2], modes[2:], n, g)
    shapes["CHAR m=7 (Q22 country codes)"] = Strings(codes, [b"%d" % c for c in range(40, 47)], n, g)
    shapes["long strings m=16"] = Strings(longs[:16], longs[16:], n, g)
    max_chunk = max(min(CHUNK, n), n)
    scratch = [(torch.zeros(max_chunk, dtype=torch.uint8, device="cuda"), torch.zeros((max_chunk + 63) // 64, dtype=torch.int64, device="cuda"))
               for _ in range(16)]
    torch.cuda.synchronize()
    for s in shapes.values():                       # warm-up
        run_in(lib, s)
        if s.m <= 16:
            run_alt(lib, s, scratch)
    t = {k: {"k": [], "c": [], "alt": []} for k in shapes}
    for _ in range(a.runs):
        for k, s in shapes.items():
            kms, cms = timed(lib, lambda: run_in(lib, s))
            t[k]["k"].append(kms); t[k]["c"].append(cms)
            if s.m <= 16:
                t[k]["alt"].append(timed(lib, lambda: run_alt(lib, s, scratch))[1])
    res = {"card": name, "power_limit": power, "rows": n, "runs": a.runs, "hbm_peak_gbps": HBM_PEAK_BPS / 1e9, "shapes": {}}
    for k, s in shapes.items():
        km = statistics.median(t[k]["k"])
        run_in(lib, s)
        torch.cuda.synchronize()
        hits = int(s.out.sum()) if isinstance(s, Fixed) else sum(int(c.out.sum()) for c in s.chunks)
        if hits != s.expected:
            raise SystemExit("in_bench: %s found %d rows in the list, %d expected" % (k, hits, s.expected))
        r = {"kernel_ms": round(km, 3), "call_ms": round(statistics.median(t[k]["c"]), 3), "build_ms": round(build_ms(lib, s, a.runs), 4),
             "rows_per_s": round(n / (km * 1e-3) / 1e9, 2), "bytes": s.bytes, "gbps": round(s.bytes / (km * 1e-3) / 1e9, 1),
             "share_of_hbm_peak": round(s.bytes / (km * 1e-3) / HBM_PEAK_BPS, 3), "spread_ms": [round(min(t[k]["k"]), 3), round(max(t[k]["k"]), 3)],
             "hits": hits}
        if t[k]["alt"]:
            r["alt_ms"] = round(statistics.median(t[k]["alt"]), 3)
        res["shapes"][k] = r
        print("%-30s kernel %8.3f ms  call %8.3f ms  build %6.3f ms  %6.2f Grows/s  %7.1f GB/s  %.3f of HBM peak%s" % (
            k, km, r["call_ms"], r["build_ms"], r["rows_per_s"], r["gbps"], r["share_of_hbm_peak"],
            "  alt %8.3f ms" % r["alt_ms"] if "alt_ms" in r else ""))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
