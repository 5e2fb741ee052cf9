#!/usr/bin/env python
"""CASE, COALESCE and CASE_SELECT on resident columns (csrc/caseexpr.cu), one GPU, one process.

    python tools/case_bench.py [--rows N] [--runs R] [--out FILE]

Shapes over --rows rows (default 10^8), conditions true on about half the rows:
  q12        CASE WHEN c THEN 1 ELSE 0 END, INT64, const branches (Q12's sum(case ...) argument)
  when3      three WHENs and an ELSE over INT64 columns
  q14        CASE WHEN c THEN v ELSE 0 END, DECIMAL128, v a column and ELSE a const (Q14's revenue argument)
  coalesce   COALESCE(a, b), INT64, a 50% NULL
  str_inline CASE WHEN c THEN a ELSE b END, VARCHAR, 10-byte values (inline)
  str_40     the same with 40-byte values (in the area)
  select     CASE_SELECT over one condition
kernel_ms is the call's main kernel between the library's CUDA events (MoB200_LastKernelMs; the strings: the write kernel); call_ms the
whole call between CUDA events on the library's stream (the strings: pick, scan, the read-back and write).  bytes are computed from the
shape: each operand row the call must read once, the result written once and the bitmap read and written; GB/s = bytes over call_ms,
next to the H100 SXM data-sheet HBM3 peak of 3.35 TB/s.  The fixed-width shapes also time torch.where over the same tensors (nested for
when3), the yardstick of a plain select.  Medians of --runs runs, ours and torch.where alternating, after one warm-up.  Each JSON line
carries the card's name and power limit, read in the same process."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from matrixone_b200 import capi  # noqa: E402
from matrixone_b200.vector import Vector, xcall  # noqa: E402
from strpred_bench import card  # noqa: E402

HBM_PEAK_BPS = 3.35e12


def dv(t, rows, nulls=None, area=None):
    """a Vector over a torch tensor (one element's bytes = const)"""
    return Vector(data_ptr=t.data_ptr(), data_nbytes=t.numel() * t.element_size(), nulls_ptr=None if nulls is None else nulls.data_ptr(),
                  length=rows, area_ptr=None if area is None else area.data_ptr(), area_nbytes=0 if area is None else area.numel())


def params(nsel, has_else):
    return Vector(data=np.frombuffer(bytes(capi.CaseParams(nsel, has_else, 0)), np.uint8).copy(), length=1)


def bits(g, n, p):
    b = torch.rand(((n + 63) // 64) * 64, generator=g, device="cuda") < p
    w = torch.zeros(b.numel() // 8, dtype=torch.uint8, device="cuda")
    b8 = b.view(-1, 8).to(torch.uint8)
    for k in range(8):
        w |= b8[:, k] << k
    return w.view(torch.int64)


def str_col(g, n, width):
    cells = torch.zeros((n, 24), dtype=torch.uint8, device="cuda")
    if width <= 23:
        cells[:, 0] = width
        cells[:, 1:1 + width] = torch.randint(32, 127, (n, width), generator=g, device="cuda", dtype=torch.uint8)
        return cells, None
    area = torch.randint(32, 127, (n * width,), generator=g, device="cuda", dtype=torch.uint8)
    u32 = cells.view(torch.int32)
    u32[:, 0] = -1
    u32[:, 1] = (torch.arange(n, device="cuda", dtype=torch.int64) * width).to(torch.int64).bitwise_and(0xffffffff).to(torch.int32)
    u32[:, 2] = width
    return cells, area


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10 ** 8)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.rows
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(-1), lib)
    name, power = card()
    g = torch.Generator(device="cuda").manual_seed(1)
    w = (n + 63) // 64
    rn = torch.zeros(w, dtype=torch.int64, device="cuda")
    c = [(torch.rand(n, generator=g, device="cuda") < p).to(torch.uint8) for p in (0.5, 0.3, 0.4)]
    x = [torch.randint(-10 ** 12, 10 ** 12, (n,), generator=g, device="cuda", dtype=torch.int64) for _ in range(4)]
    masks = [x.bool() for x in c]                        # torch.where's masks, made once outside the timing
    one, zero = torch.ones(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    out8 = torch.empty(n, dtype=torch.int64, device="cuda")
    bmw = 2 * w * 8                                   # the result bitmap, read and written

    shapes = {}

    def case_fixed(T, vecs, nsel, has_else, out, width, coalesce=False):
        fid = capi.XCALL_GO_COALESCE(T) if coalesce else capi.XCALL_GO_CASE(T)
        res = Vector(data_ptr=out.data_ptr(), data_nbytes=width * n, nulls_ptr=rn.data_ptr(), length=n)
        return lambda: xcall(fid, [res, params(nsel, has_else)] + vecs, n)

    shapes["q12"] = (case_fixed(capi.T_INT64, [dv(c[0], n), dv(one, n), dv(zero, n)], 1, 1, out8, 8), n * (1 + 8) + bmw,
                     lambda: torch.where(masks[0], one, zero))
    shapes["when3"] = (case_fixed(capi.T_INT64, [dv(c[0], n), dv(x[0], n), dv(c[1], n), dv(x[1], n), dv(c[2], n), dv(x[2], n), dv(x[3], n)], 3, 1,
                                  out8, 8), n * (3 + 8 + 8) + bmw,
                       lambda: torch.where(masks[0], x[0], torch.where(masks[1], x[1], torch.where(masks[2], x[2], x[3]))))
    v16 = torch.randint(-10 ** 12, 10 ** 12, (n, 2), generator=g, device="cuda", dtype=torch.int64)
    z16 = torch.zeros((1, 2), dtype=torch.int64, device="cuda")
    cb0_col = masks[0][:, None]
    out16 = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    shapes["q14"] = (case_fixed(capi.T_DECIMAL128, [dv(c[0], n), dv(v16, n), dv(z16, n)], 1, 1, out16, 16), n * (1 + 16 + 16) + bmw,
                     lambda: torch.where(cb0_col, v16, z16))
    an = bits(g, n, 0.5)
    an_bool = torch.rand(n, generator=g, device="cuda") < 0.5
    shapes["coalesce"] = (case_fixed(capi.T_INT64, [dv(x[0], n, an), dv(x[1], n)], 2, 0, out8, 8, coalesce=True), n * (8 + 8 + 8) + w * 8 + bmw,
                          lambda: torch.where(an_bool, x[1], x[0]))
    sel_then = torch.empty(w, dtype=torch.int64, device="cuda")
    sel_rem = torch.zeros(w, dtype=torch.int64, device="cuda")
    shapes["select"] = (lambda: xcall(capi.XCALL_GO_CASE_SELECT, [dv(sel_then, n), dv(sel_rem, n), dv(c[0], n)], n), n + 3 * w * 8, None)

    out_cells = torch.empty((n, 24), dtype=torch.uint8, device="cuda")
    for nm, width in (("str_inline", 10), ("str_40", 40)):
        (ca, aa), (cb, ab) = str_col(g, n, width), str_col(g, n, width)
        out_area = torch.empty(n * width if width > 23 else 1, dtype=torch.uint8, device="cuda")
        res = Vector(data_ptr=out_cells.data_ptr(), data_nbytes=24 * n, nulls_ptr=rn.data_ptr(), length=n, area_ptr=out_area.data_ptr(),
                     area_nbytes=out_area.numel())
        vecs = [res, params(1, 1), dv(c[0], n), dv(ca, n, area=aa), dv(cb, n, area=ab)]
        shapes[nm] = ((lambda vecs=vecs: xcall(capi.XCALL_GO_CASE(capi.T_VARCHAR), vecs, n)),
                      n * (1 + 24 + 24) + bmw + (2 * n * width if width > 23 else 0), None)
        shapes[nm + "_keep"] = (ca, aa, cb, ab, out_area)

    stream = torch.cuda.Stream()
    capi.check(lib.MoB200_SetStream(C.c_void_p(stream.cuda_stream)), lib)
    lines = []
    for nm, spec in shapes.items():
        if nm.endswith("_keep"):
            continue
        run, nbytes, ref = spec
        ours, kern, theirs = [], [], []
        for r in range(a.runs + 1):
            rn.zero_(); sel_rem.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                e0.record(stream)
                run()
                e1.record(stream)
            e1.synchronize()
            ms = C.c_float()
            capi.check(lib.MoB200_LastKernelMs(C.byref(ms)), lib)
            if ref is not None:
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record(); ref(); t1.record(); t1.synchronize()
            if r:
                ours.append(e0.elapsed_time(e1)); kern.append(ms.value)
                if ref is not None:
                    theirs.append(t0.elapsed_time(t1))
        call_ms = statistics.median(ours)
        rec = {"shape": nm, "rows": n, "card": name, "power_limit": power, "call_ms": round(call_ms, 4), "kernel_ms": round(statistics.median(kern), 4),
               "bytes": nbytes, "GBps": round(nbytes / call_ms / 1e6, 1), "hbm_share": round(nbytes / (call_ms * 1e-3) / HBM_PEAK_BPS, 3)}
        if theirs:
            rec["torch_where_ms"] = round(statistics.median(theirs), 4)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    capi.check(lib.MoB200_SetStream(None), lib)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
