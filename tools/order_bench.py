#!/usr/bin/env python
"""ORDER BY / ORDER BY ... LIMIT (MO_XCALL_ORDER_SELS) against torch.sort(stable=True) and torch.topk on the same tensors, and JOIN_SELS on
this library against another build of it (--other-lib, e.g. the parent commit's), one GPU, one process.

    python tools/order_bench.py [--rows N ...] [--runs R] [--other-lib PATH]

Every case alternates the library call and its yardstick --runs times after --warmup rounds and reports medians of the time between CUDA
events on the library's stream (asynchronous form on resident columns, then a synchronise), and G rows/s.  Results are checked once per case:
the library's sels against the yardstick's indices (single key) or against the full order's prefix (Top).  Prints one JSON line with the
card name and power limit beside the numbers.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from matrixone_b200 import capi, ops  # noqa: E402
from matrixone_b200.vector import Vector, xcall  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


class Dev:
    """a torch tensor seen as a DeviceBuffer by ops.order_sels_device"""

    def __init__(self, t):
        self.t, self.ptr, self.nbytes = t, t.data_ptr(), t.numel() * t.element_size()


def lib_ms(lib, fn):
    capi.check(lib.MoB200_TimerStart(), lib)
    fn()
    ms = C.c_float()
    capi.check(lib.MoB200_TimerStop(C.byref(ms)), lib)
    return ms.value


def torch_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def alternate(runs, warmup, fa, fb):
    ta, tb = [], []
    for i in range(warmup + runs):
        x, y = fa(), fb()
        if i >= warmup:
            ta.append(x)
            tb.append(y)
    return statistics.median(ta), statistics.median(tb)


def order_case(lib, name, cols, nulls, types, flags, n, limit, yard, runs, warmup, check):
    nout = n if limit is None else limit
    out = torch.empty(max(nout, 1), dtype=torch.int64, device="cuda")
    call = lambda: ops.order_sels_device(cols, nulls, types, flags, n, out.data_ptr(), limit=limit)  # noqa: E731
    lib_t, yard_t = alternate(runs, warmup, lambda: lib_ms(lib, call), lambda: torch_ms(yard))
    ok = check(out[:nout]) if check else None
    del out
    torch.cuda.empty_cache()
    return {"case": name, "rows": n, "limit": limit, "lib_ms": round(lib_t, 3), "yardstick_ms": round(yard_t, 3),
            "lib_grows_s": round(n / lib_t / 1e6, 2), "yardstick_grows_s": round(n / yard_t / 1e6, 2), "checked": ok}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[100_000_000, 600_000_000])
    ap.add_argument("--top-rows", type=int, default=600_000_000)
    ap.add_argument("--join-rows", type=int, default=100_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--other-lib", default=None, help="another build of libmo_b200.so to time JOIN_SELS against")
    a = ap.parse_args()
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    name, power = card()
    res = {"card": name, "power_limit": power, "runs": a.runs, "cases": []}
    g = torch.Generator(device="cuda").manual_seed(1)
    for n in a.rows:
        for kind in ("uniform", "small_range"):
            k = torch.randint(-2 ** 62, 2 ** 62, (n,), device="cuda", generator=g) if kind == "uniform" else torch.randint(0, 1000, (n,), device="cuda", generator=g)
            yard = lambda: torch.sort(k, stable=True)  # noqa: E731
            chk = lambda s: bool(torch.equal(s, torch.sort(k, stable=True)[1]))  # noqa: E731
            res["cases"].append(order_case(lib, "int64_" + kind, [Dev(k)], None, [capi.T_INT64], [0], n, None, yard, a.runs, a.warmup, chk))
            del k
        f = torch.randn(n, device="cuda", dtype=torch.float64, generator=g)
        res["cases"].append(order_case(lib, "float64", [Dev(f)], None, [capi.T_FLOAT64], [0], n, None, lambda: torch.sort(f, stable=True),
                                       a.runs, a.warmup, lambda s: bool(torch.equal(s, torch.sort(f, stable=True)[1]))))
        del f
        d = torch.randint(8000, 11000, (n,), device="cuda", dtype=torch.int32, generator=g)
        m = torch.randint(1, 10 ** 8, (n,), device="cuda", generator=g)
        nw = (n + 63) // 64
        dn = torch.randint(-2 ** 62, 2 ** 62, (nw,), device="cuda", generator=g) & torch.randint(-2 ** 62, 2 ** 62, (nw,), device="cuda", generator=g)
        mn = torch.zeros(nw, dtype=torch.int64, device="cuda")
        res["cases"].append(order_case(lib, "date_desc_decimal64_nullable", [Dev(d), Dev(m)], [Dev(dn), Dev(mn)], [capi.T_DATE, capi.T_DECIMAL64],
                                       [capi.ORDER_DESC, 0], n, None, lambda: torch.sort(m, stable=True), a.runs, a.warmup, None))
        del d, m, dn, mn
        torch.cuda.empty_cache()
    n = a.top_rows
    k = torch.randint(-2 ** 62, 2 ** 62, (n,), device="cuda", generator=g)
    for limit in (10, 100, 10_000):
        def chk(s, limit=limit):
            return bool(torch.equal(k[s], torch.topk(k, limit, largest=False, sorted=True)[0]))
        res["cases"].append(order_case(lib, "top_int64", [Dev(k)], None, [capi.T_INT64], [0], n, limit,
                                       lambda limit=limit: torch.topk(k, limit, largest=False, sorted=True), a.runs, a.warmup, chk))
    del k
    torch.cuda.empty_cache()

    # JOIN_SELS: this build against --other-lib, the same groups, alternating
    n = a.join_rows
    ng = n // 10
    groups = torch.randint(1, ng + 1, (n,), device="cuda", generator=g)
    libs = [("this", lib)]
    if a.other_lib:
        other = capi.load_library(a.other_lib)
        capi.check(other.MoB200_Init(0), other)
        libs.append(("other", other))
    outs = {}
    for tag, L in libs:
        off = torch.empty(ng + 2, dtype=torch.int32, device="cuda")
        vals = torch.empty(n, dtype=torch.int32, device="cuda")
        cnt = torch.empty(1, dtype=torch.int64, device="cuda")
        outs[tag] = (L, off, vals, cnt)

    def join(tag):
        L, off, vals, cnt = outs[tag]
        vecs = [Vector(data_ptr=off.data_ptr(), data_nbytes=4 * (ng + 2), length=ng + 2), Vector(data_ptr=vals.data_ptr(), data_nbytes=4 * n, length=n),
                Vector(data_ptr=cnt.data_ptr(), data_nbytes=8, length=1), Vector(data_ptr=groups.data_ptr(), data_nbytes=8 * n, length=n)]
        return lib_ms(L, lambda: xcall(capi.XCALL_JOIN_SELS, vecs, n, lib=L))

    if len(libs) == 2:
        t_this, t_other = alternate(a.runs, a.warmup, lambda: join("this"), lambda: join("other"))
        same = bool(torch.equal(outs["this"][1], outs["other"][1]) and torch.equal(outs["this"][2], outs["other"][2]))
        res["join_sels"] = {"rows": n, "groups": ng, "this_ms": round(t_this, 3), "other_ms": round(t_other, 3), "identical": same}
    else:
        t_this = statistics.median([join("this") for _ in range(a.warmup + a.runs)][a.warmup:])
        res["join_sels"] = {"rows": n, "groups": ng, "this_ms": round(t_this, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
