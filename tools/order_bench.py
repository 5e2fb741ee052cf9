#!/usr/bin/env python
"""ORDER BY / ORDER BY ... LIMIT (MO_XCALL_ORDER_SELS) against torch.sort(stable=True) and torch.topk on the same tensors, and JOIN_SELS on
this library against another build of it (--other-lib, e.g. the parent commit's; the fixed-width orders too, with their launch counts and
whether the sels are identical), one GPU, one process.  String keys (--only varlena): VARCHAR(25) `Customer#%09d` names (ORDER and Top 100),
random 8-100-byte TEXT, 1 KB TEXT with and without a common prefix, and the (l_returnflag, l_linestatus) pair, each beside the int64
torch.sort of the same row count; pyarrow.compute.sort_indices on the CPU when pyarrow is installed.

    python tools/order_bench.py [--rows N ...] [--runs R] [--other-lib PATH] [--only fixed|varlena]

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
    torch.cuda.synchronize()   # the columns are written on torch's stream; the library's own stream does not wait for it
    lib_t, yard_t = alternate(runs, warmup, lambda: lib_ms(lib, call), lambda: torch_ms(yard))
    ok = check(out[:nout]) if check else None
    del out
    torch.cuda.empty_cache()
    return {"case": name, "rows": n, "limit": limit, "lib_ms": round(lib_t, 3), "yardstick_ms": round(yard_t, 3),
            "lib_grows_s": round(n / lib_t / 1e6, 2), "yardstick_grows_s": round(n / yard_t / 1e6, 2), "checked": ok}


def order_ab(libs, name, cols, nulls, types, flags, n, limit, runs, warmup):
    """one fixed-width order on this build and on --other-lib, alternating: times, launch counts and whether the sels are identical"""
    nout = n if limit is None else limit
    outs = {tag: torch.empty(max(nout, 1), dtype=torch.int64, device="cuda") for tag, _ in libs}
    launches = {}

    def run(tag, L):
        vecs = [Vector(data_ptr=outs[tag].data_ptr(), data_nbytes=8 * nout, length=nout), ops._params_vec(ops._order_params(types, flags, limit, False))]
        for c, nl in zip(cols, nulls or [None] * len(cols)):
            vecs.append(Vector(data_ptr=c.ptr, data_nbytes=c.nbytes, nulls_ptr=nl.ptr if nl is not None else None, length=n))
        c0 = L.MoB200_KernelLaunchCount()
        ms = lib_ms(L, lambda: xcall(capi.XCALL_ORDER_SELS, vecs, n, lib=L))
        launches[tag] = L.MoB200_KernelLaunchCount() - c0
        return ms
    (t0, L0), (t1, L1) = libs
    a, b = alternate(runs, warmup, lambda: run(t0, L0), lambda: run(t1, L1))
    same = bool(torch.equal(outs[t0][:nout], outs[t1][:nout]))
    del outs
    torch.cuda.empty_cache()
    return {"case": name, "rows": n, "limit": limit, "this_ms": round(a, 3), "other_ms": round(b, 3), "this_launches": launches[t0],
            "other_launches": launches[t1], "identical_sels": same}


def customer_cells(ids):
    """VARCHAR(25) 'Customer#%09d' names as inline 24-byte cells, built on the device"""
    n = ids.numel()
    cells = torch.zeros((n, 24), dtype=torch.uint8, device="cuda")
    cells[:, 0] = 18
    cells[:, 1:10] = torch.tensor(list(b"Customer#"), dtype=torch.uint8, device="cuda")
    d = ids.clone()
    for j in range(9):
        cells[:, 18 - j] = (48 + d % 10).to(torch.uint8)
        d //= 10
    return cells


def area_cells(lens):
    """non-inline cells over one area: row i's value at offset sum(lens[:i]) mod 2^32 (the cell's offset field has 32 bits, so rows past
    4 GB of area read bytes of earlier rows; every cell stays inside the area), length lens[i]"""
    n = lens.numel()
    cells = torch.zeros((n, 6), dtype=torch.int32, device="cuda")
    cells[:, 0] = -1
    cells[:, 1] = (torch.cumsum(lens, 0) - lens).to(torch.int32)
    cells[:, 2] = lens.to(torch.int32)
    return cells.view(torch.uint8)


def varlena_cases(lib, res, a, g):
    """string keys: each case against the int64 torch.sort of the same row count, for scale"""
    def int64_sort(n):
        k = torch.randint(-2 ** 62, 2 ** 62, (n,), device="cuda", generator=g)
        return k, lambda: torch.sort(k, stable=True)

    def case(name, cols, types, flags, n, limit=None, check=None):
        k, yard = int64_sort(n)
        r = order_case(lib, name, cols, None, types, flags, n, limit, yard, a.runs, a.warmup, check)
        r["yardstick"] = "torch.sort int64, %d rows" % n
        res["cases"].append(r)
        del k

    n = a.varlena_rows
    ids = torch.randperm(n, device="cuda", generator=g) + 1
    cells = customer_cells(ids)
    want = torch.sort(ids, stable=True)[1]
    case("varchar25_customer_names", [(Dev(cells), None)], [capi.T_VARCHAR], [0], n, check=lambda s: bool(torch.equal(s, want)))
    case("varchar25_customer_names_top100", [(Dev(cells), None)], [capi.T_VARCHAR], [0], n, limit=100, check=lambda s: bool(torch.equal(s, want[:100])))
    del ids, cells, want
    torch.cuda.empty_cache()

    lens = torch.randint(8, 101, (n,), device="cuda", generator=g)
    area = torch.randint(0, 256, (int(lens.sum()),), device="cuda", dtype=torch.uint8, generator=g)
    cells = area_cells(lens)
    case("text_random_8_100_bytes", [(Dev(cells), Dev(area))], [capi.T_TEXT], [0], n)
    del lens, area, cells
    torch.cuda.empty_cache()

    n1k = a.kb_rows
    for prefix in (0, 16):
        area = torch.randint(0, 256, (n1k, 1000), device="cuda", dtype=torch.uint8, generator=g)
        if prefix:
            area[:, :prefix] = 0x41
        cells = area_cells(torch.full((n1k,), 1000, device="cuda", dtype=torch.int64))
        area = area.reshape(-1)
        case("text_1kb_common_prefix_%d" % prefix, [(Dev(cells), Dev(area))], [capi.T_TEXT], [0], n1k)
        del area, cells
        torch.cuda.empty_cache()

    n = a.flag_rows
    rf = torch.zeros((n, 24), dtype=torch.uint8, device="cuda")
    ls = torch.zeros((n, 24), dtype=torch.uint8, device="cuda")
    rf[:, 0] = 1
    ls[:, 0] = 1
    rf[:, 1] = torch.tensor(list(b"ANR"), dtype=torch.uint8, device="cuda")[torch.randint(0, 3, (n,), device="cuda", generator=g)]
    ls[:, 1] = torch.tensor(list(b"FO"), dtype=torch.uint8, device="cuda")[torch.randint(0, 2, (n,), device="cuda", generator=g)]
    case("returnflag_linestatus", [(Dev(rf), None), (Dev(ls), None)], [capi.T_VARCHAR, capi.T_VARCHAR], [0, 0], n)
    del rf, ls
    torch.cuda.empty_cache()
    res["pyarrow"] = pyarrow_sort(a.varlena_rows // 10)


def pyarrow_sort(n):
    """pyarrow.compute.sort_indices over Customer#%09d strings on the CPU, when pyarrow is installed"""
    try:
        import time

        import numpy as np
        import pyarrow as pa
        import pyarrow.compute as pc
    except ImportError:
        return "not installed"
    ids = np.random.default_rng(1).permutation(n) + 1
    arr = pa.array(np.char.add("Customer#", np.char.zfill(ids.astype(str), 9)))
    t0 = time.perf_counter()
    pc.sort_indices(arr)
    return {"case": "varchar25_customer_names", "rows": n, "ms": round((time.perf_counter() - t0) * 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[100_000_000, 600_000_000])
    ap.add_argument("--top-rows", type=int, default=600_000_000)
    ap.add_argument("--join-rows", type=int, default=100_000_000)
    ap.add_argument("--varlena-rows", type=int, default=100_000_000)
    ap.add_argument("--kb-rows", type=int, default=10_000_000, help="rows of the 1 KB TEXT cases")
    ap.add_argument("--flag-rows", type=int, default=600_000_000, help="rows of the (l_returnflag, l_linestatus) case")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--other-lib", default=None, help="another build of libmo_b200.so to time JOIN_SELS and the fixed-width orders against")
    ap.add_argument("--only", choices=["fixed", "varlena"], default=None)
    a = ap.parse_args()
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    name, power = card()
    res = {"card": name, "power_limit": power, "runs": a.runs, "cases": []}
    g = torch.Generator(device="cuda").manual_seed(1)
    if a.only != "fixed":
        varlena_cases(lib, res, a, g)
        if a.only == "varlena":
            print(json.dumps(res))
            return
    if a.other_lib:
        other = capi.load_library(a.other_lib)
        capi.check(other.MoB200_Init(0), other)
        ab = [("this", lib), ("other", other)]
        res["fixed_width_ab"] = []
    for n in a.rows:
        if a.other_lib:
            k = torch.randint(-2 ** 62, 2 ** 62, (n,), device="cuda", generator=g)
            s = torch.randint(0, 1000, (n,), device="cuda", generator=g)
            d = torch.randint(8000, 11000, (n,), device="cuda", dtype=torch.int32, generator=g)
            res["fixed_width_ab"].append(order_ab(ab, "int64_uniform", [Dev(k)], None, [capi.T_INT64], [0], n, None, a.runs, a.warmup))
            res["fixed_width_ab"].append(order_ab(ab, "int64_small_range", [Dev(s)], None, [capi.T_INT64], [0], n, None, a.runs, a.warmup))
            res["fixed_width_ab"].append(order_ab(ab, "date_desc_int64", [Dev(d), Dev(k)], None, [capi.T_DATE, capi.T_INT64], [capi.ORDER_DESC, 0], n,
                                                  None, a.runs, a.warmup))
            res["fixed_width_ab"].append(order_ab(ab, "top100_int64", [Dev(k)], None, [capi.T_INT64], [0], n, 100, a.runs, a.warmup))
            del k, s, d
            torch.cuda.empty_cache()
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
