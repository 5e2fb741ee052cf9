#!/usr/bin/env python
"""Decimal comparisons, division and AVG on resident columns, one GPU, one process.

    python tools/decimal_bench.py [--rows N] [--runs R] [--parent-lib PATH] [--out FILE]

Shapes, over --rows rows (default 10^8) of device-generated values: the int64 compare a > b and the decimal64 compare on the same bytes at
equal scales (2, 2) and at unequal scales (2, 4: every left value is scaled up), the decimal128 compare at (2, 2), DIV at scales (2, 2) for
decimal64 operands, for decimal128 operands with divisors below 2^64, and for decimal128 operands with divisors of 2^64 and above (the Div128
estimate-and-correct path), and DEC_AVG over --rows groups.  Every call is the asynchronous or single-read-back form on resident buffers.
kernel_ms is the library's CUDA events around the call's kernel (MoB200_LastKernelMs), a median of --runs runs alternating over the
shapes after one warm-up of each.  bytes = the operand bytes read + the result bytes written (bitmaps excluded); GB/s = bytes over
kernel_ms, next to the H100 SXM data-sheet HBM3 peak of 3.35 TB/s.  The card's name and power limit are read in the same call.
--parent-lib loads a second build of libmo_b200.so (another commit) and times every shape on it too (parent_*), alternating with this build
call by call, so that both see the same card state.
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from matrixone_b200 import capi  # noqa: E402
from matrixone_b200.vector import Vector, xcall  # noqa: E402

HBM_PEAK_BPS = 3.35e12


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
    name, power = (x.strip() for x in out.split(","))
    return name, power


def dvec(t, n, nulls=None):
    return Vector(data_ptr=t.data_ptr(), data_nbytes=t.numel() * t.element_size(), nulls_ptr=None if nulls is None else nulls.data_ptr(), length=n)


def params(struct):
    return Vector(data=np.frombuffer(bytes(struct), dtype=np.uint8).copy(), length=1, const=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decimal_bench: no CUDA device (the measurement needs the H100)")
    libs = {"": capi.load_library()}
    if a.parent_lib:
        libs["parent_"] = capi.load_library(a.parent_lib)
    for lib in libs.values():
        capi.check(lib.MoB200_Init(0), lib)
    name, power = card()
    n = a.rows
    g = torch.Generator(device="cuda").manual_seed(1)
    dev = "cuda"
    i64a = torch.randint(-10 ** 15, 10 ** 15, (n,), generator=g, device=dev, dtype=torch.int64)
    i64b = torch.randint(-10 ** 15, 10 ** 15, (n,), generator=g, device=dev, dtype=torch.int64)
    div64 = torch.randint(1, 10 ** 9, (n,), generator=g, device=dev, dtype=torch.int64)

    def d128(lo, hi):
        return torch.stack([lo, hi], dim=1).contiguous()
    d128a = d128(i64a, torch.where(i64a < 0, -1, 0))
    d128b = d128(i64b, torch.where(i64b < 0, -1, 0))
    d128_small_div = d128(div64, torch.zeros_like(div64))
    big_x = d128(torch.randint(0, 2 ** 62, (n,), generator=g, device=dev, dtype=torch.int64),
                 torch.randint(2 ** 30, 2 ** 35, (n,), generator=g, device=dev, dtype=torch.int64))
    big_y = d128(torch.randint(0, 2 ** 62, (n,), generator=g, device=dev, dtype=torch.int64),
                 torch.randint(1, 2 ** 20, (n,), generator=g, device=dev, dtype=torch.int64))
    cnts = torch.randint(1, 1000, (n,), generator=g, device=dev, dtype=torch.int64)
    res8 = torch.empty(n, dtype=torch.uint8, device=dev)
    res16 = torch.empty((n, 2), dtype=torch.int64, device=dev)
    rn = torch.zeros((n + 63) // 64, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()

    def cmp_call(fid, x, y, extra):
        def f(lib):
            rn.zero_()
            xcall(fid, [dvec(res8, n, rn), dvec(x, n), dvec(y, n)] + extra, n, lib=lib)
        return f

    def div_call(width, x, y):
        def f(lib):
            rn.zero_()
            xcall(capi.XCALL_DEC_ARITH(capi.DEC_OP_DIV, width), [dvec(res16, n, rn), dvec(x, n), dvec(y, n),
                                                                 params(capi.DecDivParams(2, 2, -1, 0, 0))], n, lib=lib)
        return f

    def avg_call(lib):
        xcall(capi.XCALL_DEC_AVG(64), [dvec(res16, n, rn), dvec(d128a, n), dvec(cnts, n), params(capi.DecParams(2, 0, -1))], n, lib=lib)

    shapes = [
        ("int64 compare a > b", cmp_call(capi.XCALL_GO_COMPARE(capi.CMP_GT, capi.T_INT64), i64a, i64b, []), 8 + 8 + 1),
        ("decimal64 compare, equal scales", cmp_call(capi.XCALL_GO_COMPARE(capi.CMP_GT, capi.T_DECIMAL64), i64a, i64b,
                                                      [params(capi.DecParams(2, 2, -1))]), 8 + 8 + 1),
        ("decimal64 compare, scales 2 / 4", cmp_call(capi.XCALL_GO_COMPARE(capi.CMP_GT, capi.T_DECIMAL64), i64a, i64b,
                                                      [params(capi.DecParams(2, 4, -1))]), 8 + 8 + 1),
        ("decimal128 compare, equal scales", cmp_call(capi.XCALL_GO_COMPARE(capi.CMP_GT, capi.T_DECIMAL128), d128a, d128b,
                                                       [params(capi.DecParams(2, 2, -1))]), 16 + 16 + 1),
        ("decimal64 div (64-bit divisor)", div_call(64, i64a, div64), 8 + 8 + 16),
        ("decimal128 div, 64-bit divisor", div_call(128, d128a, d128_small_div), 16 + 16 + 16),
        ("decimal128 div, 128-bit divisor", div_call(128, big_x, big_y), 16 + 16 + 16),
        ("DEC_AVG", avg_call, 16 + 8 + 16),
    ]
    times = {p + s[0]: [] for s in shapes for p in libs}

    def run(lib, f):
        f(lib)
        capi.check(lib.MoB200_Sync(), lib)
        ms = C.c_float()
        capi.check(lib.MoB200_LastKernelMs(C.byref(ms)), lib)
        return ms.value

    for _, f, _ in shapes:
        for lib in libs.values():
            run(lib, f)
    for _ in range(a.runs):
        for label, f, _ in shapes:
            for p, lib in libs.items():
                times[p + label].append(run(lib, f))
    res = {"card": name, "power_limit": power, "rows": n, "runs": a.runs, "hbm_peak_gbps": HBM_PEAK_BPS / 1e9, "shapes": {}}
    for label, per_row in ((p + s[0], s[2]) for s in shapes for p in libs):
        k = statistics.median(times[label])
        nbytes = per_row * n
        res["shapes"][label] = {"kernel_ms": round(k, 3), "g_rows_per_s": round(n / (k * 1e-3) / 1e9, 2), "bytes": nbytes,
                                "gbps": round(nbytes / (k * 1e-3) / 1e9, 1), "share_of_hbm_peak": round(nbytes / (k * 1e-3) / HBM_PEAK_BPS, 3),
                                "spread_ms": [round(min(times[label]), 3), round(max(times[label]), 3)]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
