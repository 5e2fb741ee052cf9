#!/usr/bin/env python
"""TPC-H Q6 over DECIMAL(15,2) columns against the float64 columns of the same rows, one GPU, one process.

    python tools/tpch_decimal_bench.py [--rows N] [--runs R] [--warmup W] [--seed S]

lineitem is generated on the device (MoB200_GenLineitem, SF100 rows by default) and its measures are converted to Decimal64 cents on the
device in chunks: round(x * 100) is exact for this generator (checked against datagen on a sample).  The float64 and the decimal calls
alternate on resident columns (synchronous calls, host result).  Two times per call, medians of --runs: the CUDA-event time of the scan kernel
(MoB200_LastKernelMs), and the whole call -- every launch, the decimal call's bound check and fold included, and the result copy --
between CUDA events on the library's stream (MoB200_TimerStart / TimerStop).  The decimal call is also timed once its magnitude bound
fails, so that it walks every row for the row-order overflow check (dec_rare_path_call_ms).  Each
decimal result is checked against the float64 one (relative 1e-9) and against the previous decimal run (identical bytes).  Prints one
JSON line with the card name and power limit beside the numbers.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tpch_decimal_reference as R  # noqa: E402
from matrixone_b200 import capi, datagen, ops  # noqa: E402
from matrixone_b200.vector import Vector, xcall  # noqa: E402

SF100_ROWS = 600_037_902
Q6_BYTES_PER_ROW = 28


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:  # the numbers still stand; say what is missing
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def vec(t):
    return Vector(data_ptr=t.data_ptr(), data_nbytes=t.numel() * t.element_size(), length=t.numel())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=SF100_ROWS)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=10)
    a = ap.parse_args()
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    n = a.rows
    dev = torch.device("cuda", 0)
    sd = torch.empty(n, dtype=torch.int32, device=dev)
    f64 = {k: torch.empty(n, dtype=torch.float64, device=dev) for k in ("quantity", "extendedprice", "discount")}
    capi.check(lib.MoB200_GenLineitem(a.seed, 0, n, sd.data_ptr(), f64["quantity"].data_ptr(), f64["extendedprice"].data_ptr(),
                                      f64["discount"].data_ptr(), None, None, None), lib)
    dec = {}
    step = 1 << 26
    for k, t in f64.items():
        out = torch.empty(n, dtype=torch.int64, device=dev)
        for r in range(0, n, step):
            out[r:r + step] = torch.round(t[r:r + step] * 100).to(torch.int64)
        dec[k] = out
    torch.cuda.synchronize()
    sample = min(n, 1 << 20)
    ref = R.lineitem_dec(a.seed, 0, sample)
    for k in dec:
        assert np.array_equal(dec[k][:sample].cpu().numpy(), ref[k]), k

    P = datagen.q6_params()
    PD = R.q6_dec_params()
    fargs = [vec(sd), vec(f64["discount"]), vec(f64["quantity"]), vec(f64["extendedprice"])]
    dargs = [vec(sd), vec(dec["discount"]), vec(dec["quantity"]), vec(dec["extendedprice"])]

    def run_f64():
        return ops.q6_filter_sum(*fargs, n, *P)

    def run_dec():
        res = np.zeros(ops.Q6_DEC_RESULT_BYTES, dtype=np.uint8)
        xcall(capi.XCALL_Q6_DEC_FILTER_SUM, [Vector(data=res, length=1)] + dargs +
              [ops._params_vec(capi.Q6DecParams(*PD[:5], PD[5], 0))], n)
        return res.tobytes()

    def kernel_ms():
        ms = C.c_float()
        capi.check(lib.MoB200_LastKernelMs(C.byref(ms)), lib)
        return ms.value

    def timed(call):
        """(result, scan-kernel ms, whole-call ms): the call's every launch and its result copy, CUDA events on the library's stream"""
        capi.check(lib.MoB200_TimerStart(), lib)
        r = call()
        k = kernel_ms()
        ms = C.c_float()
        capi.check(lib.MoB200_TimerStop(C.byref(ms)), lib)
        return r, k, ms.value

    times = {"f64": [], "dec": []}
    calls = {"f64": [], "dec": []}
    prev = None
    for i in range(a.warmup + a.runs):
        f, tf, cf = timed(run_f64)
        raw, td, cd = timed(run_dec)
        d = ops.q6_dec_result_from_bytes(raw)
        assert d["rc"] == 0 and d["count"] == f[1], (d, f)
        exact = d["revenue"] / 10 ** d["scale"]
        assert abs(exact - f[0]) <= 1e-9 * abs(exact), (exact, f[0])
        assert prev is None or raw == prev
        prev = raw
        if i >= a.warmup:
            times["f64"].append(tf)
            times["dec"].append(td)
            calls["f64"].append(cf)
            calls["dec"].append(cd)
    # The rare path: one row with a product near 2^124 (discount and price 2^62, the discount range opened to every value) lifts the magnitude
    # bound over 2^127 / rows, so the call also walks every row in row order; no running sum overflows.
    r = int(np.flatnonzero((ref["shipdate"] >= PD[0]) & (ref["shipdate"] < PD[1]) & (ref["quantity"] < PD[4]))[0])   # a row the scan keeps
    disc0, price0 = int(dec["discount"][r]), int(dec["extendedprice"][r])
    dec["discount"][r] = 1 << 62
    dec["extendedprice"][r] = 1 << 62
    wide = capi.Q6DecParams(PD[0], PD[1], -(1 << 63), (1 << 63) - 1, PD[4], PD[5], 0)
    rare = []
    for i in range(3):
        capi.check(lib.MoB200_TimerStart(), lib)
        res = np.zeros(ops.Q6_DEC_RESULT_BYTES, dtype=np.uint8)
        xcall(capi.XCALL_Q6_DEC_FILTER_SUM, [Vector(data=res, length=1)] + dargs + [ops._params_vec(wide)], n)
        ms = C.c_float()
        capi.check(lib.MoB200_TimerStop(C.byref(ms)), lib)
        got = ops.q6_dec_result_from_bytes(res.tobytes())
        assert got["rc"] == 0 and got["revenue"] >> 120, got      # the big product is in the sum: the bound failed and the walk ran
        rare.append(ms.value)
    dec["discount"][r], dec["extendedprice"][r] = disc0, price0
    name, power = card()
    out = {"workload": "tpch_q6_decimal_vs_f64", "rows": n, "runs": a.runs, "gpu": name, "power_limit": power,
           "bytes_per_row": Q6_BYTES_PER_ROW, "revenue": str(d["revenue"]), "revenue_scale": d["scale"], "qualifying_rows": d["count"]}
    for k, ts in times.items():
        ms = statistics.median(ts)
        out[k] = {"kernel_ms_median": round(ms, 4), "kernel_ms_min": round(min(ts), 4), "kernel_ms_max": round(max(ts), 4),
                  "rows_per_s": n / (ms * 1e-3), "algorithmic_GB_per_s": n * Q6_BYTES_PER_ROW / (ms * 1e-3) / 1e9,
                  "call_ms_median": round(statistics.median(calls[k]), 4)}
    out["dec_over_f64_time"] = round(out["dec"]["kernel_ms_median"] / out["f64"]["kernel_ms_median"], 4)
    out["dec_rare_path_call_ms"] = round(statistics.median(rare[1:]), 3)
    out["dec_over_f64_call_time"] = round(out["dec"]["call_ms_median"] / out["f64"]["call_ms_median"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
