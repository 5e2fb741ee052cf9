#!/usr/bin/env python
"""Byte-string keys on resident columns: PACK_STR_KEYS, STR_GROUP_IDS (one call, and 10^6-row batches on a persisting table) and
STR_JOIN_FIND (prepared against rebuilt), with 8-byte GROUP_IDS at the same cardinality for scale, one GPU, one process.

    python tools/strkey_bench.py [--rows N] [--runs R] [--out FILE]

Cases at --rows rows (default 10^8): VARCHAR(25) `Customer#%09d` keys with 10^6 and 10^7 distinct values; Q3-shaped (BIGINT, DATE, INT)
16-byte keys (has_null = 0) with 10^7 distinct values; GROUP_IDS over int64 keys with 10^7 distinct values; STR_JOIN_FIND of 10^7 probe rows
in 10^6-row batches against a 10^6-group build.  Every call is the asynchronous form on device pointers; times are the medians of --runs
alternating runs between CUDA events on the library's stream.  The card's name and power limit are read in the same call.
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

from matrixone_b200 import capi, ops  # noqa: E402
from matrixone_b200.vector import Vector, xcall  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
    name, power = (x.strip() for x in out.split(","))
    return name, power


class Dev:
    """a torch tensor seen as a DeviceBuffer"""

    def __init__(self, t):
        self.t, self.ptr, self.nbytes = t, t.data_ptr(), t.numel() * t.element_size()


def dev(shape, dtype):
    return Dev(torch.zeros(shape, dtype=dtype, device="cuda"))


def lib_ms(lib, fn):
    capi.check(lib.MoB200_TimerStart(), lib)
    fn()
    ms = C.c_float()
    capi.check(lib.MoB200_TimerStop(C.byref(ms)), lib)
    return ms.value


def name_cells(ids):
    """VARCHAR cells of b"Customer#%09d" % id: 18 bytes, inline"""
    n = ids.numel()
    cells = torch.zeros((n, 24), dtype=torch.uint8, device="cuda")
    cells[:, 0] = 18
    cells[:, 1:10] = torch.tensor(list(b"Customer#"), dtype=torch.uint8, device="cuda")
    for k in range(9):
        cells[:, 18 - k] = (ids // 10 ** k % 10 + 48).to(torch.uint8)
    return Dev(cells.reshape(-1))


def ready():
    """torch prepares the buffers on its own stream; the library runs on another one, with no order between them"""
    torch.cuda.synchronize()


def set_ngroups(ng, v):
    ng.t.fill_(v)
    ready()


def group_call(kb, ko, n, groups, ng, tb, to):
    xcall(capi.XCALL_STR_GROUP_IDS, [Vector(data_ptr=groups.ptr, data_nbytes=8 * n, length=n), Vector(data_ptr=ng.ptr, data_nbytes=8, length=1),
                                     Vector(data_ptr=tb.ptr, data_nbytes=tb.nbytes, length=1), Vector(data_ptr=to.ptr, data_nbytes=to.nbytes, length=1),
                                     Vector(data_ptr=kb.ptr, data_nbytes=kb.nbytes, length=n), Vector(data_ptr=ko.ptr, data_nbytes=8 * (n + 1), length=n),
                                     Vector(length=0)], n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--batch", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("strkey_bench: no CUDA device (the measurement needs the H100)")
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    name, power = card()
    n, B = a.rows, min(a.batch, a.rows)
    res = {"card": name, "power_limit": power, "rows": n, "runs": a.runs}
    g = torch.Generator(device="cuda").manual_seed(1)

    def med(fns):
        """fns: {label: callable}; alternating runs, one warm-up each; medians in ms"""
        t = {k: [] for k in fns}
        for r in range(a.runs + 1):
            for k, f in fns.items():
                ms = f()
                if r:
                    t[k].append(ms)
        return {k: round(statistics.median(v), 3) for k, v in t.items()}

    groups, ng = dev(n, torch.int64), dev(1, torch.int64)
    for D in (1_000_000, 10_000_000):
        ids = torch.randint(0, D, (n,), device="cuda", generator=g)
        cells = name_cells(ids)
        del ids
        kb, ko = dev(21 * n, torch.uint8), dev(n + 1, torch.int64)
        tb, to = dev(21 * D + 64, torch.uint8), dev(D + 1, torch.int64)
        ready()
        pack = lambda: lib_ms(lib, lambda: ops.pack_str_keys_device([(cells, None)], None, [capi.T_VARCHAR], n, kb, ko))   # noqa: E731
        subs = []

        def one():
            set_ngroups(ng, 0)
            return lib_ms(lib, lambda: group_call(kb, ko, n, groups, ng, tb, to))

        def batches():
            if not subs:                                 # each batch's offsets rebased to 0, once (the keys are packed by then)
                subs.extend((Dev(kb.t[21 * s:21 * (s + min(B, n - s))]), Dev(ko.t[s:s + min(B, n - s) + 1] - ko.t[s]), min(B, n - s)) for s in range(0, n, B))
            set_ngroups(ng, 0)
            return lib_ms(lib, lambda: [group_call(sb, so, m, groups, ng, tb, to) for sb, so, m in subs])
        r = med({"pack": pack, "group_one_call": one, "group_batches": batches})
        assert int(ng.t.item()) <= D
        res["names_%d" % D] = r
        del cells, kb, ko, tb, to, subs
        torch.cuda.empty_cache()

    # Q3-shaped (BIGINT, DATE, INT) keys, has_null = 0: 16 bytes per row; and 8-byte GROUP_IDS at the same cardinality
    D = 10_000_000
    ids = torch.randint(0, D, (n,), device="cuda", generator=g)
    c0, c1, c2 = Dev(ids * 7), Dev((ids % 2406).to(torch.int32)), Dev((ids % 3).to(torch.int32))
    kb, ko = dev(16 * n, torch.uint8), dev(n + 1, torch.int64)
    tb, to = dev(16 * D + 64, torch.uint8), dev(D + 1, torch.int64)
    keys8, tk8 = Dev(ids.to(torch.int64)), dev(D, torch.int64)
    ready()

    def pack3():
        return lib_ms(lib, lambda: ops.pack_str_keys_device([c0, c1, c2], None, [capi.T_INT64, capi.T_DATE, capi.T_INT32], n, kb, ko, has_null=False))

    def group3():
        set_ngroups(ng, 0)
        return lib_ms(lib, lambda: group_call(kb, ko, n, groups, ng, tb, to))

    def gid8():
        set_ngroups(ng, 0)
        return lib_ms(lib, lambda: xcall(capi.XCALL_GROUP_IDS, [Vector(data_ptr=groups.ptr, data_nbytes=8 * n, length=n), Vector(data_ptr=ng.ptr, data_nbytes=8, length=1),
                                                                Vector(data_ptr=tk8.ptr, data_nbytes=tk8.nbytes, length=D), Vector(data_ptr=keys8.ptr, data_nbytes=8 * n, length=n)], n))
    res["q3_keys_10000000"] = med({"pack": pack3, "group_one_call": group3, "group_ids_8byte": gid8})
    del ids, c0, c1, c2, kb, ko, tb, to, keys8, tk8
    torch.cuda.empty_cache()

    # STR_JOIN_FIND: 10^7 probe rows in 10^6-row batches against a 10^6-group build, prepared against rebuilt per batch
    D, P = 1_000_000, min(10_000_000, n)
    bcells = name_cells(torch.randperm(D, device="cuda", generator=g))
    bb, bo = dev(21 * D, torch.uint8), dev(D + 1, torch.int64)
    tb, to, bg = dev(21 * D + 64, torch.uint8), dev(D + 1, torch.int64), dev(D, torch.int64)
    pcells = name_cells(torch.randint(0, 2 * D, (P,), device="cuda", generator=g))
    pb, po = dev(21 * P, torch.uint8), dev(P + 1, torch.int64)
    vals = dev(P, torch.int64)
    set_ngroups(ng, 0)
    ops.pack_str_keys_device([(bcells, None)], None, [capi.T_VARCHAR], D, bb, bo)
    group_call(bb, bo, D, bg, ng, tb, to)
    ops.pack_str_keys_device([(pcells, None)], None, [capi.T_VARCHAR], P, pb, po)
    capi.check(lib.MoB200_Sync(), lib)
    psubs = [(s, min(B, P - s), Dev(po.t[s:s + min(B, P - s) + 1] - po.t[s]), int(po.t[s].item())) for s in range(0, P, B)]
    ready()
    ngv = np.array([D], np.int64)

    def find_all():
        def run():
            for s, m, so, b0 in psubs:
                xcall(capi.XCALL_STR_JOIN_FIND, [Vector(data_ptr=vals.ptr + 8 * s, data_nbytes=8 * m, length=m), Vector(data=ngv, length=1),
                                                 Vector(data_ptr=tb.ptr, data_nbytes=tb.nbytes, length=1), Vector(data_ptr=to.ptr, data_nbytes=to.nbytes, length=1),
                                                 Vector(data_ptr=pb.ptr + b0, data_nbytes=21 * m, length=m), Vector(data_ptr=so.ptr, data_nbytes=8 * (m + 1), length=m)], m)
        return lib_ms(lib, run)

    def prepared():
        capi.check(lib.MoB200_StrJoinMapPrepare(C.c_void_p(tb.ptr), C.c_void_p(to.ptr), D), lib)
        ms = find_all()
        lib.MoB200_JoinMapRelease(C.c_void_p(to.ptr))
        return ms
    res["join_find_build_1000000_probe_%d" % P] = med({"rebuilt": find_all, "prepared": prepared})
    capi.check(lib.MoB200_Sync(), lib)
    hit = (vals.t > 0).float().mean().item()
    res["join_find_hit_rate"] = round(hit, 4)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
