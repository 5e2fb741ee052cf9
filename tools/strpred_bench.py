#!/usr/bin/env python
"""String predicates on resident columns: GO_LIKE and GO_COMPARE over varlena columns in the TPC-H shapes, one GPU, one process.

    python tools/strpred_bench.py [--rows N] [--runs R] [--chunk C] [--parent-lib PATH] [--out FILE]

Shapes, over --rows rows (default 10^8) of generated values in the TPC-H formats: p_type LIKE 'PROMO%' (Q14), p_type LIKE '%BRASS' (Q2),
p_name LIKE '%green%' (Q9), o_comment NOT LIKE '%special%requests%' (Q13's wording; NOT is the negation of the same kernel's result), the
rune-level pattern '%a_b%' on p_name and o_comment, l_shipmode = 'MAIL' and p_brand <> 'Brand#45'.  A column is resident in chunks of --chunk
rows (a varlena area is addressed by 32-bit offsets), each chunk its own area with one value per row; a run calls the predicate once per
chunk, asynchronous form, const pattern in host memory.  kernel_ms sums the library's CUDA events around each call's kernel (MoB200_LastKernelMs);
call_ms is the whole run between events on the library's stream, the per-call status read-back included.  Both are medians of --runs runs,
alternating over the shapes.  bytes = cells (24 per row) + the area bytes of the non-inline values + the bool result; GB/s = bytes over
kernel_ms, next to the H100 SXM data-sheet HBM3 peak of 3.35 TB/s.  The card's name and power limit are read in the same call.
--parent-lib loads a second build of libmo_b200.so (another commit) and times every shape on it too (parent_*), alternating with this build
run by run, so that both see the same card state.
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
from matrixone_b200.vector import Vector, varlena_bytes_column, xcall  # noqa: E402

HBM_PEAK_BPS = 3.35e12

TYPES_1 = [b"STANDARD", b"SMALL", b"MEDIUM", b"LARGE", b"ECONOMY", b"PROMO"]
TYPES_2 = [b"ANODIZED", b"BURNISHED", b"PLATED", b"POLISHED", b"BRUSHED"]
TYPES_3 = [b"TIN", b"NICKEL", b"BRASS", b"STEEL", b"COPPER"]
COLORS = [b"almond", b"antique", b"aquamarine", b"azure", b"beige", b"bisque", b"black", b"blanched", b"blue", b"blush", b"brown", b"burlywood",
          b"chartreuse", b"chiffon", b"chocolate", b"coral", b"cornflower", b"cream", b"cyan", b"dark", b"deep", b"dim", b"dodger", b"drab",
          b"firebrick", b"floral", b"forest", b"frosted", b"gainsboro", b"ghost", b"goldenrod", b"green", b"grey", b"honeydew", b"hot",
          b"indian", b"ivory", b"khaki", b"lace", b"lavender", b"lawn", b"lemon", b"light", b"lime", b"linen", b"magenta", b"maroon"]
WORDS = [b"special", b"requests", b"pending", b"accounts", b"furiously", b"carefully", b"blithely", b"quickly", b"deposits", b"packages",
         b"final", b"regular", b"ironic", b"express", b"bold", b"slyly", b"even", b"theodolites", b"foxes", b"instructions", b"a", b"b"]
MODES = [b"REG AIR", b"AIR", b"RAIL", b"SHIP", b"TRUCK", b"MAIL", b"FOB"]


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
    name, power = (x.strip() for x in out.split(","))
    return name, power


def templates(kind, rng, k=4096):
    """k distinct values of one TPC-H column format"""
    out = []
    for _ in range(k):
        if kind == "p_type":
            out.append(b" ".join((TYPES_1[rng.integers(6)], TYPES_2[rng.integers(5)], TYPES_3[rng.integers(5)])))
        elif kind == "p_name":
            out.append(b" ".join(COLORS[j] for j in rng.choice(len(COLORS), 5, replace=False)))
        elif kind == "o_comment":
            w = b""
            while len(w) < rng.integers(19, 79):
                w += WORDS[rng.integers(len(WORDS))] + b" "
            out.append(w[:78].strip())
        elif kind == "l_shipmode":
            out.append(MODES[rng.integers(len(MODES))])
        else:
            out.append(b"Brand#%d%d" % (rng.integers(1, 6), rng.integers(1, 6)))
    return out


class Chunk:
    """rows of one resident column: cells and an area with a slot of W bytes per row (a non-inline value sits in its row's slot)"""

    def __init__(self, tmpl, idx):
        n = idx.numel()
        W = max(max(len(v) for v in tmpl), 1)
        tc, _ = varlena_bytes_column(tmpl)
        tcells = torch.from_numpy(tc.reshape(-1, 24).copy()).cuda()
        pad = np.zeros((len(tmpl), W), np.uint8)
        for j, v in enumerate(tmpl):
            pad[j, :len(v)] = np.frombuffer(v, np.uint8)
        lens = torch.tensor([len(v) for v in tmpl], dtype=torch.int64, device="cuda")
        cells = tcells[idx].clone()
        big = lens[idx] > 23
        if bool(big.any()):
            self.area = torch.from_numpy(pad).cuda()[idx].reshape(-1).contiguous()
            c32 = cells.view(torch.int32)
            rows = torch.arange(n, device="cuda", dtype=torch.int64)
            c32[:, 1] = torch.where(big, rows * W, c32[:, 1].to(torch.int64)).to(torch.int32)
            self.area_read = int(lens[idx][big].sum())
        else:
            self.area, self.area_read = None, 0
        self.cells, self.n = cells.reshape(-1).contiguous(), n
        self.out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        self.outn = torch.zeros((n + 63) // 64, dtype=torch.int64, device="cuda")

    def vec(self):
        a = self.area
        return Vector(data_ptr=self.cells.data_ptr(), data_nbytes=24 * self.n, length=self.n,
                      area_ptr=None if a is None else a.data_ptr(), area_nbytes=0 if a is None else a.numel())

    def call(self, lib, fid, const):
        xcall(fid, [Vector(data_ptr=self.out.data_ptr(), data_nbytes=self.n, nulls_ptr=self.outn.data_ptr(), length=self.n), self.vec(), const], self.n,
              lib=lib)


def const_vec(value):
    cells, area = varlena_bytes_column([value])
    return Vector(data=cells, area=area if area.size else None, length=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=1 << 24)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("strpred_bench: no CUDA device (the measurement needs the H100)")
    libs = {"": capi.load_library()}
    if a.parent_lib:
        libs["parent_"] = capi.load_library(a.parent_lib)
    for lib in libs.values():
        capi.check(lib.MoB200_Init(0), lib)
    name, power = card()
    rng = np.random.default_rng(1)
    g = torch.Generator(device="cuda").manual_seed(1)
    cols = {}
    for kind in ("p_type", "p_name", "o_comment", "l_shipmode", "p_brand"):
        tmpl = templates(kind, rng)
        chunks, left = [], a.rows
        while left:
            m = min(a.chunk, left)
            chunks.append(Chunk(tmpl, torch.randint(len(tmpl), (m,), generator=g, device="cuda")))
            left -= m
        cols[kind] = chunks
    torch.cuda.synchronize()
    shapes = [("p_type LIKE 'PROMO%'", "p_type", capi.XCALL_GO_LIKE, b"PROMO%"),
              ("p_type LIKE '%BRASS'", "p_type", capi.XCALL_GO_LIKE, b"%BRASS"),
              ("p_name LIKE '%green%'", "p_name", capi.XCALL_GO_LIKE, b"%green%"),
              ("o_comment NOT LIKE '%special%requests%'", "o_comment", capi.XCALL_GO_LIKE, b"%special%requests%"),
              ("p_name LIKE '%a_b%' (rune level)", "p_name", capi.XCALL_GO_LIKE, b"%a_b%"),
              ("o_comment LIKE '%a_b%' (rune level)", "o_comment", capi.XCALL_GO_LIKE, b"%a_b%"),
              ("l_shipmode = 'MAIL'", "l_shipmode", capi.XCALL_GO_COMPARE(capi.CMP_EQ, capi.T_CHAR), b"MAIL"),
              ("p_brand <> 'Brand#45'", "p_brand", capi.XCALL_GO_COMPARE(capi.CMP_NE, capi.T_CHAR), b"Brand#45")]
    times = {p + s[0]: ([], []) for s in shapes for p in libs}

    def run(shape, lib=libs[""]):
        label, kind, fid, value = shape
        cv = const_vec(value)
        kms = 0.0
        capi.check(lib.MoB200_TimerStart(), lib)
        for ch in cols[kind]:
            ch.call(lib, fid, cv)
            ms = C.c_float()
            capi.check(lib.MoB200_LastKernelMs(C.byref(ms)), lib)
            kms += ms.value
        tot = C.c_float()
        capi.check(lib.MoB200_TimerStop(C.byref(tot)), lib)
        return kms, tot.value

    for s in shapes:                                   # warm-up of every shape
        for lib in libs.values():
            run(s, lib)
    for _ in range(a.runs):
        for s in shapes:
            for p, lib in libs.items():
                k, t = run(s, lib)
                times[p + s[0]][0].append(k)
                times[p + s[0]][1].append(t)
    hits = {}
    for s in shapes:                                   # the rows each shape's LIKE / compare admits (a column's chunks share one result buffer)
        run(s)
        hits[s[0]] = sum(int(ch.out.sum()) for ch in cols[s[1]])
    res = {"card": name, "power_limit": power, "rows": a.rows, "chunk": a.chunk, "runs": a.runs, "hbm_peak_gbps": HBM_PEAK_BPS / 1e9, "shapes": {}}
    for (label, kind, fid, value), p in ((s, p) for s in shapes for p in libs):
        k, t = statistics.median(times[p + label][0]), statistics.median(times[p + label][1])
        nbytes = sum(24 * ch.n + ch.area_read + ch.n for ch in cols[kind])
        res["shapes"][p + label] = {"kernel_ms": round(k, 3), "call_ms": round(t, 3), "bytes": nbytes, "gbps": round(nbytes / (k * 1e-3) / 1e9, 1),
                                    "share_of_hbm_peak": round(nbytes / (k * 1e-3) / HBM_PEAK_BPS, 3), "spread_ms": [round(min(times[p + label][0]), 3),
                                    round(max(times[p + label][0]), 3)], "matches": hits[label]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
