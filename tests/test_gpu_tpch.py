"""GPU parity: the fused TPC-H Q6 / Q1 pipelines (BASELINE configs 2 and 3) against the oracle's operator-chain
restatement.  Counts / group sets / first-seen order exact; fp64 sums within 1e-5 relative (north_star) -- in practice
~1e-13 because only the summation order differs -- and bitwise deterministic run to run."""
import numpy as np
import pytest

import oracle_lib as O
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer, varlena_char1_column

pytestmark = pytest.mark.gpu
RTOL = 1e-5   # tolerance stated by BASELINE.json north_star for fp aggregates


def dev_lineitem(lib, seed, n, keys=True):
    bufs = {"shipdate": DeviceBuffer(4 * n), "quantity": DeviceBuffer(8 * n), "extendedprice": DeviceBuffer(8 * n),
            "discount": DeviceBuffer(8 * n), "tax": DeviceBuffer(8 * n), "returnflag": DeviceBuffer(n), "linestatus": DeviceBuffer(n)}
    capi.check(lib.MoB200_GenLineitem(seed, 0, n, bufs["shipdate"].ptr, bufs["quantity"].ptr, bufs["extendedprice"].ptr,
                                      bufs["discount"].ptr, bufs["tax"].ptr, bufs["returnflag"].ptr, bufs["linestatus"].ptr))
    return bufs


def test_device_generator_equals_numpy_twin(gpu):
    n = 300_001
    bufs = dev_lineitem(gpu, 10, n)
    cols = datagen.lineitem(10, 0, n)
    dts = {"shipdate": np.int32, "returnflag": np.uint8, "linestatus": np.uint8}
    for k, b in bufs.items():
        assert (b.to_numpy(dts.get(k, np.float64)) == cols[k]).all(), k
        b.free()


@pytest.mark.parametrize("n", [0, 1, 2, 3, 1000, 8192, 8193, 1_000_001])
def test_q6_matches_oracle_host_and_resident(gpu, n):
    cols = datagen.lineitem(10, 0, n)
    P = datagen.q6_params()
    want, ns, nul = O.q6(cols, n, P, nthreads=1)
    got = ops.q6_filter_sum(cols["shipdate"], cols["discount"], cols["quantity"], cols["extendedprice"], n, *P)    # host path
    assert got[1] == ns and got[2] == nul
    assert abs(got[0] - want) <= RTOL * abs(want)
    assert abs(got[0] - want) <= 1e-11 * abs(want) + 1e-12          # what we actually achieve
    if n:
        bufs = dev_lineitem(gpu, 10, n)
        res = ops.q6_filter_sum(bufs["shipdate"], bufs["discount"], bufs["quantity"], bufs["extendedprice"], n, *P)  # resident path
        assert res == got                                            # same kernel, same grid => bitwise equal
        assert ops.q6_filter_sum(bufs["shipdate"], bufs["discount"], bufs["quantity"], bufs["extendedprice"], n, *P) == res
        for b in bufs.values():
            b.free()


def test_q6_predicate_edges(gpu):
    """BETWEEN is inclusive on both ends, the date range is half-open, quantity strict (q6.sql:58-61)"""
    P = datagen.q6_params()
    sd = np.asarray([P[0] - 1, P[0], P[1] - 1, P[1], P[0], P[0], P[0], P[0]], dtype=np.int32)
    di = np.asarray([0.03, 0.03, 0.03, 0.03, P[2], P[3], np.nextafter(P[2], 0), np.nextafter(P[3], 1)], dtype=np.float64)
    qt = np.asarray([1, 1, 1, 1, 23, 24, 1, 1], dtype=np.float64)
    pr = np.asarray([100.0] * 8)
    cols = {"shipdate": sd, "discount": di, "quantity": qt, "extendedprice": pr}
    want, ns, nul = O.q6(cols, 8, P)
    got = ops.q6_filter_sum(sd, di, qt, pr, 8, *P)
    assert got[1] == ns == 3 and got[0] == want


def test_q6_nullable_columns_and_short_columns(gpu):
    """nullable inputs take the generic fused operator (plan.cu): a NULL predicate operand rejects the row, a NULL product is skipped by SUM;
    an all-zero bitmap gives the no-nulls answer; short columns are rejected"""
    from matrixone_b200.vector import Vector, bitmap_from_bools, xcall
    n = 100_000
    cols = datagen.lineitem(1, 0, n)
    P = datagen.q6_params()
    res = np.zeros(2); rn = np.zeros(1, dtype=np.uint64)
    p = capi.Q6Params(*P)
    pv = Vector(data=np.frombuffer(bytes(p), dtype=np.uint8).copy(), length=1)
    want = ops.q6_filter_sum(cols["shipdate"], cols["discount"], cols["quantity"], cols["extendedprice"], n, *P)
    zero = np.zeros((n + 63) // 64, dtype=np.uint64)
    xcall(capi.XCALL_Q6_FILTER_SUM, [Vector(data=res, nulls=rn, length=1), Vector(data=cols["shipdate"], nulls=zero, length=n), Vector(data=cols["discount"], length=n),
                                     Vector(data=cols["quantity"], length=n), Vector(data=cols["extendedprice"], length=n), pv], n)
    assert int(res.view(np.int64)[1]) == want[1] and abs(res[0] - want[0]) <= 1e-12 * abs(want[0])
    rng = np.random.default_rng(0)
    sdn = rng.random(n) < 0.2; prn = rng.random(n) < 0.2
    xcall(capi.XCALL_Q6_FILTER_SUM, [Vector(data=res, nulls=rn, length=1), Vector(data=cols["shipdate"], nulls=bitmap_from_bools(sdn), length=n), Vector(data=cols["discount"], length=n),
                                     Vector(data=cols["quantity"], length=n), Vector(data=cols["extendedprice"], nulls=bitmap_from_bools(prn), length=n), pv], n)
    m = (cols["shipdate"] >= P[0]) & (cols["shipdate"] < P[1]) & (cols["discount"] >= P[2]) & (cols["discount"] <= P[3]) & (cols["quantity"] < P[4]) & ~sdn
    assert int(res.view(np.int64)[1]) == int(m.sum())                                   # rows that pass the filter
    ref = float((cols["extendedprice"][m & ~prn] * cols["discount"][m & ~prn]).sum())     # SUM skips the NULL prices
    assert abs(res[0] - ref) <= 1e-11 * abs(ref)
    rc, msg = xcall(capi.XCALL_Q6_FILTER_SUM, [Vector(data=res, length=1), Vector(data=cols["shipdate"]), Vector(data=cols["discount"][:50]),
                                               Vector(data=cols["quantity"]), Vector(data=cols["extendedprice"]), pv], n, raise_on_error=False)
    assert rc == capi.RC_INVALID_ARGUMENT


def test_q1_nullable_columns(gpu):
    """Q1 with nulls bitmaps: NULL shipdate rejects the row, NULL measures are skipped by their own aggregate only (count(*) still counts), a NULL
    key forms its own group"""
    from matrixone_b200.vector import Vector, bitmap_from_bools, xcall
    import ctypes as C
    n = 200_000
    cols = datagen.lineitem(3, 0, n)
    rng = np.random.default_rng(1)
    nm = {k: rng.random(n) < 0.1 for k in ("shipdate", "quantity", "discount", "returnflag")}
    names = ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")
    vecs = [Vector(data=cols[k], nulls=bitmap_from_bools(nm[k]) if k in nm else None, length=n) for k in names]
    res = np.zeros(C.sizeof(capi.Q1Result), dtype=np.uint8)
    xcall(capi.XCALL_Q1_GROUP_AGG, [Vector(data=res, length=1)] + vecs + [Vector(data=np.asarray([datagen.Q1_CUTOFF], dtype=np.int32), length=1)], n)
    got = ops.q1_result_from_bytes(res.tobytes())
    sel = (cols["shipdate"] <= datagen.Q1_CUTOFF) & ~nm["shipdate"]
    rf = np.where(nm["returnflag"], 0, cols["returnflag"])
    seen = {}
    for g in got:
        k = (g["returnflag"], g["linestatus"])
        m = sel & (rf == k[0]) & (cols["linestatus"] == k[1]) & (nm["returnflag"] == (k[0] == 0))
        assert g["count_order"] == int(m.sum()) and g["first_row"] == int(np.flatnonzero(m)[0]), k
        q = cols["quantity"][m & ~nm["quantity"]]
        assert abs(g["sum_qty"] - q.sum()) <= 1e-11 * q.sum() and abs(g["avg_qty"] - q.mean()) <= 1e-11 * q.mean()
        dm = m & ~nm["discount"]
        dp = (cols["extendedprice"][dm] * (1 - cols["discount"][dm])).sum()
        assert abs(g["sum_disc_price"] - dp) <= 1e-11 * dp
        assert abs(g["sum_base_price"] - cols["extendedprice"][m].sum()) <= 1e-11 * cols["extendedprice"][m].sum()
        seen[k] = True
    assert sum(g["count_order"] for g in got) == int(sel.sum()) and any(k[0] == 0 for k in seen)
    assert [g["first_row"] for g in got] == sorted(g["first_row"] for g in got)


def _check_q1(got, want):
    assert [(g["returnflag"], g["linestatus"]) for g in got] == [(g["returnflag"], g["linestatus"]) for g in want]   # first-seen order
    for g, w in zip(got, want):
        assert g["count_order"] == w["count_order"] and g["first_row"] == w["first_row"]
        for k in ("sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc"):
            assert abs(g[k] - w[k]) <= RTOL * abs(w[k]), k
            assert abs(g[k] - w[k]) <= 1e-11 * abs(w[k]), k


@pytest.mark.parametrize("n", [1, 2, 5, 1000, 8192, 65_535, 65_536, 500_001])
def test_q1_matches_oracle_packed_and_varlena_keys(gpu, n):
    cols = datagen.lineitem(11, 0, n)
    want = O.q1(cols, n, datagen.Q1_CUTOFF, nthreads=1)
    got = ops.q1_group_agg(cols["shipdate"], cols["quantity"], cols["extendedprice"], cols["discount"], cols["tax"],
                           cols["returnflag"], cols["linestatus"], n, datagen.Q1_CUTOFF)
    _check_q1(got, want)
    rf = varlena_char1_column(cols["returnflag"]); ls = varlena_char1_column(cols["linestatus"])    # MatrixOne varlena layout
    got_v = ops.q1_group_agg(cols["shipdate"], cols["quantity"], cols["extendedprice"], cols["discount"], cols["tax"], rf, ls, n, datagen.Q1_CUTOFF)
    _check_q1(got_v, want)       # varlena keys run the register kernel, packed keys from 65,536 rows the TMA one: same values to 1e-11
    bufs = dev_lineitem(gpu, 11, n)
    got_d = ops.q1_group_agg(bufs["shipdate"], bufs["quantity"], bufs["extendedprice"], bufs["discount"], bufs["tax"],
                             bufs["returnflag"], bufs["linestatus"], n, datagen.Q1_CUTOFF)
    assert got_d == got           # resident vs staged-from-host: same kernel, same grid => bitwise equal
    assert got_d == ops.q1_group_agg(bufs["shipdate"], bufs["quantity"], bufs["extendedprice"], bufs["discount"], bufs["tax"],
                                     bufs["returnflag"], bufs["linestatus"], n, datagen.Q1_CUTOFF)   # run-to-run deterministic
    for b in bufs.values():
        b.free()


def test_q1_no_row_qualifies_and_many_groups(gpu):
    n = 1000
    cols = datagen.lineitem(11, 0, n)
    assert ops.q1_group_agg(cols["shipdate"], cols["quantity"], cols["extendedprice"], cols["discount"], cols["tax"],
                            cols["returnflag"], cols["linestatus"], n, 0) == []
    # 8 distinct keys: served by the wide (8-slot) variant after the 4-slot kernel reports overflow
    rf = (np.arange(n) % 4 + 65).astype(np.uint8); ls = (np.arange(n) // 4 % 2 + 70).astype(np.uint8)
    c2 = dict(cols, returnflag=rf, linestatus=ls)
    want = O.q1(c2, n, datagen.Q1_CUTOFF)
    got = ops.q1_group_agg(cols["shipdate"], cols["quantity"], cols["extendedprice"], cols["discount"], cols["tax"], rf, ls, n, datagen.Q1_CUTOFF)
    assert len(want) == 8
    _check_q1(got, want)
    rf9 = (np.arange(n) % 9 + 65).astype(np.uint8)
    with pytest.raises(capi.MoError):
        ops.q1_group_agg(cols["shipdate"], cols["quantity"], cols["extendedprice"], cols["discount"], cols["tax"], rf9, ls, n, datagen.Q1_CUTOFF)


def test_full_size_properties_block_additivity(gpu):
    """size-independent property used at SF100: the fused result over [0,n) equals the merge of the results over any
    split into block ranges (counts exactly, sums to 1e-12), and a sampled block range agrees with the oracle."""
    n = 6_000_000
    bufs = dev_lineitem(gpu, 12, n)
    P = datagen.q6_params()
    full = ops.q6_filter_sum(bufs["shipdate"], bufs["discount"], bufs["quantity"], bufs["extendedprice"], n, *P)
    cols = datagen.lineitem(12, 0, n)
    parts = []
    for r0, r1 in ((0, 8192 * 100), (8192 * 100, 8192 * 611), (8192 * 611, n)):
        m = r1 - r0
        parts.append(ops.q6_filter_sum(cols["shipdate"][r0:r1], cols["discount"][r0:r1], cols["quantity"][r0:r1], cols["extendedprice"][r0:r1], m, *P))
    assert sum(p[1] for p in parts) == full[1]
    assert abs(sum(p[0] for p in parts) - full[0]) <= 1e-12 * abs(full[0])
    want, ns, _ = O.q6(cols, n, P, nthreads=8)
    assert ns == full[1] and abs(want - full[0]) <= 1e-10 * abs(want)
    for b in bufs.values():
        b.free()


def test_kernel_variants_agree(gpu):
    """every tuning variant (tools/tune.py) computes the same counts and 1e-12-equal sums"""
    n = 300_000
    cols = datagen.lineitem(13, 0, n)
    P = datagen.q6_params()
    base = None
    try:
        for var in (0, 1):
            assert gpu.MoB200_SetTuning(b"q6_variant", var) == 0
            r = ops.q6_filter_sum(cols["shipdate"], cols["discount"], cols["quantity"], cols["extendedprice"], n, *P)
            base = base or r
            assert r[1] == base[1] and abs(r[0] - base[0]) <= 1e-12 * abs(base[0])
        want = O.q1(cols, n, datagen.Q1_CUTOFF)
        for var in (0, 1):
            assert gpu.MoB200_SetTuning(b"q1_variant", var) == 0
            _check_q1(ops.q1_group_agg(cols["shipdate"], cols["quantity"], cols["extendedprice"], cols["discount"], cols["tax"],
                                       cols["returnflag"], cols["linestatus"], n, datagen.Q1_CUTOFF), want)
    finally:
        gpu.MoB200_SetTuning(b"q6_variant", 0); gpu.MoB200_SetTuning(b"q1_variant", 0)


def test_q1_non_finite_values_stay_inside_their_group(gpu):
    """the branch-free group dispatch multiplies by 0/1 indicators; rows holding Inf/NaN must take the exact path so that
    only their own group is affected, exactly like the reference's per-group `sums[g] += v`"""
    n = 20_000
    cols = {k: v.copy() for k, v in datagen.lineitem(14, 0, n).items()}
    sel = np.flatnonzero((cols["returnflag"] == ord("A")) & (cols["shipdate"] <= datagen.Q1_CUTOFF))
    cols["quantity"][sel[5]] = np.inf
    cols["tax"][sel[9]] = np.nan
    cols["extendedprice"][sel[11]] = 1e308; cols["tax"][sel[11]] = 0.08      # finite inputs, product overflows to +Inf
    want = O.q1(cols, n, datagen.Q1_CUTOFF)
    got = ops.q1_group_agg(cols["shipdate"], cols["quantity"], cols["extendedprice"], cols["discount"], cols["tax"],
                           cols["returnflag"], cols["linestatus"], n, datagen.Q1_CUTOFF)
    assert [(g["returnflag"], g["linestatus"], g["count_order"]) for g in got] == [(g["returnflag"], g["linestatus"], g["count_order"]) for g in want]
    for g, w in zip(got, want):
        for k in ("sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc"):
            if np.isfinite(w[k]):
                assert abs(g[k] - w[k]) <= 1e-11 * abs(w[k]), (chr(g["returnflag"]), k)
            else:
                assert (np.isnan(g[k]) and np.isnan(w[k])) or g[k] == w[k], (chr(g["returnflag"]), k, g[k], w[k])
    a = [g for g in got if g["returnflag"] == ord("A")][0]
    assert np.isinf(a["sum_qty"]) and np.isnan(a["sum_charge"])


def test_q1_kernel_variants_agree(gpu):
    """the register kernel (q1_variant = 1) gives the default TMA kernel's result: same groups, counts and first rows; sums to the last
    few bits (the two kernels split the rows across threads differently, so the summation order differs)"""
    n = 5_000_011
    bufs = dev_lineitem(gpu, 10, n)
    args = [bufs[k] for k in ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")]
    want = ops.q1_group_agg(*args, n, datagen.Q1_CUTOFF)
    try:
        assert gpu.MoB200_SetTuning(b"q1_variant", 1) == 0
        got = ops.q1_group_agg(*args, n, datagen.Q1_CUTOFF)
    finally:
        gpu.MoB200_SetTuning(b"q1_variant", 0)
    assert [(g["returnflag"], g["linestatus"], g["count_order"], g["first_row"]) for g in got] == [(g["returnflag"], g["linestatus"], g["count_order"], g["first_row"]) for g in want]
    for a, b in zip(got, want):
        for f in ("sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_disc"):
            assert abs(a[f] - b[f]) <= 1e-12 * abs(b[f])
    for b in bufs.values():
        b.free()


def test_q1_more_than_four_groups_on_many_rows(gpu):
    """6 distinct keys over 300,001 rows: the 4-slot pass (the TMA kernel) overflows and the 8-slot register kernel answers, on the host
    path, on resident columns, and in the device-result form, where the 8-slot pass is enqueued behind the 4-slot one and gated on its
    overflow flag"""
    n = 300_001
    cols = datagen.lineitem(15, 0, n)
    rf = (np.arange(n) % 3 + 65).astype(np.uint8); ls = (np.arange(n) // 3 % 2 + 70).astype(np.uint8)
    want = O.q1(dict(cols, returnflag=rf, linestatus=ls), n, datagen.Q1_CUTOFF)
    assert len(want) == 6
    names = ("shipdate", "quantity", "extendedprice", "discount", "tax")
    got = ops.q1_group_agg(*[cols[k] for k in names], rf, ls, n, datagen.Q1_CUTOFF)
    _check_q1(got, want)
    bufs = dev_lineitem(gpu, 15, n)
    bufs["returnflag"].free(); bufs["returnflag"] = DeviceBuffer.from_numpy(rf)
    bufs["linestatus"].free(); bufs["linestatus"] = DeviceBuffer.from_numpy(ls)
    args = [bufs[k] for k in names + ("returnflag", "linestatus")]
    got_d = ops.q1_group_agg(*args, n, datagen.Q1_CUTOFF)
    _check_q1(got_d, want)
    assert got_d == got           # same kernels, same grids => bitwise equal
    out = DeviceBuffer(ops.Q1_RESULT_BYTES)
    ops.q1_group_agg_device(*args, n, datagen.Q1_CUTOFF, out.ptr)
    assert ops.q1_result_from_bytes(out.to_numpy(np.uint8).tobytes()) == got
    for b in list(bufs.values()) + [out]:
        b.free()
