"""The selective Q6 kernel (the default: discount, quantity and price are read only where the earlier conjuncts leave a row alive)
against the dense kernel (q6_variant = 1), which reads every column of every row.  Both run the same grid, the same pair -> thread
mapping and the same reduction, so sums and counts must agree bit for bit -- for any selectivity, size, NaN / Inf placement, and on
both the resident and the host-staged path -- and both must agree with the oracle."""
import struct

import numpy as np
import pytest

import oracle_lib as O
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer

pytestmark = pytest.mark.gpu
NAMES = ("shipdate", "discount", "quantity", "extendedprice")
SWEEP = (datagen.q6_params(),                                # Q6: 1.8 % of the rows pass
         (-2**31, 2**31 - 1, -np.inf, np.inf, np.inf),       # every row passes
         (-2**31, 2**31 - 1, 1.0, 0.0, np.inf),              # date passes everything, the discount window is empty
         (0, 0, -np.inf, np.inf, np.inf))                    # nothing passes the date test
# One batch of the selective loop is 3 pairs per thread of a 132 x 4 x 256-thread grid = 811008 rows on a 132-SM H100.  Below that
# the grid shrinks to one pair per thread and only the per-thread tail loop runs, so the tests that aim at the selective rounds use
# more rows than one batch.
SIZES = [1, 2, 3, 63, 64, 65, 1001, 270_337, 811_007, 811_008, 811_009, 811_072, 1_622_017, 5_000_003]


def bits(r):
    return struct.pack("<d", r[0]), r[1], r[2]


def q6(gpu, cols, n, P, variant):
    try:
        assert gpu.MoB200_SetTuning(b"q6_variant", variant) == 0
        return ops.q6_filter_sum(*(cols[k] for k in NAMES), n, *P)
    finally:
        gpu.MoB200_SetTuning(b"q6_variant", 0)


def resident(cols):
    return {k: DeviceBuffer.from_numpy(np.ascontiguousarray(cols[k])) for k in NAMES}


def check_against_dense(gpu, cols, n, P, oracle=True):
    """selective == dense bit for bit on the host-staged and the resident path; both agree with the oracle.  Returns the result."""
    host = q6(gpu, cols, n, P, 0)
    assert bits(host) == bits(q6(gpu, cols, n, P, 1))
    bufs = resident(cols)
    try:
        dev = q6(gpu, bufs, n, P, 0)
        assert bits(dev) == bits(q6(gpu, bufs, n, P, 1))
    finally:
        for b in bufs.values():
            b.free()
    assert bits(dev) == bits(host)       # same kernel, same grid (one host chunk at these sizes)
    if oracle:
        want, ns, nul = O.q6(cols, n, P)
        assert host[1] == ns and host[2] == nul
        assert abs(host[0] - want) <= 1e-11 * abs(want) + 1e-12
    return host


@pytest.mark.parametrize("P", SWEEP, ids=["q6", "every_row_passes", "discount_window_empty", "no_row_passes"])
def test_selectivity_sweep_matches_dense(gpu, P):
    n = 3_000_017
    cols = datagen.lineitem(10, 0, n)
    got = check_against_dense(gpu, cols, n, P)
    expect_rows = {0: None, 1: n, 2: 0, 3: 0}[SWEEP.index(P)]
    if expect_rows is not None:
        assert got[1] == expect_rows


@pytest.mark.parametrize("n", SIZES)
def test_sizes_and_tails(gpu, n):
    """odd n, n below one batch, and sizes around the batch and grid boundaries (the per-thread tail loop and the odd last row)"""
    cols = datagen.lineitem(21, 0, n)
    check_against_dense(gpu, cols, n, datagen.q6_params())
    check_against_dense(gpu, cols, n, SWEEP[1], oracle=False)


def sparse_table(n, seed, pass_rate):
    """rows that each fail exactly one conjunct -- date (both sides), discount (both sides) or quantity -- or pass all three"""
    rng = np.random.default_rng(seed)
    lo, hi, dlo, dhi, qhi = datagen.q6_params()
    stage = rng.choice(6, size=n, p=[(1 - pass_rate) / 5] * 5 + [pass_rate])
    sd = np.where(stage == 0, lo - 1, np.where(stage == 1, hi, lo + rng.integers(0, hi - lo, n))).astype(np.int32)
    di = np.where(stage == 2, dlo - 0.01, np.where(stage == 3, dhi + 0.01, dlo + rng.integers(0, 3, n) * 0.01))
    qt = np.where(stage == 4, qhi + rng.integers(0, 26, n), rng.integers(1, 24, n)).astype(np.float64)
    pr = rng.integers(90_000, 10_500_000, n) / 100.0
    return {"shipdate": sd, "discount": di, "quantity": qt, "extendedprice": pr}, stage == 5


def test_lone_survivors(gpu):
    """one passing row in an otherwise failing column: alone in its warp's 64 rows, alone in its 32-byte sector, and next to a pair
    partner that failed at each later conjunct (so its lane read discount / quantity but must still reject the partner)"""
    n = 1_622_021
    P = datagen.q6_params()
    cols, _ = sparse_table(n, 1, 0.0)
    for r in (0, 1, 2, 3, 62, 63, 64, 65, 4095, 4096, 811_007, 811_008, n - 2, n - 1):
        c = {k: v.copy() for k, v in cols.items()}
        c["shipdate"][r], c["discount"][r], c["quantity"][r], c["extendedprice"][r] = P[0], 0.03, 1.0, 1234.5
        got = check_against_dense(gpu, c, n, P)
        assert got[1] == 1 and got[0] == 1234.5 * 0.03
        mate = r ^ 1
        if mate >= n:           # the odd last row has no partner
            continue
        for k, v in (("shipdate", P[0] - 1), ("discount", 0.05), ("quantity", 24.0)):   # partner fails date / discount / quantity
            c2 = {kk: vv.copy() for kk, vv in c.items()}
            c2["shipdate"][mate], c2["discount"][mate], c2["quantity"][mate], c2["extendedprice"][mate] = P[0], 0.03, 1.0, 99.0
            c2[k][mate] = v
            got = check_against_dense(gpu, c2, n, P)
            assert got[1] == 1 and got[0] == 1234.5 * 0.03


@pytest.mark.parametrize("pass_rate", [0.0005, 0.02, 0.5])
def test_random_failure_stages(gpu, pass_rate):
    n = 1_000_003
    cols, passing = sparse_table(n, 2, pass_rate)
    got = check_against_dense(gpu, cols, n, datagen.q6_params())
    assert got[1] == int(passing.sum())


def test_nan_and_inf(gpu):
    """NaN / Inf in rows that fail the filter change nothing; in rows that pass they reach the sum (or fail the comparison, as NaN does)"""
    n = 1_000_001
    P = datagen.q6_params()
    base = datagen.lineitem(12, 0, n)
    ok = (base["shipdate"] >= P[0]) & (base["shipdate"] < P[1]) & (base["discount"] >= P[2]) & (base["discount"] <= P[3]) & (base["quantity"] < P[4])
    fail, good = np.flatnonzero(~ok), np.flatnonzero(ok)
    c = {k: v.copy() for k, v in base.items()}
    for i, (k, v) in enumerate((("extendedprice", np.nan), ("extendedprice", np.inf), ("discount", np.nan), ("quantity", np.inf),
                                ("discount", -np.inf), ("extendedprice", -np.inf))):
        c[k][fail[37 * i]] = v
    c["discount"][fail[1000:1500]] = np.nan                   # whole sectors of NaN where nothing passes
    got = check_against_dense(gpu, c, n, P)
    clean = check_against_dense(gpu, base, n, P)
    assert bits(got) == bits(clean)
    c["discount"][good[3]] = np.nan                            # a NaN discount fails BETWEEN: one row fewer
    c["quantity"][good[4]] = np.nan                            # a NaN quantity fails qty < 24
    got = check_against_dense(gpu, c, n, P)
    assert got[1] == clean[1] - 2
    c["extendedprice"][good[5]] = np.inf
    got = check_against_dense(gpu, c, n, P, oracle=False)
    assert got[0] == np.inf and got[1] == clean[1] - 2
    c["extendedprice"][good[6]] = -np.inf
    got = check_against_dense(gpu, c, n, P, oracle=False)
    assert np.isnan(got[0]) and got[1] == clean[1] - 2
    want, ns, _ = O.q6(c, n, P)
    assert np.isnan(want) and ns == got[1]


def test_device_result_form(gpu):
    """the asynchronous form (resident columns, result written to device memory) runs the same kernel"""
    n = 1_000_001
    cols = datagen.lineitem(13, 0, n)
    P = datagen.q6_params()
    bufs = resident(cols)
    out = DeviceBuffer(16)
    try:
        for variant in (0, 1):
            try:
                assert gpu.MoB200_SetTuning(b"q6_variant", variant) == 0
                ops.q6_filter_sum_device(*(bufs[k] for k in NAMES), n, *P, out_ptr=out.ptr)
                capi.check(gpu.MoB200_Sync(), gpu)
            finally:
                gpu.MoB200_SetTuning(b"q6_variant", 0)
            r = out.to_numpy(np.float64)
            assert (r[0], int(r.view(np.int64)[1])) == q6(gpu, cols, n, P, 1)[:2]
    finally:
        for b in list(bufs.values()) + [out]:
            b.free()
