"""GPU: the fused TPC-H Q6 over DECIMAL(15,2) columns (MO_XCALL_Q6_DEC_FILTER_SUM / _MERGE) -- digit for digit against q6.result, byte for
byte against the Python-integer restatement of the operator chain (tpch_decimal_reference.py) and against the GPU operator chain, on both
kernel variants, host and resident columns; the Decimal128 Add overflow at its row, through the magnitude bound and the row-order rare path."""
import numpy as np
import pytest

import golden_tables as G
import oracle_lib as O
import tpch_decimal_reference as R
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, xcall
from test_oracle_tpch_decimal import BIG, WIDE, big_rows, first_overflow

pytestmark = pytest.mark.gpu
NAMES = ("shipdate", "discount", "quantity", "extendedprice")


@pytest.fixture(params=[0, 1], ids=["selective", "dense"])
def variant(request, gpu):
    assert gpu.MoB200_SetTuning(b"q6_variant", request.param) == 0
    yield request.param
    gpu.MoB200_SetTuning(b"q6_variant", 0)


def run_host(cols, n, P):
    return ops.q6_dec_filter_sum(*[cols[k] for k in NAMES], n, *P)


def run_resident(cols, n, P):
    bufs = [DeviceBuffer.from_numpy(cols[k][:n]) for k in NAMES]
    try:
        return ops.q6_dec_filter_sum(*bufs, n, *P)
    finally:
        for b in bufs:
            b.free()


def want(cols, n, P):
    return R.q6_dec(*[cols[k] for k in NAMES], n, *P)


def test_q6_dec_fixture_equals_q6_result(variant):
    cols, ints, expected = G.tpch_fixture()
    n = len(cols["shipdate"])
    dec = {"shipdate": cols["shipdate"], "discount": ints["discount_pct"], "quantity": ints["quantity"] * 100, "extendedprice": ints["extendedprice_cents"]}
    for got in (run_host(dec, n, R.q6_dec_params()), run_resident(dec, n, R.q6_dec_params())):
        assert got["rc"] == 0 and got["scale"] == 4
        assert O.decimal_str(got["revenue"], 4) == expected["q6_revenue"]


@pytest.mark.parametrize("n", [0, 1, 2, 3, 1000, 8192, 8193, 65_535, 65_536, 1_000_001])
def test_q6_dec_matches_reference_host_and_resident(variant, n):
    cols = R.lineitem_dec(10, 0, n)
    P = R.q6_dec_params()
    w = want(cols, n, P)
    assert run_host(cols, n, P) == w
    if n:
        assert run_resident(cols, n, P) == w


def test_q6_dec_equals_gpu_operator_chain(gpu):
    """compare -> sels -> Shrink -> d64Mul -> Decimal128 SUM, each node its own call, on the same rows"""
    n = 300_001
    cols = R.lineitem_dec(3, 0, n)
    lo, hi, dlo, dhi, qhi, s = R.q6_dec_params()
    m = ((cols["shipdate"] >= lo) & (cols["shipdate"] < hi) & (cols["discount"] >= dlo) & (cols["discount"] <= dhi) & (cols["quantity"] < qhi)).astype(np.uint8)
    sels = ops.filter_sels(m)
    rc, prod, _, _ = ops.dec_arith(2, 64, ops.shuffle(cols["extendedprice"], sels), ops.shuffle(cols["discount"], sels), s, s, len(sels))
    assert rc == 0
    acc = np.zeros((1, 2), dtype=np.uint64); cnt = np.zeros(1, dtype=np.int64)
    ops.dec_sum(128, prod, acc, cnt, None, None, len(sels))
    got = run_host(cols, n, (lo, hi, dlo, dhi, qhi, s))
    assert got["revenue"] == O.d128_to_int(acc)[0] and got["count"] == cnt[0] == len(sels)


def test_q6_dec_predicate_edges(gpu):
    """BETWEEN inclusive on both ends, the date range half-open, quantity strict"""
    lo, hi, dlo, dhi, qhi, s = R.q6_dec_params()
    cols = {"shipdate": np.asarray([lo - 1, lo, hi - 1, hi, lo, lo, lo, lo, lo, lo], dtype=np.int32),
            "discount": np.asarray([3, 3, 3, 3, dlo, dhi, dlo - 1, dhi + 1, 3, 3], dtype=np.int64),
            "quantity": np.asarray([100, 100, 100, 100, 100, 100, 100, 100, qhi - 1, qhi], dtype=np.int64),
            "extendedprice": np.arange(1, 11, dtype=np.int64) * 1000}
    got = run_host(cols, 10, (lo, hi, dlo, dhi, qhi, s))
    assert got == want(cols, 10, (lo, hi, dlo, dhi, qhi, s))
    assert got["count"] == 5 and got["revenue"] == 2000 * 3 + 3000 * 3 + 5000 * dlo + 6000 * dhi + 9000 * 3


def test_q6_dec_overflow_rows(variant):
    """the Decimal128 Add overflow of SUM at its row; a failing row that does not pass the filter does not count; a bound exceeded by
    (+big, -big, ...) takes the row-order rare path and succeeds"""
    k = first_overflow(10)
    for n in (10, 70_001):
        cols = dict(zip(NAMES, big_rows([BIG] * n)))
        got = run_resident(cols, n, WIDE)
        assert got == want(cols, n, WIDE) and got["rc"] == capi.RC_INVALID_ARGUMENT and got["err_row"] == k
        cols["quantity"][k] = 2400
        assert run_host(cols, n, WIDE)["err_row"] == k + 1
    alt = dict(zip(NAMES, big_rows([BIG if i % 2 == 0 else -BIG for i in range(100_001)])))
    got = run_resident(alt, 100_001, WIDE)
    assert got == want(alt, 100_001, WIDE) and got["rc"] == 0 and got["revenue"] == BIG * BIG
    # the overflow late in a long column: (+big, -big) pairs, then a run of +big
    n = 200_000
    prices = [BIG if i % 2 == 0 else -BIG for i in range(n)]
    prices[150_000:150_004] = [BIG] * 4
    cols = dict(zip(NAMES, big_rows(prices)))
    got = run_resident(cols, n, WIDE)
    assert got == want(cols, n, WIDE) and got["err_row"] == 150_000 + first_overflow(4)


def test_q6_dec_merge_of_ranges_equals_whole(gpu):
    n = 1_000_003
    cols = R.lineitem_dec(5, 0, n)
    P = R.q6_dec_params()
    whole = run_host(cols, n, P)
    cuts = [0, 1, 400_000, 400_001, 777_777, n]
    parts = b""
    for a, b in zip(cuts[:-1], cuts[1:]):
        res = np.zeros(ops.Q6_DEC_RESULT_BYTES, dtype=np.uint8)
        sub = {k: cols[k][a:b].copy() for k in NAMES}
        d = [DeviceBuffer.from_numpy(sub[k]) for k in NAMES]
        out = DeviceBuffer(ops.Q6_DEC_RESULT_BYTES)
        ops.q6_dec_filter_sum_device(*d, b - a, *P, out.ptr)          # asynchronous form: enqueued, read back below
        parts += out.to_numpy(np.uint8).tobytes()
        assert ops.q6_dec_result_from_bytes(parts[-ops.Q6_DEC_RESULT_BYTES:]) == run_host(sub, b - a, P)
        for x in d + [out]:
            x.free()
    merged = ops.q6_dec_merge(parts, len(cuts) - 1)
    assert merged == whole
    empty = ops.q6_dec_merge(b"", 0)
    assert empty["count"] == 0 and empty["is_null"] and empty["rc"] == 0


def test_q6_dec_merge_checks_the_sum(gpu):
    cols = dict(zip(NAMES, big_rows([BIG])))
    one = run_host(cols, 1, WIDE)
    res = np.zeros(ops.Q6_DEC_RESULT_BYTES, dtype=np.uint8)
    xcall(capi.XCALL_Q6_DEC_FILTER_SUM, [Vector(data=res, length=1)] + [ops._vec(cols[k], 1) for k in NAMES] +
          [ops._params_vec(capi.Q6DecParams(*WIDE[:5], WIDE[5], 0))], 1)
    raw = res.tobytes()
    assert ops.q6_dec_result_from_bytes(raw) == one
    merged = ops.q6_dec_merge(raw * 3, 3)            # 3 * BIG^2 leaves int128 in BatchMerge's checked add
    assert merged["rc"] == capi.RC_INVALID_ARGUMENT and merged["err_row"] == -1
    assert ops.q6_dec_merge(raw * 2, 2)["rc"] == 0


def test_q6_dec_chunked_host_input_equals_resident(gpu):
    """host columns over 32 M rows are staged in chunks and folded on the device; the result equals one resident pass, and an overflow in
    the second chunk is found at its row from the first chunk's running sum"""
    n = (32 << 20) + 1001
    cols = R.lineitem_dec(7, 0, n)
    P = R.q6_dec_params()
    host = run_host(cols, n, P)
    assert host == run_resident(cols, n, P) and host["rc"] == 0 and host["count"] > 0
    big = {"shipdate": np.full(n, 9000, np.int32), "discount": np.full(n, BIG, np.int64), "quantity": np.full(n, 2400, np.int64),
           "extendedprice": np.zeros(n, np.int64)}
    r = (32 << 20) - 1                               # last row of chunk 0 and the first rows of chunk 1 qualify
    big["quantity"][r:r + 4] = 1
    big["extendedprice"][r:r + 4] = BIG
    got = run_host(big, n, WIDE)
    assert got["rc"] == capi.RC_INVALID_ARGUMENT and got["err_row"] == r + first_overflow(4)
    assert got == run_resident(big, n, WIDE)


def test_q6_dec_rejects(gpu):
    cols = R.lineitem_dec(1, 0, 1000)
    P = list(R.q6_dec_params())
    args = lambda: [Vector(data=np.zeros(ops.Q6_DEC_RESULT_BYTES, np.uint8), length=1)] + [ops._vec(cols[k], 1000) for k in NAMES]
    for scale in (5, -1):
        rc, _ = xcall(capi.XCALL_Q6_DEC_FILTER_SUM, args() + [ops._params_vec(capi.Q6DecParams(*P[:5], scale, 0))], 1000, raise_on_error=False)
        assert rc == capi.RC_INVALID_ARGUMENT
    a = args()
    a[2].nulls = np.zeros(16, dtype=np.uint64)                      # a nulls bitmap: the schema's columns are NOT NULL
    rc, msg = xcall(capi.XCALL_Q6_DEC_FILTER_SUM, a + [ops._params_vec(capi.Q6DecParams(*P, 0))], 1000, raise_on_error=False)
    assert rc == capi.RC_INVALID_ARGUMENT and "NOT NULL" in msg
    rc, _ = xcall(capi.XCALL_Q6_DEC_FILTER_SUM, args() + [ops._params_vec(capi.Q6DecParams(*P, 0))], 1001, raise_on_error=False)
    assert rc == capi.RC_INVALID_ARGUMENT                            # columns shorter than len
    buf = DeviceBuffer.from_numpy(np.concatenate([np.zeros(1, np.int64), cols["discount"]]))
    a = args()
    a[2] = Vector(data_ptr=buf.ptr + 8, data_nbytes=8000, length=1000)   # 8-byte aligned, not 16
    d = [DeviceBuffer.from_numpy(cols[k]) for k in ("shipdate", "quantity", "extendedprice")]
    a[1], a[3], a[4] = (ops._vec(x, 1000) for x in d)
    rc, _ = xcall(capi.XCALL_Q6_DEC_FILTER_SUM, a + [ops._params_vec(capi.Q6DecParams(*P, 0))], 1000, raise_on_error=False)
    assert rc == capi.RC_INVALID_ARGUMENT
    for x in d + [buf]:
        x.free()


def test_q6_dec_asynchronous_form_enqueues_without_synchronising(gpu):
    """device columns and a device result: the call returns while its kernels are still queued.  20 calls over 64 M resident rows keep the
    device busy far longer than the host needs to enqueue them; a form that synchronised would take at least as long on the host."""
    import ctypes as C
    import time
    n = 64 << 20
    cols = {"shipdate": np.full(n, 9000, np.int32), "discount": np.full(n, 3, np.int64), "quantity": np.full(n, 100, np.int64),
            "extendedprice": np.full(n, 1000, np.int64)}
    bufs = [DeviceBuffer.from_numpy(cols[k]) for k in NAMES]
    out = DeviceBuffer(ops.Q6_DEC_RESULT_BYTES)
    P = R.q6_dec_params()
    ops.q6_dec_filter_sum_device(*bufs, n, *P, out.ptr)
    capi.check(gpu.MoB200_Sync(), gpu)
    capi.check(gpu.MoB200_TimerStart(), gpu)
    t0 = time.perf_counter()
    for _ in range(20):
        ops.q6_dec_filter_sum_device(*bufs, n, *P, out.ptr)
    host_ms = (time.perf_counter() - t0) * 1e3
    dev_ms = C.c_float()
    capi.check(gpu.MoB200_TimerStop(C.byref(dev_ms)), gpu)
    assert host_ms < 0.5 * dev_ms.value, (host_ms, dev_ms.value)
    got = ops.q6_dec_result_from_bytes(out.to_numpy(np.uint8).tobytes())
    assert got["rc"] == 0 and got["count"] == n and got["revenue"] == 3000 * n
    for b in bufs + [out]:
        b.free()


def test_q6_dec_row_base_gives_global_err_rows_through_the_merge(gpu):
    """ranges scanned with their row_base report global failing rows; the merge reports the lowest one, whatever the partials' order"""
    n = 1000
    prices = [0] * n
    prices[300:304] = [BIG] * 4
    prices[700:704] = [BIG] * 4
    cols = dict(zip(NAMES, big_rows(prices)))
    whole = run_host(cols, n, WIDE)
    assert whole["rc"] == capi.RC_INVALID_ARGUMENT and whole["err_row"] == 300 + first_overflow(4)
    parts = []
    for a, b in ((0, 500), (500, n)):
        d = [DeviceBuffer.from_numpy(cols[k][a:b].copy()) for k in NAMES]
        out = DeviceBuffer(ops.Q6_DEC_RESULT_BYTES)
        ops.q6_dec_filter_sum_device(*d, b - a, *WIDE, out.ptr, row_base=a)
        parts.append(out.to_numpy(np.uint8).tobytes())
        for x in d + [out]:
            x.free()
    assert ops.q6_dec_result_from_bytes(parts[1])["err_row"] == 700 + first_overflow(4)
    for order in (parts, parts[::-1]):
        merged = ops.q6_dec_merge(b"".join(order), 2)
        assert merged["rc"] == capi.RC_INVALID_ARGUMENT and merged["err_row"] == whole["err_row"]
