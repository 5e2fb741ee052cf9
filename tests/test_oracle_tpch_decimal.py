"""The Python-integer restatement of TPC-H Q6 over DECIMAL(15,2) columns (tpch_decimal_reference.py), pinned without a GPU: digit for digit
to q6.result on the reference's lineitem, equal to the composition of the oracle's d64Mul and Decimal128 SUM, and failing at the right row
when a running sum leaves int128."""
import ctypes as C

import numpy as np

import golden_tables as G
import oracle_lib as O
import tpch_decimal_reference as R
from matrixone_b200 import capi


def test_q6_dec_reproduces_q6_result_on_reference_lineitem():
    cols, ints, expected = G.tpch_fixture()
    n = len(cols["shipdate"])
    lo, hi, dlo, dhi, qhi, s = R.q6_dec_params()
    got = R.q6_dec(cols["shipdate"], ints["discount_pct"], ints["quantity"] * 100, ints["extendedprice_cents"], n, lo, hi, dlo, dhi, qhi, s)
    assert got["rc"] == 0 and got["scale"] == 4
    assert O.decimal_str(got["revenue"], 4) == expected["q6_revenue"] == "43092.5479"


def test_q6_dec_equals_oracle_d64_mul_and_sum_d128_composition():
    rng = np.random.default_rng(6)
    n = 50_000
    sd = rng.integers(8700, 9300, n).astype(np.int32)
    disc = rng.integers(-3, 12, n).astype(np.int64)
    qty = rng.integers(-500, 5000, n).astype(np.int64)
    price = rng.integers(-10 ** 15, 10 ** 15, n).astype(np.int64)
    P = (8766, 9131, 2, 4, 2400)
    got = R.q6_dec(sd, disc, qty, price, n, *P, 2)
    m = (sd >= P[0]) & (sd < P[1]) & (disc >= P[2]) & (disc <= P[3]) & (qty < P[4])
    k = int(m.sum())
    lib = O.go()
    prod = np.zeros((k, 2), dtype=np.uint64)
    rn = np.zeros((k + 63) // 64, dtype=np.uint64)
    a, b, one = price[m].copy(), disc[m].copy(), np.ones(k, dtype=np.uint64)     # kept alive across the calls
    assert lib.og_d64_mul(O.p(prod), O.p(a), O.p(b), k, 0, 0, 2, 2, None, None, O.p(rn)) == 0
    s = np.zeros((1, 2), dtype=np.uint64); c = np.zeros(1, dtype=np.int64)
    lib.og_sum_d128(O.p(prod), None, 0, O.p(one), k, O.p(s), O.p(c))
    assert got["rc"] == 0 and got["count"] == k == c[0] and got["revenue"] == O.d128_to_int(s)[0]


BIG = (1 << 63) - 1
WIDE = (8766, 9131, -(1 << 63), BIG, 2400, 2)     # BETWEEN admits every discount: products up to (2^63 - 1)^2 ~ 2^126


def big_rows(prices):
    """rows inside the date range with discount 2^63 - 1 and quantity 1: the product of row i is prices[i] * (2^63 - 1)"""
    n = len(prices)
    return np.full(n, 9000, np.int32), np.full(n, BIG, np.int64), np.ones(n, np.int64), np.asarray(prices, dtype=np.int64)


def first_overflow(n):
    """row at which n rows of product BIG^2 have run out of int128"""
    return next(i for i in range(n) if (i + 1) * BIG * BIG > R.I128_MAX)


def test_q6_dec_sum_overflow_row_and_a_bound_exceeded_without_overflow():
    # (+big, -big, ...): the magnitude bound times the row count is exceeded, no running sum leaves range
    alt = [BIG if i % 2 == 0 else -BIG for i in range(1001)]
    got = R.q6_dec(*big_rows(alt), 1001, *WIDE)
    assert got["rc"] == 0 and got["revenue"] == BIG * BIG and got["err_row"] == -1
    k = first_overflow(10)
    assert k == 2
    got = R.q6_dec(*big_rows([BIG] * 10), 10, *WIDE)
    assert got["rc"] == R.RC_INVALID_ARGUMENT and got["err_row"] == k
    # the same row failing the filter (quantity not < 2400) does not count: the next qualifying row fails
    sd, disc, qty, price = big_rows([BIG] * 10)
    qty[k] = 2400
    got = R.q6_dec(sd, disc, qty, price, 10, *WIDE)
    assert got["rc"] == R.RC_INVALID_ARGUMENT and got["err_row"] == k + 1


def test_q6_dec_struct_layouts():
    assert C.sizeof(capi.Q6DecParams) == 48
    assert C.sizeof(capi.Q6DecResult) == 40
