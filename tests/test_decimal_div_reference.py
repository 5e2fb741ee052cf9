"""The decimal division / AVG / compare restatement (decimal_div_reference.py) pinned to the reference's own test cases, to hand-worked
Div128 and Div256 cases on both sides of their quirks, and to q1.result's averages over the reference's lineitem."""
import pytest

import decimal_div_reference as R
import golden_tables as G


def test_decimal128_over_div():
    # TestDecimal128OverDiv (decimal_test.go:253): 99999999999999999999999999999999999999 / 10000000000 at scales 0 / 0 goes through Div256
    q, scale = R.div(10 ** 38 - 1, 10 ** 10, 0, 0)
    assert scale == 6 and q == 10 ** 34


@pytest.mark.parametrize("sx,sy", [(1, -1), (-1, 1), (-1, -1), (1, 1)])
def test_decimal128_div_fallback_sign(sx, sy):
    # TestDecimal128DivFallbackSign (decimal_test.go:437): x * 10^6 leaves 127 bits, the quotient does not; the sign survives the fallback
    q, scale = R.div(sx * 3 * 10 ** 32, sy * 3, 0, 0)
    assert scale == 6 and q == sx * sy * 10 ** 38


def test_div_by_zero():
    # TestDivByZero_NullBehavior (arith_decimal_fast_test.go:43): the caller turns DivByZero into NULL or the error
    with pytest.raises(R.DivByZero):
        R.div(100, 0, 2, 2)


def test_high_scale_adj_overflows():
    # TestD128Div_DiffScale/HighScaleAdj (arith_decimal_fast_test.go:1583-1594): scale2 = 37 gives scaleAdj 43, and the quotient overflows
    with pytest.raises(R.DivOverflow):
        R.div(12345678, 1000000, 0, 37)


def test_result_scale():
    assert [R.div_scale(s) for s in (0, 2, 6, 12, 15, 38)] == [6, 8, 12, 12, 15, 38]
    assert all(R.avg_return_scale(s) == R.div_scale(s) for s in range(39))


def test_div128_below_2_126_rounds_half_up():
    # a 128-bit divisor: the quotient estimated from the divisor's top word, rounded by comparing 2x with y * v
    x, y = 7 << 64, 2 << 64
    assert R.div128(x, y) == 4                                       # 3.5 rounds up
    x, y = (7 << 120) + 1, 2 << 120
    assert R.div128(x, y) == 4
    x, y = (7 << 120) - 1, 2 << 120
    assert R.div128(x, y) == 3


def test_div128_at_and_above_2_126_rounds_down():
    # x.Left(1) wraps negative in Decimal128.Less once x >= 2^126, so an odd estimate always rounds down
    x, y = 0x77202ec9ffed9235288bc781ae662675, 0x2033e1ac4ee207f9da94e3e8ab73738f
    assert x >= 1 << 126 and R.exact_div_half_up(x, y, 0) == 4
    assert R.div128(x, y) == 3
    assert R.div(x, y, 12, 0) == (3, 12)                              # scaleAdj 0: |x| * 10^0 stays below 2^127, Div128 runs as is
    x, y = 7 << 124, 2 << 124                                        # 3.5 exactly
    assert R.div128(x, y) == 3
    # and the other side of 2^126 with the same ratio
    assert R.div128(7 << 122, 2 << 122) == 4


def test_div128_sample_differs_only_above_2_126():
    import random
    rng = random.Random(7)
    below = above = 0
    for _ in range(4000):
        y = rng.randrange(1 << 64, 1 << 125)
        x = rng.randrange(y, 1 << 126)
        below += R.div128(x, y) != R.exact_div_half_up(x, y, 0)
        x = rng.randrange(1 << 126, 1 << 127)
        above += R.div128(x, y) != R.exact_div_half_up(x, y, 0)
    assert below == 0 and above > 0


def test_div256_quirks():
    # a 64-bit divisor: the four-word long division, exact half up
    assert R.div256(10 ** 50, 3) == (10 ** 50 + 1) // 3
    # a dividend with bit 254 set doubles to a negative Decimal256: the signed long division never subtracts and the quotient is 0
    assert R.div256(1 << 254, (1 << 64) + 1) == 0
    # a dividend in [2^253, 2^254) against a power-of-two divisor: the divisor is shifted through bit 255 to zero and Go never returns
    with pytest.raises(R.NoEnd):
        R.div256(1 << 253, 1 << 64)


def test_compare_scale_quirks():
    # Decimal64: the unsigned Mul64 only fails past 2^64, so 10^18 * 10 wraps negative and compares below 0
    assert R.d64_scale_dropped(10 ** 18, 1) == 10 ** 19 - (1 << 64)
    assert R.compare(4, 10 ** 18, 0, 0, 1, 64)                        # 10^18 (scale 0) < 0 (scale 1)
    # a scale-up past 2^64 is dropped: the value compares unscaled
    assert R.d64_scale_dropped(10 ** 18, 2) == 10 ** 18
    # Decimal128 fails at 2^127 and compares unscaled
    assert R.d128_scale_dropped(10 ** 37, 2) == 10 ** 37
    assert R.d128_scale_dropped(-(10 ** 20), 18) == -(10 ** 38)
    assert R.compare(0, 15, 150, 1, 2, 128) and R.compare(5, -15, -151, 1, 2, 128) is False


def test_avg_count_zero_and_half_up():
    assert R.avg(5, 0, 2) is None
    assert R.avg(5, 2, 2) == (2500000, 8)                             # 0.05 / 2 = 0.025 at scale 8
    assert R.avg(-5, 3, 2) == (-1666667, 8)
    assert R.avg(-(1 << 127), 1, 12) == (-(1 << 127), 12)             # Div's overflow error dropped: the value it kept


def _half_up(v, from_scale, to_scale):
    f = 10 ** (from_scale - to_scale)
    q, r = divmod(abs(v), f)
    q += 2 * r >= f
    s = str(q).rjust(to_scale + 1, "0")
    return ("-" if v < 0 else "") + s[:-to_scale] + "." + s[-to_scale:]


def test_q1_averages_match_q1_result():
    """decAvg over the reference's lineitem: the three Q1 averages at scale 8, rounded half up to 2 decimals, equal q1.result's strings"""
    cols, ints, expected = G.tpch_fixture()
    import numpy as np
    from matrixone_b200 import datagen
    keep = cols["shipdate"] <= datagen.Q1_CUTOFF
    groups = {}
    for i in np.nonzero(keep)[0]:
        k = (chr(cols["returnflag"][i]), chr(cols["linestatus"][i]))
        g = groups.setdefault(k, [0, 0, 0, 0])
        g[0] += int(ints["quantity"][i]) * 100; g[1] += int(ints["extendedprice_cents"][i]); g[2] += int(ints["discount_pct"][i]); g[3] += 1
    assert len(groups) == len(expected["q1"])
    for k, (q, p, d, c) in groups.items():
        e = expected["q1"][k]
        got = [R.avg(v, c, 2) for v in (q, p, d)]
        assert all(s == 8 for _, s in got)
        assert [_half_up(v, 8, 2) for v, _ in got] == [e["avg_qty"], e["avg_price"], e["avg_disc"]]


def _kat():
    import json
    import os
    return json.load(open(os.path.join(os.path.dirname(__file__), "golden", "decimal_div_kat.json")))


def _unscaled(text, scale):
    from decimal import Decimal
    return int(Decimal(text).scaleb(scale))


def test_decimal_result_goldens_taken_and_skipped():
    """decimal.result: 4 division and 18 comparison statements have every operand exact at its column's scale; no AVG statement does (the
    one AVG over a column reads a table whose values have more fractional digits than the column).  Every other candidate is recorded as
    skipped with its reason."""
    k = _kat()
    assert (len(k["div"]), len(k["avg"]), len(k["compare"])) == (4, 0, 18)
    assert len(k["skipped"]) == 41 and all(s["reason"] for s in k["skipped"])


def _operand(o, n):
    return o["values"] if "values" in o else [o["const"]] * n


def test_decimal_result_divisions():
    for e in _kat()["div"]:
        n = len(e["a"]["values"]) if "values" in e["a"] else len(e["b"]["values"])
        a, b = _operand(e["a"], n), _operand(e["b"], n)
        got = [R.div(x, y, e["a"]["scale"], e["b"]["scale"]) for x, y in zip(a, b)]
        assert all(s == e["result_scale"] for _, s in got), e["sql"]
        assert sorted(v for v, _ in got) == sorted(_unscaled(t, e["result_scale"]) for t in e["result"]), e["sql"]


def test_decimal_result_comparisons():
    for e in _kat()["compare"]:
        width = 128 if max(e["precision"], e["const_precision"]) > 18 else 64
        hits = sum(1 for v in e["values"] if v is not None and R.compare(e["op"], v, e["const"], e["scale"], e["const_scale"], width))
        assert hits == e["rows"], e["sql"]


def test_decimal128_div_equals_div_one_for_avg():
    """decAvg's Decimal128.Div and the d128DivOne steps the device shares between DIV and AVG agree for every count, sums near +-2^127
    included: the independent restatement of Div holds the shortcut to account"""
    import random
    rng = random.Random(3)
    sums = [-(1 << 127), (1 << 127) - 1, -(1 << 127) + 1, 0, 1, -1] + [rng.randrange(-(1 << 127), 1 << 127) for _ in range(3000)]
    for scale in (0, 2, 6, 12, 18, 38):
        for t in sums:
            c = rng.choice([1, 2, 3, 7, 10 ** 6, rng.randrange(1, 1 << 63)])
            assert R.decimal128_div(t, c, scale, 0)[0] == R._div_one(t, c, R.div_scale(scale) - scale, keep=True), (t, c, scale)
