"""GPU parity of the decimal comparisons, BETWEEN, division and AVG (csrc/decimal.cu, goelem.cu) with the Python-integer restatement
(decimal_div_reference.py), exactly: values, nulls, return codes and the first failing row; then TPC-H Q6's predicates as real DECIMAL
compares and Q1's averages through DEC_SUM -> DEC_AVG over the reference's lineitem."""
import numpy as np
import pytest

import decimal_div_reference as R
import golden_tables as G
import oracle_lib as O
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer

pytestmark = pytest.mark.gpu

MAX64, MAX128 = (1 << 63) - 1, (1 << 127) - 1


def _bits(words, n):
    return [bool((int(words[i >> 6]) >> (i & 63)) & 1) for i in range(n)]


def _words(flags):
    n = len(flags)
    b = np.zeros(((n + 63) // 64) * 64, dtype=bool)
    b[:n] = flags
    return np.packbits(b, bitorder="little").view(np.uint64).copy()


def _col(width, vals):
    return np.asarray(vals, dtype=np.int64) if width == 64 else O.int_to_d128(vals)


def _values(rng, width, n, scale):
    """mixed magnitudes: small, near the type's limits, and values whose scale-up overflows"""
    top = MAX64 if width == 64 else MAX128
    out = []
    for _ in range(n):
        k = rng.integers(0, 6)
        if k == 0:
            v = int(rng.integers(-1000, 1000))
        elif k == 1:
            v = int(rng.integers(-10 ** 15, 10 ** 15))
        elif k == 2:
            v = int(rng.choice([top, -top, -top - 1, top - 1, 0, 1, -1]))
        elif k == 3:
            v = int(rng.integers(-(2 ** 62), 2 ** 62)) * (1 if width == 64 else int(rng.integers(1, 2 ** 40)))
        else:
            e = int(rng.integers(0, 18 if width == 64 else 37))
            v = int(rng.integers(1, 10)) * 10 ** e * int(rng.choice([-1, 1]))
        out.append(max(-top - 1, min(top, v)))
    return out


def _width_scales(scales):
    return [(w, s) for w in (64, 128) for s in scales if w == 128 or max(s) <= 18]


@pytest.mark.parametrize("width,scales", _width_scales([(2, 2), (2, 3), (3, 2), (0, 18), (18, 0), (0, 38), (38, 0), (5, 24)]))
@pytest.mark.parametrize("shape", ["vv", "vc", "cv"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 2000])
def test_compare_matches_restatement(gpu, width, scales, shape, n):
    rng = np.random.default_rng(n * 7 + scales[0] * 41 + scales[1] + width + len(shape))
    a = _values(rng, width, n, scales[0]); b = _values(rng, width, n, scales[1])
    c1, c2 = shape == "cv" and n > 1, shape == "vc" and n > 1
    if c1:
        a = [a[0]] * n
    if c2:
        b = [b[0]] * n
    na = None if c1 else list(rng.random(n) < 0.1)
    nb = None if c2 else list(rng.random(n) < 0.1)
    pre = list(rng.random(n) < 0.05)
    for op in range(6):
        r, rn = ops.dec_compare(op, width, _col(width, a[:1] if c1 else a), _col(width, b[:1] if c2 else b), scales[0], scales[1], n,
                                None if na is None else _words(na), None if nb is None else _words(nb), _words(pre))
        nulls = _bits(rn, n)
        for i in range(n):
            want_null = pre[i] or (na is not None and na[i]) or (nb is not None and nb[i])
            assert nulls[i] == want_null, (op, i)
            if not want_null:
                assert bool(r[i]) == R.compare(op, a[i], b[i], scales[0], scales[1], width), (op, i, a[i], b[i])


@pytest.mark.parametrize("width", [64, 128])
def test_compare_scale_up_overflow_compares_unscaled(gpu, width):
    top = MAX64 if width == 64 else MAX128
    d = 18 if width == 64 else 38
    a = [top, -top - 1, 10 ** 18 if width == 64 else 10 ** 37, 5]
    b = [0, 0, 0, 5 * 10 ** d]
    for op in range(6):
        r, rn = ops.dec_compare(op, width, _col(width, a), _col(width, b), 0, d, 4)
        assert [bool(v) for v in r] == [R.compare(op, x, y, 0, d, width) for x, y in zip(a, b)]
    r, _ = ops.dec_compare(4, 64, _col(64, [10 ** 18]), _col(64, [0]), 0, 1, 1)   # 10^18 * 10 wraps negative in Decimal64.Scale
    assert bool(r[0]) is True


@pytest.mark.parametrize("width", [64, 128])
def test_compare_const_null_nulls_every_row(gpu, width):
    n = 100
    a = _col(width, list(range(n)))
    r, rn = ops.dec_compare(0, width, a, _col(width, [3]), 2, 2, n, None, np.ones(1, dtype=np.uint64))
    assert all(_bits(rn, n))
    r, rn = ops.dec_compare(0, width, _col(width, [3]), a, 2, 2, n, np.ones(1, dtype=np.uint64), None)
    assert all(_bits(rn, n))


@pytest.mark.parametrize("width", [64, 128])
def test_compare_bad_scales_and_short_buffers(gpu, width):
    a = _col(width, [1, 2, 3])
    lim = 18 if width == 64 else 38
    for s1, s2 in ((-1, 0), (0, lim + 1), (lim + 1, 0)):
        with pytest.raises(capi.MoError) as e:
            ops.dec_compare(0, width, a, a, s1, s2, 3)
        assert e.value.rc == capi.RC_INVALID_ARGUMENT
    with pytest.raises(capi.MoError):
        ops.dec_compare(0, width, a[:2], a, 0, 0, 3)


@pytest.mark.parametrize("width", [64, 128])
def test_compare_device_form_is_async_and_exact(gpu, width):
    rng = np.random.default_rng(width)
    n = 3 * 132 * 8 * 256 + 17                              # above three grid strides
    a = [int(v) for v in rng.integers(-10 ** 12, 10 ** 12, n)]
    b = [int(v) for v in rng.integers(-10 ** 12, 10 ** 12, n)]
    ad, bd = DeviceBuffer.from_numpy(_col(width, a)), DeviceBuffer.from_numpy(_col(width, b))
    out, outn = DeviceBuffer(n), DeviceBuffer.from_numpy(np.zeros((n + 63) // 64, dtype=np.uint64))
    ops.dec_compare_device(2, width, ad, bd, 2, 4, n, out, outn)
    got = out.to_numpy(np.uint8)
    want = [R.compare(2, x, y, 2, 4, width) for x, y in zip(a, b)]
    assert [bool(v) for v in got] == want
    assert not any(outn.to_numpy(np.uint64))


@pytest.mark.parametrize("width", [64, 128])
def test_between_at_bounds(gpu, width):
    top = MAX64 if width == 64 else MAX128
    lo, hi = -5 * 10 ** 10, 7 * 10 ** 10
    vals = [lo - 1, lo, lo + 1, 0, hi - 1, hi, hi + 1, top, -top - 1, 3]
    nulls = [False] * 9 + [True]
    r, rn = ops.dec_between(width, _col(width, vals), lo, hi, len(vals), _words(nulls))
    assert [bool(v) for v in r] == [(not z) and lo <= v <= hi for v, z in zip(vals, nulls)]
    assert _bits(rn, len(vals)) == nulls


def _div_expect(width, a, b, s1, s2, pre, div0_error):
    """the serial d64Div / d128Div loop: (results by row, nulls, err_row, kind)"""
    n = len(a)
    out, nulls = [None] * n, list(pre)
    for i in range(n):
        if b[i] == 0 and not nulls[i]:
            if div0_error:
                return out, nulls, i, "zero"
            nulls[i] = True
            continue
        if nulls[i]:
            continue
        try:
            out[i] = R.div(a[i], b[i], s1, s2)[0]
        except (R.DivOverflow, R.NoEnd):
            return out, nulls, i, "overflow"
    return out, nulls, -1, None


def _div_values(rng, width, n, big):
    top = MAX64 if width == 64 else MAX128
    res = []
    for _ in range(n):
        k = rng.integers(0, 5)
        if k == 0:
            v = int(rng.integers(-10 ** 9, 10 ** 9))
        elif k == 1 or width == 64:
            v = int(rng.integers(-(2 ** 63) + 1, 2 ** 63 - 1)) >> int(rng.integers(0, 60))
        elif k == 2:
            v = int(rng.integers(1, 2 ** 62)) * (1 << 64) + int(rng.integers(0, 2 ** 62))   # just above 2^64 and beyond
        elif k == 3:
            v = top - int(rng.integers(0, 2 ** 40)) if big else (1 << 64) + int(rng.integers(0, 1000))
        else:
            v = int(rng.integers(-(2 ** 62), 2 ** 62)) << int(rng.integers(0, 64))
        if rng.random() < 0.5:
            v = -v
        res.append(max(-top - 1, min(top, v)))
    return res


@pytest.mark.parametrize("width,scales", _width_scales([(2, 2), (0, 0), (12, 0), (2, 6), (0, 18), (6, 12), (0, 30), (20, 38)]))
@pytest.mark.parametrize("shape", ["vv", "vc", "cv"])
def test_div_matches_restatement(gpu, width, scales, shape):
    rng = np.random.default_rng(scales[0] * 101 + scales[1] * 7 + width + len(shape) * 3 + (shape == "cv"))
    n = 1500
    a = _div_values(rng, width, n, True); b = _div_values(rng, width, n, False)
    # the 2^126 quirk and the 256-bit fallback, by construction
    if width == 128:
        a[:7] = [0x77202ec9ffed9235288bc781ae662675, 7 << 124, 3 * 10 ** 32, 10 ** 38 - 1, MAX128, -MAX128 - 1, MAX128 // 3]
        b[:7] = [0x2033e1ac4ee207f9da94e3e8ab73738f, 2 << 124, -3, 10 ** 10, MAX128, -MAX128, -MAX128 - 1]   # divisors near and at 2^127
    c1, c2 = shape == "cv", shape == "vc"
    if c1:
        a = [a[1] if a[1] else 7] * n
    if c2:
        b = [b[5] if b[5] else 3] * n
    for i in range(n):                                   # keep most rows clear of zero divisors; the error tests place them
        if b[i] == 0:
            b[i] = 1
    pre = list(rng.random(n) < 0.05)
    rc, r, rn, er, msg = ops.dec_div(width, _col(width, a[:1] if c1 else a), _col(width, b[:1] if c2 else b), scales[0], scales[1], n,
                                     rnulls=_words(pre))
    out, nulls, er0, kind = _div_expect(width, a, b, scales[0], scales[1], pre, False)
    assert er == er0
    assert rc == (0 if er0 < 0 else capi.RC_INVALID_ARGUMENT)
    if er0 >= 0:
        assert "Decimal128 Div overflow at row %d" % er0 in msg
    got = O.d128_to_int(r)
    gotn = _bits(rn, n)
    upto = n if er0 < 0 else er0
    assert gotn[:upto] == nulls[:upto]
    assert all(got[i] == out[i] for i in range(upto) if not nulls[i])


@pytest.mark.parametrize("width", [64, 128])
@pytest.mark.parametrize("order", ["zero_first", "overflow_first"])
def test_div_first_failing_row(gpu, width, order):
    n = 40
    top = MAX64 if width == 64 else MAX128
    a = [10 ** 3] * n; b = [7] * n
    s1, s2 = (0, 18) if width == 64 else (0, 20)
    ovf_a = top                                           # |x| * 10^adj leaves 127 bits and the quotient overflows
    zi, oi = (5, 9) if order == "zero_first" else (9, 5)
    b[zi] = 0
    a[oi] = ovf_a; b[oi] = 1
    rc, r, rn, er, msg = ops.dec_div(width, _col(width, a), _col(width, b), s1, s2, n, div0_error=True)
    assert er == min(zi, oi)
    if order == "zero_first":
        assert rc == capi.RC_DIVISION_BY_ZERO and "division by zero" in msg
    else:
        assert rc == capi.RC_INVALID_ARGUMENT and "Decimal128 Div overflow at row 5" in msg
    got = O.d128_to_int(r)
    assert all(got[i] == R.div(a[i], b[i], s1, s2)[0] for i in range(min(zi, oi)))
    # NULL mode: the zero divisor is NULL and only the overflow fails
    rc, r, rn, er, msg = ops.dec_div(width, _col(width, a), _col(width, b), s1, s2, n)
    assert er == oi and rc == capi.RC_INVALID_ARGUMENT
    if order == "zero_first":
        assert _bits(rn, n)[zi]


@pytest.mark.parametrize("width", [64, 128])
def test_div_const_zero_and_const_null(gpu, width):
    n = 70
    a = _col(width, list(range(1, n + 1)))
    rc, r, rn, er, _ = ops.dec_div(width, a, _col(width, [0]), 2, 2, n)
    assert rc == 0 and er == -1 and all(_bits(rn, n))
    rc, r, rn, er, _ = ops.dec_div(width, a, _col(width, [0]), 2, 2, n, rnulls=_words([True] * n), div0_error=True)
    assert rc == capi.RC_DIVISION_BY_ZERO and er == 0     # a const zero divisor fails before any row is looked at
    rc, r, rn, er, _ = ops.dec_div(width, a, _col(width, [5]), 2, 2, n, n2=np.ones(1, dtype=np.uint64))
    assert rc == 0 and all(_bits(rn, n))


@pytest.mark.parametrize("width", [64, 128])
def test_div_bad_scales_and_short_buffers(gpu, width):
    a = _col(width, [1, 2, 3])
    lim = 18 if width == 64 else 38
    for s in ((-1, 0), (0, lim + 1)):
        rc, *_ = ops.dec_div(width, a, a, s[0], s[1], 3)
        assert rc == capi.RC_INVALID_ARGUMENT
    rc, *_ = ops.dec_div(width, a[:2], a, 0, 0, 3)
    assert rc == capi.RC_INVALID_ARGUMENT


@pytest.mark.parametrize("width", [64, 128])
def test_div_device_form(gpu, width):
    rng = np.random.default_rng(5 + width)
    n = 3 * 132 * 8 * 256 + 5
    a = [int(v) for v in rng.integers(-10 ** 15, 10 ** 15, n)]
    b = [int(v) or 1 for v in rng.integers(-10 ** 6, 10 ** 6, n)]
    out, outn = DeviceBuffer(16 * n), DeviceBuffer.from_numpy(np.zeros((n + 63) // 64, dtype=np.uint64))
    rc, er, _ = ops.dec_div_device(width, DeviceBuffer.from_numpy(_col(width, a)), DeviceBuffer.from_numpy(_col(width, b)), 2, 2, n, out, outn)
    assert rc == 0 and er == -1
    got = O.d128_to_int(out.to_numpy(np.uint64).reshape(-1, 2))
    idx = list(range(0, n, 97)) + [n - 1]
    assert all(got[i] == R.div(a[i], b[i], 2, 2)[0] for i in idx)


@pytest.mark.parametrize("width", [64, 128])
@pytest.mark.parametrize("scale", [0, 2, 6, 12, 18])
def test_avg_matches_restatement(gpu, width, scale):
    rng = np.random.default_rng(scale + width)
    g = 1000
    sums = [int(v) for v in rng.integers(-(2 ** 62), 2 ** 62, g)]
    cnts = [int(v) for v in rng.integers(0, 5, g)]
    sums[:6] = [MAX128, -MAX128 - 1, MAX128 - 7, -(10 ** 37), 1, -1]
    cnts[:6] = [1, 1, 3, 7, 0, 2]
    r, rn = ops.dec_avg(width, O.int_to_d128(sums), np.asarray(cnts, dtype=np.int64), scale)
    got, nulls = O.d128_to_int(r), _bits(rn, g)
    for i in range(g):
        assert nulls[i] == (cnts[i] == 0)
        if cnts[i]:
            assert got[i] == R.avg(sums[i], cnts[i], scale)[0], (i, sums[i], cnts[i])


def test_avg_million_groups_device_form(gpu):
    g = 10 ** 6
    rng = np.random.default_rng(11)
    sums = rng.integers(-(2 ** 62), 2 ** 62, g).astype(np.int64)
    cnts = rng.integers(0, 1000, g).astype(np.int64)
    s128 = np.stack([sums.view(np.uint64), np.where(sums < 0, np.uint64(2 ** 64 - 1), np.uint64(0))], axis=1).copy()
    out, outn = DeviceBuffer(16 * g), DeviceBuffer((g + 63) // 64 * 8)
    ops.dec_avg_device(64, DeviceBuffer.from_numpy(s128), DeviceBuffer.from_numpy(cnts), g, 2, out, outn)
    got = out.to_numpy(np.uint64).reshape(-1, 2)
    nulls = outn.to_numpy(np.uint64)
    for i in list(range(0, g, 4999)) + [g - 1]:
        assert bool((int(nulls[i >> 6]) >> (i & 63)) & 1) == (cnts[i] == 0)
        if cnts[i]:
            assert O.d128_to_int(got[i:i + 1])[0] == R.avg(int(sums[i]), int(cnts[i]), 2)[0]


def test_avg_short_buffers_and_bad_scale(gpu):
    with pytest.raises(capi.MoError):
        ops.dec_avg(64, np.zeros((1, 2), dtype=np.uint64), np.ones(2, dtype=np.int64), 2)
    with pytest.raises(capi.MoError):
        ops.dec_avg(64, np.zeros((2, 2), dtype=np.uint64), np.ones(2, dtype=np.int64), 19)


def test_tpch_q6_with_decimal_predicates_and_q1_averages(gpu):
    """Q6's predicates as DECIMAL(15,2) compares and BETWEEN (quantity < 24 passed at scale 0), then Q1's averages through DEC_SUM -> DEC_AVG"""
    cols, ints, expected = G.tpch_fixture()
    n = len(cols["shipdate"])
    qty = ints["quantity"] * 100; price = ints["extendedprice_cents"]; disc = ints["discount_pct"]
    P = datagen.q6_params()
    from matrixone_b200.vector import Vector, xcall

    def date_cmp(op, const):
        r = np.zeros(n, dtype=np.uint8); rn = np.zeros((n + 63) // 64, dtype=np.uint64)
        xcall(capi.XCALL_GO_COMPARE(op, capi.T_DATE), [Vector(data=r, nulls=rn, length=n), Vector(data=cols["shipdate"], length=n),
                                                       Vector(data=np.asarray([const], dtype=np.int32), length=n)], n)
        return r
    btw, _ = ops.dec_between(64, disc, 2, 4, n)                                        # discount between 0.02 and 0.04 (scale 2 bounds)
    lt, _ = ops.dec_compare(4, 64, qty, np.asarray([24], dtype=np.int64), 2, 0, n)     # quantity < 24: the constant at scale 0
    m = date_cmp(3, P[0]) & date_cmp(4, P[1]) & btw & lt
    sels = ops.filter_sels(m)
    rc, prod, _, _ = ops.dec_arith(2, 64, ops.shuffle(price, sels), ops.shuffle(disc, sels), 2, 2, len(sels))
    assert rc == 0
    s = np.zeros((1, 2), dtype=np.uint64); c = np.zeros(1, dtype=np.int64)
    ops.dec_sum(128, prod, s, c, None, None, len(sels))
    assert O.decimal_str(O.d128_to_int(s)[0], 4) == expected["q6_revenue"]
    # ---- Q1 averages
    cut = np.zeros(n, dtype=np.uint8); cn = np.zeros((n + 63) // 64, dtype=np.uint64)
    xcall(capi.XCALL_GO_COMPARE(5, capi.T_DATE), [Vector(data=cut, nulls=cn, length=n), Vector(data=cols["shipdate"], length=n),
                                                  Vector(data=np.asarray([datagen.Q1_CUTOFF], dtype=np.int32), length=n)], n)
    sels = ops.filter_sels(cut)
    k = len(sels)
    keys, _ = ops.pack_keys([ops.shuffle(cols["returnflag"], sels), ops.shuffle(cols["linestatus"], sels)], has_null=False)
    table = ops.GroupTable(16)
    groups = table.insert(keys)
    ng = int(table.ngroups[0])
    avgs = []
    for col in (qty, price, disc):
        sm = np.zeros((ng, 2), dtype=np.uint64); cnt = np.zeros(ng, dtype=np.int64)
        ops.dec_sum(64, ops.shuffle(col, sels), sm, cnt, groups, None, k)
        r, rn = ops.dec_avg(64, sm, cnt, 2)
        assert not any(_bits(rn, ng))
        sums = O.d128_to_int(sm)
        vals = O.d128_to_int(r)
        assert vals == [R.avg(sums[g], int(cnt[g]), 2)[0] for g in range(ng)]
        avgs.append(vals)
    assert ng == len(expected["q1"])
    for g in range(ng):
        e = expected["q1"][(chr(int(table.keys[g]) & 0xff), chr((int(table.keys[g]) >> 8) & 0xff))]
        got = []
        for v in (avgs[0][g], avgs[1][g], avgs[2][g]):
            q, rem = divmod(abs(v), 10 ** 6)
            q += 2 * rem >= 10 ** 6
            got.append(O.decimal_str(-q if v < 0 else q, 2))
        assert got == [e["avg_qty"], e["avg_price"], e["avg_disc"]]
