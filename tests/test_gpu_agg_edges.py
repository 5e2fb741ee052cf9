"""Single-column aggregates (csrc/agg.cu, MO_XCALL_AGG), grouped aggregates (csrc/colops.cu, MO_XCALL_GROUP_AGG) and the merge of
partial states (MO_XCALL_AGG_MERGE) at the edges of their loops, against the oracle's restatement of the Go loops (oracle_go.c).

- Every row count of agg_cases.regions() (each loop path of agg_kernel, with 0 .. V - 1 scalar-tail rows), for host columns, device
  columns and device columns offset by 1 .. V - 1 elements (the whole-column scalar path), with the SM count read from the device.
- MIN / MAX are compared bit for bit through an unsigned view: the serial loop keeps the first row that reaches the extreme, so
  -0.0 and 0.0 are told apart, and NaN payloads are kept.  Integer SUM, AVG and COUNT are exact.
- Null rows hold poison (a value no live row has), so a null bit read for the wrong row changes the exact result.

Float SUM overflowing to inf during accumulation depends on the summation order; no case here reaches it."""
import math

import numpy as np
import pytest

import agg_cases as A
import oracle_lib as O
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer, bitmap_from_bools, bitmap_to_bools

pytestmark = pytest.mark.gpu

I64MAX = np.iinfo(np.int64).max
I64MIN = np.iinfo(np.int64).min
MM_TYPES = [capi.T_INT8, capi.T_INT16, capi.T_INT32, capi.T_INT64, capi.T_UINT8, capi.T_UINT16, capi.T_UINT32, capi.T_UINT64,
            capi.T_FLOAT32, capi.T_FLOAT64, capi.T_DATE, capi.T_TIMESTAMP]
UINT_OF = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dt(T):
    return np.dtype(capi.NP_OF_T[T])


def _kind(T):
    """"i", "u" or "f" for a summable type, None for DATE / TIMESTAMP (COUNT, MIN and MAX only)"""
    if capi.T_INT8 <= T <= capi.T_INT64:
        return "i"
    if capi.T_UINT8 <= T <= capi.T_UINT64:
        return "u"
    return "f" if T in (capi.T_FLOAT32, capi.T_FLOAT64) else None


def _bits(x, dt):
    """the bits of one value of type dt, as a Python int"""
    return int(np.asarray([x], dtype=dt).view(UINT_OF[np.dtype(dt).itemsize])[0])


def _words(mask):
    return bitmap_from_bools(np.asarray(mask, bool))


class Oracle:
    """the Go loops of SUM / COUNT / MIN / MAX over one column, advanced over row ranges [prev, n) so that a sweep over rising n
    reads every row once"""

    def __init__(self, T, col, words):
        self.T, self.col, self.words, self.dt, self.prev = T, col, words, col.dtype, 0
        k = _kind(T)
        self.sum = np.zeros(1, np.float64 if k == "f" else (np.uint64 if k == "u" else np.int64))
        self.snul = np.ones(1, np.uint8)
        self.scnt = np.zeros(1, np.int64)
        self.cnt = np.zeros(1, np.int64)
        self.mm = {m: np.zeros(1, self.dt) for m in (0, 1)}
        self.mmnul = {m: np.ones(1, np.uint8) for m in (0, 1)}
        self.rc = 0

    def advance(self, n):
        g, T, k, d = O.go(), self.T, _kind(self.T), n - self.prev
        c, w = O.p(self.col), O.p(self.words)
        if k == "i" and not self.rc:
            self.rc = g.og_sum_int64(T, c, w, self.prev, None, d, O.p(self.sum), O.p(self.snul), O.p(self.scnt), None)
        elif k == "u" and not self.rc:
            self.rc = g.og_sum_uint64(T, c, w, self.prev, None, d, O.p(self.sum), O.p(self.snul), O.p(self.scnt), None)
        elif k == "f":
            g.og_sum_float64(T, c, w, self.prev, None, d, O.p(self.sum), O.p(self.snul), O.p(self.scnt))
        g.og_count(0, w, self.prev, None, d, O.p(self.cnt))
        for m in (0, 1):
            assert g.og_minmax(m, T, c, w, self.prev, None, d, O.p(self.mm[m]), O.p(self.mmnul[m])) == 0
        self.prev = n

    def check(self, col, nulls, n, what):
        """run every op on (col, nulls, n) -- numpy or DeviceBuffer -- and compare with the oracle's state at n"""
        T, k = self.T, _kind(self.T)
        assert ops.agg_count(T, col, nulls, n) == int(self.cnt[0]), what
        for m, fn in ((0, ops.agg_min), (1, ops.agg_max)):
            got, isnull = fn(T, col, nulls, n)
            assert isnull == bool(self.mmnul[m][0]), what
            if not isnull:
                assert _bits(got, self.dt) == _bits(self.mm[m][0], self.dt), (what, "max" if m else "min", got, self.mm[m][0])
        if k is None:
            return
        rc, s, isnull = ops.agg_sum(T, col, nulls, n)
        assert rc == self.rc and isnull == bool(self.snul[0]), what
        if isnull or rc:
            return
        if k == "f":
            assert _bits(s, np.float64) == _bits(self.sum[0], np.float64), (what, s, self.sum[0])
        else:
            assert s == int(self.sum[0]), what
        rca, avg, nula = ops.agg_avg(T, col, nulls, n)
        assert not nula and _bits(avg, np.float64) == _bits(float(self.sum[0]) / float(self.scnt[0]), np.float64), what


# ------------------------------------------------------------------------------------------------------------------ H0 sweep
@pytest.mark.parametrize("T", MM_TYPES)
def test_h0_every_loop_region_host_device_and_unaligned(gpu, T):
    dt = _dt(T)
    sz = dt.itemsize
    V = A.vec_rows(sz)
    sms = _sms()
    sizes = [n for n, _ in A.regions(sz, sms)]
    assert A.loop_counts(sizes[-1], sz, sms)["unrolled"] > 0 and A.loop_counts(sizes[-1], sz, sms)["grid"] == 4 * sms
    rng = np.random.default_rng(T)
    N = sizes[-1] + V
    col, mask = A.poisoned_column(dt, N, rng)
    dcol = DeviceBuffer.from_numpy(col)
    for k in range(V):                      # k = 0: host and aligned device columns; k > 0: the column starts k elements in
        ck = np.ascontiguousarray(col[k:])
        wk = _words(mask[k:])               # bits past n in the last word are rows n, n + 1, ... of the longer column
        dw = DeviceBuffer.from_numpy(wk)
        dv = dcol.view(sz * (N - k), offset=sz * k)
        orc = Oracle(T, ck, wk)
        for n in sizes:
            orc.advance(n)
            orc.check(dv, dw, n, ("device", k, n))
            if k == 0:
                orc.check(ck, wk, n, ("host", n))
        dw.free()
    dcol.free()


@pytest.mark.parametrize("T", MM_TYPES)
def test_h0_planted_extremes(gpu, T):
    """the unique extreme at the first and last row, at row 64k + 63, right after a null row and at the first row of each loop path,
    with a more extreme value in the null row next to it"""
    dt = _dt(T)
    sz = dt.itemsize
    V = A.vec_rows(sz)
    sms = _sms()
    lo, hi = A.live_band(dt)
    rng = np.random.default_rng(T + 100)
    bases = A.region_bases(sz, sms)
    # below the unrolled loop: 0, 1 and V - 1 tail rows; with it (the largest columns): its first size with V - 1 tail rows and
    # its last with none
    sizes = [nvec * V + t for _, nvec in bases[:4] for t in sorted({0, 1, V - 1})] + [bases[4][1] * V + V - 1, bases[-1][1] * V]
    for n in sizes:
        if n < 2:
            continue
        col, mask = A.poisoned_column(dt, n, rng)
        for name, row in A.planted_rows(n, sz, sms, mask).items():
            for is_max in (0, 1):
                c, m = col.copy(), mask.copy()
                A.plant_extreme(c, m, row, is_max, hi + 1 if is_max else lo - 1)
                w = _words(m)
                want, wn = np.zeros(1, dt), np.ones(1, np.uint8)
                O.go().og_minmax(is_max, T, O.p(c), O.p(w), 0, None, n, O.p(want), O.p(wn))
                assert want[0] == dt.type(hi + 1 if is_max else lo - 1)          # the case is what it claims
                got, isnull = (ops.agg_max if is_max else ops.agg_min)(T, c, w, n)
                assert not isnull and _bits(got, dt) == _bits(want[0], dt), (n, name, is_max)


# ------------------------------------------------------------------------------------------------------------------ H0 +-0 and NaN
def _minmax_want(is_max, T, col, words, n):
    want, wn = np.zeros(1, col.dtype), np.ones(1, np.uint8)
    O.go().og_minmax(is_max, T, O.p(col), O.p(words), 0, None, n, O.p(want), O.p(wn))
    return want[0], bool(wn[0])


def _check_minmax_all_forms(T, col, words, n, what, offsets=(0,)):
    """host, device and device-offset columns, against the oracle, bit for bit"""
    dt = col.dtype
    for is_max, fn in ((0, ops.agg_min), (1, ops.agg_max)):
        want, wn = _minmax_want(is_max, T, col, words, n)
        got, gn = fn(T, col, words, n)
        assert gn == wn and (wn or _bits(got, dt) == _bits(want, dt)), (what, "host", is_max, got, want)
        for k in offsets:
            buf = np.zeros(n + k, dt)
            buf[k:] = col
            db = DeviceBuffer.from_numpy(buf)
            dw = DeviceBuffer.from_numpy(words) if words is not None else None
            got, gn = fn(T, db.view(n * dt.itemsize, offset=k * dt.itemsize), dw, n)
            assert gn == wn and (wn or _bits(got, dt) == _bits(want, dt)), (what, "device", k, is_max, got, want)
            db.free()
            if dw is not None:
                dw.free()


@pytest.mark.parametrize("T", [capi.T_FLOAT32, capi.T_FLOAT64])
def test_h0_min_max_keep_the_first_zero(gpu, T):
    """-0.0 and 0.0 tie under the strict compare: the result is the zero of the first row that reaches the extreme, also when a
    thread before it in lane, CTA or tail order holds the other zero"""
    dt = _dt(T)
    sz = dt.itemsize
    V = A.vec_rows(sz)
    sms = _sms()
    nt = 4 * sms * 256
    for v in ([5.0, 5.0, -0.0, -0.0, 0.0, 0.0], [1.0, -0.0, 0.0], [-1.0, -0.0, 0.0], [0.0, -0.0], [-0.0, 0.0], [-0.0], [0.0, 0.0, -0.0]):
        c = np.asarray(v, dt)
        _check_minmax_all_forms(T, c, None, len(c), v, offsets=(0, 1))
    for kind, n in (("lane", 3 * nt * V + 1), ("lane", 100 * V + 1), ("cta", 3 * nt * V), ("cta", 9 * nt * V + V - 1),
                    ("tail", 100 * V + 3), ("tail", 8 * nt * V + V - 1)):
        first, other = A.zero_tie_rows(n, sz, sms, kind)
        for z1, z2 in ((-0.0, 0.0), (0.0, -0.0)):
            for is_max in (0, 1):
                c = np.full(n, -1.0 if is_max else 1.0, dt)
                c[first], c[other] = z1, z2
                mask = np.zeros(n, bool)
                mask[first - 1] = True                     # a null row before the first zero holds a zero of the other sign
                c[first - 1] = z2
                w = _words(mask)
                want, _ = _minmax_want(is_max, T, c, w, n)
                assert _bits(want, dt) == _bits(z1, dt)
                got, _ = (ops.agg_max if is_max else ops.agg_min)(T, c, w, n)
                assert _bits(got, dt) == _bits(z1, dt), (kind, n, z1, is_max)
                dc, dw = DeviceBuffer.from_numpy(c), DeviceBuffer.from_numpy(w)
                got, _ = (ops.agg_max if is_max else ops.agg_min)(T, dc, dw, n)
                assert _bits(got, dt) == _bits(z1, dt), (kind, n, z1, is_max, "device")
                dc.free(); dw.free()
    # the unaligned scalar path: row r is read by thread r mod (grid threads); the first zero at thread 5, another at thread 0
    n = 2 * nt + 7
    for z1, z2 in ((-0.0, 0.0), (0.0, -0.0)):
        c = np.full(n, 1.0, dt)
        c[5], c[nt] = z1, z2
        _check_minmax_all_forms(T, c, None, n, ("unaligned", z1), offsets=(1,))


def _nan(dt, payload, neg=False):
    u = UINT_OF[np.dtype(dt).itemsize]
    if np.dtype(dt).itemsize == 8:
        b = 0x7FF8000000000000 | payload | (1 << 63 if neg else 0)
    else:
        b = 0x7FC00000 | payload | (1 << 31 if neg else 0)
    return np.asarray([b], u).view(dt)[0]


@pytest.mark.parametrize("T", [capi.T_FLOAT32, capi.T_FLOAT64])
def test_h0_nan_rules_and_payloads(gpu, T):
    """a NaN first live row is never replaced (and its payload is kept); a NaN later is never taken; all-NaN gives the first NaN"""
    dt = _dt(T)
    sz = dt.itemsize
    V = A.vec_rows(sz)
    nt = 4 * _sms() * 256
    rng = np.random.default_rng(T)
    for n in (7, 1000, 9 * nt * V + V - 1):
        base, mask = A.poisoned_column(dt, n, rng)
        mask[:3] = True
        nan1, nan2 = _nan(dt, 0x123), _nan(dt, 0x45, neg=True)
        cases = {}
        c = base.copy(); c[3] = nan1; c[n // 2] = nan2; cases["first live row NaN"] = c
        c = base.copy(); c[n // 2] = nan1; c[n - 1] = nan2; cases["NaN inside"] = c
        c = np.full(n, nan2, dt); c[n // 3] = nan1; cases["all NaN"] = c
        c = base.copy(); c[3:] = nan2; c[n - 1] = -0.0; cases["NaN then one zero"] = c
        for name, c in cases.items():
            w = _words(mask)
            _check_minmax_all_forms(T, c, w, n, (n, name), offsets=(0, 1))
            rc, s, isnull = ops.agg_sum(T, c, w, n)
            assert rc == 0 and not isnull and math.isnan(s), (n, name)
            assert math.isnan(ops.agg_avg(T, c, w, n)[1])


# ------------------------------------------------------------------------------------------------------------------ signed SUM gate
def _sum_i64_oracle(v, words):
    s, nul, c = np.zeros(1, np.int64), np.ones(1, np.uint8), np.zeros(1, np.int64)
    rc = O.go().og_sum_int64(capi.T_INT64, O.p(v), O.p(words), 0, None, len(v), O.p(s), O.p(nul), O.p(c), None)
    return rc, int(s[0]), bool(nul[0])


def _check_sum_i64(v, mask, what):
    v = np.ascontiguousarray(v, np.int64)
    words = None if mask is None else _words(mask)
    rc0, s0, n0 = _sum_i64_oracle(v, words)
    dv = DeviceBuffer.from_numpy(v)
    dw = None if words is None else DeviceBuffer.from_numpy(words)
    for col, nl, form in ((v, words, "host"), (dv, dw, "device")):
        rc, s, isnull = ops.agg_sum(capi.T_INT64, col, nl, len(v))
        assert rc == rc0, (what, form, rc, rc0)
        if rc0 == 0:
            assert (s, isnull) == (s0, n0), (what, form)
    dv.free()
    if dw is not None:
        dw.free()
    return rc0


def test_h0_signed_sum_gate_and_serial_check(gpu):
    """sum_check_needed: max|v| <= INT64_MAX / rows takes the fast path, one more runs the serial prefix check; rc equals the serial
    loop's in both"""
    R = capi.RC_OUT_OF_RANGE
    nt = 4 * _sms() * 256
    for n in (1000, 2 * 9 * nt + 1):
        m = I64MAX // n
        assert _check_sum_i64(np.full(n, m), None, ("fast path", n)) == 0
        assert _check_sum_i64(np.full(n, -m), None, ("fast path neg", n)) == 0
        assert _check_sum_i64(np.full(n, m + 1), None, ("one sign", n)) == R
        assert _check_sum_i64(np.full(n, -(m + 1)), None, ("one sign neg", n)) == R
        alt = np.full(n, m + 1); alt[1::2] = -(m + 1)
        assert _check_sum_i64(alt, None, ("alternating", n)) == 0
        mask = np.zeros(n, bool); mask[1::4] = True                   # the gate counts non-null rows only
        ml = I64MAX // int((~mask).sum())
        assert _check_sum_i64(np.where(mask, I64MAX, ml), mask, ("fast path, poisoned nulls", n)) == 0
        assert _check_sum_i64(np.where(mask, -2 ** 40, ml + 1), mask, ("one sign, nulls", n)) == R
    assert _check_sum_i64([I64MIN], None, "INT64_MIN") == 0
    assert _check_sum_i64([I64MIN, -1], None, "INT64_MIN, -1") == R
    assert _check_sum_i64([-1, I64MIN], None, "-1, INT64_MIN") == R
    assert _check_sum_i64([I64MIN, 1, -1], None, "INT64_MIN, 1, -1") == 0
    # the serial check splits the rows in 256 segments of seg = ceil(n / 256); prefixes that leave int64 exactly at a boundary
    for n in (256 * 40, 256 * 40 + 17, 2 * 9 * nt + 1):
        seg = -(-n // 256)
        for b in (seg, 3 * seg, 255 * seg):
            if b + 2 >= n:
                continue
            base = np.zeros(n, np.int64); base[0] = I64MAX
            mask = np.zeros(n, bool); mask[b] = True                      # null on the first row of the next segment, poisoned
            v = base.copy(); v[b - 1] = 1; v[b] = -2 ** 40; v[b + 1] = -5
            assert _check_sum_i64(v, mask, ("overflow on the segment's last row", n, b)) == R
            v = base.copy(); v[b - 1] = -5; v[b] = 2 ** 40; v[b + 1] = 1
            assert _check_sum_i64(v, mask, ("no overflow, poison in the null", n, b)) == 0
            v = base.copy(); v[b] = 1; v[b + 1] = -5
            assert _check_sum_i64(v, mask, ("the overflowing value is null", n, b)) == 0
            v = base.copy(); v[b + 1] = 1; v[b - 1] = -5
            assert _check_sum_i64(v, mask, ("after the boundary", n, b)) == 0
            v = base.copy(); v[b + 1] = 1; v[n - 1] = -5
            assert _check_sum_i64(v, mask, ("overflow on the next segment's second row", n, b)) == R


# ------------------------------------------------------------------------------------------------------------------ float SUM / AVG
@pytest.mark.parametrize("T", [capi.T_FLOAT32, capi.T_FLOAT64])
def test_h0_float_sum_error_bound_and_determinism(gpu, T):
    """|got - exact| <= (cnt - 1) 2^-53 sum |x| on data that cancels heavily; the bits repeat run to run and agree between the
    synchronous and the asynchronous (device state) forms"""
    dt = _dt(T)
    V = A.vec_rows(dt.itemsize)
    nt = 4 * _sms() * 256
    rng = np.random.default_rng(T)
    for n in (1000, 3 * nt * V + 5, 9 * nt * V + V - 1):
        h = n // 2
        a = rng.standard_normal(h) * 10.0 ** rng.integers(0, 12, h)
        x = np.empty(n)
        x[:h], x[h:2 * h] = a, -a + rng.standard_normal(h)
        x[2 * h:] = 1.0
        x = x[rng.permutation(n)].astype(dt)
        mask = rng.random(n) < 0.05
        x[mask] = 1e30 if dt == np.float64 else 3e38                 # poison
        live = x[~mask].astype(np.float64)
        exact, mag, cnt = math.fsum(live), float(np.abs(live).sum()), len(live)
        bound = (cnt - 1) * 2.0 ** -53 * mag * (1 + 1e-12)
        w = _words(mask)
        rc, s, isnull = ops.agg_sum(T, x, w, n)
        assert rc == 0 and not isnull and abs(s - exact) <= bound, (n, s, exact, bound)
        rca, avg, _ = ops.agg_avg(T, x, w, n)
        assert abs(avg - exact / cnt) <= bound / cnt + 2.0 ** -52 * abs(avg), n
        assert _bits(ops.agg_sum(T, x, w, n)[1], np.float64) == _bits(s, np.float64)
        dx, dw = DeviceBuffer.from_numpy(x), DeviceBuffer.from_numpy(w)
        for op in (capi.AGG_SUM, capi.AGG_AVG):
            st = ops.agg_state(op, T, x, w, n)
            out = DeviceBuffer(24)
            ops.agg_state_device(op, T, dx, dw, n, out.ptr)
            assert np.array_equal(out.to_numpy(np.uint64), st) and int(st[0]) == _bits(s, np.float64), (n, op)
            out.free()
        dx.free(); dw.free()
    for v, want in (([1.0, np.nan, 2.0], "nan"), ([np.inf, 1.0], "inf"), ([np.inf, -1.0, -np.inf], "nan"), ([-np.inf], "-inf"),
                    ([np.inf, np.nan], "nan")):
        for n in (len(v), 3 * nt * V + 1):
            c = np.zeros(n, dt)
            c[np.linspace(0, n - 1, len(v)).astype(int)] = v
            s = ops.agg_sum(T, c)[1]
            assert (math.isnan(s) if want == "nan" else s == float(want)), (v, n, s)


# ------------------------------------------------------------------------------------------------------------------ shared ticket
def test_shared_ticket_word_across_h0_q6_and_q1(gpu):
    """H0, Q6 and Q1 count their CTAs in the same device word, which wraps to 0 after each launch's last CTA: calls with grids of
    1, 2 and every SM, interleaved with Q6 and with Q1 (whose wide retry exits through its gate before the ticket), stay exact"""
    sms = _sms()
    nt = 4 * sms * 256
    rng = np.random.default_rng(5)
    h0 = []
    for n in (100, 2 * 2 * 256, 9 * nt * 2 + 1):
        v, mask = A.poisoned_column(np.int64, n, rng)
        w = _words(mask)
        assert A.grid_of(n, 8, sms) in (1, 2, 4 * sms)
        h0.append((v, w, n, _sum_i64_oracle(v, w), _minmax_want(0, capi.T_INT64, v, w, n)[0]))
    nq = 300_000
    cols = datagen.lineitem(10, 0, nq)
    P = datagen.q6_params()
    q6_want = O.q6(cols, nq, P, nthreads=4)
    q1_want = O.q1(cols, nq, datagen.Q1_CUTOFF, nthreads=4)
    names = ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")

    def run(step):
        if step < 3:
            v, w, n, (rc0, s0, _), mn = h0[step]
            assert ops.agg_sum(capi.T_INT64, v, w, n)[:2] == (rc0, s0), step
            assert ops.agg_min(capi.T_INT64, v, w, n)[0] == mn, step
        elif step == 3:
            s, rows, _ = ops.q6_filter_sum(cols["shipdate"], cols["discount"], cols["quantity"], cols["extendedprice"], nq, *P)
            assert rows == q6_want[1] and abs(s - q6_want[0]) <= 1e-9 * abs(q6_want[0])
        else:
            got = ops.q1_group_agg(*[cols[k] for k in names], nq, datagen.Q1_CUTOFF)
            assert [(g["returnflag"], g["linestatus"], g["count_order"]) for g in got] == \
                   [(g["returnflag"], g["linestatus"], g["count_order"]) for g in q1_want]
            assert all(abs(a["sum_charge"] - b["sum_charge"]) <= 1e-9 * abs(b["sum_charge"]) for a, b in zip(got, q1_want))

    for order in ([0, 1, 2, 3, 4], [2, 4, 0, 3, 1], [1, 3, 2, 0, 4, 2, 1, 0, 3], [4, 4, 0, 3, 3, 2, 2, 1, 1]):
        for step in order:
            run(step)


# ------------------------------------------------------------------------------------------------------------------ GROUP_AGG
NGROUPS = [1, 2, 512, 513, 1024, 1025, 5000]


def _group_data(T, ngroups, n, rng, op):
    dt = _dt(T)
    if dt.kind == "f" and op in (capi.AGG_MIN, capi.AGG_MAX):
        s = -1.0 if op == capi.AGG_MAX else 1.0
        col = rng.choice(np.asarray([0.0, -0.0, 1.5 * s, 3.0 * s]), n).astype(dt)     # most groups' extreme is a zero of either sign
        mask = rng.random(n) < 0.1
        col[mask] = -2.0 ** 40 * s
    else:
        col, mask = A.poisoned_column(dt, n, rng)
    groups = rng.integers(0, ngroups + 1, n).astype(np.uint64)                         # 0 = GroupNotMatched
    return col, mask, groups


@pytest.mark.parametrize("ngroups", NGROUPS)
def test_group_agg_group_table_edges(gpu, ngroups):
    """SUM, COUNT, MIN and MAX at the group counts where the shared-memory replication changes (512 / 513), where the global path
    starts (1025) and beyond, in two batches into one state; MIN / MAX bit for bit"""
    rng = np.random.default_rng(ngroups)
    n = max(20_000, 40 * ngroups) // 64 * 64 + 37
    h = (n // 3) // 64 * 64
    cases = [(capi.AGG_SUM, T) for T in (capi.T_INT8, capi.T_INT32, capi.T_INT64, capi.T_UINT16, capi.T_UINT64, capi.T_FLOAT32, capi.T_FLOAT64)]
    cases += [(capi.AGG_COUNT, capi.T_INT32)]
    cases += [(op, T) for op in (capi.AGG_MIN, capi.AGG_MAX) for T in (capi.T_INT8, capi.T_INT64, capi.T_UINT32, capi.T_UINT64,
                                                                        capi.T_FLOAT32, capi.T_FLOAT64)]
    for op, T in cases:
        dt = _dt(T)
        col, mask, groups = _group_data(T, ngroups, n, rng, op)
        if dt.kind == "f" and op in (capi.AGG_MIN, capi.AGG_MAX) and ngroups > 2:
            for g in (1, 2):                               # groups 2 and 3: batch 1 leaves NaN (first value) or +-0 in the state
                rows = np.flatnonzero((groups == g + 1) & ~mask)
                col[rows[0]] = np.nan if g == 1 else -0.0
        nulls = _words(mask)
        k = _kind(T)
        if op == capi.AGG_COUNT:
            want = np.zeros(ngroups, np.int64)
            O.go().og_count(0, O.p(nulls), 0, O.p(groups), n, O.p(want))
            got = np.zeros(ngroups, np.int64)
            assert ops.group_agg(op, T, got, None, None, groups[:h], col[:h], nulls[:h // 64], h) == 0
            assert ops.group_agg(op, T, got, None, None, groups[h:], col[h:], nulls[h // 64:], n - h) == 0
            assert np.array_equal(got, want), (ngroups, T)
            continue
        if op == capi.AGG_SUM:
            st_dt = np.float64 if k == "f" else (np.uint64 if k == "u" else np.int64)
            want, wn, wc = np.zeros(ngroups, st_dt), np.ones(ngroups, np.uint8), np.zeros(ngroups, np.int64)
            fn = {"f": O.go().og_sum_float64, "u": O.go().og_sum_uint64, "i": O.go().og_sum_int64}[k]
            args = [T, O.p(col), O.p(nulls), 0, O.p(groups), n, O.p(want), O.p(wn), O.p(wc)] + ([] if k == "f" else [None])
            assert fn(*args) == 0
            state = np.zeros(ngroups, st_dt)
        else:
            want, wn = np.zeros(ngroups, dt), np.ones(ngroups, np.uint8)
            assert O.go().og_minmax(int(op == capi.AGG_MAX), T, O.p(col), O.p(nulls), 0, O.p(groups), n, O.p(want), O.p(wn)) == 0
            state = np.zeros(ngroups, np.uint64)
        snull = _words(np.ones(ngroups, bool))
        assert ops.group_agg(op, T, state, snull, None, groups[:h], col[:h], nulls[:h // 64], h) == 0
        assert ops.group_agg(op, T, state, snull, None, groups[h:], col[h:], nulls[h // 64:], n - h) == 0
        assert np.array_equal(bitmap_to_bools(snull, ngroups), wn.astype(bool)), (ngroups, op, T)
        live = wn == 0
        if op == capi.AGG_SUM:
            # float columns hold small integers: every partial sum is exact, so the atomics' order cannot show
            assert np.array_equal(state.view(np.uint64)[live], want.view(np.uint64)[live]), (ngroups, T)
        else:
            u = UINT_OF[dt.itemsize]
            got = state.view(np.uint8).reshape(ngroups, 8)[:, :dt.itemsize].copy().view(u).reshape(-1)
            wb = want.view(u)
            if dt.kind == "f":                              # a NaN is kept as a NaN; its payload may change in the float64 fold
                gn, wnan = np.isnan(got.view(dt)), np.isnan(want)
                assert np.array_equal(gn[live], wnan[live]), (ngroups, op, T)
                ok = live & ~wnan
                bad = np.flatnonzero(got[ok] != wb[ok])
                assert len(bad) == 0, (ngroups, op, T, got.view(dt)[ok][bad[:5]], want[ok][bad[:5]])
                if ngroups > 2:
                    assert gn[1] and _bits(got.view(dt)[2], dt) == _bits(-0.0, dt)
            else:
                assert np.array_equal(got[live], wb[live]), (ngroups, op, T)


@pytest.mark.parametrize("ngroups", [1, 1025])
def test_group_sum_overflow_depends_on_the_second_batch_order(gpu, ngroups):
    """batch 1 leaves group 1 at INT64_MAX - 10; batch 2 adds +20 then -30 (the running sum leaves int64) or -30 then +20 (it does
    not).  rc and the state follow the serial loop across the two calls"""
    R = capi.RC_OUT_OF_RANGE
    for second, rc_want in (([20, -30], R), ([-30, 20], 0)):
        g1 = np.ones(3, np.uint64) * ngroups
        c1 = np.asarray([I64MAX - 1000, 490, 500], np.int64)
        mask1 = np.zeros(3, bool)
        g2 = np.asarray([ngroups, 0, ngroups, ngroups], np.uint64)
        c2 = np.asarray([second[0], I64MAX, -2 ** 40, second[1]], np.int64)         # a GroupNotMatched row and a poisoned null
        mask2 = np.asarray([False, False, True, False])
        want, wn = np.zeros(ngroups, np.int64), np.ones(ngroups, np.uint8)
        rcs = []
        for g, c, m in ((g1, c1, mask1), (g2, c2, mask2)):
            rcs.append(O.go().og_sum_int64(capi.T_INT64, O.p(c), O.p(_words(m)), 0, O.p(g), len(c), O.p(want), O.p(wn), None, None))
        assert rcs == [0, rc_want]
        st, sn = np.zeros(ngroups, np.int64), _words(np.ones(ngroups, bool))
        assert ops.group_agg(capi.AGG_SUM, capi.T_INT64, st, sn, None, g1, c1, _words(mask1)) == 0
        assert st[ngroups - 1] == I64MAX - 10
        assert ops.group_agg(capi.AGG_SUM, capi.T_INT64, st, sn, None, g2, c2, _words(mask2)) == rc_want
        if rc_want == 0:
            assert st[ngroups - 1] == want[ngroups - 1] == I64MAX - 20


# ------------------------------------------------------------------------------------------------------------------ AGG_MERGE
@pytest.mark.parametrize("T", [capi.T_FLOAT32, capi.T_FLOAT64])
def test_agg_merge_of_ragged_partials_keeps_the_first_zero(gpu, T):
    """partial states of ragged row ranges, merged in order (the earlier partial wins a tie), equal the aggregate of the whole
    column bit for bit"""
    dt = _dt(T)
    rng = np.random.default_rng(T)
    n = 50_000
    cut_sets = [[0, 1, 2, 3, n], [0, 13_000, 13_001, 40_000, 40_064, n], [0, 64, 128, 129, 30_000, n]]
    for op in (capi.AGG_MIN, capi.AGG_MAX):
        s = -1.0 if op == capi.AGG_MAX else 1.0
        for case in ("zeros", "nan first", "nan inside", "first zero late"):
            col = rng.choice(np.asarray([0.0, -0.0, 2.0 * s, 4.0 * s]), n).astype(dt)
            mask = rng.random(n) < 0.1
            mask[13_000:13_001] = True
            if case == "nan first":
                col[np.flatnonzero(~mask)[0]] = np.nan
            elif case == "nan inside":                   # never the first live row of a partial: that partial's state would be NaN
                mask[3:6] = False
                col[[5, 20_000, 45_000]] = np.nan
            elif case == "first zero late":
                col[:40_000] = 4.0 * s
                col[45_000], col[40_100] = 0.0, -0.0
            col[mask] = -2.0 ** 40 * s
            want, wn = _minmax_want(int(op == capi.AGG_MAX), T, col, _words(mask), n)
            for cuts in cut_sets:
                states = np.stack([ops.agg_state(op, T, np.ascontiguousarray(col[a:b]), _words(mask[a:b]), b - a)
                                   for a, b in zip(cuts[:-1], cuts[1:])])
                rc, bits, cnt, isnull = ops.agg_merge(op, T, states)
                assert rc == 0 and not isnull and cnt == int((~mask).sum())
                got = np.asarray([bits], np.uint64).view(np.uint8)[:dt.itemsize].view(dt)[0]
                if np.isnan(want):
                    assert np.isnan(got), (op, case, cuts)
                else:
                    assert _bits(got, dt) == _bits(want, dt), (op, case, cuts, got, want)
                whole, _ = (ops.agg_max if op == capi.AGG_MAX else ops.agg_min)(T, col, _words(mask), n)
                assert _bits(whole, dt) == _bits(got, dt) or (np.isnan(whole) and np.isnan(got))
