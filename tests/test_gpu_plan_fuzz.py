"""The generic fused operator (csrc/plan.cu, MO_XCALL_PLAN) over seeded random descriptors, against its exact restatement
(plan_reference.py, itself checked against the oracle in test_plan_reference.py).  Every plan runs in both dispatch modes (plan_specialise 1
and 0) and in both forms (host columns and result; resident columns, nulls and result = the asynchronous form).  Families aim at the
kernel's structure: the three group tiers (private state, CTA table, global table) and the unsorted emit, one row per group, the largest
shared-memory footprint, near misses of the recognised Q6 / Q1 shapes; then targeted edges."""
import numpy as np
import pytest

import plan_reference as R
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer, bitmap_from_bools

pytestmark = pytest.mark.gpu

INT_TYPES = [capi.T_BOOL, capi.T_INT8, capi.T_INT16, capi.T_INT32, capi.T_INT64, capi.T_UINT8, capi.T_UINT16, capi.T_UINT32, capi.T_UINT64,
             capi.T_DATE, capi.T_TIME, capi.T_DATETIME, capi.T_TIMESTAMP]
ALL_TYPES = INT_TYPES + [capi.T_FLOAT32, capi.T_FLOAT64]
KINDS = [capi.AGG_SUM, capi.AGG_COUNT, capi.AGG_MIN, capi.AGG_MAX, capi.AGG_AVG]
OPS = ["==", "!=", ">", ">=", "<", "<=", "between"]
Q1COLS = ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")


# ---------------------------------------------------------------------------------------------------------------- running and checking
def run_all(gpu, p, cols, nulls, n, max_groups):
    """[(plan_specialise, form, groups)] for both dispatch modes and both forms"""
    out = []
    for spec in (1, 0):
        assert gpu.MoB200_SetTuning(b"plan_specialise", spec) == 0
        try:
            out.append((spec, "host", p.run(cols, n, nulls=nulls, max_groups=max_groups)))
            dev = [DeviceBuffer.from_numpy(np.ascontiguousarray(c)) for c in cols]
            dnul = None if nulls is None else [None if w is None else DeviceBuffer.from_numpy(w) for w in nulls]
            res = DeviceBuffer(p.result_bytes(max_groups))
            assert p.run(dev, n, nulls=dnul, max_groups=max_groups, out_ptr=res.ptr) is None
            out.append((spec, "device", p.parse(res.to_numpy(np.uint8).tobytes())))
            for b in dev + [w for w in (dnul or []) if w is not None] + [res]:
                b.free()
        finally:
            gpu.MoB200_SetTuning(b"plan_specialise", 1)
    return out


def check(gpu, p, cols, nulls, n, max_groups=None, first_row_unknown_when_specialised=False):
    """the kernel in every mode and form against the reference; the result buffer holds exactly the groups there are unless given"""
    want = R.run(p.P, cols, nulls, n)
    mg = max_groups if max_groups is not None else max(len(want), 1)
    for spec, form, got in run_all(gpu, p, cols, nulls, n, mg):
        try:
            R.assert_matches(got, want, p.P, first_row_unknown=first_row_unknown_when_specialised and spec == 1)
        except AssertionError as e:
            raise AssertionError("plan_specialise=%d %s form: %s" % (spec, form, e)) from None
    return want


# ---------------------------------------------------------------------------------------------------------------- random descriptors
def gen_values(rng, T, n, specials=True):
    dt = R.DTYPE[T]
    if T == capi.T_BOOL:
        return rng.integers(0, 2, n).astype(np.uint8)
    if T in R.FLOAT_TYPES:
        v = rng.standard_normal(n) * 10.0 ** int(rng.integers(-1, 4))
        if rng.random() < 0.5:
            v = np.round(v, 1)                                   # duplicates and exact ties
        if specials and rng.random() < 0.5:
            pick = rng.random(n)
            v[pick < 0.01] = np.nan
            v[(pick >= 0.01) & (pick < 0.015)] = np.inf
            v[(pick >= 0.015) & (pick < 0.02)] = -np.inf
            v[(pick >= 0.02) & (pick < 0.04)] = -0.0
            v[(pick >= 0.04) & (pick < 0.06)] = 0.0
        return v.astype(dt)
    info = np.iinfo(dt)
    r = rng.random()
    if r < 0.5 or info.bits < 64:
        lo, hi = max(int(info.min), -1000), min(int(info.max), 1000)
        if rng.random() < 0.3:
            lo, hi = int(info.min), int(info.max)
        return rng.integers(lo, hi, n, dtype=dt, endpoint=True)
    if r < 0.85:                                                 # around a power of two where float64 stops being exact
        bases = [2 ** 53, 2 ** 60, 2 ** 62] if info.min < 0 else [2 ** 53, 2 ** 63, 2 ** 64 - 8]
        base = bases[int(rng.integers(0, 3))]
        sign = -1 if info.min < 0 and rng.random() < 0.3 else 1
        return np.full(n, dt(sign * base), dtype=dt) + rng.integers(-4, 5, n).astype(dt)
    return rng.integers(int(info.min), int(info.max), n, dtype=dt, endpoint=True)


def gen_const(rng, T, data, live):
    """a predicate constant: a data value, a data value + 0.5, or an extreme"""
    x = data[live] if live.any() else data
    r = rng.random()
    if r < 0.55 and x.size:
        return float(x[rng.integers(0, x.size)])
    if r < 0.7 and x.size:
        return float(x[rng.integers(0, x.size)]) + 0.5
    ext = [0.0, -0.5, 2.0 ** 53, -2.0 ** 53, 2.0 ** 60, 2.0 ** 63, -2.0 ** 63, 2.0 ** 64, np.inf, -np.inf]
    if T not in R.FLOAT_TYPES:
        info = np.iinfo(R.DTYPE[T])
        ext += [float(info.min), float(info.max)]
    return float(rng.choice(ext))


def gen_nulls(rng, n, allow=True):
    if not allow or rng.random() < 0.4:
        return None
    d = float(rng.choice([0.0, 0.01, 0.2, 0.5, 0.9, 1.0]))
    return bitmap_from_bools(rng.random(n) < d)


def key_vocab(rng, T, card):
    """card distinct values of type T (fewer when the type has fewer)"""
    if T == capi.T_BOOL:
        return np.arange(min(card, 2), dtype=np.uint8)
    if T in R.FLOAT_TYPES:
        v = np.unique(np.round(rng.standard_normal(card * 2 + 4) * 100, 2))
        v = np.concatenate([[-0.0, 0.0], v])[:card]
        return v.astype(R.DTYPE[T])
    info = np.iinfo(R.DTYPE[T])
    span = int(info.max) - int(info.min) + 1
    if span <= 4 * card:
        v = np.arange(int(info.min), int(info.max) + 1)
        return rng.permutation(v)[:card].astype(R.DTYPE[T])
    v = set()
    while len(v) < card:
        v.update(int(x) for x in rng.integers(int(info.min), int(info.max), card, dtype=R.DTYPE[T], endpoint=True))
    return np.array(sorted(v)[:card], dtype=R.DTYPE[T])


def random_plan(rng, n, ncols=None, ninstr=None, naggs=None, card=None, skew=False, row_base=None, npreds=None):
    """a random descriptor and its data.  card: distinct key tuples wanted (None: random); skew: each tile's first rows carry rare keys"""
    ncols = ncols or int(rng.integers(1, 13))
    types = [int(rng.choice(ALL_TYPES)) for _ in range(ncols)]
    has_null_keys = bool(rng.random() < 0.5)
    rb = int(rng.integers(0, 1 << 40)) if row_base is None and rng.random() < 0.3 else (row_base or 0)
    p = ops.FusedPlan(types, has_null_keys=has_null_keys, row_base=rb)
    cols = [gen_values(rng, T, n) for T in types]
    nulls = [gen_nulls(rng, n) for _ in types]
    # keys: 1-4 columns within the 8 key bytes (a marker byte each with has_null_keys), fed from a vocabulary of the wanted cardinality
    nkeys = int(rng.integers(0 if card is None else 1, 5))
    budget, keys = 8, []
    for c in rng.permutation(ncols):
        sz = R.DTYPE[types[c]]().itemsize + (1 if has_null_keys else 0)
        if len(keys) < nkeys and sz <= budget and (types[c] != capi.T_FLOAT64 or rng.random() < 0.3):
            keys.append(int(c)); budget -= sz
    if keys:
        tot = card or int(rng.choice([1, 3, 20, 300, 5000]))
        per = max(1, int(round(tot ** (1.0 / len(keys)))))
        for c in keys:
            vocab = key_vocab(rng, types[c], per)
            idx = rng.integers(0, vocab.shape[0], n)
            if skew and vocab.shape[0] > 8:
                common = rng.integers(0, 4, n)                   # most rows: 4 common keys; every tile's first rows: rare ones
                first = (np.arange(n) % 512) < 6
                idx = np.where(first, rng.integers(4, vocab.shape[0], n), common)
            cols[c] = vocab[idx]
            if rng.random() < 0.5:
                nulls[c] = None if rng.random() < 0.5 else bitmap_from_bools(rng.random(n) < 0.05)
        p.group_by(*keys)
    # predicates with moderate selectivity: quantiles for the inequalities, data values and extremes now and then; a candidate that keeps
    # less than a third of the rows still standing is usually drawn again
    kept = np.ones(n, bool)
    for _ in range(int(rng.integers(0, 9)) if npreds is None else npreds):
        for attempt in range(4):
            c = int(rng.integers(0, ncols)); T = types[c]
            live = ~R.null_mask(nulls[c], n)
            x = cols[c].astype(np.float64)
            fin = x[live & np.isfinite(x)]
            op = OPS[int(rng.integers(0, 7))]
            if op == "==" and (np.unique(fin).size if fin.size else 0) > 64:
                op = "!="
            if fin.size and rng.random() < 0.7 and op not in ("==", "!="):
                if op == "between":
                    lo, hi = np.quantile(fin, [rng.uniform(0, 0.3), rng.uniform(0.7, 1.0)], method="nearest")
                else:
                    q = rng.uniform(0.02, 0.5) if op in (">", ">=") else rng.uniform(0.5, 0.98)
                    lo, hi = np.quantile(fin, q, method="nearest"), 0.0
            else:
                lo, hi = gen_const(rng, T, cols[c], live), gen_const(rng, T, cols[c], live)
                if op == "between" and lo > hi:
                    lo, hi = hi, lo
            m = kept & live & R.predicate(T, cols[c], R.OPS_BY_NAME[op], float(lo), float(hi))
            if m.sum() * 3 >= kept.sum() or rng.random() < 0.04:
                p.where(c, op, float(lo), float(hi))
                kept = m
                break
    # an SSA program: random DAG over columns and earlier nodes, favouring recent nodes; x * x, constants, nodes nobody reads
    k = int(rng.integers(0, 17)) if ninstr is None else ninstr
    for i in range(k):
        nslots = ncols + i
        pick = lambda: int(rng.integers(max(0, nslots - 3), nslots)) if rng.random() < 0.5 else int(rng.integers(0, nslots))
        r = rng.random()
        if r < 0.1:
            p._emit(capi.PLAN_OP_COL, int(rng.integers(0, ncols)))
        elif r < 0.2:
            p.const(float(rng.choice([0.0, -0.0, 1.0, 2.5, -3.0, 1e-3, 7.0])))
        else:
            a = pick(); b = a if rng.random() < 0.15 else pick()
            [p.add, p.sub, p.mul, p.div][int(rng.integers(0, 4))](a, b)
    for _ in range(int(rng.integers(1, 13)) if naggs is None else naggs):
        kind = KINDS[int(rng.integers(0, 5))]
        v = -1 if kind == capi.AGG_COUNT and rng.random() < 0.3 else int(rng.integers(0, ncols + k))
        p.agg(kind, v)
    return p, cols, nulls


@pytest.mark.parametrize("seed", range(24))
def test_fuzz_random_descriptors(gpu, seed):
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.choice([1, 63, 64, 513, 4097, 30_011, 200_003]))
    p, cols, nulls = random_plan(rng, n)
    check(gpu, p, cols, nulls, n)


@pytest.mark.parametrize("card,skew,n", [(1, False, 50_000), (3, False, 100_003), (4, True, 100_003), (20, False, 100_003), (32, True, 50_000),
                                          (300, False, 200_003), (5000, True, 100_003), (8192, False, 60_000), (20_000, False, 300_007)],
                         ids=lambda v: str(v))
def test_fuzz_group_tiers(gpu, card, skew, n):
    """1-4 keys: private state; 5-32: the CTA table; more: the global table; above 8192 groups: unsorted emit + host sort.  Skewed data puts
    rare keys first in every tile so the private dictionary holds keys the bulk of the rows never use.  row_base is set throughout."""
    rng = np.random.default_rng(card * 7 + skew)
    p, cols, nulls = random_plan(rng, n, ncols=int(rng.integers(2, 8)), card=card, skew=skew, row_base=123_456_789, npreds=int(rng.integers(0, 3)))
    want = check(gpu, p, cols, nulls, n)
    if card > 32 and not skew:
        assert len(want) > 32


@pytest.mark.parametrize("T,n", [(capi.T_INT32, 5000), (capi.T_INT64, 20_000), (capi.T_UINT32, 9000)])
def test_fuzz_one_row_per_group(gpu, T, n):
    """key = row id: MIN, MAX and SUM of every group are the row's expression value itself -- per-node rounding checked bit for bit"""
    rng = np.random.default_rng(n)
    for rep in range(3):
        types = [T, capi.T_FLOAT64, capi.T_FLOAT32, capi.T_INT16]
        cols = [np.arange(n).astype(R.DTYPE[T]), gen_values(rng, capi.T_FLOAT64, n, specials=False), gen_values(rng, capi.T_FLOAT32, n, specials=False),
                rng.integers(-300, 300, n).astype(np.int16)]
        p = ops.FusedPlan(types, row_base=rep * 1000)
        e = p.div(p.sub(p.mul(p.col(1), p.col(2)), p.col(3)), p.add(p.col(2), p.const(0.3)))
        f = p.add(p.mul(e, e), p.sub(p.col(3), p.col(1)))
        p.group_by(0)
        for v in (e, f):
            for kind in (capi.AGG_SUM, capi.AGG_MIN, capi.AGG_MAX):
                p.agg(kind, v)
        want = check(gpu, p, cols, None, n)
        assert len(want) == n
        assert gpu.MoB200_SetTuning(b"plan_specialise", 0) == 0
        try:
            got = p.run(cols, n, max_groups=n)
        finally:
            gpu.MoB200_SetTuning(b"plan_specialise", 1)
        gv = np.array([[a[0] for a in g["aggs"]] for g in got]); wv = np.array([[a[0] for a in g["aggs"]] for g in want])
        has = np.array([[a[1] for a in g["aggs"]] for g in want]) > 0
        assert has.sum() > n and ((gv == wv) | (np.isnan(gv) & np.isnan(wv)) | ~has).all()


@pytest.mark.parametrize("seed", range(4))
def test_fuzz_largest_footprint(gpu, seed):
    """12 columns, 16 nodes, 12 aggregates: the most shared memory; dead slots reused, x * x, unread nodes, aggregates over raw columns that
    are also instruction operands"""
    rng = np.random.default_rng(50 + seed)
    n = 70_001
    p, cols, nulls = random_plan(rng, n, ncols=12, ninstr=0, naggs=0, card=int(rng.choice([3, 40, 2000])), npreds=int(rng.integers(0, 4)))
    one = p.const(1.0)
    sq = p.mul(0, 0)                                             # x * x on one operand
    p.mul(1, 2)                                                  # a node nobody reads
    d = p.div(p.sub(3, 4), p.add(5, one))
    for i in range(12):
        d = p._emit([capi.PLAN_OP_ADD, capi.PLAN_OP_SUB, capi.PLAN_OP_MUL, capi.PLAN_OP_DIV][i % 4], d, [sq, 6 + i % 6, one, d][i % 4]) \
            if p.P.ninstr < 16 else d
    for a in range(12):
        p.agg(KINDS[a % 5], [0, 3, 4, sq, d, 7, -1 if a % 5 == 1 else 11][a % 7])
    assert p.P.ncols == 12 and p.P.ninstr == 16 and p.P.naggs == 12
    check(gpu, p, cols, nulls, n)


def near_misses():
    """descriptors one field away from the recognised Q6 / Q1 shapes"""
    out = []

    def q6(f, exact=False):
        p = ops.q6_plan(); f(p.P); return ("q6", p, exact)

    def q1(f):
        p = ops.q1_plan(datagen.Q1_CUTOFF, row_base=9); f(p.P); return ("q1", p, False)
    out.append(q6(lambda P: None, exact=True))
    out.append(q6(lambda P: setattr(P.pred[0], "op", 2)))                 # > instead of >=
    out.append(q6(lambda P: setattr(P.pred[1], "lo", P.pred[1].lo + 0.5)))   # a non-integral date constant
    out.append(q6(lambda P: (setattr(P.instr[0], "a", 1), setattr(P.instr[0], "b", 3)), exact=True))   # swapped operands: still Q6
    out.append(q6(lambda P: setattr(P.instr[0], "op", capi.PLAN_OP_ADD)))
    out.append(q6(lambda P: setattr(P.agg[0], "kind", capi.AGG_AVG)))
    out.append(q6(lambda P: P.col_type.__setitem__(0, capi.T_INT32), exact=True))   # INT32 instead of DATE: still Q6
    out.append(q6(lambda P: setattr(P.pred[2], "col", 2)))               # BETWEEN on another column
    out.append(q1(lambda P: None))
    out.append(q1(lambda P: setattr(P.pred[0], "op", 4)))                 # < instead of <=
    out.append(q1(lambda P: setattr(P.pred[0], "lo", P.pred[0].lo - 0.25)))
    out.append(q1(lambda P: (setattr(P.agg[0], "value", 2), setattr(P.agg[1], "value", 1))))   # aggregate order
    out.append(q1(lambda P: setattr(P, "has_null_keys", 1)))
    out.append(q1(lambda P: setattr(P.instr[1], "a", 3)))                 # 1 - disc -> disc - disc
    out.append(q1(lambda P: setattr(P.agg[7], "value", 1)))            # COUNT(quantity) instead of COUNT(*)
    return out


@pytest.mark.parametrize("i", range(len(near_misses())))
@pytest.mark.parametrize("nullable", [False, True])
def test_fuzz_q6_q1_near_misses(gpu, i, nullable):
    """identical results whether or not the specialised kernel answers; a nullable column takes the shape off the specialised path"""
    shape, p, exact = near_misses()[i]
    n = 100_003
    li = datagen.lineitem(10, 0, n)
    names = ("shipdate", "discount", "quantity", "extendedprice") if shape == "q6" else Q1COLS
    cols = [li[k] for k in names]
    nulls = None
    if nullable:
        rng = np.random.default_rng(i)
        nulls = [None] * len(cols); nulls[1] = bitmap_from_bools(rng.random(n) < 0.05)
    # the specialised Q6 kernel does not track the first qualifying row (first_row = -1)
    check(gpu, p, cols, nulls, n, max_groups=8 if shape == "q1" else None, first_row_unknown_when_specialised=exact and not nullable)


# ---------------------------------------------------------------------------------------------------------------- targeted edges
def test_null_group_keys_without_null_mode_join_no_group(gpu):
    """has_null_keys = 0: a row whose key is NULL is in no group, even when the bytes under the NULL equal another row's key"""
    n = 10_000
    rng = np.random.default_rng(3)
    key = rng.integers(0, 50, n).astype(np.int32)
    x = rng.standard_normal(n)
    kn = rng.random(n) < 0.1
    p = ops.FusedPlan([capi.T_INT32, capi.T_FLOAT64]).group_by(0).agg(capi.AGG_COUNT, -1).agg(capi.AGG_SUM, 1)
    want = check(gpu, p, [key, x], [bitmap_from_bools(kn), None], n)
    assert sum(g["rows"] for g in want) == int((~kn).sum())
    for tier_card in (3, 30, 3000):                              # the private, CTA-table and global paths
        k2 = rng.integers(0, tier_card, n).astype(np.int32)
        p2 = ops.FusedPlan([capi.T_INT32, capi.T_INT8]).group_by(0, 1).agg(capi.AGG_COUNT, -1)
        check(gpu, p2, [k2, np.zeros(n, np.int8)], [bitmap_from_bools(rng.random(n) < 0.2), bitmap_from_bools(rng.random(n) < 0.1)], n)


def test_integer_predicates_beyond_2_53(gpu):
    """constants of magnitude >= 2^53 compare exactly in the column's integer domain, also when the column feeds an expression"""
    def count(T, vals, op, c, feeds_expr=False, hi=0.0):
        p = ops.FusedPlan([T]).where(0, op, c, hi)
        p.agg(capi.AGG_COUNT, -1)
        if feeds_expr:
            p.agg(capi.AGG_COUNT, p.add(p.col(0), p.const(1.0)))
        arr = np.array(vals, dtype=R.DTYPE[T])
        want = check(gpu, p, [arr], None, arr.shape[0])
        return want[0]["rows"] if want else 0
    for fe in (False, True):
        assert count(capi.T_INT64, [2 ** 60 - 1, 2 ** 60, 2 ** 60 + 1], ">=", 2.0 ** 60, fe) == 2
        assert count(capi.T_INT64, [2 ** 53, 2 ** 53 + 1], "==", 2.0 ** 53, fe) == 1
        assert count(capi.T_INT64, [2 ** 53, 2 ** 53 + 1], "!=", 2.0 ** 53, fe) == 1
        assert count(capi.T_UINT64, [2 ** 63 + 1, 2 ** 63, 5], ">", 2.0 ** 63, fe) == 1
        assert count(capi.T_UINT64, [2 ** 64 - 1, 2 ** 63, 0], ">=", 2.0 ** 64, fe) == 0
        assert count(capi.T_UINT64, [2 ** 64 - 1, 2 ** 63, 0], "<", 2.0 ** 64, fe) == 3
        assert count(capi.T_INT64, [-2 ** 63, -2 ** 63 + 1, 0], "<=", -2.0 ** 63, fe) == 1
        assert count(capi.T_INT64, [-2 ** 63, 2 ** 63 - 1, 0], ">", -2.0 ** 64, fe) == 3
        assert count(capi.T_INT64, [2 ** 62, 2 ** 62 + 1, 2 ** 62 + 3], "between", 2.0 ** 62 + 0.0, fe, 2.0 ** 62 + 1024) == 3
        assert count(capi.T_TIMESTAMP, [2 ** 60 - 1, 2 ** 60, 7], "<", 2.0 ** 60, fe) == 2
        assert count(capi.T_INT32, [-5, 3, 2 ** 31 - 1], "between", -2.0 ** 70, fe, np.inf) == 3


def test_nan_constant_and_non_integral_constants(gpu):
    """a NaN constant: only != holds (IEEE, like the reference's float compare); an integer column against x.5 constants"""
    n = 1000
    x = np.arange(n, dtype=np.int16) - 500
    f = np.linspace(-3, 3, n)
    for T, col in ((capi.T_INT16, x), (capi.T_FLOAT64, f)):
        for op in OPS:
            p = ops.FusedPlan([T]).where(0, op, np.nan, np.nan if op == "between" else 0.0).agg(capi.AGG_COUNT, -1)
            want = check(gpu, p, [col], None, n)
            assert (want[0]["rows"] if want else 0) == (n if op == "!=" else 0)
    for op in OPS:
        p = ops.FusedPlan([capi.T_INT16]).where(0, op, -2.5, 3.5).agg(capi.AGG_COUNT, -1).agg(capi.AGG_MIN, 0)
        check(gpu, p, [x], None, n)


def test_sentinel_keys(gpu):
    """the all-ones packed key takes the table's extra slot (mask + 1): an int64 key of -1, two int32 keys of -1 -- in every tier"""
    rng = np.random.default_rng(8)
    n = 40_000
    for card in (2, 20, 2000):
        k = rng.integers(-1, card - 1, n).astype(np.int64)
        v = rng.standard_normal(n)
        p = ops.FusedPlan([capi.T_INT64, capi.T_FLOAT64]).group_by(0).agg(capi.AGG_SUM, 1).agg(capi.AGG_COUNT, -1).agg(capi.AGG_MAX, 1)
        want = check(gpu, p, [k, v], None, n)
        assert any(g["key"] == 0xffffffffffffffff for g in want)
        a, b = rng.integers(-1, 2, n).astype(np.int32), (rng.integers(-1, card // 2 + 1, n)).astype(np.int32)
        p = ops.FusedPlan([capi.T_INT32, capi.T_INT32, capi.T_FLOAT64]).group_by(0, 1).agg(capi.AGG_MIN, 2).agg(capi.AGG_COUNT, -1)
        want = check(gpu, p, [a, b, v], None, n)
        assert any(g["key"] == 0xffffffffffffffff for g in want)


def test_key_encodings(gpu):
    """negative INT8 keys (sign extension, masked to a byte), UINT32 keys above 2^31, FLOAT32 keys where -0.0 and +0.0 are distinct keys;
    both null modes, and keys that also feed an expression (the slot is float64, the key its integer / float32 bits)"""
    rng = np.random.default_rng(9)
    n = 20_000
    i8 = rng.integers(-128, 128, n).astype(np.int8)
    u32 = (np.uint32(2 ** 31) + rng.integers(0, 40, n).astype(np.uint32) * np.uint32(2 ** 25)).astype(np.uint32)
    f32 = rng.choice(np.array([-0.0, 0.0, 1.5, -2.25, 3e-40], np.float32), n)
    nw = bitmap_from_bools(rng.random(n) < 0.05)
    for hn in (False, True):
        p = ops.FusedPlan([capi.T_INT8, capi.T_UINT32, capi.T_FLOAT32], has_null_keys=hn).group_by(0, 1)
        p.agg(capi.AGG_SUM, p.add(p.col(0), p.col(1))).agg(capi.AGG_COUNT, -1)
        check(gpu, p, [i8, u32, f32], [None, nw, None], n, max_groups=n)
        p = ops.FusedPlan([capi.T_FLOAT32, capi.T_INT8], has_null_keys=hn).group_by(0, 1)
        p.agg(capi.AGG_MIN, p.mul(p.col(0), p.const(2.0))).agg(capi.AGG_MAX, 1)
        want = check(gpu, p, [f32, i8], [nw, None], n, max_groups=n)
        zeros = {g["key"] & 0xffffffff if not hn else (g["key"] >> 8) & 0xffffffff for g in want}
        assert 0 in zeros and 0x80000000 in zeros


@pytest.mark.parametrize("n", [1, 511, 512, 513, 8193, 65_599])
def test_row_counts_and_null_tails(gpu, n):
    """tile edges and a nulls bitmap whose last word is partly used"""
    rng = np.random.default_rng(n)
    k = rng.integers(0, 7, n).astype(np.int16)
    x = rng.standard_normal(n); y = rng.integers(-9, 9, n).astype(np.int32)
    xn = rng.random(n) < 0.3
    xn[-1] = True
    p = ops.FusedPlan([capi.T_INT16, capi.T_FLOAT64, capi.T_INT32], has_null_keys=True, row_base=77).where(2, "!=", 0).group_by(0)
    e = p.div(p.col(1), p.col(2))
    for kind in KINDS:
        p.agg(kind, e)
    p.agg(capi.AGG_COUNT, -1)
    check(gpu, p, [k, x, y], [bitmap_from_bools(rng.random(n) < 0.1), bitmap_from_bools(xn), None], n)


def test_result_buffer_exact_and_one_short(gpu):
    """exactly ngroups fits; ngroups - 1 fails loudly in the synchronous form and sets header.overflow in the asynchronous form"""
    n = 30_000
    rng = np.random.default_rng(5)
    for card in (3, 25, 700):
        key = rng.integers(0, card, n).astype(np.int32)
        p = ops.FusedPlan([capi.T_INT32]).group_by(0).agg(capi.AGG_COUNT, -1)
        want = check(gpu, p, [key], None, n, max_groups=card)
        assert len(want) == card
        for spec in (1, 0):
            assert gpu.MoB200_SetTuning(b"plan_specialise", spec) == 0
            try:
                with pytest.raises(capi.MoError) as e:
                    p.run([key], n, max_groups=card - 1)
                assert e.value.rc == capi.RC_INVALID_ARGUMENT
                dev = DeviceBuffer.from_numpy(key)
                res = DeviceBuffer(p.result_bytes(card - 1))
                p.run([dev], n, max_groups=card - 1, out_ptr=res.ptr)
                h = capi.PlanHeader.from_buffer_copy(res.to_numpy(np.uint8).tobytes())
                assert h.overflow == 1
                dev.free(); res.free()
            finally:
                gpu.MoB200_SetTuning(b"plan_specialise", 1)


def test_count_paths(gpu):
    """per-aggregate counts are kept only when an aggregate input can be NULL: no nullable input at all, versus a division that can be"""
    n = 50_000
    rng = np.random.default_rng(6)
    key = rng.integers(0, 3, n).astype(np.uint8)
    x = rng.integers(-3, 4, n).astype(np.int64); y = rng.standard_normal(n)
    for divides in (False, True):
        p = ops.FusedPlan([capi.T_UINT8, capi.T_INT64, capi.T_FLOAT64]).group_by(0)
        e = p.div(p.col(2), p.col(1)) if divides else p.mul(p.col(2), p.col(1))
        for kind in KINDS:
            p.agg(kind, e)
        p.agg(capi.AGG_COUNT, -1).agg(capi.AGG_MIN, 1)
        want = check(gpu, p, [key, x, y], None, n)
        assert any(g["aggs"][1][1] < g["rows"] for g in want) == divides


def test_min_max_nan_and_integer_columns(gpu):
    """an all-NaN group: MIN / MAX are NaN with a count; NaN is skipped elsewhere; integer columns below 2^53 exactly"""
    n = 3000
    key = (np.arange(n) % 3).astype(np.int32)
    v = np.where(key == 0, np.nan, np.linspace(-1, 1, n))
    v[5] = np.nan
    big = (np.arange(n, dtype=np.int64) * 1_000_003 + 2 ** 52)
    p = ops.FusedPlan([capi.T_INT32, capi.T_FLOAT64, capi.T_INT64]).group_by(0)
    p.agg(capi.AGG_MIN, 1).agg(capi.AGG_MAX, 1).agg(capi.AGG_MIN, 2).agg(capi.AGG_MAX, 2).agg(capi.AGG_SUM, 1)
    want = check(gpu, p, [key, v, big], None, n)
    g0 = want[0]["aggs"]
    assert np.isnan(g0[0][0]) and g0[0][1] == n // 3 and np.isnan(g0[1][0]) and np.isnan(g0[4][0])
    assert want[1]["aggs"][2][0] == float(big[1]) and want[1]["aggs"][3][0] == float(big[-2])


def test_malformed_descriptors_are_refused(gpu):
    def refused(p, cols):
        with pytest.raises(capi.MoError) as e:
            p.run(cols, len(cols[0]))
        assert e.value.rc == capi.RC_INVALID_ARGUMENT
    x = np.zeros(8, np.float64)
    p = ops.FusedPlan([capi.T_FLOAT64]); p._emit(capi.PLAN_OP_ADD, 0, 2); p._emit(capi.PLAN_OP_CONST, imm=1.0); p.agg(capi.AGG_SUM, 1)
    refused(p, [x])                                              # forward SSA reference
    p = ops.FusedPlan([capi.T_INT64, capi.T_INT8]).group_by(0, 1).agg(capi.AGG_COUNT, -1)
    refused(p, [np.zeros(8, np.int64), np.zeros(8, np.int8)])   # 9 key bytes
    p = ops.FusedPlan([capi.T_INT64], has_null_keys=True).group_by(0).agg(capi.AGG_COUNT, -1)
    refused(p, [np.zeros(8, np.int64)])                          # 8 value bytes + a marker
    p = ops.FusedPlan([capi.T_FLOAT64]).agg(capi.AGG_SUM, 1)
    refused(p, [x])                                              # aggregate slot out of range
    for kind in (capi.AGG_SUM, capi.AGG_MIN, capi.AGG_MAX, capi.AGG_AVG):
        refused(ops.FusedPlan([capi.T_FLOAT64]).agg(kind, -1), [x])   # COUNT(*) tagged with another kind
