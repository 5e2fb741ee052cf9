"""Go elementwise engine conventions behind XCall (csrc/goelem.cu) vs the oracle restatement of baseTemplate.go / arithmetic.go /
func_compare.go / operator_between.go / logicalOperator.go (oracle/oracle_go.c og_arith, og_compare, og_between, og_multi_logic).
Bit-exact: results, result nulls, return code and the first offending row."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from matrixone_b200 import capi
from matrixone_b200.vector import Vector, xcall

pytestmark = pytest.mark.gpu

TYPES = {capi.T_INT8: np.int8, capi.T_INT16: np.int16, capi.T_INT32: np.int32, capi.T_INT64: np.int64,
         capi.T_UINT8: np.uint8, capi.T_UINT16: np.uint16, capi.T_UINT32: np.uint32, capi.T_UINT64: np.uint64,
         capi.T_FLOAT32: np.float32, capi.T_FLOAT64: np.float64}
N = 5000


def _words(n):
    return (n + 63) // 64


def _bits(words, n):
    return np.unpackbits(words.view(np.uint8), bitorder="little")[:n].astype(bool)


def _rand_nulls(rng, n, p):
    b = rng.random(_words(n) * 64) < p
    b[n:] = False
    return np.packbits(b, bitorder="little").view(np.uint64).copy()


def _operands(rng, dt, n, op):
    """values that overflow in a few rows only (so both the OK and the error paths are exercised across seeds)"""
    if np.issubdtype(dt, np.floating):
        a = (rng.standard_normal(n) * 100).astype(dt); b = (rng.standard_normal(n) * 100).astype(dt)
        b[rng.random(n) < 0.02] = 0
        return a, b
    info = np.iinfo(dt)
    if op == 2:      # products: mostly small, a handful near the limits
        lim = max(2, int(np.sqrt(float(info.max))) // 2)
        lo = -lim if info.min < 0 else 0
        a = rng.integers(lo, lim, n).astype(dt); b = rng.integers(lo, lim, n).astype(dt)
    else:
        lo = info.min // 4; hi = info.max // 4
        a = rng.integers(lo, hi, n, dtype=np.int64 if dt != np.uint64 else np.uint64).astype(dt)
        b = rng.integers(lo, hi, n, dtype=np.int64 if dt != np.uint64 else np.uint64).astype(dt)
    b[rng.random(n) < 0.02] = 0
    return a, b


@pytest.mark.parametrize("T", sorted(TYPES))
@pytest.mark.parametrize("op", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("shape", ["vv", "vc", "cv", "cnull", "nullc"])
@pytest.mark.parametrize("case", ["clean", "offender", "div0_null"])
def test_go_arithmetic_matches_oracle(gpu, T, op, shape, case):
    dt = TYPES[T]
    rng = np.random.default_rng(T * 1000 + op * 100 + ["vv", "vc", "cv", "cnull", "nullc"].index(shape) * 10 + ["clean", "offender", "div0_null"].index(case))
    n = N
    a, b = _operands(rng, dt, n, op)
    if case != "div0_null" and op in (3, 4):
        if case == "clean":
            b[b == 0] = 1
    if case == "offender" and op in (0, 1, 2) and not np.issubdtype(dt, np.floating):
        info = np.iinfo(dt)
        rows = rng.choice(n, 3, replace=False)
        a[rows] = info.max if op != 1 else info.min
        b[rows] = info.max if op != 2 else 2
        if op == 1 and info.min == 0:
            a[rows] = 0; b[rows] = 1
    if case == "offender" and np.issubdtype(dt, np.floating) and op in (0, 1):
        rows = rng.choice(n, 2, replace=False)
        a[rows] = np.finfo(dt).max; b[rows] = np.finfo(dt).max if op == 0 else -np.finfo(dt).max
    c1, c2 = shape in ("cv", "nullc"), shape in ("vc", "cnull")   # cnull / nullc: a const NULL b / a nulls every row
    if c1: a = a[:1].copy()
    if c2:
        b = b[:1].copy()
        if case == "clean" and op in (3, 4) and b[0] == 0: b[0] = 3
    n1 = np.array([1], dtype=np.uint64) if shape == "nullc" else (None if c1 else _rand_nulls(rng, n, 0.05))
    n2 = np.array([1], dtype=np.uint64) if shape == "cnull" else (None if c2 else _rand_nulls(rng, n, 0.05))
    sel = _rand_nulls(rng, n, 0.1)                    # NOT selectList, pre-filled by the caller
    div0_null = 1 if case == "div0_null" else 0
    # oracle
    r0 = np.full(n, 77, dtype=dt); rn0 = sel.copy(); row0 = np.array([-1], dtype=np.int64)
    rc0 = O.go().og_arith(op, T, O.p(r0), O.p(a), O.p(b), n, int(c1), int(c2), O.p(n1) if n1 is not None else None,
                          O.p(n2) if n2 is not None else None, O.p(rn0), div0_null, O.p(row0))
    # GPU
    r1 = np.full(n, 77, dtype=dt); rn1 = sel.copy()
    params = np.zeros(2, dtype=np.int64); params.view(np.int32)[0] = div0_null; params[1] = -1
    rc1, msg = xcall(capi.XCALL_GO_ARITH(op, T), [Vector(data=r1, nulls=rn1, length=n), Vector(data=a, nulls=n1, length=n),
                                                    Vector(data=b, nulls=n2, length=n), Vector(data=params.view(np.uint8), length=n)], n, raise_on_error=False)
    if op == 3 and not np.issubdtype(dt, np.floating):
        # "/" is defined on floats only (arithmetic.go:481-514): the oracle and the library both refuse integer operands, and the
        # library leaves the result, its nulls and the offending-row slot untouched.  The library refuses the type before it looks at
        # the operands, so a const NULL operand does not change that; the oracle nulls every row first.
        assert rc1 == capi.RC_INVALID_ARGUMENT and "not defined" in msg, (rc1, msg)
        assert rc0 == (0 if shape in ("cnull", "nullc") else capi.RC_INVALID_ARGUMENT), rc0
        assert (r1 == 77).all() and (rn1 == sel).all() and params[1] == -1
        return
    assert rc1 == rc0, (rc1, rc0, msg)
    if rc0 == 0:
        assert params[1] == -1
        assert (rn1 == rn0).all()
        live = ~_bits(rn0, n)
        assert (r1[live].view(np.uint8) == r0[live].view(np.uint8)).all() if dt in (np.float32, np.float64) else (r1[live] == r0[live]).all()
        assert (r1[~live] == 77).all()                # null rows are left untouched
    else:
        assert params[1] == row0[0], (params[1], row0[0])
        f = int(row0[0])
        live = ~_bits(rn0, n); live[f:] = False      # rows before the first offender are what the Go loop leaves behind
        assert (r1[live] == r0[live]).all()
        assert ("out of range" in msg) or ("division by zero" in msg)
        if rc0 == capi.RC_OUT_OF_RANGE:
            assert str(a[0 if c1 else f]) in msg or np.issubdtype(dt, np.floating)


@pytest.mark.parametrize("T", sorted(TYPES) + [capi.T_BOOL, capi.T_DATE, capi.T_DATETIME])
@pytest.mark.parametrize("op", range(6))
def test_go_compare_matches_oracle(gpu, T, op):
    dt = TYPES.get(T, {capi.T_BOOL: np.uint8, capi.T_DATE: np.int32, capi.T_DATETIME: np.int64}.get(T))
    rng = np.random.default_rng(T * 16 + op)
    n = N
    if np.issubdtype(dt, np.floating):
        a = rng.integers(-5, 5, n).astype(dt); b = rng.integers(-5, 5, n).astype(dt)
    elif T == capi.T_BOOL:
        a = rng.integers(0, 2, n).astype(dt); b = rng.integers(0, 2, n).astype(dt)
    else:
        info = np.iinfo(dt); lo = max(info.min, -5); a = rng.integers(lo, 6, n).astype(dt); b = rng.integers(lo, 6, n).astype(dt)
    for shape in ("vv", "vc", "cv", "cnull"):
        c1, c2 = shape == "cv", shape in ("vc", "cnull")
        aa = a[:1].copy() if c1 else a; bb = b[:1].copy() if c2 else b
        n1 = None if c1 else _rand_nulls(rng, n, 0.05)
        n2 = np.array([1], dtype=np.uint64) if shape == "cnull" else (None if c2 else _rand_nulls(rng, n, 0.05))
        sel = _rand_nulls(rng, n, 0.1)
        r0 = np.full(n, 7, dtype=np.uint8); rn0 = sel.copy()
        rc0 = O.go().og_compare(op, T, O.p(r0), O.p(aa), O.p(bb), n, int(c1), int(c2), O.p(n1) if n1 is not None else None,
                                O.p(n2) if n2 is not None else None, O.p(rn0))
        r1 = np.full(n, 7, dtype=np.uint8); rn1 = sel.copy()
        rc1, msg = xcall(capi.XCALL_GO_COMPARE(op, T), [Vector(data=r1, nulls=rn1, length=n), Vector(data=aa, nulls=n1, length=n),
                                                         Vector(data=bb, nulls=n2, length=n)], n, raise_on_error=False)
        assert rc1 == rc0 == 0, (shape, rc1, rc0, msg)
        assert (rn1 == rn0).all(), shape
        assert (r1 == r0).all(), shape


@pytest.mark.parametrize("T", sorted(TYPES) + [capi.T_DATE])
def test_go_between_matches_oracle(gpu, T):
    dt = TYPES.get(T, np.int32)
    rng = np.random.default_rng(T)
    for n in (1, 31, 64, 4097):
        col = rng.integers(0, 100, n).astype(dt)
        lo = np.array([20], dtype=dt); hi = np.array([60], dtype=dt)
        nulls = _rand_nulls(rng, n, 0.1); pre = _rand_nulls(rng, n, 0.05)
        r0 = np.full(n, 9, dtype=np.uint8); rn0 = pre.copy()
        assert O.go().og_between(T, O.p(r0), O.p(col), O.p(lo), O.p(hi), n, O.p(nulls), O.p(rn0)) == 0
        r1 = np.full(n, 9, dtype=np.uint8); rn1 = pre.copy()
        xcall(capi.XCALL_GO_BETWEEN(T), [Vector(data=r1, nulls=rn1, length=n), Vector(data=col, nulls=nulls, length=n),
                                          Vector(data=lo, length=n), Vector(data=hi, length=n)], n)
        assert (r1 == r0).all() and (rn1 == rn0).all(), n


@pytest.mark.parametrize("is_or", [0, 1])
@pytest.mark.parametrize("kinds", [(0, 0), (0, 0, 0, 0), (0, 1, 0), (1, 0), (0, 2, 0), (2, 0, 1), (0, 0, 2)])
def test_go_multi_logic_matches_oracle(gpu, is_or, kinds):
    rng = np.random.default_rng(len(kinds) * 7 + is_or)
    for n in (1, 33, 1000, 4099):
        cols, nulls = [], []
        for kd in kinds:
            if kd == 0:
                cols.append(rng.integers(0, 2, n).astype(np.uint8)); nulls.append(_rand_nulls(rng, n, 0.2))
            elif kd == 1:
                cols.append(rng.integers(0, 2, 1).astype(np.uint8)); nulls.append(None)
            else:
                cols.append(np.zeros(1, dtype=np.uint8)); nulls.append(np.array([1], dtype=np.uint64))
        k = len(kinds)
        colp = (C.c_void_p * k)(*[c.ctypes.data for c in cols])
        nullp = (C.c_void_p * k)(*[(x.ctypes.data if x is not None else None) for x in nulls])
        kindp = (C.c_int32 * k)(*kinds)
        r0 = np.zeros(n, dtype=np.uint8); rn0 = np.zeros(_words(n), dtype=np.uint64)
        assert O.go().og_multi_logic(is_or, O.p(r0), O.p(rn0), k, colp, nullp, kindp, n) == 0
        r1 = np.full(n, 5, dtype=np.uint8); rn1 = np.full(_words(n), 0xdeadbeef, dtype=np.uint64)
        cnt = np.array([k], dtype=np.int32)
        vecs = [Vector(data=r1, nulls=rn1, length=n), Vector(data=cnt.view(np.uint8), length=n)]
        vecs += [Vector(data=c, nulls=x, length=n) for c, x in zip(cols, nulls)]
        xcall(capi.XCALL_GO_MULTI_OR if is_or else capi.XCALL_GO_MULTI_AND, vecs, n)
        assert (rn1 == rn0).all(), (kinds, n)
        live = ~_bits(rn0, n)
        assert (r1[live] == r0[live]).all(), (kinds, n)     # the value under a NULL is not observable
