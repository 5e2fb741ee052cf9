"""The operand contract every Go expression call shares (include/mo_b200.h, csrc/goengine.cuh), table-driven over GO_ARITH, GO_COMPARE
(fixed-width, float32 with a scale, decimal and varlena), GO_BETWEEN, MULTI_AND / OR, GO_LIKE, DEC_ARITH and DEC_AVG:

- a const operand is a one-element vector, except when len == 1, where a one-element operand is a column;
- a const NULL operand nulls every row;
- the host form and the all-device form, parameter block included, leave the same bytes in every slot and return the same code;
- each call launches a fixed number of kernels, the all-NULL case included;
- the bits of the last result-bitmap word past len are pinned per call (a caller's ones kept or cleared);
- a short operand, a short result and a missing result bitmap are refused alike on both sides;
- the first failing row decides the code, err_row and the message, in both forms;
- decimal GO_COMPARE and DEC_AVG on device operands only enqueue work."""
import ctypes as C

import numpy as np
import pytest

from matrixone_b200 import capi
from matrixone_b200.vector import DeviceBuffer, varlena_bytes_column

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

N = 1000                      # not a multiple of 64: the last bitmap word has bits past len
SLEEP_CYCLES = 100_000_000    # about 50 ms at H100 clocks
SHAPES = ["vv", "vc", "cv", "nc", "cn", "len1"]   # n: const NULL, c: const, v: vector; len1: one row, one-element operands as columns


class Arg:
    def __init__(self, data=None, nulls=None, area=None):
        area = None if area is not None and not len(area) else area
        self.slots = {k: None if v is None else np.ascontiguousarray(v).view(np.uint8).reshape(-1).copy()
                      for k, v in (("pdata", data), ("pnulls", nulls), ("parea", area))}


def call(lib, fid, args, n, device, stream=None, host_args=()):
    """one XCall with every slot in host or in device memory (args[i] for i in host_args stays on the host) -> (rc, message, kernel
    launches, stream idle on return, {slot: bytes})"""
    arr = (capi.XCallArgs * len(args))()
    bufs = {}
    for i, a in enumerate(args):
        for s, v in a.slots.items():
            if v is None:
                continue
            b = DeviceBuffer.from_numpy(v, lib) if device and i not in host_args else v.copy()
            bufs[(i, s)] = b
            setattr(arr[i], s, b.ptr if isinstance(b, DeviceBuffer) else b.ctypes.data)
        if a.slots["pdata"] is not None:
            arr[i].dataSz = a.slots["pdata"].nbytes
        if a.slots["pnulls"] is not None:
            arr[i].nullCnt = n
        if a.slots["parea"] is not None:
            arr[i].areaSz = a.slots["parea"].nbytes
    capi.check(lib.MoB200_Sync(), lib)
    if stream is not None:
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SLEEP_CYCLES)
    err = (C.c_uint8 * 256)()
    c0 = lib.MoB200_KernelLaunchCount()
    rc = lib.XCall(1, fid, err, C.cast(arr, C.c_void_p), n)
    launches = lib.MoB200_KernelLaunchCount() - c0
    idle = stream.query() if stream is not None else None
    capi.check(lib.MoB200_Sync(), lib)
    msg = bytes(err[1:1 + err[0]]).decode(errors="replace")   # "mo_b200 rc=<rc>: <text>"
    out = {k: b.to_numpy(np.uint8).tobytes() if isinstance(b, DeviceBuffer) else b.tobytes() for k, b in bufs.items()}
    for b in bufs.values():
        if isinstance(b, DeviceBuffer):
            b.free()
    return rc, msg, launches, idle, out


# ---- operands
def words(n):
    return (n + 63) // 64


def rand_bits(rng, n, p):
    b = np.zeros(words(n) * 64, dtype=bool)
    b[:n] = rng.random(n) < p
    return np.packbits(b, bitorder="little").view(np.uint64).copy()


def result_nulls(rng, n):
    """NOT selectList for rows [0, n) and ones past n"""
    w = rand_bits(rng, n, 0.1)
    if n & 63:
        w[-1] |= np.uint64(~((1 << (n & 63)) - 1) & 0xffffffffffffffff)
    return w


def d128(vals):
    v = np.asarray(vals, dtype=np.int64)
    out = np.empty((len(v), 2), dtype=np.int64)
    out[:, 0] = v
    out[:, 1] = np.where(v < 0, -1, 0)
    return out


ONE_NULL = np.array([1], dtype=np.uint64)


def operand_pair(rng, shape, n, make):
    """two Args in the given shape; make(rng, k) -> (data, area or None) of k rows"""
    def one(kind):
        if kind == "v":
            d, area = make(rng, n)
            return Arg(d, rand_bits(rng, n, 0.1), area)
        d, area = make(rng, 1)
        return Arg(d, ONE_NULL if kind == "n" else np.zeros(1, np.uint64), area)
    return [one("v"), one("v")] if shape == "len1" else [one(shape[0]), one(shape[1])]


def ints(lo, hi, dt):
    return lambda rng, k: (rng.integers(lo, hi, k).astype(dt), None)


def strings(rng, k):
    vocab = [b"", b"ab", b"abc", b"xaby", b"a" * 30, b"zz-ab-" * 7, b"\xe4\xb8\xad", b"B"]
    return varlena_bytes_column([vocab[i] for i in rng.integers(0, len(vocab), k)])


def pattern(rng, k):
    vocab = [b"%ab%", b"a_c", b"%", b"x%y", b"_" * 30 + b"%", b"B"]
    return varlena_bytes_column([vocab[i] for i in rng.integers(0, len(vocab), k)])


def go_params(div0_null=0):
    p = np.zeros(2, np.int64)
    p.view(np.int32)[0] = div0_null
    p[1] = -1
    return Arg(p)


def dec_params(s1, s2, div0_error=0):
    p = np.zeros(3, np.int64)
    p.view(np.int32)[0:2] = (s1, s2)
    p[1] = -1
    p.view(np.int32)[4] = div0_error
    return Arg(p)


# ---- the table: name -> (funcId, builder(rng, shape, n) -> (args, result width), shapes, launches(shape), tail rule)
# tail rule: "merge" = cleared, or kept where a const NULL operand nulls every row; "clear"; "keep"
def binary(fid, make, out_w, params=None):
    def build(rng, shape, n):
        res = Arg(np.full(out_w * n, 0x5a, np.uint8), result_nulls(rng, n))
        return [res] + operand_pair(rng, shape, n, make) + ([params()] if params else [])
    return fid, build


def between(T, make, bounds):
    def build(rng, shape, n):
        d, _ = make(rng, n)
        return [Arg(np.full(n, 0x5a, np.uint8), result_nulls(rng, n)), Arg(d, rand_bits(rng, n, 0.1)), Arg(bounds[0]), Arg(bounds[1])]
    return capi.XCALL_GO_BETWEEN(T), build


def multi(is_or):
    def build(rng, shape, n):
        kinds = {"vv": "vvv", "vc": "vvc", "cv": "cvv", "nc": "nvv", "cn": "vvn", "len1": "vvv"}[shape]
        ops = []
        for k in kinds:
            if k == "v":
                ops.append(Arg(rng.integers(0, 2, n).astype(np.uint8), rand_bits(rng, n, 0.2)))
            else:
                ops.append(Arg(np.array([1 if is_or else 0], np.uint8) if k == "c" else np.zeros(1, np.uint8), ONE_NULL if k == "n" else None))
        return [Arg(np.full(n, 0x5a, np.uint8), result_nulls(rng, n)), Arg(np.array([len(ops)], np.int32))] + ops
    return (capi.XCALL_GO_MULTI_OR if is_or else capi.XCALL_GO_MULTI_AND), build


def avg(width):
    def build(rng, shape, n):
        sums = d128(rng.integers(-10 ** 12, 10 ** 12, n))
        cnts = rng.integers(0, 5, n).astype(np.int64)
        return [Arg(np.full(16 * n, 0x5a, np.uint8), result_nulls(rng, n)), Arg(sums), Arg(cnts), dec_params(2, 0)]
    return capi.XCALL_DEC_AVG(width), build


def build_like(rng, shape, n):
    """GO_LIKE's subject and pattern: a const pattern, a const subject, either const NULL"""
    res = Arg(np.full(n, 0x5a, np.uint8), result_nulls(rng, n))
    subj = operand_pair(rng, shape, n, strings)[0]
    pat = operand_pair(rng, shape, n, pattern)[1]
    return [res, subj, pat]


ALL, COLUMNS = SHAPES, ["vv", "len1"]
KERNELS_2 = lambda shape: 1 if shape in ("nc", "cn") else 2   # the null merge, then the row kernel unless every row is NULL
CALLS = {
    "arith_add_i64": (*binary(capi.XCALL_GO_ARITH(0, capi.T_INT64), ints(-10 ** 9, 10 ** 9, np.int64), 8, go_params), ALL, KERNELS_2, "merge"),
    "arith_mod_f32": (*binary(capi.XCALL_GO_ARITH(4, capi.T_FLOAT32), ints(1, 50, np.float32), 4, lambda: go_params(1)), ALL, KERNELS_2, "merge"),
    "arith_mul_u16": (*binary(capi.XCALL_GO_ARITH(2, capi.T_UINT16), ints(0, 200, np.uint16), 2, go_params), ALL, KERNELS_2, "merge"),
    "compare_i64": (*binary(capi.XCALL_GO_COMPARE(3, capi.T_INT64), ints(-5, 5, np.int64), 1), ALL, KERNELS_2, "merge"),
    "compare_i8": (*binary(capi.XCALL_GO_COMPARE(4, capi.T_INT8), ints(-5, 5, np.int8), 1), ALL, KERNELS_2, "merge"),
    "compare_f32_scale": (*binary(capi.XCALL_GO_COMPARE_F32_SCALE(0, 1), lambda r, k: ((r.integers(0, 40, k) / 8).astype(np.float32), None), 1),
                          ALL, KERNELS_2, "merge"),
    "compare_dec64": (*binary(capi.XCALL_GO_COMPARE(2, capi.T_DECIMAL64), ints(-500, 500, np.int64), 1, lambda: dec_params(2, 3)),
                      ALL, lambda s: 2, "merge"),
    "compare_dec128": (*binary(capi.XCALL_GO_COMPARE(5, capi.T_DECIMAL128), lambda r, k: (d128(r.integers(-500, 500, k)), None), 1,
                               lambda: dec_params(3, 2)), ALL, lambda s: 2, "merge"),
    "compare_varchar": (*binary(capi.XCALL_GO_COMPARE(4, capi.T_VARCHAR), strings, 1), ALL, lambda s: 1, "clear"),
    "like": (capi.XCALL_GO_LIKE, build_like, ALL, lambda s: 1, "clear"),
    "between_i32": (*between(capi.T_INT32, ints(0, 100, np.int32), (np.array([20], np.int32), np.array([60], np.int32))),
                    COLUMNS, lambda s: 1, "keep"),
    "between_dec128": (*between(capi.T_DECIMAL128, lambda r, k: (d128(r.integers(-100, 100, k)), None), (d128([-20]), d128([60]))),
                       COLUMNS, lambda s: 1, "keep"),
    "multi_and": (*multi(0), ALL, lambda s: 1, "clear"),
    "multi_or": (*multi(1), ALL, lambda s: 1, "clear"),
    "dec_add_64": (*binary(capi.XCALL_DEC_ARITH(0, 64), ints(-10 ** 9, 10 ** 9, np.int64), 8, lambda: dec_params(2, 3)), ALL, KERNELS_2, "merge"),
    "dec_mul_128": (*binary(capi.XCALL_DEC_ARITH(2, 128), lambda r, k: (d128(r.integers(-10 ** 9, 10 ** 9, k)), None), 16,
                            lambda: dec_params(2, 3)), ALL, KERNELS_2, "merge"),
    "dec_div_64": (*binary(capi.XCALL_DEC_ARITH(3, 64), ints(1, 10 ** 9, np.int64), 16, lambda: dec_params(2, 3)), ALL, KERNELS_2, "merge"),
    "dec_div_128": (*binary(capi.XCALL_DEC_ARITH(3, 128), lambda r, k: (d128(r.integers(1, 10 ** 12, k)), None), 16,
                            lambda: dec_params(4, 1, 1)), ALL, KERNELS_2, "merge"),
    "dec_avg_64": (*avg(64), COLUMNS, lambda s: 1, "clear"),
    "dec_avg_128": (*avg(128), COLUMNS, lambda s: 1, "clear"),
}


PARAMS = [(name, shape) for name, c in CALLS.items() for shape in c[2]]


def build(name, shape):
    fid, make, _, _, _ = CALLS[name]
    n = 1 if shape == "len1" else N
    rng = np.random.default_rng(sum(map(ord, name + shape)))
    return fid, make(rng, shape, n), n


@pytest.mark.parametrize("name,shape", PARAMS)
def test_host_and_device_forms_agree(gpu, name, shape):
    fid, args, n = build(name, shape)
    rc_h, msg_h, k_h, _, host = call(gpu, fid, args, n, device=False)
    rc_d, msg_d, k_d, _, dev = call(gpu, fid, args, n, device=True)
    assert rc_h == rc_d == 0, (msg_h, msg_d)
    assert k_h == k_d == CALLS[name][3](shape), (k_h, k_d)
    for slot in host:
        assert host[slot] == dev[slot], slot
    rn_in = args[0].slots["pnulls"].view(np.uint64)
    rn = np.frombuffer(host[(0, "pnulls")], np.uint64)
    if shape in ("nc", "cn") and not name.startswith("multi"):   # AND / OR are three-valued: a NULL operand may leave a row decided
        assert (np.unpackbits(rn.view(np.uint8), bitorder="little")[:n] == 1).all(), "a const NULL operand nulls every row"
    rule = CALLS[name][4]
    if n & 63:
        past = np.uint64(~((1 << (n & 63)) - 1) & 0xffffffffffffffff)
        keep = rule == "keep" or (rule == "merge" and shape in ("nc", "cn"))
        assert rn[-1] & past == (rn_in[-1] & past if keep else 0), (rule, hex(int(rn[-1])))


def short(args, k, n):
    """args with operand k's data one row short (or None: a short result; "nulls": no result bitmap)"""
    out = [Arg() for _ in args]
    for i, a in enumerate(args):
        out[i].slots = dict(a.slots)
    if k == "nulls":
        out[0].slots["pnulls"] = None
    else:
        d = out[k].slots["pdata"]
        out[k].slots["pdata"] = d[: d.nbytes * (n - 1) // n]
    return out


@pytest.mark.parametrize("name", list(CALLS))
@pytest.mark.parametrize("what", ["operand", "result", "nulls"])
def test_short_buffers_are_refused_alike(gpu, name, what):
    fid, args, n = build(name, "vv")
    bad = short(args, {"operand": 2 if name.startswith("multi") else 1, "result": 0, "nulls": "nulls"}[what], n)
    rc_h, msg_h, k_h, _, _ = call(gpu, fid, bad, n, device=False)
    rc_d, msg_d, k_d, _, _ = call(gpu, fid, bad, n, device=True)
    assert rc_h == rc_d == capi.RC_INVALID_ARGUMENT, (msg_h, msg_d)
    assert msg_h == msg_d and k_h == k_d == 0


def test_dec_div_const_null_dividend_before_const_zero_divisor(gpu):
    n = 300
    for width in (64, 128):
        a = np.zeros(1, np.int64) if width == 64 else d128([5])
        b = np.zeros(1, np.int64) if width == 64 else d128([0])
        args = [Arg(np.full(16 * n, 0x5a, np.uint8), np.zeros(words(n), np.uint64)), Arg(a, ONE_NULL), Arg(b), dec_params(2, 2, 1)]
        for device in (False, True):
            rc, msg, k, _, out = call(gpu, capi.XCALL_DEC_ARITH(3, width), args, n, device)
            assert rc == 0 and k == 1, msg
            rn = np.frombuffer(out[(0, "pnulls")], np.uint64)
            assert (np.unpackbits(rn.view(np.uint8), bitorder="little")[:n] == 1).all()
            assert np.frombuffer(out[(3, "pdata")], np.int64)[1] == -1


@pytest.mark.parametrize("width", [64, 128])
@pytest.mark.parametrize("zero_first", [True, False])
def test_dec_div_earlier_failing_row_wins(gpu, width, zero_first):
    n = 700
    a = np.full(n, 7, np.int64)
    b = np.full(n, 3, np.int64)
    big = (1 << 63) - 1
    zero_row, over_row = (100, 500) if zero_first else (500, 100)
    b[zero_row] = 0
    if width == 64:
        a[over_row] = big; b[over_row] = 1                  # needs scale 18 + 6: the Decimal128 quotient overflows only at 128 bits
        A, B, s1, s2 = a, b, 0, 18
    else:
        A, B, s1, s2 = d128(a), d128(b), 0, 20
        A[over_row] = (-1, 0x7fffffffffffffff)
    args = [Arg(np.full(16 * n, 0x5a, np.uint8), np.zeros(words(n), np.uint64)), Arg(A), Arg(B), dec_params(s1, s2, 1)]
    got = [call(gpu, capi.XCALL_DEC_ARITH(3, width), args, n, device) for device in (False, True)]
    (rc_h, msg_h, _, _, host), (rc_d, msg_d, _, _, dev) = got
    assert rc_h == rc_d and msg_h == msg_d
    err_h, err_d = (np.frombuffer(o[(3, "pdata")], np.int64)[1] for o in (host, dev))
    assert err_h == err_d == min(zero_row, over_row)
    if zero_first:
        assert rc_h == capi.RC_DIVISION_BY_ZERO and msg_h.endswith(": division by zero"), msg_h
    else:
        assert rc_h == capi.RC_INVALID_ARGUMENT and msg_h.endswith("Decimal128 Div overflow at row %d" % over_row), msg_h
    assert host[(0, "pdata")][:16 * min(zero_row, over_row)] == dev[(0, "pdata")][:16 * min(zero_row, over_row)]


@pytest.mark.parametrize("op,T,a_bad,b_bad,sym", [
    (0, capi.T_INT64, (1 << 62) + 5, (1 << 62), "+"), (1, capi.T_INT32, -(1 << 31) + 2, 3, "-"), (2, capi.T_INT16, 300, 200, "*"),
    (2, capi.T_UINT64, 1 << 40, 1 << 30, "*"), (3, capi.T_FLOAT64, 5, 0, None), (4, capi.T_INT32, 5, 0, None), (4, capi.T_FLOAT32, 5, 0, None)])
def test_go_arith_first_failing_row(gpu, op, T, a_bad, b_bad, sym):
    dt = {capi.T_INT64: np.int64, capi.T_INT32: np.int32, capi.T_INT16: np.int16, capi.T_UINT64: np.uint64, capi.T_FLOAT64: np.float64,
          capi.T_FLOAT32: np.float32}[T]
    n = 900
    a = np.full(n, 2, dt); b = np.full(n, 1, dt)
    for row in (611, 222, 800):
        a[row], b[row] = a_bad, b_bad
    args = [Arg(np.full(n * a.itemsize, 0x5a, np.uint8), np.zeros(words(n), np.uint64)), Arg(a), Arg(b), go_params()]
    got = [call(gpu, capi.XCALL_GO_ARITH(op, T), args, n, device) for device in (False, True)]
    (rc_h, msg_h, k_h, _, host), (rc_d, msg_d, k_d, _, dev) = got
    assert rc_h == rc_d and msg_h == msg_d and k_h == k_d == 2
    assert np.frombuffer(host[(3, "pdata")], np.int64)[1] == np.frombuffer(dev[(3, "pdata")], np.int64)[1] == 222
    assert host[(0, "pdata")][:222 * a.itemsize] == dev[(0, "pdata")][:222 * a.itemsize]
    if sym is None:
        assert rc_h == capi.RC_DIVISION_BY_ZERO and msg_h.endswith(": division by zero"), msg_h
    else:
        assert rc_h == capi.RC_OUT_OF_RANGE
        assert "data out of range" in msg_h and "'(%s %s %s)'" % (a_bad, sym, b_bad) in msg_h, msg_h


@pytest.fixture
def stream(gpu):
    s = torch.cuda.Stream()
    capi.check(gpu.MoB200_SetStream(C.c_void_p(s.cuda_stream)), gpu)
    yield s
    capi.check(gpu.MoB200_SetStream(None), gpu)


@pytest.mark.parametrize("name,shape", [(name, shape) for name in ("compare_dec64", "compare_dec128") for shape in ("vv", "vc", "nc", "cn")] +
                         [("dec_avg_64", "vv"), ("dec_avg_128", "vv")])
def test_decimal_compare_and_avg_only_enqueue_on_device_operands(gpu, stream, name, shape):
    fid, args, n = build(name, shape)
    # a device parameter block is read back before the call enqueues work, so the block stays on the host here
    rc, msg, _, idle, dev = call(gpu, fid, args, n, device=True, stream=stream, host_args=(3,))
    assert rc == 0, msg
    assert not idle, "the all-device call waited for its stream"
    rc, msg, _, idle, host = call(gpu, fid, args, n, device=False, stream=stream)
    assert rc == 0 and idle, msg
    assert host == dev
