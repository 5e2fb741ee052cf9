"""One rule for every entry point with an asynchronous form: the call only enqueues work exactly when every data pointer, nulls bitmap and
varlena area it touches is device memory; otherwise it copies back and synchronises once.  Host parameter blocks do not count.

Every case starts from its all-device call and moves one pointer slot (or, for calls whose columns must all live on one side, the column
group) to the host at a time.  After MoB200_Sync every slot, inputs, results and nulls words alike, must hold the bytes of the all-host
form.  The calls run on an adopted torch stream behind a ~50 ms device sleep: a call with a host slot must return with that stream idle,
and an all-device call that never reads back must return while the sleep is still running."""
import ctypes as C

import numpy as np
import pytest

from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer, bitmap_from_bools, varlena_bytes_column

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 100_000_000     # about 50 ms at H100 clocks
N = 5000
FILL = 0xabababababababab


class Arg:
    """one mo_xcall_args_t: numpy contents of its pointer slots (None = NULL); host=True keeps it in host memory (a parameter block)"""

    def __init__(self, data=None, nulls=None, area=None, null_bits=None, host=False):
        self.slots = {k: None if v is None else np.ascontiguousarray(v).view(np.uint8).reshape(-1).copy()
                      for k, v in (("pdata", data), ("pnulls", nulls), ("parea", area))}
        self.null_bits, self.host = null_bits, host


class Case:
    """fid, args, len; groups: slot groups that change residency together (default: every pointer slot of a non-host argument alone);
    reads_back: the asynchronous form reads one record back by design, so only the host-slot synchronisation applies"""

    def __init__(self, fid, args, n, groups=None, reads_back=False):
        self.fid, self.args, self.n, self.reads_back = fid, args, n, reads_back
        self.groups = groups or [[(i, s)] for i, a in enumerate(args) if not a.host for s, v in a.slots.items() if v is not None]


def params(struct):
    return Arg(np.frombuffer(bytes(struct), dtype=np.uint8), host=True)


def run(lib, case, host_slots, stream=None):
    """one call with `host_slots` in host memory (every other slot on the device) -> (rc, stream idle on return, {slot: its bytes})"""
    arr = (capi.XCallArgs * len(case.args))()
    bufs = {}
    for i, a in enumerate(case.args):
        for s, v in a.slots.items():
            if v is None:
                continue
            if a.host or (i, s) in host_slots:
                b = v.copy(); ptr = b.ctypes.data
            else:
                b = DeviceBuffer.from_numpy(v, lib); ptr = b.ptr
            bufs[(i, s)] = b
            setattr(arr[i], s, ptr)
        if a.slots["pdata"] is not None:
            arr[i].dataSz = a.slots["pdata"].nbytes
        if a.slots["pnulls"] is not None:
            arr[i].nullCnt = a.null_bits if a.null_bits is not None else case.n
        if a.slots["parea"] is not None:
            arr[i].areaSz = a.slots["parea"].nbytes
    if stream is not None:
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SLEEP_CYCLES)
    err = (C.c_uint8 * 256)()
    rc = lib.XCall(1, case.fid, err, C.cast(arr, C.c_void_p), case.n)
    idle = stream.query() if stream is not None else None
    capi.check(lib.MoB200_Sync(), lib)
    out = {k: b.tobytes() if isinstance(b, np.ndarray) else b.to_numpy(np.uint8).tobytes() for k, b in bufs.items()}
    for b in bufs.values():
        if isinstance(b, DeviceBuffer):
            b.free()
    return rc, idle, out


def forms(case):
    """(label, host slots): all host, all device, then each group alone on the host"""
    every = {x for g in case.groups for x in g}
    return [("host", every), ("device", set())] + [("host %s" % g, set(g)) for g in case.groups]


# ---- the cases: one per entry point with an asynchronous form
def rng(seed):
    return np.random.default_rng(seed)


def nulls_of(r, n, p=0.2):
    return bitmap_from_bools(r.random(n) < p)


def result24():
    return np.full(24, 0xab, np.uint8), np.full(1, FILL, np.uint64)


def case_agg():
    r = rng(1)
    res, rn = result24()
    return Case(capi.XCALL_AGG(capi.AGG_SUM, capi.T_INT64), [Arg(res, rn), Arg(r.integers(-1000, 1000, N), nulls_of(r, N))], N)


def case_agg_merge():
    parts = np.array([[5, 2, 0], [0, 0, 0], [-7, 3, 0]], dtype=np.int64)
    res, rn = result24()
    return Case(capi.XCALL_AGG_MERGE(capi.AGG_SUM, capi.T_INT64), [Arg(res, rn), Arg(parts)], len(parts))


def case_filter_sels():
    r = rng(2)
    bools = (r.random(N) < 0.4).astype(np.uint8)
    nulls = r.random(N) < 0.1
    count = int((bools.astype(bool) & ~nulls).sum())
    sels = np.full(count, -1, np.int64)       # a host sels buffer only has to hold the selected rows
    return Case(capi.XCALL_FILTER_SELS, [Arg(sels), Arg(np.full(1, -1, np.int64)), Arg(bools, bitmap_from_bools(nulls))], N)


def case_shuffle():
    r = rng(3)
    m = 3 * N
    src, sels = r.integers(0, 1 << 40, m), r.integers(0, m, N)
    return Case(capi.XCALL_SHUFFLE(8), [Arg(np.full(N, -1, np.int64), np.full((N + 63) // 64, FILL, np.uint64)),
                                        Arg(src, nulls_of(r, m), null_bits=m), Arg(sels)], N)


def str_keys(r, n, vocab):
    vals = [vocab[i] for i in r.integers(0, len(vocab), n)]
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum([len(v) for v in vals])
    return np.frombuffer(b"".join(vals), np.uint8), off


VOCAB = [(b"key-%d-" % i) * (1 + i % 5) for i in range(40)]


def case_pack_str_keys():
    r = rng(4)
    cells, area = varlena_bytes_column([VOCAB[i] for i in r.integers(0, len(VOCAB), N)])
    P = ops._strkey_params([capi.T_VARCHAR, capi.T_INT64], False)
    return Case(capi.XCALL_PACK_STR_KEYS, [Arg(np.full(64 * N, 0xab, np.uint8)), Arg(np.full(N + 1, 7, np.uint64), np.full((N + 63) // 64, FILL, np.uint64)),
                                           params(P), Arg(cells, nulls_of(r, N), area), Arg(r.integers(0, 9, N), nulls_of(r, N))], N,
                reads_back=True)


def case_str_group_ids():
    r = rng(5)
    kb, ko = str_keys(r, N, VOCAB)
    cap = 64
    return Case(capi.XCALL_STR_GROUP_IDS, [Arg(np.full(N, 7, np.uint64)), Arg(np.zeros(1, np.int64)), Arg(np.full(4096, 0xab, np.uint8)),
                                           Arg(np.zeros(cap + 1, np.uint64)), Arg(kb), Arg(ko, nulls_of(r, N)), Arg(np.full(N, -1, np.int64))], N,
                reads_back=True)


def case_str_join_find():
    r = rng(6)
    table = VOCAB[:30]
    toff = np.zeros(len(table) + 1, np.uint64)
    toff[1:] = np.cumsum([len(v) for v in table])
    kb, ko = str_keys(r, N, VOCAB)
    return Case(capi.XCALL_STR_JOIN_FIND, [Arg(np.full(N, 7, np.uint64)), params(C.c_int64(len(table))),
                                           Arg(np.frombuffer(b"".join(table), np.uint8)), Arg(toff), Arg(kb), Arg(ko, nulls_of(r, N))], N)


def case_order(varlena):
    r = rng(7)
    sels = np.full(N, -1, np.int64)
    if varlena:
        cells, area = varlena_bytes_column([VOCAB[i] for i in r.integers(0, len(VOCAB), N)])
        P = ops._order_params([capi.T_VARCHAR, capi.T_INT32], [capi.ORDER_DESC, 0], None, False)
        keys = [Arg(cells, nulls_of(r, N), area), Arg(r.integers(0, 50, N).astype(np.int32))]
    else:
        P = ops._order_params([capi.T_INT64, capi.T_FLOAT64], [capi.ORDER_DESC, 0], None, True)
        keys = [Arg(r.integers(0, 100, N), nulls_of(r, N)), Arg(r.integers(0, 8, N) / 4.0), Arg(np.arange(N, dtype=np.int64) * 3)]
    return Case(capi.XCALL_ORDER_SELS, [Arg(sels), params(P)] + keys, N, reads_back=varlena)


Q6_NAMES = ("shipdate", "discount", "quantity", "extendedprice")
Q1_NAMES = ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")


def col_group(first, count):
    return [[(first + c, "pdata") for c in range(count)]]


def lineitem():
    return datagen.lineitem(10, 0, N)


def case_q6():
    cols = lineitem()
    res = np.full(16, 0xab, np.uint8)
    args = [Arg(res, np.full(1, FILL, np.uint64))] + [Arg(cols[k]) for k in Q6_NAMES] + [params(capi.Q6Params(*datagen.q6_params()))]
    return Case(capi.XCALL_Q6_FILTER_SUM, args, N, groups=[[(0, "pdata")], [(0, "pnulls")]] + col_group(1, 4))


def case_q6_dec():
    cols = lineitem()
    lo, hi = datagen.q6_params()[:2]
    meas = [np.round(cols[k] * 100).astype(np.int64) for k in ("discount", "quantity", "extendedprice")]
    args = [Arg(np.full(C.sizeof(capi.Q6DecResult), 0xab, np.uint8), np.full(1, FILL, np.uint64)), Arg(cols["shipdate"])] + \
           [Arg(m) for m in meas] + [params(capi.Q6DecParams(lo, hi, 2, 4, 2400, 2, 0, 0))]   # q6.sql at DECIMAL(15,2)
    return Case(capi.XCALL_Q6_DEC_FILTER_SUM, args, N, groups=[[(0, "pdata")], [(0, "pnulls")]] + col_group(1, 4))


def case_q6_dec_merge():
    parts = b"".join(bytes(capi.Q6DecResult(lo, 0, cnt, -1, 0, 2)) for lo, cnt in ((12345, 3), (0, 0), (678, 1)))
    return Case(capi.XCALL_Q6_DEC_MERGE, [Arg(np.full(C.sizeof(capi.Q6DecResult), 0xab, np.uint8), np.full(1, FILL, np.uint64)),
                                          Arg(np.frombuffer(parts, np.uint8))], 3)


def case_q6_merge():
    parts = np.zeros(3, dtype=[("sum", np.float64), ("count", np.int64)])
    parts["sum"], parts["count"] = (1.5, 0.0, 2.25), (3, 0, 7)
    return Case(capi.XCALL_Q6_MERGE, [Arg(np.full(16, 0xab, np.uint8), np.full(1, FILL, np.uint64)), Arg(parts)], 3)


def q1_args(cols, r0, r1, res):
    return [Arg(res)] + [Arg(cols[k][r0:r1]) for k in Q1_NAMES] + [params(capi.Q1Params(datagen.Q1_CUTOFF, 0, r0))]


def case_q1():
    return Case(capi.XCALL_Q1_GROUP_AGG, q1_args(lineitem(), 0, N, np.full(ops.Q1_RESULT_BYTES, 0xab, np.uint8)), N,
                groups=[[(0, "pdata")]] + col_group(1, 7))


def case_q1_merge(lib):
    cols = lineitem()
    parts = []
    for r0, r1 in ((0, 2000), (2000, N)):
        c = Case(capi.XCALL_Q1_GROUP_AGG, q1_args(cols, r0, r1, np.zeros(ops.Q1_RESULT_BYTES, np.uint8)), r1 - r0, groups=[])
        rc, _, out = run(lib, c, set())
        assert rc == 0
        parts.append(out[(0, "pdata")])
    return Case(capi.XCALL_Q1_MERGE, [Arg(np.full(ops.Q1_RESULT_BYTES, 0xab, np.uint8)), Arg(np.frombuffer(b"".join(parts), np.uint8))], 2)


def case_plan(shape):
    if shape == "interpreter":
        r = rng(8)
        p = ops.FusedPlan([capi.T_INT32, capi.T_FLOAT64]).where(1, "<", 1.0).group_by(0).agg(capi.AGG_SUM, 1).agg(capi.AGG_COUNT, -1)
        # quarters: every partial sum is exact, so the order in which the atomics add them cannot change the bytes
        args = [Arg(np.full(p.result_bytes(5), 0xab, np.uint8)), params(p.P), Arg((np.arange(N) % 5).astype(np.int32)),
                Arg(r.integers(0, 8, N) / 4.0, nulls_of(r, N))]
        return Case(capi.XCALL_PLAN, args, N, reads_back=True)   # the descriptor is staged behind a synchronise
    cols = lineitem()
    p, names, groups = (ops.q6_plan(), Q6_NAMES, 1) if shape == "q6" else (ops.q1_plan(datagen.Q1_CUTOFF, row_base=3), Q1_NAMES, 4)
    args = [Arg(np.full(p.result_bytes(groups), 0xab, np.uint8)), params(p.P)] + [Arg(cols[k]) for k in names]
    return Case(capi.XCALL_PLAN, args, N, groups=[[(0, "pdata")]] + col_group(2, len(names)), reads_back=shape == "q1")


CASES = {
    "agg": case_agg, "agg_merge": case_agg_merge, "filter_sels": case_filter_sels, "shuffle": case_shuffle,
    "pack_str_keys": case_pack_str_keys, "str_group_ids": case_str_group_ids, "str_join_find": case_str_join_find,
    "order": lambda: case_order(False), "order_varlena": lambda: case_order(True),
    "q6": case_q6, "q6_dec": case_q6_dec, "q6_dec_merge": case_q6_dec_merge, "q6_merge": case_q6_merge, "q1": case_q1, "q1_merge": None,
    "plan_q6": lambda: case_plan("q6"), "plan_q1": lambda: case_plan("q1"), "plan_interpreter": lambda: case_plan("interpreter"),
}


def make(lib, name):
    return case_q1_merge(lib) if name == "q1_merge" else CASES[name]()


@pytest.fixture
def stream(gpu):
    """the library runs on a torch stream for the test; the finaliser gives it back its own"""
    s = torch.cuda.Stream()
    capi.check(gpu.MoB200_SetStream(C.c_void_p(s.cuda_stream)), gpu)
    yield s
    capi.check(gpu.MoB200_SetStream(None), gpu)


@pytest.mark.parametrize("name", list(CASES))
def test_every_host_slot_gives_the_bytes_of_the_host_form(gpu, stream, name):
    case = make(gpu, name)
    want = None
    for label, host in forms(case):
        rc, _, out = run(gpu, case, host)
        assert rc == 0, (label, capi.last_error(gpu))
        if want is None:
            want = out
        for slot in want:
            assert out[slot] == want[slot], (label, slot)


@pytest.mark.parametrize("name", list(CASES))
def test_the_call_synchronises_exactly_when_a_slot_is_host(gpu, stream, name):
    case = make(gpu, name)
    for label, host in forms(case):
        rc, idle, _ = run(gpu, case, host, stream)
        assert rc == 0, (label, capi.last_error(gpu))
        if host:
            assert idle, "%s: returned before its stream ran" % label
        elif not case.reads_back:
            assert not idle, "the all-device call waited for its stream"
