"""Parameter blocks and scalar arguments may be host or device memory at every entry point (include/mo_b200.h).

Every case calls its XCall twice per data placement with identical bytes: once with its parameter slots in host memory and once in device
memory, the data slots staying where they are (all host, then all device).  The return code and every pointer slot must match, the words a
call writes into its block included (err_row, ngroups, the k-means iteration count).  A parameter block too short to read is refused with
the same return code and message in both forms."""
import ctypes as C

import numpy as np
import pytest

from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import bitmap_from_bools, varlena_bytes_column
from test_gpu_async_forms import Arg, Case, run

pytestmark = pytest.mark.gpu

N = 2000
FILL = 0xabababababababab


def rng(seed):
    return np.random.default_rng(seed)


def nulls_of(r, n, p=0.2, keep=None):
    """a nulls bitmap; row `keep` is not NULL"""
    mask = r.random(n) < p
    if keep is not None:
        mask[keep] = False
    return bitmap_from_bools(mask)


def block(struct):
    return Arg(np.frombuffer(bytes(struct), np.uint8))


def scalar(v, dtype):
    return Arg(np.array([v], dtype))


# ---- the cases: (Case, indices of its parameter arguments)
LINEITEM = None


def lineitem():
    global LINEITEM
    if LINEITEM is None:
        LINEITEM = datagen.lineitem(10, 0, N)
    return LINEITEM


Q6_NAMES = ("shipdate", "discount", "quantity", "extendedprice")
Q1_NAMES = ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")


def dyadic(r, cols):
    """the measures of `cols` as small multiples of 1/4: with nulls the scans run through the generic operator, whose float64 sums are
    accumulated with atomics, and on these values every order of the additions gives the same bytes"""
    return dict(cols, quantity=r.integers(1, 51, N) * 1.0, extendedprice=r.integers(1, 100_000, N) / 4, discount=r.integers(0, 3, N) / 4,
                tax=r.integers(0, 2, N) / 4)


def case_q6(nullable):
    r = rng(1)
    cols = dyadic(r, lineitem()) if nullable else lineitem()
    data = [Arg(cols[k], nulls_of(r, N) if nullable and k == "discount" else None) for k in Q6_NAMES]
    lo, hi, dlo, dhi, qhi = datagen.q6_params()
    if nullable:
        dlo, dhi = 0.25, 0.5
    args = [Arg(np.full(16, 0xab, np.uint8), np.full(1, FILL, np.uint64))] + data + [block(capi.Q6Params(lo, hi, dlo, dhi, qhi))]
    return Case(capi.XCALL_Q6_FILTER_SUM, args, N), [5]


def case_q6_dec():
    cols = lineitem()
    lo, hi = datagen.q6_params()[:2]
    meas = [np.round(cols[k] * 100).astype(np.int64) for k in ("discount", "quantity", "extendedprice")]
    args = [Arg(np.full(C.sizeof(capi.Q6DecResult), 0xab, np.uint8), np.full(1, FILL, np.uint64)), Arg(cols["shipdate"])] + \
           [Arg(m) for m in meas] + [block(capi.Q6DecParams(lo, hi, 2, 4, 2400, 2, 0, 700))]
    return Case(capi.XCALL_Q6_DEC_FILTER_SUM, args, N), [5]


Q1_ROW_BASE = 1_000_003


def case_q1(nullable=False, cutoff_only=False):
    r = rng(2)
    cols = dyadic(r, lineitem()) if nullable else lineitem()
    data = [Arg(cols[k], nulls_of(r, N) if nullable and k == "tax" else None) for k in Q1_NAMES]
    prm = scalar(datagen.Q1_CUTOFF, np.int32) if cutoff_only else block(capi.Q1Params(datagen.Q1_CUTOFF, 0, Q1_ROW_BASE))
    return Case(capi.XCALL_Q1_GROUP_AGG, [Arg(np.full(ops.Q1_RESULT_BYTES, 0xab, np.uint8))] + data + [prm], N), [8]


class GoParams(C.Structure):
    _fields_ = [("div0_null", C.c_int32), ("reserved", C.c_int32), ("err_row", C.c_int64)]


def case_go_arith(overflow):
    r = rng(3)
    a, b = r.integers(-1000, 1000, N), r.integers(-1000, 1000, N)
    if overflow:
        a[700] = b[700] = 1 << 62
    args = [Arg(np.full(N, -1, np.int64), np.zeros((N + 63) // 64, np.uint64)), Arg(a, nulls_of(r, N, keep=700)), Arg(b), block(GoParams(0, 0, 12345))]
    return Case(capi.XCALL_GO_ARITH(0, capi.T_INT64), args, N), [3]


def case_go_between():
    r = rng(4)
    args = [Arg(np.full(N, 7, np.uint8), np.zeros((N + 63) // 64, np.uint64)), Arg(r.integers(0, 100, N).astype(np.int32), nulls_of(r, N)),
            scalar(20, np.int32), scalar(60, np.int32)]
    return Case(capi.XCALL_GO_BETWEEN(capi.T_INT32), args, N), [2, 3]


def case_go_multi_and():
    r = rng(5)
    operands = [Arg((r.random(N) < 0.7).astype(np.uint8), nulls_of(r, N, 0.1)) for _ in range(3)]
    return Case(capi.XCALL_GO_MULTI_AND, [Arg(np.full(N, 7, np.uint8), np.full((N + 63) // 64, FILL, np.uint64)), scalar(3, np.int32)] + operands, N), [1]


def case_pack_keys(ncols_only):
    r = rng(6)
    prm = scalar(2, np.int32) if ncols_only else Arg(np.array([2, 0], np.int32))
    keys = Arg(np.full(N, FILL, np.uint64), None if ncols_only else np.full((N + 63) // 64, FILL, np.uint64))
    args = [keys, prm, Arg(r.integers(0, 1 << 20, N).astype(np.int32), nulls_of(r, N)), Arg(r.integers(0, 300, N).astype(np.int16))]
    return Case(capi.XCALL_PACK_KEYS, args, N), [1]


def case_group_ids():
    r = rng(7)
    table = np.full(4096, FILL, np.uint64)
    table[:3] = (5, 9, 100)
    args = [Arg(np.full(N, 7, np.uint64)), scalar(3, np.int64), Arg(table), Arg(r.integers(0, 500, N).astype(np.uint64), nulls_of(r, N))]
    return Case(capi.XCALL_GROUP_IDS, args, N), [1]


VOCAB = [(b"key-%d-" % i) * (1 + i % 5) for i in range(40)]


def str_keys(r, n, vocab):
    vals = [vocab[i] for i in r.integers(0, len(vocab), n)]
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum([len(v) for v in vals])
    return np.frombuffer(b"".join(vals), np.uint8), off


def str_table(words, cap_groups, cap_bytes):
    tb = np.full(cap_bytes, 0xab, np.uint8)
    raw = b"".join(words)
    tb[:len(raw)] = np.frombuffer(raw, np.uint8)
    toff = np.zeros(cap_groups + 1, np.uint64)
    toff[1:len(words) + 1] = np.cumsum([len(w) for w in words])
    return tb, toff


def case_str_group_ids():
    r = rng(8)
    kb, ko = str_keys(r, N, VOCAB)
    tb, toff = str_table(VOCAB[:2], 64, 4096)
    args = [Arg(np.full(N, 7, np.uint64)), scalar(2, np.int64), Arg(tb), Arg(toff), Arg(kb), Arg(ko, nulls_of(r, N)), Arg(np.full(N, -1, np.int64))]
    return Case(capi.XCALL_STR_GROUP_IDS, args, N), [1]


def case_pack_str_keys():
    r = rng(9)
    cells, area = varlena_bytes_column([VOCAB[i] for i in r.integers(0, len(VOCAB), N)])
    args = [Arg(np.full(64 * N, 0xab, np.uint8)), Arg(np.full(N + 1, 7, np.uint64), np.full((N + 63) // 64, FILL, np.uint64)),
            block(ops._strkey_params([capi.T_VARCHAR, capi.T_INT64], False)), Arg(cells, nulls_of(r, N), area), Arg(r.integers(0, 9, N), nulls_of(r, N))]
    return Case(capi.XCALL_PACK_STR_KEYS, args, N), [2]


def case_str_join_find():
    r = rng(10)
    kb, ko = str_keys(r, N, VOCAB)
    tb, toff = str_table(VOCAB[:30], 30, len(b"".join(VOCAB[:30])))
    args = [Arg(np.full(N, 7, np.uint64)), scalar(30, np.int64), Arg(tb), Arg(toff), Arg(kb), Arg(ko, nulls_of(r, N))]
    return Case(capi.XCALL_STR_JOIN_FIND, args, N), [1]


def case_dec_arith(overflow):
    r = rng(11)
    a, b = r.integers(-10 ** 9, 10 ** 9, N), r.integers(-10 ** 9, 10 ** 9, N)
    if overflow:
        a[300] = b[300] = 1 << 62
    args = [Arg(np.full(N, -1, np.int64), np.zeros((N + 63) // 64, np.uint64)), Arg(a, nulls_of(r, N, keep=300)), Arg(b), block(capi.DecParams(2, 3, 12345))]
    return Case(capi.XCALL_DEC_ARITH(0, 64), args, N), [3]


def join_probe_args(r, gids):
    """JOIN_PROBE / JOIN_PROBE_GIDS over a unique map of 100 groups, LEFT join: one result row per probe row"""
    ngroups = 100
    head = [Arg(np.full(N, -2, np.int64)), Arg(np.full(N, -2, np.int64)), Arg(np.full(1, -1, np.int64)), Arg(np.array([capi.JOIN_LEFT, 0], np.int32))]
    if gids:
        return head + [scalar(ngroups, np.int64), Arg(), Arg(), Arg(r.integers(0, ngroups + 1, N).astype(np.uint64))]
    return head + [Arg(np.arange(ngroups, dtype=np.uint64) * 3), Arg(), Arg(), Arg(r.integers(0, 400, N).astype(np.uint64), nulls_of(r, N))]


def case_join_probe():
    return Case(capi.XCALL_JOIN_PROBE, join_probe_args(rng(12), False), N), [3]


def case_join_probe_gids():
    return Case(capi.XCALL_JOIN_PROBE_GIDS, join_probe_args(rng(13), True), N), [3, 4]


def case_kmeans():
    r = rng(14)
    n, dim, k = 600, 8, 5
    vec = (r.standard_normal((n, dim)) + np.repeat(r.standard_normal((k, dim)) * 4, n // k, axis=0)).astype(np.float32)
    args = [Arg(vec[::n // k].copy()), Arg(np.full(n, -1, np.int64)), Arg(np.full(1, -1, np.int64)), Arg(np.array([n, dim, k, 50], np.int64)), Arg(vec), Arg()]
    return Case(capi.XCALL_KMEANS_ELKAN_F32, args, n), [2, 3]


def case_order():
    r = rng(15)
    P = ops._order_params([capi.T_INT64, capi.T_FLOAT64], [capi.ORDER_DESC, 0], 700, True)
    args = [Arg(np.full(700, -1, np.int64)), block(P), Arg(r.integers(0, 100, N), nulls_of(r, N)), Arg(r.integers(0, 8, N) / 4.0),
            Arg(np.arange(N, dtype=np.int64) * 3)]
    return Case(capi.XCALL_ORDER_SELS, args, N), [1]


def case_plan():
    r = rng(16)
    p = ops.FusedPlan([capi.T_INT32, capi.T_FLOAT64], row_base=77).where(1, "<", 1.0).group_by(0).agg(capi.AGG_SUM, 1).agg(capi.AGG_COUNT, -1)
    # quarters: every partial sum is exact, so the order of the atomic additions cannot change the bytes
    args = [Arg(np.full(p.result_bytes(5), 0xab, np.uint8)), block(p.P), Arg((np.arange(N) % 5).astype(np.int32)), Arg(r.integers(0, 8, N) / 4.0, nulls_of(r, N))]
    return Case(capi.XCALL_PLAN, args, N), [1]


NQ, K, DIM = 8, 10, 32
FILTER_WORDS = np.zeros(16, np.uint64)   # kept alive for the descriptor, which points at it
FILTER_WORDS[:] = 0x5555555555555555


def search_head(r, n):
    ds, qs = r.standard_normal((n, DIM)).astype(np.float32), r.standard_normal((NQ, DIM)).astype(np.float32)
    return ds, qs, [Arg(np.full(NQ * K, -2, np.int64)), Arg(np.full(NQ * K, np.nan))]


def case_bruteforce(filtered):
    r, n = rng(17), 900
    ds, qs, out = search_head(r, n)
    args = out + [Arg(ds), Arg(qs), block(ops._search_params(n, DIM, NQ, K, capi.METRIC_L2, key_base=40))]
    if not filtered:
        return Case(capi.XCALL_BRUTEFORCE_TOPK_F32, args, NQ), [4]
    desc = capi.SearchFilter(capi.SEARCH_FILTER_KEY_BITMAP, 0, FILTER_WORDS.ctypes.data, FILTER_WORDS.size)
    return Case(capi.XCALL_BRUTEFORCE_TOPK_FILTERED_F32, args + [block(desc)], NQ), [4, 5]


def case_ivf():
    r, n, nlist = rng(18), 1000, 4
    ds, qs, out = search_head(r, n)
    cent = r.standard_normal((nlist, DIM)).astype(np.float32)
    assign = np.argmin(((ds[:, None, :] - cent[None]) ** 2).sum(-1), axis=1)
    order = np.argsort(assign, kind="stable")
    offsets = np.concatenate([[0], np.cumsum(np.bincount(assign, minlength=nlist))]).astype(np.int64)
    P = ops._search_params(n, DIM, NQ, K, capi.METRIC_L2, nprobe=2, nlist=nlist)
    args = out + [Arg(ds[order]), Arg(qs), block(P), Arg(cent), Arg(offsets), Arg(order.astype(np.int64))]
    return Case(capi.XCALL_IVF_TOPK_F32, args, NQ), [4]


def case_topk_merge():
    r, nshards = rng(19), 3
    dists = np.sort(r.random((nshards, NQ, K)), axis=2)
    keys = r.integers(0, 10_000, (nshards, NQ, K))
    args = [Arg(np.full(NQ * K, -2, np.int64)), Arg(np.full(NQ * K, np.nan)), Arg(keys), Arg(dists),
            block(ops._search_params(nshards, 0, NQ, K, 0))]
    return Case(capi.XCALL_TOPK_MERGE, args, NQ), [4]


CASES = {
    "q6": lambda: case_q6(False), "q6_nullable": lambda: case_q6(True), "q6_dec": case_q6_dec,
    "q1": case_q1, "q1_nullable": lambda: case_q1(nullable=True), "q1_cutoff_only": lambda: case_q1(cutoff_only=True),
    "go_arith": lambda: case_go_arith(False), "go_arith_err_row": lambda: case_go_arith(True), "go_between": case_go_between,
    "go_multi_and": case_go_multi_and, "pack_keys": lambda: case_pack_keys(False), "pack_keys_ncols_only": lambda: case_pack_keys(True),
    "group_ids": case_group_ids, "str_group_ids": case_str_group_ids, "pack_str_keys": case_pack_str_keys, "str_join_find": case_str_join_find,
    "dec_arith": lambda: case_dec_arith(False), "dec_arith_err_row": lambda: case_dec_arith(True),
    "join_probe": case_join_probe, "join_probe_gids": case_join_probe_gids, "kmeans": case_kmeans, "order": case_order, "plan": case_plan,
    "bruteforce": lambda: case_bruteforce(False), "bruteforce_filtered": lambda: case_bruteforce(True), "ivf": case_ivf,
    "topk_merge": case_topk_merge,
}


EXPECTED_RC = {"go_arith_err_row": capi.RC_OUT_OF_RANGE, "dec_arith_err_row": capi.RC_INVALID_ARGUMENT}
ERR_ROW = {"go_arith": -1, "go_arith_err_row": 700, "dec_arith": -1, "dec_arith_err_row": 300}


def slots(case, indices):
    return {(i, s) for i in indices for s, v in case.args[i].slots.items() if v is not None}


def both_forms(lib, case, params, data_on_host):
    """(rc, error text, slot bytes) with the parameter slots on the host, then on the device; the data slots on one side throughout"""
    every = slots(case, range(len(case.args)))
    data = every - params
    res = []
    for params_on_host in (True, False):
        host = (data if data_on_host else set()) | (params if params_on_host else set())
        rc, _, out = run(lib, case, host)
        res.append((rc, capi.last_error(lib) if rc else "", out))
    return res


@pytest.mark.parametrize("data_on_host", [True, False], ids=["host data", "device data"])
@pytest.mark.parametrize("name", list(CASES))
def test_a_device_block_gives_the_bytes_of_the_host_block(gpu, name, data_on_host):
    case, idx = CASES[name]()
    (rc_h, err_h, out_h), (rc_d, err_d, out_d) = both_forms(gpu, case, slots(case, idx), data_on_host)
    assert rc_h == EXPECTED_RC.get(name, 0), err_h
    assert (rc_d, err_d) == (rc_h, err_h)
    for slot in out_h:
        assert out_d[slot] == out_h[slot], slot
    if name in ERR_ROW:   # the failing row lands in the caller's block, replacing 12345
        assert np.frombuffer(out_d[(3, "pdata")], np.int64)[1] == ERR_ROW[name]


def test_q1_device_params_shift_first_row_by_row_base(gpu):
    case, idx = case_q1()
    (_, _, out_h), (rc, err, out_d) = both_forms(gpu, case, slots(case, idx), True)
    assert rc == 0, err
    res = capi.Q1Result.from_buffer_copy(out_d[(0, "pdata")])
    first = [res.groups[g].first_row for g in range(res.ngroups)]
    first_qualifying = int(np.flatnonzero(lineitem()["shipdate"] <= datagen.Q1_CUTOFF)[0])
    assert res.ngroups > 0 and min(first) == Q1_ROW_BASE + first_qualifying, first
    assert out_d[(0, "pdata")] == out_h[(0, "pdata")]


@pytest.mark.parametrize("name", list(CASES))
def test_a_short_block_is_refused_alike_on_both_sides(gpu, name):
    case, idx = CASES[name]()
    first = case.args[idx[0]]
    first.slots["pdata"] = first.slots["pdata"][:1].copy()
    (rc_h, err_h, out_h), (rc_d, err_d, out_d) = both_forms(gpu, case, slots(case, idx), True)
    if name.startswith("go_arith"):    # the block is optional: a short one is not read
        assert rc_h in (0, capi.RC_OUT_OF_RANGE)
    else:
        assert rc_h == capi.RC_INVALID_ARGUMENT and err_h, name
    assert (rc_d, err_d) == (rc_h, err_h)
    assert out_d == out_h
