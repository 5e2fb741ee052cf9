"""The synchronous and asynchronous forms of MO_XCALL_AGG, Q6_FILTER_SUM, Q1_GROUP_AGG and the plan's specialised shapes run the same
kernels; the forms differ only in staging and in whether the call synchronises.  Checked here: host columns staged in more than one chunk,
every mix of host and device columns and results against the all-host form, the errors of the synchronous form, and the launch cost of
the asynchronous paths the benchmark times."""
import numpy as np
import pytest

import oracle_lib as O
from matrixone_b200 import capi, datagen, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, xcall

pytestmark = pytest.mark.gpu

CHUNK = 2 ** 25                    # rows per staged chunk of host columns (kHostChunkRows)
N_BIG = CHUNK + 12_345             # two chunks
Q1_NAMES = ("shipdate", "quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus")
Q6_NAMES = ("shipdate", "discount", "quantity", "extendedprice")


@pytest.fixture(scope="module")
def big():
    return datagen.lineitem(10, 0, N_BIG)


def six_keys(cols, n):
    """the same rows with 6 distinct keys: the 4-slot pass overflows and the 8-slot pass answers"""
    c = dict(cols)
    c["returnflag"] = (65 + np.arange(n) * 7 % 6).astype(np.uint8)
    c["linestatus"] = np.full(n, ord("F"), dtype=np.uint8)
    return c


def test_q6_two_host_chunks_equal_merge_of_the_ranges(gpu, big):
    P = datagen.q6_params()
    got = ops.q6_filter_sum(*[big[k] for k in Q6_NAMES], N_BIG, *P)
    parts = [ops.q6_filter_sum(*[big[k][r0:r1] for k in Q6_NAMES], r1 - r0, *P)[:2] for r0, r1 in ((0, CHUNK), (CHUNK, N_BIG))]
    assert got == ops.q6_merge(parts)
    want, ns, _ = O.q6(big, N_BIG, P, nthreads=4)
    assert got[1] == ns and abs(got[0] - want) <= 1e-9 * abs(want)


@pytest.mark.parametrize("keys", ["tpch", "six"])
def test_q1_two_host_chunks_equal_merge_of_the_ranges(gpu, big, keys):
    cols = big if keys == "tpch" else six_keys(big, N_BIG)
    cut, RB = datagen.Q1_CUTOFF, ops.Q1_RESULT_BYTES
    got = ops.q1_group_agg(*[cols[k] for k in Q1_NAMES], N_BIG, cut, row_base=5)
    parts = DeviceBuffer(2 * RB)
    for i, (r0, r1) in enumerate(((0, CHUNK), (CHUNK, N_BIG))):
        dev = [DeviceBuffer.from_numpy(cols[k][r0:r1]) for k in Q1_NAMES]
        ops.q1_group_agg_device(*dev, r1 - r0, cut, parts.ptr + RB * i, row_base=5 + r0)
        for b in dev:
            b.free()
    assert got == ops.q1_merge(parts.to_numpy(np.uint8).tobytes(), 2)
    parts.free()
    ores = O.q1(cols, N_BIG, cut, nthreads=4)
    assert len(got) == (4 if keys == "tpch" else 6)
    assert [(g["returnflag"], g["linestatus"], g["count_order"], g["first_row"] - 5) for g in got] == \
           [(g["returnflag"], g["linestatus"], g["count_order"], g["first_row"]) for g in ores]
    for a, b in zip(got, ores):
        for f in ("sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc"):
            assert abs(a[f] - b[f]) <= 1e-9 * abs(b[f]), f


# ---- mixed forms: each must give the bytes of the all-host form
FORMS = [("host", "host"), ("host", "device"), ("device", "host")]    # (columns, result); device + device is the asynchronous form


def col_vec(x, n, nulls, where, keep):
    if where == "host":
        return Vector(data=x, nulls=nulls, length=n)
    d = DeviceBuffer.from_numpy(x); keep.append(d)
    dn = None
    if nulls is not None:
        dn = DeviceBuffer.from_numpy(nulls); keep.append(dn)
    return Vector(data_ptr=d.ptr, data_nbytes=x.nbytes, nulls_ptr=None if dn is None else dn.ptr, length=n)


class Result:
    """a result vector of `nbytes` (+ an 8-byte nulls word) in host or device memory, pre-filled with 0xab"""

    def __init__(self, nbytes, where, nulls_word, keep):
        self.where = where
        fill = np.full(nbytes, 0xab, dtype=np.uint8)
        fn = np.full(1, 0xabababababababab, dtype=np.uint64)
        if where == "host":
            self.h, self.hn = fill, (fn if nulls_word else None)
            self.vec = Vector(data=self.h, nulls=self.hn, length=1)
        else:
            self.d = DeviceBuffer.from_numpy(fill); keep.append(self.d)
            self.dn = DeviceBuffer.from_numpy(fn) if nulls_word else None
            if self.dn is not None:
                keep.append(self.dn)
            self.vec = Vector(data_ptr=self.d.ptr, data_nbytes=nbytes, nulls_ptr=None if self.dn is None else self.dn.ptr, length=1)

    def bytes(self):
        if self.where == "host":
            return self.h.tobytes(), None if self.hn is None else self.hn.tobytes()
        return self.d.to_numpy(np.uint8).tobytes(), None if self.dn is None else self.dn.to_numpy(np.uint8).tobytes()


def run_forms(call):
    """call(col_where, res_where, keep) -> (rc, bytes); every form must return what the all-host form returns"""
    outs = []
    for cw, rw in FORMS:
        keep = []
        outs.append(call(cw, rw, keep))
        for b in keep:
            b.free()
    assert outs[1] == outs[0] and outs[2] == outs[0]
    return outs[0]


@pytest.mark.parametrize("op", [capi.AGG_SUM, capi.AGG_AVG, capi.AGG_COUNT, capi.AGG_MIN, capi.AGG_MAX])
@pytest.mark.parametrize("T", [capi.T_INT64, capi.T_UINT32, capi.T_FLOAT64])
def test_agg_mixed_forms_equal_host_form(gpu, op, T):
    n = 50_001
    rng = np.random.default_rng(op * 31 + T)
    dt = np.dtype(capi.NP_OF_T[T])
    col = (rng.standard_normal(n) * 1000).astype(dt) if dt.kind == "f" else rng.integers(0, 10_000, n).astype(dt)
    nulls = bitmap_from_bools(rng.random(n) < 0.2)
    for nbytes in (8, 16, 24):
        for nulls_word in (False, True):
            for cn in (None, nulls):
                def call(cw, rw, keep):
                    r = Result(nbytes, rw, nulls_word, keep)
                    rc, _ = xcall(capi.XCALL_AGG(op, T), [r.vec, col_vec(col, n, cn, cw, keep)], n, raise_on_error=False)
                    return rc, r.bytes()
                rc, _ = run_forms(call)
                assert rc == 0


def test_q6_q1_mixed_forms_equal_host_form(gpu):
    n = 200_003
    cols = datagen.lineitem(10, 0, n)
    P = capi.Q6Params(*datagen.q6_params())
    pv = np.frombuffer(bytes(P), dtype=np.uint8).copy()

    def q6(cw, rw, keep):
        r = Result(16, rw, True, keep)
        rc, _ = xcall(capi.XCALL_Q6_FILTER_SUM, [r.vec] + [col_vec(cols[k], n, None, cw, keep) for k in Q6_NAMES] +
                      [Vector(data=pv, length=1, const=True)], n, raise_on_error=False)
        return rc, r.bytes()
    rc, (raw, rn) = run_forms(q6)
    assert rc == 0 and np.frombuffer(raw, dtype=np.int64)[1] > 0
    q1p = np.frombuffer(bytes(capi.Q1Params(datagen.Q1_CUTOFF, 0, 9)), dtype=np.uint8).copy()

    def q1(cw, rw, keep):
        r = Result(ops.Q1_RESULT_BYTES, rw, False, keep)
        rc, _ = xcall(capi.XCALL_Q1_GROUP_AGG, [r.vec] + [col_vec(cols[k], n, None, cw, keep) for k in Q1_NAMES] +
                      [Vector(data=q1p, length=1, const=True)], n, raise_on_error=False)
        return rc, r.bytes()
    rc, (raw, _) = run_forms(q1)
    assert rc == 0 and len(ops.q1_result_from_bytes(raw)) == 4


@pytest.mark.parametrize("shape", ["q6", "q1"])
def test_plan_shapes_mixed_forms_equal_host_form(gpu, shape):
    n = 150_001
    cols = datagen.lineitem(10, 0, n)
    p = ops.q6_plan() if shape == "q6" else ops.q1_plan(datagen.Q1_CUTOFF, row_base=3)
    names = Q6_NAMES if shape == "q6" else Q1_NAMES
    for max_groups in ((1, 4) if shape == "q6" else (4, 16)):
        nbytes = p.result_bytes(max_groups)

        def call(cw, rw, keep):
            r = Result(nbytes, rw, False, keep)
            vecs = [col_vec(np.ascontiguousarray(cols[k]).view(np.uint8).reshape(-1), n, None, cw, keep) for k in names]
            rc, _ = xcall(capi.XCALL_PLAN, [r.vec, ops._params_vec(p.P)] + vecs, n, raise_on_error=False)
            return rc, r.bytes()
        rc, (raw, _) = run_forms(call)
        assert rc == 0 and len(p.parse(raw)) == (1 if shape == "q6" else 4)


# ---- errors of the synchronous form
def agg_rc(op, T, col, cw, rw, keep):
    r = Result(24, rw, True, keep)
    rc, _ = xcall(capi.XCALL_AGG(op, T), [r.vec, col_vec(col, len(col), None, cw, keep)], len(col), raise_on_error=False)
    return rc, np.frombuffer(r.bytes()[0], dtype=np.uint64)


def test_sum_overflow_in_every_synchronous_form(gpu):
    signed = np.zeros(300_000, dtype=np.int64)
    signed[0] = np.iinfo(np.int64).max; signed[1] = 1; signed[2] = -5     # the total fits, the prefix at row 1 does not
    unsigned = np.full(2, 2 ** 63, dtype=np.uint64)
    for T, col in ((capi.T_INT64, signed), (capi.T_UINT64, unsigned)):
        for cw, rw in FORMS:
            keep = []
            rc, words = agg_rc(capi.AGG_SUM, T, col, cw, rw, keep)
            assert rc == capi.RC_OUT_OF_RANGE and int(words[2]) == capi.RC_OUT_OF_RANGE, (T, cw, rw)
            for b in keep:
                b.free()


def test_q1_nine_keys_in_every_form(gpu):
    n = 50_000
    cols = datagen.lineitem(10, 0, n)
    cols["returnflag"] = (65 + np.arange(n) % 9).astype(np.uint8)
    q1p = np.frombuffer(bytes(capi.Q1Params(datagen.Q1_CUTOFF, 0, 0)), dtype=np.uint8).copy()
    for cw, rw in FORMS + [("device", "device")]:
        keep = []
        r = Result(ops.Q1_RESULT_BYTES, rw, False, keep)
        rc, _ = xcall(capi.XCALL_Q1_GROUP_AGG, [r.vec] + [col_vec(cols[k], n, None, cw, keep) for k in Q1_NAMES] +
                      [Vector(data=q1p, length=1, const=True)], n, raise_on_error=False)
        if (cw, rw) == ("device", "device"):
            assert rc == 0 and capi.Q1Result.from_buffer_copy(r.bytes()[0]).ngroups == -1
        else:
            assert rc == capi.RC_INVALID_ARGUMENT, (cw, rw)
        for b in keep:
            b.free()


# ---- the asynchronous paths the benchmark times stay one launch each
def test_async_sum_and_resident_q6_cost_one_launch(gpu):
    n = 1_000_003
    col = DeviceBuffer.from_numpy(np.arange(n, dtype=np.int64))
    st = DeviceBuffer(24)
    ops.agg_state_device(capi.AGG_SUM, capi.T_INT64, col, None, n, st.ptr)       # warm: first-call set-up is not a launch either way
    l0 = gpu.MoB200_KernelLaunchCount()
    ops.agg_state_device(capi.AGG_SUM, capi.T_INT64, col, None, n, st.ptr)
    assert gpu.MoB200_KernelLaunchCount() - l0 == 1
    assert int(st.to_numpy(np.int64)[0]) == n * (n - 1) // 2
    cols = datagen.lineitem(10, 0, n)
    dev = {k: DeviceBuffer.from_numpy(cols[k]) for k in Q6_NAMES}
    out = DeviceBuffer(16)
    l0 = gpu.MoB200_KernelLaunchCount()
    ops.q6_filter_sum_device(*[dev[k] for k in Q6_NAMES], n, *datagen.q6_params(), out_ptr=out.ptr)
    assert gpu.MoB200_KernelLaunchCount() - l0 == 1
    assert int(out.to_numpy(np.int64)[1]) == ops.q6_filter_sum(*[cols[k] for k in Q6_NAMES], n, *datagen.q6_params())[1]
    for b in list(dev.values()) + [col, st, out]:
        b.free()
