"""Reference-facing operator calls over the C-ABI (what the Go side would do through cgo, written in Python).

Each function only marshals arguments into mo_xcall_args_t blocks (Vector.FillRawPtrLen layout) and calls XCall /
the mo.h entry points of libmo_b200.so.  Inputs may be numpy arrays (host path: the library stages them) or
DeviceBuffer objects (resident path).  Names follow the reference:

  q6_filter_sum / q1_group_agg     the fused TableScan->Filter->Projection->Group pipelines of TPC-H Q6 / Q1
  agg_sum / agg_count / agg_min / agg_max / agg_avg      aggexec sumAvgExec / countColumnExec / minMaxExecFixed (H0)
  BruteForceIndex                  brute_force.NewBruteForceIndex / .Search / .Destroy (brute_force.go:65-84,248-341)
  IvfflatSearchIndex               ivfflat.IvfflatSearchIndex.Search (ivfflat/search.go:509-630)
  topk_merge                       MergeTop / hnsw sub-index merge
"""
import ctypes as C

import numpy as np

from . import capi
from .vector import VARLENA_SZ, DeviceBuffer, Vector, bitmap_to_bools, varlena_bytes_column, xcall


def _vec(x, length=None, nulls=None, dtype=None):
    """one input column of a call -> Vector.  x: a numpy array (converted to dtype when one is given), a DeviceBuffer, a (cells, area) pair
    of either kind (area None: every value inline) or a list of bytes (a varlena column); nulls: bitmap words (numpy) or a DeviceBuffer.
    Its row count (the bits of its nulls) is length, else the host array's rows (a varlena column's cells)."""
    if isinstance(x, list):
        x = varlena_bytes_column(x)
    data, area = x if isinstance(x, tuple) else (x, None)
    if isinstance(data, DeviceBuffer):
        return Vector(data, nulls, area, length=length)
    if isinstance(x, tuple):
        data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        area = None if area is None else np.ascontiguousarray(area, dtype=np.uint8)
        rows = data.shape[0] // VARLENA_SZ
    else:
        data = np.ascontiguousarray(data, dtype)
        rows = data.shape[0]
    return Vector(data, nulls, area, length=rows if length is None else length)


def _params_vec(block):
    """a parameter block or scalar argument (a ctypes struct or a small numpy array) -> a one-row Vector over a copy of its bytes; a call
    that writes back into the block (err_row, area_len) is read from the Vector's data"""
    buf = np.frombuffer(bytes(block), dtype=np.uint8).copy()
    return Vector(data=buf, length=1, const=True)


# ------------------------------------------------------------------------------------------------ aggregates
def _agg(op, T, col, nulls, length, words=1):
    """MO_XCALL_AGG of one column into `words` result words: (rc, result, is_null)"""
    n = length if length is not None else (col.nbytes // np.dtype(capi.NP_OF_T[T]).itemsize if isinstance(col, DeviceBuffer) else len(col))
    res = np.zeros(words, dtype=np.uint64)
    rn = np.zeros(1, dtype=np.uint64)
    rc, msg = xcall(capi.XCALL_AGG(op, T), [Vector(data=res, nulls=rn, length=1), _vec(col, n, nulls)], n, raise_on_error=False)
    if rc not in (0, capi.RC_OUT_OF_RANGE):
        raise capi.MoError(rc, msg)
    return rc, res, bool(rn[0] & np.uint64(1))


def agg_sum(T, col, nulls=None, length=None):
    """SUM(col): returns (rc, value, is_null); value int64 / uint64 / float64 per SumReturnType (sumavg2.go:69-87)."""
    rc, res, isnull = _agg(capi.AGG_SUM, T, col, nulls, length)
    if T in (capi.T_FLOAT32, capi.T_FLOAT64):
        v = res.view(np.float64)[0]
    elif capi.T_UINT8 <= T <= capi.T_UINT64:
        v = int(res[0])
    else:
        v = int(res.view(np.int64)[0])
    return rc, v, isnull


def agg_avg(T, col, nulls=None, length=None):
    rc, res, isnull = _agg(capi.AGG_AVG, T, col, nulls, length)
    return rc, float(res.view(np.float64)[0]), isnull


def agg_count(T, col, nulls=None, length=None):
    rc, res, _ = _agg(capi.AGG_COUNT, T, col, nulls, length)
    return int(res.view(np.int64)[0])


def _minmax(op, T, col, nulls, length):
    rc, res, isnull = _agg(op, T, col, nulls, length)
    dt = np.dtype(capi.NP_OF_T[T])
    return res.view(np.uint8)[:dt.itemsize].view(dt)[0], isnull


def agg_min(T, col, nulls=None, length=None):
    return _minmax(capi.AGG_MIN, T, col, nulls, length)


def agg_max(T, col, nulls=None, length=None):
    return _minmax(capi.AGG_MAX, T, col, nulls, length)


# ------------------------------------------------------------------------------------------------ TPC-H shapes
def _scan_args(out, cols, n, params):
    """the arguments of the fused scans (Q6, Q6 over decimals, Q1): the result, the columns, the parameter block"""
    return [out] + [_vec(c, n) for c in cols] + [_params_vec(params)]


def q6_filter_sum(shipdate, discount, quantity, extendedprice, n, date_lo, date_hi, disc_lo, disc_hi, qty_hi):
    """SUM(l_extendedprice*l_discount) WHERE ... (q6.sql).  Returns (sum, qualifying_rows, is_null)."""
    res = np.zeros(2, dtype=np.float64)
    rn = np.zeros(1, dtype=np.uint64)
    xcall(capi.XCALL_Q6_FILTER_SUM, _scan_args(Vector(data=res, nulls=rn, length=1), (shipdate, discount, quantity, extendedprice), n,
                                               capi.Q6Params(date_lo, date_hi, disc_lo, disc_hi, qty_hi)), n)
    return float(res[0]), int(res.view(np.int64)[1]), bool(rn[0] & np.uint64(1))


Q6_RESULT_BYTES = 16
Q1_RESULT_BYTES = C.sizeof(capi.Q1Result)


def q6_filter_sum_device(shipdate, discount, quantity, extendedprice, n, date_lo, date_hi, disc_lo, disc_hi, qty_hi, out_ptr, out_nulls_ptr=None):
    """asynchronous form: resident columns, result {f64 sum, i64 rows} written to caller-owned DEVICE memory at out_ptr, nothing is
    read back and the calling thread's stream is not synchronised (the partial Group of a multi-GPU scan)"""
    rv = Vector(data_ptr=out_ptr, data_nbytes=Q6_RESULT_BYTES, nulls_ptr=out_nulls_ptr, length=1)
    xcall(capi.XCALL_Q6_FILTER_SUM, _scan_args(rv, (shipdate, discount, quantity, extendedprice), n,
                                               capi.Q6Params(date_lo, date_hi, disc_lo, disc_hi, qty_hi)), n)


def q6_merge_device(parts_ptr, nparts, out_ptr, out_nulls_ptr=None):
    """MergeGroup on the device: nparts x {f64 sum, i64 rows} -> one, in order"""
    xcall(capi.XCALL_Q6_MERGE, [Vector(data_ptr=out_ptr, data_nbytes=Q6_RESULT_BYTES, nulls_ptr=out_nulls_ptr, length=1),
                                Vector(data_ptr=parts_ptr, data_nbytes=Q6_RESULT_BYTES * nparts, length=nparts)], nparts)


def q6_merge(parts):
    """host form of the same merge: parts = [(sum, rows), ...] -> (sum, rows, is_null)"""
    buf = np.zeros(2 * len(parts), dtype=np.float64)
    for i, (s_, c_) in enumerate(parts):
        buf[2 * i] = s_
        buf.view(np.int64)[2 * i + 1] = c_
    res = np.zeros(2, dtype=np.float64)
    rn = np.zeros(1, dtype=np.uint64)
    xcall(capi.XCALL_Q6_MERGE, [Vector(data=res, nulls=rn, length=1), Vector(data=buf, length=len(parts))], len(parts))
    return float(res[0]), int(res.view(np.int64)[1]), bool(rn[0] & np.uint64(1))


Q6_DEC_RESULT_BYTES = C.sizeof(capi.Q6DecResult)


def q6_dec_result_from_bytes(raw, null_word=None):
    """mo_q6_dec_result_t bytes -> dict: revenue (Python int, unscaled at `scale`), scale, count, rc, err_row, is_null"""
    r = capi.Q6DecResult.from_buffer_copy(bytes(raw)[:Q6_DEC_RESULT_BYTES])
    rev = r.revenue_lo | (r.revenue_hi << 64)
    return {"revenue": rev - (1 << 128) if rev >> 127 else rev, "scale": r.scale, "count": r.count, "rc": r.rc, "err_row": r.err_row,
            "is_null": r.count == 0 if null_word is None else bool(int(null_word) & 1)}


def q6_dec_filter_sum(shipdate, discount, quantity, extendedprice, n, date_lo, date_hi, disc_lo, disc_hi, qty_hi, scale, row_base=0):
    """TPC-H Q6 over DECIMAL columns: shipdate int32 days, the three measures Decimal64 (int64 unscaled) at `scale` (0..4), the constants
    already unscaled at `scale`.  Returns the q6_dec_result_from_bytes dict; a Decimal128 Add overflow comes back as rc / err_row (the
    failing row + row_base)."""
    res = np.zeros(Q6_DEC_RESULT_BYTES, dtype=np.uint8)
    rn = np.zeros(1, dtype=np.uint64)
    rc, msg = xcall(capi.XCALL_Q6_DEC_FILTER_SUM, _scan_args(Vector(data=res, nulls=rn, length=1), (shipdate, discount, quantity, extendedprice), n,
                                                             capi.Q6DecParams(date_lo, date_hi, disc_lo, disc_hi, qty_hi, scale, 0, row_base)), n,
                    raise_on_error=False)
    if rc not in (0, capi.RC_INVALID_ARGUMENT):
        raise capi.MoError(rc, msg)
    out = q6_dec_result_from_bytes(res.tobytes(), rn[0])
    if rc and out["rc"] == 0:      # rejected before the scan (bad scale, nulls bitmap, short or misaligned column)
        raise capi.MoError(rc, msg)
    return out


def q6_dec_filter_sum_device(shipdate, discount, quantity, extendedprice, n, date_lo, date_hi, disc_lo, disc_hi, qty_hi, scale, out_ptr,
                             out_nulls_ptr=None, row_base=0):
    """asynchronous form: resident columns, mo_q6_dec_result_t written to DEVICE memory at out_ptr, nothing read back or synchronised"""
    rv = Vector(data_ptr=out_ptr, data_nbytes=Q6_DEC_RESULT_BYTES, nulls_ptr=out_nulls_ptr, length=1)
    xcall(capi.XCALL_Q6_DEC_FILTER_SUM, _scan_args(rv, (shipdate, discount, quantity, extendedprice), n,
                                                   capi.Q6DecParams(date_lo, date_hi, disc_lo, disc_hi, qty_hi, scale, 0, row_base)), n)


def q6_dec_merge(parts_bytes, nparts):
    """MergeGroup of nparts concatenated mo_q6_dec_result_t, in order -> the q6_dec_result_from_bytes dict"""
    buf = np.frombuffer(bytes(parts_bytes), dtype=np.uint8).copy()
    res = np.zeros(Q6_DEC_RESULT_BYTES, dtype=np.uint8)
    rn = np.zeros(1, dtype=np.uint64)
    rc, msg = xcall(capi.XCALL_Q6_DEC_MERGE, [Vector(data=res, nulls=rn, length=1), Vector(data=buf, length=nparts)], nparts,
                    raise_on_error=False)
    if rc not in (0, capi.RC_INVALID_ARGUMENT):
        raise capi.MoError(rc, msg)
    return q6_dec_result_from_bytes(res.tobytes(), rn[0])


def q6_dec_merge_device(parts_ptr, nparts, out_ptr, out_nulls_ptr=None):
    xcall(capi.XCALL_Q6_DEC_MERGE, [Vector(data_ptr=out_ptr, data_nbytes=Q6_DEC_RESULT_BYTES, nulls_ptr=out_nulls_ptr, length=1),
                                    Vector(data_ptr=parts_ptr, data_nbytes=Q6_DEC_RESULT_BYTES * nparts, length=nparts)], nparts)


def _q1_groups(r):
    out = []
    for g in range(r.ngroups):
        s = r.groups[g]
        out.append({k: getattr(s, k) for k in ("returnflag", "linestatus", "first_row", "sum_qty", "sum_base_price", "sum_disc_price",
                                               "sum_charge", "avg_qty", "avg_price", "avg_disc", "sum_disc", "count_order")})
    return out


def q1_result_from_bytes(raw):
    """mo_q1_result_t bytes -> list of group dicts (ngroups = -1: too many distinct keys)"""
    r = capi.Q1Result.from_buffer_copy(bytes(raw))
    if r.ngroups < 0:
        raise capi.MoError(capi.RC_INVALID_ARGUMENT, "q1: more than %d distinct group keys" % capi.Q1_MAX_GROUPS)
    return _q1_groups(r)


def q1_group_agg_device(shipdate, quantity, extendedprice, discount, tax, returnflag, linestatus, n, cutoff, out_ptr, row_base=0):
    """asynchronous form of q1_group_agg: mo_q1_result_t written to DEVICE memory at out_ptr; first_row values are offset by row_base"""
    xcall(capi.XCALL_Q1_GROUP_AGG, _scan_args(Vector(data_ptr=out_ptr, data_nbytes=Q1_RESULT_BYTES, length=1),
                                              (shipdate, quantity, extendedprice, discount, tax, returnflag, linestatus), n,
                                              capi.Q1Params(cutoff, 0, row_base)), n)


def q1_merge_device(parts_ptr, nparts, out_ptr):
    xcall(capi.XCALL_Q1_MERGE, [Vector(data_ptr=out_ptr, data_nbytes=Q1_RESULT_BYTES, length=1),
                                Vector(data_ptr=parts_ptr, data_nbytes=Q1_RESULT_BYTES * nparts, length=nparts)], nparts)


def q1_merge(parts_bytes, nparts):
    """host form: nparts concatenated mo_q1_result_t -> merged list of group dicts"""
    buf = np.frombuffer(bytes(parts_bytes), dtype=np.uint8).copy()
    res = np.zeros(Q1_RESULT_BYTES, dtype=np.uint8)
    xcall(capi.XCALL_Q1_MERGE, [Vector(data=res, length=1), Vector(data=buf, length=nparts)], nparts)
    return q1_result_from_bytes(res.tobytes())


def agg_state_device(op, T, col, nulls, n, out_ptr, out_nulls_ptr=None):
    """asynchronous MO_XCALL_AGG: mo_agg_state_t (24 bytes) written to DEVICE memory"""
    xcall(capi.XCALL_AGG(op, T), [Vector(data_ptr=out_ptr, data_nbytes=capi.AGG_STATE_BYTES, nulls_ptr=out_nulls_ptr, length=1),
                                  _vec(col, n, nulls)], n)


def agg_merge_device(op, T, parts_ptr, nparts, out_ptr, out_bytes=capi.AGG_STATE_BYTES, out_nulls_ptr=None):
    xcall(capi.XCALL_AGG_MERGE(op, T), [Vector(data_ptr=out_ptr, data_nbytes=out_bytes, nulls_ptr=out_nulls_ptr, length=1),
                                        Vector(data_ptr=parts_ptr, data_nbytes=capi.AGG_STATE_BYTES * nparts, length=nparts)], nparts)


def agg_state(op, T, col, nulls=None, length=None):
    """synchronous partial state (bits, count, rc) of one column"""
    return _agg(op, T, col, nulls, length, 3)[1]


def agg_merge(op, T, states, final=True):
    """MergeGroup of partial states (array [n, 3] uint64).  final=True: (rc, value bits as uint64, count, is_null); else the merged state"""
    st = np.ascontiguousarray(states, dtype=np.uint64).reshape(-1, 3)
    res = np.zeros(3 if not final else 2, dtype=np.uint64)
    rn = np.zeros(1, dtype=np.uint64)
    rc, msg = xcall(capi.XCALL_AGG_MERGE(op, T), [Vector(data=res, nulls=rn, length=1), Vector(data=st.reshape(-1), length=st.shape[0])], st.shape[0],
                    raise_on_error=False)
    if rc not in (0, capi.RC_OUT_OF_RANGE):
        raise capi.MoError(rc, msg)
    if not final:
        return res
    return rc, res[0], int(res[1]), bool(rn[0] & np.uint64(1))


def q1_group_agg(shipdate, quantity, extendedprice, discount, tax, returnflag, linestatus, n, cutoff, row_base=0):
    """TPC-H Q1 grouped aggregates (q1.sql).  returnflag/linestatus: packed uint8 columns or varlena cell buffers.
    Returns a list of dicts in first-seen group order."""
    res = np.zeros(Q1_RESULT_BYTES, dtype=np.uint8)
    xcall(capi.XCALL_Q1_GROUP_AGG, _scan_args(Vector(data=res, length=1), (shipdate, quantity, extendedprice, discount, tax, returnflag, linestatus),
                                              n, capi.Q1Params(cutoff, 0, row_base)), n)
    return _q1_groups(capi.Q1Result.from_buffer_copy(res.tobytes()))


# ------------------------------------------------------------------------------------------------ vector search
def _search_params(n, dim, nq, k, metric, nprobe=0, sqrt_out=0, nlist=0, key_base=0):
    return capi.SearchParams(n, dim, nq, k, metric, nprobe, sqrt_out, nlist, key_base)


def _filter_vec(filt):
    """the mo_search_filter_t argument of a filtered search.  filt: key bitmap words (numpy uint64, host) or a DeviceBuffer of them
    (bit `key` set = admitted), or a bloom filter handle (bloomfilter_t * from the library's bloomfilter_* symbols, as int / c_void_p)"""
    if isinstance(filt, DeviceBuffer):
        return _params_vec(capi.SearchFilter(capi.SEARCH_FILTER_KEY_BITMAP, 0, filt.ptr, filt.nbytes // 8))
    if isinstance(filt, np.ndarray):
        w = np.ascontiguousarray(filt, dtype=np.uint64).reshape(-1)
        v = _params_vec(capi.SearchFilter(capi.SEARCH_FILTER_KEY_BITMAP, 0, w.ctypes.data, w.size))
        v._keep.append(w)                       # the block holds the words' address
        return v
    if isinstance(filt, C.c_void_p):
        filt = filt.value
    if isinstance(filt, int):
        return _params_vec(capi.SearchFilter(capi.SEARCH_FILTER_KEY_BLOOM, 0, filt, 0))
    raise TypeError("filter: numpy uint64 key bitmap, DeviceBuffer key bitmap, or bloom filter handle")


def _queries(queries, dim):
    """(query Vector, nq): float32 rows, resident (DeviceBuffer) or host"""
    if isinstance(queries, DeviceBuffer):
        nq = queries.nbytes // (4 * dim)
        return _vec(queries, nq), nq
    q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, dim)
    return _vec(q.reshape(-1), q.shape[0]), q.shape[0]


def _search(fids, out, nq, limit, args, filter):
    """one top-k search call: fids = (unfiltered, filtered) XCall ids; the keys / distances go to out = (keys_ptr, distances_ptr), device
    memory the caller owns (returns None, None), or to host arrays that are returned"""
    if out is not None:
        keys = dists = None
        res = [Vector(data_ptr=p, data_nbytes=nq * limit * 8, length=nq) for p in out]
    else:
        keys = np.zeros(nq * limit, dtype=np.int64)
        dists = np.zeros(nq * limit, dtype=np.float64)
        res = [Vector(data=keys, length=nq), Vector(data=dists, length=nq)]
    extra = [] if filter is None else [_filter_vec(filter)]
    xcall(fids[filter is not None], res + args + extra, nq)
    return keys, dists


class BruteForceIndex:
    """brute_force.GoBruteForceIndex: NewBruteForceIndex(dataset, dim, metric) keeps the dataset RESIDENT in HBM
    (the reference keeps it in C-malloc memory, brute_force.go:104-123); Search returns (keys int64[nq*limit],
    distances float64[nq*limit]) row-major, ascending, keys = row ordinals (+ key_base)."""

    def __init__(self, dataset, dim, metric=capi.METRIC_L2, key_base=0, lib=None):
        self.lib = lib or capi.load_library()
        self.dim, self.metric, self.key_base = int(dim), int(metric), int(key_base)
        if isinstance(dataset, DeviceBuffer):
            self.buf, self.owned = dataset, False
            self.n = dataset.nbytes // (4 * self.dim)
        else:
            ds = np.ascontiguousarray(dataset, dtype=np.float32)
            self.n = ds.shape[0]
            self.buf, self.owned = DeviceBuffer.from_numpy(ds, self.lib), True
        self._prepare()

    def _prepare(self):
        # Load: split the resident rows into the tensor-core operand once (L2 metrics; a no-op where it does not apply)
        self.prepared = self.metric in (capi.METRIC_L2, capi.METRIC_L2SQ, capi.METRIC_IP, capi.METRIC_COS) and self.n > 0
        if self.prepared:
            capi.check(self.lib.MoB200_SearchPrepareMetric(self.buf.ptr, self.n, self.dim, self.metric), self.lib)

    def search(self, queries, limit, out_device=False, out=None, filter=None):
        """out = (keys_device_ptr, distances_device_ptr): results stay in caller-owned device memory (int64 / float64, nq*limit
        each) and nothing is returned -- the form a multi-GPU caller hands straight to NCCL.
        filter: search only the rows whose key (key_base + row) the filter admits (see _filter_vec)"""
        qv, nq = _queries(queries, self.dim)
        if limit == 0 or nq == 0:
            return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.float64)
        p = _search_params(self.n, self.dim, nq, limit, self.metric, key_base=self.key_base)
        keys, dists = _search((capi.XCALL_BRUTEFORCE_TOPK_F32, capi.XCALL_BRUTEFORCE_TOPK_FILTERED_F32), out, nq, limit,
                              [_vec(self.buf.view(self.n * self.dim * 4), self.n), qv, _params_vec(p)], filter)
        return None if out is not None else (keys, dists)

    def destroy(self):
        if self.buf is not None and getattr(self, "prepared", False):
            self.lib.MoB200_SearchRelease(self.buf.ptr)
        if self.owned and self.buf is not None:
            self.buf.free()
        self.buf = None


class IvfflatSearchIndex:
    """ivfflat.IvfflatSearchIndex: centroids + list-ordered entries resident in HBM.  build() takes the entry matrix
    and its list assignment (what the index tables hold) and lays the lists out contiguously."""

    def __init__(self, data, assign, centroids, metric=capi.METRIC_L2, lib=None):
        self.lib = lib or capi.load_library()
        centroids = np.ascontiguousarray(centroids, dtype=np.float32)
        self.nlist, self.dim = centroids.shape
        self.metric = int(metric)
        assign = np.asarray(assign)
        order = np.argsort(assign, kind="stable")   # stable: rows of a list stay in table order
        counts = np.bincount(assign, minlength=self.nlist)
        self.offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        self.row_ids = order.astype(np.int64)
        self.n = len(order)
        self.d_ids = DeviceBuffer.from_numpy(self.row_ids, self.lib)
        if isinstance(data, DeviceBuffer):          # resident entries: lay them out list by list on the device
            self.d_data = DeviceBuffer(4 * self.n * self.dim, self.lib)
            capi.check(self.lib.MoB200_GatherRowsF32(self.d_data.ptr, data.ptr, self.d_ids.ptr, self.n, self.dim), self.lib)
        else:
            data = np.ascontiguousarray(data, dtype=np.float32)
            self.d_data = DeviceBuffer.from_numpy(data[order], self.lib)
        self.d_cent = DeviceBuffer.from_numpy(centroids, self.lib)
        self.d_off = DeviceBuffer.from_numpy(self.offsets, self.lib)
        self.prepared = self.metric in (capi.METRIC_L2, capi.METRIC_L2SQ) and self.n > 0
        if self.prepared:   # LoadIndex: the list-ordered entries are split (as residuals against their centroid) once
            capi.check(self.lib.MoB200_SearchPrepareIvf(self.d_data.ptr, self.n, self.dim, self.d_cent.ptr, self.nlist, self.d_off.ptr), self.lib)

    @classmethod
    def build(cls, data_dev, n, centroids, metric=capi.METRIC_L2, lib=None, chunk=500_000):
        """index build on resident entries: centroid assignment = Productl2 (brute-force Search(limit=1) against the
        centroids, pkg/sql/colexec/productl2/product_l2.go:317-407) run chunk by chunk, then the list-ordered layout"""
        lib = lib or capi.load_library()
        centroids = np.ascontiguousarray(centroids, dtype=np.float32)
        dim = centroids.shape[1]
        cidx = BruteForceIndex(centroids, dim, metric, lib=lib)
        assign = np.empty(n, dtype=np.int32)
        for r0 in range(0, n, chunk):
            m = min(chunk, n - r0)
            view = DeviceBuffer.__new__(DeviceBuffer)
            view.lib, view.nbytes, view.ptr = lib, 4 * m * dim, data_dev.ptr + 4 * r0 * dim
            keys, _ = cidx.search(view, 1)
            view.ptr = None
            assign[r0:r0 + m] = keys
        cidx.destroy()
        return cls(data_dev, assign, centroids, metric, lib)

    @classmethod
    def build_list_shard(cls, gen_rows, n_total, centroids, rank, world, metric=capi.METRIC_L2, lib=None, chunk=500_000):
        """index build for ONE shard of a list-sharded index (BASELINE config 5: "lists sharded 8 x B200"): every row of the table is assigned to
        its nearest centroid (Productl2, product_l2.go:317-407) and this shard keeps the WHOLE lists l with l % world == rank; the centroid table is
        replicated, the other lists are empty here.  gen_rows(row0, m, device_ptr) materialises table rows [row0, row0 + m) in device memory.
        Row ids are the table's row numbers (primary keys)."""
        lib = lib or capi.load_library()
        centroids = np.ascontiguousarray(centroids, dtype=np.float32)
        dim = centroids.shape[1]
        cidx = BruteForceIndex(centroids, dim, metric, lib=lib)
        cap = n_total if world == 1 else int(n_total / world * 1.1) + chunk
        tmp = DeviceBuffer(4 * cap * dim, lib)
        scratch = DeviceBuffer(4 * min(chunk, n_total) * dim, lib)
        ids, lists, filled = [], [], 0
        for r0 in range(0, n_total, chunk):
            m = min(chunk, n_total - r0)
            gen_rows(r0, m, scratch.ptr)
            keys, _ = cidx.search(scratch.view(4 * m * dim), 1)
            mine = np.flatnonzero(keys % world == rank).astype(np.int64)
            if filled + mine.shape[0] > cap:
                raise capi.MoError(capi.RC_INTERNAL_ERROR, "list shard larger than expected")
            if mine.shape[0]:
                didx = DeviceBuffer.from_numpy(mine, lib)
                capi.check(lib.MoB200_GatherRowsF32(tmp.ptr + 4 * filled * dim, scratch.ptr, didx.ptr, mine.shape[0], dim), lib)
                didx.free()
            ids.append(mine + r0); lists.append(keys[mine].astype(np.int32)); filled += mine.shape[0]
        cidx.destroy(); scratch.free()
        gids = np.concatenate(ids) if ids else np.zeros(0, dtype=np.int64)
        ix = cls(tmp.view(4 * filled * dim), np.concatenate(lists) if lists else np.zeros(0, dtype=np.int32), centroids, metric, lib)
        tmp.free()
        ix.row_ids = gids[ix.row_ids]                  # list-ordered position -> table row number
        ix.d_ids.free(); ix.d_ids = DeviceBuffer.from_numpy(ix.row_ids, lib)
        return ix

    def search(self, queries, limit, nprobe, sqrt_out=False, out=None, filter=None):
        """filter: search only the entries whose primary key (row id) the filter admits, in the lists the unfiltered search probes"""
        qvec, nq = _queries(queries, self.dim)
        p = _search_params(self.n, self.dim, nq, limit, self.metric, nprobe=nprobe, sqrt_out=int(sqrt_out), nlist=self.nlist)
        return _search((capi.XCALL_IVF_TOPK_F32, capi.XCALL_IVF_TOPK_FILTERED_F32), out, nq, limit,
                       [_vec(self.d_data, self.n), qvec, _params_vec(p), _vec(self.d_cent, self.nlist),
                        _vec(self.d_off, self.nlist + 1), _vec(self.d_ids, self.n)], filter)

    def destroy(self):
        if self.prepared:
            self.lib.MoB200_SearchRelease(self.d_data.ptr)
        for b in (self.d_data, self.d_cent, self.d_off, self.d_ids):
            b.free()


def topk_merge_device(keys_ptr, dists_ptr, nshards, nq, k, out_keys_ptr, out_dists_ptr):
    """topk_merge on device-resident [nshards, nq, k] results (e.g. straight out of an NCCL all_gather); outputs stay on the device"""
    xcall(capi.XCALL_TOPK_MERGE, [Vector(data_ptr=out_keys_ptr, data_nbytes=nq * k * 8, length=nq), Vector(data_ptr=out_dists_ptr, data_nbytes=nq * k * 8, length=nq),
                                  Vector(data_ptr=keys_ptr, data_nbytes=nshards * nq * k * 8, length=nq),
                                  Vector(data_ptr=dists_ptr, data_nbytes=nshards * nq * k * 8, length=nq), _params_vec(_search_params(nshards, 0, nq, k, 0))], nq)


def topk_merge(keys_shards, dists_shards, nq, k):
    """merge [nshards, nq, k] per-shard results (final keys, float64 distances) into the global top-k."""
    ks = np.ascontiguousarray(keys_shards, dtype=np.int64).reshape(-1)
    ds = np.ascontiguousarray(dists_shards, dtype=np.float64).reshape(-1)
    keys = np.zeros(nq * k, dtype=np.int64)
    dists = np.zeros(nq * k, dtype=np.float64)
    xcall(capi.XCALL_TOPK_MERGE, [Vector(data=keys, length=nq), Vector(data=dists, length=nq), Vector(data=ks, length=nq),
                                  Vector(data=ds, length=nq), _params_vec(_search_params(ks.shape[0] // (nq * k), 0, nq, k, 0))], nq)
    return keys, dists


# ------------------------------------------------------------------------------------------------ column operators (csrc/colops.cu)
def filter_sels(bools, nulls=None, length=None):
    """Filter.Call inner loop (filter.go:116-152): ascending row numbers with (!null && true).  Host arrays in, numpy sels out."""
    b = np.ascontiguousarray(bools, dtype=np.uint8)
    n = length if length is not None else b.shape[0]
    sels = np.zeros(max(n, 1), dtype=np.int64)
    cnt = np.zeros(1, dtype=np.int64)
    xcall(capi.XCALL_FILTER_SELS, [Vector(data=sels, length=n), Vector(data=cnt, length=1), _vec(b, n, nulls)], n)
    return sels[:int(cnt[0])]


def filter_sels_device(bools_dev, nulls_dev, n, sels_ptr, count_ptr):
    """asynchronous form on resident vectors: sels (int64[n] capacity) and the count stay on the device"""
    xcall(capi.XCALL_FILTER_SELS, [Vector(data_ptr=sels_ptr, data_nbytes=8 * n, length=n), Vector(data_ptr=count_ptr, data_nbytes=8, length=1),
                                   _vec(bools_dev.view(n), n, nulls_dev)], n)


def shuffle(src, sels, src_nulls=None, want_nulls=False):
    """Vector.Shrink / Union (shuffle.FixedLengthShuffle + nulls.Filter): returns dst (and dst nulls words when want_nulls)"""
    a = np.ascontiguousarray(src)
    s = np.ascontiguousarray(sels, dtype=np.int64)
    m = s.shape[0]
    dst = np.zeros(m, dtype=a.dtype)
    dn = np.zeros((m + 63) // 64, dtype=np.uint64) if want_nulls else None
    sv = _vec(a, a.shape[0], src_nulls)
    xcall(capi.XCALL_SHUFFLE(a.dtype.itemsize), [Vector(data=dst.view(np.uint8).reshape(-1), nulls=dn, length=m), sv, Vector(data=s, length=m)], m)
    return (dst, dn) if want_nulls else dst


_T_OF_DTYPE = {np.dtype(np.bool_): capi.T_BOOL, np.dtype(np.int8): capi.T_INT8, np.dtype(np.int16): capi.T_INT16,
               np.dtype(np.int32): capi.T_INT32, np.dtype(np.int64): capi.T_INT64, np.dtype(np.uint8): capi.T_UINT8,
               np.dtype(np.uint16): capi.T_UINT16, np.dtype(np.uint32): capi.T_UINT32, np.dtype(np.uint64): capi.T_UINT64,
               np.dtype(np.float32): capi.T_FLOAT32, np.dtype(np.float64): capi.T_FLOAT64}


def _order_params(types, flags, limit, has_row_ids):
    if len(types) != len(flags):
        raise ValueError("one flag word per key")
    p = capi.OrderParams()
    p.nkeys, p.has_row_ids, p.limit = len(types), 1 if has_row_ids else 0, -1 if limit is None else int(limit)
    for k, (T, f) in enumerate(zip(types[:capi.ORDER_MAX_KEYS], flags)):
        p.key[k].col_type, p.key[k].flags = int(T), int(f)
    return p


def _key_type(c):
    """ORDER_SELS' default key type: VARCHAR for a varlena key, DECIMAL128 for uint64[n, 2], else the dtype's type"""
    if isinstance(c, (list, tuple)):
        return capi.T_VARCHAR
    c = np.asarray(c)
    return capi.T_DECIMAL128 if c.ndim == 2 else _T_OF_DTYPE.get(c.dtype)


def _order_args(sels, types, flags, limit, keys, row_ids):
    """ORDER_SELS' arguments: the sels result, the parameter block, one Vector per key, the optional row ids"""
    return [sels, _params_vec(_order_params(types, flags, limit, row_ids is not None))] + keys + ([] if row_ids is None else [row_ids])


def _order_rows(n, limit):
    return n if limit is None or limit < 0 or limit >= n else int(limit)


def order_sels(cols, nulls, flags, limit=None, row_ids=None, types=None, length=None):
    """Order / Top (order.go:103, top.go:445): the row permutation by the key columns, or its first `limit` rows; reorder payload columns
    with shuffle().  cols: numpy key columns (a 1-element array = const key; DECIMAL128 as uint64[n, 2] {lo, hi}); nulls: per key bitmap
    words or None; flags: per key ORDER_DESC | ORDER_NULLS_FIRST | ORDER_NULLS_LAST; types: MO_T_* per key (default: from the dtype, so
    DATE / DECIMAL64 and friends order as their storage type).  A varlena key (CHAR, VARCHAR, TEXT, BLOB ...; its type must be given, or
    VARCHAR is assumed) is a list of bytes or a (cells, area) pair of uint8 arrays in the vector layout (vector.varlena_bytes_column).
    row_ids (int64[n]): the merge form -- ties break by them.  Returns int64 sels."""
    keys = [_vec(c, nulls=nl) for c, nl in zip(cols, nulls if nulls is not None else [None] * len(cols))]
    types = list(types) if types is not None else [_key_type(c) for c in cols]
    n = length if length is not None else (len(row_ids) if row_ids is not None else max(k.length for k in keys))
    nout = _order_rows(n, limit)
    sels = np.zeros(max(nout, 1), dtype=np.int64)
    rv = None if row_ids is None else _vec(row_ids, n, dtype=np.int64)
    xcall(capi.XCALL_ORDER_SELS, _order_args(Vector(data=sels[:nout], length=nout), types, flags, limit, keys, rv), n)
    return sels[:nout]


def order_sels_device(cols, nulls, types, flags, n, sels_ptr, limit=None, row_ids=None):
    """asynchronous form on resident vectors (DeviceBuffer key columns, nulls and row ids): enqueues the order and returns; sels_ptr
    (device, int64[min(limit, n)]) holds the result once the calling thread's stream has run it.  A varlena key is a (cells, area)
    pair of DeviceBuffers (area None: every value inline); such a call reads back one small record first, so it synchronises once."""
    keys = [_vec(c, n, nl) for c, nl in zip(cols, nulls if nulls is not None else [None] * len(cols))]
    nout = _order_rows(n, limit)
    rv = None if row_ids is None else _vec(row_ids.view(8 * n), n)
    xcall(capi.XCALL_ORDER_SELS, _order_args(Vector(data_ptr=sels_ptr, data_nbytes=8 * nout, length=nout), types, flags, limit, keys, rv), n)


def pack_keys(cols, nulls=None, has_null=True, length=None):
    """fillKeys (inthashmap.go:92-183): <= 8 key bytes per row.  cols: list of fixed-width numpy columns (a 1-element array = const vector).
    Returns (keys uint64[n], skip bitmap words or None)"""
    n = length if length is not None else max(len(c) for c in cols)
    keys = np.zeros(n, dtype=np.uint64)
    skip = None if has_null else np.zeros((n + 63) // 64, dtype=np.uint64)
    vecs = [Vector(data=keys, nulls=skip, length=n), _params_vec(np.asarray([len(cols), 1 if has_null else 0], dtype=np.int32))]
    vecs += [_vec(c, n, None if nulls is None else nulls[i]) for i, c in enumerate(cols)]
    xcall(capi.XCALL_PACK_KEYS, vecs, n)
    return keys, skip


class GroupTable:
    """IntHashMap as the group operator sees it: insert(keys) -> 1-based group ids in first-seen order; the table persists across batches"""

    def __init__(self, capacity):
        self.keys = np.zeros(capacity, dtype=np.uint64)
        self.ngroups = np.zeros(1, dtype=np.int64)

    def insert(self, keys, skip=None):
        k = np.ascontiguousarray(keys, dtype=np.uint64)
        n = k.shape[0]
        groups = np.zeros(n, dtype=np.uint64)
        xcall(capi.XCALL_GROUP_IDS, [Vector(data=groups, length=n), Vector(data=self.ngroups, length=1), Vector(data=self.keys, length=self.keys.shape[0]),
                                     _vec(k, n, skip)], n)
        return groups

    def insert_device(self, keys_dev, n, groups_dev, d_ngroups, d_table_keys, capacity):
        """all vectors resident (DeviceBuffer); the group count is read back by the call (it sizes the next operator's state)"""
        xcall(capi.XCALL_GROUP_IDS, [Vector(groups_dev.view(8 * n), length=n), Vector(d_ngroups.view(8), length=1),
                                     Vector(d_table_keys.view(8 * capacity), length=capacity), _vec(keys_dev.view(8 * n), n)], n)


def _strkey_params(types, has_null):
    if not 1 <= len(types) <= capi.STRKEY_MAX_COLS:
        raise ValueError("1..%d key columns" % capi.STRKEY_MAX_COLS)
    p = capi.StrKeyParams()
    p.ncols, p.has_null = len(types), 1 if has_null else 0
    for k, T in enumerate(types):
        p.col_type[k] = int(T)
    return p


def _strkey_args(out, offsets, types, has_null, cols):
    """PACK_STR_KEYS' arguments: the key bytes, the offsets (and skip bitmap), the parameter block, one Vector per column"""
    return [out, offsets, _params_vec(_strkey_params(types, has_null))] + cols


def pack_str_keys(cols, types, nulls=None, has_null=True, length=None, capacity=None):
    """strHashmapIterator.encodeHashKeys (strhashmap.go:92-385): the byte-string key of every row.  cols: per key column a numpy array (fixed
    width; a 1-element array = const), or for a varlena type a list of bytes or a (cells, area) pair in the vector layout; types: MO_T_* per
    column; nulls: per column bitmap words or None.  Returns (key bytes uint8[], offsets uint64[n + 1], skip bitmap words or None): row i's key is
    bytes[off[i]:off[i + 1]]; skip (has_null=False) marks the rows that join no group."""
    data = [_vec(c, nulls=nl) for c, nl in zip(cols, nulls if nulls is not None else [None] * len(cols))]
    n = length if length is not None else max(d.length for d in data)
    off = np.zeros(n + 1, dtype=np.uint64)
    skip = None if has_null else np.zeros((n + 63) // 64, dtype=np.uint64)
    cap = capacity if capacity is not None else 16 * n
    while True:
        out = np.zeros(max(cap, 1), dtype=np.uint8)
        rc, msg = xcall(capi.XCALL_PACK_STR_KEYS, _strkey_args(Vector(data=out[:cap], length=cap), Vector(data=off, nulls=skip, length=n), types,
                                                               has_null, data), n, raise_on_error=False)
        if rc == capi.RC_OUT_OF_RANGE and capacity is None:       # off[n] holds the size needed
            cap = int(off[n])
            continue
        if rc:
            raise capi.MoError(rc, msg)
        return out[:int(off[n])], off, skip


def pack_str_keys_device(cols, nulls, types, n, bytes_dev, offsets_dev, skip_dev=None, has_null=True):
    """the form on resident vectors: cols are DeviceBuffers or, for varlena types, (cells, area) DeviceBuffer pairs (area None: every value
    inline); key bytes go to bytes_dev (its whole size is the capacity), offsets (uint64[n + 1]) to offsets_dev.  Reads back one record."""
    cv = [_vec(c, n, nl) for c, nl in zip(cols, nulls if nulls is not None else [None] * len(cols))]
    xcall(capi.XCALL_PACK_STR_KEYS, _strkey_args(Vector(bytes_dev, length=n), Vector(offsets_dev.view(8 * (n + 1)), skip_dev, length=n), types,
                                                 has_null, cv), n)


class StrGroupTable:
    """StrHashMap as the group operator sees it (the twin of GroupTable): insert(key bytes, offsets) -> 1-based group ids in first-seen order.
    Owns the table: bytes, offsets (group g is bytes[offsets[g - 1]:offsets[g]]) and ngroups, and grows them when a batch does not fit."""

    def __init__(self, capacity_groups=1024, capacity_bytes=1 << 16):
        self.bytes = np.zeros(max(capacity_bytes, 1), dtype=np.uint8)
        self.offsets = np.zeros(capacity_groups + 1, dtype=np.uint64)
        self.ngroups = np.zeros(1, dtype=np.int64)

    def _grow(self, groups, nbytes):
        g = int(self.ngroups[0])
        if groups + 1 > self.offsets.shape[0]:
            o = np.zeros(groups + 1, dtype=np.uint64); o[:g + 1] = self.offsets[:g + 1]; self.offsets = o
        if nbytes > self.bytes.shape[0]:
            b = np.zeros(nbytes, dtype=np.uint8); used = int(self.offsets[g]); b[:used] = self.bytes[:used]; self.bytes = b

    def insert(self, key_bytes, key_offsets, skip=None, first_rows=False):
        """groups uint64[n] (0 = skipped row), and with first_rows the batch row that created each new group, in id order"""
        kb = np.ascontiguousarray(key_bytes, dtype=np.uint8)
        ko = np.ascontiguousarray(key_offsets, dtype=np.uint64)
        n = ko.shape[0] - 1
        groups = np.zeros(n, dtype=np.uint64)
        fr = np.zeros(max(n, 1), dtype=np.int64) if first_rows else None
        before = int(self.ngroups[0])
        for attempt in range(2):
            vecs = [Vector(data=groups, length=n), Vector(data=self.ngroups, length=1), Vector(data=self.bytes, length=self.bytes.shape[0]),
                    Vector(data=self.offsets, length=self.offsets.shape[0]), Vector(data=kb, length=kb.shape[0]), _vec(ko, n, skip),
                    Vector(data=fr, length=n)]
            rc, msg = xcall(capi.XCALL_STR_GROUP_IDS, vecs, n, raise_on_error=False)
            if rc == capi.RC_INVALID_ARGUMENT and "capacity" in msg and attempt == 0:
                # at most n new groups and their bytes: this size always fits
                used = int(self.offsets[before])
                self._grow(max(2 * (self.offsets.shape[0] - 1), before + n), max(2 * self.bytes.shape[0], used + int(ko[n] - ko[0]) if n else used))
                continue
            if rc:
                raise capi.MoError(rc, msg)
            break
        if first_rows:
            return groups, fr[:int(self.ngroups[0]) - before]
        return groups

    def insert_device(self, bytes_dev, offsets_dev, n, groups_dev, d_ngroups, table_bytes_dev, table_offsets_dev, first_rows_dev=None, skip_dev=None):
        """every vector resident (DeviceBuffer; d_ngroups may be a host int64[1] array instead); the table is the caller's and does not grow"""
        vecs = [Vector(groups_dev.view(8 * n), length=n), Vector(d_ngroups if isinstance(d_ngroups, np.ndarray) else d_ngroups.view(8), length=1),
                Vector(table_bytes_dev, length=1), Vector(table_offsets_dev, length=1), Vector(bytes_dev, length=n),
                _vec(offsets_dev.view(8 * (n + 1)), n, skip_dev), Vector(None if first_rows_dev is None else first_rows_dev.view(8 * n), length=n)]
        xcall(capi.XCALL_STR_GROUP_IDS, vecs, n)

    def keys(self):
        g, o = int(self.ngroups[0]), self.offsets
        return [self.bytes[int(o[j]):int(o[j + 1])].tobytes() for j in range(g)]


def group_agg(op, T, state, state_nulls, counts, groups, col, col_nulls=None, length=None):
    """BatchFill of one aggregate into caller-owned state arrays (numpy, modified in place): state uint64/int64/float64[ngroups] (8-byte slots),
    state_nulls bitmap words (group is NULL), counts int64[ngroups] or None.  Returns rc (0 or RC_OUT_OF_RANGE)."""
    g = np.ascontiguousarray(groups, dtype=np.uint64)
    n = length if length is not None else g.shape[0]
    sv = Vector(data=state.view(np.uint8).reshape(-1), nulls=state_nulls, length=state.shape[0])
    cv = Vector(data=counts, length=state.shape[0])
    colv = _vec(col if col is not None else np.zeros(0, dtype=np.uint8), n, col_nulls)
    rc, msg = xcall(capi.XCALL_GROUP_AGG(op, T), [sv, cv, Vector(data=g, length=n), colv], n, raise_on_error=False)
    if rc not in (0, capi.RC_OUT_OF_RANGE):
        raise capi.MoError(rc, msg)
    return rc


# ------------------------------------------------------------------------------------------------ the generic fused operator (csrc/plan.cu)
class FusedPlan:
    """Builder for mo_plan_t: table_scan -> filter -> projection -> group in one kernel.

        p = FusedPlan([capi.T_DATE, capi.T_FLOAT64, capi.T_FLOAT64, capi.T_FLOAT64])          # column types
        p.where(0, ">=", lo).where(0, "<", hi).where(1, "between", a, b).where(2, "<", 24.0)
        revenue = p.mul(p.col(3), p.col(1))                                                 # value slots
        p.agg(capi.AGG_SUM, revenue)
        groups = p.run([shipdate, discount, quantity, price], n)
    """

    def __init__(self, col_types, has_null_keys=False, row_base=0):
        self.P = capi.Plan()
        self.P.ncols = len(col_types)
        for i, t in enumerate(col_types):
            self.P.col_type[i] = t
        self.P.has_null_keys = 1 if has_null_keys else 0
        self.P.row_base = row_base

    def where(self, col, op, lo, hi=0.0):
        q = self.P.pred[self.P.npreds]
        q.col, q.op, q.lo, q.hi = col, capi.PLAN_CMP[op], float(lo), float(hi)
        self.P.npreds += 1
        return self

    def _emit(self, op, a=0, b=0, imm=0.0):
        i = self.P.ninstr
        ins = self.P.instr[i]
        ins.op, ins.a, ins.b, ins.imm = op, a, b, float(imm)
        self.P.ninstr += 1
        return self.P.ncols + i

    def col(self, c):
        return c                      # a column IS value slot c

    def const(self, x):
        return self._emit(capi.PLAN_OP_CONST, imm=x)

    def add(self, a, b):
        return self._emit(capi.PLAN_OP_ADD, a, b)

    def sub(self, a, b):
        return self._emit(capi.PLAN_OP_SUB, a, b)

    def mul(self, a, b):
        return self._emit(capi.PLAN_OP_MUL, a, b)

    def div(self, a, b):
        return self._emit(capi.PLAN_OP_DIV, a, b)

    def group_by(self, *cols):
        for c in cols:
            self.P.key_col[self.P.nkeys] = c
            self.P.nkeys += 1
        return self

    def agg(self, kind, value=-1):
        a = self.P.agg[self.P.naggs]
        a.kind, a.value = kind, value
        self.P.naggs += 1
        return self

    def result_bytes(self, max_groups):
        return C.sizeof(capi.PlanHeader) + max_groups * (24 + 16 * self.P.naggs)

    def run(self, cols, n, nulls=None, max_groups=64, out_ptr=None):
        """cols: numpy arrays or DeviceBuffers (one per declared column); nulls: optional list of bitmap words (numpy / DeviceBuffer / None).
        out_ptr: device result buffer of result_bytes(max_groups) -> asynchronous form, returns None.  Else a list of group dicts
        {key, first_row, rows, aggs: [(value, count), ...]} in first-seen order."""
        vecs = [_vec(c, n, None if nulls is None else nulls[i]) for i, c in enumerate(cols)]
        nbytes = self.result_bytes(max_groups)
        res = np.zeros(nbytes, dtype=np.uint8) if out_ptr is None else None
        rv = Vector(data=res, length=1) if out_ptr is None else Vector(data_ptr=out_ptr, data_nbytes=nbytes, length=1)
        xcall(capi.XCALL_PLAN, [rv, _params_vec(self.P)] + vecs, n)
        return None if out_ptr is not None else self.parse(res.tobytes())

    def parse(self, raw):
        h = capi.PlanHeader.from_buffer_copy(raw[:C.sizeof(capi.PlanHeader)])
        if h.overflow:
            raise capi.MoError(capi.RC_INVALID_ARGUMENT, "plan: more groups than the result buffer holds")
        rec = 24 + 16 * self.P.naggs
        out = []
        for g in range(h.ngroups):
            b = raw[C.sizeof(capi.PlanHeader) + g * rec: C.sizeof(capi.PlanHeader) + (g + 1) * rec]
            key, first_row, rows = np.frombuffer(b[:8], dtype=np.uint64)[0], np.frombuffer(b[8:16], dtype=np.int64)[0], np.frombuffer(b[16:24], dtype=np.int64)[0]
            aggs = []
            for a in range(self.P.naggs):
                v = np.frombuffer(b[24 + 16 * a: 32 + 16 * a], dtype=np.float64)[0]
                c = np.frombuffer(b[32 + 16 * a: 40 + 16 * a], dtype=np.int64)[0]
                aggs.append((float(v), int(c)))
            out.append({"key": int(key), "first_row": int(first_row), "rows": int(rows), "aggs": aggs})
        if not h.sorted:
            out.sort(key=lambda g: g["first_row"])
        return out


def q6_plan():
    """TPC-H Q6 (q6.sql) as a FusedPlan over columns [shipdate DATE, discount f64, quantity f64, extendedprice f64]"""
    from . import datagen
    lo, hi, dlo, dhi, qhi = datagen.q6_params()
    p = FusedPlan([capi.T_DATE, capi.T_FLOAT64, capi.T_FLOAT64, capi.T_FLOAT64])
    p.where(0, ">=", lo).where(0, "<", hi).where(1, "between", dlo, dhi).where(2, "<", qhi)
    p.agg(capi.AGG_SUM, p.mul(p.col(3), p.col(1)))
    return p


def q1_plan(cutoff, row_base=0):
    """TPC-H Q1 (q1.sql) as a FusedPlan over columns [shipdate, quantity, extendedprice, discount, tax, returnflag u8, linestatus u8]"""
    p = FusedPlan([capi.T_DATE, capi.T_FLOAT64, capi.T_FLOAT64, capi.T_FLOAT64, capi.T_FLOAT64, capi.T_UINT8, capi.T_UINT8], row_base=row_base)
    p.where(0, "<=", cutoff)
    one = p.const(1.0)
    disc_price = p.mul(p.col(2), p.sub(one, p.col(3)))
    charge = p.mul(disc_price, p.add(one, p.col(4)))
    p.group_by(5, 6)
    for kind, v in ((capi.AGG_SUM, 1), (capi.AGG_SUM, 2), (capi.AGG_SUM, disc_price), (capi.AGG_SUM, charge), (capi.AGG_AVG, 1), (capi.AGG_AVG, 2), (capi.AGG_AVG, 3)):
        p.agg(kind, v)
    p.agg(capi.AGG_COUNT, -1)
    return p


# ------------------------------------------------------------------------------------------------ decimals (csrc/decimal.cu)
def dec_arith(op, width, a, b, scale1, scale2, n, n1=None, n2=None, rnulls=None):
    """d64/d128 Add (op 0) / Sub (1) / Mul (2).  a, b: int64 arrays (width 64) or uint64[n, 2] {lo, hi} arrays (width 128); a 1-row operand is a
    const vector.  Returns (rc, result, result nulls words, err_row); result is int64[n] (64-bit + -) or uint64[n, 2]."""
    out128 = op == 2 or width == 128
    r = np.zeros((n, 2), dtype=np.uint64) if out128 else np.zeros(n, dtype=np.int64)
    rn = _dec_result_nulls(n, rnulls)
    args = _dec_args(Vector(data=r.view(np.uint8).reshape(-1), nulls=rn, length=n), a, b, n, n1, n2, capi.DecParams(scale1, scale2, -1))
    rc, msg = xcall(capi.XCALL_DEC_ARITH(op, width), args, n, raise_on_error=False)
    if rc not in (0, capi.RC_INVALID_ARGUMENT):
        raise capi.MoError(rc, msg)
    return rc, r, rn, _err_row(args[3])


def _dec_args(out, a, b, n, n1, n2, params):
    """the arguments of a binary decimal call (DEC_ARITH, GO_COMPARE): the result, both operands (one element = const), the parameter block"""
    return [out, _vec(a, n, n1), _vec(b, n, n2), _params_vec(params)]


def _err_row(params):
    """the first failing row a decimal call writes back into its parameter block (-1: none)"""
    return int(params.data.view(np.int64)[1])


def dec_sum(width, col, sums, counts, groups=None, nulls=None, n=None):
    """SUM/AVG accumulation into sums uint64[ngroups, 2] (Decimal128) and counts int64[ngroups], in place"""
    c = np.ascontiguousarray(col)
    n = n if n is not None else (c.shape[0])
    gv = Vector(data=None if groups is None else np.ascontiguousarray(groups, dtype=np.uint64), length=n)
    xcall(capi.XCALL_DEC_SUM(width), [Vector(data=sums.view(np.uint8).reshape(-1), length=sums.shape[0]), Vector(data=counts, length=counts.shape[0]), gv,
                                      _vec(c, n, nulls)], n)


def _dec_result_nulls(n, rnulls):
    return np.zeros((n + 63) // 64, dtype=np.uint64) if rnulls is None else np.ascontiguousarray(rnulls, dtype=np.uint64).copy()


def _dec_compare_id(op, width):
    return capi.XCALL_GO_COMPARE(op, capi.T_DECIMAL64 if width == 64 else capi.T_DECIMAL128)


def dec_compare(op, width, a, b, scale1, scale2, n, n1=None, n2=None, rnulls=None):
    """a <op> b over DECIMAL64 (int64 arrays) or DECIMAL128 (uint64[n, 2] {lo, hi}) operands at scales scale1 / scale2 (valueDecimalCompare:
    the lower-scale side is scaled up, a failed scale-up compares unscaled).  A 1-row operand is const; rnulls: the result bitmap on entry
    (rows set there are skipped).  Returns (values uint8[n], result nulls words)."""
    r = np.zeros(n, dtype=np.uint8)
    rn = _dec_result_nulls(n, rnulls)
    xcall(_dec_compare_id(op, width), _dec_args(Vector(data=r, nulls=rn, length=n), a, b, n, n1, n2, capi.DecParams(scale1, scale2, -1)), n)
    return r, rn


def dec_compare_device(op, width, a, b, scale1, scale2, n, out_dev, out_nulls_dev, n1=None, n2=None):
    """dec_compare on resident operands (DeviceBuffers; one element's bytes = const) into out_dev (bool[n]) and out_nulls_dev (its bitmap,
    in/out): enqueue-only, nothing is read back or synchronised"""
    xcall(_dec_compare_id(op, width), _dec_args(Vector(out_dev.view(n), out_nulls_dev, length=n), a, b, n, n1, n2, capi.DecParams(scale1, scale2, -1)), n)


def _between_args(out, width, col, lo, hi, n, nulls):
    """GO_BETWEEN's arguments over a decimal column: the result, the column, the two bounds as one-element consts"""
    return [out, _vec(col, n, nulls), _params_vec(_dec_bound(width, lo)), _params_vec(_dec_bound(width, hi))]


def _dec_bound(width, v):
    v = int(v)
    if width == 64:
        return np.array([v], dtype=np.int64)
    return np.array([v & ((1 << 64) - 1), (v >> 64) & ((1 << 64) - 1)], dtype=np.uint64)


def dec_between(width, col, lo, hi, n, nulls=None):
    """col BETWEEN lo AND hi over a decimal column, the bounds (Python ints) already at the column's scale: a raw signed compare.  A NULL
    row gives false and a NULL result.  col may be a numpy array or a DeviceBuffer.  Returns (values uint8[n], result nulls words)."""
    r = np.zeros(n, dtype=np.uint8)
    rn = np.zeros((n + 63) // 64, dtype=np.uint64)
    xcall(capi.XCALL_GO_BETWEEN(capi.T_DECIMAL64 if width == 64 else capi.T_DECIMAL128),
          _between_args(Vector(data=r, nulls=rn, length=n), width, col, lo, hi, n, nulls), n)
    return r, rn


def dec_between_device(width, col, lo, hi, n, out_dev, out_nulls_dev, nulls=None):
    """dec_between on a resident column into resident outputs (out_nulls_dev zeroed by the caller)"""
    xcall(capi.XCALL_GO_BETWEEN(capi.T_DECIMAL64 if width == 64 else capi.T_DECIMAL128),
          _between_args(Vector(out_dev.view(n), out_nulls_dev, length=n), width, col, lo, hi, n, nulls), n)


def _dec_div(width, out, a, b, scale1, scale2, n, n1, n2, div0_error):
    """DEC_ARITH's Div: (rc, err_row, msg); rc 0, RC_INVALID_ARGUMENT or RC_DIVISION_BY_ZERO, any other code is raised"""
    args = _dec_args(out, a, b, n, n1, n2, capi.DecDivParams(scale1, scale2, -1, 1 if div0_error else 0, 0))
    rc, msg = xcall(capi.XCALL_DEC_ARITH(capi.DEC_OP_DIV, width), args, n, raise_on_error=False)
    if rc not in (0, capi.RC_INVALID_ARGUMENT, capi.RC_DIVISION_BY_ZERO):
        raise capi.MoError(rc, msg)
    return rc, _err_row(args[3]), msg


def dec_div(width, a, b, scale1, scale2, n, n1=None, n2=None, rnulls=None, div0_error=False):
    """a / b (d64Div / d128Div): the result is Decimal128 uint64[n, 2] at scale min(12, scale1 + 6) raised to at least scale1.  A zero divisor
    makes the row NULL, or fails the call with RC_DIVISION_BY_ZERO when div0_error.  Returns (rc, result, result nulls words, err_row, msg):
    rc is 0, RC_INVALID_ARGUMENT ("Decimal128 Div overflow") or RC_DIVISION_BY_ZERO, err_row the first failing row or -1."""
    r = np.zeros((n, 2), dtype=np.uint64)
    rn = _dec_result_nulls(n, rnulls)
    rc, err_row, msg = _dec_div(width, Vector(data=r.view(np.uint8).reshape(-1), nulls=rn, length=n), a, b, scale1, scale2, n, n1, n2, div0_error)
    return rc, r, rn, err_row, msg


def dec_div_device(width, a, b, scale1, scale2, n, out_dev, out_nulls_dev, n1=None, n2=None, div0_error=False):
    """dec_div on resident operands into resident outputs (out_nulls_dev in/out).  One read-back of the first failing row; returns
    (rc, err_row, msg)."""
    return _dec_div(width, Vector(out_dev.view(16 * n), out_nulls_dev, length=n), a, b, scale1, scale2, n, n1, n2, div0_error)


def _dec_avg_args(out, sums, counts, g, scale):
    return [out, _vec(sums, g), _vec(counts, g, dtype=np.int64), _params_vec(capi.DecParams(scale, 0, -1))]


def dec_avg(width, sums, counts, scale):
    """AVG's Flush over DEC_SUM's state (decAvg): sums uint64[g, 2], counts int64[g], scale = the argument's scale.  Returns (result
    uint64[g, 2] at scale max(12, scale) capped at scale + 6, result nulls words: count 0 is NULL)."""
    g = counts.shape[0]
    r = np.zeros((g, 2), dtype=np.uint64)
    rn = np.zeros((g + 63) // 64, dtype=np.uint64)
    xcall(capi.XCALL_DEC_AVG(width), _dec_avg_args(Vector(data=r.view(np.uint8).reshape(-1), nulls=rn, length=g), sums, counts, g, scale), g)
    return r, rn


def dec_avg_device(width, sums, counts, g, scale, out_dev, out_nulls_dev):
    """dec_avg on resident state (DeviceBuffers) into resident outputs: enqueue-only"""
    xcall(capi.XCALL_DEC_AVG(width), _dec_avg_args(Vector(out_dev.view(16 * g), out_nulls_dev, length=g), sums, counts, g, scale), g)


# ---------------------------------------------------------------------------------------------- normalize_l2 (vector-valued)
def normalize_l2(cells, area, length, dtype=np.float32, nulls=None):
    """normalize_l2(v) over a varlena vector column (moarray.NormalizeL2, pkg/vectorize/moarray/external.go:262-285).  Returns
    (result cells uint8[24 * length], result area uint8[len(area)]): the result mirrors the argument's layout."""
    cells = np.ascontiguousarray(cells, dtype=np.uint8)
    area = np.ascontiguousarray(area, dtype=np.uint8)
    ocells = np.zeros(24 * length, dtype=np.uint8)
    oarea = np.zeros(max(area.nbytes, 1), dtype=np.uint8)
    res = Vector(data=ocells, area=oarea, nulls=None if nulls is None else np.array(nulls, dtype=np.uint64, copy=True), length=length)
    fid = capi.XCALL_GO_NORMALIZE_L2_F32 if np.dtype(dtype) == np.float32 else capi.XCALL_GO_NORMALIZE_L2_F64
    xcall(fid, [res, _vec((cells, area), length)], length)
    return ocells, oarea[:area.nbytes]


# ---------------------------------------------------------------------------------------------- hash join (csrc/join.cu)
def _group_sels(groups, ngroups, nbuild):
    """JOIN_SELS: (offsets, sels) of the build rows by group, or (None, None) when GroupSels.Finalize keeps none (joinMapMsg.go:83-89): every
    group has one row, or nothing was inserted (every key NULL)"""
    if ngroups == nbuild:
        return None, None
    offsets = np.zeros(ngroups + 2, dtype=np.int32)
    sels = np.zeros(max(nbuild, 1), dtype=np.int32)
    cnt = np.zeros(1, dtype=np.int64)
    xcall(capi.XCALL_JOIN_SELS, [Vector(data=offsets, length=ngroups + 2), Vector(data=sels, length=nbuild), Vector(data=cnt, length=1),
                                 Vector(data=groups, length=nbuild)], nbuild)
    if int(cnt[0]) == 0:
        return None, None
    return offsets, sels[:int(cnt[0])]


def matched_bitmap(nbuild):
    """a zeroed matched-row bitmap for the right-flavoured join types: one bit per build row, LSB-first uint64 words"""
    return np.zeros((nbuild + 63) // 64, dtype=np.uint64)


def _matched_vec(matched, join_type):
    """args[8] of JOIN_PROBE / JOIN_PROBE_GIDS: the matched bitmap (numpy uint64 words, updated in place, or a DeviceBuffer) for types >= JOIN_RIGHT"""
    if join_type < capi.JOIN_RIGHT:
        return []
    if matched is None:
        raise ValueError("join type %d needs the matched bitmap" % join_type)
    if not isinstance(matched, DeviceBuffer) and not (isinstance(matched, np.ndarray) and matched.dtype == np.uint64 and matched.flags.c_contiguous):
        raise ValueError("the matched bitmap is updated in place: pass a contiguous numpy uint64 array")
    return [Vector(data=matched, length=1)]


def _join_type(join_type):
    return _params_vec(np.array([join_type, 0], dtype=np.int32))


def _ngroups(ngroups):
    return _params_vec(np.array([ngroups], np.int64))


def _probe_args(outs, join_type, args, matched):
    """the arguments of JOIN_PROBE, JOIN_PROBE_GIDS and JOIN_COND: probe rows, build rows, count, join type, the call's own, the matched bitmap"""
    return outs + [_join_type(join_type)] + args + _matched_vec(matched, join_type)


def _probe_with(fid, join_type, args, matched, n, length, capacity):
    """the JOIN_PROBE capacity protocol on host results: a too-small buffer reports the count and the call is repeated"""
    cap = capacity if capacity is not None else max(2 * n, 1024)
    while True:
        op, ob, cnt = np.zeros(cap, np.int64), np.zeros(cap, np.int64), np.zeros(1, np.int64)
        outs = [Vector(data=op, length=cap), Vector(data=ob, length=cap), Vector(data=cnt, length=1)]
        rc, msg = xcall(fid, _probe_args(outs, join_type, args, matched), length, raise_on_error=False)
        if rc == capi.RC_OUT_OF_RANGE and capacity is None:
            cap = int(cnt[0])
            continue
        if rc:
            raise capi.MoError(rc, msg)
        return op[:int(cnt[0])], ob[:int(cnt[0])]


def _probe_gids_args(ngroups, offsets, sels, vals):
    """JOIN_PROBE_GIDS' own arguments: the group count, the GroupSels (None: unique map), the group ids"""
    return [_ngroups(ngroups), Vector(data=offsets, length=ngroups + 2), Vector(data=sels, length=1), vals]


def _str_find_args(vals, ngroups, table_bytes, table_offsets, key_bytes, key_offsets, nulls, n):
    """STR_JOIN_FIND's arguments: the ids, the table (group count, bytes, offsets), the probe keys' bytes and offsets with their nulls"""
    return [Vector(data=vals, length=n), _ngroups(ngroups), Vector(data=table_bytes, length=1), Vector(data=table_offsets, length=1),
            Vector(data=key_bytes, length=n), _vec(key_offsets, n, nulls)]


class StrJoinMap:
    """message.JoinMap over byte-string keys (the twin of JoinMap; HashmapBuilder with varlena or wide keys, hashbuild/hashmap.go:110-116,258-275):
    the build side's StrHashMap (StrGroupTable) and its GroupSels.  Keys are PACK_STR_KEYS bytes + offsets; probe = STR_JOIN_FIND + JOIN_PROBE_GIDS."""

    def __init__(self, build_bytes, build_offsets, skip=None, prepare=True):
        ko = np.ascontiguousarray(build_offsets, dtype=np.uint64)
        self.nbuild = ko.shape[0] - 1
        tab = StrGroupTable(max(self.nbuild, 1), max(int(ko[-1] - ko[0]), 1))
        groups = tab.insert(build_bytes, ko, skip)
        self.ngroups = int(tab.ngroups[0])
        self.table_offsets = tab.offsets[:self.ngroups + 1].copy()
        self.table_bytes = tab.bytes[:int(self.table_offsets[-1])].copy()
        self.offsets, self.sels = _group_sels(groups, self.ngroups, self.nbuild)
        self.prepared = False
        if prepare and self.ngroups:
            lib = capi.load_library()
            capi.check(lib.MoB200_StrJoinMapPrepare(self.table_bytes.ctypes.data, self.table_offsets.ctypes.data, self.ngroups), lib)
            self.prepared = True

    def hash_on_unique(self):
        return self.offsets is None

    def find(self, key_bytes, key_offsets, nulls=None):
        """strHashmapIterator.Find: 1-based group id per probe key, 0 = no match"""
        ko = np.ascontiguousarray(key_offsets, dtype=np.uint64)
        n = ko.shape[0] - 1
        vals = np.zeros(n, dtype=np.uint64)
        kb = np.ascontiguousarray(key_bytes, dtype=np.uint8)
        xcall(capi.XCALL_STR_JOIN_FIND, _str_find_args(vals, self.ngroups, self.table_bytes, self.table_offsets, kb, ko, nulls, n), n)
        return vals

    def probe(self, key_bytes, key_offsets, join_type=capi.JOIN_INNER, nulls=None, capacity=None, matched=None):
        """(probe rows, build rows) of the join result in the reference's emission order, as JoinMap.probe"""
        return probe_gids(self.find(key_bytes, key_offsets, nulls), self.ngroups, self.offsets, self.sels, join_type, capacity, matched)

    def release(self):
        if self.prepared:
            lib = capi.load_library()
            lib.MoB200_JoinMapRelease(self.table_offsets.ctypes.data)
            self.prepared = False


def str_join_find_device(vals_dev, n, ngroups, table_bytes_dev, table_offsets_dev, bytes_dev, offsets_dev, nulls_dev=None):
    """STR_JOIN_FIND on resident vectors (DeviceBuffers): enqueues the lookup of n probe keys (bytes_dev, offsets_dev uint64[n + 1]) in a table
    STR_GROUP_IDS built (ngroups is a host int); vals_dev (uint64[n]) holds the ids once the calling thread's stream has run it"""
    xcall(capi.XCALL_STR_JOIN_FIND, _str_find_args(vals_dev.view(8 * n), ngroups, table_bytes_dev, table_offsets_dev.view(8 * (ngroups + 1)), bytes_dev,
                                                   offsets_dev.view(8 * (n + 1)), nulls_dev, n), n)


def probe_gids_device(vals_dev, n, ngroups, offsets_dev, sels_dev, join_type, out_probe_dev, out_build_dev, count_dev, matched_dev=None):
    """JOIN_PROBE_GIDS on resident vectors: the pairs go to out_probe_dev / out_build_dev (int64, their size is the capacity) and their count to
    count_dev; offsets_dev / sels_dev None = unique map; matched_dev = the matched bitmap (DeviceBuffer) of a right-flavoured type.  Reads the count
    back (RC_OUT_OF_RANGE: the buffers are too small, the count is written)."""
    outs = [Vector(data=out_probe_dev, length=1), Vector(data=out_build_dev, length=1), Vector(data=count_dev.view(8), length=1)]
    args = _probe_gids_args(ngroups, offsets_dev, sels_dev, Vector(data=vals_dev.view(8 * n), length=n))
    xcall(capi.XCALL_JOIN_PROBE_GIDS, _probe_args(outs, join_type, args, matched_dev), n)


def probe_gids(vals, ngroups, offsets, sels, join_type=capi.JOIN_INNER, capacity=None, matched=None):
    """JOIN_PROBE_GIDS: the JOIN_PROBE emission over given group ids (JOIN_FIND's or STR_JOIN_FIND's vals); offsets / sels None = unique map;
    matched = the matched bitmap of a right-flavoured type (matched_bitmap(nbuild), updated in place)"""
    v = np.ascontiguousarray(vals, dtype=np.uint64)
    n = v.shape[0]
    return _probe_with(capi.XCALL_JOIN_PROBE_GIDS, join_type, _probe_gids_args(ngroups, offsets, sels, Vector(data=v, length=n)), matched, n, n, capacity)


class JoinMap:
    """message.JoinMap for equality joins over <= 8-byte packed keys (pkg/vm/message/joinMapMsg.go:127-210): the build side's IntHashMap
    (GroupTable: first-seen group ids + key table) and its GroupSels.  HashOnUnique (every build row its own group) keeps no sels."""

    def __init__(self, build_keys, skip=None, prepare=True):
        k = np.ascontiguousarray(build_keys, dtype=np.uint64)
        self.nbuild = k.shape[0]
        tab = GroupTable(max(self.nbuild, 1))
        groups = tab.insert(k, skip)                                   # HashmapBuilder.BuildHashmap: itr.Insert (hashmap.go:340-360)
        self.ngroups = int(tab.ngroups[0])
        self.table_keys = np.ascontiguousarray(tab.keys[:max(self.ngroups, 1)])[:self.ngroups].copy() if self.ngroups else np.zeros(0, np.uint64)
        self.offsets, self.sels = _group_sels(groups, self.ngroups, self.nbuild)
        self.prepared = False
        if prepare and self.ngroups:
            lib = capi.load_library()
            capi.check(lib.MoB200_JoinMapPrepare(self.table_keys.ctypes.data, self.ngroups), lib)
            self.prepared = True

    def hash_on_unique(self):
        return self.offsets is None

    def find(self, keys, nulls=None):
        """intHashMapIterator.Find: 1-based group id per probe key, 0 = no match"""
        k = np.ascontiguousarray(keys, dtype=np.uint64)
        n = k.shape[0]
        vals = np.zeros(n, dtype=np.uint64)
        xcall(capi.XCALL_JOIN_FIND, [Vector(data=vals, length=n), Vector(data=self.table_keys, length=self.ngroups), Vector(data=k, nulls=nulls, length=n)], n)
        return vals

    def probe(self, keys, join_type=capi.JOIN_INNER, nulls=None, capacity=None, matched=None):
        """(probe rows, build rows) of the join result in the reference's emission order; build row -1 = no build side (left outer / semi / anti /
        full / single).  The right-flavoured types (JOIN_RIGHT and above) mark `matched` (matched_bitmap(nbuild), shared by every probe batch of
        one join); join_build_rows then gives the build rows they add."""
        k = np.ascontiguousarray(keys, dtype=np.uint64)
        n = k.shape[0]
        args = [Vector(data=self.table_keys, length=self.ngroups), Vector(data=self.offsets, length=self.ngroups + 2), Vector(data=self.sels, length=1),
                _vec(k, n, nulls)]
        return _probe_with(capi.XCALL_JOIN_PROBE, join_type, args, matched, n, n, capacity)

    def release(self):
        if self.prepared:
            lib = capi.load_library()
            lib.MoB200_JoinMapRelease(self.table_keys.ctypes.data)
            self.prepared = False


def join_build_rows(matched, nbuild, join_type):
    """hashjoin finalize (join.go:682-727): the build rows a right-flavoured join adds once every probe batch has marked `matched` -- the
    unmatched ones, or for JOIN_RIGHT_SEMI the matched ones -- ascending; their probe-side columns are NULL (SHUFFLE with sel -1)"""
    m = np.ascontiguousarray(matched, dtype=np.uint64)
    sels = np.zeros(max(nbuild, 1), dtype=np.int64)
    cnt = np.zeros(1, dtype=np.int64)
    xcall(capi.XCALL_JOIN_BUILD_ROWS, [Vector(data=sels, length=nbuild), Vector(data=cnt, length=1), Vector(data=m, length=1), _join_type(join_type)], nbuild)
    return sels[:int(cnt[0])]


def join_build_rows_device(matched_dev, nbuild, join_type, sels_ptr, count_ptr):
    """JOIN_BUILD_ROWS on a resident bitmap: sels (int64[nbuild] capacity) and the count stay on the device; the call only enqueues work"""
    xcall(capi.XCALL_JOIN_BUILD_ROWS, [Vector(data_ptr=sels_ptr, data_nbytes=8 * nbuild, length=nbuild), Vector(data_ptr=count_ptr, data_nbytes=8, length=1),
                                       Vector(data=matched_dev.view(8 * ((nbuild + 63) // 64)), length=1), _join_type(join_type)], nbuild)


def _merge_vecs(out, inputs, join_type):
    return [out, _params_vec(np.array([len(inputs)], np.int32)), _join_type(join_type)] + inputs


def join_matched_merge(bitmaps, nbuild, join_type):
    """syncBitmap (join.go:650-676): the OR of the workers' matched bitmaps; JOIN_RIGHT_SINGLE fails (MoError) when a build row is set in two"""
    words = (nbuild + 63) // 64
    out = np.zeros(words, dtype=np.uint64)
    ins = [Vector(data=np.ascontiguousarray(b, dtype=np.uint64), length=words) for b in bitmaps]
    xcall(capi.XCALL_JOIN_MATCHED_MERGE, _merge_vecs(Vector(data=out, length=words), ins, join_type), nbuild)
    return out


def join_matched_merge_device(out_dev, bitmaps_dev, nbuild, join_type):
    """JOIN_MATCHED_MERGE over resident bitmaps (DeviceBuffers; out_dev may be one of them): enqueue only, except JOIN_RIGHT_SINGLE, which reads
    back whether a row is set in two inputs"""
    words = (nbuild + 63) // 64
    ins = [Vector(data=b.view(8 * words), length=1) for b in bitmaps_dev]
    xcall(capi.XCALL_JOIN_MATCHED_MERGE, _merge_vecs(Vector(data=out_dev.view(8 * words), length=1), ins, join_type), nbuild)


def _cond_args(cand_probe, cand_build, cond, cond_nulls, npairs):
    """JOIN_COND's own arguments: the candidate pairs and their condition"""
    return [_vec(cand_probe, npairs), _vec(cand_build, npairs), _vec(cond, npairs, cond_nulls)]


def join_cond(cand_probe, cand_build, cond, nprobe, join_type, cond_nulls=None, capacity=None, matched=None):
    """JOIN_COND: a join with a non-equality condition (NonEqCond, join.go:468-498,570-611) over one probe batch of nprobe rows.  cand_probe /
    cand_build are the batch's JOIN_INNER pairs (JoinMap.probe, StrJoinMap.probe or probe_gids), cond the condition evaluated over them (one
    bool per pair, cond_nulls its null bitmap words; NULL never passes).  Returns (probe rows, build rows) in the reference's order, as
    JoinMap.probe does for join_type; `matched` as there."""
    cp = np.ascontiguousarray(cand_probe, dtype=np.int64)
    cb = np.ascontiguousarray(cand_build, dtype=np.int64)
    c = np.ascontiguousarray(cond, dtype=np.bool_).view(np.uint8)
    npairs = cp.shape[0]
    # the result has at most npairs + nprobe rows: one call
    return _probe_with(capi.XCALL_JOIN_COND, join_type, _cond_args(cp, cb, c, cond_nulls, npairs), matched, max(npairs, nprobe), nprobe, capacity)


def join_cond_device(cand_probe_dev, cand_build_dev, cond_dev, cond_nulls_dev, npairs, nprobe, join_type, out_probe_dev, out_build_dev, count_dev,
                     matched_dev=None):
    """JOIN_COND on resident vectors (DeviceBuffers), the twin of probe_gids_device: npairs candidate pairs and their condition (cond_nulls_dev
    None = no NULLs); the result goes to out_probe_dev / out_build_dev (int64, their size is the capacity) and its count to count_dev.  Reads the
    count back (RC_OUT_OF_RANGE: the buffers are too small, the count is written)."""
    outs = [Vector(data=out_probe_dev, length=1), Vector(data=out_build_dev, length=1), Vector(data=count_dev.view(8), length=1)]
    args = _cond_args(cand_probe_dev.view(8 * npairs), cand_build_dev.view(8 * npairs), cond_dev.view(npairs), cond_nulls_dev, npairs)
    xcall(capi.XCALL_JOIN_COND, _probe_args(outs, join_type, args, matched_dev), nprobe)


# ---------------------------------------------------------------------------------------------- Elkan k-means (csrc/kmeans.cu)
def kmeans_elkan(vectors, init_centroids, max_iter=500, rnd=None):
    """ElkanClusterer.Cluster (pkg/vectorindex/ivfflat/kmeans/elkans/clusterer.go:330-392), dense variant.  init_centroids: an array [k, dim],
    or an int k = kmeans.Random initialisation (Random.InitCentroids with Go's PCG, gorand.py) and the matching empty-cluster stream.
    Returns (centroids [k, dim], assignments int64[n], iterations)."""
    v = np.ascontiguousarray(vectors)
    assert v.dtype in (np.float32, np.float64)
    n, dim = v.shape
    if isinstance(init_centroids, (int, np.integer)):
        from . import gorand
        k = int(init_centroids)
        if n == k:                                    # Cluster(): vectorCnt == clusterCnt returns the vectors themselves (clusterer.go:337-339)
            return v.copy(), np.arange(n, dtype=np.int64), 0
        init_centroids = v[gorand.random_init_rows(n, k)]
        if rnd is None:
            rnd = np.array(gorand.empty_cluster_stream(min(dim * k * 4, 1 << 20)), dtype=np.float32)
    cent = np.ascontiguousarray(init_centroids, dtype=v.dtype).copy()
    k = cent.shape[0]
    assign = np.zeros(n, dtype=np.int64); iters = np.zeros(1, dtype=np.int64)
    vecs = [Vector(data=cent.reshape(-1), length=k * dim), Vector(data=assign, length=n), Vector(data=iters, length=1),
            _params_vec(np.array([n, dim, k, max_iter], dtype=np.int64)),
            Vector(data=v.reshape(-1), length=n * dim),
            Vector(data=np.ascontiguousarray(rnd, dtype=np.float32), length=len(rnd)) if rnd is not None and len(rnd) else Vector(length=0)]
    xcall(capi.XCALL_KMEANS_ELKAN_F32 if v.dtype == np.float32 else capi.XCALL_KMEANS_ELKAN_F64, vecs, n)
    return cent, assign, int(iters[0])


# ---------------------------------------------------------------------------------------------- LZ4 block decode (csrc/lz4.cu)
def lz4_decode_blocks(blocks, sizes):
    """compress.Decompress over many column blocks in one call: blocks = list of compressed byte strings, sizes = their decoded sizes.
    Returns the list of decoded byte strings."""
    src = np.frombuffer(b"".join(blocks), dtype=np.uint8) if blocks else np.zeros(0, np.uint8)
    n = len(blocks)
    desc = np.zeros((n, 4), dtype=np.int64)
    so = do = 0
    for i, (b, s) in enumerate(zip(blocks, sizes)):
        desc[i] = (so, len(b), do, s)
        so += len(b); do += s
    dst = np.zeros(max(do, 1), dtype=np.uint8)
    xcall(capi.XCALL_LZ4_DECODE, [Vector(data=dst, length=do), Vector(data=src if src.size else np.zeros(1, np.uint8), length=so), Vector(data=desc.reshape(-1), length=4 * n)], n)
    return [dst[desc[i, 2]:desc[i, 2] + desc[i, 3]].tobytes() for i in range(n)]


# ---------------------------------------------------------------------------------------------- marshalled vector -> resident vector (csrc/vecdecode.cu)
class VectorView(C.Structure):
    _fields_ = [("vclass", C.c_int32), ("oid", C.c_int32), ("size", C.c_int32), ("width", C.c_int32), ("scale", C.c_int32), ("length", C.c_uint32),
                ("data_len", C.c_uint64), ("area_len", C.c_uint64), ("null_count", C.c_int64), ("nulls_words", C.c_uint64), ("sorted", C.c_int32), ("bad", C.c_int32)]


def vector_unmarshal_device(src_dev, nbytes, data_dev, area_dev, nulls_dev):
    """Vector.UnmarshalBinary on the device: src_dev holds the marshalled bytes (e.g. straight out of lz4 decode), the sections are copied to the
    aligned DeviceBuffers given.  Returns the VectorView."""
    view = np.zeros(C.sizeof(VectorView), dtype=np.uint8)
    vecs = [Vector(data=view, length=1), Vector(data=data_dev, length=1), Vector(data=area_dev, length=1), Vector(data=nulls_dev, length=1),
            Vector(data=src_dev.view(nbytes), length=1)]
    xcall(capi.XCALL_VECTOR_UNMARSHAL, vecs, 1)
    return VectorView.from_buffer_copy(view.tobytes())


# ------------------------------------------------------------------------------------------------ string predicates (csrc/strpred.cu)
def _str_pred(fid, a, b, a_nulls, b_nulls, rnulls, length):
    va, vb = _vec(a, nulls=a_nulls), _vec(b, nulls=b_nulls)
    n = length if length is not None else max(va.length, vb.length)
    r = np.zeros(max(n, 1), dtype=np.uint8)
    rn = np.zeros(max((n + 63) // 64, 1), dtype=np.uint64) if rnulls is None else np.array(rnulls, dtype=np.uint64)
    xcall(fid, [Vector(data=r[:n], nulls=rn, length=n), va, vb], n)
    return r[:n].astype(bool), bitmap_to_bools(rn, n)


def str_compare(op, T, a, b, a_nulls=None, b_nulls=None, rnulls=None, length=None):
    """a <op> b over varlena operands (T = capi.T_CHAR / T_VARCHAR / T_TEXT / ...): = and != are bytes.Equal, the orderings bytes.Compare.
    a, b: a list of bytes (one element = const) or a (cells, area) pair; *_nulls: bitmap words; rnulls: the result bitmap on entry (rows set
    there are skipped).  Returns (values bool[n], nulls bool[n])."""
    return _str_pred(capi.XCALL_GO_COMPARE(op, T), a, b, a_nulls, b_nulls, rnulls, length)


def like(col, pattern, col_nulls=None, pattern_nulls=None, rnulls=None, length=None):
    """col LIKE pattern (likeFn): pattern is bytes (a const pattern), a list of bytes or a (cells, area) pair.  NOT LIKE is the negation of
    the values with the same nulls.  Returns (values bool[n], nulls bool[n])."""
    if isinstance(pattern, (bytes, bytearray)):
        pattern = [bytes(pattern)]
    return _str_pred(capi.XCALL_GO_LIKE, col, pattern, col_nulls, pattern_nulls, rnulls, length)


def _str_pred_device(fid, a, b, n, out_dev, out_nulls_dev, a_nulls, b_nulls):
    xcall(fid, [Vector(data=out_dev.view(n), nulls=out_nulls_dev, length=n), _vec(a, n, a_nulls), _vec(b, n, b_nulls)], n)


def str_compare_device(op, T, a, b, n, out_dev, out_nulls_dev, a_nulls=None, b_nulls=None):
    """the form on resident vectors: a, b are (cells, area) DeviceBuffer pairs (area None: every value inline; 24 bytes of cells = const);
    out_dev (bool[n]) and out_nulls_dev (its bitmap, in/out) are DeviceBuffers.  Enqueues one kernel and reads back one status record."""
    _str_pred_device(capi.XCALL_GO_COMPARE(op, T), a, b, n, out_dev, out_nulls_dev, a_nulls, b_nulls)


def like_device(col, pattern, n, out_dev, out_nulls_dev, col_nulls=None, pattern_nulls=None):
    """LIKE on resident vectors, as str_compare_device; the pattern is a (cells, area) pair of DeviceBuffers or of host arrays (a const
    pattern read on the host)."""
    if isinstance(pattern, (bytes, bytearray)):
        pattern = [bytes(pattern)]
    _str_pred_device(capi.XCALL_GO_LIKE, col, pattern, n, out_dev, out_nulls_dev, col_nulls, pattern_nulls)


# ------------------------------------------------------------------------------- IN / NOT IN (csrc/goelem.cu, csrc/strpred.cu)
def go_in(T, col, values, negate=False, col_nulls=None, values_nulls=None, rnulls=None, length=None):
    """col IN values (NOT IN with negate), operator_in.go: values is the list, with its NULL elements skipped; a NULL row is NULL, every
    other row is its membership (NOT IN: its negation).  Fixed-width T: numpy arrays of the column's element type (DECIMAL128 / UUID:
    16-byte rows); the varlena T: a list of bytes or a (cells, area) pair.  A one-element col is a const.  rnulls: the result bitmap on entry
    (rows set there are skipped).  Returns (values bool[n], nulls bool[n])."""
    vc, vl = _vec(col, nulls=col_nulls), _vec(values, nulls=values_nulls)
    n = length if length is not None else vc.length
    r = np.zeros(max(n, 1), dtype=np.uint8)
    rn = np.zeros(max((n + 63) // 64, 1), dtype=np.uint64) if rnulls is None else np.array(rnulls, dtype=np.uint64)
    fid = capi.XCALL_GO_NOT_IN(T) if negate else capi.XCALL_GO_IN(T)
    xcall(fid, [Vector(data=r[:n], nulls=rn, length=n), vc, vl, _params_vec(np.array([vl.length], np.int64))], n)
    return r[:n].astype(bool), bitmap_to_bools(rn, n)


def go_in_device(T, col, values, nvalues, n, out_dev, out_nulls_dev, negate=False, col_nulls=None, values_nulls=None):
    """IN / NOT IN on resident vectors: col and values are DeviceBuffers (the varlena T: (cells, area) pairs, area None when every value is
    inline), nulls DeviceBuffers or None; out_dev (bool[n]) and out_nulls_dev (its bitmap, in/out) DeviceBuffers.  The parameter block stays
    on the host, so a fixed-width call only enqueues work; a varlena call reads back one status record."""
    fid = capi.XCALL_GO_NOT_IN(T) if negate else capi.XCALL_GO_IN(T)
    xcall(fid, [Vector(data=out_dev.view(n), nulls=out_nulls_dev, length=n), _vec(col, n, col_nulls), _vec(values, nvalues, values_nulls),
                _params_vec(np.array([nvalues], np.int64))], n)


# --------------------------------------------------------------- CASE, IF, COALESCE and the CASE select lists (csrc/caseexpr.cu)
# value bytes per row of the GO_CASE / GO_COALESCE types; the varlena types are 24-byte cells plus an area
CASE_WIDTH = {capi.T_BOOL: 1, capi.T_INT8: 1, capi.T_UINT8: 1, capi.T_INT16: 2, capi.T_UINT16: 2, capi.T_ENUM: 2, capi.T_INT32: 4,
              capi.T_UINT32: 4, capi.T_FLOAT32: 4, capi.T_DATE: 4, capi.T_INT64: 8, capi.T_UINT64: 8, capi.T_FLOAT64: 8, capi.T_TIME: 8,
              capi.T_DATETIME: 8, capi.T_TIMESTAMP: 8, capi.T_DECIMAL64: 8, capi.T_BIT: 8, capi.T_DECIMAL128: 16, capi.T_UUID: 16}
CASE_STR_TYPES = (capi.T_CHAR, capi.T_VARCHAR, capi.T_BLOB, capi.T_TEXT, capi.T_DATALINK)


def _case_value_dtype(T):
    return {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64, 16: np.uint64}[CASE_WIDTH[T]] if T not in capi.NP_OF_T else capi.NP_OF_T[T]


def _when_then(conds, values, else_value):
    """GO_CASE's operands in argument order: c1, v1, ... [, else]"""
    if len(conds) != len(values):
        raise ValueError("one value per condition")
    return [o for cv in zip(conds, values) for o in cv] + ([] if else_value is None else [else_value])


def _case_call(fid, res, nsel, has_else, vecs, n):
    """one GO_CASE / GO_COALESCE call: (rc, msg, area_len), area_len the bytes a string result's area needs"""
    prm = _params_vec(capi.CaseParams(nsel, has_else, 0))
    rc, msg = xcall(fid, [res, prm] + vecs, n, raise_on_error=False)
    return rc, msg, int(prm.data.view(np.int64)[1])


def _case_run(fid, T, operands, nsel, has_else, rnulls, length, area_cap):
    vecs = [_vec(d, nulls=nl) for d, nl in operands]
    n = length if length is not None else max(v.length for v in vecs)
    rn = np.zeros(max((n + 63) // 64, 1), dtype=np.uint64) if rnulls is None else np.array(rnulls, dtype=np.uint64)
    if T not in CASE_STR_TYPES:
        w = CASE_WIDTH.get(T, 8)
        r = np.zeros(max(n, 1) * w, dtype=np.uint8)
        rc, msg, _ = _case_call(fid, Vector(data=r[:n * w], nulls=rn, length=n), nsel, has_else, vecs, n)
        if rc:
            raise capi.MoError(rc, "xcall xfunc failed, error code %d, %s" % (rc, msg))
        out = r[:n * w].view(_case_value_dtype(T))
        return (out.reshape(n, 2) if w == 16 else out), bitmap_to_bools(rn, n)
    cap = area_cap if area_cap is not None else sum(int(v.area.nbytes) for v in vecs if v.area is not None)
    cells = np.zeros(max(n, 1) * 24, dtype=np.uint8)
    for attempt in range(2):
        area = np.zeros(cap, dtype=np.uint8)
        rc, msg, need = _case_call(fid, Vector(data=cells[:24 * n], nulls=rn, area=area, length=n), nsel, has_else, vecs, n)
        if rc == capi.RC_OUT_OF_RANGE and attempt == 0 and area_cap is None:
            cap = need                     # the JOIN_PROBE capacity protocol: the call left the result unchanged; repeat with area_len
            continue
        if rc:
            raise capi.MoError(rc, "xcall xfunc failed, error code %d, %s" % (rc, msg))
        return cells[:24 * n], area[:need], bitmap_to_bools(rn, n)


def go_case(T, conds, values, else_value=None, rnulls=None, length=None, area_cap=None):
    """CASE WHEN conds[0] THEN values[0] ... [ELSE else_value] END (caseFn).  Every operand is a (data, nulls) pair, nulls = bitmap words or
    None; a one-row operand is a const.  rnulls: the result bitmap on entry (rows set there are skipped).  Fixed-width T returns (values,
    nulls bool[n]); the string T returns (cells uint8[24 n], area, nulls bool[n]), the area sized by the call (area_cap: a fixed capacity,
    RC_OUT_OF_RANGE raised when it is too small)."""
    operands = _when_then(conds, values, else_value)
    return _case_run(capi.XCALL_GO_CASE(T), T, operands, len(conds), 0 if else_value is None else 1, rnulls, length, area_cap)


def go_iff(T, cond, a, b, rnulls=None, length=None, area_cap=None):
    """IF(cond, a, b) (iffFn): CASE with one WHEN and an ELSE -- a NULL or false condition takes b"""
    return go_case(T, [cond], [a], b, rnulls, length, area_cap)


def go_coalesce(T, operands, rnulls=None, length=None, area_cap=None):
    """COALESCE(operands...) (CoalesceGeneral / CoalesceStr): the first non-NULL operand, or NULL.  Operands and results as go_case."""
    return _case_run(capi.XCALL_GO_COALESCE(T), T, operands, len(operands), 0, rnulls, length, area_cap)


def _case_device(fid, T, operands, nsel, has_else, n, out_dev, out_nulls_dev, out_area_dev):
    width = 24 if T in CASE_STR_TYPES else CASE_WIDTH.get(T, 8)
    res = Vector(data=out_dev.view(width * n), nulls=out_nulls_dev, area=out_area_dev if T in CASE_STR_TYPES else None, length=n)
    rc, msg, area_len = _case_call(fid, res, nsel, has_else, [_vec(d, n, nl) for d, nl in operands], n)
    if rc and not (rc == capi.RC_OUT_OF_RANGE and T in CASE_STR_TYPES):
        raise capi.MoError(rc, "xcall xfunc failed, error code %d, %s" % (rc, msg))
    return rc, area_len


def go_case_device(T, conds, values, else_value, n, out_dev, out_nulls_dev, out_area_dev=None):
    """go_case on resident operands: (data, nulls) pairs of DeviceBuffers (a string value's data is a (cells, area) pair; one element's bytes
    = const) into out_dev (T[n] or 24-byte cells), out_nulls_dev (its bitmap, in/out) and out_area_dev (strings: the area, its size the
    capacity).  The parameter block stays on the host: a fixed-width call only enqueues work.  Returns (rc, area_len): rc is 0, or
    RC_OUT_OF_RANGE for a string result whose area is smaller than area_len (the result is then unchanged)."""
    operands = _when_then(conds, values, else_value)
    return _case_device(capi.XCALL_GO_CASE(T), T, operands, len(conds), 0 if else_value is None else 1, n, out_dev, out_nulls_dev, out_area_dev)


def go_coalesce_device(T, operands, n, out_dev, out_nulls_dev, out_area_dev=None):
    """go_coalesce on resident operands, as go_case_device"""
    return _case_device(capi.XCALL_GO_COALESCE(T), T, operands, len(operands), 0, n, out_dev, out_nulls_dev, out_area_dev)


def case_select(rem_words, cond, cond_nulls, n):
    """one WHEN of EvalCase's select lists as null-prefill words (set = skip the row): rem_words = the rows already taken or not selected
    (start with NOT selectList), cond the WHEN's bool values (one element: const) and cond_nulls its bitmap words or None.  Returns
    (THEN's prefill words, the new remaining words)."""
    w = (n + 63) // 64
    then = np.zeros(max(w, 1), dtype=np.uint64)
    rem = np.array(rem_words, dtype=np.uint64).reshape(-1)[:w].copy()
    c = np.ascontiguousarray(cond).view(np.uint8).reshape(-1)
    xcall(capi.XCALL_GO_CASE_SELECT, [Vector(data=then[:w], length=n), Vector(data=rem, length=n), _vec(c, nulls=cond_nulls)], n)
    return then[:w], rem


def case_select_device(then_dev, rem_dev, cond_dev, cond_nulls_dev, n):
    """case_select on resident words and condition (DeviceBuffers): enqueue-only"""
    wb = 8 * ((n + 63) // 64)
    xcall(capi.XCALL_GO_CASE_SELECT, [Vector(data=then_dev.view(wb), length=n), Vector(data=rem_dev.view(wb), length=n),
                                      _vec(cond_dev, n, cond_nulls_dev)], n)
