"""What ops.py hands the library, checked without a GPU: ops.xcall is replaced by a recorder that sees each call's argument blocks as
XCall would (func id, len, and per slot dataSz / nullCnt / areaSz and what pdata / pnulls / parea point at).  Device buffers are fakes at
fixed addresses, so no call reaches libmo_b200.so.

A call's host form and its device form (`*_device`, `search(out=...)`, `run(out_ptr=...)`) must give the library the same func id, len and
slot count, and the same sizes and set pointers in every slot, except the result slots named where the two signatures differ."""
import ctypes as C

import numpy as np
import pytest

from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, Vector, bitmap_from_bools, varlena_bytes_column

DEV_BASE = 0x7F00_0000_0000


class FakeDevice:
    """DeviceBuffers at fixed addresses; `owner` is set, so free() never calls the library"""

    def __init__(self):
        self.top = DEV_BASE

    def buf(self, nbytes):
        b = DeviceBuffer.__new__(DeviceBuffer)
        b.lib, b.nbytes, b.ptr, b.owner = None, int(nbytes), self.top, self
        self.top += (int(nbytes) + 0x1FFF) & ~0xFFF
        return b

    def like(self, x):
        """the device twin of a host operand: same bytes, fresh address (tuples and None map element-wise)"""
        if x is None:
            return None
        if isinstance(x, tuple):
            return tuple(self.like(e) for e in x)
        if isinstance(x, list):
            return self.like(varlena_bytes_column(x))
        return self.buf(np.ascontiguousarray(x).nbytes)

    def ptr(self, nbytes):
        return self.buf(nbytes).ptr

    def owns(self, addr):
        return DEV_BASE <= addr < self.top


class Recorder:
    """stands in for ops.xcall: records each call as the library would see it and returns (0, "")"""

    def __init__(self, dev):
        self.dev, self.calls, self.host_tags = dev, [], {}

    def _mem(self, addr, nbytes):
        if not addr:
            return None
        if self.dev.owns(addr):
            return ("dev", addr - DEV_BASE)
        if nbytes is None:
            return ("host", None)
        raw = C.string_at(addr, nbytes)
        for a, tag in self.host_tags.items():          # a host address inside a parameter block differs run to run
            raw = raw.replace(int(a).to_bytes(8, "little"), tag)
        return ("host", raw)

    def __call__(self, func_id, vectors, length, runtime_id=1, lib=None, raise_on_error=True):
        slots = []
        for v in vectors:
            a = v.fill_raw_ptr_len() if isinstance(v, Vector) else v
            nulls = getattr(v, "nulls", None)
            nb = nulls.nbytes if isinstance(nulls, np.ndarray) else None
            slots.append((a.dataSz, a.nullCnt, a.areaSz, self._mem(a.pdata, a.dataSz), self._mem(a.pnulls, nb), self._mem(a.parea, a.areaSz)))
        self.calls.append((func_id, length, tuple(slots)))
        return 0, ""


def _words(n, seed=0):
    rng = np.random.default_rng(seed)
    return bitmap_from_bools(rng.random(n) < 0.3)


def _strings(n, seed=0):
    rng = np.random.default_rng(seed)
    return [bytes(rng.integers(97, 123, int(rng.integers(0, 40)), dtype=np.uint8)) for _ in range(n)]


def cases(dev, rec):
    """(name, host call, device call or None, result slots whose sizes or pointers may differ between the two forms).  Every public
    function and method of ops.py that reaches XCall appears here, in both forms where it has both."""
    rng = np.random.default_rng(7)
    D = dev.like
    out = []

    def add(name, host, device=None, free=()):
        out.append((name, host, device, frozenset(free)))

    # aggregates
    def _block1(n):
        col = rng.integers(-9, 9, n).astype(np.int64)
        nl = _words(n)
        for fn in (ops.agg_sum, ops.agg_avg, ops.agg_count, ops.agg_min, ops.agg_max):
            add("%s_n%d" % (fn.__name__, n), lambda fn=fn, col=col, nl=nl: fn(capi.T_INT64, col, nl))
        add("agg_sum_dev_n%d" % n, lambda col=col, nl=nl, n=n: ops.agg_sum(capi.T_INT64, D(col), D(nl), n))
        add("agg_sum_dev_nolen_n%d" % n, lambda col=col: ops.agg_sum(capi.T_INT64, D(col)))
        add("agg_state_n%d" % n, lambda col=col, nl=nl: ops.agg_state(capi.AGG_SUM, capi.T_INT64, col, nl),
            lambda col=col, nl=nl, n=n: ops.agg_state_device(capi.AGG_SUM, capi.T_INT64, D(col), D(nl), n, dev.ptr(24), dev.ptr(8)))
        add("agg_state_nonulls_n%d" % n, lambda col=col: ops.agg_state(capi.AGG_MAX, capi.T_INT64, col),
            lambda col=col, n=n: ops.agg_state_device(capi.AGG_MAX, capi.T_INT64, D(col), None, n, dev.ptr(24), dev.ptr(8)))
        st = rng.integers(0, 9, (max(n, 1), 3)).astype(np.uint64)
        add("agg_merge_state_n%d" % n, lambda st=st: ops.agg_merge(capi.AGG_SUM, capi.T_INT64, st, final=False),
            lambda st=st: ops.agg_merge_device(capi.AGG_SUM, capi.T_INT64, dev.ptr(st.nbytes), st.shape[0], dev.ptr(24), out_nulls_ptr=dev.ptr(8)))
        add("agg_merge_final_n%d" % n, lambda st=st: ops.agg_merge(capi.AGG_SUM, capi.T_INT64, st),
            lambda st=st: ops.agg_merge_device(capi.AGG_SUM, capi.T_INT64, dev.ptr(st.nbytes), st.shape[0], dev.ptr(16), 16, dev.ptr(8)))
    for n in (0, 1, 100):
        _block1(n)

    # TPC-H shapes
    P6 = (8766, 9131, 0.05, 0.07, 24.0)
    def _block2(n):
        sd, disc, qty, pr = (rng.integers(8000, 10000, n).astype(np.int32), rng.random(n), rng.random(n) * 50, rng.random(n) * 1e4)
        add("q6_n%d" % n, lambda c=(sd, disc, qty, pr), n=n: ops.q6_filter_sum(*c, n, *P6),
            lambda c=(sd, disc, qty, pr), n=n: ops.q6_filter_sum_device(*map(D, c), n, *P6, dev.ptr(16), dev.ptr(8)))
        add("q6_nonulls_n%d" % n, lambda c=(sd, disc, qty, pr), n=n: ops.q6_filter_sum(*c, n, *P6),
            lambda c=(sd, disc, qty, pr), n=n: ops.q6_filter_sum_device(*map(D, c), n, *P6, dev.ptr(16)), free={0})
        dc = (sd, (disc * 100).astype(np.int64), (qty * 100).astype(np.int64), (pr * 100).astype(np.int64))
        add("q6_dec_n%d" % n, lambda c=dc, n=n: ops.q6_dec_filter_sum(*c, n, 8766, 9131, 5, 7, 2400, 2, 5),
            lambda c=dc, n=n: ops.q6_dec_filter_sum_device(*map(D, c), n, 8766, 9131, 5, 7, 2400, 2, dev.ptr(ops.Q6_DEC_RESULT_BYTES), dev.ptr(8), 5))
        q1 = (sd, qty, pr, disc, rng.random(n), rng.integers(65, 70, n).astype(np.uint8), rng.integers(70, 80, n).astype(np.uint8))
        add("q1_n%d" % n, lambda c=q1, n=n: ops.q1_group_agg(*c, n, 9000, 3),
            lambda c=q1, n=n: ops.q1_group_agg_device(*map(D, c), n, 9000, dev.ptr(ops.Q1_RESULT_BYTES), 3))
    for n in (0, 1, 1000):
        _block2(n)
    for k in (0, 1, 3):
        add("q6_merge_%d" % k, lambda k=k: ops.q6_merge([(1.5 * i, i) for i in range(k)]),
            lambda k=k: ops.q6_merge_device(dev.ptr(16 * k), k, dev.ptr(16), dev.ptr(8)))
        add("q6_dec_merge_%d" % k, lambda k=k: ops.q6_dec_merge(bytes(range(ops.Q6_DEC_RESULT_BYTES)) * k, k),
            lambda k=k: ops.q6_dec_merge_device(dev.ptr(ops.Q6_DEC_RESULT_BYTES * k), k, dev.ptr(ops.Q6_DEC_RESULT_BYTES), dev.ptr(8)))
        add("q1_merge_%d" % k, lambda k=k: ops.q1_merge(bytes(ops.Q1_RESULT_BYTES * k), k),
            lambda k=k: ops.q1_merge_device(dev.ptr(ops.Q1_RESULT_BYTES * k), k, dev.ptr(ops.Q1_RESULT_BYTES)))

    # vector search
    dim, n = 8, 50
    bf = ops.BruteForceIndex.__new__(ops.BruteForceIndex)
    bf.lib, bf.dim, bf.metric, bf.key_base, bf.n, bf.owned, bf.prepared = None, dim, capi.METRIC_L2, 100, n, False, False
    bf.buf = dev.buf(4 * n * dim)
    ivf = ops.IvfflatSearchIndex.__new__(ops.IvfflatSearchIndex)
    ivf.lib, ivf.dim, ivf.nlist, ivf.metric, ivf.n, ivf.prepared = None, dim, 4, capi.METRIC_L2SQ, n, False
    ivf.d_data, ivf.d_cent, ivf.d_off, ivf.d_ids = dev.buf(4 * n * dim), dev.buf(4 * 4 * dim), dev.buf(8 * 5), dev.buf(8 * n)
    keybits = rng.integers(0, 2 ** 63, 3).astype(np.uint64)
    rec.host_tags[keybits.ctypes.data] = b"KEYBITS!"
    filters = {"none": lambda: None, "bits": lambda: keybits, "dbits": lambda: dev_keybits, "bloom": lambda: 0x1234560}
    dev_keybits = dev.buf(keybits.nbytes)
    for nq in (1, 5):
        q = rng.random((nq, dim)).astype(np.float32)
        for fname, f in filters.items():
            add("bf_search_nq%d_%s" % (nq, fname), lambda q=q, f=f: bf.search(q, 3, filter=f()),
                lambda q=q, f=f, nq=nq: bf.search(D(q), 3, out=(dev.ptr(nq * 24), dev.ptr(nq * 24)), filter=f()))
            add("ivf_search_nq%d_%s" % (nq, fname), lambda q=q, f=f: ivf.search(q, 3, 2, sqrt_out=True, filter=f()),
                lambda q=q, f=f, nq=nq: ivf.search(D(q), 3, 2, sqrt_out=True, out=(dev.ptr(nq * 24), dev.ptr(nq * 24)), filter=f()))
    for nsh, nq, k in ((1, 1, 1), (3, 4, 5)):
        ks = rng.integers(0, 99, nsh * nq * k).astype(np.int64)
        ds = rng.random(nsh * nq * k)
        add("topk_merge_%d_%d_%d" % (nsh, nq, k), lambda ks=ks, ds=ds, nq=nq, k=k: ops.topk_merge(ks, ds, nq, k),
            lambda ks=ks, ds=ds, nsh=nsh, nq=nq, k=k: ops.topk_merge_device(dev.ptr(ks.nbytes), dev.ptr(ds.nbytes), nsh, nq, k,
                                                                              dev.ptr(8 * nq * k), dev.ptr(8 * nq * k)))

    # column operators
    def _block3(n):
        b = rng.integers(0, 2, n).astype(np.uint8)
        nl = _words(n, 1)
        add("filter_sels_n%d" % n, lambda b=b, nl=nl: ops.filter_sels(b, nl),
            lambda b=b, nl=nl, n=n: ops.filter_sels_device(D(b), D(nl), n, dev.ptr(8 * n), dev.ptr(8)), free={0})
        add("filter_sels_nonulls_n%d" % n, lambda b=b: ops.filter_sels(b),
            lambda b=b, n=n: ops.filter_sels_device(D(b), None, n, dev.ptr(8 * n), dev.ptr(8)), free={0})
        src = rng.integers(0, 99, max(n, 1)).astype(np.int16)
        sels = rng.integers(0, max(n, 1), n).astype(np.int64)
        add("shuffle_n%d" % n, lambda src=src, sels=sels: ops.shuffle(src, sels, _words(len(src), 2), want_nulls=True))
        add("shuffle_plain_n%d" % n, lambda src=src, sels=sels: ops.shuffle(src, sels))
        cols = [rng.integers(0, 9, n).astype(np.int32), np.array([3], np.int16), rng.integers(0, 9, n).astype(np.uint8)]
        add("pack_keys_n%d" % n, lambda cols=cols, n=n: ops.pack_keys(cols, [None, None, _words(n, 3)], length=n))
        add("pack_keys_skip_n%d" % n, lambda cols=cols: ops.pack_keys(cols, has_null=False, length=n))
        keys = rng.integers(0, 5, n).astype(np.uint64)
        gt = ops.GroupTable(16)
        add("group_ids_n%d" % n, lambda keys=keys, gt=gt: gt.insert(keys),
            lambda keys=keys, n=n: ops.GroupTable(16).insert_device(D(keys), n, dev.buf(8 * n), dev.buf(8), dev.buf(8 * 16), 16))
        g = rng.integers(0, 4, n).astype(np.uint64)
        add("group_agg_n%d" % n, lambda g=g, nl=nl, n=n: ops.group_agg(capi.AGG_SUM, capi.T_INT32, np.zeros(4, np.int64), np.zeros(1, np.uint64),
                                                                        np.zeros(4, np.int64), g, rng.integers(0, 9, n).astype(np.int32), nl))
        add("group_agg_count_n%d" % n, lambda g=g: ops.group_agg(capi.AGG_COUNT, capi.T_INT32, np.zeros(4, np.int64), np.zeros(1, np.uint64), None, g, None))
    for n in (0, 1, 70):
        _block3(n)

    # ORDER BY
    def _block4(n):
        fixed = rng.integers(0, 9, n).astype(np.int64)
        dec = rng.integers(0, 9, (n, 2)).astype(np.uint64)
        strs = _strings(n, 4)
        cells, area = varlena_bytes_column(strs)
        inl = varlena_bytes_column([s[:10] for s in strs])
        nl = [_words(n, 5), None, None, _words(n, 6)]
        T = [capi.T_INT64, capi.T_DECIMAL128, capi.T_VARCHAR, capi.T_CHAR]
        flags = [capi.ORDER_DESC, 0, capi.ORDER_NULLS_LAST, capi.ORDER_NULLS_FIRST]
        rid = np.arange(n, dtype=np.int64)
        for limit in (None, 3):
            add("order_n%d_lim%s" % (n, limit), lambda c=[fixed, dec, (cells, area), (inl[0], None)], nl=nl, limit=limit: ops.order_sels(c, nl, flags, limit, types=T),
                lambda c=[fixed, dec, (cells, area), (inl[0], None)], nl=nl, n=n, limit=limit: ops.order_sels_device(
                    [D(x) for x in c], [D(x) for x in nl], T, flags, n, dev.ptr(8 * (n if limit is None or limit >= n else limit)), limit), free={0})
            add("order_rowids_n%d_lim%s" % (n, limit), lambda c=[fixed], limit=limit: ops.order_sels(c, None, [0], limit, row_ids=rid),
                lambda c=[fixed], n=n, limit=limit: ops.order_sels_device([D(fixed)], None, [capi.T_INT64], [0], n,
                                                                           dev.ptr(8 * (n if limit is None or limit >= n else limit)), limit, D(rid)), free={0})
        add("order_list_n%d" % n, lambda: ops.order_sels([strs, np.array([2], np.int32)], None, [0, 0]))
        add("order_const_n%d" % n, lambda: ops.order_sels([fixed, np.array([2], np.int32)], None, [0, 0], length=n))

        # string keys
        kc = [fixed.astype(np.int32), (cells, area), (inl[0], None), np.array([5], np.int64)]
        kt = [capi.T_INT32, capi.T_VARCHAR, capi.T_CHAR, capi.T_INT64]
        knl = [_words(n, 7), _words(n, 8), None, None]
        for has_null in (True, False):
            add("pack_str_keys_n%d_%d" % (n, has_null), lambda kc=kc, knl=knl, h=has_null: ops.pack_str_keys(kc, kt, knl, h, length=n, capacity=64 * n),
                lambda kc=kc, knl=knl, h=has_null, n=n: ops.pack_str_keys_device([D(x) for x in kc], [D(x) for x in knl], kt, n, dev.buf(64 * n),
                                                                                 dev.buf(8 * (n + 1)), None if h else dev.buf(8 * ((n + 63) // 64)), h))
        add("pack_str_keys_list_n%d" % n, lambda: ops.pack_str_keys([strs], [capi.T_VARCHAR]))

        # string group table
        kb = np.frombuffer(b"".join(strs), np.uint8).copy() if n else np.zeros(0, np.uint8)
        ko = np.concatenate([[0], np.cumsum([len(s) for s in strs])]).astype(np.uint64)
        skip = _words(n, 9)
        for fr in (False, True):
            add("str_group_ids_n%d_%d" % (n, fr), lambda fr=fr: ops.StrGroupTable(64, 4096).insert(kb, ko, skip, first_rows=fr),
                lambda fr=fr, n=n: ops.StrGroupTable().insert_device(D(kb), D(ko), n, dev.buf(8 * n), dev.buf(8), dev.buf(4096), dev.buf(8 * 65),
                                                                     dev.buf(8 * n) if fr else None, D(skip)), free={0, 6})
        add("str_group_ids_hostcount_n%d" % n, lambda: ops.StrGroupTable().insert_device(D(kb), D(ko), n, dev.buf(8 * n), np.zeros(1, np.int64),
                                                                                        dev.buf(4096), dev.buf(8 * 65)))
    for n in (0, 1, 40):
        _block4(n)

    # the fused plan
    def _block5(n):
        cols = [rng.integers(8000, 10000, n).astype(np.int32), rng.random(n), rng.random(n), rng.random(n)]
        nl = [None, _words(n, 10), None, None]
        p = ops.q6_plan()
        add("plan_q6_n%d" % n, lambda p=p, cols=cols, nl=nl, n=n: p.run(cols, n, nl, max_groups=4),
            lambda p=p, cols=cols, nl=nl, n=n: p.run([D(c) for c in cols], n, [D(x) for x in nl], max_groups=4, out_ptr=dev.ptr(p.result_bytes(4))))
        p1 = ops.q1_plan(9000, 5)
        c1 = [cols[0], cols[1], cols[2], cols[3], rng.random(n), rng.integers(65, 70, n).astype(np.uint8), rng.integers(70, 80, n).astype(np.uint8)]
        add("plan_q1_n%d" % n, lambda p=p1, c=c1, n=n: p.run(c, n),
            lambda p=p1, c=c1, n=n: p.run([D(x) for x in c], n, out_ptr=dev.ptr(p.result_bytes(64))))
    for n in (0, 1, 30):
        _block5(n)

    # decimals
    def _block6(n):
        a64, b64 = rng.integers(-999, 999, n).astype(np.int64), rng.integers(-999, 999, n).astype(np.int64)
        a128 = rng.integers(0, 2 ** 63, (n, 2)).astype(np.uint64)
        n1, n2 = _words(n, 11), _words(n, 12)
        one = np.array([7], np.int64)
        for op in (0, 2):
            add("dec_arith_%d_n%d" % (op, n), lambda op=op: ops.dec_arith(op, 64, a64, b64, 2, 3, n, n1, n2))
        add("dec_arith_const_n%d" % n, lambda: ops.dec_arith(1, 128, a128, np.array([[5, 0]], np.uint64), 2, 2, n, None, None, _words(n, 13)))
        add("dec_sum_n%d" % n, lambda: ops.dec_sum(64, a64, np.zeros((3, 2), np.uint64), np.zeros(3, np.int64), rng.integers(0, 3, n).astype(np.uint64), n1))
        add("dec_sum_nogroups_n%d" % n, lambda: ops.dec_sum(128, a128, np.zeros((1, 2), np.uint64), np.zeros(1, np.int64)))
        for w, a, b in ((64, a64, b64), (128, a128, a128[::-1].copy()), (64, a64, one)):
            add("dec_compare_%d_n%d_b%d" % (w, n, len(b)), lambda w=w, a=a, b=b: ops.dec_compare(2, w, a, b, 2, 3, n, n1, n2),
                lambda w=w, a=a, b=b, n=n: ops.dec_compare_device(2, w, D(a), D(b), 2, 3, n, dev.buf(n), dev.buf(8 * ((n + 63) // 64)), D(n1), D(n2)),
                free={0})
            add("dec_div_%d_n%d_b%d" % (w, n, len(b)), lambda w=w, a=a, b=b: ops.dec_div(w, a, b, 2, 3, n, n1, n2, div0_error=True),
                lambda w=w, a=a, b=b, n=n: ops.dec_div_device(w, D(a), D(b), 2, 3, n, dev.buf(16 * n), dev.buf(8 * ((n + 63) // 64)), D(n1), D(n2), True))
        for w, a in ((64, a64), (128, a128)):
            add("dec_between_%d_n%d" % (w, n), lambda w=w, a=a: ops.dec_between(w, a, -5, (1 << 70) if w == 128 else 77, n, n1),
                lambda w=w, a=a, n=n: ops.dec_between_device(w, D(a), -5, (1 << 70) if w == 128 else 77, n, dev.buf(n), dev.buf(8 * ((n + 63) // 64)), D(n1)), free={0})
        add("dec_between_devcol_n%d" % n, lambda n=n: ops.dec_between(64, D(a64), 1, 2, n))
        sums, cnts = rng.integers(0, 99, (n, 2)).astype(np.uint64), rng.integers(0, 9, n).astype(np.int64)
        for w in (64, 128):
            add("dec_avg_%d_n%d" % (w, n), lambda w=w: ops.dec_avg(w, sums, cnts, 2),
                lambda w=w, n=n: ops.dec_avg_device(w, D(sums), D(cnts), n, 2, dev.buf(16 * n), dev.buf(8 * ((n + 63) // 64))))
    for n in (0, 1, 20):
        _block6(n)

    # normalize_l2, k-means, LZ4, vector unmarshal
    from matrixone_b200.vector import varlena_column
    for rows in ([], [np.ones(3)], [np.arange(10.0), np.ones(2)]):
        cells, area = varlena_column(rows)
        add("normalize_l2_%d" % len(rows), lambda c=cells, a=area, k=len(rows): ops.normalize_l2(c, a, k))
        add("normalize_l2_nulls_%d" % len(rows), lambda c=cells, a=area, k=len(rows): ops.normalize_l2(c, a, k, np.float64, _words(k, 14)))
    v = rng.random((12, 3)).astype(np.float32)
    add("kmeans", lambda: ops.kmeans_elkan(v, v[:4], 5, rnd=np.arange(6, dtype=np.float32)))
    add("kmeans_nornd", lambda: ops.kmeans_elkan(v.astype(np.float64), v[:4], 5))
    add("lz4", lambda: ops.lz4_decode_blocks([b"\x10a", b"\x20bc"], [1, 2]))
    add("lz4_empty", lambda: ops.lz4_decode_blocks([], []))
    add("vector_unmarshal", None, lambda: ops.vector_unmarshal_device(dev.buf(100), 90, dev.buf(64), dev.buf(16), dev.buf(8)))
    add("vector_unmarshal_noarea", None, lambda: ops.vector_unmarshal_device(dev.buf(100), 90, dev.buf(64), None, None))

    # hash joins
    def _block7(n):
        bk = rng.integers(0, 6, n).astype(np.uint64)
        jm = ops.JoinMap(bk, _words(n, 15), prepare=False)
        jm.ngroups, jm.table_keys = 6, np.arange(6, dtype=np.uint64)
        jm.offsets, jm.sels = np.arange(8, dtype=np.int32), np.arange(max(n, 1), dtype=np.int32)
        pk = rng.integers(0, 8, n).astype(np.uint64)
        add("join_find_n%d" % n, lambda jm=jm, pk=pk: jm.find(pk, _words(len(pk), 16)))
        strs = _strings(n, 17)
        kb = np.frombuffer(b"".join(strs), np.uint8).copy() if n else np.zeros(0, np.uint8)
        ko = np.concatenate([[0], np.cumsum([len(s) for s in strs])]).astype(np.uint64)
        sm = ops.StrJoinMap(kb, ko, prepare=False)
        sm.ngroups, sm.table_offsets, sm.table_bytes = 2, np.array([0, 3, 5], np.uint64), np.frombuffer(b"abcde", np.uint8).copy()
        add("str_join_find_n%d" % n, lambda sm=sm, kb=kb, ko=ko, n=n: sm.find(kb, ko, _words(n, 18)),
            lambda kb=kb, ko=ko, n=n: ops.str_join_find_device(dev.buf(8 * n), n, 2, dev.buf(5), dev.buf(24), D(kb), D(ko), D(_words(n, 18))))
        add("str_join_find_nonulls_n%d" % n, lambda sm=sm, kb=kb, ko=ko: sm.find(kb, ko),
            lambda kb=kb, ko=ko, n=n: ops.str_join_find_device(dev.buf(8 * n), n, 2, dev.buf(5), dev.buf(24), D(kb), D(ko)))
        vals = rng.integers(0, 3, n).astype(np.uint64)
        cap = 2 * max(n, 1)
        for jt in (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_RIGHT_SINGLE):
            mb = ops.matched_bitmap(max(n, 1)) if jt >= capi.JOIN_RIGHT else None
            add("join_probe_n%d_t%d" % (n, jt), lambda jm=jm, pk=pk, jt=jt, mb=mb: jm.probe(pk, jt, _words(len(pk), 19), cap, mb))
            add("str_join_probe_n%d_t%d" % (n, jt), lambda sm=sm, kb=kb, ko=ko, jt=jt, mb=mb: sm.probe(kb, ko, jt, None, cap, mb))
            for uniq in (False, True):
                offs, sls = (None, None) if uniq else (np.arange(5, dtype=np.int32), np.arange(4, dtype=np.int32))
                add("probe_gids_n%d_t%d_u%d" % (n, jt, uniq), lambda vals=vals, jt=jt, mb=mb, offs=offs, sls=sls: ops.probe_gids(vals, 3, offs, sls, jt, cap, mb),
                    lambda vals=vals, jt=jt, mb=mb, offs=offs, sls=sls, n=n: ops.probe_gids_device(
                        D(vals), n, 3, D(offs), D(sls), jt, dev.buf(8 * cap), dev.buf(8 * cap), dev.buf(8), D(mb)))
            npairs = n
            cp, cb = rng.integers(0, max(n, 1), npairs).astype(np.int64), rng.integers(0, 9, npairs).astype(np.int64)
            cond, cn = rng.integers(0, 2, npairs).astype(bool), _words(npairs, 20)
            for nulls in (cn, None):
                add("join_cond_n%d_t%d_%d" % (n, jt, nulls is None), lambda cp=cp, cb=cb, cond=cond, nulls=nulls, jt=jt, mb=mb, n=n: ops.join_cond(
                        cp, cb, cond, n, jt, nulls, 2 * max(n, 1), mb),
                    lambda cp=cp, cb=cb, cond=cond, nulls=nulls, jt=jt, mb=mb, n=n: ops.join_cond_device(
                        D(cp), D(cb), D(cond), D(nulls), n, n, jt, dev.buf(16 * max(n, 1)), dev.buf(16 * max(n, 1)), dev.buf(8), D(mb)))
            if mb is not None:
                mb = ops.matched_bitmap(n)
                add("join_build_rows_n%d_t%d" % (n, jt), lambda mb=mb, jt=jt, n=n: ops.join_build_rows(mb, n, jt),
                    lambda mb=mb, jt=jt, n=n: ops.join_build_rows_device(D(mb), n, jt, dev.ptr(8 * n), dev.ptr(8)), free={0})
                bms = [ops.matched_bitmap(n) | np.uint64(i) for i in range(3)]
                add("join_matched_merge_n%d_t%d" % (n, jt), lambda bms=bms, jt=jt, n=n: ops.join_matched_merge(bms, n, jt),
                    lambda bms=bms, jt=jt, n=n: ops.join_matched_merge_device(D(bms[0]), [D(b) for b in bms], n, jt))
    for n in (0, 1, 30):
        _block7(n)

    # string predicates, IN, CASE
    def _block8(n):
        a, b = _strings(n, 21), _strings(n, 22)
        ac, bc = varlena_bytes_column(a), varlena_bytes_column([s[:5] for s in b])
        an, bn = _words(n, 23), _words(n, 24)
        rn0 = _words(n, 25)
        for bop, bnl in (((bc[0], None), bn), (varlena_bytes_column([b"const-operand-longer-than-23"]), None)):
            add("str_compare_n%d_b%d" % (n, len(bop[0])), lambda bop=bop, bnl=bnl, n=n: ops.str_compare(1, capi.T_VARCHAR, ac, bop, an, bnl, rn0, n),
                lambda bop=bop, bnl=bnl, n=n: ops.str_compare_device(1, capi.T_VARCHAR, D(ac), D(bop), n, dev.buf(n), dev.buf(8 * ((n + 63) // 64)), D(an), D(bnl)),
                free={0})
        add("str_compare_lists_n%d" % n, lambda: ops.str_compare(0, capi.T_TEXT, a, b))
        for pat in (b"%ab_c%", [b"%a"] * max(n, 1)):
            add("like_n%d_%s" % (n, type(pat).__name__), lambda pat=pat, n=n: ops.like(ac, pat, an, None, None, n),
                lambda pat=pat, n=n: ops.like_device(D(ac), pat if isinstance(pat, bytes) else D(pat), n, dev.buf(n), dev.buf(8 * ((n + 63) // 64)), D(an)),
                free={0})
        add("like_hostpattern_n%d" % n, lambda n=n: ops.like(ac, varlena_bytes_column([b"x%"]), an, _words(1, 26), None, n),
            lambda n=n: ops.like_device(D(ac), varlena_bytes_column([b"x%"]), n, dev.buf(n), dev.buf(8 * ((n + 63) // 64)), D(an), _words(1, 26)), free={0})
        fx = rng.integers(0, 9, n).astype(np.int32)
        vals = np.array([1, 4, 7], np.int32)
        for T, col, vs, cn in ((capi.T_INT32, fx, vals, an), (capi.T_INT32, np.array([4], np.int32), vals, None),
                               (capi.T_VARCHAR, ac, varlena_bytes_column([b"ab", b"x" * 30]), an), (capi.T_UUID, rng.integers(0, 9, (n, 2)).astype(np.uint64),
                                                                                                      np.zeros((2, 2), np.uint64), None)):
            for neg in (False, True):
                add("in_%d_n%d_%d_%d" % (T, n, len(col if not isinstance(col, tuple) else col[0]), neg),
                    lambda T=T, col=col, vs=vs, cn=cn, neg=neg, n=n: ops.go_in(T, col, vs, neg, cn, _words(2, 27), rn0, n),
                    lambda T=T, col=col, vs=vs, cn=cn, neg=neg, n=n: ops.go_in_device(
                        T, D(col), D(vs), len(vs[0]) // 24 if isinstance(vs, tuple) else len(vs), n, dev.buf(n), dev.buf(8 * ((n + 63) // 64)), neg, D(cn),
                        D(_words(2, 27))), free={0})
        add("in_lists_n%d" % n, lambda: ops.go_in(capi.T_TEXT, a, [b"x", b""]))

        # CASE / IF / COALESCE
        c1, c2 = (rng.integers(0, 2, n).astype(bool), an), (np.array([True]), None)
        iv = [(rng.integers(0, 9, n).astype(np.int64), bn), (np.array([5], np.int64), None)]
        sv = [(ac, an), ((bc[0], None), None), (varlena_bytes_column([b"else-value-longer-than-23-bytes"]), None)]
        for T, vs, area_cap in ((capi.T_INT64, iv, None), (capi.T_DECIMAL128, [(np.zeros((n, 2), np.uint64), None), (np.ones((1, 2), np.uint64), None)], None),
                                (capi.T_VARCHAR, sv[:2], 40 * n), (capi.T_TEXT, sv, None)):
            def dv(op):
                return (D(op[0]), D(op[1]))
            els = vs[2] if len(vs) > 2 else vs[1]
            sres = T in ops.CASE_STR_TYPES
            add("case_%d_n%d" % (T, n), lambda T=T, vs=vs, els=els, n=n, ac_=area_cap: ops.go_case(T, [c1, c2], vs[:2], els, rn0, n, ac_),
                lambda T=T, vs=vs, els=els, n=n, sres=sres: ops.go_case_device(T, [dv(c1), dv(c2)], [dv(v) for v in vs[:2]], dv(els), n,
                                                                                 dev.buf((24 if sres else 16) * n), dev.buf(8 * ((n + 63) // 64)),
                                                                                 dev.buf(40 * n) if sres else None), free={0} if sres or T == capi.T_DECIMAL128 else ())
            add("case_noelse_%d_n%d" % (T, n), lambda T=T, vs=vs, n=n: ops.go_case(T, [c1], vs[:1], None, None, n, 40 * n),
                lambda T=T, vs=vs, n=n, sres=sres: ops.go_case_device(T, [dv(c1)], [dv(vs[0])], None, n, dev.buf((24 if sres else 16) * n),
                                                           dev.buf(8 * ((n + 63) // 64)), dev.buf(40 * n) if sres else None), free={0})
            add("iff_%d_n%d" % (T, n), lambda T=T, vs=vs, n=n: ops.go_iff(T, c1, vs[0], vs[1], None, n, 40 * n))
            add("coalesce_%d_n%d" % (T, n), lambda T=T, vs=vs, n=n: ops.go_coalesce(T, vs, rn0, n, 40 * n),
                lambda T=T, vs=vs, n=n, sres=sres: ops.go_coalesce_device(T, [dv(v) for v in vs], n, dev.buf((24 if sres else 16) * n), dev.buf(8 * ((n + 63) // 64)),
                                                               dev.buf(40 * n) if sres else None), free={0})
        add("coalesce_nolen_n%d" % n, lambda: ops.go_coalesce(capi.T_INT64, iv))
        rem = _words(n, 28)
        for cond, cnl in ((rng.integers(0, 2, n).astype(bool), an), (np.array([True]), None)):
            add("case_select_n%d_c%d" % (n, len(cond)), lambda cond=cond, cnl=cnl, n=n: ops.case_select(rem, cond, cnl, n),
                lambda cond=cond, cnl=cnl, n=n: ops.case_select_device(D(rem), D(rem), D(cond), D(cnl), n), free={0, 1})
    for n in (0, 1, 25):
        _block8(n)
    return out


def record(fn, rec):
    rec.calls.clear()
    fn()
    return list(rec.calls)


@pytest.fixture
def harness(monkeypatch):
    dev = FakeDevice()
    rec = Recorder(dev)
    monkeypatch.setattr(ops, "xcall", rec)
    return dev, rec


def test_every_case_reaches_xcall(harness):
    dev, rec = harness
    for name, host, device, _ in cases(dev, rec):
        for fn in (host, device):
            if fn is not None:
                assert record(fn, rec), name


def _shape(slot):
    """what both forms must agree on: a host area of 0 bytes passes no pointer, a device area its address (the library reads neither)"""
    data_sz, _, area_sz, pdata, pnulls, parea = slot
    return data_sz, area_sz, pdata is not None, pnulls is not None, parea is not None and area_sz > 0


def test_host_and_device_forms_hand_the_library_the_same_arguments(harness):
    dev, rec = harness
    pairs, bad = 0, []
    for name, host, device, free in cases(dev, rec):
        if host is None or device is None:
            continue
        h, d = record(host, rec), record(device, rec)
        assert len(h) == len(d), name
        for (hf, hn, hs), (df, dn, ds) in zip(h, d):
            assert (hf, hn, len(hs)) == (df, dn, len(ds)), name
            for i, (a, b) in enumerate(zip(hs, ds)):
                if i not in free and _shape(a) != _shape(b):
                    bad.append((name, i, _shape(a), _shape(b)))
            for a, b in zip(hs, ds):            # every pointer of the device form is a device address or a host parameter block
                for p in b[3:]:
                    assert p is None or p[0] in ("dev", "host")
        pairs += 1
    assert not bad
    assert pairs > 150


def test_one_row_operands_and_empty_columns(harness):
    dev, rec = harness
    (call,) = record(lambda: ops.dec_compare(0, 64, np.arange(3, dtype=np.int64), np.array([2], np.int64), 2, 2, 3), rec)
    assert [s[0] for s in call[2]] == [3, 24, 8, C.sizeof(capi.DecParams)]         # the const operand is one element's bytes
    (call,) = record(lambda: ops.dec_compare_device(0, 64, dev.buf(24), dev.buf(8), 2, 2, 3, dev.buf(3), dev.buf(8)), rec)
    assert [s[0] for s in call[2]] == [3, 24, 8, C.sizeof(capi.DecParams)]
    (call,) = record(lambda: ops.str_compare(0, capi.T_VARCHAR, [b"a"], [b"b"]), rec)
    assert call[1] == 1 and [s[0] for s in call[2]] == [1, 24, 24]                   # at len 1, a one-cell operand is a column of one
    (call,) = record(lambda: ops.str_compare_device(0, capi.T_VARCHAR, (dev.buf(24), dev.buf(0)), (dev.buf(24), None), 1, dev.buf(1), dev.buf(8)), rec)
    assert call[2][1][5] is not None and call[2][1][2] == 0 and call[2][2][5] is None  # a device area passes its pointer even when empty
    (call,) = record(lambda: ops.str_compare(0, capi.T_VARCHAR, [b"a"], [b"b"]), rec)
    assert call[2][1][5] is None                                                     # an empty host area passes none
    (call,) = record(lambda: ops.filter_sels(np.zeros(0, np.uint8)), rec)
    assert call[1] == 0 and call[2][2][0] == 0
