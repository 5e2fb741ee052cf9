"""Plain reference for the vector-search tests (no GPU): float64 distances, an exactness check of a top-k result, and a
restatement of the error bound of the tensor-core candidate pass (csrc/tcsearch.cu, tc_eps) together with a worst-case model
of that pass.

The model is a statement about what the bound has to cover, not a claim about the hardware: it splits the operands like
split_kernel (bf16 round-to-nearest-even hi part, bf16 residual lo part), multiplies exactly (in float64), and accumulates in
fp32 the way the H100 tensor cores were measured to behave, taken at its worst (test_gpu_tcsearch_exact.py,
hidden_neighbour_data): in every k16 step the 16 products are aligned to the largest term among them and the running sum and
TRUNCATED at that term's last fp32 bit (the hardware keeps fewer than 3 extra bits; the model keeps none), added exactly, and
the sum is ROUNDED TOWARD ZERO -- errors that do not cancel on data with same-sign products."""
import numpy as np
import torch

import oracle_lib as O
from matrixone_b200 import capi

F32 = np.float32
U23 = 2.0 ** -23


# ---- float64 distances -------------------------------------------------------------------------------------------------
def exact_dists(ds, qs, metric, block=256, rblock=4096):
    """float64 distance [nq, n] from the fp32 inputs: L2 / L2SQ squared distance, IP -q.x, COS 1 - cos (by blocks of queries
    and rows)"""
    qs = np.asarray(qs, dtype=np.float64)
    out = np.empty((qs.shape[0], ds.shape[0]))
    qn = (qs * qs).sum(axis=1)
    for r0 in range(0, ds.shape[0], rblock):
        x = np.asarray(ds[r0:r0 + rblock], dtype=np.float64)
        xn = (x * x).sum(axis=1)
        for q0 in range(0, qs.shape[0], block):
            dot = qs[q0:q0 + block] @ x.T
            o = out[q0:q0 + block, r0:r0 + rblock]
            if metric == capi.METRIC_IP:
                o[:] = -dot
            elif metric == capi.METRIC_COS:
                den = np.sqrt(qn[q0:q0 + block])[:, None] * np.sqrt(xn)[None, :]
                with np.errstate(invalid="ignore", divide="ignore"):
                    o[:] = np.where(den > 0, 1.0 - np.clip(dot / den, -1.0, 1.0), 1.0)
            else:
                o[:] = qn[q0:q0 + block, None] + xn[None, :] - 2.0 * dot
    return out


def exact_l2_rows(ds, q, rows):
    """squared distances of q to ds[rows] by differences (no cancellation)"""
    diff = np.asarray(ds[rows], dtype=np.float64) - np.asarray(q, dtype=np.float64)[None, :]
    return (diff * diff).sum(axis=1)


def go_error(metric, dim, d, qnorm2, xmax2):
    """|Go-order fp32 value - real value| bound, as tc_final_kernel prices it: relative dim 2^-23 for L2, dim 2^-23 |q||x|max for
    the inner product, dim 2^-22 + 2^-19 for cosine"""
    if metric == capi.METRIC_IP:
        return dim * U23 * np.sqrt(qnorm2 * xmax2)
    if metric == capi.METRIC_COS:
        return dim * 2 * U23 + 2.0 ** -19
    return dim * U23 * abs(d)


# ---- exactness of a top-k result -----------------------------------------------------------------------------------------
def check_exact_topk(keys, dists, ds, qs, k, metric=capi.METRIC_L2, key_base=0, oracle=None, allowed=None, sqrt_out=False,
                     key_of_row=None, nthreads=8):
    """A search result must be the exact answer:
      * distances bit-equal to the Go-order oracle (O.bruteforce, or `oracle` = (keys, dists) of og_ivf_search_f32);
      * keys equal to the oracle's except among exact oracle ties; inside a tie the lower key comes first, and a tie cut by the
        k-th place keeps the lowest keys;
      * independently of the oracle, in float64: every returned row is within the Go-order error of the k-th distance, every row
        not returned is no closer than the k-th distance minus that error, and each returned distance is its row's.
    allowed[q] = row indices query q may return (IVF: rows of the probed lists); key_of_row maps a row index to its key
    (IVF row ids); keys are row + key_base otherwise."""
    ds = np.asarray(ds, dtype=np.float32); qs = np.asarray(qs, dtype=np.float32)
    n, dim = ds.shape
    nq = qs.shape[0]
    keys = np.asarray(keys).reshape(nq, k); dists = np.asarray(dists).reshape(nq, k)
    if oracle is None:
        kk = min(n, k + 8)        # a few places past k: ties across the k-th place are visible
        ok, od = O.bruteforce(ds, qs, kk, metric, nthreads=nthreads)
        ok = ok.reshape(nq, kk); od = od.reshape(nq, kk)
    else:
        kk = k
        ok = np.asarray(oracle[0]).reshape(nq, k); od = np.asarray(oracle[1]).reshape(nq, k)
    bad_d = np.flatnonzero((dists != od[:, :k]).any(axis=1))
    assert bad_d.size == 0, ("distances differ from the oracle", bad_d[:8], dists[bad_d[0]], od[bad_d[0], :k])
    if key_of_row is None:
        to_key = lambda r: np.where(r >= 0, r + key_base, -1)
    else:
        kor = np.asarray(key_of_row)
        to_key = lambda r: np.where(r >= 0, kor[np.maximum(r, 0)], -1)
    okeys = to_key(ok) if oracle is None else ok
    row_of_key = None
    if key_of_row is not None:
        row_of_key = {int(v): i for i, v in enumerate(key_of_row)}
    xn = np.concatenate([(np.asarray(ds[r0:r0 + 4096], dtype=np.float64) ** 2).sum(axis=1) for r0 in range(0, n, 4096)])
    dfull = exact_dists(ds, qs, metric) if allowed is None else None
    for q in range(nq):
        kq, dq, oq, odq = keys[q], dists[q], okeys[q], od[q]
        # ties: equal distances come in ascending key order
        for j in range(1, k):
            if kq[j - 1] >= 0 and dq[j] == dq[j - 1]:
                assert kq[j] > kq[j - 1], ("tie not in key order", q, j, kq)
        for j in np.flatnonzero(kq != oq[:k]):
            tied = odq == odq[j]
            assert tied.sum() > 1, ("key differs where the oracle has no tie", q, j, kq[j], oq[j])
            if oracle is None and not (tied[-1] and kk < n):
                # every oracle row at this distance is in view: the result holds the lowest keys of the tie, in order
                ties = np.sort(oq[tied])
                got = kq[:k][dq[:k] == odq[j]]
                assert (got == ties[:got.size]).all(), ("tie not resolved to the lowest keys", q, got, ties)
        # float64 check, oracle-free
        rows_ok = np.arange(n) if allowed is None else np.sort(np.asarray(allowed[q], dtype=np.int64))
        valid = kq >= 0
        assert valid.sum() == min(k, rows_ok.size), ("wrong number of results", q, kq)
        assert not valid[:k - valid.sum()].any(), ("padding must come first", q, kq)
        if rows_ok.size == 0:
            continue
        if row_of_key is None:
            ret = kq[valid] - key_base
        else:
            ret = np.asarray([row_of_key[int(v)] for v in kq[valid]], dtype=np.int64)
        assert np.isin(ret, rows_ok).all(), ("a returned row is not a candidate of this query", q, ret)
        qn2 = float((qs[q].astype(np.float64) ** 2).sum())
        xm2 = float(xn[rows_ok].max())
        dall = _row_dists(ds, xn, qs[q], qn2, rows_ok, metric, k, None if dfull is None else dfull[q].copy())
        kth = np.partition(dall, min(k, dall.size) - 1)[min(k, dall.size) - 1]
        # a returned row's Go value is <= the k-th Go value <= kth + err, and each Go value is within err of its real value
        err = 2 * go_error(metric, dim, kth, qn2, xm2) * (1 + 1e-6) + 1e-300
        at = np.searchsorted(rows_ok, ret)           # rows_ok is ascending
        dret = dall[at]
        assert (dret <= kth + err).all(), ("returned row farther than the k-th", q, ret, dret, kth, err)
        rest = np.ones(rows_ok.size, dtype=bool); rest[at] = False
        if rest.any():
            assert dall[rest].min() >= kth - err, ("a row not returned is closer than the k-th", q, rows_ok[rest][np.argmin(dall[rest])],
                                                   dall[rest].min(), kth, err)
        got = dq[valid] ** 2 if sqrt_out else dq[valid]
        tol = go_error(metric, dim, dret, qn2, xm2) * (1 + 1e-6) + (4 * U23 * np.abs(dret) if sqrt_out else 0) + 1e-300
        assert (np.abs(got - dret) <= tol).all(), ("returned distance is not its row's", q, got, dret)


def _row_dists(ds, xn, q, qn2, rows, metric, k, d=None):
    """float64 distances of q to ds[rows] (d: already computed by exact_dists); L2 by the norm expansion, then by differences
    wherever the expansion's cancellation error could matter for the k nearest"""
    if d is None:
        d = exact_dists(ds[rows], q[None, :], metric)[0]
    if metric not in (capi.METRIC_L2, capi.METRIC_L2SQ):
        return d
    dim = ds.shape[1]
    experr = 2 * (dim + 2) * 2.0 ** -53 * (qn2 + xn[rows])
    kk = min(k, d.size) - 1
    lim = np.partition(d, kk)[kk] + 2 * experr.max() + 4 * dim * U23 * abs(np.partition(d, kk)[kk]) + 1e-300
    close = np.flatnonzero(d - experr <= lim)
    for c0 in range(0, close.size, 4096):
        c = close[c0:c0 + 4096]
        d[c] = exact_l2_rows(ds, q, rows[c])
    return d


# ---- the candidate pass: bound and model -------------------------------------------------------------------------------
def kprime(dim):
    """K' of the split operands: [hi | hi | lo] . [hi | lo | hi], padded to whole 64-column k-blocks"""
    return (3 * dim + 63) // 64 * 64


def pass_kblocks(dim, one_term):
    """64-column k-blocks a candidate pass runs: the hi.hi columns only, or the whole K'"""
    return (dim + 63) // 64 if one_term else kprime(dim) // 64


def tc_eps(qn, ql, xm, xl, one_term, nkb):
    """tcsearch.cu tc_eps, in fp32 operation by operation: the bound on |approximate - real| squared distance of a pair"""
    qn, ql, xm, xl = (np.asarray(v, dtype=F32) for v in (qn, ql, xm, xl))
    acc = F32(4 * nkb) * F32(4.0531158447265625e-6)   # 34 steps 2^-23
    norms = F32(9.5367431640625e-7) * (qn + xm)
    if one_term:
        split = F32(2.002) * (root_mul(qn, xl) + root_mul(ql, xm) + F32(3.0) * root_mul(ql, xl))
        return split + np.maximum(F32(1.52587890625e-5), acc) * root_mul(qn, xm) + norms
    return np.maximum(F32(2.44140625e-4), F32(9.1552734375e-5) + acc) * root_mul(qn, xm) + norms


def root_mul(a, b):
    """tcsearch.cu root_mul: sqrt(a b) in fp32, as sqrt(a) sqrt(b) where a b is outside [1e-30, 1e30]"""
    with np.errstate(over="ignore", under="ignore"):
        p = a * b
        return np.where((p >= F32(1e-30)) & (p <= F32(1e30)), np.sqrt(p), np.sqrt(a) * np.sqrt(b)).astype(F32)


def tc_eps_fixed_steps(qn, ql, xm, xl, one_term):
    """the bound as it was before it depended on the pass length: accumulation priced for dim 768 (three-term) and
    64 k16 steps (one-term)"""
    qn, ql, xm, xl = (np.asarray(v, dtype=F32) for v in (qn, ql, xm, xl))
    norms = F32(9.5367431640625e-7) * (qn + xm)
    if one_term:
        split = F32(2.002) * (np.sqrt(qn * xl) + np.sqrt(ql * xm) + F32(3.0) * np.sqrt(ql * xl))
        return split + F32(1.52587890625e-5) * np.sqrt(qn * xm) + norms
    return F32(2.44140625e-4) * np.sqrt(qn * xm) + norms


def bf16_split(x):
    """hi = bf16(x) (round to nearest even), lo = bf16(x - hi); x - hi is exact in fp32"""
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=F32))
    hi = t.to(torch.bfloat16).to(torch.float32)
    lo = (t - hi).to(torch.bfloat16).to(torch.float32)
    return hi.numpy().astype(np.float64), lo.numpy().astype(np.float64)


def round_toward_zero_f32(v):
    """float64 -> the fp32 value next to it on the side of zero"""
    v = np.asarray(v, dtype=np.float64)
    f = v.astype(F32)
    over = np.abs(f.astype(np.float64)) > np.abs(v)
    f[over] = np.nextafter(f[over], F32(0))
    return f


def operands(x, mode):
    """K' columns of split_kernel: mode 0 (queries) [hi | hi | lo], mode 1 (rows) [hi | lo | hi], zero padded; plus
    |x|^2 and |x - hi|^2 accumulated in float64 and rounded to fp32"""
    x = np.asarray(x, dtype=F32)
    m, dim = x.shape
    hi, lo = bf16_split(x)
    op = np.zeros((m, kprime(dim)))
    op[:, :dim] = hi
    op[:, dim:2 * dim] = hi if mode == 0 else lo
    op[:, 2 * dim:3 * dim] = lo if mode == 0 else hi
    x64 = x.astype(np.float64)
    norm = (x64 * x64).sum(axis=1).astype(F32)
    lonorm = ((x64 - hi) ** 2).sum(axis=1).astype(F32)
    return op, norm, lonorm


def candidate_pass_model(qs, xs, one_term):
    """approximate squared distance of each pair (qs[i], xs[i]) under the worst-case model, the real distance (float64) and
    tc_eps of the pair.  The pass runs 4 nkb k16 steps; after each the fp32 accumulator is rounded toward zero; the epilogue
    forms fma(-2, acc, fl(|q|^2 + |x|^2)) in fp32."""
    qs = np.asarray(qs, dtype=F32); xs = np.asarray(xs, dtype=F32)
    dim = qs.shape[1]
    a, qn, ql = operands(qs, 0)
    b, xn, xl = operands(xs, 1)
    nkb = pass_kblocks(dim, one_term)
    steps = 4 * nkb
    prod = (a[:, :64 * nkb] * b[:, :64 * nkb]).reshape(len(qs), steps, 16)   # products exact in float64
    acc = np.zeros(len(qs), dtype=F32)
    for s in range(steps):
        p = prod[:, s]
        top = np.maximum(np.abs(acc.astype(np.float64)), np.abs(p).max(axis=1))
        res = np.exp2(np.floor(np.log2(np.where(top > 0, top, 1.0))) - 23)          # the largest term's last fp32 bit
        p = np.trunc(p / res[:, None]) * res[:, None]
        acc = round_toward_zero_f32(acc.astype(np.float64) + p.sum(axis=1))
    base = (qn + xn).astype(np.float64)                                                 # fp32 add, round to nearest
    approx = (base - 2.0 * acc.astype(np.float64)).astype(F32).astype(np.float64)       # fma: one rounding
    real = ((qs.astype(np.float64) - xs.astype(np.float64)) ** 2).sum(axis=1)
    eps = tc_eps(qn, ql if one_term else 0.0, xn, xl if one_term else 0.0, one_term, nkb).astype(np.float64)
    return approx, real, eps


# ---- data -------------------------------------------------------------------------------------------------------------
TAIL = 181.0 * 2.0 ** -19      # bf16; its square is 2^-23 (1 - 7 2^-15): just under one ulp of an accumulator in [1, 2)
TAIL16 = {8: 255.0 * 2.0 ** -21,   # bf16; its square is 2^-26 (1 - 2^-7.98): just under an eighth of that ulp
          4: 181.0 * 2.0 ** -20}   # bf16; its square is 2^-25 (1 - 7 2^-15): just under a quarter of it


def lost_tail_rows(dim, head_block=0, per_step=1, frac=8):
    """a bf16-exact non-negative row whose products, multiplied with itself, lose the most under truncation: one k16 block of
    0.25 (its step brings the accumulator to 1.0) and, in every other k16 block,
      per_step=1:  one TAIL component -- the step adds just under one ulp: all of it lost if the step sum is truncated, none
                   of it if it is rounded to nearest;
      per_step=16: sixteen TAIL16[frac] components -- products of just under 1/frac ulp: truncated once, the exact step sum loses
                   one ulp; with every product truncated below 1/4 ulp first (the H100), all of them are lost: 16/frac ulps.
    tail = the tail components, ordered so that the first T of them lie in T different k16 blocks"""
    x = np.zeros(dim, dtype=F32)
    h0 = 16 * head_block
    x[h0:h0 + 16] = 0.25
    blocks = [c for c in range(0, dim - dim % 16, 16) if c != h0]
    if per_step == 1:
        tail = np.array(blocks, dtype=np.int64)
        x[tail] = TAIL
    else:
        tail = np.array([b + i for i in range(16) for b in blocks], dtype=np.int64)
        x[tail] = TAIL16[frac]
    return x, tail
