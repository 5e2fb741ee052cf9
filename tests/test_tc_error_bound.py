"""The error bound of the tensor-core candidate pass (tcsearch.cu tc_eps) against a worst-case model of the pass
(search_reference.candidate_pass_model: bf16 hi/lo split, exact products, fp32 accumulation rounded toward zero after every
k16 step).  The completeness proof of brute-force, IVF and centroid-probe searches is only as good as this bound."""
import numpy as np
import pytest

import search_reference as S

DIMS = [16, 17, 100, 768, 1024, 1536, 3072, 4096, 8192]
FAMILIES = ["gaussian", "nonneg", "bf16_nonneg", "wide_range", "lost_tail", "lost_tail16_8", "lost_tail16_4"]


def _bf16(x):
    hi, _ = S.bf16_split(x)
    return hi.astype(np.float32)


def pairs(family, dim, m=24, seed=0):
    """m (query, row) pairs; every family puts some rows next to their query, where |d~ - d| is the whole error"""
    rng = np.random.default_rng(seed + dim)
    if family == "gaussian":
        q = rng.standard_normal((m, dim)).astype(np.float32)
        x = rng.standard_normal((m, dim)).astype(np.float32)
        x[: m // 2] = q[: m // 2] + np.float32(1e-3) * rng.standard_normal((m // 2, dim)).astype(np.float32)
    elif family in ("nonneg", "bf16_nonneg"):
        q = rng.random((m, dim), dtype=np.float32)
        x = rng.random((m, dim), dtype=np.float32)
        x[: m // 2] = q[: m // 2] * np.float32(1.001)
        if family == "bf16_nonneg":
            q, x = _bf16(q), _bf16(x)
    elif family == "wide_range":
        # every component a random power of 2 between 2^-24 and 1 (times a random mantissa), the first k16 block the largest
        e = rng.uniform(-24, 0, (m, dim))
        e[:, :16] = 0
        q = (np.exp2(e) * rng.uniform(1, 2, (m, dim))).astype(np.float32)
        x = q.copy()
        x[m // 2:] = (q[m // 2:] * rng.uniform(0.99, 1.01, (m - m // 2, dim))).astype(np.float32)
    else:   # lost_tail(16): the constructions that lose the most under truncation, as their own query and next to it
        per_step, frac = (16, int(family[-1])) if family.startswith("lost_tail16") else (1, 8)
        rows = np.stack([S.lost_tail_rows(dim, h % max(1, dim // 16), per_step, frac)[0] for h in range(m)])
        q = rows
        x = rows.copy()
        x[m // 2:, 16:] = 0.0
    return q.astype(np.float32), x.astype(np.float32)


@pytest.mark.parametrize("one_term", [True, False], ids=["one_term", "three_term"])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("dim", DIMS)
def test_bound_covers_the_worst_case_model(dim, family, one_term):
    q, x = pairs(family, dim)
    approx, real, eps = S.candidate_pass_model(q, x, one_term)
    err = np.abs(approx - real)
    worst = int(np.argmax(err / eps))
    assert (err <= eps).all(), "dim %d: |d~ - d| = %.4g exceeds tc_eps = %.4g (%.3gx)" % (dim, err[worst], eps[worst], err[worst] / eps[worst])


@pytest.mark.parametrize("dim", [1536, 3072, 4096, 8192])
def test_fixed_step_bound_is_exceeded_at_large_dims(dim):
    """the model has teeth: the bound with accumulation priced for a fixed number of k16 steps fails on the one-term pass
    beyond 1024 columns, which is what the step-dependent bound repairs"""
    q, x = pairs("lost_tail16_8", dim)
    approx, real, _ = S.candidate_pass_model(q, x, True)
    a, qn, ql = S.operands(q, 0)
    b, xn, xl = S.operands(x, 1)
    old = S.tc_eps_fixed_steps(qn, ql, xn, xl, True).astype(np.float64)
    assert (np.abs(approx - real) > old).any()


@pytest.mark.parametrize("one_term", [True, False])
def test_bound_never_shrinks_and_is_unchanged_where_the_fixed_coefficient_covers_the_steps(one_term):
    """the step-dependent bound is never below the fixed-step one, and bit for bit equal to it for the three-term pass up to
    dim 192"""
    rng = np.random.default_rng(3)
    qn, ql, xm, xl = (np.exp2(rng.uniform(-24, 24, 1000)).astype(np.float32) for _ in range(4))
    old = S.tc_eps_fixed_steps(qn, ql, xm, xl, one_term)
    for dim in (16, 17, 64, 100, 129, 192, 320, 768, 1024, 4096):
        new = S.tc_eps(qn, ql, xm, xl, one_term, S.pass_kblocks(dim, one_term))
        assert (new >= old).all(), dim
        if not one_term and dim <= 192:
            assert (new.view(np.uint32) == old.view(np.uint32)).all(), dim


def test_round_toward_zero():
    v = np.array([1.0 + 2.0 ** -30, -(1.0 + 2.0 ** -30), 1.0 - 2.0 ** -30, 3.0, 0.0, 2.0 ** -149 * 1.5])
    r = S.round_toward_zero_f32(v)
    assert r.tolist() == [1.0, -1.0, float(np.nextafter(np.float32(1.0), np.float32(0))), 3.0, 0.0, 2.0 ** -149]


def test_lost_tail_rows_lose_their_tail_under_truncation_only():
    x, tail = S.lost_tail_rows(1024)
    assert (S.bf16_split(x[None, :])[1] == 0).all()              # bf16-exact: the lo part is zero
    assert float(S.TAIL) ** 2 < 2.0 ** -23
    # one-term model: the accumulator stays at 1.0 after the head step, so every tail step is lost
    approx, real, _ = S.candidate_pass_model(x[None, :], x[None, :], True)
    assert real[0] == 0.0
    assert abs(approx[0] - 2 * tail.size * float(S.TAIL) ** 2) <= 2.0 ** -21


@pytest.mark.parametrize("scale", [1e-36, 1e36])
def test_bound_keeps_its_size_where_the_norm_product_leaves_fp32(scale):
    """rows scaled by 1e-18 (|q|^2 |x|^2 underflows) or 1e18 (it overflows): the bound stays 2^-12 |q||x|, not 0 or inf"""
    n = np.float32(64 * scale)
    for one_term in (True, False):
        e = float(S.tc_eps(n, n * np.float32(2.0 ** -18), n, n * np.float32(2.0 ** -18), one_term, 1))
        assert np.isfinite(e) and 2.0 ** -17 * float(n) < e < 2.0 ** -5 * float(n), (one_term, e)
