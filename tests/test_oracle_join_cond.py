"""The host restatement of the hash join with a non-equality condition (join_cond_reference) against itself and against the equality-only
restatement (join_outer_reference): row loop == numpy form, always-true == the equality join, always-false == nothing matched, a build-only
condition == the equality join over the filtered build side, probe batches sharing one bitmap, and hand-worked pair lists."""
import numpy as np
import pytest

import join_cond_reference as C
import join_outer_reference as J
from matrixone_b200 import capi

ALL_TYPES = tuple(J.FLAVOUR)
UNMATCHED_ALL = (capi.JOIN_LEFT, capi.JOIN_ANTI, capi.JOIN_SINGLE, capi.JOIN_FULL)


def case(seed, nbuild, nprobe, card, unique):
    r = np.random.default_rng(seed)
    if unique:
        build = r.permutation(2 * nbuild)[:nbuild].astype(np.uint64)
        bnull = np.zeros(nbuild, bool)
    else:
        build = r.integers(0, card, nbuild).astype(np.uint64)
        bnull = r.random(nbuild) < 0.05
    probe = r.integers(0, (2 * nbuild) if unique else card + card // 4 + 1, nprobe).astype(np.uint64)
    _, tk, off, sels = J.build_map(build, bnull)
    vals = J.find(tk, probe, r.random(nprobe) < 0.05)
    return build, bnull, vals, off, sels


def candidates(vals, off, sels):
    return J.probe(vals, off, sels, capi.JOIN_INNER)


def run(fn, *a):
    """the result, or the SingleError raised, with the bitmap it leaves"""
    try:
        return fn(*a)
    except J.SingleError as e:
        return ("error", e.probe_row, e.build_row)


def same(a, b):
    if isinstance(a, tuple) and a and isinstance(a[0], str):
        return a == b
    return not (isinstance(b, tuple) and b and isinstance(b[0], str)) and np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def both(vals, off, sels, jt, cond, null, nbuild, batch_size=C.DEFAULT_BATCH_SIZE):
    """row loop and numpy form on the same batch: equal results and bitmaps; returns (result, bitmap)"""
    cp, cb = candidates(vals, off, sels)
    c3 = [None if n else bool(x) for x, n in zip(cond, null)]
    m1, m2 = np.zeros(nbuild, bool), np.zeros(nbuild, bool)
    r1 = run(C.probe, vals, off, sels, jt, c3, m1, batch_size)
    r2 = run(C.probe_fast, cp, cb, cond, null, len(vals), jt, m2)
    assert same(r1, r2), (jt, r1, r2)
    if not isinstance(r1[0], str):
        assert np.array_equal(m1, m2)
    return r1, m1


@pytest.mark.parametrize("jt", ALL_TYPES)
@pytest.mark.parametrize("unique", [False, True])
@pytest.mark.parametrize("rate", [0.0, 0.01, 0.5, 1.0])
def test_row_loop_equals_numpy(jt, unique, rate):
    build, bnull, vals, off, sels = case(jt * 11 + int(rate * 100) + unique, 400, 900, 150, unique)
    cp, _ = candidates(vals, off, sels)
    r = np.random.default_rng(jt)
    cond = r.random(len(cp)) < rate
    null = r.random(len(cp)) < 0.1
    for bs in (C.DEFAULT_BATCH_SIZE, 7, 1):              # chunking of a row's sels into result batches changes nothing
        both(vals, off, sels, jt, cond, null, len(build), bs)


@pytest.mark.parametrize("jt", ALL_TYPES)
@pytest.mark.parametrize("unique", [False, True])
def test_always_true_is_the_equality_join(jt, unique):
    build, bnull, vals, off, sels = case(jt + 100 * unique, 300, 700, 120, unique)
    cp, _ = candidates(vals, off, sels)
    got, gm = both(vals, off, sels, jt, np.ones(len(cp), bool), np.zeros(len(cp), bool), len(build))
    wm = np.zeros(len(build), bool)
    want = run(J.probe, vals, off, sels, jt, wm)
    assert same(got, want)
    if not isinstance(want[0], str):
        assert np.array_equal(gm, wm)


@pytest.mark.parametrize("jt", ALL_TYPES)
@pytest.mark.parametrize("unique", [False, True])
def test_always_false_matches_nothing(jt, unique):
    build, bnull, vals, off, sels = case(jt + 7, 300, 500, 100, unique)
    cp, _ = candidates(vals, off, sels)
    (p, b), m = both(vals, off, sels, jt, np.zeros(len(cp), bool), np.zeros(len(cp), bool), len(build))
    if jt in UNMATCHED_ALL:
        assert p.tolist() == list(range(len(vals))) and (b == -1).all()
    else:
        assert len(p) == 0 and len(b) == 0
    assert not m.any()


@pytest.mark.parametrize("jt", ALL_TYPES)
@pytest.mark.parametrize("unique", [False, True])
def test_build_only_condition_is_the_filtered_build_side(jt, unique):
    """a condition on build columns only == the equality join against the build rows it keeps (the others take part as NULL keys)"""
    build, bnull, vals, off, sels = case(jt + 31, 500, 1200, 90, unique)
    keep = np.random.default_rng(jt).random(len(build)) < 0.6
    cp, cb = candidates(vals, off, sels)
    got, gm = both(vals, off, sels, jt, keep[cb], np.zeros(len(cp), bool), len(build))
    _, tk1, _, _ = J.build_map(build, bnull)
    _, tk2, off2, sels2 = J.build_map(build, bnull | ~keep)
    keys = np.where(vals > 0, tk1[np.maximum(vals.astype(np.int64) - 1, 0)], 0).astype(np.uint64)   # the probe keys again, by group id
    vals2 = J.find(tk2, keys, vals == 0)
    wm = np.zeros(len(build), bool)
    want = run(J.probe, vals2, off2, sels2, jt, wm)
    assert same(got, want)
    if not isinstance(want[0], str):
        assert np.array_equal(gm, wm)


@pytest.mark.parametrize("jt", [capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_RIGHT_SEMI, capi.JOIN_RIGHT_ANTI, capi.JOIN_INNER, capi.JOIN_LEFT])
@pytest.mark.parametrize("nbatch", [1, 3, 17])
def test_probe_batches_share_one_bitmap(jt, nbatch):
    build, bnull, vals, off, sels = case(nbatch, 600, 2000, 200, False)
    cp, cb = candidates(vals, off, sels)
    r = np.random.default_rng(nbatch)
    cond, null = r.random(len(cp)) < 0.4, r.random(len(cp)) < 0.1
    want, wm = both(vals, off, sels, jt, cond, null, len(build))
    m = np.zeros(len(build), bool)
    cuts = np.linspace(0, len(vals), nbatch + 1).astype(int)
    gp, gb = [], []
    for a, z in zip(cuts[:-1], cuts[1:]):
        sel = (cp >= a) & (cp < z)
        p, b = C.probe_fast(cp[sel] - a, cb[sel], cond[sel], null[sel], z - a, jt, m)
        gp.append(p + a); gb.append(b)
    assert np.array_equal(np.concatenate(gp), want[0]) and np.array_equal(np.concatenate(gb), want[1]) and np.array_equal(m, wm)
    if jt in J.RIGHT_TYPES:
        assert np.array_equal(J.finalize(m, jt), J.finalize(wm, jt))


# ---- hand-worked: build keys [10, 20, 20, 30, 30, 30], probe keys [20, 99, 30, 10, 20]; INNER candidates in order
#   k: 0      1      2      3      4      5      6      7
#      (0,1)  (0,2)  (2,3)  (2,4)  (2,5)  (3,0)  (4,1)  (4,2)
#   cond: F    T      None   T      F      None   T      T
HAND_BUILD = np.array([10, 20, 20, 30, 30, 30], np.uint64)
HAND_PROBE = np.array([20, 99, 30, 10, 20], np.uint64)
HAND_COND = [False, True, None, True, False, None, True, True]
HAND_WANT = {
    capi.JOIN_INNER: ([0, 2, 4, 4], [2, 4, 1, 2]),
    capi.JOIN_LEFT: ([0, 1, 2, 3, 4, 4], [2, -1, 4, -1, 1, 2]),
    capi.JOIN_SEMI: ([0, 2, 4], [-1, -1, -1]),
    capi.JOIN_ANTI: ([1, 3], [-1, -1]),
    capi.JOIN_SINGLE: ("error", 4, None),               # probe row 4 has two passing pairs
    capi.JOIN_RIGHT: ([0, 2, 4, 4], [2, 4, 1, 2]),
    capi.JOIN_FULL: ([0, 1, 2, 3, 4, 4], [2, -1, 4, -1, 1, 2]),
    capi.JOIN_RIGHT_SEMI: ([], []),
    capi.JOIN_RIGHT_ANTI: ([], []),
    capi.JOIN_RIGHT_SINGLE: ("error", None, 2),         # build row 2 is passed by probe rows 0 and 4
}


@pytest.mark.parametrize("jt", ALL_TYPES)
def test_hand_worked(jt):
    _, tk, off, sels = J.build_map(HAND_BUILD)
    vals = J.find(tk, HAND_PROBE)
    cp, cb = candidates(vals, off, sels)
    assert cp.tolist() == [0, 0, 2, 2, 2, 3, 4, 4] and cb.tolist() == [1, 2, 3, 4, 5, 0, 1, 2]
    m = np.zeros(6, bool)
    got = run(C.probe, vals, off, sels, jt, HAND_COND, m)
    want = HAND_WANT[jt]
    if isinstance(want[0], str):
        assert got == want
    else:
        assert got[0].tolist() == want[0] and got[1].tolist() == want[1]
        if jt in J.RIGHT_TYPES:
            assert np.flatnonzero(m).tolist() == [1, 2, 4]
    cond = np.array([bool(c) for c in HAND_COND])
    null = np.array([c is None for c in HAND_COND])
    got2 = run(C.probe_fast, cp, cb, cond, null, len(vals), jt, np.zeros(6, bool))
    assert same(got, got2)


def test_left_single_fails_only_on_two_passing_pairs():
    _, tk, off, sels = J.build_map(HAND_BUILD)
    vals = J.find(tk, HAND_PROBE)
    cond = [False, True, None, True, False, None, True, False]      # every row at most one passing pair: no failure
    p, b = C.probe(vals, off, sels, capi.JOIN_SINGLE, cond)
    assert p.tolist() == [0, 1, 2, 3, 4] and b.tolist() == [2, -1, 4, -1, 1]


def test_unique_map_path():
    """HashOnUnique: one candidate per matched row; a failing condition makes the row unmatched"""
    _, tk, off, sels = J.build_map(np.array([5, 6, 7], np.uint64))
    assert off is None
    vals = J.find(tk, np.array([7, 8, 5, 6], np.uint64))
    cond = [True, None, False]                                        # (0,2) (2,0) (3,1)
    assert [x.tolist() for x in C.probe(vals, off, sels, capi.JOIN_LEFT, cond)] == [[0, 1, 2, 3], [2, -1, -1, -1]]
    assert [x.tolist() for x in C.probe(vals, off, sels, capi.JOIN_ANTI, cond)] == [[1, 2, 3], [-1, -1, -1]]
    m = np.zeros(3, bool)
    assert [x.tolist() for x in C.probe(vals, off, sels, capi.JOIN_RIGHT_SEMI, cond, m)] == [[], []] and m.tolist() == [False, False, True]


def test_q21_fixture():
    """tests/golden/tpch_q21.json: the row counts of 10_select_count.result, and the Q21 subquery counts of a nested loop over its rows"""
    import json
    import os
    d = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tpch_q21.json")))
    assert d["counts"] == {"lineitem": 6005, "orders": 1500, "supplier": 10, "nation": 25}
    assert [len(d[k]) for k in ("l_orderkey", "l_suppkey", "l_commitdate", "l_receiptdate")] == [6005] * 4
    assert (len(d["o_orderkey"]), len(d["o_orderstatus"]), len(d["s_suppkey"]), len(d["n_name"])) == (1500, 1500, 10, 25)
    okey, supp = np.array(d["l_orderkey"]), np.array(d["l_suppkey"])
    late = np.array(d["l_receiptdate"]) > np.array(d["l_commitdate"])
    same, other = okey[:, None] == okey[None, :], supp[:, None] != supp[None, :]
    exists, not_exists = (same & other).any(1), ~(same & other & late[None, :]).any(1)
    assert (late.sum(), same[late].sum(), (late & exists & not_exists).sum()) == (3752, 18788, 307)
