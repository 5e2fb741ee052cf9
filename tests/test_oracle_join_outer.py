"""The host restatement of the right-flavoured and single hash joins (join_outer_reference): the reference's type table, hand-worked pair lists
for every new type, the set identities that tie them to INNER / LEFT, batch and worker splits, and the numpy form the GPU tests use."""
import numpy as np
import pytest

import join_outer_reference as J
from matrixone_b200 import capi

# TestHashJoinTypeCheckers (pkg/sql/colexec/hashjoin/join_test.go:332-440): (join type, IsRightJoin, the checks it pins)
TYPE_CHECKS = [
    ("INNER", False, {"IsInner": True, "IsLeftOuter": False, "IsRightOuter": False, "IsFullOuter": False, "IsSemi": False, "IsAnti": False,
                      "IsSingle": False, "EmitUnmatchedProbe": False, "EmitUnmatchedBuild": False}),
    ("LEFT", False, {"IsInner": False, "IsLeftOuter": True, "IsRightOuter": False, "EmitUnmatchedProbe": True, "EmitUnmatchedBuild": False}),
    ("RIGHT", True, {"IsInner": False, "IsLeftOuter": False, "IsRightOuter": True, "EmitUnmatchedProbe": False, "EmitUnmatchedBuild": True}),
    ("OUTER", True, {"IsFullOuter": True, "IsInner": False, "IsLeftOuter": False, "IsRightOuter": False, "IsLeftSemi": False, "IsRightSemi": False,
                     "IsLeftAnti": False, "IsRightAnti": False, "IsLeftSingle": False, "IsRightSingle": False,
                     "EmitUnmatchedProbe": True, "EmitUnmatchedBuild": True}),
    ("SEMI", False, {"IsSemi": True, "IsLeftSemi": True, "IsRightSemi": False}),
    ("SEMI", True, {"IsSemi": True, "IsLeftSemi": False, "IsRightSemi": True}),
    ("ANTI", False, {"IsAnti": True, "IsLeftAnti": True, "IsRightAnti": False}),
    ("ANTI", True, {"IsAnti": True, "IsLeftAnti": False, "IsRightAnti": True}),
    ("SINGLE", False, {"IsSingle": True, "IsLeftSingle": True, "IsRightSingle": False}),
    ("SINGLE", True, {"IsSingle": True, "IsLeftSingle": False, "IsRightSingle": True}),
]


@pytest.mark.parametrize("jt,right,checks", TYPE_CHECKS)
def test_type_table_is_the_references(jt, right, checks):
    h = J.Checkers(jt, right)
    for name, want in checks.items():
        assert getattr(h, name)() == want, (jt, right, name)


def test_every_type_maps_to_one_flavour():
    assert sorted(J.FLAVOUR.values()) == sorted((jt, r) for jt, r, _ in TYPE_CHECKS)
    for t in J.RIGHT_TYPES:
        assert J.checkers(t).EmitUnmatchedBuild()
    for t in (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI, capi.JOIN_SINGLE):
        assert not J.checkers(t).EmitUnmatchedBuild()


# ---- hand-worked: build keys 10 20 10 NULL 30 (rows 0..4), probe keys 10 NULL 40 30 20 (rows 0..4)
BUILD = np.array([10, 20, 10, 0, 30], np.uint64)
BNULL = np.array([0, 0, 0, 1, 0], bool)
PROBE = np.array([10, 0, 40, 30, 20], np.uint64)
PNULL = np.array([0, 1, 0, 0, 0], bool)


def run(build, bnull, probe_keys, pnull, jt, matched=None):
    _, tk, off, sels = J.build_map(build, bnull)
    vals = J.find(tk, probe_keys, pnull)
    m = np.zeros(len(build), bool) if matched is None else matched
    p, b = J.probe(vals, off, sels, jt, m)
    return list(zip(p.tolist(), b.tolist())), m


def test_map_of_the_hand_case():
    groups, tk, off, sels = J.build_map(BUILD, BNULL)
    assert groups.tolist() == [1, 2, 1, 0, 3] and tk.tolist() == [10, 20, 30]
    assert off.tolist() == [0, 2, 3, 4, 4] and sels.tolist() == [0, 2, 1, 4]


@pytest.mark.parametrize("jt,pairs,marked,final", [
    (capi.JOIN_RIGHT, [(0, 0), (0, 2), (3, 4), (4, 1)], [0, 1, 2, 4], [3]),
    (capi.JOIN_FULL, [(0, 0), (0, 2), (1, -1), (2, -1), (3, 4), (4, 1)], [0, 1, 2, 4], [3]),
    (capi.JOIN_RIGHT_SEMI, [], [0, 1, 2, 4], [0, 1, 2, 4]),
    (capi.JOIN_RIGHT_ANTI, [], [0, 1, 2, 4], [3]),
    (capi.JOIN_RIGHT_SINGLE, [(0, 0), (0, 2), (3, 4), (4, 1)], [0, 1, 2, 4], [3]),
])
def test_hand_worked_right_types(jt, pairs, marked, final):
    got, m = run(BUILD, BNULL, PROBE, PNULL, jt)
    assert got == pairs and np.flatnonzero(m).tolist() == marked
    assert J.finalize(m, jt).tolist() == final                          # the NULL-key build row 3 is never matched


def test_hand_worked_left_single():
    with pytest.raises(J.SingleError) as e:                              # key 10 has two build rows
        run(BUILD, BNULL, PROBE, PNULL, capi.JOIN_SINGLE)
    assert e.value.probe_row == 0
    pk = np.array([20, 0, 40, 30, 30], np.uint64)
    got, m = run(BUILD, BNULL, pk, PNULL, capi.JOIN_SINGLE)
    assert got == [(0, 1), (1, -1), (2, -1), (3, 4), (4, 4)] and not m.any()


def test_hand_worked_right_single_fails_on_a_second_match():
    pk = np.array([20, 30, 20], np.uint64)                               # build row 1 matched twice
    with pytest.raises(J.SingleError) as e:
        run(BUILD, BNULL, pk, None, capi.JOIN_RIGHT_SINGLE)
    assert e.value.build_row == 1
    m = np.zeros(5, bool)
    run(BUILD, BNULL, pk[:1], None, capi.JOIN_RIGHT_SINGLE, m)           # ... or across batches
    with pytest.raises(J.SingleError) as e:
        run(BUILD, BNULL, pk[2:], None, capi.JOIN_RIGHT_SINGLE, m)
    assert e.value.build_row == 1


def test_hand_worked_unique_map():
    build = np.array([7, 5, 9], np.uint64)
    _, tk, off, sels = J.build_map(build)
    assert off is None and sels is None
    got, m = run(build, None, np.array([9, 9, 4, 5], np.uint64), None, capi.JOIN_FULL)
    assert got == [(0, 2), (1, 2), (2, -1), (3, 1)] and J.finalize(m, capi.JOIN_FULL).tolist() == [0]
    with pytest.raises(J.SingleError):
        run(build, None, np.array([9, 9], np.uint64), None, capi.JOIN_RIGHT_SINGLE)


@pytest.mark.parametrize("jt", J.RIGHT_TYPES)
def test_empty_build_side(jt):
    got, m = run(np.zeros(0, np.uint64), None, PROBE, PNULL, jt)
    want = [(i, -1) for i in range(5)] if jt == capi.JOIN_FULL else []
    assert got == want and J.finalize(m, jt).tolist() == []


@pytest.mark.parametrize("jt", J.RIGHT_TYPES)
def test_empty_probe_side(jt):
    got, m = run(BUILD, BNULL, np.zeros(0, np.uint64), None, jt)
    assert got == [] and J.finalize(m, jt).tolist() == ([] if jt == capi.JOIN_RIGHT_SEMI else [0, 1, 2, 3, 4])


# ---- set identities over random seeds
def random_case(seed, nbuild=300, nprobe=500, keys=120, unique=False):
    r = np.random.default_rng(seed)
    if unique:
        build = r.permutation(keys * 4)[:nbuild].astype(np.uint64); bnull = None
    else:
        build = r.integers(0, keys, nbuild).astype(np.uint64); bnull = r.random(nbuild) < 0.1
    probe_keys = r.integers(0, keys * 4 if unique else keys + keys // 4, nprobe).astype(np.uint64)
    pnull = r.random(nprobe) < 0.1
    _, tk, off, sels = J.build_map(build, bnull)
    return nbuild, off, sels, J.find(tk, probe_keys, pnull)


def pairs_of(vals, off, sels, jt, m=None):
    p, b = J.probe(vals, off, sels, jt, m)
    return list(zip(p.tolist(), b.tolist()))


@pytest.mark.parametrize("seed", range(12))
def test_set_identities(seed):
    nbuild, off, sels, vals = random_case(seed, unique=seed % 3 == 0)
    inner = pairs_of(vals, off, sels, capi.JOIN_INNER)
    left = pairs_of(vals, off, sels, capi.JOIN_LEFT)
    touched = sorted({b for _, b in inner})
    for jt, pairs in ((capi.JOIN_RIGHT, inner), (capi.JOIN_FULL, left)):
        m = np.zeros(nbuild, bool)
        assert pairs_of(vals, off, sels, jt, m) == pairs
        assert np.flatnonzero(m).tolist() == touched
        assert J.finalize(m, jt).tolist() == sorted(set(range(nbuild)) - set(touched))
    for jt, want in ((capi.JOIN_RIGHT_SEMI, touched), (capi.JOIN_RIGHT_ANTI, sorted(set(range(nbuild)) - set(touched)))):
        m = np.zeros(nbuild, bool)
        assert pairs_of(vals, off, sels, jt, m) == [] and J.finalize(m, jt).tolist() == want
    twice = sorted(b for b in touched if sum(1 for _, x in inner if x == b) > 1)
    m = np.zeros(nbuild, bool)
    if twice:
        with pytest.raises(J.SingleError) as e:
            J.probe(vals, off, sels, capi.JOIN_RIGHT_SINGLE, m)
        assert e.value.build_row == twice[0]
    else:
        assert pairs_of(vals, off, sels, capi.JOIN_RIGHT_SINGLE, m) == inner


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("jt", J.NEW_TYPES + (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI))
def test_numpy_form_equals_the_row_loop(seed, jt):
    nbuild, off, sels, vals = random_case(seed, keys=[120, 40, 2000][seed % 3], unique=seed % 4 == 0)
    res = []
    for fn in (J.probe, J.probe_fast):
        m = np.zeros(nbuild, bool)
        try:
            p, b = fn(vals, off, sels, jt, m)
            res.append((p.tolist(), b.tolist(), m.tolist()))
        except J.SingleError as e:
            res.append(("err", e.probe_row, e.build_row))
    assert res[0] == res[1]


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("jt", J.RIGHT_TYPES)
@pytest.mark.parametrize("nbatch", [3, 17])
def test_batches_and_workers_equal_one_batch(seed, jt, nbatch):
    nbuild, off, sels, vals = random_case(seed, keys=2000)             # few duplicates: RIGHT SINGLE mostly passes
    m1 = np.zeros(nbuild, bool)
    try:
        whole = pairs_of(vals, off, sels, jt, m1)
    except J.SingleError:
        whole = None
    cuts = np.linspace(0, len(vals), nbatch + 1).astype(int)
    # one prober over nbatch batches, one bitmap
    m2 = np.zeros(nbuild, bool)
    got = []
    try:
        for a, z in zip(cuts[:-1], cuts[1:]):
            got += [(p + a, b) for p, b in pairs_of(vals[a:z], off, sels, jt, m2)]
    except J.SingleError:
        got = None
    assert got == whole
    if whole is None:
        return
    assert (m1 == m2).all()
    # nbatch workers, one batch each, their bitmaps merged (syncBitmap)
    maps = []
    for a, z in zip(cuts[:-1], cuts[1:]):
        mw = np.zeros(nbuild, bool)
        J.probe(vals[a:z], off, sels, jt, mw)
        maps.append(mw)
    assert (J.sync_bitmap(maps, jt) == m1).all()


def test_right_single_fails_at_the_merge_only():
    _, tk, off, sels = J.build_map(BUILD, BNULL)
    vals = J.find(tk, np.array([20, 20], np.uint64))
    nbuild = len(BUILD)
    ma, mb = np.zeros(nbuild, bool), np.zeros(nbuild, bool)
    J.probe(vals[:1], off, sels, capi.JOIN_RIGHT_SINGLE, ma)
    J.probe(vals[1:], off, sels, capi.JOIN_RIGHT_SINGLE, mb)            # each worker alone is fine
    with pytest.raises(J.SingleError) as e:
        J.sync_bitmap([ma, mb], capi.JOIN_RIGHT_SINGLE)
    assert e.value.build_row == 1
    assert J.sync_bitmap([ma, mb], capi.JOIN_RIGHT).tolist() == [False, True, False, False, False]
