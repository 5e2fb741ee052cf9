"""Hash join pieces (csrc/join.cu: JOIN_SELS, JOIN_FIND, JOIN_PROBE) against the oracle restatement of GroupSels.Finalize
(pkg/vm/message/joinMapMsg.go:72-125), intHashMapIterator.Find and the emission loop of hashjoin container.probe
(pkg/sql/colexec/hashjoin/join.go:383-628, equality conditions only): offsets / sels / ids / result pairs bit-exact, in the reference's order."""
import numpy as np
import pytest

import oracle_lib as O
from matrixone_b200 import capi, ops
from matrixone_b200.vector import Vector, bitmap_from_bools, xcall

pytestmark = pytest.mark.gpu


def _first_seen_ids(keys, skip=None):
    """IntHashMap insert: 1-based ids in first-seen order (numpy restatement for sizes the oracle's linear og_group_ids cannot do)"""
    keys = np.asarray(keys, dtype=np.uint64)
    live = np.ones(len(keys), bool) if skip is None else ~skip
    uniq, first = np.unique(keys[live], return_index=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty(len(uniq), np.int64); rank[order] = np.arange(len(uniq))
    ids = np.zeros(len(keys), np.uint64)
    ids[live] = rank[np.searchsorted(uniq, keys[live])] + 1
    return ids, uniq[order]


def _oracle_join(build, probe, jt, bskip=None, pnull=None):
    ids, table = _first_seen_ids(build, bskip)
    ng = len(table)
    offsets = np.zeros(ng + 2, np.int32); sels = np.zeros(max(len(build), 1), np.int32)
    m = O.go().og_join_sels(O.p(ids), len(build), ng, O.p(offsets), O.p(sels))
    vals = np.zeros(len(probe), np.uint64)
    pn = bitmap_from_bools(pnull) if pnull is not None else None
    O.go().og_join_find(O.p(table), ng, O.p(np.ascontiguousarray(probe, dtype=np.uint64)), O.p(pn) if pn is not None else None, len(probe), O.p(vals))
    unique = ng == len(build)
    cap = int(len(probe) + (0 if unique else 4 * len(probe) + len(build) * 4)) + 1024
    while True:
        op, ob = np.zeros(cap, np.int64), np.zeros(cap, np.int64)
        r = O.go().og_join_probe(O.p(vals), len(probe), None if unique else O.p(offsets), None if unique else O.p(sels), jt, O.p(op), O.p(ob), cap)
        if r <= cap:
            return ids, table, offsets, sels[:m], vals, op[:r], ob[:r]
        cap = r


@pytest.mark.parametrize("nbuild,card,nprobe", [(1, 1, 5), (1000, 1000, 3000), (5000, 37, 2000), (200_000, 50_000, 300_000), (70_000, 3, 100), (100_000, 100_000, 100_000)])
@pytest.mark.parametrize("jt", [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI])
def test_join_matches_the_reference_emission_order(gpu, nbuild, card, nprobe, jt):
    rng = np.random.default_rng(nbuild * 7 + card + jt)
    pool = rng.integers(0, 1 << 63, card, dtype=np.uint64)
    if card == nbuild:
        build = rng.permutation(pool)                      # unique build side: HashOnUnique
    else:
        build = pool[rng.integers(0, card, nbuild)]
    if nbuild > 10:
        build[3] = 0xFFFFFFFFFFFFFFFF                      # the all-ones key is a legal key
    bskip = rng.random(nbuild) < 0.05 if nbuild > 10 else None
    probe = np.where(rng.random(nprobe) < 0.6, pool[rng.integers(0, card, nprobe)], rng.integers(0, 1 << 63, nprobe, dtype=np.uint64)).astype(np.uint64)
    probe[0] = 0xFFFFFFFFFFFFFFFF
    pnull = rng.random(nprobe) < 0.05
    ids, table, offsets, sels, vals, op, ob = _oracle_join(build, probe, jt, bskip, pnull)
    jm = ops.JoinMap(build, skip=bitmap_from_bools(bskip) if bskip is not None else None, prepare=(nbuild % 2 == 0))
    assert jm.ngroups == len(table) and (jm.table_keys == table).all()
    if len(table) != nbuild:
        assert not jm.hash_on_unique()
        assert (jm.offsets == offsets).all()
        assert (jm.sels == sels).all()
    got_vals = jm.find(probe, bitmap_from_bools(pnull))
    assert (got_vals == vals).all()
    gp, gb = jm.probe(probe, jt, bitmap_from_bools(pnull))
    assert len(gp) == len(op)
    assert (gp == op).all() and (gb == ob).all()
    jm.release()


def test_heavy_hitters_and_capacity_protocol(gpu):
    rng = np.random.default_rng(5)
    build = np.concatenate([np.full(5000, 42, np.uint64), np.full(33, 7, np.uint64), rng.integers(100, 1000, 2000).astype(np.uint64)])
    rng.shuffle(build)
    probe = np.array([42, 7, 5, 42, 999999], np.uint64)
    ids, table, offsets, sels, vals, op, ob = _oracle_join(build, probe, capi.JOIN_LEFT)
    jm = ops.JoinMap(build)
    gp, gb = jm.probe(probe, capi.JOIN_LEFT)               # default capacity is too small: the count comes back with RC_OUT_OF_RANGE and the call is repeated
    assert (gp == op).all() and (gb == ob).all() and len(gp) > 10_000
    with pytest.raises(capi.MoError):
        jm.probe(probe, capi.JOIN_INNER, capacity=100)
    jm.release()


def test_empty_sides(gpu):
    jm = ops.JoinMap(np.zeros(0, np.uint64))
    p, b = jm.probe(np.array([1, 2, 3], np.uint64), capi.JOIN_LEFT)
    assert (p == [0, 1, 2]).all() and (b == -1).all()
    p, b = jm.probe(np.array([1, 2, 3], np.uint64), capi.JOIN_INNER)
    assert len(p) == 0
    jm2 = ops.JoinMap(np.array([5, 6], np.uint64))
    p, b = jm2.probe(np.zeros(0, np.uint64), capi.JOIN_INNER)
    assert len(p) == 0
    jm2.release()


def test_empty_table_without_a_pointer(gpu):
    """an empty build side passed with no pointer (a Go nil slice, an empty tensor) is an empty 8-byte table, scratch or prepared: the all-ones
    key, which has a slot of its own, matches nothing"""
    keys = np.array([2**64 - 1, 0, 5], np.uint64)
    prm = {jt: np.array([jt, 0], np.int32).view(np.uint8) for jt in (capi.JOIN_INNER, capi.JOIN_LEFT)}

    def find():
        vals = np.full(3, 7, np.uint64)
        xcall(capi.XCALL_JOIN_FIND, [Vector(data=vals, length=3), Vector(length=0), Vector(data=keys, length=3)], 3)
        return vals

    def probe(jt):
        op, ob, cnt = np.zeros(8, np.int64), np.zeros(8, np.int64), np.zeros(1, np.int64)
        xcall(capi.XCALL_JOIN_PROBE, [Vector(data=op, length=8), Vector(data=ob, length=8), Vector(data=cnt, length=1), Vector(data=prm[jt], length=1),
                                      Vector(length=0), Vector(length=0), Vector(length=0), Vector(data=keys, length=3)], 3)
        return op[:cnt[0]], ob[:cnt[0]]

    lib = capi.load_library()
    for prepared in (False, True):
        if prepared:
            capi.check(lib.MoB200_JoinMapPrepare(None, 0), lib)
        assert (find() == 0).all()
        assert len(probe(capi.JOIN_INNER)[0]) == 0
        p, b = probe(capi.JOIN_LEFT)
        assert (p == [0, 1, 2]).all() and (b == -1).all()
    lib.MoB200_JoinMapRelease(None)
