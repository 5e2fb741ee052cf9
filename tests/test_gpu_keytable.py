"""The one 8-byte-key hash table (csrc/keytable.cuh) on keys that collide.  mix64 is invertible, so keys whose mix64 has its low 16 bits all
ones can be made on the host: in any table of at most 65,536 slots every one of them starts at the last slot, so they form one long probe
chain that wraps to slot 0.  Each user of the table -- GROUP_IDS, the join map behind JOIN_FIND / JOIN_PROBE, the plan's CTA and global group
tables -- runs on such keys mixed with random keys and the all-ones key, against the exact restatements the other GPU tests use."""
import os
import re

import numpy as np
import pytest

import oracle_lib as O
import plan_reference as R
from matrixone_b200 import capi, ops
from matrixone_b200.vector import DeviceBuffer, bitmap_from_bools

M64 = (1 << 64) - 1
C1, C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
ALL_ONES = np.uint64(M64)


def mix64(x):
    x ^= x >> 33; x = x * C1 & M64; x ^= x >> 33; x = x * C2 & M64
    return x ^ (x >> 33)


def unmix64(h):
    """x ^= x >> 33 undoes itself on 64 bits, and the odd constants have inverses mod 2^64"""
    h ^= h >> 33; h = h * pow(C2, -1, 1 << 64) & M64; h ^= h >> 33; h = h * pow(C1, -1, 1 << 64) & M64
    return h ^ (h >> 33)


def colliding_keys(rng, n):
    """n distinct keys whose mix64 has its low 16 bits all ones; the high 48 bits of the hash stay below 2^47, so no key is all ones"""
    hi = np.unique(rng.integers(0, 1 << 47, 2 * n, dtype=np.uint64))[:n]
    assert hi.shape[0] == n
    return np.array([unmix64((int(h) << 16) | 0xFFFF) for h in rng.permutation(hi)], dtype=np.uint64)


def test_mix64_inverse_and_colliding_keys():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "matrixone_b200", "csrc", "keytable.cuh")) as f:
        body = re.search(r"uint64_t mix64\(uint64_t x\) \{(.*?)\n\}", f.read(), re.S).group(1)
    assert re.findall(r"0x([0-9a-f]+)ull", body) == ["%x" % C1, "%x" % C2] and re.findall(r">> (\d+)", body) == ["33"] * 3   # the device's mix64
    rng = np.random.default_rng(1)
    for x in [0, 1, M64, M64 - 1, 1 << 63] + [int(v) for v in rng.integers(0, 1 << 64, 2000, dtype=np.uint64)]:
        assert unmix64(mix64(x)) == x and mix64(unmix64(x)) == x
    keys = colliding_keys(rng, 3000)
    assert len(set(keys.tolist())) == 3000 and ALL_ONES not in keys
    assert all(mix64(int(k)) & 0xFFFF == 0xFFFF for k in keys)


def _first_seen_ids(keys, skip=None):
    """IntHashMap insert: 1-based ids in first-seen order, and the keys in id order"""
    keys = np.asarray(keys, dtype=np.uint64)
    live = np.ones(len(keys), bool) if skip is None else ~skip
    uniq, first = np.unique(keys[live], return_index=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty(len(uniq), np.int64); rank[order] = np.arange(len(uniq))
    ids = np.zeros(len(keys), np.uint64)
    ids[live] = rank[np.searchsorted(uniq, keys[live])] + 1
    return ids, uniq[order]


@pytest.mark.gpu
def test_group_ids_on_colliding_keys(gpu):
    rng = np.random.default_rng(11)
    universe = np.concatenate([colliding_keys(rng, 3000), rng.integers(0, 1 << 63, 2000, dtype=np.uint64), [ALL_ONES]])
    n = 300_000
    keys = universe[rng.integers(0, universe.shape[0], n)]
    keys[n // 3] = ALL_ONES
    table = ops.GroupTable(universe.shape[0] + 8)              # 16,384 slots: every colliding key starts at the last one
    half = n // 2
    g1 = table.insert(keys[:half]); ng1 = int(table.ngroups[0])
    g2 = table.insert(keys[half:]); ng2 = int(table.ngroups[0])
    want, order = _first_seen_ids(keys)
    assert np.array_equal(np.concatenate([g1, g2]), want)
    assert ng1 == int(want[:half].max()) and ng2 == order.shape[0]
    assert np.array_equal(table.keys[:ng2], order)
    small = ops.GroupTable(16)                                 # 32 slots: 100 colliding keys fill it, every slot visited
    with pytest.raises(capi.MoError):
        small.insert(colliding_keys(rng, 100))


def _oracle_join(build, probe, jt, pnull):
    ids, table = _first_seen_ids(build)
    ng = len(table)
    offsets = np.zeros(ng + 2, np.int32); sels = np.zeros(len(build), np.int32)
    m = O.go().og_join_sels(O.p(ids), len(build), ng, O.p(offsets), O.p(sels))
    vals = np.zeros(len(probe), np.uint64)
    pn = bitmap_from_bools(pnull)
    O.go().og_join_find(O.p(table), ng, O.p(probe), O.p(pn), len(probe), O.p(vals))
    cap = 8 * len(probe) + 4 * len(build)
    op, ob = np.zeros(cap, np.int64), np.zeros(cap, np.int64)
    r = O.go().og_join_probe(O.p(vals), len(probe), O.p(offsets), O.p(sels), jt, O.p(op), O.p(ob), cap)
    assert r <= cap
    return table, offsets, sels[:m], vals, op[:r], ob[:r]


@pytest.mark.gpu
@pytest.mark.parametrize("prepare", [False, True])
@pytest.mark.parametrize("jt", [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI])
def test_join_on_colliding_keys(gpu, jt, prepare):
    """build keys repeat (the sels path); probe keys hit, miss at the end of the colliding chain, or are all ones"""
    rng = np.random.default_rng(21 + jt)
    coll = colliding_keys(rng, 4000)
    pool = np.concatenate([coll[:2500], rng.integers(0, 1 << 63, 1500, dtype=np.uint64), [ALL_ONES]])
    build = pool[rng.integers(0, pool.shape[0], 20_000)]
    build[7] = ALL_ONES
    absent = np.concatenate([coll[2500:], rng.integers(0, 1 << 63, 500, dtype=np.uint64)])
    nprobe = 50_000
    probe = np.where(rng.random(nprobe) < 0.7, pool[rng.integers(0, pool.shape[0], nprobe)], absent[rng.integers(0, absent.shape[0], nprobe)]).astype(np.uint64)
    probe[0] = ALL_ONES
    pnull = rng.random(nprobe) < 0.05
    table, offsets, sels, vals, op, ob = _oracle_join(build, probe, jt, pnull)
    jm = ops.JoinMap(build, prepare=prepare)                   # <= 4001 groups: 8192 slots
    assert jm.ngroups == len(table) and (jm.table_keys == table).all()
    assert (jm.offsets == offsets).all() and (jm.sels == sels).all()
    assert (jm.find(probe, bitmap_from_bools(pnull)) == vals).all()
    gp, gb = jm.probe(probe, jt, bitmap_from_bools(pnull))
    assert len(gp) == len(op) and (gp == op).all() and (gb == ob).all()
    jm.release()


@pytest.mark.gpu
def test_plan_group_by_colliding_uint64_keys(gpu):
    """2,501 distinct keys spread over every tile: each CTA fills its 4 private slots and its 32-slot CTA table (colliding keys start at CTA
    slot 31 and wrap) and sends the rest to the global table (8,192 slots).  Exact fit, one short, and a global table too small to hold
    the keys"""
    rng = np.random.default_rng(31)
    n = 200_000
    vocab = np.concatenate([colliding_keys(rng, 2000), rng.integers(0, 1 << 63, 500, dtype=np.uint64), [ALL_ONES]])
    key = vocab[rng.integers(0, vocab.shape[0], n)]
    key[n // 2] = ALL_ONES
    x = rng.standard_normal(n)
    p = ops.FusedPlan([capi.T_UINT64, capi.T_FLOAT64], row_base=1000).group_by(0)
    p.agg(capi.AGG_SUM, 1).agg(capi.AGG_COUNT, -1).agg(capi.AGG_MIN, 1).agg(capi.AGG_MAX, 1)
    want = R.run(p.P, [key, x], None, n)
    ng = len(want)
    assert ng == vocab.shape[0]
    R.assert_matches(p.run([key, x], n, max_groups=ng), want, p.P)
    with pytest.raises(capi.MoError) as e:
        p.run([key, x], n, max_groups=ng - 1)
    assert e.value.rc == capi.RC_INVALID_ARGUMENT
    dev = [DeviceBuffer.from_numpy(key), DeviceBuffer.from_numpy(x)]
    for mg in (ng, ng - 1):                                     # the asynchronous form: header.overflow instead of an error
        res = DeviceBuffer(p.result_bytes(mg))
        p.run(dev, n, max_groups=mg, out_ptr=res.ptr)
        raw = res.to_numpy(np.uint8).tobytes()
        if mg == ng:
            R.assert_matches(p.parse(raw), want, p.P)
        else:
            assert capi.PlanHeader.from_buffer_copy(raw).overflow == 1
        res.free()
    for b in dev:
        b.free()
    with pytest.raises(capi.MoError):                          # 1,024 global slots for 2,501 keys: the table fills
        p.run([key, x], n, max_groups=100)
