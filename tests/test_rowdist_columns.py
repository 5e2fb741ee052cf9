"""The column builder and per-row references of the row-wise distance edge tests (rowdist_columns.py), checked without a GPU: every
built column decodes back to its rows by the cell rules of varlena_ref, has the storage kinds and alignment classes it is meant to
have, and the per-row oracle calls agree with one matrix og_distance_rows call."""
import numpy as np
import pytest

import rowdist_columns as R

DTYPES = [np.float32, np.float64]


def _columns(dt):
    x, q = R.ragged_pair(dt, 1)
    sx, sq = R.ragged_pair(dt, 2, special=True)
    return {"ragged x": x, "ragged q": q, "special x": sx, "special q": sq, "normalize": R.normalize_column(dt, 3),
            "uniform": R.uniform_column(dt, 4, 40, 3 * R.slice_elems(dt) + 9, list(range(16)))}


@pytest.mark.parametrize("dt", DTYPES)
def test_every_row_decodes_back(dt):
    for name, col in _columns(dt).items():
        for i in range(col.n):
            got = R.decode(col.cells, col.area, i, dt)
            assert got is not None and got.tobytes() == col.rows[i].tobytes(), (name, i, col.kind[i])
            if col.offset[i] is not None:
                assert col.offset[i] + col.rows[i].nbytes <= col.area.nbytes
        owned = np.zeros(col.area.nbytes, bool)
        for i in range(col.n):
            if col.kind[i] == "area":
                owned[col.offset[i]:col.offset[i] + col.rows[i].nbytes] = True
        assert (col.area[~owned] == R.FILL).all(), name        # the bytes between rows are padding, and there is padding behind the last


@pytest.mark.parametrize("dt", DTYPES)
def test_layout_classes_are_present(dt):
    x, q = R.ragged_pair(dt, 1)
    eps = R.slice_elems(dt)
    for col in (x, q):
        kinds = set(col.kind)
        assert kinds == {"inline", "area", "dup"}
        assert {o % 16 for o, k in zip(col.offset, col.kind) if k == "area"} == set(range(16))
        lens = [r.size for r in col.rows]
        assert col.kind[0] == "inline" and lens[0] == 0 and col.kind[1] == "area" and lens[1] == 0
        assert any(k == "area" and r.nbytes <= R.INLINE_MAX and r.size for k, r in zip(col.kind, col.rows))   # short rows in the area
        assert any(k == "inline" and r.size for k, r in zip(col.kind, col.rows))
    # row i has one length on both sides, and x and q sit at different offsets mod 16
    assert all(a.size == b.size for a, b in zip(x.rows, q.rows))
    assert any(ox % 16 != oq % 16 for ox, oq in zip(x.offset, q.offset) if ox is not None and oq is not None)
    lens = [r.size for r in x.rows]
    for chunk in (8, 4):
        for w in range(0, len(lens), 32):     # every warp mixes slice counts
            assert len({R.slices(n, dt, chunk) for n in lens[w:w + 32]}) >= 5
        nsl = {R.slices(n, dt, chunk) for n in lens}
        assert set(range(7)) <= nsl and max(nsl) >= 10
    for b in range(1, 7):
        assert {b * eps - 1, b * eps, b * eps + 1} <= set(lens)
    assert {3, 4, 5, 7, 8, 9} <= set(lens)


@pytest.mark.parametrize("dt", DTYPES)
def test_specials_are_present(dt):
    x, q = R.ragged_pair(dt, 2, special=True)
    vals = np.concatenate(x.rows + q.rows)
    assert np.isnan(vals).any() and np.isposinf(vals).any() and np.isneginf(vals).any()
    assert ((vals == 0) & np.signbit(vals)).any()
    assert ((vals != 0) & (np.abs(vals) < np.finfo(dt).tiny)).any()
    if dt == np.float32:
        assert any(np.isinf(R.row_distance(R.L2SQ, a, b)[0]) and np.isfinite(a).all() and np.isfinite(b).all() for a, b in zip(x.rows, q.rows))
    sims = [R.row_distance(R.COSSIM, a, b) for a, b in zip(x.rows, q.rows)]
    assert any(v == 1.0 and not e for v, e in sims) and any(v == -1.0 and not e for v, e in sims)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("dim", [1, 5, 8, 9, 37, 65])
def test_per_row_references_equal_one_matrix_call(dt, dim):
    rng = np.random.default_rng(dim)
    n = 70
    a = rng.standard_normal((n, dim)).astype(dt)
    b = rng.standard_normal((n, dim)).astype(dt)
    a[3] = b[3]
    a[5, 0] = np.nan
    for kind in (R.L2, R.L2SQ, R.IP, R.COSDIST, R.L1):
        for bb in (b, b[:1]):
            whole = R.matrix_distance(kind, a, bb)
            rows = np.array([R.row_distance(kind, a[i], bb[0 if bb.shape[0] == 1 else i])[0] for i in range(n)])
            assert R.same(rows, whole).all(), (kind, dim)


def test_same_accepts_any_nan_and_tells_signed_zeros_apart():
    nan2 = np.array([0x7FF8000000000001], np.uint64).view(np.float64)
    assert R.same(np.array([np.nan, 1.0, 0.0]), np.array([nan2[0], 1.0, 0.0])).all()
    assert not R.same(np.array([-0.0]), np.array([0.0])).any()
    assert not R.same(np.array([np.nan]), np.array([1.0])).any()


def test_normalize_reference_and_decode_of_out_of_area_cells():
    assert R.normalize(np.zeros(0, np.float32)) is None
    v = np.array([3.0, 4.0])
    assert R.normalize(v).tolist() == [0.6, 0.8]
    z = np.array([-0.0, 0.0], np.float32)
    assert R.normalize(z).tobytes() == z.tobytes()          # a zero row is copied as it is
    col = R.Column([np.arange(8, dtype=np.float32)], np.float32)
    cells = col.cells.copy()
    cells.view(np.uint32)[1] = col.area.nbytes - 4
    assert R.decode(cells, col.area, 0, np.float32) is None
