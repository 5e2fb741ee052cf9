"""The byte model of the selective Q6 kernel (tools/tune.py q6_touched_bytes), on the generator's rows: the bytes per row it must
read at 32 / 64 / 128-byte DRAM granularity, as DESIGN 5.1 states them.  No GPU needed."""
import importlib.util
import os

import numpy as np

from matrixone_b200 import datagen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tune():
    spec = importlib.util.spec_from_file_location("tune", os.path.join(ROOT, "tools", "tune.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_q6_bytes_per_row_by_grain():
    T = tune()
    n = 1 << 23
    c = datagen.lineitem(10, 0, n)
    per_row = {name: {g: T.q6_touched_bytes(c["shipdate"], c["discount"], c["quantity"], P, g) / n for g in T.Q6_GRAINS}
               for name, P in T.Q6_SWEEP}
    assert [round(per_row["q6"][g], 1) for g in (32, 64, 128)] == [9.5, 13.0, 17.2]
    assert all(per_row["every_row_passes"][g] == 28.0 for g in T.Q6_GRAINS)
    assert all(per_row["discount_window_empty"][g] == 12.0 for g in T.Q6_GRAINS)
    assert all(per_row["no_row_passes"][g] == 4.0 for g in T.Q6_GRAINS)


def test_q6_bytes_block_edges():
    """a block is read when any of its rows is alive; a ragged last block counts whole"""
    T = tune()
    P = datagen.q6_params()
    n = 20
    sd = np.full(n, P[0] - 1, dtype=np.int32)
    di = np.full(n, 0.03); qt = np.full(n, 1.0)
    assert T.q6_touched_bytes(sd, di, qt, P, 32) == 3 * 32            # shipdate only: 80 bytes -> 3 blocks
    sd[17] = P[0]                                                        # one row alive in the last, ragged block
    assert T.q6_touched_bytes(sd, di, qt, P, 32) == 3 * 32 + 3 * 32      # + one block each of discount, quantity, price
