"""TPC-H Q6 over the DECIMAL(15,2) lineitem schema, restated in Python integers serially in row order: filter, Shrink, d64Mul(extendedprice,
discount) -> Decimal128 at scale 2s, SUM with the checked Add128 (sum_decimal_fast.go).  The reference the fused MO_XCALL_Q6_DEC_FILTER_SUM
is tested against, byte for byte."""
import numpy as np

from matrixone_b200 import datagen

I128_MIN, I128_MAX = -(1 << 127), (1 << 127) - 1
RC_INVALID_ARGUMENT = 20203


def wrap128(v):
    v &= (1 << 128) - 1
    return v - (1 << 128) if v >> 127 else v


def q6_dec(sd, disc, qty, price, n, date_lo, date_hi, disc_lo, disc_hi, qty_hi, scale):
    """the fields of ops.q6_dec_filter_sum: revenue is the exact sum (modulo 2^128 when the call fails), err_row the first row whose running
    sum leaves int128"""
    sd, disc, qty, price = (np.asarray(c)[:n] for c in (sd, disc, qty, price))
    rows = np.flatnonzero((sd >= date_lo) & (sd < date_hi) & (disc >= disc_lo) & (disc <= disc_hi) & (qty < qty_hi))
    s, err = 0, -1
    for r, v in zip(rows.tolist(), (price[rows].astype(object) * disc[rows].astype(object)).tolist()):
        s += v
        if err < 0 and not I128_MIN <= s <= I128_MAX:
            err = r
    return {"revenue": wrap128(s), "scale": 2 * scale, "count": len(rows), "rc": RC_INVALID_ARGUMENT if err >= 0 else 0, "err_row": err,
            "is_null": len(rows) == 0}


def lineitem_dec(seed, row0, n):
    """datagen.lineitem as the DECIMAL(15,2) schema stores it: shipdate int32, quantity / extendedprice / discount as int64 cents.
    round(x * 100) is exact for this generator: quantity is integral, price a whole number of cents, discount a whole percent."""
    c = datagen.lineitem(seed, row0, n)
    return {"shipdate": c["shipdate"], "quantity": (c["quantity"] * 100).round().astype(np.int64),
            "extendedprice": (c["extendedprice"] * 100).round().astype(np.int64), "discount": (c["discount"] * 100).round().astype(np.int64)}


def q6_dec_params():
    """q6.sql's constants cast to DECIMAL(15,2) as the reference's constant folder does: 0.03 - 0.01 -> 0.02 (2), 0.03 + 0.01 -> 4, 24 -> 2400"""
    lo, hi, _, _, _ = datagen.q6_params()
    return lo, hi, 2, 4, 2400, 2
