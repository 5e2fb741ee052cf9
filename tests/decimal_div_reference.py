"""Python-integer restatement of the reference's decimal comparison, division and AVG, path by path, so the device can be held to it.

Values are Python ints: a Decimal64 is its signed 64-bit value, a Decimal128 its signed 128-bit value, and intermediate Go words are kept
as unsigned ints masked to their width.  Every Go function restated here keeps its name:
  Decimal64.Scale / Decimal128.Scale with the compare wrapper's discarded error (func_compare.go:634-650)
  Decimal128.Div128, Mul128, Left, Right, Less; Decimal256.Div256 (pkg/container/types/decimal.go:297-313, 841-861, 982-1017, 1041-1081)
  d128DivOne / d128DivInline / d64Div / d128Div routing (pkg/sql/plan/function/arith_decimal_fast.go:734-1055, 4096-4320)
  Decimal128.Div (decimal.go:1403-1446), decAvg and AvgReturnType (pkg/sql/colexec/aggexec/sumavg2.go:37-56, 545-559)
"""

M64, M128, M256 = (1 << 64) - 1, (1 << 128) - 1, (1 << 256) - 1
POW10 = [10 ** k for k in range(20)]


class DivOverflow(Exception):
    """moerr "Decimal128 Div overflow" (ErrInvalidInput)"""


class DivByZero(Exception):
    """moerr ErrDivByZero "division by zero\""""


class NoEnd(Exception):
    """Decimal256.Div256's long division shifts its divisor out to zero and never returns"""


def _signed(x, bits):
    x &= (1 << bits) - 1
    return x - (1 << bits) if x >> (bits - 1) else x


# ---- Scale as the compare wrapper calls it ---------------------------------------------------------------------------------------------
def d64_scale_dropped(x, n):
    """Decimal64.Scale(n) for 0 <= n <= 18 with the error dropped: |x| * 10^n by an unsigned Mul64 (error only past 2^64), sign restored
    modulo 2^64; on error the value is x unscaled."""
    if n == 0 or x == 0:
        return x
    ab = (-x) & M64 if x < 0 else x
    z = ab * POW10[n]
    if z > M64:
        return x
    return _signed(-z if x < 0 else z, 64)


def d128_scale_dropped(x, n):
    """Decimal128.Scale(n) for 0 <= n <= 38 with the error dropped: each Mul128 step fails once |x| * 10^k reaches 2^127; any failure leaves
    x unscaled."""
    if n == 0:
        return x
    ab = abs(x)
    if ab * 10 ** n >= 1 << 127:
        return x
    return ab * 10 ** n if x >= 0 else -(ab * 10 ** n)


def compare(op, x, y, scale1, scale2, width):
    """valueDecimalCompare: m = scale2 - scale1, the lower-scale side scaled up by |m|, then a signed compare (Less / ==)."""
    sc = d64_scale_dropped if width == 64 else d128_scale_dropped
    m = scale2 - scale1
    if m >= 0:
        x = sc(x, m)
    else:
        y = sc(y, -m)
    return {0: x == y, 1: x != y, 2: x > y, 3: x >= y, 4: x < y, 5: x <= y}[op]


# ---- Decimal128 words -------------------------------------------------------------------------------------------------------------------
def d128_right(x, n):
    """Decimal128.Right: the magnitude (two's complement of a negative) shifted, the sign restored; x unsigned 128-bit"""
    sign = x >> 127
    if sign:
        x = (-x) & M128
    y = x >> n if n < 128 else 0
    return (-y) & M128 if sign else y


def d128_less(x, y):
    """Decimal128.Less: signed"""
    return _signed(x, 128) < _signed(y, 128)


def mul128(x, y):
    """Decimal128.Mul128(x, y) with y < 2^64 (as Div128 calls it); returns the value the Go code returns, error or not"""
    xlo, xhi = x & M64, x >> 64
    ylo, yhi = y & M64, y >> 64
    if xhi and yhi:
        return x
    z = xlo * ylo
    w = (xlo * yhi) if xhi == 0 else (xhi * ylo)
    w_b0, w_b64 = w >> 64, w & M64          # w.B0_63, w.B64_127 = bits.Mul64(...): (hi, lo)
    if w_b0 != 0 or w_b64 >> 63 or z >> 127:
        return z
    return (z + (w_b64 << 64)) & M128


def div128(x, y):
    """Decimal128.Div128 for x >= 0 (unsigned 128-bit), y > 0"""
    if y >> 64 == 0:
        q, rem = divmod(x, y)
        if rem * 2 >= y:
            q += 1
        return q & M128
    if d128_less(x, y):
        return 0
    n = 64 - (y >> 64).bit_length()                   # bits.LeadingZeros64(y.B64_127)
    d = d128_right(y, 64 - n) & M64
    v = (x // d) & M64                                 # bits.Div64(x.hi, x.lo, d): x.hi < d here
    v >>= 63 - n
    if v & 1 == 0:
        return v >> 1
    z = mul128(y, v)
    return (v >> 1) if d128_less((x << 1) & M128, z) else (v >> 1) + 1


# ---- Decimal256 words -------------------------------------------------------------------------------------------------------------------
def d256_right1(x):
    sign = x >> 255
    if sign:
        x = (-x) & M256
    y = x >> 1
    return (-y) & M256 if sign else y


def d256_less(x, y):
    return _signed(x, 256) < _signed(y, 256)


def div256(x, y):
    """Decimal256.Div256 for x >= 0, 0 < y < 2^128"""
    x = (x << 1) & M256
    if y >> 64 == 0:
        z = x // y
    else:
        w, z = 1, 0
        while not d256_less(x, y):                      # y.Compare(x) <= 0
            y = (y << 1) & M256
            w = (w << 1) & M256
            if y == 0:
                raise NoEnd()
        while y != 0:
            y = d256_right1(y)
            w = d256_right1(w)
            if not d256_less(x, y):
                z = (z + w) & M256
                x = (x - y) & M256
    odd = z & 1
    z = d256_right1(z)
    return (z + odd) & M256


def mul_pow10_128(x, n):
    """d128MulPow10: at most two limbs (10^19, 10^(n - 19)), each d128Mul1Limb failing once the product reaches 2^127; n > 38 fails"""
    if n > 38:
        return None
    for k in ([n] if n <= 19 else [19, n - 19]):
        x *= POW10[k]
        if x >> 127:
            return None
    return x


def mul_pow10_256(x, n):
    """d256MulPow10: limbs of 10^19 while n > 19, then 10^n; each fails once the product reaches 2^255"""
    ks = []
    while n > 19:
        ks.append(19)
        n -= 19
    ks.append(n)
    for k in ks:
        x *= POW10[k]
        if x >> 255:
            return None
    return x


def div_scale(scale1):
    """the quotient's scale (Decimal128.Div): min(12, scale1 + 6), at least scale1"""
    s = 12
    if s > scale1 + 6:
        s = scale1 + 6
    if s < scale1:
        s = scale1
    return s


def avg_return_scale(scale):
    """AvgReturnType for decimal64 / decimal128: max(12, scale), at most scale + 6"""
    s = 12
    if s < scale:
        s = scale
    if s > scale + 6:
        s = scale + 6
    return s


def _div_one(x, y, adj, keep=False):
    """d128DivOne (keep=False) / Decimal128.Div's arithmetic (keep=True, returns what decAvg keeps when Div errs).  x, y signed, y != 0."""
    neg = (x < 0) != (y < 0)
    ax, ay = abs(x), abs(y)                            # d128Abs: |MIN| = 2^127 as an unsigned word
    z = mul_pow10_128(ax, adj)
    if z is not None:
        q = div128(z, ay)
        return _signed(-q if neg else q, 128)
    x2 = mul_pow10_256(ax, adj)
    if x2 is None:
        if keep:
            return ax                                  # Decimal128.Div returns x1 = |x| with the scale error
        raise DivOverflow()
    q = div256(x2, ay)
    low = q & M128
    val = _signed(-low if neg else low, 128)
    if q >> 127:
        if keep:
            return val
        raise DivOverflow()
    return val


def div(x, y, scale1, scale2):
    """x / y for Decimal64 or Decimal128 operands (d64Div / d128Div): returns (Decimal128 value, result scale); DivByZero for y == 0
    (the caller's division-by-zero mode decides NULL or error), DivOverflow, NoEnd."""
    if y == 0:
        raise DivByZero()
    scale = div_scale(scale1)
    return _div_one(x, y, scale - scale1 + scale2), scale


def d128_scale_go(x, n):
    """Decimal128.Scale(n) for n >= 0 on a non-negative word x (unsigned 128-bit): Mul128 by 10^19 while n - m > 19, then by 10^(n - m);
    returns (value, error)"""
    if n == 0:
        return x, False
    m = 0
    while n - m > 19:
        m += 19
        x2 = mul128(x, POW10[19])
        if _mul128_failed(x, POW10[19]):
            return x, True
        x = x2
    if _mul128_failed(x, POW10[n - m]):
        return x, True
    return mul128(x, POW10[n - m]), False


def _mul128_failed(x, y):
    """Decimal128.Mul128's error for y < 2^64"""
    xlo, xhi = x & M64, x >> 64
    z = xlo * y
    w = xhi * y
    if (w >> 64) != 0 or (w & M64) >> 63 or z >> 127:
        return True
    return (z + ((w & M64) << 64)) >> 127 != 0


def decimal128_div(x, y, scale1, scale2):
    """Decimal128.Div (decimal.go:1403-1446) as written, for decAvg: returns (value, scale, error).  x, y signed, y != 0."""
    scale = div_scale(scale1)
    signx, signy = x < 0, y < 0
    x1, y1 = (-x) & M128 if signx else x, (-y) & M128 if signy else y           # Minus: |MIN| stays the word 2^127
    z, err = d128_scale_go(x1, scale - scale1 + scale2)
    if err:
        x2 = x1 * 10 ** (scale - scale1 + scale2)                              # Decimal256.Scale: Mul256 steps, exact below 2^255
        if x2 >> 255:
            return x1, scale, True                                               # z is still x1, returned with the error
        q = div256(x2, y1)
        err = q >> 127 != 0
        low = q & M128
        return _signed(-low if signx != signy else low, 128), scale, err
    q = div128(z, y1)
    return _signed(-q if signx != signy else q, 128), scale, False


def avg(total, count, scale):
    """decAvg(sum, count, argScale, AvgReturnType(argScale).Scale): Decimal128.Div(sum, count) with the error dropped, then
    Scale(resultScale - scale) = Scale(0); count 0 is NULL (returns None)."""
    if count == 0:
        return None
    rs = avg_return_scale(scale)
    v, s, _ = decimal128_div(total, count, scale, 0)
    assert s == rs
    return v, rs


def exact_div_half_up(x, y, adj):
    """the mathematically exact x * 10^adj / y, rounded half up away from zero: what the Go code computes outside its quirks"""
    num, den = abs(x) * 10 ** adj, abs(y)
    q, r = divmod(num, den)
    if 2 * r >= den:
        q += 1
    return -q if (x < 0) != (y < 0) else q
