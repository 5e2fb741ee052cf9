// decimal.cu -- Decimal64 / Decimal128 batch arithmetic and decimal SUM (SURVEY.md section 8(f) row 1: the reference's native TPC-H
// column type is DECIMAL(15,2), test/distributed/cases/benchmark/tpch/01_DDL/01_create_table.sql:83-86).
//
//   MO_XCALL_DEC_ARITH(op, width)   d64Add / d64Sub / d64Mul / d128Add / d128Sub / d128Mul, pkg/sql/plan/function/arith_decimal_fast.go
//   MO_XCALL_DEC_SUM(width)         sumDecimal64FastExec / sumDecimal128FastExec.batchFill, pkg/sql/colexec/aggexec/sum_decimal_fast.go
//   MO_XCALL_DEC_ARITH(3, width)    d64Div / d128Div (arith_decimal_fast.go:734-1055, 4096-4320) = Decimal128.Div, result Decimal128
//   MO_XCALL_DEC_AVG(width)         decAvg over DEC_SUM's state, pkg/sql/colexec/aggexec/sumavg2.go:545-559
//   MO_XCALL_GO_COMPARE(op, DECIMAL64 | DECIMAL128)   valueDecimalCompare, pkg/sql/plan/function/func_compare.go:426-667
//
// Pure integer work, bit-exact: Decimal64 = int64 unscaled value, Decimal128 = two's-complement {B0_63, B64_127}; the scales travel in
// the parameter block.  The operand protocol is the Go elementwise engine's (goengine.cuh); the FIRST offending row in row order fails the
// call ("Decimal64 Add overflow", "scale overflow", "Decimal128 Mul overflow" -> MO_RC_INVALID_ARGUMENT = moerr ErrInvalidInput).
// 128-bit sums are accumulated as two 64-bit atomics with an explicit carry: integer addition is associative, so the result is exact
// and run-to-run identical whatever the order.
#include "goengine.cuh"
#include <cstring>

using namespace mob;

namespace {

constexpr int kCtasPerSm = 8;

typedef unsigned __int128 u128;
typedef __int128 i128;

__device__ __forceinline__ i128 d128_get(Dec128 v) { return (i128)(((u128)(uint64_t)v.hi << 64) | v.lo); }
__device__ __forceinline__ Dec128 d128_put(i128 x) { Dec128 r; r.lo = (uint64_t)(u128)x; r.hi = (int64_t)((u128)x >> 64); return r; }

__constant__ uint64_t kPow10[20] = {1ull, 10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull, 100000000ull, 1000000000ull,
    10000000000ull, 100000000000ull, 1000000000000ull, 10000000000000ull, 100000000000000ull, 1000000000000000ull, 10000000000000000ull,
    100000000000000000ull, 1000000000000000000ull, 10000000000000000000ull};

// d64MulPow10 (arith_decimal_fast.go:4881-4890): ok iff |x| * 10^diff < 2^63
__device__ __forceinline__ bool d64_scale_up(int64_t &x, int diff) {
    const uint64_t sign = (uint64_t)x >> 63, mask = 0ull - sign, ab = ((uint64_t)x ^ mask) + sign;
    const uint64_t hi = __umul64hi(ab, kPow10[diff]), lo = ab * kPow10[diff];
    if (hi | (lo >> 63)) return false;
    x = (int64_t)((lo ^ mask) + sign);
    return true;
}
// |v| * 10^d < 2^127 (d128ScaleUp / d128Mul1Limb :443-450, 4890-4906)
__device__ __forceinline__ bool d128_scale_up(i128 &v, int d) {
    u128 ab = v < 0 ? (u128)0 - (u128)v : (u128)v;
    const u128 lim = ((((u128)1) << 127) - 1) / kPow10[d];
    if (ab > lim) return false;
    ab *= kPow10[d];
    v = v < 0 ? -(i128)ab : (i128)ab;
    return true;
}
// magnitude (4 limbs) / d with round-half-up on the remainder (d128DivPow10Once :4913-4923)
__device__ __forceinline__ void mag_div_once(uint64_t m[4], uint64_t d) {
    u128 rem = 0;
#pragma unroll
    for (int k = 3; k >= 0; k--) { const u128 cur = (rem << 64) | m[k]; m[k] = (uint64_t)(cur / d); rem = cur % d; }
    if ((uint64_t)rem >= (d + 1) >> 1) {
#pragma unroll
        for (int k = 0; k < 4; k++) { if (++m[k] != 0) break; }
    }
}
__device__ __forceinline__ void mag_div_pow10(uint64_t m[4], int k) {
    if (k <= 0) return;
    if (k <= 19) { mag_div_once(m, kPow10[k]); return; }
    mag_div_once(m, kPow10[19]); mag_div_once(m, kPow10[k - 19]);
}

// ---- decimal division, restated limb by limb from the Go code (pkg/container/types/decimal.go, arith_decimal_fast.go) ----------------------
// Only the signed comparisons and the sign-aware right shifts of the Go types are signed; every add, subtract and left shift wraps.
__device__ __forceinline__ uint64_t shl64(uint64_t x, int s) { return s >= 64 ? 0 : x << s; }   // Go: a shift by >= 64 gives 0
__device__ __forceinline__ uint64_t shr64(uint64_t x, int s) { return s >= 64 ? 0 : x >> s; }
__device__ __forceinline__ u128 d128_minus(u128 x) { return (u128)0 - x; }                  // Decimal128.Minus: two's complement
// Decimal128.Right (:297-313): the magnitude is shifted and the sign restored
__device__ __forceinline__ u128 d128_right(u128 x, int n) {
    const bool sign = (uint64_t)(x >> 64) >> 63;
    if (sign) x = d128_minus(x);
    const uint64_t lo = (uint64_t)x, hi = (uint64_t)(x >> 64);
    uint64_t ylo, yhi;
    if (n > 64) { yhi = 0; ylo = shr64(hi, n - 64); }
    else { yhi = shr64(hi, n); ylo = shr64(lo, n) | shl64(hi, 64 - n); }
    const u128 y = ((u128)yhi << 64) | ylo;
    return sign ? d128_minus(y) : y;
}
// Decimal128.Mul128 (:841-861) for y < 2^64, as Div128 calls it on a divisor x >= 2^64: on overflow it returns the partial product
__device__ __forceinline__ u128 d128_mul128_go(u128 x, uint64_t y) {
    const uint64_t xlo = (uint64_t)x, xhi = (uint64_t)(x >> 64);
    u128 z = (u128)xlo * y;
    const u128 w = (u128)xhi * y;                                                // x.B64_127 == 0: Mul64(x.B0_63, y.B64_127 = 0) = 0
    const uint64_t w_b0 = (uint64_t)(w >> 64), w_b64 = (uint64_t)w;              // w.B0_63, w.B64_127 = bits.Mul64(...): hi, lo
    if (w_b0 != 0 || (w_b64 >> 63) || ((uint64_t)(z >> 64) >> 63)) return z;
    z += (u128)w_b64 << 64;
    return z;
}
// Decimal128.Div128 (:982-1017) on a non-negative dividend: round half up for a 64-bit divisor; above that the quotient is estimated from
// the divisor's top 64 bits and rounded by the signed Less of x.Left(1), which wraps negative for x >= 2^126
__device__ __forceinline__ u128 d128_div128_go(u128 x, u128 y) {
    const uint64_t yhi = (uint64_t)(y >> 64);
    if (yhi == 0) {
        const uint64_t d = (uint64_t)y;
        const uint64_t qh = (uint64_t)(x >> 64) / d, r1 = (uint64_t)(x >> 64) % d;
        const u128 cur = ((u128)r1 << 64) | (uint64_t)x;
        const uint64_t ql = (uint64_t)(cur / d), rem = (uint64_t)(cur % d);
        u128 q = ((u128)qh << 64) | ql;
        if (rem * 2 >= d || (rem >> 63)) q += 1;
        return q;
    }
    if ((i128)x < (i128)y) return 0;
    const int n = __clzll((long long)yhi);
    const uint64_t d = (uint64_t)d128_right(y, 64 - n);
    uint64_t v = (uint64_t)(x / d);                                              // bits.Div64(x.hi, x.lo, d): x.hi < 2^63 <= d
    v >>= 63 - n;
    if ((v & 1) == 0) return v >> 1;
    const u128 z = d128_mul128_go(y, v);
    return (i128)(x << 1) < (i128)z ? (u128)(v >> 1) : (u128)((v >> 1) + 1);
}

struct U256 { uint64_t w[4]; };   // Decimal256 {B0_63, B64_127, B128_191, B192_255}
__device__ __forceinline__ bool u256_zero(const U256 &x) { return (x.w[0] | x.w[1] | x.w[2] | x.w[3]) == 0; }
__device__ __forceinline__ U256 u256_minus(U256 x) {
    U256 y; uint64_t c = 1;
#pragma unroll
    for (int k = 0; k < 4; k++) { y.w[k] = ~x.w[k] + c; c = (c && y.w[k] == 0) ? 1 : 0; }
    return y;
}
__device__ __forceinline__ U256 u256_add(const U256 &x, const U256 &y) {
    U256 z; uint64_t c = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) { const uint64_t s = x.w[k] + y.w[k]; const uint64_t s2 = s + c; c = (s < x.w[k]) || (s2 < s); z.w[k] = s2; }
    return z;
}
__device__ __forceinline__ U256 u256_left1(const U256 &x) {
    U256 y; y.w[0] = x.w[0] << 1;
#pragma unroll
    for (int k = 1; k < 4; k++) y.w[k] = (x.w[k] << 1) | (x.w[k - 1] >> 63);
    return y;
}
// Decimal256.Right(1) (:330-350): sign-aware
__device__ __forceinline__ U256 u256_right1(U256 x) {
    const bool sign = x.w[3] >> 63;
    if (sign) x = u256_minus(x);
    U256 y;
#pragma unroll
    for (int k = 0; k < 3; k++) y.w[k] = (x.w[k] >> 1) | (x.w[k + 1] << 63);
    y.w[3] = x.w[3] >> 1;
    return sign ? u256_minus(y) : y;
}
// Decimal256.Less: signed
__device__ __forceinline__ bool u256_less(const U256 &x, const U256 &y) {
    if ((x.w[3] >> 63) != (y.w[3] >> 63)) return x.w[3] >> 63;
    for (int k = 3; k >= 0; k--) if (x.w[k] != y.w[k]) return x.w[k] < y.w[k];
    return false;
}
// d256Mul1Limb (arith_decimal_fast.go:1735-1746): false when the product leaves 255 bits
__device__ __forceinline__ bool u256_mul1(U256 &x, uint64_t p) {
    uint64_t h[4], l[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { l[k] = x.w[k] * p; h[k] = __umul64hi(x.w[k], p); }
    x.w[0] = l[0];
    uint64_t c = 0;
#pragma unroll
    for (int k = 1; k < 4; k++) { const uint64_t s = l[k] + h[k - 1]; const uint64_t s2 = s + c; c = (s < l[k]) || (s2 < s); x.w[k] = s2; }
    return (h[3] | c | (x.w[3] >> 63)) == 0;
}
enum { DIV_OK = 0, DIV_OVERFLOW = 1, DIV_SCALE_OVERFLOW = 2, DIV_NO_END = 3 };
// Decimal256.Div256 (:1041-1081) of a non-negative x by 0 < y < 2^128.  The long division compares signed: a dividend with bit 254 set
// (bit 255 after the first doubling) gives 0, and when the divisor is shifted out to zero the Go loop never ends (DIV_NO_END).
__device__ int u256_div256_go(U256 x, U256 y, U256 &z) {
    x = u256_left1(x);
    z = U256{{0, 0, 0, 0}};
    if ((y.w[1] | y.w[2] | y.w[3]) == 0) {
        const uint64_t d = y.w[0];
        uint64_t rem = 0;
        for (int k = 3; k >= 0; k--) { const u128 cur = ((u128)rem << 64) | x.w[k]; z.w[k] = (uint64_t)(cur / d); rem = (uint64_t)(cur % d); }
    } else {
        U256 w{{1, 0, 0, 0}};
        while (!u256_less(x, y)) {                                               // y.Compare(x) <= 0
            y = u256_left1(y); w = u256_left1(w);
            if (u256_zero(y)) return DIV_NO_END;
        }
        while (!u256_zero(y)) {
            y = u256_right1(y); w = u256_right1(w);
            if (!u256_less(x, y)) { z = u256_add(z, w); x = u256_add(x, u256_minus(y)); }
        }
    }
    const bool odd = z.w[0] & 1;
    z = u256_right1(z);
    if (odd) z = u256_add(z, U256{{1, 0, 0, 0}});
    return DIV_OK;
}

// x / y at scale adjustment adj = resultScale - scale1 + scale2 (>= 0), y != 0: d128DivOne (arith_decimal_fast.go:970-1012), which the
// inline 64-bit path d128DivInline equals wherever it applies, and Decimal128.Div (decimal.go:1403-1446) for AVG.  DIV_OVERFLOW leaves in z
// the value Decimal128.Div keeps (the quotient's low 128 bits, signed); DIV_SCALE_OVERFLOW leaves |x|.
__device__ int dec_div(i128 xs, i128 ys, int adj, i128 &out) {
    const bool neg = (xs < 0) != (ys < 0);
    const u128 x = xs < 0 ? d128_minus((u128)xs) : (u128)xs, y = ys < 0 ? d128_minus((u128)ys) : (u128)ys;   // d128Abs: |MIN| stays 2^127
    // d128MulPow10 (:431-439): |x| * 10^adj < 2^127, in at most two limbs of 10^19
    bool fits = adj <= 38;
    u128 z = x;
    if (fits) {
        int rest = adj;
        do {
            const int k = rest > 19 ? 19 : rest; rest -= k;
            const uint64_t p = kPow10[k], lo = (uint64_t)z, hi = (uint64_t)(z >> 64);
            uint64_t zh = __umul64hi(lo, p);
            if (hi) { const uint64_t ch = __umul64hi(hi, p), cl = hi * p; const uint64_t s = zh + cl; if (ch | (s < zh) | (s >> 63)) { fits = false; break; } zh = s; }
            else if (zh >> 63) { fits = false; break; }
            z = ((u128)zh << 64) | (lo * p);
        } while (rest > 0);
    }
    if (fits) {
        z = d128_div128_go(z, y);
        out = (i128)(neg ? d128_minus(z) : z);
        return DIV_OK;
    }
    U256 x2{{(uint64_t)x, (uint64_t)(x >> 64), 0, 0}}, y2{{(uint64_t)y, (uint64_t)(y >> 64), 0, 0}}, q;
    for (int rest = adj; ;) {                                                    // d256MulPow10 (:1750-1758)
        const int k = rest > 19 ? 19 : rest; rest -= k;
        if (!u256_mul1(x2, kPow10[k])) { out = (i128)x; return DIV_SCALE_OVERFLOW; }
        if (rest <= 0) break;
    }
    const int rc = u256_div256_go(x2, y2, q);
    z = ((u128)q.w[1] << 64) | q.w[0];
    out = (i128)(neg ? d128_minus(z) : z);
    if (rc != DIV_OK) return rc;
    return (q.w[3] | q.w[2] | (q.w[1] >> 63)) ? DIV_OVERFLOW : DIV_OK;
}

// Decimal64.Scale / Decimal128.Scale (decimal.go:352-392, 438-480) up by d as the compare wrapper calls them: the error is dropped and the
// value comes back unscaled.  Decimal64 scales |x| by an unsigned Mul64 (no error below 2^64) and restores the sign, so it can wrap.
__device__ __forceinline__ int64_t d64_scale_cmp(int64_t x, int d) {
    if (d == 0 || x == 0) return x;
    const uint64_t sign = (uint64_t)x >> 63, ab = sign ? 0ull - (uint64_t)x : (uint64_t)x;
    if (__umul64hi(ab, kPow10[d])) return x;
    const uint64_t z = ab * kPow10[d];
    return (int64_t)(sign ? 0ull - z : z);
}
__device__ __forceinline__ i128 d128_scale_cmp(i128 x, int d) {
    if (d == 0) return x;
    i128 v = x;
    if (d > 19) { if (!d128_scale_up(v, 19)) return x; d -= 19; }
    return d128_scale_up(v, d) ? v : x;
}

// the scale of a quotient and of an AVG: min(12, scale1 + 6), raised to at least scale1 (Decimal128.Div, AvgReturnType)
inline int div_scale(int s1) { int s = 12; if (s > s1 + 6) s = s1 + 6; if (s < s1) s = s1; return s; }
template <int W> constexpr int kMaxScale() { return W == 64 ? 18 : 38; }

struct DecParams { int32_t scale1, scale2; int64_t err_row; int32_t div0_error, reserved; };   // div0_error: DIV only
constexpr size_t kDecParamsV1 = 16;   // {scale1, scale2, err_row}: what + - * read and every op writes back

__device__ __forceinline__ bool row_null(const uint64_t *rnulls, uint64_t i) { return (rnulls[i >> 6] >> (i & 63)) & 1ull; }

// the failure record's kind: 1 = division by zero
// OP: 0 add, 1 sub, 2 mul, 3 div.  W: 64 or 128 (operand width).  d64 mul and div produce d128.
template <int OP, int W>
__global__ void __launch_bounds__(kThreads)
dec_arith_kernel(void *__restrict__ r, const void *__restrict__ a, const void *__restrict__ b, uint64_t n, int c1, int c2, int d1, int d2, int adj,
                 uint64_t *__restrict__ rnulls, int div0_error, unsigned long long *first_bad) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        if (OP == 3) {
            const i128 x = W == 64 ? (i128)reinterpret_cast<const int64_t *>(a)[c1 ? 0 : i] : d128_get(reinterpret_cast<const Dec128 *>(a)[c1 ? 0 : i]);
            const i128 y = W == 64 ? (i128)reinterpret_cast<const int64_t *>(b)[c2 ? 0 : i] : d128_get(reinterpret_cast<const Dec128 *>(b)[c2 ? 0 : i]);
            // a const zero divisor fails or nulls the whole vector before any row is looked at; a vector one only the rows it reaches
            if (y == 0 && (c2 || !row_null(rnulls, i))) {
                if (div0_error) note_failure(first_bad, i, 1);
                else atomicOr(reinterpret_cast<unsigned long long *>(&rnulls[i >> 6]), 1ull << (i & 63));
                continue;
            }
            if (row_null(rnulls, i)) continue;
            i128 z;
            if (dec_div(x, y, adj, z) != DIV_OK) note_failure(first_bad, i);
            else reinterpret_cast<Dec128 *>(r)[i] = d128_put(z);
            continue;
        }
        if (row_null(rnulls, i)) continue;
        bool bad = false;
        if (W == 64 && OP != 2) {
            int64_t x = reinterpret_cast<const int64_t *>(a)[c1 ? 0 : i], y = reinterpret_cast<const int64_t *>(b)[c2 ? 0 : i];
            if ((d1 && !d64_scale_up(x, d1)) || (d2 && !d64_scale_up(y, d2))) bad = true;
            else {
                const int64_t z = (int64_t)(OP == 1 ? (uint64_t)x - (uint64_t)y : (uint64_t)x + (uint64_t)y);
                const uint64_t sx = (uint64_t)x >> 63, sy = (uint64_t)y >> 63, sz = (uint64_t)z >> 63;
                bad = OP == 1 ? (sx != sy && sx != sz) : (sx == sy && sx != sz);
                reinterpret_cast<int64_t *>(r)[i] = z;                       // the Go loop stores before it checks (d64AddSameScale :3643-3648)
            }
        } else if (W == 64) {
            const int64_t x = reinterpret_cast<const int64_t *>(a)[c1 ? 0 : i], y = reinterpret_cast<const int64_t *>(b)[c2 ? 0 : i];
            const uint64_t ax = x < 0 ? 0ull - (uint64_t)x : (uint64_t)x, ay = y < 0 ? 0ull - (uint64_t)y : (uint64_t)y;
            uint64_t m[4] = {ax * ay, __umul64hi(ax, ay), 0, 0};
            mag_div_pow10(m, -adj);
            i128 v = (i128)(((u128)m[1] << 64) | m[0]);
            if ((x < 0) != (y < 0)) v = -v;
            reinterpret_cast<Dec128 *>(r)[i] = d128_put(v);
        } else if (OP != 2) {
            i128 x = d128_get(reinterpret_cast<const Dec128 *>(a)[c1 ? 0 : i]), y = d128_get(reinterpret_cast<const Dec128 *>(b)[c2 ? 0 : i]);
            if ((d1 && !d128_scale_up(x, d1)) || (d2 && !d128_scale_up(y, d2))) bad = true;
            else {
                const i128 z = (i128)(OP == 1 ? (u128)x - (u128)y : (u128)x + (u128)y);
                const bool sx = x < 0, sy = y < 0, sz = z < 0;
                bad = OP == 1 ? (sx != sy && sx != sz) : (sx == sy && sx != sz);
                reinterpret_cast<Dec128 *>(r)[i] = d128_put(z);
            }
        } else {
            const i128 x = d128_get(reinterpret_cast<const Dec128 *>(a)[c1 ? 0 : i]), y = d128_get(reinterpret_cast<const Dec128 *>(b)[c2 ? 0 : i]);
            const u128 ax = x < 0 ? (u128)0 - (u128)x : (u128)x, ay = y < 0 ? (u128)0 - (u128)y : (u128)y;
            const uint64_t xl = (uint64_t)ax, xh = (uint64_t)(ax >> 64), yl = (uint64_t)ay, yh = (uint64_t)(ay >> 64);
            uint64_t m[4];
            u128 t = (u128)xl * yl; m[0] = (uint64_t)t; u128 carry = t >> 64;
            t = (u128)xl * yh + carry; const u128 t2 = (u128)xh * yl + (uint64_t)t; m[1] = (uint64_t)t2;
            carry = (t >> 64) + (t2 >> 64);
            t = (u128)xh * yh + carry; m[2] = (uint64_t)t; m[3] = (uint64_t)(t >> 64);
            mag_div_pow10(m, -adj);
            if (m[2] | m[3] | (m[1] >> 63)) bad = true;                      // "Decimal128 Mul overflow" (d128MulInline :722-725)
            else {
                i128 v = (i128)(((u128)m[1] << 64) | m[0]);
                if ((x < 0) != (y < 0)) v = -v;
                reinterpret_cast<Dec128 *>(r)[i] = d128_put(v);
            }
        }
        if (bad) note_failure(first_bad, i);
    }
}

// 128-bit accumulate: lo then hi with the carry of THIS addition; all additions commute mod 2^128
__device__ __forceinline__ void atomic_add128(unsigned long long *acc, uint64_t lo, uint64_t hi) {
    const unsigned long long old = atomicAdd(&acc[0], (unsigned long long)lo);
    const unsigned long long carry = (old + lo) < old ? 1ull : 0ull;
    if (hi + carry) atomicAdd(&acc[1], (unsigned long long)(hi + carry));
}

constexpr int kSumSlots = 512;   // groups kept in shared memory (lo, hi, count)
template <int W, bool SMEM>
__global__ void __launch_bounds__(kThreads)
dec_sum_kernel(const uint64_t *__restrict__ groups, const void *__restrict__ col, const uint64_t *__restrict__ nulls, uint64_t n, uint64_t ngroups,
               unsigned long long *sums, unsigned long long *cnts, unsigned *bad_group) {
    __shared__ unsigned long long s_acc[SMEM ? kSumSlots * 2 : 2];
    __shared__ unsigned long long s_cnt[SMEM ? kSumSlots : 1];
    if (SMEM) {
        for (int s = threadIdx.x; s < (int)ngroups; s += kThreads) { s_acc[2 * s] = 0; s_acc[2 * s + 1] = 0; s_cnt[s] = 0; }
        __syncthreads();
    }
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        const uint64_t g = groups ? groups[i] : 1;
        if (g == 0) continue;
        if (g > ngroups) { *bad_group = 1; continue; }
        if (nulls && ((nulls[i >> 6] >> (i & 63)) & 1ull)) continue;
        uint64_t lo, hi;
        if (W == 64) { const int64_t v = reinterpret_cast<const int64_t *>(col)[i]; lo = (uint64_t)v; hi = v < 0 ? ~0ull : 0ull; }   // Decimal128FromDecimal64: sign extension
        else { const Dec128 v = reinterpret_cast<const Dec128 *>(col)[i]; lo = v.lo; hi = (uint64_t)v.hi; }
        if (SMEM) { atomic_add128(&s_acc[2 * (g - 1)], lo, hi); atomicAdd(&s_cnt[g - 1], 1ull); }
        else { atomic_add128(&sums[2 * (g - 1)], lo, hi); atomicAdd(&cnts[g - 1], 1ull); }
    }
    if (SMEM) {
        __syncthreads();
        for (int s = threadIdx.x; s < (int)ngroups; s += kThreads)
            if (s_cnt[s]) { atomic_add128(&sums[2 * s], s_acc[2 * s], s_acc[2 * s + 1]); atomicAdd(&cnts[s], s_cnt[s]); }
    }
}

template <int OP, int W>
int run_dec_arith(ThreadCtx &t, mo_xcall_args_t *args, uint64_t len) {
    const char *what = "decimal arith";
    const size_t in_sz = W / 8, out_sz = (OP >= 2 || W == 128) ? 16 : 8;
    Stager st(t);
    void *r; uint64_t *rn;
    Operand a, b;
    if (int rc = stage_result(st, args[0], out_sz, len, true, true, what, r, rn)) return rc;
    if (int rc = stage_operand(st, args[1], in_sz, len, what, 1, a)) return rc;
    if (int rc = stage_operand(st, args[2], in_sz, len, what, 2, b)) return rc;
    DecParams P{0, 0, -1, 0, 0};
    if (int rc = read_param(t, args[3], &P, kDecParamsV1, OP == 3 ? sizeof P : kDecParamsV1, "decimal arith: params {scale1, scale2, err_row}")) return rc;
    int d1 = 0, d2 = 0, adj = 0;
    if (OP == 3) {
        if (P.scale1 < 0 || P.scale2 < 0 || P.scale1 > kMaxScale<W>() || P.scale2 > kMaxScale<W>()) { set_error("decimal arith: scales out of range"); return MO_RC_INVALID_ARGUMENT; }
        adj = div_scale(P.scale1) - P.scale1 + P.scale2;
    } else if (OP == 2) { int d = 12; if (P.scale1 > d) d = P.scale1; if (P.scale2 > d) d = P.scale2; if (P.scale1 + P.scale2 < d) d = P.scale1 + P.scale2; adj = d - P.scale1 - P.scale2; }
    else { d1 = P.scale2 > P.scale1 ? P.scale2 - P.scale1 : 0; d2 = P.scale1 > P.scale2 ? P.scale1 - P.scale2 : 0; }
    if (P.scale1 < 0 || P.scale2 < 0 || d1 > (W == 64 ? 18 : 19) || d2 > (W == 64 ? 18 : 19) || -adj > 38) { set_error("decimal arith: scales out of range"); return MO_RC_INVALID_ARGUMENT; }
    RowRecord rec;
    if (int rc = rec.arm(t, st)) return rc;
    bool all_null;   // a const NULL operand nulls every row before a const zero divisor is looked at
    if (int rc = merge_nulls(t, rn, len, a, b, &all_null)) return rc;
    if (!all_null) {
        cudaEventRecord(t.kev0, t.stream);
        dec_arith_kernel<OP, W><<<grid_rows(len, kCtasPerSm), kThreads, 0, t.stream>>>(r, a.data, b.data, len, a.cst, b.cst, d1, d2, adj, rn,
                                                                                      P.div0_error, rec.dev);
        cudaEventRecord(t.kev1, t.stream);
        MOB_LAUNCH_CHECK();
    }
    if (int rc = rec.read(t)) return rc;
    if (int rc = rec.finish(t, st, args[3].pdata, &P, kDecParamsV1, P.err_row)) return rc;
    if (!rec.failed()) return MO_RC_SUCCESS;
    if (rec.kind() == 1) { set_error("division by zero"); return MO_RC_DIVISION_BY_ZERO; }
    if (OP == 3) { set_error("invalid input: Decimal128 Div overflow at row %llu", (unsigned long long)rec.row()); return MO_RC_INVALID_ARGUMENT; }
    set_error("invalid input: Decimal%d %s overflow at row %llu", W, OP == 0 ? "Add" : (OP == 1 ? "Sub" : "Mul"), (unsigned long long)rec.row());
    return MO_RC_INVALID_ARGUMENT;
}

template <int W>
int run_dec_sum(ThreadCtx &t, mo_xcall_args_t *args, uint64_t len) {
    const size_t in_sz = W / 8;
    const uint64_t ngroups = args[0].dataSz / 16;
    if (ngroups == 0 || args[1].dataSz < ngroups * 8 || args[3].dataSz < in_sz * len || (args[2].pdata && args[2].dataSz < 8 * len)) {
        set_error("decimal sum: state (16 bytes per group), counts (8 per group), groups or column too short"); return MO_RC_INVALID_ARGUMENT;
    }
    Stager st(t);
    unsigned long long *sums = (unsigned long long *)st.out(args[0].pdata, ngroups * 16, true);
    unsigned long long *cnts = (unsigned long long *)st.out(args[1].pdata, ngroups * 8, true);
    const uint64_t *groups = (const uint64_t *)st.in(args[2].pdata, args[2].pdata ? len * 8 : 0);
    const void *col = st.in(args[3].pdata, in_sz * len);
    const uint64_t *nulls = (const uint64_t *)st.in(args[3].pnulls, args[3].pnulls ? ((len + 63) / 64) * 8 : 0);
    unsigned *dbad = (unsigned *)st.tmp(4);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dbad, 0, 4, t.stream));
    if (len) {
        const int grid = grid_rows(len, kCtasPerSm);
        cudaEventRecord(t.kev0, t.stream);
        if (ngroups <= (uint64_t)kSumSlots) dec_sum_kernel<W, true><<<grid, kThreads, 0, t.stream>>>(groups, col, nulls, len, ngroups, sums, cnts, dbad);
        else dec_sum_kernel<W, false><<<grid, kThreads, 0, t.stream>>>(groups, col, nulls, len, ngroups, sums, cnts, dbad);
        cudaEventRecord(t.kev1, t.stream);
        MOB_LAUNCH_CHECK();
    }
    unsigned bad = 0;
    int rc = read_back(t, &bad, dbad, 4);
    int frc = st.finish();
    if (rc) return rc;
    if (bad) { set_error("decimal sum: a group id exceeds the state's group count %llu", (unsigned long long)ngroups); return MO_RC_INVALID_ARGUMENT; }
    return frc;
}


// GO_COMPARE(op, DECIMAL64 | DECIMAL128), valueDecimalCompare (func_compare.go:426-667): SIDE 1 scales a up by d, SIDE 2 scales b, SIDE 0
// compares as stored.  Decimal64.Less / Decimal128.Less are signed compares.
template <int W, int SIDE>
__global__ void __launch_bounds__(kThreads)
dec_cmp_kernel(uint8_t *__restrict__ r, const void *__restrict__ a, const void *__restrict__ b, uint64_t n, int c1, int c2, int d, int op,
               const uint64_t *__restrict__ rnulls) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        if (row_null(rnulls, i)) continue;
        bool v;
        if (W == 64) {
            int64_t x = reinterpret_cast<const int64_t *>(a)[c1 ? 0 : i], y = reinterpret_cast<const int64_t *>(b)[c2 ? 0 : i];
            if (SIDE == 1) x = d64_scale_cmp(x, d); else if (SIDE == 2) y = d64_scale_cmp(y, d);
            v = cmp_op(x, y, op);
        } else {
            i128 x = d128_get(reinterpret_cast<const Dec128 *>(a)[c1 ? 0 : i]), y = d128_get(reinterpret_cast<const Dec128 *>(b)[c2 ? 0 : i]);
            if (SIDE == 1) x = d128_scale_cmp(x, d); else if (SIDE == 2) y = d128_scale_cmp(y, d);
            v = cmp_op(x, y, op);
        }
        r[i] = v ? 1 : 0;
    }
}

// AVG's Flush over DEC_SUM's state: decAvg (aggexec/sumavg2.go:545-559) = Decimal128.Div(sum, count) with Div's error dropped; count 0 is
// NULL and keeps the sum as the value.  One warp writes one aligned 32-bit half of the result bitmap.
__global__ void __launch_bounds__(kThreads)
dec_avg_kernel(Dec128 *__restrict__ r, uint32_t *__restrict__ rnulls32, const Dec128 *__restrict__ sums, const int64_t *__restrict__ cnts, uint64_t n,
               int adj) {
    const uint64_t n64 = (n + 63) & ~63ull;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n64; i += (uint64_t)gridDim.x * kThreads) {
        const bool in = i < n;
        const int64_t c = in ? cnts[i] : 0;
        if (in) {
            const Dec128 s = sums[i];
            if (c == 0) r[i] = s;
            else { i128 z; dec_div(d128_get(s), (i128)c, adj, z); r[i] = d128_put(z); }
        }
        const unsigned m = __ballot_sync(0xffffffffu, in && c == 0);
        if ((threadIdx.x & 31) == 0) rnulls32[i >> 5] = m;
    }
}

template <int W>
int run_dec_compare(ThreadCtx &t, int op, mo_xcall_args_t *args, uint64_t len) {
    const char *what = "go compare";
    Stager st(t);
    uint8_t *r; uint64_t *rn;
    Operand a, b;
    if (int rc = stage_result(st, args[0], 1, len, true, true, what, r, rn)) return rc;
    if (int rc = stage_operand(st, args[1], W / 8, len, what, 1, a)) return rc;
    if (int rc = stage_operand(st, args[2], W / 8, len, what, 2, b)) return rc;
    DecParams P{0, 0, -1, 0, 0};
    if (int rc = read_param(t, args[3], &P, kDecParamsV1, kDecParamsV1, "go compare: decimal params {scale1, scale2, err_row}")) return rc;
    if (P.scale1 < 0 || P.scale2 < 0 || P.scale1 > kMaxScale<W>() || P.scale2 > kMaxScale<W>()) {
        set_error("go compare: decimal scales out of range 0..%d", kMaxScale<W>()); return MO_RC_INVALID_ARGUMENT;
    }
    const int m = P.scale2 - P.scale1;
    if (int rc = merge_nulls(t, rn, len, a, b, nullptr)) return rc;   // the const null words are read on the device: no read-back
    cudaEventRecord(t.kev0, t.stream);
    const int grid = grid_rows(len, kCtasPerSm), c1 = a.cst, c2 = b.cst;
    if (m > 0) dec_cmp_kernel<W, 1><<<grid, kThreads, 0, t.stream>>>(r, a.data, b.data, len, c1, c2, m, op, rn);
    else if (m < 0) dec_cmp_kernel<W, 2><<<grid, kThreads, 0, t.stream>>>(r, a.data, b.data, len, c1, c2, -m, op, rn);
    else dec_cmp_kernel<W, 0><<<grid, kThreads, 0, t.stream>>>(r, a.data, b.data, len, c1, c2, 0, op, rn);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.complete();
}

template <int W>
int run_dec_avg(ThreadCtx &t, mo_xcall_args_t *args, uint64_t len) {
    if (args[1].dataSz < 16 * len || args[2].dataSz < 8 * len) {
        set_error("decimal avg: sums (16 bytes per group) or counts (8 per group) shorter than len"); return MO_RC_INVALID_ARGUMENT;
    }
    DecParams P{0, 0, -1, 0, 0};
    if (int rc = read_param(t, args[3], &P, sizeof(int32_t), kDecParamsV1, "decimal avg: params {scale1 = the argument's scale}")) return rc;
    if (P.scale1 < 0 || P.scale1 > kMaxScale<W>()) { set_error("decimal avg: scale out of range 0..%d", kMaxScale<W>()); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    Dec128 *r; uint64_t *rn;
    if (int rc = stage_result(st, args[0], 16, len, false, false, "decimal avg", r, rn)) return rc;
    const Dec128 *sums = (const Dec128 *)st.in(args[1].pdata, 16 * len);
    const int64_t *cnts = (const int64_t *)st.in(args[2].pdata, 8 * len);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    cudaEventRecord(t.kev0, t.stream);
    dec_avg_kernel<<<grid_rows((len + 63) & ~63ull, kCtasPerSm), kThreads, 0, t.stream>>>(r, reinterpret_cast<uint32_t *>(rn), sums, cnts, len,
                                                                               div_scale(P.scale1) - P.scale1);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.complete();
}

}  // namespace

namespace mob {

// MO_XCALL_DEC_ARITH(op, width): args [0] result (+pnulls in/out) ; [1] a ; [2] b ; [3] host params mo_dec_params_t.  See include/mo_b200.h.
int xcall_dec_arith(int op, int width, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    if (width == 64) {
        if (op == 0) return run_dec_arith<0, 64>(t, args, len); if (op == 1) return run_dec_arith<1, 64>(t, args, len);
        if (op == 2) return run_dec_arith<2, 64>(t, args, len); if (op == 3) return run_dec_arith<3, 64>(t, args, len);
    }
    if (width == 128) {
        if (op == 0) return run_dec_arith<0, 128>(t, args, len); if (op == 1) return run_dec_arith<1, 128>(t, args, len);
        if (op == 2) return run_dec_arith<2, 128>(t, args, len); if (op == 3) return run_dec_arith<3, 128>(t, args, len);
    }
    set_error("decimal arith: op 0..3 (+ - * /), width 64 or 128");
    return MO_RC_INVALID_ARGUMENT;
}
// MO_XCALL_GO_COMPARE(op, DECIMAL64 | DECIMAL128), routed here by goelem.cu: args as GO_COMPARE plus [3] mo_dec_params_t (the scales)
int go_dec_compare(ThreadCtx &t, int op, int T, mo_xcall_args_t *args, uint64_t len) {
    return T == MO_T_DECIMAL64 ? run_dec_compare<64>(t, op, args, len) : run_dec_compare<128>(t, op, args, len);
}
// MO_XCALL_DEC_AVG(width): args [0] result Decimal128 per group (+pnulls out) ; [1] sums ; [2] counts (DEC_SUM's state) ; [3] mo_dec_params_t
int xcall_dec_avg(int width, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    if (width == 64) return run_dec_avg<64>(t, args, len);
    if (width == 128) return run_dec_avg<128>(t, args, len);
    set_error("decimal avg: width 64 or 128");
    return MO_RC_INVALID_ARGUMENT;
}
// MO_XCALL_DEC_SUM(width): args [0] sums Decimal128 per group (in/out) ; [1] counts int64 per group (in/out) ; [2] groups uint64[len] or NULL (one group) ; [3] column (+pnulls)
int xcall_dec_sum(int width, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (width == 64) return run_dec_sum<64>(t, args, len);
    if (width == 128) return run_dec_sum<128>(t, args, len);
    set_error("decimal sum: width 64 or 128");
    return MO_RC_INVALID_ARGUMENT;
}

}  // namespace mob
