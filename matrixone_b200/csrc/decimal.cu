// decimal.cu -- Decimal64 / Decimal128 batch arithmetic and decimal SUM (SURVEY.md section 8(f) row 1: the reference's native TPC-H
// column type is DECIMAL(15,2), test/distributed/cases/benchmark/tpch/01_DDL/01_create_table.sql:83-86).
//
//   MO_XCALL_DEC_ARITH(op, width)   d64Add / d64Sub / d64Mul / d128Add / d128Sub / d128Mul, pkg/sql/plan/function/arith_decimal_fast.go
//   MO_XCALL_DEC_SUM(width)         sumDecimal64FastExec / sumDecimal128FastExec.batchFill, pkg/sql/colexec/aggexec/sum_decimal_fast.go
//
// Pure integer work, bit-exact: Decimal64 = int64 unscaled value, Decimal128 = two's-complement {B0_63, B64_127}; the scales travel in
// the parameter block.  Conventions are those of the Go elementwise engine (goelem.cu): result nulls pre-filled by the caller
// (NOT selectList), OR-ed with the operand nulls; the FIRST offending row in row order fails the call ("Decimal64 Add overflow",
// "scale overflow", "Decimal128 Mul overflow" -> MO_RC_INVALID_ARGUMENT = moerr ErrInvalidInput) and is reported in the parameter block.
// 128-bit sums are accumulated as two 64-bit atomics with an explicit carry: integer addition is associative, so the result is exact
// and run-to-run identical whatever the order.
#include "common.cuh"
#include <cstring>

using namespace mob;

namespace {

constexpr int kThreads = 256;
constexpr unsigned long long kNoRow = ~0ull;

struct D128 { uint64_t lo, hi; };
typedef unsigned __int128 u128;
typedef __int128 i128;

__device__ __forceinline__ i128 d128_get(D128 v) { return (i128)(((u128)v.hi << 64) | v.lo); }
__device__ __forceinline__ D128 d128_put(i128 x) { D128 r; r.lo = (uint64_t)(u128)x; r.hi = (uint64_t)((u128)x >> 64); return r; }

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

struct DecParams { int32_t scale1, scale2; int64_t err_row; };

__device__ __forceinline__ bool row_null(const uint64_t *rnulls, uint64_t i) { return (rnulls[i >> 6] >> (i & 63)) & 1ull; }

// OP: 0 add, 1 sub, 2 mul.  W: 64 or 128 (operand width).  d64 mul produces d128.
template <int OP, int W>
__global__ void __launch_bounds__(kThreads)
dec_arith_kernel(void *__restrict__ r, const void *__restrict__ a, const void *__restrict__ b, uint64_t n, int c1, int c2, int d1, int d2, int adj,
                 const uint64_t *__restrict__ rnulls, unsigned long long *first_bad) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
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
            reinterpret_cast<D128 *>(r)[i] = d128_put(v);
        } else if (OP != 2) {
            i128 x = d128_get(reinterpret_cast<const D128 *>(a)[c1 ? 0 : i]), y = d128_get(reinterpret_cast<const D128 *>(b)[c2 ? 0 : i]);
            if ((d1 && !d128_scale_up(x, d1)) || (d2 && !d128_scale_up(y, d2))) bad = true;
            else {
                const i128 z = (i128)(OP == 1 ? (u128)x - (u128)y : (u128)x + (u128)y);
                const bool sx = x < 0, sy = y < 0, sz = z < 0;
                bad = OP == 1 ? (sx != sy && sx != sz) : (sx == sy && sx != sz);
                reinterpret_cast<D128 *>(r)[i] = d128_put(z);
            }
        } else {
            const i128 x = d128_get(reinterpret_cast<const D128 *>(a)[c1 ? 0 : i]), y = d128_get(reinterpret_cast<const D128 *>(b)[c2 ? 0 : i]);
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
                reinterpret_cast<D128 *>(r)[i] = d128_put(v);
            }
        }
        if (bad) atomicMin(first_bad, (unsigned long long)i);
    }
}

// rnulls |= n1 | n2 (non-const operands), tail bits cleared; a const NULL operand nulls every row
__global__ void dec_nulls_kernel(uint64_t *rnulls, const uint64_t *n1, const uint64_t *n2, uint64_t n, int all_null) {
    const uint64_t nw = (n + 63) >> 6;
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < nw; w += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t v = all_null ? ~0ull : rnulls[w];
        if (!all_null) { if (n1) v |= n1[w]; if (n2) v |= n2[w]; }
        if (w == nw - 1 && (n & 63)) { if (all_null) v = rnulls[w] | ((1ull << (n & 63)) - 1); else v &= (1ull << (n & 63)) - 1; }
        rnulls[w] = v;
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
        else { const D128 v = reinterpret_cast<const D128 *>(col)[i]; lo = v.lo; hi = v.hi; }
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
    const size_t in_sz = W / 8, out_sz = (OP == 2 || W == 128) ? 16 : 8;
    const uint64_t nwords = (len + 63) / 64;
    const bool c1 = args[1].dataSz == in_sz && len > 1, c2 = args[2].dataSz == in_sz && len > 1;
    if ((!c1 && args[1].dataSz < in_sz * len) || (!c2 && args[2].dataSz < in_sz * len) || args[0].dataSz < out_sz * len || !args[0].pnulls) {
        set_error("decimal arith: vectors shorter than len, or result without a null bitmap"); return MO_RC_INVALID_ARGUMENT;
    }
    DecParams P;
    if (int rc = read_param(t, args[3], &P, sizeof P, sizeof P, "decimal arith: params {scale1, scale2, err_row}")) return rc;
    int d1 = 0, d2 = 0, adj = 0;
    if (OP == 2) { int d = 12; if (P.scale1 > d) d = P.scale1; if (P.scale2 > d) d = P.scale2; if (P.scale1 + P.scale2 < d) d = P.scale1 + P.scale2; adj = d - P.scale1 - P.scale2; }
    else { d1 = P.scale2 > P.scale1 ? P.scale2 - P.scale1 : 0; d2 = P.scale1 > P.scale2 ? P.scale1 - P.scale2 : 0; }
    if (P.scale1 < 0 || P.scale2 < 0 || d1 > (W == 64 ? 18 : 19) || d2 > (W == 64 ? 18 : 19) || -adj > 38) { set_error("decimal arith: scales out of range"); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    void *r = st.out(args[0].pdata, out_sz * len, true);
    uint64_t *rn = (uint64_t *)st.out(args[0].pnulls, nwords * 8, true);
    const void *a = st.in(args[1].pdata, c1 ? in_sz : in_sz * len);
    const void *b = st.in(args[2].pdata, c2 ? in_sz : in_sz * len);
    const uint64_t *n1 = (const uint64_t *)st.in(args[1].pnulls, args[1].pnulls ? (c1 ? 8 : nwords * 8) : 0);
    const uint64_t *n2 = (const uint64_t *)st.in(args[2].pnulls, args[2].pnulls ? (c2 ? 8 : nwords * 8) : 0);
    unsigned long long *dbad = (unsigned long long *)st.tmp(8);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    uint64_t h1 = 0, h2 = 0;
    if (c1 && n1) { int rc = read_back(t, &h1, n1, 8); if (rc) { st.finish(); return rc; } }
    if (c2 && n2) { int rc = read_back(t, &h2, n2, 8); if (rc) { st.finish(); return rc; } }
    const bool all_null = (c1 && (h1 & 1)) || (c2 && (h2 & 1));
    MOB_CUDA_TRY(cudaMemsetAsync(dbad, 0xff, 8, t.stream));
    dec_nulls_kernel<<<(unsigned)((nwords + 255) / 256 > 1024 ? 1024 : (nwords + 255) / 256), 256, 0, t.stream>>>(rn, c1 ? nullptr : n1, c2 ? nullptr : n2, len, all_null ? 1 : 0);
    MOB_LAUNCH_CHECK();
    if (!all_null) {
        int grid = num_sms() * 8;
        const uint64_t work = (len + kThreads - 1) / kThreads;
        if ((uint64_t)grid > work) grid = (int)work;
        cudaEventRecord(t.kev0, t.stream);
        dec_arith_kernel<OP, W><<<grid, kThreads, 0, t.stream>>>(r, a, b, len, c1 ? 1 : 0, c2 ? 1 : 0, d1, d2, adj, rn, dbad);
        cudaEventRecord(t.kev1, t.stream);
        MOB_LAUNCH_CHECK();
    }
    unsigned long long bad = kNoRow;
    int rc = read_back(t, &bad, dbad, 8);
    if (rc) { st.finish(); return rc; }
    int frc = st.finish();
    P.err_row = bad == kNoRow ? -1 : (int64_t)bad;
    const int wrc = write_param(t, args[3].pdata, &P, sizeof P);
    if (frc || wrc) return frc ? frc : wrc;
    if (bad == kNoRow) return MO_RC_SUCCESS;
    set_error("invalid input: Decimal%d %s overflow at row %llu", W, OP == 0 ? "Add" : (OP == 1 ? "Sub" : "Mul"), bad);
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
        int grid = num_sms() * 8;
        const uint64_t work = (len + kThreads - 1) / kThreads;
        if ((uint64_t)grid > work) grid = (int)work;
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

}  // namespace

namespace mob {

// MO_XCALL_DEC_ARITH(op, width): args [0] result (+pnulls in/out) ; [1] a ; [2] b ; [3] host params mo_dec_params_t.  See include/mo_b200.h.
int xcall_dec_arith(int op, int width, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    if (width == 64) { if (op == 0) return run_dec_arith<0, 64>(t, args, len); if (op == 1) return run_dec_arith<1, 64>(t, args, len); if (op == 2) return run_dec_arith<2, 64>(t, args, len); }
    if (width == 128) { if (op == 0) return run_dec_arith<0, 128>(t, args, len); if (op == 1) return run_dec_arith<1, 128>(t, args, len); if (op == 2) return run_dec_arith<2, 128>(t, args, len); }
    set_error("decimal arith: op 0..2 (+ - *), width 64 or 128");
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
