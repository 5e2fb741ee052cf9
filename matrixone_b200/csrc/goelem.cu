// goelem.cu -- the Go elementwise engine's semantics behind XCall (SURVEY.md section 8, rows a7-a11).
//
// The mo.h surface (elementwise.cu) reproduces the C kernels of cgo/arith.c / compare.c / logic.c: overflow is a flag raised
// after the loop.  The LIVE engine of the reference is the Go one:
//   opBinaryFixedFixedToFixed[WithErrorCheck]   pkg/sql/plan/function/baseTemplate.go:457-578 / 580-728
//   overflow-checked + - *                       arithmetic.go:222-469, arithmetic_overflow_check.go:29-310
//   / and % with the division-by-zero mode       arithmetic.go:481-514, 704-762; baseTemplate.go:1369, 1436
//   compare                                      func_compare.go:285,677,804,931,1058,1185
//   between                                      operator_between.go:138-199
//   n-ary three-valued AND / OR                  logicalOperator.go:36-102, 104-168
// whose operand protocol (const operands, const NULL, skipped rows, the null merge, the first failing row) is goengine.cuh's.  The
// first offending row fails the call with ErrOutOfRange / ErrDivByZero; a zero divisor makes the row NULL when the session's mode says so.
//
// funcIds and argument layout: include/mo_b200.h (MO_XCALL_GO_*).  One thread per row, fully coalesced; the first offender is
// an atomicMin over row numbers, so the error is the one the serial Go loop raises.  Rows before it hold their results, as the
// Go loop leaves them; rows after it are unspecified (Go leaves them unwritten; the batch is discarded on error either way).
#include "goengine.cuh"
#include "keytable.cuh"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <type_traits>

using namespace mob;

namespace {

enum { OP_ADD = 0, OP_SUB, OP_MUL, OP_DIV, OP_MOD };

// ---- overflow-checked scalar arithmetic (arithmetic_overflow_check.go): returns true when the row must fail -----------------
template <typename T> __device__ __forceinline__ bool go_add(T a, T b, T &r) {
    if (std::is_floating_point<T>::value) { r = a + b; return isinf((double)r); }                          // :295-310
    else if (std::is_signed<T>::value) {
        using U = typename std::make_unsigned<typename std::conditional<std::is_floating_point<T>::value, int, T>::type>::type;
        const T s = (T)((U)a + (U)b); r = s;
        return (a > 0 && b > 0 && s <= 0) || (a < 0 && b < 0 && s >= 0);                                   // :32-38
    } else { const T s = (T)(a + b); r = s; return s < a || s < b; }
}
template <typename T> __device__ __forceinline__ bool go_sub(T a, T b, T &r) {
    if (std::is_floating_point<T>::value) { r = a - b; return isinf((double)r); }
    else if (std::is_signed<T>::value) {
        using U = typename std::make_unsigned<typename std::conditional<std::is_floating_point<T>::value, int, T>::type>::type;
        const T s = (T)((U)a - (U)b); r = s;
        return (a > 0 && b < 0 && s < 0) || (a < 0 && b > 0 && s > 0);                                     // :104-112
    } else { r = (T)(a - b); return a < b; }
}
template <typename T> __device__ __forceinline__ bool go_mul(T a, T b, T &r) {
    if (std::is_floating_point<T>::value) { r = a * b; return false; }                                     // unchecked, arithmetic.go:444-451
    else if (std::is_signed<T>::value) {
        using U = typename std::make_unsigned<typename std::conditional<std::is_floating_point<T>::value, int, T>::type>::type;
        if (a == 0 || b == 0) { r = 0; return false; }
        const T tmin = std::numeric_limits<T>::min();
        if ((a == tmin && b == (T)-1) || (b == tmin && a == (T)-1)) { r = 0; return true; }                // :183
        using W = typename std::conditional<(sizeof(T) < 4), unsigned, U>::type;   // no int promotion (uint16 * uint16 would overflow int)
        const T s = (T)((W)(U)a * (W)(U)b); r = s;
        return (T)(s / b) != a;                                                                            // :189
    } else {
        if (a == 0 || b == 0) { r = 0; return false; }
        using W2 = typename std::conditional<(sizeof(T) < 4), unsigned, T>::type;
        r = (T)((W2)a * (W2)b);
        return a > (T)(std::numeric_limits<T>::max() / b);                                                 // :262
    }
}
template <typename T> __device__ __forceinline__ T go_mod(T x, T y) {   // y != 0; arithmetic.go:704-762
    if (std::is_same<T, float>::value) return (T)fmod((double)x, (double)y);
    else if (std::is_same<T, double>::value) return (T)fmod((double)x, (double)y);
    else if (std::is_signed<T>::value) return y == (T)-1 ? (T)0 : (T)(x % y);
    else return (T)(x % y);
}
// integer-only helper so that `%` is never instantiated for floats
template <typename T, bool F = std::is_floating_point<T>::value> struct ModOp { static __device__ __forceinline__ T run(T x, T y) { return go_mod<T>(x, y); } };
template <typename T> struct ModOp<T, true> { static __device__ __forceinline__ T run(T x, T y) { return (T)fmod((double)x, (double)y); } };

template <typename T, int OP>
__global__ void __launch_bounds__(kThreads)
go_arith_kernel(T *__restrict__ r, const T *__restrict__ a, const T *__restrict__ b, uint64_t n, int c1, int c2,
                uint64_t *rnulls, int div0_null, unsigned long long *first_bad) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        if (bm_test(rnulls, i)) continue;                       // bit i is only ever changed by this very thread
        const T x = a[c1 ? 0 : i], y = b[c2 ? 0 : i];
        T v;
        bool bad = false;
        if (OP == OP_DIV || OP == OP_MOD) {
            if (y == (T)0) {
                if (div0_null) atomicOr(reinterpret_cast<unsigned long long *>(&rnulls[i >> 6]), 1ull << (i & 63));
                else note_failure(first_bad, i);
                continue;
            }
            if (OP == OP_DIV) v = (T)(x / y);                   // floats only (the host rejects integer types)
            else v = ModOp<T>::run(x, y);
        } else if (OP == OP_ADD) bad = go_add<T>(x, y, v);
        else if (OP == OP_SUB) bad = go_sub<T>(x, y, v);
        else bad = go_mul<T>(x, y, v);
        if (bad) { note_failure(first_bad, i); continue; }
        r[i] = v;
    }
}

// 8 consecutive rows of a column as 128-bit loads (the group never straddles a bitmap word: 8 | 64)
template <typename T> __device__ __forceinline__ void load8(const T *p, uint64_t i0, bool cst, T *out) {
    if (cst) {
        const T v = p[0];
#pragma unroll
        for (int j = 0; j < 8; j++) out[j] = v;
    } else if (sizeof(T) >= 2) {
        constexpr int NV = (int)(sizeof(T) * 8 / 16);
        const int4 *q = reinterpret_cast<const int4 *>(p + i0);
#pragma unroll
        for (int v = 0; v < NV; v++) { const int4 w = ld_stream16(q + v); memcpy(reinterpret_cast<char *>(out) + 16 * v, &w, 16); }
    } else {
        const uint64_t w = *reinterpret_cast<const uint64_t *>(p + i0);
        memcpy(out, &w, 8);
    }
}

// float32(math.Round(float64(a) * pow) / pow): math.Round = half away from zero = round(); IEEE double multiply / divide
template <typename T> __device__ __forceinline__ T round_scale(T v, double) { return v; }
template <> __device__ __forceinline__ float round_scale<float>(float v, double pw) {
    return pw > 0.0 ? (float)__ddiv_rn(round(__dmul_rn((double)v, pw)), pw) : v;
}

// compare: a thread owns 8 consecutive rows -> one 8-byte store of the bool results when none of them is null
template <typename T>
__global__ void __launch_bounds__(kThreads)
go_compare_kernel(uint8_t *__restrict__ r, const T *__restrict__ a, const T *__restrict__ b, uint64_t n, int c1, int c2,
                  const uint64_t *__restrict__ rnulls, int op, int vec_ok, double pw) {
    // pw > 0 (float32 columns declared with scale > 0, func_compare.go:725-734): both sides are rounded to `scale` decimals first
    const uint64_t ngroups = vec_ok ? n / 8 : 0;
    for (uint64_t g = blockIdx.x * (uint64_t)kThreads + threadIdx.x; g < ngroups; g += (uint64_t)gridDim.x * kThreads) {
        const uint64_t i0 = g * 8;
        const unsigned nb = (unsigned)((rnulls[i0 >> 6] >> (i0 & 63)) & 0xffu);
        if (nb == 0xffu) continue;
        T x[8], y[8];
        load8<T>(a, i0, c1 != 0, x); load8<T>(b, i0, c2 != 0, y);
        uint64_t packed = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) packed |= (uint64_t)(cmp_op<T>(round_scale<T>(x[j], pw), round_scale<T>(y[j], pw), op) ? 1 : 0) << (8 * j);
        if (nb == 0) *reinterpret_cast<uint64_t *>(r + i0) = packed;
        else {
#pragma unroll
            for (int j = 0; j < 8; j++) if (!((nb >> j) & 1u)) r[i0 + j] = (uint8_t)(packed >> (8 * j));
        }
    }
    // rows not covered by whole groups (all rows when the buffers are not 16-byte aligned)
    for (uint64_t i = ngroups * 8 + blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        if (bm_test(rnulls, i)) continue;
        r[i] = cmp_op<T>(round_scale<T>(a[c1 ? 0 : i], pw), round_scale<T>(b[c2 ? 0 : i], pw), op) ? 1 : 0;
    }
}

// rnulls |= n1 | n2 (operands that are not const), tail bits cleared; or "all rows null" (a const NULL operand, known on the host or read
// here from cn1 / cn2, so that a call on resident operands needs no read-back)
__global__ void go_nulls_kernel(uint64_t *rnulls, const uint64_t *n1, const uint64_t *n2, uint64_t n, int all_null, const uint64_t *cn1,
                                const uint64_t *cn2) {
    if ((cn1 && (cn1[0] & 1)) || (cn2 && (cn2[0] & 1))) all_null = 1;
    const uint64_t nw = (n + 63) >> 6;
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < nw; w += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t v = all_null ? ~0ull : rnulls[w];
        if (!all_null) { if (n1) v |= n1[w]; if (n2) v |= n2[w]; }
        if (w == nw - 1 && (n & 63)) { if (all_null) v = rnulls[w] | ((1ull << (n & 63)) - 1); else v &= (1ull << (n & 63)) - 1; }
        rnulls[w] = v;
    }
}

// between: null input -> res = false and the null bit set; one warp covers an aligned 32-row half word of the bitmap
template <typename T>
__global__ void __launch_bounds__(kThreads)
go_between_kernel(uint8_t *__restrict__ r, const T *__restrict__ col, T lo, T hi, uint64_t n, const uint64_t *__restrict__ nulls, uint32_t *rnulls32) {
    const uint64_t n32 = (n + 31) & ~31ull;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n32; i += (uint64_t)gridDim.x * kThreads) {
        const bool in = i < n;
        const bool isnull = in && bm_test(nulls, i);
        if (in) { const T c = col[i]; r[i] = (!isnull && c >= lo && c <= hi) ? 1 : 0; }
        const unsigned m = __ballot_sync(0xffffffffu, isnull);
        if ((threadIdx.x & 31) == 0 && m) rnulls32[i >> 5] |= m;
    }
}

// n-ary three-valued AND / OR, folded left to right exactly as opMultiAnd / opMultiOr do, row by row
struct LogicParam { const uint8_t *col; const uint64_t *nulls; int kind; };   // kind 0 = flat, 1 = const, 2 = const NULL
constexpr int kMaxLogicParams = 16;
struct LogicParams { LogicParam p[kMaxLogicParams]; int n; };
__global__ void __launch_bounds__(kThreads)
go_multi_logic_kernel(uint8_t *__restrict__ r, uint32_t *__restrict__ rnulls32, uint64_t n, LogicParams P, int is_or, int any_null_from) {
    const uint64_t n32 = (n + 31) & ~31ull;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n32; i += (uint64_t)gridDim.x * kThreads) {
        const bool in = i < n;
        bool val = false, isnull = false;
        if (in) {
            const LogicParam p0 = P.p[0];
            if (p0.kind == 2) { val = false; isnull = true; }
            else if (p0.kind == 1) val = p0.col[0] != 0;
            else { val = p0.col[i] != 0; isnull = bm_test(p0.nulls, i); }
            for (int k = 1; k < P.n; k++) {
                const LogicParam pk = P.p[k];
                if (pk.kind == 2) {
                    if (!is_or) { if (val) { val = false; isnull = true; } }
                    else { if (!val) isnull = true; }
                } else if (pk.kind == 1) {
                    const bool c = pk.col[0] != 0;
                    if (!is_or ? !c : c) { val = is_or != 0; isnull = false; }
                } else {
                    const bool a1 = pk.col[i] != 0, null2 = bm_test(pk.nulls, i);
                    // the vector-level "no nulls anywhere" fast path of the reference gives the same per-row result as this branch
                    if (isnull && !null2) {
                        if (!is_or) { if (!a1) { isnull = false; val = false; } }
                        else { if (a1) { isnull = false; val = true; } }
                    } else if (!isnull && null2) {
                        if (!is_or) { if (val) { isnull = true; val = false; } }
                        else { if (!val) isnull = true; }
                    } else if (!isnull && !null2) {
                        val = is_or ? (val || a1) : (val && a1);
                    }
                }
            }
            r[i] = val ? 1 : 0;
        }
        const unsigned m = __ballot_sync(0xffffffffu, in && isnull);
        if ((threadIdx.x & 31) == 0) rnulls32[i >> 5] = m;
    }
    (void)any_null_from;
}

constexpr int kCtasPerSm = 16;

const char *type_name(int T) {
    switch (T) {
    case MO_T_INT8: return "int8"; case MO_T_INT16: return "int16"; case MO_T_INT32: return "int32"; case MO_T_INT64: return "int64";
    case MO_T_UINT8: return "uint8"; case MO_T_UINT16: return "uint16"; case MO_T_UINT32: return "uint32"; case MO_T_UINT64: return "uint64";
    case MO_T_FLOAT32: return "float32"; case MO_T_FLOAT64: return "float64";
    }
    return "?";
}
template <typename T> void fmt_val(char *out, size_t cap, T v) {
    if (std::is_floating_point<T>::value) snprintf(out, cap, "%g", (double)v);
    else if (std::is_signed<T>::value) snprintf(out, cap, "%lld", (long long)v);
    else snprintf(out, cap, "%llu", (unsigned long long)v);
}

struct GoParams { int32_t div0_null; int32_t pad; int64_t err_row; };

template <typename T, int OP>
int run_go_arith(ThreadCtx &t, int Tid, mo_xcall_args_t *args, uint64_t len) {
    const char *what = "go arithmetic";
    Stager st(t);
    T *r; uint64_t *rn;
    Operand a, b;
    if (int rc = stage_result(st, args[0], sizeof(T), len, true, true, what, r, rn)) return rc;
    if (int rc = stage_operand(st, args[1], sizeof(T), len, what, 1, a)) return rc;
    if (int rc = stage_operand(st, args[2], sizeof(T), len, what, 2, b)) return rc;
    GoParams P{0, 0, -1};
    const bool has_params = args[3].pdata && args[3].dataSz >= sizeof P;   // optional
    if (has_params) { int rc = read_param(t, args[3], &P, sizeof P, sizeof P, "go arithmetic: params"); if (rc) return rc; }
    RowRecord rec;
    if (int rc = rec.arm(t, st)) return rc;
    bool all_null;   // a const NULL operand: every row is NULL (baseTemplate.go:600-700)
    if (int rc = merge_nulls(t, rn, len, a, b, &all_null)) return rc;
    const T *pa = (const T *)a.data, *pb = (const T *)b.data;
    if (!all_null) {
        cudaEventRecord(t.kev0, t.stream);
        go_arith_kernel<T, OP><<<grid_rows(len, kCtasPerSm), kThreads, 0, t.stream>>>(r, pa, pb, len, a.cst, b.cst, rn, P.div0_null, rec.dev);
        cudaEventRecord(t.kev1, t.stream);
        MOB_LAUNCH_CHECK();
        if (int rc = rec.read(t)) return rc;
    }
    T xa = 0, xb = 0;
    if (rec.failed()) {   // operands of the offending row for the message (moerr.NewOutOfRange(ctx, "int64", "(%d + %d)", v1, v2))
        read_back(t, &xa, pa + (a.cst ? 0 : rec.row()), sizeof(T));
        read_back(t, &xb, pb + (b.cst ? 0 : rec.row()), sizeof(T));
    }
    if (int rc = rec.finish(t, st, has_params ? args[3].pdata : nullptr, &P, sizeof P, P.err_row)) return rc;
    if (!rec.failed()) return MO_RC_SUCCESS;
    if (OP == OP_DIV || OP == OP_MOD) { set_error("division by zero"); return MO_RC_DIVISION_BY_ZERO; }
    char sa[48], sb[48];
    fmt_val<T>(sa, sizeof sa, xa); fmt_val<T>(sb, sizeof sb, xb);
    set_error("data out of range: data type %s, value '(%s %c %s)'", type_name(Tid), sa, OP == OP_ADD ? '+' : (OP == OP_SUB ? '-' : '*'), sb);
    return MO_RC_OUT_OF_RANGE;
}

template <typename T>
int go_arith_op(ThreadCtx &t, int op, int Tid, mo_xcall_args_t *args, uint64_t len) {
    switch (op) {
    case OP_ADD: return run_go_arith<T, OP_ADD>(t, Tid, args, len);
    case OP_SUB: return run_go_arith<T, OP_SUB>(t, Tid, args, len);
    case OP_MUL: return run_go_arith<T, OP_MUL>(t, Tid, args, len);
    case OP_DIV:
        if (!std::is_floating_point<T>::value) break;   // "/" is defined on floats only (arithmetic.go:481-514)
        return run_go_arith<T, OP_DIV>(t, Tid, args, len);
    case OP_MOD: return run_go_arith<T, OP_MOD>(t, Tid, args, len);
    }
    set_error("go arithmetic: operator %d is not defined for type %d", op, Tid);
    return MO_RC_INVALID_ARGUMENT;
}

template <typename T>
int run_go_compare(ThreadCtx &t, int op, mo_xcall_args_t *args, uint64_t len, double pw = 0.0) {
    const char *what = "go compare";
    Stager st(t);
    uint8_t *r; uint64_t *rn;
    Operand a, b;
    if (int rc = stage_result(st, args[0], 1, len, true, true, what, r, rn)) return rc;
    if (int rc = stage_operand(st, args[1], sizeof(T), len, what, 1, a)) return rc;
    if (int rc = stage_operand(st, args[2], sizeof(T), len, what, 2, b)) return rc;
    bool all_null;   // a const NULL operand: every row is NULL (baseTemplate.go:600-700)
    if (int rc = merge_nulls(t, rn, len, a, b, &all_null)) return rc;
    if (!all_null) {
        const T *pa = (const T *)a.data, *pb = (const T *)b.data;
        cudaEventRecord(t.kev0, t.stream);
        const int vec_ok = ((((uintptr_t)r) | ((uintptr_t)pa) | ((uintptr_t)pb)) & 15) == 0 ? 1 : 0;
        go_compare_kernel<T><<<grid_rows(vec_ok ? (len + 7) / 8 : len, kCtasPerSm), kThreads, 0, t.stream>>>(r, pa, pb, len, a.cst, b.cst, rn, op,
                                                                                                             vec_ok, pw);
        cudaEventRecord(t.kev1, t.stream);
        MOB_LAUNCH_CHECK();
    }
    return st.finish();
}

template <typename T>
int run_go_between(ThreadCtx &t, mo_xcall_args_t *args, uint64_t len) {
    // the column is never const: a one-element column with len > 1 is short
    if (args[1].dataSz < sizeof(T) * len) {
        set_error("go between: the column holds %llu bytes, %llu needed", (unsigned long long)args[1].dataSz, (unsigned long long)(sizeof(T) * len));
        return MO_RC_INVALID_ARGUMENT;
    }
    T lo, hi;
    if (int rc = read_param(t, args[2], &lo, sizeof lo, sizeof lo, "go between: lo")) return rc;
    if (int rc = read_param(t, args[3], &hi, sizeof hi, sizeof hi, "go between: hi")) return rc;
    Stager st(t);
    uint8_t *r; uint64_t *rn;
    if (int rc = stage_result(st, args[0], 1, len, false, true, "go between", r, rn)) return rc;
    const T *col = (const T *)st.in(args[1].pdata, sizeof(T) * len);
    const uint64_t *nulls = (const uint64_t *)st.in(args[1].pnulls, args[1].pnulls ? ((len + 63) / 64) * 8 : 0);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    cudaEventRecord(t.kev0, t.stream);
    go_between_kernel<T><<<grid_rows(len, kCtasPerSm), kThreads, 0, t.stream>>>(r, col, lo, hi, len, nulls, reinterpret_cast<uint32_t *>(rn));
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.finish();
}

int run_go_multi_logic(ThreadCtx &t, int is_or, mo_xcall_args_t *args, uint64_t len) {
    const char *what = "go logic";
    int32_t nparams = 0;
    if (int rc = read_param(t, args[1], &nparams, 4, 4, "go logic: parameter count")) return rc;
    if (nparams < 1 || nparams > kMaxLogicParams) { set_error("go logic: 1..%d operands", kMaxLogicParams); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    uint8_t *r; uint64_t *rn;
    if (int rc = stage_result(st, args[0], 1, len, false, false, what, r, rn)) return rc;
    LogicParams P; P.n = nparams;
    for (int k = 0; k < nparams; k++) {
        Operand o;
        bool is_null;
        if (int rc = stage_operand(st, args[2 + k], 1, len, what, 2 + k, o)) return rc;
        if (int rc = const_null(t, o.cnull(), is_null)) return rc;
        P.p[k] = LogicParam{(const uint8_t *)o.data, o.nulls, is_null ? 2 : (o.cst ? 1 : 0)};
    }
    MOB_CUDA_TRY(cudaMemsetAsync(rn, 0, ((len + 63) / 64) * 8, t.stream));
    cudaEventRecord(t.kev0, t.stream);
    go_multi_logic_kernel<<<grid_rows(len, kCtasPerSm), kThreads, 0, t.stream>>>(r, reinterpret_cast<uint32_t *>(rn), len, P, is_or, 0);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.finish();
}

// ---- IN / NOT IN over fixed-width values (operator_in.go, opOperatorFixedIn): Go's map[T]bool of the list, as a keytable.cuh table.
// Values of 8 bytes or fewer are keyed on their bits (kt_insert / kt_find): mask + 2 key slots, then one word that is 1 when the all-ones
// key is in the set (that key owns slot mask + 1, which kt_find reports as found whether it was inserted or not).  16-byte values (DECIMAL128,
// UUID) are kt_insert_str words, an XXH3 tag and the list index of the value, compared as two 8-byte words: mask + 1 slots.
struct V16 { uint64_t lo, hi; };

// the key of a value; false for a NaN, which no Go map lookup finds.  -0.0 is keyed as +0.0 (they are one key of a Go map).
template <typename T> __device__ __forceinline__ bool in_key(T v, uint64_t &key) {
    if constexpr (std::is_floating_point<T>::value) {
        if (v != v) return false;
        if (v == (T)0) v = (T)0;
    }
    key = 0;
    memcpy(&key, &v, sizeof(T));
    return true;
}
__device__ __forceinline__ uint64_t v16_hash(V16 v) { return xxh3::hash_bytes(reinterpret_cast<const uint8_t *>(&v), 16, 0).lo; }

template <typename T>
__global__ void __launch_bounds__(kThreads) go_in_build_kernel(uint64_t *keys, uint64_t mask, const T *__restrict__ vals,
                                                               const uint64_t *__restrict__ vnulls, uint64_t m) {
    for (uint64_t j = blockIdx.x * (uint64_t)kThreads + threadIdx.x; j < m; j += (uint64_t)gridDim.x * kThreads) {
        uint64_t key, slot;
        if (bm_test(vnulls, j) || !in_key(vals[j], key)) continue;
        if (key == kEmptyKey) keys[mask + 2] = 1;
        else kt_insert(keys, mask, key, slot);
    }
}
__global__ void __launch_bounds__(kThreads) go_in_build16_kernel(uint64_t *slots, uint64_t mask, const V16 *__restrict__ vals,
                                                                 const uint64_t *__restrict__ vnulls, uint64_t m) {
    for (uint64_t j = blockIdx.x * (uint64_t)kThreads + threadIdx.x; j < m; j += (uint64_t)gridDim.x * kThreads) {
        if (bm_test(vnulls, j)) continue;
        const V16 v = vals[j];
        const uint64_t h = v16_hash(v);
        kt_insert_str(slots, mask, h, str_word(h, j), [&](uint32_t r) { const V16 w = vals[r]; return w.lo == v.lo && w.hi == v.hi; });
    }
}

// the probe's view of the set; words == 0: the empty set.  stage() copies the table into shared memory when it fits kInSmemBytes.
struct InTable {
    const uint64_t *t; uint64_t mask, words;
    __device__ __forceinline__ void stage(uint64_t *sm) {
        if (!words || words * 8 > kInSmemBytes) return;
        for (uint64_t k = threadIdx.x; k < words; k += kThreads) sm[k] = t[k];
        __syncthreads();
        t = sm;
    }
};
struct NarrowSet {
    InTable tab;
    template <typename T> __device__ __forceinline__ bool has(T v) const {
        uint64_t key, slot;
        if (!tab.words || !in_key(v, key)) return false;
        return key == kEmptyKey ? tab.t[tab.mask + 2] != 0 : kt_find(tab.t, tab.mask, key, slot);
    }
};
struct WideSet {
    InTable tab; const V16 *vals;
    __device__ __forceinline__ bool has(V16 v) const {
        uint32_t row;
        if (!tab.words) return false;
        return kt_find_str(tab.t, tab.mask, v16_hash(v), [&](uint32_t r) { const V16 w = vals[r]; return w.lo == v.lo && w.hi == v.hi; }, row);
    }
};

// a thread owns 8 consecutive rows, i.e. one byte of the result bitmap, which it writes whole: rnulls | the column's nulls (a const NULL column:
// every row), bits past n cleared.  The loop covers every byte of the last bitmap word.  Rows null on exit are not written.
template <typename T, class Set>
__global__ void __launch_bounds__(kThreads)
go_in_kernel(uint8_t *__restrict__ r, uint8_t *__restrict__ rn8, const T *__restrict__ col, const uint8_t *__restrict__ cn8, int cst,
             uint64_t n, Set set, int negate, int vec_ok) {
    extern __shared__ uint64_t sm_table[];
    set.tab.stage(sm_table);
    const bool cnull = cst && cn8 && (cn8[0] & 1);
    const uint64_t nbytes = ((n + 63) >> 6) * 8;
    for (uint64_t g = blockIdx.x * (uint64_t)kThreads + threadIdx.x; g < nbytes; g += (uint64_t)gridDim.x * kThreads) {
        const uint64_t i0 = g * 8;
        const unsigned valid = i0 >= n ? 0u : (n - i0 >= 8 ? 0xffu : (1u << (n - i0)) - 1);
        unsigned nb = cnull ? 0xffu : rn8[g] | (!cst && cn8 ? cn8[g] : 0u);
        nb &= valid;
        rn8[g] = (uint8_t)nb;
        if (nb == valid) continue;
        if (vec_ok && valid == 0xffu) {
            T x[8];
            load8<T>(col, i0, cst != 0, x);
            uint64_t packed = 0;
#pragma unroll
            for (int j = 0; j < 8; j++) packed |= (uint64_t)(set.has(x[j]) ? 1 ^ negate : negate) << (8 * j);
            if (nb == 0) { *reinterpret_cast<uint64_t *>(r + i0) = packed; continue; }
#pragma unroll
            for (int j = 0; j < 8; j++) if (!((nb >> j) & 1u)) r[i0 + j] = (uint8_t)(packed >> (8 * j));
            continue;
        }
        for (int j = 0; j < 8; j++)
            if (((valid & ~nb) >> j) & 1u) r[i0 + j] = (uint8_t)(set.has(col[cst ? 0 : i0 + j]) ? 1 ^ negate : negate);
    }
}

// launches: the build (nvalues > 0), then the probe.  Every pointer a device one and a host block: enqueue only.
template <typename T>
int run_go_in(ThreadCtx &t, int negate, mo_xcall_args_t *args, uint64_t len) {
    const char *what = negate ? "go not in" : "go in";
    constexpr bool wide = sizeof(T) == 16;
    Stager st(t);
    uint8_t *r; uint64_t *rn;
    Operand a, l;
    uint64_t m, mask;
    if (int rc = stage_result(st, args[0], 1, len, true, true, what, r, rn)) return rc;
    if (int rc = stage_operand(st, args[1], sizeof(T), len, what, 1, a)) return rc;
    if (int rc = stage_in_list(t, st, args, sizeof(T), what, l, m, mask)) return rc;
    InTable tab{nullptr, mask, 0};
    if (m) {
        tab.words = wide ? mask + 1 : mask + 3;
        uint64_t *keys = (uint64_t *)st.tmp(tab.words * 8);
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        MOB_CUDA_TRY(cudaMemsetAsync(keys, 0xff, tab.words * 8, t.stream));
        if (!wide) MOB_CUDA_TRY(cudaMemsetAsync(keys + mask + 2, 0, 8, t.stream));
        if constexpr (wide) go_in_build16_kernel<<<grid_rows(m, kCtasPerSm), kThreads, 0, t.stream>>>(keys, mask, (const V16 *)l.data, l.nulls, m);
        else go_in_build_kernel<T><<<grid_rows(m, kCtasPerSm), kThreads, 0, t.stream>>>(keys, mask, (const T *)l.data, l.nulls, m);
        MOB_LAUNCH_CHECK();
        tab.t = keys;
    }
    const bool smem = tab.words && tab.words * 8 <= kInSmemBytes;
    // every CTA copies the table: fewer, longer-lived CTAs when it is large (about 64 KB of copies per SM)
    const int ctas = smem ? (int)std::max<uint64_t>(2, std::min<uint64_t>(kCtasPerSm, 65536 / (tab.words * 8))) : kCtasPerSm;
    const int vec_ok = ((((uintptr_t)r) | ((uintptr_t)a.data)) & 15) == 0 ? 1 : 0;
    const uint64_t nbytes = ((len + 63) / 64) * 8;
    cudaEventRecord(t.kev0, t.stream);
    if constexpr (wide)
        go_in_kernel<V16, WideSet><<<grid_rows(nbytes, ctas), kThreads, smem ? tab.words * 8 : 0, t.stream>>>(
            r, (uint8_t *)rn, (const V16 *)a.data, (const uint8_t *)a.nulls, a.cst, len, WideSet{tab, (const V16 *)l.data}, negate, vec_ok);
    else
        go_in_kernel<T, NarrowSet><<<grid_rows(nbytes, ctas), kThreads, smem ? tab.words * 8 : 0, t.stream>>>(
            r, (uint8_t *)rn, (const T *)a.data, (const uint8_t *)a.nulls, a.cst, len, NarrowSet{tab}, negate, vec_ok);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.complete();
}

}  // namespace

namespace mob {

int read_const(ThreadCtx &t, void *dst, const void *p, size_t bytes) {
    if (!bytes) return MO_RC_SUCCESS;
    if (!is_device_ptr(p)) { memcpy(dst, p, bytes); return MO_RC_SUCCESS; }
    if (bytes <= t.pinned_sz) return read_back(t, dst, p, bytes);
    MOB_CUDA_TRY(cudaMemcpyAsync(dst, p, bytes, cudaMemcpyDeviceToHost, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    return MO_RC_SUCCESS;
}

int merge_nulls(ThreadCtx &t, uint64_t *rnulls, uint64_t n, const Operand &a, const Operand &b, bool *all_null) {
    bool null1 = false, null2 = false;
    if (all_null) {
        if (int rc = const_null(t, a.cnull(), null1)) return rc;
        if (int rc = const_null(t, b.cnull(), null2)) return rc;
        *all_null = null1 || null2;
    }
    const uint64_t blocks = ((n + 63) / 64 + 255) / 256;
    go_nulls_kernel<<<(unsigned)(blocks > 1024 ? 1024 : blocks), 256, 0, t.stream>>>(rnulls, a.col_nulls(), b.col_nulls(), n, null1 || null2,
                                                                                   all_null ? nullptr : a.cnull(), all_null ? nullptr : b.cnull());
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

int go_str_compare(ThreadCtx &t, int op, mo_xcall_args_t *args, uint64_t len);
int go_dec_compare(ThreadCtx &t, int op, int T, mo_xcall_args_t *args, uint64_t len);

int xcall_go_elementwise(int64_t funcId, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    if (funcId >= 0x4000 && funcId < 0x4800) {
        const int op = (int)((funcId - 0x4000) >> 8), T = (int)(funcId & 0xff);
        switch (T) {
        case MO_T_INT8: return go_arith_op<int8_t>(t, op, T, args, len);
        case MO_T_INT16: return go_arith_op<int16_t>(t, op, T, args, len);
        case MO_T_INT32: return go_arith_op<int32_t>(t, op, T, args, len);
        case MO_T_INT64: return go_arith_op<int64_t>(t, op, T, args, len);
        case MO_T_UINT8: return go_arith_op<uint8_t>(t, op, T, args, len);
        case MO_T_UINT16: return go_arith_op<uint16_t>(t, op, T, args, len);
        case MO_T_UINT32: return go_arith_op<uint32_t>(t, op, T, args, len);
        case MO_T_UINT64: return go_arith_op<uint64_t>(t, op, T, args, len);
        case MO_T_FLOAT32: return go_arith_op<float>(t, op, T, args, len);
        case MO_T_FLOAT64: return go_arith_op<double>(t, op, T, args, len);
        }
        set_error("go arithmetic: unsupported type %d", T);
        return MO_RC_INVALID_ARGUMENT;
    }
    if (funcId >= 0x4800 && funcId < 0x5000) {
        const int op = (int)((funcId - 0x4800) >> 8), T = (int)(funcId & 0xff);
        if (op > CMP_LE) { set_error("go compare: unknown operator %d", op); return MO_RC_INVALID_ARGUMENT; }
        switch (T) {   // DATE compares as int32, TIME / DATETIME / TIMESTAMP as int64 (types.go:187-191); BOOL via false < true
        case MO_T_BOOL: case MO_T_UINT8: return run_go_compare<uint8_t>(t, op, args, len);
        case MO_T_INT8: return run_go_compare<int8_t>(t, op, args, len);
        case MO_T_INT16: return run_go_compare<int16_t>(t, op, args, len);
        case MO_T_INT32: case MO_T_DATE: return run_go_compare<int32_t>(t, op, args, len);
        case MO_T_INT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: return run_go_compare<int64_t>(t, op, args, len);
        case MO_T_UINT16: return run_go_compare<uint16_t>(t, op, args, len);
        case MO_T_UINT32: return run_go_compare<uint32_t>(t, op, args, len);
        case MO_T_UINT64: return run_go_compare<uint64_t>(t, op, args, len);
        case MO_T_FLOAT32: return run_go_compare<float>(t, op, args, len);
        case MO_T_FLOAT64: return run_go_compare<double>(t, op, args, len);
        case MO_T_CHAR: case MO_T_VARCHAR: case MO_T_BINARY: case MO_T_VARBINARY: case MO_T_BLOB: case MO_T_TEXT: case MO_T_DATALINK:
            return go_str_compare(t, op, args, len);   // strpred.cu
        case MO_T_DECIMAL64: case MO_T_DECIMAL128: return go_dec_compare(t, op, T, args, len);   // decimal.cu
        }
        set_error("go compare: unsupported type %d", T);
        return MO_RC_INVALID_ARGUMENT;
    }
    if (funcId >= 0x5200 && funcId < 0x5800) {   // MO_XCALL_GO_COMPARE_F32_SCALE(op, scale)
        const int op = (int)((funcId - 0x5200) >> 8), scale = (int)(funcId & 0xff);
        if (op > CMP_LE || scale < 1 || scale > 22) { set_error("go compare f32 scale: operator 0..5, scale 1..22"); return MO_RC_INVALID_ARGUMENT; }
        double pw = 1.0;
        for (int k = 0; k < scale; k++) pw *= 10.0;   // math.Pow10(scale), exact
        return run_go_compare<float>(t, op, args, len, pw);
    }
    if (funcId >= 0x5000 && funcId < 0x5100) {
        const int T = (int)(funcId & 0xff);
        switch (T) {
        case MO_T_INT8: return run_go_between<int8_t>(t, args, len);
        case MO_T_INT16: return run_go_between<int16_t>(t, args, len);
        case MO_T_INT32: case MO_T_DATE: return run_go_between<int32_t>(t, args, len);
        case MO_T_INT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: return run_go_between<int64_t>(t, args, len);
        case MO_T_UINT8: return run_go_between<uint8_t>(t, args, len);
        case MO_T_UINT16: return run_go_between<uint16_t>(t, args, len);
        case MO_T_UINT32: return run_go_between<uint32_t>(t, args, len);
        case MO_T_UINT64: return run_go_between<uint64_t>(t, args, len);
        case MO_T_FLOAT32: return run_go_between<float>(t, args, len);
        case MO_T_FLOAT64: return run_go_between<double>(t, args, len);
        // CompareDecimal64 / 128 (operator_between.go:68-73): the planner casts the bounds to the column's type, so a raw signed compare (DECIMAL64 as int64, DECIMAL128 as Dec128)
        case MO_T_DECIMAL64: return run_go_between<int64_t>(t, args, len);
        case MO_T_DECIMAL128: return run_go_between<Dec128>(t, args, len);
        }
        set_error("go between: unsupported type %d", T);
        return MO_RC_INVALID_ARGUMENT;
    }
    if (funcId == 0x5100 || funcId == 0x5101) return run_go_multi_logic(t, (int)(funcId & 1), args, len);
    return -1;
}

int go_str_in(ThreadCtx &t, int negate, mo_xcall_args_t *args, uint64_t len);

// MO_XCALL_GO_IN(T) / MO_XCALL_GO_NOT_IN(T): equality is on the raw bits, so the integer types share a kernel per width
int xcall_go_in(int negate, int T, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    switch (T) {
    case MO_T_BOOL: case MO_T_INT8: case MO_T_UINT8: return run_go_in<uint8_t>(t, negate, args, len);
    case MO_T_INT16: case MO_T_UINT16: case MO_T_YEAR: return run_go_in<uint16_t>(t, negate, args, len);
    case MO_T_INT32: case MO_T_UINT32: case MO_T_DATE: return run_go_in<uint32_t>(t, negate, args, len);
    case MO_T_INT64: case MO_T_UINT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: case MO_T_DECIMAL64:
        return run_go_in<uint64_t>(t, negate, args, len);
    case MO_T_FLOAT32: return run_go_in<float>(t, negate, args, len);
    case MO_T_FLOAT64: return run_go_in<double>(t, negate, args, len);
    case MO_T_DECIMAL128: case MO_T_UUID: return run_go_in<V16>(t, negate, args, len);
    case MO_T_CHAR: case MO_T_VARCHAR: case MO_T_TEXT: case MO_T_BLOB: case MO_T_BINARY: case MO_T_VARBINARY:
        return go_str_in(t, negate, args, len);   // strpred.cu
    }
    set_error("%s: unsupported type %d", negate ? "go not in" : "go in", T);
    return MO_RC_INVALID_ARGUMENT;
}

}  // namespace mob
