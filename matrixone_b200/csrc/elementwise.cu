// elementwise.cu -- the cgo/mo.h batch operators: vector arithmetic (cgo/arith.c:316-580), compare
// (cgo/compare.c:153-383), three-valued logic (cgo/logic.c:33-221) and bitmap ops (cgo/mo.c:19-47).
//
// All are one-touch HBM streams: each thread moves 128-bit vectors (V = 16/sizeof(T) rows), the nulls word is a
// warp-broadcast load, results are written with 128-bit stores unless a row of the vector is NULL (reference
// contract: rows whose null bit is set keep their old r[i], arith.c:229-233).  Return codes and the overflow-flag
// quirks of arith.c are reproduced exactly (see the OVERFLOW notes below); they are pinned against the reference C
// compiled unchanged (oracle/_ref/libmo_ref.so) in tests/test_parity_elementwise.py.
//
// Algorithmic bytes per row: 3*sizeof(T) for arithmetic (2 for a scalar operand), 2*sizeof(T)+1 for compare.
#include "common.cuh"
#include <cstring>
#include <type_traits>

using namespace mob;

namespace {

constexpr int kThreads = 256;
constexpr int LEFT_IS_SCALAR = 1, RIGHT_IS_SCALAR = 2;  // cgo/mo_impl.h:37-38
constexpr unsigned ST_OVERFLOW = 1u, ST_DIVZERO = 2u;

enum { AR_ADD = 0, AR_SUB, AR_MUL, AR_DIV, AR_MOD, AR_INTDIV };

template <int BYTES> __device__ __forceinline__ void store_bytes(void *dst, const void *src) {
    if (BYTES == 1) *(uint8_t *)dst = *(const uint8_t *)src;
    else if (BYTES == 2) *(uint16_t *)dst = *(const uint16_t *)src;
    else if (BYTES == 4) *(uint32_t *)dst = *(const uint32_t *)src;
    else if (BYTES == 8) *(uint2 *)dst = *(const uint2 *)src;
    else {
#pragma unroll
        for (int i = 0; i < BYTES / 16; i++) st_stream16((char *)dst + 16 * i, ((const int4 *)src)[i]);
    }
}

// ---- arithmetic functors: return false when the row must not be written (division by zero) -----------------
template <typename T> struct UnsignedOf { using type = typename std::make_unsigned<T>::type; };
template <> struct UnsignedOf<float> { using type = float; };
template <> struct UnsignedOf<double> { using type = double; };

template <typename T, typename R, int OP>
__device__ __forceinline__ bool arith_apply(T a, T b, R &r, unsigned &st) {
    using UT = typename UnsignedOf<T>::type;
    constexpr bool FP = std::is_floating_point<T>::value;
    constexpr bool SG = std::is_signed<T>::value;
    if constexpr (OP == AR_ADD) {
        if constexpr (FP) { r = (R)(a + b); }
        else if constexpr (SG) {
            T s = (T)((UT)a + (UT)b); r = (R)s;
            if ((T)((s ^ a) & (s ^ b)) < 0) st |= ST_OVERFLOW;           // ADD_SIGNED_OVFLAG, arith.c:29-31
        } else { T s = (T)(a + b); r = (R)s; if (s < a) st |= ST_OVERFLOW; }   // ADD_UNSIGNED_OVFLAG :44-48
        return true;
    } else if constexpr (OP == AR_SUB) {
        if constexpr (FP) { r = (R)(a - b); }
        else if constexpr (SG) {
            T s = (T)((UT)a - (UT)b); r = (R)s;
            if ((T)((a ^ b) & (s ^ a)) < 0) st |= ST_OVERFLOW;           // SUB_SIGNED_OVFLAG :69-71
        } else { r = (R)(T)(a - b); if (a < b) st |= ST_OVERFLOW; }      // SUB_UNSIGNED_OVFLAG :84-88
        return true;
    } else if constexpr (OP == AR_MUL) {
        if constexpr (FP) r = (R)(a * b);
        else r = (R)(T)((UT)a * (UT)b);   // TGT = (ZT)temp: low bits of the product; the flag is decided by the LAST row only
        return true;
    } else if constexpr (OP == AR_DIV) {
        if (b == (T)0) { st |= ST_DIVZERO; return false; }               // DIV_FLOAT_OVFLAG :149-152
        r = (R)(a / b); return true;
    } else if constexpr (OP == AR_MOD) {
        if (b == (T)0) { st |= ST_DIVZERO; return false; }               // MOD_*_OVFLAG :163-217
        if constexpr (std::is_same<T, float>::value) r = (R)fmodf(a, b);
        else if constexpr (std::is_same<T, double>::value) r = (R)fmod(a, b);
        else if constexpr (SG) { if (b == (T)-1) r = (R)0; else r = (R)(T)(a % b); }   // INT_MIN % -1 traps on x86; defined here as 0
        else r = (R)(T)(a % b);
        return true;
    } else {
        // AR_INTDIV: (int64_t)(A / B), arith.c:515-521
        if (b == (T)0) { st |= ST_DIVZERO; return false; }
        // the reference C on x86-64 converts with cvttss2si / cvttsd2si, whose out-of-range / NaN result is the "integer indefinite" INT64_MIN;
        // a plain CUDA cast would saturate instead
        const T q = a / b;
        const double qd = (double)q;
        r = (qd >= -9223372036854775808.0 && qd < 9223372036854775808.0) ? (R)(long long)q : (R)(long long)INT64_MIN;
        return true;
    }
}

template <typename T, typename R, int OP>
__global__ void __launch_bounds__(kThreads)
arith_kernel(R *__restrict__ r, const T *__restrict__ a, const T *__restrict__ b, uint64_t n,
             const uint64_t *__restrict__ nulls, int flag, bool vec, unsigned *status) {
    constexpr int V = 16 / sizeof(T);
    const bool as = flag & LEFT_IS_SCALAR, bs = !as && (flag & RIGHT_IS_SCALAR);
    const T a0 = as ? a[0] : T(), b0 = bs ? b[0] : T();
    unsigned st = 0;
    const uint64_t tid = blockIdx.x * (uint64_t)kThreads + threadIdx.x, nthreads = (uint64_t)gridDim.x * kThreads;
    uint64_t done = 0;
    if (vec) {
        const uint64_t nvec = n / V;
        for (uint64_t v = tid; v < nvec; v += nthreads) {
            const uint64_t row0 = v * V;
            T av[V], bv[V]; R rv[V];
            if (!as) { int4 x = ld_stream16(a + row0); memcpy(av, &x, 16); }
            if (!bs) { int4 y = ld_stream16(b + row0); memcpy(bv, &y, 16); }
            const uint32_t nb = nulls ? (uint32_t)((__ldg(nulls + (row0 >> 6)) >> (row0 & 63)) & (V == 32 ? 0xffffffffu : ((1u << V) - 1u))) : 0u;
            uint32_t wr = 0;
#pragma unroll
            for (int j = 0; j < V; j++) {
                if ((nb >> j) & 1u) continue;
                if (arith_apply<T, R, OP>(as ? a0 : av[j], bs ? b0 : bv[j], rv[j], st)) wr |= 1u << j;
            }
            if (wr == (V == 32 ? 0xffffffffu : ((1u << V) - 1u))) store_bytes<sizeof(R) * V>(r + row0, rv);
            else {
#pragma unroll
                for (int j = 0; j < V; j++) if ((wr >> j) & 1u) r[row0 + j] = rv[j];
            }
        }
        done = nvec * V;
    }
    for (uint64_t i = done + tid; i < n; i += nthreads) {
        if (bm_test(nulls, i)) continue;
        R rv;
        if (arith_apply<T, R, OP>(as ? a0 : a[i], bs ? b0 : b[i], rv, st)) r[i] = rv;
    }
    if constexpr (OP != AR_MUL || std::is_floating_point<T>::value) {
        st = __reduce_or_sync(0xffffffffu, st);
        if ((threadIdx.x & 31) == 0 && st) atomicOr(status, st);
    }
}

// OVERFLOW quirk of integer multiply (arith.c:115,129): `opflag = ...` is ASSIGNED per element, so only the last
// processed (= last non-null) row decides the return code.  The formulas below are the macros MUL_SIGNED_OVFLAG /
// MUL_UNSIGNED_OVFLAG with their widening types: int8->int16, int16->int16 (never trips), int32->int64,
// int64->__int128; uint8->uint16, uint16->uint32, uint32->uint64, uint64->signed __int128.
template <typename T>
__global__ void mul_last_row_flag_kernel(const T *a, const T *b, uint64_t n, const uint64_t *nulls, int flag, unsigned *status) {
    int64_t last = -1;
    for (int64_t i = (int64_t)n - 1; i >= 0; i--) if (!bm_test(nulls, (uint64_t)i)) { last = i; break; }
    if (last < 0) return;
    const T A = (flag & LEFT_IS_SCALAR) ? a[0] : a[last];
    const T B = (!(flag & LEFT_IS_SCALAR) && (flag & RIGHT_IS_SCALAR)) ? b[0] : b[last];
    bool ov = false;
    if (std::is_signed<T>::value) {
        const int64_t x = (int64_t)(A ^ B);  // (A ^ B) after integer promotion
        if (sizeof(T) == 1) { short t = (short)((int)A * (int)B); ov = (x > 0 && t > 127) || (x < 0 && t < -128); }
        else if (sizeof(T) == 2) { short t = (short)((int)A * (int)B); ov = (x > 0 && t > 32767) || (x < 0 && t < -32768); }
        else if (sizeof(T) == 4) { long long t = (long long)A * (long long)B; ov = (x > 0 && t > 2147483647LL) || (x < 0 && t < -2147483648LL); }
        else { __int128 t = (__int128)A * (__int128)B; ov = (x > 0 && t > (__int128)INT64_MAX) || (x < 0 && t < (__int128)INT64_MIN); }
    } else {
        if (sizeof(T) == 1) { unsigned short t = (unsigned short)((unsigned)A * (unsigned)B); ov = t > 255; }
        else if (sizeof(T) == 2) { unsigned t = (unsigned)A * (unsigned)B; ov = t > 65535u; }
        else if (sizeof(T) == 4) { unsigned long long t = (unsigned long long)A * (unsigned long long)B; ov = t > 4294967295ull; }
        else { __int128 t = (__int128)((unsigned __int128)(uint64_t)A * (unsigned __int128)(uint64_t)B); ov = t > (__int128)UINT64_MAX; }
    }
    if (ov) atomicOr(status, ST_OVERFLOW);
}

// ---- compare ----------------------------------------------------------------------------------------------
template <typename T, int OP, bool ISBOOL>
__device__ __forceinline__ uint8_t cmp_apply(T a, T b) {
    if (ISBOOL) { a = (T)(a != (T)0); b = (T)(b != (T)0); }   // COMPARE_BOOL_*, compare.c:87-103
    switch (OP) {
    case CMP_EQ: return a == b; case CMP_NE: return a != b; case CMP_GT: return a > b;
    case CMP_GE: return a >= b; case CMP_LT: return a < b; default: return a <= b;
    }
}

template <typename T, int OP, bool ISBOOL>
__global__ void __launch_bounds__(kThreads)
compare_kernel(uint8_t *__restrict__ r, const T *__restrict__ a, const T *__restrict__ b, uint64_t n,
               const uint64_t *__restrict__ nulls, int flag, bool vec) {
    constexpr int V = 16 / sizeof(T);
    const bool as = flag & LEFT_IS_SCALAR, bs = !as && (flag & RIGHT_IS_SCALAR);
    const T a0 = as ? a[0] : T(), b0 = bs ? b[0] : T();
    const uint64_t tid = blockIdx.x * (uint64_t)kThreads + threadIdx.x, nthreads = (uint64_t)gridDim.x * kThreads;
    uint64_t done = 0;
    if (vec) {
        const uint64_t nvec = n / V;
        for (uint64_t v = tid; v < nvec; v += nthreads) {
            const uint64_t row0 = v * V;
            T av[V], bv[V]; uint8_t rv[V];
            if (!as) { int4 x = ld_stream16(a + row0); memcpy(av, &x, 16); }
            if (!bs) { int4 y = ld_stream16(b + row0); memcpy(bv, &y, 16); }
            const uint32_t nb = nulls ? (uint32_t)((__ldg(nulls + (row0 >> 6)) >> (row0 & 63)) & ((1u << V) - 1u)) : 0u;
#pragma unroll
            for (int j = 0; j < V; j++) rv[j] = cmp_apply<T, OP, ISBOOL>(as ? a0 : av[j], bs ? b0 : bv[j]);
            if (nb == 0) store_bytes<V>(r + row0, rv);
            else {
#pragma unroll
                for (int j = 0; j < V; j++) if (!((nb >> j) & 1u)) r[row0 + j] = rv[j];
            }
        }
        done = nvec * V;
    }
    for (uint64_t i = done + tid; i < n; i += nthreads)
        if (!bm_test(nulls, i)) r[i] = cmp_apply<T, OP, ISBOOL>(as ? a0 : a[i], bs ? b0 : b[i]);
}

// ---- logic: one thread per 64 rows (one nulls word) ----------------------------------------------------------
enum { LG_AND = 0, LG_OR, LG_XOR, LG_NOT };

template <int OP>
__global__ void __launch_bounds__(kThreads)
logic_kernel(uint8_t *__restrict__ r, const uint8_t *__restrict__ a, const uint8_t *__restrict__ b, uint64_t n,
             const uint64_t *__restrict__ anulls, const uint64_t *__restrict__ bnulls, uint64_t *__restrict__ rnulls, int flag) {
    const bool as = flag & LEFT_IS_SCALAR, bs = !as && (flag & RIGHT_IS_SCALAR);
    const bool a0 = as ? a[0] != 0 : false, b0 = (bs && b) ? b[0] != 0 : false;
    const uint64_t nwords = (n + 63) >> 6;
    for (uint64_t w = blockIdx.x * (uint64_t)kThreads + threadIdx.x; w < nwords; w += (uint64_t)gridDim.x * kThreads) {
        const uint64_t row0 = w << 6;
        const int m = (int)(n - row0 < 64 ? n - row0 : 64);
        uint64_t am = 0, bmk = 0;  // truth masks
        for (int j = 0; j < m; j++) {
            const bool av = as ? a0 : a[row0 + j] != 0;
            const bool bv = OP == LG_NOT ? false : (bs ? b0 : b[row0 + j] != 0);
            am |= (uint64_t)av << j; bmk |= (uint64_t)bv << j;
            uint8_t rv;
            if (OP == LG_AND) rv = av && bv; else if (OP == LG_OR) rv = av || bv;
            else if (OP == LG_XOR) rv = (av || bv) && !(av && bv); else rv = !av;
            r[row0 + j] = rv;
        }
        if (OP != LG_AND && OP != LG_OR) continue;
        const uint64_t valid = m == 64 ? ~0ull : ((1ull << m) - 1ull);
        // "dominating" value: false for AND, true for OR (logic.c:33-93, 110-170)
        const uint64_t adom = (OP == LG_AND ? ~am : am) & valid, bdom = (OP == LG_AND ? ~bmk : bmk) & valid;
        uint64_t clear = 0;
        if (as) { if (rnulls && (OP == LG_AND ? !a0 : a0)) clear = valid; }
        else if (bs) { if (rnulls && (OP == LG_AND ? !b0 : b0)) clear = valid; }
        else if (anulls && bnulls) { const uint64_t an = anulls[w], bn = bnulls[w]; clear = (an & ~bn & bdom) | (bn & ~an & adom); }
        else if (anulls) clear = anulls[w] & bdom;
        else if (bnulls) clear = bnulls[w] & adom;
        if (clear && rnulls) rnulls[w] &= ~clear;
    }
}

// ---- bitmap ------------------------------------------------------------------------------------------------------
enum { BM_AND = 0, BM_OR, BM_NOT };
template <int OP>
__global__ void bitmap_binop_kernel(uint64_t *dst, const uint64_t *a, const uint64_t *b, uint64_t nwords) {
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < nwords; w += (uint64_t)gridDim.x * blockDim.x)
        dst[w] = OP == BM_AND ? (a[w] & b[w]) : OP == BM_OR ? (a[w] | b[w]) : ~a[w];   // Not flips tail bits too, bitmap.h:103-108
}
__global__ void bitmap_bit_kernel(uint64_t *word, uint64_t mask, int op, int *result) {
    if (op == 0) *word |= mask; else if (op == 1) *word &= ~mask; else *result = (*word & mask) != 0;
}

int grid_for(uint64_t items) {
    uint64_t g = (items + kThreads - 1) / kThreads;
    uint64_t cap = (uint64_t)num_sms() * 8;
    if (g > cap) g = cap;
    return g ? (int)g : 1;
}

bool al16(const void *p) { return (((uintptr_t)p) & 15) == 0; }

template <typename T, typename R, int OP>
int run_arith(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (n == 0) return MO_RC_SUCCESS;
    Stager st(t);
    const bool as = flag & LEFT_IS_SCALAR, bs = !as && (flag & RIGHT_IS_SCALAR);
    const T *da = (const T *)st.in(a, sizeof(T) * (as ? 1 : n));
    const T *db = (const T *)st.in(b, sizeof(T) * (bs ? 1 : n));
    const uint64_t *dn = (const uint64_t *)st.in(nulls, nulls ? ((n + 63) / 64) * 8 : 0);
    // rows may be skipped (NULL / division by zero): start from the caller's current r
    const bool partial = nulls != nullptr || OP == AR_DIV || OP == AR_MOD || OP == AR_INTDIV;
    R *dr = (R *)st.out(r, sizeof(R) * n, partial);
    unsigned *dstatus = (unsigned *)st.tmp(4);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dstatus, 0, 4, t.stream));
    const bool vec = al16(dr) && (as || al16(da)) && (bs || al16(db));
    arith_kernel<T, R, OP><<<grid_for((n + 16 / sizeof(T) - 1) / (16 / sizeof(T))), kThreads, 0, t.stream>>>(dr, da, db, n, dn, flag, vec, dstatus);
    MOB_LAUNCH_CHECK();
    if constexpr (OP == AR_MUL && std::is_integral<T>::value) {
        mul_last_row_flag_kernel<T><<<1, 1, 0, t.stream>>>(da, db, n, dn, flag, dstatus);
        MOB_LAUNCH_CHECK();
    }
    unsigned status = 0;
    int rc = read_back(t, &status, dstatus, 4);
    int frc = st.finish();
    if (rc) return rc;
    if (frc) return frc;
    if (status & ST_DIVZERO) return MO_RC_DIVISION_BY_ZERO;
    if (status & ST_OVERFLOW) return MO_RC_OUT_OF_RANGE;
    return MO_RC_SUCCESS;
}

template <int OP>
int arith_signed(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) {
    switch (szof) {
    case 1: return run_arith<int8_t, int8_t, OP>(r, a, b, n, nulls, flag);
    case 2: return run_arith<int16_t, int16_t, OP>(r, a, b, n, nulls, flag);
    case 4: return run_arith<int32_t, int32_t, OP>(r, a, b, n, nulls, flag);
    case 8: return run_arith<int64_t, int64_t, OP>(r, a, b, n, nulls, flag);
    }
    return MO_RC_INVALID_ARGUMENT;
}
template <int OP>
int arith_unsigned(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) {
    switch (szof) {
    case 1: return run_arith<uint8_t, uint8_t, OP>(r, a, b, n, nulls, flag);
    case 2: return run_arith<uint16_t, uint16_t, OP>(r, a, b, n, nulls, flag);
    case 4: return run_arith<uint32_t, uint32_t, OP>(r, a, b, n, nulls, flag);
    case 8: return run_arith<uint64_t, uint64_t, OP>(r, a, b, n, nulls, flag);
    }
    return MO_RC_INVALID_ARGUMENT;
}
template <int OP>
int arith_float(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) {
    switch (szof) {
    case 4: return run_arith<float, float, OP>(r, a, b, n, nulls, flag);
    case 8: return run_arith<double, double, OP>(r, a, b, n, nulls, flag);
    }
    return MO_RC_INVALID_ARGUMENT;
}

template <typename T, int OP, bool ISBOOL>
int run_compare(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (n == 0) return MO_RC_SUCCESS;
    Stager st(t);
    const bool as = flag & LEFT_IS_SCALAR, bs = !as && (flag & RIGHT_IS_SCALAR);
    const T *da = (const T *)st.in(a, sizeof(T) * (as ? 1 : n));
    const T *db = (const T *)st.in(b, sizeof(T) * (bs ? 1 : n));
    const uint64_t *dn = (const uint64_t *)st.in(nulls, nulls ? ((n + 63) / 64) * 8 : 0);
    uint8_t *dr = (uint8_t *)st.out(r, n, nulls != nullptr);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    const bool vec = al16(dr) && (as || al16(da)) && (bs || al16(db));
    compare_kernel<T, OP, ISBOOL><<<grid_for((n + 16 / sizeof(T) - 1) / (16 / sizeof(T))), kThreads, 0, t.stream>>>(dr, da, db, n, dn, flag, vec);
    MOB_LAUNCH_CHECK();
    return st.finish();
}

template <int OP>
int compare_dispatch(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type) {
    switch (type) {
    case MO_T_INT8: return run_compare<int8_t, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_INT16: return run_compare<int16_t, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_INT32: case MO_T_DATE: return run_compare<int32_t, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_INT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: return run_compare<int64_t, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_UINT8: return run_compare<uint8_t, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_UINT16: return run_compare<uint16_t, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_UINT32: return run_compare<uint32_t, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_UINT64: return run_compare<uint64_t, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_FLOAT32: return run_compare<float, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_FLOAT64: return run_compare<double, OP, false>(r, a, b, n, nulls, flag);
    case MO_T_BOOL: return run_compare<uint8_t, OP, true>(r, a, b, n, nulls, flag);
    }
    return MO_RC_INVALID_ARGUMENT;
}

template <int OP>
int run_logic(void *r, void *a, void *b, uint64_t n, uint64_t *anulls, uint64_t *bnulls, uint64_t *rnulls, int32_t flag) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (n == 0) return MO_RC_SUCCESS;
    if (OP == LG_NOT && (flag & LEFT_IS_SCALAR)) n = 1;  // Logic_VecNot writes only rt[0] for a scalar, logic.c:214-216
    Stager st(t);
    const bool as = flag & LEFT_IS_SCALAR, bs = !as && (flag & RIGHT_IS_SCALAR);
    const size_t nb = ((n + 63) / 64) * 8;
    const uint8_t *da = (const uint8_t *)st.in(a, as ? 1 : n);
    const uint8_t *db = OP == LG_NOT ? nullptr : (const uint8_t *)st.in(b, bs ? 1 : n);
    const uint64_t *dan = (const uint64_t *)st.in(anulls, anulls ? nb : 0);
    const uint64_t *dbn = (const uint64_t *)st.in(bnulls, bnulls ? nb : 0);
    uint64_t *drn = (uint64_t *)st.out(rnulls, rnulls ? nb : 0, true);
    uint8_t *dr = (uint8_t *)st.out(r, n, false);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    logic_kernel<OP><<<grid_for((n + 63) / 64), kThreads, 0, t.stream>>>(dr, da, db, n, dan, dbn, drn, flag);
    MOB_LAUNCH_CHECK();
    return st.finish();
}

template <int OP>
void run_bitmap_binop(uint64_t *dst, uint64_t *a, uint64_t *b, uint64_t nbits) {
    ThreadCtx &t = tctx();
    if (!t.ready || nbits == 0) return;
    const uint64_t nw = (nbits + 63) >> 6;
    Stager st(t);
    const uint64_t *da = (const uint64_t *)st.in(a, nw * 8);
    const uint64_t *db = OP == BM_NOT ? nullptr : (const uint64_t *)st.in(b, nw * 8);
    uint64_t *dd = (uint64_t *)st.out(dst, nw * 8, false);
    if (st.failed) { st.finish(); return; }
    bitmap_binop_kernel<OP><<<grid_for(nw), kThreads, 0, t.stream>>>(dd, da, db, nw);
    g_launches.fetch_add(1);
    st.finish();
}

int run_bitmap_bit(uint64_t *p, uint64_t pos, int op) {
    ThreadCtx &t = tctx();
    if (!t.ready || !p) return 0;
    uint64_t *word = p + (pos >> 6);
    const uint64_t mask = 1ull << (pos & 63);
    Stager st(t);
    uint64_t *dw = (uint64_t *)st.out(word, 8, true);
    int *dres = (int *)st.tmp(4);
    if (st.failed) { st.finish(); return 0; }
    if (op == 2) st.backs.clear();  // Contains does not write the word back
    bitmap_bit_kernel<<<1, 1, 0, t.stream>>>(dw, mask, op, dres);
    g_launches.fetch_add(1);
    int res = 0;
    if (op == 2) read_back(t, &res, dres, 4);
    st.finish();
    return res;
}

}  // namespace

namespace mob { int bitmap_count_device(ThreadCtx &t, const uint64_t *dp, uint64_t nbits, uint64_t *count); }

extern "C" {

void Bitmap_Add(uint64_t *p, uint64_t pos) { run_bitmap_bit(p, pos, 0); }
void Bitmap_Remove(uint64_t *p, uint64_t pos) { run_bitmap_bit(p, pos, 1); }
bool Bitmap_Contains(uint64_t *p, uint64_t pos) { return p ? run_bitmap_bit(p, pos, 2) != 0 : false; }
uint64_t Bitmap_Count(uint64_t *p, uint64_t nbits) {
    ThreadCtx &t = tctx();
    if (!t.ready || nbits == 0 || !p) return 0;
    Stager st(t);
    const uint64_t *dp = (const uint64_t *)st.in(p, ((nbits + 63) / 64) * 8);
    uint64_t c = 0;
    if (!st.failed) bitmap_count_device(t, dp, nbits, &c);
    st.finish();
    return c;
}
bool Bitmap_IsEmpty(uint64_t *p, uint64_t nbits) { return Bitmap_Count(p, nbits) == 0; }
void Bitmap_And(uint64_t *dst, uint64_t *a, uint64_t *b, uint64_t nbits) { run_bitmap_binop<BM_AND>(dst, a, b, nbits); }
void Bitmap_Or(uint64_t *dst, uint64_t *a, uint64_t *b, uint64_t nbits) { run_bitmap_binop<BM_OR>(dst, a, b, nbits); }
void Bitmap_Not(uint64_t *dst, uint64_t *a, uint64_t nbits) { run_bitmap_binop<BM_NOT>(dst, a, nullptr, nbits); }

int32_t SignedInt_VecAdd(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_signed<AR_ADD>(r, a, b, n, nulls, flag, szof); }
int32_t UnsignedInt_VecAdd(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_unsigned<AR_ADD>(r, a, b, n, nulls, flag, szof); }
int32_t Float_VecAdd(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_float<AR_ADD>(r, a, b, n, nulls, flag, szof); }
int32_t SignedInt_VecSub(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_signed<AR_SUB>(r, a, b, n, nulls, flag, szof); }
int32_t UnsignedInt_VecSub(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_unsigned<AR_SUB>(r, a, b, n, nulls, flag, szof); }
int32_t Float_VecSub(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_float<AR_SUB>(r, a, b, n, nulls, flag, szof); }
int32_t SignedInt_VecMul(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_signed<AR_MUL>(r, a, b, n, nulls, flag, szof); }
int32_t UnsignedInt_VecMul(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_unsigned<AR_MUL>(r, a, b, n, nulls, flag, szof); }
int32_t Float_VecMul(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_float<AR_MUL>(r, a, b, n, nulls, flag, szof); }
int32_t Float_VecDiv(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_float<AR_DIV>(r, a, b, n, nulls, flag, szof); }
int32_t Float_VecIntegerDiv(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) {
    switch (szof) {
    case 4: return run_arith<float, int64_t, AR_INTDIV>(r, a, b, n, nulls, flag);
    case 8: return run_arith<double, int64_t, AR_INTDIV>(r, a, b, n, nulls, flag);
    }
    return MO_RC_INVALID_ARGUMENT;
}
int32_t SignedInt_VecMod(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_signed<AR_MOD>(r, a, b, n, nulls, flag, szof); }
int32_t UnsignedInt_VecMod(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_unsigned<AR_MOD>(r, a, b, n, nulls, flag, szof); }
int32_t Float_VecMod(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof) { return arith_float<AR_MOD>(r, a, b, n, nulls, flag, szof); }

int32_t Numeric_VecEq(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type) { return compare_dispatch<CMP_EQ>(r, a, b, n, nulls, flag, type); }
int32_t Numeric_VecNe(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type) { return compare_dispatch<CMP_NE>(r, a, b, n, nulls, flag, type); }
int32_t Numeric_VecGt(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type) { return compare_dispatch<CMP_GT>(r, a, b, n, nulls, flag, type); }
int32_t Numeric_VecGe(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type) { return compare_dispatch<CMP_GE>(r, a, b, n, nulls, flag, type); }
int32_t Numeric_VecLt(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type) { return compare_dispatch<CMP_LT>(r, a, b, n, nulls, flag, type); }
int32_t Numeric_VecLe(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type) { return compare_dispatch<CMP_LE>(r, a, b, n, nulls, flag, type); }

int32_t Logic_VecAnd(void *r, void *a, void *b, uint64_t n, uint64_t *anulls, uint64_t *bnulls, uint64_t *rnulls, int32_t flag) { return run_logic<LG_AND>(r, a, b, n, anulls, bnulls, rnulls, flag); }
int32_t Logic_VecOr(void *r, void *a, void *b, uint64_t n, uint64_t *anulls, uint64_t *bnulls, uint64_t *rnulls, int32_t flag) { return run_logic<LG_OR>(r, a, b, n, anulls, bnulls, rnulls, flag); }
int32_t Logic_VecXor(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag) { (void)nulls; return run_logic<LG_XOR>(r, a, b, n, nullptr, nullptr, nullptr, flag); }
int32_t Logic_VecNot(void *r, void *a, uint64_t n, uint64_t *nulls, int32_t flag) { (void)nulls; return run_logic<LG_NOT>(r, a, nullptr, n, nullptr, nullptr, nullptr, flag); }

}  // extern "C"
