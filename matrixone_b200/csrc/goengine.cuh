// goengine.cuh -- the operand protocol of the Go expression calls: GO_ARITH, GO_COMPARE, GO_COMPARE_F32_SCALE, GO_BETWEEN, MULTI_AND / OR
// (goelem.cu), varlena GO_COMPARE and GO_LIKE (strpred.cu), DEC_ARITH, decimal GO_COMPARE and DEC_AVG (decimal.cu), GO_IN / GO_NOT_IN
// (goelem.cu, its varlena types in strpred.cu), and GO_CASE / GO_COALESCE (caseexpr.cu), which stage their operands here but apply no null
// merge: a NULL operand only matters on the rows that choose it.
//
// Every one of these calls follows the Go engine's per-batch template (pkg/sql/plan/function/baseTemplate.go:457-728), and this header is
// the one place that implements it:
//   - a const operand is a one-element vector (dataSz == the element size) when len > 1; with len == 1 a one-element operand is a column;
//   - a const NULL operand (bit 0 of its null word) nulls every row;
//   - rows whose result null bit is set on entry are skipped (the caller pre-fills the bitmap with NOT selectList, baseTemplate.go:473-486);
//   - the result bitmap leaves as rnulls | n1 | n2;
//   - the first failing row in row order fails the call, and its index goes to the parameter block's err_row.
// Each entry point keeps only what is its own: its parameter block, the kernel it launches, and how it turns a failure into a message.
#pragma once
#include <cstdio>
#include "column.cuh"

namespace mob {

constexpr int kThreads = 256;                 // every row kernel of the Go expression calls
constexpr unsigned long long kNoRow = ~0ull;

// row-grid sizing: one thread per row up to ctas_per_sm CTAs per SM, grid-stride beyond
inline int grid_rows(uint64_t n, int ctas_per_sm) {
    const uint64_t b = (n + kThreads - 1) / kThreads, cap = (uint64_t)num_sms() * ctas_per_sm;
    return (int)(b > cap ? cap : (b ? b : 1));
}

// ---- operands: Operand, is_const, stage_operand and stage_rows (column.cuh)

// ---- IN / NOT IN (goelem.cu, strpred.cu): the list of args[2] with nvalues from the mo_in_params_t of args[3]; the set's hash table has
// the least power-of-two slot count >= 2 * nvalues (load <= 1/2, so kt_find / kt_find_str always meet an empty slot), and the probe copies
// a table of at most kInSmemBytes into each CTA's shared memory, reading it from global memory (L2) otherwise
constexpr uint64_t kInSmemBytes = 16384;
constexpr int64_t kInMaxValues = 0x7fffffff;   // list indices fit the 31-bit row of a kt_insert_str word
inline int stage_in_list(ThreadCtx &t, Stager &st, mo_xcall_args_t *args, size_t elem, const char *what, Operand &l, uint64_t &m, uint64_t &mask) {
    mo_in_params_t P;
    char pw[64];
    snprintf(pw, sizeof pw, "%s: params", what);
    if (int rc = read_param(t, args[3], &P, sizeof P, sizeof P, pw)) return rc;
    if (P.nvalues < 0 || P.nvalues > kInMaxValues) {
        set_error("%s: nvalues %lld outside 0..%lld", what, (long long)P.nvalues, (long long)kInMaxValues);
        return MO_RC_INVALID_ARGUMENT;
    }
    m = (uint64_t)P.nvalues;
    l = Operand{};
    mask = 0;
    if (!m) return MO_RC_SUCCESS;
    uint64_t cap = 2;
    while (cap < 2 * m) cap <<= 1;
    mask = cap - 1;
    if (int rc = stage_rows(st, args[2], elem, m, what, 2, l)) return rc;
    // a host list whose elements are all NULL is the empty set, known without a read-back: no table and no build (a device list's null
    // words stay on the device, and its build inserts nothing)
    const uint64_t *w = (const uint64_t *)args[2].pnulls;
    if (!w || is_device_ptr(w)) return MO_RC_SUCCESS;
    for (uint64_t k = 0; k < m / 64; k++) if (w[k] != ~0ull) return MO_RC_SUCCESS;
    if ((m & 63) && (~w[m / 64] & ((1ull << (m & 63)) - 1))) return MO_RC_SUCCESS;
    m = mask = 0;
    return MO_RC_SUCCESS;
}

// stages the result args[0] and its required null bitmap; preload_* uploads a host buffer's content first (the kernel leaves rows alone)
template <typename T = void>
inline int stage_result(Stager &st, const mo_xcall_args_t &r, size_t elem, uint64_t len, bool preload_data, bool preload_nulls,
                        const char *what, T *&data, uint64_t *&nulls) {
    if (!r.pdata || r.dataSz < elem * len) {
        set_error("%s: the result holds %llu bytes, %llu needed", what, (unsigned long long)r.dataSz, (unsigned long long)(elem * len));
        return MO_RC_INVALID_ARGUMENT;
    }
    if (!r.pnulls) { set_error("%s: the result has no null bitmap", what); return MO_RC_INVALID_ARGUMENT; }
    data = (T *)st.out(r.pdata, elem * len, preload_data);
    nulls = (uint64_t *)st.out(r.pnulls, ((len + 63) / 64) * 8, preload_nulls);
    return st.failed ? MO_RC_INTERNAL_ERROR : MO_RC_SUCCESS;
}

// ---- const NULL: a const operand's bytes on the host -- copied from host memory, read back from device memory (one synchronise).  The
// calls that skip their row kernel on an all-NULL batch read the staged null word this way, and GO_LIKE its const pattern.
int read_const(ThreadCtx &t, void *dst, const void *p, size_t bytes);
inline int const_null(ThreadCtx &t, const uint64_t *word, bool &is_null) {
    uint64_t w = 0;
    if (word) { if (int rc = read_const(t, &w, word, 8)) return rc; }
    is_null = w & 1;
    return MO_RC_SUCCESS;
}

// ---- the null merge, one launch (goelem.cu): rnulls |= the column operands' bitmaps, bits past n cleared; a const NULL operand nulls every
// row (the bits past n kept).  all_null: the const null words are read back first and *all_null tells the caller to skip its row kernel;
// nullptr: the kernel reads them on the device, so the call needs no read-back (decimal GO_COMPARE stays enqueue-only).
int merge_nulls(ThreadCtx &t, uint64_t *rnulls, uint64_t n, const Operand &a, const Operand &b, bool *all_null);

// ---- the first failing row: one 64-bit word min-reduced over 2 * row + kind, so the lowest row wins and its kind (0 or 1, the caller's)
// says why
#ifdef __CUDACC__
__device__ __forceinline__ void note_failure(unsigned long long *rec, uint64_t row, unsigned kind = 0) { atomicMin(rec, 2ull * row + kind); }
#endif
struct RowRecord {
    unsigned long long *dev = nullptr;
    unsigned long long bad = kNoRow;
    // the device word, set to "no row" on the stream
    int arm(ThreadCtx &t, Stager &st) {
        dev = (unsigned long long *)st.tmp(8);
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        MOB_CUDA_TRY(cudaMemsetAsync(dev, 0xff, 8, t.stream));
        return MO_RC_SUCCESS;
    }
    int read(ThreadCtx &t) { return read_back(t, &bad, dev, 8); }   // synchronises
    bool failed() const { return bad != kNoRow; }
    uint64_t row() const { return bad >> 1; }
    unsigned kind() const { return (unsigned)(bad & 1); }
    // copies back and synchronises (rows before the failing one reach host results), then writes err_row (-1: none) into the caller's
    // parameter block `block` (none: nullptr) as the first `bytes` of P
    int finish(ThreadCtx &t, Stager &st, void *block, const void *P, size_t bytes, int64_t &err_row) {
        if (int rc = st.finish()) return rc;
        err_row = failed() ? (int64_t)row() : -1;
        return block ? write_param(t, block, P, bytes) : MO_RC_SUCCESS;
    }
};

// ---- shared device pieces
#ifdef __CUDACC__
template <typename T> __device__ __forceinline__ bool cmp_op(T x, T y, int op) {
    switch (op) {
    case CMP_EQ: return x == y; case CMP_NE: return x != y;
    case CMP_GT: return x > y;  case CMP_GE: return x >= y;
    case CMP_LT: return x < y;  default: return x <= y;
    }
}
#endif

// a Decimal128 as stored {B0_63, B64_127}: two 8-byte words, so a column needs only 8-byte alignment; orders as a signed 128-bit value
struct Dec128 { uint64_t lo; int64_t hi; };
__host__ __device__ __forceinline__ bool operator<(const Dec128 &x, const Dec128 &y) { return x.hi != y.hi ? x.hi < y.hi : x.lo < y.lo; }
__host__ __device__ __forceinline__ bool operator>=(const Dec128 &x, const Dec128 &y) { return !(x < y); }
__host__ __device__ __forceinline__ bool operator<=(const Dec128 &x, const Dec128 &y) { return !(y < x); }

}  // namespace mob
