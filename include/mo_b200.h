/*
 * mo_b200.h -- C-ABI of libmo_b200.so, the H100 (sm_90a) implementation of MatrixOne's per-block batch
 * operators and vector-distance kernels.
 *
 * PART 1 is the reference's cgo surface, byte for byte the same prototypes as /root/reference/cgo/mo.h:24-73
 * (Bitmap_*, {SignedInt,UnsignedInt,Float}_Vec*, Numeric_Vec*, Logic_Vec*, XCall), so the Go side
 * (pkg/common/bitmap/cbitmap.go:33-50, pkg/sql/plan/function/cxcall.go:78-83) binds to it unchanged.
 * Rules kept from cgo/README.md:12-16: only fixed-width ints, float/double and pointers cross the boundary.
 *
 * Every pointer argument may be either a HOST pointer (pageable or pinned; the library stages it through the
 * calling thread's stream) or a DEVICE pointer obtained from MoB200_DeviceAlloc (zero-copy, the resident path).
 * The library classifies each pointer with cudaPointerGetAttributes.  All pointers of one call must live on the
 * same side unless stated otherwise.  Buffers stay owned by the caller (cgo/README.md:21-23).
 *
 * PART 2 declares the XCall argument block (reference cgo/xcall.h:24-31) and the funcIds this library adds
 * (>= 100; ids 0..3 keep the reference meaning, cgo/mo.c:49-52).
 *
 * PART 3 is the residency/runtime extension (device + pinned allocation, copies, stream adoption, timers).
 */
#ifndef _MO_B200_H_
#define _MO_B200_H_

#include <stdint.h>
#include <stdbool.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ======================================================================================================
 * PART 1 -- reference ABI (cgo/mo.h)
 * ==================================================================================================== */

/* Bitmap ops -- replaces cgo/mo.c:19-47 (bodies in cgo/bitmap.h:47-149).  LSB-first uint64 words, set = NULL. */
void Bitmap_Add(uint64_t *p, uint64_t pos);
void Bitmap_Remove(uint64_t *p, uint64_t pos);
bool Bitmap_Contains(uint64_t *p, uint64_t pos);
bool Bitmap_IsEmpty(uint64_t *p, uint64_t nbits);
uint64_t Bitmap_Count(uint64_t *p, uint64_t nbits);
void Bitmap_And(uint64_t *dst, uint64_t *a, uint64_t *b, uint64_t nbits);
void Bitmap_Or(uint64_t *dst, uint64_t *a, uint64_t *b, uint64_t nbits);
void Bitmap_Not(uint64_t *dst, uint64_t *a, uint64_t nbits);

/* Vector arithmetic -- replaces cgo/arith.c:316-580.  flag&1: a is scalar, flag&2: b is scalar
 * (cgo/mo_impl.h:37-38).  Rows whose bit is set in `nulls` are skipped (r[i] untouched).
 * Return codes as cgo/mo_impl.h:26-35 (see MO_RC_* below); overflow-flag quirks of arith.c are reproduced. */
int32_t SignedInt_VecAdd(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t UnsignedInt_VecAdd(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t Float_VecAdd(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);

int32_t SignedInt_VecSub(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t UnsignedInt_VecSub(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t Float_VecSub(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);

int32_t SignedInt_VecMul(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t UnsignedInt_VecMul(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t Float_VecMul(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);

int32_t Float_VecDiv(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t Float_VecIntegerDiv(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);

int32_t SignedInt_VecMod(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t UnsignedInt_VecMod(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);
int32_t Float_VecMod(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t szof);

/* Compare -- replaces cgo/compare.c:153-383.  r is bool[n] (1 byte each); `type` is a types.T id (MO_T_*). */
int32_t Numeric_VecEq(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type);
int32_t Numeric_VecNe(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type);
int32_t Numeric_VecGt(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type);
int32_t Numeric_VecGe(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type);
int32_t Numeric_VecLt(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type);
int32_t Numeric_VecLe(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag, int32_t type);

/* Three-valued logic -- replaces cgo/logic.c:33-221.  The caller pre-fills rnulls = anulls | bnulls;
 * And/Or clear the bits where the other operand dominates. */
int32_t Logic_VecAnd(void *r, void *a, void *b, uint64_t n, uint64_t *anulls, uint64_t *bnulls, uint64_t *rnulls, int32_t flag);
int32_t Logic_VecOr(void *r, void *a, void *b, uint64_t n, uint64_t *anulls, uint64_t *bnulls, uint64_t *rnulls, int32_t flag);
int32_t Logic_VecXor(void *r, void *a, void *b, uint64_t n, uint64_t *nulls, int32_t flag);
int32_t Logic_VecNot(void *r, void *a, uint64_t n, uint64_t *nulls, int32_t flag);

/* XCall -- replaces cgo/mo.c:54-68.  runtimeId: 0 = "C", 1 = "CUDA" (cgo/xcall.h:44-45); this library runs every
 * funcId on the GPU for BOTH runtime ids (there is no CPU implementation inside it).  errStr is the reference's
 * 256-byte Pascal string: errStr[0] = length, text from errStr[1] (cgo/cuda/cuda.cpp:45-58, cxcall.go:76-89).
 * args -> xcall_args_t[]: index 0 = result vector, 1..k = inputs.  Unknown funcId returns -1. */
int32_t XCall(int64_t runtimeId, int64_t funcId, uint8_t *errStr, uint64_t *args, uint64_t len);

/* ======================================================================================================
 * PART 2 -- XCall argument block, type ids, return codes, funcIds
 * ==================================================================================================== */

/* cgo/xcall.h:24-31; filled by Vector.FillRawPtrLen, pkg/container/vector/vector.go:5161-5172 */
typedef struct mo_xcall_args_t {
    uint64_t *pnulls;  /* nulls bitmap words or NULL */
    uint64_t nullCnt;  /* bitmap length IN BITS (field misnamed in the reference) */
    uint8_t *pdata;    /* fixed-width values, or 24-byte varlena cells */
    uint64_t dataSz;   /* bytes; typeSize*1 for a const vector */
    uint8_t *parea;    /* varlena payload area or NULL */
    uint64_t areaSz;
} mo_xcall_args_t;

#define MO_VARLENA_SZ 24         /* cgo/xcall.h:33 */
#define MO_VARLENA_INLINE_SZ 23

#define MO_RUNTIME_C 0
#define MO_RUNTIME_CUDA 1

/* return codes, cgo/mo_impl.h:26-35 */
#define MO_RC_SUCCESS 0
#define MO_RC_INTERNAL_ERROR 20101
#define MO_RC_DIVISION_BY_ZERO 20200
#define MO_RC_OUT_OF_RANGE 20201
#define MO_RC_DATA_TRUNCATED 20202
#define MO_RC_INVALID_ARGUMENT 20203

/* types.T ids, pkg/container/types/types.go:35-67 == cgo/compare.c:20-38 */
#define MO_T_BOOL 10
#define MO_T_INT8 20
#define MO_T_INT16 21
#define MO_T_INT32 22
#define MO_T_INT64 23
#define MO_T_UINT8 25
#define MO_T_UINT16 26
#define MO_T_UINT32 27
#define MO_T_UINT64 28
#define MO_T_FLOAT32 30
#define MO_T_FLOAT64 31
#define MO_T_DATE 50
#define MO_T_TIME 51
#define MO_T_DATETIME 52
#define MO_T_TIMESTAMP 53
#define MO_T_DECIMAL64 32
#define MO_T_DECIMAL128 33
#define MO_T_BIT 11
#define MO_T_YEAR 55
#define MO_T_UUID 63
#define MO_T_ENUM 66
/* varlena types: 24-byte cells + area (cgo/xcall.h:47-61) */
#define MO_T_CHAR 60
#define MO_T_VARCHAR 61
#define MO_T_BINARY 64
#define MO_T_VARBINARY 65
#define MO_T_BLOB 70
#define MO_T_TEXT 71
#define MO_T_DATALINK 72

/* reference funcIds, cgo/mo.c:49-52 == cxcall.go:33-38.  args: [0] f64 result, [1] vec col, [2] vec col
 * (varlena cells; either side may be const: dataSz == 24).  Semantics of cgo/xcall.c:23-134:
 * float diff, squares accumulated in double, optional sqrt. */
#define MO_XCALL_L2DISTANCE_F32 0
#define MO_XCALL_L2DISTANCE_F64 1
#define MO_XCALL_L2DISTANCE_SQ_F32 2
#define MO_XCALL_L2DISTANCE_SQ_F64 3

/* --- new: row-wise distances with the Go semantics of pkg/vectorindex/metric/distance_func.go (accumulator type =
 * element type, 8-way unrolled association), i.e. what the SQL builtins l2_distance / l2_distance_sq / inner_product /
 * cosine_distance / cosine_similarity compute (pkg/vectorize/moarray/external.go:171-260).  Same 3-arg layout as
 * ids 0..3, result float64[len].  Bit-exact with the Go loops.  dim mismatch -> MO_RC_INVALID_ARGUMENT. */
#define MO_XCALL_GO_L2_F32 100
#define MO_XCALL_GO_L2_F64 101
#define MO_XCALL_GO_L2SQ_F32 102
#define MO_XCALL_GO_L2SQ_F64 103
#define MO_XCALL_GO_IP_F32 104
#define MO_XCALL_GO_IP_F64 105
#define MO_XCALL_GO_COSDIST_F32 106
#define MO_XCALL_GO_COSDIST_F64 107
#define MO_XCALL_GO_COSSIM_F32 108
#define MO_XCALL_GO_COSSIM_F64 109
#define MO_XCALL_GO_L1_F32 110   /* metric.L1Distance, distance_func.go:112-154 (l1_norm of the difference) */
#define MO_XCALL_GO_L1_F64 111
/* normalize_l2(v): moarray.NormalizeL2 (pkg/vectorize/moarray/external.go:262-285): a VECTOR-valued result.
 * args: [0] the result varlena vector (pdata -> 24 * len cells, parea / areaSz -> its area, at least as large as the
 * argument's: the result area MIRRORS the argument's layout -- cell i gets the same (offset, length), inline cells
 * stay inline; pnulls = the result nulls, rows set there are skipped and get an empty cell) ; [1] the argument vector
 * (dataSz == 24: const).  sumSquares in float64 in index order, normalized[i] = T(float64(v[i]) / norm), norm == 0
 * copies the row; an empty non-null vector -> MO_RC_INTERNAL_ERROR "cannot normalize empty vector". */
#define MO_XCALL_GO_NORMALIZE_L2_F32 112
#define MO_XCALL_GO_NORMALIZE_L2_F64 113

/* --- new: single-column aggregates (aggexec sumavg2.go / count2.go / minmax2.go semantics, no group-by = H0).
 * funcId = MO_XCALL_AGG(op, T).  args: [0] result: pdata -> one 8-byte value (int64 / uint64 / float64, or the
 * column type for MIN/MAX, zero-extended), pnulls -> 1-word bitmap, bit 0 set when the result is NULL
 * (all-null input); [1] the column (fixed width, pnulls optional).  len = rows.
 * SUM over signed ints returns MO_RC_OUT_OF_RANGE exactly when the serial Go loop would (int64OfCheck).  MIN / MAX return the bits of
 * the first row that reaches the extreme, as the serial loop's strict compare does: -0.0 and 0.0 tie, so the zero of the earlier row is
 * kept, and a NaN in the first non-null row is kept with its payload. */
#define MO_AGG_SUM 0
#define MO_AGG_COUNT 1   /* COUNT(col): non-null rows; result int64 */
#define MO_AGG_MIN 2
#define MO_AGG_MAX 3
#define MO_AGG_AVG 4     /* result float64 = sum/cnt, NULL when cnt == 0 */
#define MO_XCALL_AGG(op, T) (0x1000 + ((op) << 8) + (T))
/* Wider results: dataSz >= 16 adds the non-null row count at pdata+8; dataSz >= 24 makes the result a PARTIAL STATE
 * mo_agg_state_t {value bits (SUM/AVG: the sum in the SUM return type; AVG is NOT divided yet), non-null rows, rc} -- what a partial
 * Group hands to MergeGroup (pkg/sql/colexec/group/mergeGroup.go:132-247).
 * Asynchronous form: when the column, its nulls bitmap and the result (pdata, pnulls) are all DEVICE pointers (or NULL) the call only
 * enqueues work on the calling thread's stream and returns MO_RC_SUCCESS at once; errors detected on the device (SUM overflow) are
 * reported in state.rc.  Any host pointer among them, a column-cache hit included, makes the call synchronous. */
typedef struct mo_agg_state_t { uint64_t bits; int64_t count; int64_t rc; } mo_agg_state_t;
/* MergeGroup for these aggregates: args [0] result (8 / 16 / 24 bytes as above, + nulls word) ; [1] len partial states (24 bytes each),
 * folded in order with the reference's BatchMerge rules (sumavg2.go:205-248 incl. int64OfCheck / uint64OfCheck, minmax2.go:90-110).
 * Device partials and a device result (pdata and pnulls): asynchronous as above. */
#define MO_XCALL_AGG_MERGE(op, T) (0x1800 + ((op) << 8) + (T))
/* Parameter blocks and scalar arguments -- every mo_*_params_t, mo_plan_t, mo_search_filter_t, mo_go_params_t, the BETWEEN bounds, the
 * MULTI_AND / MULTI_OR operand count and ngroups -- may be host or device memory at every entry point.  A host block is copied and does not
 * count toward the asynchronous form.  A device block is read back once before the call enqueues work, so the call waits for the work
 * already on the calling thread's stream; apart from that the call completes exactly as it does with a host block.  Words a call writes
 * into its block (err_row, the k-means iteration count) hold their value when a synchronous call returns. */

/* --- new: fused TPC-H Q6 shape  SUM(a*b) WHERE d in [d_lo,d_hi) AND b BETWEEN b_lo AND b_hi AND c < c_hi
 * args: [0] result f64 (+ 1-word nulls bitmap, bit0 = no row qualified) ; [1] d int32/DATE col ; [2] b f64 col
 * (discount) ; [3] c f64 col (quantity) ; [4] a f64 col (extendedprice) ; [5] params: pdata -> mo_q6_params_t.
 * Optional second result word: if args[0].dataSz >= 16 the qualifying row count (int64) is written at pdata+8. */
/* ---- The Go elementwise engine's conventions (pkg/sql/plan/function/baseTemplate.go:457-728, arithmetic.go:222-762,
 * func_compare.go:285-1185, operator_between.go:138-199, logicalOperator.go:36-168) -- the LIVE per-batch path of the reference;
 * the mo.h symbols above keep the C kernels' conventions.  Differences: rows whose RESULT null bit is set on entry are skipped
 * (the caller pre-fills args[0].pnulls with NOT selectList, baseTemplate.go:473-486); on return it holds rnulls | n1 | n2 (plus
 * the rows a zero divisor nulled); a const operand is a 1-element vector (dataSz == sizeof(T)), a const NULL operand nulls every
 * row; the FIRST offending row in row order fails the call (MO_RC_OUT_OF_RANGE with "data out of range: data type int64, value
 * '(a + b)'" / MO_RC_DIVISION_BY_ZERO) and its index is stored in the parameter block; rows before it hold their results.
 *   ARITH(op, T)   op: 0 + 1 - 2 * 3 / (floats) 4 %     args: [0] result T[len] + pnulls (in/out)  [1] a  [2] b  [3] mo_go_params_t
 *   COMPARE(op, T) op: 0 == 1 != 2 > 3 >= 4 < 5 <=      args: [0] result bool[len] + pnulls (in/out)  [1] a  [2] b
 *   BETWEEN(T)                                           args: [0] result bool[len] + pnulls (in/out)  [1] column (+ pnulls)  [2] lo  [3] hi
 *                                                        null input -> result false AND null bit set
 *   MULTI_AND / MULTI_OR                                 args: [0] result bool[len] + pnulls (out)  [1] int32 operand count n (<= 16)
 *                                                              [2 .. 2 + n) bool operands (+ pnulls); const = 1 byte
 * T = types.T id (MO_T_*); DATE compares as int32, TIME / DATETIME / TIMESTAMP as int64.
 *   COMPARE(op, DECIMAL64 | DECIMAL128)  valueDecimalCompare (func_compare.go:426-667), csrc/decimal.cu.  Args as COMPARE plus [3] mo_dec_params_t
 *                  {scale1 of a, scale2 of b} (required; 0..18 for DECIMAL64, 0..38 for DECIMAL128, else MO_RC_INVALID_ARGUMENT).  The side with the
 *                  lower scale is scaled up by the difference (Decimal64.Scale / Decimal128.Scale), then the values compare signed.  The Go wrapper
 *                  drops Scale's error: a scale-up that overflows compares the value unscaled, and a Decimal64 scale-up between 2^63 and 2^64
 *                  wraps (unsigned Mul64, sign restored).  Never fails on data; all-device operands give an enqueue-only call (a const
 *                  operand's null word is read on the device).
 *   BETWEEN(DECIMAL64 | DECIMAL128)      CompareDecimal64 / 128 (operator_between.go:68-73): a raw signed compare, the bounds already at the
 *                  column's scale (8- / 16-byte bounds, host or device). */
typedef struct { int32_t div0_null; int32_t reserved; int64_t err_row; } mo_go_params_t;   /* err_row: out, -1 = no error */
#define MO_XCALL_GO_ARITH(op, T) (0x4000 + ((op) << 8) + (T))
#define MO_XCALL_GO_COMPARE(op, T) (0x4800 + ((op) << 8) + (T))
/* float32 columns declared with scale > 0 compare after rounding both sides to `scale` decimals (func_compare.go:207-216,725-734,
 * 852-861,979-988,1106-1115,1233-1242): same args as COMPARE(op, MO_T_FLOAT32), scale 1..22 */
#define MO_XCALL_GO_COMPARE_F32_SCALE(op, scale) (0x5200 + ((op) << 8) + (scale))
#define MO_XCALL_GO_BETWEEN(T) (0x5000 + (T))
#define MO_XCALL_GO_MULTI_AND 0x5100
#define MO_XCALL_GO_MULTI_OR 0x5101
/* ---- string predicates (csrc/strpred.cu), the GO conventions above.  Operands are what Vector.FillRawPtrLen gives: pdata = 24-byte cells
 * (dataSz = 24 * len; dataSz == 24 with len != 1 is a const operand), parea / areaSz = the area, pnulls = the nulls (a const operand: bit 0).
 *   COMPARE(op, T) for T = CHAR, VARCHAR, BINARY, VARBINARY, BLOB, TEXT, DATALINK (func_compare.go:224-226,353-360,744-748,871-875,1125-1129,
 *                  1252-1256): == / != are bytes.Equal, > >= < <= bytes.Compare -- unsigned bytes, a proper prefix first, zero bytes count, no
 *                  trimming or collation.  Args as COMPARE.  JSON and the vector types stay refused.
 *   GO_LIKE        likeFn (func_builtin_regexp.go:51-69).  args: [0] result bool[len] + pnulls (in/out) ; [1] the string ; [2] the pattern.
 *                  A const NULL pattern nulls every row.  A const pattern that optimizeRuleForLike (:91-280) takes is matched by its byte-level
 *                  rule: empty; `%`; `_` (one BYTE); one literal byte; exact / `_lit` / `%lit` / `lit_` / `lit%` / `%lit%` / `%lit_` / `_lit%` with
 *                  no `_` or `%` inside (escapes removed by RemoveEscapeChar, which keeps a trailing lone backslash; `\` as the next-to-last byte
 *                  makes the last byte a literal, so `\%` is a prefix match on a backslash); and `%a%b%...%` without `_` or `\%` (ordered
 *                  bytes.Index of the pieces, escapes kept as bytes).  Any other pattern, and every column pattern (len == 1: the pattern is a
 *                  column), is regularMatchForLikeOp (:618-672), ^(?s:...)$ over RUNES decoded by utf8.DecodeRune (an invalid, overlong or
 *                  surrogate sequence is (U+FFFD, 1)): `_` one rune, `%` any run of runes, `\x` the literal rune x, a trailing `\` a literal
 *                  backslash; an invalid pattern byte is a literal U+FFFD, which matches U+FFFD and any invalid subject byte.
 *                  NOT LIKE is Logic_VecNot of the result.
 * Both: values of any length.  Rows whose result null bit is set on entry are skipped; on return the bitmap holds rnulls | n1 | n2.  Cells of
 * NULL and skipped rows are never read.  A non-inline cell that points outside [0, areaSz), or any when there is no area, fails the call with
 * MO_RC_INVALID_ARGUMENT naming the operand and its lowest such row.  Device cells, areas, nulls and result: the call enqueues one kernel and
 * reads back one small status record (the bad-cell check), which synchronises the calling thread's stream once; a const pattern is read on
 * the host before that (a device one is copied back first, as a device parameter block is). */
#define MO_XCALL_GO_LIKE 0x5800
/* ---- list membership: x IN (v1, ..., vm) and x NOT IN (...), operator_in.go (overloads list_operator.go:541-808 and :1094-), the GO
 * conventions above.  Fixed-width T in csrc/goelem.cu, the varlena T in csrc/strpred.cu.
 *   IN(T) / NOT_IN(T)  args: [0] result bool[len] + pnulls (in/out) ; [1] the column (+ pnulls; a const is one element) ; [2] the list:
 *                      nvalues elements (+ pnulls; the varlena types: 24-byte cells + area) ; [3] mo_in_params_t (required, host or device).
 *   T = UINT8..64, INT8..64, FLOAT32 / 64, DECIMAL64 / 128, DATE, TIME, DATETIME, TIMESTAMP, BOOL, UUID, YEAR (int16), CHAR, VARCHAR, TEXT,
 *       BLOB, BINARY, VARBINARY.  Any other T is refused.
 *   The set is Go's map[T]bool or map[string]bool of the list (op.init): NULL elements are skipped, so a const NULL or all-NULL list is the
 *   empty set.  Equality is Go map equality: the raw value's bits (+0.0 and -0.0 are one key; a NaN is never found, so a NaN row is IN-false
 *   and NOT-IN-true; decimals and UUIDs compare raw, unscaled -- the planner casts the list to the column's type), and bytes for the strings
 *   (no trimming, no collation).  A NULL row is NULL; every other row is `found` (IN) or `!found` (NOT IN) with a clear null bit, so a NULL in
 *   the list never nulls a row: 2 NOT IN (1, NULL) is true.  A const NULL column nulls every row.  Rows whose result null bit is set on entry
 *   are skipped; on return the bitmap holds rnulls | the column's nulls (a const NULL column: every row), the bits past len cleared.
 *   The set is built per call into a hash table in the calling thread's scratch: 8-byte-or-narrower values keyed on their bits, 16-byte
 *   values (DECIMAL128, UUID) and strings as a hash tag and a list index.  Launches: nvalues == 0, or a host list whose nvalues elements
 *   are all NULL -> the probe only (1 kernel); else the build and the probe (2 kernels; a device list's NULL elements are skipped by the
 *   build, whose launch does not depend on them).  Fixed-width T with device operands and a host block only enqueue work; the varlena T read back one
 *   status record, as GO_LIKE does, and a non-inline cell outside its area, in the column or in a non-NULL list element, fails the call
 *   with MO_RC_INVALID_ARGUMENT naming the operand and its lowest such row.  A negative nvalues or one above 2^31 - 1, a list shorter than
 *   nvalues elements and a missing block are refused with MO_RC_INVALID_ARGUMENT. */
typedef struct mo_in_params_t { int64_t nvalues; } mo_in_params_t;
#define MO_XCALL_GO_IN(T) (0x5900 + (T))
#define MO_XCALL_GO_NOT_IN(T) (0x5A00 + (T))
/* ---- conditional values: CASE WHEN c1 THEN v1 ... [ELSE z] END, IF(c, a, b) and COALESCE(a, b, ...), csrc/caseexpr.cu.  caseFn / generalCaseFn /
 * strCaseFn (operatorSet.go:144-316), iffFn (:389-) and CoalesceGeneral / CoalesceStr (func_binary.go:938-993).
 *   GO_CASE(T)      args: [0] the result (T[len] + pnulls in/out; the string T: 24-byte cells + an area whose areaSz is its capacity) ; [1]
 *                   mo_case_params_t (required, host or device) ; [2 + 2j] condition j (bool) ; [3 + 2j] value j (T) ; [2 + 2n] the ELSE value
 *                   when has_else.  n = the WHEN count, 1..1024 ; has_else 0 or 1.  A row takes value j of the first j whose condition is
 *                   non-NULL and true (NULL when that value is NULL); with no such j it takes ELSE, or NULL without one.  IF(c, a, b) is
 *                   GO_CASE with n = 1 and an ELSE: a NULL or false condition takes b.
 *   GO_COALESCE(T)  args: [0] the result ; [1] mo_case_params_t with n = the operand count (1..1024) and has_else 0 ; [2 .. 2 + n) the
 *                   operands (T).  A row takes its first non-NULL operand, or NULL.
 *   T = BOOL, BIT, INT8..64, UINT8..64, FLOAT32 / 64, DATE, TIME, DATETIME, TIMESTAMP, DECIMAL64, DECIMAL128, UUID, ENUM (fixed width: the
 *       value's bytes are selected, never interpreted, so -0.0 and NaN payloads pass unchanged) and CHAR, VARCHAR, BLOB, TEXT, DATALINK (strings).
 *       Any other T is refused (caseFn panics on BINARY / VARBINARY).
 *   Operands follow the GO conventions above with one difference: merge_nulls does NOT apply.  A const operand is one element when len > 1;
 *   a const NULL condition never matches, and a const NULL value gives NULL only on the rows that choose it.  Rows whose result null bit is
 *   set on entry are skipped and their value bytes / cells left as they were; every other row the call makes NULL gets zero value bytes
 *   (a string: the empty inline cell), and the bits past len in the last result word are cleared.  A condition or value is read only on
 *   the rows that reach it, so the rows a short-circuit left unset (GO_CASE_SELECT below) are never read: a condition on the rows no
 *   earlier WHEN took, a value on the rows that choose it.
 *   Strings: each chosen value is copied, as AppendBytes does: up to 23 bytes inline in its cell (zero-padded), longer ones into the result
 *   area in row order with no padding, the cell {0xffffffff, offset, length, 0...}.  area_len (out) is set to the bytes the result needs.
 *   More than areaSz, or more than 2^32 - 1: MO_RC_OUT_OF_RANGE, area_len still written, cells, area and bitmap unchanged, so the call may be
 *   repeated with an area of area_len bytes.  A chosen non-inline cell outside its operand's area fails with MO_RC_INVALID_ARGUMENT naming
 *   the operand (its argument index) and the lowest row that chose it (a const operand too); cells that are not chosen are never read.
 *   Launches: fixed width 1 (enqueue-only with device operands and a host block) ; strings 3 (pick, scan, write; the write is not launched
 *   when the call fails), with one read-back of a status record (the bad cell and the area total) between the scan and the write.
 *   Refused with MO_RC_INVALID_ARGUMENT: another T, n outside 1..1024, has_else not 0 / 1 or set for COALESCE, a short operand or result, a
 *   result without a null bitmap, a missing block.
 *   GO_CASE_SELECT  the select lists of EvalCase / EvalIff (evalExpression.go:501-573) as null-prefill words (a set bit: skip the row).  args:
 *                   [0] uint64 words out: THEN j's prefill ; [1] uint64 words in / out: the remaining rows' complement (rows taken by an earlier
 *                   WHEN, or not selected) ; [2] condition j (bool + pnulls; a const is one element; rows set in [1] are not read).  With
 *                   took = ~[1] & cond & ~cond_nulls:  [0] = ~took (bits past len set) ; [1] |= took.  One kernel, enqueue-only.  A caller
 *                   starts with [1] = NOT selectList and, per WHEN, evaluates the condition under a copy of [1] as its prefill, calls
 *                   GO_CASE_SELECT and evaluates THEN j under [0]; ELSE is evaluated under the final [1].  CASE never raises an error from a
 *                   branch a row does not reach (CASE WHEN d <> 0 THEN x / d ELSE 0 END). */
typedef struct mo_case_params_t { int32_t n; int32_t has_else; int64_t area_len; } mo_case_params_t;
#define MO_CASE_MAX_WHENS 1024
#define MO_XCALL_GO_CASE(T) (0x5B00 + (T))
#define MO_XCALL_GO_COALESCE(T) (0x5C00 + (T))
#define MO_XCALL_GO_CASE_SELECT 0x5D00

/* ---- the standalone column operators of the colexec pipeline (csrc/colops.cu).  Host or device pointers; when every data pointer and
 * nulls bitmap of every vector is a device pointer (or NULL) FILTER_SELS and SHUFFLE only enqueue work (asynchronous form, as
 * MO_XCALL_AGG).
 *
 * FILTER_SELS  Filter.Call inner loop (filter.go:116-152): rows with (!null && true), ascending.
 *              args: [0] sels int64[] (a host buffer only has to hold the selected rows) ; [1] count int64[1] ; [2] bool vector (+pnulls).  len = rows
 * SHUFFLE(sz)  Vector.Shrink / Union / shuffle.FixedLengthShuffle (vector.go:1014,2583 ; shuffle.go:21-26) with nulls.Filter
 *              (nulls.go:237-281) fused: dst[i] = src[sels[i]], dst null bit i = src null bit sels[i].  sz = element bytes: 1, 2, 4, 8, 16, 24 (varlena cell).
 *              A negative sel gathers a NULL row: zero value bytes (a 24-byte cell: the empty inline value) and the null bit set -- the side of an
 *              outer join's result row that has no match.  Without a dst bitmap the zero bytes are still written.
 *              args: [0] dst (+pnulls out) ; [1] src (+pnulls, nullCnt = its length in bits) ; [2] sels int64[len].  len = selected rows
 * PACK_KEYS    intHashMapIterator.encodeHashKeys / fillKeys (inthashmap.go:92-183): up to 8 key bytes per row from fixed-width columns, in
 *              has_null mode a marker byte (0 / 1) precedes every column's value bytes and a NULL contributes the marker only.
 *              args: [0] keys uint64[len] (+pnulls out, has_null = 0: rows with a NULL key join no group) ; [1] params {int32 ncols, int32 has_null}
 *              ; [2 .. 2+ncols) key columns (+pnulls; a const vector holds one element)
 * GROUP_IDS    IntHashMap insert as driven by Group.buildOneBatch (exec2.go:325-362): 1-based group ids in FIRST-SEEN order; the table persists across
 *              calls through (ngroups, table_keys).  The hash function is not observable (random seeds, hashtable/hash.go:41-47), the ids are.
 *              args: [0] groups uint64[len] ; [1] int64 ngroups (in/out) ; [2] table_keys uint64[capacity] (in: keys of groups 1..ngroups ; out: + new groups)
 *              ; [3] keys uint64[len] (+pnulls: such rows get id 0 = GroupNotMatched)
 * GROUP_AGG(op, T)  sumAvgExec / countColumnExec / minMaxExecFixed .BatchFill (sumavg2.go:133-199, count2.go:120-146, minmax2.go:49-80) into a
 *              caller-owned state that persists across batches: SUM into int64 / uint64 / float64 (overflow -> MO_RC_OUT_OF_RANGE exactly when
 *              the serial loop would fail), AVG = SUM + counts, COUNT into int64, MIN / MAX in 8-byte slots (value in the low bytes) with the
 *              first-value-initialises / strict-compare rule incl. NaN: the bits of the first row that reaches the extreme (-0.0 and
 *              0.0 tie: the earlier row's zero, a state's zero before a later batch's).  A group is NULL until its first value (state pnulls, in/out).
 *              args: [0] state 8 bytes per group (+pnulls) ; [1] counts int64 per group (AVG: required) ; [2] groups uint64[len] ; [3] column (+pnulls)
 * float64 group sums are accumulated with atomics: the association order is not fixed, results agree with the serial loop to ~1e-13 relative. */
#define MO_XCALL_FILTER_SELS 0x6000
#define MO_XCALL_PACK_KEYS 0x6001
#define MO_XCALL_GROUP_IDS 0x6002
#define MO_XCALL_SHUFFLE(szof) (0x6100 + (szof))
/* ---- Elkan k-means, dense variant (csrc/kmeans.cu): ElkanClusterer.Cluster from given initial centroids
 * (pkg/vectorindex/ivfflat/kmeans/elkans/clusterer.go:330-392; distance = metric.L2Distance for every metric, distance_func.go:452-476).
 * Centroids bit for bit, assignments and iteration count as the reference computes them (serial row-order sums, Go-order distances).
 * InitCentroids (initializer.go: draws from Go's PCG) stays with the caller.  args: [0] centroids T[k * dim] (in: initial, out: final) ;
 * [1] assignments int64[n] (out) ; [2] int64 iterations (out) ; [3] mo_kmeans_params_t ; [4] vectors T[n * dim] ;
 * [5] rnd float32[] (optional): the rnd.Float32() stream an EMPTY cluster re-seeds its centroid from (clusterer.go:700-707), consumed in
 * cluster order, dim values per empty cluster; running out of it fails the call with MO_RC_INVALID_ARGUMENT. */
/* ---- LZ4 block decompression of column blocks (csrc/lz4.cu): compress.Decompress = lz4.UncompressBlock (pkg/compress/compress.go:37-47), one
 * warp per block.  args: [0] dst bytes ; [1] src bytes ; [2] int64[4 * len] descriptors {src_off, src_len, dst_off, dst_len} per block (dst_len = the
 * decoded size the object metadata records; a block that decodes to anything else, or is malformed, fails the call with MO_RC_INVALID_ARGUMENT and
 * the LOWEST such block number in the error text).  len = number of blocks.  Like the Go decoder, it does not enforce the format's end-of-block
 * rules (last 5 bytes literals, no match in the last 12): a block that ends in a match decodes by the sequence rules, where liblz4 rejects it. */
#define MO_XCALL_LZ4_DECODE 0x6030
/* ---- a decompressed column block -> a resident vector (csrc/vecdecode.cu): Vector.UnmarshalBinary (pkg/container/vector/vector.go:766-819) on the device.
 * args: [0] mo_vector_view_t (out) ; [1] data bytes (out: capacity >= dataLen, aligned) ; [2] area bytes (out) ; [3] nulls uint64 words (out:
 * (length + 63) / 64 words; pdata NULL when not wanted) ; [4] the marshalled bytes (dataSz = their length; when they are device memory the buffer
 * must be readable 8 bytes past that length).  Malformed bytes or too small output buffers -> MO_RC_INVALID_ARGUMENT. */
typedef struct mo_vector_view_t {
    int32_t vclass;        /* 0 FLAT, 1 CONSTANT */
    int32_t oid;           /* types.T */
    int32_t size, width, scale;
    uint32_t length;       /* rows */
    uint64_t data_len, area_len;
    int64_t null_count;    /* bitmap.count as marshalled */
    uint64_t nulls_words;
    int32_t sorted, bad;
} mo_vector_view_t;
#define MO_XCALL_VECTOR_UNMARSHAL 0x6031
typedef struct mo_kmeans_params_t { int64_t n, dim, k, max_iter; } mo_kmeans_params_t;
#define MO_XCALL_KMEANS_ELKAN_F32 0x6020
#define MO_XCALL_KMEANS_ELKAN_F64 0x6021
/* ---- hash join, equality conditions over <= 8-byte packed keys (csrc/join.cu).  The build side inserts its keys with GROUP_IDS (IntHashMap insert):
 *   JOIN_SELS   GroupSels.Insert + Finalize (pkg/vm/message/joinMapMsg.go:72-125) as driven by HashmapBuilder.BuildHashmap (hashbuild/hashmap.go:395-412):
 *               the build rows of every group, ascending.  args: [0] offsets int32[ngroups + 2] (out: [k] = start of 0-based group k, [ngroups] =
 *               [ngroups + 1] = count) ; [1] vals int32[len] (out) ; [2] int64 count (out: rows that have a group) ; [3] groups uint64[len] (the ids
 *               GROUP_IDS returned for the build rows; 0 = the row has a NULL key and joins nothing).  len = build rows (< 2^31).
 *               (The reference keeps no sels when every row got its own group -- HashOnUnique, joinMapMsg.go:83-89,203-205: pass pdata NULL below.)
 *   JOIN_FIND   intHashMapIterator.Find (pkg/common/hashmap/inthashmap.go): vals[i] = 1-based group id of probe key i, 0 = absent or NULL key.
 *               args: [0] vals uint64[len] ; [1] table_keys uint64[ngroups] (GROUP_IDS's key table: key of group g at [g - 1]) ; [2] keys uint64[len] (+pnulls)
 *   JOIN_PROBE  the emission loop of hashjoin container.probe (pkg/sql/colexec/hashjoin/join.go:383-628) without a non-equality condition: result rows
 *               as (probe row, build row) pairs in the reference's order -- probe rows ascending, per probe row its group's sels ascending.
 *               join_type INNER: matches only; LEFT: + (row, -1) for a probe row without a match; SEMI: (row, -1) once per matching probe row;
 *               ANTI: (row, -1) per probe row WITHOUT a match.  args: [0] probe_rows int64[cap] ; [1] build_rows int64[cap] ; [2] int64 count (out; when
 *               it exceeds cap the call fails with MO_RC_OUT_OF_RANGE and the count is still written) ; [3] mo_join_params_t ; [4] table_keys ;
 *               [5] sels offsets int32[ngroups + 2] (pdata NULL: unique map, build row = id - 1) ; [6] sels vals int32[] ; [7] probe keys uint64[len] (+pnulls)
 * The device hash table is rebuilt from table_keys per call unless MoB200_JoinMapPrepare(table_keys, ngroups) cached it (keyed by that pointer). */
#define MO_JOIN_INNER 0
#define MO_JOIN_LEFT 1
#define MO_JOIN_SEMI 2
#define MO_JOIN_ANTI 3
/* ---- right-flavoured and single joins (hashjoin types.go:317-381: JoinType + IsRightJoin; FULL OUTER always runs right-flavoured).  JOIN_PROBE
 * and JOIN_PROBE_GIDS take these types too, with the same capacity protocol, count read-back and bad-group-id error:
 *   SINGLE        LEFT SINGLE: the LEFT pairs; a probe row whose group has more than one build row fails the call (join.go:504-507).
 *   RIGHT         the INNER pairs, and every emitted build row is marked in the matched bitmap.
 *   FULL          the LEFT pairs, marked as RIGHT.
 *   RIGHT_SEMI    no pairs (count 0): only marks the matched build rows.
 *   RIGHT_ANTI    no pairs: marks as RIGHT_SEMI.
 *   RIGHT_SINGLE  the INNER pairs, marked as RIGHT; a build row matched a second time, in this call or an earlier one, fails the call.
 * Types 5..9 take args[8]: the matched bitmap (rightRowsMatched, join.go:461-467,539-547), uint64[(nbuild + 63) / 64], LSB-first, one bit per build
 * row (NULL-key rows included; they are never matched), in/out.  The caller zeroes it once per join and passes the same words to every probe
 * batch.  Missing, or too short for the rows the map names: MO_RC_INVALID_ARGUMENT.  Types that emit pairs mark only when the result fits the
 * output, so a call that fails with MO_RC_OUT_OF_RANGE leaves the bitmap untouched and its repeat is safe.  A SINGLE failure is
 * MO_RC_INTERNAL_ERROR "scalar subquery returns more than 1 row" naming the lowest offending probe row (SINGLE) or the lowest build row matched
 * twice in this call (RIGHT_SINGLE; which rows fail does not depend on the probe order).  Neither adds a synchronise: both come back in the
 * record the probe already reads.
 *   JOIN_MATCHED_MERGE  syncBitmap across workers or shards (join.go:650-676): out = the OR of n bitmaps.  args: [0] out uint64[(len + 63) / 64]
 *                 (may be one of the inputs) ; [1] int32 n (1..MO_JOIN_MERGE_MAX) ; [2] mo_join_params_t (a type 5..9) ; [3 .. 3 + n) input
 *                 bitmaps.  len = build rows.  RIGHT_SINGLE: a bit set in two inputs fails the call as above, naming the lowest such row, and
 *                 the call reads back that one word; the other types only enqueue work when every bitmap is device memory.
 *   JOIN_BUILD_ROWS     finalize (join.go:682-727): the build rows whose bit is CLEAR (RIGHT, FULL, RIGHT_ANTI, RIGHT_SINGLE) or SET (RIGHT_SEMI),
 *                 ascending -- each is one result row whose probe-side columns are NULL.  Output contract of FILTER_SELS.  args: [0] sels
 *                 int64[] (a host buffer only has to hold the rows found) ; [1] count int64[1] ; [2] matched bitmap ; [3] mo_join_params_t.
 *                 len = build rows.
 * The probe-side columns of those rows, and the build-side columns of a LEFT / FULL / SINGLE pair (row, -1), come from SHUFFLE with sel -1. */
#define MO_JOIN_SINGLE 4
#define MO_JOIN_RIGHT 5
#define MO_JOIN_FULL 6
#define MO_JOIN_RIGHT_SEMI 7
#define MO_JOIN_RIGHT_ANTI 8
#define MO_JOIN_RIGHT_SINGLE 9
#define MO_JOIN_MERGE_MAX 64
#define MO_XCALL_JOIN_MATCHED_MERGE 0x6015
#define MO_XCALL_JOIN_BUILD_ROWS 0x6016
/* ---- joins with a non-equality condition (NonEqCond, hashjoin join.go:468-498,570-611).  Three steps per probe batch:
 *   1. JOIN_PROBE or JOIN_PROBE_GIDS with MO_JOIN_INNER: the candidate pairs, every (probe row, build row) whose keys are equal, in order.
 *   2. SHUFFLE of the probe columns by the candidate probe rows and of the build columns by the candidate build rows, then the condition over
 *      them with the expression entry points (GO_COMPARE, GO_ARITH, GO_MULTI_AND / OR, DEC_ARITH, ...): one bool (+ nulls) per candidate pair.
 *   3. JOIN_COND: the join's result from the pairs and the condition.  Let P(i) = probe row i's candidates whose condition is true and not NULL,
 *      in candidate order (empty for a row without candidates).  INNER: P(i) ; LEFT: P(i), or (i, -1) when P(i) is empty ; SEMI: (i, -1) once
 *      when P(i) is non-empty ; ANTI: (i, -1) when P(i) is empty ; SINGLE: as LEFT, and |P(i)| > 1 fails ; RIGHT: P(i), marking its build rows ;
 *      FULL: as LEFT, marking as RIGHT ; RIGHT_SEMI / RIGHT_ANTI: no pairs, marking as RIGHT ; RIGHT_SINGLE: as RIGHT, a build row marked a second
 *      time (this call or an earlier one) fails.  Output order: probe rows ascending, each row's pairs in candidate order.  With a condition that
 *      is always true the result equals JOIN_PROBE's for that type.  Capacity protocol, matched-bitmap rules and SINGLE errors are JOIN_PROBE's.
 *      args: [0] probe_rows int64[cap] ; [1] build_rows int64[cap] ; [2] int64 count (out) ; [3] mo_join_params_t (type 0..9) ; [4] candidate
 *      probe rows int64[npairs] (npairs = dataSz / 8) ; [5] candidate build rows int64[npairs] ; [6] the condition bool[npairs] (+pnulls) ;
 *      [7] the matched bitmap (types 5..9; JOIN_PROBE's args[8]).  len = probe rows of the batch.  A candidate probe row outside [0, len) or below
 *      the one before it, a negative build row, a build row past the bitmap or a short buffer: MO_RC_INVALID_ARGUMENT (naming the lowest bad
 *      candidate position, or the build row).  One read-back, as JOIN_PROBE.  The reference evaluates the condition pair by pair and stops a semi
 *      row at its first passing pair; here the caller evaluates every candidate, so an expression that fails on a later candidate fails here only. */
#define MO_XCALL_JOIN_COND 0x6017
typedef struct mo_join_params_t { int32_t join_type; int32_t reserved; } mo_join_params_t;
#define MO_XCALL_JOIN_SELS 0x6010
#define MO_XCALL_JOIN_FIND 0x6011
#define MO_XCALL_JOIN_PROBE 0x6012
/* ---- byte-string keys: StrHashMap (pkg/common/hashmap/strhashmap.go), for keys wider than 8 bytes and for varlena keys (csrc/colops.cu,
 * csrc/join.cu).  A key is a byte string; two rows are in one group exactly when their key bytes are equal (the reference compares 192-bit
 * hashes of them), so -0.0 and +0.0 are two groups and NaN payloads stay distinct.
 *   PACK_STR_KEYS    strHashmapIterator.encodeHashKeys (strhashmap.go:92-385): per row the concatenation over the key columns of -- fixed width:
 *                    [0x00 marker when has_null] + the value's storage bytes ; varlena (CHAR, VARCHAR, BINARY, VARBINARY, BLOB, TEXT, DATALINK):
 *                    [0x00 marker when has_null] + uint16 little-endian length + the bytes ; NULL: 0x01 alone when has_null, else the row joins no
 *                    group (empty key, bit set in args[1].pnulls).  The reference pads keys shorter than 16 bytes with zeros; the codes are
 *                    self-delimiting, so the padding never makes two keys equal and is left out.  The ROLLUP marker 0x02 is not built.
 *                    args: [0] key bytes u8[cap] (out) ; [1] offsets uint64[len + 1] (out: row i's key is bytes[off[i], off[i + 1]); +pnulls out,
 *                    has_null = 0 only: rows that join no group) ; [2] mo_strkey_params_t ; [3 .. 3+ncols) key columns of col_type[k]: fixed
 *                    width (the key types of ORDER_SELS, by storage size) or varlena cells + area as ORDER_SELS takes them (+pnulls; one element =
 *                    const).  cap too small: MO_RC_OUT_OF_RANGE and off[len] = the bytes needed.  A cell outside its area or a value longer than
 *                    MO_ORDER_MAX_VARLENA bytes: MO_RC_INVALID_ARGUMENT naming the column and its lowest such row.  Reads back one record (the byte
 *                    total, the lowest bad cell per column): one synchronise.
 *   STR_GROUP_IDS    StrHashMap insert as Group.buildOneBatch drives it (exec2.go:325-362): GROUP_IDS over byte-string keys, 1-based ids in
 *                    first-seen order, persisting across calls through (ngroups, table bytes, table offsets), which the caller owns.
 *                    args: [0] groups uint64[len] ; [1] int64 ngroups (in/out) ; [2] table bytes u8[cap_bytes] ; [3] table offsets
 *                    uint64[cap_groups + 1]: group g is bytes[off[g - 1], off[g]) (off[0] = 0 for an empty table; in: groups 1..ngroups, out: + the
 *                    new groups) ; [4] key bytes ; [5] key offsets uint64[len + 1] (PACK_STR_KEYS's; +pnulls: those rows get id 0) ; [6] first rows
 *                    int64[len] (out, pdata NULL when not wanted): the batch row that created each new group, in id order.  More groups or bytes
 *                    than the table holds: MO_RC_INVALID_ARGUMENT stating both capacities needed, with ngroups and the table untouched -- grow the
 *                    table and repeat the call.  len + ngroups < 2^31.  Reads back its overflow record (a device ngroups is read first, as GROUP_IDS does).
 *   STR_JOIN_FIND    strHashmapIterator.Find: vals[i] = 1-based id of probe key i in a table STR_GROUP_IDS built, 0 = absent or skipped.
 *                    args: [0] vals uint64[len] ; [1] int64 ngroups ; [2] table bytes ; [3] table offsets ; [4] probe key bytes ; [5] probe key
 *                    offsets (+pnulls).  The device table is rebuilt per call (O(build groups)) unless MoB200_StrJoinMapPrepare cached it, keyed by
 *                    the table offsets pointer.  Device pointers: enqueue only.
 *   JOIN_PROBE_GIDS  JOIN_PROBE with each probe row's group id given (JOIN_FIND's or STR_JOIN_FIND's vals) instead of its key: the same pairs, in
 *                    the same order.  args [0..3], [5], [6] as JOIN_PROBE ; [4] int64 ngroups ; [7] vals uint64[len] (an id above ngroups:
 *                    MO_RC_INVALID_ARGUMENT). */
#define MO_XCALL_PACK_STR_KEYS 0x6003
#define MO_XCALL_STR_GROUP_IDS 0x6004
#define MO_XCALL_STR_JOIN_FIND 0x6013
#define MO_XCALL_JOIN_PROBE_GIDS 0x6014
#define MO_STRKEY_MAX_COLS 8
typedef struct mo_strkey_params_t { int32_t ncols; int32_t has_null; int32_t col_type[MO_STRKEY_MAX_COLS]; } mo_strkey_params_t;
#define MO_XCALL_GROUP_AGG(op, T) (0x6400 + ((op) << 8) + (T))
/* ---- ORDER BY / ORDER BY ... LIMIT (csrc/order.cu): the sels of the Order operator (order.go:103) or the first `limit` of them for Top
 * (top.go:445); payload columns are then reordered with MO_XCALL_SHUFFLE, as Batch.Shuffle(sels) does.
 *   args: [0] sels int64[min(limit, len)] (out: indices into this call's rows) ; [1] mo_order_params_t ; [2 .. 2+nkeys) key columns of
 *         key[k].col_type (+pnulls; a 1-element vector is a const key) ; [2+nkeys] int64 row ids [len] when has_row_ids.  len = rows (< 2^32).
 *   limit < 0 or >= len: the whole order; otherwise the first `limit` rows.
 *   Keys compare left to right as compare.New(type, desc, nullsLast) (pkg/compare/compare.go:24-115): flags = the OrderBySpec flag word
 *   (MO_ORDER_DESC, MO_ORDER_NULLS_FIRST, MO_ORDER_NULLS_LAST; neither NULLS flag: nullsLast = desc); two NULLs are equal; -0.0 == +0.0; NaN is
 *   above every number and equal to every NaN.  Ties break by ascending row id (row_ids[i], or the row index; then the row index): a total,
 *   stable order.  Against the reference (unstable pdqsort in Order, a heap in Top) the output key tuples are identical, and the rows are
 *   wherever all key tuples are distinct.  Key types: bool, int8-64, uint8-64, float32/64, DATE, TIME, DATETIME, TIMESTAMP, DECIMAL64,
 *   DECIMAL128, BIT (uint64), YEAR (int16), ENUM (uint16), UUID (16 bytes compared byte by byte, types.CompareUuid), and the varlena types
 *   CHAR, VARCHAR, BINARY, VARBINARY, BLOB, TEXT, DATALINK.
 *   Varlena keys: the argument is what Vector.FillRawPtrLen gives -- pdata = 24-byte cells (dataSz = 24 * len; dataSz == 24 with len != 1 is
 *   a const key), parea / areaSz = the area.  Values compare as Go's string `<` (bytes.Compare; sort.go varlenaLess, compare/strcompare.go):
 *   unsigned bytes, a proper prefix sorts first, the empty value below every other.  Cells of NULL rows are never read.  A non-inline cell
 *   that points outside [0, areaSz), or any non-inline cell when there is no area, fails the call with MO_RC_INVALID_ARGUMENT; the error
 *   names the key and the lowest such row.  So does a value longer than MO_ORDER_MAX_VARLENA bytes.
 *   MergeOrder / MergeTop: each shard's keys gathered with SHUFFLE, its row ids base + sels, all shards in one call with row ids.  A varlena
 *   key of a merge is one cells vector with ONE area: the shards' cells concatenated, the offsets of their non-inline cells rebased into the
 *   concatenation of their areas (what Vector.UnionBatch produces).  Varlena payload columns are reordered with SHUFFLE(24); its output cells
 *   still point into the source area, so that area must outlive them.
 *   Another type, nkeys outside 1..MO_ORDER_MAX_KEYS, short buffers or len >= 2^32: MO_RC_INVALID_ARGUMENT.  Device sels, key columns, nulls,
 *   areas and row ids: asynchronous form (enqueue only) -- except that a call with varlena keys first reads back one small record (the
 *   longest value of every varlena key and its lowest bad cell), which synchronises the calling thread's stream once.  Calls with only
 *   fixed-width keys never synchronise. */
#define MO_XCALL_ORDER_SELS 0x6040
#define MO_ORDER_MAX_KEYS 8
#define MO_ORDER_MAX_VARLENA 65535   /* longest varlena key value in bytes (MatrixOne's VARCHAR limit) */
#define MO_ORDER_DESC 2          /* pkg/pb/plan/plan.pb.go:419-424 */
#define MO_ORDER_NULLS_FIRST 4
#define MO_ORDER_NULLS_LAST 8
typedef struct mo_order_key_t { int32_t col_type; int32_t flags; } mo_order_key_t;
typedef struct mo_order_params_t {
    int32_t nkeys;
    int32_t has_row_ids;
    int64_t limit;
    mo_order_key_t key[MO_ORDER_MAX_KEYS];
} mo_order_params_t;

/* ---- Decimal64 / Decimal128 (csrc/decimal.cu): the reference's native TPC-H column type is DECIMAL(15,2).  Decimal64 = int64 unscaled value,
 * Decimal128 = 16 bytes two's complement {B0_63, B64_127}; scales travel in the parameter block.  Conventions of the Go engine (as GO_ARITH).
 *   DEC_ARITH(op, width)  op 0 + 1 - 2 * ; width 64 / 128 = operand type.  d64Add/d64Sub/d64Mul/d128Add/d128Sub/d128Mul,
 *                         pkg/sql/plan/function/arith_decimal_fast.go:111-733,3618-4095.  + - : the lower-scale operand is scaled up, result
 *                         scale = max(scale1, scale2), result type = operand type; * : result Decimal128 with scale
 *                         min(scale1 + scale2, max(12, scale1, scale2)), scaled down with round-half-up when that is smaller than scale1 + scale2.
 *                         The first row that overflows fails the call with MO_RC_INVALID_ARGUMENT (moerr ErrInvalidInput) and err_row is set.
 *                         args: [0] result (+pnulls in/out) ; [1] a ; [2] b (const = one element) ; [3] mo_dec_params_t
 *   DEC_SUM(width)        SUM / AVG accumulation of a decimal column into Decimal128 sums + int64 counts per group (count 0 = NULL; AVG divides at
 *                         Flush), sumDecimal64FastExec / sumDecimal128FastExec.batchFill, pkg/sql/colexec/aggexec/sum_decimal_fast.go -- exact and
 *                         order independent.  args: [0] sums Decimal128 per group (in/out) ; [1] counts int64 per group (in/out) ;
 *                         [2] groups uint64[len] (1-based, 0 = skip) or pdata NULL for one group ; [3] the column (+pnulls)
 *   DEC_ARITH(3, width)   / : d64Div / d128Div (arith_decimal_fast.go:734-1055, 4096-4320), equal to Decimal128.Div (decimal.go:1403-1446).
 *                         Result Decimal128 for both widths, scale = min(12, scale1 + 6) raised to at least scale1; the dividend is scaled by
 *                         10^(scale - scale1 + scale2) and divided with round half up (Div128; a divisor of 2^64 or more takes Div128's estimate,
 *                         whose signed Less rounds an odd estimate down once the scaled dividend reaches 2^126; past 127 bits the Decimal256
 *                         Div256 fallback).  Params mo_dec_div_params_t (a 16-byte mo_dec_params_t means div0_error = 0).  A zero divisor makes
 *                         the row NULL, or with div0_error fails the call with MO_RC_DIVISION_BY_ZERO "division by zero"; a quotient past
 *                         127 bits fails with MO_RC_INVALID_ARGUMENT "Decimal128 Div overflow".  The first failing row in row order, of either
 *                         kind, wins and goes to err_row; rows before it hold their results.  A const zero divisor fails at row 0 (or nulls every
 *                         row) whatever the row nulls, as the Go loop checks it before any row.
 *   DEC_AVG(width)        AVG's Flush over DEC_SUM's state: decAvg (aggexec/sumavg2.go:545-559) = Decimal128.Div(sum, count) with its error
 *                         dropped (the value Div keeps is written).  Result scale AvgReturnType: max(12, scale) capped at scale + 6.  args: [0] result
 *                         Decimal128 per group + pnulls (out: count 0 = NULL, the value is then the sum) ; [1] sums ; [2] counts ; [3] mo_dec_params_t
 *                         with scale1 = the argument's scale (0..18 / 0..38; the rest is not read).  len = the group count.  Never fails on data;
 *                         all-device arguments give an enqueue-only call. */
typedef struct mo_dec_params_t { int32_t scale1, scale2; int64_t err_row; } mo_dec_params_t;
typedef struct mo_dec_div_params_t { int32_t scale1, scale2; int64_t err_row; int32_t div0_error, reserved; } mo_dec_div_params_t;
#define MO_XCALL_DEC_ARITH(op, width) (0x7000 + ((op) << 8) + (width))
#define MO_XCALL_DEC_SUM(width) (0x7400 + (width))
#define MO_XCALL_DEC_AVG(width) (0x7500 + (width))

/* ---- the generic fused operator: scan -> filter -> project -> (hash) group -> aggregate in ONE pass over the columns (csrc/plan.cu).
 * What the colexec pipeline runs per block as table_scan -> filter -> projection -> group (filter.go:87-153, evalExpression.go:575-640,
 * group/exec2.go:296-367, aggexec/*), described by a mo_plan_t:
 *   columns      args[2 .. 2+ncols): fixed-width columns of col_type[c] (MO_T_*), each with an optional nulls bitmap
 *   predicates   conjunction of  col OP lo  (OP: 0 == 1 != 2 > 3 >= 4 < 5 <=)  or  col BETWEEN lo AND hi (op 6, inclusive); a NULL operand
 *                rejects the row.  The column value is compared with the float64 constant exactly (integer columns of any magnitude, UINT64
 *                unsigned), as the reference does once the constant is cast to the column type; a NaN constant: only != holds (IEEE)
 *   instructions SSA program: value slot ncols + i = COL(a) | CONST(imm) | slot a (+ - * /) slot b; slots 0..ncols-1 are the columns.  float64
 *                arithmetic, one rounding per instruction (the reference evaluates one node at a time); integer columns are converted (exact
 *                below 2^53; MIN / MAX of an integer column above 2^53 is of the rounded value); NULL in -> NULL out; x / 0 and x / -0.0 -> NULL
 *   keys         nkeys columns packed into <= 8 bytes exactly like fillKeys (inthashmap.go:92-183; has_null_keys: marker byte per column, a NULL
 *                key writes the marker 1 only; without has_null_keys a row with a NULL key joins no group, inthashmap.go:171-180)
 *   aggregates   kind MO_AGG_SUM / COUNT / MIN / MAX / AVG over value slot `value`; value = -1 with MO_AGG_COUNT is COUNT(*)
 * Result: mo_plan_result_header_t followed by ngroups records {mo_plan_group_t, naggs x mo_plan_agg_value_t}, groups in first-seen row order
 * (the reference's group-id order) when header.sorted (up to 8192 groups; beyond that in table order, first_row is there to sort by).  An
 * aggregate with count 0 is NULL.  No group-by (nkeys = 0): one group, present only if a row qualified.  header.overflow = more groups than the
 * result buffer holds (synchronous form: MO_RC_INVALID_ARGUMENT).  Device columns AND a device result: asynchronous form (as MO_XCALL_AGG).
 * float64 sums are accumulated with atomics: the association order is not fixed (|sum - exact| <= count * 2^-52 * sum |x|); MIN / MAX
 * ignore NaN (a group whose values are all NaN gives NaN with count > 0) and do not tell -0.0 from 0.0.  The specialised Q6 kernel reports
 * first_row = -1.  The TPC-H Q6 / Q1 shapes below are hand-specialised instances of this operator that reach the HBM roofline. */
#define MO_XCALL_PLAN 0x2100
#define MO_PLAN_MAX_COLS 12
#define MO_PLAN_MAX_PREDS 8
#define MO_PLAN_MAX_INSTR 16
#define MO_PLAN_MAX_KEYS 4
#define MO_PLAN_MAX_AGGS 12
#define MO_PLAN_OP_COL 0
#define MO_PLAN_OP_CONST 1
#define MO_PLAN_OP_ADD 2
#define MO_PLAN_OP_SUB 3
#define MO_PLAN_OP_MUL 4
#define MO_PLAN_OP_DIV 5
typedef struct mo_plan_pred_t { int32_t col; int32_t op; double lo; double hi; } mo_plan_pred_t;
typedef struct mo_plan_instr_t { int32_t op; int32_t a; int32_t b; int32_t reserved; double imm; } mo_plan_instr_t;
typedef struct mo_plan_agg_t { int32_t kind; int32_t value; } mo_plan_agg_t;
typedef struct mo_plan_t {
    int32_t ncols, npreds, ninstr, nkeys, naggs, has_null_keys;
    int64_t row_base;                       /* added to first_row (block-range offset of a shard) */
    int32_t col_type[MO_PLAN_MAX_COLS];
    mo_plan_pred_t pred[MO_PLAN_MAX_PREDS];
    mo_plan_instr_t instr[MO_PLAN_MAX_INSTR];
    int32_t key_col[MO_PLAN_MAX_KEYS];
    mo_plan_agg_t agg[MO_PLAN_MAX_AGGS];
} mo_plan_t;
typedef struct mo_plan_result_header_t { int64_t ngroups; int32_t sorted; int32_t overflow; int64_t reserved; } mo_plan_result_header_t;
typedef struct mo_plan_group_t { uint64_t key; int64_t first_row; int64_t rows; } mo_plan_group_t;
typedef struct mo_plan_agg_value_t { double value; int64_t count; } mo_plan_agg_value_t;

#define MO_XCALL_Q6_FILTER_SUM 0x2000
typedef struct mo_q6_params_t {
    int32_t date_lo, date_hi;  /* date_lo <= d < date_hi */
    double disc_lo, disc_hi;   /* disc_lo <= b <= disc_hi (BETWEEN) */
    double qty_hi;             /* c < qty_hi */
} mo_q6_params_t;

/* Asynchronous form: device columns AND a device result (pdata 16 bytes = {f64 sum, i64 qualifying rows}, pnulls device or NULL): the
 * call enqueues the kernel on the calling thread's stream and returns at once.  A host column or result word makes it synchronous.
 * MO_XCALL_Q6_MERGE (MergeGroup): args [0] result as above ; [1] len partial results of 16 bytes each, added in order; an empty partial
 * (count 0) is NULL and skipped (sumavg2.go:222-236).  Asynchronous when the partials, pdata and pnulls are device pointers. */
#define MO_XCALL_Q6_MERGE 0x2002

/* --- new: fused TPC-H Q1 shape: filter d <= cutoff, group by two 1-byte keys, 8 aggregates (q1.sql:5-12).
 * args: [0] result: pdata -> mo_q1_result_t ; [1] shipdate int32 ; [2] quantity f64 ; [3] extendedprice f64 ;
 * [4] discount f64 ; [5] tax f64 ; [6] returnflag ; [7] linestatus ; [8] params: pdata -> int32 cutoff.
 * Key columns: dataSz == len -> packed uint8 column; dataSz == 24*len -> MatrixOne varlena cells (inline char(1)). */
#define MO_XCALL_Q1_GROUP_AGG 0x2001
/* args[8] may also hold mo_q1_params_t (dataSz >= 16): row_base is added to every first_row (the block-range offset of this shard), so
 * partial results of different shards order their groups globally.  Asynchronous form as for Q6 (device columns + device result);
 * there "more than MO_Q1_MAX_GROUPS keys" is reported as ngroups = -1 instead of MO_RC_INVALID_ARGUMENT.
 * MO_XCALL_Q1_MERGE (MergeGroup): args [0] mo_q1_result_t ; [1] len partial mo_q1_result_t, merged in order, groups re-sorted by
 * first_row, averages recomputed from the merged sums and counts. */
#define MO_XCALL_Q1_MERGE 0x2003
typedef struct mo_q1_params_t { int32_t cutoff; int32_t reserved; int64_t row_base; } mo_q1_params_t;
#define MO_Q1_MAX_GROUPS 8
typedef struct mo_q1_group_t {
    uint8_t returnflag, linestatus; uint8_t pad[6];
    int64_t first_row;      /* global row index of the first qualifying row of the group (first-seen order) */
    double sum_qty, sum_base_price, sum_disc_price, sum_charge, avg_qty, avg_price, avg_disc;
    double sum_disc;        /* numerator of avg_disc (partials for a cross-GPU reduce) */
    int64_t count_order;
} mo_q1_group_t;
typedef struct mo_q1_result_t {
    int64_t ngroups;        /* groups sorted by first_row (= reference first-seen group-id order) */
    mo_q1_group_t groups[MO_Q1_MAX_GROUPS];
} mo_q1_result_t;

/* --- new: fused TPC-H Q6 over DECIMAL(15,2) columns (the reference's own lineitem schema), exact to the digit.
 * args: [0] result: pdata -> mo_q6_dec_result_t, pnulls (optional) -> nulls word, bit 0 = no row qualified ; [1] shipdate int32 ;
 * [2] discount ; [3] quantity ; [4] extendedprice (Decimal64 = int64 unscaled, all of one scale) ; [5] params: pdata -> mo_q6_dec_params_t.
 * The result equals the reference's operator chain: filter (date_lo <= d < date_hi, disc_lo <= discount <= disc_hi, quantity < qty_hi, the
 * constants already cast to the column scale, so each compare is an int64 compare), Shrink, d64Mul(extendedprice, discount) -> Decimal128 at
 * scale 2 * scale, SUM with the checked Add128 of sumDecimal128FastExec.  The sum is exact and independent of the summation order.
 * scale must be 0..4 (every product then keeps its full scale); other scales and columns with a nulls bitmap (the schema's columns are
 * NOT NULL) are rejected with MO_RC_INVALID_ARGUMENT -- the decimal operator chain (DEC_ARITH, DEC_SUM) serves them.
 * Errors: the call fails iff one pipeline over the qualifying rows in row order would fail, i.e. the running sum leaves int128 at some row:
 * rc = MO_RC_INVALID_ARGUMENT ("Decimal128 Add overflow") and err_row = the lowest such row, params.row_base included.  The reference's message names the values, not
 * the row, and which of several errors it raises first depends on its batch order.  Asynchronous form (device columns AND a device result:
 * enqueue only) as for Q6_FILTER_SUM: the call returns MO_RC_SUCCESS and the failure is reported in result.rc / result.err_row.
 * MO_XCALL_Q6_DEC_MERGE (MergeGroup): args [0] result as above ; [1] len partial mo_q6_dec_result_t, folded in order: an empty partial
 * (count 0) is skipped, a failing partial fails the merge with the lowest err_row of the failing partials (global rows when each range was
 * scanned with its row_base), the sum is checked as BatchMerge does (an overflow there, or partials of different scales, with no failing
 * partial: rc = MO_RC_INVALID_ARGUMENT with err_row = -1). */
#define MO_XCALL_Q6_DEC_FILTER_SUM 0x2004
#define MO_XCALL_Q6_DEC_MERGE 0x2006
typedef struct mo_dec128_t { uint64_t lo, hi; } mo_dec128_t;   /* Decimal128: two's complement {B0_63, B64_127} */
typedef struct mo_q6_dec_params_t {
    int32_t date_lo, date_hi;           /* date_lo <= d < date_hi */
    int64_t disc_lo, disc_hi;           /* disc_lo <= discount <= disc_hi (BETWEEN), unscaled at `scale` */
    int64_t qty_hi;                     /* quantity < qty_hi, unscaled at `scale` */
    int32_t scale;                      /* scale of the four Decimal64 measures, 0..4 */
    int32_t reserved;
    int64_t row_base;                   /* added to err_row: the global row of this range's first row */
} mo_q6_dec_params_t;
typedef struct mo_q6_dec_result_t {
    mo_dec128_t revenue;                /* SUM(l_extendedprice * l_discount), Decimal128 at scale `scale` */
    int64_t count;                      /* qualifying rows */
    int64_t err_row;                    /* lowest failing row, -1 when rc == 0 */
    int32_t rc;                         /* MO_RC_SUCCESS or MO_RC_INVALID_ARGUMENT */
    int32_t scale;                      /* 2 * params.scale */
} mo_q6_dec_result_t;

/* --- new: brute-force top-k (GoBruteForceIndex.Search, pkg/vectorindex/brute_force/brute_force.go:248-341).
 * args: [0] result keys int64[nq*k] ; [1] result distances f64[nq*k] ; [2] dataset f32 row-major (dataSz = n*dim*4)
 * ; [3] queries f32 row-major (dataSz = nq*dim*4) ; [4] params: pdata -> mo_search_params_t.  len = nq.
 * Distances are bit-exact with the Go metric functions; ties between equal distances resolve to the lower row id. */
#define MO_XCALL_BRUTEFORCE_TOPK_F32 0x3000
/* IVF-flat probe (IvfflatSearchIndex.Search, pkg/vectorindex/ivfflat/search.go:509-630):
 * args as above plus [5] centroids f32 (nlist*dim) ; [6] list offsets int64[nlist+1] into a list-ordered dataset ;
 * [7] row ids int64[n] (original pk of each list-ordered row). */
#define MO_XCALL_IVF_TOPK_F32 0x3001
typedef struct mo_search_params_t {
    int64_t n, dim, nq;
    int32_t k;        /* RuntimeConfig.Limit */
    int32_t metric;   /* MO_METRIC_* */
    int32_t nprobe;   /* IVF only */
    int32_t sqrt_out; /* DistanceTransformIvfflat: sqrt on the final k (user asked l2_distance) */
    int64_t nlist;    /* IVF only */
    int64_t key_base; /* added to row ordinals (dataset shard offset in a multi-GPU run) */
} mo_search_params_t;
#define MO_METRIC_L2 0      /* metric/types.go MetricType: both L2 variants search with L2sq (distance_func.go:507-524) */
#define MO_METRIC_IP 1
#define MO_METRIC_COS 2
#define MO_METRIC_L1 3
#define MO_METRIC_L2SQ 4

/* merge of per-shard top-k lists (MergeTop / hnsw sub-index merge, pkg/vectorindex/hnsw/search.go:89-135):
 * args: [0] out keys int64[nq*k] ; [1] out dist f64[nq*k] ; [2] in keys int64[nshards*nq*k] ; [3] in dist f64[...] ;
 * [4] params mo_search_params_t (n = nshards, nq, k). */
#define MO_XCALL_TOPK_MERGE 0x3002

/* Filtered search: the unfiltered entry point run over the ADMITTED rows only, with the original keys.
 * MO_XCALL_BRUTEFORCE_TOPK_FILTERED_F32: args [0..4] as MO_XCALL_BRUTEFORCE_TOPK_F32, [5] filter: pdata -> mo_search_filter_t.
 *   The key of a row is key_base + row ordinal.
 * MO_XCALL_IVF_TOPK_FILTERED_F32: args [0..7] as MO_XCALL_IVF_TOPK_F32, [8] filter: pdata -> mo_search_filter_t.
 *   The key of a row is row_ids[row] (the primary key); the probes are those of the unfiltered search.
 * Admission: KEY_BITMAP admits a key whose bit is set (bitmap_test_with_len, cgo/bitmap.h:55-63; a key at or past 64 * nwords, or
 * negative, is rejected); KEY_BLOOM admits a key for which bloomfilter_test of its 8 little-endian bytes is true (the filter's
 * current bits, including those added on the device).  Fewer than k admitted rows: front padding (key -1, distance 0); brute force
 * with k = 1 and no admitted row: key -1, distance MaxFloat32 (brute_force.go:289-331).  An unknown kind, a null filter or a
 * descriptor shorter than mo_search_filter_t: MO_RC_INVALID_ARGUMENT. */
#define MO_XCALL_BRUTEFORCE_TOPK_FILTERED_F32 0x3003
#define MO_XCALL_IVF_TOPK_FILTERED_F32 0x3004
#define MO_SEARCH_FILTER_KEY_BITMAP 1
#define MO_SEARCH_FILTER_KEY_BLOOM 2
typedef struct mo_search_filter_t {
    int32_t kind;          /* MO_SEARCH_FILTER_KEY_BITMAP | MO_SEARCH_FILTER_KEY_BLOOM */
    int32_t pad;
    const void *filter;    /* KEY_BITMAP: uint64_t words (host or device); KEY_BLOOM: bloomfilter_t * of mo_b200_bloom.h */
    uint64_t nwords;       /* KEY_BITMAP only: length in 64-bit words */
} mo_search_filter_t;

/* ======================================================================================================
 * PART 3 -- runtime / residency extension
 * ==================================================================================================== */
int32_t MoB200_Init(int32_t device);          /* idempotent; device < 0 -> $MO_B200_DEVICE, $LOCAL_RANK or 0 */
const char *MoB200_Version(void);
int32_t MoB200_DeviceCount(void);
int32_t MoB200_DeviceAlloc(uint64_t bytes, void **dptr);
int32_t MoB200_DeviceFree(void *dptr);
int32_t MoB200_HostAlloc(uint64_t bytes, void **hptr);  /* pinned host memory (replaces malloc.CAllocator) */
int32_t MoB200_HostFree(void *hptr);
int32_t MoB200_HostRegister(void *hptr, uint64_t bytes);
int32_t MoB200_HostUnregister(void *hptr);
int32_t MoB200_Upload(void *dst_dev, const void *src_host, uint64_t bytes);   /* on the calling thread's stream, synchronous */
int32_t MoB200_Download(void *dst_host, const void *src_dev, uint64_t bytes);
int32_t MoB200_DownloadAsync(void *dst_host, const void *src_dev, uint64_t bytes);  /* stream-ordered, NO synchronise (pinned host memory) */
int32_t MoB200_UploadAsync(void *dst_dev, const void *src_host, uint64_t bytes);
int32_t MoB200_Memset(void *dst_dev, int32_t value, uint64_t bytes);
/* Device column cache (off by default).  The ABI hands the library HOST vectors; re-uploading a column on every call makes every call
 * PCIe-bound (the reference's CUDA shim re-allocates and re-copies per call, cgo/cuda/cuda.cpp:123-201).  A caller that knows a host range is
 * immutable -- the column of a decoded block, an index's dataset -- pins it once: ColumnPin uploads [host, host + bytes) and from then on EVERY
 * entry point that is handed a host pointer inside that range reads the device copy instead of staging it.  `generation` distinguishes reuses of
 * the same buffer (block id / version): pinning the same address with another generation replaces the copy.  LRU eviction beyond the capacity. */
int32_t MoB200_ColumnCacheConfigure(uint64_t capacity_bytes);   /* 0 = off (drops everything) */
int32_t MoB200_ColumnPin(const void *host, uint64_t bytes, uint64_t generation);
int32_t MoB200_ColumnUnpin(const void *host);
int32_t MoB200_ColumnCacheStats(uint64_t *hits, uint64_t *misses, uint64_t *bytes);

/* prepared join maps: build the probe-side device hash table of a JoinMap once (the JoinMap message lives for the whole probe phase,
 * pkg/vm/message/joinMapMsg.go:127-160); JOIN_FIND / JOIN_PROBE calls whose table_keys pointer equals `table_keys` reuse it. */
int32_t MoB200_JoinMapPrepare(const void *table_keys, uint64_t ngroups);
/* the same for a STR_GROUP_IDS table (copied to the device): STR_JOIN_FIND calls whose table offsets pointer equals `table_offsets` reuse it */
int32_t MoB200_StrJoinMapPrepare(const void *table_bytes, const void *table_offsets, uint64_t ngroups);
int32_t MoB200_JoinMapRelease(const void *table_keys);   /* either kind: table_keys, or the table_offsets of a string map */
int32_t MoB200_Sync(void);                    /* synchronize the calling thread's stream */
int32_t MoB200_SetStream(void *cuda_stream);  /* adopt an external cudaStream_t for the calling thread (NULL = own) */
int32_t MoB200_TimerStart(void);              /* CUDA event on the calling thread's stream */
int32_t MoB200_TimerStop(float *ms);          /* records, synchronizes, returns elapsed milliseconds */
uint64_t MoB200_KernelLaunchCount(void);      /* kernels launched by this library since load (all threads) */
int32_t MoB200_LastKernelMs(float *ms);       /* device time of the dominant kernel of the calling thread's last call (CUDA events) */
int32_t MoB200_LastError(char *buf, uint64_t buflen);  /* thread-local last error text */
int32_t MoB200_FlushL2(void);                 /* write a >L2-sized scratch buffer (bench hygiene) */
int32_t MoB200_SetTuning(const char *name, int32_t value);  /* kernel-variant knobs used by tools/tune.py; returns 0 if name and value are known, else -1
                                                             * (search_filter_path: 0 auto, 1 masked scan, 2 compacted admitted rows;
                                                             * strkey_hash_bits, test only: string-key hashes keep their low 1..63 bits, 0 = all,
                                                             * so that hash tags collide and the key byte compare is exercised) */

/* synthetic column generators used by bench.py / tests (counter-based, reproducible on the host: see
 * matrixone_b200/datagen.py).  All write DEVICE memory, rows [row0, row0+n). */
int32_t MoB200_GenLineitem(uint64_t seed, uint64_t row0, uint64_t n, int32_t *shipdate, double *quantity,
                           double *extendedprice, double *discount, double *tax, uint8_t *returnflag, uint8_t *linestatus);
int32_t MoB200_GenInt64(uint64_t seed, uint64_t row0, uint64_t n, int64_t *out, uint64_t *nulls, uint32_t null_per_mille);
int32_t MoB200_GenVectorsF32(uint64_t seed, uint64_t row0, uint64_t n, int64_t dim, float *out,
                             const float *centers, int64_t ncenters, float sigma);
int32_t MoB200_GatherRowsF32(float *dst, const float *src, const int64_t *idx, uint64_t m, int64_t dim);  /* device pointers */

/* Index load hooks (brute_force.go:104-123 Load / ivfflat/search.go:216-290 LoadIndex build the reference's in-memory index once;
 * Destroy frees it).  SearchPrepare splits a RESIDENT float32 dataset [n][dim] into the tensor-core operand of
 * MO_XCALL_BRUTEFORCE_TOPK_F32 / MO_XCALL_IVF_TOPK_F32 once, instead of once per search; the rows must not change until
 * SearchRelease(data).  Optional: searches return identical results with or without it.  Costs 6*dim bytes of HBM per row. */
int32_t MoB200_SearchPrepare(const void *data, uint64_t n, int64_t dim);   /* = SearchPrepareMetric(..., MO_METRIC_L2) */
/* MO_METRIC_L2 / L2SQ / IP share one operand; MO_METRIC_COS keeps the rows normalised; other metrics have nothing to prepare */
int32_t MoB200_SearchPrepareMetric(const void *data, uint64_t n, int64_t dim, int32_t metric);
/* IVF-flat: the list-ordered entries are split as residuals against their list's centroid (centroids [nlist][dim] float32,
 * offsets [nlist + 1] int64, device pointers; the same buffers MO_XCALL_IVF_TOPK_F32 is later called with). */
int32_t MoB200_SearchPrepareIvf(const void *data, uint64_t n, int64_t dim, const void *centroids, uint64_t nlist, const void *offsets);
int32_t MoB200_SearchRelease(const void *data);

#ifdef __cplusplus
}
#endif
#endif /* _MO_B200_H_ */
