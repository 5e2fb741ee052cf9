// caseexpr.cu -- conditional values of the Go expression engine: CASE WHEN ... THEN ... [ELSE ...] END and IF (caseFn / generalCaseFn /
// strCaseFn / iffFn, operatorSet.go:144-316,389-), COALESCE (CoalesceGeneral / CoalesceStr, func_binary.go:938-993), and the select lists
// of EvalCase / EvalIff (evalExpression.go:501-573) as null-prefill words.
// funcIds and argument layout: include/mo_b200.h (MO_XCALL_GO_CASE, MO_XCALL_GO_COALESCE, MO_XCALL_GO_CASE_SELECT); the operand protocol:
// goengine.cuh, except that no null merge applies -- a NULL operand only matters on the rows that reach it.
//
// Every row walks the operands in order and stops at its choice: CASE reads condition j only where no earlier WHEN matched and the chosen
// value only where it is chosen, COALESCE reads null bits up to the first non-NULL operand.  The operand descriptors are one device array
// (up to 2 * 1024 + 1 of them), read by every thread of a warp at once.
//   fixed width  one launch, templated on the value's width (1, 2, 4, 8, 16 bytes): the bytes are selected, never interpreted.  A warp owns
//                32 consecutive rows, one aligned half word of the result bitmap, which its ballot writes whole (skipped rows keep their bit).
//   strings      three launches.  pick: per row the chosen operand, the bad-cell record, and per CTA the bytes its non-inline values need;
//                scan: the exclusive scan of those sums and the total; write (after the one read-back of the status record, only when the
//                area is large enough and no chosen cell is bad): cells, bitmap and area bytes.  Each CTA owns one contiguous range of rows,
//                so the area is filled in row order; a long value is copied by a whole warp.
#include "goengine.cuh"
#include <vector>

using namespace mob;

namespace {

constexpr int kCtasPerSm = 16;
constexpr int kScanThreads = 1024;
constexpr int32_t kPickNull = -1, kPickSkip = -2;   // a row's choice besides an operand index: NULL, or skipped (result null bit set on entry)

struct V16 { uint64_t lo, hi; };
template <int W> struct Word;
template <> struct Word<1> { using T = uint8_t; };
template <> struct Word<2> { using T = uint16_t; };
template <> struct Word<4> { using T = uint32_t; };
template <> struct Word<8> { using T = uint64_t; };
template <> struct Word<16> { using T = V16; };

// the status record of the string calls: bad = min over the rows that chose a bad cell (a const operand's included) of row * 4096 +
// argument index (~0: none), total = area bytes
struct CaseStatus { unsigned long long bad, total; };

// the operand row i of the call chooses: CASE (ops: condition j at 2j, value j at 2j + 1, ELSE at 2n) or COALESCE (ops: operand j at j);
// kPickNull when the row is NULL
__device__ __forceinline__ int32_t pick_row(const Operand *__restrict__ ops, int n, int has_else, int coalesce, uint64_t i) {
    if (coalesce) {
        for (int j = 0; j < n; j++) if (!bm_test(ops[j].nulls, ops[j].cst ? 0 : i)) return j;
        return kPickNull;
    }
    int32_t k = has_else ? 2 * n : kPickNull;
    for (int j = 0; j < n; j++) {
        const Operand &c = ops[2 * j];
        const uint64_t r = c.cst ? 0 : i;
        if (!bm_test(c.nulls, r) && static_cast<const uint8_t *>(c.data)[r]) { k = 2 * j + 1; break; }
    }
    if (k >= 0 && bm_test(ops[k].nulls, ops[k].cst ? 0 : i)) k = kPickNull;
    return k;
}

template <int W>
__global__ void __launch_bounds__(kThreads)
case_fixed_kernel(typename Word<W>::T *__restrict__ r, uint32_t *__restrict__ rn32, uint64_t n, const Operand *__restrict__ ops, int nsel,
                  int has_else, int coalesce) {
    using T = typename Word<W>::T;
    const uint64_t n64 = (n + 63) & ~63ull;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n64; i += (uint64_t)gridDim.x * kThreads) {
        bool isnull = false;
        if (i < n) {
            if ((rn32[i >> 5] >> (i & 31)) & 1u) isnull = true;   // skipped: the value is left as it was
            else {
                const int32_t k = pick_row(ops, nsel, has_else, coalesce, i);
                T v{};
                if (k >= 0) v = static_cast<const T *>(ops[k].data)[ops[k].cst ? 0 : i];
                else isnull = true;
                r[i] = v;
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, isnull);
        if ((threadIdx.x & 31) == 0) rn32[i >> 5] = m;
    }
}

// inclusive scan of v over the CTA (NT threads); *total = the CTA's sum.  sm: NT / 32 words.
template <int NT>
__device__ __forceinline__ unsigned long long block_scan(unsigned long long v, unsigned long long &total, unsigned long long *sm) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) sm[wid] = x;
    __syncthreads();
    if (wid == 0) {
        unsigned long long w = lane < NT / 32 ? sm[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
        if (lane < NT / 32) sm[lane] = w;
    }
    __syncthreads();
    const unsigned long long before = wid ? sm[wid - 1] : 0;
    total = sm[NT / 32 - 1];
    __syncthreads();
    return before + x;
}

// CTA b owns rows [b * chunk, (b + 1) * chunk)
__global__ void __launch_bounds__(kThreads)
case_str_pick_kernel(int32_t *__restrict__ pick, const uint32_t *__restrict__ rn32, uint64_t n, uint64_t chunk, const Operand *__restrict__ ops,
                     int nsel, int has_else, int coalesce, unsigned long long *__restrict__ cta_sum, CaseStatus *st) {
    __shared__ unsigned long long sm[kThreads / 32];
    const uint64_t lo = blockIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
    unsigned long long sum = 0;
    for (uint64_t i = lo + threadIdx.x; i < hi; i += kThreads) {
        int32_t k = kPickSkip;
        if (!((rn32[i >> 5] >> (i & 31)) & 1u)) {
            k = pick_row(ops, nsel, has_else, coalesce, i);
            Str s;
            if (k >= 0) {
                if (!load_str(ops[k], i, s)) atomicMin(&st->bad, (unsigned long long)i * 4096ull + (unsigned)(k + 2));   // a const too: the row that chose it
                else if (!s.inl) sum += s.len;
            }
        }
        pick[i] = k;
    }
    unsigned long long total;
    block_scan<kThreads>(sum, total, sm);
    if (threadIdx.x == 0) cta_sum[blockIdx.x] = total;
}

// one CTA: cta_sum becomes its exclusive scan, st->total the sum
__global__ void __launch_bounds__(kScanThreads) case_str_scan_kernel(unsigned long long *cta_sum, int nblk, CaseStatus *st) {
    __shared__ unsigned long long sm[kScanThreads / 32];
    unsigned long long carry = 0;
    for (int base = 0; base < nblk; base += kScanThreads) {
        const int j = base + (int)threadIdx.x;
        const unsigned long long v = j < nblk ? cta_sum[j] : 0;
        unsigned long long total;
        const unsigned long long incl = block_scan<kScanThreads>(v, total, sm);
        if (j < nblk) cta_sum[j] = carry + incl - v;
        carry += total;
    }
    if (threadIdx.x == 0) st->total = carry;
}

// bytes [0, k) of an inline cell's word q (bytes 8q .. 8q + 7), the rest zero
__device__ __forceinline__ uint64_t keep_bytes(uint64_t w, uint32_t k, int q) {
    const int c = (int)k - 8 * q;
    return c >= 8 ? w : (c <= 0 ? 0 : w & ((1ull << (8 * c)) - 1));
}

__global__ void __launch_bounds__(kThreads)
case_str_write_kernel(uint8_t *__restrict__ cells, uint32_t *__restrict__ rn32, uint8_t *__restrict__ area, const int32_t *__restrict__ pick,
                      uint64_t n, uint64_t chunk, const Operand *__restrict__ ops, const unsigned long long *__restrict__ cta_base) {
    __shared__ unsigned long long sm[kThreads / 32];
    const int lane = threadIdx.x & 31;
    const uint64_t n64 = (n + 63) & ~63ull;
    const uint64_t lo = blockIdx.x * chunk, hi = lo + chunk < n64 ? lo + chunk : n64;
    const bool aligned = (reinterpret_cast<uintptr_t>(cells) & 7) == 0;
    unsigned long long base = cta_base[blockIdx.x];
    for (uint64_t t0 = lo; t0 < hi; t0 += kThreads) {
        const uint64_t i = t0 + threadIdx.x;
        const int32_t k = i < n ? pick[i] : kPickSkip;
        Str s;
        s.inl = true; s.len = 0; s.w0 = s.w1 = s.w2 = 0; s.p = nullptr;
        if (k >= 0) load_str(ops[k], i, s);          // the pick checked the cell
        const unsigned long long L = s.inl ? 0 : s.len;
        unsigned long long tot;
        const unsigned long long off = base + block_scan<kThreads>(L, tot, sm) - L;
        base += tot;
        if (k != kPickSkip) {
            uint64_t w[3];
            if (k == kPickNull) w[0] = w[1] = w[2] = 0;   // a NULL row: the empty inline cell
            else if (s.inl) { w[0] = keep_bytes(s.w0, s.len + 1, 0); w[1] = keep_bytes(s.w1, s.len + 1, 1); w[2] = keep_bytes(s.w2, s.len + 1, 2); }
            else { w[0] = 0xffffffffull | ((uint64_t)(uint32_t)off << 32); w[1] = s.len; w[2] = 0; }
            uint8_t *c = cells + 24 * i;
            if (aligned) { uint64_t *q = reinterpret_cast<uint64_t *>(c); q[0] = w[0]; q[1] = w[1]; q[2] = w[2]; }
            else for (int b = 0; b < 24; b++) c[b] = (uint8_t)(w[b >> 3] >> (8 * (b & 7)));
        }
        const unsigned m = __ballot_sync(0xffffffffu, i < n && k < 0);
        if (lane == 0 && i < n64) rn32[i >> 5] = m;
        // the warp copies its long values one after another, 32 bytes per step
        unsigned lv = __ballot_sync(0xffffffffu, L != 0);
        while (lv) {
            const int src = __ffs(lv) - 1;
            lv &= lv - 1;
            const uint8_t *p = reinterpret_cast<const uint8_t *>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(s.p), src));
            const unsigned long long o = __shfl_sync(0xffffffffu, off, src);
            const uint32_t len = __shfl_sync(0xffffffffu, s.len, src);
            for (uint32_t b = lane; b < len; b += 32) area[o + b] = __ldg(p + b);
        }
    }
}

// took = ~rem & cond & ~cond_nulls over rows [0, n): then = ~took, rem |= took; a warp owns an aligned half word of both
__global__ void __launch_bounds__(kThreads) case_select_kernel(uint32_t *__restrict__ then32, uint32_t *__restrict__ rem32, uint64_t n, Operand c) {
    const uint64_t n64 = (n + 63) & ~63ull;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n64; i += (uint64_t)gridDim.x * kThreads) {
        bool took = false;
        if (i < n && !((rem32[i >> 5] >> (i & 31)) & 1u)) {
            const uint64_t r = c.cst ? 0 : i;
            took = !bm_test(c.nulls, r) && static_cast<const uint8_t *>(c.data)[r] != 0;
        }
        const unsigned m = __ballot_sync(0xffffffffu, took);
        if ((threadIdx.x & 31) == 0) { then32[i >> 5] = ~m; rem32[i >> 5] |= m; }
    }
}

// value bytes per row of a GO_CASE / GO_COALESCE type: 1..16 fixed width, MO_VARLENA_SZ for the strings, 0 = refused
int case_width(int T) {
    switch (T) {
    case MO_T_BOOL: case MO_T_INT8: case MO_T_UINT8: return 1;
    case MO_T_INT16: case MO_T_UINT16: case MO_T_ENUM: return 2;
    case MO_T_INT32: case MO_T_UINT32: case MO_T_FLOAT32: case MO_T_DATE: return 4;
    case MO_T_INT64: case MO_T_UINT64: case MO_T_FLOAT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: case MO_T_DECIMAL64: case MO_T_BIT:
        return 8;
    case MO_T_DECIMAL128: case MO_T_UUID: return 16;
    case MO_T_CHAR: case MO_T_VARCHAR: case MO_T_BLOB: case MO_T_TEXT: case MO_T_DATALINK: return MO_VARLENA_SZ;
    }
    return 0;
}

// the parameter block and the operands, staged; dops = their descriptors in device memory.  nsel = the WHEN count (CASE) or operand count.
int stage_case(ThreadCtx &t, Stager &st, mo_xcall_args_t *args, uint64_t len, size_t elem, int coalesce, const char *what, mo_case_params_t &P,
               const Operand *&dops) {
    char pw[64];
    snprintf(pw, sizeof pw, "%s: params", what);
    if (int rc = read_param(t, args[1], &P, sizeof P, sizeof P, pw)) return rc;
    if (P.n < 1 || P.n > MO_CASE_MAX_WHENS) { set_error("%s: n %d outside 1..%d", what, P.n, MO_CASE_MAX_WHENS); return MO_RC_INVALID_ARGUMENT; }
    if (P.has_else != 0 && (P.has_else != 1 || coalesce)) {
        set_error("%s: has_else %d (%s)", what, P.has_else, coalesce ? "must be 0" : "0 or 1"); return MO_RC_INVALID_ARGUMENT;
    }
    const int nops = coalesce ? P.n : 2 * P.n + P.has_else;
    std::vector<Operand> ops(nops);
    for (int k = 0; k < nops; k++) {
        const bool cond = !coalesce && k < 2 * P.n && !(k & 1);
        if (int rc = stage_operand(st, args[2 + k], cond ? 1 : elem, len, what, 2 + k, ops[k])) return rc;
    }
    Operand *d = (Operand *)st.tmp(nops * sizeof(Operand));
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    // pageable source: the runtime copies it into its own staging before this returns, so the vector may go out of scope
    MOB_CUDA_TRY(cudaMemcpyAsync(d, ops.data(), nops * sizeof(Operand), cudaMemcpyHostToDevice, t.stream));
    dops = d;
    return MO_RC_SUCCESS;
}

template <int W>
int run_case_fixed(ThreadCtx &t, int coalesce, mo_xcall_args_t *args, uint64_t len, const char *what) {
    using T = typename Word<W>::T;
    Stager st(t);
    mo_case_params_t P;
    const Operand *ops;
    T *r; uint64_t *rn;
    if (int rc = stage_result(st, args[0], W, len, true, true, what, r, rn)) return rc;
    if (int rc = stage_case(t, st, args, len, W, coalesce, what, P, ops)) return rc;
    cudaEventRecord(t.kev0, t.stream);
    case_fixed_kernel<W><<<grid_rows((len + 63) & ~63ull, kCtasPerSm), kThreads, 0, t.stream>>>(r, reinterpret_cast<uint32_t *>(rn), len, ops, P.n,
                                                                                             P.has_else, coalesce);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.complete();
}

int run_case_str(ThreadCtx &t, int coalesce, mo_xcall_args_t *args, uint64_t len, const char *what) {
    Stager st(t);
    mo_case_params_t P;
    const Operand *ops;
    uint8_t *cells; uint64_t *rn;
    if (int rc = stage_result(st, args[0], MO_VARLENA_SZ, len, true, true, what, cells, rn)) return rc;
    if (int rc = stage_case(t, st, args, len, MO_VARLENA_SZ, coalesce, what, P, ops)) return rc;
    // contiguous row ranges, a multiple of kThreads rows each (whole bitmap words per CTA)
    const uint64_t nblk0 = (uint64_t)grid_rows(len, kCtasPerSm);
    const uint64_t chunk = ((len + nblk0 - 1) / nblk0 + kThreads - 1) / kThreads * kThreads;
    const int nblk = (int)((len + chunk - 1) / chunk);
    int32_t *pick = (int32_t *)st.tmp(len * 4);
    unsigned long long *cta = (unsigned long long *)st.tmp(nblk * 8);
    CaseStatus *dst = (CaseStatus *)st.tmp(sizeof(CaseStatus));
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dst, 0xff, sizeof(CaseStatus), t.stream));
    const uint32_t *rn32 = reinterpret_cast<const uint32_t *>(rn);
    case_str_pick_kernel<<<nblk, kThreads, 0, t.stream>>>(pick, rn32, len, chunk, ops, P.n, P.has_else, coalesce, cta, dst);
    MOB_LAUNCH_CHECK();
    case_str_scan_kernel<<<1, kScanThreads, 0, t.stream>>>(cta, nblk, dst);
    MOB_LAUNCH_CHECK();
    CaseStatus hs;
    if (int rc = read_back(t, &hs, dst, sizeof hs)) return rc;
    P.area_len = (int64_t)hs.total;
    if (int rc = write_param(t, args[1].pdata + offsetof(mo_case_params_t, area_len), &P.area_len, sizeof P.area_len)) return rc;
    // a failed call returns through the Stager's destructor: nothing is copied back, so a host result is unchanged too
    if (hs.bad != ~0ull) {
        set_error("%s: operand %d row %llu: varlena cell outside its area", what, (int)(hs.bad & 4095), hs.bad >> 12);
        return MO_RC_INVALID_ARGUMENT;
    }
    const uint64_t cap = args[0].parea ? args[0].areaSz : 0;
    if (hs.total > 0xffffffffull || hs.total > cap) {
        set_error("%s: the result needs %llu area bytes, its area holds %llu%s", what, hs.total, (unsigned long long)cap,
                  hs.total > 0xffffffffull ? " (offsets are 32-bit)" : "");
        return MO_RC_OUT_OF_RANGE;
    }
    uint8_t *area = hs.total ? (uint8_t *)st.out(args[0].parea, hs.total, false) : nullptr;
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    cudaEventRecord(t.kev0, t.stream);
    case_str_write_kernel<<<nblk, kThreads, 0, t.stream>>>(cells, reinterpret_cast<uint32_t *>(rn), area, pick, len, chunk, ops, cta);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.complete();
}

}  // namespace

namespace mob {

// MO_XCALL_GO_CASE(T) / MO_XCALL_GO_COALESCE(T)
int xcall_go_case(int coalesce, int T, mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    const char *what = coalesce ? "go coalesce" : "go case";
    switch (case_width(T)) {
    case 1: return run_case_fixed<1>(t, coalesce, args, len, what);
    case 2: return run_case_fixed<2>(t, coalesce, args, len, what);
    case 4: return run_case_fixed<4>(t, coalesce, args, len, what);
    case 8: return run_case_fixed<8>(t, coalesce, args, len, what);
    case 16: return run_case_fixed<16>(t, coalesce, args, len, what);
    case MO_VARLENA_SZ: return run_case_str(t, coalesce, args, len, what);
    }
    set_error("%s: unsupported type %d", what, T);
    return MO_RC_INVALID_ARGUMENT;
}

// MO_XCALL_GO_CASE_SELECT: args [0] THEN j's prefill words (out) ; [1] the remaining words (in / out) ; [2] condition j
int xcall_case_select(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    const char *what = "go case select";
    const uint64_t wbytes = ((len + 63) / 64) * 8;
    for (int k = 0; k < 2; k++)
        if (!args[k].pdata || args[k].dataSz < wbytes) {
            set_error("%s: operand %d holds %llu bytes, %llu needed", what, k, (unsigned long long)args[k].dataSz, (unsigned long long)wbytes);
            return MO_RC_INVALID_ARGUMENT;
        }
    Stager st(t);
    Operand c;
    uint32_t *then32 = (uint32_t *)st.out(args[0].pdata, wbytes, false);
    uint32_t *rem32 = (uint32_t *)st.out(args[1].pdata, wbytes, true);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    if (int rc = stage_operand(st, args[2], 1, len, what, 2, c)) return rc;
    cudaEventRecord(t.kev0, t.stream);
    case_select_kernel<<<grid_rows((len + 63) & ~63ull, kCtasPerSm), kThreads, 0, t.stream>>>(then32, rem32, len, c);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.complete();
}

}  // namespace mob
