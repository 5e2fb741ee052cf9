// common.cuh -- runtime plumbing shared by every translation unit of libmo_b200.so.
//
// One ThreadCtx per calling OS thread (the reference calls the cgo surface from arbitrary goroutines pinned to
// arbitrary OS threads, pkg/sql/compile/scope.go:442-499): its own CUDA stream, timing events, a device scratch
// arena and a small pinned staging buffer, so concurrent callers never share mutable state.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <vector>
#include <atomic>
#include <memory>
#include "../../include/mo_b200.h"

namespace mob {

constexpr int kSMs = 132;  // H100 SXM; grids are sized in multiples of the device's SM count (num_sms(), this until it is known)

struct ArenaBlock { char *p; size_t size; };

struct ThreadCtx {
    cudaStream_t stream = nullptr;
    bool own_stream = true;
    bool ready = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t kev0 = nullptr, kev1 = nullptr;  // bracket the dominant kernel of the last call (MoB200_LastKernelMs)
    std::vector<ArenaBlock> blocks;  // device scratch arena (bump allocated, reset per call)
    size_t cur_block = 0, cur_off = 0;
    int kev_prio = 0;                // priority of the kernel kev0/kev1 currently bracket within this call (reset with the arena)
    uint64_t arena_epoch = 0;        // bumped by arena_reset: per-call caches of arena pointers key on it
    char *pinned = nullptr;          // small pinned staging (scalar results, status words)
    size_t pinned_sz = 0;
    unsigned *ctrl = nullptr;        // 64 device words, zero between calls ("last CTA done" tickets, atomicInc wraps)
    char err[256] = {0};
};

ThreadCtx &tctx();                      // lazily initialises the runtime and the calling thread's context
int runtime_init(int device);           // idempotent
void set_error(const char *fmt, ...);
extern std::atomic<uint64_t> g_launches;
int num_sms();

// cudaPointerGetAttributes classification
bool is_device_ptr(const void *p);

// prepared search operands (tcsearch.cu) that read [p, p + bytes) are dropped: called by every library entry point that WRITES device memory
void search_invalidate(const void *p, uint64_t bytes);
// MoB200_SetTuning names of the search module (tcsearch.cu): false for any other name, else *out = the answer (0 for a knob)
bool search_tuning(const char *name, int value, int *out);
// MoB200_SetTuning("strkey_hash_bits", b), test only (colops.cu): string-key hashes keep their low b bits (1..63; 0 = all 64), so that hash tags
// collide and the byte compare of the key table runs
extern int g_strkey_hash_bits;
inline uint64_t strkey_hash_mask() { const int b = g_strkey_hash_bits; return b <= 0 || b >= 64 ? ~0ull : (1ull << b) - 1; }

// --- device scratch arena -------------------------------------------------------------------------------
void *arena_alloc(ThreadCtx &t, size_t bytes);   // 256-byte aligned; nullptr on failure (error set)
void arena_reset(ThreadCtx &t);                  // called at the end of every API call
// scoped scratch inside one call (loops that need temporaries per iteration): everything allocated after the mark is handed back by the rewind
struct ArenaMark { size_t block, off; };
inline ArenaMark arena_mark(ThreadCtx &t) { return ArenaMark{t.cur_block, t.cur_off}; }
inline void arena_rewind(ThreadCtx &t, ArenaMark m) { t.cur_block = m.block; t.cur_off = m.off; }

// --- Stager: makes every pointer argument a device pointer for the duration of one call -------------------
// It also decides how the call completes: a call that met only device memory is asynchronous (complete() enqueues nothing more and does
// not synchronise); a call that met any host range, a column-cache hit included, copies back and synchronises once.
struct Stager {
    ThreadCtx &t;
    struct Back { void *host; const void *dev; size_t bytes; };
    std::vector<Back> backs;
    std::vector<std::shared_ptr<void>> pins;   // column-cache blocks this call reads (kept alive until finish())
    bool failed = false;
    bool finished = false;   // set by finish(); the destructor cleans up otherwise
    explicit Stager(ThreadCtx &tc) : t(tc) {}
    // input: device pointers pass through, host pointers are copied into the arena (async on t.stream)
    const void *in(const void *p, size_t bytes);
    // output: device pointers pass through; host pointers get an arena buffer that is copied back by finish().
    // preload=true first uploads the host content (needed when the kernel writes only some rows).
    void *out(void *p, size_t bytes, bool preload = false);
    // classify a pointer the call reads or writes without staging it (a null pointer names no memory); a host answer counts as in() / out()
    bool device(const void *p) { if (!p || is_device_ptr(p)) return true; host_seen = true; return false; }
    // no host range met so far
    bool resident() const { return !host_seen; }
    // device temp
    void *tmp(size_t bytes) { void *q = arena_alloc(t, bytes); if (!q) failed = true; return q; }
    // copy-backs + stream sync + arena reset. Returns MO_RC_SUCCESS or MO_RC_INTERNAL_ERROR.
    int finish();
    // the end of a call with an asynchronous form: finish() once a host range was met, else hand the scratch back in stream order and return
    // without synchronising (there is then nothing to copy back and no cache block to keep)
    int complete();
    ~Stager();
private:
    bool host_seen = false;
};

#define MOB_CUDA_TRY(expr)                                                                    \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            mob::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return MO_RC_INTERNAL_ERROR;                                                      \
        }                                                                                     \
    } while (0)

// count + check a kernel launch
#define MOB_LAUNCH_CHECK()                                                                    \
    do {                                                                                      \
        mob::g_launches.fetch_add(1, std::memory_order_relaxed);                              \
        cudaError_t _e = cudaGetLastError();                                                  \
        if (_e != cudaSuccess) {                                                              \
            mob::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
            return MO_RC_INTERNAL_ERROR;                                                      \
        }                                                                                     \
    } while (0)

// read one small device value back through the pinned staging buffer (synchronises the stream)
int read_back(ThreadCtx &t, void *host_dst, const void *dev_src, size_t bytes);

// A parameter block or scalar argument, host or device memory (include/mo_b200.h): copies min(a.dataSz, max) bytes to dst, reading a device
// block back behind the work already on t.stream.  A missing block or one shorter than min bytes fails with "<what> missing".
int read_param(ThreadCtx &t, const mo_xcall_args_t &a, void *dst, size_t min, size_t max, const char *what);
// stores a host value into a word of the caller's, host or device memory (a parameter block's out word, a result computed on the host); a
// device word is written on t.stream and holds the value when this returns

int write_param(ThreadCtx &t, void *dst, const void *src, size_t bytes);

// comparison operators: the op of MO_XCALL_GO_COMPARE(op, T) and the order of the Numeric_Vec* entry points
enum { CMP_EQ = 0, CMP_NE, CMP_GT, CMP_GE, CMP_LT, CMP_LE };

// element width in bytes of a fixed-width MO_T_* type, 0 for any other type
inline int type_size(int T) {
    switch (T) {
    case MO_T_BOOL: case MO_T_INT8: case MO_T_UINT8: return 1;
    case MO_T_INT16: case MO_T_UINT16: return 2;
    case MO_T_INT32: case MO_T_UINT32: case MO_T_FLOAT32: case MO_T_DATE: return 4;
    case MO_T_INT64: case MO_T_UINT64: case MO_T_FLOAT64: case MO_T_TIME: case MO_T_DATETIME: case MO_T_TIMESTAMP: return 8;
    }
    return 0;
}

}  // namespace mob

// =========================================================================================================
// device helpers
// =========================================================================================================
#ifdef __CUDACC__
namespace mob {

// 128-bit streaming loads: read-only path, do not allocate in L1 (each byte is touched once)
__device__ __forceinline__ int4 ld_stream16(const void *p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ int2 ld_stream8(const void *p) {
    int2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
// Two float64 through ld_stream16 under a per-lane predicate: +0.0 where `pred` is false, and no memory access.  One predicated
// instruction, not a lane-dependent branch region (DESIGN 5.1).  Typed .f64: with .s32 outputs ptxas copied every result out of the
// load's destination registers, which waits for the load.
__device__ __forceinline__ double2 ld_stream16_f64_if(bool pred, const double *p) {
    double2 r;
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\tmov.f64 %0, 0d0000000000000000;\n\tmov.f64 %1, 0d0000000000000000;\n\t"
                 "@q ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%3];\n\t}"
                 : "=d"(r.x), "=d"(r.y) : "r"((int)pred), "l"(p));
    return r;
}
// the int64 twin (Decimal64 columns): 0 where `pred` is false
__device__ __forceinline__ longlong2 ld_stream16_s64_if(bool pred, const int64_t *p) {
    longlong2 r;
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\tmov.b64 %0, 0;\n\tmov.b64 %1, 0;\n\t"
                 "@q ld.global.nc.L1::no_allocate.v2.s64 {%0, %1}, [%3];\n\t}"
                 : "=l"(r.x), "=l"(r.y) : "r"((int)pred), "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream16(void *p, int4 v) {
    asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}

__device__ __forceinline__ bool bm_test(const uint64_t *p, uint64_t i) { return p && ((p[i >> 6] >> (i & 63)) & 1ull); }

// total order on non-NaN doubles as unsigned integers, so that MIN / MAX states can use the integer atomics; -0.0 is folded onto +0.0 (they
// compare equal in the reference too)
__device__ __forceinline__ unsigned long long flt_key(double d) {
    if (d == 0.0) d = 0.0;
    unsigned long long b = (unsigned long long)__double_as_longlong(d);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}
__device__ __forceinline__ double flt_unkey(unsigned long long k) {
    const unsigned long long b = (k >> 63) ? (k & ~(1ull << 63)) : ~k;
    return __longlong_as_double((long long)b);
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// fixed-order butterfly: every lane ends with the same value, association independent of data
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = v + __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace mob
#endif
