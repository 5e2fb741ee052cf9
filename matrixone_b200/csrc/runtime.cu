// runtime.cu -- process-wide runtime + per-thread contexts + the MoB200_* residency extension.
//
// Replaces the reference CUDA shim's "global CUcontext at static-init, NULL stream, alloc/copy/free per call"
// (cgo/cuda/cuda.cpp:63-219) with: lazy init, one stream + scratch arena per calling thread, pointer
// classification so resident (device) columns are used in place, and pinned host allocation for the caller.
#include "common.cuh"
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <mutex>
#include <map>
#include <list>
#include <memory>

namespace mob {

std::atomic<uint64_t> g_launches{0};
static std::once_flag g_once;
static int g_device = -1;
static int g_init_rc = MO_RC_INTERNAL_ERROR;
static int g_sms = kSMs;
static char g_init_err[256] = "runtime not initialised";

void set_error(const char *fmt, ...) {
    // the thread context may not exist yet (init failure): keep a thread-local buffer of its own
    static thread_local char buf[256];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    ThreadCtx &t = tctx();
    memcpy(t.err, buf, sizeof buf);
}

int num_sms() { return g_sms; }

int runtime_init(int device) {
    std::call_once(g_once, [device]() {
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        if (e != cudaSuccess || n == 0) {
            snprintf(g_init_err, sizeof g_init_err, "libmo_b200: no CUDA device available (%s); this library has no CPU path",
                     e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
            return;
        }
        int d = device;
        if (d < 0) {
            const char *s = getenv("MO_B200_DEVICE");
            if (!s) s = getenv("LOCAL_RANK");
            d = s ? atoi(s) : 0;
        }
        if (d >= n) d = d % n;
        e = cudaSetDevice(d);
        if (e != cudaSuccess) {
            snprintf(g_init_err, sizeof g_init_err, "cudaSetDevice(%d) failed: %s", d, cudaGetErrorString(e));
            return;
        }
        cudaDeviceProp p;
        if (cudaGetDeviceProperties(&p, d) == cudaSuccess) g_sms = p.multiProcessorCount;
        g_device = d;
        g_init_rc = MO_RC_SUCCESS;
        g_init_err[0] = 0;
    });
    return g_init_rc;
}

ThreadCtx &tctx() {
    static thread_local ThreadCtx t;
    if (!t.ready) {
        if (runtime_init(-1) != MO_RC_SUCCESS) {
            snprintf(t.err, sizeof t.err, "%s", g_init_err);
            return t;
        }
        if (cudaSetDevice(g_device) != cudaSuccess) { snprintf(t.err, sizeof t.err, "cudaSetDevice failed"); return t; }
        if (cudaStreamCreateWithFlags(&t.stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreate(&t.ev0) != cudaSuccess || cudaEventCreate(&t.ev1) != cudaSuccess ||
            cudaEventCreate(&t.kev0) != cudaSuccess || cudaEventCreate(&t.kev1) != cudaSuccess) {
            snprintf(t.err, sizeof t.err, "stream/event creation failed: %s", cudaGetErrorString(cudaGetLastError()));
            return t;
        }
        t.pinned_sz = 1 << 16;
        if (cudaHostAlloc((void **)&t.pinned, t.pinned_sz, cudaHostAllocDefault) != cudaSuccess) {
            snprintf(t.err, sizeof t.err, "pinned staging allocation failed");
            return t;
        }
        if (cudaMalloc((void **)&t.ctrl, 256) != cudaSuccess || cudaMemset(t.ctrl, 0, 256) != cudaSuccess) {
            snprintf(t.err, sizeof t.err, "control block allocation failed");
            return t;
        }
        t.own_stream = true;
        t.ready = true;
    }
    return t;
}

bool is_device_ptr(const void *p) {
    if (!p) return false;
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

void *arena_alloc(ThreadCtx &t, size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    if (bytes == 0) bytes = 256;
    while (t.cur_block < t.blocks.size()) {
        ArenaBlock &b = t.blocks[t.cur_block];
        if (t.cur_off + bytes <= b.size) { void *p = b.p + t.cur_off; t.cur_off += bytes; return p; }
        t.cur_block++; t.cur_off = 0;
    }
    size_t sz = bytes > (size_t)(64u << 20) ? bytes : (size_t)(64u << 20);
    char *p = nullptr;
    cudaError_t e = cudaMalloc((void **)&p, sz);
    if (e != cudaSuccess) { set_error("device scratch allocation of %zu bytes failed: %s", sz, cudaGetErrorString(e)); return nullptr; }
    t.blocks.push_back({p, sz});
    t.cur_block = t.blocks.size() - 1;
    t.cur_off = bytes;
    return p;
}

void arena_reset(ThreadCtx &t) {
    // consolidate a fragmented arena into one block so the steady state is a single bump allocator
    if (t.blocks.size() > 1) {
        size_t total = 0;
        for (auto &b : t.blocks) { total += b.size; cudaFree(b.p); }
        t.blocks.clear();
        char *p = nullptr;
        if (cudaMalloc((void **)&p, total) == cudaSuccess) t.blocks.push_back({p, total});
        else cudaGetLastError();
    }
    t.cur_block = 0; t.cur_off = 0; t.arena_epoch++; t.kev_prio = 0;
}

// ---- device column cache ----------------------------------------------------------------------------------------------------------
// SURVEY.md section 7 step 1: the ABI hands the library HOST vectors, and re-uploading a column on every call makes everything PCIe-bound
// (the reference's CUDA shim has exactly this flaw, cgo/cuda/cuda.cpp:123-201).  A caller that knows a host range is immutable -- a decoded
// block's column, an index's dataset -- declares it once with MoB200_ColumnPin(host, bytes, generation); from then on every entry point
// that is handed a pointer inside that range uses the device copy instead of staging it.  Explicit opt-in, because the library cannot know
// when the Go side recycles a buffer: a new generation or MoB200_ColumnUnpin drops the copy.  LRU eviction beyond the configured capacity.
struct DevBlock {
    void *d = nullptr; size_t bytes = 0; uint64_t gen = 0;
    ~DevBlock() { if (d) cudaFree(d); }
};
static std::mutex g_cache_mu;
static std::map<uintptr_t, std::shared_ptr<DevBlock>> g_cache;   // keyed by host base address
static std::list<uintptr_t> g_cache_lru;                            // front = most recently used
static size_t g_cache_bytes = 0, g_cache_cap = 0;
static std::atomic<uint64_t> g_cache_hits{0}, g_cache_misses{0};

// device pointer for [p, p + bytes) if a pinned block covers it; `keep` holds the block alive for the caller's lifetime
static const void *cache_lookup(const void *p, size_t bytes, std::shared_ptr<DevBlock> &keep) {
    if (g_cache_cap == 0) return nullptr;
    std::lock_guard<std::mutex> lk(g_cache_mu);
    const uintptr_t a = (uintptr_t)p;
    auto it = g_cache.upper_bound(a);
    if (it == g_cache.begin()) { g_cache_misses++; return nullptr; }
    --it;
    if (a + bytes > it->first + it->second->bytes) { g_cache_misses++; return nullptr; }
    keep = it->second;
    g_cache_lru.remove(it->first); g_cache_lru.push_front(it->first);
    g_cache_hits++;
    return (const char *)it->second->d + (a - it->first);
}

const void *Stager::in(const void *p, size_t bytes) {
    if (!p || bytes == 0) return p;
    if (is_device_ptr(p)) return p;
    host_seen = true;
    {
        std::shared_ptr<DevBlock> keep;
        const void *c = cache_lookup(p, bytes, keep);
        if (c) { pins.push_back(std::static_pointer_cast<void>(keep)); return c; }
    }
    void *d = arena_alloc(t, bytes);
    if (!d) { failed = true; return nullptr; }
    cudaError_t e = cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, t.stream);
    if (e != cudaSuccess) { set_error("H2D copy of %zu bytes failed: %s", bytes, cudaGetErrorString(e)); failed = true; return nullptr; }
    return d;
}

void *Stager::out(void *p, size_t bytes, bool preload) {
    if (!p || bytes == 0) return p;
    if (is_device_ptr(p)) return p;
    host_seen = true;
    void *d = arena_alloc(t, bytes);
    if (!d) { failed = true; return nullptr; }
    if (preload) {
        cudaError_t e = cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, t.stream);
        if (e != cudaSuccess) { set_error("H2D preload failed: %s", cudaGetErrorString(e)); failed = true; return nullptr; }
    }
    backs.push_back({p, d, bytes});
    return d;
}

int Stager::finish() {
    int rc = failed ? MO_RC_INTERNAL_ERROR : MO_RC_SUCCESS;
    // outputs that fit go through the pinned staging buffer: a copy into pageable memory waits for the stream by itself, and a call with
    // a few small results (an aggregate's words and nulls word) would pay that wait once per result
    size_t pinned_used = 0;
    std::vector<size_t> at(backs.size(), SIZE_MAX);
    if (!failed) {
        for (size_t i = 0; i < backs.size(); i++) {
            const Back &b = backs[i];
            if (pinned_used + b.bytes <= t.pinned_sz) { at[i] = pinned_used; pinned_used += b.bytes; }
            cudaError_t e = cudaMemcpyAsync(at[i] == SIZE_MAX ? b.host : t.pinned + at[i], b.dev, b.bytes, cudaMemcpyDeviceToHost, t.stream);
            if (e != cudaSuccess) { set_error("D2H copy failed: %s", cudaGetErrorString(e)); rc = MO_RC_INTERNAL_ERROR; break; }
        }
    }
    cudaError_t e = cudaStreamSynchronize(t.stream);
    if (e != cudaSuccess) { set_error("stream synchronize failed: %s", cudaGetErrorString(e)); rc = MO_RC_INTERNAL_ERROR; }
    if (rc == MO_RC_SUCCESS)
        for (size_t i = 0; i < backs.size(); i++) if (at[i] != SIZE_MAX) memcpy(backs[i].host, t.pinned + at[i], backs[i].bytes);
    backs.clear();
    pins.clear();   // the stream is idle: cached blocks may be evicted now
    arena_reset(t);
    finished = true;
    return rc;
}

int Stager::complete() {
    if (failed || host_seen) return finish();
    arena_reset(t);
    finished = true;
    return MO_RC_SUCCESS;
}

Stager::~Stager() {
    // an early return between construction and finish() (MOB_CUDA_TRY / MOB_LAUNCH_CHECK): wait for whatever was enqueued on the scratch and
    // give it back, so the arena does not grow and per-call caches keyed on the arena epoch are invalidated (ADVICE r01)
    if (!finished) { cudaStreamSynchronize(t.stream); backs.clear(); pins.clear(); arena_reset(t); }
}

int read_back(ThreadCtx &t, void *host_dst, const void *dev_src, size_t bytes) {
    if (bytes > t.pinned_sz) { set_error("read_back too large"); return MO_RC_INTERNAL_ERROR; }
    MOB_CUDA_TRY(cudaMemcpyAsync(t.pinned, dev_src, bytes, cudaMemcpyDeviceToHost, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    memcpy(host_dst, t.pinned, bytes);
    return MO_RC_SUCCESS;
}

int read_param(ThreadCtx &t, const mo_xcall_args_t &a, void *dst, size_t min, size_t max, const char *what) {
    if (!a.pdata || a.dataSz < min) { set_error("%s missing", what); return MO_RC_INVALID_ARGUMENT; }
    const size_t bytes = a.dataSz < max ? (size_t)a.dataSz : max;
    if (is_device_ptr(a.pdata)) return read_back(t, dst, a.pdata, bytes);
    memcpy(dst, a.pdata, bytes);
    return MO_RC_SUCCESS;
}

int write_param(ThreadCtx &t, void *dst, const void *src, size_t bytes) {
    if (!is_device_ptr(dst)) { memcpy(dst, src, bytes); return MO_RC_SUCCESS; }
    MOB_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    return MO_RC_SUCCESS;
}

}  // namespace mob

using namespace mob;

#define REQUIRE_CTX(t)                               \
    ThreadCtx &t = tctx();                           \
    if (!t.ready) return MO_RC_INTERNAL_ERROR

__global__ void flush_l2_kernel(int4 *p, size_t n16) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n16; i += stride) p[i] = make_int4((int)i, 0, 0, 0);
}

extern "C" {

int32_t MoB200_Init(int32_t device) {
    int rc = runtime_init(device);
    if (rc != MO_RC_SUCCESS) return rc;
    REQUIRE_CTX(t);
    return MO_RC_SUCCESS;
}

const char *MoB200_Version(void) { return "mo_b200 0.1 (sm_90a)"; }

int32_t MoB200_DeviceCount(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int32_t MoB200_DeviceAlloc(uint64_t bytes, void **dptr) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaMalloc(dptr, bytes ? bytes : 1));
    return MO_RC_SUCCESS;
}
int32_t MoB200_DeviceFree(void *dptr) {
    REQUIRE_CTX(t);
    MoB200_SearchRelease(dptr);   // a prepared search operand of (or built against) this buffer must not outlive it
    MOB_CUDA_TRY(cudaFree(dptr));
    return MO_RC_SUCCESS;
}
int32_t MoB200_HostAlloc(uint64_t bytes, void **hptr) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaHostAlloc(hptr, bytes ? bytes : 1, cudaHostAllocDefault));
    return MO_RC_SUCCESS;
}
int32_t MoB200_HostFree(void *hptr) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaFreeHost(hptr));
    return MO_RC_SUCCESS;
}
int32_t MoB200_HostRegister(void *hptr, uint64_t bytes) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaHostRegister(hptr, bytes, cudaHostRegisterDefault));
    return MO_RC_SUCCESS;
}
int32_t MoB200_HostUnregister(void *hptr) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaHostUnregister(hptr));
    return MO_RC_SUCCESS;
}
int32_t MoB200_Upload(void *dst_dev, const void *src_host, uint64_t bytes) {
    REQUIRE_CTX(t);
    search_invalidate(dst_dev, bytes);
    MOB_CUDA_TRY(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    return MO_RC_SUCCESS;
}
int32_t MoB200_Download(void *dst_host, const void *src_dev, uint64_t bytes) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    return MO_RC_SUCCESS;
}
// stream-ordered copies without a synchronise: the host buffer should be pinned (MoB200_HostAlloc / HostRegister) and must not be
// read (download) or reused (upload) before MoB200_Sync
int32_t MoB200_DownloadAsync(void *dst_host, const void *src_dev, uint64_t bytes) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, t.stream));
    return MO_RC_SUCCESS;
}
int32_t MoB200_UploadAsync(void *dst_dev, const void *src_host, uint64_t bytes) {
    REQUIRE_CTX(t);
    search_invalidate(dst_dev, bytes);
    MOB_CUDA_TRY(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, t.stream));
    return MO_RC_SUCCESS;
}
int32_t MoB200_ColumnCacheConfigure(uint64_t capacity_bytes) {
    REQUIRE_CTX(t);
    std::lock_guard<std::mutex> lk(g_cache_mu);
    g_cache_cap = (size_t)capacity_bytes;
    while (g_cache_bytes > g_cache_cap && !g_cache_lru.empty()) {
        const uintptr_t k = g_cache_lru.back(); g_cache_lru.pop_back();
        auto it = g_cache.find(k);
        if (it != g_cache.end()) { g_cache_bytes -= it->second->bytes; g_cache.erase(it); }
    }
    return MO_RC_SUCCESS;
}
int32_t MoB200_ColumnPin(const void *host, uint64_t bytes, uint64_t generation) {
    REQUIRE_CTX(t);
    if (!host || bytes == 0) return MO_RC_SUCCESS;
    if (is_device_ptr(host)) { set_error("ColumnPin: host pointer expected"); return MO_RC_INVALID_ARGUMENT; }
    {
        std::lock_guard<std::mutex> lk(g_cache_mu);
        if (g_cache_cap == 0 || bytes > g_cache_cap) return MO_RC_SUCCESS;     // cache off / column larger than the cache: calls keep staging it
        auto it = g_cache.find((uintptr_t)host);
        if (it != g_cache.end()) {
            if (it->second->gen == generation && it->second->bytes >= bytes) { g_cache_lru.remove(it->first); g_cache_lru.push_front(it->first); return MO_RC_SUCCESS; }
            g_cache_bytes -= it->second->bytes; g_cache_lru.remove(it->first); g_cache.erase(it);   // a new generation of the same buffer
        }
    }
    auto blk = std::make_shared<DevBlock>();
    MOB_CUDA_TRY(cudaMalloc(&blk->d, bytes));
    blk->bytes = bytes; blk->gen = generation;
    MOB_CUDA_TRY(cudaMemcpyAsync(blk->d, host, bytes, cudaMemcpyHostToDevice, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    std::lock_guard<std::mutex> lk(g_cache_mu);
    // overlapping older entries would shadow / be shadowed by this one: drop them
    for (auto it = g_cache.begin(); it != g_cache.end();) {
        if (it->first < (uintptr_t)host + bytes && (uintptr_t)host < it->first + it->second->bytes) { g_cache_bytes -= it->second->bytes; g_cache_lru.remove(it->first); it = g_cache.erase(it); }
        else ++it;
    }
    g_cache[(uintptr_t)host] = blk; g_cache_lru.push_front((uintptr_t)host); g_cache_bytes += bytes;
    while (g_cache_bytes > g_cache_cap && g_cache_lru.size() > 1) {
        const uintptr_t k = g_cache_lru.back(); g_cache_lru.pop_back();
        auto it = g_cache.find(k);
        if (it != g_cache.end()) { g_cache_bytes -= it->second->bytes; g_cache.erase(it); }   // in-flight calls hold their own reference
    }
    return MO_RC_SUCCESS;
}
int32_t MoB200_ColumnUnpin(const void *host) {
    REQUIRE_CTX(t);
    std::lock_guard<std::mutex> lk(g_cache_mu);
    auto it = g_cache.find((uintptr_t)host);
    if (it != g_cache.end()) { g_cache_bytes -= it->second->bytes; g_cache_lru.remove(it->first); g_cache.erase(it); }
    return MO_RC_SUCCESS;
}
int32_t MoB200_ColumnCacheStats(uint64_t *hits, uint64_t *misses, uint64_t *bytes) {
    if (hits) *hits = g_cache_hits.load();
    if (misses) *misses = g_cache_misses.load();
    std::lock_guard<std::mutex> lk(g_cache_mu);
    if (bytes) *bytes = g_cache_bytes;
    return MO_RC_SUCCESS;
}
int32_t MoB200_Memset(void *dst_dev, int32_t value, uint64_t bytes) {
    REQUIRE_CTX(t);
    search_invalidate(dst_dev, bytes);
    MOB_CUDA_TRY(cudaMemsetAsync(dst_dev, value, bytes, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    return MO_RC_SUCCESS;
}
int32_t MoB200_Sync(void) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    return MO_RC_SUCCESS;
}
int32_t MoB200_SetStream(void *cuda_stream) {
    REQUIRE_CTX(t);
    static thread_local cudaStream_t own = nullptr;
    if (t.own_stream) own = t.stream;
    if (cuda_stream) { t.stream = (cudaStream_t)cuda_stream; t.own_stream = false; }
    else { t.stream = own; t.own_stream = true; }
    return MO_RC_SUCCESS;
}
int32_t MoB200_TimerStart(void) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaEventRecord(t.ev0, t.stream));
    return MO_RC_SUCCESS;
}
int32_t MoB200_TimerStop(float *ms) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaEventRecord(t.ev1, t.stream));
    MOB_CUDA_TRY(cudaEventSynchronize(t.ev1));
    MOB_CUDA_TRY(cudaEventElapsedTime(ms, t.ev0, t.ev1));
    return MO_RC_SUCCESS;
}
uint64_t MoB200_KernelLaunchCount(void) { return g_launches.load(); }

int32_t MoB200_LastKernelMs(float *ms) {
    REQUIRE_CTX(t);
    MOB_CUDA_TRY(cudaEventSynchronize(t.kev1));
    MOB_CUDA_TRY(cudaEventElapsedTime(ms, t.kev0, t.kev1));
    return MO_RC_SUCCESS;
}

int32_t MoB200_LastError(char *buf, uint64_t buflen) {
    ThreadCtx &t = tctx();
    if (buf && buflen) { snprintf(buf, buflen, "%s", t.err); }
    return (int32_t)strlen(t.err);
}

int32_t MoB200_FlushL2(void) {
    REQUIRE_CTX(t);
    static thread_local void *buf = nullptr;
    const size_t bytes = (size_t)256 << 20;  // 5x the 50 MB L2
    if (!buf) MOB_CUDA_TRY(cudaMalloc(&buf, bytes));
    flush_l2_kernel<<<num_sms() * 4, 256, 0, t.stream>>>((int4 *)buf, bytes / 16);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

}  // extern "C"
