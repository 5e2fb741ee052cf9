// join.cu -- the data-parallel pieces of the reference's hash join (pkg/sql/colexec/hashbuild/hashmap.go:237-488, pkg/vm/message/joinMapMsg.go:32-132,
// pkg/sql/colexec/hashjoin/join.go:383-628) behind XCall, over the <= 8-byte packed keys of MO_XCALL_PACK_KEYS and the group ids of MO_XCALL_GROUP_IDS.
//
//   build side   GROUP_IDS over the build keys (IntHashMap insert, first-seen ids) gives vals[i]; JOIN_SELS turns them into the JoinMap's GroupSels:
//                offsets int32[groupCount + 2], vals int32[n] -- rows of group k (0-based) at vals[offsets[k] .. offsets[k + 1]), ASCENDING row ids,
//                exactly what GroupSels.Insert + Finalize (joinMapMsg.go:72-125: count, prefix sum, stable scatter) leave behind.
//                Here: order-preserving compaction of the rows with an id, then the stable radix sort of order.cu by group id (sort_u32_pairs),
//                offsets from a histogram + exclusive scan.
//   lookup       JOIN_FIND = intHashMapIterator.Find (vals[i] = group id or 0; a NULL key never matches, zvals == 0); STR_JOIN_FIND =
//                strHashmapIterator.Find over a STR_GROUP_IDS table (keytable.cuh's byte-string slots).  One builder makes both kinds of table.
//   result       JOIN_PROBE, JOIN_PROBE_GIDS and JOIN_COND are one pipeline, the emission loop of container.probe (join.go:450-611) for every
//                join type: a first pass gives each probe row its matches and, by one type rule, its result rows; an exclusive scan turns the
//                counts into positions; one emit pass writes the pairs (probe row, build row | -1) in exactly the order the reference appends
//                them, probe rows ascending, within a row the build rows in order.  Only the row source of the emit pass differs:
//                  JOIN_PROBE      the group of the probe row's key (JOIN_PROBE_GIDS: the group id JOIN_FIND or STR_JOIN_FIND returned) and its
//                                  sels (unique maps: build row = id - 1), every build row a match;
//                  JOIN_COND       the probe row's INNER candidate pairs (join.go:468-498,570-611), a match where the caller's non-equality
//                                  condition passes.
//                Right-flavoured types mark the build side's matched-row bitmap; LEFT SINGLE and RIGHT SINGLE check the single-row rule.
//   JOIN_MATCHED_MERGE = syncBitmap's OR over the workers' bitmaps (join.go:650-676); JOIN_BUILD_ROWS (colops.cu) = finalize's row list.
//   The hash table itself is not observable in the reference (random seeds): ids and pairs are.  The device table is rebuilt from table_keys per
//   call (O(groups)) unless it was prepared with MoB200_JoinMapPrepare (cached per table_keys pointer).
// All passes stream their inputs once; algorithmic bytes per probe row: 8 (key) + 16 per emitted pair + one random 8-byte table probe.
#include "common.cuh"
#include "keytable.cuh"
#include <cstring>
#include <mutex>
#include <shared_mutex>
#include <unordered_map>

namespace mob {

int sort_u32_pairs(ThreadCtx &t, uint32_t *k0, uint32_t *v0, uint32_t *k1, uint32_t *v1, const uint64_t *m_ptr, uint64_t cap);   // order.cu

namespace {

constexpr int kThreads = 256;

inline unsigned grid_for(uint64_t items) {
    uint64_t g = (items + kThreads - 1) / kThreads;
    const uint64_t mx = (uint64_t)num_sms() * 16;
    return (unsigned)(g > mx ? mx : (g ? g : 1));
}

// ---- exclusive scan of uint64 (three kernels: tile sums, scan of the sums by one CTA, apply) ---------------------------------------------------
constexpr int kScanTile = 2048;   // 256 threads x 8
__global__ void __launch_bounds__(kThreads) scan_sums_kernel(const uint64_t *__restrict__ in, uint64_t n, uint64_t *__restrict__ sums) {
    __shared__ uint64_t sw[kThreads / 32];
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile;
    uint64_t s = 0;
    for (int j = 0; j < 8; j++) { const uint64_t i = base + (uint64_t)j * kThreads + threadIdx.x; if (i < n) s += in[i]; }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) { uint64_t t = 0; for (int w = 0; w < kThreads / 32; w++) t += sw[w]; sums[blockIdx.x] = t; }
}
__global__ void __launch_bounds__(1024) scan_of_sums_kernel(uint64_t *sums, uint64_t nb, uint64_t *total) {
    __shared__ uint64_t sw[32];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint64_t b0 = 0; b0 < nb; b0 += 1024) {
        const uint64_t i = b0 + threadIdx.x;
        const uint64_t v = i < nb ? sums[i] : 0;
        uint64_t inc = v;
        for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) sw[warp] = inc;
        __syncthreads();
        uint64_t wbase = 0;
        for (int w = 0; w < warp; w++) wbase += sw[w];
        const uint64_t c = carry;
        if (i < nb) sums[i] = c + wbase + inc - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + wbase + inc;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}
__global__ void __launch_bounds__(kThreads) scan_apply_kernel(const uint64_t *__restrict__ in, uint64_t n, const uint64_t *__restrict__ sums, uint64_t *__restrict__ out) {
    // tile layout for the apply pass: thread t owns 8 CONSECUTIVE items, so its exclusive prefix is a register scan
    __shared__ uint64_t sw[kThreads / 32];
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * 8;
    uint64_t v[8], s = 0;
    for (int j = 0; j < 8; j++) { v[j] = base + j < n ? in[base + j] : 0; s += v[j]; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t inc = s;
    for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) sw[warp] = inc;
    __syncthreads();
    uint64_t run = sums[blockIdx.x] + inc - s;
    for (int w = 0; w < warp; w++) run += sw[w];
    for (int j = 0; j < 8; j++) { if (base + j < n) out[base + j] = run; run += v[j]; }
}
}  // namespace

// out[i] = sum of in[0 .. i); *total (device) = sum of all.  in == out allowed.  sums scratch from the arena.  Also used by colops.cu.
int exclusive_scan(ThreadCtx &t, const uint64_t *in, uint64_t n, uint64_t *out, uint64_t *total) {
    if (n == 0) { MOB_CUDA_TRY(cudaMemsetAsync(total, 0, 8, t.stream)); return MO_RC_SUCCESS; }
    const uint64_t nb = (n + kScanTile - 1) / kScanTile;
    uint64_t *sums = (uint64_t *)arena_alloc(t, nb * 8);
    if (!sums) return MO_RC_INTERNAL_ERROR;
    scan_sums_kernel<<<(unsigned)nb, kThreads, 0, t.stream>>>(in, n, sums);
    MOB_LAUNCH_CHECK();
    scan_of_sums_kernel<<<1, 1024, 0, t.stream>>>(sums, nb, total);
    MOB_LAUNCH_CHECK();
    scan_apply_kernel<<<(unsigned)nb, kThreads, 0, t.stream>>>(in, n, sums, out);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

// the join type of a join entry point (what): any type, or (right_only) a right-flavoured one, whose matched bitmap JOIN_MATCHED_MERGE and
// JOIN_BUILD_ROWS (colops.cu) read
int check_join_type(int join_type, const char *what, bool right_only) {
    if (join_type < (right_only ? MO_JOIN_RIGHT : MO_JOIN_INNER) || join_type > MO_JOIN_RIGHT_SINGLE) {
        set_error(right_only ? "%s: join type %d (a right-flavoured type, 5..9)" : "%s: join type %d", what, join_type);
        return MO_RC_INVALID_ARGUMENT;
    }
    return MO_RC_SUCCESS;
}

namespace {

// ---- JOIN_SELS ------------------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) sels_flag_kernel(const uint64_t *__restrict__ groups, uint64_t n, uint64_t ngroups, uint64_t *__restrict__ flag, uint64_t *__restrict__ cnt, unsigned *bad) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        const uint64_t g = groups[i];
        if (g > ngroups) { *bad = 1; flag[i] = 0; continue; }
        flag[i] = g ? 1 : 0;
        if (g) atomicAdd((unsigned long long *)&cnt[g - 1], 1ull);
    }
}
__global__ void __launch_bounds__(kThreads) sels_compact_kernel(const uint64_t *__restrict__ groups, const uint64_t *__restrict__ pos, uint64_t n, uint64_t ngroups, uint32_t *__restrict__ key, uint32_t *__restrict__ row) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        const uint64_t g = groups[i];
        if (g && g <= ngroups) { key[pos[i]] = (uint32_t)(g - 1); row[pos[i]] = (uint32_t)i; }
    }
}
__global__ void __launch_bounds__(kThreads) sels_offsets_kernel(const uint64_t *__restrict__ starts, uint64_t ngroups, const uint64_t *__restrict__ total, int32_t *__restrict__ offsets) {
    // offsets has ngroups + 2 entries: [k] = start of group k, [ngroups] = [ngroups + 1] = n (joinMapMsg.go:89-121)
    for (uint64_t k = blockIdx.x * (uint64_t)kThreads + threadIdx.x; k < ngroups + 2; k += (uint64_t)gridDim.x * kThreads)
        offsets[k] = (int32_t)(k < ngroups ? starts[k] : *total);
}
__global__ void __launch_bounds__(kThreads) copy_rows_kernel(const uint32_t *__restrict__ row, const uint64_t *__restrict__ m_ptr, int32_t *__restrict__ vals, int64_t *count_out) {
    const uint64_t m = *m_ptr;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < m; i += (uint64_t)gridDim.x * kThreads) vals[i] = (int32_t)row[i];
    if (blockIdx.x == 0 && threadIdx.x == 0) *count_out = (int64_t)m;
}

// ---- the probe-side hash table: a keytable.cuh table, key[slots + 1] and id[slots + 1] (the id of the all-ones key, or 0, in id[slots]) -----------
__global__ void __launch_bounds__(kThreads) jt_build_kernel(const uint64_t *__restrict__ table_keys, uint64_t ngroups, uint64_t *key, uint32_t *id, uint64_t mask) {
    for (uint64_t g = blockIdx.x * (uint64_t)kThreads + threadIdx.x; g < ngroups; g += (uint64_t)gridDim.x * kThreads) {
        // the table is at most half full, so a slot is always found; table_keys are distinct: one writer per slot
        uint64_t s;
        kt_insert(key, mask, table_keys[g], s);
        id[s] = (uint32_t)(g + 1);
    }
}
// the group id of probe row i looked up by its key, 0 for a NULL or absent key (JOIN_FIND, JOIN_PROBE)
struct KeyLookup {
    const uint64_t *__restrict__ keys; const uint64_t *__restrict__ knulls; const uint64_t *__restrict__ tkey; const uint32_t *__restrict__ tid; uint64_t mask;
    __device__ __forceinline__ uint32_t operator()(uint64_t i) const {
        uint64_t s;
        return !bm_test(knulls, i) && kt_find(tkey, mask, keys[i], s) ? tid[s] : 0u;
    }
};
__global__ void __launch_bounds__(kThreads) jt_find_kernel(KeyLookup lookup, uint64_t n, uint64_t *__restrict__ vals) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) vals[i] = lookup(i);
}

// ---- the string twin (STR_JOIN_FIND): keytable.cuh's byte-string slots over the table's bytes; slot row g is group g + 1 -------------------
__global__ void __launch_bounds__(kThreads) sjt_build_kernel(StrKeys K, uint64_t ngroups, uint64_t *slots, uint64_t mask, uint64_t hash_mask) {
    for (uint64_t g = blockIdx.x * (uint64_t)kThreads + threadIdx.x; g < ngroups; g += (uint64_t)gridDim.x * kThreads) {
        // the groups' keys are distinct and the table at most half full: every group claims the first empty slot of its probe
        const uint64_t h = str_hash(K.at(g), hash_mask);
        kt_insert_str(slots, mask, h, str_word(h, g), [](uint32_t) { return false; });
    }
}
__global__ void __launch_bounds__(kThreads) sjt_find_kernel(StrKeys K, const uint64_t *__restrict__ knulls, uint64_t n, const uint64_t *__restrict__ slots,
                                                            uint64_t mask, uint64_t hash_mask, uint64_t *__restrict__ vals) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        uint64_t v = 0;
        if (!bm_test(knulls, i)) {
            const ByteKey k = K.at(K.nexist + i);
            uint32_t row;
            if (kt_find_str(slots, mask, str_hash(k, hash_mask), [&](uint32_t r) { return bytes_equal(K.at(r), k); }, row)) v = (uint64_t)row + 1;
        }
        vals[i] = v;
    }
}

// a device join table: the 8-byte one (key, id), or a string one (key = its slots; sbytes / soff = the table's bytes and offsets)
struct DevTable { uint64_t *key = nullptr; uint32_t *id = nullptr; uint64_t mask = 0; uint64_t ngroups = 0; bool cached = false;
                  bool str = false; const uint8_t *sbytes = nullptr; const uint64_t *soff = nullptr; };
std::shared_mutex g_jm_mu;
std::unordered_map<const void *, DevTable> g_jm;   // prepared join maps, by table_keys pointer (string maps: by table offsets pointer)

void free_table(DevTable &T) {
    cudaFree(T.key); cudaFree(T.id);
    cudaFree((void *)T.sbytes); cudaFree((void *)T.soff);
}

// the table of groups 1..ngroups, over the 8-byte keys dkeys or, when soff is given, over the byte strings sbytes / soff, all on the device; at
// most half full.  The kind follows soff, never null for a string table (ngroups + 1 offsets); dkeys of an empty 8-byte table may be null.
// persistent: key / id from cudaMalloc (a string table's bytes and offsets stay the caller's), else from the call's arena.
int build_table(ThreadCtx &t, uint64_t ngroups, const uint64_t *dkeys, const uint8_t *sbytes, const uint64_t *soff, bool persistent, DevTable *out) {
    uint64_t slots = 64;
    while (slots < 2 * ngroups) slots <<= 1;
    DevTable T;
    T.mask = slots - 1; T.ngroups = ngroups; T.cached = persistent; T.str = soff != nullptr; T.sbytes = sbytes; T.soff = soff;
    const uint64_t nkey = T.str ? slots : slots + 1, nid = T.str ? 0 : slots + 1;   // the 8-byte table: the all-ones key in key / id[slots]
    if (persistent) {
        if (cudaMalloc(&T.key, nkey * 8) != cudaSuccess || (nid && cudaMalloc(&T.id, nid * 4) != cudaSuccess)) {
            set_error("join map: cudaMalloc of a %llu-slot table failed", (unsigned long long)slots);
            cudaFree(T.key);
            return MO_RC_INTERNAL_ERROR;
        }
    } else {
        T.key = (uint64_t *)arena_alloc(t, nkey * 8);
        T.id = nid ? (uint32_t *)arena_alloc(t, nid * 4) : nullptr;
        if (!T.key || (nid && !T.id)) return MO_RC_INTERNAL_ERROR;
    }
    cudaError_t e = cudaMemsetAsync(T.key, 0xff, nkey * 8, t.stream);   // every slot empty
    if (e == cudaSuccess && nid) e = cudaMemsetAsync(T.id, 0, nid * 4, t.stream);
    if (e != cudaSuccess) {
        set_error("join map: clearing a %llu-slot table failed: %s", (unsigned long long)slots, cudaGetErrorString(e));
        if (persistent) { cudaFree(T.key); cudaFree(T.id); }
        return MO_RC_INTERNAL_ERROR;
    }
    if (ngroups) {
        if (T.str) sjt_build_kernel<<<grid_for(ngroups), kThreads, 0, t.stream>>>(StrKeys{sbytes, soff, nullptr, nullptr, ngroups}, ngroups, T.key, T.mask, strkey_hash_mask());
        else jt_build_kernel<<<grid_for(ngroups), kThreads, 0, t.stream>>>(dkeys, ngroups, T.key, T.id, T.mask);
        MOB_LAUNCH_CHECK();
    }
    *out = T;
    return MO_RC_SUCCESS;
}

// the table prepared under key (table_keys, or a string map's offsets pointer) for ngroups groups: true, with lk holding g_jm_mu shared for as long
// as the caller reads the table, or false with lk released
bool find_prepared(const void *key, uint64_t ngroups, bool str, DevTable *T, std::shared_lock<std::shared_mutex> &lk) {
    lk = std::shared_lock<std::shared_mutex>(g_jm_mu);
    auto it = g_jm.find(key);
    if (it != g_jm.end() && it->second.ngroups == ngroups && it->second.str == str) { *T = it->second; return true; }
    lk.unlock();
    return false;
}

// makes T the table prepared under key, releasing the one it replaces
void publish_prepared(const void *key, const DevTable &T) {
    std::unique_lock<std::shared_mutex> lk(g_jm_mu);
    auto it = g_jm.find(key);
    if (it != g_jm.end()) free_table(it->second);
    g_jm[key] = T;
}

// the table for this call: the prepared one (by the caller's table_keys pointer) or a scratch one in the arena
int table_for(ThreadCtx &t, Stager &st, const mo_xcall_args_t &a, DevTable *T, std::shared_lock<std::shared_mutex> &lk) {
    const uint64_t ngroups = a.dataSz / 8;
    if (find_prepared(a.pdata, ngroups, false, T, lk)) return MO_RC_SUCCESS;
    const uint64_t *dkeys = (const uint64_t *)st.in(a.pdata, ngroups * 8);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    return build_table(t, ngroups, dkeys, nullptr, nullptr, false, T);
}

// the prepared string table keyed by the table offsets pointer, or a scratch one
int str_table_for(ThreadCtx &t, Stager &st, const mo_xcall_args_t &bytes, const mo_xcall_args_t &offs, uint64_t ngroups, DevTable *T,
                  std::shared_lock<std::shared_mutex> &lk) {
    if (find_prepared(offs.pdata, ngroups, true, T, lk)) {
        // nothing is staged, but a table prepared from host memory keeps the call synchronous, as a staged one does
        st.device(bytes.pdata); st.device(offs.pdata);
        return MO_RC_SUCCESS;
    }
    const uint8_t *db = (const uint8_t *)st.in(bytes.pdata, bytes.dataSz);
    const uint64_t *doff = (const uint64_t *)st.in(offs.pdata, (ngroups + 1) * 8);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    return build_table(t, ngroups, nullptr, db, doff, false, T);
}

// ---- JOIN_PROBE / JOIN_PROBE_GIDS ---------------------------------------------------------------------------------------------------------------
// the group id of probe row i: KeyLookup (JOIN_PROBE), or given (JOIN_PROBE_GIDS); an id above ngroups sets *bad
struct GidLookup {
    const uint64_t *__restrict__ gids; uint64_t ngroups; unsigned *bad;
    __device__ __forceinline__ uint32_t operator()(uint64_t i) const {
        const uint64_t g = gids[i];
        if (g > ngroups) { *bad = 1; return 0u; }
        return (uint32_t)g;
    }
};

// ---- the build side's matched-row bitmap (rightRowsMatched, join.go:461-467,539-547) ------------------------------------------------------------
// One bit per build row, LSB-first uint64 words, set with atomicOr.  RIGHT SINGLE looks at the bit it replaces: a build row whose bit was already
// set is matched a second time, whichever pass or batch set it first, so the lowest such row of a call does not depend on the probe order.  A row
// at or past the bitmap's last bit is not marked; the lowest one is recorded and fails the call.  A recorded row is kept as ~row with atomicMax,
// so 0 means none and the whole record starts as zeros (one memset).
struct Marks {
    unsigned long long *words = nullptr; uint64_t nbits = 0; bool single = false;
    unsigned long long *twice = nullptr, *past = nullptr;    // ~(lowest build row) matched twice (RIGHT SINGLE) / lying past the bitmap
    __device__ __forceinline__ void mark(uint64_t r) const {
        if (r >= nbits) { atomicMax(past, ~(unsigned long long)r); return; }
        const unsigned long long bit = 1ull << (r & 63);
        if (single) { if (atomicOr(&words[r >> 6], bit) & bit) atomicMax(twice, ~(unsigned long long)r); }
        else if (!(words[r >> 6] & bit)) atomicOr(&words[r >> 6], bit);   // bits only ever go from 0 to 1: a set bit needs no atomic
    }
};
// the record a join call reads back in one copy: [0] result count, [1] a group id above ngroups (JOIN_COND: ~(lowest malformed candidate)), [2]
// ~(lowest LEFT SINGLE probe row with more than one match), [3] ~(lowest build row matched twice), [4] ~(lowest build row past the bitmap); 0 = none
constexpr int kRecWords = 5;

// the result rows of probe row i with m matches (JOIN_COND: passing pairs) for the join type; LEFT SINGLE records a row with more than one
// (join.go:504-507,587-589).  RIGHT SEMI and RIGHT ANTI emit nothing: they only mark (join.go:452,549).
__device__ __forceinline__ uint64_t result_rows(int join_type, uint64_t m, uint64_t i, unsigned long long *single_row) {
    switch (join_type) {
    case MO_JOIN_INNER: case MO_JOIN_RIGHT: case MO_JOIN_RIGHT_SINGLE: return m;
    case MO_JOIN_LEFT: case MO_JOIN_FULL: return m ? m : 1;           // EmitUnmatchedProbe: one row with the build side NULL
    case MO_JOIN_SINGLE: if (m > 1) atomicMax(single_row, ~(unsigned long long)i); return m ? m : 1;
    case MO_JOIN_SEMI: return m ? 1 : 0;
    case MO_JOIN_ANTI: return m ? 0 : 1;
    default: return 0;
    }
}

// counts per probe row of the rows it emits.  RIGHT SEMI and RIGHT ANTI mark here (groups of >= 32 sels by the whole warp) and the call skips
// the scan and the emit pass (cnt == nullptr).  The types that emit pairs mark in the emit pass, once the result is known to fit, so a call that
// fails with MO_RC_OUT_OF_RANGE leaves the bitmap as it was and its repeat marks each pair once.
template <class Lookup>
__global__ void __launch_bounds__(kThreads) probe_count_kernel(Lookup lookup, uint64_t n, const int32_t *__restrict__ offsets, const int32_t *__restrict__ sels,
                                                               int join_type, uint32_t *__restrict__ vals, uint64_t *__restrict__ cnt, Marks M,
                                                               unsigned long long *single_row) {
    const unsigned lane = threadIdx.x & 31;
    const bool mark_here = join_type == MO_JOIN_RIGHT_SEMI || join_type == MO_JOIN_RIGHT_ANTI;
    for (uint64_t i0 = blockIdx.x * (uint64_t)kThreads + (threadIdx.x & ~31u); i0 < n; i0 += (uint64_t)gridDim.x * kThreads) {
        const uint64_t i = i0 + lane;                    // the loop is warp-uniform: whole warps mark heavy groups
        uint32_t v = 0;
        uint64_t m = 0;
        if (i < n) {
            v = lookup(i);
            if (v) m = offsets ? (uint64_t)(offsets[v] - offsets[v - 1]) : 1ull;
            const uint64_t c = result_rows(join_type, m, i, single_row);
            if (cnt) { vals[i] = m ? v : 0u; cnt[i] = c; }
        }
        if (mark_here) {
            const int32_t s0 = (m && offsets) ? offsets[v - 1] : 0;
            if (m && m < 32) for (uint64_t j = 0; j < m; j++) M.mark(offsets ? (uint64_t)sels[s0 + j] : (uint64_t)v - 1);
            unsigned heavy = __ballot_sync(0xffffffffu, m >= 32);
            while (heavy) {
                const int src = __ffs(heavy) - 1; heavy &= heavy - 1;
                const uint64_t hm = __shfl_sync(0xffffffffu, m, src);
                const int32_t hs0 = __shfl_sync(0xffffffffu, s0, src);
                for (uint64_t j = lane; j < hm; j += 32) M.mark((uint64_t)sels[hs0 + j]);
            }
        }
    }
}

// The emit pass reads each probe row's build rows from a row source: range(i, c, h, e) gives row i, which emits c rows, its entries [h, e);
// build(k) is the build row of entry k and pass(k) whether the entry is a match.
// JOIN_PROBE / JOIN_PROBE_GIDS: the matched group's sels (vals[i] = group id, 0 = no match), every entry a match, so the row's count from the scan
// is its entry count.  A unique map has entry v - 1 = build row v - 1.
struct ProbeRows {
    const uint32_t *__restrict__ vals; const int32_t *__restrict__ offsets; const int32_t *__restrict__ sels;
    __device__ __forceinline__ void range(uint64_t i, uint64_t c, uint64_t &h, uint64_t &e) const {
        const uint32_t v = vals[i];
        h = v ? (offsets ? (uint64_t)offsets[v - 1] : (uint64_t)v - 1) : 0;
        e = v ? h + c : 0;
    }
    __device__ __forceinline__ int64_t build(uint64_t k) const { return offsets ? (int64_t)sels[k] : (int64_t)k; }
    __device__ __forceinline__ bool pass(uint64_t) const { return true; }
};

// ---- JOIN_MATCHED_MERGE: syncBitmap's OR over the workers' bitmaps (join.go:650-676) ------------------------------------------------------------
struct MergeInputs { const unsigned long long *p[MO_JOIN_MERGE_MAX]; };
__global__ void __launch_bounds__(kThreads) matched_merge_kernel(MergeInputs in, int n, uint64_t words, uint64_t nbits, unsigned long long *out,
                                                                 unsigned long long *twice) {
    for (uint64_t w = blockIdx.x * (uint64_t)kThreads + threadIdx.x; w < words; w += (uint64_t)gridDim.x * kThreads) {
        unsigned long long o = 0, d = 0;                 // d: bits set in two inputs (summed counts > the OR's count exactly when d != 0)
        for (int k = 0; k < n; k++) { const unsigned long long x = in.p[k][w]; d |= o & x; o |= x; }
        if (w == words - 1 && (nbits & 63)) { const unsigned long long live = (1ull << (nbits & 63)) - 1; o &= live; d &= live; }
        out[w] = o;
        if (twice && d) atomicMax(twice, ~(unsigned long long)(w * 64 + __ffsll((long long)d) - 1));   // ~row: 0 = none
    }
}

// ---- JOIN_COND: a join with a non-equality condition (NonEqCond, join.go:468-498,570-611), resolved over the INNER candidate pairs ---------------
// The caller evaluates the condition once per candidate pair; P(i) = probe row i's candidates whose condition is true and not NULL.  Record word 1
// holds ~(lowest malformed candidate position) in place of the bad group id.
__device__ __forceinline__ bool cond_pass(const uint8_t *__restrict__ cond, const uint64_t *__restrict__ cnulls, uint64_t k) {
    return cond[k] && !bm_test(cnulls, k);
}
// the row source of the emit pass: row i's candidates [head[i], end[i]), a match where the condition passes
struct CondRows {
    const uint64_t *__restrict__ head; const uint64_t *__restrict__ end; const int64_t *__restrict__ cb; const uint8_t *__restrict__ cond;
    const uint64_t *__restrict__ cnulls;
    __device__ __forceinline__ void range(uint64_t i, uint64_t, uint64_t &h, uint64_t &e) const { h = head[i]; e = end[i]; }
    __device__ __forceinline__ int64_t build(uint64_t k) const { return cb[k]; }
    __device__ __forceinline__ bool pass(uint64_t k) const { return cond_pass(cond, cnulls, k); }
};

// pass 1, over the pairs: validates them (probe rows in [0, len) and ascending, build rows >= 0 and, with a bitmap, inside it), gives every probe
// row its candidate range [head, end) (candidates are sorted by probe row: segment heads and tails) and adds up its passing pairs in pc, one
// atomic per warp and row.  RIGHT SEMI / RIGHT ANTI (head == nullptr) only mark.
__global__ void __launch_bounds__(kThreads) cond_pairs_kernel(const int64_t *__restrict__ cp, const int64_t *__restrict__ cb, const uint8_t *__restrict__ cond,
                                                              const uint64_t *__restrict__ cnulls, uint64_t npairs, uint64_t len, uint64_t *__restrict__ head,
                                                              uint64_t *__restrict__ end, unsigned long long *__restrict__ pc, Marks M, unsigned long long *bad) {
    const unsigned lane = threadIdx.x & 31;
    for (uint64_t k0 = blockIdx.x * (uint64_t)kThreads + (threadIdx.x & ~31u); k0 < npairs; k0 += (uint64_t)gridDim.x * kThreads) {
        const uint64_t k = k0 + lane;                    // the loop is warp-uniform: the warp aggregates its pass counts
        int64_t p = -1;
        bool f = false;
        if (k < npairs) {
            p = cp[k];
            const int64_t b = cb[k];
            if (p < 0 || (uint64_t)p >= len || b < 0 || (k && cp[k - 1] > p)) { atomicMax(bad, ~(unsigned long long)k); p = -1; }
            else {
                f = cond_pass(cond, cnulls, k);
                if (M.past && (uint64_t)b >= M.nbits) atomicMax(M.past, ~(unsigned long long)b);
                else if (f && !head) M.mark((uint64_t)b);
                if (head) {
                    if (k == 0 || cp[k - 1] != p) head[p] = k;
                    if (k + 1 == npairs || cp[k + 1] != p) end[p] = k + 1;
                }
            }
        }
        if (head) {
            const unsigned same = __match_any_sync(0xffffffffu, (unsigned long long)p), passing = __ballot_sync(0xffffffffu, f);
            const unsigned c = __popc(passing & same);
            if (p >= 0 && c && lane == (unsigned)__ffs(same) - 1) atomicAdd(&pc[p], (unsigned long long)c);
        }
    }
}
// pass 2, over the probe rows: pass count -> result rows of the row, in place
__global__ void __launch_bounds__(kThreads) cond_count_kernel(uint64_t n, uint64_t *__restrict__ cnt, int join_type, unsigned long long *single_row) {
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads)
        cnt[i] = result_rows(join_type, cnt[i], i, single_row);
}

// ---- the emit pass, over the probe rows ------------------------------------------------------------------------------------------------------------
// Each matching entry of a row is written at the row's scanned position plus its rank among the row's matches; a row that emits without a match
// writes (i, -1), as SEMI and ANTI rows always do.  Rows with >= 32 entries are walked by their whole warp, ranks from a ballot.  Nothing is
// written when record word 1 is set; RIGHT, FULL and RIGHT SINGLE mark (M.words) only when the whole result fits.
template <class Rows>
__global__ void __launch_bounds__(kThreads) emit_kernel(Rows R, uint64_t n, const uint64_t *__restrict__ pos, const uint64_t *__restrict__ rec, int join_type,
                                                        uint64_t cap, int64_t *__restrict__ out_probe, int64_t *__restrict__ out_build, int64_t *count_out, Marks M) {
    const uint64_t total = rec[0];
    if (blockIdx.x == 0 && threadIdx.x == 0) *count_out = (int64_t)total;
    if (rec[1]) return;
    const unsigned lane = threadIdx.x & 31;
    const bool mark = M.words && total <= cap;
    const bool pairs = join_type != MO_JOIN_SEMI && join_type != MO_JOIN_ANTI;
    const uint64_t nrounds = (n + 31) / 32;
    for (uint64_t w = (blockIdx.x * (uint64_t)kThreads + threadIdx.x) >> 5; w < nrounds; w += ((uint64_t)gridDim.x * kThreads) >> 5) {
        const uint64_t i = w * 32 + lane;
        uint64_t p = 0, c = 0, h = 0, e = 0;
        if (i < n) { p = pos[i]; c = (i + 1 < n ? pos[i + 1] : total) - p; }
        if (c && pairs) R.range(i, c, h, e);
        if (c && e - h < 32) {
            uint64_t j = 0;
#pragma unroll 1   // unrolled, the probe's walk (no entry can fail) takes 40 registers and 6 CTAs per SM instead of 32 and 8
            for (uint64_t k = h; k < e; k++) {
                if (!R.pass(k)) continue;
                const int64_t b = R.build(k);
                if (p + j < cap) { out_probe[p + j] = (int64_t)i; out_build[p + j] = b; if (mark) M.mark((uint64_t)b); }
                j++;
            }
            if (j == 0 && p < cap) { out_probe[p] = (int64_t)i; out_build[p] = -1; }
        }
        unsigned heavy = __ballot_sync(0xffffffffu, c && e - h >= 32);
        while (heavy) {
            const int src = __ffs(heavy) - 1; heavy &= heavy - 1;
            const uint64_t hi = __shfl_sync(0xffffffffu, i, src), hp = __shfl_sync(0xffffffffu, p, src);
            const uint64_t hh = __shfl_sync(0xffffffffu, h, src), he = __shfl_sync(0xffffffffu, e, src);
            uint64_t base = 0;
            for (uint64_t k0 = hh; k0 < he; k0 += 32) {
                const uint64_t k = k0 + lane;
                const bool f = k < he && R.pass(k);
                const unsigned ball = __ballot_sync(0xffffffffu, f);
                const uint64_t q = hp + base + __popc(ball & ((1u << lane) - 1));
                if (f && q < cap) { const int64_t b = R.build(k); out_probe[q] = (int64_t)hi; out_build[q] = b; if (mark) M.mark((uint64_t)b); }
                base += __popc(ball);
            }
            if (base == 0 && lane == 0 && hp < cap) { out_probe[hp] = (int64_t)hi; out_build[hp] = -1; }
        }
    }
}

// The end of JOIN_PROBE, JOIN_PROBE_GIDS and JOIN_COND.  Stages args [0] probe_rows, [1] build_rows, [2] count and args[mi], the matched bitmap of
// types MO_JOIN_RIGHT and above, and zeroes the record; first(M, record) launches the first pass, which leaves each probe row's result rows in cnt
// or, for RIGHT SEMI / RIGHT ANTI (cnt == nullptr), marks.  Then the scan and the emit pass over R, and the record read back in one copy:
// word1(h[1]) sets the caller's error for word 1, the others name the caller (what).
template <class Rows, class First, class Word1>
int join_tail(ThreadCtx &t, Stager &st, mo_xcall_args_t *args, int mi, int join_type, uint64_t len, uint64_t *cnt, Rows R, First first, const char *what,
              Word1 word1) {
    const uint64_t cap = args[0].dataSz / 8;
    uint64_t *scal = (uint64_t *)st.tmp(kRecWords * 8);
    int64_t *out_probe = (int64_t *)st.out(args[0].pdata, cap * 8);
    int64_t *out_build = (int64_t *)st.out(args[1].pdata, cap * 8);
    int64_t *count = (int64_t *)st.out(args[2].pdata, 8);
    Marks M;
    if (join_type >= MO_JOIN_RIGHT) {
        const uint64_t words = args[mi].dataSz / 8;
        M.words = (unsigned long long *)st.out(args[mi].pdata, words * 8, true);   // in/out: a host bitmap is uploaded and copied back
        M.nbits = words * 64; M.single = join_type == MO_JOIN_RIGHT_SINGLE;
        M.twice = (unsigned long long *)(scal + 3); M.past = (unsigned long long *)(scal + 4);
    }
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(scal, 0, kRecWords * 8, t.stream));
    cudaEventRecord(t.kev0, t.stream);
    if (int rc = first(M, scal)) return rc;
    if (cnt) {
        int rc = exclusive_scan(t, cnt, len, cnt, scal);
        if (rc) { st.finish(); return rc; }
        const Marks EM = join_type == MO_JOIN_RIGHT || join_type == MO_JOIN_FULL || join_type == MO_JOIN_RIGHT_SINGLE ? M : Marks();
        emit_kernel<<<grid_for(len ? len : 1), kThreads, 0, t.stream>>>(R, len, cnt, scal, join_type, cap, out_probe, out_build, count, EM);
    } else {
        MOB_CUDA_TRY(cudaMemsetAsync(count, 0, 8, t.stream));   // right semi / right anti: no pairs during the probe
    }
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    uint64_t h[kRecWords] = {};
    int rc = read_back(t, h, scal, sizeof h);
    int frc = st.finish();
    if (rc) return rc;
    if (h[1]) { word1(h[1]); return MO_RC_INVALID_ARGUMENT; }
    if (h[4]) { set_error("%s: build row %llu lies past the matched bitmap (%llu rows)", what, (unsigned long long)~h[4], (unsigned long long)M.nbits); return MO_RC_INVALID_ARGUMENT; }
    if (h[2]) { set_error("scalar subquery returns more than 1 row (probe row %llu)", (unsigned long long)~h[2]); return MO_RC_INTERNAL_ERROR; }
    if (h[3]) { set_error("scalar subquery returns more than 1 row (build row %llu)", (unsigned long long)~h[3]); return MO_RC_INTERNAL_ERROR; }
    if (h[0] > cap) { set_error("%s: %lld result rows exceed the output capacity (%llu); the count is reported, call again with larger buffers", what, (long long)h[0], (unsigned long long)cap); return MO_RC_OUT_OF_RANGE; }
    return frc;
}

// JOIN_PROBE and JOIN_PROBE_GIDS after the lookup's inputs: args [5] / [6] sels, [8] the matched bitmap; lookup_at(record) is the lookup, which may
// set record word 1
template <class LookupAt>
int run_probe(ThreadCtx &t, Stager &st, mo_xcall_args_t *args, uint64_t len, int join_type, uint64_t ngroups, LookupAt lookup_at) {
    const bool multi = args[5].pdata != nullptr;
    const bool emits = join_type != MO_JOIN_RIGHT_SEMI && join_type != MO_JOIN_RIGHT_ANTI;
    const int32_t *offsets = multi ? (const int32_t *)st.in(args[5].pdata, (ngroups + 2) * 4) : nullptr;
    const int32_t *sels = multi ? (const int32_t *)st.in(args[6].pdata, args[6].dataSz) : nullptr;
    uint32_t *vals = emits ? (uint32_t *)st.tmp(len * 4 + 4) : nullptr;
    uint64_t *cnt = emits ? (uint64_t *)st.tmp((len + 1) * 8) : nullptr;
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    return join_tail(t, st, args, 8, join_type, len, cnt, ProbeRows{vals, offsets, sels}, [&](const Marks &M, uint64_t *rec) {
        probe_count_kernel<<<grid_for(len ? len : 1), kThreads, 0, t.stream>>>(lookup_at(rec), len, offsets, sels, join_type, vals, cnt, M, (unsigned long long *)(rec + 2));
        MOB_LAUNCH_CHECK();
        return MO_RC_SUCCESS;
    }, "join probe", [&](uint64_t) { set_error("join probe: a group id exceeds the group count (%llu)", (unsigned long long)ngroups); });
}

// the argument checks of JOIN_PROBE and JOIN_PROBE_GIDS; a unique map (no sels) names build rows 0 .. ngroups - 1, so its bitmap must hold ngroups
// bits (with sels, a row past the bitmap is found on the device)
int check_probe_args(const mo_xcall_args_t *args, uint64_t len, int join_type, uint64_t ngroups, const char *what) {
    if (int rc = check_join_type(join_type, what, false)) return rc;
    if (join_type >= MO_JOIN_RIGHT && !args[8].pdata) { set_error("%s: join type %d needs the matched bitmap in args[8]", what, join_type); return MO_RC_INVALID_ARGUMENT; }
    if (join_type >= MO_JOIN_RIGHT && !args[5].pdata && args[8].dataSz / 8 < (ngroups + 63) / 64) {
        set_error("%s: the matched bitmap holds %llu rows, the build side has %llu", what, (unsigned long long)(args[8].dataSz / 8 * 64), (unsigned long long)ngroups);
        return MO_RC_INVALID_ARGUMENT;
    }
    if (args[1].dataSz / 8 < args[0].dataSz / 8 || !args[2].pdata || args[2].dataSz < 8 || args[7].dataSz < 8 * len) { set_error("%s: buffers too small", what); return MO_RC_INVALID_ARGUMENT; }
    if (args[5].pdata && args[5].dataSz < (ngroups + 2) * 4) { set_error("%s: sels offsets shorter than the group count + 2", what); return MO_RC_INVALID_ARGUMENT; }
    return MO_RC_SUCCESS;
}

}  // namespace

// Stable grouping of rows by their 1-based group id (0 = the row takes no part): *starts = uint64[ngroups + 1] (start of every 0-based group in
// *rows), *rows = uint32[n] row ids, ascending inside every group, *scal[0] = how many rows have a group, scal[2] (as unsigned) != 0 = an id exceeded
// ngroups.  Everything lives in the call's arena.  Used by JOIN_SELS and by the k-means centroid update (kmeans.cu).
int group_rows_stable(ThreadCtx &t, const uint64_t *groups, uint64_t len, uint64_t ngroups, uint64_t **starts, uint32_t **rows, uint64_t **scal_out) {
    uint64_t *flag = (uint64_t *)arena_alloc(t, (len + 1) * 8), *cnt = (uint64_t *)arena_alloc(t, (ngroups + 1) * 8);
    uint32_t *k0 = (uint32_t *)arena_alloc(t, len * 4 + 4), *r0 = (uint32_t *)arena_alloc(t, len * 4 + 4), *k1 = (uint32_t *)arena_alloc(t, len * 4 + 4), *r1 = (uint32_t *)arena_alloc(t, len * 4 + 4);
    uint64_t *scal = (uint64_t *)arena_alloc(t, 32);     // [0] rows with a group, [1] scratch total, [2] bad flag
    if (!flag || !cnt || !k0 || !r0 || !k1 || !r1 || !scal) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(cnt, 0, (ngroups + 1) * 8, t.stream));
    MOB_CUDA_TRY(cudaMemsetAsync(scal, 0, 32, t.stream));
    sels_flag_kernel<<<grid_for(len ? len : 1), kThreads, 0, t.stream>>>(groups, len, ngroups, flag, cnt, (unsigned *)(scal + 2));
    MOB_LAUNCH_CHECK();
    int rc = exclusive_scan(t, flag, len, flag, scal);                 // flag -> position among the rows that have a group ; scal[0] = m
    if (rc) return rc;
    sels_compact_kernel<<<grid_for(len ? len : 1), kThreads, 0, t.stream>>>(groups, flag, len, ngroups, k0, r0);
    MOB_LAUNCH_CHECK();
    rc = sort_u32_pairs(t, k0, r0, k1, r1, scal, len);                // stable by group id: rows ascending inside every group, in r0
    if (rc) return rc;
    rc = exclusive_scan(t, cnt, ngroups, cnt, scal + 1);               // cnt[k] -> start of group k
    if (rc) return rc;
    MOB_CUDA_TRY(cudaMemcpyAsync(cnt + ngroups, scal, 8, cudaMemcpyDeviceToDevice, t.stream));   // starts[ngroups] = m
    *starts = cnt; *rows = r0; *scal_out = scal;
    return MO_RC_SUCCESS;
}

// MO_XCALL_JOIN_SELS: args [0] offsets int32[ngroups + 2] ; [1] vals int32[len] ; [2] int64 count (out: rows that have a group) ; [3] groups uint64[len]
int xcall_join_sels(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!args[0].pdata || args[0].dataSz < 8 || !args[2].pdata || args[2].dataSz < 8 || args[1].dataSz < 4 * len || args[3].dataSz < 8 * len) { set_error("join sels: buffers too small"); return MO_RC_INVALID_ARGUMENT; }
    if (len >= 0x7fffffffull) { set_error("join sels: at most 2^31 build rows (row ids are int32, joinMapMsg.go:32-40)"); return MO_RC_INVALID_ARGUMENT; }
    const uint64_t ngroups = args[0].dataSz / 4 - 2;
    Stager st(t);
    int32_t *offsets = (int32_t *)st.out(args[0].pdata, (ngroups + 2) * 4);
    int32_t *vals = (int32_t *)st.out(args[1].pdata, 4 * len);
    int64_t *count = (int64_t *)st.out(args[2].pdata, 8);
    const uint64_t *groups = (const uint64_t *)st.in(args[3].pdata, 8 * len);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    cudaEventRecord(t.kev0, t.stream);
    uint64_t *starts, *scal; uint32_t *rows;
    int rc = group_rows_stable(t, groups, len, ngroups, &starts, &rows, &scal);
    if (rc) { st.finish(); return rc; }
    sels_offsets_kernel<<<grid_for(ngroups + 2), kThreads, 0, t.stream>>>(starts, ngroups, scal, offsets);
    MOB_LAUNCH_CHECK();
    copy_rows_kernel<<<grid_for(len ? len : 1), kThreads, 0, t.stream>>>(rows, scal, vals, count);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    unsigned bad = 0;
    rc = read_back(t, &bad, scal + 2, 4);
    int frc = st.finish();
    if (rc) return rc;
    if (bad) { set_error("join sels: a group id exceeds the group count (%llu)", (unsigned long long)ngroups); return MO_RC_INVALID_ARGUMENT; }
    return frc;
}

// MO_XCALL_JOIN_FIND: args [0] vals uint64[len] ; [1] table_keys uint64[ngroups] ; [2] probe keys uint64[len] (+pnulls)
int xcall_join_find(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (args[0].dataSz < 8 * len || args[2].dataSz < 8 * len) { set_error("join find: buffers too small"); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    DevTable T;
    std::shared_lock<std::shared_mutex> lk;
    int rc = table_for(t, st, args[1], &T, lk);
    if (rc) { st.finish(); return rc; }
    uint64_t *vals = (uint64_t *)st.out(args[0].pdata, 8 * len);
    const uint64_t *keys = (const uint64_t *)st.in(args[2].pdata, 8 * len);
    const uint64_t *kn = (const uint64_t *)st.in(args[2].pnulls, args[2].pnulls ? ((len + 63) / 64) * 8 : 0);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    cudaEventRecord(t.kev0, t.stream);
    jt_find_kernel<<<grid_for(len ? len : 1), kThreads, 0, t.stream>>>(KeyLookup{keys, kn, T.key, T.id, T.mask}, len, vals);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.finish();
}

// MO_XCALL_JOIN_PROBE: args [0] probe_rows int64[cap] ; [1] build_rows int64[cap] ; [2] int64 count (out) ; [3] mo_join_params_t ; [4] table_keys uint64[ngroups]
// ; [5] sels offsets int32[ngroups + 2] (pdata NULL: unique map, build row = id - 1) ; [6] sels vals int32[] ; [7] probe keys uint64[len] (+pnulls)
int xcall_join_probe(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    mo_join_params_t P;
    if (int rc = read_param(t, args[3], &P, sizeof P, sizeof P, "join probe: mo_join_params_t")) return rc;
    const uint64_t ngroups = args[4].dataSz / 8;
    if (int rc = check_probe_args(args, len, P.join_type, ngroups, "join probe")) return rc;
    Stager st(t);
    DevTable T;
    std::shared_lock<std::shared_mutex> lk;
    int rc = table_for(t, st, args[4], &T, lk);
    if (rc) { st.finish(); return rc; }
    const uint64_t *keys = (const uint64_t *)st.in(args[7].pdata, 8 * len);
    const uint64_t *kn = (const uint64_t *)st.in(args[7].pnulls, args[7].pnulls ? ((len + 63) / 64) * 8 : 0);
    return run_probe(t, st, args, len, P.join_type, ngroups, [&](uint64_t *) { return KeyLookup{keys, kn, T.key, T.id, T.mask}; });
}

// MO_XCALL_JOIN_PROBE_GIDS: args [0..3], [5], [6] as JOIN_PROBE ; [4] int64 ngroups ; [7] vals uint64[len] (group ids, 0 = no match)
int xcall_join_probe_gids(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    mo_join_params_t P;
    if (int rc = read_param(t, args[3], &P, sizeof P, sizeof P, "join probe gids: mo_join_params_t")) return rc;
    int64_t ng;
    if (int rc = read_param(t, args[4], &ng, 8, 8, "join probe gids: [4] int64 ngroups")) return rc;
    if (ng < 0) { set_error("join probe gids: [4] must be an int64 ngroups >= 0"); return MO_RC_INVALID_ARGUMENT; }
    const uint64_t ngroups = (uint64_t)ng;
    if (int rc = check_probe_args(args, len, P.join_type, ngroups, "join probe gids")) return rc;
    Stager st(t);
    const uint64_t *gids = (const uint64_t *)st.in(args[7].pdata, 8 * len);
    return run_probe(t, st, args, len, P.join_type, ngroups, [&](uint64_t *rec) { return GidLookup{gids, ngroups, (unsigned *)(rec + 1)}; });
}

// MO_XCALL_JOIN_MATCHED_MERGE: args [0] out bitmap uint64[(len + 63) / 64] ; [1] int32 n ; [2] mo_join_params_t ; [3 .. 3 + n) input bitmaps
// (the same words).  len = build rows.  RIGHT SINGLE reads back the lowest bit set in two inputs; the other types complete as the Stager decides.
int xcall_join_matched_merge(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    int32_t n;
    if (int rc = read_param(t, args[1], &n, 4, 4, "join matched merge: [1] int32 n")) return rc;
    mo_join_params_t P;
    if (int rc = read_param(t, args[2], &P, sizeof P, sizeof P, "join matched merge: mo_join_params_t")) return rc;
    if (int rc = check_join_type(P.join_type, "join matched merge", true)) return rc;
    if (n < 1 || n > MO_JOIN_MERGE_MAX) { set_error("join matched merge: %d inputs (1..%d)", n, MO_JOIN_MERGE_MAX); return MO_RC_INVALID_ARGUMENT; }
    const uint64_t words = (len + 63) / 64;
    if (!args[0].pdata || args[0].dataSz < 8 * words) { set_error("join matched merge: the out bitmap holds fewer than %llu rows", (unsigned long long)len); return MO_RC_INVALID_ARGUMENT; }
    for (int k = 0; k < n; k++)
        if (!args[3 + k].pdata || args[3 + k].dataSz < 8 * words) { set_error("join matched merge: input %d holds fewer than %llu rows", k, (unsigned long long)len); return MO_RC_INVALID_ARGUMENT; }
    if (words == 0) return MO_RC_SUCCESS;
    const bool single = P.join_type == MO_JOIN_RIGHT_SINGLE;
    Stager st(t);
    MergeInputs in;
    for (int k = 0; k < n; k++) in.p[k] = (const unsigned long long *)st.in(args[3 + k].pdata, 8 * words);
    unsigned long long *out = (unsigned long long *)st.out(args[0].pdata, 8 * words);
    unsigned long long *twice = single ? (unsigned long long *)st.tmp(8) : nullptr;
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    if (single) MOB_CUDA_TRY(cudaMemsetAsync(twice, 0, 8, t.stream));
    cudaEventRecord(t.kev0, t.stream);
    matched_merge_kernel<<<grid_for(words), kThreads, 0, t.stream>>>(in, n, words, len, out, twice);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    if (!single) return st.complete();
    unsigned long long h = 0;
    int rc = read_back(t, &h, twice, 8);
    int frc = st.finish();
    if (rc) return rc;
    if (h) { set_error("scalar subquery returns more than 1 row (build row %llu)", ~h); return MO_RC_INTERNAL_ERROR; }
    return frc;
}

// MO_XCALL_JOIN_COND: args [0..3] as JOIN_PROBE ; [4] candidate probe rows int64[npairs] ; [5] candidate build rows int64[npairs] ; [6] the
// condition bool[npairs] (+pnulls) ; [7] the matched bitmap (types MO_JOIN_RIGHT and above).  len = probe rows of the batch.  Reads back the
// record in one copy, as JOIN_PROBE does.
int xcall_join_cond(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    mo_join_params_t P;
    if (int rc = read_param(t, args[3], &P, sizeof P, sizeof P, "join cond: mo_join_params_t")) return rc;
    const int jt = P.join_type;
    if (int rc = check_join_type(jt, "join cond", false)) return rc;
    if (jt >= MO_JOIN_RIGHT && !args[7].pdata) { set_error("join cond: join type %d needs the matched bitmap in args[7]", jt); return MO_RC_INVALID_ARGUMENT; }
    const uint64_t cap = args[0].dataSz / 8, npairs = args[4].dataSz / 8;
    if (args[1].dataSz / 8 < cap || !args[2].pdata || args[2].dataSz < 8 || args[5].dataSz < 8 * npairs || args[6].dataSz < npairs) {
        set_error("join cond: buffers too small");
        return MO_RC_INVALID_ARGUMENT;
    }
    const bool emits = jt != MO_JOIN_RIGHT_SEMI && jt != MO_JOIN_RIGHT_ANTI;
    Stager st(t);
    const int64_t *cp = (const int64_t *)st.in(args[4].pdata, npairs * 8);
    const int64_t *cb = (const int64_t *)st.in(args[5].pdata, npairs * 8);
    const uint8_t *cond = (const uint8_t *)st.in(args[6].pdata, npairs);
    const uint64_t *cn = (const uint64_t *)st.in(args[6].pnulls, args[6].pnulls ? ((npairs + 63) / 64) * 8 : 0);
    uint64_t *head = emits ? (uint64_t *)st.tmp(len * 8 + 8) : nullptr;
    uint64_t *end = emits ? (uint64_t *)st.tmp(len * 8 + 8) : nullptr;
    uint64_t *cnt = emits ? (uint64_t *)st.tmp(len * 8 + 8) : nullptr;
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    if (emits) {
        MOB_CUDA_TRY(cudaMemsetAsync(head, 0, len * 8, t.stream));
        MOB_CUDA_TRY(cudaMemsetAsync(end, 0, len * 8, t.stream));
        MOB_CUDA_TRY(cudaMemsetAsync(cnt, 0, len * 8, t.stream));
    }
    return join_tail(t, st, args, 7, jt, len, cnt, CondRows{head, end, cb, cond, cn}, [&](const Marks &M, uint64_t *rec) {
        cond_pairs_kernel<<<grid_for(npairs ? npairs : 1), kThreads, 0, t.stream>>>(cp, cb, cond, cn, npairs, len, head, end, (unsigned long long *)cnt, M,
                                                                                     (unsigned long long *)(rec + 1));
        MOB_LAUNCH_CHECK();
        if (emits) {
            cond_count_kernel<<<grid_for(len ? len : 1), kThreads, 0, t.stream>>>(len, cnt, jt, (unsigned long long *)(rec + 2));
            MOB_LAUNCH_CHECK();
        }
        return MO_RC_SUCCESS;
    }, "join cond", [&](uint64_t w) {
        set_error("join cond: candidate %llu is malformed: its probe row lies outside [0, %llu) or below the one before it, or its build row is negative",
                  (unsigned long long)~w, (unsigned long long)len);
    });
}

// MO_XCALL_STR_JOIN_FIND: args [0] vals uint64[len] ; [1] int64 ngroups ; [2] table bytes ; [3] table offsets uint64[ngroups + 1] ; [4] probe key
// bytes ; [5] probe key offsets uint64[len + 1] (+pnulls)
int xcall_str_join_find(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    int64_t ng;
    if (int rc = read_param(t, args[1], &ng, 8, 8, "str join find: [1] int64 ngroups")) return rc;
    if (ng < 0) { set_error("str join find: [1] must be an int64 ngroups >= 0"); return MO_RC_INVALID_ARGUMENT; }
    const uint64_t ngroups = (uint64_t)ng;
    if (args[0].dataSz < 8 * len || !args[3].pdata || args[3].dataSz < 8 * (ngroups + 1) || !args[5].pdata || args[5].dataSz < 8 * (len + 1)) { set_error("str join find: buffers too small"); return MO_RC_INVALID_ARGUMENT; }
    if (ngroups >= 0x7fffffffull) { set_error("str join find: at most 2^31 groups"); return MO_RC_INVALID_ARGUMENT; }
    // host offsets must lie inside their bytes (device offsets are the caller's to keep right)
    if (!is_device_ptr(args[3].pdata) && ((const uint64_t *)args[3].pdata)[ngroups] > args[2].dataSz) { set_error("str join find: table offsets end past the table bytes (%llu)", (unsigned long long)args[2].dataSz); return MO_RC_INVALID_ARGUMENT; }
    if (!is_device_ptr(args[5].pdata) && ((const uint64_t *)args[5].pdata)[len] > args[4].dataSz) { set_error("str join find: probe key offsets end past the key bytes (%llu)", (unsigned long long)args[4].dataSz); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    DevTable T;
    std::shared_lock<std::shared_mutex> lk;
    int rc = str_table_for(t, st, args[2], args[3], ngroups, &T, lk);
    if (rc) { st.finish(); return rc; }
    uint64_t *vals = (uint64_t *)st.out(args[0].pdata, 8 * len);
    const uint8_t *kbytes = (const uint8_t *)st.in(args[4].pdata, args[4].dataSz);
    const uint64_t *koff = (const uint64_t *)st.in(args[5].pdata, 8 * (len + 1));
    const uint64_t *kn = (const uint64_t *)st.in(args[5].pnulls, args[5].pnulls ? ((len + 63) / 64) * 8 : 0);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    cudaEventRecord(t.kev0, t.stream);
    sjt_find_kernel<<<grid_for(len ? len : 1), kThreads, 0, t.stream>>>(StrKeys{T.sbytes, T.soff, kbytes, koff, ngroups}, kn, len, T.key, T.mask, strkey_hash_mask(), vals);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    // asynchronous form: a prepared table may be released while this kernel still reads it; its cudaFree waits for the device's pending work
    return st.complete();
}

}  // namespace mob

// ---- prepared join maps (the JoinMap message lives for the whole probe phase: message/joinMapMsg.go:127-160) ---------------------------------------
extern "C" int32_t MoB200_JoinMapPrepare(const void *table_keys, uint64_t ngroups) {
    using namespace mob;
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    Stager st(t);
    const uint64_t *dkeys = (const uint64_t *)st.in(table_keys, ngroups * 8);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    DevTable T;
    int rc = build_table(t, ngroups, dkeys, nullptr, nullptr, true, &T);
    int frc = st.finish();
    if (rc || frc) { if (!rc) free_table(T); return rc ? rc : frc; }
    publish_prepared(table_keys, T);
    return MO_RC_SUCCESS;
}

// the string map: the table's bytes and offsets are copied to the device with it, so the caller may change or free its copy
extern "C" int32_t MoB200_StrJoinMapPrepare(const void *table_bytes, const void *table_offsets, uint64_t ngroups) {
    using namespace mob;
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!table_offsets || ngroups >= 0x7fffffffull) { set_error("str join map: table offsets missing or more than 2^31 groups"); return MO_RC_INVALID_ARGUMENT; }
    uint64_t nbytes = 0;
    if (is_device_ptr(table_offsets)) { int rc = read_back(t, &nbytes, (const uint64_t *)table_offsets + ngroups, 8); if (rc) return rc; }
    else memcpy(&nbytes, (const uint64_t *)table_offsets + ngroups, 8);
    if (nbytes && !table_bytes) { set_error("str join map: table bytes missing"); return MO_RC_INVALID_ARGUMENT; }
    uint8_t *db = nullptr;
    uint64_t *doff = nullptr;
    if (cudaMalloc(&db, nbytes ? nbytes : 1) != cudaSuccess || cudaMalloc(&doff, (ngroups + 1) * 8) != cudaSuccess) {
        set_error("str join map: cudaMalloc of %llu bytes failed", (unsigned long long)nbytes);
        cudaFree(db);
        return MO_RC_INTERNAL_ERROR;
    }
    DevTable T;
    int rc = MO_RC_SUCCESS;
    if (nbytes && cudaMemcpyAsync(db, table_bytes, nbytes, cudaMemcpyDefault, t.stream) != cudaSuccess) rc = MO_RC_INTERNAL_ERROR;
    if (!rc && cudaMemcpyAsync(doff, table_offsets, (ngroups + 1) * 8, cudaMemcpyDefault, t.stream) != cudaSuccess) rc = MO_RC_INTERNAL_ERROR;
    if (!rc) rc = build_table(t, ngroups, nullptr, db, doff, true, &T);
    if (!rc && cudaStreamSynchronize(t.stream) != cudaSuccess) rc = MO_RC_INTERNAL_ERROR;
    arena_reset(t);
    if (rc) {
        if (!t.err[0]) set_error("str join map: copying the table to the device failed");
        if (T.key) cudaFree(T.key);
        cudaFree(db); cudaFree(doff);
        return rc;
    }
    publish_prepared(table_offsets, T);
    return MO_RC_SUCCESS;
}

extern "C" int32_t MoB200_JoinMapRelease(const void *table_keys) {
    using namespace mob;
    std::unique_lock<std::shared_mutex> lk(g_jm_mu);
    auto it = g_jm.find(table_keys);
    if (it == g_jm.end()) return MO_RC_SUCCESS;
    // (8-byte probes hold the shared lock until their stream has drained, so nothing is reading the table once the unique lock is ours; an
    // asynchronous STR_JOIN_FIND may still be reading, and cudaFree waits for it)
    free_table(it->second);
    g_jm.erase(it);
    return MO_RC_SUCCESS;
}
