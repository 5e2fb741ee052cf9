// order.cu -- ORDER BY and ORDER BY ... LIMIT on the device: the sels of the Order and Top operators (pkg/sql/colexec/{order,top}), and the
// stable LSD radix sort they are built on (also the grouping of JOIN_SELS and of the k-means centroid update, join.cu).
//
// MO_XCALL_ORDER_SELS (include/mo_b200.h) -- the order:
//   * Keys compare left to right with compare.New(type, desc, nullsLast) (pkg/compare/compare.go:24-115,231-239): two NULLs are equal, a
//     NULL is below every value when !nullsLast and above it when nullsLast (nullsCompare, compare/types.go:57-80); values compare with
//     GenericAscCompare / GenericDescCompare (container/types/compare.go:52-105), DECIMAL128 as signed 128-bit (types.Decimal128.Less).
//     Neither NULLS flag set: nullsLast = desc (order.go:143-150, top.go:249-257).
//   * Floats: -0.0 == +0.0 (Go's ==).  NaN is above every number (GenericAscCompare(NaN, x) = 1): last in ASC, first in DESC, and all NaNs are
//     equal.  The reference itself is not consistent there: compare(x, NaN) is 1 as well, so with NaN keys its Top result depends on the order
//     the rows arrive, and Order's pdqsort (pkg/sort/sort.go, `<`) leaves NaN wherever the partitioning drops it.
//   * Ties break by ascending row id: the row's index in this call, or row_ids[i] when given (then by index).  The order is total and stable,
//     so it has exactly one answer.  The reference breaks ties otherwise (Order: unstable pdqsort, Top: container/heap), so against it the
//     sequence of output key tuples is identical, and so are the rows wherever all key tuples are distinct.
//   * MergeOrder / MergeTop are the same call: every shard gathers its keys with SHUFFLE, its global row ids are base + sels, and the
//     concatenation goes into one call with row ids.  A streaming Top folds the same way (the rows kept so far + the next batch).
//
// Encoding (order_word, the one place that knows the format): every key is an order-preserving unsigned image -- signed: sign bit flipped;
// floats: -0.0 and NaN canonicalised, then the sign bit flipped, or every bit when the sign is set; DECIMAL128: two 64-bit segments; UUID:
// its 16 bytes big-endian in two segments; DESC: bitwise NOT.  A varlena key (CHAR, VARCHAR, TEXT, BLOB ...) is its bytes zero-padded to
// the longest value of the column (measured on the device and read back once per call), byte aligned, then its length in as many bits as the
// longest length needs: zero padding plus the length tie-break is exactly bytes.Compare, embedded zero bytes included.  A nullable key is
// preceded by one flag bit (NULLS FIRST: 0 = NULL, NULLS LAST: 1 = NULL) and a NULL's value bits are zero, so all NULLs are equal.  The
// fields are concatenated most significant first and cut into 64-bit words; row ids, when given, are a word of their own after them.
// Comparing the word sequences as unsigned integers is comparing the rows.
//
// Sort by rounds (varlena keys whose image is longer than kRoundWords words): the words go in rounds of kRoundWords, most significant
// first, each an LSD sort as below; after a round a kernel flags the positions where the image prefix changes and numbers the runs (a scan),
// and the next round sorts by (run number, its words): its words first, the run number as the last, most significant LSD word.  Once every
// run holds one row a device flag makes the remaining rounds' kernels return at once, so the cost follows the bytes that tell the rows
// apart, not the longest value; the host launches the rounds the longest value needs and reads nothing more back.
//
// Sort: LSD over the words, last word first.  The first word is computed in row order, each later word through the current permutation
// (random reads of the key columns).  Within a word, 8-bit digits least significant first, Onesweep-style (Adinets and Merrill, 2022): one
// histogram kernel computes the word once and counts all 8 digit positions; then one scatter kernel per digit ranks a 4096-row tile in
// shared memory (warp match + per-warp counts: equal digits keep their order) and takes its global offsets by decoupled look-back over the
// tiles.  Tiles are handed out by an atomic ticket, so a tile only ever waits on tiles that are already running.  A digit position whose rows
// all fall into one bucket is skipped; the decision is taken on the device (RadixState), so nothing is read back to the host.
//
// Top (0 <= limit < len / 8): radix select on the first word -- byte histograms from the most significant byte down, each over the rows
// whose higher bytes equal the bucket holding rank `limit` -- gives a prefix P at some byte level; the rows whose first word's prefix is
// <= P (every row tied with the limit-th one included) are compacted in row order and only they are sorted.  A nearly constant first word
// makes that set approach len: correct, no faster than the full sort.  String keys with a common leading prefix of 8 bytes or more (or 7 after
// a NULL flag) are such a case.
#include "common.cuh"
#include "column.cuh"
#include <cstring>

namespace mob {
int compact_bits(ThreadCtx &t, const uint32_t *bits, uint64_t n, int32_t *sels, unsigned long long *dtotal);   // colops.cu
}

using namespace mob;

namespace {

constexpr int kThreads = 256;
constexpr int kIPT = 16;                          // items per thread of a scatter tile
constexpr int kTile = kThreads * kIPT;            // 4096 rows
constexpr int kMaxSegs = 3 * MO_ORDER_MAX_KEYS + 1;   // per key <= 3 segments (flag + 2 halves, or flag + bytes + length) + row ids
constexpr int kRoundWords = 4;                         // image words per round of a sort by rounds (varlena keys)

// ---- the key encoding ------------------------------------------------------------------------------------------------------------------
// SEG_BYTES: a varlena value's bytes, zero-padded to the longest value of the key (bits = 8 * longest, byte aligned); SEG_LEN: its length;
// SEG_RUN: the run number of a sort by rounds (col = uint32 per row)
enum SegKind { SEG_NULL = 0, SEG_VALUE = 1, SEG_D128_HI = 2, SEG_D128_LO = 3, SEG_ROWID = 4, SEG_BYTES = 5, SEG_LEN = 6, SEG_RUN = 7 };
struct OrderSeg {
    const uint8_t *col;        // key column (a const key: one element), or varlena cells
    const uint64_t *nulls;     // nulls bitmap or nullptr
    const uint8_t *area;       // varlena area or nullptr
    uint64_t area_sz;
    int kind, type, bits, off; // off: first bit of the segment in the concatenated image, counted from the most significant end
    int cst, desc, nulls_last, pad;
};
struct OrderSpec { OrderSeg seg[kMaxSegs]; int nsegs; int nwords; };

__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
    return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
}

// VAR: the spec may hold varlena, run or UUID segments; false compiles them out of the path of the other fixed-width keys
template <bool VAR>
__device__ __forceinline__ uint64_t seg_image(const OrderSeg &s, uint64_t row) {
    const uint64_t r = s.cst ? 0 : row;
    if (s.kind == SEG_ROWID) return (uint64_t)reinterpret_cast<const int64_t *>(s.col)[r] ^ (1ull << 63);
    if (VAR && s.kind == SEG_RUN) return reinterpret_cast<const uint32_t *>(s.col)[row];
    const bool isnull = s.nulls && ((s.nulls[r >> 6] >> (r & 63)) & 1ull);
    if (s.kind == SEG_NULL) return (isnull == (bool)s.nulls_last) ? 1ull : 0ull;
    if (isnull) return 0;
    uint64_t v;
    if (VAR && s.kind == SEG_LEN) v = varlena_ref(s.col, r, s.area, s.area_sz).len;
    else if (VAR && s.type == MO_T_UUID) v = bswap64(reinterpret_cast<const uint64_t *>(s.col)[2 * r + (s.kind == SEG_D128_LO)]);   // bytes big-endian
    else switch (s.type) {
    case MO_T_BOOL: case MO_T_UINT8: v = s.col[r]; break;
    case MO_T_UINT16: v = reinterpret_cast<const uint16_t *>(s.col)[r]; break;
    case MO_T_UINT32: v = reinterpret_cast<const uint32_t *>(s.col)[r]; break;
    case MO_T_UINT64: v = reinterpret_cast<const uint64_t *>(s.col)[r]; break;
    case MO_T_INT8: v = (uint8_t)s.col[r] ^ 0x80u; break;
    case MO_T_INT16: v = reinterpret_cast<const uint16_t *>(s.col)[r] ^ 0x8000u; break;
    case MO_T_INT32: case MO_T_DATE: v = reinterpret_cast<const uint32_t *>(s.col)[r] ^ 0x80000000u; break;
    case MO_T_FLOAT32: {
        const float f = reinterpret_cast<const float *>(s.col)[r];
        uint32_t b = f != f ? 0x7fc00000u : (f == 0.0f ? 0u : __float_as_uint(f));
        v = (b >> 31) ? (uint32_t)~b : (b | 0x80000000u);
        break;
    }
    case MO_T_FLOAT64: {
        const double f = reinterpret_cast<const double *>(s.col)[r];
        const uint64_t b = f != f ? 0x7ff8000000000000ull : (f == 0.0 ? 0ull : (uint64_t)__double_as_longlong(f));
        v = (b >> 63) ? ~b : (b | (1ull << 63));
        break;
    }
    default:   // INT64, TIME, DATETIME, TIMESTAMP, DECIMAL64, and the two halves of DECIMAL128 {B0_63, B64_127}
        if (s.kind == SEG_D128_LO) v = reinterpret_cast<const uint64_t *>(s.col)[2 * r];
        else if (s.kind == SEG_D128_HI) v = reinterpret_cast<const uint64_t *>(s.col)[2 * r + 1] ^ (1ull << 63);
        else v = reinterpret_cast<const uint64_t *>(s.col)[r] ^ (1ull << 63);
    }
    if (s.desc) v = ~v;
    return s.bits == 64 ? v : (v & ((1ull << s.bits) - 1));
}

// The part of a SEG_BYTES segment that falls into one word, in place: p = the segment's first bit relative to the word's most significant
// bit (a multiple of 8, negative when the segment began in an earlier word).  Word byte j holds value byte j - p / 8, zero past the value.
__device__ __forceinline__ uint64_t bytes_image(const OrderSeg &s, uint64_t row, int p) {
    const uint64_t r = s.cst ? 0 : row;
    if (s.nulls && ((s.nulls[r >> 6] >> (r & 63)) & 1ull)) return 0;
    const VarlenaRef v = varlena_ref(s.col, r, s.area, s.area_sz);
    const int b0 = -p / 8, len = (int)v.len;
    uint64_t w = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) w = (w << 8) | ((b0 + j >= 0 && b0 + j < len) ? v.ptr[b0 + j] : 0u);
    if (s.desc) {
        const int end = p + s.bits;
        w = ~w & (p <= 0 ? ~0ull : ~0ull >> p) & (end >= 64 ? ~0ull : ~(~0ull >> end));
    }
    return w;
}

// word w (0 = most significant) of row `row`'s image
template <bool VAR>
__device__ __forceinline__ uint64_t order_word(const OrderSpec &S, int w, uint64_t row) {
    uint64_t word = 0;
    const int lo = 64 * w;
    for (int i = 0; i < S.nsegs; i++) {
        const OrderSeg &s = S.seg[i];
        const int p = s.off - lo, end = p + s.bits;       // the segment's bits relative to the word's most significant bit
        if (p >= 64 || end <= 0) continue;
        if (VAR && s.kind == SEG_BYTES) { word |= bytes_image(s, row, p); continue; }
        const uint64_t v = seg_image<VAR>(s, row);
        word |= end <= 64 ? (v << (64 - end)) : (v >> (end - 64));
    }
    return word;
}

// ---- the radix sort of (key word, uint32 row) pairs --------------------------------------------------------------------------------------
struct RadixState {
    unsigned long long hist[8][256];
    unsigned long long start[8][256];
    int src[8];          // buffer the pass of digit p reads, -1 = digit skipped
    int sel;             // buffer holding the current pairs
    int done;            // sort by rounds: every run holds one row, the remaining passes return at once
};
template <typename K> struct Pairs { K *k[2]; uint32_t *v[2]; };

struct SortScratch {
    RadixState *st;
    unsigned long long *status;   // per (tile, digit): epoch | flag | value
    unsigned *tickets;            // one tile counter per scatter launch
    int epoch, max_passes;
    uint64_t ntiles;
};
constexpr int kEpochShift = 42, kFlagShift = 40;
constexpr unsigned long long kValMask = (1ull << kFlagShift) - 1, kFlagAgg = 1, kFlagPre = 2;

// How the pass over a word gets its keys: ENCODE computes the word from the key columns (rows in row order, through a candidate list or
// through the current permutation), otherwise the keys are already in the current buffer.
struct NoEncode { };

template <typename K, bool ENCODE, bool VAR>
__global__ void __launch_bounds__(kThreads)
radix_hist_kernel(Pairs<K> B, const uint64_t *__restrict__ m_ptr, RadixState *st, bool first, const uint32_t *__restrict__ cand, OrderSpec S, int w) {
    __shared__ unsigned h[sizeof(K)][256];
    if (st->done) return;
    for (int i = threadIdx.x; i < (int)sizeof(K) * 256; i += kThreads) (&h[0][0])[i] = 0;
    __syncthreads();
    const uint64_t m = *m_ptr;
    const int sel = st->sel;
    K *kb = B.k[sel];
    uint32_t *vb = B.v[sel];
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < m; i += (uint64_t)gridDim.x * kThreads) {
        K key;
        if (ENCODE) {
            uint32_t row;
            if (first) { row = cand ? cand[i] : (uint32_t)i; vb[i] = row; }
            else row = vb[i];
            key = (K)order_word<VAR>(S, w, row);
            kb[i] = key;
        } else key = kb[i];
#pragma unroll
        for (int p = 0; p < (int)sizeof(K); p++) atomicAdd(&h[p][(key >> (8 * p)) & 255u], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (int)sizeof(K) * 256; i += kThreads) {
        const unsigned c = (&h[0][0])[i];
        if (c) atomicAdd(&(&st->hist[0][0])[i], (unsigned long long)c);
    }
}

// one CTA: global digit starts, which digits are skipped, and which buffer every pass reads
__global__ void __launch_bounds__(kThreads) radix_plan_kernel(const uint64_t *__restrict__ m_ptr, RadixState *st, int ndig) {
    __shared__ unsigned long long sw[kThreads / 32];
    __shared__ int skip[8];
    const uint64_t m = *m_ptr;
    const int d = threadIdx.x, lane = d & 31, warp = d >> 5;
    if (st->done) { if (d < ndig) st->src[d] = -1; return; }
    for (int p = 0; p < ndig; p++) {
        const unsigned long long c = st->hist[p][d];
        unsigned long long inc = c;
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) sw[warp] = inc;
        if (d == 0) skip[p] = 0;
        __syncthreads();
        unsigned long long base = 0;
        for (int q = 0; q < warp; q++) base += sw[q];
        st->start[p][d] = base + inc - c;
        if (c == m) skip[p] = 1;          // one bucket holds every row (also m == 0)
        __syncthreads();
    }
    if (d == 0) {
        int sel = st->sel;
        for (int p = 0; p < ndig; p++) {
            if (skip[p]) st->src[p] = -1;
            else { st->src[p] = sel; sel ^= 1; }
        }
        st->sel = sel;
    }
}

// one stable counting pass over digit p.  Persistent CTAs take 4096-row tiles in ticket order.
template <typename K>
__global__ void __launch_bounds__(kThreads)
radix_scatter_kernel(Pairs<K> B, const uint64_t *__restrict__ m_ptr, const RadixState *__restrict__ st, int p, unsigned long long *status,
                     unsigned *ticket, unsigned epoch) {
    extern __shared__ __align__(16) unsigned char smem[];
    K *skey = reinterpret_cast<K *>(smem);
    uint32_t *sval = reinterpret_cast<uint32_t *>(smem + kTile * sizeof(K));
    unsigned *whist = sval + kTile;                          // [warp][256]: per-warp digit counts, then their exclusive prefixes
    __shared__ unsigned s_tile;
    __shared__ unsigned lstart[256];                         // start of every digit inside the staged tile
    __shared__ unsigned long long gbase[256];                // global position of the tile's first row of every digit
    __shared__ unsigned s_wsum[kThreads / 32];
    const int src = st->src[p];
    if (src < 0) return;
    const K *kin = B.k[src];
    const uint32_t *vin = B.v[src];
    K *kout = B.k[src ^ 1];
    uint32_t *vout = B.v[src ^ 1];
    const uint64_t m = *m_ptr;
    const uint64_t ntiles = (m + kTile - 1) / kTile;
    const int shift = 8 * p;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned long long tag = (unsigned long long)epoch << kEpochShift;
    for (;;) {
        for (int i = threadIdx.x; i < (kThreads / 32) * 256; i += kThreads) whist[i] = 0;
        if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
        __syncthreads();
        const uint64_t tile = s_tile;
        if (tile >= ntiles) return;
        const uint64_t t0 = tile * kTile;
        const unsigned tn = (unsigned)(m - t0 < (uint64_t)kTile ? m - t0 : (uint64_t)kTile);
        K key[kIPT];
        unsigned off[kIPT];                                  // rank among the warp's rows of the same digit
        unsigned *wh = whist + warp * 256;
#pragma unroll
        for (int r = 0; r < kIPT; r++) {
            const unsigned j = warp * 32 * kIPT + r * 32 + lane;   // warp-contiguous chunks: rank order = input order
            const bool live = j < tn;
            key[r] = live ? kin[t0 + j] : (K)0;
            const unsigned d = live ? (unsigned)((key[r] >> shift) & 255u) : 256u;
            const unsigned peers = __match_any_sync(0xffffffffu, d);
            const unsigned below = __popc(peers & ((1u << lane) - 1u));
            off[r] = live ? wh[d] + below : 0u;
            __syncwarp();
            if (live && below == 0) wh[d] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();
        // thread d: per-warp prefixes of digit d, the tile's count of d, its place in the tile and (look-back) in the output
        const int d = threadIdx.x;
        unsigned cnt = 0;
#pragma unroll
        for (int q = 0; q < kThreads / 32; q++) { const unsigned c = whist[q * 256 + d]; whist[q * 256 + d] = cnt; cnt += c; }
        unsigned inc = cnt;
        for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) s_wsum[warp] = inc;
        unsigned long long excl = 0;
        unsigned long long *my = status + tile * 256 + d;
        if (tile == 0) atomicExch(my, tag | (kFlagPre << kFlagShift) | cnt);
        else {
            atomicExch(my, tag | (kFlagAgg << kFlagShift) | cnt);
            for (long long q = (long long)tile - 1; q >= 0; q--) {
                unsigned long long s;
                do { s = *((volatile unsigned long long *)&status[(uint64_t)q * 256 + d]); } while ((s >> kEpochShift) != epoch);
                excl += s & kValMask;
                if (((s >> kFlagShift) & 3ull) == kFlagPre) break;
            }
            atomicExch(my, tag | (kFlagPre << kFlagShift) | (excl + cnt));
        }
        __syncthreads();
        unsigned wbase = 0;
        for (int q = 0; q < warp; q++) wbase += s_wsum[q];
        const unsigned ls = wbase + inc - cnt;
        lstart[d] = ls;
        gbase[d] = st->start[p][d] + excl;
        __syncthreads();
#pragma unroll
        for (int r = 0; r < kIPT; r++) {
            const unsigned j = warp * 32 * kIPT + r * 32 + lane;
            if (j < tn) {
                const unsigned dd = (unsigned)((key[r] >> shift) & 255u);
                const unsigned pos = lstart[dd] + whist[warp * 256 + dd] + off[r];
                skey[pos] = key[r];
                sval[pos] = vin[t0 + j];                     // the rows are loaded only here: fewer live registers across the look-back
            }
        }
        __syncthreads();
        for (unsigned j = threadIdx.x; j < tn; j += kThreads) {   // the staged tile is digit-sorted: runs of one digit go out coalesced
            const K k = skey[j];
            const unsigned dd = (unsigned)((k >> shift) & 255u);
            const uint64_t g = gbase[dd] + (j - lstart[dd]);
            kout[g] = k;
            vout[g] = sval[j];
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads) sels_out_kernel(const uint32_t *v0, const uint32_t *v1, const RadixState *st, uint64_t n, int64_t *__restrict__ sels) {
    const uint32_t *v = st->sel ? v1 : v0;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) sels[i] = (int64_t)v[i];
}
__global__ void __launch_bounds__(kThreads) settle_kernel(uint32_t *v0, const uint32_t *v1, const RadixState *st, const uint64_t *m_ptr) {
    if (st->sel == 0) return;
    const uint64_t m = *m_ptr;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < m; i += (uint64_t)gridDim.x * kThreads) v0[i] = v1[i];
}

inline unsigned grid_for(uint64_t items) {
    uint64_t g = (items + kThreads - 1) / kThreads;
    const uint64_t mx = (uint64_t)num_sms() * 8;
    return (unsigned)(g > mx ? mx : (g ? g : 1));
}

// passes: the most scatter passes the sort will launch (8 per 64-bit word)
int scratch_init(ThreadCtx &t, uint64_t cap, int passes, SortScratch *S) {
    S->ntiles = (cap + kTile - 1) / kTile;
    S->max_passes = passes + 1;
    S->st = (RadixState *)arena_alloc(t, sizeof(RadixState));
    S->status = (unsigned long long *)arena_alloc(t, (S->ntiles ? S->ntiles : 1) * 256 * 8);
    S->tickets = (unsigned *)arena_alloc(t, (size_t)S->max_passes * 4);
    if (!S->st || !S->status || !S->tickets) return MO_RC_INTERNAL_ERROR;
    S->epoch = 0;
    MOB_CUDA_TRY(cudaMemsetAsync(S->st, 0, sizeof(RadixState), t.stream));
    MOB_CUDA_TRY(cudaMemsetAsync(S->status, 0, (S->ntiles ? S->ntiles : 1) * 256 * 8, t.stream));
    MOB_CUDA_TRY(cudaMemsetAsync(S->tickets, 0, (size_t)S->max_passes * 4, t.stream));
    return MO_RC_SUCCESS;
}

template <typename K>
int scatter_grid() {
    static int per_sm = 0;
    if (!per_sm) {
        const int smem = kTile * (int)(sizeof(K) + 4) + (kThreads / 32) * 256 * 4;
        cudaFuncSetAttribute(radix_scatter_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        int b = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, radix_scatter_kernel<K>, kThreads, smem) != cudaSuccess || b < 1) b = 1;
        per_sm = b;
    }
    return per_sm;
}

// one word: histogram (+ encode), plan, one scatter per digit.  The pairs end in buffer st->sel.
template <typename K, bool ENCODE, bool VAR>
int radix_word(ThreadCtx &t, SortScratch &S, Pairs<K> B, const uint64_t *m_ptr, uint64_t cap, bool first, const uint32_t *cand, const OrderSpec &spec, int w) {
    if (S.epoch + (int)sizeof(K) >= S.max_passes) { set_error("order: too many radix passes"); return MO_RC_INTERNAL_ERROR; }
    const int smem = kTile * (int)(sizeof(K) + 4) + (kThreads / 32) * 256 * 4;
    const int per_sm = scatter_grid<K>();
    MOB_CUDA_TRY(cudaMemsetAsync(S.st->hist, 0, sizeof(S.st->hist), t.stream));
    radix_hist_kernel<K, ENCODE, VAR><<<grid_for(cap), kThreads, 0, t.stream>>>(B, m_ptr, S.st, first, cand, spec, w);
    MOB_LAUNCH_CHECK();
    radix_plan_kernel<<<1, kThreads, 0, t.stream>>>(m_ptr, S.st, (int)sizeof(K));
    MOB_LAUNCH_CHECK();
    uint64_t g = (uint64_t)num_sms() * per_sm;
    if (g > S.ntiles) g = S.ntiles ? S.ntiles : 1;
    for (int p = 0; p < (int)sizeof(K); p++) {
        S.epoch++;
        radix_scatter_kernel<K><<<(unsigned)g, kThreads, smem, t.stream>>>(B, m_ptr, S.st, p, S.status, S.tickets + S.epoch, (unsigned)S.epoch);
        MOB_LAUNCH_CHECK();
    }
    return MO_RC_SUCCESS;
}

// ---- top-n: radix select on the first word ----------------------------------------------------------------------------------------------
struct SelectState { unsigned long long hist[256]; unsigned long long k; uint64_t prefix; int shift; int done; };
constexpr uint64_t kSelectEnough = 1ull << 16;    // stop refining once the bucket holding rank `limit` has at most this many rows

template <bool VAR>
__global__ void __launch_bounds__(kThreads) select_hist_kernel(OrderSpec S, uint64_t n, SelectState *ss) {
    __shared__ unsigned h[256];
    if (ss->done) return;
    h[threadIdx.x] = 0;
    __syncthreads();
    const int shift = ss->shift;
    const uint64_t prefix = ss->prefix;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        const uint64_t kw = order_word<VAR>(S, 0, i);
        if (shift == 56 || (kw >> (shift + 8)) == prefix) atomicAdd(&h[(kw >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&ss->hist[threadIdx.x], (unsigned long long)h[threadIdx.x]);
}
__global__ void __launch_bounds__(kThreads) select_pick_kernel(SelectState *ss) {
    __shared__ unsigned long long sw[kThreads / 32];
    if (ss->done) return;
    const int d = threadIdx.x, lane = d & 31, warp = d >> 5;
    const unsigned long long c = ss->hist[d], k = ss->k;
    unsigned long long inc = c;
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) sw[warp] = inc;
    __syncthreads();
    unsigned long long base = 0;
    for (int q = 0; q < warp; q++) base += sw[q];
    const unsigned long long before = base + inc - c;
    __syncthreads();
    ss->hist[d] = 0;
    if (c && before <= k && k < before + c) {     // exactly one bucket holds rank k
        const int shift = ss->shift;
        ss->k = k - before;
        ss->prefix = shift == 56 ? (uint64_t)d : ((ss->prefix << 8) | (uint64_t)d);
        if (c <= kSelectEnough || shift == 0) ss->done = 1;
        else ss->shift = shift - 8;
    }
}
template <bool VAR>
__global__ void __launch_bounds__(kThreads) select_flag_kernel(OrderSpec S, uint64_t n, const SelectState *ss, uint32_t *__restrict__ bits) {
    const int shift = ss->shift;
    const uint64_t prefix = ss->prefix;
    const uint64_t n32 = (n + 31) & ~31ull;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n32; i += (uint64_t)gridDim.x * kThreads) {
        const bool keep = i < n && (order_word<VAR>(S, 0, i) >> shift) <= prefix;
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if ((threadIdx.x & 31) == 0) bits[i >> 5] = b;
    }
}

// ---- varlena keys: the one read-back record (column.cuh), and the run numbers of a sort by rounds -----------------------------------------
__global__ void __launch_bounds__(kThreads)
varlena_stat_kernel(const uint8_t *__restrict__ cells, const uint64_t *__restrict__ nulls, const uint8_t *area, uint64_t area_sz, uint64_t n,
                    VarlenaStat *vs, int k) {
    unsigned mx = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        if (bm_test(nulls, i)) continue;
        const VarlenaRef v = varlena_ref(cells, i, area, area_sz);
        if (!v.ok) atomicMax(&vs->bad_inv[k], ~(unsigned long long)i);
        else mx = v.len > mx ? v.len : mx;
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0 && mx) atomicMax(&vs->maxlen[k], mx);
}

constexpr int kRunBlocks = 1024;   // the run numbering splits the rows into this many contiguous chunks

__device__ __forceinline__ void run_chunk(uint64_t m, uint64_t *i0, uint64_t *i1) {
    const uint64_t chunk = (m + kRunBlocks - 1) / kRunBlocks;
    *i0 = blockIdx.x * chunk;
    *i1 = *i0 + chunk < m ? *i0 + chunk : m;
}

// flag[i] = position i starts a run: its image differs from position i-1's in the word last sorted (kb: word w0 - 1 in the first round, the
// run number after) or in words [w0, w1).  cnt[chunk] = the chunk's flags.
__global__ void __launch_bounds__(kThreads)
run_flag_kernel(Pairs<uint64_t> B, const uint64_t *__restrict__ m_ptr, const RadixState *st, OrderSpec S, int w0, int w1, uint8_t *__restrict__ flag,
                unsigned long long *cnt) {
    __shared__ unsigned s_cnt;
    if (st->done) return;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    uint64_t i0, i1;
    run_chunk(*m_ptr, &i0, &i1);
    const uint64_t *kb = B.k[st->sel];
    const uint32_t *vb = B.v[st->sel];
    unsigned c = 0;
    for (uint64_t i = i0 + threadIdx.x; i < i1; i += kThreads) {
        bool f = i == 0 || kb[i] != kb[i - 1];
        for (int w = w0; !f && w < w1; w++) f = order_word<true>(S, w, vb[i]) != order_word<true>(S, w, vb[i - 1]);
        flag[i] = f;
        c += f;
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) cnt[blockIdx.x] = s_cnt;
}

// one CTA: cnt becomes the exclusive prefix over the chunks; as many runs as rows -> done
__global__ void __launch_bounds__(kThreads) run_scan_kernel(const uint64_t *__restrict__ m_ptr, RadixState *st, unsigned long long *cnt) {
    constexpr int kPer = kRunBlocks / kThreads;
    __shared__ unsigned long long sw[kThreads / 32];
    if (st->done) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long v[kPer], sum = 0;
#pragma unroll
    for (int j = 0; j < kPer; j++) { v[j] = cnt[threadIdx.x * kPer + j]; sum += v[j]; }
    unsigned long long inc = sum;
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) sw[warp] = inc;
    __syncthreads();
    unsigned long long base = 0, total = 0;
    for (int q = 0; q < kThreads / 32; q++) { if (q < warp) base += sw[q]; total += sw[q]; }
    base += inc - sum;
#pragma unroll
    for (int j = 0; j < kPer; j++) { cnt[threadIdx.x * kPer + j] = base; base += v[j]; }
    if (threadIdx.x == 0 && total == *m_ptr) st->done = 1;
}

// run[row] = the 0-based run of the row's position: base of the chunk + flags up to and including the position - 1
__global__ void __launch_bounds__(kThreads)
run_number_kernel(Pairs<uint64_t> B, const uint64_t *__restrict__ m_ptr, const RadixState *st, const uint8_t *__restrict__ flag,
                  const unsigned long long *__restrict__ base, uint32_t *__restrict__ run) {
    __shared__ unsigned sw[kThreads / 32];
    if (st->done) return;
    uint64_t i0, i1;
    run_chunk(*m_ptr, &i0, &i1);
    const uint32_t *vb = B.v[st->sel];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long carry = base[blockIdx.x];
    for (uint64_t t0 = i0; t0 < i1; t0 += kThreads) {
        const uint64_t i = t0 + threadIdx.x;
        const unsigned f = i < i1 ? flag[i] : 0u;
        unsigned inc = f;
        for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) sw[warp] = inc;
        __syncthreads();
        unsigned wbase = 0, tot = 0;
        for (int q = 0; q < kThreads / 32; q++) { if (q < warp) wbase += sw[q]; tot += sw[q]; }
        if (i < i1) run[vb[i]] = (uint32_t)(carry + wbase + inc - 1);
        carry += tot;
        __syncthreads();
    }
}

}  // namespace

namespace mob {

int varlena_stats(ThreadCtx &t, const Operand *col, const int *type, int n, uint64_t len, VarlenaStat *vs) {
    for (int k = 0; k < n; k++) {
        if (!is_varlena(type[k])) continue;
        const Operand &c = col[k];
        const uint64_t rows = c.cst ? 1 : len;
        varlena_stat_kernel<<<grid_for(rows), kThreads, 0, t.stream>>>((const uint8_t *)c.data, c.nulls, c.area, c.area_sz, rows, vs, k);
        MOB_LAUNCH_CHECK();
    }
    return MO_RC_SUCCESS;
}

int varlena_stat_error(const VarlenaStat &vs, int ncols, const char *what) {
    for (int k = 0; k < ncols; k++) {
        if (vs.bad_inv[k]) { set_error("%s %d row %llu: the varlena cell points outside the area", what, k, ~vs.bad_inv[k]); return MO_RC_INVALID_ARGUMENT; }
        if (vs.maxlen[k] > MO_ORDER_MAX_VARLENA) { set_error("%s %d has a %u-byte value, at most %d supported", what, k, vs.maxlen[k], MO_ORDER_MAX_VARLENA); return MO_RC_INVALID_ARGUMENT; }
    }
    return MO_RC_SUCCESS;
}

// Stable sort of m (device count, <= cap) pairs (k[0][i], v[0][i]) by the 32-bit key; the sorted rows end in v[0].  Used by JOIN_SELS and
// the k-means centroid update (group_rows_stable, join.cu).
int sort_u32_pairs(ThreadCtx &t, uint32_t *k0, uint32_t *v0, uint32_t *k1, uint32_t *v1, const uint64_t *m_ptr, uint64_t cap) {
    SortScratch S;
    int rc = scratch_init(t, cap, (int)sizeof(uint32_t), &S);
    if (rc) return rc;
    Pairs<uint32_t> B{{k0, k1}, {v0, v1}};
    OrderSpec none;
    none.nsegs = 0; none.nwords = 0;
    rc = radix_word<uint32_t, false, false>(t, S, B, m_ptr, cap, true, nullptr, none, 0);
    if (rc) return rc;
    settle_kernel<<<grid_for(cap), kThreads, 0, t.stream>>>(v0, v1, S.st, m_ptr);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

// MO_XCALL_ORDER_SELS: args [0] sels int64[min(limit, len)] ; [1] mo_order_params_t ; [2 .. 2+nkeys) key columns (+pnulls; one element =
// const) ; [2+nkeys] int64 row ids [len] when has_row_ids.  len = rows.
int xcall_order_sels(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    mo_order_params_t P;
    if (int rc = read_param(t, args[1], &P, sizeof P, sizeof P, "order sels: mo_order_params_t")) return rc;
    if (P.nkeys < 1 || P.nkeys > MO_ORDER_MAX_KEYS) { set_error("order sels: %d keys (1..%d)", P.nkeys, MO_ORDER_MAX_KEYS); return MO_RC_INVALID_ARGUMENT; }
    if (len >= (1ull << 32)) { set_error("order sels: %llu rows, at most 2^32 - 1 per call", (unsigned long long)len); return MO_RC_INVALID_ARGUMENT; }
    const uint64_t nout = (P.limit < 0 || (uint64_t)P.limit >= len) ? len : (uint64_t)P.limit;
    if (args[0].dataSz < 8 * nout || (nout && !args[0].pdata)) { set_error("order sels: the sels buffer holds %llu rows, %llu needed", (unsigned long long)(args[0].dataSz / 8), (unsigned long long)nout); return MO_RC_INVALID_ARGUMENT; }
    const mo_xcall_args_t *rid = P.has_row_ids ? &args[2 + P.nkeys] : nullptr;
    if (rid && (rid->dataSz < 8 * len || (len && !rid->pdata))) { set_error("order sels: row ids shorter than len"); return MO_RC_INVALID_ARGUMENT; }
    OrderSpec spec;
    memset(&spec, 0, sizeof spec);
    int bit = 0, ns = 0;
    Stager st(t);
    OrderSeg base[MO_ORDER_MAX_KEYS];
    Operand key[MO_ORDER_MAX_KEYS];
    int type[MO_ORDER_MAX_KEYS];
    bool has_var = false, ext = false;   // ext: a varlena or UUID key, order_word<true>
    for (int k = 0; k < P.nkeys; k++) {
        const mo_xcall_args_t &a = args[2 + k];
        const int T = type[k] = P.key[k].col_type, fl = P.key[k].flags;
        const bool var = is_varlena(T);
        const uint64_t esz = key_elem_size(T);
        if (!esz) { st.finish(); set_error("order sels: key %d has unsupported type %d", k, T); return MO_RC_INVALID_ARGUMENT; }
        if (!is_const(a, esz, len) && a.dataSz < esz * len) { st.finish(); set_error("order sels: key %d holds %llu bytes, %llu needed", k, (unsigned long long)a.dataSz, (unsigned long long)(esz * len)); return MO_RC_INVALID_ARGUMENT; }
        if (!a.pdata && (len || a.dataSz == esz)) { st.finish(); set_error("order sels: key %d has no data", k); return MO_RC_INVALID_ARGUMENT; }
        // the checks above are the call's own; stage_operand's size check cannot fail after them
        if (len) { if (int rc = stage_operand(st, a, esz, len, "order sels", 2 + k, key[k])) return rc; }
        const bool desc = (fl & MO_ORDER_DESC) != 0;
        const bool nulls_last = (fl & MO_ORDER_NULLS_FIRST) ? false : (fl & MO_ORDER_NULLS_LAST) ? true : desc;
        OrderSeg &b = base[k];
        b = OrderSeg{};
        // BIT, YEAR and ENUM order as their storage types uint64, int16 and uint16
        b.col = (const uint8_t *)key[k].data; b.nulls = key[k].nulls; b.area = key[k].area; b.area_sz = key[k].area_sz; b.cst = key[k].cst;
        b.type = T == MO_T_BIT ? MO_T_UINT64 : T == MO_T_YEAR ? MO_T_INT16 : T == MO_T_ENUM ? MO_T_UINT16 : T; b.desc = desc; b.nulls_last = nulls_last; b.bits = 8 * (int)esz;
        has_var = has_var || var;
        ext = ext || var || T == MO_T_UUID;
    }
    // varlena keys: the longest value of every key and its lowest bad cell, read back -- the image layout depends on the longest value
    VarlenaStat vstat{};
    if (has_var && len) {
        VarlenaStat *vs = (VarlenaStat *)st.tmp(sizeof(VarlenaStat));
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        MOB_CUDA_TRY(cudaMemsetAsync(vs, 0, sizeof(VarlenaStat), t.stream));
        int rc = varlena_stats(t, key, type, P.nkeys, len, vs);
        if (rc) { st.finish(); return rc; }
        rc = read_back(t, &vstat, vs, sizeof vstat);
        if (rc) { st.finish(); return rc; }
        rc = varlena_stat_error(vstat, P.nkeys, "order sels: key");
        if (rc) { st.finish(); return rc; }
    }
    for (int k = 0; k < P.nkeys; k++) {
        const OrderSeg &b = base[k];
        if (b.nulls) { OrderSeg s = b; s.kind = SEG_NULL; s.bits = 1; s.off = bit; bit += 1; spec.seg[ns++] = s; }
        if (is_varlena(b.type)) {   // bytes, zero-padded to the longest value, then the length: bytes.Compare
            const unsigned L = vstat.maxlen[k];
            if (!L) continue;        // every value empty or NULL
            bit = (bit + 7) & ~7;
            OrderSeg by = b; by.kind = SEG_BYTES; by.bits = 8 * (int)L; by.off = bit; bit += by.bits; spec.seg[ns++] = by;
            OrderSeg ln = b; ln.kind = SEG_LEN; ln.bits = 32 - __builtin_clz(L); ln.off = bit; bit += ln.bits; spec.seg[ns++] = ln;
        } else if (b.bits == 128) {
            OrderSeg hi = b; hi.kind = SEG_D128_HI; hi.bits = 64; hi.off = bit; bit += 64; spec.seg[ns++] = hi;
            OrderSeg lo = b; lo.kind = SEG_D128_LO; lo.bits = 64; lo.off = bit; bit += 64; spec.seg[ns++] = lo;
        } else { OrderSeg s = b; s.kind = SEG_VALUE; s.off = bit; bit += b.bits; spec.seg[ns++] = s; }
    }
    int nwords = (bit + 63) / 64;
    if (rid) {
        OrderSeg s{};
        s.col = (const uint8_t *)st.in(rid->pdata, 8 * len); s.kind = SEG_ROWID; s.bits = 64; s.off = 64 * nwords;
        spec.seg[ns++] = s;
        nwords++;
    }
    if (!nwords) nwords = 1;   // only varlena keys whose every value is empty or NULL: one all-zero word keeps the rows in order
    spec.nsegs = ns; spec.nwords = nwords;
    int64_t *sels = (int64_t *)st.out(args[0].pdata, 8 * nout);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    if (nout == 0) return st.complete();

    // Top: the candidate rows of the limit-th first word, in row order; Order: every row
    const bool top = nout < len / 8;
    const uint32_t *cand = nullptr;
    uint64_t *m_ptr = (uint64_t *)st.tmp(16);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    cudaEventRecord(t.kev0, t.stream);
    if (top) {
        SelectState *ss = (SelectState *)st.tmp(sizeof(SelectState));
        uint32_t *bits = (uint32_t *)st.tmp(((len + 63) / 64) * 8);
        uint32_t *c = (uint32_t *)st.tmp(len * 4 + 16);
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        SelectState init{};
        init.k = nout - 1; init.shift = 56;
        MOB_CUDA_TRY(cudaMemcpyAsync(ss, &init, sizeof init, cudaMemcpyHostToDevice, t.stream));
        for (int level = 0; level < 8; level++) {
            if (ext) select_hist_kernel<true><<<grid_for(len), kThreads, 0, t.stream>>>(spec, len, ss);
            else select_hist_kernel<false><<<grid_for(len), kThreads, 0, t.stream>>>(spec, len, ss);
            MOB_LAUNCH_CHECK();
            select_pick_kernel<<<1, kThreads, 0, t.stream>>>(ss);
            MOB_LAUNCH_CHECK();
        }
        if (ext) select_flag_kernel<true><<<grid_for(len), kThreads, 0, t.stream>>>(spec, len, ss, bits);
        else select_flag_kernel<false><<<grid_for(len), kThreads, 0, t.stream>>>(spec, len, ss, bits);
        MOB_LAUNCH_CHECK();
        int rc = compact_bits(t, bits, len, (int32_t *)c, (unsigned long long *)m_ptr);
        if (rc) { st.finish(); return rc; }
        cand = c;
    } else {
        MOB_CUDA_TRY(cudaMemcpyAsync(m_ptr, &len, 8, cudaMemcpyHostToDevice, t.stream));
    }
    Pairs<uint64_t> B;
    B.k[0] = (uint64_t *)st.tmp(len * 8); B.k[1] = (uint64_t *)st.tmp(len * 8);
    B.v[0] = (uint32_t *)st.tmp(len * 4); B.v[1] = (uint32_t *)st.tmp(len * 4);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    // One LSD round over every word, or -- varlena keys with a long image -- rounds of kRoundWords words, most significant first: each round
    // after the first sorts by (run number, its words), and the device stops sorting once every run holds one row.
    const bool rounds = has_var && nwords > kRoundWords;
    const int nrounds = rounds ? (nwords + kRoundWords - 1) / kRoundWords : 1;
    SortScratch S;
    int rc = scratch_init(t, len, 8 * (nwords + nrounds - 1), &S);
    if (rc) { st.finish(); return rc; }
    if (!rounds) {
        for (int w = nwords - 1; w >= 0; w--) {
            rc = ext ? radix_word<uint64_t, true, true>(t, S, B, m_ptr, len, w == nwords - 1, cand, spec, w)
                     : radix_word<uint64_t, true, false>(t, S, B, m_ptr, len, w == nwords - 1, cand, spec, w);
            if (rc) { st.finish(); return rc; }
        }
    } else {
        uint8_t *flag = (uint8_t *)st.tmp(len);
        unsigned long long *cnt = (unsigned long long *)st.tmp(kRunBlocks * 8);
        uint32_t *run = (uint32_t *)st.tmp(len * 4);
        if (st.failed) return MO_RC_INTERNAL_ERROR;
        OrderSpec runspec;
        memset(&runspec, 0, sizeof runspec);
        runspec.seg[0].col = (const uint8_t *)run; runspec.seg[0].kind = SEG_RUN; runspec.seg[0].bits = 32;
        runspec.nsegs = 1; runspec.nwords = 1;
        for (int a = 0; a < nwords; a += kRoundWords) {
            const int b = a + kRoundWords < nwords ? a + kRoundWords : nwords;
            for (int w = b - 1; w >= a; w--) {
                rc = radix_word<uint64_t, true, true>(t, S, B, m_ptr, len, a == 0 && w == b - 1, cand, spec, w);
                if (rc) { st.finish(); return rc; }
            }
            if (a) {
                rc = radix_word<uint64_t, true, true>(t, S, B, m_ptr, len, false, nullptr, runspec, 0);
                if (rc) { st.finish(); return rc; }
            }
            if (b == nwords) break;
            run_flag_kernel<<<kRunBlocks, kThreads, 0, t.stream>>>(B, m_ptr, S.st, spec, a ? a : 1, b, flag, cnt);
            MOB_LAUNCH_CHECK();
            run_scan_kernel<<<1, kThreads, 0, t.stream>>>(m_ptr, S.st, cnt);
            MOB_LAUNCH_CHECK();
            run_number_kernel<<<kRunBlocks, kThreads, 0, t.stream>>>(B, m_ptr, S.st, flag, cnt, run);
            MOB_LAUNCH_CHECK();
        }
    }
    sels_out_kernel<<<grid_for(nout), kThreads, 0, t.stream>>>(B.v[0], B.v[1], S.st, nout, sels);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return st.complete();
}

}  // namespace mob
