// vecdecode.cu -- the second half of "block decode -> device" (SURVEY.md section 8(f)-2): a decompressed column block is a marshalled
// vector.Vector (Vector.MarshalBinary / UnmarshalBinary, pkg/container/vector/vector.go:718-819):
//
//     [0]        class        uint8   (0 FLAT, 1 CONSTANT, vector.go:36-39)
//     [1, 17)    types.Type   16 bytes {Oid u8, Charset u8, notNull u8, dummy u8, Size i32, Width i32, Scale i32} (types.go:110-126, TSize encoding.go:35)
//     [17, 21)   length       uint32
//     [21, 25)   dataLen      uint32, then the data bytes
//                areaLen      uint32, then the area bytes (varlena payloads)
//                nspLen       uint32, then the nulls bitmap as bitmap.Marshal wrote it (bitmap.go:395-404): count i64, len u64, size u64, words
//                sorted       uint8
//
// The fields sit at byte offsets that are not aligned for their element type (the data starts at byte 25), so a view is not enough: one thread
// parses the header into a descriptor, then the whole grid copies data / area / nulls to the caller's ALIGNED device buffers (unaligned 8-byte
// reads assembled from two aligned words).  After this call the column is an ordinary resident vector every XCall entry point takes.
// A malformed header (lengths past the buffer, a bitmap longer than its section) fails the call.
#include "common.cuh"
#include <cstring>

namespace mob {
namespace {

constexpr int kThreads = 256;

struct Sections { uint64_t data_off, data_len, area_off, area_len, words_off, words_len; int bad; };

__device__ __forceinline__ uint32_t rd_u32(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint64_t rd_u64(const uint8_t *p) { return (uint64_t)rd_u32(p) | ((uint64_t)rd_u32(p + 4) << 32); }

__global__ void vec_parse_kernel(const uint8_t *__restrict__ src, uint64_t n, mo_vector_view_t *__restrict__ view, Sections *__restrict__ S) {
    if (blockIdx.x || threadIdx.x) return;
    mo_vector_view_t V; memset(&V, 0, sizeof V);
    Sections s; memset(&s, 0, sizeof s);
    uint64_t o = 0;
    bool bad = n < 1 + 16 + 4 + 4;
    if (!bad) {
        V.vclass = src[0];
        V.oid = src[1]; V.size = (int32_t)rd_u32(src + 5); V.width = (int32_t)rd_u32(src + 9); V.scale = (int32_t)rd_u32(src + 13);
        V.length = rd_u32(src + 17);
        s.data_len = rd_u32(src + 21); s.data_off = 25;
        o = 25 + s.data_len;
        bad = o + 4 > n;
    }
    if (!bad) { s.area_len = rd_u32(src + o); s.area_off = o + 4; o = s.area_off + s.area_len; bad = o + 4 > n; }
    if (!bad) {
        const uint64_t nsp_len = rd_u32(src + o); o += 4;
        bad = o + nsp_len + 1 > n;
        if (!bad && nsp_len) {
            if (nsp_len < 24) bad = true;
            else {
                V.null_count = (int64_t)rd_u64(src + o);
                const uint64_t bytes = rd_u64(src + o + 16);
                // compared as bytes > nsp_len - 24 (nsp_len >= 24 here): 24 + bytes wraps for a size field near 2^64 and would pass a bitmap
                // that runs far past its section
                if (bytes > nsp_len - 24 || (bytes & 7)) bad = true;
                else { s.words_off = o + 24; s.words_len = bytes / 8; }
            }
        }
        if (!bad) V.sorted = src[o + nsp_len];
    }
    V.data_len = s.data_len; V.area_len = s.area_len; V.nulls_words = ((uint64_t)V.length + 63) / 64;
    s.bad = bad ? 1 : 0;
    V.bad = s.bad;
    *view = V; *S = s;
}

// dst[0 .. len) = src[off .. off + len) with dst 16-byte aligned and src at any byte offset: 8 bytes per thread per step
__device__ __forceinline__ void copy_unaligned(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, uint64_t len, uint64_t tid, uint64_t nthreads) {
    const uint64_t nwords = len / 8;
    const unsigned sh = (unsigned)((uintptr_t)src & 7) * 8;
    const uint64_t *base = reinterpret_cast<const uint64_t *>((uintptr_t)src & ~(uintptr_t)7);
    for (uint64_t w = tid; w < nwords; w += nthreads) {
        uint64_t v = base[w] >> sh;
        if (sh) v |= base[w + 1] << (64 - sh);            // base[w + 1] holds at least one byte of this word: inside the buffer
        reinterpret_cast<uint64_t *>(dst)[w] = v;
    }
    for (uint64_t i = nwords * 8 + tid; i < len; i += nthreads) dst[i] = src[i];
}

__global__ void __launch_bounds__(kThreads) vec_copy_kernel(const uint8_t *__restrict__ src, const Sections *__restrict__ Sp, uint8_t *data, uint64_t data_cap, uint8_t *area,
                                                            uint64_t area_cap, uint64_t *nulls, uint64_t nulls_cap_words, uint64_t want_words, int *overflow) {
    const Sections S = *Sp;
    if (S.bad) return;
    const uint64_t tid = blockIdx.x * (uint64_t)kThreads + threadIdx.x, nthreads = (uint64_t)gridDim.x * kThreads;
    if (S.data_len > data_cap || S.area_len > area_cap || (nulls && want_words > nulls_cap_words)) { if (tid == 0) *overflow = 1; return; }
    if (S.data_len) copy_unaligned(data, src + S.data_off, S.data_len, tid, nthreads);
    if (S.area_len) copy_unaligned(area, src + S.area_off, S.area_len, tid, nthreads);
    if (nulls) {
        for (uint64_t w = tid; w < want_words; w += nthreads) nulls[w] = w < S.words_len ? rd_u64(src + S.words_off + 8 * w) : 0ull;
    }
}

}  // namespace

// MO_XCALL_VECTOR_UNMARSHAL: args [0] mo_vector_view_t (out; host or device) ; [1] data bytes (out, 16-byte aligned capacity) ; [2] area bytes (out) ;
// [3] nulls uint64 words (out: (length + 63) / 64 words, zero where the marshalled bitmap is shorter; pdata NULL: the caller does not want them) ;
// [4] the marshalled vector bytes (dataSz = their length).  len is ignored.
int xcall_vector_unmarshal(mo_xcall_args_t *args, uint64_t len) {
    (void)len;
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!args[0].pdata || args[0].dataSz < sizeof(mo_vector_view_t) || !args[4].pdata) { set_error("vector unmarshal: view or source missing"); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    const uint8_t *src;
    if (is_device_ptr(args[4].pdata)) src = (const uint8_t *)args[4].pdata;
    else {   // staged with 16 spare bytes: the unaligned word reads may touch the word after the last byte
        uint8_t *tmp = (uint8_t *)st.tmp(args[4].dataSz + 16);
        if (!tmp) { st.finish(); return MO_RC_INTERNAL_ERROR; }
        MOB_CUDA_TRY(cudaMemcpyAsync(tmp, args[4].pdata, args[4].dataSz, cudaMemcpyHostToDevice, t.stream));
        src = tmp;
    }
    mo_vector_view_t *view = (mo_vector_view_t *)st.out(args[0].pdata, sizeof(mo_vector_view_t));
    uint8_t *data = (uint8_t *)st.out(args[1].pdata, args[1].dataSz);
    uint8_t *area = (uint8_t *)st.out(args[2].pdata, args[2].dataSz);
    uint64_t *nulls = (uint64_t *)st.out(args[3].pdata, args[3].dataSz);
    Sections *S = (Sections *)st.tmp(sizeof(Sections));
    int *overflow = (int *)st.tmp(8);
    mo_vector_view_t *dview = (mo_vector_view_t *)st.tmp(sizeof(mo_vector_view_t));
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(overflow, 0, 8, t.stream));
    vec_parse_kernel<<<1, 32, 0, t.stream>>>(src, args[4].dataSz, dview, S);
    MOB_LAUNCH_CHECK();
    mo_vector_view_t V;
    int rc = read_back(t, &V, dview, sizeof V);
    if (rc) { st.finish(); return rc; }
    if (V.bad) { st.finish(); set_error("vector unmarshal: malformed vector bytes (a section runs past the buffer)"); return MO_RC_INVALID_ARGUMENT; }
    const uint64_t big = V.data_len + V.area_len + V.nulls_words * 8;
    uint64_t grid = (big / 8 + kThreads - 1) / kThreads;
    if (grid > (uint64_t)num_sms() * 8) grid = (uint64_t)num_sms() * 8;
    if (grid < 1) grid = 1;
    cudaEventRecord(t.kev0, t.stream);
    vec_copy_kernel<<<(unsigned)grid, kThreads, 0, t.stream>>>(src, S, data, args[1].dataSz, area, args[2].dataSz, nulls, args[3].dataSz / 8, V.nulls_words, overflow);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    MOB_CUDA_TRY(cudaMemcpyAsync(view, dview, sizeof V, cudaMemcpyDeviceToDevice, t.stream));
    int ov = 0;
    rc = read_back(t, &ov, overflow, 4);
    int frc = st.finish();
    if (rc) return rc;
    if (ov) { set_error("vector unmarshal: output buffers too small (data %llu, area %llu bytes, %llu null words)", (unsigned long long)V.data_len, (unsigned long long)V.area_len, (unsigned long long)V.nulls_words); return MO_RC_INVALID_ARGUMENT; }
    return frc;
}

}  // namespace mob
