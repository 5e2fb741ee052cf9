// lz4.cu -- LZ4 block decompression of column blocks on the device (SURVEY.md section 8(f)-2: "block decode -> device").
//
// Reference: pkg/compress/compress.go:37-47 (Decompress = lz4.UncompressBlock of github.com/pierrec/lz4/v4 v4.1.21, go.mod:73) as called by the
// object reader for every column block (pkg/objectio).  The Go module is a third-party dependency that is not part of /root/reference; the LZ4
// BLOCK format itself is published (lz4_Block_format.md): a block is a series of sequences
//     token (hi nibble: literal length, lo nibble: match length - 4; 15 = continued in 255-terminated extension bytes)
//     literals, 2-byte little-endian match offset (1 .. 65535, back from the write position), match copy (may overlap itself)
// and the last sequence ends after its literals.  The restatement is pinned against liblz4 (pyarrow's lz4_raw codec) in the tests.
//
// Mapping: a block is inherently sequential, a table scan has thousands of them: ONE WARP PER BLOCK.  All lanes parse the token stream
// redundantly (uniform control flow, broadcast loads); literal and match copies are cooperative, lane l takes bytes l, l + 32, ...; an
// overlapping match (offset < length) is a periodic pattern, byte i of the match is byte (i mod offset) of the last `offset` output bytes, so it is
// copied in parallel too.  A __syncwarp() between sequences orders the output bytes a later match reads.  Malformed input (offset 0 or before the
// block, lengths past either buffer, decoded size != the descriptor's) fails the call and names the block.
// Algorithmic bytes per block: compressed bytes in + decoded bytes out.
#include "common.cuh"
#include <cstring>

namespace mob {
namespace {

constexpr int kWarpsPerCta = 8;

// The token stream is read through a per-warp shared-memory WINDOW of the compressed block (kWin bytes, refilled cooperatively with 16-byte loads
// when the cursor runs past it): a sequence costs a handful of dependent byte reads (token, length extensions, offset), and from global memory each
// of them is a full memory latency (measured: 14 MB/s per warp, 27 GB/s for 2000 blocks); from shared memory they are ~30 cycles.
constexpr int kWin = 512;

struct SrcWin {
    const uint8_t *src; int64_t sl; unsigned char *buf; int64_t base;   // buf holds src[base .. base + kWin) (base is 16-byte aligned in ABSOLUTE address terms)
    __device__ __forceinline__ void fill(int64_t ip, unsigned lane) {
        const uintptr_t a0 = (uintptr_t)(src + ip) & ~(uintptr_t)15;
        base = (int64_t)(a0 - (uintptr_t)src);                            // may be slightly negative for the first window of an unaligned block
        __syncwarp();
        for (int i = lane * 16; i < kWin; i += 32 * 16) {
            const int64_t o = base + i;
            int4 v = make_int4(0, 0, 0, 0);
            if (o >= 0 && o + 16 <= sl) v = *reinterpret_cast<const int4 *>(src + o);
            else { unsigned char t[16]; for (int k = 0; k < 16; k++) t[k] = (o + k >= 0 && o + k < sl) ? src[o + k] : 0; memcpy(&v, t, 16); }
            *reinterpret_cast<int4 *>(buf + i) = v;
        }
        __syncwarp();
    }
    __device__ __forceinline__ unsigned byte(int64_t ip, unsigned lane) {   // src[ip], ip < sl
        if (ip - base >= kWin) fill(ip, lane);
        return buf[ip - base];
    }
};

// The OUTPUT goes through shared memory too: a match reads bytes the warp wrote a moment ago, and from global memory that is an L2 round trip per
// sequence (the measured bound once the token stream was in shared memory: ~0.6 us per sequence per warp).  Every output byte is written to the
// block in global memory AND to a per-warp ring of the last kRing bytes; matches whose source lies inside the ring (offset <= kRing: the common
// case in column data, where a value repeats its neighbours' bytes) are served from it, farther ones from global memory.
constexpr int kRing = 4096;    // 4.5 KB of shared memory per warp: up to 48 warps (= blocks in flight) per SM
constexpr size_t kLz4Smem = (size_t)kWarpsPerCta * (kWin + kRing);

__global__ void __launch_bounds__(32 * kWarpsPerCta)
lz4_decode_kernel(uint8_t *__restrict__ dst_base, uint64_t dst_cap, const uint8_t *__restrict__ src_base, uint64_t src_cap, const int64_t *__restrict__ desc, uint64_t nblocks,
                  unsigned long long *first_bad) {
    extern __shared__ __align__(16) unsigned char lz4_smem[];
    unsigned char (*win)[kWin] = reinterpret_cast<unsigned char (*)[kWin]>(lz4_smem);
    unsigned char *ring = lz4_smem + (size_t)kWarpsPerCta * kWin + (size_t)(threadIdx.x >> 5) * kRing;
    const unsigned lane = threadIdx.x & 31;
    const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t b = warp; b < nblocks; b += nwarps) {
        const int64_t so = desc[4 * b], sl = desc[4 * b + 1], dof = desc[4 * b + 2], dl = desc[4 * b + 3];
        bool bad = so < 0 || sl < 0 || dof < 0 || dl < 0 || (uint64_t)so + (uint64_t)sl > src_cap || (uint64_t)dof + (uint64_t)dl > dst_cap;
        if (!bad) {
            const uint8_t *src = src_base + so;
            volatile uint8_t *dst = dst_base + dof;
            SrcWin W{src, sl, win[threadIdx.x >> 5], 0};
            int64_t ip = 0, op = 0;
            if (sl == 0) bad = dl != 0;
            else W.fill(0, lane);
            while (!bad && ip < sl) {
                const unsigned token = W.byte(ip++, lane);
                int64_t lit = token >> 4;
                if (lit == 15) { unsigned e; do { if (ip >= sl) { bad = true; break; } e = W.byte(ip++, lane); lit += e; } while (e == 255); }
                if (bad || ip + lit > sl || op + lit > dl) { bad = true; break; }
                if (lit) {
                    if (ip + lit - W.base > kWin && lit <= kWin - 16) W.fill(ip, lane);           // bring the whole literal run into the window when it fits
                    if (ip + lit - W.base <= kWin) { for (int64_t i = lane; i < lit; i += 32) { const unsigned char v = W.buf[ip - W.base + i]; dst[op + i] = v; ring[(op + i) & (kRing - 1)] = v; } }
                    else { __syncwarp(); for (int64_t i = lane; i < lit; i += 32) { const unsigned char v = src[ip + i]; dst[op + i] = v; ring[(op + i) & (kRing - 1)] = v; } }   // a long run (incompressible data): straight from global memory (it may wrap the ring: the previous match must be done reading)
                }
                ip += lit; op += lit;
                if (ip >= sl) break;                                   // the last sequence: literals only
                if (ip + 2 > sl) { bad = true; break; }
                const int64_t offset = (int64_t)W.byte(ip, lane) | ((int64_t)W.byte(ip + 1, lane) << 8);
                ip += 2;
                int64_t mlen = token & 15;
                if (mlen == 15) { unsigned e; do { if (ip >= sl) { bad = true; break; } e = W.byte(ip++, lane); mlen += e; } while (e == 255); }
                mlen += 4;
                if (bad || offset == 0 || offset > op || op + mlen > dl) { bad = true; break; }
                __syncwarp();                                          // the bytes this match reads were written by other lanes
                const int64_t from = op - offset;
                // (an overlapping match, offset < length, is periodic with period `offset`: byte i is byte i mod offset of the last `offset` output bytes)
                if (offset <= kRing && mlen <= kRing - offset) {
                    // source [from, op) and destination [op, op + mlen) occupy disjoint ring slots (offset + mlen <= kRing): no ordering needed inside the copy
                    if (offset >= mlen) { for (int64_t i = lane; i < mlen; i += 32) { const unsigned char v = ring[(from + i) & (kRing - 1)]; dst[op + i] = v; ring[(op + i) & (kRing - 1)] = v; } }
                    else { for (int64_t i = lane; i < mlen; i += 32) { const unsigned char v = ring[(from + (i % offset)) & (kRing - 1)]; dst[op + i] = v; ring[(op + i) & (kRing - 1)] = v; } }
                } else {   // a far or very long match: its source is (or would get) evicted from the ring -> read the block in global memory
                    if (offset >= mlen) { for (int64_t i = lane; i < mlen; i += 32) { const unsigned char v = dst[from + i]; dst[op + i] = v; ring[(op + i) & (kRing - 1)] = v; } }
                    else { for (int64_t i = lane; i < mlen; i += 32) { const unsigned char v = dst[from + (i % offset)]; dst[op + i] = v; ring[(op + i) & (kRing - 1)] = v; } }
                }
                op += mlen;
                // the next sequence's literal copy writes ring slots that are at most kWin + its length ahead: it can only collide with this match's
                // reads when the match reached back almost a whole ring; otherwise the __syncwarp() before the next match orders everything
                if (offset + mlen + 2 * kWin > kRing) __syncwarp();
            }
            if (!bad && op != dl) bad = true;
        }
        if (bad && lane == 0) atomicMin(first_bad, (unsigned long long)b);
        __syncwarp();
    }
}

}  // namespace

// MO_XCALL_LZ4_DECODE: args [0] dst bytes ; [1] src bytes ; [2] descriptors int64[4 * len]: {src_off, src_len, dst_off, dst_len} per block.  len = blocks.
int xcall_lz4_decode(mo_xcall_args_t *args, uint64_t len) {
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (len == 0) return MO_RC_SUCCESS;
    if (!args[2].pdata || args[2].dataSz < 32 * len) { set_error("lz4 decode: descriptor vector shorter than 4 int64 per block"); return MO_RC_INVALID_ARGUMENT; }
    Stager st(t);
    uint8_t *dst = (uint8_t *)st.out(args[0].pdata, args[0].dataSz);
    const uint8_t *src = (const uint8_t *)st.in(args[1].pdata, args[1].dataSz);
    const int64_t *desc = (const int64_t *)st.in(args[2].pdata, 32 * len);
    unsigned long long *dbad = (unsigned long long *)st.tmp(8);
    if (st.failed) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dbad, 0xff, 8, t.stream));
    uint64_t ctas = (len + kWarpsPerCta - 1) / kWarpsPerCta;

    cudaEventRecord(t.kev0, t.stream);
    static bool attr = false;
    if (!attr) { MOB_CUDA_TRY(cudaFuncSetAttribute(lz4_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLz4Smem)); attr = true; }
    int occ = 1;   // exactly the resident CTAs: blocks are dealt statically over the warps, a partial second wave would cost a whole block time
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, lz4_decode_kernel, 32 * kWarpsPerCta, kLz4Smem) != cudaSuccess || occ < 1) occ = 1;
    if (ctas > (uint64_t)num_sms() * occ) ctas = (uint64_t)num_sms() * occ;
    lz4_decode_kernel<<<(unsigned)ctas, 32 * kWarpsPerCta, kLz4Smem, t.stream>>>(dst, args[0].dataSz, src, args[1].dataSz, desc, len, dbad);
    cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    unsigned long long bad = ~0ull;
    int rc = read_back(t, &bad, dbad, 8);
    int frc = st.finish();
    if (rc) return rc;
    if (bad != ~0ull) { set_error("lz4 decode: block %llu is malformed or does not decode to its descriptor's size", bad); return MO_RC_INVALID_ARGUMENT; }
    return frc;
}

}  // namespace mob
