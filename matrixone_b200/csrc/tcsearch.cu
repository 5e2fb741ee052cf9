// tcsearch.cu -- tensor-core candidate generation for batched brute-force search (wgmma + TMA + mbarrier, sm_90a).
//
// The exact kernel in search.cu replays the Go distance loop (3 fp32 ops per element pair).  For large query batches the L2
// distance is a dense contraction, so candidates are generated on the tensor cores and only the survivors are re-scored exactly:
//
//   1. split_kernel:   x (fp32) = hi + lo with hi = bf16(x), lo = bf16(x - hi); operands are stored K-concatenated,
//                      A' = [q_hi | q_hi | q_lo], B' = [x_hi | x_lo | x_hi]  (K' = 3*dim, padded to a multiple of 64), so ONE
//                      bf16 GEMM yields q_hi.x_hi + q_hi.x_lo + q_lo.x_hi = q.x up to ~2^-16 relative (the lo.lo term is
//                      dropped); squared norms are computed in fp64 and rounded to fp32.
//   2. tc_candidates_kernel: persistent, warp-specialised.  CTA tile 128 queries x 128 rows, K' streamed in 64-element
//                      (128-byte, SWIZZLE_128B) slabs by TMA through a 4-stage mbarrier ring; one warpgroup issues
//                      wgmma.mma_async m64n128k16 (two per K16 step, one per 64 query rows) into registers and, once a tile is
//                      complete, stores the accumulator to a shared-memory tile; four epilogue warps read that tile (each thread =
//                      one query row) while the warpgroup already multiplies the next one, form d~ = |q|^2 + |x|^2 - 2 q.x and
//                      keep the KP smallest per (query, row range) in registers.
//   3. rescore (search.cu path): the approximate lists of all ranges are merged per query, the best KR candidates are
//                      re-scored with the bit-exact Go-order distance, sorted by (distance, id), and the top k returned.
//   4. proof of completeness: a row that was never a candidate has d~ >= t, the smallest "list-full threshold" of its
//                      range; with |d~ - d| <= eps (eps from the split error bound), d_k(exact) + eps < t proves no such
//                      row can enter the top k.  Queries that fail the test (near-ties, tiny lists) are re-run on the exact
//                      kernel, so results are ALWAYS the exact answer.
//
// Work per launch: 2 * Q * N * K' flop on the tensor pipe (K' = 2304 for dim 768) + exact re-scoring of Q * KR rows.
#include "common.cuh"
#include "godist.cuh"
#include "search_internal.cuh"
#include <mutex>
#include <shared_mutex>
#include <atomic>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstring>
#include <cmath>
#include <vector>
#include <algorithm>

using namespace mob;

namespace {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int KP = 16;                      // candidates kept per (query, row range)
constexpr int KP_LONG = 32;                 // ... by the one-term pass over IVF lists (short ranges: the list threshold must sit well above the k-th result)
constexpr int kTcThreads = 288;             // warps 0-3 MMA warpgroup, warps 4-7 epilogue, warp 8 TMA
constexpr int kStages = 4;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int B_STAGE_BYTES = BN * BK * 2;  // 16 KB
constexpr int kAccStride = BM + 4;          // accumulator tile [row][query], padded so that the fragment stores are conflict-free

// PAIR = false: one CTA per unit, 128 queries, the CTA loads the whole 128-row B tile.
// PAIR = true : a cluster of two CTAs per unit (256 queries, 128 per CTA) that share the B tile: each CTA loads HALF of it with a
//               TMA multicast into both CTAs' shared memory, so a k-block costs 24 instead of 32 KB of L2 -> SM traffic per CTA --
//               the candidate pass is bound by those bytes where there are enough queries to fill 256-row units.
template <bool PAIR>
struct TcCfg {
    static constexpr int kBRows = PAIR ? BN / 2 : BN;            // B rows each CTA loads per k-block
    static constexpr int kTileM = PAIR ? 2 * BM : BM;            // query rows per unit
};

struct TcSmem {
    unsigned char a[kStages][A_STAGE_BYTES];  // 1024-byte aligned (SWIZZLE_128B atoms)
    unsigned char b[kStages][B_STAGE_BYTES];
    float acc[BN][kAccStride];                // the finished accumulator of one tile, [row of the tile][query row of the CTA]
    float xn[2][BN];                          // |x|^2 of the current tile's rows (double buffered across tiles)
    unsigned long long full[kStages], empty[kStages], acc_full, acc_empty;
    unsigned long long sched_full[2], sched_empty[2];   // dynamic unit feed (single-CTA units): the producer publishes the next unit index
    int sched_unit[2];
};

// ---- PTX wrappers ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long *bar, unsigned parity) {
    unsigned ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
    while (!mbar_try_wait(bar, parity)) { }
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap *map, unsigned long long *bar, void *dst, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// the box lands at the same shared-memory offset in every CTA of `mask` and completes bytes on the barrier at the same offset in each
__device__ __forceinline__ void tma_load_2d_multicast(const CUtensorMap *map, unsigned long long *bar, void *dst, int c0, int c1, unsigned short mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask) : "memory");
}
__device__ __forceinline__ unsigned cluster_ctarank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ unsigned mapa_rank(unsigned local_addr, unsigned rank) {
    unsigned r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank)); return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_cluster(unsigned bar_cluster_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(bar_cluster_addr) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// ties the accumulator registers to the preceding wait, so that no read of them is scheduled above it
__device__ __forceinline__ void fence_operands(float *d) {
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, both operands K-major in shared memory; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n128k16(float *d, unsigned long long desc_a, unsigned long long desc_b, unsigned scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma: start>>4 | LBO(=1, unused for swizzled K-major)<<16 |
// SBO(=1024 B: 8 rows x 128 B)>>4 <<32 | layout 1 (128-byte swizzle) <<62
__device__ __forceinline__ unsigned long long make_desc(unsigned smem_addr) {
    return (unsigned long long)((smem_addr & 0x3ffff) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// bound on |approximate - real| squared distance of one (query operand, row operand) pair, from the operand norms:
//   fp32 accumulation: a pass of nkb k-blocks runs steps = 4 nkb k16 MMA steps.  The H100 aligns the 16 products of a step to
//     the largest term (a product or the running sum) and truncates what falls below a few bits past that term's last fp32 bit,
//     then truncates the sum (measured: sixteen products of just under 1/4 ulp of the running sum are all lost, so fewer than
//     3 extra bits; tests/test_gpu_tcsearch_exact.py, hidden_neighbour_data).  Priced with no extra bit at all, each product
//     loses less than one ulp of the largest term and the sum one more: 17 ulps a step.  Every term is at most
//     sum |q_i x_i| <= |q||x|, so |q.x error| <= 17 steps 2^-23 |q||x| and the distance (2 q.x) carries 34 steps 2^-23 |q||x|
//   three-term product (K' = 3 dim): 2 * 3 * 2^-16 [dropped lo.lo + bf16 residuals] + accumulation; up to 37 steps (dim <= 192)
//     that stays under 2^-12, the coefficient used there
//   one-term (hi-only) product: q.x - qh.xh = qh.xL + qL.xh + qL.xL with qL = q - qh, xL = x - xh known exactly, so
//     |error| <= |q||xL| + |qL||x| + 3 |qL||xL|  (|qh| <= |q| + |qL|), plus accumulation (at least 2^-16)
//   both: norm / final-formula / residual-formation rounding 2^-20 (|q|^2 + |x|^2)
// qn, ql = |q|^2, |q - hi(q)|^2 of the query operand; xm, xl = the largest |x|^2, |x - hi(x)|^2 over the row operand;
// nkb = the 64-column k-blocks the candidate pass ran.
// sqrt(a b) of two squared norms; where a b leaves the normal fp32 range (rows scaled by 1e-18 or 1e18) it is taken as
// sqrt(a) sqrt(b), so that the bound neither underflows to nothing nor overflows to infinity
__device__ __forceinline__ float root_mul(float a, float b) {
    const float p = a * b;
    return p >= 1e-30f && p <= 1e30f ? sqrtf(p) : sqrtf(a) * sqrtf(b);
}
__device__ __forceinline__ float tc_eps(float qn, float ql, float xm, float xl, int one_term, int nkb) {
    const float acc = (float)(4 * nkb) * 4.0531158447265625e-6f;   // 34 steps 2^-23
    if (one_term)
        return 2.002f * (root_mul(qn, xl) + root_mul(ql, xm) + 3.0f * root_mul(ql, xl)) + fmaxf(1.52587890625e-5f, acc) * root_mul(qn, xm) + 9.5367431640625e-7f * (qn + xm);
    return fmaxf(2.44140625e-4f, 9.1552734375e-5f + acc) * root_mul(qn, xm) + 9.5367431640625e-7f * (qn + xm);
}

// one work unit: up to kTileM rows of the A' operand (queries) x dataset rows [n_begin, n_end); lists are written at out_base + row
struct TcUnit { int a_row0; int a_valid; int n_begin; int n_end; long long out_base; };

template <bool PAIR, int KPT>
__global__ void __launch_bounds__(kTcThreads, 1)
tc_candidates_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                     const TcUnit *__restrict__ units, int nunits, int nkb /* 64-element k-blocks of K' to run */,
                     const float *__restrict__ qnorm, const float *__restrict__ xnorm,
                     float *__restrict__ part_d, int *__restrict__ part_i, float *__restrict__ part_thr,
                     // cross-unit threshold sharing (qbound == nullptr: off): the units of one query run on different SMs at
                     // different times; each publishes an upper bound of the query's k-th real distance and prunes with the best one
                     float *qbound, const int *__restrict__ row_query, const float *__restrict__ alonorm,
                     const float *__restrict__ xmax2, int one_term, int topk, float rel_margin, float abs_margin,
                     // dynamic unit feed of single-CTA launches (CTA pairs: unit u = worker, worker + nworkers, ...): the producer thread takes
                     // the next unit from this counter when it has issued the last load of the current one, and hands the index to the MMA and
                     // epilogue warps through a two-slot shared-memory queue.  Units are ordered list-major, so the query tiles of one IVF list
                     // start within a few microseconds of each other on different SMs and stream the list's B' tiles through L2 together (with a
                     // static deal they drift apart and every tile of a list re-reads it from HBM), and the tail is balanced.
                     int *sched) {
    constexpr bool dyn = !PAIR;
    extern __shared__ unsigned char smem_raw[];
    // SWIZZLE_128B atoms need 1024-byte alignment in the shared window: align by hand (the launch adds 1024 spare bytes)
    TcSmem &S = *reinterpret_cast<TcSmem *>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned rank = PAIR ? cluster_ctarank() : 0u;            // a pair's CTAs take query rows rank*128.. of the unit and B half `rank`
    const int worker = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
    const int nworkers = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;

    if (threadIdx.x == 0) {
        // a stage is free again once the four MMA warps of this CTA -- and of the peer, whose half of B was multicast into it -- are done
        for (int s = 0; s < kStages; s++) { mbar_init(&S.full[s], 1); mbar_init(&S.empty[s], PAIR ? 8 : 4); }
        mbar_init(&S.acc_full, 128); mbar_init(&S.acc_empty, 128);
        for (int a = 0; a < 2; a++) { mbar_init(&S.sched_full[a], 1); mbar_init(&S.sched_empty[a], 128 + 128); }   // readers: the MMA warpgroup + the 128 epilogue threads
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    if (PAIR) cluster_sync_all();   // the peer's barriers must be initialised before anything signals them

    // the unit of iteration `it` (-1: done); the producer takes it from the counter, everybody else from the queue
    auto unit_of = [&](int it, bool producer) -> int {
        if (!dyn) { const int u = worker + it * nworkers; return u < nunits ? u : -1; }
        const int slot = it & 1;
        if (producer) {
            mbar_wait(&S.sched_empty[slot], ((it >> 1) & 1) ^ 1);
            int u = atomicAdd(sched, 1);
            if (u >= nunits) u = -1;
            *(volatile int *)&S.sched_unit[slot] = u;
            mbar_arrive(&S.sched_full[slot]);        // release: the index is visible to whoever observes the phase
            return u;
        }
        mbar_wait(&S.sched_full[slot], (it >> 1) & 1);
        const int u = *(volatile int *)&S.sched_unit[slot];
        mbar_arrive(&S.sched_empty[slot]);
        return u;
    };

    if (warp == 8) {
        // ===== TMA producer (one thread; in a pair both CTAs run it, each for its own query rows and its half of B) =====
        if (lane == 0) {
            int stage = 0; unsigned phase = 0;
            for (int it = 0;; it++) {
                const int u = unit_of(it, true);
                if (u < 0) break;
                const TcUnit U = units[u];
                for (int n0 = U.n_begin; n0 < U.n_end; n0 += BN) {
                    for (int kb = 0; kb < nkb; kb++) {
                        mbar_wait(&S.empty[stage], phase ^ 1);
                        mbar_expect_tx(&S.full[stage], A_STAGE_BYTES + B_STAGE_BYTES);   // a pair: own A + own B half + the peer's B half
                        tma_load_2d(&map_a, &S.full[stage], S.a[stage], kb * BK, U.a_row0 + (int)rank * BM);
                        if (PAIR) tma_load_2d_multicast(&map_b, &S.full[stage], S.b[stage] + rank * (B_STAGE_BYTES / 2), kb * BK, n0 + (int)rank * (BN / 2), 3);
                        else tma_load_2d(&map_b, &S.full[stage], S.b[stage], kb * BK, n0);
                        if (++stage == kStages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else if (warp < 4) {
        // ===== MMA warpgroup: 128 x 128 fp32 accumulator in registers (query rows 0-63 in d0, 64-127 in d1) =====
        float d0[64], d1[64];
#pragma unroll
        for (int i = 0; i < 64; i++) { d0[i] = 0.f; d1[i] = 0.f; }
        const unsigned peer = rank ^ 1u;
        auto release = [&](int s) {   // every warp has waited for its wgmma groups that read stage s
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&S.empty[s]);
                if (PAIR) mbar_arrive_cluster(mapa_rank(smem_u32(&S.empty[s]), peer));
            }
        };
        int stage = 0; unsigned phase = 0; unsigned tile = 0;
        for (int it = 0;; it++) {
            const int u = unit_of(it, false);
            if (u < 0) break;
            const TcUnit U = units[u];
            for (int n0 = U.n_begin; n0 < U.n_end; n0 += BN, tile++) {
                int prev = 0;
                for (int kb = 0; kb < nkb; kb++) {
                    mbar_wait(&S.full[stage], phase);
                    __syncwarp();
                    wgmma_fence();
                    const unsigned long long da = make_desc(smem_u32(S.a[stage])), db = make_desc(smem_u32(S.b[stage]));
#pragma unroll
                    for (int k = 0; k < BK / 16; k++) {  // +32 bytes (= 2 in the >>4 address field) per K16 step inside the 128-B swizzle atom
                        const unsigned acc = (kb | k) != 0;
                        wgmma_m64n128k16(d0, da + 2 * k, db + 2 * k, acc);
                        wgmma_m64n128k16(d1, da + 512 + 2 * k, db + 2 * k, acc);   // query rows 64..127: +8 KB
                    }
                    wgmma_commit();
                    if (kb > 0) { wgmma_wait<1>(); release(prev); }   // the previous k-block's MMAs have read their stage
                    prev = stage;
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
                wgmma_wait<0>();
                fence_operands(d0); fence_operands(d1);
                release(prev);
                // accumulator -> shared tile (once the epilogue has finished reading the previous one).  Fragment of m64nNk16:
                // d[4j + 2i + c] = (query row 16 warp + lane/4 + 8i, tile row 8j + 2 (lane%4) + c)
                mbar_wait(&S.acc_empty, (tile & 1) ^ 1);
                const int r0 = 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < 16; j++)
#pragma unroll
                    for (int i = 0; i < 2; i++)
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            S.acc[8 * j + c0 + c][r0 + 8 * i] = d0[4 * j + 2 * i + c];
                            S.acc[8 * j + c0 + c][64 + r0 + 8 * i] = d1[4 * j + 2 * i + c];
                        }
                mbar_arrive(&S.acc_full);
            }
        }
    } else {
        // ===== epilogue: thread e = query row of this CTA's 128 rows of the unit =====
        const int e = threadIdx.x - 128;
        const int row_in_unit = (int)rank * BM + e;
        unsigned tile = 0;
        for (int it = 0;; it++) {
            const int u = unit_of(it, false);
            if (u < 0) break;
            const TcUnit U = units[u];
            const bool valid_row = row_in_unit < U.a_valid;
            const float qn = valid_row ? qnorm[U.a_row0 + row_in_unit] : 0.f;
            // the KPT best (approximate distance, row) pairs of this query row live in REGISTERS, ascending; an insertion is a
            // branch-free compare/select sweep (no shared-memory dependency chain, lanes of a warp insert at different ranks at
            // the same cost).  Rows of the tile past a_valid never insert (thr = -inf).
            float ld[KPT]; int li[KPT];
#pragma unroll
            for (int j = 0; j < KPT; j++) { ld[j] = INFINITY; li[j] = -1; }
            float thr = valid_row ? INFINITY : -INFINITY;
            // sharing: `cap` = (best published bound of this query) + this pair's own error bound + the Go-order margin; rows at or
            // above it cannot displace the k-th result, so they are excluded exactly like rows beyond a full list (thr only falls)
            const bool share = qbound != nullptr && valid_row;
            const int qid = share ? (row_query ? row_query[U.a_row0 + row_in_unit] : U.a_row0 + row_in_unit) : 0;
            const float my_eps = share ? tc_eps(qn, one_term ? alonorm[U.a_row0 + row_in_unit] : 0.f, xmax2[0], one_term ? xmax2[1] : 0.f, one_term, nkb) : 0.f;
            float cap = INFINITY, published = INFINITY;
            for (int n0 = U.n_begin; n0 < U.n_end; n0 += BN, tile++) {
                const unsigned xb = tile & 1;
                // |x|^2 of this tile's rows -> shared (one per thread); named barrier over the 128 epilogue threads
                for (int j = e; j < BN; j += 128) S.xn[xb][j] = (n0 + j < U.n_end) ? xnorm[n0 + j] : INFINITY;
                asm volatile("bar.sync 1, 128;" ::: "memory");
                mbar_wait(&S.acc_full, tile & 1);
                const int ncols = U.n_end - n0 < BN ? U.n_end - n0 : BN;
                if (share) {
                    const float b = __ldcg(&qbound[qid]);
                    if (b < INFINITY) { cap = fminf(cap, b + my_eps + b * rel_margin + abs_margin + 1e-30f); thr = fminf(thr, cap); }
                }
#pragma unroll 1
                for (int c = 0; c < ncols; c += 32) {
                    // fast path: 32 approximate distances and their minimum, branch-free (independent FADD/FFMA/FMNMX chains)
                    float v[32];
                    float dmin = INFINITY;
#pragma unroll
                    for (int j4 = 0; j4 < 32; j4 += 4) {
                        const float4 xn4 = *reinterpret_cast<const float4 *>(&S.xn[xb][c + j4]);   // +inf for rows past the end
                        v[j4 + 0] = fmaf(-2.0f, S.acc[c + j4 + 0][e], qn + xn4.x); v[j4 + 1] = fmaf(-2.0f, S.acc[c + j4 + 1][e], qn + xn4.y);
                        v[j4 + 2] = fmaf(-2.0f, S.acc[c + j4 + 2][e], qn + xn4.z); v[j4 + 3] = fmaf(-2.0f, S.acc[c + j4 + 3][e], qn + xn4.w);
                        dmin = fminf(fminf(dmin, fminf(v[j4 + 0], v[j4 + 1])), fminf(v[j4 + 2], v[j4 + 3]));
                    }
                    // slow path (some element beats the list's worst entry): the insertion code exists ONCE -- the hits are walked
                    // through a bit mask and their distances recomputed from the shared tile (dynamic register indexing is impossible,
                    // and 32 unrolled copies of the sweep would not fit the instruction cache)
                    if (dmin < thr) {
                        unsigned hit = 0;
#pragma unroll
                        for (int j = 0; j < 32; j++) hit |= (v[j] < thr) ? (1u << j) : 0u;
#pragma unroll 1
                        while (hit) {
                            const int j = __ffs((int)hit) - 1;
                            hit &= hit - 1;
                            const float d = fmaf(-2.0f, S.acc[c + j][e], qn + S.xn[xb][c + j]);   // the same value as v[j]
                            if (d < thr) {   // thr may have dropped since the mask was taken
                                const int id = n0 + c + j;
#pragma unroll
                                for (int p = KPT - 1; p > 0; p--) {     // descending: ld[p - 1] is still the old value when read
                                    const bool shift = d < ld[p - 1];  // the old neighbour moves down to p
                                    const bool here = !shift && d < ld[p];
                                    li[p] = shift ? li[p - 1] : (here ? id : li[p]);
                                    ld[p] = shift ? ld[p - 1] : (here ? d : ld[p]);
                                }
                                if (d < ld[0]) { ld[0] = d; li[0] = id; }
                                thr = fminf(ld[KPT - 1], cap);
                            }
                        }
                    }
                }
                mbar_arrive(&S.acc_empty);   // 128 arrivals release the shared tile to the MMA warpgroup
                if (share && topk <= KPT) {   // the k best rows seen by this unit bound the query's k-th real distance from above
                    float kth = INFINITY;
#pragma unroll
                    for (int j = 0; j < KPT; j++) if (j == topk - 1) kth = ld[j];
                    const float pb = fmaxf(kth + my_eps, 0.f);
                    if (pb < published) { published = pb; atomicMin(reinterpret_cast<int *>(&qbound[qid]), __float_as_int(pb)); }
                }
            }
            if (valid_row) {
                const size_t base = (size_t)(U.out_base + row_in_unit) * KPT;
#pragma unroll
                for (int j = 0; j < KPT; j++) { part_d[base + j] = ld[j]; part_i[base + j] = li[j]; }   // empty slots: (+inf, -1)
                part_thr[U.out_base + row_in_unit] = thr;        // every row of this unit that is NOT listed has d~ >= thr (+inf: list not full)
            }
        }
    }
    __syncthreads();
    if (PAIR) cluster_sync_all();   // the peer multicasts into this CTA's shared memory and arrives on its barriers: leave together
}

// ---- operand preparation -------------------------------------------------------------------------------------------------
// one row of the split, by one warp: element j of the row is elem(j).  mode 0: A' = [hi | hi | lo] (queries), mode 1: B' =
// [hi | lo | hi] (dataset); K' is padded with zeros.  norm = |v|^2, lonorm = |v - hi|^2 (the part of v a hi-only product does
// not see), both accumulated in double; an Inf / NaN element raises *nonfinite (the caller falls back to the exact kernel).
template <class Elem>
__device__ __forceinline__ void split_row(Elem elem, int lane, int dim, int kprime, int mode, __nv_bfloat16 *__restrict__ o,
                                          float *__restrict__ norm, float *__restrict__ lonorm, int *__restrict__ nonfinite) {
    double s = 0.0, sl = 0.0;
    for (int j = lane; j < dim; j += 32) {
        const float v = elem(j);
        const __nv_bfloat16 hi = __float2bfloat16_rn(v);
        const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
        o[j] = hi;
        o[dim + j] = mode == 0 ? hi : lo;
        o[2 * dim + j] = mode == 0 ? lo : hi;
        s += (double)v * (double)v;
        const double l = (double)(v - __bfloat162float(hi));   // exact in fp32
        sl += l * l;
        if (!(fabsf(v) <= 3.0e38f)) *nonfinite = 1;
    }
    for (int j = 3 * dim + lane; j < kprime; j += 32) o[j] = __float2bfloat16_rn(0.f);
    s = warp_sum_f64(s); sl = warp_sum_f64(sl);
    if (lane == 0) { *norm = (float)s; *lonorm = (float)sl; }
}

__global__ void split_kernel(const float *__restrict__ x, int64_t n, int dim, int kprime, int mode, int normalize, __nv_bfloat16 *__restrict__ out,
                             float *__restrict__ norm, float *__restrict__ lonorm, int *__restrict__ nonfinite) {
    // normalize (cosine): the row is first divided by its length, so 1 - cos(q, x) = |q^ - x^|^2 / 2 and the L2 machinery applies;
    // a zero (or non-finite) row raises *nonfinite and the caller answers the whole call with the exact kernel.
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const float *p = x + r * dim;
        __nv_bfloat16 *o = out + r * kprime;
        float len = 1.0f;
        if (normalize) {
            double s0 = 0.0;
            for (int j = lane; j < dim; j += 32) { const double v = (double)p[j]; s0 += v * v; }
            s0 = warp_sum_f64(s0);
            len = (float)sqrt(s0);
            if (!(len > 0.f && len <= 3.0e38f)) { if (lane == 0) *nonfinite = 1; len = 1.0f; }
        }
        split_row([&](int j) { return normalize ? __fdiv_rn(p[j], len) : p[j]; }, lane, dim, kprime, mode, o, norm + r, lonorm + r, nonfinite);
    }
}

// IVF operands are RESIDUALS: x - centroid(list of x) for the entries, q - centroid(l) for every (query, probed list l) pair.
// |q - x|^2 = |(q - c) - (x - c)|^2, and residual norms are the within-list spread instead of the distance from the origin, so
// the error bounds of the candidate pass (proportional to |a||b|) shrink with them.  fl(v - c) differs from v - c by 2^-24
// relative per element, covered by the 2^-20 (|a|^2 + |b|^2) term of the proof.
// mode 1 (entries): src row r belongs to the list l with offsets[l] <= r < offsets[l + 1]; mode 0 (pairs): row g = (idx_q[g], idx_l[g]).
__global__ void split_residual_kernel(const float *__restrict__ x, int64_t n, int dim, int kprime, int mode,
                                      const float *__restrict__ cent, const int64_t *__restrict__ offsets, int64_t nlist,
                                      const int32_t *__restrict__ idx_q, const int32_t *__restrict__ idx_l,
                                      __nv_bfloat16 *__restrict__ out, float *__restrict__ norm, float *__restrict__ lonorm, int *__restrict__ nonfinite,
                                      int hi_only) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        int64_t src = r, l;
        if (mode == 0) { src = idx_q[r]; l = idx_l[r]; }
        else {   // largest l with offsets[l] <= r (empty lists share an offset: any of them gives the same answer only if non-empty => upper bound - 1)
            int64_t lo = 0, hi = nlist;          // invariant: offsets[lo] <= r < offsets[hi]
            while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (offsets[mid] <= r) lo = mid; else hi = mid; }
            l = lo;
        }
        const float *p = x + src * dim, *c = cent + l * dim;
        __nv_bfloat16 *o = out + r * kprime;
        if (hi_only && (dim & 7) == 0 && (kprime & 7) == 0) {
            // one-term level: the candidate pass multiplies only the first `dim` columns (hi . hi), so only they are written -- a third
            // of the bytes; 8 elements per lane: two 128-bit loads per operand, one 128-bit store
            double s = 0.0, sl = 0.0;
            for (int j = lane * 8; j < dim; j += 256) {
                const float4 p0 = *reinterpret_cast<const float4 *>(p + j), p1 = *reinterpret_cast<const float4 *>(p + j + 4);
                const float4 c0 = *reinterpret_cast<const float4 *>(c + j), c1 = *reinterpret_cast<const float4 *>(c + j + 4);
                const float v[8] = {__fsub_rn(p0.x, c0.x), __fsub_rn(p0.y, c0.y), __fsub_rn(p0.z, c0.z), __fsub_rn(p0.w, c0.w),
                                    __fsub_rn(p1.x, c1.x), __fsub_rn(p1.y, c1.y), __fsub_rn(p1.z, c1.z), __fsub_rn(p1.w, c1.w)};
                __align__(16) __nv_bfloat16 h[8];
#pragma unroll
                for (int e = 0; e < 8; e++) {
                    h[e] = __float2bfloat16_rn(v[e]);
                    s += (double)v[e] * (double)v[e];
                    const double d = (double)(v[e] - __bfloat162float(h[e]));
                    sl += d * d;
                    if (!(fabsf(v[e]) <= 3.0e38f)) *nonfinite = 1;
                }
                *reinterpret_cast<int4 *>(o + j) = *reinterpret_cast<const int4 *>(h);
            }
            // the pass reads whole 64-column k-blocks: the columns from dim to the next multiple of 64 must be zero, not stale scratch
            for (int j = dim + lane; j < kprime && j < (dim + BK - 1) / BK * BK; j += 32) o[j] = __float2bfloat16_rn(0.f);
            s = warp_sum_f64(s); sl = warp_sum_f64(sl);
            if (lane == 0) { norm[r] = (float)s; lonorm[r] = (float)sl; }
            continue;
        }
        split_row([&](int j) { return __fsub_rn(p[j], c[j]); }, lane, dim, kprime, mode, o, norm + r, lonorm + r, nonfinite);
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_map(CUtensorMap *map, void *base, uint64_t rows, uint64_t kprime, uint32_t box_rows) {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        cudaDriverEntryPointQueryResult qres;
        void *p = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) {
            set_error("cuTensorMapEncodeTiled entry point not available"); return MO_RC_INTERNAL_ERROR;
        }
        fn = (EncodeTiledFn)p;
    }
    const cuuint64_t gdim[2] = {kprime, rows};              // innermost first
    const cuuint64_t gstride[1] = {kprime * 2};             // bytes, dims 1..
    const cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};  // 64 bf16 = 128 B = the swizzle span
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return MO_RC_INTERNAL_ERROR; }
    return MO_RC_SUCCESS;
}

// ---- post-processing: merge approximate lists, exact re-score, final order + completeness proof -----------------------------
constexpr int KR = 32;      // candidates re-scored exactly per query (k <= KP)
constexpr int KR_WIDE = 64; // ... and for KP < k <= KW (centroid probes with nprobe up to 32)
constexpr int KW = 32;

// one warp per query: R-way merge of the (ascending) approximate lists -> KR best candidate ids; t_excl = smallest approximate
// distance any row NOT among them can have (first unconsumed entry of every list, and the list-full threshold of every range).
// Lane l owns lists l, l+32, ...; every round the warp picks the smallest head (ties: lower list number).
// list (q, r) lives at index  r * nq + q  without pos_map; with it (IVF) r = s * pos_cols + p names sub-range s of probe rank p:
// index = s * pos_stride + pos_map[q * pos_cols + p]  (pos_map < 0 = no such list)
constexpr int kMaxMergeLists = 256;
constexpr int kMergeSlots = kMaxMergeLists / 32;

// pnorm / plonorm (IVF): the query operand differs per probed list (residual against that list's centroid), so every list's
// exclusion bound is lowered by ITS error bound before the minimum is taken: t_excl = min_l (t_l - eps_l)
__global__ void tc_merge_kernel(int nq, int R, const float *__restrict__ part_d, const int *__restrict__ part_i,
                                const float *__restrict__ part_thr, const int *__restrict__ pos_map, int pos_cols, long long pos_stride,
                                const float *__restrict__ pnorm, const float *__restrict__ plonorm, const float *__restrict__ xmax2, int one_term,
                                const float *__restrict__ qnorm, const float *__restrict__ qlonorm, int k, int dim, int nkb,
                                int kp, int kr, int *__restrict__ cand, float *__restrict__ t_excl) {
    const int lane = threadIdx.x & 31;
    const int q = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5);
    if (q >= nq) return;   // whole warps leave together
    // error bound of every list of this query when it does not depend on the list (brute force: one query operand)
    const float eps_q = (!pnorm && qnorm) ? tc_eps(qnorm[q], one_term ? qlonorm[q] : 0.f, xmax2[0], one_term ? xmax2[1] : 0.f, one_term, nkb) : 0.f;
    float sel_d0 = 0.f, sel_d1 = 0.f, sel_e0 = 0.f, sel_e1 = 0.f;   // approximate distance / bound of selections lane and lane + 32
    int nsel = 0;
    long long L[kMergeSlots]; int head[kMergeSlots]; float cur[kMergeSlots], tl[kMergeSlots], eps[kMergeSlots];
#pragma unroll
    for (int i = 0; i < kMergeSlots; i++) {
        const int r = lane + 32 * i;
        long long l = -1; int p = -1;
        if (r < R) {
            if (!pos_map) l = (long long)r * nq + q;
            else { p = pos_map[(size_t)q * pos_cols + r % pos_cols]; l = p < 0 ? -1ll : (long long)(r / pos_cols) * pos_stride + p; }
        }
        L[i] = l; head[i] = 0; cur[i] = INFINITY; tl[i] = INFINITY; eps[i] = 0.f;
        if (l >= 0) {
            tl[i] = part_thr[l];
            if (part_i[(size_t)l * kp] >= 0) cur[i] = part_d[(size_t)l * kp];
            if (pnorm && p >= 0) eps[i] = tc_eps(pnorm[p], plonorm[p], xmax2[0], xmax2[1], one_term, nkb);
        }
    }
    for (int j = 0; j < kr; j++) {
        float bd = INFINITY; int br = 0x7fffffff;
#pragma unroll
        for (int i = 0; i < kMergeSlots; i++) if (cur[i] < bd) { bd = cur[i]; br = lane + 32 * i; }   // ascending i = ascending list number
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float od = __shfl_xor_sync(0xffffffffu, bd, o); const int orr = __shfl_xor_sync(0xffffffffu, br, o);
            if (od < bd || (od == bd && orr < br)) { bd = od; br = orr; }
        }
        if (br == 0x7fffffff) { if (lane == 0) cand[(size_t)q * kr + j] = -1; continue; }   // every list is exhausted (warp-uniform)
        float we = eps_q;
        if ((br & 31) == lane) {
#pragma unroll
            for (int i = 0; i < kMergeSlots; i++)
                if (i == (br >> 5)) {
                    const size_t idx = (size_t)L[i] * kp + head[i];
                    cand[(size_t)q * kr + j] = part_i[idx];
                    head[i]++;
                    cur[i] = (head[i] < kp && part_i[idx + 1] >= 0) ? part_d[idx + 1] : INFINITY;
                    if (pnorm) we = eps[i];
                }
        }
        we = __shfl_sync(0xffffffffu, we, br & 31);
        if ((j & 31) == lane) { if (j < 32) { sel_d0 = bd; sel_e0 = we; } else { sel_d1 = bd; sel_e1 = we; } }
        nsel = j + 1;   // selections are made in order: the first nsel slots are the valid ones
    }
    // prune before the exact re-score: with U = the k-th smallest UPPER bound (d~ + eps) among the selections, at least k rows have
    // a real distance <= U, so a selection whose LOWER bound (d~ - eps) exceeds U cannot be in the top k (gamma = the Go-order
    // fp32 evaluation error relative to the real distance)
    if ((pnorm || qnorm) && nsel > k && kr <= 64) {
        const bool v0 = lane < nsel, v1 = lane + 32 < nsel;
        const float u0 = v0 ? sel_d0 + sel_e0 : INFINITY, u1 = v1 ? sel_d1 + sel_e1 : INFINITY;
        int rank0 = 0, rank1 = 0;
        for (int jj = 0; jj < nsel; jj++) {
            const float v = __shfl_sync(0xffffffffu, jj < 32 ? u0 : u1, jj & 31);
            rank0 += (v < u0 || (v == u0 && jj < lane)) ? 1 : 0;
            rank1 += (v < u1 || (v == u1 && jj < lane + 32)) ? 1 : 0;
        }
        float U = (v0 && rank0 == k - 1) ? u0 : ((v1 && rank1 == k - 1) ? u1 : INFINITY);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) U = fminf(U, __shfl_xor_sync(0xffffffffu, U, o));
        const float gamma = (float)dim * 1.1920928955078125e-7f;
        const float lim = U * (1.0f + 2.0f * gamma) + 1e-30f;
        __syncwarp();   // the selections above were written by other lanes
        if (v0 && (sel_d0 - sel_e0) * (1.0f - 2.0f * gamma) > lim) cand[(size_t)q * kr + lane] = -1;
        if (v1 && (sel_d1 - sel_e1) * (1.0f - 2.0f * gamma) > lim) cand[(size_t)q * kr + lane + 32] = -1;
    }
    float t = INFINITY;
#pragma unroll
    for (int i = 0; i < kMergeSlots; i++) t = fminf(t, fminf(tl[i], cur[i]) - eps[i]);   // list-full threshold / first unconsumed entry (inf - eps = inf)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = fminf(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (lane == 0) t_excl[q] = t;
}

// exact re-scoring: one warp per (query, 32 candidates) batch, lane = candidate row, the query is the constant operand: the
// bit-exact Go-order L2sq through the lane-per-row batch machinery of godist.cuh (rows stream through a per-warp cp.async ring)
constexpr int kRescoreThreads = 128;
template <int METRIC>   // MO_METRIC_L2SQ, MO_METRIC_IP, MO_METRIC_COS: the value the exact kernel (search.cu) would produce for the pair
__global__ void __launch_bounds__(kRescoreThreads)
tc_rescore_kernel(const float *__restrict__ data, const float *__restrict__ queries, int dim, int nq, int kr,
                  const int *__restrict__ cand, float *__restrict__ exact) {
    using Cfg = godist::RingCfg<false>;
    constexpr int KIND = METRIC == MO_METRIC_IP ? godist::K_GO_IP : (METRIC == MO_METRIC_COS ? godist::K_GO_COSDIST : godist::K_GO_L2SQ);
    extern __shared__ __align__(16) unsigned char rescore_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    unsigned char *ring = rescore_smem + (size_t)wib * Cfg::kStages * Cfg::kStageBytes;
    const int nb = kr / 32;
    const int64_t w0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t w = w0; w < (int64_t)nq * nb; w += nw) {
        const int64_t q = w / nb; const int h = (int)(w % nb);
        const size_t slot = (size_t)q * kr + (size_t)h * 32 + lane;
        const int id = cand[slot];
        const bool good = id >= 0;
        // operand order (query, row) as in the exact kernel: the cosine accumulators n1 / n2 belong to the query / the row
        const uint8_t *px = good ? reinterpret_cast<const uint8_t *>(data + (int64_t)id * dim) : nullptr;
        const uint8_t *pq = reinterpret_cast<const uint8_t *>(queries + q * dim);
        const godist::RowAcc<float, KIND> acc = godist::row_batch<float, KIND, false>(ring, lane, px, pq, dim, good);
        float d = acc.sum;
        if (METRIC == MO_METRIC_IP) d = -acc.sum;
        if (METRIC == MO_METRIC_COS) {     // distance_func.go:264-284, as bf_topk_kernel evaluates it
            const double den = sqrt((double)acc.n1) * sqrt((double)acc.n2);
            if (den == 0.0) d = 1.0f;
            else { double sim = (double)acc.sum / den; sim = sim > 1.0 ? 1.0 : (sim < -1.0 ? -1.0 : sim); d = (float)(1.0 - sim); }
        }
        exact[slot] = good ? d : INFINITY;
    }
}

// IVF: seed the shared bound of every query with the exact k-th distance among the first 32 rows of its nearest list -- loose
// (k-th of 32 instead of k-th of ~nprobe lists), but enough to keep the rows of far lists out of the candidate lists from the
// first tile on.  One warp per query, lane = row, through the same batch machinery as the re-score.
__global__ void __launch_bounds__(kRescoreThreads)
ivf_seed_bound_kernel(const float *__restrict__ data, const float *__restrict__ queries, int dim, int nq, int nprobe, int k,
                      const int64_t *__restrict__ probes, const int64_t *__restrict__ offsets, float *__restrict__ qbound,
                      const uint32_t *__restrict__ admit /* filtered search: only admitted rows seed the bound */) {
    using Cfg = godist::RingCfg<false>;
    extern __shared__ __align__(16) unsigned char rescore_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    unsigned char *ring = rescore_smem + (size_t)wib * Cfg::kStages * Cfg::kStageBytes;
    const int64_t w0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t q = w0; q < nq; q += nw) {
        int64_t l = -1;   // the nearest probed list that has rows here (a list-sharded index holds only some of them)
        for (int r = 0; r < nprobe && l < 0; r++) { const int64_t c = probes[q * nprobe + r]; if (c >= 0 && offsets[c + 1] > offsets[c]) l = c; }
        const int64_t b = l >= 0 ? offsets[l] : 0, e = l >= 0 ? offsets[l + 1] : 0;
        const bool good = b + lane < e && (!admit || ((admit[(b + lane) >> 5] >> ((b + lane) & 31)) & 1u));
        const uint8_t *px = good ? reinterpret_cast<const uint8_t *>(data + (b + lane) * dim) : nullptr;
        const uint8_t *pq = reinterpret_cast<const uint8_t *>(queries + q * dim);
        const godist::RowAcc<float, godist::K_GO_L2SQ> acc = godist::row_batch<float, godist::K_GO_L2SQ, false>(ring, lane, px, pq, dim, good);
        const float d = good ? acc.sum : INFINITY;
        int rank = 0;
        for (int j = 0; j < 32; j++) { const float o = __shfl_sync(0xffffffffu, d, j); rank += (o < d || (o == d && j < lane)) ? 1 : 0; }
        // the lane holding the k-th smallest: its Go-order value, inflated by the Go-order error, bounds the real k-th distance
        if (rank == k - 1 && d < INFINITY) qbound[q] = d * (1.0f + (float)dim * 2.384185791015625e-7f);
    }
}

__global__ void tc_max_kernel(const float *__restrict__ v, int64_t n, float *out) {   // max of non-negative floats
    float m = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, v[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int *>(out), __float_as_int(m));
}

// one thread per query: order the KR exact candidates by (distance, id), emit the top k with the reference's front padding, and
// prove completeness:  every excluded row has approximate distance >= t_excl, |approx - real| <= eps_tc, |real - go| <= eps_go,
// so d_k + eps_tc + eps_go < t_excl  =>  no excluded row can displace the k-th result.  flag = 1 when the proof fails.
template <int KRT>
__global__ void tc_final_kernel(int nq, int k, int dim, int nkb, const int *__restrict__ cand, const float *__restrict__ exact,
                                const float *__restrict__ t_excl, const float *__restrict__ qnorm, const float *__restrict__ xnorm_max,
                                const float *__restrict__ qlonorm, const float *__restrict__ xlonorm_max, int one_term, int eps_applied, int metric,
                                const int64_t *__restrict__ id_map, int64_t key_base, int sqrt_out, int64_t *__restrict__ out_k,
                                double *__restrict__ out_d, int *__restrict__ flags) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    float d[KRT]; int64_t id[KRT]; int m = 0;
    for (int j = 0; j < KRT; j++) {
        const int lc = cand[(size_t)q * KRT + j];
        if (lc < 0) continue;
        const int64_t c = id_map ? id_map[lc] : (int64_t)lc + key_base;   // final key; ties are ordered by it
        const float v = exact[(size_t)q * KRT + j];
        int pos = m++;
        while (pos > 0 && (v < d[pos - 1] || (v == d[pos - 1] && c < id[pos - 1]))) { d[pos] = d[pos - 1]; id[pos] = id[pos - 1]; pos--; }
        d[pos] = v; id[pos] = c;
    }
    const int total = m < k ? m : k;
    const int pad = k - total;
    int64_t *ok = out_k + (size_t)q * k; double *od = out_d + (size_t)q * k;
    // padding (fewer than k rows exist -- with a filter, fewer than k admitted): key -1, distance 0; brute force with k = 1 and no row
    // leaves the running minimum untouched: MaxFloat32 (brute_force.go:289-331).  eps_applied = the IVF list scan, which pads with 0.
    const double pad_d = (k == 1 && !eps_applied) ? (double)3.40282346638528859811704183484516925440e+38f : 0.0;
    for (int j = 0; j < pad; j++) { ok[j] = -1; od[j] = pad_d; }
    for (int j = 0; j < total; j++) { ok[pad + j] = id[j]; od[pad + j] = sqrt_out ? sqrt((double)d[j]) : (double)d[j]; }
    // the candidate kernel works in units of |q|^2 + |x|^2 - 2 q.x: that IS the L2 distance; for inner product (norms left out)
    // and cosine (normalised operands) it is twice the metric's distance
    const float scale = (metric == MO_METRIC_IP || metric == MO_METRIC_COS) ? 0.5f : 1.0f;
    const float t = t_excl[q] * scale;
    bool proven;
    if (t == INFINITY) proven = true;                       // nothing was excluded (every row of every range is listed)
    else if (m < k) proven = false;
    else {
        // eps_applied: the merge already lowered t by every list's own bound (IVF residual operands)
        const float eps_tc = eps_applied ? 0.f : scale * tc_eps(qnorm[q], one_term ? qlonorm[q] : 0.f, *xnorm_max, one_term ? *xlonorm_max : 0.f, one_term, nkb);
        // |Go-order fp32 value - real value|: relative dim * 2^-23 for L2; absolute dim * 2^-23 |q||x| for the inner product;
        // for cosine 4 dim 2^-24 (dot product and both norms) + 2^-19 (normalisation of the operands of the candidate pass)
        float eps_go = (float)dim * 1.1920928955078125e-7f * t;
        if (metric == MO_METRIC_IP) eps_go = (float)dim * 1.1920928955078125e-7f * root_mul(qnorm[q], *xnorm_max);
        if (metric == MO_METRIC_COS) eps_go = (float)dim * 2.384185791015625e-7f + 1.9073486328125e-6f;
        proven = d[k - 1] + eps_tc + eps_go < t;
    }
    flags[q] = proven ? 0 : 1;
}

__global__ void tc_fill_kernel(float *thr, int *ids, int64_t nlists, int kp) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nlists * kp; i += (int64_t)gridDim.x * blockDim.x) {
        ids[i] = -1;
        if (i < nlists) thr[i] = INFINITY;
    }
}

}  // namespace

namespace mob {

// knobs (MoB200_SetTuning): they reach paths that production selects from the input
static int g_search_mode = 0;        // 0 = auto, 1 = exact kernel only, 2 = force the tensor-core path
static int g_tc_pair_mode = 0;       // 0 = auto, 1 = single-CTA units only, 2 = CTA pairs wherever the brute-force path runs
static int g_tc_ladder_mode = 0;     // 0 = auto (one-term level first unless it has been failing), 1 = never, 2 = always
static int g_tc_share_mode = 0;      // 1 = no cross-unit threshold sharing
static int g_tc_range_mb = 0;        // L2 budget of one row range of the brute-force candidate pass, MB (0 = ignore the L2)
static int g_filter_path = 0;        // filtered search: 0 = auto (from the admitted count), 1 = masked scan, 2 = compacted admitted rows
static std::atomic<int> g_one_term_skip{0};   // searches left before the one-term level is tried again (shared by all callers: a property of the data)
thread_local SearchStats g_search_stats;

bool search_tuning(const char *name, int value, int *out) {
    static const struct { const char *name; int *knob; } knobs[] = {
        {"search_mode", &g_search_mode}, {"search_filter_path", &g_filter_path}, {"tc_pair", &g_tc_pair_mode}, {"tc_ladder", &g_tc_ladder_mode}, {"tc_share", &g_tc_share_mode}, {"tc_range_mb", &g_tc_range_mb}};
    for (const auto &k : knobs)
        if (!strcmp(name, k.name)) {
            *k.knob = value;
            if (k.knob == &g_tc_ladder_mode) g_one_term_skip.store(0);
            *out = 0;
            return true;
        }
    const SearchStats &s = g_search_stats;
    const struct { const char *name; int value; } stats[] = {
        {"get_tc_kused", s.kused}, {"get_tc_probe_kused", s.probe_kused}, {"get_tc_refined", s.refined}, {"get_tc_fallbacks", s.fallbacks},
        {"get_filter_admitted", s.filter_admitted}, {"get_filter_compacted", s.filter_compacted}};
    for (const auto &st : stats)
        if (!strcmp(name, st.name)) { *out = st.value; return true; }
    return false;
}

struct TcOperand { __nv_bfloat16 *bf = nullptr; float *norm = nullptr; float *lonorm = nullptr; const float *enorm = nullptr; int kprime = 0; };   // enorm: what the epilogue adds (null = norm; zeros for inner product)   // norm = |x|^2, lonorm = |x - bf16(x)|^2 per row

static int tc_kprime(int dim) { return ((3 * dim + BK - 1) / BK) * BK; }   // K' = 3 dim in whole k-blocks

// an operand of `rows` rows in the call's arena
static int tc_alloc(ThreadCtx &t, int64_t rows, int dim, TcOperand &op) {
    const size_t r = (size_t)(rows > 0 ? rows : 1);
    op.kprime = tc_kprime(dim);
    op.bf = (__nv_bfloat16 *)arena_alloc(t, r * op.kprime * 2 + 1024);
    op.norm = (float *)arena_alloc(t, r * 4);
    op.lonorm = (float *)arena_alloc(t, r * 4);
    return op.bf && op.norm && op.lonorm ? MO_RC_SUCCESS : MO_RC_INTERNAL_ERROR;
}

// datasets split once by MoB200_SearchPrepare (index load); looked up by (pointer, rows, dim)
struct PreparedOperand { const float *x; int64_t n; int dim; TcOperand op; const float *cent = nullptr; int64_t nlist = 0; int normalized = 0; const int64_t *offsets = nullptr; };   // cent != nullptr: IVF residual operand; normalized: cosine
static std::mutex g_prepared_mu;
static std::vector<PreparedOperand> g_prepared;
// A search holds this shared for its whole call (the kernels it launched have finished when it returns); whoever frees or rebuilds a
// prepared operand -- SearchRelease, DeviceFree, Upload / Memset over the dataset, SearchPrepare* -- takes it exclusively, so a concurrent
// search on another OS thread never runs TMA loads on freed memory (ADVICE r01).
static std::shared_mutex g_search_rw;
SearchReadGuard::SearchReadGuard() { g_search_rw.lock_shared(); }
SearchReadGuard::~SearchReadGuard() { g_search_rw.unlock_shared(); }

static void free_prepared(const TcOperand &op) { cudaFree(op.bf); cudaFree(op.norm); }   // lonorm shares norm's allocation

// frees and forgets every prepared operand for which pred holds.  The pre-check takes only the list mutex: most calls (scratch
// uploads, generators) touch no prepared dataset and must not wait for running searches.
template <class Pred>
static void drop_prepared(Pred pred) {
    {
        std::lock_guard<std::mutex> lk(g_prepared_mu);
        if (std::none_of(g_prepared.begin(), g_prepared.end(), pred)) return;
    }
    std::unique_lock<std::shared_mutex> wr(g_search_rw);   // wait for running searches to finish before freeing their operand
    std::lock_guard<std::mutex> lk(g_prepared_mu);
    for (size_t i = 0; i < g_prepared.size();) {
        if (pred(g_prepared[i])) { free_prepared(g_prepared[i].op); g_prepared.erase(g_prepared.begin() + (long)i); }
        else i++;
    }
}

// the operand of x prepared at index load: brute force (cent == nullptr) with normalisation `normalized`, or IVF residuals against
// (cent, nlist, offsets)
static bool find_prepared(const float *x, int64_t n, int dim, const float *cent, int64_t nlist, const int64_t *offsets, int normalized, TcOperand &op) {
    std::lock_guard<std::mutex> lk(g_prepared_mu);
    for (const PreparedOperand &e : g_prepared)
        if (e.x == x && e.n == n && e.dim == dim && e.cent == cent && e.nlist == nlist && e.offsets == offsets && e.normalized == normalized) { op = e.op; return true; }
    return false;
}

// split an fp32 row-major matrix into the K-concatenated bf16 operand: mode 0 = queries (A'), mode 1 = dataset (B'); cent != nullptr:
// IVF entries as residuals against their list's centroid (see split_residual_kernel).  *nonfinite (device flag) is raised on Inf/NaN.
static int tc_prepare(ThreadCtx &t, const float *x, int64_t n, int dim, int mode, int normalize, const float *cent, int64_t nlist,
                      const int64_t *offsets, int *dnonfinite, TcOperand &op) {
    if (mode == 1 && find_prepared(x, n, dim, cent, nlist, offsets, normalize, op)) return MO_RC_SUCCESS;
    // one API call may split the same matrix more than once (the levels of a precision ladder): the operand lives in the call's
    // arena, so it is reused while the arena epoch lasts.  A nonfinite input was already reported by the split that filled the cache.
    struct Cached { const float *x = nullptr, *cent = nullptr; int64_t n = 0; int dim = 0, normalize = 0; uint64_t epoch = ~0ull; const ThreadCtx *t = nullptr; TcOperand op; };
    static thread_local Cached cache[3];   // queries, dataset, IVF entries
    Cached &c = cache[cent ? 2 : mode];
    if (c.t == &t && c.epoch == t.arena_epoch && c.x == x && c.cent == cent && c.n == n && c.dim == dim && c.normalize == normalize) { op = c.op; return MO_RC_SUCCESS; }
    int rc = tc_alloc(t, n, dim, op);
    if (rc) return rc;
    if (n > 0) {
        if (cent) split_residual_kernel<<<num_sms() * 8, 256, 0, t.stream>>>(x, n, dim, op.kprime, 1, cent, offsets, nlist, nullptr, nullptr, op.bf, op.norm, op.lonorm, dnonfinite, 0);
        else split_kernel<<<num_sms() * 8, 256, 0, t.stream>>>(x, n, dim, op.kprime, mode, normalize, op.bf, op.norm, op.lonorm, dnonfinite);
        MOB_LAUNCH_CHECK();
    }
    c = Cached{x, cent, n, dim, normalize, t.arena_epoch, &t, op};
    return MO_RC_SUCCESS;
}

// run the candidate kernel over `units`; lists are written at unit.out_base + row (nlists lists in total, pre-initialised empty)
// cross-unit threshold sharing (see the kernel): nq queries, row_query maps an A row to its query (nullptr: identity)
struct TcShare { int64_t nq; const int *row_query; int topk; int one_term; float rel_margin, abs_margin; const float *xmax2; float *qbound = nullptr; };   // qbound: pre-seeded bounds (else +inf)
__global__ void tc_fill_inf_kernel(float *p, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = INFINITY;
}

// nkb = the 64-column k-blocks of K' to multiply; a timed pass records its K in the search statistics
static int tc_run_units(ThreadCtx &t, const TcOperand &A, int64_t a_rows, const TcOperand &B, int64_t b_rows, const std::vector<TcUnit> &units,
                        int64_t nlists, float **part_d, int **part_i, float **part_thr, bool timed, bool pair, int nkb, int kp, const TcShare *share) {
    CUtensorMap map_a, map_b;
    int rc = make_map(&map_a, A.bf, (uint64_t)a_rows, (uint64_t)A.kprime, BM);
    if (rc) return rc;
    rc = make_map(&map_b, B.bf, (uint64_t)b_rows, (uint64_t)B.kprime, pair ? TcCfg<true>::kBRows : TcCfg<false>::kBRows);
    if (rc) return rc;
    TcUnit *dunits = (TcUnit *)arena_alloc(t, sizeof(TcUnit) * (units.size() ? units.size() : 1));
    *part_d = (float *)arena_alloc(t, sizeof(float) * (size_t)nlists * kp);
    *part_i = (int *)arena_alloc(t, sizeof(int) * (size_t)nlists * kp);
    *part_thr = (float *)arena_alloc(t, sizeof(float) * (size_t)nlists);
    if (!dunits || !*part_d || !*part_i || !*part_thr) return MO_RC_INTERNAL_ERROR;
    tc_fill_kernel<<<num_sms() * 4, 256, 0, t.stream>>>(*part_thr, *part_i, nlists, kp);
    MOB_LAUNCH_CHECK();
    if (units.empty()) return MO_RC_SUCCESS;
    MOB_CUDA_TRY(cudaMemcpyAsync(dunits, units.data(), sizeof(TcUnit) * units.size(), cudaMemcpyHostToDevice, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    static bool attr = false;
    const size_t smem = sizeof(TcSmem) + 1024;
    if (!attr) {
        MOB_CUDA_TRY(cudaFuncSetAttribute(tc_candidates_kernel<false, KP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        MOB_CUDA_TRY(cudaFuncSetAttribute(tc_candidates_kernel<false, KP_LONG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        MOB_CUDA_TRY(cudaFuncSetAttribute(tc_candidates_kernel<true, KP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    const int nunits = (int)units.size();
    float *qbound = nullptr; const int *row_query = nullptr; const float *alonorm = A.lonorm, *xmax2 = nullptr;
    int sh_one = 0, sh_k = 0; float sh_rel = 0.f, sh_abs = 0.f;
    if (share && !A.enorm && g_tc_share_mode != 1) {   // inner product leaves the norms out of the epilogue (A.enorm = zeros): no sharing there
        qbound = share->qbound;
        if (!qbound) {
            qbound = (float *)arena_alloc(t, (size_t)share->nq * 4);
            if (!qbound) return MO_RC_INTERNAL_ERROR;
            tc_fill_inf_kernel<<<num_sms() * 2, 256, 0, t.stream>>>(qbound, share->nq);
            MOB_LAUNCH_CHECK();
        }
        row_query = share->row_query; xmax2 = share->xmax2; sh_one = share->one_term; sh_k = share->topk; sh_rel = share->rel_margin; sh_abs = share->abs_margin;
    }
    int *sched = nullptr;   // the unit counter of single-CTA launches
    if (!pair) {
        sched = (int *)arena_alloc(t, 4);
        if (!sched) return MO_RC_INTERNAL_ERROR;
        MOB_CUDA_TRY(cudaMemsetAsync(sched, 0, 4, t.stream));
    }
    if (timed) { t.kev_prio = 2; g_search_stats.kused = nkb * BK; cudaEventRecord(t.kev0, t.stream); }   // MoB200_LastKernelMs reports the first (whole-list) pass, not the refine pass
    if (!pair) {
        int grid = num_sms();
        if (grid > nunits) grid = nunits;
        if (kp == KP_LONG) tc_candidates_kernel<false, KP_LONG><<<grid, kTcThreads, smem, t.stream>>>(map_a, map_b, dunits, nunits, nkb, A.enorm ? A.enorm : A.norm, B.enorm ? B.enorm : B.norm, *part_d, *part_i, *part_thr, qbound, row_query, alonorm, xmax2, sh_one, sh_k, sh_rel, sh_abs, sched);
        else tc_candidates_kernel<false, KP><<<grid, kTcThreads, smem, t.stream>>>(map_a, map_b, dunits, nunits, nkb, A.enorm ? A.enorm : A.norm, B.enorm ? B.enorm : B.norm, *part_d, *part_i, *part_thr, qbound, row_query, alonorm, xmax2, sh_one, sh_k, sh_rel, sh_abs, sched);
    } else {
        if (kp != KP) { set_error("tc search: CTA pairs keep %d candidates per list", KP); return MO_RC_INTERNAL_ERROR; }
        // clusters of two CTAs that share the B tile: one persistent pair per two SMs
        int pairs = num_sms() / 2;
        if (pairs > nunits) pairs = nunits;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(2 * pairs)); cfg.blockDim = dim3(kTcThreads); cfg.dynamicSmemBytes = smem; cfg.stream = t.stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        const float *an = A.enorm ? A.enorm : A.norm, *bn = B.enorm ? B.enorm : B.norm;
        MOB_CUDA_TRY(cudaLaunchKernelEx(&cfg, tc_candidates_kernel<true, KP>, map_a, map_b, (const TcUnit *)dunits, nunits, nkb, an, bn, *part_d, *part_i, *part_thr, qbound, row_query, alonorm, xmax2, sh_one, sh_k, sh_rel, sh_abs, (int *)nullptr));
    }
    if (timed) cudaEventRecord(t.kev1, t.stream);
    MOB_LAUNCH_CHECK();
    return MO_RC_SUCCESS;
}

// largest |x|^2 and |x - hi(x)|^2 over the row operand (the error bounds use them): two floats in the call's arena
static int tc_operand_max(ThreadCtx &t, const TcOperand &B, int64_t n, bool with_lo, float **xmax2) {
    *xmax2 = (float *)arena_alloc(t, 16);
    if (!*xmax2) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(*xmax2, 0, 8, t.stream));
    tc_max_kernel<<<num_sms() * 2, 256, 0, t.stream>>>(B.norm, n, *xmax2);
    MOB_LAUNCH_CHECK();
    if (with_lo) { tc_max_kernel<<<num_sms() * 2, 256, 0, t.stream>>>(B.lonorm, n, *xmax2 + 1); MOB_LAUNCH_CHECK(); }
    return MO_RC_SUCCESS;
}

// filtered search, masked scan: the norms the epilogue adds become +inf for rows that are not admitted, so every approximate distance
// of such a row is +inf -- it is never listed and never lowers a list's threshold (DESIGN.md section 5.7)
__global__ void tc_mask_norms_kernel(const float *__restrict__ norm, const uint32_t *__restrict__ admit, int64_t n, float *__restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = ((admit[i >> 5] >> (i & 31)) & 1u) ? norm[i] : INFINITY;
}
static int tc_mask_norms(ThreadCtx &t, TcOperand &B, int64_t n, const uint32_t *admit) {
    float *masked = (float *)arena_alloc(t, (size_t)(n > 0 ? n : 1) * 4);
    if (!masked) return MO_RC_INTERNAL_ERROR;
    if (n > 0) { tc_mask_norms_kernel<<<num_sms() * 4, 256, 0, t.stream>>>(B.enorm ? B.enorm : B.norm, admit, n, masked); MOB_LAUNCH_CHECK(); }
    B.enorm = masked;
    return MO_RC_SUCCESS;
}

// merge approximate lists -> exact re-score -> final order + proof; returns the queries whose proof failed
// A = the query operand of the candidate pass, one row per query, or per (query, probed list) pair (IVF: pairs, lists found
// through pos_map); nkb = the k-blocks the pass ran and one_term = it was hi-only (its error bound depends on both);
// xmax2 = the largest |x|^2 and |x - hi(x)|^2 of the row operand (tc_operand_max)
static int tc_finish(ThreadCtx &t, const float *ddata, int dim, const float *dq, int64_t nq, int k, int metric, const TcOperand &A, bool pairs,
                     bool one_term, int nkb, const float *xmax2, int R, const int *pos_map, int pos_cols, long long pos_stride,
                     const float *part_d, const int *part_i, const float *part_thr, int kp,
                     const int64_t *id_map, int64_t key_base, int sqrt_out, int64_t *out_k, double *out_d, std::vector<int> &redo) {
    const bool l2 = metric != MO_METRIC_IP && metric != MO_METRIC_COS;
    const int kr = (k > KP || one_term) ? KR_WIDE : KR;   // a looser approximation needs more exact re-scores to prove the top k
    int *cand = (int *)arena_alloc(t, sizeof(int) * (size_t)nq * kr);
    float *exact = (float *)arena_alloc(t, sizeof(float) * (size_t)nq * kr);
    float *t_excl = (float *)arena_alloc(t, sizeof(float) * (size_t)nq);
    int *flags = (int *)arena_alloc(t, sizeof(int) * (size_t)nq);
    if (!cand || !exact || !t_excl || !flags) return MO_RC_INTERNAL_ERROR;
    const float *qnorm = pairs ? nullptr : A.norm, *qlonorm = pairs ? nullptr : A.lonorm;
    const float *pair_norm = pairs ? A.norm : nullptr, *pair_lonorm = pairs ? A.lonorm : nullptr;
    if (R > kMaxMergeLists) { set_error("tc search: %d candidate lists per query exceed the merge limit %d", R, kMaxMergeLists); return MO_RC_INTERNAL_ERROR; }
    tc_merge_kernel<<<(unsigned)((nq + 3) / 4), 128, 0, t.stream>>>((int)nq, R, part_d, part_i, part_thr, pos_map, pos_cols, pos_stride, pair_norm, pair_lonorm, xmax2, one_term, qnorm, qlonorm, l2 ? k : (1 << 30) /* pruning bound is L2-specific */, dim, nkb, kp, kr, cand, t_excl);
    MOB_LAUNCH_CHECK();
    {
        const size_t smem = (size_t)(kRescoreThreads / 32) * godist::RingCfg<false>::kStages * godist::RingCfg<false>::kStageBytes;
        static bool attr = false;
        if (!attr) {
            MOB_CUDA_TRY(cudaFuncSetAttribute(tc_rescore_kernel<MO_METRIC_L2SQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            MOB_CUDA_TRY(cudaFuncSetAttribute(tc_rescore_kernel<MO_METRIC_IP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            MOB_CUDA_TRY(cudaFuncSetAttribute(tc_rescore_kernel<MO_METRIC_COS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr = true;
        }
        int64_t blocks = (nq * (kr / 32) + kRescoreThreads / 32 - 1) / (kRescoreThreads / 32);
        if (blocks > 2ll * num_sms()) blocks = 2ll * num_sms();
        if (metric == MO_METRIC_IP) tc_rescore_kernel<MO_METRIC_IP><<<(unsigned)blocks, kRescoreThreads, smem, t.stream>>>(ddata, dq, dim, (int)nq, kr, cand, exact);
        else if (metric == MO_METRIC_COS) tc_rescore_kernel<MO_METRIC_COS><<<(unsigned)blocks, kRescoreThreads, smem, t.stream>>>(ddata, dq, dim, (int)nq, kr, cand, exact);
        else tc_rescore_kernel<MO_METRIC_L2SQ><<<(unsigned)blocks, kRescoreThreads, smem, t.stream>>>(ddata, dq, dim, (int)nq, kr, cand, exact);
        MOB_LAUNCH_CHECK();
    }
    if (kr == KR) tc_final_kernel<KR><<<(unsigned)((nq + 127) / 128), 128, 0, t.stream>>>((int)nq, k, dim, nkb, cand, exact, t_excl, qnorm, xmax2, qlonorm, xmax2 + 1, one_term, pairs, metric, id_map, key_base, sqrt_out, out_k, out_d, flags);
    else tc_final_kernel<KR_WIDE><<<(unsigned)((nq + 127) / 128), 128, 0, t.stream>>>((int)nq, k, dim, nkb, cand, exact, t_excl, qnorm, xmax2, qlonorm, xmax2 + 1, one_term, pairs, metric, id_map, key_base, sqrt_out, out_k, out_d, flags);
    MOB_LAUNCH_CHECK();
    std::vector<int> hflags((size_t)nq);
    MOB_CUDA_TRY(cudaMemcpyAsync(hflags.data(), flags, sizeof(int) * (size_t)nq, cudaMemcpyDeviceToHost, t.stream));
    MOB_CUDA_TRY(cudaStreamSynchronize(t.stream));
    redo.clear();
    for (int64_t q = 0; q < nq; q++) if (hflags[(size_t)q]) redo.push_back((int)q);
    return MO_RC_SUCCESS;
}

// Number of row ranges for a brute-force search: units (range r, query tile m) are dealt round-robin to `workers` persistent
// CTAs, so the makespan is the heaviest worker's tile count.  Pick the R in [rmin, rcap] with the smallest makespan;
// every unit also pays a fixed cost (list init + write-out, more insertions while the list is young) counted as one tile.
// rmin comes from the L2: the query tiles of a range run on different SMs at about the same time, and only a range that
// stays L2-resident while they sweep it is read from HBM once.
static int plan_ranges(int64_t ntiles, int mt, int workers, int rmin, int rcap) {
    int best = 1; double best_cost = 1e300;
    const int rmax = (int)(ntiles < rcap ? ntiles : rcap);
    if (rmin > rmax) rmin = rmax;
    if (rmin < 1) rmin = 1;
    std::vector<double> load((size_t)workers);
    for (int R = rmin; R <= rmax; R++) {
        const int64_t per = (ntiles + R - 1) / R;
        const int reff = (int)((ntiles + per - 1) / per);
        if (reff != R) continue;   // same partition as a smaller R
        std::fill(load.begin(), load.end(), 0.0);
        size_t u = 0;
        for (int r = 0; r < R; r++) {
            const double tiles = (double)((r + 1) * per <= ntiles ? per : ntiles - r * per) + 1.0;
            for (int m = 0; m < mt; m++, u++) load[u % (size_t)workers] += tiles;
        }
        double cost = 0;
        for (double l : load) cost = l > cost ? l : cost;
        if (cost < best_cost * 0.999) { best_cost = cost; best = R; }
    }
    return best;
}

// the masked scan costs what the unfiltered search costs; the compacted search costs the gather of the admitted rows plus a search
// over them whose operand is split per call, not prepared.  Measured crossover (DESIGN.md section 5.12): brute force between 1/2 and
// all rows admitted, IVF between 1/10 and 1/2 (the unfiltered IVF scan is cheap next to the per-call residual split).
bool filter_compact_wanted(int64_t n, int64_t admitted, bool ivf) {
    if (g_filter_path == 1) return false;
    if (g_filter_path == 2) return true;
    return ivf ? admitted * 5 <= n : admitted * 4 <= 3 * n;
}

bool tc_search_applicable(int64_t n, int dim, int64_t nq, int k, int metric) {
    if (g_search_mode == 1) return false;
    // k <= KP: one candidate list per (query, row range); KP < k <= KW ("wide", centroid probes): ranges of >= 128 rows, at least 8 of them
    const bool metric_ok = metric == MO_METRIC_L2 || metric == MO_METRIC_L2SQ || metric == MO_METRIC_IP || metric == MO_METRIC_COS;
    const bool shape_ok = metric_ok && k >= 1 && dim >= 16 && n < (1ll << 31) - BN && (k <= KP ? n >= BN : (k <= KW && n >= 1024));
    if (g_search_mode == 2) return shape_ok;
    // below this the exact kernel wins (operand split + launch overheads).  The second clause is centroid assignment at index build
    // (Productl2.probeRun, product_l2.go:317-407): a small table (nlist rows) against a very large batch of queries.
    return shape_ok && nq >= 256 && dim >= 64 && (n >= 16384 || (n >= 1024 && nq >= 65536));
}

// centroid probe of an IVF search (findCentroids): many queries against a small table, k = nprobe
bool tc_probe_applicable(int64_t nlist, int dim, int64_t nq, int nprobe, int metric) {
    if (g_search_mode == 1) return false;
    const bool shape_ok = (metric == MO_METRIC_L2 || metric == MO_METRIC_L2SQ) && nprobe >= 1 && dim >= 16 &&
                          (nprobe <= KP ? nlist >= BN : (nprobe <= KW && nlist >= 1024));
    if (g_search_mode == 2) return shape_ok;
    return shape_ok && nq >= 1024 && dim >= 64;
}

bool tc_ivf_applicable(int64_t n, int dim, int64_t nq, int k, int nprobe, int metric, bool refine) {
    if (g_search_mode == 1) return false;
    const bool shape_ok = (metric == MO_METRIC_L2 || metric == MO_METRIC_L2SQ) && k >= 1 && k <= KP && dim >= 16 && n >= 1 && n < (1ll << 31) - BN &&
                          nprobe <= 64 && nq * (int64_t)nprobe < (1ll << 31);
    if (g_search_mode == 2 || refine) return shape_ok;
    return shape_ok && nq * (int64_t)nprobe >= 8192 && dim >= 64;
}

// Brute-force top-k through the tensor-core candidate pass; results are the exact answer (see file header).
// A precision ladder: level 0 runs only the first dim columns of K' (the hi.hi product, a third of the flop) and proves what it
// can with the looser one-term error bound; level 1 re-runs the unproven queries over the whole K' (three-term product); what is
// still unproven goes to the exact kernel.  Every level answers its queries exactly or hands them down.
void tc_one_term_report(int64_t nq, int64_t failed);
static int bf_tc_level(ThreadCtx &t, int level, int metric, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq, int k,
                       int64_t key_base, int sqrt_out, int64_t *out_k, double *out_d, bool record_stats, bool timed, const uint32_t *admit) {
    if (level >= 2) {
        if (record_stats) g_search_stats.fallbacks = (int)nq;
        return bruteforce_topk_device(t, ddata, n, dim, dq, nq, k, metric, key_base, sqrt_out, out_k, out_d, admit);
    }
    const int normalize = metric == MO_METRIC_COS ? 1 : 0;
    int *dnonfinite = (int *)arena_alloc(t, 4);
    if (!dnonfinite) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dnonfinite, 0, 4, t.stream));
    TcOperand A, B;
    int rc = tc_prepare(t, dq, nq, dim, 0, normalize, nullptr, 0, nullptr, dnonfinite, A);
    if (!rc) rc = tc_prepare(t, ddata, n, dim, 1, normalize, nullptr, 0, nullptr, dnonfinite, B);
    if (rc) return rc;
    int hnonfinite = 0;
    rc = read_back(t, &hnonfinite, dnonfinite, 4);
    if (rc) return rc;
    if (hnonfinite)   // the error bound of the tensor-core pass does not apply to Inf/NaN inputs (cosine: nor to zero vectors)
        return bf_tc_level(t, 2, metric, ddata, n, dim, dq, nq, k, key_base, sqrt_out, out_k, out_d, record_stats, false, admit);
    if (metric == MO_METRIC_IP) {   // -q.x: the epilogue adds no norms (the candidate kernel then works in units of -2 q.x)
        float *zeros = (float *)arena_alloc(t, (size_t)(n > nq ? n : nq) * 4);
        if (!zeros) return MO_RC_INTERNAL_ERROR;
        MOB_CUDA_TRY(cudaMemsetAsync(zeros, 0, (size_t)(n > nq ? n : nq) * 4, t.stream));
        A.enorm = zeros; B.enorm = zeros;
    }
    if (admit) {   // filtered search: the prepared operand is used as it is; only the norms its epilogue adds are masked
        int rc2 = tc_mask_norms(t, B, n, admit);
        if (rc2) return rc2;
    }
    const bool one_term = level == 0;
    const int nkb = one_term ? (dim + BK - 1) / BK : A.kprime / BK;
    // work units: (query tile, row range); ranges sized so that units ~ a whole number of waves over the SMs
    // enough queries to fill 256-row units: CTA pairs share the B tile (TMA multicast) and load 1.33x fewer bytes per flop
    const bool pair = g_tc_pair_mode == 2 || (g_tc_pair_mode == 0 && nq >= 1024);
    const int tile_m = pair ? TcCfg<true>::kTileM : TcCfg<false>::kTileM;
    const int mt = (int)((nq + tile_m - 1) / tile_m);
    const int64_t ntiles = (n + BN - 1) / BN;
    const int workers = pair ? num_sms() / 2 : num_sms();
    int rmin = 1;
    if (g_tc_range_mb > 0) {   // experiment knob: cap the bytes of one row range (L2 residency)
        const int64_t tile_bytes = (int64_t)BN * nkb * BK * 2;
        int64_t tiles_fit = ((int64_t)g_tc_range_mb << 20) / tile_bytes;
        if (tiles_fit < 4) tiles_fit = 4;
        rmin = (int)((ntiles + tiles_fit - 1) / tiles_fit);
    }
    int R = plan_ranges(ntiles, mt, workers, rmin, rmin > 64 ? kMaxMergeLists : 64);
    int64_t range_rows = (ntiles + R - 1) / R * BN;
    if (k > KP) {   // wide mode: R * KP candidates must comfortably exceed k -> short ranges (the MMA tile is masked beyond n_end)
        range_rows = ((n + 63) / 64 + 127) / 128 * 128;
        if (range_rows < 128) range_rows = 128;
    }
    R = (int)((n + range_rows - 1) / range_rows);
    std::vector<TcUnit> units;
    for (int r = 0; r < R; r++)
        for (int m = 0; m < mt; m++) {
            TcUnit u; u.a_row0 = m * tile_m; u.a_valid = (int)(nq - u.a_row0 < tile_m ? nq - u.a_row0 : tile_m);
            u.n_begin = (int)(r * range_rows); u.n_end = (int)((r + 1) * range_rows < n ? (r + 1) * range_rows : n);
            u.out_base = (long long)r * nq + u.a_row0;
            if (u.n_begin < u.n_end) units.push_back(u);
        }
    float *part_d, *part_thr; int *part_i;
    float *xmax2 = nullptr;
    rc = tc_operand_max(t, B, n, one_term, &xmax2);
    if (rc) return rc;
    // margins of the shared bound in kernel units: L2 relative 4 dim 2^-23; cosine absolute (its Go-order error does not scale with the distance)
    TcShare sh{nq, nullptr, k, one_term ? 1 : 0, metric == MO_METRIC_COS ? 0.f : (float)dim * 4.76837158203125e-7f,
               metric == MO_METRIC_COS ? 2.0f * ((float)dim * 4.76837158203125e-7f + 3.814697265625e-6f) : 0.f, xmax2};
    rc = tc_run_units(t, A, nq, B, n, units, (int64_t)R * nq, &part_d, &part_i, &part_thr, timed, pair, nkb, KP, k <= KP ? &sh : nullptr);
    if (rc) return rc;
    if (!record_stats) g_search_stats.probe_kused = nkb * BK;   // an IVF centroid probe: the K of its last pass
    std::vector<int> redo;
    rc = tc_finish(t, ddata, dim, dq, nq, k, metric, A, false, one_term, nkb, xmax2, R, nullptr, 0, 0, part_d, part_i, part_thr, KP,
                   nullptr, key_base, sqrt_out, out_k, out_d, redo);
    if (rc) return rc;
    if (record_stats && level == 0) {
        g_search_stats.refined = (int)redo.size();
        tc_one_term_report(nq, (int64_t)redo.size());
    }
    // queries whose completeness could not be proven: next level
    return redo_queries(t, redo, dq, dim, k, out_k, out_d, [&](const float *sub, int64_t m, int64_t *sk, double *sd) {
        return bf_tc_level(t, level + 1, metric, ddata, n, dim, sub, m, k, key_base, sqrt_out, sk, sd, record_stats, false, admit);
    });
}

void search_invalidate(const void *p, uint64_t bytes) {
    const char *lo = (const char *)p, *hi = lo + bytes;
    auto overlaps = [&](const void *b, size_t len) { return b && lo < (const char *)b + len && (const char *)b < hi; };
    drop_prepared([&](const PreparedOperand &e) {   // the residual operand depends on the centroids and the list boundaries too
        return overlaps(e.x, (size_t)e.n * e.dim * 4) || overlaps(e.cent, (size_t)e.nlist * e.dim * 4) || overlaps(e.offsets, (size_t)(e.nlist + 1) * 8);
    });
}

// the one-term level needs k <= KP (its proof re-scores 64 candidates) and is skipped while it has recently been failing
bool tc_one_term_wanted(int k, bool record) {
    if (k > KP || g_tc_ladder_mode == 1) return false;
    if (g_tc_ladder_mode == 2) return true;
    if (g_one_term_skip.load() > 0) { if (record) g_one_term_skip.fetch_sub(1); return false; }
    return true;
}
// a dataset whose norms dwarf its neighbour distances defeats the one-term bound: stop trying for a while
void tc_one_term_report(int64_t nq, int64_t failed) { if (nq >= 64 && failed * 5 > nq * 2) g_one_term_skip.store(16); }

int bruteforce_topk_tc_device(ThreadCtx &t, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq, int k,
                              int64_t key_base, int sqrt_out, int64_t *out_k, double *out_d, bool record_stats, int metric, const uint32_t *admit) {
    const bool ladder = tc_one_term_wanted(k, record_stats);
    if (record_stats) g_search_stats.fallbacks = 0;   // the search reached the tensor cores
    if (metric == MO_METRIC_L2) metric = MO_METRIC_L2SQ;
    return bf_tc_level(t, ladder ? 0 : 1, metric, ddata, n, dim, dq, nq, k, key_base, sqrt_out, out_k, out_d, record_stats, record_stats, admit);
}

// IVF list scan on the tensor cores: the queries probing a list are gathered (as split bf16 rows) next to each other, so
// a (list, 128-query tile) pair is one work unit of the same candidate kernel; every (query, probe rank) pair owns one list.
int ivf_tc_scan(ThreadCtx &t, const IvfPlan &plan, const float *ddata, int64_t n, int dim, const float *dq, int64_t nq,
                const float *dcent, const int64_t *doffsets, const std::vector<int64_t> &offsets, const int64_t *drowids, int k, int sqrt_out,
                int pass, int64_t *ok, double *od, std::vector<int> &redo, bool *nonfinite, const uint32_t *admit) {
    // pass 0: hi-only product over whole lists (one term), pass 1: three-term product over whole lists, pass 2 (refine): three-term
    // product with every list cut into sub-ranges of `chunk` rows, each keeping its own KP candidates, so the excluded-row
    // threshold of a (query, list) pair moves far away from the k-th result
    *nonfinite = false;
    const bool one_term = pass == 0, refine = pass == 2;
    const int64_t nlist = (int64_t)offsets.size() - 1;
    int split = 1; int64_t chunk = (int64_t)1 << 40;
    int64_t maxlen = 1;
    for (int64_t l = 0; l < nlist; l++) if (plan.hcnt[(size_t)l] > 0 && offsets[(size_t)l + 1] - offsets[(size_t)l] > maxlen) maxlen = offsets[(size_t)l + 1] - offsets[(size_t)l];
    if (refine) split = (int)((maxlen + BN - 1) / BN);
    if (split > 1) {
        const int cap = kMaxMergeLists / plan.nprobe > 0 ? kMaxMergeLists / plan.nprobe : 1;
        if (split > cap) split = cap;
        chunk = ((maxlen + split - 1) / split + BN - 1) / BN * BN;
    }
    int *dnonfinite = (int *)arena_alloc(t, 4);
    if (!dnonfinite) return MO_RC_INTERNAL_ERROR;
    MOB_CUDA_TRY(cudaMemsetAsync(dnonfinite, 0, 4, t.stream));
    // operands are residuals against the list centroid: entries prepared at index load (or once per call), queries per (query, list) pair
    TcOperand B, A;
    int rc = tc_prepare(t, ddata, n, dim, 1, 0, dcent, nlist, doffsets, dnonfinite, B);
    if (!rc) rc = tc_alloc(t, plan.npairs, dim, A);
    if (rc) return rc;
    split_residual_kernel<<<num_sms() * 8, 256, 0, t.stream>>>(dq, plan.nvalid, dim, A.kprime, 0, dcent, nullptr, nlist, plan.bucket_q, plan.bucket_l,
                                                               A.bf, A.norm, A.lonorm, dnonfinite, one_term ? 1 : 0);
    MOB_LAUNCH_CHECK();
    int hnonfinite = 0;
    rc = read_back(t, &hnonfinite, dnonfinite, 4);
    if (rc) return rc;
    if (hnonfinite) { *nonfinite = true; redo.resize((size_t)nq); for (int64_t q = 0; q < nq; q++) redo[(size_t)q] = (int)q; return MO_RC_SUCCESS; }
    if (admit && (rc = tc_mask_norms(t, B, n, admit)) != 0) return rc;
    std::vector<TcUnit> units;
    for (int64_t l = 0; l < nlist; l++) {
        const int c = plan.hcnt[(size_t)l];
        if (c == 0 || offsets[(size_t)l + 1] <= offsets[(size_t)l]) continue;
        for (int q0 = 0; q0 < c; q0 += BM)
            for (int s = 0; s < split; s++) {
                TcUnit u; u.a_row0 = plan.hstart[(size_t)l] + q0; u.a_valid = c - q0 < BM ? c - q0 : BM;
                const int64_t b = offsets[(size_t)l] + s * chunk, e = b + chunk < offsets[(size_t)l + 1] ? b + chunk : offsets[(size_t)l + 1];
                if (b >= e) break;
                u.n_begin = (int)b; u.n_end = (int)e; u.out_base = (long long)s * plan.npairs + u.a_row0;
                units.push_back(u);
            }
    }
    float *part_d, *part_thr; int *part_i;
    // one-term pass: the looser bound needs the list threshold further from the k-th result -> 32 candidates per (query, list).
    // (Measured alternative: two half-lists of 16 each made the kernel 16 % faster but left a few queries to the refine pass, whose
    // fixed cost outweighs that.)
    const int kp = one_term ? KP_LONG : KP;
    float *xmax2 = nullptr;
    rc = tc_operand_max(t, B, n, one_term, &xmax2);
    if (rc) return rc;
    TcShare sh{nq, plan.bucket_q, k, one_term ? 1 : 0, (float)dim * 4.76837158203125e-7f, 0.f, xmax2};
    if (k <= 32 && g_tc_share_mode == 0) {
        sh.qbound = (float *)arena_alloc(t, (size_t)nq * 4);
        if (!sh.qbound) return MO_RC_INTERNAL_ERROR;
        tc_fill_inf_kernel<<<num_sms() * 2, 256, 0, t.stream>>>(sh.qbound, nq);
        MOB_LAUNCH_CHECK();
        const size_t smem = (size_t)(kRescoreThreads / 32) * godist::RingCfg<false>::kStages * godist::RingCfg<false>::kStageBytes;
        static bool attr = false;
        if (!attr) { MOB_CUDA_TRY(cudaFuncSetAttribute(ivf_seed_bound_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
        int64_t blocks = (nq + kRescoreThreads / 32 - 1) / (kRescoreThreads / 32);
        if (blocks > 2ll * num_sms()) blocks = 2ll * num_sms();
        ivf_seed_bound_kernel<<<(unsigned)blocks, kRescoreThreads, smem, t.stream>>>(ddata, dq, dim, (int)nq, plan.nprobe, k, plan.probes, doffsets, sh.qbound, admit);
        MOB_LAUNCH_CHECK();
    }
    const int nkb = one_term ? (dim + BK - 1) / BK : A.kprime / BK;
    rc = tc_run_units(t, A, plan.npairs, B, n, units, plan.npairs * split, &part_d, &part_i, &part_thr, !refine, false, nkb, kp, &sh);
    if (rc) return rc;
    // the approximate lists are indexed by bucket position; tc_finish walks them per query through pair_pos; the final keys are
    // the primary keys row_ids[local row]; every probed list's exclusion bound is lowered by the error bound of ITS operand pair
    return tc_finish(t, ddata, dim, dq, nq, k, MO_METRIC_L2SQ, A, true, one_term, nkb, xmax2, plan.nprobe * split, plan.pair_pos, plan.nprobe, plan.npairs,
                     part_d, part_i, part_thr, kp, drowids, 0, sqrt_out, ok, od, redo);
}

// index load: split e's rows (e.cent != nullptr: IVF residuals) into an operand in device memory of its own and register it.  It
// replaces only the operand of the same kind (brute force with the same normalisation, or IVF): preparing COS after L2, or IVF after
// brute force, on one dataset keeps the earlier operand (ADVICE r01).  Rows with Inf/NaN values are left unprepared.
static int32_t search_prepare(ThreadCtx &t, PreparedOperand e, const char *what) {
    drop_prepared([&](const PreparedOperand &o) { return o.x == e.x && !o.cent == !e.cent && (e.cent || o.normalized == e.normalized); });
    e.op.kprime = tc_kprime(e.dim);
    MOB_CUDA_TRY(cudaMalloc((void **)&e.op.bf, (size_t)e.n * e.op.kprime * 2 + 1024));
    if (cudaMalloc((void **)&e.op.norm, (size_t)e.n * 8) != cudaSuccess) { free_prepared(e.op); set_error("%s: out of device memory", what); return MO_RC_INTERNAL_ERROR; }
    e.op.lonorm = e.op.norm + e.n;
    int *dnonfinite = (int *)arena_alloc(t, 4);
    int hnonfinite = 1;
    int rc = dnonfinite ? MO_RC_SUCCESS : MO_RC_INTERNAL_ERROR;
    if (!rc && cudaMemsetAsync(dnonfinite, 0, 4, t.stream) != cudaSuccess) rc = MO_RC_INTERNAL_ERROR;
    if (!rc) {
        if (e.cent) split_residual_kernel<<<num_sms() * 8, 256, 0, t.stream>>>(e.x, e.n, e.dim, e.op.kprime, 1, e.cent, e.offsets, e.nlist, nullptr, nullptr,
                                                                               e.op.bf, e.op.norm, e.op.lonorm, dnonfinite, 0);
        else split_kernel<<<num_sms() * 8, 256, 0, t.stream>>>(e.x, e.n, e.dim, e.op.kprime, 1, e.normalized, e.op.bf, e.op.norm, e.op.lonorm, dnonfinite);
        g_launches++;
        if (cudaGetLastError() != cudaSuccess) rc = MO_RC_INTERNAL_ERROR;
    }
    if (!rc) rc = read_back(t, &hnonfinite, dnonfinite, 4);
    arena_reset(t);
    if (rc || hnonfinite) { free_prepared(e.op); return rc; }
    std::lock_guard<std::mutex> lk(g_prepared_mu);
    g_prepared.push_back(e);
    return MO_RC_SUCCESS;
}

}  // namespace mob

extern "C" {

// Index load: split a RESIDENT dataset into the tensor-core operand once instead of once per search.  The rows must not change
// until MoB200_SearchRelease(data).  Datasets the tensor-core path cannot serve (dim < 16, Inf/NaN values) are left unprepared:
// searches on them behave exactly as without this call.
int32_t MoB200_SearchPrepare(const void *data, uint64_t n, int64_t dim) { return MoB200_SearchPrepareMetric(data, n, dim, MO_METRIC_L2); }

// metric: MO_METRIC_L2 / L2SQ / IP share one operand; MO_METRIC_COS keeps the rows normalised; other metrics: nothing to prepare
int32_t MoB200_SearchPrepareMetric(const void *data, uint64_t n, int64_t dim, int32_t metric) {
    using namespace mob;
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (metric != MO_METRIC_L2 && metric != MO_METRIC_L2SQ && metric != MO_METRIC_IP && metric != MO_METRIC_COS) return MO_RC_SUCCESS;
    if (!data || n == 0 || dim < 16 || n >= (1ull << 31) - BN) return MO_RC_SUCCESS;
    if (!is_device_ptr(data)) { set_error("SearchPrepare: the dataset must be device memory"); return MO_RC_INVALID_ARGUMENT; }
    PreparedOperand e; e.x = (const float *)data; e.n = (int64_t)n; e.dim = (int)dim; e.normalized = metric == MO_METRIC_COS ? 1 : 0;
    return search_prepare(t, e, "SearchPrepare");
}

// Index load for an IVF-flat index: the list-ordered entries [n][dim] are split as RESIDUALS against their list's centroid
// (centroids [nlist][dim], offsets [nlist + 1] int64; all device pointers).  Same contract as MoB200_SearchPrepare.
int32_t MoB200_SearchPrepareIvf(const void *data, uint64_t n, int64_t dim, const void *centroids, uint64_t nlist, const void *offsets) {
    using namespace mob;
    ThreadCtx &t = tctx();
    if (!t.ready) return MO_RC_INTERNAL_ERROR;
    if (!data || n == 0 || dim < 16 || n >= (1ull << 31) - BN || nlist == 0) return MO_RC_SUCCESS;
    if (!is_device_ptr(data) || !is_device_ptr(centroids) || !is_device_ptr(offsets)) { set_error("SearchPrepareIvf: entries, centroids and offsets must be device memory"); return MO_RC_INVALID_ARGUMENT; }
    PreparedOperand e; e.x = (const float *)data; e.n = (int64_t)n; e.dim = (int)dim; e.cent = (const float *)centroids; e.nlist = (int64_t)nlist; e.offsets = (const int64_t *)offsets;
    return search_prepare(t, e, "SearchPrepareIvf");
}

// also drops IVF operands built against `data` as their centroid table (residuals would be stale)
int32_t MoB200_SearchRelease(const void *data) {
    mob::drop_prepared([&](const mob::PreparedOperand &e) { return e.x == data || (e.cent && (const void *)e.cent == data); });
    return MO_RC_SUCCESS;
}

}  // extern "C"
