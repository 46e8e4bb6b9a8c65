// pfz_dense.cu -- K4: dense cosine top-k for pre-computed embeddings: C = X * Y^T on the Hopper tensor cores
// (wgmma, bf16 in, fp32 accumulate in registers) fed by TMA, with the per-row top-k fused into the epilogue so
// the n_from x n_to score matrix never exists in memory.
//
// Replaces the dense branch of polyfuzz/models/_utils.py:94-102 (sklearn cosine_similarity + argsort) as
// reached from polyfuzz/models/_embeddings.py:127-131 when the caller supplies embeddings.
//
// CTA = 128 from-rows.  Per DN-wide to-tile: K loop of 64-element (128-byte, SWIZZLE_128B) TMA boxes through a
// shared-memory ring of full / empty mbarriers.  Warps 0-7 are two consumer warpgroups (from-rows 0-63 and 64-127
// of the block), each issuing wgmma m64nDNk16 into DN/2 fp32 registers per thread; warp 8 is the TMA producer.
// The wgmma accumulator layout gives each thread two rows (r and r + 8 of its warp's 16) and DN/4 columns of each:
// the thread keeps a sorted top-k per row over its columns (key: score desc, index asc), and the four threads of a
// quad merge their lists with shuffles when a (row block, split) unit is done.  DN = 128 keeps the 64 accumulators and
// both top-k lists in registers: 9 warps per CTA leave 168 registers a thread, and DN = 256 spilled.
//
// Cluster variant (MCAST): a pair of CTAs (cluster of 2) works on two adjacent 128-row blocks against the same
// to-tiles.  Each CTA loads one half of the Y tile and multicasts it into both CTAs' shared memory, which halves
// the to-operand L2 -> SM traffic per CTA; a stage is refilled only once the consumers of both CTAs released it.
//
// Exact mode (Embeddings(precision="fp64"), DESIGN.md 4.6): rows_prep_exact_kernel stages canonical fp64 rows and their fp16
// rounding with error bounds, the same GEMM kernel on fp16 operands filters k' candidates per row below a margin, and
// exact_rescore_kernel scores them in fp64 and certifies the row; exact_fallback_kernel scores the rows it could not certify
// against every to-row.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include "pfz_common.cuh"

namespace pfz {

constexpr int DM = 128, DN = 128, DK = 64, WG_K = 16, DSTAGES = 6;
constexpr int A_BYTES = DM * DK * 2, B_BYTES = DN * DK * 2;          // 16 KB, 16 KB
constexpr int DENSE_THREADS = 288;                                     // 2 consumer warpgroups + 1 producer warp
constexpr int DENSE_CONSUMER_WARPS = 8;
constexpr size_t DENSE_SMEM = (size_t)DSTAGES * (A_BYTES + B_BYTES) + 2 * DSTAGES * 8 + 1024;

__device__ __forceinline__ unsigned s32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_arrive_cta(unsigned bar, unsigned cta) {      // the barrier at the same offset in CTA `cta` of the cluster
    asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\tmbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
                 :: "r"(bar), "r"(cta) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
    asm volatile("{\n\t.reg .pred p;\n\tLAB_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE;\n\tbra LAB_WAIT;\n\tDONE:\n\t}"
                 :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(unsigned dst, const CUtensorMap *map, int c0, int c1, unsigned bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
// same box into the same shared-memory offset of every CTA in `mask`, completing bytes on each CTA's barrier at `bar`
__device__ __forceinline__ void tma_load_2d_mcast(unsigned dst, const CUtensorMap *map, int c0, int c1, unsigned bar, unsigned short mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%2, %3}], [%4], %5;"
                 :: "r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar), "h"(mask) : "memory");
}
__device__ __forceinline__ unsigned cluster_ctarank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared-memory matrix descriptor: K-major operand, 128-byte swizzle, 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t wgmma_desc(unsigned smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);               // start address  (bits 0-13)
    d |= (uint64_t)1 << 16;                                    // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;                          // stride byte offset (bits 32-45)
    d |= (uint64_t)1 << 62;                                    // layout: SWIZZLE_128B
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int R> __device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}
// D (+)= A[smem] * B[smem]^T, bf16 (or fp16) inputs, fp32 accumulate; scale_d == 0 overwrites D
#define PFZ_WGMMA_M64N128K16(AB)                                                                                          \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                       \
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32." AB "." AB " {"                                               \
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                    \
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                          \
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                          \
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"                            \
                 "}, %64, %65, p, 1, 1, 0, 0;\n\t}"                                                                         \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),           \
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),     \
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),   \
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),   \
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),   \
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),   \
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),   \
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])    \
                 : "l"(adesc), "l"(bdesc), "r"(scale_d))
template <bool F16>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
    if constexpr (F16) PFZ_WGMMA_M64N128K16("f16");
    else PFZ_WGMMA_M64N128K16("bf16");
}
#undef PFZ_WGMMA_M64N128K16

struct DenseParams {
    int n_from, n_to, d; int k; float min_sim; int self_match; long long from_base, to_base;
    int n_splits; int n_mblocks; int n_ntiles;
    int32_t *top_idx; double *top_val;          // [n_splits][n_from][k]
    // threshold epilogue only (appended, so the top-k instantiations read their fields at the same offsets)
    const float *row_thr; int32_t *cand_cnt; int32_t *cand_idx; double *cand_val; int cap;   // [n_from], [n_from][cap]
};

// sorted insert into one row's top-k list; (kv, ki) tracks the k-th key, ki relative to to_base (-1 while not full)
template <int KMAX>
__device__ __forceinline__ void topk_insert(float (&tv)[KMAX], int (&ti)[KMAX], float &kv, int &ki, int k, float cv, int ci, long long to_base) {
#pragma unroll
    for (int z = 0; z < KMAX; ++z) {
        if (z < k) {
            const bool before = cv > tv[z] || (cv == tv[z] && (ti[z] < 0 || ci < ti[z]));
            if (before) { const float fv = tv[z]; const int fi = ti[z]; tv[z] = cv; ti[z] = ci; cv = fv; ci = fi; }
            if (z == k - 1) { kv = tv[z]; ki = ti[z] < 0 ? -1 : ti[z] - (int)to_base; }
        }
    }
}

// F16: operands are fp16 instead of bf16 (the filter pass of the exact mode); nothing else differs.
// THRESH: the threshold epilogue of top_n > 32 (DESIGN.md 4.7) replaces the register top-k: every (j, score) with
// score >= row_thr[i] and score > min_sim is appended to row i's candidate buffer (capacity cap; cand_cnt[i] keeps counting
// past it).  The four threads of a quad agree on their offsets with shuffles, so a row takes one global atomic per tile.
// The mainloop is the same code, so the scores are the same fp32 bits as the top-k instantiations'.
template <int KMAX, bool MCAST, bool F16, bool THRESH = false>
__global__ void __launch_bounds__(DENSE_THREADS, 1) dense_cos_topk_kernel(const __grid_constant__ CUtensorMap map_x,
                                                                          const __grid_constant__ CUtensorMap map_y, const DenseParams P) {
    constexpr int S = DSTAGES, G = MCAST ? 2 : 1;
    extern __shared__ __align__(1024) unsigned char dsm_raw[];
    // 128-byte-swizzled TMA/wgmma tiles need 1024-byte alignment: align by hand (the launch adds 1 KB of slack).  The
    // offset is the same in every CTA of the launch, which the multicast relies on.
    unsigned char *dsm = dsm_raw + ((1024u - (s32(dsm_raw) & 1023u)) & 1023u);
    unsigned char *sa = dsm;
    unsigned char *sb = dsm + S * A_BYTES;
    const unsigned bar0 = s32(dsm + S * (A_BYTES + B_BYTES));
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (S + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned rank = MCAST ? cluster_ctarank() : 0u;

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), G * DENSE_CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (MCAST) cluster_sync_all();                                       // the peer's barriers exist before anything signals them

    // unit = (group of G adjacent row blocks, split); CTA `rank` of a cluster takes row block G * group + rank
    const int n_groups = (P.n_mblocks + G - 1) / G;
    const int n_units = n_groups * P.n_splits;
    const int tiles_per = (P.n_ntiles + P.n_splits - 1) / P.n_splits;
    const int n_kblk = (P.d + DK - 1) / DK;
    const int u0 = blockIdx.x / G, ustep = gridDim.x / G;

    if (warp == DENSE_CONSUMER_WARPS) {
        if (lane == 0) {
            int stage = 0; unsigned phase = 0;
            for (int u = u0; u < n_units; u += ustep) {
                const int mb = (u % n_groups) * G + (int)rank, sp = u / n_groups;
                const int t_lo = sp * tiles_per, t_hi = min(P.n_ntiles, t_lo + tiles_per);
                for (int t = t_lo; t < t_hi; ++t) {
                    for (int kb = 0; kb < n_kblk; ++kb) {
                        mbar_wait(empty_bar(stage), phase ^ 1);
                        mbar_expect_tx(full_bar(stage), A_BYTES + B_BYTES);
                        tma_load_2d(s32(sa + stage * A_BYTES), &map_x, kb * DK, mb * DM, full_bar(stage));
                        if (MCAST)
                            tma_load_2d_mcast(s32(sb + stage * B_BYTES) + rank * (B_BYTES / 2), &map_y, kb * DK, t * DN + (int)rank * (DN / 2),
                                              full_bar(stage), (unsigned short)0x3);
                        else
                            tma_load_2d(s32(sb + stage * B_BYTES), &map_y, kb * DK, t * DN, full_bar(stage));
                        if (++stage == S) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        __syncwarp();
    } else {
        const int wg = warp >> 2;                                        // consumer warpgroup: rows 64 wg .. 64 wg + 63 of the block
        const int q4 = lane & 3;
        auto release = [&](int s) {
            if (lane == 0) {
                if (MCAST) { mbar_arrive_cta(empty_bar(s), 0); mbar_arrive_cta(empty_bar(s), 1); }
                else mbar_arrive(empty_bar(s));
            }
        };
        int stage = 0; unsigned phase = 0;
        for (int u = u0; u < n_units; u += ustep) {
            const int mb = (u % n_groups) * G + (int)rank, sp = u / n_groups;
            const int t_lo = sp * tiles_per, t_hi = min(P.n_ntiles, t_lo + tiles_per);
            const int row0 = mb * DM + wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: row0 and row0 + 8
            float tv[2][KMAX]; int ti[2][KMAX]; float kv[2]; int ki[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int q = 0; q < KMAX; ++q) { tv[h][q] = P.min_sim; ti[h][q] = -1; }
                kv[h] = P.min_sim; ki[h] = -1;
            }
            float rthr[2];
            if constexpr (THRESH) {
#pragma unroll
                for (int h = 0; h < 2; ++h) rthr[h] = row0 + 8 * h < P.n_from ? P.row_thr[row0 + 8 * h] : INFINITY;
            }
            for (int t = t_lo; t < t_hi; ++t) {
                float acc[DN / 2];
                int prev = -1;
                for (int kb = 0; kb < n_kblk; ++kb) {
                    mbar_wait(full_bar(stage), phase);
                    const uint64_t ad = wgmma_desc(s32(sa + stage * A_BYTES + wg * (64 * DK * 2)));
                    const uint64_t bd = wgmma_desc(s32(sb + stage * B_BYTES));
                    wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < DK / WG_K; ++kk)
                        // advance 16 elements = 32 bytes along K inside the 128-byte swizzled row: +2 in the address field
                        wgmma_m64n128<F16>(acc, ad + (uint64_t)(kk * 2), bd + (uint64_t)(kk * 2), (kb | kk) ? 1 : 0);
                    wgmma_commit();
                    wgmma_wait<1>();                                     // the previous stage's MMAs have retired
                    if (prev >= 0) release(prev);
                    prev = stage;
                    if (++stage == S) { stage = 0; phase ^= 1; }
                }
                wgmma_wait<0>();
                acc_fence(acc);
                release(prev);
                // accumulator layout: acc[4 j + 2 h + e] = (row0 + 8 h, column 8 j + 2 q4 + e of the tile)
                const int colb = t * DN + 2 * q4;
                if constexpr (THRESH) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = row0 + 8 * h;
                        unsigned mask = 0u;
#pragma unroll
                        for (int q = 0; q < 32; ++q) {
                            const int j = q >> 1;
                            const float sc = acc[4 * j + 2 * h + (q & 1)];
                            if (sc >= rthr[h] && sc > P.min_sim && colb + 8 * j + (q & 1) < P.n_to) mask |= 1u << q;
                        }
                        // quad prefix of the counts; lane 0 of the quad reserves the row's slots with one atomic
                        const int cnt = __popc(mask);
                        int incl = cnt;
                        const int u1 = __shfl_up_sync(FULL, incl, 1, 4); if (q4 >= 1) incl += u1;
                        const int u2 = __shfl_up_sync(FULL, incl, 2, 4); if (q4 >= 2) incl += u2;
                        const int tot = __shfl_sync(FULL, incl, 3, 4);
                        int base = 0;
                        if (q4 == 0 && tot > 0) base = atomicAdd(P.cand_cnt + row, tot);
                        int pos = __shfl_sync(FULL, base, 0, 4) + incl - cnt;
                        while (mask) {
                            const int q = __ffs(mask) - 1; mask &= mask - 1;
                            float sc = 0.f;
#pragma unroll
                            for (int z = 0; z < 32; ++z) if (z == q) sc = acc[4 * (z >> 1) + 2 * h + (z & 1)];
                            if (pos < P.cap) {
                                const size_t o = (size_t)row * P.cap + pos;
                                P.cand_idx[o] = (int)(P.to_base + colb + 8 * (q >> 1) + (q & 1));
                                P.cand_val[o] = (double)sc;
                            }
                            ++pos;
                        }
                    }
                }
#pragma unroll
                for (int h = 0; h < (THRESH ? 0 : 2); ++h) {              // the top-k epilogue
                    const long long self_col = P.from_base + row0 + 8 * h - P.to_base;   // local to-column of the diagonal
#pragma unroll
                    for (int c = 0; c < DN / 128; ++c) {
                        // pass 1 (branch-free): which of these 32 scores rank before the k-th key?  (score desc, index asc);
                        // the sentinel (min_sim, -1) makes the test strict while the list is not full
                        unsigned mask = 0u;
#pragma unroll
                        for (int q = 0; q < 32; ++q) {
                            const int j = c * 16 + (q >> 1);
                            const float sc = acc[4 * j + 2 * h + (q & 1)];
                            if (sc > kv[h] || (sc == kv[h] && colb + 8 * j + (q & 1) < ki[h])) mask |= 1u << q;
                        }
                        // pass 2 (rare after the first tiles; the insertion code exists once per chunk, not once per value)
                        while (mask) {
                            const int q = __ffs(mask) - 1; mask &= mask - 1;
                            float sc = 0.f;
#pragma unroll
                            for (int z = 0; z < 32; ++z) if (z == q) sc = acc[4 * (c * 16 + (z >> 1)) + 2 * h + (z & 1)];
                            const int col = colb + 8 * (c * 16 + (q >> 1)) + (q & 1);
                            if (!(sc > kv[h] || (sc == kv[h] && col < ki[h]))) continue;          // the key may have risen meanwhile
                            if (col >= P.n_to || (P.self_match && (long long)col == self_col)) continue;
                            topk_insert<KMAX>(tv[h], ti[h], kv[h], ki[h], P.k, sc, (int)(P.to_base + col), P.to_base);
                        }
                    }
                }
            }
            // the four threads of a quad hold disjoint column sets of the same two rows: k rounds of "best head wins"
#pragma unroll
            for (int h = 0; h < (THRESH ? 0 : 2); ++h) {
                const int row = row0 + 8 * h;
                const size_t o = ((size_t)sp * P.n_from + row) * P.k;
#pragma unroll
                for (int z = 0; z < KMAX; ++z) {
                    if (z < P.k) {
                        float bv = tv[h][0]; int bi = ti[h][0];
#pragma unroll
                        for (int m = 1; m <= 2; m <<= 1) {
                            const float ov = __shfl_xor_sync(FULL, bv, m); const int oi = __shfl_xor_sync(FULL, bi, m);
                            if (oi >= 0 && (bi < 0 || ov > bv || (ov == bv && oi < bi))) { bv = ov; bi = oi; }
                        }
                        if (bi >= 0 && ti[h][0] == bi) {
#pragma unroll
                            for (int w = 0; w + 1 < KMAX; ++w) { tv[h][w] = tv[h][w + 1]; ti[h][w] = ti[h][w + 1]; }
                            tv[h][KMAX - 1] = P.min_sim; ti[h][KMAX - 1] = -1;
                        }
                        if (q4 == 0 && row < P.n_from) { P.top_idx[o + z] = bi; P.top_val[o + z] = bi >= 0 ? (double)bv : 0.0; }
                    }
                }
            }
        }
    }
    if (MCAST) cluster_sync_all();                                       // no CTA exits while its peer may still write into it
}

// rows -> bf16 (fp64 or fp32 in), zero padded to d_pad.  normalize = 0: bf16(float(x)), rounded to nearest even.
// normalize = 1: a faithful bf16 rounding of x / ||x|| for every element of magnitude >= 2^-100, and the same bits for
// x and 2^e x: the row is first scaled by 2^-E, E = ilogb(max |x|), which is exact, so the fp32 sum of squares lies in
// [1, 4 d] and neither overflows nor leaves the normal range at any input scale.  Zero rows stay zero.  One warp per row.
template <typename T>
__global__ void __launch_bounds__(256) rows_normalize_bf16_kernel(const T *__restrict__ x, int64_t ld, int n_rows, int d, int d_pad, int normalize,
                                                                  __nv_bfloat16 *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int r = gw; r < n_rows; r += nw) {
        const T *row = x + (int64_t)r * ld;
        __nv_bfloat16 *o = out + (int64_t)r * d_pad;
        if (!normalize) {
            for (int c = lane; c < d_pad; c += 32) o[c] = __float2bfloat16(c < d ? (float)row[c] : 0.f);
            continue;
        }
        double mx = 0.0;
        for (int c = lane; c < d; c += 32) mx = fmax(mx, fabs((double)row[c]));
#pragma unroll
        for (int s = 16; s; s >>= 1) mx = fmax(mx, __shfl_xor_sync(FULL, mx, s));
        const int e = mx > 0.0 ? -ilogb(mx) : 0;
        float ss = 0.f;
        for (int c = lane; c < d; c += 32) { const float v = (float)ldexp((double)row[c], e); ss += v * v; }
#pragma unroll
        for (int s = 16; s; s >>= 1) ss += __shfl_xor_sync(FULL, ss, s);
        const float inv = ss > 0.f ? rsqrtf(ss) : 1.f;
        for (int c = lane; c < d_pad; c += 32) o[c] = __float2bfloat16(c < d ? (float)ldexp((double)row[c], e) * inv : 0.f);
    }
}

// ---- exact mode: canonical fp64 scores, certified against an fp16 tensor-core filter pass (DESIGN.md 4.6) ----------------
//
// canonical dot(a, b): lane l sums a[32 t + l] * b[32 t + l] over ascending t (product rounded, then added; no FMA; from +0),
// then p[l] += p[l ^ o] for o = 16, 8, 4, 2, 1.  Every lane ends with the same value.  Zero padding up to d_pad adds +0 and
// changes nothing.

__device__ __forceinline__ double warp_sum_rn(double p) {
#pragma unroll
    for (int o = 16; o; o >>= 1) p = __dadd_rn(p, __shfl_xor_sync(FULL, p, o));
    return p;
}
__device__ __forceinline__ double warp_sum_ru(double p) {
#pragma unroll
    for (int o = 16; o; o >>= 1) p = __dadd_ru(p, __shfl_xor_sync(FULL, p, o));
    return p;
}

// NC canonical dots of one row a against rows b[0..NC-1], interleaved for memory-level parallelism
template <int NC>
__device__ __forceinline__ void warp_dot_canon(const double *__restrict__ a, const double *const (&b)[NC], int d_pad, int lane, double (&out)[NC]) {
    double p[NC];
#pragma unroll
    for (int u = 0; u < NC; ++u) p[u] = 0.0;
    for (int c = lane; c < d_pad; c += 32) {
        const double av = a[c];
#pragma unroll
        for (int u = 0; u < NC; ++u) p[u] = __dadd_rn(p[u], __dmul_rn(av, b[u][c]));
    }
#pragma unroll
    for (int u = 0; u < NC; ++u) out[u] = warp_sum_rn(p[u]);
}

// rows -> canonical l2-normalised fp64 rows x~ and their fp16 rounding x^ ([n_rows][d_pad], zero padded), with upper bounds
// of ||x^|| and ||x~ - x^|| per row and (maxima, may be NULL) of both over all rows.  One warp per row.
template <typename T>
__global__ void __launch_bounds__(256) rows_prep_exact_kernel(const T *__restrict__ x, int64_t ld, int n_rows, int d, int d_pad,
                                                              double *__restrict__ out64, __half *__restrict__ out16, double *__restrict__ norm16,
                                                              double *__restrict__ err16, unsigned long long *__restrict__ maxima) {
    const int lane = threadIdx.x & 31;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int r = gw; r < n_rows; r += nw) {
        const T *row = x + (int64_t)r * ld;
        double p = 0.0;
        for (int c = lane; c < d; c += 32) { const double v = (double)row[c]; p = __dadd_rn(p, __dmul_rn(v, v)); }
        p = warp_sum_rn(p);
        const double nrm = __dsqrt_rn(p);
        double sn = 0.0, se = 0.0;
        for (int c = lane; c < d_pad; c += 32) {
            double v = c < d ? (double)row[c] : 0.0;
            if (p > 0.0) v = __ddiv_rn(v, nrm);                        // a zero row stays as it is
            const __half h = __double2half(v);
            const double hv = (double)__half2float(h);
            const double e = __dsub_rn(v, hv);                         // exact: |e| <= half an fp16 ulp of v
            out64[(int64_t)r * d_pad + c] = v;
            out16[(int64_t)r * d_pad + c] = h;
            sn = __dadd_ru(sn, __dmul_ru(hv, hv));
            se = __dadd_ru(se, __dmul_ru(e, e));
        }
        const double nx = __dsqrt_ru(warp_sum_ru(sn)), ex = __dsqrt_ru(warp_sum_ru(se));
        if (lane == 0) {
            norm16[r] = nx; err16[r] = ex;
            if (maxima) {                                              // non-negative doubles order as their bit patterns
                atomicMax(&maxima[0], (unsigned long long)__double_as_longlong(nx));
                atomicMax(&maxima[1], (unsigned long long)__double_as_longlong(ex));
            }
        }
    }
}

// A-priori bound M_max >= every row's M_i (see exact_rescore_kernel) for rows of width d_pad: |x~| <= r, each fp16 rounding
// error <= 2^-11 |x~_c| (normal range) + 2^-25 (subnormal range), fp32 accumulation error <= gamma * ||x^|| ||y^||.
static double exact_gamma(int d_pad) { return d_pad * 0x1p-22; }
static double exact_margin_max(int d_pad) {
    const double r = 1.0 + d_pad * 0x1p-50;
    const double e = 0x1p-11 * r + 0x1p-25 * sqrt((double)d_pad);
    const double n = r + e;
    const double m = 2.0 * e * n + e * e + exact_gamma(d_pad) * n * n + 2.0 * d_pad * 0x1p-53 * (n + e) * (n + e);
    return m * (1.0 + 0x1p-20);
}

struct ExactParams {
    const double *x, *y; int n_from, n_to, d_pad, k, kc; double thr, gamma, m_max; int self_match; long long from_base, to_base;
    const int32_t *cand_idx; const double *cand_val; const double *x_norm, *x_err; const double *y_max;
    int32_t *top_idx; double *top_val; int32_t *fb_rows; int32_t *fb_count;
};

// M_i of from-row i (below): an upper bound on |fp32 filter score - canonical score| for every to-row
__device__ __forceinline__ double exact_row_margin(double nx, double ex, double Ny, double Ey, double gamma, int d_pad) {
    double m = __dmul_ru(ex, Ny);
    m = __dadd_ru(m, __dmul_ru(nx, Ey));
    m = __dadd_ru(m, __dmul_ru(ex, Ey));
    m = __dadd_ru(m, __dmul_ru(__dmul_ru(gamma, nx), Ny));
    m = __dadd_ru(m, __dmul_ru(__dmul_ru(2.0 * d_pad * 0x1p-53, __dadd_ru(nx, ex)), __dadd_ru(Ny, Ey)));
    return m;
}

// One warp per from-row: canonical scores of the row's <= kc filter candidates (lane c holds candidate c), the exact top-k of
// the eligible ones, and the certificate that no other to-row belongs in it.  With s_kc the kc-th filter score and
//   M_i = e_x N_y + n_x E_y + e_x E_y + gamma n_x N_y + 2 d_pad 2^-53 (n_x + e_x)(N_y + E_y)   (rounded up)
// every non-candidate's canonical score is <= B = s_kc + M_i.  Certified iff: the filter returned fewer than kc candidates
// (then every non-candidate scored <= t_f <= thr - M_max in fp32, and M_i <= M_max), or B <= thr, or the exact k-th score > B.
// Other rows are appended to fb_rows.
__global__ void __launch_bounds__(256) exact_rescore_kernel(const ExactParams P) {
    const int lane = threadIdx.x & 31;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    const double Ny = P.y_max[0], Ey = P.y_max[1];
    constexpr int NC = 4;
    for (int i = gw; i < P.n_from; i += nw) {
        const double *xr = P.x + (int64_t)i * P.d_pad;
        const int my_j = lane < P.kc ? P.cand_idx[(int64_t)i * P.kc + lane] : -1;       // global to-index; the valid ones are a prefix
        const int nc = __popc(__ballot_sync(FULL, my_j >= 0));
        double my_s = 0.0;
        for (int c0 = 0; c0 < nc; c0 += NC) {
            const double *yr[NC]; double s[NC];
#pragma unroll
            for (int u = 0; u < NC; ++u) {
                const int j = __shfl_sync(FULL, my_j, min(c0 + u, nc - 1));
                yr[u] = P.y + ((int64_t)j - P.to_base) * P.d_pad;
            }
            warp_dot_canon<NC>(xr, yr, P.d_pad, lane, s);
#pragma unroll
            for (int u = 0; u < NC; ++u) if (lane == c0 + u) my_s = s[u];
        }
        const long long self_j = P.from_base + i;
        const bool elig = my_j >= 0 && my_s > P.thr && !(P.self_match && (long long)my_j == self_j);
        const unsigned emask = __ballot_sync(FULL, elig);
        const int n_el = __popc(emask);
        int rank = 0;
#pragma unroll 4
        for (int z = 0; z < 32; ++z) {
            const double os = __shfl_sync(FULL, my_s, z); const int oj = __shfl_sync(FULL, my_j, z);
            if (((emask >> z) & 1u) && (os > my_s || (os == my_s && oj < my_j))) ++rank;
        }
        const int64_t o = (int64_t)i * P.k;
        if (elig && rank < P.k) { P.top_idx[o + rank] = my_j; P.top_val[o + rank] = my_s; }
        for (int z = n_el + lane; z < P.k; z += 32) { P.top_idx[o + z] = -1; P.top_val[o + z] = 0.0; }
        const double m = exact_row_margin(P.x_norm[i], P.x_err[i], Ny, Ey, P.gamma, P.d_pad);
        bool cert;
        if (nc < P.kc) cert = m <= P.m_max;
        else {
            const double B = __dadd_ru(P.cand_val[(int64_t)i * P.kc + P.kc - 1], m);
            cert = B <= P.thr;
            if (!cert && n_el >= P.k) {
                const unsigned km = __ballot_sync(FULL, elig && rank == P.k - 1);
                cert = __shfl_sync(FULL, my_s, __ffs(km) - 1) > B;    // strict: a to-row scoring exactly B could tie and win on index
            }
        }
        if (!cert && lane == 0) P.fb_rows[atomicAdd(P.fb_count, 1)] = i;
    }
}

// lane-distributed sorted list of a warp: lane z holds slot z < k, key (score desc, index asc), empty slots (-1) at the end
__device__ __forceinline__ void lane_list_insert(double &lv, int &li, double s, int j, int k, int lane) {
    const bool before = lane < k && li >= 0 && (lv > s || (lv == s && li < j));
    const int pos = __popc(__ballot_sync(FULL, before));
    if (pos >= k) return;
    const double uv = __shfl_up_sync(FULL, lv, 1); const int ui = __shfl_up_sync(FULL, li, 1);
    if (lane > pos) { lv = uv; li = ui; }
    else if (lane == pos) { lv = s; li = j; }
}
__device__ __forceinline__ bool lane_list_takes(double kv, int ki, double s, int j) { return ki < 0 || s > kv || (s == kv && j < ki); }

constexpr int FB_WARPS = 8, FB_CAP_ROWS = 2048, FB_MAX_SPLITS = 64, FB_ROWS_PER_SPLIT = 512;
static int fb_splits(int n_to) { return max(1, min(FB_MAX_SPLITS, (n_to + FB_ROWS_PER_SPLIT - 1) / FB_ROWS_PER_SPLIT)); }

struct FallbackParams {
    const double *x, *y; int n_to, d_pad, k; double thr; int self_match; long long from_base, to_base;
    const int32_t *fb_rows; const int32_t *fb_count; int n_splits, cap;
    double *ws_val; int32_t *ws_idx; int32_t *ws_done; int32_t *top_idx; double *top_val;
};

// Brute-force canonical top-k over every to-row for the rows listed by exact_rescore_kernel (count read on the device).
// Work item = (listed row, to-range split): the first `cap` listed rows are split n_splits ways, the CTA that finishes a
// row's last split merges the partial lists; rows beyond `cap` are one item each over the whole to-range.
__global__ void __launch_bounds__(FB_WARPS * 32) exact_fallback_kernel(const FallbackParams P) {
    __shared__ double s_v[FB_WARPS][32];
    __shared__ int s_i[FB_WARPS][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cnt = *P.fb_count;
    const int n_split_rows = min(cnt, P.cap);
    const long long n_split_items = (long long)n_split_rows * P.n_splits;
    const long long n_items = n_split_items + (cnt - n_split_rows);
    const int chunk = (P.n_to + P.n_splits - 1) / P.n_splits;
    for (long long u = blockIdx.x; u < n_items; u += gridDim.x) {
        int p, sp, lo, hi;
        if (u < n_split_items) { p = (int)(u / P.n_splits); sp = (int)(u % P.n_splits); lo = sp * chunk; hi = min(P.n_to, lo + chunk); }
        else { p = P.cap + (int)(u - n_split_items); sp = -1; lo = 0; hi = P.n_to; }
        const int i = P.fb_rows[p];
        const double *xr = P.x + (int64_t)i * P.d_pad;
        const long long self_j = P.from_base + i - P.to_base;
        double lv = 0.0, kv = 0.0; int li = -1, ki = -1;
        for (int j = lo + warp; j < hi; j += FB_WARPS) {
            const double *yr[1] = {P.y + (int64_t)j * P.d_pad}; double s[1];
            warp_dot_canon<1>(xr, yr, P.d_pad, lane, s);
            if (!(s[0] > P.thr) || (P.self_match && (long long)j == self_j)) continue;
            const int gj = (int)(P.to_base + j);
            if (!lane_list_takes(kv, ki, s[0], gj)) continue;
            lane_list_insert(lv, li, s[0], gj, P.k, lane);
            kv = __shfl_sync(FULL, lv, P.k - 1); ki = __shfl_sync(FULL, li, P.k - 1);
        }
        s_v[warp][lane] = lv; s_i[warp][lane] = li;
        __syncthreads();
        if (warp == 0) {
            for (int w = 1; w < FB_WARPS; ++w)
                for (int z = 0; z < P.k; ++z) {
                    const int oj = s_i[w][z]; const double ov = s_v[w][z];
                    if (oj < 0 || !lane_list_takes(kv, ki, ov, oj)) break;      // sorted: the rest of this list loses too
                    lane_list_insert(lv, li, ov, oj, P.k, lane);
                    kv = __shfl_sync(FULL, lv, P.k - 1); ki = __shfl_sync(FULL, li, P.k - 1);
                }
            bool write = sp < 0;
            if (!write) {
                const int64_t o = ((int64_t)p * P.n_splits + sp) * P.k;
                if (lane < P.k) { P.ws_val[o + lane] = lv; P.ws_idx[o + lane] = li; }
                __threadfence();
                int last = 0;
                if (lane == 0) last = atomicAdd(&P.ws_done[p], 1) == P.n_splits - 1;
                write = __shfl_sync(FULL, last, 0) != 0;
                if (write) {                                                   // every split of row p is in ws: merge them
                    __threadfence();
                    li = -1; ki = -1;
                    for (int q = 0; q < P.n_splits; ++q)
                        for (int z = 0; z < P.k; ++z) {
                            const int64_t oq = ((int64_t)p * P.n_splits + q) * P.k + z;
                            const int oj = __ldcg(P.ws_idx + oq); const double ov = __ldcg(P.ws_val + oq);
                            if (oj < 0 || !lane_list_takes(kv, ki, ov, oj)) break;
                            lane_list_insert(lv, li, ov, oj, P.k, lane);
                            kv = __shfl_sync(FULL, lv, P.k - 1); ki = __shfl_sync(FULL, li, P.k - 1);
                        }
                }
            }
            if (write && lane < P.k) {
                P.top_idx[(int64_t)i * P.k + lane] = li;
                P.top_val[(int64_t)i * P.k + lane] = li >= 0 ? lv : 0.0;
            }
        }
        __syncthreads();
    }
}

// ---- top_n > 32 (DESIGN.md 4.7): bound from unmerged KMAX = 16 lists, threshold pass, select --------------------------------

constexpr int SEL_THREADS = 256, SEL_PER = 8, SEL_TILE = SEL_THREADS * SEL_PER;

struct SelectParams {
    const int32_t *idx; const double *val; const int32_t *count;         // count NULL: every row has n_cand entries
    int n_rows, n_cand; long long row_stride, seg_stride; int seg_len;  // entry e of row r: r row_stride + (e / seg_len) seg_stride + e % seg_len
    const int32_t *row_map;                                             // output row of row r (NULL: r)
    int k; double thr; int self_match; long long from_base;             // eligible: index >= 0, score > thr, not the diagonal
    int32_t *top_idx; double *top_val;                                  // list mode: [output rows][k]
    float *row_thr;                                                     // bound mode (non-NULL): per output row, instead of a list
    int exact; double thr_bound; const double *x_norm, *x_err, *y_max; double gamma; int d_pad;
};

// One CTA per row: the rank of every eligible entry under (score desc, index asc) by counting the entries that rank before it;
// entries are unique by index, so the ranks 0 .. n_el - 1 are distinct.  A batch of SEL_TILE entries sits in registers (SEL_PER
// per thread) while the row streams through shared memory in tiles of SEL_TILE, so any count works; an entry stops counting
// once its rank reaches k.  List mode writes the top k (empty slots (-1, 0.0)); bound mode writes the row threshold of the
// threshold pass from the k-th entry (-inf when fewer than k entries are eligible, i.e. no bound: every score passes).
__global__ void __launch_bounds__(SEL_THREADS) topn_select_kernel(const SelectParams P) {
    __shared__ double s_v[SEL_TILE];
    __shared__ int s_i[SEL_TILE];
    __shared__ int s_nel;
    const int tid = threadIdx.x;
    for (int r = blockIdx.x; r < P.n_rows; r += gridDim.x) {
        const int orow = P.row_map ? P.row_map[r] : r;
        const int n = P.count ? min(P.count[r], P.n_cand) : P.n_cand;
        const long long self_j = P.from_base + orow;
        auto load = [&](int e, double &v, int &j) {
            const long long o = (long long)r * P.row_stride + (long long)(e / P.seg_len) * P.seg_stride + e % P.seg_len;
            j = P.idx[o]; v = P.val[o];
            if (j < 0 || !(v > P.thr) || (P.self_match && (long long)j == self_j)) j = -1;
        };
        if (tid == 0) { s_nel = 0; if (P.row_thr) P.row_thr[orow] = -INFINITY; }
        __syncthreads();
        for (int b0 = 0; b0 < n; b0 += SEL_TILE) {
            double ov[SEL_PER]; int oj[SEL_PER], rk[SEL_PER];
            int mine = 0;
#pragma unroll
            for (int q = 0; q < SEL_PER; ++q) {
                const int e = b0 + q * SEL_THREADS + tid;
                ov[q] = 0.0; oj[q] = -1; rk[q] = 0;
                if (e < n) load(e, ov[q], oj[q]);
                mine += oj[q] >= 0;
            }
            if (mine) atomicAdd(&s_nel, mine);
            for (int t0 = 0; t0 < n; t0 += SEL_TILE) {
                const int tn = min(SEL_TILE, n - t0);
                __syncthreads();
                for (int z = tid; z < tn; z += SEL_THREADS) { double v; int j; load(t0 + z, v, j); s_v[z] = v; s_i[z] = j; }
                __syncthreads();
#pragma unroll
                for (int q = 0; q < SEL_PER; ++q) {
                    if (oj[q] < 0) continue;
                    int c = rk[q];
                    for (int z = 0; z < tn && c < P.k; ++z) {
                        const int oz = s_i[z]; const double vz = s_v[z];
                        c += oz >= 0 && (vz > ov[q] || (vz == ov[q] && oz < oj[q]));
                    }
                    rk[q] = c;
                }
            }
#pragma unroll
            for (int q = 0; q < SEL_PER; ++q) {
                if (oj[q] < 0 || rk[q] >= P.k) continue;
                if (!P.row_thr) {
                    const int64_t o = (int64_t)orow * P.k + rk[q];
                    P.top_idx[o] = oj[q]; P.top_val[o] = ov[q];
                } else if (rk[q] == P.k - 1) {
                    float rt;
                    if (!P.exact) rt = (float)ov[q];                       // an fp32 score: the threshold is the k-th score itself
                    else {                                                 // tau = f_k - M_i; emit f >= tau - M_i when tau > thr
                        const double m = exact_row_margin(P.x_norm[orow], P.x_err[orow], P.y_max[0], P.y_max[1], P.gamma, P.d_pad);
                        const double tau = __dsub_rd(ov[q], m);
                        rt = tau > P.thr_bound ? __double2float_rd(__dsub_rd(tau, m)) : -INFINITY;
                    }
                    P.row_thr[orow] = rt;
                }
            }
        }
        __syncthreads();
        if (!P.row_thr)
            for (int z = s_nel + tid; z < P.k; z += SEL_THREADS) { P.top_idx[(int64_t)orow * P.k + z] = -1; P.top_val[(int64_t)orow * P.k + z] = 0.0; }
        __syncthreads();
    }
}

struct CandRescoreParams {
    const double *x, *y; int n_rows, d_pad, cap; long long to_base;
    const int32_t *row_map; const int32_t *cand_idx; double *cand_val; const int32_t *count;
};

// exact mode: every candidate's filter score is replaced by its canonical fp64 score.  One warp per (row, 32 candidates).
__global__ void __launch_bounds__(256) topn_exact_rescore_kernel(const CandRescoreParams P) {
    constexpr int NC = 4;
    const int lane = threadIdx.x & 31;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((long long)gridDim.x * blockDim.x) >> 5;
    const int slabs = (P.cap + 31) / 32;
    const long long items = (long long)P.n_rows * slabs;
    for (long long it = gw; it < items; it += nw) {
        const int r = (int)(it / slabs), c0s = (int)(it % slabs) * 32;
        const int n = min(P.count[r], P.cap);
        if (c0s >= n) continue;
        const int nc = min(32, n - c0s);
        const double *xr = P.x + (int64_t)(P.row_map ? P.row_map[r] : r) * P.d_pad;
        const size_t o = (size_t)r * P.cap + c0s;
        const int my_j = lane < nc ? P.cand_idx[o + lane] : -1;
        double my_s = 0.0;
        for (int c0 = 0; c0 < nc; c0 += NC) {
            const double *yr[NC]; double s[NC];
#pragma unroll
            for (int u = 0; u < NC; ++u) {
                const int j = __shfl_sync(FULL, my_j, min(c0 + u, nc - 1));
                yr[u] = P.y + ((int64_t)j - P.to_base) * P.d_pad;
            }
            warp_dot_canon<NC>(xr, yr, P.d_pad, lane, s);
#pragma unroll
            for (int u = 0; u < NC; ++u) if (lane == c0 + u) my_s = s[u];
        }
        if (lane < nc) P.cand_val[o + lane] = my_s;
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static int make_map(EncodeTiledFn enc, CUtensorMap *m, const void *base, int n_rows, int d, int box_rows, CUtensorMapDataType dt) {
    cuuint64_t dims[2] = {(cuuint64_t)d, (cuuint64_t)n_rows};
    cuuint64_t strides[1] = {(cuuint64_t)d * 2};
    cuuint32_t box[2] = {(cuuint32_t)DK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, dt, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return 1; }
    return 0;
}

template <int KMAX, bool MCAST, bool F16, bool THRESH = false>
static int dense_launch(EncodeTiledFn enc, const void *x_op, const void *y_op, DenseParams P, int sms, cudaStream_t st) {
    const CUtensorMapDataType dt = F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    CUtensorMap mx, my;
    if (make_map(enc, &mx, x_op, P.n_from, P.d, DM, dt)) return 1;
    if (make_map(enc, &my, y_op, P.n_to, P.d, MCAST ? DN / 2 : DN, dt)) return 1;
    const int G = MCAST ? 2 : 1;
    int units = (P.n_mblocks + G - 1) / G * P.n_splits; if (units > sms / G) units = sms / G;
    auto kern = dense_cos_topk_kernel<KMAX, MCAST, F16, THRESH>;
    PFZ_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DENSE_SMEM));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(G * units)); cfg.blockDim = dim3(DENSE_THREADS); cfg.dynamicSmemBytes = DENSE_SMEM; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = G; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    PFZ_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, mx, my, P));
    PFZ_LAUNCH_OK();
    return 0;
}

// shared by every K4 entry point: validation, tensor-map encoder, launch shape.  Sets *run = false when there is nothing to do.
static int dense_prepare(const char *fn, const void *x_op, const void *y_op, int32_t n_from, int32_t n_to, int32_t d, int32_t n_splits,
                         DenseParams &P, EncodeTiledFn &enc_out, bool &two_cta, int &sms, bool &run) {
    run = false;
    PFZ_REQUIRE(d >= 8 && d % 8 == 0, "%s: d=%d must be a multiple of 8 (16-byte row pitch for TMA)", fn, d);
    PFZ_REQUIRE(((uintptr_t)x_op % 16) == 0 && ((uintptr_t)y_op % 16) == 0, "%s: operands must be 16-byte aligned", fn);
    if (n_from <= 0) return 0;
    PFZ_REQUIRE(n_to > 0, "%s: empty to-matrix", fn);
    static EncodeTiledFn enc = nullptr;
    if (!enc) {
        void *f = nullptr; cudaDriverEntryPointQueryResult qres;
        PFZ_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres));
        PFZ_REQUIRE(f && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available in this driver");
        enc = (EncodeTiledFn)f;
    }
    enc_out = enc;
    const char *env2 = getenv("PFZ_K4_2CTA");                   // CTA pairs sharing the to-tile through TMA multicast (half the to-operand
    two_cta = env2 ? atoi(env2) != 0 : true;                    // traffic per SM); 0 = one CTA per row block
    P = DenseParams{};
    P.n_from = n_from; P.n_to = n_to; P.d = d;
    P.n_mblocks = (n_from + DM - 1) / DM; P.n_ntiles = (n_to + DN - 1) / DN;
    PFZ_REQUIRE(n_splits >= 1 && n_splits <= P.n_ntiles, "%s: n_splits %d out of range (1..%d)", fn, n_splits, P.n_ntiles);
    P.n_splits = n_splits;
    int dev = 0;
    PFZ_CUDA_OK(cudaGetDevice(&dev));
    PFZ_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    run = true;
    return 0;
}

// the bf16 and fp16 top-k entry points: KMAX dispatch; the candidate threshold is min_sim
template <bool F16>
static int dense_topk_any(const char *fn, const void *x_op, const void *y_op, int32_t n_from, int32_t n_to, int32_t d, int32_t k, float min_sim,
                          int32_t self_match, int64_t from_index_base, int64_t to_index_base, int32_t n_splits, int32_t *top_idx, double *top_val,
                          void *stream) {
    PFZ_REQUIRE(k >= 1 && k <= 32, "%s: k=%d unsupported (1..32)", fn, k);
    DenseParams P; EncodeTiledFn enc = nullptr; bool two_cta = true, run = false; int sms = 0;
    if (dense_prepare(fn, x_op, y_op, n_from, n_to, d, n_splits, P, enc, two_cta, sms, run)) return 1;
    if (!run) return 0;
    P.k = k; P.min_sim = min_sim; P.self_match = self_match; P.from_base = from_index_base; P.to_base = to_index_base;
    P.top_idx = top_idx; P.top_val = top_val;
    cudaStream_t st = as_stream(stream);
#define PFZ_DENSE_LAUNCH(KM) (two_cta ? dense_launch<KM, true, F16>(enc, x_op, y_op, P, sms, st) : dense_launch<KM, false, F16>(enc, x_op, y_op, P, sms, st))
    if (k <= 4) return PFZ_DENSE_LAUNCH(4);
    if (k <= 10) return PFZ_DENSE_LAUNCH(10);
    if (k <= 16) return PFZ_DENSE_LAUNCH(16);
    return PFZ_DENSE_LAUNCH(32);
#undef PFZ_DENSE_LAUNCH
}

// the bf16 and fp16 threshold-pass entry points (top_n > 32): appends to per-row candidate buffers, counters zeroed here
template <bool F16>
static int dense_cand_any(const char *fn, const void *x_op, const void *y_op, int32_t n_from, int32_t n_to, int32_t d, float min_sim,
                          const float *row_thr, int64_t to_index_base, int32_t n_splits, int32_t cap, int32_t *cand_idx, double *cand_val,
                          int32_t *cand_count, void *stream) {
    PFZ_REQUIRE(cap >= 1, "%s: cap=%d must be >= 1", fn, cap);
    DenseParams P; EncodeTiledFn enc = nullptr; bool two_cta = true, run = false; int sms = 0;
    if (dense_prepare(fn, x_op, y_op, n_from, n_to, d, n_splits, P, enc, two_cta, sms, run)) return 1;
    if (!run) return 0;
    cudaStream_t st = as_stream(stream);
    PFZ_CUDA_OK(cudaMemsetAsync(cand_count, 0, (size_t)n_from * sizeof(int32_t), st));
    P.k = 1; P.min_sim = min_sim; P.self_match = 0; P.from_base = 0; P.to_base = to_index_base;
    P.row_thr = row_thr; P.cand_cnt = cand_count; P.cand_idx = cand_idx; P.cand_val = cand_val; P.cap = cap;
    return two_cta ? dense_launch<1, true, F16, true>(enc, x_op, y_op, P, sms, st) : dense_launch<1, false, F16, true>(enc, x_op, y_op, P, sms, st);
}

// t_f of the fp16 filter: the largest float <= min_similarity - M_max(d)
static float filter_threshold(double min_similarity, int d) {
    const double t = nextafter(min_similarity - exact_margin_max(d), -INFINITY);
    float tf = (float)t;
    if ((double)tf > t) tf = nextafterf(tf, -INFINITY);
    return tf;
}

}  // namespace pfz

using namespace pfz;

extern "C" {

int pfz_rows_to_bf16(const void *x, int32_t is_f64, int64_t ld, int32_t n_rows, int32_t d, int32_t d_pad, int32_t normalize, void *out_bf16,
                     void *stream) {
    if (n_rows <= 0) return 0;
    PFZ_REQUIRE(d_pad >= d && d_pad % 8 == 0, "pfz_rows_to_bf16: d_pad %d must be >= d and a multiple of 8", d_pad);
    int grid = (n_rows + 7) / 8; if (grid > SM_COUNT * 16) grid = SM_COUNT * 16;
    if (is_f64) rows_normalize_bf16_kernel<double><<<grid, 256, 0, as_stream(stream)>>>((const double *)x, ld, n_rows, d, d_pad, normalize, (__nv_bfloat16 *)out_bf16);
    else        rows_normalize_bf16_kernel<float><<<grid, 256, 0, as_stream(stream)>>>((const float *)x, ld, n_rows, d, d_pad, normalize, (__nv_bfloat16 *)out_bf16);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_dense_cos_topk(const void *x_bf16, const void *y_bf16, int32_t n_from, int32_t n_to, int32_t d, int32_t k, double min_similarity,
                       int32_t self_match, int64_t from_index_base, int64_t to_index_base, int32_t n_splits, int32_t *top_idx, double *top_val,
                       void *stream) {
    return dense_topk_any<false>("pfz_dense_cos_topk", x_bf16, y_bf16, n_from, n_to, d, k, (float)min_similarity, self_match, from_index_base,
                                 to_index_base, n_splits, top_idx, top_val, stream);
}

int pfz_rows_prep_exact(const void *x, int32_t is_f64, int64_t ld, int32_t n_rows, int32_t d, int32_t d_pad, double *out_f64, void *out_f16,
                        double *norm16, double *err16, double *maxima, void *stream) {
    PFZ_REQUIRE(d_pad >= d && d_pad % 8 == 0, "pfz_rows_prep_exact: d_pad %d must be >= d and a multiple of 8", d_pad);
    cudaStream_t st = as_stream(stream);
    if (maxima) PFZ_CUDA_OK(cudaMemsetAsync(maxima, 0, 2 * sizeof(double), st));
    if (n_rows <= 0) return 0;
    int grid = (n_rows + 7) / 8; if (grid > SM_COUNT * 16) grid = SM_COUNT * 16;
    unsigned long long *mx = (unsigned long long *)maxima;
    if (is_f64) rows_prep_exact_kernel<double><<<grid, 256, 0, st>>>((const double *)x, ld, n_rows, d, d_pad, out_f64, (__half *)out_f16, norm16, err16, mx);
    else        rows_prep_exact_kernel<float><<<grid, 256, 0, st>>>((const float *)x, ld, n_rows, d, d_pad, out_f64, (__half *)out_f16, norm16, err16, mx);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_dense_cos_topk_f16(const void *x_f16, const void *y_f16, int32_t n_from, int32_t n_to, int32_t d, int32_t k, double min_similarity,
                           int32_t self_match, int64_t from_index_base, int64_t to_index_base, int32_t n_splits, int32_t *top_idx, double *top_val,
                           void *stream) {
    return dense_topk_any<true>("pfz_dense_cos_topk_f16", x_f16, y_f16, n_from, n_to, d, k, filter_threshold(min_similarity, d), self_match,
                                from_index_base, to_index_base, n_splits, top_idx, top_val, stream);
}

int pfz_dense_cos_cand(const void *x_bf16, const void *y_bf16, int32_t n_from, int32_t n_to, int32_t d, double min_similarity,
                       const float *row_thr, int64_t to_index_base, int32_t n_splits, int32_t cap, int32_t *cand_idx, double *cand_val,
                       int32_t *cand_count, void *stream) {
    return dense_cand_any<false>("pfz_dense_cos_cand", x_bf16, y_bf16, n_from, n_to, d, (float)min_similarity, row_thr, to_index_base, n_splits,
                                 cap, cand_idx, cand_val, cand_count, stream);
}

int pfz_dense_cos_cand_f16(const void *x_f16, const void *y_f16, int32_t n_from, int32_t n_to, int32_t d, double min_similarity,
                           const float *row_thr, int64_t to_index_base, int32_t n_splits, int32_t cap, int32_t *cand_idx, double *cand_val,
                           int32_t *cand_count, void *stream) {
    return dense_cand_any<true>("pfz_dense_cos_cand_f16", x_f16, y_f16, n_from, n_to, d, filter_threshold(min_similarity, d), row_thr,
                                to_index_base, n_splits, cap, cand_idx, cand_val, cand_count, stream);
}

static int topn_select_launch(const SelectParams &P, cudaStream_t st) {
    if (P.n_rows <= 0) return 0;
    const int grid = P.n_rows < SM_COUNT * 8 ? P.n_rows : SM_COUNT * 8;
    topn_select_kernel<<<grid, SEL_THREADS, 0, st>>>(P);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_dense_topn_bound(const int32_t *list_idx, const double *list_val, int32_t n_lists, int32_t n_from, int32_t k_list, int32_t k,
                         int32_t exact, const double *x_norm16, const double *x_err16, const double *y_maxima, int32_t d_pad,
                         double min_similarity, float *row_thr, void *stream) {
    PFZ_REQUIRE(n_lists >= 1 && k_list >= 1 && k >= 1, "pfz_dense_topn_bound: need n_lists, k_list, k >= 1");
    SelectParams P = {};
    P.idx = list_idx; P.val = list_val; P.count = nullptr; P.n_rows = n_from; P.n_cand = n_lists * k_list;
    P.row_stride = k_list; P.seg_len = k_list; P.seg_stride = (long long)n_from * k_list;
    P.k = k; P.thr = -INFINITY; P.self_match = 0; P.row_thr = row_thr;
    P.exact = exact; P.thr_bound = min_similarity; P.x_norm = x_norm16; P.x_err = x_err16; P.y_max = y_maxima;
    P.gamma = exact_gamma(d_pad); P.d_pad = d_pad;
    return topn_select_launch(P, as_stream(stream));
}

int pfz_dense_topn_exact_rescore(const double *x_f64, const double *y_f64, int32_t n_rows, int32_t d_pad, const int32_t *row_map,
                                 int64_t to_index_base, int32_t cap, const int32_t *cand_idx, double *cand_val, const int32_t *cand_count,
                                 void *stream) {
    PFZ_REQUIRE(d_pad >= 8 && d_pad % 8 == 0 && cap >= 1, "pfz_dense_topn_exact_rescore: d_pad=%d, cap=%d", d_pad, cap);
    if (n_rows <= 0) return 0;
    CandRescoreParams P;
    P.x = x_f64; P.y = y_f64; P.n_rows = n_rows; P.d_pad = d_pad; P.cap = cap; P.to_base = to_index_base;
    P.row_map = row_map; P.cand_idx = cand_idx; P.cand_val = cand_val; P.count = cand_count;
    const long long warps = (long long)n_rows * ((cap + 31) / 32);
    const int grid = (int)(warps < (long long)SM_COUNT * 16 * 8 ? (warps + 7) / 8 : SM_COUNT * 16);
    topn_exact_rescore_kernel<<<grid, 256, 0, as_stream(stream)>>>(P);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_dense_topn_select(const int32_t *cand_idx, const double *cand_val, const int32_t *cand_count, int32_t n_rows, int32_t cap, int32_t k,
                          double min_similarity, int32_t self_match, int64_t from_index_base, const int32_t *row_map, int32_t *top_idx,
                          double *top_val, void *stream) {
    PFZ_REQUIRE(k >= 1 && cap >= 1, "pfz_dense_topn_select: k=%d, cap=%d must be >= 1", k, cap);
    SelectParams P = {};
    P.idx = cand_idx; P.val = cand_val; P.count = cand_count; P.n_rows = n_rows; P.n_cand = cap;
    P.row_stride = cap; P.seg_len = cap; P.seg_stride = 0; P.row_map = row_map;
    P.k = k; P.thr = min_similarity; P.self_match = self_match; P.from_base = from_index_base; P.top_idx = top_idx; P.top_val = top_val;
    return topn_select_launch(P, as_stream(stream));
}

int pfz_dense_exact_rescore(const double *x_f64, const double *y_f64, int32_t n_from, int32_t n_to, int32_t d_pad, int32_t k, int32_t k_cand,
                            const int32_t *cand_idx, const double *cand_val, const double *x_norm16, const double *x_err16, const double *y_maxima,
                            double min_similarity, int32_t self_match, int64_t from_index_base, int64_t to_index_base, int32_t *top_idx,
                            double *top_val, int32_t *fb_rows, int32_t *fb_count, void *stream) {
    PFZ_REQUIRE(k >= 1 && k <= 32 && k_cand >= k && k_cand <= 32, "pfz_dense_exact_rescore: need 1 <= k (%d) <= k_cand (%d) <= 32", k, k_cand);
    PFZ_REQUIRE(d_pad >= 8 && d_pad % 8 == 0, "pfz_dense_exact_rescore: d_pad=%d must be a multiple of 8", d_pad);
    cudaStream_t st = as_stream(stream);
    PFZ_CUDA_OK(cudaMemsetAsync(fb_count, 0, sizeof(int32_t), st));
    if (n_from <= 0) return 0;
    PFZ_REQUIRE(n_to > 0, "pfz_dense_exact_rescore: empty to-matrix");
    ExactParams P;
    P.x = x_f64; P.y = y_f64; P.n_from = n_from; P.n_to = n_to; P.d_pad = d_pad; P.k = k; P.kc = k_cand;
    P.thr = min_similarity; P.gamma = exact_gamma(d_pad); P.m_max = exact_margin_max(d_pad); P.self_match = self_match;
    P.from_base = from_index_base; P.to_base = to_index_base;
    P.cand_idx = cand_idx; P.cand_val = cand_val; P.x_norm = x_norm16; P.x_err = x_err16; P.y_max = y_maxima;
    P.top_idx = top_idx; P.top_val = top_val; P.fb_rows = fb_rows; P.fb_count = fb_count;
    int grid = (n_from + 7) / 8; if (grid > SM_COUNT * 16) grid = SM_COUNT * 16;
    exact_rescore_kernel<<<grid, 256, 0, st>>>(P);
    PFZ_LAUNCH_OK();
    return 0;
}

int64_t pfz_dense_exact_fallback_ws_bytes(int32_t n_from, int32_t n_to, int32_t k) {
    const int64_t cap = n_from < FB_CAP_ROWS ? (n_from > 0 ? n_from : 1) : FB_CAP_ROWS;
    return cap * fb_splits(n_to) * (int64_t)(k > 0 ? k : 1) * 12 + cap * 4 + 256;
}

int pfz_dense_exact_fallback(const double *x_f64, const double *y_f64, int32_t n_from, int32_t n_to, int32_t d_pad, int32_t k, double min_similarity,
                             int32_t self_match, int64_t from_index_base, int64_t to_index_base, const int32_t *fb_rows, const int32_t *fb_count,
                             int32_t *top_idx, double *top_val, void *ws, void *stream) {
    PFZ_REQUIRE(k >= 1 && k <= 32, "pfz_dense_exact_fallback: k=%d unsupported (1..32)", k);
    if (n_from <= 0) return 0;
    PFZ_REQUIRE(n_to > 0, "pfz_dense_exact_fallback: empty to-matrix");
    cudaStream_t st = as_stream(stream);
    FallbackParams P;
    P.x = x_f64; P.y = y_f64; P.n_to = n_to; P.d_pad = d_pad; P.k = k; P.thr = min_similarity; P.self_match = self_match;
    P.from_base = from_index_base; P.to_base = to_index_base; P.fb_rows = fb_rows; P.fb_count = fb_count;
    P.n_splits = fb_splits(n_to); P.cap = n_from < FB_CAP_ROWS ? n_from : FB_CAP_ROWS;
    const int64_t n_part = (int64_t)P.cap * P.n_splits * k;
    P.ws_val = (double *)ws; P.ws_idx = (int32_t *)(P.ws_val + n_part); P.ws_done = P.ws_idx + n_part;
    P.top_idx = top_idx; P.top_val = top_val;
    PFZ_CUDA_OK(cudaMemsetAsync(P.ws_done, 0, (size_t)P.cap * sizeof(int32_t), st));
    exact_fallback_kernel<<<SM_COUNT * 4, FB_WARPS * 32, 0, st>>>(P);
    PFZ_LAUNCH_OK();
    return 0;
}
}
