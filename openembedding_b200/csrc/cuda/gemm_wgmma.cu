// gemm_wgmma.cu -- hand-written sm_90a GEMM for the dense side of the CTR models.
//
//   D[M,N] (+)= A[M,K] * B[N,K]^T      A, B bf16, fp32 accumulation in registers
//
// One 128xBN output tile per CTA (optionally one K-split of it), warp specialised:
//   warps 0..7  two consumer warpgroups. Warpgroup g owns rows [64 g, 64 g + 64) of the tile and issues
//               wgmma.mma_async m64nBNk16 (bf16 in, fp32 accumulator in registers) straight from the
//               128B-swizzled smem stages, then runs the fused epilogue on its accumulator fragment
//               -> swizzled smem staging tile -> TMA store
//   warp 8      TMA producer   cp.async.bulk.tensor.2d (128B swizzle) -> STAGES-deep smem ring;
//               mbarriers: full (transaction bytes of a stage landed) / empty (every consumer warp's
//               wgmma on the stage retired)
// Fused epilogues (the reference gets these from cuBLAS/cuDNN via TensorFlow, K6 in SURVEY 2.5):
//   EPI_FWD   relu, "ones" column (bias folded into the next layer's weights), bf16 store
//             plus a transposed bf16 copy (the batch-major operand of the dW GEMMs)
//   EPI_DX    relu mask from the forward activation, bf16 store (+ transposed copy)
//   EPI_DW    split-K partial sums, fp32 TMA reduce-add
//   EPI_DX_FM fp32 store of the embedding gradient with the FM second-order term fused
// The relu mask and the FM embedding columns reach the epilogue as a TMA-loaded source tile in the staging tile
// (epi_src_boxes / load_epi_src).
//
// Every GEMM of the training step (3 forward, 3 dX, 3 dW) is this one kernel. Operands reach wgmma
// either K-major (transposed copies written by the producing epilogue) or MN-major (the dW products
// straight from batch-major activations, exb_gemm_bf16_tn): wgmma transposes bf16 tiles in hardware.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include "pdl.cuh"
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>
#include <algorithm>

namespace {

constexpr int BM = 128, BK = 64;
constexpr int A_BYTES = BM * BK * 2;
// Tile width. A 128x64 tile re-reads (1/128 + 1/64) operand bytes per output element, a 128x128 tile
// (1/128 + 1/128), a third less, but a GEMM then has half as many tiles to spread over the SMs.
//   BN = 64 : 4 stages x 24 KB = 96 KB, two CTAs per SM -- the default
//   BN = 128: 3 stages x 32 KB = 96 KB, two CTAs per SM -- tall, short-K products (pick_bn)
template <int BN> constexpr int stages_for() { return BN == 64 ? 4 : 3; }
constexpr int NUM_CONSUMER_WARPS = 8;                       // two warpgroups of 64 tile rows each
constexpr int PRODUCER_WARP = NUM_CONSUMER_WARPS;
constexpr int NUM_THREADS = 32 * (NUM_CONSUMER_WARPS + 1);

enum EpiMode : int { EPI_FWD = 0, EPI_DX = 1, EPI_DW = 2, EPI_DX_FM = 3 };

struct GemmEpi {
    int mode, relu, ones_col, fm_cols;
    int M, N, D, mn_major;   // mn_major: A is stored [K, M], B is stored [K, N] (MN contiguous)
    void* out; long long ldo;
    __nv_bfloat16* outT; long long ldoT;
    const __nv_bfloat16* mask; long long ldmask;
    const float* dlogit; const float* S; const float* emb; long long ldemb;
    int swap, mc;              // mc: CTAs per cluster along the N-tile axis that share (multicast) the A tile; <= 1: off
    unsigned long long* dbg;   // optional: %globaltimer stamps of CTA (0,0,0) [start, setup, first-full, mainloop, epilogue]
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t n) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(n) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* b, uint32_t cta) {
    asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\t"
                 "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
                 ::"r"(smem_u32(b)), "r"(cta) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t* b, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
    return ok != 0;
}
// pipeline waits that gave up (mbar_wait); read and cleared by exb_gemm_timeouts()
__device__ unsigned int g_pipeline_timeouts;
// bounded: a descriptor bug must surface as an error, never as a hung GPU
__device__ __forceinline__ bool mbar_wait(uint64_t* b, uint32_t parity) {
    for (uint32_t it = 0; it < (1u << 24); ++it)
        if (mbar_try(b, parity)) return true;
    atomicAdd(&g_pipeline_timeouts, 1u);
    return false;
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// A-tile multicast: the tile lands at the same shared-memory offset of every CTA in `mask` and completes the
// transaction bytes on each destination CTA's own barrier (same offset)
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint16_t mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%4, %5}], [%2], %3;"
                 ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// wgmma shared-memory matrix descriptor, SWIZZLE_128B. K-major: [rows][64 bf16 = 128 B], 8 rows form a
// 1024-byte swizzle atom (stride byte offset); the leading byte offset is unused. MN-major: [k rows][64 MN
// elements = 128 B], 8 k-rows form an atom, 64-element MN blocks are `lbo_bytes` apart. Canonical form
// ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);   // start address
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;               // stride byte offset: 8 rows x 128 B
    d |= (uint64_t)1 << 62;                         // SWIZZLE_128B
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across a wgmma wait
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T; TRANS = 1: both operands MN-major
template <int TRANS>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
                 "}, %32, %33, p, 1, 1, %35, %35;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(scale_d), "n"(TRANS));
}
template <int TRANS>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
                 "}, %64, %65, p, 1, 1, %67, %67;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(scale_d), "n"(TRANS));
}
// one BK = 64 slice of a stage: four k16 steps for warpgroup g (A rows [64 g, 64 g + 64) of the tile)
template <int BN, int TRANS>
__device__ __forceinline__ void wgmma_stage(float (&acc)[BN / 2], uint32_t a0, uint32_t b0, int g, bool first) {
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
        // K-major: a k16 step is 32 bytes inside the 128-byte swizzled row; MN-major: 16 k rows = 2048 bytes
        const uint64_t da = TRANS ? gmma_desc(a0 + g * 8192 + k * 2048, 8192) : gmma_desc(a0 + g * 8192 + k * 32, 16);
        const uint64_t db = TRANS ? gmma_desc(b0 + k * 2048, 8192) : gmma_desc(b0 + k * 32, 16);
        const uint32_t sd = (first && k == 0) ? 0u : 1u;
        if constexpr (BN == 64) wgmma_n64<TRANS>(acc, da, db, sd);
        else wgmma_n128<TRANS>(acc, da, db, sd);
    }
}

// Main loop of one tile for a consumer warp: stages kiter .. kiter + nkb - 1 of the ring. A stage is released
// (its empty barrier, in every CTA of a multicast cluster of C CTAs) once this warp's wgmma reading it retired;
// the wgmma of the next stage is issued before that wait, so the tensor core never idles on the release.
template <int BN>
__device__ __forceinline__ void mma_tile(float (&acc)[BN / 2], const uint8_t* sA, const uint8_t* sB, uint64_t* full,
                                         uint64_t* empty, int stages, uint32_t kiter, int nkb, bool mn_major, int g,
                                         int C) {
    constexpr int B_BYTES = BN * BK * 2;
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    auto release = [&](uint32_t it) {
        const int s = it % stages;
        if (C > 1) { if (lane < C) mbar_arrive_cluster(&empty[s], (uint32_t)lane); }
        else if (lane == 0) mbar_arrive(&empty[s]);
    };
    for (int i = 0; i < nkb; ++i) {
        const uint32_t it = kiter + i;
        const int s = it % stages;
        mbar_wait(&full[s], (it / stages) & 1u);
        const uint32_t a0 = smem_u32(sA + s * A_BYTES), b0 = smem_u32(sB + s * B_BYTES);
        wgmma_fence();
        if (mn_major) wgmma_stage<BN, 1>(acc, a0, b0, g, i == 0);
        else wgmma_stage<BN, 0>(acc, a0, b0, g, i == 0);
        wgmma_commit();
        if (i > 0) {
            wgmma_wait<1>();
            acc_fence(acc);
            release(it - 1);
        }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (nkb > 0) release(kiter + nkb - 1);
}

// Epilogue source tile: the operand the fused math reads elementwise beside the accumulator -- the relu mask of
// EPI_DX (bf16 [M, N], 64-column boxes) or the FM embedding columns of EPI_DX_FM (fp32 [M, fm_cols], 32-column
// boxes). A box of it is laid out exactly like the output staging tile it lands in (rows of 128 bytes, 128B
// swizzle), so the epilogue reads each element from the address it then writes its result to.
// Boxes per 32-row quarter of a 128 x BN tile; 0: the tile has no source (every other epilogue, fm_cols = 0, a
// tile right of the embedding columns).
template <int BN>
__device__ __forceinline__ int epi_src_boxes(int mode, int fm_cols, int N, int n_blk) {
    const int n0 = n_blk * BN;
    if (mode == EPI_DX) return min(BN / 64, (N - n0 + 63) / 64);
    if (mode == EPI_DX_FM && fm_cols > n0) return min(BN / 32, (fm_cols - n0 + 31) / 32);
    return 0;
}
// TMA loads of warpgroup g's two staging quarters, completing on `bar` (issued by one thread). Quarters that start
// at or past row M are skipped: their rows are masked in the epilogue. Rows >= M of a partial quarter and columns
// past the tensor's width arrive zero-filled.
template <int BN>
__device__ __forceinline__ void load_epi_src(const CUtensorMap* tE, uint64_t* bar, uint8_t* stage, int qstride, int g,
                                             int m_blk, int n_blk, int boxes, int M, bool f32) {
    const int row0 = m_blk * BM + 2 * g * 32;
    const int quarters = row0 >= M ? 0 : (row0 + 32 >= M ? 1 : 2);
    mbar_expect_tx(bar, (uint32_t)(quarters * boxes * 4096));
#pragma unroll 1
    for (int qq = 0; qq < quarters; ++qq)
#pragma unroll 1
        for (int h = 0; h < boxes; ++h)
            tma_load_2d(stage + (2 * g + qq) * qstride + h * 4096, tE, bar, n_blk * BN + (f32 ? 32 : 64) * h, row0 + 32 * qq);
}

// Fused epilogue of warpgroup g: accumulator fragment -> fused math -> 128B-swizzled staging tiles (one per
// 32-row quarter of the tile, `qstride` bytes apart; out tiles first, the outT tile at +BN*128) -> TMA stores
// issued by the warpgroup's first thread (committed as one bulk group; the caller waits on it).
// EPI_DX / EPI_DX_FM: the caller has landed the epilogue source tile in the staging tiles (load_epi_src).
// wgmma m64nN fragment: thread (warp w, lane l) holds rows 16 w + l/4 (+8) and columns 8 j + 2 (l%4) (+1).
template <int BN>
__device__ __forceinline__ void epilogue_tile(const GemmEpi& E, float (&acc)[BN / 2], int m_blk, int n_blk, int g,
                                              uint8_t* stage, int qstride, const CUtensorMap* tO, const CUtensorMap* tT) {
    // kept in registers: in the chain the descriptor lives in shared memory, and the staging stores below could
    // alias it for the compiler, which then re-reads every field after every store
    const int mode = E.mode, relu = E.relu, ones_col = E.ones_col, fm_cols = E.fm_cols, N = E.N, D = E.D;
    const bool has_t = E.outT != nullptr;
    const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
    const bool f32out = (mode == EPI_DW || mode == EPI_DX_FM);
    const int q = 2 * g + (w >> 1);
    uint8_t* wstage = stage + q * qstride;
    uint8_t* tstage = wstage + BN * 128;
    // The one global operand left is S of the FM term ([M, D] fp32, small and L2-resident): read-only loads of SG
    // column pairs issued together, ahead of the math and staging stores of those pairs. At two CTAs per SM a
    // thread has 96 registers; BN = 128 with its 64 accumulators takes fewer pairs at a time.
    constexpr int SG = BN == 64 ? BN / 8 : 2;
    // BN = 64: the S column n % D of this thread's first pair and the step to the next pair (8 columns on), so one
    // division per tile instead of two per pair; D is even (host-checked) and n is even, so n % D + 1 < D and a pair
    // is one float2 load. BN = 128 keeps the per-pair divisions: with this its registers spill 64 bytes instead of 8.
    const bool fm_tile = mode == EPI_DX_FM && n_blk * BN < fm_cols;
    const int dcol0 = (BN == 64 && fm_tile) ? (n_blk * BN + 2 * (l & 3)) % D : 0;
    const int dstep = (BN == 64 && fm_tile) ? 8 % D : 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int qrow = (w & 1) * 16 + (l >> 2) + 8 * i;
        const int row = m_blk * BM + q * 32 + qrow;
        const bool rv = row < E.M;
        // dlogit / S / emb exist only when the tile has FM columns (fm_cols = 0: plain fp32 dX, null pointers)
        const bool fm_row = mode == EPI_DX_FM && rv && n_blk * BN < fm_cols;
        const float dl = fm_row ? __ldg(E.dlogit + row) : 0.f;
        const float* sb = E.S + (size_t)row * D;
        int dcol = dcol0;
#pragma unroll
        for (int j0 = 0; j0 < BN / 8; j0 += SG) {
            float2 s[SG];       // S at the two columns of the pair (the FM term's dimension n % D)
#pragma unroll
            for (int jj = 0; jj < SG; ++jj) {
                const int n = n_blk * BN + 8 * (j0 + jj) + 2 * (l & 3);
                s[jj] = make_float2(0.f, 0.f);
                // per column pair: n is even and fm_cols = nf * Dp a multiple of 4, so n + 1 < fm_cols as well.
                // fm_cols need not be a multiple of 32 (nf * Dp = 208 at dim 8): the columns of a partial
                // 32-column group are embedding columns too and need the FM term
                if constexpr (BN == 64) {
                    if (fm_row && n < fm_cols) s[jj] = __ldg(reinterpret_cast<const float2*>(sb + dcol));
                    dcol += dstep;
                    if (dcol >= D) dcol -= D;
                } else if (fm_row && n < fm_cols) {
                    s[jj] = make_float2(__ldg(sb + n % D), __ldg(sb + (n + 1) % D));
                }
            }
#pragma unroll
            for (int jj = 0; jj < SG; ++jj) {
                const int j = j0 + jj;
                const int c = 8 * j + 2 * (l & 3);
                const int n = n_blk * BN + c;
                float x[2] = {acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]};
                // this pair's slot in the swizzled staging tile (rows of 128 bytes, 16-byte chunk index ^ (row & 7)):
                // fp32 [32 rows][32 fp32] per 32 columns | bf16 [32 rows][64 bf16] per 64 columns
                const int cc = f32out ? (c & 31) : (c & 63);
                uint8_t* slot = f32out
                    ? wstage + (c >> 5) * 4096 + qrow * 128 + ((((cc >> 2) ^ (qrow & 7))) << 4) + (cc & 3) * 4
                    : wstage + (c >> 6) * 4096 + qrow * 128 + ((((cc >> 3) ^ (qrow & 7))) << 4) + (cc & 7) * 2;
                if (mode == EPI_FWD) {
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        if (relu) x[u] = fmaxf(x[u], 0.f);
                        if (n + u == ones_col) x[u] = 1.f;
                        if (n + u >= N) x[u] = 0.f;
                    }
                } else if (mode == EPI_DX) {
                    float2 mk = make_float2(0.f, 0.f);     // relu mask, from the source tile
                    if (rv && n < N) mk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(slot));
                    const float mv[2] = {mk.x, mk.y};
#pragma unroll
                    for (int u = 0; u < 2; ++u)
                        if (!rv || !(mv[u] > 0.f) || n + u == ones_col || n + u >= N) x[u] = 0.f;
                } else if (fm_row && n < fm_cols) {
                    const float2 e = *reinterpret_cast<const float2*>(slot);   // embedding pair, from the source tile
                    x[0] += dl * (s[jj].x - e.x);
                    x[1] += dl * (s[jj].y - e.y);
                }
                if (f32out) {
                    *reinterpret_cast<float2*>(slot) = make_float2(x[0], x[1]);
                } else {
                    *reinterpret_cast<__nv_bfloat162*>(slot) = __floats2bfloat162_rn(x[0], x[1]);
                    if (has_t) {    // [BN n][32 rows] bf16
                        *reinterpret_cast<__nv_bfloat16*>(tstage + c * 64 + qrow * 2) = __float2bfloat16_rn(x[0]);
                        *reinterpret_cast<__nv_bfloat16*>(tstage + (c + 1) * 64 + qrow * 2) = __float2bfloat16_rn(x[1]);
                    }
                }
            }
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy smem writes -> TMA reads
    named_bar_sync(2 + g, 128);
    if (t == 0) {
        if (E.fm_cols != -7) {   // -7: timing probe without stores
#pragma unroll 1
            for (int qq = 2 * g; qq < 2 * g + 2; ++qq) {
                const int row0 = m_blk * BM + qq * 32;
                uint8_t* ws = stage + qq * qstride;
                if (f32out) {
#pragma unroll 1
                    for (int h = 0; h < BN / 32; ++h) {
                        const int n0 = n_blk * BN + 32 * h;
                        if (E.mode == EPI_DW)
                            asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
                                         ::"l"(tO), "r"(smem_u32(ws + h * 4096)), "r"(n0), "r"(row0) : "memory");
                        else
                            asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                         ::"l"(tO), "r"(smem_u32(ws + h * 4096)), "r"(n0), "r"(row0) : "memory");
                    }
                } else {
#pragma unroll 1
                    for (int h = 0; h < BN / 64; ++h)
                        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                     ::"l"(tO), "r"(smem_u32(ws + h * 4096)), "r"(n_blk * BN + 64 * h), "r"(row0) : "memory");
                    if (E.outT)
                        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                     ::"l"(tT), "r"(smem_u32(ws + BN * 128)), "r"(row0), "r"(n_blk * BN) : "memory");
                }
            }
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
}

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 2)
exb_gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmT,
                      const __grid_constant__ CUtensorMap tmE, GemmEpi E, int num_k_blocks, int k_blocks_per_split) {
    static_assert(BN == 64 || BN == 128, "tile width");
    constexpr int STAGES = stages_for<BN>();
    constexpr int B_BYTES = BN * BK * 2;
    constexpr int QSTAGE = BN * 128 + BN * 64;     // per 32-row quarter: out tiles | outT tile
    static_assert(4 * QSTAGE <= STAGES * (A_BYTES + B_BYTES), "epilogue staging aliases the stage memory");
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte aligned bases; do not rely on the toolchain for it
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
    uint64_t* empty = full + STAGES;
    uint64_t* srcfull = empty + STAGES;            // per warpgroup: its quarters of the epilogue source tile landed

    exb::pdl_trigger();   // the next kernel of the step may be scheduled once all CTAs are resident
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // E.swap: N tiles vary fastest over the launch order (neighbouring CTAs share the A tile, not the B tile)
    const int m_blk = E.swap ? blockIdx.y : blockIdx.x, n_blk = E.swap ? blockIdx.x : blockIdx.y;
    const bool dbg = E.dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0;
#define GSTAMP(i) do { if (dbg) { unsigned long long _t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_t)); E.dbg[i] = _t; } } while (0)
    if (threadIdx.x == 0) GSTAMP(0);
    const int kb0 = blockIdx.z * k_blocks_per_split;
    const int kb1 = min(num_k_blocks, kb0 + k_blocks_per_split);
    const int nkb = kb1 - kb0;
    // E.mc > 1: launched as clusters of E.mc CTAs with the same M block and consecutive N blocks. Rank 0 loads the A
    // tile ONCE and multicasts it into every CTA of the cluster (A is 2/3 of the operand bytes of a 128x64 tile);
    // each CTA loads its own B tile. A stage is re-filled only when EVERY CTA of the cluster has consumed it: the
    // consumer warps arrive on all CTAs' empty barriers.
    const int C = E.mc > 1 ? E.mc : 1;
    uint32_t crank = 0;
    if (C > 1) asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(crank));
    const uint16_t cmask = (uint16_t)((1u << C) - 1u);

    if (threadIdx.x == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], (uint32_t)(NUM_CONSUMER_WARPS * C)); }
        mbar_init(&srcfull[0], 1); mbar_init(&srcfull[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    }
    __syncthreads();
    if (C > 1) cluster_sync_all();     // every CTA's barriers exist before a peer multicasts into / arrives on them
    exb::pdl_wait();      // barriers and tensor maps are ready; operands come from the previous kernel
    if (threadIdx.x == 0) GSTAMP(1);

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {   // ===== TMA producer
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                const uint32_t ph = (uint32_t)(i / STAGES) & 1u;
                mbar_wait(&empty[s], ph ^ 1u);
                mbar_expect_tx(&full[s], A_BYTES + B_BYTES);
                if (E.mn_major) {   // boxes of 64 MN elements x 64 k rows; the A tile is two MN blocks
                    if (C > 1) {
                        if (crank == 0) {
                            tma_load_2d_mc(sA + s * A_BYTES, &tmA, &full[s], m_blk * BM, (kb0 + i) * BK, cmask);
                            tma_load_2d_mc(sA + s * A_BYTES + A_BYTES / 2, &tmA, &full[s], m_blk * BM + 64, (kb0 + i) * BK, cmask);
                        }
                    } else {
                        tma_load_2d(sA + s * A_BYTES, &tmA, &full[s], m_blk * BM, (kb0 + i) * BK);
                        tma_load_2d(sA + s * A_BYTES + A_BYTES / 2, &tmA, &full[s], m_blk * BM + 64, (kb0 + i) * BK);
                    }
#pragma unroll
                    for (int h = 0; h < BN / 64; ++h)
                        tma_load_2d(sB + s * B_BYTES + h * 8192, &tmB, &full[s], n_blk * BN + 64 * h, (kb0 + i) * BK);
                    continue;
                }
                if (C > 1) {
                    if (crank == 0) tma_load_2d_mc(sA + s * A_BYTES, &tmA, &full[s], (kb0 + i) * BK, m_blk * BM, cmask);
                } else {
                    tma_load_2d(sA + s * A_BYTES, &tmA, &full[s], (kb0 + i) * BK, m_blk * BM);
                }
                tma_load_2d(sB + s * B_BYTES, &tmB, &full[s], (kb0 + i) * BK, n_blk * BN);
            }
        }
    } else {
        // ===== consumer warpgroups
        const int g = warp >> 2;
        float acc[BN / 2];
        if (dbg && threadIdx.x == 0 && nkb > 0) { mbar_wait(&full[0], 0); GSTAMP(2); }
        mma_tile<BN>(acc, sA, sB, full, empty, STAGES, 0u, nkb, E.mn_major != 0, g, C);
        if (threadIdx.x == 0) GSTAMP(3);
        // the staging tiles alias the stage ring: both warpgroups' wgmma reads must have retired
        named_bar_sync(1, 32 * NUM_CONSUMER_WARPS);
        // so the epilogue source tile can only be requested now: one bulk round trip per warpgroup
        const int boxes = epi_src_boxes<BN>(E.mode, E.fm_cols, E.N, n_blk);
        if (boxes) {
            if ((threadIdx.x & 127) == 0)
                load_epi_src<BN>(&tmE, &srcfull[g], smem, QSTAGE, g, m_blk, n_blk, boxes, E.M, E.mode == EPI_DX_FM);
            mbar_wait(&srcfull[g], 0);
        }
        epilogue_tile<BN>(E, acc, m_blk, n_blk, g, smem, QSTAGE, &tmO, &tmT);
        if ((threadIdx.x & 127) == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        if (threadIdx.x == 0) GSTAMP(4);
    }
    __syncthreads();
    if (threadIdx.x == 0) GSTAMP(5);
    if (C > 1) cluster_sync_all();     // no CTA leaves while a peer may still multicast into / arrive on its memory
}

// =====================================================================================================
// Persistent GEMM CHAIN: several dependent GEMMs of the training step in ONE launch.
//
// The dense side of a CTR step is nine small GEMMs (M = batch 4096, N / K in {448, 1728}); launched one by one
// every kernel pays launch + barrier init + pipeline fill + epilogue drain + a partial last wave for a few
// microseconds of tensor work, and a layer cannot start before the previous kernel has fully drained.
// Here the tiles of all GEMMs of a chain (forward: fwd1 -> fwd2 -> fwd3; backward: dX3, dW3, dX2, dW2, dX1, dW1)
// form ONE static work list consumed by persistent CTAs (two per SM):
//   * set-up once per CTA; the TMA -> wgmma smem ring and its phases run on ACROSS tiles, so the producer
//     loads the next tile's stages while the consumers run the epilogue of this one;
//   * dependencies are per 128-row block, not per kernel: a tile of layer l+1 starts as soon as the row block of
//     layer l it reads is complete (`ready` counters, release / acquire at gpu scope + async-proxy fences) -- the
//     batch-parallel structure of an MLP (row blocks are independent through forward AND backward) pipelines
//     naturally; the split-K weight-gradient tiles wait for the row blocks of their K range only;
//   * the static order puts every producer before its consumers, and each CTA walks its items in increasing order,
//     so the smallest unfinished item can always run: no deadlock.
// Tile code (TMA boxes, wgmma descriptors, main loop, fused epilogues) is the one of exb_gemm_wgmma_kernel<64>,
// so a chain computes bit for bit what the single launches compute.
constexpr int CH_STAGES = 3;                  // 3 x 24 KB ring + 32 KB epilogue staging: two CTAs per SM
constexpr int CH_BN = 64;
constexpr int CH_B_BYTES = CH_BN * BK * 2;
constexpr int CH_MAX_PROB = 8;

struct ChainMaps { CUtensorMap tmA, tmB, tmO, tmE; };  // tmE: epilogue source tile (zeroed when the GEMM has none)
struct ChainMapsAll { ChainMaps m[CH_MAX_PROB]; };    // passed as a __grid_constant__ parameter (4 KB): descriptors in param space
struct ChainMeta {
    GemmEpi E;
    int m_tiles, n_tiles, splits, nkb, per;
    int item0, items;
    int dep, dep_kind, dep_need;              // dep_kind 0 none | 1 A rows = my row block | 2 my K range (batch rows)
    int signal;
};

__device__ __forceinline__ void ch_decode(const ChainMeta* M, int nprob, int item, int& p, int& m, int& n, int& z) {
    p = 0;
#pragma unroll 1
    for (int i = 1; i < nprob; ++i)
        if (item >= M[i].item0) p = i;
    const int local = item - M[p].item0;
    const int mn = M[p].m_tiles * M[p].n_tiles;
    z = local / mn;
    const int r = local - z * mn;
    m = r / M[p].n_tiles;
    n = r - m * M[p].n_tiles;
}
__device__ __forceinline__ unsigned ch_ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// ready: one counter per (GEMM p, row block m) at p * mb_stride + m (mb_stride: the largest row-block count of the
// chain), then the counter of CTAs that have left
__global__ void __launch_bounds__(NUM_THREADS, 2)
exb_gemm_chain_kernel(const __grid_constant__ ChainMapsAll MAPS, const ChainMeta* __restrict__ metas, int nprob, int total_items,
                      unsigned* __restrict__ ready, int mb_stride, int* __restrict__ err) {
    const ChainMaps* maps = MAPS.m;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + CH_STAGES * A_BYTES;
    uint8_t* sStage = sB + CH_STAGES * CH_B_BYTES;                 // 4 quarters x 8 KB (1024-byte aligned)
    uint64_t* full = reinterpret_cast<uint64_t*>(sStage + 4 * 8192);
    uint64_t* empty = full + CH_STAGES;
    // per consumer warpgroup g, for its two staging quarters: sfree -- the TMA store of its previous tile has read
    // them; srcfull -- the epilogue source boxes of its current tile landed in them
    uint64_t* sfree = empty + CH_STAGES;
    uint64_t* srcfull = sfree + 2;
    ChainMeta* M = reinterpret_cast<ChainMeta*>(srcfull + 2);

    exb::pdl_trigger();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < nprob * (int)(sizeof(ChainMeta) / 4); i += blockDim.x)
        reinterpret_cast<uint32_t*>(M)[i] = reinterpret_cast<const uint32_t*>(metas)[i];     // host-written
    if (threadIdx.x == 0) {
        for (int i = 0; i < CH_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], NUM_CONSUMER_WARPS); }
        for (int i = 0; i < 2; ++i) { mbar_init(&sfree[i], 1); mbar_init(&srcfull[i], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    exb::pdl_wait();

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {   // ===== TMA producer
            uint32_t kiter = 0, tile = 0;
            for (int item = blockIdx.x; item < total_items; item += gridDim.x, ++tile) {
                int p, m_blk, n_blk, z;
                ch_decode(M, nprob, item, p, m_blk, n_blk, z);
                const ChainMeta& Q = M[p];
                const int kb0 = z * Q.per, kb1 = min(Q.nkb, kb0 + Q.per);
                if (Q.dep_kind) {      // the row blocks this tile reads must be complete
                    int mb0 = m_blk, mb1 = m_blk + 1;
                    if (Q.dep_kind == 2) { mb0 = (kb0 * BK) / BM; mb1 = (kb1 * BK + BM - 1) / BM; }
                    const unsigned* cnt = ready + Q.dep * mb_stride;
                    for (int mb = mb0; mb < mb1; ++mb) {
                        uint32_t it = 0;
                        while (ch_ld_acquire(cnt + mb) < (unsigned)Q.dep_need) {
                            __nanosleep(64);
                            if (++it > (1u << 22)) { atomicCAS(err, 0, 100 + p); break; }
                        }
                    }
                    asm volatile("fence.proxy.async;" ::: "memory");   // generic acquire -> async-proxy (TMA) reads
                }
                const CUtensorMap* tA = &maps[p].tmA;
                const CUtensorMap* tB = &maps[p].tmB;
                const int boxes = epi_src_boxes<CH_BN>(Q.E.mode, Q.E.fm_cols, Q.E.N, n_blk);
                // Staging hand-off, after the ring stages that are free while the consumers finish the previous
                // tile and before the last k-block: wait until both warpgroups' stores of the previous tile have read
                // the staging quarters, then load this tile's epilogue source into them. Waiting first would
                // serialise the ring behind the store; waiting before the last k-block keeps a consumer from
                // completing this tile's hand-off before the wait for the previous one (one phase in flight).
                const int handoff = kb0 + min(CH_STAGES, kb1 - kb0 - 1);
                for (int kb = kb0; kb < kb1; ++kb, ++kiter) {
                    if (kb == handoff) {
                        if (tile > 0) { mbar_wait(&sfree[0], (tile - 1) & 1u); mbar_wait(&sfree[1], (tile - 1) & 1u); }
                        if (boxes)
                            for (int g = 0; g < 2; ++g)
                                load_epi_src<CH_BN>(&maps[p].tmE, &srcfull[g], sStage, 8192, g, m_blk, n_blk, boxes, Q.E.M,
                                                    Q.E.mode == EPI_DX_FM);
                    }
                    const int s = kiter % CH_STAGES;
                    const uint32_t ph = (kiter / CH_STAGES) & 1u;
                    mbar_wait(&empty[s], ph ^ 1u);
                    mbar_expect_tx(&full[s], A_BYTES + CH_B_BYTES);
                    if (Q.E.mn_major) {
                        tma_load_2d(sA + s * A_BYTES, tA, &full[s], m_blk * BM, kb * BK);
                        tma_load_2d(sA + s * A_BYTES + A_BYTES / 2, tA, &full[s], m_blk * BM + 64, kb * BK);
                        tma_load_2d(sB + s * CH_B_BYTES, tB, &full[s], n_blk * CH_BN, kb * BK);
                    } else {
                        tma_load_2d(sA + s * A_BYTES, tA, &full[s], kb * BK, m_blk * BM);
                        tma_load_2d(sB + s * CH_B_BYTES, tB, &full[s], kb * BK, n_blk * CH_BN);
                    }
                }
            }
        }
    } else {
        // ===== consumer warpgroups: main loop + epilogue of every item of this CTA
        const int g = warp >> 2;
        uint32_t kiter = 0, nsrc = 0;
        float acc[CH_BN / 2];
        for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
            int p, m_blk, n_blk, z;
            ch_decode(M, nprob, item, p, m_blk, n_blk, z);
            const ChainMeta& Q = M[p];
            const int kb0 = z * Q.per, kb1 = min(Q.nkb, kb0 + Q.per);
            // broadcast from lane 0: the compiler then knows the wgmma path is warp-uniform (values read from shared
            // memory are not, and a divergent path makes ptxas serialize every wgmma)
            const int nk = __shfl_sync(0xffffffffu, kb1 - kb0, 0);
            const int mn = __shfl_sync(0xffffffffu, Q.E.mn_major, 0);
            mma_tile<CH_BN>(acc, sA, sB, full, empty, CH_STAGES, kiter, nk, mn != 0, g, 1);
            kiter += nk;
            if (epi_src_boxes<CH_BN>(Q.E.mode, Q.E.fm_cols, Q.E.N, n_blk)) mbar_wait(&srcfull[g], (nsrc++) & 1u);
            epilogue_tile<CH_BN>(Q.E, acc, m_blk, n_blk, g, sStage, 8192, &maps[p].tmO, &maps[p].tmO);
            if ((threadIdx.x & 127) == 0) {
                if (Q.signal) {
                    // a later GEMM of the chain reads this row block: its writes must have COMPLETED before the release
                    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
                    asm volatile("fence.proxy.async;" ::: "memory");
                    __threadfence();
                    atomicAdd(&ready[p * mb_stride + m_blk], 1u);
                } else {
                    // nobody inside this launch reads the tile (dW, the last dX): only the staging tile has to be free
                    // again; kernel completion makes the writes visible to the next kernel
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                }
                mbar_arrive(&sfree[g]);   // the producer may load the next tile's epilogue source into the staging
            }
            named_bar_sync(2 + g, 128);   // the staging tiles are free for the next item
        }
    }
    __syncthreads();
    // self-cleaning dependency counters: the LAST CTA to leave zeroes them for the next launch (no memset node in
    // front of the kernel, so the launch keeps its programmatic-dependent-launch edge inside a CUDA graph)
    if (warp == 0) {
        const int ncnt = nprob * mb_stride;
        unsigned last = 0;
        if (lane == 0) {
            __threadfence();
            last = (atomicAdd(&ready[ncnt], 1u) == gridDim.x - 1) ? 1u : 0u;
        }
        last = __shfl_sync(0xffffffffu, last, 0);
        if (last) {
            for (int i = lane; i < ncnt; i += 32) ready[i] = 0u;
            __syncwarp();
            if (lane == 0) { __threadfence(); ready[ncnt] = 0u; }
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
thread_local std::string g_gemm_err;

bool make_map_ex(CUtensorMap* map, CUtensorMapDataType dt, int esize, const void* ptr, long long rows, long long cols,
                 long long ld, int box_cols, int box_rows, CUtensorMapSwizzle sw);

bool make_map(CUtensorMap* map, const void* ptr, long long rows, long long cols, long long ld, int box_rows) {
    return make_map_ex(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, rows, cols, ld, BK, box_rows, CU_TENSOR_MAP_SWIZZLE_128B);
}

bool make_map_ex(CUtensorMap* map, CUtensorMapDataType dt, int esize, const void* ptr, long long rows, long long cols,
                 long long ld, int box_cols, int box_rows, CUtensorMapSwizzle sw) {
    if (!g_encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
            g_gemm_err = "cuTensorMapEncodeTiled entry point not found";
            return false;
        }
        g_encode = (EncodeTiledFn)fn;
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(map, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        g_gemm_err = "cuTensorMapEncodeTiled failed: " + std::to_string((int)r);
        return false;
    }
    return true;
}

template <int BN>
constexpr size_t gemm_smem() { return stages_for<BN>() * (A_BYTES + BN * BK * 2) + (2 * stages_for<BN>() + 2) * 8 + 16 + 1024; }

// Tensor map of the epilogue source tile (epi_src_boxes): the relu mask of EPI_DX, the embedding columns of
// EPI_DX_FM with fm_cols > 0. Returns true and leaves `map` untouched when the epilogue has no source.
bool make_epi_src_map(CUtensorMap* map, int mode, int fm_cols, int M, int N, const void* mask, long long ldmask,
                      const void* emb, long long ldemb) {
    const bool dx = mode == EPI_DX, fm = mode == EPI_DX_FM && fm_cols > 0;
    if (!dx && !fm) return true;
    const void* p = dx ? mask : emb;
    const long long ld = dx ? ldmask : ldemb;
    const int esize = dx ? 2 : 4;
    if (!p) { g_gemm_err = dx ? "gemm: EPI_DX needs the relu mask" : "gemm: fm_cols > 0 needs the embedding rows"; return false; }
    // TMA: 16-byte aligned base and row stride
    if (((uintptr_t)p & 15) != 0 || (ld * esize) % 16 != 0) {
        g_gemm_err = dx ? "gemm: relu mask base / row stride not 16-byte aligned"
                        : "gemm: embedding rows base / row stride not 16-byte aligned";
        return false;
    }
    if (dx) return make_map_ex(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, p, M, N, ld, 64, 32, CU_TENSOR_MAP_SWIZZLE_128B);
    return make_map_ex(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, p, M, fm_cols, ld, 32, 32, CU_TENSOR_MAP_SWIZZLE_128B);
}

// FM term of EPI_DX_FM: the epilogue reads S a column pair at a time as one float2 (epilogue_tile), so the padded
// dimension D must be even and S 8-byte aligned
bool fm_operands_ok(int mode, int fm_cols, int D, uint64_t S) {
    if (mode != EPI_DX_FM || fm_cols <= 0) return true;
    if (D < 2 || D % 2 != 0 || (S & 7) != 0) { g_gemm_err = "gemm: the FM term needs an even D and an 8-byte aligned S"; return false; }
    return true;
}

// tile width: env EXB_GEMM_BN (64 | 128) overrides
int pick_swap() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("EXB_GEMM_SWAP"); v = e ? atoi(e) : 0; }
    return v;
}
int pick_bn(int M, int N, int K) {
    static int forced = -1;
    if (forced < 0) { const char* e = getenv("EXB_GEMM_BN"); forced = e ? atoi(e) : 0; }
    if (forced == 64 || forced == 128) return forced;
    // default 64: the step's GEMMs (M = batch, N <= 1 728) have few tiles, and 64-wide tiles give twice as many to
    // spread over the SMs. Tall, short-K products (the CIN input-gradient GEMM: M 36 864, N 1 728, K 128 -- two
    // k-blocks per tile, thousands of tiles) take 128: their tiles are mostly set-up and epilogue, and the wider
    // tile halves their number. The DeepFM step keeps 64 by measurement on H100 (docs/benchmark.md): with 128 for
    // the two 448-K forward GEMMs only (fwd2, fwd3), bench.py ran 0.361-0.362 ms/step against 0.332 at 64, three
    // runs each, alternated; 128 for all three forward GEMMs was slower as well. Isolated back-to-back launches of
    // one GEMM (benchmarks/step_gemms.py) do not predict this: they swing by more than the width difference
    // between runs of the same code.
    if (K <= 128 && N >= 512 && M >= 8192) return 128;
    return 64;
}

template <int BN>
cudaError_t launch_gemm(dim3 grid, cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO,
                        const CUtensorMap& tmT, const CUtensorMap& tmE, const GemmEpi& E, int nkb, int per) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(exb_gemm_wgmma_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gemm_smem<BN>());
        attr_set = true;
    }
    if (E.mc > 1) {       // clusters of E.mc CTAs along grid.y (the N-tile axis when swap == 0)
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = grid; cfg.blockDim = dim3(NUM_THREADS); cfg.dynamicSmemBytes = gemm_smem<BN>(); cfg.stream = stream;
        cudaLaunchAttribute attr[2];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = (unsigned)E.mc; attr[0].val.clusterDim.z = 1;
        attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[1].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = exb::pdl_enabled() ? 2 : 1;
        return cudaLaunchKernelEx(&cfg, exb_gemm_wgmma_kernel<BN>, tmA, tmB, tmO, tmT, tmE, E, nkb, per);
    }
    return exb::launch_pdl(exb_gemm_wgmma_kernel<BN>, grid, dim3(NUM_THREADS), gemm_smem<BN>(), stream, tmA, tmB, tmO, tmT,
                           tmE, E, nkb, per);
}

// cluster size for the A-tile multicast: the largest divisor (<= EXB_GEMM_MC, <= 8) of the number of N tiles.
// OFF by default (EXB_GEMM_MC unset / 0): on H100 it makes every GEMM of the DeepFM step slower although it cuts the
// L2 operand bytes by 42-57% (benchmarks/step_gemms.py --mc, docs/benchmark.md; 400 W card, 3 alternated runs):
// dX1 without FM operands 32.8-33.1 us off, 51.8-52.3 us at 3 CTAs per cluster; fwd1 21.5-21.7 us off, 35.8-36.4 us
// at 7. The step's GEMMs are not bound by L2 operand bandwidth, and the lock step of a cluster costs more than the
// bytes it saves.
int pick_mc(int n_tiles) {
    static int lim = -1;
    if (lim < 0) { const char* e = getenv("EXB_GEMM_MC"); lim = e ? atoi(e) : 0; }
    if (lim <= 1 || pick_swap()) return 1;
    int best = 1;
    for (int c = 2; c <= 8 && c <= lim; ++c)
        if (n_tiles % c == 0) best = c;
    return best;
}

}  // namespace

extern "C" {

const char* exb_gemm_last_error() { return g_gemm_err.c_str(); }

// device sync; number of pipeline barrier waits of the GEMM kernels that timed out since the last call (their
// results are wrong), then reset to 0; -1 if the counter could not be read
int exb_gemm_timeouts() {
    unsigned v = 0, z = 0;
    if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(&v, g_pipeline_timeouts, sizeof(v)) != cudaSuccess ||
        cudaMemcpyToSymbol(g_pipeline_timeouts, &z, sizeof(z)) != cudaSuccess) return -1;
    return (int)v;
}

// D (+)= A[M,K](lda) * B[N,K](ldb)^T, bf16 in. K must be a multiple of 64 (pad the operands);
// lda/ldb in elements, multiples of 8. epi: see GemmEpi. splits > 1: EPI_DW only (the other epilogues store their
// tile, so the K splits would overwrite each other's partial sums).
int exb_gemm_bf16_nt(uint64_t A, long long lda, uint64_t B, long long ldb, int M, int N, int K, int mode, int relu,
                     int ones_col, uint64_t out, long long ldo, uint64_t outT, long long ldoT, uint64_t mask,
                     long long ldmask, uint64_t dlogit, uint64_t S, uint64_t emb, long long ldemb, int fm_cols, int D,
                     int splits, uint64_t stream, uint64_t dbg) {
    if (K % BK != 0 || lda % 8 != 0 || ldb % 8 != 0) { g_gemm_err = "gemm: K %% 64 / ld %% 8 violated"; return -1; }
    if (splits > 1 && mode != EPI_DW) { g_gemm_err = "gemm: splits > 1 needs EPI_DW (split-K sums are reduce-added)"; return -1; }
    if (!fm_operands_ok(mode, fm_cols, D, S)) return -1;
    CUtensorMap tmA, tmB;
    if (!make_map(&tmA, (const void*)A, M, K, lda, BM)) return -1;
    const int BN = pick_bn(M, N, K);
    if (!make_map(&tmB, (const void*)B, N, K, ldb, BN)) return -1;
    CUtensorMap tmO, tmT;
    const bool f32out = (mode == EPI_DW || mode == EPI_DX_FM);
    if (f32out) {   // fp32 [M, N] (ld ldo): 32x32 boxes = 128-byte rows
        if (!make_map_ex(&tmO, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (const void*)out, M, N, ldo, 32, 32, CU_TENSOR_MAP_SWIZZLE_128B)) return -1;
    } else {        // bf16 [M, ceil64(N)] : 64x32 boxes = 128-byte rows
        if (!make_map_ex(&tmO, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (const void*)out, M, (N + 63) / 64 * 64, ldo, 64, 32, CU_TENSOR_MAP_SWIZZLE_128B)) return -1;
    }
    tmT = tmO;
    CUtensorMap tmE = tmO;    // placeholder when the epilogue has no source tile
    if (!make_epi_src_map(&tmE, mode, fm_cols, M, N, (const void*)mask, ldmask, (const void*)emb, ldemb)) return -1;
    if (outT && !make_map_ex(&tmT, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (const void*)outT, (N + 63) / 64 * 64, M, ldoT, 32, BN, CU_TENSOR_MAP_SWIZZLE_NONE)) return -1;
    GemmEpi E;
    E.mode = mode; E.relu = relu; E.ones_col = ones_col; E.fm_cols = fm_cols; E.M = M; E.N = N; E.D = D > 0 ? D : 1; E.mn_major = 0;
    E.out = (void*)out; E.ldo = ldo; E.outT = (__nv_bfloat16*)outT; E.ldoT = ldoT;
    E.mask = (const __nv_bfloat16*)mask; E.ldmask = ldmask;
    E.dlogit = (const float*)dlogit; E.S = (const float*)S; E.emb = (const float*)emb; E.ldemb = ldemb;
    E.dbg = (unsigned long long*)dbg;
    const int nkb = K / BK;
    if (splits < 1) splits = 1;
    if (splits > nkb) splits = nkb;
    const int per = (nkb + splits - 1) / splits;
    splits = (nkb + per - 1) / per;
    dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, splits);
    E.swap = pick_swap(); E.mc = pick_mc((int)grid.y);
    if (E.swap) grid = dim3(grid.y, grid.x, grid.z);
    cudaError_t err = BN == 128 ? launch_gemm<128>(grid, (cudaStream_t)stream, tmA, tmB, tmO, tmT, tmE, E, nkb, per)
                                : launch_gemm<64>(grid, (cudaStream_t)stream, tmA, tmB, tmO, tmT, tmE, E, nkb, per);
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err != cudaSuccess) { g_gemm_err = std::string("gemm launch: ") + cudaGetErrorString(err); return -1; }
    return 0;
}

// dW-style product from batch-major operands, no transposed copies needed:
//   out[M, N] (fp32, += via TMA reduce-add) = A[K, M]^T * B[K, N],  A/B bf16 row-major with K rows
// (e.g. M = features of dZ, N = features of the layer input, K = batch). M, N: any; K % 64 == 0;
// lda/ldb multiples of 8 elements. Both operands reach the tensor core as MN-major tiles.
int exb_gemm_bf16_tn(uint64_t A, long long lda, uint64_t B, long long ldb, int M, int N, int K, uint64_t out,
                     long long ldo, int splits, uint64_t stream) {
    if (K % BK != 0 || lda % 8 != 0 || ldb % 8 != 0) { g_gemm_err = "gemm_tn: K %% 64 / ld %% 8 violated"; return -1; }
    CUtensorMap tmA, tmB, tmO, tmT, tmE;
    if (!make_map_ex(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (const void*)A, K, M, lda, 64, BK, CU_TENSOR_MAP_SWIZZLE_128B)) return -1;
    if (!make_map_ex(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (const void*)B, K, N, ldb, 64, BK, CU_TENSOR_MAP_SWIZZLE_128B)) return -1;
    if (!make_map_ex(&tmO, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (const void*)out, M, N, ldo, 32, 32, CU_TENSOR_MAP_SWIZZLE_128B)) return -1;
    tmT = tmE = tmO;
    GemmEpi E;
    memset(&E, 0, sizeof(E));
    E.mode = EPI_DW; E.ones_col = -1; E.M = M; E.N = N; E.D = 1; E.mn_major = 1;
    E.out = (void*)out; E.ldo = ldo;
    const int BN = pick_bn(M, N, K);
    const int nkb = K / BK;
    if (splits < 1) splits = 1;
    if (splits > nkb) splits = nkb;
    const int per = (nkb + splits - 1) / splits;
    splits = (nkb + per - 1) / per;
    dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, splits);
    E.swap = pick_swap(); E.mc = pick_mc((int)grid.y);
    if (E.swap) grid = dim3(grid.y, grid.x, grid.z);
    cudaError_t err = BN == 128 ? launch_gemm<128>(grid, (cudaStream_t)stream, tmA, tmB, tmO, tmT, tmE, E, nkb, per)
                                : launch_gemm<64>(grid, (cudaStream_t)stream, tmA, tmB, tmO, tmT, tmE, E, nkb, per);
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err != cudaSuccess) { g_gemm_err = std::string("gemm_tn launch: ") + cudaGetErrorString(err); return -1; }
    return 0;
}

// ---------------------------------------------------------------- GEMM chains (persistent, one launch)
struct ChainDesc {      // one GEMM of a chain (python: ops/gemm.py ChainDesc)
    int tn;             // 0: D = A[M,K] B[N,K]^T (K-major operands); 1: D[M,N] += A[K,M]^T B[K,N] (split-K, fp32 reduce-add)
    int M, N, K;
    unsigned long long A, B, out;
    long long lda, ldb, ldo;
    int mode, relu, ones_col, fm_cols, D, splits;
    unsigned long long mask; long long ldmask;
    unsigned long long dlogit, S, emb; long long ldemb;
    int dep, dep_kind;  // index of the GEMM of this chain that produces this one's A operand (-1: none); kind 1 row block, 2 K range
};
struct Chain {
    int nprob = 0, total = 0, grid = 0, mb_stride = 1;
    ChainMapsAll maps;
    ChainMeta* d_meta = nullptr;
    unsigned* d_ready = nullptr;
    int* d_err = nullptr;
    size_t smem = 0;
};

int exb_chain_desc_size() { return (int)sizeof(ChainDesc); }

void* exb_chain_create(const void* descs, int n, int sms) {
    if (n < 1 || n > CH_MAX_PROB) { g_gemm_err = "chain: 1..8 GEMMs"; return nullptr; }
    const ChainDesc* D = reinterpret_cast<const ChainDesc*>(descs);
    std::vector<ChainMaps> maps(n);
    std::vector<ChainMeta> meta(n);
    int item0 = 0;
    for (int i = 0; i < n; ++i) {
        const ChainDesc& d = D[i];
        ChainMeta& Q = meta[i];
        memset(&Q, 0, sizeof(Q));
        if (d.K % BK != 0 || d.lda % 8 != 0 || d.ldb % 8 != 0) { g_gemm_err = "chain: K % 64 / ld % 8 violated"; return nullptr; }
        if (!d.tn && !fm_operands_ok(d.mode, d.fm_cols, d.D, d.S)) return nullptr;
        GemmEpi& E = Q.E;
        E.mode = d.tn ? EPI_DW : d.mode; E.relu = d.relu; E.ones_col = d.tn ? -1 : d.ones_col; E.fm_cols = d.fm_cols;
        E.M = d.M; E.N = d.N; E.D = d.D > 0 ? d.D : 1; E.mn_major = d.tn ? 1 : 0;
        E.out = (void*)d.out; E.ldo = d.ldo; E.outT = nullptr; E.ldoT = 0;
        E.mask = (const __nv_bfloat16*)d.mask; E.ldmask = d.ldmask;
        E.dlogit = (const float*)d.dlogit; E.S = (const float*)d.S; E.emb = (const float*)d.emb; E.ldemb = d.ldemb;
        E.swap = 0; E.mc = 1; E.dbg = nullptr;
        const bool f32out = (E.mode == EPI_DW || E.mode == EPI_DX_FM);
        bool ok;
        if (d.tn) {
            ok = make_map_ex(&maps[i].tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (const void*)d.A, d.K, d.M, d.lda, 64, BK, CU_TENSOR_MAP_SWIZZLE_128B) &&
                 make_map_ex(&maps[i].tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (const void*)d.B, d.K, d.N, d.ldb, 64, BK, CU_TENSOR_MAP_SWIZZLE_128B);
        } else {
            ok = make_map(&maps[i].tmA, (const void*)d.A, d.M, d.K, d.lda, BM) && make_map(&maps[i].tmB, (const void*)d.B, d.N, d.K, d.ldb, CH_BN);
        }
        if (ok) {
            if (f32out) ok = make_map_ex(&maps[i].tmO, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (const void*)d.out, d.M, d.N, d.ldo, 32, 32, CU_TENSOR_MAP_SWIZZLE_128B);
            else ok = make_map_ex(&maps[i].tmO, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (const void*)d.out, d.M, (d.N + 63) / 64 * 64, d.ldo, 64, 32, CU_TENSOR_MAP_SWIZZLE_128B);
        }
        if (ok && !d.tn)
            ok = make_epi_src_map(&maps[i].tmE, E.mode, d.fm_cols, d.M, d.N, (const void*)d.mask, d.ldmask, (const void*)d.emb, d.ldemb);
        if (!ok) return nullptr;
        Q.nkb = d.K / BK;
        int splits = d.tn ? std::max(1, d.splits) : 1;
        if (splits > Q.nkb) splits = Q.nkb;
        Q.per = (Q.nkb + splits - 1) / splits;
        Q.splits = (Q.nkb + Q.per - 1) / Q.per;
        Q.m_tiles = (d.M + BM - 1) / BM; Q.n_tiles = (d.N + CH_BN - 1) / CH_BN;
        Q.item0 = item0; Q.items = Q.m_tiles * Q.n_tiles * Q.splits;
        item0 += Q.items;
        Q.dep = d.dep; Q.dep_kind = d.dep >= 0 ? d.dep_kind : 0; Q.dep_need = 0; Q.signal = 0;
        if (Q.dep_kind) {
            if (d.dep >= i) { g_gemm_err = "chain: a GEMM may only depend on an earlier one"; return nullptr; }
            // the row blocks a tile waits on must be row blocks its producer writes: the counters of the next GEMM
            // (or past the table) would otherwise be read as this producer's
            const int rows_read = Q.dep_kind == 1 ? Q.m_tiles : Q.dep_kind == 2 ? (d.K + BM - 1) / BM : -1;
            if (rows_read < 0 || rows_read > meta[d.dep].m_tiles) {
                g_gemm_err = "chain: a dependency reads row blocks its producer does not write";
                return nullptr;
            }
            meta[d.dep].signal = 1;
            Q.dep_need = (NUM_CONSUMER_WARPS / 4) * meta[d.dep].n_tiles;   // each consumer warpgroup signs off every tile of the row block
        }
    }
    int mb_stride = 1;     // ready counters per GEMM: its row blocks (the largest count of the chain)
    for (int i = 0; i < n; ++i) mb_stride = std::max(mb_stride, meta[i].m_tiles);
    const size_t ready_bytes = ((size_t)n * mb_stride + 1) * sizeof(unsigned);
    Chain* c = new Chain();
    c->nprob = n; c->total = item0; c->mb_stride = mb_stride;
    c->smem = CH_STAGES * (A_BYTES + CH_B_BYTES) + 4 * 8192 + (2 * CH_STAGES + 4) * 8 + CH_MAX_PROB * sizeof(ChainMeta) + 1024;
    cudaFuncSetAttribute(exb_gemm_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem);
    cudaFuncSetAttribute(exb_gemm_chain_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    // two CTAs per SM by construction: 2 x (smem + 1 KB reserved) <= 227 KB, and __launch_bounds__(288, 2) keeps
    // 2 x 288 threads within the 64 K registers of an SM
    // (the occupancy API answers 1 here when it is asked before the carve-out is configured)
    int occ = (2 * (c->smem + 1024) <= 232448) ? 2 : 1;
    if (const char* ev = getenv("EXB_CHAIN_CTAS_PER_SM")) occ = std::max(1, std::min(2, atoi(ev)));
    // dependencies are spin-waits: every CTA has to be resident
    c->grid = std::min(c->total, (sms > 0 ? sms : 132) * occ);
    memset(&c->maps, 0, sizeof(c->maps));
    for (int i = 0; i < n; ++i) c->maps.m[i] = maps[i];
    if (cudaMalloc(&c->d_meta, n * sizeof(ChainMeta)) != cudaSuccess ||
        cudaMalloc(&c->d_ready, ready_bytes) != cudaSuccess || cudaMalloc(&c->d_err, 4) != cudaSuccess) {
        g_gemm_err = "chain: cudaMalloc failed"; delete c; return nullptr;
    }
    cudaMemcpy(c->d_meta, meta.data(), n * sizeof(ChainMeta), cudaMemcpyHostToDevice);
    cudaMemset(c->d_ready, 0, ready_bytes);
    cudaMemset(c->d_err, 0, 4);
    return c;
}
void exb_chain_destroy(void* h) {
    Chain* c = (Chain*)h;
    cudaFree(c->d_meta); cudaFree(c->d_ready); cudaFree(c->d_err);
    delete c;
}
int exb_chain_launch(void* h, uint64_t stream) {
    Chain* c = (Chain*)h;
    cudaError_t err = exb::launch_pdl(exb_gemm_chain_kernel, dim3(c->grid), dim3(NUM_THREADS), c->smem, (cudaStream_t)stream,
                              c->maps, (const ChainMeta*)c->d_meta, c->nprob, c->total, c->d_ready, c->mb_stride, c->d_err);
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err != cudaSuccess) { g_gemm_err = std::string("chain launch: ") + cudaGetErrorString(err); return -1; }
    return 0;
}
// device sync; returns the error word (0 ok, 100 + p: GEMM p timed out waiting for its producer)
int exb_chain_status(void* h) {
    Chain* c = (Chain*)h;
    int v = 0;
    cudaDeviceSynchronize();
    cudaMemcpy(&v, c->d_err, 4, cudaMemcpyDeviceToHost);
    return v;
}
int exb_chain_info(void* h, int* out) { Chain* c = (Chain*)h; out[0] = c->total; out[1] = c->grid; out[2] = (int)c->smem; return 0; }

}  // extern "C"
