// sparse_kernels.cuh -- the two fused sparse hot paths of the engine (sm_90a).
//
//  exb_pull_kernel        K1+K2+K3 of SURVEY 2.5: bucketize by owner (id % S), one-sided
//                         peer loads of the rows over NVLink (array: direct address, hash:
//                         probe in the owner's key slab), scatter into request order.
//                         Missing hash rows are answered with the Philox initial value.
//  exb_push_update_kernel K4a+K4b: persistent kernel, phases separated by grid barriers:
//     P1 dispatch   (id, grad) -> owner inbox with P2P vector stores; local ids skip the
//                   inbox and go straight to the combine map
//     B1            publish counts, cross-GPU flag barrier (release/acquire .sys)
//     P3 combine    owner folds inbox entries into a per-step open-addressing map
//                   (atomicCAS on key, red.global.add.v4.f32 on the accumulator row)
//     B2
//     P5 apply      one lane group per unique row: (hash: find-or-insert, Philox init of
//                   new rows) -> optimizer functor -> write back, reset map entry
//     B3            cross-GPU "update done" barrier (next pull may read any shard)
//
// Both kernels are latency-bound gather/scatter machines, so: (1) every descriptor the
// inner loops touch (table structs, plan index arrays) is staged in shared memory once
// per CTA, (2) each lane group issues a batch of independent 128-bit loads before it
// consumes any of them (memory-level parallelism instead of occupancy), (3) barriers
// poll with relaxed loads.
//
// Reference semantics preserved: gradients of duplicate ids are SUMMED, counts are
// summed (MpscGradientReducer.h:30-53); rows are materialised at their first update.
#pragma once
#include "exb_common.cuh"
#include "pdl.cuh"
#include "bulk_rows.cuh"

namespace exb {

#define EXB_MAX_SEG 1024  // max W*PT segments of the combine phase
#define EXB_MAX_PT 128

struct SmemView {
    TableDev* tab;                 // [PT] copies of the plan's table descriptors
    unsigned long long* key_off;   // [PT]
    unsigned long long* grad_off;  // [PT]
    unsigned long long* map_off;   // [PT]
    unsigned long long* acc_off;   // [PT]
    unsigned long long* ulist_off; // [PT]
    unsigned* cap;                 // [PT]
    unsigned* map_mask;            // [PT]
    int* task_prefix;              // [F+1]
    int* feat_pt;                  // [F]
    int* feat_off;                 // [F]
    int* feat_col;                 // [F]
    int* feat_off2;                // [F]
    int* feat_split;               // [F]
    int* seg_prefix;               // [EXB_MAX_SEG+1] (push kernel only)
};

__host__ __device__ inline size_t exb_smem_bytes(int PT, int F, bool push) {
    size_t b = (size_t)PT * sizeof(TableDev) + (size_t)PT * 8 * 5 + (size_t)PT * 4 * 2 +
               (size_t)(F + 1) * 4 + (size_t)F * 4 * 5;
    if (push) b += (EXB_MAX_SEG + 1) * 4;
    return (b + 127) & ~(size_t)127;
}
// total dynamic shared memory of a 256-thread CTA: staged descriptors | per-warp row buffers |
// (push: per-warp metadata)
__host__ __device__ inline size_t exb_smem_total(int PT, int F, bool push) {
    size_t b = exb_smem_bytes(PT, F, push);
    b += 8 * (size_t)(push ? EXB_APPLY_WARP_BUF : EXB_PULL_WARP_BUF);
    if (push) b += 8 * sizeof(WarpMeta);
    return b;
}

__device__ __forceinline__ SmemView stage_plan(const TableDev* __restrict__ tables, const PlanDev& P,
                                               unsigned char* smem) {
    SmemView S;
    const int PT = P.PT, F = P.F;
    unsigned char* p = smem;
    S.tab = (TableDev*)p; p += (size_t)PT * sizeof(TableDev);
    S.key_off = (unsigned long long*)p; p += PT * 8;
    S.grad_off = (unsigned long long*)p; p += PT * 8;
    S.map_off = (unsigned long long*)p; p += PT * 8;
    S.acc_off = (unsigned long long*)p; p += PT * 8;
    S.ulist_off = (unsigned long long*)p; p += PT * 8;
    S.cap = (unsigned*)p; p += PT * 4;
    S.map_mask = (unsigned*)p; p += PT * 4;
    S.task_prefix = (int*)p; p += (F + 1) * 4;
    S.feat_pt = (int*)p; p += F * 4;
    S.feat_off = (int*)p; p += F * 4;
    S.feat_col = (int*)p; p += F * 4;
    S.feat_off2 = (int*)p; p += F * 4;
    S.feat_split = (int*)p; p += F * 4;
    S.seg_prefix = (int*)p;
    constexpr int TW = sizeof(TableDev) / 4;
    for (int i = threadIdx.x; i < PT * TW; i += blockDim.x) {
        int pt = i / TW, w = i - pt * TW;
        ((unsigned*)S.tab)[i] = ((const unsigned*)(tables + P.pt_table[pt]))[w];
    }
    for (int i = threadIdx.x; i < PT; i += blockDim.x) {
        S.key_off[i] = P.pt_key_off[i]; S.grad_off[i] = P.pt_grad_off[i]; S.map_off[i] = P.pt_map_off[i];
        S.acc_off[i] = P.pt_acc_off[i]; S.ulist_off[i] = P.pt_ulist_off[i];
        S.cap[i] = P.pt_cap[i]; S.map_mask[i] = P.pt_map_mask[i];
    }
    for (int i = threadIdx.x; i <= F; i += blockDim.x) S.task_prefix[i] = P.task_prefix[i];
    for (int i = threadIdx.x; i < F; i += blockDim.x) {
        S.feat_pt[i] = P.feat_pt[i]; S.feat_off[i] = P.feat_off[i]; S.feat_col[i] = P.feat_col[i];
        S.feat_off2[i] = P.feat_off2[i]; S.feat_split[i] = P.feat_split[i];
    }
    __syncthreads();
    return S;
}

__device__ __forceinline__ int find_segment(const int* prefix, int n, int task) {
    int lo = 0, hi = n;  // prefix[lo] <= task < prefix[hi]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (prefix[mid] <= task) lo = mid; else hi = mid;
    }
    return lo;
}

// initializer values of elements c..c+3 of row `id` (cold path: kept out of line so the hot
// gather loops do not carry Philox in registers)
__device__ __noinline__ float4 init_block_masked(const InitParams* I, unsigned long long id, int c,
                                                 int dim) {
    float t[4];
    InitGen<float>::block4(*I, id, (uint32_t)(c >> 2), t);
    float4 v;
    v.x = (c + 0 < dim) ? t[0] : 0.f;
    v.y = (c + 1 < dim) ? t[1] : 0.f;
    v.z = (c + 2 < dim) ? t[2] : 0.f;
    v.w = (c + 3 < dim) ? t[3] : 0.f;
    return v;
}
__device__ __noinline__ float init_scalar(const InitParams* I, unsigned long long id, int c) {
    float t[4];
    InitGen<float>::block4(*I, id, (uint32_t)(c >> 2), t);
    return t[c & 3];
}

// ------------------------------------------------------------------ pull
// flag: 0 -> zeros (invalid id / padding row), 1 -> load from src, 2 -> initializer value
template <int LPR>
__device__ __forceinline__ void pull_rows(const TableDev& T, const float* src, unsigned long long id,
                                          int flag, int b0, int n_rows, float* __restrict__ out,
                                          int io_stride, int off, int lane) {
    constexpr int RP = 32 / LPR;
    constexpr int U = LPR >= 8 ? 8 : LPR;  // rows in flight per lane group
    const int gl = lane % LPR;
    const int wstride = T.wstride, dim = T.dim;
    if (T.vec4) {
        // warp-uniform trip count (the body shuffles): one iteration unless dim > 128
        for (int cb = 0; cb < wstride; cb += LPR * 4) {
            const int c0 = cb + gl * 4;
            const bool cin = c0 < wstride;
#pragma unroll 1
            for (int p0 = 0; p0 < LPR; p0 += U) {
                float4 v[U];
                int fl[U];
                unsigned long long idr[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    int r = (p0 + u) * RP + lane / LPR;
                    const float* s = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src, r);
                    idr[u] = __shfl_sync(0xffffffffu, id, r);
                    fl[u] = __shfl_sync(0xffffffffu, flag, r);
                    v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (fl[u] == 1 && cin) v[u] = ld_stream_v4(s + c0);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    int b = b0 + (p0 + u) * RP + lane / LPR;
                    if (b >= n_rows || !cin) continue;
                    if (fl[u] == 2) v[u] = init_block_masked(&T.init, idr[u], c0, dim);
                    *reinterpret_cast<float4*>(out + (size_t)b * io_stride + off + c0) = v[u];
                }
            }
        }
    } else {  // dim < 4: one lane per row
        int b = b0 + lane;
        if (b < n_rows) {
            for (int c = 0; c < dim; ++c) {
                float v = 0.f;
                if (flag == 1) v = src[c];
                else if (flag == 2) v = init_scalar(&T.init, id, c);
                out[(size_t)b * io_stride + off + c] = v;
            }
        }
    }
}

// every row shape the single-pass form does not cover (rows wider than the warp buffer / 32, dim < 4, multi-pass
// split rows). Out of line on purpose: these paths hold 8 float4 of rows in registers per lane group and would
// otherwise set the register budget (and the spills) of the whole kernel.
__device__ __noinline__ void pull_rows_slow(const TableDev& T, const float* src, unsigned long long id, int flag,
                                            int b0, int n_rows, float* __restrict__ out, int io_stride, int off,
                                            int off2, int split, int lane, unsigned char* wbuf, int use_bulk) {
    if (split < T.dim) {       // split-row feature (plan creation guarantees vec4 rows that fit the buffer)
        pull_rows_split(T, src, id, flag, b0, n_rows, out, io_stride, off, off2, split, lane, wbuf);
        return;
    }
    if (use_bulk && T.vec4 && T.wstride * 4 <= EXB_PULL_WARP_BUF) {
        pull_rows_bulk(T, src, id, flag, b0, n_rows, out, io_stride, off, lane, wbuf);
        return;
    }
    switch (T.lpr) {
        case 1: pull_rows<1>(T, src, id, flag, b0, n_rows, out, io_stride, off, lane); break;
        case 2: pull_rows<2>(T, src, id, flag, b0, n_rows, out, io_stride, off, lane); break;
        case 4: pull_rows<4>(T, src, id, flag, b0, n_rows, out, io_stride, off, lane); break;
        case 8: pull_rows<8>(T, src, id, flag, b0, n_rows, out, io_stride, off, lane); break;
        case 16: pull_rows<16>(T, src, id, flag, b0, n_rows, out, io_stride, off, lane); break;
        default: pull_rows<32>(T, src, id, flag, b0, n_rows, out, io_stride, off, lane); break;
    }
}

// where does the row of lookup (f, b) live? flag: 0 invalid id / padding, 1 row at *src, 2 initializer value
__device__ __forceinline__ int pull_resolve(const TableDev& T, const PlanDev& P, unsigned long long id,
                                            const float** srcp) {
    const int W = P.W;
    const float* src = nullptr;
    int flag = 0;
    {
        if (!T.is_hash) {
            if (id < T.vocab) {
                int o = owner_of(T, id, W);
                src = T.w[o] + local_row_of(T, id) * (unsigned long long)T.wstride;
                flag = 1;
            }
        } else if ((id >> 63) == 0) {
            int o = owner_of(T, id, W);
            const unsigned long long* keys = T.keys[o];
            unsigned long long mask = T.rows - 1, h = exb_hash64(id) & mask;
            flag = 2;
            for (unsigned long long probe = 0; probe <= mask; ++probe) {
                unsigned long long k = keys[h];
                if (k == id) {
                    src = T.w[o] + h * (unsigned long long)T.wstride;
                    flag = 1;
                    break;
                }
                if (k == EXB_EMPTY_KEY) break;
                h = (h + 1) & mask;
            }
        }
    }
    *srcp = src;
    return flag;
}

// one warp task of the pull: the 32 lookups (f, b0 .. b0+31)
__device__ __forceinline__ void pull_one_task(const SmemView& S, const PlanDev& P, const long long* __restrict__ ids,
                                              float* __restrict__ out, int n_rows, int task, int lane,
                                              unsigned char* wbuf) {
    const int W = P.W;
    const int f = find_segment(S.task_prefix, P.F, task);
    const int b0 = (task - S.task_prefix[f]) * 32;
    if (b0 >= n_rows) return;
    const TableDev& T = S.tab[S.feat_pt[f]];
    const int b = b0 + lane;
    unsigned long long id = 0;
    const float* src = nullptr;
    int flag = 0;
    if (b < n_rows) {
        id = (unsigned long long)__ldg(ids + (size_t)b * P.ncols + S.feat_col[f]);
        if (!T.is_hash) {
            if (id < T.vocab) {
                int o = owner_of(T, id, W);
                src = T.w[o] + local_row_of(T, id) * (unsigned long long)T.wstride;
                flag = 1;
            }
        } else if ((id >> 63) == 0) {
            int o = owner_of(T, id, W);
            const unsigned long long* keys = T.keys[o];
            unsigned long long mask = T.rows - 1, h = exb_hash64(id) & mask;
            flag = 2;
            for (unsigned long long probe = 0; probe <= mask; ++probe) {
                unsigned long long k = keys[h];
                if (k == id) {
                    src = T.w[o] + h * (unsigned long long)T.wstride;
                    flag = 1;
                    break;
                }
                if (k == EXB_EMPTY_KEY) break;
                h = (h + 1) & mask;
            }
        }
    }
    const int off = S.feat_off[f];
    int bulk;
    if (P.use_bulk && pull_fast_geometry(T, S.feat_split[f], &bulk)) {     // one pass: the benchmark's row shapes
        pull_rows_fast(T, src, id, flag, b0, n_rows, out, P.io_stride, off, S.feat_off2[f], S.feat_split[f], bulk, lane,
                       wbuf, [] {});
        return;
    }
    pull_rows_slow(T, src, id, flag, b0, n_rows, out, P.io_stride, off, S.feat_off2[f], S.feat_split[f], lane, wbuf,
                   P.use_bulk);
}

__global__ void __launch_bounds__(256, 2)
exb_pull_kernel(const TableDev* __restrict__ tables, PlanDev P, const long long* __restrict__ ids,
                float* __restrict__ out, int n_rows) {
    extern __shared__ __align__(16) unsigned char exb_smem[];
    pdl_trigger();
    const SmemView S = stage_plan(tables, P, exb_smem);   // descriptors are written by the host only
    pdl_wait();
    ctx_check(P);
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    if (P.W > 1) peer_wait(P);   // peers' last update is complete (deferred half of the push "done" barrier)
    const int wic = threadIdx.x >> 5;
    unsigned char* stage_end = exb_smem + exb_smem_bytes(P.PT, P.F, false);
    unsigned char* wbuf = stage_end + (size_t)wic * EXB_PULL_WARP_BUF;
    for (int task = warp; task < P.num_tasks; task += nwarps)
        pull_one_task(S, P, ids, out, n_rows, task, lane, wbuf);
    if (threadIdx.x == 0 && blockIdx.x == 0)
        atomicAdd(&P.stats[0], (unsigned long long)n_rows * (unsigned long long)P.F);
}

// ------------------------------------------------------------ push + update
// Per-table counters live on their own 128-byte line (EXB_CTR_STRIDE words apart): every
// table's appends would otherwise serialise in ONE L2 slice (measured: 19 us per warp task).
#define EXB_CTR_STRIDE 32

// Warp-collective find-or-insert of `key` (lanes with active == false only take part in
// the vote) into plan-table pt's combine map; returns the map position. New keys are
// appended to the table's unique list with ONE counter atomic per warp.
__device__ __forceinline__ unsigned cmap_insert_warp(const PlanDev& P, const SmemView& S, int pt,
                                                     unsigned long long key, bool active, int lane) {
    const unsigned mask = S.map_mask[pt];
    unsigned long long* keys = P.cmap_keys + S.map_off[pt];
    unsigned h = (unsigned)(exb_hash64(key) >> 20) & mask;
    bool won = false, done = !active;
    for (unsigned probe = 0; probe <= mask && !done; ++probe) {
        unsigned long long prev = atomicCAS(&keys[h], EXB_EMPTY_KEY, key);
        if (prev == EXB_EMPTY_KEY) { won = true; done = true; }
        else if (prev == key) done = true;
        else h = (h + 1) & mask;
    }
    if (!done) { set_error(P.status, EXB_ERR_CMAP_FULL); h = 0xFFFFFFFFu; }
    const unsigned wmask = __ballot_sync(0xffffffffu, won);
    if (wmask) {
        const int leader = __ffs(wmask) - 1;
        unsigned base = 0;
        if (lane == leader) base = atomicAdd(&P.ucount[pt * EXB_CTR_STRIDE], (unsigned)__popc(wmask));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (won) {
            const unsigned long long up = S.ulist_off[pt] + base + (unsigned)__popc(wmask & ((1u << lane) - 1u));
            P.ulist[up] = h;
            P.ukeys[up] = key;     // the apply phase reads key and slot side by side (one dependent load less)
        }
    }
    return active ? h : 0xFFFFFFFFu;
}

// Move / accumulate the 32 rows of a warp task.
// mode: 0 skip, 1 accumulate row into dst (red.add), 2 store row to dst (peer inbox)
template <int LPR>
__device__ __forceinline__ void move_rows(const TableDev& T, const float* src, float* dst, int mode,
                                          int lane) {
    constexpr int RP = 32 / LPR;
    constexpr int U = LPR >= 8 ? 8 : LPR;
    const int gl = lane % LPR;
    const int wstride = T.wstride, dim = T.dim;
    if (T.vec4) {
        for (int cb = 0; cb < wstride; cb += LPR * 4) {  // warp-uniform trip count
            const int c0 = cb + gl * 4;
            const bool cin = c0 < wstride;
#pragma unroll 1
            for (int p0 = 0; p0 < LPR; p0 += U) {
                float4 v[U];
                float* d[U];
                int m[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    int r = (p0 + u) * RP + lane / LPR;
                    const float* s = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src, r);
                    d[u] = (float*)__shfl_sync(0xffffffffu, (unsigned long long)dst, r);
                    m[u] = __shfl_sync(0xffffffffu, mode, r);
                    v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (!cin) m[u] = 0;
                    if (m[u]) v[u] = ld_stream_v4(s + c0);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    if (m[u] == 1) red_add_v4(d[u] + c0, v[u]);
                    else if (m[u] == 2) *reinterpret_cast<float4*>(d[u] + c0) = v[u];
                }
            }
        }
    } else {
        if (mode) {
            for (int c = 0; c < dim; ++c) {
                float v = src[c];
                if (mode == 1) red_add_f32(dst + c, v);
                else dst[c] = v;
            }
        }
    }
}

__device__ __noinline__ void move_rows_dispatch(const TableDev& T, const float* src, float* dst,
                                               int mode, int lane) {
    switch (T.lpr) {
        case 1: move_rows<1>(T, src, dst, mode, lane); break;
        case 2: move_rows<2>(T, src, dst, mode, lane); break;
        case 4: move_rows<4>(T, src, dst, mode, lane); break;
        case 8: move_rows<8>(T, src, dst, mode, lane); break;
        case 16: move_rows<16>(T, src, dst, mode, lane); break;
        default: move_rows<32>(T, src, dst, mode, lane); break;
    }
}

// gradient rows of a split-row feature (see pull_rows_split) are gathered from two places of the gradient row
// and added into the accumulator row (mode 1) or stored into an inbox row (mode 2): columns [0, split) from src,
// [split, dim) from src2, pad columns 0
template <int LPR>
__device__ __forceinline__ void accum_rows_split_t(const TableDev& T, const float* src, const float* src2, int split,
                                                   float* dst, int mode, int lane) {
    const int wstride = T.wstride, dim = T.dim;
    constexpr int RP = 32 / LPR;
    constexpr int U = LPR >= 8 ? 8 : LPR;              // rows in flight per lane group
    const int gl = lane % LPR, sub = lane / LPR;
    for (int cb = 0; cb < wstride; cb += LPR * 4) {    // one iteration unless the row is wider than 128 floats
        const int c = cb + gl * 4;
        const bool cin = c < wstride;
#pragma unroll 1
        for (int p0 = 0; p0 < LPR; p0 += U) {
            float4 v[U];
            float* d[U];
            int m[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int r = (p0 + u) * RP + sub;
                const float* s = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src, r);
                const float* s2 = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src2, r);
                d[u] = (float*)__shfl_sync(0xffffffffu, (unsigned long long)dst, r);
                m[u] = __shfl_sync(0xffffffffu, mode, r);
                if (!cin) m[u] = 0;
                v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (m[u]) {
                    if (c + 4 <= split) v[u] = ld_stream_v4(s + c);
                    else {
                        float t[4];
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int col = c + e;
                            t[e] = col < split ? s[col] : (col < dim ? s2[col - split] : 0.f);
                        }
                        v[u] = make_float4(t[0], t[1], t[2], t[3]);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (m[u] == 1) red_add_v4(d[u] + c, v[u]);                                   // accumulate
                else if (m[u] == 2) *reinterpret_cast<float4*>(d[u] + c) = v[u];              // store (peer inbox)
            }
        }
    }
}
__device__ __noinline__ void accum_rows_split(const TableDev& T, const float* src, const float* src2, int split,
                                              float* dst, int mode, int lane) {
    switch (T.lpr) {
        case 1: accum_rows_split_t<1>(T, src, src2, split, dst, mode, lane); break;
        case 2: accum_rows_split_t<2>(T, src, src2, split, dst, mode, lane); break;
        case 4: accum_rows_split_t<4>(T, src, src2, split, dst, mode, lane); break;
        case 8: accum_rows_split_t<8>(T, src, src2, split, dst, mode, lane); break;
        case 16: accum_rows_split_t<16>(T, src, src2, split, dst, mode, lane); break;
        default: accum_rows_split_t<32>(T, src, src2, split, dst, mode, lane); break;
    }
}

// Dense-gradient all-reduce riding on the push kernel (P.ar_n > 0): the two-shot all-reduce of exb_ar_fused_kernel
// (dense_kernels.cu) without a launch or cross-GPU barriers of its own. Two calls by every thread of the grid:
//   dense_reduce_gather   after the cross-GPU "counts published" barrier (every peer has entered its push kernel, so
//                         its dense gradients are final): this rank sums its 1/W chunk of the flat gradient over every
//                         rank's buffer (peer loads, their latency hides under the combine phase) into its own buffer;
//   dense_reduce_scatter  after the next grid barrier: the summed chunk goes to every peer's buffer (peer stores, in
//                         flight under the apply phase; the kernel's last barrier releases them at system scope).
// Chunk r of a peer's buffer is read and then written by rank r only, so the in-place update needs no extra ordering;
// the sums are bit-identical on every rank. The caller's last barrier must WAIT for the peers (peer_barrier(P, true)):
// the dense optimizer runs next. (One call doing both cost 8-10 us of grid-barrier time at 8 GPUs: the barrier's
// fence waits for the NVLink stores in flight.)
__device__ __forceinline__ void dense_reduce_span(const PlanDev& P, long long& lo, long long& hi) {
    const long long n = (long long)P.ar_n;
    const long long per = ((n + P.W - 1) / P.W + 3) & ~3ll;
    lo = per * P.rank;
    hi = min(n, lo + per);
}
__device__ __forceinline__ void dense_reduce_gather(const PlanDev& P) {
    const int W = P.W;
    long long lo, hi;
    dense_reduce_span(P, lo, hi);
    const long long stride = (long long)gridDim.x * blockDim.x * 4;
    for (long long i = lo + (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4; i < hi; i += stride) {
        float4 v[EXB_MAX_PEERS];
#pragma unroll
        for (int r = 0; r < EXB_MAX_PEERS; ++r)
            if (r < W) v[r] = __ldcg(reinterpret_cast<const float4*>(P.ar_buf[r] + i));
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int r = 0; r < EXB_MAX_PEERS; ++r)
            if (r < W) { s.x += v[r].x; s.y += v[r].y; s.z += v[r].z; s.w += v[r].w; }
        __stcg(reinterpret_cast<float4*>(P.ar_buf[P.rank] + i), s);
    }
}
__device__ __forceinline__ void dense_reduce_scatter(const PlanDev& P) {
    const int W = P.W, rank = P.rank;
    long long lo, hi;
    dense_reduce_span(P, lo, hi);
    const long long stride = (long long)gridDim.x * blockDim.x * 4;
    for (long long i = lo + (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4; i < hi; i += stride) {
        const float4 s = __ldcg(reinterpret_cast<const float4*>(P.ar_buf[rank] + i));
#pragma unroll
        for (int r = 0; r < EXB_MAX_PEERS; ++r)
            if (r < W && r != rank) __stcg(reinterpret_cast<float4*>(P.ar_buf[r] + i), s);
    }
}

// non-bulk optimizer path (rows that do not fit the warp buffer, dim < 4): out of line, see pull_rows_slow
template <int LPR>
__device__ __forceinline__ void apply_rows(const TableDev& T, const PlanDev& P, float* accbase,
                                           unsigned long long key, unsigned long long row, unsigned h,
                                           unsigned cnt, int flag, int lane);
__device__ __noinline__ void apply_rows_slow(const TableDev& T, const PlanDev& P, float* accbase,
                                             unsigned long long key, unsigned long long row, unsigned h,
                                             unsigned cnt, int flag, int lane);

// A unique id whose hash-shard insert failed (EXB_ERR_HASH_FULL) is skipped by the apply paths, so its summed
// gradient would stay in accumulator row h and be added to whichever id the next batch maps to h (the same id
// retried after a rehash: applied twice). One lane clears the row; cold path, out of line.
__device__ __noinline__ void clear_acc_row(float* arow, int wstride) {
    for (int c = 0; c < wstride; ++c) arow[c] = 0.f;
}

// block-wide exclusive prefix of ceil(cnt/32) over n (<= EXB_MAX_SEG) segments -> s_prefix[0..n]
__device__ __forceinline__ void block_task_prefix(const unsigned* cnt, int n, int* s_prefix,
                                                  int stride = 1) {
    __syncthreads();
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        const int chunk = (n + 31) / 32;
        int beg = lane * chunk, end = min(n, beg + chunk);
        int sum = 0;
        for (int i = beg; i < end; ++i)
            sum += (int)((__ldcg(&cnt[(size_t)i * stride]) + 31u) >> 5);
        int incl = sum;
        for (int d = 1; d < 32; d <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        int run = incl - sum;
        for (int i = beg; i < end; ++i) {
            s_prefix[i] = run;
            run += (int)((__ldcg(&cnt[(size_t)i * stride]) + 31u) >> 5);
        }
        if (lane == 31) s_prefix[n] = incl;
    }
    __syncthreads();
}

// ---- work split of the apply phase ----------------------------------------------------
// A warp task is `chunk` unique rows of one table, gathered in ONE pass through the warp's row
// buffer (weights + state + accumulated gradient). The chunk is chosen per step from the actual
// unique counts: the phase is split into the smallest number of rounds that fits the buffers and
// every task gets the same number of row BYTES, instead of a full round of maximal tasks plus a
// straggler round (measured before: warps finished after 15 us on average, the slowest after
// 43 us, because 2589 13-row tasks were dealt to 2368 warps).
__device__ __forceinline__ unsigned apply_need(const TableDev& T) {    // weights + accumulated gradient + state
    return (2u * (unsigned)T.wstride + (unsigned)T.sstride) * 4u;
}
__device__ __forceinline__ bool apply_is_bulk(const TableDev& T, int use_bulk) {
    return use_bulk && T.vec4 && apply_need(T) <= EXB_APPLY_WARP_BUF;
}
__device__ __forceinline__ int apply_max_rows(const TableDev& T, int use_bulk) {
    if (!apply_is_bulk(T, use_bulk)) return 32;
    return min(32, (int)(EXB_APPLY_WARP_BUF / apply_need(T)));
}
// s_prefix[0..n]: task prefix; s_chunk[i]: rows per task of table i; s_cnt[i]: unique rows of table i
__device__ __forceinline__ void block_apply_prefix(const unsigned* cnt, int n, int* s_prefix, int* s_chunk, int* s_cnt,
                                                   int stride, const TableDev* tab, int use_bulk) {
    __syncthreads();
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        const int per = (n + 31) / 32;
        const int beg = lane * per, end = min(n, beg + per);
        unsigned long long bytes = 0;
        for (int i = beg; i < end; ++i) {
            const unsigned c = __ldcg(&cnt[(size_t)i * stride]);
            s_cnt[i] = (int)c;
            bytes += (unsigned long long)c * apply_need(tab[i]);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
        // rounds the phase needs when every task fills a warp buffer; then equal tasks over exactly that many rounds
        const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
        const unsigned long long rounds = max(1ull, (bytes + nw * EXB_APPLY_WARP_BUF - 1) / (nw * EXB_APPLY_WARP_BUF));
        const unsigned budget = (unsigned)((bytes + nw * rounds - 1) / (nw * rounds));   // row bytes per task
        int sum = 0;
        for (int i = beg; i < end; ++i) {
            const int c = max(1, min(apply_max_rows(tab[i], use_bulk), (int)(budget / apply_need(tab[i])) + 1));
            s_chunk[i] = c;
            sum += (s_cnt[i] + c - 1) / c;
        }
        int incl = sum;
        for (int d = 1; d < 32; d <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        int run = incl - sum;
        for (int i = beg; i < end; ++i) {
            s_prefix[i] = run;
            run += (s_cnt[i] + s_chunk[i] - 1) / s_chunk[i];
        }
        if (lane == 31) s_prefix[n] = incl;
    }
    __syncthreads();
}

template <int LPR>
__device__ __forceinline__ void apply_rows(const TableDev& T, const PlanDev& P, float* accbase,
                                           unsigned long long key, unsigned long long row, unsigned h,
                                           unsigned cnt, int flag /*0 skip,1 existing,2 new*/,
                                           int lane) {
    constexpr int RP = 32 / LPR;
    constexpr int U = LPR >= 2 ? 2 : LPR;
    const int gl = lane % LPR;
    const int wstride = T.wstride, dim = T.dim, nslots = T.nslots, nsc = T.nscalars;
    float* wloc = T.w[P.rank];
    const OptParams opt = T.opt;
    const float s0i = opt_slot_init<float>(opt, 0), s1i = opt_slot_init<float>(opt, 1);
    if (T.vec4) {
#pragma unroll 1
        for (int p0 = 0; p0 < LPR; p0 += U) {
            float4 g4[U], w4[U], a4[U], b4[U];
            float scv[U][2];
            int fl[U];
            unsigned long long rowr[U], keyr[U];
            unsigned hr[U], cr[U];
            // ---- issue every load of the batch
#pragma unroll
            for (int u = 0; u < U; ++u) {
                int r = (p0 + u) * RP + lane / LPR;
                keyr[u] = __shfl_sync(0xffffffffu, key, r);
                rowr[u] = __shfl_sync(0xffffffffu, row, r);
                hr[u] = __shfl_sync(0xffffffffu, h, r);
                cr[u] = __shfl_sync(0xffffffffu, cnt, r);
                fl[u] = __shfl_sync(0xffffffffu, flag, r);
                const int c = gl * 4;
                g4[u] = w4[u] = a4[u] = b4[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                scv[u][0] = scv[u][1] = 0.f;
                if (fl[u] && c < wstride) {
                    float* arow = accbase + (unsigned long long)hr[u] * wstride;
                    g4[u] = *reinterpret_cast<float4*>(arow + c);
                    if (fl[u] == 1) {
                        const float* wrow = wloc + rowr[u] * (unsigned long long)wstride;
                        const float* srow = T.state + rowr[u] * (unsigned long long)T.sstride;
                        w4[u] = *reinterpret_cast<const float4*>(wrow + c);
                        if (nslots > 0) a4[u] = *reinterpret_cast<const float4*>(srow + c);
                        if (nslots > 1) b4[u] = *reinterpret_cast<const float4*>(srow + wstride + c);
                        for (int i = 0; i < nsc; ++i) scv[u][i] = srow[(size_t)nslots * wstride + i];
                    }
                }
            }
            // ---- compute + write back
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (!fl[u]) continue;
                float* wrow = wloc + rowr[u] * (unsigned long long)wstride;
                float* srow = T.state + rowr[u] * (unsigned long long)T.sstride;
                float* arow = accbase + (unsigned long long)hr[u] * wstride;
                float sc[2] = {scv[u][0], scv[u][1]}, nsc_v[2];
                if (fl[u] == 2)
                    for (int i = 0; i < nsc; ++i) sc[i] = opt_scalar_init<float>(opt, i);
                RowCtx<float> rc = opt_row_prologue_pure<float>(opt, sc, (uint64_t)cr[u], nsc_v);
                for (int c = gl * 4; c < wstride; c += LPR * 4) {
                    float4 g, w, a, b;
                    if (c == gl * 4) { g = g4[u]; w = w4[u]; a = a4[u]; b = b4[u]; }
                    else {  // dim > 128: remaining chunks, simple path
                        g = *reinterpret_cast<float4*>(arow + c);
                        w = a = b = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (fl[u] == 1) {
                            w = *reinterpret_cast<float4*>(wrow + c);
                            if (nslots > 0) a = *reinterpret_cast<float4*>(srow + c);
                            if (nslots > 1) b = *reinterpret_cast<float4*>(srow + wstride + c);
                        }
                    }
                    if (fl[u] == 2) {
                        w = init_block_masked(&T.init, keyr[u], c, dim);
                        a = make_float4(s0i, s0i, s0i, s0i);
                        b = make_float4(s1i, s1i, s1i, s1i);
                    }
                    *reinterpret_cast<float4*>(arow + c) = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (c + 0 < dim) opt_elem<float>(opt, rc, w.x, a.x, b.x, g.x);
                    if (c + 1 < dim) opt_elem<float>(opt, rc, w.y, a.y, b.y, g.y);
                    if (c + 2 < dim) opt_elem<float>(opt, rc, w.z, a.z, b.z, g.z);
                    if (c + 3 < dim) opt_elem<float>(opt, rc, w.w, a.w, b.w, g.w);
                    *reinterpret_cast<float4*>(wrow + c) = w;
                    if (nslots > 0) *reinterpret_cast<float4*>(srow + c) = a;
                    if (nslots > 1) *reinterpret_cast<float4*>(srow + wstride + c) = b;
                }
                if (gl == 0)
                    for (int i = 0; i < nsc; ++i) srow[(size_t)nslots * wstride + i] = nsc_v[i];
            }
        }
    } else if (flag) {  // dim < 4: one lane per row
        float* wrow = wloc + row * (unsigned long long)wstride;
        float* srow = T.state + row * (unsigned long long)T.sstride;
        float* arow = accbase + (unsigned long long)h * wstride;
        float sc[2] = {0.f, 0.f}, nsc_v[2];
        for (int i = 0; i < nsc; ++i)
            sc[i] = (flag == 2) ? opt_scalar_init<float>(opt, i) : srow[(size_t)nslots * wstride + i];
        RowCtx<float> rc = opt_row_prologue_pure<float>(opt, sc, (uint64_t)cnt, nsc_v);
        for (int c = 0; c < dim; ++c) {
            float g = arow[c];
            arow[c] = 0.f;
            float w, a = s0i, b = s1i;
            if (flag == 2) {
                w = init_scalar(&T.init, key, c);
            } else {
                w = wrow[c];
                if (nslots > 0) a = srow[c];
                if (nslots > 1) b = srow[wstride + c];
            }
            opt_elem<float>(opt, rc, w, a, b, g);
            wrow[c] = w;
            if (nslots > 0) srow[c] = a;
            if (nslots > 1) srow[wstride + c] = b;
        }
        for (int i = 0; i < nsc; ++i) srow[(size_t)nslots * wstride + i] = nsc_v[i];
    }
}

__device__ __noinline__ void apply_rows_slow(const TableDev& T, const PlanDev& P, float* accbase,
                                             unsigned long long key, unsigned long long row, unsigned h,
                                             unsigned cnt, int flag, int lane) {
    switch (T.lpr) {
        case 1: apply_rows<1>(T, P, accbase, key, row, h, cnt, flag, lane); break;
        case 2: apply_rows<2>(T, P, accbase, key, row, h, cnt, flag, lane); break;
        case 4: apply_rows<4>(T, P, accbase, key, row, h, cnt, flag, lane); break;
        case 8: apply_rows<8>(T, P, accbase, key, row, h, cnt, flag, lane); break;
        case 16: apply_rows<16>(T, P, accbase, key, row, h, cnt, flag, lane); break;
        default: apply_rows<32>(T, P, accbase, key, row, h, cnt, flag, lane); break;
    }
}

__global__ void __launch_bounds__(256, 2)
exb_push_update_kernel(const TableDev* __restrict__ tables, PlanDev P,
                       const long long* __restrict__ ids, const float* __restrict__ grads,
                       int n_rows) {
    extern __shared__ __align__(16) unsigned char exb_smem[];
    pdl_trigger();
    const SmemView S = stage_plan(tables, P, exb_smem);
    pdl_wait();
    ctx_check(P);
    int* s_prefix = S.seg_prefix;
    const int wic = threadIdx.x >> 5;
    unsigned char* stage_end = exb_smem + exb_smem_bytes(P.PT, P.F, true);
    unsigned char* wbuf = stage_end + (size_t)wic * EXB_APPLY_WARP_BUF;
    WarpMeta* wmeta = reinterpret_cast<WarpMeta*>(stage_end + 8 * (size_t)EXB_APPLY_WARP_BUF) + wic;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    const int W = P.W, PT = P.PT, rank = P.rank;
    // phase clock: CTA 0 / thread 0 stamps %globaltimer at every phase boundary into
    // stats[8..15] (read by utils.timers; the in-kernel equivalent of the reference's VTIMER)
#define EXB_STAMP(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) P.stats[8 + (i)] = globaltimer_ns(); } while (0)
    EXB_STAMP(0);
    if (blockIdx.x == 0 && threadIdx.x == 0) P.stats[7] = 1ull;     // phase-clock layout marker (v2 kernel writes 2)

    // ---------------- P1: dispatch (remote ids -> owner inbox, local ids -> combine map)
    for (int task = warp; task < P.num_tasks; task += nwarps) {
        const int f = find_segment(S.task_prefix, P.F, task);
        const int b0 = (task - S.task_prefix[f]) * 32;
        if (b0 >= n_rows) continue;
        const int pt = S.feat_pt[f];
        const TableDev& T = S.tab[pt];
        const int b = b0 + lane;
        unsigned long long id = 0;
        int owner = -1;
        if (b < n_rows) {
            id = (unsigned long long)__ldg(ids + (size_t)b * P.ncols + S.feat_col[f]);
            bool ok = T.is_hash ? ((id >> 63) == 0) : (id < T.vocab);
            if (ok) owner = owner_of(T, id, W);
        }
        const float* src = grads + (size_t)b * P.io_stride + S.feat_off[f];
        float* dst = nullptr;
        int mode = 0;
        {
            unsigned h = cmap_insert_warp(P, S, pt, id, owner == rank, lane);
            if (h != 0xFFFFFFFFu) {
                unsigned old = atomicAdd(&P.cmap_cnt[S.map_off[pt] + h], 1u);
                (void)old;
                dst = P.acc + S.acc_off[pt] + (unsigned long long)h * T.wstride;
                mode = 1;
            }
        }
        if (W > 1) {
            unsigned m = __match_any_sync(0xffffffffu, owner);
            if (owner >= 0 && owner != rank) {
                int leader = __ffs(m) - 1;
                unsigned base = 0;
                if (lane == leader)
                    base = atomicAdd(&P.send_cnt[(owner * PT + pt) * EXB_CTR_STRIDE], (unsigned)__popc(m));
                base = __shfl_sync(m, base, leader);
                unsigned pos = base + (unsigned)__popc(m & ((1u << lane) - 1u));
                if (pos < S.cap[pt]) {
                    P.inbox_keys[owner][(unsigned long long)rank * P.src_key_stride + S.key_off[pt] + pos] = id;
                    dst = P.inbox_grads[owner] + (unsigned long long)rank * P.src_grad_stride +
                          S.grad_off[pt] + (unsigned long long)pos * T.wstride;
                    mode = 2;
                } else {
                    set_error(P.status, EXB_ERR_INBOX_OVERFLOW);
                }
            }
        }
        if (S.feat_split[f] < T.dim)      // split-row feature: the gradient row comes from two places of the gradient matrix
            accum_rows_split(T, src, grads + (size_t)b * P.io_stride + S.feat_off2[f], S.feat_split[f], dst, mode, lane);
        else
            move_rows_dispatch(T, src, dst, mode, lane);
    }

    EXB_STAMP(1);
    if (W > 1) {
        // ---------------- B1: publish counts, cross-GPU barrier
        // CTAs arrive with a gpu-scope release; the one system-scope release (cumulative over the whole
        // grid's inbox stores) is the flag store in peer_barrier
        grid_barrier(P, false, [&]() {
            for (int i = threadIdx.x; i < W * PT; i += blockDim.x) {
                int o = i / PT, pt = i - o * PT;
                unsigned c = __ldcg(&P.send_cnt[i * EXB_CTR_STRIDE]);
                if (c > S.cap[pt]) c = S.cap[pt];
                if (o != rank) P.inbox_cnt[o][rank * PT + pt] = c;
                P.send_cnt[i * EXB_CTR_STRIDE] = 0;
            }
            peer_barrier(P);
        });
        EXB_STAMP(2);
        if (P.ar_n) dense_reduce_gather(P);    // peer loads in flight under the combine phase
        // ---------------- P3: combine inbox entries of every remote source
        const unsigned* mycnt = P.inbox_cnt[rank];
        block_task_prefix(mycnt, W * PT, s_prefix);
        const int ntask3 = s_prefix[W * PT];
        for (int task = warp; task < ntask3; task += nwarps) {
            const int seg = find_segment(s_prefix, W * PT, task);
            const int s = seg / PT, pt = seg - s * PT;
            if (s == rank) continue;  // local ids never travel through the inbox
            const TableDev& T = S.tab[pt];
            const unsigned e = (unsigned)(task - s_prefix[seg]) * 32u + lane;
            const unsigned n = __ldcg(&mycnt[seg]);
            const float* src = nullptr;
            float* dst = nullptr;
            int mode = 0;
            {
                unsigned long long key = 0;
                if (e < n)
                    key = P.inbox_keys[rank][(unsigned long long)s * P.src_key_stride + S.key_off[pt] + e];
                unsigned h = cmap_insert_warp(P, S, pt, key, e < n, lane);
                if (h != 0xFFFFFFFFu) {
                    atomicAdd(&P.cmap_cnt[S.map_off[pt] + h], 1u);
                    src = P.inbox_grads[rank] + (unsigned long long)s * P.src_grad_stride +
                          S.grad_off[pt] + (unsigned long long)e * T.wstride;
                    dst = P.acc + S.acc_off[pt] + (unsigned long long)h * T.wstride;
                    mode = 1;
                }
            }
            move_rows_dispatch(T, src, dst, mode, lane);
        }
    }

    // ---------------- B2: all accumulations visible
    EXB_STAMP(3);
    grid_barrier(P, false, [&]() {});
    EXB_STAMP(4);
    if (P.ar_n) dense_reduce_scatter(P);       // peer stores drain under the apply phase

    // ---------------- P5: apply optimizer to every unique row
    int* s_chunk = s_prefix + 256;     // the combine phase is over: its 1025-entry prefix array is free again
    int* s_cnt5 = s_prefix + 512;
    block_apply_prefix(P.ucount, PT, s_prefix, s_chunk, s_cnt5, EXB_CTR_STRIDE, S.tab, P.use_bulk);
    const int ntask5 = s_prefix[PT];
    unsigned n_unique_local = 0;
    unsigned long long* tr = P.trace ? P.trace + (size_t)warp * EXB_TRACE_SLOTS : nullptr;
    int trk = 1;
    if (tr && lane == 0) tr[0] = globaltimer_ns();
    for (int task = warp; task < ntask5; task += nwarps) {
        const int pt = find_segment(s_prefix, PT, task);
        const TableDev& T = S.tab[pt];
        const int chunk = s_chunk[pt];
        const unsigned n = (unsigned)s_cnt5[pt];
        const unsigned u = lane < chunk ? (unsigned)(task - s_prefix[pt]) * (unsigned)chunk + lane : n;
        unsigned long long* trt = (tr && trk + 8 <= EXB_TRACE_SLOTS) ? tr + trk : nullptr;
        trk += 8;
        if (trt && lane == 0) { trt[0] = (unsigned long long)task | ((unsigned long long)pt << 32); trt[1] = globaltimer_after(n); }
        unsigned long long key = 0, row = 0;
        unsigned h = 0, cnt = 0;
        int flag = 0;
        if (u < n) {
            h = __ldcg(&P.ulist[S.ulist_off[pt] + u]);
            key = __ldcg(&P.ukeys[S.ulist_off[pt] + u]);
            if (trt && lane == 0) trt[2] = globaltimer_after(h + key);
            const unsigned long long mo = S.map_off[pt] + h;
            cnt = (T.opt.kind == OPT_TEST) ? __ldcg(&P.cmap_cnt[mo]) : 1u;   // only the test optimizer uses the count
            if (trt && lane == 0) trt[3] = globaltimer_after(cnt);
            P.cmap_keys[mo] = EXB_EMPTY_KEY;
            P.cmap_cnt[mo] = 0;
            if (!T.is_hash) {
                row = local_row_of(T, key);
                atomicOr(&T.touched[row >> 5], 1u << (row & 31));
                flag = 1;
            } else {
                unsigned long long* keys = const_cast<unsigned long long*>(T.keys[rank]);
                unsigned long long mask = T.rows - 1, hh = exb_hash64(key) & mask;
                for (unsigned long long probe = 0; probe <= mask; ++probe) {
                    unsigned long long k = ld_relaxed_gpu_u64(&keys[hh]);
                    if (k == key) { flag = 1; break; }
                    if (k == EXB_EMPTY_KEY) {
                        unsigned long long prev = atomicCAS(&keys[hh], EXB_EMPTY_KEY, key);
                        if (prev == EXB_EMPTY_KEY) { flag = 2; break; }
                        if (prev == key) { flag = 1; break; }
                    }
                    hh = (hh + 1) & mask;
                }
                if (flag == 0) {
                    set_error(P.status, EXB_ERR_HASH_FULL);
                    clear_acc_row(P.acc + S.acc_off[pt] + (unsigned long long)h * T.wstride, T.wstride);
                }
                row = hh;
            }
            if (flag) ++n_unique_local;
        }
        if (T.is_hash) {   // one size-counter atomic per warp
            const unsigned nm = __ballot_sync(0xffffffffu, flag == 2);
            if (nm && lane == __ffs(nm) - 1) atomicAdd(T.size_ctr, (unsigned long long)__popc(nm));
        }
        float* accbase = P.acc + S.acc_off[pt];
        if (trt && lane == 0) trt[4] = globaltimer_after(row + (unsigned)flag);
        if (apply_is_bulk(T, P.use_bulk)) {
            apply_rows_bulk(T, P, accbase, key, row, h, cnt, flag, lane, wbuf, wmeta, chunk, trt);
            if (trt && lane == 0) { __threadfence(); trt[6] = globaltimer_ns(); }
            continue;
        }
        apply_rows_slow(T, P, accbase, key, row, h, cnt, flag, lane);
    }
    n_unique_local = __reduce_add_sync(0xffffffffu, n_unique_local);
    if (lane == 0 && n_unique_local) atomicAdd(&P.stats[2], (unsigned long long)n_unique_local);
    EXB_STAMP(5);

    // ---------------- B3: reset per-step counters; cross-GPU "update done"
    grid_barrier(P, false, [&]() {   // P5 wrote local memory only; the sys release is in peer_barrier
        for (int i = threadIdx.x; i < PT; i += blockDim.x) P.ucount[i * EXB_CTR_STRIDE] = 0;
        if (threadIdx.x == 0) atomicAdd(&P.stats[1], (unsigned long long)n_rows * P.F);
        // signal only: the next pull waits (peer_wait) -- unless the dense reduction rode along, whose result the
        // next kernel of this stream (the dense optimizer) reads
        if (W > 1) peer_barrier(P, P.ar_n != 0);
    });
    EXB_STAMP(6);
#undef EXB_STAMP
}

}  // namespace exb
