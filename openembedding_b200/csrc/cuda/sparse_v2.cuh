// sparse_v2.cuh -- "plan once per step": id de-duplication, unique-row pulls, pre-reduced pushes.
//
// Reference semantics being matched (the v1 kernels in sparse_kernels.cuh moved every LOOKUP over
// NVLink; the reference moves every UNIQUE id):
//   * pull  : the client de-duplicates the ids of a batch per variable before it asks the servers
//             (EmbeddingPullOperator.cpp:60-84) and scatters the unique rows back to request order
//             (:232-243); counters pull_indices / pull_unique (:208-209, 244-247);
//   * push  : the client sums the gradients of duplicate ids and counts them BEFORE sending
//             (EmbeddingPushOperator.cpp:29-62): one (id, summed gradient, count) per unique id;
//   * prefetch: a future batch's pull may be issued early and is parked until batch_id catches up
//             (exb_ops.cpp:139-175, EmbeddingPullOperator.cpp:117-145, Prefetch.h:11-72).
//
// Design. A plan owns TWO batch slots (double buffer). A slot is the per-step state:
//   per-table open-addressing map  id -> h   (h doubles as the row index of the slot's slabs)
//   slot_of[f][b]                   h of every lookup of the batch
//   ulist/ukeys/ucount              unique ids in insertion order
//   urows[h]                        staging row of a REMOTE unique id (pull)
//   acc[h], cmap_cnt[h]             summed gradient / count of a unique id (push)
// and three kernels work on it:
//   exb_plan_kernel   ids only (no table access): insert every id of the batch, record slot_of. Because it
//                     touches no table it may run any time after the ids are on the device -- for batch k+1
//                     on a side stream while step k computes: this is the prefetch (the parked pull of the
//                     reference), and it takes the hashing off the critical path of pull AND push.
//   exb_pull2_kernel  (W > 1) G: one peer load per UNIQUE remote id into urows (NVLink traffic / 2.2 at the
//                     benchmark's duplicate rate); L: local lookups straight from the local shard (duplicates
//                     hit L2); grid barrier; E: remote lookups expand from urows (L2). Gated by peer_wait on
//                     the "update done" epoch = batch_id gating.
//   exb_push2_kernel  P1 red.add of every gradient row into acc[slot_of] (no hashing); P2 ONE entry
//                     (id, summed row, count) per unique remote id to the owner's inbox (P2P stores); B1;
//                     P3 owner folds the pre-reduced entries of the other ranks into its map; B2; P5 optimizer
//                     on every owned unique row, map reset; B3 + slot parity flip.
// Which slot is "current" is a device-resident parity word (flipped by the push), so ONE captured CUDA graph
// serves even and odd steps.
#pragma once
#include "sparse_kernels.cuh"

namespace exb {

__device__ __forceinline__ SlotDev pick_slot(const PlanDev& P, int which) {
    const unsigned par = __ldcg(P.parity);
    SlotDev L;
    const bool one = ((par + (unsigned)which) & 1u) != 0u;
    L.cmap_keys = one ? P.slot[1].cmap_keys : P.slot[0].cmap_keys;
    L.cmap_cnt = one ? P.slot[1].cmap_cnt : P.slot[0].cmap_cnt;
    L.acc = one ? P.slot[1].acc : P.slot[0].acc;
    L.urows = one ? P.slot[1].urows : P.slot[0].urows;
    L.ulist = one ? P.slot[1].ulist : P.slot[0].ulist;
    L.ukeys = one ? P.slot[1].ukeys : P.slot[0].ukeys;
    L.ucount = one ? P.slot[1].ucount : P.slot[0].ucount;
    L.slot_of = one ? P.slot[1].slot_of : P.slot[0].slot_of;
    L.olist = one ? P.slot[1].olist : P.slot[0].olist;
    L.okeys = one ? P.slot[1].okeys : P.slot[0].okeys;
    L.ocount = one ? P.slot[1].ocount : P.slot[0].ocount;
    return L;
}

// warp-collective find-or-insert into the slot's map of plan-table pt (see cmap_insert_warp)
// new keys are appended to (list, lkeys, lcount): the unique list while a batch is planned, the owned list when
// the owner folds in the other ranks' entries
__device__ __forceinline__ unsigned slot_insert_warp(const PlanDev& P, const SlotDev& L, const SmemView& S, int pt,
                                                     unsigned long long key, bool active, int lane,
                                                     unsigned* list, unsigned long long* lkeys, unsigned* lcount) {
    const unsigned mask = S.map_mask[pt];
    unsigned long long* keys = L.cmap_keys + S.map_off[pt];
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
        if (lane == leader) base = atomicAdd(&lcount[pt * EXB_CTR_STRIDE], (unsigned)__popc(wmask));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (won) {
            const unsigned long long up = S.ulist_off[pt] + base + (unsigned)__popc(wmask & ((1u << lane) - 1u));
            list[up] = h;
            lkeys[up] = key;
        }
    }
    return active ? h : 0xFFFFFFFFu;
}

// one warp task of the planner: insert the 32 ids (f, b0 .. b0+31) into the slot's map
__device__ __forceinline__ void plan_one_task(const SmemView& S, const PlanDev& P, const SlotDev& L,
                                              const long long* __restrict__ ids, int n_rows, int task, int lane) {
    const int f = find_segment(S.task_prefix, P.F, task);
    const int b0 = (task - S.task_prefix[f]) * 32;
    if (b0 >= n_rows) return;
    const int pt = S.feat_pt[f];
    const TableDev& T = S.tab[pt];
    const int b = b0 + lane;
    unsigned long long id = 0;
    bool ok = false;
    if (b < n_rows) {
        id = (unsigned long long)__ldg(ids + (size_t)b * P.ncols + S.feat_col[f]);
        ok = T.is_hash ? ((id >> 63) == 0) : (id < T.vocab);
    }
    const unsigned h = slot_insert_warp(P, L, S, pt, id, ok, lane, L.ulist, L.ukeys, L.ucount);
    if (h != 0xFFFFFFFFu) atomicAdd(&L.cmap_cnt[S.map_off[pt] + h], 1u);
    if (b < n_rows) L.slot_of[(size_t)f * P.B + b] = h;
}

// ------------------------------------------------------------------ plan (de-duplicate)
__global__ void __launch_bounds__(256)
exb_plan_kernel(const TableDev* __restrict__ tables, PlanDev P, const long long* __restrict__ ids, int n_rows, int which) {
    extern __shared__ __align__(16) unsigned char exb_smem[];
    pdl_trigger();
    const SmemView S = stage_plan(tables, P, exb_smem);
    pdl_wait();
    ctx_check(P);
    const SlotDev L = pick_slot(P, which);
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int task = warp; task < P.num_tasks; task += nwarps) plan_one_task(S, P, L, ids, n_rows, task, lane);
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        atomicAdd(&P.stats[3], 1ull);                                            // plans built
    }
}

// Training pull: the stateless one-pass gather of exb_pull_kernel (every lookup reads its row where it lives --
// on several GPUs the step is bound by the NUMBER of dependent phases, not by NVLink bytes, so the
// one-pass gather beats the unique-row pull of exb_pull2_kernel) with the batch's de-duplication plan built IN
// THE SAME LAUNCH and in the shadow of the gather: every warp issues the cp.async loads of its 32 rows, inserts
// the same 32 ids into the slot's map while the rows are in flight, then waits and writes the rows out. The
// plan costs no launch, no stream fork, no second read of the ids and (nearly) no time.
__global__ void __launch_bounds__(256, 2)
exb_pull_plan_kernel(const TableDev* __restrict__ tables, PlanDev P, const long long* __restrict__ ids,
                     float* __restrict__ out, int n_rows, int which) {
    extern __shared__ __align__(16) unsigned char exb_smem[];
    // in-kernel phase clock of warp 0 of the LAST CTA (stats[16..23], "probe" in CudaEngine.status())
#define PP_STAMP(i) do { if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) P.stats[16 + (i)] = globaltimer_ns(); } while (0)
    PP_STAMP(0);
    pdl_trigger();
    const SmemView S = stage_plan(tables, P, exb_smem);
    PP_STAMP(1);
    pdl_wait();
    ctx_check(P);
    PP_STAMP(2);
    const SlotDev L = pick_slot(P, which);
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    if (P.W > 1) peer_wait(P);
    PP_STAMP(3);
    unsigned char* wbuf = exb_smem + exb_smem_bytes(P.PT, P.F, false) + (size_t)wic * EXB_PULL_WARP_BUF;
    for (int task = warp; task < P.num_tasks; task += nwarps) {
        const int f = find_segment(S.task_prefix, P.F, task);
        const int b0 = (task - S.task_prefix[f]) * 32;
        if (b0 >= n_rows) continue;
        const int pt = S.feat_pt[f];
        const TableDev& T = S.tab[pt];
        const int b = b0 + lane;
        int bulk;
        if (!(P.use_bulk && pull_fast_geometry(T, S.feat_split[f], &bulk))) {   // odd row shapes: plan, then gather
            plan_one_task(S, P, L, ids, n_rows, task, lane);
            pull_one_task(S, P, ids, out, n_rows, task, lane, wbuf);
            continue;
        }
        unsigned long long id = 0;
        const float* src = nullptr;
        int flag = 0;
        if (b < n_rows) {
            id = (unsigned long long)__ldg(ids + (size_t)b * P.ncols + S.feat_col[f]);
            flag = pull_resolve(T, P, id, &src);
        }
        if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) P.stats[20] = globaltimer_after(id + (unsigned long long)src);
        pull_rows_fast(T, src, id, flag, b0, n_rows, out, P.io_stride, S.feat_off[f], S.feat_off2[f], S.feat_split[f],
                       bulk, lane, wbuf, [&] {
            PP_STAMP(5);
            const unsigned h = slot_insert_warp(P, L, S, pt, id, flag != 0, lane, L.ulist, L.ukeys, L.ucount);
            if (h != 0xFFFFFFFFu) atomicAdd(&L.cmap_cnt[S.map_off[pt] + h], 1u);
            if (b < n_rows) L.slot_of[(size_t)f * P.B + b] = h;
            if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) P.stats[22] = globaltimer_after(h);
        });
    }
    PP_STAMP(7);
#undef PP_STAMP
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        atomicAdd(&P.stats[0], (unsigned long long)n_rows * (unsigned long long)P.F);
        atomicAdd(&P.stats[3], 1ull);
    }
}

// drop a prepared batch that will never be pushed (ONE CTA; rare path: evaluation pulls with grad enabled,
// a prefetched batch that is not the one trained next)
__global__ void __launch_bounds__(1024)
exb_plan_reset_kernel(PlanDev P, int which) {
    const SlotDev L = pick_slot(P, which);
    __shared__ unsigned s_n[EXB_MAX_PT];
    for (int pt = threadIdx.x; pt < P.PT; pt += blockDim.x) s_n[pt] = __ldcg(&L.ucount[pt * EXB_CTR_STRIDE]);
    __syncthreads();
    for (int pt = 0; pt < P.PT; ++pt) {
        const unsigned long long mo = P.pt_map_off[pt], uo = P.pt_ulist_off[pt];
        for (unsigned u = threadIdx.x; u < s_n[pt]; u += blockDim.x) {
            const unsigned h = L.ulist[uo + u];
            L.cmap_keys[mo + h] = EXB_EMPTY_KEY;
            L.cmap_cnt[mo + h] = 0u;
        }
    }
    __syncthreads();
    for (int pt = threadIdx.x; pt < P.PT; pt += blockDim.x) L.ucount[pt * EXB_CTR_STRIDE] = 0u;
}

// ------------------------------------------------------------------ row movers with a per-row destination
// mode per row (lane l describes row l of the warp task): 0 skip, 1 copy src -> dst, 2 initializer value of `id`,
// 3 zeros
__device__ __forceinline__ void rows_to(const TableDev& T, const float* src, unsigned long long id, int mode,
                                        float* dst, int lane, unsigned char* buf, int bufbytes) {
    const int wstride = T.wstride, dim = T.dim;
    if (!T.vec4) {                       // dim < 4: one lane per row
        if (mode) {
            for (int c = 0; c < dim; ++c) {
                float v = 0.f;
                if (mode == 1) v = src[c];
                else if (mode == 2) v = init_scalar(&T.init, id, c);
                dst[c] = v;
            }
        }
        return;
    }
    const unsigned rowbytes = (unsigned)wstride * 4u;
    if ((int)rowbytes > bufbytes) {      // very wide rows: the whole warp moves one row at a time
        for (int r = 0; r < 32; ++r) {
            const float* s = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src, r);
            float* d = (float*)__shfl_sync(0xffffffffu, (unsigned long long)dst, r);
            const int m = __shfl_sync(0xffffffffu, mode, r);
            const unsigned long long idr = __shfl_sync(0xffffffffu, id, r);
            if (!m) continue;
            for (int c = lane * 4; c < wstride; c += 128) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (m == 1) v = ld_stream_v4(s + c);
                else if (m == 2) v = init_block_masked(&T.init, idr, c, dim);
                *reinterpret_cast<float4*>(d + c) = v;
            }
        }
        return;
    }
    const int R = min(32, bufbytes / (int)rowbytes);   // rows per pass (warp uniform)
    const int lpr = T.lpr, gl = lane % lpr, RP = 32 / lpr;
    float* rows = reinterpret_cast<float*>(buf);
    for (int r0 = 0; r0 < 32; r0 += R) {
        for (int jb = 0; jb < R; jb += RP) {             // warp-uniform trip count (body shuffles)
            const int j = jb + lane / lpr, r = r0 + j;
            const float* s = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src, r & 31);
            const int m = __shfl_sync(0xffffffffu, mode, r & 31);
            if (j < R && r < 32 && m == 1)
                for (int c = gl * 4; c < wstride; c += lpr * 4) cp_async16(rows + (size_t)j * wstride + c, s + c);
        }
        cp_async_commit_wait();
        __syncwarp();
        for (int jb = 0; jb < R; jb += RP) {
            const int j = jb + lane / lpr, r = r0 + j;
            const unsigned long long idr = __shfl_sync(0xffffffffu, id, r & 31);
            const int m = __shfl_sync(0xffffffffu, mode, r & 31);
            float* d = (float*)__shfl_sync(0xffffffffu, (unsigned long long)dst, r & 31);
            if (j >= R || r >= 32 || m == 0) continue;
            for (int c = gl * 4; c < wstride; c += lpr * 4) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (m == 1) v = *reinterpret_cast<const float4*>(rows + (size_t)j * wstride + c);
                else if (m == 2) v = init_block_masked(&T.init, idr, c, dim);
                *reinterpret_cast<float4*>(d + c) = v;
            }
        }
        __syncwarp();
    }
}

// zero the rows flagged `on` (lane l describes row l)
__device__ __forceinline__ void zero_rows(const TableDev& T, float* dst, int on, int lane) {
    if (!T.vec4) {
        if (on) for (int c = 0; c < T.dim; ++c) dst[c] = 0.f;
        return;
    }
    const int wstride = T.wstride;
    const int lpr = T.lpr, gl = lane % lpr, RP = 32 / lpr;
    for (int jb = 0; jb < 32; jb += RP) {
        const int r = jb + lane / lpr;
        float* d = (float*)__shfl_sync(0xffffffffu, (unsigned long long)dst, r);
        const int m = __shfl_sync(0xffffffffu, on, r);
        if (!m) continue;
        for (int c = gl * 4; c < wstride; c += lpr * 4) *reinterpret_cast<float4*>(d + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// where does row `id` of table T live on rank `o`? (array: direct address; hash: probe in the owner's key slab)
// returns the mode for rows_to: 1 (src valid) or 2 (row not materialised yet -> initializer value)
__device__ __forceinline__ int resolve_row(const TableDev& T, unsigned long long id, int o, const float** src) {
    if (!T.is_hash) {
        *src = T.w[o] + local_row_of(T, id) * (unsigned long long)T.wstride;
        return 1;
    }
    const unsigned long long* keys = T.keys[o];
    const unsigned long long mask = T.rows - 1;
    unsigned long long h = exb_hash64(id) & mask;
    for (unsigned long long probe = 0; probe <= mask; ++probe) {
        const unsigned long long k = keys[h];
        if (k == id) { *src = T.w[o] + h * (unsigned long long)T.wstride; return 1; }
        if (k == EXB_EMPTY_KEY) break;
        h = (h + 1) & mask;
    }
    return 2;
}

// ------------------------------------------------------------------ pull, W > 1
__global__ void __launch_bounds__(256, 2)
exb_pull2_kernel(const TableDev* __restrict__ tables, PlanDev P, const long long* __restrict__ ids,
                 float* __restrict__ out, int n_rows, int which) {
    extern __shared__ __align__(16) unsigned char exb_smem[];
    pdl_trigger();
    const SmemView S = stage_plan(tables, P, exb_smem);
    pdl_wait();
    ctx_check(P);
    const SlotDev L = pick_slot(P, which);
    int* s_prefix = S.seg_prefix;
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    const int W = P.W, PT = P.PT, rank = P.rank;
    unsigned char* wbuf = exb_smem + exb_smem_bytes(PT, P.F, true) + (size_t)wic * EXB_PULL_WARP_BUF;
    if (W > 1) peer_wait(P);          // every peer's last update is complete and visible (batch_id gating)

    // ---- G: one peer load per unique remote id -> urows[h]
    block_task_prefix(L.ucount, PT, s_prefix, EXB_CTR_STRIDE);
    const int ntaskG = s_prefix[PT];
    unsigned n_remote_unique = 0;
    for (int task = warp; task < ntaskG; task += nwarps) {
        const int pt = find_segment(s_prefix, PT, task);
        const TableDev& T = S.tab[pt];
        const unsigned n = __ldcg(&L.ucount[pt * EXB_CTR_STRIDE]);
        const unsigned u = (unsigned)(task - s_prefix[pt]) * 32u + lane;
        const float* src = nullptr;
        float* dst = nullptr;
        unsigned long long key = 0;
        int mode = 0;
        if (u < n) {
            const unsigned h = __ldcg(&L.ulist[S.ulist_off[pt] + u]);
            key = __ldcg(&L.ukeys[S.ulist_off[pt] + u]);
            const int o = owner_of(T, key, W);
            if (o != rank) {
                mode = resolve_row(T, key, o, &src);
                dst = L.urows + S.acc_off[pt] + (unsigned long long)h * T.wstride;
                ++n_remote_unique;
            }
        }
        rows_to(T, src, key, mode, dst, lane, wbuf, EXB_PULL_WARP_BUF);
    }
    // ---- L: lookups owned by this rank come straight from the local shard (duplicates hit L2)
    for (int task = warp; task < P.num_tasks; task += nwarps) {
        const int f = find_segment(S.task_prefix, P.F, task);
        const int b0 = (task - S.task_prefix[f]) * 32;
        if (b0 >= n_rows) continue;
        const TableDev& T = S.tab[S.feat_pt[f]];
        const int b = b0 + lane;
        const float* src = nullptr;
        unsigned long long id = 0;
        int mode = 0;
        if (b < n_rows) {
            id = (unsigned long long)__ldg(ids + (size_t)b * P.ncols + S.feat_col[f]);
            const bool ok = T.is_hash ? ((id >> 63) == 0) : (id < T.vocab);
            if (!ok) mode = 3;                                   // invalid id / padding: zeros
            else if (owner_of(T, id, W) == rank) mode = resolve_row(T, id, rank, &src);
        }
        float* dst = out + (size_t)b * P.io_stride + S.feat_off[f];
        rows_to(T, src, id, mode, dst, lane, wbuf, EXB_PULL_WARP_BUF);
    }
    // ---- every unique remote row has landed in urows
    grid_barrier(P, false, [&]() {});
    // ---- E: remote lookups expand from urows (local L2)
    for (int task = warp; task < P.num_tasks; task += nwarps) {
        const int f = find_segment(S.task_prefix, P.F, task);
        const int b0 = (task - S.task_prefix[f]) * 32;
        if (b0 >= n_rows) continue;
        const int pt = S.feat_pt[f];
        const TableDev& T = S.tab[pt];
        const int b = b0 + lane;
        const float* src = nullptr;
        int mode = 0;
        if (b < n_rows) {
            const unsigned long long id = (unsigned long long)__ldg(ids + (size_t)b * P.ncols + S.feat_col[f]);
            const bool ok = T.is_hash ? ((id >> 63) == 0) : (id < T.vocab);
            if (ok && owner_of(T, id, W) != rank) {
                const unsigned h = __ldcg(&L.slot_of[(size_t)f * P.B + b]);
                if (h != 0xFFFFFFFFu) {
                    src = L.urows + S.acc_off[pt] + (unsigned long long)h * T.wstride;
                    mode = 1;
                } else mode = 3;
            }
        }
        float* dst = out + (size_t)b * P.io_stride + S.feat_off[f];
        rows_to(T, src, 0ull, mode, dst, lane, wbuf, EXB_PULL_WARP_BUF);
    }
    n_remote_unique = __reduce_add_sync(0xffffffffu, n_remote_unique);
    if (lane == 0 && n_remote_unique) atomicAdd(&P.stats[5], (unsigned long long)n_remote_unique);   // rows over NVLink
    if (threadIdx.x == 0 && blockIdx.x == 0)
        atomicAdd(&P.stats[0], (unsigned long long)n_rows * (unsigned long long)P.F);
}

// ------------------------------------------------------------------ push + update on a prepared slot
__global__ void __launch_bounds__(256, 2)
exb_push2_kernel(const TableDev* __restrict__ tables, PlanDev P, const float* __restrict__ grads, int n_rows,
                 int which) {
    extern __shared__ __align__(16) unsigned char exb_smem[];
    pdl_trigger();
    const SmemView S = stage_plan(tables, P, exb_smem);
    pdl_wait();
    ctx_check(P);
    const SlotDev L = pick_slot(P, which);
    int* s_prefix = S.seg_prefix;
    const int wic = threadIdx.x >> 5;
    unsigned char* stage_end = exb_smem + exb_smem_bytes(P.PT, P.F, true);
    unsigned char* wbuf = stage_end + (size_t)wic * EXB_APPLY_WARP_BUF;
    WarpMeta* wmeta = reinterpret_cast<WarpMeta*>(stage_end + 8 * (size_t)EXB_APPLY_WARP_BUF) + wic;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    const int W = P.W, PT = P.PT, rank = P.rank;
#define EXB_STAMP(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) P.stats[8 + (i)] = globaltimer_ns(); } while (0)
    EXB_STAMP(0);
    if (blockIdx.x == 0 && threadIdx.x < 32) {     // unique ids of this rank's batch (reference accumulator pull_unique)
        unsigned long long s = 0;
        for (int pt = lane; pt < PT; pt += 32) s += __ldcg(&L.ucount[pt * EXB_CTR_STRIDE]);
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) { atomicAdd(&P.stats[4], s); P.stats[7] = 2ull; }
    }

    // ---------------- P1: every gradient row is added into the accumulator row of its unique id (no hashing)
    for (int task = warp; task < P.num_tasks; task += nwarps) {
        const int f = find_segment(S.task_prefix, P.F, task);
        const int b0 = (task - S.task_prefix[f]) * 32;
        if (b0 >= n_rows) continue;
        const int pt = S.feat_pt[f];
        const TableDev& T = S.tab[pt];
        const int b = b0 + lane;
        unsigned h = 0xFFFFFFFFu;
        if (b < n_rows) h = __ldcg(&L.slot_of[(size_t)f * P.B + b]);
        const float* src = grads + (size_t)b * P.io_stride + S.feat_off[f];
        float* dst = nullptr;
        int mode = 0;
        if (h != 0xFFFFFFFFu) { dst = L.acc + S.acc_off[pt] + (unsigned long long)h * T.wstride; mode = 1; }
        if (S.feat_split[f] < T.dim)
            accum_rows_split(T, src, grads + (size_t)b * P.io_stride + S.feat_off2[f], S.feat_split[f], dst, mode, lane);
        else
            move_rows_dispatch(T, src, dst, mode, lane);
    }
    EXB_STAMP(1);
    unsigned n_sent = 0;
    if (W > 1) {
        // ---------------- B0: the local sums are complete
        grid_barrier(P, false, [&]() {});
        // ---------------- P2: ONE (id, summed gradient, count) entry per unique remote id -> owner inbox
        block_task_prefix(L.ucount, PT, s_prefix, EXB_CTR_STRIDE);
        const int ntask2 = s_prefix[PT];
        for (int task = warp; task < ntask2; task += nwarps) {
            const int pt = find_segment(s_prefix, PT, task);
            const TableDev& T = S.tab[pt];
            const unsigned n = __ldcg(&L.ucount[pt * EXB_CTR_STRIDE]);
            const unsigned u = (unsigned)(task - s_prefix[pt]) * 32u + lane;
            int owner = -1;
            unsigned h = 0;
            unsigned long long key = 0;
            if (u < n) {
                h = __ldcg(&L.ulist[S.ulist_off[pt] + u]);
                key = __ldcg(&L.ukeys[S.ulist_off[pt] + u]);
                owner = owner_of(T, key, W);
            }
            const bool remote = owner >= 0 && owner != rank;
            {   // ids this rank owns go onto the optimizer's work list (one counter atomic per warp)
                const unsigned om = __ballot_sync(0xffffffffu, owner == rank);
                if (om) {
                    const int ol = __ffs(om) - 1;
                    unsigned ob = 0;
                    if (lane == ol) ob = atomicAdd(&L.ocount[pt * EXB_CTR_STRIDE], (unsigned)__popc(om));
                    ob = __shfl_sync(0xffffffffu, ob, ol);
                    if (owner == rank) {
                        const unsigned long long op = S.ulist_off[pt] + ob + (unsigned)__popc(om & ((1u << lane) - 1u));
                        L.olist[op] = h;
                        L.okeys[op] = key;
                    }
                }
            }
            float* arow = L.acc + S.acc_off[pt] + (unsigned long long)h * T.wstride;
            float* dst = nullptr;
            int mode = 0;
            const unsigned m = __match_any_sync(0xffffffffu, remote ? owner : -1);
            if (remote) {
                const int leader = __ffs(m) - 1;
                unsigned base = 0;
                if (lane == leader)
                    base = atomicAdd(&P.send_cnt[(owner * PT + pt) * EXB_CTR_STRIDE], (unsigned)__popc(m));
                base = __shfl_sync(m, base, leader);
                const unsigned pos = base + (unsigned)__popc(m & ((1u << lane) - 1u));
                if (pos < S.cap[pt]) {
                    const unsigned long long kp = (unsigned long long)rank * P.src_key_stride + S.key_off[pt] + pos;
                    P.inbox_keys[owner][kp] = key;
                    P.inbox_vals[owner][kp] = __ldcg(&L.cmap_cnt[S.map_off[pt] + h]);
                    dst = P.inbox_grads[owner] + (unsigned long long)rank * P.src_grad_stride + S.grad_off[pt] +
                          (unsigned long long)pos * T.wstride;
                    mode = 2;
                    ++n_sent;
                } else {
                    set_error(P.status, EXB_ERR_INBOX_OVERFLOW);
                }
            }
            move_rows_dispatch(T, arow, dst, mode, lane);     // accumulator row -> peer inbox (P2P stores)
            zero_rows(T, arow, remote ? 1 : 0, lane);         // the accumulator slab is clean again for the next batch
        }
        EXB_STAMP(2);
        // ---------------- B1: publish counts, cross-GPU barrier
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
        EXB_STAMP(3);
        if (P.ar_n) dense_reduce_gather(P);    // dense-gradient all-reduce on this kernel's barriers (sparse_kernels.cuh)
        // ---------------- P3: fold the other ranks' pre-reduced entries into this rank's map
        const unsigned* mycnt = P.inbox_cnt[rank];
        block_task_prefix(mycnt, W * PT, s_prefix);
        const int ntask3 = s_prefix[W * PT];
        for (int task = warp; task < ntask3; task += nwarps) {
            const int seg = find_segment(s_prefix, W * PT, task);
            const int s = seg / PT, pt = seg - s * PT;
            if (s == rank) continue;
            const TableDev& T = S.tab[pt];
            const unsigned e = (unsigned)(task - s_prefix[seg]) * 32u + lane;
            const unsigned n = __ldcg(&mycnt[seg]);
            const float* src = nullptr;
            float* dst = nullptr;
            int mode = 0;
            unsigned long long key = 0;
            unsigned c = 0;
            const unsigned long long kp = (unsigned long long)s * P.src_key_stride + S.key_off[pt] + e;
            if (e < n) { key = P.inbox_keys[rank][kp]; c = P.inbox_vals[rank][kp]; }
            const unsigned h = slot_insert_warp(P, L, S, pt, key, e < n, lane, L.olist, L.okeys, L.ocount);
            if (h != 0xFFFFFFFFu) {
                atomicAdd(&L.cmap_cnt[S.map_off[pt] + h], c);
                src = P.inbox_grads[rank] + (unsigned long long)s * P.src_grad_stride + S.grad_off[pt] +
                      (unsigned long long)e * T.wstride;
                dst = L.acc + S.acc_off[pt] + (unsigned long long)h * T.wstride;
                mode = 1;
            }
            move_rows_dispatch(T, src, dst, mode, lane);
        }
    }
    // ---------------- B2: all accumulations visible
    EXB_STAMP(4);
    grid_barrier(P, false, [&]() {});
    EXB_STAMP(5);
    if (P.ar_n) dense_reduce_scatter(P);       // peer stores drain under the apply phase

    // ---------------- P5: optimizer on every unique row this rank owns; every map entry is reset
    int* s_chunk = s_prefix + 256;
    int* s_cnt5 = s_prefix + 512;
    // world > 1: the work list is the owned list (own unique ids this rank owns + ids received from peers);
    // world == 1: every unique id is owned
    const unsigned* wl_h = (W > 1) ? L.olist : L.ulist;
    const unsigned long long* wl_k = (W > 1) ? L.okeys : L.ukeys;
    const unsigned* wl_n = (W > 1) ? L.ocount : L.ucount;
    block_apply_prefix(wl_n, PT, s_prefix, s_chunk, s_cnt5, EXB_CTR_STRIDE, S.tab, P.use_bulk);
    const int ntask5 = s_prefix[PT];
    unsigned n_unique_local = 0;
    for (int task = warp; task < ntask5; task += nwarps) {
        const int pt = find_segment(s_prefix, PT, task);
        const TableDev& T = S.tab[pt];
        const int chunk = s_chunk[pt];
        const unsigned n = (unsigned)s_cnt5[pt];
        const unsigned u = lane < chunk ? (unsigned)(task - s_prefix[pt]) * (unsigned)chunk + lane : n;
        unsigned long long key = 0, row = 0;
        unsigned h = 0, cnt = 0;
        int flag = 0;
        if (u < n) {
            h = __ldcg(&wl_h[S.ulist_off[pt] + u]);
            key = __ldcg(&wl_k[S.ulist_off[pt] + u]);
            const unsigned long long mo = S.map_off[pt] + h;
            cnt = (T.opt.kind == OPT_TEST) ? __ldcg(&L.cmap_cnt[mo]) : 1u;
            L.cmap_keys[mo] = EXB_EMPTY_KEY;
            L.cmap_cnt[mo] = 0;
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
                    clear_acc_row(L.acc + S.acc_off[pt] + (unsigned long long)h * T.wstride, T.wstride);
                }
                row = hh;
            }
            if (flag) ++n_unique_local;
        }
        if (T.is_hash) {
            const unsigned nm = __ballot_sync(0xffffffffu, flag == 2);
            if (nm && lane == __ffs(nm) - 1) atomicAdd(T.size_ctr, (unsigned long long)__popc(nm));
        }
        float* accbase = L.acc + S.acc_off[pt];
        if (apply_is_bulk(T, P.use_bulk)) {
            apply_rows_bulk(T, P, accbase, key, row, h, cnt, flag, lane, wbuf, wmeta, chunk, nullptr);
            continue;
        }
        apply_rows_slow(T, P, accbase, key, row, h, cnt, flag, lane);
    }
    if (W > 1) {
        // map entries of the ids other ranks own (shipped in P2) are cleared here: no insert is in flight any more
        const unsigned gtid = blockIdx.x * blockDim.x + threadIdx.x, gthreads = gridDim.x * blockDim.x;
        for (int pt = 0; pt < PT; ++pt) {
            const TableDev& T = S.tab[pt];
            const unsigned n = __ldcg(&L.ucount[pt * EXB_CTR_STRIDE]);
            for (unsigned u = gtid; u < n; u += gthreads) {
                const unsigned long long key = __ldcg(&L.ukeys[S.ulist_off[pt] + u]);
                if (owner_of(T, key, W) != rank) {
                    const unsigned long long mo = S.map_off[pt] + __ldcg(&L.ulist[S.ulist_off[pt] + u]);
                    L.cmap_keys[mo] = EXB_EMPTY_KEY;
                    L.cmap_cnt[mo] = 0;
                }
            }
        }
    }
    n_unique_local = __reduce_add_sync(0xffffffffu, n_unique_local);
    if (lane == 0 && n_unique_local) atomicAdd(&P.stats[2], (unsigned long long)n_unique_local);
    n_sent = __reduce_add_sync(0xffffffffu, n_sent);
    if (lane == 0 && n_sent) atomicAdd(&P.stats[6], (unsigned long long)n_sent);                      // rows over NVLink
    EXB_STAMP(6);

    // ---------------- B3: reset per-step counters; flip the slot parity; cross-GPU "update done"
    grid_barrier(P, false, [&]() {
        for (int i = threadIdx.x; i < PT; i += blockDim.x) { L.ucount[i * EXB_CTR_STRIDE] = 0; L.ocount[i * EXB_CTR_STRIDE] = 0; }
        if (threadIdx.x == 0) {
            atomicAdd(&P.stats[1], (unsigned long long)n_rows * P.F);
            *P.parity = __ldcg(P.parity) ^ 1u;
        }
        if (W > 1) peer_barrier(P, P.ar_n != 0);
    });
    EXB_STAMP(7);
#undef EXB_STAMP
}

}  // namespace exb
