// exb_common.cuh -- device-side data model of the sparse engine.
//
// The reference is a CPU parameter server: worker -> RPC -> server thread -> RPC -> worker
// (SURVEY 3.2/3.3). Here every rank maps every peer's table slabs, inbox and flag words
// (CUDA IPC over NVLink/NVSwitch) and the PS verbs are kernels:
//   pull          = ids -> owner = id % W -> one-sided peer *loads* of rows     (K1+K2+K3)
//   push + update = P2P *stores* of (id, grad) into the owner's inbox -> flag barrier
//                   -> owner combines duplicates with atomics -> optimizer        (K4a+K4b)
// `batch_id` gating of the reference (EmbeddingPullOperator.cpp:117-145) becomes a device
// epoch counter exchanged through system-scope release/acquire flags.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "exb_math.h"

#define EXB_MAX_PEERS 8
#define EXB_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull

namespace exb {

struct TableDev {
    float* w[EXB_MAX_PEERS];                        // weight slab of every rank's shard (peer mapped)
    const unsigned long long* keys[EXB_MAX_PEERS];  // hash keys of every rank's shard (hash tables)
    float* state;                                   // local optimizer-state slab
    unsigned* touched;                              // local bitmap of updated rows (array tables)
    unsigned long long* size_ctr;                   // local number of occupied slots (hash tables)
    unsigned long long rows;   // array: rows per shard = ceil(vocab / W); hash: capacity (pow2)
    unsigned long long vocab;  // array: vocabulary; hash: 2^63
    int dim, wstride, sstride, nslots, nscalars;
    int is_hash, lpr, vec4;
    int shard_num, shard_base;  // owner(id) = (shard_base + id % shard_num) % W, local row = id / shard_num
    InitParams init;
    OptParams opt;
};

// One batch slot of a plan (sparse_v2.cuh): the per-step de-duplication state. A plan owns two (double buffer:
// the plan of batch k+1 is built while batch k trains); slot[0] aliases the v1 work arrays below.
struct SlotDev {
    unsigned long long* cmap_keys;   // per-table open-addressing maps id -> h
    unsigned* cmap_cnt;              // [h] lookups of the id in the batch (+ counts received from peers)
    float* acc;                      // [h] summed gradient row
    float* urows;                    // [h] staging row of a remote unique id (pull)
    unsigned* ulist;                 // unique entries in insertion order: h ...
    unsigned long long* ukeys;       // ... and id
    unsigned* ucount;                // [PT * EXB_CTR_STRIDE]
    unsigned* slot_of;               // [F][B] h of every lookup (0xFFFFFFFF: invalid id)
    unsigned* olist;                 // world > 1: unique entries OWNED by this rank (own lookups + received), the
    unsigned long long* okeys;       //            work list of the optimizer phase
    unsigned* ocount;                // [PT * EXB_CTR_STRIDE]
};

struct PlanDev {
    int F, B, PT, W, rank;
    int num_tasks;          // sum_f ceil(B/32)
    int io_stride;          // floats per row of out / grad
    int ncols;              // id columns per batch row (several features may share one column)
    int use_bulk;           // 1: rows move through per-warp shared-memory buffers with cp.async (bulk_rows.cuh)
    int _pad1;
    const int* feat_pt;     // [F] feature -> plan-table
    const int* feat_off;    // [F] column offset of the feature in out / grad rows
    const int* feat_col;    // [F] id column of the feature
    const int* feat_off2;   // [F] split-row features: columns >= feat_split[f] of the table row live at this offset
    const int* feat_split;  // [F] first column that goes to feat_off2 (>= row width: the feature is not split)
    const int* task_prefix; // [F+1]
    const int* pt_table;    // [PT] plan-table -> engine table id
    const unsigned* pt_cap; // [PT] max entries one source can send for this table per step
    const unsigned long long* pt_key_off;   // [PT] offset (u64 elements) inside one source block
    const unsigned long long* pt_grad_off;  // [PT] offset (floats) inside one source block
    unsigned long long src_key_stride, src_grad_stride;
    unsigned long long* inbox_keys[EXB_MAX_PEERS];  // peer mapped, indexed by owner rank
    float* inbox_grads[EXB_MAX_PEERS];
    unsigned* inbox_cnt[EXB_MAX_PEERS];             // [W src][PT]
    unsigned* send_cnt;                             // local [W owner][PT]
    const unsigned long long* pt_map_off;           // [PT] offset into cmap arrays
    const unsigned* pt_map_mask;                    // [PT] capacity-1 (pow2)
    const unsigned long long* pt_acc_off;           // [PT] offset (floats) into acc
    const unsigned long long* pt_ulist_off;         // [PT]
    unsigned long long* cmap_keys;
    unsigned* cmap_cnt;
    float* acc;
    unsigned* ulist;
    unsigned long long* ukeys;                      // key of every unique-list entry (parallel to ulist)
    unsigned* ucount;                               // [PT]
    unsigned* flags[EXB_MAX_PEERS];                 // peer mapped [W]
    unsigned* gbar;                                 // [0] arrive count, [1] generation
    unsigned* epoch;                                // device-resident barrier epoch
    int* status;                                    // 0 ok; else first error code
    unsigned long long* stats;                      // [0] pull ids, [1] push ids, [2] unique rows updated
    unsigned long long* trace;                      // optional per-warp %globaltimer trace (EXB_TRACE_SLOTS per warp)
    SlotDev slot[2];                                // v2 batch slots
    unsigned* parity;                               // which slot is "current" (flipped by exb_push2_kernel)
    unsigned* inbox_vals[EXB_MAX_PEERS];            // peer mapped: count of every inbox entry (parallel to inbox_keys)
    // dense-gradient all-reduce riding on the push kernel's cross-GPU barriers (exb_plan_set_dense_reduce; 0: off)
    float* ar_buf[EXB_MAX_PEERS];                   // peer mapped flat gradient buffer of every rank
    unsigned long long ar_n;                        // floats (multiple of 4)
};
#define EXB_TRACE_SLOTS 32

enum ExbStatus : int {
    EXB_OK = 0,
    EXB_ERR_TIMEOUT_GRID = 1,
    EXB_ERR_TIMEOUT_PEER = 2,
    EXB_ERR_HASH_FULL = 3,
    EXB_ERR_INBOX_OVERFLOW = 4,
    EXB_ERR_CMAP_FULL = 5,
    EXB_ERR_CTX_VERSION = 6,     // a rank announced a newer context (moved a slab) than this rank's mappings were built for
};
// u32 word offsets inside a rank's sync block (PlanDev::flags[rank] points at its start)
#define EXB_CTX_ANNOUNCED_WORD 16
#define EXB_CTX_EXPECTED_WORD 24

// ---------------------------------------------------------------- PTX helpers
__device__ __forceinline__ unsigned ld_acquire_sys_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_u32(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_gpu_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu_u32(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// timer read that cannot issue before `dep` has been produced (scoreboard dependency)
__device__ __forceinline__ unsigned long long globaltimer_after(unsigned long long dep) {
    unsigned long long t;
    asm volatile("{ .reg .b64 d; mov.b64 d, %1; mov.u64 %0, %%globaltimer; }" : "=l"(t) : "l"(dep));
    return t;
}
// fire-and-forget vector reduction (sm_90+): 4 fp32 adds in one L2 atomic transaction
__device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void red_add_f32(float* addr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
// streaming 128-bit load that does not pollute L1 (rows are touched once per step)
__device__ __forceinline__ float4 ld_stream_v4(const float* p) {
    float4 v;
    asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}

#define EXB_SPIN_TIMEOUT_NS 4000000000ull  // 4 s: a hung peer becomes an error code, not a hung box

__device__ __forceinline__ void set_error(int* status, int code) { atomicCAS(status, 0, code); }

// row sharding: the reference routes shard = id % global_shard_num, local = id / global_shard_num
// (EmbeddingPullOperator.cpp:74-76) and places shards round-robin on servers
// (WorkerContext.cpp:66-85); shard_base is that round-robin offset.
__device__ __forceinline__ int owner_of(const TableDev& T, unsigned long long id, int W) {
    return (int)(((unsigned)T.shard_base + (unsigned)(id % (unsigned)T.shard_num)) % (unsigned)W);
}
__device__ __forceinline__ unsigned long long local_row_of(const TableDev& T, unsigned long long id) {
    return id / (unsigned)T.shard_num;
}
// shard index held by `rank` (>= shard_num means: this rank holds no shard of the table)
__device__ __forceinline__ int shard_of_rank(const TableDev& T, int rank, int W) {
    return (rank - T.shard_base % W + W) % W;
}

// NEVER read shared words through `volatile`: it lowers to LDG.STRONG.SYS, and those loads
// took ~5 us each in the apply phase (trace: 15.9 us -> 4.4 us per task after switching the
// four dependent loads to ld.global.cg / ld.relaxed.gpu).
// Polling loads are RELAXED (no per-iteration L1 invalidate: `ld.acquire` lowers to
// LDG + CCTL.IVALL, and a spinning thread would keep flushing the L1 that co-resident
// CTAs are still working out of); one acquire fence is issued after the loop exits.
__device__ __forceinline__ unsigned ld_relaxed_gpu_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ld_relaxed_sys_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// Grid-wide barrier for a persistent kernel whose CTAs are all resident
// (grid <= SMs * occupancy, enforced by the host). `master` runs on every thread of
// CTA 0 while all other CTAs are parked -- this is where the cross-GPU flag exchange and
// the count publication happen.
template <class MasterFn>
__device__ __forceinline__ void grid_barrier(const PlanDev& P, bool sys_scope, MasterFn master) {
    // bar.sync orders every thread's writes before thread 0's fence, and fence + atomic is a
    // cumulative release: ONE fence per CTA covers the whole CTA (a system fence costs an
    // NVLink round trip when peer stores are in flight -- 256 of them in series per barrier
    // was most of the 17-25 us the first version spent here).
    __syncthreads();
    __shared__ unsigned s_gen;
    if (blockIdx.x == 0) {
        if (threadIdx.x == 0) {
            if (sys_scope) fence_acq_rel_sys(); else fence_acq_rel_gpu();
            unsigned gen = ld_relaxed_gpu_u32(&P.gbar[1]);
            s_gen = gen;
            atomicAdd(&P.gbar[0], 1u);
            unsigned long long t0 = globaltimer_ns();
            unsigned it = 0;
            while (ld_relaxed_gpu_u32(&P.gbar[0]) != gridDim.x) {
                __nanosleep(20);
                if ((++it & 1023u) == 0 && globaltimer_ns() - t0 > EXB_SPIN_TIMEOUT_NS) {
                    set_error(P.status, EXB_ERR_TIMEOUT_GRID);
                    break;
                }
            }
            fence_acq_rel_gpu();
        }
        __syncthreads();
        master();
        __syncthreads();
        if (threadIdx.x == 0) {
            P.gbar[0] = 0;
            st_release_gpu_u32(&P.gbar[1], s_gen + 1);   // release orders the reset before the new generation
        }
    } else {
        if (threadIdx.x == 0) {
            unsigned gen = ld_relaxed_gpu_u32(&P.gbar[1]);
            if (sys_scope) fence_acq_rel_sys(); else fence_acq_rel_gpu();
            atomicAdd(&P.gbar[0], 1u);
            unsigned long long t0 = globaltimer_ns();
            unsigned it = 0, ns = 32;
            while (ld_relaxed_gpu_u32(&P.gbar[1]) == gen) {
                __nanosleep(ns);             // growing back-off: ~300 CTAs poll this one line
                if (ns < 128) ns += 32;
                if ((++it & 1023u) == 0 && globaltimer_ns() - t0 > EXB_SPIN_TIMEOUT_NS) {
                    set_error(P.status, EXB_ERR_TIMEOUT_GRID);
                    break;
                }
            }
            fence_acq_rel_gpu();
        }
    }
    __syncthreads();
}

// Cross-GPU barrier executed by CTA 0 (all its threads call this). Every rank writes its
// new epoch into slot [rank] of every peer's flag array with a system-scope release
// (cumulative over everything CTA 0 has observed, i.e. the whole grid's peer stores) and,
// if `wait`, polls its own array until all peers have reached the epoch.
// wait == false is the "update done" signal at the end of a push: nobody has to stand still
// for it -- the next kernel that reads peer shards (pull) calls peer_wait() first, by which
// time the flags have long arrived.
__device__ __forceinline__ void peer_barrier(const PlanDev& P, bool wait = true) {
    __syncthreads();
    const unsigned e = *(volatile unsigned*)P.epoch + 1;
    __syncthreads();
    if ((int)threadIdx.x < P.W) {
        st_release_sys_u32(&P.flags[threadIdx.x][P.rank], e);
        if (wait) {
            unsigned long long t0 = globaltimer_ns();
            unsigned it = 0;
            while ((int)(ld_relaxed_sys_u32(&P.flags[P.rank][threadIdx.x]) - e) < 0) {
                if ((++it & 255u) == 0 && globaltimer_ns() - t0 > EXB_SPIN_TIMEOUT_NS) {
                    set_error(P.status, EXB_ERR_TIMEOUT_PEER);
                    break;
                }
            }
            fence_acq_rel_sys();
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) *(volatile unsigned*)P.epoch = e;
    __syncthreads();
}

// Context-version guard (engine.cu: announce_ctx / exb_engine_accept_ctx), first thing in every plan kernel: the versions
// the ranks have announced into this rank's sync block must be the ones this rank's peer mappings were built against.
// Local loads only (two words per rank, CTA 0).
__device__ __forceinline__ void ctx_check(const PlanDev& P) {
    if (blockIdx.x == 0 && (int)threadIdx.x < P.W) {
        const unsigned* blk = P.flags[P.rank];
        const unsigned announced = ld_relaxed_sys_u32(blk + EXB_CTX_ANNOUNCED_WORD + threadIdx.x);
        const unsigned expected = ld_relaxed_sys_u32(blk + EXB_CTX_EXPECTED_WORD + threadIdx.x);
        if (announced != expected) set_error(P.status, EXB_ERR_CTX_VERSION);
    }
}

// Every CTA of a kernel that reads peer shards: wait until all peers have signalled the
// epoch this rank has reached (their last update is complete and visible).
__device__ __forceinline__ void peer_wait(const PlanDev& P) {
    // one polling thread per CTA, whole flag row per poll (two 16-byte loads), growing back-off: several
    // hundred CTAs x W threads re-reading one L2 line saturate its slice and delay everybody
    if (threadIdx.x == 0) {
        const unsigned e = *(volatile unsigned*)P.epoch;
        const unsigned* row = P.flags[P.rank];
        unsigned long long t0 = globaltimer_ns();
        unsigned it = 0, ns = 32;
        for (;;) {
            unsigned v[8];
            asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(row) : "memory");
            asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7]) : "l"(row + 4) : "memory");
            bool ok = true;
#pragma unroll
            for (int i = 0; i < 8; ++i) ok = ok && (i >= P.W || (int)(v[i] - e) >= 0);
            if (ok) break;
            __nanosleep(ns);
            if (ns < 256) ns += 32;
            if ((++it & 255u) == 0 && globaltimer_ns() - t0 > EXB_SPIN_TIMEOUT_NS) {
                set_error(P.status, EXB_ERR_TIMEOUT_PEER);
                break;
            }
        }
        fence_acq_rel_sys();
    }
    __syncthreads();
}

}  // namespace exb
