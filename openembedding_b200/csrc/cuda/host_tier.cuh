// host_tier.cuh -- host-DRAM overflow tier of a hash table (included by engine.cu).
//
// Reference: the PMem tables (openembedding/variable/PmemEmbeddingTable.h:107-417: every row lives in persistent
// memory, hot rows in a DRAM LRU cache, each item carries the batch id `work_id`; :237-270 promote / evict;
// :285-328 checkpoint flush of exactly the rows older than the checkpoint batch), their item pools
// (PmemEmbeddingItemPool.h:133-365), the pull-triggered ASYNC promotion of
// PmemEmbeddingOptimizerVariable.h:129-192 and the cache budget of PersistManager.h:12-83.
//
// GPU mapping (one tier per rank and table):
//   PMem pool   -> `hrows`: PINNED host DRAM (cudaHostAlloc), one slab of [weights | optimizer state] rows. The GPU
//                  reads and writes it directly over PCIe (zero-copy): no CPU thread, no staging copy, no ids.cpu().
//   pool index  -> `hkeys`: open-addressing id -> host-row index kept in HBM (8 B per host row), so every atomic of the
//                  store is an HBM atomic and only row payloads cross PCIe.
//   DRAM cache  -> the table's ordinary HBM hash shard (the RESIDENCY MAP is that hash table itself: a miss is found
//                  by the same probe the pull kernel uses) + `stamp` / `clean` words per slot:
//                  stamp = work_id of the last batch that needed the row (CLOCK / LRU approximation),
//                  dirty <=> stamp >= clean (clean = work_id at which HBM and host copy were last equal).
//   promotion   -> tier_admit_kernel, one launch per batch, enqueued on a SIDE STREAM one batch ahead by the python
//                  layer (VariableAsyncTask analogue): ids -> probe cache -> on a miss claim a slot, look the id up in
//                  the host index, warp-cooperative copy host row -> HBM slot (or first-touch initialisation).
//                  After it every row the batch touches is resident: pull / push kernels run unchanged.
//   eviction    -> tier_scan_kernel + in-place rebuild at a quiescent point: age histogram -> cutoff that keeps the
//                  `target` most recently used rows; dirty victims are written back (HBM -> host over PCIe); survivors
//                  are compacted through a scratch slab and re-inserted (no tombstones in the probe chains).
//   checkpoint  -> tier flush (write back every dirty row, keep the cache) + dump of the host slab.
#pragma once

namespace {

struct Tier {
    Engine* e = nullptr;
    int table = -1;
    unsigned long long hcap = 0;          // host rows capacity (pow2)
    int HR = 0;                           // floats per host row = wstride + sstride
    unsigned long long* hkeys = nullptr;  // HBM [hcap]
    float* hrows = nullptr;               // pinned host [hcap * HR]
    unsigned* stamp = nullptr;            // HBM [cache capacity]
    unsigned* clean = nullptr;            // HBM [cache capacity]
    unsigned long long* ctr = nullptr;    // HBM counters, see TIER_* below
    unsigned* hist = nullptr;             // HBM age histogram [TIER_BINS]
    // scratch for the rebuild (allocated at the first eviction)
    unsigned long long* sk = nullptr;
    float* srow = nullptr;
    unsigned* sst = nullptr;
    unsigned* scl = nullptr;
    unsigned long long scap = 0;
};

enum { TIER_HITS = 0, TIER_MISS_HOST = 1, TIER_MISS_NEW = 2, TIER_EVICTED = 3, TIER_WRITEBACK = 4, TIER_HOST_ROWS = 5,
       TIER_KEEP = 6, TIER_CUTOFF = 7, TIER_NCTR = 8 };
#define TIER_BINS 1024

__device__ __forceinline__ long long tier_host_find(const unsigned long long* hkeys, unsigned long long hmask,
                                                    unsigned long long id) {
    unsigned long long h = exb_hash64(id ^ 0x9E3779B97F4A7C15ull) & hmask;
    for (unsigned long long probe = 0; probe <= hmask; ++probe) {
        const unsigned long long k = ld_relaxed_gpu_u64(&hkeys[h]);
        if (k == id) return (long long)h;
        if (k == EXB_EMPTY_KEY) return -1;
        h = (h + 1) & hmask;
    }
    return -1;
}
__device__ __forceinline__ long long tier_host_insert(unsigned long long* hkeys, unsigned long long hmask,
                                                      unsigned long long id, unsigned long long* ctr) {
    unsigned long long h = exb_hash64(id ^ 0x9E3779B97F4A7C15ull) & hmask;
    for (unsigned long long probe = 0; probe <= hmask; ++probe) {
        const unsigned long long k = ld_relaxed_gpu_u64(&hkeys[h]);
        if (k == id) return (long long)h;
        if (k == EXB_EMPTY_KEY) {
            const unsigned long long prev = atomicCAS(&hkeys[h], EXB_EMPTY_KEY, id);
            if (prev == EXB_EMPTY_KEY) { atomicAdd(&ctr[TIER_HOST_ROWS], 1ull); return (long long)h; }
            if (prev == id) return (long long)h;
        }
        h = (h + 1) & hmask;
    }
    return -1;
}

// warp-cooperative copy of one [w | state] row between an HBM slot and a host row
__device__ __forceinline__ void tier_copy_row(const TableDev& T, int rank, unsigned long long slot, float* hrow,
                                              bool to_host, int lane) {
    float* w = T.w[rank] + slot * (unsigned long long)T.wstride;
    float* s = T.state + slot * (unsigned long long)T.sstride;
    if (T.vec4) {
        for (int c = lane * 4; c < T.wstride; c += 128) {
            if (to_host) *reinterpret_cast<float4*>(hrow + c) = *reinterpret_cast<const float4*>(w + c);
            else *reinterpret_cast<float4*>(w + c) = *reinterpret_cast<const float4*>(hrow + c);
        }
        for (int c = lane * 4; c < T.sstride; c += 128) {
            if (to_host) *reinterpret_cast<float4*>(hrow + T.wstride + c) = *reinterpret_cast<const float4*>(s + c);
            else *reinterpret_cast<float4*>(s + c) = *reinterpret_cast<const float4*>(hrow + T.wstride + c);
        }
    } else {
        for (int c = lane; c < T.wstride; c += 32) { if (to_host) hrow[c] = w[c]; else w[c] = hrow[c]; }
        for (int c = lane; c < T.sstride; c += 32) { if (to_host) hrow[T.wstride + c] = s[c]; else s[c] = hrow[T.wstride + c]; }
    }
}
// first touch: initializer weights + optimizer-state initial values
__device__ __forceinline__ void tier_init_row(const TableDev& T, int rank, unsigned long long slot,
                                              unsigned long long id, int lane) {
    float* w = T.w[rank] + slot * (unsigned long long)T.wstride;
    float* s = T.state + slot * (unsigned long long)T.sstride;
    for (int c = lane; c < T.wstride; c += 32) w[c] = c < T.dim ? init_scalar(&T.init, id, c) : 0.f;
    const int slot_w = T.nslots * T.wstride;
    for (int c = lane; c < T.sstride; c += 32) {
        float v = 0.f;
        if (c < slot_w) v = opt_slot_init<float>(T.opt, c / T.wstride);
        else if (c - slot_w < T.nscalars) v = opt_scalar_init<float>(T.opt, c - slot_w);
        s[c] = v;
    }
}

// ids: any int64 array (every rank's lookups of the batch); rows this rank owns become resident
__global__ void __launch_bounds__(256)
tier_admit_kernel(TableDev T, int rank, int W, const long long* __restrict__ ids, unsigned long long n, unsigned work,
                  unsigned long long* hkeys, unsigned long long hmask, float* hrows, int HR, unsigned* stamp,
                  unsigned* clean, unsigned long long* ctr, int* status) {
    const int lane = threadIdx.x & 31;
    const unsigned long long warp = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    unsigned long long* keys = const_cast<unsigned long long*>(T.keys[rank]);
    const unsigned long long mask = T.rows - 1;
    for (unsigned long long base = warp * 32; base < n; base += nwarps * 32) {
        const unsigned long long i = base + lane;
        unsigned long long id = 0, slot = 0;
        long long hs = -1;
        int act = 0;          // 0 nothing, 1 load from host row hs, 2 first touch
        if (i < n) {
            id = (unsigned long long)ids[i];
            if ((id >> 63) == 0 && owner_of(T, id, W) == rank) {
                unsigned long long h = exb_hash64(id) & mask;
                bool done = false;
                for (unsigned long long probe = 0; probe <= mask && !done; ++probe) {
                    const unsigned long long k = ld_relaxed_gpu_u64(&keys[h]);
                    if (k == id) { stamp[h] = work; atomicAdd(&ctr[TIER_HITS], 1ull); done = true; break; }
                    if (k == EXB_EMPTY_KEY) {
                        const unsigned long long prev = atomicCAS(&keys[h], EXB_EMPTY_KEY, id);
                        if (prev == EXB_EMPTY_KEY) {                 // this lane loads the row
                            slot = h;
                            stamp[h] = work;
                            atomicAdd(T.size_ctr, 1ull);
                            hs = tier_host_find(hkeys, hmask, id);
                            if (hs >= 0) { act = 1; clean[h] = work; atomicAdd(&ctr[TIER_MISS_HOST], 1ull); }
                            else { act = 2; clean[h] = 0u; atomicAdd(&ctr[TIER_MISS_NEW], 1ull); }
                            done = true;
                            break;
                        }
                        if (prev == id) { stamp[h] = work; atomicAdd(&ctr[TIER_HITS], 1ull); done = true; break; }
                    }
                    h = (h + 1) & mask;
                }
                if (!done) atomicCAS(status, 0, EXB_ERR_HASH_FULL);
            }
        }
        unsigned todo = __ballot_sync(0xffffffffu, act != 0);
        while (todo) {
            const int r = __ffs(todo) - 1;
            todo &= todo - 1;
            const int a = __shfl_sync(0xffffffffu, act, r);
            const unsigned long long sl = __shfl_sync(0xffffffffu, slot, r);
            const unsigned long long idr = __shfl_sync(0xffffffffu, id, r);
            const long long hr = __shfl_sync(0xffffffffu, hs, r);
            if (a == 1) tier_copy_row(T, rank, sl, hrows + (unsigned long long)hr * HR, false, lane);
            else tier_init_row(T, rank, sl, idr, lane);
        }
    }
}

// age histogram of the resident rows (age = work - stamp, clipped)
__global__ void tier_hist_kernel(TableDev T, int rank, unsigned work, const unsigned* stamp, unsigned* hist) {
    const unsigned long long* keys = T.keys[rank];
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < T.rows;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        if (keys[i] == EXB_EMPTY_KEY) continue;
        unsigned age = work - stamp[i];
        if (age >= TIER_BINS) age = TIER_BINS - 1;
        atomicAdd(&hist[age], 1u);
    }
}
// cutoff age: keep the youngest rows up to `target` (whole age classes; class 0 = needed right now, always kept)
__global__ void tier_cutoff_kernel(const unsigned* hist, unsigned long long target, unsigned long long* ctr) {
    if (threadIdx.x || blockIdx.x) return;
    unsigned long long kept = 0;
    unsigned cut = 1;
    for (unsigned a = 0; a < TIER_BINS; ++a) {
        if (a > 0 && kept + hist[a] > target) break;
        kept += hist[a];
        cut = a + 1;
    }
    ctr[TIER_CUTOFF] = cut;          // rows with age < cut survive
    ctr[TIER_KEEP] = 0;
}

// One pass over the cache. flush_only: write back every dirty row, keep everything.
// Otherwise: rows with age >= cutoff are victims (written back if dirty); survivors are appended to the scratch slab.
__global__ void __launch_bounds__(256)
tier_scan_kernel(TableDev T, int rank, unsigned work, int flush_only, unsigned long long* hkeys,
                 unsigned long long hmask, float* hrows, int HR, unsigned* stamp, unsigned* clean,
                 unsigned long long* ctr, unsigned long long* sk, float* srow, unsigned* sst, unsigned* scl, int* status) {
    const int lane = threadIdx.x & 31;
    const unsigned long long warp = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const unsigned long long* keys = T.keys[rank];
    const unsigned cut = flush_only ? 0xFFFFFFFFu : (unsigned)ctr[TIER_CUTOFF];
    for (unsigned long long base = warp * 32; base < T.rows; base += nwarps * 32) {
        const unsigned long long i = base + lane;
        unsigned long long key = EXB_EMPTY_KEY;
        bool keep = false, wb = false;
        long long hs = -1;
        unsigned long long spos = 0;
        if (i < T.rows) key = keys[i];
        if (key != EXB_EMPTY_KEY) {
            const unsigned st = stamp[i], cl = clean[i];
            keep = flush_only || (work - st) < cut;
            wb = st >= cl;                       // dirty
            if (wb && (flush_only || !keep)) {
                hs = tier_host_insert(hkeys, hmask, key, ctr);
                if (hs < 0) { atomicCAS(status, 0, EXB_ERR_HASH_FULL); wb = false; }
            } else wb = false;
            if (wb) clean[i] = work + 1;
        }
        if (!flush_only) {
            const unsigned km = __ballot_sync(0xffffffffu, keep);
            if (km) {
                const int leader = __ffs(km) - 1;
                unsigned long long b = 0;
                if (lane == leader) b = atomicAdd(&ctr[TIER_KEEP], (unsigned long long)__popc(km));
                b = __shfl_sync(0xffffffffu, b, leader);
                if (keep) {
                    spos = b + (unsigned)__popc(km & ((1u << lane) - 1u));
                    sk[spos] = key; sst[spos] = stamp[i]; scl[spos] = clean[i];
                }
            }
            const unsigned em = __ballot_sync(0xffffffffu, key != EXB_EMPTY_KEY && !keep);
            if (em && lane == __ffs(em) - 1) atomicAdd(&ctr[TIER_EVICTED], (unsigned long long)__popc(em));
        }
        unsigned wm = __ballot_sync(0xffffffffu, wb);
        if (wm && lane == __ffs(wm) - 1) atomicAdd(&ctr[TIER_WRITEBACK], (unsigned long long)__popc(wm));
        while (wm) {                             // HBM -> host over PCIe
            const int r = __ffs(wm) - 1;
            wm &= wm - 1;
            const long long hr = __shfl_sync(0xffffffffu, hs, r);
            tier_copy_row(T, rank, base + r, hrows + (unsigned long long)hr * HR, true, lane);
        }
        if (!flush_only) {
            unsigned km = __ballot_sync(0xffffffffu, keep);
            while (km) {                         // survivor -> scratch slab
                const int r = __ffs(km) - 1;
                km &= km - 1;
                const unsigned long long sp = __shfl_sync(0xffffffffu, spos, r);
                tier_copy_row(T, rank, base + r, srow + sp * HR, true, lane);
            }
        }
    }
}

__global__ void tier_clear_cache_kernel(TableDev T, int rank, unsigned* stamp, unsigned* clean) {
    unsigned long long* keys = const_cast<unsigned long long*>(T.keys[rank]);
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < T.rows;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        keys[i] = EXB_EMPTY_KEY; stamp[i] = 0u; clean[i] = 0u;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *T.size_ctr = 0ull;
}

__global__ void __launch_bounds__(256)
tier_reinsert_kernel(TableDev T, int rank, const unsigned long long* ctr, const unsigned long long* sk,
                     float* srow, const unsigned* sst, const unsigned* scl, int HR, unsigned* stamp, unsigned* clean,
                     int* status) {
    const int lane = threadIdx.x & 31;
    const unsigned long long warp = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const unsigned long long n = ctr[TIER_KEEP];
    unsigned long long* keys = const_cast<unsigned long long*>(T.keys[rank]);
    const unsigned long long mask = T.rows - 1;
    for (unsigned long long i = warp; i < n; i += nwarps) {
        long long slot = -1;
        if (lane == 0) {
            const unsigned long long key = sk[i];
            unsigned long long h = exb_hash64(key) & mask;
            for (unsigned long long probe = 0; probe <= mask; ++probe) {
                const unsigned long long prev = atomicCAS(&keys[h], EXB_EMPTY_KEY, key);
                if (prev == EXB_EMPTY_KEY) { slot = (long long)h; break; }
                h = (h + 1) & mask;
            }
            if (slot >= 0) { stamp[slot] = sst[i]; clean[slot] = scl[i]; }
            else atomicCAS(status, 0, EXB_ERR_HASH_FULL);
        }
        slot = __shfl_sync(0xffffffffu, slot, 0);
        if (slot >= 0) tier_copy_row(T, rank, (unsigned long long)slot, srow + i * HR, false, lane);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *T.size_ctr = n;
}

// host rows -> (ids, weights, states) in the reference layout, for dumps: one warp per host slot range
__global__ void tier_host_enumerate_kernel(const unsigned long long* hkeys, unsigned long long hcap,
                                           unsigned long long* out_slots, unsigned long long* counter) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < hcap;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        if (hkeys[i] == EXB_EMPTY_KEY) continue;
        out_slots[atomicAdd(counter, 1ull)] = i;
    }
}

int tier_alloc_scratch(Tier* t) {
    const TableDev& T = t->e->tables[t->table].d;
    if (t->scap >= T.rows) return 0;
    if (t->sk) { cudaFree(t->sk); cudaFree(t->srow); cudaFree(t->sst); cudaFree(t->scl); }
    t->scap = T.rows;
    CK(cudaMalloc(&t->sk, t->scap * 8));
    CK(cudaMalloc(&t->srow, t->scap * (size_t)t->HR * 4));
    CK(cudaMalloc(&t->sst, t->scap * 4));
    CK(cudaMalloc(&t->scl, t->scap * 4));
    return 0;
}

}  // namespace

extern "C" {

// Attach a host tier to an allocated hash table. host_rows: capacity of the pinned host slab (rows).
void* exb_tier_create(void* h, int ti, uint64_t host_rows) {
    Engine* e = (Engine*)h;
    if (ti < 0 || ti >= (int)e->tables.size() || !e->tables[ti].allocated || !e->tables[ti].d.is_hash) {
        fail_msg("tier: needs an allocated hash table");
        return nullptr;
    }
    CKP(cudaSetDevice(e->device));
    Tier* t = new Tier();
    t->e = e; t->table = ti;
    const TableDev& T = e->tables[ti].d;
    t->HR = T.wstride + T.sstride;
    unsigned long long cap = 1024;
    while (cap < 2 * host_rows) cap <<= 1;             // load <= 1/2
    t->hcap = cap;
    CKP(cudaMalloc(&t->hkeys, cap * 8));
    fill_u64_kernel<<<e->sms * 4, 256>>>(t->hkeys, cap, EXB_EMPTY_KEY);
    cudaError_t err = cudaHostAlloc((void**)&t->hrows, cap * (size_t)t->HR * 4, cudaHostAllocMapped | cudaHostAllocPortable);
    if (err != cudaSuccess) { fail("cudaHostAlloc (host tier slab)", err); cudaFree(t->hkeys); delete t; return nullptr; }
    CKP(cudaMalloc(&t->stamp, T.rows * 4)); CKP(cudaMemset(t->stamp, 0, T.rows * 4));
    CKP(cudaMalloc(&t->clean, T.rows * 4)); CKP(cudaMemset(t->clean, 0, T.rows * 4));
    CKP(cudaMalloc(&t->ctr, TIER_NCTR * 8)); CKP(cudaMemset(t->ctr, 0, TIER_NCTR * 8));
    CKP(cudaMalloc(&t->hist, TIER_BINS * 4));
    CKP(cudaDeviceSynchronize());
    return t;
}
void exb_tier_destroy(void* th) {
    Tier* t = (Tier*)th;
    cudaSetDevice(t->e->device);
    cudaFree(t->hkeys); cudaFreeHost(t->hrows); cudaFree(t->stamp); cudaFree(t->clean); cudaFree(t->ctr); cudaFree(t->hist);
    if (t->sk) { cudaFree(t->sk); cudaFree(t->srow); cudaFree(t->sst); cudaFree(t->scl); }
    delete t;
}
// Make every row of `ids` (int64 device array of n lookups of ANY rank) that this rank owns resident in HBM.
int exb_tier_admit(void* th, uint64_t ids, uint64_t n, uint32_t work, uint64_t stream) {
    Tier* t = (Tier*)th;
    Engine* e = t->e;
    if (n == 0) return 0;
    const TableDev& T = e->tables[t->table].d;
    int grid = (int)std::min<uint64_t>((n + 255) / 256, (uint64_t)e->sms * 8);
    tier_admit_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(T, e->rank, e->world, (const long long*)ids, n, work,
        t->hkeys, t->hcap - 1, t->hrows, t->HR, t->stamp, t->clean, t->ctr, (int*)(e->sync_local + OFF_STATUS));
    CK(cudaGetLastError());
    return 0;
}
// Write back every dirty row (checkpoint / persist); the cache keeps its contents.
int exb_tier_flush(void* th, uint32_t work, uint64_t stream) {
    Tier* t = (Tier*)th;
    Engine* e = t->e;
    const TableDev& T = e->tables[t->table].d;
    tier_scan_kernel<<<e->sms * 8, 256, 0, (cudaStream_t)stream>>>(T, e->rank, work, 1, t->hkeys, t->hcap - 1, t->hrows,
        t->HR, t->stamp, t->clean, t->ctr, nullptr, nullptr, nullptr, nullptr, (int*)(e->sync_local + OFF_STATUS));
    CK(cudaGetLastError());
    return 0;
}
// Evict down to (about) `target` resident rows, least recently used first; dirty victims are written back.
// Must run at a quiescent point (no pull / push of this table in flight on any rank).
int exb_tier_evict(void* th, uint64_t target, uint32_t work, uint64_t stream) {
    Tier* t = (Tier*)th;
    Engine* e = t->e;
    const TableDev& T = e->tables[t->table].d;
    cudaStream_t st = (cudaStream_t)stream;
    if (tier_alloc_scratch(t)) return -1;
    CK(cudaMemsetAsync(t->hist, 0, TIER_BINS * 4, st));
    tier_hist_kernel<<<e->sms * 8, 256, 0, st>>>(T, e->rank, work, t->stamp, t->hist);
    tier_cutoff_kernel<<<1, 32, 0, st>>>(t->hist, target, t->ctr);
    tier_scan_kernel<<<e->sms * 8, 256, 0, st>>>(T, e->rank, work, 0, t->hkeys, t->hcap - 1, t->hrows, t->HR, t->stamp,
        t->clean, t->ctr, t->sk, t->srow, t->sst, t->scl, (int*)(e->sync_local + OFF_STATUS));
    tier_clear_cache_kernel<<<e->sms * 8, 256, 0, st>>>(T, e->rank, t->stamp, t->clean);
    tier_reinsert_kernel<<<e->sms * 8, 256, 0, st>>>(T, e->rank, t->ctr, t->sk, t->srow, t->sst, t->scl, t->HR, t->stamp,
        t->clean, (int*)(e->sync_local + OFF_STATUS));
    CK(cudaGetLastError());
    return 0;
}
// drop the cache (and the host store when host_too)
int exb_tier_clear(void* th, int host_too) {
    Tier* t = (Tier*)th;
    Engine* e = t->e;
    const TableDev& T = e->tables[t->table].d;
    CK(cudaSetDevice(e->device));
    tier_clear_cache_kernel<<<e->sms * 8, 256>>>(T, e->rank, t->stamp, t->clean);
    if (host_too) {
        fill_u64_kernel<<<e->sms * 4, 256>>>(t->hkeys, t->hcap, EXB_EMPTY_KEY);
        CK(cudaMemset(t->ctr, 0, TIER_NCTR * 8));
    }
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    return 0;
}
// out[0..7] = hits, misses served from host, first-touch misses, evicted rows, written-back rows, host rows,
//             resident rows, host capacity (rows)   (device sync)
int exb_tier_stats(void* th, uint64_t* out) {
    Tier* t = (Tier*)th;
    Engine* e = t->e;
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    unsigned long long c[TIER_NCTR];
    CK(cudaMemcpy(c, t->ctr, sizeof(c), cudaMemcpyDeviceToHost));
    for (int i = 0; i < 6; ++i) out[i] = c[i];
    unsigned long long sz = 0;
    CK(cudaMemcpy(&sz, e->tables[t->table].d.size_ctr, 8, cudaMemcpyDeviceToHost));
    out[6] = sz; out[7] = t->hcap / 2;
    return 0;
}
// out: [0] host slab pointer (pinned host memory, HR floats per row), [1] HR, [2] host index capacity,
//      [3] bytes of pinned host memory, [4] bytes of HBM held by the tier (index + stamps + scratch)
int exb_tier_info(void* th, uint64_t* out) {
    Tier* t = (Tier*)th;
    const TableDev& T = t->e->tables[t->table].d;
    out[0] = (uint64_t)t->hrows; out[1] = (uint64_t)t->HR; out[2] = t->hcap;
    out[3] = t->hcap * (uint64_t)t->HR * 4;
    out[4] = t->hcap * 8 + T.rows * 8 + t->scap * ((uint64_t)t->HR * 4 + 16);
    return 0;
}
// ids (global) and host-slab row index of every row in the host store: ids_out / slots_out device arrays of
// capacity cap; *n_out = rows found. Rows are then read straight from the pinned slab by the caller.
int exb_tier_host_enumerate(void* th, uint64_t slots_out_dev, uint64_t cap, uint64_t* n_out) {
    Tier* t = (Tier*)th;
    Engine* e = t->e;
    CK(cudaSetDevice(e->device));
    unsigned long long* ctr;
    CK(cudaMalloc(&ctr, 8));
    CK(cudaMemset(ctr, 0, 8));
    (void)cap;
    tier_host_enumerate_kernel<<<e->sms * 8, 256>>>(t->hkeys, t->hcap, (unsigned long long*)slots_out_dev, ctr);
    CK(cudaGetLastError());
    CK(cudaMemcpy(n_out, ctr, 8, cudaMemcpyDeviceToHost));
    cudaFree(ctr);
    return 0;
}
// host index keys (device pointer) for the dump: id of host slot i = hkeys[i]
uint64_t exb_tier_hkeys_ptr(void* th) { return (uint64_t)((Tier*)th)->hkeys; }

// The optimizer of the table changed (it is configured lazily at the first optimizer step, like the reference:
// exb.py:460-462): the state width -- and with it the host-row layout -- may differ. Weights of rows already in
// the host store are kept, their optimizer state restarts from the initial values (a category change resets the
// state everywhere, EmbeddingVariable.cpp:44-47). The HBM side was re-laid out by exb_table_set_optimizer.
int exb_tier_relayout(void* th) {
    Tier* t = (Tier*)th;
    Engine* e = t->e;
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    const TableDev& T = e->tables[t->table].d;
    const int newHR = T.wstride + T.sstride;
    if (newHR == t->HR) {
        // same width: only the state values restart
    }
    float* nrows = nullptr;
    cudaError_t err = cudaHostAlloc((void**)&nrows, t->hcap * (size_t)newHR * 4, cudaHostAllocMapped | cudaHostAllocPortable);
    if (err != cudaSuccess) return fail("cudaHostAlloc (host tier relayout)", err);
    std::vector<unsigned long long> hk(t->hcap);
    CK(cudaMemcpy(hk.data(), t->hkeys, t->hcap * 8, cudaMemcpyDeviceToHost));
    const int slot_w = T.nslots * T.wstride;
    for (unsigned long long i = 0; i < t->hcap; ++i) {
        if (hk[i] == EXB_EMPTY_KEY) continue;
        float* dst = nrows + i * (size_t)newHR;
        memcpy(dst, t->hrows + i * (size_t)t->HR, (size_t)T.wstride * 4);
        for (int c = 0; c < T.sstride; ++c) {
            float v = 0.f;
            if (c < slot_w) v = opt_slot_init<float>(T.opt, c / T.wstride);
            else if (c - slot_w < T.nscalars) v = opt_scalar_init<float>(T.opt, c - slot_w);
            dst[T.wstride + c] = v;
        }
    }
    cudaFreeHost(t->hrows);
    t->hrows = nrows;
    t->HR = newHR;
    if (t->sk) { cudaFree(t->sk); cudaFree(t->srow); cudaFree(t->sst); cudaFree(t->scl); t->sk = nullptr; t->scap = 0; }
    // every resident row now carries a fresh state: it differs from its host copy
    CK(cudaMemset(t->clean, 0, T.rows * 4));
    return 0;
}

// bulk insert into the host store from HOST arrays (load_model / restore): ids[n], rows[n][HR] in slab layout
int exb_tier_host_put(void* th, const uint64_t* ids, uint64_t n, const float* rows) {
    Tier* t = (Tier*)th;
    Engine* e = t->e;
    CK(cudaSetDevice(e->device));
    if (n == 0) return 0;
    // the index lives in HBM: pull it to the host, insert, push it back (load is a cold path)
    std::vector<unsigned long long> hk(t->hcap);
    CK(cudaMemcpy(hk.data(), t->hkeys, t->hcap * 8, cudaMemcpyDeviceToHost));
    const unsigned long long hmask = t->hcap - 1;
    unsigned long long added = 0;
    for (uint64_t i = 0; i < n; ++i) {
        unsigned long long id = ids[i];
        unsigned long long hh = exb_hash64(id ^ 0x9E3779B97F4A7C15ull) & hmask;
        bool ok = false;
        for (unsigned long long probe = 0; probe <= hmask; ++probe) {
            if (hk[hh] == id) { ok = true; break; }
            if (hk[hh] == EXB_EMPTY_KEY) { hk[hh] = id; ++added; ok = true; break; }
            hh = (hh + 1) & hmask;
        }
        if (!ok) return fail_msg("tier: host store full");
        memcpy(t->hrows + hh * (size_t)t->HR, rows + i * (size_t)t->HR, (size_t)t->HR * 4);
    }
    CK(cudaMemcpy(t->hkeys, hk.data(), t->hcap * 8, cudaMemcpyHostToDevice));
    unsigned long long c = 0;
    CK(cudaMemcpy(&c, t->ctr + TIER_HOST_ROWS, 8, cudaMemcpyDeviceToHost));
    c += added;
    CK(cudaMemcpy(t->ctr + TIER_HOST_ROWS, &c, 8, cudaMemcpyHostToDevice));
    return 0;
}

}  // extern "C"
