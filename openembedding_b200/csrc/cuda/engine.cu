// engine.cu -- host runtime of the sparse engine + C ABI ("exb_cuda_*").
//
// Owns the HBM slabs of every table shard, the peer mapping (CUDA IPC), the per-plan
// inbox / combine-map work areas and the launch logic of the fused kernels in
// sparse_kernels.cuh. Replaces, for one NVSwitch box, the reference's
// Connection/WorkerContext/EmbeddingVariableHandle client runtime and the
// ps::Server request loop (openembedding/client/*.cpp, pico-ps/service/Service.cpp).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "sparse_kernels.cuh"
#include "sparse_v2.cuh"

using namespace exb;

static thread_local std::string g_err;
static int fail(const char* what, cudaError_t e) {
    g_err = std::string(what) + ": " + cudaGetErrorString(e);
    return -1;
}
static int fail_msg(const std::string& m) { g_err = m; return -1; }
#define CK(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return fail(#x, _e); } while (0)
#define CKP(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { fail(#x, _e); return nullptr; } } while (0)

namespace {

const size_t SYNC_BYTES = 2u << 20;
const size_t OFF_FLAGS = 0, OFF_EPOCH = 128, OFF_STATUS = 132, OFF_GBAR = 136, OFF_STATS = 256;
// context versions (exb_common.cuh: ctx_check): [64, 96) announced by every rank's host into this block, [96, 128) the
// versions this rank's mappings were built against (accepted at the last connect)
const size_t OFF_CTX_ANNOUNCED = 4 * EXB_CTX_ANNOUNCED_WORD, OFF_CTX_EXPECTED = 4 * EXB_CTX_EXPECTED_WORD;

struct HostTable {
    TableDev d;
    float* w_local = nullptr;
    unsigned long long* keys_local = nullptr;
    size_t w_bytes = 0, s_bytes = 0, k_bytes = 0, t_bytes = 0;
    bool allocated = false;
    bool opt_set = false;
};

struct Engine {
    int device = 0, rank = 0, world = 1, sms = 132, max_ctas = 0;
    std::vector<HostTable> tables;
    TableDev* d_tables = nullptr;
    size_t d_tables_cap = 0;
    char* sync_local = nullptr;
    char* sync_peer[EXB_MAX_PEERS] = {nullptr};
    unsigned ctx_version = 1;   // bumped whenever a table slab of this rank moves (alloc, rehash): peers' mappings are stale
};

struct Plan {
    Engine* e = nullptr;
    PlanDev d;
    char* meta = nullptr;   // small index arrays
    char* inbox = nullptr;  // keys | grads | cnt (peer mapped)
    size_t inbox_bytes = 0, inbox_grads_off = 0, inbox_cnt_off = 0;
    char* work = nullptr;   // send_cnt | parity | 2 x (ucount | cmap_keys | cmap_cnt | ulist | ukeys | slot_of | acc | urows)
    size_t inbox_vals_off = 0, work_bytes = 0;
    int grid_pull = 1, grid_push = 1, grid_pull2 = 1, grid_plan = 1;
    size_t smem_pull = 0, smem_push = 0, smem_pull2 = 0, smem_plan = 0;
};

int pow2_ceil_int(int x) { int p = 1; while (p < x) p <<= 1; return p; }
size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Context versioning (reference: pico-ps ctx version, Status SERVER_TOO_{NEW,OLD}_CTX): a rank announces its version
// into its own sync block and into every peer's (mapped) block; kernels compare the announced versions with the ones
// accepted at the last connect and raise EXB_ERR_CTX_VERSION on a mismatch (a peer moved a slab, this rank still
// holds the old mapping).
cudaError_t announce_ctx(Engine* e, int only_peer = -1) {
    for (int r = 0; r < e->world; ++r) {
        if (only_peer >= 0 && r != only_peer) continue;
        char* base = e->sync_peer[r];
        if (!base) continue;
        cudaError_t err = cudaMemcpy(base + OFF_CTX_ANNOUNCED + 4 * e->rank, &e->ctx_version, 4, cudaMemcpyDefault);
        if (err != cudaSuccess) return err;
    }
    return cudaSuccess;
}
cudaError_t bump_ctx(Engine* e) {
    ++e->ctx_version;
    return announce_ctx(e);
}
cudaError_t accept_own_ctx(Engine* e) {
    return cudaMemcpy(e->sync_local + OFF_CTX_EXPECTED + 4 * e->rank, &e->ctx_version, 4, cudaMemcpyHostToDevice);
}

// ------------------------------------------------------------ utility kernels
__global__ void fill_u64_kernel(unsigned long long* p, unsigned long long n, unsigned long long v) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x)
        p[i] = v;
}

// array table: materialise every local row with its Philox initial value
__global__ void array_fill_weights_kernel(TableDev T, int rank, int W) {
    const unsigned long long chunks = T.vec4 ? (unsigned long long)(T.wstride / 4) : 1ull;
    const unsigned long long total = T.rows * chunks;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < total;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned long long row = i / chunks;
        int c = (int)(i % chunks) * 4;
        unsigned long long id = row * (unsigned long long)T.shard_num + shard_of_rank(T, rank, W);
        float* wrow = T.w[rank] + row * T.wstride;
        if (T.vec4) {
            *reinterpret_cast<float4*>(wrow + c) = init_block_masked(&T.init, id, c, T.dim);
        } else {
            float t[4];
            InitGen<float>::block4(T.init, id, 0u, t);
            for (int k = 0; k < T.dim; ++k) wrow[k] = t[k & 3];
        }
    }
}

// (re)initialise the optimizer state of every row / slot
__global__ void fill_state_kernel(TableDev T) {
    const unsigned long long total = T.rows * (unsigned long long)T.sstride;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < total;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        int c = (int)(i % T.sstride);
        float v = 0.f;
        int slot_w = T.nslots * T.wstride;
        if (c < slot_w) v = opt_slot_init<float>(T.opt, c / T.wstride);
        else if (c - slot_w < T.nscalars) v = opt_scalar_init<float>(T.opt, c - slot_w);
        T.state[i] = v;
    }
}

// append the global ids of all materialised rows (array: touched bit, hash: occupied slot)
__global__ void enumerate_kernel(TableDev T, int rank, int W, unsigned long long* out,
                                 unsigned long long* counter, unsigned long long cap) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < T.rows;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned long long id = EXB_EMPTY_KEY;
        if (T.is_hash) {
            id = T.keys[rank][i];
        } else if ((T.touched[i >> 5] >> (i & 31)) & 1u) {
            id = i * (unsigned long long)T.shard_num + shard_of_rank(T, rank, W);
        }
        if (id != EXB_EMPTY_KEY) {
            unsigned long long pos = atomicAdd(counter, 1ull);
            if (pos < cap) out[pos] = id;
        }
    }
}

__device__ __forceinline__ long long resolve_local_row(const TableDev& T, int rank, int W,
                                                       unsigned long long id) {
    if (!T.is_hash) {
        if (id >= T.vocab || owner_of(T, id, W) != rank) return -1;
        return (long long)local_row_of(T, id);
    }
    if ((id >> 63) || owner_of(T, id, W) != rank) return -1;
    const unsigned long long* keys = T.keys[rank];
    unsigned long long mask = T.rows - 1, h = exb_hash64(id) & mask;
    for (unsigned long long probe = 0; probe <= mask; ++probe) {
        unsigned long long k = keys[h];
        if (k == id) return (long long)h;
        if (k == EXB_EMPTY_KEY) return -1;
        h = (h + 1) & mask;
    }
    return -1;
}

// one warp per requested id; state is re-packed to the reference layout
// [slot0[dim] | slot1[dim] | scalars] (EmbeddingOptimizer.h state_view order)
__global__ void gather_rows_kernel(TableDev T, int rank, int W, const unsigned long long* ids,
                                   unsigned long long n, float* w_out, float* s_out) {
    const int lane = threadIdx.x & 31;
    const unsigned long long warp = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const int sd = T.nslots * T.dim + T.nscalars;
    for (unsigned long long i = warp; i < n; i += nwarps) {
        unsigned long long id = ids[i];
        long long row = 0;
        if (lane == 0) row = resolve_local_row(T, rank, W, id);
        row = __shfl_sync(0xffffffffu, row, 0);
        if (row >= 0) {
            const float* wrow = T.w[rank] + (unsigned long long)row * T.wstride;
            const float* srow = T.state + (unsigned long long)row * T.sstride;
            for (int c = lane; c < T.dim; c += 32) w_out[i * T.dim + c] = wrow[c];
            if (s_out) {
                for (int s = 0; s < T.nslots; ++s)
                    for (int c = lane; c < T.dim; c += 32)
                        s_out[i * sd + s * T.dim + c] = srow[s * T.wstride + c];
                for (int c = lane; c < T.nscalars; c += 32)
                    s_out[i * sd + T.nslots * T.dim + c] = srow[T.nslots * T.wstride + c];
            }
        } else {
            for (int c = lane; c < T.dim; c += 32) {
                float t[4];
                InitGen<float>::block4(T.init, id, (uint32_t)(c >> 2), t);
                w_out[i * T.dim + c] = t[c & 3];
            }
            if (s_out) {
                for (int s = 0; s < T.nslots; ++s)
                    for (int c = lane; c < T.dim; c += 32)
                        s_out[i * sd + s * T.dim + c] = opt_slot_init<float>(T.opt, s);
                for (int c = lane; c < T.nscalars; c += 32)
                    s_out[i * sd + T.nslots * T.dim + c] = opt_scalar_init<float>(T.opt, c);
            }
        }
    }
}

// one warp per id (ids unique, all owned by this rank); inserts hash keys as needed
__global__ void scatter_rows_kernel(TableDev T, int rank, int W, const unsigned long long* ids,
                                    unsigned long long n, const float* w_in, const float* s_in,
                                    int* status) {
    const int lane = threadIdx.x & 31;
    const unsigned long long warp = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const int sd = T.nslots * T.dim + T.nscalars;
    for (unsigned long long i = warp; i < n; i += nwarps) {
        unsigned long long id = ids[i];
        long long row = -1;
        if (lane == 0) {
            if (!T.is_hash) {
                if (id < T.vocab && owner_of(T, id, W) == rank) {
                    row = (long long)local_row_of(T, id);
                    atomicOr(&T.touched[row >> 5], 1u << (row & 31));
                }
            } else if ((id >> 63) == 0 && owner_of(T, id, W) == rank) {
                unsigned long long* keys = const_cast<unsigned long long*>(T.keys[rank]);
                unsigned long long mask = T.rows - 1, h = exb_hash64(id) & mask;
                for (unsigned long long probe = 0; probe <= mask; ++probe) {
                    unsigned long long k = *(volatile unsigned long long*)&keys[h];
                    if (k == id) { row = (long long)h; break; }
                    if (k == EXB_EMPTY_KEY) {
                        unsigned long long prev = atomicCAS(&keys[h], EXB_EMPTY_KEY, id);
                        if (prev == EXB_EMPTY_KEY) { atomicAdd(T.size_ctr, 1ull); row = (long long)h; break; }
                        if (prev == id) { row = (long long)h; break; }
                    }
                    h = (h + 1) & mask;
                }
                if (row < 0) atomicCAS(status, 0, EXB_ERR_HASH_FULL);
            }
        }
        row = __shfl_sync(0xffffffffu, row, 0);
        if (row < 0) continue;
        float* wrow = T.w[rank] + (unsigned long long)row * T.wstride;
        float* srow = T.state + (unsigned long long)row * T.sstride;
        for (int c = lane; c < T.wstride; c += 32) wrow[c] = c < T.dim ? w_in[i * T.dim + c] : 0.f;
        for (int s = 0; s < T.nslots; ++s)
            for (int c = lane; c < T.wstride; c += 32) {
                float v = opt_slot_init<float>(T.opt, s);
                if (s_in && c < T.dim) v = s_in[i * sd + s * T.dim + c];
                srow[s * T.wstride + c] = v;
            }
        for (int c = lane; c < T.nscalars; c += 32)
            srow[T.nslots * T.wstride + c] =
                s_in ? s_in[i * sd + T.nslots * T.dim + c] : opt_scalar_init<float>(T.opt, c);
    }
}

// move every occupied slot of an old hash shard into a new (bigger) one
__global__ void rehash_kernel(const unsigned long long* okeys, const float* ow, const float* os,
                              unsigned long long ocap, TableDev N, int rank, int* status) {
    const int lane = threadIdx.x & 31;
    const unsigned long long warp = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    for (unsigned long long i = warp; i < ocap; i += nwarps) {
        unsigned long long key = okeys[i];
        if (key == EXB_EMPTY_KEY) continue;
        long long row = -1;
        if (lane == 0) {
            unsigned long long* keys = const_cast<unsigned long long*>(N.keys[rank]);
            unsigned long long mask = N.rows - 1, h = exb_hash64(key) & mask;
            for (unsigned long long probe = 0; probe <= mask; ++probe) {
                unsigned long long prev = atomicCAS(&keys[h], EXB_EMPTY_KEY, key);
                if (prev == EXB_EMPTY_KEY) { row = (long long)h; break; }
                h = (h + 1) & mask;
            }
            if (row < 0) atomicCAS(status, 0, EXB_ERR_HASH_FULL);
        }
        row = __shfl_sync(0xffffffffu, row, 0);
        if (row < 0) continue;
        for (int c = lane; c < N.wstride; c += 32)
            N.w[rank][(unsigned long long)row * N.wstride + c] = ow[i * N.wstride + c];
        for (int c = lane; c < N.sstride; c += 32)
            N.state[(unsigned long long)row * N.sstride + c] = os[i * N.sstride + c];
    }
}

void layout_table(TableDev& d) {
    d.nslots = opt_num_slots(d.opt.kind);
    d.nscalars = opt_num_scalars(d.opt.kind);
    if (d.dim >= 4) { d.wstride = (d.dim + 3) & ~3; d.vec4 = 1; }
    else { d.wstride = d.dim; d.vec4 = 0; }
    int st = d.nslots * d.wstride + d.nscalars;
    d.sstride = d.vec4 ? ((st + 3) & ~3) : st;
    if (d.sstride == 0) d.sstride = d.vec4 ? 4 : 1;  // keep a valid (tiny) allocation
    int chunks = d.vec4 ? d.wstride / 4 : 1;
    d.lpr = std::min(32, pow2_ceil_int(chunks));
}

int upload_tables(Engine* e) {
    size_t n = e->tables.size();
    if (n == 0) return 0;
    if (n > e->d_tables_cap) {
        if (e->d_tables) cudaFree(e->d_tables);
        e->d_tables_cap = std::max<size_t>(64, n * 2);
        CK(cudaMalloc(&e->d_tables, e->d_tables_cap * sizeof(TableDev)));
    }
    std::vector<TableDev> h(n);
    for (size_t i = 0; i < n; ++i) h[i] = e->tables[i].d;
    CK(cudaMemcpy(e->d_tables, h.data(), n * sizeof(TableDev), cudaMemcpyHostToDevice));
    return 0;
}

int alloc_state(Engine* e, HostTable& t) {
    if (t.d.state) { cudaFree(t.d.state); t.d.state = nullptr; }
    t.s_bytes = align_up((size_t)t.d.rows * t.d.sstride * sizeof(float), 256);
    CK(cudaMalloc(&t.d.state, t.s_bytes));
    fill_state_kernel<<<e->sms * 8, 256>>>(t.d);
    CK(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" {

const char* exb_cuda_last_error() { return g_err.c_str(); }

int exb_cuda_device_count() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

void* exb_engine_create(int device, int rank, int world) {
    if (world < 1 || world > EXB_MAX_PEERS || rank < 0 || rank >= world) {
        fail_msg("world size must be in [1, 8] for one NVSwitch box");
        return nullptr;
    }
    CKP(cudaSetDevice(device));
    Engine* e = new Engine();
    e->device = device; e->rank = rank; e->world = world;
    cudaDeviceProp prop;
    CKP(cudaGetDeviceProperties(&prop, device));
    e->sms = prop.multiProcessorCount;
    CKP(cudaMalloc(&e->sync_local, SYNC_BYTES));
    CKP(cudaMemset(e->sync_local, 0, SYNC_BYTES));
    for (int i = 0; i < EXB_MAX_PEERS; ++i) e->sync_peer[i] = nullptr;
    e->sync_peer[rank] = e->sync_local;
    if (announce_ctx(e) != cudaSuccess || accept_own_ctx(e) != cudaSuccess) { fail_msg("engine: context version"); return nullptr; }
    return e;
}
void exb_engine_destroy(void* h) {
    Engine* e = (Engine*)h;
    cudaSetDevice(e->device);
    for (HostTable& t : e->tables) {
        if (t.w_local) cudaFree(t.w_local);
        if (t.keys_local) cudaFree(t.keys_local);
        if (t.d.state) cudaFree(t.d.state);
        if (t.d.touched) cudaFree(t.d.touched);
        if (t.d.size_ctr) cudaFree(t.d.size_ctr);
    }
    if (e->d_tables) cudaFree(e->d_tables);
    if (e->sync_local) cudaFree(e->sync_local);
    delete e;
}
int exb_engine_sms(void* h) { return ((Engine*)h)->sms; }
void exb_engine_set_max_ctas(void* h, int n) { ((Engine*)h)->max_ctas = n; }
uint64_t exb_engine_sync_ptr(void* h) { return (uint64_t)((Engine*)h)->sync_local; }
uint64_t exb_engine_sync_bytes() { return SYNC_BYTES; }
void exb_engine_set_peer_sync(void* h, int peer, uint64_t ptr) {
    Engine* e = (Engine*)h;
    e->sync_peer[peer] = (char*)ptr;
    cudaSetDevice(e->device);
    announce_ctx(e, peer);       // the newly mapped peer learns this rank's current context version
}
// accept every rank's announced context version as the one this rank's mappings are built against. Collective
// protocol (ops/sparse_engine.py: connect): all ranks have exchanged their mappings, a barrier, then this call.
int exb_engine_accept_ctx(void* h) {
    Engine* e = (Engine*)h;
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(e->sync_local + OFF_CTX_EXPECTED, e->sync_local + OFF_CTX_ANNOUNCED, 4 * EXB_MAX_PEERS, cudaMemcpyDeviceToDevice));
    return 0;
}
unsigned exb_engine_ctx_version(void* h) { return ((Engine*)h)->ctx_version; }

// returns 0 and the error status word (device sync!)
int exb_engine_status(void* h, int* status, uint64_t* stats16) {
    Engine* e = (Engine*)h;
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(status, e->sync_local + OFF_STATUS, 4, cudaMemcpyDeviceToHost));
    if (stats16) CK(cudaMemcpy(stats16, e->sync_local + OFF_STATS, 256, cudaMemcpyDeviceToHost));
    return 0;
}
int exb_engine_reset_status(void* h) {
    Engine* e = (Engine*)h;
    CK(cudaSetDevice(e->device));
    CK(cudaMemset(e->sync_local + OFF_STATUS, 0, 4));
    return 0;
}

// ---- tables
int exb_table_add(void* h, int is_hash, int dim, uint64_t vocab, uint64_t capacity, int shard_num, int shard_base) {
    Engine* e = (Engine*)h;
    HostTable t;
    memset(&t.d, 0, sizeof(TableDev));
    t.d.dim = dim; t.d.is_hash = is_hash ? 1 : 0;
    t.d.vocab = is_hash ? (1ull << 63) : vocab;
    if (is_hash) {
        unsigned long long cap = 1024;
        while (cap < capacity) cap <<= 1;
        t.d.rows = cap;
    } else {
        t.d.rows = 0;
    }
    if (shard_num <= 0 || shard_num > e->world) shard_num = e->world;
    t.d.shard_num = shard_num;
    t.d.shard_base = ((shard_base % e->world) + e->world) % e->world;
    {
        int my_shard = (e->rank - t.d.shard_base + e->world) % e->world;
        bool owner = my_shard < shard_num;
        if (!is_hash) t.d.rows = owner ? (vocab + shard_num - 1) / shard_num : 1;
        // hash shards keep a symmetric capacity: peers probe the owner's slab with T.rows
        if (t.d.rows == 0) t.d.rows = 1;
    }
    t.d.init.kind = INIT_CONSTANT; t.d.init.p[0] = t.d.init.p[1] = t.d.init.p[2] = 0; t.d.init.seed = 0;
    t.d.opt.kind = OPT_DEFAULT; for (double& v : t.d.opt.p) v = 0;
    layout_table(t.d);
    e->tables.push_back(t);
    return (int)e->tables.size() - 1;
}
int exb_table_set_initializer(void* h, int t, int kind, double p0, double p1, double p2, uint64_t seed) {
    Engine* e = (Engine*)h;
    InitParams& I = e->tables[t].d.init;
    I.kind = kind; I._pad = 0; I.p[0] = p0; I.p[1] = p1; I.p[2] = p2; I.seed = seed;
    return 0;
}
// May be called before or after allocation; a category change re-initialises the state
// (reference: EmbeddingVariable.cpp:44-47).
int exb_table_set_optimizer(void* h, int ti, int kind, const double* p, int np) {
    Engine* e = (Engine*)h;
    HostTable& t = e->tables[ti];
    CK(cudaSetDevice(e->device));
    bool changed = !t.opt_set || kind != t.d.opt.kind;
    t.d.opt.kind = kind; t.d.opt._pad = 0;
    for (int i = 0; i < 8; ++i) t.d.opt.p[i] = i < np ? p[i] : 0.0;
    t.opt_set = true;
    if (changed) {
        layout_table(t.d);
        if (t.allocated) { if (alloc_state(e, t)) return -1; }
    }
    return 0;
}
int exb_table_alloc(void* h, int ti) {
    Engine* e = (Engine*)h;
    HostTable& t = e->tables[ti];
    CK(cudaSetDevice(e->device));
    if (t.allocated) return 0;
    CK(bump_ctx(e));
    layout_table(t.d);
    t.w_bytes = align_up((size_t)t.d.rows * t.d.wstride * sizeof(float), 2u << 20);
    CK(cudaMalloc(&t.w_local, t.w_bytes));
    t.d.w[e->rank] = t.w_local;
    if (t.d.is_hash) {
        t.k_bytes = align_up((size_t)t.d.rows * 8, 2u << 20);
        CK(cudaMalloc(&t.keys_local, t.k_bytes));
        fill_u64_kernel<<<e->sms * 4, 256>>>(t.keys_local, t.d.rows, EXB_EMPTY_KEY);
        t.d.keys[e->rank] = t.keys_local;
        CK(cudaMalloc(&t.d.size_ctr, 256));
        CK(cudaMemset(t.d.size_ctr, 0, 256));
        CK(cudaMemset(t.w_local, 0, t.w_bytes));
    } else {
        t.t_bytes = align_up((size_t)(t.d.rows + 31) / 32 * 4, 256);
        CK(cudaMalloc(&t.d.touched, t.t_bytes));
        CK(cudaMemset(t.d.touched, 0, t.t_bytes));
        if (t.d.init.kind == INIT_CONSTANT && t.d.init.p[0] == 0.0) {
            CK(cudaMemset(t.w_local, 0, t.w_bytes));
        } else {
            array_fill_weights_kernel<<<e->sms * 8, 256>>>(t.d, e->rank, e->world);
        }
    }
    CK(cudaGetLastError());
    if (alloc_state(e, t)) return -1;
    t.allocated = true;
    return 0;
}
// out[0]=w ptr, out[1]=w bytes, out[2]=keys ptr, out[3]=keys bytes, out[4]=rows, out[5]=wstride, out[6]=sstride
int exb_table_info(void* h, int ti, uint64_t* out) {
    HostTable& t = ((Engine*)h)->tables[ti];
    out[0] = (uint64_t)t.w_local; out[1] = t.w_bytes; out[2] = (uint64_t)t.keys_local; out[3] = t.k_bytes;
    out[4] = t.d.rows; out[5] = (uint64_t)t.d.wstride; out[6] = (uint64_t)t.d.sstride;
    out[7] = (uint64_t)(t.d.nslots * t.d.dim + t.d.nscalars);
    return 0;
}
int exb_table_set_peer(void* h, int ti, int peer, uint64_t w_ptr, uint64_t keys_ptr) {
    HostTable& t = ((Engine*)h)->tables[ti];
    t.d.w[peer] = (float*)w_ptr;
    t.d.keys[peer] = (const unsigned long long*)keys_ptr;
    return 0;
}
int exb_engine_commit(void* h) {
    Engine* e = (Engine*)h;
    CK(cudaSetDevice(e->device));
    CK(accept_own_ctx(e));        // the device table descriptors are refreshed below: this rank's own view is current
    return upload_tables(e);
}
int exb_table_size(void* h, int ti, uint64_t* out) {
    Engine* e = (Engine*)h;
    HostTable& t = e->tables[ti];
    CK(cudaSetDevice(e->device));
    if (t.d.is_hash) {
        CK(cudaMemcpy(out, t.d.size_ctr, 8, cudaMemcpyDeviceToHost));
    } else {
        *out = t.d.rows;
    }
    return 0;
}
// writes up to cap global ids of materialised rows into out_dev; *n_out = total found
int exb_table_enumerate(void* h, int ti, uint64_t out_dev, uint64_t cap, uint64_t* n_out, uint64_t stream) {
    Engine* e = (Engine*)h;
    HostTable& t = e->tables[ti];
    CK(cudaSetDevice(e->device));
    unsigned long long* ctr;
    CK(cudaMalloc(&ctr, 8));
    CK(cudaMemsetAsync(ctr, 0, 8, (cudaStream_t)stream));
    enumerate_kernel<<<e->sms * 8, 256, 0, (cudaStream_t)stream>>>(t.d, e->rank, e->world,
                                                                   (unsigned long long*)out_dev, ctr, cap);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(n_out, ctr, 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CK(cudaStreamSynchronize((cudaStream_t)stream));
    cudaFree(ctr);
    return 0;
}
int exb_table_gather(void* h, int ti, uint64_t ids_dev, uint64_t n, uint64_t w_out, uint64_t s_out, uint64_t stream) {
    Engine* e = (Engine*)h;
    HostTable& t = e->tables[ti];
    CK(cudaSetDevice(e->device));
    if (n == 0) return 0;
    int grid = (int)std::min<uint64_t>((n + 7) / 8, (uint64_t)e->sms * 8);
    gather_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(t.d, e->rank, e->world,
        (const unsigned long long*)ids_dev, n, (float*)w_out, (float*)s_out);
    CK(cudaGetLastError());
    return 0;
}
int exb_table_scatter(void* h, int ti, uint64_t ids_dev, uint64_t n, uint64_t w_in, uint64_t s_in, uint64_t stream) {
    Engine* e = (Engine*)h;
    HostTable& t = e->tables[ti];
    CK(cudaSetDevice(e->device));
    if (n == 0) return 0;
    int grid = (int)std::min<uint64_t>((n + 7) / 8, (uint64_t)e->sms * 8);
    scatter_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(t.d, e->rank, e->world,
        (const unsigned long long*)ids_dev, n, (const float*)w_in, (const float*)s_in,
        (int*)(e->sync_local + OFF_STATUS));
    CK(cudaGetLastError());
    return 0;
}
// drop all rows (array: re-fill initial values, hash: empty) -- used by load_model
int exb_table_clear(void* h, int ti) {
    Engine* e = (Engine*)h;
    HostTable& t = e->tables[ti];
    CK(cudaSetDevice(e->device));
    if (!t.allocated) return 0;
    if (t.d.is_hash) {
        fill_u64_kernel<<<e->sms * 4, 256>>>(t.keys_local, t.d.rows, EXB_EMPTY_KEY);
        CK(cudaMemset(t.d.size_ctr, 0, 8));
    } else {
        CK(cudaMemset(t.d.touched, 0, t.t_bytes));
        if (t.d.init.kind == INIT_CONSTANT && t.d.init.p[0] == 0.0) CK(cudaMemset(t.w_local, 0, t.w_bytes));
        else array_fill_weights_kernel<<<e->sms * 8, 256>>>(t.d, e->rank, e->world);
    }
    fill_state_kernel<<<e->sms * 8, 256>>>(t.d);
    CK(cudaGetLastError());
    return 0;
}
// grow a hash shard to new_capacity (pow2). Peers must re-import the new slabs afterwards.
int exb_table_rehash(void* h, int ti, uint64_t new_capacity) {
    Engine* e = (Engine*)h;
    HostTable& t = e->tables[ti];
    CK(cudaSetDevice(e->device));
    if (!t.d.is_hash || !t.allocated) return fail_msg("rehash: not an allocated hash table");
    unsigned long long cap = 1024;
    while (cap < new_capacity) cap <<= 1;
    if (cap <= t.d.rows) return 0;
    HostTable n = t;
    n.d.rows = cap;
    n.w_bytes = align_up((size_t)cap * n.d.wstride * sizeof(float), 2u << 20);
    n.k_bytes = align_up((size_t)cap * 8, 2u << 20);
    n.s_bytes = align_up((size_t)cap * n.d.sstride * sizeof(float), 256);
    CK(cudaMalloc(&n.w_local, n.w_bytes));
    CK(cudaMemset(n.w_local, 0, n.w_bytes));
    CK(cudaMalloc(&n.keys_local, n.k_bytes));
    CK(cudaMalloc(&n.d.state, n.s_bytes));
    fill_u64_kernel<<<e->sms * 4, 256>>>(n.keys_local, cap, EXB_EMPTY_KEY);
    n.d.w[e->rank] = n.w_local;
    n.d.keys[e->rank] = n.keys_local;
    fill_state_kernel<<<e->sms * 8, 256>>>(n.d);
    rehash_kernel<<<e->sms * 8, 256>>>(t.keys_local, t.w_local, t.d.state, t.d.rows, n.d, e->rank,
                                       (int*)(e->sync_local + OFF_STATUS));
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    cudaFree(t.w_local); cudaFree(t.keys_local); cudaFree(t.d.state);
    for (int p = 0; p < EXB_MAX_PEERS; ++p)
        if (p != e->rank) { n.d.w[p] = nullptr; n.d.keys[p] = nullptr; }
    t = n;
    CK(bump_ctx(e));              // peers still map the freed slabs: their kernels must notice until they reconnect
    return 0;
}

// ---- raw (cudaMalloc-owned, IPC-exportable) buffers for python-side peer-mapped tensors
uint64_t exb_raw_alloc(int device, uint64_t nbytes) {
    if (cudaSetDevice(device) != cudaSuccess) return 0;
    void* p = nullptr;
    nbytes = align_up(nbytes, 2u << 20);
    cudaError_t err = cudaMalloc(&p, nbytes);
    if (err != cudaSuccess) { fail("cudaMalloc", err); return 0; }
    cudaMemset(p, 0, nbytes);
    cudaDeviceSynchronize();
    return (uint64_t)p;
}
int exb_raw_free(uint64_t ptr) { CK(cudaFree((void*)ptr)); return 0; }

// ---- IPC
int exb_ipc_get_handle(uint64_t ptr, char* out64) {
    cudaIpcMemHandle_t hdl;
    CK(cudaIpcGetMemHandle(&hdl, (void*)ptr));
    memcpy(out64, &hdl, sizeof(hdl));
    return 0;
}
uint64_t exb_ipc_open_handle(const char* in64) {
    cudaIpcMemHandle_t hdl;
    memcpy(&hdl, in64, sizeof(hdl));
    void* p = nullptr;
    cudaError_t err = cudaIpcOpenMemHandle(&p, hdl, cudaIpcMemLazyEnablePeerAccess);
    if (err != cudaSuccess) { fail("cudaIpcOpenMemHandle", err); return 0; }
    return (uint64_t)p;
}
int exb_ipc_close_handle(uint64_t ptr) { CK(cudaIpcCloseMemHandle((void*)ptr)); return 0; }
int exb_enable_peer_access(int device, int peer_device) {
    CK(cudaSetDevice(device));
    int can = 0;
    CK(cudaDeviceCanAccessPeer(&can, device, peer_device));
    if (!can) return fail_msg("peer access not supported between devices");
    cudaError_t err = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (err != cudaSuccess && err != cudaErrorPeerAccessAlreadyEnabled) return fail("cudaDeviceEnablePeerAccess", err);
    cudaGetLastError();
    return 0;
}

// ---- plans
// feat_off2 / feat_split (both may be null): split-row features, see pull_rows_split in bulk_rows.cuh
void* exb_plan_create2(void* h, int F, const int* feat_table, const int* feat_off, const int* feat_col, int ncols,
                       int B, int io_stride, const int* feat_off2, const int* feat_split) {
    Engine* e = (Engine*)h;
    CKP(cudaSetDevice(e->device));
    const int W = e->world;
    std::vector<int> pt_table, feat_pt(F);
    for (int f = 0; f < F; ++f) {
        int t = feat_table[f];
        if (t < 0 || t >= (int)e->tables.size() || !e->tables[t].allocated) { fail_msg("plan: bad table id or table not allocated"); return nullptr; }
        auto it = std::find(pt_table.begin(), pt_table.end(), t);
        if (it == pt_table.end()) { pt_table.push_back(t); feat_pt[f] = (int)pt_table.size() - 1; }
        else feat_pt[f] = (int)(it - pt_table.begin());
    }
    const int PT = (int)pt_table.size();
    if (PT > 128 || W * PT > EXB_MAX_SEG) { fail_msg("plan: too many tables for one plan (max 128)"); return nullptr; }
    std::vector<int> off2(F, 0), split(F, 0x7fffffff);
    for (int f = 0; f < F; ++f) {
        if (!feat_split || !feat_off2) break;
        const TableDev& T = e->tables[feat_table[f]].d;
        if (feat_split[f] <= 0 || feat_split[f] >= T.dim) continue;
        if (!T.vec4 || T.wstride * 4 > (int)EXB_PULL_WARP_BUF) { fail_msg("plan: a split-row feature needs 4 <= dim <= 2048"); return nullptr; }
        off2[f] = feat_off2[f]; split[f] = feat_split[f];
    }
    Plan* p = new Plan();
    p->e = e;
    PlanDev& d = p->d;
    memset(&d, 0, sizeof(d));
    d.F = F; d.B = B; d.PT = PT; d.W = W; d.rank = e->rank; d.io_stride = io_stride; d.ncols = ncols;
    std::vector<unsigned> pt_cap(PT, 0);
    std::vector<int> task_prefix(F + 1, 0);
    for (int f = 0; f < F; ++f) { pt_cap[feat_pt[f]] += (unsigned)B; task_prefix[f + 1] = task_prefix[f] + (B + 31) / 32; }
    d.num_tasks = task_prefix[F];
    std::vector<unsigned long long> key_off(PT), grad_off(PT), map_off(PT), acc_off(PT), ulist_off(PT);
    std::vector<unsigned> map_mask(PT);
    unsigned long long ko = 0, go = 0, mo = 0, ao = 0, uo = 0;
    for (int i = 0; i < PT; ++i) {
        const TableDev& T = e->tables[pt_table[i]].d;
        key_off[i] = ko; grad_off[i] = go;
        ko += pt_cap[i]; go += (unsigned long long)pt_cap[i] * T.wstride;
        go = (go + 3) & ~3ull;
        unsigned long long need = 2ull * W * pt_cap[i];
        unsigned long long cap = 64; while (cap < need) cap <<= 1;
        map_off[i] = mo; map_mask[i] = (unsigned)(cap - 1); acc_off[i] = ao; ulist_off[i] = uo;
        mo += cap; ao += cap * T.wstride; ao = (ao + 3) & ~3ull; uo += (unsigned long long)W * pt_cap[i];
    }
    d.src_key_stride = ko; d.src_grad_stride = go;
    // ---- meta buffer
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 16); return o; };
    size_t o_feat_col = take(F * 4), o_feat_off2 = take(F * 4), o_feat_split = take(F * 4);
    size_t o_feat_pt = take(F * 4), o_feat_off = take(F * 4), o_prefix = take((F + 1) * 4), o_pt_table = take(PT * 4),
           o_cap = take(PT * 4), o_koff = take(PT * 8), o_goff = take(PT * 8), o_moff = take(PT * 8),
           o_mask = take(PT * 4), o_aoff = take(PT * 8), o_uoff = take(PT * 8);
    std::vector<char> hm(off);
    memcpy(&hm[o_feat_pt], feat_pt.data(), F * 4); memcpy(&hm[o_feat_off], feat_off, F * 4);
    memcpy(&hm[o_feat_col], feat_col, F * 4);
    memcpy(&hm[o_feat_off2], off2.data(), F * 4); memcpy(&hm[o_feat_split], split.data(), F * 4);
    memcpy(&hm[o_prefix], task_prefix.data(), (F + 1) * 4); memcpy(&hm[o_pt_table], pt_table.data(), PT * 4);
    memcpy(&hm[o_cap], pt_cap.data(), PT * 4); memcpy(&hm[o_koff], key_off.data(), PT * 8);
    memcpy(&hm[o_goff], grad_off.data(), PT * 8); memcpy(&hm[o_moff], map_off.data(), PT * 8);
    memcpy(&hm[o_mask], map_mask.data(), PT * 4); memcpy(&hm[o_aoff], acc_off.data(), PT * 8);
    memcpy(&hm[o_uoff], ulist_off.data(), PT * 8);
    CKP(cudaMalloc(&p->meta, off));
    CKP(cudaMemcpy(p->meta, hm.data(), off, cudaMemcpyHostToDevice));
    d.feat_pt = (const int*)(p->meta + o_feat_pt); d.feat_off = (const int*)(p->meta + o_feat_off);
    d.feat_col = (const int*)(p->meta + o_feat_col);
    d.feat_off2 = (const int*)(p->meta + o_feat_off2); d.feat_split = (const int*)(p->meta + o_feat_split);
    d.task_prefix = (const int*)(p->meta + o_prefix); d.pt_table = (const int*)(p->meta + o_pt_table);
    d.pt_cap = (const unsigned*)(p->meta + o_cap);
    d.pt_key_off = (const unsigned long long*)(p->meta + o_koff);
    d.pt_grad_off = (const unsigned long long*)(p->meta + o_goff);
    d.pt_map_off = (const unsigned long long*)(p->meta + o_moff);
    d.pt_map_mask = (const unsigned*)(p->meta + o_mask);
    d.pt_acc_off = (const unsigned long long*)(p->meta + o_aoff);
    d.pt_ulist_off = (const unsigned long long*)(p->meta + o_uoff);
    // ---- inbox (peer visible): keys | grads | cnt
    size_t kb = align_up((size_t)W * ko * 8, 256), gb = align_up((size_t)W * go * 4, 256), cb = align_up((size_t)W * PT * 4, 256);
    size_t vb = align_up((size_t)W * ko * 4, 256);
    if (W == 1) { kb = 256; gb = 256; vb = 256; }
    p->inbox_grads_off = kb; p->inbox_cnt_off = kb + gb; p->inbox_vals_off = kb + gb + cb;
    p->inbox_bytes = align_up(kb + gb + cb + vb, 2u << 20);
    CKP(cudaMalloc(&p->inbox, p->inbox_bytes));
    CKP(cudaMemset(p->inbox + p->inbox_cnt_off, 0, cb));
    d.inbox_keys[e->rank] = (unsigned long long*)p->inbox;
    d.inbox_grads[e->rank] = (float*)(p->inbox + p->inbox_grads_off);
    d.inbox_cnt[e->rank] = (unsigned*)(p->inbox + p->inbox_cnt_off);
    d.inbox_vals[e->rank] = (unsigned*)(p->inbox + p->inbox_vals_off);
    // ---- local work: send_cnt | parity | 2 slots x (ucount | cmap_keys | cmap_cnt | ulist | ukeys | slot_of | acc | urows)
    size_t woff = 0;
    auto wtake = [&](size_t bytes) { size_t o = woff; woff = align_up(woff + bytes, 256); return o; };
    size_t o_send = wtake((size_t)W * PT * 4 * EXB_CTR_STRIDE), o_par = wtake(256);
    size_t o_ucount[2], o_ckeys[2], o_ccnt[2], o_ulist[2], o_ukeys[2], o_slotof[2], o_acc[2], o_urows[2];
    size_t o_ocount[2], o_olist[2], o_okeys[2];
    for (int s = 0; s < 2; ++s) {
        o_ucount[s] = wtake((size_t)PT * 4 * EXB_CTR_STRIDE); o_ckeys[s] = wtake(mo * 8); o_ccnt[s] = wtake(mo * 4);
        o_ulist[s] = wtake(uo * 4); o_ukeys[s] = wtake(uo * 8); o_slotof[s] = wtake((size_t)F * B * 4);
        o_acc[s] = wtake(ao * 4); o_urows[s] = wtake(W > 1 ? ao * 4 : 256);
        o_ocount[s] = wtake((size_t)PT * 4 * EXB_CTR_STRIDE);
        o_olist[s] = wtake(W > 1 ? uo * 4 : 256); o_okeys[s] = wtake(W > 1 ? uo * 8 : 256);
    }
    p->work_bytes = woff;
    CKP(cudaMalloc(&p->work, woff));
    CKP(cudaMemset(p->work, 0, woff));
    for (int s = 0; s < 2; ++s) {
        fill_u64_kernel<<<e->sms * 4, 256>>>((unsigned long long*)(p->work + o_ckeys[s]), mo, EXB_EMPTY_KEY);
        CKP(cudaGetLastError());
        SlotDev& L = d.slot[s];
        L.ucount = (unsigned*)(p->work + o_ucount[s]); L.cmap_keys = (unsigned long long*)(p->work + o_ckeys[s]);
        L.cmap_cnt = (unsigned*)(p->work + o_ccnt[s]); L.ulist = (unsigned*)(p->work + o_ulist[s]);
        L.ukeys = (unsigned long long*)(p->work + o_ukeys[s]); L.slot_of = (unsigned*)(p->work + o_slotof[s]);
        L.acc = (float*)(p->work + o_acc[s]); L.urows = (float*)(p->work + o_urows[s]);
        L.ocount = (unsigned*)(p->work + o_ocount[s]); L.olist = (unsigned*)(p->work + o_olist[s]);
        L.okeys = (unsigned long long*)(p->work + o_okeys[s]);
    }
    d.send_cnt = (unsigned*)(p->work + o_send); d.parity = (unsigned*)(p->work + o_par);
    // the v1 kernels work on slot 0
    d.ucount = d.slot[0].ucount; d.cmap_keys = d.slot[0].cmap_keys; d.cmap_cnt = d.slot[0].cmap_cnt;
    d.ulist = d.slot[0].ulist; d.ukeys = d.slot[0].ukeys; d.acc = d.slot[0].acc;
    // ---- sync words
    for (int r = 0; r < W; ++r) d.flags[r] = (unsigned*)(e->sync_peer[r] + OFF_FLAGS);
    d.gbar = (unsigned*)(e->sync_local + OFF_GBAR);
    d.epoch = (unsigned*)(e->sync_local + OFF_EPOCH);
    d.status = (int*)(e->sync_local + OFF_STATUS);
    d.stats = (unsigned long long*)(e->sync_local + OFF_STATS);
    d.trace = nullptr;
    // ---- launch geometry: persistent push kernel must be fully resident
    p->smem_pull = exb_smem_total(PT, F, false);
    p->smem_push = exb_smem_total(PT, F, true);
    {
        const char* eb = getenv("EXB_BULK");
        d.use_bulk = (eb && eb[0] == '0') ? 0 : 1;
    }
    cudaFuncSetAttribute(exb_pull_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(exb_push_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    int occ = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, exb_push_update_kernel, 256, p->smem_push);
    if (occ < 1) occ = 1;
    int per_sm = std::min(occ, 4);
    if (const char* ev = getenv("EXB_PUSH_CTAS_PER_SM")) per_sm = std::max(1, std::min(per_sm, atoi(ev)));
    int resident = e->sms * per_sm;
    int want = std::max(1, (d.num_tasks * std::max(1, W / 2 + 1) + 7) / 8);
    p->grid_push = std::min(resident, want);
    int occ_pull = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_pull, exb_pull_kernel, 256, p->smem_pull);
    if (occ_pull < 1) occ_pull = 1;
    p->grid_pull = std::max(1, std::min(e->sms * occ_pull, (d.num_tasks + 7) / 8));
    // ---- v2 kernels (sparse_v2.cuh)
    p->smem_plan = exb_smem_bytes(PT, F, false);
    p->smem_pull2 = exb_smem_bytes(PT, F, true) + 8 * (size_t)EXB_PULL_WARP_BUF;
    cudaFuncSetAttribute(exb_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(exb_pull2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(exb_pull_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(exb_push2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    p->grid_plan = std::max(1, (d.num_tasks + 7) / 8);
    {
        int occ2 = 1;      // the pull2 kernel contains a grid barrier: all CTAs resident
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ2, exb_pull2_kernel, 256, p->smem_pull2);
        occ2 = std::max(1, std::min(occ2, 2));
        p->grid_pull2 = std::max(1, std::min(e->sms * occ2, (d.num_tasks + 7) / 8));
        int occ3 = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ3, exb_push2_kernel, 256, p->smem_push);
        if (occ3 < per_sm) p->grid_push = std::min(p->grid_push, e->sms * std::max(1, occ3));
    }
    if (e->max_ctas > 0) {
        p->grid_push = std::min(p->grid_push, e->max_ctas); p->grid_pull = std::min(p->grid_pull, e->max_ctas);
        p->grid_pull2 = std::min(p->grid_pull2, e->max_ctas); p->grid_plan = std::min(p->grid_plan, 4 * e->max_ctas);
    }
    CKP(cudaDeviceSynchronize());
    return p;
}
void* exb_plan_create(void* h, int F, const int* feat_table, const int* feat_off, const int* feat_col, int ncols,
                      int B, int io_stride) {
    return exb_plan_create2(h, F, feat_table, feat_off, feat_col, ncols, B, io_stride, nullptr, nullptr);
}
void exb_plan_destroy(void* ph) {
    Plan* p = (Plan*)ph;
    cudaSetDevice(p->e->device);
    cudaFree(p->meta); cudaFree(p->inbox); cudaFree(p->work);
    delete p;
}
// out: [0]=inbox base, [1]=inbox bytes
int exb_plan_inbox_info(void* ph, uint64_t* out) {
    Plan* p = (Plan*)ph;
    out[0] = (uint64_t)p->inbox; out[1] = p->inbox_bytes;
    return 0;
}
int exb_plan_set_peer_inbox(void* ph, int peer, uint64_t base) {
    Plan* p = (Plan*)ph;
    p->d.inbox_keys[peer] = (unsigned long long*)base;
    p->d.inbox_grads[peer] = (float*)((char*)base + p->inbox_grads_off);
    p->d.inbox_cnt[peer] = (unsigned*)((char*)base + p->inbox_cnt_off);
    p->d.inbox_vals[peer] = (unsigned*)((char*)base + p->inbox_vals_off);
    return 0;
}
// refresh flag pointers after peers' sync blocks were imported
int exb_plan_commit(void* ph) {
    Plan* p = (Plan*)ph;
    Engine* e = p->e;
    for (int r = 0; r < e->world; ++r) {
        if (!e->sync_peer[r]) return fail_msg("plan commit: peer sync block not mapped");
        p->d.flags[r] = (unsigned*)(e->sync_peer[r] + OFF_FLAGS);
        if (e->world > 1 && (!p->d.inbox_keys[r])) return fail_msg("plan commit: peer inbox not mapped");
    }
    return 0;
}
// per-warp phase trace of the push kernel: buffer of grid_push*8*EXB_TRACE_SLOTS u64 (0 = off)
int exb_plan_set_trace(void* ph, uint64_t ptr) { ((Plan*)ph)->d.trace = (unsigned long long*)ptr; return 0; }
int exb_plan_grid(void* ph, int which) { Plan* p = (Plan*)ph; return which ? p->grid_push : p->grid_pull; }

int exb_pull(void* ph, uint64_t ids, uint64_t out, int n_rows, uint64_t stream) {
    Plan* p = (Plan*)ph;
    Engine* e = p->e;
    if (n_rows > p->d.B) return fail_msg("pull: n_rows exceeds plan batch");
    CK(launch_pdl(exb_pull_kernel, dim3(p->grid_pull), dim3(256), p->smem_pull, (cudaStream_t)stream,
                  (const TableDev*)e->d_tables, p->d, (const long long*)ids, (float*)out, n_rows));
    return 0;
}
// Attach (n > 0) or detach (n == 0) a dense-gradient all-reduce to this plan's push kernels: bufs[r] is rank r's
// flat fp32 gradient buffer as mapped into this process (P2PAllReduce), n its length in floats (multiple of 4).
// Every rank must attach the same n before its next push; the push then leaves the summed gradients in every buffer.
int exb_plan_set_dense_reduce(void* ph, const uint64_t* bufs, uint64_t n) {
    Plan* p = (Plan*)ph;
    if (n % 4) return fail_msg("dense reduce: length must be a multiple of 4 floats");
    for (int r = 0; r < EXB_MAX_PEERS; ++r) p->d.ar_buf[r] = (n && r < p->d.W) ? (float*)bufs[r] : nullptr;
    for (int r = 0; r < p->d.W && n; ++r)
        if (!p->d.ar_buf[r]) return fail_msg("dense reduce: peer buffer not mapped");
    p->d.ar_n = p->d.W > 1 ? n : 0;
    return 0;
}
int exb_push_update(void* ph, uint64_t ids, uint64_t grads, int n_rows, uint64_t stream) {
    Plan* p = (Plan*)ph;
    Engine* e = p->e;
    if (n_rows > p->d.B) return fail_msg("push: n_rows exceeds plan batch");
    CK(launch_pdl(exb_push_update_kernel, dim3(p->grid_push), dim3(256), p->smem_push, (cudaStream_t)stream,
                  (const TableDev*)e->d_tables, p->d, (const long long*)ids, (const float*)grads, n_rows));
    return 0;
}

// ---- v2: plan once per step (sparse_v2.cuh). which: 0 = current slot, 1 = next slot (prefetch)
int exb_plan_prepare(void* ph, uint64_t ids, int n_rows, int which, uint64_t stream) {
    Plan* p = (Plan*)ph;
    Engine* e = p->e;
    if (n_rows > p->d.B) return fail_msg("prepare: n_rows exceeds plan batch");
    CK(launch_pdl(exb_plan_kernel, dim3(p->grid_plan), dim3(256), p->smem_plan, (cudaStream_t)stream,
                  (const TableDev*)e->d_tables, p->d, (const long long*)ids, n_rows, which));
    return 0;
}
int exb_plan_reset(void* ph, int which, uint64_t stream) {
    Plan* p = (Plan*)ph;
    exb_plan_reset_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(p->d, which);
    CK(cudaGetLastError());
    return 0;
}
int exb_pull2(void* ph, uint64_t ids, uint64_t out, int n_rows, int which, uint64_t stream) {
    Plan* p = (Plan*)ph;
    Engine* e = p->e;
    if (n_rows > p->d.B) return fail_msg("pull: n_rows exceeds plan batch");
    CK(launch_pdl(exb_pull2_kernel, dim3(p->grid_pull2), dim3(256), p->smem_pull2, (cudaStream_t)stream,
                  (const TableDev*)e->d_tables, p->d, (const long long*)ids, (float*)out, n_rows, which));
    return 0;
}
// training pull: one-pass gather + plan of the batch in the same launch (exb_pull_plan_kernel)
int exb_pull_plan(void* ph, uint64_t ids, uint64_t out, int n_rows, int which, uint64_t stream) {
    Plan* p = (Plan*)ph;
    Engine* e = p->e;
    if (n_rows > p->d.B) return fail_msg("pull: n_rows exceeds plan batch");
    CK(launch_pdl(exb_pull_plan_kernel, dim3(p->grid_pull), dim3(256), p->smem_pull, (cudaStream_t)stream,
                  (const TableDev*)e->d_tables, p->d, (const long long*)ids, (float*)out, n_rows, which));
    return 0;
}
int exb_push2(void* ph, uint64_t grads, int n_rows, int which, uint64_t stream) {
    Plan* p = (Plan*)ph;
    Engine* e = p->e;
    if (n_rows > p->d.B) return fail_msg("push: n_rows exceeds plan batch");
    CK(launch_pdl(exb_push2_kernel, dim3(p->grid_push), dim3(256), p->smem_push, (cudaStream_t)stream,
                  (const TableDev*)e->d_tables, p->d, (const float*)grads, n_rows, which));
    return 0;
}
// bytes of device memory held by a plan: out[0] = peer-visible inbox, out[1] = local work area (both slots)
int exb_plan_memory(void* ph, uint64_t* out) {
    Plan* p = (Plan*)ph;
    out[0] = p->inbox_bytes; out[1] = p->work_bytes;
    return 0;
}
uint64_t exb_engine_status_ptr(void* h) { return (uint64_t)(((Engine*)h)->sync_local + OFF_STATUS); }

}  // extern "C"

#include "host_tier.cuh"
