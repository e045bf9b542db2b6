// dev_shard.cu -- generic (templated on the element type) device-resident table shard: float64 tables on the GPU.
//
// The reference registers float AND double tables (openembedding/variable/EmbeddingVariable.cpp:277-278) and its
// optimizer parity test runs both (test/optimizer_test.py:6-72). The fused fp32 engine (engine.cu) is built around
// 128-bit fp32 vectors and fp32 atomics; double precision is not the throughput path of these
// tables (fp64 runs at a fraction of the fp32 rate and doubles the bytes per row), so fp64 tables get this small, exact engine instead: every row is [weights | optimizer state] in the
// reference's own layout (EmbeddingOptimizerVariable.h:141), rows live in an open-addressing slab in HBM, and the
// verbs are the same four as the CPU oracle's (exb_core.cpp: pull / update / get / set) executed by kernels with the
// SAME shared math header (exb_math.h) in the same per-row order, and this file is built without multiply-add
// contraction (_build.py) -- the results are bit-identical to the CPU engine, except FTRL with learning_rate_power
// != -0.5: CUDA's pow is not the host libm's.
// Routing between ranks (unique ids -> owner, NCCL all_to_all) is done by the python layer (backend.py).
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <string>

#include "exb_math.h"

#define DS_EMPTY 0xFFFFFFFFFFFFFFFFull

namespace {

thread_local std::string g_ds_err;
int ds_fail(const char* what, cudaError_t e) { g_ds_err = std::string(what) + ": " + cudaGetErrorString(e); return -1; }
#define DCK(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return ds_fail(#x, _e); } while (0)

template <class T>
struct ShardDev {
    unsigned long long* keys;     // local row index -> slot (open addressing)
    T* rows;                      // [cap][rowlen]: weights[dim] | state[sdim]
    unsigned long long cap;       // pow2
    int dim, sdim, rowlen;
    int shard_id, shard_num;
    unsigned long long vocab;     // array tables: ids >= vocab are invalid (zeros); hash: 2^63
    exb::InitParams init;
    exb::OptParams opt;
    unsigned long long* count;    // occupied slots
    int* status;                  // 1: table full
};

template <class T>
struct Shard {
    ShardDev<T> d;
    int device = 0;
    bool is_hash = false;
};

__device__ __forceinline__ long long ds_find(const unsigned long long* keys, unsigned long long mask, unsigned long long k) {
    unsigned long long h = exb::exb_hash64(k) & mask;
    for (unsigned long long p = 0; p <= mask; ++p) {
        const unsigned long long v = keys[h];
        if (v == k) return (long long)h;
        if (v == DS_EMPTY) return -1;
        h = (h + 1) & mask;
    }
    return -1;
}
__device__ __forceinline__ long long ds_find_or_insert(unsigned long long* keys, unsigned long long mask, unsigned long long k,
                                                       bool* inserted) {
    unsigned long long h = exb::exb_hash64(k) & mask;
    *inserted = false;
    for (unsigned long long p = 0; p <= mask; ++p) {
        const unsigned long long v = *(volatile unsigned long long*)&keys[h];
        if (v == k) return (long long)h;
        if (v == DS_EMPTY) {
            const unsigned long long prev = atomicCAS(&keys[h], DS_EMPTY, k);
            if (prev == DS_EMPTY) { *inserted = true; return (long long)h; }
            if (prev == k) return (long long)h;
        }
        h = (h + 1) & mask;
    }
    return -1;
}

template <class T>
__global__ void ds_pull_kernel(ShardDev<T> S, const unsigned long long* ids, unsigned long long n, T* out) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = ids[i];
        T* o = out + i * S.dim;
        const unsigned long long gid = k * (unsigned long long)S.shard_num + S.shard_id;
        if (gid >= S.vocab) { for (int c = 0; c < S.dim; ++c) o[c] = (T)0; continue; }
        const long long s = ds_find(S.keys, S.cap - 1, k);
        if (s >= 0) { const T* r = S.rows + (unsigned long long)s * S.rowlen; for (int c = 0; c < S.dim; ++c) o[c] = r[c]; }
        else exb::init_row<T>(S.init, gid, o, S.dim);
    }
}
// ids unique; one thread per row: the per-row arithmetic order is the CPU oracle's
template <class T>
__global__ void ds_update_kernel(ShardDev<T> S, const unsigned long long* ids, unsigned long long n, const T* grads,
                                 const unsigned long long* counts) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = ids[i];
        const unsigned long long gid = k * (unsigned long long)S.shard_num + S.shard_id;
        if (gid >= S.vocab) continue;
        bool ins;
        const long long s = ds_find_or_insert(S.keys, S.cap - 1, k, &ins);
        if (s < 0) { atomicCAS(S.status, 0, 1); continue; }
        T* r = S.rows + (unsigned long long)s * S.rowlen;
        if (ins) {
            atomicAdd(S.count, 1ull);
            exb::init_row<T>(S.init, gid, r, S.dim);
            exb::opt_init_state<T>(S.opt, r + S.dim, S.dim);
        }
        exb::opt_update_row<T>(S.opt, r, r + S.dim, S.dim, counts ? counts[i] : 1ull, grads + i * S.dim);
    }
}
template <class T>
__global__ void ds_get_kernel(ShardDev<T> S, const unsigned long long* ids, unsigned long long n, T* w, T* st) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = ids[i];
        const long long s = ds_find(S.keys, S.cap - 1, k);
        if (s >= 0) {
            const T* r = S.rows + (unsigned long long)s * S.rowlen;
            for (int c = 0; c < S.dim; ++c) w[i * S.dim + c] = r[c];
            if (st) for (int c = 0; c < S.sdim; ++c) st[i * S.sdim + c] = r[S.dim + c];
        } else {
            exb::init_row<T>(S.init, k * (unsigned long long)S.shard_num + S.shard_id, w + i * S.dim, S.dim);
            if (st) exb::opt_init_state<T>(S.opt, st + i * S.sdim, S.dim);
        }
    }
}
template <class T>
__global__ void ds_set_kernel(ShardDev<T> S, const unsigned long long* ids, unsigned long long n, const T* w, const T* st) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        bool ins;
        const long long s = ds_find_or_insert(S.keys, S.cap - 1, ids[i], &ins);
        if (s < 0) { atomicCAS(S.status, 0, 1); continue; }
        if (ins) atomicAdd(S.count, 1ull);
        T* r = S.rows + (unsigned long long)s * S.rowlen;
        for (int c = 0; c < S.dim; ++c) r[c] = w[i * S.dim + c];
        if (st) for (int c = 0; c < S.sdim; ++c) r[S.dim + c] = st[i * S.sdim + c];
        else exb::opt_init_state<T>(S.opt, r + S.dim, S.dim);
    }
}
__global__ void ds_enumerate_kernel(const unsigned long long* keys, unsigned long long cap, unsigned long long* out,
                                    unsigned long long* counter) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < cap;
         i += (unsigned long long)gridDim.x * blockDim.x)
        if (keys[i] != DS_EMPTY) out[atomicAdd(counter, 1ull)] = keys[i];
}
template <class T>
__global__ void ds_rehash_kernel(ShardDev<T> O, ShardDev<T> N) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < O.cap;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = O.keys[i];
        if (k == DS_EMPTY) continue;
        bool ins;
        const long long s = ds_find_or_insert(N.keys, N.cap - 1, k, &ins);
        if (s < 0) continue;
        const T* a = O.rows + i * O.rowlen;
        T* b = N.rows + (unsigned long long)s * N.rowlen;
        for (int c = 0; c < O.rowlen; ++c) b[c] = a[c];
    }
}
// optimizer category change: state width changes, weights are kept, states restart
template <class T>
__global__ void ds_restate_kernel(ShardDev<T> O, ShardDev<T> N) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < O.cap;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        if (O.keys[i] == DS_EMPTY) continue;
        const T* a = O.rows + i * O.rowlen;
        T* b = N.rows + i * N.rowlen;
        for (int c = 0; c < O.dim; ++c) b[c] = a[c];
        exb::opt_init_state<T>(N.opt, b + N.dim, N.dim);
    }
}
__global__ void ds_fill_kernel(unsigned long long* p, unsigned long long n, unsigned long long v) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) p[i] = v;
}

template <class T>
int ds_alloc(Shard<T>* s, unsigned long long cap) {
    ShardDev<T>& d = s->d;
    d.cap = cap;
    DCK(cudaMalloc(&d.keys, cap * 8));
    DCK(cudaMalloc(&d.rows, cap * (size_t)d.rowlen * sizeof(T)));
    ds_fill_kernel<<<256, 256>>>(d.keys, cap, DS_EMPTY);
    DCK(cudaGetLastError());
    return 0;
}
template <class T>
int ds_grow(Shard<T>* s, unsigned long long need) {
    ShardDev<T>& d = s->d;
    unsigned long long cap = d.cap;
    while (need * 2 > cap) cap <<= 1;
    if (cap == d.cap) return 0;
    ShardDev<T> old = d;
    if (ds_alloc(s, cap)) return -1;
    ds_rehash_kernel<T><<<512, 256>>>(old, d);
    DCK(cudaGetLastError());
    DCK(cudaDeviceSynchronize());
    cudaFree(old.keys); cudaFree(old.rows);
    return 0;
}

}  // namespace

extern "C" {

const char* exb_ds_last_error() { return g_ds_err.c_str(); }

// dtype: 8 = float64, 4 = float32 (the fp32 instantiation exists for parity tests of this engine)
void* exb_ds_create(int device, int esize, int dim, uint64_t vocab, int shard_id, int shard_num, int is_hash, uint64_t capacity) {
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    if (esize != 8) { g_ds_err = "dev shard: float64 only"; return nullptr; }
    Shard<double>* s = new Shard<double>();
    s->device = device; s->is_hash = is_hash != 0;
    ShardDev<double>& d = s->d;
    memset(&d, 0, sizeof(d));
    d.dim = dim; d.sdim = 0; d.rowlen = dim;
    d.shard_id = shard_id; d.shard_num = shard_num;
    d.vocab = is_hash ? (1ull << 63) : vocab;
    d.init.kind = exb::INIT_CONSTANT; d.opt.kind = exb::OPT_DEFAULT;
    unsigned long long cap = 1024;
    while (cap < capacity) cap <<= 1;
    if (cudaMalloc(&d.count, 8) != cudaSuccess || cudaMalloc(&d.status, 4) != cudaSuccess) { delete s; return nullptr; }
    cudaMemset(d.count, 0, 8); cudaMemset(d.status, 0, 4);
    if (ds_alloc(s, cap)) { delete s; return nullptr; }
    return s;
}
void exb_ds_destroy(void* h) {
    Shard<double>* s = (Shard<double>*)h;
    cudaSetDevice(s->device);
    cudaFree(s->d.keys); cudaFree(s->d.rows); cudaFree(s->d.count); cudaFree(s->d.status);
    delete s;
}
int exb_ds_set_initializer(void* h, int kind, double p0, double p1, double p2, uint64_t seed) {
    exb::InitParams& I = ((Shard<double>*)h)->d.init;
    I.kind = kind; I._pad = 0; I.p[0] = p0; I.p[1] = p1; I.p[2] = p2; I.seed = seed;
    return 0;
}
int exb_ds_set_optimizer(void* h, int kind, const double* p, int np) {
    Shard<double>* s = (Shard<double>*)h;
    DCK(cudaSetDevice(s->device));
    ShardDev<double>& d = s->d;
    const bool changed = kind != d.opt.kind;
    d.opt.kind = kind; d.opt._pad = 0;
    for (int i = 0; i < 8; ++i) d.opt.p[i] = i < np ? p[i] : 0.0;
    if (changed) {        // new state width: rebuild the slab in place (same slots), states restart
        ShardDev<double> old = d;
        d.sdim = exb::opt_state_dim(kind, d.dim);
        d.rowlen = d.dim + d.sdim;
        DCK(cudaMalloc(&d.rows, d.cap * (size_t)d.rowlen * sizeof(double)));
        ds_restate_kernel<double><<<512, 256>>>(old, d);
        DCK(cudaGetLastError());
        DCK(cudaDeviceSynchronize());
        cudaFree(old.rows);
    }
    return 0;
}
int exb_ds_state_dim(void* h) { return ((Shard<double>*)h)->d.sdim; }
uint64_t exb_ds_num_items(void* h) {
    Shard<double>* s = (Shard<double>*)h;
    unsigned long long c = 0;
    cudaSetDevice(s->device);
    cudaMemcpy(&c, s->d.count, 8, cudaMemcpyDeviceToHost);
    return c;
}
static int ds_grid(uint64_t n) { return (int)((n + 255) / 256 > 2048 ? 2048 : (n + 255) / 256 ? (n + 255) / 256 : 1); }
// ids: LOCAL row indices (global id / shard_num), device pointers everywhere
int exb_ds_pull(void* h, uint64_t ids, uint64_t n, uint64_t out, uint64_t stream) {
    Shard<double>* s = (Shard<double>*)h;
    if (!n) return 0;
    ds_pull_kernel<double><<<ds_grid(n), 256, 0, (cudaStream_t)stream>>>(s->d, (const unsigned long long*)ids, n, (double*)out);
    DCK(cudaGetLastError());
    return 0;
}
int exb_ds_update(void* h, uint64_t ids, uint64_t n, uint64_t grads, uint64_t counts, uint64_t stream) {
    Shard<double>* s = (Shard<double>*)h;
    if (!n) return 0;
    DCK(cudaSetDevice(s->device));
    if (ds_grow(s, exb_ds_num_items(h) + n)) return -1;     // never more than half full after the inserts
    ds_update_kernel<double><<<ds_grid(n), 256, 0, (cudaStream_t)stream>>>(s->d, (const unsigned long long*)ids, n,
        (const double*)grads, (const unsigned long long*)counts);
    DCK(cudaGetLastError());
    return 0;
}
int exb_ds_get(void* h, uint64_t ids, uint64_t n, uint64_t w, uint64_t st, uint64_t stream) {
    Shard<double>* s = (Shard<double>*)h;
    if (!n) return 0;
    ds_get_kernel<double><<<ds_grid(n), 256, 0, (cudaStream_t)stream>>>(s->d, (const unsigned long long*)ids, n, (double*)w, (double*)st);
    DCK(cudaGetLastError());
    return 0;
}
int exb_ds_set(void* h, uint64_t ids, uint64_t n, uint64_t w, uint64_t st, uint64_t stream) {
    Shard<double>* s = (Shard<double>*)h;
    if (!n) return 0;
    DCK(cudaSetDevice(s->device));
    if (ds_grow(s, exb_ds_num_items(h) + n)) return -1;
    ds_set_kernel<double><<<ds_grid(n), 256, 0, (cudaStream_t)stream>>>(s->d, (const unsigned long long*)ids, n, (const double*)w, (const double*)st);
    DCK(cudaGetLastError());
    return 0;
}
// local row indices of all materialised rows -> out (device, capacity >= num_items); returns the count
int exb_ds_enumerate(void* h, uint64_t out, uint64_t* n_out) {
    Shard<double>* s = (Shard<double>*)h;
    DCK(cudaSetDevice(s->device));
    unsigned long long* ctr;
    DCK(cudaMalloc(&ctr, 8));
    DCK(cudaMemset(ctr, 0, 8));
    ds_enumerate_kernel<<<512, 256>>>(s->d.keys, s->d.cap, (unsigned long long*)out, ctr);
    DCK(cudaGetLastError());
    DCK(cudaMemcpy(n_out, ctr, 8, cudaMemcpyDeviceToHost));
    cudaFree(ctr);
    return 0;
}
int exb_ds_clear(void* h) {
    Shard<double>* s = (Shard<double>*)h;
    DCK(cudaSetDevice(s->device));
    ds_fill_kernel<<<256, 256>>>(s->d.keys, s->d.cap, DS_EMPTY);
    DCK(cudaMemset(s->d.count, 0, 8));
    DCK(cudaDeviceSynchronize());
    return 0;
}
int exb_ds_status(void* h) {
    Shard<double>* s = (Shard<double>*)h;
    int v = 0;
    cudaSetDevice(s->device);
    cudaDeviceSynchronize();
    cudaMemcpy(&v, s->d.status, 4, cudaMemcpyDeviceToHost);
    return v;
}
uint64_t exb_ds_bytes(void* h) {
    Shard<double>* s = (Shard<double>*)h;
    return s->d.cap * (8 + (uint64_t)s->d.rowlen * 8);
}

}  // extern "C"
