// exb_core.cpp -- CPU parameter-shard engine + checkpoint shard-file IO, C ABI ("exb_*").
//
// Role in the framework: (1) the numerical oracle every CUDA kernel is tested
// against, (2) the data path of the CPU/gloo configuration, (3) the native checkpoint
// reader/writer that speaks the reference's on-disk format bit for bit, (4) the backing
// store of the host-DRAM overflow tier.
//
// Reference behaviour mirrored here (read-only, cited for parity checks):
//   per-shard variable  openembedding/variable/EmbeddingOptimizerVariable.h:134-300
//   tables              openembedding/variable/EmbeddingTable.h:23-197
//   gradient reducer    openembedding/variable/MpscGradientReducer.h:12-69 (sum, not mean; counts summed)
//   shard file          openembedding/server/EmbeddingShardFile.h:13-86,
//                       openembedding/server/EmbeddingDumpOperator.cpp:58-94
// Differences: pulls never insert (initial values are a pure Philox function of the
// global id, so a missing row can be answered without mutating the table; rows are
// materialised by the first update), and the open-addressing map is linear-probing.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <vector>

#include "exb_math.h"

namespace exb {

static const uint64_t EMPTY_KEY = ~0ull;

// key -> dense slot index; power-of-two capacity, load <= 1/2, linear probing.
class SlotMap {
public:
    SlotMap() { rehash(1024); }
    int64_t find(uint64_t key) const {
        uint64_t m = _keys.size() - 1, h = exb_hash64(key) & m;
        for (;;) {
            uint64_t k = _keys[h];
            if (k == key) return _vals[h];
            if (k == EMPTY_KEY) return -1;
            h = (h + 1) & m;
        }
    }
    // returns slot; *inserted tells whether it is new (value = next_slot)
    int64_t find_or_insert(uint64_t key, int64_t next_slot, bool* inserted) {
        if ((_size + 1) * 2 > _keys.size()) rehash(_keys.size() * 2);
        uint64_t m = _keys.size() - 1, h = exb_hash64(key) & m;
        for (;;) {
            uint64_t k = _keys[h];
            if (k == key) { *inserted = false; return _vals[h]; }
            if (k == EMPTY_KEY) {
                _keys[h] = key; _vals[h] = next_slot; ++_size; *inserted = true;
                return next_slot;
            }
            h = (h + 1) & m;
        }
    }
    void reserve(size_t n) {
        size_t cap = _keys.size();
        while (cap < n * 2) cap *= 2;
        if (cap != _keys.size()) rehash(cap);
    }
    void clear() { _keys.assign(1024, EMPTY_KEY); _vals.assign(1024, 0); _size = 0; }
    size_t size() const { return _size; }

private:
    void rehash(size_t cap) {
        std::vector<uint64_t> ok; std::vector<int64_t> ov;
        ok.swap(_keys); ov.swap(_vals);
        _keys.assign(cap, EMPTY_KEY); _vals.assign(cap, 0);
        uint64_t m = cap - 1;
        for (size_t i = 0; i < ok.size(); ++i) {
            if (ok[i] == EMPTY_KEY) continue;
            uint64_t h = exb_hash64(ok[i]) & m;
            while (_keys[h] != EMPTY_KEY) h = (h + 1) & m;
            _keys[h] = ok[i]; _vals[h] = ov[i];
        }
    }
    std::vector<uint64_t> _keys;
    std::vector<int64_t> _vals;
    size_t _size = 0;
};

struct VariableBase {
    virtual ~VariableBase() {}
    virtual void set_initializer(const InitParams& I) = 0;
    virtual void set_optimizer(const OptParams& P) = 0;
    virtual void pull(const uint64_t* keys, size_t n, void* out) = 0;
    virtual void push(const uint64_t* keys, size_t n, const void* grads, const uint64_t* counts) = 0;
    virtual void update() = 0;
    virtual uint64_t num_items() = 0;
    virtual size_t read_indices(uint64_t* cursor, uint64_t* out, size_t cap) = 0;
    virtual void get_weights(const uint64_t* keys, size_t n, void* w, void* s) = 0;
    virtual void set_weights(const uint64_t* keys, size_t n, const void* w, const void* s,
                             uint64_t state_line_size) = 0;
    virtual void clear() = 0;
    virtual int state_dim() = 0;
    virtual uint64_t pending() = 0;
};

template <class T>
class Variable : public VariableBase {
public:
    Variable(int dim, uint64_t vocab, int shard_id, int shard_num, bool hash)
        : _dim(dim), _vocab(vocab), _shard_id(shard_id), _shard_num(shard_num), _hash(hash) {
        _init.kind = INIT_CONSTANT; _init.p[0] = _init.p[1] = _init.p[2] = 0; _init.seed = 0;
        _opt.kind = OPT_DEFAULT; for (double& v : _opt.p) v = 0;
        if (!_hash) {
            // local rows of this shard: ids {shard_id, shard_id+S, ...} < vocab
            _rows = vocab > (uint64_t)shard_id ? (vocab - shard_id + shard_num - 1) / shard_num : 0;
            _valid.assign(_rows, 0);
        }
    }
    void set_initializer(const InitParams& I) override {
        std::unique_lock<std::shared_mutex> l(_mu);
        _init = I;
    }
    void set_optimizer(const OptParams& P) override {
        std::unique_lock<std::shared_mutex> l(_mu);
        bool reset = P.kind != _opt.kind;  // category change resets the states (EmbeddingVariable.cpp:44-47)
        _opt = P;
        if (reset && (_hash || (_alloc_rows == _rows && _rows))) {
            int sd = state_dim();
            size_t n = _hash ? _slot_keys.size() : _rows;
            _states.assign(n * (size_t)sd, (T)0);
            for (size_t r = 0; r < n; ++r)
                if (_hash || _valid[r]) opt_init_state<T>(_opt, state_ptr(r), _dim);
        }
    }
    int state_dim() override { return opt_state_dim(_opt.kind, _dim); }

    void pull(const uint64_t* keys, size_t n, void* out_) override {
        std::shared_lock<std::shared_mutex> l(_mu);
        T* out = (T*)out_;
        for (size_t i = 0; i < n; ++i) {
            int64_t r = row_of(keys[i]);
            if (r >= 0) memcpy(out + i * _dim, &_weights[(size_t)r * _dim], sizeof(T) * _dim);
            else init_row<T>(_init, global_id(keys[i]), out + i * _dim, _dim);
        }
    }
    void push(const uint64_t* keys, size_t n, const void* grads, const uint64_t* counts) override {
        Block b;
        b.keys.assign(keys, keys + n);
        b.grads.assign((const T*)grads, (const T*)grads + n * _dim);
        if (counts) b.counts.assign(counts, counts + n); else b.counts.assign(n, 1);
        std::lock_guard<std::mutex> l(_qmu);
        _queue.push_back(std::move(b));
    }
    uint64_t pending() override { std::lock_guard<std::mutex> l(_qmu); return _queue.size(); }
    void update() override {
        std::vector<Block> blocks;
        { std::lock_guard<std::mutex> l(_qmu); blocks.swap(_queue); }
        if (blocks.empty()) return;
        std::unique_lock<std::shared_mutex> l(_mu);
        // reduce: unique key -> (sum grad, sum count), first-seen order
        SlotMap idx; std::vector<uint64_t> ukeys, ucnt; std::vector<T> ugrad;
        for (Block& b : blocks) {
            for (size_t i = 0; i < b.keys.size(); ++i) {
                bool ins; int64_t u = idx.find_or_insert(b.keys[i], (int64_t)ukeys.size(), &ins);
                if (ins) {
                    ukeys.push_back(b.keys[i]); ucnt.push_back(0);
                    ugrad.resize(ugrad.size() + _dim, (T)0);
                }
                ucnt[u] += b.counts[i];
                T* g = &ugrad[(size_t)u * _dim]; const T* s = &b.grads[i * _dim];
                for (int d = 0; d < _dim; ++d) g[d] += s[d];
            }
        }
        for (size_t u = 0; u < ukeys.size(); ++u) {
            size_t r = materialize(ukeys[u]);
            opt_update_row<T>(_opt, &_weights[r * _dim], state_ptr(r), _dim, ucnt[u],
                              &ugrad[u * _dim]);
        }
    }
    uint64_t num_items() override {
        std::shared_lock<std::shared_mutex> l(_mu);
        if (_hash) return _slot_keys.size();
        uint64_t c = 0; for (uint8_t v : _valid) c += v; return c;
    }
    size_t read_indices(uint64_t* cursor, uint64_t* out, size_t cap) override {
        std::shared_lock<std::shared_mutex> l(_mu);
        size_t n = 0; uint64_t c = *cursor;
        if (_hash) {
            while (c < _slot_keys.size() && n < cap) out[n++] = _slot_keys[c++];
        } else {
            while (c < _rows && n < cap) { if (_valid[c]) out[n++] = c; ++c; }
        }
        *cursor = c;
        return n;
    }
    void get_weights(const uint64_t* keys, size_t n, void* w_, void* s_) override {
        std::shared_lock<std::shared_mutex> l(_mu);
        T* w = (T*)w_; T* s = (T*)s_; int sd = state_dim();
        for (size_t i = 0; i < n; ++i) {
            int64_t r = row_of(keys[i]);
            if (r >= 0) {
                memcpy(w + i * _dim, &_weights[(size_t)r * _dim], sizeof(T) * _dim);
                if (s && sd) memcpy(s + i * sd, state_ptr(r), sizeof(T) * sd);
            } else {
                init_row<T>(_init, global_id(keys[i]), w + i * _dim, _dim);
                if (s && sd) opt_init_state<T>(_opt, s + i * sd, _dim);
            }
        }
    }
    void set_weights(const uint64_t* keys, size_t n, const void* w_, const void* s_,
                     uint64_t state_line_size) override {
        std::unique_lock<std::shared_mutex> l(_mu);
        const T* w = (const T*)w_; const T* s = (const T*)s_; int sd = state_dim();
        bool has_state = s && state_line_size == (uint64_t)sd * sizeof(T) && sd > 0;
        for (size_t i = 0; i < n; ++i) {
            size_t r = materialize(keys[i]);
            memcpy(&_weights[r * _dim], w + i * _dim, sizeof(T) * _dim);
            if (has_state) memcpy(state_ptr(r), s + i * sd, sizeof(T) * sd);
        }
    }
    void clear() override {
        std::unique_lock<std::shared_mutex> l(_mu);
        _weights.clear(); _states.clear(); _map.clear(); _slot_keys.clear();
        if (!_hash) { _valid.assign(_rows, 0); }
        _alloc_rows = 0;
    }

private:
    struct Block { std::vector<uint64_t> keys, counts; std::vector<T> grads; };
    uint64_t global_id(uint64_t local) const { return local * (uint64_t)_shard_num + _shard_id; }
    T* state_ptr(size_t r) { return _states.data() + r * (size_t)state_dim(); }
    int64_t row_of(uint64_t key) const {
        if (_hash) return _map.find(key);
        if (key >= _rows) return -1;
        return _valid[key] ? (int64_t)key : -1;
    }
    void ensure_array_alloc() {
        if (_alloc_rows == _rows) return;
        _weights.assign(_rows * (size_t)_dim, (T)0);
        _states.assign(_rows * (size_t)state_dim(), (T)0);
        _alloc_rows = _rows;
    }
    size_t materialize(uint64_t key) {
        int sd = state_dim();
        if (_hash) {
            bool ins; int64_t r = _map.find_or_insert(key, (int64_t)_slot_keys.size(), &ins);
            if (ins) {
                _slot_keys.push_back(key);
                _weights.resize(_weights.size() + _dim);
                _states.resize(_states.size() + sd);
                init_row<T>(_init, global_id(key), &_weights[(size_t)r * _dim], _dim);
                opt_init_state<T>(_opt, state_ptr(r), _dim);
            }
            return (size_t)r;
        }
        if (key >= _rows) { fprintf(stderr, "exb_core: index %llu out of range\n", (unsigned long long)key); abort(); }
        ensure_array_alloc();
        if (!_valid[key]) {
            _valid[key] = 1;
            init_row<T>(_init, global_id(key), &_weights[key * _dim], _dim);
            opt_init_state<T>(_opt, state_ptr(key), _dim);
        }
        return key;
    }

    int _dim; uint64_t _vocab; int _shard_id, _shard_num; bool _hash;
    InitParams _init; OptParams _opt;
    uint64_t _rows = 0, _alloc_rows = 0;
    std::vector<T> _weights, _states;
    std::vector<uint8_t> _valid;
    SlotMap _map; std::vector<uint64_t> _slot_keys;
    std::shared_mutex _mu; std::mutex _qmu; std::vector<Block> _queue;
};

// ---------------------------------------------------------------- shard files
struct ShardHeader {
    uint32_t variable_id; int32_t dtype; uint64_t dim, vocab; std::string config;
    int32_t shard_id, shard_num; uint64_t state_line_size, num_items;
};

struct FileWriter {
    FILE* f = nullptr; bool null_sink = false;
    void w(const void* p, size_t n) { if (!null_sink && n) { if (fwrite(p, 1, n, f) != n) { perror("exb write"); abort(); } } }
};
struct FileReader { FILE* f = nullptr; };

}  // namespace exb

using namespace exb;

extern "C" {

const char* exb_core_version() { return "openembedding-b200-core 0.1"; }

void* exb_var_create(int dtype, int dim, uint64_t vocab, int shard_id, int shard_num, int use_hash) {
    if (dtype == 0x104) return (VariableBase*)new Variable<float>(dim, vocab, shard_id, shard_num, use_hash != 0);
    if (dtype == 0x108) return (VariableBase*)new Variable<double>(dim, vocab, shard_id, shard_num, use_hash != 0);
    return nullptr;
}
void exb_var_destroy(void* v) { delete (VariableBase*)v; }
void exb_var_set_initializer(void* v, int kind, double p0, double p1, double p2, uint64_t seed) {
    InitParams I; I.kind = kind; I._pad = 0; I.p[0] = p0; I.p[1] = p1; I.p[2] = p2; I.seed = seed;
    ((VariableBase*)v)->set_initializer(I);
}
void exb_var_set_optimizer(void* v, int kind, const double* p, int np) {
    OptParams P; P.kind = kind; P._pad = 0; for (int i = 0; i < 8; ++i) P.p[i] = i < np ? p[i] : 0.0;
    ((VariableBase*)v)->set_optimizer(P);
}
int exb_var_state_dim(void* v) { return ((VariableBase*)v)->state_dim(); }
void exb_var_pull(void* v, const uint64_t* keys, uint64_t n, void* out) { ((VariableBase*)v)->pull(keys, n, out); }
void exb_var_push(void* v, const uint64_t* keys, uint64_t n, const void* grads, const uint64_t* counts) {
    ((VariableBase*)v)->push(keys, n, grads, counts);
}
void exb_var_update(void* v) { ((VariableBase*)v)->update(); }
uint64_t exb_var_pending(void* v) { return ((VariableBase*)v)->pending(); }
uint64_t exb_var_num_items(void* v) { return ((VariableBase*)v)->num_items(); }
uint64_t exb_var_read_indices(void* v, uint64_t* cursor, uint64_t* out, uint64_t cap) {
    return ((VariableBase*)v)->read_indices(cursor, out, cap);
}
void exb_var_get_weights(void* v, const uint64_t* keys, uint64_t n, void* w, void* s) {
    ((VariableBase*)v)->get_weights(keys, n, w, s);
}
void exb_var_set_weights(void* v, const uint64_t* keys, uint64_t n, const void* w, const void* s,
                         uint64_t state_line_size) {
    ((VariableBase*)v)->set_weights(keys, n, w, s, state_line_size);
}
void exb_var_clear(void* v) { ((VariableBase*)v)->clear(); }

// standalone math entry points (oracle for kernel tests)
void exb_opt_update_rows_f32(int kind, const double* p, float* w, float* state, int dim,
                             const uint64_t* counts, const float* g, uint64_t nrows) {
    OptParams P; P.kind = kind; P._pad = 0; for (int i = 0; i < 8; ++i) P.p[i] = p[i];
    int sd = opt_state_dim(kind, dim);
    for (uint64_t r = 0; r < nrows; ++r)
        opt_update_row<float>(P, w + r * dim, state + r * sd, dim, counts ? counts[r] : 1, g + r * dim);
}
void exb_opt_update_rows_f64(int kind, const double* p, double* w, double* state, int dim,
                             const uint64_t* counts, const double* g, uint64_t nrows) {
    OptParams P; P.kind = kind; P._pad = 0; for (int i = 0; i < 8; ++i) P.p[i] = p[i];
    int sd = opt_state_dim(kind, dim);
    for (uint64_t r = 0; r < nrows; ++r)
        opt_update_row<double>(P, w + r * dim, state + r * sd, dim, counts ? counts[r] : 1, g + r * dim);
}
void exb_opt_init_state_f32(int kind, const double* p, float* state, int dim, uint64_t nrows) {
    OptParams P; P.kind = kind; P._pad = 0; for (int i = 0; i < 8; ++i) P.p[i] = p[i];
    int sd = opt_state_dim(kind, dim);
    for (uint64_t r = 0; r < nrows; ++r) opt_init_state<float>(P, state + r * sd, dim);
}
int exb_opt_state_dim(int kind, int dim) { return opt_state_dim(kind, dim); }
void exb_init_rows_f32(int kind, double p0, double p1, double p2, uint64_t seed, const uint64_t* ids,
                       uint64_t n, int dim, float* out) {
    InitParams I; I.kind = kind; I._pad = 0; I.p[0] = p0; I.p[1] = p1; I.p[2] = p2; I.seed = seed;
    for (uint64_t i = 0; i < n; ++i) init_row<float>(I, ids[i], out + i * dim, dim);
}
void exb_init_rows_f64(int kind, double p0, double p1, double p2, uint64_t seed, const uint64_t* ids,
                       uint64_t n, int dim, double* out) {
    InitParams I; I.kind = kind; I._pad = 0; I.p[0] = p0; I.p[1] = p1; I.p[2] = p2; I.seed = seed;
    for (uint64_t i = 0; i < n; ++i) init_row<double>(I, ids[i], out + i * dim, dim);
}
uint64_t exb_hash64_c(uint64_t x) { return exb_hash64(x); }

// ---- shard file writer: header + blocks, little-endian raw (format: SURVEY 5.4)
void* exb_fw_open(const char* path) {
    FileWriter* w = new FileWriter();
    if (strncmp(path, "mem://null/", 11) == 0) { w->null_sink = true; return w; }
    w->f = fopen(path, "wb");
    if (!w->f) { delete w; return nullptr; }
    setvbuf(w->f, nullptr, _IOFBF, 8 << 20);
    return w;
}
void exb_fw_header(void* h, uint32_t variable_id, int32_t dtype, uint64_t dim, uint64_t vocab,
                   const char* config, uint64_t config_len, int32_t shard_id, int32_t shard_num,
                   uint64_t state_line_size, uint64_t num_items) {
    FileWriter* w = (FileWriter*)h;
    w->w(&variable_id, 4); w->w(&dtype, 4); w->w(&dim, 8); w->w(&vocab, 8);
    w->w(&config_len, 8); w->w(config, config_len);
    w->w(&shard_id, 4); w->w(&shard_num, 4); w->w(&state_line_size, 8); w->w(&num_items, 8);
}
void exb_fw_block(void* h, uint64_t n, const uint64_t* indices, const void* weights, uint64_t wbytes,
                  const void* states, uint64_t sbytes) {
    FileWriter* w = (FileWriter*)h;
    w->w(&n, 8); w->w(indices, n * 8); w->w(weights, wbytes); w->w(states, sbytes);
}
void exb_fw_close(void* h) { FileWriter* w = (FileWriter*)h; if (w->f) fclose(w->f); delete w; }

void* exb_fr_open(const char* path) {
    FILE* f = fopen(path, "rb");
    if (!f) return nullptr;
    setvbuf(f, nullptr, _IOFBF, 8 << 20);
    FileReader* r = new FileReader(); r->f = f; return r;
}
// returns 1 on success, 0 on clean EOF, -1 on corrupt; config copied into cfg (cap bytes)
int exb_fr_header(void* h, uint32_t* variable_id, int32_t* dtype, uint64_t* dim, uint64_t* vocab,
                  char* cfg, uint64_t cfg_cap, uint64_t* cfg_len, int32_t* shard_id,
                  int32_t* shard_num, uint64_t* state_line_size, uint64_t* num_items) {
    FILE* f = ((FileReader*)h)->f;
    size_t got = fread(variable_id, 1, 4, f);
    if (got == 0) return 0;
    if (got != 4) return -1;
    if (fread(dtype, 4, 1, f) != 1 || fread(dim, 8, 1, f) != 1 || fread(vocab, 8, 1, f) != 1 ||
        fread(cfg_len, 8, 1, f) != 1) return -1;
    if (*cfg_len >= cfg_cap) return -1;
    if (*cfg_len && fread(cfg, 1, *cfg_len, f) != *cfg_len) return -1;
    cfg[*cfg_len] = 0;
    if (fread(shard_id, 4, 1, f) != 1 || fread(shard_num, 4, 1, f) != 1 ||
        fread(state_line_size, 8, 1, f) != 1 || fread(num_items, 8, 1, f) != 1) return -1;
    return 1;
}
int64_t exb_fr_block_size(void* h) {
    uint64_t n; if (fread(&n, 8, 1, ((FileReader*)h)->f) != 1) return -1; return (int64_t)n;
}
// skip a block of n rows (after exb_fr_block_size) without reading it: the loader of a rank that does not own the
// segment's shard seeks past it
int exb_fr_skip_block(void* h, uint64_t n, uint64_t wbytes, uint64_t sbytes) {
    FILE* f = ((FileReader*)h)->f;
    const uint64_t total = n * 8 + wbytes + sbytes;
    return fseeko(f, (off_t)total, SEEK_CUR) == 0 ? 0 : -1;
}
int exb_fr_block(void* h, uint64_t n, uint64_t* indices, void* weights, uint64_t wbytes, void* states,
                 uint64_t sbytes) {
    FILE* f = ((FileReader*)h)->f;
    if (n && fread(indices, 8, n, f) != n) return -1;
    if (wbytes && fread(weights, 1, wbytes, f) != wbytes) return -1;
    if (sbytes && fread(states, 1, sbytes, f) != sbytes) return -1;
    return 0;
}
void exb_fr_close(void* h) { FileReader* r = (FileReader*)h; fclose(r->f); delete r; }

// ---- host-side id utilities (K1 on CPU): unique + inverse, shard bucketize
// out_unique must hold n entries; returns number of unique ids; inverse[i] = position in unique
uint64_t exb_unique_indices(const uint64_t* ids, uint64_t n, uint64_t* out_unique, uint64_t* inverse) {
    SlotMap m; m.reserve(n);
    uint64_t u = 0;
    for (uint64_t i = 0; i < n; ++i) {
        bool ins; int64_t s = m.find_or_insert(ids[i], (int64_t)u, &ins);
        if (ins) out_unique[u++] = ids[i];
        if (inverse) inverse[i] = (uint64_t)s;
    }
    return u;
}

// ---- LZ4 block codec (message / payload compression; the reference's RpcView / Compress offers snappy, lz4 and zlib,
// pico-core/include/pico-core/Compress.h). Standard LZ4 block format: sequences of [token | literal length bytes |
// literals | 2-byte offset | match length bytes]; greedy single-probe compressor with a 64 K-entry hash table.
// The decompressor checks every bound: corrupt input yields -1, never an out-of-range access.
int64_t exb_lz4_bound(int64_t n) { return n + n / 255 + 16; }

static inline uint32_t lz4_read32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

int64_t exb_lz4_compress(const uint8_t* src, int64_t n, uint8_t* dst, int64_t cap) {
    if (n < 0 || cap < exb_lz4_bound(n)) return -1;
    const int HASH_LOG = 16;
    std::vector<int64_t> table((size_t)1 << HASH_LOG, -1);
    uint8_t* op = dst;
    int64_t anchor = 0, ip = 0;
    const int64_t mflimit = n - 12, matchlimit = n - 5;
    auto emit_length = [&](int64_t len) { while (len >= 255) { *op++ = 255; len -= 255; } *op++ = (uint8_t)len; };
    while (ip <= mflimit) {
        const uint32_t seq = lz4_read32(src + ip);
        const uint32_t h = (seq * 2654435761u) >> (32 - HASH_LOG);
        const int64_t ref = table[h];
        table[h] = ip;
        if (ref < 0 || ip - ref > 65535 || lz4_read32(src + ref) != seq) { ++ip; continue; }
        int64_t mlen = 4;
        while (ip + mlen < matchlimit && src[ref + mlen] == src[ip + mlen]) ++mlen;
        const int64_t lit = ip - anchor;
        uint8_t* token = op++;
        *token = (uint8_t)((lit >= 15 ? 15 : lit) << 4);
        if (lit >= 15) emit_length(lit - 15);
        memcpy(op, src + anchor, (size_t)lit); op += lit;
        const uint16_t off = (uint16_t)(ip - ref);
        *op++ = (uint8_t)(off & 255); *op++ = (uint8_t)(off >> 8);
        const int64_t ml = mlen - 4;
        *token |= (uint8_t)(ml >= 15 ? 15 : ml);
        if (ml >= 15) emit_length(ml - 15);
        ip += mlen;
        anchor = ip;
    }
    const int64_t lit = n - anchor;       // last sequence: literals only
    uint8_t* token = op++;
    *token = (uint8_t)((lit >= 15 ? 15 : lit) << 4);
    if (lit >= 15) emit_length(lit - 15);
    memcpy(op, src + anchor, (size_t)lit); op += lit;
    return (int64_t)(op - dst);
}

int64_t exb_lz4_decompress(const uint8_t* src, int64_t n, uint8_t* dst, int64_t cap) {
    const uint8_t* ip = src; const uint8_t* const iend = src + n;
    uint8_t* op = dst; uint8_t* const oend = dst + cap;
    if (n <= 0) return n == 0 ? 0 : -1;
    for (;;) {
        if (ip >= iend) return -1;
        const uint8_t token = *ip++;
        int64_t lit = token >> 4;
        if (lit == 15) { uint8_t b; do { if (ip >= iend) return -1; b = *ip++; lit += b; } while (b == 255); }
        if (lit > iend - ip || lit > oend - op) return -1;
        memcpy(op, ip, (size_t)lit); op += lit; ip += lit;
        if (ip == iend) break;            // the last sequence carries no match
        if (iend - ip < 2) return -1;
        const int64_t off = ip[0] | (ip[1] << 8); ip += 2;
        if (off == 0 || off > op - dst) return -1;
        int64_t ml = token & 15;
        if (ml == 15) { uint8_t b; do { if (ip >= iend) return -1; b = *ip++; ml += b; } while (b == 255); }
        ml += 4;
        if (ml > oend - op) return -1;
        const uint8_t* m = op - off;
        for (int64_t i = 0; i < ml; ++i) op[i] = m[i];     // overlapping copies are the format's run-length trick
        op += ml;
    }
    return (int64_t)(op - dst);
}

}  // extern "C"
