// bulk_rows.cuh -- asynchronous row movement through shared memory.
//
// Random rows of a large table are fetched with DRAM and TLB misses, so a gather that stages
// rows in registers is bound by how many rows it keeps in flight. Rows therefore move with
// cp.async 16-byte copies (LDGSTS), which hold no registers while in flight and queue deep;
// one 1-D TMA copy (cp.async.bulk) per row was the other candidate. The choice was made by
// measurement on the GPUs the engine was first written for and has not been re-measured
// on H100.
// A warp keeps a whole task (32 weight rows, or up to 13 x {weights, state, accumulator}) in
// flight; peer-mapped (NVLink) addresses take the same path.
#pragma once
#include "exb_common.cuh"

namespace exb {

#define EXB_PULL_WARP_BUF 8192    // bytes of row staging per warp in the pull kernel
#define EXB_APPLY_WARP_BUF 10240  // bytes per warp in the apply phase (w | state | acc rows)

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __noinline__ float4 init_block_masked(const InitParams* I, unsigned long long id, int c, int dim);

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit_wait() {
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Pull the 32 rows of a warp task through shared memory (cp.async gather, coalesced write-out).
// Lane l holds (src, id, flag) of row l. buf: EXB_PULL_WARP_BUF bytes owned by this warp.
__device__ __forceinline__ void pull_rows_bulk(const TableDev& T, const float* src, unsigned long long id,
                                               int flag, int b0, int n_rows, float* __restrict__ out,
                                               int io_stride, int off, int lane, unsigned char* buf) {
    const int wstride = T.wstride;
    const unsigned rowbytes = (unsigned)wstride * 4u;
    const int R = min(32, (int)(EXB_PULL_WARP_BUF / rowbytes));   // rows per pass (warp uniform)
    const int lpr = T.lpr, gl = lane % lpr, RP = 32 / lpr;
    float* rows = reinterpret_cast<float*>(buf);
    for (int r0 = 0; r0 < 32; r0 += R) {
        // ---- issue: lane group g copies rows g, g+RP, ... of this pass, 16 bytes per lane
        for (int jb = 0; jb < R; jb += RP) {             // warp-uniform trip count (body shuffles)
            const int j = jb + lane / lpr, r = r0 + j;
            const float* s = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src, r & 31);
            const int fl = __shfl_sync(0xffffffffu, flag, r & 31);
            if (j < R && r < 32 && fl == 1)
                for (int c = gl * 4; c < wstride; c += lpr * 4) cp_async16(rows + (size_t)j * wstride + c, s + c);
        }
        cp_async_commit_wait();
        __syncwarp();
        // ---- write out (request order), zeros / initializer values for rows that were not loaded
        for (int jb = 0; jb < R; jb += RP) {
            const int j = jb + lane / lpr, r = r0 + j;
            const unsigned long long idr = __shfl_sync(0xffffffffu, id, r & 31);
            const int fl = __shfl_sync(0xffffffffu, flag, r & 31);
            const int b = b0 + r;
            if (j >= R || r >= 32 || b >= n_rows) continue;
            float* dst = out + (size_t)b * io_stride + off;
            for (int c = gl * 4; c < wstride; c += lpr * 4) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (fl == 1) v = *reinterpret_cast<const float4*>(rows + (size_t)j * wstride + c);
                else if (fl == 2) v = init_block_masked(&T.init, idr, c, T.dim);
                *reinterpret_cast<float4*>(dst + c) = v;
            }
        }
        __syncwarp();
    }
}

// Single-pass pull of a warp task: columns [0, bulk) of the 32 rows are gathered with cp.async through the warp's
// buffer, the remaining (< 8) columns of row l by lane l into registers -- so a [D | 1] split row of D = 64 needs
// the same 8 KB as a plain 64-column row and never a second pass. `mid()` runs while the loads are in flight
// (the training pull builds the batch's de-duplication plan there). Requires 32 * bulk * 4 <= EXB_PULL_WARP_BUF.
//   split >= dim: not a split feature (bulk = wstride); else columns [split, dim) go to out[b, off2 ...].
// LPR (lanes per row of the bulk part, power of two >= bulk / 4) is a template parameter: every loop below has a
// compile-time trip count and unrolls -- the run-time form executed ~1300 instructions per warp task, and a warp
// task is one dependent chain.
template <int LPR, class Mid>
__device__ __forceinline__ void pull_rows_fast_t(const TableDev& T, const float* src, unsigned long long id, int flag,
                                                 int b0, int n_rows, float* __restrict__ out, int io_stride, int off,
                                                 int off2, int split, int bulk, int lane, unsigned char* buf, Mid mid) {
    constexpr int RP = 32 / LPR;
    const int wstride = T.wstride, dim = T.dim;
    const int gl = lane % LPR, sub = lane / LPR;
    const int c = gl * 4;
    const bool cin = c < bulk;
    float* rows = reinterpret_cast<float*>(buf);
#pragma unroll
    for (int jb = 0; jb < 32; jb += RP) {
        const int j = jb + sub;
        const float* s = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src, j);
        const int fl = __shfl_sync(0xffffffffu, flag, j);
        if (fl == 1 && cin) cp_async16(rows + (size_t)j * bulk + c, s + c);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    float4 tl[2];
    tl[0] = tl[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int ntail = (wstride - bulk) >> 2;           // 0, 1 or 2 float4 per row
    if (flag == 1) {
        if (ntail > 0) tl[0] = ld_stream_v4(src + bulk);
        if (ntail > 1) tl[1] = ld_stream_v4(src + bulk + 4);
    } else if (flag == 2) {
        if (ntail > 0) tl[0] = init_block_masked(&T.init, id, bulk, dim);
        if (ntail > 1) tl[1] = init_block_masked(&T.init, id, bulk + 4, dim);
    }
    mid();
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    const unsigned any2 = __ballot_sync(0xffffffffu, flag == 2);
#pragma unroll
    for (int jb = 0; jb < 32; jb += RP) {
        const int j = jb + sub;
        const int fl = __shfl_sync(0xffffffffu, flag, j);
        const int b = b0 + j;
        if (b >= n_rows || !cin) continue;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (fl == 1) v = *reinterpret_cast<const float4*>(rows + (size_t)j * bulk + c);
        *reinterpret_cast<float4*>(out + (size_t)b * io_stride + off + c) = v;
    }
    if (any2) {                                        // rows answered with their initializer value (cold)
        for (int j = 0; j < 32; ++j) {
            if (!((any2 >> j) & 1u)) continue;
            const unsigned long long idr = __shfl_sync(0xffffffffu, id, j);
            if (b0 + j < n_rows)
                for (int cc = lane * 4; cc < bulk; cc += 128)
                    *reinterpret_cast<float4*>(out + (size_t)(b0 + j) * io_stride + off + cc) = init_block_masked(&T.init, idr, cc, dim);
        }
    }
    if (ntail > 0 && b0 + lane < n_rows) {             // lane l finishes row l
        float* dst = out + (size_t)(b0 + lane) * io_stride + off;
        float* dst2 = out + (size_t)(b0 + lane) * io_stride + off2;
        const float t[8] = {tl[0].x, tl[0].y, tl[0].z, tl[0].w, tl[1].x, tl[1].y, tl[1].z, tl[1].w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int col = bulk + e;
            if (e < 4 * ntail) {
                if (col < split) { if (col < wstride) dst[col] = t[e]; }
                else if (col < dim) dst2[col - split] = t[e];
            }
        }
    }
    __syncwarp();
}

template <class Mid>
__device__ __forceinline__ void pull_rows_fast(const TableDev& T, const float* src, unsigned long long id, int flag,
                                               int b0, int n_rows, float* __restrict__ out, int io_stride, int off,
                                               int off2, int split, int bulk, int lane, unsigned char* buf, Mid mid) {
    const int chunks = bulk >> 2;
#define EXB_PRF(L) pull_rows_fast_t<L>(T, src, id, flag, b0, n_rows, out, io_stride, off, off2, split, bulk, lane, buf, mid)
    if (chunks <= 1) EXB_PRF(1);
    else if (chunks <= 2) EXB_PRF(2);
    else if (chunks <= 4) EXB_PRF(4);
    else if (chunks <= 8) EXB_PRF(8);
    else if (chunks <= 16) EXB_PRF(16);
    else EXB_PRF(32);
#undef EXB_PRF
}
// column split of pull_rows_fast for a feature: bulk columns and whether the single-pass form applies
__device__ __forceinline__ bool pull_fast_geometry(const TableDev& T, int split, int* bulk) {
    const bool is_split = split < T.dim;
    *bulk = is_split ? (split & ~3) : T.wstride;
    if (!T.vec4 || *bulk <= 0) return false;
    if (T.wstride - *bulk > 8 || *bulk > 128) return false;
    return 32 * (*bulk) * 4 <= (int)EXB_PULL_WARP_BUF;
}

// Split-row feature: ONE table row feeds two places of the activation row -- columns [0, split) go to
// out[b, off ...], columns [split, dim) to out[b, off2 ...] (e.g. DeepFM: the dim-D embedding and the dim-1
// linear weight of a sparse feature share one row of dim D+1, so one lookup / one unique id / one optimizer
// row serves both; the reference keeps them as two variables = two RPCs, criteo_deepctr.py:60-110).
// Same cp.async gather as pull_rows_bulk; only the write-out differs. Pad columns are not written.
__device__ __forceinline__ void pull_rows_split(const TableDev& T, const float* src, unsigned long long id,
                                                int flag, int b0, int n_rows, float* __restrict__ out,
                                                int io_stride, int off, int off2, int split, int lane,
                                                unsigned char* buf) {
    const int wstride = T.wstride, dim = T.dim;
    const unsigned rowbytes = (unsigned)wstride * 4u;
    const int R = min(32, (int)(EXB_PULL_WARP_BUF / rowbytes));
    const int lpr = T.lpr, gl = lane % lpr, RP = 32 / lpr;
    float* rows = reinterpret_cast<float*>(buf);
    for (int r0 = 0; r0 < 32; r0 += R) {
        for (int jb = 0; jb < R; jb += RP) {
            const int j = jb + lane / lpr, r = r0 + j;
            const float* s = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)src, r & 31);
            const int fl = __shfl_sync(0xffffffffu, flag, r & 31);
            if (j < R && r < 32 && fl == 1)
                for (int c = gl * 4; c < wstride; c += lpr * 4) cp_async16(rows + (size_t)j * wstride + c, s + c);
        }
        cp_async_commit_wait();
        __syncwarp();
        for (int jb = 0; jb < R; jb += RP) {
            const int j = jb + lane / lpr, r = r0 + j;
            const unsigned long long idr = __shfl_sync(0xffffffffu, id, r & 31);
            const int fl = __shfl_sync(0xffffffffu, flag, r & 31);
            const int b = b0 + r;
            if (j >= R || r >= 32 || b >= n_rows) continue;
            float* dst = out + (size_t)b * io_stride + off;
            float* dst2 = out + (size_t)b * io_stride + off2;
            for (int c = gl * 4; c < wstride; c += lpr * 4) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (fl == 1) v = *reinterpret_cast<const float4*>(rows + (size_t)j * wstride + c);
                else if (fl == 2) v = init_block_masked(&T.init, idr, c, dim);
                if (c + 4 <= split) {
                    *reinterpret_cast<float4*>(dst + c) = v;
                } else {
                    const float t[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int col = c + e;
                        if (col < split) dst[col] = t[e];
                        else if (col < dim) dst2[col - split] = t[e];
                    }
                }
            }
        }
        __syncwarp();
    }
}

struct WarpMeta {   // per-warp row metadata of the apply phase (shared memory)
    unsigned long long key[32];
    unsigned long long row[32];
    unsigned h[32];
    unsigned cnt[32];
    int flag[32];
};

// Apply the optimizer to the (up to) 32 unique rows of a warp task: weights, state and
// accumulator rows are gathered into shared memory with cp.async, the math reads them from
// there and writes results straight back to global memory.
// Lane l holds (key,row,h,cnt,flag) of row l on entry.
// KIND is the optimizer category as a compile-time constant: the per-element switch of
// opt_elem folds away and the four elements of a float4 become straight-line, independent
// instruction streams (the runtime-switch version was issue-latency bound: ~10 us per pass).
template <int KIND>
__device__ __noinline__ void apply_rows_bulk_k(const TableDev& T, const PlanDev& P, float* accbase,
                                               unsigned long long key, unsigned long long row, unsigned h,
                                               unsigned cnt, int flag, int lane, unsigned char* buf,
                                               WarpMeta* M, int nrows, unsigned long long* trt) {
    const int wstride = T.wstride, sstride = T.sstride, dim = T.dim, nslots = T.nslots, nsc = T.nscalars;
    const unsigned wb = (unsigned)wstride * 4u, sb = (unsigned)sstride * 4u;
    const int R = min(32, (int)(EXB_APPLY_WARP_BUF / (2u * wb + sb)));
    const int lpr = T.lpr, gl = lane % lpr, RP = 32 / lpr;
    float* wloc = T.w[P.rank];
    OptParams opt = T.opt;
    opt.kind = KIND;
    const float s0i = opt_slot_init<float>(opt, 0), s1i = opt_slot_init<float>(opt, 1);
    M->key[lane] = key; M->row[lane] = row; M->h[lane] = h; M->cnt[lane] = cnt; M->flag[lane] = flag;
    __syncwarp();
    float* wbuf = reinterpret_cast<float*>(buf);
    float* sbuf = reinterpret_cast<float*>(buf + (size_t)R * wb);
    float* abuf = reinterpret_cast<float*>(buf + (size_t)R * (wb + sb));
    for (int r0 = 0; r0 < nrows; r0 += R) {
        // ---- gather: lane group g fetches rows g, g+RP, ... of the pass
        for (int jj = lane / lpr; jj < R; jj += RP) {
            const int rr = r0 + jj;
            if (rr >= 32) break;
            const int f = M->flag[rr];
            if (!f) continue;
            const float* ga = accbase + (unsigned long long)M->h[rr] * wstride;
            for (int c = gl * 4; c < wstride; c += lpr * 4) cp_async16(abuf + (size_t)jj * wstride + c, ga + c);
            if (f == 1) {
                const float* gw = wloc + M->row[rr] * (unsigned long long)wstride;
                const float* gs = T.state + M->row[rr] * (unsigned long long)sstride;
                for (int c = gl * 4; c < wstride; c += lpr * 4) cp_async16(wbuf + (size_t)jj * wstride + c, gw + c);
                for (int c = gl * 4; c < sstride; c += lpr * 4) cp_async16(sbuf + (size_t)jj * sstride + c, gs + c);
            }
        }
        cp_async_commit_wait();
        __syncwarp();
        if (trt && lane == 0) trt[5] = globaltimer_ns();
        // ---- math out of shared memory, results go straight to global
        for (int jj = lane / lpr; jj < R; jj += RP) {
            const int rr = r0 + jj;
            if (rr >= 32) break;
            const int f = M->flag[rr];
            if (!f) continue;
            const float* wr = wbuf + (size_t)jj * wstride;
            const float* sr = sbuf + (size_t)jj * sstride;
            const float* ar = abuf + (size_t)jj * wstride;
            float* gw = wloc + M->row[rr] * (unsigned long long)wstride;
            float* gs = T.state + M->row[rr] * (unsigned long long)sstride;
            float* ga = accbase + (unsigned long long)M->h[rr] * wstride;
            float sc[2] = {0.f, 0.f}, nsc_v[2];
            for (int i = 0; i < nsc; ++i)
                sc[i] = (f == 2) ? opt_scalar_init<float>(opt, i) : sr[(size_t)nslots * wstride + i];
            RowCtx<float> rc = opt_row_prologue_pure<float>(opt, sc, (uint64_t)M->cnt[rr], nsc_v);
            for (int c = gl * 4; c < wstride; c += lpr * 4) {
                float4 g = *reinterpret_cast<const float4*>(ar + c);
                float4 w, a = make_float4(s0i, s0i, s0i, s0i), b = make_float4(s1i, s1i, s1i, s1i);
                if (f == 2) {
                    w = init_block_masked(&T.init, M->key[rr], c, dim);
                } else {
                    w = *reinterpret_cast<const float4*>(wr + c);
                    if (nslots > 0) a = *reinterpret_cast<const float4*>(sr + c);
                    if (nslots > 1) b = *reinterpret_cast<const float4*>(sr + wstride + c);
                }
                if (c + 0 < dim) opt_elem<float>(opt, rc, w.x, a.x, b.x, g.x);
                if (c + 1 < dim) opt_elem<float>(opt, rc, w.y, a.y, b.y, g.y);
                if (c + 2 < dim) opt_elem<float>(opt, rc, w.z, a.z, b.z, g.z);
                if (c + 3 < dim) opt_elem<float>(opt, rc, w.w, a.w, b.w, g.w);
                *reinterpret_cast<float4*>(gw + c) = w;
                if (nslots > 0) *reinterpret_cast<float4*>(gs + c) = a;
                if (nslots > 1) *reinterpret_cast<float4*>(gs + wstride + c) = b;
                *reinterpret_cast<float4*>(ga + c) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            if (gl == 0) {
                for (int i = 0; i < nsc; ++i) gs[(size_t)nslots * wstride + i] = nsc_v[i];
                if (f == 2)   // pad words of a brand-new state row
                    for (int i = nslots * wstride + nsc; i < sstride; ++i) gs[i] = 0.f;
            }
        }
        __syncwarp();
    }
}

__device__ __forceinline__ void apply_rows_bulk(const TableDev& T, const PlanDev& P, float* accbase,
                                                unsigned long long key, unsigned long long row, unsigned h,
                                                unsigned cnt, int flag, int lane, unsigned char* buf,
                                                WarpMeta* M, int nrows, unsigned long long* trt) {
    switch (T.opt.kind) {   // warp uniform
        case OPT_ADADELTA: apply_rows_bulk_k<OPT_ADADELTA>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
        case OPT_ADAGRAD: apply_rows_bulk_k<OPT_ADAGRAD>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
        case OPT_ADAM: apply_rows_bulk_k<OPT_ADAM>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
        case OPT_ADAMAX: apply_rows_bulk_k<OPT_ADAMAX>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
        case OPT_FTRL: apply_rows_bulk_k<OPT_FTRL>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
        case OPT_RMSPROP: apply_rows_bulk_k<OPT_RMSPROP>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
        case OPT_SGD: apply_rows_bulk_k<OPT_SGD>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
        case OPT_TEST: apply_rows_bulk_k<OPT_TEST>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
        default: apply_rows_bulk_k<OPT_DEFAULT>(T, P, accbase, key, row, h, cnt, flag, lane, buf, M, nrows, trt); break;
    }
}

}  // namespace exb
