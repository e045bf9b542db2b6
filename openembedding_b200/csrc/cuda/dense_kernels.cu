// dense_kernels.cu -- the non-GEMM kernels of the fused dense step (DeepFM / Wide&Deep).
//
//   prep      X32 (pull output) -> bf16 MLP input A0 and its transpose A0T, FM field sums S,
//             per-sample base logit (linear + FM + bias); cached ("sparse_as_dense") tables
//             are gathered here
//   head      final dot with w_out, sigmoid, BCE loss, dlogit, dZ_last (+ transpose), gradients
//             of the small parameters, linear-term gradients of the sparse rows
//   predict   evaluation head: final dot with w_out, logits and sigmoid probabilities only
//   cachegrad scatter-add of the cached tables' gradient rows
//   adagrad   tf.keras Adagrad over the flat fp32 parameter buffer + refresh of the bf16
//             K-major weight copies (W and W^T) consumed by the wgmma GEMMs
//   allreduce one-shot / two-shot sum over peer-mapped gradient buffers (NVLink P2P), fused
//             with nothing else on purpose: it replaces the NCCL call of the reference's
//             Horovod DistributedOptimizer (K5 in SURVEY 2.5)
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include "pdl.cuh"
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <string>

namespace {

thread_local std::string g_dense_err;

struct PrepArgs {
    float* X32; long long xs;            // [B, XS] fp32: server emb cols filled by pull
    __nv_bfloat16* A0; __nv_bfloat16* A0T;   // [B, K0p], [K0p, B]
    const long long* ids; int ncols;     // [B, ncols] int64
    const float* dense; int nd;          // [B, nd]
    const float* cache_emb; const float* cache_lin;   // [Vc, Dp], [Vc]
    const int* cache_col; const long long* cache_off; int nc;   // cached features: id column, row offset
    const float* wd; const float* bias;  // dense-linear weights [nd], global bias [1]
    float* S; float* base;               // [B, Dp], [B]
    int B, K0p, Dp, nf, ns, lin0, use_fm;   // lin0 = first column of the server linear terms in X32
    float* loss;                         // [1] step loss accumulator, cleared here (head A adds to it)
    int* opt_step;                       // [1] dense-optimizer step counter (Adam bias correction), advanced here
};

// prep A: grid (B/32, ceil(K0p/256)); thread t owns ONE column of 32 batch rows: gathers cached
//         rows / dense features / the ones column, writes A0 (row major) and A0T (batch major,
//         64-byte runs). 7x more CTAs than a per-row-block loop: the kernel is latency bound.
__global__ void __launch_bounds__(256) exb_prep_a_kernel(PrepArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const int b0 = blockIdx.x * 32;
    const int col = blockIdx.y * 256 + threadIdx.x;
    if (col >= a.K0p) return;
    const int emb_cols = a.nf * a.Dp, srv_cols = a.ns * a.Dp;
    const bool full = b0 + 31 < a.B;
    float v[32];
    // every path below is a fully unrolled batch of 32 INDEPENDENT loads (v[] stays in registers)
    if (col < srv_cols) {
        const float* src = a.X32 + (size_t)b0 * a.xs + col;
#pragma unroll
        for (int r = 0; r < 32; ++r) v[r] = (full || b0 + r < a.B) ? src[(size_t)r * a.xs] : 0.f;
    } else if (col < emb_cols) {
        const int cj = (col - srv_cols) / a.Dp, d = col % a.Dp;
        const long long coff = a.cache_off[cj];
        const long long* idp = a.ids + (size_t)b0 * a.ncols + a.cache_col[cj];
        long long id[32];
#pragma unroll
        for (int r = 0; r < 32; ++r) id[r] = (full || b0 + r < a.B) ? idp[(size_t)r * a.ncols] : 0;
#pragma unroll
        for (int r = 0; r < 32; ++r) v[r] = a.cache_emb[(size_t)(coff + id[r]) * a.Dp + d];
        float* dst = a.X32 + (size_t)b0 * a.xs + col;
#pragma unroll
        for (int r = 0; r < 32; ++r)
            if (full || b0 + r < a.B) dst[(size_t)r * a.xs] = v[r];
    } else if (col < emb_cols + a.nd) {
        const float* src = a.dense + (size_t)b0 * a.nd + (col - emb_cols);
#pragma unroll
        for (int r = 0; r < 32; ++r) v[r] = (full || b0 + r < a.B) ? src[(size_t)r * a.nd] : 0.f;
    } else {
        const float c = (col == a.K0p - 1) ? 1.f : 0.f;
#pragma unroll
        for (int r = 0; r < 32; ++r) v[r] = c;
    }
    uint32_t pk[16];
    __nv_bfloat16* a0 = a.A0 + (size_t)b0 * a.K0p + col;
#pragma unroll
    for (int r = 0; r < 32; r += 2) {
        const __nv_bfloat16 h0 = __float2bfloat16_rn(v[r]), h1 = __float2bfloat16_rn(v[r + 1]);
        if (full || b0 + r < a.B) a0[(size_t)r * a.K0p] = h0;
        if (full || b0 + r + 1 < a.B) a0[(size_t)(r + 1) * a.K0p] = h1;
        pk[r >> 1] = (uint32_t)(*reinterpret_cast<const uint16_t*>(&h0)) |
                     ((uint32_t)(*reinterpret_cast<const uint16_t*>(&h1)) << 16);
    }
    if (a.A0T == nullptr) return;   // dW GEMMs read A0 itself as an MN-major operand
    if (full) {
        uint4* tp = reinterpret_cast<uint4*>(a.A0T + (size_t)col * a.B + b0);
#pragma unroll
        for (int j = 0; j < 4; ++j) tp[j] = make_uint4(pk[4 * j], pk[4 * j + 1], pk[4 * j + 2], pk[4 * j + 3]);
    } else {
#pragma unroll
        for (int r = 0; r < 32; ++r)
            if (b0 + r < a.B) a.A0T[(size_t)col * a.B + b0 + r] = __float2bfloat16_rn(v[r]);
    }
}

// prep B: one CTA per 8 batch rows: FM field sums with float4 loads (X32 is complete after
//         prep A), linear terms, per-sample base logit
__global__ void __launch_bounds__(256) exb_prep_b_kernel(PrepArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    __shared__ float sq[8], sfm[8], sl[8];
    const int b0 = blockIdx.x * 8;
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss) *a.loss = 0.f;
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.opt_step) *a.opt_step += 1;
    if (threadIdx.x < 8) { sq[threadIdx.x] = 0.f; sfm[threadIdx.x] = 0.f; sl[threadIdx.x] = 0.f; }
    __syncthreads();
    const int q4 = a.Dp / 4;
    for (int i = threadIdx.x; i < 8 * q4; i += blockDim.x) {
        const int r = i / q4, c = (i % q4) * 4, b = b0 + r;
        if (b >= a.B) continue;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        float q = 0.f;
        const float* xr = a.X32 + (size_t)b * a.xs + c;
#pragma unroll 13
        for (int f = 0; f < a.nf; ++f) {
            const float4 e = *reinterpret_cast<const float4*>(xr + (size_t)f * a.Dp);
            s.x += e.x; s.y += e.y; s.z += e.z; s.w += e.w;
            q += e.x * e.x + e.y * e.y + e.z * e.z + e.w * e.w;
        }
        *reinterpret_cast<float4*>(a.S + (size_t)b * a.Dp + c) = s;
        if (a.use_fm) {
            atomicAdd(&sq[r], q);
            atomicAdd(&sfm[r], s.x * s.x + s.y * s.y + s.z * s.z + s.w * s.w);
        }
    }
    const int per = a.ns + a.nc + 1;
    for (int i = threadIdx.x; i < 8 * per; i += blockDim.x) {
        const int r = i / per, j = i % per, b = b0 + r;
        if (b >= a.B) continue;
        float x = 0.f;
        if (j < a.ns) x = a.X32[(size_t)b * a.xs + a.lin0 + j];
        else if (j < a.ns + a.nc) {
            long long id = a.ids[(size_t)b * a.ncols + a.cache_col[j - a.ns]];
            x = a.cache_lin[a.cache_off[j - a.ns] + id];
        } else {
            for (int k = 0; k < a.nd; ++k) x += a.dense[(size_t)b * a.nd + k] * a.wd[k];
        }
        atomicAdd(&sl[r], x);
    }
    __syncthreads();
    if (threadIdx.x < 8 && b0 + threadIdx.x < a.B) {
        const int r = threadIdx.x;
        a.base[b0 + r] = sl[r] + (a.use_fm ? 0.5f * (sfm[r] - sq[r]) : 0.f) + a.bias[0];
    }
}

// prep, row-wise (Dp divides 128): ONE pass over X32 per batch row by one warp.
//   lane l handles the float4 at columns 4l + 128 i, so its embedding sub-range d = (4l) % Dp is the
//   same in every iteration: FM field sums and squares accumulate in registers, lanes that share
//   d are combined with xor-shuffles at the end. The same pass writes the bf16 MLP input row
//   (8 bytes per lane, 256 contiguous bytes per warp instruction), gathers the cached tables'
//   rows (and copies them into X32 for the FM gradient), appends dense features / padding /
//   the ones column, and reduces the linear terms into the per-sample base logit.
//   Replaces prep A (column per thread, needed only while A0^T was materialised) + prep B
//   (second pass over X32).
__global__ void __launch_bounds__(256) exb_prep_row_kernel(PrepArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss) *a.loss = 0.f;
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.opt_step) *a.opt_step += 1;
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (b >= a.B) return;
    const int emb_cols = a.nf * a.Dp, srv_cols = a.ns * a.Dp;
    float* xr = a.X32 + (size_t)b * a.xs;
    __nv_bfloat16* ar = a.A0 + (size_t)b * a.K0p;
    const long long* idr = a.ids + (size_t)b * a.ncols;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    float q = 0.f;
    constexpr int U = 7;
    for (int c0 = lane * 4; c0 < a.K0p; c0 += 128 * U) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {           // batch of independent loads
            const int c = c0 + 128 * u;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (c < srv_cols) {
                v[u] = *reinterpret_cast<const float4*>(xr + c);
            } else if (c < emb_cols) {
                const int cj = (c - srv_cols) / a.Dp, d = c % a.Dp;
                const long long id = idr[a.cache_col[cj]];
                v[u] = *reinterpret_cast<const float4*>(a.cache_emb + (size_t)(a.cache_off[cj] + id) * a.Dp + d);
            } else if (c < a.K0p) {
                float t[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int k = c + e - emb_cols;
                    t[e] = (k < a.nd) ? a.dense[(size_t)b * a.nd + k] : ((c + e == a.K0p - 1) ? 1.f : 0.f);
                }
                v[u] = make_float4(t[0], t[1], t[2], t[3]);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int c = c0 + 128 * u;
            if (c >= a.K0p) continue;
            if (c < emb_cols) {
                s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w;
                q += v[u].x * v[u].x + v[u].y * v[u].y + v[u].z * v[u].z + v[u].w * v[u].w;
                if (c >= srv_cols) *reinterpret_cast<float4*>(xr + c) = v[u];
            }
            const __nv_bfloat162 lo = __floats2bfloat162_rn(v[u].x, v[u].y), hi = __floats2bfloat162_rn(v[u].z, v[u].w);
            uint2 pk;
            pk.x = *reinterpret_cast<const uint32_t*>(&lo);
            pk.y = *reinterpret_cast<const uint32_t*>(&hi);
            *reinterpret_cast<uint2*>(ar + c) = pk;
        }
    }
    // lanes l, l + Dp/4, l + 2 Dp/4, ... hold partial sums of the same d
    for (int off = a.Dp >> 2; off < 32; off <<= 1) {
        s.x += __shfl_xor_sync(0xffffffffu, s.x, off); s.y += __shfl_xor_sync(0xffffffffu, s.y, off);
        s.z += __shfl_xor_sync(0xffffffffu, s.z, off); s.w += __shfl_xor_sync(0xffffffffu, s.w, off);
    }
    float fm = 0.f;
    if (lane < (a.Dp >> 2)) {
        *reinterpret_cast<float4*>(a.S + (size_t)b * a.Dp + lane * 4) = s;
        fm = s.x * s.x + s.y * s.y + s.z * s.z + s.w * s.w;
    }
    // linear terms: server rows (pulled into X32), cached rows, dense features
    float lin = 0.f;
    for (int j = lane; j < a.ns; j += 32) lin += xr[a.lin0 + j];
    for (int j = lane; j < a.nc; j += 32) lin += a.cache_lin[a.cache_off[j] + idr[a.cache_col[j]]];
    for (int k = lane; k < a.nd; k += 32) lin += a.dense[(size_t)b * a.nd + k] * a.wd[k];
    float tot = lin + (a.use_fm ? 0.5f * (fm - q) : 0.f);
#pragma unroll
    for (int off = 16; off; off >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, off);
    if (lane == 0) a.base[b] = tot + a.bias[0];
}

struct HeadArgs {
    const __nv_bfloat16* H; int Hp, ones_col;     // last hidden activation [B, Hp]
    const float* wout;                            // [Hp] (ones_col entry = output bias)
    const float* base; const float* labels;       // [B]
    float* dlogit; float* loss;                   // [B], [1] (sum of per-sample loss / B)
    __nv_bfloat16* dZ; __nv_bfloat16* dZT;        // [B, Hp], [Hp, B]
    float* g_wout; float* g_wd; float* g_bias;    // gradients of the small parameters
    const float* dense; int nd;
    float* G32; long long xs; int lin0, ns;       // linear-term grads of server rows
    const long long* ids; int ncols;
    const int* cache_col; const long long* cache_off; int nc; float* g_cache_lin;
    int B;
    float grad_scale;                             // 1/B (mean loss)
};

// head A: one warp per batch row: logit, loss, dlogit; linear-term gradients of that row
__global__ void __launch_bounds__(256) exb_head_a_kernel(HeadArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    __shared__ float s_loss[8], s_dl[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + warp;
    float z = 0.f, dl = 0.f, l = 0.f;
    if (b < a.B) {
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(a.H + (size_t)b * a.Hp);
        const float2* w2 = reinterpret_cast<const float2*>(a.wout);
        for (int n = lane; n < a.Hp / 2; n += 32) {
            const float2 hv = __bfloat1622float2(h2[n]);
            const float2 wv = w2[n];
            z += hv.x * wv.x + hv.y * wv.y;
        }
    }
    for (int o = 16; o; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    if (b < a.B) {
        z += a.base[b];
        const float y = a.labels[b];
        l = (fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)))) * a.grad_scale;   // stable BCE with logits
        dl = (1.f / (1.f + expf(-z)) - y) * a.grad_scale;
        if (lane == 0) a.dlogit[b] = dl;
        // linear-term gradients: server rows -> G32, cached rows -> dense grad
        for (int j = lane; j < a.ns + a.nc; j += 32) {
            if (j < a.ns) a.G32[(size_t)b * a.xs + a.lin0 + j] = dl;
            else {
                long long id = a.ids[(size_t)b * a.ncols + a.cache_col[j - a.ns]];
                atomicAdd(&a.g_cache_lin[a.cache_off[j - a.ns] + id], dl);
            }
        }
    }
    if (lane == 0) { s_loss[warp] = l; s_dl[warp] = dl; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f, gb = 0.f;
        for (int i = 0; i < 8; ++i) { t += s_loss[i]; gb += s_dl[i]; }
        atomicAdd(a.loss, t);
        atomicAdd(a.g_bias, gb);
    }
    if ((int)threadIdx.x < a.nd) {     // dense-linear weight gradient, reduced over the CTA's 8 rows
        float g = 0.f;
        for (int r = 0; r < 8; ++r) {
            const int bb = blockIdx.x * 8 + r;
            if (bb < a.B) g += s_dl[r] * a.dense[(size_t)bb * a.nd + threadIdx.x];
        }
        atomicAdd(&a.g_wd[threadIdx.x], g);
    }
}

// head B: grid (B/32, ceil(Hp/256)); thread = one column of 32 rows:
//         dZ = dl * wout * relu'(H) in both layouts, g_wout
__global__ void __launch_bounds__(256) exb_head_b_kernel(HeadArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    __shared__ float s_dl[32];
    const int b0 = blockIdx.x * 32;
    if (threadIdx.x < 32) s_dl[threadIdx.x] = (b0 + threadIdx.x < a.B) ? a.dlogit[b0 + threadIdx.x] : 0.f;
    __syncthreads();
    const int n = blockIdx.y * 256 + threadIdx.x;
    if (n >= a.Hp) return;
    const float w = a.wout[n];
    float gw = 0.f;
    float hv[32];
#pragma unroll
    for (int r = 0; r < 32; ++r) hv[r] = (b0 + r < a.B) ? __bfloat162float(a.H[(size_t)(b0 + r) * a.Hp + n]) : 0.f;
    uint32_t pk[16];
#pragma unroll
    for (int r = 0; r < 32; ++r) {
        float dz = 0.f;
        gw += s_dl[r] * hv[r];
        if (hv[r] > 0.f && n != a.ones_col) dz = s_dl[r] * w;
        const __nv_bfloat16 hb = __float2bfloat16_rn(dz);
        if (b0 + r < a.B) a.dZ[(size_t)(b0 + r) * a.Hp + n] = hb;
        const uint16_t u = *reinterpret_cast<const uint16_t*>(&hb);
        if (r & 1) pk[r >> 1] |= (uint32_t)u << 16; else pk[r >> 1] = u;
    }
    if (a.dZT == nullptr) {
    } else if (b0 + 31 < a.B) {
        uint4* tp = reinterpret_cast<uint4*>(a.dZT + (size_t)n * a.B + b0);
#pragma unroll
        for (int j = 0; j < 4; ++j) tp[j] = make_uint4(pk[4 * j], pk[4 * j + 1], pk[4 * j + 2], pk[4 * j + 3]);
    } else {
        for (int r = 0; r < 32 && b0 + r < a.B; ++r) {
            const uint16_t u = (pk[r >> 1] >> ((r & 1) * 16)) & 0xffffu;
            a.dZT[(size_t)n * a.B + b0 + r] = *reinterpret_cast<const __nv_bfloat16*>(&u);
        }
    }
    atomicAdd(&a.g_wout[n], gw);
}

// head, row-wise (Hp <= 512): one warp per batch row, 4 rows per warp, 32 rows per CTA.
//   pass 1: z = base + H[b,:] . wout (H row kept in registers), loss, dlogit
//   pass 2: dZ[b,:] = dlogit * wout * relu'(H) straight from those registers; dlogit * H
//           accumulates per lane into the output-weight gradient, reduced over the CTA's 32
//           rows in shared memory -> one global atomic per (CTA, column)
//   server linear-term gradients go to G32; the cached tables' linear gradients are produced
//   by the cachegrad kernel (which already groups duplicate ids).
// Replaces head A + head B (the second existed for the transposed dZ copy).
#define EXB_HEAD_MAXP 8
__global__ void __launch_bounds__(256) exb_head_row_kernel(HeadArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    __shared__ float s_gw[512];
    __shared__ float s_dl[32];
    __shared__ float s_loss[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 512; i += blockDim.x) s_gw[i] = 0.f;
    __syncthreads();
    const int np = a.Hp >> 1;                       // bf16x2 pairs per row
    float2 wv[EXB_HEAD_MAXP], gw[EXB_HEAD_MAXP];
#pragma unroll
    for (int p = 0; p < EXB_HEAD_MAXP; ++p) {
        const int n = lane + 32 * p;
        wv[p] = (n < np) ? reinterpret_cast<const float2*>(a.wout)[n] : make_float2(0.f, 0.f);
        gw[p] = make_float2(0.f, 0.f);
    }
    float lsum = 0.f;
    // the warp's 4 rows are processed together: all H loads first, then 4 interleaved reductions
    float2 hv[4][EXB_HEAD_MAXP];
    float z[4], dlv[4];
    const int brow = blockIdx.x * 32 + warp * 4;
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
        const int b = brow + rr;
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(a.H + (size_t)min(b, a.B - 1) * a.Hp);
#pragma unroll
        for (int p = 0; p < EXB_HEAD_MAXP; ++p) {
            const int n = lane + 32 * p;
            hv[rr][p] = (n < np && b < a.B) ? __bfloat1622float2(h2[n]) : make_float2(0.f, 0.f);
        }
    }
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
        z[rr] = 0.f;
#pragma unroll
        for (int p = 0; p < EXB_HEAD_MAXP; ++p) z[rr] += hv[rr][p].x * wv[p].x + hv[rr][p].y * wv[p].y;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) z[rr] += __shfl_xor_sync(0xffffffffu, z[rr], o);
    }
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
        const int b = brow + rr;
        dlv[rr] = 0.f;
        if (b < a.B) {                              // warp uniform
            const float zz = z[rr] + a.base[b];
            const float y = a.labels[b];
            lsum += (fmaxf(zz, 0.f) - zz * y + log1pf(expf(-fabsf(zz)))) * a.grad_scale;   // stable BCE with logits
            dlv[rr] = (1.f / (1.f + expf(-zz)) - y) * a.grad_scale;
        }
    }
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
        const int b = brow + rr;
        const float dl = dlv[rr];
        if (b < a.B) {
            if (lane == 0) a.dlogit[b] = dl;
            for (int j = lane; j < a.ns; j += 32) a.G32[(size_t)b * a.xs + a.lin0 + j] = dl;
            __nv_bfloat162* dz2 = reinterpret_cast<__nv_bfloat162*>(a.dZ + (size_t)b * a.Hp);
#pragma unroll
            for (int p = 0; p < EXB_HEAD_MAXP; ++p) {
                const int n = lane + 32 * p;
                if (n >= np) continue;
                gw[p].x += dl * hv[rr][p].x; gw[p].y += dl * hv[rr][p].y;
                const float dx = (hv[rr][p].x > 0.f && 2 * n != a.ones_col) ? dl * wv[p].x : 0.f;
                const float dy = (hv[rr][p].y > 0.f && 2 * n + 1 != a.ones_col) ? dl * wv[p].y : 0.f;
                dz2[n] = __floats2bfloat162_rn(dx, dy);
            }
        }
        if (lane == 0) s_dl[warp * 4 + rr] = dl;
    }
#pragma unroll
    for (int p = 0; p < EXB_HEAD_MAXP; ++p) {
        const int n = lane + 32 * p;
        if (n < np) { atomicAdd(&s_gw[2 * n], gw[p].x); atomicAdd(&s_gw[2 * n + 1], gw[p].y); }
    }
    if (lane == 0) s_loss[warp] = lsum;
    __syncthreads();
    for (int n = threadIdx.x; n < a.Hp; n += blockDim.x) atomicAdd(&a.g_wout[n], s_gw[n]);
    if (threadIdx.x == 0) {
        float t = 0.f, gb = 0.f;
        for (int i = 0; i < 8; ++i) t += s_loss[i];
        for (int i = 0; i < 32; ++i) gb += s_dl[i];
        atomicAdd(a.loss, t);
        atomicAdd(a.g_bias, gb);
    }
    if ((int)threadIdx.x < a.nd) {     // dense-linear weight gradient, reduced over the CTA's 32 rows
        float g = 0.f;
        for (int r = 0; r < 32; ++r) {
            const int bb = blockIdx.x * 32 + r;
            if (bb < a.B) g += s_dl[r] * a.dense[(size_t)bb * a.nd + threadIdx.x];
        }
        atomicAdd(&a.g_wd[threadIdx.x], g);
    }
}

struct PredictArgs {
    const __nv_bfloat16* H; int Hp;               // last hidden activation [B, Hp]
    const float* wout;                            // [Hp] (ones-column entry = output bias)
    const float* base;                            // [B] linear + FM / CIN / cross terms
    float* logits; float* probs;                  // [B], [B]
    int B;
};

// predict head (evaluation): one warp per batch row, any Hp: z = base + H[b,:] . wout, sigmoid(z).
// Writes logits and probs only -- no loss, dlogit, dZ or gradient.
__global__ void __launch_bounds__(256) exb_predict_head_kernel(PredictArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (b >= a.B) return;
    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(a.H + (size_t)b * a.Hp);
    const float2* w2 = reinterpret_cast<const float2*>(a.wout);
    float z = 0.f;
    for (int n = lane; n < a.Hp / 2; n += 32) {
        const float2 hv = __bfloat1622float2(h2[n]);
        const float2 wv = w2[n];
        z += hv.x * wv.x + hv.y * wv.y;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    if (lane == 0) {
        z += a.base[b];
        a.logits[b] = z;
        a.probs[b] = 1.f / (1.f + expf(-z));
    }
}

// Scatter-add the gradient rows of the cached (replicated) embedding tables.
// CTA = (cached feature, 256 batch rows), warp = 32 rows. The 32 gradient rows go through a
// per-warp shared-memory tile; rows with the SAME id are grouped with __match_any_sync, the first
// row of a group (its leader) owns the sum. The (row, 4-column chunk) pairs are then spread over
// the lanes: a pair whose row is a leader adds up the group's tile rows and issues one
// red.global.add.v4 -- distinct ids proceed in parallel (a large-vocabulary tile is 16 fully
// parallel steps), duplicates cost one shared-memory read each instead of a global atomic.
// Cached tables are the small-vocabulary ones (3..4096 rows): the first version issued one global
// atomic per (sample, chunk) and serialised on the hot rows. Shared-memory float atomics were
// tried for the tiniest tables and were slower.
// The kernel also produces the cached tables' linear-term gradients (dlogit summed per id).
#define EXB_CG_MAXDP 128
__global__ void __launch_bounds__(256) exb_cachegrad_kernel(const float* G32, long long xs, int col0, int Dp,
                                                            const long long* ids, int ncols, const int* cache_col,
                                                            const long long* cache_off, int nc, float* g_cache_emb,
                                                            int B, const float* dlogit, float* g_cache_lin) {
    exb::pdl_trigger();
    extern __shared__ __align__(16) float cg_smem[];
    __shared__ unsigned s_mem[8][32];       // group mask of a leader row, 0 otherwise
    __shared__ long long s_id[8][32];
    __shared__ float s_dl[8][32];
    exb::pdl_wait();
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
    const int chunks = Dp >> 2;
    const int j = blockIdx.x % nc, blk = blockIdx.x / nc;
    float* tile = cg_smem + (size_t)wic * 32 * Dp;
    const int b0 = blk * 256 + wic * 32;
    if (b0 >= B) return;
    const int b = b0 + lane;
    const long long id = (b < B) ? ids[(size_t)b * ncols + cache_col[j]] : -1ll - lane;
    const float* src = G32 + (size_t)b0 * xs + col0 + j * Dp;
    constexpr int LU = 8;                                       // batches of independent loads
    for (int i0 = 0; i0 < chunks; i0 += LU) {                   // idx = lane + 32 i: coalesced float4s
        float4 v[LU];
#pragma unroll
        for (int u = 0; u < LU; ++u) {
            const int idx = lane + 32 * (i0 + u);
            const int r = idx / chunks, c = idx - r * chunks;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i0 + u < chunks && b0 + r < B) v[u] = __ldcg(reinterpret_cast<const float4*>(src + (size_t)r * xs) + c);
        }
#pragma unroll
        for (int u = 0; u < LU; ++u)
            if (i0 + u < chunks) reinterpret_cast<float4*>(tile)[lane + 32 * (i0 + u)] = v[u];
    }
    const unsigned grp = __match_any_sync(0xffffffffu, id);
    s_mem[wic][lane] = (b < B && lane == __ffs(grp) - 1) ? grp : 0u;
    s_id[wic][lane] = id;
    s_dl[wic][lane] = (g_cache_lin != nullptr && b < B) ? dlogit[b] : 0.f;
    __syncwarp();
    const long long base = cache_off[j];
    for (int i = 0; i < chunks; ++i) {
        const int idx = lane + 32 * i;
        const int r = idx / chunks, c = idx - r * chunks;
        const unsigned members = s_mem[wic][r];
        if (!members) continue;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        float dl = 0.f;
        for (unsigned m = members; m; m &= m - 1) {
            const int q = __ffs(m) - 1;
            const float4 v = reinterpret_cast<const float4*>(tile)[q * chunks + c];
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            if (c == 0) dl += s_dl[wic][q];
        }
        const long long row = base + s_id[wic][r];
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(g_cache_emb + (size_t)row * Dp + c * 4), "f"(acc.x),
                     "f"(acc.y), "f"(acc.z), "f"(acc.w) : "memory");
        if (c == 0 && g_cache_lin != nullptr) atomicAdd(&g_cache_lin[row], dl);
    }
}

// ---- dense optimizer step: Adagrad + bf16 weight refresh + gradient clearing in ONE pass ----
// theta is the flat fp32 parameter buffer; the first `nmat` segments are the MLP weight matrices
// [R, C] whose bf16 copy Wb [R, C] and transposed copy WTb [C, R] feed the wgmma GEMMs of the
// next step. A 256-thread CTA (32x8) walks 32x32 tiles: read g/accum/w once, write w/accum, the
// bf16 tile, the transposed bf16 tile (through shared memory) and zero the gradient, so the
// step needs no separate memset / Adagrad / 3x refresh launches. Elements outside the matrices
// (output weights, dense-linear weights, bias, cached embedding tables) are updated flat.
// Up to EXB_OPT_MAX_MATS matrices: the DNN layers, then (xDeepFM) the CIN layer filters.
constexpr int EXB_OPT_MAX_MATS = 8;
struct OptMat { long long off; int R, C; __nv_bfloat16* Wb; __nv_bfloat16* WTb; };
struct DenseOptArgs {
    float* theta; float* accum; float* grad;
    long long n, flat_lo;          // [flat_lo, n) is the flat region (matrices come first)
    float lr, eps;
    int nmat, zero_grad;
    OptMat mat[EXB_OPT_MAX_MATS];
    // optimizer of the dense parameters (tf.keras semantics, the ones the reference benchmark sweeps:
    // test/benchmark/criteo_deepctr.py --optimizer Adagrad | Adam | Ftrl): 0 adagrad, 1 adam, 2 ftrl
    int kind, _pad;
    float* accum2;                 // second state slot (adam: v, ftrl: linear); accum = adam m / ftrl accumulator
    const int* step;               // device step counter (adam bias correction)
    float b1, b2;                  // adam
    float l1, l2, l2s, lrp, beta;  // ftrl: l1, l2, l2 shrinkage, learning_rate_power, beta
    float c1, c2;                  // adam: bias-corrected step size factors are computed per launch from *step
};

struct OptRun { int kind; float lr, eps, b1, b2, lr_t, l1, l2s, lrp, adj_l2; };

__device__ __forceinline__ OptRun opt_run(const DenseOptArgs& o) {
    OptRun r;
    r.kind = o.kind; r.lr = o.lr; r.eps = o.eps; r.b1 = o.b1; r.b2 = o.b2; r.l1 = o.l1; r.l2s = o.l2s; r.lrp = o.lrp;
    r.adj_l2 = o.l2 + o.beta / o.lr * 0.5f;
    r.lr_t = o.lr;
    if (o.kind == 1) {
        const float t = (float)(o.step ? *o.step : 1);
        r.lr_t = o.lr * sqrtf(1.f - powf(o.b2, t)) / (1.f - powf(o.b1, t));
    }
    return r;
}

// one parameter: w, state slots a (accum / m / ftrl accumulator) and b (adam v / ftrl linear)
__device__ __forceinline__ void dense_opt_one(const OptRun& r, float& w, float& a, float& b, float g) {
    if (r.kind == 0) {                       // adagrad: a += g^2; w -= lr g / (sqrt(a) + eps)
        a += g * g;
        float q;
        asm("sqrt.approx.f32 %0, %1;" : "=f"(q) : "f"(a));      // 1 ulp; the IEEE sequences made this kernel issue bound
        w -= __fdividef(r.lr * g, q + r.eps);
    } else if (r.kind == 1) {                // adam (keras): m, v moments; w -= lr_t m / (sqrt(v) + eps)
        a = r.b1 * a + (1.f - r.b1) * g;
        b = r.b2 * b + (1.f - r.b2) * g * g;
        w -= r.lr_t * a / (sqrtf(b) + r.eps);
    } else {                                 // ftrl (keras / EmbeddingOptimizer.h:230-293)
        const float gs = g + 2.f * r.l2s * w;
        const float an = a + g * g;
        const float pa = powf(an, -r.lrp), po = powf(a, -r.lrp);
        b += gs - (pa - po) / r.lr * w;
        a = an;
        const float quad = pa / r.lr + 2.f * r.adj_l2;
        const float l1a = fminf(fmaxf(b, -r.l1), r.l1);
        w = (l1a - b) / quad;
    }
}

__device__ __forceinline__ float adagrad_one(float& w, float& a, float g, float lr, float eps) {
    a += g * g;
    float r;
    asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(a));      // 1 ulp; the IEEE sequences made this kernel issue bound
    w -= __fdividef(lr * g, r + eps);
    return w;
}

__device__ __forceinline__ void dense_opt_step(const DenseOptArgs& o, float (*tile)[33]) {
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // launched with 256 threads
    const OptRun R = opt_run(o);
    const bool two = o.kind != 0 && o.accum2 != nullptr;
    int tile_base = 0;
    for (int mi = 0; mi < o.nmat; ++mi) {
        const OptMat M = o.mat[mi];
        const int tc = (M.C + 31) / 32, tr = (M.R + 31) / 32, nt = tc * tr;
        // tiles of all matrices form one global list; CTA b takes tiles b, b+grid, ...
        const int G = (int)gridDim.x;
        for (int t = ((int)blockIdx.x - tile_base % G + G) % G; t < nt; t += G) {
            const int r0 = (t / tc) * 32, c0 = (t % tc) * 32;
            float g4[4], a4[4], w4[4], b4[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {          // 12 independent loads in flight per thread
                const int r = r0 + ty + 8 * u, c = c0 + tx;
                g4[u] = a4[u] = w4[u] = b4[u] = 0.f;
                if (r < M.R && c < M.C) {
                    const long long k = M.off + (long long)r * M.C + c;
                    g4[u] = __ldcg(o.grad + k); a4[u] = o.accum[k]; w4[u] = o.theta[k];
                    if (two) b4[u] = o.accum2[k];
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int i = ty + 8 * u, r = r0 + i, c = c0 + tx;
                if (r < M.R && c < M.C) {
                    const long long k = M.off + (long long)r * M.C + c;
                    dense_opt_one(R, w4[u], a4[u], b4[u], g4[u]);
                    o.accum[k] = a4[u];
                    if (two) o.accum2[k] = b4[u];
                    o.theta[k] = w4[u];
                    if (o.zero_grad) o.grad[k] = 0.f;
                    M.Wb[(size_t)r * M.C + c] = __float2bfloat16_rn(w4[u]);
                }
                tile[i][tx] = w4[u];
            }
            __syncthreads();
            for (int i = ty; i < 32; i += 8) {
                const int c = c0 + i, r = r0 + tx;
                if (r < M.R && c < M.C) M.WTb[(size_t)c * M.R + r] = __float2bfloat16_rn(tile[tx][i]);
            }
            __syncthreads();
        }
        tile_base += nt;
    }
    for (long long i = o.flat_lo + (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4; i < o.n;
         i += (long long)gridDim.x * blockDim.x * 4) {
        if (i + 3 < o.n) {
            const float4 g = __ldcg(reinterpret_cast<const float4*>(o.grad + i));
            float4 a = *reinterpret_cast<float4*>(o.accum + i);
            float4 w = *reinterpret_cast<float4*>(o.theta + i);
            float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
            if (two) b = *reinterpret_cast<float4*>(o.accum2 + i);
            dense_opt_one(R, w.x, a.x, b.x, g.x); dense_opt_one(R, w.y, a.y, b.y, g.y);
            dense_opt_one(R, w.z, a.z, b.z, g.z); dense_opt_one(R, w.w, a.w, b.w, g.w);
            *reinterpret_cast<float4*>(o.accum + i) = a;
            if (two) *reinterpret_cast<float4*>(o.accum2 + i) = b;
            *reinterpret_cast<float4*>(o.theta + i) = w;
            if (o.zero_grad) *reinterpret_cast<float4*>(o.grad + i) = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            for (long long k = i; k < o.n; ++k) {
                float a = o.accum[k], w = o.theta[k], b = two ? o.accum2[k] : 0.f;
                dense_opt_one(R, w, a, b, o.grad[k]);
                o.accum[k] = a; o.theta[k] = w;
                if (two) o.accum2[k] = b;
                if (o.zero_grad) o.grad[k] = 0.f;
            }
        }
    }
}

__global__ void __launch_bounds__(256) exb_dense_opt_kernel(DenseOptArgs o) {
    __shared__ float tile[32][33];
    exb::pdl_trigger();
    exb::pdl_wait();
    dense_opt_step(o, tile);
}

// Adagrad on the flat fp32 buffer (tf.keras semantics: accum += g^2; w -= lr * g / (sqrt(accum) + eps))
__global__ void exb_adagrad_flat_kernel(float* theta, float* accum, const float* grad, long long n, float lr, float eps) {
    exb::pdl_trigger();
    exb::pdl_wait();
    for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4; i < n;
         i += (long long)gridDim.x * blockDim.x * 4) {
        if (i + 3 < n) {
            float4 g = *reinterpret_cast<const float4*>(grad + i);
            float4 a = *reinterpret_cast<float4*>(accum + i);
            float4 w = *reinterpret_cast<float4*>(theta + i);
            a.x += g.x * g.x; a.y += g.y * g.y; a.z += g.z * g.z; a.w += g.w * g.w;
            w.x -= lr * g.x / (sqrtf(a.x) + eps); w.y -= lr * g.y / (sqrtf(a.y) + eps);
            w.z -= lr * g.z / (sqrtf(a.z) + eps); w.w -= lr * g.w / (sqrtf(a.w) + eps);
            *reinterpret_cast<float4*>(accum + i) = a;
            *reinterpret_cast<float4*>(theta + i) = w;
        } else {
            for (long long k = i; k < n; ++k) {
                float g = grad[k], a = accum[k] + g * g;
                accum[k] = a;
                theta[k] -= lr * g / (sqrtf(a) + eps);
            }
        }
    }
}

// W fp32 [R, C] -> Wb bf16 [R, C] and WTb bf16 [C, R] (32x32 smem tile transpose)
__global__ void exb_refresh_bf16_kernel(const float* W, __nv_bfloat16* Wb, __nv_bfloat16* WTb, int R, int C) {
    exb::pdl_trigger();
    exb::pdl_wait();
    __shared__ float tile[32][33];
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        float v = (r < R && c < C) ? W[(size_t)r * C + c] : 0.f;
        tile[i][threadIdx.x] = v;
        if (r < R && c < C) Wb[(size_t)r * C + c] = __float2bfloat16_rn(v);
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < R && c < C) WTb[(size_t)c * R + r] = __float2bfloat16_rn(tile[threadIdx.x][i]);
    }
}

// ---- P2P all-reduce (sum) over peer-mapped buffers, fused with the dense optimizer ------
// ONE persistent kernel (grid <= resident CTAs):
//   signal "my gradients are complete"  | every CTA polls its LOCAL flag row for all peers
//   reduce-scatter + all-gather in one pass: this rank sums its 1/W slice with peer LOADS
//     from every rank and peer-STORES the sum back into every rank's buffer in place (the
//     slice of a buffer is read only by its reducing rank, by the very thread that then
//     overwrites it, so no scratch and no barrier between the two halves)
//   last CTA to finish signals "my stores have landed" | every CTA polls for all peers
//   Adagrad over the whole (now identical on every rank) gradient, fused behind the wait.
// Two flag exchanges per call instead of the three barrier kernels + two memcpys of the
// first version. Flags are monotonically increasing epochs.
struct ArArgs {
    float* buf[8];          // every rank's gradient buffer (peer mapped), index = rank
    unsigned* flags[8];     // every rank's flag array [8]
    unsigned* epoch;        // local
    unsigned* gcount;       // local: CTA arrival counter
    unsigned long long* stamps;   // local, optional: %globaltimer of CTA 0 [start, ready, reduced, landed, done]
    int* status;
    long long n;
    int W, rank;
};

__device__ __forceinline__ void ar_signal(const ArArgs& a, unsigned e) {   // threads < W of one CTA
    if ((int)threadIdx.x < a.W)
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(&a.flags[threadIdx.x][a.rank]), "r"(e) : "memory");
}
// ONE polling thread per CTA reads the whole local flag row (<= 8 words) with two 16-byte loads and
// backs off between polls: W threads x several hundred CTAs re-reading one L2 line every ~0.5 us
// saturated its slice -- CTAs noticed a flag many microseconds after it had been set (per-CTA stamps).
__device__ __forceinline__ bool ar_flags_reached(const unsigned* row, int W, unsigned e) {
    unsigned v[8];
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(row) : "memory");
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7]) : "l"(row + 4) : "memory");
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 8; ++i) ok = ok && (i >= W || (int)(v[i] - e) >= 0);
    return ok;
}
__device__ __forceinline__ void ar_wait(const ArArgs& a, unsigned e) {     // every CTA
    if (threadIdx.x == 0) {
        unsigned long long t0, t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        unsigned ns = 32;
        for (unsigned it = 0; !ar_flags_reached(a.flags[a.rank], a.W, e); ++it) {
            __nanosleep(ns);
            if (ns < 256) ns += 32;
            if ((it & 255u) == 255u) {
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
                if (t1 - t0 > 4000000000ull) { atomicCAS(a.status, 0, 2); break; }
            }
        }
        asm volatile("fence.acq_rel.sys;" ::: "memory");
    }
    __syncthreads();
}

__global__ void __launch_bounds__(256) exb_ar_fused_kernel(ArArgs a, DenseOptArgs o) {
    exb::pdl_trigger();
    exb::pdl_wait();
    __shared__ int s_last;
    __shared__ float opt_tile[32][33];
    const unsigned e0 = *(volatile unsigned*)a.epoch;
#define AR_STAMP(i) do { if (a.stamps && blockIdx.x == 0 && threadIdx.x == 0) { unsigned long long _t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_t)); a.stamps[i] = _t; } } while (0)
    AR_STAMP(0);
#define AR_CTA_STAMP(i) do { if (a.stamps && threadIdx.x == 0) { unsigned long long _t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_t)); a.stamps[16 + 4 * blockIdx.x + (i)] = _t; } } while (0)
    AR_CTA_STAMP(0);
    if (blockIdx.x == 0) ar_signal(a, e0 + 1);     // earlier kernels of this stream wrote the gradients
    ar_wait(a, e0 + 1);
    AR_STAMP(1);
    AR_CTA_STAMP(1);
    const long long per = ((a.n + a.W - 1) / a.W + 3) & ~3ll;
    const long long lo = per * a.rank, hi = min(a.n, lo + per);
    // two float4 per thread and iteration: 2 W independent peer loads in flight before the first use
    const long long stride = (long long)gridDim.x * blockDim.x * 4;
    for (long long i = lo + (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4; i < hi; i += 2 * stride) {
        const long long i2 = i + stride;
        const bool two = i2 < hi;
        float4 v[8], u[8];
#pragma unroll
        for (int r = 0; r < 8; ++r)
            if (r < a.W) {
                v[r] = __ldcg(reinterpret_cast<const float4*>(a.buf[r] + i));   // peer loads over NVLink
                if (two) u[r] = __ldcg(reinterpret_cast<const float4*>(a.buf[r] + i2));
            }
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f), t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int r = 0; r < 8; ++r)
            if (r < a.W) {
                s.x += v[r].x; s.y += v[r].y; s.z += v[r].z; s.w += v[r].w;
                if (two) { t.x += u[r].x; t.y += u[r].y; t.z += u[r].z; t.w += u[r].w; }
            }
#pragma unroll
        for (int r = 0; r < 8; ++r)
            if (r < a.W) {
                __stcg(reinterpret_cast<float4*>(a.buf[r] + i), s);             // peer stores
                if (two) __stcg(reinterpret_cast<float4*>(a.buf[r] + i2), t);
            }
    }
    __syncthreads();
    AR_STAMP(2);
    AR_CTA_STAMP(2);
    if (threadIdx.x == 0) {
        // gpu-scope release of the CTA's (peer) stores into the arrival count; the LAST CTA's
        // st.release.sys below is cumulative over everything it acquired through that count, so only
        // one system-scope fence sits on the critical path (a MEMBAR.SYS with NVLink stores in flight
        // costs microseconds at 8 GPUs)
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
        s_last = atomicAdd(a.gcount, 1u) == gridDim.x - 1;
    }
    AR_CTA_STAMP(3);
    __syncthreads();
    if (s_last) {
        if (threadIdx.x == 0) {
            asm volatile("fence.acq_rel.gpu;" ::: "memory");
            *(volatile unsigned*)a.gcount = 0;
            *(volatile unsigned*)a.epoch = e0 + 2;
            if (a.stamps) { unsigned long long _t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_t)); a.stamps[5] = _t; }
        }
        __syncthreads();
        ar_signal(a, e0 + 2);
        if (a.stamps && threadIdx.x == 0) { unsigned long long _t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_t)); a.stamps[6] = _t; }
    }
    ar_wait(a, e0 + 2);
    AR_STAMP(3);
    if (o.theta == nullptr) return;
    dense_opt_step(o, opt_tile);     // o.grad == a.buf[a.rank]: identical on every rank now
    AR_STAMP(4);
#undef AR_STAMP
}

}  // namespace

extern "C" {

const char* exb_dense_last_error() { return g_dense_err.c_str(); }

int exb_prep(const void* args, int B, int Dp, uint64_t stream) {
    PrepArgs a = *reinterpret_cast<const PrepArgs*>(args);
    (void)Dp;
    dim3 ga((B + 31) / 32, (a.K0p + 255) / 256);
    cudaError_t e;
    if (a.A0T == nullptr && a.Dp >= 4 && 128 % a.Dp == 0 && a.K0p % 4 == 0) {   // one row-wise pass
        e = exb::launch_pdl(exb_prep_row_kernel, dim3((B + 7) / 8), dim3(256), 0, (cudaStream_t)stream, a);
    } else {
        e = exb::launch_pdl(exb_prep_a_kernel, ga, dim3(256), 0, (cudaStream_t)stream, a);
        if (e == cudaSuccess) e = exb::launch_pdl(exb_prep_b_kernel, dim3((B + 7) / 8), dim3(256), 0, (cudaStream_t)stream, a);
    }
    if (e != cudaSuccess) { g_dense_err = cudaGetErrorString(e); return -1; }
    return 0;
}
int exb_prep_args_size() { return (int)sizeof(PrepArgs); }
int exb_head(const void* args, int B, uint64_t stream) {
    HeadArgs a = *reinterpret_cast<const HeadArgs*>(args);
    cudaError_t e;
    if (a.dZT == nullptr && a.Hp <= 64 * EXB_HEAD_MAXP && a.Hp % 2 == 0 && a.g_cache_lin == nullptr) {
        e = exb::launch_pdl(exb_head_row_kernel, dim3((B + 31) / 32), dim3(256), 0, (cudaStream_t)stream, a);
    } else {
        e = exb::launch_pdl(exb_head_a_kernel, dim3((B + 7) / 8), dim3(256), 0, (cudaStream_t)stream, a);
        dim3 gb((B + 31) / 32, (a.Hp + 255) / 256);
        if (e == cudaSuccess) e = exb::launch_pdl(exb_head_b_kernel, gb, dim3(256), 0, (cudaStream_t)stream, a);
    }
    if (e != cudaSuccess) { g_dense_err = cudaGetErrorString(e); return -1; }
    return 0;
}
int exb_head_args_size() { return (int)sizeof(HeadArgs); }
int exb_predict_head(const void* args, uint64_t stream) {
    const PredictArgs a = *reinterpret_cast<const PredictArgs*>(args);
    if (a.Hp < 2 || a.Hp % 2 || ((uintptr_t)a.H & 3) || ((uintptr_t)a.wout & 7) || !a.base || !a.logits || !a.probs) {
        g_dense_err = "predict_head: even Hp, 4-byte aligned H, 8-byte aligned w_out, base / logits / probs required";
        return -1;
    }
    const int grid = a.B > 0 ? (a.B + 7) / 8 : 1;
    cudaError_t e = exb::launch_pdl(exb_predict_head_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, a);
    if (e != cudaSuccess) { g_dense_err = cudaGetErrorString(e); return -1; }
    return 0;
}
int exb_predict_args_size() { return (int)sizeof(PredictArgs); }
int exb_cachegrad(uint64_t G32, long long xs, int col0, int Dp, uint64_t ids, int ncols, uint64_t cache_col,
                  uint64_t cache_off, int nc, uint64_t g_cache_emb, int B, uint64_t dlogit, uint64_t g_cache_lin,
                  uint64_t cache_vocab, uint64_t stream) {
    if (nc == 0) return 0;
    if (Dp % 4 || Dp > EXB_CG_MAXDP) { g_dense_err = "cachegrad: Dp must be a multiple of 4 and <= 128"; return -1; }
    const int grid = nc * ((B + 255) / 256);     // CTA = (cached feature, 256 batch rows)
    const size_t smem = (size_t)8 * 32 * Dp * sizeof(float);
    static bool attr = false;
    if (!attr) { cudaFuncSetAttribute(exb_cachegrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 32 * EXB_CG_MAXDP * 4); attr = true; }
    cudaError_t e = exb::launch_pdl(exb_cachegrad_kernel, dim3(grid), dim3(256), smem, (cudaStream_t)stream, (const float*)G32,
                                    xs, col0, Dp, (const long long*)ids, ncols, (const int*)cache_col,
                                    (const long long*)cache_off, nc, (float*)g_cache_emb, B, (const float*)dlogit,
                                    (float*)g_cache_lin);
    (void)cache_vocab;
    if (e != cudaSuccess) { g_dense_err = cudaGetErrorString(e); return -1; }
    return 0;
}
int exb_adagrad_flat(uint64_t theta, uint64_t accum, uint64_t grad, long long n, float lr, float eps, uint64_t stream) {
    int grid = (int)((n / 4 + 255) / 256);
    if (grid > 132 * 4) grid = 132 * 4;
    if (grid < 1) grid = 1;
    cudaError_t e = exb::launch_pdl(exb_adagrad_flat_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, (float*)theta,
                                    (float*)accum, (const float*)grad, n, lr, eps);
    if (e != cudaSuccess) { g_dense_err = cudaGetErrorString(e); return -1; }
    return 0;
}
int exb_refresh_bf16(uint64_t W, uint64_t Wb, uint64_t WTb, int R, int C, uint64_t stream) {
    dim3 grid((C + 31) / 32, (R + 31) / 32), block(32, 8);
    cudaError_t e = exb::launch_pdl(exb_refresh_bf16_kernel, grid, block, 0, (cudaStream_t)stream, (const float*)W,
                                    (__nv_bfloat16*)Wb, (__nv_bfloat16*)WTb, R, C);
    if (e != cudaSuccess) { g_dense_err = cudaGetErrorString(e); return -1; }
    return 0;
}
// Adagrad + bf16 refresh + gradient clearing of the whole dense parameter buffer in one launch
int exb_dense_opt(const void* args, uint64_t stream) {
    DenseOptArgs o = *reinterpret_cast<const DenseOptArgs*>(args);
    if (o.nmat < 0 || o.nmat > EXB_OPT_MAX_MATS) { g_dense_err = "dense_opt: at most 8 weight matrices"; return -1; }
    int tiles = 0;
    for (int i = 0; i < o.nmat; ++i) tiles += ((o.mat[i].R + 31) / 32) * ((o.mat[i].C + 31) / 32);
    int grid = tiles > 0 ? tiles : 1;
    if (grid > 132 * 8) grid = 132 * 8;
    cudaError_t e = exb::launch_pdl(exb_dense_opt_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, o);
    if (e != cudaSuccess) { g_dense_err = cudaGetErrorString(e); return -1; }
    return 0;
}
int exb_dense_opt_args_size() { return (int)sizeof(DenseOptArgs); }

// all-reduce (sum, in place) of a flat fp32 buffer of n elements (n % 4 == 0, 16-byte aligned)
// that every rank has peer-mapped; bufs/flags: W pointers each; epoch/gcount/status: local words.
// theta/accum != 0: Adagrad step on the reduced gradient inside the same kernel.
int exb_allreduce_adagrad(const uint64_t* bufs, const uint64_t* flags, uint64_t epoch, uint64_t gcount, uint64_t status,
                          long long n, int W, int rank, int ctas, const void* opt_args, uint64_t stream) {
    ArArgs a;
    for (int i = 0; i < 8; ++i) { a.buf[i] = i < W ? (float*)bufs[i] : nullptr; a.flags[i] = i < W ? (unsigned*)flags[i] : nullptr; }
    a.epoch = (unsigned*)epoch; a.gcount = (unsigned*)gcount; a.status = (int*)status; a.n = n; a.W = W; a.rank = rank;
    a.stamps = (unsigned long long*)(gcount + 1024);   // flag block + 4096: phase clock of CTA 0
    if (n % 4) { g_dense_err = "allreduce: n must be a multiple of 4"; return -1; }
    DenseOptArgs o;
    memset(&o, 0, sizeof(o));
    if (opt_args) o = *reinterpret_cast<const DenseOptArgs*>(opt_args);
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // CTAs wait on each other (flag polls, arrival counter): the grid must be resident. Up to 4 CTAs per
    // SM: the optimizer phase walks 32x32 weight tiles grid-strided and wants the parallelism.
    int occ = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, exb_ar_fused_kernel, 256, 0);
    const int resident = sms * std::max(1, std::min(occ, 4));
    if (ctas < 1) ctas = opt_args ? resident : sms;
    if (ctas > resident) ctas = resident;
    cudaError_t e = exb::launch_pdl(exb_ar_fused_kernel, dim3(ctas), dim3(256), 0, (cudaStream_t)stream, a, o);
    if (e != cudaSuccess) { g_dense_err = cudaGetErrorString(e); return -1; }
    return 0;
}

}  // extern "C"
