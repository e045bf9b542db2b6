// cross_kernels.cu -- the elementwise half of DCN-v2's cross network in the fused step (models/fused_dense.py); the
// wgmma GEMM (gemm_wgmma.cu, single launches) does the other half.
//
// A cross layer is  x_{l+1} = x0 * (W_l x_l + b_l) + x_l  over the n = nf*D + nd real columns of the step's A0 layout
//   [nf*Dp embedding columns | nd dense | zero pad | ones column at K0p-1].
// b_l sits in W_l's ones column, so U_l = x_l W_l^T is one GEMM with a plain fp32 store (EPI_DX_FM, fm_cols = 0).
// Rows are samples, one warp per sample, 4 columns per lane and access:
//   exb_cross_fwd_kernel      Xf_{l+1} = x0 * U_l + X_l (fp32, rounded product then rounded sum: no contraction),
//                             Xb_{l+1} = bf16(Xf_{l+1}) (the next layer's GEMM operand), ones column 1, other columns 0;
//                             the last layer's launch also adds x_L . w_cross to base[b] (the warp is its only writer)
//   exb_cross_bwd_top_kernel  g_L = dlogit w_cross, dU_{L-1} = bf16(g_L x0), gx0 = g_L U_{L-1};
//                             CTAs past `main_ctas`: g_wcross[c] += sum_b dlogit[b] Xf_L[b, c]
//   exb_cross_bwd_kernel      g_l = g_{l+1} + P_l  (P_l = dU_l W_l, the GEMM launched before it);
//                             l > 0: dU_{l-1} = bf16(g_l x0), gx0 += g_l U_{l-1};
//                             l = 0: G32[b, c] += gx0 + g_0 on the real embedding columns (before cachegrad and the push)
// x0 is never copied: its embedding columns are X32's (the pulled rows; prep copies the cached rows there) and its
// dense columns the caller's fp32 dense input. The columns that are not real (embedding pad Dp - D, pad, ones) carry
// zero weights; the kernels mask them anyway, so every gradient that reaches them is exactly 0.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "pdl.cuh"

namespace {

std::string g_cross_err;

constexpr int CROSS_WARPS = 8;
constexpr int WC_COLS = 256;       // g_wcross CTAs: one column per thread ...
constexpr int WC_ROWS = 128;       // ... over this many samples

struct CrossX0 {                   // x0[b] = [X32[b, :E] | dense[b, :nd] | 0 ... | 1]
    const float* X32; long long xs;
    const float* dense; int nd;
    int E, Dp, D, K0p, B;          // E = nf * Dp
};

struct CrossFwdArgs {
    CrossX0 x;
    const float* U;                // [B, K0p] U_l
    const float* Xin;              // [B, K0p] X_l; nullptr: x0 (layer 0)
    float* Xf;                     // [B, K0p] X_{l+1}
    __nv_bfloat16* Xb;             // [B, K0p] bf16(X_{l+1}); nullptr on the last layer (no GEMM reads it)
    const float* wcross;           // [K0p]; the last layer: base[b] += X_L[b] . w_cross
    float* base;                   // nullptr below the last layer
};

struct CrossBwdArgs {
    CrossX0 x;
    const float* dlogit;           // [B] (top)
    const float* wcross;           // [K0p] (top)
    const float* gin;              // [B, K0p] g_{l+1} (layer)
    const float* P;                // [B, K0p] P_l (layer)
    float* gout;                   // [B, K0p] g_L (top) / g_l (layer; nullptr: not stored)
    const float* U;                // [B, K0p] U_{L-1} (top) / U_{l-1} (layer l > 0)
    __nv_bfloat16* dU;             // [B, K0p] dU_{L-1} (top) / dU_{l-1} (layer l > 0)
    float* gx0;                    // [B, K0p] written (top), accumulated (l > 0), read (l = 0)
    float* G32;                    // layer 0: the embedding-gradient buffer, row stride x.xs; nullptr for l > 0
    const float* XfL;              // [B, K0p] X_L (top: g_wcross)
    float* g_wcross;               // [K0p]
    int main_ctas;                 // set by the launcher
};

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void unpack(const float4& f, float (&v)[4]) { v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w; }
__device__ __forceinline__ void st_bf16x4(__nv_bfloat16* p, const float (&v)[4]) {
    __align__(8) __nv_bfloat162 h[2] = {__floats2bfloat162_rn(v[0], v[1]), __floats2bfloat162_rn(v[2], v[3])};
    *reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(h);
}

// real columns among c0 .. c0+3 (c0 % 4 == 0; E and Dp are multiples of 4, so the group lies in one feature or past E)
__device__ __forceinline__ void real_mask(const CrossX0& x, int c0, bool (&r)[4]) {
    if (c0 < x.E) {
        const int d0 = c0 % x.Dp;
#pragma unroll
        for (int k = 0; k < 4; ++k) r[k] = d0 + k < x.D;
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) r[k] = c0 + k - x.E < x.nd;
    }
}

__device__ __forceinline__ void load_x0(const CrossX0& x, int b, int c0, float (&v)[4]) {
    if (c0 < x.E) {
        unpack(ld4(x.X32 + (size_t)b * x.xs + c0), v);
        return;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int i = c0 + k - x.E;
        v[k] = i < x.nd ? x.dense[(size_t)b * x.nd + i] : 0.f;
    }
}

__global__ void __launch_bounds__(CROSS_WARPS * 32) exb_cross_fwd_kernel(CrossFwdArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const CrossX0& x = a.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int b = blockIdx.x * CROSS_WARPS + warp; b < x.B; b += gridDim.x * CROSS_WARPS) {
        const size_t row = (size_t)b * x.K0p;
        float acc = 0.f;
        for (int c0 = lane * 4; c0 < x.K0p; c0 += 128) {
            bool r[4];
            float x0[4], u[4], xi[4], o[4];
            real_mask(x, c0, r);
            load_x0(x, b, c0, x0);
            unpack(ld4(a.U + row + c0), u);
            if (a.Xin) unpack(ld4(a.Xin + row + c0), xi);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float xl = a.Xin ? xi[k] : x0[k];
                o[k] = r[k] ? __fadd_rn(__fmul_rn(x0[k], u[k]), xl) : (c0 + k == x.K0p - 1 ? 1.f : 0.f);
            }
            if (a.base) {
                float w[4];
                unpack(ld4(a.wcross + c0), w);
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (r[k]) acc += o[k] * w[k];
            }
            st4(a.Xf + row + c0, o);
            if (a.Xb) st_bf16x4(a.Xb + row + c0, o);
        }
        if (a.base) {
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
            if (lane == 0) a.base[b] += acc;
        }
    }
}

__global__ void __launch_bounds__(CROSS_WARPS * 32) exb_cross_bwd_top_kernel(CrossBwdArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const CrossX0& x = a.x;
    if ((int)blockIdx.x >= a.main_ctas) {        // g_wcross: WC_COLS columns x WC_ROWS samples per CTA
        const int e = (int)blockIdx.x - a.main_ctas;
        const int ncb = (x.K0p + WC_COLS - 1) / WC_COLS;
        const int c = (e % ncb) * WC_COLS + (int)threadIdx.x, b0 = (e / ncb) * WC_ROWS;
        if (c >= x.K0p) return;
        const bool real = c < x.E ? c % x.Dp < x.D : c - x.E < x.nd;
        if (!real) return;
        const int b1 = min(b0 + WC_ROWS, x.B);
        float s = 0.f;
        for (int b = b0; b < b1; ++b) s += a.dlogit[b] * a.XfL[(size_t)b * x.K0p + c];
        atomicAdd(a.g_wcross + c, s);
        return;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int b = blockIdx.x * CROSS_WARPS + warp; b < x.B; b += a.main_ctas * CROSS_WARPS) {
        const size_t row = (size_t)b * x.K0p;
        const float dl = a.dlogit[b];
        for (int c0 = lane * 4; c0 < x.K0p; c0 += 128) {
            bool r[4];
            float x0[4], w[4], u[4], g[4], du[4], gx[4];
            real_mask(x, c0, r);
            load_x0(x, b, c0, x0);
            unpack(ld4(a.wcross + c0), w);
            unpack(ld4(a.U + row + c0), u);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                g[k] = r[k] ? __fmul_rn(dl, w[k]) : 0.f;
                du[k] = r[k] ? __fmul_rn(g[k], x0[k]) : 0.f;
                gx[k] = r[k] ? __fmul_rn(g[k], u[k]) : 0.f;
            }
            st4(a.gout + row + c0, g);
            st_bf16x4(a.dU + row + c0, du);
            st4(a.gx0 + row + c0, gx);
        }
    }
}

__global__ void __launch_bounds__(CROSS_WARPS * 32) exb_cross_bwd_kernel(CrossBwdArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const CrossX0& x = a.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cend = a.G32 ? x.E : x.K0p;        // layer 0 only folds into the embedding columns
    for (int b = blockIdx.x * CROSS_WARPS + warp; b < x.B; b += gridDim.x * CROSS_WARPS) {
        const size_t row = (size_t)b * x.K0p;
        for (int c0 = lane * 4; c0 < cend; c0 += 128) {
            bool r[4];
            float gi[4], p[4], g[4], gx[4];
            real_mask(x, c0, r);
            unpack(ld4(a.gin + row + c0), gi);
            unpack(ld4(a.P + row + c0), p);
#pragma unroll
            for (int k = 0; k < 4; ++k) g[k] = r[k] ? __fadd_rn(gi[k], p[k]) : 0.f;
            if (a.gout) st4(a.gout + row + c0, g);
            unpack(ld4(a.gx0 + row + c0), gx);
            if (a.G32) {
                float* gp = a.G32 + (size_t)b * x.xs + c0;
                float G[4];
                unpack(ld4(gp), G);
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (r[k]) G[k] = __fadd_rn(G[k], __fadd_rn(gx[k], g[k]));
                st4(gp, G);
            } else {
                float x0[4], u[4], du[4];
                load_x0(x, b, c0, x0);
                unpack(ld4(a.U + row + c0), u);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    du[k] = r[k] ? __fmul_rn(g[k], x0[k]) : 0.f;
                    gx[k] = r[k] ? __fadd_rn(gx[k], __fmul_rn(g[k], u[k])) : 0.f;
                }
                st_bf16x4(a.dU + row + c0, du);
                st4(a.gx0 + row + c0, gx);
            }
        }
    }
}

bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

bool check_x0(const CrossX0& x, const char* who) {
    if (x.B < 0 || x.K0p % 64 || x.Dp % 4 || x.E % x.Dp || x.D < 1 || x.D > x.Dp || x.nd < 0 ||
        x.E + x.nd >= x.K0p || x.xs % 4 || x.xs < x.E || !al16(x.X32) || (x.nd > 0 && !x.dense)) {
        g_cross_err = std::string(who) + ": layout [nf*Dp | nd | pad | 1] with K0p % 64 == 0, Dp % 4 == 0, "
                      "16-byte aligned X32 rows";
        return false;
    }
    return true;
}

int grid_rows(int B) {
    const int g = (B + CROSS_WARPS - 1) / CROSS_WARPS;
    return g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g);
}

}  // namespace

extern "C" {

const char* exb_cross_last_error() { return g_cross_err.c_str(); }
int exb_cross_fwd_args_size() { return (int)sizeof(CrossFwdArgs); }
int exb_cross_bwd_args_size() { return (int)sizeof(CrossBwdArgs); }

int exb_cross_fwd(const void* args, uint64_t stream) {
    const CrossFwdArgs a = *reinterpret_cast<const CrossFwdArgs*>(args);
    if (!check_x0(a.x, "cross_fwd")) return -1;
    if (!al16(a.U) || !al16(a.Xin) || !al16(a.Xf) || !a.Xf || !a.U || ((uintptr_t)a.Xb & 7) ||
        (a.base && (!a.wcross || !al16(a.wcross)))) {
        g_cross_err = "cross_fwd: U / X_l / X_{l+1} / w_cross must be 16-byte aligned (bf16 X: 8-byte)";
        return -1;
    }
    cudaError_t e = exb::launch_pdl(exb_cross_fwd_kernel, dim3(grid_rows(a.x.B)), dim3(CROSS_WARPS * 32), 0,
                                    (cudaStream_t)stream, a);
    if (e != cudaSuccess) { g_cross_err = cudaGetErrorString(e); return -1; }
    return 0;
}

int exb_cross_bwd_top(const void* args, uint64_t stream) {
    CrossBwdArgs a = *reinterpret_cast<const CrossBwdArgs*>(args);
    if (!check_x0(a.x, "cross_bwd_top")) return -1;
    if (!a.dlogit || !a.wcross || !al16(a.wcross) || !a.U || !al16(a.U) || !a.gout || !al16(a.gout) || !a.dU ||
        ((uintptr_t)a.dU & 7) || !a.gx0 || !al16(a.gx0) || !a.XfL || !a.g_wcross) {
        g_cross_err = "cross_bwd_top: dlogit, w_cross, U, g, dU, gx0, X_L and g_wcross are required and aligned";
        return -1;
    }
    a.main_ctas = grid_rows(a.x.B);
    const int extra = ((a.x.K0p + WC_COLS - 1) / WC_COLS) * ((a.x.B + WC_ROWS - 1) / WC_ROWS);
    static_assert(WC_COLS == CROSS_WARPS * 32, "one g_wcross column per thread");
    cudaError_t e = exb::launch_pdl(exb_cross_bwd_top_kernel, dim3(a.main_ctas + extra), dim3(CROSS_WARPS * 32), 0,
                                    (cudaStream_t)stream, a);
    if (e != cudaSuccess) { g_cross_err = cudaGetErrorString(e); return -1; }
    return 0;
}

int exb_cross_bwd(const void* args, uint64_t stream) {
    const CrossBwdArgs a = *reinterpret_cast<const CrossBwdArgs*>(args);
    if (!check_x0(a.x, "cross_bwd")) return -1;
    const bool fold = a.G32 != nullptr;
    if (!a.gin || !al16(a.gin) || !a.P || !al16(a.P) || !al16(a.gout) || !a.gx0 || !al16(a.gx0) ||
        (fold ? !al16(a.G32) : (!a.U || !al16(a.U) || !a.dU || ((uintptr_t)a.dU & 7)))) {
        g_cross_err = "cross_bwd: g_{l+1}, P, gx0 and (l = 0) G32 or (l > 0) U, dU are required and aligned";
        return -1;
    }
    cudaError_t e = exb::launch_pdl(exb_cross_bwd_kernel, dim3(grid_rows(a.x.B)), dim3(CROSS_WARPS * 32), 0,
                                    (cudaStream_t)stream, a);
    if (e != cudaSuccess) { g_cross_err = cudaGetErrorString(e); return -1; }
    return 0;
}

}  // extern "C"
