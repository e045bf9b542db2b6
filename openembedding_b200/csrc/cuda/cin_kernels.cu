// cin_kernels.cu -- the interaction (outer product) half of xDeepFM's Compressed Interaction Network, laid out for the
// wgmma GEMM that does the other half (the 1x1 convolution over the H_k x m interaction channels).
//
// A CIN layer is  out[b, n, d] = relu( sum_{h, j} W[n, h*m + j] * hid[b, h, d] * x[b, j, d] + bias[n] ).
// With rows r = (b, d) this is ONE GEMM  out[R, N] = Z[R, C] W^T  with  Z[r, h*m + j] = hid[r, h] * x[r, j],  C = H_k*m.
// The reference gets it from DeepCTR: tf.einsum / tf.nn.conv1d through TensorFlow -> cuBLAS / cuDNN
// (test/benchmark/criteo_deepctr.py; K6 in SURVEY 2.5), materialising the fp32 interaction tensor and several
// transposed copies. Here:
//   exb_cin_outer_kernel      writes Z directly as the GEMM's K-major bf16 A operand (row stride Kp, a constant-one
//                             column at C that carries the bias, zero padding up to Kp) -- one pass, no fp32 tensor
//   exb_cin_outer_bwd_kernel  folds dZ (the GEMM's dX output, bf16) back into d hid and d x, one warp per row
// Everything stays in the [R = B*D, channels] layout between layers (ops/cin.py).
//
// The fused xDeepFM step (models/fused_dense.py) adds the kernels around them that the eager path leaves to torch:
//   exb_cin_gather_kernel  X32 [B, nf*Dp + ...] (the pulled rows) -> X0 [R, m] fp32, the CIN input
//   exb_cin_pool_kernel    p[b] = concat_k sum_d direct_k[(b, d), :]  and  base[b] += p[b] . w_cin   (all layers)
//   exb_cin_dy_kernel      dY_k = bf16([Y_k > 0] * (dlogit w_cin on direct channels + d hid_{k+1} on handed-on ones)),
//                          and on the last layer's launch g_wcin += sum_b dlogit[b] p[b]
//   exb_cin_fold_kernel    G32[b, j*Dp + d] += dx_0 + dhid_0 + sum_{k>=1} dx_k   at row (b, d), field j
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "pdl.cuh"

namespace {

std::string g_cin_err;

constexpr int CIN_MAX_H = 256;     // channels of the previous layer handed on (DeepCTR: 128 / 2 = 64)
constexpr int CIN_MAX_M = 64;      // fields
constexpr int CIN_WARPS = 8;
constexpr int CIN_MAX_LAYERS = 8;  // layers of the fused step (pool / fold argument arrays)

__device__ __forceinline__ float load_as_float(const void* p, int is_bf16, size_t i) {
    return is_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]) : reinterpret_cast<const float*>(p)[i];
}

// one warp per row r: Z[r, h*m + j] = hid[r, h] * x[r, j]; Z[r, C] = 1; Z[r, C+1 .. Kp) = 0
__global__ void __launch_bounds__(CIN_WARPS * 32) exb_cin_outer_kernel(const void* hid, int hid_bf16, long long ld_hid, int H,
                                                                        const float* x, long long ld_x, int m,
                                                                        __nv_bfloat16* Z, long long ldz, int Kp, int R) {
    exb::pdl_trigger();
    exb::pdl_wait();
    __shared__ float s_h[CIN_WARPS][CIN_MAX_H];
    __shared__ float s_x[CIN_WARPS][CIN_MAX_M];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int C = H * m;
    for (int r = blockIdx.x * CIN_WARPS + warp; r < R; r += gridDim.x * CIN_WARPS) {
        for (int h = lane; h < H; h += 32) s_h[warp][h] = load_as_float(hid, hid_bf16, (size_t)r * ld_hid + h);
        for (int j = lane; j < m; j += 32) s_x[warp][j] = x[(size_t)r * ld_x + j];
        __syncwarp();
        __nv_bfloat16* zr = Z + (size_t)r * ldz;
        // (h, j) of the lane's first column, then advanced by 256 columns per iteration without dividing again
        const int dh = 256 / m, dj = 256 - dh * m;
        int h0 = (lane * 8) / m, j0 = lane * 8 - h0 * m;
        for (int c0 = lane * 8; c0 < Kp; c0 += 32 * 8) {       // 16 bytes per lane and iteration
            int h = h0, j = j0;
            h0 += dh; j0 += dj;
            if (j0 >= m) { j0 -= m; ++h0; }
            __align__(16) __nv_bfloat16 v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int c = c0 + k;
                float f = 0.f;
                if (c < C) f = s_h[warp][h] * s_x[warp][j];
                else if (c == C) f = 1.f;
                v[k] = __float2bfloat16_rn(f);
                if (++j == m) { j = 0; ++h; }
            }
            *reinterpret_cast<uint4*>(zr + c0) = *reinterpret_cast<const uint4*>(v);
        }
        __syncwarp();
    }
}

// one warp per row r:  dhid[r, h] = sum_j dZ[r, h*m + j] * x[r, j],   dx[r, j] = sum_h dZ[r, h*m + j] * hid[r, h]
// The dZ row is staged in shared memory AS bf16 (16-byte copies, no conversion pass): both reductions then read 2-byte
// elements -- lane h walks m consecutive elements (word stride m/2 between lanes: odd for the usual even m = 26, so no
// bank conflicts), lane j reads element h*m + j (consecutive lanes, consecutive elements).
__global__ void __launch_bounds__(CIN_WARPS * 32) exb_cin_outer_bwd_kernel(const __nv_bfloat16* dZ, long long ldz,
                                                                            const void* hid, int hid_bf16, long long ld_hid, int H,
                                                                            const float* x, long long ld_x, int m,
                                                                            float* dhid, long long ld_dhid, float* dx, long long ld_dx,
                                                                            int R) {
    exb::pdl_trigger();
    exb::pdl_wait();
    extern __shared__ __align__(16) unsigned char cin_smem[];
    __shared__ float s_hx[CIN_WARPS][CIN_MAX_H + CIN_MAX_M];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int C = H * m;
    const int Cp = (C + 7) & ~7;
    __nv_bfloat16* s_dz = reinterpret_cast<__nv_bfloat16*>(cin_smem) + (size_t)warp * Cp;
    float* s_h = s_hx[warp];
    float* s_x = s_h + CIN_MAX_H;
    for (int r = blockIdx.x * CIN_WARPS + warp; r < R; r += gridDim.x * CIN_WARPS) {
        const __nv_bfloat16* zr = dZ + (size_t)r * ldz;
        for (int c0 = lane * 8; c0 < Cp; c0 += 32 * 8)
            *reinterpret_cast<uint4*>(s_dz + c0) = *reinterpret_cast<const uint4*>(zr + c0);
        for (int h = lane; h < H; h += 32) s_h[h] = load_as_float(hid, hid_bf16, (size_t)r * ld_hid + h);
        for (int j = lane; j < m; j += 32) s_x[j] = x[(size_t)r * ld_x + j];
        __syncwarp();
        for (int h = lane; h < H; h += 32) {
            const __nv_bfloat16* p = s_dz + h * m;
            float a = 0.f;
            for (int j = 0; j < m; ++j) a += __bfloat162float(p[j]) * s_x[j];
            dhid[(size_t)r * ld_dhid + h] = a;
        }
        for (int j = lane; j < m; j += 32) {
            float a0 = 0.f, a1 = 0.f;
            int h = 0;
            for (; h + 1 < H; h += 2) {
                a0 += __bfloat162float(s_dz[h * m + j]) * s_h[h];
                a1 += __bfloat162float(s_dz[(h + 1) * m + j]) * s_h[h + 1];
            }
            if (h < H) a0 += __bfloat162float(s_dz[h * m + j]) * s_h[h];
            dx[(size_t)r * ld_dx + j] = a0 + a1;
        }
        __syncwarp();
    }
}

// ---- the fused step ----

// one CTA per sample b: X0[b*D + d, j] = X32[b, j*Dp + d] (d < D: the pad columns Dp - D are not CIN input)
__global__ void __launch_bounds__(256) exb_cin_gather_kernel(const float* __restrict__ X32, long long xs, int Dp, int D,
                                                             int m, float* __restrict__ X0, int B) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const int n = m * D;
    for (int b = blockIdx.x; b < B; b += gridDim.x) {
        const float* xr = X32 + (size_t)b * xs;
        float* out = X0 + (size_t)b * n;             // the D rows of sample b are contiguous
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int j = i / D, d = i - j * D;       // d fastest: coalesced reads of X32
            out[d * m + j] = xr[j * Dp + d];
        }
    }
}

struct CinPoolArgs {
    const __nv_bfloat16* Y[CIN_MAX_LAYERS];   // layer outputs [R, ldy]
    long long ldy[CIN_MAX_LAYERS];
    int lo[CIN_MAX_LAYERS], hi[CIN_MAX_LAYERS];   // direct channels [lo, hi) of each layer
    int K, T, D, B;                            // T = sum of (hi - lo): width of p
    const float* wcin;                         // [T]
    float* p;                                  // [B, T]
    float* base;                               // [B]
};

// one warp per sample: p[b, t] = sum_d Y_k[b*D + d, lo_k + t - t0_k]; base[b] += p[b] . wcin (the warp is the only
// writer of base[b])
__global__ void __launch_bounds__(CIN_WARPS * 32) exb_cin_pool_kernel(CinPoolArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int b = blockIdx.x * CIN_WARPS + warp; b < a.B; b += gridDim.x * CIN_WARPS) {
        float acc = 0.f;
        int t0 = 0;
        for (int k = 0; k < a.K; ++k) {
            const __nv_bfloat16* y = a.Y[k] + (size_t)b * a.D * a.ldy[k];
            const int w = a.hi[k] - a.lo[k];
            for (int t = lane; t < w; t += 32) {
                const __nv_bfloat16* col = y + a.lo[k] + t;
                float s = 0.f;
                for (int d = 0; d < a.D; ++d) s += __bfloat162float(col[(size_t)d * a.ldy[k]]);
                a.p[(size_t)b * a.T + t0 + t] = s;
                acc += s * a.wcin[t0 + t];
            }
            t0 += w;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) a.base[b] += acc;
    }
}

struct CinDyArgs {
    const __nv_bfloat16* Y; long long ldy;     // layer output [R, Np]
    int N, Np;                                  // real / padded channels
    int dir_lo, t0;                             // direct channels [dir_lo, N): weight wcin[t0 + n - dir_lo]
    const float* wcin;
    const float* dhid; long long ld_dhid;       // gradient of the next layer's input [R, Hn] (fp32)
    int Hn;                                     // channels [0, Hn) are handed on (0 on the last layer)
    int D, R;
    const float* dlogit;                        // [B]
    __nv_bfloat16* dY; long long lddy;          // [R, Np]
    // g_wcin[t] += sum_b dlogit[b] p[b, t] by the CTAs past `main_ctas` (g_wcin == nullptr: none)
    const float* p; float* g_wcin; int T, B, main_ctas;
};

// dY[r, n] = bf16([Y[r, n] > 0] * g), g = dlogit[r / D] * wcin[..] on a direct channel, dhid[r, n] on a handed-on one
// (both without split_half), 0 on a pad channel. 8 channels (16 bytes) per thread.
__global__ void __launch_bounds__(256) exb_cin_dy_kernel(CinDyArgs a) {
    exb::pdl_trigger();
    exb::pdl_wait();
    if ((int)blockIdx.x >= a.main_ctas) {        // g_wcin: 256 samples per CTA, 32 per warp, lanes over channels
        __shared__ float s_part[8][32];
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const int b0 = ((int)blockIdx.x - a.main_ctas) * 256 + warp * 32;
        for (int tb = 0; tb < a.T; tb += 32) {
            const int t = tb + lane;
            float s = 0.f;
            if (t < a.T)
                for (int i = 0; i < 32; ++i) {
                    const int b = b0 + i;
                    if (b < a.B) s += a.dlogit[b] * a.p[(size_t)b * a.T + t];
                }
            s_part[warp][lane] = s;
            __syncthreads();
            if (warp == 0 && t < a.T) {
                float tot = 0.f;
#pragma unroll
                for (int w = 0; w < 8; ++w) tot += s_part[w][lane];
                atomicAdd(a.g_wcin + t, tot);
            }
            __syncthreads();
        }
        return;
    }
    const int per_row = a.Np / 8;
    const long long total = (long long)a.R * per_row;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)a.main_ctas * blockDim.x) {
        const int r = (int)(i / per_row), c0 = (int)(i - (long long)r * per_row) * 8;
        const float dl = a.dlogit[r / a.D];
        const uint4 yv = *reinterpret_cast<const uint4*>(a.Y + (size_t)r * a.ldy + c0);
        const __nv_bfloat16* y = reinterpret_cast<const __nv_bfloat16*>(&yv);
        __align__(16) __nv_bfloat16 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int n = c0 + k;
            float g = 0.f;
            if (n < a.N && __bfloat162float(y[k]) > 0.f) {
                const bool dir = n >= a.dir_lo, hid = n < a.Hn;
                if (dir) g = __fmul_rn(dl, a.wcin[a.t0 + n - a.dir_lo]);
                if (hid) {
                    const float h = a.dhid[(size_t)r * a.ld_dhid + n];
                    g = dir ? __fadd_rn(g, h) : h;
                }
            }
            v[k] = __float2bfloat16_rn(g);
        }
        *reinterpret_cast<uint4*>(a.dY + (size_t)r * a.lddy + c0) = *reinterpret_cast<const uint4*>(v);
    }
}

struct CinFoldArgs {
    const float* src[CIN_MAX_LAYERS + 1];       // [R, m] each, summed in this order
    int nsrc;
};

// one CTA per sample b: G32[b, j*Dp + d] += sum_q src_q[b*D + d, j]   (d < D)
__global__ void __launch_bounds__(256) exb_cin_fold_kernel(float* __restrict__ G32, long long xs, int Dp, int D, int m,
                                                           int B, CinFoldArgs s) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const int n = m * D;
    for (int b = blockIdx.x; b < B; b += gridDim.x) {
        float* gr = G32 + (size_t)b * xs;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int j = i / D, d = i - j * D;       // d fastest: coalesced G32 read-modify-write
            const size_t k = (size_t)b * n + d * m + j;
            float acc = s.src[0][k];
#pragma unroll
            for (int q = 1; q < CIN_MAX_LAYERS + 1; ++q)     // constant indices: the pointers stay in parameter space
                if (q < s.nsrc) acc += s.src[q][k];
            gr[j * Dp + d] += acc;
        }
    }
}

}  // namespace

extern "C" {

const char* exb_cin_last_error() { return g_cin_err.c_str(); }

int exb_cin_outer(uint64_t hid, int hid_bf16, long long ld_hid, int H, uint64_t x, long long ld_x, int m, uint64_t Z,
                  long long ldz, int Kp, int R, uint64_t stream) {
    if (H > CIN_MAX_H || m > CIN_MAX_M || H < 1 || m < 1) { g_cin_err = "cin_outer: H <= 256, m <= 64"; return -1; }
    if (Kp % 8 || H * m + 1 > Kp || ldz % 8) { g_cin_err = "cin_outer: Kp must be a multiple of 8 and hold H*m + 1 columns"; return -1; }
    int grid = (R + CIN_WARPS - 1) / CIN_WARPS;
    if (grid > 132 * 16) grid = 132 * 16;
    cudaError_t e = exb::launch_pdl(exb_cin_outer_kernel, dim3(grid), dim3(CIN_WARPS * 32), 0, (cudaStream_t)stream,
                                    (const void*)hid, hid_bf16, ld_hid, H, (const float*)x, ld_x, m, (__nv_bfloat16*)Z, ldz, Kp, R);
    if (e != cudaSuccess) { g_cin_err = cudaGetErrorString(e); return -1; }
    return 0;
}

int exb_cin_outer_bwd(uint64_t dZ, long long ldz, uint64_t hid, int hid_bf16, long long ld_hid, int H, uint64_t x,
                      long long ld_x, int m, uint64_t dhid, long long ld_dhid, uint64_t dx, long long ld_dx, int R,
                      uint64_t stream) {
    if (H > CIN_MAX_H || m > CIN_MAX_M || H < 1 || m < 1) { g_cin_err = "cin_outer_bwd: H <= 256, m <= 64"; return -1; }
    const int C = H * m, Cp = (C + 7) & ~7;
    if (ldz % 8 || Cp > ldz) { g_cin_err = "cin_outer_bwd: dZ rows must be 16-byte aligned and hold H*m columns"; return -1; }
    const size_t smem = (size_t)CIN_WARPS * Cp * sizeof(__nv_bfloat16);
    if (smem > 200 * 1024) { g_cin_err = "cin_outer_bwd: H*m too large for the shared-memory row buffers"; return -1; }
    static size_t attr = 0;
    if (smem > attr) {
        cudaFuncSetAttribute(exb_cin_outer_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr = smem;
    }
    int grid = (R + CIN_WARPS - 1) / CIN_WARPS;
    if (grid > 132 * 8) grid = 132 * 8;
    cudaError_t e = exb::launch_pdl(exb_cin_outer_bwd_kernel, dim3(grid), dim3(CIN_WARPS * 32), smem, (cudaStream_t)stream,
                                    (const __nv_bfloat16*)dZ, ldz, (const void*)hid, hid_bf16, ld_hid, H, (const float*)x, ld_x, m,
                                    (float*)dhid, ld_dhid, (float*)dx, ld_dx, R);
    if (e != cudaSuccess) { g_cin_err = cudaGetErrorString(e); return -1; }
    return 0;
}

int exb_cin_gather(uint64_t X32, long long xs, int Dp, int D, int m, uint64_t X0, int B, uint64_t stream) {
    if (m < 1 || m > CIN_MAX_M || D < 1 || D > Dp) { g_cin_err = "cin_gather: 1 <= m <= 64, 1 <= D <= Dp"; return -1; }
    const int grid = B < 132 * 16 ? B : 132 * 16;
    cudaError_t e = exb::launch_pdl(exb_cin_gather_kernel, dim3(grid > 0 ? grid : 1), dim3(256), 0, (cudaStream_t)stream,
                                    (const float*)X32, xs, Dp, D, m, (float*)X0, B);
    if (e != cudaSuccess) { g_cin_err = cudaGetErrorString(e); return -1; }
    return 0;
}

int exb_cin_pool(const void* args, uint64_t stream) {
    const CinPoolArgs a = *reinterpret_cast<const CinPoolArgs*>(args);
    if (a.K < 1 || a.K > CIN_MAX_LAYERS) { g_cin_err = "cin_pool: 1..8 layers"; return -1; }
    int grid = (a.B + CIN_WARPS - 1) / CIN_WARPS;
    if (grid > 132 * 8) grid = 132 * 8;
    cudaError_t e = exb::launch_pdl(exb_cin_pool_kernel, dim3(grid > 0 ? grid : 1), dim3(CIN_WARPS * 32), 0,
                                    (cudaStream_t)stream, a);
    if (e != cudaSuccess) { g_cin_err = cudaGetErrorString(e); return -1; }
    return 0;
}
int exb_cin_pool_args_size() { return (int)sizeof(CinPoolArgs); }

int exb_cin_dy(const void* args, uint64_t stream) {
    CinDyArgs a = *reinterpret_cast<const CinDyArgs*>(args);
    if (a.Np % 8 || a.ldy % 8 || a.lddy % 8 || a.N > a.Np) { g_cin_err = "cin_dy: Np and the row strides must be multiples of 8"; return -1; }
    long long main = ((long long)a.R * (a.Np / 8) + 255) / 256;
    if (main > 132 * 16) main = 132 * 16;
    a.main_ctas = (int)(main > 0 ? main : 1);
    const int extra = a.g_wcin ? (a.B + 255) / 256 : 0;
    cudaError_t e = exb::launch_pdl(exb_cin_dy_kernel, dim3(a.main_ctas + extra), dim3(256), 0, (cudaStream_t)stream, a);
    if (e != cudaSuccess) { g_cin_err = cudaGetErrorString(e); return -1; }
    return 0;
}
int exb_cin_dy_args_size() { return (int)sizeof(CinDyArgs); }

int exb_cin_fold(uint64_t G32, long long xs, int Dp, int D, int m, int B, const uint64_t* srcs, int nsrc, uint64_t stream) {
    if (nsrc < 1 || nsrc > CIN_MAX_LAYERS + 1) { g_cin_err = "cin_fold: 1..9 source buffers"; return -1; }
    if (m < 1 || m > CIN_MAX_M || D < 1 || D > Dp) { g_cin_err = "cin_fold: 1 <= m <= 64, 1 <= D <= Dp"; return -1; }
    CinFoldArgs s = {};
    for (int q = 0; q < nsrc; ++q) s.src[q] = (const float*)srcs[q];
    s.nsrc = nsrc;
    const int grid = B < 132 * 16 ? B : 132 * 16;
    cudaError_t e = exb::launch_pdl(exb_cin_fold_kernel, dim3(grid > 0 ? grid : 1), dim3(256), 0, (cudaStream_t)stream,
                                    (float*)G32, xs, Dp, D, m, B, s);
    if (e != cudaSuccess) { g_cin_err = cudaGetErrorString(e); return -1; }
    return 0;
}

}  // extern "C"
