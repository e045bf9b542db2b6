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

}  // extern "C"
