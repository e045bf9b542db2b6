// autoint_kernels.cu -- the attention half of AutoInt's stacked field self-attention in the fused step
// (models/fused_dense.py); the wgmma GEMM (gemm_wgmma.cu, single launches) does the projections and their gradients.
//
// Rows are r = (sample b, field i) = b * nf + i, fields in the A0 order (server features, then cached ones). A layer
// with input X_l [B*nf, d_l] projects once: QKVR = X_l T_l with the stacked weight T_l = [W_Q | W_K | W_V | W_R]
// (fp32 out, [B*nf, Np], column blocks of dh = d * h). Per sample and head (columns eta*d .. eta*d + d - 1 of a block):
//   exb_att_gather_kernel  layer 0's operand: Xb0[r, c] = bf16(X32[b, i*Dp + c]) for c < D, 0 up to Kp0 (prep has
//                          copied the cached rows into X32)
//   exb_att_fwd_kernel     S = Q K^T, P = softmax(S) (max-subtracted, expf), X_{l+1} = relu(P V + R) in fp32 and its
//                          bf16 copy (zero-padded, the next layer's GEMM operand); P [B, h, nf, nf] is kept for the
//                          backward. The last layer's launch adds flatten(X_L) . w_att to base[b].
//   exb_att_bwd_kernel     dY = dX_{l+1} * [X_{l+1} > 0] (the last layer: dX_L = dlogit w_att), dO = dR = dY,
//                          dS = P * (dO V^T - rowsum(dO V^T * P)), dQ = dS K, dK = dS^T Q, dV = P^T dO, written as one
//                          bf16 operand [dQ | dK | dV | dR | 0] [B*nf, Np] for the weight- and input-gradient GEMMs.
//                          The last layer's launch has extra CTAs that write per-128-sample partial sums of
//                          g_watt = sum_b dlogit[b] flatten(X_L[b]).
//   exb_att_fold_kernel    G32[b, i*Dp + c] += dX_0[r, c] for c < D (before cachegrad and the push), and
//                          g_watt += the partial sums in chunk order (no atomics: the result is deterministic).
// One CTA per sample: its Q, K, V (and dO, P, dS in the backward) sit in shared memory; every sum runs in a fixed order.
// Limits (checked on the host, models/fused_dense.py: autoint_dims): nf <= 64 (two score columns per lane),
// dh <= 64 (the bf16 X_{l+1} operand is one 64-column K block).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <string>

#include "pdl.cuh"

namespace {

std::string g_att_err;

constexpr int ATT_WARPS = 8;
constexpr int ATT_THREADS = ATT_WARPS * 32;
constexpr int ATT_MAX_NF = 64;
constexpr int ATT_MAX_DH = 64;
constexpr int GW_ROWS = 128;       // samples per partial sum of g_watt

struct AttFwdArgs {
    const float* QKVR; int Np;     // [B*nf, Np] projections (Q | K | V | R)
    float* P;                      // [B, h, nf, nf] softmax
    float* Xf;                     // [B*nf, dh] X_{l+1}
    __nv_bfloat16* Xb; int ldxb;   // [B*nf, ldxb] bf16(X_{l+1}), zero past dh; nullptr on the last layer
    const float* watt;             // [nf*dh] (last layer)
    float* base;                   // [B]; nullptr below the last layer
    int B, nf, d, h, res;
};

struct AttBwdArgs {
    const float* QKVR; int Np;
    const float* P;                // [B, h, nf, nf]
    const float* Xf;               // [B*nf, dh] X_{l+1} (relu mask; the last layer: g_watt input)
    const float* dX; int lddx;     // [B*nf, lddx] gradient of X_{l+1}; nullptr on the last layer
    const float* dlogit;           // [B] (last layer)
    const float* watt;             // [nf*dh] (last layer)
    __nv_bfloat16* dQKVR;          // [B*nf, Np]
    float* gpart;                  // [ceil(B / 128), nf*dh] partial sums of g_watt (last layer)
    int B, nf, d, h, res;
    int main_ctas;                 // set by the launcher
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, s));
    return v;
}

__global__ void __launch_bounds__(ATT_THREADS) exb_att_gather_kernel(const float* X32, long long xs, int Dp, int D,
                                                                     int nf, __nv_bfloat16* Xb, int Kp, int B) {
    exb::pdl_trigger();
    exb::pdl_wait();
    const size_t n = (size_t)B * nf * Kp;
    for (size_t e = (size_t)blockIdx.x * ATT_THREADS + threadIdx.x; e < n; e += (size_t)gridDim.x * ATT_THREADS) {
        const size_t r = e / Kp;
        const int c = (int)(e % Kp);
        const size_t b = r / nf;
        const int i = (int)(r % nf);
        Xb[e] = __float2bfloat16_rn(c < D ? X32[b * xs + (size_t)i * Dp + c] : 0.f);
    }
}

__global__ void __launch_bounds__(ATT_THREADS) exb_att_fwd_kernel(AttFwdArgs a) {
    extern __shared__ float sm[];
    __shared__ float red[ATT_WARPS];
    exb::pdl_trigger();
    exb::pdl_wait();
    const int b = blockIdx.x, nf = a.nf, d = a.d, h = a.h, dh = d * h;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* sQ = sm;
    float* sK = sQ + nf * dh;
    float* sV = sK + nf * dh;
    float* prow = sV + nf * dh + warp * ATT_MAX_NF;
    const size_t r0 = (size_t)b * nf;
    for (int e = threadIdx.x; e < nf * dh; e += ATT_THREADS) {
        const int i = e / dh, c = e % dh;
        const float* q = a.QKVR + (r0 + i) * a.Np;
        sQ[e] = q[c];
        sK[e] = q[dh + c];
        sV[e] = q[2 * dh + c];
    }
    __syncthreads();
    float acc = 0.f;                                   // this thread's share of flatten(X_L) . w_att
    for (int t = warp; t < h * nf; t += ATT_WARPS) {
        const int eta = t / nf, i = t % nf;
        const float* q = sQ + i * dh + eta * d;
        float s[2], p[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int j = lane + 32 * u;
            s[u] = -INFINITY;
            if (j < nf) {
                const float* k = sK + j * dh + eta * d;
                float v = 0.f;
                for (int kk = 0; kk < d; ++kk) v = fmaf(q[kk], k[kk], v);
                s[u] = v;
            }
        }
        const float m = warp_max(fmaxf(s[0], s[1]));
        float e[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) e[u] = lane + 32 * u < nf ? expf(s[u] - m) : 0.f;
        const float sum = warp_sum(e[0] + e[1]);
        float* Pg = a.P + (((size_t)b * h + eta) * nf + i) * nf;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int j = lane + 32 * u;
            p[u] = e[u] / sum;
            if (j < nf) {
                Pg[j] = p[u];
                prow[j] = p[u];
            }
        }
        __syncwarp();
        const size_t r = r0 + i;
        for (int kk = lane; kk < d; kk += 32) {
            const int c = eta * d + kk;
            float o = 0.f;
            for (int j = 0; j < nf; ++j) o = fmaf(prow[j], sV[j * dh + c], o);
            if (a.res) o = __fadd_rn(o, a.QKVR[r * a.Np + 3 * dh + c]);
            o = o > 0.f ? o : 0.f;
            a.Xf[r * dh + c] = o;
            if (a.Xb) a.Xb[r * a.ldxb + c] = __float2bfloat16_rn(o);
            if (a.base) acc = fmaf(o, a.watt[i * dh + c], acc);
        }
        __syncwarp();
    }
    if (a.Xb) {
        const int pad = a.ldxb - dh;
        for (int e = threadIdx.x; e < nf * pad; e += ATT_THREADS)
            a.Xb[(r0 + e / pad) * a.ldxb + dh + e % pad] = __float2bfloat16_rn(0.f);
    }
    if (a.base) {
        acc = warp_sum(acc);
        if (lane == 0) red[warp] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int w = 0; w < ATT_WARPS; ++w) s += red[w];
            a.base[b] += s;
        }
    }
}

__global__ void __launch_bounds__(ATT_THREADS) exb_att_bwd_kernel(AttBwdArgs a) {
    extern __shared__ float sm[];
    exb::pdl_trigger();
    exb::pdl_wait();
    const int nf = a.nf, d = a.d, h = a.h, dh = d * h;
    if ((int)blockIdx.x >= a.main_ctas) {             // partial g_watt: ATT_THREADS columns x GW_ROWS samples per CTA
        const int T = nf * dh, ncb = (T + ATT_THREADS - 1) / ATT_THREADS;
        const int e = (int)blockIdx.x - a.main_ctas;
        const int t = (e % ncb) * ATT_THREADS + (int)threadIdx.x, chunk = e / ncb;
        if (t >= T) return;
        const int b0 = chunk * GW_ROWS, b1 = min(b0 + GW_ROWS, a.B);
        float s = 0.f;
        for (int b = b0; b < b1; ++b) s = fmaf(a.dlogit[b], a.Xf[(size_t)b * T + t], s);
        a.gpart[(size_t)chunk * T + t] = s;
        return;
    }
    const int b = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* sQ = sm;
    float* sK = sQ + nf * dh;
    float* sV = sK + nf * dh;
    float* sdO = sV + nf * dh;
    float* sP = sdO + nf * dh;
    float* sdS = sP + nf * nf;
    const size_t r0 = (size_t)b * nf;
    const int nblk = a.res ? 4 : 3;
    for (int e = threadIdx.x; e < nf * dh; e += ATT_THREADS) {
        const int i = e / dh, c = e % dh;
        const size_t r = r0 + i;
        const float* q = a.QKVR + r * a.Np;
        sQ[e] = q[c];
        sK[e] = q[dh + c];
        sV[e] = q[2 * dh + c];
        const float g = a.dX ? a.dX[r * a.lddx + c] : __fmul_rn(a.dlogit[b], a.watt[i * dh + c]);
        const float dy = a.Xf[r * dh + c] > 0.f ? g : 0.f;
        sdO[e] = dy;
        if (a.res) a.dQKVR[r * a.Np + 3 * dh + c] = __float2bfloat16_rn(dy);
    }
    const int pad = a.Np - nblk * dh;
    for (int e = threadIdx.x; e < nf * pad; e += ATT_THREADS)
        a.dQKVR[(r0 + e / pad) * a.Np + nblk * dh + e % pad] = __float2bfloat16_rn(0.f);
    for (int eta = 0; eta < h; ++eta) {
        const float* Pg = a.P + ((size_t)b * h + eta) * nf * nf;
        for (int e = threadIdx.x; e < nf * nf; e += ATT_THREADS) sP[e] = Pg[e];
        __syncthreads();                               // sP, and (first head) sQ / sK / sV / sdO
        for (int i = warp; i < nf; i += ATT_WARPS) {
            const float* go = sdO + i * dh + eta * d;
            float dp[2], p[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int j = lane + 32 * u;
                dp[u] = 0.f;
                p[u] = 0.f;
                if (j < nf) {
                    const float* v = sV + j * dh + eta * d;
                    float s = 0.f;
                    for (int kk = 0; kk < d; ++kk) s = fmaf(go[kk], v[kk], s);
                    dp[u] = s;
                    p[u] = sP[i * nf + j];
                }
            }
            const float t = warp_sum(fmaf(dp[0], p[0], dp[1] * p[1]));
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int j = lane + 32 * u;
                if (j < nf) sdS[i * nf + j] = p[u] * (dp[u] - t);
            }
        }
        __syncthreads();
        for (int e = threadIdx.x; e < nf * d; e += ATT_THREADS) {
            const int i = e / d, c = eta * d + e % d;
            float dq = 0.f, dk = 0.f, dv = 0.f;
            for (int j = 0; j < nf; ++j) {
                dq = fmaf(sdS[i * nf + j], sK[j * dh + c], dq);
                dk = fmaf(sdS[j * nf + i], sQ[j * dh + c], dk);
                dv = fmaf(sP[j * nf + i], sdO[j * dh + c], dv);
            }
            __nv_bfloat16* o = a.dQKVR + (r0 + i) * a.Np;
            o[c] = __float2bfloat16_rn(dq);
            o[dh + c] = __float2bfloat16_rn(dk);
            o[2 * dh + c] = __float2bfloat16_rn(dv);
        }
        __syncthreads();                               // before the next head overwrites sP / sdS
    }
}

__global__ void __launch_bounds__(ATT_THREADS) exb_att_fold_kernel(float* G32, long long xs, int Dp, int D, int nf,
                                                                   const float* dX0, int Kp, int B, const float* gpart,
                                                                   int nchunks, float* g_watt, int T, int main_ctas) {
    exb::pdl_trigger();
    exb::pdl_wait();
    if ((int)blockIdx.x >= main_ctas) {                // g_watt += partial sums, in chunk order
        const int t = ((int)blockIdx.x - main_ctas) * ATT_THREADS + (int)threadIdx.x;
        if (t >= T) return;
        float s = 0.f;
        for (int c = 0; c < nchunks; ++c) s += gpart[(size_t)c * T + t];
        g_watt[t] += s;
        return;
    }
    const size_t n = (size_t)B * nf * D;
    for (size_t e = (size_t)blockIdx.x * ATT_THREADS + threadIdx.x; e < n; e += (size_t)main_ctas * ATT_THREADS) {
        const size_t r = e / D;
        const int c = (int)(e % D);
        float* g = G32 + (r / nf) * xs + (size_t)(r % nf) * Dp + c;
        *g = __fadd_rn(*g, dX0[r * Kp + c]);
    }
}

int grid_elems(size_t n) {
    const size_t g = (n + ATT_THREADS - 1) / ATT_THREADS;
    return g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : (int)g);
}

bool check_dims(int B, int nf, int d, int h, int Np, int res, const char* who) {
    const int dh = d * h;
    if (B < 0 || nf < 1 || nf > ATT_MAX_NF || d < 1 || h < 1 || dh > ATT_MAX_DH || Np < (res ? 4 : 3) * dh) {
        g_att_err = std::string(who) + ": needs 1 <= nf <= 64, 1 <= d * h <= 64, Np >= (3 + res) * d * h";
        return false;
    }
    return true;
}

// dynamic shared memory above 48 KB has to be allowed once per kernel
cudaError_t allow_smem(const void* kernel, size_t bytes, int& allowed) {
    if ((int)bytes <= allowed) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) allowed = (int)bytes;
    return e;
}

int fail(cudaError_t e) {
    if (e == cudaSuccess) return 0;
    g_att_err = cudaGetErrorString(e);
    return -1;
}

}  // namespace

extern "C" {

const char* exb_att_last_error() { return g_att_err.c_str(); }
int exb_att_fwd_args_size() { return (int)sizeof(AttFwdArgs); }
int exb_att_bwd_args_size() { return (int)sizeof(AttBwdArgs); }

int exb_att_gather(uint64_t X32, long long xs, int Dp, int D, int nf, uint64_t Xb, int Kp, int B, uint64_t stream) {
    if (!X32 || !Xb || D < 1 || D > Dp || Kp < D || Kp % 64 || nf < 1 || xs < (long long)nf * Dp || B < 0) {
        g_att_err = "att_gather: needs X32 rows of nf*Dp >= nf*D columns and Kp >= D, Kp % 64 == 0";
        return -1;
    }
    return fail(exb::launch_pdl(exb_att_gather_kernel, dim3(grid_elems((size_t)B * nf * Kp)), dim3(ATT_THREADS), 0,
                                (cudaStream_t)stream, (const float*)X32, xs, Dp, D, nf, (__nv_bfloat16*)Xb, Kp, B));
}

int exb_att_fwd(const void* args, uint64_t stream) {
    const AttFwdArgs a = *reinterpret_cast<const AttFwdArgs*>(args);
    if (!check_dims(a.B, a.nf, a.d, a.h, a.Np, a.res, "att_fwd")) return -1;
    if (!a.QKVR || !a.P || !a.Xf || (a.Xb && a.ldxb < a.d * a.h) || (a.base && !a.watt)) {
        g_att_err = "att_fwd: QKVR, P, X_{l+1} (and on the last layer w_att) are required";
        return -1;
    }
    static int allowed = 48 * 1024;
    const size_t smem = sizeof(float) * (3 * a.nf * a.d * a.h + ATT_WARPS * ATT_MAX_NF);
    if (fail(allow_smem((const void*)exb_att_fwd_kernel, smem, allowed))) return -1;
    return fail(exb::launch_pdl(exb_att_fwd_kernel, dim3(a.B > 0 ? a.B : 1), dim3(ATT_THREADS), smem,
                                (cudaStream_t)stream, a));
}

int exb_att_bwd(const void* args, uint64_t stream) {
    AttBwdArgs a = *reinterpret_cast<const AttBwdArgs*>(args);
    if (!check_dims(a.B, a.nf, a.d, a.h, a.Np, a.res, "att_bwd")) return -1;
    const bool top = a.dX == nullptr;
    if (!a.QKVR || !a.P || !a.Xf || !a.dQKVR ||
        (top ? (!a.dlogit || !a.watt || !a.gpart) : a.lddx < a.d * a.h)) {
        g_att_err = "att_bwd: QKVR, P, X_{l+1}, dQKVR and either dX_{l+1} or (last layer) dlogit, w_att, g_watt parts";
        return -1;
    }
    static int allowed = 48 * 1024;
    const int dh = a.d * a.h;
    const size_t smem = sizeof(float) * (4 * a.nf * dh + 2 * a.nf * a.nf);
    if (fail(allow_smem((const void*)exb_att_bwd_kernel, smem, allowed))) return -1;
    a.main_ctas = a.B;
    const int T = a.nf * dh;
    const int extra = top ? ((T + ATT_THREADS - 1) / ATT_THREADS) * ((a.B + GW_ROWS - 1) / GW_ROWS) : 0;
    if (a.main_ctas + extra < 1) return 0;
    return fail(exb::launch_pdl(exb_att_bwd_kernel, dim3(a.main_ctas + extra), dim3(ATT_THREADS), smem,
                                (cudaStream_t)stream, a));
}

int exb_att_fold(uint64_t G32, long long xs, int Dp, int D, int nf, uint64_t dX0, int Kp, int B, uint64_t gpart,
                 int T, uint64_t g_watt, uint64_t stream) {
    if (!G32 || !dX0 || !gpart || !g_watt || D < 1 || D > Dp || Kp < D || nf < 1 || xs < (long long)nf * Dp ||
        T < 1 || B < 0) {
        g_att_err = "att_fold: needs G32 rows of nf*Dp >= nf*D columns, dX_0 rows of Kp >= D, and the g_watt parts";
        return -1;
    }
    const int main_ctas = grid_elems((size_t)B * nf * D);
    const int nchunks = (B + GW_ROWS - 1) / GW_ROWS;
    return fail(exb::launch_pdl(exb_att_fold_kernel, dim3(main_ctas + (T + ATT_THREADS - 1) / ATT_THREADS),
                                dim3(ATT_THREADS), 0, (cudaStream_t)stream, (float*)G32, xs, Dp, D, nf,
                                (const float*)dX0, Kp, B, (const float*)gpart, nchunks, (float*)g_watt, T, main_ctas));
}

}  // extern "C"
