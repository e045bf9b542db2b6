// metric_kernels.cu -- streaming binary-classification metrics on the device (models/metrics.py: BinaryMetrics).
//
//   exb_binary_metrics_kernel  one launch per batch: logits + labels in, counters in device memory accumulated.
//     AUC: the confusion counts of Keras' tf.keras.metrics.AUC(num_thresholds=T). With the float32 threshold table
//          t_0 = -1e-7 < t_1 < ... < t_{T-1} = 1 + 1e-7, a sample with probability p is predicted positive at t_i iff
//          p > t_i, so its whole contribution is its bucket k = #{i : t_i < p} in [0, T] (found by binary search:
//          exact at ties, unlike ceil(p (T-1))). Per bucket, positives (label != 0, Keras casts labels to bool) and
//          negatives are counted; the host turns the suffix sums into tp / fp / tn / fn at every threshold.
//     log loss: sum of max(z, 0) - z y + log1p(exp(-|z|)) (the training head's formula) in an fp64 counter, plus
//          the number of samples.
//   p = 1 / (1 + exp(-z)) is the expression of the predict head (dense_kernels.cu), so the buckets agree with the
//   probabilities it returns. Each CTA counts into a private shared-memory histogram and flushes its non-zero bins
//   to the 64-bit global counters. The number of valid rows n is read from device memory (clamped to the capacity
//   the grid was sized for): one captured graph serves every batch size up to that capacity.
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "pdl.cuh"

namespace {

std::string g_metric_err;

constexpr int MET_THREADS = 256;
constexpr int MET_MAX_T = 8192;        // 2 (T + 1) 32-bit bins = 64 KiB of shared memory per CTA

__global__ void __launch_bounds__(MET_THREADS) exb_binary_metrics_kernel(
        const float* __restrict__ logits, const float* __restrict__ labels, const int* __restrict__ n_dev, int cap,
        const float* __restrict__ thr, int T, unsigned long long* hist, double* loss_sum, unsigned long long* count) {
    extern __shared__ unsigned s_hist[];     // [positives: T + 1 | negatives: T + 1]
    __shared__ double s_loss[MET_THREADS / 32];
    exb::pdl_trigger();
    const int nb = T + 1;
    for (int i = threadIdx.x; i < 2 * nb; i += blockDim.x) s_hist[i] = 0u;
    exb::pdl_wait();
    __syncthreads();
    int n = cap;
    if (n_dev) n = min(max(*n_dev, 0), cap);
    double ls = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float z = logits[i], y = labels[i];
        const float p = 1.f / (1.f + expf(-z));
        int lo = 0, hi = T;                  // lower bound of p in the ascending table = #{i : t_i < p} (NaN: 0)
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(thr + mid) < p) lo = mid + 1; else hi = mid;
        }
        atomicAdd(&s_hist[(y != 0.f ? 0 : nb) + lo], 1u);
        ls += (double)(fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z))));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) ls += __shfl_xor_sync(0xffffffffu, ls, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) s_loss[warp] = ls;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < MET_THREADS / 32; ++w) t += s_loss[w];
        if (n > 0) atomicAdd(loss_sum, t);
        if (blockIdx.x == 0) atomicAdd(count, (unsigned long long)n);
    }
    for (int i = threadIdx.x; i < 2 * nb; i += blockDim.x) {
        const unsigned c = s_hist[i];
        if (c) atomicAdd(hist + i, (unsigned long long)c);
    }
}

}  // namespace

extern "C" {

const char* exb_metric_last_error() { return g_metric_err.c_str(); }
int exb_metric_max_thresholds() { return MET_MAX_T; }

// logits, labels: fp32 [>= cap]; n_dev: int32 on the device (0: all cap rows); thr: fp32 [T] ascending;
// hist: int64 [2, T + 1] (positives, negatives per bucket); loss_sum: fp64 [1]; count: int64 [1]
int exb_binary_metrics_update(uint64_t logits, uint64_t labels, uint64_t n_dev, int cap, uint64_t thr, int T,
                              uint64_t hist, uint64_t loss_sum, uint64_t count, uint64_t stream) {
    if (T < 2 || T > MET_MAX_T) { g_metric_err = "binary_metrics: 2 <= num_thresholds <= 8192"; return -1; }
    if (cap < 0 || (cap > 0 && (!logits || !labels)) || !thr || !hist || !loss_sum || !count) {
        g_metric_err = "binary_metrics: logits, labels, thresholds and the counters are required";
        return -1;
    }
    const size_t smem = (size_t)2 * (T + 1) * sizeof(unsigned);
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(exb_binary_metrics_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             2 * (MET_MAX_T + 1) * (int)sizeof(unsigned));
        attr = true;
    }
    int grid = (cap + 4 * MET_THREADS - 1) / (4 * MET_THREADS);     // about 4 samples per thread
    grid = grid < 1 ? 1 : (grid > 264 ? 264 : grid);
    cudaError_t e = exb::launch_pdl(exb_binary_metrics_kernel, dim3(grid), dim3(MET_THREADS), smem,
                                    (cudaStream_t)stream, (const float*)logits, (const float*)labels,
                                    (const int*)n_dev, cap, (const float*)thr, T, (unsigned long long*)hist,
                                    (double*)loss_sum, (unsigned long long*)count);
    if (e != cudaSuccess) { g_metric_err = cudaGetErrorString(e); return -1; }
    return 0;
}

}  // extern "C"
