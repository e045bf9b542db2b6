"""Streaming binary-classification metrics on the GPU: AUC (Keras ``tf.keras.metrics.AUC``) and log loss.

``BinaryMetrics`` owns device counters that one kernel launch per batch accumulates into
(csrc/cuda/metric_kernels.cu): per threshold bucket the positives and negatives, an fp64 sum of the per-sample
log loss and the sample count. ``result()`` finalises on the host in fp64 with the formulas of Keras' AUC
(ROC curve, interpolation summation). The host half (``keras_thresholds``, ``confusion``, ``auc_from_counts``)
needs no GPU.

Reference: the examples and the benchmark of the reference compile their models with ``metrics=['AUC']``.
"""
import ctypes

import numpy as np
import torch

MAX_THRESHOLDS = 8192          # csrc/cuda/metric_kernels.cu: MET_MAX_T


def keras_thresholds(num_thresholds=200):
    """The float32 threshold table of ``tf.keras.metrics.AUC(num_thresholds=T)``: -1e-7, i / (T - 1) for
    1 <= i <= T - 2 (divided in double, then cast), 1 + 1e-7."""
    T = _check_thresholds(num_thresholds)
    inner = [(i + 1) * 1.0 / (T - 1) for i in range(T - 2)]
    return np.array([0.0 - 1e-7] + inner + [1.0 + 1e-7], dtype=np.float64).astype(np.float32)


def _check_thresholds(num_thresholds):
    if isinstance(num_thresholds, bool) or int(num_thresholds) != num_thresholds:
        raise ValueError("num_thresholds must be an integer (got %r)" % (num_thresholds,))
    T = int(num_thresholds)
    if T < 2 or T > MAX_THRESHOLDS:
        raise ValueError("num_thresholds must be in [2, %d] (got %d)" % (MAX_THRESHOLDS, T))
    return T


def confusion(pos, neg):
    """tp, fp, tn, fn (int64 [T]) at every threshold from the bucket counts pos, neg (int [T + 1]; bucket k holds
    the samples above exactly k thresholds)."""
    pos, neg = np.asarray(pos, dtype=np.int64), np.asarray(neg, dtype=np.int64)
    assert pos.shape == neg.shape and pos.ndim == 1 and pos.size >= 3, (pos.shape, neg.shape)
    T = pos.size - 1
    # predicted positive at threshold i <=> bucket > i: suffix sums over buckets i + 1 .. T
    tp = np.cumsum(pos[::-1])[::-1][1:]
    fp = np.cumsum(neg[::-1])[::-1][1:]
    assert tp.size == T
    return tp, fp, int(neg.sum()) - fp, int(pos.sum()) - tp


def _div_no_nan(a, b):
    out = np.zeros_like(a, dtype=np.float64)
    np.divide(a, b, out=out, where=b != 0)
    return out


def auc_from_counts(pos, neg):
    """Keras' ROC AUC with interpolation summation from bucket counts, in fp64: tpr = tp / (tp + fn),
    fpr = fp / (fp + tn) (0 where the denominator is 0), auc = sum_i (fpr_i - fpr_{i+1}) (tpr_i + tpr_{i+1}) / 2."""
    tp, fp, tn, fn = (x.astype(np.float64) for x in confusion(pos, neg))
    tpr = _div_no_nan(tp, tp + fn)
    fpr = _div_no_nan(fp, fp + tn)
    return float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2.0))


def _lib():
    from .. import _native
    lib = _native.cuda()
    if lib.exb_binary_metrics_update.argtypes is None:
        u64 = ctypes.c_uint64
        lib.exb_binary_metrics_update.restype = ctypes.c_int
        lib.exb_binary_metrics_update.argtypes = [u64, u64, u64, ctypes.c_int, u64, ctypes.c_int, u64, u64, u64, u64]
        lib.exb_metric_last_error.restype = ctypes.c_char_p
        assert lib.exb_metric_max_thresholds() == MAX_THRESHOLDS, "metric_kernels.cu: MET_MAX_T mismatch"
    return lib


class BinaryMetrics:
    """AUC (Keras ``AUC(num_thresholds)``: ROC, interpolation) and mean log loss over every batch passed to
    ``update`` since the last ``reset``.

    ``update(logits, labels, n=None)``: one kernel launch, no host synchronisation. ``n`` is an int (the first n
    rows count) or an int32 CUDA tensor of one element read on the device, so a captured CUDA graph serves every
    batch size up to ``logits.numel()``. ``result()`` returns ``{"auc", "logloss", "count", "positives"}``; with
    several ranks it is collective and all-reduces the counters over the context's process group once."""

    def __init__(self, num_thresholds=200, device=None):
        self.num_thresholds = T = _check_thresholds(num_thresholds)
        if device is None:
            from ..context import get_context
            device = get_context().device
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("BinaryMetrics accumulates on a CUDA device (got %s)" % self.device)
        self.lib = _lib()
        self.thresholds = torch.from_numpy(keras_thresholds(T)).to(self.device)
        self.hist = torch.zeros(2, T + 1, dtype=torch.int64, device=self.device)    # positives, negatives per bucket
        self.loss_sum = torch.zeros(1, dtype=torch.float64, device=self.device)
        self.count = torch.zeros(1, dtype=torch.int64, device=self.device)

    def reset(self):
        self.hist.zero_()
        self.loss_sum.zero_()
        self.count.zero_()

    def update(self, logits, labels, n=None):
        """accumulate the first n rows of logits / labels (any float dtype, CUDA, one value per sample)"""
        logits = logits.detach().reshape(-1)
        labels = labels.detach().reshape(-1)
        if not (logits.is_cuda and labels.is_cuda):
            raise ValueError("BinaryMetrics.update takes CUDA tensors")
        logits = logits.to(device=self.device, dtype=torch.float32).contiguous()
        labels = labels.to(device=self.device, dtype=torch.float32).contiguous()
        cap, n_ptr = logits.numel(), 0
        if isinstance(n, torch.Tensor):
            if not (n.is_cuda and n.dtype == torch.int32 and n.numel() == 1):
                raise ValueError("a device row count is an int32 CUDA tensor of one element")
            n_ptr = n.data_ptr()
        elif n is not None:
            if not 0 <= int(n) <= cap:
                raise ValueError("n = %d rows of %d" % (int(n), cap))
            cap = int(n)
        if labels.numel() < cap:
            raise ValueError("%d labels for %d logits" % (labels.numel(), cap))
        st = torch.cuda.current_stream(self.device).cuda_stream
        rc = self.lib.exb_binary_metrics_update(logits.data_ptr(), labels.data_ptr(), n_ptr, cap,
                                                self.thresholds.data_ptr(), self.num_thresholds, self.hist.data_ptr(),
                                                self.loss_sum.data_ptr(), self.count.data_ptr(), st)
        if rc != 0:
            raise RuntimeError("binary_metrics_update: " + self.lib.exb_metric_last_error().decode())

    def counts(self):
        """(positives, negatives, loss sum, count) summed over the ranks; collective when world > 1"""
        from ..context import get_context
        ints = torch.cat([self.hist.reshape(-1), self.count])
        loss = self.loss_sum.clone()
        ctx = get_context()
        if ctx.world > 1:
            import torch.distributed as dist
            dist.all_reduce(ints, group=ctx.group)
            dist.all_reduce(loss, group=ctx.group)
        ints = ints.cpu().numpy()
        T1 = self.num_thresholds + 1
        return ints[:T1], ints[T1:2 * T1], float(loss.item()), int(ints[-1])

    def result(self):
        pos, neg, loss, count = self.counts()
        return {"auc": auc_from_counts(pos, neg), "logloss": loss / count if count else 0.0, "count": count,
                "positives": int(pos.sum())}
