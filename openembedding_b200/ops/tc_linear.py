"""``TcLinear`` / ``tc_matmul``: ``torch.nn.Linear`` whose three GEMMs (forward, input gradient, weight gradient) run
on the hand-written wgmma kernel (``csrc/cuda/gemm_wgmma.cu``) instead of cuBLAS.

Used by the eager model zoo (``models/ctr.py``) for everything that is GEMM-shaped and not covered by the fully fused
DeepFM / WDL step: the DNN towers of xDeepFM / DCN-v2, the DCN-v2 cross layers (``x0 * (W x + b) + x``) and the CIN's
1x1 convolutions (a GEMM over the ``H_k x m`` interaction channels, xDeepFM). The reference gets these from
TensorFlow -> cuBLAS / cuDNN (K6 in SURVEY 2.5).

bf16 operands, fp32 accumulation in registers, fp32 master weights / bias / gradients. Operands are padded to the tile
geometry (K to a multiple of 64, the batch to a multiple of 64 for the weight-gradient product, which reads the
batch-major activations as MN-major wgmma operands -- no transposed copies).
"""
import torch
from torch import nn

from . import gemm as G


def _r(x, m):
    return (x + m - 1) // m * m


def _pad_bf16(x, rows, cols):
    """[r, c] float -> zero-padded bf16 [rows, cols]: ONE cast-copy over the data, the pad strips zeroed separately
    (a zeros() + copy pair was two full passes over every operand: ~0.1 ms of a DCN-v2 step)"""
    if x.dtype == torch.bfloat16 and x.shape == (rows, cols) and x.is_contiguous():
        return x
    r, c = x.shape
    out = torch.empty((rows, cols), dtype=torch.bfloat16, device=x.device)
    out[:r, :c] = x
    if c < cols:
        out[:, c:].zero_()
    if r < rows:
        out[r:, :c].zero_()
    return out


class _TcLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        M, K = x.shape
        N = weight.shape[0]
        Mp, Kp, Np = _r(M, 64), _r(K, 64), _r(N, 64)
        xb = _pad_bf16(x, Mp, Kp)
        wb = _pad_bf16(weight, Np, Kp)
        out = torch.empty((Mp, Np), dtype=torch.bfloat16, device=x.device)
        G.gemm_nt(xb, wb, M, N, Kp, out, mode=G.EPI_FWD, relu=False, ones_col=-1)
        ctx.save_for_backward(xb, weight)
        ctx.shape = (M, K, N)
        ctx.has_bias = bias is not None
        # bf16 + fp32 promotes to fp32 in one kernel (no separate .float() pass)
        return out[:M, :N] + bias if bias is not None else out[:M, :N].float()

    @staticmethod
    def backward(ctx, dy):
        xb, weight = ctx.saved_tensors
        M, K, N = ctx.shape
        Mp, Kp, Np = xb.shape[0], xb.shape[1], _r(N, 64)
        dyb = _pad_bf16(dy, Mp, Np)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            wtb = _pad_bf16(weight.t(), Kp, Np)                     # [K, N]: K-major in N for dX = dY W
            dxb = torch.empty((Mp, Kp), dtype=torch.bfloat16, device=dy.device)
            G.gemm_nt(dyb, wtb, M, K, Np, dxb, mode=G.EPI_FWD, relu=False, ones_col=-1)
            dx = dxb[:M, :K].float()
        if ctx.needs_input_grad[1]:
            gw = torch.zeros((Np, Kp), dtype=torch.float32, device=dy.device)
            G.gemm_tn(dyb, xb, N, K, Mp, gw, splits=max(1, min(8, Mp // 512)))    # dW = dY^T X, batch-major operands
            dw = gw[:N, :K]
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum(0)
        return dx, dw, db


def tc_linear(x, weight, bias=None):
    """``x @ weight.T + bias`` on the wgmma GEMM; x may have any leading shape"""
    lead = x.shape[:-1]
    y = _TcLinearFn.apply(x.reshape(-1, x.shape[-1]), weight, bias)
    return y.reshape(lead + (weight.shape[0],))


class TcLinear(nn.Linear):
    """drop-in ``nn.Linear`` (fp32 parameters) computing on the hand-written GEMM when the input is on a CUDA device"""

    def forward(self, x):
        if x.is_cuda and x.numel() > 0:
            return tc_linear(x, self.weight, self.bias)
        return super().forward(x)


class TcConv1x1(nn.Module):
    """``nn.Conv1d(cin, cout, 1)`` as a GEMM over the channel axis (the CIN layer of xDeepFM): [B, cin, D] -> [B, cout, D]"""

    def __init__(self, cin, cout):
        super().__init__()
        self.lin = TcLinear(cin, cout)

    def forward(self, z):
        B, C, D = z.shape
        y = self.lin(z.transpose(1, 2).reshape(B * D, C))
        return y.reshape(B, D, -1).transpose(1, 2)
