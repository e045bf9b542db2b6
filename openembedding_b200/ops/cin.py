"""One Compressed-Interaction-Network layer (xDeepFM) on own kernels: interaction + 1x1 convolution + bias + relu.

``out[r, n] = relu(sum_{h, j} W[n, h*m + j] * hid[r, h] * x[r, j] + bias[n])`` with rows ``r = (batch, embedding column)``.
The interaction tensor is written once, directly as the bf16 K-major operand of the wgmma GEMM
(``csrc/cuda/cin_kernels.cu: exb_cin_outer_kernel``; a constant-one column carries the bias), the GEMM applies the relu
in its epilogue, and the backward folds the GEMM's input gradient back into ``d hid`` / ``d x`` with one warp per row
(``exb_cin_outer_bwd_kernel``). Everything stays in the ``[B*D, channels]`` layout between layers -- no fp32 interaction
tensor, no transposes, no pad copies. The reference runs this layer as DeepCTR's ``tf.einsum`` + ``conv1d`` through
TensorFlow (test/benchmark/criteo_deepctr.py:268-282, K6 in SURVEY 2.5).
"""
import ctypes
from ctypes import c_int, c_longlong, c_uint64

import torch

from .. import _native
from . import gemm as G

_proto_done = False


def _lib():
    global _proto_done
    lib = _native.cuda()
    if not _proto_done:
        lib.exb_cin_outer.restype = c_int
        lib.exb_cin_outer.argtypes = [c_uint64, c_int, c_longlong, c_int, c_uint64, c_longlong, c_int, c_uint64, c_longlong,
                                      c_int, c_int, c_uint64]
        lib.exb_cin_outer_bwd.restype = c_int
        lib.exb_cin_outer_bwd.argtypes = [c_uint64, c_longlong, c_uint64, c_int, c_longlong, c_int, c_uint64, c_longlong, c_int,
                                          c_uint64, c_longlong, c_uint64, c_longlong, c_int, c_uint64]
        lib.exb_cin_last_error.restype = ctypes.c_char_p
        # the fused xDeepFM step (models/fused_dense.py)
        lib.exb_cin_gather.restype = c_int
        lib.exb_cin_gather.argtypes = [c_uint64, c_longlong, c_int, c_int, c_int, c_uint64, c_int, c_uint64]
        lib.exb_cin_pool.restype = c_int
        lib.exb_cin_pool.argtypes = [ctypes.c_void_p, c_uint64]
        lib.exb_cin_pool_args_size.restype = c_int
        lib.exb_cin_dy.restype = c_int
        lib.exb_cin_dy.argtypes = [ctypes.c_void_p, c_uint64]
        lib.exb_cin_dy_args_size.restype = c_int
        lib.exb_cin_fold.restype = c_int
        lib.exb_cin_fold.argtypes = [c_uint64, c_longlong, c_int, c_int, c_int, c_int, ctypes.POINTER(c_uint64), c_int,
                                     c_uint64]
        _proto_done = True
    return lib


def _r(x, m):
    return (x + m - 1) // m * m


def _ck(rc, lib, what):
    if rc != 0:
        raise RuntimeError("%s: %s" % (what, lib.exb_cin_last_error().decode()))


class _CinLayerFn(torch.autograd.Function):
    """hid [R, H] (fp32, or the bf16 output of the previous layer), x [R, m] fp32, weight [N, H*m], bias [N] -> [R, N] fp32"""

    @staticmethod
    def forward(ctx, hid, x, weight, bias, relu):
        lib = _lib()
        R, H = hid.shape
        m = x.shape[1]
        N, C = weight.shape
        assert C == H * m and x.shape[0] == R
        assert hid.stride(-1) == 1 and x.stride(-1) == 1 and x.dtype == torch.float32
        assert hid.dtype in (torch.float32, torch.bfloat16)
        Mp, Kp, Np = _r(R, 128), _r(C + 1, 64), _r(N, 64)
        dev = x.device
        st = torch.cuda.current_stream(dev).cuda_stream
        Z = torch.empty((Mp, Kp), dtype=torch.bfloat16, device=dev)
        if Mp > R:
            Z[R:].zero_()
        _ck(lib.exb_cin_outer(hid.data_ptr(), int(hid.dtype == torch.bfloat16), hid.stride(0), H, x.data_ptr(), x.stride(0), m,
                              Z.data_ptr(), Z.stride(0), Kp, R, st), lib, "cin_outer")
        Wb = torch.zeros((Np, Kp), dtype=torch.bfloat16, device=dev)
        Wb[:N, :C] = weight
        if bias is not None:
            Wb[:N, C] = bias                    # meets the constant-one column of Z
        out = torch.empty((Mp, Np), dtype=torch.bfloat16, device=dev)
        G.gemm_nt(Z, Wb, R, N, Kp, out, mode=G.EPI_FWD, relu=bool(relu), ones_col=-1)
        ctx.save_for_backward(hid, x, Z, Wb, out)
        ctx.dims = (R, H, m, N, C, Mp, Kp, Np, bool(relu), bias is not None)
        return out[:R, :N].float()

    @staticmethod
    def backward(ctx, dy):
        lib = _lib()
        hid, x, Z, Wb, out = ctx.saved_tensors
        R, H, m, N, C, Mp, Kp, Np, relu, has_bias = ctx.dims
        dev = dy.device
        st = torch.cuda.current_stream(dev).cuda_stream
        dyb = torch.empty((Mp, Np), dtype=torch.bfloat16, device=dev)
        dyb[:R, :N] = dy * (out[:R, :N] > 0) if relu else dy
        if N < Np:
            dyb[:, N:].zero_()
        if R < Mp:
            dyb[R:, :N].zero_()
        dhid = dx = dw = db = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            WTb = Wb.t().contiguous()                                   # [Kp, Np]: K-major in N for dZ = dY W
            dZ = torch.empty((Mp, Kp), dtype=torch.bfloat16, device=dev)
            G.gemm_nt(dyb, WTb, R, Kp, Np, dZ, mode=G.EPI_FWD, relu=False, ones_col=-1)
            dhid = torch.empty((R, H), dtype=torch.float32, device=dev)
            dx = torch.empty((R, m), dtype=torch.float32, device=dev)
            _ck(lib.exb_cin_outer_bwd(dZ.data_ptr(), dZ.stride(0), hid.data_ptr(), int(hid.dtype == torch.bfloat16),
                                      hid.stride(0), H, x.data_ptr(), x.stride(0), m, dhid.data_ptr(), dhid.stride(0),
                                      dx.data_ptr(), dx.stride(0), R, st), lib, "cin_outer_bwd")
            if hid.dtype != torch.float32:
                dhid = dhid.to(hid.dtype)
        if ctx.needs_input_grad[2] or (has_bias and ctx.needs_input_grad[3]):
            gw = torch.zeros((Np, Kp), dtype=torch.float32, device=dev)
            G.gemm_tn(dyb, Z, N, Kp, Mp, gw, splits=max(1, min(8, Mp // 512)))     # dW = dY^T Z; column C is d bias
            dw = gw[:N, :C]
            if has_bias:
                db = gw[:N, C]
        return dhid, dx, dw, db, None


def cin_layer(hid, x, weight, bias=None, relu=True):
    """hid [R, H], x [R, m] (rows = batch x embedding column), weight [N, H*m] -> relu(interaction @ weight.T + bias) [R, N]"""
    return _CinLayerFn.apply(hid, x, weight, bias, relu)
