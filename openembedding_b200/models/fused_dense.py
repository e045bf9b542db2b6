"""Fused DeepFM / Wide&Deep / xDeepFM / DCN-v2 / AutoInt training step on hand-written sm_90a kernels only.

Per step and per GPU (10 launches at world 1, captured in one CUDA graph by ``FusedTrainer``):

    pull + plan (peer loads, cp.async)   sparse_v2.cuh / sparse_kernels.cuh   (prefetched in the previous step's tail)
    prep                                 dense_kernels.cu   X32 -> A0 (bf16), FM sums, base logit
    3x GEMM fwd  (wgmma, relu, ones)     gemm_wgmma.cu
    head         (loss, dlogit, dZ_L)    dense_kernels.cu
    backward chain: 3x dX (relu mask / FM-fused fp32 embedding gradient) + 3x dW (MN-major operands, split-K,
                 TMA reduce-add) as ONE persistent kernel (exb_gemm_chain_kernel)
    cachegrad, push_update (P2P dispatch + combine + sparse optimizer; world > 1: the dense-gradient all-reduce
                 rides on its cross-GPU barriers),
    Adagrad / Adam / FTRL (flat) + bf16 weight refresh  ||  pull + plan of the NEXT batch on a side stream

No cuBLAS, no NCCL, no torch op on the step. Biases are folded into the GEMMs through a
constant "ones" column, so a layer is exactly one GEMM in each direction.

Model definition = DeepCTR's DeepFM / WDL / xDeepFM as used by the reference benchmark
(test/benchmark/criteo_deepctr.py:243-282) and the zoo's DCN-v2; see ``models/ctr.py`` for the eager version
of the same architecture (used as the numerical reference in tests).

xDeepFM adds the CIN branch (csrc/cuda/cin_kernels.cu + the wgmma GEMM), 3 + 6 K launches for K layers:
gather + K x (interaction operand, GEMM) + pool after prep; after the dX GEMM, K x (dY, dZ GEMM, row-wise
interaction backward, filter-gradient GEMM) and the fold of the CIN embedding gradient into G32.

DCN-v2 adds the cross network on the A0 layout (csrc/cuda/cross_kernels.cu + the wgmma GEMM), 1 + 5 L launches for
L layers: L x (U_l GEMM, cross forward) before the head; after the dX GEMM, the top of the cross backward and
L x (P_l GEMM, weight-gradient GEMM, cross backward), the last of which folds the embedding gradient into G32.

AutoInt adds stacked multi-head self-attention over the fields (csrc/cuda/autoint_kernels.cu + the wgmma GEMM) on rows
r = (sample, field), 2 + 5 A launches for A layers: gather + A x (projection GEMM, attention forward) before the head;
after the dX GEMM, A x (attention backward, weight-gradient GEMM, input-gradient GEMM) and the fold of the embedding
gradient (and of the partial sums of the output weight's gradient) into G32 / gtheta.

Evaluation (``predict_forward``; ``FusedTrainer.predict`` / ``evaluate``) runs the forward half alone: stateless pull,
prep, the forward GEMMs, the CIN / cross forward and the predict head (logits + probabilities, dense_kernels.cu).
"""
import ctypes
import os
import math
import shutil
from ctypes import c_float, c_int, c_longlong, c_void_p

import torch

from .. import _native
from ..context import get_context
from ..ops import gemm as G
from ..utils import timers as _timers


class _PrepArgs(ctypes.Structure):
    _fields_ = [("X32", c_void_p), ("xs", c_longlong), ("A0", c_void_p), ("A0T", c_void_p), ("ids", c_void_p),
                ("ncols", c_int), ("dense", c_void_p), ("nd", c_int), ("cache_emb", c_void_p),
                ("cache_lin", c_void_p), ("cache_col", c_void_p), ("cache_off", c_void_p), ("nc", c_int),
                ("wd", c_void_p), ("bias", c_void_p), ("S", c_void_p), ("base", c_void_p), ("B", c_int),
                ("K0p", c_int), ("Dp", c_int), ("nf", c_int), ("ns", c_int), ("lin0", c_int), ("use_fm", c_int),
                ("loss", c_void_p), ("opt_step", c_void_p)]


class _HeadArgs(ctypes.Structure):
    _fields_ = [("H", c_void_p), ("Hp", c_int), ("ones_col", c_int), ("wout", c_void_p), ("base", c_void_p),
                ("labels", c_void_p), ("dlogit", c_void_p), ("loss", c_void_p), ("dZ", c_void_p), ("dZT", c_void_p),
                ("g_wout", c_void_p), ("g_wd", c_void_p), ("g_bias", c_void_p), ("dense", c_void_p), ("nd", c_int),
                ("G32", c_void_p), ("xs", c_longlong), ("lin0", c_int), ("ns", c_int), ("ids", c_void_p),
                ("ncols", c_int), ("cache_col", c_void_p), ("cache_off", c_void_p), ("nc", c_int),
                ("g_cache_lin", c_void_p), ("B", c_int), ("grad_scale", c_float)]


class _PredictArgs(ctypes.Structure):
    _fields_ = [("H", c_void_p), ("Hp", c_int), ("wout", c_void_p), ("base", c_void_p), ("logits", c_void_p),
                ("probs", c_void_p), ("B", c_int)]


_OPT_MAX_MATS = 8          # csrc/cuda/dense_kernels.cu: EXB_OPT_MAX_MATS (DNN layers + CIN layers)


class _OptMat(ctypes.Structure):
    _fields_ = [("off", c_longlong), ("R", c_int), ("C", c_int), ("Wb", c_void_p), ("WTb", c_void_p)]


class _DenseOptArgs(ctypes.Structure):
    _fields_ = [("theta", c_void_p), ("accum", c_void_p), ("grad", c_void_p), ("n", c_longlong), ("flat_lo", c_longlong),
                ("lr", c_float), ("eps", c_float), ("nmat", c_int), ("zero_grad", c_int),
                ("mat", _OptMat * _OPT_MAX_MATS),
                ("kind", c_int), ("_pad", c_int), ("accum2", c_void_p), ("step", c_void_p), ("b1", c_float), ("b2", c_float),
                ("l1", c_float), ("l2", c_float), ("l2s", c_float), ("lrp", c_float), ("beta", c_float),
                ("c1", c_float), ("c2", c_float)]


_CIN_MAX_LAYERS = 8        # csrc/cuda/cin_kernels.cu: CIN_MAX_LAYERS


class _CinPoolArgs(ctypes.Structure):
    _fields_ = [("Y", c_void_p * _CIN_MAX_LAYERS), ("ldy", c_longlong * _CIN_MAX_LAYERS),
                ("lo", c_int * _CIN_MAX_LAYERS), ("hi", c_int * _CIN_MAX_LAYERS), ("K", c_int), ("T", c_int),
                ("D", c_int), ("B", c_int), ("wcin", c_void_p), ("p", c_void_p), ("base", c_void_p)]


class _CinDyArgs(ctypes.Structure):
    _fields_ = [("Y", c_void_p), ("ldy", c_longlong), ("N", c_int), ("Np", c_int), ("dir_lo", c_int), ("t0", c_int),
                ("wcin", c_void_p), ("dhid", c_void_p), ("ld_dhid", c_longlong), ("Hn", c_int), ("D", c_int),
                ("R", c_int), ("dlogit", c_void_p), ("dY", c_void_p), ("lddy", c_longlong), ("p", c_void_p),
                ("g_wcin", c_void_p), ("T", c_int), ("B", c_int), ("main_ctas", c_int)]


class _CrossX0(ctypes.Structure):
    _fields_ = [("X32", c_void_p), ("xs", c_longlong), ("dense", c_void_p), ("nd", c_int), ("E", c_int), ("Dp", c_int),
                ("D", c_int), ("K0p", c_int), ("B", c_int)]


class _CrossFwdArgs(ctypes.Structure):
    _fields_ = [("x", _CrossX0), ("U", c_void_p), ("Xin", c_void_p), ("Xf", c_void_p), ("Xb", c_void_p),
                ("wcross", c_void_p), ("base", c_void_p)]


class _CrossBwdArgs(ctypes.Structure):
    _fields_ = [("x", _CrossX0), ("dlogit", c_void_p), ("wcross", c_void_p), ("gin", c_void_p), ("P", c_void_p),
                ("gout", c_void_p), ("U", c_void_p), ("dU", c_void_p), ("gx0", c_void_p), ("G32", c_void_p),
                ("XfL", c_void_p), ("g_wcross", c_void_p), ("main_ctas", c_int)]


class _AttFwdArgs(ctypes.Structure):
    _fields_ = [("QKVR", c_void_p), ("Np", c_int), ("P", c_void_p), ("Xf", c_void_p), ("Xb", c_void_p), ("ldxb", c_int),
                ("watt", c_void_p), ("base", c_void_p), ("B", c_int), ("nf", c_int), ("d", c_int), ("h", c_int),
                ("res", c_int)]


class _AttBwdArgs(ctypes.Structure):
    _fields_ = [("QKVR", c_void_p), ("Np", c_int), ("P", c_void_p), ("Xf", c_void_p), ("dX", c_void_p), ("lddx", c_int),
                ("dlogit", c_void_p), ("watt", c_void_p), ("dQKVR", c_void_p), ("gpart", c_void_p), ("B", c_int),
                ("nf", c_int), ("d", c_int), ("h", c_int), ("res", c_int), ("main_ctas", c_int)]


def _r(x, m):
    return (x + m - 1) // m * m


_proto = False


def _lib():
    global _proto
    lib = _native.cuda()
    if not _proto:
        u64 = ctypes.c_uint64
        lib.exb_prep.restype = c_int
        lib.exb_prep.argtypes = [c_void_p, c_int, c_int, u64]
        lib.exb_head.restype = c_int
        lib.exb_head.argtypes = [c_void_p, c_int, u64]
        lib.exb_prep_args_size.restype = c_int
        lib.exb_head_args_size.restype = c_int
        lib.exb_predict_head.restype = c_int
        lib.exb_predict_head.argtypes = [c_void_p, u64]
        assert lib.exb_predict_args_size() == ctypes.sizeof(_PredictArgs), "PredictArgs ABI mismatch"
        lib.exb_cachegrad.restype = c_int
        lib.exb_cachegrad.argtypes = [u64, c_longlong, c_int, c_int, u64, c_int, u64, u64, c_int, u64, c_int, u64, u64, u64,
                                      u64]
        lib.exb_adagrad_flat.restype = c_int
        lib.exb_adagrad_flat.argtypes = [u64, u64, u64, c_longlong, c_float, c_float, u64]
        lib.exb_refresh_bf16.restype = c_int
        lib.exb_refresh_bf16.argtypes = [u64, u64, u64, c_int, c_int, u64]
        lib.exb_allreduce_adagrad.restype = c_int
        lib.exb_allreduce_adagrad.argtypes = [ctypes.POINTER(u64), ctypes.POINTER(u64), u64, u64, u64, c_longlong, c_int,
                                              c_int, c_int, c_void_p, u64]
        lib.exb_dense_opt.restype = c_int
        lib.exb_dense_opt.argtypes = [c_void_p, u64]
        assert lib.exb_dense_opt_args_size() == ctypes.sizeof(_DenseOptArgs), "DenseOptArgs ABI mismatch"
        lib.exb_dense_last_error.restype = ctypes.c_char_p
        assert lib.exb_prep_args_size() == ctypes.sizeof(_PrepArgs), "PrepArgs ABI mismatch"
        assert lib.exb_head_args_size() == ctypes.sizeof(_HeadArgs), "HeadArgs ABI mismatch"
        _proto = True
    return lib


def _ck(rc, what):
    if rc != 0:
        raise RuntimeError("%s: %s" % (what, _lib().exb_dense_last_error().decode()))


def _cin_lib():
    from ..ops import cin as C
    lib = C._lib()
    assert lib.exb_cin_pool_args_size() == ctypes.sizeof(_CinPoolArgs), "CinPoolArgs ABI mismatch"
    assert lib.exb_cin_dy_args_size() == ctypes.sizeof(_CinDyArgs), "CinDyArgs ABI mismatch"
    return lib


def _cin_ck(rc, what):
    if rc != 0:
        raise RuntimeError("%s: %s" % (what, _cin_lib().exb_cin_last_error().decode()))


_cross_proto = False


def _cross_lib():
    global _cross_proto
    lib = _native.cuda()
    if not _cross_proto:
        for fn in (lib.exb_cross_fwd, lib.exb_cross_bwd_top, lib.exb_cross_bwd):
            fn.restype = c_int
            fn.argtypes = [c_void_p, ctypes.c_uint64]
        lib.exb_cross_last_error.restype = ctypes.c_char_p
        assert lib.exb_cross_fwd_args_size() == ctypes.sizeof(_CrossFwdArgs), "CrossFwdArgs ABI mismatch"
        assert lib.exb_cross_bwd_args_size() == ctypes.sizeof(_CrossBwdArgs), "CrossBwdArgs ABI mismatch"
        _cross_proto = True
    return lib


def _cross_ck(rc, what):
    if rc != 0:
        raise RuntimeError("%s: %s" % (what, _cross_lib().exb_cross_last_error().decode()))


_att_proto = False


def _att_lib():
    global _att_proto
    lib = _native.cuda()
    if not _att_proto:
        u64 = ctypes.c_uint64
        for fn in (lib.exb_att_fwd, lib.exb_att_bwd):
            fn.restype = c_int
            fn.argtypes = [c_void_p, u64]
        lib.exb_att_gather.restype = c_int
        lib.exb_att_gather.argtypes = [u64, c_longlong, c_int, c_int, c_int, u64, c_int, c_int, u64]
        lib.exb_att_fold.restype = c_int
        lib.exb_att_fold.argtypes = [u64, c_longlong, c_int, c_int, c_int, u64, c_int, c_int, u64, c_int, u64, u64]
        lib.exb_att_last_error.restype = ctypes.c_char_p
        assert lib.exb_att_fwd_args_size() == ctypes.sizeof(_AttFwdArgs), "AttFwdArgs ABI mismatch"
        assert lib.exb_att_bwd_args_size() == ctypes.sizeof(_AttBwdArgs), "AttBwdArgs ABI mismatch"
        _att_proto = True
    return lib


def _att_ck(rc, what):
    if rc != 0:
        raise RuntimeError("%s: %s" % (what, _att_lib().exb_att_last_error().decode()))


AUTOINT_MAX_FIELDS = 64    # csrc/cuda/autoint_kernels.cu: two attention scores per lane of a warp
AUTOINT_MAX_WIDTH = 64     # d * heads: X_{l+1}'s bf16 operand is one 64-column K block of the next projection


def autoint_dims(nf, layers, d, h, res, embedding_dim=1, dnn_layers=0):
    """Sizes of the fused AutoInt: (dh, Np, Kp). dh = d * h is a layer's output width, Np = r(4 dh, 64)
    (r(3 dh, 64) without the residual) the width of the stacked projection [Q | K | V | R], Kp[l] the padded input
    width of layer l: r(embedding_dim, 64), then r(dh, 64) = 64. Raises ValueError for the sizes the kernels and the
    dense optimizer do not take: no layer, nf outside 1 .. 64, d or h below 1, d * h above 64, or more than 8 weight
    matrices with the ``dnn_layers`` of the DNN."""
    layers, d, h = int(layers), int(d), int(h)
    if layers < 1:
        raise ValueError("AutoInt needs at least one attention layer (got %d)" % layers)
    if not 1 <= nf <= AUTOINT_MAX_FIELDS:
        raise ValueError("the attention kernels take 1 .. %d fields (got %d)" % (AUTOINT_MAX_FIELDS, nf))
    if d < 1 or h < 1:
        raise ValueError("att_embedding_size and att_head_num must be positive (got %d, %d)" % (d, h))
    if d * h > AUTOINT_MAX_WIDTH:
        raise ValueError("att_embedding_size * att_head_num = %d is above %d" % (d * h, AUTOINT_MAX_WIDTH))
    if dnn_layers + layers > _OPT_MAX_MATS:
        raise ValueError("the fused optimizer kernel takes at most %d weight matrices (DNN + attention layers)"
                         % _OPT_MAX_MATS)
    dh = d * h
    Np = _r((4 if res else 3) * dh, 64)
    return dh, Np, [_r(int(embedding_dim), 64)] + [_r(dh, 64)] * (layers - 1)


def cross_cols(nf, D, Dp, nd):
    """Columns of the A0 layout [nf*Dp embedding | nd dense | pad | ones] that hold DCN-v2's input
    x = [emb (nf*D) | dense (nd)], in the order of x: field j's embedding column d < D is column j*Dp + d, the
    dense features follow at nf*Dp."""
    return [j * Dp + d for j in range(nf) for d in range(D)] + [nf * Dp + i for i in range(nd)]


def cin_dims(nf, cin_layers, split_half):
    """Per-layer sizes of the fused CIN: (H, N, Kp, Np, dir_lo) lists. H[k] channels enter layer k (H[0] = nf),
    the interaction operand Z_k has C_k = H[k] * nf columns plus the bias column, padded to Kp[k]; the layer has
    N[k] channels padded to Np[k]; its direct (pooled) channels are [dir_lo[k], N[k]). Raises ValueError for the
    sizes the CIN kernels cannot run."""
    layers = [int(n) for n in cin_layers]
    K = len(layers)
    if K < 1:
        raise ValueError("xDeepFM needs at least one CIN layer")
    if nf > 64:
        raise ValueError("the CIN kernels take at most 64 fields (got %d)" % nf)
    H, dir_lo = [nf], []
    for k, n in enumerate(layers):
        if n < 1:
            raise ValueError("CIN layer sizes must be positive: %r" % (layers,))
        last = k == K - 1
        if split_half and not last and n % 2:
            raise ValueError("cin_split_half needs even sizes below the last layer: %r" % (layers,))
        dir_lo.append(n // 2 if split_half and not last else 0)
        if not last:
            h = n // 2 if split_half else n
            if h > 256:
                raise ValueError("a CIN layer hands at most 256 channels on (got %d)" % h)
            H.append(h)
    for h in H:
        if _r(h * nf, 8) > 12800:       # exb_cin_outer_bwd stages 8 rows of dZ (bf16) in 200 KB of shared memory
            raise ValueError("CIN interaction width H * fields = %d is above 12800" % (h * nf))
    Kp = [_r(H[k] * nf + 1, 64) for k in range(K)]
    Np = [_r(n, 64) for n in layers]
    return H, layers, Kp, Np, dir_lo


class DenseLayout:
    """What ``FusedCTR``'s flat padded fp32 buffer (``theta``, and alike ``gtheta`` / ``accum`` / ``accum2``) holds.

    ``segs``    {segment: (offset, size)}, ``n_theta`` the buffer's length;
    ``shapes``  {segment: (R, C)}: the DNN / CIN / cross matrices ``W{l}`` / ``C{k}`` / ``X{l}`` are [R, C], the
                replicated table ``cache_emb`` is [rows, Dp], every other segment is one row of C entries;
    ``params``  {logical name: (shape, blocks)}: a block (segment, rows, cols) is the sub-matrix of real rows and
                columns of one segment; a parameter is its blocks side by side, reshaped to ``shape``.

    The logical names and shapes are those of ``models.ctr.CTRModel``'s dense parameters, plus ``dnn_out.bias``
    (the output weight that faces the last hidden layer's ones column). The embedding columns of the first DNN
    layer and of the cross network are in the order server features, then cached features (the A0 order)."""

    def __init__(self, segs, n_theta, shapes, params):
        self.segs, self.n_theta, self.shapes, self.params = segs, n_theta, shapes, params

    def index(self, name):
        """flat indices (int64, the parameter's shape) of a logical parameter in the buffer"""
        def ix(v):
            return torch.arange(v.start, v.stop) if isinstance(v, range) else torch.as_tensor(v, dtype=torch.long)

        shape, blocks = self.params[name]
        parts = []
        for seg, rows, cols in blocks:
            off, C = self.segs[seg][0], self.shapes[seg][1]
            parts.append(off + ix(rows)[:, None] * C + ix(cols)[None, :])
        return torch.cat(parts, 1).reshape(shape)

    def gather(self, flat):
        """{logical name: tensor} read out of a flat buffer"""
        return {name: flat[self.index(name).to(flat.device)] for name in self.params}

    def scatter(self, flat, tensors):
        """write every logical parameter of ``tensors`` into the flat buffer (in place)"""
        for name in self.params:
            idx = self.index(name).to(flat.device)
            flat[idx] = tensors[name].to(device=flat.device, dtype=flat.dtype).reshape(idx.shape)


def dense_layout(vocab_sizes, num_dense, embedding_dim, model, hidden, cached=(), cin_layers=(128, 128),
                 cin_split_half=True, cross_layers=3, att_layers=3, att_embedding_size=8, att_head_num=2, att_res=True):
    """The ``DenseLayout`` of a ``FusedCTR`` configuration (``cached``: the features held in the replicated table).
    Needs no GPU: save, load and export read and write the dense state through this map alone."""
    vocab, model, hidden = list(vocab_sizes), model.lower(), [int(h) for h in hidden]
    nf, nd, D, Dp = len(vocab), int(num_dense), int(embedding_dim), _r(int(embedding_dim), 4)
    Hp = [_r(h + 1, 64) for h in hidden]
    K0p = _r(nf * Dp + nd + 1, 64)
    dims = [K0p] + Hp
    segs, shapes, off = {}, {}, 0

    def seg(name, R, C, n=None):
        nonlocal off
        segs[name], shapes[name] = (off, R * C), (R, C)
        off = _r(off + (R * C if n is None else n), 4)

    for l in range(len(hidden)):
        seg("W%d" % l, Hp[l], dims[l])
    cin = model == "xdeepfm"
    if cin:
        cH, cN, cKp, cNp, clo = cin_dims(nf, cin_layers, cin_split_half)
        for k in range(len(cN)):        # bias in column H_k * nf
            seg("C%d" % k, cNp[k], cKp[k])
    Lc = int(cross_layers) if model == "dcn" else 0
    for l in range(Lc):                 # bias in the ones column K0p - 1
        seg("X%d" % l, K0p, K0p)
    La = int(att_layers) if model == "autoint" else 0
    if La:                              # [W_query | W_key | W_value | W_res] of layer l, [in, out] as in DeepCTR
        adh, aNp, aKp = autoint_dims(nf, La, att_embedding_size, att_head_num, att_res, D, len(hidden))
        for l in range(La):
            seg("T%d" % l, aKp[l], aNp)
    seg("wout", 1, Hp[-1])
    seg("wd", 1, max(nd, 1))
    seg("bias", 1, 1)
    if cin:
        T = sum(n - lo for n, lo in zip(cN, clo))
        seg("wcin", 1, T)
    if Lc:
        seg("wcross", 1, K0p)
    if La:
        seg("watt", 1, nf * adh)
    vc = sum(vocab[f] for f in cached)
    seg("cache_emb", vc, Dp)
    seg("cache_lin", 1, vc, n=max(vc, 1))

    real0 = cross_cols(nf, D, Dp, nd)   # [emb (nf*D) | dense (nd)] among the A0 columns
    params = {}
    for l, h in enumerate(hidden):
        cols = real0 if l == 0 else range(hidden[l - 1])
        params["dnn.%d.weight" % (2 * l)] = ((h, len(cols)), [("W%d" % l, range(h), cols)])
        params["dnn.%d.bias" % (2 * l)] = ((h,), [("W%d" % l, range(h), [dims[l] - 1])])
    hL = hidden[-1]
    if Lc:                              # CTRModel's order: cat([cross(x), dnn(x)])
        params["dnn_out.weight"] = ((1, len(real0) + hL), [("wcross", [0], real0), ("wout", [0], range(hL))])
    elif La:                            # CTRModel's order: cat([flatten(att(emb)), dnn(x)])
        params["dnn_out.weight"] = ((1, nf * adh + hL), [("watt", [0], range(nf * adh)), ("wout", [0], range(hL))])
    else:
        params["dnn_out.weight"] = ((1, hL), [("wout", [0], range(hL))])
    params["dnn_out.bias"] = ((1,), [("wout", [0], [Hp[-1] - 1])])
    if nd:
        params["dense_linear.weight"] = ((1, nd), [("wd", [0], range(nd))])
    params["bias"] = ((1,), [("bias", [0], [0])])
    if vc:
        params["cache_emb"] = ((vc, D), [("cache_emb", range(vc), range(D))])
        params["cache_lin"] = ((vc, 1), [("cache_lin", [0], range(vc))])
    if cin:
        for k, n in enumerate(cN):
            C = cH[k] * nf
            params["cin.convs.%d.weight" % k] = ((n, C, 1), [("C%d" % k, range(n), range(C))])
            params["cin.convs.%d.bias" % k] = ((n,), [("C%d" % k, range(n), [C])])
        params["cin_out.weight"] = ((1, T), [("wcin", [0], range(T))])
    for l in range(Lc):
        n = len(real0)
        params["cross.w.%d.weight" % l] = ((n, n), [("X%d" % l, real0, real0)])
        params["cross.w.%d.bias" % l] = ((n,), [("X%d" % l, real0, [K0p - 1])])
    names = ("W_query", "W_key", "W_value") + (("W_res",) if att_res else ())
    for l in range(La):
        d_in = D if l == 0 else adh
        for k, name in enumerate(names):
            params["att.layers.%d.%s" % (l, name)] = ((d_in, adh), [("T%d" % l, range(d_in), range(k * adh, (k + 1) * adh))])
    return DenseLayout(segs, off, shapes, params)


# the dense optimizer's state slots: accum holds the first, accum2 the second (csrc/cuda/dense_kernels.cu: dense_opt_one)
DENSE_OPT_SLOTS = {"adagrad": ("accumulator",), "adam": ("m", "v"), "ftrl": ("accumulator", "linear")}
CHECKPOINT_FORMAT = "openembedding_b200.FusedCTR/1"
# what a checkpoint must agree on with the model that loads it (batch, world size and optimizer may differ)
CONFIG_KEYS = ("model", "vocab", "cached", "embedding_dim", "num_dense", "hidden", "cin_layers", "cin_split_half",
               "cross_layers", "pack_linear", "att_layers", "att_embedding_size", "att_head_num", "att_res")


class FusedCTR:
    """DeepFM (use_fm=True), Wide&Deep, xDeepFM, DCN-v2 or AutoInt (use_fm=False; xDeepFM adds the CIN branch, DCN-v2
    the cross network, AutoInt the field self-attention) with the whole step on own kernels."""

    def __init__(self, vocab_sizes, num_dense=13, embedding_dim=64, model="deepfm", batch=4096, hidden=None,
                 sparse_optimizer=None, cache_threshold=0, lr=0.001, initial_accumulator_value=0.1, eps=1e-7,
                 num_shards=None, dw_splits=8, seed=0, pack_linear=None, dense_optimizer=None,
                 cin_layers=(128, 128), cin_split_half=True, cross_layers=3, att_layers=3, att_embedding_size=8,
                 att_head_num=2, att_res=True):
        from .ctr import FusedEmbeddings, _default_hidden
        ctx = get_context()
        if ctx.device.type != "cuda":
            raise RuntimeError("FusedCTR runs on the CUDA engine only (use models.ctr.CTRModel on CPU)")
        assert batch % 128 == 0, "the fused dense path needs batch % 128 == 0"
        self.ctx, self.dev, self.lib = ctx, ctx.device, _lib()
        self.model = model.lower()
        assert self.model in ("deepfm", "wdl", "xdeepfm", "dcn", "autoint")
        self.use_fm = self.model == "deepfm"
        self.B, self.nd, self.D = batch, num_dense, embedding_dim
        self.Dp = _r(embedding_dim, 4)
        self.vocab = list(vocab_sizes)
        self.nf = len(self.vocab)
        if hidden is None:
            hidden = _default_hidden(self.model)
        self.hidden = list(hidden)
        # xDeepFM: Compressed Interaction Network over the nf embeddings, rows r = (sample, embedding column)
        self.cin = self.model == "xdeepfm"
        self.cin_split_half = bool(cin_split_half)
        self.cin_layers = []
        if self.cin:
            self.cin_H, self.cin_layers, self.cin_Kp, self.cin_Np, self.cin_lo = cin_dims(self.nf, cin_layers,
                                                                                          self.cin_split_half)
            if len(self.hidden) + len(self.cin_layers) > _OPT_MAX_MATS:
                raise ValueError("the fused optimizer kernel takes at most %d weight matrices (DNN + CIN layers)"
                                 % _OPT_MAX_MATS)
        # DCN-v2: cross network x_{l+1} = x0 * (W_l x_l + b_l) + x_l on the A0 layout, one [K0p, K0p] matrix per layer
        self.dcn = self.model == "dcn"
        self.cross_layers = int(cross_layers) if self.dcn else 0
        if self.dcn:
            if self.cross_layers < 1:
                raise ValueError("DCN-v2 needs at least one cross layer (got %d)" % self.cross_layers)
            if len(self.hidden) + self.cross_layers > _OPT_MAX_MATS:
                raise ValueError("the fused optimizer kernel takes at most %d weight matrices (DNN + cross layers)"
                                 % _OPT_MAX_MATS)
        # AutoInt: stacked self-attention over the fields, rows r = (sample, field), one stacked projection per layer
        self.autoint = self.model == "autoint"
        self.att_layers = int(att_layers) if self.autoint else 0
        if self.autoint:
            self.att_d, self.att_h, self.att_res = int(att_embedding_size), int(att_head_num), bool(att_res)
            self.att_dh, self.att_Np, self.att_Kp = autoint_dims(self.nf, self.att_layers, self.att_d, self.att_h,
                                                                 self.att_res, embedding_dim, len(self.hidden))
        self.Hp = [_r(h + 1, 64) for h in self.hidden]
        self.lr, self.eps, self.dw_splits = lr, eps, int(os.environ.get("EXB_DW_SPLITS", dw_splits))
        self.cached = [f for f, v in enumerate(self.vocab) if 0 < v < cache_threshold]
        self.server = [f for f in range(self.nf) if f not in self.cached]
        self.ns, self.nc = len(self.server), len(self.cached)
        nf, Dp = self.nf, self.Dp
        self.K0p = _r(nf * Dp + num_dense + 1, 64)
        self.lin0 = self.K0p
        self.XS = _r(self.K0p + self.ns, 4)
        sparse_optimizer = sparse_optimizer or {"category": "adagrad"}
        zero = {"category": "constant", "value": 0.0}
        # pack_linear: the dim-D embedding and the dim-1 linear ("wide") weight of a sparse feature share ONE
        # server row of dim D+1 (split-row feature): half the lookups, unique ids, hash inserts, NVLink rows and
        # optimizer rows of the two-variables-per-feature layout of the reference benchmark
        # (criteo_deepctr.py:60-110). Same math per element; the checkpoint then holds one variable per feature.
        if pack_linear is None:
            pack_linear = os.environ.get("EXB_PACK_LINEAR", "1") != "0"
        self.pack_linear = bool(pack_linear)
        if self.pack_linear:
            specs = [{"vocab": self.vocab[f], "dim": embedding_dim + 1, "col": f, "initializer": zero} for f in self.server]
            self.sparse = FusedEmbeddings(specs, batch, sparse_optimizer, num_shards=num_shards, ncols=nf,
                                          feat_offsets=[j * Dp for j in range(self.ns)], io_stride=self.XS,
                                          feat_offsets2=[self.lin0 + j for j in range(self.ns)],
                                          feat_split=[embedding_dim] * self.ns)
        else:
            specs = [{"vocab": self.vocab[f], "dim": embedding_dim, "col": f, "initializer": zero} for f in self.server]
            specs += [{"vocab": self.vocab[f], "dim": 1, "col": f, "initializer": zero} for f in self.server]
            offs = [j * Dp for j in range(self.ns)] + [self.lin0 + j for j in range(self.ns)]
            self.sparse = FusedEmbeddings(specs, batch, sparse_optimizer, num_shards=num_shards, ncols=nf,
                                          feat_offsets=offs, io_stride=self.XS)
        self.group = self.sparse.group
        dev = self.dev
        f32, bf16 = torch.float32, torch.bfloat16
        # ---- flat parameter buffer: the matrices (DNN, CIN filters [Np_k, Kp_k], cross [K0p, K0p]; refreshed to bf16
        # by the optimizer), then wout, wd, bias, wcin, wcross (x_L's output weights, zero outside the real columns),
        # cache_emb, cache_lin (dense_layout)
        self.layout = dense_layout(self.vocab, num_dense, embedding_dim, self.model, self.hidden, self.cached,
                                   self.cin_layers, self.cin_split_half, self.cross_layers, self.att_layers,
                                   *((self.att_d, self.att_h, self.att_res) if self.autoint else ()))
        segs, off = self.layout.segs, self.layout.n_theta
        dims = [self.K0p] + self.Hp
        L = len(self.hidden)
        K = len(self.cin_layers)
        Lc = self.cross_layers
        La = self.att_layers
        if self.cin:
            self.cin_T = sum(n - lo for n, lo in zip(self.cin_layers, self.cin_lo))    # pooled CIN features
        self.cache_rows = sum(self.vocab[f] for f in self.cached)
        self.segs, self.n_theta = segs, off
        self.theta = torch.zeros(off, dtype=f32, device=dev)
        # dense optimizer (tf.keras semantics): {"category": "adagrad" | "adam" | "ftrl", ...}; default Adagrad(lr)
        from ..config import normalize_optimizer
        dopt = normalize_optimizer(dense_optimizer or {"category": "adagrad", "learning_rate": lr,
                                                        "initial_accumulator_value": initial_accumulator_value, "epsilon": eps})
        if dopt["category"] not in ("adagrad", "adam", "ftrl"):
            raise ValueError("fused dense optimizer: adagrad, adam or ftrl")
        self.dense_opt = dopt
        self.lr = lr = float(dopt["learning_rate"])
        acc0 = float(dopt.get("initial_accumulator_value", 0.0)) if dopt["category"] in ("adagrad", "ftrl") else 0.0
        self._acc0 = acc0
        self.accum = torch.full((off,), acc0, dtype=f32, device=dev)
        self.accum2 = torch.zeros(off if dopt["category"] != "adagrad" else 4, dtype=f32, device=dev)
        self.opt_step = torch.zeros(1, dtype=torch.int32, device=dev)
        self._ar = None
        self._rider = False
        self.overlap = os.environ.get("EXB_OVERLAP", "0") == "1"
        self.late_cachegrad = os.environ.get("EXB_LATE_CACHEGRAD", "0") == "1"     # measured: no gain (0.2260 vs 0.2240), the tail pull owns the SMs
        if ctx.world > 1:     # gradients are produced straight into the peer-mapped all-reduce buffer
            from ..ops.p2p_allreduce import P2PAllReduce
            self._ar = P2PAllReduce(ctx, off)
            self.gtheta = self._ar.grad
            # the reduction rides on the sparse push kernel's cross-GPU barriers instead of being a kernel with two
            # barriers of its own (EXB_AR_RIDER=0: separate exb_ar_fused_kernel launch)
            self._rider = (os.environ.get("EXB_AR_RIDER", "1") != "0" and not self.overlap
                           and hasattr(self.group, "set_dense_reduce"))
            if self._rider:
                self.group.set_dense_reduce(self._ar.bufs, off)
        else:
            self.gtheta = torch.zeros(off, dtype=f32, device=dev)
        gen = torch.Generator(device="cpu").manual_seed(seed)
        fan_in = [nf * embedding_dim + num_dense] + self.hidden
        for l in range(L):
            W = self.view("W%d" % l).view(self.Hp[l], dims[l])
            h_out = self.hidden[l]
            std = math.sqrt(2.0 / (fan_in[l] + h_out))            # glorot normal (DeepCTR DNN default)
            real_in = nf * Dp + num_dense if l == 0 else self.hidden[l - 1]
            blk = torch.randn(h_out, real_in, generator=gen) * std
            if l == 0 and Dp != embedding_dim:                     # zero the weights that face pad columns
                m = torch.ones(nf, Dp)
                m[:, embedding_dim:] = 0
                blk[:, :nf * Dp] *= m.reshape(-1)
            W[:h_out, :real_in] = blk.to(dev)
        # DCN-v2: w_cross and wout are one Dense(1) over [x_L | h_dnn] (glorot normal over the concatenation)
        self.cross_n = nf * embedding_dim + num_dense if self.dcn else 0
        std_out = math.sqrt(2.0 / (self.hidden[-1] + self.cross_n + 1))
        self.view("wout")[: self.hidden[-1]] = (torch.randn(self.hidden[-1], generator=gen) * std_out).to(dev)
        if num_dense:
            self.view("wd")[:num_dense] = (torch.randn(num_dense, generator=gen) * math.sqrt(2.0 / (num_dense + 1))).to(dev)
        if self.dcn:                # DeepCTR CrossNet (matrix): glorot-normal kernels over the real block, zero biases
            self.cross_real = torch.tensor(cross_cols(nf, embedding_dim, Dp, num_dense), dtype=torch.long, device=dev)
            n = self.cross_n
            self.view("wcross")[self.cross_real] = (torch.randn(n, generator=gen) * std_out).to(dev)
            for l in range(Lc):
                blk = torch.randn(n, n, generator=gen) * math.sqrt(2.0 / (n + n))
                self.xview(l)[self.cross_real[:, None], self.cross_real[None, :]] = blk.to(dev)
        if self.autoint:            # DeepCTR InteractingLayer: TruncatedNormal(stddev 0.05); w_att, wout one Dense(1)
            dh, T = self.att_dh, nf * self.att_dh
            std = math.sqrt(2.0 / (self.hidden[-1] + T + 1))
            self.view("wout")[: self.hidden[-1]] = (torch.randn(self.hidden[-1], generator=gen) * std).to(dev)
            self.view("watt")[:] = (torch.randn(T, generator=gen) * std).to(dev)
            nmat = 4 if self.att_res else 3
            for l in range(La):
                d_in = embedding_dim if l == 0 else dh
                w = torch.empty(d_in, nmat * dh)
                torch.nn.init.trunc_normal_(w, std=0.05, a=-0.1, b=0.1, generator=gen)
                self.aview(l)[:d_in, :nmat * dh] = w.to(dev)
        for k in range(K):          # DeepCTR CIN: glorot-uniform filters (fan_in H_k * nf, fan_out N_k), zero biases
            C, n = self.cin_H[k] * nf, self.cin_layers[k]
            lim = math.sqrt(6.0 / (C + n))
            self.cview(k)[:n, :C] = ((torch.rand(n, C, generator=gen) * 2 - 1) * lim).to(dev)
        if self.cin:                # exFM_logit = Dense(1, use_bias=False, glorot_normal)
            self.view("wcin")[:] = (torch.randn(self.cin_T, generator=gen) * math.sqrt(2.0 / (self.cin_T + 1))).to(dev)
        # ---- bf16 K-major weight copies
        self.Wb = [torch.zeros(self.Hp[l], dims[l], dtype=bf16, device=dev) for l in range(L)]
        self.WTb = [torch.zeros(dims[l], self.Hp[l], dtype=bf16, device=dev) for l in range(L)]
        self.cWb = [torch.zeros(self.cin_Np[k], self.cin_Kp[k], dtype=bf16, device=dev) for k in range(K)]
        self.cWTb = [torch.zeros(self.cin_Kp[k], self.cin_Np[k], dtype=bf16, device=dev) for k in range(K)]
        self.xWb = [torch.zeros(self.K0p, self.K0p, dtype=bf16, device=dev) for l in range(Lc)]
        self.xWTb = [torch.zeros(self.K0p, self.K0p, dtype=bf16, device=dev) for l in range(Lc)]
        self.aWb = [torch.zeros(self.att_Kp[l], self.att_Np, dtype=bf16, device=dev) for l in range(La)]
        self.aWTb = [torch.zeros(self.att_Np, self.att_Kp[l], dtype=bf16, device=dev) for l in range(La)]
        # ---- activations
        B = batch
        self.X32 = torch.zeros(B, self.XS, dtype=f32, device=dev)
        self.G32 = torch.zeros(B, self.XS, dtype=f32, device=dev)
        self.A0 = torch.zeros(B, self.K0p, dtype=bf16, device=dev)
        self.A0T = torch.zeros(self.K0p, B, dtype=bf16, device=dev)
        self.H = [torch.zeros(B, hp, dtype=bf16, device=dev) for hp in self.Hp]
        self.HT = [torch.zeros(hp, B, dtype=bf16, device=dev) for hp in self.Hp]
        self.dZ = [torch.zeros(B, hp, dtype=bf16, device=dev) for hp in self.Hp]
        self.dZT = [torch.zeros(hp, B, dtype=bf16, device=dev) for hp in self.Hp]
        self.S = torch.zeros(B, Dp, dtype=f32, device=dev)
        self.base = torch.zeros(B, dtype=f32, device=dev)
        self.dlogit = torch.zeros(B, dtype=f32, device=dev)
        self.loss = torch.zeros(1, dtype=f32, device=dev)
        self.logits = torch.zeros(B, dtype=f32, device=dev)       # predict_forward's outputs
        self.probs = torch.zeros(B, dtype=f32, device=dev)
        self._predict_args = _PredictArgs(self.H[-1].data_ptr(), self.Hp[-1], self.view("wout").data_ptr(),
                                          self.base.data_ptr(), self.logits.data_ptr(), self.probs.data_ptr(), B)
        offs_c, o = [], 0
        for f in self.cached:
            offs_c.append(o)
            o += self.vocab[f]
        self.cache_col = torch.tensor(self.cached or [0], dtype=torch.int32, device=dev)
        self.cache_off = torch.tensor(offs_c or [0], dtype=torch.int64, device=dev)
        self.cache_vocab = torch.tensor([self.vocab[f] for f in self.cached] or [0], dtype=torch.int32, device=dev)
        # push+update runs on a second stream next to the dW GEMMs / dense optimizer (fork after dX1, join at step end)
        self.overlap = os.environ.get("EXB_OVERLAP", "0") == "1"
        # weight-gradient GEMMs read the batch-major activations as MN-major operands: no A0^T / H^T / dZ^T copies
        self.mn_major = os.environ.get("EXB_MN_MAJOR", "1") != "0"
        self._s2 = torch.cuda.Stream(device=dev)
        self._ev_fork, self._ev_join, self._ev_plan = torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()
        assert L + K + Lc + La <= _OPT_MAX_MATS, "the fused optimizer kernel takes at most %d weight matrices" % _OPT_MAX_MATS
        oa = _DenseOptArgs()
        oa.theta, oa.accum, oa.grad = self.theta.data_ptr(), self.accum.data_ptr(), self.gtheta.data_ptr()
        oa.n, oa.flat_lo, oa.lr, oa.eps = self.n_theta, segs["wout"][0], self.lr, float(self.dense_opt.get("epsilon", self.eps))
        oa.nmat, oa.zero_grad = L + K + Lc + La, 1
        d = self.dense_opt
        oa.kind = {"adagrad": 0, "adam": 1, "ftrl": 2}[d["category"]]
        oa.accum2, oa.step = self.accum2.data_ptr(), self.opt_step.data_ptr()
        oa.b1, oa.b2 = float(d.get("beta_1", 0.9)), float(d.get("beta_2", 0.999))
        oa.l1, oa.l2 = float(d.get("l1_regularization_strength", 0.0)), float(d.get("l2_regularization_strength", 0.0))
        oa.l2s, oa.lrp = float(d.get("l2_shrinkage_regularization_strength", 0.0)), float(d.get("learning_rate_power", -0.5))
        oa.beta = float(d.get("beta", 0.0))
        for l in range(L):
            oa.mat[l].off, oa.mat[l].R, oa.mat[l].C = segs["W%d" % l][0], self.Hp[l], dims[l]
            oa.mat[l].Wb, oa.mat[l].WTb = self.Wb[l].data_ptr(), self.WTb[l].data_ptr()
        for k in range(K):
            oa.mat[L + k].off, oa.mat[L + k].R, oa.mat[L + k].C = segs["C%d" % k][0], self.cin_Np[k], self.cin_Kp[k]
            oa.mat[L + k].Wb, oa.mat[L + k].WTb = self.cWb[k].data_ptr(), self.cWTb[k].data_ptr()
        for l in range(Lc):
            i = L + K + l
            oa.mat[i].off, oa.mat[i].R, oa.mat[i].C = segs["X%d" % l][0], self.K0p, self.K0p
            oa.mat[i].Wb, oa.mat[i].WTb = self.xWb[l].data_ptr(), self.xWTb[l].data_ptr()
        for l in range(La):
            i = L + K + Lc + l
            oa.mat[i].off, oa.mat[i].R, oa.mat[i].C = segs["T%d" % l][0], self.att_Kp[l], self.att_Np
            oa.mat[i].Wb, oa.mat[i].WTb = self.aWb[l].data_ptr(), self.aWTb[l].data_ptr()
        self._opt_args = oa
        if self.cin:
            self._cin_init_buffers()
        if self.dcn:
            self._cross_init_buffers()
        if self.autoint:
            self._att_init_buffers()
        self._grad_dirty = False
        self.load_generation = 0     # counts ``load`` calls: rows and plans prefetched before one are stale
        # persistent GEMM chains: forward (fwd1 -> ... -> fwdL) and backward (dX / dW of every layer) in ONE launch
        # each (csrc/cuda/gemm_wgmma.cu: exb_gemm_chain_kernel). EXB_GEMM_CHAIN=0: one launch per GEMM.
        mode = os.environ.get("EXB_GEMM_CHAIN", "bwd")          # "0" | "bwd" | "1" (forward and backward)
        self.use_chain = mode != "0" and self.mn_major and L <= 4
        self.chain_fwd = self.use_chain and mode == "1"
        self.fwd_chain = self.bwd_chain = None
        if self.use_chain:
            fd, src = [], self.A0
            for l in range(L):
                fd.append(G.chain_nt(src, self.Wb[l], B, self.Hp[l], dims[l], self.H[l], mode=G.EPI_FWD, relu=True,
                                     ones_col=self.Hp[l] - 1, dep=l - 1))
                src = self.H[l]
            self.fwd_chain = G.GemmChain(fd, dev)
            bd, prod = [], -1          # prod: index (in the chain) of the GEMM that produced dZ[l]
            for l in range(L - 1, -1, -1):
                gW = self.gview("W%d" % l).view(self.Hp[l], dims[l])
                if l > 0:
                    bd.append(G.chain_nt(self.dZ[l], self.WTb[l], B, self.Hp[l - 1], self.Hp[l], self.dZ[l - 1], mode=G.EPI_DX,
                                         ones_col=self.Hp[l - 1] - 1, mask=self.H[l - 1], dep=prod))
                else:
                    bd.append(G.chain_nt(self.dZ[0], self.WTb[0], B, self.K0p, self.Hp[0], self.G32, mode=G.EPI_DX_FM,
                                         dlogit=self.dlogit, S=self.S, emb=self.X32,
                                         fm_cols=self.nf * self.Dp if self.use_fm else 0, D=self.Dp, dep=prod))
                nxt = len(bd) - 1
                bd.append(G.chain_tn(self.dZ[l], self.A0 if l == 0 else self.H[l - 1], self.Hp[l], dims[l], B, gW,
                                     splits=self.dw_splits, dep=prod))
                prod = nxt
            self.bwd_chain = G.GemmChain(bd, dev)
        self.refresh_weights()
        torch.cuda.synchronize(dev)

    # ---- helpers
    def view(self, name):
        o, n = self.segs[name]
        return self.theta[o:o + n]

    def gview(self, name):
        o, n = self.segs[name]
        return self.gtheta[o:o + n]

    def cview(self, k, grad=False):
        """CIN layer k's filter matrix [Np_k, Kp_k] (bias in column H_k * nf) in theta, or in gtheta"""
        return (self.gview if grad else self.view)("C%d" % k).view(self.cin_Np[k], self.cin_Kp[k])

    def xview(self, l, grad=False):
        """cross layer l's matrix [K0p, K0p] (out, in; bias in the ones column K0p - 1) in theta, or in gtheta"""
        return (self.gview if grad else self.view)("X%d" % l).view(self.K0p, self.K0p)

    def aview(self, l, grad=False):
        """AutoInt layer l's stacked projection [Kp_l, Np] = [W_query | W_key | W_value | W_res] (in, out) in theta, or
        in gtheta"""
        return (self.gview if grad else self.view)("T%d" % l).view(self.att_Kp[l], self.att_Np)

    # ---- xDeepFM: the CIN branch (csrc/cuda/cin_kernels.cu + the wgmma GEMM), every buffer allocated here once
    def _cin_init_buffers(self):
        B, D, m, K, dev = self.B, self.D, self.nf, len(self.cin_layers), self.dev
        f32, bf16 = torch.float32, torch.bfloat16
        self.cin_lib = _cin_lib()
        self.cin_R = R = B * D            # rows (sample, embedding column); the pad columns Dp - D are no CIN input
        H, Kp, Np = self.cin_H, self.cin_Kp, self.cin_Np
        self.cin_X0 = torch.zeros(R, m, dtype=f32, device=dev)
        self.cin_Z = [torch.zeros(R, Kp[k], dtype=bf16, device=dev) for k in range(K)]       # interaction operands
        self.cin_Y = [torch.zeros(R, Np[k], dtype=bf16, device=dev) for k in range(K)]       # layer outputs
        self.cin_dY = [torch.zeros(R, Np[k], dtype=bf16, device=dev) for k in range(K)]
        self.cin_dZ = [torch.zeros(R, Kp[k], dtype=bf16, device=dev) for k in range(K)]
        self.cin_dhid = [torch.zeros(R, H[k], dtype=f32, device=dev) for k in range(K)]
        self.cin_dx = [torch.zeros(R, m, dtype=f32, device=dev) for k in range(K)]
        self.cin_p = torch.zeros(B, self.cin_T, dtype=f32, device=dev)                        # pooled features
        pa = _CinPoolArgs()
        t0s, t0 = [], 0
        for k in range(K):
            pa.Y[k], pa.ldy[k] = self.cin_Y[k].data_ptr(), Np[k]
            pa.lo[k], pa.hi[k] = self.cin_lo[k], self.cin_layers[k]
            t0s.append(t0)
            t0 += self.cin_layers[k] - self.cin_lo[k]
        pa.K, pa.T, pa.D, pa.B = K, self.cin_T, D, B
        pa.wcin, pa.p, pa.base = self.view("wcin").data_ptr(), self.cin_p.data_ptr(), self.base.data_ptr()
        self._cin_pool_args = pa
        self._cin_dy_args = []
        for k in range(K):
            last = k == K - 1
            a = _CinDyArgs()
            a.Y, a.ldy, a.N, a.Np = self.cin_Y[k].data_ptr(), Np[k], self.cin_layers[k], Np[k]
            a.dir_lo, a.t0, a.wcin = self.cin_lo[k], t0s[k], self.view("wcin").data_ptr()
            a.dhid = 0 if last else self.cin_dhid[k + 1].data_ptr()
            a.ld_dhid, a.Hn = (0, 0) if last else (H[k + 1], H[k + 1])
            a.D, a.R, a.dlogit = D, R, self.dlogit.data_ptr()
            a.dY, a.lddy = self.cin_dY[k].data_ptr(), Np[k]
            a.p, a.g_wcin = self.cin_p.data_ptr(), self.gview("wcin").data_ptr() if last else 0
            a.T, a.B = self.cin_T, B
            self._cin_dy_args.append(a)
        srcs = [self.cin_dx[0], self.cin_dhid[0]] + self.cin_dx[1:]
        self._cin_fold_srcs = (ctypes.c_uint64 * len(srcs))(*[t.data_ptr() for t in srcs])
        # split-K of the filter-gradient GEMMs (K = R rows): about two waves of output tiles
        self.cin_splits = [max(1, min(R // 1024, 264 // ((Np[k] // 128 + 1) * (Kp[k] // 128 + 1)))) for k in range(K)]

    def _cin_hid(self, k):
        """(tensor, is_bf16, row stride) of layer k's input: X0 (fp32), then the handed-on channels of Y_{k-1}"""
        if k == 0:
            return self.cin_X0, 0, self.nf
        return self.cin_Y[k - 1], 1, self.cin_Np[k - 1]

    def _cin_forward(self, st):
        """X0 from X32, Z_k / Y_k of every layer, then p and base += p . w_cin (after prep, before the head)"""
        lib, B, R, m = self.cin_lib, self.B, self.cin_R, self.nf
        _cin_ck(lib.exb_cin_gather(self.X32.data_ptr(), self.XS, self.Dp, self.D, m, self.cin_X0.data_ptr(), B, st),
                "cin_gather")
        for k in range(len(self.cin_layers)):
            hid, hb, ld = self._cin_hid(k)
            Kp, Np = self.cin_Kp[k], self.cin_Np[k]
            _cin_ck(lib.exb_cin_outer(hid.data_ptr(), hb, ld, self.cin_H[k], self.cin_X0.data_ptr(), m, m,
                                      self.cin_Z[k].data_ptr(), Kp, Kp, R, st), "cin_outer")
            G.gemm_nt(self.cin_Z[k], self.cWb[k], R, Np, Kp, self.cin_Y[k], mode=G.EPI_FWD, relu=True, ones_col=-1,
                      stream=st)
        _cin_ck(lib.exb_cin_pool(ctypes.byref(self._cin_pool_args), st), "cin_pool")

    def _cin_backward(self, st):
        """dY / dZ / d hid / d x / filter gradients from the last layer down, g_wcin, then the fold of the embedding
        gradients into G32 (after the DNN's dX GEMM wrote those columns, before cachegrad and the push)"""
        lib, B, R, m = self.cin_lib, self.B, self.cin_R, self.nf
        for k in range(len(self.cin_layers) - 1, -1, -1):
            Kp, Np = self.cin_Kp[k], self.cin_Np[k]
            _cin_ck(lib.exb_cin_dy(ctypes.byref(self._cin_dy_args[k]), st), "cin_dy")
            G.gemm_nt(self.cin_dY[k], self.cWTb[k], R, Kp, Np, self.cin_dZ[k], mode=G.EPI_FWD, relu=False, ones_col=-1,
                      stream=st)
            hid, hb, ld = self._cin_hid(k)
            _cin_ck(lib.exb_cin_outer_bwd(self.cin_dZ[k].data_ptr(), Kp, hid.data_ptr(), hb, ld, self.cin_H[k],
                                          self.cin_X0.data_ptr(), m, m, self.cin_dhid[k].data_ptr(), self.cin_H[k],
                                          self.cin_dx[k].data_ptr(), m, R, st), "cin_outer_bwd")
            G.gemm_tn(self.cin_dY[k], self.cin_Z[k], Np, Kp, R, self.cview(k, grad=True), splits=self.cin_splits[k],
                      stream=st)
        _cin_ck(lib.exb_cin_fold(self.G32.data_ptr(), self.XS, self.Dp, self.D, m, B, self._cin_fold_srcs,
                                 len(self._cin_fold_srcs), st), "cin_fold")

    # ---- DCN-v2: the cross network (csrc/cuda/cross_kernels.cu + the wgmma GEMM), every buffer allocated here once
    def _cross_init_buffers(self):
        B, K0p, Lc, dev = self.B, self.K0p, self.cross_layers, self.dev
        f32, bf16 = torch.float32, torch.bfloat16
        self.cross_lib = _cross_lib()
        self.cross_U = [torch.zeros(B, K0p, dtype=f32, device=dev) for _ in range(Lc)]        # U_l = x_l W_l^T
        self.cross_Xf = [torch.zeros(B, K0p, dtype=f32, device=dev) for _ in range(Lc)]       # x_{l+1}
        self.cross_Xb = [torch.zeros(B, K0p, dtype=bf16, device=dev) for _ in range(Lc - 1)]  # bf16 x_{l+1} (GEMM A)
        self.cross_g = [torch.zeros(B, K0p, dtype=f32, device=dev) for _ in range(2)]         # g_l in cross_g[l % 2]
        self.cross_gx0 = torch.zeros(B, K0p, dtype=f32, device=dev)
        self.cross_P = torch.zeros(B, K0p, dtype=f32, device=dev)                             # P_l = dU_l W_l
        self.cross_dU = torch.zeros(B, K0p, dtype=bf16, device=dev)
        p = lambda t: t.data_ptr() if t is not None else 0

        def x0():
            return _CrossX0(self.X32.data_ptr(), self.XS, 0, self.nd, self.nf * self.Dp, self.Dp, self.D, K0p, B)
        wcross = self.view("wcross").data_ptr()
        self._cross_fwd_args = []
        for l in range(Lc):
            last = l == Lc - 1
            self._cross_fwd_args.append(_CrossFwdArgs(
                x0(), p(self.cross_U[l]), p(self.cross_Xf[l - 1]) if l else 0, p(self.cross_Xf[l]),
                0 if last else p(self.cross_Xb[l]), wcross, p(self.base) if last else 0))
        a = _CrossBwdArgs()
        a.x, a.dlogit, a.wcross, a.gout = x0(), p(self.dlogit), wcross, p(self.cross_g[Lc % 2])
        a.U, a.dU, a.gx0 = p(self.cross_U[Lc - 1]), p(self.cross_dU), p(self.cross_gx0)
        a.XfL, a.g_wcross = p(self.cross_Xf[Lc - 1]), self.gview("wcross").data_ptr()
        self._cross_top_args = a
        self._cross_bwd_args = []
        for l in range(Lc):
            a = _CrossBwdArgs()
            a.x, a.gin, a.P, a.gx0 = x0(), p(self.cross_g[(l + 1) % 2]), p(self.cross_P), p(self.cross_gx0)
            if l:
                a.gout, a.U, a.dU = p(self.cross_g[l % 2]), p(self.cross_U[l - 1]), p(self.cross_dU)
            else:
                a.G32 = p(self.G32)
            self._cross_bwd_args.append(a)
        # split-K of the weight-gradient GEMMs (K = batch): about two waves of 128 x 128 output tiles
        self.cross_splits = max(1, min(B // 1024, 264 // (K0p // 128 + 1) ** 2))

    def _cross_forward(self, st, dense):
        """U_l and x_{l+1} of every layer, then base += x_L . w_cross (after the forward GEMMs, before the head)"""
        lib, B, K0p = self.cross_lib, self.B, self.K0p
        for l in range(self.cross_layers):
            src = self.A0 if l == 0 else self.cross_Xb[l - 1]
            G.gemm_nt(src, self.xWb[l], B, K0p, K0p, self.cross_U[l], mode=G.EPI_DX_FM, fm_cols=0, stream=st)
            a = self._cross_fwd_args[l]
            a.x.dense = dense.data_ptr()
            _cross_ck(lib.exb_cross_fwd(ctypes.byref(a), st), "cross_fwd")

    def _cross_backward(self, st, dense):
        """g_L, then per layer from the last: P_l, the weight gradient, g_l / dU_{l-1} / gx0, and at layer 0 the fold
        of the cross network's input gradient into G32 (after the DNN's dX GEMM wrote those columns, before cachegrad
        and the push)"""
        lib, B, K0p = self.cross_lib, self.B, self.K0p
        self._cross_top_args.x.dense = dense.data_ptr()
        _cross_ck(lib.exb_cross_bwd_top(ctypes.byref(self._cross_top_args), st), "cross_bwd_top")
        for l in range(self.cross_layers - 1, -1, -1):
            G.gemm_nt(self.cross_dU, self.xWTb[l], B, K0p, K0p, self.cross_P, mode=G.EPI_DX_FM, fm_cols=0, stream=st)
            G.gemm_tn(self.cross_dU, self.A0 if l == 0 else self.cross_Xb[l - 1], K0p, K0p, B, self.xview(l, grad=True),
                      splits=self.cross_splits, stream=st)
            a = self._cross_bwd_args[l]
            a.x.dense = dense.data_ptr()
            _cross_ck(lib.exb_cross_bwd(ctypes.byref(a), st), "cross_bwd")

    # ---- AutoInt: the field self-attention (csrc/cuda/autoint_kernels.cu + the wgmma GEMM), buffers allocated once
    def _att_init_buffers(self):
        B, nf, La, dev = self.B, self.nf, self.att_layers, self.dev
        f32, bf16 = torch.float32, torch.bfloat16
        dh, Np, Kp = self.att_dh, self.att_Np, self.att_Kp
        self.att_lib = _att_lib()
        self.att_R = R = B * nf             # rows (sample, field)
        self.att_X = [torch.zeros(R, Kp[l], dtype=bf16, device=dev) for l in range(La)]        # layer inputs (GEMM A)
        self.att_QKVR = [torch.zeros(R, Np, dtype=f32, device=dev) for _ in range(La)]          # projections
        self.att_P = [torch.zeros(B, self.att_h, nf, nf, dtype=f32, device=dev) for _ in range(La)]   # softmax
        self.att_Xf = [torch.zeros(R, dh, dtype=f32, device=dev) for _ in range(La)]            # layer outputs
        self.att_dQKVR = [torch.zeros(R, Np, dtype=bf16, device=dev) for _ in range(La)]
        self.att_dX = [torch.zeros(R, Kp[l], dtype=f32, device=dev) for l in range(La)]         # input gradients
        self.att_gpart = torch.zeros((B + 127) // 128, nf * dh, dtype=f32, device=dev)          # g_watt partial sums
        p = lambda t: t.data_ptr() if t is not None else 0
        watt, res = self.view("watt").data_ptr(), int(self.att_res)
        self._att_fwd_args, self._att_bwd_args = [], []
        for l in range(La):
            last = l == La - 1
            self._att_fwd_args.append(_AttFwdArgs(
                p(self.att_QKVR[l]), Np, p(self.att_P[l]), p(self.att_Xf[l]), 0 if last else p(self.att_X[l + 1]),
                0 if last else Kp[l + 1], watt if last else 0, p(self.base) if last else 0, B, nf, self.att_d,
                self.att_h, res))
            self._att_bwd_args.append(_AttBwdArgs(
                p(self.att_QKVR[l]), Np, p(self.att_P[l]), p(self.att_Xf[l]), 0 if last else p(self.att_dX[l + 1]),
                0 if last else Kp[l + 1], p(self.dlogit) if last else 0, watt if last else 0, p(self.att_dQKVR[l]),
                p(self.att_gpart) if last else 0, B, nf, self.att_d, self.att_h, res, 0))
        # split-K of the weight-gradient GEMMs (K = R rows): about two waves of output tiles
        self.att_splits = [max(1, min(R // 1024, 264 // ((Kp[l] // 128 + 1) * (Np // 128 + 1)))) for l in range(La)]

    def _att_forward(self, st):
        """layer 0's operand from X32, then the projection and attention of every layer; the last adds
        flatten(X_L) . w_att to base (after the forward GEMMs, before the head)"""
        lib, R, Np, Kp = self.att_lib, self.att_R, self.att_Np, self.att_Kp
        _att_ck(lib.exb_att_gather(self.X32.data_ptr(), self.XS, self.Dp, self.D, self.nf, self.att_X[0].data_ptr(),
                                   Kp[0], self.B, st), "att_gather")
        for l in range(self.att_layers):
            G.gemm_nt(self.att_X[l], self.aWTb[l], R, Np, Kp[l], self.att_QKVR[l], mode=G.EPI_DX_FM, fm_cols=0, stream=st)
            _att_ck(lib.exb_att_fwd(ctypes.byref(self._att_fwd_args[l]), st), "att_fwd")

    def _att_backward(self, st):
        """per layer from the last: [dQ | dK | dV | dR], the weight gradient, the input gradient; then the fold of
        layer 0's input gradient into G32 (after the DNN's dX GEMM wrote those columns, before cachegrad and the push)
        and of g_watt's partial sums into gtheta"""
        lib, R, Np, Kp = self.att_lib, self.att_R, self.att_Np, self.att_Kp
        for l in range(self.att_layers - 1, -1, -1):
            _att_ck(lib.exb_att_bwd(ctypes.byref(self._att_bwd_args[l]), st), "att_bwd")
            G.gemm_tn(self.att_X[l], self.att_dQKVR[l], Kp[l], Np, R, self.aview(l, grad=True),
                      splits=self.att_splits[l], stream=st)
            G.gemm_nt(self.att_dQKVR[l], self.aWb[l], R, Kp[l], Np, self.att_dX[l], mode=G.EPI_DX_FM, fm_cols=0,
                      stream=st)
        _att_ck(lib.exb_att_fold(self.G32.data_ptr(), self.XS, self.Dp, self.D, self.nf, self.att_dX[0].data_ptr(),
                                 Kp[0], self.B, self.att_gpart.data_ptr(), self.nf * self.att_dh,
                                 self.gview("watt").data_ptr(), st), "att_fold")

    def _st(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    _trace = None          # list of (name, event) when stage tracing is on (tools/mp_timeline.py)

    def _mark(self, name):
        _timers.nvtx_mark(name)              # EXB_NVTX=1: stage boundaries on the nsys / ncu timeline
        if self._trace is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(torch.cuda.current_stream(self.dev))
            self._trace.append((name, ev))

    def refresh_weights(self):
        dims = [self.K0p] + self.Hp
        for l in range(len(self.hidden)):
            _ck(self.lib.exb_refresh_bf16(self.view("W%d" % l).data_ptr(), self.Wb[l].data_ptr(),
                                          self.WTb[l].data_ptr(), self.Hp[l], dims[l], self._st()), "refresh_bf16")
        for k in range(len(self.cin_layers)):
            _ck(self.lib.exb_refresh_bf16(self.view("C%d" % k).data_ptr(), self.cWb[k].data_ptr(), self.cWTb[k].data_ptr(),
                                          self.cin_Np[k], self.cin_Kp[k], self._st()), "refresh_bf16")
        for l in range(self.cross_layers):
            _ck(self.lib.exb_refresh_bf16(self.view("X%d" % l).data_ptr(), self.xWb[l].data_ptr(), self.xWTb[l].data_ptr(),
                                          self.K0p, self.K0p, self._st()), "refresh_bf16")
        for l in range(self.att_layers):
            _ck(self.lib.exb_refresh_bf16(self.view("T%d" % l).data_ptr(), self.aWb[l].data_ptr(), self.aWTb[l].data_ptr(),
                                          self.att_Kp[l], self.att_Np, self._st()), "refresh_bf16")

    def _forward(self, ids, dense, st, loss, opt_step):
        """prep, the forward GEMMs and the CIN / cross branches on the rows in X32: leaves H[-1] and base for a
        head. ``loss`` / ``opt_step``: device addresses prep clears / advances, 0 for neither."""
        B, L, tn = self.B, len(self.hidden), self.mn_major
        pa = _PrepArgs(self.X32.data_ptr(), self.XS, self.A0.data_ptr(), 0 if tn else self.A0T.data_ptr(), ids.data_ptr(), self.nf,
                       dense.data_ptr(), self.nd, self.view("cache_emb").data_ptr(), self.view("cache_lin").data_ptr(),
                       self.cache_col.data_ptr(), self.cache_off.data_ptr(), self.nc, self.view("wd").data_ptr(),
                       self.view("bias").data_ptr(), self.S.data_ptr(), self.base.data_ptr(), B, self.K0p, self.Dp,
                       self.nf, self.ns, self.lin0, int(self.use_fm), loss, opt_step)
        _ck(self.lib.exb_prep(ctypes.byref(pa), B, self.Dp, st), "prep")
        self._mark("prep")
        dims = [self.K0p] + self.Hp
        src = self.A0
        if self.chain_fwd:
            self.fwd_chain.launch(st)
        else:
            for l in range(L):
                G.gemm_nt(src, self.Wb[l], B, self.Hp[l], dims[l], self.H[l], mode=G.EPI_FWD, relu=True,
                          ones_col=self.Hp[l] - 1, outT=self.HT[l] if (l < L - 1 and not tn) else None, stream=st)
                src = self.H[l]
        self._mark("fwd_gemm")
        if self.cin:
            self._cin_forward(st)
            self._mark("cin_fwd")
        if self.dcn:
            self._cross_forward(st, dense)
            self._mark("cross_fwd")
        if self.autoint:
            self._att_forward(st)
            self._mark("att_fwd")

    # ---- forward-only pass (evaluation; all launches on the current stream)
    def predict_forward(self, ids, dense):
        """Logits and sigmoid probabilities of a full batch into ``self.logits`` / ``self.probs`` (fp32 [B]):
        stateless pull of the rows into X32, prep (the training loss and the optimizer step counter untouched), the
        forward GEMMs, the CIN / cross branches, then the predict head. No parameter, optimizer state, gradient,
        sparse plan or table row changes -- but X32 and the other activation buffers are overwritten, so rows that
        a training step prefetched into X32 are gone (``FusedTrainer`` makes the next step pull again)."""
        B = self.B
        assert ids.shape == (B, self.nf) and ids.dtype == torch.int64 and ids.is_contiguous()
        assert dense.shape == (B, self.nd) and dense.dtype == torch.float32 and dense.is_contiguous()
        st = self._st()
        self.group.pull(ids, out=self.X32)
        self._mark("pull")
        self._forward(ids, dense, st, 0, 0)
        _ck(self.lib.exb_predict_head(ctypes.byref(self._predict_args), st), "predict_head")
        self._mark("predict_head")
        return self.logits

    def kernels_per_eval(self, metric=False):
        """launches of our own kernels in one ``predict_forward`` (+ 1 for the metric update of an evaluation)"""
        L = len(self.hidden)
        prep = 1 if (self.mn_major and 128 % self.Dp == 0) else 2
        n = 1 + prep + (1 if self.chain_fwd else L) + 1                # pull prep GEMMs head
        n += 2 + 2 * len(self.cin_layers) if self.cin else 0          # gather + pool, per layer outer + GEMM
        n += 2 * self.cross_layers if self.dcn else 0                 # per layer GEMM + cross forward
        n += 1 + 2 * self.att_layers if self.autoint else 0           # gather, per layer GEMM + attention forward
        return n + (1 if metric else 0)

    # ---- one training step (all launches on the current stream)
    def forward_backward(self, ids, dense, labels, update=True, next_ids=None, pulled=False):
        """One training step. ``next_ids``: ids of the NEXT batch (a device tensor that stays unchanged until that
        batch has been trained): after this batch's push+update the rows AND the de-duplication plan of the next
        batch are pulled on a side stream, next to the dense all-reduce / optimizer of this step -- the prefetch of
        the reference's ``pulling`` (exb.py:645-691; parked pulls, EmbeddingPullOperator.cpp:117-145: a pull of batch
        k+1 may only see the tables after update k, which the stream order guarantees). ``pulled=True``: the caller
        passes the batch that the previous step prefetched this way: X32 and the plan are ready, no pull up front."""
        B, L, lib, st = self.B, len(self.hidden), self.lib, self._st()
        assert ids.shape == (B, self.nf) and ids.dtype == torch.int64 and ids.is_contiguous()
        if self._grad_dirty:          # the optimizer kernel clears the gradients it consumed; a call with
            self.gtheta.zero_()       # update=False leaves them behind
            self._grad_dirty = False
        self._mark("start")
        g = self.group
        v2 = getattr(g, "v2", False) and update
        if pulled:
            if v2:
                g._armed[0] = (g._key(ids), "pull")    # rows + plan of this batch came with the previous step's tail
        elif v2:
            g.pull(ids, out=self.X32, train=True)      # gather + plan of the batch in one launch
        else:
            g.pull(ids, out=self.X32)
        self._mark("pull")
        tn = self.mn_major
        self._forward(ids, dense, st, self.loss.data_ptr(), self.opt_step.data_ptr() if update else 0)
        dims = [self.K0p] + self.Hp
        row_head = tn and self.Hp[-1] <= 512       # merged row-wise head; cachegrad then owns the cached linear grads
        ha = _HeadArgs(self.H[-1].data_ptr(), self.Hp[-1], self.Hp[-1] - 1, self.view("wout").data_ptr(),
                       self.base.data_ptr(), labels.data_ptr(), self.dlogit.data_ptr(), self.loss.data_ptr(),
                       self.dZ[-1].data_ptr(), 0 if tn else self.dZT[-1].data_ptr(), self.gview("wout").data_ptr(),
                       self.gview("wd").data_ptr(), self.gview("bias").data_ptr(), dense.data_ptr(), self.nd,
                       self.G32.data_ptr(), self.XS, self.lin0, self.ns, ids.data_ptr(), self.nf,
                       self.cache_col.data_ptr(), self.cache_off.data_ptr(), self.nc,
                       0 if row_head else self.gview("cache_lin").data_ptr(), B, 1.0 / B)
        _ck(lib.exb_head(ctypes.byref(ha), B, st), "head")
        self._mark("head")
        if self.use_chain:
            self.bwd_chain.launch(st)          # dX and dW of every layer: one persistent launch
        else:
            for l in range(L - 1, 0, -1):      # dZ_{l-1} = (dZ_l @ W_l) * relu'(H_{l-1})
                G.gemm_nt(self.dZ[l], self.WTb[l], B, self.Hp[l - 1], self.Hp[l], self.dZ[l - 1], mode=G.EPI_DX,
                          ones_col=self.Hp[l - 1] - 1, outT=None if tn else self.dZT[l - 1], mask=self.H[l - 1], stream=st)
            G.gemm_nt(self.dZ[0], self.WTb[0], B, self.K0p, self.Hp[0], self.G32, mode=G.EPI_DX_FM, dlogit=self.dlogit,
                      S=self.S, emb=self.X32, fm_cols=self.nf * self.Dp if self.use_fm else 0, D=self.Dp, stream=st)
        self._mark("dx_gemm")
        if self.cin:
            self._cin_backward(st)
            self._mark("cin_bwd")
        if self.dcn:
            self._cross_backward(st, dense)
            self._mark("cross_bwd")
        if self.autoint:
            self._att_backward(st)
            self._mark("att_bwd")
        forked = update and self.overlap
        if forked:
            cur = torch.cuda.current_stream(self.dev)
            self._ev_fork.record(cur)
            with torch.cuda.stream(self._s2):
                self._s2.wait_event(self._ev_fork)
                self.group.push_update(ids, self.G32)
                self._ev_join.record(self._s2)
        for l in range(L if not self.use_chain else 0):                 # dW_l = dZ_l^T @ H_{l-1}
            prevT = self.A0T if l == 0 else self.HT[l - 1]
            gW = self.gview("W%d" % l).view(self.Hp[l], dims[l])
            if tn:
                G.gemm_tn(self.dZ[l], self.A0 if l == 0 else self.H[l - 1], self.Hp[l], dims[l], B, gW,
                          splits=self.dw_splits, stream=st)
                continue
            G.gemm_nt(self.dZT[l], prevT, self.Hp[l], dims[l], B, gW, mode=G.EPI_DW, splits=self.dw_splits, stream=st)
        def cachegrad():
            _ck(lib.exb_cachegrad(self.G32.data_ptr(), self.XS, self.ns * self.Dp, self.Dp, ids.data_ptr(), self.nf,
                                  self.cache_col.data_ptr(), self.cache_off.data_ptr(), self.nc,
                                  self.gview("cache_emb").data_ptr(), B, self.dlogit.data_ptr(),
                                  self.gview("cache_lin").data_ptr() if row_head else 0,
                                  self.cache_vocab.data_ptr(), st), "cachegrad")
        tail = update and next_ids is not None and not forked
        # one GPU: the gradients of the replicated tables are only needed by the dense optimizer, so their kernel moves
        # behind push+update, next to the tail pull (several GPUs: the push kernel all-reduces them, they come first)
        late_cg = bool(self.nc) and tail and self._ar is None and self.late_cachegrad
        if self.nc and not late_cg:
            cachegrad()
        self._mark("dw_gemm+cachegrad")
        if update:
            if not forked:
                self.group.push_update(ids, self.G32)
                self._mark("push_update")
            if tail:      # next batch: rows into X32 (free since the dX1 GEMM) + plan, beside the dense optimizer
                cur = torch.cuda.current_stream(self.dev)
                self._ev_fork.record(cur)
                self._s2.wait_event(self._ev_fork)
                with torch.cuda.stream(self._s2):
                    g.pull(next_ids, out=self.X32, train=v2)
                    self._ev_plan.record(self._s2)
            # Adagrad + bf16 weight refresh + gradient clearing: one kernel (world > 1: behind the all-reduce,
            # in the same kernel)
            # world > 1: the all-reduce runs on one CTA per SM (every CTA polls peer flags); the optimizer kernel
            # is chained behind it with a programmatic dependent launch instead of sharing its grid
            if self._ar is not None and not self._rider:
                self._ar()
                self._mark("allreduce")
            if late_cg:
                cachegrad()
            _ck(lib.exb_dense_opt(ctypes.byref(self._opt_args), st), "dense_opt")
            self._mark("optimizer")
            if forked:
                torch.cuda.current_stream(self.dev).wait_event(self._ev_join)
                self._mark("join(push_update)")
            if tail:
                torch.cuda.current_stream(self.dev).wait_event(self._ev_plan)
                self._mark("join(prefetch pull)")
        else:
            self._grad_dirty = True
        return self.loss.view(())

    def warmup(self, ids, dense, labels):
        """Launch every kernel of a training step once WITHOUT changing a parameter: forward + backward of the batch
        with the gradients discarded, the planned pull and push+update of a zero-row batch (all phases and barriers,
        no row; world > 1: the ride-along all-reduce sums zero gradients), the dense optimizer on a snapshot that is
        restored afterwards. Used before a CUDA-graph capture -- lazy kernel loading and allocator growth may not
        happen inside one. Collective when world > 1."""
        lib, st = self.lib, self._st()
        keep = [t.clone() for t in (self.theta, self.accum, self.accum2, self.opt_step)]
        self.forward_backward(ids, dense, labels, update=False)
        g = self.group
        none_ids, none_g = ids[:0], self.G32[:0]
        if getattr(g, "v2", False):
            g.pull(none_ids, out=self.X32, train=True)
        self.gtheta.zero_()
        g.push_update(none_ids, none_g)
        if self._ar is not None and not self._rider:
            self._ar()
        _ck(lib.exb_dense_opt(ctypes.byref(self._opt_args), st), "dense_opt")
        for t, k in zip((self.theta, self.accum, self.accum2, self.opt_step), keep):
            t.copy_(k)
        self.gtheta.zero_()
        self._grad_dirty = False
        self.refresh_weights()

    def kernels_per_step(self):
        """launches of our own kernels in one training step"""
        L = len(self.hidden)
        prep = 1 if (self.mn_major and 128 % self.Dp == 0) else 2
        head = 1 if (self.mn_major and self.Hp[-1] <= 512) else 2
        gemms = (1 if self.chain_fwd else L) + (1 if self.use_chain else 2 * L)   # persistent chains: fwd, bwd
        n = 1 + prep + gemms + head + (1 if self.nc else 0) + 1 + 1      # pull prep GEMMs head cache push optimizer
        # CIN: gather + pool + fold, per layer outer + GEMM forward, dY + dZ GEMM + outer_bwd + filter-gradient GEMM
        n += 3 + 6 * len(self.cin_layers) if self.cin else 0
        # DCN-v2: per layer GEMM + cross forward; backward top, per layer P GEMM + weight-gradient GEMM + cross backward
        n += 1 + 5 * self.cross_layers if self.dcn else 0
        # AutoInt: gather + fold, per layer projection GEMM + attention forward, attention backward + two GEMMs
        n += 2 + 5 * self.att_layers if self.autoint else 0
        return n + (1 if self._ar is not None and not self._rider else 0)

    # ---- dense state, checkpoints and export (all through ``self.layout``)
    def config(self):
        """the configuration a checkpoint records; ``CONFIG_KEYS`` must match on load"""
        return {"model": self.model, "vocab": list(self.vocab), "cached": list(self.cached), "embedding_dim": self.D,
                "num_dense": self.nd, "hidden": list(self.hidden), "cin_layers": list(self.cin_layers),
                "cin_split_half": self.cin_split_half if self.cin else None, "cross_layers": self.cross_layers,
                "pack_linear": self.pack_linear, "batch": self.B, "world": self.ctx.world,
                "dense_optimizer": self.dense_opt["category"], "att_layers": self.att_layers or None,
                "att_embedding_size": self.att_d if self.autoint else None,
                "att_head_num": self.att_h if self.autoint else None,
                "att_res": self.att_res if self.autoint else None}

    def config_mismatches(self, config):
        """one line per configuration entry in which ``config`` differs from this model's"""
        mine = self.config()
        return ["%s: checkpoint %r, model %r" % (k, config.get(k), mine[k]) for k in CONFIG_KEYS if config.get(k) != mine[k]]

    def dense_state_dict(self, include_optimizer=True):
        """The dense parameters as fp32 CPU tensors under ``layout``'s logical names. ``include_optimizer``: plus the
        dense optimizer's state slots ("<category>.<slot>/<name>", ``DENSE_OPT_SLOTS``) and its step counter
        ("opt_step"). Reads the buffers after every step launched so far on the current stream."""
        sd = self.layout.gather(self.theta.cpu())
        if include_optimizer:
            cat = self.dense_opt["category"]
            for slot, buf in zip(DENSE_OPT_SLOTS[cat], (self.accum, self.accum2)):
                for name, t in self.layout.gather(buf.cpu()).items():
                    sd["%s.%s/%s" % (cat, slot, name)] = t
            sd["opt_step"] = self.opt_step.cpu()
        return sd

    def _dense_buffers(self, sd, config=None):
        """(theta, accum, accum2, opt_step) on the CPU from a dense state dict: every slot outside the layout at its
        construction value, the optimizer state fresh unless ``sd`` holds all of this model's dense-optimizer slots.
        Raises ValueError (nothing changed yet) on a configuration or parameter mismatch."""
        errs = self.config_mismatches(config) if config is not None else []
        for name, (shape, _) in self.layout.params.items():
            t = sd.get(name)
            if t is None:
                errs.append("%s: missing" % name)
            elif tuple(t.shape) != tuple(shape):
                errs.append("%s: checkpoint shape %s, model %s" % (name, tuple(t.shape), tuple(shape)))
        if errs:
            raise ValueError("the checkpoint does not fit this FusedCTR:\n  " + "\n  ".join(errs))
        f32, n = torch.float32, self.n_theta
        theta = torch.zeros(n, dtype=f32)
        self.layout.scatter(theta, sd)
        accum = torch.full((n,), self._acc0, dtype=f32)
        accum2 = torch.zeros(self.accum2.numel(), dtype=f32)
        step = torch.zeros(1, dtype=torch.int32)
        # a checkpoint without optimizer state, or of another category: the weights load, the state starts fresh
        # (as the sparse tables do, checkpoint.load_model); the hyper-parameters are always the model's own
        cat = self.dense_opt["category"]
        slots = DENSE_OPT_SLOTS[cat]
        if "opt_step" in sd and all("%s.%s/%s" % (cat, s, p) in sd for s in slots for p in self.layout.params):
            for s, buf in zip(slots, (accum, accum2)):
                self.layout.scatter(buf, {p: sd["%s.%s/%s" % (cat, s, p)] for p in self.layout.params})
            step.copy_(sd["opt_step"].reshape(1))
        return theta, accum, accum2, step

    def _set_dense(self, bufs):
        """copy (theta, accum, accum2, opt_step) IN PLACE (captured graphs hold these addresses), clear the
        gradients, refresh the bf16 weight copies"""
        for dst, src in zip((self.theta, self.accum, self.accum2, self.opt_step), bufs):
            dst.copy_(src)
        self.gtheta.zero_()
        self._grad_dirty = False
        self.refresh_weights()

    def load_dense_state_dict(self, sd, config=None):
        """Load ``dense_state_dict`` output in place (``config``: a checkpoint's ``config()``, checked first). Slots
        outside the layout (padding) return to their construction values; the gradients are cleared. A different
        batch size or world size is fine."""
        self._set_dense(self._dense_buffers(sd, config))

    def save(self, path, include_optimizer=True):
        """Collective checkpoint into the directory ``path`` (a local path): ``model.pt`` (rank 0, ``torch.save`` of
        {"format", "config", "dense": dense_state_dict}) and the sparse tables under ``openembedding/`` in the
        server-model format (``checkpoint.save_model``). Holds the state after every step launched so far; changes
        nothing, so a prefetched next batch stays valid. The dense state is replicated: every rank holds the same."""
        ctx = self.ctx
        torch.cuda.synchronize(self.dev)
        if ctx.rank == 0:
            os.makedirs(path, exist_ok=True)
            torch.save({"format": CHECKPOINT_FORMAT, "config": self.config(),
                        "dense": self.dense_state_dict(include_optimizer)}, os.path.join(path, "model.pt"))
            if os.path.exists(os.path.join(path, "openembedding")):
                shutil.rmtree(os.path.join(path, "openembedding"))
        ctx.barrier()
        from .. import checkpoint
        checkpoint.save_model(ctx, os.path.join(path, "openembedding"), include_optimizer=include_optimizer)

    def load(self, path):
        """Collective: restore a ``save`` checkpoint -- the tables (rows, hash slots, optimizer states) and the dense
        state, in place. The configuration must match (ValueError naming each difference, model untouched); batch
        and world size may differ. A checkpoint without dense-optimizer state, or of another optimizer category,
        loads the weights and starts that state fresh. Rows or plans prefetched before the load are stale:
        ``load_generation`` advances and ``FusedTrainer.step`` pulls up front again."""
        blob = torch.load(os.path.join(path, "model.pt"), map_location="cpu", weights_only=True)
        if not isinstance(blob, dict) or blob.get("format") != CHECKPOINT_FORMAT:
            raise ValueError("%s is not a FusedCTR checkpoint" % os.path.join(path, "model.pt"))
        bufs = self._dense_buffers(blob["dense"], blob["config"])
        torch.cuda.synchronize(self.dev)
        from .. import checkpoint
        checkpoint.load_model(self.ctx, os.path.join(path, "openembedding"))
        self._set_dense(bufs)
        self.load_generation += 1
        torch.cuda.synchronize(self.dev)

    def to_original(self):
        """The model as a ``models.ctr.StandaloneCTR`` on the CPU: every table row pulled through the engine
        (collective), the dense weights through ``layout``, ``dnn_out.bias`` folded into ``bias``."""
        from .ctr import StandaloneCTR
        if any(self.vocab[f] <= 0 for f in self.server):
            raise ValueError("can not convert sparse variable to nn.Embedding.")
        mod = StandaloneCTR(self.vocab, num_dense=self.nd, embedding_dim=self.D, model=self.model, hidden=self.hidden,
                            cached=self.cached, cin_layers=self.cin_layers or (128, 128),
                            cin_split_half=self.cin_split_half, cross_layers=self.cross_layers or 3,
                            **(dict(att_layers=self.att_layers, att_embedding_size=self.att_d, att_head_num=self.att_h,
                                    att_res=self.att_res) if self.autoint else {}))
        sd = self.dense_state_dict(include_optimizer=False)
        sd["bias"] = sd["bias"] + sd.pop("dnn_out.bias")
        missing, unexpected = mod.load_state_dict(sd, strict=False)
        assert not unexpected and all(k.startswith(("emb.", "lin.", "cache_cols", "cache_offsets")) for k in missing), \
            (missing, unexpected)
        ns, D = self.ns, self.D
        metas = self.sparse.metas
        with torch.no_grad():
            for j, f in enumerate(self.server):
                if self.pack_linear:
                    rows = self._pull_table(metas[j], self.vocab[f])
                    mod.emb[j].weight.copy_(rows[:, :D])
                    mod.lin[j].weight.copy_(rows[:, D:])
                else:
                    mod.emb[j].weight.copy_(self._pull_table(metas[j], self.vocab[f]))
                    mod.lin[j].weight.copy_(self._pull_table(metas[ns + j], self.vocab[f]))
        return mod

    def _pull_table(self, meta, vocab):
        """all rows of a table (CPU fp32 [vocab, dim]), pulled in blocks (collective)"""
        out = torch.empty(vocab, meta.dim, dtype=torch.float32)
        blk = 2 ** 20 // meta.dim + 1
        for i in range(0, vocab, blk):
            idx = torch.arange(i, min(vocab, i + blk), device=self.dev)
            out[i:i + idx.numel()] = self.ctx.backend.pull(meta, idx).cpu()
        return out

    def save_as_original_model(self, path):
        """Collective export of a stand-alone ``models.ctr.StandaloneCTR`` (fp32, no engine, no GPU) to the file
        ``path``: every rank pulls, rank 0 writes ``torch.save(module)``. Returns the module (CPU). A hash-table
        feature (vocab <= 0) cannot become an ``nn.Embedding``: ValueError."""
        mod = self.to_original()
        if self.ctx.rank == 0:
            os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
            torch.save(mod.cpu(), path)
        self.ctx.barrier()
        return mod

    # ---- fp32 torch reference of the dense math on the current X32 (tests)
    def reference(self, ids, dense, labels, return_logits=False):
        """returns (loss, grads dict) computed with torch autograd in fp32 from the same
        parameters and the same pulled embeddings (self.X32 after a forward); ``return_logits``: (loss, grads,
        logits [B])."""
        B, nf, Dp, L = self.B, self.nf, self.Dp, len(self.hidden)
        theta = self.theta.detach().clone().requires_grad_(True)
        X = self.X32.detach().clone()
        emb = X[:, :nf * Dp].clone()
        if self.nc:
            ce = theta[self.segs["cache_emb"][0]:self.segs["cache_emb"][0] + self.cache_rows * Dp].view(-1, Dp)
            cid = ids[:, self.cache_col.long()] + self.cache_off
            emb = torch.cat([emb[:, :self.ns * Dp], ce[cid].reshape(B, -1)], dim=1)
        emb = emb.detach().requires_grad_(True) if not self.nc else emb
        emb_leaf = X[:, :self.ns * Dp].clone().requires_grad_(True)
        if self.nc:
            emb = torch.cat([emb_leaf, ce[cid].reshape(B, -1)], dim=1)
        else:
            emb = emb_leaf
        lin_leaf = X[:, self.lin0:self.lin0 + self.ns].clone().requires_grad_(True)
        lin = lin_leaf.sum(1)
        if self.nc:
            cl = theta[self.segs["cache_lin"][0]:self.segs["cache_lin"][0] + self.cache_rows]
            lin = lin + cl[cid].sum(1)
        wd = theta[self.segs["wd"][0]:self.segs["wd"][0] + self.nd]
        bias = theta[self.segs["bias"][0]]
        z = lin + dense @ wd + bias
        if self.use_fm:
            e = emb.view(B, nf, Dp)
            s = e.sum(1)
            z = z + 0.5 * (s * s - (e * e).sum(1)).sum(1)
        ones = torch.ones(B, 1, device=self.dev)
        dims = [self.K0p] + self.Hp
        pad0 = self.K0p - 1 - nf * Dp - self.nd
        h = torch.cat([emb, dense, torch.zeros(B, pad0, device=self.dev), ones], dim=1)
        for l in range(L):
            o, n = self.segs["W%d" % l]
            W = theta[o:o + n].view(self.Hp[l], dims[l])
            h = torch.relu(h.to(torch.bfloat16).float() @ W.to(torch.bfloat16).float().t())
            h = torch.cat([h[:, :-1], ones], dim=1)
        o, n = self.segs["wout"]
        z = z + h.to(torch.bfloat16).float() @ theta[o:o + n]
        if self.cin:
            z = z + self._reference_cin(emb.view(B, nf, Dp)[:, :, :self.D], theta)
        if self.dcn:
            z = z + self._reference_cross(torch.cat([emb.view(B, nf, Dp)[:, :, :self.D].reshape(B, -1), dense], 1), theta)
        if self.autoint:
            z = z + self._reference_att(emb.view(B, nf, Dp)[:, :, :self.D], theta)
        loss =torch.nn.functional.binary_cross_entropy_with_logits(z, labels)
        loss.backward()
        grads = {"theta": theta.grad, "emb": emb_leaf.grad, "lin": lin_leaf.grad}
        if return_logits:
            return loss.detach(), grads, z.detach()
        return loss.detach(), grads

    def _reference_cin(self, x, theta):
        """CIN(x) . w_cin for ``reference``: the eager zoo's ``models.ctr.CIN`` (plain torch) run on the filters in
        ``theta``, rounded to bf16 where the kernels round -- Z and W on the way into a layer, Y on the way out (the
        gradients of Z and Y then arrive rounded too, like the kernels' bf16 dZ and dY). x: [B, nf, D] fp32."""
        from .ctr import CIN
        bf16 = torch.bfloat16
        if getattr(self, "_ref_cin", None) is None:
            cin = CIN(self.nf, tuple(self.cin_layers), split_half=self.cin_split_half, tc=False).to(self.dev)
            for conv in cin.convs:
                conv.register_forward_pre_hook(lambda mod, args: (args[0].to(bf16).float(),))
                conv.register_forward_hook(lambda mod, args, out: out.to(bf16).float())
            self._ref_cin = cin
        params = {}
        for k, n in enumerate(self.cin_layers):
            o, sz = self.segs["C%d" % k]
            W = theta[o:o + sz].view(self.cin_Np[k], self.cin_Kp[k])
            W = W + (W.to(bf16).float() - W).detach()          # bf16 value, fp32 gradient (the kernels' gW)
            C = self.cin_H[k] * self.nf
            params["convs.%d.weight" % k] = W[:n, :C].contiguous().unsqueeze(-1)
            params["convs.%d.bias" % k] = W[:n, C].contiguous()
        p = torch.func.functional_call(self._ref_cin, params, (x,))
        o, n = self.segs["wcin"]
        return p @ theta[o:o + n]

    def _reference_cross(self, x, theta):
        """CrossNetV2(x) . w_cross for ``reference``: the eager zoo's ``models.ctr.CrossNetV2`` (plain torch) run on the
        cross matrices in ``theta``, rounded to bf16 where the kernels round -- x_l and W_l (bias included) on the way
        into a layer's GEMM with an fp32 gradient passed straight through, and the gradient of U_l (the kernels' bf16
        dU). U_l itself stays fp32. x: [B, nf*D + nd] fp32."""
        from .ctr import CrossNetV2
        bf16 = torch.bfloat16
        st = lambda t: t + (t.to(bf16).float() - t).detach()        # bf16 value, fp32 gradient

        def round_grad(mod, args, out):
            out.register_hook(lambda g: g.to(bf16).float())

        if getattr(self, "_ref_cross", None) is None:
            net = CrossNetV2(self.cross_n, self.cross_layers, tc=False).to(self.dev)
            for lin in net.w:
                lin.register_forward_pre_hook(lambda mod, args: (st(args[0]),))
                lin.register_forward_hook(round_grad)
            self._ref_cross = net
        cols, ones = self.cross_real, self.K0p - 1
        params = {}
        for l in range(self.cross_layers):
            o, sz = self.segs["X%d" % l]
            W = st(theta[o:o + sz].view(self.K0p, self.K0p))
            params["w.%d.weight" % l] = W[cols[:, None], cols[None, :]]
            params["w.%d.bias" % l] = W[cols, ones]
        xL = torch.func.functional_call(self._ref_cross, params, (x,))
        o, n = self.segs["wcross"]
        return xL @ theta[o:o + n][cols]


    def _reference_att(self, x, theta):
        """flatten(AutoInt(x)) . w_att for ``reference``: the eager zoo's ``InteractingLayer.attend`` (plain torch, fp32)
        on the projections of the stacked weights in ``theta``, rounded to bf16 where the kernels round -- X_l and T_l
        on the way into the projection GEMM with an fp32 gradient passed straight through, and the gradient of the
        projections (the kernels' bf16 [dQ | dK | dV | dR]). The projections themselves stay fp32. x: [B, nf, D]."""
        from .ctr import InteractingLayer
        bf16 = torch.bfloat16
        st = lambda t: t + (t.to(bf16).float() - t).detach()        # bf16 value, fp32 gradient
        dh = self.att_dh
        for l in range(self.att_layers):
            o, sz = self.segs["T%d" % l]
            T = st(theta[o:o + sz].view(self.att_Kp[l], self.att_Np))[:x.shape[-1]]
            proj = st(x) @ T
            proj.register_hook(lambda g: g.to(bf16).float())
            q, k, v = proj[..., :dh], proj[..., dh:2 * dh], proj[..., 2 * dh:3 * dh]
            x = InteractingLayer.attend(q, k, v, proj[..., 3 * dh:4 * dh] if self.att_res else None, self.att_h)
        o, n = self.segs["watt"]
        return x.reshape(x.shape[0], -1) @ theta[o:o + n]


class FusedTrainer:
    """CUDA-graph driver for ``FusedCTR`` with the same interface as ``models.trainer.Trainer``.

    ``step(ids, dense, labels, next_ids=...)``: with ``next_ids`` (the device ids of the batch that will be passed
    as ``ids`` to the NEXT call) the de-duplication plan of the next batch is built inside this step on a side
    stream -- the prefetch of the reference's ``pulling`` (exb.py:645-691).

    Before the first capture every kernel of the step is launched eagerly twice through ``FusedCTR.warmup`` (lazy
    kernel loading and allocator growth may not happen inside a capture); the warm-up changes no parameter, so the
    graph-driven trajectory is the eager one from the first step on.

    ``predict(ids, dense)`` / ``evaluate(ids, dense, labels, metrics)``: the forward-only pass over n <= B rows,
    replayed from one more graph (key ``"eval"``); an evaluation drops a prefetched next batch, whose step then
    pulls up front."""

    supports_prefetch = True
    want_prefetch = True         # ``make_pipeline`` runs one batch ahead: the next batch's pull overlaps this step's tail
    supports_stable_inputs = True
    MAX_STABLE_GRAPHS = 64

    def __init__(self, model, use_graph=True):
        self.m, self.ctx = model, model.ctx
        self.device, self.world = model.dev, model.ctx.world
        self.use_graph = use_graph
        self._graphs, self._static = {}, None      # (pull up front?, prefetch pull at the tail?[, input addresses]) -> CUDAGraph
        self._stable = {}                          # stable-input graph key -> the caller's tensors (kept alive)
        self.graph = None
        self._ar = model._ar
        self._x32_key = None         # key of the batch whose rows + plan the last step prefetched into X32
        self._load_gen = model.load_generation     # a model ``load`` since the prefetch makes it stale
        self._warm = False
        self._eval = None            # static eval inputs (ids, dense, labels, n on the device) of predict / evaluate

    def step(self, ids, dense, labels, next_ids=None, stable=False):
        """``stable=True``: the caller keeps the four input tensors alive at fixed addresses and refills them in place
        (an input pipeline's device buffers, a resident pool of batches). In the steady state (this batch was
        prefetched, the next one is announced) the graph is then captured directly on those tensors -- one graph per
        distinct (ids, dense, labels, next_ids) address tuple, at most MAX_STABLE_GRAPHS -- instead of copying the
        inputs into the trainer's own static buffers first (four device copies per step)."""
        g = self.m.group
        v2 = getattr(g, "v2", False)
        self._drop_stale_prefetch()
        pulled = self._x32_key is not None and self._x32_key == g._key(ids)
        tail = next_ids is not None
        if not self.use_graph:
            if v2 and not pulled and self._x32_key is not None:
                g.reset_slot(0)                     # a prefetched batch that is not the one trained now
            loss = self.m.forward_backward(ids, dense, labels, next_ids=next_ids, pulled=pulled)
            self._x32_key = g._key(next_ids) if tail else None
            self.ctx.step_done()
            return loss
        if self._static is None:
            self._static = {"ids": ids.clone(), "dense": dense.clone(), "labels": labels.clone(), "next_ids": ids.clone()}
        s = self._static
        key = (not pulled, tail)
        if stable and pulled and tail and self._warm:
            skey = key + (ids.data_ptr(), dense.data_ptr(), labels.data_ptr(), next_ids.data_ptr())
            if skey in self._graphs or len(self._stable) < self.MAX_STABLE_GRAPHS:
                key = skey
                s = self._stable.setdefault(skey, {"ids": ids, "dense": dense, "labels": labels, "next_ids": next_ids})
        if s is self._static:
            if ids.data_ptr() != s["ids"].data_ptr():
                s["ids"].copy_(ids, non_blocking=True)
                s["dense"].copy_(dense, non_blocking=True)
                s["labels"].copy_(labels, non_blocking=True)
            if tail:
                s["next_ids"].copy_(next_ids, non_blocking=True)
        if v2 and not pulled and self._x32_key is not None:
            g.reset_slot(0)                         # drop the prefetched plan: this is a different batch
        gr = self._graphs.get(key)
        if gr is None:
            gr = self._capture(key, s)
        gr.replay()
        # replays bypass the plan's python bookkeeping: if a batch was prefetched the current slot is armed on the
        # device under a key no tensor can match -- any eager use of the plan re-plans
        if v2:
            g._armed = [(("graph", id(self)), "pull") if tail else None, None]
        self._x32_key = g._key(next_ids) if tail else None
        self.graph = gr
        self.ctx.step_done()
        return self._static["loss"]

    def _drop_stale_prefetch(self):
        """after a ``FusedCTR.load`` the prefetched rows (and, v2, the plan: hash-slot positions) describe tables
        that are gone: the next step pulls and plans up front"""
        if self._load_gen == self.m.load_generation:
            return
        if self._x32_key is not None and getattr(self.m.group, "v2", False):
            self.m.group.reset_slot(0)
        self._x32_key = None
        self._load_gen = self.m.load_generation

    def _capture(self, key, s):
        head, tail = key[:2]
        g = self.m.group
        if not self._warm:          # allocator / lazy init warm-up, outside any capture
            assert head, "the first step of a trainer always pulls up front"
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):
                for _ in range(2):      # every kernel of the step runs, no parameter changes (FusedCTR.warmup)
                    self.m.warmup(s["ids"], s["dense"], s["labels"])
            torch.cuda.current_stream(self.device).wait_stream(side)
            torch.cuda.synchronize(self.device)
            if self.world > 1:
                self.ctx.barrier()
            self._warm = True
        torch.cuda.synchronize(self.device)
        saved = list(getattr(g, "_armed", [None, None]))
        if getattr(g, "v2", False):
            g._armed = [None, None]
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            loss = self.m.forward_backward(s["ids"], s["dense"], s["labels"], next_ids=s["next_ids"] if tail else None,
                                           pulled=not head)
        self._static["loss"] = loss          # the model's own loss buffer: the same tensor in every variant
        if getattr(g, "v2", False):
            g._armed = saved            # capture only recorded launches: the device-side slots are untouched
        self._graphs[key] = gr
        return gr

    # ---- evaluation: forward-only pass on the trainer's static, zero-padded eval buffers
    def _eval_forward(self, ids, dense, labels=None):
        """copy n <= B rows into the eval buffers (rows >= n zero), set n on the device, run the forward-only pass
        (graph replay, or eagerly); returns n"""
        m = self.m
        n = ids.shape[0]
        if not (1 <= n <= m.B) or ids.shape[1] != m.nf or dense.shape != (n, m.nd):
            raise ValueError("evaluation takes 1 .. %d rows of ids [n, %d] and dense [n, %d]" % (m.B, m.nf, m.nd))
        if labels is not None and labels.numel() != n:
            raise ValueError("%d labels for %d rows" % (labels.numel(), n))
        e = self._eval
        if e is None:
            dev = self.device
            e = self._eval = {"ids": torch.zeros(m.B, m.nf, dtype=torch.int64, device=dev),
                              "dense": torch.zeros(m.B, m.nd, dtype=torch.float32, device=dev),
                              "labels": torch.zeros(m.B, dtype=torch.float32, device=dev),
                              "n": torch.zeros(1, dtype=torch.int32, device=dev)}
        for name, src in (("ids", ids), ("dense", dense), ("labels", labels)):
            if src is None:
                continue
            e[name][:n].copy_(src.reshape(e[name][:n].shape), non_blocking=True)
            e[name][n:].zero_()
        e["n"].fill_(n)
        # the forward overwrites X32: rows (and, v2, the plan) a step prefetched for the next batch are dropped the
        # way ``step`` drops a prefetch that is not followed, and that step pulls up front again
        if self._x32_key is not None:
            if getattr(m.group, "v2", False):
                m.group.reset_slot(0)
            self._x32_key = None
        if not self.use_graph:
            m.predict_forward(e["ids"], e["dense"])
            return n
        gr = self._graphs.get("eval")
        if gr is None:
            torch.cuda.synchronize(self.device)
            m.predict_forward(e["ids"], e["dense"])    # side-effect free: one eager run loads every kernel
            torch.cuda.synchronize(self.device)
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                m.predict_forward(e["ids"], e["dense"])
            self._graphs["eval"] = gr
        gr.replay()
        return n

    def predict(self, ids, dense):
        """probabilities of n <= B rows (device ids [n, nf] int64, dense [n, nd] fp32) as a new fp32 tensor [n]"""
        n = self._eval_forward(ids, dense)
        return self.m.probs[:n].clone()

    def evaluate(self, ids, dense, labels, metrics):
        """forward-only pass over n <= B rows, accumulated into ``metrics`` (``models.metrics.BinaryMetrics``)"""
        self._eval_forward(ids, dense, labels)
        metrics.update(self.m.logits, self._eval["labels"], n=self._eval["n"])

    def make_pipeline(self, batch, num_sparse, num_dense):
        from .trainer import _Pipeline
        return _Pipeline(self, batch, num_sparse, num_dense)
