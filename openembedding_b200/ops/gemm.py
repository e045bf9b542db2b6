"""Python face of the hand-written wgmma GEMM (``csrc/cuda/gemm_wgmma.cu``).

``gemm_nt(A, B, ...)`` computes ``A[M,K] @ B[N,K].T`` on bf16 operands with one of the
fused epilogues. Operands must be K-padded to a multiple of 64 and have leading
dimensions that are multiples of 8 elements (the dense engine allocates them that way).

Outputs are stored by TMA in whole 16-byte units of a row: when an output row (or a row of ``outT``) is not a
multiple of 16 bytes wide, the elements up to the next 16-byte boundary, inside the row stride, are overwritten too.
``splits > 1`` is for EPI_DW only (split-K partial sums are reduce-added); other epilogues refuse it.
"""
import ctypes
from ctypes import c_int, c_longlong, c_uint64

import torch

from .. import _native

EPI_FWD, EPI_DX, EPI_DW, EPI_DX_FM = 0, 1, 2, 3
_proto_done = False


def _lib():
    global _proto_done
    lib = _native.cuda()
    if not _proto_done:
        lib.exb_gemm_bf16_nt.restype = c_int
        lib.exb_gemm_bf16_nt.argtypes = [c_uint64, c_longlong, c_uint64, c_longlong, c_int, c_int, c_int, c_int, c_int,
                                         c_int, c_uint64, c_longlong, c_uint64, c_longlong, c_uint64, c_longlong,
                                         c_uint64, c_uint64, c_uint64, c_longlong, c_int, c_int, c_int, c_uint64,
                                         c_uint64]
        lib.exb_gemm_bf16_tn.restype = c_int
        lib.exb_gemm_bf16_tn.argtypes = [c_uint64, c_longlong, c_uint64, c_longlong, c_int, c_int, c_int, c_uint64,
                                         c_longlong, c_int, c_uint64]
        lib.exb_gemm_last_error.restype = ctypes.c_char_p
        lib.exb_gemm_timeouts.restype = c_int
        lib.exb_chain_desc_size.restype = c_int
        lib.exb_chain_create.restype = ctypes.c_void_p
        lib.exb_chain_create.argtypes = [ctypes.c_void_p, c_int, c_int]
        lib.exb_chain_destroy.argtypes = [ctypes.c_void_p]
        lib.exb_chain_launch.restype = c_int
        lib.exb_chain_launch.argtypes = [ctypes.c_void_p, c_uint64]
        lib.exb_chain_status.restype = c_int
        lib.exb_chain_status.argtypes = [ctypes.c_void_p]
        lib.exb_chain_info.argtypes = [ctypes.c_void_p, ctypes.POINTER(c_int)]
        _proto_done = True
    return lib


def check():
    """Synchronise the device and raise if a GEMM kernel launched since the last check gave up waiting on its
    shared-memory pipeline (its output is then wrong)."""
    n = _lib().exb_gemm_timeouts()
    if n != 0:
        raise RuntimeError("GEMM pipeline: %s" % ("%d barrier waits timed out" % n if n > 0 else "status unreadable"))


def _p(t):
    return t.data_ptr() if t is not None else 0


class ChainDesc(ctypes.Structure):
    """one GEMM of a persistent chain (csrc/cuda/gemm_wgmma.cu: struct ChainDesc)"""
    _fields_ = [("tn", c_int), ("M", c_int), ("N", c_int), ("K", c_int),
                ("A", c_uint64), ("B", c_uint64), ("out", c_uint64),
                ("lda", c_longlong), ("ldb", c_longlong), ("ldo", c_longlong),
                ("mode", c_int), ("relu", c_int), ("ones_col", c_int), ("fm_cols", c_int), ("D", c_int), ("splits", c_int),
                ("mask", c_uint64), ("ldmask", c_longlong),
                ("dlogit", c_uint64), ("S", c_uint64), ("emb", c_uint64), ("ldemb", c_longlong),
                ("dep", c_int), ("dep_kind", c_int)]


def chain_nt(A, B, M, N, K, out, mode=EPI_FWD, relu=False, ones_col=-1, mask=None, dlogit=None, S=None, emb=None,
             fm_cols=0, D=1, dep=-1):
    d = ChainDesc()
    d.tn, d.M, d.N, d.K = 0, M, N, K
    d.A, d.B, d.out = A.data_ptr(), B.data_ptr(), out.data_ptr()
    d.lda, d.ldb, d.ldo = A.stride(0), B.stride(0), out.stride(0)
    d.mode, d.relu, d.ones_col, d.fm_cols, d.D, d.splits = mode, int(relu), ones_col, fm_cols, D, 1
    d.mask, d.ldmask = _p(mask), (mask.stride(0) if mask is not None else 0)
    d.dlogit, d.S, d.emb, d.ldemb = _p(dlogit), _p(S), _p(emb), (emb.stride(0) if emb is not None else 0)
    d.dep, d.dep_kind = dep, (1 if dep >= 0 else 0)
    return d


def chain_tn(A, B, M, N, K, out, splits=8, dep=-1):
    """out[M, N] (fp32) += A[K, M]^T B[K, N]; dep: GEMM of the chain producing A (its rows = this GEMM's K range)"""
    d = ChainDesc()
    d.tn, d.M, d.N, d.K = 1, M, N, K
    d.A, d.B, d.out = A.data_ptr(), B.data_ptr(), out.data_ptr()
    d.lda, d.ldb, d.ldo = A.stride(0), B.stride(0), out.stride(0)
    d.mode, d.ones_col, d.D, d.splits = EPI_DW, -1, 1, splits
    d.dep, d.dep_kind = dep, (2 if dep >= 0 else 0)
    return d


class GemmChain:
    """Several dependent GEMMs in ONE persistent launch (``exb_gemm_chain_kernel``): tensor maps encoded once,
    tiles of all GEMMs in one static work list, dependencies tracked per 128-row block on the device."""

    def __init__(self, descs, device):
        lib = _lib()
        assert lib.exb_chain_desc_size() == ctypes.sizeof(ChainDesc), "ChainDesc ABI mismatch"
        arr = (ChainDesc * len(descs))(*descs)
        sms = torch.cuda.get_device_properties(device).multi_processor_count
        self.lib, self.device = lib, device
        self.h = lib.exb_chain_create(ctypes.byref(arr), len(descs), sms)
        if not self.h:
            raise RuntimeError("exb_chain_create: " + lib.exb_gemm_last_error().decode())
        out = (c_int * 3)()
        lib.exb_chain_info(self.h, out)
        self.items, self.grid, self.smem = int(out[0]), int(out[1]), int(out[2])

    def launch(self, stream=None):
        st = stream if stream is not None else torch.cuda.current_stream(self.device).cuda_stream
        if self.lib.exb_chain_launch(self.h, st) != 0:
            raise RuntimeError("exb_chain_launch: " + self.lib.exb_gemm_last_error().decode())

    def check(self):
        code = self.lib.exb_chain_status(self.h)
        if code:
            raise RuntimeError("GEMM chain error %d (GEMM %d timed out waiting for its producer)" % (code, code - 100))
        check()

    def close(self):
        if self.h:
            self.lib.exb_chain_destroy(self.h)
            self.h = None


def gemm_nt(A, B, M, N, K, out, mode=EPI_FWD, relu=False, ones_col=-1, outT=None, mask=None, dlogit=None, S=None,
            emb=None, fm_cols=0, D=1, splits=1, stream=None, dbg=None):
    """A: [>=M, lda] bf16 view, B: [>=N, ldb] bf16 view (both row-major, K contiguous)."""
    lib = _lib()
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    assert A.stride(-1) == 1 and B.stride(-1) == 1
    st = stream if stream is not None else torch.cuda.current_stream(A.device).cuda_stream
    rc = lib.exb_gemm_bf16_nt(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), M, N, K, mode, int(relu), ones_col,
                              out.data_ptr(), out.stride(0), _p(outT), outT.stride(0) if outT is not None else 0,
                              _p(mask), mask.stride(0) if mask is not None else 0, _p(dlogit), _p(S), _p(emb),
                              emb.stride(0) if emb is not None else 0, fm_cols, D, splits, st, _p(dbg))
    if rc != 0:
        raise RuntimeError("exb_gemm_bf16_nt: " + lib.exb_gemm_last_error().decode())
    return out


def gemm_tn(A, B, M, N, K, out, splits=1, stream=None):
    """out[M, N] (fp32) += A[K, M].T @ B[K, N] with A, B row-major bf16 (K rows): the weight-gradient
    product straight from batch-major activations -- both operands are fed to the tensor core as
    MN-major tiles, so no transposed copies have to be materialised. ``out`` must be zeroed (or
    hold the value to accumulate onto); split-K partial sums arrive by TMA reduce-add."""
    lib = _lib()
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16 and out.dtype == torch.float32
    assert A.stride(-1) == 1 and B.stride(-1) == 1
    st = stream if stream is not None else torch.cuda.current_stream(A.device).cuda_stream
    rc = lib.exb_gemm_bf16_tn(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), M, N, K, out.data_ptr(),
                              out.stride(0), splits, st)
    if rc != 0:
        raise RuntimeError("exb_gemm_bf16_tn: " + lib.exb_gemm_last_error().decode())
    return out
