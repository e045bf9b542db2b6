"""The wgmma GEMM (csrc/cuda/gemm_wgmma.cu) against the float64 reference of its contract (tests/gemm_reference.py),
on every launch path: single launches at the default 64-wide tile, the automatically chosen 128-wide tile, split-K,
the persistent chain, and (in subprocesses, their switches are read once per process) the forced 128-wide tile,
the swapped launch order and the A-tile multicast.

Every case runs in two operand families:
  * exact: small integers, every output must equal the reference bit for bit after one round-to-nearest-even;
  * real: bf16 normals, within the derived bound; the largest error / bound ratio per path is reported.
Every output lives inside a NaN-sentinel canvas (rows below, columns to the right): nothing outside the contract
region may change, and no input may change. EXB_GEMM_EXACT_REPORT=<file> appends the ratios there as JSON.
"""
import json
import os
import re
import subprocess
import sys

import pytest
import torch

import gemm_reference as R

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
FAMILIES = ("exact", "real")
RATIOS = {}
HERE = os.path.dirname(os.path.abspath(__file__))


def _path():
    """the launch path the process runs single launches on (the variant switches are read once per process)"""
    if os.environ.get("EXB_GEMM_BN") == "128":
        return "bn128_forced"
    if os.environ.get("EXB_GEMM_SWAP", "0") not in ("", "0"):
        return "swap"
    mc = os.environ.get("EXB_GEMM_MC", "0")
    if mc not in ("", "0", "1"):
        return "mc" + mc
    return "bn64"


def _note(path, family, ratio):
    if family == "real":
        RATIOS[path] = max(RATIOS.get(path, 0.0), ratio)


@pytest.fixture(autouse=True)
def _no_pipeline_timeouts():
    """every GEMM launched by a test must have completed its shared-memory pipeline"""
    yield
    from openembedding_b200.ops.gemm import check
    check()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest real-family error / bound ratio per path:", json.dumps(RATIOS, sort_keys=True))
    f = os.environ.get("EXB_GEMM_EXACT_REPORT")
    if f:
        with open(f, "a") as fh:
            fh.write(json.dumps(RATIOS, sort_keys=True) + "\n")


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _vals(shape, family, g, scale=1.0):
    return R.ints(shape, R.EXACT_LIM, g, "cuda") if family == "exact" else R.normals(shape, g, "cuda", scale)


def _in(values, dtype=BF16, extra_cols=8, align=None):
    """an input operand inside a sentinel canvas"""
    c = R.Canvas(values.shape[0], values.shape[1], dtype, "cuda", extra_cols=extra_cols, align=align)
    return c.set(values)


def _fm_operands(M, fm_cols, D, family, g):
    """dlogit [M], S [M, D] (contiguous, no row padding) and emb [M, fm_cols] (fp32), each inside a canvas"""
    if family == "exact":
        dl, S, e = R.ints((1, M), 4, g, "cuda", -2), R.ints((M, D), 8, g, "cuda", -2), R.ints((M, fm_cols), 8, g, "cuda", -2)
    else:
        dl, S, e = (torch.randn(s, generator=g, device="cuda").to(F64) for s in ((1, M), (M, D), (M, fm_cols)))
    return _in(dl, F32), _in(S, F32, extra_cols=0, align=1), _in(e, F32, extra_cols=4)


def _check(family, got, v, c, bound, what):
    if family == "exact":
        R.check_exact(got, v, c, what)
        return 0.0
    return R.check_bound(got, v, bound, c, what)


def run_nt(case, mode, family, seed, path=None):
    """one gemm_nt launch of `case` (a dict of gemm_reference's case lists) with epilogue `mode`, checked against
    the float64 reference; returns the real family's largest error / bound ratio"""
    from openembedding_b200.ops import gemm as G
    path = path or _path()
    M, N, K = case["M"], case["N"], case["K"]
    Np = R.ceil64(N)
    what = "%s %s mode %d M=%d N=%d K=%d" % (path, family, mode, M, N, K)
    g = _gen(seed)
    A = _in(_vals((M, K), family, g), extra_cols=case.get("lda_extra", 0) or 8)
    B = _in(_vals((N, K), family, g, scale=K ** -0.5))
    ins = [A, B]
    kw = {}
    f32 = mode in (R.EPI_DW, R.EPI_DX_FM)
    if mode == R.EPI_DX:
        mask = _in(_vals((M, N), family, g))
        mask.buf[:M, N:] = 2.0                     # columns past N hold positive values: not part of the mask
        kw["mask"] = mask.view
        ins.append(mask)
    fm_cols, D = (case.get("fm_cols", 0), case.get("D", 2)) if mode == R.EPI_DX_FM else (0, 1)
    if fm_cols:
        dl, S, emb = _fm_operands(M, fm_cols, D, family, g)
        kw.update(dlogit=dl.view[0], S=S.view, emb=emb.view)
        ins += [dl, S, emb]
    out = R.Canvas(M, N if f32 else Np, F32 if f32 else BF16, "cuda", extra_cols=8 + case.get("ldo_extra", 0))
    init = None
    if mode == R.EPI_DW:
        init = _vals((M, N), family, g)
        out.set(init)
    outT = R.Canvas(Np, M, BF16, "cuda") if case.get("outT") and not f32 else None
    ones = case.get("ones_col", -1) if mode in (R.EPI_FWD, R.EPI_DX) else -1
    for c in ins + [out] + ([outT] if outT else []):
        c.snapshot()
    G.gemm_nt(A.view, B.view, M, N, K, out.view, mode=mode, relu=bool(case.get("relu", True)), ones_col=ones,
              outT=outT.view if outT else None, fm_cols=fm_cols, D=D, splits=case.get("splits", 1), **kw)
    torch.cuda.synchronize()
    for c, name in zip(ins, ("A", "B", "mask" if mode == R.EPI_DX else "dlogit", "S", "emb")):
        c.check_unchanged(what + " input " + name)
    out.check_untouched(M, N if f32 else Np, what + " out")
    v, c, absp = R.ref_nt(A.view, B.view, M, N, K, mode, relu=bool(case.get("relu", True)), ones_col=ones,
                          mask=kw.get("mask"), dl=kw.get("dlogit"), S=kw.get("S"), emb=kw.get("emb"), fm_cols=fm_cols,
                          D=D, init=init)
    if family == "exact":
        assert float(absp.max()) + R.EXACT_LIM < R.EXACT_BUDGET, what
    bound = None
    if family == "real":
        ab = torch.zeros_like(v)
        ab[:, :N] = absp
        extra = None
        if fm_cols:
            n = torch.arange(fm_cols, device="cuda")
            fa = kw["dlogit"].to(F64).abs()[:, None] * (kw["S"].to(F64).abs()[:, n % D] + kw["emb"].to(F64).abs())
            extra = torch.zeros_like(v)
            extra[:, :fm_cols] = 4 * R.U32 * fa
            extra = extra + R.U32 * v.abs()
        bound = R.real_bound(ab, K, v, bf16_out=not f32, splits=case.get("splits", 1), init=init, extra=extra)
    r = _check(family, out.view, v, c, bound, what)
    if outT:
        outT.check_untouched(Np, M, what + " outT")
        r = max(r, _check(family, outT.view, R.transposed(v, M), R.transposed(c, M),
                          None if bound is None else R.transposed(bound, M), what + " outT"))
    _note(path, family, r)
    return r


def run_tn(case, family, seed, path=None):
    """gemm_tn: out[M, N] += A[K, M]^T B[K, N] with split-K reduce-add onto a non-zero initial out"""
    from openembedding_b200.ops import gemm as G
    path = path or _path()
    M, N, K, s = case["M"], case["N"], case["K"], case["splits"]
    what = "%s %s tn M=%d N=%d K=%d splits=%d" % (path, family, M, N, K, s)
    g = _gen(seed)
    A, B = _in(_vals((K, M), family, g)), _in(_vals((K, N), family, g, scale=K ** -0.5))
    init = _vals((M, N), family, g)
    out = R.Canvas(M, N, F32, "cuda").set(init)
    for c in (A, B, out):
        c.snapshot()
    G.gemm_tn(A.view, B.view, M, N, K, out.view, splits=s)
    torch.cuda.synchronize()
    A.check_unchanged(what + " A")
    B.check_unchanged(what + " B")
    out.check_untouched(M, N, what + " out")
    v, absp = R.ref_tn(A.view, B.view, M, N, K, init)
    bound = R.real_bound(absp, K, v, False, splits=s, init=init) if family == "real" else None
    r = _check(family, out.view, v, torch.zeros_like(v, dtype=torch.bool), bound, what)
    _note(path, family, r)
    return r


# ---------------------------------------------------------------------------------------------- single launches

@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("mode", [R.EPI_FWD, R.EPI_DX, R.EPI_DX_FM])
def test_single_launch(mode, family):
    """pairwise cover of M x N x K at the default tile (BN = 64 below the 128-wide threshold), strided A and out"""
    for i, case in enumerate(R.single_cases()):
        if mode == R.EPI_FWD:
            case = dict(case, relu=i % 5 != 0)
        run_nt(case, mode, family, seed=1000 * mode + i)


@pytest.mark.parametrize("family", FAMILIES)
def test_split_k(family):
    """uneven split-K ranges, splits > and == the number of k-blocks, onto a non-zero initial out, M and N tails"""
    for i, case in enumerate(R.split_cases()):
        run_tn(case, family, seed=2000 + i)
        run_nt(dict(case), R.EPI_DW, family, seed=3000 + i)


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in p.events() if "exb_gemm" in e.name]


@pytest.mark.parametrize("family", FAMILIES)
def test_auto_wide_tile(family):
    """pick_bn's 128-wide tile, chosen in-process: the xDeepFM CIN GEMM shape and the M = 8192 threshold"""
    for i, case in enumerate(R.AUTO128_CASES):
        names = _kernel_names(lambda: run_nt(dict(case, relu=True), R.EPI_FWD, family, seed=4000 + i, path="bn128_auto"))
        assert any("exb_gemm_wgmma_kernel<128>" in n for n in names), names
    # one row block less: the default tile
    names = _kernel_names(lambda: run_nt(dict(M=8064, N=512, K=64, relu=True), R.EPI_FWD, family, seed=4100))
    assert any("exb_gemm_wgmma_kernel<64>" in n for n in names), names


@pytest.mark.parametrize("family", FAMILIES)
def test_dx_fm_d_and_fm_cols(family):
    """the FM term at every even D (66, 68 wrap mid-tile, 130 is wider than a tile) and three fm_cols positions,
    single launch and one-GEMM chain; fm_cols = 0 is the plain fp32 store DCN uses"""
    i = 0
    for D in R.FM_D:
        for fm_cols in R.FM_COLS:
            case = dict(M=R.FM_M, N=R.FM_N, K=R.FM_K, fm_cols=fm_cols, D=D)
            run_nt(case, R.EPI_DX_FM, family, seed=5000 + i)
            run_chain_single_fm(case, family, seed=5500 + i)
            i += 1
    run_nt(dict(M=R.FM_M, N=R.FM_N, K=R.FM_K, fm_cols=0), R.EPI_DX_FM, family, seed=5999)


@pytest.mark.parametrize("family", FAMILIES)
def test_dx_mask_edge_values(family):
    """the relu mask at +0, -0, NaN, the smallest positive bf16 (subnormal), negatives and positives; columns past N
    hold positive values and must not count"""
    from openembedding_b200.ops import gemm as G
    M, N, K = 300, 129, 192
    g = _gen(6000)
    A, B = _in(_vals((M, K), family, g)), _in(_vals((N, K), family, g, scale=K ** -0.5))
    edge = torch.tensor([0.0, -0.0, float("nan"), 2.0 ** -133, -2.0 ** -133, 1.0, -1.0, float("inf"), -float("inf")],
                        dtype=F64, device="cuda")
    pick = torch.randint(0, edge.numel(), (M, N), generator=g, device="cuda")
    mask = R.Canvas(M, N, BF16, "cuda")
    mask.buf[:M, :N] = edge[pick].to(BF16)
    mask.buf[:M, N:] = 2.0 ** -133
    assert int(mask.view.view(torch.int16)[pick == 3].unique().numel()) == 1 and int(mask.view.view(torch.int16)[pick == 3][0]) == 1
    assert bool((mask.view.view(torch.int16)[pick == 1] == -32768).all())       # -0 kept its sign
    out, outT = R.Canvas(M, R.ceil64(N), BF16, "cuda"), R.Canvas(R.ceil64(N), M, BF16, "cuda")
    for c in (A, B, mask, out, outT):
        c.snapshot()
    G.gemm_nt(A.view, B.view, M, N, K, out.view, mode=G.EPI_DX, ones_col=7, outT=outT.view, mask=mask.view)
    torch.cuda.synchronize()
    for c in (A, B, mask):
        c.check_unchanged("dx edge input")
    out.check_untouched(M, R.ceil64(N), "dx edge out")
    outT.check_untouched(R.ceil64(N), M, "dx edge outT")
    v, c, absp = R.ref_nt(A.view, B.view, M, N, K, R.EPI_DX, ones_col=7, mask=mask.view)
    kept = ~c[:, :N]
    off_ones = torch.ones_like(kept)
    off_ones[:, 7] = False                         # the ones column is zeroed whatever its mask
    assert bool(kept[((pick == 3) | (pick == 5) | (pick == 7)) & off_ones].all())
    assert not bool(kept[(pick <= 2) | (pick == 4) | (pick == 6) | (pick == 8)].any())
    bound = None
    if family == "real":
        ab = torch.zeros_like(v)
        ab[:, :N] = absp
        bound = R.real_bound(ab, K, v, True)
    r = _check(family, out.view, v, c, bound, "dx edge")
    r = max(r, _check(family, outT.view, R.transposed(v, M), R.transposed(c, M),
                      None if bound is None else R.transposed(bound, M), "dx edge outT"))
    _note(_path(), family, r)


def test_argument_errors_raise():
    """arguments the kernel cannot honour are refused before anything is launched"""
    from openembedding_b200.ops import gemm as G
    M, N, K = 128, 64, 128
    A = torch.ones(M, K + 8, device="cuda", dtype=BF16)
    B = torch.ones(N, K, device="cuda", dtype=BF16)
    out = torch.full((M + 1, N + 4), 7.0, device="cuda", dtype=F32)
    outb = torch.full((M, N + 8), 7.0, device="cuda", dtype=BF16)
    flat = torch.full((M * (N + 8) + 64,), 7.0, device="cuda", dtype=F32)
    flatb = torch.full((M * (N + 8) + 64,), 7.0, device="cuda", dtype=BF16)
    before = (out.clone(), outb.clone(), flat.clone(), flatb.clone())
    shape, tma, split = "K %% 64 / ld %% 8 violated", "cuTensorMapEncodeTiled failed", "splits > 1 needs EPI_DW"
    bad = [
        (shape, dict(K=100)),                                                   # K not a multiple of 64
        (shape, dict(A=torch.ones(M, K + 4, device="cuda", dtype=BF16)[:, :K])),   # lda % 8 != 0
        (shape, dict(B=torch.ones(N, K + 2, device="cuda", dtype=BF16)[:, :K])),   # ldb % 8 != 0
        (tma, dict(out=flat[1:1 + M * (N + 4)].view(M, N + 4)[:, :N], mode=G.EPI_DW)),     # fp32 out base at 4 bytes
        (tma, dict(out=flat[:M * (N + 1)].view(M, N + 1)[:, :N], mode=G.EPI_DW)),         # fp32 row stride 65 * 4 bytes
        (tma, dict(out=flatb[4:4 + M * (N + 8)].view(M, N + 8)[:, :N])),                 # bf16 out base at 8 bytes
        (tma, dict(out=flatb[:M * (N + 4)].view(M, N + 4)[:, :N])),                      # bf16 row stride 136 bytes
        (tma, dict(outT=torch.zeros(N, M + 4, device="cuda", dtype=BF16)[:, :M - 4])),   # outT row stride 264 bytes
        (split, dict(splits=2)),                                                # split-K onto a plain store
        (split, dict(splits=4, mode=G.EPI_DX, mask=outb)),
        (split, dict(splits=2, mode=G.EPI_DX_FM, out=out[:M, :N])),
    ]
    for msg, b in bad:
        kw = dict(A=A[:, :K], B=B, M=M, N=N, K=K, out=outb[:, :N], mode=G.EPI_FWD)
        kw.update(b)
        with pytest.raises(RuntimeError, match=re.escape(msg)):
            G.gemm_nt(kw.pop("A"), kw.pop("B"), kw.pop("M"), kw.pop("N"), kw.pop("K"), kw.pop("out"), **kw)
    with pytest.raises(RuntimeError, match=re.escape("gemm_tn: " + shape)):
        G.gemm_tn(A[:, :K], B, K, N, 96, out[:K, :N])                        # K % 64
    with pytest.raises(RuntimeError, match=re.escape("gemm_tn: " + shape)):    # lda % 8
        G.gemm_tn(torch.ones(K, M + 4, device="cuda", dtype=BF16)[:, :M], B.t().contiguous(), M, N, K, out[:M, :N])
    torch.cuda.synchronize()
    for t, b in zip((out, outb, flat, flatb), before):
        assert torch.equal(t, b)


# ---------------------------------------------------------------------------------------------- chains

def run_chain_single_fm(case, family, seed):
    """EPI_DX_FM as a one-GEMM persistent chain"""
    from openembedding_b200.ops import gemm as G
    M, N, K, fm_cols, D = case["M"], case["N"], case["K"], case["fm_cols"], case["D"]
    what = "chain %s dX_FM M=%d N=%d K=%d fm_cols=%d D=%d" % (family, M, N, K, fm_cols, D)
    g = _gen(seed)
    A, B = _in(_vals((M, K), family, g)), _in(_vals((N, K), family, g, scale=K ** -0.5))
    dl, S, emb = _fm_operands(M, fm_cols, D, family, g)
    out = R.Canvas(M, N, F32, "cuda")
    ins = [A, B, dl, S, emb]
    for c in ins + [out]:
        c.snapshot()
    ch = G.GemmChain([G.chain_nt(A.view, B.view, M, N, K, out.view, mode=G.EPI_DX_FM, dlogit=dl.view[0], S=S.view,
                                 emb=emb.view, fm_cols=fm_cols, D=D)], torch.device("cuda"))
    try:
        ch.launch()
        ch.check()
    finally:
        ch.close()
    for c in ins:
        c.check_unchanged(what + " input")
    out.check_untouched(M, N, what)
    v, c, absp = R.ref_nt(A.view, B.view, M, N, K, R.EPI_DX_FM, dl=dl.view[0], S=S.view, emb=emb.view,
                          fm_cols=fm_cols, D=D)
    bound = None
    if family == "real":
        n = torch.arange(fm_cols, device="cuda")
        fa = torch.zeros_like(v)
        fa[:, :fm_cols] = dl.view[0].to(F64).abs()[:, None] * (S.view.to(F64).abs()[:, n % D] + emb.view.to(F64).abs())
        bound = R.real_bound(absp, K, v, False, extra=4 * R.U32 * fa + R.U32 * v.abs())
    _note("chain", family, _check(family, out.view, v, c, bound, what))


class ChainRun:
    """a forward chain (fwd1 -> ... -> fwdL) and a backward chain (dX / dW of every layer, the dependency structure
    of FusedCTR's step) on canvases, each GEMM checked directly against the float64 reference"""

    def __init__(self, M, widths, family, seed, splits, fm_cols=R.CHAIN_FM_COLS, D=R.CHAIN_FM_D):
        from openembedding_b200.ops import gemm as G
        self.G, self.M, self.w, self.family, self.splits = G, M, widths, family, splits
        self.fm_cols, self.D = fm_cols, D
        L = self.L = len(widths) - 1
        g = _gen(seed)
        ops = R.chain_operands(M, widths, g, "cuda", fm_cols=fm_cols, D=D)
        if family == "real":
            for l in range(L):
                for key in ("W", "WT"):
                    t = ops[key][l]
                    ops[key][l] = R.normals(t.shape, g, "cuda", scale=t.shape[1] ** -0.5)
            for key, wdt in (("A0", widths[0]), ("dtop", widths[L])):
                ops[key][:M, :wdt] = R.normals((M, wdt), g, "cuda")
            ops["fm"] = {k: torch.randn(v.shape, generator=g, device="cuda").to(F64) for k, v in ops["fm"].items()}
        p, Kb = self.p, self.Kb = ops["p"], ops["Kb"]
        self.A0 = _in(ops["A0"])
        self.W = [_in(t) for t in ops["W"]]
        self.WT = [_in(t) for t in ops["WT"]]
        self.dl, self.S, self.emb = (_in(ops["fm"]["dl"][None], F32), _in(ops["fm"]["S"], F32, extra_cols=0, align=1),
                                     _in(ops["fm"]["emb"], F32, extra_cols=4))

        def act(cols):   # rows [M, Kb) are zero: the dW GEMMs read Kb batch rows
            c = R.Canvas(Kb, cols, BF16, "cuda")
            c.buf[M:Kb, :cols] = 0
            return c
        self.H = [act(p[l + 1]) for l in range(L)]
        self.dZ = [act(p[l + 1]) for l in range(L)]
        self.dZ[L - 1].set(ops["dtop"])
        self.G32 = R.Canvas(M, widths[0], F32, "cuda")
        self.gW = [R.Canvas(widths[l + 1], p[l], F32, "cuda") for l in range(L)]
        dev = torch.device("cuda")
        fd, src = [], self.A0
        for l in range(L):
            fd.append(G.chain_nt(src.view[:, :p[l]], self.W[l].view, M, widths[l + 1], p[l], self.H[l].view, mode=G.EPI_FWD,
                                 relu=True, ones_col=widths[l + 1] - 1, dep=l - 1))
            src = self.H[l]
        bd, prod = [], -1
        for l in range(L - 1, -1, -1):
            if l > 0:
                bd.append(G.chain_nt(self.dZ[l].view, self.WT[l].view, M, widths[l], p[l + 1], self.dZ[l - 1].view,
                                     mode=G.EPI_DX, ones_col=widths[l] - 1, mask=self.H[l - 1].view[:, :widths[l]], dep=prod))
            else:
                bd.append(G.chain_nt(self.dZ[0].view, self.WT[0].view, M, widths[0], p[1], self.G32.view, mode=G.EPI_DX_FM,
                                     dlogit=self.dl.view[0], S=self.S.view, emb=self.emb.view, fm_cols=fm_cols, D=D,
                                     dep=prod))
            nxt = len(bd) - 1
            srcl = self.A0 if l == 0 else self.H[l - 1]
            bd.append(G.chain_tn(self.dZ[l].view[:, :widths[l + 1]], srcl.view[:, :p[l]], widths[l + 1], p[l], Kb,
                                 self.gW[l].view, splits=splits, dep=prod))
            prod = nxt
        self.fwd = G.GemmChain(fd, dev)
        self.nbwd = len(bd)
        self.bwd = G.GemmChain(bd, dev)
        self.zero_grads()
        self.ins = [self.A0, self.dl, self.S, self.emb] + self.W + self.WT

    def close(self):
        self.fwd.close()
        self.bwd.close()

    def refresh(self, seed):
        """new chain inputs written in place, every intermediate the chains read (H, dZ below the top, G32) refilled
        with the NaN sentinel, dW outputs zeroed: a tile that reads its producer's row block before it is written
        then gives NaN or a stale value, never the right answer"""
        M, w, L = self.M, self.w, self.L
        g = _gen(seed)
        def vals(shape):    # the distribution of chain_operands
            return R.ints(shape, 4, g, "cuda") if self.family == "exact" else R.normals(shape, g, "cuda")
        self.A0.view[:M, :w[0]] = vals((M, w[0])).to(BF16)
        self.dZ[L - 1].view[:M, :w[L]] = vals((M, w[L])).to(BF16)
        for c in self.H + self.dZ[:L - 1] + [self.G32]:
            c.buf.view(R.INT_VIEW[c.buf.dtype]).fill_(R.SENTINEL[c.buf.dtype])
            c.buf[M:self.Kb, :c.view.shape[1]] = 0
        self.zero_grads()

    def launch(self, which=("fwd", "bwd")):
        for c in self.ins + self.H + self.dZ + [self.G32] + self.gW:
            c.snapshot()
        for name in which:
            ch = getattr(self, name)
            ch.launch()
            ch.check()
        torch.cuda.synchronize()
        for c in self.ins:
            c.check_unchanged("chain input")
        self.dZ[self.L - 1].check_unchanged("chain dZ top")

    def check(self, bwd=True, tag="chain"):
        M, w, p, Kb, L, fam = self.M, self.w, self.p, self.Kb, self.L, self.family
        r = 0.0
        src = self.A0
        for l in range(L):
            what = "%s %s M=%d fwd%d" % (tag, fam, M, l + 1)
            self.H[l].check_untouched(M, p[l + 1], what)
            v, c, absp = R.ref_nt(src.view, self.W[l].view, M, w[l + 1], p[l], R.EPI_FWD, relu=True, ones_col=w[l + 1] - 1)
            r = max(r, self._cmp(self.H[l].view[:M], v, c, absp, p[l], True, what))
            src = self.H[l]
        if not bwd:
            return r
        for l in range(L - 1, -1, -1):
            what = "%s %s M=%d dX%d" % (tag, fam, M, l + 1)
            if l > 0:
                self.dZ[l - 1].check_untouched(M, p[l], what)
                v, c, absp = R.ref_nt(self.dZ[l].view, self.WT[l].view, M, w[l], p[l + 1], R.EPI_DX, ones_col=w[l] - 1,
                                      mask=self.H[l - 1].view)
                r = max(r, self._cmp(self.dZ[l - 1].view[:M], v, c, absp, p[l + 1], True, what))
            else:
                self.G32.check_untouched(M, w[0], what)
                v, c, absp = R.ref_nt(self.dZ[0].view, self.WT[0].view, M, w[0], p[1], R.EPI_DX_FM, dl=self.dl.view[0],
                                      S=self.S.view, emb=self.emb.view, fm_cols=self.fm_cols, D=self.D)
                extra = None
                if fam == "real":
                    n = torch.arange(self.fm_cols, device="cuda")
                    extra = torch.zeros_like(v)
                    extra[:, :self.fm_cols] = 4 * R.U32 * self.dl.view[0, :M].to(F64).abs()[:, None] * (
                        self.S.view[:M].to(F64).abs()[:, n % self.D] + self.emb.view[:M].to(F64).abs())
                    extra += R.U32 * v.abs()
                r = max(r, self._cmp(self.G32.view, v, c, absp, p[1], False, what, extra=extra))
            what = "%s %s M=%d dW%d" % (tag, fam, M, l + 1)
            self.gW[l].check_untouched(w[l + 1], p[l], what)
            srcl = self.A0 if l == 0 else self.H[l - 1]
            zero = torch.zeros(w[l + 1], p[l], dtype=F64, device="cuda")
            v, absp = R.ref_tn(self.dZ[l].view, srcl.view, w[l + 1], p[l], Kb, zero)
            if fam == "exact":
                assert float(absp.max()) < R.EXACT_BUDGET, what
            r = max(r, self._cmp(self.gW[l].view, v, torch.zeros_like(v, dtype=torch.bool), absp, Kb, False, what,
                                 splits=self.splits))
        return r

    def _cmp(self, got, v, c, absp, K, bf16, what, extra=None, splits=1):
        if self.family == "exact":
            assert float(absp.max()) < R.EXACT_BUDGET, what
            R.check_exact(got, v, c, what)
            return 0.0
        ab = torch.zeros_like(v)
        ab[:, :absp.shape[1]] = absp
        return R.check_bound(got, v, R.real_bound(ab, K, v, bf16, splits=splits, extra=extra), c, what)

    def zero_grads(self):
        for c in self.gW:
            c.view.zero_()


def _dw_splits(M):
    # M = 4096: 64 k-blocks in 5 splits of 13, so split-K ranges straddle 128-row blocks
    return {4096: 5, 300: 3}.get(M, 8)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("M", R.CHAIN_M)
def test_chain_forward_backward(M, family):
    """every GEMM of a 3-layer forward chain and of its backward chain (row-block and K-range dependencies) against
    the reference; M = 8320 and 16384 have more row blocks than a fixed table of 64 would hold"""
    run = ChainRun(M, R.CHAIN_W, family, seed=7000 + M, splits=_dw_splits(M))
    try:
        run.launch()
        _note("chain", family, run.check())
    finally:
        run.close()


@pytest.mark.parametrize("family", FAMILIES)
def test_chain_eight_gemms(family):
    """a 4-layer backward chain is 8 GEMMs, the most a chain takes"""
    run = ChainRun(4096, R.CHAIN_W8, family, seed=7100, splits=8)
    try:
        assert run.nbwd == 8
        run.launch()
        _note("chain", family, run.check())
    finally:
        run.close()


@pytest.mark.parametrize("family", FAMILIES)
def test_chain_mixed_k(family):
    """independent GEMMs of K = 4096 and K = 64 in one chain: persistent CTAs run tiles of both lengths back to back,
    so the ring phases and the epilogue staging hand-off carry across very different tiles"""
    from openembedding_b200.ops import gemm as G
    g = _gen(7200)
    specs = [(2048, 448, 4096, G.EPI_FWD), (4096, 448, 64, G.EPI_DX), (2048, 320, 4096, G.EPI_DX_FM),
             (4096, 1728, 64, G.EPI_FWD), (448, 448, 4096, G.EPI_DW)]
    descs, checks, keep = [], [], []
    for i, (M, N, K, mode) in enumerate(specs):
        if mode == G.EPI_DW:
            A, B = _in(_vals((K, M), family, g)), _in(_vals((K, N), family, g, scale=K ** -0.5))
            out = R.Canvas(M, N, F32, "cuda").set(torch.zeros(M, N, dtype=F64, device="cuda"))
            descs.append(G.chain_tn(A.view, B.view, M, N, K, out.view, splits=5))
            checks.append((mode, M, N, K, A, B, out, {}))
            keep += [A, B, out]
            continue
        A, B = _in(_vals((M, K), family, g)), _in(_vals((N, K), family, g, scale=K ** -0.5))
        kw = {}
        if mode == G.EPI_DX:
            kw["mask"] = _in(_vals((M, N), family, g))
        if mode == G.EPI_DX_FM:
            dl, S, emb = _fm_operands(M, 208, 66, family, g)
            kw.update(dl=dl, S=S, emb=emb)
        f32 = mode == G.EPI_DX_FM
        out = R.Canvas(M, N if f32 else R.ceil64(N), F32 if f32 else BF16, "cuda")
        ckw = dict(mask=kw["mask"].view) if "mask" in kw else {}
        if f32:
            ckw = dict(dlogit=kw["dl"].view[0], S=kw["S"].view, emb=kw["emb"].view, fm_cols=208, D=66)
        descs.append(G.chain_nt(A.view, B.view, M, N, K, out.view, mode=mode, relu=True, ones_col=N - 1, **ckw))
        checks.append((mode, M, N, K, A, B, out, ckw))
        keep += [A, B, out] + list(kw.values())
    for c in keep:
        c.snapshot()
    ch = G.GemmChain(descs, torch.device("cuda"))
    try:
        assert ch.items > 2 * ch.grid, (ch.items, ch.grid)     # CTAs take several tiles of different K
        ch.launch()
        ch.check()
    finally:
        ch.close()
    r = 0.0
    for mode, M, N, K, A, B, out, ckw in checks:
        what = "mixed-K chain %s mode %d M=%d N=%d K=%d" % (family, mode, M, N, K)
        A.check_unchanged(what)
        B.check_unchanged(what)
        if mode == G.EPI_DW:
            out.check_untouched(M, N, what)
            v, absp = R.ref_tn(A.view, B.view, M, N, K, torch.zeros(M, N, dtype=F64, device="cuda"))
            bound = R.real_bound(absp, K, v, False, splits=5) if family == "real" else None
            r = max(r, _check(family, out.view, v, torch.zeros_like(v, dtype=torch.bool), bound, what))
            continue
        f32 = mode == G.EPI_DX_FM
        out.check_untouched(M, N if f32 else R.ceil64(N), what)
        v, c, absp = R.ref_nt(A.view, B.view, M, N, K, mode, relu=True, ones_col=N - 1, mask=ckw.get("mask"),
                              dl=ckw.get("dlogit"), S=ckw.get("S"), emb=ckw.get("emb"), fm_cols=ckw.get("fm_cols", 0),
                              D=ckw.get("D", 1))
        bound = None
        if family == "real":
            ab = torch.zeros_like(v)
            ab[:, :N] = absp
            extra = None
            if f32:
                n = torch.arange(208, device="cuda")
                extra = torch.zeros_like(v)
                extra[:, :208] = 4 * R.U32 * ckw["dlogit"].to(F64).abs()[:, None] * (
                    ckw["S"].to(F64).abs()[:, n % 66] + ckw["emb"].to(F64).abs())
                extra += R.U32 * v.abs()
            bound = R.real_bound(ab, K, v, not f32, extra=extra)
        r = max(r, _check(family, out.view, v, c, bound, what))
    _note("chain", family, r)


def test_chain_relaunch_and_alternate():
    """the same chains launched again and again, each launch checked against the reference. Before every launch the
    inputs change in place and every intermediate the chains read is refilled with the NaN sentinel, so a tile that
    read its producer's row block too early -- a dependency counter left over from an earlier launch lets its wait
    pass at once -- would show as NaN or a stale value. The last CTA of a launch zeroes the counters for the next one;
    the third launch of a chain is the first that depends on a clean-up done by a launch after the first. Then two
    chains of different sizes (separate counters) alternate."""
    a = ChainRun(4096, R.CHAIN_W, "exact", seed=7300, splits=5)
    b = ChainRun(8320, R.CHAIN_W, "exact", seed=7301, splits=8)
    try:
        for k in range(4):
            a.refresh(7310 + k)
            a.launch()
            a.check(tag="relaunch %d" % k)
        for k in range(3):
            for i, run in enumerate((b, a)):
                run.refresh(7320 + 2 * k + i)
                run.launch()
                run.check(tag="alternate %d" % k)
    finally:
        a.close()
        b.close()


def test_chain_refuses_bad_structure():
    from openembedding_b200.ops import gemm as G
    A = torch.zeros(128, 64, device="cuda", dtype=BF16)
    out = torch.zeros(128, 64, device="cuda", dtype=BF16)
    d = [G.chain_nt(A, A, 128, 64, 64, out) for _ in range(9)]
    with pytest.raises(RuntimeError, match="1..8 GEMMs"):
        G.GemmChain(d, torch.device("cuda"))
    d = [G.chain_nt(A, A, 128, 64, 64, out, dep=1), G.chain_nt(A, A, 128, 64, 64, out)]
    with pytest.raises(RuntimeError, match="only depend on an earlier one"):
        G.GemmChain(d, torch.device("cuda"))
    # dependencies on row blocks the producer does not write: a dW whose K range (256 batch rows) runs past a
    # 128-row producer, and a 256-row GEMM waiting on the row blocks of a 128-row one
    A2 = torch.zeros(256, 64, device="cuda", dtype=BF16)
    out2 = torch.zeros(256, 64, device="cuda", dtype=BF16)
    gw = torch.zeros(64, 64, device="cuda", dtype=F32)
    for second in (G.chain_tn(A2, A2, 64, 64, 256, gw, splits=2, dep=0), G.chain_nt(A2, A, 256, 64, 64, out2, dep=0)):
        with pytest.raises(RuntimeError, match="reads row blocks its producer does not write"):
            G.GemmChain([G.chain_nt(A, A, 128, 64, 64, out), second], torch.device("cuda"))
    # the largest legal K range is accepted: K = 128 over a 128-row producer
    G.GemmChain([G.chain_nt(A, A, 128, 64, 64, out), G.chain_tn(A, A, 64, 64, 128, gw, dep=0)], torch.device("cuda")).close()


def test_fused_step_batch_16384(cuda_context):
    """FusedCTR at a batch of 16384 (128 row blocks) builds its persistent chains and its step matches reference()"""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedCTR
    ctx = get_context()
    vocab = [1000, 50, 20000, 7, 3000] + [300] * 21
    B = 16384
    m = FusedCTR(vocab, embedding_dim=8, model="deepfm", batch=B, cache_threshold=64, lr=0.05,
                 sparse_optimizer={"category": "adagrad", "learning_rate": 0.05})
    assert m.use_chain
    gcpu = torch.Generator().manual_seed(5)
    ids = torch.stack([torch.randint(0, v, (B,), generator=gcpu) for v in vocab], dim=1).contiguous().to(ctx.device)
    dense = torch.rand(B, 13, generator=gcpu).to(ctx.device)
    labels = (torch.rand(B, generator=gcpu) < 0.3).float().to(ctx.device)
    m.forward_backward(ids, dense, labels)
    loss = m.forward_backward(ids, dense, labels, update=False)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    m.bwd_chain.check()
    ref_loss, g = m.reference(ids, dense, labels)
    assert abs(float(loss) - float(ref_loss)) < 5e-3, (float(loss), float(ref_loss))
    for name in [n for n in ["W0", "W1", "W2", "wout", "wd", "bias"] if n in m.segs]:
        o, n = m.segs[name]
        a, b = m.gtheta[o:o + n], g["theta"][o:o + n]
        assert float((a - b).abs().max()) < 0.05 * (float(b.abs().max()) + 1e-6) + 2e-4, name
    ge = m.G32[:, :m.ns * m.Dp]
    assert float((ge - g["emb"]).abs().max()) < 0.05 * float(g["emb"].abs().max()) + 2e-5


# ---------------------------------------------------------------------------------------------- cached variants

def variant_main():
    """reduced case list for a process started with one of the cached switches (EXB_GEMM_BN / _SWAP / _MC)"""
    cases = [dict(M=300, N=100, K=192, outT=True, fm_cols=64, D=66, ones_col=99, lda_extra=64),
             dict(M=129, N=448, K=448, outT=False, fm_cols=208, D=68, ones_col=447, ldo_extra=8),
             dict(M=4096, N=1728, K=320, outT=True, fm_cols=1664, D=64, ones_col=1727),
             dict(M=7, N=65, K=64, outT=True, fm_cols=64, D=130, ones_col=64),
             dict(M=1024, N=256, K=256, outT=True, fm_cols=256, D=4, ones_col=255),     # 4 N tiles
             dict(M=1024, N=384, K=1728, outT=False, fm_cols=384, D=6, ones_col=383),   # 6 N tiles
             dict(M=1024, N=512, K=256, outT=True, fm_cols=512, D=8, ones_col=511)]     # 8 N tiles
    n = 0
    for family in FAMILIES:
        for case in cases:
            for mode in (R.EPI_FWD, R.EPI_DX, R.EPI_DX_FM):
                run_nt(case, mode, family, seed=8000 + n)
                n += 1
        for case in (dict(M=448, N=1728, K=4096, splits=8), dict(M=100, N=72, K=448, splits=4),
                     dict(M=448, N=512, K=320, splits=3), dict(M=63, N=256, K=128, splits=5)):
            run_tn(case, family, seed=8000 + n)
            run_nt(case, R.EPI_DW, family, seed=8500 + n)
            n += 1
    from openembedding_b200.ops.gemm import check
    check()
    print("VARIANT_RATIOS " + json.dumps(RATIOS))


@pytest.mark.parametrize("env", [{"EXB_GEMM_BN": "128"}, {"EXB_GEMM_SWAP": "1"}, {"EXB_GEMM_MC": "2"},
                                 {"EXB_GEMM_MC": "4"}, {"EXB_GEMM_MC": "8"}], ids=["bn128", "swap", "mc2", "mc4", "mc8"])
def test_cached_variant(env):
    code = ("import sys; sys.path[:0] = [%r, %r]\nimport test_gpu_gemm_exact as T\nT.variant_main()\n"
            % (os.path.dirname(HERE), HERE))
    envs = {k: v for k, v in os.environ.items() if k not in ("EXB_GEMM_BN", "EXB_GEMM_SWAP", "EXB_GEMM_MC")}
    r = subprocess.run([sys.executable, "-c", code], env=dict(envs, **env), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=400)
    line = [s for s in r.stdout.splitlines() if s.startswith("VARIANT_RATIOS ")]
    assert r.returncode == 0 and line, r.stdout[-3000:]
    for k, v in json.loads(line[-1][len("VARIANT_RATIOS "):]).items():
        RATIOS[k] = max(RATIOS.get(k, 0.0), v)
