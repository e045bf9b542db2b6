"""The epilogue source tile of the wgmma GEMM (relu mask of EPI_DX, FM embedding columns of EPI_DX_FM), which
reaches the epilogue by TMA through its staging tile: exact checks against the same GEMM's plain store, for the
single launch and the persistent chain."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_pipeline_timeouts():
    """every GEMM launched by a test must have completed its shared-memory pipeline"""
    yield
    from openembedding_b200.ops.gemm import check
    check()


def _bf16(rows, cols, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(rows, cols, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _grid(rows, cols, seed, step):
    """values on a grid of `step` in [-4, 4): their differences and products with a grid-valued dlogit are exact in
    fp32, so the fused FM term has one rounding only and the fp64 reference is exact"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randint(-int(4 / step), int(4 / step), (rows, cols), device="cuda", generator=g) * step).float()


def _run(chain, A, B, M, N, K, out, **kw):
    from openembedding_b200.ops import gemm as G
    if chain:
        kw.pop("outT", None)
        c = G.GemmChain([G.chain_nt(A, B, M, N, K, out, **kw)], torch.device("cuda"))
        c.launch()
        c.check()
        c.close()
    else:
        G.gemm_nt(A, B, M, N, K, out, **kw)
    torch.cuda.synchronize()


# (M, N, K): the step's shape; N not a multiple of 64 (a partial mask box); M not a multiple of 128
DX_SHAPES = [(4096, 448, 448), (512, 200, 448), (300, 448, 448)]


@pytest.mark.parametrize("chain", [False, True])
@pytest.mark.parametrize("M,N,K", DX_SHAPES)
def test_dx_mask_equals_masked_plain_store(M, N, K, chain):
    """EPI_DX == the plain bf16 store of the same GEMM with the relu mask, ones_col and n >= N applied in torch"""
    from openembedding_b200.ops import gemm as G
    Np = (N + 63) // 64 * 64
    dZ, WT = _bf16(M, K, 1), _bf16(N, K, 2, scale=0.1)
    # mask buffer wider than N: the columns past N hold positive values the epilogue must not read
    Hbuf = _bf16(M, Np + 64, 3)
    Hbuf[:, N:] = 1.0
    plain = torch.full((M, Np), 5.0, device="cuda", dtype=torch.bfloat16)
    _run(False, dZ, WT, M, N, K, plain, mode=G.EPI_FWD, relu=False, ones_col=-1)
    out = torch.full((M, Np), 5.0, device="cuda", dtype=torch.bfloat16)
    outT = None if chain else torch.full((Np, M + (-M) % 8), 5.0, device="cuda", dtype=torch.bfloat16)[:, :M]
    _run(chain, dZ, WT, M, N, K, out, mode=G.EPI_DX, ones_col=N - 1, mask=Hbuf, outT=outT)
    ref = torch.where(Hbuf[:, :N] > 0, plain[:, :N], torch.zeros_like(plain[:, :N]))
    ref[:, N - 1] = 0
    assert torch.equal(out[:, :N], ref), float((out[:, :N].float() - ref.float()).abs().max())
    if Np > N:                                         # n >= N: zero in both
        assert torch.equal(out[:, N:], plain[:, N:])
        assert float(out[:, N:].float().abs().max()) == 0.0
    if outT is not None:
        assert torch.equal(outT[:N].t(), out[:, :N])


# (F fields, D padded dim, M, N): dim 64 at the step's shape; nf * Dp = 208, not a multiple of 64 (or 32);
# M = 300, not a multiple of 128, with nf * Dp = 416
FM_SHAPES = [(26, 64, 4096, 1728), (26, 8, 512, 256), (26, 16, 300, 448)]


@pytest.mark.parametrize("chain", [False, True])
@pytest.mark.parametrize("F,D,M,N", FM_SHAPES)
def test_dx_fm_equals_plain_store_plus_fm_term(F, D, M, N, chain):
    """EPI_DX_FM == the fm_cols = 0 fp32 store of the same GEMM + dl * (S - e) in fp64: within 1 ulp in the
    embedding columns, bit for bit in every other column"""
    from openembedding_b200.ops import gemm as G
    K = 448
    fm_cols = F * D
    ld = N + 4                                   # row stride a multiple of 4 floats, like the model's XS
    dZ, WT = _bf16(M, K, 4), _bf16(N, K, 5, scale=0.1)
    emb = _grid(M, ld, 6, 1.0 / 64)
    S = _grid(M, D, 7, 1.0 / 64)
    dl = _grid(M, 1, 8, 1.0 / 256).reshape(M).contiguous()
    plain = torch.full((M, ld), 3.0, device="cuda")
    _run(False, dZ, WT, M, N, K, plain, mode=G.EPI_DX_FM, fm_cols=0)
    out = torch.full((M, ld), 3.0, device="cuda")
    _run(chain, dZ, WT, M, N, K, out, mode=G.EPI_DX_FM, dlogit=dl, S=S, emb=emb, fm_cols=fm_cols, D=D)
    fm = dl.double()[:, None, None] * (S.double()[:, None, :] - emb[:, :fm_cols].double().reshape(M, F, D))
    ref = (plain[:, :fm_cols].double() + fm.reshape(M, fm_cols)).float()
    got = out[:, :fm_cols]
    ulp = (torch.nextafter(ref.abs(), torch.full_like(ref, float("inf"))) - ref.abs())
    assert bool(((got - ref).abs() <= ulp).all()), float((got - ref).abs().max())
    # plain columns after the embedding columns, and the untouched columns past N, bit for bit
    assert torch.equal(out[:, fm_cols:], plain[:, fm_cols:])


def test_epilogue_source_alignment_is_checked():
    """the TMA map of the source tile needs a 16-byte aligned base and row stride: anything else is refused"""
    from openembedding_b200.ops import gemm as G
    M, N, K, D = 256, 256, 448, 8
    dZ, WT = _bf16(M, K, 9), _bf16(N, K, 10, scale=0.1)
    S = torch.zeros(M, D, device="cuda")
    dl = torch.zeros(M, device="cuda")
    out = torch.zeros(M, N + 4, device="cuda")
    emb = torch.zeros(M, N + 5, device="cuda")[:, 1:]       # base 4 bytes off
    with pytest.raises(RuntimeError, match="16-byte"):
        G.gemm_nt(dZ, WT, M, N, K, out, mode=G.EPI_DX_FM, dlogit=dl, S=S, emb=emb, fm_cols=208, D=D)
    emb = torch.zeros(M, N + 2, device="cuda")               # row stride 2 floats past a multiple of 4
    with pytest.raises(RuntimeError, match="16-byte"):
        G.GemmChain([G.chain_nt(dZ, WT, M, N, K, out, mode=G.EPI_DX_FM, dlogit=dl, S=S, emb=emb, fm_cols=208, D=D)],
                    torch.device("cuda"))


def test_wide_tile_epilogue_source():
    """EXB_GEMM_BN=128: the single launch's 128-wide tile (two mask boxes, four embedding boxes per quarter)"""
    here = os.path.dirname(os.path.abspath(__file__))
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import test_gpu_gemm_epilogue_src as T\n"
        "from openembedding_b200.ops.gemm import check\n"
        "for shape in T.DX_SHAPES:\n"
        "    T.test_dx_mask_equals_masked_plain_store(*shape, chain=False)\n"
        "for shape in T.FM_SHAPES:\n"
        "    T.test_dx_fm_equals_plain_store_plus_fm_term(*shape, chain=False)\n"
        "check()\n"
        "print('BN128_SRC_OK')\n" % (os.path.dirname(here), here))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, EXB_GEMM_BN="128"), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert "BN128_SRC_OK" in r.stdout, r.stdout[-2000:]
