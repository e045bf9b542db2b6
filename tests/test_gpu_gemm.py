"""wgmma GEMM vs a plain PyTorch fp32 reference of the same op, every fused epilogue."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_pipeline_timeouts():
    """every GEMM launched by a test must have completed its shared-memory pipeline"""
    yield
    from openembedding_b200.ops.gemm import check
    check()


def _mk(rows, cols, ld=None, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ld = ld or cols
    buf = torch.zeros(rows, ld, device="cuda", dtype=torch.bfloat16)
    buf[:, :cols] = (torch.randn(rows, cols, device="cuda", generator=g) * scale).to(torch.bfloat16)
    return buf


@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 128, 192), (4096, 448, 1728), (4096, 448, 448), (300, 100, 128)])
def test_fwd_relu_ones_transposed(M, N, K):
    from openembedding_b200.ops.gemm import EPI_FWD, gemm_nt
    Np = (N + 63) // 64 * 64
    A, B = _mk(M, K, seed=1), _mk(Np, K, scale=0.1, seed=2)
    B[N:] = 0
    out = torch.full((M, Np), 7.0, device="cuda", dtype=torch.bfloat16)
    Mp = (M + 7) // 8 * 8        # TMA store: leading dimensions must be multiples of 16 bytes
    outT = torch.full((Np, Mp), 7.0, device="cuda", dtype=torch.bfloat16)[:, :M]
    ones_col = N - 1
    gemm_nt(A, B, M, N, K, out, mode=EPI_FWD, relu=True, ones_col=ones_col, outT=outT)
    torch.cuda.synchronize()
    ref = torch.relu(A.float() @ B[:N].float().t())
    ref[:, ones_col] = 1.0
    assert torch.allclose(out[:, :N].float(), ref, atol=2e-2, rtol=2e-2), (out[:, :N].float() - ref).abs().max()
    assert torch.equal(outT[:N].t().contiguous(), out[:, :N].contiguous())


def test_dx_mask():
    from openembedding_b200.ops.gemm import EPI_DX, gemm_nt
    M, N, K = 512, 448, 448
    dZ, WT = _mk(M, K, seed=3), _mk(N, K, scale=0.1, seed=4)
    H = _mk(M, N, seed=5)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    outT = torch.zeros(N, M, device="cuda", dtype=torch.bfloat16)
    gemm_nt(dZ, WT, M, N, K, out, mode=EPI_DX, ones_col=N - 1, outT=outT, mask=H)
    torch.cuda.synchronize()
    ref = (dZ.float() @ WT.float().t()) * (H.float() > 0)
    ref[:, N - 1] = 0
    assert torch.allclose(out.float(), ref, atol=3e-2, rtol=3e-2)
    assert torch.equal(outT.t().contiguous(), out)


@pytest.mark.parametrize("splits", [1, 4, 16])
def test_dw_splitk(splits):
    from openembedding_b200.ops.gemm import EPI_DW, gemm_nt
    M, N, K = 448, 1728, 4096      # dW1 = dZ1^T[448,B] @ A0^T[1728,B]^T
    A, B = _mk(M, K, scale=0.1, seed=6), _mk(N, K, scale=0.1, seed=7)
    out = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    gemm_nt(A, B, M, N, K, out, mode=EPI_DW, splits=splits)
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    assert torch.allclose(out, ref, atol=5e-2, rtol=2e-2), (out - ref).abs().max()


# (F fields, D = padded dim, persistent chain): F * D = 1664 is a multiple of 32; 208, 312, 108 and 340 are not,
# so their last embedding columns share a 32-column group with plain dX columns
DX_FM_CASES = [(26, 64, False), (26, 8, False), (26, 12, False), (27, 4, False), (5, 68, False), (26, 8, True)]


def test_dx_fm():
    """fp32 embedding gradient dZ @ W + dlogit * (S - e) on the F * D embedding columns, plain dX after them"""
    for F, D, chain in DX_FM_CASES:
        _dx_fm_case(F, D, chain)


def _dx_fm_case(F, D, chain):
    from openembedding_b200.ops import gemm as G
    case = "F=%d D=%d chain=%s" % (F, D, chain)
    Bsz, N, K = 256, 1728, 448
    dZ, WT = _mk(Bsz, K, seed=8), _mk(N, K, scale=0.1, seed=9)
    g = torch.Generator(device="cuda").manual_seed(10)
    emb = torch.randn(Bsz, 1800, device="cuda", generator=g)
    S = emb[:, :F * D].reshape(Bsz, F, D).sum(1).contiguous()
    dl = torch.randn(Bsz, device="cuda", generator=g)
    out = torch.zeros(Bsz, 1800, device="cuda")
    if chain:
        c = G.GemmChain([G.chain_nt(dZ, WT, Bsz, N, K, out, mode=G.EPI_DX_FM, dlogit=dl, S=S, emb=emb, fm_cols=F * D,
                                    D=D)], torch.device("cuda"))
        c.launch()
        c.check()
        c.close()
    else:
        G.gemm_nt(dZ, WT, Bsz, N, K, out, mode=G.EPI_DX_FM, dlogit=dl, S=S, emb=emb, fm_cols=F * D, D=D)
    torch.cuda.synchronize()
    out = out.double()
    plain = dZ.double() @ WT.double().t()
    ref = plain.clone()
    e64, S64 = emb.double(), S.double()
    fm = dl.double()[:, None, None] * (S64[:, None, :] - e64[:, :F * D].reshape(Bsz, F, D))
    ref[:, :F * D] += fm.reshape(Bsz, -1)
    assert torch.allclose(out[:, :N], ref, atol=5e-2, rtol=2e-2), (case, float((out[:, :N] - ref).abs().max()))
    # the columns after the embedding columns carry plain dX, without an FM term
    assert torch.allclose(out[:, F * D:N], plain[:, F * D:], atol=5e-2, rtol=2e-2), \
        (case, float((out[:, F * D:N] - plain[:, F * D:]).abs().max()))
    assert float(out[:, N:].abs().max()) == 0.0, case


@pytest.mark.parametrize("M,N,K,splits", [(128, 64, 64, 1), (64, 64, 128, 1), (448, 1728, 4096, 8), (448, 448, 4096, 8),
                                          (100, 72, 256, 2)])
def test_dw_mn_major(M, N, K, splits):
    """out = A[K,M]^T @ B[K,N] from batch-major operands (MN-major wgmma tiles, no transposed copies)"""
    from openembedding_b200.ops.gemm import gemm_tn
    ldm, ldn = (M + 7) // 8 * 8, (N + 7) // 8 * 8
    A, B = _mk(K, M, ld=ldm, scale=0.1, seed=11), _mk(K, N, ld=ldn, scale=0.1, seed=12)
    out = torch.zeros(M, ldn, device="cuda", dtype=torch.float32)
    gemm_tn(A[:, :M], B[:, :N], M, N, K, out[:, :N] if ldn == N else out, splits=splits)
    torch.cuda.synchronize()
    ref = A[:, :M].float().t() @ B[:, :N].float()
    assert torch.allclose(out[:, :N], ref, atol=5e-2, rtol=2e-2), (out[:, :N] - ref).abs().max()


@pytest.mark.parametrize("M", [512, 4096])
def test_chain_matches_single_launches(M):
    """persistent chain (forward 3 layers; backward dX/dW of 3 layers with row-block dependencies) == the same GEMMs
    launched one by one, bit for bit (same tiles, same K order)"""
    from openembedding_b200.ops import gemm as G
    K0, H1, H2, H3 = 320, 192, 192, 128
    dev = torch.device("cuda")
    A0 = _mk(M, K0, seed=1)
    W = [_mk(H1, K0, scale=0.1, seed=2), _mk(H2, H1, scale=0.1, seed=3), _mk(H3, H2, scale=0.1, seed=4)]
    WT = [w.t().contiguous() for w in W]
    dims = [K0, H1, H2, H3]

    def run(chain):
        H = [torch.zeros(M, d, device=dev, dtype=torch.bfloat16) for d in dims[1:]]
        dZ = [torch.zeros(M, d, device=dev, dtype=torch.bfloat16) for d in dims[1:]]
        dZ[2].copy_(_mk(M, H3, scale=0.05, seed=9))
        gW = [torch.zeros(dims[l + 1], dims[l], device=dev, dtype=torch.float32) for l in range(3)]
        G32 = torch.zeros(M, K0, device=dev, dtype=torch.float32)
        if chain:
            src, fd = A0, []
            for l in range(3):
                fd.append(G.chain_nt(src, W[l], M, dims[l + 1], dims[l], H[l], mode=G.EPI_FWD, relu=True, ones_col=dims[l + 1] - 1, dep=l - 1))
                src = H[l]
            c1 = G.GemmChain(fd, dev)
            c1.launch()
            bd, prod = [], -1
            for l in (2, 1, 0):
                if l > 0:
                    bd.append(G.chain_nt(dZ[l], WT[l], M, dims[l], dims[l + 1], dZ[l - 1], mode=G.EPI_DX, ones_col=dims[l] - 1,
                                         mask=H[l - 1], dep=prod))
                else:
                    bd.append(G.chain_nt(dZ[0], WT[0], M, K0, H1, G32, mode=G.EPI_DX_FM, fm_cols=0, D=4, dep=prod))
                nxt = len(bd) - 1
                bd.append(G.chain_tn(dZ[l], A0 if l == 0 else H[l - 1], dims[l + 1], dims[l], M, gW[l], splits=4, dep=prod))
                prod = nxt
            c2 = G.GemmChain(bd, dev)
            c2.launch()
            c1.check(); c2.check()
            c1.close(); c2.close()
        else:
            src = A0
            for l in range(3):
                G.gemm_nt(src, W[l], M, dims[l + 1], dims[l], H[l], mode=G.EPI_FWD, relu=True, ones_col=dims[l + 1] - 1)
                src = H[l]
            for l in (2, 1):
                G.gemm_nt(dZ[l], WT[l], M, dims[l], dims[l + 1], dZ[l - 1], mode=G.EPI_DX, ones_col=dims[l] - 1, mask=H[l - 1])
            G.gemm_nt(dZ[0], WT[0], M, K0, H1, G32, mode=G.EPI_DX_FM, fm_cols=0, D=4)
            for l in range(3):
                G.gemm_tn(dZ[l], A0 if l == 0 else H[l - 1], dims[l + 1], dims[l], M, gW[l], splits=4)
        torch.cuda.synchronize()
        return H, dZ, gW, G32

    a, b = run(False), run(True)
    for l in range(3):
        assert torch.equal(a[0][l], b[0][l]), ("H", l, float((a[0][l].float() - b[0][l].float()).abs().max()))
        assert torch.equal(a[1][l], b[1][l]), ("dZ", l)
        assert torch.allclose(a[2][l], b[2][l], atol=1e-3, rtol=1e-4), ("gW", l, float((a[2][l] - b[2][l]).abs().max()))
    assert torch.equal(a[3], b[3])
    ref = torch.relu(A0.float() @ W[0].float().t())
    ref[:, H1 - 1] = 1.0
    assert torch.allclose(b[0][0].float(), ref, atol=3e-2, rtol=3e-2)


@pytest.mark.parametrize("M,K,N", [(256, 100, 40), (1000, 247, 400), (130, 64, 1)])
def test_tc_linear_matches_torch(M, K, N):
    """forward, dX, dW, db of TcLinear (wgmma GEMMs) vs nn.Linear in fp32"""
    from openembedding_b200.ops.tc_linear import TcLinear
    torch.manual_seed(0)
    ref = torch.nn.Linear(K, N).cuda()
    tc = TcLinear(K, N).cuda()
    tc.load_state_dict(ref.state_dict())
    x = torch.randn(M, K, device="cuda")
    x1, x2 = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    g = torch.randn(M, N, device="cuda")
    y1, y2 = ref(x1), tc(x2)
    y1.backward(g)
    y2.backward(g)
    torch.cuda.synchronize()

    def close(a, b, what):
        err = float((a - b).abs().max())
        assert err < 0.03 * float(b.abs().max()) + 1e-2, (what, err, float(b.abs().max()))
    close(y2, y1, "y")
    close(x2.grad, x1.grad, "dx")
    close(tc.weight.grad, ref.weight.grad, "dw")
    close(tc.bias.grad, ref.bias.grad, "db")


@pytest.mark.parametrize("B,Fn,D,layers,split", [(64, 26, 9, (128, 128), True), (50, 7, 16, (32, 16, 8), True),
                                                 (33, 5, 4, (24,), False)])
def test_cin_own_kernels_match_torch(B, Fn, D, layers, split):
    """xDeepFM CIN on own kernels (interaction written as the GEMM operand + wgmma GEMM with bias/relu + row-wise
    backward, ops/cin.py) vs the einsum + Conv1d definition in fp32: output and every gradient"""
    from openembedding_b200.models.ctr import CIN
    torch.manual_seed(1)
    ref = CIN(Fn, layers, split_half=split, tc=False).cuda()
    own = CIN(Fn, layers, split_half=split, tc=True).cuda()
    for cr, co in zip(ref.convs, own.convs):
        with torch.no_grad():
            # pre-activations far from zero (half of the channels on, half off): a relu whose input sits within the
            # bf16 rounding error of zero flips between the two implementations and moves a whole gradient term
            cr.bias.copy_(torch.where(torch.arange(cr.bias.numel(), device="cuda") % 2 == 0, 4.0, -4.0))
            co.lin.weight.copy_(cr.weight.squeeze(-1))
            co.lin.bias.copy_(cr.bias)
    x = torch.randn(B, Fn, D, device="cuda") * 0.5
    x1, x2 = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    y1, y2 = ref(x1), own(x2)
    assert y1.shape == y2.shape == (B, ref.out_dim)
    g = torch.randn_like(y1)
    y1.backward(g)
    y2.backward(g)
    torch.cuda.synchronize()

    def close(a, b, what):
        err = float((a - b).abs().max())
        assert err < 0.03 * float(b.abs().max()) + 1e-2, (what, err, float(b.abs().max()))
    close(y2, y1, "y")
    close(x2.grad, x1.grad, "dx")
    for i, (cr, co) in enumerate(zip(ref.convs, own.convs)):
        close(co.lin.weight.grad, cr.weight.grad.squeeze(-1), "dw%d" % i)
        close(co.lin.bias.grad, cr.bias.grad, "db%d" % i)


def test_cluster_multicast_variant_matches(monkeypatch):
    """EXB_GEMM_MC: the A tile is loaded once per cluster and multicast into the CTAs that share it"""
    import subprocess, sys, os
    code = (
        "import torch, sys; sys.path.insert(0, %r)\n"
        "from openembedding_b200.ops.gemm import EPI_FWD, gemm_nt, gemm_tn\n"
        "g = torch.Generator(device='cuda').manual_seed(0)\n"
        "A = (torch.randn(1024, 448, device='cuda', generator=g)).to(torch.bfloat16)\n"
        "B = (torch.randn(448, 448, device='cuda', generator=g) * 0.1).to(torch.bfloat16)\n"
        "out = torch.zeros(1024, 448, device='cuda', dtype=torch.bfloat16)\n"
        "gemm_nt(A, B, 1024, 448, 448, out, mode=EPI_FWD, relu=True, ones_col=447)\n"
        "gw = torch.zeros(448, 448, device='cuda')\n"
        "gemm_tn(A, A, 448, 448, 1024, gw, splits=4)\n"
        "torch.cuda.synchronize()\n"
        "ref = torch.relu(A.float() @ B.float().t()); ref[:, 447] = 1\n"
        "assert torch.allclose(out.float(), ref, atol=3e-2, rtol=3e-2), float((out.float() - ref).abs().max())\n"
        "refw = A.float().t() @ A.float()\n"
        "assert torch.allclose(gw, refw, atol=0.5, rtol=2e-2), float((gw - refw).abs().max())\n"
        "print('MC_OK')\n" % os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, EXB_GEMM_MC="8"), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert "MC_OK" in r.stdout, r.stdout[-2000:]


def test_wide_tile_variant_matches():
    """EXB_GEMM_BN=128: the 128-wide tile (m64n128k16 wgmma, 3-stage ring, two-block MN-major operands) for every
    epilogue of gemm_nt and for gemm_tn, through the same checks as the default 64-wide tile"""
    import subprocess, sys, os
    here = os.path.dirname(os.path.abspath(__file__))
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import test_gpu_gemm as T\n"
        "from openembedding_b200.ops.gemm import check\n"
        "for shape in [(128, 64, 64), (256, 128, 192), (300, 200, 128), (4096, 448, 448)]:\n"
        "    T.test_fwd_relu_ones_transposed(*shape)\n"
        "T.test_dx_mask()\n"
        "for s in (1, 4):\n"
        "    T.test_dw_splitk(s)\n"
        "T.test_dx_fm()\n"
        "for shape in [(128, 64, 64, 1), (448, 1728, 4096, 8), (100, 200, 256, 2)]:\n"
        "    T.test_dw_mn_major(*shape)\n"
        "check()\n"
        "print('BN128_OK')\n" % (os.path.dirname(here), here))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, EXB_GEMM_BN="128"), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert "BN128_OK" in r.stdout, r.stdout[-2000:]
