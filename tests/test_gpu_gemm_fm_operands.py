"""The FM term of the dX1 epilogue reads S one column pair at a time as a float2: an odd padded dimension D is
refused by the single launch and by the chain instead of producing misaligned loads."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("chain", [False, True])
def test_odd_fm_dimension_is_refused(chain):
    from openembedding_b200.ops import gemm as G
    B, K, F, D = 128, 64, 4, 9
    N = 64
    dZ = torch.zeros(B, K, device="cuda", dtype=torch.bfloat16)
    WT = torch.zeros(N, K, device="cuda", dtype=torch.bfloat16)
    emb = torch.zeros(B, N, device="cuda")
    S = torch.zeros(B, D, device="cuda")
    dl = torch.zeros(B, device="cuda")
    out = torch.zeros(B, N, device="cuda")
    kw = dict(mode=G.EPI_DX_FM, dlogit=dl, S=S, emb=emb, fm_cols=F * D, D=D)
    with pytest.raises(RuntimeError, match="even D"):
        if chain:
            G.GemmChain([G.chain_nt(dZ, WT, B, N, K, out, **kw)], torch.device("cuda"))
        else:
            G.gemm_nt(dZ, WT, B, N, K, out, **kw)
