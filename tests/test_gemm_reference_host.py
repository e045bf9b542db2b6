"""The float64 GEMM reference (tests/gemm_reference.py), checked without a GPU:

  * every epilogue's reference equals a naive triple loop plus the contract written out element by element;
  * the exact family stays within its 2^20-grain budget and its FM term is exact, at every shape the GPU file uses;
  * the real-family bound is tight enough to matter: a round-toward-zero bf16 conversion breaks it.
"""
import pytest
import torch

import gemm_reference as R

F64 = torch.float64


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _small(M, N, K, seed):
    g = _gen(seed)
    return R.ints((M, K), 8, g, "cpu"), R.ints((N, K), 8, g, "cpu")


@pytest.mark.parametrize("M,N,K", [(3, 5, 64), (5, 70, 64), (2, 1, 128)])
def test_fwd_matches_loop(M, N, K):
    A, B = _small(M, N, K, 1)
    acc = R.naive_nt(A, B, M, N, K)
    for relu in (False, True):
        for ones in (-1, 0, N - 1, N + 3):
            v, c, _ = R.ref_nt(A, B, M, N, K, R.EPI_FWD, relu=relu, ones_col=ones)
            assert v.shape == (M, R.ceil64(N))
            for m in range(M):
                for n in range(R.ceil64(N)):
                    if n >= N:
                        e, const = 0.0, True
                    elif n == ones:
                        e, const = 1.0, True
                    else:
                        e, const = (max(float(acc[m, n]), 0.0) if relu else float(acc[m, n])), False
                    assert float(v[m, n]) == e and bool(c[m, n]) == const, (relu, ones, m, n)


def test_dx_matches_loop():
    M, N, K = 4, 67, 64
    A, B = _small(M, N, K, 2)
    acc = R.naive_nt(A, B, M, N, K)
    mask = R.ints((M, 80), 2, _gen(3), "cpu")
    mask[0, :4] = torch.tensor([0.0, -0.0, float("nan"), 2.0 ** -133])
    mask[:, N:] = 5.0                       # columns past N are not part of the mask
    ones = 10
    v, c, _ = R.ref_nt(A, B, M, N, K, R.EPI_DX, ones_col=ones, mask=mask)
    for m in range(M):
        for n in range(R.ceil64(N)):
            keep = n < N and n != ones and float(mask[m, n]) > 0
            assert float(v[m, n]) == (float(acc[m, n]) if keep else 0.0), (m, n)
            assert bool(c[m, n]) == (not keep)
    assert bool(c[0, :3].all()) and not bool(c[0, 3])


@pytest.mark.parametrize("fm_cols,D", [(0, 2), (12, 4), (40, 6), (64, 130), (66, 66)])
def test_dx_fm_matches_loop(fm_cols, D):
    M, N, K = 3, 70, 64
    A, B = _small(M, N, K, 4)
    g = _gen(5)
    dl, S, emb = R.ints((M,), 4, g, "cpu", -2), R.ints((M, D), 8, g, "cpu", -2), R.ints((M, max(fm_cols, 1)), 8, g, "cpu", -2)
    acc = R.naive_nt(A, B, M, N, K)
    v, c, _ = R.ref_nt(A, B, M, N, K, R.EPI_DX_FM, dl=dl, S=S, emb=emb, fm_cols=fm_cols, D=D)
    assert v.shape == (M, N) and not bool(c.any())
    for m in range(M):
        for n in range(N):
            e = float(acc[m, n])
            if n < fm_cols:
                e += float(dl[m]) * (float(S[m, n % D]) - float(emb[m, n]))
            assert float(v[m, n]) == e, (m, n)
    assert R.fm_exact(acc, N, fm_cols, D, dl, S, emb)


def test_dw_and_tn_match_loop():
    M, N, K = 6, 9, 128
    A, B = _small(M, N, K, 6)
    init = R.ints((M, N), 8, _gen(7), "cpu")
    acc = R.naive_nt(A, B, M, N, K)
    v, c, _ = R.ref_nt(A, B, M, N, K, R.EPI_DW, init=init)
    assert torch.equal(v, init + acc) and not bool(c.any())
    vt, _ = R.ref_tn(A.t().contiguous(), B.t().contiguous(), M, N, K, init)
    assert torch.equal(vt, v)


def test_transposed_region():
    v = torch.arange(3 * 64, dtype=F64).view(3, 64)
    t = R.transposed(v, 3)
    assert t.shape == (64, 3) and float(t[5, 2]) == float(v[2, 5])


def test_grain_and_rounding_helpers():
    assert R.grain(torch.tensor([3.0, -6.0, 0.0])) == 1.0
    assert R.grain(torch.tensor([0.75, 1.5])) == 0.25
    x = torch.tensor([257.0, 259.0, 258.0, -257.0, 1.0 + 2.0 ** -8])
    # ties go to even: 257 -> 256, 259 -> 260; toward zero: 259 -> 258
    assert R.bf16_rne(x).to(F64).tolist() == [256.0, 260.0, 258.0, -256.0, 1.0]
    assert R.bf16_rz(x).to(F64).tolist() == [256.0, 258.0, 258.0, -256.0, 1.0]


def test_check_exact_and_footprint_detect_mistakes():
    ref = torch.tensor([[1.0, 257.0, 0.0]], dtype=F64)
    const = torch.tensor([[False, False, True]])
    good = R.bf16_rne(ref)
    R.check_exact(good, ref, const)
    R.check_exact(torch.tensor([[1.0, 256.0, -0.0]]).to(torch.bfloat16), ref, torch.zeros_like(const))   # -0 == +0
    with pytest.raises(AssertionError):
        R.check_exact(torch.tensor([[1.0, 256.0, -0.0]]).to(torch.bfloat16), ref, const)     # a constant must be +0
    with pytest.raises(AssertionError):
        R.check_exact(R.bf16_rz(torch.tensor([[1.0, 259.0, 0.0]], dtype=F64)), torch.tensor([[1.0, 259.0, 0.0]], dtype=F64), const)
    c = R.Canvas(4, 5, torch.bfloat16, "cpu")
    assert c.ld % 8 == 0 and c.ld >= 13 and c.buf.shape[0] == 7
    c.snapshot()
    c.view.fill_(1.0)
    c.check_untouched(4, 5)
    c.buf[1, 7] = 0.0                       # inside the 16-byte unit of columns [0, 8): counts as written
    c.check_untouched(4, 5)
    c.buf[1, 8] = 0.0
    with pytest.raises(AssertionError):
        c.check_untouched(4, 5)
    c.snapshot()
    c.buf[4, 0] = 0.0                       # a row below the written rows
    with pytest.raises(AssertionError):
        c.check_untouched(4, 5)


def test_exact_budget_single_shapes():
    """dense exact operands: the worst case of every single-launch and split-K shape stays within 2^20 grains"""
    ks = {c["K"] for c in R.single_cases()} | {c["K"] for c in R.split_cases()} | {c["K"] for c in R.AUTO128_CASES}
    ks |= {R.FM_K}
    for k in ks:
        assert R.single_headroom(k) < R.EXACT_BUDGET, k
    # the pairwise cover really covers every pair
    cases = R.single_cases()
    assert {(c["M"], c["N"]) for c in cases} == {(m, n) for m in R.SINGLE_M for n in R.SINGLE_N}
    assert {(c["M"], c["K"]) for c in cases} == {(m, k) for m in R.SINGLE_M for k in R.SINGLE_K}
    assert {(c["N"], c["K"]) for c in cases} == {(n, k) for n in R.SINGLE_N for k in R.SINGLE_K}


def test_exact_fm_term_single_shapes():
    """the FM operand grids keep x + dl (s - e) exact at every FM shape (the accumulator at its worst case)"""
    g = _gen(8)
    shapes = [(R.FM_N, R.FM_K, D, fm) for D in R.FM_D for fm in R.FM_COLS]
    shapes += [(c["N"], c["K"], c["D"], c["fm_cols"]) for c in R.single_cases()]
    shapes += [(320, 4096, 66, 208)]                 # the mixed-K chain's dX1
    for N, K, D, fm_cols in shapes:
        M = 64
        dl, S, emb = R.ints((M,), 4, g, "cpu", -2), R.ints((M, D), 8, g, "cpu", -2), R.ints((M, fm_cols), 8, g, "cpu", -2)
        acc = torch.full((M, N), float(R.single_headroom(K, init=False)), dtype=F64)
        acc[::2] *= -1
        assert R.fm_exact(acc, N, fm_cols, D, dl, S, emb), (N, K, D, fm_cols)


@pytest.mark.parametrize("M,widths", [(m, R.CHAIN_W) for m in R.CHAIN_M] + [(4096, R.CHAIN_W8)])
def test_exact_budget_chains(M, widths):
    """forward + backward chain of the GPU file, simulated in float64 with every bf16 rounding: each GEMM's
    accumulator headroom stays within 2^20 grains, and the FM term of dX1 is exact"""
    g = _gen(100 + M)
    ops = R.chain_operands(M, widths, g, "cpu", fm_cols=R.CHAIN_FM_COLS, D=R.CHAIN_FM_D)
    H, dZ, heads, fm_ok = R.simulate_chain(M, widths, ops, fm_cols=R.CHAIN_FM_COLS, D=R.CHAIN_FM_D)
    print(M, widths, "largest headroom %.0f grains" % max(heads))
    assert max(heads) < R.EXACT_BUDGET, heads
    assert fm_ok
    # the chain is not trivial: activations and gradients are non-zero in every layer
    for t in H + dZ:
        assert float(t.abs().max()) > 0


@pytest.mark.parametrize("K", [64, 192, 256, 320, 448])
def test_real_bound_catches_round_toward_zero(K):
    """at the bf16-output shapes up to K = 448, a round-toward-zero conversion of the reference breaks the
    real-family bound on some elements. (For K >= 1728 the accumulation term dominates the bound: there the exact
    family is what tells the two roundings apart.)"""
    g = _gen(K)
    M, N = 129, 129
    A, B = R.normals((M, K), g, "cpu"), R.normals((N, K), g, "cpu")
    v, c, absp = R.ref_nt(A, B, M, N, K, R.EPI_FWD)
    b = R.real_bound(absp, K, v[:, :N], bf16_out=True)
    rz = R.bf16_rz(v[:, :N]).to(F64)
    rne = R.bf16_rne(v[:, :N]).to(F64)
    assert bool(((rne - v[:, :N]).abs() <= b).all())
    assert int(((rz - v[:, :N]).abs() > b).sum()) > 0
