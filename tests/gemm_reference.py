"""Float64 reference of the wgmma GEMM contract (csrc/cuda/gemm_wgmma.cu), plus the operand families, error bounds
and footprint checks the exact GEMM tests use. Plain torch float64; runs on any device, no GPU needed.

The contract, per epilogue (D = A[M, K] @ B[N, K]^T, fp32 accumulation):
  EPI_FWD    bf16 [M, ceil64(N)]: relu (optional), column ``ones_col`` set to 1, columns n >= N set to +0
  EPI_DX     bf16 [M, ceil64(N)]: +0 wherever !(mask > 0), at ``ones_col`` and at n >= N
  EPI_DX_FM  fp32 [M, N]: D + dl * (S[:, n mod D] - emb[:, n]) on the columns n < fm_cols, plain D after them
  EPI_DW     fp32 [M, N]: out += D onto the initial contents (split-K partial sums arrive by reduce-add);
             gemm_tn is the same with A stored [K, M] and B stored [K, N]
  outT       bf16 [ceil64(N), M]: the transposed copy of a bf16 output, pad rows included

Two operand families:
  * exact: small integers (optionally times a power of two) whose accumulations stay below 2^20 grains, so the fp32
    accumulation is exact in any order, split-K included. The kernel must then equal the reference bit for bit after
    one round-to-nearest-even to the output type.
  * real: random normals in bf16, checked within the derived bound C_ACC * K * 2^-24 * (|A| @ |B|^T), plus half a
    bf16 ulp (2^-8 |ref|) for a bf16 store and (splits + 1) * 2^-24 * (sum + |init|) for reduce-added partial sums.
"""
import torch

EPI_FWD, EPI_DX, EPI_DW, EPI_DX_FM = 0, 1, 2, 3

U32 = 2.0 ** -24            # fp32 unit roundoff (the same constants as test_gpu_fused_stages.py)
C_ACC = 4.0                 # constant of the fp32 accumulation bound
BF16_HALF_ULP = 2.0 ** -8   # half a bf16 ulp, relative: one round-to-nearest
EXACT_BUDGET = 2.0 ** 20    # exact family: largest accumulator magnitude, in grains

F64 = torch.float64
SENTINEL = {torch.bfloat16: 0x7FAB, torch.float32: 0x7FA5A5A5}   # NaN bit patterns outside the written region
INT_VIEW = {torch.bfloat16: torch.int16, torch.float32: torch.int32}


def ceil64(n):
    return (n + 63) // 64 * 64


# ---------------------------------------------------------------------------------------------- epilogues

def epi_fwd(acc, N, relu, ones_col):
    """acc [M, >= N] -> (value [M, ceil64(N)], const mask: positions the kernel writes as a constant)"""
    M, Np = acc.shape[0], ceil64(N)
    out = torch.zeros(M, Np, dtype=F64, device=acc.device)
    const = torch.zeros(M, Np, dtype=torch.bool, device=acc.device)
    x = acc[:, :N]
    out[:, :N] = x.clamp_min(0.0) if relu else x
    const[:, N:] = True
    if 0 <= ones_col < N:
        out[:, ones_col] = 1.0
        const[:, ones_col] = True
    return out, const


def epi_dx(acc, mask, N, ones_col):
    """relu-mask gradient: zero where !(mask > 0) (NaN, +-0 and negatives), at ones_col and at n >= N"""
    M, Np = acc.shape[0], ceil64(N)
    keep = mask[:M, :N] > 0
    if 0 <= ones_col < N:
        keep[:, ones_col] = False
    out = torch.zeros(M, Np, dtype=F64, device=acc.device)
    out[:, :N] = torch.where(keep, acc[:, :N], torch.zeros((), dtype=F64, device=acc.device))
    const = torch.ones(M, Np, dtype=torch.bool, device=acc.device)
    const[:, :N] = ~keep
    return out, const


def fm_term(M, fm_cols, D, dl, S, emb):
    """dl * (S[:, n mod D] - emb[:, n]) for n < fm_cols, [M, fm_cols]"""
    n = torch.arange(fm_cols, device=S.device)
    return dl[:M, None] * (S[:M][:, n % D] - emb[:M, :fm_cols])


def epi_dx_fm(acc, N, fm_cols, D, dl=None, S=None, emb=None):
    out = acc[:, :N].clone()
    if fm_cols > 0:
        out[:, :fm_cols] += fm_term(acc.shape[0], fm_cols, D, dl, S, emb)
    return out, torch.zeros_like(out, dtype=torch.bool)


def ref_nt(A, B, M, N, K, mode, relu=False, ones_col=-1, mask=None, dl=None, S=None, emb=None, fm_cols=0, D=1,
           init=None):
    """float64 reference of gemm_nt: (value, const mask, |A| @ |B|^T) over the output's contract region"""
    a, b = A[:M, :K].to(F64), B[:N, :K].to(F64)
    acc, absp = a @ b.t(), a.abs() @ b.abs().t()
    if mode == EPI_FWD:
        v, c = epi_fwd(acc, N, relu, ones_col)
    elif mode == EPI_DX:
        v, c = epi_dx(acc, mask.to(F64), N, ones_col)
    elif mode == EPI_DX_FM:
        v, c = epi_dx_fm(acc, N, fm_cols, D, *(None if t is None else t.to(F64) for t in (dl, S, emb)))
    else:
        v, c = init[:M, :N].to(F64) + acc, torch.zeros(M, N, dtype=torch.bool, device=acc.device)
    return v, c, absp


def ref_tn(A, B, M, N, K, init):
    """float64 reference of gemm_tn: init + A[K, M]^T @ B[K, N]"""
    a, b = A[:K, :M].to(F64), B[:K, :N].to(F64)
    return init[:M, :N].to(F64) + a.t() @ b, a.abs().t() @ b.abs()


def transposed(v, M):
    """the outT contract region [ceil64(N), M] of a bf16 output value [M, ceil64(N)]"""
    return v[:M].t()


def naive_nt(A, B, M, N, K):
    """triple loop, for checking the matmul form above on small shapes"""
    out = torch.zeros(M, N, dtype=F64)
    for m in range(M):
        for n in range(N):
            s = 0.0
            for k in range(K):
                s += float(A[m, k]) * float(B[n, k])
            out[m, n] = s
    return out


# ---------------------------------------------------------------------------------------------- operand families

def ints(shape, lim, gen, device, scale_log2=0, density=1.0):
    """exact family: integers in [-lim, lim] (a fraction `density` of them non-zero) times 2^scale_log2, float64"""
    x = torch.randint(-lim, lim + 1, shape, generator=gen, device=device).to(F64)
    if density < 1.0:
        x = x * (torch.rand(shape, generator=gen, device=device) < density)
    return x * 2.0 ** scale_log2


def normals(shape, gen, device, scale=1.0):
    """real family: normals rounded to bf16, returned as float64"""
    return (torch.randn(shape, generator=gen, device=device) * scale).to(torch.bfloat16).to(F64)


def grain(x):
    """largest power of two that divides every element of x (float64); 2^1023 for an all-zero tensor"""
    nz = x[x != 0].abs()
    if nz.numel() == 0:
        return 2.0 ** 1023
    m, e = torch.frexp(nz)
    v = (m * 2.0 ** 53).to(torch.int64)
    low = (v & -v).to(F64)                     # lowest set bit of the 53-bit significand
    return float((torch.log2(low).round() + e.to(F64) - 53).min().exp2())


def exact_headroom(A, B, M, N, K, tn=False, init=None):
    """largest accumulator bound of the exact family, in grains (must stay below EXACT_BUDGET): every partial sum of
    init + sum_k a_mk b_nk is a multiple of the grain and at most (|A| @ |B|^T + |init|) in magnitude"""
    a = (A[:K, :M].t() if tn else A[:M, :K]).to(F64)
    b = (B[:K, :N].t() if tn else B[:N, :K]).to(F64)
    s = a.abs() @ b.abs().t()
    g = grain(a) * grain(b)
    if init is not None:
        s = s + init[:M, :N].to(F64).abs()
        g = min(g, grain(init[:M, :N].to(F64)))
    return float(s.max()) / g if s.numel() else 0.0


def fm_exact(acc, N, fm_cols, D, dl, S, emb):
    """True when every step of x + dl * (s - e) in fp32 is exact for these operands"""
    if fm_cols == 0:
        return True
    M = acc.shape[0]
    n = torch.arange(fm_cols, device=S.device)
    d = S.to(F64)[:M][:, n % D] - emb.to(F64)[:M, :fm_cols]
    p = dl.to(F64)[:M, None] * d
    r = acc[:, :fm_cols] + p
    return all(bool((t.float().to(F64) == t).all()) for t in (d, p, r))


# ---------------------------------------------------------------------------------------------- checks

def bf16_rne(v):
    return v.to(torch.float32).to(torch.bfloat16)


def bf16_rz(v):
    """round toward zero to bf16 (the mistake a truncating conversion makes), from the fp32 value"""
    f = v.to(torch.float32).contiguous()
    return (f.view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)


def expected_exact(ref, dtype):
    """exact family: the one correctly rounded output the kernel must produce"""
    f = ref.to(torch.float32)
    assert bool((f.to(F64) == ref).all()), "exact family: reference not representable in fp32"
    return f.to(torch.bfloat16) if dtype == torch.bfloat16 else f


def check_exact(got, ref, const, what=""):
    """got == round(ref) on values (-0 == +0), and bit for bit +0.0 / 1.0 where the kernel writes a constant"""
    exp = expected_exact(ref, got.dtype)
    bad = ~(got.to(F64) == exp.to(F64))
    if bool(bad.any()):
        i = tuple(int(t) for t in bad.nonzero()[0])
        raise AssertionError("%s: %d of %d elements not exact, first at %s: got %r expected %r (ref %r)" % (
            what, int(bad.sum()), bad.numel(), i, float(got[i]), float(exp[i]), float(ref[i])))
    iv = INT_VIEW[got.dtype]
    gb, eb = got.contiguous().view(iv), exp.contiguous().view(iv)
    cbad = const & (gb != eb)
    if bool(cbad.any()):
        i = tuple(int(t) for t in cbad.nonzero()[0])
        raise AssertionError("%s: constant element at %s has bits %#x, expected %#x" % (what, i, int(gb[i]), int(eb[i])))


def real_bound(absp, K, ref, bf16_out, splits=1, init=None, extra=None):
    """derived error bound of the real family (float64, shape of ref)"""
    b = C_ACC * K * U32 * absp
    if init is not None or splits > 1:
        b = b + (splits + 1) * U32 * (absp + (init.to(F64).abs() if init is not None else 0.0))
    if extra is not None:
        b = b + extra
    if bf16_out:
        b = b * (1 + BF16_HALF_ULP) + BF16_HALF_ULP * ref.abs()
    return b


def check_bound(got, ref, bound, const=None, what=""):
    """|got - ref| <= bound (NaN fails); constants exact. Returns the largest error / bound ratio."""
    g = got.to(F64)
    err = (g - ref).abs()
    bad = ~(err <= bound)
    if const is not None:
        bad |= const & ~(g == ref)
    if bool(bad.any()):
        i = tuple(int(t) for t in bad.nonzero()[0])
        raise AssertionError("%s: %d elements out of bound, first at %s: got %r ref %r bound %r" % (
            what, int(bad.sum()), i, float(g[i]), float(ref[i]), float(bound[i])))
    pos = bound > 0
    return float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0


# ---------------------------------------------------------------------------------------------- footprint

class Canvas:
    """a [rows, cols] view inside a larger buffer: `extra_rows` rows below, `extra_cols` columns to the right
    inside the row stride, everything filled with a NaN sentinel bit pattern"""

    def __init__(self, rows, cols, dtype, device, extra_rows=3, extra_cols=8, align=None):
        if align is None:
            align = 16 // torch.tensor([], dtype=dtype).element_size()     # TMA: row stride a multiple of 16 bytes
        self.ld = (cols + extra_cols + align - 1) // align * align
        self.buf = torch.empty(rows + extra_rows, self.ld, dtype=dtype, device=device)
        self.buf.view(INT_VIEW[dtype]).fill_(SENTINEL[dtype])
        self.view = self.buf[:rows, :cols]
        self.before = None

    def set(self, values):
        """write float64 values into the top-left corner (exactly representable in the dtype)"""
        r, c = values.shape
        self.buf[:r, :c] = values.to(self.buf.dtype)
        return self

    def snapshot(self):
        self.before = self.buf.clone()

    def check_untouched(self, rows=0, cols=0, what=""):
        """every element outside [:rows, :cols] still has the bits it had at snapshot(). The GEMM's TMA stores write
        whole 16-byte units of a row (measured on H100), so the columns up to the next 16-byte boundary, inside the
        row stride, count as written; rows >= `rows` and the rest of the row padding must keep their bits."""
        iv = INT_VIEW[self.buf.dtype]
        unit = 16 // self.buf.element_size()
        cols = min(self.ld, (cols + unit - 1) // unit * unit)
        changed = self.buf.view(iv) != self.before.view(iv)
        changed[:rows, :cols] = False
        if bool(changed.any()):
            i = tuple(int(t) for t in changed.nonzero()[0])
            raise AssertionError("%s: element %s outside the written region [:%d, :%d] changed" % (what, i, rows, cols))

    def check_unchanged(self, what=""):
        self.check_untouched(0, 0, what)


# ---------------------------------------------------------------------------------------------- case lists

EXACT_LIM = 8               # exact family: integers in [-8, 8]; K <= 4096 keeps K * 64 + 8 below 2^20
SINGLE_M = (1, 7, 127, 128, 129, 300, 4096)
SINGLE_N = (1, 8, 63, 64, 65, 100, 129, 448, 1728)
# one k-block, the 3- and 4-stage ring depths exactly, a ring wrap, the step's K values
SINGLE_K = (64, 192, 256, 320, 448, 1728, 4096)
FM_D = (2, 4, 6, 8, 10, 12, 64, 66, 68, 130)


def single_cases():
    """pairwise cover of SINGLE_M x SINGLE_N x SINGLE_K: every (M, N), (M, K) and (N, K) pair occurs. Per case: a
    transposed copy on every other case, strided A (lda = K + 64) and a wider output row stride on some, and on every
    fourth case the ones column at n = N (a pad column, which must stay +0)"""
    out = []
    for i, (m, n) in enumerate((m, n) for m in SINGLE_M for n in SINGLE_N):
        k = SINGLE_K[i % len(SINGLE_K)]
        fm = (n * 2 // 3) // 4 * 4
        out.append(dict(M=m, N=n, K=k, outT=i % 2 == 0, lda_extra=64 if i % 3 == 0 else 0, ldo_extra=8 * (i % 4),
                        fm_cols=fm, D=FM_D[i % len(FM_D)], ones_col=n if i % 4 == 3 else (n - 1 - i % 3) if n > 2 else -1))
    return out


# split-K: 7 k-blocks in 4 splits (2, 2, 2, 1), 5 in 3, splits > nkb, splits == nkb, the step's dW, no split
SPLIT_KS = ((448, 4), (320, 3), (128, 5), (256, 4), (4096, 8), (448, 1))


def split_cases():
    out = []
    for i, (m, n) in enumerate((m, n) for m in (1, 63, 100, 448) for n in (1, 8, 72, 1728)):
        k, s = SPLIT_KS[i % len(SPLIT_KS)]
        out.append(dict(M=m, N=n, K=k, splits=s))
    return out


# the automatically chosen 128-wide tile (pick_bn: K <= 128, N >= 512, M >= 8192): the CIN GEMM and the threshold
AUTO128_CASES = (dict(M=36864, N=1728, K=128, outT=False), dict(M=8192, N=1728, K=128, outT=True),
                 dict(M=8192, N=512, K=64, outT=True))
# fm_cols: a multiple of 64 inside N, inside a 32-column group, on the edge of a 32-column group inside a tile (the
# group after it is not loaded), ending on the last tile edge (= N)
FM_N, FM_K, FM_M = 448, 192, 300
FM_COLS = (320, 208, 224, 448)
CHAIN_M = (128, 300, 4096, 8192, 8320, 16384)
CHAIN_W8 = (256, 192, 136, 128, 64)   # four layers: the backward chain is 8 GEMMs, the most a chain takes
CHAIN_FM_COLS, CHAIN_FM_D = 208, 68   # the chains' dX1: FM columns end inside a 32-column group; D wraps mid-tile


def single_headroom(K, init=True):
    """worst case of the dense exact family in grains: K products of at most 8 * 8, plus an initial value <= 8"""
    return K * EXACT_LIM * EXACT_LIM + (EXACT_LIM if init else 0)


# ---------------------------------------------------------------------------------------------- chains

CHAIN_W = (320, 180, 192, 128)      # widths: chain input, then the output of each layer (180: pad columns)


def chain_shapes(widths):
    p = [ceil64(w) for w in widths]
    return p


def chain_operands(M, widths, gen, device, fm_cols=0, D=2):
    """exact-family operands of a forward chain and a backward chain (fused_dense.py's dependency structure).
    Inputs are integers in [-4, 4]; weights are sparse {-1, 0, 1} (about four non-zeros per row) so activations keep
    their size from layer to layer and the batch-long dW sums stay within the budget. Batch rows are padded to Kb = ceil64(M) with zeros."""
    L = len(widths) - 1
    p = chain_shapes(widths)
    Kb = ceil64(M)
    A0 = torch.zeros(Kb, p[0], dtype=F64, device=device)
    A0[:M, :widths[0]] = ints((M, widths[0]), 4, gen, device)
    W = [ints((widths[l + 1], p[l]), 1, gen, device, density=4.0 / widths[l]) for l in range(L)]
    WT = [ints((widths[l], p[l + 1]), 1, gen, device, density=4.0 / widths[l + 1]) for l in range(L)]
    dtop = torch.zeros(Kb, p[L], dtype=F64, device=device)
    dtop[:M, :widths[L]] = ints((M, widths[L]), 4, gen, device)
    fm = None
    if fm_cols:
        fm = dict(dl=ints((Kb,), 4, gen, device, -2), S=ints((Kb, D), 8, gen, device, -2),
                  emb=ints((Kb, fm_cols), 8, gen, device, -2))
    return dict(A0=A0, W=W, WT=WT, dtop=dtop, fm=fm, p=p, Kb=Kb)


def simulate_chain(M, widths, ops, fm_cols=0, D=2):
    """float64 simulation of the forward and backward chains with the exact family: every bf16 output rounded as the
    kernel must round it. Returns the activations, the per-GEMM exact headroom and whether the FM term is exact."""
    L = len(widths) - 1
    p, Kb = ops["p"], ops["Kb"]
    heads = []
    src, H = ops["A0"], []
    for l in range(L):
        heads.append(exact_headroom(src, ops["W"][l], M, widths[l + 1], p[l]))
        v, _, _ = ref_nt(src, ops["W"][l], M, widths[l + 1], p[l], EPI_FWD, relu=True, ones_col=widths[l + 1] - 1)
        h = torch.zeros(Kb, p[l + 1], dtype=F64, device=src.device)
        h[:M] = bf16_rne(v).to(F64)
        H.append(h)
        src = h
    dZ = [None] * L
    dZ[L - 1] = ops["dtop"]
    fm_ok = True
    for l in range(L - 1, -1, -1):
        heads.append(exact_headroom(dZ[l], ops["WT"][l], M, widths[l], p[l + 1]))
        if l > 0:
            v, _, _ = ref_nt(dZ[l], ops["WT"][l], M, widths[l], p[l + 1], EPI_DX, ones_col=widths[l] - 1, mask=H[l - 1])
            d = torch.zeros(Kb, p[l], dtype=F64, device=src.device)
            d[:M] = bf16_rne(v).to(F64)
            dZ[l - 1] = d
        elif fm_cols:
            f = ops["fm"]
            acc = dZ[0][:M, :p[1]] @ ops["WT"][0][:widths[0], :p[1]].t()
            fm_ok = fm_exact(acc, widths[0], fm_cols, D, f["dl"], f["S"], f["emb"])
        srcl = ops["A0"] if l == 0 else H[l - 1]
        heads.append(exact_headroom(dZ[l], srcl, widths[l + 1], p[l], Kb, tn=True))
    return H, dZ, heads, fm_ok
