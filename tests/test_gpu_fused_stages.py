"""The fused DeepFM / WDL step (models/fused_dense.py) checked one stage at a time against float64 references.

After one ``forward_backward(..., update=False)`` every intermediate of the step is still in the model's buffers
(X32, A0, H[l], dZ[l], S, base, dlogit, loss, G32, gtheta, Wb, WTb). Each stage is compared with plain float64
math whose inputs are the buffers the previous stage actually wrote, so an error cannot compound from one stage
to the next and a failure names the kernel that is wrong.

Error bounds are derived, not tuned: an fp32-accumulated dot product of length K is within
``C_ACC * K * 2^-24 * sum|a_i b_i|`` of the exact value (sum computed in float64), plus one bf16 ulp
(2^-7 |ref|) when the result is stored as bf16. Values the kernels copy or write as constants are compared
bit for bit; sums made with atomics or split-K reduce-add never are.
"""
import ctypes
import json
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # fp32 unit roundoff
BF16_ULP = 2.0 ** -7      # one bf16 ulp, relative
C_ACC = 4.0               # constant of the fp32 accumulation bound
POW_ULP = 8.0             # powf (ftrl): CUDA documents at most 4 ulp; 8 leaves room for the argument's rounding
C_OPT = 8.0               # relative error of one optimizer step: about 6.5 roundings (sqrt.approx 2 ulp,
                          # __fdividef 2 ulp, and the products / sums around them)

BASE_VOCAB = [1000, 50, 20000, 7, 3000] + [300] * 21     # 26 features; cache 64 -> features 1 and 3 replicated

# name -> FusedCTR arguments. ``hit``: nf * Dp is not a multiple of 32, so the FM term of the columns
# [32 * floor(nf * Dp / 32), nf * Dp) needs per-column-pair handling in the dX GEMM epilogue.
CONFIGS = {
    # partial FM group on server features, row-wise prep
    "fm26_d8": dict(vocab=BASE_VOCAB, dim=8, cache=0, B=256, dense_opt="adagrad"),
    # partial FM group on the cached features, prep A + B (128 % 12 != 0)
    "fm26_d9_cache": dict(vocab=BASE_VOCAB, dim=9, cache=64, B=384, dense_opt="adam"),
    # Dp 4: three features in the partial group (the packed embedding + linear row needs dim + 1 >= 4, so the
    # embeddings and linear weights are separate tables here)
    "fm27_d1": dict(vocab=BASE_VOCAB + [300], dim=1, cache=0, B=256, dense_opt="ftrl", pack_linear=False),
    # Dp 68: partial group inside one feature, cachegrad at Dp 68
    "fm5_d65_cache": dict(vocab=BASE_VOCAB[:5], dim=65, cache=64, B=384, dense_opt="adagrad"),
    # cachegrad at its largest Dp
    "fm3_d128_cache": dict(vocab=[1000, 50, 7], dim=128, cache=64, B=256, dense_opt="ftrl"),
    # aligned controls (dim 64 is the benchmark layout)
    "fm26_d16_cache": dict(vocab=BASE_VOCAB, dim=16, cache=64, B=256, dense_opt="adam"),
    "fm26_d64_cache": dict(vocab=BASE_VOCAB, dim=64, cache=64, B=256, dense_opt="adagrad"),
    # fm_cols = 0, four layers (the dense optimizer kernel's maximum)
    "wdl_d9_cache": dict(vocab=BASE_VOCAB, dim=9, cache=64, B=256, dense_opt="adagrad", model="wdl"),
    # Hp 640 > 512: head A + B with a single layer (head A owns the cached linear gradients)
    "fm26_d8_h600_cache": dict(vocab=BASE_VOCAB, dim=8, cache=64, B=256, dense_opt="adam", hidden=(600,)),
    # Hp 64 and 128 without pad columns: the ones column is the last column of the layer
    "fm26_d16_h63_127": dict(vocab=BASE_VOCAB, dim=16, cache=0, B=256, dense_opt="ftrl", hidden=(63, 127)),
    # no dense features. The replicated tables are what starts training here: with zero server rows and no dense
    # input the first layer sees only its bias column, almost every relu is off and no embedding would move
    "fm26_d8_nodense_cache": dict(vocab=BASE_VOCAB, dim=8, cache=64, B=256, dense_opt="adagrad", nd=0),
}

DENSE_OPT = {"adagrad": {"category": "adagrad", "learning_rate": 0.05},
             "adam": {"category": "adam", "learning_rate": 0.01},
             "ftrl": {"category": "ftrl", "learning_rate": 0.05, "l1_regularization_strength": 0.001}}


def _batch(vocab, B, nd, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randint(0, v, (B,), generator=g) for v in vocab], dim=1).contiguous()
    dense = torch.rand(B, nd, generator=g)
    labels = (torch.rand(B, generator=g) < 0.3).float()
    return ids, dense, labels


class _Ratios(dict):
    """largest |got - ref| / bound seen per stage"""

    def check(self, stage, got, ref, bound, what=""):
        got, ref, bound = got.double(), ref.double(), bound.double()
        assert bool(torch.isfinite(ref).all() and torch.isfinite(bound).all()), (stage, what, "non-finite reference")
        err = (got - ref).abs()
        bad = ~(err <= bound)           # a NaN in got is a failure too
        if bool(bad.any()):
            idx = tuple(int(i) for i in bad.nonzero()[0])
            raise AssertionError("%s %s: %d elements out of bound, first at %s: got %r ref %r bound %r" % (
                stage, what, int(bad.sum()), idx, float(got[idx]), float(ref[idx]), float(bound[idx])))
        pos = bound > 0
        r = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
        self[stage] = max(self.get(stage, 0.0), r)


def _bits_equal(a, b):
    """bitwise equality of two bf16 / fp32 tensors"""
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    iv = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    return torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


def _dot_bound(A, B_):
    """C_ACC * K * u * (|A| @ |B|): fp32-accumulation bound of A @ B (float64 operands)"""
    return C_ACC * A.shape[-1] * U32 * (A.abs() @ B_.abs())


def run_stages(name):
    """Build the model of CONFIGS[name], run one step without update and check every stage; returns the
    error/bound ratios per stage plus the FM sensitivity ratio. Needs the CUDA context to be set up."""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedCTR
    from openembedding_b200.ops import gemm as G
    cfg = dict(CONFIGS[name])
    ctx = get_context()
    dev = ctx.device
    vocab, B, nd = cfg["vocab"], cfg["B"], cfg.get("nd", 13)
    model = cfg.get("model", "deepfm")
    m = FusedCTR(vocab, num_dense=nd, embedding_dim=cfg["dim"], model=model, batch=B, hidden=cfg.get("hidden"),
                 cache_threshold=cfg["cache"], sparse_optimizer={"category": "adam", "learning_rate": 0.2},
                 dense_optimizer=dict(DENSE_OPT[cfg["dense_opt"]]), dw_splits=2, pack_linear=cfg.get("pack_linear"))
    nf, Dp, D, ns, nc, L = m.nf, m.Dp, m.D, m.ns, m.nc, len(m.hidden)
    K0p, lin0, Hp = m.K0p, m.lin0, m.Hp
    dims = [K0p] + Hp
    g = torch.Generator().manual_seed(7)
    if nc:      # random replicated tables, pad columns Dp - D kept at zero (their gradient is zero: they stay so)
        ce = torch.randn(m.cache_rows, Dp, generator=g) * 0.3
        ce[:, D:] = 0
        m.view("cache_emb").copy_(ce.reshape(-1).to(dev))
        m.view("cache_lin").copy_((torch.randn(m.cache_rows, generator=g) * 0.3).to(dev))
    # Adam moves every touched embedding element by about lr whatever its gradient: the pulled rows are far from
    # zero afterwards, so the FM term (which vanishes with the embeddings) is large
    for s in range(2):
        m.forward_backward(*[t.to(dev) for t in _batch(vocab, B, nd, seed=s)])
    ids_c, dense_c, labels_c = _batch(vocab, B, nd, seed=99)
    ids, dense, labels = ids_c.to(dev), dense_c.to(dev), labels_c.to(dev)
    m.forward_backward(ids, dense, labels, update=False)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    G.check()

    R = _Ratios()
    f64 = torch.float64
    dd = lambda t: t.detach().to(f64)
    theta = dd(m.theta)
    X = dd(m.X32)
    A0 = m.A0.clone()
    S = dd(m.S)
    dl = dd(m.dlogit)
    dense64, labels64 = dense.to(f64), labels.to(f64)
    ids_l = ids.long()
    cache_col = m.cache_col.long()
    cache_off = m.cache_off.long()
    rows_c = (ids_l[:, cache_col] + cache_off) if nc else None          # [B, nc] rows of the replicated tables
    seg = lambda name_: theta[m.segs[name_][0]:m.segs[name_][0] + m.segs[name_][1]]
    gseg = lambda name_: dd(m.gview(name_))

    # ---------------- prep: A0 (bitwise), cached X32 columns (bitwise), S, base
    emb_cols, srv_cols = nf * Dp, ns * Dp
    if nc:
        cemb = m.view("cache_emb").view(-1, Dp)
        want = cemb[rows_c].reshape(B, nc * Dp)
        assert _bits_equal(m.X32[:, srv_cols:emb_cols], want), "prep: cached X32 columns != cache_emb rows"
    a0_ref = torch.zeros(B, K0p, dtype=torch.float32, device=dev)
    a0_ref[:, :emb_cols] = m.X32[:, :emb_cols]
    a0_ref[:, emb_cols:emb_cols + nd] = dense
    a0_ref[:, K0p - 1] = 1.0
    assert _bits_equal(A0, a0_ref.to(torch.bfloat16)), "prep: A0 != bf16(emb, dense, 0, 1)"
    if not m.mn_major:
        assert _bits_equal(m.A0T, A0.t()), "prep: A0T is not the transpose of A0"
    e = X[:, :emb_cols].view(B, nf, Dp)
    s_ref = e.sum(1)
    absA = e.abs().sum(1)
    R.check("prep", S, s_ref, C_ACC * nf * U32 * absA, "S")
    lin_terms = [X[:, lin0:lin0 + ns]]
    if nc:
        lin_terms.append(seg("cache_lin")[rows_c])
    if nd:
        lin_terms.append(dense64 * seg("wd")[:nd])
    lin_t = torch.cat(lin_terms, dim=1)
    bias = seg("bias")[0]
    n_lin = lin_t.shape[1]
    base_ref = lin_t.sum(1) + bias
    fm_abs = torch.zeros(B, dtype=f64, device=dev)
    fm_err = torch.zeros(B, dtype=f64, device=dev)
    if m.use_fm:
        sq_s, sq_e = (s_ref * s_ref).sum(1), (e * e).sum((1, 2))
        base_ref = base_ref + 0.5 * (sq_s - sq_e)
        fm_abs = sq_s + sq_e
        # error of sum_d s_d^2 through the error of s_d (nf-term sums), plus the two squared-norm sums
        fm_err = 0.5 * (2 * nf * (s_ref.abs() * absA).sum(1) + (Dp + 1) * sq_s + nf * Dp * sq_e)
    base_bound = C_ACC * U32 * (n_lin * lin_t.abs().sum(1) + fm_err + 32 * (lin_t.abs().sum(1) + fm_abs + bias.abs()))
    R.check("prep", dd(m.base), base_ref, base_bound, "base")

    # ---------------- forward: H[l] = bf16(relu(prev @ Wb[l]^T)), ones column 1, pad columns 0
    for l in range(L):
        W = seg("W%d" % l).view(Hp[l], dims[l])
        assert _bits_equal(m.Wb[l], W.float().to(torch.bfloat16)), ("Wb != bf16(theta)", l)
        assert _bits_equal(m.WTb[l], m.Wb[l].t()), ("WTb != Wb^T", l)
        prev = A0 if l == 0 else m.H[l - 1]
        P = dd(prev) @ dd(m.Wb[l]).t()
        bnd = _dot_bound(dd(prev), dd(m.Wb[l]).t())
        ref = torch.relu(P)
        # relu is 1-Lipschitz: a pre-activation within the bound of 0 may land on either side
        bound = bnd * (1 + BF16_ULP) + BF16_ULP * ref
        h = m.H[l]
        hl = m.hidden[l]
        R.check("forward", dd(h[:, :hl]), ref[:, :hl], bound[:, :hl], "H%d" % l)
        assert bool((h[:, Hp[l] - 1] == 1).all()), ("forward: ones column", l)
        assert bool((h[:, hl:Hp[l] - 1] == 0).all()), ("forward: pad columns", l)
        if not m.mn_major and l < L - 1:
            assert _bits_equal(m.HT[l], h.t()), ("HT is not the transpose of H", l)

    # ---------------- head: dlogit, loss, dZ[L-1], g_wout, g_wd, g_bias, G32 linear columns
    Hl = dd(m.H[-1])
    wout = seg("wout")
    z = Hl @ wout + dd(m.base)
    z_err = C_ACC * U32 * (Hp[-1] * (Hl.abs() @ wout.abs()) + dd(m.base).abs() + z.abs())
    sig = torch.sigmoid(z)
    dl_ref = (sig - labels64) / B
    dl_bound = (0.25 * z_err + C_ACC * U32 * (1 + sig)) / B + 2 * U32 * dl_ref.abs()
    R.check("head", dl, dl_ref, dl_bound, "dlogit")
    lb = torch.clamp(z, min=0) - z * labels64 + torch.log1p(torch.exp(-z.abs()))
    loss_bound = (z_err.sum() + C_ACC * U32 * (z.abs() * 2 + 1).sum() + C_ACC * B * U32 * lb.sum()) / B
    R.check("head", dd(m.loss).view(()), lb.sum() / B, loss_bound, "loss")
    ones = Hp[-1] - 1
    dz_ref = dl[:, None] * wout[None, :] * (Hl > 0)
    dz_ref[:, ones] = 0
    R.check("head", dd(m.dZ[-1]), dz_ref, (BF16_ULP + 2 * U32) * dz_ref.abs(), "dZ%d" % (L - 1))
    assert bool((m.dZ[-1][:, ones] == 0).all()), "head: ones column of dZ"
    R.check("head", gseg("wout"), dl @ Hl, C_ACC * B * U32 * (dl.abs() @ Hl.abs()), "g_wout")
    if nd:
        R.check("head", gseg("wd")[:nd], dl @ dense64, C_ACC * B * U32 * (dl.abs() @ dense64.abs()), "g_wd")
    R.check("head", gseg("bias"), dl.sum().view(1), (C_ACC * B * U32 * dl.abs().sum()).view(1), "g_bias")
    assert _bits_equal(m.G32[:, lin0:lin0 + ns], m.dlogit[:, None].expand(B, ns)), "head: G32 linear columns != dlogit"
    if not m.mn_major:
        assert _bits_equal(m.dZT[-1], m.dZ[-1].t()), "head: dZT is not the transpose of dZ"

    # ---------------- dX: dZ[l-1] = bf16((dZ[l] @ WTb[l]^T) * (H[l-1] > 0)), ones column 0
    for l in range(L - 1, 0, -1):
        dZ, WT = dd(m.dZ[l]), dd(m.WTb[l])
        mask = (dd(m.H[l - 1]) > 0).to(f64)
        mask[:, Hp[l - 1] - 1] = 0
        ref = (dZ @ WT.t()) * mask
        bound = _dot_bound(dZ, WT.t()) * mask * (1 + BF16_ULP) + BF16_ULP * ref.abs()
        R.check("dX", dd(m.dZ[l - 1]), ref, bound, "dZ%d" % (l - 1))
        assert bool((m.dZ[l - 1][:, Hp[l - 1] - 1] == 0).all()), ("dX: ones column", l - 1)
        if not m.mn_major:
            assert _bits_equal(m.dZT[l - 1], m.dZ[l - 1].t()), ("dZT is not the transpose of dZ", l - 1)

    # ---------------- dX + FM: G32[:, :K0p] = dZ0 @ W0 (+ dlogit * (S - e) on the nf * Dp embedding columns)
    dZ0, WT0 = dd(m.dZ[0]), dd(m.WTb[0])
    mlp = dZ0 @ WT0.t()
    mlp_bound = _dot_bound(dZ0, WT0.t())
    fm_cols = emb_cols if m.use_fm else 0
    fm = torch.zeros_like(mlp)
    fm_bound = torch.zeros_like(mlp)
    if fm_cols:
        Sx = S.repeat(1, nf)                                     # S[b, c % Dp] for every embedding column c
        fm[:, :fm_cols] = dl[:, None] * (Sx - X[:, :fm_cols])
        fm_bound[:, :fm_cols] = 3 * U32 * dl.abs()[:, None] * (Sx.abs() + X[:, :fm_cols].abs())
    ref = mlp + fm
    bound = mlp_bound + fm_bound + U32 * ref.abs()
    got = dd(m.G32[:, :K0p])
    R.check("dX+FM", got[:, :fm_cols], ref[:, :fm_cols], bound[:, :fm_cols], "embedding columns")
    R.check("dX+FM", got[:, fm_cols:], mlp[:, fm_cols:], mlp_bound[:, fm_cols:] + U32 * mlp[:, fm_cols:].abs(),
            "plain dX columns")
    sens = None
    lo = fm_cols // 32 * 32
    if fm_cols % 32:
        # the columns a per-32-column-group FM epilogue leaves without the FM term: without it the reference
        # must move by far more than the bound, or the check above could not see that mistake
        # (pad columns Dp - D have neither an FM term nor a bound)
        sens = float((fm[:, lo:fm_cols].abs() / bound[:, lo:fm_cols]).nan_to_num(0.0).max())
        assert sens >= 10, ("sensitivity of the dX+FM check on columns [%d, %d)" % (lo, fm_cols), sens)

    # ---------------- dW: gW[l] = dZ[l]^T @ act[l-1] (split-K partial sums)
    for l in range(L):
        act = dd(A0 if l == 0 else m.H[l - 1])
        dZ = dd(m.dZ[l])
        ref = dZ.t() @ act
        R.check("dW", gseg("W%d" % l).view(Hp[l], dims[l]), ref, _dot_bound(dZ.t(), act), "W%d" % l)

    # ---------------- cachegrad: index_add of the G32 cached columns and of dlogit
    if nc:
        Gc = dd(m.G32[:, srv_cols:emb_cols]).view(B, nc, Dp)
        ref_e = torch.zeros(m.cache_rows, Dp, dtype=f64, device=dev)
        abs_e = torch.zeros_like(ref_e)
        ref_l = torch.zeros(m.cache_rows, dtype=f64, device=dev)
        abs_l = torch.zeros_like(ref_l)
        for j in range(nc):
            ref_e.index_add_(0, rows_c[:, j], Gc[:, j])
            abs_e.index_add_(0, rows_c[:, j], Gc[:, j].abs())
            ref_l.index_add_(0, rows_c[:, j], dl)
            abs_l.index_add_(0, rows_c[:, j], dl.abs())
        R.check("cachegrad", gseg("cache_emb").view(-1, Dp), ref_e, C_ACC * B * U32 * abs_e, "g_cache_emb")
        R.check("cachegrad", gseg("cache_lin"), ref_l, C_ACC * B * U32 * abs_l, "g_cache_lin")

    # ---------------- dense optimizer on the gradients checked above
    _check_optimizer(m, R)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    G.check()
    out = dict(R)
    out["sensitivity"] = sens
    return out


def _check_optimizer(m, R):
    """exb_dense_opt_kernel, launched directly, vs the tf.keras update in float64"""
    from openembedding_b200.models.fused_dense import _ck
    d = m.dense_opt
    kind = d["category"]
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))    # the kernel receives fp32 hyper-parameters
    lr, eps = f32(d["learning_rate"]), f32(d.get("epsilon", m.eps))
    if kind == "adam":
        m.opt_step.fill_(1)
    torch.cuda.synchronize()
    w, a, b, gr = (t.detach().double().clone() for t in (m.theta, m.accum, m.accum2, m.gtheta))
    _ck(m.lib.exb_dense_opt(ctypes.byref(m._opt_args), m._st()), "dense_opt")
    torch.cuda.synchronize()
    u = U32
    if kind == "adagrad":
        a1 = a + gr * gr
        step = lr * gr / (a1.sqrt() + eps)
        w1 = w - step
        R.check("optimizer", m.theta.double(), w1, C_OPT * u * step.abs() + 2 * u * w1.abs(), "adagrad theta")
        R.check("optimizer", m.accum.double(), a1, 2 * u * a1, "adagrad accum")
    elif kind == "adam":
        b1, b2 = f32(d["beta_1"]), f32(d["beta_2"])
        lr_t = lr * math.sqrt(1 - b2) / (1 - b1)                 # step 1
        m1 = b1 * a + (1 - b1) * gr
        v1 = b2 * b + (1 - b2) * gr * gr
        m1_err = C_ACC * u * (b1 * a.abs() + (1 - b1) * gr.abs())
        v1_err = C_ACC * u * (b2 * b + (1 - b2) * gr * gr)
        den = v1.sqrt() + eps
        step = lr_t * m1 / den
        w1 = w - step
        sq = v1.sqrt().clamp(min=1e-30)
        step_err = lr_t * m1_err / den + step.abs() * (v1_err / (2 * sq * den) + C_OPT * u)
        step_err = torch.where(v1 > 0, step_err, lr_t * m1_err / den + C_OPT * u * step.abs())
        R.check("optimizer", m.theta.double(), w1, step_err + 2 * u * w1.abs(), "adam theta")
        R.check("optimizer", m.accum.double(), m1, m1_err, "adam m")
        R.check("optimizer", m.accum2.double(), v1, v1_err, "adam v")
    else:
        l1, l2, l2s = f32(d["l1_regularization_strength"]), f32(d["l2_regularization_strength"]), \
            f32(d["l2_shrinkage_regularization_strength"])
        lrp, beta = f32(d["learning_rate_power"]), f32(d["beta"])
        adj_l2 = l2 + beta / lr * 0.5
        gs = gr + 2 * l2s * w
        an = a + gr * gr
        pa, po = an.pow(-lrp), a.pow(-lrp)
        sigma = (pa - po) / lr
        t = sigma * w
        b1_ = b + gs - t
        quad = pa / lr + 2 * adj_l2
        w1 = (b1_.clamp(-l1, l1) - b1_) / quad
        # first-order propagation of the roundings: powf within POW_ULP ulp, every other operation within 1 ulp
        pa_err, po_err = POW_ULP * u * pa, POW_ULP * u * po
        sigma_err = (pa_err + po_err + u * (pa - po).abs()) / lr + u * sigma.abs()
        t_err = sigma_err * w.abs() + u * t.abs()
        b_err = C_ACC * u * (b.abs() + gs.abs() + t.abs() + b1_.abs()) + t_err
        quad_err = pa_err / lr + u * quad
        w_err = (b_err + u * (b1_.clamp(-l1, l1) - b1_).abs()) / quad + w1.abs() * (quad_err / quad + C_ACC * u)
        R.check("optimizer", m.theta.double(), w1, w_err, "ftrl theta")
        R.check("optimizer", m.accum.double(), an, 2 * u * an, "ftrl accum")
        R.check("optimizer", m.accum2.double(), b1_, b_err, "ftrl linear")
    for l in range(len(m.hidden)):
        W = m.view("W%d" % l).view(m.Hp[l], -1)
        assert _bits_equal(m.Wb[l], W.to(torch.bfloat16)), ("optimizer: Wb != bf16(theta)", l)
        assert _bits_equal(m.WTb[l], m.Wb[l].t()), ("optimizer: WTb != Wb^T", l)
    assert bool((m.gtheta == 0).all()), "optimizer: gradients not cleared"


def _record(record_property, ratios):
    for k, v in ratios.items():
        record_property(k, v)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_fused_stages_match_fp64(cuda_context, record_property, name):
    _record(record_property, run_stages(name))


# the two partial-FM-group layouts under every GEMM path the step can take
PATHS = {"chain_fwd_bwd": {"EXB_GEMM_CHAIN": "1"},       # forward and backward chains
         "single_launch": {"EXB_GEMM_CHAIN": "0"},       # one launch per GEMM, MN-major dW
         "k_major": {"EXB_MN_MAJOR": "0"}}               # A0T / HT / dZT copies, K-major dW, prep A, head A + B


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("name", ["fm26_d8", "fm26_d9_cache"])
def test_fused_stages_gemm_paths(cuda_context, record_property, monkeypatch, name, path):
    for k, v in PATHS[path].items():
        monkeypatch.setenv(k, v)
    _record(record_property, run_stages(name))


@pytest.mark.parametrize("name", ["fm26_d8", "fm26_d9_cache"])
def test_fused_stages_wide_tile(cuda_context, record_property, name):
    """EXB_GEMM_BN=128 (read once per process, hence the subprocess) with one launch per GEMM"""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import openembedding_b200 as oe\n"
            "from openembedding_b200.context import reset_context\n"
            "oe.flags.device = 'cuda'; reset_context()\n"
            "import test_gpu_fused_stages as T\n"
            "print('STAGES ' + json.dumps(T.run_stages(%r)))\n" % (os.path.dirname(here), here, name))
    env = dict(os.environ, EXB_GEMM_BN="128", EXB_GEMM_CHAIN="0")
    r = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600)
    lines = [x for x in r.stdout.splitlines() if x.startswith("STAGES ")]
    assert r.returncode == 0 and lines, r.stdout[-3000:]
    _record(record_property, json.loads(lines[-1][len("STAGES "):]))
