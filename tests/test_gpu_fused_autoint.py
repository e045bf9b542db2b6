"""The fused AutoInt step (FusedCTR model="autoint": stacked field self-attention inside the one graph-captured step).

``run_stages`` checks every attention stage of one step against float64, with the method and the bound constants of
test_gpu_fused_stages.py. Every layer keeps its own buffers (operand, projections, softmax, output, gradient operand,
input gradient), so each stage is checked on what the step left behind, from the inputs the kernels actually read.
Values made by one rounded operation on stored inputs are compared bit for bit (the gather, the bf16 copies, dR, the
fold), sums within a derived bound. The other tests check the whole step against ``FusedCTR.reference()`` (the eager
zoo's ``InteractingLayer`` in fp32 autograd), the dense optimizer over the attention matrices against the Keras
formulas, the graph / prefetch drivers, the constructor checks, the launch count, predict, resume and the export.
"""
import copy
import ctypes
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

from test_gpu_fused_stages import (BF16_ULP, C_ACC, DENSE_OPT, U32, _batch, _bits_equal, _check_optimizer, _dot_bound,
                                   _Ratios, _record)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_VOCAB = [1000, 50, 20000, 7, 3000] + [300] * 21     # 26 features; cache 64 -> features 1 and 3 replicated

CONFIGS = {
    # Dp 12 != D 9, cached features folded through cachegrad; DeepCTR's defaults (3 layers, d 8, 2 heads, residual)
    "d26_d9_cache": dict(vocab=BASE_VOCAB, dim=9, cache=64, att={}, dense_opt="adagrad"),
    # the benchmark layout (dim 64) at batch 256
    "d26_d64_cache": dict(vocab=BASE_VOCAB, dim=64, cache=64, att={}, dense_opt="adam"),
    # one layer without residual (Np = r(3 dh, 64)) and without dense features
    "d7_d16_1layer_nores_nodense": dict(vocab=BASE_VOCAB[:7], dim=16, cache=0, nd=0, dense_opt="ftrl",
                                        att=dict(att_layers=1, att_res=False)),
    # four attention layers beside a four-layer DNN: all 8 matrices of the dense optimizer
    "d5_d12_4layers_cache": dict(vocab=BASE_VOCAB[:5], dim=12, cache=64, hidden=(64, 48, 32, 16), dense_opt="adagrad",
                                 att=dict(att_layers=4)),
    # one head with d * h = 64 (Np 256), D above 64 (layer 0's operand has 128 columns)
    "d6_d70_1head64_cache": dict(vocab=BASE_VOCAB[:6], dim=70, cache=64, dense_opt="adam",
                                 att=dict(att_layers=2, att_embedding_size=64, att_head_num=1)),
    # nf at the kernels' maximum of 64 fields
    "d64_d8_maxfields": dict(vocab=BASE_VOCAB + [500] * 38, dim=8, cache=64, dense_opt="ftrl", att={}),
}


def _model(cfg, B, **kw):
    from openembedding_b200.models.fused_dense import FusedCTR
    args = dict(num_dense=cfg.get("nd", 13), embedding_dim=cfg["dim"], model="autoint", batch=B,
                cache_threshold=cfg["cache"], hidden=cfg.get("hidden"), **cfg["att"])
    args.update(kw)
    return FusedCTR(cfg["vocab"], **args)


def _zero_outside_real(m):
    """every entry of a stacked attention matrix outside its real rows and columns is bit-zero"""
    nmat = 4 if m.att_res else 3
    for l in range(m.att_layers):
        W = m.aview(l).clone()
        W[:m.D if l == 0 else m.att_dh, :nmat * m.att_dh] = 0
        assert bool((W == 0).all()), ("attention matrix outside the real block", l)


def _fill_cache(m, seed=7):
    if m.nc:
        g = torch.Generator().manual_seed(seed)
        ce = torch.randn(m.cache_rows, m.Dp, generator=g) * 0.3
        ce[:, m.D:] = 0
        m.view("cache_emb").copy_(ce.reshape(-1).to(m.dev))


def _fresh_att_weights(m, seed=11):
    """attention weights large enough that the softmax is far from uniform, and a fresh w_att. Keras FTRL's first
    update rebuilds each weight from its accumulators alone, so after warm-up steps the initial weights may be gone"""
    g = torch.Generator().manual_seed(seed)
    dh, nmat = m.att_dh, 4 if m.att_res else 3
    for l in range(m.att_layers):
        d_in = m.D if l == 0 else dh
        m.aview(l)[:d_in, :nmat * dh] = (torch.randn(d_in, nmat * dh, generator=g) * (1.5 / d_in) ** 0.5).to(m.dev)
    T = m.nf * dh
    m.view("watt")[:] = (torch.randn(T, generator=g) * (2.0 / (T + 1)) ** 0.5).to(m.dev)
    m.refresh_weights()


def run_stages(name, B=256):
    """One step without update on the model of CONFIGS[name]; every attention stage checked. Returns the error/bound
    ratio per stage."""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import _att_lib
    from openembedding_b200.ops import gemm as G
    cfg = CONFIGS[name]
    ctx = get_context()
    dev = ctx.device
    nd = cfg.get("nd", 13)
    m = _model(cfg, B, sparse_optimizer={"category": "adam", "learning_rate": 0.2},
               dense_optimizer=dict(DENSE_OPT[cfg["dense_opt"]]), dw_splits=2)
    nf, Dp, D, La, h, dh, Np = m.nf, m.Dp, m.D, m.att_layers, m.att_h, m.att_dh, m.att_Np
    d, res, Kp = m.att_d, m.att_res, m.att_Kp
    nblk = 4 if res else 3
    _fill_cache(m)
    for s in range(2):
        m.forward_backward(*[t.to(dev) for t in _batch(cfg["vocab"], B, nd, seed=s)])
    _zero_outside_real(m)
    _fresh_att_weights(m)
    ids, dense, labels = [t.to(dev) for t in _batch(cfg["vocab"], B, nd, seed=99)]
    m.forward_backward(ids, dense, labels, update=False)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    G.check()

    R = _Ratios()
    f64, f32, bf16 = torch.float64, torch.float32, torch.bfloat16
    dd = lambda t: t.detach().to(f64)
    lib, st = _att_lib(), torch.cuda.current_stream(dev).cuda_stream
    heads = lambda t: t.reshape(B, nf, h, d).transpose(1, 2)          # [B*nf, dh] -> [B, h, nf, d]

    # ---------------- gather: bf16 of the embedding columns of X32 (server and cached rows), zero-padded
    want = torch.zeros(B * nf, Kp[0], dtype=f32, device=dev)
    want[:, :D] = m.X32[:, :nf * Dp].reshape(B * nf, Dp)[:, :D]
    assert _bits_equal(m.att_X[0], want.to(bf16)), "gather"

    # ---------------- forward, layer by layer
    for l in range(La):
        assert _bits_equal(m.aWb[l], m.aview(l).to(bf16)), ("aWb != bf16(theta)", l)
        assert _bits_equal(m.aWTb[l], m.aWb[l].t()), ("aWTb != aWb^T", l)
        A, Wt = dd(m.att_X[l]), dd(m.aWTb[l]).t()
        ref = A @ Wt
        R.check("att_proj", dd(m.att_QKVR[l]), ref, _dot_bound(A, Wt) + U32 * ref.abs(), "QKVR%d" % l)
        qkvr = dd(m.att_QKVR[l])
        q, k, v = (heads(qkvr[:, i * dh:(i + 1) * dh]) for i in range(3))
        S = q @ k.transpose(-1, -2)                                   # [B, h, nf, nf]
        dS_row = (C_ACC * d * U32 * (q.abs() @ k.abs().transpose(-1, -2))).amax(-1, keepdim=True)
        P = torch.softmax(S, -1)
        # first order: rel. error of p_j <= |e_j| + |sum_k p_k e_k| with e the error of s_j - max, plus expf (2 ulp),
        # the fp32 sum of the exponentials and the division; 2^-140 covers quotients in the subnormal range
        R.check("att_softmax", dd(m.att_P[l]), P, P * (4 * dS_row + (C_ACC * nf + 8) * U32) + 2.0 ** -140, "P%d" % l)
        Pk = dd(m.att_P[l])
        o = Pk @ v
        ob = C_ACC * nf * U32 * (Pk.abs() @ v.abs())
        o = o.transpose(1, 2).reshape(B * nf, dh)
        ob = ob.transpose(1, 2).reshape(B * nf, dh)
        pre = o + (qkvr[:, 3 * dh:4 * dh] if res else 0)
        R.check("att_out", dd(m.att_Xf[l]), pre.clamp(min=0), ob + U32 * pre.abs(), "X%d" % (l + 1))
        if l < La - 1:
            want = torch.zeros(B * nf, Kp[l + 1], dtype=f32, device=dev)
            want[:, :dh] = m.att_Xf[l]
            assert _bits_equal(m.att_X[l + 1], want.to(bf16)), ("X_{l+1} bf16 != bf16(Xf), zero pad", l)

    # ---------------- base increment flatten(X_L) . w_att: the last forward launch once more on top of the base
    XL = m.att_Xf[-1].clone()
    base0 = m.base.clone()
    assert lib.exb_att_fwd(ctypes.byref(m._att_fwd_args[-1]), st) == 0
    torch.cuda.synchronize()
    assert _bits_equal(m.att_Xf[-1], XL), "att_fwd: X_L differs between two launches"
    XL64, w64 = dd(XL).view(B, nf * dh), dd(m.view("watt"))
    inc_ref = XL64 @ w64
    inc_bound = C_ACC * nf * dh * U32 * (XL64.abs() @ w64.abs()) + U32 * dd(m.base).abs()
    R.check("att_base", dd(m.base) - dd(base0), inc_ref, inc_bound, "base increment")
    m.base.copy_(base0)

    # ---------------- backward, layer by layer from the last
    dl = m.dlogit
    for l in range(La - 1, -1, -1):
        if l == La - 1:
            g = dl.repeat_interleave(nf)[:, None] * m.view("watt").view(nf, dh).repeat(B, 1)     # one rounding
        else:
            g = m.att_dX[l + 1][:, :dh]
        dy = torch.where(m.att_Xf[l] > 0, g, torch.zeros_like(g))
        dq = m.att_dQKVR[l]
        if res:
            assert _bits_equal(dq[:, 3 * dh:4 * dh], dy.to(bf16)), ("dR != bf16(dY)", l)
        assert bool((dq[:, nblk * dh:] == 0).all()), ("dQKVR pad columns", l)
        qkvr = dd(m.att_QKVR[l])
        q, k, v = (heads(qkvr[:, i * dh:(i + 1) * dh]) for i in range(3))
        Pk, go = dd(m.att_P[l]), heads(dd(dy))
        dP = go @ v.transpose(-1, -2)
        dP_b = C_ACC * d * U32 * (go.abs() @ v.abs().transpose(-1, -2))
        t = (dP * Pk).sum(-1, keepdim=True)
        t_b = (Pk * dP_b).sum(-1, keepdim=True) + C_ACC * nf * U32 * (dP * Pk).abs().sum(-1, keepdim=True)
        dS = Pk * (dP - t)
        dS_b = Pk * (dP_b + t_b + U32 * (dP - t).abs()) + U32 * dS.abs()
        for i, (ref, bound, what) in enumerate((
                (dS @ k, dS_b @ k.abs() + C_ACC * nf * U32 * (dS.abs() @ k.abs()), "dQ"),
                (dS.transpose(-1, -2) @ q, dS_b.transpose(-1, -2) @ q.abs()
                 + C_ACC * nf * U32 * (dS.abs().transpose(-1, -2) @ q.abs()), "dK"),
                (Pk.transpose(-1, -2) @ go, C_ACC * nf * U32 * (Pk.transpose(-1, -2) @ go.abs()), "dV"))):
            ref = ref.transpose(1, 2).reshape(B * nf, dh)
            bound = bound.transpose(1, 2).reshape(B * nf, dh)
            R.check("att_" + what, dd(dq[:, i * dh:(i + 1) * dh]), ref, bound + BF16_ULP * (ref.abs() + bound),
                    "%s%d" % (what, l))
        # weight gradient (split-K into gtheta) and input gradient
        A, Dq = dd(m.att_X[l]), dd(dq)
        ref = A.t() @ Dq
        R.check("att_dW", dd(m.aview(l, grad=True)), ref, _dot_bound(A.t(), Dq), "T%d" % l)
        Wt = dd(m.aWb[l]).t()
        ref = Dq @ Wt
        R.check("att_dX", dd(m.att_dX[l]), ref, _dot_bound(Dq, Wt) + U32 * ref.abs(), "dX%d" % l)

    # ---------------- g_watt: the partial sums per 128 samples, the step's sum, and the fold launched once more
    T = nf * dh
    XLs, dl64 = dd(m.att_Xf[-1]).view(B, T), dd(dl)
    for c in range(m.att_gpart.shape[0]):
        rows = slice(128 * c, min(128 * (c + 1), B))
        ref = dl64[rows] @ XLs[rows]
        R.check("att_gwatt", dd(m.att_gpart[c]), ref, C_ACC * 128 * U32 * (dl64[rows].abs() @ XLs[rows].abs()),
                "partial %d" % c)
    ref = dl64 @ XLs
    R.check("att_gwatt", dd(m.gview("watt")), ref, C_ACC * B * U32 * (dl64.abs() @ XLs.abs()), "g_watt")
    G32_0, gw0 = m.G32.clone(), m.gview("watt").clone()
    assert lib.exb_att_fold(m.G32.data_ptr(), m.XS, Dp, D, nf, m.att_dX[0].data_ptr(), Kp[0], B,
                            m.att_gpart.data_ptr(), T, m.gview("watt").data_ptr(), st) == 0
    torch.cuda.synchronize()
    emb = G32_0[:, :nf * Dp].reshape(B * nf, Dp).clone()
    emb[:, :D] = emb[:, :D] + m.att_dX[0][:, :D]
    want = G32_0.clone()
    want[:, :nf * Dp] = emb.reshape(B, nf * Dp)
    assert _bits_equal(m.G32, want), "fold: G32 != G32 + dX_0 on the real embedding columns"
    s = torch.zeros(T, dtype=f32, device=dev)
    for c in range(m.att_gpart.shape[0]):
        s = s + m.att_gpart[c]
    assert _bits_equal(m.gview("watt"), gw0 + s), "fold: g_watt != g_watt + the partial sums in chunk order"
    m.G32.copy_(G32_0)
    m.gview("watt").copy_(gw0)

    # ---------------- dense optimizer over DNN + attention matrices and the flat region (w_att)
    _check_optimizer(m, R)
    for l in range(La):
        assert _bits_equal(m.aWb[l], m.aview(l).to(bf16)), ("optimizer: aWb", l)
        assert _bits_equal(m.aWTb[l], m.aWb[l].t()), ("optimizer: aWTb", l)
    _zero_outside_real(m)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    G.check()
    return dict(R)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_fused_autoint_stages_match_fp64(cuda_context, record_property, name):
    _record(record_property, run_stages(name))


def _grads_match_reference(m, ids, dense, labels, loss):
    ref_loss, g = m.reference(ids, dense, labels)
    assert abs(float(loss) - float(ref_loss)) < 5e-3, (float(loss), float(ref_loss))
    names = ["W%d" % l for l in range(len(m.hidden))] + ["T%d" % l for l in range(m.att_layers)]
    for name_ in names + ["wout", "bias", "watt"] + (["wd"] if m.nd else []) + (["cache_emb", "cache_lin"] if m.nc else []):
        o, n = m.segs[name_]
        a, b = m.gtheta[o:o + n], g["theta"][o:o + n]
        err = float((a - b).abs().max())
        scale = float(b.abs().max()) + 1e-6
        assert err < 0.05 * scale + 2e-4, (name_, err, scale)
    ge = m.G32[:, :m.ns * m.Dp]
    err = float((ge - g["emb"]).abs().max())
    assert err < 0.05 * float(g["emb"].abs().max()) + 2e-5, err
    gl = m.G32[:, m.lin0:m.lin0 + m.ns]
    assert torch.allclose(gl, g["lin"], atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_fused_autoint_step_matches_reference(cuda_context, name):
    from openembedding_b200.context import get_context
    ctx = get_context()
    cfg = CONFIGS[name]
    B, nd = 256, cfg.get("nd", 13)
    m = _model(cfg, B, lr=0.05, sparse_optimizer={"category": "adagrad", "learning_rate": 0.05}, dw_splits=2)
    _fill_cache(m)
    for s in range(3):
        m.forward_backward(*[t.to(ctx.device) for t in _batch(cfg["vocab"], B, nd, seed=s)])
    ids, dense, labels = [t.to(ctx.device) for t in _batch(cfg["vocab"], B, nd, seed=99)]
    loss = m.forward_backward(ids, dense, labels, update=False)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    _grads_match_reference(m, ids, dense, labels, loss)


@pytest.mark.parametrize("cfg,name", [({"category": "adam", "learning_rate": 0.01}, "d26_d9_cache"),
                                      ({"category": "ftrl", "learning_rate": 0.05, "l1_regularization_strength": 0.001},
                                       "d5_d12_4layers_cache"),
                                      ({"category": "adagrad", "learning_rate": 0.05}, "d5_d12_4layers_cache")])
def test_fused_autoint_dense_optimizers_match_keras(cuda_context, cfg, name):
    """exb_dense_opt_kernel over 6 (DNN 3 + attention 3) or 8 (4 + 4) refreshed matrices vs the Keras formulas"""
    from test_optimizers import keras_reference
    from openembedding_b200.context import get_context
    ctx = get_context()
    B = 256
    m = _model(CONFIGS[name], B, sparse_optimizer={"category": "adagrad", "learning_rate": 0.05},
               dense_optimizer=dict(cfg))
    assert m._opt_args.nmat == len(m.hidden) + m.att_layers >= 6
    theta0 = m.theta.detach().cpu().double().clone()
    grads = []
    for s in range(4):
        b = [t.to(ctx.device) for t in _batch(CONFIGS[name]["vocab"], B, 13, seed=s)]
        m.forward_backward(*b, update=False)
        torch.cuda.synchronize()
        grads.append(m.gtheta.detach().cpu().double().clone())
        m.forward_backward(*b, update=True)
        torch.cuda.synchronize()
    ctx.backend.engine.check()
    ref = keras_reference(cfg, theta0.view(1, -1), [g.view(1, -1) for g in grads]).view(-1)
    got = m.theta.detach().cpu().double()
    err = float((got - ref).abs().max())
    moved = float((ref - theta0).abs().max())
    assert moved > 1e-4 and err < 2e-2 * moved + 1e-6, (cfg, err, moved)
    for l in range(m.att_layers):
        o, n = m.segs["T%d" % l]
        assert float((ref[o:o + n] - theta0[o:o + n]).abs().max()) > 0, ("attention matrix did not move", l)
        assert torch.equal(m.aWb[l], m.aview(l).to(torch.bfloat16)), ("bf16 refresh", l)
    _zero_outside_real(m)


@pytest.mark.parametrize("dense_opt", ["adagrad", "ftrl"])
def test_fused_autoint_graph_equals_eager_and_warmup_is_neutral(cuda_context, dense_opt):
    from openembedding_b200.context import get_context, reset_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg = CONFIGS["d26_d9_cache"]
    B = 256
    curves = []
    for graph in (False, True):
        reset_context()
        ctx = get_context()
        m = _model(cfg, B, lr=0.05, sparse_optimizer={"category": "adagrad", "learning_rate": 0.05},
                   dense_optimizer={"category": dense_opt, "learning_rate": 0.05})
        batches = [[t.to(ctx.device) for t in _batch(cfg["vocab"], B, 13, seed=s)] for s in range(3)]
        if graph:
            theta0, acc0 = m.theta.clone(), m.accum.clone()
            m.warmup(*batches[0])
            torch.cuda.synchronize()
            assert torch.equal(m.theta, theta0) and torch.equal(m.accum, acc0)
            assert int(m.opt_step.item()) == 0
            for l in range(m.att_layers):
                assert torch.equal(m.aWb[l], m.aview(l).to(torch.bfloat16)), l
        tr = FusedTrainer(m, use_graph=graph)
        curves.append([float(tr.step(*batches[k % 3])) for k in range(7)])
        torch.cuda.synchronize()
        ctx.backend.engine.check()
    assert curves[0][-1] < curves[0][0], curves
    for a, b in zip(*curves):
        assert abs(a - b) < 2e-4, curves


@pytest.mark.parametrize("graph", [False, True])
def test_fused_autoint_prefetch_matches_plain(cuda_context, graph):
    from openembedding_b200.context import get_context, reset_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg = CONFIGS["d26_d9_cache"]
    B = 256
    curves = []
    for prefetch in (False, True, "stable"):
        reset_context()
        ctx = get_context()
        m = _model(cfg, B, lr=0.05, sparse_optimizer={"category": "adagrad", "learning_rate": 0.05})
        tr = FusedTrainer(m, use_graph=graph)
        batches = [[t.to(ctx.device) for t in _batch(cfg["vocab"], B, 13, seed=s)] for s in range(4)]
        order = [0, 1, 2, 3, 0, 2, 1, 3, 3, 0]
        losses = []
        for k, i in enumerate(order):
            nxt = None
            if prefetch and k + 1 < len(order) and k != 4:
                nxt = batches[order[k + 1]][0]
            if prefetch and k == 6:                 # announce one batch, train another
                nxt = batches[0][0]
            losses.append(float(tr.step(*batches[i], next_ids=nxt, stable=prefetch == "stable")))
        torch.cuda.synchronize()
        ctx.backend.engine.check()
        curves.append(losses)
    for a, b, c in zip(*curves):
        assert abs(a - b) < 2e-4 and abs(a - c) < 2e-4, curves


@pytest.mark.parametrize("kw,match", [(dict(att_layers=0), "at least one"),
                                      (dict(att_layers=6), "weight matrices"),                 # 3 DNN + 6 > 8
                                      (dict(att_layers=4, hidden=(64,) * 5), "weight matrices"),
                                      (dict(att_embedding_size=33, att_head_num=2), "above 64"),
                                      (dict(att_head_num=0), "positive"),
                                      (dict(vocab=[300] * 65), "fields")])
def test_fused_autoint_constructor_errors(cuda_context, kw, match):
    from openembedding_b200.models.fused_dense import FusedCTR
    kw = dict(kw)
    vocab = kw.pop("vocab", BASE_VOCAB)
    with pytest.raises(ValueError, match=match):
        FusedCTR(vocab, embedding_dim=8, model="autoint", batch=256, **kw)


def _profiled_step_kernels():
    """names of the kernels two eager steps of CONFIGS["d26_d9_cache"] launch, and kernels_per_step(); run in a
    subprocess of its own (test_fused_autoint_kernels_per_step)"""
    from torch.profiler import ProfilerActivity, profile
    from openembedding_b200.context import get_context
    dev = get_context().device
    cfg = CONFIGS["d26_d9_cache"]
    m = _model(cfg, 256)
    b = [t.to(dev) for t in _batch(cfg["vocab"], 256, 13, seed=0)]
    m.forward_backward(*b)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            m.forward_backward(*b)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and not e.name.startswith(("Memcpy", "Memset"))]
    return {"names": names, "per_step": m.kernels_per_step(), "att_layers": m.att_layers}


def test_fused_autoint_kernels_per_step(cuda_context):
    """the attention adds 2 + 5 launches per layer to the WDL-shaped step around it, 1 + 2 per layer to the
    evaluation pass; the step's count is a torch.profiler count of two eager steps. The profiler runs in a subprocess:
    a profiling session changes what later sessions of the same process record of graph replays, and other test files
    count graph replays with the profiler."""
    from openembedding_b200.models.fused_dense import FusedCTR
    kw = dict(embedding_dim=8, batch=256, hidden=(64, 32))
    wdl = FusedCTR(BASE_VOCAB, model="wdl", **kw)
    m3 = FusedCTR(BASE_VOCAB, model="autoint", att_layers=3, **kw)
    assert m3.kernels_per_step() == wdl.kernels_per_step() + 17
    assert m3.kernels_per_eval() == wdl.kernels_per_eval() + 7
    assert FusedCTR(BASE_VOCAB, model="autoint", att_layers=1, **kw).kernels_per_step() == wdl.kernels_per_step() + 7
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import openembedding_b200 as oe\n"
            "from openembedding_b200.context import reset_context\n"
            "oe.flags.device = 'cuda'; reset_context()\n"
            "import test_gpu_fused_autoint as T\n"
            "print('KERNELS ' + json.dumps(T._profiled_step_kernels()))\n" % (ROOT, here))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    lines = [x for x in r.stdout.splitlines() if x.startswith("KERNELS ")]
    assert r.returncode == 0 and lines, r.stdout[-3000:]
    out = json.loads(lines[-1][len("KERNELS "):])
    names = out["names"]
    assert len(names) == 2 * out["per_step"], (out["per_step"], names)
    assert sum("exb_att_" in n for n in names) == 2 * (2 + 2 * out["att_layers"]), names     # gather, fwd, bwd, fold


def test_fused_autoint_predict_matches_reference(cuda_context):
    """predict's logits against reference() on the rows the stateless pull left in X32; no parameter, optimizer
    state, gradient or loss changes"""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg = CONFIGS["d26_d9_cache"]
    B = 256
    dev = get_context().device
    m = _model(cfg, B, lr=0.05, sparse_optimizer={"category": "adam", "learning_rate": 0.2},
               dense_optimizer={"category": "adam", "learning_rate": 0.01})
    _fill_cache(m)
    tr = FusedTrainer(m, use_graph=True)
    for s in range(3):
        tr.step(*[t.to(dev) for t in _batch(cfg["vocab"], B, 13, seed=s)])
    torch.cuda.synchronize()
    state = [t.clone() for t in (m.theta, m.accum, m.accum2, m.opt_step, m.gtheta, m.loss)]
    ids, dense, labels = [t.to(dev) for t in _batch(cfg["vocab"], B, 13, seed=42)]
    p = tr.predict(ids, dense)
    z = m.logits.clone()
    torch.cuda.synchronize()
    for a, b in zip(state, (m.theta, m.accum, m.accum2, m.opt_step, m.gtheta, m.loss)):
        assert torch.equal(a, b)
    assert torch.equal(p, torch.sigmoid(z))
    _, _, zr = m.reference(ids, dense, labels, return_logits=True)
    assert bool(((z - zr).abs() <= 1e-2 * (1 + zr.abs())).all()), float((z - zr).abs().max())


def test_fused_autoint_resume_equals_uninterrupted(cuda_context, tmp_path):
    """save after 3 of 6 batches in the middle of a graph-driven pipeline (prefetch armed): a model built with another
    seed in a fresh context loads exactly the state of the save, bit for bit (dense buffers with the optimizer state,
    table rows), and the other 3 batches then train as the uninterrupted run does.

    The step's atomics make two runs of the same trajectory differ, and Adam turns the ulp-level noise of an almost
    dead unit into steps of up to the learning rate, so the largest difference between two runs is heavy-tailed. The
    trajectory check therefore compares the mean difference to the uninterrupted run with the one of a resume that lost
    the dense optimizer state (a weights-only checkpoint): a correct resume is far closer."""
    from test_gpu_fused_eval import _rows, _rows_equal
    from openembedding_b200.context import get_context, reset_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg, B, k = CONFIGS["d26_d9_cache"], 256, 3
    batches = [[t.pin_memory() for t in _batch(cfg["vocab"], B, 13, seed=s)] for s in range(2 * k)]
    ck, ckw = str(tmp_path / "ck"), str(tmp_path / "weights")
    dense = lambda m: [t.detach().clone().cpu() for t in (m.theta, m.accum, m.accum2, m.opt_step)]

    def model(seed):
        reset_context()
        ctx = get_context()
        m = _model(cfg, B, seed=seed, sparse_optimizer={"category": "adam", "learning_rate": 0.2},
                   dense_optimizer={"category": "adam", "learning_rate": 0.01}, dw_splits=2)
        _fill_cache(m, 7 + seed)
        return ctx, m

    def run(bs, seed=0, load=None, save_at=None):
        ctx, m = model(seed)
        if load:
            m.load(load)
        tr = FusedTrainer(m, use_graph=True)
        pipe = tr.make_pipeline(B, m.nf, m.nd)
        at_save = None
        for b in bs:
            pipe.submit(*b)
            if save_at is not None and pipe.trained == save_at:
                assert tr._x32_key is not None              # a prefetch is armed
                m.save(ck)
                m.save(ckw, include_optimizer=False)
                at_save = (dense(m), _rows(ctx, m))
                save_at = None
        loss = pipe.last_loss()
        torch.cuda.synchronize()
        ctx.backend.engine.check()
        return loss, dense(m), at_save

    plain_loss, plain, at_save = run(batches, save_at=k)
    ctx, m = model(1)                                        # the load restores the state of the save exactly
    m.load(ck)
    torch.cuda.synchronize()
    for a, b in zip(at_save[0], dense(m)):
        assert torch.equal(a, b)
    _rows_equal(at_save[1], _rows(ctx, m))
    resumed_loss, resumed, _ = run(batches[k:], seed=1, load=ck)
    _, stateless, _ = run(batches[k:], seed=1, load=ckw)
    assert torch.equal(resumed[3], plain[3])                 # the optimizer step counter
    mean = lambda a, b: float((a.double() - b.double()).abs().mean())
    for i, name in enumerate(("theta", "m", "v")):
        good, lost = mean(resumed[i], plain[i]), mean(stateless[i], plain[i])
        assert good <= 0.25 * lost, (name, good, lost)
    assert abs(resumed_loss - plain_loss) <= 1e-3, (resumed_loss, plain_loss)


def _rounding_bound(mod, ids, dense):
    """per-sample first-order bound on |fused logit - fp32 logit| from the fused path's bf16 rounding points (as in
    test_gpu_fused_checkpoint.py): the DNN's and the attention's weights, the DNN's layer inputs and every attention
    layer's input, each taken at 2^-8 |dz/dv| |v| (twice the first-order term, for the higher orders)"""
    from torch import nn
    from openembedding_b200.models.ctr import InteractingLayer
    mod = copy.deepcopy(mod).double()
    acts = []

    def grab(t):
        t = t.clone() if t.requires_grad else t.detach().clone().requires_grad_(True)
        t.retain_grad()
        acts.append(t)
        return t

    hooks = [mm.register_forward_pre_hook(lambda m_, args: (grab(args[0]),)) for mm in mod.modules()
             if isinstance(mm, (nn.Linear, InteractingLayer))]
    rounded = [p for n, p in mod.named_parameters() if n.startswith(("dnn.", "att."))]
    out = []
    for b in range(ids.shape[0]):
        acts.clear()
        mod.zero_grad()
        z = mod(ids[b:b + 1], dense[b:b + 1].double())
        z.sum().backward()
        s = sum(float((p.grad * p.detach()).abs().sum()) for p in rounded)
        s += sum(float((a.grad * a).abs().sum()) for a in acts if a.grad is not None)
        out.append(s)
    for h_ in hooks:
        h_.remove()
    return torch.tensor(out, dtype=torch.float64)


def test_fused_autoint_export_matches_predict(cuda_context, tmp_path):
    """the stand-alone export holds the model's dense tensors bit for bit (dnn_out.bias folded into bias) and its
    logits agree with predict within the bf16 rounding bound"""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg, B = CONFIGS["d26_d9_cache"], 256
    dev = get_context().device
    m = _model(cfg, B, sparse_optimizer={"category": "adam", "learning_rate": 0.2},
               dense_optimizer={"category": "adam", "learning_rate": 0.01})
    _fill_cache(m)
    tr = FusedTrainer(m, use_graph=True)
    for s in range(4):
        tr.step(*[t.to(dev) for t in _batch(cfg["vocab"], B, 13, seed=s)])
    torch.cuda.synchronize()
    path = str(tmp_path / "export" / "model.pt")
    mod = m.save_as_original_model(path)
    assert os.path.exists(path) and type(mod).__name__ == "StandaloneCTR"
    sd, got = m.dense_state_dict(include_optimizer=False), mod.state_dict()
    for k, v in sd.items():
        if k != "dnn_out.bias":
            assert torch.equal(got[k], v + sd["dnn_out.bias"] if k == "bias" else v), k
    ids, dense, _ = [t.to(dev) for t in _batch(cfg["vocab"], B, 13, seed=99)]
    tr.predict(ids, dense)
    zf = m.logits.detach().double().cpu()
    with torch.no_grad():
        ze = mod.cpu()(ids.cpu(), dense.cpu()).double()
    n = 48
    bound = 2.0 ** -8 * _rounding_bound(mod, ids[:n].cpu(), dense[:n].cpu())
    bound += 4 * m.K0p * 2.0 ** -24 * (bound * 2 ** 8 + ze[:n].abs()) + 1e-6
    err = (zf[:n] - ze[:n]).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    assert float((zf - ze).abs().max()) <= 1e-2 * (1 + float(ze.abs().max()))


def _torchrun(env=None):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_gpu_fused_autoint_check.py")]
    p = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600,
                       env=dict(os.environ, **(env or {})))
    return p.returncode, p.stdout


def test_mp_fused_autoint_two_ranks():
    """world 2: the loss falls, the dense replicas (attention matrices and w_att included) stay bit-identical, and the
    all-reduce riding on the push kernel gives the parameters of the stand-alone all-reduce kernel"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs on the box")
    rc, out = _torchrun()
    assert rc == 0 and "MP_GPU_FUSED_AUTOINT_PASSED" in out and "rider 1" in out, out[-4000:]
    rc2, out2 = _torchrun({"EXB_AR_RIDER": "0"})
    assert rc2 == 0 and "MP_GPU_FUSED_AUTOINT_PASSED" in out2 and "rider 0" in out2, out2[-4000:]
    tsum = lambda o: float(o.split("theta_sum ")[1].split()[0])
    assert abs(tsum(out) - tsum(out2)) < 1e-6 * abs(tsum(out2)), (tsum(out), tsum(out2))
