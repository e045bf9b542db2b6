"""The fused DCN-v2 step (FusedCTR model="dcn": the cross network inside the one graph-captured step).

``run_stages`` checks the cross kernels of one step stage by stage against float64, with the method and the bound
constants of test_gpu_fused_stages.py. The forward buffers of every layer stay in the model after a step; the backward
keeps only a ping-pong of g and one dU / P buffer, so its launches are replayed one at a time on the step's state and
each result is checked before the next launch overwrites it. Values the kernels compute with one rounded operation on
stored inputs are compared bit for bit, sums within a derived bound. The other tests check the whole step against
``FusedCTR.reference()`` (the eager zoo's CrossNetV2 in fp32 autograd), the dense optimizer over the cross matrices
against the Keras formulas, the graph / prefetch drivers and the constructor checks.
"""
import ctypes
import os
import socket
import subprocess
import sys

import pytest
import torch

from test_gpu_fused_stages import (C_ACC, DENSE_OPT, U32, _batch, _bits_equal, _check_optimizer, _dot_bound, _Ratios,
                                   _record)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_VOCAB = [1000, 50, 20000, 7, 3000] + [300] * 21     # 26 features; cache 64 -> features 1 and 3 replicated

CONFIGS = {
    # Dp 12 != D 9: embedding pad columns inside the cross layout, cached features folded through cachegrad
    "d26_d9_cache": dict(vocab=BASE_VOCAB, dim=9, cache=64, cross=3, dense_opt="adagrad"),
    # the benchmark layout (dim 64, K0p 1728) at batch 256
    "d26_d64_cache": dict(vocab=BASE_VOCAB, dim=64, cache=64, cross=3, dense_opt="adam"),
    # one cross layer (the top launch feeds layer 0 directly) and no dense features
    "d7_d16_1layer_nodense": dict(vocab=BASE_VOCAB[:7], dim=16, cache=0, cross=1, nd=0, dense_opt="ftrl"),
    # four cross layers beside a four-layer DNN: all 8 matrices of the dense optimizer
    "d5_d12_4layers_cache": dict(vocab=BASE_VOCAB[:5], dim=12, cache=64, cross=4, hidden=(64, 48, 32, 16),
                                 dense_opt="adagrad"),
}


def _model(cfg, B, **kw):
    from openembedding_b200.models.fused_dense import FusedCTR
    args = dict(num_dense=cfg.get("nd", 13), embedding_dim=cfg["dim"], model="dcn", batch=B,
                cache_threshold=cfg["cache"], cross_layers=cfg["cross"], hidden=cfg.get("hidden"))
    args.update(kw)
    return FusedCTR(cfg["vocab"], **args)


def _zero_outside_real(m):
    """every cross-matrix entry outside the real block and its bias column, and w_cross outside the real columns,
    is bit-zero"""
    keep = torch.zeros(m.K0p, m.K0p, dtype=torch.bool, device=m.dev)
    keep[m.cross_real[:, None], m.cross_real[None, :]] = True
    keep[m.cross_real, m.K0p - 1] = True
    for l in range(m.cross_layers):
        assert bool((m.xview(l)[~keep] == 0).all()), ("cross matrix outside the real block", l)
    w = m.view("wcross").clone()
    w[m.cross_real] = 0
    assert bool((w == 0).all()), "w_cross outside the real columns"


def _fresh_cross_weights(m, seed=11):
    """glorot-normal cross matrices, biases and w_cross on the real block. Keras FTRL's first update rebuilds each
    weight from its accumulators alone (about -lr g / sqrt(a), exactly 0 under L1), so after warm-up steps the
    initial cross weights may be gone and the stage checks would see nothing"""
    g = torch.Generator().manual_seed(seed)
    n, cols = m.cross_n, m.cross_real
    for l in range(m.cross_layers):
        W = m.xview(l)
        W[cols[:, None], cols[None, :]] = (torch.randn(n, n, generator=g) * (1.0 / n) ** 0.5).to(m.dev)
        W[cols, m.K0p - 1] = (torch.randn(n, generator=g) * 0.1).to(m.dev)
    m.view("wcross")[cols] = (torch.randn(n, generator=g) * (2.0 / (n + 1)) ** 0.5).to(m.dev)
    m.refresh_weights()


def run_stages(name, B=256):
    """One step without update on the model of CONFIGS[name]; every cross stage checked. Returns the error/bound
    ratio per stage and the two sensitivity ratios."""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import _cross_lib
    from openembedding_b200.ops import gemm as G
    cfg = CONFIGS[name]
    ctx = get_context()
    dev = ctx.device
    nd = cfg.get("nd", 13)
    m = _model(cfg, B, sparse_optimizer={"category": "adam", "learning_rate": 0.2},
               dense_optimizer=dict(DENSE_OPT[cfg["dense_opt"]]), dw_splits=2)
    nf, Dp, D, K0p, Lc = m.nf, m.Dp, m.D, m.K0p, m.cross_layers
    E, ones = nf * Dp, K0p - 1
    g = torch.Generator().manual_seed(7)
    if m.nc:
        ce = torch.randn(m.cache_rows, Dp, generator=g) * 0.3
        ce[:, D:] = 0
        m.view("cache_emb").copy_(ce.reshape(-1).to(dev))
    for s in range(2):
        m.forward_backward(*[t.to(dev) for t in _batch(cfg["vocab"], B, nd, seed=s)])
    _zero_outside_real(m)
    _fresh_cross_weights(m)
    ids, dense, labels = [t.to(dev) for t in _batch(cfg["vocab"], B, nd, seed=99)]
    m.forward_backward(ids, dense, labels, update=False)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    G.check()

    R = _Ratios()
    f64, f32, bf16 = torch.float64, torch.float32, torch.bfloat16
    dd = lambda t: t.detach().to(f64)
    lib, st = _cross_lib(), torch.cuda.current_stream(dev).cuda_stream
    real = torch.zeros(K0p, dtype=torch.bool, device=dev)
    real[m.cross_real] = True
    zero = lambda t: torch.where(real[None, :], t, torch.zeros_like(t))       # the kernels' mask
    x0 = torch.zeros(B, K0p, dtype=f32, device=dev)                            # fp32 x0 on the A0 layout
    x0[:, :E] = m.X32[:, :E]
    x0[:, E:E + nd] = dense
    x0 = zero(x0)
    wc = m.view("wcross")
    dl = m.dlogit

    # ---------------- forward: Wb / WTb (bitwise), U_l, X_{l+1} and bf16 X_{l+1} (bitwise), ones and pad columns
    xin = x0
    for l in range(Lc):
        assert _bits_equal(m.xWb[l], m.xview(l).to(bf16)), ("xWb != bf16(theta)", l)
        assert _bits_equal(m.xWTb[l], m.xWb[l].t()), ("xWTb != xWb^T", l)
        src = m.A0 if l == 0 else m.cross_Xb[l - 1]
        A, Wt = dd(src), dd(m.xWb[l]).t()
        ref = A @ Wt
        R.check("cross_U", dd(m.cross_U[l]), ref, _dot_bound(A, Wt) + U32 * ref.abs(), "U%d" % l)
        want = zero(x0 * m.cross_U[l] + xin)                 # two roundings, like __fmul_rn then __fadd_rn
        want[:, ones] = 1.0
        assert _bits_equal(m.cross_Xf[l], want), ("X_{l+1} != x0 * U_l + X_l (masked, ones column 1)", l)
        if l < Lc - 1:
            assert _bits_equal(m.cross_Xb[l], want.to(bf16)), ("Xb != bf16(Xf)", l)
        xin = m.cross_Xf[l]
    assert bool((m.cross_Xf[-1][:, ones] == 1).all()) and bool((m.cross_Xf[-1][:, ~real].sum(1) == 1).all())

    # ---------------- base increment x_L . w_cross: the last forward launch once more on top of the step's base
    XL = m.cross_Xf[-1].clone()
    base0 = m.base.clone()
    assert lib.exb_cross_fwd(ctypes.byref(m._cross_fwd_args[-1]), st) == 0
    torch.cuda.synchronize()
    assert _bits_equal(m.cross_Xf[-1], XL), "cross_fwd: X_L differs between two launches"
    XL64, wc64 = dd(XL)[:, real], dd(wc)[real]
    inc_ref = XL64 @ wc64
    inc_bound = C_ACC * int(real.sum()) * U32 * (XL64.abs() @ wc64.abs()) + U32 * dd(m.base).abs()
    R.check("cross_base", dd(m.base) - dd(base0), inc_ref, inc_bound, "base increment")
    m.base.copy_(base0)
    # without the x0 * term of the last layer the increment would move by far more than its bound
    drop = (dd(x0) * dd(m.cross_U[-1]))[:, real] @ wc64
    sens_x0 = float((drop.abs() / inc_bound).nan_to_num(0.0).max())
    assert sens_x0 >= 10, ("sensitivity of the base check to the x0 * U term", sens_x0)

    # ---------------- the step's fold: G32[:, :K0p] = dZ0 @ W0 (the DNN's dX GEMM) + gx0 + g_0 on real embedding columns
    g1 = m.cross_g[1 % 2].clone()
    g0 = zero(g1 + m.cross_P)
    fold = dd(m.cross_gx0 + g0)
    fold[:, E:] = 0
    dZ0, WT0 = dd(m.dZ[0]), dd(m.WTb[0])
    mlp = dZ0 @ WT0.t()
    ref = mlp + fold
    bound = _dot_bound(dZ0, WT0.t()) + U32 * fold.abs() + U32 * ref.abs()
    R.check("cross_fold", dd(m.G32[:, :K0p]), ref, bound, "G32")
    sens_fold = float((fold.abs() / bound).nan_to_num(0.0).max())     # 0 / 0 off the fold
    assert sens_fold >= 10, ("sensitivity of the G32 check to the cross fold", sens_fold)
    step_gW = [m.xview(l, grad=True).clone() for l in range(Lc)]
    step_gwc = m.gview("wcross").clone()

    # ---------------- backward replayed launch by launch on the step's state
    for l in range(Lc):
        m.xview(l, grad=True).zero_()
    m.gview("wcross").zero_()
    m._cross_top_args.x.dense = dense.data_ptr()
    assert lib.exb_cross_bwd_top(ctypes.byref(m._cross_top_args), st) == 0
    torch.cuda.synchronize()
    gL = zero(dl[:, None] * wc[None, :])
    assert _bits_equal(m.cross_g[Lc % 2], gL), "g_L != dlogit w_cross (masked)"
    assert _bits_equal(m.cross_dU, zero(gL * x0).to(bf16)), "dU_{L-1} != bf16(g_L x0)"
    assert _bits_equal(m.cross_gx0, zero(gL * m.cross_U[-1])), "gx0 != g_L U_{L-1}"
    dl64 = dd(dl)
    ref = dl64 @ dd(XL)
    ref[~real] = 0
    R.check("cross_g_wcross", dd(m.gview("wcross")), ref, C_ACC * B * U32 * (dl64.abs() @ dd(XL).abs()), "g_wcross")
    R.check("cross_g_wcross", dd(step_gwc), ref, C_ACC * B * U32 * (dl64.abs() @ dd(XL).abs()), "step g_wcross")
    assert bool((m.gview("wcross")[~real] == 0).all()), "g_wcross outside the real columns"
    for l in range(Lc - 1, -1, -1):
        dU, gin, gx_in = m.cross_dU.clone(), m.cross_g[(l + 1) % 2].clone(), m.cross_gx0.clone()
        G.gemm_nt(m.cross_dU, m.xWTb[l], B, K0p, K0p, m.cross_P, mode=G.EPI_DX_FM, fm_cols=0, stream=st)
        src = m.A0 if l == 0 else m.cross_Xb[l - 1]
        G.gemm_tn(m.cross_dU, src, K0p, K0p, B, m.xview(l, grad=True), splits=m.cross_splits, stream=st)
        torch.cuda.synchronize()
        A, Wt = dd(dU), dd(m.xWTb[l]).t()
        ref = A @ Wt
        R.check("cross_P", dd(m.cross_P), ref, _dot_bound(A, Wt) + U32 * ref.abs(), "P%d" % l)
        S = dd(src)
        ref = A.t() @ S
        for gw, what in ((m.xview(l, grad=True), "X%d" % l), (step_gW[l], "step X%d" % l)):
            R.check("cross_dW", dd(gw), ref, _dot_bound(A.t(), S), what)
            assert bool((gw[~real, :] == 0).all()), ("gradient of a pad / ones row", l)
            assert bool((gw[:, ~real][:, :-1] == 0).all()), ("gradient of a pad column", l)
        P = m.cross_P.clone()
        G32_before = m.G32.clone()
        assert lib.exb_cross_bwd(ctypes.byref(m._cross_bwd_args[l]), st) == 0
        torch.cuda.synchronize()
        gl = zero(gin + P)
        if l > 0:
            assert _bits_equal(m.cross_g[l % 2], gl), ("g_l != g_{l+1} + P_l (masked)", l)
            assert _bits_equal(m.cross_dU, zero(gl * x0).to(bf16)), ("dU_{l-1} != bf16(g_l x0)", l)
            assert _bits_equal(m.cross_gx0, zero(gx_in + gl * m.cross_U[l - 1])), ("gx0 += g_l U_{l-1}", l)
        else:
            want = G32_before.clone()
            emb_real = real.clone()
            emb_real[E:] = False
            want[:, :K0p] = torch.where(emb_real[None, :], G32_before[:, :K0p] + (gx_in + gl), G32_before[:, :K0p])
            assert _bits_equal(m.G32, want), "fold: G32 != G32 + (gx0 + g_0) on the real embedding columns"

    # ---------------- dense optimizer over DNN + cross matrices and the flat region (w_cross)
    _check_optimizer(m, R)
    for l in range(Lc):
        assert _bits_equal(m.xWb[l], m.xview(l).to(bf16)), ("optimizer: xWb", l)
        assert _bits_equal(m.xWTb[l], m.xWb[l].t()), ("optimizer: xWTb", l)
    _zero_outside_real(m)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    G.check()
    out = dict(R)
    out["sensitivity_x0"], out["sensitivity_fold"] = sens_x0, sens_fold
    return out


@pytest.mark.parametrize("name", list(CONFIGS))
def test_fused_dcn_stages_match_fp64(cuda_context, record_property, name):
    _record(record_property, run_stages(name))


@pytest.mark.parametrize("name", ["d26_d9_cache", "d7_d16_1layer_nodense", "d5_d12_4layers_cache"])
def test_fused_dcn_step_matches_reference(cuda_context, name):
    from openembedding_b200.context import get_context
    ctx = get_context()
    cfg = CONFIGS[name]
    B, nd = 256, cfg.get("nd", 13)
    m = _model(cfg, B, lr=0.05, sparse_optimizer={"category": "adagrad", "learning_rate": 0.05}, dw_splits=2)
    for s in range(3):
        m.forward_backward(*[t.to(ctx.device) for t in _batch(cfg["vocab"], B, nd, seed=s)])
    ids, dense, labels = [t.to(ctx.device) for t in _batch(cfg["vocab"], B, nd, seed=99)]
    loss = m.forward_backward(ids, dense, labels, update=False)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    ref_loss, g = m.reference(ids, dense, labels)
    assert abs(float(loss) - float(ref_loss)) < 5e-3, (float(loss), float(ref_loss))
    names = ["W%d" % l for l in range(len(m.hidden))] + ["X%d" % l for l in range(m.cross_layers)]
    for name_ in names + ["wout", "wd", "bias", "wcross"] + (["cache_emb", "cache_lin"] if m.nc else []):
        if name_ == "wd" and not nd:
            continue
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


@pytest.mark.parametrize("cfg,name", [({"category": "adam", "learning_rate": 0.01}, "d26_d9_cache"),
                                      ({"category": "ftrl", "learning_rate": 0.05, "l1_regularization_strength": 0.001},
                                       "d5_d12_4layers_cache"),
                                      ({"category": "adagrad", "learning_rate": 0.05}, "d5_d12_4layers_cache")])
def test_fused_dcn_dense_optimizers_match_keras(cuda_context, cfg, name):
    """exb_dense_opt_kernel over 6 (DNN 3 + cross 3) or 8 (4 + 4) refreshed matrices vs the Keras formulas"""
    from test_optimizers import keras_reference
    from openembedding_b200.context import get_context
    ctx = get_context()
    B = 256
    m = _model(CONFIGS[name], B, sparse_optimizer={"category": "adagrad", "learning_rate": 0.05},
               dense_optimizer=dict(cfg))
    assert m._opt_args.nmat == len(m.hidden) + m.cross_layers >= 6
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
    for l in range(m.cross_layers):
        o, n = m.segs["X%d" % l]
        assert float((ref[o:o + n] - theta0[o:o + n]).abs().max()) > 0, ("cross matrix did not move", l)
        assert torch.equal(m.xWb[l], m.xview(l).to(torch.bfloat16)), ("bf16 refresh", l)
    _zero_outside_real(m)


@pytest.mark.parametrize("dense_opt", ["adagrad", "ftrl"])
def test_fused_dcn_graph_equals_eager_and_warmup_is_neutral(cuda_context, dense_opt):
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
            for l in range(m.cross_layers):
                assert torch.equal(m.xWb[l], m.xview(l).to(torch.bfloat16)), l
        tr = FusedTrainer(m, use_graph=graph)
        curves.append([float(tr.step(*batches[k % 3])) for k in range(7)])
        torch.cuda.synchronize()
        ctx.backend.engine.check()
    assert curves[0][-1] < curves[0][0], curves
    for a, b in zip(*curves):
        assert abs(a - b) < 2e-4, curves


@pytest.mark.parametrize("graph", [False, True])
def test_fused_dcn_prefetch_matches_plain(cuda_context, graph):
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


@pytest.mark.parametrize("kw", [dict(cross_layers=0),                               # no cross layer
                                dict(cross_layers=-1),
                                dict(cross_layers=6),                               # 3 DNN + 6 cross matrices > 8
                                dict(cross_layers=4, hidden=(64, 64, 64, 64, 64))])  # 5 + 4 > 8
def test_fused_dcn_constructor_errors(cuda_context, kw):
    from openembedding_b200.models.fused_dense import FusedCTR
    with pytest.raises(ValueError):
        FusedCTR(BASE_VOCAB, embedding_dim=8, model="dcn", batch=256, **kw)


def test_fused_dcn_kernels_per_step(cuda_context):
    """the cross network adds 1 + 5 launches per layer to the WDL-shaped step around it"""
    from openembedding_b200.models.fused_dense import FusedCTR
    kw = dict(embedding_dim=8, batch=256, hidden=(64, 32))
    wdl = FusedCTR(BASE_VOCAB, model="wdl", **kw).kernels_per_step()
    assert FusedCTR(BASE_VOCAB, model="dcn", cross_layers=3, **kw).kernels_per_step() == wdl + 16
    assert FusedCTR(BASE_VOCAB, model="dcn", cross_layers=1, **kw).kernels_per_step() == wdl + 6


def _torchrun(env=None):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_gpu_fused_dcn_check.py")]
    p = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600,
                       env=dict(os.environ, **(env or {})))
    return p.returncode, p.stdout


def test_mp_fused_dcn_two_ranks():
    """world 2: the loss falls, the dense replicas (cross matrices and w_cross included) stay bit-identical, and the
    all-reduce riding on the push kernel gives the parameters of the stand-alone all-reduce kernel"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs on the box")
    rc, out = _torchrun()
    assert rc == 0 and "MP_GPU_FUSED_DCN_PASSED" in out and "rider 1" in out, out[-4000:]
    rc2, out2 = _torchrun({"EXB_AR_RIDER": "0"})
    assert rc2 == 0 and "MP_GPU_FUSED_DCN_PASSED" in out2 and "rider 0" in out2, out2[-4000:]
    # not bit for bit: the sparse gradient accumulation uses float atomics, whose order varies from run to run
    tsum = lambda o: float(o.split("theta_sum ")[1].split()[0])
    assert abs(tsum(out) - tsum(out2)) < 1e-6 * abs(tsum(out2)), (tsum(out), tsum(out2))
