"""The fused xDeepFM step (FusedCTR model="xdeepfm": the CIN branch inside the one graph-captured step).

``run_stages`` checks the CIN kernels of one step stage by stage against float64, with the method and the bound
constants of test_gpu_fused_stages.py: every stage is computed from the buffers the previous stage actually wrote,
values the kernels copy or round once are compared bit for bit, sums within a derived bound. The other tests check
the whole step against ``FusedCTR.reference()`` (the eager zoo's CIN definition in fp32 autograd), the dense
optimizer over the CIN matrices against the Keras formulas, the graph / prefetch drivers and the constructor checks.
"""
import ctypes
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
    # Dp 12 != D 9: pad columns outside the CIN, cached features folded through cachegrad
    "x26_d9_cache": dict(vocab=BASE_VOCAB, dim=9, cache=64, cin=(128, 128), split=True, dense_opt="adagrad"),
    # the benchmark layout (dim 64) at batch 256
    "x26_d64_cache": dict(vocab=BASE_VOCAB, dim=64, cache=64, cin=(128, 128), split=True, dense_opt="adam"),
    # three CIN layers: 6 refreshed matrices, hidden channels handed on twice
    "x7_d16_3layers": dict(vocab=BASE_VOCAB[:7], dim=16, cache=0, cin=(32, 16, 8), split=True, dense_opt="ftrl"),
    # one layer without split_half
    "x5_d4_nosplit": dict(vocab=BASE_VOCAB[:5], dim=4, cache=0, cin=(24,), split=False, dense_opt="adagrad"),
}


def _model(cfg, B, **kw):
    from openembedding_b200.models.fused_dense import FusedCTR
    args = dict(embedding_dim=cfg["dim"], model="xdeepfm", batch=B, cache_threshold=cfg["cache"],
                cin_layers=cfg["cin"], cin_split_half=cfg["split"])
    args.update(kw)
    return FusedCTR(cfg["vocab"], **args)


def run_stages(name, B=256):
    """One step without update on the model of CONFIGS[name]; every CIN stage checked. Returns the error/bound ratio
    per stage."""
    from openembedding_b200.context import get_context
    from openembedding_b200.ops import cin as C
    from openembedding_b200.ops import gemm as G
    cfg = CONFIGS[name]
    ctx = get_context()
    dev = ctx.device
    nd = 13
    m = _model(cfg, B, sparse_optimizer={"category": "adam", "learning_rate": 0.2},
               dense_optimizer=dict(DENSE_OPT[cfg["dense_opt"]]), dw_splits=2)
    nf, Dp, D, K = m.nf, m.Dp, m.D, len(m.cin_layers)
    R_, H, Kp, Np, lo, N = m.cin_R, m.cin_H, m.cin_Kp, m.cin_Np, m.cin_lo, m.cin_layers
    g = torch.Generator().manual_seed(7)
    if m.nc:
        ce = torch.randn(m.cache_rows, Dp, generator=g) * 0.3
        ce[:, D:] = 0
        m.view("cache_emb").copy_(ce.reshape(-1).to(dev))
    for s in range(2):
        m.forward_backward(*[t.to(dev) for t in _batch(cfg["vocab"], B, nd, seed=s)])
    ids, dense, labels = [t.to(dev) for t in _batch(cfg["vocab"], B, nd, seed=99)]
    m.forward_backward(ids, dense, labels, update=False)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    G.check()

    R = _Ratios()
    f64, bf16 = torch.float64, torch.bfloat16
    dd = lambda t: t.detach().to(f64)
    theta = dd(m.theta)
    seg = lambda n_: theta[m.segs[n_][0]:m.segs[n_][0] + m.segs[n_][1]]
    wcin = m.view("wcin")
    dl = m.dlogit

    # ---------------- gather: X0[b*D + d, j] = X32[b, j*Dp + d]
    x0_ref = m.X32[:, :nf * Dp].view(B, nf, Dp)[:, :, :D].permute(0, 2, 1).reshape(R_, nf)
    assert _bits_equal(m.cin_X0, x0_ref), "gather: X0 != X32 embedding columns"
    X0 = m.cin_X0

    # ---------------- forward: Z_k (bitwise), Y_k
    def hid(k):
        return X0 if k == 0 else m.cin_Y[k - 1][:, :H[k]].float()
    for k in range(K):
        Ck = H[k] * nf
        z_ref = torch.zeros(R_, Kp[k], dtype=torch.float32, device=dev)
        z_ref[:, :Ck] = (hid(k)[:, :, None] * X0[:, None, :]).reshape(R_, Ck)
        z_ref[:, Ck] = 1.0
        assert _bits_equal(m.cin_Z[k], z_ref.to(bf16)), ("Z != bf16(hid x X0), ones column, zero pad", k)
        W = seg("C%d" % k).view(Np[k], Kp[k])
        assert _bits_equal(m.cWb[k], W.float().to(bf16)), ("cWb != bf16(theta)", k)
        assert _bits_equal(m.cWTb[k], m.cWb[k].t()), ("cWTb != cWb^T", k)
        Z, Wb = dd(m.cin_Z[k]), dd(m.cWb[k])
        ref = torch.relu(Z @ Wb.t())
        bound = _dot_bound(Z, Wb.t()) * (1 + BF16_ULP) + BF16_ULP * ref
        R.check("cin_forward", dd(m.cin_Y[k][:, :N[k]]), ref[:, :N[k]], bound[:, :N[k]], "Y%d" % k)
        assert bool((m.cin_Y[k][:, N[k]:] == 0).all()), ("cin_forward: pad channels", k)

    # ---------------- pool: p (stored), base increment (pool launched once more on top of the step's base)
    p_ref = torch.cat([dd(m.cin_Y[k][:, lo[k]:N[k]]).view(B, D, -1).sum(1) for k in range(K)], dim=1)
    R.check("cin_pool", dd(m.cin_p), p_ref, C_ACC * D * U32 * p_ref, "p")
    p = m.cin_p.clone()
    base0 = m.base.clone()
    st = torch.cuda.current_stream(dev).cuda_stream
    assert C._lib().exb_cin_pool(ctypes.byref(m._cin_pool_args), st) == 0
    torch.cuda.synchronize()
    assert _bits_equal(m.cin_p, p), "cin_pool: p differs between two launches"
    inc_ref = dd(p) @ dd(wcin)
    inc_bound = C_ACC * m.cin_T * U32 * (dd(p).abs() @ dd(wcin).abs()) + U32 * dd(m.base).abs()
    R.check("cin_pool", dd(m.base) - dd(base0), inc_ref, inc_bound, "base increment")
    m.base.copy_(base0)

    # ---------------- backward, last layer first: dY_k (bitwise), dZ_k, dhid_k / dx_k, gW_k
    dl_r = dl.repeat_interleave(D)                                  # dlogit of row r = b*D + d
    t0 = [sum(N[i] - lo[i] for i in range(k)) for k in range(K)]
    for k in range(K - 1, -1, -1):
        Yf = m.cin_Y[k].float()
        gk = torch.zeros(R_, Np[k], dtype=torch.float32, device=dev)
        gk[:, lo[k]:N[k]] = dl_r[:, None] * wcin[t0[k]:t0[k] + N[k] - lo[k]][None, :]
        if k < K - 1:
            Hn = H[k + 1]
            dh = m.cin_dhid[k + 1]
            gk[:, :Hn] = dh if lo[k] >= Hn else gk[:, :Hn] + dh
        gk = torch.where(Yf > 0, gk, torch.zeros_like(gk))
        gk[:, N[k]:] = 0
        assert _bits_equal(m.cin_dY[k], gk.to(bf16)), ("dY != bf16([Y > 0] * (dlogit w_cin | dhid))", k)
        dY, WT = dd(m.cin_dY[k]), dd(m.cWTb[k])
        ref = dY @ WT.t()
        bound = _dot_bound(dY, WT.t()) * (1 + BF16_ULP) + BF16_ULP * ref.abs()
        R.check("cin_dZ", dd(m.cin_dZ[k]), ref, bound, "dZ%d" % k)
        Ck = H[k] * nf
        dZ3 = dd(m.cin_dZ[k][:, :Ck]).view(R_, H[k], nf)
        x, h = dd(X0), dd(hid(k))
        ref_h = (dZ3 * x[:, None, :]).sum(2)
        R.check("cin_outer_bwd", dd(m.cin_dhid[k]), ref_h, C_ACC * nf * U32 * (dZ3.abs() * x.abs()[:, None, :]).sum(2),
                "dhid%d" % k)
        ref_x = (dZ3 * h[:, :, None]).sum(1)
        R.check("cin_outer_bwd", dd(m.cin_dx[k]), ref_x, C_ACC * H[k] * U32 * (dZ3.abs() * h.abs()[:, :, None]).sum(1),
                "dx%d" % k)
        Z = dd(m.cin_Z[k])
        R.check("cin_dW", dd(m.cview(k, grad=True)), dY.t() @ Z, _dot_bound(dY.t(), Z), "C%d" % k)
    dl64, p64 = dd(dl), dd(p)
    R.check("cin_dW", dd(m.gview("wcin")), dl64 @ p64, C_ACC * B * U32 * (dl64.abs() @ p64.abs()), "w_cin")

    # ---------------- fold: G32 = dZ0 @ W0 (the DNN's dX GEMM) + dx_0 + dhid_0 + sum_k>=1 dx_k on the embedding columns
    dZ0, WT0 = dd(m.dZ[0]), dd(m.WTb[0])
    mlp = dZ0 @ WT0.t()
    mlp_bound = _dot_bound(dZ0, WT0.t())
    srcs = [m.cin_dx[0], m.cin_dhid[0]] + m.cin_dx[1:]
    fsum = sum(dd(s) for s in srcs)
    fabs = sum(dd(s).abs() for s in srcs)
    to_cols = lambda t: torch.nn.functional.pad(t.view(B, D, nf).permute(0, 2, 1), (0, Dp - D)).reshape(B, nf * Dp)
    ref = mlp.clone()
    ref[:, :nf * Dp] += to_cols(fsum)
    bound = mlp_bound.clone()
    bound[:, :nf * Dp] += to_cols(C_ACC * len(srcs) * U32 * fabs)
    bound += U32 * ref.abs()
    R.check("cin_fold", dd(m.G32[:, :m.K0p]), ref, bound, "G32")

    # ---------------- dense optimizer over DNN + CIN matrices and the flat region (w_cin)
    _check_optimizer(m, R)
    for k in range(K):
        assert _bits_equal(m.cWb[k], m.view("C%d" % k).view(Np[k], Kp[k]).to(bf16)), ("optimizer: cWb", k)
        assert _bits_equal(m.cWTb[k], m.cWb[k].t()), ("optimizer: cWTb", k)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    G.check()
    return dict(R)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_fused_xdeepfm_stages_match_fp64(cuda_context, record_property, name):
    _record(record_property, run_stages(name))


def _far_biases(m):
    """CIN pre-activations far from 0 (half the channels on, half off): a relu flipping inside bf16 rounding
    would otherwise move whole gradient terms between the kernels and the fp32 reference"""
    for k, n in enumerate(m.cin_layers):
        col = m.cview(k)[:n, m.cin_H[k] * m.nf]
        col.copy_(torch.where(torch.arange(n, device=m.dev) % 2 == 0, 4.0, -4.0))
    m.refresh_weights()


@pytest.mark.parametrize("name", ["x26_d9_cache", "x7_d16_3layers", "x5_d4_nosplit"])
def test_fused_xdeepfm_step_matches_reference(cuda_context, name):
    from openembedding_b200.context import get_context
    ctx = get_context()
    cfg = CONFIGS[name]
    B = 256
    m = _model(cfg, B, lr=0.05, sparse_optimizer={"category": "adagrad", "learning_rate": 0.05}, dw_splits=2)
    _far_biases(m)
    for s in range(3):
        m.forward_backward(*[t.to(ctx.device) for t in _batch(cfg["vocab"], B, 13, seed=s)])
    ids, dense, labels = [t.to(ctx.device) for t in _batch(cfg["vocab"], B, 13, seed=99)]
    loss = m.forward_backward(ids, dense, labels, update=False)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    ref_loss, g = m.reference(ids, dense, labels)
    assert abs(float(loss) - float(ref_loss)) < 5e-3, (float(loss), float(ref_loss))
    names = ["W%d" % l for l in range(len(m.hidden))] + ["C%d" % k for k in range(len(m.cin_layers))]
    for name_ in names + ["wout", "wd", "bias", "wcin"] + (["cache_emb", "cache_lin"] if m.nc else []):
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


@pytest.mark.parametrize("cfg,name", [({"category": "adam", "learning_rate": 0.01}, "x26_d9_cache"),
                                      ({"category": "ftrl", "learning_rate": 0.05, "l1_regularization_strength": 0.001},
                                       "x7_d16_3layers"),
                                      ({"category": "adagrad", "learning_rate": 0.05}, "x7_d16_3layers")])
def test_fused_xdeepfm_dense_optimizers_match_keras(cuda_context, cfg, name):
    """exb_dense_opt_kernel over 5 (DNN 3 + CIN 2) or 6 (3 + 3) refreshed matrices vs the Keras formulas"""
    from test_optimizers import keras_reference
    from openembedding_b200.context import get_context
    ctx = get_context()
    B = 256
    m = _model(CONFIGS[name], B, sparse_optimizer={"category": "adagrad", "learning_rate": 0.05},
               dense_optimizer=dict(cfg))
    assert m._opt_args.nmat == len(m.hidden) + len(m.cin_layers) >= 5
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
    for k in range(len(m.cin_layers)):
        o, n = m.segs["C%d" % k]
        assert float((ref[o:o + n] - theta0[o:o + n]).abs().max()) > 0, ("CIN filters did not move", k)
        assert torch.equal(m.cWb[k], m.cview(k).to(torch.bfloat16)), ("bf16 refresh", k)


@pytest.mark.parametrize("dense_opt", ["adagrad", "ftrl"])
def test_fused_xdeepfm_graph_equals_eager_and_warmup_is_neutral(cuda_context, dense_opt):
    from openembedding_b200.context import get_context, reset_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg = CONFIGS["x26_d9_cache"]
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
            for k in range(len(m.cin_layers)):
                assert torch.equal(m.cWb[k], m.cview(k).to(torch.bfloat16)), k
        tr = FusedTrainer(m, use_graph=graph)
        curves.append([float(tr.step(*batches[k % 3])) for k in range(7)])
        torch.cuda.synchronize()
        ctx.backend.engine.check()
    assert curves[0][-1] < curves[0][0], curves
    for a, b in zip(*curves):
        assert abs(a - b) < 2e-4, curves


@pytest.mark.parametrize("graph", [False, True])
def test_fused_xdeepfm_prefetch_matches_plain(cuda_context, graph):
    from openembedding_b200.context import get_context, reset_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg = CONFIGS["x26_d9_cache"]
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


@pytest.mark.parametrize("kw", [dict(cin_layers=(127, 128)),                       # odd size under split_half
                                dict(cin_layers=(64, 31, 16)),                     # odd size below the last layer
                                dict(cin_layers=(1024, 128)),                      # hands 512 channels on
                                dict(cin_layers=(600, 8), cin_split_half=False),   # hands 600 channels on
                                dict(vocab=[100] * 65),                            # 65 fields
                                dict(cin_layers=())])
def test_fused_xdeepfm_constructor_errors(cuda_context, kw):
    from openembedding_b200.models.fused_dense import FusedCTR
    kw = dict(kw)
    vocab = kw.pop("vocab", BASE_VOCAB)
    with pytest.raises(ValueError):
        FusedCTR(vocab, embedding_dim=8, model="xdeepfm", batch=256, **kw)


def test_mp_fused_xdeepfm_two_ranks():
    """world 2: the loss falls and the dense replicas (CIN filters and w_cin included) stay bit-identical"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs on the box")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_gpu_fused_xdeepfm_check.py")]
    p = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0 and "MP_GPU_FUSED_XDEEPFM_PASSED" in p.stdout, p.stdout[-4000:]
