"""Checkpoints and export of the fused models (models/fused_dense.py: FusedCTR.save / load / load_dense_state_dict /
save_as_original_model, FusedTrainer after a load) on one GPU.

Where run-to-run atomics make the step nondeterministic (shared-memory and global atomics of prep, cachegrad, the
split-K reduce-adds) two trajectories are compared with the spread rule of test_gpu_fused_eval.py: two runs of the same
trajectory set the spread, and a resumed run must stay within a few spreads of them, in the largest and in the mean
difference of every buffer; when the two runs agree bit for bit, the resumed run must too. The largest difference is
heavy-tailed (with Adam an element whose gradient is ulp-level noise around zero moves by up to the learning rate in
either direction), hence the factor 8 and the 1e-4 floor; the mean is stable, and a run that lost an optimizer state or
a step, or trained on stale prefetched rows, misses it by far."""
import copy
import os

import numpy as np
import pytest
import torch

from test_gpu_fused_eval import LAYOUTS, _batch, _pinned, _rows, _rows_equal, _vocab

pytestmark = pytest.mark.gpu

MODELS = ["deepfm_d9_cache", "wdl_d16", "xdeepfm_d9_cache", "dcn_d8_cache"]
DENSE_OPT = {"adam": {"category": "adam", "learning_rate": 0.01},
             "ftrl": {"category": "ftrl", "learning_rate": 0.05, "l1_regularization_strength": 0.001,
                      "l2_regularization_strength": 0.001}}
SPARSE_OPT = {"adam": {"category": "adam", "learning_rate": 0.2}, "ftrl": {"category": "ftrl", "learning_rate": 0.2}}


def _model(cfg, opt="adam", seed=0, **over):
    from openembedding_b200.models.fused_dense import FusedCTR
    kw = {k: cfg[k] for k in ("hidden", "cin_layers", "cross_layers") if k in cfg}
    kw.update(over)
    m = FusedCTR(_vocab(cfg), num_dense=cfg.get("nd", 13), embedding_dim=cfg["dim"], model=cfg["model"],
                 batch=kw.pop("batch", cfg["B"]), cache_threshold=kw.pop("cache", cfg["cache"]),
                 sparse_optimizer=SPARSE_OPT[opt], dense_optimizer=DENSE_OPT[opt], dw_splits=2, seed=seed, **kw)
    if m.nc:                       # replicated tables away from zero, so that they take part from the first step
        g = torch.Generator().manual_seed(7 + seed)
        ce = torch.randn(m.cache_rows, m.Dp, generator=g) * 0.3
        ce[:, m.D:] = 0
        m.view("cache_emb").copy_(ce.reshape(-1).to(m.dev))
        m.view("cache_lin").copy_((torch.randn(m.cache_rows, generator=g) * 0.3).to(m.dev))
    return m


def _dense(m):
    """the full dense buffers, padding included, on the CPU"""
    return [t.detach().clone().cpu() for t in (m.theta, m.accum, m.accum2, m.opt_step)]


def _fresh_ctx():
    from openembedding_b200.context import get_context, reset_context
    reset_context()
    return get_context()


def _run(cfg, opt, batches, seed=0, load=None, save_at=None, save_path=None):
    """a graph-driven pipeline over ``batches`` (pinned host tensors); ``load``: checkpoint loaded before the
    trainer exists; ``save_at``: ``save`` once the pipeline has trained that many batches (the next batch's rows and
    plan are then prefetched). Returns (last loss, dense buffers, table rows)."""
    ctx = _fresh_ctx()
    from openembedding_b200.models.fused_dense import FusedTrainer
    m = _model(cfg, opt, seed)
    if load is not None:
        m.load(load)
    tr = FusedTrainer(m, use_graph=True)
    pipe = tr.make_pipeline(cfg["B"], m.nf, m.nd)
    for b in batches:
        pipe.submit(*b)
        if save_at is not None and pipe.trained == save_at:
            assert tr._x32_key is not None          # a prefetch is armed
            m.save(save_path)
            save_at = None
    loss = pipe.last_loss()
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    return loss, _dense(m), _rows(ctx, m)


def _same_trajectory(a, b, ref):
    """``b`` trains as ``a`` does: bit for bit when ``ref`` (another run of ``a``'s trajectory) equals ``a`` bit for bit,
    otherwise within a few times the spread between ``a`` and ``ref``"""
    (la, da, ra), (lb, db, rb), (lr, dr, _) = a, b, ref
    if la == lr and all(torch.equal(x, y) for x, y in zip(da, dr)):
        assert lb == la, (la, lb)
        for x, y in zip(da, db):
            assert torch.equal(x.view(torch.int32) if x.is_floating_point() else x,
                               y.view(torch.int32) if y.is_floating_point() else y)
        _rows_equal(ra, rb)
        return
    assert abs(lb - la) <= 4 * abs(la - lr) + 2e-4, (la, lb, lr)
    for x, y, r in zip(da, db, dr):
        d, s = (x.double() - y.double()).abs(), (x.double() - r.double()).abs()
        assert float(d.max()) <= 8 * float(s.max()) + 1e-4, (float(d.max()), float(s.max()))
        assert float(d.mean()) <= 8 * float(s.mean()) + 1e-7, (float(d.mean()), float(s.mean()))
    assert torch.equal(da[3], db[3])                   # the optimizer step counter


GRID = [(n, o, v) for n in MODELS for o in ("adam", "ftrl") for v in ("1", "0")] + \
       [("deepfm_d8_h600_nodense_hash", "adam", v) for v in ("1", "0")]


@pytest.mark.parametrize("name,opt,v2", GRID)
def test_resume_equals_uninterrupted(cuda_context, monkeypatch, tmp_path, name, opt, v2):
    """save after k of 2k batches in the middle of a pipeline (prefetch armed), load into a model built with another
    seed in a fresh context, train the other k: the same final loss, dense buffers, rows and optimizer states as the
    uninterrupted run -- which the save did not disturb"""
    monkeypatch.setenv("EXB_SPARSE_V2", v2)
    cfg, k = LAYOUTS[name], 3
    dev = torch.device("cuda")
    batches = [[_pinned(t) for t in _batch(cfg, s, dev)] for s in range(2 * k)]
    ck = str(tmp_path / "ck")
    saved = _run(cfg, opt, batches, save_at=k, save_path=ck)
    plain = _run(cfg, opt, batches)
    resumed = _run(cfg, opt, batches[k:], seed=1, load=ck)
    _same_trajectory(plain, saved, _run(cfg, opt, batches))        # the save is invisible
    _same_trajectory(plain, resumed, saved)


@pytest.mark.parametrize("v2", ["1", "0"])
def test_load_into_live_trainer(cuda_context, monkeypatch, tmp_path, v2):
    """a trainer with captured graphs and an armed prefetch, loaded (on the model) and stepped, trains as a freshly
    loaded model on the same batches: its graphs are reused, the prefetched rows and plan are dropped"""
    from openembedding_b200.models.fused_dense import FusedTrainer
    monkeypatch.setenv("EXB_SPARSE_V2", v2)
    cfg, opt = LAYOUTS["deepfm_d9_cache"], "adam"
    dev = torch.device("cuda")
    first = [[_pinned(t) for t in _batch(cfg, s, dev)] for s in range(3)]
    other = [[_pinned(t) for t in _batch(cfg, 50 + s, dev)] for s in range(3)]
    after = [[_pinned(t) for t in _batch(cfg, 100 + s, dev)] for s in range(4)]
    ck = str(tmp_path / "ck")
    _run(cfg, opt, first, save_at=len(first) - 1, save_path=ck)

    ctx = _fresh_ctx()
    m = _model(cfg, opt, seed=3)
    tr = FusedTrainer(m, use_graph=True)
    pipe = tr.make_pipeline(cfg["B"], m.nf, m.nd)
    for b in other:
        pipe.submit(*b)
    assert tr._x32_key is not None
    graphs = dict(tr._graphs)
    m.load(ck)
    pipe.submit(*after[0])          # trains other[-1]: pulls up front on the graph captured for the first step
    assert tr._graphs.keys() == graphs.keys() and all(tr._graphs[k] is g for k, g in graphs.items())
    for b in after[1:]:
        pipe.submit(*b)
    live = (pipe.last_loss(), _dense(m), _rows(ctx, m))
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    assert all(tr._graphs[k] is g for k, g in graphs.items())
    # the batch trained first after the load (other[-1], prefetched before it) -- then ``after``
    fresh = _run(cfg, opt, [other[-1]] + after, seed=4, load=ck)
    _same_trajectory(fresh, live, _run(cfg, opt, [other[-1]] + after, seed=5, load=ck))


ROUND_TRIP = [(n, o, True) for n in MODELS for o in ("adam", "ftrl")] + [("deepfm_d9_cache", "adam", False),
                                                                         ("wdl_d16", "ftrl", False)]


@pytest.mark.parametrize("name,opt,pack", ROUND_TRIP)
def test_round_trip(cuda_context, tmp_path, name, opt, pack):
    """load(save(m)) restores the full dense buffers bit for bit, padding included, with the gradients cleared and
    the bf16 weight copies those of refresh_weights(); without the optimizer the dense optimizer state is the
    construction value"""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg = LAYOUTS[name]
    ctx, dev = get_context(), torch.device("cuda")
    m = _model(cfg, opt, pack_linear=pack)
    init = _dense(m)
    tr = FusedTrainer(m, use_graph=True)
    for s in range(3):
        tr.step(*_batch(cfg, s, dev))
    torch.cuda.synchronize()
    state, rows = _dense(m), _rows(ctx, m)
    m.save(str(tmp_path / "full"))
    m.save(str(tmp_path / "weights"), include_optimizer=False)
    for s in range(3, 5):
        tr.step(*_batch(cfg, s, dev))
    m.forward_backward(*_batch(cfg, 9, dev), update=False)       # gradients left behind
    m.load(str(tmp_path / "full"))
    torch.cuda.synchronize()
    for a, b in zip(state, _dense(m)):
        assert torch.equal(a, b)
    assert not bool(m.gtheta.any()) and not m._grad_dirty
    _rows_equal(rows, _rows(ctx, m))
    copies = [t.clone() for t in m.Wb + m.WTb + m.cWb + m.cWTb + m.xWb + m.xWTb]
    m.refresh_weights()
    for a, b in zip(copies, m.Wb + m.WTb + m.cWb + m.cWTb + m.xWb + m.xWTb):
        assert torch.equal(a, b)
    m.load(str(tmp_path / "weights"))
    torch.cuda.synchronize()
    got = _dense(m)
    assert torch.equal(got[0], state[0])
    for a, b in zip(init[1:], got[1:]):              # accum, accum2, opt_step as constructed
        assert torch.equal(a, b)
    for a, b in zip(rows, _rows(ctx, m)):            # table weights (their optimizer states start fresh)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint8), b[1].view(np.uint8))
    # a dense state dict of another optimizer category: the weights load, the state starts fresh
    sd = m.dense_state_dict()
    other = "ftrl" if opt == "adam" else "adam"
    foreign = {k.replace(opt + ".", other + ".", 1) if "/" in k else k: v for k, v in sd.items()}
    m.load_dense_state_dict(foreign)
    got = _dense(m)
    assert torch.equal(got[0], state[0]) and all(torch.equal(a, b) for a, b in zip(init[1:], got[1:]))


def test_other_batch_and_mismatch(cuda_context, tmp_path):
    """a checkpoint saved at batch 256 loads at batch 128 and predicts the same; a different hidden, model, dim or
    cached set raises ValueError naming it and leaves the model as it was"""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg = dict(LAYOUTS["dcn_d8_cache"], model="deepfm")      # Dp = D = 8: row-wise prep, a deterministic forward
    dev = torch.device("cuda")
    m = _model(cfg)
    tr = FusedTrainer(m, use_graph=True)
    for s in range(3):
        tr.step(*_batch(cfg, s, dev))
    ids, dense, _ = _batch(cfg, 77, dev, n=128)
    p256 = tr.predict(ids, dense).cpu()
    ck = str(tmp_path / "ck")
    m.save(ck)
    _fresh_ctx()
    m = _model(cfg, seed=1, batch=128)
    m.load(ck)
    p128 = FusedTrainer(m, use_graph=True).predict(ids, dense).cpu()
    assert torch.equal(p128.view(torch.int32), p256.view(torch.int32)), float((p128 - p256).abs().max())
    for key, over in (("hidden", dict(hidden=(64,))), ("model", dict(model="wdl")), ("embedding_dim", dict(dim=16)),
                      ("cached", dict(cache=40))):
        ctx = _fresh_ctx()
        c = dict(cfg, **{k: v for k, v in over.items() if k in ("model", "dim", "cache")})
        m = _model(c, seed=2, **{k: v for k, v in over.items() if k == "hidden"})
        m.forward_backward(*_batch(c, 1, dev))
        torch.cuda.synchronize()
        before, rows = _dense(m), _rows(ctx, m)
        with pytest.raises(ValueError, match=key):
            m.load(ck)
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(before, _dense(m)))
        _rows_equal(rows, _rows(ctx, m))
        assert m.load_generation == 0


def _rounding_bound(mod, ids, dense):
    """per-sample first-order bound on |fused logit - fp32 logit| from the fused path's bf16 rounding points.

    The fused forward rounds to bf16 (relative error <= 2^-9, round to nearest): the GEMM operands -- the DNN's and
    the cross network's weights and biases, the DNN input A0 (embeddings + dense), every hidden activation, the cross
    layers' inputs x_l, the CIN filters, interaction operands Z_k and layer outputs Y_k -- and accumulates in fp32.
    To first order, rounding a value v moves the logit by at most |dz/dv| |v| 2^-9; the bound is the sum over every
    rounded value (per-sample gradients in fp64 through the exported module, whose layers are exactly these rounding
    points) taken at 2^-8 -- twice the first-order term, for the higher orders -- plus fp32 accumulation over the
    longest dot product (K0p terms) on the same magnitudes and on |z|."""
    from torch import nn
    mod = copy.deepcopy(mod).double()
    acts = []

    def grab(t):                   # every use of a rounded value gets a node (and a gradient) of its own
        t = t.clone() if t.requires_grad else t.detach().clone().requires_grad_(True)
        t.retain_grad()
        acts.append(t)
        return t

    layers = [mm for mm in mod.modules() if isinstance(mm, (nn.Linear, nn.Conv1d))]
    hooks = [mm.register_forward_pre_hook(lambda m_, args: (grab(args[0]),)) for mm in layers]
    hooks += [mm.register_forward_hook(lambda m_, args, out: grab(out)) for mm in mod.modules()
              if isinstance(mm, nn.Conv1d)]            # CIN layer outputs Y_k
    rounded = [p for n, p in mod.named_parameters() if n.startswith(("dnn.", "cross.", "cin.convs."))]
    out = []
    for b in range(ids.shape[0]):
        acts.clear()
        mod.zero_grad()
        z = mod(ids[b:b + 1], dense[b:b + 1].double())
        z.sum().backward()
        s = sum(float((p.grad * p.detach()).abs().sum()) for p in rounded)
        s += sum(float((a.grad * a).abs().sum()) for a in acts if a.grad is not None)
        out.append(s)
    for h in hooks:
        h.remove()
    return torch.tensor(out, dtype=torch.float64)


EXPORT = [(n, True) for n in MODELS] + [("deepfm_d9_cache", False)]


@pytest.mark.parametrize("name,pack", EXPORT)
def test_export(cuda_context, tmp_path, name, pack):
    """the stand-alone export: its tensors are the model's weights and rows bit for bit (dnn_out.bias folded into
    bias), its logits agree with predict within the bf16 rounding bound, and the file loaded without the engine on
    the CPU gives the GPU's logits"""
    import openembedding_b200 as oe
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    cfg = LAYOUTS[name]
    ctx, dev = get_context(), torch.device("cuda")
    m = _model(cfg, pack_linear=pack)
    tr = FusedTrainer(m, use_graph=True)
    for s in range(4):
        tr.step(*_batch(cfg, s, dev))
    torch.cuda.synchronize()
    path = str(tmp_path / "export" / "model.pt")
    mod = m.save_as_original_model(path)
    assert os.path.exists(path)
    sd, got = m.dense_state_dict(include_optimizer=False), mod.state_dict()
    for k, v in sd.items():
        if k == "dnn_out.bias":
            continue
        want = v + sd["dnn_out.bias"] if k == "bias" else v
        assert torch.equal(got[k], want), k
    D = m.D
    for j, f in enumerate(m.server):
        tabs = [(m.sparse.metas[j], slice(0, D + 1))] if pack else [(m.sparse.metas[j], slice(0, D)),
                                                                  (m.sparse.metas[m.ns + j], slice(D, D + 1))]
        full = torch.cat([mod.emb[j].weight, mod.lin[j].weight], 1)
        seen = torch.zeros(full.shape[0], dtype=torch.bool)
        for meta, cols in tabs:
            for idx, w, _ in ctx.backend.iter_local_rows(meta, 1 << 16):
                ii = torch.from_numpy(np.array(idx, dtype=np.int64) * meta.shard_num + ctx.backend.shard_id(meta))
                assert torch.equal(full[ii, cols], torch.from_numpy(np.array(w)))
                seen[ii] = True
        assert not bool(full[~seen].any())            # rows never trained: the zero initializer
    ids, dense, _ = _batch(cfg, 99, dev)
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
    with torch.no_grad():
        zg = copy.deepcopy(mod).to(dev)(ids, dense).cpu()
    old = oe.flags.device
    try:                                               # the file alone, without the engine, on the CPU
        from openembedding_b200.context import reset_context
        reset_context()
        oe.flags.device = "cpu"
        get_context()
        loaded = torch.load(path, weights_only=False)
        with torch.no_grad():
            zc = loaded(ids.cpu(), dense.cpu())
    finally:
        oe.flags.device = old
    assert type(loaded).__name__ == "StandaloneCTR"
    assert float((zc - zg).abs().max()) <= 1e-5 * (1 + float(zg.abs().max()))


def test_export_hash_feature_raises(cuda_context, tmp_path):
    cfg = LAYOUTS["deepfm_d8_h600_nodense_hash"]
    m = _model(cfg)
    path = str(tmp_path / "model.pt")
    with pytest.raises(ValueError, match="nn.Embedding"):
        m.save_as_original_model(path)
    assert not os.path.exists(path)


def test_two_ranks_and_load_at_world_one(cuda_context, tmp_path):
    """tests/mp_gpu_fused_ckpt_check.py at world 2 (resume equals uninterrupted, theta identical across the ranks),
    then its world-2 checkpoint loads at world 1 with the same dense state and every table row"""
    import socket
    import subprocess
    import sys
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedCTR
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs on the box")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_gpu_fused_ckpt_check.py"),
           str(tmp_path)]
    p = subprocess.run(cmd, cwd=root, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0 and "MP_GPU_FUSED_CKPT_PASSED" in p.stdout, p.stdout[-4000:]
    sys.path.insert(0, os.path.join(root, "tests"))
    import mp_gpu_fused_ckpt_check as mp
    ctx = get_context()
    m = mp.model(seed=9)
    assert isinstance(m, FusedCTR) and ctx.world == 1
    m.load(str(tmp_path / "ck"))
    want = torch.load(str(tmp_path / "dense.pt"), weights_only=True)
    got = m.dense_state_dict()
    assert want.keys() == got.keys() and all(torch.equal(want[k], got[k]) for k in want)
    saved = [np.load(str(tmp_path / ("rows_%d.npz" % r))) for r in range(2)]
    for t, r in enumerate(mp.rows(ctx, m)):
        idx = np.concatenate([z["i_%d" % t] for z in saved])
        o = np.argsort(idx)
        assert np.array_equal(idx[o], r[0])
        for k, a in zip("ws", r[1:]):
            b = np.concatenate([z["%s_%d" % (k, t)] for z in saved])[o]
            assert np.array_equal(b.view(np.uint8), a.view(np.uint8))
