"""Evaluation on the fused models (models/fused_dense.py: FusedCTR.predict_forward, FusedTrainer.predict /
evaluate): logits against fp64 and fp32 references, the metric's buckets against the returned probabilities, partial
batches, graph against eager, no side effect on any training state, and training unchanged by evaluations.

Bit-for-bit comparisons of two forward passes need a deterministic forward: prep B (the path when Dp does not divide
128) sums each row's FM and linear terms with shared-memory atomics, so for those layouts the comparison is within
the logit bound instead."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
C_ACC = 4.0

BASE_VOCAB = [1000, 50, 20000, 7, 3000] + [300] * 21

LAYOUTS = {
    # Dp 12 != D, cached features, prep A + B
    "deepfm_d9_cache": dict(model="deepfm", dim=9, cache=64, B=384),
    # Hp 640 > 512, no dense features, a hash-table feature (vocab 0)
    "deepfm_d8_h600_nodense_hash": dict(model="deepfm", dim=8, cache=64, B=256, hidden=(600,), nd=0, hash=True),
    "wdl_d16": dict(model="wdl", dim=16, cache=0, B=256),
    "xdeepfm_d9_cache": dict(model="xdeepfm", dim=9, cache=64, B=256, cin_layers=(16, 16)),
    "dcn_d8_cache": dict(model="dcn", dim=8, cache=64, B=256, cross_layers=2),
}


def _vocab(cfg):
    return BASE_VOCAB + ([0] if cfg.get("hash") else [])


def _batch(cfg, seed, dev, n=None):
    vocab, nd = _vocab(cfg), cfg.get("nd", 13)
    n = n or cfg["B"]
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randint(0, v if v else 2 ** 62, (n,), generator=g) for v in vocab], 1).contiguous()
    dense = torch.rand(n, nd, generator=g)
    labels = (torch.rand(n, generator=g) < 0.3).float()
    return ids.to(dev), dense.to(dev), labels.to(dev)


def _model(cfg):
    from openembedding_b200.models.fused_dense import FusedCTR
    kw = {k: cfg[k] for k in ("hidden", "cin_layers", "cross_layers") if k in cfg}
    m = FusedCTR(_vocab(cfg), num_dense=cfg.get("nd", 13), embedding_dim=cfg["dim"], model=cfg["model"],
                 batch=cfg["B"], cache_threshold=cfg["cache"], sparse_optimizer={"category": "adam", "learning_rate": 0.2},
                 dense_optimizer={"category": "adam", "learning_rate": 0.01}, dw_splits=2, **kw)
    if m.nc:
        g = torch.Generator().manual_seed(7)
        ce = torch.randn(m.cache_rows, m.Dp, generator=g) * 0.3
        ce[:, m.D:] = 0
        m.view("cache_emb").copy_(ce.reshape(-1).to(m.dev))
        m.view("cache_lin").copy_((torch.randn(m.cache_rows, generator=g) * 0.3).to(m.dev))
    return m


def _state(m):
    return [t.clone() for t in (m.theta, m.accum, m.accum2, m.opt_step, m.gtheta, m.loss)]


def _rows(ctx, m):
    """every table row this rank owns, with its optimizer state, sorted by index"""
    out = []
    for meta in m.sparse.metas:
        parts = [(np.array(i, copy=True), np.array(w, copy=True), np.array(s, copy=True))
                 for i, w, s in ctx.backend.iter_local_rows(meta, 1 << 16)]
        if not parts:
            out.append(None)
            continue
        idx = np.concatenate([p[0] for p in parts])
        o = np.argsort(idx)
        out.append((idx[o], np.concatenate([p[1] for p in parts])[o], np.concatenate([p[2] for p in parts])[o]))
    return out


def _rows_equal(a, b):
    for x, y in zip(a, b):
        if x is None or y is None:
            assert x is None and y is None
            continue
        for u, v in zip(x, y):
            assert u.shape == v.shape and np.array_equal(u.view(np.uint8), v.view(np.uint8))


def _ref_counts(p, y, T=200):
    from openembedding_b200.models.metrics import keras_thresholds
    t = keras_thresholds(T)
    k = (np.asarray(p, dtype=np.float32)[:, None] > t[None, :]).sum(1)
    real = np.asarray(y) != 0
    return np.bincount(k[real], minlength=T + 1), np.bincount(k[~real], minlength=T + 1)


def _logit_bound(m):
    """fp64 logits from the stored H_L, base and w_out, and the fp32 accumulation bound of the head's dot"""
    H, w, base = m.H[-1].double(), m.view("wout").double(), m.base.double()
    ref = base + H @ w
    return ref, C_ACC * (m.Hp[-1] + 1) * U32 * (H.abs() @ w.abs() + base.abs())


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_fused_eval(cuda_context, name):
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    from openembedding_b200.models.metrics import BinaryMetrics, auc_from_counts
    cfg = LAYOUTS[name]
    ctx = get_context()
    dev, B = ctx.device, cfg["B"]
    m = _model(cfg)
    for s in range(2):
        m.forward_backward(*_batch(cfg, s, dev))
    ids, dense, labels = _batch(cfg, 99, dev)
    torch.cuda.synchronize()
    state0, rows0 = _state(m), _rows(ctx, m)
    row_prep = m.mn_major and 128 % m.Dp == 0

    eager, graph = FusedTrainer(m, use_graph=False), FusedTrainer(m, use_graph=True)
    met = BinaryMetrics(200, device=dev)
    eager.evaluate(ids, dense, labels, met)
    probs, z = m.probs.clone(), m.logits.clone()
    torch.cuda.synchronize()
    ref64, bound = _logit_bound(m)
    err = (z.double() - ref64).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    # fp32 torch forward (reference()) from theta and the rows the stateless pull left in X32
    _, _, zr = m.reference(ids, dense, labels, return_logits=True)
    assert bool(((z - zr).abs() <= 1e-2 * (1 + zr.abs())).all()), float((z - zr).abs().max())
    # the metric's buckets are those of the returned probabilities
    pos, neg = _ref_counts(probs.cpu().numpy(), labels.cpu().numpy())
    gp, gn, _, count = met.counts()
    assert np.array_equal(gp, pos) and np.array_equal(gn, neg), "metric buckets differ from the probabilities"
    assert count == B and met.result()["auc"] == auc_from_counts(pos, neg)

    # partial batch: rows < n as in the full batch, rows >= n not counted
    n = B - 37
    part = BinaryMetrics(200, device=dev)
    graph.evaluate(ids[:n], dense[:n], labels[:n], part)
    pos_n, neg_n = _ref_counts(m.probs[:n].cpu().numpy(), labels[:n].cpu().numpy())
    gp, gn, _, count = part.counts()
    assert count == n and np.array_equal(gp, pos_n) and np.array_equal(gn, neg_n)
    pn = graph.predict(ids[:n], dense[:n])
    pf = graph.predict(ids, dense)
    torch.cuda.synchronize()
    assert pn.shape == (n,)
    if row_prep:
        assert torch.equal(pn.view(torch.int32), pf[:n].view(torch.int32))
        assert torch.equal(pf.view(torch.int32), probs.view(torch.int32))       # graph == eager, bit for bit
    else:                              # prep B's atomic order moves base by a few ulps of its partial sums
        assert float((pn - pf[:n]).abs().max()) <= 1e-4
        assert float((pf - probs).abs().max()) <= 1e-4

    # no side effect on parameters, optimizer state, gradients, the loss buffer or the tables (unseen hash ids
    # insert no row)
    unseen = _batch(cfg, 12345, dev)
    graph.evaluate(unseen[0], unseen[1], unseen[2], part)
    torch.cuda.synchronize()
    for a, b in zip(state0, _state(m)):
        assert torch.equal(a, b)
    _rows_equal(rows0, _rows(ctx, m))

    # the mean BCE of the full batch is the training step's loss
    eager.evaluate(ids, dense, labels, BinaryMetrics(200, device=dev))
    z = m.logits.double()
    y = labels.double()
    per = torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-z.abs()))
    loss = float(m.forward_backward(ids, dense, labels, update=False))
    _, bound = _logit_bound(m)
    tol = C_ACC * B * U32 * float(per.mean()) + float(bound.mean()) + 1e-7
    assert abs(loss - float(per.mean())) <= tol, (loss, float(per.mean()), tol)
    ctx.backend.engine.check()


def test_kernels_per_eval_matches_profiler(cuda_context):
    from torch.profiler import ProfilerActivity, profile
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    from openembedding_b200.models.metrics import BinaryMetrics
    dev = get_context().device
    for name in ("deepfm_d9_cache", "xdeepfm_d9_cache", "dcn_d8_cache"):
        cfg = LAYOUTS[name]
        m = _model(cfg)
        tr = FusedTrainer(m, use_graph=True)
        met = BinaryMetrics(200, device=dev)
        ids, dense, labels = _batch(cfg, 1, dev)
        tr.evaluate(ids, dense, labels, met)
        torch.cuda.synchronize()
        gr = tr._graphs["eval"]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                gr.replay()
                met.update(m.logits, tr._eval["labels"], n=tr._eval["n"])
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and not e.name.startswith(("Memcpy", "Memset"))]
        assert len(names) == 3 * m.kernels_per_eval(metric=True), (name, m.kernels_per_eval(metric=True), names)


def _pinned(t):
    return t.cpu().pin_memory()


@pytest.mark.parametrize("v2", ["1", "0"])
def test_evaluation_is_invisible_to_training(cuda_context, monkeypatch, v2):
    """a graph-driven pipeline with prefetch, evaluated every few steps, trains as the same run without evaluation"""
    from openembedding_b200.context import get_context, reset_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    from openembedding_b200.models.metrics import BinaryMetrics
    monkeypatch.setenv("EXB_SPARSE_V2", v2)
    cfg = LAYOUTS["deepfm_d8_h600_nodense_hash"]
    cfg = dict(cfg, hidden=(64, 64), nd=13, B=256)
    runs = []
    for evaluate in (False, True, False):
        reset_context()
        ctx = get_context()
        dev = ctx.device
        m = _model(cfg)
        tr = FusedTrainer(m, use_graph=True)
        pipe = tr.make_pipeline(cfg["B"], m.nf, m.nd)
        batches = [[_pinned(t) for t in _batch(cfg, s, dev)] for s in range(4)]
        val = _batch(cfg, 777, dev)
        met = BinaryMetrics(200, device=dev)
        for k in range(12):
            pipe.submit(*batches[k % 4])
            if evaluate and k % 3 == 2:
                tr.evaluate(*val, met)
        loss = pipe.last_loss()
        torch.cuda.synchronize()
        ctx.backend.engine.check()
        runs.append((loss, m.theta.clone().cpu(), m.accum.clone().cpu(), _rows(ctx, m)))
        if evaluate:
            assert met.result()["count"] == 4 * cfg["B"]
    (l0, t0, a0, r0), (l1, t1, a1, r1), (l2, t2, a2, r2) = runs
    if torch.equal(t0, t2) and l0 == l2:          # the step is deterministic here: demand bit identity
        assert l1 == l0 and torch.equal(t1, t0) and torch.equal(a1, a0)
        _rows_equal(r0, r1)
    else:                                         # atomics reorder fp32 sums from run to run
        spread = float((t0 - t2).abs().max())
        assert abs(l1 - l0) < 2e-4 and float((t1 - t0).abs().max()) <= 4 * spread + 1e-5, (l0, l1, l2, spread)


def test_validation_auc_on_planted_signal(cuda_context):
    """training on a planted logistic signal gives a validation AUC well above 0.5, and evaluate's metric equals
    the NumPy formula on predict's probabilities"""
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedCTR, FusedTrainer
    from openembedding_b200.models.metrics import BinaryMetrics, auc_from_counts
    dev = get_context().device
    vocab, B, nd = [200, 50, 1000, 30], 512, 4
    g = torch.Generator().manual_seed(3)
    w_true = torch.randn(vocab[0], generator=g) * 2
    v_true = torch.randn(nd, generator=g)

    def batch():
        ids = torch.stack([torch.randint(0, v, (B,), generator=g) for v in vocab], 1).contiguous()
        dense = torch.rand(B, nd, generator=g)
        p = torch.sigmoid(w_true[ids[:, 0]] + (dense - 0.5) @ v_true)
        return ids.to(dev), dense.to(dev), (torch.rand(B, generator=g) < p).float().to(dev)

    m = FusedCTR(vocab, num_dense=nd, embedding_dim=8, model="deepfm", batch=B, hidden=(64, 32),
                 sparse_optimizer={"category": "adam", "learning_rate": 0.05},
                 dense_optimizer={"category": "adam", "learning_rate": 0.01})
    tr = FusedTrainer(m, use_graph=True)
    for _ in range(150):
        tr.step(*batch())
    met, from_logits = BinaryMetrics(200, device=dev), BinaryMetrics(200, device=dev)
    probs, labels = [], []
    for _ in range(4):
        ids, dense, y = batch()
        tr.evaluate(ids, dense, y, met)
        probs.append(tr.predict(ids, dense).cpu().numpy())
        from_logits.update(m.logits, y)
        labels.append(y.cpu().numpy())
    r = met.result()
    pos, neg = _ref_counts(np.concatenate(probs), np.concatenate(labels))
    assert r["auc"] > 0.7, r
    assert r["auc"] == auc_from_counts(pos, neg) == from_logits.result()["auc"]
    assert r["count"] == 4 * B
