"""The streaming AUC / log-loss kernel (csrc/cuda/metric_kernels.cu through models/metrics.py: BinaryMetrics)
against NumPy: bucket counts exactly, AUC and log loss in fp64."""
import numpy as np
import pytest
import torch

from openembedding_b200.models import metrics as M

pytestmark = pytest.mark.gpu


def _probs_f32(z):
    """p = 1 / (1 + exp(-z)) as the kernels compute it, read back from a CUDA float32 evaluation"""
    z = torch.as_tensor(z, dtype=torch.float32, device="cuda")
    return (1.0 / (1.0 + torch.exp(-z))).cpu().numpy()


def _ref_counts(p, y, T):
    """NumPy direct comparison p > t_i (float32) per threshold -> the bucket counts the kernel keeps"""
    t = M.keras_thresholds(T)
    above = (np.asarray(p, dtype=np.float32)[:, None] > t[None, :]).sum(1)
    real = np.asarray(y) != 0
    return np.bincount(above[real], minlength=T + 1), np.bincount(above[~real], minlength=T + 1)


def _logits_on_thresholds(T, rng):
    """logits whose float32 sigmoid lands exactly on a threshold or on a neighbour of one"""
    t = M.keras_thresholds(T)[1:-1].astype(np.float32)
    cand = []
    for p in t[rng.choice(len(t), size=min(len(t), 300), replace=False)] if len(t) else []:
        for q in (np.nextafter(p, np.float32(0)), p, np.nextafter(p, np.float32(1))):
            q = float(np.clip(q, 1e-6, 1 - 1e-6))
            cand.append(np.log(q / (1 - q)))
    z = np.array(cand, dtype=np.float32)
    # nudge each logit by a few ulps so that some sigmoids hit the table values exactly
    zz = np.concatenate([z] + [np.nextafter(z, np.float32(s) * np.inf).astype(np.float32) for s in (1, -1)])
    return zz.astype(np.float32)


def _run(metric, batches, n=None):
    for z, y in batches:
        metric.update(torch.as_tensor(z, device="cuda"), torch.as_tensor(y, device="cuda"), n=n)
    torch.cuda.synchronize()


@pytest.mark.parametrize("T", [3, 200, 8192])
def test_counts_exact_and_auc_logloss(cuda_context, T):
    rng = np.random.default_rng(T)
    batches = []
    for k in range(7):                  # many batches, n not a multiple of 32
        n = int(rng.integers(1, 3000)) | 1
        z = (rng.standard_normal(n) * 3).astype(np.float32)
        y = (rng.random(n) < 0.3).astype(np.float32)
        batches.append((z, y))
    zt = _logits_on_thresholds(T, rng)
    batches.append((zt, (rng.random(zt.size) < 0.5).astype(np.float32)))
    a, b = zt[:333], zt[-77:]
    batches.append((a, np.ones(a.size, np.float32)))                 # all positive
    batches.append((b, np.zeros(b.size, np.float32)))                # all negative
    batches.append((np.array([0.0, 40.0, -40.0, 1e-8], np.float32), np.array([2.0, 1.0, 0.0, -1.0], np.float32)))
    m = M.BinaryMetrics(T, device="cuda")
    _run(m, batches)
    z = np.concatenate([b[0] for b in batches])
    y = np.concatenate([b[1] for b in batches])
    p = _probs_f32(z)
    assert np.isin(p, M.keras_thresholds(T)).any(), "no probability lies exactly on a threshold"
    pos, neg = _ref_counts(p, y, T)
    gp, gn, loss, count = m.counts()
    assert np.array_equal(gp, pos) and np.array_equal(gn, neg)
    assert count == z.size
    r = m.result()
    assert r["count"] == z.size and r["positives"] == int((y != 0).sum())
    assert r["auc"] == M.auc_from_counts(pos, neg)
    zd, yd = z.astype(np.float64), y.astype(np.float64)
    ref_loss = np.sum(np.maximum(zd, 0) - zd * yd + np.log1p(np.exp(-np.abs(zd))))
    assert abs(loss - ref_loss) <= 1e-6 * abs(ref_loss)
    assert r["logloss"] == pytest.approx(ref_loss / z.size, rel=1e-6)


def test_auc_close_to_rank_auc(cuda_context):
    """with 8192 thresholds the interpolated AUC is within 1e-3 of the exact Mann-Whitney AUC"""
    from scipy.stats import rankdata
    rng = np.random.default_rng(5)
    n = 200000
    y = (rng.random(n) < 0.25).astype(np.float32)
    z = (rng.standard_normal(n) + 1.2 * y).astype(np.float32)
    m = M.BinaryMetrics(8192, device="cuda")
    _run(m, [(z, y)])
    p = _probs_f32(z).astype(np.float64)
    r = rankdata(p)
    npos = int(y.sum())
    exact = (r[y != 0].sum() - npos * (npos + 1) / 2) / (npos * (n - npos))
    assert abs(m.result()["auc"] - exact) < 1e-3, (m.result()["auc"], exact)


def test_rows_past_n_reset_and_graph(cuda_context):
    rng = np.random.default_rng(3)
    B = 4096
    z = torch.as_tensor((rng.standard_normal(B) * 2).astype(np.float32), device="cuda")
    y = torch.as_tensor((rng.random(B) < 0.4).astype(np.float32), device="cuda")
    n_dev = torch.zeros(1, dtype=torch.int32, device="cuda")
    ref = M.BinaryMetrics(200, device="cuda")
    got = M.BinaryMetrics(200, device="cuda")
    got.update(z, y)
    got.reset()
    torch.cuda.synchronize()
    assert int(got.hist.abs().sum()) == 0 and int(got.count) == 0 and float(got.loss_sum) == 0.0
    # one captured graph, n read on the device
    n_dev.fill_(1)
    got.update(z, y, n=n_dev)              # warm-up outside the capture
    torch.cuda.synchronize()
    got.reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got.update(z, y, n=n_dev)
    for n in (B, 1000, 31, 4095):
        n_dev.fill_(n)
        g.replay()
        ref.update(z[:n], y[:n])
    torch.cuda.synchronize()
    assert torch.equal(got.hist, ref.hist) and torch.equal(got.count, ref.count)
    assert int(got.count) == B + 1000 + 31 + 4095
    assert float(got.loss_sum) == pytest.approx(float(ref.loss_sum), rel=1e-12)
    # an int n counts the first n rows only
    a, b = M.BinaryMetrics(200, device="cuda"), M.BinaryMetrics(200, device="cuda")
    a.update(z, y, n=100)
    b.update(z[:100].clone(), y[:100].clone())
    torch.cuda.synchronize()
    assert torch.equal(a.hist, b.hist) and torch.equal(a.count, b.count)


@pytest.mark.parametrize("T", [1, 8193])
def test_threshold_range(cuda_context, T):
    with pytest.raises(ValueError):
        M.BinaryMetrics(T, device="cuda")


def test_eager_ctrmodel_logits(cuda_context):
    """the metric takes any CUDA logits: the eager CTRModel (LR included) under no_grad"""
    from openembedding_b200.models.ctr import CTRModel
    vocab = [100, 50, 7]
    B = 256
    torch.manual_seed(0)
    ids = torch.stack([torch.randint(0, v, (B,)) for v in vocab], 1).cuda()
    dense = torch.rand(B, 13, device="cuda")
    y = (torch.rand(B, device="cuda") < 0.3).float()
    for model in ("lr", "deepfm"):
        net = CTRModel(vocab, num_dense=13, embedding_dim=8, model=model, batch=B)
        with torch.no_grad():
            z = net(ids, dense).reshape(-1)
        m = M.BinaryMetrics(200, device="cuda")
        m.update(z, y)
        torch.cuda.synchronize()
        pos, neg = _ref_counts(_probs_f32(z.float().cpu().numpy()), y.cpu().numpy(), 200)
        gp, gn, _, count = m.counts()
        assert np.array_equal(gp, pos) and np.array_equal(gn, neg) and count == B
