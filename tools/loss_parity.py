#!/usr/bin/env python
"""Loss-trajectory parity: the fused engine (bf16 wgmma GEMMs, fp32 tables / master weights) vs the plain-PyTorch
baseline in FP32 (benchmarks/nccl_baseline.py), SAME initial weights, SAME batches, SAME optimizers.

Answers "does the bf16 dense path train like an fp32 model?" (VERDICT r1, weak #3). Prints one JSON line with the
mean / max absolute loss difference per window of steps and the final-window means.

    python tools/loss_parity.py --steps 2000 --dim 16 --vocab tiny
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--dim", type=int, default=16)
    ap.add_argument("--model", default="deepfm")
    ap.add_argument("--vocab", default="tiny", choices=["tiny", "kaggle"])
    ap.add_argument("--lr", type=float, default=0.01)
    ap.add_argument("--window", type=int, default=100)
    a = ap.parse_args()
    import openembedding_b200 as oe
    from benchmarks.nccl_baseline import NcclBaselineCTR
    from openembedding_b200.context import get_context
    from openembedding_b200.models.ctr import CRITEO_KAGGLE_VOCAB
    from openembedding_b200.models.fused_dense import FusedCTR, FusedTrainer
    oe.flags.device = "cuda"
    ctx = get_context()
    dev = ctx.device
    vocab = CRITEO_KAGGLE_VOCAB if a.vocab == "kaggle" else [min(v, 10007) for v in CRITEO_KAGGLE_VOCAB]
    sparse_opt = {"category": "adagrad", "learning_rate": a.lr}
    fused = FusedCTR(vocab, embedding_dim=a.dim, model=a.model, batch=a.batch, cache_threshold=64, lr=a.lr,
                     sparse_optimizer=sparse_opt)
    tr = FusedTrainer(fused, use_graph=True)
    res = {}
    for name, dt in (("baseline_fp32", torch.float32), ("baseline_bf16", torch.bfloat16)):
        base = NcclBaselineCTR(vocab, embedding_dim=a.dim, model=a.model, batch=a.batch, cache_threshold=64,
                               compute_dtype=dt, lr=a.lr, sparse_lr=a.lr, device=dev)
        base.load_from_fused(fused)
        res[name] = base
    g = torch.Generator().manual_seed(11)
    v = torch.tensor(vocab, dtype=torch.float64)
    wtrue = torch.randn(len(vocab), generator=g)
    curves = {"fused_bf16": [], "baseline_fp32": [], "baseline_bf16": []}
    for step in range(a.steps):
        u = torch.rand((a.batch, len(vocab)), generator=g, dtype=torch.float64)
        ids = (torch.floor(torch.exp(u * torch.log(v))) - 1).clamp_(min=0).to(torch.int64)
        dense = torch.rand((a.batch, 13), generator=g)
        # a learnable synthetic target: the label depends on a few id parities and dense features
        logit = ((ids % 2).double() * 2 - 1).float() @ wtrue * 0.3 + (dense[:, :4].sum(1) - 2.0)
        labels = (torch.rand(a.batch, generator=g) < torch.sigmoid(logit)).float()
        ids, dense, labels = ids.to(dev), dense.to(dev), labels.to(dev)
        curves["fused_bf16"].append(float(tr.step(ids, dense, labels)))
        for name in ("baseline_fp32", "baseline_bf16"):
            curves[name].append(float(res[name].step(ids, dense, labels)))
    ctx.backend.engine.check()
    t = {k: torch.tensor(c) for k, c in curves.items()}
    W = a.window

    def windows(x):
        n = x.numel() // W * W
        return x[:n].view(-1, W).mean(1)
    out = {"steps": a.steps, "batch": a.batch, "dim": a.dim, "model": a.model, "vocab": a.vocab, "lr": a.lr, "window": W,
           "first_window": {k: float(windows(x)[0]) for k, x in t.items()},
           "last_window": {k: float(windows(x)[-1]) for k, x in t.items()},
           "fused_vs_fp32": {"mean_abs_diff": float((t["fused_bf16"] - t["baseline_fp32"]).abs().mean()),
                             "max_abs_diff": float((t["fused_bf16"] - t["baseline_fp32"]).abs().max()),
                             "max_window_diff": float((windows(t["fused_bf16"]) - windows(t["baseline_fp32"])).abs().max())},
           "bf16_baseline_vs_fp32": {"mean_abs_diff": float((t["baseline_bf16"] - t["baseline_fp32"]).abs().mean()),
                                     "max_window_diff": float((windows(t["baseline_bf16"]) - windows(t["baseline_fp32"])).abs().max())},
           "curve_windows": {k: [round(float(y), 5) for y in windows(x)] for k, x in t.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
