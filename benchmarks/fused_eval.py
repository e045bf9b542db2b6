"""Evaluation throughput of the fused models: FusedTrainer.evaluate (graph-captured forward-only pass + the streaming
AUC / log-loss kernel) against the training step of the same model in the same run, and against the eager CTRModel
forward under no_grad with the same metric.

    python benchmarks/fused_eval.py                                  # deepfm, wdl, xdeepfm, dcn at dim 9 and 64
    python benchmarks/fused_eval.py --model deepfm --embedding_dim 64 --steps 200

Synthetic Criteo-shaped data (26 log-uniform sparse ids + 13 dense), batch 4096, one GPU. Device-timed with CUDA
events around ``--steps`` calls after ``--warmup`` calls; prints the card and its power limit, then one JSON line per
(model, dim).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import openembedding_b200 as oe  # noqa: E402
from openembedding_b200.context import get_context, reset_context  # noqa: E402
from openembedding_b200.models.ctr import CRITEO_1TB_VOCAB_20M, CRITEO_KAGGLE_VOCAB, CTRModel  # noqa: E402
from openembedding_b200.models.fused_dense import FusedCTR, FusedTrainer  # noqa: E402
from openembedding_b200.models.metrics import BinaryMetrics  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="all", help="deepfm|wdl|xdeepfm|dcn|all")
ap.add_argument("--embedding_dim", default="9,64", help="comma list")
ap.add_argument("--batch_size", type=int, default=4096)
ap.add_argument("--vocab", default="kaggle", choices=["kaggle", "1tb"])
ap.add_argument("--steps", type=int, default=100)
ap.add_argument("--warmup", type=int, default=10)
ap.add_argument("--no-eager", dest="eager", action="store_false", help="skip the eager CTRModel baseline")
a = ap.parse_args()

if not torch.cuda.is_available():
    raise SystemExit("benchmarks/fused_eval.py measures on a CUDA device")
oe.flags.device = "cuda"
vocab = CRITEO_KAGGLE_VOCAB if a.vocab == "kaggle" else CRITEO_1TB_VOCAB_20M
B = a.batch_size


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], stdout=subprocess.PIPE, text=True, timeout=30).stdout
        name, power = [s.strip() for s in q.strip().split(",")]
        return name, power
    except Exception:           # no nvidia-smi: the name from the runtime, power limit unknown
        return torch.cuda.get_device_name(), "unknown"


def data(dev, n=8, seed=1):
    g = torch.Generator().manual_seed(seed)
    v = torch.tensor(vocab, dtype=torch.float64)
    out = []
    for _ in range(n):
        u = torch.rand((B, len(vocab)), generator=g, dtype=torch.float64)
        ids = (torch.floor(torch.exp(u * torch.log(v))) - 1).clamp_(min=0).to(torch.int64).contiguous()
        out.append((ids.to(dev), torch.rand(B, 13, generator=g).to(dev), (torch.rand(B, generator=g) < 0.25).float().to(dev)))
    return out


def timed(fn):
    """ms per call over a.steps calls, device-timed, after a.warmup calls"""
    for i in range(a.warmup):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.steps


name, power = card()
print(json.dumps({"card": name, "power_limit": power, "batch": B, "vocab": a.vocab, "steps": a.steps}), flush=True)
models = ["deepfm", "wdl", "xdeepfm", "dcn"] if a.model == "all" else [a.model.lower()]
for model in models:
    for dim in (int(x) for x in a.embedding_dim.split(",")):
        reset_context()
        dev = get_context().device
        dd = data(dev)
        val = data(dev, seed=2)
        m = FusedCTR(vocab, embedding_dim=dim, model=model, batch=B, cache_threshold=B)
        tr = FusedTrainer(m, use_graph=True)
        train_ms = timed(lambda i: tr.step(*dd[i % 8], next_ids=dd[(i + 1) % 8][0]))
        met = BinaryMetrics(200, device=dev)
        eval_ms = timed(lambda i: tr.evaluate(*val[i % 8], met))
        auc = met.result()["auc"]
        row = {"model": model, "dim": dim, "eval_ms": round(eval_ms, 4), "eval_samples_per_s": round(B / eval_ms * 1e3),
               "train_ms": round(train_ms, 4), "train_samples_per_s": round(B / train_ms * 1e3),
               "kernels_per_eval": m.kernels_per_eval(metric=True), "auc": round(auc, 6)}
        del tr, m
        if a.eager:
            reset_context()
            dev = get_context().device
            em = CTRModel(vocab, embedding_dim=dim, model=model, batch=B, cache_threshold=B)
            emet = BinaryMetrics(200, device=dev)

            def eager_eval(i):
                ids, dense, labels = val[i % 8]
                with torch.no_grad():
                    emet.update(em(ids, dense), labels)
            ems = timed(eager_eval)
            row.update({"eager_eval_ms": round(ems, 4), "eager_eval_samples_per_s": round(B / ems * 1e3)})
            del em
        row.update({"card": name, "power_limit": power})
        print(json.dumps(row), flush=True)
reset_context()
