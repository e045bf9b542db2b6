"""Training-throughput sweep over the model zoo -- counterpart of the reference's
test/benchmark/criteo_deepctr.py (models WDL/DeepFM/xDeepFM/..., --embedding_dim 9|64,
--optimizer, --cache, --prefetch, batch 4096 per GPU; documents/en/benchmark.md:5-15).

    python benchmarks/criteo_deepctr.py --model DeepFM --embedding_dim 64              # 1 GPU
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 benchmarks/criteo_deepctr.py --model all

Synthetic Criteo-shaped data (26 log-uniform sparse ids + 13 dense); prints one JSON line per
(model, dim): samples/s over all ranks, device-timed with CUDA events, max over ranks.
`bench.py` at the repo root is the single-config headline driver; this is the sweep.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import openembedding_b200 as oe  # noqa: E402
from openembedding_b200.context import get_context, reset_context  # noqa: E402
from openembedding_b200.models.ctr import CRITEO_1TB_VOCAB_20M, CRITEO_KAGGLE_VOCAB, CTRModel  # noqa: E402
from openembedding_b200.models.trainer import Trainer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="DeepFM", help="LR|WDL|DeepFM|xDeepFM|DCN|AutoInt|all")
ap.add_argument("--embedding_dim", default="64", help="comma list, e.g. 9,64")
ap.add_argument("--optimizer", default="adagrad")
ap.add_argument("--batch_size", type=int, default=4096)
ap.add_argument("--vocab", default="1tb", choices=["kaggle", "1tb"])
ap.add_argument("--cache", action="store_true", default=True, help="replicate tables smaller than the batch")
ap.add_argument("--no-cache", dest="cache", action="store_false")
ap.add_argument("--prefetch", action="store_true", help="pinned-host input pipeline (pulling())")
ap.add_argument("--steps", type=int, default=100)
ap.add_argument("--warmup", type=int, default=10)
ap.add_argument("--cpu", action="store_true")
ap.add_argument("--engine", default="auto", choices=["auto", "fused", "eager"],
                help="fused: FusedCTR + FusedTrainer (WDL / DeepFM / xDeepFM / DCN / AutoInt, CUDA); eager: CTRModel + Trainer; "
                     "auto: fused where it exists")
ap.add_argument("--profile", default="", help="directory: write a chrome trace of 10 steps after the timed run "
                                                "(reference: --profile / TensorBoard profile_batch, criteo_deepctr.py:290-293), "
                                                "the vtimer table and the process RSS")
a = ap.parse_args()

world = int(os.environ.get("WORLD_SIZE", "1"))
use_cuda = torch.cuda.is_available() and not a.cpu
if use_cuda:
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
if world > 1:
    dist.init_process_group("nccl" if use_cuda else "gloo")
oe.flags.device = "cuda" if use_cuda else "cpu"
vocab = CRITEO_KAGGLE_VOCAB if a.vocab == "kaggle" else CRITEO_1TB_VOCAB_20M
if a.cpu:
    vocab = [min(v, 100000) for v in vocab]
models = ["LR", "WDL", "DeepFM", "xDeepFM", "DCN", "AutoInt"] if a.model == "all" else [a.model]
for name in models:
    for dim in (int(x) for x in a.embedding_dim.split(",")):
        reset_context()
        ctx = get_context()
        dev = ctx.device
        can_fuse = use_cuda and name.lower() in ("deepfm", "wdl", "xdeepfm", "dcn", "autoint") and a.batch_size % 128 == 0
        if a.engine == "fused" and not can_fuse:
            raise SystemExit("--engine fused: %s at batch %d has no fused step (CUDA, WDL / DeepFM / xDeepFM / DCN / "
                             "AutoInt, batch %% 128 == 0)" % (name, a.batch_size))
        fused = can_fuse and a.engine != "eager"
        cache = a.batch_size if a.cache else 0
        if fused:
            from openembedding_b200.models.fused_dense import FusedCTR, FusedTrainer
            m = FusedCTR(vocab, embedding_dim=dim, model=name.lower(), batch=a.batch_size, cache_threshold=cache,
                         sparse_optimizer={"category": a.optimizer})
            tr = FusedTrainer(m, use_graph=True)
        else:
            m = CTRModel(vocab, embedding_dim=dim, model=name.lower(), batch=a.batch_size, cache_threshold=cache,
                         sparse_optimizer={"category": a.optimizer},
                         compute_dtype=torch.bfloat16 if use_cuda else torch.float32)
            tr = Trainer(m, use_graph=use_cuda)
        g = torch.Generator().manual_seed(1 + ctx.rank)
        v = torch.tensor(vocab, dtype=torch.float64)
        data = []
        for _ in range(8):
            u = torch.rand((a.batch_size, 26), generator=g, dtype=torch.float64)
            ids = (torch.floor(torch.exp(u * torch.log(v))) - 1).clamp_(min=0).to(torch.int64).contiguous()
            data.append((ids, torch.rand(a.batch_size, 13, generator=g), (torch.rand(a.batch_size, generator=g) < 0.3).float()))
        if a.prefetch and use_cuda:
            pipe = tr.make_pipeline(a.batch_size, 26, 13)      # pinned H2D double buffering, loss read back lazily

            def step(i):
                pipe.submit(*data[i % 8])
                return None
        else:
            dd = [tuple(t.to(dev) for t in b) for b in data]
            step = lambda i: tr.step(*dd[i % 8])
        for i in range(a.warmup):
            step(i)
        ctx.barrier()
        if use_cuda:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(a.steps):
                loss = step(i)
            if loss is None:
                loss = pipe.last_loss()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.steps
        else:
            import time
            t0 = time.time()
            for i in range(a.steps):
                loss = step(i)
            ms = (time.time() - t0) * 1e3 / a.steps
        t = torch.tensor([ms], dtype=torch.float64, device=dev if use_cuda else "cpu")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            from openembedding_b200.utils import timers
            os.makedirs(a.profile, exist_ok=True)
            acts = [ProfilerActivity.CPU] + ([ProfilerActivity.CUDA] if use_cuda else [])
            timers.enabled = True
            with profile(activities=acts) as prof:
                for i in range(10):
                    step(i)
                if use_cuda:
                    torch.cuda.synchronize()
            timers.enabled = False
            trace = os.path.join(a.profile, "%s_dim%d_rank%d.trace.json" % (name, dim, ctx.rank))
            prof.export_chrome_trace(trace)
            if ctx.rank == 0:
                import psutil
                print("profile: %s ; rss %.1f GB" % (trace, psutil.Process().memory_info().rss / 2 ** 30), flush=True)
                print(prof.key_averages().table(sort_by="cuda_time_total" if use_cuda else "cpu_time_total", row_limit=15,
                                                max_name_column_width=60), flush=True)
        if ctx.rank == 0:
            print(json.dumps({"model": name, "embedding_dim": dim, "optimizer": a.optimizer, "n_gpus": world,
                              "batch_per_gpu": a.batch_size, "engine": "fused" if fused else "eager",
                              "ms_per_step": round(float(t), 4), "samples_per_s": round(a.batch_size * world / float(t) * 1e3),
                              "loss": round(float(loss), 5)}), flush=True)
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
