"""DeepFM / WDL / xDeepFM / DCN / AutoInt on Criteo-shaped data -- counterpart of the reference's
examples/criteo_deepctr_network{,_mirrored,_mpi}.py and test/benchmark/criteo_deepctr.py.

single GPU / CPU :  python examples/criteo_deepctr_network.py --model DeepFM
multi GPU        :  python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 \
                        examples/criteo_deepctr_network.py --model DeepFM --fused
(torchrun replaces horovodrun / MirroredStrategy / mpirun of the reference: one rank per GPU,
dense gradients are summed across ranks, the embedding tables are row-sharded over the GPUs)
"""
import argparse
import os
import sys

import pandas
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import openembedding_b200 as oe  # noqa: E402
import openembedding_b200.torch as embed  # noqa: E402
from openembedding_b200.context import get_context  # noqa: E402
from openembedding_b200.models.ctr import CTRModel  # noqa: E402
from openembedding_b200.models.trainer import Trainer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--data", default="")
ap.add_argument("--model", default="DeepFM", choices=["LR", "WDL", "DeepFM", "xDeepFM", "DCN", "AutoInt"])
ap.add_argument("--optimizer", default="Adagrad", choices=["Adam", "Adagrad", "Ftrl", "SGD"])
ap.add_argument("--embedding_dim", type=int, default=9)
ap.add_argument("--batch_size", type=int, default=16)
ap.add_argument("--epochs", type=int, default=3)
ap.add_argument("--cache", action="store_true", help="replicate tables smaller than the batch (sparse_as_dense)")
ap.add_argument("--fused", action="store_true", help="whole step on the hand-written kernels (CUDA, DeepFM/WDL/xDeepFM/DCN/AutoInt)")
ap.add_argument("--validation_batches", type=int, default=0,
                help="with --fused: hold out the last N batches of each rank, print val_auc / val_logloss per epoch")
ap.add_argument("--cpu", action="store_true")
ap.add_argument("--checkpoint", default="")
ap.add_argument("--load", default="")
ap.add_argument("--save", default="")
ap.add_argument("--export", default="", help="with --fused: stand-alone PyTorch model file (no engine, no GPU needed)")
args = ap.parse_args()

world = int(os.environ.get("WORLD_SIZE", "1"))
if world > 1:
    local = int(os.environ.get("LOCAL_RANK", "0"))
    use_cuda = torch.cuda.is_available() and not args.cpu
    if use_cuda:
        torch.cuda.set_device(local)
    dist.init_process_group("nccl" if use_cuda else "gloo")
oe.flags.device = "cpu" if args.cpu else "auto"
ctx = get_context()

if args.data:
    data = pandas.read_csv(args.data)
else:
    from make_sample_data import make
    data = make(128)
vocab = [int(data["C%d" % i].max()) + 1 for i in range(1, 27)]
n = len(data) // (world * args.batch_size) * args.batch_size
part = data.iloc[ctx.rank * n:(ctx.rank + 1) * n]
ids = torch.tensor(part[["C%d" % i for i in range(1, 27)]].values, dtype=torch.int64)
dense = torch.tensor(part[["I%d" % i for i in range(1, 14)]].values, dtype=torch.float32)
label = torch.tensor(part["label"].values, dtype=torch.float32)

if args.validation_batches and not args.fused:
    raise SystemExit("--validation_batches: evaluation runs on the fused step (--fused)")
if args.export and not args.fused:
    raise SystemExit("--export: the stand-alone export is of the fused models (--fused)")
n_val = args.validation_batches * args.batch_size
if n_val >= n:
    raise SystemExit("--validation_batches %d leaves no training batch" % args.validation_batches)
n_train = n - n_val

sparse_opt = {"category": args.optimizer.lower()}
cache = args.batch_size if args.cache else 0
if args.fused:
    if args.model not in ("WDL", "DeepFM", "xDeepFM", "DCN", "AutoInt"):
        raise SystemExit("--fused: WDL, DeepFM, xDeepFM, DCN or AutoInt")
    from openembedding_b200.models.fused_dense import FusedCTR, FusedTrainer
    model = FusedCTR(vocab, embedding_dim=args.embedding_dim, model=args.model.lower(), batch=args.batch_size,
                     sparse_optimizer=sparse_opt, cache_threshold=cache)
    trainer = FusedTrainer(model, use_graph=True)
else:
    model = CTRModel(vocab, embedding_dim=args.embedding_dim, model=args.model.lower(), batch=args.batch_size,
                     sparse_optimizer=sparse_opt, cache_threshold=cache,
                     compute_dtype=torch.float32 if ctx.device.type == "cpu" else torch.bfloat16)
    trainer = Trainer(model, use_graph=False)
if args.load:
    if args.fused:               # dense weights, dense optimizer and the tables
        model.load(args.load)
    else:
        embed.load_server_model(model, args.load)
for epoch in range(args.epochs):
    tot, cnt = 0.0, 0
    for i in range(0, n_train, args.batch_size):
        sl = slice(i, i + args.batch_size)
        loss = trainer.step(ids[sl].contiguous().to(ctx.device), dense[sl].to(ctx.device), label[sl].to(ctx.device))
        tot += float(loss)
        cnt += 1
    if ctx.rank == 0:
        print("epoch %d loss %.4f" % (epoch + 1, tot / max(cnt, 1)))
    if n_val:
        from openembedding_b200.models.metrics import BinaryMetrics
        metrics = BinaryMetrics()          # tf.keras.metrics.AUC(): 200 thresholds
        for i in range(n_train, n, args.batch_size):
            sl = slice(i, i + args.batch_size)
            trainer.evaluate(ids[sl].contiguous().to(ctx.device), dense[sl].to(ctx.device), label[sl].to(ctx.device),
                             metrics)
        r = metrics.result()                # all ranks: the counters are summed over them
        if ctx.rank == 0:
            print("epoch %d val_auc %.4f val_logloss %.4f" % (epoch + 1, r["auc"], r["logloss"]))
    if args.checkpoint:                                                            # include optimizer
        if args.fused:
            model.save(args.checkpoint + str(epoch + 1))
        else:
            embed.save_server_model(model, args.checkpoint + str(epoch + 1))
if args.save:
    if args.fused:
        model.save(args.save, include_optimizer=False)
    else:
        embed.save_server_model(model, args.save, include_optimizer=False)
if args.export:
    model.save_as_original_model(args.export)
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
