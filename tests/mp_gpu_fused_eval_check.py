"""torchrun script: distributed evaluation of a fused DeepFM (FusedTrainer.evaluate + BinaryMetrics) on W ranks.
After a few training steps every rank evaluates its own disjoint slice of one validation set; the all-reduced
counters of ``BinaryMetrics.result()`` must equal those of rank 0 evaluating the whole set alone. Launched by
tests/test_gpu_fused_eval_mp.py."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import openembedding_b200 as oe
    from openembedding_b200.context import get_context
    from openembedding_b200.models.fused_dense import FusedCTR, FusedTrainer
    from openembedding_b200.models.metrics import BinaryMetrics
    oe.flags.device = "cuda"
    ctx = get_context()
    vocab = [1000, 50, 20000, 7, 3000] + [300] * 21
    B = 256
    m = FusedCTR(vocab, embedding_dim=16, model="deepfm", batch=B, cache_threshold=64, lr=0.05,
                 sparse_optimizer={"category": "adagrad", "learning_rate": 0.05})
    tr = FusedTrainer(m, use_graph=True)

    def batch(seed, n):
        g = torch.Generator().manual_seed(seed)
        ids = torch.stack([torch.randint(0, v, (n,), generator=g) for v in vocab], dim=1).contiguous()
        return ids.to(ctx.device), torch.rand(n, 13, generator=g).to(ctx.device), \
            (torch.rand(n, generator=g) < 0.3).float().to(ctx.device)

    ids, dense, labels = batch(7 + rank, B)
    for _ in range(6):
        tr.step(ids, dense, labels, next_ids=ids)
    # one validation set of 3 * B rows, identical on every rank; rank r takes rows [r * n, (r + 1) * n)
    vids, vdense, vlab = batch(1000, 3 * B)
    n = 3 * B // world
    mine = BinaryMetrics(200)
    for lo in range(rank * n, (rank + 1) * n, B):
        hi = min(lo + B, (rank + 1) * n)
        tr.evaluate(vids[lo:hi], vdense[lo:hi], vlab[lo:hi], mine)
    # the union on this rank alone (no collective: counts of the local accumulator, before any all-reduce)
    whole = BinaryMetrics(200)
    for lo in range(0, world * n, B):
        hi = min(lo + B, world * n)
        tr.evaluate(vids[lo:hi], vdense[lo:hi], vlab[lo:hi], whole)
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    pos, neg, loss, count = mine.counts()           # collective
    local = torch.cat([whole.hist.reshape(-1), whole.count]).cpu().numpy()
    T1 = whole.num_thresholds + 1
    assert count == world * n == int(local[-1]), (count, local[-1])
    assert np.array_equal(pos, local[:T1]) and np.array_equal(neg, local[T1:2 * T1])
    assert abs(loss - float(whole.loss_sum)) <= 1e-9 * abs(float(whole.loss_sum))
    r = mine.result()                               # collective
    dist.barrier()
    if rank == 0:
        print("MP_GPU_FUSED_EVAL_PASSED auc %.6f logloss %.6f count %d" % (r["auc"], r["logloss"], r["count"]))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
