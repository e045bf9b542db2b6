"""torchrun script: the fused AutoInt step (FusedCTR model="autoint" + FusedTrainer, graph on) on W ranks. Checks that the
loss falls, that the dense replicas -- attention matrices and w_att included -- stay bit-identical on every rank and that
the engine reports no error. Prints the sum of |theta| so that the ride-along all-reduce (default) can be compared with
the stand-alone one (EXB_AR_RIDER=0). Launched by tests/test_gpu_fused_autoint.py."""
import os
import sys

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
    oe.flags.device = "cuda"
    ctx = get_context()
    vocab = [1000, 50, 20000, 7, 3000] + [300] * 21
    B = 256
    m = FusedCTR(vocab, embedding_dim=9, model="autoint", batch=B, cache_threshold=64, lr=0.05,
                 sparse_optimizer={"category": "adagrad", "learning_rate": 0.05})
    tr = FusedTrainer(m, use_graph=True)
    g = torch.Generator().manual_seed(7 + rank)
    ids = torch.stack([torch.randint(0, v, (B,), generator=g) for v in vocab], dim=1).contiguous().to(ctx.device)
    dense = torch.rand(B, 13, generator=g).to(ctx.device)
    labels = (torch.rand(B, generator=g) < 0.3).float().to(ctx.device)
    losses = [float(tr.step(ids, dense, labels, next_ids=ids)) for _ in range(12)]
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    assert losses[-1] < losses[0] - 0.01, losses
    theta = m.theta.clone()
    ref = theta.clone()
    dist.broadcast(ref, src=0)
    assert torch.equal(theta, ref), "dense replicas diverged: %g" % float((theta - ref).abs().max())
    dist.barrier()
    if rank == 0:
        print("MP_GPU_FUSED_AUTOINT_PASSED loss %.4f -> %.4f theta_sum %.17g rider %d" %
              (losses[0], losses[-1], float(theta.double().abs().sum()), int(m._rider)))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
