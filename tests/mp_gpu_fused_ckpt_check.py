"""torchrun script: checkpoints of a fused DeepFM on W ranks. Run 1 trains 2k batches through a graph-driven pipeline
and saves after k (prefetch armed); run 2 builds the model with another seed, loads and trains the last k; run 3
trains all 2k without a save. Run 2 must train as run 1 (bit for bit when runs 1 and 3 agree bit for bit, otherwise
within a few times their spread), and theta must be bit-identical across the ranks. Rank 0 leaves the saved dense state
and every rank its table rows at the time of the save under ``argv[1]``, for the single-rank load of
tests/test_gpu_fused_checkpoint.py. Launched by that test."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VOCAB = [1000, 50, 20000, 7, 3000] + [300] * 21
B, K = 256, 3


def model(seed):
    from openembedding_b200.models.fused_dense import FusedCTR
    return FusedCTR(VOCAB, embedding_dim=16, model="deepfm", batch=B, cache_threshold=64, hidden=(64, 32), seed=seed,
                    sparse_optimizer={"category": "adam", "learning_rate": 0.05},
                    dense_optimizer={"category": "adam", "learning_rate": 0.01})


def rows(ctx, m):
    out = []
    for meta in m.sparse.metas:
        parts = [(np.array(i, dtype=np.int64) * meta.shard_num + ctx.backend.shard_id(meta), np.array(w, copy=True),
                  np.array(s, copy=True)) for i, w, s in ctx.backend.iter_local_rows(meta, 1 << 16)]
        if not parts:
            out.append((np.zeros(0, np.int64), np.zeros((0, meta.dim), np.float32), np.zeros((0, 0), np.float32)))
            continue
        idx = np.concatenate([p[0] for p in parts])
        o = np.argsort(idx)
        out.append((idx[o], np.concatenate([p[1] for p in parts])[o], np.concatenate([p[2] for p in parts])[o]))
    return out


def run(batches, seed=0, load=None, save_at=None, save_path=None, out=None):
    from openembedding_b200.context import get_context, reset_context
    from openembedding_b200.models.fused_dense import FusedTrainer
    reset_context()
    ctx = get_context()
    m = model(seed)
    if load is not None:
        m.load(load)
    tr = FusedTrainer(m, use_graph=True)
    pipe = tr.make_pipeline(B, m.nf, m.nd)
    for b in batches:
        pipe.submit(*b)
        if save_at is not None and pipe.trained == save_at:
            assert tr._x32_key is not None
            m.save(save_path)
            if out is not None:
                if ctx.rank == 0:
                    torch.save(m.dense_state_dict(), os.path.join(out, "dense.pt"))
                np.savez(os.path.join(out, "rows_%d.npz" % ctx.rank),
                         **{"%s_%d" % (k, t): a for t, r in enumerate(rows(ctx, m)) for k, a in zip("iws", r)})
            save_at = None
    loss = pipe.last_loss()
    torch.cuda.synchronize()
    ctx.backend.engine.check()
    return loss, [t.clone() for t in (m.theta, m.accum, m.accum2, m.opt_step)]


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import openembedding_b200 as oe
    oe.flags.device = "cuda"
    out = sys.argv[1]
    dev = torch.device("cuda", local)

    def batch(seed):
        g = torch.Generator().manual_seed(seed)
        ids = torch.stack([torch.randint(0, v, (B,), generator=g) for v in VOCAB], 1).contiguous()
        return [ids.pin_memory(), torch.rand(B, 13, generator=g).pin_memory(),
                (torch.rand(B, generator=g) < 0.3).float().pin_memory()]

    batches = [batch(100 * rank + s) for s in range(2 * K)]
    ck = os.path.join(out, "ck")
    l1, s1 = run(batches, save_at=K, save_path=ck, out=out)
    l2, s2 = run(batches[K:], seed=1, load=ck)
    l3, s3 = run(batches)
    if l1 == l3 and all(torch.equal(a, b) for a, b in zip(s1, s3)):
        assert l2 == l1 and all(torch.equal(a, b) for a, b in zip(s1, s2)), (l1, l2)
    else:
        assert abs(l2 - l1) <= 4 * abs(l1 - l3) + 2e-4, (l1, l2, l3)
        for a, b, r in zip(s1, s2, s3):         # the rule of tests/test_gpu_fused_checkpoint.py: _same_trajectory
            d, s = (a.double() - b.double()).abs(), (a.double() - r.double()).abs()
            assert float(d.max()) <= 8 * float(s.max()) + 1e-4 and float(d.mean()) <= 8 * float(s.mean()) + 1e-7
    # the dense state is replicated: theta bit-identical on every rank
    th = [torch.empty_like(s1[0]) for _ in range(world)]
    dist.all_gather(th, s1[0])
    assert all(torch.equal(t.view(torch.int32), th[0].view(torch.int32)) for t in th)
    dist.barrier()
    if rank == 0:
        print("MP_GPU_FUSED_CKPT_PASSED loss %.6f %.6f %.6f" % (l1, l2, l3))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
