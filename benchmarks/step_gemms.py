"""Time the nine GEMMs of the fused DeepFM training step one by one, at both wgmma tile widths.

    python benchmarks/step_gemms.py                       # batch 4096, dim 64, hidden (400, 400, 400)
    python benchmarks/step_gemms.py --steps 500 --widths 64,128
    python benchmarks/step_gemms.py --widths 64 --mc 0,7 --rounds 3     # A-tile multicast off / on, alternated

For every GEMM of the step (fwd1..3, then dX3, dW3, dX2, dW2, dX1 with the FM term, dW1 split-K) this prints, per
single-launch tile width BN: the time of the single launch (``gemm_nt`` / ``gemm_tn``), the achieved TFLOP/s and the
operand bytes the tiles read from L2, and the time of the same GEMM as a one-GEMM persistent chain (64-wide tiles).
A last row, "dX1 (no FM)", is dX1 with a plain fp32 store (``fm_cols=0``): the same GEMM without the FM epilogue's
operands, so its gap to "dX1 (FM)" bounds what the FM epilogue costs. It also times the whole forward (three single launches, and the forward chain) and the whole backward (six single
launches, and the backward chain that the step runs). Device-timed with CUDA events over
``--steps`` launches after ``--warmup``; the card and its power limit are read in the same run.

L2 operand bytes of a tiled GEMM: every 128 x BN output tile reads its 128 rows of A and its BN rows of B over the
whole K range (split-K only cuts that range into pieces), so

    bytes = M*K*2 * ceil(N / BN) + N*K*2 * ceil(M / 128)

With the A tile multicast to the C CTAs of a cluster (consecutive N tiles), A is read once per cluster: the first
term becomes M*K*2 * ceil(ceil(N / BN) / C).

The single-launch width follows ``EXB_GEMM_BN`` and the single-launch A-tile multicast ``EXB_GEMM_MC`` (``--mc``: the
cluster size is the largest divisor of the N-tile count up to that value). Both are read once per process, so each
combination runs in a child process of its own; with ``--rounds R`` the whole list of combinations runs R times in
turn, so that the arms are compared under the same drift of a shared card. The GEMM shapes depend on batch, dim,
hidden and the dense-feature count only, so the embedding tables are kept small. Output: one JSON line per
measurement, then a markdown table.
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=4096)
ap.add_argument("--dim", type=int, default=64)
ap.add_argument("--steps", type=int, default=300)
ap.add_argument("--warmup", type=int, default=30)
ap.add_argument("--widths", default="64,128", help="tile widths to time, comma list")
ap.add_argument("--mc", default="0", help="EXB_GEMM_MC values to time, comma list (0: no multicast)")
ap.add_argument("--rounds", type=int, default=1, help="run the list of combinations this many times, alternated")
ap.add_argument("--child", type=int, default=0, help=argparse.SUPPRESS)   # single-launch width of this process
a = ap.parse_args()

BM = 128


def l2_bytes(M, N, K, bn, c=1):
    return M * K * 2 * math.ceil(math.ceil(N / bn) / c) + N * K * 2 * math.ceil(M / BM)


def single_mc(mc, n_tiles):
    """cluster size of a single launch under EXB_GEMM_MC = mc (gemm_wgmma.cu pick_mc)"""
    return max([1] + [c for c in range(2, min(mc, 8) + 1) if n_tiles % c == 0])


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], stdout=subprocess.PIPE, text=True, timeout=30).stdout
        name, power = [s.strip() for s in q.strip().split(",")]
        return name, power
    except Exception:           # no nvidia-smi: the name from the runtime, power limit unknown
        return torch.cuda.get_device_name(), "unknown"


def child(bn, mc):
    import torch
    import openembedding_b200 as oe
    from openembedding_b200.context import get_context
    from openembedding_b200.models.ctr import CRITEO_KAGGLE_VOCAB
    from openembedding_b200.models.fused_dense import FusedCTR
    from openembedding_b200.ops import gemm as G

    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/step_gemms.py measures on a CUDA device")
    oe.flags.device = "cuda"
    dev = get_context().device
    vocab = [min(v, 10007) for v in CRITEO_KAGGLE_VOCAB]
    B = a.batch
    torch.manual_seed(1234)
    m = FusedCTR(vocab, num_dense=13, embedding_dim=a.dim, model="deepfm", batch=B)
    g = torch.Generator().manual_seed(1)
    ids = torch.stack([torch.randint(0, v, (B,), generator=g) for v in vocab], 1).contiguous().to(dev)
    dense = torch.rand(B, 13, generator=g).to(dev)
    labels = (torch.rand(B, generator=g) < 0.25).float().to(dev)
    m.forward_backward(ids, dense, labels)     # real activations and gradients in every buffer the GEMMs read
    torch.cuda.synchronize()
    st = torch.cuda.current_stream().cuda_stream
    L, dims, Hp = len(m.hidden), [m.K0p] + m.Hp, m.Hp

    # (name, M, N, K, single launch, chain descriptor) -- the step's GEMMs as FusedCTR issues them
    gemms = []
    # dX1 with a plain fp32 store and no FM operands (fm_cols = 0): timed after the step's GEMMs, not part of the
    # whole forward / backward. Its gap to "dX1 (FM)" is what the FM epilogue costs.
    nofm = []
    src = m.A0
    for l in range(L):
        def fwd(l=l, src=src):
            G.gemm_nt(src, m.Wb[l], B, Hp[l], dims[l], m.H[l], mode=G.EPI_FWD, relu=True, ones_col=Hp[l] - 1, stream=st)
        gemms.append(("fwd%d" % (l + 1), B, Hp[l], dims[l], fwd,
                      lambda l=l, src=src: G.chain_nt(src, m.Wb[l], B, Hp[l], dims[l], m.H[l], mode=G.EPI_FWD,
                                                      relu=True, ones_col=Hp[l] - 1)))
        src = m.H[l]
    for l in range(L - 1, -1, -1):
        gW = m.gview("W%d" % l).view(Hp[l], dims[l])
        if l > 0:
            def dx(l=l):
                G.gemm_nt(m.dZ[l], m.WTb[l], B, Hp[l - 1], Hp[l], m.dZ[l - 1], mode=G.EPI_DX, ones_col=Hp[l - 1] - 1,
                          mask=m.H[l - 1], stream=st)
            gemms.append(("dX%d" % (l + 1), B, Hp[l - 1], Hp[l], dx,
                          lambda l=l: G.chain_nt(m.dZ[l], m.WTb[l], B, Hp[l - 1], Hp[l], m.dZ[l - 1], mode=G.EPI_DX,
                                                 ones_col=Hp[l - 1] - 1, mask=m.H[l - 1])))
        else:
            fm = dict(dlogit=m.dlogit, S=m.S, emb=m.X32, fm_cols=m.nf * m.Dp, D=m.Dp)

            def dx(fm=fm):
                G.gemm_nt(m.dZ[0], m.WTb[0], B, m.K0p, Hp[0], m.G32, mode=G.EPI_DX_FM, stream=st, **fm)
            gemms.append(("dX1 (FM)", B, m.K0p, Hp[0], dx,
                          lambda fm=fm: G.chain_nt(m.dZ[0], m.WTb[0], B, m.K0p, Hp[0], m.G32, mode=G.EPI_DX_FM, **fm)))
            nofm.append(("dX1 (no FM)", B, m.K0p, Hp[0],
                         lambda: G.gemm_nt(m.dZ[0], m.WTb[0], B, m.K0p, Hp[0], m.G32, mode=G.EPI_DX_FM, fm_cols=0, stream=st),
                         lambda: G.chain_nt(m.dZ[0], m.WTb[0], B, m.K0p, Hp[0], m.G32, mode=G.EPI_DX_FM, fm_cols=0)))
        prev = m.A0 if l == 0 else m.H[l - 1]

        def dw(l=l, prev=prev, gW=gW):
            G.gemm_tn(m.dZ[l], prev, Hp[l], dims[l], B, gW, splits=m.dw_splits, stream=st)
        gemms.append(("dW%d (split %d)" % (l + 1, m.dw_splits), Hp[l], dims[l], B, dw,
                      lambda l=l, prev=prev, gW=gW: G.chain_tn(m.dZ[l], prev, Hp[l], dims[l], B, gW, splits=m.dw_splits)))

    def timed(fn):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        G.check()
        return e0.elapsed_time(e1) * 1e3 / a.steps     # us per launch

    def run_chain(descs):
        c = G.GemmChain(descs, dev)
        us = timed(lambda: c.launch(st))
        c.check()
        c.close()
        return us

    name, power = card()
    out = []
    for nm, M, N, K, single, desc in gemms + nofm:
        row = {"gemm": nm, "M": M, "N": N, "K": K, "bn": bn, "mc": mc, "single_us": timed(single)}
        row["chain_us"] = run_chain([desc()])
        row["gflop"] = 2.0 * M * N * K / 1e9
        row["l2_MB"] = l2_bytes(M, N, K, bn, single_mc(mc, math.ceil(N / bn))) / 1e6
        row["tflops_single"] = row["gflop"] / row["single_us"] * 1e3
        out.append(row)

    fwd_single = timed(lambda: [gm[4]() for gm in gemms[:L]])
    whole = {"bn": bn, "mc": mc, "fwd_3_single_us": fwd_single, "bwd_6_single_us": timed(lambda: [gm[4]() for gm in gemms[L:]])}
    # whole chains with their dependencies, built as FusedCTR builds them
    fd = []
    for l in range(L):
        d = gemms[l][5]()
        d.dep, d.dep_kind = l - 1, (1 if l > 0 else 0)
        fd.append(d)
    whole["fwd_chain_us"] = run_chain(fd)
    bd, prod = [], -1
    for i in range(L):
        dx, dw = gemms[L + 2 * i][5](), gemms[L + 2 * i + 1][5]()
        dx.dep, dx.dep_kind = prod, (1 if prod >= 0 else 0)
        dw.dep, dw.dep_kind = prod, (2 if prod >= 0 else 0)
        bd += [dx, dw]
        prod = len(bd) - 2
    whole["bwd_chain_us"] = run_chain(bd)
    whole["bwd_chain_l2_MB"] = sum(l2_bytes(gm[1], gm[2], gm[3], 64) for gm in gemms[L:]) / 1e6
    print(json.dumps({"card": name, "power_limit": power, "rows": out, "whole": whole}), flush=True)


if a.child:
    child(a.child, int(os.environ.get("EXB_GEMM_MC", "0")))
    sys.exit(0)

ints = lambda s: [int(x) for x in s.split(",")]
combos = [(w, mc) for w in ints(a.widths) for mc in ints(a.mc)]
results = []
for _ in range(a.rounds):
    for w, mc in combos:
        env = dict(os.environ, EXB_GEMM_BN=str(w), EXB_GEMM_MC=str(mc))
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", str(w), "--batch", str(a.batch),
                            "--dim", str(a.dim), "--steps", str(a.steps), "--warmup", str(a.warmup)],
                           env=env, stdout=subprocess.PIPE, text=True)
        if p.returncode != 0:
            raise SystemExit("child for BN=%d, EXB_GEMM_MC=%d failed (exit %d)" % (w, mc, p.returncode))
        r = json.loads(p.stdout.strip().splitlines()[-1])
        print(json.dumps(r), flush=True)
        results.append(r)

r0 = results[0]
print("\n%s, power limit %s; batch %d, dim %d; us per launch over %d launches after %d\n"
      % (r0["card"], r0["power_limit"], a.batch, a.dim, a.steps, a.warmup))
f = lambda v: "%.1f" % v
print("| GEMM | M x N x K | GFLOP | BN | MC | L2 operand MB | single us | TFLOP/s | one-GEMM chain us |")
print("|---|---|---|---|---|---|---|---|---|")
for i in range(len(r0["rows"])):
    for r in results:
        x = r["rows"][i]
        print("| %s | %d x %d x %d | %.2f | %d | %d | %.0f | %s | %.0f | %s |"
              % (x["gemm"], x["M"], x["N"], x["K"], x["gflop"], x["bn"], x["mc"], x["l2_MB"], f(x["single_us"]),
                 x["tflops_single"], f(x["chain_us"])))
print("\n| BN | MC | forward: 3 single launches us | forward chain us | backward: 6 single launches us "
      "| backward chain L2 operand MB | backward chain us |")
print("|---|---|---|---|---|---|---|")
for r in results:
    w = r["whole"]
    print("| %d | %d | %s | %s | %s | %.0f | %s |"
          % (w["bn"], w["mc"], f(w["fwd_3_single_us"]), f(w["fwd_chain_us"]), f(w["bwd_6_single_us"]),
             w["bwd_chain_l2_MB"], f(w["bwd_chain_us"])))
