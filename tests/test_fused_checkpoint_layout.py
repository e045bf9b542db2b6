"""The layout map of the fused models' dense buffer (models/fused_dense.py: dense_layout) and the stand-alone export
module (models/ctr.py: StandaloneCTR), on the CPU.

The map is checked on its own (gather + scatter round trip, blocks that do not overlap, every block inside its
segment) and against the eager zoo: the logical names and shapes are those of ``CTRModel``'s dense parameters, plus
the fused-only ``dnn_out.bias``. ``StandaloneCTR`` shares ``CTRModel``'s math after the row lookup, so given the same
parameters and table rows it returns the same fp32 logits bit for bit. The table layout (``pack_linear``) does not
enter the dense map; the GPU tests cover it."""
import numpy as np
import pytest
import torch

VOCAB = [1000, 50, 2000, 7, 3000, 30, 500, 20]       # features 1, 3, 5, 7 are cached below threshold 64

CONFIGS = {
    # Dp 12 != D 9, cached features between server features, odd hidden sizes
    "deepfm_d9_cache_odd": dict(model="deepfm", dim=9, nd=13, hidden=(37, 21), cache=64),
    # no dense features, no cached feature
    "wdl_d16_nodense": dict(model="wdl", dim=16, nd=0, hidden=(33, 17, 5), cache=0),
    "deepfm_d8_nodense_cache": dict(model="deepfm", dim=8, nd=0, hidden=(63,), cache=64),
    "xdeepfm_d5_cache": dict(model="xdeepfm", dim=5, nd=13, hidden=(19, 7), cache=64, cin_layers=(6, 5)),
    "xdeepfm_d6_nosplit": dict(model="xdeepfm", dim=6, nd=2, hidden=(11,), cache=64, cin_layers=(3, 5),
                               cin_split_half=False),
    "dcn_d6_cache": dict(model="dcn", dim=6, nd=3, hidden=(19, 9), cache=64, cross_layers=2),
    "dcn_d7_nodense": dict(model="dcn", dim=7, nd=0, hidden=(13,), cache=0, cross_layers=1),
}


def _cached(cfg):
    return [f for f, v in enumerate(VOCAB) if 0 < v < cfg["cache"]]


def _layout(cfg):
    from openembedding_b200.models.fused_dense import dense_layout
    return dense_layout(VOCAB, cfg["nd"], cfg["dim"], cfg["model"], cfg["hidden"], _cached(cfg),
                        cfg.get("cin_layers", (128, 128)), cfg.get("cin_split_half", True), cfg.get("cross_layers", 3))


def _ctr(cfg):
    from openembedding_b200.models.ctr import CTRModel
    return CTRModel(VOCAB, num_dense=cfg["nd"], embedding_dim=cfg["dim"], model=cfg["model"], batch=64,
                    dnn_hidden=cfg["hidden"], cache_threshold=cfg["cache"], compute_dtype=torch.float32,
                    cin_layers=cfg.get("cin_layers", (128, 128)), cross_layers=cfg.get("cross_layers", 3))


def _standalone(cfg):
    from openembedding_b200.models.ctr import StandaloneCTR
    return StandaloneCTR(VOCAB, num_dense=cfg["nd"], embedding_dim=cfg["dim"], model=cfg["model"], hidden=cfg["hidden"],
                         cached=_cached(cfg), cin_layers=cfg.get("cin_layers", (128, 128)),
                         cin_split_half=cfg.get("cin_split_half", True), cross_layers=cfg.get("cross_layers", 3))


def _dense_shapes(module):
    """names and shapes of a zoo module's dense parameters (not its tables)"""
    return {n: tuple(p.shape) for n, p in module.named_parameters() if not n.startswith(("sparse.", "emb.", "lin."))}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_layout_round_trip_and_disjoint_blocks(name):
    lay = _layout(CONFIGS[name])
    g = torch.Generator().manual_seed(1)
    flat = torch.randn(lay.n_theta, generator=g)
    sd = lay.gather(flat)
    back = torch.zeros(lay.n_theta)
    lay.scatter(back, sd)
    mapped = torch.zeros(lay.n_theta, dtype=torch.bool)
    for pname, (shape, blocks) in lay.params.items():
        idx = lay.index(pname)
        assert tuple(idx.shape) == tuple(shape) == tuple(sd[pname].shape), pname
        assert not bool(mapped[idx].any()), "%s overlaps another parameter" % pname
        mapped[idx] = True
        for seg, rows, cols in blocks:            # every block lies inside its segment's [R, C] matrix
            R, C = lay.shapes[seg]
            off, n = lay.segs[seg]
            assert R * C == n and 0 <= min(rows) and max(rows) < R and 0 <= min(cols) and max(cols) < C, (pname, seg)
    assert torch.equal(back[mapped], flat[mapped])        # every mapped slot reproduced
    assert not bool(back[~mapped].any())                  # nothing else written
    # segments do not overlap and stay inside the buffer
    spans = sorted(lay.segs.values())
    for (o0, n0), (o1, _) in zip(spans, spans[1:]):
        assert o0 + n0 <= o1
    assert spans[-1][0] + spans[-1][1] <= lay.n_theta


@pytest.mark.parametrize("name", list(CONFIGS))
def test_layout_names_and_shapes_are_the_zoo_models(cpu_context, name):
    cfg = CONFIGS[name]
    want = _dense_shapes(_standalone(cfg))
    if cfg.get("cin_split_half", True):               # CTRModel's CIN always splits its layers in half
        assert _dense_shapes(_ctr(cfg)) == want
    got = {n: tuple(s) for n, (s, _) in _layout(cfg).params.items()}
    assert got == dict(want, **{"dnn_out.bias": (1,)})


def _fill_tables(ctx, model, g):
    """random rows in every table of a CPU CTRModel"""
    for meta in model.sparse.metas:
        n = meta.vocab
        w = (torch.randn(n, meta.dim, generator=g) * 0.5).numpy()
        ctx.backend.load_rows(meta, np.arange(n, dtype=np.uint64), w, np.empty((n, 0), dtype=np.float32))


@pytest.mark.parametrize("name", list(n for n in CONFIGS if CONFIGS[n].get("cin_split_half", True)))
def test_standalone_logits_equal_ctr_model(cpu_context, name):
    from openembedding_b200.context import get_context
    cfg = CONFIGS[name]
    ctx = get_context()
    torch.manual_seed(3)
    ref = _ctr(cfg)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n, p in ref.named_parameters():
            if not n.startswith("sparse."):
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
    _fill_tables(ctx, ref, g)
    mod = _standalone(cfg)
    params = {n: p for n, p in ref.state_dict().items() if not n.startswith("sparse.")}
    missing, unexpected = mod.load_state_dict(params, strict=False)
    assert not unexpected and all(k.startswith(("emb.", "lin.")) for k in missing)
    ns = len(ref.server)
    with torch.no_grad():
        for j, f in enumerate(ref.server):
            ids = torch.arange(VOCAB[f])
            mod.emb[j].weight.copy_(ctx.backend.pull(ref.sparse.metas[j], ids))
            mod.lin[j].weight.copy_(ctx.backend.pull(ref.sparse.metas[ns + j], ids))
    B = 96
    ids = torch.stack([torch.randint(0, v, (B,), generator=g) for v in VOCAB], 1).contiguous()
    dense = torch.rand(B, cfg["nd"], generator=g)
    with torch.no_grad():
        z_ref = ref(ids, dense)
        z = mod(ids, dense)
    assert z.dtype == torch.float32 and z.shape == (B,)
    assert torch.equal(z.view(torch.int32), z_ref.view(torch.int32)), float((z - z_ref).abs().max())
