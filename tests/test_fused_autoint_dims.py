"""The fused AutoInt's sizes and dense map on the CPU (models/fused_dense.py: autoint_dims, dense_layout), the eager zoo's
AutoInt against its stand-alone export (models/ctr.py), and the configuration keys AutoInt adds to checkpoints."""
import pytest
import torch

from test_fused_checkpoint_layout import VOCAB, _cached, _fill_tables

CONFIGS = {
    # the defaults: 3 layers, d 8, 2 heads, residual; Dp 12 != D 9, cached features between server features
    "autoint_d9_cache": dict(model="autoint", dim=9, nd=13, hidden=(37, 21), cache=64, att=dict()),
    # one layer without residual and without dense features
    "autoint_d16_1layer_nores_nodense": dict(model="autoint", dim=16, nd=0, hidden=(17,), cache=0,
                                             att=dict(att_layers=1, att_res=False)),
    # one head with d * h = 64, D above 64 (layer 0's operand has 128 columns)
    "autoint_d70_1head": dict(model="autoint", dim=70, nd=2, hidden=(19, 7), cache=64,
                              att=dict(att_layers=2, att_embedding_size=64, att_head_num=1)),
}


def _layout(cfg):
    from openembedding_b200.models.fused_dense import dense_layout
    return dense_layout(VOCAB, cfg["nd"], cfg["dim"], cfg["model"], cfg["hidden"], _cached(cfg), **cfg["att"])


def _ctr(cfg):
    from openembedding_b200.models.ctr import CTRModel
    return CTRModel(VOCAB, num_dense=cfg["nd"], embedding_dim=cfg["dim"], model=cfg["model"], batch=64,
                    dnn_hidden=cfg["hidden"], cache_threshold=cfg["cache"], compute_dtype=torch.float32, **cfg["att"])


def _standalone(cfg):
    from openembedding_b200.models.ctr import StandaloneCTR
    return StandaloneCTR(VOCAB, num_dense=cfg["nd"], embedding_dim=cfg["dim"], model=cfg["model"], hidden=cfg["hidden"],
                         cached=_cached(cfg), **cfg["att"])


def test_autoint_dims_sizes():
    from openembedding_b200.models.fused_dense import autoint_dims
    assert autoint_dims(26, 3, 8, 2, True, 9, 3) == (16, 64, [64, 64, 64])
    assert autoint_dims(26, 3, 8, 2, False, 64, 3) == (16, 64, [64, 64, 64])
    assert autoint_dims(26, 2, 16, 2, True, 65, 3) == (32, 128, [128, 64])
    assert autoint_dims(64, 1, 64, 1, True, 8, 7) == (64, 256, [64])           # every limit at its maximum
    assert autoint_dims(1, 4, 1, 64, False, 1, 4) == (64, 192, [64] * 4)


@pytest.mark.parametrize("args,match", [((26, 0, 8, 2, True), "at least one"),
                                        ((26, -1, 8, 2, True), "at least one"),
                                        ((65, 3, 8, 2, True), "fields"),
                                        ((0, 3, 8, 2, True), "fields"),
                                        ((26, 3, 0, 2, True), "positive"),
                                        ((26, 3, 8, 0, True), "positive"),
                                        ((26, 3, 65, 1, True), "above 64"),
                                        ((26, 3, 8, 9, True), "above 64")])
def test_autoint_dims_errors(args, match):
    from openembedding_b200.models.fused_dense import autoint_dims
    with pytest.raises(ValueError, match=match):
        autoint_dims(*args)


def test_autoint_dims_matrix_count():
    from openembedding_b200.models.fused_dense import autoint_dims
    autoint_dims(26, 4, 8, 2, True, 9, dnn_layers=4)                           # 8 matrices: the optimizer's maximum
    for layers, dnn in ((5, 4), (6, 3), (8, 1)):
        with pytest.raises(ValueError, match="weight matrices"):
            autoint_dims(26, layers, 8, 2, True, 9, dnn_layers=dnn)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_autoint_layout_names_and_shapes(cpu_context, name):
    """the map's names and shapes are CTRModel's and StandaloneCTR's (plus dnn_out.bias); the attention weights sit in
    segments T{l} [Kp_l, Np] as [W_query | W_key | W_value | W_res] column blocks, w_att in the flat region"""
    from openembedding_b200.models.fused_dense import autoint_dims
    cfg = CONFIGS[name]
    lay = _layout(cfg)
    want = {n: tuple(p.shape) for n, p in _standalone(cfg).named_parameters() if not n.startswith(("emb.", "lin."))}
    assert {n: tuple(p.shape) for n, p in _ctr(cfg).named_parameters() if not n.startswith("sparse.")} == want
    assert {n: tuple(s) for n, (s, _) in lay.params.items()} == dict(want, **{"dnn_out.bias": (1,)})
    a = dict(dict(att_layers=3, att_embedding_size=8, att_head_num=2, att_res=True), **cfg["att"])
    dh, Np, Kp = autoint_dims(len(VOCAB), a["att_layers"], a["att_embedding_size"], a["att_head_num"], a["att_res"],
                              cfg["dim"], len(cfg["hidden"]))
    names = ["W_query", "W_key", "W_value"] + (["W_res"] if a["att_res"] else [])
    for l in range(a["att_layers"]):
        assert lay.shapes["T%d" % l] == (Kp[l], Np)
        for k, n in enumerate(names):
            (seg, rows, cols), = lay.params["att.layers.%d.%s" % (l, n)][1]
            assert seg == "T%d" % l and list(rows) == list(range(cfg["dim"] if l == 0 else dh))
            assert list(cols) == list(range(k * dh, (k + 1) * dh))
    assert lay.shapes["watt"] == (1, len(VOCAB) * dh)
    assert lay.segs["watt"][0] > lay.segs["wout"][0]          # the flat region starts at wout
    assert all(lay.segs["T%d" % l][0] < lay.segs["wout"][0] for l in range(a["att_layers"]))
    blocks = lay.params["dnn_out.weight"][1]
    assert [b[0] for b in blocks] == ["watt", "wout"] and list(blocks[0][2]) == list(range(len(VOCAB) * dh))


@pytest.mark.parametrize("name", list(CONFIGS))
def test_autoint_standalone_logits_equal_ctr_model(cpu_context, name):
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
    # the attention reaches the logit: zeroing its output weights moves it
    with torch.no_grad():
        mod.dnn_out.weight[:, :len(VOCAB) * mod.att.out_dim] = 0
        assert not torch.equal(mod(ids, dense), z)


def test_autoint_matches_attention_by_hand(cpu_context):
    """InteractingLayer against an explicit per-sample, per-head loop (DeepCTR's formulas, scaling=False)"""
    from openembedding_b200.models.ctr import InteractingLayer
    torch.manual_seed(0)
    lay = InteractingLayer(5, att_embedding_size=3, head_num=2, use_res=True).double()
    x = torch.randn(4, 7, 5, dtype=torch.float64)
    with torch.no_grad():
        got = lay(x)
        want = torch.empty(4, 7, 6, dtype=torch.float64)
        for b in range(4):
            q, k, v, r = (x[b] @ w for w in (lay.W_query, lay.W_key, lay.W_value, lay.W_res))
            for h in range(2):
                c = slice(3 * h, 3 * h + 3)
                s = q[:, c] @ k[:, c].t()
                p = torch.exp(s - s.max(1, keepdim=True).values)
                p = p / p.sum(1, keepdim=True)
                want[b, :, c] = p @ v[:, c]
            want[b] = torch.relu(want[b] + r)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_config_keys_of_existing_models_unchanged():
    """a configuration written before AutoInt joined (no att_* keys) still matches a model of the other families:
    their value of every new key is None"""
    from openembedding_b200.models.fused_dense import CONFIG_KEYS, FusedCTR
    new = ("att_layers", "att_embedding_size", "att_head_num", "att_res")
    assert all(k in CONFIG_KEYS for k in new)

    class _Fake:                                     # config() / config_mismatches() read these attributes only
        pass

    for model, extra in (("deepfm", {}), ("wdl", {}), ("xdeepfm", {"cin_split_half": True}), ("dcn", {})):
        m = _Fake()
        m.model, m.vocab, m.cached, m.D, m.nd, m.hidden = model, [10, 20], [], 8, 13, [64]
        m.cin_layers = [4] if model == "xdeepfm" else []
        m.cin, m.cin_split_half = model == "xdeepfm", True
        m.cross_layers = 3 if model == "dcn" else 0
        m.autoint, m.att_layers = False, 0
        m.pack_linear, m.B = True, 256
        m.ctx = type("C", (), {"world": 1})()
        m.dense_opt = {"category": "adagrad"}
        cfg = FusedCTR.config(m)
        assert all(cfg[k] is None for k in new), cfg
        old = {k: v for k, v in cfg.items() if k not in new}
        m.config = lambda m=m: FusedCTR.config(m)
        assert FusedCTR.config_mismatches(m, old) == []
        assert FusedCTR.config_mismatches(m, dict(old, att_layers=3)) != []
