"""CTR model zoo on the sharded engine: LR, Wide&Deep, DeepFM, xDeepFM, DCN-v2, AutoInt.

The reference benchmarks DeepCTR's WDL / DeepFM / xDeepFM with every
``keras.layers.Embedding`` swapped for the PS embedding
(test/benchmark/criteo_deepctr.py:60-110, 243-282): per sparse feature one embedding of
``embedding_dim`` (FM / DNN / CIN input) and one of dim 1 (the linear "wide" term);
13 dense features; DNN (400,400,400) for DeepFM/xDeepFM and (512,256,128,32) for WDL;
``task='binary'``. The same architectures are built here:

* all server-side tables of the model form ONE fused ``SparsePlan`` -- one pull launch
  and one push+update launch per step for all 2x26 tables (the reference issues one
  RPC round per table);
* tables with ``vocab < cache_threshold`` are replicated ("sparse_as_dense" cache mode of
  the reference, criteo_deepctr.py:79-81) and trained with the dense parameters;
* the dense part runs in bf16 with fp32 master weights.
"""
import math

import torch
from torch import nn
import torch.nn.functional as F

from ..context import get_context

# Criteo-Terabyte cardinalities (label-encoded, as produced by test/criteo_preprocess.cpp
# style preprocessing) capped at 20M rows per table -> 104M rows in total ("100M-row tables").
CRITEO_1TB_VOCAB_20M = [20000000, 39043, 17289, 7420, 20263, 3, 7120, 1543, 63, 20000000, 2953546, 403346, 10,
                        2208, 11938, 155, 4, 976, 14, 20000000, 20000000, 20000000, 585935, 12972, 108, 36]
# Criteo-Kaggle cardinalities (33.8M rows)
CRITEO_KAGGLE_VOCAB = [1460, 583, 10131227, 2202608, 305, 24, 12517, 633, 3, 93145, 5683, 8351593, 3194, 27,
                       14992, 5461306, 10, 5652, 2173, 4, 7046547, 18, 15, 286181, 105, 142572]


class _GroupLookup(torch.autograd.Function):
    """pull in forward; fused dispatch+combine+optimizer in backward (no fake gradient
    round trip: the cross-GPU barrier inside the kernel plays the role of the reference's
    fake-gradient allreduce, exb.py:89-97)."""

    @staticmethod
    def forward(ctx, anchor, ids, owner):
        ctx.owner = owner
        ctx.ids = ids
        return owner.group.pull(ids, train=True)    # push_update of the same ids follows in backward

    @staticmethod
    def backward(ctx, grad):
        owner = ctx.owner
        owner.group.push_update(ctx.ids, grad.contiguous())
        owner.steps += 1
        return torch.zeros_like(owner.anchor), None, None


class FusedEmbeddings(nn.Module):
    """All server-side tables of a model behind one plan.

    specs: list of dict(vocab, dim, col, initializer) -- several specs may share an id
    column (`col`), e.g. the dim-D and the dim-1 table of one sparse feature.
    """

    def __init__(self, specs, batch, optimizer, num_shards=None, ncols=None, feat_offsets=None, io_stride=None,
                 feat_offsets2=None, feat_split=None):
        super().__init__()
        ctx = get_context()
        self.ctx = ctx
        self.specs = specs
        self.metas = []
        for s in specs:
            st = ctx.create_storage(num_shards)
            vocab = s["vocab"] if s["vocab"] and s["vocab"] > 0 else 2 ** 63
            m = ctx.create_variable(st, vocab, s["dim"], "float32")
            ctx.set_initializer(m, s.get("initializer", {"category": "constant", "value": 0.0}))
            ctx.set_optimizer(m, optimizer)
            self.metas.append(m)
        if feat_offsets is not None:
            ctx.backend.ensure_allocated(self.metas)
            self.group = ctx.backend.engine.make_plan([m.handle for m in self.metas], batch, feat_offsets=feat_offsets,
                                                      io_stride=io_stride, feat_cols=[s["col"] for s in specs],
                                                      ncols=ncols, feat_offsets2=feat_offsets2, feat_split=feat_split)
            ctx.backend.engine.connect(ctx.backend.group)
        else:
            self.group = ctx.backend.make_group(self.metas, batch, feat_cols=[s["col"] for s in specs], ncols=ncols)
        self.slices = self.group.feature_slices()
        self.io_stride = self.group.io_stride
        self.anchor = nn.Parameter(torch.zeros(1, device=ctx.device))  # keeps autograd attached
        self.steps = 0

    def forward(self, ids):
        if torch.is_grad_enabled():
            return _GroupLookup.apply(self.anchor, ids, self)
        return self.group.pull(ids)


def _gemm_layers(tc):
    """(Linear, Conv1x1) layer classes: on the CUDA engine every GEMM-shaped op of the eager zoo runs on the
    hand-written wgmma kernel (ops/tc_linear.py); on CPU plain torch"""
    if tc:
        from ..ops.tc_linear import TcConv1x1, TcLinear
        return TcLinear, TcConv1x1
    return nn.Linear, lambda cin, cout: nn.Conv1d(cin, cout, 1)


class _GatherRows(torch.autograd.Function):
    """``weight[idx]`` for the small replicated ("cache") tables whose backward is an atomic ``index_add_`` instead of
    ``embedding_dense_backward``'s radix sort of all indices (8 sort passes + a segmented reduction per table group:
    ~170 us of a step at batch 4096 x 11 cached features)"""

    @staticmethod
    def forward(ctx, weight, idx):
        ctx.save_for_backward(idx)
        ctx.rows = weight.shape[0]
        return weight.index_select(0, idx.reshape(-1)).reshape(tuple(idx.shape) + (weight.shape[1],))

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        gw = torch.zeros((ctx.rows, g.shape[-1]), dtype=g.dtype, device=g.device)
        gw.index_add_(0, idx.reshape(-1), g.reshape(-1, g.shape[-1]))
        return gw, None


class CIN(nn.Module):
    """Compressed Interaction Network (xDeepFM), DeepCTR defaults: split_half, relu."""

    def __init__(self, num_fields, layer_sizes=(128, 128), split_half=True, tc=False):
        super().__init__()
        _, Conv = _gemm_layers(tc)
        self.tc = tc
        self.split_half = split_half
        self.layer_sizes = layer_sizes
        self.convs = nn.ModuleList()
        prev, total = num_fields, 0
        for i, size in enumerate(layer_sizes):
            self.convs.append(Conv(num_fields * prev, size))
            if split_half and i != len(layer_sizes) - 1:
                prev = size // 2
                total += size // 2
            else:
                prev = size
                total += size
        self.out_dim = total

    def forward(self, x):                      # x [B, F, D]
        B, Fn, D = x.shape
        if self.tc and x.is_cuda:
            # own kernels (ops/cin.py): rows = (sample, embedding column); the interaction tensor is written once as
            # the bf16 operand of the wgmma GEMM, bias + relu in its epilogue; no transposes between layers
            from ..ops.cin import cin_layer
            xr = x.transpose(1, 2).reshape(B * D, Fn).contiguous().float()
            hidden, outs = xr, []
            for i, conv in enumerate(self.convs):
                z = cin_layer(hidden, xr, conv.lin.weight, conv.lin.bias, relu=True)        # [B*D, size]
                if self.split_half and i != len(self.convs) - 1:
                    half = z.shape[1] // 2
                    hidden, direct = z[:, :half], z[:, half:]
                else:
                    hidden, direct = z, z
                outs.append(direct.reshape(B, D, -1).sum(1))
            return torch.cat(outs, dim=1)      # [B, total]
        hidden, outs = x, []
        for i, conv in enumerate(self.convs):
            z = torch.einsum("bhd,bmd->bhmd", hidden, x).reshape(B, -1, D)
            z = F.relu(conv(z))
            if self.split_half and i != len(self.convs) - 1:
                hidden, direct = torch.split(z, z.shape[1] // 2, dim=1)
            else:
                hidden, direct = z, z
            outs.append(direct)
        return torch.cat(outs, dim=1).sum(-1)  # [B, total]


class CrossNetV2(nn.Module):
    def __init__(self, dim, layers=3, tc=False):
        super().__init__()
        Linear, _ = _gemm_layers(tc)
        self.w = nn.ModuleList([Linear(dim, dim) for _ in range(layers)])

    def forward(self, x0):
        x = x0
        for lin in self.w:
            x = x0 * lin(x) + x
        return x


class InteractingLayer(nn.Module):
    """AutoInt's multi-head self-attention over the fields (DeepCTR ``InteractingLayer``, ``scaling=False``) in fp32
    torch: x [B, nf, in_dim] -> relu(concat_heads(softmax(Q K^T) V) + x W_res) [B, nf, d * heads], with
    Q = x W_query, K = x W_key, V = x W_value; head h owns the columns h*d .. h*d + d - 1. Weights [in_dim, d * heads],
    no bias, Keras TruncatedNormal(stddev 0.05) initial values."""

    def __init__(self, in_dim, att_embedding_size=8, head_num=2, use_res=True):
        super().__init__()
        self.d, self.heads, self.use_res = att_embedding_size, head_num, use_res
        names = ("W_query", "W_key", "W_value") + (("W_res",) if use_res else ())
        for n in names:
            w = nn.Parameter(torch.empty(in_dim, att_embedding_size * head_num))
            nn.init.trunc_normal_(w, std=0.05, a=-0.1, b=0.1)
            setattr(self, n, w)

    @staticmethod
    def attend(q, k, v, r, heads):
        """relu(concat_heads(softmax(q_h k_h^T) v_h) + r) from the projections q, k, v [B, nf, d * heads] and r (the
        residual projection, or None)"""
        B, nf, dh = q.shape
        split = lambda t: t.view(B, nf, heads, dh // heads).transpose(1, 2)       # [B, heads, nf, d]
        p = torch.softmax(split(q) @ split(k).transpose(-1, -2), dim=-1)
        o = (p @ split(v)).transpose(1, 2).reshape(B, nf, dh)
        return F.relu(o + r if r is not None else o)

    def forward(self, x):
        r = x @ self.W_res if self.use_res else None
        return self.attend(x @ self.W_query, x @ self.W_key, x @ self.W_value, r, self.heads)


class AutoIntNet(nn.Module):
    """``layers`` stacked ``InteractingLayer``s: the first takes the embedding dim, the others d * heads"""

    def __init__(self, embedding_dim, layers=3, att_embedding_size=8, head_num=2, use_res=True):
        super().__init__()
        dims = [embedding_dim] + [att_embedding_size * head_num] * layers
        self.layers = nn.ModuleList([InteractingLayer(dims[l], att_embedding_size, head_num, use_res)
                                     for l in range(layers)])
        self.out_dim = att_embedding_size * head_num

    def forward(self, x):
        for layer in self.layers:
            x = layer(x)
        return x


AUTOINT_DEFAULTS = dict(att_layers=3, att_embedding_size=8, att_head_num=2, att_res=True)


class _CTRHead(nn.Module):
    """The dense part of the zoo's CTR models, shared by ``CTRModel`` and ``StandaloneCTR``: the layers after the
    row lookup, and the logit from the looked-up rows."""

    def _build_dense(self, num_dense, dnn_hidden, tc, cin_layers, cross_layers, cin_split_half=True, autoint=None):
        """dense_linear, bias and (models with embeddings) dnn, dnn_out, cin / cin_out, cross, att (``autoint``:
        ``AUTOINT_DEFAULTS``' keys)"""
        nf, embedding_dim = self.nf, self.D
        dnn_in = nf * embedding_dim + num_dense
        self.tc = tc
        Linear, _ = _gemm_layers(tc)
        self.dense_linear = nn.Linear(num_dense, 1, bias=False) if num_dense else None
        self.bias = nn.Parameter(torch.zeros(1))
        layers, prev = [], dnn_in
        if self.has_emb:
            for h in dnn_hidden:
                layers += [Linear(prev, h), nn.ReLU()]
                prev = h
            self.dnn = nn.Sequential(*layers)
            self.dnn_out = nn.Linear(prev, 1, bias=False)
        if self.model_name == "xdeepfm":
            self.cin = CIN(nf, cin_layers, split_half=cin_split_half, tc=tc)
            self.cin_out = nn.Linear(self.cin.out_dim, 1, bias=False)
        if self.model_name == "dcn":
            self.cross = CrossNetV2(dnn_in, cross_layers, tc=tc)
            self.dnn_out = nn.Linear(prev + dnn_in, 1, bias=False)
        if self.model_name == "autoint":        # DeepCTR's concat order: flatten(attention output), then the DNN
            a = dict(AUTOINT_DEFAULTS, **(autoint or {}))
            self.att = AutoIntNet(embedding_dim, a["att_layers"], a["att_embedding_size"], a["att_head_num"],
                                  a["att_res"])
            self.dnn_out = nn.Linear(nf * self.att.out_dim + prev, 1, bias=False)

    def _cached_rows(self, ids, embs, lins):
        """append the rows of the replicated ("cache") tables to the embedding / linear parts"""
        if self.cached:
            cid = ids[:, self.cache_cols] + self.cache_offsets            # [B, nc]
            if self.has_emb:
                embs.append(_GatherRows.apply(self.cache_emb, cid))
            lins.append(_GatherRows.apply(self.cache_lin, cid).squeeze(-1))

    def _logit(self, embs, lins, dense):
        """logits [B] from the embedding parts ([B, n, D] each; server features, then cached ones), the linear
        parts ([B, n] each) and the dense input"""
        linear = torch.cat(lins, dim=1).sum(dim=1)
        if self.dense_linear is not None:
            linear = linear + self.dense_linear(dense).squeeze(-1)
        logit = linear + self.bias
        if not self.has_emb:
            return logit
        B = dense.shape[0]
        emb = torch.cat(embs, dim=1) if len(embs) > 1 else embs[0]        # [B, nf, D] fp32
        with torch.autocast(device_type=emb.device.type, dtype=self.compute_dtype,
                            enabled=self.compute_dtype != torch.float32 and not self.tc):
            x = torch.cat([emb.reshape(B, -1), dense], dim=1)
            if self.model_name == "dcn":
                h = torch.cat([self.cross(x), self.dnn(x)], dim=1)
                logit = logit + self.dnn_out(h).squeeze(-1).float()
            elif self.model_name == "autoint":
                with torch.autocast(device_type=emb.device.type, enabled=False):      # the attention runs in fp32
                    att = self.att(emb).reshape(B, -1)
                h = torch.cat([att, self.dnn(x)], dim=1)
                logit = logit + self.dnn_out(h).squeeze(-1).float()
            else:
                logit = logit + self.dnn_out(self.dnn(x)).squeeze(-1).float()
            if self.model_name == "xdeepfm":
                logit = logit + self.cin_out(self.cin(emb)).squeeze(-1).float()
        if self.model_name == "deepfm":
            s = emb.sum(dim=1)
            logit = logit + 0.5 * (s * s - (emb * emb).sum(dim=1)).sum(dim=1)
        return logit


def _default_hidden(model):
    """DeepCTR's default DNN of each model"""
    return {"wdl": (512, 256, 128, 32), "autoint": (256, 128, 64)}.get(model, (400, 400, 400))


class CTRModel(_CTRHead):
    """model in {"lr", "wdl", "deepfm", "xdeepfm", "dcn", "autoint"}"""

    def __init__(self, vocab_sizes, num_dense=13, embedding_dim=9, model="deepfm", batch=4096,
                 sparse_optimizer=None, dnn_hidden=None, cache_threshold=0, num_shards=None,
                 compute_dtype=torch.bfloat16, cin_layers=(128, 128), cross_layers=3, att_layers=3, att_embedding_size=8,
                 att_head_num=2, att_res=True):
        super().__init__()
        ctx = get_context()
        self.model_name = model.lower()
        self.num_dense, self.D = num_dense, embedding_dim
        self.vocab_sizes = list(vocab_sizes)
        self.compute_dtype = compute_dtype
        nf = len(vocab_sizes)
        self.nf = nf
        if dnn_hidden is None:
            dnn_hidden = _default_hidden(self.model_name)
        if sparse_optimizer is None:
            sparse_optimizer = {"category": "adagrad"}   # tf.keras.optimizers.Adagrad() defaults
        zero = {"category": "constant", "value": 0.0}    # benchmark uses zeros initializer (criteo_deepctr.py:82)
        self.has_emb = self.model_name != "lr"
        self.cached = [f for f, v in enumerate(vocab_sizes) if 0 < v < cache_threshold]
        self.server = [f for f in range(nf) if f not in self.cached]
        specs = []
        if self.has_emb:
            specs += [{"vocab": vocab_sizes[f], "dim": embedding_dim, "col": f, "initializer": zero}
                      for f in self.server]
        specs += [{"vocab": vocab_sizes[f], "dim": 1, "col": f, "initializer": zero} for f in self.server]
        self.sparse = FusedEmbeddings(specs, batch, sparse_optimizer, num_shards=num_shards, ncols=nf) if specs else None
        ns = len(self.server)
        if self.sparse is not None:
            sl = self.sparse.slices
            self._emb_slices = sl[:ns] if self.has_emb else []
            self._lin_slices = sl[ns:] if self.has_emb else sl
            if self.has_emb:
                self._emb_stride = (sl[1].start - sl[0].start) if ns > 1 else (self._lin_slices[0].start - sl[0].start)
        # replicated ("cache") small tables, trained with the dense parameters
        if self.cached:
            off, offs = 0, []
            for f in self.cached:
                offs.append(off)
                off += vocab_sizes[f]
            self.register_buffer("cache_offsets", torch.tensor(offs, dtype=torch.int64, device=ctx.device))
            self.register_buffer("cache_cols", torch.tensor(self.cached, dtype=torch.int64, device=ctx.device))
            self.cache_emb = nn.Parameter(torch.zeros(off, embedding_dim, device=ctx.device)) if self.has_emb else None
            self.cache_lin = nn.Parameter(torch.zeros(off, 1, device=ctx.device))
        # GEMM-shaped layers on the hand-written wgmma kernel (bf16 operands) when the model computes in bf16 on CUDA
        tc = ctx.device.type == "cuda" and compute_dtype == torch.bfloat16
        self._build_dense(num_dense, dnn_hidden, tc, cin_layers, cross_layers,
                          autoint=dict(att_layers=att_layers, att_embedding_size=att_embedding_size,
                                       att_head_num=att_head_num, att_res=att_res))
        self.to(ctx.device)

    def dense_parameters(self):
        skip = {id(self.sparse.anchor)} if self.sparse is not None else set()
        return [p for p in self.parameters() if id(p) not in skip]

    def forward(self, ids, dense):
        """ids [B, 26] int64, dense [B, 13] fp32 -> logits [B] (fp32)"""
        B = ids.shape[0]
        embs, lins = [], []
        if self.sparse is not None:
            out = self.sparse(ids)                                        # [B, io_stride] fp32
            if self.has_emb:
                ns = len(self.server)
                s0 = self._emb_slices[0].start
                es = self._emb_stride
                embs.append(out[:, s0:s0 + ns * es].reshape(B, ns, es)[:, :, :self.D])
            l0 = self._lin_slices[0].start
            lins.append(out[:, l0:l0 + len(self.server)])
        self._cached_rows(ids, embs, lins)
        return self._logit(embs, lins, dense)


class StandaloneCTR(_CTRHead):
    """A trained Wide&Deep / DeepFM / xDeepFM / DCN-v2 / AutoInt as a plain fp32 module that needs no engine and no GPU (the
    export of ``FusedCTR.save_as_original_model``): ``emb[j]`` (dim D) and ``lin[j]`` (dim 1) are the
    ``nn.Embedding`` tables of the j-th server feature, ``cache_emb`` / ``cache_lin`` the replicated tables of the
    ``cached`` features, and the dense layers carry ``CTRModel``'s names. ``forward(ids [B, nf], dense [B, nd])``
    returns fp32 logits [B]."""

    def __init__(self, vocab_sizes, num_dense=13, embedding_dim=9, model="deepfm", hidden=None, cached=(),
                 cin_layers=(128, 128), cin_split_half=True, cross_layers=3, att_layers=3, att_embedding_size=8,
                 att_head_num=2, att_res=True):
        super().__init__()
        self.model_name = model.lower()
        if self.model_name not in ("wdl", "deepfm", "xdeepfm", "dcn", "autoint"):
            raise ValueError("StandaloneCTR: wdl, deepfm, xdeepfm, dcn or autoint")
        self.num_dense, self.D = num_dense, embedding_dim
        self.vocab_sizes = list(vocab_sizes)
        self.nf = nf = len(self.vocab_sizes)
        self.compute_dtype, self.has_emb = torch.float32, True
        if hidden is None:
            hidden = _default_hidden(self.model_name)
        self.cached = list(cached)
        self.server = [f for f in range(nf) if f not in self.cached]
        self.emb = nn.ModuleList([nn.Embedding(self.vocab_sizes[f], embedding_dim) for f in self.server])
        self.lin = nn.ModuleList([nn.Embedding(self.vocab_sizes[f], 1) for f in self.server])
        if self.cached:
            offs = [sum(self.vocab_sizes[g] for g in self.cached[:i]) for i in range(len(self.cached))]
            rows = sum(self.vocab_sizes[f] for f in self.cached)
            self.register_buffer("cache_offsets", torch.tensor(offs, dtype=torch.int64))
            self.register_buffer("cache_cols", torch.tensor(self.cached, dtype=torch.int64))
            self.cache_emb = nn.Parameter(torch.zeros(rows, embedding_dim))
            self.cache_lin = nn.Parameter(torch.zeros(rows, 1))
        self._build_dense(num_dense, hidden, False, cin_layers, cross_layers, cin_split_half,
                          autoint=dict(att_layers=att_layers, att_embedding_size=att_embedding_size,
                                       att_head_num=att_head_num, att_res=att_res))

    def forward(self, ids, dense):
        embs, lins = [], []
        if self.server:
            embs.append(torch.stack([t(ids[:, f]) for t, f in zip(self.emb, self.server)], dim=1))
            lins.append(torch.cat([t(ids[:, f]) for t, f in zip(self.lin, self.server)], dim=1))
        self._cached_rows(ids, embs, lins)
        return self._logit(embs, lins, dense)


class CriteoLR(nn.Module):
    """examples/criteo_lr_subclass.py: ONE hashed dim-1 table shared by all 26 sparse
    columns (ids pre-hashed by column), dense features concatenated, sigmoid(Dense(1))."""

    def __init__(self, num_sparse=26, num_dense=13, num_shards=16, input_dim=-1):
        super().__init__()
        from ..api import Embedding
        self.embeddings = Embedding(input_dim=input_dim, output_dim=1, embeddings_initializer="zeros",
                                    num_shards=num_shards)
        self.out = nn.Linear(num_sparse + num_dense, 1)
        self.out.to(get_context().device)

    def forward(self, sparse_ids, dense):
        e = self.embeddings(sparse_ids).squeeze(-1)          # [B, 26]
        return self.out(torch.cat([e, dense.to(e.device)], dim=1)).squeeze(-1)
