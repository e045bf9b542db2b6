"""The fp32 sparse engine (sparse_kernels.cuh, sparse_v2.cuh, bulk_rows.cuh) against the NumPy reference of
tests/sparse_reference.py, on every kernel path and row shape the code can take.

Exact wherever exactness is possible: with `default`, `sgd` and `test`, power-of-two learning rates and momenta and
dyadic gradients, every pulled value, weight, state word and counter must equal the float32 replica bit for bit
(see sparse_reference.py for why no rounding or atomic order can change them). Adam / Adamax beta powers are exact
too. The other optimizers (sqrt.approx / __fdividef on the device) are compared with the float64 Keras form within
a per-element bound derived from the float64 trajectory, and the bound is shown to be tight enough to see one
lookup's gradient.

Kernel paths (environment set before the plan is created):
  v1        EXB_SPARSE_V2=0: exb_pull_kernel + exb_push_update_kernel
  v2        exb_pull_plan_kernel + exb_push2_kernel
  v2next    v2 with the next batch planned during the step (prepare(next=True)): the pull is exb_pull_kernel
  pull2     v2 with EXB_PULL2=1 at world > 1: exb_pull2_kernel (unique remote rows, rows_to)
  stateless pull(train=False), then push_update (the push plans the batch)
each with EXB_BULK=1 (cp.async row movers, single-pass fast pull, apply_rows_bulk_k) and EXB_BULK=0 (register pull
and apply_rows). Row geometry selects the rest: fast pull pull_rows_fast_t<LPR> for wstride <= 128 (LPR 1..32 for
dims 4, 5-8, 9-16, 17-32, 33-64, 65-128), pull_rows_bulk up to wstride 2048, the register pull_rows<LPR> and the
whole-warp rows_to beyond; the bulk apply while apply_need <= EXB_APPLY_WARP_BUF, apply_rows (with its column loop
for dim > 128) beyond; one lane per row for dim < 4.
"""
import ctypes

import numpy as np
import pytest
import torch

from sparse_reference import BOUND_C, TableRef, dyadic, hash64, valid_ids
from test_optimizers import CONFIGS

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

INIT = 0.25                      # constant initializer: exact tests seed their rows through scatter_rows
APPLY_WARP_BUF = 10240           # bulk_rows.cuh EXB_APPLY_WARP_BUF
EXACT = {
    "default": {"category": "default", "learning_rate": 0.125},
    "sgd": {"category": "sgd", "learning_rate": 0.25, "momentum": 0.5, "nesterov": True},
    "test": {"category": "test", "learning_rate": 0.5, "flip": 3.0, "init": 0.75},
}
DIMS = [1, 2, 3, 4, 5, 8, 12, 16, 17, 31, 32, 33, 64, 65, 127, 128, 129, 132, 200, 2048, 2049, 2052]
SPLIT_DIMS = [3, 4, 8, 9, 64, 127, 128, 129, 200]           # [D | 1] rows: table dim D + 1
PATHS = {
    "v1": {"EXB_SPARSE_V2": "0"},
    "v2": {"EXB_SPARSE_V2": "1"},
    "v2next": {"EXB_SPARSE_V2": "1"},
    "pull2": {"EXB_SPARSE_V2": "1", "EXB_PULL2": "1"},
    "stateless": {"EXB_SPARSE_V2": "1"},
}
STREAMS = ["unique", "uniform", "zipf", "same", "invalid"]


def _slots(cfg):
    from openembedding_b200.config import OPTIMIZER_SLOTS
    return OPTIMIZER_SLOTS(cfg)


def apply_need(dim, cfg):
    """bytes of one row in the apply phase (sparse_kernels.cuh apply_need), from engine.cu layout_table"""
    nslots, nsc = _slots(cfg)
    if dim < 4:
        return None                                  # never the bulk apply
    ws = (dim + 3) // 4 * 4
    ss = max(4, (nslots * ws + nsc + 3) // 4 * 4)
    return (2 * ws + ss) * 4


def boundary_dims(cfg):
    """the dims on either side of the optimizer's bulk-apply limit apply_need <= EXB_APPLY_WARP_BUF"""
    d = 4
    while apply_need(d + 1, cfg) <= APPLY_WARP_BUF:
        d += 1
    return [d, d + 1]


def _set_env(monkeypatch, path, bulk):
    for k in ("EXB_SPARSE_V2", "EXB_PULL2", "EXB_BULK"):
        monkeypatch.delenv(k, raising=False)
    for k, v in PATHS[path].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("EXB_BULK", "1" if bulk else "0")


class Rig:
    """W virtual ranks (engines on one GPU wired with connect_local), one plan each, and the reference."""

    def __init__(self, world, tables, feats, batch, path, exact=True, max_ctas=6, layout=None, seed=0):
        from openembedding_b200.ops.sparse_engine import CudaEngine
        self.world, self.tables, self.feats, self.B, self.path = world, tables, feats, batch, path
        self.rng = np.random.default_rng(seed)
        self.dev = torch.device("cuda", 0)
        self.engines = [CudaEngine(0, r, world, max_ctas=max_ctas) for r in range(world)]
        for e in self.engines:
            for vid, t in enumerate(tables):
                i = e.add_table(t["dim"], t.get("vocab", 0), t["is_hash"], capacity=t.get("capacity", 4096),
                                shard_num=t.get("shard_num", -1), shard_base=t.get("shard_base", 0))
                e.set_initializer(i, {"category": "constant", "value": INIT}, vid)
                e.set_optimizer(i, t["cfg"])
                e.alloc(i)
        layout = layout or {}
        self.plans = [e.make_plan(feats, batch, **layout) for e in self.engines]
        if world > 1:
            CudaEngine.connect_local(self.engines)
        self.streams = [torch.cuda.Stream(device=self.dev) for _ in range(world)]
        self.refs = [TableRef(t["dim"], t.get("vocab", 0), t["is_hash"], t["cfg"], INIT, exact) for t in tables]
        self.info = [self.engines[0].table_info(i) for i in range(len(tables))]
        p = self.plans[0]
        self.io, self.ncols = p.io_stride, p.ncols
        self.hist = []                               # per step: [(table, ids, grads)] of every lookup
        self.expect_unique = [0] * world
        self.steps = 0
        self.seen = [set() for _ in tables]
        self.seeded = [(np.zeros(0, np.int64), np.zeros((0, t["dim"]), np.float32)) for t in tables]

    # ---- owners (exb_common.cuh owner_of)
    def owner(self, t, ids):
        T = self.tables[t]
        sn = T.get("shard_num", -1)
        sn = self.world if sn <= 0 or sn > self.world else sn
        base = T.get("shard_base", 0) % self.world
        return (base + np.asarray(ids, dtype=np.uint64) % np.uint64(sn)).astype(np.int64) % self.world

    # ---- seeding
    def seed_rows(self, t, ids):
        T = self.tables[t]
        ids = np.unique(np.asarray(ids, dtype=np.int64))
        w = self.rng.standard_normal((ids.size, T["dim"])).astype(np.float32)
        for e in self.engines:
            e.scatter_rows(t, torch.from_numpy(ids), torch.from_numpy(w))
        self.refs[t].seed(ids, w)
        self.seeded[t] = (ids, w)
        self.seen[t].update(ids.tolist())

    # ---- batches
    def ids_for(self, t, kind, n):
        T, rng = self.tables[t], self.rng
        vocab = T.get("vocab", 0)
        if kind == "unique":
            x = rng.choice(min(vocab, 4000) if not T["is_hash"] else 100000, size=n, replace=False)
        elif kind == "uniform":
            x = rng.integers(0, 40, size=n)
        elif kind == "zipf":
            x = rng.integers(0, 300, size=n)
            x[rng.random(n) < 0.6] = 7                     # one id in more than half of the batch
        elif kind == "same":
            x = np.full(n, 3)
        else:
            x = rng.integers(0, 60, size=n)
        x = x.astype(np.int64)
        if T["is_hash"]:
            x = x * 1000003 + 11
        if kind == "invalid":
            bad = rng.random(n) < 0.3
            inv = (rng.integers(0, 1 << 40, size=n) | (1 << 62)) * -1 if T["is_hash"] else \
                vocab + rng.integers(0, 1000, size=n)
            inv[rng.random(n) < 0.3] = -1
            x = np.where(bad, inv, x)
        return x

    def make_batch(self, step, kinds=None):
        out = []
        for r in range(self.world):
            ids = self.rng.integers(-50, 50, size=(self.B, self.ncols)).astype(np.int64)   # unused columns: junk
            for f, t in enumerate(self.feats):
                kind = kinds[f] if kinds else STREAMS[(f + step + r) % len(STREAMS)]
                ids[:, self.plans[0].feat_cols[f]] = self.ids_for(t, kind, self.B)
            out.append(ids)
        return out

    def feature_cols(self, f):
        """(columns of the activation row the feature's table columns map to, pad columns)"""
        p, t = self.plans[0], self.feats[f]
        d, ws, off = self.tables[t]["dim"], int(self.info[t]["wstride"]), p.feat_offsets[f]
        sp = p.feat_split[f] if p.feat_split is not None else d
        if sp < d:
            o2 = p.feat_offsets2[f]
            return list(range(off, off + sp)) + list(range(o2, o2 + d - sp)), []
        return list(range(off, off + d)), list(range(off + d, off + ws))

    def make_grads(self, step):
        fill = np.float32(np.nan) if step % 2 == 0 else np.float32(1e30)     # pad / gap columns: must not matter
        out = []
        for r in range(self.world):
            g = np.full((self.B, self.io), fill, dtype=np.float32)
            for f in range(len(self.feats)):
                cols, _ = self.feature_cols(f)
                g[:, cols] = dyadic(self.rng, (self.B, len(cols)))
            out.append(g)
        return out

    # ---- checks
    def expected_pull(self, ids):
        exp = np.full((ids.shape[0], self.io), np.nan, dtype=np.float32)
        for f, t in enumerate(self.feats):
            cols, pad = self.feature_cols(f)
            exp[:, cols] = self.refs[t].pull(ids[:, self.plans[0].feat_cols[f]])
            exp[:, pad] = 0.0
        return exp

    def pull_all(self, ids_t, train, nxt=None):
        outs = []
        torch.cuda.synchronize()
        for r in range(self.world):
            with torch.cuda.stream(self.streams[r]):
                out = torch.full((self.B, self.io), float("nan"), device=self.dev)
                outs.append(self.plans[r].pull(ids_t[r], out=out, train=train))
                if nxt is not None:
                    self.plans[r].prepare(nxt[r], next=True)
        torch.cuda.synchronize()
        return outs

    def check_pull(self, ids, outs):
        for r in range(self.world):
            np.testing.assert_array_equal(outs[r].cpu().numpy(), self.expected_pull(ids[r]),
                                          err_msg="pull rank %d (%s)" % (r, self.path))

    def step(self, ids, grads, ids_t, check_pull=True, nxt_t=None):
        train = self.path != "stateless"
        outs = self.pull_all(ids_t, train, nxt_t if self.path == "v2next" else None)
        if check_pull:
            self.check_pull(ids, outs)
        gt = [torch.from_numpy(g).to(self.dev) for g in grads]
        torch.cuda.synchronize()
        for r in range(self.world):
            with torch.cuda.stream(self.streams[r]):
                self.plans[r].push_update(ids_t[r], gt[r])
        torch.cuda.synchronize()
        for e in self.engines:
            e.check()
        rec = []
        for t in range(len(self.tables)):
            fs = [f for f, ft in enumerate(self.feats) if ft == t]
            if not fs:
                continue
            li, lg = [], []
            for r in range(self.world):
                for f in fs:
                    cols, _ = self.feature_cols(f)
                    li.append(ids[r][:, self.plans[0].feat_cols[f]])
                    lg.append(grads[r][:, cols])
            li, lg = np.concatenate(li), np.concatenate(lg)
            rec.append((t, li, lg))
            u = self.refs[t].step(li, lg)
            self.seen[t].update(u.tolist())
            own = self.owner(t, u)
            for r in range(self.world):
                self.expect_unique[r] += int((own == r).sum())
        self.hist.append(rec)
        self.steps += 1

    def run(self, steps, check_pull=True):
        batches = [self.make_batch(s) for s in range(steps + 1)]
        ids_t = [[torch.from_numpy(b).to(self.dev) for b in bs] for bs in batches]
        for s in range(steps):
            self.step(batches[s], self.make_grads(s), ids_t[s], check_pull, ids_t[s + 1])
        if check_pull:            # later pulls: weights and zero pad columns after the last update (stateless read)
            outs = []
            for r in range(self.world):
                out = torch.full((self.B, self.io), float("nan"), device=self.dev)
                outs.append(self.plans[r].pull(ids_t[steps][r], out=out))
            torch.cuda.synchronize()
            self.check_pull(batches[steps], outs)

    def probe_ids(self, t):
        T = self.tables[t]
        if not T["is_hash"]:
            return np.arange(T["vocab"], dtype=np.int64)          # every row: untouched rows must be unchanged
        never = np.arange(5, dtype=np.int64) * 1000003 + 5     # never pushed: initial values
        return np.unique(np.concatenate([np.array(sorted(self.seen[t]), dtype=np.int64), never]))

    def gathered(self, t):
        """(ids, weights, state) of table t as the owning ranks hold them"""
        ids = self.probe_ids(t)
        own = self.owner(t, ids)
        w = np.zeros((ids.size, self.tables[t]["dim"]), np.float32)
        s = np.zeros((ids.size, self.refs[t].sd), np.float32)
        for r, e in enumerate(self.engines):
            m = own == r
            if m.any():
                gw, gs = e.gather_rows(t, torch.from_numpy(ids[m]))
                w[m] = gw.cpu().numpy()
                if gs is not None and gs.numel():
                    s[m] = gs.cpu().numpy()
        return ids, w, s

    def check_tables_exact(self):
        for t in range(len(self.tables)):
            ids, w, s = self.gathered(t)
            ww, ws = self.refs[t].get(ids)
            np.testing.assert_array_equal(w, ww, err_msg="weights of table %d (%s)" % (t, self.path))
            np.testing.assert_array_equal(s, ws, err_msg="state of table %d (%s)" % (t, self.path))
            if self.tables[t]["is_hash"]:
                mat = np.array(sorted(self.refs[t].materialized()), dtype=np.int64)
                own = self.owner(t, mat)
                for r, e in enumerate(self.engines):
                    assert e.table_size(t) == int((own == r).sum())
                    np.testing.assert_array_equal(e.enumerate_ids(t).cpu().numpy(), mat[own == r])

    def check_counters(self):
        for r, e in enumerate(self.engines):
            st = e.status()[1]
            assert st["push_indices"] == self.steps * self.B * len(self.feats), st
            assert st["update_unique"] == self.expect_unique[r], (r, st["update_unique"], self.expect_unique[r])

    def close(self):
        for e in self.engines:
            e.close()


def _dims_tables(dims, cfg, flip=0):
    return [{"dim": d, "vocab": 4096, "is_hash": (i + flip) % 2 == 1, "cfg": cfg} for i, d in enumerate(dims)]


# ------------------------------------------------------------------ row shape x kernel path x {default, sgd, test}
MATRIX = [(p, b) for p in PATHS for b in (1, 0)]


@pytest.mark.parametrize("opt", list(EXACT))
@pytest.mark.parametrize("path,bulk", MATRIX)
def test_row_shapes_exact(path, bulk, opt, monkeypatch):
    _set_env(monkeypatch, path, bulk)
    cfg = EXACT[opt]
    k = list(PATHS).index(path) + list(EXACT).index(opt)
    dims = DIMS + boundary_dims(cfg)
    world = 2 if path == "pull2" else 1
    batch = [31, 257, 1, 100][k % 4]
    rig = Rig(world, _dims_tables(dims, cfg, flip=k), list(range(len(dims))), batch, path,
              max_ctas=(1 if k % 2 == 0 else None) if world == 1 else 6, seed=k)
    try:
        for t in range(len(dims)):
            rig.seed_rows(t, np.arange(0, 80, 3) if not rig.tables[t]["is_hash"] else np.arange(0, 60, 2) * 1000003 + 11)
        rig.run(3)
        rig.check_tables_exact()
        rig.check_counters()
    finally:
        rig.close()


@pytest.mark.parametrize("opt", list(EXACT))
@pytest.mark.parametrize("path,bulk", [(p, b) for p in PATHS if p != "pull2" for b in (1, 0)])
def test_split_rows_exact(path, bulk, opt, monkeypatch):
    """[D | 1] rows: columns [0, D) at the feature's offset, column D among the linear columns"""
    _set_env(monkeypatch, path, bulk)
    cfg = EXACT[opt]
    k = list(PATHS).index(path) + list(EXACT).index(opt)
    tables = _dims_tables([d + 1 for d in SPLIT_DIMS], cfg, flip=k)
    offs, o = [], 4                                        # a gap in front, and one between features
    for d in SPLIT_DIMS:
        offs.append(o)
        o += (d + 3) // 4 * 4 + 4
    lin = [o + 3 + i for i in range(len(SPLIT_DIMS))]
    layout = {"feat_offsets": offs, "io_stride": (lin[-1] + 8) // 4 * 4, "feat_offsets2": lin, "feat_split": SPLIT_DIMS}
    rig = Rig(1, tables, list(range(len(tables))), [257, 33, 1000][k % 3], path, layout=layout,
              max_ctas=1 if k % 2 else None, seed=100 + k)
    try:
        rig.run(3)
        rig.check_tables_exact()
        rig.check_counters()
    finally:
        rig.close()


LAYOUT_TABLES = [(8, False), (1, False), (1, True), (1, False), (17, True)]


@pytest.mark.parametrize("path,bulk", MATRIX)
def test_layouts_exact(path, bulk, monkeypatch):
    """two features on one table, adjacent dim-1 features, permuted id columns with an unused one, gaps in io_stride"""
    _set_env(monkeypatch, path, bulk)
    cfg = EXACT["test"]                     # counts: duplicates across features of one table must add up
    tables = [{"dim": d, "vocab": 500, "is_hash": h, "cfg": cfg} for d, h in LAYOUT_TABLES]
    feats = [0, 1, 2, 3, 0, 4]
    layout = {"feat_offsets": [4, 13, 14, 15, 24, 40], "io_stride": 68, "feat_cols": [3, 0, 6, 2, 5, 1], "ncols": 7}
    world = 2 if path == "pull2" else 1
    rig = Rig(world, tables, feats, 96, path, layout=layout, seed=7)
    try:
        for t in range(len(tables)):
            rig.seed_rows(t, np.arange(0, 30) * (1000003 if tables[t]["is_hash"] else 1) + (11 if tables[t]["is_hash"] else 0))
        rig.run(3)
        rig.check_tables_exact()
        rig.check_counters()
    finally:
        rig.close()


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("path", list(PATHS))
def test_virtual_ranks_exact(world, path, monkeypatch):
    """every rank's push kernel resident at once (max_ctas=6); shards with shard_num < W and shard_base != 0"""
    _set_env(monkeypatch, path, 1)
    opt = list(EXACT)[(world + list(PATHS).index(path)) % 3]
    cfg = EXACT[opt]
    tables = [{"dim": 16, "vocab": 3000, "is_hash": False, "cfg": cfg},
              {"dim": 4, "vocab": 0, "is_hash": True, "cfg": cfg},
              {"dim": 1, "vocab": 3000, "is_hash": False, "cfg": cfg, "shard_num": world - 1, "shard_base": 1},
              {"dim": 33, "vocab": 0, "is_hash": True, "cfg": cfg, "shard_num": world - 1, "shard_base": world - 1},
              {"dim": 200, "vocab": 3000, "is_hash": False, "cfg": cfg, "shard_num": 1, "shard_base": 1},
              {"dim": 2049, "vocab": 0, "is_hash": True, "cfg": cfg}]
    rig = Rig(world, tables, [0, 1, 2, 3, 4, 5, 0], [257, 31][world % 2], path, seed=world)
    try:
        for t in range(len(tables)):
            rig.seed_rows(t, np.arange(0, 40) * (1000003 if tables[t]["is_hash"] else 1) + (11 if tables[t]["is_hash"] else 0))
        rig.run(3)
        rig.check_tables_exact()
        rig.check_counters()
    finally:
        rig.close()


# ------------------------------------------------------------------ stateful optimizers: within a derived bound
STATEFUL = [c for c in CONFIGS if c["category"] not in ("default", "sgd")]
BOUNDED_PATHS = [("v2", 1), ("v1", 0), ("v2next", 1), ("stateless", 0), ("v1", 1), ("v2", 0)]
REPORT = {}


@pytest.mark.parametrize("idx", range(len(STATEFUL)), ids=lambda i: "-".join("%s=%s" % kv for kv in STATEFUL[i].items()))
def test_stateful_optimizers_within_bound(idx, monkeypatch):
    cfg = STATEFUL[idx]
    path, bulk = BOUNDED_PATHS[idx % len(BOUNDED_PATHS)]
    _set_env(monkeypatch, path, bulk)
    dims = [3, 5, 64, 200, 2052] + boundary_dims(cfg)           # one per row-shape class + the bulk-apply limit
    tables = _dims_tables(dims, cfg, flip=idx)
    rig = Rig(1, tables, list(range(len(dims))), 64, path, exact=False, seed=200 + idx)
    try:
        for t in range(len(dims)):
            rig.seed_rows(t, np.arange(0, 40) * (1000003 if tables[t]["is_hash"] else 1) + (11 if tables[t]["is_hash"] else 0))
        kinds = ["uniform"] * len(dims)                          # rows touched repeatedly: the optimizer state matters
        batches = [rig.make_batch(s, kinds) for s in range(5)]
        for s in range(5):
            rig.step(batches[s], rig.make_grads(s), [torch.from_numpy(b).to(rig.dev) for b in batches[s]],
                     check_pull=False)
        worst, sens = 0.0, np.inf
        for t in range(len(dims)):
            ids, w, s = rig.gathered(t)
            ref = rig.refs[t]
            ww, ws = ref.get(ids)
            wb, sb = ref.bound(ids)
            nsd = s.shape[1]
            if ref.c["category"] in ("adam", "adamax"):        # per-row beta powers: the float32 replica, exactly
                nsc = 2 if ref.c["category"] == "adam" else 1
                exact = TableRef(ref.dim, ref.vocab, ref.is_hash, cfg, INIT, exact=True)
                exact.seed(ids, np.zeros((ids.size, ref.dim), np.float32))
                for rec in rig.hist:
                    for (tt, li, lg) in rec:
                        if tt == t:
                            exact.step(li, lg)
                np.testing.assert_array_equal(s[:, nsd - nsc:], exact.get(ids)[1][:, nsd - nsc:])
            rw = np.abs(w - ww) / np.maximum(wb, 1e-45)
            rs = np.abs(s - ws) / np.maximum(sb, 1e-45)
            worst = max(worst, float(rw.max()), float(rs.max()))
            assert rw.max() <= 1 and rs.max() <= 1, (t, dims[t], float(rw.max()), float(rs.max()))
            # sensitivity: the reference without one lookup's gradient (an id with a single lookup in step 0)
            t0, li, lg = next(r for r in rig.hist[0] if r[0] == t)
            ok = valid_ids(li, ref.vocab, ref.is_hash)
            u, c = np.unique(li[ok], return_counts=True)
            target = u[c == 1][0] if (c == 1).any() else u[0]
            j = int(np.nonzero(li == target)[0][0])
            alt = TableRef(ref.dim, ref.vocab, ref.is_hash, cfg, INIT, exact=False)
            alt.seed(*rig.seeded[t])
            for s_i, rec in enumerate(rig.hist):
                for (tt, li2, lg2) in rec:
                    if tt == t:
                        lg2 = lg2.copy()
                        if s_i == 0:
                            lg2[j] = 0
                        alt.step(li2, lg2)
            k = int(np.nonzero(ids == target)[0][0])
            moved = np.abs(alt.get([target])[0][0] - ww[k]) / np.maximum(wb[k], 1e-45)
            sens = min(sens, float(moved.max()))
            assert moved.max() >= 10, (t, dims[t], float(moved.max()))
        REPORT[idx] = (cfg, worst, sens)
        print("\n[bound] %s: path %s bulk %d, largest error/bound %.3g, sensitivity %.3g (C = %g)"
              % (cfg, path, bulk, worst, sens, BOUND_C))
    finally:
        rig.close()


# ------------------------------------------------------------------ cold rows: the initializers against the CPU engine's
INITS = {"uniform": {"category": "uniform", "minval": -0.5, "maxval": 0.5, "seed": 3},
         "normal": {"category": "normal", "mean": 2.0, "stddev": 0.25, "seed": 4},          # no value near zero:
         "truncated": {"category": "normal", "mean": 2.0, "stddev": 0.25, "truncated": 1.5, "seed": 5}}   # ulps stay meaningful
INIT_MAX_ULPS = 8


def _ulps(a, b):
    return np.abs(a.astype(np.float32).view(np.int32).astype(np.int64) - b.astype(np.float32).view(np.int32).astype(np.int64))


@pytest.mark.parametrize("init", list(INITS))
def test_cold_rows_match_cpu_initializer(init, monkeypatch):
    """cold rows: array rows are filled at allocation, hash rows are generated by the pull (flag 2); both against
    exb_init_rows_f32. The float32 Philox / Box-Muller path uses logf / sinf / cosf / sqrtf on both sides."""
    from openembedding_b200 import _native
    from openembedding_b200.config import initializer_params, mix_seed
    from openembedding_b200.ops.sparse_engine import CudaEngine
    monkeypatch.setenv("EXB_SPARSE_V2", "1")
    lib = _native.core()
    e = CudaEngine(0, 0, 1)
    dims = [3, 5, 64, 200]
    for vid, d in enumerate(dims):
        for h in (False, True):
            t = e.add_table(d, 3000, h)
            e.set_initializer(t, INITS[init], 2 * vid + h)
            e.set_optimizer(t, EXACT["sgd"])
            e.alloc(t)
    plan = e.make_plan(list(range(2 * len(dims))), 2000)
    worst = 0
    try:
        keys = np.arange(2000, dtype=np.int64)
        ids = np.stack([keys if t % 2 == 0 else keys * 7919 + 1 for t in range(2 * len(dims))], 1)
        out = plan.pull(torch.from_numpy(ids).cuda()).cpu().numpy()
        kind, p, seed = initializer_params(INITS[init])
        for t, sl in enumerate(plan.feature_slices()):
            d = dims[t // 2]
            want = np.empty((2000, d), np.float32)
            k = np.ascontiguousarray(ids[:, t], dtype=np.uint64)
            lib.exb_init_rows_f32(kind, p[0], p[1], p[2], mix_seed(seed, t), k.ctypes.data, k.size, d, want.ctypes.data)
            u = _ulps(out[:, sl], want)
            worst = max(worst, int(u.max()))
            if init == "uniform":
                assert u.max() == 0, t           # one FMA on both sides
        print("\n[init] %s: largest difference %d ulps" % (init, worst))
        assert worst <= INIT_MAX_ULPS, worst
    finally:
        e.close()


# ------------------------------------------------------------------ a hash shard at and over capacity
@pytest.mark.parametrize("v2", [0, 1])
def test_hash_shard_capacity(v2, monkeypatch):
    """Near capacity: a 1024-slot shard filled to ~97 % with probe chains that wrap past the end of the slab and new
    colliding ids in one batch. Over capacity: check() raises Status.OOM, rows present before are unchanged and the
    ids that got a slot got exactly their update. After rehash: the ids that failed train again, and their dropped
    gradient must not come back (it used to stay in the accumulator row of the failed id and was applied later)."""
    from openembedding_b200.ops.sparse_engine import CudaEngine
    from openembedding_b200.status import Status, StatusError
    monkeypatch.setenv("EXB_SPARSE_V2", str(v2))
    monkeypatch.delenv("EXB_BULK", raising=False)
    cfg = {"category": "sgd", "learning_rate": 0.25}
    dim, B = 8, 320
    rng = np.random.default_rng(11)
    e = CudaEngine(0, 0, 1)
    t = e.add_table(dim, 0, True, capacity=1024)
    e.set_initializer(t, {"category": "constant", "value": INIT}, 0)
    e.set_optimizer(t, cfg)
    e.alloc(t)
    plan = e.make_plan([t], B)
    ref = TableRef(dim, 0, True, cfg, INIT)
    pool = np.arange(1, 40000, dtype=np.int64) * 7919 + 13
    home = np.array([hash64(int(x)) & 1023 for x in pool])
    tail = pool[home >= 1016][:48]                          # probe chains wrap past slot 1023
    rest = pool[home < 1016]
    fresh = list(np.concatenate([tail, rest[:993 - tail.size]]))
    order = rng.permutation(len(fresh))
    fresh = [fresh[i] for i in order]

    def push(ids):
        ids = np.asarray(ids, dtype=np.int64)
        g = dyadic(rng, (ids.size, dim))
        it = torch.from_numpy(ids.reshape(-1, 1)).cuda()
        plan.pull(it, train=True)
        plan.push_update(it, torch.from_numpy(g).cuda())
        torch.cuda.synchronize()
        return ids, g

    def check_rows(ids):
        ids = np.unique(np.asarray(ids, dtype=np.int64))
        w, s = e.gather_rows(t, torch.from_numpy(ids))
        ww, ws = ref.get(ids)
        np.testing.assert_array_equal(w.cpu().numpy(), ww)
        np.testing.assert_array_equal(s.cpu().numpy(), ws)

    try:
        done = []
        for step in range(4):                                   # ~248 new ids per step + repeats, tail ids together
            new = fresh[step * 249:(step + 1) * 249] if step < 3 else fresh[3 * 249:]
            old = list(rng.choice(done, size=B - len(new))) if done else list(rng.choice(new, size=B - len(new)))
            ids, g = push(new + old)
            e.check()
            ref.step(ids, g)
            done += new
            check_rows(done)
            assert e.table_size(t) == len(ref.materialized())
        assert len(ref.materialized()) == 993
        before = np.array(done, dtype=np.int64)
        extra = list(rest[993 - tail.size:993 - tail.size + 100])
        ids, g = push(extra + extra[:B - 100])                  # 100 new ids, 31 free slots
        with pytest.raises(StatusError) as ei:
            e.check()
        assert ei.value.status == Status.OOM
        keys = set(e.enumerate_ids(t).cpu().numpy().tolist())
        got = [x for x in extra if x in keys]
        failed = [x for x in extra if x not in keys]
        assert len(got) == 1024 - 993 and len(failed) == 100 - len(got) and e.table_size(t) == 1024
        keep = np.isin(ids, got)
        ref.step(ids[keep], g[keep])                            # the failed ids' gradients are dropped
        check_rows(before)
        check_rows(got)
        e.rehash(t, 4096)
        e.commit()
        for step in range(4):                                   # v2 alternates its two batch slots
            ids, g = push(failed + got + list(rng.choice(done, size=B - 100)))
            e.check()
            ref.step(ids, g)
            check_rows(done + extra)
        assert e.table_size(t) == len(ref.materialized())
    finally:
        e.close()


# ------------------------------------------------------------------ fp64 tables: bit-identical to the CPU engine
FP64_POW_RTOL = 1e-13


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: "-".join("%s=%s" % kv for kv in c.items()))
def test_float64_tables_bit_identical_to_cpu_engine(cuda_context, cfg):
    """dev_shard.cu shares exb_math.h with the CPU engine and is built without multiply-add contraction"""
    import openembedding_b200.torch as embed
    from openembedding_b200 import _native
    from openembedding_b200.config import optimizer_params
    from openembedding_b200.context import get_context
    ctx = get_context()
    lib = _native.core()
    kind, p = optimizer_params(cfg)
    for dim in (1, 5, 64):
        torch.manual_seed(dim)
        rows = 9
        w0 = torch.randn(rows, dim, dtype=torch.float64)
        var = embed.Variable(initializer="zeros", dtype=torch.float64, shape=(rows, dim))
        var.set_server_optimizer(dict(cfg))
        keys = np.arange(rows, dtype=np.uint64)
        ctx.backend.load_rows(var.variable, keys, w0.numpy(), np.empty((rows, 0)))
        h = lib.exb_var_create(0x108, dim, rows, 0, 1, 0)
        lib.exb_var_set_optimizer(h, kind, (ctypes.c_double * 8)(*p), 8)
        w0n = np.ascontiguousarray(w0.numpy())
        lib.exb_var_set_weights(h, keys.ctypes.data, rows, w0n.ctypes.data, None, 0)
        for step in range(6):
            ids = np.random.default_rng(step).permutation(rows)[:rows - step % 3]     # unique ids, some rows skipped
            g = torch.randn(ids.size, dim, dtype=torch.float64)
            var.push_gradients(torch.from_numpy(ids).to(ctx.device), g.to(ctx.device))
            var.update_weights()
            k = np.ascontiguousarray(ids, dtype=np.uint64)
            gn = np.ascontiguousarray(g.numpy())
            lib.exb_var_push(h, k.ctypes.data, k.size, gn.ctypes.data, None)
            lib.exb_var_update(h)
        got = var.sparse_read(torch.arange(rows, device=ctx.device)).detach().cpu().numpy()
        want = np.empty((rows, dim), np.float64)
        lib.exb_var_pull(h, keys.ctypes.data, rows, want.ctypes.data)
        lib.exb_var_destroy(h)
        ulps = np.abs(got.view(np.int64) - want.view(np.int64))
        print("\n[fp64] %s dim %d: largest difference %d ulps, %.3g absolute"
              % (cfg, dim, int(ulps.max()), float(np.abs(got - want).max())))
        if cfg["category"] == "ftrl" and cfg.get("learning_rate_power", -0.5) != -0.5:
            # pow(): CUDA's double pow (<= 2 ulps) is not the host libm's. Weights near zero make ulps meaningless
            # (229 ulps measured on H100); the largest difference was below 1e-15 absolute
            np.testing.assert_allclose(got, want, rtol=FP64_POW_RTOL, atol=FP64_POW_RTOL)
        else:
            assert ulps.max() == 0, (dim, int(ulps.max()))
