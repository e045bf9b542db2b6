"""Sparse-table backends behind ``Context``.

* ``CudaBackend`` -- the product: HBM shards + fused sm_90a kernels + NVLink peer memory
  (``ops/sparse_engine.py``).
* ``CpuBackend``  -- the plumbing/oracle configuration (BASELINE config 1: CPU + gloo):
  shards live in ``libexb_core`` and ids / rows / grads travel with
  ``all_to_all_single`` -- structurally the reference's pull/push RPC
  (EmbeddingPullOperator.cpp:40-252, EmbeddingPushOperator.cpp:29-161) on torch
  collectives.

Both expose per-variable verbs (``pull`` / ``push`` / ``update``) and a fused multi-table
group (``make_group``) used by the model zoo.
"""
import ctypes

import numpy as np
import torch

from . import _native
from .config import DTYPES, initializer_params, mix_seed, optimizer_params, optimizer_state_dim


class VarMeta:
    def __init__(self, variable_id, storage_id, vocab, dim, dtype, is_hash, shard_num, shard_base):
        self.variable_id, self.storage_id = variable_id, storage_id
        self.vocab, self.dim, self.dtype, self.is_hash = vocab, dim, dtype, is_hash
        self.shard_num, self.shard_base = shard_num, shard_base
        self.initializer = {"category": "constant", "value": 0.0}
        self.optimizer = {"category": "default"}
        self.handle = None     # backend specific


def _owner_local(ids, meta, world):
    shard = ids % meta.shard_num
    owner = (meta.shard_base + shard) % world
    return owner, ids // meta.shard_num


# ======================================================================= CPU
class CpuBackend:
    name = "cpu"

    def __init__(self, rank, world, group=None):
        self.rank, self.world, self.group = rank, world, group
        self.lib = _native.core()
        self.device = torch.device("cpu")
        self.vars = []
        self.counters = {"pull_indices": 0, "pull_unique": 0, "push_indices": 0}

    # ---- variables
    def create_variable(self, meta):
        my_shard = (self.rank - meta.shard_base) % self.world
        meta.my_shard = my_shard if my_shard < meta.shard_num else -1
        sid = max(meta.my_shard, 0)
        h = self.lib.exb_var_create(DTYPES[meta.dtype], meta.dim, 0 if meta.is_hash else meta.vocab, sid,
                                    meta.shard_num, 1 if meta.is_hash else 0)
        if not h:
            raise ValueError("unsupported dtype for server variable: %s" % meta.dtype)
        meta.handle = h
        self.vars.append(meta)
        return meta

    def set_initializer(self, meta, cfg):
        kind, p, seed = initializer_params(cfg)
        self.lib.exb_var_set_initializer(meta.handle, kind, p[0], p[1], p[2], mix_seed(seed, meta.variable_id))

    def set_optimizer(self, meta, cfg):
        kind, p = optimizer_params(cfg)
        self.lib.exb_var_set_optimizer(meta.handle, kind, (ctypes.c_double * 8)(*p), 8)

    def _tdtype(self, meta):
        return torch.float32 if meta.dtype == "float32" else torch.float64

    # ---- exchange helpers
    def _a2a(self, send, send_counts, width, dtype):
        import torch.distributed as dist
        counts_in = torch.tensor(send_counts, dtype=torch.int64)
        counts_out = torch.empty(self.world, dtype=torch.int64)
        dist.all_to_all_single(counts_out, counts_in, group=self.group)
        recv_counts = counts_out.tolist()
        recv = torch.empty((sum(recv_counts),) + ((width,) if width else ()), dtype=dtype)
        dist.all_to_all_single(recv, send.contiguous(), output_split_sizes=recv_counts,
                               input_split_sizes=list(send_counts), group=self.group)
        return recv, recv_counts

    def _a2a_known(self, send, send_counts, recv_counts, width, dtype):
        import torch.distributed as dist
        recv = torch.empty((sum(recv_counts),) + ((width,) if width else ()), dtype=dtype)
        dist.all_to_all_single(recv, send.contiguous(), output_split_sizes=list(recv_counts),
                               input_split_sizes=list(send_counts), group=self.group)
        return recv

    # ---- verbs
    def pull(self, meta, ids):
        ids = ids.reshape(-1).to(torch.int64).contiguous()
        n = ids.numel()
        dt = self._tdtype(meta)
        self.counters["pull_indices"] += n
        # K1: dedup (reference client dedups per variable, EmbeddingPullOperator.cpp:60-84)
        uniq, inverse = torch.unique(ids, return_inverse=True)
        self.counters["pull_unique"] += uniq.numel()
        if self.world == 1:
            local = (uniq // meta.shard_num).contiguous()
            rows = torch.empty((uniq.numel(), meta.dim), dtype=dt)
            self.lib.exb_var_pull(meta.handle, local.data_ptr(), uniq.numel(), rows.data_ptr())
            return rows[inverse]
        owner, local = _owner_local(uniq, meta, self.world)
        order = torch.argsort(owner, stable=True)
        send_counts = torch.bincount(owner, minlength=self.world).tolist()
        req, recv_counts = self._a2a(local[order], send_counts, 0, torch.int64)
        rows = torch.empty((req.numel(), meta.dim), dtype=dt)
        if req.numel():
            self.lib.exb_var_pull(meta.handle, req.data_ptr(), req.numel(), rows.data_ptr())
        back = self._a2a_known(rows, recv_counts, send_counts, meta.dim, dt)
        urows = torch.empty((uniq.numel(), meta.dim), dtype=dt)
        urows[order] = back
        return urows[inverse]

    def push(self, meta, ids, grads):
        ids = ids.reshape(-1).to(torch.int64).contiguous()
        dt = self._tdtype(meta)
        grads = grads.reshape(-1, meta.dim).to(dt).contiguous()
        self.counters["push_indices"] += ids.numel()
        # K4a: per-worker pre-reduce (sum grads, count duplicates; EmbeddingPushOperator.cpp:29-62)
        uniq, inverse, counts = torch.unique(ids, return_inverse=True, return_counts=True)
        g = torch.zeros((uniq.numel(), meta.dim), dtype=dt)
        g.index_add_(0, inverse, grads)
        counts = counts.to(torch.int64)
        if self.world == 1:
            local = (uniq // meta.shard_num).contiguous()
            self.lib.exb_var_push(meta.handle, local.data_ptr(), uniq.numel(), g.data_ptr(), counts.data_ptr())
            return
        owner, local = _owner_local(uniq, meta, self.world)
        order = torch.argsort(owner, stable=True)
        send_counts = torch.bincount(owner, minlength=self.world).tolist()
        rid, recv_counts = self._a2a(local[order], send_counts, 0, torch.int64)
        rg = self._a2a_known(g[order], send_counts, recv_counts, meta.dim, dt)
        rc = self._a2a_known(counts[order], send_counts, recv_counts, 0, torch.int64)
        if rid.numel():
            self.lib.exb_var_push(meta.handle, rid.data_ptr(), rid.numel(), rg.data_ptr(), rc.data_ptr())

    def update(self, metas=None):
        import torch.distributed as dist
        if self.world > 1:
            dist.barrier(group=self.group)   # every worker's push has landed (the fake-gradient allreduce of the reference)
        for meta in (metas or self.vars):
            self.lib.exb_var_update(meta.handle)
        if self.world > 1:
            dist.barrier(group=self.group)

    # ---- fused group (loop of per-variable verbs on CPU)
    def make_group(self, metas, batch, feat_cols=None, ncols=None):
        return _CpuGroup(self, metas, batch, feat_cols)

    # ---- checkpoint side
    def num_items(self, meta):
        return int(self.lib.exb_var_num_items(meta.handle))

    def state_dim(self, meta):
        return optimizer_state_dim(meta.optimizer, meta.dim)

    def iter_local_rows(self, meta, block_rows, with_state=True):
        """yields (local_indices u64 ndarray, weights ndarray, states ndarray) of this rank's shard"""
        if getattr(meta, "my_shard", 0) < 0:
            return
        cursor = ctypes.c_uint64(0)
        np_dt = np.float32 if meta.dtype == "float32" else np.float64
        sd = self.state_dim(meta)
        while True:
            idx = np.empty(block_rows, dtype=np.uint64)
            n = int(self.lib.exb_var_read_indices(meta.handle, ctypes.byref(cursor), idx.ctypes.data, block_rows))
            if n == 0:
                break
            idx = idx[:n]
            w = np.empty((n, meta.dim), dtype=np_dt)
            s = np.empty((n, sd), dtype=np_dt)
            self.lib.exb_var_get_weights(meta.handle, idx.ctypes.data, n, w.ctypes.data,
                                         s.ctypes.data if (with_state and sd) else None)
            yield idx, w, (s if with_state else np.empty((n, 0), dtype=np_dt))

    def read_rows(self, meta, global_ids):
        """(weights, states) of the given rows of this rank's shard (host tier write-back)"""
        ids = np.ascontiguousarray(np.asarray(global_ids, dtype=np.uint64) // np.uint64(meta.shard_num))
        np_dt = np.float32 if meta.dtype == "float32" else np.float64
        sd = self.state_dim(meta)
        w = np.empty((ids.size, meta.dim), dtype=np_dt)
        s = np.empty((ids.size, max(sd, 1)), dtype=np_dt)
        if ids.size:
            self.lib.exb_var_get_weights(meta.handle, ids.ctypes.data, ids.size, w.ctypes.data, s.ctypes.data if sd else None)
        return w, s[:, :sd]

    def load_rows(self, meta, global_ids, weights, states):
        """rows whose owner is this rank are stored, the rest ignored (load re-shards)."""
        ids = np.asarray(global_ids, dtype=np.uint64)
        owner = (meta.shard_base + (ids % np.uint64(meta.shard_num)).astype(np.int64)) % self.world
        m = owner == self.rank
        if not m.any():
            return
        local = np.ascontiguousarray(ids[m] // np.uint64(meta.shard_num))
        np_dt = np.float32 if meta.dtype == "float32" else np.float64
        w = np.ascontiguousarray(np.asarray(weights)[m], dtype=np_dt)
        sd = self.state_dim(meta)
        st = np.asarray(states)
        has_state = st.size > 0 and st.shape[1] == sd and sd > 0
        s = np.ascontiguousarray(st[m], dtype=np_dt) if has_state else None
        self.lib.exb_var_set_weights(meta.handle, local.ctypes.data, local.size, w.ctypes.data,
                                     s.ctypes.data if s is not None else None,
                                     sd * w.itemsize if s is not None else 0)

    def clear(self, meta):
        self.lib.exb_var_clear(meta.handle)

    def table_kind(self, meta):
        return "hash" if meta.is_hash else "array"

    def shard_id(self, meta):
        return getattr(meta, "my_shard", 0)

    def synchronize(self):
        pass

    def close(self):
        for m in self.vars:
            if m.handle:
                self.lib.exb_var_destroy(m.handle)
                m.handle = None
        self.vars = []


class _CpuGroup:
    def __init__(self, backend, metas, batch, feat_cols=None):
        self.b, self.metas, self.B = backend, list(metas), batch
        self.feat_cols = list(feat_cols) if feat_cols is not None else list(range(len(self.metas)))
        self.dims = [m.dim for m in metas]
        offs, o = [], 0
        for d in self.dims:
            offs.append(o)
            o += d
        self.feat_offsets, self.io_stride = offs, o

    def feature_slices(self):
        return [slice(o, o + d) for o, d in zip(self.feat_offsets, self.dims)]

    def pull(self, ids, out=None, train=False):
        out = torch.empty((ids.shape[0], self.io_stride), dtype=torch.float32)
        for f, m in enumerate(self.metas):
            out[:, self.feat_offsets[f]:self.feat_offsets[f] + m.dim] = self.b.pull(m, ids[:, self.feat_cols[f]]).to(torch.float32)
        return out

    def push_update(self, ids, grads):
        for f, m in enumerate(self.metas):
            self.b.push(m, ids[:, self.feat_cols[f]], grads[:, self.feat_offsets[f]:self.feat_offsets[f] + m.dim])
        self.b.update(list(dict.fromkeys(self.metas)))


# ====================================================================== CUDA, float64 tables
class _F64Tables:
    """float64 variables on the GPU (``csrc/cuda/dev_shard.cu``): device-resident shards with the CPU oracle's four
    verbs executed by kernels (bit-identical math), ids / rows / gradients routed between ranks with NCCL
    ``all_to_all_single`` on device tensors -- the structure of ``CpuBackend`` with every buffer in HBM.
    Reference: float and double tables are both registered (EmbeddingVariable.cpp:277-278)."""

    def __init__(self, be):
        self.be = be
        self.lib = be.engine.lib
        self.dev = be.device
        self.pending = {}

    def _ck(self, rc, what):
        if rc != 0:
            raise RuntimeError("dev shard %s: %s" % (what, self.lib.exb_ds_last_error().decode()))

    def _st(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def create(self, meta):
        be = self.be
        my = (be.rank - meta.shard_base) % be.world
        meta.my_shard = my if my < meta.shard_num else -1
        cap = getattr(meta, "capacity", None) or (1 << 16)
        h = self.lib.exb_ds_create(be.engine.device_index, 8, meta.dim, 0 if meta.is_hash else meta.vocab,
                                   max(meta.my_shard, 0), meta.shard_num, 1 if meta.is_hash else 0, int(cap))
        if not h:
            raise RuntimeError("exb_ds_create: " + self.lib.exb_ds_last_error().decode())
        meta.handle, meta.f64, meta.allocated = h, True, True
        return meta

    def set_initializer(self, meta, cfg):
        kind, p, seed = initializer_params(cfg)
        self._ck(self.lib.exb_ds_set_initializer(meta.handle, kind, p[0], p[1], p[2], mix_seed(seed, meta.variable_id)), "init")

    def set_optimizer(self, meta, cfg):
        kind, p = optimizer_params(cfg)
        self._ck(self.lib.exb_ds_set_optimizer(meta.handle, kind, (ctypes.c_double * 8)(*p), 8), "optimizer")

    # ---- exchange (device tensors, NCCL)
    def _a2a(self, send, send_counts, width, dtype):
        import torch.distributed as dist
        ci = torch.tensor(send_counts, dtype=torch.int64, device=self.dev)
        co = torch.empty(self.be.world, dtype=torch.int64, device=self.dev)
        dist.all_to_all_single(co, ci, group=self.be.group)
        rc = co.tolist()
        recv = torch.empty((sum(rc),) + ((width,) if width else ()), dtype=dtype, device=self.dev)
        dist.all_to_all_single(recv, send.contiguous(), output_split_sizes=rc, input_split_sizes=list(send_counts),
                               group=self.be.group)
        return recv, rc

    def _a2a_known(self, send, sc, rc, width, dtype):
        import torch.distributed as dist
        recv = torch.empty((sum(rc),) + ((width,) if width else ()), dtype=dtype, device=self.dev)
        dist.all_to_all_single(recv, send.contiguous(), output_split_sizes=list(rc), input_split_sizes=list(sc),
                               group=self.be.group)
        return recv

    def _pull_local(self, meta, local):
        rows = torch.empty((local.numel(), meta.dim), dtype=torch.float64, device=self.dev)
        self._ck(self.lib.exb_ds_pull(meta.handle, local.data_ptr(), local.numel(), rows.data_ptr(), self._st()), "pull")
        return rows

    def pull(self, meta, ids):
        ids = ids.reshape(-1).to(device=self.dev, dtype=torch.int64).contiguous()
        uniq, inverse = torch.unique(ids, return_inverse=True)
        W = self.be.world
        if W == 1:
            return self._pull_local(meta, (uniq // meta.shard_num).contiguous())[inverse]
        owner, local = _owner_local(uniq, meta, W)
        order = torch.argsort(owner, stable=True)
        sc = torch.bincount(owner, minlength=W).tolist()
        req, rc = self._a2a(local[order], sc, 0, torch.int64)
        rows = self._pull_local(meta, req.contiguous())
        back = self._a2a_known(rows, rc, sc, meta.dim, torch.float64)
        urows = torch.empty((uniq.numel(), meta.dim), dtype=torch.float64, device=self.dev)
        urows[order] = back
        return urows[inverse]

    def push(self, meta, ids, grads):
        ids = ids.reshape(-1).to(device=self.dev, dtype=torch.int64)
        grads = grads.reshape(-1, meta.dim).to(device=self.dev, dtype=torch.float64)
        self.pending.setdefault(meta.variable_id, []).append((ids, grads))

    def update(self, meta):
        pend = self.pending.pop(meta.variable_id, None)
        W = self.be.world
        if not pend:
            if W == 1:
                return
            ids = torch.zeros(0, dtype=torch.int64, device=self.dev)
            g = torch.zeros((0, meta.dim), dtype=torch.float64, device=self.dev)
        else:
            ids = torch.cat([p[0] for p in pend])
            g = torch.cat([p[1] for p in pend])
        # K4a: per-worker pre-reduce (sum duplicate gradients, count them)
        uniq, inverse, counts = torch.unique(ids, return_inverse=True, return_counts=True)
        gs = torch.zeros((uniq.numel(), meta.dim), dtype=torch.float64, device=self.dev).index_add_(0, inverse, g)
        if W == 1:
            local, cnt = (uniq // meta.shard_num).contiguous(), counts.contiguous()
        else:
            owner, loc = _owner_local(uniq, meta, W)
            order = torch.argsort(owner, stable=True)
            sc = torch.bincount(owner, minlength=W).tolist()
            rid, rc = self._a2a(loc[order], sc, 0, torch.int64)
            rg = self._a2a_known(gs[order], sc, rc, meta.dim, torch.float64)
            rcnt = self._a2a_known(counts[order], sc, rc, 0, torch.int64)
            local, inv2 = torch.unique(rid, return_inverse=True)          # K4b: combine the sources
            gs = torch.zeros((local.numel(), meta.dim), dtype=torch.float64, device=self.dev).index_add_(0, inv2, rg)
            cnt = torch.zeros(local.numel(), dtype=torch.int64, device=self.dev).index_add_(0, inv2, rcnt)
        if local.numel():
            self._ck(self.lib.exb_ds_update(meta.handle, local.data_ptr(), local.numel(), gs.data_ptr(), cnt.data_ptr(),
                                            self._st()), "update")
        torch.cuda.current_stream(self.dev).synchronize()      # keeps local / gs / cnt alive until the kernel ran
        if self.lib.exb_ds_status(meta.handle):
            from .status import Status, StatusError
            raise StatusError(Status.OOM, "float64 shard full")

    # ---- checkpoint side
    def num_items(self, meta):
        return int(self.lib.exb_ds_num_items(meta.handle))

    def local_ids(self, meta):
        n = self.num_items(meta)
        out = torch.empty(max(n, 1), dtype=torch.int64, device=self.dev)
        cnt = (ctypes.c_uint64 * 1)()
        self._ck(self.lib.exb_ds_enumerate(meta.handle, out.data_ptr(), cnt), "enumerate")
        return torch.sort(out[: int(cnt[0])])[0]

    def get(self, meta, local, with_state=True):
        local = local.to(device=self.dev, dtype=torch.int64).contiguous()
        sd = int(self.lib.exb_ds_state_dim(meta.handle))
        w = torch.empty((local.numel(), meta.dim), dtype=torch.float64, device=self.dev)
        s = torch.empty((local.numel(), max(sd, 1)), dtype=torch.float64, device=self.dev)
        self._ck(self.lib.exb_ds_get(meta.handle, local.data_ptr(), local.numel(), w.data_ptr(),
                                     s.data_ptr() if (with_state and sd) else 0, self._st()), "get")
        torch.cuda.current_stream(self.dev).synchronize()
        return w, (s[:, :sd] if with_state else s[:, :0])

    def set(self, meta, local, w, s):
        local = local.to(device=self.dev, dtype=torch.int64).contiguous()
        w = w.to(device=self.dev, dtype=torch.float64).contiguous()
        s = s.to(device=self.dev, dtype=torch.float64).contiguous() if s is not None else None
        self._ck(self.lib.exb_ds_set(meta.handle, local.data_ptr(), local.numel(), w.data_ptr(),
                                     s.data_ptr() if s is not None else 0, self._st()), "set")
        torch.cuda.current_stream(self.dev).synchronize()


# ====================================================================== CUDA
class CudaBackend:
    name = "cuda"

    def __init__(self, rank, world, device_index, group=None):
        from .ops.sparse_engine import CudaEngine
        self.rank, self.world, self.group = rank, world, group
        self.engine = CudaEngine(device_index, rank, world)
        self.device = self.engine.device
        self.vars = []
        self._plans = {}      # (variable_id, B) -> SparsePlan
        self._pending = {}    # variable_id -> [(ids, grads)]
        self.hash_reserve = 1 << 20
        self._f64 = None      # float64 tables (dev_shard.cu)

    def create_variable(self, meta):
        if meta.dtype == "float64":          # exact fp64 shard engine (dev_shard.cu); fp32 = the fused engine
            if self._f64 is None:
                self._f64 = _F64Tables(self)
            self._f64.create(meta)
            self.vars.append(meta)
            return meta
        if meta.dtype != "float32":
            raise ValueError("unsupported dtype for server variable: %s" % meta.dtype)
        t = self.engine.add_table(meta.dim, meta.vocab, meta.is_hash,
                                  capacity=getattr(meta, "capacity", None) or self.hash_reserve,
                                  shard_num=meta.shard_num, shard_base=meta.shard_base)
        meta.handle = t
        meta.allocated = False
        self.vars.append(meta)
        return meta

    def set_initializer(self, meta, cfg):
        if getattr(meta, "f64", False):
            return self._f64.set_initializer(meta, cfg)
        if getattr(meta, "allocated", False):
            # weights are materialised eagerly; a later initializer only affects rows
            # that are (re)created from now on (hash misses, clear()).
            pass
        self.engine.set_initializer(meta.handle, cfg, meta.variable_id)

    def set_optimizer(self, meta, cfg):
        if getattr(meta, "f64", False):
            return self._f64.set_optimizer(meta, cfg)
        self.engine.set_optimizer(meta.handle, cfg)
        if getattr(meta, "allocated", False):
            self.engine.commit()
        if getattr(meta, "tiered", False):
            from .host_tier import tier_of
            t = tier_of(meta)
            if t is not None and hasattr(t, "on_optimizer_change"):
                t.on_optimizer_change()

    def ensure_allocated(self, metas=None):
        """Collective: materialise not-yet-allocated tables and map them on every peer."""
        todo = [m for m in (metas or self.vars) if not m.allocated and not getattr(m, "f64", False)]
        if not todo:
            return
        self._check_memory_limits(todo)
        for m in todo:
            self.engine.alloc(m.handle)
            m.allocated = True
        self.engine.connect(self.group)

    soft_limit_mb = hard_limit_mb = 0

    def _check_memory_limits(self, todo):
        """ShardStorageMemory analogue: refuse (hard) / warn about (soft) allocations beyond the configured budget"""
        if not (self.soft_limit_mb or self.hard_limit_mb):
            return
        from .status import Status, StatusError
        from .utils import log
        held = self.engine.memory_info()
        want = held["tables_bytes"] + held["plans_bytes"] + sum(self.engine.table_bytes_estimate(m.handle) for m in todo)
        if self.hard_limit_mb and want > self.hard_limit_mb << 20:
            raise StatusError(Status.OOM, "sparse engine would hold %d MB, server.memory_hard_limit_mb is %d"
                              % (want >> 20, self.hard_limit_mb))
        if self.soft_limit_mb and want > self.soft_limit_mb << 20:
            log.warning("sparse engine holds %d MB, above server.memory_soft_limit_mb = %d" % (want >> 20, self.soft_limit_mb))

    def memory_info(self):
        info = self.engine.memory_info()
        from .host_tier import _tiers
        tiers = {vid: t.memory() for vid, t in _tiers.items() if hasattr(t, "memory")}
        info["tiers"] = tiers
        info["tiers_bytes"] = sum(t["hbm_index_bytes"] for t in tiers.values())
        info["pinned_host_bytes"] = sum(t["pinned_host_bytes"] for t in tiers.values())
        return info

    def _plan_for(self, meta, n):
        """Per-variable plan of capacity next_pow2(n). Creating a plan is collective (IPC exchange) and the
        push kernel contains cross-GPU barriers, so every rank must pick the SAME plan: with world > 1 the
        capacity is agreed on first (MAX of n over the ranks) -- uneven last batches / ragged features would
        otherwise send ranks into different collectives."""
        if self.world > 1:
            import torch.distributed as dist
            t = torch.tensor([int(n)], dtype=torch.int64, device=self.device)
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
            n = int(t[0])
        cap = 1024
        while cap < n:
            cap *= 2
        key = (meta.variable_id, cap)
        plan = self._plans.get(key)
        if plan is None:
            self.ensure_allocated([meta])
            plan = self.engine.make_plan([meta.handle], cap)
            self.engine.connect(self.group)
            self._plans[key] = plan
        return plan

    def pull(self, meta, ids):
        if getattr(meta, "f64", False):
            return self._f64.pull(meta, ids)
        ids = ids.reshape(-1, 1).to(device=self.device, dtype=torch.int64).contiguous()
        plan = self._plan_for(meta, ids.shape[0])
        out = plan.pull(ids)
        return out[:, :meta.dim] if out.shape[1] != meta.dim else out

    def push(self, meta, ids, grads):
        if getattr(meta, "f64", False):
            return self._f64.push(meta, ids, grads)
        ids = ids.reshape(-1, 1).to(device=self.device, dtype=torch.int64).contiguous()
        grads = grads.reshape(-1, meta.dim).to(device=self.device, dtype=torch.float32)
        self._pending.setdefault(meta.variable_id, []).append((ids, grads))

    def update(self, metas=None):
        """Apply the pushed gradients. Collective when world > 1: the kernel is launched on EVERY rank for every
        variable some rank may have pushed to (n = 0 where this rank has nothing) -- a rank that skipped the
        launch would leave its peers waiting in the in-kernel barrier."""
        for meta in (metas or self.vars):
            if getattr(meta, "f64", False):
                self._f64.update(meta)
                continue
            pend = self._pending.pop(meta.variable_id, None)
            if not pend:
                if self.world == 1:
                    continue
                ids = torch.zeros((0, 1), dtype=torch.int64, device=self.device)
                g = torch.zeros((0, meta.dim), dtype=torch.float32, device=self.device)
            else:
                ids = torch.cat([p[0] for p in pend]) if len(pend) > 1 else pend[0][0]
                g = torch.cat([p[1] for p in pend]) if len(pend) > 1 else pend[0][1]
            plan = self._plan_for(meta, ids.shape[0])
            if g.shape[1] != plan.io_stride:
                gp = torch.zeros((g.shape[0], plan.io_stride), dtype=torch.float32, device=self.device)
                gp[:, :meta.dim] = g
                g = gp
            plan.push_update(ids, g.contiguous())

    def make_group(self, metas, batch, feat_cols=None, ncols=None):
        if any(getattr(m, "f64", False) for m in metas):
            raise ValueError("fused plans are float32; float64 variables use the per-variable path")
        self.ensure_allocated(list(metas))
        plan = self.engine.make_plan([m.handle for m in metas], batch, feat_cols=feat_cols, ncols=ncols)
        self.engine.connect(self.group)
        return plan

    # ---- checkpoint side
    def num_items(self, meta):
        if getattr(meta, "f64", False):
            return self._f64.num_items(meta) if meta.my_shard >= 0 else 0
        self.ensure_allocated([meta])
        if meta.is_hash:
            return self.engine.table_size(meta.handle)
        return int(self.engine.enumerate_ids(meta.handle).numel())

    def state_dim(self, meta):
        return optimizer_state_dim(meta.optimizer, meta.dim)

    def shard_id(self, meta):
        s = (self.rank - meta.shard_base) % self.world
        return s if s < meta.shard_num else -1

    def iter_local_rows(self, meta, block_rows, with_state=True):
        """Streaming dump (K8 of SURVEY 2.5): device key compaction, then the rows travel in CHUNKS of many file
        blocks -- gather kernel into a device staging buffer, asynchronous D2H into one of two PINNED host buffers
        on a copy stream -- while the caller writes the previous chunk's blocks: the copy of chunk i+1 overlaps the
        file writes of chunk i. Yields (local indices, weights, states) per file block (views of the pinned buffer)."""
        if getattr(meta, "f64", False):
            if meta.my_shard < 0:
                return
            local = self._f64.local_ids(meta)
            for i in range(0, local.numel(), block_rows):
                blk = local[i:i + block_rows]
                w, s = self._f64.get(meta, blk, with_state=with_state)
                yield blk.cpu().numpy().astype(np.uint64), w.cpu().numpy(), s.cpu().numpy()
            return
        self.ensure_allocated([meta])
        if self.shard_id(meta) < 0:
            return
        ids = self.engine.enumerate_ids(meta.handle)   # device key compaction, sorted
        n = int(ids.numel())
        if n == 0:
            return
        sd = self.state_dim(meta) if with_state else 0
        chunk = max(block_rows, min(n, block_rows * 64))
        dev = self.device
        copy = torch.cuda.Stream(device=dev)
        pinned = [dict(i=torch.empty(chunk, dtype=torch.int64).pin_memory(),
                       w=torch.empty((chunk, meta.dim), dtype=torch.float32).pin_memory(),
                       s=torch.empty((chunk, max(sd, 1)), dtype=torch.float32).pin_memory(),
                       ev=torch.cuda.Event()) for _ in range(2)]

        def launch(c0, buf):
            blk = ids[c0:c0 + chunk]
            w, s = self.engine.gather_rows(meta.handle, blk, with_state=bool(sd))
            cur = torch.cuda.current_stream(dev)
            copy.wait_stream(cur)
            with torch.cuda.stream(copy):
                k = blk.numel()
                buf["i"][:k].copy_(blk // meta.shard_num, non_blocking=True)
                buf["w"][:k].copy_(w, non_blocking=True)
                if sd:
                    buf["s"][:k].copy_(s, non_blocking=True)
                for t in (blk, w, s):
                    if t is not None:
                        t.record_stream(copy)
                buf["ev"].record(copy)
            return k

        k_next = launch(0, pinned[0])
        c0, which = 0, 0
        while c0 < n:
            buf, k = pinned[which], k_next
            if c0 + chunk < n:
                k_next = launch(c0 + chunk, pinned[which ^ 1])      # in flight while this chunk is written
            buf["ev"].synchronize()
            li = buf["i"].numpy().view(np.uint64)
            wv, sv = buf["w"].numpy(), buf["s"].numpy()
            for b0 in range(0, k, block_rows):
                b1 = min(k, b0 + block_rows)
                yield li[b0:b1], wv[b0:b1], (sv[b0:b1, :sd] if sd else np.empty((b1 - b0, 0), dtype=np.float32))
            c0 += chunk
            which ^= 1

    def read_rows(self, meta, global_ids):
        """(weights, states) of the given rows of this rank's shard (host tier write-back): device gather + D2H"""
        self.ensure_allocated([meta])
        ids = torch.from_numpy(np.ascontiguousarray(np.asarray(global_ids, dtype=np.uint64).astype(np.int64)))
        sd = self.state_dim(meta)
        if ids.numel() == 0:
            return np.empty((0, meta.dim), np.float32), np.empty((0, sd), np.float32)
        w, s = self.engine.gather_rows(meta.handle, ids, with_state=True)
        return w.cpu().numpy(), (s.cpu().numpy() if (s is not None and sd) else np.empty((ids.numel(), 0), np.float32))

    def load_rows(self, meta, global_ids, weights, states):
        if getattr(meta, "f64", False):
            ids = np.asarray(global_ids, dtype=np.uint64)
            owner = (meta.shard_base + (ids % np.uint64(meta.shard_num)).astype(np.int64)) % self.world
            m = owner == self.rank
            if not m.any():
                return
            sd = self.state_dim(meta)
            st = np.asarray(states)
            has_state = st.size > 0 and st.shape[1] == sd and sd > 0
            self._f64.set(meta, torch.from_numpy((ids[m] // np.uint64(meta.shard_num)).astype(np.int64)),
                          torch.from_numpy(np.ascontiguousarray(np.asarray(weights)[m], dtype=np.float64)),
                          torch.from_numpy(np.ascontiguousarray(st[m], dtype=np.float64)) if has_state else None)
            return
        self.ensure_allocated([meta])
        ids = np.asarray(global_ids, dtype=np.uint64)
        owner = (meta.shard_base + (ids % np.uint64(meta.shard_num)).astype(np.int64)) % self.world
        m = owner == self.rank
        if not m.any():
            return
        sd = self.state_dim(meta)
        st = np.asarray(states)
        has_state = st.size > 0 and st.shape[1] == sd and sd > 0
        self.engine.scatter_rows(meta.handle, torch.from_numpy(ids[m].astype(np.int64)),
                                 torch.from_numpy(np.ascontiguousarray(np.asarray(weights)[m], dtype=np.float32)),
                                 torch.from_numpy(np.ascontiguousarray(st[m], dtype=np.float32)) if has_state else None)

    def clear(self, meta):
        if getattr(meta, "f64", False):
            self.lib_ds_clear(meta)
            return
        if meta.allocated:
            self.engine.clear_table(meta.handle)

    def lib_ds_clear(self, meta):
        self._f64._ck(self._f64.lib.exb_ds_clear(meta.handle), "clear")

    def table_kind(self, meta):
        return "hash" if meta.is_hash else "array"

    grow_interval, max_load, _steps = 16, 0.5, 0

    def tick(self, n=1):
        """Per training step (``Context.step_done``).

        * every step: ``engine.poll()`` -- the device error word (hash shard full, inbox / combine-map
          overflow, barrier timeout) is read back asynchronously and raised as ``StatusError``; no update is
          ever dropped silently.
        * every ``grow_interval`` steps: occupancy of the hash shards is read back and shards that would pass
          ``max_load`` before the NEXT inspection -- judged from the insert rate seen since the last one -- are
          rehashed to the capacity that keeps them below it (reference: EasyHashMap grows on insert at load 1/2)."""
        before = self._steps
        self._steps += n
        self.engine.poll()
        if self.grow_interval > 0 and before // self.grow_interval != self._steps // self.grow_interval:
            if any(m.is_hash and m.allocated for m in self.vars):
                self.maybe_grow(self.max_load)

    def maybe_grow(self, load_factor=0.5):
        """Collective: grow hash shards whose (projected) load exceeds `load_factor` (all ranks agree)."""
        import torch.distributed as dist
        grew = False
        for meta in self.vars:
            if not (meta.is_hash and meta.allocated) or getattr(meta, "tiered", False):
                continue          # a tiered table's HBM shard is a fixed-size cache: it evicts, it does not grow
            size = self.engine.table_size(meta.handle)
            cap = self.engine.table_info(meta.handle)["rows"]
            last = getattr(meta, "_last_size", 0)
            rate = max(0, size - last)            # inserts since the previous inspection
            meta._last_size = size
            projected = size + 2 * rate           # two more inspection periods of head room
            need = torch.tensor([projected, cap], dtype=torch.int64, device=self.device)
            if self.world > 1:
                dist.all_reduce(need, op=dist.ReduceOp.MAX, group=self.group)
            projected, cap = int(need[0]), int(need[1])
            if projected > cap * load_factor:
                new_cap = cap
                while projected > new_cap * load_factor:
                    new_cap *= 2
                self.engine.rehash(meta.handle, new_cap)
                grew = True
        if grew:
            self.engine.connect(self.group)
        return grew

    def synchronize(self):
        torch.cuda.synchronize(self.device)

    def close(self):
        if self._f64 is not None:
            for m in self.vars:
                if getattr(m, "f64", False) and m.handle:
                    self._f64.lib.exb_ds_destroy(m.handle)
                    m.handle = None
        self.engine.close()
