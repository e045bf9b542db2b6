"""Python face of the sm_90a sparse engine (``csrc/cuda/engine.cu``).

``CudaEngine`` owns the table shards of one rank; ``SparsePlan`` is a fused
multi-table lookup/update plan: ONE ``pull`` launch gathers every feature of a batch
(peer loads over NVLink), ONE ``push_update`` launch dispatches, combines and applies
the optimizer. The reference needs one RPC round per table per verb
(openembedding/client/EmbeddingVariableHandle.cpp:106-155).
"""
import ctypes
import os

import torch

from .. import _native
from ..config import initializer_params, mix_seed, optimizer_params
from ..status import ENGINE_STATUS, Status, StatusError

_STATUS_TEXT = {
    0: "ok", 1: "grid barrier timeout", 2: "peer barrier timeout (a rank did not arrive)",
    3: "hash table full (grow it)", 4: "inbox overflow", 5: "combine map full",
    6: "context version mismatch: a rank moved a table slab (alloc / rehash) after the last connect()",
}


def cuda_available():
    return torch.cuda.is_available()


def _u64arr(n):
    return (ctypes.c_uint64 * n)()


class CudaEngine:
    def __init__(self, device_index=0, rank=0, world=1, max_ctas=None):
        if not torch.cuda.is_available():
            raise RuntimeError("CudaEngine needs a CUDA device; libexb_cuda has no CPU fallback")
        self.lib = _native.cuda()
        self.device_index = int(device_index)
        self.device = torch.device("cuda", self.device_index)
        self.rank, self.world = int(rank), int(world)
        torch.cuda.set_device(self.device)
        torch.zeros(1, device=self.device)  # make sure the primary context exists
        self.h = self.lib.exb_engine_create(self.device_index, self.rank, self.world)
        if not self.h:
            raise RuntimeError("exb_engine_create: " + self.lib.exb_cuda_last_error().decode())
        env_ctas = os.environ.get("EXB_MAX_CTAS")
        if max_ctas is None and env_ctas:
            max_ctas = int(env_ctas)
        if max_ctas:
            self.lib.exb_engine_set_max_ctas(self.h, int(max_ctas))
        self.tables = []          # per table: dict(dim, vocab, is_hash, connected)
        self.plans = []
        self._sync_connected = self.world == 1
        self._peer_open = []      # opened IPC pointers (closed at destroy)
        # asynchronous status read-back (poll()): the error word travels D2H on a side stream into pinned memory
        self._st_stream = torch.cuda.Stream(device=self.device)
        self._st_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._st_ev = torch.cuda.Event()
        self._st_pending = False
        self._st_dev = None

    # ---------------------------------------------------------------- tables
    def add_table(self, dim, vocab, is_hash=False, capacity=0, shard_num=-1, shard_base=0):
        t = self.lib.exb_table_add(self.h, int(bool(is_hash)), int(dim), int(vocab if not is_hash else 0),
                                   int(capacity), int(shard_num), int(shard_base))
        self.tables.append({"dim": int(dim), "vocab": int(vocab), "is_hash": bool(is_hash),
                            "connected": self.world == 1, "allocated": False})
        return t

    def set_initializer(self, t, config, variable_id=0):
        kind, p, seed = initializer_params(config)
        _native.cuda_check(self.lib.exb_table_set_initializer(self.h, t, kind, p[0], p[1], p[2],
                                                              mix_seed(seed, variable_id)), "set_initializer")

    def set_optimizer(self, t, config):
        kind, p = optimizer_params(config)
        arr = (ctypes.c_double * 8)(*p)
        _native.cuda_check(self.lib.exb_table_set_optimizer(self.h, t, kind, arr, 8), "set_optimizer")

    def alloc(self, t):
        _native.cuda_check(self.lib.exb_table_alloc(self.h, t), "table_alloc")
        self.tables[t]["allocated"] = True

    def table_info(self, t):
        out = _u64arr(8)
        self.lib.exb_table_info(self.h, t, out)
        return {"w_ptr": out[0], "w_bytes": out[1], "keys_ptr": out[2], "keys_bytes": out[3],
                "rows": out[4], "wstride": out[5], "sstride": out[6], "state_dim": out[7]}

    def table_size(self, t):
        out = _u64arr(1)
        _native.cuda_check(self.lib.exb_table_size(self.h, t, out), "table_size")
        return int(out[0])

    def commit(self):
        _native.cuda_check(self.lib.exb_engine_commit(self.h), "commit")

    # ------------------------------------------------------- peer connection
    def _export(self, ptr):
        buf = ctypes.create_string_buffer(64)
        _native.cuda_check(self.lib.exb_ipc_get_handle(ptr, buf), "ipc_get_handle")
        return buf.raw

    def _open(self, raw):
        p = self.lib.exb_ipc_open_handle(ctypes.create_string_buffer(raw, 64))
        if not p:
            raise RuntimeError("cudaIpcOpenMemHandle: " + self.lib.exb_cuda_last_error().decode())
        self._peer_open.append(p)
        return p

    def connect(self, group=None):
        """Collective: exchange CUDA-IPC handles of everything not yet peer-mapped."""
        if self.world == 1:
            self.commit()
            return
        import torch.distributed as dist
        mine = {"sync": None, "tables": {}, "plans": {}}
        if not self._sync_connected:
            mine["sync"] = self._export(self.lib.exb_engine_sync_ptr(self.h))
        for t, meta in enumerate(self.tables):
            if meta["allocated"] and not meta["connected"]:
                info = self.table_info(t)
                mine["tables"][t] = (self._export(info["w_ptr"]),
                                     self._export(info["keys_ptr"]) if info["keys_ptr"] else None)
        for i, plan in enumerate(self.plans):
            if not plan.connected:
                mine["plans"][i] = self._export(plan.inbox_info()[0])
        gathered = [None] * self.world
        dist.all_gather_object(gathered, mine, group=group)
        for r, theirs in enumerate(gathered):
            if r == self.rank:
                continue
            if theirs["sync"] is not None:
                self.lib.exb_engine_set_peer_sync(self.h, r, self._open(theirs["sync"]))
            for t, (wh, kh) in theirs["tables"].items():
                self.lib.exb_table_set_peer(self.h, t, r, self._open(wh), self._open(kh) if kh else 0)
            for i, ih in theirs["plans"].items():
                self.lib.exb_plan_set_peer_inbox(self.plans[i].h, r, self._open(ih))
        self._sync_connected = True
        for meta in self.tables:
            if meta["allocated"]:
                meta["connected"] = True
        self.commit()
        for plan in self.plans:
            if not plan.connected:
                _native.cuda_check(self.lib.exb_plan_commit(plan.h), "plan_commit")
                plan.connected = True
        torch.cuda.synchronize(self.device)
        dist.barrier(group=group)
        # every rank has mapped every slab and announced its context version: these are the versions the kernels
        # will insist on (ctx_check) until the next connect
        _native.cuda_check(self.lib.exb_engine_accept_ctx(self.h), "accept_ctx")

    @staticmethod
    def connect_local(engines):
        """Wire several engines living in ONE process on ONE device as virtual ranks
        (test harness for the multi-rank protocol without multiple GPUs)."""
        W = len(engines)
        for e in engines:
            assert e.world == W
        for a in engines:
            for b in engines:
                if a is b:
                    continue
                a.lib.exb_engine_set_peer_sync(a.h, b.rank, b.lib.exb_engine_sync_ptr(b.h))
                for t in range(len(a.tables)):
                    info = b.table_info(t)
                    a.lib.exb_table_set_peer(a.h, t, b.rank, info["w_ptr"], info["keys_ptr"])
                for i, plan in enumerate(a.plans):
                    a.lib.exb_plan_set_peer_inbox(plan.h, b.rank, b.plans[i].inbox_info()[0])
        for e in engines:
            e._sync_connected = True
            for meta in e.tables:
                meta["connected"] = True
            e.commit()
            for plan in e.plans:
                _native.cuda_check(e.lib.exb_plan_commit(plan.h), "plan_commit")
                plan.connected = True
        for e in engines:
            _native.cuda_check(e.lib.exb_engine_accept_ctx(e.h), "accept_ctx")

    # ---------------------------------------------------------------- plans
    def make_plan(self, feat_tables, batch, feat_offsets=None, io_stride=None, feat_cols=None, ncols=None,
                  feat_offsets2=None, feat_split=None):
        return SparsePlan(self, feat_tables, batch, feat_offsets, io_stride, feat_cols, ncols, feat_offsets2, feat_split)

    # --------------------------------------------------------------- memory accounting
    def memory_info(self):
        """Bytes of device memory held by this rank's engine (reference: pico_memory accounting + the MEMORY_INFO
        request, pico-ps service/Service.cpp:511-518)."""
        tables = []
        for t, meta in enumerate(self.tables):
            if not meta["allocated"]:
                tables.append({"table": t, "allocated": False, "bytes": 0})
                continue
            info = self.table_info(t)
            state = int(info["rows"]) * int(info["sstride"]) * 4
            touched = 0 if meta["is_hash"] else (int(info["rows"]) + 31) // 32 * 4
            tables.append({"table": t, "allocated": True, "rows": int(info["rows"]), "dim": meta["dim"],
                           "hash": meta["is_hash"], "weights": int(info["w_bytes"]), "keys": int(info["keys_bytes"]),
                           "state": state, "bytes": int(info["w_bytes"]) + int(info["keys_bytes"]) + state + touched})
        plans = []
        for p in self.plans:
            if p.h:
                inbox, work = p.memory()
                plans.append({"features": p.F, "batch": p.B, "inbox": inbox, "work": work, "bytes": inbox + work})
        free, total = torch.cuda.mem_get_info(self.device)
        return {"tables": tables, "plans": plans, "tables_bytes": sum(t["bytes"] for t in tables),
                "plans_bytes": sum(p["bytes"] for p in plans), "device_free": int(free), "device_total": int(total)}

    def table_bytes_estimate(self, t):
        """bytes exb_table_alloc will take for a not-yet-allocated table (rows are known at add time)"""
        info = self.table_info(t)
        rows, ws, ss = int(info["rows"]), int(info["wstride"]), int(info["sstride"])
        return rows * (ws + ss) * 4 + (rows * 8 if self.tables[t]["is_hash"] else (rows + 31) // 32 * 4)

    # --------------------------------------------------------------- status
    def status(self):
        st = ctypes.c_int32(0)
        stats = _u64arr(32)
        _native.cuda_check(self.lib.exb_engine_status(self.h, ctypes.byref(st), stats), "status")
        v2 = int(stats[7]) == 2          # which push kernel stamped the phase clock last
        nst = 8 if v2 else 7
        t = [int(stats[8 + i]) for i in range(nst)]
        names = (["reduce", "dispatch", "barrier_publish", "combine", "barrier_acc", "apply", "barrier_done"] if v2
                 else ["dispatch", "barrier_publish", "combine", "barrier_acc", "apply", "barrier_done"])
        phases = {}
        if t[0] and t[nst - 1] >= t[0]:
            prev = t[0]
            for i, nm in enumerate(names):
                cur = t[i + 1] if t[i + 1] >= prev else prev     # phases skipped at world==1 keep the clock
                phases[nm] = (cur - prev) / 1e3
                prev = cur
            phases["total"] = (t[nst - 1] - t[0]) / 1e3
        return int(st.value), {"pull_indices": int(stats[0]), "push_indices": int(stats[1]),
                               "update_unique": int(stats[2]), "plans": int(stats[3]), "pull_unique": int(stats[4]),
                               "nvlink_rows_pulled": int(stats[5]), "nvlink_rows_pushed": int(stats[6]),
                               "last_push_update_us": phases,
                               "probe": [int(stats[i]) for i in range(16, 28)]}

    def _raise(self, code):
        self.lib.exb_engine_reset_status(self.h)
        raise StatusError(ENGINE_STATUS.get(code, Status.ERROR),
                          "sparse engine error %d: %s" % (code, _STATUS_TEXT.get(code, "?")))

    def check(self):
        """Blocking (device sync): raise ``StatusError`` if any kernel since the last check left an error
        code (hash shard full, inbox / combine-map overflow, barrier timeout)."""
        code, _ = self.status()
        if code != 0:
            self._raise(code)

    def poll(self):
        """Non-blocking status check for the per-step product path: consumes the previous asynchronous
        read-back of the device error word (raises ``StatusError`` if it was non-zero) and enqueues the next
        one on a side stream -- an error surfaces at most two polls after the kernel that hit it, without a
        device synchronisation on the training stream."""
        if self._st_pending and self._st_ev.query():
            self._st_pending = False
            code = int(self._st_host[0])
            if code != 0:
                self._raise(code)
        if not self._st_pending:
            if self._st_dev is None:
                from .p2p_allreduce import tensor_from_ptr
                self._st_dev = tensor_from_ptr(self.lib.exb_engine_status_ptr(self.h), 1, self.device,
                                               dtype=torch.int32)
            with torch.cuda.stream(self._st_stream):
                self._st_host.copy_(self._st_dev, non_blocking=True)
                self._st_ev.record(self._st_stream)
            self._st_pending = True

    # ---------------------------------------------- checkpoint-side row access
    def enumerate_ids(self, t):
        """Global ids of all materialised local rows, sorted (device tensor, int64)."""
        info = self.table_info(t)
        cap = int(info["rows"])
        out = torch.empty(max(cap, 1), dtype=torch.int64, device=self.device)
        n = _u64arr(1)
        s = torch.cuda.current_stream(self.device).cuda_stream
        _native.cuda_check(self.lib.exb_table_enumerate(self.h, t, out.data_ptr(), cap, n, s), "enumerate")
        return torch.sort(out[: int(n[0])])[0]

    def gather_rows(self, t, ids, with_state=True):
        info = self.table_info(t)
        dim = self.tables[t]["dim"]
        ids = ids.to(device=self.device, dtype=torch.int64).contiguous()
        n = ids.numel()
        w = torch.empty((n, dim), dtype=torch.float32, device=self.device)
        sd = int(info["state_dim"])
        s = torch.empty((n, sd), dtype=torch.float32, device=self.device) if with_state else None
        st = torch.cuda.current_stream(self.device).cuda_stream
        _native.cuda_check(self.lib.exb_table_gather(self.h, t, ids.data_ptr(), n, w.data_ptr(),
                                                     s.data_ptr() if (with_state and sd) else 0, st), "gather")
        return w, s

    def scatter_rows(self, t, ids, weights, states=None):
        ids = ids.to(device=self.device, dtype=torch.int64).contiguous()
        w = weights.to(device=self.device, dtype=torch.float32).contiguous()
        s = states.to(device=self.device, dtype=torch.float32).contiguous() if states is not None and states.numel() else None
        st = torch.cuda.current_stream(self.device).cuda_stream
        _native.cuda_check(self.lib.exb_table_scatter(self.h, t, ids.data_ptr(), ids.numel(), w.data_ptr(),
                                                      s.data_ptr() if s is not None else 0, st), "scatter")
        torch.cuda.current_stream(self.device).synchronize()

    def clear_table(self, t):
        _native.cuda_check(self.lib.exb_table_clear(self.h, t), "clear")

    def rehash(self, t, new_capacity):
        _native.cuda_check(self.lib.exb_table_rehash(self.h, t, int(new_capacity)), "rehash")
        self.tables[t]["connected"] = self.world == 1

    def close(self):
        if getattr(self, "h", None):
            for p in self.plans:
                p.close()
            for ptr in self._peer_open:
                self.lib.exb_ipc_close_handle(ptr)
            self._peer_open = []
            self.lib.exb_engine_destroy(self.h)
            self.h = None


class SparsePlan:
    """Fused lookup/update over F features of one batch (ids ``[B, F]`` int64)."""

    def __init__(self, engine, feat_tables, batch, feat_offsets=None, io_stride=None, feat_cols=None, ncols=None,
                 feat_offsets2=None, feat_split=None):
        """``feat_split`` / ``feat_offsets2``: SPLIT-ROW features -- columns ``[0, split)`` of a feature's table row are
        read / written at ``feat_offsets[f]`` of the activation row and columns ``[split, dim)`` at
        ``feat_offsets2[f]`` (one table row, e.g. [embedding | linear weight], feeding two places of the model)."""
        self.e = engine
        self.lib = engine.lib
        self.F = len(feat_tables)
        self.B = int(batch)
        self.feat_tables = [int(t) for t in feat_tables]
        widths = [int(engine.table_info(t)["wstride"]) for t in self.feat_tables]
        self.dims = [engine.tables[t]["dim"] for t in self.feat_tables]
        if feat_offsets is None:
            feat_offsets, o = [], 0
            for w in widths:
                o = (o + 3) // 4 * 4 if w % 4 == 0 else o
                feat_offsets.append(o)
                o += w
            total = (o + 3) // 4 * 4
        elif feat_split is not None:
            total = max([o + min(w, sp) for o, w, sp in zip(feat_offsets, widths, feat_split)] +
                        [o2 + d - sp for o2, d, sp in zip(feat_offsets2, self.dims, feat_split) if sp < d])
        else:
            total = max(o + w for o, w in zip(feat_offsets, widths))
        self.feat_offsets = [int(o) for o in feat_offsets]
        self.io_stride = int(io_stride) if io_stride is not None else total
        self.feat_cols = [int(c) for c in (feat_cols if feat_cols is not None else range(self.F))]
        self.ncols = int(ncols) if ncols else max(self.feat_cols) + 1
        ft = (ctypes.c_int32 * self.F)(*self.feat_tables)
        fo = (ctypes.c_int32 * self.F)(*self.feat_offsets)
        fc = (ctypes.c_int32 * self.F)(*self.feat_cols)
        self.feat_split = [int(x) for x in feat_split] if feat_split is not None else None
        self.feat_offsets2 = [int(x) for x in feat_offsets2] if feat_offsets2 is not None else None
        if self.feat_split is not None:
            fo2 = (ctypes.c_int32 * self.F)(*self.feat_offsets2)
            fsp = (ctypes.c_int32 * self.F)(*self.feat_split)
            self.h = self.lib.exb_plan_create2(engine.h, self.F, ft, fo, fc, self.ncols, self.B, self.io_stride, fo2, fsp)
        else:
            self.h = self.lib.exb_plan_create(engine.h, self.F, ft, fo, fc, self.ncols, self.B, self.io_stride)
        if not self.h:
            raise RuntimeError("exb_plan_create: " + self.lib.exb_cuda_last_error().decode())
        self.connected = engine.world == 1
        # v2 ("plan once per step", csrc/cuda/sparse_v2.cuh): ids are de-duplicated once per batch into one of two
        # batch slots; pull moves unique remote rows, push moves pre-reduced rows. EXB_SPARSE_V2=0: v1 kernels.
        # default: v2 on one GPU, v1 with more (the extra phases of the pre-reduced push cost more than the halved
        # NVLink rows buy)
        env = os.environ.get("EXB_SPARSE_V2")
        self.v2 = (env != "0") if env is not None else (engine.world == 1)
        # EXB_PULL2=1: training pulls of world > 1 move UNIQUE remote rows (exb_pull2_kernel: gather unique rows,
        # grid barrier, expand). It adds dependent phases, and on several GPUs the step is bound by the number of
        # dependent phases rather than by NVLink bytes, hence off by default.
        self.pull2 = os.environ.get("EXB_PULL2", "0") == "1" and self.feat_split is None
        self._armed = [None, None]       # relative slots (0 current, 1 next): ((ids ptr, n), origin) or None
        engine.plans.append(self)
        if engine.world == 1:
            engine.commit()
            _native.cuda_check(self.lib.exb_plan_commit(self.h), "plan_commit")

    def inbox_info(self):
        out = _u64arr(2)
        self.lib.exb_plan_inbox_info(self.h, out)
        return int(out[0]), int(out[1])

    def _stream(self):
        return torch.cuda.current_stream(self.e.device).cuda_stream

    # ---- v2 slot bookkeeping (mirrors the device-side parity word: push_update flips current <-> next)
    @staticmethod
    def _key(ids):
        return (ids.data_ptr(), ids.shape[0])

    def reset_slot(self, which=0):
        """drop a prepared batch that will not be pushed"""
        _native.cuda_check(self.lib.exb_plan_reset(self.h, which, self._stream()), "plan_reset")
        self._armed[which] = None

    def prepare(self, ids, next=False, stream=None):
        """De-duplicate the ids of a batch into a batch slot (ids only, no table access).

        ``next=True`` is the PREFETCH of the reference (``pulling`` / PrefetchPullWeights): the plan of batch
        k+1 is built -- typically on a side stream -- while batch k trains; after the ``push_update`` of batch k
        that slot becomes the current one and ``pull(train=True)`` / ``push_update`` of batch k+1 find their plan
        ready. The ids tensor must stay unchanged until that push."""
        assert ids.is_cuda and ids.dtype == torch.int64 and ids.is_contiguous() and ids.shape[1] == self.ncols
        which = 1 if next else 0
        if self._armed[which] is not None:
            self.reset_slot(which)
        st = stream if stream is not None else self._stream()
        _native.cuda_check(self.lib.exb_plan_prepare(self.h, ids.data_ptr(), ids.shape[0], which, st), "plan_prepare")
        self._armed[which] = (self._key(ids), "prefetch" if next else "pull")

    def _ensure(self, ids, for_push):
        a = self._armed[0]
        if a is not None and a[0] == self._key(ids) and (for_push or a[1] == "prefetch"):
            return
        self.prepare(ids, next=False)

    def pull(self, ids, out=None, train=False):
        """ids [n, ncols] int64 (cuda, contiguous) -> out [n, io_stride] fp32.

        ``train=True`` announces that ``push_update`` of the same ids follows: the batch is planned (or its
        prefetched plan is used) and, with world > 1, only UNIQUE remote rows cross NVLink. ``train=False``
        is the stateless read (evaluation, export, serving)."""
        assert ids.is_cuda and ids.dtype == torch.int64 and ids.is_contiguous() and ids.shape[1] == self.ncols
        n = ids.shape[0]
        if out is None:
            out = torch.empty((n, self.io_stride), dtype=torch.float32, device=ids.device)
        if self.v2 and train:
            if self.pull2 and self.e.world > 1:
                self._ensure(ids, for_push=False)
                _native.cuda_check(self.lib.exb_pull2(self.h, ids.data_ptr(), out.data_ptr(), n, 0, self._stream()), "pull2")
                return out
            a = self._armed[0]
            if not (a is not None and a[0] == self._key(ids) and a[1] == "prefetch"):
                # one launch: gather (6 warps per CTA) + de-duplication plan of the batch (2 warps per CTA)
                if a is not None:
                    self.reset_slot(0)
                _native.cuda_check(self.lib.exb_pull_plan(self.h, ids.data_ptr(), out.data_ptr(), n, 0, self._stream()),
                                   "pull_plan")
                self._armed[0] = (self._key(ids), "pull")
                return out
            # the plan was prefetched: plain gather
        _native.cuda_check(self.lib.exb_pull(self.h, ids.data_ptr(), out.data_ptr(), n, self._stream()), "pull")
        return out

    def set_dense_reduce(self, bufs, n):
        """attach (n > 0) / detach (n == 0) a dense-gradient all-reduce to this plan's push kernels: `bufs` are every
        rank's peer-mapped flat fp32 gradient buffers (P2PAllReduce.bufs). Collective: every rank, same n."""
        _native.cuda_check(self.lib.exb_plan_set_dense_reduce(self.h, bufs, int(n)), "set_dense_reduce")

    def push_update(self, ids, grads):
        assert ids.is_cuda and ids.dtype == torch.int64 and ids.is_contiguous()
        assert grads.dtype == torch.float32 and grads.is_contiguous() and grads.shape[1] == self.io_stride
        if not self.v2:
            _native.cuda_check(self.lib.exb_push_update(self.h, ids.data_ptr(), grads.data_ptr(), ids.shape[0],
                                                        self._stream()), "push_update")
            return
        self._ensure(ids, for_push=True)
        _native.cuda_check(self.lib.exb_push2(self.h, grads.data_ptr(), ids.shape[0], 0, self._stream()), "push2")
        self._armed = [self._armed[1], None]          # the kernel flipped the parity word

    def memory(self):
        """bytes of device memory held by the plan: (peer-visible inbox, local work area of both slots)"""
        out = _u64arr(2)
        self.lib.exb_plan_memory(self.h, out)
        return int(out[0]), int(out[1])

    def grid(self):
        return self.lib.exb_plan_grid(self.h, 0), self.lib.exb_plan_grid(self.h, 1)

    TRACE_SLOTS = 32

    def enable_trace(self, on=True):
        """per-warp %globaltimer trace of the apply phase of push_update (tools/sparse_probe.py);
        returns the int64 tensor [warps, TRACE_SLOTS]: slot 0 = phase start, then per task
        8 slots: task id, t_count, t_ulist, t_cmap, t_resolved, t_gathered, t_done, -."""
        if not on:
            self.lib.exb_plan_set_trace(self.h, 0)
            self._trace = None
            return None
        warps = self.grid()[1] * 8
        self._trace = torch.zeros((warps, self.TRACE_SLOTS), dtype=torch.int64, device=self.e.device)
        self.lib.exb_plan_set_trace(self.h, self._trace.data_ptr())
        return self._trace

    def feature_slices(self):
        if self.feat_split is not None:
            return [slice(o, o + min(d, sp)) for o, d, sp in zip(self.feat_offsets, self.dims, self.feat_split)]
        return [slice(o, o + d) for o, d in zip(self.feat_offsets, self.dims)]

    def close(self):
        if self.h:
            self.lib.exb_plan_destroy(self.h)
            self.h = None
