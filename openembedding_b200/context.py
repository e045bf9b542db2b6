"""Process-wide training context (one per rank).

Reference: ``_get_context()`` / ``Context`` in openembedding/tensorflow/exb.py:107-219 and
the C++ ``WorkerContext`` (openembedding/client/WorkerContext.cpp:7-163): connection to
the master, storage / variable creation broadcast to all workers, model uuid, barrier.

Design: rendezvous and object broadcast ride on ``torch.distributed`` (NCCL group
for GPUs, gloo for the CPU configuration); the data plane is ``backend.CudaBackend``.
"""
import atexit
import os
import uuid

import torch

from . import flags
from .backend import CpuBackend, CudaBackend, VarMeta
from .config import HASH_KEY_RANGE, EnvConfig, normalize_initializer, normalize_optimizer

_context = None


class Storage:
    def __init__(self, storage_id, shard_num, shard_base):
        self.storage_id, self.shard_num, self.shard_base = storage_id, shard_num, shard_base
        self.variables = []


class Context:
    def __init__(self):
        import torch.distributed as dist
        self.dist_on = dist.is_available() and dist.is_initialized()
        self.rank = dist.get_rank() if self.dist_on else 0
        self.world = dist.get_world_size() if self.dist_on else 1
        if flags.num_workers < 1:
            raise ValueError("error num_workers")
        if flags.wait_num_servers < -1:
            raise ValueError("error wait_num_servers")
        flags.num_workers = self.world
        self.env = EnvConfig(flags.config)
        want = flags.device
        use_cuda = torch.cuda.is_available() if want == "auto" else (want == "cuda")
        if use_cuda and not torch.cuda.is_available():
            raise RuntimeError("flags.device='cuda' but no CUDA device is visible")
        self.group = None
        if use_cuda:
            local_rank = int(os.environ.get("LOCAL_RANK", self.rank % max(1, torch.cuda.device_count())))
            self.backend = CudaBackend(self.rank, self.world, local_rank, group=None)
            self.backend.hash_reserve = int(self.env["server"]["hash_table_reserve"])
            self.backend.grow_interval = int(self.env["server"]["hash_table_grow_interval"])
            self.backend.max_load = float(self.env["server"]["hash_table_max_load"])
            self.backend.soft_limit_mb = int(self.env["server"]["memory_soft_limit_mb"])
            self.backend.hard_limit_mb = int(self.env["server"]["memory_hard_limit_mb"])
        else:
            if self.dist_on and dist.get_backend() != "gloo":
                self.group = dist.new_group(backend="gloo")
            self.backend = CpuBackend(self.rank, self.world, group=self.group)
        self.device = self.backend.device
        self.model_uuid = self.sync_bcast(lambda: str(uuid.uuid1()))
        self.model_version = 0.1     # floor() gives the number of applied steps (exb.py:213-218)
        self.storages = []
        self.variables = []          # VarMeta by variable_id
        self.tracks = {}             # id(graph_var) -> api.Variable
        # server.report_interval > 0: timers/counters on, rank 0 prints the table periodically
        # (reference: WorkerContext.cpp:24-41, 140-163)
        self.monitor = None
        interval = float(self.env["server"]["report_interval"])
        if interval > 0:
            from .utils import timers
            self.monitor = timers.Monitor(self, interval).start()
        atexit.register(self.finalize)

    # ---- control plane (reference: client/Communication.h:12-73)
    def barrier(self):
        if self.dist_on:
            import torch.distributed as dist
            dist.barrier(group=self.group)

    def sync_bcast(self, fn):
        """Run fn on exactly one rank and broadcast its result."""
        if not self.dist_on:
            return fn()
        import torch.distributed as dist
        obj = [fn() if self.rank == 0 else None]
        dist.broadcast_object_list(obj, src=0, group=self.group)
        return obj[0]

    # ---- storages / variables
    def create_storage(self, num_shards=None):
        sid = len(self.storages)
        if not num_shards or num_shards < 0 or num_shards > self.world:
            shard_num = self.world        # one shard per rank; more shards than ranks is an internal detail
        else:
            shard_num = int(num_shards)
        st = Storage(sid, shard_num, sid % self.world)   # round-robin placement (WorkerContext.cpp:66-85)
        self.storages.append(st)
        return st

    def create_variable(self, storage, vocabulary_size, embedding_dim, dtype="float32", force_hash=False,
                        capacity=None):
        is_hash = vocabulary_size >= HASH_KEY_RANGE or force_hash
        meta = VarMeta(len(self.variables), storage.storage_id, int(vocabulary_size), int(embedding_dim),
                       dtype, is_hash, storage.shard_num, storage.shard_base)
        meta.capacity = capacity
        self.backend.create_variable(meta)
        self.backend.set_initializer(meta, meta.initializer)
        storage.variables.append(meta)
        self.variables.append(meta)
        return meta

    def set_initializer(self, meta, config):
        meta.initializer = normalize_initializer(config)
        if "seed" not in meta.initializer:
            meta.initializer["seed"] = int(flags.seed)
        self.backend.set_initializer(meta, meta.initializer)

    def set_optimizer(self, meta, config):
        meta.optimizer = normalize_optimizer(config)
        self.backend.set_optimizer(meta, meta.optimizer)

    def step_done(self, n=1):
        """once per training step: advances the model version and lets the backend do its periodic
        maintenance (hash shards above the load factor are grown, collectively)"""
        self.model_version += n
        tick = getattr(self.backend, "tick", None)
        if tick is not None:
            tick(n)

    def memory_info(self):
        """device / pinned-host memory held by the sparse engine of this rank (tables, plans, host tiers)"""
        fn = getattr(self.backend, "memory_info", None)
        return fn() if fn is not None else {}

    def model_sign(self):
        return "%s-%d" % (self.model_uuid, int(self.model_version))

    def finalize(self):
        global _context
        if getattr(self, "monitor", None) is not None:
            self.monitor.stop()
            self.monitor = None
        if getattr(self, "backend", None) is not None:
            try:
                from . import host_tier
                host_tier.close_all()          # tiers hold engine handles: before the backend goes away
            except Exception:
                pass
            try:
                self.backend.close()
            except Exception:
                pass
            self.backend = None
        if _context is self:
            _context = None


def get_context():
    global _context
    if _context is None:
        _context = Context()
    return _context


def reset_context():
    """Drop the process context (tests)."""
    global _context
    if _context is not None:
        _context.finalize()
    _context = None
