"""openembedding_b200 -- a Hopper-native (H100, sm_90a) sparse-embedding training/serving engine.

Same capabilities and Python surface as 4paradigm/OpenEmbedding (``Embedding``,
``Variable`` a.k.a. ``distributed_variable``, ``distributed_model``,
``distributed_optimizer``, server-model save/load, standalone export, ``flags``,
``Master``/``Server``), rebuilt for one NVSwitch box of H100s on PyTorch: tables are
row-sharded over the GPUs' HBM and pull / push+update are fused sm_90a kernels that
talk to peer memory directly (see ``DESIGN.md``).

Reference package root: openembedding/__init__.py:33-76.
"""
__version__ = "0.1.0"


class Flags:
    """Process-wide knobs (reference: openembedding/__init__.py:33-40)."""

    def __init__(self):
        self.config = ""            # YAML/JSON EnvConfig string
        self.master_endpoint = ""   # host:port of the control-plane master ("" -> in-process)
        self.bind_ip = ""
        self.num_workers = 1
        self.wait_num_servers = -1  # -1: every worker hosts its shards in-process (the only GPU mode)
        # additions of this engine
        self.device = "auto"        # auto | cuda | cpu
        self.seed = 0               # Philox seed of the server-side initializers


flags = Flags()

from .master import Master, Server  # noqa: E402,F401


def __getattr__(name):
    # lazy: the torch-facing API pulls in torch
    if name in ("Embedding", "Variable", "distributed_variable", "distributed_model", "distributed_optimizer",
                "Model", "save_server_model", "load_server_model", "save_as_original_model", "pulling",
                "Adadelta", "Adagrad", "Adam", "Adamax", "Ftrl", "Nadam", "RMSprop", "SGD",
                "should_persist_server_model", "persist_server_model", "restore_server_model"):
        from . import api
        return getattr(api, name)
    raise AttributeError(name)
