"""Optimizer / initializer / environment configuration.

Mirrors the reference's three config tiers (SURVEY 5.6):

1. ``flags`` (python object)                    openembedding/__init__.py:33-40
2. ``EnvConfig`` (YAML/JSON string in flags.config)  openembedding/client/EnvConfig.h:14-84
3. per-object ``str -> str`` property bags for optimizer/initializer
   (openembedding/entry/c_api.cc:273-293 -> Factory.h CONFIGURE_PROPERTY), serialised as
   YAML inside checkpoints (EmbeddingOptimizerVariable.h:93-107).
"""
import copy
import json

import yaml

# ---- optimizer categories: name -> (kind, [(property, default), ...] in p[] order)
# defaults: openembedding/variable/EmbeddingOptimizer.h CONFIGURE_PROPERTY lines
OPTIMIZERS = {
    "default": (0, [("learning_rate", 0.0)]),
    "adadelta": (1, [("learning_rate", 0.001), ("rho", 0.95), ("epsilon", 1e-7)]),
    "adagrad": (2, [("learning_rate", 0.001), ("initial_accumulator_value", 0.1), ("epsilon", 1e-7)]),
    "adam": (3, [("learning_rate", 0.001), ("beta_1", 0.9), ("beta_2", 0.999), ("epsilon", 1e-7)]),
    "adamax": (4, [("learning_rate", 0.001), ("beta_1", 0.9), ("beta_2", 0.999), ("epsilon", 1e-7)]),
    "ftrl": (5, [("learning_rate", 0.001), ("initial_accumulator_value", 0.1),
                 ("l1_regularization_strength", 0.0), ("l2_regularization_strength", 0.0),
                 ("l2_shrinkage_regularization_strength", 0.0), ("learning_rate_power", -0.5),
                 ("beta", 0.0)]),
    "rmsprop": (6, [("learning_rate", 0.001), ("rho", 0.9), ("momentum", 0.0), ("epsilon", 1e-7)]),
    "sgd": (7, [("learning_rate", 0.01), ("momentum", 0.0), ("nesterov", False)]),
    "test": (8, [("learning_rate", 0.1), ("flip", 10000.0), ("init", 0.0)]),
}
OPT_KIND_TO_NAME = {v[0]: k for k, v in OPTIMIZERS.items()}

INITIALIZERS = {
    "constant": (0, [("value", 0.0)]),
    "uniform": (1, [("minval", 0.0), ("maxval", 1.0)]),
    "normal": (2, [("mean", 0.0), ("stddev", 1.0), ("truncated", 0.0)]),
}

DTYPES = {"float32": 0x104, "float64": 0x108, "int8": 0x1, "int16": 0x2, "int32": 0x4, "int64": 0x8}
DTYPE_NAMES = {v: k for k, v in DTYPES.items()}


class DataType:
    """dtype tag of a table (reference: openembedding/variable/DataType.h:20-134: the low byte of
    the tag is the element size; only float32/float64 are registered for tables,
    EmbeddingVariable.cpp:277-278). ``DataType("float32").size == 4``; ``int(dt)`` is the tag
    stored in shard-file headers."""

    def __init__(self, v):
        if isinstance(v, DataType):
            v = v.name
        if isinstance(v, int):
            if v not in DTYPE_NAMES:
                raise ValueError("unknown datatype tag: %r" % v)
            v = DTYPE_NAMES[v]
        v = str(v).replace("torch.", "")
        if v not in DTYPES:
            raise ValueError("unknown datatype: %r" % v)
        self.name, self.tag = v, DTYPES[v]

    @property
    def size(self):
        return self.tag & 0xFF

    @property
    def is_table_type(self):
        return self.name in ("float32", "float64")

    def __int__(self):
        return self.tag

    def __str__(self):
        return self.name

    def __eq__(self, o):
        try:
            return self.tag == DataType(o).tag
        except ValueError:
            return False

    def __hash__(self):
        return hash(self.tag)
HASH_KEY_RANGE = 2 ** 63


def _to_float(v):
    if isinstance(v, bool):
        return 1.0 if v else 0.0
    if isinstance(v, str):
        s = v.strip().lower()
        if s in ("true", "yes"):
            return 1.0
        if s in ("false", "no"):
            return 0.0
        return float(s)
    return float(v)


def str_dict(config):
    return {str(k): str(v) for k, v in config.items()}


def normalize_optimizer(config):
    """dict(category=..., prop=...) of anything -> canonical dict with every property set."""
    config = dict(config)
    category = str(config.pop("category", "default")).lower()
    if category not in OPTIMIZERS:
        # Nadam & friends are wrapped by the reference's python but have no server
        # implementation (EmbeddingOptimizer.h:393-395 TODO) -> factory failure there too.
        raise ValueError("unsupported server optimizer category: %r" % category)
    out = {"category": category}
    props = dict(OPTIMIZERS[category][1])
    for k, v in config.items():
        if k not in props:
            # reference warns on unknown keys (Factory.h:64-75)
            continue
        out[k] = (_to_float(v) != 0.0) if isinstance(props[k], bool) else _to_float(v)
    for k, d in props.items():
        out.setdefault(k, d)
    return out


def optimizer_params(config):
    """canonical optimizer config -> (kind, [p0..p7])"""
    c = normalize_optimizer(config)
    kind, props = OPTIMIZERS[c["category"]]
    p = [_to_float(c[name]) for name, _ in props]
    p += [0.0] * (8 - len(p))
    return kind, p


def optimizer_state_dim(config, dim):
    kind, _ = optimizer_params(config)
    slots = {0: 0, 1: 2, 2: 1, 3: 2, 4: 2, 5: 2, 6: 2, 7: 1, 8: 0}[kind]
    scalars = {3: 2, 4: 1, 8: 2}.get(kind, 0)
    return slots * dim + scalars


def OPTIMIZER_SLOTS(config):
    """(per-element state slots, trailing per-row scalars) of an optimizer -- exb_math.h opt_num_slots/scalars"""
    kind, _ = optimizer_params(config)
    return {0: 0, 1: 2, 2: 1, 3: 2, 4: 2, 5: 2, 6: 2, 7: 1, 8: 0}[kind], {3: 2, 4: 1, 8: 2}.get(kind, 0)


def optimizer_slot_inits(config):
    """initial values ([per slot], [per scalar]) of a fresh optimizer state -- exb_math.h opt_slot_init/opt_scalar_init"""
    kind, p = optimizer_params(config)
    nslots, nsc = OPTIMIZER_SLOTS(config)
    slots = [float(p[1]) if (kind in (2, 5) and s == 0) else 0.0 for s in range(nslots)]
    if kind in (3, 4):
        scal = [1.0] * nsc
    elif kind == 8:
        scal = [float(p[2]), 0.0][:nsc]
    else:
        scal = [0.0] * nsc
    return slots, scal


_INIT_ALIASES = {
    # keras string identifiers used by tf.keras.layers.Embedding (exb.py:25-63)
    "uniform": {"category": "uniform", "minval": -0.05, "maxval": 0.05},
    "random_uniform": {"category": "uniform", "minval": -0.05, "maxval": 0.05},
    "normal": {"category": "normal", "mean": 0.0, "stddev": 0.05, "truncated": 0.0},
    "random_normal": {"category": "normal", "mean": 0.0, "stddev": 0.05, "truncated": 0.0},
    "zeros": {"category": "constant", "value": 0.0},
    "ones": {"category": "constant", "value": 1.0},
    "constant": {"category": "constant", "value": 0.0},
}


def normalize_initializer(init, explicit=True):
    if init is None:
        init = "uniform"
    if isinstance(init, str):
        key = init.lower()
        if key not in _INIT_ALIASES:
            if explicit:
                raise ValueError("error initializer: " + str(init))
            key = "zeros"
        config = dict(_INIT_ALIASES[key])
    elif isinstance(init, dict):
        config = dict(init)
    elif isinstance(init, (int, float)):
        config = {"category": "constant", "value": float(init)}
    else:
        if explicit:
            raise ValueError("error initializer: " + str(init))
        config = {"category": "constant", "value": 0.0}
    category = str(config.pop("category", "constant")).lower()
    if category not in INITIALIZERS:
        raise ValueError("error initializer category: " + category)
    out = {"category": category}
    props = dict(INITIALIZERS[category][1])
    seed = config.pop("seed", None)
    config.pop("dtype", None)
    for k, v in config.items():
        if k in props:
            out[k] = _to_float(v)
    for k, d in props.items():
        out.setdefault(k, d)
    if seed is not None:
        out["seed"] = int(seed)
    return out


def initializer_params(config):
    c = normalize_initializer(config)
    kind, props = INITIALIZERS[c["category"]]
    p = [_to_float(c[name]) for name, _ in props]
    p += [0.0] * (3 - len(p))
    return kind, p, int(c.get("seed", 0))


def mix_seed(seed, variable_id):
    """64-bit Philox key from (user seed, variable id) -- splitmix64."""
    x = (int(seed) * 0x9E3779B97F4A7C15 + int(variable_id) + 0x632BE59BD9B4E019) & (2 ** 64 - 1)
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & (2 ** 64 - 1)
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & (2 ** 64 - 1)
    x ^= x >> 31
    return x


# ---- YAML variable config stored in checkpoint shard headers
def dump_variable_config(table, reserve_items, optimizer, initializer, include_optimizer=True, extra=None):
    opt = normalize_optimizer(optimizer)
    ini = normalize_initializer(initializer)
    doc = {"table": table, "reserve_items": int(reserve_items)}
    oc, ic = opt.pop("category"), ini.pop("category")
    seed = ini.pop("seed", None)
    if include_optimizer:
        doc["optimizer"] = oc
    doc["initializer"] = ic
    if include_optimizer:
        doc[oc] = opt
    doc[ic] = ini
    # addition of this engine: pulls never insert, so never-updated rows are regenerated from Philox(seed, variable_id).
    # The seed therefore has to travel with the checkpoint (the reference loader only warns about unknown keys,
    # Factory.h:64-75); seed 0 (the default) is left out so that default dumps stay byte-identical.
    if seed:
        doc["initializer_seed"] = int(seed)
    if extra:
        doc.update(extra)
    return yaml.safe_dump(doc, sort_keys=False, default_flow_style=False)


def load_variable_config(text):
    doc = yaml.safe_load(text) if text else {}
    doc = doc or {}
    out = {"table": doc.get("table", "array"), "reserve_items": int(doc.get("reserve_items", 0)), "raw": doc}
    if "optimizer" in doc:
        oc = str(doc["optimizer"])
        cfg = dict(doc.get(oc) or {})
        cfg["category"] = oc
        out["optimizer"] = normalize_optimizer(cfg)
    if "initializer" in doc:
        ic = str(doc["initializer"])
        cfg = dict(doc.get(ic) or {})
        cfg["category"] = ic
        out["initializer"] = normalize_initializer(cfg)
        out["initializer"]["seed"] = int(doc.get("initializer_seed", 0))
    return out


# ---- EnvConfig (tier 2): schema + defaults + validation
_ENV_DEFAULTS = {
    "rpc": {
        "bind_ip": "", "io_thread_num": 2, "protocol": "nvlink",  # reference: tcp | rdma
        "tcp": {"keepalive_time": -1, "keepalive_intvl": -1, "keepalive_probes": -1, "connect_timeout": 3600},
        "rdma": {"ib_devname": "", "gid_index": 0, "ib_port": 1, "traffic_class": 4, "sl": 4,
                 "mtu": 1024, "pkey_index": 0, "min_rnr_timer": 12, "retry_cnt": 7, "timeout": 12},
    },
    "master": {"endpoint": "", "type": "tcp", "root_path": "/openembedding", "recv_timeout": 10000,
               "cache_timeout": 20},
    "server": {
        "pmem_pool_root_path": "", "cache_size": 1024, "message_compress": "",
        "server_dump_files": 1, "server_concurrency": -1, "recv_timeout": -1, "report_interval": -1,
        "update_early_return": True,
        # additions of this engine
        "hash_table_reserve": 1 << 20, "host_tier_root_path": "", "deterministic": False,
        # HBM accounting (reference: ShardStorageMemory soft / hard limits, pico-ps storage/Storage.h:261-289): MB of
        # device memory the sparse engine of ONE rank may hold (tables + optimizer state + plans + tier caches);
        # 0 = unlimited. Above the soft limit a warning is logged, above the hard limit allocation fails with OOM.
        "memory_soft_limit_mb": 0, "memory_hard_limit_mb": 0,
        "hash_table_grow_interval": 64, "hash_table_max_load": 0.5,
    },
}
_ENV_CHECKS = {
    ("rpc", "protocol"): lambda v: v in ("nvlink", "tcp", "rdma", "gloo"),
    ("master", "type"): lambda v: v in ("tcp", "zk", "store"),
    ("server", "message_compress"): lambda v: v in ("", "snappy", "lz4", "zlib"),
    ("server", "server_dump_files"): lambda v: int(v) >= 1,
    ("server", "cache_size"): lambda v: int(v) >= 0,
}


class EnvConfig(dict):
    """Nested dict with the reference's schema; unknown keys are rejected."""

    def __init__(self, text=None):
        super().__init__(copy.deepcopy(_ENV_DEFAULTS))
        if text:
            self.load(text)

    def load(self, text):
        if isinstance(text, str):
            text = text.strip()
            doc = json.loads(text) if text.startswith("{") else yaml.safe_load(text)
        else:
            doc = text
        self._merge(self, doc or {}, ())
        return self

    def _merge(self, dst, src, path):
        for k, v in src.items():
            if k not in dst:
                raise ValueError("unknown config key: " + ".".join(path + (k,)))
            if isinstance(dst[k], dict):
                if not isinstance(v, dict):
                    raise ValueError("config key %s must be a mapping" % ".".join(path + (k,)))
                self._merge(dst[k], v, path + (k,))
            else:
                chk = _ENV_CHECKS.get(path + (k,))
                if chk and not chk(v):
                    raise ValueError("invalid value for %s: %r" % (".".join(path + (k,)), v))
                dst[k] = type(dst[k])(v) if not isinstance(dst[k], bool) else bool(v)

    def dump_yaml(self):
        return yaml.safe_dump(dict(self), sort_keys=False)
