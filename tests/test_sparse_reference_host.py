"""The NumPy reference of the sparse engine (tests/sparse_reference.py), checked without a GPU:

  * its float32 replicas equal the CPU engine (libexb_core, float tables) bit for bit, duplicates included;
  * its float64 form equals the Keras transcription of tests/test_optimizers.py for every configuration;
  * updates are lazy: a row skipped for a step keeps its state and its own step count.
"""
import ctypes

import numpy as np
import pytest
import torch

from openembedding_b200 import _native
from openembedding_b200.config import optimizer_params
from sparse_reference import TableRef, dyadic, f32_config, hash64, valid_ids
from test_optimizers import CONFIGS, keras_reference

EXACT_CONFIGS = [
    {"category": "default", "learning_rate": 0.125},
    {"category": "sgd", "learning_rate": 0.25, "momentum": 0.0},
    {"category": "sgd", "learning_rate": 0.25, "momentum": 0.5},
    {"category": "sgd", "learning_rate": 0.25, "momentum": 0.5, "nesterov": True},
    {"category": "test", "learning_rate": 0.5, "flip": 3.0, "init": 0.75},
    {"category": "adam", "learning_rate": 0.01},          # the per-row beta powers only
    {"category": "adamax", "learning_rate": 0.01},
]


def _cfg_id(c):
    return "-".join("%s=%s" % kv for kv in c.items())


def _oracle(dim, vocab, cfg):
    lib = _native.core()
    h = lib.exb_var_create(0x104, dim, vocab, 0, 1, 0)
    kind, p = optimizer_params(cfg)
    lib.exb_var_set_optimizer(h, kind, (ctypes.c_double * 8)(*p), 8)
    return lib, h


@pytest.mark.parametrize("cfg", EXACT_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("dim", [1, 5, 64])
def test_float32_replica_equals_cpu_engine(cfg, dim):
    rng = np.random.default_rng(dim)
    vocab = 40
    lib, h = _oracle(dim, vocab, cfg)
    ref = TableRef(dim, vocab, False, cfg, exact=True)
    seeded = np.arange(0, vocab, 2, dtype=np.uint64)              # odd ids keep the (zero) initial row
    w0 = rng.standard_normal((seeded.size, dim)).astype(np.float32)
    lib.exb_var_set_weights(h, seeded.ctypes.data, seeded.size, w0.ctypes.data, None, 0)
    ref.seed(seeded, w0)
    for step in range(4):
        # duplicates within a push and across the two pushes of a step (two "ranks"); ids 30.. are skipped on odd steps
        hi = vocab if step % 2 == 0 else 30
        ids = [rng.integers(0, hi, size=97).astype(np.uint64) for _ in range(2)]
        g = [dyadic(rng, (97, dim)) for _ in range(2)]
        for i, gi in zip(ids, g):
            lib.exb_var_push(h, i.ctypes.data, i.size, gi.ctypes.data, None)
        lib.exb_var_update(h)
        ref.step(np.concatenate(ids).astype(np.int64), np.concatenate(g))
    probe = np.arange(vocab, dtype=np.uint64)
    sd = lib.exb_var_state_dim(h)
    w = np.empty((vocab, dim), dtype=np.float32)
    s = np.empty((vocab, max(sd, 1)), dtype=np.float32)
    lib.exb_var_get_weights(h, probe.ctypes.data, vocab, w.ctypes.data, s.ctypes.data)
    lib.exb_var_destroy(h)
    want_w, want_s = ref.get(probe.astype(np.int64))
    assert want_s.shape[1] == sd
    if cfg["category"] in ("adam", "adamax"):          # the replica covers the trailing scalars only
        nsc = 2 if cfg["category"] == "adam" else 1
        np.testing.assert_array_equal(s[:, sd - nsc:sd], want_s[:, sd - nsc:])
        return
    np.testing.assert_array_equal(w, want_w)
    np.testing.assert_array_equal(s[:, :sd], want_s)


@pytest.mark.parametrize("cfg", CONFIGS, ids=_cfg_id)
def test_float64_form_equals_keras(cfg):
    torch.manual_seed(1)
    c = f32_config(cfg)
    dim, steps = 6, 5
    ref = TableRef(dim, 10, False, c, exact=False)
    w0 = torch.randn(3, dim, dtype=torch.float64)
    ref.seed(np.arange(3), w0.numpy())
    grads = [torch.randn(3, dim, dtype=torch.float64) for _ in range(steps)]
    touched = {0: range(steps), 1: [0, 2, 3], 2: [4]}     # rows 1 and 2 skip steps: lazy, per-row step counts
    for t in range(steps):
        ids = np.array([r for r in range(3) if t in touched[r]], dtype=np.int64)
        ref.step(ids, grads[t].numpy()[ids])
    got, _ = ref.get(np.arange(3))
    for r in range(3):
        want = keras_reference(c, w0[r:r + 1], [grads[t][r:r + 1] for t in touched[r]])
        np.testing.assert_allclose(got[r], want.numpy()[0], rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("cat", ["adam", "adamax", "adagrad", "sgd"])
def test_lazy_rows_keep_state_and_step_count(cat):
    cfg = {"category": cat, "learning_rate": 0.05}
    ref = TableRef(3, 10, False, cfg, exact=False)
    g = np.ones((1, 3))
    ref.step(np.array([1]), g)
    w1, s1 = ref.get([1])
    ref.step(np.array([2]), g)                              # row 1 untouched
    w1b, s1b = ref.get([1])
    np.testing.assert_array_equal(w1, w1b)
    np.testing.assert_array_equal(s1, s1b)
    ref.step(np.array([1, 2]), np.ones((2, 3)))
    _, s = ref.get([1, 2])
    np.testing.assert_array_equal(s[0], s[1])                   # both at their own second step
    if cat == "adam":
        np.testing.assert_allclose(s[0, -2:], [0.9 ** 2, 0.999 ** 2], rtol=1e-7)
    # the float32 replica of the beta powers counts steps per row the same way
    if cat in ("adam", "adamax"):
        r32 = TableRef(3, 10, False, cfg, exact=True)
        r32.step(np.array([1]), g.astype(np.float32))
        r32.step(np.array([2]), g.astype(np.float32))
        r32.step(np.array([1, 2]), np.ones((2, 3), np.float32))
        _, s32 = r32.get([1, 2, 3])
        b1 = np.float32(0.9)
        np.testing.assert_array_equal(s32[0, 6], b1 * b1)
        np.testing.assert_array_equal(s32[0], s32[1])
        np.testing.assert_array_equal(s32[2, 6], np.float32(1))           # never touched: initial scalars


def test_invalid_ids_and_hash():
    ids = np.array([-1, 0, 5, 9, 10, -(2 ** 63), 2 ** 62], dtype=np.int64)
    np.testing.assert_array_equal(valid_ids(ids, 10, False), [0, 1, 1, 1, 0, 0, 0])
    np.testing.assert_array_equal(valid_ids(ids, 10, True), [0, 1, 1, 1, 1, 0, 1])
    ref = TableRef(2, 10, True, {"category": "sgd", "learning_rate": 1.0}, init_value=0.5)
    ref.step(ids, np.ones((ids.size, 2), np.float32))
    assert ref.materialized() == {0, 5, 9, 10, 2 ** 62}
    np.testing.assert_array_equal(ref.pull(ids)[0], [0, 0])
    np.testing.assert_array_equal(ref.pull(ids)[1], [-0.5, -0.5])
    lib = _native.core()
    for x in [0, 1, 7, 2 ** 40 + 3, 2 ** 63 - 1, 12345678901234]:
        assert hash64(x) == lib.exb_hash64_c(x)
