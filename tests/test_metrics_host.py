"""Host half of models/metrics.py (no GPU): the Keras threshold table and the AUC finalisation from bucket counts."""
import numpy as np
import pytest

from openembedding_b200.models import metrics as M


def _keras_table(T):
    """tf.keras.metrics.AUC's construction (metrics_utils / AUC.__init__), then the float32 cast of the tensor"""
    eps = 1e-7
    thresholds = [(i + 1) * 1.0 / (T - 1) for i in range(T - 2)]
    return np.array([0.0 - eps] + thresholds + [1.0 + eps]).astype(np.float32)


@pytest.mark.parametrize("T", [2, 3, 200, 8192])
def test_threshold_table_is_keras(T):
    t = M.keras_thresholds(T)
    assert t.dtype == np.float32 and t.shape == (T,)
    assert np.array_equal(t.view(np.int32), _keras_table(T).view(np.int32))
    assert np.all(np.diff(t.astype(np.float64)) > 0)
    assert t[0] < 0 and t[-1] > 1


def _counts(probs, labels, T):
    """bucket counts the kernel produces: bucket = #{i : t_i < p}, positive iff label != 0"""
    t = M.keras_thresholds(T)
    k = (t[None, :] < np.asarray(probs, dtype=np.float32)[:, None]).sum(1)
    pos = np.bincount(k[np.asarray(labels) != 0], minlength=T + 1)
    neg = np.bincount(k[np.asarray(labels) == 0], minlength=T + 1)
    return pos, neg


def test_confusion_matches_direct_comparison():
    rng = np.random.default_rng(0)
    T = 50
    p = rng.random(1000).astype(np.float32)
    y = (rng.random(1000) < 0.3).astype(np.float32)
    tp, fp, tn, fn = M.confusion(*_counts(p, y, T))
    t = M.keras_thresholds(T)
    pred = p[:, None] > t[None, :]
    assert np.array_equal(tp, (pred & (y[:, None] != 0)).sum(0))
    assert np.array_equal(fp, (pred & (y[:, None] == 0)).sum(0))
    assert np.array_equal(tn, (~pred & (y[:, None] == 0)).sum(0))
    assert np.array_equal(fn, (~pred & (y[:, None] != 0)).sum(0))


def test_auc_hand_made_counts():
    T = 200
    # perfect ranking (every positive above every negative) and its inverse
    pos, neg = _counts([0.9, 0.8, 0.1, 0.2], [1, 1, 0, 0], T)
    assert M.auc_from_counts(pos, neg) == pytest.approx(1.0, abs=1e-12)
    pos, neg = _counts([0.1, 0.2, 0.9, 0.8], [1, 1, 0, 0], T)
    assert M.auc_from_counts(pos, neg) == pytest.approx(0.0, abs=1e-12)
    # one class only: 0, as Keras' divide_no_nan gives
    assert M.auc_from_counts(*_counts([0.9, 0.8, 0.95], [1, 1, 1], T)) == 0.0
    assert M.auc_from_counts(*_counts([0.1, 0.2], [0, 0], T)) == 0.0
    # all in one bucket: the ROC is the diagonal
    pos, neg = _counts([0.5, 0.5, 0.5, 0.5], [1, 0, 1, 0], T)
    assert M.auc_from_counts(pos, neg) == pytest.approx(0.5, abs=1e-12)


def test_auc_formula_in_fp64():
    rng = np.random.default_rng(1)
    T = 17
    pos, neg = rng.integers(0, 50, T + 1), rng.integers(0, 50, T + 1)
    tp, fp, tn, fn = (x.astype(np.float64) for x in M.confusion(pos, neg))
    tpr, fpr = tp / (tp + fn), fp / (fp + tn)
    ref = sum((fpr[i] - fpr[i + 1]) * (tpr[i] + tpr[i + 1]) / 2 for i in range(T - 1))
    assert M.auc_from_counts(pos, neg) == pytest.approx(ref, rel=1e-14)


@pytest.mark.parametrize("T", [0, 1, 8193, 2.5, True])
def test_threshold_count_is_checked(T):
    with pytest.raises(ValueError):
        M.keras_thresholds(T)
