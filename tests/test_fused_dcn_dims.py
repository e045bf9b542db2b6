"""Column layout of the fused DCN-v2 cross network (models/fused_dense.py: cross_cols); no GPU needed."""
from openembedding_b200.models.fused_dense import _r, cross_cols


def test_cross_cols_skip_the_embedding_pad_columns():
    # dim 9 is stored as Dp = 12 columns per field: columns 9..11 of every field are not cross input
    cols = cross_cols(3, 9, 12, 2)
    assert cols == list(range(0, 9)) + list(range(12, 21)) + list(range(24, 33)) + [36, 37]


def test_cross_cols_benchmark_layouts():
    for D, Dp, K0p in ((64, 64, 1728), (9, 12, 384)):
        cols = cross_cols(26, D, Dp, 13)
        assert len(cols) == 26 * D + 13 and len(set(cols)) == len(cols)
        assert cols == sorted(cols) and cols[-1] == 26 * Dp + 12
        assert _r(26 * Dp + 13 + 1, 64) == K0p and cols[-1] < K0p - 1     # the ones column stays outside


def test_cross_cols_without_dense_features():
    assert cross_cols(2, 4, 4, 0) == list(range(8))
