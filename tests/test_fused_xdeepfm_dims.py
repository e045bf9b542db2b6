"""Layer sizes and argument checks of the fused xDeepFM CIN (models/fused_dense.py: cin_dims); no GPU needed."""
import pytest

from openembedding_b200.models.fused_dense import cin_dims


def test_cin_dims_deepctr_default():
    # 26 fields, (128, 128) split_half: 64 channels handed on, 64 + 128 pooled
    H, N, Kp, Np, lo = cin_dims(26, (128, 128), True)
    assert H == [26, 64] and N == [128, 128]
    assert Kp == [704, 1728]               # round_up(H * 26 + 1, 64): the bias column needs one more
    assert Np == [128, 128] and lo == [64, 0]


def test_cin_dims_three_layers_and_no_split():
    assert cin_dims(7, (32, 16, 8), True) == ([7, 16, 8], [32, 16, 8], [64, 128, 64], [64, 64, 64], [16, 8, 0])
    assert cin_dims(5, (24,), False) == ([5], [24], [64], [64], [0])
    # without split_half every channel is pooled and handed on
    assert cin_dims(4, (20, 12), False) == ([4, 20], [20, 12], [64, 128], [64, 64], [0, 0])


@pytest.mark.parametrize("nf,layers,split", [(26, (127, 128), True), (26, (64, 31, 16), True), (26, (1024, 128), True),
                                             (26, (600, 8), False), (65, (128, 128), True), (26, (), True),
                                             (64, (402, 8), True)])
def test_cin_dims_rejects_what_the_kernels_cannot_run(nf, layers, split):
    with pytest.raises(ValueError):
        cin_dims(nf, layers, split)
