"""The grouping of mixed-size images into ragged network passes (pipeline.ragged_groups): CPU only."""
import numpy as np
import pytest

from dirb200 import pipeline


def _check(sizes, batch_size):
    groups = pipeline.ragged_groups(sizes, batch_size)
    flat = [i for g in groups for i in g]
    assert sorted(flat) == list(range(len(sizes)))                      # every image exactly once
    num, den = pipeline.RAGGED_AREA_BOUND
    for g in groups:
        assert 1 <= len(g) <= batch_size
        hh, ww = max(sizes[i][0] for i in g), max(sizes[i][1] for i in g)
        assert den * len(g) * hh * ww <= num * sum(sizes[i][0] * sizes[i][1] for i in g) or len(g) == 1
    # scattering the per-group outputs back restores dataset order
    out = [None] * len(sizes)
    for g in groups:
        for i in g:
            out[i] = sizes[i]
    assert out == list(sizes)
    return groups


@pytest.mark.parametrize("seed", range(20))
def test_random_oxford_like_mixes(seed):
    rs = np.random.RandomState(seed)
    sizes = []
    for _ in range(int(rs.randint(1, 200))):
        r = rs.rand()
        if r < 0.4:
            sizes.append((768, 1024))
        elif r < 0.7:
            sizes.append((1024, 768))
        elif r < 0.85:
            a = int(rs.randint(400, 1024))
            sizes.append((1024, a) if rs.rand() < 0.5 else (a, 1024))
        else:
            sizes.append((int(rs.randint(32, 700)), int(rs.randint(32, 700))))     # query crops
    _check(sizes, int(rs.choice([2, 4, 8, 16, 64])))


def test_one_image():
    assert _check([(333, 517)], 16) == [[0]]


def test_all_equal_sizes_fill_whole_batches():
    groups = _check([(768, 1024)] * 37, 16)
    assert [len(g) for g in groups] == [16, 16, 5]


def test_batch_size_one_is_one_image_per_pass():
    sizes = [(100, 200), (50, 60), (100, 200)]
    assert sorted(map(tuple, _check(sizes, 1))) == [(0,), (1,), (2,)]


def test_area_bound_splits_dissimilar_shapes():
    groups = _check([(1024, 768), (768, 1024)], 16)        # one slot of 1024 x 1024 would pad 33%
    assert len(groups) == 2
    assert len(_check([(1024, 768), (1000, 768)], 16)) == 1
