"""CPU checks of the brute-force distCUDA2 oracle (oracle/knn_oracle.c) that tests/test_gpu_knn.py compares against."""
import numpy as np
import pytest

from oracle.knn_oracle import knn_mean_dist3
from tests.knn_clouds import SHAPES, cloud, mean_dist3_float64

FLT_MAX = np.float32(np.finfo(np.float32).max)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("P", [4, 33, 1025, 20000])
def test_oracle_matches_float64_kdtree(shape, P):
    x = cloud(shape, P, seed=P)
    got = knn_mean_dist3(x).astype(np.float64)
    want = mean_dist3_float64(x)
    err = np.abs(got - want)
    assert np.all(err <= 1e-6 * want), f"{shape} P={P}: max rel err {np.max(err / np.maximum(want, 1e-300)):.3g}"


def test_oracle_placeholders_for_fewer_than_four_points():
    assert knn_mean_dist3(np.zeros((0, 3), np.float32)).shape == (0,)
    # the missing neighbours are the reference's FLT_MAX slots (simple_knn.cu:154), summed as (b0 + b1) + b2 then / 3
    for P in (1, 2):
        assert np.all(np.isposinf(knn_mean_dist3(cloud("uniform", P))))
    out = knn_mean_dist3(cloud("uniform", 3))
    assert np.all(out == FLT_MAX / np.float32(3.0))
    assert np.all(knn_mean_dist3(cloud("identical", 3)) == FLT_MAX / np.float32(3.0))


def test_oracle_keeps_duplicates_and_excludes_only_self():
    x = np.array([[0, 0, 0], [0, 0, 0], [1, 0, 0], [0, 2, 0]], np.float32)
    out = knn_mean_dist3(x)
    # point 0: neighbours at 0 (its duplicate), 1, 4
    assert out[0] == np.float32(5.0) / np.float32(3.0)
    assert out[2] == np.float32(1.0 + 1.0 + 5.0) / np.float32(3.0)
