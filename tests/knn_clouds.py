"""Seeded point clouds for the distCUDA2 tests (tests/test_knn_oracle.py, tests/test_gpu_knn.py, scripts/time_knn.py)."""
from __future__ import annotations

import numpy as np

# leaf (32 points) and node (1024 points) boundaries of csrc/lgr_knn.cuh, and the oracle's practical limit
SIZES = [4, 5, 31, 32, 33, 63, 1023, 1024, 1025, 4097, 20000]
SHAPES = ["uniform", "offset_cube", "planar", "collinear", "identical", "duplicated", "outlier", "two_clusters", "lattice"]


def cloud(shape: str, P: int, seed: int = 0) -> np.ndarray:
    """float32 [P, 3]"""
    rng = np.random.default_rng(seed)
    if shape == "uniform":            # cube of side 2 at the origin
        x = rng.uniform(-1.0, 1.0, (P, 3))
    elif shape == "offset_cube":      # cube of side 0.05 at offset 10: where fp32 |x|^2 + |y|^2 - 2x.y cancels
        x = 10.0 + rng.uniform(0.0, 0.05, (P, 3))
    elif shape == "planar":           # exactly z = 0
        x = rng.uniform(-1.0, 1.0, (P, 3))
        x[:, 2] = 0.0
    elif shape == "collinear":
        t = rng.uniform(-1.0, 1.0, P)
        x = np.stack([t, 0.5 * t + 1.0, np.full(P, 3.0)], axis=1)
    elif shape == "identical":        # every output is 0
        x = np.tile(np.array([[0.3, -1.2, 5.0]]), (P, 1))
    elif shape == "duplicated":       # every point twice (one extra copy when P is odd), shuffled
        base = rng.uniform(-1.0, 1.0, ((P + 1) // 2, 3))
        x = np.concatenate([base, base])[:P][rng.permutation(P)]
    elif shape == "outlier":          # one point 1e4 away
        x = rng.uniform(-1.0, 1.0, (P, 3))
        x[rng.integers(P)] = (1.0e4, 0.0, 0.0)
    elif shape == "two_clusters":     # 100 apart
        x = rng.uniform(-0.5, 0.5, (P, 3))
        x[rng.random(P) < 0.5] += 100.0
    elif shape == "lattice":          # integer lattice, shuffled: massive ties
        n = int(np.ceil(P ** (1.0 / 3.0))) + 1
        g = np.stack(np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij"), axis=-1).reshape(-1, 3)
        x = g[rng.permutation(len(g))[:P]].astype(np.float64)
    else:
        raise ValueError(shape)
    return np.ascontiguousarray(x, dtype=np.float32)


def sfm_like(P: int, seed: int = 0) -> np.ndarray:
    """An SfM-like cloud: 300 anisotropic clusters of varying density tens of units from the origin, plus 1 % scattered outliers."""
    rng = np.random.default_rng(seed)
    k = 300
    centres = rng.uniform(20.0, 60.0, (k, 3))
    spread = rng.uniform(0.05, 2.0, (k, 3))
    which = rng.integers(0, k, P)
    x = centres[which] + rng.standard_normal((P, 3)) * spread[which]
    far = rng.random(P) < 0.01
    x[far] = rng.uniform(-100.0, 150.0, (int(far.sum()), 3))
    return np.ascontiguousarray(x, dtype=np.float32)


def mean_dist3_float64(x: np.ndarray) -> np.ndarray:
    """float64 mean squared distance to the three nearest other points (scipy cKDTree) of the float32 coordinates"""
    from scipy.spatial import cKDTree
    xd = np.asarray(x, np.float64)
    d, _ = cKDTree(xd).query(xd, k=4)
    # column 0 is the point itself (distance 0); with duplicates the tree may list a duplicate there instead, at the same distance
    return (d[:, 1:] ** 2).mean(axis=1)
