"""Full-size checks (BASELINE.json config 1: 1M Gaussians, 1920x1080) where the CPU oracle is too slow:
size-independent properties, and parity with the reference's own kernels on the same GPU."""
import numpy as np
import pytest
import torch

from lightgaussian_b200.synth import make_scene, make_cameras
from tests import util
from tests.util import run_ours, run_ref, rel_inf, rel_l2, view_from_camera, assert_elementwise

pytestmark = pytest.mark.gpu

P, W, H = 1_000_000, 1920, 1080


@pytest.fixture(scope="module")
def big():
    scene = make_scene(P, sh_degree=3, seed=0)
    cam = make_cameras(16, W, H)[5]
    view = view_from_camera(cam, (0.0, 0.0, 0.0), 3, 1.0)
    dpix = np.random.default_rng(7).standard_normal((3, H, W)).astype(np.float32)
    return scene["act"], view, dpix


def test_forward_is_deterministic_and_lists_are_depth_sorted(big):
    act, view, _ = big
    a = run_ours(view, act, count=True)
    b = run_ours(view, act, count=True)
    np.testing.assert_array_equal(a["color"], b["color"])
    np.testing.assert_array_equal(a["gaussians_count"], b["gaussians_count"])     # exact integer significance: run-to-run identical
    np.testing.assert_array_equal(a["point_list"], b["point_list"])
    assert a["num_rendered"] == int(a["geom"]["tiles_touched"].sum()) >= a["num_listed"] > 0
    depth, pl, rg = a["geom"]["depths"], a["point_list"], a["ranges"]
    rng = np.random.default_rng(1)
    covered = int((rg[:, 1] - rg[:, 0]).sum())
    assert covered == a["num_listed"]
    for t in rng.choice(rg.shape[0], 300, replace=False):
        s, e = rg[t]
        if e > s:
            ids = pl[s:e].astype(np.int64)
            d = depth[ids]
            assert np.all(np.diff(d) >= 0)
            assert np.all(np.diff(ids)[np.diff(d) == 0] > 0)          # equal depth -> ascending id (stable order of the reference)
    # a Gaussian is counted at most once per pixel and only if it is listed somewhere
    assert a["gaussians_count"].max() <= W * H
    listed = np.zeros(P, bool)
    listed[pl] = True
    assert not np.any(a["gaussians_count"][~listed])
    assert np.isfinite(a["color"]).all() and a["color"].min() >= 0.0


def test_backward_is_linear_in_the_pixel_gradient(big):
    act, view, dpix = big
    g1 = run_ours(view, act, dL_dpix=dpix)["grads"]
    g2 = run_ours(view, act, dL_dpix=(2.0 * dpix).astype(np.float32))["grads"]
    for k in g1:
        assert np.isfinite(g1[k]).all(), k
        assert rel_inf(g2[k], 2.0 * g1[k]) <= 1e-4, (k, rel_inf(g2[k], 2.0 * g1[k]))   # float atomics reorder sums run to run
    cul = run_ours(view, act)["radii"] <= 0
    for k in g1:
        assert np.all(g1[k][cul] == 0), k


@pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref/libref_rasterizer.so not built (needs the reference checkout)")
def test_full_size_parity_with_reference_kernels(big):
    act, view, dpix = big
    ours = run_ours(view, act, dL_dpix=dpix)
    ref = run_ref(view, act, dL_dpix=dpix)
    assert ours["num_rendered"] == ref["num_rendered"]
    np.testing.assert_array_equal(ours["radii"], ref["radii"])
    assert np.abs(ours["color"] - ref["color"]).max() <= 1e-4          # the contract ...
    np.testing.assert_array_equal(ours["color"], ref["color"])         # ... and in fact bit-identical
    np.testing.assert_array_equal(ours["final_T"], ref["final_T"])
    for k in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations"):
        a, b = ours["grads"][k], ref["grads"][k].reshape(ours["grads"][k].shape)
        assert rel_inf(a, b) <= 1e-3, f"{k}: rel_inf {rel_inf(a, b)}"
        assert rel_l2(a, b) <= 1e-3, f"{k}: rel_l2 {rel_l2(a, b)}"
        assert_elementwise(a, b, k)
    cnt = run_ours(view, act, count=True)
    refc = run_ref(view, act, count=True)
    assert np.all(refc["gaussians_count"] <= cnt["gaussians_count"])   # the reference's racy counter only loses updates
    # how much the racy counter loses (measured 97 % on this scene: lanes of a warp hitting the same Gaussian collapse to one
    # increment, forward.cu:473-474) and how the two rankings correlate -- reported, not part of the contract (SURVEY.md 8c)
    lost = 1.0 - refc["gaussians_count"].sum() / cnt["gaussians_count"].sum()
    v = cnt["gaussians_count"] > 0
    ra, rb = np.argsort(np.argsort(cnt["important_score"][v])), np.argsort(np.argsort(refc["important_score"][v]))
    rho = np.corrcoef(ra, rb)[0, 1]
    print(f"reference racy counter loses {100 * lost:.1f} % of the updates; Spearman rho(exact score, racy score) = {rho:.3f}")
    assert 0.0 <= lost < 1.0 and np.isfinite(rho)


@pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref/libref_rasterizer.so not built (needs the reference checkout)")
def test_bench_config_3m_1080p_parity_with_reference_kernels():
    """The exact bench.py workload (BASELINE.json configs[2] scene: 3M Gaussians, SH degree 3, 1920x1080, camera 0 of the bench's
    16): forward bit-identical to the reference's kernels, gradients to 1e-3."""
    scene = make_scene(3_000_000, sh_degree=3, seed=0)
    view = view_from_camera(make_cameras(16, W, H)[0], (0.0, 0.0, 0.0), 3, 1.0)
    dpix = np.random.default_rng(11).standard_normal((3, H, W)).astype(np.float32)
    ours = run_ours(view, scene["act"], dL_dpix=dpix)
    ref = run_ref(view, scene["act"], dL_dpix=dpix)
    assert ours["num_rendered"] == ref["num_rendered"]
    np.testing.assert_array_equal(ours["radii"], ref["radii"])
    np.testing.assert_array_equal(ours["color"], ref["color"])
    np.testing.assert_array_equal(ours["final_T"], ref["final_T"])
    for k in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations"):
        a, b = ours["grads"][k], ref["grads"][k].reshape(ours["grads"][k].shape)
        assert rel_inf(a, b) <= 1e-3, f"{k}: rel_inf {rel_inf(a, b)}"
        assert rel_l2(a, b) <= 1e-3, f"{k}: rel_l2 {rel_l2(a, b)}"
        assert_elementwise(a, b, k)
