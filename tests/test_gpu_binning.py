"""The hand-written binning kernels (csrc/lgr_bin.cuh: three-pass depth sort, single-pass stable tile bucketing, blob sized from
an estimate) against the round-1 library path and against the reference's own kernels: per-tile lists, ranges, depth order and
image must be bit-identical in every mode, also when the estimate is too small and scatter + blend are repeated."""
import numpy as np
import pytest

from lightgaussian_b200.synth import make_scene, make_cameras
from tests import util
from tests.util import CONFIGS, make_config, run_ours, run_ref, view_from_camera

pytestmark = pytest.mark.gpu


def _same(a, b, grads=False):
    assert a["num_rendered"] == b["num_rendered"]
    assert a["num_listed"] == b["num_listed"]
    np.testing.assert_array_equal(a["geom"]["sorted_ids"], b["geom"]["sorted_ids"])
    np.testing.assert_array_equal(a["geom"]["tiles_touched"], b["geom"]["tiles_touched"])
    np.testing.assert_array_equal(a["ranges"], b["ranges"])
    np.testing.assert_array_equal(a["point_list"], b["point_list"])
    np.testing.assert_array_equal(a["n_contrib"], b["n_contrib"])
    np.testing.assert_array_equal(a["final_T"], b["final_T"])
    np.testing.assert_array_equal(a["color"], b["color"])
    if "gaussians_count" in a:
        np.testing.assert_array_equal(a["gaussians_count"], b["gaussians_count"])


@pytest.mark.parametrize("tile_cull", [True, False])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_binning_modes_agree(name, tile_cull):
    from lightgaussian_b200 import capi
    act, view, dpix = make_config(name)
    lib = run_ours(view, act, tile_cull=tile_cull, bin_mode=2)
    exact = run_ours(view, act, tile_cull=tile_cull, bin_mode=1)
    _same(exact, lib)
    capi.set_binning_estimate(0)          # forget the estimate: the first view overflows the 4096-instance floor and is repeated
    n0 = capi.binning_overflows()
    est = run_ours(view, act, tile_cull=tile_cull, bin_mode=0)
    if lib["num_listed"] > 4096:
        assert capi.binning_overflows() == n0 + 1
    _same(est, lib)
    n1 = capi.binning_overflows()
    est2 = run_ours(view, act, tile_cull=tile_cull, bin_mode=0, count=True)   # now the estimate fits: no repeat
    assert capi.binning_overflows() == n1
    libc = run_ours(view, act, tile_cull=tile_cull, bin_mode=2, count=True)
    _same(est2, libc)


def test_overflow_repeat_keeps_the_significance_exact():
    from lightgaussian_b200 import capi
    act, view, _ = make_config("outside")
    ref = run_ours(view, act, count=True, bin_mode=2)
    capi.set_binning_estimate(0)
    n0 = capi.binning_overflows()
    got = run_ours(view, act, count=True, bin_mode=0)
    assert capi.binning_overflows() == n0 + 1
    np.testing.assert_array_equal(got["gaussians_count"], ref["gaussians_count"])   # the repeat re-zeroes the counters
    np.testing.assert_array_equal(got["important_score"], ref["important_score"])


def test_backward_after_estimated_and_repeated_forward():
    """the ring backward finds the per-instance records through the capacity word of the geometry header"""
    from lightgaussian_b200 import capi
    act, view, dpix = make_config("outside")
    ref = run_ours(view, act, dL_dpix=dpix, bin_mode=2)
    for estimate in (0, 10_000_000):
        capi.set_binning_estimate(estimate)
        got = run_ours(view, act, dL_dpix=dpix, bin_mode=0)
        for k in ref["grads"]:
            assert util.rel_inf(got["grads"][k], ref["grads"][k]) <= 1e-4, k     # same kernels, atomics reorder the sums


needs_ref = pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref/libref_rasterizer.so not built (needs the reference checkout)")


@needs_ref
@pytest.mark.parametrize("P,W,H", [(200_000, 1920, 1080), (50_000, 4096, 2304), (7, 64, 48), (100_000, 33, 17)])
def test_lists_vs_reference_kernels_other_shapes(P, W, H):
    """more tiles than the 1080p bench (36 864), a handful of Gaussians, an image smaller than two tiles"""
    scene = make_scene(P, sh_degree=3, seed=3, scale_mult=1.0 if P > 1000 else 20.0)
    cam = make_cameras(7, W, H)[3]
    view = view_from_camera(cam, (0.0, 0.0, 0.0), 3, 1.0)
    ours = run_ours(view, scene["act"], tile_cull=False)
    ref = run_ref(view, scene["act"])
    assert ours["num_rendered"] == ref["num_rendered"]
    np.testing.assert_array_equal(ours["point_list"], ref["point_list"])
    np.testing.assert_array_equal(ours["ranges"], ref["ranges"])
    np.testing.assert_array_equal(ours["color"], ref["color"])


def test_full_size_lists_match_the_library_path():
    P, W, H = 1_000_000, 1920, 1080
    scene = make_scene(P, sh_degree=3, seed=0)
    cam = make_cameras(16, W, H)[5]
    view = view_from_camera(cam, (0.0, 0.0, 0.0), 3, 1.0)
    _same(run_ours(view, scene["act"], bin_mode=0), run_ours(view, scene["act"], bin_mode=2))
