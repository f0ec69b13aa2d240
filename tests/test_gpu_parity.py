"""GPU parity tests: our sm_90a path (through the C-ABI) against
  (a) the CPU oracle (oracle/lgo.c), stage by stage, and
  (b) the reference's own CUDA kernels compiled into oracle/_ref (where oracle/Makefile could build it).

Tolerances (BASELINE.json north_star): rendered RGB 1e-4 abs, gradients 1e-3 rel, significance exact.
Forward comparisons against the reference kernels are expected to be BIT-EXACT because lgr_math.cuh pins
the reference's compiled operation order; the asserted bound is still the contractual 1e-4.
"""
import numpy as np
import pytest

from tests import util
from tests.util import CONFIGS, make_config, run_ours, run_ref, rel_inf, rel_l2, oracle_from_geometry, assert_elementwise
from tests.util import oracle_backward_on_our_state
from oracle.lgo import Oracle

pytestmark = pytest.mark.gpu

RGB_TOL = 1e-4     # abs, north_star
GRAD_TOL = 1e-3    # rel, north_star


def _clamp_bits(clamped3):
    return (clamped3[:, 0].astype(np.uint8) | (clamped3[:, 1].astype(np.uint8) << 1) | (clamped3[:, 2].astype(np.uint8) << 2))


@pytest.mark.parametrize("name", list(CONFIGS))
def test_preprocess_bit_exact_vs_oracle(name):
    """K1: every per-Gaussian quantity equals the oracle bit for bit (same pinned operation order;
    sqrt / div are correctly rounded on both sides)."""
    act, view, _ = make_config(name)
    ours = run_ours(view, act)
    o = Oracle()
    g = o.preprocess(view, act["means3D"], act["opacities"], shs=act["shs"], scales=act["scales"], rotations=act["rotations"])
    og = ours["geom"]
    vis = g["radii"] > 0
    assert vis.sum() > 50
    np.testing.assert_array_equal(ours["radii"], g["radii"])
    np.testing.assert_array_equal(og["tiles_touched"], g["tiles_touched"])
    assert ours["num_rendered"] == int(g["tiles_touched"].sum())
    for k in ("depths", "means2D", "conic_opacity", "rgb"):
        np.testing.assert_array_equal(og[k][vis], g[k][vis], err_msg=k)
    np.testing.assert_array_equal(og["cov3D"][vis], g["cov3D"][vis])
    np.testing.assert_array_equal(og["clamped_bits"][vis], _clamp_bits(g["clamped"])[vis])


@pytest.mark.parametrize("name", list(CONFIGS))
def test_binning_and_blend_vs_oracle(name):
    """binning order identical; image within 1e-4 wherever no threshold test is within rounding noise
    (the oracle's exp() is glibc's, the GPU's is libdevice's on MUFU.EX2)."""
    act, view, _ = make_config(name)
    ours = run_ours(view, act, count=True, tile_cull=False)
    o = Oracle()
    ref = oracle_from_geometry(o, view, ours["geom"], count=True)
    np.testing.assert_array_equal(ours["point_list"], ref["point_list"])
    np.testing.assert_array_equal(ours["ranges"], ref["ranges"])
    frag = ref["fragile"]
    assert frag.mean() < 0.01
    err = np.abs(ours["color"] - ref["color"]).max(axis=0)
    assert err[~frag].max() <= RGB_TOL, f"max abs RGB error {err[~frag].max()} on non-fragile pixels"
    assert err.max() <= 2e-2
    ok = ~frag.reshape(-1)
    np.testing.assert_array_equal(ours["n_contrib"][ok], ref["n_contrib"][ok])
    np.testing.assert_allclose(ours["final_T"][ok], ref["final_T"][ok], atol=1e-5)
    # significance: exact wherever no fragile pixel can have touched the Gaussian
    dc = ours["gaussians_count"].astype(np.int64) - ref["gaussians_count"]
    assert np.abs(dc).sum() <= 64 * max(1, int(frag.sum()))
    if frag.sum() == 0:
        assert np.abs(dc).max() == 0
    np.testing.assert_array_equal(ours["important_score"],
                                  (ours["gaussians_count"].astype(np.float32) * act["opacities"].reshape(-1)).astype(np.float32))


@pytest.mark.parametrize("name", list(CONFIGS))
def test_backward_vs_oracle(name):
    """K6..K8 against the oracle's backward evaluated on OUR forward state (so no threshold can differ)."""
    act, view, dpix = make_config(name)
    ours = run_ours(view, act, dL_dpix=dpix)
    o = Oracle()
    g2, g3 = oracle_backward_on_our_state(o, view, act, ours, dpix)
    mine = ours["grads"]
    checks = {
        "dL_dmeans2D": (mine["dL_dmeans2D"][:, :2], g2["dL_dmean2D"]),
        "dL_dcolors": (mine["dL_dcolors"], g2["dL_dcolor"]),
        "dL_dopacity": (mine["dL_dopacity"].reshape(-1), g2["dL_dopacity"]),
        "dL_dmeans3D": (mine["dL_dmeans3D"], g3["dL_dmeans3D"]),
        "dL_dcov3D": (mine["dL_dcov3D"], g3["dL_dcov3D"]),
        "dL_dsh": (mine["dL_dsh"], g3["dL_dsh"]),
        "dL_dscales": (mine["dL_dscales"], g3["dL_dscales"]),
        "dL_drotations": (mine["dL_drotations"], g3["dL_drotations"]),
    }
    assert np.all(mine["dL_dmeans2D"][:, 2] == 0)
    for k, (a, b) in checks.items():
        assert np.isfinite(a).all(), k
        assert rel_inf(a, b) <= GRAD_TOL, f"{k}: rel_inf {rel_inf(a, b)}"
        assert rel_l2(a, b) <= GRAD_TOL, f"{k}: rel_l2 {rel_l2(a, b)}"
        assert_elementwise(a, b, k)
    # culled Gaussians get exact zeros in every output
    cul = ours["radii"] <= 0
    for k in mine:
        assert np.all(mine[k][cul] == 0), k


def test_precomputed_inputs_vs_oracle():
    """colors_precomp + cov3D_precomp path (render() with convert_SHs_python / compute_cov3D_python)."""
    act, view, dpix = make_config("deg1")
    o = Oracle()
    g = o.preprocess(view, act["means3D"], act["opacities"], shs=act["shs"], scales=act["scales"], rotations=act["rotations"])
    rng = np.random.default_rng(5)
    P = act["means3D"].shape[0]
    colors = rng.uniform(0, 1, (P, 3)).astype(np.float32)
    cov = g["cov3D"].copy()
    cov[g["radii"] <= 0] = np.array([1e-4, 0, 0, 1e-4, 0, 1e-4], np.float32)
    ours = run_ours(view, act, dL_dpix=dpix, colors_precomp=colors, cov3D_precomp=cov)
    gp = o.preprocess(view, act["means3D"], act["opacities"], colors_precomp=colors, cov3D_precomp=cov)
    np.testing.assert_array_equal(ours["radii"], gp["radii"])
    np.testing.assert_array_equal(ours["geom"]["rgb"][gp["radii"] > 0], colors[gp["radii"] > 0])
    ref = oracle_from_geometry(o, view, ours["geom"])
    err = np.abs(ours["color"] - ref["color"]).max(axis=0)
    assert err[~ref["fragile"]].max() <= RGB_TOL
    g2, g3 = oracle_backward_on_our_state(o, view, act, ours, dpix, colors=colors, cov=cov)
    mine = ours["grads"]
    for a, b, k in ((mine["dL_dcolors"], g2["dL_dcolor"], "dL_dcolors"), (mine["dL_dcov3D"], g3["dL_dcov3D"], "dL_dcov3D"),
                    (mine["dL_dmeans3D"], g3["dL_dmeans3D"], "dL_dmeans3D"), (mine["dL_dopacity"].reshape(-1), g2["dL_dopacity"], "dL_dopacity")):
        assert rel_inf(a, b) <= GRAD_TOL, f"{k}: {rel_inf(a, b)}"
    assert mine["dL_dsh"].shape == (P, 0, 3)
    assert np.all(mine["dL_dscales"] == 0) and np.all(mine["dL_drotations"] == 0)


# ------------------------------------------------------------------------------------------------
# against the reference's own kernels (oracle/_ref), same GPU
# ------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref/libref_rasterizer.so not built (needs the reference checkout)")


@needs_ref
@pytest.mark.parametrize("name", list(CONFIGS))
def test_forward_vs_reference_kernels(name):
    act, view, _ = make_config(name)
    ours = run_ours(view, act, tile_cull=False)
    ref = run_ref(view, act)
    assert ours["num_rendered"] == ref["num_rendered"]
    np.testing.assert_array_equal(ours["radii"], ref["radii"])
    vis = ref["radii"] > 0
    for k in ("depths", "means2D", "conic_opacity", "rgb"):
        np.testing.assert_array_equal(ours["geom"][k][vis], ref["geom"][k][vis], err_msg=k)
    np.testing.assert_array_equal(ours["point_list"], ref["point_list"])
    np.testing.assert_array_equal(ours["ranges"], ref["ranges"])
    np.testing.assert_array_equal(ours["n_contrib"], ref["n_contrib"])
    assert np.abs(ours["color"] - ref["color"]).max() <= RGB_TOL
    # stronger than the contract: bit-identical image and transmittance
    np.testing.assert_array_equal(ours["color"], ref["color"])
    np.testing.assert_array_equal(ours["final_T"], ref["final_T"])


@needs_ref
@pytest.mark.parametrize("name", list(CONFIGS))
def test_backward_vs_reference_kernels(name):
    act, view, dpix = make_config(name)
    ours = run_ours(view, act, dL_dpix=dpix)
    ref = run_ref(view, act, dL_dpix=dpix)
    for k in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations"):
        a, b = ours["grads"][k], ref["grads"][k].reshape(ours["grads"][k].shape)
        assert rel_inf(a, b) <= GRAD_TOL, f"{k}: rel_inf {rel_inf(a, b)}"
        assert rel_l2(a, b) <= GRAD_TOL, f"{k}: rel_l2 {rel_l2(a, b)}"
        assert_elementwise(a, b, k)


@needs_ref
def test_precomputed_inputs_vs_reference_kernels():
    """colors_precomp + cov3D_precomp (the convert_SHs_python / compute_cov3D_python pipeline flags) against the reference's own
    kernels: forward bit-identical, gradients to tolerance, no SH / scale / rotation gradients."""
    act, view, dpix = make_config("deg1")
    o = Oracle()
    g = o.preprocess(view, act["means3D"], act["opacities"], shs=act["shs"], scales=act["scales"], rotations=act["rotations"])
    P = act["means3D"].shape[0]
    colors = np.random.default_rng(5).uniform(0, 1, (P, 3)).astype(np.float32)
    cov = g["cov3D"].copy()
    cov[g["radii"] <= 0] = np.array([1e-4, 0, 0, 1e-4, 0, 1e-4], np.float32)
    ours = run_ours(view, act, dL_dpix=dpix, colors_precomp=colors, cov3D_precomp=cov, tile_cull=False)
    ref = run_ref(view, act, dL_dpix=dpix, colors_precomp=colors, cov3D_precomp=cov)
    assert ours["num_rendered"] == ref["num_rendered"]
    np.testing.assert_array_equal(ours["radii"], ref["radii"])
    np.testing.assert_array_equal(ours["point_list"], ref["point_list"])
    np.testing.assert_array_equal(ours["color"], ref["color"])
    np.testing.assert_array_equal(ours["final_T"], ref["final_T"])
    for k in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D"):
        a, b = ours["grads"][k], ref["grads"][k].reshape(ours["grads"][k].shape)
        assert rel_inf(a, b) <= GRAD_TOL, f"{k}: rel_inf {rel_inf(a, b)}"
        assert_elementwise(a, b, k)


@needs_ref
@pytest.mark.parametrize("cam", ["sphere", "inside"])
def test_config_c1_10k_400x400_vs_reference_kernels(cam):
    """BASELINE.json configs[0] literally: 10 000 synthetic Gaussians, one 400x400 camera, forward render -- plus the correctness-only
    camera INSIDE the cube (z <= 0.2 cull, 1.3 tanfov clamp, huge splats) of SURVEY.md section 8d, and the backward on both."""
    from lightgaussian_b200.synth import make_scene, make_cameras, inside_camera
    scene = make_scene(10_000, sh_degree=3, seed=0)
    c = inside_camera(400, 400) if cam == "inside" else make_cameras(1, 400, 400)[0]
    view = util.view_from_camera(c, (0.0, 0.0, 0.0), 3, 1.0)
    dpix = np.random.default_rng(3).standard_normal((3, 400, 400)).astype(np.float32)
    ours = run_ours(view, scene["act"], dL_dpix=dpix, tile_cull=False)
    ref = run_ref(view, scene["act"], dL_dpix=dpix)
    assert ours["num_rendered"] == ref["num_rendered"] > 0
    np.testing.assert_array_equal(ours["radii"], ref["radii"])
    np.testing.assert_array_equal(ours["point_list"], ref["point_list"])
    np.testing.assert_array_equal(ours["ranges"], ref["ranges"])
    assert np.abs(ours["color"] - ref["color"]).max() <= RGB_TOL
    np.testing.assert_array_equal(ours["color"], ref["color"])
    np.testing.assert_array_equal(ours["n_contrib"], ref["n_contrib"])
    culled = run_ours(view, scene["act"])                       # the product default (exact tile culling): same image
    np.testing.assert_array_equal(culled["color"], ref["color"])
    # arbiter for the per-element check: the float64 oracle's backward on the (bit-identical) forward state
    g2, g3 = oracle_backward_on_our_state(Oracle(double=True), view, scene["act"], ours, dpix)
    exact = {"dL_dmeans2D": np.concatenate([g2["dL_dmean2D"], np.zeros((g2["dL_dmean2D"].shape[0], 1))], axis=1), "dL_dcolors": g2["dL_dcolor"],
             "dL_dopacity": g2["dL_dopacity"], "dL_dmeans3D": g3["dL_dmeans3D"], "dL_dcov3D": g3["dL_dcov3D"], "dL_dsh": g3["dL_dsh"],
             "dL_dscales": g3["dL_dscales"], "dL_drotations": g3["dL_drotations"]}
    for k in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations"):
        a, b = ours["grads"][k], ref["grads"][k].reshape(ours["grads"][k].shape)
        assert rel_inf(a, b) <= GRAD_TOL, f"{k}: rel_inf {rel_inf(a, b)}"
        assert_elementwise(a, b, k, exact=np.asarray(exact[k], np.float64).reshape(a.shape))


@needs_ref
def test_significance_vs_reference_kernels():
    """The reference's counter is a racy, non-atomic ++ (forward.cu:473-474): it can only LOSE updates.
    Ours is exact, so ref <= ours everywhere, image and radii identical."""
    act, view, _ = make_config("outside")
    ours = run_ours(view, act, count=True)
    ref = run_ref(view, act, count=True)
    np.testing.assert_array_equal(ours["color"], ref["color"])
    assert np.all(ref["gaussians_count"] <= ours["gaussians_count"])
    assert ours["gaussians_count"].sum() > 0
    # count-mode image == plain forward image
    plain = run_ours(view, act)
    np.testing.assert_array_equal(ours["color"], plain["color"])


@pytest.mark.parametrize("name", list(CONFIGS))
def test_tile_culling_changes_lists_but_not_results(name):
    """The product default drops (tile, Gaussian) instances in which no pixel can reach alpha >= 1/255.  Outputs must be
    bit-identical to the unculled run (= the reference's lists), the kept list an order-preserving subsequence."""
    act, view, dpix = make_config(name)
    full = run_ours(view, act, count=True, tile_cull=False)
    cull = run_ours(view, act, count=True)
    assert cull["num_rendered"] == full["num_rendered"]               # API value = the reference's definition
    assert cull["num_listed"] <= full["num_listed"] == full["num_rendered"]
    np.testing.assert_array_equal(cull["color"], full["color"])
    np.testing.assert_array_equal(cull["final_T"], full["final_T"])
    np.testing.assert_array_equal(cull["gaussians_count"], full["gaussians_count"])
    np.testing.assert_array_equal(cull["radii"], full["radii"])
    for t in range(full["ranges"].shape[0]):
        a = full["point_list"][full["ranges"][t, 0]:full["ranges"][t, 1]].tolist()
        b = cull["point_list"][cull["ranges"][t, 0]:cull["ranges"][t, 1]].tolist()
        it = iter(a)
        assert all(x in it for x in b), f"tile {t}: culled list is not an ordered subsequence"
    gf = run_ours(view, act, dL_dpix=dpix, tile_cull=False)["grads"]
    gc = run_ours(view, act, dL_dpix=dpix)["grads"]
    for k in gf:
        assert rel_inf(gc[k], gf[k]) <= GRAD_TOL, k
    if name == "outside":
        assert cull["num_listed"] < full["num_listed"]


@pytest.mark.parametrize("name", list(CONFIGS))
def test_ring_kernels_equal_the_round1_kernels(name):
    """The shared-ring blend kernels (producer warp, TMA-staged records, sign-of-T termination, two-scalar backward reduction) against
    the round-1 per-warp kernels of the same library: forward outputs and significance counts bit-identical, gradients to tolerance."""
    act, view, dpix = make_config(name)
    new = run_ours(view, act, count=True)
    old = run_ours(view, act, count=True, blend_mode=1)
    for k in ("color", "final_T", "n_contrib", "gaussians_count", "important_score", "radii"):
        np.testing.assert_array_equal(new[k], old[k], err_msg=k)
    gn = run_ours(view, act, dL_dpix=dpix)
    go = run_ours(view, act, dL_dpix=dpix, blend_mode=1)
    np.testing.assert_array_equal(gn["color"], go["color"])
    for k in gn["grads"]:
        assert rel_inf(gn["grads"][k], go["grads"][k]) <= GRAD_TOL, f"{k}: {rel_inf(gn['grads'][k], go['grads'][k])}"
        assert_elementwise(gn["grads"][k], go["grads"][k], k)


# ------------------------------------------------------------------------------------------------
# edge cases (empty / ragged / degenerate inputs)
# ------------------------------------------------------------------------------------------------
def test_empty_scene_is_zero_image():
    act, view, _ = make_config("deg0")
    empty = {k: v[:0] for k, v in act.items()}
    ours = run_ours(view, empty)
    assert ours["num_rendered"] == 0 and ours["radii"].shape == (0,)
    assert np.all(ours["color"] == 0)  # rasterize_points.cu:79-93: P == 0 leaves the zero-filled image


def test_all_culled_gives_background():
    act, view, dpix = make_config("deg1")
    far = dict(act)
    far["means3D"] = (act["means3D"] * 0.01 + np.array([50.0, 50.0, 50.0], np.float32)).astype(np.float32)
    ours = run_ours(view, far, dL_dpix=dpix)
    assert ours["num_rendered"] == 0 and np.all(ours["radii"] == 0)
    for c in range(3):
        assert np.all(ours["color"][c] == view.bg[c])
    for k, g in ours["grads"].items():
        assert np.all(g == 0), k


@pytest.mark.parametrize("wh", [(1, 1), (17, 5), (16, 16), (33, 47)])
def test_ragged_image_sizes(wh):
    from lightgaussian_b200.synth import make_scene, make_cameras
    W, H = wh
    scene = make_scene(500, seed=21, scale_mult=3.0)
    view = util.view_from_camera(make_cameras(3, W, H)[1], (0.1, 0.2, 0.3), 3, 1.0)
    ours = run_ours(view, scene["act"], count=True, tile_cull=False)
    o = Oracle()
    ref = oracle_from_geometry(o, view, ours["geom"], count=True)
    err = np.abs(ours["color"] - ref["color"]).max(axis=0)
    assert err[~ref["fragile"]].max(initial=0.0) <= RGB_TOL
    np.testing.assert_array_equal(ours["point_list"], ref["point_list"])
    culled = run_ours(view, scene["act"], count=True)
    np.testing.assert_array_equal(culled["color"], ours["color"])
    np.testing.assert_array_equal(culled["gaussians_count"], ours["gaussians_count"])


def test_single_gaussian_and_huge_splat():
    """one Gaussian covering the whole image: every tile lists it once."""
    from lightgaussian_b200.synth import make_cameras
    W, H = 64, 48
    act = dict(means3D=np.zeros((1, 3), np.float32), scales=np.full((1, 3), 2.0, np.float32),
               rotations=np.array([[1, 0, 0, 0]], np.float32), opacities=np.array([[0.7]], np.float32),
               shs=np.zeros((1, 16, 3), np.float32))
    act["shs"][0, 0] = [1.0, 0.5, -3.0]
    view = util.view_from_camera(make_cameras(3, W, H)[1], (0.0, 0.0, 0.0), 0, 1.0)
    ours = run_ours(view, act, count=True)
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    assert ours["num_rendered"] == tiles == ours["num_listed"]
    assert ours["gaussians_count"][0] == W * H
    assert ours["geom"]["clamped_bits"][0] == 4  # blue channel clamped at 0
    assert np.all(ours["color"][2] == 0)


def test_mark_visible():
    import torch
    from lightgaussian_b200.rasterizer import _C
    act, view, _ = make_config("inside")
    vis = _C.mark_visible(torch.from_numpy(act["means3D"]).cuda(), torch.from_numpy(view.viewmatrix).cuda(),
                          torch.from_numpy(view.projmatrix).cuda()).cpu().numpy()
    np.testing.assert_array_equal(vis, Oracle().mark_visible(view, act["means3D"]))
    assert 0 < vis.sum() < vis.size
