"""Absolute-gradient densification statistic (LGR_DENSIFY_GRAD=abs, lgr_backward_raw_absgrad, DESIGN.md section 7):
  1. absgrad equals the sum over pixels of |dL/dmeans2D| of the existing lgr_backward_raw run with dL/dpix non-zero at one pixel only;
  2. absgrad against float64 (tests/native/absgrad_host.c: the reference's blend backward terms) on the fused forward's own state, every element, from P = 0 to the bench view, 1x1 to 1080p,
     a fully culled view, every binning mode with tile culling on and off and every K7+K8 mode; the six leaf gradients and dL/dmeans2D
     of the same call pass the default backward's BOUNDS, and absgrad >= |dL/dmeans2D[:, :2]|;
  3. render(): the forward bit for bit, .absgrad on the view-space tensor, the refusals before any launch, nothing new when unset;
  4. add_densification_stats in abs mode over 20 real views, bit for bit and without a host synchronisation;
  5. the unmodified train_densify_prune.py opting in."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from lightgaussian_b200 import capi, trace
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
from lightgaussian_b200.rasterizer import (_forward_raw_native, _make_view, _raw_grads_struct, _raw_struct, enable_gradient_exchange)
from lightgaussian_b200.renderer import render
from lightgaussian_b200.synth import make_cameras, make_scene
from tests import scripts_harness as sh
from tests.test_absgrad_cpu import absgrad_float64
from tests.test_gpu_leafgrad import BOUNDS, GRADS, _activated, _leaves, _raw_np, _settings
from tests.util import assert_every_element, element_ratios, leaf_grads_float64, read_state, view_from_camera

pytestmark = pytest.mark.gpu

ABS_BOUND = BOUNDS["means2D"]   # (1e-3, 3e-5): no looser than dL/dmeans2D's
WORST = {}                       # case -> worst ratio to ABS_BOUND, printed at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print(f"\nabsgrad vs float64, bound {ABS_BOUND}: worst ratio {max(WORST.values()):.3g} over {len(WORST)} cases")
        for k, v in sorted(WORST.items(), key=lambda kv: -kv[1])[:8]:
            print(f"  {k}: {v:.3g}")


def _scene(P, seed, needles=0, scale_mult=1.0):
    """make_scene with the first `needles` Gaussians turned into needles (one long axis, two very short ones)"""
    raw = dict(make_scene(max(P, 1), sh_degree=3, seed=seed, scale_mult=scale_mult)["raw"])
    raw = {k: np.ascontiguousarray(v[:P]) for k, v in raw.items()}
    if needles:
        s = raw["scaling"].copy()
        s[:needles, 0] += 3.0
        s[:needles, 1:] -= 2.5
        raw["scaling"] = s
    return raw


def _setup(raw, cam, bg=(0.1, 0.2, 0.3)):
    pc = GaussianParams(raw, 3, "cuda", requires_grad=False)
    leaves = _leaves(pc)
    tcam = TorchCamera(cam, "cuda")
    rs = _settings(tcam, torch.tensor(bg, device="cuda"), 3)
    return leaves, rs, view_from_camera(cam, bg, 3, 1.0)


def _backward(rs, R, dpix, leaves, radii, blobs, absgrad=True):
    """lgr_backward_raw_absgrad (or lgr_backward_raw) into NaN-filled outputs: (the six leaf gradients + dL/dmeans2D, absgrad)"""
    lib = capi.load()
    P, M = leaves[0].shape[0], 1 + leaves[2].shape[1]
    H, W = dpix.shape[1], dpix.shape[2]
    nan = lambda *s: torch.full(s, float("nan"), device="cuda")  # noqa: E731
    outs = [nan(*t.shape) for t in leaves] + [nan(P, 3)]
    ag = nan(P, 2)
    with torch.cuda.device(dpix.device):
        view, keep = _make_view(dpix.device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W,
                                rs.scale_modifier, rs.sh_degree, False, rs.debug)
        args = (C.byref(view), P, M, int(R), C.byref(_raw_struct(*leaves)), radii.data_ptr(), blobs[0].data_ptr(), blobs[1].data_ptr(),
                blobs[2].data_ptr(), dpix.data_ptr(), C.byref(_raw_grads_struct(*outs[:6])), outs[6].data_ptr())
        if absgrad:
            st = lib.lgr_backward_raw_absgrad(*args, ag.data_ptr(), capi.current_stream_ptr(dpix.device))
        else:
            st = lib.lgr_backward_raw(*args, capi.current_stream_ptr(dpix.device))
    capi.check(st, "lgr_backward_raw_absgrad" if absgrad else "lgr_backward_raw")
    torch.cuda.synchronize()
    return {n: t.cpu().numpy() for n, t in zip(GRADS, outs)}, ag.cpu().numpy()


def _check_case(tag, raw, cam, seed=0, leaf_bounds=True):
    """absgrad against the float64 arbiter on our own forward state, plus the other outputs against BOUNDS"""
    leaves, rs, view = _setup(raw, cam)
    P = leaves[0].shape[0]
    with torch.no_grad():
        _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
    radii_np = radii.cpu().numpy()
    H, W = cam.image_height, cam.image_width
    dpix = torch.randn(3, H, W, generator=torch.Generator().manual_seed(seed + W + 7 * H)).cuda()
    grads, ag = _backward(rs, R, dpix, leaves, radii, (geom, binning, img))
    assert ag.shape == (P, 2) and np.isfinite(ag).all(), tag
    assert np.all(ag[radii_np <= 0] == 0), f"{tag}: absgrad rows of culled Gaussians are not exact zeros"
    if R == 0 or P == 0:
        assert np.all(ag == 0)
        for n in GRADS:
            assert np.all(grads[n] == 0), (tag, n)
        return
    state = read_state(view, P, R, radii_np, geom, binning, img)
    g = state["geom"]
    ex = absgrad_float64(W, H, P, state["ranges"], state["point_list"], g["means2D"], g["conic_opacity"], g["rgb"], view.bg,
                         state["final_T"], state["n_contrib"], dpix.cpu().numpy())
    WORST[tag] = assert_every_element(ag, ex, *ABS_BOUND, f"{tag} absgrad")
    # absgrad >= |dL/dmeans2D| element by element, up to the rounding of the two float32 sums
    m2 = np.abs(grads["means2D"][:, :2].astype(np.float64))
    scale = np.abs(ex).max(initial=0.0)
    assert np.all(ag >= m2 - (2e-3 * ag + 2 * ABS_BOUND[1] * scale)), tag
    if leaf_bounds:
        # the other outputs are the default backward's, up to the order of the float atomics: against float64 they pass BOUNDS, or,
        # where the default lgr_backward_raw on the same state does not either, they are no further off than it is
        exact = leaf_grads_float64(view, _raw_np(leaves), state, dpix.cpu().numpy(), act=_activated(leaves, 3))
        default, _ = _backward(rs, R, dpix, leaves, radii, (geom, binning, img), absgrad=False)
        for n in GRADS:
            assert np.isfinite(grads[n]).all() and np.all(grads[n][radii_np <= 0] == 0), (tag, n)
            r_abs = float(element_ratios(grads[n], exact[n], *BOUNDS[n]).max(initial=0.0))
            r_def = float(element_ratios(default[n], exact[n], *BOUNDS[n]).max(initial=0.0))
            if r_def > 1.0:
                print(f"{tag} {n}: the default backward itself is at {r_def:.3g} of BOUNDS, the absgrad call at {r_abs:.3g}")
            assert r_abs <= max(1.0, 1.1 * r_def), (tag, n, r_abs, r_def)
        assert np.all(grads["means2D"][:, 2] == 0)


# ------------------------------------------------------------------------------------------------
# 1. the per-pixel definition, from the existing backward
# ------------------------------------------------------------------------------------------------
def test_absgrad_is_the_sum_of_one_pixel_backwards():
    W, H = 24, 16
    raw = _scene(3000, seed=11, needles=300, scale_mult=2.0)
    cam = make_cameras(4, W, H)[1]
    leaves, rs, view = _setup(raw, cam)
    P = leaves[0].shape[0]
    with torch.no_grad():
        _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
    assert R > 0
    dpix = torch.randn(3, H, W, generator=torch.Generator().manual_seed(3)).cuda()
    blobs = (geom, binning, img)
    _, ag = _backward(rs, R, dpix, leaves, radii, blobs)
    total = np.zeros((P, 2))
    npix = np.zeros(P, np.int64)   # pixels whose one-pixel backward reaches the Gaussian
    one = torch.zeros_like(dpix)
    for py in range(H):
        for px in range(W):
            one.zero_()
            one[:, py, px] = dpix[:, py, px]
            g, _ = _backward(rs, R, one, leaves, radii, blobs, absgrad=False)
            total += np.abs(g["means2D"][:, :2].astype(np.float64))
            npix += np.abs(g["means2D"][:, :2]).sum(1) > 0
    worst = assert_every_element(ag, total, *ABS_BOUND, "absgrad vs sum of one-pixel backwards")
    print(f"absgrad vs sum over {W * H} one-pixel lgr_backward_raw calls: worst ratio {worst:.3g} of {ABS_BOUND}")
    # a Gaussian that one pixel reaches: absgrad == |dL/dmeans2D| up to rounding (both are that pixel's term)
    full, _ = _backward(rs, R, dpix, leaves, radii, blobs, absgrad=False)
    single = npix == 1
    print(f"Gaussians reached by exactly one pixel: {int(single.sum())}")
    if single.any():
        np.testing.assert_allclose(ag[single], np.abs(full["means2D"][single, :2]), rtol=1e-3, atol=1e-6 * float(np.abs(total).max()))


# ------------------------------------------------------------------------------------------------
# 2. against float64.  The scenes are make_scene's, whose scales already spread over e^(+-1.5).  Far needles stay in test 1: there
# float32 and float64 take different alpha-threshold decisions on pairs whose |dL/dmean2D| term is among the largest (the term grows
# with the distance to the needle's axis), the same decisions the reference's float32 kernels take.
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,wh", [(0, (64, 48)), (1, (64, 48)), (5, (17, 5)), (4099, (1, 1)), (4099, (17, 5)), (4099, (64, 48)),
                                  (30001, (640, 360)), (30001, (1920, 1080))])
def test_absgrad_against_float64(P, wh):
    W, H = wh
    raw = _scene(P, seed=100 + P, scale_mult=3.0 if P < 10 else 1.5)
    _check_case(f"P={P} {W}x{H}", raw, make_cameras(3, W, H)[1], seed=P)


def test_absgrad_fully_culled_view():
    raw = _scene(2000, seed=4)
    cam = make_cameras(3, 64, 48)[1]
    raw = dict(raw)
    raw["xyz"] = (1.5 * cam.camera_center[None, :] + 0.01 * np.random.default_rng(0).standard_normal((2000, 3))).astype(np.float32)
    _check_case("culled", raw, cam)


@pytest.mark.parametrize("binning", [0, 1, 2])
@pytest.mark.parametrize("cull", [True, False])
def test_absgrad_binning_modes(binning, cull):
    capi.set_binning_mode(binning)
    capi.set_tile_culling(cull)
    try:
        _check_case(f"binning={binning} cull={cull}", _scene(20000, seed=21), make_cameras(3, 320, 240)[2], leaf_bounds=False)
    finally:
        capi.set_binning_mode(0)
        capi.set_tile_culling(True)


@pytest.mark.parametrize("kback", [0, 1, 2])
def test_absgrad_kback_modes(kback):
    capi.set_kback_mode(kback)
    try:
        _check_case(f"kback={kback}", _scene(20000, seed=22), make_cameras(3, 320, 240)[0])
    finally:
        capi.set_kback_mode(0)


def test_absgrad_bench_view():
    """one bench-size view: 3M Gaussians at 1080p"""
    _check_case("bench 3M 1920x1080", _scene(3_000_000, seed=0), make_cameras(16, 1920, 1080)[0], leaf_bounds=False)


def test_depth_forward_gives_nan():
    """a geometry blob from the depth / alpha forward is refused on the device: NaN absgrad and NaN gradients of visible Gaussians"""
    raw = _scene(4000, seed=9)
    leaves, rs, _ = _setup(raw, make_cameras(3, 64, 48)[1])
    d = torch.empty((1, 48, 64), device="cuda")
    with torch.no_grad():
        _, _, R, _, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves, depth=(1, d, None))
    grads, ag = _backward(rs, R, torch.ones(3, 48, 64, device="cuda"), leaves, radii, (geom, binning, img))
    vis = radii.cpu().numpy() > 0
    assert vis.any() and np.isnan(ag).all() and np.isnan(grads["xyz"][vis]).all()


# ------------------------------------------------------------------------------------------------
# 3. render()
# ------------------------------------------------------------------------------------------------
def _small(P=4000, W=208, H=160):
    pc = GaussianParams(_scene(P, seed=5), 3, "cuda")
    return pc, TorchCamera(make_cameras(3, W, H)[1], "cuda"), torch.tensor([0.1, 0.2, 0.3], device="cuda")


def _step(pc, tcam, bg, pipe=None, **kw):
    for p in pc.parameters():
        p.grad = None
    pkg = render(tcam, pc, pipe or pipeline_params(), bg, **kw)
    (pkg["render"] * torch.linspace(-1, 1, pkg["render"].numel(), device="cuda").view_as(pkg["render"])).sum().backward()
    return pkg, [p.grad.clone() for p in pc.parameters()]


def test_render_abs_mode(monkeypatch):
    pc, tcam, bg = _small()
    base, g0 = _step(pc, tcam, bg)
    assert not hasattr(base["viewspace_points"], "absgrad")
    c0 = dict(trace.counters)
    n0 = capi.launch_count()
    _step(pc, tcam, bg)
    per_step = capi.launch_count() - n0
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "abs")
    pkg, g1 = _step(pc, tcam, bg)
    assert set(pkg) == set(base)
    assert torch.equal(pkg["render"], base["render"]) and torch.equal(pkg["radii"], base["radii"])
    vp = pkg["viewspace_points"]
    assert vp.absgrad.shape == (vp.shape[0], 2) and vp.absgrad.dtype == torch.float32
    assert trace.counters.get("raw_backward_absgrad", 0) == c0.get("raw_backward_absgrad", 0) + 1
    assert trace.counters.get("render_absgrad", 0) == c0.get("render_absgrad", 0) + 1
    # .grad stays dL/dmeans2D, and the leaves get the default backward's gradients up to the order of float atomics
    for a, b in zip(g1 + [vp.grad], g0 + [base["viewspace_points"].grad]):
        torch.testing.assert_close(a, b, rtol=1e-3, atol=1e-5 * float(b.abs().max()))
    vis = pkg["radii"] > 0
    assert torch.all(vp.absgrad[~vis] == 0) and bool((vp.absgrad[vis].sum(1) > 0).any())
    # a permuted _xyz (create_from_pcd's layout) goes to the node as a contiguous copy; its gradient reaches the leaf
    xyz = pc._xyz.detach()
    pc._xyz = torch.nn.Parameter(xyz.t().contiguous().t())
    assert not pc._xyz.is_contiguous()
    perm, g2 = _step(pc, tcam, bg)
    assert torch.equal(perm["render"], base["render"]) and perm["viewspace_points"].absgrad.shape == vp.absgrad.shape
    torch.testing.assert_close(perm["viewspace_points"].absgrad, vp.absgrad, rtol=1e-4, atol=1e-6 * float(vp.absgrad.abs().max()))
    torch.testing.assert_close(g2[0], g1[0], rtol=1e-3, atol=1e-5 * float(g1[0].abs().max()))
    pc._xyz = torch.nn.Parameter(xyz)
    # no_grad and count_render are unchanged by the variable
    with torch.no_grad():
        ng = render(tcam, pc, pipeline_params(), bg)
    assert torch.equal(ng["render"], base["render"]) and not hasattr(ng["viewspace_points"], "absgrad")
    from lightgaussian_b200.renderer import count_render
    cr = count_render(tcam, pc, pipeline_params(), bg)
    assert not hasattr(cr["viewspace_points"], "absgrad") and "gaussians_count" in cr
    # unset again: the same launches and dictionary as the default step before
    monkeypatch.delenv("LGR_DENSIFY_GRAD")
    n2 = capi.launch_count()
    again, _ = _step(pc, tcam, bg)
    assert capi.launch_count() - n2 == per_step and set(again) == set(base)
    assert not hasattr(again["viewspace_points"], "absgrad")


def test_refusals_before_any_launch(monkeypatch):
    pc, tcam, bg = _small()
    pipe = pipeline_params()
    render(tcam, pc, pipe, bg)          # the fused path's one-time self-check runs here, not inside a refused call
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "abs")
    n0 = capi.launch_count()
    c0 = dict(trace.counters)

    def refuses(match, **kw):
        with pytest.raises(RuntimeError, match=match):
            render(tcam, pc, kw.pop("pipe", pipe), bg, **kw)
        assert capi.launch_count() == n0

    refuses("override_color", override_color=torch.rand(4000, 3, device="cuda"))
    refuses("convert_SHs_python", pipe=pipeline_params(convert_SHs_python=True))
    refuses("compute_cov3D_python", pipe=pipeline_params(compute_cov3D_python=True))
    monkeypatch.setenv("LGR_FUSED", "0")
    refuses("LGR_FUSED=0")
    monkeypatch.delenv("LGR_FUSED")
    pc.scaling_activation = lambda x: torch.exp(x)
    refuses("activations")
    del pc.scaling_activation
    monkeypatch.setenv("LGR_DETERMINISTIC", "1")
    refuses("deterministic")
    monkeypatch.delenv("LGR_DETERMINISTIC")
    capi.set_blend_mode(1)
    try:
        refuses("blend mode 1")
    finally:
        capi.set_blend_mode(0)
    enable_gradient_exchange(2)
    try:
        refuses("view-parallel")
    finally:
        enable_gradient_exchange(1)
    monkeypatch.setenv("LGR_SPARSE_SINGLE", "1")
    refuses("LGR_SPARSE_SINGLE")
    monkeypatch.delenv("LGR_SPARSE_SINGLE")
    refuses("depth=", depth="z")
    refuses("depth=", alpha=True)
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "absolute")
    refuses("LGR_DENSIFY_GRAD='absolute'")
    assert capi.launch_count() == n0
    assert trace.counters.get("render_fused", 0) == c0.get("render_fused", 0)
    # the library refuses deterministic mode and blend mode 1 itself, with nothing launched
    lib = capi.load()
    for setup, reset in ((lambda: capi.set_deterministic(True), lambda: capi.set_deterministic(False)),
                         (lambda: capi.set_blend_mode(1), lambda: capi.set_blend_mode(0))):
        setup()
        try:
            st = lib.lgr_backward_raw_absgrad(None, 1, 16, 1, None, None, None, None, None, None, None, None, None, None)
        finally:
            reset()
        assert st != 0
    assert capi.launch_count() == n0


# ------------------------------------------------------------------------------------------------
# 4. add_densification_stats
# ------------------------------------------------------------------------------------------------
def test_add_densification_stats_abs(monkeypatch):
    from lightgaussian_b200 import densify
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "abs")
    P = 20000
    pc = GaussianParams(_scene(P, seed=8, needles=1000), 3, "cuda")
    cams = make_cameras(20, 320, 240)
    bg = torch.zeros(3, device="cuda")
    gs = type("G", (), {})()
    gs.xyz_gradient_accum = torch.zeros((P, 1), device="cuda")
    gs.denom = torch.zeros((P, 1), device="cuda")
    acc_ref, den_ref = torch.zeros((P, 1), device="cuda"), torch.zeros((P, 1), device="cuda")
    for cam in cams:
        pkg, _ = _step(pc, TorchCamera(cam, "cuda"), bg)
        vp, f = pkg["viewspace_points"], pkg["visibility_filter"]
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            densify.add_densification_stats(gs, vp, f)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        acc_ref[f] += torch.norm(vp.absgrad[f], dim=-1, keepdim=True)
        den_ref[f] += 1
    assert torch.equal(gs.xyz_gradient_accum, acc_ref) and torch.equal(gs.denom, den_ref)
    assert gs.xyz_gradient_accum.sum() > 0
    with pytest.raises(RuntimeError, match="absgrad"):
        densify.add_densification_stats(gs, torch.zeros((P, 3), device="cuda"), f)


# ------------------------------------------------------------------------------------------------
# 5. the unmodified training script
# ------------------------------------------------------------------------------------------------
def test_train_densify_prune_opts_in(tmp_path, monkeypatch):
    reason = sh.stacks_available()
    if reason:
        pytest.skip(reason)
    from lightgaussian_b200.synth import write_colmap_dataset
    from tests.test_gpu_densify import _ply_count
    scene = make_scene(20000, sh_degree=3, seed=5, scale_mult=1.5)
    cams = make_cameras(24, 320, 240)
    gt = sh.render_ground_truth(scene["raw"], cams)
    data = os.path.join(str(tmp_path), "data")
    write_colmap_dataset(data, list(zip(cams, gt)), n_points=20000)
    last = 600
    res = {}
    for mode, thr in (("grad", "0.0002"), ("abs", "0.0008")):
        monkeypatch.setenv("LGR_DENSIFY_GRAD", mode)
        out, tr = os.path.join(str(tmp_path), f"tdp_{mode}"), os.path.join(str(tmp_path), f"tdp_{mode}.trace.json")
        sh.run("ours", ["train_densify_prune.py", "-s", data, "-m", out, "--eval", "-r", "1", "--port", str(6290 + len(res)),
                        "--iterations", str(last), "--densify_from_iter", "100", "--densification_interval", "100",
                        "--densify_until_iter", "550", "--opacity_reset_interval", "300", "--prune_iterations", "560",
                        "--position_lr_max_steps", str(last), "--test_iterations", "999999", "--save_iterations", str(last),
                        "--checkpoint_iterations", str(last), "--densify_grad_threshold", thr], trace=tr)
        t = sh.read_trace(tr)
        assert t.get("densify_native") == 4, t
        if mode == "abs":
            assert t.get("raw_backward_absgrad", 0) >= last and t.get("densify_stats_absgrad", 0) >= 500, t
        else:
            assert "raw_backward_absgrad" not in t, t
        test_idx = [k for k in range(len(cams)) if k % 8 == 0]
        psnr = sh.psnr_of_leaves(sh.load_checkpoint_leaves(os.path.join(out, f"chkpnt{last}.pth"))["leaves"], 3,
                                 [cams[k] for k in test_idx], [gt[k] for k in test_idx])
        res[mode] = (_ply_count(os.path.join(out, "point_cloud", f"iteration_{last}", "point_cloud.ply")), psnr)
    print("train_densify_prune (Gaussians, held-out PSNR): default grad 0.0002", res["grad"], "| abs 0.0008", res["abs"])
