"""Depth and alpha planes of the fused renderer (render(depth=..., alpha=...), lgr_forward_raw_depth / lgr_backward_raw_depth):
  1. the forward bit for bit: every other output equals the default forward's; the depth plane equals channel 0 of the plain API
     path (bit-identical to the reference) rendering colours (v, v, v) on black, v = z or torch's 1 / z read from our geometry blob;
     alpha equals 1 - final_T -- at P = 0 and 1, ragged P, 1x1 to 1080p, a fully culled view, every binning mode, tile culling on/off;
  2. leaf gradients against float64, every element: the C oracle's backward on the fused forward's own state, once with the colours
     and dL/dpix, once with colours (v, 1, 0), dL/dpix = (dL/ddepth, dL/dalpha, 0) and a black background; dL/dv is that call's
     channel-0 colour gradient, chained to xyz by float64 torch autograd of v(xyz);
  3. the default path untouched, the combinations without a depth output refused before any launch, mismatched pairings NaN;
  4. use: fused AdamW on a depth + alpha L1 loss moves a perturbed scene toward a target's maps."""
import ctypes as C
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lightgaussian_b200 import capi, optim, trace
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
from lightgaussian_b200.rasterizer import (GaussianRasterizer, _forward_raw_native, _make_view, _raw_grads_struct, _raw_struct,
                                           enable_gradient_exchange, rasterize_raw_leaves_depth)
from lightgaussian_b200.renderer import render
from lightgaussian_b200.synth import make_cameras, make_scene
from oracle.lgo import Oracle
from tests import util
from tests.test_gpu_leafgrad import BOUNDS, GRADS, STACK_BOUNDS, _activated, _leaves, _raw_np, _settings, _stack_scene
from tests.util import LEAVES, assert_every_element, leaf_grads_from_activated, read_state, view_from_camera

pytestmark = pytest.mark.gpu

MODES = {"z": 1, "inverse": 2}


def _planes_forward(rs, leaves, mode, want_depth=True, want_alpha=True):
    H, W = int(rs.image_height), int(rs.image_width)
    d = torch.full((1, H, W), float("nan"), device="cuda") if want_depth else None
    a = torch.full((1, H, W), float("nan"), device="cuda") if want_alpha else None
    with torch.no_grad():
        out = _forward_raw_native(False, rs, *leaves, depth=(MODES.get(mode, 0), d, a))
    return out, d, a


def _values(z, radii, mode):
    """the depth value of every Gaussian as torch computes it from the geometry blob's z (0 for culled ones)"""
    zt = torch.from_numpy(z).cuda()
    v = zt if mode == "z" else 1.0 / zt
    return torch.where(torch.from_numpy(radii > 0).cuda(), v, torch.zeros_like(v))


def _api_channel0(rs_black, leaves, vals):
    xyz, dc, rest, scaling, rotation, opacity = leaves
    with torch.no_grad():
        color, _ = GaussianRasterizer(rs_black)(means3D=xyz, means2D=torch.zeros_like(xyz), opacities=torch.sigmoid(opacity),
                                                colors_precomp=vals[:, None].expand(-1, 3).contiguous(), scales=torch.exp(scaling),
                                                rotations=F.normalize(rotation))
    return color[0]


def _check_forward(cam, raw, mode="z"):
    P = raw["xyz"].shape[0]
    pc = GaussianParams(raw, 3, "cuda", requires_grad=False)
    leaves = _leaves(pc)
    tcam = TorchCamera(cam, "cuda")
    bg = torch.tensor([0.3, 0.2, 0.1], device="cuda")
    rs = _settings(tcam, bg, 3)
    view = view_from_camera(cam, (0.3, 0.2, 0.1), 3, 1.0)
    with torch.no_grad():
        base = _forward_raw_native(False, rs, *leaves)
    out, d, a = _planes_forward(rs, leaves, mode)
    _, _, R0, color0, radii0, geom0, bin0, img0, _ = base
    _, _, R, color, radii, geom, binning, img, _ = out
    assert R == R0
    assert torch.equal(color, color0) and torch.equal(radii, radii0)
    W, H = cam.image_width, cam.image_height
    if P == 0:
        assert torch.all(d == 0) and torch.all(a == 0) and torch.all(color == 0)
        return R
    s0 = read_state(view, P, R0, radii0.cpu().numpy(), geom0, bin0, img0)
    s = read_state(view, P, R, radii.cpu().numpy(), geom, binning, img)
    np.testing.assert_array_equal(s["final_T"], s0["final_T"])
    np.testing.assert_array_equal(s["n_contrib"], s0["n_contrib"])
    ft = torch.from_numpy(s["final_T"]).cuda().view(1, H, W)
    assert torch.equal(a, 1.0 - ft)
    rs_black = _settings(tcam, torch.zeros(3, device="cuda"), 3)
    vals = _values(s["geom"]["depths"], s["radii"], mode)
    ref = _api_channel0(rs_black, leaves, vals)
    assert torch.equal(d[0], ref), f"depth plane differs from the API path's blend in {(d[0] != ref).sum().item()} pixels"
    out2, d2, _ = _planes_forward(rs, leaves, "inverse" if mode == "z" else "z")
    s2 = read_state(view, P, out2[2], out2[4].cpu().numpy(), *out2[5:8])
    assert torch.equal(d2[0], _api_channel0(rs_black, leaves, _values(s2["geom"]["depths"], s2["radii"], "inverse" if mode == "z" else "z")))
    return R


# ------------------------------------------------------------------------------------------------
# 1. forward
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,wh", [(0, (17, 5)), (1, (64, 48)), (1, (1, 1)), (4099, (1, 1)), (4099, (17, 5)), (5003, (333, 211)),
                                  (20011, (1920, 1080))])
@pytest.mark.parametrize("mode", ["z", "inverse"])
def test_forward_planes_bit_for_bit(P, wh, mode):
    W, H = wh
    scene = make_scene(max(P, 1), sh_degree=3, seed=50 + P, scale_mult=2.0)
    raw = {k: v[:P] for k, v in scene["raw"].items()}
    R = _check_forward(make_cameras(4, W, H)[1], raw, mode)
    if P > 1000:
        assert R > 0


def test_forward_fully_culled_view():
    scene = make_scene(3001, sh_degree=3, seed=9)
    cam = make_cameras(3, 96, 64)[0]
    raw = dict(scene["raw"])
    raw["xyz"] = (1.5 * cam.camera_center[None, :] + 0.05 * np.random.default_rng(0).standard_normal((3001, 3))).astype(np.float32)
    assert _check_forward(cam, raw) == 0


@pytest.mark.parametrize("bin_mode", [0, 1, 2])
@pytest.mark.parametrize("cull", [True, False])
def test_forward_every_binning_mode(bin_mode, cull):
    scene = make_scene(30011, sh_degree=3, seed=11, scale_mult=1.5)
    capi.set_binning_mode(bin_mode)
    capi.set_tile_culling(cull)
    try:
        for i, (W, H) in enumerate([(640, 360), (1920, 1080)]):
            _check_forward(make_cameras(4, W, H)[i + 1], scene["raw"], ("z", "inverse")[i])
    finally:
        capi.set_binning_mode(capi.DEFAULT_BINNING_MODE)
        capi.set_tile_culling(True)


# ------------------------------------------------------------------------------------------------
# 2. gradients against float64
# ------------------------------------------------------------------------------------------------
def _exact(view, view_black, wv, raw, act, state, gC, gD, gA, mode):
    o = Oracle(double=True)
    P = raw["xyz"].shape[0]
    g2a, g3a = util.oracle_backward_on_our_state(o, view, act, state, gC)
    vals = _values(state["geom"]["depths"], state["radii"], mode).cpu().numpy()
    cols = np.stack([vals, np.ones(P, np.float32), np.zeros(P, np.float32)], 1).astype(np.float32)
    dpix2 = np.stack([gD, gA, np.zeros_like(gD)]).astype(np.float32)
    g2b, g3b = util.oracle_backward_on_our_state(o, view_black, act, state, dpix2, colors=cols)
    dval = torch.from_numpy(np.asarray(g2b["dL_dcolor"], np.float64).reshape(P, 3)[:, 0].copy())
    x = torch.from_numpy(np.asarray(raw["xyz"], np.float64)).requires_grad_(True)
    z = (torch.cat([x, torch.ones(P, 1, dtype=torch.float64)], 1) @ wv.double().cpu())[:, 2]
    ((z if mode == "z" else 1.0 / z) * dval).sum().backward()
    f = lambda k, a, b: np.asarray(a[k], np.float64) + np.asarray(b[k], np.float64)  # noqa: E731
    g = dict(dL_dmeans2D=np.asarray(g2a["dL_dmean2D"], np.float64) + np.asarray(g2b["dL_dmean2D"], np.float64),
             dL_dopacity=f("dL_dopacity", g2a, g2b), dL_dmeans3D=f("dL_dmeans3D", g3a, g3b) + x.grad.numpy(),
             dL_dsh=np.asarray(g3a["dL_dsh"], np.float64), dL_dscales=f("dL_dscales", g3a, g3b), dL_drotations=f("dL_drotations", g3a, g3b))
    return leaf_grads_from_activated(raw, g)


def _grads_through_render(pc, tcam, bg, mode, loss, gC, gD, gA):
    for p in pc.parameters():
        p.grad = None
    pkg = render(tcam, pc, pipeline_params(), bg, depth=mode, alpha=True)
    outs, gs = [], []
    if "color" in loss:
        outs.append(pkg["render"]); gs.append(torch.from_numpy(gC).cuda())
    if "depth" in loss:
        outs.append(pkg["depth"]); gs.append(torch.from_numpy(gD).cuda()[None])
    if "alpha" in loss:
        outs.append(pkg["alpha"]); gs.append(torch.from_numpy(gA).cuda()[None])
    n0 = trace.counters.get("raw_backward_depth", 0)
    torch.autograd.backward(outs, gs)
    torch.cuda.synchronize()
    assert trace.counters.get("raw_backward_depth", 0) == n0 + 1
    grads = {n: getattr(pc, "_" + n).grad.cpu().numpy() for n in LEAVES}
    grads["means2D"] = pkg["viewspace_points"].grad.cpu().numpy()
    return pkg, grads


def _check_grads(grads, exact, bounds, tag, radii):
    for n in GRADS:
        a = grads[n]
        assert np.isfinite(a).all(), f"{tag} {n}: non-finite entries"
        rho, alpha = bounds[n] if isinstance(bounds, dict) else bounds
        assert_every_element(a, exact[n], rho, alpha, f"{tag} {n}")
        assert np.all(a[radii <= 0] == 0), f"{tag} {n}: culled rows are not exact zeros"


LOSSES = {"depth": ("depth",), "alpha": ("alpha",), "all": ("color", "depth", "alpha")}


def _upstream(loss, H, W, seed):
    """random-sign upstream gradients, the shape of an L1 loss's (test_gpu_leafgrad's bounds are set for those)"""
    rng = np.random.default_rng(seed)
    g = lambda *s: np.sign(rng.standard_normal(s)).astype(np.float32)  # noqa: E731
    gC = g(3, H, W) if "color" in loss else np.zeros((3, H, W), np.float32)
    gD = g(H, W) if "depth" in loss else np.zeros((H, W), np.float32)
    gA = g(H, W) if "alpha" in loss else np.zeros((H, W), np.float32)
    return gC, gD, gA


@pytest.mark.parametrize("kback", [0, 1, 2])
@pytest.mark.parametrize("loss", list(LOSSES))
@pytest.mark.parametrize("mode", ["z", "inverse"])
def test_stack_grads_every_element(mode, loss, kback):
    """the blend ring's chunk / flush / wrap boundaries (test_gpu_leafgrad's stacks)"""
    raw, cam, _ = _stack_scene()
    pc = GaussianParams(raw, 3, "cuda")
    tcam = TorchCamera(cam, "cuda")
    bg = torch.tensor([0.3, 0.2, 0.1], device="cuda")
    view, view_black = view_from_camera(cam, (0.3, 0.2, 0.1), 3, 1.0), view_from_camera(cam, (0.0, 0.0, 0.0), 3, 1.0)
    leaves = _leaves(pc)
    out, _, _ = _planes_forward(_settings(tcam, bg, 3), leaves, mode)
    state = read_state(view, raw["xyz"].shape[0], out[2], out[4].cpu().numpy(), *out[5:8])
    gC, gD, gA = _upstream(LOSSES[loss], cam.image_height, cam.image_width, 7)
    capi.set_kback_mode(kback)
    try:
        _, grads = _grads_through_render(pc, tcam, bg, mode, LOSSES[loss], gC, gD, gA)
    finally:
        capi.set_kback_mode(0)
    exact = _exact(view, view_black, tcam.world_view_transform, _raw_np(leaves), _activated(leaves, 3), state, gC, gD, gA, mode)
    _check_grads(grads, exact, STACK_BOUNDS, f"stacks/{mode}/{loss}/kback{kback}", state["radii"])


def test_bench_size_grads_every_element():
    """3M Gaussians at 1080p (bench.py's scene, camera 0 and colour target), L1 losses on colour, depth and alpha, default backward"""
    BW, BH = 1920, 1080
    scene = make_scene(3_000_000, sh_degree=3, seed=0)
    cam = make_cameras(16, BW, BH)[0]
    pc = GaussianParams(scene["raw"], 3, "cuda")
    del scene
    tcam = TorchCamera(cam, "cuda")
    bg = torch.zeros(3, device="cuda")
    view = view_from_camera(cam, (0.0, 0.0, 0.0), 3, 1.0)
    leaves = _leaves(pc)
    out, d, a = _planes_forward(_settings(tcam, bg, 3), leaves, "z")
    state = read_state(view, leaves[0].shape[0], out[2], out[4].cpu().numpy(), *out[5:8])
    g = torch.Generator().manual_seed(1234)
    target = torch.rand(3, BH, BW, generator=g).cuda()
    t_depth, t_alpha = torch.rand(BH, BW, generator=g).cuda() * d.max(), torch.rand(BH, BW, generator=g).cuda()
    gC = (torch.sign(out[3] - target) / (3 * BH * BW)).cpu().numpy()
    gD = (torch.sign(d[0] - t_depth) / (BH * BW)).cpu().numpy()
    gA = (torch.sign(a[0] - t_alpha) / (BH * BW)).cpu().numpy()
    _, grads = _grads_through_render(pc, tcam, bg, "z", LOSSES["all"], gC, gD, gA)
    exact = _exact(view, view, tcam.world_view_transform, _raw_np(leaves), _activated(leaves, 3), state, gC, gD, gA, "z")
    _check_grads(grads, exact, BOUNDS, "bench/z/all", state["radii"])


# ------------------------------------------------------------------------------------------------
# 3. default path, refusals, mismatched pairings
# ------------------------------------------------------------------------------------------------
def _small():
    scene = make_scene(4000, sh_degree=3, seed=7, scale_mult=1.5)
    cam = make_cameras(4, 208, 160)[1]
    return GaussianParams(scene["raw"], 3, "cuda"), TorchCamera(cam, "cuda"), torch.tensor([0.1, 0.2, 0.3], device="cuda")


def test_default_path_untouched():
    pc, tcam, bg = _small()
    c0 = dict(trace.counters)
    pkg = render(tcam, pc, pipeline_params(), bg)
    assert set(pkg) == {"render", "viewspace_points", "visibility_filter", "radii"}
    pkg["render"].sum().backward()
    pkg2 = render(tcam, pc, pipeline_params(), bg, depth="z", alpha=True)
    assert torch.equal(pkg2["render"], pkg["render"]) and torch.equal(pkg2["radii"], pkg["radii"])
    assert pkg2["depth"].shape == (1, 160, 208) and pkg2["alpha"].shape == (1, 160, 208)
    (pkg2["render"].sum() + 0 * pkg2["radii"].sum()).backward()          # depth and alpha requested, outside the loss
    c1 = trace.counters
    assert c1.get("render_depth_alpha", 0) == c0.get("render_depth_alpha", 0) + 1
    assert c1.get("raw_backward_plain", 0) == c0.get("raw_backward_plain", 0) + 1
    assert c1.get("raw_backward_depth", 0) == c0.get("raw_backward_depth", 0)
    only_alpha = render(tcam, pc, pipeline_params(), bg, alpha=True)
    assert "depth" not in only_alpha and "alpha" in only_alpha


def test_combinations_without_depth_raise_before_any_launch(monkeypatch):
    pc, tcam, bg = _small()
    pipe = pipeline_params()
    render(tcam, pc, pipe, bg)          # the fused path's one-time self-check runs here, not inside a refused call
    n0 = capi.launch_count()

    def refuses(match, **kw):
        with pytest.raises(RuntimeError, match=match):
            render(tcam, pc, kw.pop("pipe", pipe), bg, depth="z", alpha=True, **kw)
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
    with pytest.raises(RuntimeError, match="expected None"):
        render(tcam, pc, pipe, bg, depth="disparity")
    rs = _settings(tcam, bg, 3)._replace(f_count=True)
    with pytest.raises(RuntimeError, match="count mode"):
        rasterize_raw_leaves_depth(pc._xyz, torch.zeros_like(pc._xyz), pc._features_dc, pc._features_rest, pc._scaling, pc._rotation,
                                   pc._opacity, rs, depth="z")
    assert capi.launch_count() == n0


def _depth_backward(rs, R, leaves, radii, blobs, mode, gD, gA):
    lib = capi.load()
    P, M = leaves[0].shape[0], 1 + leaves[2].shape[1]
    H, W = gD.shape
    outs = [torch.empty(t.shape, device="cuda") for t in leaves] + [torch.empty(P, 3, device="cuda")]
    dpix = torch.zeros(3, H, W, device="cuda")
    with torch.cuda.device(0):
        view, keep = _make_view(dpix.device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W,
                                rs.scale_modifier, rs.sh_degree, False, rs.debug)
        st = lib.lgr_backward_raw_depth(C.byref(view), P, M, int(R), C.byref(_raw_struct(*leaves)), radii.data_ptr(), blobs[0].data_ptr(),
                                        blobs[1].data_ptr(), blobs[2].data_ptr(), dpix.data_ptr(), mode, capi.ptr(gD), capi.ptr(gA),
                                        C.byref(_raw_grads_struct(*outs[:6])), outs[6].data_ptr(), capi.current_stream_ptr(dpix.device))
    capi.check(st, "lgr_backward_raw_depth")
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("pairing", [("none", 1), ("z", 2), ("inverse", 1), ("alpha", 1), ("z", 1)])
def test_mismatched_pairing_gives_nan(pairing):
    fwd, bwd = pairing
    pc, tcam, bg = _small()
    leaves = _leaves(pc)
    rs = _settings(tcam, bg, 3)
    H, W = 160, 208
    if fwd == "none":
        with torch.no_grad():
            out = _forward_raw_native(False, rs, *leaves)
    else:
        out, _, _ = _planes_forward(rs, leaves, None if fwd == "alpha" else fwd, want_depth=fwd != "alpha")
    R, radii, blobs = out[2], out[4], out[5:8]
    gD = torch.randn(H, W, device="cuda")
    outs = _depth_backward(rs, R, leaves, radii, blobs, bwd, gD, None)
    vis = radii > 0
    assert vis.sum() > 100
    if fwd in ("z", "inverse") and MODES[fwd] == bwd:
        assert all(torch.isfinite(t).all() for t in outs) and outs[0][vis].abs().sum() > 0
    else:
        # xyz, scaling, rotation, opacity and dL/dmeans2D of every visible Gaussian (the SH rows keep the exact zeros of clamped colour
        # channels)
        for t in (outs[0], outs[3], outs[4], outs[5], outs[6][:, :2]):
            assert torch.isnan(t[vis]).all()


# ------------------------------------------------------------------------------------------------
# 4. use
# ------------------------------------------------------------------------------------------------
def test_depth_alpha_loss_moves_a_perturbed_scene_toward_the_target():
    """a perturbed copy of a synthetic scene, trained on an L1 loss on its depth and alpha maps only (fused AdamW on xyz, opacity and
    scaling, 300 steps over 4 views), moves toward the target scene's maps"""
    P, W, H = 3000, 160, 120
    scene = make_scene(P, sh_degree=3, seed=21, scale_mult=2.0)
    cams = [TorchCamera(c, "cuda") for c in make_cameras(4, W, H)]
    bg = torch.zeros(3, device="cuda")
    pipe = pipeline_params()
    target = GaussianParams(scene["raw"], 3, "cuda", requires_grad=False)
    with torch.no_grad():
        tmaps = [render(c, target, pipe, bg, depth="z", alpha=True) for c in cams]
        tmaps = [(m["depth"].clone(), m["alpha"].clone()) for m in tmaps]
    rng = np.random.default_rng(5)
    raw = dict(scene["raw"])
    raw["xyz"] = (raw["xyz"] + 0.08 * rng.standard_normal(raw["xyz"].shape)).astype(np.float32)
    raw["opacity"] = (raw["opacity"] + 0.8 * rng.standard_normal(raw["opacity"].shape)).astype(np.float32)
    pc = GaussianParams(raw, 3, "cuda")
    opt = optim.FusedAdamW([{"params": [pc._xyz], "lr": 2e-3, "name": "xyz"}, {"params": [pc._opacity], "lr": 5e-2, "name": "opacity"},
                            {"params": [pc._scaling], "lr": 5e-3, "name": "scaling"}], lr=0.0, eps=1e-15)

    def loss_of(i):
        pkg = render(cams[i], pc, pipe, bg, depth="z", alpha=True)
        return (pkg["depth"] - tmaps[i][0]).abs().mean() + (pkg["alpha"] - tmaps[i][1]).abs().mean()

    with torch.no_grad():
        before = sum(float(loss_of(i)) for i in range(4))
    for step in range(300):
        opt.zero_grad(set_to_none=True)
        loss_of(step % 4).backward()
        opt.step()
    with torch.no_grad():
        after = sum(float(loss_of(i)) for i in range(4))
    print(f"\ndepth + alpha L1 over 4 views: {before:.5f} -> {after:.5f} ({after / before:.3f})")
    # measured on an H100: 0.597 -> 0.022 (0.037 of the start)
    assert after < 0.1 * before, (before, after)
