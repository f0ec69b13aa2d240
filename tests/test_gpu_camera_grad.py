"""Camera gradients of the fused renderer (render(..., camera_grad=True), lgr_backward_raw_camera):
  1. dL/dviewmatrix, dL/dprojmatrix and dL/dcampos against the float64 arbiter (tests/camgrad_util.py) on the fused forward's own
     state, every entry: |ours - exact| <= RHO * sum_i |term_i|; the eight unread entries exactly 0 -- on the seeded configs in every
     single-GPU mode (kback 0/1/2, hand-written binning, blend mode 1, deterministic mode), with depth / alpha planes, at bench size, for
     a fully culled view and at P = 0;
  2. deterministic mode: bit-identical camera gradients run to run, leaf gradients equal to those without the camera request; in the
     default mode the leaf gradients keep test_gpu_leafgrad's float64 bounds;
  3. refusals before any launch, and the default path untouched;
  4. use: a perturbed pose converges back to the true one under Adam on an L1 loss."""
import json
import math
import os

import numpy as np
import pytest
import torch

from lightgaussian_b200 import capi, trace
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
from lightgaussian_b200.rasterizer import enable_gradient_exchange
from lightgaussian_b200.renderer import render
from lightgaussian_b200.synth import look_at, camera_from_pose, make_cameras, make_scene
from oracle.lgo import Oracle
from tests import util
from tests.camgrad_util import PROJ_LIVE, VIEW_LIVE, camera_grads_float64
from tests.test_gpu_leafgrad import BOUNDS, _activated, _leaves, _raw_np, _settings
from tests.util import CONFIGS, LEAVES, assert_every_element, leaf_grads_float64, read_state, view_from_camera

pytestmark = pytest.mark.gpu

RHO = 1e-5          # |ours - exact| <= RHO * sum_i |term_i|; the worst measured is 1.4e-6 (DESIGN.md section 7)
CAMS = ("world_view_transform", "full_proj_transform", "camera_center")
_WORST = {}


def _record(tag, worst):
    _WORST[tag] = worst
    out = os.environ.get("LGR_CAMGRAD_REPORT")
    if out:
        with open(out, "w") as f:
            json.dump(_WORST, f, indent=1)


def _cam_tensors(tcam):
    for n in CAMS:
        setattr(tcam, n, getattr(tcam, n).detach().clone().requires_grad_(True))
    return tcam


class _Mode:
    """one single-GPU configuration of the library, restored on exit"""

    def __init__(self, kback=0, bin_mode=None, blend=0, det=False):
        self.kback, self.bin_mode, self.blend, self.det = kback, bin_mode, blend, det

    def __enter__(self):
        capi.set_kback_mode(self.kback)
        capi.set_binning_mode(capi.DEFAULT_BINNING_MODE if self.bin_mode is None else self.bin_mode)
        capi.set_blend_mode(self.blend)
        if self.det:
            os.environ["LGR_DETERMINISTIC"] = "1"
        return self

    def __exit__(self, *exc):
        capi.set_kback_mode(0)
        capi.set_binning_mode(capi.DEFAULT_BINNING_MODE)
        capi.set_blend_mode(0)
        os.environ.pop("LGR_DETERMINISTIC", None)
        capi.set_deterministic(False)


MODES = {"kback0": _Mode(0), "kback1": _Mode(1), "kback2": _Mode(2), "hand_binning": _Mode(bin_mode=0), "blend1": _Mode(blend=1),
         "deterministic": _Mode(det=True)}


def _upstream(H, W, seed):
    rng = np.random.default_rng(seed)
    return np.sign(rng.standard_normal((3, H, W))).astype(np.float32)


def _render_backward(pc, tcam, bg, dpix, camera_grad=True, depth=None, alpha=False, gD=None, gA=None):
    for p in pc.parameters():
        p.grad = None
    for n in CAMS:
        getattr(tcam, n).grad = None
    pkg = render(tcam, pc, pipeline_params(), bg, depth=depth, alpha=alpha, camera_grad=camera_grad)
    outs, gs = [pkg["render"]], [torch.from_numpy(dpix).cuda()]
    if depth is not None:
        outs.append(pkg["depth"]); gs.append(torch.from_numpy(gD).cuda()[None])
    if alpha:
        outs.append(pkg["alpha"]); gs.append(torch.from_numpy(gA).cuda()[None])
    torch.autograd.backward(outs, gs)
    torch.cuda.synchronize()
    leaves = {n: getattr(pc, "_" + n).grad.clone() for n in LEAVES}
    leaves["means2D"] = pkg["viewspace_points"].grad.clone()
    cams = {n: (getattr(tcam, n).grad.clone() if getattr(tcam, n).grad is not None else None) for n in CAMS}
    return pkg, leaves, cams


def _state(view, tcam, pc, bg):
    from lightgaussian_b200.rasterizer import _forward_raw_native
    leaves = _leaves(pc)
    with torch.no_grad():
        _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, _settings(tcam, bg, pc.active_sh_degree), *leaves)
    P = leaves[0].shape[0]
    st = read_state(view, P, R, radii.cpu().numpy(), geom, binning, img) if P else {}
    st.update(radii=radii.cpu().numpy(), num_rendered=R)
    return st, leaves


def _check_cam(cams, exact, tag, rho=RHO):
    """every entry within rho * sum_i |term_i|; unread entries exactly 0; returns the worst ratio"""
    worst = 0.0
    for n, k in zip(CAMS, ("view", "proj", "campos")):
        g = cams[n]
        assert g is not None, f"{tag}: no gradient for {n}"
        assert g.dtype == torch.float32 and tuple(g.shape) == ((3,) if k == "campos" else (4, 4)), (tag, n, g.dtype, g.shape)
        a = g.detach().cpu().numpy().astype(np.float64).ravel()
        assert np.isfinite(a).all(), f"{tag} {n}: non-finite {a}"
        e, s = exact[k], exact["abs_" + k]
        err = np.abs(a - e)
        bound = rho * s
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(err == 0, 0.0, err / bound)
        worst = max(worst, float(r.max()))
        assert np.all(err <= bound), (f"{tag} {n}: entries outside {rho:g} sum|term|:\n ours  {a}\n exact {e}\n sum|term| {s}\n ratio {r}")
        if k != "campos":
            dead = [j for j in range(16) if j not in (VIEW_LIVE if k == "view" else PROJ_LIVE)]
            assert np.all(a[dead] == 0.0), f"{tag} {n}: unread entries not 0: {a[dead]}"
    _record(tag, worst)
    return worst


def _config(name):
    c = CONFIGS[name]
    scene = make_scene(c["P"], sh_degree=3, seed=c["seed"], scale_mult=c["scale_mult"])
    cam = util.inside_camera(c["W"], c["H"]) if c["cam"] == "inside" else make_cameras(5, c["W"], c["H"])[2]
    pc = GaussianParams(scene["raw"], 3, "cuda")
    pc.active_sh_degree = c["deg"]
    tcam = _cam_tensors(TorchCamera(cam, "cuda"))
    bg = torch.tensor(c["bg"], dtype=torch.float32, device="cuda")
    view = view_from_camera(cam, c["bg"], c["deg"], 1.0)
    return pc, tcam, bg, view, cam


# ------------------------------------------------------------------------------------------------
# 1. against float64
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CONFIGS))
def test_configs_every_mode(name, mode):
    pc, tcam, bg, view, cam = _config(name)
    with MODES[mode]:
        state, leaves = _state(view, tcam, pc, bg)
        dpix = _upstream(cam.image_height, cam.image_width, 3)
        _, got, cams = _render_backward(pc, tcam, bg, dpix)
    exact = camera_grads_float64(view, _raw_np(leaves), state, dpix, act=_activated(leaves, pc.active_sh_degree))
    _check_cam(cams, exact, f"{name}/{mode}")


def _depth_exact(view, view_black, tcam, pc, state, leaves, dpix, gD, gA, mode):
    """camera gradients of colour + depth + alpha: the colour call, plus the planes' blend backward (colours (v, 1, 0) on black, as
    test_gpu_depth_alpha's arbiter) whose dL/dmean2D and dL/dconic add to the camera terms, and dL/dv chained to dL/dz"""
    o = Oracle(double=True)
    P = leaves[0].shape[0]
    z = state["geom"]["depths"].astype(np.float64)
    vis = state["radii"] > 0
    v32 = state["geom"]["depths"] if mode == "z" else (1.0 / torch.from_numpy(state["geom"]["depths"])).numpy()
    vals = np.where(vis, v32, 0).astype(np.float32)
    cols = np.stack([vals, np.ones(P, np.float32), np.zeros(P, np.float32)], 1)
    dpix2 = np.stack([gD, gA, np.zeros_like(gD)]).astype(np.float32)
    act = _activated(leaves, pc.active_sh_degree)
    g2b, _ = util.oracle_backward_on_our_state(o, view_black, act, state, dpix2, colors=cols)
    dval = np.asarray(g2b["dL_dcolor"], np.float64).reshape(P, 3)[:, 0]
    dz = dval if mode == "z" else -dval / (z * z)
    return camera_grads_float64(view, _raw_np(leaves), state, dpix, act=act, extra2d=(g2b["dL_dmean2D"], g2b["dL_dconic"]),
                                dL_dz=np.where(vis, dz, 0.0))


@pytest.mark.parametrize("kback", [0, 1, 2])
@pytest.mark.parametrize("mode", ["z", "inverse"])
def test_depth_alpha_planes(mode, kback):
    pc, tcam, bg, view, cam = _config("outside")
    view_black = view_from_camera(cam, (0.0, 0.0, 0.0), view.sh_degree, 1.0)
    H, W = cam.image_height, cam.image_width
    rng = np.random.default_rng(9)
    gD, gA = np.sign(rng.standard_normal((H, W))).astype(np.float32), np.sign(rng.standard_normal((H, W))).astype(np.float32)
    dpix = _upstream(H, W, 4)
    with _Mode(kback):
        state, leaves = _state(view, tcam, pc, bg)
        _, _, cams = _render_backward(pc, tcam, bg, dpix, depth=mode, alpha=True, gD=gD, gA=gA)
    exact = _depth_exact(view, view_black, tcam, pc, state, leaves, dpix, gD, gA, mode)
    _check_cam(cams, exact, f"planes/{mode}/kback{kback}")


def test_bench_step():
    """3M Gaussians at 1080p (bench.py's scene, camera 0), an L1 loss's upstream gradient, default mode"""
    BW, BH = 1920, 1080
    scene = make_scene(3_000_000, sh_degree=3, seed=0)
    cam = make_cameras(16, BW, BH)[0]
    pc = GaussianParams(scene["raw"], 3, "cuda")
    del scene
    tcam = _cam_tensors(TorchCamera(cam, "cuda"))
    bg = torch.zeros(3, device="cuda")
    view = view_from_camera(cam, (0.0, 0.0, 0.0), 3, 1.0)
    state, leaves = _state(view, tcam, pc, bg)
    dpix = (_upstream(BH, BW, 5) / (3 * BH * BW)).astype(np.float32)
    _, _, cams = _render_backward(pc, tcam, bg, dpix)
    exact = camera_grads_float64(view, _raw_np(leaves), state, dpix, act=_activated(leaves, 3))
    _check_cam(cams, exact, "bench")


def test_fully_culled_view_and_empty_model():
    pc, tcam, bg, view, cam = _config("deg1")
    # looking away from the cloud: every Gaussian behind the near plane
    R, t = look_at((8.0, 0.0, 0.0), target=(16.0, 0.0, 0.0))
    away = _cam_tensors(TorchCamera(camera_from_pose(R, t, 96, 64, math.radians(60.0)), "cuda"))
    dpix = _upstream(64, 96, 6)
    pkg, leaves, cams = _render_backward(pc, away, bg, dpix)
    assert int((pkg["radii"] > 0).sum()) == 0
    for n in CAMS:
        assert torch.equal(cams[n], torch.zeros_like(cams[n])), n
    for n, g in leaves.items():
        assert torch.count_nonzero(g) == 0, n
    empty = GaussianParams({k: v[:0] for k, v in make_scene(8, sh_degree=3, seed=1)["raw"].items()}, 3, "cuda")
    tcam = _cam_tensors(TorchCamera(cam, "cuda"))
    _, _, cams = _render_backward(empty, tcam, bg, _upstream(cam.image_height, cam.image_width, 7))
    for n in CAMS:
        assert torch.equal(cams[n], torch.zeros_like(cams[n])), n


# ------------------------------------------------------------------------------------------------
# 2. determinism and the leaf gradients
# ------------------------------------------------------------------------------------------------
def test_deterministic_mode_is_bitwise_and_leaves_unchanged():
    pc, tcam, bg, view, cam = _config("outside")
    dpix = _upstream(cam.image_height, cam.image_width, 8)
    with _Mode(det=True):
        pkg = render(tcam, pc, pipeline_params(), bg, camera_grad=True)
        img = pkg["render"]
        runs = [torch.autograd.grad(img, [getattr(tcam, n) for n in CAMS], torch.from_numpy(dpix).cuda(), retain_graph=True)
                for _ in range(2)]                                   # two backward runs of one forward
        for a, b in zip(*runs):
            assert torch.equal(a, b) and torch.count_nonzero(a) > 0
        _, with_cam, _ = _render_backward(pc, tcam, bg, dpix, camera_grad=True)
        _, without, cams = _render_backward(pc, tcam, bg, dpix, camera_grad=False)
    assert all(c is None for c in cams.values())
    for n in with_cam:
        assert torch.equal(with_cam[n], without[n]), n


@pytest.mark.parametrize("name", ["outside", "deg1"])
def test_default_mode_leaf_grads_keep_their_float64_bounds(name):
    pc, tcam, bg, view, cam = _config(name)
    state, leaves = _state(view, tcam, pc, bg)
    dpix = _upstream(cam.image_height, cam.image_width, 10)
    _, got, cams = _render_backward(pc, tcam, bg, dpix)
    exact = leaf_grads_float64(view, _raw_np(leaves), state, dpix, act=_activated(leaves, pc.active_sh_degree))
    for n in LEAVES + ("means2D",):
        rho, alpha = BOUNDS[n]
        assert_every_element(got[n].cpu().numpy(), exact[n], rho, alpha, f"{name} {n}")


# ------------------------------------------------------------------------------------------------
# 3. refusals and the default path
# ------------------------------------------------------------------------------------------------
def test_refusals_before_any_launch(monkeypatch):
    pc, tcam, bg, view, cam = _config("deg1")
    pipe = pipeline_params()
    render(tcam, pc, pipe, bg)          # the fused path's one-time self-check runs here, not inside a refused call
    n0, c0 = capi.launch_count(), dict(trace.counters)

    def refuses(match, cam_=None, pipe_=None, **kw):
        with pytest.raises(RuntimeError, match=match):
            render(cam_ or tcam, pc, pipe_ or pipe, bg, camera_grad=True, **kw)
        assert capi.launch_count() == n0
        assert trace.counters == c0

    refuses("override_color", override_color=torch.zeros((pc._xyz.shape[0], 3), device="cuda"))
    refuses("convert_SHs_python", pipe_=pipeline_params(convert_SHs_python=True))
    monkeypatch.setenv("LGR_FUSED", "0")
    refuses("LGR_FUSED=0")
    monkeypatch.delenv("LGR_FUSED")
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "abs")
    refuses("LGR_DENSIFY_GRAD=abs")
    monkeypatch.delenv("LGR_DENSIFY_GRAD")
    monkeypatch.setenv("LGR_SPARSE_SINGLE", "1")
    refuses("LGR_SPARSE_SINGLE=1")
    monkeypatch.delenv("LGR_SPARSE_SINGLE")
    enable_gradient_exchange(2)
    try:
        refuses("view-parallel gradient exchange")
    finally:
        enable_gradient_exchange(1)
    bad = TorchCamera(cam, "cuda")
    bad.world_view_transform = bad.world_view_transform.double()
    refuses("world_view_transform must be a float32 CUDA tensor", cam_=bad)
    bad = TorchCamera(cam, "cuda")
    bad.camera_center = bad.camera_center.cpu()
    refuses("camera_center must be a float32 CUDA tensor", cam_=bad)
    bad = TorchCamera(cam, "cuda")
    bad.full_proj_transform = bad.full_proj_transform.reshape(16)
    refuses("full_proj_transform must be a float32 CUDA tensor of shape", cam_=bad)


def test_default_path_untouched():
    pc, tcam, bg, view, cam = _config("outside")
    dpix = _upstream(cam.image_height, cam.image_width, 11)
    keys = ("render_fused", "render_camera_grad", "raw_backward_camera", "render_depth_alpha", "raw_backward_plain")
    counts = []
    for _ in range(2):
        c0, n0 = {k: trace.counters.get(k, 0) for k in keys}, capi.launch_count()
        pkg, g0, cams = _render_backward(pc, tcam, bg, dpix, camera_grad=False)
        counts.append(({k: trace.counters.get(k, 0) - c0[k] for k in keys}, capi.launch_count() - n0))
    assert counts[0] == counts[1]
    assert counts[0][0] == {"render_fused": 1, "render_camera_grad": 0, "raw_backward_camera": 0, "render_depth_alpha": 0,
                            "raw_backward_plain": 0}
    assert all(c is None for c in cams.values())
    with torch.no_grad():
        a = render(tcam, pc, pipeline_params(), bg, camera_grad=True)
    assert torch.equal(a["render"], pkg["render"])
    c0 = dict(trace.counters)
    pkg2, g1, cams = _render_backward(pc, tcam, bg, dpix, camera_grad=True)
    assert torch.equal(pkg2["render"], pkg["render"])
    assert trace.counters.get("render_camera_grad", 0) == c0.get("render_camera_grad", 0) + 1
    assert trace.counters.get("raw_backward_camera", 0) == c0.get("raw_backward_camera", 0) + 1
    # only the camera tensors that require grad are differentiated
    tcam.camera_center = tcam.camera_center.detach()
    _, _, cams = _render_backward(pc, tcam, bg, dpix, camera_grad=True)
    assert cams["camera_center"] is None and cams["world_view_transform"] is not None


# ------------------------------------------------------------------------------------------------
# 4. pose recovery
# ------------------------------------------------------------------------------------------------
def _hat(w):
    z = torch.zeros((), dtype=w.dtype, device=w.device)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def test_pose_recovery():
    """~20k Gaussians, 320x240: from a pose 3 degrees and 3 % of the camera distance off, Adam on a 6-vector se(3) delta with the
    Gaussians frozen brings both errors down by at least 10x"""
    W, H = 320, 240
    scene = make_scene(20_000, sh_degree=3, seed=21, scale_mult=1.0)
    pc = GaussianParams(scene["raw"], 3, "cuda", requires_grad=False)
    true_cam = make_cameras(5, W, H)[1]
    bg = torch.zeros(3, device="cuda")
    tc = TorchCamera(true_cam, "cuda")
    with torch.no_grad():
        target = render(tc, pc, pipeline_params(), bg)["render"]
    V_true = tc.world_view_transform.double()
    K = torch.linalg.inv(V_true) @ tc.full_proj_transform.double()
    R_true, t_true = V_true.T[:3, :3], V_true.T[:3, 3]
    c_true = torch.linalg.inv(V_true)[3, :3]
    dist = float(torch.linalg.norm(c_true))
    g = torch.Generator().manual_seed(3)
    axis = torch.nn.functional.normalize(torch.randn(3, generator=g, dtype=torch.float64), dim=0).cuda()
    shift = torch.nn.functional.normalize(torch.randn(3, generator=g, dtype=torch.float64), dim=0).cuda()
    R0 = torch.linalg.matrix_exp(_hat(axis * math.radians(3.0))) @ R_true
    c0 = c_true + shift * 0.03 * dist
    t0 = -R0 @ c0

    def pose_of(delta):
        Rd = torch.linalg.matrix_exp(_hat(delta[:3]))
        R, t = Rd @ R0, Rd @ t0 + delta[3:]
        top = torch.cat([R, t[:, None]], 1)
        last = torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=torch.float64, device="cuda")
        return torch.cat([top, last], 0).T, R, t

    def errors(delta):
        with torch.no_grad():
            V, R, t = pose_of(delta)
            c = torch.linalg.inv(V)[3, :3]
            ang = torch.arccos(torch.clamp((torch.trace(R.T @ R_true) - 1) / 2, -1.0, 1.0))
            return math.degrees(float(ang)), float(torch.linalg.norm(c - c_true))

    delta = torch.zeros(6, dtype=torch.float64, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([delta], lr=2e-3)
    steps = 300
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, steps, eta_min=1e-5)
    e0 = errors(delta)
    cam = TorchCamera(true_cam, "cuda")
    for _ in range(steps):
        V, _, _ = pose_of(delta)
        Vf = V.float()
        cam.world_view_transform, cam.full_proj_transform = Vf, (V @ K).float()
        cam.camera_center = torch.linalg.inv(V)[3, :3].float()
        loss = (render(cam, pc, pipeline_params(), bg, camera_grad=True)["render"] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
    e1 = errors(delta)
    _record("pose_recovery", dict(start_deg=e0[0], start_dist=e0[1], end_deg=e1[0], end_dist=e1[1], camera_distance=dist))
    assert e1[0] <= e0[0] / 10 and e1[1] <= e0[1] / 10, (e0, e1)
