"""render() on GaussianModel's raw leaves -- the path users train with and bench.py times: in-kernel activations (lgr_raw.cuh), the
ring blend backward that also clears the dense gradient rows (lgr_blend.cuh), K7+K8 on the compacted list -- against exact float64
leaf gradients, EVERY element (util.assert_every_element, no quantile):
  (a) the bench step itself at full size (3M Gaussians, 1080p, L1 loss) in every single-GPU backward mode,
  (b) stacks of Gaussians whose per-tile lists end on and next to the blend ring's chunk / flush / wrap boundaries,
  (c) ragged Gaussian counts, where the row clearing has a tail, with culled rows that must come back as exact zeros.
The float64 arbiter is the C oracle's backward evaluated on the fused forward's own state (util.leaf_grads_float64)."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lightgaussian_b200 import capi, trace
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
from lightgaussian_b200.synth import make_scene, make_cameras, camera_from_pose
from tests import util
from tests.util import LEAVES, assert_every_element, element_ratios, leaf_grads_float64, leaf_grads_from_activated, read_state, view_from_camera

pytestmark = pytest.mark.gpu

GRADS = LEAVES + ("means2D",)          # the six leaves and viewspace_points

# |ours - exact| <= rho |exact| + alpha max|exact|, per tensor.  The float64 value is exact for the kernels' forward state; what is left
# is float32 rounding (the reference's operation order, which the kernels keep) and the order of the float atomics.  The alphas are
# what that rounding needs on the bench step: the reference's own kernels need the same (xyz: 2.3e-5, scaling 1.2e-5, means2D 1.4e-5
# at rho = 1e-3, measured on an H100), test_bench_step_reference_kernels_pass_the_same_bounds checks that they pass.
BOUNDS = {"xyz": (1e-3, 5e-5), "features_dc": (1e-3, 1e-5), "features_rest": (1e-3, 1e-5), "scaling": (1e-3, 3e-5),
          "rotation": (1e-3, 2e-5), "opacity": (1e-3, 1e-5), "means2D": (1e-3, 3e-5)}
# stacks: at most a few hundred terms per pixel and few per Gaussian, so little cancels -- 10x tighter than the 1e-3 contract
STACK_BOUNDS = (1e-4, 1e-5)


# ------------------------------------------------------------------------------------------------
# shared pieces
# ------------------------------------------------------------------------------------------------
def _settings(tcam, bg, deg):
    from lightgaussian_b200.rasterizer import GaussianRasterizationSettings
    return GaussianRasterizationSettings(int(tcam.image_height), int(tcam.image_width), math.tan(tcam.FoVx * 0.5), math.tan(tcam.FoVy * 0.5),
                                         bg, 1.0, tcam.world_view_transform, tcam.full_proj_transform, deg, tcam.camera_center, False, False,
                                         False)


def _leaves(pc):
    return [p.detach() for p in pc.parameters()]


def _fused_state(view, rs, leaves):
    """the fused forward (lgr_forward_raw) of the leaves, with the state its backward reads"""
    from lightgaussian_b200.rasterizer import _forward_raw_native
    with torch.no_grad():
        _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
    st = read_state(view, leaves[0].shape[0], R, radii.cpu().numpy(), geom, binning, img) if leaves[0].shape[0] else {}
    st.update(color=color.cpu().numpy(), radii=radii.cpu().numpy(), num_rendered=R)
    return st


def _activated(leaves, deg):
    """the activated inputs exactly as torch computes them (the fused kernels reproduce these bit for bit)"""
    xyz, dc, rest, scaling, rotation, opacity = leaves
    M = (deg + 1) ** 2
    with torch.no_grad():
        act = dict(means3D=xyz, scales=torch.exp(scaling), rotations=F.normalize(rotation), opacities=torch.sigmoid(opacity),
                   shs=torch.cat((dc, rest), dim=1)[:, :M])
    return {k: np.ascontiguousarray(v.cpu().numpy()) for k, v in act.items()}


def _raw_np(leaves):
    return {n: np.ascontiguousarray(t.cpu().numpy()) for n, t in zip(LEAVES, leaves)}


def _check_all(grads, exact, bounds, tag, radii):
    worst = {}
    for n in GRADS:
        a = grads[n]
        assert a.shape == exact[n].shape, (tag, n, a.shape, exact[n].shape)
        assert np.isfinite(a).all(), f"{tag} {n}: non-finite entries"
        rho, alpha = bounds[n] if isinstance(bounds, dict) else bounds
        worst[n] = assert_every_element(a, exact[n], rho, alpha, f"{tag} {n}")
        assert np.all(a[radii <= 0] == 0), f"{tag} {n}: culled rows are not exact zeros"
    assert np.all(grads["means2D"][:, 2] == 0)
    return worst


# ------------------------------------------------------------------------------------------------
# (a) the bench step at full size
# ------------------------------------------------------------------------------------------------
BW, BH = 1920, 1080
MODES = ("default", "kback_dense", "kback_separate_zero", "sparse_single")


def _student(raw):
    """GaussianModel.onedownSHdegree()'s leaf for 3 -> 2: a NON-contiguous [P,8,3] view of a [P,15,3] tensor (as test_gpu_fused.py)"""
    pc = GaussianParams(raw, 3, "cuda")
    full = pc._features_rest.clone().detach()
    pc._features_rest = full[:, :8, :]
    pc._features_rest.requires_grad = True
    pc.max_sh_degree, pc.active_sh_degree = 2, 2
    return pc


def _train_step(pc, tcam, bg, target):
    """trainstep.train_view with bench.py's loss; returns the image, radii, the upstream gradient the rasterizer received and the
    gradients of the six leaves and of viewspace_points"""
    from lightgaussian_b200.loss import l1_loss
    from lightgaussian_b200.renderer import render
    from lightgaussian_b200.trainstep import train_view
    for p in pc.parameters():
        p.grad = None
    seen = {}

    def render_fn(*a):
        pkg = render(*a)
        seen["pkg"] = pkg
        pkg["render"].register_hook(lambda g: seen.__setitem__("dpix", g.detach().clone()))
        return pkg
    n0 = trace.counters.get("render_fused", 0)
    train_view(render_fn, tcam, pc, pipeline_params(), bg, target, loss_fn=l1_loss)
    torch.cuda.synchronize()
    assert trace.counters.get("render_fused", 0) == n0 + 1, "render() did not take the fused path"
    pkg = seen["pkg"]
    grads = {n: getattr(pc, "_" + n).grad.cpu().numpy() for n in LEAVES}
    grads["means2D"] = pkg["viewspace_points"].grad.cpu().numpy()
    return pkg["render"].detach().cpu().numpy(), pkg["radii"].cpu().numpy(), seen["dpix"].cpu().numpy(), grads


def _with_mode(mode, fn):
    old = os.environ.get("LGR_SPARSE_SINGLE")
    capi.set_kback_mode({"kback_dense": 1, "kback_separate_zero": 2}.get(mode, 0))
    if mode == "sparse_single":
        os.environ["LGR_SPARSE_SINGLE"] = "1"
    try:
        return fn()
    finally:
        capi.set_kback_mode(0)
        if old is None:
            os.environ.pop("LGR_SPARSE_SINGLE", None)
        else:
            os.environ["LGR_SPARSE_SINGLE"] = old


@pytest.fixture(scope="module", params=["deg3", "student"])
def bench_step(request):
    """bench.py's step (bench.py:366-421): make_scene(3M, seed 0), camera 0 of 16 at 1920x1080, black background, the first target of
    Generator().manual_seed(1234), lightgaussian_b200.loss.l1_loss -- plus the float64 leaf gradients of that step, computed once."""
    scene = make_scene(3_000_000, sh_degree=3, seed=0)
    cam = make_cameras(16, BW, BH)[0]
    tcam = TorchCamera(cam, "cuda")
    bg = torch.zeros(3, device="cuda")
    target = torch.rand(3, BH, BW, generator=torch.Generator().manual_seed(1234)).cuda()
    pc = _student(scene["raw"]) if request.param == "student" else GaussianParams(scene["raw"], 3, "cuda")
    del scene
    deg = pc.active_sh_degree
    view = view_from_camera(cam, (0.0, 0.0, 0.0), deg, 1.0)
    img, radii, dpix, grads = _train_step(pc, tcam, bg, target)
    # the upstream gradient is the L1's sign(img - target) / N, not Gaussian noise
    np.testing.assert_allclose(dpix, np.sign(img - target.cpu().numpy()) / np.float32(3 * BH * BW), rtol=1e-6, atol=0)
    leaves = _leaves(pc)
    state = _fused_state(view, _settings(tcam, bg, deg), leaves)
    raw, act = _raw_np(leaves), _activated(leaves, deg)      # raw features_rest: a contiguous copy of the student's view
    exact = leaf_grads_float64(view, raw, state, dpix, act=act)
    yield dict(case=request.param, pc=pc, tcam=tcam, bg=bg, target=target, view=view, img=img, radii=radii, dpix=dpix, grads=grads,
               state=state, raw=raw, act=act, exact=exact)


@pytest.mark.parametrize("mode", MODES)
def test_bench_step_leaf_grads_every_element(bench_step, mode):
    s = bench_step
    # the state the oracle used is the training forward's: image and radii bit-identical
    np.testing.assert_array_equal(s["state"]["color"], s["img"])
    np.testing.assert_array_equal(s["state"]["radii"], s["radii"])
    assert (s["radii"] > 0).sum() > 100_000
    if mode == "default":
        grads = s["grads"]
    else:
        img, radii, dpix, grads = _with_mode(mode, lambda: _train_step(s["pc"], s["tcam"], s["bg"], s["target"]))
        np.testing.assert_array_equal(img, s["img"])
        np.testing.assert_array_equal(radii, s["radii"])
        np.testing.assert_array_equal(dpix, s["dpix"])
    worst = _check_all(grads, s["exact"], BOUNDS, f"{s['case']}/{mode}", s["radii"])
    print(f"\n{s['case']}/{mode}: worst ratio to the bound " + ", ".join(f"{n} {w:.3f}" for n, w in worst.items()))


@pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref/libref_rasterizer.so not built (needs the reference checkout)")
def test_bench_step_reference_kernels_pass_the_same_bounds(bench_step):
    """the bounds are fair: the reference's own kernels, on the same activated inputs and upstream gradient (their gradients mapped to
    the leaves by the same chain rule), pass them too.  The forward is bit-identical to ours."""
    s = bench_step
    ref = util.run_ref(s["view"], s["act"], dL_dpix=s["dpix"])
    np.testing.assert_array_equal(ref["color"], s["img"])
    np.testing.assert_array_equal(ref["radii"], s["radii"])
    rg = leaf_grads_from_activated(s["raw"], ref["grads"])
    lines = []
    for n in GRADS:
        rho, alpha = BOUNDS[n]
        wo = float(element_ratios(s["grads"][n], s["exact"][n], rho, alpha).max())
        wr = float(element_ratios(rg[n], s["exact"][n], rho, alpha).max())
        lines.append(f"  {n:14s} rho {rho:g} alpha {alpha:g}: worst ratio ours {wo:.3f}  reference kernels {wr:.3f}")
    print(f"\n{s['case']}: worst |err| / (rho |exact| + alpha max|exact|) against float64\n" + "\n".join(lines))
    for n in GRADS:
        assert_every_element(rg[n], s["exact"][n], *BOUNDS[n], f"reference kernels {s['case']} {n}")


# ------------------------------------------------------------------------------------------------
# (b) blend-ring boundaries: one stack of N Gaussians per tile
# ------------------------------------------------------------------------------------------------
STACKS = (1, 15, 16, 17, 31, 32, 33, 127, 128, 129, 255, 256, 257, 600)   # around BL_CH = 32, BL_FLUSH = 16, the 4 x 32 ring
CORNER_N = 40
SW, SHT = 96, 64                        # 6 x 4 tiles; the corner stack sits at the corner of tiles (4,2), (5,2), (4,3), (5,3)
CORNER_TILES = {(4, 2), (5, 2), (4, 3), (5, 3)}


def _stack_scene(seed=0):
    """Gaussians on the camera ray through one screen point, at strictly increasing depth, each about 1.2 px wide on screen (radius
    <= 7 px: inside its 16x16 tile).  Opacity ~0.1: centre pixels saturate (T < 1e-4) after ~90 Gaussians, edge pixels never."""
    rng = np.random.default_rng(seed)
    fovx = math.radians(60.0)
    cam = camera_from_pose(np.eye(3), np.zeros(3), SW, SHT, fovx)
    tanx, tany = cam.tanfovx, cam.tanfovy
    focal = SW / (2.0 * tanx)
    free = [(tx, ty) for ty in range(SHT // 16) for tx in range(SW // 16) if (tx, ty) not in CORNER_TILES]
    # centres off the pixel grid's symmetry (so that dL/dmean2D does not cancel to nothing), radius <= 7 px keeps a stack in its tile
    off = rng.uniform(-0.4, 0.4, (len(STACKS) + 1, 2))
    centres = [((16 * tx + 7.5 + off[i, 0], 16 * ty + 7.5 + off[i, 1]), n) for i, ((tx, ty), n) in enumerate(zip(free, STACKS))]
    centres.append(((79.5 + off[-1, 0], 47.5 + off[-1, 1]), CORNER_N))
    xyz, scaling = [], []
    for (cx, cy), n in centres:
        ray = np.array([(2 * cx + 1 - SW) / SW * tanx, (2 * cy + 1 - SHT) / SHT * tany, 1.0])
        z = np.linspace(2.0, 4.0, n + 2)[1:-1]                       # strictly increasing depth
        xyz.append(ray[None, :] * z[:, None])
        sig = 1.2 * z / focal                                        # world size of 1.2 px at depth z
        scaling.append(np.log(sig[:, None] * rng.uniform(0.7, 1.3, (n, 3))))
    P = sum(n for _, n in centres)
    op = rng.uniform(0.06, 0.16, (P, 1))
    raw = dict(xyz=np.concatenate(xyz).astype(np.float32), scaling=np.concatenate(scaling).astype(np.float32),
               rotation=rng.standard_normal((P, 4)).astype(np.float32), opacity=np.log(op / (1 - op)).astype(np.float32),
               features_dc=(0.8 * rng.standard_normal((P, 1, 3))).astype(np.float32),
               features_rest=(0.2 * rng.standard_normal((P, 15, 3))).astype(np.float32))
    return raw, cam, free


@pytest.mark.parametrize("dpix_kind", ["constant", "random_sign"])
def test_blend_ring_boundaries(dpix_kind):
    raw, cam, free = _stack_scene()
    pc = GaussianParams(raw, 3, "cuda")
    tcam = TorchCamera(cam, "cuda")
    bg = torch.tensor([0.3, 0.2, 0.1], device="cuda")
    view = view_from_camera(cam, (0.3, 0.2, 0.1), 3, 1.0)
    leaves = _leaves(pc)
    state = _fused_state(view, _settings(tcam, bg, 3), leaves)
    # the construction: tile lists of exactly N (tile culling keeps every instance), n_contrib on both sides of 32 and 128
    gx = SW // 16
    lens = (state["ranges"][:, 1].astype(np.int64) - state["ranges"][:, 0]).reshape(SHT // 16, gx)
    want = np.zeros_like(lens)
    for (tx, ty), n in zip(free, STACKS):
        want[ty, tx] = n
    for tx, ty in CORNER_TILES:
        want[ty, tx] = CORNER_N
    np.testing.assert_array_equal(lens, want)
    assert (state["radii"] > 0).all() and state["radii"].max() <= 7
    nc = state["n_contrib"]
    assert (nc[(nc > 0) & (nc < 32)]).size and (nc[(nc > 32) & (nc < 128)]).size and (nc[nc > 128]).size
    assert ((nc > 0) & (nc % 32 == 0)).any()                         # some pixels end exactly on a chunk boundary
    assert (state["final_T"][nc > 0] < 1e-3).any()                   # some pixels saturated inside a stack
    if dpix_kind == "constant":
        dpix = np.full((3, SHT, SW), 0.5, np.float32)
    else:
        dpix = np.sign(np.random.default_rng(1).standard_normal((3, SHT, SW))).astype(np.float32)
    from lightgaussian_b200.renderer import render
    pkg = render(tcam, pc, pipeline_params(), bg)
    np.testing.assert_array_equal(pkg["render"].detach().cpu().numpy(), state["color"])
    pkg["render"].backward(torch.from_numpy(dpix).cuda())
    grads = {n: getattr(pc, "_" + n).grad.cpu().numpy() for n in LEAVES}
    grads["means2D"] = pkg["viewspace_points"].grad.cpu().numpy()
    exact = leaf_grads_float64(view, raw, state, dpix, act=_activated(leaves, 3))
    _check_all(grads, exact, STACK_BOUNDS, f"stacks/{dpix_kind}", state["radii"])


# ------------------------------------------------------------------------------------------------
# (c) row clearing at ragged P
# ------------------------------------------------------------------------------------------------
def _backward_into(rs, R, dpix, leaves, radii, blobs, outs):
    """lgr_backward_raw (what the fused node's backward calls on one GPU) writing into the given output tensors"""
    import ctypes as C
    from lightgaussian_b200.rasterizer import _make_view, _raw_struct, _raw_grads_struct
    lib = capi.load()
    P, M = leaves[0].shape[0], 1 + leaves[2].shape[1]
    H, W = dpix.shape[1], dpix.shape[2]
    with torch.cuda.device(dpix.device):
        view, keep = _make_view(dpix.device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W,
                                rs.scale_modifier, rs.sh_degree, False, rs.debug)
        st = lib.lgr_backward_raw(C.byref(view), P, M, int(R), C.byref(_raw_struct(*leaves)), radii.data_ptr(), blobs[0].data_ptr(),
                                  blobs[1].data_ptr(), blobs[2].data_ptr(), dpix.data_ptr(), C.byref(_raw_grads_struct(*outs[:6])),
                                  outs[6].data_ptr(), capi.current_stream_ptr(dpix.device))
    capi.check(st, "lgr_backward_raw")
    torch.cuda.synchronize()


@pytest.mark.parametrize("wh", [(1, 1), (17, 5), (64, 48)])
@pytest.mark.parametrize("P", [1, 2, 3, 5, 4097, 4099])
def test_row_clearing_at_ragged_P(P, wh):
    """tile_zero_rows clears [0, P) in runs of 4 rows with bulk stores and the last P % 4 rows with plain stores.  The gradient
    buffers are handed to the backward filled with NaN: every row the kernels do not write must still come back as exact zeros.
    Odd rows and the last row sit behind the camera (culled); P is below and above the tile count."""
    from lightgaussian_b200.rasterizer import _forward_raw_native
    W, H = wh
    scene = make_scene(P, sh_degree=3, seed=300 + P, scale_mult=3.0)
    cam = make_cameras(3, W, H)[1]
    raw = dict(scene["raw"])
    behind = np.zeros(P, bool)
    behind[1::2] = True
    if P >= 2:
        behind[-1] = True
    rng = np.random.default_rng(P)
    raw["xyz"] = raw["xyz"].copy()
    raw["xyz"][behind] = (1.5 * cam.camera_center[None, :] + 0.1 * rng.standard_normal((int(behind.sum()), 3))).astype(np.float32)
    pc = GaussianParams(raw, 3, "cuda", requires_grad=False)
    leaves = _leaves(pc)
    tcam = TorchCamera(cam, "cuda")
    bg = torch.tensor([0.1, 0.2, 0.3], device="cuda")
    rs = _settings(tcam, bg, 3)
    view = view_from_camera(cam, (0.1, 0.2, 0.3), 3, 1.0)
    with torch.no_grad():
        _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
    radii_np = radii.cpu().numpy()
    assert np.all(radii_np[behind] == 0)
    dpix = torch.randn(3, H, W, generator=torch.Generator().manual_seed(P + W)).cuda()
    nan = lambda *s: torch.full(s, float("nan"), device="cuda")  # noqa: E731
    outs = [nan(P, 3), nan(P, 1, 3), nan(P, 15, 3), nan(P, 3), nan(P, 4), nan(P, 1), nan(P, 3)]
    _backward_into(rs, R, dpix, leaves, radii, (geom, binning, img), outs)
    grads = {n: t.cpu().numpy() for n, t in zip(GRADS, outs)}
    for n in GRADS:
        assert np.all(grads[n][radii_np <= 0] == 0), f"{n}: rows of culled Gaussians are not exact zeros"
    if R == 0:
        for n in GRADS:
            assert np.all(grads[n] == 0), n
        return
    state = read_state(view, P, R, radii_np, geom, binning, img)
    exact = leaf_grads_float64(view, _raw_np(leaves), state, dpix.cpu().numpy(), act=_activated(leaves, 3))
    _check_all(grads, exact, BOUNDS, f"P={P} {W}x{H}", radii_np)
