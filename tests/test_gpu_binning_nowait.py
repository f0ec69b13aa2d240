"""The default library binning sizes its blob from a running estimate and queues emit, tile sort, ranges and blend before the host
learns the instance count; it repeats them with an exact blob when the estimate was too small, and sorts pad keys past the count when it
was large.  Everything it produces must be bit-identical to the library binning that synchronises for the count first
(LGR_BINNING_SYNC=1) and to the hand-written exact binning (mode 1); gradients must agree up to the order of float atomics."""
import os

import numpy as np
import pytest
import torch

from lightgaussian_b200 import capi
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
from lightgaussian_b200.rasterizer import _C
from lightgaussian_b200.renderer import count_render, render
from lightgaussian_b200.synth import make_scene, make_cameras
from tests import util
from tests.util import CONFIGS, make_config, run_ours, view_from_camera, _t, _empty

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore():
    yield
    os.environ.pop("LGR_BINNING_SYNC", None)
    os.environ.pop("LGR_DETERMINISTIC", None)
    capi.set_deterministic(False)
    capi.set_binning_estimate(0)


def synced(fn, *a, **kw):
    os.environ["LGR_BINNING_SYNC"] = "1"
    try:
        return fn(*a, **kw)
    finally:
        os.environ.pop("LGR_BINNING_SYNC", None)


def _same(a, b):
    assert a["num_rendered"] == b["num_rendered"]
    assert a["num_listed"] == b["num_listed"]
    for k in ("radii", "ranges", "point_list", "n_contrib", "final_T", "color"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    np.testing.assert_array_equal(a["geom"]["sorted_ids"], b["geom"]["sorted_ids"])
    for k in ("gaussians_count", "important_score"):
        if k in a:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def _default(view, act, estimate, expect_repeat, **kw):
    """one default forward (+ backward) with the running estimate set to `estimate` instances; checks whether it repeated"""
    capi.set_binning_estimate(estimate)
    n0, s0 = capi.binning_overflows(), capi.forward_stream_syncs()
    out = run_ours(view, act, **kw)
    assert capi.binning_overflows() - n0 == (1 if expect_repeat else 0)
    assert capi.forward_stream_syncs() == s0
    return out


def _estimates(R):
    """(estimate, repeat expected): first view, a jump of more than 25 %, well under the estimate (pads sorted), about right"""
    cases = [(0, R > 4096), (10 * R + 100_000, False), (R + R // 4 + 4096, False)]
    if R > 8192:
        cases.append((int(R / 1.3), True))
    return cases


@pytest.mark.parametrize("count", [False, True])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_lists_and_image_match_the_synchronised_path(name, count):
    act, view, _ = make_config(name)
    ref = synced(run_ours, view, act, count=count)
    _same(run_ours(view, act, count=count, bin_mode=1), ref)
    for est, rep in _estimates(ref["num_listed"]):
        _same(_default(view, act, est, rep, count=count), ref)


@pytest.mark.parametrize("W,H", [(240, 272),       # 255 tiles: 8 key bits, the pad (255) one above the last tile
                                 (256, 256),       # 256 tiles: 9 key bits
                                 (16, 4112),       # 257 tiles, one tile wide
                                 (4080, 4112),     # 65 535 tiles: the widest 16-bit keys
                                 (4096, 4096)])    # 65 536 tiles: 32-bit keys (17 bits)
def test_key_width_boundaries(W, H):
    scene = make_scene(30_000, sh_degree=3, seed=5, scale_mult=2.0)
    view = view_from_camera(make_cameras(5, W, H)[1], (0.1, 0.2, 0.3), 3, 1.0)
    ref = synced(run_ours, view, scene["act"])
    assert ref["num_listed"] > 0
    _same(run_ours(view, scene["act"], bin_mode=1), ref)
    for est, rep in _estimates(ref["num_listed"]):
        _same(_default(view, scene["act"], est, rep), ref)


def test_nothing_listed():
    """R = 0 (every Gaussian below the alpha threshold everywhere, so tile culling lists none) with the reference's count > 0"""
    act, view, _ = make_config("outside")
    act = dict(act, opacities=np.full_like(act["opacities"], 1e-3))
    ref = synced(run_ours, view, act, count=True)
    assert ref["num_listed"] == 0 and ref["num_rendered"] > 0
    for est in (0, 100_000):
        got = _default(view, act, est, False, count=True)
        _same(got, ref)
        assert not got["ranges"].any()


def test_backward_after_repeated_and_padded_forwards():
    """the ring backward finds the records through the capacity word of the header, whether the blob was exact or padded"""
    act, view, dpix = make_config("outside")
    ref = synced(run_ours, view, act, dL_dpix=dpix)
    for est, rep in _estimates(ref["num_listed"]):
        got = _default(view, act, est, rep, dL_dpix=dpix)
        for k in ref["grads"]:
            assert util.rel_inf(got["grads"][k], ref["grads"][k]) <= 1e-4, (est, k)


def _weights(view, act):
    P = act["means3D"].shape[0]
    fx = torch.zeros(P, dtype=torch.int64, device="cuda")
    args = (_t(view.bg), _t(act["means3D"]), _empty(), _t(act["opacities"]), _t(act["scales"]), _t(act["rotations"]), view.scale_modifier,
            _empty(), _t(view.viewmatrix), _t(view.projmatrix), view.tanfovx, view.tanfovy, view.H, view.W, _t(act["shs"]), view.sh_degree,
            _t(view.campos), False, False)
    cnt, score, *_ = _C.count_gaussians(*args, True, blend_weight=fx)
    return cnt.cpu().numpy(), score.cpu().numpy(), fx.cpu().numpy()


def test_blending_weights_after_repeated_and_padded_forwards():
    act, view, _ = make_config("inside")
    ref = synced(_weights, view, act)
    R = synced(run_ours, view, act)["num_listed"]
    for est in (0, 10 * R + 100_000):
        capi.set_binning_estimate(est)
        for a, b in zip(_weights(view, act), ref):
            np.testing.assert_array_equal(a, b)


def _train_grads(pc, cam, pipe, bg, target):
    for p in pc.parameters():
        p.grad = None
    pkg = render(cam, pc, pipe, bg)
    (pkg["render"] - target).abs().mean().backward()
    return pkg["render"].detach().clone(), [p.grad.detach().clone() for p in pc.parameters()]


def test_training_view_gradients_and_no_host_synchronisation():
    """the fused training path (raw leaves): image bit-identical and leaf gradients equal up to atomics order; the default forwards,
    render and count_render, synchronise nothing while the synchronised and deterministic ones do once per forward"""
    P, W, H = 200_000, 640, 480
    scene = make_scene(P, sh_degree=3, seed=2)
    pc = GaussianParams(scene["raw"], 3, "cuda")
    cams = [TorchCamera(c, "cuda") for c in make_cameras(4, W, H)]
    pipe, bg = pipeline_params(), torch.tensor([0.1, 0.2, 0.3], device="cuda")
    target = torch.rand(3, H, W, generator=torch.Generator().manual_seed(3)).cuda()
    for cam in cams:
        img_ref, g_ref = synced(_train_grads, pc, cam, pipe, bg, target)
        for est in (0, 10_000_000):
            capi.set_binning_estimate(est)
            s0 = capi.forward_stream_syncs()
            img, g = _train_grads(pc, cam, pipe, bg, target)
            with torch.no_grad():
                count_render(cam, pc, pipe, bg)
            assert capi.forward_stream_syncs() == s0
            assert torch.equal(img, img_ref)
            for a, b in zip(g, g_ref):
                assert float((a - b).abs().max() / b.abs().max()) <= 1e-4
    s0 = capi.forward_stream_syncs()
    synced(_train_grads, pc, cams[0], pipe, bg, target)
    os.environ["LGR_DETERMINISTIC"] = "1"
    _train_grads(pc, cams[0], pipe, bg, target)
    os.environ.pop("LGR_DETERMINISTIC")
    assert capi.forward_stream_syncs() == s0 + 2


def test_bench_view_and_no_repeat_after_warm_up():
    """the bench workload (3M Gaussians, 1080p, 16 cameras): lists of one view bit-identical to the synchronised path, and after the
    bench's warm-up of 5 views no camera takes the repeat"""
    P, W, H = 3_000_000, 1920, 1080
    scene = make_scene(P, sh_degree=3, seed=0)
    cams_np = make_cameras(16, W, H)
    view = view_from_camera(cams_np[5], (0.0, 0.0, 0.0), 3, 1.0)
    ref = synced(run_ours, view, scene["act"])
    _same(_default(view, scene["act"], 0, True), ref)
    capi.set_binning_estimate(0)
    pc = GaussianParams(scene["raw"], 3, "cuda")
    cams = [TorchCamera(c, "cuda") for c in cams_np]
    pipe, bg = pipeline_params(), torch.zeros(3, device="cuda")
    with torch.no_grad():
        for cam in cams[:5]:
            render(cam, pc, pipe, bg)
        n0 = capi.binning_overflows()
        for k in range(32):
            render(cams[(5 + k) % 16], pc, pipe, bg)
    torch.cuda.synchronize()
    assert capi.binning_overflows() == n0
