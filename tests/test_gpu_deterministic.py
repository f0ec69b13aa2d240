"""Deterministic mode (lgr_set_deterministic; on when torch.are_deterministic_algorithms_enabled() or LGR_DETERMINISTIC=1):
  * the forward is bit-identical to the default mode's (images, radii, final_T, n_contrib, per-tile lists, counts, scores);
  * every leaf gradient is bit-identical over repeats of the same forward + backward, on other streams and next to other GPU work;
  * the gradients still meet test_gpu_leafgrad.py's per-element bounds against float64;
  * a backward runs in the mode of its forward; combinations without a deterministic path raise before any launch;
  * the VecTree EMA k-means is bit-identical between runs.
For each repeatability case the number of elements that differ between two DEFAULT-mode runs is printed (not asserted): it shows
that the input exercises the float atomics the deterministic mode replaces."""
import contextlib
import os

import numpy as np
import pytest
import torch

from lightgaussian_b200 import capi
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
from lightgaussian_b200.synth import make_scene, make_cameras
from tests import util
from tests.test_gpu_leafgrad import (BOUNDS, STACK_BOUNDS, BW, BH, GRADS, _activated, _check_all, _fused_state, _leaves, _raw_np,
                                     _settings, _stack_scene, _student, _train_step, _with_mode)
from tests.util import LEAVES, element_ratios, leaf_grads_float64, view_from_camera

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def det(on=True):
    old = os.environ.get("LGR_DETERMINISTIC")
    os.environ["LGR_DETERMINISTIC"] = "1" if on else "0"
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("LGR_DETERMINISTIC", None)
        else:
            os.environ["LGR_DETERMINISTIC"] = old
        capi.set_deterministic(False)


def _n_diff(a, b):
    return int(sum((x != y).sum() for x, y in zip(a.values(), b.values())))


def _repeat(run, tag, n=3):
    """run() -> {name: ndarray}; n runs in deterministic mode must agree bitwise, two default-mode runs are compared for the print"""
    with det(False):
        d0, d1 = run(), run()
    with det(True):
        runs = [run() for _ in range(n)]
    for r in runs[1:]:
        for k in runs[0]:
            assert np.array_equal(runs[0][k], r[k]), f"{tag}: {k} differs between deterministic runs"
    print(f"\n{tag}: {_n_diff(d0, d1)} elements differ between two default-mode runs; deterministic runs bit-identical")
    return runs[0], d0


def _leaf_step(pc, tcam, bg, dpix, settings=None):
    """render() + backward with the given upstream gradient; the leaves' and viewspace_points' gradients"""
    from lightgaussian_b200.renderer import render
    for p in pc.parameters():
        p.grad = None
    pkg = render(tcam, pc, pipeline_params(**(settings or {})), bg)
    pkg["render"].backward(dpix)
    torch.cuda.synchronize()
    g = {n: getattr(pc, "_" + n).grad.cpu().numpy() for n in LEAVES}
    if pkg["viewspace_points"].grad is not None:
        g["means2D"] = pkg["viewspace_points"].grad.cpu().numpy()
    g["image"] = pkg["render"].detach().cpu().numpy()
    return g


# ------------------------------------------------------------------------------------------------
# 1. forward unchanged
# ------------------------------------------------------------------------------------------------
def _forward_fields(view, act, count):
    o = util.run_ours(view, act, count=count)
    keys = ["color", "radii", "final_T", "n_contrib", "ranges", "point_list", "num_rendered"]
    if count:
        keys += ["gaussians_count", "important_score"]
    return {k: np.asarray(o[k]) for k in keys}


@pytest.mark.parametrize("count", [False, True])
@pytest.mark.parametrize("name", sorted(util.CONFIGS))
def test_forward_bit_identical_small(name, count):
    act, view, _ = util.make_config(name)
    with det(False):
        a = _forward_fields(view, act, count)
    with det(True):
        b = _forward_fields(view, act, count)
    for k in a:
        assert np.array_equal(a[k], b[k]), f"{name}: {k} differs between default and deterministic mode"


@pytest.mark.parametrize("count", [False, True])
def test_forward_bit_identical_bench_size(count):
    scene = make_scene(3_000_000, sh_degree=3, seed=0)
    cam = make_cameras(16, BW, BH)[0]
    view = view_from_camera(cam, (0.0, 0.0, 0.0), 3, 1.0)
    act = scene["act"]
    del scene
    with det(False):
        a = _forward_fields(view, act, count)
    with det(True):
        b = _forward_fields(view, act, count)
    assert a["point_list"].size > 1_000_000
    for k in a:
        assert np.array_equal(a[k], b[k]), f"bench size: {k} differs between default and deterministic mode"


# ------------------------------------------------------------------------------------------------
# 2 + 3. the bench step: repeatable in every single-GPU backward mode, and still within the float64 bounds
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["deg3", "student"])
def bench(request):
    scene = make_scene(3_000_000, sh_degree=3, seed=0)
    cam = make_cameras(16, BW, BH)[0]
    tcam = TorchCamera(cam, "cuda")
    bg = torch.zeros(3, device="cuda")
    target = torch.rand(3, BH, BW, generator=torch.Generator().manual_seed(1234)).cuda()
    pc = _student(scene["raw"]) if request.param == "student" else GaussianParams(scene["raw"], 3, "cuda")
    del scene
    yield dict(case=request.param, pc=pc, tcam=tcam, bg=bg, target=target, cam=cam)


def _bench_grads(b):
    img, radii, dpix, grads = _train_step(b["pc"], b["tcam"], b["bg"], b["target"])
    grads = dict(grads)
    grads["image"] = img
    return grads


@pytest.mark.parametrize("mode", ["default", "kback_dense", "kback_separate_zero", "sparse_single"])
def test_bench_step_repeatable(bench, mode):
    if bench["case"] == "student" and mode != "default":
        pytest.skip("the student runs in the default backward mode only")
    _repeat(lambda: _with_mode(mode, lambda: _bench_grads(bench)), f"bench {bench['case']}/{mode}")


def test_bench_step_within_float64_bounds(bench):
    """deterministic-mode gradients against the float64 oracle on every element, with test_gpu_leafgrad.py's bounds"""
    b = bench
    pc, deg = b["pc"], b["pc"].active_sh_degree
    with det(False):
        img, radii, dpix, g_def = _train_step(pc, b["tcam"], b["bg"], b["target"])
    with det(True):
        img_d, radii_d, dpix_d, g_det = _train_step(pc, b["tcam"], b["bg"], b["target"])
    assert np.array_equal(img, img_d) and np.array_equal(radii, radii_d) and np.array_equal(dpix, dpix_d)
    view = view_from_camera(b["cam"], (0.0, 0.0, 0.0), deg, 1.0)
    leaves = _leaves(pc)
    state = _fused_state(view, _settings(b["tcam"], b["bg"], deg), leaves)
    exact = leaf_grads_float64(view, _raw_np(leaves), state, dpix, act=_activated(leaves, deg))
    _check_all(g_det, exact, BOUNDS, f"{b['case']}/deterministic", radii)
    lines = []
    for n in GRADS:
        rho, alpha = BOUNDS[n]
        wd = float(element_ratios(g_det[n], exact[n], rho, alpha).max())
        wo = float(element_ratios(g_def[n], exact[n], rho, alpha).max())
        lines.append(f"  {n:14s} worst ratio to the bound: deterministic {wd:.3f}  default {wo:.3f}")
    print(f"\n{b['case']}:\n" + "\n".join(lines))


def test_bench_step_other_stream_and_concurrent_work(bench):
    """the same step on a non-default stream, and while a matmul loop runs on another stream, matches the deterministic run bitwise"""
    if bench["case"] != "deg3":
        pytest.skip("deg3 only")
    with det(True):
        ref = _bench_grads(bench)
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            on_stream = _bench_grads(bench)
        torch.cuda.synchronize()
        busy = torch.cuda.Stream()
        a = torch.randn(4096, 4096, device="cuda")
        with torch.cuda.stream(busy):
            for _ in range(40):
                a = torch.tanh(a @ a * 1e-3)
        loaded = _bench_grads(bench)
        torch.cuda.synchronize()
    for k in ref:
        assert np.array_equal(ref[k], on_stream[k]), f"{k}: non-default stream differs"
        assert np.array_equal(ref[k], loaded[k]), f"{k}: concurrent work changed the result"


# ------------------------------------------------------------------------------------------------
# 2. small and edge configurations
# ------------------------------------------------------------------------------------------------
def _scene_case(P, W, H, seed=5, bg=(0.1, 0.2, 0.3), scale_mult=1.5, cull_all=False):
    scene = make_scene(max(P, 1), sh_degree=3, seed=seed, scale_mult=scale_mult)
    raw = {k: v[:P] for k, v in scene["raw"].items()}
    cam = make_cameras(4, W, H)[1]
    if cull_all:
        raw["xyz"] = (1.5 * cam.camera_center[None, :] + 0.01 * np.random.default_rng(seed).standard_normal((P, 3))).astype(np.float32)
    pc = GaussianParams(raw, 3, "cuda")
    tcam = TorchCamera(cam, "cuda")
    return pc, tcam, torch.tensor(bg, device="cuda")


@pytest.mark.parametrize("case", ["P0", "1x1", "culled", "mod07", "white", "small"])
def test_edge_cases_repeatable(case):
    cfg = dict(P0=(0, 64, 48), culled=(2000, 96, 64), mod07=(4000, 160, 112), white=(4000, 160, 112), small=(4000, 208, 160))
    P, W, H = (3000, 1, 1) if case == "1x1" else cfg[case]
    bg = (1.0, 1.0, 1.0) if case == "white" else (0.1, 0.2, 0.3)
    pc, tcam, bgt = _scene_case(P, W, H, bg=bg, cull_all=case == "culled", scale_mult=8.0 if case == "1x1" else 1.5)
    dpix = torch.randn(3, H, W, generator=torch.Generator().manual_seed(3)).cuda()
    if case == "mod07":
        from lightgaussian_b200.renderer import render

        def run():
            for p in pc.parameters():
                p.grad = None
            pkg = render(tcam, pc, pipeline_params(), bgt, scaling_modifier=0.7)
            pkg["render"].backward(dpix)
            torch.cuda.synchronize()
            return {n: getattr(pc, "_" + n).grad.cpu().numpy() for n in LEAVES}
    else:
        def run():
            return _leaf_step(pc, tcam, bgt, dpix)
    _repeat(run, f"edge {case}")


def test_api_path_python_flags_repeatable():
    """the reference API node (_RasterizeGaussians): compute_cov3D_python and override_color"""
    from lightgaussian_b200.renderer import render
    pc, tcam, bg = _scene_case(20000, 320, 240, seed=9, scale_mult=2.0)
    dpix = torch.randn(3, 240, 320, generator=torch.Generator().manual_seed(4)).cuda()
    colors = torch.rand(20000, 3, device="cuda", requires_grad=True)

    def run(kind):
        def f():
            for p in pc.parameters():
                p.grad = None
            colors.grad = None
            if kind == "cov3D":
                pkg = render(tcam, pc, pipeline_params(compute_cov3D_python=True), bg)
            else:
                pkg = render(tcam, pc, pipeline_params(), bg, override_color=colors)
            pkg["render"].backward(dpix)
            torch.cuda.synchronize()
            g = {n: getattr(pc, "_" + n).grad.cpu().numpy() for n in LEAVES if getattr(pc, "_" + n).grad is not None}
            if kind == "color":
                g["colors"] = colors.grad.cpu().numpy()
            return g
        return f
    _repeat(run("cov3D"), "API path compute_cov3D_python")
    _repeat(run("color"), "API path override_color")


def test_whole_frame_gaussian_repeatable():
    """one Gaussian covering the whole 1080p frame, behind 2000 small ones"""
    cam = make_cameras(16, BW, BH)[0]
    scene = make_scene(2001, sh_degree=3, seed=21, scale_mult=1.0)
    raw = {k: v.copy() for k, v in scene["raw"].items()}
    # the first Gaussian: just in front of the camera centre along the view axis, huge and opaque-ish
    R = np.asarray(cam.world_view_transform, np.float64)[:3, :3]
    fwd = R[:, 2] if abs(np.linalg.det(R)) > 0 else np.array([0, 0, 1.0])
    raw["xyz"][0] = (np.asarray(cam.camera_center) + 3.0 * fwd / np.linalg.norm(fwd)).astype(np.float32)
    raw["scaling"][0] = np.log(np.full(3, 20.0, np.float32))
    raw["opacity"][0] = 0.0
    pc = GaussianParams(raw, 3, "cuda")
    tcam = TorchCamera(cam, "cuda")
    bg = torch.zeros(3, device="cuda")
    dpix = torch.randn(3, BH, BW, generator=torch.Generator().manual_seed(5)).cuda()
    from lightgaussian_b200.rasterizer import _forward_raw_native
    with torch.no_grad():
        radii = _forward_raw_native(False, _settings(tcam, bg, 3), *_leaves(pc))[4]
    assert int(radii[0]) > 1000, "the big Gaussian does not cover the frame"
    _repeat(lambda: _leaf_step(pc, tcam, bg, dpix), "whole-frame Gaussian")


@pytest.mark.parametrize("dpix_kind", ["constant", "random_sign"])
def test_blend_ring_stacks_repeatable_and_accurate(dpix_kind):
    """test_gpu_leafgrad.py's stacks of 1 .. 600 Gaussians per tile (chunk, flush and ring boundaries, a tile corner)"""
    raw, cam, free = _stack_scene()
    pc = GaussianParams(raw, 3, "cuda")
    tcam = TorchCamera(cam, "cuda")
    bg = torch.tensor([0.3, 0.2, 0.1], device="cuda")
    H, W = cam.image_height, cam.image_width
    if dpix_kind == "constant":
        dpix = np.full((3, H, W), 0.5, np.float32)
    else:
        dpix = np.sign(np.random.default_rng(1).standard_normal((3, H, W))).astype(np.float32)
    dpix_t = torch.from_numpy(dpix).cuda()
    g, _ = _repeat(lambda: _leaf_step(pc, tcam, bg, dpix_t), f"stacks/{dpix_kind}")
    view = view_from_camera(cam, (0.3, 0.2, 0.1), 3, 1.0)
    leaves = _leaves(pc)
    with det(True):
        state = _fused_state(view, _settings(tcam, bg, 3), leaves)
    exact = leaf_grads_float64(view, raw, state, dpix, act=_activated(leaves, 3))
    _check_all(g, exact, STACK_BOUNDS, f"stacks/{dpix_kind}/deterministic", state["radii"])


# ------------------------------------------------------------------------------------------------
# 4. mode pinning and refused combinations
# ------------------------------------------------------------------------------------------------
def _pinned_run(fwd_det, bwd_det, pc, tcam, bg, dpix, api=False):
    from lightgaussian_b200.renderer import render
    for p in pc.parameters():
        p.grad = None
    with det(fwd_det):
        pkg = render(tcam, pc, pipeline_params(compute_cov3D_python=api), bg)
    with det(bwd_det):
        pkg["render"].backward(dpix)
    torch.cuda.synchronize()
    return {n: getattr(pc, "_" + n).grad.cpu().numpy() for n in LEAVES}


@pytest.mark.parametrize("api", [False, True])
def test_backward_runs_in_the_mode_of_its_forward(api):
    pc, tcam, bg = _scene_case(20000, 320, 240, seed=31, scale_mult=2.0)
    dpix = torch.randn(3, 240, 320, generator=torch.Generator().manual_seed(6)).cuda()
    all_det = _pinned_run(True, True, pc, tcam, bg, dpix, api)
    flag_off = _pinned_run(True, False, pc, tcam, bg, dpix, api)
    for k in all_det:
        assert np.array_equal(all_det[k], flag_off[k]), f"{k}: a deterministic forward's backward ran in default mode"
    # the reverse: a default forward keeps the default backward even when the flag is on by then.  Two default-mode runs differ in
    # the last bits (float atomics), so the check is test_gpu_leafgrad.py's per-element bound between them, not bit-equality; a
    # deterministic backward of a default forward would read records without the permutation word and miss it by far.
    all_def = _pinned_run(False, False, pc, tcam, bg, dpix, api)
    flag_on = _pinned_run(False, True, pc, tcam, bg, dpix, api)
    for k in all_def:
        util.assert_every_element(flag_on[k], all_def[k], 1e-3, 1e-5, f"default forward, flag on at backward: {k}")


def test_torch_flag_turns_the_mode_on():
    pc, tcam, bg = _scene_case(20000, 320, 240, seed=32, scale_mult=2.0)
    dpix = torch.randn(3, 240, 320, generator=torch.Generator().manual_seed(7)).cuda()
    with det(True):
        ref = _leaf_step(pc, tcam, bg, dpix)
    torch.use_deterministic_algorithms(True)
    try:
        with det(False):
            via_torch = _leaf_step(pc, tcam, bg, dpix)
    finally:
        torch.use_deterministic_algorithms(False)
    for k in ref:
        assert np.array_equal(ref[k], via_torch[k]), k


@pytest.mark.parametrize("switch", ["binning0", "binning1", "blend1"])
def test_unsupported_combinations_raise_before_any_launch(switch):
    from lightgaussian_b200.renderer import render
    pc, tcam, bg = _scene_case(2000, 96, 64, seed=33)
    render(tcam, pc, pipeline_params(), bg)   # one-time self-checks of the fused path happen here, in the default modes
    torch.cuda.synchronize()
    try:
        if switch == "blend1":
            capi.set_blend_mode(1)
        else:
            capi.set_binning_mode(int(switch[-1]))
        with det(True):
            n0 = capi.launch_count()
            with pytest.raises(RuntimeError, match="lgr_set_binning_mode" if switch != "blend1" else "lgr_set_blend_mode"):
                render(tcam, pc, pipeline_params(), bg)
            assert capi.launch_count() == n0
            with pytest.raises(RuntimeError, match="deterministic"):
                util.run_ours(*util.make_config("deg1")[1::-1], blend_mode=1 if switch == "blend1" else 0,
                              bin_mode=None if switch == "blend1" else int(switch[-1]))
            assert capi.launch_count() == n0
    finally:
        capi.set_blend_mode(0)
        capi.set_binning_mode(capi.DEFAULT_BINNING_MODE)


# ------------------------------------------------------------------------------------------------
# 5. VecTree
# ------------------------------------------------------------------------------------------------
def _vq_run(kind, seed=0, n=80_000, K=8192, d=27, iters=20):
    from lightgaussian_b200.vectree import VectorQuantize
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "random":
        feats = torch.randn(n * 4, d, device="cuda", generator=g)
    else:
        centres = torch.randn(64, d, device="cuda", generator=g) * 3
        feats = centres[torch.randint(0, 64, (n * 4,), device="cuda", generator=g)] + 0.05 * torch.randn(n * 4, d, device="cuda", generator=g)
    imp = torch.rand(n * 4, device="cuda", generator=g) + 0.01
    torch.manual_seed(seed)
    vq = VectorQuantize(dim=d, codebook_size=K, decay=0.8, commitment_weight=0.0, use_cosine_sim=False,
                        threshold_ema_dead_code=0).cuda()
    vq.train()
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    k_expire = 10
    for it in range(iters):
        sel = torch.randint(0, n * 4, (n,), device="cuda", generator=gen)
        vq(feats[sel].unsqueeze(0), weight=imp[sel].reshape(1, -1, 1))
        # the k_expire replacement of Quantization.train_codebook: the least used codes take random samples
        replace = torch.argsort(vq._codebook.cluster_size[0], stable=True)[:k_expire]
        vq._codebook.embed[0, replace] = feats[sel[:k_expire]]
    vq.eval()
    q, idx, _ = vq(feats[:n].unsqueeze(0))
    torch.cuda.synchronize()
    return {"embed": vq._codebook.embed.cpu().numpy(), "cluster_size": vq._codebook.cluster_size.cpu().numpy(),
            "idx": idx.cpu().numpy()}


@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_vectree_ema_bit_identical(kind):
    _repeat(lambda: _vq_run(kind), f"VecTree 20 EMA iterations, {kind}", n=2)



def _vq_data(kind, n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "random":
        x = torch.randn(n, d, device="cuda", generator=g)
    else:   # few, tight clusters: thousands of samples per code, the segmented sum's longest segments
        centres = torch.randn(64, d, device="cuda", generator=g) * 3
        x = centres[torch.randint(0, 64, (n,), device="cuda", generator=g)] + 0.05 * torch.randn(n, d, device="cuda", generator=g)
    return x, torch.rand(n, device="cuda", generator=g) + 0.01


@pytest.mark.parametrize("kind,n,d,K_,weighted", [("random", 80_000, 27, 8192, True), ("clustered", 80_000, 27, 8192, True),
                                                  ("random", 80_000, 27, 8192, False), ("random", 5000, 48, 300, True),
                                                  ("clustered", 20_000, 64, 1000, True), ("random", 777, 3, 7, True)])
def test_vq_assign_sums_against_the_oracle(kind, n, d, K_, weighted):
    """lgr_vq_assign's cluster_batch / embed_sum in deterministic mode against vq_oracle's float64 sums over the SAME indices (so no
    tie can differ): the weight normalisation, both outputs, the sort's bit count for K not a power of two, d > 32 (three columns per
    lane) and d < 32, empty codes (exact zeros)"""
    from lightgaussian_b200.vectree import vq_assign
    x, w = _vq_data(kind, n, d, n + d)
    embed = x[torch.randperm(n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))[:K_]].clone()
    if kind == "clustered":   # 64 codes on the data, the rest far away: every sample lands on one of 64 codes (hundreds each)
        embed = 100.0 + torch.randn(K_, d, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        embed[:64] = x[:64]
    with det(True):
        idx, cb, es = vq_assign(x, embed, w if weighted else None, want_sums=True)
        idx2, cb2, es2 = vq_assign(x, embed, w if weighted else None, want_sums=True)
    torch.cuda.synchronize()
    assert torch.equal(idx, idx2) and torch.equal(cb, cb2) and torch.equal(es, es2)
    with det(False):
        idx_def = vq_assign(x, embed)
    assert torch.equal(idx, idx_def), "deterministic mode changed the nearest-code search"
    i = idx.cpu().numpy().astype(np.int64)
    x64 = x.cpu().numpy().astype(np.float64)
    w64 = np.ones(n) if not weighted else w.cpu().numpy().astype(np.float64) * n / w.cpu().numpy().astype(np.float64).sum()
    batch = np.bincount(i, weights=w64, minlength=K_)
    esum = np.zeros((K_, d))
    np.add.at(esum, i, x64 * w64[:, None])
    np.testing.assert_allclose(cb.cpu().numpy(), batch, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(es.cpu().numpy(), esum, rtol=1e-4, atol=1e-4 * max(1.0, float(np.abs(esum).max())))
    empty = batch == 0
    assert np.all(cb.cpu().numpy()[empty] == 0) and np.all(es.cpu().numpy()[empty] == 0)
    if kind == "clustered":
        assert batch.max() > 250   # the input really has long segments


@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_vectree_ema_iterations_against_the_oracle(kind):
    """20 weighted EMA iterations with the k_expire replacement in deterministic mode: every iteration's cluster_size and codebook
    against vq_oracle.ema_step from the same pre-iteration state and the same indices, within test_gpu_vq.py's tolerances"""
    from oracle import vq_oracle as vo
    from lightgaussian_b200.vectree import VectorQuantize
    n, d, K_ = 80_000, 27, 8192
    feats, imp = _vq_data(kind, 4 * n, d, 7)
    torch.manual_seed(0)
    vq = VectorQuantize(dim=d, codebook_size=K_, decay=0.8, commitment_weight=0.0).cuda().train()
    gen = torch.Generator(device="cuda").manual_seed(8)
    with det(True):
        for it in range(20):
            sel = torch.randint(0, 4 * n, (n,), device="cuda", generator=gen)
            x, w = feats[sel], imp[sel]
            e0, c0 = vq._codebook.embed[0].cpu().numpy(), vq._codebook.cluster_size[0].cpu().numpy()
            _, idx, _ = vq(x.unsqueeze(0), weight=w.reshape(1, -1, 1))
            _, e_ref, c_ref = vo.ema_step(x.cpu().numpy(), w.cpu().numpy(), e0, c0, idx=idx[0].cpu().numpy().astype(np.int64))
            np.testing.assert_allclose(vq._codebook.cluster_size[0].cpu().numpy(), c_ref, rtol=1e-4, atol=1e-4, err_msg=f"iteration {it}")
            np.testing.assert_allclose(vq._codebook.embed[0].cpu().numpy(), e_ref, rtol=1e-4, atol=2e-5, err_msg=f"iteration {it}")
            replace = torch.argsort(vq._codebook.cluster_size[0], stable=True)[:10]
            vq._codebook.embed[0, replace] = x[:10]


def _quantize_files(tmp, seed=3):
    from lightgaussian_b200.vectree import Quantization
    rng = np.random.default_rng(seed)
    n = 200_000
    feats = rng.standard_normal((n, 6 + 27 + 8)).astype(np.float32)
    imp = rng.random(n).astype(np.float32)
    torch.manual_seed(seed)
    q = Quantization(feats, importance=imp, sh_degree=2, save_path=str(tmp), codebook_size=8192, iteration_num=20, vq_ratio=0.6)
    q.quantize()
    ex = os.path.join(str(tmp), "extreme_saving")
    out = {}
    for f in sorted(os.listdir(ex)):
        z = np.load(os.path.join(ex, f), allow_pickle=True)
        for k in z.files:
            v = z[k]
            out[f"{f}/{k}"] = v.item() if v.dtype == object else v
    return out


def test_quantization_files_bit_identical(tmp_path):
    """Quantization.quantize() twice (importance split, 20 EMA iterations with k_expire, encode): every array of every
    extreme_saving/*.npz is bit-identical between the runs"""
    with det(True):
        a = _quantize_files(tmp_path / "a")
        b = _quantize_files(tmp_path / "b")
    assert sorted(a) == sorted(b) and any(k.startswith("vq_indexs") for k in a)
    for k in a:
        if isinstance(a[k], dict):
            assert a[k] == b[k], k
        else:
            assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------------------
# 4. a deterministic backward of a default forward is refused (NaN), not run on foreign data
# ------------------------------------------------------------------------------------------------
def test_deterministic_backward_of_a_default_forward_gives_nan():
    from lightgaussian_b200.rasterizer import _forward_raw_native, backward_raw_native
    pc, tcam, bg = _scene_case(20000, 320, 240, seed=34, scale_mult=2.0)
    rs = _settings(tcam, bg, 3)
    leaves = _leaves(pc)
    dpix = torch.randn(3, 240, 320, generator=torch.Generator().manual_seed(8)).cuda()
    with det(False):
        with torch.no_grad():
            _, _, R, _, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
        capi.set_deterministic(True)
        g, g2d, _, _ = backward_raw_native(rs, R, dpix, *leaves, radii, geom, binning, img)
        torch.cuda.synchronize()
    vis = radii > 0
    assert int(vis.sum()) > 100
    assert torch.isnan(g[0][vis]).all() and torch.isnan(g2d[vis, :2]).all()


# ------------------------------------------------------------------------------------------------
# 8. multi-GPU: a view-parallel step in deterministic mode
# ------------------------------------------------------------------------------------------------
def _mgpu_worker(rank, world, port, out):
    from tests.test_gpu_multi import _setup
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      LGR_DETERMINISTIC="1")
    from lightgaussian_b200 import parallel
    from lightgaussian_b200.renderer import render
    parallel.init_from_env("nccl")
    dev = torch.device("cuda", rank)
    pc, cams, pipe, bg = _setup(dev)
    parallel.enable_gradient_exchange(world)
    res = []
    for _ in range(2):
        for p in pc.parameters():
            p.grad = None
        render(cams[rank], pc, pipe, bg)["render"].sum().backward()
        res.append(torch.cat([p.grad.reshape(-1) for p in pc.parameters()]).cpu())
    torch.cuda.synchronize()
    torch.save(res, os.path.join(out, f"det_r{rank}.pt"))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_view_parallel_step_bit_identical_over_repeats_and_ranks(tmp_path):
    import torch.multiprocessing as mp
    from tests.test_gpu_multi import _free_port
    world = 2
    mp.spawn(_mgpu_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    runs = [torch.load(os.path.join(tmp_path, f"det_r{r}.pt")) for r in range(world)]
    for r in range(world):
        assert torch.equal(runs[r][0], runs[r][1]), f"rank {r}: repeats differ"
        assert torch.equal(runs[r][0], runs[0][0]), f"rank {r} differs from rank 0"
