"""Blending-weight significance on the GPU (LGR_SIGNIFICANCE=blend_weight, lgr_forward_*_weight).

Two references: the GPU's own per-pair alpha*T, read from images rendered with one-hot colours on a black background (the colour
accumulator then holds exactly fl(alpha*T) of one Gaussian per pixel, and colours change no decision of the blend), which the
weights must match bit for bit; and the float32 CPU oracle, whose exp() is glibc's rather than the GPU's, so it is matched within a
stated tolerance."""
import math
import os

import numpy as np
import pytest
import torch

from lightgaussian_b200 import capi, parallel
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
from lightgaussian_b200.rasterizer import _C
from lightgaussian_b200.renderer import count_render, weight_score
from lightgaussian_b200.synth import camera_from_pose, make_cameras, make_scene
from tests.test_significance_weight_cpu import reference, touches_fragile, weight_fx
from tests.util import CONFIGS, make_config, _t, _empty

pytestmark = pytest.mark.gpu

DEV = "cuda"
TWO32 = 2.0 ** 32


def _api(view, act, weight=True, colors=None, bg=None):
    """the API count path (_C.count_gaussians) on activated arrays; returns count, score, color, radii, blend_weight_fx, image blob"""
    P = act["means3D"].shape[0]
    fx = torch.full((P,), -7, dtype=torch.int64, device=DEV) if weight else None
    bgv = view.bg if bg is None else bg
    args = (_t(bgv), _t(act["means3D"]), _t(colors) if colors is not None else _empty(), _t(act["opacities"]), _t(act["scales"]),
            _t(act["rotations"]), view.scale_modifier, _empty(), _t(view.viewmatrix), _t(view.projmatrix), view.tanfovx, view.tanfovy,
            view.H, view.W, _empty() if colors is not None else _t(act["shs"]), view.sh_degree, _t(view.campos), False, False)
    cnt, score, R, color, radii, geom, binning, img = _C.count_gaussians(*args, True, blend_weight=fx)
    return dict(count=cnt, score=score, color=color, radii=radii, fx=fx, img=img)


def _gpu_pair_fx(view, act, ids):
    """sum over pixels of rint(fl(alpha*T) * 2^32) per Gaussian, from one-hot colour renders (three Gaussians per render)"""
    P = act["means3D"].shape[0]
    out = np.zeros(P, np.int64)
    zero = np.zeros(3, np.float32)
    for k in range(0, len(ids), 3):
        grp = ids[k:k + 3]
        col = np.zeros((P, 3), np.float32)
        col[grp, np.arange(len(grp))] = 1.0
        r = _api(view, act, weight=False, colors=col, bg=zero)
        q = torch.round(r["color"].double() * TWO32).to(torch.int64).reshape(3, -1).sum(dim=1).cpu().numpy()
        out[grp] = q[:len(grp)]
    return out


@pytest.mark.parametrize("name", list(CONFIGS))
def test_against_the_gpu_blend_and_the_oracle(name):
    act, view, _ = make_config(name)
    ours = _api(view, act)
    fx = ours["fx"].cpu().numpy()
    ids = np.nonzero(ours["radii"].cpu().numpy() > 0)[0]
    np.testing.assert_array_equal(fx, _gpu_pair_fx(view, act, ids))        # every Gaussian, bit for bit
    ref = reference(name)
    rfx = weight_fx(ref)
    frag = touches_fragile(ref)
    cnt = ref["count"]
    err = np.abs(fx - rfx).astype(np.float64)
    ok = ~frag
    # off fragile tiles the pairs are the same; alpha differs by the two exp() implementations' ulps, and T carries that on
    assert (err[ok] <= 1e-4 * rfx[ok] + 2.0 * cnt[ok]).all(), np.max(err[ok] - 1e-4 * rfx[ok])
    assert (err <= 2e-2 * rfx + 2e-3 * TWO32 * cnt + 1).all()
    print(f"{name}: {np.mean(err[ok] == 0) * 100:.1f} % of {ok.sum()} Gaussians off fragile tiles bit-identical to the oracle, "
          f"max relative difference {np.max(err[ok] / np.maximum(rfx[ok], 1)):.2e}")


# ---------------------------------------------------------------------------------------------------------------------------------
def _vq_models(tmp_path, P=20000):
    from lightgaussian_b200.vqresident import ResidentVQ
    from tests.test_gpu_vq_render import ResidentModel, dense_model, make_model
    make_model(str(tmp_path), P, 3, 0.6, True, seed=3, writer="direct")
    store = ResidentVQ.load(str(tmp_path), 3, DEV)
    return ResidentModel(store, 3), dense_model(store, 3)


def _count_render(cam, pc, weight, fused=True, bg=None):
    env = {"LGR_SIGNIFICANCE": "blend_weight" if weight else "count", "LGR_FUSED": "1" if fused else "0"}
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        with torch.no_grad():
            return count_render(cam, pc, pipeline_params(), torch.zeros(3, device=DEV) if bg is None else bg)
    finally:
        for k, v in saved.items():
            os.environ.pop(k) if v is None else os.environ.__setitem__(k, v)


def test_three_paths_agree_and_opt_in_changes_nothing_else(tmp_path):
    from lightgaussian_b200 import trace
    resident, dense = _vq_models(tmp_path)
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    for c in make_cameras(3, 320, 240):
        cam = TorchCamera(c)
        weights = []
        for pc, fused, counter in ((resident, True, "render_vq_resident"), (dense, True, "render_fused"), (dense, False, "render_unfused")):
            before = trace.counters.get(counter, 0)
            d = _count_render(cam, pc, False, fused, bg)
            w = _count_render(cam, pc, True, fused, bg)
            assert trace.counters.get(counter, 0) == before + 2, counter
            for k in ("render", "radii", "visibility_filter", "gaussians_count"):
                assert torch.equal(d[k], w[k]), (counter, k)
            assert "blend_weight_fx" not in d and w["blend_weight_fx"].dtype == torch.int64
            assert torch.equal(w["important_score"], weight_score(w["blend_weight_fx"]))
            assert int((w["blend_weight_fx"] > 0).sum()) == int((w["gaussians_count"] > 0).sum())
            weights.append((d, w))
        for (d, w) in weights[1:]:
            assert torch.equal(w["blend_weight_fx"], weights[0][1]["blend_weight_fx"])
            assert torch.equal(d["important_score"], weights[0][0]["important_score"])


def _scene(P, W, H, n_cams, seed=21):
    s = make_scene(P, sh_degree=3, seed=seed, scale_mult=1.5)
    pc = GaussianParams(s["raw"], 3, DEV, requires_grad=False)
    return pc, [TorchCamera(c) for c in make_cameras(n_cams, W, H)]


def test_bit_identical_across_runs_streams_modes_binning_and_culling(monkeypatch):
    pc, cams = _scene(200_000, 640, 480, 2)
    monkeypatch.setenv("LGR_SIGNIFICANCE", "blend_weight")
    pipe, bg = pipeline_params(), torch.zeros(3, device=DEV)

    def run():
        with torch.no_grad():
            return [count_render(c, pc, pipe, bg)["blend_weight_fx"].clone() for c in cams]
    base = run()
    assert all(int(b.sum()) > 0 for b in base)

    def same(tag):
        for a, b in zip(run(), base):
            assert torch.equal(a, b), tag
    same("second run")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = run()
    s.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(got, base)), "side stream"
    monkeypatch.setenv("LGR_DETERMINISTIC", "1")
    same("deterministic mode")
    monkeypatch.delenv("LGR_DETERMINISTIC")
    try:
        for m in (0, 1, 2):
            capi.set_binning_mode(m)
            same(f"binning mode {m}")
        capi.set_binning_mode(capi.DEFAULT_BINNING_MODE)
        capi.set_tile_culling(False)
        same("tile culling off")
    finally:
        capi.set_binning_mode(capi.DEFAULT_BINNING_MODE)
        capi.set_tile_culling(True)


def test_round1_blend_kernels_refuse_before_any_launch():
    act, view, _ = make_config("deg1")
    P = act["means3D"].shape[0]
    fx = torch.full((P,), -7, dtype=torch.int64, device=DEV)
    args = (_t(view.bg), _t(act["means3D"]), _empty(), _t(act["opacities"]), _t(act["scales"]), _t(act["rotations"]), 1.0, _empty(),
            _t(view.viewmatrix), _t(view.projmatrix), view.tanfovx, view.tanfovy, view.H, view.W, _t(act["shs"]), view.sh_degree,
            _t(view.campos), False, False)
    torch.cuda.synchronize()
    capi.set_blend_mode(1)
    try:
        n0 = capi.launch_count()
        with pytest.raises(capi.LgrError, match="ring blend kernels"):
            _C.count_gaussians(*args, True, blend_weight=fx)
        torch.cuda.synchronize()
        assert capi.launch_count() == n0
        assert bool((fx == -7).all())
        _C.count_gaussians(*args, True)          # the plain count forward still runs in that mode
    finally:
        capi.set_blend_mode(0)


def test_bench_size_weights_sum_to_coverage():
    """3M Gaussians, 1080p, 4 cameras: sum_i weight_i = sum_p (1 - final_T), up to the float32 rounding of each pixel's blend"""
    s = make_scene(3_000_000, sh_degree=3, seed=0)
    act = {k: v for k, v in s["act"].items()}
    from tests.util import view_from_camera
    il, _ = capi.image_layout(1920, 1080)
    N = 1920 * 1080
    for c in make_cameras(4, 1920, 1080):
        r = _api(view_from_camera(c), act)
        final_T = r["img"][il["final_T"]:il["final_T"] + 4 * N].view(torch.float32)
        cover = float((1.0 - final_T.double()).sum())
        total = float(r["fx"].double().sum()) / TWO32
        print(f"bench camera: sum of weights {total:.4f}, sum of 1 - final_T {cover:.4f}, relative {abs(total - cover) / cover:.2e}")
        assert abs(total - cover) <= 2e-5 * cover, (total, cover)


def test_partition_independence_bit_identical():
    pc, cams = _scene(200_000, 480, 360, 8, seed=22)
    os.environ["LGR_SIGNIFICANCE"] = "blend_weight"
    try:
        per_view = [count_render(c, pc, pipeline_params(), torch.zeros(3, device=DEV))["blend_weight_fx"].clone() for c in cams]
        cnt1, imp1 = parallel.sharded_prune_list(pc, cams, pipeline_params(), torch.zeros(3, device=DEV), count_render, 0, 1)
    finally:
        os.environ.pop("LGR_SIGNIFICANCE")
    serial = torch.stack(per_view).sum(dim=0)
    assert torch.equal(weight_score(serial), imp1)
    rng = np.random.default_rng(0)
    for world in (1, 2, 3, 8):
        partial = [sum((per_view[i] for i in parallel.shard_views(len(cams), r, world)), torch.zeros_like(serial)) for r in range(world)]
        for _ in range(3):
            total = torch.zeros_like(serial)
            for r in rng.permutation(world):
                total += partial[r]
            assert torch.equal(total, serial), world


def _occlusion_scene():
    """an opaque wide Gaussian in front of a small one of equal opacity, and six unoccluded copies of the small one around them"""
    logit = math.log(0.99 / 0.01)
    xyz = [[0.0, 0.0, -1.0], [0.0, 0.0, 0.0]] + [[2.6 * math.cos(a), 2.6 * math.sin(a), 0.0] for a in np.arange(6) * math.pi / 3]
    scale = [1.0, 0.1] + [0.1] * 6
    P = len(xyz)
    raw = dict(xyz=np.array(xyz, np.float32), features_dc=np.full((P, 1, 3), 0.5, np.float32), features_rest=np.zeros((P, 15, 3), np.float32),
               scaling=np.log(np.repeat(np.array(scale, np.float32)[:, None], 3, 1)), rotation=np.tile(np.array([1, 0, 0, 0], np.float32), (P, 1)),
               opacity=np.full((P, 1), logit, np.float32))
    pc = GaussianParams(raw, 0, DEV, requires_grad=False)
    pc.active_sh_degree = 0
    cam = TorchCamera(camera_from_pose(np.eye(3), np.array([0.0, 0.0, 5.0]), 256, 256, math.radians(60.0)))
    return pc, cam


def test_weight_ranks_an_occluded_gaussian_far_lower():
    pc, cam = _occlusion_scene()
    d = _count_render(cam, pc, False)
    w = _count_render(cam, pc, True)
    cnt = d["gaussians_count"].cpu().numpy()
    imp, wt = d["important_score"].cpu().numpy(), w["important_score"].cpu().numpy()
    rear, ctrl = 1, slice(2, 8)
    print(f"opacity*count: front {imp[0]:.1f} rear {imp[1]:.1f} controls {imp[ctrl].mean():.1f};  "
          f"weight: front {wt[0]:.3f} rear {wt[1]:.4f} controls {wt[ctrl].mean():.3f}")
    assert cnt[rear] > 0 and imp[rear] >= 0.9 * imp[ctrl].min()          # the count ranks it with the unoccluded copies
    assert wt[rear] <= wt[ctrl].min() / 20.0                              # the weight: the front leaves it T = 0.01 to 0.03
    # prune_gaussians(0.5, score) of the reference (scene/gaussian_model.py): drop every score <= the value at int(0.5 * (P - 1))
    thr = np.sort(wt)[int(0.5 * (len(wt) - 1))]
    pruned = wt <= thr
    assert pruned[rear] and not pruned[0]


def test_prune_finetune_opts_in_unmodified(tmp_path):
    """prune_finetune.py on the drop-ins with LGR_SIGNIFICANCE=blend_weight --prune_type important_score: it prunes by weight and
    writes imp_score.npz at its last checkpoint, equal to calculate_v_imp_score of sharded_prune_list's weights on that checkpoint"""
    from tests import scripts_harness as sh
    reason = sh.stacks_available()
    if reason:
        pytest.skip(reason)
    it0, steps = 30000, 20
    w = sh.build_workdir(str(tmp_path), iteration=it0)
    last = it0 + steps
    model = os.path.join(str(tmp_path), "pf")
    saved = os.environ.get("LGR_SIGNIFICANCE")
    os.environ["LGR_SIGNIFICANCE"] = "blend_weight"
    try:
        sh.run("ours", ["prune_finetune.py", "-s", w["data"], "-m", model, "--eval", "-r", "1", "--port", str(6131),
                        "--start_checkpoint", w["ckpt"], "--iterations", str(last), "--prune_percent", "0.5", "--prune_type",
                        "important_score", "--prune_decay", "1", "--v_pow", "0.1", "--position_lr_max_steps", str(last),
                        "--prune_iterations", str(it0 + 1), "--test_iterations", "999999", "--save_iterations", str(last),
                        "--checkpoint_iterations", str(last)])
        ck = sh.load_checkpoint_leaves(os.path.join(model, f"chkpnt{last}.pth"))
        P = ck["leaves"]["xyz"].shape[0]
        assert P <= 0.55 * w["P"], P                                        # the prune event ran
        saved_v = np.load(os.path.join(model, "imp_score.npz"))["arr_0"]
        pc = GaussianParams(ck["leaves"], 3, DEV, requires_grad=False)
        train = [TorchCamera(c) for k, c in enumerate(w["cams"]) if k % 8 != 0]
        with torch.no_grad():
            _, imp = parallel.sharded_prune_list(pc, train, pipeline_params(), torch.zeros(3, device=DEV), count_render)
            volume = torch.prod(pc.get_scaling, dim=1)
            kth = torch.sort(volume, descending=True)[0][int(len(volume) * 0.9)]
            v = ((volume / kth) ** 0.1 * imp).cpu().numpy()
    finally:
        os.environ.pop("LGR_SIGNIFICANCE") if saved is None else os.environ.__setitem__("LGR_SIGNIFICANCE", saved)
    assert saved_v.shape == v.shape
    rel = np.abs(saved_v - v) / np.maximum(np.abs(v), 1e-6)
    print(f"imp_score.npz against sharded_prune_list: median relative difference {np.median(rel):.2e}, max {rel.max():.2e}")
    np.testing.assert_allclose(saved_v, v, rtol=1e-4, atol=1e-6)


def test_psnr_after_a_066_prune_report_only():
    """Report only: training-view PSNR of the scripts' synthetic scene right after pruning 66 % by each score, no finetuning"""
    from tests.scripts_harness import render_ground_truth
    from lightgaussian_b200.renderer import render
    s = make_scene(20000, sh_degree=3, seed=5, scale_mult=1.5)
    cams = make_cameras(24, 320, 240)
    gt = render_ground_truth(s["raw"], cams)
    train = [TorchCamera(c) for k, c in enumerate(cams) if k % 8 != 0]
    gtt = [torch.from_numpy(g).to(DEV) for k, g in enumerate(gt) if k % 8 != 0]
    pc = GaussianParams(s["raw"], 3, DEV, requires_grad=False)
    pipe, bg = pipeline_params(), torch.zeros(3, device=DEV)
    out = {}
    for mode in ("count", "blend_weight"):
        os.environ["LGR_SIGNIFICANCE"] = mode
        try:
            with torch.no_grad():
                _, imp = parallel.sharded_prune_list(pc, train, pipe, bg, count_render)
        finally:
            os.environ.pop("LGR_SIGNIFICANCE")
        thr = torch.sort(imp)[0][int(0.66 * (imp.numel() - 1))]
        keep = (imp > thr).cpu().numpy()
        kept = GaussianParams({k: v[keep] for k, v in s["raw"].items()}, 3, DEV, requires_grad=False)
        vals = []
        with torch.no_grad():
            for c, g in zip(train, gtt):
                mse = ((render(c, kept, pipe, bg)["render"].clamp(0, 1) - g.clamp(0, 1)) ** 2).mean().item()
                vals.append(-10.0 * math.log10(max(mse, 1e-12)))
        out[mode] = (float(np.mean(vals)), int(keep.sum()))
    print(f"training-view PSNR after a 0.66 prune, no finetuning: count {out['count'][0]:.2f} dB ({out['count'][1]} kept), "
          f"blend_weight {out['blend_weight'][0]:.2f} dB ({out['blend_weight'][1]} kept)")
    assert all(np.isfinite(v[0]) for v in out.values())
