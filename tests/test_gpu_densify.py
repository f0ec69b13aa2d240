"""Native densification (lightgaussian_b200/densify.py, csrc/lgr_densify.cuh) against the reference's own GaussianModel methods.

Both stacks of tests/scripts_harness.py run tests/helpers/densify_event.py on the same states (tests/helpers/densify_state.py):
under the stock stack the reference's torch add_densification_stats / densify_and_prune and torch.optim.AdamW, under ours the same
unmodified class with FusedAdamW and the native methods installed.  Every parameter, Adam moment, `step`, optimizer state key and
auxiliary buffer must be bit-identical, and so must the CUDA generator's state afterwards, one rendered view of the result (each
stack's own renderer; their forward passes are bit-identical), and the parameters after one more optimizer step.  Then
train_densify_prune.py, unmodified, from Scene creation on both stacks."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from tests import scripts_harness as sh

pytestmark = pytest.mark.gpu

sys.path.insert(0, sh.HELPERS)
import densify_state  # noqa: E402

P_BASE = 100_000
PORT = 6200


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    reason = sh.stacks_available()
    if reason:
        pytest.skip(reason)
    return str(tmp_path_factory.mktemp("densify"))


def _views(base, P, n_views=20, W=320, H=240):
    """view-space gradients and visibility filters of real render() + backward passes of our renderer"""
    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.renderer import render
    from lightgaussian_b200.synth import make_cameras, make_scene
    scene = make_scene(P, sh_degree=3, seed=3, scale_mult=1.5)
    pc = GaussianParams(scene["raw"], 3, "cuda")
    bg = torch.zeros(3, device="cuda")
    g = torch.Generator().manual_seed(1)
    views = []
    for cam in make_cameras(n_views, W, H):
        pkg = render(TorchCamera(cam, "cuda"), pc, pipeline_params(), bg)
        target = torch.rand(3, H, W, generator=g).cuda()
        (pkg["render"] - target).abs().mean().backward()
        views.append((pkg["viewspace_points"].grad.detach().cpu(), pkg["visibility_filter"].cpu()))
        for p in pc.parameters():
            p.grad = None
    path = os.path.join(base, "views.pt")
    torch.save(views, path)
    return path, views


def _run(work, stack, mode, cases, tag, extra=()):
    cases_path = os.path.join(work, f"{tag}_cases.pt")
    out = os.path.join(work, f"{tag}_{stack}.pt")
    trace = os.path.join(work, f"{tag}_{stack}.trace.json")
    torch.save(cases, cases_path)
    sh.run(stack, [os.path.join(sh.HELPERS, "densify_event.py"), mode, cases_path, out, *extra], trace=trace if stack == "ours" else None)
    return torch.load(out, weights_only=False), (sh.read_trace(trace) if stack == "ours" else None)


@pytest.fixture(scope="module")
def stats(work):
    path, views = _views(work, P_BASE)
    case = dict(P_base=P_BASE, seed=3, P=P_BASE, views=path)
    ours, tr = _run(work, "ours", "stats", [case], "stats", ["--sync-error"])
    stock, _ = _run(work, "stock", "stats", [case], "stats")
    out = os.path.join(work, "accum.pt")
    torch.save(stock, out)
    return dict(ours=ours, stock=stock, trace=tr, views=views, path=out)


def test_statistics_bit_identical_to_reference(stats):
    ours, stock, views = stats["ours"], stats["stock"], stats["views"]
    culled = sum(int((~f).sum()) for _, f in views)
    assert culled > 0 and all(f.any() for _, f in views)
    assert torch.equal(ours["accum"].view(torch.int32), stock["accum"].view(torch.int32))
    assert torch.equal(ours["denom"].view(torch.int32), stock["denom"].view(torch.int32))
    # the native call ran under torch.cuda.set_sync_debug_mode("error") once per view
    assert stats["trace"].get("densify_stats_native") == len(views), stats["trace"]


def test_statistics_native_without_host_sync():
    from lightgaussian_b200 import densify
    P = 4097
    holder = types.SimpleNamespace(xyz_gradient_accum=torch.zeros(P, 1, device="cuda"), denom=torch.zeros(P, 1, device="cuda"))
    vs = types.SimpleNamespace(grad=torch.randn(P, 3, device="cuda"))
    filt = torch.rand(P, device="cuda") > 0.5
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        densify.add_densification_stats(holder, vs, filt)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want = torch.zeros(P, 1, device="cuda")
    want[filt] += torch.norm(vs.grad[filt, :2], dim=-1, keepdim=True)
    assert torch.equal(holder.xyz_gradient_accum, want)
    assert torch.equal(holder.denom[:, 0], filt.float())


def _grads_and_scales(case):
    st = densify_state.build(case)
    grads = (st["accum"].cuda() / st["denom"].cuda())[:, 0]
    grads[grads.isnan()] = 0.0
    ms = torch.exp(st["scaling"].cuda()).max(dim=1).values
    return grads, ms


def _stats_3m(base):
    """densification statistics of the 3M-Gaussian case: two 1080p render() + backward views through our renderer, accumulated by the
    native add_densification_stats (bit-identical to the reference's, test_statistics_bit_identical_to_reference)"""
    from lightgaussian_b200 import densify
    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.renderer import render
    from lightgaussian_b200.synth import make_cameras, make_scene
    pc = GaussianParams(make_scene(3_000_000, sh_degree=3, seed=9, scale_mult=1.5)["raw"], 3, "cuda")
    holder = types.SimpleNamespace(xyz_gradient_accum=torch.zeros(3_000_000, 1, device="cuda"), denom=torch.zeros(3_000_000, 1, device="cuda"))
    for cam in make_cameras(4, 1920, 1080)[:2]:
        pkg = render(TorchCamera(cam, "cuda"), pc, pipeline_params(), torch.zeros(3, device="cuda"))
        pkg["render"].mean().backward()
        densify.add_densification_stats(holder, pkg["viewspace_points"], pkg["visibility_filter"])
        for p in pc.parameters():
            p.grad = None
    path = os.path.join(base, "accum_3m.pt")
    torch.save({"accum": holder.xyz_gradient_accum.cpu(), "denom": holder.denom.cpu()}, path)
    return path


def _coverage(case):
    """rows of each kind on either side of the world-space size prune `max exp(s) > 0.1*extent` (scene/gaussian_model.py:755-757)"""
    grads, ms = _grads_and_scales(case)
    dense, big, mg = np.float32(0.01 * case["extent"]), np.float32(0.1 * case["extent"]), np.float32(case["max_grad"])
    split = (grads >= mg) & (ms > dense)
    clone = (grads >= mg) & (ms <= dense)
    child = ms / 1.6                                      # the child's max scale up to rounding: enough to count coverage
    return {"unsplit above": int((~split & (ms > big)).sum()), "unsplit at": int((~split & (ms == big)).sum()),
            "unsplit below": int((~split & (ms <= big)).sum()),
            "clones": int(clone.sum()), "children above": int((split & (child > big)).sum()),
            "children below, parent above": int((split & (child <= big) & (ms > big)).sum()), "children below": int((split & (child <= big)).sum())}


def _event_cases(stats_path, work):
    cases = []
    base = dict(P_base=P_BASE, seed=3, stats=stats_path, min_opacity=0.005)
    for P in (1, 2, 33, 4097, 100_000):
        for mss in (None, 20):
            c = dict(base, P=P, max_screen_size=mss, rng_seed=P + (mss or 0), zero_denom_every=7)
            grads, ms = _grads_and_scales(c)
            # C and S a few percent each: the top 8 % of the gradients, the scale threshold at the median of max scale
            c["max_grad"] = float(torch.quantile(grads.double(), 0.92)) if P > 1 else float(grads[0])
            c["extent"] = float(ms.median().double()) / 0.01
            cases.append(c)
    c0 = dict(base, P=100_000, max_screen_size=20, rng_seed=5)
    grads, ms = _grads_and_scales(c0)
    cases.append(dict(c0, max_grad=1e9, extent=float(ms.median().double()) / 0.01))           # C = S = 0
    cases.append(dict(c0, max_grad=0.0, extent=float(ms.median().double()) / 0.01))           # every row selected
    # thresholds met with equality: gradients exactly at max_grad, max scale exactly at percent_dense*extent
    k = int(torch.argsort(grads)[int(0.9 * len(grads))])
    j = int(torch.argsort(ms)[len(ms) // 2])
    extent = float(ms[j].double()) / 0.01
    assert np.float32(0.01 * extent) == np.float32(ms[j].item())
    for mss in (None, 20):
        cases.append(dict(c0, max_grad=float(grads[k].double()), extent=extent, max_screen_size=mss, rng_seed=7))
    # the world-space size prune inside the distribution: log-scales spread over 6 units, 0.1*extent at the 70th percentile of the max
    # scale (percent_dense*extent ten times lower, near the 30th), the top 20 % of the gradients selected.  max_screen_size 20 and its
    # None twin: the first must prune rows the second keeps.
    for mss in (20, None):
        c = dict(base, P=100_000, max_screen_size=mss, rng_seed=11, wide_scales=True)
        grads, ms = _grads_and_scales(c)
        c["max_grad"] = float(torch.quantile(grads.double(), 0.8))
        # 0.1*extent equal to the max scale of an unselected row: `>` keeps it, `>=` would not
        order = torch.argsort(ms).tolist()
        j = next(i for i in order[int(0.7 * len(order)):] if grads[i] < np.float32(c["max_grad"]))
        c["extent"] = float(ms[j].double()) / 0.1
        assert np.float32(0.1 * c["extent"]) == np.float32(ms[j].item())
        cases.append(c)
    # SH degree 0 (`--sh_degree 0`): _features_rest is [P, 0, 3]
    c = dict(base, P=4097, max_screen_size=20, rng_seed=13, sh_degree=0)
    grads, ms = _grads_and_scales(c)
    cases.append(dict(c, max_grad=float(torch.quantile(grads.double(), 0.92)), extent=float(ms.median().double()) / 0.01))
    # bench size: 3M Gaussians, statistics of two 1080p views
    c = dict(P_base=3_000_000, seed=9, P=3_000_000, stats=_stats_3m(work), min_opacity=0.005, max_screen_size=20, rng_seed=9)
    grads, ms = _grads_and_scales(c)
    cases.append(dict(c, max_grad=float(torch.quantile(grads[grads > 0].double(), 0.9)), extent=float(ms.median().double()) / 0.01))
    return cases


def test_densify_and_prune_bit_identical_to_reference(work, stats):
    cases = _event_cases(stats["path"], work)
    ours, tr = _run(work, "ours", "event", cases, "event")
    stock, _ = _run(work, "stock", "event", cases, "event")
    assert tr.get("densify_native") == len(cases), tr
    for c, o, s in zip(cases, ours, stock):
        label = {k: c[k] for k in ("P", "max_grad", "extent", "max_screen_size")}
        print("case", label, "rows", c["P"], "->", s["rows"])
        assert o["rows"] == s["rows"], label
        assert o["order"] == s["order"], label
        bad = [k for k in s["hash"] if o["hash"][k] != s["hash"][k]]
        for k in o["full"]:
            if not torch.equal(o["full"][k].view(torch.int32), s["full"][k].view(torch.int32)):
                d = o["full"][k].view(torch.int32) != s["full"][k].view(torch.int32)
                print(f"  {k}: {int(d.any(dim=tuple(range(1, d.dim()))).sum())} rows differ, first {d.nonzero()[:4].tolist()}")
        assert not bad, (label, bad)
        assert torch.equal(o["rng"], s["rng"]), label
        assert o["image_nonzero"] > 0 and torch.equal(o["image"].view(torch.int32), s["image"].view(torch.int32)), label
        after = [k for k in s["after_step"] if o["after_step"][k] != s["after_step"][k]]
        assert not after, (label, after)
    # the cases really cover clone, split, prune and the empty event
    rows = {(c["P"], c["max_grad"]): s["rows"] for c, s in zip(cases, stock) if not c.get("wide_scales")}
    assert rows[(100_000, 1e9)] < 100_000 and rows[(100_000, 0.0)] > 100_000
    (big, big_c), (none, none_c) = [(s["rows"], c) for c, s in zip(cases, stock) if c.get("wide_scales")]
    cover = _coverage(big_c)
    print("size-prune case", cover, "rows with max_screen_size 20:", big, "with None:", none)
    assert all(v > 0 for v in cover.values()), cover
    assert big < none


def _ply_count(path):
    with open(path, "rb") as f:
        for line in f:
            if line.startswith(b"element vertex"):
                return int(line.split()[-1])
    raise AssertionError(path)


def test_train_densify_prune_runs_unmodified_and_matches_the_stock_stack(work):
    from lightgaussian_b200.synth import make_cameras, make_scene, write_colmap_dataset
    # a 20 000-point SfM cloud: a handful of threshold decisions that flip with last-bit gradient differences stay a small share
    scene = make_scene(20000, sh_degree=3, seed=5, scale_mult=1.5)
    cams = make_cameras(24, 320, 240)
    gt = sh.render_ground_truth(scene["raw"], cams)
    data = os.path.join(work, "script", "data")
    write_colmap_dataset(data, list(zip(cams, gt)), n_points=20000)
    last = 600
    runs = {}
    for stack in ("ours", "stock"):
        out = os.path.join(work, f"tdp_{stack}")
        trace = os.path.join(work, f"tdp_{stack}.trace.json")
        sh.run(stack, ["train_densify_prune.py", "-s", data, "-m", out, "--eval", "-r", "1", "--port", str(PORT + (stack == "ours")),
                       "--iterations", str(last), "--densify_from_iter", "100", "--densification_interval", "100",
                       "--densify_until_iter", "550", "--opacity_reset_interval", "300", "--prune_iterations", "560",
                       "--position_lr_max_steps", str(last), "--test_iterations", "999999", "--save_iterations", str(last),
                       "--checkpoint_iterations", str(last)], trace=trace)
        runs[stack] = dict(out=out, trace=sh.read_trace(trace) if stack == "ours" else None)
    c = {s: sh.read_scalars(runs[s]["out"], "train_loss_patches/total_loss") for s in runs}
    steps = sorted(c["ours"])
    assert steps == sorted(c["stock"]) and steps[0] == 1
    co, cs = np.array([c["ours"][k] for k in steps]), np.array([c["stock"][k] for k in steps])
    assert abs(co[0] - cs[0]) <= 1e-6, (co[0], cs[0])
    win = lambda x: np.convolve(x, np.ones(20) / 20, mode="valid")  # noqa: E731
    rel = (win(co) - win(cs)) / win(cs)
    print(f"train_densify_prune smoothed (ours-stock)/stock in [{rel.min():+.3f}, {rel.max():+.3f}], tail ours {co[-50:].mean():.5f} "
          f"stock {cs[-50:].mean():.5f}")
    # the criteria of tests/test_gpu_scripts.py: our smoothed curve nowhere worse than the stock stack's by more than 3 %, tail within 3 %
    assert rel.max() <= 0.03, rel.max()
    assert abs(co[-50:].mean() - cs[-50:].mean()) <= 0.03 * cs[-50:].mean()
    # densify_and_prune at iterations 200, 300, 400, 500 (iteration > densify_from_iter, < densify_until_iter).  The importance
    # prune runs after them, at 560: the stock stack ranks by its racy significance counter (tests/test_gpu_scripts.py), so the two
    # stacks keep different survivors, and densifying after that would compare two different models.
    t = runs["ours"]["trace"]
    assert t.get("densify_native") == 4 and t.get("densify_stats_native", 0) >= 500, t
    counts = {s: _ply_count(os.path.join(runs[s]["out"], "point_cloud", f"iteration_{last}", "point_cloud.ply")) for s in runs}
    print("saved Gaussians", counts)
    assert abs(counts["ours"] - counts["stock"]) <= 0.02 * counts["stock"], counts
    test_idx = [k for k in range(len(cams)) if k % 8 == 0]
    p = {s: sh.psnr_of_leaves(sh.load_checkpoint_leaves(os.path.join(runs[s]["out"], f"chkpnt{last}.pth"))["leaves"], 3,
                              [cams[k] for k in test_idx], [gt[k] for k in test_idx]) for s in runs}
    print("held-out PSNR", p)
    assert p["ours"] >= 0.97 * p["stock"], p


def test_fused_adamw_updates_a_permuted_dense_parameter_bit_exactly():
    """GaussianModel.create_from_pcd builds _xyz from a transposed numpy array (strides (1, P)); train_densify_prune.py steps it
    before its first densification.  FusedAdamW must match torch.optim.AdamW on it, in place."""
    from lightgaussian_b200.optim import FusedAdamW
    g = torch.Generator().manual_seed(4)
    base = torch.randn(3, 2001, generator=g)
    grads = [torch.randn(3, 2001, generator=g) for _ in range(3)]
    ps = [torch.nn.Parameter(base.clone().cuda().t()) for _ in range(2)]
    assert not ps[0].is_contiguous()
    opts = [torch.optim.AdamW([ps[0]], lr=1e-2, eps=1e-15), FusedAdamW([ps[1]], lr=1e-2, eps=1e-15)]
    for gr in grads:
        for p, o in zip(ps, opts):
            p.grad = gr.cuda().t().contiguous()
            o.step()
    assert ps[1].stride() == (1, 2001)
    assert torch.equal(ps[0].detach().view(torch.int32), ps[1].detach().view(torch.int32))
    for k in ("exp_avg", "exp_avg_sq"):
        assert torch.equal(opts[0].state[ps[0]][k], opts[1].state[ps[1]][k])
