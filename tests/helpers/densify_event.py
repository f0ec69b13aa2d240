"""Run with a stack's PYTHONPATH (tests/scripts_harness.py): build the reference's GaussianModel on the states of
tests/helpers/densify_state.py, with the optimizer of its own training_setup, and run the class's add_densification_stats /
densify_and_prune -- the reference's torch code under the stock stack, the native one under ours.

  densify_event.py stats <cases.pt> <out.pt> [--sync-error]   accumulate the views of case 0, save accum / denom
  densify_event.py event <cases.pt> <out.pt>                  one densify_and_prune per case, one render of the result through the
                                                              stack's gaussian_renderer, then one optimizer step
"""
import hashlib
import os
import sys
from argparse import ArgumentParser

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import densify_state  # noqa: E402
from arguments import OptimizationParams, PipelineParams  # noqa: E402
import gaussian_renderer  # noqa: E402  (under our stack: FusedAdamW and the native densification are installed)
from scene.cameras import MiniCam  # noqa: E402
from scene.gaussian_model import GaussianModel  # noqa: E402
from lightgaussian_b200.synth import make_cameras  # noqa: E402  (numpy only; densify_state put the repository on the path)


def model(st):
    g = GaussianModel(3)
    for name, attr in densify_state.ATTR.items():
        setattr(g, attr, torch.nn.Parameter(st[name].cuda().requires_grad_(True)))
    g.spatial_lr_scale = 1.0
    parser = ArgumentParser()
    op = OptimizationParams(parser)
    g.training_setup(op.extract(parser.parse_args([])))
    g.xyz_gradient_accum, g.denom, g.max_radii2D = st["accum"].cuda(), st["denom"].cuda(), st["max_radii2D"].cuda()
    for group in g.optimizer.param_groups:
        n = group["name"]
        g.optimizer.state[group["params"][0]] = {"step": torch.tensor(densify_state.STEP), "exp_avg": st["m_" + n].cuda(),
                                                 "exp_avg_sq": st["v_" + n].cuda()}
    return g


def digest(t):
    return (tuple(t.shape), hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest())


def snapshot(g, full):
    opt = g.optimizer
    names = {id(grp["params"][0]): grp["name"] for grp in opt.param_groups}
    out = {"order": [names[id(p)] for p in opt.state], "hash": {}, "full": {}}
    for grp in opt.param_groups:
        n, p = grp["name"], grp["params"][0]
        st = opt.state[p]
        out["hash"][n] = digest(p)
        out["hash"]["m_" + n], out["hash"]["v_" + n] = digest(st["exp_avg"]), digest(st["exp_avg_sq"])
        out["hash"]["step_" + n] = float(st["step"])
        out["hash"]["keys_" + n] = sorted(st)
        if full:
            out["full"][n] = p.detach().cpu()
    for a in ("xyz_gradient_accum", "denom", "max_radii2D"):
        out["hash"][a] = digest(getattr(g, a))
    return out


mode, cases_path, out_path = sys.argv[1], sys.argv[2], sys.argv[3]
cases = torch.load(cases_path)
results = []
if mode == "stats":
    case = cases[0]
    g = model(densify_state.build(case))
    views = []
    for grad, filt in torch.load(case["views"]):
        vs = torch.zeros(grad.shape, device="cuda", requires_grad=True)
        vs.grad = grad.cuda()
        views.append((vs, filt.cuda()))
    torch.cuda.synchronize()
    if "--sync-error" in sys.argv:
        torch.cuda.set_sync_debug_mode("error")
    for vs, filt in views:
        g.add_densification_stats(vs, filt)
    torch.cuda.set_sync_debug_mode(0)
    results = {"accum": g.xyz_gradient_accum.cpu(), "denom": g.denom.cpu()}
else:
    for case in cases:
        g = model(densify_state.build(case))
        torch.manual_seed(case["rng_seed"])
        g.densify_and_prune(case["max_grad"], case["min_opacity"], case["extent"], case["max_screen_size"])
        res = snapshot(g, full=case["P"] <= 100_000)
        res["rng"] = torch.cuda.get_rng_state()
        res["rows"] = g._xyz.shape[0]
        # one view of the densified model through the stack's own renderer: the reference's extension, or our kernels
        c = make_cameras(4, 320, 240)[1]
        cam = MiniCam(c.image_width, c.image_height, c.FoVy, c.FoVx, c.znear, c.zfar, torch.from_numpy(c.world_view_transform).cuda(),
                      torch.from_numpy(c.full_proj_transform).cuda())
        parser = ArgumentParser()
        pipe = PipelineParams(parser).extract(parser.parse_args([]))
        img = gaussian_renderer.render(cam, g, pipe, torch.zeros(3, device="cuda"))["render"].detach()
        res["image"] = img.cpu()
        res["image_nonzero"] = int((img != 0).sum())
        for grp in g.optimizer.param_groups:
            p = grp["params"][0]
            p.grad = torch.sin(p.detach() * 7.0) * 1e-3
        g.optimizer.step()
        res["after_step"] = snapshot(g, full=False)["hash"]
        results.append(res)
        del g
        torch.cuda.empty_cache()
torch.save(results, out_path)
print("done", mode, len(results))
