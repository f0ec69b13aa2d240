"""Time one densify_and_prune event and one add_densification_stats call at 3M Gaussians: the native functions of
lightgaussian_b200/densify.py against the reference's own GaussianModel methods (torch code, torch.optim.AdamW state), in one process,
alternating rounds, CUDA events, warm-up first.  Prints the card name and power limit with the numbers.

    python scripts/time_densify.py [--rounds 5]

Needs the staged reference tree (oracle/_ref/stock, see oracle/stage_reference.py)."""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFDIR = os.path.join(ROOT, "oracle", "_ref", "stock")
sys.path[:0] = [REFDIR, os.path.join(REFDIR, "shims"), os.path.join(REFDIR, "LightGaussian"), ROOT, os.path.join(ROOT, "tests", "helpers")]

from arguments import OptimizationParams  # noqa: E402
from scene.gaussian_model import GaussianModel  # noqa: E402

import densify_state  # noqa: E402
from lightgaussian_b200 import densify  # noqa: E402
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params  # noqa: E402
from lightgaussian_b200.renderer import render  # noqa: E402
from lightgaussian_b200.synth import make_cameras  # noqa: E402

P = 3_000_000
CASE = dict(P_base=P, seed=9, P=P, stats=None)
MAX_GRAD, MIN_OPACITY, EXTENT, MAX_SCREEN = 3.6e-4, 0.005, 0.9, 20


def model(st):
    g = GaussianModel(3)
    for name, attr in densify_state.ATTR.items():
        setattr(g, attr, torch.nn.Parameter(st[name].clone().requires_grad_(True)))
    g.spatial_lr_scale = 1.0
    parser = argparse.ArgumentParser()
    op = OptimizationParams(parser)
    g.training_setup(op.extract(parser.parse_args([])))
    g.xyz_gradient_accum, g.denom, g.max_radii2D = st["accum"].clone(), st["denom"].clone(), st["max_radii2D"].clone()
    for group in g.optimizer.param_groups:
        n = group["name"]
        g.optimizer.state[group["params"][0]] = {"step": torch.tensor(densify_state.STEP), "exp_avg": st["m_" + n].clone(),
                                                 "exp_avg_sq": st["v_" + n].clone()}
    return g


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU:", smi.stdout.strip() or torch.cuda.get_device_name(0))
    st = {k: v.cuda() for k, v in densify_state.build(CASE).items()}

    # statistics of one 1080p view of the same Gaussians (render + backward through our renderer)
    pc = GaussianParams({densify_state.RAW[n]: st[n].cpu().numpy() for n in densify_state.ATTR}, 3, "cuda")
    pkg = render(TorchCamera(make_cameras(1, 1920, 1080)[0], "cuda"), pc, pipeline_params(), torch.zeros(3, device="cuda"))
    pkg["render"].mean().backward()
    vs, vis = pkg["viewspace_points"], pkg["visibility_filter"]
    print(f"P = {P}, visible in the 1080p view: {int(vis.sum())}")
    del pc, pkg

    impl = {"reference": lambda g: GaussianModel.densify_and_prune(g, MAX_GRAD, MIN_OPACITY, EXTENT, MAX_SCREEN),
            "native": lambda g: densify.densify_and_prune(g, MAX_GRAD, MIN_OPACITY, EXTENT, MAX_SCREEN)}
    stats = {"reference": lambda g: GaussianModel.add_densification_stats(g, vs, vis),
             "native": lambda g: densify.add_densification_stats(g, vs, vis)}
    times = {k: {"event": [], "stats": []} for k in impl}
    rows = {}
    for rnd in range(args.rounds + 1):                       # round 0 is the warm-up
        for name in (("reference", "native") if rnd % 2 == 0 else ("native", "reference")):
            g = model(st)
            t_stats = sum(timed(lambda: stats[name](g)) for _ in range(10)) / 10
            g.xyz_gradient_accum.copy_(st["accum"])
            g.denom.copy_(st["denom"])
            torch.manual_seed(rnd)
            t_event = timed(lambda: impl[name](g))
            rows[name] = g._xyz.shape[0]
            if rnd:
                times[name]["stats"].append(t_stats)
                times[name]["event"].append(t_event)
            del g
            torch.cuda.empty_cache()
    assert rows["native"] == rows["reference"], rows
    print(f"rows after the event: {rows['native']}")
    for what in ("event", "stats"):
        r, n = sorted(times["reference"][what]), sorted(times["native"][what])
        label = "densify_and_prune" if what == "event" else "add_densification_stats"
        print(f"{label}: reference median {r[len(r) // 2]:.3f} ms (min {r[0]:.3f}), native median {n[len(n) // 2]:.3f} ms "
              f"(min {n[0]:.3f}), speed-up {r[len(r) // 2] / n[len(n) // 2]:.1f}x")


if __name__ == "__main__":
    main()
